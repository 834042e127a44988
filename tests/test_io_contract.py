"""On-disk contract around the path: official-Swin key/row conversion, checkpoint ingestion, KITTI PNG values."""
import numpy as np
import pytest
import torch

from diffusiondepth_b200 import io as ddio
from diffusiondepth_b200.model.backbone.convert_ckpt import swin_convert
from oracle import ref_import


def _official_like(C=8):
    g = torch.Generator().manual_seed(0)
    r = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    return {"patch_embed.proj.weight": r(C, 3, 4, 4), "patch_embed.norm.weight": r(C),
            "layers.0.blocks.0.attn.qkv.weight": r(3 * C, C), "layers.0.blocks.0.attn.relative_position_bias_table": r(169, 2),
            "layers.0.blocks.0.mlp.fc1.weight": r(4 * C, C), "layers.0.blocks.0.mlp.fc2.bias": r(C),
            "layers.0.blocks.0.norm1.weight": r(C), "layers.0.downsample.reduction.weight": r(2 * C, 4 * C),
            "layers.0.downsample.norm.weight": r(4 * C), "layers.0.downsample.norm.bias": r(4 * C),
            "norm.weight": r(8 * C), "head.weight": r(10, 8 * C)}


def test_swin_convert_names_and_merge_order():
    src = _official_like()
    out = swin_convert(src)
    assert "head.weight" not in out
    for k in ("patch_embed.projection.weight", "stages.0.blocks.0.attn.w_msa.qkv.weight",
              "stages.0.blocks.0.attn.w_msa.relative_position_bias_table", "stages.0.blocks.0.ffn.layers.0.0.weight",
              "stages.0.blocks.0.ffn.layers.1.bias", "stages.0.blocks.0.norm1.weight",
              "stages.0.downsample.reduction.weight", "stages.0.downsample.norm.bias", "norm.weight"):
        assert k in out, k
    # semantic check of the permutation: official concat [x0,x1,x2,x3] (positions (0,0),(1,0),(0,1),(1,1)) vs unfold
    C = 8
    x = torch.randn(1, C, 4, 6)
    x0, x1, x2, x3 = x[:, :, 0::2, 0::2], x[:, :, 1::2, 0::2], x[:, :, 0::2, 1::2], x[:, :, 1::2, 1::2]
    official = torch.cat([x0, x1, x2, x3], 1).flatten(2).transpose(1, 2)          # [1, L, 4C]
    unfold = torch.nn.functional.unfold(x, 2, stride=2).transpose(1, 2)          # [1, L, 4C] channel-major
    w = src["layers.0.downsample.reduction.weight"]
    assert torch.allclose(official @ w.t(), unfold @ out["stages.0.downsample.reduction.weight"].t(), atol=1e-5)
    g = src["layers.0.downsample.norm.weight"]
    assert torch.allclose((official * g).sum(-1), (unfold * out["stages.0.downsample.norm.weight"]).sum(-1), atol=1e-5)


def test_swin_convert_matches_reference():
    """Against the reference's own swin_convert on the same input (outputs stored by oracle/make_ref_fixtures.py)."""
    import dd_helpers
    ref = dd_helpers.ref_fixtures()
    b = swin_convert(dict(_official_like()))
    assert list(b) == [str(k) for k in ref["convert_keys"]]
    for i, k in enumerate(b):
        assert torch.equal(torch.from_numpy(ref[f"convert_{i}"]), b[k]), k


def test_checkpoint_ingestion_and_png(tmp_path):
    import dd_helpers
    m = dd_helpers.build_mirror("res18", 5)
    path = tmp_path / "model_00001.pt"
    torch.save({"net": {"module." + k: v for k, v in m.state_dict().items()}, "args": {"inference_steps": 5}}, path)
    args = ddio.load_reference_checkpoint(m, str(path))
    assert args == {"inference_steps": 5}
    sd = m.state_dict()
    sd.pop("depth_head.model.pred.0.weight")
    torch.save({"net": sd}, path)
    with pytest.raises(KeyError, match="Missing keys"):
        ddio.load_reference_checkpoint(m, str(path))
    pred = torch.tensor([[[[0.5, -1.0], [80.0, 255.99]]]])
    png = ddio.depth_to_kitti_png(pred)
    assert png.dtype == np.uint16 and png.tolist() == [[128, 0], [20480, 65533]]
    ddio.save_kitti_png(pred, str(tmp_path / "x.png"))
    from PIL import Image
    assert np.array(Image.open(tmp_path / "x.png")).tolist() == png.tolist()
