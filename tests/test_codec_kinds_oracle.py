"""The reference's other learned depth codecs in the mirror (CPU): module layout and torch `t` / `inv_t` against the
real reference (live, where its sources exist), the fp64 restatement (oracle/restate_codecs.py) against the reference,
and the head-level refusals that need no engine."""
import os

import pytest
import torch

from diffusiondepth_b200._cabi import EngineError
from diffusiondepth_b200.model.registry import DEPTH_TRANSFORM, HEADS
from oracle import ref_import, restate_codecs

KINDS = {"DeepDepthTransformWithUpsampling1x1": 1, "DeepDepthTransformWithUpsamplingX4": 2, "DeepDepthTransform": 3}
live = pytest.mark.skipif(not ref_import.available(), reason="reference sources not present")


def _head(kind_name, head="DDIMDepthEstimate_Swin_ADDHAHI", **cfg):
    return HEADS.build(dict(type=head, in_channels=[64, 128, 256, 512], inference_steps=3, num_train_timesteps=1000,
                            depth_feature_dim=16, loss_cfgs=[], init_cfg=None,
                            depth_transform_cfg=dict(type=kind_name, **cfg)))


def test_registry_has_all_six_transforms():
    for n in ("DeepDepthTransformWithUpsampling", "DeepDepthTransformWithUpsampling1x1",
              "DeepDepthTransformWithUpsamplingX4", "DeepDepthTransform", "ReciprocalDepthTransform",
              "ReciprocalDepthTransformII"):
        assert DEPTH_TRANSFORM.get(n) is not None, n


@pytest.mark.parametrize("name", sorted(KINDS))
def test_latent_geometry(name):
    m = DEPTH_TRANSFORM.build(dict(type=name)).eval()
    assert m.ENGINE_KIND == KINDS[name]
    for hw in ((1, 1), (2, 3), (17, 23), (352, 1216)):
        with torch.no_grad():
            lat = m.t(torch.rand(1, 1, *hw))
            dec = m.inv_t(torch.randn(1, 16, *lat.shape[-2:]))
        assert tuple(lat.shape[-2:]) == m.latent_hw(hw)
        assert tuple(dec.shape[-2:]) == (m.UP * lat.shape[-2], m.UP * lat.shape[-1])


@live
@pytest.mark.parametrize("name", sorted(KINDS))
def test_codec_matches_reference(name):
    """state_dict keys and shapes in order; torch t / inv_t equal to the reference's; the fp64 restatement within fp32
    rounding of the reference, with trained-like BatchNorms, at an even and an odd size."""
    ref = ref_import.reference_modules()
    torch.manual_seed(3)
    r = restate_codecs.trainedify_codec(getattr(ref.depth_transform, name)(hidden=16), KINDS[name]).eval()
    m = DEPTH_TRANSFORM.build(dict(type=name)).eval()
    assert [(k, tuple(v.shape)) for k, v in r.state_dict().items()] == \
        [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    m.load_state_dict(r.state_dict())
    sd = {"depth_head.depth_transform." + k: v.double() for k, v in r.state_dict().items()}
    worst = {}
    for hw in ((20, 28), (17, 23)):
        depth = torch.rand(2, 1, *hw) * 8
        latent = torch.randn(2, 16, *m.latent_hw(hw))
        with torch.no_grad():
            t_ref, t_m = r.t(depth), m.t(depth)
            z_ref = r.conv_inv_transform[:-1](latent)
            assert torch.equal(t_ref, t_m) and torch.equal(r.inv_t(latent), m.inv_t(latent))
        t64 = restate_codecs.encode(sd, depth.double(), KINDS[name])
        z64 = restate_codecs.decode_logits(sd, latent.double(), KINDS[name])
        worst[hw] = ((t_ref.double() - t64).abs().max().item(),
                     (z_ref.double() - z64).abs().max().item() / max(1.0, z64.abs().max().item()))
        assert worst[hw][0] < 2e-4 and worst[hw][1] < 1e-5, worst  # the reference's own fp32 rounding
    print(f"{name}: reference fp32 vs restatement fp64 (|dt|, |dz| / max(1, max|z|)): {worst}")


@live
@pytest.mark.parametrize("name", sorted(KINDS))
def test_head_codec_keys_match_reference(name):
    """A head built with each depth_transform_cfg carries the reference codec's keys under `depth_transform.`."""
    ref = ref_import.reference_modules()
    r = getattr(ref.depth_transform, name)(hidden=16)
    h = _head(name)
    got = {k: tuple(v.shape) for k, v in h.state_dict().items() if k.startswith("depth_transform.")}
    assert got == {"depth_transform." + k: tuple(v.shape) for k, v in r.state_dict().items()}


def test_unsupported_pairings_and_hidden_raise():
    res = _head("DeepDepthTransformWithUpsamplingX4", head="DDIMDepthEstimate_Res")
    with pytest.raises(EngineError, match=r"\(10, 14\).*\(5, 7\)"):
        res._engine(1, (5, 7), (10, 14), "cpu")  # refused before any engine is created
    full = _head("DeepDepthTransform", head="DDIMDepthEstimate_Res")
    with pytest.raises(EngineError, match="without resampling"):
        full._engine(1, (20, 28), (10, 14), "cpu")
    with pytest.raises(EngineError, match="hidden=8"):
        _head("DeepDepthTransformWithUpsamplingX4", hidden=8)._codec_kind()
    with pytest.raises(EngineError, match="no engine codec"):
        _head("ReciprocalDepthTransformII")._codec_kind()


@pytest.mark.parametrize("flag", ["grad_through_loop", "grad_through_encoder", "codec_train_bn"])
def test_codec_training_is_refused_before_engine_work(flag):
    h = _head("DeepDepthTransformWithUpsamplingX4")
    setattr(h, flag, True)
    h.train()
    fp = [torch.zeros(1, c, 4, 4) for c in (64, 128, 256, 512)]
    with pytest.raises(EngineError, match="DeepDepthTransformWithUpsamplingX4"):
        h(fp, None, None, gt_depth_map=torch.zeros(1, 1, 16, 16))
    assert len(h._engines) == 0


def test_restatement_matches_reference_golden():
    """oracle/restate_codecs.py in fp64 against the real reference's `t` / `inv_t` stored in g_codec_kinds.npz
    (oracle/make_codec_kinds.py), every codec at an even and an odd size, margins printed."""
    import numpy as np
    from oracle import make_codec_kinds as mk
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "g_codec_kinds.npz"))
    for kind in mk.NAMES:
        sd = {"depth_head.depth_transform." + k: v.double() for k, v in mk.mirror_codec(kind).state_dict().items()}
        for hw in mk.CODEC_SIZES:
            depth, latent = mk.codec_inputs(kind, hw)
            t_ref = torch.from_numpy(g[f"codec{kind}_{hw[0]}x{hw[1]}_t"]).double()
            z_ref = torch.from_numpy(g[f"codec{kind}_{hw[0]}x{hw[1]}_z"]).double()
            dt = (restate_codecs.encode(sd, depth.double(), kind) - t_ref).abs().max().item()
            dz = (restate_codecs.decode_logits(sd, latent.double(), kind) - z_ref).abs().max().item() / \
                max(1.0, z_ref.abs().max().item())
            print(f"{mk.NAMES[kind]} {hw}: fp64 restatement vs reference golden |dt| {dt:.2e}, |dz| rel {dz:.2e}")
            assert dt < 2e-4 and dz < 1e-5  # the reference's own fp32 rounding
