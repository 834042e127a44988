"""TEST INFRASTRUCTURE ONLY — the REAL reference Swin-L backbone (src/model/backbone/swin.py, the
`swin_large_naive_nopretrain` architecture) in training mode (`.train()`, as src/main.py trains), on CPU in the
reference's own fp32, with stochastic depth on: `drop_path_rate = RATE`, so the rates run linspace(0, RATE, 24) over
the 24 blocks and both residual branches of every block but the first draw one mmcv DropPath mask per call from the
global CPU generator, seeded with case_seed(name) before the forward.  B = 3, at 70 x 106 (the patch embedding pads,
odd grids 18x27 .. 3x4) and at 64 x 96.  The weights are the trained-like mirror state (oracle.configs.trainedify).

RATE is 0.9, not 1.0: at 1.0 the last block has keep = 0 and mmcv's x.div(keep) * floor(keep + U) is NaN.

The in-repo mmcv stub's DropPath draws with `bernoulli_`, which consumes the generator differently from mmcv 1.x's
`drop_path` (cnn/bricks/drop.py: torch.rand, then floor).  This script leaves the stub as it is and gives each of the
reference's DropPath modules mmcv's own forward (`mmcv_drop_path`) for the run.

Stored per case:
  input_checksum, weight_checksum
  masks            [draws][B] the masks the DropPath modules drew, in call order (stage, block, attention then FFN)
  rng_state        the CPU generator's state after the forward (uint8)
  feats/i          the four stage outputs, sub-sampled (sample_index) + their checksum and absmax
Written to tests/golden/g_swin_drop_path.npz.  Run in the build container:
    python -m oracle.make_swin_drop_path"""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_import  # noqa: E402
from oracle.make_denoiser_grads import checksum, sample_index  # noqa: E402
from oracle.make_producer_train import mirror_state  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "g_swin_drop_path.npz")
B = 3
RATE = 0.9
SEED = 2024
FAMILY = "swinl"
CASES = {"swin_70x106": (70, 106), "swin_64x96": (64, 96)}
SWIN_L = dict(pretrain_img_size=224, in_channels=3, embed_dims=192, patch_size=4, window_size=7, mlp_ratio=4,
              depths=(2, 2, 18, 2), num_heads=(6, 12, 24, 48), strides=(4, 2, 2, 2), out_indices=(0, 1, 2, 3),
              pretrain_style="official", pretrained=None)


def mmcv_drop_path(module, x):
    """mmcv 1.x cnn/bricks/drop.py `drop_path(x, module.drop_prob, module.training)`."""
    if module.drop_prob == 0. or not module.training:
        return x
    keep_prob = 1 - module.drop_prob
    shape = (x.shape[0],) + (1,) * (x.ndim - 1)
    random_tensor = keep_prob + torch.rand(shape, dtype=x.dtype, device=x.device)
    return x.div(keep_prob) * random_tensor.floor()


def case_seed(name):
    return SEED + list(CASES).index(name)


def case_rgb(name):
    H, W = CASES[name]
    return torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(H * 1000 + W))


def backbone_state():
    """The trained-like mirror Swin-L's state dict, keys relative to the backbone."""
    p = "depth_backbone."
    return {k[len(p):]: v for k, v in mirror_state(FAMILY).items() if k.startswith(p)}


def reference_case(name, sd):
    ref_import._activate()
    import importlib
    swin = importlib.import_module("model.backbone.swin")
    net = swin.SwinTransformer(drop_path_rate=RATE, **SWIN_L)
    net.load_state_dict(sd, strict=True)
    net.train()
    rgb = case_rgb(name)
    drawn, hooks = [], []
    for m in net.modules():
        if type(m).__name__ == "DropPath":
            m.forward = types.MethodType(mmcv_drop_path, m)
        if type(m).__name__ == "DropPath" and m.drop_prob > 0:
            hooks.append(m.register_forward_hook(lambda mod, a, o: drawn.append(o.flatten(1).abs().amax(1) > 0)))
    torch.manual_seed(case_seed(name))
    try:
        with torch.no_grad():
            feats = net(rgb)
    finally:
        for h in hooks:
            h.remove()
    masks = torch.stack(drawn).to(torch.uint8)
    out = {name + "/input_checksum": np.float64(checksum(rgb)),
           name + "/weight_checksum": np.float64(checksum(*[v for v in sd.values() if v.is_floating_point()])),
           name + "/masks": masks.numpy(),
           name + "/rng_state": torch.get_rng_state().numpy()}
    for i, f in enumerate(feats):
        flat = f.reshape(-1)
        out[f"{name}/feats/{i}/checksum"] = np.float64(checksum(f))
        out[f"{name}/feats/{i}/absmax"] = np.float64(flat.abs().max())
        out[f"{name}/feats/{i}/values"] = flat[torch.from_numpy(sample_index(flat.numel()))].numpy()
    print(f"[{name}] {masks.shape[0]} draws, {int(masks.sum())} of {masks.numel()} kept; feats absmax "
          + " ".join(f"{float(out[f'{name}/feats/{i}/absmax']):.3g}" for i in range(4)), flush=True)
    return out


def main():
    torch.set_num_threads(os.cpu_count() or 8)
    sd = backbone_state()
    arrays = {}
    for name in CASES:
        arrays.update(reference_case(name, sd))
    np.savez_compressed(OUT, **arrays)
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1e3:.0f} kB)")


if __name__ == "__main__":
    main()
