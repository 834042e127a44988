"""TEST INFRASTRUCTURE ONLY — gradients of the REAL reference's `ScheduledCNNRefine` (Swin: head
ddim_depth_estimate_res_swin_addHAHI.py:336-382, Res: ddim_depth_estimate_res.py:301-344) under torch.autograd on CPU, in
the reference's own fp32, stored in tests/golden/g_denoiser_grads.npz.  Run in the build container:
    python -m oracle.make_denoiser_grads

Weights and inputs are regenerated from seeds by `case_inputs` (which needs no reference), so the golden holds only t,
checksums and the gradients: small tensors in full, large ones at a fixed set of sampled indices, plus max |g| of each.
Weights are in the trained-like regime (`oracle.configs.trainedify`: GroupNorm gamma != 1, beta != 0)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import configs  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "g_denoiser_grads.npz")
SAMPLES = 1024  # sampled entries per large gradient
# name -> (variant, batch, latent (h, w), condition (h, w), t per image: a repeated t shares a time-embedding row)
CASES = {
    "swin_19x27": ("swin", 3, (19, 27), (10, 14), (417, 417, 12)),
    "swin_35x53": ("swin", 3, (35, 53), (18, 27), (999, 3, 999)),
    "res_19x27": ("res", 3, (19, 27), (19, 27), (417, 417, 12)),
    "res_35x53": ("res", 3, (35, 53), (35, 53), (999, 3, 999)),
}


def denoiser_state(variant, seed=configs.SEED_WEIGHTS):
    """The mirror's ScheduledCNNRefine (same keys as the reference's) under a fixed seed, then trainedify'd: a state_dict
    with keys `model.*` (relative to `depth_head.`)."""
    from diffusiondepth_b200.model.head._ddim_head import ScheduledCNNRefine
    torch.manual_seed(seed)
    m = configs.trainedify(ScheduledCNNRefine(256, 16, with_fuse=variant == "swin"))
    return {"model." + k: v.detach().clone() for k, v in m.state_dict().items()}


def case_inputs(name):
    """(variant, state_dict, noisy, cond, t LongTensor [B], d_eps) of a case, all fp32 CPU."""
    variant, B, (h, w), (hc, wc), t = CASES[name]
    sd = denoiser_state(variant)
    g = torch.Generator().manual_seed(2024)
    noisy = torch.randn(B, 16, h, w, generator=g)
    cond = torch.randn(B, 256, hc, wc, generator=g).abs()  # the FPN's condition map is post-ReLU
    d_eps = torch.randn(B, 16, h, w, generator=g) * (2.0 / (B * 16 * h * w))  # the scale of an MSE loss's gradient
    return variant, sd, noisy, cond, torch.tensor(t, dtype=torch.long), d_eps


def checksum(*tensors):
    return float(sum(t.double().abs().sum() for t in tensors))


def sample_index(n):
    return np.sort(np.random.default_rng(0).choice(n, min(n, SAMPLES), replace=False)).astype(np.int64)


def reference_grads(name):
    """Run the real reference's module: eps = model(noisy, t, cond, None, None, None); (eps * d_eps).sum().backward()."""
    from oracle import ref_import
    variant, sd, noisy, cond, t, d_eps = case_inputs(name)
    mods = ref_import.reference_modules()
    cls = (mods.head_swin if variant == "swin" else mods.head_res).ScheduledCNNRefine
    ref = cls(256, 16)
    ref.load_state_dict({k[len("model."):]: v for k, v in sd.items()}, strict=True)
    noisy = noisy.clone().requires_grad_(True)
    cond = cond.clone().requires_grad_(True)
    eps = ref(noisy, t, cond, None, None, None)
    (eps * d_eps).sum().backward()
    grads = {"d_noisy": noisy.grad, "d_cond": cond.grad}
    for k, p in ref.named_parameters():
        grads["model." + k] = p.grad
    return variant, sd, grads


def main():
    torch.set_num_threads(os.cpu_count() or 8)
    arrays = {}
    for name in CASES:
        variant, sd, grads = reference_grads(name)
        _, _, noisy, cond, t, d_eps = case_inputs(name)
        arrays[name + "/t"] = t.numpy()
        arrays[name + "/weight_checksum"] = np.float64(checksum(*sd.values()))
        arrays[name + "/input_checksum"] = np.float64(checksum(noisy, cond, d_eps))
        for k, gr in grads.items():
            flat = gr.detach().reshape(-1)
            arrays[f"{name}/{k}/absmax"] = np.float64(flat.abs().max())
            if flat.numel() <= SAMPLES:
                arrays[f"{name}/{k}/values"] = flat.numpy()
            else:
                idx = sample_index(flat.numel())
                arrays[f"{name}/{k}/index"] = idx
                arrays[f"{name}/{k}/values"] = flat[torch.from_numpy(idx)].numpy()
        print(f"[{name}] {len(grads)} gradients, max|d_cond| {grads['d_cond'].abs().max():.3e}", flush=True)
    np.savez_compressed(OUT, **arrays)
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1e3:.0f} kB)")


if __name__ == "__main__":
    main()
