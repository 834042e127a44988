"""TEST INFRASTRUCTURE ONLY — gradients of the REAL reference's sampling loop and decoder: `CNNDDIMPipiline` (head
ddim_depth_estimate_res_swin_addHAHI.py:244-303) over its `ScheduledCNNRefine` (Swin :336-382, Res
ddim_depth_estimate_res.py:301-344), then `DeepDepthTransformWithUpsampling.inv_t` (ops/depth_transform.py:33-35) with the
decoder in eval mode, under torch.autograd on CPU in the reference's own fp32.  The initial latent is injected as
oracle/reference_runner.py does.  Loss L = sum(depth * d_depth) + sum(latent * d_latent).  Stored in
tests/golden/g_loop_grads.npz with the layout of g_denoiser_grads.npz.  Run in the build container:
    python -m oracle.make_loop_grads"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import configs  # noqa: E402
from oracle.make_denoiser_grads import SAMPLES, checksum, denoiser_state, sample_index  # noqa: E402,F401

OUT = os.path.join(ROOT, "tests", "golden", "g_loop_grads.npz")
STEPS = 3
# name -> (variant, batch, latent (h, w), condition (h, w))
CASES = {
    "swin_19x27": ("swin", 3, (19, 27), (10, 14)),
    "swin_35x53": ("swin", 3, (35, 53), (18, 27)),
    "res_19x27": ("res", 3, (19, 27), (19, 27)),
    "res_35x53": ("res", 3, (35, 53), (35, 53)),
}


def decoder_state(seed=configs.SEED_WEIGHTS):
    """The mirror's DeepDepthTransformWithUpsampling (same keys as the reference's) under a fixed seed, trainedify'd so
    that the decoder's BatchNorm statistics are non-trivial: keys `depth_transform.*` (relative to `depth_head.`)."""
    from diffusiondepth_b200.model.ops.depth_transform import DeepDepthTransformWithUpsampling
    torch.manual_seed(seed + 1)
    m = configs.trainedify(DeepDepthTransformWithUpsampling(16, 1e-6))
    return {"depth_transform." + k: v.detach().clone() for k, v in m.state_dict().items()
            if not k.endswith("num_batches_tracked")}


def loop_state(variant):
    sd = denoiser_state(variant)
    sd.update(decoder_state())
    return sd


def case_inputs(name):
    """(variant, state_dict, cond, noise, d_depth, d_latent) of a case, all fp32 CPU."""
    variant, B, (h, w), (hc, wc) = CASES[name]
    sd = loop_state(variant)
    g = torch.Generator().manual_seed(2025)
    cond = torch.randn(B, 256, hc, wc, generator=g).abs()  # the FPN's condition map is post-ReLU
    noise = torch.randn(B, 16, h, w, generator=g)
    d_depth = torch.randn(B, 1, 2 * h, 2 * w, generator=g) * (1.0 / (B * 4 * h * w))  # the scale of an L1 / L2 gradient
    d_latent = torch.randn(B, 16, h, w, generator=g) * (2.0 / (B * 16 * h * w))
    return variant, sd, cond, noise, d_depth, d_latent


def reference_grads(name):
    from oracle import ref_import
    from oracle.reference_runner import _inject_first_randn
    variant, sd, cond, noise, d_depth, d_latent = case_inputs(name)
    mods = ref_import.reference_modules()
    head = mods.head_swin if variant == "swin" else mods.head_res
    model = head.ScheduledCNNRefine(256, 16)
    model.load_state_dict({k[len("model."):]: v for k, v in sd.items() if k.startswith("model.")}, strict=True)
    codec = mods.depth_transform.DeepDepthTransformWithUpsampling(16, 1e-6)
    codec.load_state_dict({k[len("depth_transform."):]: v for k, v in sd.items() if k.startswith("depth_transform.")},
                          strict=False)
    codec.eval()
    pipe = head.CNNDDIMPipiline(model, mods.scheduling_ddim.DDIMScheduler(num_train_timesteps=1000, clip_sample=False))
    cond = cond.clone().requires_grad_(True)
    with _inject_first_randn(noise) as st:
        latent, = pipe(batch_size=noise.shape[0], device=noise.device, dtype=noise.dtype, shape=noise.shape[-3:],
                       input_args=(cond, None, None, None), num_inference_steps=STEPS, return_dict=False)
    assert st["used"]
    depth = codec.inv_t(latent)
    ((depth * d_depth).sum() + (latent * d_latent).sum()).backward()
    grads = {"d_cond": cond.grad}
    for k, p in model.named_parameters():
        grads["model." + k] = p.grad
    for k, p in codec.conv_inv_transform.named_parameters():
        grads["depth_transform.conv_inv_transform." + k] = p.grad
    return variant, sd, grads


def main():
    torch.set_num_threads(os.cpu_count() or 8)
    arrays = {}
    for name in CASES:
        variant, sd, grads = reference_grads(name)
        _, _, cond, noise, d_depth, d_latent = case_inputs(name)
        arrays[name + "/weight_checksum"] = np.float64(checksum(*sd.values()))
        arrays[name + "/input_checksum"] = np.float64(checksum(cond, noise, d_depth, d_latent))
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
