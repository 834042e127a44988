"""TEST INFRASTRUCTURE ONLY — the REAL reference's depth codec `DeepDepthTransformWithUpsampling`
(ops/depth_transform.py:10-35, conv_bn_relu = common.py:45-60) in training mode (`.train()`, as src/main.py:181 trains),
on CPU in the reference's own fp32:
  codec/*      inv_t and t outputs; the decoder's and the encoder's running statistics after one call; the decoder's
               after a *Vis head's T + 1 calls (the final map's, then steps 1 .. T: ..._swin_addHAHI_vis.py:146-149);
               autograd gradients of sum(inv_t(latent) * d_depth) with respect to the latent and the decoder parameters;
  <loop case>/ gradients of the sampling loop + decoder as oracle/make_loop_grads.py stores them (T = 3, B = 3), with the
               codec in training mode.
Stored in tests/golden/g_codec_train.npz.  Run in the build container:
    python -m oracle.make_codec_train"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import make_loop_grads as mlg  # noqa: E402
from oracle.make_denoiser_grads import SAMPLES, checksum, sample_index  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "g_codec_train.npz")
B, HW, VIS_T = 2, (13, 21), 3
LOOP_CASES = ("swin_19x27", "res_19x27")
BN_KEYS = {"dec": "conv_inv_transform.1", "enc1": "conv_transform.0.1", "enc2": "conv_transform.1.1"}


def codec_state():
    """The codec's parameters and running statistics (keys relative to `depth_transform.`), as the loop goldens use."""
    return {k[len("depth_transform."):]: v for k, v in mlg.decoder_state().items()}


def codec_inputs():
    """(latent [B,16,h,w], depth [B,1,2h,2w], d_depth [B,1,2h,2w], Vis latents [T][B,16,h,w]), fp32 CPU."""
    g = torch.Generator().manual_seed(4711)
    h, w = HW
    latent = torch.randn(B, 16, h, w, generator=g)
    depth = torch.rand(B, 1, 2 * h, 2 * w, generator=g) * 80 + 0.5
    d_depth = torch.randn(B, 1, 2 * h, 2 * w, generator=g) * (1.0 / (B * 4 * h * w))
    vis = [torch.randn(B, 16, h, w, generator=g) for _ in range(VIS_T)]
    return latent, depth, d_depth, vis


def _reference_codec():
    from oracle import ref_import
    codec = ref_import.reference_modules().depth_transform.DeepDepthTransformWithUpsampling(16, 1e-6)
    codec.load_state_dict(codec_state(), strict=False)  # num_batches_tracked starts at 0
    return codec.train()


def _running(codec, name):
    bn = codec.get_submodule(BN_KEYS[name])
    return {"running_mean": bn.running_mean, "running_var": bn.running_var,
            "num_batches_tracked": bn.num_batches_tracked}


def codec_arrays():
    latent, depth, d_depth, vis = codec_inputs()
    out = {"codec/weight_checksum": np.float64(checksum(*codec_state().values())),
           "codec/input_checksum": np.float64(checksum(latent, depth, d_depth, *vis))}
    codec = _reference_codec()
    x = latent.clone().requires_grad_(True)
    inv = codec.inv_t(x)
    (inv * d_depth).sum().backward()
    out["codec/inv_t"] = inv.detach().numpy()
    out["codec/grad/d_latent"] = x.grad.numpy()
    for k, p in codec.conv_inv_transform.named_parameters():
        out["codec/grad/conv_inv_transform." + k] = p.grad.numpy()
    for k, v in _running(codec, "dec").items():
        out["codec/after_decode/dec/" + k] = v.numpy()
    codec = _reference_codec()
    with torch.no_grad():
        out["codec/t"] = codec.t(depth).numpy()
    for name in ("enc1", "enc2"):
        for k, v in _running(codec, name).items():
            out[f"codec/after_encode/{name}/{k}"] = v.numpy()
    codec = _reference_codec()
    with torch.no_grad():
        for lat in [vis[-1]] + vis:
            codec.inv_t(lat)
    for k, v in _running(codec, "dec").items():
        out["codec/after_vis/dec/" + k] = v.numpy()
    return out


def loop_grads(name):
    """make_loop_grads.reference_grads with the codec in training mode."""
    from oracle import ref_import
    from oracle.reference_runner import _inject_first_randn
    variant, sd, cond, noise, d_depth, d_latent = mlg.case_inputs(name)
    mods = ref_import.reference_modules()
    head = mods.head_swin if variant == "swin" else mods.head_res
    model = head.ScheduledCNNRefine(256, 16)
    model.load_state_dict({k[len("model."):]: v for k, v in sd.items() if k.startswith("model.")}, strict=True)
    codec = _reference_codec()
    pipe = head.CNNDDIMPipiline(model, mods.scheduling_ddim.DDIMScheduler(num_train_timesteps=1000, clip_sample=False))
    cond = cond.clone().requires_grad_(True)
    with _inject_first_randn(noise) as st:
        latent, = pipe(batch_size=noise.shape[0], device=noise.device, dtype=noise.dtype, shape=noise.shape[-3:],
                       input_args=(cond, None, None, None), num_inference_steps=mlg.STEPS, return_dict=False)
    assert st["used"]
    depth = codec.inv_t(latent)
    ((depth * d_depth).sum() + (latent * d_latent).sum()).backward()
    grads = {"d_cond": cond.grad}
    for k, p in model.named_parameters():
        grads["model." + k] = p.grad
    for k, p in codec.conv_inv_transform.named_parameters():
        grads["depth_transform.conv_inv_transform." + k] = p.grad
    return sd, grads


def main():
    torch.set_num_threads(os.cpu_count() or 8)
    arrays = codec_arrays()
    for name in LOOP_CASES:
        sd, grads = loop_grads(name)
        _, _, cond, noise, d_depth, d_latent = mlg.case_inputs(name)
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
        print(f"[{name}] {len(grads)} gradients", flush=True)
    np.savez_compressed(OUT, **arrays)
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1e3:.0f} kB)")


if __name__ == "__main__":
    main()
