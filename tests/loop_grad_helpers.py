"""Helpers of the loop-gradient tests (dd_denoise_backward / dd_decode_backward): autograd through the restated
sampling loop and decoder, and a DDIM head holding a given denoiser + decoder.  Test infrastructure; may import oracle/."""
import torch

from grad_helpers import _FlipReluTorch, make_head
from oracle import restate


# ------------------------------------------------------------------ the sampling loop + decoder (dd_denoise_backward)
def _with_relu_band(band, fn):
    if band == 0:
        return fn()
    restate.torch = _FlipReluTorch(band)
    try:
        return fn()
    finally:
        restate.torch = torch


def loop_restatement_grads(variant, sd, cond, noise, d_depth, d_latent, steps, dtype=torch.float64, band=0.0):
    """Gradients of sum(depth * d_depth) + sum(latent * d_latent) for latent = restate.ddim_loop(cond, noise),
    depth = restate.decode(latent), by torch autograd in `dtype` on CPU (keys relative to `depth_head.`, plus d_cond and
    d_noise); `band` > 0 flips every ReLU mask within `band` of the kink, at every step and in the decoder."""
    p = {"depth_head." + k: v.detach().cpu().to(dtype).requires_grad_("running" not in k) for k, v in sd.items()}
    c = cond.detach().cpu().to(dtype).requires_grad_(True)
    x = noise.detach().cpu().to(dtype).requires_grad_(True)

    def run():
        latent = restate.ddim_loop(p, c, x, steps, variant)
        return latent, restate.decode(p, latent)

    latent, depth = _with_relu_band(band, run)
    loss = 0
    if d_depth is not None:
        loss = loss + (depth * d_depth.detach().cpu().to(dtype)).sum()
    if d_latent is not None:
        loss = loss + (latent * d_latent.detach().cpu().to(dtype)).sum()
    loss.backward()
    out = {"d_cond": c.grad, "d_noise": x.grad}
    out.update({k[len("depth_head."):]: v.grad for k, v in p.items() if v.grad is not None})
    return out


def decode_restatement_grads(sd, latent, d_depth, dtype=torch.float64, band=0.0):
    """Gradients of sum(restate.decode(latent) * d_depth): d_latent and the decoder parameters."""
    p = {"depth_head." + k: v.detach().cpu().to(dtype).requires_grad_("running" not in k)
         for k, v in sd.items() if k.startswith("depth_transform.")}
    x = latent.detach().cpu().to(dtype).requires_grad_(True)
    depth = _with_relu_band(band, lambda: restate.decode(p, x))
    (depth * d_depth.detach().cpu().to(dtype)).sum().backward()
    out = {"d_latent": x.grad}
    out.update({k[len("depth_head."):]: v.grad for k, v in p.items() if v.grad is not None})
    return out


def make_loop_head(variant, sd, steps, device):
    """A DDIM head with the denoiser and decoder of `sd` (keys `model.*`, `depth_transform.*`) running `steps` steps."""
    head = make_head(variant, {k: v for k, v in sd.items() if k.startswith("model.")}, device)
    head.depth_transform.load_state_dict({k[len("depth_transform."):]: v for k, v in sd.items()
                                          if k.startswith("depth_transform.")}, strict=False)
    head.diffusion_inference_steps = steps
    return head
