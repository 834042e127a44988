"""Helpers of the denoiser-gradient tests (test infrastructure; may import oracle/)."""
import os

import numpy as np
import torch

from oracle import restate
from oracle.make_denoiser_grads import CASES, case_inputs, checksum, denoiser_state  # noqa: F401

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "g_denoiser_grads.npz")
HEAD_TYPES = {"swin": "DDIMDepthEstimate_Swin_ADDHAHI", "res": "DDIMDepthEstimate_Res"}


class _FlipReluTorch:
    """Stands in for the `torch` module inside oracle.restate during one call: everything is torch's, except relu,
    whose gradient mask is flipped wherever |z| < band (what a computation whose ReLU inputs are off by up to `band`
    may do at the kinks).  torch itself is never modified."""

    def __init__(self, band):
        self._band = band

    def relu(self, z):
        return z * ((z > 0) ^ (z.abs() < self._band)).to(z.dtype)

    def __getattr__(self, name):
        return getattr(torch, name)


class _MaskedReluTorch:
    """Stands in for the `torch` module inside oracle.restate during one denoiser call: everything is torch's, except
    that its k-th relu(z) returns z * masks[k] (masks: the four ReLUs' 0 / 1 masks in forward order, e.g. the engine's
    own; None: z > 0, the restatement's own) and records z in fp64.  A call that runs more or fewer than len(masks) relus
    is an error."""

    def __init__(self, masks):
        self._masks = list(masks)
        self.z = []

    def relu(self, z):
        if len(self.z) == len(self._masks):
            raise RuntimeError(f"more than {len(self._masks)} relu calls")
        m = self._masks[len(self.z)]
        if m is None:
            m = z.detach() > 0
        if tuple(m.shape) != tuple(z.shape):
            raise RuntimeError(f"mask {len(self.z)} has shape {tuple(m.shape)}, relu input {tuple(z.shape)}")
        self.z.append(z.detach().to(torch.float64))
        return z * m.to(z.dtype)

    def check_complete(self):
        if len(self.z) != len(self._masks):
            raise RuntimeError(f"{len(self.z)} relu calls, {len(self._masks)} masks")

    def __getattr__(self, name):
        return getattr(torch, name)


def _grads_with(stand_in, variant, sd, noisy, cond, t, d_eps, dtype):
    """Gradients of sum(eps * d_eps), eps = restate.denoiser with `stand_in` (None: torch itself) as restate's torch."""
    p = {k: v.detach().cpu().to(dtype).requires_grad_(True) for k, v in sd.items()}
    x = noisy.detach().cpu().to(dtype).requires_grad_(True)
    c = cond.detach().cpu().to(dtype).requires_grad_(True)
    if stand_in is not None:
        restate.torch = stand_in
    try:
        eps = restate.denoiser(p, x, torch.as_tensor(t).cpu(), c, variant, prefix="model.")
    finally:
        restate.torch = torch
    (eps * d_eps.detach().cpu().to(dtype)).sum().backward()
    out = {"d_noisy": x.grad, "d_cond": c.grad}
    out.update({k: v.grad for k, v in p.items()})
    return out


def restatement_grads(variant, sd, noisy, cond, t, d_eps, dtype=torch.float64, band=0.0):
    """Gradients of sum(eps * d_eps) for eps = restate.denoiser, by torch autograd in `dtype` on CPU; `band` > 0 flips
    the ReLU masks within `band` of the kink (see kink_envelope)."""
    return _grads_with(_FlipReluTorch(band) if band != 0 else None, variant, sd, noisy, cond, t, d_eps, dtype)


def masked_restatement_grads(variant, sd, noisy, cond, t, d_eps, masks):
    """As restatement_grads in fp64, but with the four ReLU masks given (forward order, [B,C,h,w] each, e.g. the
    engine's `z > 0`; None: the fp64 forward's own) instead of taken from the fp64 forward: (gradients, the four ReLU
    inputs z in fp64).  At the
    engine's own masks the gradients differ from the engine's by rounding alone, with no kink to allow for."""
    relu = _MaskedReluTorch(masks)
    grads = _grads_with(relu, variant, sd, noisy, cond, t, d_eps, torch.float64)
    relu.check_complete()
    return grads, relu.z


def golden_margins(golden, case, grads):
    """max |g - g_ref| / max |g_ref| per gradient, at the golden's sampled entries."""
    out = {}
    for key in [k[len(case) + 1:-len("/absmax")] for k in golden.files if k.startswith(case + "/") and k.endswith("/absmax")]:
        g = grads[key].detach().double().cpu().reshape(-1).numpy()
        if case + "/" + key + "/index" in golden.files:
            g = g[golden[case + "/" + key + "/index"]]
        ref = golden[case + "/" + key + "/values"].astype(np.float64)
        out[key] = float(np.abs(g - ref).max() / float(golden[case + "/" + key + "/absmax"]))
    return out


def tensor_margins(grads, ref):
    """max |g - g_ref| / max |g_ref| per gradient, over every entry."""
    return {k: float((grads[k].detach().double().cpu() - ref[k].double()).abs().max() / ref[k].double().abs().max())
            for k in ref}


def make_head(variant, sd, device):
    """A DDIM head of `variant` on `device` whose denoiser holds `sd` (keys `model.*`)."""
    from diffusiondepth_b200.model.registry import HEADS
    torch.manual_seed(0)
    head = HEADS.build(dict(type=HEAD_TYPES[variant], in_channels=[64, 128, 256, 512], inference_steps=2,
                            num_train_timesteps=1000, depth_feature_dim=16, loss_cfgs=[], init_cfg=None))
    head.model.load_state_dict({k[len("model."):]: v for k, v in sd.items()}, strict=True)
    return head.to(device)


def kink_envelope(variant, sd, noisy, cond, t, d_eps, ref, band):
    """Per gradient: max |g_flipped - g_ref| / max |g_ref|, g_flipped = the fp64 gradient with every ReLU mask flipped
    within `band` of zero.  A ReLU input that an fp32-grade forward puts on the other side of zero changes the gradient
    by a whole masked element, far more than rounding does; this is the size of that effect on a given case (zero when
    no ReLU input lies that close to zero)."""
    flipped = restatement_grads(variant, sd, noisy, cond, t, d_eps, band=band)
    return tensor_margins(flipped, ref)
