"""TEST INFRASTRUCTURE ONLY — the stochastic DDIM step (eta > 0) of the reference's sampler, restated in torch next to
oracle/restate.py (whose denoiser, alpha table and timesteps it uses): `DDIMScheduler.step(..., eta,
use_clipped_model_output=True, variance_noise=z)` (scheduling_ddim.py:285-350, epsilon prediction, clip_sample False) in
the reference's three-expression form, and `CNNDDIMPipiline.__call__` (head :254-303) with every draw injected."""
from typing import Dict

import torch

from oracle import restate

SD = Dict[str, torch.Tensor]


def ddim_step(eps, t: int, x, alphas_cumprod, num_inference_steps, eta, z, num_train_timesteps=1000):
    """One reverse step with sigma_t = eta sqrt(variance) and its variance noise z; scalars as 0-dim tensors."""
    prev_t = t - num_train_timesteps // num_inference_steps
    a_t = alphas_cumprod[t].to(x.dtype)
    a_prev = alphas_cumprod[prev_t].to(x.dtype) if prev_t >= 0 else torch.tensor(1.0, dtype=x.dtype)
    b_t = 1 - a_t
    x0 = (x - b_t ** 0.5 * eps) / a_t ** 0.5
    std = eta * (((1 - a_prev) / (1 - a_t)) * (1 - a_t / a_prev)) ** 0.5
    eps2 = (x - a_t ** 0.5 * x0) / b_t ** 0.5
    return a_prev ** 0.5 * x0 + (1 - a_prev - std ** 2) ** 0.5 * eps2 + std * z


def ddim_loop(sd: SD, cond, noise, num_inference_steps, variant, eta, zs, num_train_timesteps=1000):
    """The T-step sampler from x_T = noise with zs [T, B, 16, h, w] the per-step variance noise: (final latent, the
    latent after every step)."""
    acp = restate.ddim_tables(num_train_timesteps)
    x, trace = noise, []
    for i, t in enumerate(restate.ddim_timesteps(num_inference_steps, num_train_timesteps)):
        eps = restate.denoiser(sd, x, t, cond, variant)
        x = ddim_step(eps, t, x, acp, num_inference_steps, eta, zs[i], num_train_timesteps)
        trace.append(x)
    return x, trace
