"""The fp64 restatement of the encoder's gradients (encoder_grad_helpers) against the real reference
(tests/golden/g_encoder_grads.npz, oracle/make_encoder_grads.py): `t` in both BatchNorm modes, and one Res head
`ddim_loss_gt` through the training-mode encoder and the denoiser.  CPU only."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from encoder_grad_helpers import encode, encode_grads, encoder_params
from grad_helpers import golden_margins
from oracle import restate
from oracle.make_denoiser_grads import checksum
from oracle.make_encoder_grads import CASES, case_inputs, loss_gt_inputs
from oracle.make_loop_grads import loop_state

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "g_encoder_grads.npz")
TOL = 1e-6  # of max |g_ref|: fp64 against the reference's fp32
# plus, per gradient, twice the spread of the restatement run in fp32 from its fp64 self: in training mode the weight
# gradients behind a BatchNorm cancel (sum du = 0 over the batch), and with few values per channel the reference's own
# fp32 rounding reaches 1e-4 of max |g| there


def _fp32_envelope(fn):
    g64, g32 = fn(torch.float64), fn(torch.float32)
    return {k: 2 * float((g32[k].double() - g64[k]).abs().max() / g64[k].abs().max()) for k in g64}, g64


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def test_golden_inputs_unchanged(golden):
    sd = loop_state("res")
    assert checksum(*[v for k, v in sd.items() if k.startswith("depth_transform.")]) == \
        pytest.approx(float(golden["weight_checksum"]), rel=1e-12)
    for name in CASES:
        assert checksum(*case_inputs(name)) == pytest.approx(float(golden[f"enc/eval/{name}/input_checksum"]), rel=1e-12)


@pytest.mark.parametrize("mode", ("eval", "train"))
@pytest.mark.parametrize("name", tuple(CASES))
def test_restated_encoder_grads_match_reference(golden, name, mode):
    depth, d_latent = case_inputs(name)
    sd = loop_state("res")
    env, grads = _fp32_envelope(lambda dt: encode_grads(sd, depth, d_latent, mode == "train", dtype=dt)[0])
    m = golden_margins(golden, f"enc/{mode}/{name}", grads)
    assert len(m) == 6
    for k, v in m.items():
        assert v <= TOL + env[k], (k, v, env[k])


def _loss_gt_grads(golden, dtype, box=None):
    """The restated Res head ddim_loss_gt (training-mode encoder) on the golden's noise and timesteps, in `dtype`."""
    from diffusiondepth_b200.model.diffusers.schedulers.scheduling_ddim import DDIMScheduler
    sd = loop_state("res")
    gt, cond = loss_gt_inputs()
    noise = torch.from_numpy(golden["loss_gt/noise"]).to(dtype)
    t = torch.from_numpy(golden["loss_gt/t"])
    p = encoder_params(sd, dtype)
    pm = {k: v.detach().to(dtype).requires_grad_(True) for k, v in sd.items() if k.startswith("model.")}
    c = cond.to(dtype).requires_grad_(True)
    gt_t, _ = encode(p, gt.to(dtype), True)
    acp = DDIMScheduler(num_train_timesteps=1000, clip_sample=False).alphas_cumprod.to(dtype)[t]
    noisy = acp.sqrt().view(-1, 1, 1, 1) * gt_t + (1 - acp).sqrt().view(-1, 1, 1, 1) * noise
    loss = F.mse_loss(restate.denoiser(pm, noisy, t, c, "res", prefix="model."), noise)
    loss.backward()
    if box is not None:
        box["loss"] = float(loss.detach())
    grads = {"d_cond": c.grad}
    grads.update({k: v.grad for k, v in pm.items()})
    grads.update({k: v.grad for k, v in p.items() if v.grad is not None})
    return grads


def test_restated_ddim_loss_gt_matches_reference(golden):
    box = {}
    env, grads = _fp32_envelope(lambda dt: _loss_gt_grads(golden, dt, box if dt == torch.float64 else None))
    assert box["loss"] == pytest.approx(float(golden["loss_gt/loss"]), rel=1e-5)
    m = golden_margins(golden, "loss_gt", grads)
    assert sum(k.startswith("depth_transform.") for k in m) == 6 and "d_cond" in m
    for k, v in m.items():
        assert v <= TOL + env[k], (k, v, env[k])
