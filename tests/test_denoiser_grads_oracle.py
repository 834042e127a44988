"""The fp64 restatement of ScheduledCNNRefine differentiates like the real reference: its autograd gradients reproduce
the ones oracle/make_denoiser_grads.py stored from the reference's own autograd (fp32, trained-like weights, odd sizes, a
repeated t).  This pins the restatement that the GPU gradient tests compare the engine against."""
import numpy as np
import pytest
import torch

from grad_helpers import (CASES, GOLDEN, case_inputs, checksum, golden_margins, kink_envelope, masked_restatement_grads,
                          restatement_grads, tensor_margins)

TOL = 1e-4


@pytest.mark.parametrize("case", list(CASES))
def test_restatement_gradients_match_reference(case):
    golden = np.load(GOLDEN, allow_pickle=False)
    variant, sd, noisy, cond, t, d_eps = case_inputs(case)
    assert np.array_equal(golden[case + "/t"], t.numpy())
    assert checksum(*sd.values()) == pytest.approx(float(golden[case + "/weight_checksum"]), rel=1e-12)
    assert checksum(noisy, cond, d_eps) == pytest.approx(float(golden[case + "/input_checksum"]), rel=1e-12)
    # in the reference's own fp32 the restatement's autograd reproduces the reference's (measured: bit for bit)
    m32 = golden_margins(golden, case, restatement_grads(variant, sd, noisy, cond, t, d_eps, dtype=torch.float32))
    assert len(m32) == (23 if variant == "swin" else 19)
    assert max(m32.values()) <= 1e-6, m32
    # in fp64 it differs from the fp32 reference by rounding (measured 1.5e-6 .. 6.1e-6 of max |g|) plus, where an fp32
    # ReLU input lies within rounding of zero, one flipped mask element (measured up to 1.0e-2 on the 19 x 27 cases)
    g64 = restatement_grads(variant, sd, noisy, cond, t, d_eps)
    m64 = golden_margins(golden, case, g64)
    env = kink_envelope(variant, sd, noisy, cond, t, d_eps, g64, band=1e-6)
    worst = max(m64, key=lambda k: m64[k] - env[k])
    print(f"\n[{case}] restatement fp64 vs reference fp32: worst {worst} {m64[worst]:.2e} (kink envelope {env[worst]:.2e})")
    for k in m64:
        assert m64[k] <= TOL + env[k], (k, m64[k], env[k])


@pytest.mark.parametrize("variant", ["swin", "res"])
def test_masked_restatement_at_its_own_masks(variant):
    """masked_restatement_grads, the fp64 reference the GPU tests evaluate at the engine's own ReLU masks: handed the
    fp64 forward's masks it is the plain fp64 restatement, and flipping one mask element of any layer moves a gradient."""
    _, sd, noisy, cond, t, d_eps = case_inputs(f"{variant}_19x27")
    ref = restatement_grads(variant, sd, noisy, cond, t, d_eps)
    _, z64 = masked_restatement_grads(variant, sd, noisy, cond, t, d_eps, [None] * 4)
    assert [z.shape[1] for z in z64] == [64, 256, 64, 16] and all(z.dtype == torch.float64 for z in z64)
    masks = [z > 0 for z in z64]
    got, z = masked_restatement_grads(variant, sd, noisy, cond, t, d_eps, masks)
    assert all(torch.equal(a, b) for a, b in zip(z, z64))
    m = tensor_margins(got, ref)
    assert max(m.values()) <= 1e-12, m
    for k in range(4):  # the element nearest the kink, where an fp32 forward may disagree with fp64
        flipped = [mk.clone() for mk in masks]
        i = int(z64[k].abs().argmin())
        flipped[k].view(-1)[i] = ~flipped[k].view(-1)[i]
        moved = tensor_margins(masked_restatement_grads(variant, sd, noisy, cond, t, d_eps, flipped)[0], ref)
        assert max(moved.values()) > 1e-9, (k, moved)
    with pytest.raises(RuntimeError):  # one mask per ReLU, no more and no fewer
        masked_restatement_grads(variant, sd, noisy, cond, t, d_eps, masks[:3])
    with pytest.raises(RuntimeError):
        masked_restatement_grads(variant, sd, noisy, cond, t, d_eps, masks + [None])
