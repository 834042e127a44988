"""The fp32 / fp64 restatement of the sampling loop + decoder differentiates like the real reference: autograd through
restate.ddim_loop + restate.decode reproduces the gradients oracle/make_loop_grads.py stored from the reference's own
CNNDDIMPipiline + ScheduledCNNRefine + DeepDepthTransformWithUpsampling.inv_t (fp32, trained-like weights and decoder
BatchNorm statistics, odd sizes, T = 3).  This pins the restatement that the GPU loop-gradient tests compare against."""
import numpy as np
import pytest
import torch

from grad_helpers import golden_margins, tensor_margins
from loop_grad_helpers import loop_restatement_grads
from oracle.make_loop_grads import CASES, OUT, STEPS, case_inputs, checksum

TOL = 1e-4


@pytest.mark.parametrize("case", list(CASES))
def test_loop_restatement_gradients_match_reference(case):
    golden = np.load(OUT, allow_pickle=False)
    variant, sd, cond, noise, d_depth, d_latent = case_inputs(case)
    assert checksum(*sd.values()) == pytest.approx(float(golden[case + "/weight_checksum"]), rel=1e-12)
    assert checksum(cond, noise, d_depth, d_latent) == pytest.approx(float(golden[case + "/input_checksum"]), rel=1e-12)
    g32 = loop_restatement_grads(variant, sd, cond, noise, d_depth, d_latent, STEPS, dtype=torch.float32)
    m32 = golden_margins(golden, case, g32)
    assert len(m32) == (28 if variant == "swin" else 24)  # d_cond, the denoiser's 21 / 17, the decoder's 6
    print(f"\n[{case}] restatement fp32 vs reference fp32: worst {max(m32.values()):.2e}")
    # fp32 rounding only: the T steps carry last-bit differences of the scheduler arithmetic into every sum (measured up to
    # 1.7e-6, and 1.1e-5 on the final conv bias, whose gradient sums e^-z over the map)
    assert max(m32.values()) <= 2e-5, m32
    g64 = loop_restatement_grads(variant, sd, cond, noise, d_depth, d_latent, STEPS)
    m64 = golden_margins(golden, case, g64)
    env = tensor_margins(loop_restatement_grads(variant, sd, cond, noise, d_depth, d_latent, STEPS, band=1e-6), g64)
    worst = max(m64, key=lambda k: m64[k] - env[k])
    print(f"[{case}] restatement fp64 vs reference fp32: worst {worst} {m64[worst]:.2e} (kink envelope {env[worst]:.2e})")
    for k in m64:
        assert m64[k] <= TOL + env[k], (k, m64[k], env[k])
