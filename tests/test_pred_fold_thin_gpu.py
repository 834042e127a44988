"""The composed convB -> pred.0 on latents that are all ring: one or two rows (ring_fix_kernel cuts them into rows) and
one or two columns (cut into columns).  A row of height 1 has both the top and the bottom edge kernel as its own sides,
a column of width 1 both the left and the right one, and every end pixel adds a crossing side and its corner terms.  As
on larger latents, the fold must be as accurate as the two-conv chain and bit-reproducible.

A 1 x 1 latent is left out: there the composed conv's centre tap carries all nine pred.0 . convB tap products and the
correction takes eight of them back, so the fp32 cancellation sets the error, not the correction's terms (on an H100,
max |d eps| 5.6e-6 for the fold against 1.3e-6 for the chain; 9.6e-6 when the correction was built from b_ext).  Its
algebra is checked in fp64 by tests/test_ring_edge_math.py."""
import pytest
import torch

from oracle import restate
from test_pred_fold_gpu import DEV, _engine, _errors, _head, _ring_mask

pytestmark = pytest.mark.gpu
# (latent h, w), (cond h, w)
THIN = [((2, 9), (1, 5)), ((9, 2), (5, 1)), ((1, 6), (1, 3)), ((6, 1), (3, 1))]


@pytest.mark.parametrize("hw,chw", THIN)
def test_operator_fold_vs_chain_thin(hw, chw):
    head = _head(5)
    sd = {"depth_head." + k: v.detach().cpu() for k, v in head.state_dict().items()}
    B, (h, w) = 2, hw
    g = torch.Generator().manual_seed(h * 100 + w + 3)
    noisy = torch.randn(B, 16, h, w, generator=g) * 4
    cond = torch.randn(B, 256, *chw, generator=g)
    t = [950, 40]
    ref = restate.denoiser(sd, noisy.double(), torch.tensor(t), cond.double(), "swin")
    mask = _ring_mask(h, w)
    err = {}
    for name, chain in (("fold", False), ("chain", True)):
        eng = _engine(head, B, hw, chw, 5, chain_pred=chain, cuda_graph=False)
        eps = eng.denoiser_forward(cond.to(DEV), noisy.to(DEV), t)
        eps2 = eng.denoiser_forward(cond.to(DEV), noisy.to(DEV), t)
        eng.poll_status()
        assert torch.equal(eps, eps2), (name, "repeat call")
        err[name] = _errors(eps, ref, mask)
        eng.close()
    print(f"{hw}: ring / interior max |d eps| fold {err['fold']}, chain {err['chain']}")
    assert err["fold"][0] <= 1.5 * err["chain"][0] + 1e-7, (hw, err)
