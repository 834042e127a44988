"""The algebra behind the Swin step's composed convB -> pred.0 (pred_fold.cuh), in fp64 on the CPU: the 5x5 composed
weights and bias on zero-padded input, minus the ring correction
  corr(p) = sum_{d: p + d outside} Wp0[d] b_ext(p + d),   b_ext(q) = bB + sum_{d': q + d' inside} WB[d'] a(q + d'),
equal the restatement's convB -> pred.0 chain on every pixel, for even, odd and tiny latents."""
import pytest
import torch
import torch.nn.functional as F

from oracle import restate

P = "depth_head.model."


def compose(wp, bp, wb, bb):
    """K5[co][ci][D] = sum_{cm, d + d' = D} Wp0[co][cm][d] WB[cm][ci][d'];  b5 = bp0 + sum_{cm, d} Wp0[co][cm][d] bB[cm]."""
    k5 = torch.zeros(wp.shape[0], wb.shape[1], 5, 5, dtype=wp.dtype)
    for ky in range(3):
        for kx in range(3):
            for ey in range(3):
                for ex in range(3):
                    k5[:, :, ky + ey, kx + ex] += wp[:, :, ky, kx] @ wb[:, :, ey, ex]
    return k5, bp + wp.sum((2, 3)) @ bb


def fold(a, wp, bp, wb, bb):
    k5, b5 = compose(wp, bp, wb, bb)
    y = F.conv2d(a, k5, b5, padding=2)
    h, w = a.shape[-2:]
    b_ext = F.conv2d(a, wb, bb, padding=2)           # b on [-1, h] x [-1, w], zero-padded a
    outside = torch.ones(h + 2, w + 2, dtype=torch.bool)
    outside[1:-1, 1:-1] = False
    return y - F.conv2d(b_ext * outside, wp)         # pred.0 taps that land outside the image


@pytest.mark.parametrize("h,w", [(18, 26), (35, 53), (3, 5), (1, 7), (2, 2)])
def test_fold_equals_chain_every_pixel(h, w):
    g = torch.Generator().manual_seed(h * 100 + w)
    c, cm, co = 24, 20, 12  # channel counts shrunk from 256 / 256 / 64: the identity does not depend on them
    sd = {P + "upsample_fuse.convB.conv.weight": torch.randn(cm, c, 3, 3, generator=g, dtype=torch.float64) * 0.1,
          P + "upsample_fuse.convB.conv.bias": torch.randn(cm, generator=g, dtype=torch.float64),
          P + "pred.0.weight": torch.randn(co, cm, 3, 3, generator=g, dtype=torch.float64) * 0.1,
          P + "pred.0.bias": torch.randn(co, generator=g, dtype=torch.float64)}
    a = torch.randn(2, c, h, w, generator=g, dtype=torch.float64)
    chain = restate.conv(restate.conv(a, sd, P + "upsample_fuse.convB.conv"), sd, P + "pred.0")
    got = fold(a, sd[P + "pred.0.weight"], sd[P + "pred.0.bias"], sd[P + "upsample_fuse.convB.conv.weight"],
               sd[P + "upsample_fuse.convB.conv.bias"])
    assert ((got - chain).abs().max() / chain.abs().max()).item() <= 1e-12
