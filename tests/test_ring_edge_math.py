"""The ring correction of the Swin step's composed convB -> pred.0 (pred_fold.cuh) as ring_fix_kernel computes it, in
fp64 on the CPU: four 1-D 5-tap edge convs of a's border rows and columns plus a fix-up at each corner,
  corr(p) = [y = 0] T(x) + [y = h-1] B(x) + [x = 0] (L(y) - C_TL - C_BL) + [x = w-1] (R(y) - C_TR - C_BR),
composed from the layer weights as compose_edge_kernel composes them.  The 5x5 composed conv minus this correction
equals the restatement's convB -> pred.0 chain on every pixel, down to latents with a side of 1."""
import pytest
import torch
import torch.nn.functional as F

from oracle import restate
from test_pred_fold_math import P, compose


def edge_kernels(wp, wb, bb):
    """Side s in T, B, L, R: pred.0's outer tap row / column o with convB's opposite one, tap k + e along the side.
    Corner (dy, dx): Wp0[d] WB[-d].  Returns {side: (kernel [co][ci][5], constant [co])}, {corner: (matrix, constant)}."""
    sides, corners = {}, {}
    for s in "TBLR":
        o = 0 if s in "TL" else 2
        k = torch.zeros(wp.shape[0], wb.shape[1], 5, dtype=wp.dtype)
        for kp in range(3):
            for e in range(3):
                k[:, :, kp + e] += (wp[:, :, o, kp] @ wb[:, :, 2 - o, e] if s in "TB"
                                    else wp[:, :, kp, o] @ wb[:, :, e, 2 - o])
        sides[s] = (k, (wp[:, :, o, :] if s in "TB" else wp[:, :, :, o]).sum(-1) @ bb)
    for c, (ky, kx) in {"TL": (0, 0), "TR": (0, 2), "BL": (2, 0), "BR": (2, 2)}.items():
        corners[c] = (wp[:, :, ky, kx] @ wb[:, :, 2 - ky, 2 - kx], wp[:, :, ky, kx] @ bb)
    return sides, corners


def ring_correction(a, wp, wb, bb):
    h, w = a.shape[-2:]
    sides, corners = edge_kernels(wp, wb, bb)
    corr = torch.zeros(a.shape[0], wp.shape[0], h, w, dtype=a.dtype)

    def conv1d(s, line):  # 5 taps along a border row / column, zero-padded
        k, c = sides[s]
        return F.conv1d(line, k, c, padding=2)

    corr[:, :, 0, :] += conv1d("T", a[:, :, 0, :])
    corr[:, :, h - 1, :] += conv1d("B", a[:, :, h - 1, :])
    corr[:, :, :, 0] += conv1d("L", a[:, :, :, 0])
    corr[:, :, :, w - 1] += conv1d("R", a[:, :, :, w - 1])
    for c, (y, x) in {"TL": (0, 0), "TR": (0, w - 1), "BL": (h - 1, 0), "BR": (h - 1, w - 1)}.items():
        m, k = corners[c]
        corr[:, :, y, x] -= a[:, :, y, x] @ m.T + k
    return corr


@pytest.mark.parametrize("h,w", [(18, 26), (35, 53), (3, 5), (1, 7), (2, 2), (1, 1), (1, 2), (2, 1), (3, 3), (4, 4),
                                 (1, 4), (4, 1), (2, 3), (3, 2), (4, 2), (2, 4), (3, 1), (1, 3)])
def test_edge_correction_equals_chain_every_pixel(h, w):
    g = torch.Generator().manual_seed(h * 100 + w + 7)
    c, cm, co = 24, 20, 12  # channel counts shrunk from 256 / 256 / 64: the identity does not depend on them
    sd = {P + "upsample_fuse.convB.conv.weight": torch.randn(cm, c, 3, 3, generator=g, dtype=torch.float64) * 0.1,
          P + "upsample_fuse.convB.conv.bias": torch.randn(cm, generator=g, dtype=torch.float64),
          P + "pred.0.weight": torch.randn(co, cm, 3, 3, generator=g, dtype=torch.float64) * 0.1,
          P + "pred.0.bias": torch.randn(co, generator=g, dtype=torch.float64)}
    wp, bp = sd[P + "pred.0.weight"], sd[P + "pred.0.bias"]
    wb, bb = sd[P + "upsample_fuse.convB.conv.weight"], sd[P + "upsample_fuse.convB.conv.bias"]
    a = torch.randn(2, c, h, w, generator=g, dtype=torch.float64)
    chain = restate.conv(restate.conv(a, sd, P + "upsample_fuse.convB.conv"), sd, P + "pred.0")
    k5, b5 = compose(wp, bp, wb, bb)
    got = F.conv2d(a, k5, b5, padding=2) - ring_correction(a, wp, wb, bb)
    assert ((got - chain).abs().max() / chain.abs().max()).item() <= 1e-12
