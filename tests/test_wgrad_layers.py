"""dd_conv3x3_wgrad: the weight and bias gradient of one 3x3 conv on the backward's own kernels (wgrad_wgmma_kernel for
the three 256-wide shapes, wgrad_simt_kernel for 16->64 and 64->16) against fp64 on the CPU, at every hot-path shape and
at geometries that engage the tensor-core kernel's machinery: rows wider than one 64-pixel segment with a partial tail
segment, a CTA that sums its full 128 segments, several split-K chunks whose ranges break mid-row and mid-image, and the
training geometry.  Exact checks (every product an exact zero) pin cross-image leakage and the zero fill at the padding
and the row tail; the status word and run-to-run determinism are checked too."""
import pytest
import torch

import diffusiondepth_b200 as dd
from diffusiondepth_b200 import _cabi

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SHAPES = [(16, 64), (64, 256), (256, 256), (256, 64), (64, 16)]  # (cin, cout)
# (B, H, W); for the tensor-core shapes: xsegs = ceil(W / 64), segments = B * H * xsegs, chunks = ceil(segments / 128)
GEOMS = [
    (1, 3, 5),       # everything in one tail segment
    (1, 8, 64),      # a row exactly one segment wide
    (2, 5, 65),      # a 1-pixel tail segment: 2 / 20 / 1
    (1, 128, 64),    # one full CTA, the deepest fp32 accumulation: 1 / 128 / 1
    (1, 129, 64),    # a second chunk holding a single segment: 1 / 129 / 2
    (3, 43, 129),    # 3 / 387 / 4: CTA ranges break mid-row and mid-image; SIMT: 66 chunks, the last one 1 pixel
    (2, 176, 352),   # a 352 x 704 crop's latent: 6 / 2112 / 17; SIMT: 125 chunks that cross the image boundary
]
TOL_DW = 3e-5  # of max |dW_ref|: the forward layer test's bound
TOL_DB = 1e-6  # of max |db_ref|
DY_SCALES = [1e-9, 1.0, 3e4]


def _gid(g):
    return "B{}_{}x{}".format(*g)


@pytest.fixture(scope="module")
def eng():
    e = dd.DenoiseEngine("swin", 1, (8, 16), (4, 8), 2, DEV, cuda_graph=False)
    yield e
    e.close()


def _ref(x, dy):
    """fp64 weight and bias gradient of conv2d(x, w, b, padding=1) on the CPU, from the exact fp32 inputs."""
    xd, dyd = x.double().cpu(), dy.double().cpu()
    dw = torch.nn.grad.conv2d_weight(xd, (dy.shape[1], x.shape[1], 3, 3), dyd, padding=1)
    return dw, dyd.sum((0, 2, 3))


def _margin(got, ref):
    return (got.double().cpu() - ref).abs().max().item() / ref.abs().max().item()


@pytest.mark.parametrize("geom", GEOMS, ids=_gid)
@pytest.mark.parametrize("cin,cout", SHAPES)
def test_wgrad_vs_fp64(eng, cin, cout, geom):
    """Random data, independent per image: X = 3 randn (signed) and relu(randn) (the post-ReLU activations the engine
    feeds), dY = randn at 1e-9, 1 and 3e4 (the on-device split scale must follow)."""
    B, H, W = geom
    g = torch.Generator().manual_seed(cin * 1000 + cout + H * 7 + W)
    worst = 0.0
    for xk in ("randn*3", "relu"):
        x = torch.randn(B, cin, H, W, generator=g)
        x = x * 3 if xk == "randn*3" else torch.relu(x)
        for s in DY_SCALES:
            dy = torch.randn(B, cout, H, W, generator=g) * s
            dw, db = eng.conv3x3_wgrad(x.to(DEV), dy.to(DEV))
            ref_w, ref_b = _ref(x, dy)
            ew, eb = _margin(dw, ref_w), _margin(db, ref_b)
            print(f"\n[wgrad {cin}->{cout} {_gid(geom)} x={xk} dy*{s:g}] dW {ew:.2e} (bound {TOL_DW:.0e}) "
                  f"db {eb:.2e} (bound {TOL_DB:.0e})")
            assert ew <= TOL_DW, (xk, s, ew)
            assert eb <= TOL_DB, (xk, s, eb)
            worst = max(worst, ew / TOL_DW)
            if s == 1.0 and xk == "relu":  # determinism: a second call is bit-identical
                dw2, db2 = eng.conv3x3_wgrad(x.to(DEV), dy.to(DEV))
                assert torch.equal(dw, dw2) and torch.equal(db, db2)
    print(f"\n[wgrad {cin}->{cout} {_gid(geom)}] worst dW margin = {worst:.2f} of the bound")


@pytest.mark.parametrize("geom", GEOMS, ids=_gid)
@pytest.mark.parametrize("cin,cout", SHAPES)
def test_wgrad_exact_zeros(eng, cin, cout, geom):
    """Inputs for which every product of a tap is an exact zero, so the gradient must be exactly zero there."""
    B, H, W = geom
    g = torch.Generator().manual_seed(cin + cout + H + W)
    x = torch.randn(B, cin, H, W, generator=g).to(DEV)
    dy = torch.randn(B, cout, H, W, generator=g).to(DEV)
    # dY only on one border line: the taps that would read past it see the padding / the row tail's zero fill
    # (dW[..., ky, kx] pairs dY at p with X at p + (ky - 1, kx - 1))
    for name, sl, tap in [("col W-1", (..., slice(W - 1, W)), (..., 2)), ("col 0", (..., slice(0, 1)), (..., 0)),
                          ("row 0", (..., slice(0, 1), slice(None)), (..., 0, slice(None))),
                          ("row H-1", (..., slice(H - 1, H), slice(None)), (..., 2, slice(None)))]:
        d = torch.zeros_like(dy)
        d[sl] = dy[sl]
        dw, _ = eng.conv3x3_wgrad(x, d)
        assert dw[tap].abs().max().item() == 0.0, name
        assert dw.abs().max().item() > 0.0, name  # the other taps did see the data
    # dY only in image 1, X only in image 0: nothing may leak across an image (or CTA / chunk) boundary
    if B >= 2:
        xa, da = torch.zeros_like(x), torch.zeros_like(dy)
        xa[0], da[1] = x[0], dy[1]
        dw, _ = eng.conv3x3_wgrad(xa, da)
        assert dw.abs().max().item() == 0.0
    # dY all zero: exactly zero gradients, and the call succeeds
    dw, db = eng.conv3x3_wgrad(x, torch.zeros_like(dy))
    assert dw.abs().max().item() == 0.0 and db.abs().max().item() == 0.0


@pytest.mark.parametrize("cin,cout", SHAPES)
def test_wgrad_status_and_recovery(eng, cin, cout):
    """A single NaN in dY is reported as DD_ERR_RANGE; the next clean call on the same handle succeeds and equals a
    call made before the NaN, bit for bit."""
    B, H, W = 3, 43, 129
    g = torch.Generator().manual_seed(cin * 3 + cout)
    x = torch.randn(B, cin, H, W, generator=g).to(DEV)
    dy = torch.randn(B, cout, H, W, generator=g).to(DEV)
    dw0, db0 = eng.conv3x3_wgrad(x, dy)
    bad = dy.clone()
    bad[2, cout - 1, H - 1, W - 1] = float("nan")
    with pytest.raises(_cabi.EngineError, match="DD_ERR_RANGE"):
        eng.conv3x3_wgrad(x, bad)
    dw1, db1 = eng.conv3x3_wgrad(x, dy)
    assert torch.equal(dw0, dw1) and torch.equal(db0, db1)


def test_wgrad_rejects_off_path_shapes(eng):
    x, dy = torch.zeros(1, 32, 4, 4, device=DEV), torch.zeros(1, 64, 4, 4, device=DEV)
    with pytest.raises(_cabi.EngineError, match="DD_ERR_UNSUPPORTED"):
        eng.conv3x3_wgrad(x, dy)
