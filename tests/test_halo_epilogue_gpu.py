"""conv3x3_halo_kernel's output at the image's right and bottom edges, for every loop conv shape and each epilogue, on
grids whose sides are not multiples of the 16 x 8 tile (and 1 x n, n x 1), against the fp32 CUDA-core convolution
(DD_FLAG_SIMT_CONV).  The kernel writes its outputs as 8-channel boxes with TMA tensor stores, which the hardware clips
to the image, and sums GroupNorm partials over the pixels inside it only: a box written past an edge lands on the next
row's or image's pixels, and a partial that counts a clipped pixel moves the group's statistics.
  * EPI_F32: dd_conv3x3.
  * EPI_F32_STATS: dd_conv_groupnorm, its conv output and the per-group mean / rstd.
  * EPI_SPLIT: the Swin denoiser, whose 256 -> 256 conv (convA) hands its output to the next conv as fp16 hi / lo
    planes."""
import pytest
import torch

import diffusiondepth_b200 as dd
from oracle import restate
from test_pred_fold_gpu import DEV, _engine, _head

pytestmark = pytest.mark.gpu
SHAPES = [(16, 64), (64, 256), (256, 256), (256, 64), (64, 16)]
GRIDS = [(2, 35, 53), (1, 1, 37), (1, 29, 1), (1, 17, 9)]  # (B, H, W)
# the GroupNorm'd convs of the loop and the apply mode dd_conv_groupnorm runs them with (test_groupnorm_layers.LAYERS)
GN_CONVS = [(16, 64, 0), (64, 256, 1), (256, 64, 0), (64, 16, 3)]
TOL = 6e-5  # of max |simt|: both paths are within 3e-5 of an fp64 conv (test_gpu_parity)


def _conv_engines():
    return {k: dd.DenoiseEngine("swin", 1, (8, 16), (4, 8), 2, DEV, cuda_graph=False, simt_conv=k == "simt")
            for k in ("halo", "simt")}


def _inputs(cin, cout, B, H, W):
    g = torch.Generator().manual_seed(cin * 1000 + cout + 7 * H + W)
    x = (torch.randn(B, cin, H, W, generator=g) * 3).to(DEV)
    w = (torch.randn(cout, cin, 3, 3, generator=g) * 0.05).to(DEV)
    b = torch.randn(cout, generator=g).to(DEV)
    return g, x, w, b


def _rel(a, ref):
    return (a.double() - ref.double()).abs().max().item() / ref.abs().max().item()


@pytest.mark.parametrize("B,H,W", GRIDS)
def test_f32_epilogue_edges(B, H, W):
    engs = _conv_engines()
    for cin, cout in SHAPES:
        _, x, w, b = _inputs(cin, cout, B, H, W)
        y = {k: e.conv3x3(x, w, b) for k, e in engs.items()}
        assert torch.isfinite(y["halo"]).all(), (cin, cout)
        assert _rel(y["halo"], y["simt"]) < TOL, (cin, cout, _rel(y["halo"], y["simt"]))
    for e in engs.values():
        e.close()


@pytest.mark.parametrize("B,H,W", GRIDS)
def test_stats_epilogue_edges(B, H, W):
    engs = _conv_engines()
    for cin, cout, mode in GN_CONVS:
        g, x, w, b = _inputs(cin, cout, B, H, W)
        gamma = (torch.rand(cout, generator=g) + 0.5).to(DEV)
        beta = torch.randn(cout, generator=g).to(DEV)
        kw = {}
        if mode == 1:
            kw = dict(cond=torch.randn(B, 256, H, W, generator=g).to(DEV), temb=torch.randn(B, 256, generator=g).to(DEV))
        res = {k: e.conv_groupnorm(x, w, b, gamma, beta, mode, **kw) for k, e in engs.items()}
        (y, mr, _), (ys, mrs, _) = res["halo"], res["simt"]
        assert torch.isfinite(y).all() and torch.isfinite(mr).all(), (cin, cout)
        assert _rel(y, ys) < TOL, (cin, cout, _rel(y, ys))
        # mean against the conv output's scale, rstd relative to itself
        assert (mr[..., 0] - mrs[..., 0]).abs().max().item() < TOL * ys.abs().max().item(), (cin, cout)
        assert ((mr[..., 1] - mrs[..., 1]).abs() / mrs[..., 1]).max().item() < 1e-4, (cin, cout)
    for e in engs.values():
        e.close()


@pytest.mark.parametrize("hw,chw", [((35, 53), (18, 27)), ((1, 37), (1, 19)), ((29, 1), (15, 1))])
def test_split_epilogue_edges(hw, chw):
    head = _head(5)
    sd = {"depth_head." + k: v.detach().cpu() for k, v in head.state_dict().items()}
    B, (h, w) = 2, hw
    g = torch.Generator().manual_seed(h * 100 + w + 11)
    noisy = torch.randn(B, 16, h, w, generator=g) * 4
    cond = torch.randn(B, 256, *chw, generator=g)
    t = [950, 40]
    ref = restate.denoiser(sd, noisy.double(), torch.tensor(t), cond.double(), "swin")
    eps = {}
    for k in ("halo", "simt"):
        eng = _engine(head, B, hw, chw, 5, cuda_graph=False, simt_conv=k == "simt")
        eps[k] = eng.denoiser_forward(cond.to(DEV), noisy.to(DEV), t).double().cpu()
        eng.poll_status()
        eng.close()
    scale = max(1.0, ref.abs().max().item())
    assert (eps["halo"] - ref).abs().max().item() < 2e-4 * scale, hw
    assert (eps["halo"] - eps["simt"]).abs().max().item() < 2e-4 * scale, hw
