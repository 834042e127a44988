"""The DDIM loop's four GroupNorm(4, C) + ReLU layers (noise_embedding.1 / .4, pred.1 / .4) one layer at a time against
fp64, through dd_conv_groupnorm: the 3x3 conv with its statistics epilogue (conv3x3_halo_kernel, or conv3x3_simt_kernel
under DD_FLAG_SIMT_CONV), gn_finalize_kernel and the loop's apply kernel of the layer (GroupNorm + ReLU; + the
condition and time embedding at the same grid; + their align_corners=True bilinear upsampling; the collapsed DDIM
update).  The statistics are single-pass fp32 sums of v and v^2 per tile, combined in fp64, so the cases aim at groups
whose mean dominates their spread: bias offsets and non-negative (post-ReLU-like) inputs through non-zero-sum weights
at mean / std up to 1000, constant groups, groups where eps matters, negative and near-zero gamma.

Each layer is held to 3e-5 of its own max |ref| in three parts:
  * the conv output y32 against an fp64 conv of the same x;
  * mean / rstd against fp64 statistics of the engine's own y32, and the layer's output against fp64 GroupNorm (+ its
    apply) of that y32.  Comparing the norm with its own input isolates it: at mean / std = 1000 the fp32 rounding of y
    alone is 6e-5 of a group's std, which no norm can undo;
  * end to end against fp64 from x, where the offset leaves y's fp32 rounding below the bound (mean / std <= 10).

Measured on an H100 80GB HBM3 (700 W), worst over each group of cases, as a fraction of the bound (`-s` prints every
case).  Layers at every size: conv 0.30, mean 0.00, rstd 0.00, output 0.05, end to end 0.20.  Offset groups at mean /
std 10, 100, 300, 1000: rstd 0.00 at all four and output 0.05, 0.07, 0.28, 0.54.  The fp32 sums these kernels used
before gave rstd 0.05, 4.6, 81 and 576 times the bound there (rstd off by 1.7e-2 at 1000), the whole denoiser at mean
/ std ~300 eps 131 times its bound.  Degenerate groups (mean 0) 0.33; the constant group at mean 50 still misses
(3-6x, the apply kernels' fp32 affine; marked xfail).  Up-add geometries 0.06.  Denoiser with offset groups: eps 0.36,
ReLU inputs 0.33.

Operator-level cases run the whole denoiser with offset conv biases (and, separately, an offset latent): eps against
the fp64 restatement, and each ReLU input of dd_denoiser_relu_inputs against fp64 GroupNorm of the conv of the engine's
own upstream activations.  Exact checks pin cross-image isolation and run-to-run determinism.

The CPU test at the end pins this file's fp64 layer reference to oracle.restate's GroupNorm, upsampling and DDIM step."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import diffusiondepth_b200 as dd
from diffusiondepth_b200.engine import GN_LAYERS, ddim_coefficients
from oracle import restate

DEV = torch.device("cuda:0")
TOL = 3e-5        # of max |ref|: the bound of the hot-path conv layer tests
RSTD_TOL = 3e-5   # relative error of rstd against fp64 statistics of the engine's own conv output
ZTOL = 5e-5       # of max |z64| per GroupNorm at operator level (as the backward's recompute is held)
# eps of the whole denoiser with every norm's groups at mean / std ~300, against fp64 from the input: each pre-norm conv
# output carries fp32 rounding of ~300 x 6e-8 of its std, through four layers (measured up to 3.6e-5)
EPS_TOL = 1e-4
gpu = pytest.mark.gpu

# (cin, cout, mode): 16 -> 64 (noise_embedding.1), 64 -> 256 (noise_embedding.4: Res head at the same grid, Swin head
# up-add), 256 -> 64 (pred.1 after the Res head's feat or the chained pred.0), 64 -> 16 (pred.4 + the DDIM update)
LAYERS = [(16, 64, 0), (64, 256, 1), (64, 256, 2), (256, 64, 0), (64, 16, 3)]
KERNELS = ["halo", "simt"]
RATIOS = [0, 10, 100, 300, 1000]
C_X, C_EPS = 1.0207, -0.1931  # a mid-schedule DDIM step's coefficients


# ------------------------------------------------------------------------------------------------ fp64 reference
def gn_stats64(y):
    """Per (image, group) mean and rstd = 1 / sqrt(var + 1e-5), biased variance, of y [B, C, H, W] in fp64."""
    v = y.double().reshape(y.shape[0], 4, -1)
    mean = v.mean(-1)
    var = ((v - mean[..., None]) ** 2).mean(-1)
    return mean, 1.0 / torch.sqrt(var + 1e-5)


def apply64(y, gamma, beta, mode, cond=None, temb=None, latent=None, c_x=C_X, c_eps=C_EPS):
    """GroupNorm(4, C) (eps 1e-5) + ReLU of y in fp64, then the loop's injection of the layer's mode: 1 adds cond + temb
    (Res head :340, feat = cond + temb first), 2 adds up(cond + temb), bilinear, align_corners=True (UpSample_add), 3 the
    DDIM update c_x x + c_eps eps when a latent is given."""
    h = torch.relu(F.group_norm(y.double(), 4, gamma.double(), beta.double(), 1e-5))
    if mode in (1, 2):
        feat = cond.double() + temb.double()[..., None, None]
        if mode == 2:
            feat = F.interpolate(feat, size=y.shape[-2:], mode="bilinear", align_corners=True)
        h = feat + h
    if mode == 3 and latent is not None:
        h = c_x * latent.double() + c_eps * h
    return h


def conv64(x, w, b):
    return F.conv2d(x.double(), w.double(), b.double(), padding=1)


# ------------------------------------------------------------------------------------------------ cases
def _engine(kernel):
    return dd.DenoiseEngine("swin", 1, (8, 16), (4, 8), 2, DEV, cuda_graph=False, simt_conv=kernel == "simt")


@pytest.fixture(scope="module")
def engines():
    e = {k: _engine(k) for k in KERNELS}
    yield e
    for v in e.values():
        v.close()


def _cond_hw(mode, H, W):
    return ((H + 1) // 2, (W + 1) // 2) if mode == 2 else (H, W)


def make_case(cin, cout, mode, B, H, W, seed, ratio=0, offset="bias", degenerate=False):
    """Inputs of one layer.  ratio > 0: each group's mean / std is set to `ratio` by a per-group bias offset
    ("bias": zero-mean x, random 3x3 weights) or by the input ("input": x = |N(0, 1)| + s through centre-tap weights
    whose rows sum to 1, so every pixel, border included, carries the same offset).  degenerate: group 0 constant (0 for
    even seeds, 50 for odd ones), group 1 with std ~1e-3 (eps matters), group 2 with negative gamma, group 3 with gamma
    ~1e-6."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, cin, H, W, generator=g)
    if offset == "input" and ratio > 0:
        x = x.abs()
        w = torch.zeros(cout, cin, 3, 3, dtype=torch.float64)
        wc = torch.randn(cout, cin, generator=g, dtype=torch.float64) * 0.3 / cin ** 0.5
        w[:, :, 1, 1] = wc - wc.mean(1, keepdim=True) + 1.0 / cin
        w = w.float()
    else:
        w = torch.randn(cout, cin, 3, 3, generator=g) * (1.0 / (3 * cin ** 0.5))
    b = torch.randn(cout, generator=g) * 0.1
    gamma = 1.0 + 0.3 * torch.randn(cout, generator=g)
    beta = 0.2 * torch.randn(cout, generator=g)
    gc = cout // 4
    if degenerate:
        w[:gc] = 0.0
        b[:gc] = 0.0 if seed % 2 == 0 else 50.0
        w[gc:2 * gc] *= 1e-3
        gamma[2 * gc:3 * gc] = -gamma[2 * gc:3 * gc].abs()
        gamma[3 * gc:] = 1e-6 * torch.randn(gc, generator=g)
    if ratio > 0:
        y0 = conv64(x, w, b)
        mean, rstd = gn_stats64(y0)
        m, s = mean.mean(0), (1.0 / rstd).mean(0)  # per group, over the batch
        if offset == "input":
            shift = (ratio * s.min() - m.min()).clamp(min=0.0)  # every output channel's weights sum to 1
            x = x + float(shift)
        else:
            b = (b.double() + (ratio * s - m).repeat_interleave(gc)).float()
    ch, cw = _cond_hw(mode, H, W)
    cond = torch.randn(B, 256, ch, cw, generator=g) if mode in (1, 2) else None
    temb = torch.randn(B, 256, generator=g) if mode in (1, 2) else None  # one row per image
    latent = torch.randn(B, 16, H, W, generator=g) * 3 if mode == 3 else None
    return dict(x=x, w=w, b=b, gamma=gamma, beta=beta, cond=cond, temb=temb, latent=latent)


def run(eng, case, mode, up_qpb=4, update=False):
    dev = {k: (v.to(DEV) if v is not None else None) for k, v in case.items()}
    lat = dev["latent"].clone() if (mode == 3 and update) else None
    y, mr, out = eng.conv_groupnorm(dev["x"], dev["w"], dev["b"], dev["gamma"], dev["beta"], mode, cond=dev["cond"],
                                    temb=dev["temb"], latent=lat, c_x=C_X, c_eps=C_EPS, up_qpb=up_qpb)
    torch.cuda.synchronize()
    return y.cpu(), mr.cpu(), out.cpu(), (lat.cpu() if lat is not None else None)


def margins(case, mode, got, update=False, end_to_end=True):
    """Fractions of the bound: conv, mean, rstd, output vs GN of the engine's y, (output end to end), (updated latent)."""
    y, mr, out, lat = got
    y_ref = conv64(case["x"], case["w"], case["b"])
    m = {"conv": float((y.double() - y_ref).abs().max() / y_ref.abs().max()) / TOL}
    mean_e, rstd_e = gn_stats64(y)
    # the mean is returned in fp32: against the fp32 rounding of the fp64 mean (at mean / std = 1000 that rounding alone
    # is 6e-5 of the std)
    m["mean"] = float(((mr[..., 0].double() - mean_e.float().double()) * rstd_e).abs().max()) / RSTD_TOL
    m["rstd"] = float(((mr[..., 1].double() - rstd_e) / rstd_e).abs().max()) / RSTD_TOL
    lat_in = case["latent"] if update else None
    extra = dict(cond=case["cond"], temb=case["temb"], latent=lat_in)
    ref = apply64(y, case["gamma"], case["beta"], mode, **extra)
    scale = float(ref.abs().max())
    m["out"] = float((out.double() - ref).abs().max()) / scale / TOL
    if end_to_end:
        ref2 = apply64(y_ref, case["gamma"], case["beta"], mode, **extra)
        m["e2e"] = float((out.double() - ref2).abs().max()) / float(ref2.abs().max()) / TOL
    if lat is not None:
        m["latent"] = float((lat.double() - ref).abs().max()) / scale / TOL
    return m


def _report(tag, m):
    print(f"\n[{tag}] " + " ".join(f"{k}={v:.2f}" for k, v in m.items()))


def _assert(tag, m):
    _report(tag, m)
    for k, v in m.items():
        assert v <= 1.0, (tag, k, v)


# ------------------------------------------------------------------------------------------------ layers
SIZES = [(2, 32, 32), (1, 16, 8), (1, 13, 21), (4, 5, 9), (2, 57, 76)]  # exact tiles of both kernels, one tile, ragged


@gpu
@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("cin,cout,mode", LAYERS)
def test_layer_vs_fp64(engines, kernel, cin, cout, mode):
    """Every loop layer on both conv kernels at exact, ragged, single-tile and sub-tile sizes, B in {1, 2, 4}: pixels
    outside the image must not enter the partials (they would move mean and rstd)."""
    for i, (B, H, W) in enumerate(SIZES):
        case = make_case(cin, cout, mode, B, H, W, seed=100 * cin + cout + i)
        for update in ([False, True] if mode == 3 else [False]):
            qpbs = [4, 1] if mode == 2 else [4]
            for qpb in qpbs:
                got = run(engines[kernel], case, mode, qpb, update)
                _assert(f"{kernel} {cin}->{cout} mode {mode} B={B} {H}x{W} qpb={qpb} update={update}",
                        margins(case, mode, got, update))


@gpu
@pytest.mark.parametrize("offset", ["bias", "input"])
@pytest.mark.parametrize("ratio", RATIOS)
@pytest.mark.parametrize("cin,cout,mode", LAYERS)
def test_offset_dominated_groups(engines, cin, cout, mode, ratio, offset):
    """Groups whose mean is `ratio` times their std, from the bias or from a non-negative input through non-zero-sum
    weights (an offset no per-channel bias trick removes), on the tensor-core kernel at a ragged multi-tile size, and on
    the CUDA-core kernel at one size."""
    for kernel, (B, H, W) in [("halo", (2, 57, 76)), ("simt", (1, 19, 27))]:
        case = make_case(cin, cout, mode, B, H, W, seed=7 * ratio + cin + cout, ratio=ratio, offset=offset)
        mean, rstd = gn_stats64(conv64(case["x"], case["w"], case["b"]))
        got_ratio = float((mean * rstd).abs().min())
        assert ratio == 0 or got_ratio > 0.6 * ratio, got_ratio
        m = margins(case, mode, run(engines[kernel], case, mode), end_to_end=ratio <= 10)
        _assert(f"{kernel} {cin}->{cout} mode {mode} {offset} mean/std {got_ratio:.0f}", m)


@gpu
@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("cin,cout,mode", LAYERS)
@pytest.mark.parametrize("seed", [0, pytest.param(1, marks=pytest.mark.xfail(
    strict=True, reason="the apply kernels form beta - (rstd gamma) mean in fp32: at mean 50, rstd 316 its rounding "
                        "(~1e-3) reaches the output (measured 3-6x the bound)"))])  # constant group at 0, at 50
def test_degenerate_groups(engines, kernel, cin, cout, mode, seed):
    """A constant group (std 0, mean 0 or 50), a group with std ~1e-3 (eps is 10x its variance), negative and near-zero
    gamma.  A constant group's output is relu(beta) (to the fp16 hi/lo split's 2^-21): the statistics must not invent a
    spread."""
    B, H, W = 2, 19, 27
    case = make_case(cin, cout, mode, B, H, W, seed=seed, degenerate=True)
    got = run(engines[kernel], case, mode)
    _assert(f"{kernel} {cin}->{cout} mode {mode} degenerate seed {seed}", margins(case, mode, got))
    if mode in (0, 3):
        gc = cout // 4
        out = got[2][:, :gc].double()
        want = torch.relu(case["beta"][:gc]).double()[None, :, None, None]
        assert float((out - want).abs().max()) <= 2.0 ** -21 * float(want.abs().max())


@gpu
@pytest.mark.parametrize("hw,chw", [((19, 27), (10, 14)), ((35, 53), (18, 27)), ((18, 26), (9, 13))])
@pytest.mark.parametrize("qpb", [4, 1])
def test_up_add_odd_geometry(engines, hw, chw, qpb):
    """The bilinear up-add at latent / condition pairs that send quads down the per-tap path, both block shapes,
    distinct time-embedding rows per image, with an offset group statistic."""
    B = 2
    case = make_case(64, 256, 2, B, *hw, seed=hw[0] + qpb, ratio=100)
    g = torch.Generator().manual_seed(5)
    case["cond"] = torch.randn(B, 256, *chw, generator=g)
    got = run(engines["halo"], case, 2, qpb)
    _assert(f"up-add {hw} over {chw} qpb={qpb}", margins(case, 2, got, end_to_end=False))


@gpu
@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("cin,cout,mode", LAYERS)
def test_isolation_and_determinism(engines, kernel, cin, cout, mode):
    """Scaling image 1 by 1e3 leaves image 0's conv output, statistics and output bit-identical; two runs are
    bit-identical."""
    B, H, W = 2, 21, 35
    case = make_case(cin, cout, mode, B, H, W, seed=11)
    eng = engines[kernel]
    update = mode == 3
    a, b = run(eng, case, mode, update=update), run(eng, case, mode, update=update)
    for u, v in zip(a, b):
        if u is not None:
            assert torch.equal(u, v)
    case["x"] *= 0.5  # image 1 at 1e3 stays inside the fp16 split's range of the loop's activation planes
    a = run(eng, case, mode, update=update)
    big = dict(case, x=case["x"].clone())
    big["x"][1] *= 1e3
    c = run(eng, big, mode, update=update)
    for u, v in zip(a, c):
        if u is not None:
            assert torch.equal(u[0], v[0])


# ------------------------------------------------------------------------------------------------ operator level
def _offset_state(variant, ratio, kind, noisy, cond, t):
    """denoiser_state with every GroupNorm'd conv's bias shifted so that its groups' mean / std is about `ratio`
    (kind "bias"), or unchanged (kind "latent", where the latent carries the offset)."""
    from grad_helpers import denoiser_state
    sd = {k: v.clone() for k, v in denoiser_state(variant).items()}
    if kind != "bias":
        return sd
    for prefix in ("noise_embedding.0", "noise_embedding.3", "pred.0", "pred.3"):
        ys = _chain(sd, variant, noisy.double(), cond.double(), t)[0]
        y = ys[["noise_embedding.0", "noise_embedding.3", "pred.0", "pred.3"].index(prefix)]
        mean, rstd = gn_stats64(y)
        m, s = mean.mean(0), (1.0 / rstd).mean(0)
        key = f"model.{prefix}.bias"
        sd[key] = (sd[key].double() + (ratio * s - m).repeat_interleave(sd[key].shape[0] // 4)).float()
    return sd


def _chain(sd, variant, x, cond, t, z_eng=None):
    """The denoiser in fp64 as pre-GN conv outputs ys and ReLU inputs zs; with z_eng, each conv reads the ReLU of the
    engine's own upstream ReLU input instead of the fp64 one."""
    p = lambda k: sd["model." + k].double()  # noqa: E731
    cv = lambda h, k: F.conv2d(h, p(k + ".weight"), p(k + ".bias"), padding=1)  # noqa: E731
    gn = lambda h, k: F.group_norm(h, 4, p(k + ".weight"), p(k + ".bias"), 1e-5)  # noqa: E731
    src = lambda i, zs: torch.relu(zs[i] if z_eng is None else z_eng[i])  # noqa: E731
    temb = p("time_embedding.weight")[torch.as_tensor(t)]
    ys, zs = [], []
    ys.append(cv(x, "noise_embedding.0"))
    zs.append(gn(ys[-1], "noise_embedding.1"))
    ys.append(cv(src(0, zs), "noise_embedding.3"))
    zs.append(gn(ys[-1], "noise_embedding.4"))
    feat = cond + temb[..., None, None]
    if variant == "swin":
        up = F.interpolate(feat, size=x.shape[-2:], mode="bilinear", align_corners=True)
        feat = cv(cv(up + src(1, zs), "upsample_fuse.convA.conv"), "upsample_fuse.convB.conv")
    else:
        feat = feat + src(1, zs)
    ys.append(cv(feat, "pred.0"))
    zs.append(gn(ys[-1], "pred.1"))
    ys.append(cv(src(2, zs), "pred.3"))
    zs.append(gn(ys[-1], "pred.4"))
    return ys, zs


@gpu
@pytest.mark.parametrize("variant,hw", [("res", (19, 27)), ("swin", (19, 27)), ("swin", (35, 53))])
@pytest.mark.parametrize("kind", ["bias", "latent"])
def test_denoiser_with_offset_groups(variant, hw, kind):
    """The whole denoiser with every GroupNorm'd conv's groups at mean / std ~300 (kind "bias"), or a latent offset by
    300 (kind "latent"): eps of dd_denoiser_forward (Swin: the composed pred.0 and its ring partials) against the fp64
    restatement, and each ReLU input of dd_denoiser_relu_inputs (the backward's recomputation) against fp64 GroupNorm of
    the conv of the engine's own upstream activations."""
    from grad_helpers import make_head
    B, (h, w) = 2, hw
    ch, cw = ((h + 1) // 2, (w + 1) // 2) if variant == "swin" else (h, w)
    g = torch.Generator().manual_seed(13)
    noisy = torch.randn(B, 16, h, w, generator=g) + (300.0 if kind == "latent" else 0.0)
    cond = torch.randn(B, 256, ch, cw, generator=g).abs()
    t = [417, 12]
    sd = _offset_state(variant, 300, kind, noisy, cond, t)
    head = make_head(variant, sd, DEV)
    eng = head._engine(B, hw, (ch, cw), DEV, backward=True)
    c, x = cond.to(DEV), noisy.to(DEV)
    eps = eng.denoiser_forward(c, x, t).double().cpu()
    z_dev = eng.denoiser_relu_inputs(c, x, t)
    eng.poll_status()
    z_eng = [v.double().cpu() for v in z_dev.values()]
    ref = restate.denoiser(sd, noisy.double(), t, cond.double(), variant, prefix="model.")
    m = {"eps": float((eps - ref).abs().max()) / float(ref.abs().max()) / EPS_TOL}
    ys, zs = _chain(sd, variant, noisy.double(), cond.double(), t, z_eng=z_eng)
    ratios = []
    for k, ze, zr, y in zip(GN_LAYERS, z_eng, zs, ys):
        mean, rstd = gn_stats64(y)
        ratios.append(float((mean * rstd).abs().max()))
        m[k] = float((ze - zr).abs().max()) / float(zr.abs().max()) / ZTOL
    _assert(f"denoiser {variant} {hw} {kind}: mean/std " + ", ".join(f"{r:.0f}" for r in ratios), m)


# ------------------------------------------------------------------------------------------------ CPU
def test_reference_matches_restated_modules():
    """apply64 against oracle.restate's GroupNorm, the reference's F.interpolate order (interpolate cond + temb, then
    add) and DDIM step (the three-expression form equals c_x x + c_eps eps); gn_stats64 against F.group_norm."""
    g = torch.Generator().manual_seed(0)
    B, C, H, W = 2, 64, 7, 9
    y = torch.randn(B, C, H, W, generator=g, dtype=torch.float64) * 3 + 40
    sd = {"gn.weight": torch.randn(C, generator=g, dtype=torch.float64),
          "gn.bias": torch.randn(C, generator=g, dtype=torch.float64)}
    gn = restate.group_norm4(y, sd, "gn")
    assert torch.allclose(apply64(y, sd["gn.weight"], sd["gn.bias"], 0), torch.relu(gn), rtol=0, atol=1e-12)
    mean, rstd = gn_stats64(y)
    ones, zeros = torch.ones(C, dtype=torch.float64), torch.zeros(C, dtype=torch.float64)
    v = y.reshape(B, 4, -1)
    norm = ((v - mean[..., None]) * rstd[..., None]).reshape_as(y)
    assert torch.allclose(norm, F.group_norm(y, 4, ones, zeros, 1e-5), rtol=0, atol=1e-12)
    cond = torch.randn(B, C, 4, 5, generator=g, dtype=torch.float64)
    temb = torch.randn(B, C, generator=g, dtype=torch.float64)
    up = F.interpolate(cond + temb[..., None, None], size=(H, W), mode="bilinear", align_corners=True)
    assert torch.allclose(apply64(y, sd["gn.weight"], sd["gn.bias"], 2, cond=cond, temb=temb), up + torch.relu(gn),
                          rtol=0, atol=1e-12)
    same = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    assert torch.allclose(apply64(y, sd["gn.weight"], sd["gn.bias"], 1, cond=same, temb=temb),
                          same + temb[..., None, None] + torch.relu(gn), rtol=0, atol=1e-12)
    acp = restate.ddim_tables()
    ts, cx, ce = ddim_coefficients(acp, 20, 1000)
    x = torch.randn(B, 16, H, W, generator=g, dtype=torch.float64) * 3
    y16 = y[:, :16]
    sd16 = {"gn.weight": sd["gn.weight"][:16], "gn.bias": sd["gn.bias"][:16]}
    eps = torch.relu(restate.group_norm4(y16, sd16, "gn"))
    step = restate.ddim_step(eps, ts[5], x, acp.double(), 20)
    got = apply64(y16, sd16["gn.weight"], sd16["gn.bias"], 3, latent=x, c_x=cx[5], c_eps=ce[5])
    assert float((got - step).abs().max()) < 1e-12 * float(step.abs().max()) * 1e3
    assert np.isfinite(float(got.abs().max()))
