"""MPViT's hand-written kernels outside the GEMM path one layer at a time against fp64: the factorised attention
(ksoftmax_partial -> ktv_partial -> ktv_combine -> factor_att_apply) through dd_factor_attention, the depthwise conv
(dwconv_nhwc_kernel) through dd_depthwise_conv and the any-width LayerNorm (ln_split_generic_kernel) through
dd_layer_norm, each packed and launched by the backbone's own host code.  Stage-level tests dilute a one-layer error
through residuals and LayerNorms and only ever ran small images; here each layer is held to 3e-5 of its own output's max
|ref| (attention: of each (image, head) slice's max) at every MPViT stage width (Ch = 8 ... 60: the float4 channel groups
that straddle two heads with different crpe windows, two channel trips of ksoftmax_partial above 256, every heads-per-
block grouping of ktv_partial), at token counts from one token to the real stage-0 grids of NYU and KITTI images
(> 16,384 tokens: chunks of 65 ... 418 tokens, not multiples of the 32-token staging tile, up to 256 chunks), and with
k columns whose exp underflows for most tokens or whose maximum sits in the last token of the last chunk.  Exact checks
pin run-to-run determinism, that an image of a batch equals the same image run alone, and the DD_ERR_RANGE status with
its recovery."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import restate

DEV = torch.device("cuda:0")
TOL = 3e-5       # of max |ref|: the bound of the other layer tests
SPLIT = 16.0     # the producers' fp16 split scale: planes hold 16 x
HEADS = 8
WINDOWS = ((3, 2), (5, 3), (7, 3))  # crpe window: heads
gpu = pytest.mark.gpu
_WORST = {}


@pytest.fixture(scope="module")
def eng():
    import diffusiondepth_b200 as dd
    e = dd.DenoiseEngine("swin", 1, (8, 16), (4, 8), 2, DEV, cuda_graph=False)
    yield e
    e.close()
    if _WORST:
        print("\n[mpvit layers] worst margin per family:")
        for fam in sorted({k.split(":")[0] for k in _WORST}):
            k = max((k for k in _WORST if k.split(":")[0] == fam), key=_WORST.get)
            print(f"  {fam}: {_WORST[k]:.2e} ({k})")


def _log(key, e):
    _WORST[key] = max(_WORST.get(key, 0.0), e)


def chunking(N):
    """The host's token chunking of the factorised attention: (tokens per chunk, chunks)."""
    tpc = max(64, -(-N // 256))
    return tpc, -(-N // tpc)


def heads_per_block(Ch):
    return max(1, min(HEADS, min(4096 // (Ch * Ch), 160 // Ch)))


# ------------------------------------------------------------------------------------------------ factorised attention
def _att_inputs(B, H, W, C, regime, seed):
    """qkv [B*H*W, 3C] fp32 on the device and the crpe weights / biases in the reference layout.  k regimes: flat
    (softmax close to uniform), peaked (logits N(0, 25^2): a column spans > 150, exp underflows for most tokens), edge
    (one column's max in the last token of the last chunk, one column's max in chunk 0 with every later chunk 120
    below it)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    N, Ch = H * W, C // HEADS
    q, k, v = (torch.randn(B, N, C, generator=g, device=DEV) for _ in range(3))
    if regime == "flat":
        k *= 0.05
    elif regime == "peaked":
        k *= 25.0
    else:
        k *= 0.5
        tpc, _ = chunking(N)
        k[:, N - 1, 1] = 30.0                    # head 0: max in the very last token
        cb = C - Ch                              # last head: max in chunk 0, nothing survives exp in later chunks
        k[:, tpc:, cb] = -100.0
        k[:, 0, cb] = 20.0
        k[:, N // 2, 3 * Ch + 2] = 25.0          # a 5 x 5 head: one token in the middle dominates
    # crpe on the flat regime; zero elsewhere, so that q (k^T v) alone is measured (q * crpe(v) would dominate it)
    gc = torch.Generator().manual_seed(seed + 1)
    cs = 1.0 if regime == "flat" else 0.0
    cw = [(torch.randn(nh * Ch, 1, win, win, generator=gc) * (cs * 0.5 / win)).to(DEV) for win, nh in WINDOWS]
    cb_ = [(cs * 0.1 * torch.randn(nh * Ch, generator=gc)).to(DEV) for _, nh in WINDOWS]
    return torch.cat([q, k, v], -1).reshape(B * N, 3 * C), cw, cb_


def ref_factor_att(qkv, cw, cb, B, H, W):
    """restate.factor_att_crpe (the oracle's restatement of the reference module, pinned by the MPViT goldens) in fp64
    on qkv's device: [B, H*W, C]."""
    C = qkv.shape[1] // 3
    t = qkv.double().reshape(B, H * W, 3, HEADS, C // HEADS).permute(2, 0, 3, 1, 4)
    sd = {}
    for i in range(3):
        sd[f"crpe.conv_list.{i}.weight"] = cw[i].double()
        sd[f"crpe.conv_list.{i}.bias"] = cb[i].double()
    return restate.factor_att_crpe(t[0], t[1], t[2], (H, W), sd, "", WINDOWS)


def _head_margin(out, ref, B):
    """Worst (image, head) slice error over that slice's max |ref|."""
    C = ref.shape[-1]
    o = out.double().reshape(B, -1, HEADS, C // HEADS)
    r = ref.reshape(B, -1, HEADS, C // HEADS)
    return ((o - r).abs().amax((1, 3)) / r.abs().amax((1, 3))).max().item()


def _check_att(eng, B, H, W, C, seed, regimes=("flat", "peaked", "edge")):
    info = None
    for regime in regimes:
        qkv, cw, cb = _att_inputs(B, H, W, C, regime, seed)
        ref = ref_factor_att(qkv, cw, cb, B, H, W)
        out, info = eng.factor_attention(qkv, cw, cb, B, (H, W))
        e = _head_margin(out, ref, B)
        print(f"\n[fa C{C} B{B} {H}x{W} {regime}] {e:.2e} (bound {TOL:.0e}) tpc={info['tpc']} "
              f"chunks={info['chunks']} HB={info['hb']} grid={info['grid']}")
        _log(f"factor_att:C{C}.{H}x{W}.{regime}", e)
        assert e <= TOL, (C, H, W, regime, e)
        if regime == "peaked":  # a repeat call is bit-identical
            assert torch.equal(out, eng.factor_attention(qkv, cw, cb, B, (H, W))[0])
        del ref, out, qkv
    N, Ch = H * W, C // HEADS
    tpc, chunks = chunking(N)
    grid = B * -(-H // 8) * -(-W // 16) * -(-(C // 4) // 16)
    assert info == {"tpc": tpc, "chunks": chunks, "hb": heads_per_block(Ch), "grid": grid}, info
    return info


WIDTHS = [64, 96, 128, 176, 216, 224, 288, 368, 480]  # every MPViT factory's stage widths: Ch = 8 ... 60
TINY = [(1, 1), (1, 7), (2, 3), (5, 7)]                # chunks with fewer tokens than ksoftmax_partial has slices


@gpu
@pytest.mark.parametrize("C", WIDTHS)
def test_factor_attention_small_vs_fp64(eng, C):
    for H, W in TINY + [(35, 53)]:
        _check_att(eng, 2, H, W, C, C * 7 + H * 31 + W)


# (C, B, H, W): every width just past the 16,384-token boundary (tpc 65); the boundary itself (tpc 64, 256 chunks);
# the stage-0 grids of NYU 228x304 / 480x640 and KITTI 352x1216 images (tpc 68 / 300 / 418)
LARGE = [(C, 1, 113, 145) for C in WIDTHS] + [
    (64, 1, 128, 128), (216, 1, 128, 128),
    (64, 2, 114, 152), (128, 1, 114, 152),
    (64, 1, 240, 320), (128, 1, 240, 320),
    (64, 2, 176, 608), (128, 2, 176, 608),
]


@gpu
@pytest.mark.parametrize("C,B,H,W", LARGE, ids=[f"C{c}_B{b}_{h}x{w}" for c, b, h, w in LARGE])
def test_factor_attention_large_vs_fp64(eng, C, B, H, W):
    info = _check_att(eng, B, H, W, C, C + B * 1000 + H * 31 + W)
    N = H * W
    if N > 16384:
        assert info["tpc"] > 64 and info["tpc"] % 32 != 0, info  # chunks are no multiple of the 32-token tile
    else:
        assert info["tpc"] == 64 and info["chunks"] == 256, info
    if (H, W) == (176, 608):
        assert info["chunks"] == 256 and info["tpc"] == 418, info


@gpu
@pytest.mark.parametrize("C,H,W", [(64, 114, 152), (176, 113, 145), (480, 5, 7)])
def test_factor_attention_batch_equals_single_image(eng, C, H, W):
    """The chunking depends on H W only: image b of a batch is bit-identical to the same image run alone."""
    qkv, cw, cb = _att_inputs(2, H, W, C, "peaked", 3)
    N = H * W
    out, _ = eng.factor_attention(qkv, cw, cb, 2, (H, W))
    for b in range(2):
        alone, _ = eng.factor_attention(qkv[b * N:(b + 1) * N], cw, cb, 1, (H, W))
        assert torch.equal(out[b * N:(b + 1) * N], alone), b


@gpu
def test_factor_attention_status_and_recovery(eng):
    """A NaN or +inf in k (fmaxf drops a NaN from the column max: only the sums carry it) and a v that pushes 16 x out
    past 6e4 are DD_ERR_RANGE; the next clean call equals a call made before, bit for bit."""
    from diffusiondepth_b200 import _cabi
    B, H, W, C = 2, 23, 37, 96
    N, Ch = H * W, C // HEADS
    qkv, cw, cb = _att_inputs(B, H, W, C, "flat", 17)
    out0, _ = eng.factor_attention(qkv, cw, cb, B, (H, W))
    bads = []
    for val in (float("nan"), float("inf")):
        for tok in (N + 300, N + 301):  # image 1, two different token slices of ksoftmax_partial
            bad = qkv.clone()
            bad[tok, C + 7] = val
            bads.append(bad)
    bad = qkv.clone()
    bad[:, 2 * C:2 * C + Ch] = 1e5       # head 0's v everywhere
    bads.append(bad)
    for bad in bads:
        with pytest.raises(_cabi.EngineError, match="DD_ERR_RANGE"):
            eng.factor_attention(bad, cw, cb, B, (H, W))
        out1, _ = eng.factor_attention(qkv, cw, cb, B, (H, W))
        assert torch.equal(out0, out1)


# ------------------------------------------------------------------------------------------------ depthwise conv
def ref_dw(x, w, bias=None, bn=None, stride=1, act=0, residual=False):
    """Depthwise 3x3 (pad 1) in fp64, NHWC, then eval-BN folded or bias, + x (residual), Hardswish (act 3)."""
    xc = x.double().permute(0, 3, 1, 2)
    y = F.conv2d(xc, w.double(), None, stride, 1, 1, x.shape[-1])
    if bn is not None:
        g, b, m, v = (t.double()[:, None, None] for t in bn)
        s = g / torch.sqrt(v + 1e-5)
        y = y * s + (b - m * s)
    elif bias is not None:
        y = y + bias.double()[:, None, None]
    if residual:
        y = y + xc
    if act == 3:
        y = F.hardswish(y)
    return y.permute(0, 2, 3, 1)


# (name, B, H, W, C, stride, affine, act, residual, out): H x W the source grid
DW = [
    ("pe.kitti.352x1216.s2", 1, 352, 1216, 64, 2, None, 0, False, "planes"),  # > 3 grid-stride trips
    ("pe.nyu.228x304.s2", 2, 228, 304, 64, 2, None, 0, False, "planes"),
    ("pe.35x53.s2", 2, 35, 53, 216, 2, None, 0, False, "planes"),              # odd source -> 18 x 27
    ("pe.18x27.s2", 1, 18, 27, 288, 2, None, 0, False, "both"),
    ("cpe.114x152", 2, 114, 152, 64, 1, "bias", 0, True, "y32"),
    ("cpe.176x608", 1, 176, 608, 128, 1, "bias", 0, True, "y32"),              # > 3 grid-stride trips
    ("cpe.18x27", 1, 18, 27, 216, 1, "bias", 0, True, "both"),
    ("invres.57x76.bn", 2, 57, 76, 128, 1, "bn", 3, False, "planes"),
    ("invres.9x14.bn", 1, 9, 14, 480, 1, "bn", 3, False, "both"),
    ("invres.35x53.bn", 1, 35, 53, 368, 1, "bn", 3, False, "planes"),
]


def _dw_inputs(B, H, W, C, affine, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, H, W, C, generator=g)
    w = torch.randn(C, 1, 3, 3, generator=g) * 0.4
    bias = 0.2 * torch.randn(C, generator=g) if affine == "bias" else None
    bn = None
    if affine == "bn":  # folded scales spread over 1e-2 .. 1e2
        bn = (10.0 ** (torch.rand(C, generator=g) * 4 - 2), 0.1 * torch.randn(C, generator=g),
              0.1 * torch.randn(C, generator=g), 0.5 + 1.5 * torch.rand(C, generator=g))
    d = lambda t: None if t is None else t.to(DEV)  # noqa: E731
    return d(x), d(w), d(bias), None if bn is None else [t.to(DEV) for t in bn]


@gpu
@pytest.mark.parametrize("name,B,H,W,C,stride,affine,act,residual,out", DW, ids=[c[0] for c in DW])
def test_depthwise_conv_vs_fp64(eng, name, B, H, W, C, stride, affine, act, residual, out):
    x, w, bias, bn = _dw_inputs(B, H, W, C, affine, C + H * 7 + W)
    ref = ref_dw(x, w, bias, bn, stride, act, residual)
    y, p, info = eng.depthwise_conv(x, w, bias=bias, bn=bn, stride=stride, act=act, residual=residual,
                                    y32=out in ("y32", "both"), planes=out in ("planes", "both"))
    outs = ([("y32", y.double())] if y is not None else []) + \
        ([("planes", (p[0].double() + p[1].double()) / SPLIT)] if p is not None else [])
    for what, got in outs:
        assert got.shape == ref.shape
        e = ((got - ref).abs().max() / ref.abs().max()).item()
        # per channel as well: the folded BN scales span four decades
        err_c, ref_c = (got - ref).abs().flatten(0, -2).amax(0), ref.abs().flatten(0, -2).amax(0)
        per = (err_c / ref_c.clamp_min(1e-30)).max().item()
        print(f"\n[dw {name} {what}] {e:.2e}, per channel {per:.2e} (bound {TOL:.0e}) grid={info['grid']} "
              f"work={info['work']}")
        _log(f"dwconv:{name}.{what}", per)
        assert e <= TOL and per <= TOL, (name, what, e, per)
    assert info["work"] == B * ref.shape[1] * ref.shape[2] * C // 4
    if name in ("pe.kitti.352x1216.s2", "cpe.176x608"):
        assert info["work"] > 3 * 256 * info["grid"], info  # the grid-stride loop takes more than three trips
    y2, p2, _ = eng.depthwise_conv(x, w, bias=bias, bn=bn, stride=stride, act=act, residual=residual,
                                   y32=y is not None, planes=p is not None)
    assert (y is None or torch.equal(y, y2)) and (p is None or (torch.equal(p[0], p2[0]) and torch.equal(p[1], p2[1])))


@gpu
def test_depthwise_conv_status_and_recovery(eng):
    from diffusiondepth_b200 import _cabi
    x, w, bias, _ = _dw_inputs(2, 18, 27, 216, "bias", 5)
    y0, p0, _ = eng.depthwise_conv(x, w, bias=bias, residual=True, planes=True)
    for val in (float("nan"), 5000.0):
        bad = x.clone()
        bad[1, 17, 26, 215] = val
        with pytest.raises(_cabi.EngineError, match="DD_ERR_RANGE"):
            eng.depthwise_conv(bad, w, bias=bias, residual=True, planes=True)
        y1, p1, _ = eng.depthwise_conv(x, w, bias=bias, residual=True, planes=True)
        assert torch.equal(y0, y1) and torch.equal(p0[0], p1[0]) and torch.equal(p0[1], p1[1])


# ------------------------------------------------------------------------------------------------ LayerNorm
LN_WIDTHS = [64, 96, 128, 176, 216, 256, 288, 480, 512]  # at and around every template bucket edge (64 / 128 / 256 / 512)


def _ln_inputs(M, C, seed):
    """Rows: signed with an offset; 100 rows of mean 1e3 and std 1e-2; constant rows (variance 0)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, C, generator=g) * 2 + 0.5
    x[:100] = 1e3 + 1e-2 * torch.randn(100, C, generator=g)
    x[100:110] = torch.randn(10, 1, generator=g) * 3
    x[110] = 0.0
    x[111] = 1e3
    gamma = 1 + 0.3 * torch.randn(C, generator=g)
    beta = 0.2 * torch.randn(C, generator=g)
    return x.to(DEV), gamma.to(DEV), beta.to(DEV)


@gpu
@pytest.mark.parametrize("C", LN_WIDTHS)
def test_layer_norm_vs_fp64(eng, C):
    M = 1001  # not a multiple of the 8 tokens per block
    x, gamma, beta = _ln_inputs(M, C, C)
    for eps in (1e-6, 1e-5):
        ref = F.layer_norm(x.double(), (C,), gamma.double(), beta.double(), eps)
        out = eng.layer_norm(x, gamma, beta, eps)
        per_row = ((out.double() - ref).abs().amax(1) / ref.abs().amax(1))
        e = per_row.max().item()
        print(f"\n[ln C{C} eps{eps:.0e}] worst row {e:.2e} (bound {TOL:.0e}); mean-1e3 rows "
              f"{per_row[:100].max().item():.2e}, constant rows {per_row[100:112].max().item():.2e}")
        _log(f"layernorm:C{C}.eps{eps:.0e}", e)
        assert e <= TOL, (C, eps, e)
        assert torch.equal(out, eng.layer_norm(x, gamma, beta, eps))


@gpu
def test_layer_norm_status_and_recovery(eng):
    from diffusiondepth_b200 import _cabi
    x, gamma, beta = _ln_inputs(203, 216, 9)
    out0 = eng.layer_norm(x, gamma, beta)
    bad = x.clone()
    bad[202, 215] = float("nan")
    with pytest.raises(_cabi.EngineError, match="DD_ERR_RANGE"):
        eng.layer_norm(bad, gamma, beta)
    assert torch.equal(out0, eng.layer_norm(x, gamma, beta))


# ------------------------------------------------------------------------------------------------ argument checks
@gpu
def test_mpvit_layers_reject_bad_arguments(eng):
    from diffusiondepth_b200 import _cabi
    cw = [torch.zeros(8, 1, k, k, device=DEV) for k in (3, 5, 7)]
    cb = [torch.zeros(8, device=DEV) for _ in range(3)]
    for C, B, status in ((100, 1, "DD_ERR_UNSUPPORTED"), (520, 1, "DD_ERR_UNSUPPORTED"), (64, 0, "DD_ERR_INVALID")):
        with pytest.raises(_cabi.EngineError, match=status):
            eng.factor_attention(torch.zeros(max(B, 1) * 12, 3 * C, device=DEV), cw, cb, B, (3, 4))
    x, w, _, bn = _dw_inputs(1, 6, 7, 64, "bn", 1)
    with pytest.raises(_cabi.EngineError, match="DD_ERR_UNSUPPORTED"):  # channels not a multiple of 4
        eng.depthwise_conv(x[..., :6], w[:6])
    for kw in (dict(stride=2, residual=True), dict(act=1), dict(stride=3), dict(bn=bn, bias=bn[1])):
        with pytest.raises(_cabi.EngineError, match="DD_ERR_INVALID"):
            eng.depthwise_conv(x, w, **kw)
    xl = torch.zeros(9, 520, device=DEV)
    with pytest.raises(_cabi.EngineError, match="DD_ERR_UNSUPPORTED"):
        eng.layer_norm(xl, xl[0], xl[0])
    with pytest.raises(_cabi.EngineError, match="DD_ERR_INVALID"):
        eng.layer_norm(xl[:, :64], xl[0, :64], xl[0, :64], eps=0.0)


# ------------------------------------------------------------------------------------------------ CPU: the reference
def test_factor_att_reference_is_the_module():
    """ref_factor_att's head layout and window grouping agree with a direct fp64 statement of FactorAtt_ConvRelPosEnc
    (softmax of k over the tokens, k^T v, q (k^T v) Ch^-0.5 + q * per-head-group depthwise conv of v)."""
    B, H, W, C = 2, 5, 6, 64
    Ch, N = C // HEADS, H * W
    g = torch.Generator().manual_seed(0)
    qkv = torch.randn(B * N, 3 * C, generator=g)
    cw = [torch.randn(nh * Ch, 1, win, win, generator=g) for win, nh in WINDOWS]
    cb = [torch.randn(nh * Ch, generator=g) for _, nh in WINDOWS]
    got = ref_factor_att(qkv, cw, cb, B, H, W)
    t = qkv.double().reshape(B, N, 3, C)
    q, k, v = t[:, :, 0], t[:, :, 1], t[:, :, 2]
    want = torch.empty(B, N, C, dtype=torch.float64)
    h = 0
    for (win, nh), w_, b_ in zip(WINDOWS, cw, cb):
        for j in range(nh):
            sl = slice(h * Ch, (h + 1) * Ch)
            ktv = torch.softmax(k[:, :, sl], 1).transpose(1, 2) @ v[:, :, sl]
            vi = v[:, :, sl].transpose(1, 2).reshape(B, Ch, H, W)
            conv = F.conv2d(vi, w_[j * Ch:(j + 1) * Ch].double(), b_[j * Ch:(j + 1) * Ch].double(), padding=win // 2,
                            groups=Ch).reshape(B, Ch, N).transpose(1, 2)
            want[:, :, sl] = (q[:, :, sl] @ ktv) / math.sqrt(Ch) + q[:, :, sl] * conv
            h += 1
    assert (got - want).abs().max().item() <= 1e-12 * want.abs().max().item()
