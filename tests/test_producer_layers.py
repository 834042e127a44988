"""The producers' two hand-written tensor-core kernels one layer at a time against fp64: convgen_wgmma_kernel (every
Linear of Swin-L and MPViT, every BasicBlock conv, every HAHI neck and FPN ConvModule) through dd_gen_layer, and the
Swin window attention (window_attention_wgmma_kernel and its fp32 CUDA-core check path window_attention_kernel) through
dd_window_attention.  Stage-level tests dilute a one-layer error through the residual stream and the LayerNorms; here
each layer is held to 3e-5 of its own output's max |ref| at the shapes the models run — the deepest K accumulations
(3,456 wgmma into one accumulator in the level-3 HAHI fusion conv), persistent CTAs that take more than one work item,
partial K chunks on the second concat source, partial N tiles, every N-tile width and the 192-wide alternative maps,
pixel-shuffle stores, channel-offset writes into wider planes, both addend orders, every activation, token tails and
stride-2 boxes on odd sources.  Exact checks pin what must not be written, cross-image leakage, run-to-run determinism
and the DD_ERR_RANGE status with its recovery.

The CPU test at the end pins this file's fp64 layer reference (BN fold, ConvT + pixel shuffle, addend order) to the
oracle restatement of the reference's ConvModule and FPN."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import restate

DEV = torch.device("cuda:0")
TOL = 3e-5       # of max |ref|: the bound of the hot-path conv and weight-gradient layer tests
# per output channel when the folded BN scales span 1e-3 .. 1e3: one power-of-two weight scale per layer leaves the
# smallest channels' lo plane in fp16 subnormals (measured 2.7e-4 on a 256 -> 256 3x3; DESIGN.md section 6)
TOL_SPAN_CHANNEL = 5e-4
SPLIT = 16.0     # the producers' fp16 split scale: planes hold 16 x
Y_SENT, P_SENT = -12345.0, -7.0  # what outputs must keep where a layer does not write
ACTS = {0: lambda y: y, 1: torch.relu, 2: F.gelu, 3: F.hardswish}
gpu = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ fp64 reference
def ref_layer(x0, w, x1=None, bias=None, bn=None, add=None, stride=1, transposed=False, act=0, add_first=False):
    """One producer layer in fp64 (any device), NHWC: x0 [M, c0] with a 2-D Linear weight, or [B, H, W, c0] with a conv
    weight [cout, cin, k, k] (pad k // 2; input channels past cin are zero padding) or a ConvT weight [c0, cout, 2, 2]
    (stride 2); x1 concatenated after x0 on the channel axis; eval-BN bn = (weight, bias, mean, var) folded into a
    per-channel scale and shift, else `bias`; the addend before (add_first) or after the activation."""
    x = (x0 if x1 is None else torch.cat([x0, x1], -1)).double()
    w = w.double()
    if w.dim() == 2:
        y = x @ w.t()
    else:
        xc = x.permute(0, 3, 1, 2)
        if transposed:
            y = F.conv_transpose2d(xc, w, stride=2)
        else:
            y = F.conv2d(xc[:, :w.shape[1]], w, stride=stride, padding=w.shape[-1] // 2)
        y = y.permute(0, 2, 3, 1)
    if bn is not None:
        g, b, m, v = (t.double() for t in bn)
        s = g / torch.sqrt(v + 1e-5)
        y = y * s + (b - m * s)
    elif bias is not None:
        y = y + bias.double()
    if add is not None and add_first:
        y = y + add.double()
    y = ACTS[act](y)
    if add is not None and not add_first:
        y = y + add.double()
    return y


def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def _margin(got, ref):
    return ((got.double() - ref).abs().max() / ref.abs().max()).item()


# ------------------------------------------------------------------------------------------------ engine
@pytest.fixture(scope="module")
def eng():
    import diffusiondepth_b200 as dd
    e = dd.DenoiseEngine("swin", 1, (8, 16), (4, 8), 2, DEV, cuda_graph=False)
    yield e
    e.close()


def _bn(c, g, span=None):
    gamma = (10.0 ** (torch.rand(c, generator=g) * 2 * span - span)) if span else 1 + 0.1 * torch.randn(c, generator=g)
    return (gamma, 0.1 * torch.randn(c, generator=g), 0.1 * torch.randn(c, generator=g),
            0.5 + 1.5 * torch.rand(c, generator=g))


def _x(shape, regime, g, real=None):
    """signed O(1), post-ReLU, or signed with max |x| = 3000 (16 x 3000 stays inside the split's 6e4)."""
    x = torch.randn(*shape, generator=g)
    if regime == "relu":
        x = torch.relu(x)
    elif regime == "big":
        x = x * (3000.0 / x.abs().max())
    if real is not None:  # channels past `real` are the zero padding of a padded input (RGB -> 64)
        x[..., real:] = 0
    return x


class Case:
    """One layer: GEMM mode (M tokens) or conv mode (B images of H x W source pixels)."""

    def __init__(self, name, c0, cout, M=None, B=1, H=None, W=None, c1=0, k=1, stride=1, xp=False, cin=0, act=0,
                 add=None, bn=False, bias=False, out="y32", ld_out=0, ch_off=0, n_tile=0, alt_tile=0, bn_span=None,
                 regimes=("signed", "relu", "big")):
        self.__dict__.update(locals())
        del self.__dict__["self"]

    def __repr__(self):
        return self.name

    @property
    def gemm(self):
        return self.M is not None

    def out_hw(self):
        return (self.H, self.W) if self.stride == 1 else ((self.H + 1) // 2, (self.W + 1) // 2)

    def build(self, regime, seed):
        g = torch.Generator().manual_seed(seed)
        Ho, Wo = (None, None) if self.gemm else self.out_hw()
        lead0 = (self.M,) if self.gemm else (self.B, self.H, self.W)
        lead1 = (self.M,) if self.gemm else (self.B, Ho, Wo)
        cin_w = self.cin or self.c0 + self.c1
        x0 = _x(lead0 + (self.c0,), regime, g, real=self.cin or None)
        x1 = _x(lead1 + (self.c1,), regime, g) if self.c1 else None
        if self.xp:
            w = torch.randn(self.c0, self.cout, 2, 2, generator=g) * (0.5 / math.sqrt(self.c0))
        elif self.gemm:
            w = torch.randn(self.cout, cin_w, generator=g) * (0.5 / math.sqrt(cin_w))
        else:
            w = torch.randn(self.cout, cin_w, self.k, self.k, generator=g) * (0.5 / math.sqrt(cin_w * self.k ** 2))
        bn = _bn(self.cout, g, self.bn_span) if self.bn else None
        bias = 0.1 * torch.randn(self.cout, generator=g) if self.bias else None
        add = None
        if self.add:
            ashape = (self.B, 2 * Ho, 2 * Wo, self.cout) if self.xp else lead1 + (self.cout,)
            add = torch.randn(*ashape, generator=g)
        return x0, x1, w, bn, bias, add

    def outputs(self):
        """Sentinel-filled outputs, larger than what the layer writes: GEMM rows up to the whole last 128-row tile,
        rows ld_out wide."""
        width = self.ld_out or self.cout
        if self.gemm:
            shape = ((self.M + 127) // 128 * 128, width)
        elif self.xp:
            shape = (self.B, 2 * self.H, 2 * self.W, self.cout)
        else:
            shape = (self.B,) + self.out_hw() + (width,)
        y = torch.full(shape, Y_SENT, device=DEV) if self.out in ("y32", "both") else False
        p = tuple(torch.full(shape, P_SENT, dtype=torch.float16, device=DEV) for _ in range(2)) \
            if self.out in ("planes", "both") else False
        return y, p

    def written(self, t):
        """The part of an output tensor the layer writes, and the rest (flattened)."""
        if self.gemm:
            region = t[:self.M, self.ch_off:self.ch_off + self.cout]
            mask = torch.ones(t.shape, dtype=torch.bool, device=t.device)
            mask[:self.M, self.ch_off:self.ch_off + self.cout] = False
        else:
            region = t[..., self.ch_off:self.ch_off + self.cout]
            mask = torch.ones(t.shape, dtype=torch.bool, device=t.device)
            mask[..., self.ch_off:self.ch_off + self.cout] = False
        return region, t[mask]

    def run(self, eng, x0, x1, w, bn, bias, add):
        y, p = self.outputs()
        y, p, info = eng.gen_layer(x0.to(DEV), w.to(DEV), x1=None if x1 is None else x1.to(DEV),
                                   bias=None if bias is None else bias.to(DEV),
                                   bn=None if bn is None else [t.to(DEV) for t in bn],
                                   add=None if add is None else add.to(DEV), stride=self.stride, transposed=self.xp,
                                   act=self.act, add_first=self.add == "first", cin=self.cin, ld_out=self.ld_out,
                                   ch_off=self.ch_off, n_tile=self.n_tile, alt_tile=self.alt_tile, y32=y, planes=p)
        return y, p, info

    def reference(self, x0, x1, w, bn, bias, add):
        d = lambda t: None if t is None else t.to(DEV)  # noqa: E731
        return ref_layer(d(x0), d(w), d(x1), d(bias), None if bn is None else [t.to(DEV) for t in bn], d(add),
                         self.stride, self.xp, self.act, self.add == "first")


# Swin-L at a 96 x 160 image: stages of 24x40 / 12x20 / 6x10 / 3x5 tokens per image, C = 192 / 384 / 768 / 1536
SWIN_GEMMS = [
    ("qkv.s0", dict(c0=192, cout=576, bias=True)),
    ("proj.s1", dict(c0=384, cout=384, bias=True, add="after")),
    ("ffn1.s2", dict(c0=768, cout=3072, bias=True, act=2, out="planes")),
    ("ffn2.s3", dict(c0=6144, cout=1536, bias=True, add="after")),          # K = 6144: 1,152 wgmma per accumulator
    ("merge.s2", dict(c0=3072, cout=1536)),
]
TOKENS = [1, 15, 17, 30, 1920, 9000]  # 9000: 71 M tiles, more work items than 132 persistent CTAs

CONVS = [
    # HAHI neck: 1x1 lateral / proj ConvModules, two-source 3x3 fusion (cat never materialises)
    Case("hahi.lateral.0", 192, 192, B=1, H=24, W=40, bn=True, act=1, out="planes"),
    Case("hahi.lateral.2", 768, 768, B=2, H=6, W=10, bn=True, act=1, out="planes"),
    Case("hahi.proj.3", 1536, 512, B=1, H=3, W=5, bn=True, act=1, out="planes"),
    Case("hahi.fusion.0", 512, 192, c1=192, B=1, H=24, W=40, k=3, bn=True, act=1, out="planes"),
    Case("hahi.fusion.2", 768, 768, c1=512, B=2, H=6, W=10, k=3, bn=True, act=1, out="planes"),
    # level 3: (1536 + 512) channels x 9 taps = 288 K iterations = 3,456 wgmma into one accumulator
    Case("hahi.fusion.3", 1536, 1536, c1=512, B=1, H=3, W=5, k=3, bn=True, act=1, out="planes"),
    Case("hahi.fusion.3.12x20", 1536, 1536, c1=512, B=1, H=12, W=20, k=3, bn=True, act=1, out="planes"),
    # MPViT-small widths: partial K chunk of source 0 (216 = 3 x 64 + 24, 288 = 4 x 64 + 32), partial N tile
    Case("hahi.fusion.mpvit216", 216, 216, c1=512, B=2, H=6, W=10, k=3, bn=True, act=1, out="planes"),
    Case("hahi.fusion.mpvit288", 288, 288, c1=512, B=1, H=3, W=5, k=3, bn=True, act=1, out="planes"),
    # FPN: 3x3 laterals (+ top-down addend after the ReLU), ConvT 2x2/s2 with its pixel-shuffle store
    Case("fpn.lateral.3", 1536, 256, B=1, H=3, W=5, k=3, bn=True, act=1, out="both"),  # 2,592 wgmma
    Case("fpn.lateral.2", 768, 256, B=1, H=6, W=10, k=3, bn=True, act=1, add="after", out="both"),  # 1,296 wgmma
    Case("fpn.lateral.0", 192, 256, B=2, H=24, W=40, k=3, bn=True, act=1, add="after", out="both"),
    Case("fpn.up.1", 256, 256, B=2, H=6, W=10, xp=True, bn=True, act=1, add="after", out="y32"),
    Case("fpn.up.0", 256, 256, B=1, H=12, W=20, xp=True, bn=True, act=1, out="y32"),
    # ResNet BasicBlocks on odd sources: stride-2 conv1 on RGB padded to 64 channels, the biased stride-2
    # downsample, conv2 with the residual added before the ReLU
    Case("resnet.conv1.rgb", 64, 64, cin=3, B=2, H=57, W=57, k=3, stride=2, bn=True, act=1, out="planes"),
    Case("resnet.ds.57to29", 64, 128, B=2, H=57, W=57, k=3, stride=2, bias=True, out="y32"),
    Case("resnet.ds.29to15", 128, 256, B=1, H=29, W=29, k=3, stride=2, bias=True, out="y32"),
    Case("resnet.conv1.29to15", 128, 256, B=1, H=29, W=29, k=3, stride=2, bn=True, act=1, out="planes"),
    Case("resnet.conv2", 256, 256, B=1, H=15, W=15, k=3, bn=True, act=1, add="first", out="both"),
    Case("resnet.conv2.s3", 512, 512, B=1, H=8, W=8, k=3, bn=True, act=1, add="first", out="both"),
    # MPViT 1x1 + BN + Hardswish written at a channel offset of the concatenated planes
    Case("mpvit.pw.choff", 216, 216, B=1, H=6, W=10, bn=True, act=3, ld_out=864, ch_off=432, out="planes"),
    Case("mpvit.pw.choff.y32", 288, 288, B=2, H=3, W=5, bn=True, act=3, ld_out=1152, ch_off=288, out="both"),
    Case("mpvit.fc1.gelu", 216, 864, M=60, bias=True, act=2, out="planes"),
    # MPViT encoder Linears at stage 0 of two KITTI 352x1216 images (2 x 176 x 608 tokens): qkv, proj + residual,
    # fc1 + GELU to planes, fc2 + residual into the stage's concatenated planes (3 x 64 wide, path 1 at offset 128)
    Case("mpvit.qkv.s0.M214016", 64, 192, M=214016, bias=True, out="y32"),
    Case("mpvit.proj.s0.M214016", 64, 64, M=214016, bias=True, add="after", out="y32"),
    Case("mpvit.fc1.s0.M214016", 64, 256, M=214016, bias=True, act=2, out="planes"),
    Case("mpvit.fc2.s0.M214016", 256, 64, M=214016, bias=True, add="after", ld_out=192, ch_off=128, out="planes"),
]
# one layer (ffn1 of stage 0: 768 = 3 x 256 = 4 x 192 columns) at every N-tile width; (n_tile, alt_tile, width hit)
WIDTHS = [(64, -1, 64), (128, -1, 128), (192, -1, 192), (256, -1, 256), (0, -1, 256), (0, 1, 192)]


def _check(case, eng, seed, log):
    worst = 0.0
    for regime in case.regimes:
        args = case.build(regime, seed)
        ref = case.reference(*args)
        y, p, info = case.run(eng, *args)
        errs = []
        if y is not None:
            got, rest = case.written(y)
            errs.append(("y32", _margin(got, ref)))
            assert (rest == Y_SENT).all(), f"{case}: fp32 output written outside its rows / channels"
        if p is not None:
            (hi, rest_h), (lo, rest_l) = case.written(p[0]), case.written(p[1])
            errs.append(("planes", _margin((hi.double() + lo.double()) / SPLIT, ref)))
            assert (rest_h == P_SENT).all() and (rest_l == P_SENT).all(), f"{case}: planes written outside"
        for what, e in errs:
            print(f"\n[gen {case} {regime}] {what} {e:.2e} (bound {TOL:.0e}) nt={info['nt']} work={info['work']} "
                  f"grid={info['grid']} launches={info['parts']}")
            assert e <= TOL, (case.name, regime, what, e)
            worst = max(worst, e)
        if case.bn_span:  # per output channel as well: the folded scales span 1e-3 .. 1e3
            got = case.written(y)[0].double() if y is not None else \
                (case.written(p[0])[0].double() + case.written(p[1])[0].double()) / SPLIT
            err_c, ref_c = (got - ref).abs().flatten(0, -2).amax(0), ref.abs().flatten(0, -2).amax(0)
            assert (err_c[ref_c == 0] == 0).all()  # channels the ReLU zeroed everywhere stay exactly zero
            per = (err_c[ref_c > 0] / ref_c[ref_c > 0]).max().item()
            print(f"\n[gen {case} {regime}] worst per-channel {per:.2e} (bound {TOL_SPAN_CHANNEL:.0e})")
            assert per <= TOL_SPAN_CHANNEL, (case.name, regime, per)
        if regime == "signed":  # a repeat call is bit-identical
            y2, p2, _ = case.run(eng, *args)
            if y is not None:
                assert torch.equal(y, y2)
            if p is not None:
                assert torch.equal(p[0], p2[0]) and torch.equal(p[1], p2[1])
    log[case.name] = worst
    print(f"\n[gen {case}] worst margin {worst:.2e} = {worst / TOL:.2f} of the bound")
    return info


_WORST = {}


@gpu
@pytest.mark.parametrize("M", TOKENS)
@pytest.mark.parametrize("name,kw", SWIN_GEMMS, ids=[n for n, _ in SWIN_GEMMS])
def test_swin_gemm_vs_fp64(eng, name, kw, M):
    info = _check(Case(f"{name}.M{M}", M=M, **kw), eng, M * 31 + kw["c0"], _WORST)
    if M == 9000:
        assert info["work"] > info["grid"], info  # persistent CTAs take a second work item


@gpu
@pytest.mark.parametrize("case", CONVS, ids=repr)
def test_producer_conv_vs_fp64(eng, case):
    _check(case, eng, case.c0 * 7 + case.cout + (case.H or 0), _WORST)


@gpu
def test_bn_scales_per_channel(eng):
    """Folded eval-BN scales spanning 1e-3 .. 1e3 (one power-of-two weight scale for the whole layer): every output
    channel is held to the bound of its own max."""
    for case in (Case("bn.span.1x1", 192, 192, B=1, H=24, W=40, bn=True, bn_span=3, act=0, regimes=("signed",)),
                 Case("bn.span.3x3", 256, 256, B=1, H=12, W=20, k=3, bn=True, bn_span=3, act=1, out="both",
                      regimes=("signed", "relu"))):
        _check(case, eng, 4242, _WORST)


@gpu
def test_every_n_tile_width(eng):
    hit = set()
    for n_tile, alt, want in WIDTHS:
        case = Case(f"ffn1.s0.nt{n_tile}.alt{alt}", 192, 768, M=1920, bias=True, act=2, out="both", n_tile=n_tile,
                    alt_tile=alt, regimes=("signed",))
        info = _check(case, eng, 99, _WORST)
        assert info["nt"] == want, (n_tile, alt, info)
        hit.add((want, alt))
    assert {64, 128, 192, 256} <= {w for w, _ in hit} and (192, 1) in hit


@gpu
@pytest.mark.parametrize("case", [
    Case("leak.fusion", 512, 192, c1=192, B=2, H=12, W=20, k=3, act=1, out="both"),
    Case("leak.resnet.s2", 64, 128, B=3, H=29, W=29, k=3, stride=2, act=0, out="both"),
    Case("leak.convT", 256, 256, B=2, H=6, W=10, xp=True, act=1, out="y32"),
], ids=repr)
def test_no_leak_across_images(eng, case):
    """Source data in image 0 only: every other image's output is exactly zero (no bias / BN / addend)."""
    x0, x1, w, _, _, _ = case.build("signed", 5)
    x0[1:] = 0
    if x1 is not None:
        x1[1:] = 0
    y, p, _ = case.run(eng, x0, x1, w, None, None, None)
    for t in ([y] if y is not None else []) + (list(p) if p is not None else []):
        assert t[1:].abs().max().item() == 0.0
        assert t[0].abs().max().item() > 0.0


@gpu
@pytest.mark.parametrize("case", [
    Case("range.fusion.mpvit216", 216, 216, c1=512, B=2, H=6, W=10, k=3, bn=True, act=1, out="planes"),
    Case("range.ffn2.y32", 6144, 1536, M=30, bias=True, add="after", out="y32"),
], ids=repr)
def test_gen_status_and_recovery(eng, case):
    """A NaN or a value past the split's range in either source is DD_ERR_RANGE; the next clean call equals a call made
    before, bit for bit."""
    from diffusiondepth_b200 import _cabi
    args = list(case.build("signed", 11))
    y0, p0, _ = case.run(eng, *args)
    for src, val in ((0, float("nan")), (0, 5000.0)) + (((1, float("nan")),) if args[1] is not None else ()):
        bad = list(args)
        bad[src] = args[src].clone()
        bad[src].view(-1)[-1] = val
        with pytest.raises(_cabi.EngineError, match="DD_ERR_RANGE"):
            case.run(eng, *bad)
        y1, p1, _ = case.run(eng, *args)
        if y0 is not None:
            assert torch.equal(y0, y1)
        if p0 is not None:
            assert torch.equal(p0[0], p1[0]) and torch.equal(p0[1], p1[1])


# ------------------------------------------------------------------------------------------------ window attention
def _rpi(ws=7):
    c = torch.stack(torch.meshgrid(torch.arange(ws), torch.arange(ws), indexing="ij")).flatten(1)
    rel = c[:, :, None] - c[:, None, :] + (ws - 1)
    return rel[0] * (2 * ws - 1) + rel[1]


def _attn_case(B, H, W, nH, shift, peak, seed):
    """x, qkv weight / bias in fp64 (q / k rows scaled by `peak`: small = flat softmax, large = peaked), the table
    N(0, 2); returns the engine's fp32 qkv / bias / table and the restated reference's fp64 output (proj = identity)."""
    g = torch.Generator().manual_seed(seed)
    C = 32 * nH
    x = torch.randn(B, H * W, C, generator=g, dtype=torch.float64)
    w = torch.randn(3 * C, C, generator=g, dtype=torch.float64) / math.sqrt(C)
    w[:2 * C] *= peak
    b = 0.3 * torch.randn(3 * C, generator=g, dtype=torch.float64)
    table = 2.0 * torch.randn(169, nH, generator=g, dtype=torch.float64)
    p = "attn."
    sd = {p + "w_msa.qkv.weight": w, p + "w_msa.qkv.bias": b, p + "w_msa.relative_position_bias_table": table,
          p + "w_msa.relative_position_index": _rpi(), p + "w_msa.proj.weight": torch.eye(C, dtype=torch.float64),
          p + "w_msa.proj.bias": torch.zeros(C, dtype=torch.float64)}
    ref = restate._shift_window_msa(sd, x, (H, W), p, nH, 7, shift)  # [B, H*W, C]
    qkv = (x @ w.t() + b).reshape(B * H * W, 3 * C)
    return qkv.float(), b.float(), table.float(), ref


ATTN = [  # (B, H, W, nH)
    (1, 7, 7, 2), (2, 3, 5, 6), (3, 13, 9, 12), (3, 24, 40, 12), (1, 56, 56, 12), (2, 24, 40, 6), (1, 13, 9, 3),
]


def _attn_margin(out, ref, B, nH):
    """Worst (image, head) slice error over that slice's max |ref|."""
    o = out.double().cpu().reshape(B, -1, nH, 32)
    r = ref.reshape(B, -1, nH, 32)
    return ((o - r).abs().amax((1, 3)) / r.abs().amax((1, 3))).max().item()


@gpu
@pytest.mark.parametrize("shift", [0, 3])
@pytest.mark.parametrize("B,H,W,nH", ATTN, ids=[f"B{b}_{h}x{w}_nH{n}" for b, h, w, n in ATTN])
def test_window_attention_vs_fp64(eng, B, H, W, nH, shift):
    kernels = (1,) if nH & 1 else (1, 2)
    for peak in (0.1, 3.0):
        qkv, b, table, ref = _attn_case(B, H, W, nH, shift, peak, B * 1000 + H * 31 + W + nH + shift)
        outs = {}
        for k in kernels:
            out, info = eng.window_attention(qkv.to(DEV), b.to(DEV), table.to(DEV), B, (H, W), nH, shift, kernel=k)
            e = _attn_margin(out, ref, B, nH)
            name = {1: "simt", 2: "wgmma"}[k]
            print(f"\n[attn B{B} {H}x{W} nH{nH} shift{shift} peak{peak} {name}] {e:.2e} (bound {TOL:.0e}) "
                  f"work={info['work']} grid={info['grid']}")
            assert e <= TOL, (name, peak, e)
            _WORST[f"attn.{H}x{W}.nH{nH}.{name}"] = max(_WORST.get(f"attn.{H}x{W}.nH{nH}.{name}", 0.0), e)
            outs[k] = out
            if k == 2 and B * ((H + 6) // 7) * ((W + 6) // 7) * nH // 2 > 2 * _sms():
                assert info["work"] > info["grid"] and info["work"] % info["grid"] != 0, info
            if peak == 3.0:  # a repeat call is bit-identical
                assert torch.equal(out, eng.window_attention(qkv.to(DEV), b.to(DEV), table.to(DEV), B, (H, W), nH,
                                                             shift, kernel=k)[0])
        if len(outs) == 2:  # the two kernels agree with each other as closely as each does with fp64
            e = _attn_margin(outs[2], outs[1].double().cpu().reshape(B, H * W, -1), B, nH)
            assert e <= TOL, ("simt vs wgmma", peak, e)


@gpu
def test_window_attention_work_exceeds_grid(eng):
    """The shapes above include persistent wgmma CTAs that take a second (and a partial third) head pair, reusing
    their shared tiles and token tables."""
    qkv, b, table, _ = _attn_case(1, 56, 56, 12, 3, 1.0, 3)
    _, info = eng.window_attention(qkv.to(DEV), b.to(DEV), table.to(DEV), 1, (56, 56), 12, 3, kernel=2)
    assert info["work"] == 64 * 6 and info["grid"] == 2 * _sms() and info["work"] > info["grid"], info


@gpu
@pytest.mark.parametrize("kernel", [1, 2])
def test_window_attention_status_and_recovery(eng, kernel):
    from diffusiondepth_b200 import _cabi
    B, H, W, nH = 2, 13, 9, 6
    qkv, b, table, _ = _attn_case(B, H, W, nH, 3, 1.0, 77)
    qkv, b, table = qkv.to(DEV), b.to(DEV), table.to(DEV)
    out0, _ = eng.window_attention(qkv, b, table, B, (H, W), nH, 3, kernel=kernel)
    C = 32 * nH
    bad_nan = qkv.clone()
    bad_nan[B * H * W - 1, 2 * C + 5] = float("nan")  # one v entry of the last token
    bad_big = qkv.clone()
    bad_big[:, 2 * C:2 * C + 32] = 5000.0             # head 0's v everywhere: 16 x 5000 is past the split's range
    for bad in (bad_nan, bad_big):
        with pytest.raises(_cabi.EngineError, match="DD_ERR_RANGE"):
            eng.window_attention(bad, b, table, B, (H, W), nH, 3, kernel=kernel)
        out1, _ = eng.window_attention(qkv, b, table, B, (H, W), nH, 3, kernel=kernel)
        assert torch.equal(out0, out1)


# ------------------------------------------------------------------------------------------------ CPU: the reference
def test_reference_matches_restated_modules():
    """ref_layer's fp64 BN fold, ConvT + pixel shuffle and addend order equal the oracle restatement's ConvModule
    (1x1 and 3x3 over a concatenation) and its FPN (3x3 laterals + ConvT top-down, add after the ReLU) to 1e-12."""
    g = torch.Generator().manual_seed(0)
    dt = torch.float64
    sd = {}

    def bn(prefix, c):
        w_, b_, m_, v_ = _bn(c, g, span=2)
        sd.update({prefix + ".weight": w_.to(dt), prefix + ".bias": b_.to(dt), prefix + ".running_mean": m_.to(dt),
                   prefix + ".running_var": v_.to(dt)})
        return [sd[prefix + s] for s in (".weight", ".bias", ".running_mean", ".running_var")]

    # ConvModule, 3x3 over cat([a, b]) and 1x1
    a, b = torch.randn(2, 24, 7, 9, generator=g, dtype=dt), torch.randn(2, 40, 7, 9, generator=g, dtype=dt)
    for k, pad in ((3, 1), (1, 0)):
        sd["m.conv.weight"] = torch.randn(32, 64, k, k, generator=g, dtype=dt)
        bnp = bn("m.bn", 32)
        want = restate._conv_module(torch.cat([a, b], 1), sd, "m", padding=pad).permute(0, 2, 3, 1)
        got = ref_layer(a.permute(0, 2, 3, 1), sd["m.conv.weight"], x1=b.permute(0, 2, 3, 1), bn=bnp, act=1)
        assert (got - want).abs().max().item() <= 1e-12 * want.abs().max().item()
    # FPN over two levels at exactly 2x (the adaptive pool is the identity there)
    f0, f1 = torch.randn(2, 16, 10, 12, generator=g, dtype=dt), torch.randn(2, 24, 5, 6, generator=g, dtype=dt)
    p = "depth_head."
    sd[p + "conv_lateral.0.0.weight"] = torch.randn(256, 16, 3, 3, generator=g, dtype=dt)
    sd[p + "conv_lateral.1.0.weight"] = torch.randn(256, 24, 3, 3, generator=g, dtype=dt)
    sd[p + "conv_up.0.0.weight"] = torch.randn(256, 256, 2, 2, generator=g, dtype=dt) * 0.05
    bn0, bn1, bnu = bn(p + "conv_lateral.0.1", 256), bn(p + "conv_lateral.1.1", 256), bn(p + "conv_up.0.1", 256)
    want = restate.fpn_condition(sd, [f0, f1]).permute(0, 2, 3, 1)
    lat1 = ref_layer(f1.permute(0, 2, 3, 1), sd[p + "conv_lateral.1.0.weight"], bn=bn1, act=1)
    up = ref_layer(lat1, sd[p + "conv_up.0.0.weight"], bn=bnu, act=1, transposed=True)
    got = ref_layer(f0.permute(0, 2, 3, 1), sd[p + "conv_lateral.0.0.weight"], bn=bn0, act=1, add=up)
    assert (got - want).abs().max().item() <= 1e-12 * want.abs().max().item()
