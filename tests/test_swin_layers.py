"""Swin-L's hand-written kernels outside the GEMMs and the window attention one layer at a time against fp64: the patch
embedding (patch_embed_kernel: 4x4/s4 conv, bias, LayerNorm(192)) through dd_swin_patch_embed, the block and
stage-output LayerNorms (ln_split_kernel, with the neck's fp32 NCHW copy) through dd_swin_layer_norm and the patch
merging (merge_ln_split_kernel: 2x2 unfold gather, zero padding, LayerNorm(4C)) through dd_swin_patch_merge, each
launched by the backbone's own host code.  The stage-level tests run token grids that are all even and divisible by 4;
here each layer is held to 3e-5 of its own token's max |ref| at odd and padded grids (the patch embedding's right /
bottom padding, partial and one-token 32-token segments, the merge's odd last row and column), at the full KITTI
352x1216 shapes, and on tokens whose mean dominates their spread (1e3 +- 1e-2), constant tokens and tokens with one
massive channel.  Exact checks pin run-to-run determinism, that a NaN pixel poisons its own token only, and the
DD_ERR_RANGE status with its recovery.  A stage-level companion runs the whole backbone at odd grids.

The CPU test at the end pins this file's three fp64 references to the oracle restatement of the reference's
SwinTransformer."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from oracle import restate

DEV = torch.device("cuda:0")
TOL = 3e-5       # of each token's max |ref|: the bound of the other layer tests
E = 192          # Swin-L's embedding width
gpu = pytest.mark.gpu
_WORST = {}


@pytest.fixture(scope="module")
def eng():
    import diffusiondepth_b200 as dd
    e = dd.DenoiseEngine("swin", 1, (8, 16), (4, 8), 2, DEV, cuda_graph=False)
    yield e
    e.close()
    if _WORST:
        print("\n[swin layers] worst margin per family:")
        for fam in sorted({k.split(":")[0] for k in _WORST}):
            k = max((k for k in _WORST if k.split(":")[0] == fam), key=_WORST.get)
            print(f"  {fam}: {_WORST[k]:.2e} ({k})")


def _log(key, e):
    _WORST[key] = max(_WORST.get(key, 0.0), e)


# ------------------------------------------------------------------------------------------------ fp64 references
def ref_patch_embed(rgb, w, bias, gamma, beta):
    """PatchEmbedSwin in fp64: rgb [B, 3, H, W] zero-padded right / bottom to a multiple of 4, 4x4/s4 conv + bias,
    LayerNorm(E) -> tokens [B * Hp * Wp, E] (row-major over the token grid)."""
    x = rgb.double()
    H, W = x.shape[-2:]
    x = F.pad(x, (0, (4 - W % 4) % 4, 0, (4 - H % 4) % 4))
    x = F.conv2d(x, w.double(), bias.double(), stride=4)
    x = x.flatten(2).transpose(1, 2).reshape(-1, w.shape[0])
    return F.layer_norm(x, (w.shape[0],), gamma.double(), beta.double(), 1e-5)


def ref_layer_norm(x, gamma, beta):
    """LayerNorm over the last axis in fp64, eps 1e-5."""
    return F.layer_norm(x.double(), (x.shape[-1],), gamma.double(), beta.double(), 1e-5)


def ref_patch_merge(x, gamma, beta):
    """PatchMerging's gather + norm in fp64: x [B, H, W, C] zero-padded to even H / W, 2x2 unfold (feature c * 4 + ky
    * 2 + kx), LayerNorm(4C) -> tokens [B * ceil(H / 2) * ceil(W / 2), 4C]."""
    B, H, W, Cc = x.shape
    z = F.pad(x.double().permute(0, 3, 1, 2), (0, W % 2, 0, H % 2))
    z = F.unfold(z, kernel_size=2, stride=2).transpose(1, 2).reshape(-1, 4 * Cc)
    return F.layer_norm(z, (4 * Cc,), gamma.double(), beta.double(), 1e-5)


def to_nchw(tokens, B, hw):
    """Tokens [B * hw, C] -> the stage-output layout [B, C, hw]."""
    return tokens.reshape(B, hw, tokens.shape[-1]).transpose(1, 2)


def _row_margin(got, ref, dim=-1):
    """Per token: error over that token's max |ref| (dim: the channel axis)."""
    return (got.double() - ref).abs().amax(dim) / ref.abs().amax(dim)


def _affine(n, seed):
    g = torch.Generator().manual_seed(seed)
    return (1 + 0.3 * torch.randn(n, generator=g)).to(DEV), (0.2 * torch.randn(n, generator=g)).to(DEV)


# ------------------------------------------------------------------------------------------------ patch embedding
def _pe_inputs(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    rgb = torch.randn(B, 3, H, W, generator=g)
    w = torch.randn(E, 3, 4, 4, generator=g) * 0.2
    bias = 0.1 * torch.randn(E, generator=g)
    gamma, beta = _affine(E, seed + 1)
    return rgb.to(DEV), w.to(DEV), bias.to(DEV), gamma, beta


# (B, H, W): both axes padded (-> 18 x 27, 15 x 21); a second, partial 32-token segment (24 x 40); a one-token tail
# segment, where the 8-token group loop stops early (2 x 33); a single token; the full KITTI batch (88 x 304)
PE = [(2, 70, 106), (2, 57, 83), (2, 96, 160), (2, 5, 129), (2, 4, 4), (4, 352, 1216)]


@gpu
@pytest.mark.parametrize("B,H,W", PE, ids=[f"B{b}_{h}x{w}" for b, h, w in PE])
def test_patch_embed_vs_fp64(eng, B, H, W):
    rgb, w, bias, gamma, beta = _pe_inputs(B, H, W, H * 31 + W)
    ref = ref_patch_embed(rgb, w, bias, gamma, beta)
    out = eng.swin_patch_embed(rgb, w, bias, gamma, beta)
    assert out.shape == ref.shape == (B * ((H + 3) // 4) * ((W + 3) // 4), E)
    e = _row_margin(out, ref).max().item()
    print(f"\n[patch embed B{B} {H}x{W}] worst token {e:.2e} (bound {TOL:.0e})")
    _log(f"patch_embed:{H}x{W}", e)
    assert e <= TOL, (B, H, W, e)
    assert torch.equal(out, eng.swin_patch_embed(rgb, w, bias, gamma, beta))


@gpu
@pytest.mark.parametrize("c", [0.7, 3.7, -33.3])
def test_patch_embed_constant_tokens_give_beta(eng, c):
    """A zero image with a bias constant across channels: every token, the padded ones included, is constant before
    the norm and must come out as beta."""
    B, H, W = 2, 57, 83
    _, w, _, gamma, beta = _pe_inputs(B, H, W, 3)
    rgb = torch.zeros(B, 3, H, W, device=DEV)
    bias = torch.full((E,), c, device=DEV)
    out = eng.swin_patch_embed(rgb, w, bias, gamma, beta)
    ref = beta.double().expand(out.shape[0], E)
    e = _row_margin(out, ref).max().item()
    print(f"\n[patch embed constant {c}] worst token {e:.2e} (bound {TOL:.0e})")
    _log(f"patch_embed:constant{c}", e)
    assert e <= TOL, (c, e)


@gpu
def test_patch_embed_nan_stays_in_its_token(eng):
    """The patch embedding writes fp32 (no split, no range check): a NaN pixel makes its own token NaN and leaves every
    other token bit-identical, the tokens of its 8-token group and 32-token segment included."""
    B, H, W = 2, 57, 83
    rgb, w, bias, gamma, beta = _pe_inputs(B, H, W, 8)
    out0 = eng.swin_patch_embed(rgb, w, bias, gamma, beta)
    Hp, Wp = (H + 3) // 4, (W + 3) // 4
    for b, y, x in ((1, H - 1, W - 1), (0, 9, 37)):
        bad = rgb.clone()
        bad[b, 2, y, x] = float("nan")
        out = eng.swin_patch_embed(bad, w, bias, gamma, beta)
        tok = (b * Hp + y // 4) * Wp + x // 4
        assert torch.isnan(out[tok]).all()
        keep = torch.ones(out.shape[0], dtype=torch.bool, device=DEV)
        keep[tok] = False
        assert torch.equal(out[keep], out0[keep])
    assert torch.equal(out0, eng.swin_patch_embed(rgb, w, bias, gamma, beta))


# ------------------------------------------------------------------------------------------------ LayerNorm
LN_WIDTHS = [192, 384, 768, 1536]


def _ln_inputs(M, Cc, seed):
    """Rows: signed with an offset; 100 rows of mean 1e3 and std 1e-2; constant rows (variance 0: random, 0, 1e3);
    8 rows with one massive channel (1e3 in one channel, N(0, 1) elsewhere)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, Cc, generator=g) * 2 + 0.5
    x[:100] = 1e3 + 1e-2 * torch.randn(100, Cc, generator=g)
    x[100:110] = torch.randn(10, 1, generator=g) * 3
    x[110] = 0.0
    x[111] = 1e3
    x[112:120] = torch.randn(8, Cc, generator=g)
    x[torch.arange(112, 120), torch.randint(0, Cc, (8,), generator=g)] = 1e3
    gamma, beta = _affine(Cc, seed + 1)
    return x.to(DEV), gamma, beta


# (B, H, W) of the stage-output copy: KITTI's stage-3 grid (11 x 38) at B = 3, an odd hw (9 x 15); neither token
# count is a multiple of the 8 tokens per block
LN_GRIDS = [(3, 11, 38), (2, 9, 15)]


@gpu
@pytest.mark.parametrize("Cc", LN_WIDTHS)
def test_layer_norm_vs_fp64(eng, Cc):
    for B, H, W in LN_GRIDS:
        hw = H * W
        M = B * hw
        x, gamma, beta = _ln_inputs(M, Cc, Cc + hw)
        ref = ref_layer_norm(x, gamma, beta)
        out, nchw = eng.swin_layer_norm(x, gamma, beta, hw=hw)
        assert nchw.shape == (B, Cc, hw)
        per_row = _row_margin(out, ref)
        per_col = _row_margin(nchw, to_nchw(ref, B, hw), dim=1).flatten()  # the copy, per token
        e, ec = per_row.max().item(), per_col.max().item()
        print(f"\n[ln C{Cc} B{B} {H}x{W}] worst token {e:.2e}, NCHW copy {ec:.2e} (bound {TOL:.0e}); mean-1e3 rows "
              f"{per_row[:100].max().item():.2e}, constant rows {per_row[100:112].max().item():.2e}, massive-channel "
              f"rows {per_row[112:120].max().item():.2e}")
        _log(f"layernorm:C{Cc}.{H}x{W}", max(e, ec))
        assert e <= TOL and ec <= TOL, (Cc, H, W, e, ec)
        out2, nchw2 = eng.swin_layer_norm(x, gamma, beta, hw=hw)
        assert torch.equal(out, out2) and torch.equal(nchw, nchw2)
        # without the copy: the same planes
        assert torch.equal(out, eng.swin_layer_norm(x, gamma, beta)[0])


# ------------------------------------------------------------------------------------------------ patch merging
MERGE_GRIDS = [(2, 18, 27), (1, 15, 21), (2, 9, 14), (1, 5, 7), (1, 1, 1), (2, 88, 304)]
MERGE = [(Cc, *g) for Cc in (192, 384, 768) for g in MERGE_GRIDS]


def _merge_inputs(B, H, W, Cc, seed):
    """Signed values with an offset; the last three rows and columns (the odd padded row / column included) at mean
    1e3 and std 1e-2, so that the padded tokens mix 1e3-valued and zero features and the inner ones are dominated by
    their mean; a constant 1e3 and a constant 0 token at the top left."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, H, W, Cc, generator=g) * 2 + 0.5
    x[:, -3:] = 1e3 + 1e-2 * torch.randn(B, min(3, H), W, Cc, generator=g)
    x[:, :, -3:] = 1e3 + 1e-2 * torch.randn(B, H, min(3, W), Cc, generator=g)
    if H >= 4 and W >= 2:
        x[:, 0:2, 0:2] = 1e3
        x[:, 2:4, 0:2] = 0.0
    gamma, beta = _affine(4 * Cc, seed + 1)
    return x.to(DEV), gamma, beta


@gpu
@pytest.mark.parametrize("Cc,B,H,W", MERGE, ids=[f"C{c}_B{b}_{h}x{w}" for c, b, h, w in MERGE])
def test_patch_merge_vs_fp64(eng, Cc, B, H, W):
    x, gamma, beta = _merge_inputs(B, H, W, Cc, Cc + H * 31 + W)
    ref = ref_patch_merge(x, gamma, beta)
    out = eng.swin_patch_merge(x, gamma, beta)
    H2, W2 = (H + 1) // 2, (W + 1) // 2
    assert out.shape == ref.shape == (B * H2 * W2, 4 * Cc)
    per = _row_margin(out, ref).reshape(B, H2, W2)
    e = per.max().item()
    edge = torch.cat([per[:, -1].flatten(), per[:, :, -1].flatten()]).max().item()
    print(f"\n[merge C{Cc} B{B} {H}x{W}] worst token {e:.2e} (bound {TOL:.0e}); last row / column {edge:.2e}")
    _log(f"merge:C{Cc}.{H}x{W}", e)
    assert e <= TOL, (Cc, B, H, W, e)
    assert torch.equal(out, eng.swin_patch_merge(x, gamma, beta))


# ------------------------------------------------------------------------------------------------ status and recovery
@gpu
def test_layer_norm_and_merge_status_and_recovery(eng):
    """A NaN in the input and a gamma that drives 16 |y| past 6e4 are DD_ERR_RANGE; the next clean call equals a call
    made before, bit for bit."""
    from diffusiondepth_b200 import _cabi
    B, H, W, Cc = 2, 9, 15, 384
    x, gamma, beta = _ln_inputs(B * H * W, Cc, 4)
    out0, nchw0 = eng.swin_layer_norm(x, gamma, beta, hw=H * W)
    xm, gm, bm = _merge_inputs(B, H, W, Cc, 6)
    m0 = eng.swin_patch_merge(xm, gm, bm)
    bad = x.clone()
    bad[B * H * W - 1, Cc - 1] = float("nan")
    for args in ((bad, gamma, beta), (x, gamma * 5000, beta)):
        with pytest.raises(_cabi.EngineError, match="DD_ERR_RANGE"):
            eng.swin_layer_norm(*args, hw=H * W)
        out1, nchw1 = eng.swin_layer_norm(x, gamma, beta, hw=H * W)
        assert torch.equal(out0, out1) and torch.equal(nchw0, nchw1)
    bad = xm.clone()
    bad[1, H - 1, W - 1, Cc - 1] = float("nan")  # a real feature of the padded corner token
    for args in ((bad, gm, bm), (xm, gm * 5000, bm)):
        with pytest.raises(_cabi.EngineError, match="DD_ERR_RANGE"):
            eng.swin_patch_merge(*args)
        assert torch.equal(m0, eng.swin_patch_merge(xm, gm, bm))


# ------------------------------------------------------------------------------------------------ argument checks
@gpu
def test_swin_layers_reject_bad_arguments(eng):
    from diffusiondepth_b200 import _cabi
    lib, h, st = eng.lib, eng._h, C.c_void_p(0)
    rgb, w, bias, gamma, beta = _pe_inputs(1, 8, 8, 1)
    with pytest.raises(_cabi.EngineError, match="DD_ERR_UNSUPPORTED"):  # E = 96: not instantiated
        eng.swin_patch_embed(rgb, w[:96], bias[:96], gamma[:96], beta[:96])
    for Cc in (96, 256, 512, 3072):
        x = torch.zeros(12, Cc, device=DEV)
        with pytest.raises(_cabi.EngineError, match="DD_ERR_UNSUPPORTED"):
            eng.swin_layer_norm(x, x[0], x[0])
    x = torch.zeros(12, 1536, device=DEV)
    with pytest.raises(_cabi.EngineError, match="DD_ERR_INVALID"):  # 12 tokens are no whole number of 5-token images
        eng.swin_layer_norm(x[:, :192], x[0, :192], x[0, :192], hw=5)
    xm = torch.zeros(1, 4, 6, 1536, device=DEV)
    for Cc in (96, 1536):
        with pytest.raises(_cabi.EngineError, match="DD_ERR_UNSUPPORTED"):
            eng.swin_patch_merge(xm[..., :Cc], xm[0, 0, 0, :1], xm[0, 0, 0, :1])
    # through the C ABI directly: null pointers and bad geometry are DD_ERR_INVALID
    p = C.c_void_p(x.data_ptr())
    out = torch.empty(12, 1536, device=DEV)
    o = C.c_void_p(out.data_ptr())
    n = None
    assert lib.dd_swin_patch_embed(h, n, p, p, p, p, o, 1, 8, 8, E, st) == 1
    assert lib.dd_swin_patch_embed(h, p, p, p, p, p, n, 1, 8, 8, E, st) == 1
    assert lib.dd_swin_patch_embed(h, p, p, p, p, p, o, 0, 8, 8, E, st) == 1
    assert lib.dd_swin_patch_embed(h, p, p, p, p, p, o, 1, 8, 0, E, st) == 1
    assert lib.dd_swin_layer_norm(h, n, p, p, o, n, 12, 192, 0, st) == 1
    assert lib.dd_swin_layer_norm(h, p, p, n, o, n, 12, 192, 0, st) == 1
    assert lib.dd_swin_layer_norm(h, p, p, p, o, n, 0, 192, 0, st) == 1
    assert lib.dd_swin_layer_norm(h, p, p, p, o, o, 12, 192, 0, st) == 1      # a copy needs hw >= 1
    assert lib.dd_swin_layer_norm(h, p, p, p, o, o, 12, 192, 5, st) == 1      # tokens % hw != 0
    assert lib.dd_swin_patch_merge(h, p, n, p, o, 1, 2, 2, 192, st) == 1
    assert lib.dd_swin_patch_merge(h, p, p, p, o, 1, 0, 2, 192, st) == 1
    assert lib.dd_swin_patch_merge(h, p, p, p, o, 0, 2, 2, 192, st) == 1


# ------------------------------------------------------------------------------------------------ the whole backbone
@gpu
@pytest.mark.parametrize("hw", [(70, 106), (57, 83)])
def test_native_swin_backbone_odd_grids_vs_oracle(hw):
    """dd_run_backbone on Swin-L where the padding runs: 70x106 -> 18x27 / 9x14 / 5x7 / 3x4 tokens (the patch
    embedding pads both axes, three merges pad an odd row or column), 57x83 -> 15x21 / 8x11 / 4x6 / 2x3; vs the fp64
    restatement of reference backbone/swin.py:756-777, stage by stage, with non-zero relative-position tables."""
    import dd_helpers as helpers
    m = helpers.build_mirror("swinl", 2).to(DEV)
    bb, head = m.depth_backbone, m.depth_head
    g = torch.Generator().manual_seed(23)
    saved = {}
    with torch.no_grad():  # the mirror is cached across tests: restored below
        for n, p in bb.named_parameters():
            if n.endswith("relative_position_bias_table"):
                saved[n] = p.detach().clone()
                p.copy_(torch.randn(p.shape, generator=g).to(DEV) * 0.5)
    try:
        sd = {"depth_backbone." + k: v.detach().cpu() for k, v in bb.state_dict().items()}
        rgb = torch.randn(2, 3, *hw, generator=g)
        ref = restate.swin_backbone(sd, rgb.double())
        sizes = head.swin_pyramid(hw)
        assert [tuple(r.shape[-2:]) for r in ref] == sizes
        eng = head._engine(2, ((hw[0] + 1) // 2, (hw[1] + 1) // 2), sizes[0], DEV,
                           feats=([192, 384, 768, 1536], sizes), image_hw=hw)
        feats = eng.run_backbone(rgb.to(DEV), want_feats=True)
        eng.poll_status()
        errs = []
        for f, r in zip(feats, ref):
            assert f.shape == r.shape
            errs.append((f.double().cpu() - r).abs().max().item() / r.abs().max().item())
        print(f"\n[swin stages {hw[0]}x{hw[1]}] rel err", ["%.2e" % e for e in errs])
        assert max(errs) < 1e-4, errs
    finally:
        with torch.no_grad():
            for n, p in bb.named_parameters():
                if n in saved:
                    p.copy_(saved[n])


# ------------------------------------------------------------------------------------------------ CPU: the references
def test_layer_references_compose_to_the_restated_backbone():
    """ref_patch_embed, ref_layer_norm and ref_patch_merge (+ the reduction Linear) with the to_nchw layout reproduce
    restate.swin_backbone with no blocks stage by stage: the references restate PatchEmbedSwin, the stage-output norms
    and PatchMerging, at odd grids (37x53 -> 10x14 / 5x7 / 3x4 / 2x2)."""
    P = "depth_backbone."
    g = torch.Generator().manual_seed(5)
    B, Hi, Wi = 2, 37, 53
    sd = {P + "patch_embed.projection.weight": torch.randn(E, 3, 4, 4, generator=g) * 0.2,
          P + "patch_embed.projection.bias": 0.1 * torch.randn(E, generator=g),
          P + "patch_embed.norm.weight": 1 + 0.3 * torch.randn(E, generator=g),
          P + "patch_embed.norm.bias": 0.2 * torch.randn(E, generator=g)}
    for s in range(4):
        Cs = E << s
        sd[f"{P}norm{s}.weight"] = 1 + 0.3 * torch.randn(Cs, generator=g)
        sd[f"{P}norm{s}.bias"] = 0.2 * torch.randn(Cs, generator=g)
        if s < 3:
            sd[f"{P}stages.{s}.downsample.norm.weight"] = 1 + 0.3 * torch.randn(4 * Cs, generator=g)
            sd[f"{P}stages.{s}.downsample.norm.bias"] = 0.2 * torch.randn(4 * Cs, generator=g)
            sd[f"{P}stages.{s}.downsample.reduction.weight"] = torch.randn(2 * Cs, 4 * Cs, generator=g) / (4 * Cs) ** 0.5
    rgb = torch.randn(B, 3, Hi, Wi, generator=g)
    want = restate.swin_backbone(sd, rgb.double(), depths=(0, 0, 0, 0))
    x = ref_patch_embed(rgb, *(sd[P + k] for k in ("patch_embed.projection.weight", "patch_embed.projection.bias",
                                                    "patch_embed.norm.weight", "patch_embed.norm.bias")))
    H, W = (Hi + 3) // 4, (Wi + 3) // 4
    for s in range(4):
        Cs = E << s
        out = to_nchw(ref_layer_norm(x, sd[f"{P}norm{s}.weight"], sd[f"{P}norm{s}.bias"]), B, H * W)
        assert want[s].shape == (B, Cs, H, W)
        assert (out.reshape(B, Cs, H, W) - want[s]).abs().max().item() <= 1e-12 * want[s].abs().max().item(), s
        if s < 3:
            p = f"{P}stages.{s}.downsample."
            z = ref_patch_merge(x.reshape(B, H, W, Cs), sd[p + "norm.weight"], sd[p + "norm.bias"])
            x = F.linear(z, sd[p + "reduction.weight"].double())
            H, W = (H + 1) // 2, (W + 1) // 2
