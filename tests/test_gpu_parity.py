"""GPU parity tests proper (-m gpu): the CUDA path through the C ABI against the oracle restatement on the
same seeded inputs, against golden vectors from the real reference, and size-independent properties at
BASELINE.json's full sizes.  Tolerance: 1e-3 on the decoder logit z (== relative depth error, BASELINE.md)."""
import pytest
import torch

import diffusiondepth_b200 as dd
from oracle import configs, restate
import dd_helpers as helpers

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
TOL = 1e-3
SHAPES = [(16, 64), (64, 256), (256, 256), (256, 64), (64, 16)]


def _swin_head(steps, seed=7):
    from diffusiondepth_b200.model.registry import HEADS
    torch.manual_seed(seed)
    return HEADS.build(dict(type="DDIMDepthEstimate_Swin_ADDHAHI", in_channels=[64, 128, 256, 512],
                            inference_steps=steps, num_train_timesteps=1000, depth_feature_dim=16, loss_cfgs=[],
                            init_cfg=None)).eval()


def _res_head(steps, seed=7):
    from diffusiondepth_b200.model.registry import HEADS
    torch.manual_seed(seed)
    return HEADS.build(dict(type="DDIMDepthEstimate_Res", in_channels=[64, 128, 256, 512], inference_steps=steps,
                            num_train_timesteps=1000, depth_feature_dim=16, loss_cfgs=[], init_cfg=None)).eval()


def _mpvit_head(steps, seed=7):
    from diffusiondepth_b200.model.registry import HEADS
    torch.manual_seed(seed)
    return HEADS.build(dict(type="DDIMDepthEstimate_MPVIT_ADDHAHI", in_channels=[64, 128, 256, 512],
                            inference_steps=steps, num_train_timesteps=1000, depth_feature_dim=16, loss_cfgs=[],
                            init_cfg=None)).eval()


def _head_sd(head):
    return {"depth_head." + k: v.detach().cpu() for k, v in head.state_dict().items()}


# ------------------------------------------------------------------------------------------------ single layers
@pytest.mark.parametrize("path", ["classic", "halo", "pair", "swap", "swap_halo", "simt"])
@pytest.mark.parametrize("cin,cout", SHAPES)
def test_conv3x3_all_hot_path_shapes(cin, cout, path):
    """3-pass fp16 split on wgmma (row-halo-reuse kernel; every combination of the kernel-selection flags, which pick
    Blackwell-only kernels elsewhere, must reach it) and the fp32 CUDA-core check path, vs an fp64 reference; ragged
    tiles, a single tile, sub-tile images."""
    tol = 3e-5
    eng = dd.DenoiseEngine("swin", 1, (8, 16), (4, 8), 2, DEV, cuda_graph=False, simt_conv=path == "simt",
                           halo_conv=path in ("halo", "pair", "swap_halo"), swap_narrow=path in ("swap", "swap_halo"),
                           pair_wide=path == "pair")
    for (B, H, W) in [(2, 24, 40), (1, 8, 16), (1, 13, 21), (1, 5, 9), (2, 57, 76)]:
        g = torch.Generator().manual_seed(cin * 1000 + cout + H)
        x = torch.randn(B, cin, H, W, generator=g).to(DEV) * 3
        w = (torch.randn(cout, cin, 3, 3, generator=g) * 0.05).to(DEV)
        b = torch.randn(cout, generator=g).to(DEV)
        y = eng.conv3x3(x, w, b)
        ref = torch.nn.functional.conv2d(x.double(), w.double(), b.double(), padding=1)
        err = (y.double() - ref).abs().max().item() / ref.abs().max().item()
        assert err < tol, (cin, cout, B, H, W, err)
    eng.close()


def test_conv_linearity_and_zero():
    eng = dd.DenoiseEngine("swin", 1, (8, 16), (4, 8), 2, DEV, cuda_graph=False, fp8_corr=False)
    g = torch.Generator().manual_seed(1)
    x1, x2 = (torch.randn(1, 256, 16, 32, generator=g).to(DEV) for _ in range(2))
    w = (torch.randn(256, 256, 3, 3, generator=g) * 0.02).to(DEV)
    zero = torch.zeros(256, device=DEV)
    y1, y2, y12 = eng.conv3x3(x1, w, zero), eng.conv3x3(x2, w, zero), eng.conv3x3(x1 + x2, w, zero)
    assert (y12 - y1 - y2).abs().max().item() < 2e-5 * y12.abs().max().item()
    assert eng.conv3x3(torch.zeros_like(x1), w, zero).abs().max().item() == 0.0
    eng.close()


# ------------------------------------------------------------------------------------------------ operators
@pytest.mark.parametrize("variant,hw,fp8", [("res", (19, 27), False), ("swin", (18, 26), False), ("swin", (8, 16), False),
                                            ("swin", (18, 26), True), ("swin", (19, 27), False), ("swin", (35, 53), True)])
def test_denoiser_operator_vs_oracle(variant, hw, fp8):
    """eps = ScheduledCNNRefine(noisy, t, cond) with per-image t — vs the fp64 restatement (exact 3-pass split, and the
    fp8-correction mode of the wide convs at its own error level).  Odd latent sizes (19 x 27, 35 x 53 over a 10 x 14 /
    18 x 27 condition map) are not an exact 2x upsampling: some outputs of the quad-based condition injection kernel take
    their per-tap path."""
    head = (_res_head if variant == "res" else _swin_head)(5).to(DEV)
    head.fp8_corrections = fp8
    sd = _head_sd(head)
    B, (h, w) = 2, hw
    chw = (h, w) if variant == "res" else ((h + 1) // 2, (w + 1) // 2)
    g = torch.Generator().manual_seed(3)
    noisy = torch.randn(B, 16, h, w, generator=g) * 4
    cond = torch.randn(B, 256, *chw, generator=g)
    t = torch.tensor([950, 40])
    eps = head.model(noisy.to(DEV), t.to(DEV), cond.to(DEV), None, None, None)
    ref = restate.denoiser(sd, noisy.double(), t, cond.double(), variant)
    assert eps.shape == ref.shape and (eps >= 0).all()
    assert (eps.double().cpu() - ref).abs().max().item() < (2e-3 if fp8 else 2e-4) * max(1.0, ref.abs().max().item())


def test_decoder_vs_oracle():
    head = _res_head(5).to(DEV)
    sd = _head_sd(head)
    g = torch.Generator().manual_seed(4)
    for (h, w) in [(19, 27), (8, 16), (33, 5)]:
        lat = torch.randn(2, 16, h, w, generator=g) * 20
        eng = head._engine(2, (h, w), (h, w), DEV)
        depth, logits = eng.decode(lat.to(DEV), want_logits=True)
        z = restate.decode_logits(sd, lat.double())
        assert (logits.double().cpu() - z).abs().max().item() < 1e-4 * max(1.0, z.abs().max().item())
        d32 = restate.decode(sd, lat)
        pm = restate.parity_metrics(logits.cpu(), z.float(), depth.cpu(), d32)
        assert pm["max_rel_depth_wellcond"] < TOL
        assert (depth.cpu()[z.float() < -14.5] == 999999.0).all()  # clamp(1e-6) branch of inv_t


@pytest.mark.parametrize("HW", [(38, 54), (37, 53), (352, 1216)])
def test_encoder_vs_oracle(HW):
    """dd_encode = depth_transform.t (reference depth_transform.py:15-19,29-31), odd sizes included."""
    head = _res_head(2).to(DEV)
    with torch.no_grad():
        for m in head.depth_transform.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.running_mean.normal_(0, 0.3)
                m.running_var.uniform_(0.5, 1.5)
                m.weight.uniform_(0.5, 1.5)
                m.bias.normal_(0, 0.2)
    sd = _head_sd(head)
    g = torch.Generator().manual_seed(8)
    depth = torch.rand(2, 1, *HW, generator=g) * 80
    lat = ((HW[0] + 1) // 2, (HW[1] + 1) // 2)
    eng = head._engine(2, lat, lat, DEV)
    out = eng.encode(depth.to(DEV))
    ref = restate.encode(sd, depth.double())
    assert out.shape == ref.shape
    assert (out.double().cpu() - ref).abs().max().item() < 2e-5
    from diffusiondepth_b200.model._blocks import exact_fp32
    with torch.no_grad(), exact_fp32():  # (cuDNN's default TF32 would itself be off by more than the tolerance)
        assert torch.allclose(out, head.depth_transform.t(depth.to(DEV)), atol=2e-5)


@pytest.mark.parametrize("variant,hw,T", [("res", (19, 27), 5), ("swin", (18, 26), 5), ("swin", (24, 40), 20)])
def test_loop_and_decode_vs_oracle(variant, hw, T):
    """T-step DDIM loop + decoder through dd_denoise_decode vs the fp64 restatement; CUDA-graph replay and the
    fp32 CUDA-core conv path must agree with it too."""
    head = (_res_head if variant == "res" else _swin_head)(T).to(DEV)
    sd = _head_sd(head)
    B, (h, w) = 2, hw
    chw = (h, w) if variant == "res" else ((h + 1) // 2, (w + 1) // 2)
    g = torch.Generator().manual_seed(5)
    noise = torch.randn(B, 16, h, w, generator=g)
    cond = torch.randn(B, 256, *chw, generator=g).abs()
    lat_ref = restate.ddim_loop(sd, cond.double(), noise.double(), T, variant)
    z_ref = restate.decode_logits(sd, lat_ref)
    outs = {}
    for name, kw in (("graph", dict(cuda_graph=True, fp8_corr=False)), ("eager", dict(cuda_graph=False, fp8_corr=False)),
                     ("simt", dict(cuda_graph=False, simt_conv=True)), ("fp8", dict(cuda_graph=True, fp8_corr=True))):
        if name == "fp8" and variant != "swin":
            continue
        eng = dd.DenoiseEngine(variant, B, (h, w), chw, T, DEV, check_range=True, **kw)
        eng.load_weights(head._engine_tensors())
        eng.set_schedule(*head.scheduler.fused_coefficients(T))
        depth, lat, z = eng.denoise_decode(cond.to(DEV), noise.to(DEV), want_latent=True, want_logits=True)
        depth2, _, z2 = eng.denoise_decode(cond.to(DEV), noise.to(DEV), want_latent=True, want_logits=True)
        if name != "simt":  # the tensor-core path is bit-reproducible; the debug SIMT path sums stats with atomics
            assert torch.equal(z, z2) and torch.equal(depth, depth2), "run-to-run determinism"
        outs[name] = z
        scale = max(1.0, lat_ref.abs().max().item())
        assert (lat.double().cpu() - lat_ref).abs().max().item() < (2e-3 if name == "fp8" else 2e-4) * scale, name
        assert (z.double().cpu() - z_ref).abs().max().item() < TOL, name
        assert eng.last_launch_count == 3 + T * (14 if variant == "swin" else 12) + 2
        eng.close()
    assert torch.equal(outs["graph"], outs["eager"])


# ------------------------------------------------------------------------------------------------ producers
@pytest.mark.parametrize("variant,hw0", [("swin", (16, 32)), ("swin", (24, 40)), ("res", (32, 48)), ("mpvit", (32, 48)),
                                         ("mpvit", (24, 40))])
def test_native_neck_and_fpn_vs_oracle(variant, hw0):
    """dd_build_condition (HAHI neck + FPN on the tensor-core conv path, BN folded, concat-free) vs the fp64
    restatement of reference necks/hahi.py:165-276 + head :112-122, and vs the mirror's torch-op producers.
    mpvit: channels 128/216/288/288 — partial 64-channel K chunks (216 = 3.375 x 64, the second concat source starting
    at weight column 216) and partial N tiles (216 of 256, 288 of 2 x 192), completed by TMA out-of-bounds zero fill."""
    head = {"res": _res_head, "swin": _swin_head, "mpvit": _mpvit_head}[variant](2).to(DEV)
    with torch.no_grad():  # make BN non-trivial
        for m in head.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.running_mean.normal_(0, 0.2)
                m.running_var.uniform_(0.5, 1.5)
                m.weight.uniform_(0.5, 1.5)
                m.bias.normal_(0, 0.2)
    sd = _head_sd(head)
    chans = {"swin": (192, 384, 768, 1536), "res": (64, 128, 256, 512), "mpvit": (128, 216, 288, 288)}[variant]
    g = torch.Generator().manual_seed(11)
    feats = [torch.randn(2, c, hw0[0] >> i, hw0[1] >> i, generator=g) for i, c in enumerate(chans)]
    fd = [f.to(DEV) for f in feats]
    lat = (2 * hw0[0], 2 * hw0[1]) if variant == "swin" else hw0
    assert head._pyramid_ok(fd)
    eng = head._engine(2, lat, hw0, DEV, feats=fd)
    cond = eng.build_condition(fd, want_cond=True)
    eng.poll_status()
    f64 = [f.double() for f in feats]
    ref = restate.fpn_condition(sd, restate.hahi_neck(sd, f64) if variant != "res" else f64)
    err = (cond.double().cpu() - ref).abs().max().item() / ref.abs().max().item()
    assert err < 5e-5, err
    from diffusiondepth_b200.model._blocks import exact_fp32
    with torch.no_grad(), exact_fp32():  # with cuDNN's default TF32 the torch path itself is off by ~5e-3 here
        torch_cond = head._condition(head._neck(fd))
    assert (cond - torch_cond).abs().max().item() < 1e-4 * ref.abs().max().item()
    # the loop consumes the internally built condition: same result as passing it explicitly
    noise = torch.randn(2, 16, *lat, generator=g).to(DEV)
    eng.set_schedule(*head.scheduler.fused_coefficients(2))
    a = eng.denoise_decode(None, noise, want_logits=True)[2]
    b = head._engine(2, lat, hw0, DEV).denoise_decode(cond, noise, want_logits=True)[2]
    assert torch.equal(a, b)
    with pytest.raises(dd.EngineError):
        eng.denoise_decode(None, noise)  # the built condition is consumed once


@pytest.mark.parametrize("hw", [(96, 160), (64, 96)])
def test_native_swin_backbone_vs_oracle(hw):
    """dd_run_backbone (patch embed, LN, 3-pass GEMMs, shifted-window attention with padding, patch merging) vs
    the fp64 restatement of reference backbone/swin.py:756-777, stage by stage; non-zero relative-position tables
    so the bias path is exercised.  96x160 -> 24x40 tokens (pads to 28x42), 64x96 -> 16x24 (pads to 21x28)."""
    m = helpers.build_mirror("swinl", 2).to(DEV)
    bb, head = m.depth_backbone, m.depth_head
    g = torch.Generator().manual_seed(21)
    saved = {}
    with torch.no_grad():
        for n, p in bb.named_parameters():
            if n.endswith("relative_position_bias_table"):
                saved[n] = p.detach().clone()
                p.copy_(torch.randn(p.shape, generator=g).to(DEV) * 0.5)
    try:
        sd = {"depth_backbone." + k: v.detach().cpu() for k, v in bb.state_dict().items()}
        rgb = torch.randn(2, 3, *hw, generator=g)
        ref = restate.swin_backbone(sd, rgb.double())
        sizes = head.swin_pyramid(hw)
        eng = head._engine(2, (hw[0] // 2, hw[1] // 2), sizes[0], DEV, feats=([192, 384, 768, 1536], sizes), image_hw=hw)
        feats = eng.run_backbone(rgb.to(DEV), want_feats=True)
        eng.poll_status()
        for s, (f, r) in enumerate(zip(feats, ref)):
            assert f.shape == r.shape
            err = (f.double().cpu() - r).abs().max().item() / r.abs().max().item()
            assert err < 1e-4, (s, err)
        # the planes left in the workspace feed the neck directly: same condition map as via the NCHW round trip
        c1 = eng.build_condition(None, want_cond=True)
        c2 = eng.build_condition(feats, want_cond=True)
        assert (c1 - c2).abs().max().item() < 1e-5 * c2.abs().max().item()
    finally:
        with torch.no_grad():
            for n, p in bb.named_parameters():
                if n in saved:
                    p.copy_(saved[n])


@pytest.mark.parametrize("family,hw", [("res18", (228, 304)), ("res18", (70, 106)), ("res50", (64, 96))])
def test_native_resnet_backbone_and_resampling_fpn_vs_oracle(family, hw):
    """dd_run_backbone(kind = ResNet): stride-2 3x3 convs via TMA element strides, BN folded, residual add before
    ReLU, biased strided skip convs — vs the fp64 restatement of reference mmbev_resnet.py:124-160; then the FPN on
    the odd-sized pyramid (228x304 -> 114/57/29/15), where adaptive_avg_pool2d really resamples (head :121)."""
    m = helpers.build_mirror(family, 2).to(DEV)
    bb, head = m.depth_backbone, m.depth_head
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.running_mean.normal_(0, 0.1)
                mod.running_var.uniform_(0.7, 1.3)
    try:
        sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
        g = torch.Generator().manual_seed(31)
        rgb = torch.randn(2, 3, *hw, generator=g)
        depths = restate.RESNET_DEPTHS["mmbev_" + family]
        ref = restate.resnet_backbone(sd, rgb.double(), depths)
        sizes = head.resnet_pyramid(hw)
        assert [tuple(r.shape[-2:]) for r in ref] == sizes
        eng = head._engine(2, sizes[0], sizes[0], DEV, feats=([64, 128, 256, 512], sizes), image_hw=hw)
        feats = eng.run_backbone(rgb.to(DEV), want_feats=True)
        eng.poll_status()
        for s, (f, r) in enumerate(zip(feats, ref)):
            err = (f.double().cpu() - r).abs().max().item() / r.abs().max().item()
            assert err < 5e-5, (s, err)
        cond = eng.build_condition(None, want_cond=True)
        cref = restate.fpn_condition(sd, ref)
        err = (cond.double().cpu() - cref).abs().max().item() / cref.abs().max().item()
        assert err < 5e-5, err
    finally:
        with torch.no_grad():
            for mod in m.modules():
                if isinstance(mod, torch.nn.BatchNorm2d):
                    mod.running_mean.zero_()
                    mod.running_var.fill_(1.0)


@pytest.mark.parametrize("hw", [(64, 96), (70, 106), (228, 304)])
def test_native_mpvit_backbone_vs_oracle(hw):
    """dd_run_backbone(kind = MPViT): full-resolution stem, chained depthwise-separable patch embeddings, conv path,
    factorised-attention encoders (token-axis softmax of k, k^T v, convolutional relative position encoding with 3 / 5 / 7
    windows), 1x1 aggregate — vs the fp64 restatement of reference backbone/mpvit.py:601-730, stage by stage; then neck +
    FPN on the resulting planes.  70x106 -> 35x53 / 18x27 / 9x14 / 5x7: odd sizes on every level.  228x304 (an NYU
    image): stage 0 at 114x152 = 17,328 tokens, past the 16,384 where the attention's token chunks grow beyond 64
    tokens.  The restatement runs in fp64 on the GPU."""
    m = helpers.build_mirror("mpvit_s", 2).to(DEV)
    bb, head = m.depth_backbone, m.depth_head
    g = torch.Generator().manual_seed(41)
    bns = [mod for mod in m.modules() if isinstance(mod, torch.nn.BatchNorm2d)]
    with torch.no_grad():
        for mod in bns:  # the mirror is cached across tests: restored below
            mod.running_mean.copy_(torch.randn(mod.running_mean.shape, generator=g) * 0.1)
            mod.running_var.copy_(torch.rand(mod.running_var.shape, generator=g) * 0.6 + 0.7)
    try:
        sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
        rgb = torch.randn(2, 3, *hw, generator=g)
        ref = restate.mpvit_backbone(sd, rgb.double().to(DEV), "mpvit_small")
        sizes = head.backbone_pyramid(hw, bb)
        assert [tuple(r.shape[-2:]) for r in ref] == sizes and head.can_run_backbone(bb, rgb.to(DEV))
        eng = head._engine(2, sizes[0], sizes[0], DEV, feats=([128, 216, 288, 288], sizes), image_hw=hw, backbone=bb)
        feats = eng.run_backbone(rgb.to(DEV), want_feats=True)
        eng.poll_status()
        errs = []
        for s, (f, r) in enumerate(zip(feats, ref)):
            assert f.shape == r.shape
            errs.append((f.double() - r).abs().max().item() / r.abs().max().item())
        print("[mpvit stages] rel err", ["%.2e" % e for e in errs])
        assert max(errs) < 1e-4, errs
        c1 = eng.build_condition(None, want_cond=True)
        cref = restate.fpn_condition(sd, restate.hahi_neck(sd, ref))
        err = (c1.double() - cref).abs().max().item() / cref.abs().max().item()
        assert err < 1e-4, err
        feats2 = eng.run_backbone(rgb.to(DEV), want_feats=True)
        assert all(torch.equal(a, b) for a, b in zip(feats, feats2)), "run-to-run determinism"
    finally:
        with torch.no_grad():
            for mod in bns:
                mod.running_mean.zero_()
                mod.running_var.fill_(1.0)


def test_producers_reject_unsupported_pyramids():
    eng = dd.DenoiseEngine("res", 1, (32, 48), (32, 48), 2, DEV)
    with pytest.raises(dd.EngineError, match="DD_ERR_UNSUPPORTED"):
        eng.enable_producers([64, 128, 256, 512], [(32, 48), (10, 19), (5, 10), (3, 5)], has_neck=False)  # > 2x jump
    with pytest.raises(dd.EngineError, match="DD_ERR_UNSUPPORTED"):
        eng.enable_producers([60, 128, 256, 512], [(32, 48), (16, 24), (8, 12), (4, 6)], has_neck=False)  # 60 % 8 != 0


# ------------------------------------------------------------------------------------------------ whole plugin
def _run_plugin(case, batch=None, fp8=True):
    g = helpers.load_golden(case)
    m = helpers.build_mirror(g["family"], g["T"], helpers.is_trained_case(case)).to(DEV)
    m.depth_head.fp8_corrections = fp8
    ck = helpers.weight_checksum({k: v.cpu() for k, v in m.state_dict().items()})
    assert abs(ck - float(g["z"]["weight_checksum"])) <= 1e-5 * ck, "regenerated weights differ from the golden's"
    B = batch or g["B"]
    sample = restate.synthetic_sample(B, g["H"], g["W"], configs.SEED_INPUTS)
    sample["noise"] = restate.synthetic_noise(B, g["H"], g["W"], configs.SEED_NOISE)
    sample = {k: v.to(DEV) for k, v in sample.items()}
    m.depth_head.capture_logits = True
    m.depth_head.capture_cond = True
    with torch.no_grad():
        out = m(sample)
    return g, m, out


@pytest.mark.parametrize("case", ["g_res18_c1", "g_res18_ragged", "g_swinl_small", "g_res50_c2", "g_swinl_c3",
                                  "g_swinl_c5", "g_swinl_add_small", "g_mpvit_small", "g_mpvit_trained", "g_res18_trained",
                                  "g_swinl_small_trained", "g_swinl_odd_trained"])
def test_plugin_forward_matches_reference_golden(case, parity_log):
    """`Diffusion_DCbase_Model.forward(sample)` on the GPU vs the real reference's own forward (golden).  `*_trained`:
    the trained-like regime (non-zero Swin relative-position tables, non-trivial BN statistics, LN / GN affines)."""
    g, m, out = _run_plugin(case)
    assert all(e.producers is not None for e in m.depth_head._engines.values()), \
        "neck + FPN must run on the engine for every family"
    z = m.depth_head.last_logits.cpu()
    z_ref = torch.from_numpy(g["z"]["logits"])
    dz = (helpers.golden_view(g, "logits", z) - z_ref).abs()
    lat_rel = (helpers.golden_view(g, "latent", m.depth_head.last_latent.cpu()) - torch.from_numpy(g["z"]["latent"])
               ).abs().max().item() / float(g["z"]["latent_absmax"])
    cond_rel = (helpers.golden_view(g, "cond", m.depth_head.last_cond.cpu()) - torch.from_numpy(g["z"]["cond"])
                ).abs().max().item() / float(g["z"]["cond_absmax"])
    parity_log(case, "reference golden (logits sub-sampled x%d)" % int(g["z"]["logits_stride"]), dz,
               latent_rel=lat_rel, cond_rel=cond_rel)
    assert dz.max().item() < TOL, f"{case}: max|dz| {dz.max().item():.3e}"
    pm = restate.parity_metrics(helpers.golden_view(g, "logits", z), z_ref, helpers.golden_view(g, "pred", out["pred"].cpu()),
                                torch.from_numpy(g["z"]["pred"]))
    assert pm["max_rel_depth_wellcond"] < TOL
    lat = helpers.golden_view(g, "latent", m.depth_head.last_latent.cpu())
    assert (lat - torch.from_numpy(g["z"]["latent"])).abs().max().item() < 5e-4 * float(g["z"]["latent_absmax"])
    cond = helpers.golden_view(g, "cond", m.depth_head.last_cond.cpu())
    assert (cond - torch.from_numpy(g["z"]["cond"])).abs().max().item() < 1e-4 * float(g["z"]["cond_absmax"])
    assert sorted(out.keys()) == sorted(str(k) for k in g["z"]["output_keys"])
    assert out["pred"].shape == (g["B"], 1, g["H"], g["W"]) and out["pred_init"].shape[1] == 16
    for k in ("pred_uncertainty", "pred_inter", "weight_map", "guidance", "offset", "aff", "gamma", "confidence"):
        assert out[k] is None


@pytest.mark.parametrize("case", ["g_res18_vis_trained", "g_swinl_vis_trained"])
def test_vis_plugin_matches_reference_golden(case, parity_log):
    """The `*Vis` heads through `Diffusion_DCbase_Model.forward` vs the REAL reference's Vis heads (goldens generated by
    oracle/make_golden.py from ..._res_vis.py / ..._swin_addHAHI_vis.py): the final logits as for the other heads, and
    `pred_inter` — the depth map the engine decodes after every DDIM step inside its captured graph
    (dd_denoise_decode_steps) — step by step against the reference's list."""
    g, m, out = _run_plugin(case)
    z = m.depth_head.last_logits.cpu()
    dz = (helpers.golden_view(g, "logits", z) - torch.from_numpy(g["z"]["logits"])).abs()
    parity_log(case, "reference golden (logits sub-sampled x%d)" % int(g["z"]["logits_stride"]), dz)
    assert dz.max().item() < TOL
    ref_inter = torch.from_numpy(g["z"]["pred_inter"])  # [T, B, 1, H, W]
    assert out["pred_inter"] is not None and len(out["pred_inter"]) == g["T"] == ref_inter.shape[0]
    worst = 0.0
    for i, d in enumerate(out["pred_inter"]):
        d, r = d.cpu(), ref_inter[i]
        assert d.shape == r.shape == (g["B"], 1, g["H"], g["W"])
        # depth = 1 / sigmoid(z) - 1 = exp(-z): relative depth error == |dz| where the reference's own fp32 evaluation is well
        # conditioned, -13 < z < 6 as in the other tests (below 2.5e-3 its `1 / sigmoid - 1` cancels: 6e-8 / depth)
        well = (r > 2.5e-3) & (r < 4.4e5)
        assert well.float().mean().item() > 0.25
        rel = ((d - r).abs() / r.clamp_min(1e-30))[well].max().item()
        worst = max(worst, rel)
        assert rel < TOL, (case, i, rel)
    assert torch.equal(out["pred"], out["pred_inter"][-1])
    print(f"[vis] {case}: max relative depth error over {g['T']} intermediate maps = {worst:.3e}")


@pytest.mark.parametrize("case", ["g_swinl_small", "g_swinl_c3", "g_swinl_c5", "g_swinl_small_trained", "g_swinl_odd_trained"])
def test_plugin_forward_exact_split_mode(case, parity_log):
    """The Swin goldens again with `fp8_corrections = False`: the exact 3-pass fp16 split everywhere (the round-1 path)."""
    g, m, out = _run_plugin(case, fp8=False)
    z_ref = torch.from_numpy(g["z"]["logits"])
    dz = (helpers.golden_view(g, "logits", m.depth_head.last_logits.cpu()) - z_ref).abs()
    cond_rel = (helpers.golden_view(g, "cond", m.depth_head.last_cond.cpu()) - torch.from_numpy(g["z"]["cond"])
                ).abs().max().item() / float(g["z"]["cond_absmax"])
    parity_log(case + " [exact 3-pass split]", "reference golden (logits sub-sampled x%d)" % int(g["z"]["logits_stride"]), dz,
               cond_rel=cond_rel)
    assert dz.max().item() < 5e-4, f"{case}: max|dz| {dz.max().item():.3e}"
    m.depth_head.fp8_corrections = True


def test_full_size_c3_batch_properties():
    """BASELINE config 3 (Swin-L, T=20, 4 x 352 x 1216): image 0 of the batch equals the batch-1 golden, images are
    independent of their batch neighbours, and the run is deterministic."""
    g, m, out = _run_plugin("g_swinl_c3", batch=4)
    z4 = m.depth_head.last_logits.clone()
    z_ref = torch.from_numpy(g["z"]["logits"])
    assert (helpers.golden_view(g, "logits", z4[:1].cpu()) - z_ref).abs().max().item() < TOL
    sample = restate.synthetic_sample(1, g["H"], g["W"], configs.SEED_INPUTS, first=2)
    sample["noise"] = restate.synthetic_noise(1, g["H"], g["W"], configs.SEED_NOISE, first=2)
    with torch.no_grad():
        m({k: v.to(DEV) for k, v in sample.items()})
    z1 = m.depth_head.last_logits
    assert (z1[0] - z4[2]).abs().max().item() < 2e-4  # same image alone vs inside a batch of 4
    _, m2, _ = _run_plugin("g_swinl_c3", batch=4)
    assert torch.equal(m2.depth_head.last_logits, z4)
    frac_clamped = (out["pred"] >= 999998.0).float().mean().item()
    assert abs(frac_clamped - float(g["z"]["frac_clamped"])) < 0.05  # random-init outputs saturate (SURVEY §7.2-2)


def _full_res_vs_restatement(family, T, B, H, W, images, parity_log, tag):
    """The plugin at the CONFIGURED batch; images `images` compared on ALL pixels (logits, latent, condition map) with
    the fp32 restatement (itself pinned to the real reference at 4e-6 .. 3e-5, oracle/make_golden.py)."""
    m = helpers.build_mirror(family, T).to(DEV)
    sample = restate.synthetic_sample(B, H, W, configs.SEED_INPUTS)
    sample["noise"] = restate.synthetic_noise(B, H, W, configs.SEED_NOISE)
    m.depth_head.capture_logits = m.depth_head.capture_cond = True
    m.depth_head.check_range = True
    with torch.no_grad():
        out = m({k: v.to(DEV) for k, v in sample.items()})
    z, lat, cond = (t.cpu() for t in (m.depth_head.last_logits, m.depth_head.last_latent, m.depth_head.last_cond))
    sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    bb = configs.FAMILIES[family]["backbone_name"]
    for i in images:
        one = {k: v[i:i + 1] for k, v in sample.items() if k != "noise"}
        ref = restate.forward(sd, one, bb, T, sample["noise"][i:i + 1])
        dz = (z[i:i + 1] - ref["logits"]).abs()
        parity_log(f"{tag} image {i} of {B}", "fp32 restatement, all %d pixels" % dz.numel(), dz)
        assert dz.max().item() < TOL, (tag, i, dz.max().item())
        assert (lat[i:i + 1] - ref["latent"]).abs().max().item() < 5e-4 * ref["latent"].abs().max().item()
        assert (cond[i:i + 1] - ref["cond"]).abs().max().item() < 1e-4 * ref["cond"].abs().max().item()
        pm = restate.parity_metrics(z[i:i + 1], ref["logits"], out["pred"][i:i + 1].cpu(), ref["pred"])
        assert pm["max_rel_depth_wellcond"] < TOL
    return m, out, z


def test_c3_full_resolution_every_pixel(parity_log):
    """BASELINE config 3 at full resolution (Swin-L, T=20, 352 x 1216): every pixel of the decoder logit against the
    restatement — the goldens keep 1/16 of the logits of the large cases, so a defect at odd tile coordinates would
    pass them (round-1 VERDICT)."""
    _full_res_vs_restatement("swinl", 20, 1, 352, 1216, [0], parity_log, "C3")


def test_c2_at_configured_batch(parity_log):
    """BASELINE config 2 as configured: ResNet-50, T=20, batch 8 x 228 x 304 — all 8 images, every pixel."""
    m, out, z = _full_res_vs_restatement("res50", 20, 8, 228, 304, list(range(8)), parity_log, "C2")
    g = helpers.load_golden("g_res50_c2")
    assert (helpers.golden_view(g, "logits", z[:1]) - torch.from_numpy(g["z"]["logits"])).abs().max().item() < TOL


def test_c5_at_configured_per_gpu_batch(parity_log):
    """BASELINE config 5 as configured per GPU: Swin-L, T=50, batch 8 x 480 x 640 (64 over 8 GPUs): image 0 against the
    real reference's golden, image 5 on every pixel against the restatement."""
    m, out, z = _full_res_vs_restatement("swinl", 50, 8, 480, 640, [5], parity_log, "C5")
    g = helpers.load_golden("g_swinl_c5")
    dz = (helpers.golden_view(g, "logits", z[:1]) - torch.from_numpy(g["z"]["logits"])).abs()
    parity_log("C5 image 0 of 8", "reference golden (logits sub-sampled x%d)" % int(g["z"]["logits_stride"]), dz)
    assert dz.max().item() < TOL
    assert out["pred"].shape == (8, 1, 480, 640)


def test_vis_head_and_ddim_loss_key():
    """`*Vis` heads (reference ..._swin_addHAHI_vis.py:130-149): `pred_inter` = inv_t of the latent after EVERY step,
    decoded inside the captured graph (dd_denoise_decode_steps) on the fully native path — against the same loop driven
    one step at a time through the bare operators (dd_denoiser_forward -> axpby -> dd_decode)."""
    from diffusiondepth_b200.model.registry import HEADS
    torch.manual_seed(7)
    T = 5
    vis = HEADS.build(dict(type="DDIMDepthEstimate_ResVis", in_channels=[64, 128, 256, 512], inference_steps=T,
                           num_train_timesteps=1000, depth_feature_dim=16, loss_cfgs=[], init_cfg=None)).eval().to(DEV)
    base = _res_head(T).to(DEV)
    base.load_state_dict(vis.state_dict())
    g = torch.Generator().manual_seed(9)
    fp = [torch.randn(1, c, -(-40 // s), -(-56 // s), generator=g).to(DEV) for c, s in
          ((64, 2), (128, 4), (256, 8), (512, 16))]
    gt = (torch.rand(1, 1, 40, 56, generator=g) * 80).to(DEV)
    noise = torch.randn(1, 16, 20, 28, generator=g).to(DEV)
    vis.capture_cond = True
    a = vis(fp, gt, gt > 0, gt_depth_map=gt, noise=noise)
    base.eval_ddim_loss = True
    b = base(fp, gt, gt > 0, gt_depth_map=gt, noise=noise)
    assert len(a["pred_inter"]) == T and a["pred_inter"][0].shape == (1, 1, 40, 56)
    assert torch.equal(a["pred"], a["pred_inter"][-1]) and torch.equal(a["pred"], b["pred"])
    assert torch.equal(vis.last_latent, base.last_latent)
    assert b["ddim_loss"].dim() == 0 and torch.isfinite(b["ddim_loss"]) and b["ddim_loss"] > 0
    # step by step through the bare operators
    eng = vis._any_engine(1, (20, 28), (20, 28), DEV)
    ts, cx, ce = vis.scheduler.fused_coefficients(T)
    x, cond = noise.clone(), vis.last_cond
    for i, (t, ca, cb) in enumerate(zip(ts, cx, ce)):
        x = (ca * x.double() + cb * eng.denoiser_forward(cond, x, t).double()).float().contiguous()
        d, z = eng.decode(x, want_logits=True)
        well = (z < 6) & (z > -13)
        rel = (a["pred_inter"][i] - d).abs() / d.abs().clamp_min(1e-6)
        assert rel[well].max().item() < 1e-3, (i, rel[well].max().item())
    # the Swin Vis head takes the fully native path as well (backbone included when called through the model)
    assert HEADS.get("DDIMDepthEstimate_Swin_ADDHAHIVis").return_intermediates


def test_vis_head_reports_range_overflow():
    """round-1 ADVICE: an overflow in an early step must not be cleared by a later one."""
    from diffusiondepth_b200.model.registry import HEADS
    torch.manual_seed(7)
    vis = HEADS.build(dict(type="DDIMDepthEstimate_ResVis", in_channels=[64, 128, 256, 512], inference_steps=3,
                           num_train_timesteps=1000, depth_feature_dim=16, loss_cfgs=[], init_cfg=None)).eval().to(DEV)
    g = torch.Generator().manual_seed(1)
    fp = [torch.full((1, c, 32 // s, 48 // s), 3.0e4, device=DEV) for c, s in ((64, 1), (128, 2), (256, 4), (512, 8))]
    gt = (torch.rand(1, 1, 64, 96, generator=g) * 80).to(DEV)
    with pytest.raises(dd.EngineError, match="DD_ERR_RANGE"):
        vis(fp, gt, gt > 0, gt_depth_map=gt)


def test_range_overflow_is_reported_not_silent():
    head = _res_head(2).to(DEV)
    g = torch.Generator().manual_seed(1)
    cond = torch.full((1, 256, 16, 32), 1.0e4)  # 1e4 * 16 > fp16 max
    noise = torch.randn(1, 16, 16, 32, generator=g)
    eng = head._engine(1, (16, 32), (16, 32), DEV)
    eng.denoise_decode(cond.to(DEV), noise.to(DEV))
    with pytest.raises(dd.EngineError, match="DD_ERR_RANGE"):
        eng.poll_status()


def test_weights_are_repacked_after_load_state_dict():
    head = _res_head(3).to(DEV)
    other = _res_head(3, seed=8).to(DEV)
    g = torch.Generator().manual_seed(2)
    cond, noise = torch.randn(1, 256, 16, 32, generator=g).abs().to(DEV), torch.randn(1, 16, 16, 32, generator=g).to(DEV)
    eng = head._engine(1, (16, 32), (16, 32), DEV)
    d1 = eng.denoise_decode(cond, noise)[0].clone()
    head.load_state_dict(other.state_dict())
    eng2 = head._engine(1, (16, 32), (16, 32), DEV)
    assert eng2 is eng
    d2 = eng2.denoise_decode(cond, noise)[0]
    d3 = other._engine(1, (16, 32), (16, 32), DEV).denoise_decode(cond, noise)[0]
    assert not torch.equal(d1, d2) and torch.equal(d2, d3)


def test_host_buffer_end_to_end_call():
    """The call a user makes (reference src/main.py:456-470): host sample -> .cuda() -> net(sample) -> host."""
    g = helpers.load_golden("g_res18_ragged")
    m = helpers.build_mirror(g["family"], g["T"]).to(DEV)
    sample = restate.synthetic_sample(g["B"], g["H"], g["W"], configs.SEED_INPUTS)
    sample["noise"] = restate.synthetic_noise(g["B"], g["H"], g["W"], configs.SEED_NOISE)
    pinned = {k: v.pin_memory() for k, v in sample.items()}
    with torch.no_grad():
        out = m({k: v.to(DEV, non_blocking=True) for k, v in pinned.items()})
    pred = out["pred"].cpu()
    ref = torch.from_numpy(g["z"]["pred"])
    z_ref = torch.from_numpy(g["z"]["logits"])
    rel = (pred - ref).abs() / ref.abs().clamp_min(1e-6)
    assert rel[(z_ref < 6) & (z_ref > -13)].max().item() < TOL


def test_one_step_loop_equals_operator_plus_update_plus_decode():
    """Size-independent property tying the three C-ABI entry points together: a T = 1 `dd_denoise_decode` must equal
    eps = `dd_denoiser_forward`(x_T, t_0) -> x_0 = c_x x_T + c_eps eps -> `dd_decode`(x_0), and depth = exp(-z)
    where it is well conditioned."""
    head = _swin_head(1).to(DEV)
    g = torch.Generator().manual_seed(11)
    B, (h, w) = 2, (24, 40)
    cond = torch.randn(B, 256, 12, 20, generator=g).abs().to(DEV)
    noise = torch.randn(B, 16, h, w, generator=g).to(DEV)
    eng = head._engine(B, (h, w), (12, 20), DEV)
    depth, latent, z = eng.denoise_decode(cond, noise, want_latent=True, want_logits=True)
    ts, cx, ce = head.scheduler.fused_coefficients(1)
    eps = eng.denoiser_forward(cond, noise, int(ts[0]))
    x0 = (cx[0] * noise.double() + ce[0] * eps.double()).float()
    assert (x0 - latent).abs().max().item() < 2e-5 * max(1.0, latent.abs().max().item())
    depth2, z2 = eng.decode(latent, want_logits=True)
    assert torch.equal(depth2, depth) and torch.equal(z2, z)
    well = (z < 6) & (z > -13)
    assert ((depth - torch.exp(-z)).abs() / torch.exp(-z))[well].max().item() < 1e-3
    eng.poll_status()


def test_cabi_rejects_bad_arguments_with_status_codes():
    """Error behaviour of the boundary: int status + dd_last_error(), never a crash or a silent fallback."""
    import ctypes as C
    from diffusiondepth_b200 import _cabi
    lib = _cabi.load_library()
    h = C.c_void_p()
    bad = _cabi.DDConfig(_cabi.ABI_VERSION + 7, _cabi.VARIANT_SWIN, 1, 8, 16, 4, 8, 2, 0, 0)
    assert lib.dd_create(C.byref(bad), C.byref(h)) != 0 and b"abi" in lib.dd_last_error().lower()
    res_mismatch = _cabi.DDConfig(_cabi.ABI_VERSION, _cabi.VARIANT_RES, 1, 8, 16, 4, 8, 2, 0, 0)
    assert lib.dd_create(C.byref(res_mismatch), C.byref(h)) != 0  # Res heads condition at latent resolution
    eng = dd.DenoiseEngine("swin", 1, (8, 16), (4, 8), 2, DEV, cuda_graph=False)
    noise = torch.zeros(1, 16, 8, 16, device=DEV)
    cond = torch.zeros(1, 256, 4, 8, device=DEV)
    with pytest.raises(dd.EngineError):  # weights never registered
        eng.denoise_decode(cond, noise)
    with pytest.raises(dd.EngineError):  # wrong shape is refused on the host side
        eng.denoise_decode(cond, torch.zeros(1, 16, 8, 17, device=DEV))
    head = _swin_head(2).to(DEV)
    eng.load_weights(head._engine_tensors())
    eng.set_schedule(*head.scheduler.fused_coefficients(2))
    depth = torch.empty(1, 1, 16, 32, device=DEV)
    small = torch.empty(4096, dtype=torch.uint8, device=DEV)
    rc = lib.dd_denoise_decode(eng._h, C.c_void_p(cond.data_ptr()), C.c_void_p(noise.data_ptr()), C.c_void_p(0),
                               C.c_void_p(0), C.c_void_p(depth.data_ptr()), C.c_void_p(small.data_ptr()), 4096,
                               C.c_void_p(0))
    assert rc != 0 and b"workspace" in lib.dd_last_error().lower()
    assert eng.denoise_decode(cond, noise)[0].shape == (1, 1, 16, 32)  # the handle is still usable afterwards
    eng.close()
