"""The reference's other learned depth codecs on the engine (H100): dd_encode / dd_decode per codec kind against the
fp64 restatement (oracle/restate_codecs.py), the DDIM loop + decoder at the geometries each codec gives the Swin and
Res denoisers, the step decodes of the *Vis heads, in-place weight updates and the refusals."""
import ctypes as C

import pytest
import torch

from diffusiondepth_b200._cabi import EngineError
from diffusiondepth_b200.engine import CODEC_KEYS, DenoiseEngine
from diffusiondepth_b200.model.registry import HEADS
from oracle import configs, restate, restate_codecs

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
NAMES = {1: "DeepDepthTransformWithUpsampling1x1", 2: "DeepDepthTransformWithUpsamplingX4", 3: "DeepDepthTransform"}


def _head(kind, head="DDIMDepthEstimate_Swin_ADDHAHI", steps=3, seed=0, in_channels=(64, 128, 256, 512)):
    torch.manual_seed(seed)
    h = HEADS.build(dict(type=head, in_channels=list(in_channels), inference_steps=steps, num_train_timesteps=1000,
                         depth_feature_dim=16, loss_cfgs=[], init_cfg=None,
                         depth_transform_cfg=dict(type=NAMES[kind])))
    restate_codecs.trainedify_codec(h.depth_transform, seed)
    return h.eval().to(DEV)


def _sd(head):
    return {"depth_head." + k: v.detach().double().cpu() for k, v in head.state_dict().items()}


def _engine(head, batch, latent_hw, cond_hw, **kw):
    eng = DenoiseEngine(head.variant, batch, latent_hw, cond_hw, head.diffusion_inference_steps, DEV,
                        codec_kind=head._codec_kind(), **kw)
    eng.load_weights(head._engine_tensors())
    eng.set_schedule(*head.scheduler.fused_coefficients(head.diffusion_inference_steps))
    return eng


@pytest.mark.parametrize("kind", [1, 2, 3])
@pytest.mark.parametrize("B,H,W", [(1, 1, 1), (2, 37, 53), (4, 352, 1216)])
def test_encode_decode_vs_fp64(kind, B, H, W):
    """dd_encode / dd_decode against fp64 at a 1 x 1 latent, odd sizes and config-3 size, BN scales 1e-2 .. 1e2;
    the default codec's bounds (|dt| < 2e-5, |dz| < 1e-4 max(1, max|z|))."""
    head = _head(kind)
    sd = _sd(head)
    if H == 1:  # a 1 x 1 latent
        H = W = {1: 2, 2: 3, 3: 1}[kind]
    lat_hw = head.depth_transform.latent_hw((H, W))
    eng = _engine(head, B, lat_hw, (4, 4))
    g = torch.Generator().manual_seed(H * W + kind)
    depth = torch.rand(B, 1, H, W, generator=g) * 10
    latent = torch.randn(B, 16, *lat_hw, generator=g)
    t = eng.encode(depth.to(DEV))
    d, z = eng.decode(latent.to(DEV), want_logits=True)
    torch.cuda.synchronize()
    t64 = restate_codecs.encode(sd, depth.double(), kind)
    z64 = restate_codecs.decode_logits(sd, latent.double(), kind)
    dt = (t.cpu().double() - t64).abs().max().item()
    dz = (z.cpu().double() - z64).abs().max().item() / max(1.0, z64.abs().max().item())
    print(f"kind {kind} B{B} {H}x{W}: max|dt| {dt:.3e}, max|dz| / max(1, max|z|) {dz:.3e}")
    assert t.shape == t64.shape and z.shape == z64.shape == d.shape
    assert dt < 2e-5 and dz < 1e-4
    assert torch.equal(d, 1.0 / torch.sigmoid(z).clamp(1e-6) - 1) or \
        ((d - (1.0 / torch.sigmoid(z).clamp(1e-6) - 1)).abs() / (d.abs() + 1)).max().item() < 1e-5


# (kind, variant head, latent, cond): Swin + UP4 (cond at half the latent), Swin + FULL (cond upsampled 4x),
# MPViT-like Swin + UP4 (cond twice the latent: sampled down), Res + UP2_1X1 (cond == latent)
LOOPS = [(2, "DDIMDepthEstimate_Swin_ADDHAHI", (11, 19), (6, 10)),
         (3, "DDIMDepthEstimate_Swin_ADD", (24, 40), (6, 10)),
         (2, "DDIMDepthEstimate_MPVIT_ADDHAHI", (11, 19), (22, 38)),
         (1, "DDIMDepthEstimate_Res", (12, 20), (12, 20))]


@pytest.mark.parametrize("kind,head_name,lat,cond_hw", LOOPS)
def test_loop_and_decode_vs_fp64(kind, head_name, lat, cond_hw):
    head = _head(kind, head_name)
    sd = _sd(head)
    g = torch.Generator().manual_seed(5)
    noise = torch.randn(2, 16, *lat, generator=g)
    cond = torch.randn(2, 256, *cond_hw, generator=g).abs()
    eng = _engine(head, 2, lat, cond_hw)
    depth, latent, z = eng.denoise_decode(cond.to(DEV), noise.to(DEV), want_latent=True, want_logits=True)
    eng.poll_status()
    variant = "res" if head.variant == "res" else "swin"
    lat_ref = restate.ddim_loop(sd, cond.double(), noise.double(), 3, variant)
    z_ref = restate_codecs.decode_logits(sd, lat_ref, kind)
    err = (z.cpu().double() - z_ref).abs().max().item()
    print(f"{head_name} + {NAMES[kind]}: max|dz| {err:.3e}, latent {(latent.cpu().double() - lat_ref).abs().max():.3e}")
    assert depth.shape == (2, 1, eng.up * lat[0], eng.up * lat[1])
    assert err < 1e-3


@pytest.mark.parametrize("kind", [2, 3])
def test_config3_every_pixel(kind):
    """Swin_ADDHAHI + UP4 and Swin + FULL at BASELINE config-3 geometry (B = 4, 352 x 1216 depth), T = 3, every pixel
    of the logit against the fp64 restatement."""
    head = _head(kind, "DDIMDepthEstimate_Swin_ADDHAHI" if kind == 2 else "DDIMDepthEstimate_Swin_ADD")
    sd = _sd(head)
    lat = head.depth_transform.latent_hw((352, 1216))
    cond_hw = (44, 152)
    g = torch.Generator().manual_seed(9)
    noise = torch.randn(4, 16, *lat, generator=g)
    cond = torch.randn(4, 256, *cond_hw, generator=g).abs()
    eng = _engine(head, 4, lat, cond_hw)
    _, _, z = eng.denoise_decode(cond.to(DEV), noise.to(DEV), want_logits=True)
    eng.poll_status()
    worst = 0.0
    for b in range(4):  # one image at a time keeps the fp64 restatement's memory small
        lat_ref = restate.ddim_loop(sd, cond[b:b + 1].double(), noise[b:b + 1].double(), 3, "swin")
        z_ref = restate_codecs.decode_logits(sd, lat_ref, kind)
        worst = max(worst, (z[b:b + 1].cpu().double() - z_ref).abs().max().item())
    print(f"config 3, {NAMES[kind]}: latent {lat}, max|dz| over every pixel {worst:.3e}")
    assert z.shape == (4, 1, 352, 1216) and worst < 1e-3


def test_vis_pred_inter_x4():
    head = _head(2, "DDIMDepthEstimate_Swin_ADDHAHIVis")
    sd = _sd(head)
    lat, cond_hw = (9, 13), (5, 7)
    g = torch.Generator().manual_seed(11)
    noise, cond = torch.randn(1, 16, *lat, generator=g), torch.randn(1, 256, *cond_hw, generator=g).abs()
    eng = _engine(head, 1, lat, cond_hw, step_decode=True)
    steps, latent, _ = eng.denoise_decode_steps(cond.to(DEV), noise.to(DEV), want_latent=True)
    eng.poll_status()
    _, trace = restate.ddim_loop(sd, cond.double(), noise.double(), 3, "swin", collect=True)
    assert steps.shape == (3, 1, 1, 36, 52)
    for i, x in enumerate(trace):
        ref = restate_codecs.decode(sd, x, 2)
        well = ref < 1e3
        assert ((steps[i].cpu().double() - ref).abs() / (ref.abs() + 1))[well].max().item() < 1e-3


@pytest.mark.parametrize("kind", [1, 2, 3])
def test_update_weights_matches_fresh_pack(kind):
    """After an in-place change of codec tensors, update_weights gives outputs bit-identical to a fresh pack, and the
    loop graphs are kept (the new decoders read every constant from device memory)."""
    head = _head(kind)
    lat, cond_hw = head.depth_transform.latent_hw((30, 44)), (8, 11)
    g = torch.Generator().manual_seed(2)
    noise, cond = torch.randn(1, 16, *lat, generator=g).to(DEV), torch.randn(1, 256, *cond_hw, generator=g).abs().to(DEV)
    depth_in = (torch.rand(1, 1, 30, 44, generator=g) * 5).to(DEV)
    eng = _engine(head, 1, lat, cond_hw, step_decode=True)
    eng.denoise_decode(cond, noise)
    eng.denoise_decode_steps(cond, noise)
    captures = eng.graph_capture_count()
    enc_keys, dec_keys = CODEC_KEYS[kind]
    tensors = head._engine_tensors()
    changed = {}
    with torch.no_grad():
        for k in (enc_keys[0], dec_keys[0], dec_keys[-1]):
            tensors[k].mul_(1.25).add_(0.01)
            changed[k] = tensors[k]
    eng.update_weights(changed)
    a = eng.denoise_decode(cond, noise, want_logits=True)
    s = eng.denoise_decode_steps(cond, noise)[0]
    e = eng.encode(depth_in)
    # UP2_1X1 keeps the default decoder, whose final bias the step-decode graph holds by value: that graph alone is
    # captured again
    assert eng.graph_capture_count() == captures + (1 if kind == 1 else 0)
    fresh = _engine(head, 1, lat, cond_hw, step_decode=True)
    b = fresh.denoise_decode(cond, noise, want_logits=True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[2], b[2])
    assert torch.equal(s, fresh.denoise_decode_steps(cond, noise)[0])
    assert torch.equal(e, fresh.encode(depth_in))


def test_refusals():
    head = _head(2)
    lat = (5, 7)
    with pytest.raises(EngineError, match="DeepDepthTransformWithUpsamplingX4"):
        DenoiseEngine("swin", 1, lat, (3, 4), 3, DEV, loop_backward=True, codec_kind=2)
    eng = _engine(head, 1, lat, (3, 4), backward=True)
    with pytest.raises(EngineError, match="DD_CODEC_TRAIN"):
        eng.set_codec_mode(True)
    depth = torch.rand(1, 1, 20, 28, device=DEV)
    with pytest.raises(EngineError, match="no encoder backward"):
        eng.encode_backward(depth, torch.zeros(1, 16, *lat, device=DEV))
    buf = torch.zeros(1 << 20, device=DEV)
    ws = eng._workspace()
    rc = eng.lib.dd_decode_backward(eng._h, C.c_void_p(buf.data_ptr()), C.c_void_p(buf.data_ptr()), None, None,
                                    C.c_void_p(ws.data_ptr()), C.c_size_t(ws.numel()), C.c_void_p(0))
    assert rc == 3  # DD_ERR_UNSUPPORTED
    with pytest.raises(EngineError):  # the encoder's size check follows the codec's latent formula
        eng.encode(torch.rand(1, 1, 10, 14, device=DEV))
    with pytest.raises(EngineError, match="unknown weight key"):  # another kind's key
        eng.update_weights({"depth_transform.conv_inv_transform.3.0.weight": torch.zeros(1, 16, 3, 3)})
    # the denoiser operators do not involve the codec
    x = torch.randn(1, 16, *lat, device=DEV)
    eps = eng.denoiser_forward(torch.rand(1, 256, 3, 4, device=DEV), x, [500])
    assert eps.shape == x.shape and torch.isfinite(eps).all()


def test_head_forward_x4_native():
    """A Swin_ADDHAHI head with the X4 codec end to end on the engine: latent at a quarter of the depth map."""
    head = _head(2, in_channels=(192, 384, 768, 1536))  # the HAHI neck's Swin-L widths
    fp = [torch.randn(1, c, 44 // 2 ** i, 64 // 2 ** i, device=DEV).abs() for i, c in enumerate((192, 384, 768, 1536))]
    gt = torch.rand(1, 1, 88, 128, device=DEV) * 10
    head.capture_logits = True
    out = head(fp, None, None, gt_depth_map=gt)
    assert out["pred"].shape == (1, 1, 88, 128)
    assert out["gt_map_t"].shape == (1, 16, 22, 32)
    assert torch.isfinite(out["pred"]).all()


# ------------------------------------------------------------------ against the real reference (g_codec_kinds.npz)
def _golden():
    import numpy as np
    import os
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "g_codec_kinds.npz"))


@pytest.mark.parametrize("kind", [1, 2, 3])
def test_codec_vs_reference_golden(kind):
    """dd_encode / dd_decode against the real reference's `t` / `inv_t` (oracle/make_codec_kinds.py) at an even and
    an odd size; the bound on t is the reference's own fp32 rounding with BatchNorm scales up to 1e2."""
    from oracle import make_codec_kinds as mk
    g = _golden()
    head = _head(kind)
    head.depth_transform.load_state_dict(mk.mirror_codec(kind).state_dict())
    for hw in mk.CODEC_SIZES:
        depth, latent = mk.codec_inputs(kind, hw)
        eng = _engine(head, 1, latent.shape[-2:], (4, 4))
        t = eng.encode(depth.to(DEV)).cpu().double()
        _, z = eng.decode(latent.to(DEV), want_logits=True)
        t_ref = torch.from_numpy(g[f"codec{kind}_{hw[0]}x{hw[1]}_t"]).double()
        z_ref = torch.from_numpy(g[f"codec{kind}_{hw[0]}x{hw[1]}_z"]).double()
        dt, dz = (t - t_ref).abs().max().item(), (z.cpu().double() - z_ref).abs().max().item()
        print(f"{NAMES[kind]} {hw}: vs reference |dt| {dt:.2e}, |dz| {dz:.2e}")
        assert dt < 2e-4 and dz < 1e-4 * max(1.0, z_ref.abs().max().item())


@pytest.mark.parametrize("case", ["swinl_x4", "swinl_add_full", "res18_1x1", "mpvit_x4", "swinl_vis_x4"])
def test_head_matches_reference_golden(case):
    """`Diffusion_DCbase_Model.forward(sample)` of the mirror with the case's codec, everything native on the engine
    (backbone where it runs natively, neck, FPN, encoder, loop, decoder), against the real reference's forward: max |dz|
    on the decoder logit < 1e-3, the final latent, `pred_init` (the encoder through the head) and the Vis head's
    `pred_inter`."""
    from oracle import make_codec_kinds as mk
    g = _golden()
    family, kind, T, B, H, W = mk.HEAD_CASES[case]
    m = mk.build_mirror_model(family, kind, T).to(DEV)
    sample = restate.synthetic_sample(B, H, W, configs.SEED_INPUTS)
    sample["noise"] = mk.head_noise(kind, B, H, W)
    sample = {k: v.to(DEV) for k, v in sample.items()}
    head = m.depth_head
    head.capture_logits = True
    with torch.no_grad():
        out = m(sample)
    assert all(e.producers is not None for e in head._engines.values()), "neck + FPN must run on the engine"
    assert all(e.codec_kind == kind for e in head._engines.values())
    s = int(g["stride"])
    z_ref = torch.from_numpy(g[case + "_logits"])
    dz = (head.last_logits.cpu()[..., ::s, ::s] - z_ref).abs().max().item()
    lat_ref = torch.from_numpy(g[case + "_latent"])
    dlat = (head.last_latent.cpu()[..., ::s, ::s] - lat_ref).abs().max().item() / lat_ref.abs().max().item()
    dinit = (out["pred_init"].cpu()[:, ::4, ::s, ::s] - torch.from_numpy(g[case + "_pred_init"])).abs().max().item()
    print(f"{case}: max|dz| {dz:.2e} (|z| up to {float(g[case + '_logits_absmax']):.1f}), latent rel {dlat:.2e}, "
          f"pred_init {dinit:.2e}")
    assert out["pred"].shape == (B, 1, H, W)
    assert dz < 1e-3 and dlat < 1e-3 and dinit < 2e-4
    if case + "_pred_inter" in g:
        ref = torch.from_numpy(g[case + "_pred_inter"]).double()
        got = torch.stack(out["pred_inter"]).cpu()[..., ::s, ::s].double()
        well = ref < 1e3
        assert got.shape == ref.shape
        assert ((got - ref).abs() / (ref.abs() + 1))[well].max().item() < 1e-3


def test_set_weight_rejects_other_kinds_keys_and_kind0_workspace():
    """dd_set_weight itself (not the Python pre-check) rejects a key of another codec; the workspace of kind 0 is the
    parent engine's: the step-decode region is T x B x 2h x 2w floats, as before codec kinds existed."""
    head = _head(2)
    eng = _engine(head, 1, (5, 7), (3, 4))
    w = torch.zeros(1, 16, 3, 3, device=DEV)
    shape = (C.c_int64 * 4)(*w.shape)
    for key in (b"depth_transform.conv_inv_transform.3.0.weight", b"depth_transform.conv_transform.0.weight"):
        assert eng.lib.dd_set_weight(eng._h, key, C.c_void_p(w.data_ptr()), shape, 4) == 1  # DD_ERR_INVALID
    assert eng.lib.dd_set_weight(eng._h, b"depth_transform.conv_inv_transform.4.0.weight", C.c_void_p(w.data_ptr()),
                                 shape, 4) == 0
    T, B, h, wd = 3, 2, 24, 40
    sizes = {}
    for kind in (0, 1, 2, 3):
        for step in (False, True):
            e = DenoiseEngine("swin", B, (h, wd), (12, 20), T, DEV, step_decode=step, codec_kind=kind)
            sizes[kind, step] = int(e.lib.dd_workspace_bytes(e._h))
            e.close()
    for kind, u in ((0, 2), (1, 2), (2, 4), (3, 1)):
        assert sizes[kind, False] == sizes[0, False]
        assert sizes[kind, True] - sizes[kind, False] == -(-T * B * (u * h) * (u * wd) * 4 // 1024) * 1024  # 1 KB carve
