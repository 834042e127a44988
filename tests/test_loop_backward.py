"""dd_denoise_backward / dd_decode_backward: reverse mode through the DDIM sampling loop and the depth decoder.  Checked
against a Python chain of the merged operator backward (same engine, free of kinks), against fp64 autograd of the
restatement (itself pinned to the real reference by test_loop_grads_oracle.py), for determinism and argument checks,
and at head level through `grad_through_loop`."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from diffusiondepth_b200 import _cabi
from diffusiondepth_b200.engine import DECODER_PARAM_KEYS, DenoiseEngine
from grad_helpers import masked_restatement_grads, tensor_margins
from loop_grad_helpers import decode_restatement_grads, loop_restatement_grads, make_loop_head
from oracle import restate
from oracle.make_loop_grads import loop_state

DEV = torch.device("cuda:0")
TOL = 2e-4      # of max |g_ref| per gradient, engine vs fp64 restatement
CHAIN_TOL = 1e-5
BAND = 5e-5     # ReLU inputs this close to zero may land on the other side in the fp32-grade loop (kink envelope)
# dd_workspace_bytes of a DD_FLAG_BACKWARD engine (Res, B = 3, 8 x 16, T = 2), measured with the library of the commit
# before the loop backward existed: the loop backward must not grow it
BACKWARD_WS_BYTES = 8752128


def _inputs(variant, hw, B=3, seed=7):
    h, w = hw
    ch, cw = ((h + 1) // 2, (w + 1) // 2) if variant == "swin" else (h, w)
    g = torch.Generator().manual_seed(seed)
    cond = torch.randn(B, 256, ch, cw, generator=g).abs()
    noise = torch.randn(B, 16, h, w, generator=g)
    d_depth = torch.randn(B, 1, 2 * h, 2 * w, generator=g) * (1.0 / (B * 4 * h * w))
    d_latent = torch.randn(B, 16, h, w, generator=g) * (2.0 / (B * 16 * h * w))
    return cond, noise, d_depth, d_latent


def _loop_engine(head, B, hw, chw):
    return head._engine(B, hw, chw, DEV, loop_backward=True)


def _native(eng, cond, noise, d_depth, d_latent, want_latents=False):
    d_cond, d_noise, grads, lat = eng.denoise_backward(cond.to(DEV), noise.to(DEV),
                                                       d_depth.to(DEV) if d_depth is not None else None,
                                                       d_latent.to(DEV) if d_latent is not None else None,
                                                       want_latents=want_latents)
    eng.poll_status()
    out = {"d_cond": d_cond, "d_noise": d_noise}
    out.update(grads)
    return out, lat


def _report(tag, m, env=None):
    worst = max(m, key=m.get)
    extra = f" (env {env[worst]:.1e})" if env is not None else ""
    print(f"\n[{tag}] worst {worst} {m[worst]:.2e}{extra}; " +
          " ".join(f"{k.replace('model.', '').replace('depth_transform.conv_inv_transform', 'dec')}={v:.1e}"
                   for k, v in m.items()))


@pytest.mark.gpu
@pytest.mark.parametrize("variant,hw,T,B", [("swin", (19, 27), 3, 3), ("res", (19, 27), 3, 3), ("swin", (88, 304), 20, 2)])
def test_composition_of_operator_backwards(variant, hw, T, B):
    """At the engine's own latents the loop backward is T operator backwards, the c_x / c_eps recurrence and the decoder
    backward; latents_out[T] is dd_denoise_decode's latent bit for bit (with and without the CUDA graph)."""
    sd = loop_state(variant)
    head = make_loop_head(variant, sd, T, DEV)
    cond, noise, d_depth, d_latent = (x.to(DEV) for x in _inputs(variant, hw, B))
    chw = tuple(cond.shape[-2:])
    eng = _loop_engine(head, B, hw, chw)
    got, lat = _native(eng, cond, noise, d_depth, d_latent, want_latents=True)
    assert torch.equal(lat[0], noise)
    for graph in (True, False):
        head.use_cuda_graph = graph
        _, latent, _ = head._engine(B, hw, chw, DEV).denoise_decode(cond, noise, want_latent=True)
        assert torch.equal(lat[T], latent), graph
    ts, cx, ce = head.scheduler.fused_coefficients(T)
    d_lat_dec, ref = eng.decode_backward(lat[T].contiguous(), d_depth)
    ref = {k: v.double().cpu() for k, v in ref.items()}
    g = d_latent + d_lat_dec
    d_cond = torch.zeros_like(cond, dtype=torch.float64)
    for s in reversed(range(T)):
        dc, dn, gr = eng.denoiser_backward(cond, lat[s].contiguous(), ts[s], float(np.float32(ce[s])) * g)
        d_cond += dc.double()
        for k, v in gr.items():
            ref[k] = ref.get(k, 0) + v.double().cpu()
        g = float(np.float32(cx[s])) * g + dn
    ref.update(d_cond=d_cond.cpu(), d_noise=g.double().cpu())
    m = tensor_margins(got, ref)
    _report(f"chain {variant} {hw} T={T}", m)
    for k in m:
        assert m[k] <= CHAIN_TOL, (k, m[k])


# the last two run the wide layers' weight gradients over 6 and 5 split-K chunks, rows of 4 and 3 segments (the second
# with a 2-pixel tail segment)
CASES = [(v, hw, 3) for v in ("swin", "res") for hw in ((19, 27), (18, 26), (35, 53), (8, 16))] + [("swin", (19, 27), 20)]
CASES += [("swin", (64, 200), 3), ("res", (67, 130), 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("variant,hw,T", CASES)
def test_loop_gradients_vs_fp64_restatement(variant, hw, T):
    sd = loop_state(variant)
    cond, noise, d_depth, d_latent = _inputs(variant, hw)
    clamp = hw == (8, 16)
    if clamp:  # push part of the map below sigmoid(z) = 1e-6, where the clamp's gradient is zero
        p = {"depth_head." + k: v.double() for k, v in sd.items()}
        z = restate.decode_logits(p, restate.ddim_loop(p, cond.double(), noise.double(), T, variant))
        zs = z.flatten().sort().values
        n = zs.numel()
        gaps = zs[1:] - zs[:-1]
        i = int(gaps[n // 4: 3 * n // 4].argmax()) + n // 4  # put the threshold in the widest gap of the middle half
        thr = -13.815510557964274  # logit(1e-6)
        key = "depth_transform.conv_inv_transform.3.0.bias"
        sd[key] = sd[key] + (thr - float(zs[i] + zs[i + 1]) / 2)
        print(f"\n[clamp] {i + 1} of {n} pixels clamped; nearest logit {float(gaps[i]) / 2:.1e} from the threshold")
    head = make_loop_head(variant, sd, T, DEV)
    eng = _loop_engine(head, 3, hw, tuple(cond.shape[-2:]))
    got, lat = _native(eng, cond, noise, d_depth, d_latent, want_latents=True)
    ref = loop_restatement_grads(variant, sd, cond, noise, d_depth, d_latent, T)
    env = tensor_margins(loop_restatement_grads(variant, sd, cond, noise, d_depth, d_latent, T, band=BAND), ref)
    # The decoder's gradients depend on x_0 alone, which the fp32-grade loop reproduces to ~1e-4 (more at T = 20); the
    # final conv bias sums e^-z d_depth with heavy cancellation, so that drift shows in it beyond rounding.  Allow the
    # change the fp64 decoder gradients see between the fp64 x_0 and the engine's x_0.
    p = {"depth_head." + k: v.double() for k, v in sd.items()}
    x0 = restate.ddim_loop(p, cond.double(), noise.double(), T, variant)
    drift = tensor_margins(decode_restatement_grads(sd, lat[T].cpu(), d_depth),
                           decode_restatement_grads(sd, x0, d_depth))
    for k in DECODER_PARAM_KEYS:
        env[k] += drift[k] / 2
    m = tensor_margins(got, ref)
    _report(f"fp64 {variant} {hw} T={T}{' clamp' if clamp else ''}", m, env)
    for k in m:
        assert m[k] <= TOL + 2 * env[k], (k, m[k], env[k])
    rows = got["model.time_embedding.weight"].abs().sum(1).nonzero().flatten().tolist()
    assert rows == sorted(head.scheduler.fused_coefficients(T)[0])


# the last two run the wide layers' weight gradients over 6 and 5 split-K chunks (the second with a 2-pixel tail segment)
MASK_CASES = [("swin", (19, 27), 3), ("swin", (19, 27), 20), ("res", (35, 53), 3), ("swin", (64, 200), 3),
              ("res", (67, 130), 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("variant,hw,T", MASK_CASES)
def test_loop_gradients_vs_fp64_at_engine_masks(variant, hw, T):
    """d_latent only: the loop backward against an fp64 chain of operator VJPs at the engine's own latents, each step
    evaluated at the ReLU masks the engine's backward applied there (denoiser_relu_inputs on the same engine), so that
    rounding is the only difference left: no kink envelope."""
    sd = loop_state(variant)
    cond, noise, _, d_latent = _inputs(variant, hw)
    B = cond.shape[0]
    head = make_loop_head(variant, sd, T, DEV)
    eng = _loop_engine(head, B, hw, tuple(cond.shape[-2:]))
    got, lat = _native(eng, cond, noise, None, d_latent, want_latents=True)
    for k in DECODER_PARAM_KEYS:  # the depth does not enter the loss
        assert float(got[k].abs().max()) == 0.0, k
    ts, cx, ce = head.scheduler.fused_coefficients(T)
    msd = {k: v for k, v in sd.items() if k.startswith("model.")}
    c = cond.to(DEV)
    g = d_latent.double()
    ref = {"d_cond": torch.zeros(cond.shape, dtype=torch.float64)}
    flips = 0
    for s in reversed(range(T)):
        x = lat[s].contiguous()
        z = eng.denoiser_relu_inputs(c, x, ts[s])
        masks = [v.cpu() > 0 for v in z.values()]
        gr, z64 = masked_restatement_grads(variant, msd, x.cpu(), cond, [ts[s]] * B, float(np.float32(ce[s])) * g, masks)
        flips += sum(int((m != (zr > 0)).sum()) for m, zr in zip(masks, z64))
        ref["d_cond"] += gr["d_cond"]
        for k in msd:
            ref[k] = ref.get(k, 0) + gr[k]
        g = float(np.float32(cx[s])) * g + gr["d_noisy"]
    ref["d_noise"] = g
    m = tensor_margins(got, ref)
    _report(f"fp64 at engine masks {variant} {hw} T={T}; {flips} masks differ from fp64's", m)
    for k in m:
        assert m[k] <= 1e-4, (k, m[k])


@pytest.mark.gpu
def test_decode_backward_vs_fp64():
    sd = loop_state("res")
    head = make_loop_head("res", sd, 2, DEV)
    g = torch.Generator().manual_seed(9)
    hw = (13, 21)
    latent = torch.randn(2, 16, *hw, generator=g)
    d_depth = torch.randn(2, 1, 2 * hw[0], 2 * hw[1], generator=g)
    eng = _loop_engine(head, 2, hw, hw)
    d_lat, grads = eng.decode_backward(latent.to(DEV), d_depth.to(DEV))
    got = dict(grads, d_latent=d_lat)
    assert set(grads) == set(DECODER_PARAM_KEYS)
    ref = decode_restatement_grads(sd, latent, d_depth)
    env = tensor_margins(decode_restatement_grads(sd, latent, d_depth, band=BAND), ref)
    m = tensor_margins(got, ref)
    _report("decode", m, env)
    for k in m:
        assert m[k] <= 1e-5 + 2 * env[k], (k, m[k], env[k])


@pytest.mark.gpu
def test_deterministic_and_argument_checks():
    lib = _cabi.load_library()
    variant, hw, B = "res", (8, 16), 3
    sd = loop_state(variant)
    head = make_loop_head(variant, sd, 2, DEV)
    cond, noise, d_depth, d_latent = (x.to(DEV) for x in _inputs(variant, hw, B))
    eng = _loop_engine(head, B, hw, hw)
    a, lat_a = _native(eng, cond, noise, d_depth, d_latent, want_latents=True)
    b, lat_b = _native(eng, cond, noise, d_depth, d_latent, want_latents=True)
    assert torch.equal(lat_a, lat_b)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    # d_depth only / d_latent only are accepted; the decoder gradients are zero without d_depth
    _, _, gr, _ = eng.denoise_backward(cond, noise, None, d_latent)
    assert all(float(gr[k].abs().max()) == 0.0 for k in DECODER_PARAM_KEYS)
    eng.denoise_backward(cond, noise, d_depth, None)

    def call(e, dd=d_depth, dl=d_latent, nbytes=None):
        ws = e._workspace()
        n = ws.numel() - 1024 if nbytes is None else nbytes
        return lib.dd_denoise_backward(e._h, C.c_void_p(cond.data_ptr()), C.c_void_p(noise.data_ptr()),
                                       C.c_void_p(dd.data_ptr() if dd is not None else 0),
                                       C.c_void_p(dl.data_ptr() if dl is not None else 0), None, None, None, None, None,
                                       C.c_void_p(e._aligned(ws)), n, C.c_void_p(e._stream()))

    fwd = head._engine(B, hw, hw, DEV)
    bwd = head._engine(B, hw, hw, DEV, backward=True)
    assert call(fwd) == 1 and b"DD_FLAG_LOOP_BACKWARD" in lib.dd_last_error()
    assert call(bwd) == 1
    assert call(eng, dd=None, dl=None) == 1
    assert call(eng, nbytes=int(lib.dd_workspace_bytes(eng._h)) - 1) == 1 and b"workspace" in lib.dd_last_error()
    bare = DenoiseEngine(variant, B, hw, hw, 2, DEV, loop_backward=True)
    bare.load_weights(head._engine_tensors())
    assert call(bare) == 1 and b"dd_set_schedule" in lib.dd_last_error()
    assert call(eng) == 0
    torch.cuda.synchronize()
    assert int(lib.dd_workspace_bytes(eng._h)) > int(lib.dd_workspace_bytes(bwd._h)) > int(lib.dd_workspace_bytes(fwd._h))
    assert int(lib.dd_workspace_bytes(bwd._h)) == BACKWARD_WS_BYTES
    with pytest.raises(_cabi.EngineError):
        bwd.denoise_backward(cond, noise, d_depth, d_latent)


def _head_inputs(B=2, hw=(19, 27), seed=4):
    g = torch.Generator().manual_seed(seed)
    sizes = [hw, ((hw[0] + 1) // 2, (hw[1] + 1) // 2), ((hw[0] + 3) // 4, (hw[1] + 3) // 4),
             ((hw[0] + 7) // 8, (hw[1] + 7) // 8)]
    fp = [torch.randn(B, c, *s, generator=g).to(DEV) for c, s in zip((64, 128, 256, 512), sizes)]
    gt = (torch.rand(B, 1, 2 * hw[0], 2 * hw[1], generator=g) * 2 + 0.1).to(DEV)
    noise = torch.randn(B, 16, *hw, generator=g).to(DEV)
    return fp, gt, noise


def _run_head(head, fp, gt, noise, seed=21):
    torch.manual_seed(seed)  # ddim_loss draws its noise and t from the global RNG
    return head(fp, gt, gt > 0, gt_depth_map=gt, noise=noise)


@pytest.mark.gpu
def test_head_grad_through_loop_reaches_every_parameter():
    sd = loop_state("res")
    head = make_loop_head("res", sd, 2, DEV)
    head.train()
    fp, gt, noise = _head_inputs()
    out0 = _run_head(head, fp, gt, noise)
    lat0 = head.last_latent
    assert out0["pred"].grad_fn is None and lat0.grad_fn is None
    head.grad_through_loop = True
    out = _run_head(head, fp, gt, noise)
    assert torch.equal(out["pred"], out0["pred"]) and torch.equal(head.last_latent, lat0)
    assert out["pred"].grad_fn is not None
    head.zero_grad(set_to_none=True)
    (F.l1_loss(out["pred"], gt) + F.mse_loss(out["pred"], gt) + out["ddim_loss"]).backward()
    keys, params = head._loop_params()
    for k, p in zip(keys, params):
        assert p.grad is not None and float(p.grad.abs().max()) > 0, k
    # the operator backward of ddim_loss ran on the loop engine: no backward-only engine was created
    assert not any(key.backward for key in head._engines)


@pytest.mark.gpu
def test_vis_head_refuses_grad_through_loop():
    from diffusiondepth_b200.model.registry import HEADS
    head = HEADS.build(dict(type="DDIMDepthEstimate_ResVis", in_channels=[64, 128, 256, 512], inference_steps=2,
                            num_train_timesteps=1000, depth_feature_dim=16, loss_cfgs=[], init_cfg=None)).to(DEV)
    head.grad_through_loop = True
    fp, gt, noise = _head_inputs()
    with pytest.raises(_cabi.EngineError):
        _run_head(head, fp, gt, noise)


@pytest.mark.gpu
def test_sgd_on_depth_losses_tracks_fp64():
    variant, T = "res", 2
    sd = loop_state(variant)
    head = make_loop_head(variant, sd, T, DEV)
    head.train()
    head.grad_through_loop = True
    fp, gt, noise = _head_inputs()
    keys, params = head._loop_params()
    lr, steps = 0.05, 5
    opt = torch.optim.SGD(params, lr=lr)
    ref = {k: v.double().clone().requires_grad_("running" not in k) for k, v in sd.items()}
    rkeys = [k for k in keys]
    losses, ref_losses = [], []
    for _ in range(steps):
        opt.zero_grad()
        out = _run_head(head, fp, gt, noise)
        loss = F.l1_loss(out["pred"], gt) + F.mse_loss(out["pred"], gt)
        loss.backward()
        opt.step()  # in-place: the next forward re-packs the engines' weights
        losses.append(float(loss.detach()))
        cond = head.last_cond.double().cpu()
        p = {"depth_head." + k: v for k, v in ref.items()}
        pred = restate.decode(p, restate.ddim_loop(p, cond, noise.double().cpu(), T, variant))
        g64 = gt.double().cpu()
        rl = F.l1_loss(pred, g64) + F.mse_loss(pred, g64)
        gr = torch.autograd.grad(rl, [ref[k] for k in rkeys])
        with torch.no_grad():
            for k, gv in zip(rkeys, gr):
                ref[k] -= lr * gv
        ref_losses.append(float(rl))
    moved = {k: float((ref[k].detach() - sd[k].double()).abs().max()) for k in rkeys}
    got = dict(zip(keys, params))
    rel = {k: float((got[k].detach().double().cpu() - ref[k].detach()).abs().max()) / max(moved[k], 1e-30) for k in rkeys}
    worst = max(rel, key=rel.get)
    print(f"\n[train loop {variant}] losses {losses} (fp64 {ref_losses}); worst drift / movement: {worst} {rel[worst]:.2e}")
    assert losses[-1] < losses[0]
    assert abs(losses[0] - ref_losses[0]) <= 1e-4 * ref_losses[0]
    assert rel[worst] <= 1e-2
