"""Training-mode BatchNorm of the depth codec (dd_set_codec_mode(DD_CODEC_TRAIN), head.codec_train_bn): batch
statistics, the forward outputs, the decoder backward through the statistics and the running-statistic updates, against
the fp64 training-mode restatement (codec_train_helpers, pinned to the reference by test_codec_train_oracle.py) and the
reference's own golden; the running-update helper and the re-pack decision also on the CPU."""
import ctypes as C

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from codec_train_helpers import DEC, decode_train, decode_train_grads, encode_train, loop_train_grads
from diffusiondepth_b200 import _cabi
from diffusiondepth_b200.engine import DECODER_PARAM_KEYS
from diffusiondepth_b200.model.head._ddim_head import bn_running_update, repack_plan

DEV = torch.device("cuda:0")
BAND = 5e-5  # ReLU inputs this close to zero may land on the other side in fp32 (kink envelope)


def _codec_state(head, dtype=torch.float64):
    return {k: v.detach().cpu().to(dtype) for k, v in head.state_dict().items() if k.startswith("depth_transform.")}


def _make_head(variant="res", T=2, seed=0):
    from diffusiondepth_b200.model.registry import HEADS
    torch.manual_seed(seed)
    kind = {"res": "DDIMDepthEstimate_Res", "swin": "DDIMDepthEstimate_Swin_ADDHAHI",
            "resvis": "DDIMDepthEstimate_ResVis"}[variant]
    head = HEADS.build(dict(type=kind, in_channels=[64, 128, 256, 512], inference_steps=T, num_train_timesteps=1000,
                            depth_feature_dim=16, loss_cfgs=[], init_cfg=None))
    with torch.no_grad():  # non-trivial BatchNorm affines and running statistics
        for bn in head._codec_bns():
            bn.weight.uniform_(0.5, 1.5)
            bn.bias.uniform_(-0.3, 0.3)
            bn.running_mean.uniform_(-0.2, 0.2)
            bn.running_var.uniform_(0.5, 2.0)
    return head.to(DEV)


def _stat_errors(rec, ref):
    """(max |mean - mean_ref| / sigma, max |var - var_ref| / var_ref) of one record [2][16] against (mean, var)."""
    mean, var = (t.detach().double().cpu() for t in rec)
    sigma = ref[1].sqrt()
    return float(((mean - ref[0]).abs() / sigma).max()), float(((var - ref[1]).abs() / ref[1]).max())


# ------------------------------------------------------------------ CPU
@pytest.mark.parametrize("momentum", [0.1, None])
def test_running_update_matches_torch(momentum):
    g = torch.Generator().manual_seed(3)
    ours, ref = nn.BatchNorm2d(16, momentum=momentum), nn.BatchNorm2d(16, momentum=momentum)
    ref.train()
    for _ in range(3):
        x = torch.randn(2, 16, 5, 7, generator=g) * 3 + 1
        ref(x)
        bn_running_update(ours, x.mean((0, 2, 3)), x.var((0, 2, 3), unbiased=True))
    assert int(ours.num_batches_tracked) == int(ref.num_batches_tracked) == 3
    torch.testing.assert_close(ours.running_mean, ref.running_mean, rtol=1e-6, atol=1e-7)
    torch.testing.assert_close(ours.running_var, ref.running_var, rtol=1e-6, atol=1e-7)


def test_running_statistics_change_is_an_update_not_a_load():
    from diffusiondepth_b200.model.registry import HEADS
    head = HEADS.build(dict(type="DDIMDepthEstimate_Res", in_channels=[64, 128, 256, 512], inference_steps=2,
                            num_train_timesteps=1000, depth_feature_dim=16, loss_cfgs=[], init_cfg=None))
    tensors = head._engine_tensors()
    keys, sig = list(tensors), [(t.data_ptr(), t._version) for t in tensors.values()]
    bn = head._codec_bns()
    for b in bn:
        bn_running_update(b, torch.zeros(16), torch.ones(16))
    new_sig = [(t.data_ptr(), t._version) for t in head._engine_tensors().values()]
    changed = repack_plan(keys, sig, keys, new_sig)
    assert changed is not None
    assert sorted(changed) == sorted(k for k in keys if "running_" in k)


def test_codec_bn_eps_is_checked():
    from diffusiondepth_b200.model.registry import HEADS
    head = HEADS.build(dict(type="DDIMDepthEstimate_Res", in_channels=[64, 128, 256, 512], inference_steps=2,
                            num_train_timesteps=1000, depth_feature_dim=16, loss_cfgs=[], init_cfg=None))
    assert not head._codec_training()  # flag off
    head.codec_train_bn = True
    assert head._codec_training()
    head.depth_transform.eval()
    assert not head._codec_training()
    head.depth_transform.train()
    head.depth_transform.conv_inv_transform[1].eps = 1e-3
    with pytest.raises(_cabi.EngineError):
        head._codec_training()


# ------------------------------------------------------------------ GPU: the engine entries
def _engine(head, B, hw, loop_backward=False):
    eng = head._engine(B, hw, hw, DEV, loop_backward=loop_backward)
    eng.set_codec_mode(True)
    return eng


@pytest.mark.gpu
def _latent_dc_case(head, latent, offset):
    """Weights and a latent whose ConvT output ITSELF (without the bias) has |mean| = offset * std in every channel:
    only the taps (ky, kx) in {1, 2}^2 carry weight, all four the same matrix M, so every output pixel sees exactly one
    latent pixel through M (no border effect), and the latent carries a per-channel DC offset o with o^T M =
    offset * |M[:, co]|.  Returns the offset latent."""
    with torch.no_grad():
        w = head.depth_transform.conv_inv_transform[0].weight
        m = w[:, :, 1, 1].detach().cpu().double()
        w.zero_()
        for ky in (1, 2):
            for kx in (1, 2):
                w[:, :, ky, kx] = m.float().to(w.device)
        o = torch.linalg.solve(m.T, offset * m.norm(dim=0))
    return latent + o.float()[None, :, None, None]


@pytest.mark.gpu
@pytest.mark.parametrize("B,hw,offset,where", [(2, (13, 21), 0.0, None), (3, (35, 53), 0.0, None),
                                               (4, (176, 608), 0.0, None), (2, (88, 304), 1e3, "bias"),
                                               (2, (176, 608), 1e3, "latent")])
def test_decode_train_vs_fp64(B, hw, offset, where):
    head = _make_head()
    g = torch.Generator().manual_seed(11)
    latent = torch.randn(B, 16, *hw, generator=g)
    if where == "bias":  # u = ConvT + b with |mean| ~ offset * std from the bias (added to the mean in fp64)
        with torch.no_grad():
            u = F.conv_transpose2d(latent, head.depth_transform.conv_inv_transform[0].weight.cpu(), None, 2, 1)
            head.depth_transform.conv_inv_transform[0].bias.copy_(offset * u.std((0, 2, 3)))
    if where == "latent":  # the statistics kernel itself sees |mean| ~ offset * std: E[u^2] - mean^2 would cancel
        latent = _latent_dc_case(head, latent, offset)
    p = _codec_state(head)
    eng = _engine(head, B, hw)
    depth, z = eng.decode(latent.to(DEV), want_logits=True)
    rec = eng.codec_batch_stats()
    _, z_ref, stats = decode_train(p, latent.double())
    dmean, dvar = _stat_errors(rec[0], stats)
    dz = float((z.double().cpu() - z_ref).abs().max() / z_ref.abs().max())
    # the record is fp32: a mean of ~offset * sigma carries its own rounding, 2^-24 |mean|
    rounding = float((stats[0].abs() / stats[1].sqrt()).max()) * 2.0 ** -24
    # with the DC offset in the latent, the fp32 forward (decoder_kernel on the folded weights, or torch's own fp32
    # BatchNorm) loses ~offset ulps to the cancellation of the mean: the bound on z is that of torch in fp32
    z_tol = 1e-5
    if where == "latent":
        _, z32, _ = decode_train({k: v.float() for k, v in p.items()}, latent)
        z_tol += 4 * float((z32.double() - z_ref).abs().max() / z_ref.abs().max())
    print(f"\n[decode train B={B} {hw} offset={offset} in {where}] mean {dmean:.1e} sigma (fp32 rounding "
          f"{rounding:.1e}), var {dvar:.1e} rel, |dz| {dz:.1e} max|z| (bound {z_tol:.1e})")
    assert rec.shape == (1, 2, 16)
    assert dmean <= 1e-6 + rounding and dvar <= 1e-5 and dz <= z_tol
    # eval mode afterwards: the running-statistics decode again, and no record
    eng.set_codec_mode(False)
    _, z_eval = eng.decode(latent.to(DEV), want_logits=True)
    assert eng.codec_batch_stats().shape[0] == 0
    assert not torch.equal(z_eval, z)


@pytest.mark.gpu
@pytest.mark.parametrize("B,hw", [(2, (13, 21)), (4, (176, 608))])
def test_encode_train_vs_fp64(B, hw):
    head = _make_head()
    g = torch.Generator().manual_seed(12)
    gt = torch.rand(B, 1, 2 * hw[0], 2 * hw[1], generator=g) * 80 + 0.5
    p = _codec_state(head)
    eng = _engine(head, B, hw)
    lat = eng.encode(gt.to(DEV))
    rec = eng.codec_batch_stats()
    ref, stats = encode_train(p, gt.double())
    errs = [_stat_errors(rec[i], stats[i]) for i in range(2)]
    dl = float((lat.double().cpu() - ref).abs().max() / ref.abs().max())
    print(f"\n[encode train B={B} {hw}] stats {errs}, |dlatent| {dl:.1e}")
    assert rec.shape == (2, 2, 16)
    for dmean, dvar in errs:
        assert dmean <= 1e-6 and dvar <= 1e-5
    assert dl <= 1e-5


def _margins(got, ref):
    return {k: float((got[k].detach().double().cpu() - ref[k]).abs().max() / ref[k].abs().max().clamp_min(1e-300))
            for k in ref}


@pytest.mark.gpu
def test_decode_backward_train_vs_fp64():
    head = _make_head()
    B, hw = 2, (13, 21)
    g = torch.Generator().manual_seed(9)
    latent = torch.randn(B, 16, *hw, generator=g)
    d_depth = torch.randn(B, 1, 2 * hw[0], 2 * hw[1], generator=g)
    p = _codec_state(head)
    eng = _engine(head, B, hw, loop_backward=True)
    d_lat, grads = eng.decode_backward(latent.to(DEV), d_depth.to(DEV))
    got = dict(grads, d_latent=d_lat)
    ref = decode_train_grads(p, latent, d_depth)
    env = _margins(decode_train_grads(p, latent, d_depth, band=BAND), ref)
    bias_key = DEC + "0.bias"
    ref_nb = {k: v for k, v in ref.items() if k != bias_key}
    m = _margins(got, ref_nb)
    db = float(got[bias_key].abs().max() / got[DEC + "0.weight"].abs().max())
    print(f"\n[decode bwd train] {m} env {env}; |d b_t| / max |dW_t| = {db:.1e}")
    for k in m:
        assert m[k] <= 1e-5 + 2 * env[k], (k, m[k], env[k])
    assert db <= 1e-6
    # bit-reproducible
    d_lat2, grads2 = eng.decode_backward(latent.to(DEV), d_depth.to(DEV))
    assert torch.equal(d_lat, d_lat2) and all(torch.equal(grads[k], grads2[k]) for k in grads)


@pytest.mark.gpu
def test_denoise_backward_train_matches_decode_backward_at_x0():
    """The loop backward's decoder part in training mode is dd_decode_backward's at the loop's own x_0, bit for bit;
    its decode recompute records nothing."""
    head = _make_head()
    B, hw, T = 2, (8, 16), 2
    head.diffusion_inference_steps = T
    g = torch.Generator().manual_seed(5)
    cond = torch.randn(B, 256, *hw, generator=g).abs().to(DEV)
    noise = torch.randn(B, 16, *hw, generator=g).to(DEV)
    d_depth = torch.randn(B, 1, 2 * hw[0], 2 * hw[1], generator=g).to(DEV)
    eng = _engine(head, B, hw, loop_backward=True)
    depth, latent, _ = eng.denoise_decode(cond, noise, want_latent=True)
    rec = eng.codec_batch_stats().clone()
    _, _, grads, lats = eng.denoise_backward(cond, noise, d_depth, None, want_latents=True)
    assert torch.equal(lats[-1], latent)
    assert torch.equal(eng.codec_batch_stats(), rec)  # backward records nothing
    _, dgrads = eng.decode_backward(latent, d_depth)
    for k in DECODER_PARAM_KEYS:
        assert torch.equal(grads[k], dgrads[k]), k
    # and the forward's depth is the train-mode decode of its latent
    d2, _ = eng.decode(latent)
    assert torch.equal(d2, depth) and torch.equal(eng.codec_batch_stats(), rec)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["swin_19x27", "res_19x27"])
def test_denoise_backward_train_vs_golden_and_fp64(case):
    """dd_denoise_backward in DD_CODEC_TRAIN (T = 3, B = 3) against the real reference's gradients with its codec in
    .train() (g_codec_train.npz) and the fp64 training-mode chain, under the bounds of the eval-mode loop tests
    (test_loop_backward.py: 2e-4 of max |g| plus the kink envelope; the decoder's part also allows the drift of the
    fp32-grade x_0); and the decoder's gradients against the fp64 training-mode decoder at the engine's own x_0."""
    import numpy as np
    from grad_helpers import golden_margins, tensor_margins
    from loop_grad_helpers import make_loop_head
    from oracle.make_codec_train import OUT
    from oracle.make_loop_grads import STEPS, case_inputs
    tol, bias = 2e-4, DEC + "0.bias"
    golden = np.load(OUT, allow_pickle=False)
    variant, sd, cond, noise, d_depth, d_latent = case_inputs(case)
    head = make_loop_head(variant, sd, STEPS, DEV)
    eng = head._engine(cond.shape[0], noise.shape[-2:], cond.shape[-2:], DEV, loop_backward=True)
    eng.set_codec_mode(True)
    d_cond, d_noise, grads, lat = eng.denoise_backward(cond.to(DEV), noise.to(DEV), d_depth.to(DEV), d_latent.to(DEV),
                                                       want_latents=True)
    eng.poll_status()
    got = dict(grads, d_cond=d_cond, d_noise=d_noise)
    ref = loop_train_grads(variant, sd, cond, noise, d_depth, d_latent, STEPS)
    env = tensor_margins(loop_train_grads(variant, sd, cond, noise, d_depth, d_latent, STEPS, band=BAND), ref)
    x0 = lat[STEPS].cpu()
    dec64 = decode_train_grads(sd, x0, d_depth)
    dec_env = tensor_margins(decode_train_grads(sd, x0, d_depth, band=BAND), dec64)
    p = {"depth_head." + k: v.double() for k, v in sd.items()}
    from oracle import restate
    drift = tensor_margins(dec64, decode_train_grads(sd, restate.ddim_loop(p, cond.double(), noise.double(), STEPS,
                                                                            variant), d_depth))
    for k in DECODER_PARAM_KEYS:
        env[k] += drift[k] / 2
    db = float(got[bias].abs().max() / got[DEC + "0.weight"].abs().max())
    for m in (ref, env):
        m.pop(bias)
    m64 = tensor_margins(got, ref)
    mg = golden_margins(golden, case, got)
    mg.pop(bias)
    md = tensor_margins({k: got[k] for k in DECODER_PARAM_KEYS if k != bias},
                        {k: dec64[k] for k in DECODER_PARAM_KEYS if k != bias})
    wf, wg = max(m64, key=lambda k: m64[k] - 2 * env[k]), max(mg, key=lambda k: mg[k] - 2 * env[k])
    print(f"\n[loop bwd train {case}] vs fp64 worst {wf} {m64[wf]:.1e} (env {env[wf]:.1e}), vs reference worst {wg} "
          f"{mg[wg]:.1e} (env {env[wg]:.1e}), decoder vs fp64 at x_0 worst {max(md.values()):.1e}; |d b_t| / max |dW_t| {db:.1e}")
    for k in m64:
        assert m64[k] <= tol + 2 * env[k], (k, m64[k], env[k])
    for k in mg:  # d_cond and the parameters (the golden holds no d_noise)
        assert mg[k] <= tol + 2 * env[k], (k, mg[k], env[k])
    for k in md:
        assert md[k] <= 1e-5 + 2 * dec_env[k], (k, md[k], dec_env[k])
    assert db <= 1e-6


@pytest.mark.gpu
def test_deterministic_and_argument_checks():
    lib = _cabi.load_library()
    head = _make_head()
    B, hw = 2, (13, 21)
    g = torch.Generator().manual_seed(2)
    latent = torch.randn(B, 16, *hw, generator=g).to(DEV)
    gt = (torch.rand(B, 1, 2 * hw[0], 2 * hw[1], generator=g) * 10 + 0.5).to(DEV)
    eng = _engine(head, B, hw)
    outs = []
    for _ in range(2):
        d, z = eng.decode(latent, want_logits=True)
        r1 = eng.codec_batch_stats().clone()
        lt = eng.encode(gt)
        r2 = eng.codec_batch_stats().clone()
        outs.append((d, z, r1, lt, r2))
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    ws_train = int(lib.dd_workspace_bytes(eng._h))
    assert lib.dd_set_codec_mode(eng._h, 2) == 1 and lib.dd_set_codec_mode(eng._h, -1) == 1
    eng.set_codec_mode(False)
    assert int(lib.dd_workspace_bytes(eng._h)) == ws_train
    n = C.c_int32()
    assert lib.dd_codec_batch_stats(eng._h, None, 0, C.byref(n), None) == 1  # the last encode wrote 2 records
    assert lib.dd_codec_batch_stats(eng._h, None, 0, None, None) == 1
    assert eng.codec_batch_stats().shape == (2, 2, 16)
    # one value per channel in the encoder: refused in training mode only
    one = _make_head()
    e1 = one._engine(1, (1, 1), (1, 1), DEV)
    depth1 = torch.rand(1, 1, 2, 2, device=DEV) + 0.5
    e1.encode(depth1)
    e1.set_codec_mode(True)
    with pytest.raises(_cabi.EngineError, match="more than 1 value"):
        e1.encode(depth1)


# ------------------------------------------------------------------ GPU: the head
def _head_inputs(head, B=2, hw=(19, 27), seed=4):
    g = torch.Generator().manual_seed(seed)
    sizes = [hw, ((hw[0] + 1) // 2, (hw[1] + 1) // 2), ((hw[0] + 3) // 4, (hw[1] + 3) // 4),
             ((hw[0] + 7) // 8, (hw[1] + 7) // 8)]
    fp = [torch.randn(B, c, *s, generator=g).to(DEV) for c, s in zip(head.fpn_in_channels, sizes)]
    gt = (torch.rand(B, 1, 2 * hw[0], 2 * hw[1], generator=g) * 2 + 0.1).to(DEV)
    noise = torch.randn(B, 16, *hw, generator=g).to(DEV)
    return fp, gt, noise


def _run_head(head, fp, gt, noise, seed=21):
    torch.manual_seed(seed)
    return head(fp, gt, gt > 0, gt_depth_map=gt, noise=noise)


def _expected_running(bn0, stats, momentum=0.1):
    mean, var = stats
    return (1 - momentum) * bn0[0] + momentum * mean, (1 - momentum) * bn0[1] + momentum * var


def _rel(a, b):
    return float(((a.detach().double().cpu() - b).abs() / b.abs().clamp_min(1e-12)).max())


def _running_errors(bn, mean, var):
    """(max |running_mean - mean| / sqrt(var), max |running_var - var| / var)"""
    return max(float(((bn.running_mean.double().cpu() - mean).abs() / var.sqrt()).max()), _rel(bn.running_var, var))


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["res", "swin"])
def test_head_train_codec_vs_fp64(variant):
    from oracle import restate
    T = 2
    head = _make_head(variant, T)
    head.train()
    head.codec_train_bn = True
    fp, gt, noise = _head_inputs(head)
    p0 = _codec_state(head)
    run0 = [(bn.running_mean.double().cpu().clone(), bn.running_var.double().cpu().clone()) for bn in head._codec_bns()]
    out = _run_head(head, fp, gt, noise)
    torch.cuda.synchronize()
    # pred against the fp64 train-mode decode of the fp64 loop at the cond the head produced
    sd = {"depth_head." + k: v.detach().cpu().double() for k, v in head.state_dict().items()}
    lat = restate.ddim_loop(sd, head.last_cond.double().cpu(), noise.double().cpu(), T, variant)
    depth_ref, _, _ = decode_train(p0, lat)
    _, _, dstats = decode_train(p0, head.last_latent.double().cpu())  # the statistics at the engine's own latent
    _, estats = encode_train(p0, gt.double().cpu())
    dpred = float((out["pred"].double().cpu() - depth_ref).abs().max() / depth_ref.abs().max())
    bns = head._codec_bns()
    errs = []
    for bn, r0, st in zip(bns, run0, estats + [dstats]):
        errs.append(_running_errors(bn, *_expected_running(r0, st)))
        assert int(bn.num_batches_tracked) == 1
    print(f"\n[head train codec {variant}] |dpred| {dpred:.1e} max|pred|; running stats rel err {errs}")
    assert dpred <= 5e-5  # measured 5.0e-6 (Swin)
    assert max(errs) <= 1e-6
    # an eval() forward now uses the updated statistics, through update_weights and never load_weights
    head.eval()
    head.capture_cond = True
    loads = []
    for e in head._engines.values():
        orig = e.load_weights
        e.load_weights = lambda t, _o=orig: (loads.append(1), _o(t))
    out_e = _run_head(head, fp, gt, noise)
    assert not loads
    sd = {"depth_head." + k: v.detach().cpu().double() for k, v in head.state_dict().items()}
    lat = restate.ddim_loop(sd, head.last_cond.double().cpu(), noise.double().cpu(), T, variant)
    ref_e = restate.decode(sd, lat)
    assert float((out_e["pred"].double().cpu() - ref_e).abs().max() / ref_e.abs().max()) <= 5e-5
    assert all(int(bn.num_batches_tracked) == 1 for bn in bns)


@pytest.mark.gpu
def test_vis_head_applies_T_plus_1_updates_in_reference_order():
    T = 3
    head = _make_head("resvis", T)
    head.train()
    head.codec_train_bn = True
    bn = head.depth_transform.conv_inv_transform[1]
    assert bn.momentum == 0.1  # an exponential average: the order of the updates shows in the result
    fp, gt, noise = _head_inputs(head)
    r0 = (bn.running_mean.double().cpu().clone(), bn.running_var.double().cpu().clone())
    out = _run_head(head, fp, gt, noise)
    eng = next(e for k, e in head._engines.items() if k.step_decode)
    rec = eng.codec_batch_stats().double().cpu()
    assert rec.shape == (T, 2, 16)

    def apply(order):
        m, v = r0
        for j in order:
            m, v = 0.9 * m + 0.1 * rec[j, 0], 0.9 * v + 0.1 * rec[j, 1]
        return m, v

    assert int(bn.num_batches_tracked) == T + 1
    err = _running_errors(bn, *apply([T - 1] + list(range(T))))
    wrong = _running_errors(bn, *apply(list(range(T)) + [T - 1]))  # steps 1 .. T, then the final map
    print(f"\n[vis order] reference order {err:.1e}, final map last {wrong:.1e}")
    assert err <= 1e-6 and wrong > 100 * max(err, 1e-7)
    # every step's map is the train-mode decode of that step's latent: the last one is `pred`
    assert torch.equal(out["pred_inter"][-1], out["pred"])


@pytest.mark.gpu
def test_flag_off_leaves_codec_in_eval():
    """Off (the default), a training forward runs the codec on its running statistics, as the parent commit did: `pred`
    and `gt_map_t` against the fp64 eval-mode restatement (oracle/restate.py), running statistics untouched."""
    from oracle import restate
    T = 2
    head = _make_head("res", T)
    head.train()
    fp, gt, noise = _head_inputs(head)
    r0 = [(b.running_mean.clone(), b.running_var.clone()) for b in head._codec_bns()]
    out = _run_head(head, fp, gt, noise)
    sd = {"depth_head." + k: v.detach().cpu().double() for k, v in head.state_dict().items()}
    ref = restate.decode(sd, restate.ddim_loop(sd, head.last_cond.double().cpu(), noise.double().cpu(), T, "res"))
    ref_t = restate.encode(sd, gt.double().cpu())
    dpred = float((out["pred"].double().cpu() - ref).abs().max() / ref.abs().max())
    dt = float((out["gt_map_t"].double().cpu() - ref_t).abs().max() / ref_t.abs().max())
    print(f"\n[flag off] |dpred| {dpred:.1e}, |dt| {dt:.1e}")
    assert dpred <= 5e-5 and dt <= 2e-5
    for b, (m, v) in zip(head._codec_bns(), r0):
        assert torch.equal(b.running_mean, m) and torch.equal(b.running_var, v) and int(b.num_batches_tracked) == 0


@pytest.mark.gpu
def test_sgd_with_train_codec_tracks_fp64():
    from oracle import restate
    variant, T = "res", 2
    head = _make_head(variant, T)
    head.train()
    head.grad_through_loop = True
    head.codec_train_bn = True
    fp, gt, noise = _head_inputs(head)
    keys, params = head._loop_params()
    lr, steps = 0.01, 4
    opt = torch.optim.SGD(params, lr=lr)
    ref = {k: v.detach().cpu().double().clone().requires_grad_("running" not in k and "num_batches" not in k)
           for k, v in head.state_dict().items() if k.startswith(("model.", "depth_transform."))}
    p0 = {k: ref[k].detach().clone() for k in keys}
    losses, ref_losses = [], []
    for _ in range(steps):
        opt.zero_grad()
        out = _run_head(head, fp, gt, noise)
        loss = F.l1_loss(out["pred"], gt) + F.mse_loss(out["pred"], gt)
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
        cond = head.last_cond.double().cpu()
        sd = {"depth_head." + k: v for k, v in ref.items()}
        lat = restate.ddim_loop(sd, cond, noise.double().cpu(), T, variant)
        pred, _, _ = decode_train({k: v for k, v in ref.items() if k.startswith("depth_transform.")}, lat)
        g64 = gt.double().cpu()
        rl = F.l1_loss(pred, g64) + F.mse_loss(pred, g64)
        gr = torch.autograd.grad(rl, [ref[k] for k in keys])
        with torch.no_grad():
            for k, gv in zip(keys, gr):
                ref[k] -= lr * gv
        ref_losses.append(float(rl))
    got = dict(zip(keys, params))
    moved = {k: float((ref[k].detach() - p0[k]).abs().max()) for k in keys}
    rel = {k: float((got[k].detach().double().cpu() - ref[k].detach()).abs().max()) / max(moved[k], 1e-30) for k in keys}
    # the ConvT bias has no effect through a training-mode BatchNorm: its gradient is zero up to rounding
    bias = DEC + "0.bias"
    assert float((got[bias].detach().double().cpu() - p0[bias]).abs().max()) <= 1e-6 * lr * steps
    rel.pop(bias)
    worst = max(rel, key=rel.get)
    print(f"\n[train codec sgd] losses {losses} (fp64 {ref_losses}); worst drift / movement: {worst} {rel[worst]:.2e}")
    assert losses[-1] < losses[0]
    assert abs(losses[0] - ref_losses[0]) <= 1e-4 * ref_losses[0]
    assert rel[worst] <= 1e-2
