"""dd_encode_backward / DenoiseEngine.encode_backward: reverse mode of the depth encoder `depth_transform.t` in both
codec BatchNorm modes, checked against fp64 autograd of the restatement (itself pinned to the real reference by
test_encoder_backward_oracle.py), for determinism, argument checks and workspace size, at head level through
`grad_through_encoder` + `ddim_loss_gt`, and across two ranks with a synchronised BatchNorm."""
import ctypes as C
import datetime
import os
import traceback

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

from diffusiondepth_b200 import _cabi
from diffusiondepth_b200.engine import DENOISER_KEYS, DECODER_KEYS, ENCODER_PARAM_KEYS, GN_LAYERS, DenoiseEngine
from encoder_grad_helpers import ENC_PARAMS, encode, encode_grads, encoder_params
from grad_helpers import _MaskedReluTorch
from oracle import restate
from oracle.make_loop_grads import loop_state

DEV = torch.device("cuda:0") if torch.cuda.is_available() else None
TOL = 1e-5        # of max |g_ref| per gradient, engine vs fp64 restatement
KINK = 1e-5       # LeakyReLU inputs within KINK * max |v1| of zero may take the other slope in fp32 (kink envelope)
OP_TOL = 1e-4     # the operator backward's bound (test_denoiser_backward.py) for the head-level chain
SHAPES = ((1, 2, 3), (3, 37, 53), (2, 351, 1215), (4, 352, 1216))
SCALES = (1e-7, 1.0, 1e4)
# dd_workspace_bytes of test_loop_backward's geometry (Res, B = 3, 8 x 16, T = 2): DD_FLAG_BACKWARD as pinned there,
# DD_FLAG_LOOP_BACKWARD as the commit before the encoder backward gave it; the encoder backward adds no workspace
BACKWARD_WS_BYTES, LOOP_WS_BYTES = 8752128, 17583104


def _state():
    return loop_state("res")


def _engine_head(sd=None, steps=2):
    from loop_grad_helpers import make_loop_head
    return make_loop_head("res", sd if sd is not None else _state(), steps, DEV)


def _inputs(B, H, W, seed=11):
    g = torch.Generator().manual_seed(seed + B * 7 + H)
    depth = torch.rand(B, 1, H, W, generator=g) * 2 + 0.1
    d_latent = torch.randn(B, 16, (H + 1) // 2, (W + 1) // 2, generator=g)
    return depth, d_latent


def _margins(grads, ref):
    return {k: float((grads[k].double().cpu() - ref[k]).abs().max() / ref[k].abs().max()) for k in ref}


@pytest.mark.gpu
@pytest.mark.parametrize("train", (False, True), ids=("eval", "train"))
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_encode_backward_matches_fp64(shape, train):
    B, H, W = shape
    sd = _state()
    head = _engine_head(sd)
    hw = ((H + 1) // 2, (W + 1) // 2)
    eng = head._engine(B, hw, hw, DEV, backward=True)
    eng.set_codec_mode(train)
    depth, d_latent = _inputs(B, H, W)
    ref, vmax = encode_grads(sd, depth, d_latent, train)
    flip, _ = encode_grads(sd, depth, d_latent, train, band=KINK * vmax)
    f32, _ = encode_grads(sd, depth, d_latent, train, dtype=torch.float32)
    # the kink envelope plus four times the fp32 restatement's own spread (one sample of an fp32 rounding, which the
    # engine's independent rounding may exceed): with two values per channel (1 x 2 x 3 in training mode) the gradients
    # behind a BatchNorm cancel (sum du = 0), and any fp32 evaluation rounds at 1e-5 of max |g| there
    env = {k: e + 4 * r for (k, e), r in zip(_margins(flip, ref).items(), _margins(f32, ref).values())}
    dd = depth.to(DEV)
    for s in SCALES:
        grads = eng.encode_backward(dd, (d_latent * s).to(DEV))
        m = _margins({k: g / s for k, g in grads.items()}, ref)
        print(f"\n[{'x'.join(map(str, shape))} {'train' if train else 'eval'} x{s:g}] " +
              " ".join(f"{k[len('depth_transform.conv_transform.'):]}={v:.1e}(env {env[k]:.1e})" for k, v in m.items()))
        for k in ENC_PARAMS:
            assert torch.isfinite(grads[k]).all(), k
            assert m[k] <= TOL + env[k], (s, k, m[k], env[k])


@pytest.mark.gpu
def test_encode_backward_repeatable_and_records_untouched():
    B, H, W = 3, 37, 53
    head = _engine_head()
    hw = ((H + 1) // 2, (W + 1) // 2)
    eng = head._engine(B, hw, hw, DEV, backward=True)
    depth, d_latent = (t.to(DEV) for t in _inputs(B, H, W))
    for train in (False, True):
        eng.set_codec_mode(train)
        lat0 = eng.encode(depth)
        rec0 = eng.codec_batch_stats().clone()
        g1 = eng.encode_backward(depth, d_latent)
        rec1 = eng.codec_batch_stats().clone()
        g2 = eng.encode_backward(depth, d_latent)
        assert all(torch.equal(g1[k], g2[k]) for k in ENCODER_PARAM_KEYS)
        assert rec0.shape == rec1.shape == ((2, 2, 16) if train else (0, 2, 16))
        assert torch.equal(rec0, rec1)  # the backward records nothing
        # its batch fold is dd_encode's own: the forward after it is bit-identical, with the same records
        assert torch.equal(eng.encode(depth), lat0) and torch.equal(eng.codec_batch_stats(), rec0)
        assert set(eng.encode_backward(depth, d_latent, want_params=False)) == set()


def _call(eng, depth, d_latent, H, W):
    lib = _cabi.load_library()
    n = int(lib.dd_workspace_bytes(eng._h))
    wsb = eng._workspace()
    out = [torch.empty(16, 1, 3, 3, device=DEV) for _ in range(6)]
    return lib.dd_encode_backward(eng._h, C.c_void_p(depth.data_ptr() if depth is not None else 0), H, W,
                                  C.c_void_p(d_latent.data_ptr() if d_latent is not None else 0),
                                  (C.c_void_p * 6)(*[o.data_ptr() for o in out]), C.c_void_p(eng._aligned(wsb)), n,
                                  C.c_void_p(eng._stream()))


@pytest.mark.gpu
def test_encode_backward_invalid_arguments():
    sd = _state()
    head = _engine_head(sd)
    B, H, W = 2, 6, 10
    hw = (3, 5)
    depth, d_latent = (t.to(DEV) for t in _inputs(B, H, W))
    fwd = head._engine(B, hw, hw, DEV)
    bwd = head._engine(B, hw, hw, DEV, backward=True)
    INVALID = 1
    assert _call(fwd, depth, d_latent, H, W) == INVALID                    # neither backward flag
    with pytest.raises(_cabi.EngineError):
        fwd.encode_backward(depth, d_latent)
    assert _call(bwd, depth, d_latent, H, W) == 0
    torch.cuda.synchronize()
    assert _call(bwd, None, d_latent, H, W) == INVALID
    assert _call(bwd, depth, None, H, W) == INVALID
    assert _call(bwd, depth, d_latent, H + 2, W) == INVALID            # latent grid 4 x 5
    assert _call(bwd, depth, d_latent, H, W - 2) == INVALID
    fresh = DenoiseEngine("res", B, hw, hw, 2, DEV, backward=True)     # before dd_finalize_weights
    assert _call(fresh, depth, d_latent, H, W) == INVALID
    tensors = head._engine_tensors()
    plain = DenoiseEngine("res", B, hw, hw, 2, DEV, backward=True)     # without encoder weights
    plain.load_weights({k: tensors[k] for k in DENOISER_KEYS + DECODER_KEYS})
    assert _call(plain, depth, d_latent, H, W) == INVALID
    assert b"encoder" in _cabi.load_library().dd_last_error()
    one = head._engine(1, (1, 1), (1, 1), DEV, loop_backward=True)    # batch x latent = 1
    d1, l1 = (t.to(DEV) for t in _inputs(1, 1, 2))
    one.set_codec_mode(True)
    assert _call(one, d1, l1, 1, 2) == INVALID
    one.set_codec_mode(False)
    assert _call(one, d1, l1, 1, 2) == 0
    torch.cuda.synchronize()
    for e in (fresh, plain):
        e.close()


@pytest.mark.gpu
def test_workspace_unchanged():
    head = _engine_head()
    lib = _cabi.load_library()
    bwd = head._engine(3, (8, 16), (8, 16), DEV, backward=True)
    loop = head._engine(3, (8, 16), (8, 16), DEV, loop_backward=True)
    assert int(lib.dd_workspace_bytes(bwd._h)) == BACKWARD_WS_BYTES
    assert int(lib.dd_workspace_bytes(loop._h)) == LOOP_WS_BYTES


# ------------------------------------------------------------------------------------------------ head level
def _head_inputs(head, B=2, hw=(19, 27), seed=4):
    g = torch.Generator().manual_seed(seed)
    sizes = [hw, ((hw[0] + 1) // 2, (hw[1] + 1) // 2), ((hw[0] + 3) // 4, (hw[1] + 3) // 4),
             ((hw[0] + 7) // 8, (hw[1] + 7) // 8)]
    fp = [torch.randn(B, c, *s, generator=g).to(DEV) for c, s in zip(head.fpn_in_channels, sizes)]
    gt = (torch.rand(B, 1, 2 * hw[0], 2 * hw[1], generator=g) * 2 + 0.1).to(DEV)
    noise = torch.randn(B, 16, *hw, generator=g).to(DEV)
    return fp, gt, noise


def _make_head(variant, codec_train):
    from loop_grad_helpers import make_loop_head
    sd = loop_state(variant)
    head = make_loop_head(variant, sd, 2, DEV)
    head.train()
    head.codec_train_bn = codec_train
    return head, sd


def _loss_gt(head, out, cond, seed=33):
    torch.manual_seed(seed)
    head.zero_grad(set_to_none=True)
    loss = head.ddim_loss_gt(gt_depth=out["gt_map_t"], refine_module_inputs=(cond, None, None, None),
                             blur_depth_t=out["blur_depth_t"], weight=1.0)
    loss.backward()
    return loss


def _fp64_loss_gt(head, variant, sd, gt, cond, codec_train, eng_noisy, seed=33, band=0.0):
    """fp64 autograd of ddim_loss_gt over the restated encoder and denoiser, with the same noise and timesteps and the
    engine's own denoiser ReLU masks."""
    torch.manual_seed(seed)
    B = gt.shape[0]
    shape = (B, 16, (gt.shape[-2] + 1) // 2, (gt.shape[-1] + 1) // 2)
    noise = torch.randn(shape).double()
    t = torch.randint(0, head.scheduler.num_train_timesteps, (B,), device=DEV).long().cpu()
    z = head._grad_engine(B, shape[-2:], cond.shape[-2:], DEV).denoiser_relu_inputs(cond.detach(), eng_noisy, t.tolist())
    masks = [z[k] > 0 for k in GN_LAYERS]
    p = encoder_params(sd)
    pm = {k: v.detach().cpu().double().requires_grad_(True) for k, v in sd.items() if k.startswith("model.")}
    c = cond.detach().cpu().double().requires_grad_(True)
    gt_t, _ = encode(p, gt.detach().cpu().double(), codec_train, band)
    acp = head.scheduler.alphas_cumprod.detach().cpu().double()[t]
    noisy = acp.sqrt().view(-1, 1, 1, 1) * gt_t + (1 - acp).sqrt().view(-1, 1, 1, 1) * noise
    relu = _MaskedReluTorch([m.cpu() for m in masks])
    restate.torch = relu
    try:
        eps = restate.denoiser(pm, noisy, t, c, variant, prefix="model.")
    finally:
        restate.torch = torch
    F.mse_loss(eps, noise).backward()
    out = {k: p[k].grad for k in ENC_PARAMS}
    out.update({k: v.grad for k, v in pm.items()})
    out["d_cond"] = c.grad
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("variant,codec_train", (("res", False), ("swin", False), ("res", True)),
                         ids=("res", "swin", "res-codec-train"))
def test_head_ddim_loss_gt_trains_encoder(variant, codec_train):
    head, sd = _make_head(variant, codec_train)
    fp, gt, noise = _head_inputs(head)
    torch.manual_seed(21)
    out0 = head(fp, gt, gt > 0, gt_depth_map=gt, noise=noise)
    assert out0["gt_map_t"].grad_fn is None
    cond = head.last_cond.detach().requires_grad_(True)
    _loss_gt(head, out0, cond)
    off = {k: p.grad.clone() for k, p in head.named_parameters() if p.grad is not None}
    off_cond = cond.grad.clone()
    assert all(head.get_parameter(k).grad is None for k in ENC_PARAMS)
    bns = head._codec_bns()[:2]
    before = [(bn.running_mean.clone(), int(bn.num_batches_tracked)) for bn in bns]
    head.grad_through_encoder = True
    torch.manual_seed(21)
    out = head(fp, gt, gt > 0, gt_depth_map=gt, noise=noise)
    if codec_train:  # one running-statistic update per forward
        assert all(int(bn.num_batches_tracked) == n + 1 for bn, (_, n) in zip(bns, before))
    assert out["gt_map_t"].grad_fn is not None
    assert out["pred_init"] is out["gt_map_t"] is out["blur_depth_t"]
    assert torch.equal(out["gt_map_t"].detach(), out0["gt_map_t"])
    cond = head.last_cond.detach().requires_grad_(True)
    noisy_box = {}
    orig = head.denoiser

    def spy(noisy, t, c):
        noisy_box["noisy"] = noisy.detach().clone()
        return orig(noisy, t, c)
    head.denoiser = spy
    try:
        _loss_gt(head, out, cond)
    finally:
        del head.denoiser
    # with the flag off the same loss trains the denoiser and cond alone, bit for bit as with it on
    assert off.keys() == {k for k, p in head.named_parameters() if p.grad is not None} - set(ENC_PARAMS)
    for k, g in off.items():
        assert torch.equal(head.get_parameter(k).grad, g), k
    assert torch.equal(cond.grad, off_cond)
    # fp64 chain (in training mode the encoder's batch statistics do not read the running ones the forward updated)
    ref = _fp64_loss_gt(head, variant, sd, gt, cond, codec_train, noisy_box["noisy"])
    vmax = float(encode(encoder_params(sd), gt.cpu().double(), codec_train)[1].detach().abs().max())
    flip = _fp64_loss_gt(head, variant, sd, gt, cond, codec_train, noisy_box["noisy"], band=KINK * vmax)
    got = {k: head.get_parameter(k).grad for k in ref if k != "d_cond"}
    got["d_cond"] = cond.grad
    m, env = _margins(got, ref), _margins(flip, ref)
    worst = max(m, key=m.get)
    print(f"\n[{variant}{' codec-train' if codec_train else ''}] worst {worst} {m[worst]:.2e} (env {env[worst]:.1e}); "
          + " ".join(f"{k.rpartition('.')[0][-12:]}.{k.rpartition('.')[2]}={v:.1e}" for k, v in m.items() if k in ENC_PARAMS))
    for k in ref:
        assert m[k] <= OP_TOL + env[k], (k, m[k], env[k])


@pytest.mark.gpu
def test_head_encoder_repacks_in_place_after_step():
    head, _ = _make_head("res", False)
    head.grad_through_encoder = True
    fp, gt, noise = _head_inputs(head)
    opt = torch.optim.SGD([head.get_parameter(k) for k in ENC_PARAMS], lr=1e-2)
    for _ in range(2):  # the first backward grows the shared workspace pool: the forward engine then captures again once
        torch.manual_seed(21)
        out = head(fp, gt, gt > 0, gt_depth_map=gt, noise=noise)
        _loss_gt(head, out, head.last_cond)
    captures = {k: e.graph_capture_count() for k, e in head._engines.items()}
    opt.step()
    torch.manual_seed(21)
    out2 = head(fp, gt, gt > 0, gt_depth_map=gt, noise=noise)
    with torch.no_grad():
        from encoder_grad_helpers import encode as enc
        p = {k: v.detach().cpu().double() for k, v in head.state_dict().items() if k.startswith("depth_transform.conv_transform.")}
        want = enc(p, gt.cpu().double(), False)[0]
    assert not torch.equal(out2["gt_map_t"], out["gt_map_t"])
    assert float((out2["gt_map_t"].detach().cpu().double() - want).abs().max()) < 1e-5
    assert {k: e.graph_capture_count() for k, e in head._engines.items() if k in captures} == captures


# ------------------------------------------------------------------------------------------------ two ranks
def _rank_case(rank, world, group, dev):
    from test_bn_sync import _rows
    B, H, W = 2, 37, 53
    head = _engine_head()
    head.bn_sync_group = group
    hw = ((H + 1) // 2, (W + 1) // 2)
    depth, d_latent = _inputs(B, H, W)
    eng = head._engine(B // world, hw, hw, dev, backward=True)
    eng.set_codec_mode(True)
    dd, dl = _rows(depth, rank, world).to(dev), _rows(d_latent, rank, world).to(dev)
    eng.encode(dd)
    grads = eng.encode_backward(dd, dl)
    return {k: v.cpu().numpy() for k, v in grads.items()}


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=300))
    try:
        q.put((rank, _rank_case(rank, world, dist.group.WORLD, dev)))
    except BaseException:
        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
def test_two_ranks_encoder_gradients_match_full_batch():
    from test_bn_sync import _free_port
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        res = dict(q.get(timeout=600) for _ in procs)
        for p in procs:
            p.join(120)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(30)
    for r in range(2):
        assert not isinstance(res[r], str), f"rank {r}:\n{res[r]}"
    depth, d_latent = _inputs(2, 37, 53)
    ref, _ = encode_grads(_state(), depth, d_latent, True)
    total = {k: torch.from_numpy(res[0][k]).double() + torch.from_numpy(res[1][k]).double() for k in ref}
    m = _margins(total, ref)
    print("\n[two ranks] " + " ".join(f"{k[len('depth_transform.conv_transform.'):]}={v:.1e}" for k, v in m.items()))
    for k in ref:
        assert m[k] <= 1e-6, (k, m[k])
