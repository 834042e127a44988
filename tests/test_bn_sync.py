"""Synchronised BatchNorm across ranks (`bn_sync_group`, DenoiseEngine.set_bn_allgather, dd_set_bn_allgather): every
training-mode BatchNorm of the depth codec and the condition producers normalises with the statistics of all ranks'
batches together, as the reference's apex SyncBatchNorm (src/main.py:128) does.

World size 1 with a gatherer installed is bit-identical to no gatherer.  Two ranks run as two processes on one GPU over
gloo on 127.0.0.1 (NCCL cannot place two ranks on one GPU): the goldens' full batches split over the two ranks must come
out as the reference's full batch.  The NCCL branch is checked only with two GPUs."""
import copy
import datetime
import os
import socket
import traceback

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

from diffusiondepth_b200 import EngineError
from diffusiondepth_b200.engine import DECODER_PARAM_KEYS
from diffusiondepth_b200.model.head._ddim_head import bn_running_update

DEV = torch.device("cuda:0") if torch.cuda.is_available() else None
COND_BOUND, MEAN_BOUND, VAR_BOUND = 1e-4, 1e-4, 2e-4  # test_producer_train_bn.py's bounds
PRODUCER_CASES = ("swinl_70x106", "res18_64x128")     # g_producer_train.npz, B = 2 as 1 + 1
LOOP_CASES = ("swin_19x27", "res_19x27")               # g_codec_train.npz, B = 3 as 2 + 1


def _span(B, rank, world):
    """Rows [first, first + count) of rank's shard: the first ranks take the larger shards (3 as 2 + 1)."""
    base, extra = divmod(B, world)
    first = rank * base + min(rank, extra)
    return first, base + (rank < extra)


def _rows(t, rank, world):
    first, count = _span(t.shape[0], rank, world)
    return t[first:first + count].contiguous()


def _records_equal(a, b):
    return a.keys() == b.keys() and all(torch.equal(a[k][0], b[k][0]) and torch.equal(a[k][1], b[k][1]) for k in a)


@pytest.fixture
def group1():
    """A one-process gloo group: the gatherer's full path at world size 1."""
    dist.init_process_group("gloo", store=dist.HashStore(), rank=0, world_size=1)
    try:
        yield dist.group.WORLD
    finally:
        dist.destroy_process_group()


# ------------------------------------------------------------------------------------------------ world size 1
@pytest.mark.gpu
def test_world_size_one_producers_bit_identical(group1):
    from diffusiondepth_b200.model.backbone.mmbev_resnet import mmbev_res18
    from test_producer_train_bn import _feats, _head, _randomize, _swin_sizes
    # Swin HAHI at the 70 x 106 image's pyramid: neck + FPN from feature maps
    B, sizes = 2, _swin_sizes(18, 27)
    head = _head("DDIMDepthEstimate_Swin_ADDHAHI", 31).to(DEV)
    head.producer_train_bn = True
    head.train()
    fp = _feats(head, B, sizes, 38)
    eng = head._engine(B, (36, 54), sizes[0], DEV, feats=fp, producer_train=True)
    eng.set_producer_mode(True)
    runs = []
    for group in (None, group1, None):
        eng.set_bn_allgather(group)
        runs.append((eng.build_condition(fp, want_cond=True), eng.producer_batch_stats(), eng.graph_capture_count()))
    (c0, r0, n0), (c1, r1, n1), (c2, r2, n2) = runs
    assert torch.equal(c0, c1) and _records_equal(r0, r1) and len(r0) == 19
    assert n1 == n0, "the eager path captured a graph"
    assert torch.equal(c0, c2) and _records_equal(r0, r2) and n2 == n0  # back on the graph captured before
    # the native ResNet backbone + FPN
    head = _head("DDIMDepthEstimate_Res", 5).to(DEV)
    bb = _randomize(mmbev_res18(), 6).to(DEV)
    head.producer_train_bn = True
    head.train()
    bb.train()
    img = (70, 106)
    sizes = head.resnet_pyramid(img)
    rgb = torch.randn(B, 3, *img, generator=torch.Generator().manual_seed(9)).to(DEV)
    eng = head._engine(B, sizes[0], sizes[0], DEV, feats=(list(head.fpn_in_channels), sizes), image_hw=img,
                       backbone=bb, producer_train=True)
    eng.set_producer_mode(True)
    runs = []
    for group in (None, group1):
        eng.set_bn_allgather(group)
        eng.run_backbone(rgb)
        runs.append((eng.build_condition(None, want_cond=True), eng.producer_batch_stats()))
    eng.set_bn_allgather(None)
    assert torch.equal(runs[0][0], runs[1][0]) and _records_equal(runs[0][1], runs[1][1]) and len(runs[0][1]) == 23


@pytest.mark.gpu
def test_world_size_one_codec_bit_identical(group1):
    from test_codec_train import _make_head
    head = _make_head()
    B, hw = 2, (13, 21)
    g = torch.Generator().manual_seed(3)
    latent = torch.randn(B, 16, *hw, generator=g).to(DEV)
    d_depth = torch.randn(B, 1, 2 * hw[0], 2 * hw[1], generator=g).to(DEV)
    gt = (torch.rand(B, 1, 2 * hw[0], 2 * hw[1], generator=g) * 80 + 0.5).to(DEV)
    eng = head._engine(B, hw, hw, DEV, loop_backward=True)
    eng.set_codec_mode(True)

    def run():
        lat = eng.encode(gt)
        rec_enc = eng.codec_batch_stats().clone()
        depth, z = eng.decode(latent, want_logits=True)
        rec_dec = eng.codec_batch_stats().clone()
        d_lat, grads = eng.decode_backward(latent, d_depth)
        return [lat, rec_enc, depth, z, rec_dec, d_lat] + [grads[k] for k in DECODER_PARAM_KEYS]

    plain = run()
    eng.set_bn_allgather(group1)
    synced = run()
    eng.set_bn_allgather(None)
    assert all(torch.equal(a, b) for a, b in zip(plain, synced))


@pytest.mark.gpu
def test_world_size_one_head_running_stats_bit_identical(group1):
    from test_producer_train_bn import _feats, _forward, _head, _swin_sizes
    B, sizes = 2, _swin_sizes(18, 27)
    head = _head("DDIMDepthEstimate_Swin_ADDHAHI", 21).to(DEV)
    head.producer_train_bn = head.codec_train_bn = True
    head.train()
    synced = copy.deepcopy(head)
    synced.bn_sync_group = group1
    fp = _feats(head, B, sizes, 22)
    a, b = _forward(head, fp, B, sizes, 30), _forward(synced, fp, B, sizes, 30)
    assert torch.equal(a["pred"], b["pred"]) and torch.equal(a["gt_map_t"], b["gt_map_t"])
    n = 0
    for (name, x), y in zip(head.named_buffers(), synced.buffers()):
        assert torch.equal(x, y), name
        n += name.endswith("num_batches_tracked") and int(x) == 1
    assert n == 19 + 3  # every producer and codec BatchNorm moved once


@pytest.mark.gpu
def test_gather_failure_and_vis_heads(group1, monkeypatch):
    from test_codec_train import _make_head
    head = _make_head()
    B, hw = 2, (13, 21)
    latent = torch.randn(B, 16, *hw, generator=torch.Generator().manual_seed(4)).to(DEV)
    eng = head._engine(B, hw, hw, DEV)
    eng.set_codec_mode(True)
    eng.set_bn_allgather(group1)
    d0, _ = eng.decode(latent)

    def down(*args, **kwargs):
        raise RuntimeError("gather down")

    monkeypatch.setattr(dist, "all_gather", down)
    with pytest.raises(EngineError, match="all-gather callback failed"):
        eng.decode(latent)
    assert isinstance(eng.bn_allgather_error, RuntimeError)
    monkeypatch.undo()
    d1, _ = eng.decode(latent)  # the engine is still usable
    assert torch.equal(d0, d1)
    # *Vis heads: the head refuses, and so does the engine's step-decode loop in codec training mode
    vis = _make_head("resvis", T=2)
    vis.codec_train_bn = True
    vis.train()
    vis.bn_sync_group = group1
    gt = torch.rand(B, 1, 2 * hw[0], 2 * hw[1], device=DEV) + 0.5
    with pytest.raises(EngineError, match="Vis"):
        vis([torch.zeros(B, 64, *hw, device=DEV)], gt, gt > 0, gt_depth_map=gt)
    veng = vis._engine(B, hw, hw, DEV)
    assert veng.step_decode and veng.bn_allgather_group is group1
    veng.set_codec_mode(True)
    with pytest.raises(EngineError, match="DD_ERR_UNSUPPORTED"):
        veng.denoise_decode_steps(torch.rand(B, 256, *hw, device=DEV), latent)


# ------------------------------------------------------------------------------------------------ two ranks
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _producer_case(case, rank, world, group, dev):
    """One model forward of a g_producer_train case on this rank's images: condition map, records, running statistics."""
    import dd_helpers as helpers
    from oracle.make_producer_train import case_inputs
    family, sample = case_inputs(case)
    model = copy.deepcopy(helpers.build_mirror(family, 2, trained=True)).to(dev).train()
    if family.startswith("swin"):
        model.depth_backbone.eval()
    head = model.depth_head
    head.producer_train_bn = True
    head.bn_sync_group = group
    sample = {k: _rows(v, rank, world).to(dev) for k, v in sample.items()}
    assert head.can_run_backbone(model.depth_backbone, sample["rgb"])
    with torch.no_grad():
        model(sample)
    eng = next(e for e in head._engines.values() if e.producer_train)
    rec = {("depth_head." + k if not k.startswith("backbone.") else "depth_" + k): (m.cpu(), v.cpu())
           for k, (m, v) in eng.producer_batch_stats().items()}
    running = {k: (bn.running_mean.cpu(), bn.running_var.cpu(), int(bn.num_batches_tracked))
               for k in rec for bn in [model.get_submodule(k)]}
    return {"cond": head.last_cond.cpu(), "rec": rec, "running": running}


def _codec_head(dev, variant="res", sd=None, steps=2):
    from loop_grad_helpers import make_loop_head
    from oracle.make_codec_train import codec_state
    from oracle.make_loop_grads import loop_state
    sd = sd if sd is not None else dict(loop_state(variant), **{"depth_transform." + k: v for k, v in codec_state().items()})
    return make_loop_head(variant, sd, steps, dev)


def _codec_case(rank, world, group, dev):
    """The g_codec_train codec case (B = 2) on this rank's rows: inv_t, t, records and the decoder backward."""
    from oracle.make_codec_train import HW, codec_inputs
    latent, depth, d_depth, _ = codec_inputs()
    head = _codec_head(dev)
    head.bn_sync_group = group
    B = _span(latent.shape[0], rank, world)[1]
    eng = head._engine(B, HW, HW, dev, loop_backward=True)
    eng.set_codec_mode(True)
    inv, _ = eng.decode(_rows(latent, rank, world).to(dev))
    rec_dec = eng.codec_batch_stats().cpu()
    t = eng.encode(_rows(depth, rank, world).to(dev))
    rec_enc = eng.codec_batch_stats().cpu()
    d_lat, grads = eng.decode_backward(_rows(latent, rank, world).to(dev), _rows(d_depth, rank, world).to(dev))
    return {"inv_t": inv.cpu(), "t": t.cpu(), "rec_dec": rec_dec, "rec_enc": rec_enc, "d_latent": d_lat.cpu(),
            "grads": {k: v.cpu() for k, v in grads.items()}}


def _loop_case(case, rank, world, group, dev):
    """dd_denoise_backward of a g_codec_train loop case (T = 3, B = 3) with the codec in training mode, on this rank's
    rows; the forward's records first."""
    from oracle.make_loop_grads import STEPS, case_inputs
    variant, sd, cond, noise, d_depth, d_latent = case_inputs(case)
    head = _codec_head(dev, variant, sd, STEPS)
    head.bn_sync_group = group
    cond, noise, d_depth, d_latent = (_rows(t, rank, world).to(dev) for t in (cond, noise, d_depth, d_latent))
    eng = head._engine(cond.shape[0], noise.shape[-2:], cond.shape[-2:], dev, loop_backward=True)
    eng.set_codec_mode(True)
    eng.denoise_decode(cond, noise)
    rec = eng.codec_batch_stats().cpu()
    d_cond, _, grads, _ = eng.denoise_backward(cond, noise, d_depth, d_latent, want_noise=False)
    eng.poll_status()
    return {"rec": rec, "d_cond": d_cond.cpu(), "grads": {k: v.cpu() for k, v in grads.items()}}


def _plain(obj, conv):
    """obj with every tensor / array converted by conv: results cross the queue as numpy arrays, which do not depend
    on the sending process staying alive."""
    if isinstance(obj, dict):
        return {k: _plain(v, conv) for k, v in obj.items()}
    if isinstance(obj, (tuple, list)):
        return type(obj)(_plain(v, conv) for v in obj)
    return conv(obj) if isinstance(obj, (torch.Tensor, np.ndarray)) else obj


def _worker(rank, world, port, backend, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(seconds=300))
    try:
        group = dist.group.WORLD
        if backend == "nccl":
            out = {"codec": _codec_case(rank, world, group, dev)}
        else:
            out = {case: _producer_case(case, rank, world, group, dev) for case in PRODUCER_CASES}
            out["codec"] = _codec_case(rank, world, group, dev)
            out.update({case: _loop_case(case, rank, world, group, dev) for case in LOOP_CASES})
        q.put((rank, _plain(out, lambda t: t.numpy())))
    except BaseException:
        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


def _run_ranks(backend, world=2):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, backend, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        res = dict(q.get(timeout=1200) for _ in procs)
        for p in procs:
            p.join(120)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(30)
    for r in range(world):
        assert not isinstance(res[r], str), f"rank {r}:\n{res[r]}"
    return [_plain(res[r], torch.from_numpy) for r in range(world)]


@pytest.fixture(scope="module")
def two_ranks():
    return _run_ranks("gloo")


def _stat_margins(mean, var, m64, v64):
    sd = v64.clamp_min(1e-30).sqrt()
    return (((mean.double() - m64).abs() / sd).max().item(),
            ((var.double() - v64).abs() / v64.abs().clamp_min(1e-30)).max().item())


@pytest.mark.gpu
@pytest.mark.parametrize("case", PRODUCER_CASES)
def test_two_ranks_producers_match_reference_batch(two_ranks, case):
    from oracle.make_denoiser_grads import sample_index
    from oracle.make_producer_train import OUT
    golden = np.load(OUT, allow_pickle=False)
    r0, r1 = two_ranks[0][case], two_ranks[1][case]
    cond = torch.cat([r0["cond"], r1["cond"]]).reshape(-1)
    ref = torch.from_numpy(golden[case + "/cond/values"]).double()
    ec = ((cond[torch.from_numpy(sample_index(cond.numel()))].double() - ref).abs().max()
          / float(golden[case + "/cond/absmax"])).item()
    p = case + "/bn/"
    keys = sorted({k[len(p):-len("/mean")] for k in golden.files if k.startswith(p) and k.endswith("/mean")})
    assert set(r0["rec"]) == set(keys)
    em = ev = rm = rv = 0.0
    for k in keys:
        assert torch.equal(r0["rec"][k][0], r1["rec"][k][0]) and torch.equal(r0["rec"][k][1], r1["rec"][k][1]), k
        assert all(torch.equal(a, b) for a, b in zip(r0["running"][k][:2], r1["running"][k][:2])), k
        m64, v64 = (torch.from_numpy(golden[p + k + s]).double() for s in ("/mean", "/var"))
        e = _stat_margins(*r0["rec"][k], m64, v64)
        em, ev = max(em, e[0]), max(ev, e[1])
        mean, var, nbt = r0["running"][k]
        assert nbt == int(golden[p + k + "/num_batches_tracked"]) == 1, k
        rm64, rv64 = (torch.from_numpy(golden[p + k + s]).double() for s in ("/running_mean", "/running_var"))
        rm = max(rm, ((mean.double() - rm64).abs() / v64.sqrt()).max().item())
        rv = max(rv, ((var.double() - rv64).abs() / rv64).max().item())
    print(f"\n[{case} 1 + 1] cond {ec:.2e}, records mean {em:.2e} sigma, var {ev:.2e}; running mean {rm:.2e} sigma, "
          f"running var {rv:.2e} ({len(keys)} BatchNorms)")
    assert ec <= COND_BOUND
    assert em <= MEAN_BOUND and ev <= VAR_BOUND and rm <= MEAN_BOUND and rv <= VAR_BOUND


def _codec_bn(name):
    from oracle.make_codec_train import BN_KEYS, codec_state
    st = codec_state()
    bn = nn.BatchNorm2d(16)
    bn.running_mean.copy_(st[BN_KEYS[name] + ".running_mean"])
    bn.running_var.copy_(st[BN_KEYS[name] + ".running_var"])
    return bn


def _running_margins(bn, golden, prefix):
    assert int(bn.num_batches_tracked) == int(golden[prefix + "num_batches_tracked"]) == 1
    rm64, rv64 = (torch.from_numpy(golden[prefix + k]).double() for k in ("running_mean", "running_var"))
    return (((bn.running_mean.double() - rm64).abs() / rv64.sqrt()).max().item(),
            ((bn.running_var.double() - rv64).abs() / rv64).max().item())


def _check_codec(ranks, tag):
    from codec_train_helpers import DEC, decode_train_grads
    from oracle.make_codec_train import OUT, codec_inputs, codec_state
    golden = np.load(OUT, allow_pickle=False)
    r0, r1 = ranks[0]["codec"], ranks[1]["codec"]
    for k in ("rec_dec", "rec_enc"):
        assert torch.equal(r0[k], r1[k]), k
    e_inv = ((torch.cat([r0["inv_t"], r1["inv_t"]]).double() - torch.from_numpy(golden["codec/inv_t"])).abs().max()
             / float(np.abs(golden["codec/inv_t"]).max())).item()
    e_t = ((torch.cat([r0["t"], r1["t"]]).double() - torch.from_numpy(golden["codec/t"])).abs().max()
           / float(np.abs(golden["codec/t"]).max())).item()
    worst = (0.0, 0.0)
    for name, rec, prefix in (("dec", r0["rec_dec"][0], "codec/after_decode/dec/"),
                              ("enc1", r0["rec_enc"][0], "codec/after_encode/enc1/"),
                              ("enc2", r0["rec_enc"][1], "codec/after_encode/enc2/")):
        bn = _codec_bn(name)
        bn_running_update(bn, rec[0], rec[1])
        m = _running_margins(bn, golden, prefix)
        worst = (max(worst[0], m[0]), max(worst[1], m[1]))
    # the decoder backward: the ranks' parameter gradients sum to the full batch's, d_latent rows are the full batch's
    latent, _, d_depth, _ = codec_inputs()
    sd = {"depth_transform." + k: v for k, v in codec_state().items()}
    ref = decode_train_grads(sd, latent, d_depth)
    got = {k: r0["grads"][k].double() + r1["grads"][k].double() for k in DECODER_PARAM_KEYS if k != DEC + "0.bias"}
    got["d_latent"] = torch.cat([r0["d_latent"], r1["d_latent"]]).double()
    eg = {k: ((got[k] - ref[k]).abs().max() / ref[k].abs().max()).item() for k in got}
    print(f"\n[codec {tag} 1 + 1] inv_t {e_inv:.2e}, t {e_t:.2e}, running mean {worst[0]:.2e} sigma, running var "
          f"{worst[1]:.2e}, gradients worst {max(eg.values()):.2e}")
    assert e_inv <= 1e-4 and e_t <= 1e-4
    assert worst[0] <= MEAN_BOUND and worst[1] <= VAR_BOUND
    for k, e in eg.items():
        assert e <= 1e-4, (k, e)


@pytest.mark.gpu
def test_two_ranks_codec_matches_reference_batch(two_ranks):
    _check_codec(two_ranks, "gloo")


@pytest.mark.gpu
@pytest.mark.parametrize("case", LOOP_CASES)
def test_two_ranks_loop_gradients_match_reference_batch(two_ranks, case):
    """The ragged 2 + 1 split of the loop goldens (T = 3, B = 3, codec in training mode): d_cond rows and the summed
    parameter gradients against the reference's full batch, under test_codec_train.py's bound (2e-4 of max |g| plus the
    fp64 kink envelope)."""
    from codec_train_helpers import DEC, loop_train_grads
    from grad_helpers import golden_margins, tensor_margins
    from oracle.make_codec_train import OUT
    from oracle.make_loop_grads import STEPS, case_inputs
    golden = np.load(OUT, allow_pickle=False)
    r0, r1 = two_ranks[0][case], two_ranks[1][case]
    assert r0["rec"].shape == (1, 2, 16) and torch.equal(r0["rec"], r1["rec"])
    got = {k: r0["grads"][k].double() + r1["grads"][k].double() for k in r0["grads"]}
    got["d_cond"] = torch.cat([r0["d_cond"], r1["d_cond"]])
    variant, sd, cond, noise, d_depth, d_latent = case_inputs(case)
    ref = loop_train_grads(variant, sd, cond, noise, d_depth, d_latent, STEPS)
    env = tensor_margins(loop_train_grads(variant, sd, cond, noise, d_depth, d_latent, STEPS, band=5e-5), ref)
    mg = golden_margins(golden, case, got)
    mg.pop(DEC + "0.bias")  # no effect through a training-mode BatchNorm: rounding noise in the reference too
    worst = max(mg, key=lambda k: mg[k] - 2 * env[k])
    print(f"\n[loop {case} 2 + 1] vs reference worst {worst} {mg[worst]:.1e} (env {env[worst]:.1e})")
    for k in mg:
        assert mg[k] <= 2e-4 + 2 * env[k], (k, mg[k], env[k])


@pytest.mark.gpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="NCCL places one rank per GPU: needs 2 GPUs")
def test_two_ranks_nccl_codec():
    _check_codec(_run_ranks("nccl"), "nccl")
