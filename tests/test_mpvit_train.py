"""The MPViT backbone in training mode on the engine (`mpvit_native_train` with `producer_train_bn`): its 29 BatchNorms on
batch statistics (DD_PRODUCER_TRAIN) and stochastic depth on every MHCABlock (dd_set_drop_path), against fp64 torch of
the mirror MPViT in `.train()` from the same fp32 image, against the real reference's golden (g_mpvit_train.npz), and
against the torch backbone the head falls back to.  With the flag off, or the backbone in eval, nothing changes.

Each GPU test prints its worst margin (error over max |x64| of the features and condition map, mean error over sigma,
relative variance error)."""
import copy
import datetime
import os
import traceback

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

import dd_helpers as helpers
from diffusiondepth_b200 import _cabi
from diffusiondepth_b200.model._blocks import DropPath
from oracle import restate
from oracle.make_denoiser_grads import sample_index
from oracle.make_mpvit_train import CASES, FAMILY, OUT as GOLDEN, case_inputs
from test_bn_sync import _free_port, _plain, _records_equal, _rows, group1  # noqa: F401  (group1: fixture)
from test_producer_train_bn import COND_BOUND, MEAN_BOUND, VAR_BOUND, _StatHooks, _check_stats, _eval_order

DEV = torch.device("cuda:0") if torch.cuda.is_available() else None


def mpvit_bn_keys(paths=(2, 3, 3, 3)):
    """The MPViT's 29 (mpvit_small) BatchNorm keys in evaluation order: the stem, then per stage the patch embeddings,
    InvRes conv1 / norm / conv2 and the aggregate."""
    keys = ["backbone.stem.0.bn", "backbone.stem.1.bn"]
    for s, n in enumerate(paths):
        keys += [f"backbone.patch_embed_stages.{s}.patch_embeds.{p}.patch_conv.bn" for p in range(n)]
        keys += [f"backbone.mhca_stages.{s}.InvRes.{k}" for k in ("conv1.bn", "norm", "conv2.bn")]
        keys.append(f"backbone.mhca_stages.{s}.aggregate.bn")
    return keys


def _model(drop=None):
    """The trained-like mirror MPViT model in training mode: DropPath modules in eval (drop None) or at rate `drop`."""
    model = copy.deepcopy(helpers.build_mirror(FAMILY, 2, trained=True)).to(DEV).train()
    for m in model.modules():
        if isinstance(m, DropPath):
            if drop is None:
                m.eval()
            else:
                m.p = drop
    head = model.depth_head
    head.producer_train_bn = True
    head.mpvit_native_train = True
    return model


def _engine(head, bb, B, img):
    sizes = head.backbone_pyramid(img, bb)
    return head._engine(B, sizes[0], sizes[0], DEV, feats=(list(head.fpn_in_channels), sizes), image_hw=img,
                        backbone=bb, producer_train=True)


def _err(x, x64):
    return ((x.double() - x64).abs().max() / x64.abs().max()).item()


def _ref64(model, rgb, masks=None):
    """fp64 torch of the mirror's backbone + neck + FPN in `model`'s modes: features, condition map, BatchNorm stats.
    masks: per-sample scales [branch][B] the DropPath modules apply in call order instead of drawing."""
    ref = copy.deepcopy(model).double()
    if masks is not None:
        it = iter(masks)
        for m in ref.modules():
            if isinstance(m, DropPath):
                m.forward = lambda x: x * next(it).to(x).reshape(-1, *([1] * (x.dim() - 1)))
    hooks = [_StatHooks(ref.depth_backbone, "backbone."), _StatHooks(ref.depth_head)]
    with torch.no_grad():
        feats = list(ref.depth_backbone(rgb.double()))
        cond = ref.depth_head._condition(ref.depth_head._neck(feats))
    for h in hooks:
        h.close()
    return feats, cond, {**hooks[0].stats, **hooks[1].stats}


# ------------------------------------------------------------------------------------------------ CPU
def test_drop_path_layout_and_decision():
    model = copy.deepcopy(helpers.build_mirror(FAMILY, 2, trained=True)).train()
    head, bb = model.depth_head, model.depth_backbone
    masks, mods = head.mpvit_drop_paths(bb)
    # mpvit_small: linspace(0, 0.2, 13) over the layers (1, 3, 6, 3): only stage 0's layer has rate 0
    assert masks == (0, 0b111, 0b111111, 0b111) and len(mods) == 3 * (3 + 6 + 3)
    img = torch.zeros(1, 3, 64, 128)
    head.producer_train_bn = True
    assert not head.can_run_backbone(bb, img)  # CPU input
    assert head._producer_training(bb) == (True, False)  # mpvit_native_train off: the backbone stays in torch
    head.mpvit_native_train = True
    assert head._producer_training(bb) == (True, True)
    bb.mhca_stages[1].InvRes.norm.eval()
    assert head._producer_training(bb) == (True, False) and len(head._bn_modes(bb)) == 2
    bb.mhca_stages[2].mhca_blks[1].MHCA_layers[0].drop_path = nn.Identity()
    assert head.mpvit_drop_paths(bb) is None  # the paths of stage 2 differ


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("B,img", [(2, (70, 106)), (2, (64, 128)), (4, (352, 1216))])
def test_engine_matches_fp64_mirror(B, img):
    """Stage features, condition map and every record against fp64 torch of the mirror in `.train()` (DropPath off)."""
    model = _model()
    head, bb = model.depth_head, model.depth_backbone
    rgb = torch.randn(B, 3, *img, generator=torch.Generator().manual_seed(5)).to(DEV)
    assert head.can_run_backbone(bb, rgb)
    eng = _engine(head, bb, B, img)
    eng.set_producer_mode(True)
    eng.set_drop_path(None)
    feats = eng.run_backbone(rgb, want_feats=True)
    cond = eng.build_condition(None, want_cond=True)
    rec = eng.producer_batch_stats()
    eng.poll_status()
    keys = mpvit_bn_keys()
    assert [k for k, _, _ in eng.producer_bn_keys()] == keys + _eval_order(True)
    assert list(rec) == keys + _eval_order(True)
    feats64, cond64, stats = _ref64(model, rgb)
    ef = max(_err(f, f64) for f, f64 in zip(feats, feats64))
    ec = _err(cond, cond64)
    margins = []
    _check_stats(rec, stats, margins, "mpvit")
    print(f"mpvit B={B} {img}: feats {ef:.2e}, cond {ec:.2e}, mean {max(m[2] for m in margins):.2e} sigma, "
          f"var {max(m[3] for m in margins):.2e}")
    assert ef <= COND_BOUND and ec <= COND_BOUND


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_whole_model_matches_reference_golden(case):
    """A training-mode forward of the whole model with the MPViT on the engine, against the real reference's golden:
    stage features, condition map, every producer BatchNorm's running statistics after the call."""
    golden = np.load(GOLDEN, allow_pickle=False)
    model = _model()
    head = model.depth_head
    sample = {k: v.to(DEV) for k, v in case_inputs(case).items()}
    assert head.can_run_backbone(model.depth_backbone, sample["rgb"])
    with torch.no_grad():
        model(sample)
    eng = next(e for e in head._engines.values() if e.backbone is not None)
    feats = eng.run_backbone(sample["rgb"], want_feats=True)  # the same batch again: the same batch statistics
    ef = 0.0
    for i, f in enumerate(feats):
        flat = f.reshape(-1)
        ref = torch.from_numpy(golden[f"{case}/feats/{i}/values"]).double()
        ef = max(ef, ((flat[torch.from_numpy(sample_index(flat.numel())).to(DEV)].double().cpu() - ref).abs().max()
                      / ref.abs().max()).item())
    cond = head.last_cond.reshape(-1)
    ref = torch.from_numpy(golden[case + "/cond/values"]).double()
    ec = ((cond[torch.from_numpy(sample_index(cond.numel())).to(DEV)].double().cpu() - ref).abs().max()
          / float(golden[case + "/cond/absmax"])).item()
    p = case + "/bn/"
    keys = sorted({k[len(p):-len("/mean")] for k in golden.files if k.startswith(p) and k.endswith("/mean")})
    assert sum(k.startswith("depth_backbone.") for k in keys) == 29
    em = ev = 0.0
    for k in keys:
        bn = model.get_submodule(k)
        assert int(bn.num_batches_tracked) == int(golden[p + k + "/num_batches_tracked"]) == 1, k
        sd = torch.from_numpy(golden[p + k + "/var"]).double().sqrt()
        rm = torch.from_numpy(golden[p + k + "/running_mean"]).double()
        rv = torch.from_numpy(golden[p + k + "/running_var"]).double()
        em = max(em, ((bn.running_mean.double().cpu() - rm).abs() / sd).max().item())
        ev = max(ev, ((bn.running_var.double().cpu() - rv).abs() / rv).max().item())
    print(f"{case}: engine vs reference golden: feats {ef:.2e}, cond {ec:.2e}, running mean {em:.2e} sigma, "
          f"running var {ev:.2e} ({len(keys)} BatchNorms)")
    assert ef <= COND_BOUND and ec <= COND_BOUND and em <= MEAN_BOUND and ev <= VAR_BOUND


def _fallback_forward(model, sample, native, seed):
    """One training-mode model forward from CUDA seed `seed`, the MPViT natively or in torch: (condition map, CUDA
    generator state after the forward, the masks torch's DropPath modules drew, per call)."""
    head = model.depth_head
    head.mpvit_native_train = native
    drawn, hooks = [], []
    for m in model.depth_backbone.modules():
        if isinstance(m, DropPath):
            hooks.append(m.register_forward_hook(
                lambda mod, a, o: drawn.append((o.flatten(1).abs().amax(1) > 0).float().cpu())))
    torch.cuda.manual_seed(seed)
    try:
        with torch.no_grad():
            model(sample)
    finally:
        for h in hooks:
            h.remove()
    return head.last_cond.clone(), torch.cuda.get_rng_state(), drawn


@pytest.mark.gpu
def test_drop_path_matches_torch_fallback():
    """Every DropPath at rate 0.5 and the same CUDA seed for the engine and the torch backbone: the same masks, the same
    generator state after the forward (ddim_loss's draws included), features and condition map within the bounds."""
    B, img, seed = 2, (70, 106), 1234
    sample = {k: v.to(DEV) for k, v in restate.synthetic_sample(B, *img, 3).items()}
    sample["noise"] = restate.synthetic_noise(B, *img, 3).to(DEV)
    torch_model = _model(drop=0.5)
    native_model = copy.deepcopy(torch_model)
    start = copy.deepcopy(torch_model)
    assert native_model.depth_head.can_run_backbone(native_model.depth_backbone, sample["rgb"])
    cond_t, rng_t, drawn = _fallback_forward(torch_model, sample, False, seed)
    cond_n, rng_n, none = _fallback_forward(native_model, sample, True, seed)
    assert not none and len(drawn) == 2 * 36  # the engine ran the backbone; torch drew two masks per active block
    assert torch.equal(rng_t, rng_n)
    head, bb = start.depth_head, start.depth_backbone
    torch.cuda.manual_seed(seed)
    scales = head._mpvit_drop_scales(bb, B, DEV)
    masks = (scales.reshape(-1, B) > 0).float().cpu()
    assert torch.equal(masks, torch.stack(drawn))
    assert 0 < int(masks.sum()) < masks.numel()  # some samples dropped, some kept
    eng = _engine(head, bb, B, img)
    eng.set_producer_mode(True)
    eng.set_drop_path(scales)
    feats = eng.run_backbone(sample["rgb"], want_feats=True)
    cond = eng.build_condition(None, want_cond=True)
    eng.poll_status()
    feats64, cond64, _ = _ref64(start, sample["rgb"], masks=list(scales.reshape(-1, B).cpu().double()))
    ef = max(_err(f, f64) for f, f64 in zip(feats, feats64))
    ec, et = _err(cond, cond64), _err(cond_n, cond_t.double())
    print(f"drop path 0.5: {int(masks.sum())} of {masks.numel()} kept; feats {ef:.2e}, cond {ec:.2e}, "
          f"engine vs torch fallback cond {et:.2e}")
    assert ef <= COND_BOUND and ec <= COND_BOUND and et <= COND_BOUND
    with pytest.raises(_cabi.EngineError, match="DD_ERR_INVALID"):
        eng.set_drop_path(scales[:-1].contiguous())


@pytest.mark.gpu
def test_flag_off_and_eval_unchanged():
    """With mpvit_native_train off, or the backbone in eval, the engine computes what it did before: the same features,
    workspace size, graph count and launch count as an engine without the training-mode packs."""
    B, img = 2, (70, 106)
    model = _model()
    head, bb = model.depth_head, model.depth_backbone
    rgb = torch.randn(B, 3, *img, generator=torch.Generator().manual_seed(5)).to(DEV)
    runs = []
    for native_train, producer_train in ((False, False), (True, True)):
        h = copy.deepcopy(head)
        h.mpvit_native_train, h.producer_train_bn = native_train, producer_train
        eng = _engine(h, bb, B, img)
        if eng.producer_train:
            eng.set_producer_mode(False)
            eng.set_drop_path(None)
        eng.run_backbone(rgb)
        n_bb = eng.last_launch_count
        cond = eng.build_condition(None, want_cond=True)
        eng.poll_status()
        runs.append((cond, eng.lib.dd_workspace_bytes(eng._h), eng.graph_capture_count(), n_bb, eng.last_launch_count))
    assert torch.equal(runs[0][0], runs[1][0]) and runs[0][1:] == runs[1][1:]
    model.eval()  # the whole model in eval: torch-free, eval packs, no stochastic depth
    assert head.can_run_backbone(bb, rgb) and head._producer_training(bb) == (False, False)


@pytest.mark.gpu
def test_world_size_one_bit_identical(group1):  # noqa: F811
    B, img = 2, (70, 106)
    model = _model(drop=0.5)
    head, bb = model.depth_head, model.depth_backbone
    rgb = torch.randn(B, 3, *img, generator=torch.Generator().manual_seed(5)).to(DEV)
    eng = _engine(head, bb, B, img)
    eng.set_producer_mode(True)
    torch.cuda.manual_seed(3)
    eng.set_drop_path(head._mpvit_drop_scales(bb, B, DEV))
    runs = []
    for group in (None, group1):
        eng.set_bn_allgather(group)
        eng.run_backbone(rgb)
        runs.append((eng.build_condition(None, want_cond=True), eng.producer_batch_stats()))
    eng.set_bn_allgather(None)
    assert torch.equal(runs[0][0], runs[1][0]) and _records_equal(runs[0][1], runs[1][1])
    assert len(runs[0][1]) == 29 + 19  # the backbone's, then the neck's and the FPN's


def _rank_case(case, rank, world, group, dev):
    model = _model()
    model.to(dev)
    head = model.depth_head
    head.bn_sync_group = group
    sample = {k: _rows(v, rank, world).to(dev) for k, v in case_inputs(case).items()}
    assert head.can_run_backbone(model.depth_backbone, sample["rgb"])
    with torch.no_grad():
        model(sample)
    eng = next(e for e in head._engines.values() if e.backbone is not None)
    rec = {k: (m.cpu(), v.cpu()) for k, (m, v) in eng.producer_batch_stats().items()}
    running = {k: (bn.running_mean.cpu(), bn.running_var.cpu(), int(bn.num_batches_tracked))
               for k in rec if k.startswith("backbone.") for bn in [model.depth_backbone.get_submodule(k[9:])]}
    return {"rec": rec, "running": running}


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=300))
    try:
        q.put((rank, _plain({"mpvit_70x106": _rank_case("mpvit_70x106", rank, world, dist.group.WORLD, DEV)},
                            lambda t: t.numpy())))
    except BaseException:
        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
def test_two_ranks_match_reference_batch():
    """The golden's B = 2 split 1 + 1 over two gloo processes on one GPU: every rank records the full batch's
    statistics, bit-identical across ranks, and its running statistics follow the reference's."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
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
    for r in range(2):
        assert not isinstance(res[r], str), f"rank {r}:\n{res[r]}"
    r0, r1 = (_plain(res[r], torch.from_numpy)["mpvit_70x106"] for r in range(2))
    golden = np.load(GOLDEN, allow_pickle=False)
    p = "mpvit_70x106/bn/depth_"
    em = ev = rm = 0.0
    assert [k for k in r0["rec"] if k.startswith("backbone.")] == mpvit_bn_keys()
    for k in mpvit_bn_keys():
        assert torch.equal(r0["rec"][k][0], r1["rec"][k][0]) and torch.equal(r0["rec"][k][1], r1["rec"][k][1]), k
        assert all(torch.equal(a, b) for a, b in zip(r0["running"][k][:2], r1["running"][k][:2])), k
        m64, v64 = (torch.from_numpy(golden[p + k + s]).double() for s in ("/mean", "/var"))
        sd = v64.sqrt()
        em = max(em, ((r0["rec"][k][0].double() - m64).abs() / sd).max().item())
        ev = max(ev, ((r0["rec"][k][1].double() - v64).abs() / v64).max().item())
        rm64 = torch.from_numpy(golden[p + k + "/running_mean"]).double()
        rm = max(rm, ((r0["running"][k][0].double() - rm64).abs() / sd).max().item())
    print(f"\n[mpvit 1 + 1] records mean {em:.2e} sigma, var {ev:.2e}; running mean {rm:.2e} sigma")
    assert em <= MEAN_BOUND and ev <= VAR_BOUND and rm <= MEAN_BOUND


def test_drop_path_symbol_exported():
    import diffusiondepth_b200
    lib = diffusiondepth_b200.load_library()
    assert hasattr(lib, "dd_set_drop_path") and "dd_set_drop_path" in _cabi.SIGNATURES
