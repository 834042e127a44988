"""Training-mode BatchNorm of the condition producers (`producer_train_bn`, dd_set_producer_mode): the HAHI neck, the FPN
and the native ResNet backbone on batch statistics, against fp64 torch of the mirror modules in `.train()` from the
same fp32 inputs; running-statistic updates, records, the re-pack rule, and no change with the mode off.

Each GPU test prints its worst margin (cond error over max |cond64|, mean error over sigma, relative variance error)."""
import copy
import math

import numpy as np
import pytest
import torch
import torch.nn as nn

from diffusiondepth_b200.model.backbone.mmbev_resnet import mmbev_res18
from diffusiondepth_b200.model.head import _ddim_head
from diffusiondepth_b200.model.head._ddim_head import is_producer_running_stat, repack_plan
from diffusiondepth_b200.model.registry import HEADS
from oracle import restate
from oracle.make_denoiser_grads import sample_index
from oracle.make_producer_train import OUT as GOLDEN
from oracle.make_producer_train import case_inputs as golden_case_inputs

import dd_helpers as helpers

DEV = torch.device("cuda:0") if torch.cuda.is_available() else None
COND_BOUND = 1e-4    # of max |cond64|
MEAN_BOUND = 1e-4    # of the batch sigma
VAR_BOUND = 2e-4     # relative


def _bns(module):
    return [m for m in module.modules() if isinstance(m, nn.BatchNorm2d)]


def _randomize(module, seed):
    """Non-trivial BatchNorm affines and running statistics (fresh BatchNorms are the identity at init)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for bn in _bns(module):
            C = bn.num_features
            bn.weight.copy_(torch.rand(C, generator=g) + 0.5)
            bn.bias.copy_(torch.rand(C, generator=g) * 0.6 - 0.3)
            bn.running_mean.copy_(torch.rand(C, generator=g) * 0.4 - 0.2)
            bn.running_var.copy_(torch.rand(C, generator=g) + 0.5)
    return module


def _head(kind, seed=11):
    torch.manual_seed(seed)
    head = HEADS.build(dict(type=kind, in_channels=[64, 128, 256, 512], inference_steps=2, num_train_timesteps=1000,
                            depth_feature_dim=16, loss_cfgs=[], init_cfg=None))
    return _randomize(head, seed + 1)


def _swin_sizes(h0, w0):
    sizes = [(h0, w0)]
    for _ in range(3):
        h, w = sizes[-1]
        sizes.append(((h + 1) // 2, (w + 1) // 2))
    return sizes


def _feats(head, B, sizes, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(B, c, *s, generator=g).to(DEV) for c, s in zip(head.fpn_in_channels, sizes)]


class _StatHooks:
    """Batch mean / unbiased variance of every BatchNorm's input in a torch forward, by module name."""

    def __init__(self, module, prefix=""):
        self.stats, self.handles = {}, []
        for name, m in module.named_modules():
            if isinstance(m, nn.BatchNorm2d):
                self.handles.append(m.register_forward_pre_hook(self._hook(prefix + name)))

    def _hook(self, name):
        def f(_, inp):
            x = inp[0]
            self.stats[name] = (x.mean((0, 2, 3)), x.var((0, 2, 3), unbiased=True))
        return f

    def close(self):
        for h in self.handles:
            h.remove()


def _ref_cond(head, fp):
    ref = copy.deepcopy(head).double().train()
    hooks = _StatHooks(ref)
    with torch.no_grad():
        cond = ref._condition(ref._neck([f.double() for f in fp]))
    hooks.close()
    return ref, cond, hooks.stats


def _check_stats(rec, ref_stats, margins, tag):
    assert rec, "no records"
    for key, (mean, var) in rec.items():
        m64, v64 = ref_stats[key]
        sd = v64.clamp_min(1e-30).sqrt()
        em = ((mean.double() - m64).abs() / sd).max().item()
        ev = ((var.double() - v64).abs() / v64.abs().clamp_min(1e-30)).max().item()
        margins.append((tag, key, em, ev))
        assert em <= MEAN_BOUND, (tag, key, em)
        assert ev <= VAR_BOUND, (tag, key, ev)


def _cond_err(cond, cond64):
    return ((cond.double() - cond64).abs().max() / cond64.abs().max()).item()


def _eval_order(neck, res_depths=(), nlev=4):
    """Producer BatchNorm keys in evaluation order: the ResNet block by block, then the neck level by level (lateral,
    proj, fusion), then the FPN top-down (lateral, conv_up)."""
    keys = [f"backbone.layers.{s}.{b}.bn{j}" for s, d in enumerate(res_depths) for b in range(d) for j in (1, 2)]
    for i in range(nlev if neck else 0):
        t, j = ("conv", 0) if i == 0 else ("trans", i - 1)
        keys += [f"hahineck.lateral_convs.{i}.bn", f"hahineck.{t}_proj.{j}.bn", f"hahineck.{t}_fusion.{j}.bn"]
    for i in reversed(range(nlev)):
        keys += [f"conv_lateral.{i}.1"] + ([f"conv_up.{i - 1}.1"] if i else [])
    return keys


def _bn_channels(module, prefix=""):
    return {prefix + n: m.num_features for n, m in module.named_modules() if isinstance(m, nn.BatchNorm2d)}


def _check_record_order(eng, keys, channels):
    """The records are those of `keys`, in that order, each 2 x C floats, back to back from offset 0."""
    info = eng.producer_bn_keys()
    assert [k for k, _, _ in info] == keys
    off = 0
    for k, c, o in info:
        assert (c, o) == (channels[k], off), k
        off += 2 * c


# ------------------------------------------------------------------------------------------------ CPU
def test_repack_plan_defers_producer_running_stats():
    keys = ["model.pred.0.weight", "hahineck.lateral_convs.0.bn.running_mean", "conv_up.0.1.num_batches_tracked",
            "backbone.layers.0.0.bn1.running_var", "conv_lateral.0.1.weight"]
    old = [(1, 0)] * 5
    new = [(1, 1), (1, 1), (1, 1), (1, 1), (1, 0)]
    assert repack_plan(keys, old, keys, new) is None  # unchanged behaviour without the argument
    assert repack_plan(keys, old, keys, new, deferred=is_producer_running_stat) == ["model.pred.0.weight"]
    new[4] = (1, 1)  # a producer weight: still a full pack
    assert repack_plan(keys, old, keys, new, deferred=is_producer_running_stat) is None
    assert not is_producer_running_stat("depth_transform.conv_inv_transform.1.running_mean")


def test_producer_training_decision():
    head = HEADS.build(dict(type="DDIMDepthEstimate_Swin_ADDHAHI", in_channels=[64, 128, 256, 512], inference_steps=2,
                            num_train_timesteps=1000, depth_feature_dim=16, loss_cfgs=[], init_cfg=None)).train()
    assert head._producer_training() == (False, False)  # flag off
    head.producer_train_bn = True
    assert head._producer_training() == (True, False)
    bb = mmbev_res18().train()
    assert head._producer_training(bb) == (True, True)
    bb.eval()
    assert head._producer_training(bb) == (True, False)
    head.eval()
    assert head._producer_training() == (False, False)
    head.train()
    head.hahineck.lateral_convs[0].bn.eps = 1e-3
    with pytest.raises(Exception, match="eps"):
        head._producer_training()


# ------------------------------------------------------------------------------------------------ GPU
def _cond_case(kind, B, sizes, seed, margins):
    head = _head(kind, seed).to(DEV)
    head.producer_train_bn = True
    head.train()
    fp = _feats(head, B, sizes, seed + 7)
    h0, w0 = sizes[0]
    eng = head._engine(B, (2 * h0, 2 * w0), (h0, w0), DEV, feats=fp, producer_train=True)
    eng.set_producer_mode(True)
    cond = eng.build_condition(fp, want_cond=True)
    rec = eng.producer_batch_stats()
    eng.poll_status()
    ref, cond64, stats = _ref_cond(head, fp)
    err = _cond_err(cond, cond64)
    margins.append((kind, sizes[0], "cond", err))
    assert err <= COND_BOUND, err
    assert set(rec) == set(stats)
    _check_record_order(eng, _eval_order("HAHI" in kind), _bn_channels(head))
    _check_stats(rec, stats, margins, kind)
    # determinism: a second call gives the same bits
    cond2 = eng.build_condition(fp, want_cond=True)
    rec2 = eng.producer_batch_stats()
    assert torch.equal(cond, cond2)
    assert all(torch.equal(rec[k][0], rec2[k][0]) and torch.equal(rec[k][1], rec2[k][1]) for k in rec)
    return head, eng, fp


@pytest.mark.gpu
@pytest.mark.parametrize("kind,B,h0w0", [
    ("DDIMDepthEstimate_Swin_ADDHAHI", 2, (18, 27)),   # the 70 x 106 image: the FPN resamples
    ("DDIMDepthEstimate_Swin_ADDHAHI", 3, (16, 32)),   # exact 2x pyramid
    ("DDIMDepthEstimate_Swin_ADDHAHI", 4, (88, 304)),  # C3 geometry
    ("DDIMDepthEstimate_Swin_ADD", 2, (18, 27)),       # FPN only
])
def test_condition_train_mode(kind, B, h0w0):
    margins = []
    _cond_case(kind, B, _swin_sizes(*h0w0), 31, margins)
    stats = [m for m in margins if m[2] != "cond"]
    print(kind, B, h0w0, "cond", margins[0][3], "mean/sigma", max(m[2] for m in stats), "var rel", max(m[3] for m in stats))


@pytest.mark.gpu
@pytest.mark.parametrize("img", [(228, 304), (70, 106)])
def test_resnet_backbone_train_mode(img):
    B = 2
    head = _head("DDIMDepthEstimate_Res", 5).to(DEV)
    bb = _randomize(mmbev_res18(), 6).to(DEV)
    head.producer_train_bn = True
    head.train()
    bb.train()
    sizes = head.resnet_pyramid(img)
    g = torch.Generator().manual_seed(9)
    rgb = torch.randn(B, 3, *img, generator=g).to(DEV)
    eng = head._engine(B, sizes[0], sizes[0], DEV, feats=(list(head.fpn_in_channels), sizes), image_hw=img,
                       backbone=bb, producer_train=True)
    eng.set_producer_mode(True)
    eng.run_backbone(rgb)
    cond = eng.build_condition(None, want_cond=True)
    rec = eng.producer_batch_stats()
    eng.poll_status()
    ref = copy.deepcopy(head).double().train()
    bb64 = copy.deepcopy(bb).double().train()
    hooks = [_StatHooks(ref), _StatHooks(bb64, "backbone.")]
    with torch.no_grad():
        cond64 = ref._condition(ref._neck(list(bb64(rgb.double()))))
    stats = {**hooks[0].stats, **hooks[1].stats}
    err = _cond_err(cond, cond64)
    print("res", img, "cond", err)
    assert err <= COND_BOUND, err
    assert set(rec) == set(stats) and len(rec) == 16 + 7
    _check_record_order(eng, _eval_order(False, res_depths=(2, 2, 2, 2)),
                        {**_bn_channels(head), **_bn_channels(bb, "backbone.")})
    margins = []
    _check_stats(rec, stats, margins, "res")
    print("res", img, "stats", max(m[2] for m in margins), max(m[3] for m in margins))


@pytest.mark.gpu
def test_flag_off_and_eval_mode_unchanged():
    kind, B, sizes = "DDIMDepthEstimate_Swin_ADDHAHI", 2, _swin_sizes(18, 27)
    head = _head(kind, 3).to(DEV).eval()
    fp = _feats(head, B, sizes, 4)
    plain = head._engine(B, (36, 54), (18, 27), DEV, feats=fp)
    head.producer_train_bn = True
    flagged = head._engine(B, (36, 54), (18, 27), DEV, feats=fp, producer_train=False)
    assert flagged is not plain and flagged.producer_train and not plain.producer_train
    assert plain.lib.dd_workspace_bytes(plain._h) == flagged.lib.dd_workspace_bytes(flagged._h)
    a = plain.build_condition(fp, want_cond=True)
    b = flagged.build_condition(fp, want_cond=True)
    assert torch.equal(a, b)
    assert plain.graph_capture_count() == flagged.graph_capture_count() == 1
    with pytest.raises(Exception, match="DD_FLAG_PRODUCER_TRAIN"):
        plain.set_producer_mode(True)
    # a train-mode call captures its own graph and leaves the eval graph in place
    flagged.set_producer_mode(True)
    flagged.build_condition(fp)
    flagged.set_producer_mode(False)
    c = flagged.build_condition(fp, want_cond=True)
    assert torch.equal(a, c) and flagged.graph_capture_count() == 2
    assert flagged.producer_batch_stats() == {}  # eval call: no current record


@pytest.mark.gpu
def test_constant_channel_outputs_beta():
    """A pre-BN channel that is constant (zero conv weights) has batch variance 0: no NaN, and the layer outputs beta.
    At level 0 both the FPN lateral and the ConvT above it are made constant in channel 5, so the condition map's
    channel 5 is relu(beta_lateral) + adaptive_avg_pool(relu(beta_up)) = 0.25 + 0.125 exactly."""
    kind, B, sizes = "DDIMDepthEstimate_Swin_ADD", 2, _swin_sizes(18, 27)
    head = _head(kind, 8).to(DEV)
    with torch.no_grad():
        head.conv_lateral[0][0].weight[5].zero_()
        head.conv_lateral[0][1].bias[5] = 0.25
        head.conv_up[0][0].weight[:, 5].zero_()  # ConvTranspose2d weight [cin][cout][2][2]
        head.conv_up[0][1].bias[5] = 0.125
    head.producer_train_bn = True
    head.train()
    fp = _feats(head, B, sizes, 2)
    eng = head._engine(B, (36, 54), sizes[0], DEV, feats=fp, producer_train=True)
    eng.set_producer_mode(True)
    cond = eng.build_condition(fp, want_cond=True)
    rec = eng.producer_batch_stats()
    eng.poll_status()
    assert torch.isfinite(cond).all()
    for key in ("conv_lateral.0.1", "conv_up.0.1"):
        m, v = rec[key]
        assert m[5].item() == 0.0 and v[5].item() == 0.0, key
    assert torch.equal(cond[:, 5], torch.full_like(cond[:, 5], 0.375))
    _, cond64, _ = _ref_cond(head, fp)
    assert _cond_err(cond, cond64) <= COND_BOUND


@pytest.mark.gpu
def test_large_mean_costs_only_the_record_rounding():
    """A pre-BN channel with |mean| ~ 1e3 sigma: the neck's 1x1 lateral conv at level 0 with row 7 = 2^-7 everywhere on an
    input of 1000 + 14 N(0, 1) rounded to multiples of 1/8, so the channel is 1500 + 1.5 N(0, 1).  Weights, inputs, their
    fp16 split and every partial sum are exact, so the conv's output is exact and the recorded mean may differ from the
    fp64 batch mean by no more than the fp32 record's own rounding (one ulp); the variance stays within the usual
    bound."""
    kind, B, sizes = "DDIMDepthEstimate_Swin_ADDHAHI", 2, _swin_sizes(16, 32)
    head = _head(kind, 8).to(DEV)
    with torch.no_grad():
        head.hahineck.lateral_convs[0].conv.weight[7].fill_(2.0 ** -7)
    head.producer_train_bn = True
    head.train()
    fp = _feats(head, B, sizes, 2)
    fp[0] = (torch.round(fp[0] * 14.0 * 8.0) / 8.0 + 1000.0).contiguous()
    eng = head._engine(B, (32, 64), sizes[0], DEV, feats=fp, producer_train=True)
    eng.set_producer_mode(True)
    cond = eng.build_condition(fp, want_cond=True)
    rec = eng.producer_batch_stats()
    eng.poll_status()
    _, cond64, stats = _ref_cond(head, fp)
    m64, v64 = (t[7].item() for t in stats["hahineck.lateral_convs.0.bn"])
    mean, var = (t[7].item() for t in rec["hahineck.lateral_convs.0.bn"])
    ratio = abs(m64) / v64 ** 0.5
    ulp = 2.0 ** (math.floor(math.log2(abs(m64))) - 23)
    print(f"large mean: |mean| / sigma {ratio:.0f}, |d mean| {abs(mean - m64):.2e} (fp32 ulp {ulp:.2e}), "
          f"var rel {abs(var - v64) / v64:.2e}")
    assert ratio >= 500
    assert abs(mean - m64) <= ulp
    assert abs(var - v64) / v64 <= VAR_BOUND
    # that layer's other channels carry the 1e3 offset through inexact random weights, so their means inherit the
    # conv's own rounding (up to ~1.5e-4 sigma measured); every later layer sees normalised inputs again
    _check_stats({k: v for k, v in rec.items() if k != "hahineck.lateral_convs.0.bn"}, stats, [], kind)
    assert _cond_err(cond, cond64) <= COND_BOUND


@pytest.mark.gpu
def test_mpvit_torch_backbone_native_neck_and_fpn():
    """MPViT's BatchNorms are not on the engine: with producer_train_bn and the backbone in training mode the model runs
    it in torch (which moves its BatchNorm buffers), while the neck and FPN run natively in training mode and their
    running statistics follow fp64 torch from the same features."""
    family, B, H, W = "mpvit_s", 2, 70, 106
    model = copy.deepcopy(helpers.build_mirror(family, 2, trained=True)).to(DEV).train()
    head, bb = model.depth_head, model.depth_backbone
    head.producer_train_bn = True
    sample = {k: v.to(DEV) for k, v in restate.synthetic_sample(B, H, W, 3).items()}
    sample["noise"] = restate.synthetic_noise(B, H, W, 3).to(DEV)
    assert not head.can_run_backbone(bb, sample["rgb"])
    head.producer_train_bn = False
    assert head.can_run_backbone(bb, sample["rgb"])  # only the training-mode MPViT falls back
    head.producer_train_bn = True
    start = copy.deepcopy(head)
    feats = {}
    h = bb.register_forward_hook(lambda m, a, o: feats.__setitem__("fp", [f.detach().clone() for f in o]))
    try:
        with torch.no_grad():
            model(sample)
    finally:
        h.remove()
    bb_bns = [m for m in bb.modules() if isinstance(m, nn.BatchNorm2d)]
    assert bb_bns and all(int(m.num_batches_tracked) == 1 for m in bb_bns)  # torch ran the backbone in train mode
    ref = start.double().train()
    with torch.no_grad():
        cond64 = ref._condition(ref._neck([f.double() for f in feats["fp"]]))
    assert _cond_err(head.last_cond, cond64) <= COND_BOUND
    worst, n = 0.0, 0
    for (name, bn), bn64 in zip(((n_, m) for n_, m in head.named_modules() if isinstance(m, nn.BatchNorm2d)
                                 and n_.startswith(("hahineck", "conv_lateral", "conv_up"))),
                                (m for n_, m in ref.named_modules() if isinstance(m, nn.BatchNorm2d)
                                 and n_.startswith(("hahineck", "conv_lateral", "conv_up")))):
        assert int(bn.num_batches_tracked) == int(bn64.num_batches_tracked) == 1, name
        em = ((bn.running_mean.double() - bn64.running_mean).abs() / bn64.running_var.sqrt()).max().item()
        ev = ((bn.running_var.double() - bn64.running_var).abs() / bn64.running_var).max().item()
        worst, n = max(worst, em, ev), n + 1
        assert em <= MEAN_BOUND and ev <= VAR_BOUND, (name, em, ev)
    print(f"mpvit: cond {_cond_err(head.last_cond, cond64):.2e}, {n} neck / FPN BatchNorms, worst {worst:.2e}")
    assert n == 19


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["swinl_70x106", "res18_64x128"])
def test_engine_matches_reference_golden(case):
    """A training-mode forward of the whole model on the engine (native backbone; Swin-L in eval, DropPath off) against
    the real reference's golden: the condition map and every producer BatchNorm's running statistics after one call."""
    golden = np.load(GOLDEN, allow_pickle=False)
    family, sample = golden_case_inputs(case)
    model = copy.deepcopy(helpers.build_mirror(family, 2, trained=True)).to(DEV).train()
    if family.startswith("swin"):
        model.depth_backbone.eval()
    head = model.depth_head
    head.producer_train_bn = True
    sample = {k: v.to(DEV) for k, v in sample.items()}
    assert head.can_run_backbone(model.depth_backbone, sample["rgb"])
    with torch.no_grad():
        model(sample)
    cond = head.last_cond.reshape(-1)
    ref = torch.from_numpy(golden[case + "/cond/values"]).double()
    ec = ((cond[torch.from_numpy(sample_index(cond.numel())).to(DEV)].double().cpu() - ref).abs().max()
          / float(golden[case + "/cond/absmax"])).item()
    p = case + "/bn/"
    keys = sorted({k[len(p):-len("/mean")] for k in golden.files if k.startswith(p) and k.endswith("/mean")})
    em = ev = 0.0
    for k in keys:
        bn = model.get_submodule(k)
        assert int(bn.num_batches_tracked) == int(golden[p + k + "/num_batches_tracked"]) == 1, k
        sd = torch.from_numpy(golden[p + k + "/var"]).double().sqrt()
        rm = torch.from_numpy(golden[p + k + "/running_mean"]).double()
        rv = torch.from_numpy(golden[p + k + "/running_var"]).double()
        em = max(em, ((bn.running_mean.double().cpu() - rm).abs() / sd).max().item())
        ev = max(ev, ((bn.running_var.double().cpu() - rv).abs() / rv).max().item())
    print(f"{case}: engine vs reference golden: cond {ec:.2e}, running mean {em:.2e} sigma, running var {ev:.2e} "
          f"({len(keys)} BatchNorms)")
    assert ec <= COND_BOUND and em <= MEAN_BOUND and ev <= VAR_BOUND


def _forward(head, fp, B, sizes, seed):
    g = torch.Generator().manual_seed(seed)
    gt = (torch.rand(B, 1, 4 * sizes[0][0], 4 * sizes[0][1], generator=g) * 2 + 0.1).to(DEV)
    noise = torch.randn(B, 16, 2 * sizes[0][0], 2 * sizes[0][1], generator=g).to(DEV)
    return head(fp, gt, torch.ones_like(gt), gt_depth_map=gt, noise=noise)


@pytest.mark.gpu
def test_running_stats_after_head_forward():
    kind, B, sizes = "DDIMDepthEstimate_Swin_ADDHAHI", 2, _swin_sizes(18, 27)
    head = _head(kind, 21).to(DEV)
    head.producer_train_bn = True
    head.train()
    head.conv_up[0][1].momentum = None  # cumulative average
    fp = _feats(head, B, sizes, 22)
    ref = copy.deepcopy(head).double().train()
    for it in range(2):
        _forward(head, fp, B, sizes, 30 + it)
        with torch.no_grad():
            ref._condition(ref._neck([f.double() for f in fp]))
    worst = 0.0
    for (name, bn), bn64 in zip(((n, m) for n, m in head.named_modules() if isinstance(m, nn.BatchNorm2d)
                                 and not n.startswith("depth_transform")),
                                (m for n, m in ref.named_modules() if isinstance(m, nn.BatchNorm2d)
                                 and not n.startswith("depth_transform"))):
        assert bn.num_batches_tracked.item() == bn64.num_batches_tracked.item() == 2, name
        sd = bn64.running_var.sqrt()
        em = ((bn.running_mean.double() - bn64.running_mean).abs() / sd).max().item()
        ev = ((bn.running_var.double() - bn64.running_var).abs() / bn64.running_var).max().item()
        worst = max(worst, em, ev)
        assert em <= MEAN_BOUND and ev <= VAR_BOUND, (name, em, ev)
    print("running stats worst", worst)


@pytest.mark.gpu
def test_repack_rule_and_eval_after_training(monkeypatch):
    kind, B, sizes = "DDIMDepthEstimate_Swin_ADD", 2, _swin_sizes(16, 32)
    head = _head(kind, 41).to(DEV)
    head.producer_train_bn = True
    head.train()
    fp = _feats(head, B, sizes, 42)
    loads = []
    orig = _ddim_head.DenoiseEngine.load_weights
    monkeypatch.setattr(_ddim_head.DenoiseEngine, "load_weights",
                        lambda self, t: (loads.append(self), orig(self, t))[1])
    opt = torch.optim.Adam(head.model.parameters(), lr=1e-4)

    def step(seed):
        out = _forward(head, fp, B, sizes, seed)
        opt.zero_grad()
        out["ddim_loss"].backward()
        opt.step()

    step(1)  # packs the forward's engine and creates the backward's
    n0 = len(loads)
    step(2)
    step(3)
    assert len(loads) == n0, "a training-mode iteration re-packed in full"
    head.eval()
    out = _forward(head, fp, B, sizes, 9)
    assert len(loads) == n0 + 1
    fresh = copy.deepcopy(head)
    ref = _forward(fresh, fp, B, sizes, 9)
    assert torch.equal(out["pred"], ref["pred"])
