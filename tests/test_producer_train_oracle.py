"""The fp64 training-mode mirror producers (the head's own `_condition(_neck(.))` and the mirror backbone in `.train()`)
and the head's running-statistic update (`bn_running_update`) behave like the real reference in `.train()`: which
BatchNorms run and update, their batch statistics, the condition map, and the running statistics after one call,
against tests/golden/g_producer_train.npz (oracle/make_producer_train.py).  This pins the mirror modules the GPU tests of
tests/test_producer_train_bn.py compare against."""
import copy

import numpy as np
import pytest
import torch
import torch.nn as nn

import dd_helpers as helpers
from diffusiondepth_b200.model.head._ddim_head import bn_running_update
from oracle.make_denoiser_grads import checksum, sample_index
from oracle.make_producer_train import CASES, OUT, PRODUCER_PREFIXES, case_inputs


@pytest.fixture(scope="module")
def golden():
    return np.load(OUT, allow_pickle=False)


def golden_bn_keys(golden, case):
    p = case + "/bn/"
    return sorted({k[len(p):-len("/mean")] for k in golden.files if k.startswith(p) and k.endswith("/mean")})


def mirror_train(family, dtype=torch.float64):
    """The trained-like mirror model in training mode (a Swin backbone in eval: DropPath off)."""
    m = copy.deepcopy(helpers.build_mirror(family, 2, trained=True)).to("cpu", dtype).train()
    if family.startswith("swin"):
        m.depth_backbone.eval()
    return m


def mirror_forward(model, rgb):
    """-> (feats, cond, {BatchNorm name: (batch mean, unbiased batch variance)}) of one training-mode call."""
    stats, hooks = {}, []
    for n, mod in model.named_modules():
        if isinstance(mod, nn.BatchNorm2d) and n.startswith(PRODUCER_PREFIXES):
            def pre(m, a, n=n):
                x = a[0].detach()
                stats[n] = (x.mean((0, 2, 3)), x.var((0, 2, 3), unbiased=True))
            hooks.append(mod.register_forward_pre_hook(pre))
    try:
        with torch.no_grad():
            feats = list(model.depth_backbone(rgb))
            head = model.depth_head
            cond = head._condition(head._neck(feats))
    finally:
        for h in hooks:
            h.remove()
    return feats, cond, stats


def _sampled(t):
    flat = t.reshape(-1)
    return flat[torch.from_numpy(sample_index(flat.numel()))]


@pytest.mark.parametrize("case", list(CASES))
def test_mirror_producers_match_reference_train(case, golden):
    family, sample = case_inputs(case)
    assert checksum(sample["rgb"]) == pytest.approx(float(golden[case + "/input_checksum"]), rel=1e-12)
    start = mirror_train(family)
    model = copy.deepcopy(start)
    feats, cond, stats = mirror_forward(model, sample["rgb"].double())
    keys = golden_bn_keys(golden, case)
    assert sorted(stats) == keys  # the same BatchNorms run on the way to the condition map
    worst = {}
    for i, f in enumerate(feats):
        ref = golden[f"{case}/feats/{i}/values"]
        worst["feats"] = max(worst.get("feats", 0.0),
                             float((_sampled(f) - torch.from_numpy(ref).double()).abs().max() / np.abs(ref).max()))
    worst["cond"] = float((_sampled(cond) - torch.from_numpy(golden[case + "/cond/values"]).double()).abs().max()
                          / float(golden[case + "/cond/absmax"]))
    em = ev = er = 0.0
    for k in keys:
        g = {f: torch.from_numpy(golden[f"{case}/bn/{k}/{f}"]).double() for f in ("mean", "var", "running_mean",
                                                                                 "running_var")}
        mean, var = stats[k]
        sd = g["var"].sqrt()
        em = max(em, float(((mean - g["mean"]).abs() / sd).max()))
        ev = max(ev, float(((var - g["var"]).abs() / g["var"]).max()))
        # the head's update from the mirror's statistics, on the BatchNorm's starting state
        bn = copy.deepcopy(start.get_submodule(k))
        assert bn.num_batches_tracked.item() == 0
        assert (bn.momentum if bn.momentum is not None else -1.0) == float(golden[f"{case}/bn/{k}/momentum"])
        bn_running_update(bn, mean, var)
        assert int(bn.num_batches_tracked) == int(golden[f"{case}/bn/{k}/num_batches_tracked"]) == 1
        # running mean in units of the batch sigma (it may sit near 0), running variance relative
        er = max(er, float(((bn.running_mean - g["running_mean"]).abs() / sd).max()),
                 float(((bn.running_var - g["running_var"]).abs() / g["running_var"]).max()))
        # torch's own training-mode update in the mirror agrees with it
        torch.testing.assert_close(model.get_submodule(k).running_mean, bn.running_mean, rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(model.get_submodule(k).running_var, bn.running_var, rtol=1e-12, atol=1e-12)
    print(f"\n[{case}] fp64 mirror vs fp32 reference: feats {worst['feats']:.1e}, cond {worst['cond']:.1e}, "
          f"batch mean {em:.1e} sigma, variance {ev:.1e}, running statistics {er:.1e} ({len(keys)} BatchNorms)")
    assert worst["feats"] <= 1e-4 and worst["cond"] <= 1e-4
    assert em <= 1e-4 and ev <= 2e-4 and er <= 2e-5
