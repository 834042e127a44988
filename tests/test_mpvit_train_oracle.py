"""The fp64 mirror MPViT head in training mode (mirror `mpvit_small` in `.train()` with its DropPath modules in eval,
then the head's own `_condition(_neck(.))`) and the head's running-statistic update (`bn_running_update`) behave like
the real reference in `.train()`: which BatchNorms run and update, their batch statistics, the four stage outputs, the
condition map and the running statistics after one call, against tests/golden/g_mpvit_train.npz
(oracle/make_mpvit_train.py).  This pins the mirror modules the GPU tests of tests/test_mpvit_train.py compare against."""
import copy

import numpy as np
import pytest
import torch
import torch.nn as nn

import dd_helpers as helpers
from diffusiondepth_b200.model._blocks import DropPath
from diffusiondepth_b200.model.head._ddim_head import bn_running_update
from oracle.make_denoiser_grads import checksum, sample_index
from oracle.make_mpvit_train import CASES, FAMILY, OUT, case_inputs
from oracle.make_producer_train import PRODUCER_PREFIXES


@pytest.fixture(scope="module")
def golden():
    return np.load(OUT, allow_pickle=False)


def mirror_mpvit_train(dtype=torch.float64):
    """The trained-like mirror MPViT model in training mode with stochastic depth off."""
    m = copy.deepcopy(helpers.build_mirror(FAMILY, 2, trained=True)).to("cpu", dtype).train()
    for mod in m.modules():
        if isinstance(mod, DropPath):
            mod.eval()
    return m


def _sampled(t):
    flat = t.reshape(-1)
    return flat[torch.from_numpy(sample_index(flat.numel()))]


@pytest.mark.parametrize("case", list(CASES))
def test_mirror_mpvit_matches_reference_train(case, golden):
    sample = case_inputs(case)
    assert checksum(sample["rgb"]) == pytest.approx(float(golden[case + "/input_checksum"]), rel=1e-12)
    start = mirror_mpvit_train()
    model = copy.deepcopy(start)
    stats, hooks, order = {}, [], []
    for n, mod in model.named_modules():
        if isinstance(mod, nn.BatchNorm2d) and n.startswith(PRODUCER_PREFIXES):
            def pre(m, a, n=n):
                x = a[0].detach()
                stats[n] = (x.mean((0, 2, 3)), x.var((0, 2, 3), unbiased=True))
                order.append(n)
            hooks.append(mod.register_forward_pre_hook(pre))
    try:
        with torch.no_grad():
            feats = list(model.depth_backbone(sample["rgb"].double()))
            head = model.depth_head
            cond = head._condition(head._neck(feats))
    finally:
        for h in hooks:
            h.remove()
    p = case + "/bn/"
    keys = sorted({k[len(p):-len("/mean")] for k in golden.files if k.startswith(p) and k.endswith("/mean")})
    assert sorted(stats) == keys  # the same BatchNorms run on the way to the condition map
    assert sum(1 for n in order if n.startswith("depth_backbone.")) == 29
    worst = {"feats": 0.0}
    for i, f in enumerate(feats):
        ref = golden[f"{case}/feats/{i}/values"]
        worst["feats"] = max(worst["feats"],
                             float((_sampled(f) - torch.from_numpy(ref).double()).abs().max() / np.abs(ref).max()))
    worst["cond"] = float((_sampled(cond) - torch.from_numpy(golden[case + "/cond/values"]).double()).abs().max()
                          / float(golden[case + "/cond/absmax"]))
    em = ev = er = 0.0
    for k in keys:
        g = {f: torch.from_numpy(golden[f"{case}/bn/{k}/{f}"]).double()
             for f in ("mean", "var", "running_mean", "running_var")}
        mean, var = stats[k]
        sd = g["var"].sqrt()
        em = max(em, float(((mean - g["mean"]).abs() / sd).max()))
        ev = max(ev, float(((var - g["var"]).abs() / g["var"]).max()))
        bn = copy.deepcopy(start.get_submodule(k))
        assert bn.num_batches_tracked.item() == 0
        assert (bn.momentum if bn.momentum is not None else -1.0) == float(golden[f"{case}/bn/{k}/momentum"])
        bn_running_update(bn, mean, var)
        assert int(bn.num_batches_tracked) == int(golden[f"{case}/bn/{k}/num_batches_tracked"]) == 1
        er = max(er, float(((bn.running_mean - g["running_mean"]).abs() / sd).max()),
                 float(((bn.running_var - g["running_var"]).abs() / g["running_var"]).max()))
        torch.testing.assert_close(model.get_submodule(k).running_mean, bn.running_mean, rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(model.get_submodule(k).running_var, bn.running_var, rtol=1e-12, atol=1e-12)
    print(f"\n[{case}] fp64 mirror vs fp32 reference: feats {worst['feats']:.1e}, cond {worst['cond']:.1e}, "
          f"batch mean {em:.1e} sigma, variance {ev:.1e}, running statistics {er:.1e} ({len(keys)} BatchNorms)")
    assert worst["feats"] <= 1e-4 and worst["cond"] <= 1e-4
    assert em <= 1e-4 and ev <= 2e-4 and er <= 2e-5
