"""Swin-L's stochastic depth on the engine (dd_backbone_config.mp_drop_path marks, dd_set_drop_path scales): against the
torch backbone the head falls back to (`native_backbone = False`) from the same CUDA seed, against the real reference's
golden (g_swin_drop_path.npz) at its masks, against fp64 torch of the mirror at BASELINE config 3's shape, and with an
image whose every branch is dropped.  At rate 0, or with the backbone in eval, nothing changes.

Each test prints its worst error over max |ref|."""
import copy

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import dd_helpers as helpers
from diffusiondepth_b200 import _cabi
from diffusiondepth_b200.engine import DenoiseEngine
from diffusiondepth_b200.model._blocks import MMCVDropPath
from oracle import restate
from oracle.make_denoiser_grads import sample_index
from oracle.make_swin_drop_path import CASES, OUT as GOLDEN, RATE, case_rgb

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0") if torch.cuda.is_available() else None
BOUND = 1e-4


def _model(rate, trained=True):
    """The mirror Swin_ADDHAHI model on the GPU in training mode, its backbone at drop-path rate `rate`."""
    model = copy.deepcopy(helpers.build_mirror("swinl", 2, trained=trained)).to(DEV).train()
    model.depth_backbone.set_drop_path_rate(rate)
    return model


def _engine(head, bb, B, hw):
    sizes = head.swin_pyramid(hw)
    return head._engine(B, ((hw[0] + 1) // 2, (hw[1] + 1) // 2), sizes[0], DEV,
                        feats=([192, 384, 768, 1536], sizes), image_hw=hw, backbone=bb)


def _ref64(bb, rgb, scales=None):
    """fp64 torch of the mirror backbone; scales [branch][B]: what its marked branches multiply by, in draw order."""
    ref = copy.deepcopy(bb).double()
    if scales is not None:
        from diffusiondepth_b200.model.head._ddim_head import DDIMHeadBase
        mods = DDIMHeadBase.swin_drop_paths(ref)[1]
        assert len(mods) == len(scales)
        for m, s in zip(mods, scales):
            m.forward = lambda x, s=s: x * s.to(x).reshape(-1, 1, 1)
    with torch.no_grad():
        return list(ref(rgb.double()))


def _err(x, ref):
    return ((x.double() - ref).abs().max() / ref.abs().max()).item()


def _forward(model, sample, seed):
    """One training-mode model forward from CUDA seed `seed`: (condition map, CUDA generator state after the forward,
    the masks the torch backbone's MMCVDropPath modules at a rate above 0 drew, per call)."""
    drawn, hooks = [], []
    for m in model.depth_backbone.modules():
        if isinstance(m, MMCVDropPath) and m.drop_prob > 0:
            hooks.append(m.register_forward_hook(
                lambda mod, a, o: drawn.append((o.flatten(1).abs().amax(1) > 0).float().cpu())))
    torch.cuda.manual_seed(seed)
    try:
        with torch.no_grad():
            model(sample)
    finally:
        for h in hooks:
            h.remove()
    return model.depth_head.last_cond.clone(), torch.cuda.get_rng_state(), drawn


def _sample(B, hw, seed=3):
    sample = {k: v.to(DEV) for k, v in restate.synthetic_sample(B, *hw, seed).items()}
    sample["noise"] = restate.synthetic_noise(B, *hw, seed).to(DEV)
    return sample


def test_native_matches_torch_fallback():
    """Rate 0.5, the same CUDA seed for the engine and the torch backbone: the same masks and generator state after the
    forward (ddim_loss's draws included), condition maps within 1e-4 of max."""
    B, hw, seed = 2, (70, 106), 77
    sample = _sample(B, hw)
    torch_model = _model(0.5)
    torch_model.depth_head.native_backbone = False
    native_model = copy.deepcopy(torch_model)
    native_model.depth_head.native_backbone = True
    assert native_model.depth_head.can_run_backbone(native_model.depth_backbone, sample["rgb"])
    assert not torch_model.depth_head.can_run_backbone(torch_model.depth_backbone, sample["rgb"])
    cond_t, rng_t, drawn = _forward(torch_model, sample, seed)
    cond_n, rng_n, none = _forward(native_model, sample, seed)
    assert not none and len(drawn) == 2 * 23  # the engine ran the backbone; torch drew a mask per marked branch
    assert torch.equal(rng_t, rng_n)
    head, bb = native_model.depth_head, native_model.depth_backbone
    torch.cuda.manual_seed(seed)
    masks = (head._swin_drop_scales(bb, B, DEV).reshape(-1, B) > 0).float().cpu()
    assert torch.equal(masks, torch.stack(drawn))
    assert 0 < int(masks.sum()) < masks.numel()
    ec = _err(cond_n, cond_t.double())
    print(f"\nswin drop path 0.5: {int(masks.sum())} of {masks.numel()} kept; engine vs torch fallback cond {ec:.2e}")
    assert ec <= BOUND


@pytest.mark.parametrize("case", list(CASES))
def test_golden_masks_give_golden_features(case):
    """dd_set_drop_path with the masks the real reference drew: its stage features within 1e-4 of their max."""
    golden = np.load(GOLDEN, allow_pickle=False)
    masks = torch.from_numpy(golden[case + "/masks"]).float()
    rgb = case_rgb(case).to(DEV)
    B, hw = rgb.shape[0], CASES[case]
    model = _model(RATE)
    head, bb = model.depth_head, model.depth_backbone
    keep = torch.tensor([1.0 - m.drop_prob for m in head.swin_drop_paths(bb)[1]])
    eng = _engine(head, bb, B, hw)
    eng.set_drop_path((masks / keep[:, None]).reshape(-1).contiguous().to(DEV))
    feats = eng.run_backbone(rgb, want_feats=True)
    eng.poll_status()
    worst = 0.0
    for i, f in enumerate(feats):
        flat = f.reshape(-1)
        got = flat[torch.from_numpy(sample_index(flat.numel())).to(DEV)].double().cpu()
        ref = torch.from_numpy(golden[f"{case}/feats/{i}/values"]).double()
        worst = max(worst, ((got - ref).abs().max() / float(golden[f"{case}/feats/{i}/absmax"])).item())
    print(f"\n[{case}] engine vs reference golden at its masks ({int(masks.sum())} of {masks.numel()} kept): {worst:.2e}")
    assert worst <= BOUND


def test_c3_shape_vs_fp64_mirror():
    """B = 4, 352 x 1216 (BASELINE config 3), rate 0.5, masks drawn by the head: stage features within 1e-4 relative of
    fp64 torch of the mirror at the same masks."""
    B, hw = 4, (352, 1216)
    model = _model(0.5)
    head, bb = model.depth_head, model.depth_backbone
    rgb = torch.randn(B, 3, *hw, generator=torch.Generator().manual_seed(8)).to(DEV)
    eng = _engine(head, bb, B, hw)
    torch.cuda.manual_seed(5)
    scales = head._swin_drop_scales(bb, B, DEV)
    eng.set_drop_path(scales)
    feats = eng.run_backbone(rgb, want_feats=True)
    eng.poll_status()
    ref = _ref64(bb, rgb, scales.reshape(-1, B).double())
    errs = [_err(f, r) for f, r in zip(feats, ref)]
    print(f"\nswin C3 drop path: {int((scales > 0).sum())} of {scales.numel()} kept; stages", ["%.2e" % e for e in errs])
    assert max(errs) <= BOUND


def test_every_branch_dropped():
    """Image 0 drops every marked branch (all but stage 0's block 0): the restatement with those blocks removed.  Image
    1 keeps every branch: the mirror at scale 1 / keep."""
    B, hw = 2, (70, 106)
    model = _model(0.3)
    head, bb = model.depth_head, model.depth_backbone
    rgb = torch.randn(B, 3, *hw, generator=torch.Generator().manual_seed(9)).to(DEV)
    keep = torch.tensor([1.0 - m.drop_prob for m in head.swin_drop_paths(bb)[1]], dtype=torch.float32)
    scales = torch.stack([torch.zeros_like(keep), 1.0 / keep], 1)  # [branch][B]
    eng = _engine(head, bb, B, hw)
    eng.set_drop_path(scales.reshape(-1).contiguous().to(DEV))
    feats = eng.run_backbone(rgb, want_feats=True)
    eng.poll_status()
    bare = copy.deepcopy(bb)
    bare.stages[0].blocks = bare.stages[0].blocks[:1]
    for st in bare.stages[1:]:
        st.blocks = nn.ModuleList()
    ref0 = _ref64(bare.eval(), rgb[:1])
    ref1 = _ref64(bb, rgb[1:], scales[:, 1:].double())
    e0 = max(_err(f[:1], r) for f, r in zip(feats, ref0))
    e1 = max(_err(f[1:], r) for f, r in zip(feats, ref1))
    print(f"\nevery branch dropped: {e0:.2e}; every branch kept: {e1:.2e}")
    assert e0 <= BOUND and e1 <= BOUND


def test_rate_zero_and_eval_unchanged():
    """At rate 0, or with the backbone in eval, the forward is what it was: the same condition map bit for bit, workspace
    size, graph captures and launches as an engine without marks.  Switching stochastic depth on, off and on again
    captures nothing new."""
    B, hw, seed = 2, (70, 106), 11
    sample = _sample(B, hw)
    runs = []
    for rate in (0.0, 0.1):
        model = _model(rate)
        model.depth_head.capture_cond = True
        model.depth_backbone.eval()
        cond, rng, drawn = _forward(model, sample, seed)
        eng = next(e for e in model.depth_head._engines.values() if e.backbone is not None)
        assert not drawn
        runs.append((model, cond, rng, eng.lib.dd_workspace_bytes(eng._h), eng.graph_capture_count(),
                     eng.last_launch_count))
    (_, c0, r0, *rest0), (model, c1, r1, *rest1) = runs
    assert torch.equal(c0, c1) and torch.equal(r0, r1) and rest0 == rest1
    assert model.depth_head._native_drop_paths(hw, model.depth_backbone) is not None
    eng = next(e for e in model.depth_head._engines.values() if e.backbone is not None)
    counts = []
    for train in (True, False, True, False, True):
        model.depth_backbone.train(train)
        cond, _, _ = _forward(model, sample, seed)
        counts.append(eng.graph_capture_count())
        if not train:
            assert torch.equal(cond, c0)
    print(f"\ngraph captures while switching: {counts}")
    assert counts[1:] == [counts[1]] * 4 and counts[0] == counts[1]  # eval's graph existed; on was captured once


def test_wrong_count_is_invalid_and_engine_stays_usable():
    B, hw = 2, (64, 96)
    model = _model(0.5)
    head, bb = model.depth_head, model.depth_backbone
    rgb = torch.randn(B, 3, *hw, generator=torch.Generator().manual_seed(2)).to(DEV)
    eng = _engine(head, bb, B, hw)
    torch.cuda.manual_seed(1)
    scales = head._swin_drop_scales(bb, B, DEV)
    eng.set_drop_path(scales)
    before = eng.run_backbone(rgb, want_feats=True)
    for bad in (scales[:-1], torch.cat([scales, scales[:B]])):
        with pytest.raises(_cabi.EngineError, match="DD_ERR_INVALID"):
            eng.set_drop_path(bad.contiguous())
    after = eng.run_backbone(rgb, want_feats=True)  # the earlier scales stay in force
    eng.poll_status()
    assert all(torch.equal(a, b) for a, b in zip(before, after))


def test_adam_iteration_with_grad_through_loop(monkeypatch):
    """A training-mode Swin_ADDHAHI at rate 0.1 with grad_through_loop: Adam iterations on the loop's parameters re-pack
    by update, never by a full load_weights, once the engines exist."""
    B, hw = 2, (64, 96)
    model = _model(0.1, trained=False)
    head = model.depth_head
    head.grad_through_loop = True
    sample = _sample(B, hw, seed=4)
    loads = []
    real = DenoiseEngine.load_weights
    monkeypatch.setattr(DenoiseEngine, "load_weights", lambda self, t: (loads.append(len(t)), real(self, t))[1])
    keys, params = head._loop_params()
    opt = torch.optim.Adam(params, lr=1e-4)
    counts = []
    for i in range(3):
        torch.manual_seed(60 + i)
        opt.zero_grad()
        out = model(sample)
        loss = F.l1_loss(out["pred"], sample["gt"]) + out["ddim_loss"]
        loss.backward()
        assert torch.isfinite(loss) and all(p.grad is not None and torch.isfinite(p.grad).all() for p in params)
        opt.step()
        counts.append(len(loads))
    print(f"\nfull loads after each iteration: {counts}")
    assert counts[1:] == [counts[0]] * 2
