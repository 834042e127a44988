"""dd_update_weights: after an optimizer step only the changed denoiser / codec tensors are re-packed, in place.  The
result must be bit-identical to a full dd_finalize_weights from the same tensors, CUDA graphs must survive unless a
kernel argument they hold by value changed (a conv's power-of-two weight scale, the decoder's final bias), and a rejected
update must leave the engine as it was.  The head's decision between update and full pack is checked without a device."""
import copy

import pytest
import torch
import torch.nn.functional as F

import dd_helpers as helpers
from diffusiondepth_b200._cabi import EngineError
from diffusiondepth_b200.engine import (DECODER_PARAM_KEYS, DENOISER_KEYS, ENCODER_KEYS, FUSE_KEYS, DenoiseEngine,
                                        is_updatable)
from diffusiondepth_b200.model.head import _ddim_head
from diffusiondepth_b200.model.head._ddim_head import repack_plan
from diffusiondepth_b200.model.registry import HEADS

DEV = torch.device("cuda:0")
DEC = "depth_transform.conv_inv_transform."
ENC = "depth_transform.conv_transform."


# ---------------------------------------------------------------------------------------------- the head's decision (CPU)
def test_repack_plan():
    keys = ["model.pred.0.weight", DEC + "1.running_var", ENC + "0.0.weight", "conv_lateral.0.0.weight", "backbone.x"]
    sig = tuple((100 + i, 0) for i in range(5))

    def bump(*idx):
        return tuple((p, v + (i in idx)) for i, (p, v) in enumerate(sig))

    assert repack_plan(keys, sig, keys, sig) == []
    assert repack_plan(keys, sig, keys, bump(0, 1, 2)) == keys[:3]
    assert repack_plan(keys, sig, keys, bump(1)) == [keys[1]]
    assert repack_plan(keys, sig, keys, bump(0, 3)) is None       # the FPN changed too
    assert repack_plan(keys, sig, keys, bump(4)) is None          # the backbone changed
    assert repack_plan(keys, sig, keys[:4], sig[:4]) is None      # a different key set
    assert repack_plan(keys, None, keys, sig) is None             # never packed
    assert repack_plan(keys, sig, keys, bump(0), incremental=False) is None
    assert all(is_updatable(k) for k in DENOISER_KEYS + FUSE_KEYS + DECODER_PARAM_KEYS + ENCODER_KEYS)
    assert not any(is_updatable(k) for k in ("hahineck.a", "conv_lateral.0.0.weight", "conv_up.0.0.weight", "backbone.x"))


class _FakeEngine:
    """Stands in for DenoiseEngine inside _ddim_head: records which tensors each pack call received."""
    calls = []

    def __init__(self, *args, **kwargs):
        pass

    def set_schedule(self, *args):
        pass

    def enable_producers(self, *args, **kwargs):
        pass

    def load_weights(self, tensors):
        _FakeEngine.calls.append(("load", sorted(tensors)))

    def update_weights(self, tensors):
        _FakeEngine.calls.append(("update", sorted(tensors)))

    def close(self):
        pass


def test_head_chooses_update_or_full_load(monkeypatch):
    monkeypatch.setattr(_ddim_head, "DenoiseEngine", _FakeEngine)
    _FakeEngine.calls = calls = []
    head = HEADS.build(dict(type="DDIMDepthEstimate_Res", in_channels=[64, 128, 256, 512], inference_steps=2,
                            num_train_timesteps=1000, depth_feature_dim=16, loss_cfgs=[], init_cfg=None))
    feats = ([64, 128, 256, 512], [(8, 16), (4, 8), (2, 4), (1, 2)])

    def fetch(**kw):
        return head._engine(1, (8, 16), (8, 16), "cpu", feats=feats, **kw)

    fetch()
    assert [c[0] for c in calls] == ["load"] and "conv_lateral.0.0.weight" in calls[0][1]
    fetch()
    assert len(calls) == 1  # nothing changed
    with torch.no_grad():
        head.model.pred[0].weight.add_(1.0)  # in place, as an optimizer does
        head.depth_transform.conv_inv_transform[1].running_var.mul_(2.0)
    fetch()
    assert calls[-1] == ("update", sorted(["model.pred.0.weight", DEC + "1.running_var"]))
    head.model.time_embedding.weight.data = torch.zeros(1280, 256)  # a new tensor behind the same Parameter
    fetch()
    assert calls[-1] == ("update", ["model.time_embedding.weight"])
    fetch(loop_backward=True)  # another engine of the head: never packed
    assert calls[-1][0] == "load" and len(calls) == 4
    with torch.no_grad():
        head.model.pred[0].bias.add_(1.0)
        head.conv_lateral[0][0].weight.add_(1.0)  # the update does not re-pack the FPN
    fetch()
    assert calls[-1][0] == "load" and len(calls) == 5
    fetch(loop_backward=True)
    assert calls[-1][0] == "load" and len(calls) == 6
    head.incremental_repack = False
    with torch.no_grad():
        head.model.pred[0].bias.add_(1.0)
    fetch()
    assert calls[-1][0] == "load" and len(calls) == 7
    fetch()
    assert len(calls) == 7


# ---------------------------------------------------------------------------------------------- engine level (GPU)
def _state(variant):
    from oracle.make_loop_grads import loop_state
    return {k: v.to(DEV) for k, v in loop_state(variant).items()}


def _engine(variant, sd, B, hw, T, **flags):
    from diffusiondepth_b200.model.diffusers.schedulers.scheduling_ddim import DDIMScheduler
    chw = ((hw[0] + 1) // 2, (hw[1] + 1) // 2) if variant == "swin" else hw
    eng = DenoiseEngine(variant, B, hw, chw, T, DEV, **flags)
    eng.set_schedule(*DDIMScheduler(num_train_timesteps=1000, clip_sample=False).fused_coefficients(T))
    if sd is not None:
        eng.load_weights(sd)
    return eng


def _inputs(variant, B, hw, seed=5):
    h, w = hw
    chw = ((h + 1) // 2, (w + 1) // 2) if variant == "swin" else hw
    g = torch.Generator().manual_seed(seed)
    return dict(cond=torch.randn(B, 256, *chw, generator=g).abs().to(DEV), noise=torch.randn(B, 16, h, w, generator=g).to(DEV),
                gt=(torch.rand(B, 1, 2 * h, 2 * w, generator=g) * 80).to(DEV),
                d_eps=(torch.randn(B, 16, h, w, generator=g) / (B * 16 * h * w)).to(DEV),
                d_depth=(torch.randn(B, 1, 2 * h, 2 * w, generator=g) / (B * 4 * h * w)).to(DEV))


def _outputs(eng, x):
    """Everything the engine computes from its packed weights, as one dict of tensors."""
    out = {}
    if eng.step_decode:
        out["steps"], out["latent"], out["logits"] = eng.denoise_decode_steps(x["cond"], x["noise"], True, True)
    else:
        out["depth"], out["latent"], out["logits"] = eng.denoise_decode(x["cond"], x["noise"], True, True)
    out["eps"] = eng.denoiser_forward(x["cond"], x["noise"], 417)
    out["encode"] = eng.encode(x["gt"])
    if eng.backward:
        dc, dn, gr = eng.denoiser_backward(x["cond"], x["noise"], 417, x["d_eps"])
        out.update({"op/" + k: v for k, v in gr.items()}, op_d_cond=dc, op_d_noisy=dn)
    if eng.loop_backward:
        dc, dn, gr, _ = eng.denoise_backward(x["cond"], x["noise"], x["d_depth"], out["latent"] * 1e-3)
        out.update({"loop/" + k: v for k, v in gr.items()}, loop_d_cond=dc, loop_d_noise=dn)
    eng.poll_status()
    return out


def _assert_same(got, want, tag):
    assert got.keys() == want.keys()
    for k in want:
        assert torch.equal(got[k], want[k]), (tag, k, float((got[k] - want[k]).abs().max()))


def _nudge(sd, keys, gen, rel=1e-3):
    """In place, the size of an SGD step: each tensor moves by `rel` of its mean magnitude."""
    for k in keys:
        t = sd[k]
        t.add_(torch.randn(t.shape, generator=gen).to(DEV) * t.abs().mean() * rel)
    return {k: sd[k] for k in keys}


def _cases(variant):
    fuse = FUSE_KEYS if variant == "swin" else ()
    return [("sgd", DENOISER_KEYS + fuse + DECODER_PARAM_KEYS),
            ("pred.0.weight", ("model.pred.0.weight",)),
            ("bias", ("model.upsample_fuse.convB.conv.bias" if variant == "swin" else "model.pred.0.bias",)),
            ("groupnorm", ("model.noise_embedding.4.weight",)),
            ("time_embedding", ("model.time_embedding.weight",)),
            ("running_var", (DEC + "1.running_var",)),
            ("encoder", (ENC + "0.0.weight", ENC + "1.1.running_mean"))]


MODES = {"plain": {}, "backward": dict(backward=True), "loop_backward": dict(loop_backward=True),
         "step_decode": dict(step_decode=True)}
EQUIV = [(v, hw, B, 3, m, None) for v, hw, B in (("swin", (19, 27), 3), ("res", (35, 53), 2)) for m in MODES]
EQUIV += [("swin", (35, 53), 2, 3, "loop_backward", None), ("res", (19, 27), 3, 3, "loop_backward", None),
          ("swin", (88, 304), 2, 20, "loop_backward", ("sgd", "pred.0.weight"))]


@pytest.mark.gpu
@pytest.mark.parametrize("variant,hw,B,T,mode,only", EQUIV)
def test_update_equals_fresh_finalize(variant, hw, B, T, mode, only):
    """Engine A is packed once and then updated case after case; after each, a fresh engine B finalized from the same
    tensors must compute the same bits, forward and backward."""
    sd = _state(variant)
    x = _inputs(variant, B, hw)
    a = _engine(variant, sd, B, hw, T, **MODES[mode])
    _outputs(a, x)  # captures A's loop graph before any update
    gen = torch.Generator().manual_seed(11)
    for name, keys in _cases(variant):
        if only is not None and name not in only:
            continue
        rel = 0.3 if name == "running_var" else 1e-2
        if name == "running_var":
            sd[keys[0]].mul_(1.5)
            changed = {keys[0]: sd[keys[0]]}
        else:
            changed = _nudge(sd, keys, gen, rel)
        a.update_weights(changed)
        b = _engine(variant, sd, B, hw, T, **MODES[mode])
        _assert_same(_outputs(a, x), _outputs(b, x), name)
        b.close()
    a.close()


@pytest.mark.gpu
@pytest.mark.parametrize("variant,scaled", [("swin", "model.upsample_fuse.convA.conv.weight"), ("res", "model.pred.0.weight")])
def test_loop_graph_survives_unless_a_scale_changes(variant, scaled):
    B, hw, T = 2, (19, 27), 3
    sd = _state(variant)
    x = _inputs(variant, B, hw)
    a = _engine(variant, sd, B, hw, T)
    _outputs(a, x)
    assert a.graph_capture_count() == 1
    gen = torch.Generator().manual_seed(3)
    trained = DENOISER_KEYS + (FUSE_KEYS if variant == "swin" else ()) + DECODER_PARAM_KEYS
    a.update_weights(_nudge(sd, trained, gen, 1e-3))  # no max |w| crosses a power of two
    out = _outputs(a, x)
    assert a.graph_capture_count() == 1
    b = _engine(variant, sd, B, hw, T)
    _assert_same(out, _outputs(b, x), "nudge")
    b.close()
    sd[scaled].mul_(4.0)  # its split scale drops by 4: the captured acc_scale would be a silent 4x error
    a.update_weights({scaled: sd[scaled]})
    out = _outputs(a, x)
    assert a.graph_capture_count() == 2
    b = _engine(variant, sd, B, hw, T)
    _assert_same(out, _outputs(b, x), "x4")
    a.update_weights({})
    assert a.graph_capture_count() == 2
    _assert_same(_outputs(a, x), out, "empty update")


@pytest.mark.gpu
def test_step_decode_graph_follows_the_decoder_bias():
    B, hw, T = 2, (19, 27), 3
    sd = _state("res")
    x = _inputs("res", B, hw)
    a = _engine("res", sd, B, hw, T, step_decode=True)
    a.denoise_decode(x["cond"], x["noise"])
    _outputs(a, x)
    assert a.graph_capture_count() == 2  # the plain loop and the step-decode loop
    key = DEC + "3.0.bias"
    sd[key].add_(0.25)
    a.update_weights({key: sd[key]})
    a.denoise_decode(x["cond"], x["noise"])
    assert a.graph_capture_count() == 2  # the plain loop graph does not hold the bias
    out = _outputs(a, x)
    assert a.graph_capture_count() == 3
    _assert_same(out, _outputs(_engine("res", sd, B, hw, T, step_decode=True), x), "decoder bias")


@pytest.mark.gpu
def test_rejected_update_leaves_the_engine_intact():
    B, hw, T = 2, (19, 27), 3
    sd = _state("swin")
    x = _inputs("swin", B, hw)
    fresh = _engine("swin", None, B, hw, T)
    with pytest.raises(EngineError, match="dd_finalize_weights"):
        fresh.update_weights({"model.pred.0.bias": sd["model.pred.0.bias"]})
    fresh.load_weights(sd)  # the early registration was forgotten: a full set is needed and accepted
    before = _outputs(fresh, x)
    captures = fresh.graph_capture_count()
    bad = {"model.pred.0.bias": sd["model.pred.0.bias"] + 1, "model.pred.3.weight": torch.zeros(16, 64, 3, 1, device=DEV)}
    with pytest.raises(EngineError, match="shape"):
        fresh.update_weights(bad)
    _assert_same(_outputs(fresh, x), before, "after a wrong shape")
    with pytest.raises(EngineError, match="DD_ERR_UNSUPPORTED.*dd_finalize_weights"):
        fresh.update_weights({"model.pred.0.bias": sd["model.pred.0.bias"] + 1,
                              "conv_lateral.0.0.weight": torch.zeros(256, 192, 3, 3, device=DEV)})
    with pytest.raises(EngineError):
        fresh.update_weights({"model.nonsense": torch.zeros(3, device=DEV)})
    _assert_same(_outputs(fresh, x), before, "after an unsupported key")
    assert fresh.graph_capture_count() == captures
    lib = fresh.lib  # dd_set_weight without finalize or update still blocks the forward
    t = sd["model.pred.0.bias"]
    import ctypes as C
    assert lib.dd_set_weight(fresh._h, b"model.pred.0.bias", C.c_void_p(t.data_ptr()), (C.c_int64 * 1)(64), 1) == 0
    with pytest.raises(EngineError, match="dd_finalize_weights has not been called"):
        fresh.denoise_decode(x["cond"], x["noise"])
    fresh.update_weights({})
    _assert_same(_outputs(fresh, x), before, "after the pending registration was applied")


# ---------------------------------------------------------------------------------------------- head level (GPU)
def _train(step_fn, head, iters=4, lr=1e-3):
    """`iters` iterations of forward, L1 + ddim_loss, backward, SGD on the head's loop parameters: per iteration
    (pred, loss, parameters after the step) and the head's graph captures so far."""
    head.train()
    head.grad_through_loop = True
    keys, params = head._loop_params()
    opt = torch.optim.SGD(params, lr=lr)
    log, captures = [], []
    for i in range(iters):
        torch.manual_seed(40 + i)  # ddim_loss draws its noise and t from the global RNG
        opt.zero_grad()
        out, gt = step_fn()
        loss = F.l1_loss(out["pred"], gt) + out["ddim_loss"]
        loss.backward()
        opt.step()
        log.append([out["pred"].detach().clone(), loss.detach().clone()] + [p.detach().clone() for p in params])
        captures.append(sum(e.graph_capture_count() for e in head._engines.values()))
    return log, captures


def _assert_runs_equal(on, off):
    for i, (a, b) in enumerate(zip(on, off)):
        for j, (u, v) in enumerate(zip(a, b)):
            assert torch.equal(u, v), (i, j)


@pytest.mark.gpu
def test_training_res_model_with_native_backbone():
    from oracle import restate
    m_on = copy.deepcopy(helpers.build_mirror("res18", 3)).to(DEV)
    m_off = copy.deepcopy(m_on)
    m_off.depth_head.incremental_repack = False
    sample = {k: v.to(DEV) for k, v in restate.synthetic_sample(2, 76, 108, 9).items()}
    sample["noise"] = restate.synthetic_noise(2, 76, 108, 9).to(DEV)
    assert m_on.depth_head.can_run_backbone(m_on.depth_backbone, sample["rgb"])
    runs = []
    for m in (m_on, m_off):
        log, captures = _train(lambda: (m(sample), sample["gt"]), m.depth_head)
        runs.append((log, captures))
    _assert_runs_equal(runs[0][0], runs[1][0])
    on, off = runs[0][1], runs[1][1]
    # backbone, condition and loop graph.  The first backward creates the loop-backward engine and grows the workspace
    # the head's engines share, so the second forward binds a new workspace and captures once more; from then on an
    # optimizer step costs no capture, while the full re-pack captures all three every iteration.
    assert on[0] == 3 and on[1:] == [on[1]] * 3, on
    assert [b - a for a, b in zip(off, off[1:])] == [3, 3, 3], off


@pytest.mark.gpu
def test_training_swin_head_on_a_pyramid():
    torch.manual_seed(7)
    h_on = HEADS.build(dict(type="DDIMDepthEstimate_Swin_ADDHAHI", in_channels=[64, 128, 256, 512], inference_steps=3,
                            num_train_timesteps=1000, depth_feature_dim=16, loss_cfgs=[], init_cfg=None)).to(DEV)
    h_off = copy.deepcopy(h_on)
    h_off.incremental_repack = False
    g = torch.Generator().manual_seed(2)
    fp = [torch.randn(2, c, *s, generator=g).to(DEV) for c, s in
          zip(h_on.fpn_in_channels, [(10, 14), (5, 7), (3, 4), (2, 2)])]
    gt = (torch.rand(2, 1, 38, 54, generator=g) * 2 + 0.1).to(DEV)
    noise = torch.randn(2, 16, 19, 27, generator=g).to(DEV)
    runs = []
    for head in (h_on, h_off):
        runs.append(_train(lambda: (head(fp, gt, gt > 0, gt_depth_map=gt, noise=noise), gt), head))
    _assert_runs_equal(runs[0][0], runs[1][0])
    on, off = runs[0][1], runs[1][1]
    assert on[1:] == [on[1]] * 3, on  # as above: nothing is captured once both engines exist
    assert off[-1] > off[1], off
