"""dd_denoiser_backward: the native backward of ScheduledCNNRefine against the fp64 restatement (itself pinned to the real
reference's autograd by test_denoiser_grads_oracle.py) and against the reference's stored gradients, its determinism,
the autograd Function around it, training through it, and its argument checks."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from diffusiondepth_b200 import _cabi
from diffusiondepth_b200.engine import DenoiseEngine
from diffusiondepth_b200.model._blocks import exact_fp32
from grad_helpers import (CASES, GOLDEN, case_inputs, denoiser_state, golden_margins, kink_envelope, make_head,
                          restatement_grads, tensor_margins)
from oracle import restate

DEV = torch.device("cuda:0")
TOL = 1e-4    # of max |g_ref| per gradient
BAND = 2e-5   # ReLU inputs this close to zero may land on the other side in an fp32-grade forward (kink_envelope)
T3 = (417, 417, 12)


def _inputs(variant, hw, seed=5):
    h, w = hw
    ch, cw = ((h + 1) // 2, (w + 1) // 2) if variant == "swin" else (h, w)
    g = torch.Generator().manual_seed(seed)
    noisy = torch.randn(3, 16, h, w, generator=g)
    cond = torch.randn(3, 256, ch, cw, generator=g).abs()
    d_eps = torch.randn(3, 16, h, w, generator=g) * (2.0 / (3 * 16 * h * w))
    return noisy, cond, d_eps


def _engine_grads(head, variant, noisy, cond, t, d_eps):
    eng = head._engine(noisy.shape[0], noisy.shape[-2:], cond.shape[-2:], DEV, backward=True)
    d_cond, d_noisy, grads = eng.denoiser_backward(cond.to(DEV), noisy.to(DEV), list(t), d_eps.to(DEV))
    eng.poll_status()
    out = {"d_cond": d_cond, "d_noisy": d_noisy}
    out.update(grads)
    return out


def _check(tag, got, ref, env):
    m = tensor_margins(got, ref)
    worst = max(m, key=m.get)
    print(f"\n[{tag}] worst {worst} {m[worst]:.2e}; " + " ".join(f"{k.replace('model.', '')}={v:.1e}" for k, v in m.items()))
    for k in m:  # the envelope flips every near-kink mask at once; a subset of them may move a sum a little further
        assert m[k] <= TOL + 2 * env[k], (tag, k, m[k], env[k])


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["swin", "res"])
# (176, 352), B = 3: the wide layers' weight gradients sum 25 split-K chunks of 6-segment rows (a 352 x 704 crop)
@pytest.mark.parametrize("hw", [(19, 27), (18, 26), (35, 53), (8, 16), (176, 352)])
def test_gradients_vs_fp64_restatement(variant, hw):
    sd = denoiser_state(variant)
    head = make_head(variant, sd, DEV)
    noisy, cond, d_eps = _inputs(variant, hw)
    got = _engine_grads(head, variant, noisy, cond, T3, d_eps)
    ref = restatement_grads(variant, sd, noisy, cond, T3, d_eps)
    env = kink_envelope(variant, sd, noisy, cond, T3, d_eps, ref, BAND)
    _check(f"{variant} {hw[0]}x{hw[1]}", got, ref, env)
    rows = got["model.time_embedding.weight"].abs().sum(1).nonzero().flatten().tolist()
    assert rows == sorted(set(T3))


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_gradients_vs_reference_golden(case):
    golden = np.load(GOLDEN, allow_pickle=False)
    variant, sd, noisy, cond, t, d_eps = case_inputs(case)
    head = make_head(variant, sd, DEV)
    got = _engine_grads(head, variant, noisy, cond, t.tolist(), d_eps)
    m = golden_margins(golden, case, got)
    ref = restatement_grads(variant, sd, noisy, cond, t, d_eps)
    env = kink_envelope(variant, sd, noisy, cond, t, d_eps, ref, BAND)
    worst = max(m, key=m.get)
    print(f"\n[{case}] engine vs reference golden: worst {worst} {m[worst]:.2e}")
    for k in m:  # the fp32 reference carries its own kink flips: allow the envelope of both sides
        assert m[k] <= 2 * TOL + 2 * env[k], (k, m[k], env[k])


@pytest.mark.gpu
def test_function_forward_bit_identical_and_backward_deterministic():
    variant = "swin"
    sd = denoiser_state(variant)
    head = make_head(variant, sd, DEV)
    noisy, cond, d_eps = (x.to(DEV) for x in _inputs(variant, (19, 27)))
    t = torch.tensor(T3, device=DEV)
    with torch.no_grad():
        eps0 = head.model(noisy, t, cond, None, None, None)
    assert eps0.grad_fn is None
    x = noisy.clone().requires_grad_(True)
    c = cond.clone().requires_grad_(True)
    grads = []
    for _ in range(2):
        head.zero_grad(set_to_none=True)
        eps = head.model(x, t, c, None, None, None)
        assert eps.grad_fn is not None
        assert torch.equal(eps, eps0)
        x.grad = c.grad = None
        (eps * d_eps).sum().backward()
        grads.append([x.grad.clone(), c.grad.clone()] + [p.grad.clone() for p in head.model.parameters()])
    for a, b in zip(*grads):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_chain_rule_through_a_torch_conv():
    variant = "swin"
    sd = denoiser_state(variant)
    head = make_head(variant, sd, DEV)
    g = torch.Generator().manual_seed(11)
    feat = torch.randn(3, 8, 10, 14, generator=g)
    noisy = torch.randn(3, 16, 19, 27, generator=g)
    noise = torch.randn(3, 16, 19, 27, generator=g)
    w0 = torch.randn(256, 8, 3, 3, generator=g) * 0.2
    t = torch.tensor(T3)
    conv = torch.nn.Conv2d(8, 256, 3, padding=1, bias=False).to(DEV)
    with torch.no_grad():
        conv.weight.copy_(w0)
    with exact_fp32():
        cond = torch.relu(conv(feat.to(DEV)))
        F.mse_loss(head.model(noisy.to(DEV), t.to(DEV), cond, None, None, None), noise.to(DEV)).backward()
    w = w0.double().requires_grad_(True)
    p = {k: v.double() for k, v in sd.items()}
    c = torch.relu(F.conv2d(feat.double(), w, padding=1))
    F.mse_loss(restate.denoiser(p, noisy.double(), t, c, variant, prefix="model."), noise.double()).backward()
    err = float((conv.weight.grad.double().cpu() - w.grad).abs().max() / w.grad.abs().max())
    print(f"\n[chain rule] torch conv weight grad through the engine vs fp64: {err:.2e}")
    assert err <= 1e-3


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["swin", "res"])
def test_sgd_training_loop_tracks_fp64(variant):
    sd = denoiser_state(variant)
    head = make_head(variant, sd, DEV)
    g = torch.Generator().manual_seed(3)
    h, w = 19, 27
    ch, cw = ((h + 1) // 2, (w + 1) // 2) if variant == "swin" else (h, w)
    latent = torch.randn(2, 16, h, w, generator=g)
    noise = torch.randn(2, 16, h, w, generator=g)
    cond = torch.randn(2, 256, ch, cw, generator=g).abs()
    t = torch.tensor([600, 31])
    noisy = head.scheduler.add_noise(latent, noise, t)  # the `_ddim_loss` recipe with fixed noise and t
    lr, steps = 0.1, 5
    opt = torch.optim.SGD(head.model.parameters(), lr=lr)
    ref = {k: v.double().clone().requires_grad_(True) for k, v in sd.items()}
    losses, ref_losses = [], []
    for _ in range(steps):
        opt.zero_grad()
        loss = F.mse_loss(head.model(noisy.to(DEV), t.to(DEV), cond.to(DEV), None, None, None), noise.to(DEV))
        loss.backward()
        opt.step()  # in-place update: the next call re-packs the engine's weights ((data_ptr, _version) check)
        losses.append(float(loss.detach()))
        rl = F.mse_loss(restate.denoiser(ref, noisy.double(), t, cond.double(), variant, prefix="model."), noise.double())
        gr = torch.autograd.grad(rl, list(ref.values()))
        with torch.no_grad():
            for v, gv in zip(ref.values(), gr):
                v -= lr * gv
        ref_losses.append(float(rl))
    moved = {k: float((ref[k].detach() - sd[k].double()).abs().max()) for k in sd}
    got = dict(head.model.named_parameters())
    rel = {k: float((got[k[len("model."):]].detach().double().cpu() - ref[k].detach()).abs().max()) / max(moved[k], 1e-30)
           for k in sd}
    worst = max(rel, key=rel.get)
    print(f"\n[train {variant}] losses {losses} (fp64 {ref_losses}); worst parameter drift / movement: {worst} {rel[worst]:.2e}")
    assert losses[-1] < losses[0]
    assert abs(losses[0] - ref_losses[0]) <= 1e-4 * ref_losses[0]
    assert rel[worst] <= 1e-2


@pytest.mark.gpu
def test_argument_checks():
    lib = _cabi.load_library()
    noisy, cond, d_eps = (x.to(DEV) for x in _inputs("res", (8, 16)))
    sd = denoiser_state("res")
    head = make_head("res", sd, DEV)
    fwd = head._engine(3, (8, 16), (8, 16), DEV)
    bwd = head._engine(3, (8, 16), (8, 16), DEV, backward=True)
    assert int(lib.dd_workspace_bytes(bwd._h)) > int(lib.dd_workspace_bytes(fwd._h))

    def call(eng, t=T3, nbytes=None):
        ws = eng._workspace()
        n = ws.numel() - 1024 if nbytes is None else nbytes
        ptrs = (C.c_void_p * 17)()
        return lib.dd_denoiser_backward(eng._h, C.c_void_p(cond.data_ptr()), C.c_void_p(noisy.data_ptr()),
                                        (C.c_int64 * 3)(*t), C.c_void_p(d_eps.data_ptr()), None, None, ptrs,
                                        C.c_void_p(eng._aligned(ws)), n, C.c_void_p(eng._stream()))

    assert call(fwd) == 1 and b"DD_FLAG_BACKWARD" in lib.dd_last_error()
    assert call(bwd, nbytes=int(lib.dd_workspace_bytes(bwd._h)) - 1) == 1 and b"workspace" in lib.dd_last_error()
    assert call(bwd, t=(0, 1280, 3)) == 1
    assert call(bwd, t=(0, -1, 3)) == 1
    assert call(bwd) == 0
    torch.cuda.synchronize()
    with pytest.raises(_cabi.EngineError):
        DenoiseEngine.denoiser_backward(fwd, cond, noisy, T3, d_eps)
