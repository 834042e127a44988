"""`head.pipeline` (the reference's `CNNDDIMPipiline`) on the engine: the stochastic DDIM step (eta > 0) inside the fused
loop against the real reference's golden and the fp64 restatement, its random draws, its refusals, and the eta = 0
path against the head's own forward."""
import contextlib
import os

import numpy as np
import pytest
import torch

from diffusiondepth_b200._cabi import EngineError
from diffusiondepth_b200.engine import DenoiseEngine
from diffusiondepth_b200.model.registry import HEADS
from oracle import restate, restate_eta
from oracle.make_loop_grads import loop_state
from oracle.make_pipeline import BATCH, ETAS, HEADS as CASE_HEADS, LATENT, STEPS, case_inputs, case_name

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "g_pipeline_eta.npz")


def _head(kind, sd, steps):
    torch.manual_seed(0)
    head = HEADS.build(dict(type=kind, in_channels=[64, 128, 256, 512], inference_steps=steps, num_train_timesteps=1000,
                            depth_feature_dim=16, loss_cfgs=[], init_cfg=None)).eval()
    head.model.load_state_dict({k[len("model."):]: v for k, v in sd.items() if k.startswith("model.")})
    head.depth_transform.load_state_dict({k[len("depth_transform."):]: v for k, v in sd.items()
                                          if k.startswith("depth_transform.")}, strict=False)
    return head.to(DEV)


@contextlib.contextmanager
def _feed_randn(draws):
    """torch.randn hands out `draws` in order (on the requested device), as the injected draws of the reference."""
    real, queue = torch.randn, list(draws)

    def fake(*a, **k):
        t = queue.pop(0)
        return t.to(device=k.get("device") or "cpu", dtype=k.get("dtype") or t.dtype)

    torch.randn = fake
    try:
        yield queue
    finally:
        torch.randn = real


def _call(head, cond, shape, eta, T, **kw):
    return head.pipeline(batch_size=cond.shape[0], device=DEV, dtype=torch.float32, shape=shape,
                         input_args=(cond, None, None, None), eta=eta, num_inference_steps=T, return_dict=False, **kw)


@pytest.mark.parametrize("head_name", list(CASE_HEADS))
@pytest.mark.parametrize("T", STEPS)
@pytest.mark.parametrize("eta", ETAS)
def test_pipeline_matches_reference_golden(head_name, T, eta):
    g = np.load(GOLDEN)
    variant, sd, cond = case_inputs(head_name)
    head = _head(CASE_HEADS[head_name][3], sd, T)
    draws = torch.from_numpy(g["draws"])[:T + 1]
    with torch.no_grad(), _feed_randn(draws) as left:
        out = _call(head, cond.to(DEV), (16, *LATENT), eta, T)
    assert not left
    name = case_name(head_name, T, eta)
    latent = out[0]
    eng = head._any_engine(BATCH, LATENT, cond.shape[-2:], DEV)
    _, logit = eng.decode(latent.contiguous(), want_logits=True)
    d_logit = (logit.cpu() - torch.from_numpy(g[name + "_logit"])).abs().max().item()
    ref_lat = torch.from_numpy(g[name + "_latent"])
    d_lat = (latent.cpu() - ref_lat).abs().max().item()
    print(f"{name}: logit max|dz| {d_logit:.3g}; latent max|d| {d_lat:.3g} of max {ref_lat.abs().max():.3g}")
    assert d_logit < 1e-3
    assert d_lat < 1e-3 * ref_lat.abs().max().item()
    if name + "_image_list" in g:
        ref_list = torch.from_numpy(g[name + "_image_list"])
        assert len(out[1]) == T and torch.equal(out[1][-1], latent)
        for i, (a, b) in enumerate(zip(out[1], ref_list)):
            d = (a.cpu() - b).abs().max().item()
            print(f"  image_list[{i}]: max|d| {d:.3g} of max {b.abs().max():.3g}")
            assert d < 1e-3 * b.abs().max().item()
        # the Vis heads' graphed step-decode loop runs the same stochastic steps
        steps_eng = head._engine(BATCH, LATENT, cond.shape[-2:], DEV, steps=T, eta=eta)
        z = draws[1:].to(DEV).contiguous()
        _, lat_steps, _ = steps_eng.denoise_decode_steps(cond.to(DEV), draws[0].to(DEV).contiguous(), want_latent=True,
                                                         variance_noise=z)
        assert torch.equal(lat_steps, latent)


def _swin_feats(B, hw, seed=3):
    g = torch.Generator().manual_seed(seed)
    fp = [torch.randn(B, c, -(-hw[0] // s), -(-hw[1] // s), generator=g).to(DEV) for c, s in
          ((192, 4), (384, 8), (768, 16), (1536, 32))]
    gt = (torch.rand(B, 1, *hw, generator=g) * 80).to(DEV)
    return fp, gt


def test_eta0_pipeline_is_bit_identical_to_forward():
    T = 5
    head = _head("DDIMDepthEstimate_Swin_ADDHAHI", loop_state("swin"), T)
    fp, gt = _swin_feats(2, (32, 64))
    x_T = torch.randn(2, 16, 16, 32, generator=torch.Generator().manual_seed(5)).to(DEV)
    head.capture_cond = True
    with torch.no_grad():
        head(fp, gt, gt > 0, gt_depth_map=gt, noise=x_T)
        with _feed_randn([x_T]):
            latent, = _call(head, head.last_cond, (16, 16, 32), 0.0, T)
    assert torch.equal(latent, head.last_latent)


def test_config3_every_pixel_against_fp64():
    """BASELINE config 3 geometry (B = 4, 352 x 1216 -> latent 176 x 608, condition 88 x 304), T = 20, eta = 1."""
    B, T, (h, w), (hc, wc) = 4, 20, (176, 608), (88, 304)
    sd = loop_state("swin")
    head = _head("DDIMDepthEstimate_Swin_ADDHAHI", sd, T)
    g = torch.Generator().manual_seed(11)
    cond = torch.randn(B, 256, hc, wc, generator=g).abs().to(DEV)
    draws = [torch.randn(B, 16, h, w, generator=g) for _ in range(T + 1)]
    with torch.no_grad(), _feed_randn(draws):
        latent, = _call(head, cond, (16, h, w), 1.0, T)
    sd64 = {"depth_head." + k: v.to(DEV, torch.float64) for k, v in sd.items()}
    with torch.no_grad():
        ref, _ = restate_eta.ddim_loop(sd64, cond.double(), draws[0].to(DEV).double(), T, "swin", 1.0,
                                       torch.stack(draws[1:]).to(DEV).double())
        z_ref = restate.decode_logits(sd64, ref)
        _, z = head._any_engine(B, (h, w), (hc, wc), DEV).decode(latent.contiguous(), want_logits=True)
    d_lat = (latent.double() - ref).abs().max().item()
    d_z = (z.double() - z_ref).abs().max().item()
    print(f"config 3, eta 1: latent max|d| {d_lat:.3g} of max {ref.abs().max().item():.3g}; logit max|dz| {d_z:.3g}")
    assert d_z < 1e-3
    assert d_lat < 1e-3 * ref.abs().max().item()


def test_rng_order_and_generator():
    """x_T, then one draw per step (T of them), nothing in between: the pipeline under a seed equals the engine fed
    the same draws made by hand; a generator is used for every draw."""
    T, shape = 4, (16, 16, 32)
    head = _head("DDIMDepthEstimate_Swin_ADDHAHI", loop_state("swin"), T)
    cond = torch.rand(2, 256, 8, 16, generator=torch.Generator().manual_seed(1)).to(DEV)
    with torch.no_grad():
        torch.manual_seed(123)
        a, = _call(head, cond, shape, 1.0, T)
        torch.manual_seed(123)
        x_T = torch.randn((2, *shape), device=DEV)
        z = torch.stack([torch.randn((2, *shape), device=DEV) for _ in range(T)])
        eng = head._engine(2, shape[1:], (8, 16), DEV, steps=T, eta=1.0)
        _, b, _ = eng.denoise_decode(cond, x_T, want_latent=True, variance_noise=z)
        assert torch.equal(a, b)
        gen = torch.Generator(device=DEV).manual_seed(77)
        c, = _call(head, cond, shape, 1.0, T, generator=gen)
        gen.manual_seed(77)
        x_T = torch.randn((2, *shape), generator=gen, device=DEV)
        z = torch.stack([torch.randn((2, *shape), generator=gen, device=DEV) for _ in range(T)])
        _, d, _ = eng.denoise_decode(cond, x_T, want_latent=True, variance_noise=z)
        assert torch.equal(c, d) and not torch.equal(a, c)
        # eta = 0 draws x_T only
        torch.manual_seed(5)
        _call(head, cond, shape, 0.0, T)
        after = torch.randn(1, device=DEV)
        torch.manual_seed(5)
        torch.randn((2, *shape), device=DEV)
        assert torch.equal(after, torch.randn(1, device=DEV))


def test_refusals():
    T, (h, w) = 3, (16, 32)
    sd = loop_state("swin")
    head = _head("DDIMDepthEstimate_Swin_ADDHAHI", sd, T)
    ts, cx, ce, sg = head.scheduler.fused_coefficients(T, eta=1.0)
    # the loop backward does not differentiate a stochastic sample
    lb = DenoiseEngine("swin", 1, (h, w), (8, 16), T, DEV, loop_backward=True)
    with pytest.raises(EngineError, match="DD_ERR_UNSUPPORTED"):
        lb.set_schedule(ts, cx, ce, sg)
    lb.close()
    # a stochastic schedule without its noise
    eng = head._engine(1, (h, w), (8, 16), DEV, steps=T, eta=1.0)
    cond = torch.rand(1, 256, 8, 16, device=DEV)
    x = torch.randn(1, 16, h, w, device=DEV)
    with pytest.raises(EngineError, match="DD_ERR_INVALID"):
        eng.denoise_decode(cond, x)
    with pytest.raises(EngineError, match="DD_ERR_INVALID"):
        eng.set_schedule(ts, cx, ce, [-1.0] * T)
    # the noise is borrowed for one call: the next call without it is refused again
    eng.denoise_decode(cond, x, variance_noise=torch.randn(T, 1, 16, h, w, device=DEV))
    with pytest.raises(EngineError, match="DD_ERR_INVALID"):
        eng.denoise_decode(cond, x)
    # under autograd
    with pytest.raises(EngineError, match="eta"):
        _call(head, cond, (16, h, w), 0.5, T)
    head.grad_through_loop = True
    with pytest.raises(EngineError, match="grad_through_loop"):
        _call(head, cond, (16, h, w), 0.0, T)
    head.grad_through_loop = False
    out, = _call(head, cond, (16, h, w), 0.0, T)
    assert not out.requires_grad


def test_switching_eta_between_calls():
    T, shape = 5, (16, 16, 32)
    head = _head("DDIMDepthEstimate_Swin_ADDHAHI", loop_state("swin"), T)
    cond = torch.rand(2, 256, 8, 16, generator=torch.Generator().manual_seed(2)).to(DEV)

    def run(eta):
        torch.manual_seed(9)
        with torch.no_grad():
            return _call(head, cond, shape, eta, T)[0]

    first = {eta: run(eta) for eta in (0.0, 1.0)}
    counts = {eta: head._engine(2, shape[1:], (8, 16), DEV, steps=T, eta=eta).graph_capture_count()
              for eta in (0.0, 1.0)}
    for eta in (0.0, 1.0, 0.0, 1.0, 0.5):
        got = run(eta)
        if eta in first:
            assert torch.equal(got, first[eta])
        else:
            assert not torch.equal(got, first[1.0])
    after = {eta: head._engine(2, shape[1:], (8, 16), DEV, steps=T, eta=eta).graph_capture_count()
             for eta in (0.0, 1.0)}
    print(f"graph captures per engine before / after alternating eta: {counts} / {after}")
    assert after == counts  # each eta keeps its own engine and graph
    # one engine switched between schedules captures its loop graph again
    eng = head._engine(2, shape[1:], (8, 16), DEV, steps=T, eta=1.0)
    x = torch.randn(2, *shape, device=DEV)
    z = torch.randn(T, 2, *shape, device=DEV)
    n0 = eng.graph_capture_count()
    eng.set_schedule(*head.scheduler.fused_coefficients(T))
    _, a, _ = eng.denoise_decode(cond, x, want_latent=True)
    eng.set_schedule(*head.scheduler.fused_coefficients(T, eta=1.0))
    _, b, _ = eng.denoise_decode(cond, x, want_latent=True, variance_noise=z)
    print(f"one engine switched eta 1 -> 0 -> 1: {eng.graph_capture_count() - n0} graph captures")
    assert eng.graph_capture_count() - n0 == 2
    assert not torch.equal(a, b)
