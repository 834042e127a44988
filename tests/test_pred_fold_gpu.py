"""The Swin denoiser's composed convB -> pred.0 (one 5x5 conv + the ring correction, pred_fold.cuh) against the
two-conv chain (DD_FLAG_CHAIN_PRED) and the fp64 restatement: the operator and the T-step loop, over even, odd and tiny
latents.  The composed path must be as accurate as the chain, on the border ring and in the interior alike, and
bit-reproducible, with CUDA-graph replay equal to eager launches."""
import pytest
import torch

import diffusiondepth_b200 as dd
from oracle import restate

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
# (latent h, w), (cond h, w)
SIZES = [((18, 26), (9, 13)), ((24, 40), (12, 20)), ((35, 53), (18, 27)), ((3, 5), (2, 3))]


def _head(steps):
    from diffusiondepth_b200.model.registry import HEADS
    torch.manual_seed(11)
    return HEADS.build(dict(type="DDIMDepthEstimate_Swin_ADDHAHI", in_channels=[64, 128, 256, 512],
                            inference_steps=steps, num_train_timesteps=1000, depth_feature_dim=16, loss_cfgs=[],
                            init_cfg=None)).eval().to(DEV)


def _engine(head, B, hw, chw, T, **kw):
    eng = dd.DenoiseEngine("swin", B, hw, chw, T, DEV, check_range=True, fp8_corr=False, **kw)
    eng.load_weights(head._engine_tensors())
    eng.set_schedule(*head.scheduler.fused_coefficients(T))
    return eng


def _ring_mask(h, w, width=2):
    """Pixels within `width` of the border: pred.0's ring and the pred.3 outputs that read it."""
    m = torch.zeros(h, w, dtype=torch.bool)
    m[:width], m[-width:], m[:, :width], m[:, -width:] = True, True, True, True
    return m


def _errors(out, ref, mask):
    d = (out.double().cpu() - ref).abs()
    ring = d[..., mask].max().item()
    inner = d[..., ~mask].max().item() if (~mask).any() else 0.0
    return ring, inner


@pytest.mark.parametrize("hw,chw", SIZES)
def test_operator_fold_vs_chain(hw, chw):
    head = _head(5)
    sd = {"depth_head." + k: v.detach().cpu() for k, v in head.state_dict().items()}
    B, (h, w) = 2, hw
    g = torch.Generator().manual_seed(h * 100 + w)
    noisy = torch.randn(B, 16, h, w, generator=g) * 4
    cond = torch.randn(B, 256, *chw, generator=g)
    t = [950, 40]
    ref = restate.denoiser(sd, noisy.double(), torch.tensor(t), cond.double(), "swin")
    mask = _ring_mask(h, w)
    err = {}
    for name, chain in (("fold", False), ("chain", True)):
        eng = _engine(head, B, hw, chw, 5, chain_pred=chain, cuda_graph=False)
        eps = eng.denoiser_forward(cond.to(DEV), noisy.to(DEV), t)
        eps2 = eng.denoiser_forward(cond.to(DEV), noisy.to(DEV), t)
        eng.poll_status()
        assert torch.equal(eps, eps2), (name, "repeat call")
        err[name] = _errors(eps, ref, mask)
        eng.close()
    print(f"{hw}: ring / interior max |d eps| fold {err['fold']}, chain {err['chain']}")
    for i in range(2):
        assert err["fold"][i] <= 1.5 * err["chain"][i] + 1e-7, (hw, err)


@pytest.mark.parametrize("hw,chw", SIZES)
def test_loop_fold_vs_chain(hw, chw):
    T = 5
    head = _head(T)
    sd = {"depth_head." + k: v.detach().cpu() for k, v in head.state_dict().items()}
    B, (h, w) = 2, hw
    g = torch.Generator().manual_seed(5 + h)
    noise = torch.randn(B, 16, h, w, generator=g)
    cond = torch.randn(B, 256, *chw, generator=g).abs()
    lat_ref = restate.ddim_loop(sd, cond.double(), noise.double(), T, "swin")
    mask = _ring_mask(h, w)
    err, outs = {}, {}
    for name, kw in (("graph", dict(cuda_graph=True)), ("eager", dict(cuda_graph=False)),
                     ("chain", dict(cuda_graph=True, chain_pred=True))):
        eng = _engine(head, B, hw, chw, T, **kw)
        _, lat, z = eng.denoise_decode(cond.to(DEV), noise.to(DEV), want_latent=True, want_logits=True)
        _, lat2, z2 = eng.denoise_decode(cond.to(DEV), noise.to(DEV), want_latent=True, want_logits=True)
        assert torch.equal(lat, lat2) and torch.equal(z, z2), (name, "run-to-run determinism")
        assert eng.last_launch_count == 3 + T * 14 + 2
        err[name] = _errors(lat, lat_ref, mask)
        outs[name] = lat
        eng.close()
    print(f"{hw}: ring / interior max |d latent| fold {err['graph']}, chain {err['chain']}")
    assert torch.equal(outs["graph"], outs["eager"])
    for i in range(2):
        assert err["graph"][i] <= 1.5 * err["chain"][i] + 1e-7, (hw, err)


def test_bench_pred_fold_entry():
    head = _head(2)
    eng = _engine(head, 1, (24, 40), (12, 20), 2)
    assert eng.bench_pred_fold(2) > 0.0
    eng.close()
    chain = _engine(head, 1, (24, 40), (12, 20), 2, chain_pred=True)
    with pytest.raises(dd.EngineError):
        chain.bench_pred_fold(2)
    chain.close()
