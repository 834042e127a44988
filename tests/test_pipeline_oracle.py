"""The heads' stochastic DDIM sampler (`head.pipeline`, reference `CNNDDIMPipiline`) without a GPU: the fp32 restatement
against the golden of the real reference (oracle/make_pipeline.py), the collapsed step c_x x + c_eps eps + sigma z
against the scheduler's own `step` in fp64, the eta = 0 coefficients, and the pipeline's public surface on every head."""
import inspect
import os

import numpy as np
import pytest
import torch

from diffusiondepth_b200._cabi import EngineError
from diffusiondepth_b200.engine import ddim_coefficients
from diffusiondepth_b200.model.diffusers.schedulers.scheduling_ddim import DDIMScheduler
from diffusiondepth_b200.model.registry import HEADS
from oracle import ref_import, restate, restate_eta
from oracle.make_pipeline import BATCH, ETAS, HEADS as CASE_HEADS, LATENT, STEPS, case_inputs, case_name

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "g_pipeline_eta.npz")
DDIM_HEADS = ["DDIMDepthEstimate_Res", "DDIMDepthEstimate_ResVis", "DDIMDepthEstimate_Swin_ADD",
              "DDIMDepthEstimate_Swin_ADDHAHI", "DDIMDepthEstimate_Swin_ADDHAHIVis", "DDIMDepthEstimate_MPVIT_ADDHAHI"]


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


@pytest.mark.parametrize("head", list(CASE_HEADS))
@pytest.mark.parametrize("T", STEPS)
@pytest.mark.parametrize("eta", ETAS)
def test_restatement_matches_reference_pipeline(golden, head, T, eta):
    """oracle/restate_eta.py's loop with the reference's three-expression step at eta > 0, fed the golden's x_T and z_t,
    against the reference pipeline's latent, per-step latents (Vis) and decoded logit."""
    variant, sd, cond = case_inputs(head)
    draws = torch.from_numpy(golden["draws"])
    assert draws.shape == (1 + max(STEPS), BATCH, 16, *LATENT)
    name = case_name(head, T, eta)
    with torch.no_grad():
        latent, trace = restate_eta.ddim_loop({"depth_head." + k: v for k, v in sd.items()}, cond, draws[0], T, variant,
                                              eta, draws[1:T + 1])
        logit = restate.decode_logits(sd, latent, prefix="depth_transform.conv_inv_transform.")
    checks = [("latent", latent, golden[name + "_latent"]), ("logit", logit, golden[name + "_logit"])]
    if name + "_image_list" in golden:
        checks.append(("image_list", torch.stack(trace), golden[name + "_image_list"]))
    for what, got, want in checks:
        want = torch.from_numpy(want)
        err, scale = (got - want).abs().max().item(), want.abs().max().item()
        print(f"{name} {what}: max|d| {err:.3g} of max {scale:.3g}")
        assert err <= 1e-5 * max(1.0, scale), (what, err, scale)


def _reference_scheduler_cls():
    if not ref_import.available():
        pytest.skip("reference sources not available")
    return ref_import.reference_modules().scheduling_ddim.DDIMScheduler


@pytest.mark.parametrize("source", ["reference", "mirror"])
@pytest.mark.parametrize("T", [3, 20, 50])
@pytest.mark.parametrize("eta", [0.0, 0.5, 1.0])
def test_collapsed_step_equals_scheduler_step_fp64(source, T, eta):
    """x <- c_x x + c_eps eps + sigma z with the fp64 coefficients of `fused_coefficients(T, eta)` is the scheduler's
    `step(eps, t, x, eta, use_clipped_model_output=True, variance_noise=z)` for every step, in fp64."""
    cls = _reference_scheduler_cls() if source == "reference" else DDIMScheduler
    ref = cls(num_train_timesteps=1000, clip_sample=False)
    ref.alphas_cumprod = ref.alphas_cumprod.double()  # the same fp32 table, evaluated in fp64
    ref.final_alpha_cumprod = torch.as_tensor(ref.final_alpha_cumprod).double()
    ref.set_timesteps(T)
    ts, cx, ce, sg = DDIMScheduler(num_train_timesteps=1000, clip_sample=False).fused_coefficients(T, eta=eta)
    assert ts == [int(t) for t in ref.timesteps.tolist()]
    assert sg[-1] == 0.0 and (eta == 0) == all(s == 0 for s in sg)
    g = torch.Generator().manual_seed(T)
    worst = 0.0
    for i, t in enumerate(ts):
        x, eps, z = (torch.randn(2, 16, 5, 7, generator=g, dtype=torch.float64) for _ in range(3))
        want = ref.step(eps, t, x, eta=eta, use_clipped_model_output=True, variance_noise=z, return_dict=False)[0]
        got = cx[i] * x + ce[i] * eps + sg[i] * z
        err = (got - want).abs().max().item() / max(1.0, want.abs().max().item())
        worst = max(worst, err)
        assert err < 1e-12, (i, t, err)
    print(f"{source} T={T} eta={eta}: worst relative |d| {worst:.3g}")


@pytest.mark.parametrize("T", [1, 3, 5, 20, 50])
def test_fused_coefficients_eta0_unchanged(T):
    s = DDIMScheduler(num_train_timesteps=1000, clip_sample=False)
    base = s.fused_coefficients(T)
    assert len(base) == 3
    ts, cx, ce, sg = s.fused_coefficients(T, eta=0.0)
    assert (ts, cx, ce) == base and sg == [0.0] * T
    assert (ts, cx, ce) == ddim_coefficients(s.alphas_cumprod, T, 1000)
    with pytest.raises(ValueError):
        s.fused_coefficients(T, eta=-0.1)


def _build(kind, steps=3):
    torch.manual_seed(0)
    return HEADS.build(dict(type=kind, in_channels=[64, 128, 256, 512], inference_steps=steps, num_train_timesteps=1000,
                            depth_feature_dim=16, loss_cfgs=[], init_cfg=None)).eval()


def _reference_call_signature(vis):
    if not ref_import.available():
        return None
    import importlib
    ref_import.reference_modules()
    mod = importlib.import_module("model.head.ddim_depth_estimate_res_swin_addHAHI" + ("_vis" if vis else ""))
    return inspect.signature(mod.CNNDDIMPipiline.__call__)


@pytest.mark.parametrize("kind", DDIM_HEADS)
def test_every_head_has_the_reference_pipeline(kind):
    head = _build(kind)
    pipe = head.pipeline
    assert type(pipe).__name__ == "CNNDDIMPipiline"
    assert pipe.model is head.model and pipe.scheduler is head.scheduler
    assert pipe.image_list == kind.endswith("Vis")
    sig = inspect.signature(type(pipe).__call__)
    names = ["self", "batch_size", "device", "dtype", "shape", "input_args", "generator", "eta", "num_inference_steps",
             "return_dict", "kwargs"]
    assert list(sig.parameters) == names
    defaults = {k: p.default for k, p in sig.parameters.items() if p.default is not inspect.Parameter.empty}
    assert defaults == {"generator": None, "eta": 0.0, "num_inference_steps": 50, "return_dict": True}
    ref = _reference_call_signature(kind.endswith("Vis"))
    if ref is not None:
        assert list(ref.parameters) == names
        assert {k: p.default for k, p in ref.parameters.items() if p.default is not inspect.Parameter.empty} == defaults


def test_pipeline_has_no_cpu_path():
    head = _build("DDIMDepthEstimate_Swin_ADDHAHI")
    cond = torch.rand(1, 256, 4, 8)
    with pytest.raises(EngineError):
        head.pipeline(batch_size=1, device=torch.device("cpu"), dtype=torch.float32, shape=(16, 8, 16),
                      input_args=(cond, None, None, None), eta=1.0, num_inference_steps=3)
