"""TEST INFRASTRUCTURE ONLY — the REAL reference's stochastic DDIM sampler: `CNNDDIMPipiline.__call__` of the Res head
(ddim_depth_estimate_res.py:238-297), the Swin_ADDHAHI head (ddim_depth_estimate_res_swin_addHAHI.py:244-303) and the
Swin_ADDHAHIVis head (..._vis.py:246-306, which also returns `image_list`), unmodified, over each module's own
`ScheduledCNNRefine` with trained-like weights, at eta in {0.5, 1.0} and T in {3, 5}, on the CPU in fp32, seeded with
torch.manual_seed (the reference pipeline cannot take a `generator`: it reads a `self.device` it never sets).  The
decoder (`DeepDepthTransformWithUpsampling.inv_t`, eval BatchNorm) gives the logit.  Stored in
tests/golden/g_pipeline_eta.npz:
  draws                          [1 + 5, B, 16, h, w]: x_T, then z_1 .. z_5 — every case draws x_T, then one z per step,
                                 and the draws of one seed do not depend on the head or eta, so T = 3 uses the first 4
  <case>_latent / _logit         the final latent [B,16,h,w] and the decoder's pre-sigmoid logit [B,1,2h,2w]
  <case>_image_list              (Vis) the latent after every step [T,B,16,h,w]
with <case> = <head>_T<T>_eta<eta*10>.  Weights and the condition map are regenerated from seeds by `case_inputs`.
Run in the build container:
    python -m oracle.make_pipeline"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

OUT = os.path.join(ROOT, "tests", "golden", "g_pipeline_eta.npz")
SEED = 4242
BATCH, LATENT = 1, (8, 16)
# head -> (variant, condition (h, w), reference module, mirror head type)
HEADS = {
    "res18": ("res", (8, 16), "model.head.ddim_depth_estimate_res", "DDIMDepthEstimate_Res"),
    "swin": ("swin", (4, 8), "model.head.ddim_depth_estimate_res_swin_addHAHI", "DDIMDepthEstimate_Swin_ADDHAHI"),
    "swin_vis": ("swin", (4, 8), "model.head.ddim_depth_estimate_res_swin_addHAHI_vis",
                 "DDIMDepthEstimate_Swin_ADDHAHIVis"),
}
ETAS = (0.5, 1.0)
STEPS = (3, 5)


def case_name(head, T, eta):
    return f"{head}_T{T}_eta{int(round(eta * 10))}"


def case_inputs(head):
    """(variant, state_dict with keys `model.*` / `depth_transform.*`, cond [B,256,hc,wc]) of a head, fp32 CPU."""
    from oracle.make_loop_grads import loop_state
    variant, (hc, wc), _, _ = HEADS[head]
    g = torch.Generator().manual_seed(2026)
    cond = torch.randn(BATCH, 256, hc, wc, generator=g).abs()  # the FPN's condition map is post-ReLU
    return variant, loop_state(variant), cond


class _RecordRandn:
    """Pass every torch.randn through, keeping what it drew."""

    def __enter__(self):
        self.real, self.draws = torch.randn, []

        def rec(*a, **k):
            out = self.real(*a, **k)
            self.draws.append(out.detach().clone())
            return out

        torch.randn = rec
        return self

    def __exit__(self, *exc):
        torch.randn = self.real


def reference_case(head, T, eta):
    import importlib
    from oracle import ref_import
    mods = ref_import.reference_modules()
    variant, sd, cond = case_inputs(head)
    mod = importlib.import_module(HEADS[head][2])
    model = mod.ScheduledCNNRefine(256, 16)
    model.load_state_dict({k[len("model."):]: v for k, v in sd.items() if k.startswith("model.")}, strict=True)
    model.eval()
    codec = mods.depth_transform.DeepDepthTransformWithUpsampling(16, 1e-6)
    codec.load_state_dict({k[len("depth_transform."):]: v for k, v in sd.items() if k.startswith("depth_transform.")},
                          strict=False)
    codec.eval()
    pipe = mod.CNNDDIMPipiline(model, mods.scheduling_ddim.DDIMScheduler(num_train_timesteps=1000, clip_sample=False))
    torch.manual_seed(SEED)
    with torch.no_grad(), _RecordRandn() as rec:
        out = pipe(batch_size=BATCH, device=torch.device("cpu"), dtype=torch.float32, shape=(16, *LATENT),
                   input_args=(cond, None, None, None), eta=eta, num_inference_steps=T, return_dict=False)
    draws = torch.stack(rec.draws)
    assert draws.shape[0] == T + 1, draws.shape
    with torch.no_grad():  # the pre-sigmoid output of conv_inv_transform (inv_t, depth_transform.py:33-35)
        logit = codec.conv_inv_transform[:4](out[0])
    return draws, out[0], logit, (torch.stack(out[1]) if len(out) > 1 else None)


def main():
    arrays = {}
    for head in HEADS:
        for T in STEPS:
            for eta in ETAS:
                draws, latent, logit, image_list = reference_case(head, T, eta)
                if "draws" not in arrays or arrays["draws"].shape[0] < draws.shape[0]:
                    prev = arrays.get("draws")
                    if prev is not None:
                        assert np.array_equal(prev, draws[:prev.shape[0]].numpy())
                    arrays["draws"] = draws.numpy()
                else:
                    assert np.array_equal(arrays["draws"][:T + 1], draws.numpy())
                name = case_name(head, T, eta)
                arrays[name + "_latent"] = latent.numpy()
                arrays[name + "_logit"] = logit.numpy()
                if image_list is not None:
                    arrays[name + "_image_list"] = image_list.numpy()
                print(f"{name}: max|latent| {latent.abs().max():.4g}  max|logit| {logit.abs().max():.4g}")
    np.savez_compressed(OUT, **arrays)
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1024:.0f} kB)")


if __name__ == "__main__":
    main()
