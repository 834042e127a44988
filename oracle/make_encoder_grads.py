"""TEST INFRASTRUCTURE ONLY — gradients of the REAL reference's depth encoder `DeepDepthTransformWithUpsampling.t`
(ops/depth_transform.py:15-19,29-31) by autograd, on CPU in the reference's own fp32:
  enc/<mode>/<case>/  gradients of sum(t(depth) * d_latent) with respect to the encoder's six parameters, the codec in
                      eval (running statistics) or `.train()` (batch statistics) mode; cases B = 3 at 37 x 53 (latent
                      19 x 27, odd: a stride-2 tail) and B = 1 at 2 x 3;
  loss_gt/            one reference Res head `ddim_loss_gt` (ddim_depth_estimate_res.py:219-235) on gt_map_t = t(gt)
                      with the codec in training mode: its noise and timesteps, the loss, and the encoder, denoiser and
                      cond gradients.
Stored in tests/golden/g_encoder_grads.npz.  Run in the build container:
    python -m oracle.make_encoder_grads"""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import make_loop_grads as mlg  # noqa: E402
from oracle.make_codec_train import codec_state  # noqa: E402
from oracle.make_denoiser_grads import SAMPLES, checksum, sample_index  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "g_encoder_grads.npz")
CASES = {"b3_37x53": (3, 37, 53), "b1_2x3": (1, 2, 3)}
LOSS_GT = (2, 19, 27)  # B, depth map (latent 10 x 14); condition map at the latent's size (Res)
LOSS_SEED = 1234


def case_inputs(name):
    """(depth [B,1,H,W], d_latent [B,16,ceil(H/2),ceil(W/2)]), fp32 CPU."""
    B, H, W = CASES[name]
    g = torch.Generator().manual_seed(808 + H)
    depth = torch.rand(B, 1, H, W, generator=g) * 2 + 0.1
    d_latent = torch.randn(B, 16, (H + 1) // 2, (W + 1) // 2, generator=g)
    return depth, d_latent


def loss_gt_inputs():
    """(gt depth [B,1,H,W], cond [B,256,h,w]), fp32 CPU."""
    B, H, W = LOSS_GT
    g = torch.Generator().manual_seed(99)
    gt = torch.rand(B, 1, H, W, generator=g) * 2 + 0.1
    cond = torch.randn(B, 256, (H + 1) // 2, (W + 1) // 2, generator=g).abs()
    return gt, cond


def _reference_codec(train):
    from oracle import ref_import
    codec = ref_import.reference_modules().depth_transform.DeepDepthTransformWithUpsampling(16, 1e-6)
    codec.load_state_dict(codec_state(), strict=False)
    return codec.train(train)


def _store(out, prefix, grads):
    for k, gr in grads.items():
        flat = gr.detach().reshape(-1)
        out[f"{prefix}/{k}/absmax"] = np.float64(flat.abs().max())
        if flat.numel() <= SAMPLES:
            out[f"{prefix}/{k}/values"] = flat.numpy()
        else:
            idx = sample_index(flat.numel())
            out[f"{prefix}/{k}/index"] = idx
            out[f"{prefix}/{k}/values"] = flat[torch.from_numpy(idx)].numpy()


def encoder_arrays():
    out = {"weight_checksum": np.float64(checksum(*codec_state().values()))}
    for mode in ("eval", "train"):
        for name in CASES:
            depth, d_latent = case_inputs(name)
            codec = _reference_codec(mode == "train")
            (codec.t(depth) * d_latent).sum().backward()
            _store(out, f"enc/{mode}/{name}", {"depth_transform.conv_transform." + k: p.grad
                                               for k, p in codec.conv_transform.named_parameters()})
            out[f"enc/{mode}/{name}/input_checksum"] = np.float64(checksum(depth, d_latent))
    return out


def loss_gt_arrays():
    from oracle import ref_import
    mods = ref_import.reference_modules()
    sd = mlg.loop_state("res")
    model = mods.head_res.ScheduledCNNRefine(256, 16)
    model.load_state_dict({k[len("model."):]: v for k, v in sd.items() if k.startswith("model.")}, strict=True)
    codec = _reference_codec(True)
    gt, cond = loss_gt_inputs()
    cond = cond.clone().requires_grad_(True)
    gt_map_t = codec.t(gt)
    # the reference method itself, on a stand-in holding the two attributes it reads
    head = types.SimpleNamespace(model=model,
                                 scheduler=mods.scheduling_ddim.DDIMScheduler(num_train_timesteps=1000, clip_sample=False))
    torch.manual_seed(LOSS_SEED)
    noise = torch.randn(gt_map_t.shape)
    t = torch.randint(0, 1000, (gt.shape[0],)).long()
    torch.manual_seed(LOSS_SEED)
    loss = mods.head_res.DDIMDepthEstimate_Res.ddim_loss_gt(head, gt_map_t, (cond, None, None, None), gt_map_t, 1.0)
    loss.backward()
    grads = {"d_cond": cond.grad}
    grads.update({"model." + k: p.grad for k, p in model.named_parameters()})
    grads.update({"depth_transform.conv_transform." + k: p.grad for k, p in codec.conv_transform.named_parameters()})
    out = {"loss_gt/noise": noise.numpy(), "loss_gt/t": t.numpy(), "loss_gt/loss": np.float64(loss.item()),
           "loss_gt/weight_checksum": np.float64(checksum(*sd.values())),
           "loss_gt/input_checksum": np.float64(checksum(gt, cond.detach()))}
    _store(out, "loss_gt", grads)
    return out


def main():
    torch.set_num_threads(os.cpu_count() or 8)
    arrays = encoder_arrays()
    arrays.update(loss_gt_arrays())
    np.savez_compressed(OUT, **arrays)
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1e3:.0f} kB)")


if __name__ == "__main__":
    main()
