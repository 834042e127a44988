"""Time one dd_denoise_backward (re-run of the T-step loop + T operator backwards + the decoder backward) on the GPU with
CUDA events, at B = 4, T = 20 on the C3 latent (176 x 608) and on a training-crop latent (120 x 608), next to the forward
dd_denoise_decode and torch fp32 autograd (TF32 off) of restate.ddim_loop + restate.decode with torch.utils.checkpoint
per step (so that the baseline fits in memory).  Prints the card's name and power limit and one JSON line.

    python profiles/loop_backward_bench.py [--iters 2] [--steps 20]"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.utils.checkpoint as ckpt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from loop_grad_helpers import make_loop_head  # noqa: E402
from oracle import restate  # noqa: E402
from oracle.make_loop_grads import loop_state  # noqa: E402

DEV = torch.device("cuda:0")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def events(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def run(hw, steps, iters, torch_ref):
    B, (h, w) = 4, hw
    sd = loop_state("swin")
    head = make_loop_head("swin", sd, steps, DEV)
    g = torch.Generator(device=DEV).manual_seed(0)
    noise = torch.randn(B, 16, h, w, device=DEV, generator=g)
    cond = torch.randn(B, 256, h // 2, w // 2, device=DEV, generator=g).abs()
    d_depth = torch.randn(B, 1, 2 * h, 2 * w, device=DEV, generator=g) / (B * 4 * h * w)
    d_latent = torch.randn(B, 16, h, w, device=DEV, generator=g) / (B * 16 * h * w)
    eng = head._engine(B, (h, w), (h // 2, w // 2), DEV, loop_backward=True)
    fwd = head._engine(B, (h, w), (h // 2, w // 2), DEV)
    out = {"latent": [h, w], "batch": B, "steps": steps,
           "native_loop_backward_ms": events(lambda: eng.denoise_backward(cond, noise, d_depth, d_latent), iters),
           "native_forward_ms": events(lambda: fwd.denoise_decode(cond, noise), iters),
           "native_operator_backward_ms": events(lambda: eng.denoiser_backward(cond, noise, 417, d_latent), iters)}
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        eng.denoise_backward(cond, noise, d_depth, d_latent)
        torch.cuda.synchronize()
    ker = {e.key.split("(")[0][:60]: round(e.device_time_total / 1e3, 3) for e in prof.key_averages()}
    out["kernel_ms"] = dict(sorted(ker.items(), key=lambda kv: -kv[1])[:10])
    out["decoder_backward_kernel_ms"] = round(sum(v for k, v in ker.items() if "dec_" in k), 3)
    if torch_ref:
        p = {"depth_head." + k: v.to(DEV).requires_grad_(k.startswith(("model.", "depth_transform.conv_inv")) and
                                                        "running" not in k) for k, v in sd.items()}
        params = [v for v in p.values() if v.requires_grad]
        x, c = noise.clone().requires_grad_(True), cond.clone().requires_grad_(True)
        acp = restate.ddim_tables().to(DEV)

        def ref():
            lat = x
            for t in restate.ddim_timesteps(steps):
                lat = ckpt.checkpoint(lambda z, t=t: restate.ddim_step(restate.denoiser(p, z, t, c, "swin"), t, z, acp,
                                                                       steps), lat, use_reentrant=False)
            loss = (restate.decode(p, lat) * d_depth).sum() + (lat * d_latent).sum()
            torch.autograd.grad(loss, [x, c] + params)

        torch.backends.cuda.matmul.allow_tf32 = False
        torch.backends.cudnn.allow_tf32 = False
        out["torch_fp32_autograd_checkpointed_ms"] = events(ref, 1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=2)
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    res = {"card": card(), "runs": [run((176, 608), a.steps, a.iters, True), run((120, 608), a.steps, a.iters, True)]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
