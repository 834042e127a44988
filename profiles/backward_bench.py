"""Time dd_denoiser_backward on the GPU with CUDA events: ms per call at B = 4 on the C3 latent (176 x 608) and on a
training-crop latent (120 x 608), the tensor-core weight-gradient kernel's algorithmic TFLOP/s per 256-wide shape (from
a torch.profiler run), and torch fp32 autograd (TF32 off) of the restatement on the same card.  Prints one JSON line.

    python profiles/backward_bench.py [--iters 5]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from grad_helpers import denoiser_state, make_head  # noqa: E402
from oracle import restate  # noqa: E402

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


def run(hw, iters, torch_ref):
    B, (h, w) = 4, hw
    sd = denoiser_state("swin")
    head = make_head("swin", sd, DEV)
    g = torch.Generator(device=DEV).manual_seed(0)
    noisy = torch.randn(B, 16, h, w, device=DEV, generator=g)
    cond = torch.randn(B, 256, h // 2, w // 2, device=DEV, generator=g).abs()
    d_eps = torch.randn(B, 16, h, w, device=DEV, generator=g) * 1e-6
    t = [417, 31, 999, 417]
    eng = head._engine(B, (h, w), (h // 2, w // 2), DEV, backward=True)
    out = {"latent": [h, w], "batch": B,
           "native_backward_ms": events(lambda: eng.denoiser_backward(cond, noisy, t, d_eps), iters),
           "native_forward_ms": events(lambda: eng.denoiser_forward(cond, noisy, t), iters)}
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        eng.denoiser_backward(cond, noisy, t, d_eps)
        torch.cuda.synchronize()
    wg = [e.device_time_total / 1e3 for e in prof.key_averages() if "wgrad_simt_kernel" in e.key]
    ker = {e.key.split("(")[0][:60]: round(e.device_time_total / 1e3, 3) for e in prof.key_averages()}
    out["kernel_ms"] = dict(sorted(ker.items(), key=lambda kv: -kv[1])[:12])
    # wgrad_wgmma_kernel per 256-wide shape: <128, 128> = convA + convB, <128, 64> = noise_embedding.3, <64, 128> = pred.0
    shapes = {"<128, 128>": (256, 256), "<128, 64>": (256, 64), "<64, 128>": (64, 256)}
    per = {}
    for e in prof.key_averages():
        for tag, (co, ci) in shapes.items():
            if "wgrad_wgmma_kernel" + tag in e.key:
                ms = e.device_time_total / 1e3 / e.count
                per[f"{co}x{ci}"] = {"ms_per_launch": round(ms, 3),
                                     "algorithmic_tflops": round(2.0 * co * ci * 9 * B * h * w / 1e12 / (ms / 1e3), 1)}
    out["wgrad_wgmma"] = per
    out["wgrad_simt_ms"] = round(sum(wg), 3)
    if torch_ref:
        p = {k: v.to(DEV).requires_grad_(True) for k, v in sd.items()}
        x, c = noisy.clone().requires_grad_(True), cond.clone().requires_grad_(True)
        tt = torch.tensor(t, device=DEV)

        def ref():
            eps = restate.denoiser(p, x, tt, c, "swin", prefix="model.")
            torch.autograd.grad((eps * d_eps).sum(), [x, c] + list(p.values()))

        torch.backends.cuda.matmul.allow_tf32 = False
        torch.backends.cudnn.allow_tf32 = False
        out["torch_fp32_autograd_fwd_bwd_ms"] = events(ref, iters)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    a = ap.parse_args()
    res = {"card": card(), "runs": [run((176, 608), a.iters, True), run((120, 608), a.iters, True)]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
