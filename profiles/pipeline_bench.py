"""`head.pipeline` of a Swin_ADDHAHI head at BASELINE config 3 geometry (B = 4, 352 x 1216 -> latent 176 x 608, condition
88 x 304, T = 20): eta = 0 (the deterministic loop) against eta = 1 (the same loop plus sigma_t z_t, one 16-channel
fp32 read per pixel per step, 4 x 16 x 176 x 608 x 4 B = 27 MB), alternating in one process, timed with CUDA events
around the engine call (the random draws of the pipeline are made up front and not timed).  Prints the card, its power
limit, the per-round medians and their spread.

    python profiles/pipeline_bench.py [--rounds 7] [--iters 10]"""
import argparse
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name(0) + " (power limit not readable)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    from diffusiondepth_b200.model.registry import HEADS
    dev = torch.device("cuda:0")
    B, T, (h, w), (hc, wc) = 4, 20, (176, 608), (88, 304)
    torch.manual_seed(0)
    head = HEADS.build(dict(type="DDIMDepthEstimate_Swin_ADDHAHI", in_channels=[64, 128, 256, 512], inference_steps=T,
                            num_train_timesteps=1000, depth_feature_dim=16, loss_cfgs=[], init_cfg=None)).eval().to(dev)
    cond = torch.rand(B, 256, hc, wc, device=dev)
    x_T = torch.randn(B, 16, h, w, device=dev)
    z = torch.randn(T, B, 16, h, w, device=dev)
    engines = {}
    with torch.no_grad():
        for eta in (0.0, 1.0):  # each eta has its engine, schedule and CUDA graph (head.pipeline does the same)
            head.pipeline(batch_size=B, device=dev, dtype=torch.float32, shape=(16, h, w),
                          input_args=(cond, None, None, None), eta=eta, num_inference_steps=T)
            engines[eta] = head._engine(B, (h, w), (hc, wc), dev, steps=T, eta=eta)

    def run(eta):
        return engines[eta].denoise_decode(cond, x_T, variance_noise=z if eta > 0 else None)

    for eta in engines:  # warm-up
        run(eta)
    torch.cuda.synchronize()
    per = {0.0: [], 1.0: []}
    for _ in range(args.rounds):
        for eta in (0.0, 1.0):
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(args.iters):
                run(eta)
            t1.record()
            t1.synchronize()
            per[eta].append(t0.elapsed_time(t1) / args.iters)
    print(f"card: {card()}")
    print(f"Swin_ADDHAHI pipeline, B={B}, latent {h}x{w}, T={T}, {args.rounds} rounds x {args.iters} calls")
    for eta, ms in per.items():
        print(f"eta={eta}: median {statistics.median(ms):.3f} ms/call, min {min(ms):.3f}, max {max(ms):.3f}")
    over = [b / a - 1 for a, b in zip(per[0.0], per[1.0])]
    print(f"eta=1 over eta=0 per round: median {100 * statistics.median(over):+.2f}%, "
          f"range {100 * min(over):+.2f}% .. {100 * max(over):+.2f}%")
    print(f"added noise traffic per step: {B * 16 * h * w * 4 / 1e6:.1f} MB")


if __name__ == "__main__":
    main()
