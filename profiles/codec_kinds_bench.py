"""Time a DDIMDepthEstimate_Swin_ADDHAHI forward (native HAHI neck + FPN, T = 20 DDIM steps, decoder) at BASELINE
config-3 geometry (B = 4, 352 x 1216 depth map, Swin-L pyramid at 1/4 .. 1/32) for each learned depth codec, the
default DeepDepthTransformWithUpsampling as the control, the kinds alternating round by round; then each codec's
decoder kernel alone (dd_bench_decoder) with CUDA events.  Prints the card and its power limit with the numbers.

    python profiles/codec_kinds_bench.py [--rounds 5] [--iters 20]
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from diffusiondepth_b200.model.registry import HEADS  # noqa: E402

NAMES = ["DeepDepthTransformWithUpsampling", "DeepDepthTransformWithUpsampling1x1",
         "DeepDepthTransformWithUpsamplingX4", "DeepDepthTransform"]
CH = [192, 384, 768, 1536]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    B, H, W = 4, 352, 1216
    g = torch.Generator().manual_seed(0)
    fp = [torch.randn(B, c, H // 4 >> i, W // 4 >> i, generator=g).abs().to(dev) for i, c in enumerate(CH)]
    gt = (torch.rand(B, 1, H, W, generator=g) * 80).to(dev)
    heads = []
    for n in NAMES:
        torch.manual_seed(0)
        h = HEADS.build(dict(type="DDIMDepthEstimate_Swin_ADDHAHI", in_channels=CH, inference_steps=20,
                             num_train_timesteps=1000, depth_feature_dim=16, loss_cfgs=[], init_cfg=None,
                             depth_transform_cfg=dict(type=n))).eval().to(dev)
        h.check_range = False
        heads.append(h)
    times = {n: [] for n in NAMES}
    with torch.no_grad():
        for h in heads:  # warm up: engine creation, pack, graph capture
            for _ in range(2):
                h(fp, None, None, gt_depth_map=gt)
        torch.cuda.synchronize()
        for _ in range(args.rounds):
            for n, h in zip(NAMES, heads):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(args.iters):
                    h(fp, None, None, gt_depth_map=gt)
                b.record()
                b.synchronize()
                times[n].append(a.elapsed_time(b) / args.iters)
    print(f"card: {card()}")
    print(f"Swin_ADDHAHI forward (neck + FPN + T=20 loop + decode + encode), B={B}, {H}x{W}, ms per forward, "
          f"median of {args.rounds} alternating rounds of {args.iters}:")
    base = sorted(times[NAMES[0]])[len(times[NAMES[0]]) // 2]
    for n, h in zip(NAMES, heads):
        med = sorted(times[n])[len(times[n]) // 2]
        lat = h.depth_transform.latent_hw((H, W))
        print(f"  {n:38s} latent {lat[0]}x{lat[1]:4d}  {med:8.2f} ms  (min {min(times[n]):.2f}, max {max(times[n]):.2f})"
              f"  x{base / med:.2f} vs default")
    print("decoder kernel alone (CUDA events around its launches, dd_bench_decoder), ms per launch:")
    with torch.no_grad():
        for n, h in zip(NAMES, heads):
            lat = h.depth_transform.latent_hw((H, W))
            eng = h._any_engine(B, lat, (H // 4, W // 4), dev)
            eng.decode(torch.randn(B, 16, *lat, device=dev))  # the latent the timed launches decode
            ms = eng.bench_decoder(args.iters * 5)
            print(f"  {n:38s} -> {eng.up * lat[0]}x{eng.up * lat[1]}  {ms:.3f} ms")


if __name__ == "__main__":
    main()
