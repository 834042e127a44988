#!/usr/bin/env python
"""A/B timing of the DDIM loop's 3x3 convs (conv3x3_halo_kernel) between two builds of the engine library.

  python profiles/halo_ab.py --lib base=diffusiondepth_b200/libddengine_base.so --lib new=diffusiondepth_b200/libddengine.so
  python profiles/halo_ab.py --profile [--out DIR]     per-kernel breakdown of one C3 forward (torch.profiler)

Every loop conv shape is timed with DenoiseEngine.bench_conv (CUDA events around `--iters` back-to-back launches) on
the C3 latent grid: B = 4, 176 x 608.  Each library runs in its own process (the library is chosen when the package
loads it, through DD_ENGINE_LIB), and the libraries alternate for `--rounds` rounds so that clock and load drift hit
both alike.  Rates are algorithmic: 2 * pixels * COUT * 9 * CIN FLOPs per launch (the 3-pass split issues 3x that).
The Swin step runs convB + pred.0 as one composed 5x5 conv + its ring correction (DenoiseEngine.bench_pred_fold,
row "fold", rate counted as 2 * pixels * 64 * 25 * 256 FLOPs); 256->256 is convA, 256->64 the chain's pred.0.

The profile mode runs the full C3 forward (Swin-L, T = 20) once with the profiler on, without CUDA graphs so that
every kernel is recorded, and groups device time by kernel name.  It is a breakdown, not a timing: take times from
bench.py or from the A/B mode, which run with the profiler off.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(16, 64), (64, 256), (256, 256), (256, 64), (64, 16)]  # the loop's conv shapes (CIN, COUT)
B, LH, LW = 4, 176, 608  # C3 latent grid: 352 x 1216 at half resolution
PER_STEP = {(16, 64): 1, (64, 256): 1, (256, 256): 1, (256, 64): 0, (64, 16): 1}  # launches per DDIM step (+ fold)


def worker(iters, warmup):
    sys.path.insert(0, ROOT)
    import torch
    from diffusiondepth_b200 import lib_path
    from diffusiondepth_b200.model.registry import HEADS

    if not torch.cuda.is_available():
        raise SystemExit("halo_ab.py times kernels on an H100; there is no CPU path")
    dev = torch.device("cuda:0")
    torch.manual_seed(7240)
    head = HEADS.build(dict(type="DDIMDepthEstimate_Swin_ADDHAHI", in_channels=[64, 128, 256, 512],
                            inference_steps=20, num_train_timesteps=1000, depth_feature_dim=16, loss_cfgs=[],
                            init_cfg=None)).eval().to(dev)
    eng = head._engine(B, (LH, LW), (LH // 2, LW // 2), dev)
    res = {"lib": lib_path(), "gpu": torch.cuda.get_device_name(0), "ms": {}}
    for cin, cout in SHAPES:
        eng.bench_conv(cin, cout, warmup)
        res["ms"][f"{cin}->{cout}"] = eng.bench_conv(cin, cout, iters)
    eng.bench_pred_fold(warmup)
    res["ms"]["fold"] = eng.bench_pred_fold(iters)
    print(json.dumps(res), flush=True)


def tflops(cin, cout, ms):
    return 2.0 * B * LH * LW * cout * 9 * cin / (ms * 1e-3) / 1e12


def ab(libs, rounds, iters, warmup):
    runs = {name: [] for name, _ in libs}
    for _ in range(rounds):
        for name, path in libs:
            env = dict(os.environ, DD_ENGINE_LIB=os.path.abspath(path))
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", "--iters", str(iters),
                                  "--warmup", str(warmup)], env=env, cwd=ROOT, check=True, capture_output=True,
                                 text=True).stdout
            runs[name].append(json.loads(out.strip().splitlines()[-1]))
    print(f"{'shape':>9} " + " ".join(f"{n + ' ms (runs)':>28} {n + ' TF/s':>9}" for n, _ in libs))
    summary = {}
    for cin, cout in SHAPES:
        key = f"{cin}->{cout}"
        cells = []
        for name, _ in libs:
            ms = [r["ms"][key] for r in runs[name]]
            best = min(ms)
            summary.setdefault(key, {})[name] = {"ms": ms, "tflops_best": tflops(cin, cout, best)}
            cells.append(f"{' '.join(f'{m:.3f}' for m in ms):>28} {tflops(cin, cout, best):9.1f}")
        print(f"{key:>9} " + " ".join(cells))
    cells = []
    for name, _ in libs:
        ms = [r["ms"]["fold"] for r in runs[name]]
        summary.setdefault("fold", {})[name] = {"ms": ms, "tflops_best": tflops(256, 64, min(ms)) * 25 / 9}
        cells.append(f"{' '.join(f'{m:.3f}' for m in ms):>28} {tflops(256, 64, min(ms)) * 25 / 9:9.1f}")
    print(f"{'fold':>9} " + " ".join(cells))
    per_step = {name: min(summary["fold"][name]["ms"]) +
                sum(PER_STEP[(ci, co)] * min(summary[f"{ci}->{co}"][name]["ms"]) for ci, co in SHAPES)
                for name, _ in libs}
    print("loop conv ms per DDIM step (best runs): " + ", ".join(f"{n} {v:.2f}" for n, v in per_step.items()))
    print(json.dumps({"gpu": runs[libs[0][0]][0]["gpu"], "grid": [B, LH, LW], "iters": iters, "summary": summary,
                      "conv_ms_per_step": per_step}))


def profile(out_dir):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile
    import dd_helpers
    from oracle import configs, restate

    dev = torch.device("cuda:0")
    model = dd_helpers.build_mirror("swinl", 20).to(dev)
    model.depth_head.use_cuda_graph = False
    sample = {k: v.to(dev) for k, v in restate.synthetic_sample(B, 352, 1216, configs.SEED_INPUTS).items()}
    with torch.no_grad():
        for _ in range(2):
            model(sample)
        torch.cuda.synchronize()
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            model(sample)
            torch.cuda.synchronize()
    rows = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            r = rows.setdefault(e.name, [0, 0.0])
            r[0] += 1
            r[1] += e.device_time / 1e3  # ms
    total = sum(v[1] for v in rows.values())
    top = sorted(rows.items(), key=lambda kv: -kv[1][1])
    print(f"one C3 forward, profiler on, no CUDA graph: {total:.1f} ms of kernel time in {len(rows)} kernels")
    for name, (n, ms) in top[:25]:
        print(f"{ms:9.2f} ms {100 * ms / total:5.1f} % {n:5d}x  {name[:110]}")
    halo = sum(ms for name, (n, ms) in rows.items() if "conv3x3_halo_kernel" in name)
    print(f"conv3x3_halo_kernel, all shapes: {halo:.1f} ms = {100 * halo / total:.1f} % of kernel time")
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "kernels.json"), "w") as f:
            json.dump({"gpu": torch.cuda.get_device_name(0), "total_ms": total,
                       "kernels": [{"name": k, "count": n, "ms": ms} for k, (n, ms) in top]}, f, indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], metavar="NAME=PATH", help="library to time (repeatable)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None, help="profile mode: directory for kernels.json")
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args.iters, args.warmup)
    if args.profile:
        return profile(args.out)
    libs = [tuple(s.split("=", 1)) for s in args.lib] or [("current", os.path.join(ROOT, "diffusiondepth_b200",
                                                                                    "libddengine.so"))]
    ab(libs, args.rounds, args.iters, args.warmup)


if __name__ == "__main__":
    main()
