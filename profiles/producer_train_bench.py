"""What training-mode BatchNorm in the condition producers (`head.producer_train_bn`, dd_set_producer_mode) costs, on
the GPU.  Per configuration, in one process after warm-up, alternating the two settings:
  (a) the graphed producer chain (dd_run_backbone + dd_build_condition) in DD_PRODUCER_EVAL vs DD_PRODUCER_TRAIN on
      the same engine (CUDA events);
  (b) one training iteration (forward with the native backbone, ddim_loss, backward, Adam.step) with
      `producer_train_bn` off vs on (host clock around device synchronisations).
Configurations: C3 (Swin-L + HAHI neck + FPN, B = 4, 352 x 1216; Swin-L has no BatchNorm, so TRAIN changes the neck and
FPN only) and C2 (res50-shaped native ResNet + FPN, B = 8, 228 x 304).  Prints the card's name, power limit and max SM
clock, and one JSON line.

    python profiles/producer_train_bench.py [--iters 5] [--configs C3,C2]"""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import dd_helpers as helpers  # noqa: E402
from oracle import configs, restate  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def event_ms(fn, reps):
    """Device milliseconds per fn() over reps back-to-back calls (CUDA events)."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def summary(xs):
    return {"median": round(statistics.median(xs), 4), "min": round(min(xs), 4), "max": round(max(xs), 4)}


def run_config(name, iters, dev):
    family, steps, B, H, W = configs.CONFIGS[name]
    base = helpers.build_mirror(family, steps).to(dev)
    sample = {k: v.to(dev) for k, v in restate.synthetic_sample(B, H, W, 3).items()}
    sample["noise"] = restate.synthetic_noise(B, H, W, 3).to(dev)
    # one model per setting: the running updates of one must not reach the other's packed weights
    models, opts = {}, {}
    for mode in (False, True):
        m = copy.deepcopy(base).train()
        m.depth_head.check_range = False
        m.depth_head.producer_train_bn = mode
        models[mode], opts[mode] = m, torch.optim.Adam(m.depth_head.model.parameters(), lr=1e-5)

    def iteration(mode):
        opts[mode].zero_grad()
        out = models[mode](sample)
        out["ddim_loss"].backward()
        opts[mode].step()

    for mode in (False, True, False, True):  # warm-up: every engine exists, every graph is captured
        iteration(mode)
    it = {False: [], True: []}
    for i in range(2 * iters):
        mode = i % 2 == 1
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        iteration(mode)
        torch.cuda.synchronize()
        it[mode].append((time.perf_counter() - t0) * 1e3)

    head = models[True].depth_head
    eng = next(e for k, e in head._engines.items() if k.image_hw is not None and k.producer_train)
    img = sample["rgb"].contiguous().float()

    def chain(train):
        eng.set_producer_mode(train)
        eng.run_backbone(img)
        eng.build_condition(None)

    for mode in (False, True):
        chain(mode)
    ch = {False: [], True: []}
    for i in range(2 * iters):
        mode = i % 2 == 1
        ch[mode].append(event_ms(lambda: chain(mode), 10))
    eng.set_producer_mode(False)
    res = {"config": name, "family": family, "batch": B, "image": [H, W],
           "bn_layers": len(eng.producer_bn_keys())}
    for mode, tag in ((False, "eval"), (True, "train")):
        res["chain_ms_" + tag] = summary(ch[mode])
        res["iteration_ms_producer_train_bn_" + ("on" if mode else "off")] = summary(it[mode])
    for m in models.values():
        m.depth_head.invalidate_engines()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5, help="timed rounds per setting")
    ap.add_argument("--configs", default="C3,C2")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("producer_train_bench.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda:0")
    out = {"card (name, power limit, max SM clock)": card(),
           "results": [run_config(c, a.iters, dev) for c in a.configs.split(",")]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
