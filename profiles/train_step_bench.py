"""What an optimizer step costs the engine, on the GPU: at BASELINE config 3's geometry (B = 4, 352 x 1216, Swin-L native
backbone, T = 20) time
  (a) `load_weights` of the whole model (dd_finalize_weights: what every iteration paid per engine before),
  (b) `update_weights` of the 27 trained tensors (21 denoiser + 6 decoder parameters; dd_update_weights),
  (c) one whole training iteration (forward, L1 + ddim_loss, backward through the loop, Adam.step) with
      `head.incremental_repack` off and on, alternating the two in one process after warm-up,
and count the CUDA graph captures per iteration of both.  (a) and (b) contain host synchronisations, so all three are
host-clock times around a device synchronise.  Prints the card's name, power limit and max SM clock, and one JSON line.

    python profiles/train_step_bench.py [--iters 4] [--family swinl --batch 4 --height 352 --width 1216 --steps 20]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import dd_helpers as helpers  # noqa: E402
from oracle import restate  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def wall_ms(fn, reps):
    """Host milliseconds of fn() between two device synchronisations: (median, min, max) over reps."""
    out = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
    return {"median": round(statistics.median(out), 3), "min": round(min(out), 3), "max": round(max(out), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=4, help="timed iterations per setting")
    ap.add_argument("--family", default="swinl")
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--height", type=int, default=352)
    ap.add_argument("--width", type=int, default=1216)
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("train_step_bench.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda:0")
    model = helpers.build_mirror(a.family, a.steps).to(dev)
    head = model.depth_head
    head.train()
    head.grad_through_loop = True
    head.check_range = False
    sample = {k: v.to(dev) for k, v in restate.synthetic_sample(a.batch, a.height, a.width, 3).items()}
    sample["noise"] = restate.synthetic_noise(a.batch, a.height, a.width, 3).to(dev)
    keys, params = head._loop_params()
    opt = torch.optim.Adam(params, lr=1e-5)

    def captures():
        return sum(e.graph_capture_count() for e in head._engines.values())

    def iteration():
        opt.zero_grad()
        out = model(sample)
        loss = F.l1_loss(out["pred"], sample["gt"]) + out["ddim_loss"]
        loss.backward()
        opt.step()

    for mode in (True, False, True):  # warm-up: both engines exist, every graph has been captured, both paths have run
        head.incremental_repack = mode
        iteration()
    times, caps = {True: [], False: []}, {True: [], False: []}
    for i in range(2 * a.iters):
        mode = i % 2 == 1
        head.incremental_repack = mode
        before = captures()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        iteration()
        torch.cuda.synchronize()
        times[mode].append((time.perf_counter() - t0) * 1e3)
        caps[mode].append(captures() - before)

    # (a) and (b) on the forward engine (native backbone + producers), from the tensors it was last packed with
    fwd_key = next(k for k in head._engines if k.image_hw is not None)
    eng, tensors = head._engines[fwd_key], head._packed[fwd_key][0]
    trained = {k: tensors[k] for k in keys}
    res = {"card (name, power limit, max SM clock)": card(), "family": a.family, "batch": a.batch,
           "image": [a.height, a.width], "steps": a.steps, "packed_tensors": len(tensors), "updated_tensors": len(trained),
           "load_weights_ms": wall_ms(lambda: eng.load_weights(tensors), 3),
           "update_weights_ms": wall_ms(lambda: eng.update_weights(trained), 5)}
    for mode, name in ((False, "full_repack"), (True, "incremental")):
        res["iteration_ms_" + name] = {"median": round(statistics.median(times[mode]), 2),
                                       "all": [round(t, 2) for t in times[mode]]}
        res["graph_captures_per_iteration_" + name] = caps[mode]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
