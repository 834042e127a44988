"""What training-mode BatchNorm in the depth codec (`head.codec_train_bn`, dd_set_codec_mode) costs, on the GPU: at
BASELINE config 3's geometry (B = 4, 352 x 1216, Swin-L native backbone, T = 20), alternating the two modes in one
process after warm-up, time
  (a) one decode (dd_decode) with the running-statistics fold vs batch statistics (CUDA events),
  (b) one dd_denoise_backward (the loop backward, decoder included) in both modes (CUDA events),
  (c) one training iteration (forward, L1 + L2 + ddim_loss, backward through the loop, Adam.step) with
      `codec_train_bn` off vs on (host clock around device synchronisations).
Prints the card's name, power limit and max SM clock, and one JSON line.

    python profiles/codec_train_bench.py [--iters 4] [--family swinl --batch 4 --height 352 --width 1216 --steps 20]"""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=4, help="timed rounds per setting")
    ap.add_argument("--family", default="swinl")
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--height", type=int, default=352)
    ap.add_argument("--width", type=int, default=1216)
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("codec_train_bench.py measures on the GPU; no CUDA device found")
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

    def iteration():
        opt.zero_grad()
        out = model(sample)
        gt = sample["gt"]
        loss = F.l1_loss(out["pred"], gt) + F.mse_loss(out["pred"], gt) + out["ddim_loss"]
        loss.backward()
        opt.step()

    for mode in (False, True, False, True):  # warm-up: every engine exists and both modes' graphs are captured
        head.codec_train_bn = mode
        iteration()
    it = {False: [], True: []}
    for i in range(2 * a.iters):
        mode = i % 2 == 1
        head.codec_train_bn = mode
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        iteration()
        torch.cuda.synchronize()
        it[mode].append((time.perf_counter() - t0) * 1e3)

    # (a) and (b) on the head's engines, at its own latent, condition map and noise
    fwd = next(e for k, e in head._engines.items() if k.image_hw is not None)
    loop = next(e for k, e in head._engines.items() if k.loop_backward)
    latent, cond = head.last_latent.detach().contiguous(), head.last_cond.detach().contiguous()
    noise = sample["noise"].contiguous()
    d_depth = torch.randn(a.batch, 1, 2 * latent.shape[2], 2 * latent.shape[3], device=dev) * 1e-6
    dec, bwd = {False: [], True: []}, {False: [], True: []}
    for mode in (False, True):
        fwd.set_codec_mode(mode)
        fwd.decode(latent)
        loop.set_codec_mode(mode)
        loop.denoise_backward(cond, noise, d_depth, None)
    for i in range(2 * a.iters):
        mode = i % 2 == 1
        fwd.set_codec_mode(mode)
        dec[mode].append(event_ms(lambda: fwd.decode(latent), 50))
        loop.set_codec_mode(mode)
        bwd[mode].append(event_ms(lambda: loop.denoise_backward(cond, noise, d_depth, None), 2))
    res = {"card (name, power limit, max SM clock)": card(), "family": a.family, "batch": a.batch,
           "image": [a.height, a.width], "steps": a.steps}
    for mode, name in ((False, "eval"), (True, "train")):
        res["decode_ms_" + name] = summary(dec[mode])
        res["denoise_backward_ms_" + name] = summary(bwd[mode])
        res["iteration_ms_codec_train_bn_" + ("on" if mode else "off")] = summary(it[mode])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
