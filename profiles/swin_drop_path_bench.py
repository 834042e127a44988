"""Swin-L's stochastic depth on the engine at BASELINE config 3 (B = 4, 352 x 1216), on the GPU: the graphed backbone +
neck + FPN (dd_run_backbone, then dd_build_condition) of the Swin_ADDHAHI head in three settings, in one process after
warm-up, alternating the settings, CUDA events around back-to-back calls, medians over the rounds:
  eval        the backbone in eval: no stochastic depth, today's fused launches (G_BACKBONE);
  train       the backbone in `.train()` at drop_path_rate 0.1: fresh scales drawn on the device, dd_set_drop_path, the
              marked blocks' proj / ffn2 without their addend plus drop_path_add_kernel (G_BACKBONE_DROP);
  torch       the torch fallback at rate 0.1: the mirror Swin-L's forward in `.train()` in fp32 (TF32 off, as the model
              runs it), no grad, then the engine's neck + FPN on its features.
Also the HBM bytes the unfused adds add, from shapes: per marked branch, the branch written and read back (fp32) and x
read (the fused epilogue reads x too).  Prints the card's name, power limit and max SM clock, and one JSON line.

    python profiles/swin_drop_path_bench.py [--iters 5] [--reps 5]"""
import argparse
import copy
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "profiles"))

import dd_helpers as helpers  # noqa: E402
from diffusiondepth_b200.model._blocks import exact_fp32  # noqa: E402
from producer_train_bench import card, event_ms, summary  # noqa: E402

B, IMG, RATE = 4, (352, 1216), 0.1


def extra_bytes(head, bb):
    """HBM bytes the unfused adds move beyond the fused epilogues, per forward with every marked branch on."""
    sizes = head.swin_pyramid(IMG)
    masks = head.swin_drop_paths(bb)[0]
    total = 0
    for s, (h, w) in enumerate(sizes):
        tokens_c = B * h * w * (192 << s)
        total += bin(masks[s]).count("1") * 2 * 2 * tokens_c * 4  # 2 branches x (branch written + read back) x fp32
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5, help="timed rounds per setting")
    ap.add_argument("--reps", type=int, default=5, help="calls per timed round")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("swin_drop_path_bench.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda:0")
    model = copy.deepcopy(helpers.build_mirror("swinl", 2)).to(dev)
    head, bb = model.depth_head, model.depth_backbone
    bb.set_drop_path_rate(RATE)
    rgb = torch.randn(B, 3, *IMG, generator=torch.Generator().manual_seed(1)).to(dev)
    assert head.can_run_backbone(bb, rgb)
    sizes = head.swin_pyramid(IMG)
    eng = head._engine(B, ((IMG[0] + 1) // 2, (IMG[1] + 1) // 2), sizes[0], dev,
                       feats=([192, 384, 768, 1536], sizes), image_hw=IMG, backbone=bb)

    def engine(train):
        bb.train(train)
        eng.set_drop_path(head._swin_drop_scales(bb, B, dev))
        eng.run_backbone(rgb)
        eng.build_condition(None)

    def torch_train():
        bb.train()
        with torch.no_grad(), exact_fp32():
            feats = [f.contiguous() for f in bb(rgb)]
        eng.build_condition(feats)

    runs = {"eval": lambda: engine(False), "train": lambda: engine(True), "torch": torch_train}
    for fn in list(runs.values()) * 2:  # warm-up: every graph captured, every torch kernel chosen
        fn()
    captures = eng.graph_capture_count()
    times = {k: [] for k in runs}
    for _ in range(a.iters):
        for k, fn in runs.items():
            times[k].append(event_ms(fn, a.reps))
    assert eng.graph_capture_count() == captures  # switching never re-captured
    res = {"card (name, power limit, max SM clock)": card(), "batch": B, "image": list(IMG), "rate": RATE,
           "marked_blocks": sum(bin(m).count("1") for m in head.swin_drop_paths(bb)[0]),
           "extra_hbm_gb_all_marked": round(extra_bytes(head, bb) / 1e9, 3)}
    res.update({k + "_ms": summary(v) for k, v in times.items()})
    res["train_minus_eval_ms"] = round(res["train_ms"]["median"] - res["eval_ms"]["median"], 3)
    res["torch_over_train"] = round(res["torch_ms"]["median"] / res["train_ms"]["median"], 3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
