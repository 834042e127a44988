"""The training-mode MPViT backbone (`mpvit_small`, `head.mpvit_native_train`) on the engine against the torch backbone the
head otherwise falls back to, on the GPU.  Per size, in one process after warm-up, alternating the settings, CUDA events
around back-to-back calls, medians:
  engine_train  dd_set_drop_path (fresh masks at the model's rates, drawn on the device) + dd_run_backbone in
                DD_PRODUCER_TRAIN (batch-statistics BatchNorms, stochastic depth; its CUDA graph);
  engine_eval   dd_run_backbone in DD_PRODUCER_EVAL without stochastic depth (the inference network, for scale);
  torch_train   the mirror MPViT's forward in `.train()` in fp32 (TF32 off, as the head runs it), no grad.
Sizes: B = 2 at 70 x 106 and B = 4 at 352 x 1216 (the KITTI crop).  Prints the card's name, power limit and max SM
clock, and one JSON line.

    python profiles/mpvit_train_bench.py [--iters 5] [--reps 5]"""
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

SIZES = ((2, (70, 106)), (4, (352, 1216)))


def run_size(B, img, iters, reps, dev):
    model = copy.deepcopy(helpers.build_mirror("mpvit_s", 2, trained=True)).to(dev).train()
    head, bb = model.depth_head, model.depth_backbone
    head.producer_train_bn = head.mpvit_native_train = True
    rgb = torch.randn(B, 3, *img, generator=torch.Generator().manual_seed(1)).to(dev)
    assert head.can_run_backbone(bb, rgb)
    sizes = head.backbone_pyramid(img, bb)
    eng = head._engine(B, sizes[0], sizes[0], dev, feats=(list(head.fpn_in_channels), sizes), image_hw=img,
                       backbone=bb, producer_train=True)

    def engine(train):
        eng.set_producer_mode(train)
        eng.set_drop_path(head._mpvit_drop_scales(bb, B, dev) if train else None)
        eng.run_backbone(rgb)

    def torch_train():
        with torch.no_grad(), exact_fp32():
            bb(rgb)

    runs = {"engine_train": lambda: engine(True), "engine_eval": lambda: engine(False), "torch_train": torch_train}
    for fn in list(runs.values()) * 2:  # warm-up: every graph captured, every torch kernel chosen
        fn()
    times = {k: [] for k in runs}
    for _ in range(iters):
        for k, fn in runs.items():
            times[k].append(event_ms(fn, reps))
    eng.set_producer_mode(False)
    eng.set_drop_path(None)
    res = {"batch": B, "image": list(img), "bn_records": len(eng.producer_bn_keys()),
           "drop_path_blocks": len(head.mpvit_drop_paths(bb)[1])}
    res.update({k + "_ms": summary(v) for k, v in times.items()})
    res["torch_over_engine_train"] = round(res["torch_train_ms"]["median"] / res["engine_train_ms"]["median"], 3)
    head.invalidate_engines()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5, help="timed rounds per setting")
    ap.add_argument("--reps", type=int, default=5, help="calls per timed round")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("mpvit_train_bench.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda:0")
    out = {"card (name, power limit, max SM clock)": card(),
           "results": [run_size(B, img, a.iters, a.reps, dev) for B, img in SIZES]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
