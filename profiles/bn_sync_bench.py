"""What synchronised BatchNorm (`head.bn_sync_group`, dd_set_bn_allgather) costs at world size 1, on the GPU: the eager
launches that replace the training-mode producer graphs, plus two all-gathers per BatchNorm in the forward.  Per
configuration, in one process after warm-up, alternating the settings on the same engine (CUDA events):
  chain:  dd_run_backbone + dd_build_condition in DD_PRODUCER_TRAIN (graphed without a gatherer);
  decode: one dd_decode in DD_CODEC_TRAIN (its BatchNorm's statistics, fold and the decoder);
each without a gatherer, with an NCCL gatherer (a one-rank NCCL group: the collective runs on the engine's stream) and
with a gloo gatherer (a one-rank gloo group: staged through host memory, synchronous).
Configurations: C3 (Swin-L + HAHI neck + FPN, B = 4, 352 x 1216) and C2 (res50-shaped native ResNet + FPN, B = 8,
228 x 304).  Prints the card's name, power limit and max SM clock, and one JSON line.

    python profiles/bn_sync_bench.py [--iters 5] [--configs C3,C2]"""
import argparse
import copy
import json
import os
import statistics
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import dd_helpers as helpers  # noqa: E402
from oracle import configs, restate  # noqa: E402
from producer_train_bench import card, event_ms, summary  # noqa: E402


def run_config(name, iters, dev, groups):
    family, steps, B, H, W = configs.CONFIGS[name]
    model = copy.deepcopy(helpers.build_mirror(family, steps)).to(dev).train()
    head = model.depth_head
    head.check_range = False
    head.producer_train_bn = head.codec_train_bn = True
    sample = {k: v.to(dev) for k, v in restate.synthetic_sample(B, H, W, 3).items()}
    sample["noise"] = restate.synthetic_noise(B, H, W, 3).to(dev)
    with torch.no_grad():
        model(sample)  # creates and packs the native engine
    eng = next(e for k, e in head._engines.items() if k.image_hw is not None and k.producer_train)
    img = sample["rgb"].contiguous().float()
    latent = torch.randn(B, 16, *eng.latent_hw, generator=torch.Generator().manual_seed(0)).to(dev)
    eng.set_producer_mode(True)
    eng.set_codec_mode(True)

    def chain():
        eng.run_backbone(img)
        eng.build_condition(None)

    def decode():
        eng.decode(latent)

    settings = ["none"] + list(groups)
    for s in settings:  # warm-up: the graphs, the gather buffers, the collectives' first calls
        eng.set_bn_allgather(groups.get(s))
        chain()
        decode()
    times = {(s, w): [] for s in settings for w in ("chain", "decode")}
    for _ in range(iters):
        for s in settings:
            eng.set_bn_allgather(groups.get(s))
            times[(s, "chain")].append(event_ms(chain, 5))
            times[(s, "decode")].append(event_ms(decode, 20))
    eng.set_bn_allgather(None)
    res = {"config": name, "family": family, "batch": B, "image": [H, W], "producer_bn_layers": len(eng.producer_bn_keys())}
    for (s, w), xs in times.items():
        res[f"{w}_ms_{s}"] = summary(xs)
    head.invalidate_engines()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5, help="timed rounds per setting")
    ap.add_argument("--configs", default="C3,C2")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bn_sync_bench.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", store=dist.HashStore(), rank=0, world_size=1, device_id=dev)
    try:
        groups = {"nccl": dist.group.WORLD, "gloo": dist.new_group([0], backend="gloo")}
        out = {"card (name, power limit, max SM clock)": card(), "world_size": 1,
               "results": [run_config(c, a.iters, dev, groups) for c in a.configs.split(",")]}
    finally:
        dist.destroy_process_group()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
