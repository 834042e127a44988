"""What training the depth encoder costs (`dd_encode_backward`, `head.grad_through_encoder`), on the GPU, at BASELINE
config 3's geometry (B = 4, 352 x 1216 depth map -> latent 176 x 608; Swin head, condition map 88 x 304), eval-mode
codec, after warm-up, CUDA events:
  (a) one encode_backward, and one encode + encode_backward;
  (b) torch fp32 autograd (TF32 off) of the same encoder: forward + backward of sum(t(depth) * d_latent);
  (c) one head.ddim_loss_gt forward + backward with gt_map_t through the encoder (`_EncodeFunction`) and the denoiser.
Prints the card's name, power limit and max SM clock, and one JSON line.

    python profiles/encoder_backward_bench.py [--reps 20] [--batch 4 --height 352 --width 1216]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def event_ms(fn, reps):
    """Device milliseconds per fn() over reps back-to-back calls (CUDA events), after two warm-up calls."""
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--height", type=int, default=352)
    ap.add_argument("--width", type=int, default=1216)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    from loop_grad_helpers import make_loop_head
    from oracle.make_loop_grads import loop_state
    dev = torch.device("cuda:0")
    B, H, W = a.batch, a.height, a.width
    hw, chw = ((H + 1) // 2, (W + 1) // 2), ((H + 3) // 4, (W + 3) // 4)
    head = make_loop_head("swin", loop_state("swin"), 20, dev)
    head.train()
    eng = head._engine(B, hw, chw, dev, backward=True)
    eng.set_codec_mode(False)
    g = torch.Generator().manual_seed(3)
    depth = (torch.rand(B, 1, H, W, generator=g) * 2 + 0.1).to(dev)
    d_latent = torch.randn(B, 16, *hw, generator=g).to(dev)
    cond = torch.randn(B, 256, *chw, generator=g).abs().to(dev)
    res = {"card": card(), "batch": B, "depth_hw": [H, W], "latent_hw": list(hw)}
    res["encode_backward_ms"] = event_ms(lambda: eng.encode_backward(depth, d_latent), a.reps)
    res["encode_plus_backward_ms"] = event_ms(lambda: (eng.encode(depth), eng.encode_backward(depth, d_latent)), a.reps)

    codec = head.depth_transform  # eval BatchNorm, as the engine above
    codec.eval()

    def torch_step():
        for p in codec.conv_transform.parameters():
            p.grad = None
        (codec.t(depth) * d_latent).sum().backward()
    res["torch_fp32_encoder_fwd_bwd_ms"] = event_ms(torch_step, a.reps)
    codec.train()

    head.grad_through_encoder = True
    enc = head._encoder_params()

    def loss_gt_step():
        head.zero_grad(set_to_none=True)
        gt_map_t = head._encode(eng, depth, False, enc)
        head.ddim_loss_gt(gt_map_t, (cond, None, None, None), gt_map_t, 1.0).backward()
    res["ddim_loss_gt_fwd_bwd_ms"] = event_ms(loss_gt_step, max(1, a.reps // 4))
    res = {k: (round(v, 4) if isinstance(v, float) else v) for k, v in res.items()}
    print(f"card: {res['card']}")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
