"""TEST INFRASTRUCTURE ONLY — the REAL reference model with the MPViT backbone (`DDIMDepthEstimate_MPVIT_ADDHAHI` on
`mpvit_small`, `norm_eval=False`) in training mode (`.train()`, as src/main.py trains), on CPU in the reference's own
fp32, with its DropPath modules in eval (stochastic depth off, so the result is deterministic); B = 2, at an odd image
(70 x 106: odd sizes on every MPViT level, the FPN resamples) and an exact-2x one (64 x 128).
The weights are the trained-like mirror state (oracle.configs.trainedify).  `head.pipeline` is replaced by a recorder
that keeps the condition map and stops the forward, so backbone, neck and FPN run exactly once.  Stored per case:
  feats/i      the four MPViT stage outputs, sub-sampled (sample_index) + their checksum,
  cond         the condition map, sub-sampled,
  bn/<key>/{mean,var}                    batch mean and unbiased batch variance of every producer BatchNorm's input
                                         (the backbone's 29, then the neck's and the FPN's),
  bn/<key>/{momentum,running_mean,running_var,num_batches_tracked}   the running statistics after the call.
Written to tests/golden/g_mpvit_train.npz.  Run in the build container:
    python -m oracle.make_mpvit_train"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import configs, ref_import, restate  # noqa: E402
from oracle.make_denoiser_grads import checksum, sample_index  # noqa: E402
from oracle.make_producer_train import _Stop, mirror_state, producer_bn_names  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "g_mpvit_train.npz")
B = 2
FAMILY = "mpvit_s"
CASES = {"mpvit_70x106": (70, 106), "mpvit_64x128": (64, 128)}


def case_inputs(name):
    H, W = CASES[name]
    return restate.synthetic_sample(B, H, W, configs.SEED_INPUTS)


def drop_path_off(model):
    """Every DropPath module of `model` in eval (identity); the rest keeps its mode."""
    for m in model.modules():
        if type(m).__name__ == "DropPath":
            m.eval()


def reference_case(name):
    sample = case_inputs(name)
    sd = mirror_state(FAMILY)
    fam = configs.FAMILIES[FAMILY]
    net = ref_import.build_reference_model(ref_import.make_args(fam["backbone_module"], fam["backbone_name"],
                                                                fam["head_specify"], 2))
    net.load_state_dict(sd, strict=True)
    net.train()
    drop_path_off(net)
    cap = {"stats": {}}

    def pipeline(*a, **kw):
        cap["cond"] = kw["input_args"][0].detach().clone()
        raise _Stop

    net.depth_head.pipeline = pipeline
    hooks = [net.depth_backbone.register_forward_hook(lambda m, a, o: cap.__setitem__("feats", [f.detach() for f in o]))]
    names = producer_bn_names(net)
    for n in names:
        def pre(m, a, n=n):
            x = a[0].detach().double()
            cap["stats"][n] = (x.mean((0, 2, 3)), x.var((0, 2, 3), unbiased=True))
        hooks.append(net.get_submodule(n).register_forward_pre_hook(pre))
    try:
        with torch.no_grad():
            net(sample)
        raise RuntimeError("the reference forward did not reach its pipeline")
    except _Stop:
        pass
    finally:
        for h in hooks:
            h.remove()
    out = {name + "/input_checksum": np.float64(checksum(sample["rgb"])),
           name + "/weight_checksum": np.float64(checksum(*[v for v in sd.values() if v.is_floating_point()]))}
    for i, f in enumerate(cap["feats"]):
        flat = f.reshape(-1)
        out[f"{name}/feats/{i}/checksum"] = np.float64(checksum(f))
        out[f"{name}/feats/{i}/values"] = flat[torch.from_numpy(sample_index(flat.numel()))].numpy()
    flat = cap["cond"].reshape(-1)
    out[name + "/cond/values"] = flat[torch.from_numpy(sample_index(flat.numel()))].numpy()
    out[name + "/cond/absmax"] = np.float64(flat.abs().max())
    for n in names:
        if n not in cap["stats"]:
            continue  # not on the way to the condition map
        bn = net.get_submodule(n)
        mean, var = cap["stats"][n]
        out[f"{name}/bn/{n}/mean"] = mean.numpy()
        out[f"{name}/bn/{n}/var"] = var.numpy()
        out[f"{name}/bn/{n}/running_mean"] = bn.running_mean.numpy()
        out[f"{name}/bn/{n}/running_var"] = bn.running_var.numpy()
        out[f"{name}/bn/{n}/num_batches_tracked"] = bn.num_batches_tracked.numpy()
        out[f"{name}/bn/{n}/momentum"] = np.float64(bn.momentum if bn.momentum is not None else -1.0)
    nbb = sum(1 for k in out if k.endswith("/mean") and "/bn/depth_backbone." in k)
    print(f"[{name}] {sum(1 for k in out if k.endswith('/mean'))} BatchNorms ({nbb} in the backbone), cond absmax "
          f"{float(out[name + '/cond/absmax']):.3g}", flush=True)
    return out


def main():
    torch.set_num_threads(os.cpu_count() or 8)
    arrays = {}
    for name in CASES:
        arrays.update(reference_case(name))
    np.savez_compressed(OUT, **arrays)
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1e3:.0f} kB)")


if __name__ == "__main__":
    main()
