"""TEST INFRASTRUCTURE ONLY — the REAL reference model in training mode (`.train()`, as src/main.py trains), on CPU in
the reference's own fp32, for the condition producers' BatchNorms:
  Swin_ADDHAHI (swinl family) with the backbone in eval (DropPath off), and the Res head with mmbev_res18, the whole
  model in train mode; B = 2, at an odd image (70 x 106: the FPN resamples) and an exact-2x one (64 x 128).
The weights are the trained-like mirror state (oracle.configs.trainedify).  `head.pipeline` is replaced by a recorder
that keeps the condition map and stops the forward, so the neck / FPN / backbone run exactly once.  Stored per case:
  feats/i      backbone features, sub-sampled (sample_index) + their checksum,
  cond         the condition map, sub-sampled,
  bn/<key>/{mean,var}                    batch mean and unbiased batch variance of every producer BatchNorm's input,
  bn/<key>/{running_mean,running_var,num_batches_tracked}   the running statistics after the call.
Written to tests/golden/g_producer_train.npz.  Run in the build container:
    python -m oracle.make_producer_train"""
import os
import sys

import numpy as np
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import configs, ref_import, restate  # noqa: E402
from oracle.make_denoiser_grads import checksum, sample_index  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "g_producer_train.npz")
B = 2
# name -> (family, image (H, W))
CASES = {"swinl_70x106": ("swinl", (70, 106)), "swinl_64x128": ("swinl", (64, 128)),
         "res18_70x106": ("res18", (70, 106)), "res18_64x128": ("res18", (64, 128))}
PRODUCER_PREFIXES = ("depth_head.hahineck.", "depth_head.conv_lateral.", "depth_head.conv_up.", "depth_backbone.")


def mirror_state(family):
    """The trained-like mirror state dict (reference keys) the golden was made from."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import dd_helpers
    m = dd_helpers.build_mirror(family, 2, trained=True)
    return {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}


def case_inputs(name):
    family, (H, W) = CASES[name]
    return family, restate.synthetic_sample(B, H, W, configs.SEED_INPUTS)


def producer_bn_names(model):
    """Names (reference keys) of every BatchNorm in the backbone, neck and FPN, in module order."""
    return [n for n, m in model.named_modules() if isinstance(m, nn.BatchNorm2d) and n.startswith(PRODUCER_PREFIXES)]


class _Stop(Exception):
    pass


def reference_case(name):
    family, sample = case_inputs(name)
    sd = mirror_state(family)
    fam = configs.FAMILIES[family]
    net = ref_import.build_reference_model(ref_import.make_args(fam["backbone_module"], fam["backbone_name"],
                                                                fam["head_specify"], 2))
    net.load_state_dict(sd, strict=True)
    net.train()
    if family.startswith("swin"):
        net.depth_backbone.eval()  # DropPath off: the engine's Swin-L is the eval network
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
    print(f"[{name}] {sum(1 for k in out if k.endswith('/mean'))} BatchNorms, cond absmax "
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
