"""TEST INFRASTRUCTURE ONLY — generate tests/golden/g_codec_kinds.npz from the REAL reference (/root/reference, imported
unmodified under oracle/refstub) for the learned depth codecs other than the default one.  Run in the build container:
python -m oracle.make_codec_kinds

Codec level, per codec: `t` and `inv_t` in eval mode with trained-like BatchNorms (oracle.restate_codecs.
trainedify_codec), at an even and an odd depth-map size.  Weights: `DEPTH_TRANSFORM.build` of the mirror under
torch.manual_seed(SEED_CODEC + kind), then trainedify_codec(seed = kind); inputs from seeded CPU generators.

Head level, T = 3, per case below: the whole model (`Diffusion_DCbase_Model.forward(sample)`) with the head's codec
replaced by the case's codec.  Weights: the mirror's default construction under SEED_WEIGHTS (as oracle/make_golden.py),
its `depth_head.depth_transform` replaced by the codec-level one, loaded into the reference with load_state_dict
(strict=True).  Inputs: oracle.restate.synthetic_sample; the initial latent: randn of the codec's latent shape from a
CPU generator seeded SEED_NOISE.  Stored: the decoder logit z of the final latent, the final latent, `pred_init`
(= depth_transform.t(gt)) and, for the Vis head, `pred_inter`, sub-sampled where large."""
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import configs, ref_import, restate_codecs  # noqa: E402
from oracle.reference_runner import _inject_first_randn  # noqa: E402
from oracle import restate  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "g_codec_kinds.npz")
SEED_CODEC = 500
NAMES = {1: "DeepDepthTransformWithUpsampling1x1", 2: "DeepDepthTransformWithUpsamplingX4", 3: "DeepDepthTransform"}
CODEC_SIZES = ((20, 28), (17, 23))
# name -> (family, codec kind, T, batch, H, W)
HEAD_CASES = {
    "swinl_x4": ("swinl", 2, 3, 1, 96, 160),          # Swin_ADDHAHI + X4: condition 24x40 -> latent 24x40
    "swinl_add_full": ("swinl_add", 3, 3, 1, 64, 96),  # neck-less Swin_ADD + DeepDepthTransform: condition up 4x
    "res18_1x1": ("res18", 1, 3, 2, 70, 106),         # Res18 + 1x1: condition == latent (35x53)
    "mpvit_x4": ("mpvit_s", 2, 3, 1, 64, 112),        # MPViT_ADDHAHI + X4: condition 32x56 above the 16x28 latent
    "swinl_vis_x4": ("swinl_vis", 2, 3, 1, 96, 160),  # Swin_ADDHAHIVis + X4: pred_inter
}
STRIDE = 2  # spatial sub-sampling of the stored head outputs (pred_init also keeps every 4th channel)


def mirror_codec(kind):
    from diffusiondepth_b200.model.registry import DEPTH_TRANSFORM
    torch.manual_seed(SEED_CODEC + kind)
    return restate_codecs.trainedify_codec(DEPTH_TRANSFORM.build(dict(type=NAMES[kind])), kind).eval()


def codec_inputs(kind, hw):
    g = torch.Generator().manual_seed(kind * 1000 + hw[0] * 100 + hw[1])
    depth = torch.rand(1, 1, *hw, generator=g) * 80
    latent = torch.randn(1, 16, *mirror_codec_latent(kind, hw), generator=g)
    return depth, latent


def mirror_codec_latent(kind, hw):
    from diffusiondepth_b200.model.registry import DEPTH_TRANSFORM
    return DEPTH_TRANSFORM.get(NAMES[kind]).latent_hw(hw)


def build_mirror_model(family, kind, steps):
    """The mirror model of `family` (SEED_WEIGHTS) with the head's codec replaced by mirror_codec(kind)."""
    from diffusiondepth_b200.model import get
    args = configs.make_args(family, steps)
    torch.manual_seed(configs.SEED_WEIGHTS)
    m = get(args)(args).eval()
    m.depth_head.depth_transform = mirror_codec(kind)
    return m


def head_noise(kind, B, H, W):
    return torch.randn(B, 16, *mirror_codec_latent(kind, (H, W)), generator=torch.Generator().manual_seed(configs.SEED_NOISE))


def run_reference(net, sample, noise):
    """The reference forward with the initial latent injected; z = the input of the decoder's final Sigmoid on the last
    inv_t call (the final latent: the Vis head decodes it first, then every step, the last of which is the same)."""
    cap = {}
    dt = net.depth_head.depth_transform
    hooks = [dt.conv_inv_transform.register_forward_pre_hook(lambda m, a: cap.__setitem__("latent", a[0].clone())),
             dt.conv_inv_transform[-1].register_forward_pre_hook(lambda m, a: cap.__setitem__("logits", a[0].clone()))]
    try:
        with torch.no_grad(), _inject_first_randn(noise) as st:
            out = net(sample)
        assert st["used"], "the reference did not draw the initial latent with the expected shape"
    finally:
        for h in hooks:
            h.remove()
    r = dict(logits=cap["logits"], latent=cap["latent"], pred=out["pred"], pred_init=out["pred_init"])
    if out.get("pred_inter") is not None:
        r["pred_inter"] = torch.stack([p.detach() for p in out["pred_inter"]])
    return r


def main():
    arrays = {}
    ref = ref_import.reference_modules()
    for kind, name in NAMES.items():
        m = mirror_codec(kind)
        r = getattr(ref.depth_transform, name)(hidden=16).eval()
        r.load_state_dict(m.state_dict(), strict=True)
        for hw in CODEC_SIZES:
            depth, latent = codec_inputs(kind, hw)
            with torch.no_grad():
                arrays[f"codec{kind}_{hw[0]}x{hw[1]}_t"] = r.t(depth).numpy()
                arrays[f"codec{kind}_{hw[0]}x{hw[1]}_z"] = r.conv_inv_transform[:-1](latent).numpy()
    for case, (family, kind, T, B, H, W) in HEAD_CASES.items():
        t0 = time.time()
        mirror = build_mirror_model(family, kind, T)
        sd = {k: v.detach().clone() for k, v in mirror.state_dict().items()}
        fam = configs.FAMILIES[family]
        net = ref_import.build_reference_model(ref_import.make_args(fam["backbone_module"], fam["backbone_name"],
                                                                    fam["head_specify"], T))
        net.depth_head.depth_transform = getattr(ref.depth_transform, NAMES[kind])(hidden=16)
        net.load_state_dict(sd, strict=True)
        net.eval()
        sample = restate.synthetic_sample(B, H, W, configs.SEED_INPUTS)
        torch.manual_seed(0)
        r = run_reference(net, sample, head_noise(kind, B, H, W))
        s = STRIDE
        arrays[case + "_logits"] = r["logits"][..., ::s, ::s].float().numpy()
        arrays[case + "_latent"] = r["latent"][..., ::s, ::s].float().numpy()
        arrays[case + "_pred_init"] = r["pred_init"][:, ::4, ::s, ::s].float().numpy()
        arrays[case + "_logits_absmax"] = np.float64(r["logits"].abs().max())
        arrays[case + "_meta"] = np.array([kind, T, B, H, W], dtype=np.int32)
        if "pred_inter" in r:
            arrays[case + "_pred_inter"] = r["pred_inter"][..., ::s, ::s].float().numpy()
        print(f"[{case}] {NAMES[kind]}: reference {time.time() - t0:.1f}s, latent {tuple(r['latent'].shape)}, "
              f"logits {tuple(r['logits'].shape)}", flush=True)
    arrays["stride"] = np.int32(STRIDE)
    np.savez_compressed(OUT, **arrays)
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1e3:.0f} kB)", flush=True)


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count() or 8)
    main()
