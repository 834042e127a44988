"""The keys of the denoiser + codec pack, per variant and codec kind (H100, tiny geometry): dd_set_weight accepts exactly
the kind's keys, dd_finalize_weights names every missing one, refuses every key of the wrong shape (biases, GroupNorm
and BatchNorm vectors included) and a partial encoder, and packs without an encoder, after which dd_encode refuses."""
import ctypes as C

import pytest
import torch

from diffusiondepth_b200.engine import CODEC_KEYS, CODEC_UP, DENOISER_KEYS, FUSE_KEYS, DenoiseEngine
from diffusiondepth_b200.model.registry import HEADS

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
DD_ERR_INVALID = 1
CODECS = {0: "DeepDepthTransformWithUpsampling", 1: "DeepDepthTransformWithUpsampling1x1",
          2: "DeepDepthTransformWithUpsamplingX4", 3: "DeepDepthTransform"}
HEAD = {"swin": "DDIMDepthEstimate_Swin_ADDHAHI", "res": "DDIMDepthEstimate_Res"}
LAT = (4, 6)


def _tensors(variant, kind):
    torch.manual_seed(0)
    head = HEADS.build(dict(type=HEAD[variant], in_channels=[64, 128, 256, 512], inference_steps=1,
                            num_train_timesteps=1000, depth_feature_dim=16, loss_cfgs=[], init_cfg=None,
                            depth_transform_cfg=dict(type=CODECS[kind])))
    return {k: v.detach().to(DEV, torch.float32).contiguous() for k, v in head._engine_tensors().items()}


def _engine(variant, kind):
    cond = LAT if variant == "res" else (LAT[0] // 2, LAT[1] // 2)
    return DenoiseEngine(variant, 1, LAT, cond, 1, DEV, codec_kind=kind)


def _set(eng, key, t, shape=None):
    shape = tuple(t.shape) if shape is None else shape
    return eng.lib.dd_set_weight(eng._h, key.encode(), C.c_void_p(t.data_ptr()), (C.c_int64 * len(shape))(*shape),
                                 len(shape))


def _finalize(eng):
    rc = eng.lib.dd_finalize_weights(eng._h, C.c_void_p(eng._stream()))
    return rc, eng.lib.dd_last_error().decode()


def _required(variant, kind):
    return DENOISER_KEYS + (FUSE_KEYS if variant == "swin" else ()) + CODEC_KEYS[kind][1]


@pytest.mark.parametrize("kind", [0, 1, 2, 3])
@pytest.mark.parametrize("variant", ["swin", "res"])
def test_pack_keys(variant, kind):
    ts = _tensors(variant, kind)
    enc_keys = CODEC_KEYS[kind][0]
    required = _required(variant, kind)
    assert set(ts) == set(required + enc_keys)
    big = torch.zeros(1 << 20, device=DEV)

    # dd_set_weight: the kind's keys (and the fuse convs' on either variant), not another kind's
    eng = _engine(variant, kind)
    for k in DENOISER_KEYS + FUSE_KEYS + sum(CODEC_KEYS[kind], ()):
        assert _set(eng, k, big, tuple(ts[k].shape) if k in ts else (256,)) == 0, k
    for other in set(sum(sum(CODEC_KEYS.values(), ()), ())) - set(sum(CODEC_KEYS[kind], ())):
        assert _set(eng, other, big, (16,)) == DD_ERR_INVALID, other
    eng.close()

    # every key of the wrong shape, one at a time (a failed finalize keeps what was registered)
    eng = _engine(variant, kind)
    for k in required + enc_keys:
        assert _set(eng, k, ts[k]) == 0
    for k in required + enc_keys:
        s = ts[k].shape
        assert _set(eng, k, big, (s[0] + 1,) + tuple(s[1:])) == 0
        rc, msg = _finalize(eng)
        assert rc == DD_ERR_INVALID and k in msg and "shape" in msg, (k, msg)
        assert _set(eng, k, ts[k]) == 0
    assert _finalize(eng)[0] == 0
    eng.close()

    # each key missing: a required one, or one of the encoder's (a partial encoder)
    for k in required + enc_keys:
        eng = _engine(variant, kind)
        for j in required + enc_keys:
            if j != k:
                assert _set(eng, j, ts[j]) == 0
        rc, msg = _finalize(eng)
        assert rc == DD_ERR_INVALID and "missing weights" in msg and k in msg, (k, msg)
        eng.close()

    # no encoder: packs, and dd_encode refuses
    eng = _engine(variant, kind)
    for k in required:
        assert _set(eng, k, ts[k]) == 0
    assert _finalize(eng)[0] == 0
    u = CODEC_UP[kind]
    depth = torch.rand(1, 1, LAT[0] * u, LAT[1] * u, device=DEV)
    out = torch.empty(1, 16, *LAT, device=DEV)
    rc = eng.lib.dd_encode(eng._h, C.c_void_p(depth.data_ptr()), depth.shape[2], depth.shape[3],
                           C.c_void_p(out.data_ptr()), C.c_void_p(eng._stream()))
    assert rc == DD_ERR_INVALID and "not registered" in eng.lib.dd_last_error().decode()
    eng.close()
