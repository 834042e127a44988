"""The training-mode codec restatement (codec_train_helpers) and the head's running-statistic update behave like the real
reference's DeepDepthTransformWithUpsampling in `.train()`: outputs, running statistics after one call and after a *Vis
head's T + 1 calls, gradients, and the sampling loop's gradients with the codec in training mode, against
tests/golden/g_codec_train.npz (oracle/make_codec_train.py).  This pins the restatement the GPU tests of
tests/test_codec_train.py compare against."""
import numpy as np
import pytest
import torch
import torch.nn as nn

from codec_train_helpers import DEC, decode_train, decode_train_grads, encode_train, loop_train_grads
from diffusiondepth_b200.model.head._ddim_head import bn_running_update
from grad_helpers import golden_margins, tensor_margins
from oracle.make_codec_train import BN_KEYS, LOOP_CASES, OUT, codec_inputs, codec_state
from oracle.make_denoiser_grads import checksum
from oracle.make_loop_grads import STEPS, case_inputs

BIAS = DEC + "0.bias"  # no effect through a training-mode BatchNorm: its gradient is rounding noise in the reference too


@pytest.fixture(scope="module")
def golden():
    return np.load(OUT, allow_pickle=False)


def _state(dtype):
    return {"depth_transform." + k: v.to(dtype) for k, v in codec_state().items()}


def _bn(name):
    """A BatchNorm2d holding the golden's starting state of codec BatchNorm `name` (num_batches_tracked = 0)."""
    st = codec_state()
    bn = nn.BatchNorm2d(16)
    bn.running_mean.copy_(st[BN_KEYS[name] + ".running_mean"])
    bn.running_var.copy_(st[BN_KEYS[name] + ".running_var"])
    return bn


def _check_running(bn, golden, prefix):
    assert int(bn.num_batches_tracked) == int(golden[prefix + "num_batches_tracked"])
    for k in ("running_mean", "running_var"):
        ref = torch.from_numpy(golden[prefix + k]).double()
        err = float(((getattr(bn, k).double() - ref).abs() / ref.abs().clamp_min(1e-3)).max())
        assert err <= 2e-6, (prefix + k, err)


def _rel(a, ref):
    ref = torch.from_numpy(ref).double()
    return float((a.detach().double() - ref).abs().max() / ref.abs().max())


def test_codec_restatement_matches_reference_train(golden):
    latent, depth, d_depth, vis = codec_inputs()
    assert checksum(*codec_state().values()) == pytest.approx(float(golden["codec/weight_checksum"]), rel=1e-12)
    assert checksum(latent, depth, d_depth, *vis) == pytest.approx(float(golden["codec/input_checksum"]), rel=1e-12)
    p = _state(torch.float64)
    inv, _, dstats = decode_train(p, latent.double())
    lat, estats = encode_train(p, depth.double())
    e_inv, e_t = _rel(inv, golden["codec/inv_t"]), _rel(lat, golden["codec/t"])
    print(f"\n[codec train] inv_t {e_inv:.1e}, t {e_t:.1e} (fp64 restatement vs fp32 reference)")
    assert e_inv <= 2e-5 and e_t <= 2e-5
    # the head's running update (bn_running_update) from the restatement's statistics
    bn = _bn("dec")
    bn_running_update(bn, *dstats)
    _check_running(bn, golden, "codec/after_decode/dec/")
    for name, st in zip(("enc1", "enc2"), estats):
        bn = _bn(name)
        bn_running_update(bn, *st)
        _check_running(bn, golden, f"codec/after_encode/{name}/")
    bn = _bn("dec")  # a *Vis head: the final map's statistics first, then steps 1 .. T
    for x in [vis[-1]] + vis:
        bn_running_update(bn, *decode_train(p, x.double())[2])
    _check_running(bn, golden, "codec/after_vis/dec/")


def test_codec_gradients_match_reference_train(golden):
    latent, _, d_depth, _ = codec_inputs()
    sd = _state(torch.float32)
    g64 = decode_train_grads(sd, latent, d_depth)
    env = tensor_margins(decode_train_grads(sd, latent, d_depth, band=1e-6), g64)
    m = {}
    for k, v in g64.items():
        name = "d_latent" if k == "d_latent" else k[len("depth_transform."):]
        m[k] = _rel(v, golden["codec/grad/" + name])
    bias = float(np.abs(golden["codec/grad/conv_inv_transform.0.bias"]).max() /
                 np.abs(golden["codec/grad/conv_inv_transform.0.weight"]).max())
    print(f"\n[codec train grads] {m}; reference |d b_t| / max |dW_t| = {bias:.1e}")
    assert bias <= 1e-5 and float(g64[BIAS].abs().max() / g64[DEC + "0.weight"].abs().max()) <= 1e-12
    for k in m:
        if k != BIAS:
            assert m[k] <= 1e-4 + env[k], (k, m[k], env[k])


@pytest.mark.parametrize("case", LOOP_CASES)
def test_loop_train_restatement_matches_reference(case, golden):
    variant, sd, cond, noise, d_depth, d_latent = case_inputs(case)
    assert checksum(*sd.values()) == pytest.approx(float(golden[case + "/weight_checksum"]), rel=1e-12)
    assert checksum(cond, noise, d_depth, d_latent) == pytest.approx(float(golden[case + "/input_checksum"]), rel=1e-12)
    g64 = loop_train_grads(variant, sd, cond, noise, d_depth, d_latent, STEPS)
    m64 = golden_margins(golden, case, g64)
    assert len(m64) == (28 if variant == "swin" else 24)
    env = tensor_margins(loop_train_grads(variant, sd, cond, noise, d_depth, d_latent, STEPS, band=1e-6), g64)
    m64.pop(BIAS)
    worst = max(m64, key=lambda k: m64[k] - env[k])
    print(f"\n[{case} train codec] restatement fp64 vs reference fp32: worst {worst} {m64[worst]:.2e} "
          f"(kink envelope {env[worst]:.2e})")
    for k in m64:
        assert m64[k] <= 1e-4 + env[k], (k, m64[k], env[k])
