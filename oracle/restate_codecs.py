"""TEST INFRASTRUCTURE ONLY — restatement of the reference's other learned depth codecs (paths relative to
/root/reference/src/model), on a plain `state_dict` in the reference key layout with functional torch ops, in the
dtype of the input (fp64: ground truth for the engine's error budgets).  Eval-mode BatchNorm (running statistics).

Kinds follow include/dd_engine.h `dd_codec_kind`: 0 DeepDepthTransformWithUpsampling (oracle/restate.py encode /
decode_logits), 1 DeepDepthTransformWithUpsampling1x1, 2 DeepDepthTransformWithUpsamplingX4, 3 DeepDepthTransform.
Nothing under `diffusiondepth_b200/` imports this module."""
import torch
import torch.nn.functional as F

from oracle import restate
from oracle.restate import _p, batchnorm_eval

ENC = "depth_head.depth_transform.conv_transform."
DEC = "depth_head.depth_transform.conv_inv_transform."


def _conv_bn(x, sd, prefix, stride, act):
    """conv_bn_relu (common.py:45-60): conv without bias, BatchNorm, LeakyReLU(0.2) when `act`."""
    h = F.conv2d(x, _p(sd, prefix + "0.weight", x.dtype), None, stride=stride, padding=1)
    h = batchnorm_eval(h, sd, prefix + "1")
    return F.leaky_relu(h, 0.2) if act else h


def encode(sd, depth, kind, prefix=ENC):
    """depth_transform.t of codec `kind`."""
    if kind == 0:
        return restate.encode(sd, depth, prefix)
    if kind == 1:  # ops/depth_transform.py:43-48
        h = F.conv2d(depth, _p(sd, prefix + "0.weight", depth.dtype))
        h = torch.tanh(F.conv2d(h, _p(sd, prefix + "1.weight", depth.dtype)))
        return F.max_pool2d(h, 3, 2, 1)
    if kind == 2:  # :72-77
        h = _conv_bn(depth, sd, prefix + "0.", 2, True)
        h = _conv_bn(h, sd, prefix + "1.", 2, True)
        return torch.tanh(_conv_bn(h, sd, prefix + "2.", 1, False))
    h = _conv_bn(depth, sd, prefix + "0.", 1, True)  # :101-105
    return torch.tanh(_conv_bn(h, sd, prefix + "1.", 1, False))


def decode_logits(sd, latent, kind, prefix=DEC):
    """depth_transform.conv_inv_transform of codec `kind` up to (not including) the sigmoid: the logit z."""
    if kind in (0, 1):  # :49-55 are the default decoder's modules
        return restate.decode_logits(sd, latent, prefix)
    dt = latent.dtype
    if kind == 2:  # :78-85
        h = F.conv_transpose2d(latent, _p(sd, prefix + "0.weight", dt), _p(sd, prefix + "0.bias", dt), stride=2, padding=1)
        h = F.conv_transpose2d(h, _p(sd, prefix + "1.weight", dt), _p(sd, prefix + "1.bias", dt), stride=2, padding=1)
        h = torch.relu(batchnorm_eval(h, sd, prefix + "2"))
        return restate.conv(h, sd, prefix + "4.0")
    h = _conv_bn(latent, sd, prefix + "0.", 1, True)  # :106-110
    return _conv_bn(h, sd, prefix + "1.", 1, False)


def decode(sd, latent, kind, eps=1e-6):
    """depth_transform.inv_t: 1 / clamp(sigmoid(z), eps) - 1 (:33-35, :62-64, :92-94, :116-117)."""
    return 1.0 / torch.sigmoid(decode_logits(sd, latent, kind)).clamp(eps) - 1


def trainedify_codec(module, seed=0, scale_range=(1e-2, 1e2)):
    """Trained-like BatchNorm statistics and affine on every BatchNorm of a codec module (in place): running means
    away from 0, variances and weights spread log-uniformly over `scale_range`."""
    g = torch.Generator().manual_seed(seed)
    lo, hi = torch.log(torch.tensor(scale_range[0])), torch.log(torch.tensor(scale_range[1]))
    with torch.no_grad():
        for m in module.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                n = m.num_features
                m.running_mean.copy_(torch.randn(n, generator=g) * 0.3)
                m.running_var.copy_(torch.exp(lo + (hi - lo) * torch.rand(n, generator=g)) * 0.1)
                m.weight.copy_(torch.exp(lo + (hi - lo) * torch.rand(n, generator=g)) * 0.05 *
                               torch.sign(torch.randn(n, generator=g)))
                m.bias.copy_(torch.randn(n, generator=g) * 0.2)
    return module
