"""The depth encoder `depth_transform.t` restated in torch for any dtype, in either BatchNorm mode, and its autograd
gradients (test infrastructure; pinned to the real reference by tests/test_encoder_backward_oracle.py against
tests/golden/g_encoder_grads.npz)."""
import torch
import torch.nn.functional as F

from codec_train_helpers import ENC, bn_train

ENC_PARAMS = tuple(ENC + k for k in ("0.0.weight", "0.1.weight", "0.1.bias", "1.0.weight", "1.1.weight", "1.1.bias"))


def _leaky(v, band):
    """LeakyReLU(0.2); `band` > 0 moves every input within `band` of zero to the other slope (value and gradient)."""
    pos = v > 0
    if band:
        pos = pos ^ (v.detach().abs() < band)
    return v * torch.where(pos, 1.0, 0.2).to(v.dtype)


def encode(p, depth, train, band=0.0):
    """(t(depth), the first BatchNorm's output v1).  `p`: keys `depth_transform.conv_transform.*`; `train`: both
    BatchNorms on batch statistics, else on the running statistics."""
    def bn(u, k):
        if train:
            return bn_train(u, p[k + "weight"], p[k + "bias"])[0]
        return F.batch_norm(u, p[k + "running_mean"], p[k + "running_var"], p[k + "weight"], p[k + "bias"], False,
                            0.0, 1e-5)
    v1 = bn(F.conv2d(depth, p[ENC + "0.0.weight"], None, 2, 1), ENC + "0.1.")
    v2 = bn(F.conv2d(_leaky(v1, band), p[ENC + "1.0.weight"], None, 1, 1), ENC + "1.1.")
    return torch.tanh(v2), v1


def encoder_params(sd, dtype=torch.float64):
    """The encoder's tensors of `sd` (keys relative to `depth_head.`) on the CPU in `dtype`, parameters requiring grad."""
    return {k: v.detach().cpu().to(dtype).requires_grad_("running" not in k) for k, v in sd.items()
            if k.startswith(ENC)}


def encode_grads(sd, depth, d_latent, train, dtype=torch.float64, band=0.0):
    """Gradients of sum(t(depth) * d_latent) with respect to the encoder's parameters (ENC_PARAMS), and max |v1|."""
    p = encoder_params(sd, dtype)
    out, v1 = encode(p, depth.detach().cpu().to(dtype), train, band)
    (out * d_latent.detach().cpu().to(dtype)).sum().backward()
    return {k: p[k].grad for k in ENC_PARAMS}, float(v1.detach().abs().max())
