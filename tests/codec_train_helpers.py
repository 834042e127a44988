"""The depth codec with its BatchNorms in training mode, restated in torch for any dtype (test infrastructure; pinned to
the real reference by tests/test_codec_train_oracle.py against tests/golden/g_codec_train.npz): the forward with its
batch statistics, and autograd gradients through the sampling loop + training-mode decoder."""
import torch
import torch.nn.functional as F

from loop_grad_helpers import _with_relu_band
from oracle import restate

DEC = "depth_transform.conv_inv_transform."
ENC = "depth_transform.conv_transform."


def bn_train(u, g, b):
    """F.batch_norm(training=True, eps=1e-5) and the batch (mean, unbiased variance) it records."""
    mean, var = u.mean((0, 2, 3)), u.var((0, 2, 3), unbiased=False)
    n = u.numel() // u.shape[1]
    v = (u - mean[None, :, None, None]) / torch.sqrt(var + 1e-5)[None, :, None, None] * g[None, :, None, None] \
        + b[None, :, None, None]
    return v, (mean, var * n / (n - 1))


def _relu(v, band):
    return torch.relu(v) if band == 0 else v * ((v > 0) ^ (v.abs() < band)).to(v.dtype)


def decode_train(p, latent, band=0.0):
    """inv_t with the decoder's BatchNorm in training mode: (depth, logit z, batch statistics).  `p`: keys
    `depth_transform.*`; `band` > 0 flips the ReLU's gradient mask within `band` of the kink."""
    u = F.conv_transpose2d(latent, p[DEC + "0.weight"], p[DEC + "0.bias"], stride=2, padding=1)
    v, stats = bn_train(u, p[DEC + "1.weight"], p[DEC + "1.bias"])
    z = F.conv2d(_relu(v, band), p[DEC + "3.0.weight"], p[DEC + "3.0.bias"], padding=1)
    return 1.0 / torch.sigmoid(z).clamp(1e-6) - 1, z, stats


def encode_train(p, depth):
    """t with both BatchNorms in training mode: (latent, [stats of BN1, stats of BN2])."""
    h, s1 = bn_train(F.conv2d(depth, p[ENC + "0.0.weight"], None, 2, 1), p[ENC + "0.1.weight"], p[ENC + "0.1.bias"])
    h, s2 = bn_train(F.conv2d(F.leaky_relu(h, 0.2), p[ENC + "1.0.weight"], None, 1, 1), p[ENC + "1.1.weight"],
                     p[ENC + "1.1.bias"])
    return torch.tanh(h), [s1, s2]


def decode_train_grads(sd, latent, d_depth, dtype=torch.float64, band=0.0):
    """Gradients of sum(decode_train(latent) * d_depth): d_latent and the decoder parameters (keys of `sd`)."""
    p = {k: v.detach().cpu().to(dtype).requires_grad_("running" not in k)
         for k, v in sd.items() if k.startswith("depth_transform.")}
    x = latent.detach().cpu().to(dtype).requires_grad_(True)
    depth, _, _ = decode_train(p, x, band)
    (depth * d_depth.detach().cpu().to(dtype)).sum().backward()
    out = {"d_latent": x.grad}
    out.update({k: v.grad for k, v in p.items() if v.grad is not None})
    return out


def loop_train_grads(variant, sd, cond, noise, d_depth, d_latent, steps, dtype=torch.float64, band=0.0):
    """As loop_grad_helpers.loop_restatement_grads, with the decoder's BatchNorm in training mode."""
    p = {"depth_head." + k: v.detach().cpu().to(dtype).requires_grad_("running" not in k) for k, v in sd.items()}
    c = cond.detach().cpu().to(dtype).requires_grad_(True)
    x = noise.detach().cpu().to(dtype).requires_grad_(True)
    codec = {k[len("depth_head."):]: v for k, v in p.items() if k.startswith("depth_head.depth_transform.")}
    latent = _with_relu_band(band, lambda: restate.ddim_loop(p, c, x, steps, variant))
    depth, _, _ = decode_train(codec, latent, band)
    loss = (depth * d_depth.detach().cpu().to(dtype)).sum()
    if d_latent is not None:
        loss = loss + (latent * d_latent.detach().cpu().to(dtype)).sum()
    loss.backward()
    out = {"d_cond": c.grad, "d_noise": x.grad}
    out.update({k[len("depth_head."):]: v.grad for k, v in p.items() if v.grad is not None})
    return out
