"""Depth <-> latent codec registry (reference src/model/ops/depth_transform.py): all six transforms of the reference's
`DEPTH_TRANSFORM`, with its module layout and state_dict keys.

The four learned codecs (hidden = 16, the DDIM denoiser's `channels_noise`) are PARAMETER CONTAINERS inside a head:
`t()` (encoder; its value is only returned as `pred_init` / `gt_map_t`) runs through `dd_encode`, `inv_t()` (decoder,
on the hot path) through `dd_denoise_decode` / `dd_decode` (`DenoiseEngine.encode / .decode`), each on the engine's
kernels for its `ENGINE_KIND` (include/dd_engine.h, dd_codec_kind).  A codec also states the latent grid of an image
size (`latent_hw`) and the decoder's upsampling `UP`.  The default codec (`DeepDepthTransformWithUpsampling`) alone
trains its BatchNorms and encoder / decoder on the engine.  The torch expressions below exist for API parity when a
caller invokes `t` / `inv_t` directly on a tensor (and for the torch-op fallback of architectures the engine does not
instantiate).  The two reciprocal transforms are parameter-free torch only: the 16-channel DDIM heads cannot use
them, as in the reference."""
import torch
import torch.nn as nn

from ..registry import DEPTH_TRANSFORM


def _conv_block(cin, cout, k, stride, pad, bn=True, act=True):
    """conv(bias iff no BN) [+ BatchNorm2d] [+ LeakyReLU(0.2)] — key layout `0.weight`, `1.*`
    (reference src/model/common.py:45-60)."""
    mods = [nn.Conv2d(cin, cout, k, stride, pad, bias=not bn)]
    if bn:
        mods.append(nn.BatchNorm2d(cout))
    if act:
        mods.append(nn.LeakyReLU(0.2, inplace=True))
    return nn.Sequential(*mods)


class _LearnedCodec(nn.Module):
    """t = conv_transform, inv_t = 1 / clamp(conv_inv_transform, eps) - 1 (reference :29-35, :58-64, :88-94, :113-117).
    ENGINE_KIND: the engine's dd_codec_kind; UP: the decoder's upsampling (decoded map u h x u w)."""
    ENGINE_KIND = 0
    UP = 2

    @staticmethod
    def latent_hw(image_hw):
        """Latent grid of an H x W depth map: one stride-2 stage, ceil(H / 2) x ceil(W / 2)."""
        return tuple((int(n) + 1) // 2 for n in image_hw)

    def t(self, depth):
        return self.conv_transform(depth)

    def inv_t(self, value):
        return 1.0 / self.conv_inv_transform(value).clamp(self.eps) - 1


def _up2_decoder(hidden):
    """ConvT(k4, s2, p1) + BatchNorm + ReLU + 3x3 conv -> 1 + sigmoid (reference :20-26, :49-55)."""
    return nn.Sequential(
        nn.ConvTranspose2d(hidden, hidden, kernel_size=4, stride=2, padding=1),
        nn.BatchNorm2d(hidden),
        nn.ReLU(inplace=True),
        _conv_block(hidden, 1, 3, 1, 1, bn=False, act=False),
        nn.Sigmoid())


@DEPTH_TRANSFORM.register_module()
class DeepDepthTransformWithUpsampling(nn.Module):
    ENGINE_KIND = 0
    UP = 2
    latent_hw = staticmethod(_LearnedCodec.latent_hw)

    def __init__(self, hidden=16, eps=1e-6):
        super().__init__()
        self.conv_transform = nn.Sequential(
            _conv_block(1, hidden, 3, 2, 1),
            _conv_block(hidden, hidden, 3, 1, 1, act=False),
            nn.Tanh())
        self.conv_inv_transform = nn.Sequential(
            nn.ConvTranspose2d(hidden, hidden, kernel_size=4, stride=2, padding=1),
            nn.BatchNorm2d(hidden),
            nn.ReLU(inplace=True),
            _conv_block(hidden, 1, 3, 1, 1, bn=False, act=False),
            nn.Sigmoid())
        self.eps = eps

    def t(self, depth):
        return self.conv_transform(depth)

    def inv_t(self, value):
        return 1.0 / self.conv_inv_transform(value).clamp(self.eps) - 1


@DEPTH_TRANSFORM.register_module()
class DeepDepthTransformWithUpsampling1x1(_LearnedCodec):
    """Reference :38-64: two bias-free 1x1 convs, tanh, MaxPool 3x3 s2 p1; the default codec's decoder."""
    ENGINE_KIND = 1

    def __init__(self, hidden=16, eps=1e-6):
        super().__init__()
        self.conv_transform = nn.Sequential(
            nn.Conv2d(1, hidden, 1, 1, 0, bias=False),
            nn.Conv2d(hidden, hidden, 1, 1, 0, bias=False),
            nn.Tanh(),
            nn.MaxPool2d(kernel_size=3, stride=2, padding=1))
        self.conv_inv_transform = _up2_decoder(hidden)
        self.eps = eps


@DEPTH_TRANSFORM.register_module()
class DeepDepthTransformWithUpsamplingX4(_LearnedCodec):
    """Reference :67-94: two stride-2 conv_bn_relu stages (latent at a quarter of the resolution), two ConvTs up."""
    ENGINE_KIND = 2
    UP = 4

    @staticmethod
    def latent_hw(image_hw):
        return tuple(((int(n) + 1) // 2 + 1) // 2 for n in image_hw)

    def __init__(self, hidden=16, eps=1e-6):
        super().__init__()
        self.conv_transform = nn.Sequential(
            _conv_block(1, hidden, 3, 2, 1),
            _conv_block(hidden, hidden, 3, 2, 1),
            _conv_block(hidden, hidden, 3, 1, 1, act=False),
            nn.Tanh())
        self.conv_inv_transform = nn.Sequential(
            nn.ConvTranspose2d(hidden, hidden, kernel_size=4, stride=2, padding=1),
            nn.ConvTranspose2d(hidden, hidden, kernel_size=4, stride=2, padding=1),
            nn.BatchNorm2d(hidden),
            nn.ReLU(inplace=True),
            _conv_block(hidden, 1, 3, 1, 1, bn=False, act=False),
            nn.Sigmoid())
        self.eps = eps


@DEPTH_TRANSFORM.register_module()
class DeepDepthTransform(_LearnedCodec):
    """Reference :97-117: stride-1 conv_bn_relu stages both ways; the latent is at the depth map's resolution."""
    ENGINE_KIND = 3
    UP = 1

    @staticmethod
    def latent_hw(image_hw):
        return tuple(int(n) for n in image_hw)

    def __init__(self, hidden=16, eps=1e-6):
        super().__init__()
        self.conv_transform = nn.Sequential(
            _conv_block(1, hidden, 3, 1, 1),
            _conv_block(hidden, hidden, 3, 1, 1, act=False),
            nn.Tanh())
        self.conv_inv_transform = nn.Sequential(
            _conv_block(hidden, hidden, 3, 1, 1),
            _conv_block(hidden, 1, 3, 1, 1, act=False),
            nn.Sigmoid())
        self.eps = eps


@DEPTH_TRANSFORM.register_module()
class ReciprocalDepthTransform:
    """Parameter-free transform BaseDepthRefine builds by default before the DDIM heads replace it
    (reference mmbev_base_depth_refine.py:21, depth_transform.py:120-133)."""

    def __init__(self, linear=(1, 0), eps=1e-6):
        self.linear, self.eps = linear, eps

    def t(self, depth):
        return self.linear[0] / (1 + depth.clamp(0.)).clamp(self.eps) + self.linear[1]

    def inv_t(self, value):
        return self.linear[0] / (value - self.linear[1]).clamp(self.eps) - 1


@DEPTH_TRANSFORM.register_module()
class ReciprocalDepthTransformII:
    """Reference :136-145: parameter-free, registry parity only."""

    def __init__(self, min_depth=0.5):
        self.min_depth = min_depth

    def t(self, depth):
        return self.min_depth / depth.clamp(self.min_depth)

    def inv_t(self, value):
        return self.min_depth / value
