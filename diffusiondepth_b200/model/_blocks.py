"""Small building blocks with the parameter names the reference's mmcv wrappers produce, so the mirror
loads reference checkpoints key-for-key (SURVEY.md Appendix A), plus the fp32-exact execution context the
step-invariant producers (backbone / neck / FPN) run under."""
import contextlib

import torch
import torch.nn as nn


class ConvModule(nn.Module):
    """conv -> [BatchNorm2d as `.bn`] -> [ReLU]; bias iff no norm; kaiming-normal(fan_out) conv init —
    the semantics of mmcv.cnn.ConvModule the reference relies on (hahi.py:54-97, head :328-329)."""

    def __init__(self, cin, cout, k, padding=0, stride=1, norm=True, act=True):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, k, stride=stride, padding=padding, bias=not norm)
        if norm:
            self.bn = nn.BatchNorm2d(cout)
        self.with_norm, self.with_act = norm, act
        nn.init.kaiming_normal_(self.conv.weight, a=0, mode="fan_out", nonlinearity="relu")
        if self.conv.bias is not None:
            nn.init.zeros_(self.conv.bias)

    def forward(self, x):
        x = self.conv(x)
        if self.with_norm:
            x = self.bn(x)
        return torch.relu_(x) if self.with_act else x


class DropPath(nn.Module):
    """Stochastic depth; identity in eval (the only mode the engine serves)."""

    def __init__(self, p=0.0):
        super().__init__()
        self.p = p

    def forward(self, x):
        if not self.training or self.p == 0.0:
            return x
        keep = 1.0 - self.p
        return x * x.new_empty((x.shape[0],) + (1,) * (x.dim() - 1)).bernoulli_(keep) / keep


class MMCVDropPath(nn.Module):
    """Stochastic depth as mmcv 1.x's DropPath draws it (mmcv/cnn/bricks/drop.py, the Swin backbone's): in training mode
    at a rate above 0, x / keep * floor(keep + torch.rand((B, 1, ...))); otherwise identity, drawing nothing.  Its draw
    consumes the generator differently from DropPath's `bernoulli_`, so the two are separate classes."""

    def __init__(self, drop_prob=0.0):
        super().__init__()
        self.drop_prob = drop_prob

    def forward(self, x):
        if self.drop_prob == 0.0 or not self.training:
            return x
        keep = 1 - self.drop_prob
        r = keep + torch.rand((x.shape[0],) + (1,) * (x.dim() - 1), dtype=x.dtype, device=x.device)
        return x.div(keep) * r.floor()


@contextlib.contextmanager
def exact_fp32():
    """cuDNN/cuBLAS default to TF32 for fp32 convs/matmuls on GPU, which alone breaks the 1e-3 parity bar
    (SURVEY.md §7.2: a 4.9e-4 relative perturbation of the condition features gives 4.5e-3 on the output)."""
    c, m = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = c, m
