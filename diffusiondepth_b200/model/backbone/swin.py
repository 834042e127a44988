"""Swin Transformer condition-feature producer (reference src/model/backbone/swin.py:23-793 and
backbone/utils.py:201-302), restated compactly.  Step-invariant: runs once per image, outside the loop.

Parity traps honoured (SURVEY.md Appendix C): q is scaled before q@k^T; the shift mask is a finite -100;
tokens are zero-padded to a multiple of the window *before* the roll; patch merging groups channels
channel-major (nn.Unfold order); every stage output has its own LayerNorm; GELU is exact (erf);
`swin_large_naive_nopretrain` never initialises the relative-position table (all zeros)."""
import torch
import torch.nn as nn
import torch.nn.functional as F

from .._blocks import MMCVDropPath


class PatchEmbed(nn.Module):
    def __init__(self, cin, dim, patch):
        super().__init__()
        self.patch = patch
        self.projection = nn.Conv2d(cin, dim, patch, patch)
        self.norm = nn.LayerNorm(dim)

    def forward(self, x):
        H, W = x.shape[-2:]
        x = F.pad(x, (0, -W % self.patch, 0, -H % self.patch))
        x = self.projection(x)
        hw = x.shape[-2:]
        return self.norm(x.flatten(2).transpose(1, 2)), (int(hw[0]), int(hw[1]))


class PatchMerging(nn.Module):
    def __init__(self, dim, out_dim):
        super().__init__()
        self.norm = nn.LayerNorm(4 * dim)
        self.reduction = nn.Linear(4 * dim, out_dim, bias=False)

    def forward(self, x, hw):
        B, _, C = x.shape
        H, W = hw
        x = x.view(B, H, W, C).permute(0, 3, 1, 2)
        x = F.pad(x, (0, W % 2, 0, H % 2))
        x = F.unfold(x, kernel_size=2, stride=2).transpose(1, 2)  # [B, L/4, C*4], feature = c*4 + ky*2 + kx
        return self.reduction(self.norm(x)), ((H + 1) // 2, (W + 1) // 2)


class WindowMSA(nn.Module):
    def __init__(self, dim, heads, ws):
        super().__init__()
        self.heads, self.ws, self.scale = heads, ws, (dim // heads) ** -0.5
        self.relative_position_bias_table = nn.Parameter(torch.zeros((2 * ws - 1) ** 2, heads))
        coords = torch.stack(torch.meshgrid(torch.arange(ws), torch.arange(ws), indexing="ij")).flatten(1)
        rel = coords[:, :, None] - coords[:, None, :] + (ws - 1)
        self.register_buffer("relative_position_index", rel[0] * (2 * ws - 1) + rel[1])
        self.qkv = nn.Linear(dim, 3 * dim)
        self.proj = nn.Linear(dim, dim)

    def forward(self, x, mask=None):
        Bw, N, C = x.shape
        qkv = self.qkv(x).view(Bw, N, 3, self.heads, C // self.heads).permute(2, 0, 3, 1, 4)
        attn = (qkv[0] * self.scale) @ qkv[1].transpose(-2, -1)
        bias = self.relative_position_bias_table[self.relative_position_index.reshape(-1)]
        attn = attn + bias.view(N, N, -1).permute(2, 0, 1)
        if mask is not None:
            nW = mask.shape[0]
            attn = (attn.view(Bw // nW, nW, self.heads, N, N) + mask[None, :, None]).view(-1, self.heads, N, N)
        x = (attn.softmax(-1) @ qkv[2]).transpose(1, 2).reshape(Bw, N, C)
        return self.proj(x)


def _windows(x, ws):  # [B,H,W,C] -> [B*nW, ws*ws, C]
    B, H, W, C = x.shape
    return x.view(B, H // ws, ws, W // ws, ws, C).transpose(2, 3).reshape(-1, ws * ws, C)


def _unwindows(w, ws, B, H, W):
    return w.view(B, H // ws, W // ws, ws, ws, -1).transpose(2, 3).reshape(B, H, W, -1)


class ShiftWindowMSA(nn.Module):
    def __init__(self, dim, heads, ws, shift):
        super().__init__()
        self.ws, self.shift = ws, shift
        self.w_msa = WindowMSA(dim, heads, ws)
        self.drop = MMCVDropPath(0.0)  # stochastic depth of the attention branch (reference :248)

    def forward(self, x, hw):
        B, _, C = x.shape
        H, W = hw
        ws, s = self.ws, self.shift
        x = F.pad(x.view(B, H, W, C), (0, 0, 0, -W % ws, 0, -H % ws))
        Hp, Wp = x.shape[1:3]
        mask = None
        if s > 0:
            x = torch.roll(x, (-s, -s), (1, 2))
            region = torch.zeros(1, Hp, Wp, 1, device=x.device)
            bands = (slice(0, -ws), slice(-ws, -s), slice(-s, None))
            for i, hs in enumerate(bands):
                for j, wsl in enumerate(bands):
                    region[:, hs, wsl] = 3 * i + j
            ids = _windows(region, ws).squeeze(-1)
            mask = (ids[:, None, :] != ids[:, :, None]).to(x.dtype) * -100.0
        y = _unwindows(self.w_msa(_windows(x, ws), mask), ws, B, Hp, Wp)
        if s > 0:
            y = torch.roll(y, (s, s), (1, 2))
        return self.drop(y[:, :H, :W].reshape(B, H * W, C))


class FFN(nn.Module):
    """Keys `layers.0.0.*` / `layers.1.*` as mmcv's FFN lays them out; `dropout_layer`: stochastic depth of the branch."""

    def __init__(self, dim, hidden):
        super().__init__()
        self.layers = nn.Sequential(nn.Sequential(nn.Linear(dim, hidden), nn.GELU(), nn.Dropout(0.0)),
                                    nn.Linear(hidden, dim), nn.Dropout(0.0))
        self.dropout_layer = MMCVDropPath(0.0)

    def forward(self, x, identity):
        return identity + self.dropout_layer(self.layers(x))


class SwinBlock(nn.Module):
    def __init__(self, dim, heads, hidden, ws, shift):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim)
        self.attn = ShiftWindowMSA(dim, heads, ws, ws // 2 if shift else 0)
        self.norm2 = nn.LayerNorm(dim)
        self.ffn = FFN(dim, hidden)

    def set_drop_path_rate(self, rate):
        """Both branches' stochastic-depth rate (reference :412,421: one rate per block)."""
        self.attn.drop.drop_prob = self.ffn.dropout_layer.drop_prob = float(rate)

    def forward(self, x, hw):
        x = x + self.attn(self.norm1(x), hw)
        return self.ffn(self.norm2(x), x)


class SwinStage(nn.Module):
    def __init__(self, dim, heads, hidden, depth, ws, downsample):
        super().__init__()
        self.blocks = nn.ModuleList(SwinBlock(dim, heads, hidden, ws, shift=i % 2 == 1) for i in range(depth))
        self.downsample = downsample

    def forward(self, x, hw):
        for blk in self.blocks:
            x = blk(x, hw)
        if self.downsample is None:
            return x, hw, x, hw
        down, dhw = self.downsample(x, hw)
        return down, dhw, x, hw


class SwinTransformer(nn.Module):
    """`drop_path_rate`: stochastic depth in training mode (mmcv DropPath on both residual branches of every block).  The
    reference class defaults to 0.1; the mirror's factories build at 0, so nothing changes unless a user calls
    `set_drop_path_rate`."""

    def __init__(self, pretrain_img_size=224, in_channels=3, embed_dims=96, patch_size=4, window_size=7,
                 mlp_ratio=4, depths=(2, 2, 6, 2), num_heads=(3, 6, 12, 24), strides=(4, 2, 2, 2),
                 out_indices=(0, 1, 2, 3), pretrain_style="official", pretrained=None, drop_path_rate=0.0, **unused):
        super().__init__()
        self.out_indices = out_indices
        self.patch_embed = PatchEmbed(in_channels, embed_dims, patch_size)
        self.stages = nn.ModuleList()
        dim = embed_dims
        for i, (depth, heads) in enumerate(zip(depths, num_heads)):
            down = PatchMerging(dim, 2 * dim) if i < len(depths) - 1 else None
            self.stages.append(SwinStage(dim, heads, mlp_ratio * dim, depth, window_size, down))
            if down is not None:
                dim *= 2
        self.num_features = [embed_dims * 2 ** i for i in range(len(depths))]
        for i in out_indices:
            self.add_module(f"norm{i}", nn.LayerNorm(self.num_features[i]))
        self.set_drop_path_rate(drop_path_rate)

    def set_drop_path_rate(self, rate):
        """Re-derive every block's stochastic-depth rate from `rate`, as the reference's constructor does (:639-674):
        linspace(0, rate, sum(depths)) over the blocks in order, so block 0 of stage 0 has rate 0 and the last block has
        `rate`.  The reference hands stage i `dpr[:depths[i]]` and then advances `dpr = dpr[depths[i]:]`, a running
        slice.  The rate is the switch: in training mode every block with a rate above 0 draws one mask per branch."""
        blocks = [blk for st in self.stages for blk in st.blocks]
        for blk, r in zip(blocks, torch.linspace(0, rate, len(blocks))):
            blk.set_drop_path_rate(r.item())
        self.drop_path_rate = float(rate)

    def forward(self, x):
        x, hw = self.patch_embed(x)
        outs = []
        for i, stage in enumerate(self.stages):
            x, hw, out, ohw = stage(x, hw)
            if i in self.out_indices:
                out = getattr(self, f"norm{i}")(out)
                outs.append(out.view(-1, *ohw, self.num_features[i]).permute(0, 3, 1, 2).contiguous())
        return outs


def _swin_large(pretrained=None):
    return SwinTransformer(embed_dims=192, depths=(2, 2, 18, 2), num_heads=(6, 12, 24, 48), pretrained=pretrained)


def swin_large_naive_nopretrain():
    """Random-init Swin-L (reference swin.py:780-793) — the factory parity and benchmarks use."""
    return _swin_large()


def swin_large_naive_l4w722422k():
    """Reference :796-810 loads an ImageNet-22k checkpoint from a hard-coded cluster path; here the weights
    arrive through `load_state_dict` (same key layout), so the factory only builds the architecture."""
    return _swin_large()


swin_large_naive_swinlargepreatrain_add = swin_large_naive_l4w722422k
