"""Python handle over the C ABI: packs a head's parameters into the engine and runs the hot path.

PyTorch is used only for device memory (tensors, caching allocator) and the current stream."""
import ctypes as C
from typing import Dict, Optional, Sequence, Tuple

import torch

from . import _cabi
from ._cabi import EngineError  # noqa: F401

# reference state_dict keys (relative to `depth_head.`) the engine consumes — SURVEY.md Appendix A
DENOISER_KEYS = (
    "model.noise_embedding.0.weight", "model.noise_embedding.0.bias", "model.noise_embedding.1.weight",
    "model.noise_embedding.1.bias", "model.noise_embedding.3.weight", "model.noise_embedding.3.bias",
    "model.noise_embedding.4.weight", "model.noise_embedding.4.bias", "model.time_embedding.weight",
    "model.pred.0.weight", "model.pred.0.bias", "model.pred.1.weight", "model.pred.1.bias",
    "model.pred.3.weight", "model.pred.3.bias", "model.pred.4.weight", "model.pred.4.bias")
FUSE_KEYS = ("model.upsample_fuse.convA.conv.weight", "model.upsample_fuse.convA.conv.bias",
             "model.upsample_fuse.convB.conv.weight", "model.upsample_fuse.convB.conv.bias")
ENCODER_KEYS = (
    "depth_transform.conv_transform.0.0.weight", "depth_transform.conv_transform.0.1.weight",
    "depth_transform.conv_transform.0.1.bias", "depth_transform.conv_transform.0.1.running_mean",
    "depth_transform.conv_transform.0.1.running_var", "depth_transform.conv_transform.1.0.weight",
    "depth_transform.conv_transform.1.1.weight", "depth_transform.conv_transform.1.1.bias",
    "depth_transform.conv_transform.1.1.running_mean", "depth_transform.conv_transform.1.1.running_var")
# the encoder's parameters (ENCODER_KEYS without the running statistics): the order of dd_encode_backward's d_enc_params
ENCODER_PARAM_KEYS = tuple(k for k in ENCODER_KEYS if "running" not in k)
_ENCODER_SHAPES = {"depth_transform.conv_transform.0.0.weight": (16, 1, 3, 3),
                   "depth_transform.conv_transform.1.0.weight": (16, 16, 3, 3)}
# shapes of the denoiser's parameters (reference ScheduledCNNRefine, head :336-359) in DENOISER_KEYS + FUSE_KEYS order
_PARAM_SHAPES = {
    "model.noise_embedding.0.weight": (64, 16, 3, 3), "model.noise_embedding.0.bias": (64,),
    "model.noise_embedding.1.weight": (64,), "model.noise_embedding.1.bias": (64,),
    "model.noise_embedding.3.weight": (256, 64, 3, 3), "model.noise_embedding.3.bias": (256,),
    "model.noise_embedding.4.weight": (256,), "model.noise_embedding.4.bias": (256,),
    "model.time_embedding.weight": (1280, 256),
    "model.pred.0.weight": (64, 256, 3, 3), "model.pred.0.bias": (64,), "model.pred.1.weight": (64,),
    "model.pred.1.bias": (64,), "model.pred.3.weight": (16, 64, 3, 3), "model.pred.3.bias": (16,),
    "model.pred.4.weight": (16,), "model.pred.4.bias": (16,),
    "model.upsample_fuse.convA.conv.weight": (256, 256, 3, 3), "model.upsample_fuse.convA.conv.bias": (256,),
    "model.upsample_fuse.convB.conv.weight": (256, 256, 3, 3), "model.upsample_fuse.convB.conv.bias": (256,)}
# the denoiser's GroupNorm(4, C) + ReLU layers in forward order (dd_denoiser_relu_inputs' z_out order): channels
GN_LAYERS = {"noise_embedding.1": 64, "noise_embedding.4": 256, "pred.1": 64, "pred.4": 16}
DECODER_KEYS = (
    "depth_transform.conv_inv_transform.0.weight", "depth_transform.conv_inv_transform.0.bias",
    "depth_transform.conv_inv_transform.1.weight", "depth_transform.conv_inv_transform.1.bias",
    "depth_transform.conv_inv_transform.1.running_mean", "depth_transform.conv_inv_transform.1.running_var",
    "depth_transform.conv_inv_transform.3.0.weight", "depth_transform.conv_inv_transform.3.0.bias")
# the decoder's parameters (DECODER_KEYS without the running statistics): the order of dd_denoise_backward's d_dec_params
DECODER_PARAM_KEYS = tuple(k for k in DECODER_KEYS if "running" not in k)
_DECODER_SHAPES = {"depth_transform.conv_inv_transform.0.weight": (16, 16, 4, 4),
                   "depth_transform.conv_inv_transform.3.0.weight": (1, 16, 3, 3),
                   "depth_transform.conv_inv_transform.3.0.bias": (1,)}

def _conv_bn_keys(prefix):
    return (prefix + "0.weight",) + tuple(prefix + "1." + leaf for leaf in ("weight", "bias", "running_mean", "running_var"))


# The codec's keys per dd_codec_kind (the `ENGINE_KIND` of the depth_transform classes): (encoder, decoder).  Kind 0 is
# the default codec's ENCODER_KEYS / DECODER_KEYS.
_T, _IT = "depth_transform.conv_transform.", "depth_transform.conv_inv_transform."
CODEC_KEYS = {
    0: (ENCODER_KEYS, DECODER_KEYS),
    1: ((_T + "0.weight", _T + "1.weight"), DECODER_KEYS),
    2: (_conv_bn_keys(_T + "0.") + _conv_bn_keys(_T + "1.") + _conv_bn_keys(_T + "2."),
        (_IT + "0.weight", _IT + "0.bias", _IT + "1.weight", _IT + "1.bias") +
        tuple(_IT + "2." + leaf for leaf in ("weight", "bias", "running_mean", "running_var")) +
        (_IT + "4.0.weight", _IT + "4.0.bias")),
    3: (ENCODER_KEYS, _conv_bn_keys(_IT + "0.") + _conv_bn_keys(_IT + "1.")),
}
CODEC_UP = {0: 2, 1: 2, 2: 4, 3: 1}  # the decoder's upsampling: decoded map [B, 1, u h, u w]
# keys `DenoiseEngine.update_weights` re-packs in place (the denoiser and the depth codec); the neck, FPN and backbone
# packs are rebuilt by `load_weights` only
UPDATABLE_PREFIXES = ("model.", "depth_transform.conv_inv_transform.", "depth_transform.conv_transform.")


def is_updatable(key: str) -> bool:
    return key.startswith(UPDATABLE_PREFIXES)


def _ptr(t: Optional[torch.Tensor]) -> C.c_void_p:
    """The device pointer the C ABI takes for a tensor; NULL for None."""
    return C.c_void_p(0 if t is None else t.data_ptr())


def _f32(t: Optional[torch.Tensor], device) -> Optional[torch.Tensor]:
    """t as a contiguous fp32 tensor on device, copied only when it is not one already; None stays None."""
    return None if t is None else t.detach().to(device, torch.float32).contiguous()


def ddim_coefficients(alphas_cumprod: torch.Tensor, num_inference_steps: int, num_train_timesteps: int,
                      final_alpha_cumprod: float = 1.0) -> Tuple[list, list, list]:
    """Timesteps of `DDIMScheduler.set_timesteps` (reference scheduling_ddim.py:215-229) and the two scalars
    that `DDIMScheduler.step` (:285-326, eta=0, epsilon prediction, no clipping) reduces to:
        x_{t-1} = c_x * x_t + c_eps * eps,
        c_x = sqrt(a_prev / a_t),  c_eps = sqrt(1 - a_prev) - sqrt(a_prev * (1 - a_t) / a_t)
    evaluated in fp64 from the scheduler's fp32 `alphas_cumprod` table (SURVEY.md §3.3)."""
    ratio = num_train_timesteps // num_inference_steps
    ts = [int(round(i * ratio)) for i in range(num_inference_steps)][::-1]
    acp = alphas_cumprod.detach().to("cpu", torch.float64)
    cx, ce = [], []
    for t in ts:
        prev = t - ratio
        a_t = float(acp[t])
        a_p = float(acp[prev]) if prev >= 0 else float(final_alpha_cumprod)
        cx.append((a_p / a_t) ** 0.5)
        ce.append((1.0 - a_p) ** 0.5 - (a_p * (1.0 - a_t) / a_t) ** 0.5)
    return ts, cx, ce


class _DeviceDoubles:
    """`count` fp64 values at device address `ptr`, viewable as a tensor through __cuda_array_interface__."""

    def __init__(self, ptr: int, count: int):
        self.__cuda_array_interface__ = {"shape": (int(count),), "typestr": "<f8", "data": (int(ptr), False),
                                         "version": 3, "strides": None}


class WorkspacePool:
    """One growing device buffer shared by several engines that never run concurrently (the engines of one head):
    a ragged last batch or a second image size then costs packed weights only, not another workspace (1.3 GB at C3)."""

    def __init__(self, device):
        self.device, self.buf = torch.device(device), None

    def get(self, nbytes: int) -> torch.Tensor:
        if self.buf is None or self.buf.numel() < nbytes:
            self.buf = None  # release before growing
            self.buf = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        return self.buf


class DenoiseEngine:
    """One engine per (device, geometry).  `variant`: 'swin' (cond at half the latent resolution, bilinear
    upsample + convA/convB) or 'res' (cond at latent resolution)."""

    def __init__(self, variant: str, batch: int, latent_hw: Sequence[int], cond_hw: Sequence[int],
                 num_inference_steps: int, device: torch.device, cuda_graph: bool = True,
                 simt_conv: bool = False, check_range: bool = False, halo_conv: bool = True,
                 swap_narrow: bool = True, pair_wide: bool = True, step_decode: bool = False, workspace_pool=None,
                 fp8_corr: bool = True, backward: bool = False, loop_backward: bool = False,
                 chain_pred: bool = False, producer_train: bool = False, codec_kind: int = 0):
        self.lib = _cabi.load_library()
        device = torch.device(device)
        if device.type != "cuda":
            raise EngineError("DenoiseEngine runs on CUDA (sm_90a) only; there is no CPU path")
        self.device = device
        self.variant = variant
        self.batch, self.latent_hw, self.cond_hw = int(batch), tuple(latent_hw), tuple(cond_hw)
        self.steps = int(num_inference_steps)
        flags = (_cabi.FLAG_CUDA_GRAPH if cuda_graph else 0) | (_cabi.FLAG_SIMT_CONV if simt_conv else 0) | \
                (_cabi.FLAG_CHECK_RANGE if check_range else 0) | (_cabi.FLAG_HALO_CONV if halo_conv else 0) | \
                (_cabi.FLAG_SWAP_NARROW if swap_narrow else 0) | (_cabi.FLAG_PAIR_WIDE if pair_wide else 0) | \
                (_cabi.FLAG_STEP_DECODE if step_decode else 0) | (_cabi.FLAG_FP8_CORR if fp8_corr else 0) | \
                (_cabi.FLAG_BACKWARD if backward else 0) | (_cabi.FLAG_LOOP_BACKWARD if loop_backward else 0) | \
                (_cabi.FLAG_CHAIN_PRED if chain_pred else 0) | (_cabi.FLAG_PRODUCER_TRAIN if producer_train else 0)
        if codec_kind not in CODEC_KEYS:
            raise EngineError(f"unknown codec kind {codec_kind}")
        flags |= int(codec_kind) << _cabi.FLAG_CODEC_SHIFT
        self.codec_kind = int(codec_kind)
        self.up = CODEC_UP[self.codec_kind]  # decoded map [B, 1, up h, up w]
        self.producer_train = bool(producer_train)
        self.fp8_corr = bool(fp8_corr)
        self.backward = bool(backward or loop_backward)  # the loop backward includes the operator's
        self.loop_backward = bool(loop_backward)
        self.step_decode = bool(step_decode)
        cfg = _cabi.DDConfig(_cabi.ABI_VERSION, {"res": _cabi.VARIANT_RES, "swin": _cabi.VARIANT_SWIN}[variant],
                             self.batch, self.latent_hw[0], self.latent_hw[1], self.cond_hw[0], self.cond_hw[1],
                             self.steps, device.index if device.index is not None else torch.cuda.current_device(),
                             flags)
        h = C.c_void_p()
        _cabi.check(self.lib.dd_create(C.byref(cfg), C.byref(h)))
        self._h = h
        self._ws: Optional[torch.Tensor] = None
        self._pool = workspace_pool  # optional WorkspacePool shared by the engines of one head (one buffer per device)
        self._keep = []  # fp32 contiguous copies handed to dd_set_weight must outlive finalize
        self.producers = None
        self.backbone = None
        self.bn_allgather_group = None  # the process group set_bn_allgather installed
        self.bn_allgather_error: Optional[BaseException] = None  # what the last failed gather raised
        self._allgather = None  # the installed ctypes callback: must outlive its installation

    # ---------------------------------------------------------------- setup
    def load_weights(self, tensors: Dict[str, torch.Tensor]):
        enc_keys, dec_keys = CODEC_KEYS[self.codec_kind]
        keys = DENOISER_KEYS + dec_keys + (FUSE_KEYS if self.variant == "swin" else ())
        if all(k in tensors for k in enc_keys):
            keys = keys + enc_keys
        if self.backbone is not None:
            keys = keys + tuple(k for k in tensors if k.startswith("backbone.") and tensors[k].is_floating_point())
        if self.producers is not None:
            keys = keys + tuple(k for k in tensors if k.startswith(("hahineck.", "conv_lateral.", "conv_up."))
                                and not k.endswith("num_batches_tracked") and tensors[k].dim() <= 4
                                and not k.startswith(("hahineck.multi_att", "hahineck.self_attn",
                                                      "hahineck.reference_points", "hahineck.level_embed")))
        for k in keys:
            if k not in tensors:
                raise EngineError(f"missing parameter {k}")
        self._register((k, tensors[k]) for k in keys)
        _cabi.check(self.lib.dd_finalize_weights(self._h, C.c_void_p(self._stream())))
        self._keep = []

    def update_weights(self, tensors: Dict[str, torch.Tensor]):
        """After `load_weights`: re-pack, in place, what depends on `tensors` — only the parameters / buffers that
        changed, all of them `is_updatable`.  Buffers, TMA descriptors and CUDA graphs are kept (a loop graph is
        captured again only when a conv's power-of-two weight scale changed); the result is bit-identical to a
        `load_weights` of the whole model.  On EngineError the previous pack is intact."""
        known = DENOISER_KEYS + FUSE_KEYS + sum(CODEC_KEYS[self.codec_kind], ())
        for k, v in tensors.items():  # what dd_set_weight would reject, before anything is registered
            if not (k in known or k.startswith(("hahineck.", "conv_lateral.", "conv_up.", "backbone."))) or v.dim() > 4:
                raise EngineError(f"unknown weight key: {k}")
        self._register(tensors.items())
        status = self.lib.dd_update_weights(self._h, C.c_void_p(self._stream()))
        self._keep = []  # still read on the stream: the caching allocator reuses the memory in stream order
        _cabi.check(status)

    def _register(self, items):
        """dd_set_weight for every (key, tensor) of items, from fp32 copies kept in `_keep` for the pack to read."""
        self._keep = []
        for k, v in items:
            t = _f32(v, self.device)
            self._keep.append(t)
            _cabi.check(self.lib.dd_set_weight(self._h, k.encode(), _ptr(t), (C.c_int64 * t.dim())(*t.shape), t.dim()))

    def graph_capture_count(self) -> int:
        """CUDA graph instantiations of this engine so far."""
        return int(self.lib.dd_graph_capture_count(self._h))

    def enable_producers(self, channels, sizes, has_neck: bool):
        """Run the HAHI neck (if any) + FPN natively too; call before load_weights.  `sizes`: [(h, w)] per level."""
        pc = _cabi.DDProducerConfig()
        pc.num_levels = len(channels)
        for i, (c, (hh, ww)) in enumerate(zip(channels, sizes)):
            pc.channels[i], pc.heights[i], pc.widths[i] = int(c), int(hh), int(ww)
        pc.has_neck = 1 if has_neck else 0
        _cabi.check(self.lib.dd_enable_producers(self._h, C.byref(pc)))
        self.producers = (tuple(channels), tuple(tuple(s_) for s_ in sizes), bool(has_neck))
        self._ws = None

    def enable_backbone(self, image_hw, embed_dims=192, depths=(2, 2, 18, 2), num_heads=(6, 12, 24, 48), window=7,
                        kind="swin", mp_dims=(64, 128, 216, 288), mp_paths=(2, 3, 3, 3), mlp_ratio=4,
                        mp_drop_path=(0, 0, 0, 0)):
        """Run the backbone natively as well (after enable_producers, before load_weights).  kind: 'swin' (Swin-L),
        'resnet' (ResNetForMMBEV BasicBlock stages; only `depths` is used) or 'mpvit' (`depths` = encoder layers per
        stage, `mp_dims` / `mp_paths` / `mlp_ratio`).  `mp_drop_path[s]` bit k (MPViT and Swin): block k of stage s
        has stochastic depth, see `set_drop_path`."""
        bc = _cabi.DDBackboneConfig()
        bc.kind, bc.embed_dims, bc.window = {"swin": 1, "resnet": 2, "mpvit": 3}[kind], int(embed_dims), int(window)
        bc.height, bc.width = int(image_hw[0]), int(image_hw[1])
        bc.mlp_ratio = int(mlp_ratio)
        for i in range(4):
            bc.depths[i], bc.num_heads[i] = int(depths[i]), int(num_heads[i])
            bc.mp_dims[i], bc.mp_paths[i] = int(mp_dims[i]), int(mp_paths[i])
            bc.mp_drop_path[i] = int(mp_drop_path[i])
        _cabi.check(self.lib.dd_enable_backbone(self._h, C.byref(bc)))
        self.backbone = (tuple(image_hw), int(embed_dims))
        self._ws = None

    def set_schedule(self, timesteps, c_x, c_eps, sigma=None):
        """The loop's timesteps and fp64 step coefficients (`DDIMScheduler.fused_coefficients`); `sigma` (per step,
        optional) makes it the stochastic step of eta > 0, which needs `variance_noise` on every denoise call."""
        n = len(timesteps)
        ts, cx, ce = (C.c_int64 * n)(*[int(t) for t in timesteps]), (C.c_double * n)(*c_x), (C.c_double * n)(*c_eps)
        if sigma is None:
            _cabi.check(self.lib.dd_set_schedule(self._h, ts, cx, ce, n))
        else:
            _cabi.check(self.lib.dd_set_schedule_eta(self._h, ts, cx, ce, (C.c_double * n)(*sigma), n))

    # ---------------------------------------------------------------- calls
    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def _workspace(self) -> torch.Tensor:
        need = int(self.lib.dd_workspace_bytes(self._h))
        if self._pool is not None:
            return self._pool.get(need + 1024)
        if self._ws is None or self._ws.numel() < need + 1024:
            self._ws = torch.empty(need + 1024, dtype=torch.uint8, device=self.device)
        return self._ws

    @staticmethod
    def _aligned(ws: torch.Tensor) -> int:
        return (ws.data_ptr() + 1023) // 1024 * 1024

    def _ws_args(self):
        """The last three arguments of every entry that runs on the engine's workspace: its 1024-byte aligned start,
        the bytes usable from there, the current stream."""
        ws = self._workspace()
        return C.c_void_p(self._aligned(ws)), ws.numel() - 1024, C.c_void_p(self._stream())

    def _check_in(self, t: torch.Tensor, shape):
        if t.device != self.device or t.dtype != torch.float32 or not t.is_contiguous() or tuple(t.shape) != tuple(shape):
            raise EngineError(f"expected contiguous fp32 {tuple(shape)} on {self.device}, got {tuple(t.shape)} "
                              f"{t.dtype} {t.device}")

    def run_backbone(self, rgb: torch.Tensor, want_feats=False):
        """rgb [B,3,H,W] -> the four Swin stage outputs, left inside the workspace for `build_condition(None)`;
        `want_feats` also returns them as fp32 NCHW tensors."""
        if self.backbone is None:
            raise EngineError("enable_backbone() was not called")
        self._check_in(rgb, (self.batch, 3, *self.backbone[0]))
        chans, sizes, _ = self.producers
        feats = [torch.empty(self.batch, c, *hw, device=self.device) for c, hw in zip(chans, sizes)] if want_feats else None
        ptrs = (C.c_void_p * 4)(*[f.data_ptr() for f in feats]) if want_feats else None
        _cabi.check(self.lib.dd_run_backbone(self._h, _ptr(rgb), ptrs, *self._ws_args()))
        return feats

    def build_condition(self, feats, want_cond=False):
        """Backbone feature maps (fp32 NCHW, finest first) -> condition map, natively (neck + FPN).  The result
        stays inside the workspace for the next `denoise_decode(None, noise)`; `want_cond` also returns it."""
        if self.producers is None:
            raise EngineError("enable_producers() was not called")
        chans, sizes, _ = self.producers
        ptrs = None
        if feats is not None:
            for f, c, hw in zip(feats, chans, sizes):
                self._check_in(f, (self.batch, c, *hw))
            ptrs = (C.c_void_p * 4)(*([f.data_ptr() for f in feats] + [0] * (4 - len(feats))))
        cond = torch.empty(self.batch, 256, *self.cond_hw, device=self.device) if want_cond else None
        _cabi.check(self.lib.dd_build_condition(self._h, ptrs, _ptr(cond), *self._ws_args()))
        return cond

    def _step_io(self, variance_noise: Optional[torch.Tensor], latent_steps: Optional[torch.Tensor]):
        """dd_set_step_io for the next denoise call: the [T,B,16,h,w] noise of a stochastic schedule and / or the
        buffer that receives the latent after every step."""
        shape = (self.steps, self.batch, 16, *self.latent_hw)
        for t in (variance_noise, latent_steps):
            if t is not None:
                self._check_in(t, shape)
        _cabi.check(self.lib.dd_set_step_io(self._h, _ptr(variance_noise), _ptr(latent_steps)))

    def denoise_decode(self, cond: Optional[torch.Tensor], noise: torch.Tensor, want_latent=False, want_logits=False,
                       variance_noise: Optional[torch.Tensor] = None, latent_steps: Optional[torch.Tensor] = None):
        """cond [B,256,hc,wc] (or None right after build_condition), noise [B,16,h,w] -> depth [B,1,u h,u w]
        (u = `self.up`, the codec's upsampling; + latent [B,16,h,w], logits).  `variance_noise` [T,B,16,h,w]: z_t of
        every step, required by a schedule set with sigma (eta > 0); `latent_steps` [T,B,16,h,w] (optional) receives
        the latent after every step (the call then runs without its CUDA graph)."""
        B, (h, w), u = self.batch, self.latent_hw, self.up
        if cond is not None:
            self._check_in(cond, (B, 256, *self.cond_hw))
        self._check_in(noise, (B, 16, h, w))
        depth = torch.empty(B, 1, u * h, u * w, device=self.device, dtype=torch.float32)
        latent = torch.empty(B, 16, h, w, device=self.device, dtype=torch.float32) if want_latent else None
        logits = torch.empty_like(depth) if want_logits else None
        self._step_io(variance_noise, latent_steps)
        _cabi.check(self.lib.dd_denoise_decode(self._h, _ptr(cond), _ptr(noise), _ptr(latent), _ptr(logits), _ptr(depth),
                                               *self._ws_args()))
        return depth, latent, logits

    def denoise_decode_steps(self, cond: Optional[torch.Tensor], noise: torch.Tensor, want_latent=False,
                             want_logits=False, variance_noise: Optional[torch.Tensor] = None):
        """As `denoise_decode`, additionally decoding the latent after every step inside the captured graph (the *Vis
        heads' `pred_inter`): returns (depth_steps [T,B,1,u h,u w], latent, logits of the final step)."""
        if not self.step_decode:
            raise EngineError("engine was created without step_decode=True")
        B, (h, w), u = self.batch, self.latent_hw, self.up
        if cond is not None:
            self._check_in(cond, (B, 256, *self.cond_hw))
        self._check_in(noise, (B, 16, h, w))
        steps = torch.empty(self.steps, B, 1, u * h, u * w, device=self.device, dtype=torch.float32)
        latent = torch.empty(B, 16, h, w, device=self.device, dtype=torch.float32) if want_latent else None
        logits = torch.empty(B, 1, u * h, u * w, device=self.device, dtype=torch.float32) if want_logits else None
        self._step_io(variance_noise, None)
        _cabi.check(self.lib.dd_denoise_decode_steps(self._h, _ptr(cond), _ptr(noise), _ptr(latent), _ptr(logits),
                                                     _ptr(steps), *self._ws_args()))
        return steps, latent, logits

    def denoiser_forward(self, cond: torch.Tensor, noisy: torch.Tensor, t) -> torch.Tensor:
        """eps = ScheduledCNNRefine(noisy, t, cond); t: int or per-image sequence."""
        B, (h, w) = self.batch, self.latent_hw
        self._check_in(cond, (B, 256, *self.cond_hw))
        self._check_in(noisy, (B, 16, h, w))
        ts = self._timesteps(t)
        eps = torch.empty_like(noisy)
        _cabi.check(self.lib.dd_denoiser_forward(self._h, _ptr(cond), _ptr(noisy), (C.c_int64 * B)(*ts), _ptr(eps),
                                                 *self._ws_args()))
        return eps

    def _timesteps(self, t):
        B = self.batch
        ts = [int(t)] * B if not hasattr(t, "__len__") else [int(v) for v in t]
        return ts * B if len(ts) == 1 else ts

    def denoiser_backward(self, cond: torch.Tensor, noisy: torch.Tensor, t, d_eps: torch.Tensor, want_cond=True,
                          want_noisy=True, want_params=True):
        """Gradients of eps = ScheduledCNNRefine(noisy, t, cond) given d_eps = dL/d eps (engine created with
        backward=True): (d_cond or None, d_noisy or None, {reference key relative to `depth_head.`: gradient}).
        time_embedding.weight's gradient is dense [1280, 256]; rows used by several images are summed in image order."""
        if not self.backward:
            raise EngineError("engine was created without backward=True")
        B, (h, w) = self.batch, self.latent_hw
        self._check_in(cond, (B, 256, *self.cond_hw))
        self._check_in(noisy, (B, 16, h, w))
        self._check_in(d_eps, (B, 16, h, w))
        ts = self._timesteps(t)
        d_cond = torch.empty_like(cond) if want_cond else None
        d_noisy = torch.empty_like(noisy) if want_noisy else None
        keys = DENOISER_KEYS + (FUSE_KEYS if self.variant == "swin" else ())
        grads = {}
        if want_params:
            for k in keys:
                grads[k] = torch.empty(_PARAM_SHAPES[k], device=self.device, dtype=torch.float32)
        ptrs = (C.c_void_p * len(keys))(*[grads[k].data_ptr() if k in grads else 0 for k in keys])
        _cabi.check(self.lib.dd_denoiser_backward(self._h, _ptr(cond), _ptr(noisy), (C.c_int64 * B)(*ts), _ptr(d_eps),
                                                  _ptr(d_cond), _ptr(d_noisy), ptrs, *self._ws_args()))
        return d_cond, d_noisy, grads

    def denoiser_relu_inputs(self, cond: torch.Tensor, noisy: torch.Tensor, t) -> Dict[str, torch.Tensor]:
        """The inputs of the denoiser's four ReLUs, z = GroupNorm(y) [B,C,h,w], as `denoiser_backward` recomputes them
        (engine created with backward=True): {GroupNorm layer name: z}, in GN_LAYERS order.  z > 0 is exactly the mask
        that backward applies."""
        if not self.backward:
            raise EngineError("engine was created without backward=True")
        B, (h, w) = self.batch, self.latent_hw
        self._check_in(cond, (B, 256, *self.cond_hw))
        self._check_in(noisy, (B, 16, h, w))
        ts = self._timesteps(t)
        z = {k: torch.empty(B, c, h, w, device=self.device, dtype=torch.float32) for k, c in GN_LAYERS.items()}
        _cabi.check(self.lib.dd_denoiser_relu_inputs(self._h, _ptr(cond), _ptr(noisy), (C.c_int64 * B)(*ts),
                                                     (C.c_void_p * 4)(*[v.data_ptr() for v in z.values()]),
                                                     *self._ws_args()))
        return z

    def _grad_buffers(self, keys, shapes, default=None):
        grads = {k: torch.empty(shapes.get(k, default), device=self.device, dtype=torch.float32) for k in keys}
        return grads, (C.c_void_p * len(keys))(*[grads[k].data_ptr() for k in keys])

    def denoise_backward(self, cond: Optional[torch.Tensor], noise: torch.Tensor, d_depth: Optional[torch.Tensor],
                         d_latent: Optional[torch.Tensor], want_latents=False, want_cond=True, want_noise=True,
                         want_params=True):
        """Gradients of (depth, latent) = denoise_decode(cond, noise) through all T steps and the decoder (engine
        created with loop_backward=True), given d_depth [B,1,2h,2w] and / or d_latent [B,16,h,w]:
        (d_cond or None, d_noise or None, {reference key relative to `depth_head.`: gradient} for the denoiser and the
        decoder parameters, latents [T+1,B,16,h,w] (x_T .. x_0 as recomputed) or None).  time_embedding.weight's
        gradient is dense [1280, 256].  `cond` may be None right after build_condition."""
        if not self.loop_backward:
            raise EngineError("engine was created without loop_backward=True")
        if d_depth is None and d_latent is None:
            raise EngineError("denoise_backward needs d_depth or d_latent")
        B, (h, w) = self.batch, self.latent_hw
        if cond is not None:
            self._check_in(cond, (B, 256, *self.cond_hw))
        self._check_in(noise, (B, 16, h, w))
        if d_depth is not None:
            self._check_in(d_depth, (B, 1, self.up * h, self.up * w))
        if d_latent is not None:
            self._check_in(d_latent, (B, 16, h, w))
        d_cond = torch.empty(B, 256, *self.cond_hw, device=self.device) if want_cond else None
        d_noise = torch.empty_like(noise) if want_noise else None
        latents = torch.empty(self.steps + 1, B, 16, h, w, device=self.device) if want_latents else None
        keys = DENOISER_KEYS + (FUSE_KEYS if self.variant == "swin" else ())
        grads, ptrs = self._grad_buffers(keys if want_params else (), _PARAM_SHAPES)
        dgrads, dptrs = self._grad_buffers(DECODER_PARAM_KEYS if want_params else (), _DECODER_SHAPES, (16,))
        _cabi.check(self.lib.dd_denoise_backward(
            self._h, _ptr(cond), _ptr(noise), _ptr(d_depth), _ptr(d_latent), _ptr(d_cond), _ptr(d_noise),
            ptrs if want_params else None, dptrs if want_params else None, _ptr(latents), *self._ws_args()))
        grads.update(dgrads)
        return d_cond, d_noise, grads, latents

    def decode_backward(self, latent: torch.Tensor, d_depth: torch.Tensor, want_latent=True, want_params=True):
        """Gradients of depth = decode(latent) given d_depth [B,1,2h,2w] (engine created with loop_backward=True):
        (d_latent or None, {decoder key relative to `depth_head.`: gradient})."""
        if not self.loop_backward:
            raise EngineError("engine was created without loop_backward=True")
        B, (h, w) = self.batch, self.latent_hw
        self._check_in(latent, (B, 16, h, w))
        self._check_in(d_depth, (B, 1, self.up * h, self.up * w))
        d_latent = torch.empty_like(latent) if want_latent else None
        grads, ptrs = self._grad_buffers(DECODER_PARAM_KEYS if want_params else (), _DECODER_SHAPES, (16,))
        _cabi.check(self.lib.dd_decode_backward(self._h, _ptr(latent), _ptr(d_depth), _ptr(d_latent),
                                                ptrs if want_params else None, *self._ws_args()))
        return d_latent, grads

    def encode(self, depth: torch.Tensor) -> torch.Tensor:
        """latent = depth_transform.t(depth): [B,1,H,W] -> [B,16,h,w], the codec's latent grid of H x W (the default
        codec: ceil(H/2) x ceil(W/2))."""
        B, (h, w) = self.batch, self.latent_hw
        H, W = depth.shape[-2:]
        self._check_in(depth, (B, 1, H, W))
        out = torch.empty(B, 16, h, w, device=self.device, dtype=torch.float32)
        _cabi.check(self.lib.dd_encode(self._h, _ptr(depth), H, W, _ptr(out), C.c_void_p(self._stream())))
        return out

    def encode_backward(self, depth: torch.Tensor, d_latent: torch.Tensor, want_params=True) -> Dict[str, torch.Tensor]:
        """Gradients of latent = encode(depth) given d_latent [B,16,h,w], in the current codec mode (engine created with
        backward=True or loop_backward=True): {encoder key relative to `depth_head.`: gradient} (ENCODER_PARAM_KEYS;
        empty without `want_params`).  In training mode it differentiates through the batch statistics and records
        nothing: `codec_batch_stats` still reports the last forward.  No gradient with respect to depth."""
        if not self.backward:
            raise EngineError("engine was created without backward=True or loop_backward=True")
        B, (h, w) = self.batch, self.latent_hw
        H, W = depth.shape[-2:]
        self._check_in(depth, (B, 1, H, W))
        self._check_in(d_latent, (B, 16, h, w))
        grads, ptrs = self._grad_buffers(ENCODER_PARAM_KEYS if want_params else (), _ENCODER_SHAPES, (16,))
        _cabi.check(self.lib.dd_encode_backward(self._h, _ptr(depth), H, W, _ptr(d_latent),
                                                ptrs if want_params else None, *self._ws_args()))
        return grads

    def set_codec_mode(self, training: bool):
        """The depth codec's BatchNorms on batch statistics (`training`, as torch's BatchNorm2d in training mode) or on
        their running statistics (the default) for every later encode / decode / denoise_decode(_steps) and their
        backward.  The engine never updates running statistics; `codec_batch_stats` returns what a caller needs to."""
        _cabi.check(self.lib.dd_set_codec_mode(self._h, _cabi.CODEC_TRAIN if training else _cabi.CODEC_EVAL))

    def codec_batch_stats(self) -> torch.Tensor:
        """[n, 2, 16]: (batch mean, unbiased batch variance) of every codec BatchNorm the last forward call evaluated in
        training mode, in evaluation order (decode: 1, denoise_decode_steps: T, encode: 2; n = 0 after an eval-mode
        call).  Ordered on the current stream; no synchronisation."""
        out = torch.empty(max(self.steps, 2), 2, 16, device=self.device, dtype=torch.float32)
        n = C.c_int32()
        _cabi.check(self.lib.dd_codec_batch_stats(self._h, _ptr(out), out.shape[0], C.byref(n), C.c_void_p(self._stream())))
        return out[:n.value]

    def set_producer_mode(self, training: bool):
        """The condition producers' BatchNorms (ResNet backbone, HAHI neck, FPN) on batch statistics (`training`, as
        torch's BatchNorm2d in training mode; engine created with producer_train=True) or on their running statistics
        (the default) for every later run_backbone / build_condition.  The engine never updates running statistics;
        `producer_batch_stats` returns what a caller needs to."""
        _cabi.check(self.lib.dd_set_producer_mode(self._h, _cabi.PRODUCER_TRAIN if training else _cabi.PRODUCER_EVAL))

    def set_drop_path(self, scales: Optional[torch.Tensor]):
        """Stochastic depth of the MPViT or Swin backbone for every later run_backbone (dd_set_drop_path): `scales`
        (fp32 on the engine's device) = mask / keep of every DropPath branch, [block][attention, MLP][B] for the blocks
        `enable_backbone(mp_drop_path=...)` marked, in stage, path, layer order (Swin: stage, block order); copied on
        the current stream.  None turns it off."""
        if scales is None:
            _cabi.check(self.lib.dd_set_drop_path(self._h, None, 0, C.c_void_p(self._stream())))
            return
        if scales.device != self.device or scales.dtype != torch.float32 or not scales.is_contiguous():
            raise EngineError(f"drop-path scales must be contiguous fp32 on {self.device}")
        _cabi.check(self.lib.dd_set_drop_path(self._h, _ptr(scales), scales.numel(), C.c_void_p(self._stream())))

    def _producer_records(self):
        n = C.c_int32()
        _cabi.check(self.lib.dd_producer_batch_stats(self._h, None, 0, C.byref(n), None))
        buf, ch, off, fresh = C.create_string_buffer(256), C.c_int32(), C.c_int64(), C.c_int32()
        info = []
        for i in range(n.value):
            _cabi.check(self.lib.dd_producer_bn_info(self._h, i, buf, 256, C.byref(ch), C.byref(off), C.byref(fresh)))
            info.append((buf.value.decode(), ch.value, off.value, bool(fresh.value)))
        return info

    def producer_bn_keys(self):
        """[(BatchNorm key prefix, channels, offset into the records)] of every BatchNorm'ed producer layer, in
        evaluation order (empty without producer_train=True)."""
        return [(k, c, o) for k, c, o, _ in self._producer_records()]

    def producer_batch_stats(self) -> Dict[str, Tuple[torch.Tensor, torch.Tensor]]:
        """{BatchNorm key prefix: (batch mean [C], unbiased batch variance [C])} of every producer BatchNorm the forward
        that last started (run_backbone, or build_condition with feature maps) evaluated in training mode, in
        evaluation order.  Ordered on the current stream; no synchronisation."""
        info = self._producer_records()
        total = max((o + 2 * c for _, c, o, _ in info), default=0)
        if total == 0:
            return {}
        rec = torch.empty(total, device=self.device, dtype=torch.float32)
        n = C.c_int32()
        _cabi.check(self.lib.dd_producer_batch_stats(self._h, _ptr(rec), total, C.byref(n), C.c_void_p(self._stream())))
        return {k: (rec[o:o + c], rec[o + c:o + 2 * c]) for k, c, o, f in info if f}

    def set_bn_allgather(self, group):
        """Synchronised BatchNorm (dd_set_bn_allgather): with a torch.distributed process group, every BatchNorm this
        engine runs on batch statistics (`set_codec_mode(True)`, `set_producer_mode(True)`) normalises with the
        statistics of all the group's ranks' batches together, and every rank gets the same records bit for bit.  Every
        rank must then make the same engine calls in the same order.  NCCL gathers on the engine's stream, other
        backends (gloo) through host memory.  None (the default) turns it off.  A gather that raises fails the engine
        call with EngineError (the exception is kept in `bn_allgather_error`); the engine stays usable."""
        if group is None:
            _cabi.check(self.lib.dd_set_bn_allgather(self._h, _cabi.ALLGATHER_FN(), None, 0))
            self._allgather, self.bn_allgather_group = None, None
            return
        import torch.distributed as dist
        world = dist.get_world_size(group)
        nccl = dist.get_backend(group) == "nccl"
        device = self.device

        def gather(inp, out, count, stream, _user):
            try:
                src = torch.as_tensor(_DeviceDoubles(inp, count), device=device)
                dst = torch.as_tensor(_DeviceDoubles(out, world * count), device=device)
                cur = torch.cuda.current_stream(device)
                st = cur if cur.cuda_stream == (stream or 0) else torch.cuda.ExternalStream(stream, device=device)
                with torch.cuda.stream(st):
                    if nccl:
                        dist.all_gather_into_tensor(dst, src, group=group)
                    else:  # synchronous copies through the host, in order on the engine's stream
                        rows = [torch.empty(count, dtype=torch.float64) for _ in range(world)]
                        dist.all_gather(rows, src.cpu(), group=group)
                        dst.copy_(torch.cat(rows))
                return 0
            except Exception as e:  # noqa: BLE001 - any failure becomes the engine call's error
                self.bn_allgather_error = e
                return 1

        fn = _cabi.ALLGATHER_FN(gather)
        _cabi.check(self.lib.dd_set_bn_allgather(self._h, fn, None, world))
        self._allgather, self.bn_allgather_group = fn, group

    def decode(self, latent: torch.Tensor, want_logits=False):
        B, (h, w), u = self.batch, self.latent_hw, self.up
        self._check_in(latent, (B, 16, h, w))
        depth = torch.empty(B, 1, u * h, u * w, device=self.device, dtype=torch.float32)
        logits = torch.empty_like(depth) if want_logits else None
        _cabi.check(self.lib.dd_decode(self._h, _ptr(latent), _ptr(logits), _ptr(depth), *self._ws_args()))
        return depth, logits

    def conv3x3(self, x: torch.Tensor, w: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
        """Single 3x3/s1/p1 conv + bias on the engine's convolution path (parity tests, roofline)."""
        B, cin, H, W = x.shape
        cout = w.shape[0]
        x, w, b = (_f32(t, self.device) for t in (x, w, b))
        y = torch.empty(B, cout, H, W, device=self.device, dtype=torch.float32)
        need = int(self.lib.dd_conv3x3_workspace_bytes(B, cin, cout, H, W))
        ws = torch.empty(need + 1024, dtype=torch.uint8, device=self.device)
        _cabi.check(self.lib.dd_conv3x3(self._h, _ptr(x), _ptr(w), _ptr(b), _ptr(y), B, cin, cout, H, W,
                                        C.c_void_p(self._aligned(ws)), need, C.c_void_p(self._stream())))
        return y

    def conv3x3_wgrad(self, x: torch.Tensor, dy: torch.Tensor):
        """Weight and bias gradient of that conv on the backward's kernels: x [B,Cin,H,W], dy [B,Cout,H,W] ->
        (dw [Cout,Cin,3,3], db [Cout]).  Raises EngineError (DD_ERR_RANGE) for a non-finite x or dy."""
        B, cin, H, W = x.shape
        cout = dy.shape[1]
        if tuple(dy.shape) != (B, cout, H, W):
            raise EngineError(f"dy {tuple(dy.shape)} does not match x {tuple(x.shape)}")
        x, dy = _f32(x, self.device), _f32(dy, self.device)
        dw = torch.empty(cout, cin, 3, 3, device=self.device, dtype=torch.float32)
        db = torch.empty(cout, device=self.device, dtype=torch.float32)
        need = int(self.lib.dd_conv3x3_wgrad_workspace_bytes(B, cin, cout, H, W))
        ws = torch.empty(need + 1024, dtype=torch.uint8, device=self.device)
        _cabi.check(self.lib.dd_conv3x3_wgrad(self._h, _ptr(x), _ptr(dy), _ptr(dw), _ptr(db), B, cin, cout, H, W,
                                              C.c_void_p(self._aligned(ws)), need, C.c_void_p(self._stream())))
        return dw, db

    def gen_layer(self, x0: torch.Tensor, w: torch.Tensor, x1: Optional[torch.Tensor] = None,
                  bias: Optional[torch.Tensor] = None, bn=None, add: Optional[torch.Tensor] = None,
                  stride: int = 1, transposed: bool = False, act: int = 0, add_first: bool = False, cin: int = 0,
                  ld_out: int = 0, ch_off: int = 0, n_tile: int = 0, alt_tile: int = 0, y32=True, planes=None):
        """One producer layer on the engine's tensor-core conv / GEMM kernel (dd_gen_layer), NHWC in and out.
        x0 [M, c0] (GEMM mode) or [B, Hs, Ws, c0] (conv mode), x1 (second source, concatenated after x0) on the output
        grid; w in the reference layout (Linear [cout, cin], conv [cout, cin, k, k], ConvT [c0, cout, 2, 2]); bn =
        (weight, bias, running_mean, running_var) folded after the conv, else `bias`; `add` the fp32 addend.
        y32 / planes: True allocates the output (planes: fp16 hi / lo at the producers' scale), a tensor (pair) is
        written in place (rows ld_out wide, columns [ch_off, ch_off + cout)), None / False skips it.
        Returns (y32, (hi, lo), {"nt", "work", "grid", "parts"}) with None for a skipped output; "parts" > 1: the
        layer ran split along K."""
        dev = self.device
        x0, x1, w, bias, add = (_f32(t, dev) for t in (x0, x1, w, bias, add))
        bn = None if bn is None else [_f32(t, dev) for t in bn]
        d = _cabi.DDGenLayerDesc()
        d.taps = 1 if (transposed or w.dim() == 2) else w.shape[2] * w.shape[3]
        d.stride, d.transposed, d.act, d.add_first = int(stride), int(transposed), int(act), int(add_first)
        d.c0, d.c1 = x0.shape[-1], (0 if x1 is None else x1.shape[-1])
        d.cin, d.cout = int(cin), (w.shape[1] if transposed else w.shape[0])
        d.ld_out, d.ch_off, d.n_tile, d.alt_tile = int(ld_out), int(ch_off), int(n_tile), int(alt_tile)
        width = int(ld_out) or d.cout
        if x0.dim() == 2:
            d.tokens = x0.shape[0]
            shape = (x0.shape[0], width)
        else:
            d.batch, d.src_h, d.src_w = x0.shape[0], x0.shape[1], x0.shape[2]
            d.height, d.width = (d.src_h, d.src_w) if stride == 1 else ((d.src_h + 1) // 2, (d.src_w + 1) // 2)
            shape = (d.batch, 2 * d.height, 2 * d.width, d.cout) if transposed else (d.batch, d.height, d.width, width)
        if y32 is True:
            y32 = torch.full(shape, float("nan"), device=dev)
        if planes is True:
            planes = tuple(torch.zeros(shape, dtype=torch.float16, device=dev) for _ in range(2))
        y32 = None if y32 is False else y32
        planes = None if planes is False else planes
        info = (C.c_int32 * 4)()
        bn_ptrs = None if bn is None else (C.c_void_p * 4)(*[t.data_ptr() for t in bn])
        _cabi.check(self.lib.dd_gen_layer(self._h, C.byref(d), _ptr(x0), _ptr(x1), _ptr(w), _ptr(bias), bn_ptrs,
                                          _ptr(add), _ptr(y32), _ptr(planes[0] if planes else None),
                                          _ptr(planes[1] if planes else None), info, C.c_void_p(self._stream())))
        return y32, planes, {"nt": info[0], "work": info[1], "grid": info[2], "parts": info[3]}

    def window_attention(self, qkv: torch.Tensor, qkv_bias: torch.Tensor, table: torch.Tensor, batch: int,
                         hw: Sequence[int], num_heads: int, shift: int, kernel: int = 0):
        """Swin (shifted-)window attention on the engine's kernels (dd_window_attention): qkv [B*H*W, 3C] fp32 (padded
        tokens carry qkv_bias [3C]), table [169, nH].  kernel: 0 the engine's choice, 1 fp32 CUDA cores, 2 wgmma.
        Returns (out [B*H*W, C] fp32, {"work", "grid"})."""
        qkv, qkv_bias, table = (_f32(t, self.device) for t in (qkv, qkv_bias, table))
        out = torch.empty(qkv.shape[0], qkv.shape[1] // 3, device=self.device, dtype=torch.float32)
        info = (C.c_int32 * 2)()
        _cabi.check(self.lib.dd_window_attention(self._h, _ptr(qkv), _ptr(qkv_bias), _ptr(table), _ptr(out), int(batch),
                                                 int(hw[0]), int(hw[1]), int(num_heads), int(shift), int(kernel), info,
                                                 C.c_void_p(self._stream())))
        return out, {"work": info[0], "grid": info[1]}

    def factor_attention(self, qkv: torch.Tensor, crpe_w: Sequence[torch.Tensor], crpe_b: Sequence[torch.Tensor],
                         batch: int, hw: Sequence[int]):
        """MPViT's factorised attention with convolutional relative position encoding on the engine's kernels
        (dd_factor_attention; 8 heads, crpe windows {3: 2, 5: 3, 7: 3}): qkv [B*H*W, 3C] fp32, crpe_w / crpe_b the three
        crpe.conv_list weights [nh*Ch, 1, k, k] / biases.  Returns (out [B*H*W, C] fp32, {"tpc", "chunks", "hb",
        "grid"})."""
        qkv = _f32(qkv, self.device)
        crpe_w, crpe_b = [_f32(t, self.device) for t in crpe_w], [_f32(t, self.device) for t in crpe_b]
        out = torch.empty(qkv.shape[0], qkv.shape[1] // 3, device=self.device, dtype=torch.float32)
        info = (C.c_int32 * 4)()
        _cabi.check(self.lib.dd_factor_attention(self._h, _ptr(qkv), (C.c_void_p * 3)(*[t.data_ptr() for t in crpe_w]),
                                                 (C.c_void_p * 3)(*[t.data_ptr() for t in crpe_b]), _ptr(out),
                                                 int(batch), int(hw[0]), int(hw[1]), out.shape[1], info,
                                                 C.c_void_p(self._stream())))
        return out, {"tpc": info[0], "chunks": info[1], "hb": info[2], "grid": info[3]}

    def depthwise_conv(self, x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, bn=None,
                       stride: int = 1, act: int = 0, residual: bool = False, y32=True, planes=False):
        """MPViT's depthwise 3x3 conv on the engine's kernel (dd_depthwise_conv): x [B, H, W, C] fp32 NHWC, w [C, 1, 3,
        3], then bn = (weight, bias, running_mean, running_var) folded or `bias`; act 0 / 3 (Hardswish); residual adds x
        (stride 1).  y32 / planes: True allocates the output (planes: fp16 hi / lo at the producers' scale), False skips
        it.  Returns (y32, (hi, lo), {"grid", "work"}) with None for a skipped output."""
        x, w, bias = (_f32(t, self.device) for t in (x, w, bias))
        bn = None if bn is None else [_f32(t, self.device) for t in bn]
        B, H, W, Cc = x.shape
        shape = (B, (H - 1) // stride + 1, (W - 1) // stride + 1, Cc)
        y32 = torch.full(shape, float("nan"), device=self.device) if y32 else None
        planes = tuple(torch.zeros(shape, dtype=torch.float16, device=self.device) for _ in range(2)) if planes else None
        info = (C.c_int32 * 2)()
        bn_ptrs = None if bn is None else (C.c_void_p * 4)(*[t.data_ptr() for t in bn])
        _cabi.check(self.lib.dd_depthwise_conv(self._h, _ptr(x), _ptr(w), _ptr(bias), bn_ptrs, _ptr(y32),
                                               _ptr(planes[0] if planes else None), _ptr(planes[1] if planes else None),
                                               B, H, W, Cc, int(stride), int(act), int(residual), info,
                                               C.c_void_p(self._stream())))
        return y32, planes, {"grid": info[0], "work": info[1]}

    def layer_norm(self, x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float = 1e-6) -> torch.Tensor:
        """LayerNorm over the last axis on the MPViT encoders' kernel (dd_layer_norm, C <= 512): x [M, C] fp32 ->
        fp32 [M, C], rebuilt from the kernel's hi / lo planes."""
        x, gamma, beta = (_f32(t, self.device) for t in (x, gamma, beta))
        out = torch.empty_like(x)
        _cabi.check(self.lib.dd_layer_norm(self._h, _ptr(x), _ptr(gamma), _ptr(beta), _ptr(out), x.shape[0], x.shape[1],
                                           float(eps), C.c_void_p(self._stream())))
        return out

    def swin_patch_embed(self, rgb: torch.Tensor, w: torch.Tensor, bias: torch.Tensor, gamma: torch.Tensor,
                         beta: torch.Tensor) -> torch.Tensor:
        """Swin's patch embedding on the backbone's kernel (dd_swin_patch_embed, E = 192): rgb [B, 3, H, W] fp32, w [E,
        3, 4, 4] -> 4x4/s4 conv (zero pad right / bottom) + bias + LayerNorm(E) -> fp32 [B * ceil(H/4) * ceil(W/4),
        E]."""
        rgb, w, bias, gamma, beta = (_f32(t, self.device) for t in (rgb, w, bias, gamma, beta))
        B, _, H, W = rgb.shape
        E = w.shape[0]
        out = torch.full((B * ((H + 3) // 4) * ((W + 3) // 4), E), float("nan"), device=self.device)
        _cabi.check(self.lib.dd_swin_patch_embed(self._h, _ptr(rgb), _ptr(w), _ptr(bias), _ptr(gamma), _ptr(beta),
                                                 _ptr(out), B, H, W, E, C.c_void_p(self._stream())))
        return out

    def swin_layer_norm(self, x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, hw: int = 0):
        """Swin's LayerNorm on the backbone's kernel (dd_swin_layer_norm, C in {192, 384, 768, 1536}, eps 1e-5): x
        [M, C] fp32 -> (out [M, C] fp32 rebuilt from the kernel's hi / lo planes, the stage-output copy [M / hw, C, hw]
        fp32 when hw > 0, else None)."""
        x, gamma, beta = (_f32(t, self.device) for t in (x, gamma, beta))
        M, Cc = x.shape
        out = torch.empty_like(x)
        nchw = torch.full((M // hw, Cc, hw), float("nan"), device=self.device) if hw > 0 else None
        _cabi.check(self.lib.dd_swin_layer_norm(self._h, _ptr(x), _ptr(gamma), _ptr(beta), _ptr(out), _ptr(nchw), M,
                                                Cc, int(hw), C.c_void_p(self._stream())))
        return out, nchw

    def swin_patch_merge(self, x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor) -> torch.Tensor:
        """Swin's patch merging on the backbone's kernel (dd_swin_patch_merge, C in {192, 384, 768}): x [B, H, W, C]
        fp32 -> 2x2 unfold (zero pad for odd H / W) + LayerNorm(4C) -> fp32 [B * ceil(H/2) * ceil(W/2), 4C], rebuilt
        from the kernel's hi / lo planes."""
        x, gamma, beta = (_f32(t, self.device) for t in (x, gamma, beta))
        B, H, W, Cc = x.shape
        out = torch.empty(B * ((H + 1) // 2) * ((W + 1) // 2), 4 * Cc, device=self.device)
        _cabi.check(self.lib.dd_swin_patch_merge(self._h, _ptr(x), _ptr(gamma), _ptr(beta), _ptr(out), B, H, W, Cc,
                                                 C.c_void_p(self._stream())))
        return out

    def conv_groupnorm(self, x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, gamma: torch.Tensor,
                       beta: torch.Tensor, mode: int, cond: Optional[torch.Tensor] = None,
                       temb: Optional[torch.Tensor] = None, latent: Optional[torch.Tensor] = None, c_x: float = 0.0,
                       c_eps: float = 0.0, up_qpb: int = 4):
        """One GroupNorm(4, Cout)'d conv of the DDIM loop on the loop's kernels (dd_conv_groupnorm): x [B, Cin, H, W]
        -> conv -> GroupNorm + ReLU, then mode 0 nothing, 1 + cond [B, 256, H, W] + temb [B, 256], 2 + bilinear
        up(cond [B, 256, h, w] + temb), 3 the DDIM update (latent [B, 16, H, W] is updated in place; None: eps only).
        Returns (y32 the conv output, mean_rstd [B, 4, 2], out [B, Cout, H, W])."""
        dev = self.device
        x, w, b, gamma, beta, cond, temb = (_f32(t, dev) for t in (x, w, b, gamma, beta, cond, temb))
        B, cin, H, W = x.shape
        cout = w.shape[0]
        d = _cabi.DDConvGnDesc()
        d.batch, d.cin, d.cout, d.height, d.width, d.mode = B, cin, cout, H, W, int(mode)
        d.cond_h, d.cond_w = (cond.shape[2], cond.shape[3]) if cond is not None else (0, 0)
        d.up_qpb, d.c_x, d.c_eps = int(up_qpb), float(c_x), float(c_eps)
        y32 = torch.full((B, cout, H, W), float("nan"), device=dev)
        mean_rstd = torch.full((B, 4, 2), float("nan"), device=dev)
        out = torch.full((B, cout, H, W), float("nan"), device=dev)
        _cabi.check(self.lib.dd_conv_groupnorm(self._h, C.byref(d), _ptr(x), _ptr(w), _ptr(b), _ptr(gamma), _ptr(beta),
                                               _ptr(cond), _ptr(temb), _ptr(latent), _ptr(y32), _ptr(mean_rstd),
                                               _ptr(out), C.c_void_p(self._stream())))
        return y32, mean_rstd, out

    def bench_conv(self, cin: int, cout: int, iters: int = 20) -> float:
        """Average milliseconds per launch of the (cin -> cout) conv on this engine's latent grid."""
        ms = C.c_float()
        _cabi.check(self.lib.dd_bench_conv(self._h, cin, cout, iters, C.byref(ms), *self._ws_args()))
        return float(ms.value)

    def bench_decoder(self, iters: int = 20) -> float:
        """Average milliseconds per launch of the codec's decoder kernel alone (CUDA events), on the latent the
        workspace holds from the last call."""
        B, (h, w), u = self.batch, self.latent_hw, self.up
        depth = torch.empty(B, 1, u * h, u * w, device=self.device, dtype=torch.float32)
        ms = C.c_float()
        _cabi.check(self.lib.dd_bench_decoder(self._h, _ptr(depth), iters, C.byref(ms), *self._ws_args()))
        return float(ms.value)

    def bench_pred_fold(self, iters: int = 20) -> float:
        """Average milliseconds of the Swin step's composed convB -> pred.0 (5x5 conv + ring correction)."""
        ms = C.c_float()
        _cabi.check(self.lib.dd_bench_pred_fold(self._h, iters, C.byref(ms), *self._ws_args()))
        return float(ms.value)

    def bench_gemm(self, M: int, K: int, N: int, mode: int = 0, iters: int = 20) -> float:
        ms = C.c_float()
        _cabi.check(self.lib.dd_bench_gemm(self._h, M, K, N, mode, iters, C.byref(ms)))
        return float(ms.value)

    def poll_status(self) -> None:
        """Synchronise the current stream; raises EngineError(DD_ERR_RANGE) if the fp16 split overflowed."""
        _cabi.check(self.lib.dd_poll_status(self._h, C.c_void_p(self._stream())))

    @property
    def last_launch_count(self) -> int:
        return int(self.lib.dd_last_launch_count(self._h))

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            self.lib.dd_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # pragma: no cover
            pass
