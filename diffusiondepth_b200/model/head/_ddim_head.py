"""Shared machinery of the DDIM depth heads: parameter containers with the reference's key layout and the
bridge to the CUDA engine.

Reference call chain being replaced (src/model/head/ddim_depth_estimate_res_swin_addHAHI.py):
  forward :87-185  ->  encoder t() :102, hahineck :110, FPN :112-122, pipeline(...) :130-144 =
  CNNDDIMPipiline.__call__ :254-303 (T x {denoiser :361-382, DDIMScheduler.step})  ->  depth_transform.inv_t :146.
Here all of it — and the backbone in front of it — runs inside the CUDA engine (C ABI, include/dd_engine.h) whenever the
engine instantiates the architecture; the torch modules below only hold the parameters under the reference's keys.
The torch-op producer path (TF32 off) remains for architectures the engine does not instantiate.

The engine bits are imported absolutely (`diffusiondepth_b200.*`), everything else relatively, so that this package
works both as `diffusiondepth_b200.model` and as the reference's top-level `model` (INTEGRATION.md: symlink into
`src/`, tested by tests/test_dropin.py)."""
import collections
import copy
import threading
import weakref
from typing import Dict, NamedTuple, Optional, Tuple, Union

import torch
import torch.nn as nn
import torch.nn.functional as F

from diffusiondepth_b200._cabi import EngineError
from diffusiondepth_b200.engine import (CODEC_KEYS, DECODER_KEYS, DECODER_PARAM_KEYS, DENOISER_KEYS, ENCODER_KEYS,
                                        ENCODER_PARAM_KEYS, FUSE_KEYS, DenoiseEngine, WorkspacePool, is_updatable)
from .._blocks import ConvModule, DropPath, MMCVDropPath, exact_fp32
from ..diffusers.schedulers.scheduling_ddim import DDIMScheduler
from ..ops import depth_transform as _codec  # noqa: F401  (registers the codec classes)
from ..registry import DEPTH_TRANSFORM

FPN_DIM = 256
MAX_ENGINES = 4  # per head: least-recently-used engines beyond this are closed (packed weights + CUDA graphs freed)


def collect_tensors(module: nn.Module, prefix: str = "") -> Dict[str, torch.Tensor]:
    """`module.state_dict(keep_vars=True)` that also works on `nn.DataParallel` replicas, whose parameters are plain
    tensor attributes listed in `_former_parameters` (torch/nn/parallel/replicate.py) and absent from `state_dict()`."""
    out: Dict[str, torch.Tensor] = {}

    def walk(m, pre):
        for k, v in m._parameters.items():
            if v is not None:
                out[pre + k] = v
        for k, v in getattr(m, "_former_parameters", {}).items():
            if v is not None:
                out.setdefault(pre + k, v)
        for k, v in m._buffers.items():
            if v is not None and k not in m._non_persistent_buffers_set:
                out[pre + k] = v
        for k, c in m._modules.items():
            if c is not None:
                walk(c, pre + k + ".")

    walk(module, prefix)
    return out


class EngineKey(NamedTuple):
    """What a head's cached engine was created for: geometry, schedule and the creation flags."""
    batch: int
    latent_hw: Tuple[int, int]
    cond_hw: Tuple[int, int]
    device: str
    steps: int
    cuda_graph: bool
    native: bool                          # neck + FPN on the engine
    image_hw: Optional[Tuple[int, int]]   # and the backbone (None: not native)
    step_decode: bool
    producer_train: bool
    backward: bool
    loop_backward: bool
    drop_path: Tuple[int, ...] = ()       # native backbone with stochastic depth: per stage, the bit mask of its MPViT
                                          # layers / Swin blocks (dd_backbone_config.mp_drop_path)
    codec_kind: int = 0                   # the depth codec's dd_codec_kind (`depth_transform.ENGINE_KIND`)
    eta: float = 0.0                      # the DDIM step's eta (> 0: `pipeline(eta=...)`, the stochastic schedule)

    @property
    def geometry(self):
        """What an engine serving the bare operators (denoiser / decode) must match."""
        return self.batch, self.latent_hw, self.cond_hw, self.device, self.steps, self.codec_kind


def _signature(tensors):
    return tuple((t.data_ptr(), t._version) for t in tensors.values())


def repack_plan(old_keys, old_sig, new_keys, new_sig, incremental=True, deferred=None):
    """What an engine packed from tensors `old_keys` with signature `old_sig` (None: never packed) needs to serve the
    tensors `new_keys` / `new_sig`: the list of changed keys for `DenoiseEngine.update_weights` (empty: nothing), or
    None for a full `load_weights` — a different key set, a changed tensor the update does not re-pack (neck, FPN,
    backbone), or `incremental` off.  `deferred` (a predicate on keys, optional): changes of those keys are left out
    of the plan; the caller re-packs them later."""
    if not incremental or old_sig is None or tuple(old_keys) != tuple(new_keys):
        return None
    changed = [k for k, a, b in zip(new_keys, old_sig, new_sig) if a != b and not (deferred and deferred(k))]
    return changed if all(is_updatable(k) for k in changed) else None


_PRODUCER_PREFIXES = ("hahineck.", "conv_lateral.", "conv_up.", "backbone.")


def is_producer_running_stat(key: str) -> bool:
    """A running-statistic buffer of a producer BatchNorm: what the running update of a training-mode forward changes,
    and what the training-mode producers do not read."""
    return key.startswith(_PRODUCER_PREFIXES) and key.endswith((".running_mean", ".running_var", ".num_batches_tracked"))


def _gn_conv_stack(cin, mid, cout):
    """conv3x3 -> GN(4) -> ReLU -> conv3x3 -> GN(4) -> ReLU; indices 0,1,3,4 carry parameters."""
    return nn.Sequential(nn.Conv2d(cin, mid, 3, 1, 1), nn.GroupNorm(4, mid), nn.ReLU(True),
                         nn.Conv2d(mid, cout, 3, 1, 1), nn.GroupNorm(4, cout), nn.ReLU(True))


class UpSample_add(nn.Module):
    """Parameters of the Swin heads' fusion block: convA / convB = bare 3x3 conv + bias (head :321-333)."""

    def __init__(self, cin, cout):
        super().__init__()
        self.convA = ConvModule(cin, cout, 3, padding=1, norm=False, act=False)
        self.convB = ConvModule(cout, cout, 3, padding=1, norm=False, act=False)


class ScheduledCNNRefine(nn.Module):
    """The denoiser's parameters (head :336-359 / res.py:301-322).  It has no torch forward: the operator
    `model(noisy, t, cond, None, None, None) -> eps` is served by the engine (`DenoiseEngine.denoiser_forward`)."""

    def __init__(self, channels_in, channels_noise, with_fuse):
        super().__init__()
        self.noise_embedding = _gn_conv_stack(channels_noise, 64, channels_in)
        if with_fuse:
            self.upsample_fuse = UpSample_add(channels_in, channels_in)
        self.time_embedding = nn.Embedding(1280, channels_in)
        self.pred = _gn_conv_stack(channels_in, 64, channels_noise)
        self.__dict__['_bridge'] = None  # weakref to the owning head, set by it

    def forward(self, noisy_image, t, feat, *unused):
        head = self._bridge() if self._bridge is not None else None
        if head is None:
            raise EngineError("ScheduledCNNRefine is not attached to a DDIM head / CUDA engine")
        return head.denoiser(noisy_image, t, feat)


def _fpn_lateral(cin):
    return nn.Sequential(nn.Conv2d(cin, FPN_DIM, 3, 1, 1, bias=False), nn.BatchNorm2d(FPN_DIM), nn.ReLU(True))


def _fpn_up():
    return nn.Sequential(nn.ConvTranspose2d(FPN_DIM, FPN_DIM, 2, 2, bias=False), nn.BatchNorm2d(FPN_DIM), nn.ReLU(True))


class _DenoiserFunction(torch.autograd.Function):
    """eps = ScheduledCNNRefine(noisy, t, cond) as an autograd node over (noisy, cond, *denoiser parameters).  The forward
    is the head's plain `dd_denoiser_forward` call (eps bit-identical to the no-grad path) and keeps only the inputs; the
    backward runs `dd_denoiser_backward` on an engine of the same geometry created with backward=True, which recomputes
    the activations from those inputs."""

    @staticmethod
    def forward(ctx, head, t, keys, noisy, cond, *params):
        eng = head._any_engine(noisy.shape[0], noisy.shape[-2:], cond.shape[-2:], noisy.device)
        eps = eng.denoiser_forward(cond.contiguous().float(), noisy.contiguous().float(), t)
        ctx.save_for_backward(noisy, cond, *params)
        ctx.head, ctx.t, ctx.keys = head, t, keys
        return eps

    @staticmethod
    def backward(ctx, d_eps):
        noisy, cond = ctx.saved_tensors[:2]
        need = ctx.needs_input_grad
        eng = ctx.head._grad_engine(noisy.shape[0], noisy.shape[-2:], cond.shape[-2:], noisy.device)
        d_cond, d_noisy, grads = eng.denoiser_backward(
            cond.contiguous().float(), noisy.contiguous().float(), ctx.t, d_eps.contiguous().float(),
            want_cond=need[4], want_noisy=need[3], want_params=any(need[5:]))
        return (None, None, None, d_noisy, d_cond) + tuple(grads[k] if need[5 + i] else None for i, k in enumerate(ctx.keys))


class _LoopFunction(torch.autograd.Function):
    """(depth, latent) = inv_t(CNNDDIMPipiline(cond, noise)) as an autograd node over (cond, noise, *denoiser parameters,
    *decoder parameters).  The forward is the head's own `denoise_decode` call on `eng` (with native producers
    cond = None: the condition map is already in the workspace), so both outputs are bit-identical to the no-grad path;
    it keeps cond and noise.  The backward runs `dd_denoise_backward` on an engine of the same geometry created with
    loop_backward=True, which re-runs the loop and walks back through every step and the decoder."""

    @staticmethod
    def forward(ctx, head, eng, box, cond_in_workspace, keys, codec_train, cond, noise, *params):
        eng.set_codec_mode(codec_train)
        depth, latent, logits = eng.denoise_decode(None if cond_in_workspace else cond, noise, want_latent=True,
                                                   want_logits=head.capture_logits)
        box["logits"] = logits
        ctx.save_for_backward(cond, noise)
        ctx.head, ctx.keys, ctx.codec_train = head, keys, codec_train
        ctx.set_materialize_grads(False)
        return depth, latent

    @staticmethod
    def backward(ctx, d_depth, d_latent):
        cond, noise = ctx.saved_tensors
        need = ctx.needs_input_grad
        if d_depth is None and d_latent is None:
            return (None,) * len(need)
        eng = ctx.head._engine(noise.shape[0], noise.shape[-2:], cond.shape[-2:], noise.device, loop_backward=True)
        eng.set_codec_mode(ctx.codec_train)  # differentiate the decoder the forward ran
        d_cond, d_noise, grads, _ = eng.denoise_backward(
            cond.contiguous().float(), noise, None if d_depth is None else d_depth.contiguous().float(),
            None if d_latent is None else d_latent.contiguous().float(),
            want_cond=need[6], want_noise=need[7], want_params=any(need[8:]))
        return (None,) * 6 + (d_cond, d_noise) + tuple(grads[k] if need[8 + i] else None for i, k in enumerate(ctx.keys))


class _EncodeFunction(torch.autograd.Function):
    """gt_map_t = depth_transform.t(depth) as an autograd node over (depth, *encoder parameters).  The forward is the
    head's plain `encode` call on `eng`, in the codec mode the caller set (gt_map_t bit-identical to the no-grad path),
    and keeps depth and that mode; the backward runs `dd_encode_backward` in the same mode on the engine the denoiser
    backward runs on, which recomputes the forward from depth.  Ground truth gets no gradient."""

    @staticmethod
    def forward(ctx, head, eng, keys, codec_train, depth, *params):
        latent = eng.encode(depth)
        ctx.save_for_backward(depth)
        ctx.head, ctx.keys, ctx.codec_train, ctx.cond_hw = head, keys, codec_train, eng.cond_hw
        return latent

    @staticmethod
    def backward(ctx, d_latent):
        depth, = ctx.saved_tensors
        need = ctx.needs_input_grad
        eng = ctx.head._grad_engine(depth.shape[0], d_latent.shape[-2:], ctx.cond_hw, depth.device)
        eng.set_codec_mode(ctx.codec_train)  # differentiate the encoder the forward ran
        grads = eng.encode_backward(depth, d_latent.contiguous().float(), want_params=any(need[5:]))
        return (None,) * 5 + tuple(grads[k] if need[5 + i] else None for i, k in enumerate(ctx.keys))


def bn_running_update(bn: nn.BatchNorm2d, mean: torch.Tensor, var: torch.Tensor):
    """The running-statistic update torch's training-mode BatchNorm (F.batch_norm) makes after one batch with mean `mean`
    and UNBIASED variance `var`: num_batches_tracked += 1, then running = (1 - f) running + f batch with f = momentum,
    or 1 / num_batches_tracked when momentum is None.  Stays on the buffers' device (no synchronisation)."""
    if not bn.track_running_stats:
        return
    with torch.no_grad():
        bn.num_batches_tracked.add_(1)
        f = bn.momentum if bn.momentum is not None else 1.0 / bn.num_batches_tracked.to(bn.running_mean.dtype)
        bn.running_mean.mul_(1 - f).add_(mean.to(bn.running_mean) * f)
        bn.running_var.mul_(1 - f).add_(var.to(bn.running_var) * f)


class DDIMHeadBase(nn.Module):
    """Common ctor surface: HEADS.build(dict(type=..., in_channels, inference_steps, num_train_timesteps,
    depth_feature_dim=16, loss_cfgs, init_cfg=args)) as in reference diffusion_dcbase_model.py:77-91."""

    variant = "res"          # engine variant
    fpn_in_channels = (64, 128, 256, 512)
    has_neck = False         # HAHI neck in front of the FPN (the *HAHI heads)
    return_intermediates = False  # *Vis heads: also decode every intermediate latent -> 'pred_inter'
    # Training through the sampling loop: when True, grad is enabled and a denoiser / decoder parameter (or cond) requires
    # grad, `pred` and the final latent carry the reference's training-graph gradients through all T steps and the
    # decoder (native dd_denoise_backward), so the L1 / L2 depth losses train the head and `ddim_loss` also reaches the
    # loop through its re-noised latent.  Off by default: it changes what `ddim_loss.backward()` costs and computes.
    grad_through_loop = False
    # Training the depth encoder through `gt_map_t`: when True, grad is enabled and an encoder parameter
    # (`depth_transform.conv_transform.*`) requires grad, `gt_map_t` (= `pred_init` = `blur_depth_t`) is the engine's
    # encoding as an autograd node (native dd_encode_backward, in the codec's BatchNorm mode), so `ddim_loss_gt` trains
    # the encoder as well as the denoiser.  Without native producers the engine then encodes too, instead of torch's
    # `t()` under no_grad.  Off by default: `gt_map_t` then carries no gradient.
    grad_through_encoder = False
    # Training-mode BatchNorm in the depth codec (reference `net.train()`): when True and `depth_transform.training`, the
    # engine's encoder and decoder normalise with the statistics of the batch they see, the decoder's gradients flow
    # through those statistics, and every forward applies torch's running-statistic update to the codec's BatchNorm
    # buffers (re-packed by `update_weights` before the next call).  Off by default: the codec then runs on its running
    # statistics in every mode.
    codec_train_bn = False
    # Training-mode BatchNorm in the condition producers (reference `net.train()`): when True, the HAHI neck and the FPN
    # (when `hahineck` / `conv_lateral` are in training mode) and the native ResNet backbone (when it is in training
    # mode) normalise with the statistics of the batch, and every forward applies torch's running-statistic update to
    # their BatchNorm buffers.  Engines are created with DenoiseEngine(producer_train=True).  While they run in training
    # mode those buffer updates do not re-pack; the first eval-mode forward on the engine re-packs once.  An MPViT
    # backbone in training mode runs in torch unless `mpvit_native_train` is set.  Off by default: the producers then run
    # on their running statistics in every mode.
    producer_train_bn = False
    # Training-mode MPViT backbone on the engine (the MPViT head, together with `producer_train_bn`): when True, an MPViT
    # in training mode runs natively as well — its 29 BatchNorms on batch statistics when all are in training mode (on
    # running statistics when all are in eval, `norm_eval`; a mix runs in torch), and stochastic depth on every
    # MHCABlock whose DropPath is in training mode, with the masks drawn on the device in the order torch's forward
    # draws them, so every later random draw is the same as with the torch backbone.  Off by default: a training-mode
    # MPViT then runs in torch under `producer_train_bn`.
    mpvit_native_train = False
    # Synchronised BatchNorm across ranks (reference src/main.py:128, apex `convert_syncbn_model`): a torch.distributed
    # process group, or None (the default: each rank's own batch).  When set, every BatchNorm that `codec_train_bn` /
    # `producer_train_bn` run in training mode normalises with the statistics of all the group's ranks' batches
    # together, its decoder backward reduces over all of them, and every rank records the same statistics, so the
    # running statistics stay identical on every rank.  Every rank must run the same forwards.  The *Vis heads do not
    # support it (their step decodes run inside one CUDA graph).
    bn_sync_group = None

    def __init__(self, in_channels=None, up_scale_factor=1, inference_steps=20, num_train_timesteps=1000,
                 return_indices=None, depth_transform_cfg=None, detach_fp=False, depth_embed_dim=16,
                 depth_feature_dim=16, loss_cfgs=(), init_cfg=None, **unused):
        super().__init__()
        self.init_cfg, self.detach_fp, self.loss_cfgs = init_cfg, detach_fp, list(loss_cfgs)
        self.return_indices = return_indices
        self.depth_embed_dim = depth_embed_dim
        cfg = depth_transform_cfg or dict(type="DeepDepthTransformWithUpsampling", hidden=16, eps=1e-6)
        self.depth_transform = DEPTH_TRANSFORM.build(cfg)
        self.model = ScheduledCNNRefine(FPN_DIM, depth_feature_dim, with_fuse=self.variant == "swin")
        self.model.__dict__['_bridge'] = weakref.ref(self)  # plain attribute: must not register as a submodule
        self.diffusion_inference_steps = inference_steps
        self.scheduler = DDIMScheduler(num_train_timesteps=num_train_timesteps, clip_sample=False)
        self.conv_lateral = nn.ModuleList(_fpn_lateral(c) for c in self.fpn_in_channels)
        self.conv_up = nn.ModuleList(_fpn_up() for _ in self.fpn_in_channels[1:])
        # engine state (not parameters)
        self.eval_ddim_loss = False       # reference computes it in eval too; it is RNG noise there
        self.use_cuda_graph = True
        self.check_range = True
        self.capture_logits = False      # tests: also keep the decoder's pre-sigmoid z of the last forward
        self.native_producers = True     # neck + FPN on the engine's tensor-core conv path when the pyramid allows
        self.incremental_repack = True   # after an optimizer step re-pack only the changed denoiser / codec tensors, in
        #                                  place (DenoiseEngine.update_weights; bit-identical); False: always the full pack
        self.native_backbone = True      # Swin-L backbone on the engine's GEMM/attention path (needs native_producers)
        self.fp8_corrections = True      # accepted and selects nothing on sm_90a: every conv runs the exact 3-pass fp16
        #                                  split (Hopper's e4m3 wgmma accumulates at reduced precision; DESIGN.md §3)
        self.__dict__['_backbone_ref'] = None  # weakref to the model's depth_backbone (Diffusion_DCbase_Model passes the
        #                                        backbone with every call; this is the fallback for direct head calls)
        self.capture_cond = False        # tests: keep the NCHW condition map of the last forward
        self.noise_generator: Optional[torch.Generator] = None
        self._reset_engine_state()

    def _reset_engine_state(self):
        self.__dict__['_engines'] = collections.OrderedDict()  # key -> DenoiseEngine, least recently used first
        self.__dict__['_packed'] = {}                          # key -> (tensor list, signature) of the packed weights
        self.__dict__['_pools'] = {}                           # device -> WorkspacePool
        self.__dict__['_lock'] = threading.RLock()             # nn.DataParallel replicas (threads) share the three dicts
        self.__dict__['_stale'] = set()  # keys of engines whose eval producer pack predates a running-statistic update

    def invalidate_engines(self):
        """Close every engine (call after replacing Parameter OBJECTS; in-place updates, load_state_dict and .to() are
        picked up automatically through data_ptr / _version: a change confined to denoiser / codec tensors is re-packed
        in place by `DenoiseEngine.update_weights`, anything else by a full `load_weights`)."""
        for e in self._engines.values():
            e.close()
        self._reset_engine_state()

    def __deepcopy__(self, memo):
        """copy.deepcopy(model) (EMA / eval copies): the copy gets its own engines, packed from ITS parameters, and its
        denoiser operator bridges to the copy — never to the original's ctypes handles or weights."""
        new = self.__class__.__new__(self.__class__)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            if k in ("_engines", "_packed", "_pools", "_backbone_ref", "_lock", "_stale"):
                continue
            if k == "bn_sync_group":  # a process group is shared, not copied
                new.__dict__[k] = v
                continue
            new.__dict__[k] = copy.deepcopy(v, memo)
        new.__dict__['_backbone_ref'] = None
        new._reset_engine_state()
        new.model.__dict__['_bridge'] = weakref.ref(new)
        return new

    def _replicate_for_data_parallel(self):
        """nn.DataParallel replicas (reference src/main.py:434): same idea — the replica bridges to itself and reads the
        replica's (broadcast) tensors; engines are cached per device in the dict shared with the original."""
        replica = super()._replicate_for_data_parallel()
        replica.__dict__['_backbone_ref'] = None
        return replica

    @property
    def pipeline(self) -> "CNNDDIMPipiline":
        """The reference's sampler object (`self.pipeline = CNNDDIMPipiline(self.model, self.scheduler)`, head :49),
        built on each access: it holds nothing but this head's `model` and `scheduler`, so deep copies and DataParallel
        replicas get their own."""
        pipe = CNNDDIMPipiline(self.model, self.scheduler, image_list=self.return_intermediates)
        pipe._head = self
        return pipe

    # ------------------------------------------------------------------------------------------ engine bridge
    def _engine_tensors(self):
        sd = {}
        enc_keys, dec_keys = CODEC_KEYS[self._codec_kind()]
        for k in DENOISER_KEYS + dec_keys + enc_keys + (FUSE_KEYS if self.variant == "swin" else ()):
            mod, _, leaf = k.rpartition(".")
            obj = self.get_submodule(mod)
            sd[k] = getattr(obj, leaf)
        return sd

    def _codec_kind(self) -> int:
        """The engine's dd_codec_kind for `depth_transform`: one of the four learned codecs, with hidden = 16 (the
        denoiser's `channels_noise`)."""
        dt = self.depth_transform
        kind = getattr(dt, "ENGINE_KIND", None)
        if kind is None:
            raise EngineError(f"{type(dt).__name__} has no engine codec: the DDIM heads denoise a 16-channel latent "
                              "of a learned depth transform")
        hidden = next(m.out_channels for m in dt.conv_transform.modules() if isinstance(m, nn.Conv2d))
        if hidden != 16:
            raise EngineError(f"{type(dt).__name__}(hidden={hidden}): the engine's latent has 16 channels (the "
                              "denoiser's channels_noise)")
        return kind

    def _check_codec_trains(self):
        """Training the codec on the engine (batch-statistics BatchNorms, encoder / decoder backward) exists for the
        default codec only."""
        if self._codec_kind() == 0:
            return
        name = type(self.depth_transform).__name__
        if self.grad_through_loop:
            raise EngineError(f"grad_through_loop: no decoder backward for {name} on the engine")
        if self.grad_through_encoder:
            raise EngineError(f"grad_through_encoder: no encoder backward for {name} on the engine")
        if self.codec_train_bn and getattr(self.depth_transform, "training", False):
            raise EngineError(f"codec_train_bn: no batch-statistics BatchNorms for {name} on the engine")

    def _producer_tensors(self):
        sd = {}
        for name in ("hahineck", "conv_lateral", "conv_up"):
            if name in self._modules:
                sd.update(collect_tensors(self._modules[name], name + "."))
        return sd

    @staticmethod
    def _sizes_ok(sizes):
        """Native FPN: each level at most 2x its coarser neighbour (== 2x: adaptive_avg_pool2d is the identity;
        smaller, e.g. 57 vs 2*29: the engine's pooling kernel resamples)."""
        return all(b[0] <= a[0] <= 2 * b[0] and b[1] <= a[1] <= 2 * b[1] for a, b in zip(sizes[:-1], sizes[1:]))

    @classmethod
    def _pyramid_ok(cls, feats):
        return cls._sizes_ok([tuple(f.shape[-2:]) for f in feats]) and all(f.shape[1] % 8 == 0 for f in feats)  # 16-byte NHWC rows (TMA)

    def attach_backbone(self, backbone):
        self.__dict__['_backbone_ref'] = weakref.ref(backbone)

    def _backbone(self, given=None):
        if given is not None:
            return given
        bb = self._backbone_ref() if self._backbone_ref is not None else None
        if bb is None:
            raise EngineError("native backbone requested but no backbone module is attached to this head "
                              "(Diffusion_DCbase_Model passes it; direct callers use head.attach_backbone)")
        return bb

    @staticmethod
    def swin_pyramid(image_hw):
        """Stage output sizes of a patch-4 Swin for an (H, W) image, finest first."""
        h, w = (image_hw[0] + 3) // 4, (image_hw[1] + 3) // 4
        sizes = []
        for _ in range(4):
            sizes.append((h, w))
            h, w = (h + 1) // 2, (w + 1) // 2
        return sizes

    @staticmethod
    def resnet_pyramid(image_hw):
        """Stage output sizes of the stem-less stride-2-per-stage ResNet (3x3, pad 1), finest first."""
        h, w = image_hw
        sizes = []
        for _ in range(4):
            h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
            sizes.append((h, w))
        return sizes

    def backbone_pyramid(self, image_hw, backbone=None):
        """Stage output sizes of this head's backbone family (MPViT halves per stage like the stem-less ResNet)."""
        if self.variant == "swin" and type(backbone).__name__ != "MPViT":
            return self.swin_pyramid(image_hw)
        return self.resnet_pyramid(image_hw)

    @staticmethod
    def mpvit_spec(backbone):
        """(layers per stage, stage widths, paths per stage, mlp ratio) of an MPViT module, or None when it is not one of
        the shapes the engine instantiates (8 heads, crpe windows {3: 2, 5: 3, 7: 3}, <= 3 paths, widths <= 512)."""
        try:
            stages = backbone.mhca_stages
            dims = [st.InvRes.conv1.conv.in_channels for st in stages]
            paths = [len(st.mhca_blks) for st in stages]
            layers = [len(st.mhca_blks[0].MHCA_layers) for st in stages]
            blk = stages[0].mhca_blks[0].MHCA_layers[0]
            ratio = blk.mlp.fc1.out_features // dims[0]
            ok = (len(stages) == 4 and max(paths) <= 3 and max(dims) <= 512 and all(d % 8 == 0 for d in dims)
                  and dims[0] % 16 == 0 and blk.factoratt_crpe.num_heads == 8
                  and [c.kernel_size[0] for c in stages[0].mhca_blks[0].crpe.conv_list] == [3, 5, 7]
                  and all(st.mhca_blks[0].MHCA_layers[0].mlp.fc1.out_features == ratio * d for st, d in zip(stages, dims))
                  and list(backbone.out_channels) == dims[1:] + dims[-1:])
            return (layers, dims, paths, ratio) if ok else None
        except (AttributeError, IndexError):
            return None

    @staticmethod
    def mpvit_drop_paths(backbone):
        """(per-stage bit masks of the encoder layers with stochastic depth, their DropPath modules in torch's draw order:
        stage, path, layer) of an MPViT module, or None when the layers with a DropPath of rate > 0 differ between the
        paths of a stage."""
        masks, mods = [], []
        for st in backbone.mhca_stages:
            bits = None
            for enc in st.mhca_blks:
                b = 0
                for l, blk in enumerate(enc.MHCA_layers):
                    if isinstance(blk.drop_path, DropPath) and blk.drop_path.p > 0.0:
                        b |= 1 << l
                        mods.append(blk.drop_path)
                if bits is not None and b != bits:
                    return None
                bits = b
            masks.append(bits or 0)
        return tuple(masks), mods

    @staticmethod
    def swin_drop_paths(backbone):
        """(per-stage bit masks of the blocks with stochastic depth, their MMCVDropPath modules in torch's draw order:
        stage, block, then the attention branch before the FFN branch) of a Swin module.  A block is marked when one of
        its two branches has a rate above 0 (the reference gives both the block's rate, swin.py:412,421)."""
        masks, mods = [], []
        for st in backbone.stages:
            bits = 0
            for k, blk in enumerate(st.blocks):
                pair = (getattr(blk.attn, "drop", None), getattr(blk.ffn, "dropout_layer", None))
                if all(isinstance(m, MMCVDropPath) for m in pair) and max(m.drop_prob for m in pair) > 0.0:
                    bits |= 1 << k
                    mods += pair
            masks.append(bits)
        return tuple(masks), mods

    @staticmethod
    def _draw_drop_scales(branches, batch, device):
        """Per-sample scales mask / keep of stochastic-depth branches, [branch][B] (set_drop_path), `branches` holding
        one DropPath or MMCVDropPath module per branch in torch's draw order.  Each is drawn on the device as its module's
        forward draws it: DropPath `x.new_empty((B, 1, 1)).bernoulli_(keep)`, MMCVDropPath
        `floor(keep + torch.rand((B, 1, 1)))`; a module in eval or at rate 0 draws nothing (scale 1).  None when no
        module draws."""
        def rate(m):
            return m.p if isinstance(m, DropPath) else m.drop_prob

        if not any(m.training and rate(m) > 0.0 for m in branches):
            return None
        out = []
        for m in branches:
            if not (m.training and rate(m) > 0.0):
                out.append(torch.ones(batch, device=device, dtype=torch.float32))
                continue
            keep = 1.0 - rate(m)
            if isinstance(m, MMCVDropPath):
                mask = (keep + torch.rand((batch, 1, 1), dtype=torch.float32, device=device)).floor()
            else:
                mask = torch.empty((batch, 1, 1), device=device, dtype=torch.float32).bernoulli_(keep)
            out.append(mask.reshape(batch) / keep)
        return torch.cat(out)

    def _mpvit_drop_scales(self, backbone, batch, device):
        """The scales of a natively run MPViT, [block][attention, MLP][B]: one DropPath module serves both branches of
        its block, called twice.  None when none is in training mode."""
        _, mods = self.mpvit_drop_paths(backbone)
        return self._draw_drop_scales([m for m in mods for _ in range(2)], batch, device)

    def _swin_drop_scales(self, backbone, batch, device):
        """The scales of a natively run Swin, [block][attention, FFN][B]; None when no branch draws."""
        return self._draw_drop_scales(self.swin_drop_paths(backbone)[1], batch, device)

    @staticmethod
    def _bn_modes(module):
        """{training flags} of the BatchNorms in `module`."""
        return {m.training for m in module.modules() if isinstance(m, nn.modules.batchnorm._BatchNorm)}

    def can_run_backbone(self, backbone, img) -> bool:
        """Native backbone path: CUDA input and an architecture the engine instantiates — Swin-L for the Swin heads,
        BasicBlock ResNetForMMBEV (64/128/256/512, stride 2 per stage) for the Res heads, MPViT for the MPViT head."""
        if not (self.native_producers and self.native_backbone and img.is_cuda):
            return False
        name = type(backbone).__name__
        if name == "MPViT":
            if self.producer_train_bn and backbone.training:
                # natively with mpvit_native_train, when its BatchNorms share one mode and its paths one DropPath
                # layout; otherwise torch runs it and the neck and FPN stay native
                if not self.mpvit_native_train or len(self._bn_modes(backbone)) > 1 \
                        or self.mpvit_drop_paths(backbone) is None:
                    return False
            spec = self.mpvit_spec(backbone)
            if spec is None or self.variant != "swin" or list(self.fpn_in_channels) != list(backbone.out_channels):
                return False
        elif self.variant == "swin":
            if name != "SwinTransformer" or getattr(backbone, "num_features", None) != [192, 384, 768, 1536]:
                return False
            if [len(s.blocks) for s in backbone.stages] != [2, 2, 18, 2]:
                return False
        else:
            if name != "ResNetForMMBEV" or list(backbone.backbone_output_ids) != [0, 1, 2, 3]:
                return False
            if [st[0].conv2.out_channels for st in backbone.layers] != [64, 128, 256, 512]:
                return False
        return self._sizes_ok(self.backbone_pyramid(img.shape[-2:], backbone))

    def _gather(self, native, image_hw, backbone):
        tensors = self._engine_tensors()
        if native:
            tensors.update(self._producer_tensors())
        if image_hw is not None:
            for k, v in collect_tensors(self._backbone(backbone), "backbone.").items():
                if v.is_floating_point():
                    tensors[k] = v
        return tensors

    def _engine(self, batch, latent_hw, cond_hw, device, feats=None, image_hw=None, backbone=None,
                backward=False, loop_backward=False, producer_train=False, steps=None, eta=0.0) -> DenoiseEngine:
        """feats: backbone feature maps, or a (channels, sizes) pyramid spec -> native neck/FPN;
        image_hw: additionally run the backbone natively (`backbone`: the module holding its parameters);
        backward: an engine that also serves `denoiser_backward`; loop_backward: one that also serves
        `denoise_backward` / `decode_backward` (and `denoiser_backward`); producer_train: this forward runs a producer
        BatchNorm in training mode (the eval producer pack may then lag behind their running statistics); steps, eta:
        the schedule (default: the head's own steps, eta = 0)."""
        with self._lock:
            return self._engine_locked(batch, latent_hw, cond_hw, device, feats, image_hw, backbone, backward,
                                       loop_backward, producer_train, steps, eta)

    def _engine_key(self, batch, latent_hw, cond_hw, device, native=False, image_hw=None, backward=False,
                    loop_backward=False, drop_path=(), steps=None, eta=0.0) -> EngineKey:
        return EngineKey(batch, tuple(latent_hw), tuple(cond_hw), str(torch.device(device)),
                         int(steps or self.diffusion_inference_steps), self.use_cuda_graph, native,
                         tuple(image_hw) if image_hw is not None else None, bool(self.return_intermediates),
                         native and bool(self.producer_train_bn), bool(backward), bool(loop_backward), tuple(drop_path),
                         self._codec_kind(), float(eta))

    def _mpvit_native_train(self, image_hw, backbone):
        """Whether the engine running this backbone also runs it in training mode (stochastic depth included)."""
        return (image_hw is not None and self.mpvit_native_train and self.producer_train_bn
                and type(self._backbone(backbone)).__name__ == "MPViT")

    def _native_drop_paths(self, image_hw, backbone):
        """(per-stage marks, scale drawer) of the stochastic depth the engine runs on this backbone, or None: an MPViT
        under `mpvit_native_train`, or a Swin whose drop-path rate is above 0 (`set_drop_path_rate`; the factories
        build at 0).  The drawer returns the scales of this forward, or None when no module is in training mode."""
        if image_hw is None:
            return None
        bb = self._backbone(backbone)
        if self._mpvit_native_train(image_hw, bb):
            return self.mpvit_drop_paths(bb)[0], lambda B, dev: self._mpvit_drop_scales(bb, B, dev)
        if type(bb).__name__ == "SwinTransformer":
            masks = self.swin_drop_paths(bb)[0]
            if any(masks):
                return masks, lambda B, dev: self._swin_drop_scales(bb, B, dev)
        return None

    def _grad_engine(self, batch, latent_hw, cond_hw, device) -> DenoiseEngine:
        """The engine `denoiser_backward` runs on: the loop-backward engine of this geometry when the head trains through
        the loop or that engine exists (its flag is a superset), else a backward-only one."""
        loop = self.grad_through_loop or \
            self._engine_key(batch, latent_hw, cond_hw, device, loop_backward=True) in self._engines
        return self._engine(batch, latent_hw, cond_hw, device, backward=not loop, loop_backward=loop)

    def _engine_locked(self, batch, latent_hw, cond_hw, device, feats, image_hw, backbone, backward,
                       loop_backward, producer_train=False, steps=None, eta=0.0) -> DenoiseEngine:
        native = feats is not None
        if native and not isinstance(feats, tuple):
            feats = ([f.shape[1] for f in feats], [tuple(f.shape[-2:]) for f in feats])
        device = torch.device(device)
        drop = self._native_drop_paths(image_hw, backbone)
        key = self._engine_key(batch, latent_hw, cond_hw, device, native, image_hw, backward, loop_backward,
                               drop[0] if drop else (), steps, eta)
        eng = self._engines.get(key)
        if eng is None:
            if key.codec_kind != 0 and self.variant == "res" and tuple(cond_hw) != tuple(latent_hw):
                raise EngineError(f"{type(self.depth_transform).__name__}: the Res denoiser adds the condition map "
                                  f"{tuple(cond_hw)} to the latent {tuple(latent_hw)} without resampling")
            pool = self._pools.setdefault(str(device), WorkspacePool(device))
            eng = DenoiseEngine(self.variant, batch, latent_hw, cond_hw, key.steps, device, cuda_graph=key.cuda_graph,
                                check_range=False, step_decode=key.step_decode, workspace_pool=pool,
                                backward=key.backward, loop_backward=key.loop_backward, producer_train=key.producer_train,
                                codec_kind=key.codec_kind)
            if native:
                eng.enable_producers(feats[0], feats[1], has_neck=self.has_neck)
            if image_hw is not None:
                if type(self._backbone(backbone)).__name__ == "MPViT":
                    layers, dims, paths, ratio = self.mpvit_spec(self._backbone(backbone))
                    eng.enable_backbone(image_hw, depths=layers, kind="mpvit", mp_dims=dims, mp_paths=paths, mlp_ratio=ratio,
                                        mp_drop_path=key.drop_path or (0, 0, 0, 0))
                elif self.variant == "swin":
                    eng.enable_backbone(image_hw, mp_drop_path=key.drop_path or (0, 0, 0, 0))
                else:
                    eng.enable_backbone(image_hw, depths=[len(st) for st in self._backbone(backbone).layers], kind="resnet")
            if key.eta > 0:
                eng.set_schedule(*self.scheduler.fused_coefficients(key.steps, eta=key.eta))
            else:
                eng.set_schedule(*self.scheduler.fused_coefficients(key.steps))
            self._engines[key] = eng
            self._packed.pop(key, None)
            self._stale.discard(key)
            while len(self._engines) > MAX_ENGINES:  # a ragged last batch / a new image size must not pile up engines
                old_key, old = self._engines.popitem(last=False)
                old.close()
                self._packed.pop(old_key, None)
                self._stale.discard(old_key)
        else:
            self._engines.move_to_end(key)
        if getattr(eng, "bn_allgather_group", None) is not self.bn_sync_group:  # every engine follows bn_sync_group
            eng.set_bn_allgather(self.bn_sync_group)
        # Re-pack when a parameter changed.  The ~500 tensors are walked once per pack; per forward only their
        # (data_ptr, _version) pairs are compared (0.3 ms instead of 2.6 ms for a Swin-L model).
        packed = self._packed.get(key)
        if packed is not None and packed[2] is not (backbone if image_hw is not None else None):
            packed = None  # a different backbone module (DataParallel replica): look its tensors up again
        if packed is None:
            tensors = self._gather(native, image_hw, backbone)
            sig = None
        else:
            tensors = packed[0]
            sig = _signature(tensors)
        # In a training-mode producer forward, changes confined to producer running statistics (the previous forward's
        # running update) are deferred: the batch-statistics path does not read them.  The eval pack is then stale and
        # the next eval-mode forward re-packs it in full.
        stale = key in self._stale and not producer_train
        if packed is None or sig != packed[1] or stale:
            changed = None
            if packed is not None:  # something changed: the owning modules may hold new tensors
                tensors = self._gather(native, image_hw, backbone)
                new_sig = _signature(tensors)
                defer = is_producer_running_stat if producer_train else None
                changed = None if stale else repack_plan(packed[0].keys(), packed[1], tensors.keys(), new_sig,
                                                         self.incremental_repack, defer)
                if changed is not None and defer is not None and any(
                        a != b and defer(k) for k, a, b in zip(tensors.keys(), packed[1], new_sig)):
                    self._stale.add(key)
            if changed is None:
                eng.load_weights(tensors)
                self._stale.discard(key)
            elif changed:
                eng.update_weights({k: tensors[k] for k in changed})
            self._packed[key] = (tensors, _signature(tensors), backbone if image_hw is not None else None)
        return eng

    def _any_engine(self, batch, latent_hw, cond_hw, device):
        """An engine of this geometry for the bare operators (denoiser / decode): reuse the forward's engine (same
        packed denoiser + codec weights) instead of packing a second one."""
        want = self._engine_key(batch, latent_hw, cond_hw, device)
        for key in reversed(self._engines):
            if key.geometry == want.geometry and self._packed.get(key) is not None:
                tensors, sig, _ = self._packed[key]
                if _signature(tensors) == sig:
                    self._engines.move_to_end(key)
                    return self._engines[key]
                break
        return self._engine(batch, latent_hw, cond_hw, device)

    def _denoiser_params(self):
        """The denoiser's parameters in DENOISER_KEYS (+ FUSE_KEYS) order: the order of dd_denoiser_backward's gradients."""
        keys = DENOISER_KEYS + (FUSE_KEYS if self.variant == "swin" else ())
        return keys, [self.get_submodule(k.rpartition(".")[0]).get_parameter(k.rpartition(".")[2]) for k in keys]

    def _loop_params(self):
        """The denoiser's then the decoder's parameters: the order of dd_denoise_backward's d_params, d_dec_params."""
        keys, params = self._denoiser_params()
        keys = keys + DECODER_PARAM_KEYS
        params = params + [self.get_submodule(k.rpartition(".")[0]).get_parameter(k.rpartition(".")[2])
                           for k in DECODER_PARAM_KEYS]
        return keys, params

    def denoiser(self, noisy, t, cond):
        """`self.model(noisy, t, cond, None, None, None)` of the reference, on the engine.  Differentiable (through
        `_DenoiserFunction`, native backward) when grad is enabled and `noisy`, `cond` or a denoiser parameter requires
        grad; otherwise the plain forward call."""
        tl = t.reshape(-1).tolist() if torch.is_tensor(t) else t
        if torch.is_grad_enabled():
            keys, params = self._denoiser_params()
            if noisy.requires_grad or cond.requires_grad or any(p.requires_grad for p in params):
                return _DenoiserFunction.apply(self, tl, keys, noisy, cond, *params)
        B = noisy.shape[0]
        eng = self._any_engine(B, noisy.shape[-2:], cond.shape[-2:], noisy.device)
        return eng.denoiser_forward(cond.contiguous().float(), noisy.contiguous().float(), tl)

    # ------------------------------------------------------------------------------------------ codec BatchNorms
    def _codec_bns(self):
        """The codec's BatchNorms: encoder (conv_transform.0.1, .1.1), decoder (conv_inv_transform.1)."""
        dt = self.depth_transform
        return dt.conv_transform[0][1], dt.conv_transform[1][1], dt.conv_inv_transform[1]

    def _codec_training(self) -> bool:
        """Whether this forward runs the codec's BatchNorms on batch statistics (`codec_train_bn` and the codec in
        training mode); the engine's BatchNorms use eps = 1e-5 only."""
        if not (self.codec_train_bn and getattr(self.depth_transform, "training", False)):
            return False
        for bn in self._codec_bns():
            if bn.eps != 1e-5:
                raise EngineError(f"codec_train_bn: the engine's codec BatchNorms use eps = 1e-5, got {bn.eps}")
        return True

    @staticmethod
    def _codec_records(eng, bns, order=None):
        """[(BatchNorm, batch mean, unbiased batch variance)] from `eng`'s records of its last forward call: record
        `order[i]` (default: i) for the i-th entry of `bns`."""
        rec = eng.codec_batch_stats()
        return [(bn, rec[i if order is None else order[i], 0], rec[i if order is None else order[i], 1])
                for i, bn in enumerate(bns)]

    # ------------------------------------------------------------------------------------------ producer BatchNorms
    def _producer_training(self, backbone=None):
        """(neck + FPN, native backbone) run their BatchNorms on batch statistics in this forward: `producer_train_bn`
        and the modules in training mode.  `backbone`: the natively run backbone module (None: torch runs it); the
        ResNet's BatchNorms are on the engine, and the MPViT's under `mpvit_native_train` (all of them in training mode).
        The engine's BatchNorms use eps = 1e-5 and track running statistics."""
        if not self.producer_train_bn:
            return False, False
        cond_mods = [self._modules[n] for n in ("hahineck", "conv_lateral") if n in self._modules]
        cond = any(m.training for m in cond_mods)
        name = type(backbone).__name__ if backbone is not None else None
        bb = (name == "ResNetForMMBEV" and backbone.training) or \
            (name == "MPViT" and self.mpvit_native_train and self._bn_modes(backbone) == {True})
        mods = ([self._modules[n] for n in ("hahineck", "conv_lateral", "conv_up") if n in self._modules] if cond else []) \
            + ([backbone] if bb else [])
        for m in mods:
            for bn in m.modules():
                if isinstance(bn, nn.modules.batchnorm._BatchNorm):
                    if bn.eps != 1e-5 or not bn.track_running_stats:
                        raise EngineError("producer_train_bn: the engine's producer BatchNorms use eps = 1e-5 and "
                                          f"running statistics, got eps = {bn.eps}, track_running_stats = "
                                          f"{bn.track_running_stats}")
        return cond, bb

    def _producer_records(self, eng, backbone=None):
        """[(BatchNorm, batch mean, unbiased batch variance)] of the producer BatchNorms `eng`'s last forward ran in
        training mode (keys `backbone.*` name modules of `backbone`)."""
        out = []
        for key, (mean, var) in eng.producer_batch_stats().items():
            bn = backbone.get_submodule(key[len("backbone."):]) if key.startswith("backbone.") else self.get_submodule(key)
            out.append((bn, mean, var))
        return out

    # ------------------------------------------------------------------------------------------ condition path
    def _condition(self, fp):
        """Top-down FPN that builds the 256-channel condition map x (head :112-122 / res.py:108-118)."""
        x = None
        for i in reversed(range(len(fp))):
            lat = self.conv_lateral[i](fp[i])
            if x is not None:
                lat = lat + F.adaptive_avg_pool2d(self.conv_up[i](x), lat.shape[-2:])
            x = lat
        return x

    def _neck(self, fp):
        return fp

    def _draw_noise(self, shape, device, dtype, override):
        if override is not None:
            return override.to(device=device, dtype=dtype).contiguous()
        g = self.noise_generator
        if g is not None and g.device.type != torch.device(device).type:
            return torch.randn(shape, generator=g, dtype=dtype).to(device)
        return torch.randn(shape, generator=g, device=device, dtype=dtype)

    # ------------------------------------------------------------------------------------------ forward
    def forward(self, fp, depth_map, depth_mask, gt_depth_map=None, return_loss=False, noise=None, image=None,
                backbone=None, **kwargs):
        """fp: backbone feature maps — or None, meaning "run the backbone natively from `image`" (the model
        wrapper does that when `can_run_backbone` holds, and passes `backbone` = the module holding its weights).

        Gradients: the condition map comes from the native producers (or the torch producers under no_grad) and carries
        no gradient, so `ddim_loss` trains the denoiser's parameters only.  A caller who trains the producers passes a
        differentiable `cond` to the operator itself, `self.model(noisy, t, cond)`, whose backward also returns d_cond.
        With `grad_through_loop = True`, `pred` and the final latent are differentiable too (denoiser and decoder
        parameters, through every step: `_LoopFunction`)."""
        self._check_codec_trains()
        if self.bn_sync_group is not None and self.return_intermediates:
            raise EngineError("bn_sync_group is not supported by the *Vis heads (their step decodes run in one CUDA graph)")
        with_backbone = fp is None
        drop_scales = None
        if with_backbone:
            B, dev, dtype = image.shape[0], image.device, torch.float32
            sizes = self.backbone_pyramid(image.shape[-2:], self._backbone(backbone))
            native = True
            drop = self._native_drop_paths(image.shape[-2:], backbone)
            if drop is not None:  # drawn first, as the torch backbone's forward would before the head draws x_T
                drop_scales = drop[1](B, dev)
        else:
            if self.detach_fp is not False and self.detach_fp is not None:
                idx = self.detach_fp if isinstance(self.detach_fp, (list, tuple, range)) else range(len(fp))
                fp = [f.detach() if i in idx else f for i, f in enumerate(fp)]
            fp = [f.contiguous().float() for f in fp]
            B, dev, dtype = fp[0].shape[0], fp[0].device, fp[0].dtype
            native = self.native_producers and fp[0].is_cuda and self._pyramid_ok(fp)
        latent_hw = tuple(self.depth_transform.latent_hw(gt_depth_map.shape[-2:]))  # shape of depth_transform.t(gt)
        gt_map_t = None
        enc_grad = None  # (keys, parameters) when gt_map_t is differentiable
        if self.grad_through_encoder and torch.is_grad_enabled():
            enc_grad = self._encoder_params()
            if not any(p.requires_grad for p in enc_grad[1]):
                enc_grad = None
        if not native:
            with torch.no_grad(), exact_fp32():
                if enc_grad is None:
                    gt_map_t = self.depth_transform.t(gt_depth_map)
                cond = self._condition(self._neck(fp)).contiguous()
        else:
            cond = None
        x_T = self._draw_noise((B, 16, *latent_hw), dev, dtype, noise)
        if self.grad_through_loop and self.return_intermediates:
            raise EngineError("grad_through_loop is not supported by the *Vis heads (pred_inter has no backward)")
        codec_train = self._codec_training()
        enc_bn1, enc_bn2, dec_bn = self._codec_bns() if codec_train else (None,) * 3
        bn_updates = []  # applied at the end: the buffers keep the signature the engines were packed with until then
        if native:  # (backbone +) neck + FPN + loop + decoder inside the engine; the condition map never leaves NHWC
            want_cond = self.capture_cond or self.training or self.eval_ddim_loss or self.grad_through_loop
            bb_mod = self._backbone(backbone) if with_backbone else None
            ptrain_cond, ptrain_bb = self._producer_training(bb_mod)
            ptrain = ptrain_cond or ptrain_bb
            if with_backbone:
                eng = self._engine(B, latent_hw, sizes[0], dev, feats=(list(self.fpn_in_channels), sizes),
                                   image_hw=tuple(image.shape[-2:]), backbone=backbone, producer_train=ptrain)
                if eng.producer_train:
                    eng.set_producer_mode(ptrain_bb)
                if drop is not None:
                    eng.set_drop_path(drop_scales)
                eng.run_backbone(image.contiguous().float())
                if eng.producer_train:
                    eng.set_producer_mode(ptrain_cond)
                cond = eng.build_condition(None, want_cond=want_cond)
            else:
                eng = self._engine(B, latent_hw, tuple(fp[0].shape[-2:]), dev, feats=fp, producer_train=ptrain)
                if eng.producer_train:
                    eng.set_producer_mode(ptrain_cond)
                cond = eng.build_condition(fp, want_cond=want_cond)
            if ptrain:
                bn_updates += self._producer_records(eng, bb_mod)
            gt_map_t = self._encode(eng, gt_depth_map, codec_train, enc_grad)  # returned as pred_init / gt_map_t only
            if codec_train:
                bn_updates += self._codec_records(eng, (enc_bn1, enc_bn2))
            loop_cond = None
        else:
            eng = self._engine(B, latent_hw, tuple(cond.shape[-2:]), dev)
            if enc_grad is not None:
                gt_map_t = self._encode(eng, gt_depth_map, codec_train, enc_grad)
                if codec_train:
                    bn_updates += self._codec_records(eng, (enc_bn1, enc_bn2))
            loop_cond = cond
        inter = None
        loop_keys, loop_params = None, None
        if self.grad_through_loop and torch.is_grad_enabled():
            loop_keys, loop_params = self._loop_params()
            if not (cond.requires_grad or any(p.requires_grad for p in loop_params)):
                loop_keys = None
        if loop_keys is not None:  # the same denoise_decode call, as an autograd node (native backward through the loop)
            box = {}
            refined_depth, refined_depth_t = _LoopFunction.apply(self, eng, box, loop_cond is None, loop_keys,
                                                                 codec_train, cond, x_T, *loop_params)
            logits = box["logits"]
        elif self.return_intermediates:  # *Vis heads: inv_t of every intermediate latent, decoded inside the graph
            eng.set_codec_mode(codec_train)
            steps, refined_depth_t, logits = eng.denoise_decode_steps(loop_cond, x_T, want_latent=True,
                                                                      want_logits=self.capture_logits)
            inter = list(steps.unbind(0))
            refined_depth = inter[-1]
        else:
            eng.set_codec_mode(codec_train)
            refined_depth, refined_depth_t, logits = eng.denoise_decode(loop_cond, x_T, want_latent=True,
                                                                        want_logits=self.capture_logits)
        if codec_train:
            if self.return_intermediates:  # the reference's order: inv_t of the final map, then of steps 1 .. T
                T = self.diffusion_inference_steps
                bn_updates += self._codec_records(eng, (dec_bn,) * (T + 1), order=[T - 1] + list(range(T)))
            else:
                bn_updates += self._codec_records(eng, (dec_bn,))
        self.last_latent, self.last_logits, self.last_cond = refined_depth_t, logits, cond
        if self.check_range:
            eng.poll_status()  # syncs; raises if an activation left the fp16 split range (DESIGN.md "Numerics")
        ddim_loss = self._ddim_loss(cond, refined_depth_t) if (self.eval_ddim_loss or self.training) \
            else refined_depth.new_zeros(())
        for bn, mean, var in bn_updates:
            bn_running_update(bn, mean, var)
        return {'pred': refined_depth, 'pred_init': gt_map_t, 'blur_depth_t': gt_map_t, 'ddim_loss': ddim_loss,
                'gt_map_t': gt_map_t, 'pred_uncertainty': None, 'pred_inter': inter, 'weight_map': None,
                'guidance': None, 'offset': None, 'aff': None, 'gamma': None, 'confidence': None}

    def _encoder_params(self):
        """The encoder's parameters in ENCODER_PARAM_KEYS order: the order of dd_encode_backward's gradients."""
        return ENCODER_PARAM_KEYS, [self.get_submodule(k.rpartition(".")[0]).get_parameter(k.rpartition(".")[2])
                                    for k in ENCODER_PARAM_KEYS]

    def _encode(self, eng, gt_depth_map, codec_train, enc_grad):
        """depth_transform.t(gt_depth_map) on `eng` in the codec mode `codec_train`; through `_EncodeFunction` when
        `enc_grad` = (keys, parameters) is given."""
        eng.set_codec_mode(codec_train)
        depth = gt_depth_map.contiguous().float()
        if enc_grad is None:
            return eng.encode(depth)
        return _EncodeFunction.apply(self, eng, enc_grad[0], codec_train, depth, *enc_grad[1])

    def ddim_loss_gt(self, gt_depth, refine_module_inputs, blur_depth_t, weight, **kwargs):
        """Reference head :225-240: the diffusion objective on the encoded ground truth `gt_depth` (the forward's
        `gt_map_t`), re-noised at a random timestep per image; `self.model(noisy, t, *refine_module_inputs)` must
        predict the noise.  Random draws in the reference's order: the noise on the CPU, then the timesteps on the
        device.  `blur_depth_t` and `weight` are unused, as in the reference.  The denoiser's parameters (and `cond`,
        when it requires grad) are trained through `_DenoiserFunction`; with `grad_through_encoder` the encoder too,
        through `gt_depth`."""
        noise = torch.randn(gt_depth.shape).to(gt_depth.device)
        timesteps = torch.randint(0, self.scheduler.num_train_timesteps, (gt_depth.shape[0],),
                                  device=gt_depth.device).long()
        noisy = self.scheduler.add_noise(gt_depth, noise, timesteps)
        return F.mse_loss(self.model(noisy, timesteps, *refine_module_inputs), noise)

    def _ddim_loss(self, cond, latent):
        """Reference head :207-223 — one extra denoiser call on a re-noised latent; RNG-dependent."""
        noise = torch.randn(latent.shape).to(latent.device)
        t = torch.randint(0, self.scheduler.num_train_timesteps, (latent.shape[0],), device=latent.device).long()
        noisy = self.scheduler.add_noise(latent, noise, t)
        return F.mse_loss(self.denoiser(noisy, t, cond), noise)  # == self.model(noisy, t, cond, None, None, None)

    ddim_loss = _ddim_loss


class CNNDDIMPipiline:
    """The reference's DDIM sampler (head :244-303; the *Vis heads' copy also returns `image_list`, ..._vis.py:254-306):
    `pipeline(batch_size, device, dtype, shape, input_args, generator, eta, num_inference_steps, return_dict)` ->
    `(latent,)` or `{'images': latent}` (Vis: `(latent, image_list)` / `{'images', 'image_list'}`, the latent after
    every step).  It draws x_T = randn((batch_size, *shape)), then, only when eta > 0, one randn of that shape per step
    (the reference scheduler's `variance_noise`, the last step's included), each with `generator` when given, and runs
    the T steps of `scheduler.step(..., eta, use_clipped_model_output=True)` on the head's engine in one call: the
    condition map `input_args[0]` must be a CUDA tensor and `model` the head's ScheduledCNNRefine.  It returns the
    latent; decoding it (`depth_transform.inv_t`) is the caller's.  No gradient: under autograd, with the condition
    map or a denoiser / decoder parameter requiring grad, eta > 0 raises, as does eta = 0 on a head set to
    `grad_through_loop` (the head's forward is the differentiable path); otherwise the result carries no graph."""

    def __init__(self, model, scheduler, image_list=False):
        self.model = model
        self.scheduler = scheduler
        self.image_list = image_list
        self._head = None

    def __call__(self, batch_size, device, dtype, shape, input_args, generator: Optional[torch.Generator] = None,
                 eta: float = 0.0, num_inference_steps: int = 50, return_dict: bool = True,
                 **kwargs) -> Union[Dict, Tuple]:
        head = self._head if self._head is not None else (self.model._bridge() if self.model._bridge else None)
        cond = input_args[0]
        if head is None or head.model is not self.model or not (torch.is_tensor(cond) and cond.is_cuda):
            raise EngineError("CNNDDIMPipiline runs on the head's CUDA engine: `model` must be the head's "
                              "ScheduledCNNRefine and input_args[0] a CUDA condition map")
        eta = float(eta)
        if eta < 0:
            raise ValueError(f"eta must be >= 0, got {eta}")
        if torch.is_grad_enabled():
            _, params = head._denoiser_params()
            if cond.requires_grad or any(p.requires_grad for p in params):
                if eta > 0:
                    raise EngineError(f"CNNDDIMPipiline(eta={eta}) has no backward: a stochastic sample (eta > 0) is "
                                      "not differentiated; run it under torch.no_grad()")
                if head.grad_through_loop:
                    raise EngineError("CNNDDIMPipiline has no backward: with grad_through_loop, train through the "
                                      "head's forward, or run the pipeline under torch.no_grad()")
        image_shape = (batch_size, *shape)
        image = torch.randn(image_shape, generator=generator, device=device, dtype=dtype)
        self.scheduler.set_timesteps(num_inference_steps)
        T = len(self.scheduler.timesteps)
        z = None
        if eta > 0:
            z = torch.stack([torch.randn(image_shape, generator=generator, device=device, dtype=dtype)
                             for _ in range(T)]).float()
        x_T = image.detach().float().contiguous()
        eng = head._engine(batch_size, tuple(shape[-2:]), tuple(cond.shape[-2:]), cond.device, steps=T, eta=eta)
        eng.set_codec_mode(False)
        steps = torch.empty(T, *x_T.shape, device=x_T.device) if self.image_list else None
        _, latent, _ = eng.denoise_decode(cond.detach().contiguous().float(), x_T, want_latent=True, variance_noise=z,
                                          latent_steps=steps)
        if head.check_range:
            eng.poll_status()
        image = latent.to(dtype)
        if self.image_list:
            image_list = [s.to(dtype) for s in steps.unbind(0)]
            return (image, image_list) if not return_dict else {'images': image, 'image_list': image_list}
        return (image,) if not return_dict else {'images': image}
