/*
 * dd_engine.h — C ABI of libddengine.so: the H100-native (sm_90a) DiffusionDepth hot path.
 *
 * The reference (duanyiqun/DiffusionDepth @ e1ca9d5) has no FFI on this path; these entry points
 * are what a binding for it would bind.  Each one names the reference interface it replaces:
 *
 *   dd_create / dd_destroy        <- construction of `ScheduledCNNRefine` + `CNNDDIMPipiline` +
 *                                    `DeepDepthTransformWithUpsampling` inside the head ctor
 *                                    (src/model/head/ddim_depth_estimate_res_swin_addHAHI.py:45-49,
 *                                     src/model/head/ddim_depth_estimate_res.py:36-40)
 *   dd_set_weight / dd_finalize_weights / dd_update_weights
 *                                 <- `load_state_dict(ckpt['net'])` for the keys under
 *                                    `depth_head.model.*` and `depth_head.depth_transform.*`
 *                                    (src/main.py:418-432; key layout SURVEY.md Appendix A)
 *   dd_set_schedule               <- `DDIMScheduler.set_timesteps` + the per-step scalar algebra of
 *                                    `DDIMScheduler.step` (src/model/diffusers/schedulers/
 *                                    scheduling_ddim.py:215-229, 285-326) collapsed to
 *                                    x_{t-1} = c_x * x_t + c_eps * eps
 *   dd_set_schedule_eta           <- the same with `eta` > 0: `DDIMScheduler.step(..., eta,
 *                                    use_clipped_model_output=True)` (scheduling_ddim.py:285-350) collapsed to
 *                                    x_{t-1} = c_x * x_t + c_eps * eps + sigma_t * z_t
 *   dd_set_step_io                <- the per-step `randn` draws of that `step` (:336-345) passed in as
 *                                    `variance_noise`, and the Vis pipeline's `image_list` (..._vis.py:289-306)
 *   dd_denoise_decode             <- `CNNDDIMPipiline.__call__` (head :254-303) = T x
 *                                    {`ScheduledCNNRefine.forward` (:361-382 / res.py:324-344),
 *                                    `DDIMScheduler.step`} followed by
 *                                    `DeepDepthTransformWithUpsampling.inv_t`
 *                                    (src/model/ops/depth_transform.py:33-35)
 *   dd_denoiser_forward           <- one bare `ScheduledCNNRefine.forward(noisy, t, cond, ...)` call
 *                                    (the operator `ddim_loss` invokes, head :207-223)
 *   dd_denoiser_backward          <- reverse-mode differentiation of that call: the gradients of
 *                                    `ScheduledCNNRefine` (head :336-382 / res.py:301-344) that `ddim_loss`
 *                                    (head :207-223) needs for training
 *   dd_denoiser_relu_inputs       <- the inputs of that call's four `nn.ReLU` after `nn.GroupNorm(4, C)`
 *                                    (head :341-358 / res.py:305-321), as the backward recomputes them
 *   dd_denoise_backward          <- reverse-mode differentiation of dd_denoise_decode: the training graph of
 *                                    `pred` and the final latent under the reference's L1 + L2 + DDIM loss
 *                                    (head :130-146, :165-175, :207-223) through every step and the decoder
 *   dd_decode                     <- `depth_transform.inv_t(latent)` alone (the *Vis heads call it
 *                                    per step, ..._swin_addHAHI_vis.py)
 *   dd_decode_backward            <- reverse-mode differentiation of `inv_t` (eval BatchNorm)
 *   dd_encode_backward            <- reverse-mode differentiation of `t` with respect to the encoder's parameters
 *                                    (the heads' `ddim_loss_gt`, head :225-240, trains the encoder through `gt_map_t`)
 *
 * Conventions (inherited from the reference, SURVEY.md §8b): every tensor is fp32, NCHW, contiguous,
 * resident on the engine's CUDA device; no autograd.  Ownership: the caller (PyTorch's allocator)
 * owns every buffer including the workspace; the engine borrows raw pointers for the duration of a
 * call and owns only its pre-packed weights / descriptors / CUDA graph.  Calls are enqueued on the
 * given stream and return without synchronising.  One handle per (process, device); a handle is not
 * re-entrant.  Errors: int status (0 = ok), never an exception across the ABI; text via
 * dd_last_error() (thread-local).  There is NO CPU path: dd_create fails if no sm_90 device is present.
 */
#ifndef DD_ENGINE_H_
#define DD_ENGINE_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DD_ABI_VERSION 3

typedef struct dd_engine* dd_handle;

enum dd_status {
  DD_OK = 0,
  DD_ERR_INVALID = 1,     /* bad argument / shape / missing weight */
  DD_ERR_CUDA = 2,        /* a CUDA runtime or driver call failed */
  DD_ERR_UNSUPPORTED = 3, /* no sm_90 device, unsupported shape */
  DD_ERR_RANGE = 4        /* an activation left the fp16 split's range (see DESIGN.md "Numerics") */
};

enum dd_variant {
  DD_VARIANT_RES = 0,  /* DDIMDepthEstimate_Res: cond at latent resolution, no upsample_fuse */
  DD_VARIANT_SWIN = 1  /* DDIMDepthEstimate_Swin_ADDHAHI: cond upsampled (bilinear, align_corners)
                          to the latent grid, then convA/convB */
};

enum dd_flags {
  DD_FLAG_CUDA_GRAPH = 1 << 0, /* capture the T-step loop once and replay it */
  DD_FLAG_SIMT_CONV = 1 << 1,  /* debug: fp32 CUDA-core convolutions instead of the tensor cores */
  DD_FLAG_CHECK_RANGE = 1 << 2,/* after the call, sync and report DD_ERR_RANGE if the split overflowed */
  DD_FLAG_HALO_CONV = 1 << 3,  /* kernel selection on Blackwell; the sm_90a build always runs the row-halo kernel */
  DD_FLAG_SWAP_NARROW = 1 << 4, /* swapped-operand narrow convs (Blackwell only; accepted without effect on sm_90a) */
  DD_FLAG_PAIR_WIDE = 1 << 5,   /* Cout = 256 convs on CTA pairs (Blackwell only; accepted without effect on sm_90a) */
  DD_FLAG_STEP_DECODE = 1 << 6, /* reserve workspace for dd_denoise_decode_steps (T decoded maps; the *Vis heads) */
  DD_FLAG_FP8_CORR = 1 << 7,    /* correction products of the split as e4m3 MMAs (Blackwell only: Hopper's e4m3 MMA
                                   accumulates at reduced precision, DESIGN.md "Numerics"); the sm_90a build accepts the
                                   flag and runs the exact 3-pass fp16 split everywhere */
  DD_FLAG_BACKWARD = 1 << 8,    /* enable dd_denoiser_backward: dd_finalize_weights also packs the flipped, transposed
                                   conv weights of the data gradients, and dd_workspace_bytes includes the backward's
                                   region (recomputed activations, gradient buffers; DESIGN.md "Backward") */
  DD_FLAG_LOOP_BACKWARD = 1 << 9, /* everything DD_FLAG_BACKWARD does, and enable dd_denoise_backward / dd_decode_backward:
                                   dd_finalize_weights also keeps the decoder's unfolded ConvTranspose weights and
                                   BatchNorm scale, and the workspace adds the loop backward's region (the T + 1 latents
                                   [T+1][B,P,16] fp32, fp64 gradient accumulators, the running latent gradient, the
                                   decoder backward's scratch) */
  DD_FLAG_CHAIN_PRED = 1 << 10, /* Swin: run convB and pred.0 as two 3x3 convs instead of one composed 5x5 conv + its
                                   border correction (A/B runs and tests; DD_FLAG_SIMT_CONV always runs the chain) */
  DD_FLAG_PRODUCER_TRAIN = 1 << 11 /* enable dd_set_producer_mode(DD_PRODUCER_TRAIN): dd_finalize_weights also packs every
                                   BatchNorm'ed producer layer (ResNet bn1 / bn2, HAHI neck, FPN) unfolded — its conv
                                   alone, with gamma / beta kept on the device — and allocates engine-owned scratch for
                                   the largest pre-BN output.  The eval pack, graphs and dd_workspace_bytes are those of
                                   an engine without the flag. */
};

/* The depth codec (`depth_transform_cfg` of the reference heads, src/model/ops/depth_transform.py), carried in flag bits
 * DD_FLAG_CODEC_SHIFT .. +1 (kind << DD_FLAG_CODEC_SHIFT).  It fixes the latent grid of an H x W depth map and the
 * upsampling u of the decoder (decoded map [B,1,u h,u w]):
 *   DD_CODEC_UP2      DeepDepthTransformWithUpsampling (:10-35)     latent ceil(H/2) x ceil(W/2),           u = 2
 *   DD_CODEC_UP2_1X1  DeepDepthTransformWithUpsampling1x1 (:38-64)  latent ceil(H/2) x ceil(W/2),           u = 2
 *   DD_CODEC_UP4      DeepDepthTransformWithUpsamplingX4 (:67-94)   latent ceil(ceil(H/2)/2) (each side),   u = 4
 *   DD_CODEC_FULL     DeepDepthTransform (:97-117)                  latent H x W,                           u = 1
 * dd_set_weight takes the kind's `depth_transform.*` keys and rejects the other kinds'; dd_finalize_weights needs the
 * decoder's, the encoder's stay optional (all of them or none).  Kinds other than DD_CODEC_UP2 run with eval-mode BatchNorm only: they
 * answer dd_set_codec_mode(DD_CODEC_TRAIN), dd_encode_backward and dd_decode_backward with DD_ERR_UNSUPPORTED, and
 * dd_create refuses them with DD_FLAG_LOOP_BACKWARD.  dd_denoiser_forward / dd_denoiser_backward do not involve the
 * codec. */
enum dd_codec_kind { DD_CODEC_UP2 = 0, DD_CODEC_UP2_1X1 = 1, DD_CODEC_UP4 = 2, DD_CODEC_FULL = 3 };
#define DD_FLAG_CODEC_SHIFT 12

typedef struct dd_config {
  int32_t abi_version;          /* must be DD_ABI_VERSION */
  int32_t variant;              /* enum dd_variant */
  int32_t batch;                /* images per call on this device */
  int32_t latent_h, latent_w;   /* shape of depth_transform.t(gt): h = ceil(H/2), w = ceil(W/2) for the default
                                   codec (dd_codec_kind: ceil(ceil(H/2)/2) for DD_CODEC_UP4, H for DD_CODEC_FULL) */
  int32_t cond_h, cond_w;       /* spatial size of the FPN condition map x (256 channels) */
  int32_t num_inference_steps;  /* T */
  int32_t device;               /* CUDA ordinal */
  int32_t flags;                /* enum dd_flags */
} dd_config;

/* Fixed by the reference architecture (head ctor): 16 latent channels, 256 condition channels,
 * GroupNorm(4, C), time_embedding rows = 1280. */
#define DD_LATENT_C 16
#define DD_COND_C 256
#define DD_TIME_ROWS 1280

int dd_abi_version(void);
const char* dd_last_error(void);

int dd_create(const dd_config* cfg, dd_handle* out);
int dd_destroy(dd_handle h);

/* Register one parameter/buffer by its reference state_dict key relative to `depth_head.`
 * (e.g. "model.noise_embedding.0.weight", "depth_transform.conv_inv_transform.1.running_var").
 * `dev_ptr` is a device fp32 pointer in the reference's own layout/shape; it is read by the next
 * dd_finalize_weights or dd_update_weights only, which then forgets every registered pointer (a re-pack registers
 * all keys again, an update the changed ones).  Unknown keys are rejected (DD_ERR_INVALID). */
int dd_set_weight(dd_handle h, const char* name, const float* dev_ptr, const int64_t* shape, int32_t ndim);

/* Pre-pack: fold eval-BatchNorm into the decoder, repack conv weights tap-major, split them into
 * scaled fp16 hi/lo planes for the 3-pass tensor-core product.  Fails listing any missing key, and on any key of the
 * denoiser or codec whose shape is not the reference's (DD_ERR_INVALID). */
int dd_finalize_weights(dd_handle h, void* cuda_stream);

/* After an optimizer step: re-pack, in place, what depends on the tensors registered with dd_set_weight since the
 * last successful dd_finalize_weights / dd_update_weights: ONLY the tensors that changed, under the same keys and
 * shapes.  Every refreshed buffer ends up with exactly the bytes a dd_finalize_weights from the same tensors would
 * write, at the address that finalize allocated: nothing is allocated or freed, no TMA descriptor is re-encoded.
 *   a denoiser conv's `.weight` / `.bias`     that layer's split planes, bias and scale (and, with DD_FLAG_BACKWARD /
 *                                             DD_FLAG_LOOP_BACKWARD, its data-gradient layer)
 *   `upsample_fuse.convB.conv.*`, `pred.0.*`  also the composed 5x5 conv, where the engine runs it
 *   a GroupNorm `.weight` / `.bias`, `model.time_embedding.weight`
 *                                             the engine's copy
 *   `depth_transform.conv_inv_transform.*`    the folded decoder (and the unfolded one of DD_FLAG_LOOP_BACKWARD)
 *   `depth_transform.conv_transform.*`        the folded encoder
 *   `hahineck.*`, `conv_lateral.*`, `conv_up.*`, `backbone.*`
 *                                             DD_ERR_UNSUPPORTED: those packs are rebuilt by dd_finalize_weights only
 * CUDA graphs are kept.  The one exception: the loop graphs hold each conv's power-of-two weight scale (and the
 * step-decode graph the decoder's final bias) as kernel arguments, so when such a value changes (max |w| of a layer
 * crosses a power of two) the graphs holding it are captured again on their next use.
 * The work is enqueued on `cuda_stream` and the call synchronises that stream once; the registered tensors are read on
 * the stream after the call returns as well, so free them in stream order.  Successive calls that touch the weights
 * belong on one stream, or on streams the caller orders.
 * Every key and shape is validated before anything is written: on DD_ERR_INVALID (a key this engine did not pack, a
 * different shape, no finalize yet) or DD_ERR_UNSUPPORTED the registrations are forgotten and the engine is as it was
 * before the dd_set_weight calls.  With nothing registered the call does nothing. */
int dd_update_weights(dd_handle h, void* cuda_stream);

/* CUDA graph instantiations since dd_create: lets a test or a timing script see which calls captured a graph. */
int64_t dd_graph_capture_count(dd_handle h);

/* Per-step timesteps (descending, as DDIMScheduler.set_timesteps produces) and the collapsed DDIM
 * coefficients; n must equal num_inference_steps. */
int dd_set_schedule(dd_handle h, const int64_t* timesteps, const double* c_x, const double* c_eps, int32_t n);

/* As dd_set_schedule, for the reference's stochastic DDIM step (`CNNDDIMPipiline.__call__(eta=...)`, head :254-303,
 * calling `DDIMScheduler.step(..., eta, use_clipped_model_output=True)`, scheduling_ddim.py:285-350, clip_sample
 * False, epsilon prediction): step i runs x <- c_x[i] x + c_eps[i] eps + sigma[i] z_i with
 *   sigma = eta sqrt((1 - a_prev) / (1 - a_t) (1 - a_t / a_prev)),
 *   c_eps = sqrt(1 - a_prev - sigma^2) - sqrt(a_prev (1 - a_t) / a_t),   c_x = sqrt(a_prev / a_t),
 * computed by the caller in fp64 (DDIMScheduler.fused_coefficients(eta=...)).  sigma NULL or all zero: exactly
 * dd_set_schedule (the eta = 0 kernels and graphs).  A schedule with a non-zero sigma makes every dd_denoise_decode(_steps)
 * need the noise of dd_set_step_io (DD_ERR_INVALID without it).  DD_ERR_UNSUPPORTED on an engine created with
 * DD_FLAG_LOOP_BACKWARD (a stochastic sample is not differentiated); DD_ERR_INVALID for a negative or non-finite sigma.
 * Either setter drops the loop graphs: the next call captures them again. */
int dd_set_schedule_eta(dd_handle h, const int64_t* timesteps, const double* c_x, const double* c_eps,
                        const double* sigma, int32_t n);

/* Borrowed for the next dd_denoise_decode or dd_denoise_decode_steps call only, which then forgets both (NULL: none):
 *   variance_noise    [T][B,16,h,w] device fp32: z_i of step i (the reference's `variance_noise`, one `randn(shape)`
 *                     per step in step order, the last step's included); read in place by the loop's kernels, through
 *                     an engine-owned device slot the call writes before the loop (or its CUDA graph) runs.  Ignored
 *                     by a schedule without sigma.
 *   latent_steps_out  [T][B,16,h,w] device fp32: the latent after every step (the Vis pipeline's `image_list`); the
 *                     call then runs its loop without a CUDA graph. */
int dd_set_step_io(dd_handle h, const float* variance_noise, float* latent_steps_out);

/* Optional: also run the step-invariant condition producers natively — HAHI neck (attention gates off, as
 * the shipped heads configure it: src/model/necks/hahi.py:165-276) and the FPN (head :112-122) — on the same
 * 3-pass tensor-core path.  Call before dd_finalize_weights; additionally register the reference keys
 * `hahineck.*` (only if has_neck), `conv_lateral.*`, `conv_up.*`.  Pyramid levels may be anything up to 2x their
 * coarser neighbour (an exact 2x pyramid makes the FPN's adaptive_avg_pool2d the identity; otherwise it is a real
 * resample kernel).  Channel counts: any positive multiples of 8 (Swin 192..1536, ResNet 64..512, MPViT 128/216/288/288);
 * partial 64-channel K chunks and partial N tiles are completed with zeros by TMA's out-of-bounds fill. */
typedef struct dd_producer_config {
  int32_t num_levels;   /* 2..4 */
  int32_t channels[4];  /* backbone feature channels, finest level first */
  int32_t heights[4];
  int32_t widths[4];
  int32_t has_neck;     /* 1: *HAHI heads (HAHIHeteroNeck in front of the FPN), 0: Res heads and Swin_ADD */
} dd_producer_config;
int dd_enable_producers(dd_handle h, const dd_producer_config* pc);

/* feats[i]: device fp32 NCHW [B, channels[i], heights[i], widths[i]] (the backbone's outputs).  Builds the
 * (feats may be NULL right after dd_run_backbone.)  256-channel condition map inside the workspace; a following dd_denoise_decode(cond = NULL, ...) consumes it.
 * cond_out (nullable): also write it as NCHW [B,256,cond_h,cond_w]. */
int dd_build_condition(dd_handle h, const float* const* feats, float* cond_out, void* workspace,
                       size_t workspace_bytes, void* cuda_stream);

/* Optional: also run the Swin backbone natively (reference src/model/backbone/swin.py:756-777): patch embed,
 * LayerNorms, QKV / proj / FFN / patch-merging Linears on the 3-pass tensor-core GEMM path, 7x7 (shifted-)window
 * attention with relative-position bias and the finite -100 mask, per-stage output norms written straight into the
 * neck's (or, without a neck, the FPN's) input planes.  Requires dd_enable_producers(4 levels) with matching geometry; register the
 * reference keys of `depth_backbone.*` as "backbone.<key>" (the int64 `relative_position_index` buffers are not
 * needed).  Instantiated for Swin-L (embed_dims 192, head_dim 32, window 7). */
enum dd_backbone_kind {
  DD_BACKBONE_SWIN = 1,   /* SwinTransformer (reference backbone/swin.py) */
  DD_BACKBONE_RESNET = 2, /* ResNetForMMBEV with BasicBlocks, no stem (reference backbone/mmbev_resnet.py:124-187): depths[] =
                             blocks per stage, channels 64/128/256/512, every stage stride 2; needs
                             dd_enable_producers(4 levels, has_neck = 0); embed_dims / num_heads / window ignored */
  DD_BACKBONE_MPVIT = 3   /* MPViT (reference backbone/mpvit.py:601-730; tiny / xsmall / small / base factories :743-870):
                             full-resolution stem, then 4 x { chained depthwise-separable patch embeddings (first one
                             stride 2), a conv path + one factorised-attention encoder per embedding, 1x1 aggregate }.
                             depths[] = encoder layers per stage, mp_dims[] = stage widths (multiples of 8, <= 512; stage
                             s outputs mp_dims[s + 1], the last one mp_dims[3]), mp_paths[] = embeddings per stage (<= 3),
                             mlp_ratio; 8 heads, crpe windows {3: 2, 5: 3, 7: 3} heads.  Outputs at 1/2 .. 1/16 of the image;
                             needs dd_enable_producers(4 levels) with those sizes and channels */
};
typedef struct dd_backbone_config {
  int32_t kind;        /* enum dd_backbone_kind */
  int32_t embed_dims;  /* 192 */
  int32_t depths[4];   /* 2, 2, 18, 2 */
  int32_t num_heads[4];/* 6, 12, 24, 48 */
  int32_t window;      /* 7 */
  int32_t height, width; /* input image size */
  int32_t mp_dims[4];  /* DD_BACKBONE_MPVIT only: 64, 128, 216, 288 (mpvit_small) */
  int32_t mp_paths[4]; /* 2, 3, 3, 3 */
  int32_t mlp_ratio;   /* 4 */
  int32_t mp_drop_path[4]; /* DD_BACKBONE_MPVIT and DD_BACKBONE_SWIN: bit k of entry s set = block k of stage s has
                              stochastic depth (a DropPath of rate > 0) on its two residual branches, attention then
                              MLP / FFN; see dd_set_drop_path.  MPViT: encoder layer k in every path of the stage;
                              Swin: SwinBlock k.  All zero: none.  Ignored by DD_BACKBONE_RESNET */
} dd_backbone_config;
int dd_enable_backbone(dd_handle h, const dd_backbone_config* bc);

/* rgb: device fp32 NCHW [B,3,height,width].  Leaves the four stage outputs in the workspace for a following
 * dd_build_condition(feats = NULL, ...); feats_out (nullable array of 4 nullable pointers) also receives them as
 * fp32 NCHW [B, C_s, H_s, W_s]. */
int dd_run_backbone(dd_handle h, const float* rgb, float* const* feats_out, void* workspace, size_t workspace_bytes,
                    void* cuda_stream);

size_t dd_workspace_bytes(dd_handle h);

/* cond [B,256,cond_h,cond_w], noise [B,16,h,w] -> latent_out [B,16,h,w] (nullable),
 * logit_out [B,1,u h,u w] (nullable; the decoder's pre-sigmoid z), depth_out [B,1,u h,u w]; u = 2 for the default
 * codec (dd_codec_kind).
 * cond may be NULL right after dd_build_condition. */
int dd_denoise_decode(dd_handle h, const float* cond, const float* noise, float* latent_out, float* logit_out,
                      float* depth_out, void* workspace, size_t workspace_bytes, void* cuda_stream);

/* The *Vis heads' variant (reference src/model/head/ddim_depth_estimate_res_swin_addHAHI_vis.py:130-149, pipeline
 * :289-304 `image_list`): same loop, and `inv_t` of the latent after EVERY step, all inside the captured graph.
 * depth_steps_out [T][B,1,u h,u w] (slice T-1 is the final `pred`); latent_out / logit_out (nullable) refer to the
 * final step.  Needs DD_FLAG_STEP_DECODE at dd_create. */
int dd_denoise_decode_steps(dd_handle h, const float* cond, const float* noise, float* latent_out, float* logit_out,
                            float* depth_steps_out, void* workspace, size_t workspace_bytes, void* cuda_stream);

/* eps = ScheduledCNNRefine(noisy, t, cond): noisy [B,16,h,w], t[b] int64 host array (one per image),
 * eps_out [B,16,h,w]. */
int dd_denoiser_forward(dd_handle h, const float* cond, const float* noisy, const int64_t* t_host, float* eps_out,
                        void* workspace, size_t workspace_bytes, void* cuda_stream);

/* Backward of dd_denoiser_forward (reference ScheduledCNNRefine.forward, head :361-382 / res.py:324-344, differentiated
 * in reverse mode): given d_eps [B,16,h,w] = dL/d eps for eps = ScheduledCNNRefine(noisy, t, cond), write
 *   d_cond_out  [B,256,cond_h,cond_w]  dL/d cond   (nullable)
 *   d_noisy_out [B,16,h,w]             dL/d noisy  (nullable)
 *   d_params[i]                        dL/d parameter i in the reference layout (the array and each entry nullable), in
 *                                      the order of the reference state_dict keys under `depth_head.model.`:
 *      0 noise_embedding.0.weight [64,16,3,3]   1 noise_embedding.0.bias   2 noise_embedding.1.weight [64]
 *      3 noise_embedding.1.bias               4 noise_embedding.3.weight [256,64,3,3]   5 noise_embedding.3.bias
 *      6 noise_embedding.4.weight [256]       7 noise_embedding.4.bias   8 time_embedding.weight [1280,256]
 *      9 pred.0.weight [64,256,3,3]          10 pred.0.bias   11 pred.1.weight [64]   12 pred.1.bias
 *     13 pred.3.weight [16,64,3,3]           14 pred.3.bias   15 pred.4.weight [16]   16 pred.4.bias
 *   and for DD_VARIANT_SWIN also
 *     17 upsample_fuse.convA.conv.weight [256,256,3,3]   18 convA.conv.bias   19 convB.conv.weight   20 convB.conv.bias.
 * time_embedding.weight's gradient is dense: zero except at the rows t_host[b]; a row shared by several images is the sum
 * of their contributions in image order.  The call recomputes the forward from (cond, noisy, t) into the backward's own
 * workspace region, then runs the backward; it does not synchronise.  Results are bit-identical run to run.
 * Needs DD_FLAG_BACKWARD at dd_create (else DD_ERR_INVALID), as does a null cond / noisy / t_host / d_eps or a timestep
 * outside [0, 1280).  DD_FLAG_CHECK_RANGE and dd_poll_status also report an overflow of the gradient split. */
int dd_denoiser_backward(dd_handle h, const float* cond, const float* noisy, const int64_t* t_host, const float* d_eps,
                         float* d_cond_out, float* d_noisy_out, float* const* d_params, void* workspace,
                         size_t workspace_bytes, void* cuda_stream);

/* The inputs of the four ReLUs of ScheduledCNNRefine (reference head :341-358 / res.py:305-321, `nn.ReLU` after each
 * `nn.GroupNorm(4, C)`) as dd_denoiser_backward's recompute produces them: z = gamma * xhat + beta of
 *   z_out[0] noise_embedding.1 [B,64,h,w]    z_out[1] noise_embedding.4 [B,256,h,w]
 *   z_out[2] pred.1            [B,64,h,w]    z_out[3] pred.4            [B,16,h,w]
 * (fp32 NCHW, each entry nullable) for eps = ScheduledCNNRefine(noisy, t, cond).  The inputs are staged and the
 * forward recomputed exactly as dd_denoiser_backward does, and z comes from the expression its GroupNorm + ReLU
 * backward evaluates, so z > 0 is, bit for bit, the mask that backward applies.  For checking the backward against a
 * higher-precision computation at the same masks.  Argument checks as dd_denoiser_backward (DD_FLAG_BACKWARD or
 * DD_FLAG_LOOP_BACKWARD, null arguments, timesteps, workspace); DD_FLAG_CHECK_RANGE is honoured; does not synchronise
 * otherwise.  Results are bit-identical run to run. */
int dd_denoiser_relu_inputs(dd_handle h, const float* cond, const float* noisy, const int64_t* t_host,
                            float* const* z_out, void* workspace, size_t workspace_bytes, void* cuda_stream);

/* Backward of dd_denoise_decode (reference CNNDDIMPipiline.__call__ + DeepDepthTransformWithUpsampling.inv_t, head
 * :254-303 / depth_transform.py:33-35, differentiated in reverse mode through all T denoiser calls, the T DDIM updates
 * and the decoder; the decoder's BatchNorm uses its running statistics, as the forward does).  Given
 *   d_depth  [B,1,2h,2w]  dL/d depth         (nullable)
 *   d_latent [B,16,h,w]   dL/d final latent  (nullable; not both NULL)
 * for depth, latent = dd_denoise_decode(cond, noise), write (every output nullable)
 *   d_cond_out [B,256,cond_h,cond_w], d_noise_out [B,16,h,w] (dL/d x_T),
 *   d_params[i]      the denoiser's 17 / 21 gradients in dd_denoiser_backward's order; time_embedding.weight is dense,
 *                    non-zero at the rows of the schedule's timesteps,
 *   d_dec_params[i]  6 decoder gradients: conv_inv_transform.0.weight [16,16,4,4], .0.bias, .1.weight, .1.bias,
 *                    .3.0.weight [1,16,3,3], .3.0.bias (zero when d_depth is NULL),
 *   latents_out      [T+1][B,16,h,w]: x_T = noise, then the latent after every step, as the call recomputed them.
 * The call re-runs the loop un-graphed with the forward's kernels (bit-identical to dd_denoise_decode's), keeping every
 * latent, then walks back: at each step the recompute + backward chain of dd_denoiser_backward, with per-step gradients
 * summed in fp64 in step order.  Results are bit-identical run to run; the call does not synchronise.  cond may be NULL
 * right after dd_build_condition.  Needs DD_FLAG_LOOP_BACKWARD and dd_set_schedule (else DD_ERR_INVALID).
 * DD_FLAG_CHECK_RANGE and dd_poll_status also report an overflow of the gradient split. */
int dd_denoise_backward(dd_handle h, const float* cond, const float* noise, const float* d_depth, const float* d_latent,
                        float* d_cond_out, float* d_noise_out, float* const* d_params, float* const* d_dec_params,
                        float* latents_out, void* workspace, size_t workspace_bytes, void* cuda_stream);

/* depth = inv_t(latent): latent [B,16,h,w] -> logit_out (nullable), depth_out [B,1,u h,u w] (dd_codec_kind). */
int dd_decode(dd_handle h, const float* latent, float* logit_out, float* depth_out, void* workspace,
              size_t workspace_bytes, void* cuda_stream);

/* Backward of dd_decode: d_depth [B,1,2h,2w] -> d_latent_out [B,16,h,w] and d_dec_params[0..5] (as in
 * dd_denoise_backward; the array and every output nullable).  Needs DD_FLAG_LOOP_BACKWARD. */
int dd_decode_backward(dd_handle h, const float* latent, const float* d_depth, float* d_latent_out,
                       float* const* d_dec_params, void* workspace, size_t workspace_bytes, void* cuda_stream);

/* latent = depth_transform.t(depth) (reference src/model/ops/depth_transform.py:29-31): depth [B,1,height,width] ->
 * latent_out [B,16,ceil(height/2),ceil(width/2)] (other codec kinds: their latent grid, dd_codec_kind).  Needs the
 * optional keys `depth_transform.conv_transform.*`. */
int dd_encode(dd_handle h, const float* depth, int32_t height, int32_t width, float* latent_out, void* cuda_stream);

/* Backward of dd_encode in the current codec mode: d_latent [B,16,ceil(height/2),ceil(width/2)] -> d_enc_params[0..5]
 * = the gradients of conv_transform.0.0.weight [16,1,3,3], .0.1.weight, .0.1.bias, .1.0.weight [16,16,3,3],
 * .1.1.weight, .1.1.bias (the array and every entry nullable).  It recomputes the forward from depth; in DD_CODEC_TRAIN
 * it recomputes the two batch statistics as dd_encode does (bit-identical) and differentiates through them, across
 * ranks with each BatchNorm's backward sums gathered once.  It records nothing (dd_codec_batch_stats still reports the
 * last forward).  No gradient with respect to depth.  Bit-identical run to run; no synchronisation.  Its scratch
 * aliases the operator backward's region of the workspace.  DD_ERR_INVALID without DD_FLAG_BACKWARD or
 * DD_FLAG_LOOP_BACKWARD, before dd_finalize_weights, without encoder weights, for a size that does not match the
 * latent grid, for a NULL depth or d_latent, and in DD_CODEC_TRAIN when batch x latent is 1. */
int dd_encode_backward(dd_handle h, const float* depth, int32_t height, int32_t width, const float* d_latent,
                       float* const* d_enc_params, void* workspace, size_t workspace_bytes, void* cuda_stream);

/* How the depth codec's BatchNorms normalise.  DD_CODEC_EVAL (the default): running statistics, folded into the
 * weights at dd_finalize_weights.  DD_CODEC_TRAIN: as BatchNorm2d in training mode, the statistics of the batch
 * each call sees (biased variance, eps 1e-5), computed and folded on the device without synchronising:
 *   dd_decode, dd_denoise_decode           one batch-statistics decode                      (1 record)
 *   dd_denoise_decode_steps                one per step, inside a CUDA graph of its own      (T records)
 *   dd_encode                              both BatchNorms, the second after the first       (2 records)
 *   dd_decode_backward, dd_denoise_backward, dd_encode_backward  differentiate through the batch mean and variance
 * The backward's recompute and the steps variant's extra logit decode record nothing.  The engine never writes running
 * statistics: the caller applies the running update from the records and registers the new buffers with
 * dd_update_weights.  In DD_CODEC_TRAIN dd_encode returns DD_ERR_INVALID when batch x latent is 1 (one value per
 * channel).  The mode is engine state; DD_ERR_INVALID for a value other than the two below. */
enum dd_codec_mode { DD_CODEC_EVAL = 0, DD_CODEC_TRAIN = 1 };
int dd_set_codec_mode(dd_handle h, int32_t mode);

/* Batch statistics of every codec BatchNorm the last forward entry (dd_decode, dd_denoise_decode(_steps), dd_encode)
 * evaluated in DD_CODEC_TRAIN, in evaluation order: dev_out [n][2][16] fp32 (batch mean, unbiased variance),
 * *n_out = n (0 after a forward in DD_CODEC_EVAL).  Enqueued on cuda_stream, no synchronisation; DD_ERR_INVALID when
 * capacity < n. */
int dd_codec_batch_stats(dd_handle h, float* dev_out, int32_t capacity, int32_t* n_out, void* cuda_stream);

/* How the condition producers' BatchNorms normalise: the ResNet backbone's BasicBlock bn1 / bn2 (reference
 * mmbev_resnet.py:150-160), the HAHI neck's ConvModules (necks/hahi.py:54-97) and the FPN's conv_lateral.i.1 /
 * conv_up.i.1 (head :112-122).  DD_PRODUCER_EVAL (the default): running statistics, folded into the weights at
 * dd_finalize_weights.  DD_PRODUCER_TRAIN (needs DD_FLAG_PRODUCER_TRAIN, else DD_ERR_INVALID): as BatchNorm2d in
 * training mode, the statistics of the batch each call sees (biased variance, eps 1e-5).  dd_run_backbone (ResNet) and
 * dd_build_condition then run each such layer as the conv on its unfolded pack into engine-owned fp32 scratch (a ConvT
 * pixel-shuffled: its statistics cover all B x 2H x 2W pixels before the FPN's adaptive_avg_pool2d), two statistics
 * passes, a fold s = gamma / sqrt(var + 1e-5), t = beta - s mean, and act(s u + t) with the eval layer's addend and
 * outputs; no host synchronisation, CUDA graphs of their own (the eval graphs are kept).  dd_run_backbone (MPViT) does the
 * same for the stem, the patch embeddings' pointwise convs, InvRes conv1 / conv2, the aggregate and InvRes.norm after
 * its depthwise conv, with Hardswish where the layer has it (records: stem, then per stage the patch embeddings,
 * conv1, norm, conv2, aggregate).  The Swin backbone is not affected.  The engine never writes running statistics: the caller applies the running update from the
 * records (dd_producer_batch_stats) and re-packs the eval weights with dd_finalize_weights when it next runs in
 * DD_PRODUCER_EVAL.  The mode is engine state, read by each call. */
enum dd_producer_mode { DD_PRODUCER_EVAL = 0, DD_PRODUCER_TRAIN = 1 };
int dd_set_producer_mode(dd_handle h, int32_t mode);

/* Records of the producers' BatchNorms: one per BatchNorm'ed layer, in evaluation order, [2][C] fp32 (batch mean,
 * unbiased batch variance) at a fixed offset (dd_producer_bn_info).  Copies all of them back to back into dev_out
 * (capacity in floats; dev_out may be NULL to query *n_out, the number of records); enqueued on cuda_stream, no
 * synchronisation.  A record is current when the forward that last started (dd_run_backbone, or dd_build_condition
 * with feature maps) evaluated its layer in DD_PRODUCER_TRAIN (dd_producer_bn_info's *fresh). */
int dd_producer_batch_stats(dd_handle h, float* dev_out, int64_t capacity, int32_t* n_out, void* cuda_stream);

/* Stochastic depth of the MPViT backbone (reference mpvit.py:432,435, timm DropPath in training mode) or of the Swin
 * backbone (reference swin.py:412,421, mmcv DropPath in training mode): dev_scales (device fp32, n of them) holds, for
 * every block dd_backbone_config.mp_drop_path marks, the B per-sample scales mask / (1 - rate) of its attention branch,
 * then the B of its MLP / FFN branch; blocks in stage, path, layer order (MPViT) or stage, block order (Swin).  They are
 * copied on cuda_stream into an engine-owned buffer that every later dd_run_backbone reads (graphs included), in either
 * producer mode: x = x + scale[b] branch.  n = 0 turns stochastic depth off (the default; dev_scales may be NULL).
 * DD_ERR_INVALID when n is neither 0 nor 2 x batch x the marked blocks, or before dd_finalize_weights of an MPViT or
 * Swin backbone (which also turns it off). */
int dd_set_drop_path(dd_handle h, const float* dev_scales, int32_t n, void* cuda_stream);

/* Record i: the registered key prefix of its BatchNorm (e.g. `hahineck.trans_fusion.1.bn`, `conv_up.0.1`,
 * `backbone.layers.2.0.bn1`; NUL-terminated, truncated to key_capacity), its channels, its offset in floats into
 * dd_producer_batch_stats' output, and whether it is current.  DD_ERR_INVALID for i out of range. */
int dd_producer_bn_info(dd_handle h, int32_t i, char* key, int32_t key_capacity, int32_t* channels, int64_t* offset,
                        int32_t* fresh);

/* Cross-rank all-gather of BatchNorm statistics: fill out[world_size][count] with every rank's in[count], ordered by
 * rank, in stream order on cuda_stream (in and out are device memory the engine owns); return 0 on success.  Every
 * rank must make the same sequence of calls with the same counts. */
typedef int (*dd_allgather_fn)(const double* in, double* out, int64_t count, void* cuda_stream, void* user);

/* Synchronised BatchNorm (as apex's SyncBatchNorm): with fn installed, every BatchNorm that runs on batch statistics
 * (DD_CODEC_TRAIN, DD_PRODUCER_TRAIN) normalises with the statistics of the union of all world_size ranks' batches,
 * which may be ragged.  Each statistics pass gathers this rank's fp64 totals with its pixel count and sums the gathered
 * rows in rank order, so every rank folds and records the same values bit for bit: the mean and variance of the union,
 * the unbiased variance with N = the union's pixel count.  Gathers per BatchNorm: two in the forward, one in the
 * decoder backward (its sum dv and sum dv xhat over the union).  While fn is installed the training-mode producer
 * calls run their launches eagerly instead of from their CUDA graphs, and dd_denoise_decode_steps in DD_CODEC_TRAIN
 * returns DD_ERR_UNSUPPORTED.  A non-zero return of fn fails the call with DD_ERR_CUDA; the engine stays usable.
 * fn = NULL (the default) turns it off: nothing changes.  Synchronises the device. */
int dd_set_bn_allgather(dd_handle h, dd_allgather_fn fn, void* user, int32_t world_size);

/* Synchronise `cuda_stream` and report DD_ERR_RANGE if any activation left the fp16 split's range since the
 * last hot-path call started (DD_OK otherwise).  The hot-path calls themselves never synchronise unless
 * DD_FLAG_CHECK_RANGE is set. */
int dd_poll_status(dd_handle h, void* cuda_stream);

/* Number of kernel launches the last forward (dd_run_backbone .. dd_denoise_decode) enqueued; graph nodes count
 * individually. */
int64_t dd_last_launch_count(dd_handle h);

/* Standalone layer entry used by the parity tests and the roofline bench: one 3x3/s1/p1 convolution
 * + bias on the engine's tensor-core (or SIMT, per flags) path.
 * x [B,Cin,H,W], w [Cout,Cin,3,3], b [Cout] -> y [B,Cout,H,W]; all device fp32 NCHW. */
int dd_conv3x3(dd_handle h, const float* x, const float* w, const float* b, float* y, int32_t batch, int32_t cin,
               int32_t cout, int32_t height, int32_t width, void* workspace, size_t workspace_bytes,
               void* cuda_stream);
size_t dd_conv3x3_workspace_bytes(int32_t batch, int32_t cin, int32_t cout, int32_t height, int32_t width);

/* Standalone weight gradient of that convolution on the backward's own kernels (the tensor-core kernel for the
 * 256-wide shapes, the fp32 CUDA-core kernel for 16->64 and 64->16), chosen by shape as dd_denoiser_backward chooses
 * them.  x [B,Cin,H,W] and dy [B,Cout,H,W] (device fp32 NCHW) -> dw [Cout,Cin,3,3] = sum over images and pixels of
 * dy (x) x, db [Cout] = sum of dy.  dy is split to fp16 hi/lo with the backward's on-device power-of-two scale.
 * DD_ERR_UNSUPPORTED for a shape off the hot path; synchronises `cuda_stream` and returns DD_ERR_RANGE when x or dy held
 * a non-finite value or left the split's range.  Does not touch the engine's workspace. */
int dd_conv3x3_wgrad(dd_handle h, const float* x, const float* dy, float* dw, float* db, int32_t batch, int32_t cin,
                     int32_t cout, int32_t height, int32_t width, void* workspace, size_t workspace_bytes,
                     void* cuda_stream);
size_t dd_conv3x3_wgrad_workspace_bytes(int32_t batch, int32_t cin, int32_t cout, int32_t height, int32_t width);

/* One layer of the producers (backbone, HAHI neck, FPN) on their tensor-core conv / GEMM kernel, described by: */
typedef struct dd_gen_layer_desc {
  int32_t taps;                 /* 1 (1x1 conv, Linear) or 9 (3x3, pad 1) */
  int32_t stride;               /* 1, or 2 (conv mode, one source, not transposed) */
  int32_t transposed;           /* 1: ConvTranspose2d(k=2, s=2), taps 1, one source; pixel-shuffled output */
  int32_t act;                  /* 0 none, 1 ReLU, 2 exact (erf) GELU, 3 Hardswish */
  int32_t add_first;            /* 1: the addend goes in before the activation, 0: after it */
  int32_t tokens;               /* > 0: GEMM mode on that many token rows (batch .. src_w ignored) */
  int32_t batch, height, width; /* conv mode: the output grid */
  int32_t src_h, src_w;         /* stride 2: the source grid */
  int32_t c0, c1;               /* channels of source 0 and of source 1 (concatenated after it; 0: none) */
  int32_t cin;                  /* the weight's input channels: 0 = c0 + c1; below c0 (one source) zero-pads it to c0 */
  int32_t cout;                 /* output channels (transposed: per output pixel) */
  int32_t ld_out, ch_off;       /* output rows are ld_out channels wide (0: cout), written from channel ch_off */
  int32_t n_tile;               /* N-tile width 64 / 128 / 192 / 256, 0: the engine's choice */
  int32_t alt_tile;             /* layers with 192-wide alternative maps: 0 by wave cost, 1 always, -1 never */
} dd_gen_layer_desc;

/* Standalone run of that kernel for layer tests, packing and launching the layer exactly as the engine does:
 *   x0 [tokens][c0] or [B][src grid][c0], x1 [.. output grid ..][c1] (nullable when c1 = 0): device fp32 NHWC, split at
 *      the producers' scale;
 *   w  the reference layout: conv [cout][cin][k][k], Linear [cout][cin], ConvT [c0][cout][2][2];
 *   bn (nullable) four device vectors [cout] (weight, bias, running_mean, running_var) of an eval-BN folded after the
 *      conv, otherwise bias [cout] (nullable);
 *   add32 (nullable) fp32 addend, dense [rows][cout] (transposed: [B][2H][2W][cout]);
 *   y32 fp32 and / or out_hi, out_lo fp16 planes (at the producers' scale) of [rows][ld_out]: only the layer's rows
 *      (not the GEMM tail) and channels [ch_off, ch_off + cout) are written (transposed: [B][2H][2W][cout]).
 * launch_out (nullable) receives {N-tile width, work items, grid, launches}: a layer deeper than one fp32 accumulator
 * should take runs as that many launches over channel ranges, summed in fp32 in a fixed order.  Allocates and frees its own buffers, touches neither
 * the workspace nor the packed weights; synchronises `cuda_stream` and returns DD_ERR_RANGE when an input or an output
 * plane held a non-finite value or left the split's range. */
int dd_gen_layer(dd_handle h, const dd_gen_layer_desc* d, const float* x0, const float* x1, const float* w,
                 const float* bias, const float* const* bn, const float* add32, float* y32, void* out_hi, void* out_lo,
                 int32_t* launch_out, void* cuda_stream);

/* Standalone (shifted-)window attention of a Swin block (7 x 7 windows, head_dim 32, C = 32 nH): qkv [B*H*W][3C] (device
 * fp32, the qkv Linear's output; padded tokens carry qkv_bias [3C]), table [169][nH] -> out [B*H*W][C] fp32, rebuilt from
 * the kernel's hi/lo output planes.  kernel: 0 the engine's choice, 1 the fp32 CUDA-core kernel, 2 the wgmma kernel (nH
 * even).  launch_out (nullable) receives {units of work, grid}.  Allocates and frees its own buffers; synchronises and
 * returns DD_ERR_RANGE as dd_gen_layer does. */
int dd_window_attention(dd_handle h, const float* qkv, const float* qkv_bias, const float* table, float* out,
                        int32_t batch, int32_t height, int32_t width, int32_t num_heads, int32_t shift, int32_t kernel,
                        int32_t* launch_out, void* cuda_stream);

/* Standalone factorised attention of an MPViT encoder layer (8 heads, crpe windows {3: 2 heads, 5: 3, 7: 3}, C = 8 Ch,
 * Ch <= 64), through the backbone's own launch sequence: qkv [B*H*W][3C] (device fp32, the qkv Linear's output, q | k |
 * v head-major), crpe_w[g] / crpe_b[g] the reference's crpe.conv_list.{0,1,2}.weight [nh Ch][1][k][k] / .bias [nh Ch]
 * -> out [B*H*W][C] = Ch^-0.5 q (softmax over the tokens of k)^T v + q * crpe(v) in fp32, rebuilt from the kernel's hi/lo
 * output planes.  launch_out (nullable) receives {tokens per chunk, chunks, heads per k^T v block, apply grid}.
 * DD_ERR_UNSUPPORTED for C not a multiple of 8 or above 512.  Allocates and frees its own buffers; synchronises and
 * returns DD_ERR_RANGE as dd_gen_layer does. */
int dd_factor_attention(dd_handle h, const float* qkv, const float* const* crpe_w, const float* const* crpe_b, float* out,
                        int32_t batch, int32_t height, int32_t width, int32_t channels, int32_t* launch_out,
                        void* cuda_stream);

/* Standalone depthwise 3x3 conv of the MPViT backbone (pad 1), packed and launched as the backbone does: x [B][H][W][C]
 * (device fp32 NHWC, the source grid), w [C][1][3][3] followed by eval-BN bn (nullable: four device vectors [C] weight,
 * bias, running_mean, running_var, folded) or by bias [C] (nullable; not both); stride 1 or 2; act 0 none, 3 Hardswish;
 * residual 1 adds x before the activation (ConvPosEnc; stride 1 only) -> y32 fp32 and / or out_hi, out_lo fp16 planes
 * (at the producers' scale) of [B][ceil(H / stride)][ceil(W / stride)][C].  launch_out (nullable) receives {grid, work
 * items of 4 channels}.  DD_ERR_UNSUPPORTED for C not a multiple of 4.  Allocates and frees its own buffers;
 * synchronises and returns DD_ERR_RANGE when an output plane held a non-finite value or left the split's range (an fp32
 * output alone is not range-checked). */
int dd_depthwise_conv(dd_handle h, const float* x, const float* w, const float* bias, const float* const* bn, float* y32,
                      void* out_hi, void* out_lo, int32_t batch, int32_t height, int32_t width, int32_t channels,
                      int32_t stride, int32_t act, int32_t residual, int32_t* launch_out, void* cuda_stream);

/* Standalone LayerNorm of the MPViT encoders (any C <= 512): x [tokens][C] (device fp32), gamma / beta [C] -> out
 * [tokens][C] fp32, rebuilt from the kernel's hi/lo output planes.  DD_ERR_UNSUPPORTED for C above 512.  Allocates and
 * frees its own buffers; synchronises and returns DD_ERR_RANGE as dd_gen_layer does. */
int dd_layer_norm(dd_handle h, const float* x, const float* gamma, const float* beta, float* out, int32_t tokens,
                  int32_t channels, float eps, void* cuda_stream);

/* Standalone patch embedding of the Swin backbone, launched as the backbone does: rgb [B][3][H][W] (device fp32,
 * zero-padded right / bottom to a multiple of 4), w [E][3][4][4], bias / gamma / beta [E] -> 4x4/s4 conv + bias +
 * LayerNorm(E) (eps 1e-5) -> out [B * ceil(H / 4) * ceil(W / 4)][E] fp32, written by the kernel itself (not
 * range-checked).  DD_ERR_UNSUPPORTED for E other than 192.  Allocates and frees its own buffers; synchronises. */
int dd_swin_patch_embed(dd_handle h, const float* rgb, const float* w, const float* bias, const float* gamma,
                        const float* beta, float* out, int32_t batch, int32_t height, int32_t width, int32_t embed,
                        void* cuda_stream);

/* Standalone LayerNorm of the Swin backbone (norm1 / norm2 of every block, the stage-output norms; eps 1e-5): x
 * [tokens][C] (device fp32), gamma / beta [C] -> out [tokens][C] fp32, rebuilt from the kernel's hi/lo output planes,
 * and, when nchw_out is not null, the stage-output copy nchw_out [tokens / hw][C][hw] fp32 (tokens a multiple of hw;
 * hw is ignored otherwise).  DD_ERR_UNSUPPORTED for C outside {192, 384, 768, 1536}.  Allocates and frees its own
 * buffers; synchronises and returns DD_ERR_RANGE as dd_gen_layer does. */
int dd_swin_layer_norm(dd_handle h, const float* x, const float* gamma, const float* beta, float* out, float* nchw_out,
                       int32_t tokens, int32_t channels, int32_t hw, void* cuda_stream);

/* Standalone patch merging of the Swin backbone, launched as the backbone does: x [B][H][W][C] (device fp32) -> 2x2
 * unfold (feature c * 4 + ky * 2 + kx; zero pad for odd H / W) + LayerNorm(4C) (eps 1e-5) with gamma / beta [4C] ->
 * out [B * ceil(H / 2) * ceil(W / 2)][4C] fp32, rebuilt from the kernel's hi/lo output planes.  DD_ERR_UNSUPPORTED for
 * C outside {192, 384, 768}.  Allocates and frees its own buffers; synchronises and returns DD_ERR_RANGE as
 * dd_gen_layer does. */
int dd_swin_patch_merge(dd_handle h, const float* x, const float* gamma, const float* beta, float* out, int32_t batch,
                        int32_t height, int32_t width, int32_t channels, void* cuda_stream);

typedef struct dd_conv_gn_desc {
  int32_t batch, cin, cout, height, width; /* one of the loop's GroupNorm'd convs: 16->64, 64->256, 256->64, 64->16 */
  int32_t mode;            /* 0 GN + ReLU (Cout 64); 1 + cond (same grid) + temb (Cout 256); 2 + bilinear up(cond + temb),
                              align_corners=True (Cout 256); 3 GN + ReLU -> the DDIM update (Cout 16) */
  int32_t cond_h, cond_w;  /* mode 2: the condition's grid */
  int32_t up_qpb;          /* mode 2: quads per block of the up-add kernel, 4 or 1 */
  float c_x, c_eps;        /* mode 3 with a latent: x <- c_x x + c_eps eps */
} dd_conv_gn_desc;

/* Standalone GroupNorm(4, Cout)'d conv of the DDIM loop, through the loop's own kernels: the 3x3 conv (the engine's
 * choice, DD_FLAG_SIMT_CONV honoured) with its GroupNorm-statistics epilogue, the fp64 finalize and the apply kernel of
 * `mode`.  x [B][cin][H][W], w [cout][cin][3][3], b / gamma / beta [cout]; cond [B][256][cond grid] and temb [B][256]
 * (modes 1 and 2); latent [B][16][H][W] (mode 3, nullable: null writes eps, otherwise it is updated in place), all
 * device fp32.  Outputs, each nullable: y32 [B][cout][H][W] the conv output before the norm, mean_rstd [B][4][2], out
 * [B][cout][H][W] the layer's output in fp32, rebuilt from the hi/lo planes the apply kernel wrote (mode 3: eps, or
 * the updated latent's planes).  Allocates and frees its own buffers; synchronises and returns DD_ERR_RANGE as
 * dd_gen_layer does. */
int dd_conv_groupnorm(dd_handle h, const dd_conv_gn_desc* d, const float* x, const float* w, const float* b,
                      const float* gamma, const float* beta, const float* cond, const float* temb, float* latent,
                      float* y32, float* mean_rstd, float* out, void* cuda_stream);

/* Time the dominant kernel (convA-shaped 256->256 3x3 on the engine's latent grid) `iters` times with
 * CUDA events on `cuda_stream`; returns average milliseconds per launch in *ms_out. */
int dd_bench_conv(dd_handle h, int32_t cin, int32_t cout, int32_t iters, float* ms_out, void* workspace,
                  size_t workspace_bytes, void* cuda_stream);

/* Time the Swin step's composed convB -> pred.0 (the 5x5 conv + its ring correction, two launches) `iters` times with
 * CUDA events; average milliseconds per pair in *ms_out.  DD_ERR_UNSUPPORTED when the engine runs the chain. */
int dd_bench_pred_fold(dd_handle h, int32_t iters, float* ms_out, void* workspace, size_t workspace_bytes,
                       void* cuda_stream);

/* Time the codec's decoder kernel alone (decoder_kernel, or the UP4 / FULL kind's own) `iters` times with CUDA events
 * on `cuda_stream`, decoding the latent the workspace holds from the last call into depth_out [B,1,u h,u w]; average
 * milliseconds per launch in *ms_out. */
int dd_bench_decoder(dd_handle h, float* depth_out, int32_t iters, float* ms_out, void* workspace, size_t workspace_bytes,
                     void* cuda_stream);

/* Tuning aid: average milliseconds per launch of the GEMM-mode kernel (tokens [M,K] x weights [N,K]^T) on
 * synthetic operands.  mode 0: fp32 out, 1: fp32 out + residual add, 2: GELU -> fp16 planes, 3: no output. */
int dd_bench_gemm(dd_handle h, int32_t M, int32_t K, int32_t N, int32_t mode, int32_t iters, float* ms_out);

#ifdef __cplusplus
}
#endif
#endif /* DD_ENGINE_H_ */
