// libddengine.so — C ABI (include/dd_engine.h) over the sm_90a kernels in conv_halo.cuh / convgen.cuh / kernels.cuh.
// Host side: weight pre-pack, workspace carving, TMA descriptor construction, per-step launch schedule
// (captured once into a CUDA graph), status polling.  No CPU compute path exists in this library.
#include <cuda.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <string>
#include <vector>

#include "../../include/dd_engine.h"
#include "kernels.cuh"
#include "convgen.cuh"
#include "conv_halo.cuh"
#include "pred_fold.cuh"
#include "swin.cuh"
#include "mpvit.cuh"
#include "backward.cuh"
#include "codec_train.cuh"
#include "producer_train.cuh"

namespace {

thread_local std::string g_err;

int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}
#define CUDA_TRY(expr)                                                                          \
  do {                                                                                          \
    cudaError_t _e = (expr);                                                                    \
    if (_e != cudaSuccess)                                                                      \
      return fail(DD_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));             \
  } while (0)

// The check after every kernel launch.  check_launch leaves the engine's launch count alone (weight packing, the
// standalone layer entries, and the transposes / splits whose callers count them); launched() counts one launch.
int check_launch(const char* what) {
  const cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) return fail(DD_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(err));
  return DD_OK;
}
// Blocks of per_block elements each for a grid-stride kernel over n elements, capped at 16 per SM of an H100 (132 SMs).
int grid_of(size_t n, int per_block = 256) {
  const size_t b = (n + per_block - 1) / per_block;
  return static_cast<int>(std::max<size_t>(1, std::min<size_t>(b, 132 * 16)));
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;

int load_driver() {
  if (g_encode) return DD_OK;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q);
  if (e != cudaSuccess || fn == nullptr || q != cudaDriverEntryPointSuccess)
    return fail(DD_ERR_CUDA, "cuTensorMapEncodeTiled not available from the driver");
  g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  return DD_OK;
}

int absmax_grid(size_t n) {  // blocks of 256 threads, ~4 elements per thread, at most two per SM
  const size_t b = (n + 1023) / 1024;
  return static_cast<int>(b < 1 ? 1 : (b > 296 ? 296 : b));
}

// Power-of-two split scale (dd::grad_scale_of) of the absmax that `launch_absmax` leaves in the device word *amax_dev:
// the largest power of two with amax * scale < 2^15, so hi stays finite and lo = O(2^4) stays normal.  The word is
// zeroed first; st is synchronised to read it back.
template <typename Absmax>
int split_scale(float* amax_dev, cudaStream_t st, float* scale, Absmax&& launch_absmax) {
  CUDA_TRY(cudaMemsetAsync(amax_dev, 0, 4, st));
  launch_absmax();
  int rc;
  if ((rc = check_launch("absmax"))) return rc;
  float amax = 0.f;
  CUDA_TRY(cudaMemcpyAsync(&amax, amax_dev, 4, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  *scale = dd::grad_scale_of(amax);
  return DD_OK;
}
// ... of the n device floats at x
int split_scale_of(const float* x, size_t n, float* amax_dev, cudaStream_t st, float* scale) {
  return split_scale(amax_dev, st, scale, [&] {
    dd::absmax_kernel<<<absmax_grid(n), 256, 0, st>>>(x, static_cast<int>(n), amax_dev);
  });
}

CUtensorMapSwizzle swizzle_for(int bk) {
  return bk == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : (bk == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
}

// The one cuTensorMapEncodeTiled call: an fp16 tensor of `rank` dims (innermost first; strides in bytes of dims 1..),
// no interleave, out-of-bounds elements read as zero.  `what` names the map in the error message.
int encode_map(CUtensorMap* m, const char* what, cuuint32_t rank, const __half* base, const cuuint64_t* dims,
               const cuuint64_t* strides, const cuuint32_t* box, const cuuint32_t* estr, CUtensorMapSwizzle swizzle,
               CUtensorMapL2promotion l2) {
  const CUresult r = g_encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, rank, const_cast<__half*>(base), dims, strides, box, estr,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, l2, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(DD_ERR_CUDA, std::string("cuTensorMapEncodeTiled(") + what + ") failed: " + std::to_string((int)r));
  return DD_OK;
}

// NHWC fp16 plane [B][H][W][C] read in boxes of {box_c, box_w, box_h, 1}.  With stride s > 1 (stride-2 convs) the
// element strides are {1, s, s, 1}: a box spanning box_w x box_h input positions delivers box_w / s x box_h / s pixels.
//   convgen activations  box {bk, 16 s, 8 s}, swizzle_for(bk)
//   halo-kernel strip    box {bk, 8, 18},     swizzle_for(bk)
//   wgrad operand        box {64, 64, 1},     128-byte swizzle (64 channels x 64 pixels of one row)
// ld > C: the C channels from base on of rows that are ld channels wide.
int make_nhwc_map(CUtensorMap* m, const char* what, const __half* base, int B, int H, int W, int C, int box_c, int box_w,
                  int box_h, CUtensorMapSwizzle swizzle, int stride = 1, int ld = 0) {
  const cuuint64_t L = ld > 0 ? ld : C;
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  const cuuint64_t strides[3] = {L * 2, (cuuint64_t)W * L * 2, (cuuint64_t)H * W * L * 2};
  const cuuint32_t box[4] = {(cuuint32_t)box_c, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
  const cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
  return encode_map(m, what, 4, base, dims, strides, box, estr, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
}
// activations of the convgen kernel: 16 x 8 output pixels (sampled with `stride`) by bk channels
int make_act_map(CUtensorMap* m, const __half* base, int B, int H, int W, int C, int bk, int stride = 1, int ld = 0) {
  return make_nhwc_map(m, "activation", base, B, H, W, C, bk, dd::TILE_W * stride, dd::TILE_H * stride, swizzle_for(bk),
                       stride, ld);
}
// halo patch of conv5x5_fold_kernel: the NHWC [B][H][W][256] fp16 plane seen as {8 ch, y, x, channel group, image};
// box = {8, 20, 36, 2, 1} lands in shared memory as [channel group][x][y][8 ch], no swizzle
int make_patch_map(CUtensorMap* m, const __half* base, int B, int H, int W) {
  const cuuint64_t px = 256 * 2;  // bytes per pixel
  const cuuint64_t dims[5] = {8, (cuuint64_t)H, (cuuint64_t)W, 32, (cuuint64_t)B};
  const cuuint64_t strides[4] = {(cuuint64_t)W * px, px, 16, (cuuint64_t)H * W * px};
  const cuuint32_t box[5] = {8, dd::F5::PH, dd::F5::PW, 2, 1};
  const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  return encode_map(m, "patch", 5, base, dims, strides, box, estr, CU_TENSOR_MAP_SWIZZLE_NONE,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
}
// conv weights [taps][cout][cin] fp16 read in boxes of {box_k, rows, 1}: the halo kernel's (9 taps, all cout rows, its
// K chunk) and the convgen kernel's (GEN_BK, one unit's gen_unit_cols rows); ld > cin: cin columns from base on of ld-wide rows
int make_weight_map(CUtensorMap* m, const __half* base, int cout, int cin, int taps, int box_k, int rows, int ld = 0) {
  const cuuint64_t L = ld > 0 ? ld : cin;
  const cuuint64_t dims[3] = {(cuuint64_t)cin, (cuuint64_t)cout, (cuuint64_t)taps};
  const cuuint64_t strides[2] = {L * 2, (cuuint64_t)cout * L * 2};
  const cuuint32_t box[3] = {(cuuint32_t)box_k, (cuuint32_t)rows, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  return encode_map(m, "weight", 3, base, dims, strides, box, estr, swizzle_for(box_k), CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
}

// ---- conv shapes served by the engine
struct ShapeInfo {
  int cin, cout;
};
constexpr ShapeInfo kShapes[5] = {{16, 64}, {64, 256}, {256, 256}, {256, 64}, {64, 16}};
int shape_id(int cin, int cout) {
  for (int i = 0; i < 5; ++i)
    if (kShapes[i].cin == cin && kShapes[i].cout == cout) return i;
  return -1;
}

constexpr int kHaloBK[5] = {16, 32, 32, 32, 32};  // K chunk of the halo kernel per shape id

// One 3x3 conv kernel: conv3x3_simt_kernel (fp32 CUDA cores, reads sa) or the persistent conv3x3_halo_kernel (reads
// the strip maps m[0..1] of the input planes and the weight maps m[2..3]).
template <int CIN, int COUT, int BK, int EPI>
void conv3x3_kernel(bool simt, const dd::SimtArgs& sa, const CUtensorMap* m, const dd::ConvArgs& a, int sm_count,
                    cudaStream_t st) {
  if (simt) {
    constexpr int CO_T = COUT < 64 ? COUT : 64;
    dd::conv3x3_simt_kernel<CIN, COUT, EPI><<<dim3(a.num_tiles, COUT / CO_T), 256, 0, st>>>(sa);
  } else {
    using C = dd::HaloCfg<CIN, COUT, BK>;
    const int grid = a.num_tiles < sm_count ? a.num_tiles : sm_count;
    dd::conv3x3_halo_kernel<CIN, COUT, BK, EPI><<<grid, C::THREADS, C::SMEM_BYTES, st>>>(m[0], m[1], m[2], m[3], a);
  }
}
template <int CIN, int COUT, int BK>
void conv3x3_epi(int epi, bool simt, const dd::SimtArgs& sa, const CUtensorMap* m, const dd::ConvArgs& a, int sm_count,
                 cudaStream_t st) {
  if (epi == dd::EPI_F32_STATS) conv3x3_kernel<CIN, COUT, BK, dd::EPI_F32_STATS>(simt, sa, m, a, sm_count, st);
  else if (epi == dd::EPI_SPLIT) conv3x3_kernel<CIN, COUT, BK, dd::EPI_SPLIT>(simt, sa, m, a, sm_count, st);
  else conv3x3_kernel<CIN, COUT, BK, dd::EPI_F32>(simt, sa, m, a, sm_count, st);
}

// Launch the 3x3 conv of shape `sid` with epilogue `epi` on a's B x H x W grid, from fp16 hi / lo input planes at
// scale in_scale: conv3x3_simt_kernel on 16 x 8 tiles (simt; weights w_simt) or conv3x3_halo_kernel on 8 x 16 tiles
// (weight maps w_hi / w_lo).  Sets a's tile fields to the chosen kernel's tiling; the caller checks the launch.
int launch_conv3x3(int sid, int epi, bool simt, dd::ConvArgs& a, const __half* in_hi, const __half* in_lo,
                   float in_scale, const float* w_simt, const CUtensorMap& w_hi, const CUtensorMap& w_lo, int sm_count,
                   cudaStream_t st) {
  const int tw = simt ? dd::TILE_W : dd::HALO_TW, th = simt ? dd::TILE_H : dd::HALO_TH;
  a.tiles_x = (a.W + tw - 1) / tw;
  a.tiles_y = (a.H + th - 1) / th;
  a.num_tiles = a.tiles_x * a.tiles_y * a.B;
  CUtensorMap m[4] = {{}, {}, w_hi, w_lo};
  dd::SimtArgs sa{};
  if (simt) {
    sa.in_hi = in_hi;
    sa.in_lo = in_lo;
    sa.in_inv_scale = 1.f / in_scale;
    sa.w = w_simt;
    sa.c = a;
  } else {
    const int cin = kShapes[sid].cin, bk = kHaloBK[sid];
    int rc;
    if ((rc = make_nhwc_map(&m[0], "strip", in_hi, a.B, a.H, a.W, cin, bk, dd::HALO_TW, dd::HALO_TH + 2, swizzle_for(bk))))
      return rc;
    if ((rc = make_nhwc_map(&m[1], "strip", in_lo, a.B, a.H, a.W, cin, bk, dd::HALO_TW, dd::HALO_TH + 2, swizzle_for(bk))))
      return rc;
  }
  switch (sid) {
    case 0: conv3x3_epi<16, 64, kHaloBK[0]>(epi, simt, sa, m, a, sm_count, st); break;
    case 1: conv3x3_epi<64, 256, kHaloBK[1]>(epi, simt, sa, m, a, sm_count, st); break;
    case 2: conv3x3_epi<256, 256, kHaloBK[2]>(epi, simt, sa, m, a, sm_count, st); break;
    case 3: conv3x3_epi<256, 64, kHaloBK[3]>(epi, simt, sa, m, a, sm_count, st); break;
    case 4: conv3x3_epi<64, 16, kHaloBK[4]>(epi, simt, sa, m, a, sm_count, st); break;
    default: return fail(DD_ERR_UNSUPPORTED, "unsupported conv shape");
  }
  return DD_OK;
}

template <int CIN, int COUT, int BK>
cudaError_t configure_halo_all_epi() {
  using C = dd::HaloCfg<CIN, COUT, BK>;
  cudaError_t e;
  if ((e = cudaFuncSetAttribute(dd::conv3x3_halo_kernel<CIN, COUT, BK, dd::EPI_F32_STATS>,
                                cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES)) != cudaSuccess) return e;
  if ((e = cudaFuncSetAttribute(dd::conv3x3_halo_kernel<CIN, COUT, BK, dd::EPI_SPLIT>,
                                cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES)) != cudaSuccess) return e;
  return cudaFuncSetAttribute(dd::conv3x3_halo_kernel<CIN, COUT, BK, dd::EPI_F32>,
                              cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
}
template <int MCO, int NCI>
cudaError_t configure_wgm() {
  return cudaFuncSetAttribute(dd::wgrad_wgmma_kernel<MCO, NCI>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              dd::WgmCfg<MCO, NCI>::SMEM_BYTES);
}
template <int NT>
cudaError_t configure_gen() {
  return cudaFuncSetAttribute(dd::convgen_wgmma_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              dd::GenCfg<NT>::SMEM_BYTES);
}
cudaError_t configure_all_kernels() {
  cudaError_t e;
  if ((e = cudaFuncSetAttribute(dd::window_attention_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                dd::WAU_SMEM)) != cudaSuccess) return e;
  if ((e = cudaFuncSetAttribute(dd::decoder_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dd::DEC_SMEM)) != cudaSuccess)
    return e;
  if ((e = configure_halo_all_epi<16, 64, 16>()) != cudaSuccess) return e;
  if ((e = configure_halo_all_epi<64, 256, 32>()) != cudaSuccess) return e;
  if ((e = configure_halo_all_epi<256, 256, 32>()) != cudaSuccess) return e;
  if ((e = configure_halo_all_epi<256, 64, 32>()) != cudaSuccess) return e;
  if ((e = configure_halo_all_epi<64, 16, 32>()) != cudaSuccess) return e;
  if ((e = cudaFuncSetAttribute(dd::conv5x5_fold_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                dd::F5::SMEM_BYTES)) != cudaSuccess) return e;
  if ((e = cudaFuncSetAttribute(dd::ring_fix_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dd::RING_SMEM)) !=
      cudaSuccess) return e;
  if ((e = configure_wgm<128, 128>()) != cudaSuccess) return e;
  if ((e = configure_wgm<128, 64>()) != cudaSuccess) return e;
  if ((e = configure_wgm<64, 128>()) != cudaSuccess) return e;
  if ((e = configure_gen<256>()) != cudaSuccess) return e;
  if ((e = configure_gen<192>()) != cudaSuccess) return e;
  if ((e = configure_gen<128>()) != cudaSuccess) return e;
  return configure_gen<64>();
}

struct ConvLayer {
  int sid = -1;
  __half* w_hi = nullptr;
  __half* w_lo = nullptr;
  float* w_simt = nullptr;
  float* bias = nullptr;
  float wscale = 1.f;
  CUtensorMap mh_hi, mh_lo;  // box for the halo kernel's K chunk
};

// Pinned host side of the denoiser / codec pack, so that its copies are asynchronous and one synchronisation serves a
// whole pack: the abs-max words of the conv weights, the decoder's and encoder's raw tensors as last registered (an
// update re-reads only the registered ones; the BatchNorm folds need all of them), and what the host folds produce.
struct PackStage {
  float amax[16];  // slot i: conv layer i (0..5), 6 + i: its data-gradient layer, 12: the composed 5x5 conv
  // device -> host
  float dec_wt[16 * 16 * 16], dec_bt[16], dec_g[16], dec_be[16], dec_mu[16], dec_var[16], dec_wc[16 * 9], dec_bc[1];
  float enc_w1[144], enc_bn1[4][16], enc_w2[2304], enc_bn2[4][16];
  // host -> device
  float wt_f[4 * 4 * 16 * 16], bt_f[16], wc_f[9 * 16], wu[4 * 4 * 16 * 16], bn[3 * 16];
  float f1[144], t1[16], f2[2304], t2[16];
  float e1u[144], e2u[2304], enc_gb[4][16];  // unfolded encoder for DD_CODEC_TRAIN: [tap][co], [tap][ci][co]; gamma / beta
  float enc_bn[2][3][16];                     // the encoder backward's running-statistics BatchNorms: s, mean, rstd
};

struct Raw {
  const float* ptr;
  std::vector<int64_t> shape;
};

// One layer on the convgen_wgmma_kernel path: a producer convolution (neck / FPN / backbone; eval-BN folded into the
// weights and `shift`) or a Linear (taps = 1, `shift` = its bias, zeros if it has none).
struct GenLayer {
  int cin = 0, cout = 0, taps = 1, nt = 256, relu = 1, shuffle = 0;
  int stride = 1, add_first = 0;
  __half* w_hi = nullptr;
  __half* w_lo = nullptr;
  float* shift = nullptr;
  float wscale = 1.f;
  CUtensorMap mb_hi, mb_lo;
  bool alt = false;          // cout divisible by 256 and 192: launch_gen picks the width whose last wave wastes least
  CUtensorMap mb_hi_alt, mb_lo_alt;  // for N tiles of 192 columns
  float* zero_shift = nullptr;       // layers deep enough to be split along K (gen_parts): the partial launches' shift
  int bn = -1;                       // index of its training-mode BatchNorm pack in dd_engine::pt.layers (-1: none)
};

// K iterations (64-channel chunk x tap, 12 wgmma each) that one fp32 wgmma accumulator of convgen_wgmma_kernel takes.
// The accumulator loses a little at every wgmma: measured against fp64, 1,152 wgmma stay at 0.8 of the 3e-5 bound and
// 2,160 / 2,592 / 3,456 wgmma reach 3.7e-5 / 5.8e-5 / 7.9e-5.  Deeper layers (the level 1..3 fusion convs of the HAHI
// neck and the widest FPN laterals of Swin) run as gen_parts launches over contiguous channel ranges, summed in fp32 in
// a fixed order through an fp32 partial buffer (launch_gen).
constexpr int kGenSplitIters = 110;
int gen_parts(int taps, int kc_total) { return (taps * kc_total + kGenSplitIters - 1) / kGenSplitIters; }
int gen_chunks(int c) { return (c + dd::GEN_BK - 1) / dd::GEN_BK; }
struct Planes {
  __half* hi = nullptr;
  __half* lo = nullptr;
};
struct SwinBlockW {
  float *ln1_g = nullptr, *ln1_b = nullptr, *ln2_g = nullptr, *ln2_b = nullptr, *table = nullptr;
  GenLayer qkv, proj, ffn1, ffn2;
};
struct SwinStageW {
  std::vector<SwinBlockW> blocks;
  float *out_g = nullptr, *out_b = nullptr, *dn_g = nullptr, *dn_b = nullptr;
  GenLayer reduction;
};
struct Backbone {
  bool enabled = false, ready = false;
  int E = 0, window = 7, H = 0, W = 0;
  int depths[4] = {0, 0, 0, 0}, heads[4] = {0, 0, 0, 0}, Hs[4] = {0, 0, 0, 0}, Ws[4] = {0, 0, 0, 0};
  float *pe_w = nullptr, *pe_b = nullptr, *pe_g = nullptr, *pe_beta = nullptr;
  SwinStageW stage[4];
  // workspace views
  float* X[2] = {nullptr, nullptr};
  float* QKV = nullptr;
  Planes AP, HP;
};
struct Producers {
  bool enabled = false, ready = false, neck = false;
  int nlev = 0;
  int C[4] = {0, 0, 0, 0}, H[4] = {0, 0, 0, 0}, W[4] = {0, 0, 0, 0};
  GenLayer lat[4], proj[4], fus[4], fl[4], fu[3];
  Planes F[4], L[4], P[4], O[4], XP[4];
  float* X[4] = {nullptr, nullptr, nullptr, nullptr};   // fp32 NHWC FPN outputs (X[0] aliases the loop's cond)
  float* UP[3] = {nullptr, nullptr, nullptr};           // fp32 NHWC upsampled maps at level i
  bool resample = false;                                // pyramid is not exactly 2x: adaptive_avg_pool2d is a real resample
  float* UPR[3] = {nullptr, nullptr, nullptr};          // raw ConvT output [B, 2H[i+1], 2W[i+1], 256] before pooling to level i
  float* KS = nullptr;                                  // fp32 partial sums of the convs split along K (gen_parts)
};
struct ResBlockW {
  GenLayer c1, c2, ds;
  bool has_ds = false;
};
struct ResNetW {
  bool enabled = false, ready = false;
  int H = 0, W = 0;
  int depths[4] = {0, 0, 0, 0}, C[4] = {64, 128, 256, 512}, Hs[4] = {0, 0, 0, 0}, Ws[4] = {0, 0, 0, 0};
  std::vector<ResBlockW> blocks[4];
  Planes IN, T, Yp[2];
  float* Y32[2] = {nullptr, nullptr};
  float* D32 = nullptr;
};

// MPViT (reference backbone/mpvit.py): depthwise layers as tap-major fp32 tables, every 1x1 conv / Linear on the GEMM path
struct DwLayer {
  int C = 0, K = 3;
  float* w = nullptr;     // [K*K][C], eval-BN scale folded in
  float* bias = nullptr;  // [C]
  int bn = -1;            // index of its training-mode BatchNorm record in dd_engine::pt.layers (-1: none)
  float *raw_w = nullptr, *raw_bias = nullptr;  // with a record: the weights unfolded, and a zero bias
};
struct MpBlockW {
  float *ln1_g = nullptr, *ln1_b = nullptr, *ln2_g = nullptr, *ln2_b = nullptr;
  GenLayer qkv, proj, fc1, fc2;
};
struct MpEncoderW {
  DwLayer cpe;              // ConvPosEnc, shared by the encoder's layers
  float* crpe_w = nullptr;  // [49][C]: the 3 / 5 / 7 windows of the head groups, centred in one 7 x 7 layout
  float* crpe_b = nullptr;
  std::vector<MpBlockW> layers;
};
struct MpStageW {
  DwLayer pe_dw[4], inv_dw;
  GenLayer pe_pw[4], inv1, inv2, agg;
  MpEncoderW enc[4];
};
constexpr int kMpHeads = 8;        // MPViT's attention heads in every stage
constexpr int kMpChunksMax = 256;  // token chunks of the factorised attention's reductions
// the factorised attention's token-chunk partials, sized for kMpChunksMax chunks
struct FactorAttBufs {
  float *part_m = nullptr, *part_s = nullptr, *colinv = nullptr, *part_ktv = nullptr, *ktv = nullptr;
};
struct MPViTW {
  bool enabled = false, ready = false;
  int H = 0, W = 0, heads = kMpHeads, mlp_ratio = 4;
  int dims[4] = {0, 0, 0, 0}, out_dims[4] = {0, 0, 0, 0}, layers[4] = {0, 0, 0, 0}, paths[4] = {0, 0, 0, 0};
  int Hs[4] = {0, 0, 0, 0}, Ws[4] = {0, 0, 0, 0};
  GenLayer stem0, stem1;
  MpStageW stage[4];
  // workspace views
  Planes IN, S1, D, EP0, AP, HP, CAT;
  float* XS = nullptr;      // stem output, then each stage's output (fp32 NHWC)
  float* E[4] = {nullptr, nullptr, nullptr, nullptr};  // the paths' token maps + one swap buffer
  float* R1 = nullptr;
  float* QKV = nullptr;
  FactorAttBufs fab;
};

// Stochastic depth of the native backbone (dd_backbone_config.mp_drop_path, dd_set_drop_path).  Bit k of mask[s] marks
// block k of stage s: an MPViT encoder layer (in every path) or a Swin block, each with two residual branches (attention,
// then MLP / FFN); blocks counts the marked blocks (MPViT: times the stage's paths).  While on, scales holds
// [block][branch][B] per-sample scales, blocks in stage(, path), block order.
struct DropPathState {
  int mask[4] = {0, 0, 0, 0}, blocks = 0;
  bool on = false;
  float* scales = nullptr;
};

}  // namespace

struct dd_engine {
  dd_config cfg;
  int sm_count = 0;
  bool weights_ready = false;
  bool packed = false;  // a dd_finalize_weights has completed and its buffers are intact (dd_update_weights needs that)
  std::map<std::string, Raw> raw;
  // packed parameters (device memory owned by the engine)
  ConvLayer L[12];  // 0 ne.0, 1 ne.3, 2 convA, 3 convB, 4 pred.0, 5 pred.3; 6 + i: the data-gradient conv of layer i
                    // (flipped, transposed weights, zero bias; DD_FLAG_BACKWARD only)
  struct Fold {  // convB -> pred.0 composed into one 5x5 conv (Swin, unless DD_FLAG_CHAIN_PRED / DD_FLAG_SIMT_CONV)
    __half* w = nullptr;     // packed K5 hi / lo (pred_fold.cuh)
    float* bias = nullptr;   // b5 [64]
    float wscale = 1.f;
    float* src[2] = {nullptr, nullptr};  // convB's and pred.0's weights as registered: an update of one composes with the other
    double* k5 = nullptr;                // [64][256][25] the composition in fp64, and its magnitudes for the scale
    float* k5_abs = nullptr;
    float* edge = nullptr;               // the ring correction's edge kernels (dd::EDGE_ELEMS)
  } fold;
  float* w_flip[6] = {};       // data-gradient layer 6 + i: layer i's weights flipped and transposed, before the split
  float* amax = nullptr;       // [16] abs-max words of the pack (PackStage::amax)
  PackStage* stage = nullptr;  // pinned
  cudaEvent_t pack_done = nullptr;  // after the last pack's copies out of `stage`: the next pack's stream waits for it
  float* gn_gamma[4] = {nullptr, nullptr, nullptr, nullptr};  // ne.1, ne.4, pred.1, pred.4
  float* gn_beta[4] = {nullptr, nullptr, nullptr, nullptr};
  float* temb = nullptr;    // [1280][256]
  float* dec_wt = nullptr;  // [4][4][16][16] folded
  float* dec_bt = nullptr;  // [16]
  float* dec_wc = nullptr;  // [9][16]
  float dec_bc = 0.f;
  float* dec_wu = nullptr;  // [4][4][16][16] unfolded ConvT weights, [ky][kx][ci][co]
  float* dec_bu = nullptr;  // [16] unfolded ConvT bias
  float* dec_bn = nullptr;  // [3][16] BatchNorm scale gamma * rstd, running mean, rstd
  float *enc_w1 = nullptr, *enc_b1 = nullptr, *enc_w2 = nullptr, *enc_b2 = nullptr;  // folded encoder (optional)
  float* enc_bn = nullptr;  // [2][3][16] encoder BatchNorms 1, 2 on running statistics: s = gamma rstd, mean, rstd
  // DD_CODEC_TRAIN (dd_set_codec_mode): the codec's BatchNorms on batch statistics.  The unfolded parameters (filled
  // with the pack), the batch-folded copies decoder_kernel / encoder_kernel run on, and the statistics' scratch; all
  // engine-owned, so the workspace size does not depend on the mode.
  int codec_mode = DD_CODEC_EVAL;
  struct CodecTrain {
    float *dec_gb = nullptr;                                  // [2][16] decoder BatchNorm weight, bias
    float *dec_wt = nullptr, *dec_bt = nullptr, *dec_bn = nullptr;  // batch-folded decoder; [3][16] s, mean, rstd
    float* zero16 = nullptr;  // [16] zeros: the ConvT bias of the decoder backward's xhat (bn's mean is bias-free)
    float *enc_w1 = nullptr, *enc_w2 = nullptr, *enc_gb = nullptr;  // unfolded encoder; [4][16] gamma1, beta1, gamma2, beta2
    float *enc_w1f = nullptr, *enc_b1f = nullptr, *enc_w2f = nullptr, *enc_b2f = nullptr;  // batch-folded encoder
    float* enc_bn = nullptr;  // [2][3][16] the encoder backward's batch s, mean, rstd (layout of dd_engine::enc_bn)
    double *part = nullptr, *sum1 = nullptr;     // bn_stats_kernel partials [blocks][2][16]; pass-1 sums [16]
    double *sums = nullptr, *part_db = nullptr;  // decoder backward: [32] sum dv, sum dv xhat; [act blocks][16]
    float* rec = nullptr;                        // [max(T, 2)][2][16] batch mean, unbiased variance
    int nrec = 0;                                // records the last forward entry wrote
  } ct;
  // DD_PRODUCER_TRAIN (dd_set_producer_mode; DD_FLAG_PRODUCER_TRAIN): the producers' BatchNorms on batch statistics.
  // Every BatchNorm'ed producer layer, in evaluation order (ResNet bn1 / bn2 block by block, then per level the neck's
  // lateral / proj / fusion, then the FPN top-down: lateral, conv_up), keeps an unfolded pack of its conv and device
  // copies of gamma / beta; the scratch below is engine-owned and sized for the largest layer.  The eval layer names
  // its record (GenLayer::bn).
  int producer_mode = DD_PRODUCER_EVAL;
  struct ProdBn {
    GenLayer raw;                    // conv (or ConvT) weights alone: no BatchNorm, zero shift
    float *gamma = nullptr, *beta = nullptr;
    int C = 0;                       // BatchNorm channels
    int stage = 0;                   // 0: dd_run_backbone, 1: dd_build_condition
    long long n = 0;                 // pixels of the pre-BN output (a ConvT's: B x 2H x 2W)
    bool fresh = false;              // evaluated in DD_PRODUCER_TRAIN since the forward started
    size_t rec_off = 0;              // floats into `rec`: [2][C] batch mean, unbiased batch variance
    std::string key;                 // registered key prefix of the BatchNorm
  };
  struct ProdTrain {
    std::vector<ProdBn> layers;
    float* U = nullptr;                              // pre-BN conv output, fp32 NHWC
    double *part = nullptr, *sum1 = nullptr;         // pbn_stats_kernel partials [blocks][2][C]; pass-1 sums [C]
    float *s = nullptr, *t = nullptr, *rec = nullptr;  // batch scale / shift [C]; records
    size_t rec_floats = 0;
  } pt;
  // dd_set_bn_allgather: every training-mode BatchNorm takes the statistics of the union of all ranks' batches.  Each
  // statistics pass sends this rank's totals and pixel count (`row`) through `fn`; the gathered rows are summed in rank
  // order into tot1 (pass 1, and the decoder backward) or tot2 (pass 2), which the fold kernels read as one block.
  struct BnSync {
    dd_allgather_fn fn = nullptr;
    void* user = nullptr;
    int world = 1;
    int cap = 0;  // doubles per row the buffers hold (grown on first use by a wider layer)
    double *row = nullptr, *rows = nullptr, *tot1 = nullptr, *tot2 = nullptr;  // [cap], [world][cap], [cap], [cap]
  } sync;
  std::vector<void*> owned;
  // schedule
  std::vector<int64_t> ts;
  std::vector<float> cx, ce;
  // workspace views
  void* ws = nullptr;
  float *x32 = nullptr, *Y = nullptr, *cond = nullptr, *mr[4] = {}, *temb_sel = nullptr;
  double* stats[4] = {};  // GroupNorm partials [tiles][4][2] of the conv before each norm
  __half *xs_hi = nullptr, *xs_lo = nullptr, *S_hi[2] = {}, *S_lo[2] = {};
  int* status = nullptr;
  struct Bwd {  // dd_denoiser_backward's region (DD_FLAG_BACKWARD): the recomputed forward and the gradient buffers
    float *y1 = nullptr, *y2 = nullptr, *y5 = nullptr, *y6 = nullptr;  // pre-GN conv outputs
    Planes a1, f0, fa, fp, a5;               // conv input planes (noise_embedding.0 reads xs_hi / xs_lo)
    float *g[2] = {nullptr, nullptr};        // gradient ping-pong [B][P][256]
    Planes gp;                               // split planes of the gradient a data-gradient conv reads
    float *gn_part = nullptr, *ab = nullptr, *col_part = nullptr, *dtemb = nullptr, *dcond = nullptr;
    float *scales = nullptr, *amax = nullptr;  // [kBwdSlots] on-device gradient scales and their absmax inputs
    double* wg_part = nullptr;
  } bw;
  struct LoopBwd {  // dd_denoise_backward's region (DD_FLAG_LOOP_BACKWARD)
    float* stash = nullptr;     // [T + 1][B][P][16] the loop's latents x_T .. x_0
    float* gl = nullptr;        // [B][P][16] running latent gradient
    float* stage = nullptr;     // one step's parameter gradients, laid out as `acc`
    double* acc = nullptr;      // parameter gradients summed over the steps (time_embedding dense)
    double* acc_cond = nullptr; // [B][cond_h][cond_w][256]
    float *z = nullptr, *r = nullptr, *du = nullptr;  // decoder backward: logit / dz [B][2h][2w], r and du [..][16]
    double *part_act = nullptr, *part_wc = nullptr, *part_wt = nullptr;
  } lp;
  int stats_tiles_img[4] = {0, 0, 0, 0};  // tiles per image of the kernel that last filled stats[i]
  // graph
  Producers prod;
  Backbone bb;
  ResNetW rn;
  MPViTW mp;
  DropPathState drop;  // of whichever of bb / mp is enabled
  bool feats_ready = false;  // dd_run_backbone has filled the neck's input planes
  bool cond_ready = false;  // dd_build_condition has filled `cond` for the next dd_denoise_decode(cond = NULL)
  // CUDA graphs (DD_FLAG_CUDA_GRAPH), captured on first use and replayed: the T-step loop, the same loop with a decode
  // after every step (dd_denoise_decode_steps), the native backbone, the neck + FPN
  // (G_LOOP_STEPS_TRAIN: the step-decode loop in DD_CODEC_TRAIN, batch statistics before every decode)
  // (G_BACKBONE_TRAIN, G_COND_TRAIN: the native backbone and the neck + FPN in DD_PRODUCER_TRAIN; G_BACKBONE_DROP,
  // G_BACKBONE_TRAIN_DROP: the MPViT or Swin backbone with stochastic depth on, in either producer mode)
  enum {
    G_LOOP = 0, G_LOOP_STEPS = 1, G_BACKBONE = 2, G_COND = 3, G_LOOP_STEPS_TRAIN = 4, G_BACKBONE_TRAIN = 5,
    G_COND_TRAIN = 6, G_BACKBONE_DROP = 7, G_BACKBONE_TRAIN_DROP = 8, G_COUNT = 9
  };
  cudaGraphExec_t graphs[G_COUNT] = {};
  int64_t graph_launches[G_COUNT] = {};  // kernel nodes per graph (added to `launches` per replay)
  int64_t graph_captures = 0;                      // graph instantiations since dd_create (dd_graph_capture_count)
  cudaStream_t cap_stream = nullptr;  // capture happens here (the caller's stream may be the legacy default stream)
  float* rgb_stage = nullptr;         // workspace copy of the image batch the backbone graph reads
  float* inter = nullptr;             // [T][B][2h][2w] per-step decoded depth (DD_FLAG_STEP_DECODE)
  int64_t launches = 0;
  int* status_host = nullptr;  // pinned
};

namespace {

int launched(dd_engine* e, const char* what) {
  e->launches++;
  return check_launch(what);
}

constexpr float kActScale = 16.f;  // power-of-two pre-scale of conv inputs before the fp16 split
constexpr float kXScale = 1.f;     // the raw latent keeps scale 1 (random-init trajectories reach |x| ~ 5e2)

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

struct Carver {
  uint8_t* base;
  size_t off = 0;
  template <typename T>
  T* take(size_t n) {
    off = align_up(off, 1024);
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += n * sizeof(T);
    return p;
  }
};

struct Geom {
  int B, h, w, P, tiles_x, tiles_y, tiles_img, tiles;  // tiles of the conv kernel selected by cfg.flags
  int tiles_max;                                       // max over both tilings (buffer sizing)
};
Geom geom_of(const dd_config& c) {
  Geom g;
  g.B = c.batch;
  g.h = c.latent_h;
  g.w = c.latent_w;
  g.P = g.h * g.w;
  const int t816 = ((g.w + dd::TILE_W - 1) / dd::TILE_W) * ((g.h + dd::TILE_H - 1) / dd::TILE_H);
  const int t168 = ((g.w + dd::HALO_TW - 1) / dd::HALO_TW) * ((g.h + dd::HALO_TH - 1) / dd::HALO_TH);
  g.tiles_x = (g.w + dd::TILE_W - 1) / dd::TILE_W;
  g.tiles_y = (g.h + dd::TILE_H - 1) / dd::TILE_H;
  g.tiles_img = g.tiles_x * g.tiles_y;
  g.tiles = g.tiles_img * g.B;
  g.tiles_max = (t816 > t168 ? t816 : t168) * g.B;
  return g;
}

// ---- backward (DD_FLAG_BACKWARD)
constexpr int kBwdSlots = 16;  // gradient splits per dd_denoiser_backward call (at most 6 are used)
// conv layer i: reference key prefix, Cout, Cin
const char* const kConvKey[6] = {"model.noise_embedding.0", "model.noise_embedding.3", "model.upsample_fuse.convA.conv",
                                 "model.upsample_fuse.convB.conv", "model.pred.0", "model.pred.3"};
constexpr int kConvCout[6] = {64, 256, 256, 256, 64, 16};
constexpr int kConvCin[6] = {16, 64, 256, 256, 256, 64};
// Split-K plan of wgrad_simt_kernel: about 16 blocks per SM in all, each chunk a multiple of the fp32 flush interval.
struct WgPlan {
  int chunks, chunk;
};
WgPlan wgrad_plan(int cout, int cin, long long BP) {
  const int tiles = (cout / std::min(64, cout)) * (cin / std::min(64, cin)) * 9;
  long long chunks = std::max(1, std::min(128, (2112 + tiles - 1) / tiles));
  long long chunk = (BP + chunks - 1) / chunks;
  chunk = std::max<long long>(dd::WG_KS * dd::WG_FLUSH, (chunk + dd::WG_KS - 1) / dd::WG_KS * dd::WG_KS);
  chunks = (BP + chunk - 1) / chunk;
  return {static_cast<int>(chunks), static_cast<int>(chunk)};
}
int bwd_chunks(int P) { return (P + dd::BWD_CHUNK - 1) / dd::BWD_CHUNK; }
// Shapes whose weight gradient runs on wgrad_wgmma_kernel: the 256-wide ones.  The two 16-channel shapes keep
// wgrad_simt_kernel (3.6 of 192 ms of a backward call at B = 4, 176 x 608).
bool wgrad_on_tc(int cout, int cin) { return cout == 256 || cin == 256; }
constexpr int kWgmSegs = 128;  // 64-pixel row segments per CTA of wgrad_wgmma_kernel (8192 pixels summed in fp32)
int wgm_chunks(int B, int H, int W) {
  const int nseg = B * H * ((W + 63) / 64);
  return (nseg + kWgmSegs - 1) / kWgmSegs;
}
// fp64 partials run_wgrad writes for one (cout, cin) conv at B x H x W
size_t wgrad_partial_elems(int cout, int cin, int B, int H, int W) {
  const int chunks = wgrad_on_tc(cout, cin) ? wgm_chunks(B, H, W)
                                            : wgrad_plan(cout, cin, static_cast<long long>(B) * H * W).chunks;
  return static_cast<size_t>(chunks) * cout * cin * 9;
}
// DD_FLAG_LOOP_BACKWARD implies DD_FLAG_BACKWARD
bool has_backward(const dd_config& c) { return (c.flags & (DD_FLAG_BACKWARD | DD_FLAG_LOOP_BACKWARD)) != 0; }
// Elements of the denoiser's parameters in dd_denoiser_backward's order (time_embedding dense); offsets into lp.acc.
constexpr size_t kParamNumel[21] = {64 * 16 * 9, 64, 64, 64, 256 * 64 * 9, 256, 256, 256, DD_TIME_ROWS * 256,
                                    64 * 256 * 9, 64, 64, 64, 16 * 64 * 9, 16, 16, 16,
                                    256 * 256 * 9, 256, 256 * 256 * 9, 256};
int param_count(const dd_config& c) { return c.variant == DD_VARIANT_SWIN ? 21 : 17; }
size_t param_offset(int i) {
  size_t o = 0;
  for (int k = 0; k < i; ++k) o += kParamNumel[k];
  return o;
}
// block counts of the decoder backward's reductions
int dec_act_blocks(const Geom& g) { return static_cast<int>((static_cast<size_t>(g.B) * g.P * 4 + dd::DEC_ACT_PIX - 1) / dd::DEC_ACT_PIX); }
int dec_wc_blocks(const Geom& g) { return static_cast<int>((static_cast<size_t>(g.B) * g.P * 4 + dd::DEC_WC_PIX - 1) / dd::DEC_WC_PIX); }
int dec_wt_blocks(const Geom& g) { return static_cast<int>((static_cast<size_t>(g.B) * g.P + dd::DEC_WT_PIX - 1) / dd::DEC_WT_PIX); }
// blocks of bn_stats_kernel over n items (the decoder's B x 2h x 2w is the largest codec BatchNorm)
int codec_stats_blocks(long long n) { return static_cast<int>((n + dd::BNS_PIX - 1) / dd::BNS_PIX); }

void free_bn_sync(dd_engine* e) {
  dd_engine::BnSync& s = e->sync;
  for (double* p : {s.row, s.rows, s.tot1, s.tot2})
    if (p) cudaFree(p);
  s.row = s.rows = s.tot1 = s.tot2 = nullptr;
  s.cap = 0;
}

// What a consumer of batch statistics reads: totals, and the count to divide them by (null: its own item count).
struct BnTotals {
  const double* sum;
  const double* cnt;
};

// The totals of columns [0, ncols) of nblk block partials (stride doubles apart), summed in block order.  On one GPU
// they go to `local`.  Across ranks (dd_set_bn_allgather) this rank's totals and its item count n go out as one row,
// and every rank's row summed in rank order (the count last) lands in tot1 when reserve > 0: the BatchNorm's first
// gather, which makes room for its widest row of `reserve` columns; or in tot2 when reserve is 0 (its second).
int bn_totals(dd_engine* e, const double* part, int nblk, int stride, int ncols, long long n, double* local,
              int reserve, cudaStream_t st, BnTotals* out) {
  dd_engine::BnSync& s = e->sync;
  int rc;
  if (!s.fn) {
    dd::part_colsum_kernel<<<(ncols + 255) / 256, 256, 0, st>>>(part, nblk, stride, ncols, local, 0);
    *out = {local, nullptr};
    return launched(e, "part_colsum");
  }
  if (reserve > s.cap) {  // wait for the old buffers' readers (tot1 / tot2 hold nothing across BatchNorms), then grow
    CUDA_TRY(cudaStreamSynchronize(st));
    free_bn_sync(e);
    const size_t b = static_cast<size_t>(reserve) * sizeof(double);
    if (cudaMalloc(&s.row, b) != cudaSuccess || cudaMalloc(&s.rows, b * s.world) != cudaSuccess ||
        cudaMalloc(&s.tot1, b) != cudaSuccess || cudaMalloc(&s.tot2, b) != cudaSuccess) {
      free_bn_sync(e);
      return fail(DD_ERR_CUDA, std::string("cudaMalloc: ") + cudaGetErrorString(cudaGetLastError()));
    }
    s.cap = reserve;
  }
  const int cols = ncols + 1;
  dd::part_colsum_kernel<<<(cols + 255) / 256, 256, 0, st>>>(part, nblk, stride, ncols, s.row, n);
  if ((rc = launched(e, "part_colsum"))) return rc;
  const int r = s.fn(s.row, s.rows, cols, st, s.user);
  if (r != 0) return fail(DD_ERR_CUDA, "BatchNorm statistics all-gather callback failed (returned " + std::to_string(r) + ")");
  double* tot = reserve > 0 ? s.tot1 : s.tot2;
  dd::bn_rank_sum_kernel<<<(cols + 255) / 256, 256, 0, st>>>(s.rows, s.world, cols, tot);
  *out = {tot, tot + ncols};
  return launched(e, "bn_rank_sum");
}

// One training-mode BatchNorm over n items of C channels: two statistics passes into the partials part [nblk][2][C]
// (pass-1 totals on one GPU in sum1_local), then the fold.  stats(sum1, cnt) launches a pass (pass 1: both null);
// fold(const dd::BnFoldIn&) launches the fold.
template <class Stats, class Fold>
int run_bn_passes(dd_engine* e, double* part, int nblk, int C, long long n, double* sum1_local, cudaStream_t st,
                  const Stats& stats, const Fold& fold) {
  BnTotals t1, t2;
  int rc;
  if ((rc = stats(nullptr, nullptr))) return rc;
  if ((rc = bn_totals(e, part, nblk, 2 * C, C, n, sum1_local, 2 * C + 1, st, &t1))) return rc;
  if ((rc = stats(t1.sum, t1.cnt))) return rc;
  if (!e->sync.fn) return fold(dd::BnFoldIn{t1.sum, part, nblk, n, nullptr});
  if ((rc = bn_totals(e, part, nblk, 2 * C, 2 * C, n, nullptr, 0, st, &t2))) return rc;
  return fold(dd::BnFoldIn{t1.sum, t2.sum, 1, n, t2.cnt});
}

void drop_graph(dd_engine* e, int which) {
  if (e->graphs[which]) {
    cudaGraphExecDestroy(e->graphs[which]);
    e->graphs[which] = nullptr;
  }
}
void drop_graphs(dd_engine* e) {
  for (int i = 0; i < dd_engine::G_COUNT; ++i) drop_graph(e, i);
}

// Capture `body(stream)` into graph slot `which` on first use, then replay it on `st`.  Every pointer the body's kernels
// take must live in the workspace or in engine-owned memory (caller buffers are staged in / copied out around the graph).
template <typename F>
int graph_run(dd_engine* e, int which, cudaStream_t st, F&& body) {
  if (!e->graphs[which]) {
    cudaGraph_t graph = nullptr;
    const int64_t before = e->launches;
    CUDA_TRY(cudaStreamBeginCapture(e->cap_stream, cudaStreamCaptureModeThreadLocal));
    const int rc = body(e->cap_stream);
    const cudaError_t ce = cudaStreamEndCapture(e->cap_stream, &graph);
    e->graph_launches[which] = e->launches - before;
    e->launches = before;
    if (rc != DD_OK) {
      if (graph) cudaGraphDestroy(graph);
      return rc;
    }
    if (ce != cudaSuccess) return fail(DD_ERR_CUDA, std::string("graph capture: ") + cudaGetErrorString(ce));
    const cudaError_t ci = cudaGraphInstantiate(&e->graphs[which], graph, 0);
    cudaGraphDestroy(graph);
    if (ci != cudaSuccess) return fail(DD_ERR_CUDA, std::string("graph instantiate: ") + cudaGetErrorString(ci));
    e->graph_captures++;
  }
  CUDA_TRY(cudaGraphLaunch(e->graphs[which], st));
  e->launches += e->graph_launches[which];
  return DD_OK;
}

// Lay the workspace out.  With base == nullptr only the size is computed (the engine's views are untouched).
size_t carve(dd_engine* e, void* base) {
  const Geom g = geom_of(e->cfg);
  const size_t BP = static_cast<size_t>(g.B) * g.P;
  Carver c{reinterpret_cast<uint8_t*>(base)};
  dd_engine tmp_views;  // scratch target when only sizing
  dd_engine* v = base ? e : &tmp_views;
  v->status = c.take<int>(16);
  v->x32 = c.take<float>(BP * 16);
  v->xs_hi = c.take<__half>(BP * 16);
  v->xs_lo = c.take<__half>(BP * 16);
  v->Y = c.take<float>(BP * 256);
  for (int i = 0; i < 2; ++i) {
    v->S_hi[i] = c.take<__half>(BP * 256);
    v->S_lo[i] = c.take<__half>(BP * 256);
  }
  v->cond = c.take<float>(static_cast<size_t>(g.B) * e->cfg.cond_h * e->cfg.cond_w * 256);
  for (int i = 0; i < 4; ++i) {
    v->stats[i] = c.take<double>(static_cast<size_t>(g.tiles_max) * 8);
    v->mr[i] = c.take<float>(static_cast<size_t>(g.B) * 8);
  }
  v->temb_sel = c.take<float>(static_cast<size_t>(g.B) * 256);
  if (e->cfg.flags & DD_FLAG_STEP_DECODE)
    v->inter = c.take<float>(static_cast<size_t>(e->cfg.num_inference_steps) * BP * 4);
  if (e->rn.enabled || e->bb.enabled || e->mp.enabled)
    v->rgb_stage = c.take<float>(static_cast<size_t>(g.B) * 3 *
                                 (e->rn.enabled ? e->rn.H * e->rn.W : (e->mp.enabled ? e->mp.H * e->mp.W : e->bb.H * e->bb.W)));
  if (e->prod.enabled) {
    const Producers& pc = e->prod;
    Producers* pv = &v->prod;
    size_t ks = 0;  // the largest output of a conv split along K: neck fusion (C + 512 -> C), FPN lateral (C -> 256)
    for (int i = 0; i < pc.nlev; ++i) {
      const size_t px = static_cast<size_t>(g.B) * pc.H[i] * pc.W[i];
      if (pc.neck && gen_parts(9, gen_chunks(pc.C[i]) + gen_chunks(512)) > 1) ks = std::max(ks, px * pc.C[i]);
      if (gen_parts(9, gen_chunks(pc.C[i])) > 1) ks = std::max(ks, px * 256);
    }
    if (ks) pv->KS = c.take<float>(ks);
    for (int i = 0; i < pc.nlev; ++i) {
      const size_t px = static_cast<size_t>(g.B) * pc.H[i] * pc.W[i];
      auto planes = [&](Planes& pl, size_t ch) {
        pl.hi = c.take<__half>(px * ch);
        pl.lo = c.take<__half>(px * ch);
      };
      planes(pv->F[i], pc.C[i]);
      if (pc.neck) {
        planes(pv->L[i], pc.C[i]);
        planes(pv->P[i], 512);
        planes(pv->O[i], pc.C[i]);
      }
      planes(pv->XP[i], 256);
      pv->X[i] = (i == 0) ? v->cond : c.take<float>(px * 256);
      if (i < pc.nlev - 1) {
        pv->UP[i] = c.take<float>(px * 256);
        if (pc.resample) pv->UPR[i] = c.take<float>(static_cast<size_t>(g.B) * 4 * pc.H[i + 1] * pc.W[i + 1] * 256);
      }
    }
  }
  if (e->rn.enabled) {
    const ResNetW& rc = e->rn;
    ResNetW* rv = &v->rn;
    const size_t pin = static_cast<size_t>(g.B) * rc.H * rc.W;
    const size_t p0 = static_cast<size_t>(g.B) * rc.Hs[0] * rc.Ws[0] * 64;  // largest stage tensor (elements)
    rv->IN.hi = c.take<__half>(pin * dd::GEN_BK);
    rv->IN.lo = c.take<__half>(pin * dd::GEN_BK);
    rv->T.hi = c.take<__half>(p0);
    rv->T.lo = c.take<__half>(p0);
    for (int k = 0; k < 2; ++k) {
      rv->Yp[k].hi = c.take<__half>(p0);
      rv->Yp[k].lo = c.take<__half>(p0);
      rv->Y32[k] = c.take<float>(p0);
    }
    rv->D32 = c.take<float>(p0);
  }
  if (e->bb.enabled) {
    const Backbone& bc = e->bb;
    Backbone* bv = &v->bb;
    const size_t m0 = (static_cast<size_t>(g.B) * bc.Hs[0] * bc.Ws[0] + 127) / 128 * 128 + 128;  // padded token count
    const size_t c0 = bc.E;
    bv->X[0] = c.take<float>(m0 * c0);
    bv->X[1] = c.take<float>(m0 * c0);
    bv->QKV = c.take<float>(m0 * c0 * 3);
    bv->AP.hi = c.take<__half>(m0 * c0);
    bv->AP.lo = c.take<__half>(m0 * c0);
    bv->HP.hi = c.take<__half>(m0 * c0 * 4);
    bv->HP.lo = c.take<__half>(m0 * c0 * 4);
  }
  if (e->mp.enabled) {
    const MPViTW& mc = e->mp;
    MPViTW* mv = &v->mp;
    const size_t pin = static_cast<size_t>(g.B) * mc.H * mc.W;
    size_t tok = 0, cat = 0, xs = pin * mc.dims[0];
    int cmax = 0;
    for (int s = 0; s < 4; ++s) {
      const size_t M = static_cast<size_t>(g.B) * mc.Hs[s] * mc.Ws[s] + 256;  // slack: the GEMM's token "image" is 16 wide
      tok = std::max(tok, M * mc.dims[s]);
      cat = std::max(cat, M * mc.dims[s] * (mc.paths[s] + 1));
      xs = std::max(xs, M * mc.out_dims[s]);
      cmax = std::max(cmax, mc.dims[s]);
    }
    auto planes = [&](Planes& pl, size_t n) {
      pl.hi = c.take<__half>(n);
      pl.lo = c.take<__half>(n);
    };
    planes(mv->IN, pin * dd::GEN_BK);
    planes(mv->S1, pin * (mc.dims[0] / 2));
    mv->XS = c.take<float>(xs);
    for (int i = 0; i < 4; ++i) mv->E[i] = c.take<float>(tok);
    mv->R1 = c.take<float>(tok);
    mv->QKV = c.take<float>(tok * 3);
    planes(mv->D, tok);
    planes(mv->EP0, tok);
    planes(mv->AP, tok);
    planes(mv->HP, tok * mc.mlp_ratio);
    planes(mv->CAT, cat);
    const size_t chm = static_cast<size_t>(cmax / mc.heads), nk = static_cast<size_t>(mc.heads) * chm * chm;
    mv->fab.part_m = c.take<float>(static_cast<size_t>(g.B) * kMpChunksMax * cmax);
    mv->fab.part_s = c.take<float>(static_cast<size_t>(g.B) * kMpChunksMax * cmax);
    mv->fab.colinv = c.take<float>(static_cast<size_t>(g.B) * cmax);
    mv->fab.part_ktv = c.take<float>(static_cast<size_t>(g.B) * kMpChunksMax * nk);
    mv->fab.ktv = c.take<float>(static_cast<size_t>(g.B) * nk);
  }
  if (has_backward(e->cfg)) {
    dd_engine::Bwd* bv = &v->bw;
    const bool swin = e->cfg.variant == DD_VARIANT_SWIN;
    const size_t PC = static_cast<size_t>(e->cfg.cond_h) * e->cfg.cond_w;
    auto planes = [&](Planes& pl, size_t ch) {
      pl.hi = c.take<__half>(BP * ch);
      pl.lo = c.take<__half>(BP * ch);
    };
    bv->y1 = c.take<float>(BP * 64);
    bv->y2 = c.take<float>(BP * 256);
    bv->y5 = c.take<float>(BP * 64);
    bv->y6 = c.take<float>(BP * 16);
    planes(bv->a1, 64);
    if (swin) {
      planes(bv->f0, 256);
      planes(bv->fa, 256);
    }
    planes(bv->fp, 256);
    planes(bv->a5, 64);
    bv->g[0] = c.take<float>(BP * 256);
    bv->g[1] = c.take<float>(BP * 256);
    planes(bv->gp, 256);
    bv->gn_part = c.take<float>(static_cast<size_t>(g.B) * bwd_chunks(g.P) * 256 * 2);
    bv->ab = c.take<float>(static_cast<size_t>(g.B) * 8);
    bv->col_part = c.take<float>(static_cast<size_t>(g.B) * bwd_chunks(std::max<int>(g.P, static_cast<int>(PC))) * 256);
    bv->dtemb = c.take<float>(static_cast<size_t>(g.B) * 256);
    if (swin) bv->dcond = c.take<float>(static_cast<size_t>(g.B) * PC * 256);
    bv->scales = c.take<float>(kBwdSlots);
    bv->amax = c.take<float>(kBwdSlots);
    size_t wg = 0;
    for (int i = 0; i < 6; ++i) wg = std::max(wg, wgrad_partial_elems(kConvCout[i], kConvCin[i], g.B, g.h, g.w));
    bv->wg_part = c.take<double>(wg);
  }
  if (e->cfg.flags & DD_FLAG_LOOP_BACKWARD) {
    dd_engine::LoopBwd* lv = &v->lp;
    const size_t np = param_offset(param_count(e->cfg)), nout = BP * 4;
    lv->stash = c.take<float>(static_cast<size_t>(e->cfg.num_inference_steps + 1) * BP * 16);
    lv->gl = c.take<float>(BP * 16);
    lv->stage = c.take<float>(np);
    lv->acc = c.take<double>(np);
    lv->acc_cond = c.take<double>(static_cast<size_t>(g.B) * e->cfg.cond_h * e->cfg.cond_w * 256);
    lv->z = c.take<float>(nout);
    lv->r = c.take<float>(nout * 16);
    lv->du = c.take<float>(nout * 16);
    lv->part_act = c.take<double>(static_cast<size_t>(dec_act_blocks(g)) * dd::DEC_ACT_N);
    lv->part_wc = c.take<double>(static_cast<size_t>(dec_wc_blocks(g)) * 144);
    lv->part_wt = c.take<double>(static_cast<size_t>(dec_wt_blocks(g)) * 4096);
  }
  return align_up(c.off, 1024);
}

// One convolution on the engine's latent grid.  in planes have `cin` channels (scale in_scale).
int run_conv(dd_engine* e, int layer, const __half* in_hi, const __half* in_lo, float in_scale, int epi, float* y32,
             double* stats_partial, __half* out_hi, __half* out_lo, cudaStream_t st) {
  const Geom g = geom_of(e->cfg);
  ConvLayer& L = e->L[layer];
  dd::ConvArgs a;
  a.B = g.B;
  a.H = g.h;
  a.W = g.w;
  a.bias = L.bias;
  a.acc_scale = 1.f / (in_scale * L.wscale);
  a.y32 = y32;
  a.stats_partial = stats_partial;
  a.out_hi = out_hi;
  a.out_lo = out_lo;
  a.split_scale = kActScale;
  a.status = e->status;
  const bool simt = (e->cfg.flags & DD_FLAG_SIMT_CONV) != 0;
  int rc;
  if ((rc = launch_conv3x3(L.sid, epi, simt, a, in_hi, in_lo, in_scale, L.w_simt, L.mh_hi, L.mh_lo, e->sm_count, st)))
    return rc;
  for (int i = 0; i < 4; ++i)  // the GroupNorm finalize sums this kernel's tiles
    if (stats_partial == e->stats[i]) e->stats_tiles_img[i] = a.tiles_x * a.tiles_y;
  return launched(e, "conv3x3");
}

int run_finalize(dd_engine* e, int which, int channels, cudaStream_t st, const double* ring = nullptr, int ring_per_img = 0) {
  const Geom g = geom_of(e->cfg);
  const double inv = 1.0 / (static_cast<double>(g.P) * (channels / 4));
  dd::gn_finalize_kernel<<<g.B * 4, 256, 0, st>>>(e->stats[which], e->stats_tiles_img[which], ring, ring_per_img, inv,
                                                   1e-5f, e->mr[which]);
  return launched(e, "gn_finalize");
}

// The GroupNorm apply kernel of a (C, COND) layer on a's B x H x W grid; up_qpb: quads per block of the bilinear
// up-add kernel (4, or 1: one 64-thread block per quad).  The caller checks the launch.
template <int C, int COND>
void launch_apply(const dd::ApplyArgs& a, int B, int up_qpb, cudaStream_t st) {
  if (COND == 2 && C == 256) {
    // one 64-thread block per 2 x 2 output quad (rows 2i-1, 2i; columns 2j-1, 2j)
    if (up_qpb == 4) {
      dim3 grid((a.W / 2 + 1 + 3) / 4, a.H / 2 + 1, B);
      dd::gn_apply_up_split_kernel<4, 4><<<grid, 256, 0, st>>>(a);
    } else {
      dim3 grid(a.W / 2 + 1, a.H / 2 + 1, B);
      dd::gn_apply_up_split_kernel<4, 1><<<grid, 64, 0, st>>>(a);
    }
  } else {
    constexpr int PPB = 256 / (C / 8);
    dim3 grid((a.H * a.W + PPB - 1) / PPB, B);
    dd::gn_apply_split_kernel<C, COND><<<grid, 256, 0, st>>>(a);
  }
}

template <int C, int COND>
int run_apply(dd_engine* e, int which, const float* temb, int temb_bstride, __half* out_hi, __half* out_lo,
              cudaStream_t st, const float* y = nullptr) {
  const Geom g = geom_of(e->cfg);
  dd::ApplyArgs a;
  a.y = y != nullptr ? y : e->Y;
  a.mean_rstd = e->mr[which];
  a.gamma = e->gn_gamma[which];
  a.beta = e->gn_beta[which];
  a.cond = e->cond;
  a.temb = temb;
  a.temb_bstride = temb_bstride;
  a.H = g.h;
  a.W = g.w;
  a.ch = e->cfg.cond_h;
  a.cw = e->cfg.cond_w;
  a.ry = g.h > 1 ? static_cast<float>(a.ch - 1) / static_cast<float>(g.h - 1) : 0.f;
  a.rx = g.w > 1 ? static_cast<float>(a.cw - 1) / static_cast<float>(g.w - 1) : 0.f;
  a.out_hi = out_hi;
  a.out_lo = out_lo;
  a.scale = kActScale;
  a.status = e->status;
  launch_apply<C, COND>(a, g.B, 4, st);
  return launched(e, "gn_apply");
}

bool fold_active(const dd_engine* e) {
  return e->cfg.variant == DD_VARIANT_SWIN && !(e->cfg.flags & (DD_FLAG_SIMT_CONV | DD_FLAG_CHAIN_PRED));
}
// Ring partials of the composed pred.0 conv: segments spread over at most as many blocks per image as stats[3] has
// tile slots (stats[3] is free until pred.3 runs).
int ring_blocks_per_img(const Geom& g) {
  return std::min(dd::ring_segments(g.h, g.w), g.tiles_max / g.B);
}

// convB -> pred.0 as the composed 5x5 conv on convA's split output (S_hi[0] / S_lo[0]) + the ring correction: Y and the
// pred.0 GroupNorm partials (tiles in stats[2], ring in stats[3]) as the two-conv chain would leave them.
int run_fold(dd_engine* e, cudaStream_t st) {
  const Geom g = geom_of(e->cfg);
  int rc;
  CUtensorMap m_hi, m_lo;
  if ((rc = make_patch_map(&m_hi, e->S_hi[0], g.B, g.h, g.w))) return rc;
  if ((rc = make_patch_map(&m_lo, e->S_lo[0], g.B, g.h, g.w))) return rc;
  dd::FoldArgs a;
  a.B = g.B;
  a.H = g.h;
  a.W = g.w;
  a.tiles_x = (g.w + dd::F5_TW - 1) / dd::F5_TW;
  a.tiles_y = (g.h + dd::F5_TH - 1) / dd::F5_TH;
  a.num_tiles = a.tiles_x * a.tiles_y * g.B;
  a.w = e->fold.w;
  a.bias = e->fold.bias;
  a.acc_scale = 1.f / (kActScale * e->fold.wscale);
  a.y32 = e->Y;
  a.stats_partial = e->stats[2];
  e->stats_tiles_img[2] = a.tiles_x * a.tiles_y;
  const int grid = std::min(a.num_tiles, e->sm_count);
  dd::conv5x5_fold_kernel<<<grid, dd::F5::THREADS, dd::F5::SMEM_BYTES, st>>>(m_hi, m_lo, a);
  if ((rc = launched(e, "conv5x5_fold"))) return rc;
  dd::RingArgs r;
  r.H = g.h;
  r.W = g.w;
  r.nseg = dd::ring_segments(g.h, g.w);
  r.blocks_per_img = ring_blocks_per_img(g);
  r.a_hi = e->S_hi[0];
  r.a_lo = e->S_lo[0];
  r.a_inv_scale = 1.f / kActScale;
  r.edge = e->fold.edge;
  r.y32 = e->Y;
  r.ring_partial = e->stats[3];
  dd::ring_fix_kernel<<<dim3(r.blocks_per_img, g.B), dd::RING_THREADS, dd::RING_SMEM, st>>>(r);
  return launched(e, "ring_fix");
}

int run_tail(dd_engine* e, float cx, float ce, float* eps_out, cudaStream_t st);

// pred.4's GroupNorm + ReLU fused with the DDIM update over B images of f.P pixels; the caller checks the launch.
void launch_final(const dd::FinalArgs& f, int B, cudaStream_t st) {
  dim3 grid((f.P * 4 + 255) / 256, B);
  dd::gn_relu_ddim_kernel<<<grid, 256, 0, st>>>(f);
}

// One ScheduledCNNRefine.forward + (optionally) the DDIM update.
int run_step(dd_engine* e, const float* temb, int temb_bstride, float cx, float ce, float* eps_out, cudaStream_t st) {
  const Geom g = geom_of(e->cfg);
  int rc;
  // noise_embedding.0 : x (16) -> 64, GN stats
  if ((rc = run_conv(e, 0, e->xs_hi, e->xs_lo, kXScale, dd::EPI_F32_STATS, e->Y, e->stats[0], nullptr, nullptr, st))) return rc;
  if ((rc = run_finalize(e, 0, 64, st))) return rc;
  if ((rc = run_apply<64, 0>(e, 0, nullptr, 0, e->S_hi[0], e->S_lo[0], st))) return rc;
  // noise_embedding.3 : 64 -> 256, GN stats
  if ((rc = run_conv(e, 1, e->S_hi[0], e->S_lo[0], kActScale, dd::EPI_F32_STATS, e->Y, e->stats[1], nullptr, nullptr, st)))
    return rc;
  if ((rc = run_finalize(e, 1, 256, st))) return rc;
  const __half *p_hi, *p_lo;
  if (e->cfg.variant == DD_VARIANT_SWIN) {
    // feat = up(cond + temb) + relu(gn(y2));  convA ; convB   (UpSample_add)
    if ((rc = run_apply<256, 2>(e, 1, temb, temb_bstride, e->S_hi[1], e->S_lo[1], st))) return rc;
    if ((rc = run_conv(e, 2, e->S_hi[1], e->S_lo[1], kActScale, dd::EPI_SPLIT, nullptr, nullptr, e->S_hi[0], e->S_lo[0], st)))
      return rc;
    if (fold_active(e)) {  // convB + pred.0 as one composed conv + its ring correction
      if ((rc = run_fold(e, st))) return rc;
      if ((rc = run_finalize(e, 2, 64, st, e->stats[3], ring_blocks_per_img(g)))) return rc;
      return run_tail(e, cx, ce, eps_out, st);
    }
    if ((rc = run_conv(e, 3, e->S_hi[0], e->S_lo[0], kActScale, dd::EPI_SPLIT, nullptr, nullptr, e->S_hi[1], e->S_lo[1], st)))
      return rc;
    p_hi = e->S_hi[1];
    p_lo = e->S_lo[1];
  } else {
    if ((rc = run_apply<256, 1>(e, 1, temb, temb_bstride, e->S_hi[1], e->S_lo[1], st))) return rc;
    p_hi = e->S_hi[1];
    p_lo = e->S_lo[1];
  }
  // pred.0 : 256 -> 64, GN stats
  if ((rc = run_conv(e, 4, p_hi, p_lo, kActScale, dd::EPI_F32_STATS, e->Y, e->stats[2], nullptr, nullptr, st))) return rc;
  if ((rc = run_finalize(e, 2, 64, st))) return rc;
  return run_tail(e, cx, ce, eps_out, st);
}

// pred.0's GroupNorm + ReLU, pred.3 and its GroupNorm + ReLU, and the DDIM update (Y holds pred.0's output).
int run_tail(dd_engine* e, float cx, float ce, float* eps_out, cudaStream_t st) {
  const Geom g = geom_of(e->cfg);
  int rc;
  if ((rc = run_apply<64, 0>(e, 2, nullptr, 0, e->S_hi[0], e->S_lo[0], st))) return rc;
  // pred.3 : 64 -> 16, GN stats
  if ((rc = run_conv(e, 5, e->S_hi[0], e->S_lo[0], kActScale, dd::EPI_F32_STATS, e->Y, e->stats[3], nullptr, nullptr, st))) return rc;
  if ((rc = run_finalize(e, 3, 16, st))) return rc;
  dd::FinalArgs f;
  f.y = e->Y;
  f.mean_rstd = e->mr[3];
  f.gamma = e->gn_gamma[3];
  f.beta = e->gn_beta[3];
  f.x = e->x32;
  f.x_hi = e->xs_hi;
  f.x_lo = e->xs_lo;
  f.eps_out = eps_out;
  f.cx = cx;
  f.ce = ce;
  f.scale = kXScale;
  f.P = g.P;
  f.status = e->status;
  launch_final(f, g.B, st);
  return launched(e, "gn_relu_ddim");
}

// The layout changes and the latent split leave counting their launch to their callers.
int transpose_in(const float* nchw, float* nhwc, int B, int C, int P, cudaStream_t st) {
  dim3 grid((P + 31) / 32, (C + 31) / 32, B), block(32, 8);
  dd::nchw_to_nhwc_kernel<<<grid, block, 0, st>>>(nchw, nhwc, C, P);
  return check_launch("nchw_to_nhwc");
}
int transpose_out(const float* nhwc, float* nchw, int B, int C, int P, cudaStream_t st) {
  dim3 grid((P + 31) / 32, (C + 31) / 32, B), block(32, 8);
  dd::nhwc_to_nchw_kernel<<<grid, block, 0, st>>>(nhwc, nchw, C, P);
  return check_launch("nhwc_to_nchw");
}
int split_planes(dd_engine* e, const float* x, __half* hi, __half* lo, size_t n, float scale, cudaStream_t st) {
  dd::split_planes_kernel<<<grid_of(n / 4), 256, 0, st>>>(x, hi, lo, n / 4, scale, e->status);
  return check_launch("split_planes");
}

// A codec BatchNorm in training mode over n items of op's pre-BN value (run_bn_passes): bn_stats_kernel's two passes,
// then the fold of (gamma, beta) = gb[0..15], gb[16..31] into w_out / b_out (see dd::BnFoldArgs for the other pointers).
template <class Op>
int run_codec_bn(dd_engine* e, const Op& op, long long n, const float* gb, const float* bias, const float* w, int nw,
                 float* w_out, float* b_out, float* bn_out, float* rec, cudaStream_t st) {
  dd_engine::CodecTrain& ct = e->ct;
  const int nblk = codec_stats_blocks(n);
  auto stats = [&](const double* sum1, const double* cnt) {
    dd::bn_stats_kernel<Op><<<nblk, 256, 0, st>>>(op, n, sum1, cnt, ct.part);
    return launched(e, "bn_stats");
  };
  auto fold = [&](const dd::BnFoldIn& in) {
    dd::BnFoldArgs f;
    f.in = in;
    f.gamma = gb;
    f.beta = gb + 16;
    f.bias = bias;
    f.w = w;
    f.nw = nw;
    f.w_out = w_out;
    f.b_out = b_out;
    f.bn_out = bn_out;
    f.rec = rec;
    dd::bn_fold_kernel<<<1, 256, 0, st>>>(f);
    return launched(e, "bn_fold");
  };
  return run_bn_passes(e, ct.part, nblk, 16, n, ct.sum1, st, stats, fold);
}

// DD_CODEC_TRAIN: the decoder BatchNorm's statistics over the latent in x32, folded into ct.dec_wt / dec_bt / dec_bn
// (which run_decoder then reads); rec: where the record goes (null: none).
int run_dec_batch_stats(dd_engine* e, float* rec, cudaStream_t st) {
  const Geom g = geom_of(e->cfg);
  const dd::DecPreBn op{e->x32, e->dec_wu, g.h, g.w};
  dd_engine::CodecTrain& ct = e->ct;
  return run_codec_bn(e, op, static_cast<long long>(g.B) * g.P * 4, ct.dec_gb, e->dec_bu, e->dec_wu, 4096, ct.dec_wt,
                      ct.dec_bt, ct.dec_bn, rec, st);
}

// decoder_kernel on the running-statistics fold, or in DD_CODEC_TRAIN on the batch fold of the last run_dec_batch_stats
int run_decoder(dd_engine* e, float* logit, float* depth, cudaStream_t st) {
  const Geom g = geom_of(e->cfg);
  const bool train = e->codec_mode == DD_CODEC_TRAIN;
  dd::DecoderArgs a;
  a.x = e->x32;
  a.wt = train ? e->ct.dec_wt : e->dec_wt;
  a.bt = train ? e->ct.dec_bt : e->dec_bt;
  a.wc = e->dec_wc;
  a.bc = e->dec_bc;
  a.logit = logit;
  a.depth = depth;
  a.h = g.h;
  a.w = g.w;
  a.eps = 1e-6f;
  dim3 grid((2 * g.w + dd::DEC_TW - 1) / dd::DEC_TW, (2 * g.h + dd::DEC_TH - 1) / dd::DEC_TH, g.B);
  dd::decoder_kernel<<<grid, 256, dd::DEC_SMEM, st>>>(a);
  return launched(e, "decoder");
}

int bind_workspace(dd_engine* e, void* ws, size_t bytes) {
  const size_t need = carve(e, nullptr);
  if (ws == nullptr || bytes < need) return fail(DD_ERR_INVALID, "workspace too small: need " + std::to_string(need));
  if ((reinterpret_cast<uintptr_t>(ws) & 1023) != 0) return fail(DD_ERR_INVALID, "workspace must be 1024-byte aligned");
  if (ws != e->ws) {
    carve(e, ws);
    e->ws = ws;
    drop_graphs(e);
  }
  return DD_OK;
}

// The first step of every entry that runs on the engine's workspace: its device, then the workspace bound.
int enter_workspace(dd_engine* h, void* ws, size_t bytes) {
  CUDA_TRY(cudaSetDevice(h->cfg.device));
  return bind_workspace(h, ws, bytes);
}

// A forward starts: the status word its kernels flag range faults in and the launch count start from zero.
int start_forward(dd_engine* h, cudaStream_t st) {
  h->launches = 0;
  CUDA_TRY(cudaMemsetAsync(h->status, 0, 64, st));
  return DD_OK;
}

// Synchronise st and report a flagged range fault in the engine's status word.
int poll_status(dd_engine* h, cudaStream_t st) {
  CUDA_TRY(cudaMemcpyAsync(h->status_host, h->status, 4, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  if (*h->status_host & 1)
    return fail(DD_ERR_RANGE, "an activation exceeded the operand split's range (16 |v| > 6e4)");
  return DD_OK;
}

// A forward ends: with DD_FLAG_CHECK_RANGE it waits for st and reports a range fault.
int finish_forward(dd_engine* h, cudaStream_t st) {
  return (h->cfg.flags & DD_FLAG_CHECK_RANGE) ? poll_status(h, st) : DD_OK;
}

// After dd_enable_producers / dd_enable_backbone: the pack and the workspace layout no longer fit the engine, so the
// weights must be finalized again, the next entry re-carves its workspace, and every graph is captured again.
void invalidate_pack(dd_engine* h) {
  h->weights_ready = h->packed = false;
  h->ws = nullptr;
  drop_graphs(h);
}

// Copy a standalone call's status word back, synchronise st and report a flag as DD_ERR_RANGE in `what`.
int check_status_word(const int* status, cudaStream_t st, const char* what) {
  int flag = 0;
  CUDA_TRY(cudaMemcpyAsync(&flag, status, 4, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  if (flag) return fail(DD_ERR_RANGE, std::string("non-finite or out-of-range value in ") + what);
  return DD_OK;
}

const Raw* find(dd_engine* e, const std::string& k) {
  auto it = e->raw.find(k);
  return it == e->raw.end() ? nullptr : &it->second;
}

// cudaMalloc recorded in `owned`, which the owner frees (the engine's list: at dd_destroy)
int dev_alloc(std::vector<void*>& owned, void** p, size_t bytes) {
  cudaError_t err = cudaMalloc(p, bytes);
  if (err != cudaSuccess) return fail(DD_ERR_CUDA, std::string("cudaMalloc: ") + cudaGetErrorString(err));
  owned.push_back(*p);
  return DD_OK;
}
int dev_alloc(dd_engine* e, void** p, size_t bytes) { return dev_alloc(e->owned, p, bytes); }

template <typename T>
int dev_array(dd_engine* e, T** p, size_t elems) {
  return dev_alloc(e->owned, reinterpret_cast<void**>(p), elems * sizeof(T));
}

// The buffers and TMA descriptors of one conv layer; fill_pack writes the contents.
int alloc_layer(dd_engine* e, ConvLayer& L, int cout, int cin) {
  L.sid = shape_id(cin, cout);
  if (L.sid < 0) return fail(DD_ERR_UNSUPPORTED, "unsupported conv shape");
  const size_t n = static_cast<size_t>(cout) * cin * 9;
  int rc;
  if ((rc = dev_array(e, &L.w_hi, n))) return rc;
  if ((rc = dev_array(e, &L.w_lo, n))) return rc;
  if ((rc = dev_array(e, &L.w_simt, n))) return rc;
  if ((rc = dev_array(e, &L.bias, cout))) return rc;
  if ((rc = make_weight_map(&L.mh_hi, L.w_hi, cout, cin, 9, kHaloBK[L.sid], cout))) return rc;
  return make_weight_map(&L.mh_lo, L.w_lo, cout, cin, 9, kHaloBK[L.sid], cout);
}

// ------------------------------------------------------------------------------------------------ producers
constexpr float kProdScale = 16.f;  // fp16-split pre-scale of every producer activation

// Eval-BN (weight, bias, running_mean, running_var) = bn[0..3], host vectors of ch, as per-channel (scale, shift).
void bn_fold_host(const float* const* bn, int ch, float* scale, float* shift) {
  for (int c = 0; c < ch; ++c) {
    const double sc = static_cast<double>(bn[0][c]) / sqrt(static_cast<double>(bn[3][c]) + 1e-5);
    scale[c] = static_cast<float>(sc);
    shift[c] = static_cast<float>(static_cast<double>(bn[1][c]) - static_cast<double>(bn[2][c]) * sc);
  }
}
// Fold eval-BN, given as the device vectors bn[0..3] = (weight, bias, running_mean, running_var), into per-channel
// (scale, shift) on the host.
int bn_fold(const float* const* bn, int ch, std::vector<float>& scale, std::vector<float>& shift, cudaStream_t st) {
  std::vector<float> v[4];
  for (int i = 0; i < 4; ++i) {
    v[i].resize(ch);
    CUDA_TRY(cudaMemcpyAsync(v[i].data(), bn[i], ch * 4, cudaMemcpyDeviceToHost, st));
  }
  CUDA_TRY(cudaStreamSynchronize(st));
  scale.resize(ch);
  shift.resize(ch);
  const float* host[4] = {v[0].data(), v[1].data(), v[2].data(), v[3].data()};
  bn_fold_host(host, ch, scale.data(), shift.data());
  return DD_OK;
}
// the registered eval-BN vectors prefix.{weight,bias,running_mean,running_var} -> bn[0..3]
int find_bn(dd_engine* e, const std::string& prefix, const float** bn) {
  const char* parts[4] = {".weight", ".bias", ".running_mean", ".running_var"};
  for (int i = 0; i < 4; ++i) {
    const Raw* r = find(e, prefix + parts[i]);
    if (!r) return fail(DD_ERR_INVALID, "missing weights: " + prefix + parts[i]);
    bn[i] = r->ptr;
  }
  return DD_OK;
}
int copy_param(dd_engine* e, const std::string& key, size_t n, float** out, cudaStream_t st) {
  const Raw* r = find(e, key);
  if (!r) return fail(DD_ERR_INVALID, "missing weights: " + key);
  size_t have = 1;
  for (int64_t d : r->shape) have *= static_cast<size_t>(d);
  if (have != n) return fail(DD_ERR_INVALID, "weight shape mismatch: " + key);
  int rc;
  if ((rc = dev_alloc(e, reinterpret_cast<void**>(out), n * 4))) return rc;
  CUDA_TRY(cudaMemcpyAsync(*out, r->ptr, n * 4, cudaMemcpyDeviceToDevice, st));
  return DD_OK;
}

// ------------------------------------------------------------------------------------------------ denoiser + codec pack
// dd_finalize_weights allocates (alloc_pack) and fills (fill_pack) everything; dd_update_weights validates
// (check_update) and fills what depends on the registered keys, at the same addresses.
const char* const kGnKey[4] = {"model.noise_embedding.1", "model.noise_embedding.4", "model.pred.1", "model.pred.4"};
constexpr int kGnCh[4] = {64, 256, 64, 16};
const std::string kDecPrefix = "depth_transform.conv_inv_transform.";
const std::string kEncPrefix = "depth_transform.conv_transform.";
struct CodecKey {
  const char* leaf;
  size_t host_off;  // floats from the start of PackStage
  std::vector<int64_t> shape;
};
#define DD_STAGE_OFF(m) (offsetof(PackStage, m) / sizeof(float))
const CodecKey kDecKeys[8] = {{"0.weight", DD_STAGE_OFF(dec_wt), {16, 16, 4, 4}}, {"0.bias", DD_STAGE_OFF(dec_bt), {16}},
                              {"1.weight", DD_STAGE_OFF(dec_g), {16}},            {"1.bias", DD_STAGE_OFF(dec_be), {16}},
                              {"1.running_mean", DD_STAGE_OFF(dec_mu), {16}},     {"1.running_var", DD_STAGE_OFF(dec_var), {16}},
                              {"3.0.weight", DD_STAGE_OFF(dec_wc), {1, 16, 3, 3}}, {"3.0.bias", DD_STAGE_OFF(dec_bc), {1}}};
const CodecKey kEncKeys[10] = {
    {"0.0.weight", DD_STAGE_OFF(enc_w1), {16, 1, 3, 3}},        {"0.1.weight", DD_STAGE_OFF(enc_bn1[0]), {16}},
    {"0.1.bias", DD_STAGE_OFF(enc_bn1[1]), {16}},               {"0.1.running_mean", DD_STAGE_OFF(enc_bn1[2]), {16}},
    {"0.1.running_var", DD_STAGE_OFF(enc_bn1[3]), {16}},        {"1.0.weight", DD_STAGE_OFF(enc_w2), {16, 16, 3, 3}},
    {"1.1.weight", DD_STAGE_OFF(enc_bn2[0]), {16}},             {"1.1.bias", DD_STAGE_OFF(enc_bn2[1]), {16}},
    {"1.1.running_mean", DD_STAGE_OFF(enc_bn2[2]), {16}},       {"1.1.running_var", DD_STAGE_OFF(enc_bn2[3]), {16}}};
#undef DD_STAGE_OFF
size_t numel(const std::vector<int64_t>& s) {
  size_t n = 1;
  for (int64_t d : s) n *= static_cast<size_t>(d);
  return n;
}

int alloc_pack(dd_engine* h, bool encoder, cudaStream_t st) {
  const bool swin = h->cfg.variant == DD_VARIANT_SWIN;
  int rc;
  if ((rc = dev_array(h, &h->amax, 16))) return rc;
  for (int i = 0; i < 6; ++i) {
    if (!swin && (i == 2 || i == 3)) continue;
    const int co = kConvCout[i], ci = kConvCin[i];
    if ((rc = alloc_layer(h, h->L[i], co, ci))) return rc;
    if (has_backward(h->cfg)) {
      // data-gradient convs: W'[ci][co][ky][kx] = W[co][ci][2-ky][2-kx] with zero bias, packed like any forward layer
      if ((rc = dev_array(h, &h->w_flip[i], static_cast<size_t>(co) * ci * 9))) return rc;
      if ((rc = alloc_layer(h, h->L[6 + i], ci, co))) return rc;
      CUDA_TRY(cudaMemsetAsync(h->L[6 + i].bias, 0, ci * 4, st));
    }
  }
  if (fold_active(h)) {
    const size_t n5 = 64 * 256 * 25;
    if ((rc = dev_array(h, &h->fold.w, dd::F5::W_ELEMS))) return rc;
    if ((rc = dev_array(h, &h->fold.bias, 64))) return rc;
    if ((rc = dev_array(h, &h->fold.src[0], 256 * 256 * 9))) return rc;
    if ((rc = dev_array(h, &h->fold.src[1], 64 * 256 * 9))) return rc;
    if ((rc = dev_array(h, &h->fold.k5, n5))) return rc;
    if ((rc = dev_array(h, &h->fold.k5_abs, n5))) return rc;
    if ((rc = dev_array(h, &h->fold.edge, dd::EDGE_ELEMS))) return rc;
  }
  for (int i = 0; i < 4; ++i) {
    if ((rc = dev_array(h, &h->gn_gamma[i], kGnCh[i]))) return rc;
    if ((rc = dev_array(h, &h->gn_beta[i], kGnCh[i]))) return rc;
  }
  if ((rc = dev_array(h, &h->temb, DD_TIME_ROWS * 256))) return rc;
  if ((rc = dev_array(h, &h->dec_wt, 4 * 4 * 16 * 16))) return rc;
  if ((rc = dev_array(h, &h->dec_bt, 16))) return rc;
  if ((rc = dev_array(h, &h->dec_wc, 9 * 16))) return rc;
  // the decoder backward and DD_CODEC_TRAIN need the BatchNorm unfolded
  if ((rc = dev_array(h, &h->dec_wu, 4 * 4 * 16 * 16))) return rc;
  if ((rc = dev_array(h, &h->dec_bu, 16))) return rc;
  if ((rc = dev_array(h, &h->dec_bn, 3 * 16))) return rc;
  dd_engine::CodecTrain& ct = h->ct;
  if ((rc = dev_array(h, &ct.dec_gb, 2 * 16))) return rc;
  if ((rc = dev_array(h, &ct.dec_wt, 4 * 4 * 16 * 16))) return rc;
  if ((rc = dev_array(h, &ct.dec_bt, 16))) return rc;
  if ((rc = dev_array(h, &ct.dec_bn, 3 * 16))) return rc;
  if ((rc = dev_array(h, &ct.zero16, 16))) return rc;
  CUDA_TRY(cudaMemsetAsync(ct.zero16, 0, 16 * 4, st));
  const Geom g = geom_of(h->cfg);
  if ((rc = dev_array(h, &ct.part, static_cast<size_t>(codec_stats_blocks(static_cast<long long>(g.B) * g.P * 4)) *
                                         dd::BNS_COLS)))
    return rc;
  if ((rc = dev_array(h, &ct.sum1, 16))) return rc;
  if ((rc = dev_array(h, &ct.sums, 32))) return rc;
  if ((rc = dev_array(h, &ct.part_db, static_cast<size_t>(dec_act_blocks(g)) * 16))) return rc;
  if ((rc = dev_array(h, &ct.rec, static_cast<size_t>(std::max(h->cfg.num_inference_steps, 2)) * 32))) return rc;
  ct.nrec = 0;
  h->enc_w1 = nullptr;
  if (encoder) {
    if ((rc = dev_array(h, &h->enc_w1, 144))) return rc;
    if ((rc = dev_array(h, &h->enc_b1, 16))) return rc;
    if ((rc = dev_array(h, &h->enc_w2, 2304))) return rc;
    if ((rc = dev_array(h, &h->enc_b2, 16))) return rc;
    if ((rc = dev_array(h, &h->enc_bn, 2 * 3 * 16))) return rc;
    if ((rc = dev_array(h, &ct.enc_bn, 2 * 3 * 16))) return rc;
    if ((rc = dev_array(h, &ct.enc_w1, 144))) return rc;
    if ((rc = dev_array(h, &ct.enc_w2, 2304))) return rc;
    if ((rc = dev_array(h, &ct.enc_gb, 4 * 16))) return rc;
    if ((rc = dev_array(h, &ct.enc_w1f, 144))) return rc;
    if ((rc = dev_array(h, &ct.enc_b1f, 16))) return rc;
    if ((rc = dev_array(h, &ct.enc_w2f, 2304))) return rc;
    if ((rc = dev_array(h, &ct.enc_b2f, 16))) return rc;
  }
  return DD_OK;
}

// Every key registered for dd_update_weights belongs to the denoiser / codec pack and has the packed shape.
int check_update(dd_engine* h) {
  const bool swin = h->cfg.variant == DD_VARIANT_SWIN;
  std::map<std::string, std::vector<int64_t>> want;
  for (int i = 0; i < 6; ++i) {
    if (!swin && (i == 2 || i == 3)) continue;
    want[std::string(kConvKey[i]) + ".weight"] = {kConvCout[i], kConvCin[i], 3, 3};
    want[std::string(kConvKey[i]) + ".bias"] = {kConvCout[i]};
  }
  for (int i = 0; i < 4; ++i) want[std::string(kGnKey[i]) + ".weight"] = want[std::string(kGnKey[i]) + ".bias"] = {kGnCh[i]};
  want["model.time_embedding.weight"] = {DD_TIME_ROWS, 256};
  for (const CodecKey& k : kDecKeys) want[kDecPrefix + k.leaf] = k.shape;
  if (h->enc_w1)
    for (const CodecKey& k : kEncKeys) want[kEncPrefix + k.leaf] = k.shape;
  for (const auto& kv : h->raw) {
    const std::string& name = kv.first;
    for (const char* p : {"hahineck.", "conv_lateral.", "conv_up.", "backbone."})
      if (name.compare(0, strlen(p), p) == 0)
        return fail(DD_ERR_UNSUPPORTED, name + ": the neck, FPN and backbone are re-packed by dd_finalize_weights only");
    auto it = want.find(name);
    if (it == want.end()) return fail(DD_ERR_INVALID, name + " is not part of this engine's pack");
    if (kv.second.shape != it->second) return fail(DD_ERR_INVALID, name + ": shape differs from the packed tensor");
  }
  return DD_OK;
}

// The loop graphs hold acc_scale = 1 / (in_scale * wscale) of the convs run_step launches, by value.
bool loop_reads_wscale(const dd_engine* e, int layer) { return !(fold_active(e) && (layer == 3 || layer == 4)); }

// Write every packed object that depends on a key in h->raw (dd_finalize_weights: all of them).  Enqueued on st with one
// synchronisation in the middle, where the abs-max words and the registered codec tensors reach the host; the conv
// weights are read again after it, so the registered tensors must stay valid until the work enqueued here has run.
int fill_pack(dd_engine* h, cudaStream_t st) {
  const bool swin = h->cfg.variant == DD_VARIANT_SWIN;
  PackStage* sg = h->stage;
  float* sg_f = reinterpret_cast<float*>(sg);
  auto W = [&](const std::string& k) -> const float* {
    const Raw* r = find(h, k);
    return r ? r->ptr : nullptr;
  };
  int rc;
  CUDA_TRY(cudaStreamWaitEvent(st, h->pack_done, 0));
  CUDA_TRY(cudaMemsetAsync(h->amax, 0, 16 * 4, st));
  const float* w[6] = {};
  bool fold = false;
  for (int i = 0; i < 6; ++i) {
    if (!swin && (i == 2 || i == 3)) continue;
    const int co = kConvCout[i], ci = kConvCin[i];
    const int n = co * ci * 9;
    w[i] = W(std::string(kConvKey[i]) + ".weight");
    const float* b = W(std::string(kConvKey[i]) + ".bias");
    if (b) CUDA_TRY(cudaMemcpyAsync(h->L[i].bias, b, co * 4, cudaMemcpyDeviceToDevice, st));
    if (w[i]) {
      dd::absmax_kernel<<<absmax_grid(n), 256, 0, st>>>(w[i], n, h->amax + i);
      if ((rc = check_launch("absmax"))) return rc;
      if (has_backward(h->cfg)) {
        dd::flip_transpose_weight_kernel<<<64, 256, 0, st>>>(w[i], h->w_flip[i], co, ci);
        if ((rc = check_launch("flip_transpose_weight"))) return rc;
        dd::absmax_kernel<<<absmax_grid(n), 256, 0, st>>>(h->w_flip[i], n, h->amax + 6 + i);
        if ((rc = check_launch("absmax"))) return rc;
      }
    }
    if (fold_active(h) && (i == 3 || i == 4)) {
      if (w[i]) CUDA_TRY(cudaMemcpyAsync(h->fold.src[i - 3], w[i], static_cast<size_t>(n) * 4, cudaMemcpyDeviceToDevice, st));
      fold |= w[i] || b;
    }
  }
  if (fold) {  // K5 / b5 in fp64, then one fp16 hi / lo split with a power-of-two scale as for the 3x3 layers
    dd::compose_fold_kernel<<<256, 256, 0, st>>>(h->fold.src[1], h->L[4].bias, h->fold.src[0], h->L[3].bias, h->fold.k5,
                                                 h->fold.k5_abs, h->fold.bias);
    if ((rc = check_launch("compose_fold"))) return rc;
    dd::compose_edge_kernel<<<256, 256, 0, st>>>(h->fold.src[1], h->fold.src[0], h->L[3].bias, h->fold.edge);
    if ((rc = check_launch("compose_edge"))) return rc;
    dd::absmax_kernel<<<absmax_grid(64 * 256 * 25), 256, 0, st>>>(h->fold.k5_abs, 64 * 256 * 25, h->amax + 12);
    if ((rc = check_launch("absmax"))) return rc;
  }
  for (int i = 0; i < 4; ++i) {
    if (const float* g = W(std::string(kGnKey[i]) + ".weight"))
      CUDA_TRY(cudaMemcpyAsync(h->gn_gamma[i], g, kGnCh[i] * 4, cudaMemcpyDeviceToDevice, st));
    if (const float* b = W(std::string(kGnKey[i]) + ".bias"))
      CUDA_TRY(cudaMemcpyAsync(h->gn_beta[i], b, kGnCh[i] * 4, cudaMemcpyDeviceToDevice, st));
  }
  if (const float* t = W("model.time_embedding.weight"))
    CUDA_TRY(cudaMemcpyAsync(h->temb, t, DD_TIME_ROWS * 256 * 4, cudaMemcpyDeviceToDevice, st));
  bool dec = false, enc = false;
  for (const CodecKey& k : kDecKeys)
    if (const float* p = W(kDecPrefix + k.leaf)) {
      CUDA_TRY(cudaMemcpyAsync(sg_f + k.host_off, p, numel(k.shape) * 4, cudaMemcpyDeviceToHost, st));
      dec = true;
    }
  if (h->enc_w1)
    for (const CodecKey& k : kEncKeys)
      if (const float* p = W(kEncPrefix + k.leaf)) {
        CUDA_TRY(cudaMemcpyAsync(sg_f + k.host_off, p, numel(k.shape) * 4, cudaMemcpyDeviceToHost, st));
        enc = true;
      }
  CUDA_TRY(cudaMemcpyAsync(sg->amax, h->amax, 16 * 4, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));

  // A graph stays valid across a re-pack (the buffers keep their addresses) unless a kernel argument it holds by value
  // changed: a conv's or the fold's scale in both loop graphs, the decoder's final bias in the step-decode one.
  bool loop_stale = false, steps_stale = false;
  for (int i = 0; i < 6; ++i) {
    if (!w[i]) continue;
    const int co = kConvCout[i], ci = kConvCin[i];
    ConvLayer& L = h->L[i];
    const float s = dd::grad_scale_of(sg->amax[i]);
    loop_stale |= s != L.wscale && loop_reads_wscale(h, i);
    L.wscale = s;
    dd::pack_conv_weight_kernel<<<128, 256, 0, st>>>(w[i], L.w_hi, L.w_lo, L.w_simt, co, ci, L.wscale);
    if ((rc = check_launch("pack_conv_weight"))) return rc;
    if (has_backward(h->cfg)) {
      ConvLayer& D = h->L[6 + i];
      D.wscale = dd::grad_scale_of(sg->amax[6 + i]);
      dd::pack_conv_weight_kernel<<<128, 256, 0, st>>>(h->w_flip[i], D.w_hi, D.w_lo, D.w_simt, ci, co, D.wscale);
      if ((rc = check_launch("pack_conv_weight"))) return rc;
    }
  }
  if (fold) {
    const float s = dd::grad_scale_of(sg->amax[12]);
    loop_stale |= s != h->fold.wscale;
    h->fold.wscale = s;
    dd::pack_fold_kernel<<<256, 256, 0, st>>>(h->fold.k5, h->fold.w, static_cast<double>(h->fold.wscale));
    if ((rc = check_launch("pack_fold"))) return rc;
  }
  if (dec) {  // fold eval-BN into the transposed conv (tiny: on the host in fp64)
    for (int co = 0; co < 16; ++co) {
      const double sc = static_cast<double>(sg->dec_g[co]) / sqrt(static_cast<double>(sg->dec_var[co]) + 1e-5);
      sg->bt_f[co] = static_cast<float>((static_cast<double>(sg->dec_bt[co]) - sg->dec_mu[co]) * sc + sg->dec_be[co]);
      for (int ci = 0; ci < 16; ++ci)
        for (int ky = 0; ky < 4; ++ky)
          for (int kx = 0; kx < 4; ++kx)  // ConvTranspose2d weight layout: [Cin][Cout][kh][kw]
            sg->wt_f[((ky * 4 + kx) * 16 + ci) * 16 + co] =
                static_cast<float>(static_cast<double>(sg->dec_wt[((ci * 16 + co) * 4 + ky) * 4 + kx]) * sc);
    }
    for (int ci = 0; ci < 16; ++ci)
      for (int tap = 0; tap < 9; ++tap) sg->wc_f[tap * 16 + ci] = sg->dec_wc[ci * 9 + tap];
    CUDA_TRY(cudaMemcpyAsync(h->dec_wt, sg->wt_f, sizeof(sg->wt_f), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(h->dec_bt, sg->bt_f, sizeof(sg->bt_f), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(h->dec_wc, sg->wc_f, sizeof(sg->wc_f), cudaMemcpyHostToDevice, st));
    steps_stale |= sg->dec_bc[0] != h->dec_bc;
    h->dec_bc = sg->dec_bc[0];
    for (int co = 0; co < 16; ++co) {  // unfolded: the decoder backward and DD_CODEC_TRAIN
      const double rstd = 1.0 / sqrt(static_cast<double>(sg->dec_var[co]) + 1e-5);
      sg->bn[co] = static_cast<float>(static_cast<double>(sg->dec_g[co]) * rstd);
      sg->bn[16 + co] = sg->dec_mu[co];
      sg->bn[32 + co] = static_cast<float>(rstd);
      for (int ci = 0; ci < 16; ++ci)
        for (int k = 0; k < 16; ++k) sg->wu[(k * 16 + ci) * 16 + co] = sg->dec_wt[(ci * 16 + co) * 16 + k];
    }
    CUDA_TRY(cudaMemcpyAsync(h->dec_wu, sg->wu, sizeof(sg->wu), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(h->dec_bu, sg->dec_bt, sizeof(sg->dec_bt), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(h->dec_bn, sg->bn, sizeof(sg->bn), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(h->ct.dec_gb, sg->dec_g, 16 * 4, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(h->ct.dec_gb + 16, sg->dec_be, 16 * 4, cudaMemcpyHostToDevice, st));
  }
  if (enc) {
    float s1[16], s2[16];
    const float* bn1[4] = {sg->enc_bn1[0], sg->enc_bn1[1], sg->enc_bn1[2], sg->enc_bn1[3]};
    const float* bn2[4] = {sg->enc_bn2[0], sg->enc_bn2[1], sg->enc_bn2[2], sg->enc_bn2[3]};
    bn_fold_host(bn1, 16, s1, sg->t1);
    bn_fold_host(bn2, 16, s2, sg->t2);
    for (int co = 0; co < 16; ++co)
      for (int tap = 0; tap < 9; ++tap)
        sg->f1[tap * 16 + co] = static_cast<float>(static_cast<double>(sg->enc_w1[co * 9 + tap]) * s1[co]);
    for (int co = 0; co < 16; ++co)
      for (int ci = 0; ci < 16; ++ci)
        for (int tap = 0; tap < 9; ++tap)
          sg->f2[(tap * 16 + ci) * 16 + co] =
              static_cast<float>(static_cast<double>(sg->enc_w2[(co * 16 + ci) * 9 + tap]) * s2[co]);
    CUDA_TRY(cudaMemcpyAsync(h->enc_w1, sg->f1, sizeof(sg->f1), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(h->enc_b1, sg->t1, sizeof(sg->t1), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(h->enc_w2, sg->f2, sizeof(sg->f2), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(h->enc_b2, sg->t2, sizeof(sg->t2), cudaMemcpyHostToDevice, st));
    for (int co = 0; co < 16; ++co) {  // unfolded, for DD_CODEC_TRAIN
      for (int tap = 0; tap < 9; ++tap) {
        sg->e1u[tap * 16 + co] = sg->enc_w1[co * 9 + tap];
        for (int ci = 0; ci < 16; ++ci) sg->e2u[(tap * 16 + ci) * 16 + co] = sg->enc_w2[(co * 16 + ci) * 9 + tap];
      }
      sg->enc_gb[0][co] = sg->enc_bn1[0][co];
      sg->enc_gb[1][co] = sg->enc_bn1[1][co];
      sg->enc_gb[2][co] = sg->enc_bn2[0][co];
      sg->enc_gb[3][co] = sg->enc_bn2[1][co];
      for (int k = 0; k < 2; ++k) {  // the backward's eval BatchNorms, as dec_bn
        const float(*bn)[16] = k == 0 ? sg->enc_bn1 : sg->enc_bn2;  // weight, bias, running_mean, running_var
        const double rstd = 1.0 / sqrt(static_cast<double>(bn[3][co]) + 1e-5);
        sg->enc_bn[k][0][co] = static_cast<float>(static_cast<double>(bn[0][co]) * rstd);
        sg->enc_bn[k][1][co] = bn[2][co];
        sg->enc_bn[k][2][co] = static_cast<float>(rstd);
      }
    }
    CUDA_TRY(cudaMemcpyAsync(h->ct.enc_w1, sg->e1u, sizeof(sg->e1u), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(h->ct.enc_w2, sg->e2u, sizeof(sg->e2u), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(h->ct.enc_gb, sg->enc_gb, sizeof(sg->enc_gb), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(h->enc_bn, sg->enc_bn, sizeof(sg->enc_bn), cudaMemcpyHostToDevice, st));
  }
  CUDA_TRY(cudaEventRecord(h->pack_done, st));
  if (loop_stale) drop_graph(h, dd_engine::G_LOOP);
  if (loop_stale || steps_stale) {
    drop_graph(h, dd_engine::G_LOOP_STEPS);
    drop_graph(h, dd_engine::G_LOOP_STEPS_TRAIN);
  }
  return DD_OK;
}

// Pack one layer of the convgen_wgmma_kernel path, a producer conv or a Linear, from its raw weight w ([cout][cin]
// [taps], or ConvT [cin][co][2][2] when transposed) followed by eval-BN bn[0..3] (device vectors of cout_conv, see
// bn_fold; folded), or — bn null — by the plain device bias `bias` (null: none).  cin_pad >= cin zero-pads the
// input-channel axis (RGB -> 64).  nt > 0 forces the N-tile width (64, 128, 192 or 256; 0: the width chosen below).
// Every device buffer is recorded in `owned`.  `name` labels errors.
int pack_gen_weights(dd_engine* e, std::vector<void*>& owned, GenLayer& L, const float* w, const std::string& name,
                     const float* const* bn, const float* bias, int cin, int cout_conv, int taps, bool transposed,
                     int cin_pad, int nt, cudaStream_t st, float* scratch) {
  std::vector<float> scale(cout_conv, 1.f), shift(cout_conv, 0.f);
  int rc;
  if (bn) {
    if ((rc = bn_fold(bn, cout_conv, scale, shift, st))) return rc;
  } else if (bias) {
    CUDA_TRY(cudaMemcpyAsync(shift.data(), bias, cout_conv * 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
  }
  const int cp = cin_pad > 0 ? cin_pad : cin;
  L.cin = cp;
  L.taps = transposed ? 1 : taps;
  L.cout = transposed ? 4 * cout_conv : cout_conv;
  L.shuffle = transposed ? 1 : 0;
  L.relu = 1;
  // N tile: the width in {256, 192, 128} that wastes the fewest padded columns (ties -> wider); 64 for cout <= 64.
  // A last tile wider than the remaining channels reads zero weight rows (TMA out-of-bounds fill), the epilogue drops
  // them; partial K chunks are completed with zeros the same way (MPViT widths: 216, 288, 648, 864 ...).
  L.nt = 64;
  if (nt > 0) {
    if (nt != 64 && nt != 128 && nt != 192 && nt != 256) return fail(DD_ERR_INVALID, "N tile must be 64, 128, 192 or 256");
    L.nt = nt;
  } else if (L.cout > 64) {
    int best = 1 << 30;
    for (int width : {256, 192, 128}) {
      const int padded = (L.cout + width - 1) / width * width;
      if (padded < best) { best = padded; L.nt = width; }
    }
  }
  if (L.cout % 8 != 0 || cp % 8 != 0) return fail(DD_ERR_UNSUPPORTED, "channels must be multiples of 8: " + name);
  const int cout_pad = (L.cout + L.nt - 1) / L.nt * L.nt;
  const size_t n = static_cast<size_t>(L.cout) * cp * L.taps;
  float* d_scale = nullptr;  // per output channel; nullptr: 1
  if ((rc = dev_alloc(owned, reinterpret_cast<void**>(&L.w_hi), n * 2))) return rc;
  if ((rc = dev_alloc(owned, reinterpret_cast<void**>(&L.w_lo), n * 2))) return rc;
  if ((rc = dev_alloc(owned, reinterpret_cast<void**>(&L.shift), cout_pad * 4))) return rc;
  if (bn) {
    if ((rc = dev_alloc(owned, reinterpret_cast<void**>(&d_scale), cout_conv * 4))) return rc;
    CUDA_TRY(cudaMemcpyAsync(d_scale, scale.data(), cout_conv * 4, cudaMemcpyHostToDevice, st));
  }
  if (cp != cin) {
    CUDA_TRY(cudaMemsetAsync(L.w_hi, 0, n * 2, st));
    CUDA_TRY(cudaMemsetAsync(L.w_lo, 0, n * 2, st));
  }
  std::vector<float> shift_full(cout_pad, 0.f);
  for (int i = 0; i < L.cout; ++i) shift_full[i] = shift[i % cout_conv];
  CUDA_TRY(cudaMemcpyAsync(L.shift, shift_full.data(), cout_pad * 4, cudaMemcpyHostToDevice, st));
  if (gen_parts(L.taps, gen_chunks(cp) + 1) > 1) {  // two sources may add a partial chunk
    if ((rc = dev_alloc(owned, reinterpret_cast<void**>(&L.zero_shift), cout_pad * 4))) return rc;
    CUDA_TRY(cudaMemsetAsync(L.zero_shift, 0, cout_pad * 4, st));
  }
  const int nraw = static_cast<int>(static_cast<size_t>(cout_conv) * cin * (transposed ? 4 : taps));
  if ((rc = split_scale(scratch, st, &L.wscale, [&] {
         dd::absmax_scaled_kernel<<<absmax_grid(nraw), 256, 0, st>>>(w, d_scale, nraw, cin * L.taps, cout_conv,
                                                                     L.shuffle, scratch);
       })))
    return rc;
  dd::pack_gen_weight_kernel<<<256, 256, 0, st>>>(w, d_scale, L.w_hi, L.w_lo, L.cout, cin, L.taps, L.shuffle, L.wscale, cp);
  if ((rc = check_launch("pack_gen_weight"))) return rc;
  CUDA_TRY(cudaStreamSynchronize(st));
  if ((rc = make_weight_map(&L.mb_hi, L.w_hi, L.cout, cp, L.taps, dd::GEN_BK, dd::gen_unit_cols(L.nt)))) return rc;
  if ((rc = make_weight_map(&L.mb_lo, L.w_lo, L.cout, cp, L.taps, dd::GEN_BK, dd::gen_unit_cols(L.nt)))) return rc;
  // cout divisible by 256 and 192: launch_gen may pick the width whose last wave wastes least
  L.alt = (L.nt == 256 && L.cout % 256 == 0 && L.cout % 192 == 0 && !L.shuffle);
  if (L.alt) {
    if ((rc = make_weight_map(&L.mb_hi_alt, L.w_hi, L.cout, cp, L.taps, dd::GEN_BK, dd::gen_unit_cols(192)))) return rc;
    if ((rc = make_weight_map(&L.mb_lo_alt, L.w_lo, L.cout, cp, L.taps, dd::GEN_BK, dd::gen_unit_cols(192)))) return rc;
  }
  return DD_OK;
}

// Where a producer layer's BatchNorm runs in DD_PRODUCER_TRAIN: the call (0 dd_run_backbone, 1 dd_build_condition;
// -1 not at all) and the pixel count of the pre-BN output (a ConvT's: B x 2H x 2W).
struct TrainBn {
  int stage = -1;
  long long n = 0;
};

// Appends the training-mode record `b` of the BatchNorm `bnkey` (C channels; the caller packed its unfolded conv) to
// pt.layers with device copies of gamma / beta; *index receives its position.
int push_bn_record(dd_engine* e, dd_engine::ProdBn& b, const std::string& bnkey, int C, TrainBn train, int* index,
                   cudaStream_t st) {
  b.C = C;
  b.stage = train.stage;
  b.n = train.n;
  b.key = bnkey;
  int rc;
  if ((rc = copy_param(e, bnkey + ".weight", C, &b.gamma, st))) return rc;
  if ((rc = copy_param(e, bnkey + ".bias", C, &b.beta, st))) return rc;
  *index = static_cast<int>(e->pt.layers.size());
  e->pt.layers.push_back(b);
  return DD_OK;
}

// conv weight key `wkey` ([cout][cin][k][k], or ConvT [cin][co][2][2] when transposed); see pack_gen_weights.  With
// `train` and DD_FLAG_PRODUCER_TRAIN, the BatchNorm `bnkey` also gets its training-mode record in pt.layers (L.bn): the
// conv packed unfolded (no BatchNorm, no bias, zero shift) and device copies of gamma / beta.
int pack_gen(dd_engine* e, GenLayer& L, const std::string& wkey, const std::string& bnkey, int cin, int cout_conv,
             int taps, bool transposed, cudaStream_t st, float* scratch, int cin_pad = 0,
             const std::string& biaskey = std::string(), TrainBn train = TrainBn()) {
  L.bn = -1;  // the Producers' layers outlive a pack: no index from an earlier one may survive
  const Raw* w = find(e, wkey);
  if (!w) return fail(DD_ERR_INVALID, "missing weights: " + wkey);
  const int k = taps == 9 ? 3 : (transposed ? 2 : 1);
  std::vector<int64_t> want = transposed ? std::vector<int64_t>{cin, cout_conv, 2, 2}
                                         : std::vector<int64_t>{cout_conv, cin, k, k};
  if (w->shape != want) return fail(DD_ERR_INVALID, "weight shape mismatch: " + wkey);
  const float* bn[4] = {nullptr, nullptr, nullptr, nullptr};
  const float* bias = nullptr;
  int rc;
  if (!bnkey.empty()) {
    if ((rc = find_bn(e, bnkey, bn))) return rc;
  } else if (!biaskey.empty()) {
    const Raw* b = find(e, biaskey);
    if (!b) return fail(DD_ERR_INVALID, "missing weights: " + biaskey);
    bias = b->ptr;
  }
  if ((rc = pack_gen_weights(e, e->owned, L, w->ptr, wkey, bnkey.empty() ? nullptr : bn, bias, cin, cout_conv, taps,
                             transposed, cin_pad, 0, st, scratch)))
    return rc;
  if (train.stage < 0 || !(e->cfg.flags & DD_FLAG_PRODUCER_TRAIN)) return DD_OK;
  dd_engine::ProdBn b;
  if ((rc = pack_gen_weights(e, e->owned, b.raw, w->ptr, wkey, nullptr, nullptr, cin, cout_conv, taps, transposed,
                             cin_pad, 0, st, scratch)))
    return rc;
  return push_bn_record(e, b, bnkey, cout_conv, train, &L.bn, st);
}

// nn.Linear: weight key `wkey` [N][K], bias key `bkey` (empty: none).  run_gemm supplies the activation.
int pack_linear(dd_engine* e, GenLayer& L, const std::string& wkey, const std::string& bkey, int N, int K,
                cudaStream_t st, float* scratch) {
  const Raw* w = find(e, wkey);
  if (!w) return fail(DD_ERR_INVALID, "missing weights: " + wkey);
  if (w->shape != std::vector<int64_t>{N, K}) return fail(DD_ERR_INVALID, "weight shape mismatch: " + wkey);
  const Raw* b = nullptr;
  if (!bkey.empty() && !(b = find(e, bkey))) return fail(DD_ERR_INVALID, "missing weights: " + bkey);
  return pack_gen_weights(e, e->owned, L, w->ptr, wkey, nullptr, b ? b->ptr : nullptr, K, N, 1, false, 0, 0, st,
                          scratch);
}

// In evaluation order, which is that of the training-mode records: the neck level by level, then the FPN top-down.
int pack_producers(dd_engine* e, cudaStream_t st, float* scratch) {
  Producers& p = e->prod;
  const long long B = e->cfg.batch;
  int rc;
  for (int i = 0; p.neck && i < p.nlev; ++i) {
    const std::string si = std::to_string(i), h = "hahineck.";
    const TrainBn bn = {1, B * p.H[i] * p.W[i]};
    if ((rc = pack_gen(e, p.lat[i], h + "lateral_convs." + si + ".conv.weight", h + "lateral_convs." + si + ".bn",
                       p.C[i], p.C[i], 1, false, st, scratch, 0, "", bn))) return rc;
    const std::string pj = i == 0 ? h + "conv_proj.0" : h + "trans_proj." + std::to_string(i - 1);
    const std::string fs = i == 0 ? h + "conv_fusion.0" : h + "trans_fusion." + std::to_string(i - 1);
    if ((rc = pack_gen(e, p.proj[i], pj + ".conv.weight", pj + ".bn", p.C[i], 512, 1, false, st, scratch, 0, "", bn)))
      return rc;
    if ((rc = pack_gen(e, p.fus[i], fs + ".conv.weight", fs + ".bn", p.C[i] + 512, p.C[i], 9, false, st, scratch, 0, "",
                       bn))) return rc;
  }
  for (int i = p.nlev - 1; i >= 0; --i) {
    const std::string si = std::to_string(i);
    const long long n = B * p.H[i] * p.W[i];
    if ((rc = pack_gen(e, p.fl[i], "conv_lateral." + si + ".0.weight", "conv_lateral." + si + ".1", p.C[i], 256, 9, false,
                       st, scratch, 0, "", {1, n}))) return rc;
    if (i > 0) {  // the ConvT from level i up to level i - 1
      const std::string su = std::to_string(i - 1);
      if ((rc = pack_gen(e, p.fu[i - 1], "conv_up." + su + ".0.weight", "conv_up." + su + ".1", 256, 256, 1, true, st,
                         scratch, 0, "", {1, 4 * n}))) return rc;
    }
  }
  p.ready = true;
  return DD_OK;
}

template <int NT>
void convgen_kernel(int grid, cudaStream_t st, const CUtensorMap* m, const dd::GenConvArgs& a) {
  dd::convgen_wgmma_kernel<NT><<<grid, dd::GenCfg<NT>::THREADS, dd::GenCfg<NT>::SMEM_BYTES, st>>>(m[0], m[1], m[2], m[3],
                                                                                                 m[4], m[5], a);
}

// Output grid of one convgen_wgmma_kernel launch: B images of H x W pixels, the first m_valid of them real (0: all).
// A stride-2 layer reads its sources on the src_h x src_w grid.
struct GenGrid {
  int B, H, W, m_valid, src_h, src_w;
};

// What one launch_gen launched: the N-tile width, the work items (M tiles x N tiles) and the persistent grid.
struct GenLaunch {
  int nt, work, grid, parts;
};

// Every launch of layer L on convgen_wgmma_kernel (producer convs and Linears): activation act, sources a0 (c0
// channels) and a1 (c1, concatenated after a0; c1 = 0: none), outputs y32 (fp32, + add32) and / or the split planes
// *out with row width ld_out (0: L.cout) from channel ch_off on.  alt: a layer with 192-wide alternative maps uses them
// when its last wave wastes less (0), always (1) or never (-1).  info (nullable) receives what was launched (per launch
// of a layer split along K).  partial: fp32 [pixels][L.cout] for the partial sums of a layer split along K.
int launch_gen(dd_engine* e, const GenLayer& L, int act, const GenGrid& g, const Planes& a0, int c0, const Planes& a1,
               int c1, float* y32, const float* add32, const Planes* out, int ld_out, int ch_off, cudaStream_t st,
               int alt = 0, GenLaunch* info = nullptr, float* partial = nullptr) {
  if (c0 + c1 != L.cin) return fail(DD_ERR_INVALID, "producer conv: source channels do not match the layer");
  dd::GenConvArgs a;
  a.B = g.B;
  a.H = g.H;
  a.W = g.W;
  a.tiles_x = (g.W + dd::TILE_W - 1) / dd::TILE_W;
  a.tiles_y = (g.H + dd::TILE_H - 1) / dd::TILE_H;
  a.m_tiles = a.tiles_x * a.tiles_y * g.B;
  // wave quantisation: with few M tiles pick the N-tile width whose last wave wastes least — deep Swin stages, and the
  // level-2 fusion conv of the HAHI neck (768 channels, 30 tile pairs) runs 2 waves of 192 columns instead of 2 of 256
  int nt = L.nt;
  if (L.alt && alt >= 0) {
    const int units = a.m_tiles, slots = e->sm_count;
    auto cost = [&](int w) { return ((units * (L.cout / w) + slots - 1) / slots) * w; };
    if (alt > 0 || cost(192) < cost(256)) nt = 192;
  }
  a.n_tiles = (L.cout + nt - 1) / nt;
  a.kc0 = (c0 + dd::GEN_BK - 1) / dd::GEN_BK;  // a partial last chunk is zero-filled by TMA on both operands
  a.kc1 = (c1 + dd::GEN_BK - 1) / dd::GEN_BK;
  a.c0_ch = c0;
  a.taps = L.taps;
  a.cout = L.cout;
  a.ld_out = ld_out > 0 ? ld_out : L.cout;  // branches of a concatenation write straight into the concatenated planes
  a.ch_off = ch_off;
  a.shift = L.shift;
  a.acc_scale = 1.f / (kProdScale * L.wscale);
  a.relu = act;
  a.m_valid = g.m_valid;
  a.stride = L.stride;
  a.add_first = L.add_first;
  a.shuffle = L.shuffle;
  a.y32 = y32;
  a.add32 = add32;
  a.out_hi = out ? out->hi : nullptr;
  a.out_lo = out ? out->lo : nullptr;
  a.split_scale = kProdScale;
  a.status = e->status;
  const bool use_alt = nt != L.nt;
  CUtensorMap m[6];  // sources 0 and 1 (hi, lo), weights (hi, lo)
  const int sh = L.stride == 1 ? g.H : g.src_h, sw = L.stride == 1 ? g.W : g.src_w;
  const int grid = std::min(a.m_tiles * a.n_tiles, e->sm_count);
  const int parts = gen_parts(L.taps, a.kc0 + a.kc1);
  if (info) *info = {nt, a.m_tiles * a.n_tiles, grid, parts};
  auto launch = [&](const dd::GenConvArgs& args) {
    switch (nt) {
      case 256: convgen_kernel<256>(grid, st, m, args); break;
      case 192: convgen_kernel<192>(grid, st, m, args); break;
      case 128: convgen_kernel<128>(grid, st, m, args); break;
      default: convgen_kernel<64>(grid, st, m, args); break;
    }
    return launched(e, "convgen");
  };
  int rc;
  if (parts == 1) {
    if ((rc = make_act_map(&m[0], a0.hi, g.B, sh, sw, c0, dd::GEN_BK, L.stride))) return rc;
    if ((rc = make_act_map(&m[1], a0.lo, g.B, sh, sw, c0, dd::GEN_BK, L.stride))) return rc;
    if (c1 > 0) {
      if ((rc = make_act_map(&m[2], a1.hi, g.B, g.H, g.W, c1, dd::GEN_BK))) return rc;
      if ((rc = make_act_map(&m[3], a1.lo, g.B, g.H, g.W, c1, dd::GEN_BK))) return rc;
    } else {
      m[2] = m[0];
      m[3] = m[1];
    }
    m[4] = use_alt ? L.mb_hi_alt : L.mb_hi;
    m[5] = use_alt ? L.mb_lo_alt : L.mb_lo;
    return launch(a);
  }
  // Split along K (kGenSplitIters): `parts` launches over contiguous ranges of the concatenated 64-channel chunks, every
  // tap each.  Launch p < parts - 1 writes partial = acc_p (+ partial), the last one adds the partial sum before its shift
  // and activation and writes the real outputs: a fixed-order fp32 sum, bit-reproducible.
  if (add32 || L.shuffle || !partial || !L.zero_shift)
    return fail(DD_ERR_UNSUPPORTED, "producer conv deeper than one accumulator takes, with an addend or no partial buffer");
  const int kc_total = a.kc0 + a.kc1, per = (kc_total + parts - 1) / parts;
  for (int p = 0; p * per < kc_total; ++p) {
    const int ka = p * per, kb = std::min(kc_total, ka + per);
    // chunks [ka, kb): source-0 chunks [s0a, s0b) (channels from s0a * GEN_BK, w0 of them), then source-1 chunks
    const int s0a = std::min(ka, a.kc0), s0b = std::min(kb, a.kc0);
    const int s1a = std::max(ka, a.kc0) - a.kc0, s1b = std::max(kb, a.kc0) - a.kc0;
    const int w0 = std::min(s0b * dd::GEN_BK, c0) - s0a * dd::GEN_BK;
    const int w1 = std::min(s1b * dd::GEN_BK, c1) - s1a * dd::GEN_BK;
    // The part's weight columns are contiguous (a part that reaches into source 1 holds source 0's last chunk).  Every
    // map starts on a 64-channel (128-byte) boundary: a source-1-only part behind a source 0 of c0 % 64 != 0 channels
    // runs as a source 0 of no chunks whose source-1 weights start c0 % 64 columns into its map.
    dd::GenConvArgs ap = a;
    int wcol, wlen;
    if (w0 > 0) {
      if ((rc = make_act_map(&m[0], a0.hi + s0a * dd::GEN_BK, g.B, sh, sw, w0, dd::GEN_BK, L.stride, c0))) return rc;
      if ((rc = make_act_map(&m[1], a0.lo + s0a * dd::GEN_BK, g.B, sh, sw, w0, dd::GEN_BK, L.stride, c0))) return rc;
      ap.kc0 = s0b - s0a;
      ap.c0_ch = w0;
      wcol = s0a * dd::GEN_BK;
      wlen = w0 + w1;
    } else {
      ap.kc0 = 0;
      ap.c0_ch = (c0 + s1a * dd::GEN_BK) % dd::GEN_BK;
      wcol = c0 + s1a * dd::GEN_BK - ap.c0_ch;
      wlen = ap.c0_ch + w1;
    }
    ap.kc1 = s1b - s1a;
    if (w1 > 0) {
      if ((rc = make_act_map(&m[2], a1.hi + s1a * dd::GEN_BK, g.B, g.H, g.W, w1, dd::GEN_BK, 1, c1))) return rc;
      if ((rc = make_act_map(&m[3], a1.lo + s1a * dd::GEN_BK, g.B, g.H, g.W, w1, dd::GEN_BK, 1, c1))) return rc;
    }
    if (w0 == 0) {
      m[0] = m[2];
      m[1] = m[3];
    } else if (w1 == 0) {
      m[2] = m[0];
      m[3] = m[1];
    }
    if ((rc = make_weight_map(&m[4], L.w_hi + wcol, L.cout, wlen, L.taps, dd::GEN_BK, dd::gen_unit_cols(nt), L.cin))) return rc;
    if ((rc = make_weight_map(&m[5], L.w_lo + wcol, L.cout, wlen, L.taps, dd::GEN_BK, dd::gen_unit_cols(nt), L.cin))) return rc;
    const bool last = kb == kc_total;
    ap.relu = last ? act : 0;
    ap.shift = last ? L.shift : L.zero_shift;
    ap.add_first = 1;
    ap.add32 = p > 0 ? partial : nullptr;
    ap.y32 = last ? y32 : partial;
    ap.out_hi = last ? a.out_hi : nullptr;
    ap.out_lo = last ? a.out_lo : nullptr;
    ap.ld_out = last ? a.ld_out : L.cout;
    ap.ch_off = last ? ch_off : 0;
    if ((rc = launch(ap))) return rc;
  }
  return DD_OK;
}

// ------------------------------------------------------------------------------------------------ producer BatchNorms
int pbn_blocks(long long n) { return static_cast<int>((n + dd::PBN_ROWS - 1) / dd::PBN_ROWS); }

// DD_FLAG_PRODUCER_TRAIN (producer_train.cuh): the records' offsets, in the order pack_gen appended them, and the
// scratch for the largest layer.
int pack_prod_train(dd_engine* e, cudaStream_t st) {
  dd_engine::ProdTrain& pt = e->pt;
  size_t u_max = 0, part_max = 0;
  int c_max = 0;
  for (dd_engine::ProdBn& b : pt.layers) {
    b.rec_off = pt.rec_floats;
    pt.rec_floats += 2 * static_cast<size_t>(b.C);
    u_max = std::max(u_max, static_cast<size_t>(b.n) * b.C);
    part_max = std::max(part_max, static_cast<size_t>(pbn_blocks(b.n)) * 2 * b.C);
    c_max = std::max(c_max, b.C);
  }
  if (pt.layers.empty()) return DD_OK;
  int rc;
  if ((rc = dev_array(e, &pt.U, u_max))) return rc;
  if ((rc = dev_array(e, &pt.part, part_max))) return rc;
  if ((rc = dev_array(e, &pt.sum1, c_max))) return rc;
  if ((rc = dev_array(e, &pt.s, c_max))) return rc;
  if ((rc = dev_array(e, &pt.t, c_max))) return rc;
  if ((rc = dev_array(e, &pt.rec, pt.rec_floats))) return rc;
  CUDA_TRY(cudaMemsetAsync(pt.rec, 0, pt.rec_floats * 4, st));
  return DD_OK;
}

// The training-mode BatchNorm of record b on the pre-BN value in pt.U (b.n pixels): pbn_stats_kernel's two passes and
// the fold (run_bn_passes), which write the record, then act(s u + t) (`act` as the eval epilogue's code)
// with the addend add32 placed as add_first says, into y32 and / or the planes *out (row width ld_out, 0: b.C).
int run_producer_bn(dd_engine* e, const dd_engine::ProdBn& b, int act, int add_first, const float* add32, float* y32,
                    const Planes* out, int ld_out, int ch_off, cudaStream_t st) {
  dd_engine::ProdTrain& pt = e->pt;
  const long long n = b.n;
  const int C = b.C, nblk = pbn_blocks(n);
  const dim3 grid(nblk, (C + dd::PBN_CH - 1) / dd::PBN_CH), block(dd::PBN_CH, 8);
  auto stats = [&](const double* sum1, const double* cnt) {
    dd::pbn_stats_kernel<<<grid, block, 0, st>>>(pt.U, n, C, sum1, cnt, pt.part);
    return launched(e, "pbn_stats");
  };
  auto fold = [&](const dd::BnFoldIn& in) {
    dd::pbn_fold_kernel<<<(C + 255) / 256, 256, 0, st>>>(in, C, b.gamma, b.beta, pt.s, pt.t, pt.rec + b.rec_off);
    return launched(e, "pbn_fold");
  };
  int rc;
  if ((rc = run_bn_passes(e, pt.part, nblk, C, n, pt.sum1, st, stats, fold))) return rc;
  dd::PbnApplyArgs a;
  a.u = pt.U;
  a.n = n;
  a.C = C;
  a.relu = act;
  a.add_first = add_first;
  a.s = pt.s;
  a.t = pt.t;
  a.add32 = add32;
  a.y32 = y32;
  a.out_hi = out ? out->hi : nullptr;
  a.out_lo = out ? out->lo : nullptr;
  a.ld_out = ld_out > 0 ? ld_out : C;
  a.ch_off = ch_off;
  a.split_scale = kProdScale;
  a.status = e->status;
  dd::pbn_apply_kernel<<<grid_of(static_cast<size_t>(n) * C / 8), 256, 0, st>>>(a);
  return launched(e, "pbn_apply");
}

// H, W: OUTPUT grid.  With L.stride == 2 the sources live on a (src_h, src_w) grid.  A layer with a training-mode
// BatchNorm (L.bn) in DD_PRODUCER_TRAIN runs its conv on the unfolded pack into pt.U, then the batch statistics and fold
// (record written), then act(s u + t) with L's addend and outputs.
int run_gen(dd_engine* e, const GenLayer& L, const Planes& a0, int c0, const Planes& a1, int c1, int H, int W,
            float* y32, const float* add32, const Planes* out, cudaStream_t st, int src_h = 0, int src_w = 0,
            int ld_out = 0, int ch_off = 0) {
  if (L.bn < 0 || e->producer_mode != DD_PRODUCER_TRAIN)
    return launch_gen(e, L, L.relu, {e->cfg.batch, H, W, 0, src_h, src_w}, a0, c0, a1, c1, y32, add32, out, ld_out,
                      ch_off, st, 0, nullptr, e->prod.KS);
  dd_engine::ProdTrain& pt = e->pt;
  const dd_engine::ProdBn& b = pt.layers[L.bn];
  const long long n = static_cast<long long>(e->cfg.batch) * H * W * (L.shuffle ? 4 : 1);
  if (n != b.n) return fail(DD_ERR_INVALID, b.key + ": output grid differs from the packed geometry");
  GenLayer raw = b.raw;  // the unfolded weights; the layer's shape is L's
  raw.stride = L.stride;
  int rc;
  if ((rc = launch_gen(e, raw, 0, {e->cfg.batch, H, W, 0, src_h, src_w}, a0, c0, a1, c1, pt.U, nullptr, nullptr, 0, 0,
                       st, 0, nullptr, e->prod.KS)))
    return rc;
  return run_producer_bn(e, b, L.relu, L.add_first, add32, y32, out, ld_out, ch_off, st);
}

// A forward starts (dd_run_backbone, dd_build_condition with feature maps): no record is current.
void producer_forward_start(dd_engine* e) {
  for (auto& b : e->pt.layers) b.fresh = false;
}
// After a call of `stage` (0 backbone, 1 neck + FPN) in DD_PRODUCER_TRAIN: its layers' records are current.
void producer_mark_fresh(dd_engine* e, int stage) {
  for (auto& b : e->pt.layers)
    if (b.stage == stage) b.fresh = true;
}

// ------------------------------------------------------------------------------------------------ ResNet backbone
// ResNetForMMBEV with BasicBlocks and no stem (reference src/model/backbone/mmbev_resnet.py:124-160; block = mmdet
// BasicBlock): per stage, block 0 = conv3x3(s2)+BN+ReLU -> conv3x3+BN, skip = biased conv3x3(s2) without BN; other
// blocks are stride 1 with identity skips.  Stride-2 convs use TMA element strides on the same tensor-core conv kernel.
int pack_resnet(dd_engine* e, cudaStream_t st, float* scratch) {
  ResNetW& r = e->rn;
  int rc;
  for (int s = 0; s < 4; ++s) {
    r.blocks[s].assign(r.depths[s], ResBlockW());
    const int cprev = s == 0 ? 3 : r.C[s - 1];
    const TrainBn bn = {0, static_cast<long long>(e->cfg.batch) * r.Hs[s] * r.Ws[s]};
    for (int b = 0; b < r.depths[s]; ++b) {
      ResBlockW& W = r.blocks[s][b];
      const std::string bp = "backbone.layers." + std::to_string(s) + "." + std::to_string(b) + ".";
      const int cin = b == 0 ? cprev : r.C[s];
      const int pad = (cin % dd::GEN_BK) ? dd::GEN_BK : 0;
      if ((rc = pack_gen(e, W.c1, bp + "conv1.weight", bp + "bn1", cin, r.C[s], 9, false, st, scratch, pad, "", bn)))
        return rc;
      W.c1.stride = b == 0 ? 2 : 1;
      if ((rc = pack_gen(e, W.c2, bp + "conv2.weight", bp + "bn2", r.C[s], r.C[s], 9, false, st, scratch, 0, "", bn)))
        return rc;
      W.c2.add_first = 1;  // out = relu(bn2(conv2) + skip)
      W.has_ds = (b == 0);
      if (W.has_ds) {
        if ((rc = pack_gen(e, W.ds, bp + "downsample.weight", "", cin, r.C[s], 9, false, st, scratch, pad,
                           bp + "downsample.bias"))) return rc;
        W.ds.stride = 2;
        W.ds.relu = 0;
      }
    }
  }
  r.ready = true;
  return DD_OK;
}

int run_resnet(dd_engine* e, const float* rgb, float* const* feats_out, cudaStream_t st) {
  ResNetW& r = e->rn;
  const int B = e->cfg.batch;
  {
    const size_t n = static_cast<size_t>(B) * r.H * r.W * dd::GEN_BK;
    dd::rgb_to_planes_kernel<<<grid_of(n), 256, 0, st>>>(rgb, r.IN.hi, r.IN.lo, B, r.H * r.W, kProdScale, e->status);
  }
  int rc;
  if ((rc = launched(e, "rgb_to_planes"))) return rc;
  const Planes none;
  Planes src = r.IN;
  int src_c = dd::GEN_BK, src_h = r.H, src_w = r.W;
  for (int s = 0; s < 4; ++s) {
    const int C = r.C[s], H = r.Hs[s], W = r.Ws[s];
    int cur = 0;
    for (int b = 0; b < r.depths[s]; ++b) {
      const ResBlockW& Wt = r.blocks[s][b];
      const bool last = (b == r.depths[s] - 1);
      const int k = b & 1;
      const Planes& in = (b == 0) ? src : r.Yp[cur];
      const int in_c = (b == 0) ? src_c : C;
      if ((rc = run_gen(e, Wt.c1, in, in_c, none, 0, H, W, nullptr, nullptr, &r.T, st, src_h, src_w))) return rc;
      const float* skip;
      if (Wt.has_ds) {
        if ((rc = run_gen(e, Wt.ds, in, in_c, none, 0, H, W, r.D32, nullptr, nullptr, st, src_h, src_w))) return rc;
        skip = r.D32;
      } else {
        skip = r.Y32[cur];
      }
      const Planes& outp = last ? e->prod.F[s] : r.Yp[k];
      if ((rc = run_gen(e, Wt.c2, r.T, C, none, 0, H, W, r.Y32[k], skip, &outp, st))) return rc;
      cur = k;
    }
    if (feats_out && feats_out[s]) {
      if ((rc = transpose_out(r.Y32[cur], feats_out[s], B, C, H * W, st))) return rc;
      e->launches++;
    }
    src = e->prod.F[s];
    src_c = C;
    src_h = H;
    src_w = W;
  }
  return DD_OK;
}

// ------------------------------------------------------------------------------------------------ Swin backbone
constexpr float kTokScale = 16.f;  // fp16-split pre-scale of token activations (LayerNorm / GELU / attention outputs)
static_assert(kTokScale == kProdScale, "run_gemm reads token planes at the producers' split scale");

int pack_backbone(dd_engine* e, cudaStream_t st, float* scratch) {
  Backbone& b = e->bb;
  const std::string P = "backbone.";
  int rc;
  if ((rc = copy_param(e, P + "patch_embed.projection.weight", static_cast<size_t>(b.E) * 48, &b.pe_w, st))) return rc;
  if ((rc = copy_param(e, P + "patch_embed.projection.bias", b.E, &b.pe_b, st))) return rc;
  if ((rc = copy_param(e, P + "patch_embed.norm.weight", b.E, &b.pe_g, st))) return rc;
  if ((rc = copy_param(e, P + "patch_embed.norm.bias", b.E, &b.pe_beta, st))) return rc;
  for (int s = 0; s < 4; ++s) {
    const int C = b.E << s;
    SwinStageW& S = b.stage[s];
    S.blocks.assign(b.depths[s], SwinBlockW());
    for (int k = 0; k < b.depths[s]; ++k) {
      SwinBlockW& W = S.blocks[k];
      const std::string bp = P + "stages." + std::to_string(s) + ".blocks." + std::to_string(k) + ".";
      if ((rc = copy_param(e, bp + "norm1.weight", C, &W.ln1_g, st))) return rc;
      if ((rc = copy_param(e, bp + "norm1.bias", C, &W.ln1_b, st))) return rc;
      if ((rc = copy_param(e, bp + "norm2.weight", C, &W.ln2_g, st))) return rc;
      if ((rc = copy_param(e, bp + "norm2.bias", C, &W.ln2_b, st))) return rc;
      if ((rc = copy_param(e, bp + "attn.w_msa.relative_position_bias_table", static_cast<size_t>(169) * b.heads[s], &W.table, st))) return rc;
      if ((rc = pack_linear(e, W.qkv, bp + "attn.w_msa.qkv.weight", bp + "attn.w_msa.qkv.bias", 3 * C, C, st, scratch))) return rc;
      if ((rc = pack_linear(e, W.proj, bp + "attn.w_msa.proj.weight", bp + "attn.w_msa.proj.bias", C, C, st, scratch))) return rc;
      if ((rc = pack_linear(e, W.ffn1, bp + "ffn.layers.0.0.weight", bp + "ffn.layers.0.0.bias", 4 * C, C, st, scratch))) return rc;
      if ((rc = pack_linear(e, W.ffn2, bp + "ffn.layers.1.weight", bp + "ffn.layers.1.bias", C, 4 * C, st, scratch))) return rc;
    }
    const std::string np = P + "norm" + std::to_string(s) + ".";
    if ((rc = copy_param(e, np + "weight", C, &S.out_g, st))) return rc;
    if ((rc = copy_param(e, np + "bias", C, &S.out_b, st))) return rc;
    if (s < 3) {
      const std::string dp = P + "stages." + std::to_string(s) + ".downsample.";
      if ((rc = copy_param(e, dp + "norm.weight", 4 * C, &S.dn_g, st))) return rc;
      if ((rc = copy_param(e, dp + "norm.bias", 4 * C, &S.dn_b, st))) return rc;
      if ((rc = pack_linear(e, S.reduction, dp + "reduction.weight", "", 2 * C, 4 * C, st, scratch))) return rc;
    }
  }
  CUDA_TRY(cudaStreamSynchronize(st));
  b.ready = true;
  return DD_OK;
}

// y = act(A[M][K] @ W^T + bias) (+ add32): tokens are laid out as a [ceil(M/16)][16] "image" for the conv kernel
int run_gemm(dd_engine* e, const GenLayer& L, const Planes& A, int M, int act, float* y32, const float* add32,
             const Planes* out, cudaStream_t st, int ld_out = 0, int ch_off = 0) {
  return launch_gen(e, L, act, {1, (M + 15) / 16, 16, M, 0, 0}, A, L.cin, Planes(), 0, y32, add32, out, ld_out, ch_off,
                    st);
}

int run_ln(dd_engine* e, int C, const float* x, const float* g, const float* b, const Planes& out, int M, float* nchw,
           int HW, cudaStream_t st) {
  const int grid = (M + 7) / 8;
  switch (C) {
    case 192: dd::ln_split_kernel<192><<<grid, 256, 0, st>>>(x, g, b, out.hi, out.lo, kTokScale, M, nchw, HW, e->status); break;
    case 384: dd::ln_split_kernel<384><<<grid, 256, 0, st>>>(x, g, b, out.hi, out.lo, kTokScale, M, nchw, HW, e->status); break;
    case 768: dd::ln_split_kernel<768><<<grid, 256, 0, st>>>(x, g, b, out.hi, out.lo, kTokScale, M, nchw, HW, e->status); break;
    case 1536: dd::ln_split_kernel<1536><<<grid, 256, 0, st>>>(x, g, b, out.hi, out.lo, kTokScale, M, nchw, HW, e->status); break;
    default: return fail(DD_ERR_UNSUPPORTED, "LayerNorm width not instantiated");
  }
  return launched(e, "ln_split");
}

// Swin patch embedding: 4x4/s4 conv (3 -> E) + bias + LayerNorm(E), rgb [B][3][H][W] zero-padded right / bottom to a
// multiple of 4 -> x fp32 [B * ceil(H / 4) * ceil(W / 4)][E]
int run_patch_embed(dd_engine* e, int E, const float* rgb, const float* w, const float* bias, const float* g,
                    const float* beta, float* x, int B, int H, int W, cudaStream_t st) {
  if (E != 192) return fail(DD_ERR_UNSUPPORTED, "patch embedding width not instantiated");
  const int Hp = (H + 3) / 4, Wp = (W + 3) / 4;
  const int segs = (Wp + dd::PE_TOK - 1) / dd::PE_TOK;
  dd::patch_embed_kernel<192><<<segs * Hp * B, 192, 0, st>>>(rgb, w, bias, g, beta, x, B, H, W, Hp, Wp);
  return launched(e, "patch_embed");
}

// Swin patch merging: x [B][H][W][C] -> 2x2 unfold (zero pad for odd H / W) + LayerNorm(4C) -> out planes
// [B * ceil(H / 2) * ceil(W / 2)][4C]
int run_merge_ln(dd_engine* e, int C, const float* x, const float* g, const float* b, const Planes& out, int B, int H,
                 int W, cudaStream_t st) {
  const int grid = (B * ((H + 1) / 2) * ((W + 1) / 2) + 7) / 8;
  switch (C) {
    case 192: dd::merge_ln_split_kernel<192><<<grid, 256, 0, st>>>(x, g, b, out.hi, out.lo, kTokScale, B, H, W, e->status); break;
    case 384: dd::merge_ln_split_kernel<384><<<grid, 256, 0, st>>>(x, g, b, out.hi, out.lo, kTokScale, B, H, W, e->status); break;
    case 768: dd::merge_ln_split_kernel<768><<<grid, 256, 0, st>>>(x, g, b, out.hi, out.lo, kTokScale, B, H, W, e->status); break;
    default: return fail(DD_ERR_UNSUPPORTED, "patch merging width not instantiated");
  }
  return launched(e, "merge_ln_split");
}

// Window attention on the fp32 CUDA-core kernel: the check path (DD_FLAG_SIMT_CONV) and any odd head count (the wgmma
// kernel takes heads in pairs).
bool attn_simt(const dd_engine* e, int nH) {
  return (e->cfg.flags & DD_FLAG_SIMT_CONV) || (nH & 1);
}

// One (shifted-)window attention launch (7 x 7 windows, head_dim 32): qkv fp32 [B*H*W][3C] (padded tokens carry
// qkv_bias), relative-position table [169][nH] -> out planes [B*H*W][C] at kTokScale.  simt: window_attention_kernel,
// one block per (window, head); else window_attention_wgmma_kernel on pairs of heads of one window (nH even).
// work / grid (nullable) receive the units of work and the grid launched.
int launch_attention(dd_engine* e, const float* qkv, const float* qkv_bias, const float* table, const Planes& out,
                     int B, int H, int W, int C, int nH, int shift, bool simt, cudaStream_t st, int* work = nullptr,
                     int* grid_out = nullptr) {
  constexpr int ws = 7;
  const int Hp = (H + ws - 1) / ws * ws, Wp = (W + ws - 1) / ws * ws;
  dd::AttnArgs aa;
  aa.qkv = qkv;
  aa.qkv_bias = qkv_bias;
  aa.bias_table = table;
  aa.out_hi = out.hi;
  aa.out_lo = out.lo;
  aa.scale_out = kTokScale;
  aa.B = B; aa.H = H; aa.W = W; aa.C = C; aa.nH = nH;
  aa.shift = shift;
  aa.Hp = Hp; aa.Wp = Wp; aa.nWx = Wp / ws; aa.nWy = Hp / ws;
  aa.status = e->status;
  int units, grid;
  if (simt) {  // fp32 CUDA-core check path
    units = grid = B * aa.nWx * aa.nWy * nH;
    dd::window_attention_kernel<<<grid, 64, 0, st>>>(aa);
  } else {  // wgmma: pairs of heads of one window per M = 128 tile, two persistent CTAs per SM
    if (nH & 1) return fail(DD_ERR_UNSUPPORTED, "the wgmma window attention takes heads in pairs");
    units = B * aa.nWx * aa.nWy * (nH / 2);
    grid = units < 2 * e->sm_count ? units : 2 * e->sm_count;
    dd::window_attention_wgmma_kernel<<<grid, 128, dd::WAU_SMEM, st>>>(aa, units);
  }
  if (work) *work = units;
  if (grid_out) *grid_out = grid;
  return launched(e, "window_attention");
}

// x (+)= scale[b] branch over B images of n tokens of C channels (drop_path_add_kernel): into y32, or into the planes
// *out (row width ld_out, channel offset ch_off)
int run_drop_add(dd_engine* e, const float* x, const float* branch, const float* scale, int B, int n, int C, float* y32,
                 const Planes* out, int ld_out, int ch_off, cudaStream_t st) {
  dd::DropAddArgs a;
  a.x = x;
  a.branch = branch;
  a.scale = scale;
  a.per_img = n;
  a.B = B;
  a.C = C;
  a.y32 = y32;
  a.out_hi = out ? out->hi : nullptr;
  a.out_lo = out ? out->lo : nullptr;
  a.ld_out = ld_out > 0 ? ld_out : C;
  a.ch_off = ch_off;
  a.split_scale = kProdScale;
  a.status = e->status;
  dd::drop_path_add_kernel<<<grid_of(static_cast<size_t>(B) * n * C / 4), 256, 0, st>>>(a);
  return launched(e, "drop_path_add");
}

// With stochastic depth on, a marked block (reference swin.py:412,421) runs proj and ffn2 without the addend into QKV,
// dead between its attention and the next block's qkv GEMM and 3x the size of the token map, then adds each branch
// through drop_path_add_kernel; every other block adds them in the GEMM's epilogue.
int run_swin(dd_engine* e, const float* rgb, float* const* feats_out, cudaStream_t st) {
  Backbone& b = e->bb;
  const DropPathState& dp = e->drop;
  const int B = e->cfg.batch;
  int rc;
  if ((rc = run_patch_embed(e, b.E, rgb, b.pe_w, b.pe_b, b.pe_g, b.pe_beta, b.X[0], B, b.H, b.W, st))) return rc;
  int slot = 0;  // marked blocks in stage, block order
  for (int s = 0; s < 4; ++s) {
    const int C = b.E << s, H = b.Hs[s], W = b.Ws[s], M = B * H * W, nH = b.heads[s];
    float* x = b.X[s & 1];
    const int ws = b.window;
    for (int k = 0; k < b.depths[s]; ++k) {
      const SwinBlockW& Wt = b.stage[s].blocks[k];
      const float* drop = (dp.on && ((dp.mask[s] >> k) & 1)) ? dp.scales + static_cast<size_t>(slot++) * 2 * B
                                                             : nullptr;  // [attention, FFN][B]
      if ((rc = run_ln(e, C, x, Wt.ln1_g, Wt.ln1_b, b.AP, M, nullptr, 0, st))) return rc;
      if ((rc = run_gemm(e, Wt.qkv, b.AP, M, 0, b.QKV, nullptr, nullptr, st))) return rc;
      if ((rc = launch_attention(e, b.QKV, Wt.qkv.shift, Wt.table, b.AP, B, H, W, C, nH, (k & 1) ? ws / 2 : 0,
                                 attn_simt(e, nH), st))) return rc;
      if (drop) {
        if ((rc = run_gemm(e, Wt.proj, b.AP, M, 0, b.QKV, nullptr, nullptr, st))) return rc;
        if ((rc = run_drop_add(e, x, b.QKV, drop, B, H * W, C, x, nullptr, 0, 0, st))) return rc;  // x += drop(proj(attn))
      } else if ((rc = run_gemm(e, Wt.proj, b.AP, M, 0, x, x, nullptr, st))) {  // x += proj(attn)
        return rc;
      }
      if ((rc = run_ln(e, C, x, Wt.ln2_g, Wt.ln2_b, b.AP, M, nullptr, 0, st))) return rc;
      if ((rc = run_gemm(e, Wt.ffn1, b.AP, M, 2, nullptr, nullptr, &b.HP, st))) return rc;  // GELU(fc1) -> planes
      if (drop) {
        if ((rc = run_gemm(e, Wt.ffn2, b.HP, M, 0, b.QKV, nullptr, nullptr, st))) return rc;
        if ((rc = run_drop_add(e, x, b.QKV, drop + B, B, H * W, C, x, nullptr, 0, 0, st))) return rc;  // x += drop(fc2(...))
      } else if ((rc = run_gemm(e, Wt.ffn2, b.HP, M, 0, x, x, nullptr, st))) {  // x += fc2(...)
        return rc;
      }
    }
    // per-stage output norm straight into the neck's input planes (+ NCHW copy on request)
    if ((rc = run_ln(e, C, x, b.stage[s].out_g, b.stage[s].out_b, e->prod.F[s], M, feats_out ? feats_out[s] : nullptr,
                     H * W, st))) return rc;
    if (s < 3) {
      const int M2 = B * b.Hs[s + 1] * b.Ws[s + 1];
      const SwinStageW& S = b.stage[s];
      if ((rc = run_merge_ln(e, C, x, S.dn_g, S.dn_b, b.AP, B, H, W, st))) return rc;
      if ((rc = run_gemm(e, S.reduction, b.AP, M2, 0, b.X[(s + 1) & 1], nullptr, nullptr, st))) return rc;
    }
  }
  return DD_OK;
}

#include "mpvit_host.inc"

// ------------------------------------------------------------------------------------------------ backward

// GroupNorm `which` (0 ne.1, 1 ne.4, 2 pred.1, 3 pred.4) of the pre-GN output y: its mean / rstd, gamma, beta
dd::GnBwdArgs gn_args(dd_engine* e, int which, const float* y) {
  const Geom g = geom_of(e->cfg);
  dd::GnBwdArgs a{};
  a.y = y;
  a.mean_rstd = e->mr[which];
  a.gamma = e->gn_gamma[which];
  a.beta = e->gn_beta[which];
  a.B = g.B;
  a.P = g.P;
  return a;
}

// GroupNorm `which` + ReLU backward: dout (times *dscale) -> dy (unscaled)
template <int C>
int run_gn_bwd(dd_engine* e, int which, const float* dout, const float* dscale, const float* y, float* dgamma,
               float* dbeta, float* dy, cudaStream_t st) {
  const Geom g = geom_of(e->cfg);
  dd::GnBwdArgs a = gn_args(e, which, y);
  a.dout = dout;
  a.dscale = dscale;
  a.chunks = bwd_chunks(g.P);
  a.partial = e->bw.gn_part;
  a.ab = e->bw.ab;
  a.dgamma = dgamma;
  a.dbeta = dbeta;
  a.dy = dy;
  int rc;
  dd::gn_bwd_reduce_kernel<C><<<dim3(a.chunks, g.B), 256, 0, st>>>(a);
  if ((rc = launched(e, "gn_bwd_reduce"))) return rc;
  dd::gn_bwd_finalize_kernel<C><<<4, 256, 0, st>>>(a);
  if ((rc = launched(e, "gn_bwd_finalize"))) return rc;
  dd::gn_bwd_apply_kernel<C><<<grid_of(static_cast<size_t>(g.B) * g.P * C / 4), 256, 0, st>>>(a);
  return launched(e, "gn_bwd_apply");
}

// GroupNorm `which`'s output before its ReLU, fp32 NCHW [B][C][h][w]: z > 0 is run_gn_bwd's mask, bit for bit
template <int C>
int run_gn_pre_relu(dd_engine* e, int which, const float* y, float* z, cudaStream_t st) {
  const Geom g = geom_of(e->cfg);
  dd::gn_pre_relu_kernel<C><<<grid_of(static_cast<size_t>(g.B) * g.P * C), 256, 0, st>>>(gn_args(e, which, y), z);
  return launched(e, "gn_pre_relu");
}

// column sums of x [B][P][C] (times *scale): per image (out_img [B][C]) and / or over the batch in image order (out_sum
// [C]); partial holds B * bwd_chunks(P) * C floats
int run_colsum(dd_engine* e, int C, const float* x, const float* scale, int B, int P, float* partial, float* out_img,
               float* out_sum, cudaStream_t st) {
  const int chunks = bwd_chunks(P);
  const dim3 grid(chunks, B);
  switch (C) {
    case 16: dd::colsum_partial_kernel<16><<<grid, 256, 0, st>>>(x, scale, P, chunks, partial); break;
    case 64: dd::colsum_partial_kernel<64><<<grid, 256, 0, st>>>(x, scale, P, chunks, partial); break;
    case 256: dd::colsum_partial_kernel<256><<<grid, 256, 0, st>>>(x, scale, P, chunks, partial); break;
    default: return fail(DD_ERR_INVALID, "colsum: unsupported channel count");
  }
  int rc;
  if ((rc = launched(e, "colsum_partial"))) return rc;
  dd::colsum_finalize_kernel<<<C, 32, 0, st>>>(partial, B, chunks, C, out_img, out_sum);
  return launched(e, "colsum_finalize");
}

template <int TM, int TN>
void launch_wgrad(const dd::WgradArgs& a, int chunks, cudaStream_t st) {
  const dim3 grid(chunks, (a.cout / TM) * (a.cin / TN) * 9);
  dd::wgrad_simt_kernel<TM, TN><<<grid, TM * TN / 16, 0, st>>>(a);
}

// Buffers of run_wgrad: the dY split planes [B*H*W][cout] fp16, the split's absmax (zeroed before the call) and scale
// (written), the status word a non-finite dY sets, and wgrad_partial_elems fp64 partials.
struct WgradBufs {
  Planes gp;
  float* amax;
  float* scale;
  int* status;
  double* partial;
};

// Weight gradient of one 3x3 conv at B x H x W: dw [cout][cin][3][3] (nullable) = sum over pixels of dY (x) X, dY
// [B*H*W][cout] times *dscale (nullable = 1), X the conv's fp16 hi/lo input planes at scale x_scale.  dY is split into
// bufs.gp with an on-device power-of-two scale when the tensor cores read it (the 256-wide shapes) or when `split` asks
// for the planes anyway (the data-gradient conv reads them); *bufs.scale = *dscale times that scale.
int run_wgrad(dd_engine* e, int B, int H, int W, int cout, int cin, const float* dy, const float* dscale,
              const __half* x_hi, const __half* x_lo, float x_scale, float* dw, bool split, const WgradBufs& bufs,
              cudaStream_t st) {
  const size_t BP = static_cast<size_t>(B) * H * W;
  const size_t nw = static_cast<size_t>(cout) * cin * 9;
  const bool tc = dw != nullptr && wgrad_on_tc(cout, cin);
  int rc;
  if (split || tc) {
    const size_t n = BP * cout;
    dd::absmax_kernel<<<absmax_grid(n), 256, 0, st>>>(dy, static_cast<int>(n), bufs.amax);
    if ((rc = launched(e, "grad absmax"))) return rc;
    dd::grad_split_kernel<<<grid_of(n / 4), 256, 0, st>>>(dy, bufs.gp.hi, bufs.gp.lo, n / 4, bufs.amax, dscale,
                                                          bufs.scale, bufs.status);
    if ((rc = launched(e, "grad_split"))) return rc;
  }
  if (tc) {
    CUtensorMap ah, al, bh, bl;
    const CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_128B;
    if ((rc = make_nhwc_map(&ah, "wgrad operand", bufs.gp.hi, B, H, W, cout, 64, 64, 1, sw))) return rc;
    if ((rc = make_nhwc_map(&al, "wgrad operand", bufs.gp.lo, B, H, W, cout, 64, 64, 1, sw))) return rc;
    if ((rc = make_nhwc_map(&bh, "wgrad operand", x_hi, B, H, W, cin, 64, 64, 1, sw))) return rc;
    if ((rc = make_nhwc_map(&bl, "wgrad operand", x_lo, B, H, W, cin, 64, 64, 1, sw))) return rc;
    dd::WgmArgs a;
    a.cout = cout;
    a.cin = cin;
    a.B = B;
    a.H = H;
    a.W = W;
    a.xsegs = (W + 63) / 64;
    a.nseg = B * H * a.xsegs;
    a.segs = kWgmSegs;
    a.partial = bufs.partial;
    const int chunks = wgm_chunks(B, H, W);
    if (cout == 256 && cin == 256) {
      using Cf = dd::WgmCfg<128, 128>;
      dd::wgrad_wgmma_kernel<128, 128><<<dim3(chunks, 2 * 2 * 9), Cf::THREADS, Cf::SMEM_BYTES, st>>>(ah, al, bh, bl, a);
    } else if (cin == 64) {
      using Cf = dd::WgmCfg<128, 64>;
      dd::wgrad_wgmma_kernel<128, 64><<<dim3(chunks, 2 * 9), Cf::THREADS, Cf::SMEM_BYTES, st>>>(ah, al, bh, bl, a);
    } else {
      using Cf = dd::WgmCfg<64, 128>;
      dd::wgrad_wgmma_kernel<64, 128><<<dim3(chunks, 2 * 9), Cf::THREADS, Cf::SMEM_BYTES, st>>>(ah, al, bh, bl, a);
    }
    if ((rc = launched(e, "wgrad_wgmma"))) return rc;
    dd::wgrad_reduce_kernel<<<grid_of(nw), 256, 0, st>>>(bufs.partial, chunks, cout, cin, 1, 1.0 / x_scale, bufs.scale,
                                                         dw);
    return launched(e, "wgrad_reduce");
  }
  if (dw == nullptr) return DD_OK;
  const WgPlan pl = wgrad_plan(cout, cin, static_cast<long long>(BP));
  dd::WgradArgs a;
  a.dy = dy;
  a.x_hi = x_hi;
  a.x_lo = x_lo;
  a.x_inv_scale = 1.f / x_scale;
  a.cout = cout;
  a.cin = cin;
  a.B = B;
  a.H = H;
  a.W = W;
  a.chunk = pl.chunk;
  a.partial = bufs.partial;
  if (cout == 16) launch_wgrad<16, 64>(a, pl.chunks, st);
  else launch_wgrad<64, 16>(a, pl.chunks, st);
  if ((rc = launched(e, "wgrad"))) return rc;
  dd::wgrad_reduce_kernel<<<grid_of(nw), 256, 0, st>>>(bufs.partial, pl.chunks, cout, cin, 0, 1.0, dscale, dw);
  return launched(e, "wgrad_reduce");
}

// Backward of conv layer `layer` given dy [B][P][Cout] (times *dscale, nullable = 1) and the conv's input planes X (scale
// x_scale): dw [Cout][Cin][3][3] and db [Cout] (each nullable), and dx (nullable) = conv3x3(dy, W') on the forward's
// tensor-core kernel, left multiplied by bw.scales[slot].
int run_conv_bwd(dd_engine* e, int layer, const float* dy, const float* dscale, const __half* x_hi, const __half* x_lo,
                 float x_scale, float* dw, float* db, float* dx, int slot, cudaStream_t st) {
  const Geom g = geom_of(e->cfg);
  const int cout = kConvCout[layer], cin = kConvCin[layer];
  int rc;
  if (db != nullptr && (rc = run_colsum(e, cout, dy, dscale, g.B, g.P, e->bw.col_part, nullptr, db, st))) return rc;
  const WgradBufs bufs{e->bw.gp, e->bw.amax + slot, e->bw.scales + slot, e->status, e->bw.wg_part};
  if ((rc = run_wgrad(e, g.B, g.h, g.w, cout, cin, dy, dscale, x_hi, x_lo, x_scale, dw, dx != nullptr, bufs, st)))
    return rc;
  if (dx != nullptr &&
      (rc = run_conv(e, 6 + layer, e->bw.gp.hi, e->bw.gp.lo, 1.f, dd::EPI_F32, dx, nullptr, nullptr, nullptr, st)))
    return rc;
  return DD_OK;
}

// The forward again, keeping what the backward reads: pre-GN outputs, mean / rstd and every conv's input planes.
// Image b's time-embedding row is temb + b * temb_bstride.
int run_recompute(dd_engine* e, const float* temb, int temb_bstride, cudaStream_t st) {
  dd_engine::Bwd& b = e->bw;
  int rc;
  if ((rc = run_conv(e, 0, e->xs_hi, e->xs_lo, kXScale, dd::EPI_F32_STATS, b.y1, e->stats[0], nullptr, nullptr, st))) return rc;
  if ((rc = run_finalize(e, 0, 64, st))) return rc;
  if ((rc = run_apply<64, 0>(e, 0, nullptr, 0, b.a1.hi, b.a1.lo, st, b.y1))) return rc;
  if ((rc = run_conv(e, 1, b.a1.hi, b.a1.lo, kActScale, dd::EPI_F32_STATS, b.y2, e->stats[1], nullptr, nullptr, st))) return rc;
  if ((rc = run_finalize(e, 1, 256, st))) return rc;
  if (e->cfg.variant == DD_VARIANT_SWIN) {
    if ((rc = run_apply<256, 2>(e, 1, temb, temb_bstride, b.f0.hi, b.f0.lo, st, b.y2))) return rc;
    if ((rc = run_conv(e, 2, b.f0.hi, b.f0.lo, kActScale, dd::EPI_SPLIT, nullptr, nullptr, b.fa.hi, b.fa.lo, st))) return rc;
    if ((rc = run_conv(e, 3, b.fa.hi, b.fa.lo, kActScale, dd::EPI_SPLIT, nullptr, nullptr, b.fp.hi, b.fp.lo, st))) return rc;
  } else if ((rc = run_apply<256, 1>(e, 1, temb, temb_bstride, b.fp.hi, b.fp.lo, st, b.y2))) {
    return rc;
  }
  if ((rc = run_conv(e, 4, b.fp.hi, b.fp.lo, kActScale, dd::EPI_F32_STATS, b.y5, e->stats[2], nullptr, nullptr, st))) return rc;
  if ((rc = run_finalize(e, 2, 64, st))) return rc;
  if ((rc = run_apply<64, 0>(e, 2, nullptr, 0, b.a5.hi, b.a5.lo, st, b.y5))) return rc;
  if ((rc = run_conv(e, 5, b.a5.hi, b.a5.lo, kActScale, dd::EPI_F32_STATS, b.y6, e->stats[3], nullptr, nullptr, st))) return rc;
  return run_finalize(e, 3, 16, st);
}

// Reverse mode of one ScheduledCNNRefine call on the latent in x32 / xs planes and the condition map in the workspace,
// given d_eps (unscaled, NHWC) in bw.g[0].  Serves dd_denoiser_backward and every step of dd_denoise_backward.
//   P[i]        (each nullable; P[8] is never written) parameter gradients in dd_denoiser_backward's order
//   want_dtemb  per-image time-embedding gradients into bw.dtemb [B][256]; the dense table is the caller's
//   dcond_sink  called with (d_cond NHWC [B][cond_h][cond_w][256], its scale or nullptr) at the point where d_cond is
//               complete (for Res that buffer is reused right after); nullptr: d_cond is not needed
//   want_dnoisy leave d_noisy times bw.scales[5] in bw.g[0]
template <typename Sink>
int run_denoiser_bwd(dd_engine* h, const float* temb, int temb_bstride, float* const* P, bool want_dtemb,
                     const Sink* dcond_sink, bool want_dnoisy, cudaStream_t st) {
  const Geom g = geom_of(h->cfg);
  const bool swin = h->cfg.variant == DD_VARIANT_SWIN;
  dd_engine::Bwd& bw = h->bw;
  const int PC = h->cfg.cond_h * h->cfg.cond_w;
  int rc;
  CUDA_TRY(cudaMemsetAsync(bw.amax, 0, kBwdSlots * 4, st));
  if ((rc = run_recompute(h, temb, temb_bstride, st))) return rc;
  float *g0 = bw.g[0], *g1 = bw.g[1];
  const float* sc = bw.scales;
  // eps = relu(GN(y6)) -> pred.3
  if ((rc = run_gn_bwd<16>(h, 3, g0, nullptr, bw.y6, P[15], P[16], g1, st))) return rc;
  if ((rc = run_conv_bwd(h, 5, g1, nullptr, bw.a5.hi, bw.a5.lo, kActScale, P[13], P[14], g0, 0, st))) return rc;
  // pred.1 -> pred.0
  if ((rc = run_gn_bwd<64>(h, 2, g0, sc + 0, bw.y5, P[11], P[12], g1, st))) return rc;
  if ((rc = run_conv_bwd(h, 4, g1, nullptr, bw.fp.hi, bw.fp.lo, kActScale, P[9], P[10], g0, 1, st))) return rc;
  // g0 = dF (times scales[1]).  Swin: F = convB(convA(up(cond + temb) + ne)); Res: F = cond + temb + ne
  const float* dne_scale = sc + 1;
  if (swin) {
    if ((rc = run_conv_bwd(h, 3, g0, sc + 1, bw.fa.hi, bw.fa.lo, kActScale, P[19], P[20], g1, 2, st))) return rc;
    if ((rc = run_conv_bwd(h, 2, g1, sc + 2, bw.f0.hi, bw.f0.lo, kActScale, P[17], P[18], g0, 3, st))) return rc;
    dne_scale = sc + 3;
    if (dcond_sink || want_dtemb) {
      const float ry = g.h > 1 ? static_cast<float>(h->cfg.cond_h - 1) / static_cast<float>(g.h - 1) : 0.f;
      const float rx = g.w > 1 ? static_cast<float>(h->cfg.cond_w - 1) / static_cast<float>(g.w - 1) : 0.f;
      dd::up_adjoint_kernel<<<dim3(h->cfg.cond_w, h->cfg.cond_h, g.B), 256, 0, st>>>(g0, dne_scale, g.h, g.w, h->cfg.cond_h,
                                                                                      h->cfg.cond_w, ry, rx, bw.dcond);
      if ((rc = launched(h, "up_adjoint"))) return rc;
      if (want_dtemb && (rc = run_colsum(h, 256, bw.dcond, nullptr, g.B, PC, bw.col_part, bw.dtemb, nullptr, st)))
        return rc;
      if (dcond_sink && (rc = (*dcond_sink)(bw.dcond, nullptr))) return rc;
    }
  } else {
    if (want_dtemb && (rc = run_colsum(h, 256, g0, dne_scale, g.B, g.P, bw.col_part, bw.dtemb, nullptr, st))) return rc;
    if (dcond_sink && (rc = (*dcond_sink)(g0, dne_scale))) return rc;
  }
  // ne = relu(GN(y2)) -> noise_embedding.3 -> relu(GN(y1)) -> noise_embedding.0
  if ((rc = run_gn_bwd<256>(h, 1, g0, dne_scale, bw.y2, P[6], P[7], g1, st))) return rc;
  if ((rc = run_conv_bwd(h, 1, g1, nullptr, bw.a1.hi, bw.a1.lo, kActScale, P[4], P[5], g0, 4, st))) return rc;
  if ((rc = run_gn_bwd<64>(h, 0, g0, sc + 4, bw.y1, P[2], P[3], g1, st))) return rc;
  return run_conv_bwd(h, 0, g1, nullptr, h->xs_hi, h->xs_lo, kXScale, P[0], P[1], want_dnoisy ? g0 : nullptr, 5, st);
}

// Reverse mode of run_decoder for the latent in x32: d_depth [B][2h][2w] -> dx (NHWC [B][P][16], nullable) and the six
// decoder gradients dp[0..5] (array and entries nullable), in DECODER_KEYS order without the running statistics.
int run_decode_bwd(dd_engine* e, const float* d_depth, float* dx, float* const* dp, cudaStream_t st) {
  const Geom g = geom_of(e->cfg);
  dd_engine::LoopBwd& l = e->lp;
  const size_t nout = static_cast<size_t>(g.B) * g.P * 4;
  const bool train = e->codec_mode == DD_CODEC_TRAIN;
  int rc;
  // DD_CODEC_TRAIN: the same statistics in the same order as the forward's, so the fold and the ReLU mask are its own
  if (train && (rc = run_dec_batch_stats(e, nullptr, st))) return rc;
  if ((rc = run_decoder(e, l.z, l.r, st))) return rc;  // the forward's logit z; its depth lands in r (scratch until below)
  dd::dec_dz_kernel<<<grid_of(nout), 256, 0, st>>>(l.z, d_depth, nout, 1e-6f);
  if ((rc = launched(e, "dec_dz"))) return rc;
  dd::DecBwdArgs a;
  a.x = e->x32;
  a.wt = train ? e->ct.dec_wt : e->dec_wt;
  a.bt = train ? e->ct.dec_bt : e->dec_bt;
  a.wu = e->dec_wu;
  a.bu = train ? e->ct.zero16 : e->dec_bu;  // DD_CODEC_TRAIN: xhat from the bias-free conv, as its statistics
  a.bn = train ? e->ct.dec_bn : e->dec_bn;
  a.wc = e->dec_wc;
  a.dz = l.z;
  a.r = l.r;
  a.du = l.du;
  a.part_act = l.part_act;
  a.part_wc = l.part_wc;
  a.part_wt = l.part_wt;
  a.dx = dx;
  a.B = g.B;
  a.h = g.h;
  a.w = g.w;
  dd::dec_bwd_act_kernel<<<dec_act_blocks(g), 256, 0, st>>>(a);
  if ((rc = launched(e, "dec_bwd_act"))) return rc;
  if (train) {  // du through the batch mean and variance (across ranks: the union batch's sums and count)
    BnTotals t;
    if ((rc = bn_totals(e, l.part_act, dec_act_blocks(g), dd::DEC_ACT_N, 32, nout, e->ct.sums, 33, st, &t))) return rc;
    dd::dec_bwd_bn_kernel<<<dec_act_blocks(g), 256, 0, st>>>(a, t.sum, t.cnt, e->ct.part_db);
    if ((rc = launched(e, "dec_bwd_bn"))) return rc;
  }
  if (dx != nullptr) {
    dd::dec_bwd_dx_kernel<<<static_cast<int>((static_cast<size_t>(g.B) * g.P + 255) / 256), 256, 0, st>>>(a);
    if ((rc = launched(e, "dec_bwd_dx"))) return rc;
  }
  bool any = false;
  for (int i = 0; i < 6 && dp != nullptr; ++i) any |= dp[i] != nullptr;
  if (!any) return DD_OK;
  dd::dec_bwd_wc_kernel<<<dec_wc_blocks(g), 160, 0, st>>>(a);
  if ((rc = launched(e, "dec_bwd_wc"))) return rc;
  dd::dec_bwd_wt_kernel<<<dec_wt_blocks(g), 256, 0, st>>>(a);
  if ((rc = launched(e, "dec_bwd_wt"))) return rc;
  dd::DecFinishArgs f;
  f.part_act = l.part_act;
  f.part_wc = l.part_wc;
  f.part_wt = l.part_wt;
  f.nb_act = dec_act_blocks(g);
  f.nb_wc = dec_wc_blocks(g);
  f.nb_wt = dec_wt_blocks(g);
  f.bn = a.bn;
  f.part_db = train ? e->ct.part_db : nullptr;
  for (int i = 0; i < 6; ++i) f.out[i] = dp[i];
  dd::dec_bwd_finish_kernel<<<(dd::DEC_GRAD_N + 255) / 256, 256, 0, st>>>(f);
  return launched(e, "dec_bwd_finish");
}

constexpr size_t kDecGradNumel[6] = {16 * 16 * 4 * 4, 16, 16, 16, 16 * 9, 1};

// Checks of an entry that recomputes one denoiser call on the backward's region (dd_denoiser_backward,
// dd_denoiser_relu_inputs), after its own null-pointer checks.
int check_operator_bwd_call(const dd_engine* h, const char* entry) {
  if (!has_backward(h->cfg))
    return fail(DD_ERR_INVALID, std::string(entry) + " needs an engine created with DD_FLAG_BACKWARD (or DD_FLAG_LOOP_BACKWARD)");
  if (!h->weights_ready) return fail(DD_ERR_INVALID, "dd_finalize_weights has not been called");
  const Geom g = geom_of(h->cfg);
  if (static_cast<size_t>(g.B) * g.P * 256 > static_cast<size_t>(INT32_MAX))
    return fail(DD_ERR_UNSUPPORTED, "batch x latent too large for one backward call");
  return DD_OK;
}

// One denoiser call's inputs as run_step / run_recompute read them: image b's time-embedding row t_host[b] in
// temb_sel (every row checked first), cond and noisy as NHWC, the latent's fp16 split planes.
int stage_operator_inputs(dd_engine* h, const float* cond, const float* noisy, const int64_t* t_host, cudaStream_t st) {
  const Geom g = geom_of(h->cfg);
  int rc;
  for (int b = 0; b < g.B; ++b)
    if (t_host[b] < 0 || t_host[b] >= DD_TIME_ROWS) return fail(DD_ERR_INVALID, "timestep outside time_embedding");
  for (int b = 0; b < g.B; ++b)
    CUDA_TRY(cudaMemcpyAsync(h->temb_sel + b * 256, h->temb + t_host[b] * 256, 1024, cudaMemcpyDeviceToDevice, st));
  if ((rc = transpose_in(cond, h->cond, g.B, 256, h->cfg.cond_h * h->cfg.cond_w, st))) return rc;
  if ((rc = transpose_in(noisy, h->x32, g.B, 16, g.P, st))) return rc;
  return split_planes(h, h->x32, h->xs_hi, h->xs_lo, static_cast<size_t>(g.B) * g.P * 16, kXScale, st);
}

// Milliseconds per call of `body` (which returns a DD_* code) over `iters` calls on st, after `warmup` untimed calls.
template <typename F>
int time_per_call(cudaStream_t st, int warmup, int iters, float* ms_out, F&& body) {
  int rc;
  for (int i = 0; i < warmup; ++i)
    if ((rc = body())) return rc;
  struct Events {  // destroyed on every return
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    ~Events() {
      if (e0) cudaEventDestroy(e0);
      if (e1) cudaEventDestroy(e1);
    }
  } ev;
  CUDA_TRY(cudaEventCreate(&ev.e0));
  CUDA_TRY(cudaEventCreate(&ev.e1));
  CUDA_TRY(cudaEventRecord(ev.e0, st));
  for (int i = 0; i < iters; ++i)
    if ((rc = body())) return rc;
  CUDA_TRY(cudaEventRecord(ev.e1, st));
  CUDA_TRY(cudaEventSynchronize(ev.e1));
  float ms = 0.f;
  CUDA_TRY(cudaEventElapsedTime(&ms, ev.e0, ev.e1));
  *ms_out = ms / iters;
  return DD_OK;
}

// The buffers of one standalone call (the layer entries, dd_bench_gemm), freed when it returns, and the engine's
// status word pointed at the call's own word meanwhile (the launch helpers report to e->status, a workspace word).
struct StandaloneCall {
  dd_engine* e;
  int* saved;
  std::vector<void*> owned;
  int* status = nullptr;
  explicit StandaloneCall(dd_engine* eng) : e(eng), saved(eng->status) {}
  ~StandaloneCall() {
    e->status = saved;
    for (void* p : owned) cudaFree(p);
  }
  int begin(cudaStream_t st) {
    int rc;
    if ((rc = dev_alloc(owned, reinterpret_cast<void**>(&status), 64))) return rc;
    CUDA_TRY(cudaMemsetAsync(status, 0, 64, st));
    e->status = status;
    return DD_OK;
  }
  template <typename T>
  int alloc(T** p, size_t n) { return dev_alloc(owned, reinterpret_cast<void**>(p), n * sizeof(T)); }
  int finish(cudaStream_t st, const char* what) { return check_status_word(status, st, what); }
};

// Frees what dd_create and dd_finalize_weights allocated; also takes an engine whose dd_create failed part-way.
void release(dd_engine* e) {
  cudaSetDevice(e->cfg.device);
  drop_graphs(e);
  for (void* p : e->owned) cudaFree(p);
  free_bn_sync(e);
  if (e->status_host) cudaFreeHost(e->status_host);
  if (e->stage) cudaFreeHost(e->stage);
  if (e->pack_done) cudaEventDestroy(e->pack_done);
  if (e->cap_stream) cudaStreamDestroy(e->cap_stream);
  delete e;
}

// The standalone conv's workspace: the status word (+ scratch), x as NHWC fp32 and its split planes, y as NHWC fp32,
// the packed weights.  With base == nullptr only the size is computed, as carve() does.
struct Conv3x3Ws {
  int* status;
  float *xn, *yn, *wsimt;
  Planes x, w;
};
size_t conv3x3_layout(void* base, int batch, int cin, int cout, int height, int width, Conv3x3Ws& v) {
  const size_t BP = static_cast<size_t>(batch) * height * width;
  const size_t nw = static_cast<size_t>(cin) * cout * 9;
  Carver c{reinterpret_cast<uint8_t*>(base)};
  v.status = c.take<int>(16);
  v.xn = c.take<float>(BP * cin);
  v.x.hi = c.take<__half>(BP * cin);
  v.x.lo = c.take<__half>(BP * cin);
  v.yn = c.take<float>(BP * cout);
  v.w.hi = c.take<__half>(nw);
  v.w.lo = c.take<__half>(nw);
  v.wsimt = c.take<float>(nw);
  return align_up(c.off, 1024);
}

// The standalone weight gradient's workspace: the status word (+ scratch), x and dy as NHWC fp32 and their split
// planes, the fp64 weight-gradient partials, the bias-gradient partials.  base == nullptr: the size only.
struct WgradWs {
  int* status;
  float *xn, *dyn, *col_part;
  Planes x, dy;
  double* partial;
};
size_t wgrad_layout(void* base, int batch, int cin, int cout, int height, int width, WgradWs& v) {
  const size_t BP = static_cast<size_t>(batch) * height * width;
  Carver c{reinterpret_cast<uint8_t*>(base)};
  v.status = c.take<int>(16);
  v.xn = c.take<float>(BP * cin);
  v.x.hi = c.take<__half>(BP * cin);
  v.x.lo = c.take<__half>(BP * cin);
  v.dyn = c.take<float>(BP * cout);
  v.dy.hi = c.take<__half>(BP * cout);
  v.dy.lo = c.take<__half>(BP * cout);
  v.partial = c.take<double>(wgrad_partial_elems(cout, cin, batch, height, width));
  v.col_part = c.take<float>(static_cast<size_t>(batch) * bwd_chunks(height * width) * cout);
  return align_up(c.off, 1024);
}

}  // namespace

extern "C" {

int dd_abi_version(void) { return DD_ABI_VERSION; }
const char* dd_last_error(void) { return g_err.c_str(); }

int dd_create(const dd_config* cfg, dd_handle* out) {
  if (!cfg || !out) return fail(DD_ERR_INVALID, "null argument");
  if (cfg->abi_version != DD_ABI_VERSION) return fail(DD_ERR_INVALID, "ABI version mismatch");
  if (cfg->variant != DD_VARIANT_RES && cfg->variant != DD_VARIANT_SWIN) return fail(DD_ERR_INVALID, "bad variant");
  if (cfg->batch < 1 || cfg->latent_h < 1 || cfg->latent_w < 1 || cfg->num_inference_steps < 1)
    return fail(DD_ERR_INVALID, "bad geometry");
  if (cfg->variant == DD_VARIANT_RES && (cfg->cond_h != cfg->latent_h || cfg->cond_w != cfg->latent_w))
    return fail(DD_ERR_INVALID, "Res variant needs the condition map at latent resolution");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail(DD_ERR_UNSUPPORTED, "no CUDA device: libddengine has no CPU path");
  if (cfg->device < 0 || cfg->device >= ndev) return fail(DD_ERR_INVALID, "bad device ordinal");
  cudaDeviceProp prop;
  CUDA_TRY(cudaGetDeviceProperties(&prop, cfg->device));
  if (prop.major != 9 || prop.minor != 0)
    return fail(DD_ERR_UNSUPPORTED, "libddengine is built for sm_90a (Hopper H100) only");
  CUDA_TRY(cudaSetDevice(cfg->device));
  int rc;
  if ((rc = load_driver())) return rc;
  dd_engine* e = new dd_engine();
  e->cfg = *cfg;
  e->sm_count = prop.multiProcessorCount;
  if (cudaMallocHost(&e->status_host, 64) != cudaSuccess ||
      cudaMallocHost(&e->stage, sizeof(PackStage)) != cudaSuccess ||
      cudaEventCreateWithFlags(&e->pack_done, cudaEventDisableTiming) != cudaSuccess ||
      cudaStreamCreateWithFlags(&e->cap_stream, cudaStreamNonBlocking) != cudaSuccess ||
      configure_all_kernels() != cudaSuccess) {
    std::string msg = std::string("engine setup failed: ") + cudaGetErrorString(cudaGetLastError());
    release(e);
    return fail(DD_ERR_CUDA, msg);
  }
  *out = e;
  return DD_OK;
}

int dd_destroy(dd_handle h) {
  if (h) release(h);
  return DD_OK;
}

static const char* kKeys[] = {
    "model.noise_embedding.0.weight", "model.noise_embedding.0.bias", "model.noise_embedding.1.weight",
    "model.noise_embedding.1.bias", "model.noise_embedding.3.weight", "model.noise_embedding.3.bias",
    "model.noise_embedding.4.weight", "model.noise_embedding.4.bias", "model.upsample_fuse.convA.conv.weight",
    "model.upsample_fuse.convA.conv.bias", "model.upsample_fuse.convB.conv.weight",
    "model.upsample_fuse.convB.conv.bias", "model.time_embedding.weight", "model.pred.0.weight", "model.pred.0.bias",
    "model.pred.1.weight", "model.pred.1.bias", "model.pred.3.weight", "model.pred.3.bias", "model.pred.4.weight",
    "model.pred.4.bias", "depth_transform.conv_inv_transform.0.weight", "depth_transform.conv_inv_transform.0.bias",
    "depth_transform.conv_inv_transform.1.weight", "depth_transform.conv_inv_transform.1.bias",
    "depth_transform.conv_inv_transform.1.running_mean", "depth_transform.conv_inv_transform.1.running_var",
    "depth_transform.conv_inv_transform.3.0.weight", "depth_transform.conv_inv_transform.3.0.bias"};

int dd_set_weight(dd_handle h, const char* name, const float* dev_ptr, const int64_t* shape, int32_t ndim) {
  if (!h || !name || !dev_ptr || ndim < 0 || ndim > 4) return fail(DD_ERR_INVALID, "bad argument");
  bool known = strncmp(name, "hahineck.", 9) == 0 || strncmp(name, "conv_lateral.", 13) == 0 ||
               strncmp(name, "conv_up.", 8) == 0 ||  // step-invariant producers (optional, dd_enable_producers)
               strncmp(name, "backbone.", 9) == 0 ||  // native backbone (optional, dd_enable_backbone)
               strncmp(name, "depth_transform.conv_transform.", 31) == 0;  // encoder t() (optional, dd_encode)
  for (const char* k : kKeys) known |= (strcmp(k, name) == 0);
  if (!known) return fail(DD_ERR_INVALID, std::string("unknown weight key: ") + name);
  Raw r;
  r.ptr = dev_ptr;
  r.shape.assign(shape, shape + ndim);
  h->raw[name] = r;
  h->weights_ready = false;
  return DD_OK;
}

int dd_finalize_weights(dd_handle h, void* cuda_stream) {
  if (!h) return fail(DD_ERR_INVALID, "null handle");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  CUDA_TRY(cudaSetDevice(h->cfg.device));
  const bool swin = h->cfg.variant == DD_VARIANT_SWIN;
  std::string missing;
  for (const char* k : kKeys) {
    if (!swin && strstr(k, "upsample_fuse")) continue;
    if (!find(h, k)) missing += std::string(missing.empty() ? "" : ", ") + k;
  }
  if (!missing.empty()) return fail(DD_ERR_INVALID, "missing weights: " + missing);
  auto expect = [&](const char* k, std::vector<int64_t> s) { return find(h, k)->shape == s; };
  if (!expect("model.noise_embedding.0.weight", {64, 16, 3, 3}) || !expect("model.noise_embedding.3.weight", {256, 64, 3, 3}) ||
      !expect("model.pred.0.weight", {64, 256, 3, 3}) || !expect("model.pred.3.weight", {16, 64, 3, 3}) ||
      !expect("model.time_embedding.weight", {DD_TIME_ROWS, 256}) ||
      !expect("depth_transform.conv_inv_transform.0.weight", {16, 16, 4, 4}) ||
      !expect("depth_transform.conv_inv_transform.3.0.weight", {1, 16, 3, 3}) ||
      (swin && (!expect("model.upsample_fuse.convA.conv.weight", {256, 256, 3, 3}) ||
                !expect("model.upsample_fuse.convB.conv.weight", {256, 256, 3, 3}))))
    return fail(DD_ERR_INVALID, "weight shape mismatch with the reference architecture");
  const bool encoder = find(h, kEncPrefix + "0.0.weight") != nullptr;
  if (encoder) {
    const Raw *w1 = find(h, kEncPrefix + "0.0.weight"), *w2 = find(h, kEncPrefix + "1.0.weight");
    if (!w2 || w1->shape != std::vector<int64_t>{16, 1, 3, 3} || w2->shape != std::vector<int64_t>{16, 16, 3, 3})
      return fail(DD_ERR_INVALID, "encoder weights missing / wrong shape");
    for (const CodecKey& k : kEncKeys)
      if (!find(h, kEncPrefix + k.leaf)) return fail(DD_ERR_INVALID, "missing weights: " + kEncPrefix + k.leaf);
  }
  // drop any previous pack
  drop_graphs(h);
  h->packed = false;
  for (void* p : h->owned) cudaFree(p);
  h->owned.clear();
  h->pt = dd_engine::ProdTrain();  // pack_gen appends the training-mode records, the backbone's before the producers'
  int rc;
  if ((rc = alloc_pack(h, encoder, st))) return rc;
  if ((rc = fill_pack(h, st))) return rc;
  float* scratch = h->amax;
  h->rn.ready = false;
  if (h->rn.enabled)
    if ((rc = pack_resnet(h, st, scratch))) return rc;
  h->mp.ready = false;
  if (h->mp.enabled)
    if ((rc = pack_mpvit(h, st, scratch))) return rc;
  h->prod.ready = false;
  if (h->prod.enabled)
    if ((rc = pack_producers(h, st, scratch))) return rc;
  h->bb.ready = false;
  if (h->bb.enabled)
    if ((rc = pack_backbone(h, st, scratch))) return rc;
  if ((rc = pack_prod_train(h, st))) return rc;
  h->drop.on = false;  // a new buffer: dd_set_drop_path fills it
  if (h->drop.blocks > 0 && (h->mp.enabled || h->bb.enabled) &&
      (rc = dev_array(h, &h->drop.scales, static_cast<size_t>(h->drop.blocks) * 2 * h->cfg.batch)))
    return rc;
  // the registered pointers were borrowed for this call only (include/dd_engine.h): wait for the kernels that read them
  // and forget them, so a later finalize cannot read memory the caller has freed in the meantime
  CUDA_TRY(cudaStreamSynchronize(st));
  h->raw.clear();
  h->weights_ready = h->packed = true;
  return DD_OK;
}

int dd_update_weights(dd_handle h, void* cuda_stream) {
  if (!h) return fail(DD_ERR_INVALID, "null handle");
  int rc = DD_OK;
  if (!h->packed) {
    rc = fail(DD_ERR_INVALID, "dd_update_weights needs a completed dd_finalize_weights");
  } else if (!h->raw.empty() && (rc = check_update(h)) == DD_OK) {
    if (cudaSetDevice(h->cfg.device) != cudaSuccess) rc = fail(DD_ERR_CUDA, "cudaSetDevice failed");
    else rc = fill_pack(h, static_cast<cudaStream_t>(cuda_stream));
    if (rc != DD_OK) h->packed = false;  // the pack is partly written: only dd_finalize_weights restores it
  }
  h->raw.clear();
  h->weights_ready = h->packed;
  return rc;
}

int64_t dd_graph_capture_count(dd_handle h) { return h ? h->graph_captures : 0; }

int dd_set_schedule(dd_handle h, const int64_t* timesteps, const double* c_x, const double* c_eps, int32_t n) {
  if (!h || !timesteps || !c_x || !c_eps) return fail(DD_ERR_INVALID, "null argument");
  if (n != h->cfg.num_inference_steps) return fail(DD_ERR_INVALID, "schedule length != num_inference_steps");
  h->ts.assign(timesteps, timesteps + n);
  h->cx.resize(n);
  h->ce.resize(n);
  for (int i = 0; i < n; ++i) {
    if (timesteps[i] < 0 || timesteps[i] >= DD_TIME_ROWS) return fail(DD_ERR_INVALID, "timestep outside time_embedding");
    h->cx[i] = static_cast<float>(c_x[i]);
    h->ce[i] = static_cast<float>(c_eps[i]);
  }
  drop_graphs(h);
  return DD_OK;
}

size_t dd_workspace_bytes(dd_handle h) { return h ? carve(h, nullptr) : 0; }

// dd_denoise_decode and dd_denoise_decode_steps: the T-step loop (+ a decode after every step when depth_steps_out
// is given: the *Vis heads' `pred_inter`, reference ..._swin_addHAHI_vis.py:130-149,289-304), then the final decode.
static int denoise_impl(dd_handle h, const float* cond, const float* noise, float* latent_out, float* logit_out,
                        float* depth_out, float* depth_steps_out, void* workspace, size_t workspace_bytes,
                        void* cuda_stream) {
  if (!h || !noise || (!depth_out && !depth_steps_out)) return fail(DD_ERR_INVALID, "null argument");
  if (!cond && !h->cond_ready) return fail(DD_ERR_INVALID, "cond is NULL but dd_build_condition has not run");
  if (!h->weights_ready) return fail(DD_ERR_INVALID, "dd_finalize_weights has not been called");
  if (static_cast<int>(h->ts.size()) != h->cfg.num_inference_steps) return fail(DD_ERR_INVALID, "dd_set_schedule has not been called");
  if (depth_steps_out && !(h->cfg.flags & DD_FLAG_STEP_DECODE))
    return fail(DD_ERR_INVALID, "dd_denoise_decode_steps needs an engine created with DD_FLAG_STEP_DECODE");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  int rc;
  if ((rc = enter_workspace(h, workspace, workspace_bytes))) return rc;
  const Geom g = geom_of(h->cfg);
  if (cond) {
    if ((rc = start_forward(h, st))) return rc;
    if ((rc = transpose_in(cond, h->cond, g.B, 256, h->cfg.cond_h * h->cfg.cond_w, st))) return rc;
    h->launches += 1;
  }  // else: dd_build_condition left the NHWC condition map (and the launch / status counters) in place
  h->cond_ready = false;
  if ((rc = transpose_in(noise, h->x32, g.B, 16, g.P, st))) return rc;
  if ((rc = split_planes(h, h->x32, h->xs_hi, h->xs_lo, static_cast<size_t>(g.B) * g.P * 16, kXScale, st))) return rc;
  h->launches += 2;
  const int T = h->cfg.num_inference_steps;
  const size_t map_elems = static_cast<size_t>(g.B) * g.P * 4;  // one decoded batch [B][2h][2w]
  const bool steps = depth_steps_out != nullptr;
  const bool train = h->codec_mode == DD_CODEC_TRAIN;  // batch statistics before every decode, one record each
  if (steps && train && h->sync.fn)
    return fail(DD_ERR_UNSUPPORTED, "dd_denoise_decode_steps in DD_CODEC_TRAIN does not run with a BatchNorm all-gather "
                                    "installed (dd_set_bn_allgather)");
  h->ct.nrec = 0;
  auto loop = [&](cudaStream_t s) -> int {
    for (int i = 0; i < T; ++i) {
      int r = run_step(h, h->temb + h->ts[i] * 256, 0, h->cx[i], h->ce[i], nullptr, s);
      if (r == DD_OK && steps && train) r = run_dec_batch_stats(h, h->ct.rec + i * 32, s);
      if (r == DD_OK && steps) r = run_decoder(h, nullptr, h->inter + i * map_elems, s);
      if (r != DD_OK) return r;
    }
    return DD_OK;
  };
  if (h->cfg.flags & DD_FLAG_CUDA_GRAPH) {
    const int which = steps ? (train ? dd_engine::G_LOOP_STEPS_TRAIN : dd_engine::G_LOOP_STEPS) : dd_engine::G_LOOP;
    if ((rc = graph_run(h, which, st, loop))) return rc;
  } else if ((rc = loop(st))) {
    return rc;
  }
  if (steps) {
    CUDA_TRY(cudaMemcpyAsync(depth_steps_out, h->inter, static_cast<size_t>(T) * map_elems * 4, cudaMemcpyDeviceToDevice, st));
    if (depth_out)
      CUDA_TRY(cudaMemcpyAsync(depth_out, h->inter + static_cast<size_t>(T - 1) * map_elems, map_elems * 4,
                               cudaMemcpyDeviceToDevice, st));
    // the logits of the final map only: one more (cheap) decode, its depth lands in the scratch slot; in
    // DD_CODEC_TRAIN it reuses the last step's batch fold and records nothing
    if (logit_out)
      if ((rc = run_decoder(h, logit_out, h->inter + static_cast<size_t>(T - 1) * map_elems, st))) return rc;
    h->ct.nrec = train ? T : 0;
  } else {
    if (train && (rc = run_dec_batch_stats(h, h->ct.rec, st))) return rc;
    if ((rc = run_decoder(h, logit_out, depth_out, st))) return rc;
    h->ct.nrec = train ? 1 : 0;
  }
  if (latent_out) {
    if ((rc = transpose_out(h->x32, latent_out, g.B, 16, g.P, st))) return rc;
    h->launches++;
  }
  return finish_forward(h, st);
}

int dd_denoise_decode(dd_handle h, const float* cond, const float* noise, float* latent_out, float* logit_out,
                      float* depth_out, void* workspace, size_t workspace_bytes, void* cuda_stream) {
  if (!depth_out) return fail(DD_ERR_INVALID, "null argument");
  return denoise_impl(h, cond, noise, latent_out, logit_out, depth_out, nullptr, workspace, workspace_bytes, cuda_stream);
}

int dd_denoise_decode_steps(dd_handle h, const float* cond, const float* noise, float* latent_out, float* logit_out,
                            float* depth_steps_out, void* workspace, size_t workspace_bytes, void* cuda_stream) {
  if (!depth_steps_out) return fail(DD_ERR_INVALID, "null argument");
  return denoise_impl(h, cond, noise, latent_out, logit_out, nullptr, depth_steps_out, workspace, workspace_bytes, cuda_stream);
}

int dd_denoiser_forward(dd_handle h, const float* cond, const float* noisy, const int64_t* t_host, float* eps_out,
                        void* workspace, size_t workspace_bytes, void* cuda_stream) {
  if (!h || !cond || !noisy || !t_host || !eps_out) return fail(DD_ERR_INVALID, "null argument");
  if (!h->weights_ready) return fail(DD_ERR_INVALID, "dd_finalize_weights has not been called");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  int rc;
  if ((rc = enter_workspace(h, workspace, workspace_bytes))) return rc;
  if ((rc = start_forward(h, st))) return rc;
  if ((rc = stage_operator_inputs(h, cond, noisy, t_host, st))) return rc;
  const Geom g = geom_of(h->cfg);
  // eps (NHWC) lands in the tail of Y's storage: Y holds y6 in its first B*P*16 floats at that point
  float* eps_nhwc = h->Y + static_cast<size_t>(g.B) * g.P * 16;
  if ((rc = run_step(h, h->temb_sel, 256, 0.f, 0.f, eps_nhwc, st))) return rc;
  if ((rc = transpose_out(eps_nhwc, eps_out, g.B, 16, g.P, st))) return rc;
  return finish_forward(h, st);
}

int dd_denoiser_backward(dd_handle h, const float* cond, const float* noisy, const int64_t* t_host, const float* d_eps,
                         float* d_cond_out, float* d_noisy_out, float* const* d_params, void* workspace,
                         size_t workspace_bytes, void* cuda_stream) {
  if (!h || !cond || !noisy || !t_host || !d_eps) return fail(DD_ERR_INVALID, "null argument");
  int rc;
  if ((rc = check_operator_bwd_call(h, "dd_denoiser_backward"))) return rc;
  const Geom g = geom_of(h->cfg);
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  if ((rc = enter_workspace(h, workspace, workspace_bytes))) return rc;
  const bool swin = h->cfg.variant == DD_VARIANT_SWIN;
  const int npar = swin ? 21 : 17;
  float* P[21] = {};
  if (d_params)
    for (int i = 0; i < npar; ++i) P[i] = d_params[i];
  dd_engine::Bwd& bw = h->bw;
  const size_t BP = static_cast<size_t>(g.B) * g.P;
  const int PC = h->cfg.cond_h * h->cfg.cond_w;
  if ((rc = start_forward(h, st))) return rc;
  if ((rc = stage_operator_inputs(h, cond, noisy, t_host, st))) return rc;
  if ((rc = transpose_in(d_eps, bw.g[0], g.B, 16, g.P, st))) return rc;
  auto sink = [&](const float* dc, const float* scale) -> int {
    int r;
    if ((r = transpose_out(dc, d_cond_out, g.B, 256, PC, st))) return r;
    if (scale == nullptr) return DD_OK;
    dd::unscale_kernel<<<grid_of(static_cast<size_t>(g.B) * PC * 256), 256, 0, st>>>(d_cond_out,
                                                                                     static_cast<size_t>(g.B) * PC * 256, scale);
    return launched(h, "unscale");
  };
  if ((rc = run_denoiser_bwd(h, h->temb_sel, 256, P, P[8] != nullptr, d_cond_out ? &sink : nullptr, d_noisy_out != nullptr,
                             st)))
    return rc;
  if (P[8]) {  // dense [1280][256]: row t_b collects image b's d_temb, rows shared by several images sum in image order
    CUDA_TRY(cudaMemsetAsync(P[8], 0, static_cast<size_t>(DD_TIME_ROWS) * 256 * 4, st));
    for (int b = 0; b < g.B; ++b) {
      dd::temb_row_add_kernel<<<1, 256, 0, st>>>(P[8] + t_host[b] * 256, bw.dtemb + b * 256);
      if ((rc = launched(h, "temb_row_add"))) return rc;
    }
  }
  if (d_noisy_out) {
    if ((rc = transpose_out(bw.g[0], d_noisy_out, g.B, 16, g.P, st))) return rc;
    dd::unscale_kernel<<<grid_of(BP * 16), 256, 0, st>>>(d_noisy_out, BP * 16, bw.scales + 5);
    if ((rc = launched(h, "unscale"))) return rc;
  }
  return finish_forward(h, st);
}

int dd_denoiser_relu_inputs(dd_handle h, const float* cond, const float* noisy, const int64_t* t_host,
                            float* const* z_out, void* workspace, size_t workspace_bytes, void* cuda_stream) {
  if (!h || !cond || !noisy || !t_host || !z_out) return fail(DD_ERR_INVALID, "null argument");
  int rc;
  if ((rc = check_operator_bwd_call(h, "dd_denoiser_relu_inputs"))) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  if ((rc = enter_workspace(h, workspace, workspace_bytes))) return rc;
  const dd_engine::Bwd& bw = h->bw;
  if ((rc = start_forward(h, st))) return rc;
  if ((rc = stage_operator_inputs(h, cond, noisy, t_host, st))) return rc;
  if ((rc = run_recompute(h, h->temb_sel, 256, st))) return rc;
  if (z_out[0] && (rc = run_gn_pre_relu<64>(h, 0, bw.y1, z_out[0], st))) return rc;
  if (z_out[1] && (rc = run_gn_pre_relu<256>(h, 1, bw.y2, z_out[1], st))) return rc;
  if (z_out[2] && (rc = run_gn_pre_relu<64>(h, 2, bw.y5, z_out[2], st))) return rc;
  if (z_out[3] && (rc = run_gn_pre_relu<16>(h, 3, bw.y6, z_out[3], st))) return rc;
  return finish_forward(h, st);
}

int dd_denoise_backward(dd_handle h, const float* cond, const float* noise, const float* d_depth, const float* d_latent,
                        float* d_cond_out, float* d_noise_out, float* const* d_params, float* const* d_dec_params,
                        float* latents_out, void* workspace, size_t workspace_bytes, void* cuda_stream) {
  if (!h || !noise) return fail(DD_ERR_INVALID, "null argument");
  if (!(h->cfg.flags & DD_FLAG_LOOP_BACKWARD))
    return fail(DD_ERR_INVALID, "dd_denoise_backward needs an engine created with DD_FLAG_LOOP_BACKWARD");
  if (!d_depth && !d_latent) return fail(DD_ERR_INVALID, "d_depth and d_latent are both NULL");
  if (!cond && !h->cond_ready) return fail(DD_ERR_INVALID, "cond is NULL but dd_build_condition has not run");
  if (!h->weights_ready) return fail(DD_ERR_INVALID, "dd_finalize_weights has not been called");
  const int T = h->cfg.num_inference_steps;
  if (static_cast<int>(h->ts.size()) != T) return fail(DD_ERR_INVALID, "dd_set_schedule has not been called");
  const Geom g = geom_of(h->cfg);
  if (static_cast<size_t>(g.B) * g.P * 256 > static_cast<size_t>(INT32_MAX))
    return fail(DD_ERR_UNSUPPORTED, "batch x latent too large for one backward call");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  int rc;
  if ((rc = enter_workspace(h, workspace, workspace_bytes))) return rc;
  dd_engine::LoopBwd& l = h->lp;
  const size_t BP = static_cast<size_t>(g.B) * g.P, nx = BP * 16;
  const size_t ncond = static_cast<size_t>(g.B) * h->cfg.cond_h * h->cfg.cond_w * 256;
  const int npar = param_count(h->cfg);
  if (cond) {
    if ((rc = start_forward(h, st))) return rc;
    if ((rc = transpose_in(cond, h->cond, g.B, 256, h->cfg.cond_h * h->cfg.cond_w, st))) return rc;
  }  // else: dd_build_condition left the NHWC condition map in place
  h->cond_ready = false;
  // 1. the forward again, un-graphed, with the forward's kernels: stash[s] = x before step s, stash[T] = x_0
  if ((rc = transpose_in(noise, h->x32, g.B, 16, g.P, st))) return rc;
  if ((rc = split_planes(h, h->x32, h->xs_hi, h->xs_lo, nx, kXScale, st))) return rc;
  for (int s = 0; s < T; ++s) {
    CUDA_TRY(cudaMemcpyAsync(l.stash + s * nx, h->x32, nx * 4, cudaMemcpyDeviceToDevice, st));
    if ((rc = run_step(h, h->temb + h->ts[s] * 256, 0, h->cx[s], h->ce[s], nullptr, st))) return rc;
  }
  CUDA_TRY(cudaMemcpyAsync(l.stash + T * nx, h->x32, nx * 4, cudaMemcpyDeviceToDevice, st));
  if (latents_out)
    for (int s = 0; s <= T; ++s)
      if ((rc = transpose_out(l.stash + s * nx, latents_out + s * nx, g.B, 16, g.P, st))) return rc;
  // 2. seed: g = d_latent + the decoder's backward at x_0 (still in x32)
  if (d_latent) {
    if ((rc = transpose_in(d_latent, l.gl, g.B, 16, g.P, st))) return rc;
  } else {
    CUDA_TRY(cudaMemsetAsync(l.gl, 0, nx * 4, st));
  }
  if (d_depth) {
    if ((rc = run_decode_bwd(h, d_depth, h->bw.g[1], d_dec_params, st))) return rc;
    dd::latent_grad_step_kernel<<<grid_of(nx), 256, 0, st>>>(l.gl, h->bw.g[1], nullptr, 1.f, nx);
    if ((rc = launched(h, "latent_grad_step"))) return rc;
  } else if (d_dec_params) {  // the depth does not enter the loss: zero decoder gradients
    for (int i = 0; i < 6; ++i)
      if (d_dec_params[i]) CUDA_TRY(cudaMemsetAsync(d_dec_params[i], 0, kDecGradNumel[i] * 4, st));
  }
  // 3. walk back: step s maps x_s -> x_{s+1} = c_x x_s + c_eps eps(x_s)
  float* P[21] = {};
  bool want_dtemb = false;
  if (d_params) {
    for (int i = 0; i < npar; ++i)
      if (d_params[i] && i != 8) P[i] = l.stage + param_offset(i);
    want_dtemb = d_params[8] != nullptr;
  }
  CUDA_TRY(cudaMemsetAsync(l.acc, 0, param_offset(npar) * 8, st));
  if (d_cond_out) CUDA_TRY(cudaMemsetAsync(l.acc_cond, 0, ncond * 8, st));
  auto sink = [&](const float* dc, const float* scale) -> int {
    dd::acc_add_kernel<<<grid_of(ncond), 256, 0, st>>>(l.acc_cond, dc, scale, ncond);
    return launched(h, "acc_add");
  };
  for (int s = T - 1; s >= 0; --s) {
    CUDA_TRY(cudaMemcpyAsync(h->x32, l.stash + s * nx, nx * 4, cudaMemcpyDeviceToDevice, st));
    if ((rc = split_planes(h, h->x32, h->xs_hi, h->xs_lo, nx, kXScale, st))) return rc;
    dd::scale_copy_kernel<<<grid_of(nx), 256, 0, st>>>(l.gl, h->ce[s], h->bw.g[0], nx);
    if ((rc = launched(h, "scale_copy"))) return rc;
    const bool want_dnoisy = s > 0 || d_noise_out != nullptr;
    if ((rc = run_denoiser_bwd(h, h->temb + h->ts[s] * 256, 0, P, want_dtemb, d_cond_out ? &sink : nullptr, want_dnoisy, st)))
      return rc;
    for (int i = 0; i < npar; ++i) {
      if (!P[i]) continue;
      dd::acc_add_kernel<<<grid_of(kParamNumel[i]), 256, 0, st>>>(l.acc + param_offset(i), P[i], nullptr, kParamNumel[i]);
      if ((rc = launched(h, "acc_add"))) return rc;
    }
    if (want_dtemb) {
      dd::temb_acc_kernel<<<1, 256, 0, st>>>(l.acc + param_offset(8) + h->ts[s] * 256, h->bw.dtemb, g.B);
      if ((rc = launched(h, "temb_acc"))) return rc;
    }
    if (want_dnoisy) {
      dd::latent_grad_step_kernel<<<grid_of(nx), 256, 0, st>>>(l.gl, h->bw.g[0], h->bw.scales + 5, h->cx[s], nx);
      if ((rc = launched(h, "latent_grad_step"))) return rc;
    }
  }
  // 4. outputs
  if (d_noise_out && (rc = transpose_out(l.gl, d_noise_out, g.B, 16, g.P, st))) return rc;
  for (int i = 0; i < npar && d_params; ++i) {
    if (!d_params[i]) continue;
    dd::acc_store_kernel<<<grid_of(kParamNumel[i]), 256, 0, st>>>(l.acc + param_offset(i), d_params[i], kParamNumel[i]);
    if ((rc = launched(h, "acc_store"))) return rc;
  }
  if (d_cond_out) {  // fp32 NHWC in a backward buffer of at least that size, then NCHW
    float* dc32 = h->cfg.variant == DD_VARIANT_SWIN ? h->bw.dcond : h->bw.g[1];
    dd::acc_store_kernel<<<grid_of(ncond), 256, 0, st>>>(l.acc_cond, dc32, ncond);
    if ((rc = launched(h, "acc_store"))) return rc;
    if ((rc = transpose_out(dc32, d_cond_out, g.B, 256, h->cfg.cond_h * h->cfg.cond_w, st))) return rc;
  }
  return finish_forward(h, st);
}

int dd_decode_backward(dd_handle h, const float* latent, const float* d_depth, float* d_latent_out,
                       float* const* d_dec_params, void* workspace, size_t workspace_bytes, void* cuda_stream) {
  if (!h || !latent || !d_depth) return fail(DD_ERR_INVALID, "null argument");
  if (!(h->cfg.flags & DD_FLAG_LOOP_BACKWARD))
    return fail(DD_ERR_INVALID, "dd_decode_backward needs an engine created with DD_FLAG_LOOP_BACKWARD");
  if (!h->weights_ready) return fail(DD_ERR_INVALID, "dd_finalize_weights has not been called");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  int rc;
  if ((rc = enter_workspace(h, workspace, workspace_bytes))) return rc;
  const Geom g = geom_of(h->cfg);
  if ((rc = transpose_in(latent, h->x32, g.B, 16, g.P, st))) return rc;
  if ((rc = run_decode_bwd(h, d_depth, d_latent_out ? h->bw.g[1] : nullptr, d_dec_params, st))) return rc;
  if (d_latent_out) return transpose_out(h->bw.g[1], d_latent_out, g.B, 16, g.P, st);
  return DD_OK;
}

int dd_decode(dd_handle h, const float* latent, float* logit_out, float* depth_out, void* workspace,
              size_t workspace_bytes, void* cuda_stream) {
  if (!h || !latent || !depth_out) return fail(DD_ERR_INVALID, "null argument");
  if (!h->weights_ready) return fail(DD_ERR_INVALID, "dd_finalize_weights has not been called");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  int rc;
  if ((rc = enter_workspace(h, workspace, workspace_bytes))) return rc;
  const Geom g = geom_of(h->cfg);
  if ((rc = transpose_in(latent, h->x32, g.B, 16, g.P, st))) return rc;
  const bool train = h->codec_mode == DD_CODEC_TRAIN;
  h->ct.nrec = 0;
  if (train && (rc = run_dec_batch_stats(h, h->ct.rec, st))) return rc;
  h->ct.nrec = train ? 1 : 0;
  return run_decoder(h, logit_out, depth_out, st);
}

int dd_set_codec_mode(dd_handle h, int32_t mode) {
  if (!h) return fail(DD_ERR_INVALID, "null handle");
  if (mode != DD_CODEC_EVAL && mode != DD_CODEC_TRAIN) return fail(DD_ERR_INVALID, "codec mode must be DD_CODEC_EVAL or DD_CODEC_TRAIN");
  h->codec_mode = mode;
  return DD_OK;
}

int dd_codec_batch_stats(dd_handle h, float* dev_out, int32_t capacity, int32_t* n_out, void* cuda_stream) {
  if (!h || !n_out) return fail(DD_ERR_INVALID, "null argument");
  const int n = h->ct.nrec;
  if (n > 0) {
    if (!dev_out || capacity < n) return fail(DD_ERR_INVALID, "dev_out holds fewer records than the last forward wrote");
    CUDA_TRY(cudaSetDevice(h->cfg.device));
    CUDA_TRY(cudaMemcpyAsync(dev_out, h->ct.rec, static_cast<size_t>(n) * 32 * 4, cudaMemcpyDeviceToDevice,
                             static_cast<cudaStream_t>(cuda_stream)));
  }
  *n_out = n;
  return DD_OK;
}

int dd_set_bn_allgather(dd_handle h, dd_allgather_fn fn, void* user, int32_t world_size) {
  if (!h) return fail(DD_ERR_INVALID, "null handle");
  if (fn && world_size < 1) return fail(DD_ERR_INVALID, "world_size must be at least 1");
  CUDA_TRY(cudaSetDevice(h->cfg.device));
  CUDA_TRY(cudaDeviceSynchronize());  // earlier gathers may still read the buffers
  free_bn_sync(h);
  h->sync.fn = fn;
  h->sync.user = fn ? user : nullptr;
  h->sync.world = fn ? world_size : 1;
  return DD_OK;
}

int dd_set_producer_mode(dd_handle h, int32_t mode) {
  if (!h) return fail(DD_ERR_INVALID, "null handle");
  if (mode != DD_PRODUCER_EVAL && mode != DD_PRODUCER_TRAIN)
    return fail(DD_ERR_INVALID, "producer mode must be DD_PRODUCER_EVAL or DD_PRODUCER_TRAIN");
  if (mode == DD_PRODUCER_TRAIN && !(h->cfg.flags & DD_FLAG_PRODUCER_TRAIN))
    return fail(DD_ERR_INVALID, "DD_PRODUCER_TRAIN needs an engine created with DD_FLAG_PRODUCER_TRAIN");
  h->producer_mode = mode;
  return DD_OK;
}

int dd_set_drop_path(dd_handle h, const float* dev_scales, int32_t n, void* cuda_stream) {
  if (!h) return fail(DD_ERR_INVALID, "null handle");
  DropPathState& d = h->drop;
  if (n == 0) {
    d.on = false;
    return DD_OK;
  }
  if (!dev_scales) return fail(DD_ERR_INVALID, "null argument");
  if (!((h->mp.enabled && h->mp.ready) || (h->bb.enabled && h->bb.ready)))
    return fail(DD_ERR_INVALID, "dd_set_drop_path needs a finalized MPViT or Swin backbone");
  if (n != static_cast<int64_t>(d.blocks) * 2 * h->cfg.batch)
    return fail(DD_ERR_INVALID, "dd_set_drop_path: n must be 0 or 2 x batch x the blocks mp_drop_path marks (" +
                                    std::to_string(static_cast<int64_t>(d.blocks) * 2 * h->cfg.batch) + ")");
  CUDA_TRY(cudaSetDevice(h->cfg.device));
  CUDA_TRY(cudaMemcpyAsync(d.scales, dev_scales, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToDevice,
                           static_cast<cudaStream_t>(cuda_stream)));
  d.on = true;
  return DD_OK;
}

int dd_producer_batch_stats(dd_handle h, float* dev_out, int64_t capacity, int32_t* n_out, void* cuda_stream) {
  if (!h || !n_out) return fail(DD_ERR_INVALID, "null argument");
  const dd_engine::ProdTrain& pt = h->pt;
  if (dev_out && !pt.layers.empty()) {
    if (capacity < static_cast<int64_t>(pt.rec_floats))
      return fail(DD_ERR_INVALID, "dev_out holds fewer floats than the records");
    CUDA_TRY(cudaSetDevice(h->cfg.device));
    CUDA_TRY(cudaMemcpyAsync(dev_out, pt.rec, pt.rec_floats * 4, cudaMemcpyDeviceToDevice,
                             static_cast<cudaStream_t>(cuda_stream)));
  }
  *n_out = static_cast<int32_t>(pt.layers.size());
  return DD_OK;
}

int dd_producer_bn_info(dd_handle h, int32_t i, char* key, int32_t key_capacity, int32_t* channels, int64_t* offset,
                        int32_t* fresh) {
  if (!h) return fail(DD_ERR_INVALID, "null handle");
  if (i < 0 || i >= static_cast<int32_t>(h->pt.layers.size())) return fail(DD_ERR_INVALID, "record index out of range");
  const dd_engine::ProdBn& b = h->pt.layers[i];
  if (key && key_capacity > 0) {
    const size_t n = std::min(b.key.size(), static_cast<size_t>(key_capacity - 1));
    memcpy(key, b.key.data(), n);
    key[n] = 0;
  }
  if (channels) *channels = b.C;
  if (offset) *offset = static_cast<int64_t>(b.rec_off);
  if (fresh) *fresh = b.fresh ? 1 : 0;
  return DD_OK;
}

int dd_enable_producers(dd_handle h, const dd_producer_config* pc) {
  if (!h || !pc) return fail(DD_ERR_INVALID, "null argument");
  if (pc->num_levels < 2 || pc->num_levels > 4) return fail(DD_ERR_INVALID, "producers need 2..4 pyramid levels");
  Producers p;
  p.enabled = true;
  p.neck = pc->has_neck != 0;
  p.nlev = pc->num_levels;
  for (int i = 0; i < p.nlev; ++i) {
    p.C[i] = pc->channels[i];
    p.H[i] = pc->heights[i];
    p.W[i] = pc->widths[i];
    // 16-byte rows for TMA and the vector stores of the epilogues; nothing else constrains the counts (MPViT: 128/216/288/288)
    if (p.C[i] % 8 != 0 || p.C[i] <= 0) return fail(DD_ERR_UNSUPPORTED, "feature channels must be positive multiples of 8");
    // the FPN's adaptive_avg_pool2d (reference head :121) is the identity only for exact 2x pyramids; otherwise the
    // ConvT output (2x the coarser level) is average-pooled down to the lateral's size by a dedicated kernel
    if (i > 0 && (p.H[i - 1] != 2 * p.H[i] || p.W[i - 1] != 2 * p.W[i])) {
      p.resample = true;
      if (p.H[i - 1] > 2 * p.H[i] || p.W[i - 1] > 2 * p.W[i])
        return fail(DD_ERR_UNSUPPORTED, "feature pyramid level is more than 2x its coarser neighbour");
    }
  }
  if (p.H[0] != h->cfg.cond_h || p.W[0] != h->cfg.cond_w)
    return fail(DD_ERR_INVALID, "level-0 feature size must equal the condition map size");
  h->prod = p;
  invalidate_pack(h);
  return DD_OK;
}

int dd_build_condition(dd_handle h, const float* const* feats, float* cond_out, void* workspace, size_t workspace_bytes,
                       void* cuda_stream) {
  if (!h) return fail(DD_ERR_INVALID, "null argument");
  if (!feats && !h->feats_ready) return fail(DD_ERR_INVALID, "feats is NULL but dd_run_backbone has not run");
  if (!h->prod.enabled || !h->weights_ready || !h->prod.ready)
    return fail(DD_ERR_INVALID, "producers not enabled / weights not finalized");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  int rc;
  if ((rc = enter_workspace(h, workspace, workspace_bytes))) return rc;
  Producers& p = h->prod;
  const int B = h->cfg.batch;
  if (feats) {
    if ((rc = start_forward(h, st))) return rc;
    producer_forward_start(h);
  }  // else: dd_run_backbone already wrote the input planes F[i] (and owns the status / launch counters)
  h->feats_ready = false;
  for (int i = 0; feats && i < p.nlev; ++i) {
    if (!feats[i]) return fail(DD_ERR_INVALID, "null feature map");
    const int P = p.H[i] * p.W[i];
    dim3 grid((P + 31) / 32, (p.C[i] + 31) / 32, B), block(32, 8);
    dd::nchw_to_nhwc_split_kernel<<<grid, block, 0, st>>>(feats[i], p.F[i].hi, p.F[i].lo, p.C[i], P, kProdScale, h->status);
    if ((rc = launched(h, "nchw_to_nhwc_split"))) return rc;
  }
  auto build = [&](cudaStream_t s) -> int {
  const Planes none;
  for (int i = 0; i < p.nlev; ++i) {
    if (!p.neck) {
      p.O[i] = p.F[i];
      continue;
    }
    // HAHI neck, attention gates off (reference necks/hahi.py:173-176, 226-250, 253-272)
    if ((rc = run_gen(h, p.lat[i], p.F[i], p.C[i], none, 0, p.H[i], p.W[i], nullptr, nullptr, &p.L[i], s))) return rc;
    if ((rc = run_gen(h, p.proj[i], p.L[i], p.C[i], none, 0, p.H[i], p.W[i], nullptr, nullptr, &p.P[i], s))) return rc;
    if (i == 0) {  // cat([conv_proj(lat), lat])
      if ((rc = run_gen(h, p.fus[i], p.P[i], 512, p.L[i], p.C[i], p.H[i], p.W[i], nullptr, nullptr, &p.O[i], s))) return rc;
    } else {       // cat([lat, trans_proj(lat)])
      if ((rc = run_gen(h, p.fus[i], p.L[i], p.C[i], p.P[i], 512, p.H[i], p.W[i], nullptr, nullptr, &p.O[i], s))) return rc;
    }
  }
  // FPN top-down (reference head :112-122): x_i = relu(bn(conv3x3(O_i))) + relu(bn(convT2x2(x_{i+1})))
  for (int i = p.nlev - 1; i >= 0; --i) {
    const float* add = (i < p.nlev - 1) ? p.UP[i] : nullptr;
    if ((rc = run_gen(h, p.fl[i], p.O[i], p.C[i], none, 0, p.H[i], p.W[i], p.X[i], add, i > 0 ? &p.XP[i] : nullptr, s)))
      return rc;
    if (i > 0) {
      float* up_raw = p.resample ? p.UPR[i - 1] : p.UP[i - 1];
      if ((rc = run_gen(h, p.fu[i - 1], p.XP[i], 256, none, 0, p.H[i], p.W[i], up_raw, nullptr, nullptr, s))) return rc;
      if (p.resample) {  // F.adaptive_avg_pool2d(conv_up(pre_x), output_size = lateral size)  (reference head :121)
        const size_t n = static_cast<size_t>(B) * p.H[i - 1] * p.W[i - 1] * 256;
        dd::adaptive_avg_pool_nhwc_kernel<<<grid_of(n), 256, 0, s>>>(up_raw, p.UP[i - 1], B, 2 * p.H[i], 2 * p.W[i],
                                                                     p.H[i - 1], p.W[i - 1], 256);
        if ((rc = launched(h, "adaptive_avg_pool"))) return rc;
      }
    }
  }
  return DD_OK;
  };
  // every pointer of the neck / FPN kernels lives in the workspace -> replayable as a graph; with a BatchNorm all-gather
  // installed the training-mode launches run eagerly (the gathers are host calls)
  const bool train = h->producer_mode == DD_PRODUCER_TRAIN;
  if ((h->cfg.flags & DD_FLAG_CUDA_GRAPH) && !(train && h->sync.fn)) {
    if ((rc = graph_run(h, train ? dd_engine::G_COND_TRAIN : dd_engine::G_COND, st, build))) return rc;
  } else if ((rc = build(st))) {
    return rc;
  }
  if (train) producer_mark_fresh(h, 1);
  h->cond_ready = true;
  if (cond_out) {
    if ((rc = transpose_out(h->cond, cond_out, B, 256, p.H[0] * p.W[0], st))) return rc;
    h->launches++;
  }
  return DD_OK;
}

// dd_backbone_config.mp_drop_path of a backbone with depths[s] blocks per stage, each marked block counting per_mark[s]
// times (MPViT: its paths) -> *d, stochastic depth off
int drop_marks(const int32_t* marks, const int* depths, const int* per_mark, DropPathState* d) {
  *d = DropPathState();
  for (int s = 0; s < 4; ++s) {
    d->mask[s] = marks[s];
    if (d->mask[s] < 0 || (depths[s] < 31 && (d->mask[s] >> depths[s]) != 0))
      return fail(DD_ERR_INVALID, "mp_drop_path marks a block the stage does not have");
    d->blocks += per_mark[s] * __builtin_popcount(static_cast<unsigned>(d->mask[s]));
  }
  return DD_OK;
}

int dd_enable_backbone(dd_handle h, const dd_backbone_config* bc) {
  if (!h || !bc) return fail(DD_ERR_INVALID, "null argument");
  if (bc->kind == DD_BACKBONE_RESNET) {
    if (!h->prod.enabled || h->prod.neck || h->prod.nlev != 4)
      return fail(DD_ERR_INVALID, "dd_enable_producers (4 levels, no neck) must be called first");
    ResNetW r;
    r.enabled = true;
    r.H = bc->height;
    r.W = bc->width;
    int hh = bc->height, ww = bc->width;
    for (int s = 0; s < 4; ++s) {
      r.depths[s] = bc->depths[s];
      if (r.depths[s] < 1) return fail(DD_ERR_INVALID, "bad ResNet depth");
      hh = (hh - 1) / 2 + 1;  // 3x3, stride 2, pad 1
      ww = (ww - 1) / 2 + 1;
      r.Hs[s] = hh;
      r.Ws[s] = ww;
      if (hh != h->prod.H[s] || ww != h->prod.W[s] || r.C[s] != h->prod.C[s])
        return fail(DD_ERR_INVALID, "backbone stage geometry does not match the producer pyramid");
    }
    h->rn = r;
    h->drop = DropPathState();
    h->bb.enabled = false;
    h->mp.enabled = false;
    invalidate_pack(h);
    return DD_OK;
  }
  if (bc->kind == DD_BACKBONE_MPVIT) {
    if (!h->prod.enabled || h->prod.nlev != 4)
      return fail(DD_ERR_INVALID, "dd_enable_producers (4 levels) must be called first");
    MPViTW m;
    m.enabled = true;
    m.H = bc->height;
    m.W = bc->width;
    m.heads = 8;  // every MPViT variant (reference mpvit.py:743-870)
    m.mlp_ratio = bc->mlp_ratio;
    if (m.mlp_ratio < 1 || m.mlp_ratio > 8) return fail(DD_ERR_INVALID, "bad MPViT mlp_ratio");
    int hh = bc->height, ww = bc->width;
    for (int s = 0; s < 4; ++s) {
      m.dims[s] = bc->mp_dims[s];
      m.layers[s] = bc->depths[s];
      m.paths[s] = bc->mp_paths[s];
      if (m.layers[s] < 1 || m.paths[s] < 1 || m.paths[s] > 3) return fail(DD_ERR_UNSUPPORTED, "MPViT: 1..3 paths, >= 1 layer per stage");
      if (m.dims[s] <= 0 || m.dims[s] % 8 != 0 || m.dims[s] / m.heads > dd::KTV_CH_MAX || m.dims[s] > 512)
        return fail(DD_ERR_UNSUPPORTED, "MPViT: stage widths must be multiples of 8 (8 heads), at most 512");
      hh = (hh - 1) / 2 + 1;  // depthwise 3x3, stride 2, pad 1
      ww = (ww - 1) / 2 + 1;
      m.Hs[s] = hh;
      m.Ws[s] = ww;
    }
    if (m.dims[0] % 16 != 0) return fail(DD_ERR_UNSUPPORTED, "MPViT: stem width must be a multiple of 16");
    for (int s = 0; s < 4; ++s) {
      m.out_dims[s] = s < 3 ? m.dims[s + 1] : m.dims[s];
      if (m.Hs[s] != h->prod.H[s] || m.Ws[s] != h->prod.W[s] || m.out_dims[s] != h->prod.C[s])
        return fail(DD_ERR_INVALID, "backbone stage geometry does not match the producer pyramid");
    }
    DropPathState d;
    int rc;
    if ((rc = drop_marks(bc->mp_drop_path, m.layers, m.paths, &d))) return rc;
    h->mp = m;
    h->drop = d;
    h->bb.enabled = false;
    h->rn.enabled = false;
    invalidate_pack(h);
    return DD_OK;
  }
  if (bc->kind != DD_BACKBONE_SWIN) return fail(DD_ERR_UNSUPPORTED, "unknown backbone kind");
  if (!h->prod.enabled || h->prod.nlev != 4)
    return fail(DD_ERR_INVALID, "dd_enable_producers (4 levels) must be called first");
  if (bc->embed_dims != 192 || bc->window != 7)
    return fail(DD_ERR_UNSUPPORTED, "native Swin is instantiated for embed_dims 192 (Swin-L), window 7");
  Backbone b;
  b.enabled = true;
  b.E = bc->embed_dims;
  b.window = bc->window;
  b.H = bc->height;
  b.W = bc->width;
  int hh = (bc->height + 3) / 4, ww = (bc->width + 3) / 4;
  for (int s = 0; s < 4; ++s) {
    b.depths[s] = bc->depths[s];
    b.heads[s] = bc->num_heads[s];
    if (b.depths[s] < 1 || (b.E << s) != 32 * b.heads[s]) return fail(DD_ERR_UNSUPPORTED, "Swin head_dim must be 32");
    b.Hs[s] = hh;
    b.Ws[s] = ww;
    if (hh != h->prod.H[s] || ww != h->prod.W[s] || (b.E << s) != h->prod.C[s])
      return fail(DD_ERR_INVALID, "backbone stage geometry does not match the producer pyramid");
    hh = (hh + 1) / 2;
    ww = (ww + 1) / 2;
  }
  const int one[4] = {1, 1, 1, 1};
  DropPathState d;
  int rc;
  if ((rc = drop_marks(bc->mp_drop_path, b.depths, one, &d))) return rc;
  h->bb = b;
  h->drop = d;
  h->rn.enabled = false;
  h->mp.enabled = false;
  invalidate_pack(h);
  return DD_OK;
}

int dd_run_backbone(dd_handle h, const float* rgb, float* const* feats_out, void* workspace, size_t workspace_bytes,
                    void* cuda_stream) {
  if (!h || !rgb) return fail(DD_ERR_INVALID, "null argument");
  const bool swin = h->bb.enabled && h->bb.ready, resnet = h->rn.enabled && h->rn.ready, mpvit = h->mp.enabled && h->mp.ready;
  if (!h->weights_ready || !(swin || resnet || mpvit)) return fail(DD_ERR_INVALID, "backbone not enabled / weights not finalized");
  auto run = [&](const float* img, float* const* outs, cudaStream_t s) {
    return swin ? run_swin(h, img, outs, s) : (resnet ? run_resnet(h, img, outs, s) : run_mpvit(h, img, outs, s));
  };
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  int rc;
  if ((rc = enter_workspace(h, workspace, workspace_bytes))) return rc;
  if ((rc = start_forward(h, st))) return rc;
  producer_forward_start(h);
  // the ResNet's and MPViT's BatchNorms follow the producer mode (Swin has none); MPViT's and Swin's stochastic depth is
  // on while dd_set_drop_path holds scales, in either mode
  const bool train = (resnet || mpvit) && h->producer_mode == DD_PRODUCER_TRAIN;
  const bool drop = (mpvit || swin) && h->drop.on;
  bool want_out = false;
  for (int i = 0; feats_out && i < 4; ++i) want_out |= (feats_out[i] != nullptr);
  if ((h->cfg.flags & DD_FLAG_CUDA_GRAPH) && !want_out && !(train && h->sync.fn)) {
    // the graph's kernels read the image from the workspace: stage the caller's batch there first (20 MB at C3)
    const size_t n = static_cast<size_t>(h->cfg.batch) * 3 *
                     (swin ? h->bb.H * h->bb.W : (resnet ? h->rn.H * h->rn.W : h->mp.H * h->mp.W));
    CUDA_TRY(cudaMemcpyAsync(h->rgb_stage, rgb, n * 4, cudaMemcpyDeviceToDevice, st));
    const int which = train ? (drop ? dd_engine::G_BACKBONE_TRAIN_DROP : dd_engine::G_BACKBONE_TRAIN)
                            : (drop ? dd_engine::G_BACKBONE_DROP : dd_engine::G_BACKBONE);
    if ((rc = graph_run(h, which, st, [&](cudaStream_t s) { return run(h->rgb_stage, nullptr, s); })))
      return rc;
  } else if ((rc = run(rgb, feats_out, st))) {
    return rc;
  }
  if (train) producer_mark_fresh(h, 0);
  h->feats_ready = true;
  return DD_OK;
}

// Debug / tuning aid: time the GEMM-mode kernel on synthetic planes.  mode: 0 fp32 out, 1 fp32 out + residual add,
// 2 GELU -> planes, 3 no output at all (mainloop + accumulator drain only).
int dd_bench_gemm(dd_handle h, int32_t M, int32_t K, int32_t N, int32_t mode, int32_t iters, float* ms_out) {
  if (!h || !ms_out || M < 1 || K % dd::GEN_BK || N % 192 && N % 256) return fail(DD_ERR_INVALID, "bad argument");
  CUDA_TRY(cudaSetDevice(h->cfg.device));
  cudaStream_t st = h->cap_stream;
  const size_t Mp = (static_cast<size_t>(M) + 127) / 128 * 128 + 128;
  StandaloneCall call(h);
  int rc;
  if ((rc = call.begin(st))) return rc;
  Planes A, O;
  GenLayer L;
  float *y = nullptr, *bias = nullptr;
  if ((rc = call.alloc(&A.hi, Mp * K)) || (rc = call.alloc(&A.lo, Mp * K)) || (rc = call.alloc(&O.hi, Mp * N)) ||
      (rc = call.alloc(&O.lo, Mp * N)) || (rc = call.alloc(&y, Mp * N)) ||
      (rc = call.alloc(&L.w_hi, static_cast<size_t>(N) * K)) || (rc = call.alloc(&L.w_lo, static_cast<size_t>(N) * K)) ||
      (rc = call.alloc(&bias, N)))
    return rc;
  CUDA_TRY(cudaMemsetAsync(A.hi, 0x11, Mp * K * 2, st));
  CUDA_TRY(cudaMemsetAsync(A.lo, 0x01, Mp * K * 2, st));
  CUDA_TRY(cudaMemsetAsync(L.w_hi, 0x11, static_cast<size_t>(N) * K * 2, st));
  CUDA_TRY(cudaMemsetAsync(L.w_lo, 0x01, static_cast<size_t>(N) * K * 2, st));
  CUDA_TRY(cudaMemsetAsync(bias, 0, N * 4, st));
  CUDA_TRY(cudaMemsetAsync(y, 0, Mp * N * 4, st));
  L.cin = K;
  L.cout = N;
  L.nt = (N % 256 == 0) ? 256 : 192;
  L.shift = bias;
  if ((rc = make_weight_map(&L.mb_hi, L.w_hi, N, K, 1, dd::GEN_BK, dd::gen_unit_cols(L.nt)))) return rc;
  if ((rc = make_weight_map(&L.mb_lo, L.w_lo, N, K, 1, dd::GEN_BK, dd::gen_unit_cols(L.nt)))) return rc;
  return time_per_call(st, 3, iters, ms_out, [&]() {
    return run_gemm(h, L, A, M, mode == 2 ? 2 : 0, (mode == 0 || mode == 1) ? y : nullptr, mode == 1 ? y : nullptr,
                    mode == 2 ? &O : nullptr, st);
  });
}

int dd_encode(dd_handle h, const float* depth, int32_t height, int32_t width, float* latent_out, void* cuda_stream) {
  if (!h || !depth || !latent_out) return fail(DD_ERR_INVALID, "null argument");
  if (!h->weights_ready || !h->enc_w1) return fail(DD_ERR_INVALID, "encoder weights (depth_transform.conv_transform.*) not registered");
  if ((height + 1) / 2 != h->cfg.latent_h || (width + 1) / 2 != h->cfg.latent_w)
    return fail(DD_ERR_INVALID, "depth map size does not match the engine's latent grid");
  const bool train = h->codec_mode == DD_CODEC_TRAIN;
  if (train && static_cast<long long>(h->cfg.batch) * h->cfg.latent_h * h->cfg.latent_w < 2)
    return fail(DD_ERR_INVALID, "training-mode BatchNorm needs more than 1 value per channel (batch x latent = 1)");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  CUDA_TRY(cudaSetDevice(h->cfg.device));
  dd_engine::CodecTrain& ct = h->ct;
  ct.nrec = 0;
  if (train) {  // BN1 over conv1, then BN2 over conv2 of the batch-normalised, activated conv1; records 0 and 1
    const long long n = static_cast<long long>(h->cfg.batch) * h->cfg.latent_h * h->cfg.latent_w;
    const dd::EncPreBn1 op1{depth, ct.enc_w1, height, width, h->cfg.latent_h, h->cfg.latent_w};
    int rc;
    if ((rc = run_codec_bn(h, op1, n, ct.enc_gb, nullptr, ct.enc_w1, 144, ct.enc_w1f, ct.enc_b1f, nullptr, ct.rec, st)))
      return rc;
    const dd::EncPreBn2 op2{depth, ct.enc_w1f, ct.enc_b1f, ct.enc_w2, height, width, h->cfg.latent_h, h->cfg.latent_w};
    if ((rc = run_codec_bn(h, op2, n, ct.enc_gb + 32, nullptr, ct.enc_w2, 2304, ct.enc_w2f, ct.enc_b2f, nullptr,
                           ct.rec + 32, st)))
      return rc;
    ct.nrec = 2;
  }
  dd::EncoderArgs a;
  a.depth = depth;
  a.w1 = train ? ct.enc_w1f : h->enc_w1;
  a.b1 = train ? ct.enc_b1f : h->enc_b1;
  a.w2 = train ? ct.enc_w2f : h->enc_w2;
  a.b2 = train ? ct.enc_b2f : h->enc_b2;
  a.out = latent_out;
  a.H = height;
  a.W = width;
  a.h = h->cfg.latent_h;
  a.w = h->cfg.latent_w;
  dim3 grid((a.w + 15) / 16, (a.h + 15) / 16, h->cfg.batch);
  dd::encoder_kernel<<<grid, 256, 0, st>>>(a);
  return check_launch("encoder");
}

// The encoder backward's weight partials fit the smallest wgrad partials region: one chunk of a 256 -> 256 conv.
static_assert(dd::ENC_WG_BLOCKS * dd::ENC_WG_COLS <= 256 * 256 * 9, "encoder weight partials exceed bw.wg_part");

// Reverse mode of dd_encode in the current codec mode: d_latent NCHW [B][16][h][w] -> the six encoder gradients
// dp[0..5] (each nullable), in ENCODER_KEYS order without the running statistics.  Its planes and partials live in the
// operator backward's region (bw.g[0], bw.g[1], bw.wg_part), which no other call uses while this one runs.
int run_encode_bwd(dd_engine* e, const float* depth, int H, int W, const float* d_latent, float* const* dp, cudaStream_t st) {
  const Geom g = geom_of(e->cfg);
  const long long N = static_cast<long long>(g.B) * g.P;
  const bool train = e->codec_mode == DD_CODEC_TRAIN;
  dd_engine::CodecTrain& ct = e->ct;
  int rc;
  if (train) {  // dd_encode's two batch statistics, the same kernels in the same order; no record
    const dd::EncPreBn1 op1{depth, ct.enc_w1, H, W, g.h, g.w};
    if ((rc = run_codec_bn(e, op1, N, ct.enc_gb, nullptr, ct.enc_w1, 144, ct.enc_w1f, ct.enc_b1f, ct.enc_bn, nullptr, st)))
      return rc;
    const dd::EncPreBn2 op2{depth, ct.enc_w1f, ct.enc_b1f, ct.enc_w2, H, W, g.h, g.w};
    if ((rc = run_codec_bn(e, op2, N, ct.enc_gb + 32, nullptr, ct.enc_w2, 2304, ct.enc_w2f, ct.enc_b2f, ct.enc_bn + 48,
                           nullptr, st)))
      return rc;
  }
  const float* bn = train ? ct.enc_bn : e->enc_bn;
  const size_t plane = static_cast<size_t>(N) * 16;
  const int nb_pix = static_cast<int>((N + dd::ENC_PIX - 1) / dd::ENC_PIX);
  const int nb_w = static_cast<int>(std::min<long long>(dd::ENC_WG_BLOCKS, (N + 1023) / 1024));
  const int per_block = static_cast<int>((N + nb_w - 1) / nb_w);
  dd::EncBwdArgs a;
  a.depth = depth;
  a.w1f = train ? ct.enc_w1f : e->enc_w1;
  a.b1f = train ? ct.enc_b1f : e->enc_b1;
  a.w2f = train ? ct.enc_w2f : e->enc_w2;
  a.b2f = train ? ct.enc_b2f : e->enc_b2;
  a.w1u = ct.enc_w1;
  a.w2u = ct.enc_w2;
  a.bn1 = bn;
  a.bn2 = bn + 48;
  a.dlat = d_latent;
  a.a1 = e->bw.g[0];
  a.x1 = e->bw.g[0] + plane;
  a.x2 = e->bw.g[0] + 2 * plane;
  a.dz = e->bw.g[0] + 3 * plane;
  a.part2 = reinterpret_cast<double*>(e->bw.g[1]);
  a.part1 = a.part2 + static_cast<size_t>(nb_pix) * 32;
  a.part_w = e->bw.wg_part;
  a.B = g.B;
  a.H = H;
  a.W = W;
  a.h = g.h;
  a.w = g.w;
  dd::enc_bwd_mid_kernel<<<nb_pix, 256, 0, st>>>(a);
  if ((rc = launched(e, "enc_bwd_mid"))) return rc;
  dd::enc_bwd_out_kernel<<<nb_pix, 256, 0, st>>>(a);
  if ((rc = launched(e, "enc_bwd_out"))) return rc;
  // each BatchNorm's du through its statistics (training mode: the two backward sums, across ranks the union batch's)
  auto bn_bwd = [&](float* d, const float* xhat, const float* bnk, const double* part) -> int {
    BnTotals t{nullptr, nullptr};
    int r;
    if (train && (r = bn_totals(e, part, nb_pix, 32, 32, N, ct.sums, 33, st, &t))) return r;
    dd::enc_bwd_bn_kernel<<<grid_of(plane), 256, 0, st>>>(d, xhat, bnk, t.sum, t.cnt, N);
    return launched(e, "enc_bwd_bn");
  };
  if ((rc = bn_bwd(a.dz, a.x2, a.bn2, a.part2))) return rc;
  dd::enc_bwd_mid_grad_kernel<<<nb_pix, 256, 0, st>>>(a);
  if ((rc = launched(e, "enc_bwd_mid_grad"))) return rc;
  if ((rc = bn_bwd(a.x2, a.x1, a.bn1, a.part1))) return rc;
  dd::enc_bwd_wgrad_kernel<<<nb_w, 160, 0, st>>>(a, per_block);
  if ((rc = launched(e, "enc_bwd_wgrad"))) return rc;
  dd::EncFinishArgs f;
  f.part1 = a.part1;
  f.part2 = a.part2;
  f.part_w = a.part_w;
  f.nb_pix = nb_pix;
  f.nb_w = nb_w;
  for (int i = 0; i < 6; ++i) f.out[i] = dp[i];
  dd::enc_bwd_finish_kernel<<<(dd::ENC_GRAD_N + 255) / 256, 256, 0, st>>>(f);
  return launched(e, "enc_bwd_finish");
}

int dd_encode_backward(dd_handle h, const float* depth, int32_t height, int32_t width, const float* d_latent,
                       float* const* d_enc_params, void* workspace, size_t workspace_bytes, void* cuda_stream) {
  if (!h || !depth || !d_latent) return fail(DD_ERR_INVALID, "null argument");
  int rc;
  if ((rc = check_operator_bwd_call(h, "dd_encode_backward"))) return rc;
  if (!h->enc_w1) return fail(DD_ERR_INVALID, "encoder weights (depth_transform.conv_transform.*) not registered");
  if ((height + 1) / 2 != h->cfg.latent_h || (width + 1) / 2 != h->cfg.latent_w)
    return fail(DD_ERR_INVALID, "depth map size does not match the engine's latent grid");
  if (h->codec_mode == DD_CODEC_TRAIN && static_cast<long long>(h->cfg.batch) * h->cfg.latent_h * h->cfg.latent_w < 2)
    return fail(DD_ERR_INVALID, "training-mode BatchNorm needs more than 1 value per channel (batch x latent = 1)");
  if (static_cast<long long>(h->cfg.batch) * height * width > static_cast<long long>(INT32_MAX))
    return fail(DD_ERR_UNSUPPORTED, "depth map too large for one encoder backward call");
  if ((rc = enter_workspace(h, workspace, workspace_bytes))) return rc;
  float* none[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  return run_encode_bwd(h, depth, height, width, d_latent, d_enc_params ? d_enc_params : none,
                        static_cast<cudaStream_t>(cuda_stream));
}

int64_t dd_last_launch_count(dd_handle h) { return h ? h->launches : 0; }

int dd_poll_status(dd_handle h, void* cuda_stream) {
  if (!h) return fail(DD_ERR_INVALID, "null handle");
  if (!h->status) return DD_OK;  // nothing has run yet
  CUDA_TRY(cudaSetDevice(h->cfg.device));
  return poll_status(h, static_cast<cudaStream_t>(cuda_stream));
}

// ---------------------------------------------------------------- standalone conv (tests / roofline)
size_t dd_conv3x3_workspace_bytes(int32_t batch, int32_t cin, int32_t cout, int32_t height, int32_t width) {
  Conv3x3Ws v;
  return conv3x3_layout(nullptr, batch, cin, cout, height, width, v);
}

int dd_conv3x3(dd_handle h, const float* x, const float* w, const float* b, float* y, int32_t batch, int32_t cin,
               int32_t cout, int32_t height, int32_t width, void* workspace, size_t workspace_bytes, void* cuda_stream) {
  if (!h || !x || !w || !b || !y) return fail(DD_ERR_INVALID, "null argument");
  const int sid = shape_id(cin, cout);
  if (sid < 0) return fail(DD_ERR_UNSUPPORTED, "conv shape not on the DiffusionDepth hot path");
  if (workspace_bytes < dd_conv3x3_workspace_bytes(batch, cin, cout, height, width) ||
      (reinterpret_cast<uintptr_t>(workspace) & 1023))
    return fail(DD_ERR_INVALID, "conv workspace too small or misaligned");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  CUDA_TRY(cudaSetDevice(h->cfg.device));
  const size_t BP = static_cast<size_t>(batch) * height * width;
  const size_t nw = static_cast<size_t>(cin) * cout * 9;
  Conv3x3Ws v;
  conv3x3_layout(workspace, batch, cin, cout, height, width, v);
  CUDA_TRY(cudaMemsetAsync(v.status, 0, 64, st));
  int rc;
  if ((rc = transpose_in(x, v.xn, batch, cin, height * width, st))) return rc;
  float* amax_dev = reinterpret_cast<float*>(v.status) + 8;
  float sx, sw;
  if ((rc = split_scale_of(v.xn, std::min<size_t>(BP * cin, 1u << 30), amax_dev, st, &sx))) return rc;
  if ((rc = split_scale_of(w, nw, amax_dev, st, &sw))) return rc;
  dd::split_planes_kernel<<<132 * 8, 256, 0, st>>>(v.xn, v.x.hi, v.x.lo, BP * cin / 4, sx, v.status);
  if ((rc = check_launch("split_planes"))) return rc;
  dd::pack_conv_weight_kernel<<<128, 256, 0, st>>>(w, v.w.hi, v.w.lo, v.wsimt, cout, cin, sw);
  if ((rc = check_launch("pack_conv_weight"))) return rc;
  dd::ConvArgs a;
  a.B = batch;
  a.H = height;
  a.W = width;
  a.bias = b;
  a.acc_scale = 1.f / (sx * sw);
  a.y32 = v.yn;
  a.stats_partial = nullptr;
  a.out_hi = nullptr;
  a.out_lo = nullptr;
  a.split_scale = 1.f;
  a.status = v.status;
  const bool simt = (h->cfg.flags & DD_FLAG_SIMT_CONV) != 0;
  CUtensorMap mb_hi{}, mb_lo{};
  if (!simt) {
    if ((rc = make_weight_map(&mb_hi, v.w.hi, cout, cin, 9, kHaloBK[sid], cout))) return rc;
    if ((rc = make_weight_map(&mb_lo, v.w.lo, cout, cin, 9, kHaloBK[sid], cout))) return rc;
  }
  if ((rc = launch_conv3x3(sid, dd::EPI_F32, simt, a, v.x.hi, v.x.lo, sx, v.wsimt, mb_hi, mb_lo, h->sm_count, st)))
    return rc;
  if ((rc = check_launch("conv3x3"))) return rc;
  return transpose_out(v.yn, y, batch, cout, height * width, st);
}

// ---------------------------------------------------------------- standalone weight gradient (tests / roofline)
size_t dd_conv3x3_wgrad_workspace_bytes(int32_t batch, int32_t cin, int32_t cout, int32_t height, int32_t width) {
  WgradWs v;
  return wgrad_layout(nullptr, batch, cin, cout, height, width, v);
}

int dd_conv3x3_wgrad(dd_handle h, const float* x, const float* dy, float* dw, float* db, int32_t batch, int32_t cin,
                     int32_t cout, int32_t height, int32_t width, void* workspace, size_t workspace_bytes,
                     void* cuda_stream) {
  if (!h || !x || !dy || !dw || !db) return fail(DD_ERR_INVALID, "null argument");
  if (shape_id(cin, cout) < 0) return fail(DD_ERR_UNSUPPORTED, "conv shape not on the DiffusionDepth hot path");
  if (batch < 1 || height < 1 || width < 1) return fail(DD_ERR_INVALID, "empty geometry");
  if (workspace_bytes < dd_conv3x3_wgrad_workspace_bytes(batch, cin, cout, height, width) ||
      (reinterpret_cast<uintptr_t>(workspace) & 1023))
    return fail(DD_ERR_INVALID, "wgrad workspace too small or misaligned");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  CUDA_TRY(cudaSetDevice(h->cfg.device));
  const int P = height * width;
  const size_t BP = static_cast<size_t>(batch) * P;
  WgradWs v;
  wgrad_layout(workspace, batch, cin, cout, height, width, v);
  float* scratch = reinterpret_cast<float*>(v.status) + 8;  // [0] x absmax, [1] dy absmax, [2] dy split scale
  CUDA_TRY(cudaMemsetAsync(v.status, 0, 64, st));
  int rc;
  if ((rc = transpose_in(x, v.xn, batch, cin, P, st))) return rc;
  if ((rc = transpose_in(dy, v.dyn, batch, cout, P, st))) return rc;
  // X: host-side power-of-two scale, as dd_conv3x3 splits its input
  float sx;
  if ((rc = split_scale_of(v.xn, BP * cin, scratch, st, &sx))) return rc;
  dd::split_planes_kernel<<<132 * 8, 256, 0, st>>>(v.xn, v.x.hi, v.x.lo, BP * cin / 4, sx, v.status);
  if ((rc = launched(h, "split_planes"))) return rc;
  // dY: the backward's own on-device split (also for the SIMT shapes, so a non-finite dY is reported for every shape)
  if ((rc = run_colsum(h, cout, v.dyn, nullptr, batch, P, v.col_part, nullptr, db, st))) return rc;
  const WgradBufs bufs{v.dy, scratch + 1, scratch + 2, v.status, v.partial};
  if ((rc = run_wgrad(h, batch, height, width, cout, cin, v.dyn, nullptr, v.x.hi, v.x.lo, sx, dw, true, bufs, st)))
    return rc;
  return check_status_word(v.status, st, "x or dy");
}

// ---------------------------------------------------------------- standalone producer layers (tests)
int dd_gen_layer(dd_handle h, const dd_gen_layer_desc* d, const float* x0, const float* x1, const float* w,
                 const float* bias, const float* const* bn, const float* add32, float* y32, void* out_hi, void* out_lo,
                 int32_t* launch_out, void* cuda_stream) {
  if (!h || !d || !x0 || !w || (d->c1 > 0 && !x1)) return fail(DD_ERR_INVALID, "null argument");
  if (!y32 && !(out_hi && out_lo)) return fail(DD_ERR_INVALID, "no output");
  const bool gemm = d->tokens > 0, xp = d->transposed != 0;
  const int c0 = d->c0, c1 = d->c1, cout = d->cout;
  const int cin = d->cin > 0 ? d->cin : c0 + c1;
  if ((d->taps != 1 && d->taps != 9) || (d->stride != 1 && d->stride != 2) || d->act < 0 || d->act > 3 || c0 < 8 ||
      c1 < 0 || c0 % 8 || c1 % 8 || cout < 8 || cin > c0 + c1 || (cin < c0 + c1 && c1 > 0))
    return fail(DD_ERR_INVALID, "bad layer descriptor");
  if (d->stride == 2 && (gemm || c1 > 0 || xp)) return fail(DD_ERR_INVALID, "stride 2: conv mode, one source");
  if (xp && (d->taps != 1 || c1 > 0 || d->ld_out > 0 || d->ch_off > 0))
    return fail(DD_ERR_INVALID, "transposed: one 1x1 source, dense output");
  const int ld_out = d->ld_out > 0 ? d->ld_out : (xp ? 4 * cout : cout);
  if (d->ch_off < 0 || d->ch_off + cout > ld_out || ld_out % 8 || d->ch_off % 8)  // 16-byte plane stores
    return fail(DD_ERR_INVALID, "bad output row width / channel offset");
  GenGrid g;
  if (gemm) {
    g = {1, (d->tokens + dd::TILE_W - 1) / dd::TILE_W, dd::TILE_W, d->tokens, 0, 0};
  } else {
    if (d->batch < 1 || d->height < 1 || d->width < 1) return fail(DD_ERR_INVALID, "empty geometry");
    g = {d->batch, d->height, d->width, 0, d->stride == 2 ? d->src_h : d->height, d->stride == 2 ? d->src_w : d->width};
    if (d->stride == 2 && ((g.src_h + 1) / 2 != g.H || (g.src_w + 1) / 2 != g.W))
      return fail(DD_ERR_INVALID, "stride 2: the output grid must be ceil(source / 2)");
  }
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  CUDA_TRY(cudaSetDevice(h->cfg.device));
  StandaloneCall call(h);
  int rc;
  if ((rc = call.begin(st))) return rc;
  float* scratch = reinterpret_cast<float*>(call.status) + 8;
  GenLayer L;
  if ((rc = pack_gen_weights(h, call.owned, L, w, "standalone layer", bn, bias, cin, cout, d->taps, xp,
                             cin < c0 ? c0 : 0, d->n_tile, st, scratch)))
    return rc;
  L.stride = d->stride;
  L.add_first = d->add_first;
  // sources: fp32 -> split planes; a GEMM's token rows are padded to whole 16-row "image" rows with zeros
  const size_t rows0 = gemm ? static_cast<size_t>(g.H) * g.W : static_cast<size_t>(g.B) * g.src_h * g.src_w;
  const size_t rows1 = gemm ? rows0 : static_cast<size_t>(g.B) * g.H * g.W;
  const size_t real0 = gemm ? static_cast<size_t>(d->tokens) : rows0, real1 = gemm ? real0 : rows1;
  Planes a0, a1;
  if ((rc = call.alloc(&a0.hi, rows0 * c0)) || (rc = call.alloc(&a0.lo, rows0 * c0))) return rc;
  if (gemm) {
    CUDA_TRY(cudaMemsetAsync(a0.hi, 0, rows0 * c0 * 2, st));
    CUDA_TRY(cudaMemsetAsync(a0.lo, 0, rows0 * c0 * 2, st));
  }
  if ((rc = split_planes(h, x0, a0.hi, a0.lo, real0 * c0, kProdScale, st))) return rc;
  if (c1 > 0) {
    if ((rc = call.alloc(&a1.hi, rows1 * c1)) || (rc = call.alloc(&a1.lo, rows1 * c1))) return rc;
    if (gemm) {
      CUDA_TRY(cudaMemsetAsync(a1.hi, 0, rows1 * c1 * 2, st));
      CUDA_TRY(cudaMemsetAsync(a1.lo, 0, rows1 * c1 * 2, st));
    }
    if ((rc = split_planes(h, x1, a1.hi, a1.lo, real1 * c1, kProdScale, st))) return rc;
  }
  float* partial = nullptr;  // a layer split along K (gen_parts)
  if (gen_parts(L.taps, gen_chunks(c0) + gen_chunks(c1)) > 1 &&
      (rc = call.alloc(&partial, static_cast<size_t>(g.B) * g.H * g.W * L.cout)))
    return rc;
  const Planes out{static_cast<__half*>(out_hi), static_cast<__half*>(out_lo)};
  GenLaunch info;
  if ((rc = launch_gen(h, L, d->act, g, a0, c0, a1, c1, y32, add32, (out_hi && out_lo) ? &out : nullptr,
                       d->ld_out > 0 ? d->ld_out : 0, d->ch_off, st, d->alt_tile, &info, partial)))
    return rc;
  if ((rc = call.finish(st, "an input or an output plane"))) return rc;
  if (launch_out) {
    launch_out[0] = info.nt;
    launch_out[1] = info.work;
    launch_out[2] = info.grid;
    launch_out[3] = info.parts;
  }
  return DD_OK;
}

int dd_window_attention(dd_handle h, const float* qkv, const float* qkv_bias, const float* table, float* out,
                        int32_t batch, int32_t height, int32_t width, int32_t num_heads, int32_t shift, int32_t kernel,
                        int32_t* launch_out, void* cuda_stream) {
  if (!h || !qkv || !qkv_bias || !table || !out) return fail(DD_ERR_INVALID, "null argument");
  if (batch < 1 || height < 1 || width < 1 || num_heads < 1 || shift < 0 || shift >= 7 || kernel < 0 || kernel > 2)
    return fail(DD_ERR_INVALID, "bad attention geometry");
  if (kernel == 2 && (num_heads & 1)) return fail(DD_ERR_UNSUPPORTED, "the wgmma window attention takes heads in pairs");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  CUDA_TRY(cudaSetDevice(h->cfg.device));
  const int C = 32 * num_heads;
  const size_t n = static_cast<size_t>(batch) * height * width * C;
  StandaloneCall call(h);
  int rc;
  if ((rc = call.begin(st))) return rc;
  Planes o;
  if ((rc = call.alloc(&o.hi, n)) || (rc = call.alloc(&o.lo, n))) return rc;
  const bool simt = kernel == 0 ? attn_simt(h, num_heads) : kernel == 1;
  int work = 0, grid = 0;
  if ((rc = launch_attention(h, qkv, qkv_bias, table, o, batch, height, width, C, num_heads, shift, simt, st, &work,
                             &grid)))
    return rc;
  dd::join_planes_kernel<<<grid_of(n), 256, 0, st>>>(o.hi, o.lo, out, n, 1.f / kTokScale);
  if ((rc = check_launch("join_planes"))) return rc;
  if ((rc = call.finish(st, "qkv or the attention output"))) return rc;
  if (launch_out) {
    launch_out[0] = work;
    launch_out[1] = grid;
  }
  return DD_OK;
}

int dd_factor_attention(dd_handle h, const float* qkv, const float* const* crpe_w, const float* const* crpe_b, float* out,
                        int32_t batch, int32_t height, int32_t width, int32_t channels, int32_t* launch_out,
                        void* cuda_stream) {
  if (!h || !qkv || !crpe_w || !crpe_b || !out) return fail(DD_ERR_INVALID, "null argument");
  for (int g = 0; g < 3; ++g)
    if (!crpe_w[g] || !crpe_b[g]) return fail(DD_ERR_INVALID, "null argument");
  if (batch < 1 || height < 1 || width < 1 || channels < 1) return fail(DD_ERR_INVALID, "bad attention geometry");
  if (channels % kMpHeads != 0 || channels / kMpHeads > dd::KTV_CH_MAX)
    return fail(DD_ERR_UNSUPPORTED, "factorised attention: channels must be a multiple of 8 (8 heads), at most 512");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  CUDA_TRY(cudaSetDevice(h->cfg.device));
  const int C = channels, Ch = C / kMpHeads;
  const size_t n = static_cast<size_t>(batch) * height * width * C;
  const size_t nk = static_cast<size_t>(batch) * kMpHeads * Ch * Ch;
  StandaloneCall call(h);
  int rc;
  if ((rc = call.begin(st))) return rc;
  float *cw = nullptr, *cb = nullptr;
  if ((rc = pack_crpe(call.owned, crpe_w, crpe_b, C, cw, cb, st))) return rc;
  FactorAttBufs bf;
  if ((rc = call.alloc(&bf.part_m, static_cast<size_t>(batch) * kMpChunksMax * C)) ||
      (rc = call.alloc(&bf.part_s, static_cast<size_t>(batch) * kMpChunksMax * C)) ||
      (rc = call.alloc(&bf.colinv, static_cast<size_t>(batch) * C)) ||
      (rc = call.alloc(&bf.part_ktv, nk * kMpChunksMax)) || (rc = call.alloc(&bf.ktv, nk)))
    return rc;
  Planes o;
  if ((rc = call.alloc(&o.hi, n)) || (rc = call.alloc(&o.lo, n))) return rc;
  int info[4];
  if ((rc = run_factor_att(h, qkv, cw, cb, bf, o, batch, height, width, C, st, info))) return rc;
  dd::join_planes_kernel<<<grid_of(n), 256, 0, st>>>(o.hi, o.lo, out, n, 1.f / kTokScale);
  if ((rc = check_launch("join_planes"))) return rc;
  if ((rc = call.finish(st, "qkv or the attention output"))) return rc;
  if (launch_out)
    for (int i = 0; i < 4; ++i) launch_out[i] = info[i];
  return DD_OK;
}

int dd_depthwise_conv(dd_handle h, const float* x, const float* w, const float* bias, const float* const* bn, float* y32,
                      void* out_hi, void* out_lo, int32_t batch, int32_t height, int32_t width, int32_t channels,
                      int32_t stride, int32_t act, int32_t residual, int32_t* launch_out, void* cuda_stream) {
  if (!h || !x || !w) return fail(DD_ERR_INVALID, "null argument");
  if (!y32 && !(out_hi && out_lo)) return fail(DD_ERR_INVALID, "no output");
  if (bn && bias) return fail(DD_ERR_INVALID, "a bias or an eval-BN, not both");
  if (bn && !(bn[0] && bn[1] && bn[2] && bn[3])) return fail(DD_ERR_INVALID, "null argument");
  if (batch < 1 || height < 1 || width < 1 || channels < 1 || (stride != 1 && stride != 2) || (act != 0 && act != 3) ||
      (residual != 0 && residual != 1) || (residual && stride != 1))
    return fail(DD_ERR_INVALID, "bad depthwise conv descriptor");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  CUDA_TRY(cudaSetDevice(h->cfg.device));
  StandaloneCall call(h);
  int rc;
  if ((rc = call.begin(st))) return rc;
  DwLayer L;
  if ((rc = pack_dw(call.owned, L, w, bn, bias, channels, 3, "standalone depthwise conv", st))) return rc;
  const Planes o{static_cast<__half*>(out_hi), static_cast<__half*>(out_lo)};
  int info[2];
  if ((rc = run_dw(h, L, x, batch, height, width, stride, act, residual, y32, (out_hi && out_lo) ? &o : nullptr, st,
                   info)))
    return rc;
  if ((rc = call.finish(st, "the depthwise conv output"))) return rc;
  if (launch_out) {
    launch_out[0] = info[0];
    launch_out[1] = info[1];
  }
  return DD_OK;
}

int dd_layer_norm(dd_handle h, const float* x, const float* gamma, const float* beta, float* out, int32_t tokens,
                  int32_t channels, float eps, void* cuda_stream) {
  if (!h || !x || !gamma || !beta || !out) return fail(DD_ERR_INVALID, "null argument");
  if (tokens < 1 || channels < 1 || !(eps > 0.f)) return fail(DD_ERR_INVALID, "bad LayerNorm geometry");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  CUDA_TRY(cudaSetDevice(h->cfg.device));
  const size_t n = static_cast<size_t>(tokens) * channels;
  StandaloneCall call(h);
  int rc;
  if ((rc = call.begin(st))) return rc;
  Planes o;
  if ((rc = call.alloc(&o.hi, n)) || (rc = call.alloc(&o.lo, n))) return rc;
  if ((rc = run_ln_generic(h, channels, x, gamma, beta, o, tokens, eps, st))) return rc;
  dd::join_planes_kernel<<<grid_of(n), 256, 0, st>>>(o.hi, o.lo, out, n, 1.f / kTokScale);
  if ((rc = check_launch("join_planes"))) return rc;
  return call.finish(st, "x or the LayerNorm output");
}

int dd_swin_patch_embed(dd_handle h, const float* rgb, const float* w, const float* bias, const float* gamma,
                        const float* beta, float* out, int32_t batch, int32_t height, int32_t width, int32_t embed,
                        void* cuda_stream) {
  if (!h || !rgb || !w || !bias || !gamma || !beta || !out) return fail(DD_ERR_INVALID, "null argument");
  if (batch < 1 || height < 1 || width < 1 || embed < 1) return fail(DD_ERR_INVALID, "bad patch embedding geometry");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  CUDA_TRY(cudaSetDevice(h->cfg.device));
  StandaloneCall call(h);
  int rc;
  if ((rc = call.begin(st))) return rc;
  if ((rc = run_patch_embed(h, embed, rgb, w, bias, gamma, beta, out, batch, height, width, st))) return rc;
  return call.finish(st, "the patch embedding");
}

int dd_swin_layer_norm(dd_handle h, const float* x, const float* gamma, const float* beta, float* out, float* nchw_out,
                       int32_t tokens, int32_t channels, int32_t hw, void* cuda_stream) {
  if (!h || !x || !gamma || !beta || !out) return fail(DD_ERR_INVALID, "null argument");
  if (tokens < 1 || channels < 1 || (nchw_out && (hw < 1 || tokens % hw != 0)))
    return fail(DD_ERR_INVALID, "bad LayerNorm geometry");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  CUDA_TRY(cudaSetDevice(h->cfg.device));
  const size_t n = static_cast<size_t>(tokens) * channels;
  StandaloneCall call(h);
  int rc;
  if ((rc = call.begin(st))) return rc;
  Planes o;
  if ((rc = call.alloc(&o.hi, n)) || (rc = call.alloc(&o.lo, n))) return rc;
  if ((rc = run_ln(h, channels, x, gamma, beta, o, tokens, nchw_out, nchw_out ? hw : 0, st))) return rc;
  dd::join_planes_kernel<<<grid_of(n), 256, 0, st>>>(o.hi, o.lo, out, n, 1.f / kTokScale);
  if ((rc = check_launch("join_planes"))) return rc;
  return call.finish(st, "x or the LayerNorm output");
}

int dd_swin_patch_merge(dd_handle h, const float* x, const float* gamma, const float* beta, float* out, int32_t batch,
                        int32_t height, int32_t width, int32_t channels, void* cuda_stream) {
  if (!h || !x || !gamma || !beta || !out) return fail(DD_ERR_INVALID, "null argument");
  if (batch < 1 || height < 1 || width < 1 || channels < 1) return fail(DD_ERR_INVALID, "bad patch merging geometry");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  CUDA_TRY(cudaSetDevice(h->cfg.device));
  const size_t n = static_cast<size_t>(batch) * ((height + 1) / 2) * ((width + 1) / 2) * 4 * channels;
  StandaloneCall call(h);
  int rc;
  if ((rc = call.begin(st))) return rc;
  Planes o;
  if ((rc = call.alloc(&o.hi, n)) || (rc = call.alloc(&o.lo, n))) return rc;
  if ((rc = run_merge_ln(h, channels, x, gamma, beta, o, batch, height, width, st))) return rc;
  dd::join_planes_kernel<<<grid_of(n), 256, 0, st>>>(o.hi, o.lo, out, n, 1.f / kTokScale);
  if ((rc = check_launch("join_planes"))) return rc;
  return call.finish(st, "x or the patch merging output");
}

int dd_conv_groupnorm(dd_handle h, const dd_conv_gn_desc* d, const float* x, const float* w, const float* b,
                      const float* gamma, const float* beta, const float* cond, const float* temb, float* latent,
                      float* y32, float* mean_rstd, float* out, void* cuda_stream) {
  if (!h || !d || !x || !w || !b || !gamma || !beta) return fail(DD_ERR_INVALID, "null argument");
  const int B = d->batch, cin = d->cin, cout = d->cout, H = d->height, W = d->width, mode = d->mode;
  const int sid = shape_id(cin, cout);
  if (sid < 0 || (cin == 256 && cout == 256)) return fail(DD_ERR_UNSUPPORTED, "not a GroupNorm'd conv of the DDIM loop");
  if (B < 1 || H < 1 || W < 1 || mode < 0 || mode > 3) return fail(DD_ERR_INVALID, "bad conv / GroupNorm descriptor");
  if ((mode == 0 && cout != 64) || ((mode == 1 || mode == 2) && cout != 256) || (mode == 3 && cout != 16))
    return fail(DD_ERR_UNSUPPORTED, "the loop applies that mode to another conv shape");
  if ((mode == 1 || mode == 2) && (!cond || !temb)) return fail(DD_ERR_INVALID, "null condition or time embedding");
  if (mode == 2 && (d->cond_h < 1 || d->cond_w < 1 || (d->up_qpb != 4 && d->up_qpb != 1)))
    return fail(DD_ERR_INVALID, "bad up-add geometry");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  CUDA_TRY(cudaSetDevice(h->cfg.device));
  const int P = H * W;
  const size_t BP = static_cast<size_t>(B) * P;
  const size_t nw = static_cast<size_t>(cin) * cout * 9;
  const int ch = mode == 2 ? d->cond_h : H, cw = mode == 2 ? d->cond_w : W;
  StandaloneCall call(h);
  int rc;
  if ((rc = call.begin(st))) return rc;
  float* scratch = reinterpret_cast<float*>(call.status) + 8;
  const bool simt = (h->cfg.flags & DD_FLAG_SIMT_CONV) != 0;
  const int tiles_img = simt ? ((W + dd::TILE_W - 1) / dd::TILE_W) * ((H + dd::TILE_H - 1) / dd::TILE_H)
                             : ((W + dd::HALO_TW - 1) / dd::HALO_TW) * ((H + dd::HALO_TH - 1) / dd::HALO_TH);
  float *xn, *yn, *wsimt, *mr, *cn = nullptr, *xl = nullptr, *eps = nullptr;
  double* partial;
  Planes xs, wp, o;
  if ((rc = call.alloc(&xn, BP * cin)) || (rc = call.alloc(&xs.hi, BP * cin)) || (rc = call.alloc(&xs.lo, BP * cin)) ||
      (rc = call.alloc(&yn, BP * cout)) || (rc = call.alloc(&wp.hi, nw)) || (rc = call.alloc(&wp.lo, nw)) ||
      (rc = call.alloc(&wsimt, nw)) || (rc = call.alloc(&partial, static_cast<size_t>(B) * tiles_img * 8)) ||
      (rc = call.alloc(&mr, static_cast<size_t>(B) * 8)) || (rc = call.alloc(&o.hi, BP * cout)) ||
      (rc = call.alloc(&o.lo, BP * cout)))
    return rc;
  // the conv: fp32 NCHW -> NHWC split planes at the loop's scale of that input (the latent's, or the activations'), the
  // weights at their own power-of-two scale, and the loop's epilogue
  if ((rc = transpose_in(x, xn, B, cin, P, st))) return rc;
  const float sx = cin == 16 ? kXScale : kActScale;
  float sw;
  if ((rc = split_scale_of(w, nw, scratch, st, &sw))) return rc;
  if ((rc = split_planes(h, xn, xs.hi, xs.lo, BP * cin, sx, st))) return rc;
  dd::pack_conv_weight_kernel<<<128, 256, 0, st>>>(w, wp.hi, wp.lo, wsimt, cout, cin, sw);
  if ((rc = check_launch("pack_conv_weight"))) return rc;
  dd::ConvArgs a;
  a.B = B;
  a.H = H;
  a.W = W;
  a.bias = b;
  a.acc_scale = 1.f / (sx * sw);
  a.y32 = yn;
  a.stats_partial = partial;
  a.out_hi = a.out_lo = nullptr;
  a.split_scale = 1.f;
  a.status = call.status;
  CUtensorMap mb_hi{}, mb_lo{};
  if (!simt) {
    if ((rc = make_weight_map(&mb_hi, wp.hi, cout, cin, 9, kHaloBK[sid], cout))) return rc;
    if ((rc = make_weight_map(&mb_lo, wp.lo, cout, cin, 9, kHaloBK[sid], cout))) return rc;
  }
  if ((rc = launch_conv3x3(sid, dd::EPI_F32_STATS, simt, a, xs.hi, xs.lo, sx, wsimt, mb_hi, mb_lo, h->sm_count, st)))
    return rc;
  if ((rc = check_launch("conv3x3"))) return rc;
  dd::gn_finalize_kernel<<<B * 4, 256, 0, st>>>(partial, a.tiles_x * a.tiles_y, nullptr, 0,
                                                 1.0 / (static_cast<double>(P) * (cout / 4)), 1e-5f, mr);
  if ((rc = check_launch("gn_finalize"))) return rc;
  // the apply kernel the loop runs after this conv
  if (mode == 3) {
    dd::FinalArgs f;
    f.y = yn;
    f.mean_rstd = mr;
    f.gamma = gamma;
    f.beta = beta;
    f.x = nullptr;
    f.x_hi = o.hi;
    f.x_lo = o.lo;
    f.eps_out = nullptr;
    f.cx = d->c_x;
    f.ce = d->c_eps;
    f.scale = kXScale;
    f.P = P;
    f.status = call.status;
    if (latent) {
      if ((rc = call.alloc(&xl, BP * 16)) || (rc = transpose_in(latent, xl, B, 16, P, st))) return rc;
      f.x = xl;
    } else {
      if ((rc = call.alloc(&eps, BP * 16))) return rc;
      f.eps_out = eps;
    }
    launch_final(f, B, st);
    if ((rc = check_launch("gn_relu_ddim"))) return rc;
  } else {
    dd::ApplyArgs g;
    g.y = yn;
    g.mean_rstd = mr;
    g.gamma = gamma;
    g.beta = beta;
    g.cond = nullptr;
    g.temb = temb;
    g.temb_bstride = 256;
    g.H = H;
    g.W = W;
    g.ch = ch;
    g.cw = cw;
    g.ry = H > 1 ? static_cast<float>(ch - 1) / static_cast<float>(H - 1) : 0.f;
    g.rx = W > 1 ? static_cast<float>(cw - 1) / static_cast<float>(W - 1) : 0.f;
    g.out_hi = o.hi;
    g.out_lo = o.lo;
    g.scale = kActScale;
    g.status = call.status;
    if (mode != 0) {
      const size_t nc = static_cast<size_t>(B) * ch * cw * 256;
      if ((rc = call.alloc(&cn, nc)) || (rc = transpose_in(cond, cn, B, 256, ch * cw, st))) return rc;
      g.cond = cn;
    }
    if (mode == 0) launch_apply<64, 0>(g, B, 0, st);
    else if (mode == 1) launch_apply<256, 1>(g, B, 0, st);
    else launch_apply<256, 2>(g, B, d->up_qpb, st);
    if ((rc = check_launch("gn_apply"))) return rc;
  }
  // outputs, NCHW
  if (y32 && (rc = transpose_out(yn, y32, B, cout, P, st))) return rc;
  if (mean_rstd) CUDA_TRY(cudaMemcpyAsync(mean_rstd, mr, static_cast<size_t>(B) * 32, cudaMemcpyDeviceToDevice, st));
  if (xl && (rc = transpose_out(xl, latent, B, 16, P, st))) return rc;
  if (out) {
    const float* src = eps;
    if (!eps) {  // the split planes the apply kernel wrote, joined back in place of the conv output
      dd::join_planes_kernel<<<grid_of(BP * cout), 256, 0, st>>>(o.hi, o.lo, yn, BP * cout,
                                                                 1.f / (mode == 3 ? kXScale : kActScale));
      if ((rc = check_launch("join_planes"))) return rc;
      src = yn;
    }
    if ((rc = transpose_out(src, out, B, cout, P, st))) return rc;
  }
  return call.finish(st, "x or the GroupNorm'd output");
}

int dd_bench_pred_fold(dd_handle h, int32_t iters, float* ms_out, void* workspace, size_t workspace_bytes,
                       void* cuda_stream) {
  if (!h || !ms_out || iters < 1) return fail(DD_ERR_INVALID, "bad argument");
  if (!h->weights_ready) return fail(DD_ERR_INVALID, "dd_finalize_weights has not been called");
  if (!fold_active(h)) return fail(DD_ERR_UNSUPPORTED, "this engine runs convB and pred.0 as two convs");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  int rc;
  if ((rc = enter_workspace(h, workspace, workspace_bytes))) return rc;
  // whatever the planes currently hold is fine for timing: MMA time is data independent
  return time_per_call(st, 2, iters, ms_out, [&]() { return run_fold(h, st); });
}

int dd_bench_conv(dd_handle h, int32_t cin, int32_t cout, int32_t iters, float* ms_out, void* workspace,
                  size_t workspace_bytes, void* cuda_stream) {
  if (!h || !ms_out || iters < 1) return fail(DD_ERR_INVALID, "bad argument");
  if (!h->weights_ready) return fail(DD_ERR_INVALID, "dd_finalize_weights has not been called");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  int rc;
  if ((rc = enter_workspace(h, workspace, workspace_bytes))) return rc;
  int layer = -1;
  for (int i = 0; i < 6; ++i)
    if (h->L[i].sid >= 0 && kShapes[h->L[i].sid].cin == cin && kShapes[h->L[i].sid].cout == cout) layer = i;
  if (layer < 0) return fail(DD_ERR_UNSUPPORTED, "no packed layer with that shape in this engine variant");
  const bool split_out = (cin == 256 && cout == 256);
  // whatever the planes currently hold is fine for timing: MMA time is data independent
  const __half* in_hi = cin == 16 ? h->xs_hi : h->S_hi[1];
  const __half* in_lo = cin == 16 ? h->xs_lo : h->S_lo[1];
  return time_per_call(st, 2, iters, ms_out, [&]() {
    return run_conv(h, layer, in_hi, in_lo, kActScale, split_out ? dd::EPI_SPLIT : dd::EPI_F32_STATS, h->Y, h->stats[0],
                    h->S_hi[0], h->S_lo[0], st);
  });
}

}  // extern "C"
