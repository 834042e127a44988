// MPViT backbone (reference src/model/backbone/mpvit.py:57-741): the pieces that are not GEMMs.  Every 1x1 conv and Linear
// of the network runs on convgen_wgmma_kernel (3-pass fp16 split on wgmma); what is left is HBM/L2-bound pointwise and
// stencil work on fp32 NHWC token maps [B, H, W, C]:
//   dwconv_nhwc_kernel        depthwise k x k (stride 1 / 2), + bias / folded eval-BN, Hardswish, residual (ConvPosEnc),
//                             fp32 and / or fp16 hi/lo plane outputs                      (:125-175, :241-259, :482-532)
//   ln_split_generic_kernel   LayerNorm(C) for any C <= 512 -> planes                     (:396-436)
//   ksoftmax_partial_kernel   softmax of k over the TOKEN axis: per-chunk online max / sum            (:374)
//   ktv_{partial,combine}     k_softmax^T v per (image, head): per-chunk partial [Ch x Ch] sums (the chunk maxima are
//                             folded on the way in), ordered combine                              (:375)
//   factor_att_apply_kernel   scale * q (k^T v) + q * depthwise_conv_{3,5,7}(v)  -> planes (:376-386, :262-330)
// All reductions over tokens run in a fixed order (chunk partials, then an ordered combine): results are bit-reproducible.
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

#include "kernels.cuh"
#include "swin.cuh"  // warp_sum, warp_ln_centre

namespace dd {

__device__ __forceinline__ float hardswish_f(float v) { return v * fminf(fmaxf(v + 3.f, 0.f), 6.f) * (1.f / 6.f); }

// ------------------------------------------------------------------------------------------------ depthwise conv
struct DwArgs {
  const float* x;     // fp32 NHWC [B, H, W, C]
  const float* w;     // [KS*KS][C] tap-major (eval-BN scale folded in)
  const float* bias;  // [C]: conv bias / folded BN shift (zeros if neither)
  float* y32;         // nullable: fp32 NHWC [B, Ho, Wo, C]
  __half* out_hi;     // nullable: fp16 hi/lo planes of split_scale * y
  __half* out_lo;
  float split_scale;
  int B, H, W, C, Ho, Wo, stride;
  int act;            // 0 none, 3 Hardswish
  int residual;       // 1: y += x (ConvPosEnc; stride 1 only)
  int* status;
};

// one thread = one output pixel x 4 channels (float4 loads along the channel axis are coalesced across the warp)
template <int KS>
__global__ void __launch_bounds__(256) dwconv_nhwc_kernel(const DwArgs a) {
  const int C4 = a.C >> 2;
  const size_t total = static_cast<size_t>(a.B) * a.Ho * a.Wo * C4;
  bool ov = false;
  for (size_t i = blockIdx.x * static_cast<size_t>(256) + threadIdx.x; i < total; i += static_cast<size_t>(gridDim.x) * 256) {
    const int c4 = static_cast<int>(i % C4);
    const size_t px = i / C4;
    const int ox = static_cast<int>(px % a.Wo), oy = static_cast<int>((px / a.Wo) % a.Ho);
    const int b = static_cast<int>(px / (static_cast<size_t>(a.Wo) * a.Ho));
    float4 acc = __ldg(reinterpret_cast<const float4*>(a.bias) + c4);
    const int iy0 = oy * a.stride - KS / 2, ix0 = ox * a.stride - KS / 2;
    const float* img = a.x + static_cast<size_t>(b) * a.H * a.W * a.C;
#pragma unroll
    for (int ky = 0; ky < KS; ++ky) {
      const int iy = iy0 + ky;
      if (iy < 0 || iy >= a.H) continue;
#pragma unroll
      for (int kx = 0; kx < KS; ++kx) {
        const int ix = ix0 + kx;
        if (ix < 0 || ix >= a.W) continue;
        const float4 v = __ldg(reinterpret_cast<const float4*>(img + (static_cast<size_t>(iy) * a.W + ix) * a.C) + c4);
        const float4 w = __ldg(reinterpret_cast<const float4*>(a.w + (ky * KS + kx) * a.C) + c4);
        acc.x = fmaf(v.x, w.x, acc.x);
        acc.y = fmaf(v.y, w.y, acc.y);
        acc.z = fmaf(v.z, w.z, acc.z);
        acc.w = fmaf(v.w, w.w, acc.w);
      }
    }
    if (a.residual) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(img + (static_cast<size_t>(oy) * a.W + ox) * a.C) + c4);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    if (a.act == 3) {
      acc.x = hardswish_f(acc.x); acc.y = hardswish_f(acc.y); acc.z = hardswish_f(acc.z); acc.w = hardswish_f(acc.w);
    }
    const size_t o = px * a.C + 4 * c4;
    if (a.y32) *reinterpret_cast<float4*>(a.y32 + o) = acc;
    if (a.out_hi) {
      __half h[4], l[4];
      split_f16(acc.x, a.split_scale, h[0], l[0], ov);
      split_f16(acc.y, a.split_scale, h[1], l[1], ov);
      split_f16(acc.z, a.split_scale, h[2], l[2], ov);
      split_f16(acc.w, a.split_scale, h[3], l[3], ov);
      *reinterpret_cast<uint2*>(a.out_hi + o) = *reinterpret_cast<const uint2*>(h);
      *reinterpret_cast<uint2*>(a.out_lo + o) = *reinterpret_cast<const uint2*>(l);
    }
  }
  if (ov) atomicOr(a.status, 1);
}

// depthwise weights [C][1][K][K] (optionally scaled per channel) -> tap-major [KD*KD][C] at the centre of a KD x KD
// window (KD >= K; the crpe table holds its 3 / 5 / 7 windows in one 7 x 7 layout), channel offset c0 of C_total
__global__ void pack_dw_weight_kernel(const float* __restrict__ w, const float* __restrict__ ch_scale, float* __restrict__ out,
                                      int C, int K, int KD, int c0, int C_total) {
  const int n = C * K * K;
  const int off = (KD - K) / 2;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int kx = i % K, ky = (i / K) % K, c = i / (K * K);
    out[((ky + off) * KD + kx + off) * C_total + c0 + c] = w[i] * (ch_scale ? ch_scale[c] : 1.f);
  }
}

// ------------------------------------------------------------------------------------------------ LayerNorm, any width
// one warp per token, C <= 32 * VMAX (VMAX values per lane: 2 / 4 / 8 / 16 picked by the host from C)
template <int VMAX>
__global__ void __launch_bounds__(256) ln_split_generic_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                                               const float* __restrict__ beta, __half* __restrict__ hi,
                                                               __half* __restrict__ lo, float scale, int M, int C, float eps,
                                                               int* status) {
  const int token = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (token >= M) return;
  const float* row = x + static_cast<size_t>(token) * C;
  float v[VMAX];
#pragma unroll
  for (int i = 0; i < VMAX; ++i) {
    const int c = lane + 32 * i;
    v[i] = c < C ? row[c] : 0.f;
  }
  const float rstd = warp_ln_centre(v, C, eps);  // two-part mean (swin.cuh)
  bool ov = false;
#pragma unroll
  for (int i = 0; i < VMAX; ++i) {
    const int c = lane + 32 * i;
    if (c < C) {
      const float y = v[i] * rstd * gamma[c] + beta[c];
      __half h, l;
      split_f16(y, scale, h, l, ov);
      hi[static_cast<size_t>(token) * C + c] = h;
      lo[static_cast<size_t>(token) * C + c] = l;
    }
  }
  if (ov) atomicOr(status, 1);
}

// ------------------------------------------------------------------------------------------------ factorised attention
// qkv: fp32 [B][N][3C] (q | k | v, each head-major h * Ch + c).  Token chunks: chunk j of image b covers tokens
// [j * tpc, min(N, (j + 1) * tpc)).  Launch order per layer: ksoftmax_partial -> ktv_partial -> ktv_combine ->
// factor_att_apply.

// per (image, chunk, channel of k): running max m and sum s = sum exp(k - m) over the chunk's tokens.  256 threads =
// (256 / C) token slices x C channels; the slices of a channel are merged in slice order.
__global__ void __launch_bounds__(256) ksoftmax_partial_kernel(const float* __restrict__ qkv, float* __restrict__ part_m,
                                                               float* __restrict__ part_s, int N, int C, int chunks, int tpc) {
  __shared__ float sm_m[256], sm_s[256];
  const int b = blockIdx.y, ch = blockIdx.x;
  const int n0 = ch * tpc, n1 = min(N, n0 + tpc);
  const float* base = qkv + static_cast<size_t>(b) * N * 3 * C + C;
  const int nsl = C >= 256 ? 1 : 256 / C;
  const int slice = nsl == 1 ? 0 : threadIdx.x / C;
  const int c_first = nsl == 1 ? threadIdx.x : threadIdx.x - slice * C;
  for (int c = c_first; c < C; c += 256) {  // more than one trip only when C > 256 (then nsl == 1)
    float m = -INFINITY, s = 0.f;
    if (slice < nsl) {
      int n = n0 + slice;
      for (; n + 3 * nsl < n1; n += 4 * nsl) {  // four independent loads in flight, one rescale per group
        const float k0 = base[static_cast<size_t>(n) * 3 * C + c], k1 = base[static_cast<size_t>(n + nsl) * 3 * C + c];
        const float k2 = base[static_cast<size_t>(n + 2 * nsl) * 3 * C + c], k3 = base[static_cast<size_t>(n + 3 * nsl) * 3 * C + c];
        const float mm = fmaxf(fmaxf(fmaxf(k0, k1), fmaxf(k2, k3)), m);
        s = s * expf(m - mm) + ((expf(k0 - mm) + expf(k1 - mm)) + (expf(k2 - mm) + expf(k3 - mm)));
        m = mm;
      }
      for (; n < n1; n += nsl) {
        const float k = base[static_cast<size_t>(n) * 3 * C + c];
        const float mm = fmaxf(m, k);
        s = s * expf(m - mm) + expf(k - mm);
        m = mm;
      }
    }
    if (nsl > 1) {
      __syncthreads();
      if (slice < nsl) {
        sm_m[threadIdx.x] = m;
        sm_s[threadIdx.x] = s;
      }
      __syncthreads();
      if (slice == 0) {
        for (int j = 1; j < nsl; ++j) {
          const float mj = sm_m[j * C + c], sj = sm_s[j * C + c];
          if (sj > 0.f) {
            const float mm = fmaxf(m, mj);
            s = s * expf(m - mm) + sj * expf(mj - mm);
            m = mm;
          }
        }
      }
    }
    if (slice == 0) {
      part_m[(static_cast<size_t>(b) * chunks + ch) * C + c] = m;
      part_s[(static_cast<size_t>(b) * chunks + ch) * C + c] = s;
    }
  }
}

// per (image, group of HB heads, chunk): part[h][c1][c2] = sum over the chunk's tokens of exp(k[n][h][c1] - colmax) * v[n][h][c2].
// The block first folds the chunk partials of its k columns into colmax (chunk 0's blocks also store 1 / sum exp for
// ktv_combine).  256 threads own <= KTV_NP (h, c1, c2) entries each; the host picks HB with HB Ch^2 <= 4096 and
// HB Ch <= KTV_W, so that the high-resolution stages (Ch = 8, 16) take all 8 heads in one block (one block per head left
// 64 threads with 32 FMAs between two barriers).  Tokens are staged 32 at a time.
constexpr int KTV_NP = 16;
constexpr int KTV_T = 32;
constexpr int KTV_W = 160;
constexpr int KTV_CH_MAX = 64;
__global__ void __launch_bounds__(256) ktv_partial_kernel(const float* __restrict__ qkv, const float* __restrict__ part_m,
                                                          const float* __restrict__ part_s, float* __restrict__ colinv,
                                                          float* __restrict__ part, int N, int C, int Ch, int heads, int HB,
                                                          int chunks, int tpc) {
  __shared__ float ek[KTV_T][KTV_W];
  __shared__ float vv[KTV_T][KTV_W];
  __shared__ float cmax[KTV_W];
  const int ch = blockIdx.x, b = blockIdx.z;
  const int hb0 = blockIdx.y * HB, nh = min(HB, heads - hb0);
  const int width = nh * Ch, c_base = hb0 * Ch;
  const int n0 = ch * tpc, n1 = min(N, n0 + tpc);
  const int per_head = Ch * Ch, pairs = nh * per_head;
  if (threadIdx.x < width) {
    const int c = c_base + threadIdx.x;
    float M = -INFINITY;
    for (int j = 0; j < chunks; ++j) M = fmaxf(M, part_m[(static_cast<size_t>(b) * chunks + j) * C + c]);
    cmax[threadIdx.x] = M;
    if (ch == 0) {
      float S = 0.f;
      for (int j = 0; j < chunks; ++j) {
        const size_t o = (static_cast<size_t>(b) * chunks + j) * C + c;
        S += part_s[o] * expf(part_m[o] - M);
      }
      colinv[b * C + c] = 1.f / S;
    }
  }
  float acc[KTV_NP];
  int off[KTV_NP];  // column of exp(k) | column of v << 16 (both inside the block's [width] slice)
#pragma unroll
  for (int i = 0; i < KTV_NP; ++i) {
    acc[i] = 0.f;
    const int p = threadIdx.x + 256 * i;
    if (p < pairs) {
      const int hl = p / per_head, r = p - hl * per_head;
      off[i] = (hl * Ch + r / Ch) | ((hl * Ch + r % Ch) << 16);
    } else {
      off[i] = -1;
    }
  }
  __syncthreads();
  const float* base = qkv + static_cast<size_t>(b) * N * 3 * C + c_base;
  for (int t0 = n0; t0 < n1; t0 += KTV_T) {
    for (int i = threadIdx.x; i < KTV_T * width; i += 256) {
      const int tok = i / width, c = i - tok * width;
      const int n = t0 + tok;
      float e = 0.f, v = 0.f;
      if (n < n1) {
        const float* row = base + static_cast<size_t>(n) * 3 * C;
        e = expf(row[C + c] - cmax[c]);
        v = row[2 * C + c];
      }
      ek[tok][c] = e;
      vv[tok][c] = v;
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < KTV_NP; ++i) {
      if (off[i] >= 0) {
        const int c1 = off[i] & 0xffff, c2 = off[i] >> 16;
        float s = acc[i];
#pragma unroll 8
        for (int tok = 0; tok < KTV_T; ++tok) s = fmaf(ek[tok][c1], vv[tok][c2], s);
        acc[i] = s;
      }
    }
    __syncthreads();
  }
  float* dst = part + (static_cast<size_t>(b) * chunks + ch) * heads * per_head + static_cast<size_t>(hb0) * per_head;
#pragma unroll
  for (int i = 0; i < KTV_NP; ++i)
    if (off[i] >= 0) dst[threadIdx.x + 256 * i] = acc[i];
}

// sum over the chunks (8 chunk slices per entry, merged in slice order), times 1 / sum exp of the k column:
// ktv[b][h][c1][c2].  Block = 32 entries x 8 slices.
__global__ void __launch_bounds__(256) ktv_combine_kernel(const float* __restrict__ part, const float* __restrict__ colinv,
                                                          float* __restrict__ ktv, int C, int Ch, int heads, int chunks) {
  __shared__ float red[8][32];
  const int b = blockIdx.y;
  const int total = heads * Ch * Ch;
  const int lane = threadIdx.x & 31, slice = threadIdx.x >> 5;
  const int p = blockIdx.x * 32 + lane;
  float s = 0.f;
  if (p < total)
    for (int j = slice; j < chunks; j += 8) s += part[(static_cast<size_t>(b) * chunks + j) * total + p];
  red[slice][lane] = s;
  __syncthreads();
  if (slice == 0 && p < total) {
#pragma unroll
    for (int j = 1; j < 8; ++j) s += red[j][lane];
    const int h = p / (Ch * Ch), c1 = (p / Ch) % Ch;
    ktv[static_cast<size_t>(b) * total + p] = s * colinv[b * C + h * Ch + c1];
  }
}

// out[n][h Ch + c] = scale * sum_c' q[n][h][c'] ktv[h][c'][c] + q[n][h][c] * (dwconv_win(h)(v)[n][h Ch + c] + bias)
// One work item = one token x 4 channels: the convolution walks the (2r + 1)^2 window of the widest head among its channels
// with float4 loads (the table holds every channel's window centred in a 7 x 7 layout, zeros outside), k^T v and the
// token's q row come through L1.  One block = a 16 x 8 pixel tile x 64 channels, so that the window overlap of neighbouring
// pixels in BOTH directions is served by L1 (22 x 14 x 256 B = 79 KB per block: 2.4x the tile instead of the 10x that
// 16-token row segments pull from L2).
struct FactorApplyArgs {
  const float* qkv;     // [B][N][3C]
  const float* ktv;     // [B][heads][Ch][Ch]
  const float* crpe_w;  // [49][C]
  const float* crpe_b;  // [C]
  __half* out_hi;       // planes [B][N][C] of split_scale * out
  __half* out_lo;
  float split_scale, scale;
  int B, H, W, C, Ch, heads;
  int radius[16];       // per head: window / 2
  int* status;
};
constexpr int FA_TX = 16, FA_TY = 8, FA_CC = 16;  // pixel tile, float4 channel groups per block
__global__ void __launch_bounds__(256) factor_att_apply_kernel(const FactorApplyArgs a) {
  const int N = a.H * a.W, C4 = a.C >> 2;
  const int tiles_x = (a.W + FA_TX - 1) / FA_TX, tiles_y = (a.H + FA_TY - 1) / FA_TY, cchunks = (C4 + FA_CC - 1) / FA_CC;
  int blk = blockIdx.x;
  const int cchunk = blk % cchunks; blk /= cchunks;
  const int tx = blk % tiles_x; blk /= tiles_x;
  const int ty = blk % tiles_y;
  const int b = blk / tiles_y;
  const int cc = min(FA_CC, C4 - cchunk * FA_CC);
  bool ov = false;
  for (int it = threadIdx.x; it < FA_TX * FA_TY * cc; it += 256) {
    const int c4 = cchunk * FA_CC + it % cc;
    const int px = it / cc;
    const int x = tx * FA_TX + px % FA_TX, y = ty * FA_TY + px / FA_TX;
    if (x >= a.W || y >= a.H) continue;
    const int n = y * a.W + x;
    const size_t tok = static_cast<size_t>(b) * N + n;
    const int ch = 4 * c4;
    const int h0 = ch / a.Ch, h3 = (ch + 3) / a.Ch;
    const int r = max(a.radius[h0], a.radius[h3]);
    const float* img = a.qkv + static_cast<size_t>(b) * N * 3 * a.C;
    float4 conv = __ldg(reinterpret_cast<const float4*>(a.crpe_b) + c4);
    for (int dy = -r; dy <= r; ++dy) {
      const int yy = y + dy;
      if (yy < 0 || yy >= a.H) continue;
      for (int dx = -r; dx <= r; ++dx) {
        const int xx = x + dx;
        if (xx < 0 || xx >= a.W) continue;
        const float4 w = __ldg(reinterpret_cast<const float4*>(a.crpe_w + ((dy + 3) * 7 + dx + 3) * a.C) + c4);
        const float4 v = __ldg(reinterpret_cast<const float4*>(img + (static_cast<size_t>(yy) * a.W + xx) * 3 * a.C + 2 * a.C) + c4);
        conv.x = fmaf(w.x, v.x, conv.x);
        conv.y = fmaf(w.y, v.y, conv.y);
        conv.z = fmaf(w.z, v.z, conv.z);
        conv.w = fmaf(w.w, v.w, conv.w);
      }
    }
    const float* qrow = img + static_cast<size_t>(n) * 3 * a.C;
    const float* kt = a.ktv + static_cast<size_t>(b) * a.heads * a.Ch * a.Ch;
    float fa[4] = {0.f, 0.f, 0.f, 0.f};
    if (h0 == h3 && (a.Ch & 3) == 0) {  // the four channels sit in one head at a 16-byte aligned column
      const float* qh = qrow + h0 * a.Ch;
      const float* kh = kt + static_cast<size_t>(h0) * a.Ch * a.Ch + (ch - h0 * a.Ch);
      for (int k = 0; k < a.Ch; ++k) {
        const float q = __ldg(qh + k);
        const float4 t = __ldg(reinterpret_cast<const float4*>(kh + k * a.Ch));
        fa[0] = fmaf(q, t.x, fa[0]);
        fa[1] = fmaf(q, t.y, fa[1]);
        fa[2] = fmaf(q, t.z, fa[2]);
        fa[3] = fmaf(q, t.w, fa[3]);
      }
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int hj = (ch + j) / a.Ch, cj = ch + j - hj * a.Ch;
        const float* qh = qrow + hj * a.Ch;
        const float* kh = kt + static_cast<size_t>(hj) * a.Ch * a.Ch + cj;
        float s = 0.f;
        for (int k = 0; k < a.Ch; ++k) s = fmaf(__ldg(qh + k), __ldg(kh + k * a.Ch), s);
        fa[j] = s;
      }
    }
    const float4 q4 = __ldg(reinterpret_cast<const float4*>(qrow) + c4);
    const float o0 = fmaf(a.scale, fa[0], q4.x * conv.x), o1 = fmaf(a.scale, fa[1], q4.y * conv.y);
    const float o2 = fmaf(a.scale, fa[2], q4.z * conv.z), o3 = fmaf(a.scale, fa[3], q4.w * conv.w);
    __half h[4], l[4];
    split_f16(o0, a.split_scale, h[0], l[0], ov);
    split_f16(o1, a.split_scale, h[1], l[1], ov);
    split_f16(o2, a.split_scale, h[2], l[2], ov);
    split_f16(o3, a.split_scale, h[3], l[3], ov);
    const size_t o = tok * a.C + ch;
    *reinterpret_cast<uint2*>(a.out_hi + o) = *reinterpret_cast<const uint2*>(h);
    *reinterpret_cast<uint2*>(a.out_lo + o) = *reinterpret_cast<const uint2*>(l);
  }
  if (ov) atomicOr(a.status, 1);
}

}  // namespace dd
