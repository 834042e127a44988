// Training-mode BatchNorm of the condition producers (dd_set_producer_mode(DD_PRODUCER_TRAIN)): the FPN's conv_lateral /
// conv_up, the HAHI neck's ConvModules and the ResNet BasicBlocks' bn1 / bn2.  The unchanged convgen_wgmma_kernel runs
// the layer on an unfolded pack (no BatchNorm, no bias, no activation) and writes the pre-BN value u, fp32 NHWC
// [n][C]; these kernels then take its per-channel batch statistics, fold them into a scale and shift, and apply
// act(s u + t) with the eval epilogue's addend placements and outputs.  The two statistics passes, their partials and
// the cross-rank totals follow bn_stats.cuh.
#pragma once
#include <cuda_fp16.h>

#include "bn_stats.cuh"

namespace dd {

constexpr int PBN_ROWS = 512;  // pixels per block of pbn_stats_kernel (64 per thread)
constexpr int PBN_CH = 32;     // channels per block (one per lane)

// grid (ceil(n / PBN_ROWS), ceil(C / PBN_CH)), block (32, 8).  part [blocks.x][2][C]: sum d, sum d^2 of the block's
// pixels, d = u - m with m = 0 (pass 1, sum1 null) or fp32(sum1[c] / N) (pass 2), N = *cnt, or n when cnt is null.
__global__ void __launch_bounds__(256) pbn_stats_kernel(const float* __restrict__ u, long long n, int C,
                                                        const double* __restrict__ sum1, const double* __restrict__ cnt,
                                                        double* __restrict__ part) {
  const int c = blockIdx.y * PBN_CH + threadIdx.x;
  const bool ok = c < C;
  const double N = cnt ? *cnt : static_cast<double>(n);
  const float m = (sum1 && ok) ? static_cast<float>(sum1[c] / N) : 0.f;
  float s = 0.f, q = 0.f;
  const long long base = static_cast<long long>(blockIdx.x) * PBN_ROWS;
  if (ok) {
    for (int k = threadIdx.y; k < PBN_ROWS; k += 8) {
      const long long p = base + k;
      if (p >= n) break;
      const float d = __ldg(u + p * C + c) - m;
      s += d;
      q = fmaf(d, d, q);
    }
  }
  __shared__ double red[2][8][PBN_CH];
  red[0][threadIdx.y][threadIdx.x] = static_cast<double>(s);
  red[1][threadIdx.y][threadIdx.x] = static_cast<double>(q);
  __syncthreads();
  if (threadIdx.y < 2 && ok) {
    double t = 0.0;
#pragma unroll
    for (int y = 0; y < 8; ++y) t += red[threadIdx.y][y][threadIdx.x];
    part[(static_cast<size_t>(blockIdx.x) * 2 + threadIdx.y) * C + c] = t;
  }
}

// From the batch statistics (bn_batch_stats): s, t = beta - s mean in fp64, each rounded once, and the record [2][C]
// (batch mean, unbiased batch variance) that the caller's running update reads.
__global__ void __launch_bounds__(256) pbn_fold_kernel(const BnFoldIn in, int C, const float* __restrict__ gamma,
                                                       const float* __restrict__ beta, float* __restrict__ s_out,
                                                       float* __restrict__ t_out, float* __restrict__ rec) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const BnBatchStats b = bn_batch_stats(in, C, c, gamma);
  s_out[c] = static_cast<float>(b.scale);
  t_out[c] = static_cast<float>(static_cast<double>(beta[c]) - b.mean * b.scale);
  rec[c] = static_cast<float>(b.mean);
  rec[C + c] = static_cast<float>(b.var_unbiased);
}

// y = act(s u + t) over n pixels of C channels (C % 8 == 0), eight channels per item, act as the eval epilogue's `relu`
// code (0 none, 1 ReLU, 3 Hardswish), with the eval epilogue's addend placements: add32 (dense [n][C]) before the ReLU (add_first, ResNet conv2 + skip) or after it (FPN lateral + up).
// Outputs: y32 dense [n][C] and / or fp16 hi / lo planes [n][ld_out] from channel ch_off at split_scale; an output
// outside the split's range sets bit 0 of *status, as convgen_wgmma_kernel does.
struct PbnApplyArgs {
  const float* u;
  long long n;
  int C, relu, add_first;
  const float *s, *t;
  const float* add32;
  float* y32;
  __half *out_hi, *out_lo;
  int ld_out, ch_off;
  float split_scale;
  int* status;
};
__global__ void __launch_bounds__(256) pbn_apply_kernel(const PbnApplyArgs a) {
  const int c8 = a.C / 8;
  const long long items = a.n * c8;
  bool overflow = false;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < items;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long p = i / c8;
    const int c0 = static_cast<int>(i - p * c8) * 8;
    const size_t o = static_cast<size_t>(p) * a.C + c0;
    float v[8], ad[8];
    const float4* u4 = reinterpret_cast<const float4*>(a.u + o);
    const float4* s4 = reinterpret_cast<const float4*>(a.s + c0);
    const float4* t4 = reinterpret_cast<const float4*>(a.t + c0);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float4 x = __ldg(u4 + h), sc = __ldg(s4 + h), sh = __ldg(t4 + h);
      v[4 * h] = fmaf(x.x, sc.x, sh.x);
      v[4 * h + 1] = fmaf(x.y, sc.y, sh.y);
      v[4 * h + 2] = fmaf(x.z, sc.z, sh.z);
      v[4 * h + 3] = fmaf(x.w, sc.w, sh.w);
      const float4 d = a.add32 ? __ldg(reinterpret_cast<const float4*>(a.add32 + o) + h) : make_float4(0.f, 0.f, 0.f, 0.f);
      ad[4 * h] = d.x;
      ad[4 * h + 1] = d.y;
      ad[4 * h + 2] = d.z;
      ad[4 * h + 3] = d.w;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (a.add32 && a.add_first) v[j] += ad[j];
      if (a.relu == 1) v[j] = fmaxf(v[j], 0.f);
      else if (a.relu == 3) v[j] = v[j] * fminf(fmaxf(v[j] + 3.f, 0.f), 6.f) * (1.f / 6.f);
      if (a.add32 && !a.add_first) v[j] += ad[j];
    }
    if (a.y32) {
      float4* d4 = reinterpret_cast<float4*>(a.y32 + o);
      d4[0] = make_float4(v[0], v[1], v[2], v[3]);
      d4[1] = make_float4(v[4], v[5], v[6], v[7]);
    }
    if (a.out_hi) {
      __align__(16) __half2 hi[4];
      __align__(16) __half2 lo[4];
      float amax = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float s0 = v[2 * j] * a.split_scale, s1 = v[2 * j + 1] * a.split_scale;
        amax = fmaxf(amax, fmaxf(fabsf(s0), fabsf(s1)));
        hi[j] = __floats2half2_rn(s0, s1);
        const float2 back = __half22float2(hi[j]);
        lo[j] = __floats2half2_rn(s0 - back.x, s1 - back.y);
      }
      overflow |= !(amax <= 60000.f);  // also catches NaN
      const size_t po = static_cast<size_t>(p) * a.ld_out + a.ch_off + c0;
      *reinterpret_cast<uint4*>(a.out_hi + po) = *reinterpret_cast<const uint4*>(hi);
      *reinterpret_cast<uint4*>(a.out_lo + po) = *reinterpret_cast<const uint4*>(lo);
    }
  }
  if (overflow) atomicOr(a.status, 1);
}

// Stochastic depth on a residual branch (MPViT's MHCABlock, reference mpvit.py:432,435): y = x + scale[b] branch over
// B images of `per_img` rows of C channels (C % 4 == 0), scale[b] = mask / keep.  y goes to y32 (dense [rows][C]; may
// alias x) or to fp16 hi / lo planes [rows][ld_out] from channel ch_off at split_scale, where an output outside the
// split's range sets bit 0 of *status, as convgen_wgmma_kernel does.
struct DropAddArgs {
  const float* x;
  const float* branch;
  const float* scale;
  long long per_img;
  int B, C;
  float* y32;
  __half *out_hi, *out_lo;
  int ld_out, ch_off;
  float split_scale;
  int* status;
};
__global__ void __launch_bounds__(256) drop_path_add_kernel(const DropAddArgs a) {
  const int c4 = a.C / 4;
  const long long items = a.per_img * a.B * c4;
  bool overflow = false;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < items;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long p = i / c4;
    const int c0 = static_cast<int>(i - p * c4) * 4;
    const float s = __ldg(a.scale + p / a.per_img);
    const size_t o = static_cast<size_t>(p) * a.C + c0;
    const float4 x = __ldg(reinterpret_cast<const float4*>(a.x + o));
    const float4 r = __ldg(reinterpret_cast<const float4*>(a.branch + o));
    const float v[4] = {fmaf(s, r.x, x.x), fmaf(s, r.y, x.y), fmaf(s, r.z, x.z), fmaf(s, r.w, x.w)};
    if (a.y32) *reinterpret_cast<float4*>(a.y32 + o) = make_float4(v[0], v[1], v[2], v[3]);
    if (a.out_hi) {
      __align__(8) __half2 hi[2];
      __align__(8) __half2 lo[2];
      float amax = 0.f;
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const float s0 = v[2 * j] * a.split_scale, s1 = v[2 * j + 1] * a.split_scale;
        amax = fmaxf(amax, fmaxf(fabsf(s0), fabsf(s1)));
        hi[j] = __floats2half2_rn(s0, s1);
        const float2 back = __half22float2(hi[j]);
        lo[j] = __floats2half2_rn(s0 - back.x, s1 - back.y);
      }
      overflow |= !(amax <= 60000.f);  // also catches NaN
      const size_t po = static_cast<size_t>(p) * a.ld_out + a.ch_off + c0;
      *reinterpret_cast<uint2*>(a.out_hi + po) = *reinterpret_cast<const uint2*>(hi);
      *reinterpret_cast<uint2*>(a.out_lo + po) = *reinterpret_cast<const uint2*>(lo);
    }
  }
  if (overflow) atomicOr(a.status, 1);
}

}  // namespace dd
