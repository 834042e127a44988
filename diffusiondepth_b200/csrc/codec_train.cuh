// Training-mode BatchNorm of the depth codec (dd_set_codec_mode(DD_CODEC_TRAIN)): batch statistics of the pre-BN value,
// folded on the device into a copy of the weights that the unchanged decoder_kernel / encoder_kernel then run on, and
// the decoder backward's extra term through the batch mean and variance.  The two statistics passes, their partials
// and the cross-rank totals follow bn_stats.cuh.
#pragma once
#include "backward.cuh"
#include "bn_stats.cuh"

namespace dd {

constexpr int BNS_PIX = 1024;     // items per block of bn_stats_kernel (4 per thread)
constexpr int BNS_COLS = 2 * 16;  // partials per block: [2][16], sum d then sum d^2 of the 16 channels

// The pre-BatchNorm values (16 channels per item) of the codec's three BatchNorms.  load() stages what eval() reads in
// shared memory (SMEM floats).

// Decoder: u = ConvT4x4/s2/p1(x; unfolded W) at output pixel q of [B][2h][2w], without the ConvT bias: the statistics
// are taken of the convolution alone and bn_fold_kernel adds the bias to the mean in fp64, so a bias far larger than
// the spread of u costs no precision.
struct DecPreBn {
  const float* x;   // latent NHWC [B][h][w][16]
  const float* wu;  // [ky][kx][ci][co]
  int h, w;
  static constexpr int SMEM = 4096;
  __device__ void load(float* s) const {
    for (int i = threadIdx.x; i < 1024; i += blockDim.x)
      reinterpret_cast<float4*>(s)[i] = reinterpret_cast<const float4*>(wu)[i];
  }
  __device__ void eval(const float* s, long long q, float u[16]) const {
    const int H = 2 * h, W = 2 * w;
    const int b = static_cast<int>(q / (static_cast<long long>(H) * W));
    const int Y = static_cast<int>((q / W) % H), X = static_cast<int>(q % W);
#pragma unroll
    for (int c = 0; c < 16; ++c) u[c] = 0.f;
    const int ky0 = (Y + 1) & 1, kx0 = (X + 1) & 1;
#pragma unroll
    for (int a2 = 0; a2 < 2; ++a2) {
      const int ky = ky0 + 2 * a2;
      const int iy = (Y + 1 - ky) / 2;
      if (Y + 1 - ky < 0 || iy >= h) continue;
#pragma unroll
      for (int b2 = 0; b2 < 2; ++b2) {
        const int kx = kx0 + 2 * b2;
        const int ix = (X + 1 - kx) / 2;
        if (X + 1 - kx < 0 || ix >= w) continue;
        const float* lp = x + ((static_cast<size_t>(b) * h + iy) * w + ix) * 16;
        const float* wn = s + (ky * 4 + kx) * 256;
#pragma unroll
        for (int ci = 0; ci < 16; ++ci) {
          const float v = lp[ci];
#pragma unroll
          for (int c = 0; c < 16; ++c) u[c] = fmaf(v, wn[ci * 16 + c], u[c]);
        }
      }
    }
  }
};

// Encoder BatchNorm 1: c1 = Conv2d(1,16,3,s2,p1, no bias)(depth) at latent pixel q of [B][h][w].
struct EncPreBn1 {
  const float* depth;  // [B][H][W]
  const float* w1;     // unfolded [9][16] (tap, co)
  int H, W, h, w;
  static constexpr int SMEM = 144;
  __device__ void load(float* s) const {
    if (threadIdx.x < 144) s[threadIdx.x] = w1[threadIdx.x];
  }
  __device__ void eval(const float* s, long long q, float u[16]) const {
    const int b = static_cast<int>(q / (static_cast<long long>(h) * w));
    const int ly = static_cast<int>((q / w) % h), lx = static_cast<int>(q % w);
#pragma unroll
    for (int c = 0; c < 16; ++c) u[c] = 0.f;
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const int yy = 2 * ly - 1 + tap / 3, xx = 2 * lx - 1 + tap % 3;
      if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;
      const float v = depth[(static_cast<size_t>(b) * H + yy) * W + xx];
#pragma unroll
      for (int c = 0; c < 16; ++c) u[c] = fmaf(v, s[tap * 16 + c], u[c]);
    }
  }
};

// Encoder BatchNorm 2: c2 = Conv2d(16,16,3,1,1, no bias)(a1) at latent pixel q, where a1 = LeakyReLU(0.2) of the
// batch-folded first conv, evaluated as encoder_kernel evaluates its intermediate.
struct EncPreBn2 {
  const float* depth;  // [B][H][W]
  const float* w1f;    // batch-folded [9][16]
  const float* b1f;    // [16]
  const float* w2;     // unfolded [9][16][16] (tap, ci, co)
  int H, W, h, w;
  static constexpr int SMEM = 144 + 16 + 2304;
  __device__ void load(float* s) const {
    if (threadIdx.x < 144) s[threadIdx.x] = w1f[threadIdx.x];
    if (threadIdx.x < 16) s[144 + threadIdx.x] = b1f[threadIdx.x];
    for (int i = threadIdx.x; i < 2304; i += blockDim.x) s[160 + i] = w2[i];
  }
  __device__ void eval(const float* s, long long q, float u[16]) const {
    const int b = static_cast<int>(q / (static_cast<long long>(h) * w));
    const int ly = static_cast<int>((q / w) % h), lx = static_cast<int>(q % w);
#pragma unroll
    for (int c = 0; c < 16; ++c) u[c] = 0.f;
    for (int t2 = 0; t2 < 9; ++t2) {
      const int my = ly - 1 + t2 / 3, mx = lx - 1 + t2 % 3;
      if (my < 0 || my >= h || mx < 0 || mx >= w) continue;  // the second conv's zero padding
      float a[16];
#pragma unroll
      for (int c = 0; c < 16; ++c) a[c] = s[144 + c];
#pragma unroll
      for (int tap = 0; tap < 9; ++tap) {
        const int yy = 2 * my - 1 + tap / 3, xx = 2 * mx - 1 + tap % 3;
        const float v = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? depth[(static_cast<size_t>(b) * H + yy) * W + xx] : 0.f;
#pragma unroll
        for (int c = 0; c < 16; ++c) a[c] = fmaf(v, s[tap * 16 + c], a[c]);
      }
      const float* w2 = s + 160 + t2 * 256;
#pragma unroll
      for (int ci = 0; ci < 16; ++ci) {
        const float v = a[ci] > 0.f ? a[ci] : 0.2f * a[ci];
#pragma unroll
        for (int c = 0; c < 16; ++c) u[c] = fmaf(v, w2[ci * 16 + c], u[c]);
      }
    }
  }
};

// Per-block partials [2][16] over the block's BNS_PIX items: sum d, sum d^2, d = u - m.  Pass 1: sum1 null, m = 0;
// pass 2: m = fp32(sum1 / N), N = *cnt or n when cnt is null.
template <class Op>
__global__ void __launch_bounds__(256) bn_stats_kernel(const Op op, long long n, const double* __restrict__ sum1,
                                                       const double* __restrict__ cnt, double* __restrict__ part) {
  __shared__ __align__(16) float s_op[Op::SMEM];
  __shared__ double s_red[8][BNS_COLS];
  op.load(s_op);
  __syncthreads();
  const double N = cnt ? *cnt : static_cast<double>(n);
  float m[16];
#pragma unroll
  for (int c = 0; c < 16; ++c) m[c] = sum1 ? static_cast<float>(sum1[c] / N) : 0.f;
  float acc[BNS_COLS];
#pragma unroll
  for (int j = 0; j < BNS_COLS; ++j) acc[j] = 0.f;
  const long long base = static_cast<long long>(blockIdx.x) * BNS_PIX;
  for (int k = 0; k < BNS_PIX / 256; ++k) {
    const long long q = base + k * 256 + threadIdx.x;
    if (q >= n) break;
    float u[16];
    op.eval(s_op, q, u);
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      const float d = u[c] - m[c];
      acc[c] += d;
      acc[16 + c] = fmaf(d, d, acc[16 + c]);
    }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < BNS_COLS; ++j) {
    double s = static_cast<double>(acc[j]);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) s_red[warp][j] = s;
  }
  __syncthreads();
  if (threadIdx.x < BNS_COLS) {
    double s = 0.0;
    for (int w8 = 0; w8 < 8; ++w8) s += s_red[w8][threadIdx.x];
    part[static_cast<size_t>(blockIdx.x) * BNS_COLS + threadIdx.x] = s;
  }
}

// Fold the batch statistics (bn_batch_stats) into a copy of one conv's weights:
//   w_out = w s (output channel = index % 16),  b_out = (bias - mean_b) s + beta = beta - mean_conv s,
// where the statistics were taken of the convolution without its bias (mean_b = mean_conv + bias),
// and the record of this evaluation: batch mean and unbiased variance.
struct BnFoldArgs {
  BnFoldIn in;  // C = 16
  const float *gamma, *beta;
  const float* bias;  // the conv's own bias in front of the BatchNorm, not in the statistics (null: none)
  const float* w;     // unfolded weights, output channel fastest
  int nw;
  float *w_out, *b_out;
  float* bn_out;  // null, or [3][16]: s, batch mean of the conv WITHOUT its bias, rstd (the decoder backward's `bn`,
                  // which then runs with a zero ConvT bias: xhat from bias-free values, as the statistics were taken)
  float* rec;     // null, or [2][16]: batch mean, unbiased batch variance
};
__global__ void __launch_bounds__(256) bn_fold_kernel(const BnFoldArgs f) {
  __shared__ double s_sc[16];
  const int c = threadIdx.x;
  if (c < 16) {
    // read before the statistics: ptxas then keeps 11 partials' loads in flight in their latency-bound sum, not 8
    const double bias = f.bias ? static_cast<double>(f.bias[c]) : 0.0;
    const BnBatchStats b = bn_batch_stats(f.in, 16, c, f.gamma);
    s_sc[c] = b.scale;
    f.b_out[c] = static_cast<float>(static_cast<double>(f.beta[c]) - b.mean * b.scale);
    if (f.bn_out) {
      f.bn_out[c] = static_cast<float>(b.scale);
      f.bn_out[16 + c] = static_cast<float>(b.mean);
      f.bn_out[32 + c] = static_cast<float>(1.0 / sqrt(b.var + 1e-5));
    }
    if (f.rec) {
      f.rec[c] = static_cast<float>(b.mean + bias);
      f.rec[16 + c] = static_cast<float>(b.var_unbiased);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < f.nw; i += blockDim.x)
    f.w_out[i] = static_cast<float>(static_cast<double>(f.w[i]) * s_sc[i & 15]);
}

// Decoder backward through the batch statistics.  dec_bwd_act_kernel ran on the batch-folded weights, a zero ConvT bias
// and the batch `bn` = [s, bias-free mean, rstd]: du = s dv, and its partials hold sum dv and sum dv xhat.  With
// sums[32] their totals over the N output pixels, du becomes s (dv - sum dv / N - xhat sum(dv xhat) / N), xhat = (u -
// mean) rstd recomputed from the bias-free u in dec_bwd_act_kernel's order (the same xhat); the per-block sums of the
// new du (the ConvT bias gradient, zero up to rounding) go to part_db [blocks][16].
// Same block decomposition as dec_bwd_act_kernel.  Across ranks sums are the union batch's and *cnt its pixel count
// (cnt null: the local N).
__global__ void __launch_bounds__(256) dec_bwd_bn_kernel(const DecBwdArgs a, const double* __restrict__ sums,
                                                         const double* __restrict__ cnt, double* __restrict__ part_db) {
  __shared__ __align__(16) float s_op[DecPreBn::SMEM];
  __shared__ double s_red[8][16];
  const DecPreBn op{a.x, a.wu, a.h, a.w};
  op.load(s_op);
  __syncthreads();
  const long long N = static_cast<long long>(a.B) * 4 * a.h * a.w;
  const double NN = cnt ? *cnt : static_cast<double>(N);
  float ka[16], kb[16], acc[16];
#pragma unroll
  for (int c = 0; c < 16; ++c) {
    ka[c] = static_cast<float>(sums[c] / NN);
    kb[c] = static_cast<float>(sums[16 + c] / NN);
    acc[c] = 0.f;
  }
  const long long base = static_cast<long long>(blockIdx.x) * DEC_ACT_PIX;
  for (int k = 0; k < DEC_ACT_PIX / 256; ++k) {
    const long long q = base + k * 256 + threadIdx.x;
    if (q >= N) break;
    float u[16];
    op.eval(s_op, q, u);
    float4* dp = reinterpret_cast<float4*>(a.du + q * 16);
#pragma unroll
    for (int c4 = 0; c4 < 4; ++c4) {
      const float4 d4 = dp[c4];
      float d[4] = {d4.x, d4.y, d4.z, d4.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = 4 * c4 + j;
        const float xhat = (u[c] - a.bn[16 + c]) * a.bn[32 + c];
        d[j] -= a.bn[c] * fmaf(xhat, kb[c], ka[c]);
        acc[c] += d[j];
      }
      dp[c4] = make_float4(d[0], d[1], d[2], d[3]);
    }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int c = 0; c < 16; ++c) {
    double s = static_cast<double>(acc[c]);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) s_red[warp][c] = s;
  }
  __syncthreads();
  if (threadIdx.x < 16) {
    double s = 0.0;
    for (int w8 = 0; w8 < 8; ++w8) s += s_red[w8][threadIdx.x];
    part_db[static_cast<size_t>(blockIdx.x) * 16 + threadIdx.x] = s;
  }
}

}  // namespace dd
