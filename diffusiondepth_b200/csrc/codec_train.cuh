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

// ------------------------------------------------------------------ encoder backward (reverse of encoder_kernel)
// Forward (kernels.cuh encoder_kernel, on the folded weights): u1 = conv1(depth) (3x3, stride 2, pad 1, no bias),
// v1 = s1 (u1 - m1) + beta1, a1 = LeakyReLU_0.2(v1), u2 = conv2(a1) (3x3, pad 1, no bias), v2 = s2 (u2 - m2) + beta2,
// out = tanh(v2); s = gamma rstd, (m, rstd) running or batch statistics.  Reverse, with xhat = (u - m) rstd from the
// unfolded conv:
//   dv2 = d_latent (1 - out^2);  dgamma2 = sum dv2 xhat2,  dbeta2 = sum dv2;  du2 = s2 dv2, and in training mode
//   du2 = s2 (dv2 - sum dv2 / N - xhat2 sum(dv2 xhat2) / N);
//   dw2[tap][ci][co] = sum_q a1(q + d_tap)[ci] du2(q)[co],  da1(m)[ci] = sum_tap sum_co w2[tap][ci][co] du2(m - d_tap)[co];
//   dv1 = da1 [v1 > 0 ? 1 : 0.2];  BatchNorm 1 as BatchNorm 2;  dw1[tap][co] = sum_q depth(2 q - 1 + tap) du1(q)[co].
// One thread per latent pixel for the per-pixel passes; the recomputed v1 and v2 use the forward's folded weights in its
// FMA order, so the LeakyReLU mask and tanh are the forward's.  Every reduction writes fixed per-block fp64 partials
// that enc_bwd_finish_kernel sums in block order.
constexpr int ENC_PIX = 256;          // latent pixels per block of the per-pixel kernels (one per thread)
constexpr int ENC_WG_BLOCKS = 192;    // most blocks of enc_bwd_wgrad_kernel
constexpr int ENC_WG_COLS = 2304 + 144;  // its partial columns: conv2 (tap * 16 + ci) * 16 + co, then conv1 tap * 16 + co
constexpr int ENC_GRAD_N = 144 + 16 + 16 + 2304 + 16 + 16;  // the six encoder gradients, reference layouts back to back

struct EncBwdArgs {
  const float* depth;  // [B][H][W]
  const float *w1f, *b1f, *w2f, *b2f;  // the forward's folded weights: [9][16], [16], [9][16][16], [16]
  const float *w1u, *w2u;              // unfolded: [9][16] (tap, co), [9][16][16] (tap, ci, co)
  const float *bn1, *bn2;              // [3][16] each: s, mean of the bias-free conv, rstd
  const float* dlat;   // d_latent NCHW [B][16][h][w]
  float* a1;           // [N][16] LeakyReLU output
  float* x1;           // [N][16] xhat1
  float* x2;           // [N][16] xhat2, then dv1, then du1
  float* dz;           // [N][16] dv2, then du2
  double* part2;       // [blocks][32] sum dv2, sum dv2 xhat2
  double* part1;       // [blocks][32] sum dv1, sum dv1 xhat1
  double* part_w;      // [wg blocks][ENC_WG_COLS]
  int B, H, W, h, w;
};

// Block sums of acc[32] over the block's 256 threads into part[blockIdx.x][32].
__device__ __forceinline__ void enc_block_partials(const float (&acc)[32], double* __restrict__ part) {
  __shared__ double s_red[8][32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    double s = static_cast<double>(acc[j]);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) s_red[warp][j] = s;
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    double s = 0.0;
    for (int w8 = 0; w8 < 8; ++w8) s += s_red[w8][threadIdx.x];
    part[static_cast<size_t>(blockIdx.x) * 32 + threadIdx.x] = s;
  }
}

// a1 at every latent pixel: the first conv on the folded weights in encoder_kernel's order (out-of-map depth taps as 0).
__global__ void __launch_bounds__(256) enc_bwd_mid_kernel(const EncBwdArgs a) {
  __shared__ float s_w[144 + 16];
  if (threadIdx.x < 144) s_w[threadIdx.x] = a.w1f[threadIdx.x];
  if (threadIdx.x < 16) s_w[144 + threadIdx.x] = a.b1f[threadIdx.x];
  __syncthreads();
  const int P = a.h * a.w;
  const int q = blockIdx.x * ENC_PIX + threadIdx.x;
  if (q >= a.B * P) return;
  const int b = q / P, ly = (q % P) / a.w, lx = q % a.w;
  float o[16];
#pragma unroll
  for (int c = 0; c < 16; ++c) o[c] = s_w[144 + c];
#pragma unroll
  for (int tap = 0; tap < 9; ++tap) {
    const int yy = 2 * ly - 1 + tap / 3, xx = 2 * lx - 1 + tap % 3;
    const float v = (yy >= 0 && yy < a.H && xx >= 0 && xx < a.W) ? a.depth[(static_cast<size_t>(b) * a.H + yy) * a.W + xx] : 0.f;
#pragma unroll
    for (int c = 0; c < 16; ++c) o[c] = fmaf(v, s_w[tap * 16 + c], o[c]);
  }
  float4* op = reinterpret_cast<float4*>(a.a1 + static_cast<size_t>(q) * 16);
#pragma unroll
  for (int c4 = 0; c4 < 4; ++c4) {
    float r[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) r[j] = o[4 * c4 + j] > 0.f ? o[4 * c4 + j] : 0.2f * o[4 * c4 + j];
    op[c4] = make_float4(r[0], r[1], r[2], r[3]);
  }
}

// out = tanh of the folded second conv (encoder_kernel's order), xhat2 from the unfolded one, dv2 = d_latent (1 - out^2);
// partials sum dv2, sum dv2 xhat2.
__global__ void __launch_bounds__(256) enc_bwd_out_kernel(const EncBwdArgs a) {
  __shared__ __align__(16) float s_wf[2304];
  __shared__ __align__(16) float s_wu[2304];
  for (int i = threadIdx.x; i < 576; i += 256) {
    reinterpret_cast<float4*>(s_wf)[i] = reinterpret_cast<const float4*>(a.w2f)[i];
    reinterpret_cast<float4*>(s_wu)[i] = reinterpret_cast<const float4*>(a.w2u)[i];
  }
  __syncthreads();
  const int P = a.h * a.w;
  const int q = blockIdx.x * ENC_PIX + threadIdx.x;
  float acc[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) acc[j] = 0.f;
  if (q < a.B * P) {
    const int b = q / P, ly = (q % P) / a.w, lx = q % a.w;
    float of[16], ou[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      of[c] = a.b2f[c];
      ou[c] = 0.f;
    }
    for (int tap = 0; tap < 9; ++tap) {
      const int my = ly - 1 + tap / 3, mx = lx - 1 + tap % 3;
      float m[16];
      if (my >= 0 && my < a.h && mx >= 0 && mx < a.w) {
        const float4* mp = reinterpret_cast<const float4*>(a.a1 + ((static_cast<size_t>(b) * a.h + my) * a.w + mx) * 16);
#pragma unroll
        for (int c4 = 0; c4 < 4; ++c4) {
          const float4 v = mp[c4];
          m[4 * c4] = v.x;
          m[4 * c4 + 1] = v.y;
          m[4 * c4 + 2] = v.z;
          m[4 * c4 + 3] = v.w;
        }
      } else {
#pragma unroll
        for (int c = 0; c < 16; ++c) m[c] = 0.f;  // the second conv's zero padding, as encoder_kernel's s_mid holds it
      }
      const float* wf = s_wf + tap * 256;
      const float* wu = s_wu + tap * 256;
#pragma unroll
      for (int ci = 0; ci < 16; ++ci) {
#pragma unroll
        for (int co = 0; co < 16; ++co) {
          of[co] = fmaf(m[ci], wf[ci * 16 + co], of[co]);
          ou[co] = fmaf(m[ci], wu[ci * 16 + co], ou[co]);
        }
      }
    }
    float xh[16], dv[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      const float t = tanhf(of[c]);
      dv[c] = a.dlat[(static_cast<size_t>(b) * 16 + c) * P + (q % P)] * (1.f - t * t);
      xh[c] = (ou[c] - a.bn2[16 + c]) * a.bn2[32 + c];
      acc[c] = dv[c];
      acc[16 + c] = dv[c] * xh[c];
    }
    float4* xp = reinterpret_cast<float4*>(a.x2 + static_cast<size_t>(q) * 16);
    float4* dp = reinterpret_cast<float4*>(a.dz + static_cast<size_t>(q) * 16);
#pragma unroll
    for (int c4 = 0; c4 < 4; ++c4) {
      xp[c4] = make_float4(xh[4 * c4], xh[4 * c4 + 1], xh[4 * c4 + 2], xh[4 * c4 + 3]);
      dp[c4] = make_float4(dv[4 * c4], dv[4 * c4 + 1], dv[4 * c4 + 2], dv[4 * c4 + 3]);
    }
  }
  enc_block_partials(acc, a.part2);
}

// du = s (dv - sum dv / N - xhat sum(dv xhat) / N) in place over n pixels (sums null: eval, du = s dv).  Across ranks
// sums are the union batch's and *cnt its pixel count (cnt null: n).
__global__ void __launch_bounds__(256) enc_bwd_bn_kernel(float* __restrict__ d, const float* __restrict__ xhat,
                                                         const float* __restrict__ bn, const double* __restrict__ sums,
                                                         const double* __restrict__ cnt, long long n) {
  const double NN = cnt ? *cnt : static_cast<double>(n);
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < static_cast<size_t>(n) * 16;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i & 15);
    const float ka = sums ? static_cast<float>(sums[c] / NN) : 0.f;
    const float kb = sums ? static_cast<float>(sums[16 + c] / NN) : 0.f;
    d[i] = bn[c] * (d[i] - fmaf(xhat[i], kb, ka));
  }
}

// da1 from the 3 x 3 neighbourhood of du2 (unfolded conv2 transposed), dv1 through the LeakyReLU slope, xhat1 from the
// unfolded first conv in EncPreBn1's order; partials sum dv1, sum dv1 xhat1.
__global__ void __launch_bounds__(256) enc_bwd_mid_grad_kernel(const EncBwdArgs a) {
  __shared__ __align__(16) float s_w[2304];  // [tap][co][ci]
  __shared__ float s_w1[144];
  for (int i = threadIdx.x; i < 2304; i += 256) {
    const int tap = i / 256, co = (i / 16) % 16, ci = i % 16;
    s_w[i] = a.w2u[(tap * 16 + ci) * 16 + co];
  }
  if (threadIdx.x < 144) s_w1[threadIdx.x] = a.w1u[threadIdx.x];
  __syncthreads();
  const int P = a.h * a.w;
  const int q = blockIdx.x * ENC_PIX + threadIdx.x;
  float acc[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) acc[j] = 0.f;
  if (q < a.B * P) {
    const int b = q / P, ly = (q % P) / a.w, lx = q % a.w;
    float da[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) da[c] = 0.f;
    for (int tap = 0; tap < 9; ++tap) {
      const int ny = ly + 1 - tap / 3, nx = lx + 1 - tap % 3;  // the output pixel that reads this one through `tap`
      if (ny < 0 || ny >= a.h || nx < 0 || nx >= a.w) continue;
      const float4* dp = reinterpret_cast<const float4*>(a.dz + ((static_cast<size_t>(b) * a.h + ny) * a.w + nx) * 16);
      const float* wk = s_w + tap * 256;
#pragma unroll
      for (int c4 = 0; c4 < 4; ++c4) {
        const float4 d4 = dp[c4];
        const float dv[4] = {d4.x, d4.y, d4.z, d4.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float* wr = wk + (4 * c4 + j) * 16;
#pragma unroll
          for (int ci = 0; ci < 16; ++ci) da[ci] = fmaf(dv[j], wr[ci], da[ci]);
        }
      }
    }
    float u[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) u[c] = 0.f;
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const int yy = 2 * ly - 1 + tap / 3, xx = 2 * lx - 1 + tap % 3;
      if (yy < 0 || yy >= a.H || xx < 0 || xx >= a.W) continue;
      const float v = a.depth[(static_cast<size_t>(b) * a.H + yy) * a.W + xx];
#pragma unroll
      for (int c = 0; c < 16; ++c) u[c] = fmaf(v, s_w1[tap * 16 + c], u[c]);
    }
    const float4* ap = reinterpret_cast<const float4*>(a.a1 + static_cast<size_t>(q) * 16);
    float dv[16], xh[16];
#pragma unroll
    for (int c4 = 0; c4 < 4; ++c4) {
      const float4 a4 = ap[c4];
      const float av[4] = {a4.x, a4.y, a4.z, a4.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = 4 * c4 + j;
        dv[c] = av[j] > 0.f ? da[c] : 0.2f * da[c];  // a1 > 0 exactly where v1 > 0
        xh[c] = (u[c] - a.bn1[16 + c]) * a.bn1[32 + c];
        acc[c] = dv[c];
        acc[16 + c] = dv[c] * xh[c];
      }
    }
    float4* xp = reinterpret_cast<float4*>(a.x1 + static_cast<size_t>(q) * 16);
    float4* dp = reinterpret_cast<float4*>(a.x2 + static_cast<size_t>(q) * 16);
#pragma unroll
    for (int c4 = 0; c4 < 4; ++c4) {
      xp[c4] = make_float4(xh[4 * c4], xh[4 * c4 + 1], xh[4 * c4 + 2], xh[4 * c4 + 3]);
      dp[c4] = make_float4(dv[4 * c4], dv[4 * c4 + 1], dv[4 * c4 + 2], dv[4 * c4 + 3]);
    }
  }
  enc_block_partials(acc, a.part1);
}

// dw2 and dw1: thread (tap, co) = (t / 16, t % 16) holds conv2's 16 input channels and conv1's one, and walks the
// block's contiguous run of latent pixels, fp32 for 256 pixels at a time, then fp64.
__global__ void __launch_bounds__(160) enc_bwd_wgrad_kernel(const EncBwdArgs a, int per_block) {
  const int t = threadIdx.x;
  if (t >= 144) return;
  const int tap = t / 16, co = t % 16, dy = tap / 3 - 1, dx = tap % 3 - 1;
  const int P = a.h * a.w, N = a.B * P;
  const int q0 = blockIdx.x * per_block, q1 = min(N, q0 + per_block);
  double t2[16], t1 = 0.0;
#pragma unroll
  for (int c = 0; c < 16; ++c) t2[c] = 0.0;
  for (int s0 = q0; s0 < q1; s0 += 256) {
    float c2[16], c1 = 0.f;
#pragma unroll
    for (int c = 0; c < 16; ++c) c2[c] = 0.f;
    const int s1 = min(q1, s0 + 256);
    for (int q = s0; q < s1; ++q) {
      const int b = q / P, ly = (q % P) / a.w, lx = q % a.w;
      const float d2 = a.dz[static_cast<size_t>(q) * 16 + co], d1 = a.x2[static_cast<size_t>(q) * 16 + co];
      const int my = ly + dy, mx = lx + dx;
      if (my >= 0 && my < a.h && mx >= 0 && mx < a.w) {
        const float4* mp = reinterpret_cast<const float4*>(a.a1 + (static_cast<long long>(q) + dy * a.w + dx) * 16);
#pragma unroll
        for (int c4 = 0; c4 < 4; ++c4) {
          const float4 v = mp[c4];
          c2[4 * c4] = fmaf(v.x, d2, c2[4 * c4]);
          c2[4 * c4 + 1] = fmaf(v.y, d2, c2[4 * c4 + 1]);
          c2[4 * c4 + 2] = fmaf(v.z, d2, c2[4 * c4 + 2]);
          c2[4 * c4 + 3] = fmaf(v.w, d2, c2[4 * c4 + 3]);
        }
      }
      const int yy = 2 * ly + dy, xx = 2 * lx + dx;
      if (yy >= 0 && yy < a.H && xx >= 0 && xx < a.W) c1 = fmaf(a.depth[(static_cast<size_t>(b) * a.H + yy) * a.W + xx], d1, c1);
    }
#pragma unroll
    for (int c = 0; c < 16; ++c) t2[c] += static_cast<double>(c2[c]);
    t1 += static_cast<double>(c1);
  }
  double* out = a.part_w + static_cast<size_t>(blockIdx.x) * ENC_WG_COLS;
#pragma unroll
  for (int ci = 0; ci < 16; ++ci) out[(tap * 16 + ci) * 16 + co] = t2[ci];
  out[2304 + t] = t1;
}

// The six gradients in the reference layouts, each partial column summed over the blocks in block order:
// out[0] conv1 weight [16][1][3][3], out[1] BN1 weight, out[2] BN1 bias, out[3] conv2 weight [16 co][16 ci][3][3],
// out[4] BN2 weight, out[5] BN2 bias (each nullable).
struct EncFinishArgs {
  const double *part1, *part2, *part_w;
  int nb_pix, nb_w;
  float* out[6];
};
__global__ void enc_bwd_finish_kernel(const EncFinishArgs f) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ENC_GRAD_N) return;
  double s = 0.0;
  float* dst;
  int o;
  if (i < 144) {  // [co][tap] <- column 2304 + tap * 16 + co
    const int co = i / 9, tap = i % 9;
    for (int b = 0; b < f.nb_w; ++b) s += f.part_w[static_cast<size_t>(b) * ENC_WG_COLS + 2304 + tap * 16 + co];
    dst = f.out[0];
    o = i;
  } else if (i < 176) {  // BN1 weight = sum dv1 xhat1, bias = sum dv1
    const int j = i - 144, c = j % 16, which = j / 16;
    for (int b = 0; b < f.nb_pix; ++b) s += f.part1[static_cast<size_t>(b) * 32 + (which == 0 ? 16 + c : c)];
    dst = which == 0 ? f.out[1] : f.out[2];
    o = c;
  } else if (i < 176 + 2304) {  // [co][ci][tap] <- column (tap * 16 + ci) * 16 + co
    const int j = i - 176, co = j / 144, ci = (j / 9) % 16, tap = j % 9;
    for (int b = 0; b < f.nb_w; ++b) s += f.part_w[static_cast<size_t>(b) * ENC_WG_COLS + (tap * 16 + ci) * 16 + co];
    dst = f.out[3];
    o = j;
  } else {
    const int j = i - 176 - 2304, c = j % 16, which = j / 16;
    for (int b = 0; b < f.nb_pix; ++b) s += f.part2[static_cast<size_t>(b) * 32 + (which == 0 ? 16 + c : c)];
    dst = which == 0 ? f.out[4] : f.out[5];
    o = c;
  }
  if (dst != nullptr) dst[o] = static_cast<float>(s);
}

}  // namespace dd
