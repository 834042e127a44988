// Backward of one ScheduledCNNRefine call (dd_denoiser_backward): gradient split with an on-device power-of-two scale,
// GroupNorm + ReLU backward, bias / time-embedding column sums, the weight gradient of the 3x3 convs and the adjoint of
// the align-corners bilinear upsample.  The data gradients of the convs run on the forward's conv3x3_halo_kernel with
// flipped, transposed weights (engine.cu).  Every reduction is split into fixed partials that a second pass sums in a
// fixed order in fp64, so the gradients are bit-reproducible run to run.
#pragma once
#include "kernels.cuh"

namespace dd {

constexpr int BWD_CHUNK = 256;  // pixels per partial of the GroupNorm and column-sum reductions
constexpr int WG_KS = 32;       // pixels per shared-memory stage of the weight-gradient kernel
constexpr int WG_FLUSH = 8;     // stages summed in fp32 before the per-thread fp64 accumulators take them

// Largest power of two k with amax * k < 2^14 (the rule of the weight split); 1 when amax is 0, inf or NaN.
__device__ __forceinline__ float grad_scale_of(float amax) {
  if (!(amax > 0.f) || !isfinite(amax)) return 1.f;
  return exp2f(floorf(log2f(32768.f / amax)) - 1.f);
}

// fp32 gradient (already multiplied by *in_scale, nullable = 1) -> fp16 hi/lo planes of x * k, k from the on-device
// absmax *amax.  *out_scale = in_scale * k is the factor by which a conv of these planes overshoots the true gradient.
// A non-finite absmax or a split overflow sets bit 0 of the status word, as split_planes_kernel does.
__global__ void grad_split_kernel(const float* __restrict__ x, __half* __restrict__ hi, __half* __restrict__ lo, size_t n4,
                                  const float* __restrict__ amax, const float* __restrict__ in_scale,
                                  float* __restrict__ out_scale, int* status) {
  const float a = *amax;
  const float k = grad_scale_of(a);
  bool ov = false;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    out_scale[0] = (in_scale != nullptr ? in_scale[0] : 1.f) * k;
    ov = !isfinite(a);
  }
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(x)[i];
    __align__(8) __half h[4];
    __align__(8) __half l[4];
    split_f16(v.x, k, h[0], l[0], ov);
    split_f16(v.y, k, h[1], l[1], ov);
    split_f16(v.z, k, h[2], l[2], ov);
    split_f16(v.w, k, h[3], l[3], ov);
    reinterpret_cast<uint2*>(hi)[i] = *reinterpret_cast<const uint2*>(h);
    reinterpret_cast<uint2*>(lo)[i] = *reinterpret_cast<const uint2*>(l);
  }
  if (ov) atomicOr(status, 1);
}

// x *= 1 / *scale (n elements)
__global__ void unscale_kernel(float* __restrict__ x, size_t n, const float* __restrict__ scale) {
  const float inv = 1.f / *scale;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x)
    x[i] *= inv;
}

// ------------------------------------------------------------------ GroupNorm(4, C) + ReLU backward
// Forward: z = gamma * xhat + beta, out = relu(z), xhat = (y - mean) * rstd per (image, group).  With dz = dout * [z > 0]:
//   dgamma = sum dz * xhat,  dbeta = sum dz,
//   dy = rstd * (gamma * dz - mean_g(gamma * dz) - xhat * mean_g(gamma * dz * xhat)).
// Both group means follow from the per-(image, channel) sums of dz * xhat and dz, which are all the reduction keeps.
struct GnBwdArgs {
  const float* dout;       // [B][P][C] gradient of the ReLU output, multiplied by *dscale
  const float* dscale;     // nullable: 1
  const float* y;          // [B][P][C] pre-GN conv output
  const float* mean_rstd;  // [B][4][2]
  const float* gamma;      // [C]
  const float* beta;       // [C]
  int B, P, chunks;        // chunks = ceil(P / BWD_CHUNK)
  float* partial;          // [B][chunks][C][2]: sum dz * xhat, sum dz over one chunk
  float* ab;               // [B][4][2]: mean_g(gamma * dz), mean_g(gamma * dz * xhat)
  float* dgamma;           // [C], nullable
  float* dbeta;            // [C], nullable
  float* dy;               // [B][P][C]
};

// z, the ReLU's input, of channel c of image b.  The backward's mask is z > 0; gn_pre_relu_kernel exports the same z
// (dd_denoiser_relu_inputs), so both go through this one expression.
template <int C>
__device__ __forceinline__ float gn_pre_relu(const GnBwdArgs& a, int b, int c, float yv) {
  const int g = c / (C / 4);
  const float mean = a.mean_rstd[(b * 4 + g) * 2], rstd = a.mean_rstd[(b * 4 + g) * 2 + 1];
  const float sa = rstd * a.gamma[c];
  return fmaf(yv, sa, a.beta[c] - sa * mean);  // the forward's expression (gn_apply_split_kernel)
}

template <int C>
__device__ __forceinline__ void gn_bwd_point(const GnBwdArgs& a, int b, int c, float yv, float dov, float inv, float& dz,
                                             float& xh) {
  const int g = c / (C / 4);
  const float mean = a.mean_rstd[(b * 4 + g) * 2], rstd = a.mean_rstd[(b * 4 + g) * 2 + 1];
  dz = gn_pre_relu<C>(a, b, c, yv) > 0.f ? dov * inv : 0.f;
  xh = (yv - mean) * rstd;
}

// z = gn_pre_relu of every element of a.y [B][P][C], written as fp32 NCHW [B][C][P] (uses a.y, mean_rstd, gamma, beta,
// B, P only)
template <int C>
__global__ void __launch_bounds__(256) gn_pre_relu_kernel(const GnBwdArgs a, float* __restrict__ z) {
  const size_t n = static_cast<size_t>(a.B) * C * a.P;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int p = static_cast<int>(i % a.P);
    const int c = static_cast<int>(i / a.P % C);
    const int b = static_cast<int>(i / a.P / C);
    z[i] = gn_pre_relu<C>(a, b, c, a.y[(static_cast<size_t>(b) * a.P + p) * C + c]);
  }
}

template <int C>
__global__ void __launch_bounds__(256) gn_bwd_reduce_kernel(const GnBwdArgs a) {
  constexpr int LANES = 256 / C;
  __shared__ float sh[LANES][C][2];
  const int b = blockIdx.y, chunk = blockIdx.x;
  const int c = threadIdx.x % C, lane = threadIdx.x / C;
  const float inv = a.dscale != nullptr ? 1.f / a.dscale[0] : 1.f;
  const int p0 = chunk * BWD_CHUNK, p1 = min(a.P, p0 + BWD_CHUNK);
  float s1 = 0.f, s2 = 0.f;
  for (int p = p0 + lane; p < p1; p += LANES) {
    const size_t off = (static_cast<size_t>(b) * a.P + p) * C + c;
    float dz, xh;
    gn_bwd_point<C>(a, b, c, a.y[off], a.dout[off], inv, dz, xh);
    s1 = fmaf(dz, xh, s1);
    s2 += dz;
  }
  sh[lane][c][0] = s1;
  sh[lane][c][1] = s2;
  __syncthreads();
  if (threadIdx.x < C) {
    float t1 = 0.f, t2 = 0.f;
    for (int l = 0; l < LANES; ++l) {
      t1 += sh[l][threadIdx.x][0];
      t2 += sh[l][threadIdx.x][1];
    }
    float* q = a.partial + ((static_cast<size_t>(b) * a.chunks + chunk) * C + threadIdx.x) * 2;
    q[0] = t1;
    q[1] = t2;
  }
}

// One block per group, 8 warps; a warp owns the same channels for every image, so it also carries their
// dgamma / dbeta across the images in image order.
template <int C>
__global__ void __launch_bounds__(256) gn_bwd_finalize_kernel(const GnBwdArgs a) {
  constexpr int CG = C / 4;
  __shared__ double s1[CG], s2[CG], run1[CG], run2[CG];
  const int g = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int j = threadIdx.x; j < CG; j += blockDim.x) run1[j] = run2[j] = 0.0;
  __syncthreads();
  const double inv_n = 1.0 / (static_cast<double>(CG) * a.P);
  for (int b = 0; b < a.B; ++b) {
    for (int j = warp; j < CG; j += 8) {
      const int c = g * CG + j;
      double t1 = 0.0, t2 = 0.0;
      for (int k = lane; k < a.chunks; k += 32) {
        const float* q = a.partial + ((static_cast<size_t>(b) * a.chunks + k) * C + c) * 2;
        t1 += static_cast<double>(q[0]);
        t2 += static_cast<double>(q[1]);
      }
      for (int o = 16; o > 0; o >>= 1) {
        t1 += __shfl_xor_sync(0xffffffffu, t1, o);
        t2 += __shfl_xor_sync(0xffffffffu, t2, o);
      }
      if (lane == 0) {
        s1[j] = t1;
        s2[j] = t2;
        run1[j] += t1;
        run2[j] += t2;
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      double A = 0.0, Bq = 0.0;
      for (int j = 0; j < CG; ++j) {
        const double gm = static_cast<double>(a.gamma[g * CG + j]);
        A += gm * s2[j];
        Bq += gm * s1[j];
      }
      a.ab[(b * 4 + g) * 2 + 0] = static_cast<float>(A * inv_n);
      a.ab[(b * 4 + g) * 2 + 1] = static_cast<float>(Bq * inv_n);
    }
    __syncthreads();
  }
  for (int j = threadIdx.x; j < CG; j += blockDim.x) {
    if (a.dgamma != nullptr) a.dgamma[g * CG + j] = static_cast<float>(run1[j]);
    if (a.dbeta != nullptr) a.dbeta[g * CG + j] = static_cast<float>(run2[j]);
  }
}

template <int C>
__global__ void __launch_bounds__(256) gn_bwd_apply_kernel(const GnBwdArgs a) {
  const size_t n4 = static_cast<size_t>(a.B) * a.P * C / 4;
  const float inv = a.dscale != nullptr ? 1.f / a.dscale[0] : 1.f;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t e = i * 4;
    const int c0 = static_cast<int>(e % C);
    const int b = static_cast<int>(e / C / a.P);
    const float4 yv = reinterpret_cast<const float4*>(a.y)[i];
    const float4 dv = reinterpret_cast<const float4*>(a.dout)[i];
    const float ys[4] = {yv.x, yv.y, yv.z, yv.w}, ds[4] = {dv.x, dv.y, dv.z, dv.w};
    float r[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = c0 + j, g = c / (C / 4);
      float dz, xh;
      gn_bwd_point<C>(a, b, c, ys[j], ds[j], inv, dz, xh);
      const float rstd = a.mean_rstd[(b * 4 + g) * 2 + 1];
      r[j] = rstd * (a.gamma[c] * dz - a.ab[(b * 4 + g) * 2] - xh * a.ab[(b * 4 + g) * 2 + 1]);
    }
    reinterpret_cast<float4*>(a.dy)[i] = make_float4(r[0], r[1], r[2], r[3]);
  }
}

// ------------------------------------------------------------------ column sums (bias gradient, time-embedding gradient)
// x [B][P][C] (times *scale, nullable = 1) -> partial [B][chunks][C]
template <int C>
__global__ void __launch_bounds__(256) colsum_partial_kernel(const float* __restrict__ x, const float* __restrict__ scale,
                                                             int P, int chunks, float* __restrict__ partial) {
  constexpr int LANES = 256 / C;
  __shared__ float sh[LANES][C];
  const int b = blockIdx.y, chunk = blockIdx.x;
  const int c = threadIdx.x % C, lane = threadIdx.x / C;
  const float inv = scale != nullptr ? 1.f / scale[0] : 1.f;
  const int p0 = chunk * BWD_CHUNK, p1 = min(P, p0 + BWD_CHUNK);
  float s = 0.f;
  for (int p = p0 + lane; p < p1; p += LANES) s += x[(static_cast<size_t>(b) * P + p) * C + c] * inv;
  sh[lane][c] = s;
  __syncthreads();
  if (threadIdx.x < C) {
    float t = 0.f;
    for (int l = 0; l < LANES; ++l) t += sh[l][threadIdx.x];
    partial[(static_cast<size_t>(b) * chunks + chunk) * C + threadIdx.x] = t;
  }
}
// one warp per channel: per-image sums (out_img [B][C], nullable) and their total in image order (out_sum [C], nullable)
__global__ void colsum_finalize_kernel(const float* __restrict__ partial, int B, int chunks, int C,
                                       float* __restrict__ out_img, float* __restrict__ out_sum) {
  const int c = blockIdx.x, lane = threadIdx.x;
  double total = 0.0;
  for (int b = 0; b < B; ++b) {
    double s = 0.0;
    for (int k = lane; k < chunks; k += 32) s += static_cast<double>(partial[(static_cast<size_t>(b) * chunks + k) * C + c]);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0 && out_img != nullptr) out_img[b * C + c] = static_cast<float>(s);
    total += s;
  }
  if (lane == 0 && out_sum != nullptr) out_sum[c] = static_cast<float>(total);
}

// time_embedding.weight gradient: row t_b += d_temb[b] (launched once per image, in image order)
__global__ void temb_row_add_kernel(float* __restrict__ dtable_row, const float* __restrict__ dtemb_b) {
  dtable_row[threadIdx.x] += dtemb_b[threadIdx.x];
}

// ------------------------------------------------------------------ weight gradient of the two 16-channel 3x3 convs
// dW[co][ci][tap] = sum over (b, pixel) of dY[b, p, co] * X[b, p + tap, ci], X read from the conv's own fp16 hi/lo input
// planes (exactly the operand the forward multiplied).  Block = one (TM x TN) tile of (co, ci) for one tap over one chunk
// of pixels; each thread holds a 4 x 4 sub-tile, summed in fp32 over WG_FLUSH * WG_KS pixels and then in fp64.  The
// chunks' fp64 partials are summed in chunk order by wgrad_reduce_kernel.
struct WgradArgs {
  const float* dy;      // [B*P][cout]
  const __half* x_hi;   // [B*P][cin]
  const __half* x_lo;
  float x_inv_scale;    // 1 / the planes' power-of-two scale
  int cout, cin, B, H, W;
  int chunk;            // pixels per block (multiple of WG_KS)
  double* partial;      // [chunks][cout][cin][9]
};

template <int TM, int TN>
__global__ void __launch_bounds__(TM * TN / 16) wgrad_simt_kernel(const WgradArgs a) {
  constexpr int NT = TM * TN / 16;
  __shared__ __align__(16) float As[WG_KS][TM];
  __shared__ __align__(16) float Bs[WG_KS][TN];
  const int tap = blockIdx.y % 9, rest = blockIdx.y / 9;
  const int ci0 = (rest % (a.cin / TN)) * TN, co0 = (rest / (a.cin / TN)) * TM;
  const int ky = tap / 3 - 1, kx = tap % 3 - 1;
  const int P = a.H * a.W;
  const long long BP = static_cast<long long>(a.B) * P;
  const long long q_begin = static_cast<long long>(blockIdx.x) * a.chunk;
  const long long q_end = min(BP, q_begin + a.chunk);
  const int tx = threadIdx.x % (TN / 4), ty = threadIdx.x / (TN / 4);
  float acc[4][4];
  double dacc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      acc[i][j] = 0.f;
      dacc[i][j] = 0.0;
    }
  int stage = 0;
  for (long long q0 = q_begin; q0 < q_end; q0 += WG_KS) {
    for (int idx = threadIdx.x; idx < WG_KS * TM; idx += NT) {
      const int k = idx / TM, m = idx % TM;
      const long long q = q0 + k;
      As[k][m] = q < q_end ? a.dy[q * a.cout + co0 + m] : 0.f;
    }
    for (int idx = threadIdx.x; idx < WG_KS * TN; idx += NT) {
      const int k = idx / TN, n = idx % TN;
      const long long q = q0 + k;
      float v = 0.f;
      if (q < q_end) {
        const int b = static_cast<int>(q / P), p = static_cast<int>(q - static_cast<long long>(b) * P);
        const int yy = p / a.W + ky, xx = p % a.W + kx;
        if (yy >= 0 && yy < a.H && xx >= 0 && xx < a.W) {
          const size_t off = ((static_cast<size_t>(b) * a.H + yy) * a.W + xx) * a.cin + ci0 + n;
          v = (__half2float(a.x_hi[off]) + __half2float(a.x_lo[off])) * a.x_inv_scale;
        }
      }
      Bs[k][n] = v;
    }
    __syncthreads();
#pragma unroll 8
    for (int k = 0; k < WG_KS; ++k) {
      const float4 av = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 bv = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float ar[4] = {av.x, av.y, av.z, av.w}, br[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
    }
    __syncthreads();
    if (++stage == WG_FLUSH) {
      stage = 0;
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          dacc[i][j] += static_cast<double>(acc[i][j]);
          acc[i][j] = 0.f;
        }
    }
  }
  double* out = a.partial + static_cast<size_t>(blockIdx.x) * a.cout * a.cin * 9;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
      out[(static_cast<size_t>(co0 + ty * 4 + i) * a.cin + ci0 + tx * 4 + j) * 9 + tap] =
          dacc[i][j] + static_cast<double>(acc[i][j]);
}

// Weight gradient of the 256-wide layers on the tensor cores.  GEMM view: D[co][ci] (one tap) = sum over pixels k of
// dY[k][co] * X[k + tap][ci]; both operands are NHWC planes, i.e. MN-major (channels contiguous, pixels = K), and enter
// wgmma through its transpose bits.  A K step is one 64-pixel segment of an image row: TMA loads box {64 ch, 64 px} of
// the dY planes at (co, x0, y, b) and of the input planes at (ci, x0 + dx, y + dy, b) — the tap shift is a coordinate
// offset and TMA's out-of-bounds zero fill supplies the padding and the row tail.  3-pass split: dY_hi X_hi + dY_lo X_hi
// + dY_hi X_lo.  Warp 0 of warpgroup 0 produces into a STAGES-deep ring; MCO / 64 consumer warpgroups each own 64 output
// channels x NCI input channels.  A CTA sums `segs` segments (split K) and writes its fp32 tile as an fp64 partial
// [chunk][tap][cout][cin]; wgrad_reduce_kernel adds the chunks in order.
// A tensor-core accumulator loses a little at every wgmma that adds into it: one accumulator over a CTA's 128 segments
// (1,536 wgmmas) was 3.0-3.4e-5 of max |dW| from fp64 on an H100.  So the wgmma accumulator only ever holds WGM_FLUSH
// segments; it is then added into a second, ordinary fp32 register accumulator and cleared.
constexpr int WGM_STAGES = 3;
constexpr int WGM_FLUSH = 4;
template <int MCO, int NCI>
struct WgmCfg {
  static constexpr int NCWG = MCO / 64;
  static constexpr int THREADS = 128 * (1 + NCWG);
  static constexpr int BOX = 64 * 64 * 2;                    // one TMA box: 64 pixels x 64 channels fp16
  static constexpr int A_BYTES = (MCO / 64) * BOX;           // one plane of the dY tile
  static constexpr int B_BYTES = (NCI / 64) * BOX;
  static constexpr int STAGE = 2 * A_BYTES + 2 * B_BYTES;    // hi + lo of both operands
  static constexpr int SMEM_BYTES = WGM_STAGES * STAGE + 1024;
  static_assert(SMEM_BYTES <= 232448, "exceeds the 227 KB dynamic shared memory limit");
};

struct WgmArgs {
  int cout, cin, B, H, W;
  int xsegs;       // ceil(W / 64) segments per image row
  int nseg;        // B * H * xsegs
  int segs;        // segments per CTA (split K)
  double* partial; // [chunks][9][cout][cin]
};

template <int MCO, int NCI>
__global__ void __launch_bounds__(WgmCfg<MCO, NCI>::THREADS, 1)
    wgrad_wgmma_kernel(const __grid_constant__ CUtensorMap dy_hi, const __grid_constant__ CUtensorMap dy_lo,
                       const __grid_constant__ CUtensorMap x_hi, const __grid_constant__ CUtensorMap x_lo,
                       const WgmArgs a) {
  using Cfg = WgmCfg<MCO, NCI>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ __align__(8) uint64_t full[WGM_STAGES], empty[WGM_STAGES];
  const int tap = blockIdx.y % 9, rest = blockIdx.y / 9;
  const int ci0 = (rest % (a.cin / NCI)) * NCI, co0 = (rest / (a.cin / NCI)) * MCO;
  const int dy = tap / 3 - 1, dx = tap % 3 - 1;
  const int s_begin = blockIdx.x * a.segs, s_end = min(a.nseg, s_begin + a.segs);
  const int wg = threadIdx.x >> 7;
  if (threadIdx.x == 0) {
    for (int i = 0; i < WGM_STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], Cfg::NCWG * 128);
    }
    fence_barrier_init();
  }
  __syncthreads();
  // setmaxnreg at the top of each role's branch, branches meeting only at the exit (see conv3x3_halo_kernel): the two
  // consumer warpgroups' 2 x NCI / 2 accumulators do not fit the 168-register launch bound of a 384-thread CTA
  if (wg == 0) {
    if constexpr (Cfg::NCWG > 1) setmaxnreg_dec<40>();
    if (threadIdx.x < 32) {
      const bool leader = elect_one();
      for (int s = s_begin, it = 0; s < s_end; ++s, ++it) {
        const int st = it % WGM_STAGES;
        mbar_wait(&empty[st], ((it / WGM_STAGES) & 1) ^ 1);
        if (leader) {
          const int xs = s % a.xsegs, yb = s / a.xsegs, y = yb % a.H, b = yb / a.H;
          const int x0 = xs * 64;
          uint8_t* base = smem + st * Cfg::STAGE;
          mbar_arrive_expect_tx(&full[st], Cfg::STAGE);
#pragma unroll
          for (int j = 0; j < MCO / 64; ++j) {
            tma_load_4d(base + j * Cfg::BOX, &dy_hi, &full[st], co0 + 64 * j, x0, y, b);
            tma_load_4d(base + Cfg::A_BYTES + j * Cfg::BOX, &dy_lo, &full[st], co0 + 64 * j, x0, y, b);
          }
#pragma unroll
          for (int j = 0; j < NCI / 64; ++j) {
            tma_load_4d(base + 2 * Cfg::A_BYTES + j * Cfg::BOX, &x_hi, &full[st], ci0 + 64 * j, x0 + dx, y + dy, b);
            tma_load_4d(base + 2 * Cfg::A_BYTES + Cfg::B_BYTES + j * Cfg::BOX, &x_lo, &full[st], ci0 + 64 * j, x0 + dx,
                        y + dy, b);
          }
        }
        __syncwarp();
      }
    }
  } else {
    if constexpr (Cfg::NCWG > 1) setmaxnreg_inc<232>();
    float d[NCI / 2], acc[NCI / 2];  // d: the wgmma accumulator of the current WGM_FLUSH segments; acc: their fp32 sum
#pragma unroll
    for (int i = 0; i < NCI / 2; ++i) d[i] = acc[i] = 0.f;
    const int cw = wg - 1;  // this warpgroup's 64 output channels
    for (int s = s_begin, it = 0; s < s_end; ++s, ++it) {
      const int st = it % WGM_STAGES;
      mbar_wait(&full[st], (it / WGM_STAGES) & 1);
      const uint32_t base = smem_u32(smem + st * Cfg::STAGE);
      const uint32_t ah = base + cw * Cfg::BOX, al = ah + Cfg::A_BYTES;
      const uint32_t bh = base + 2 * Cfg::A_BYTES, bl = bh + Cfg::B_BYTES;
      wgmma_fence_regs(d);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const uint32_t ko = kk * 2048;
        wgmma_f16_mn<NCI>(d, wgmma_desc_mn(al + ko, Cfg::BOX), wgmma_desc_mn(bh + ko, Cfg::BOX));
        wgmma_f16_mn<NCI>(d, wgmma_desc_mn(ah + ko, Cfg::BOX), wgmma_desc_mn(bl + ko, Cfg::BOX));
        wgmma_f16_mn<NCI>(d, wgmma_desc_mn(ah + ko, Cfg::BOX), wgmma_desc_mn(bh + ko, Cfg::BOX));
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(d);
      mbar_arrive(&empty[st]);
      if ((it + 1) % WGM_FLUSH == 0 || s + 1 == s_end) {
#pragma unroll
        for (int i = 0; i < NCI / 2; ++i) {
          acc[i] += d[i];
          d[i] = 0.f;
        }
      }
    }
    // acc[4 i + e] (d's layout) = D[16 (t / 32) + (t % 32) / 4 + 8 (e / 2)][8 i + 2 (t % 4) + (e % 2)]
    const int t = threadIdx.x & 127;
    double* out = a.partial + (static_cast<size_t>(blockIdx.x) * 9 + tap) * a.cout * a.cin;
#pragma unroll
    for (int i = 0; i < NCI / 8; ++i)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int co = co0 + 64 * cw + 16 * (t >> 5) + ((t & 31) >> 2) + 8 * (e >> 1);
        const int ci = ci0 + 8 * i + 2 * (t & 3) + (e & 1);
        out[static_cast<size_t>(co) * a.cin + ci] = static_cast<double>(acc[4 * i + e]);
      }
  }
}

// dW = (sum over chunks, in chunk order) * post / *dscale, in the reference layout [cout][cin][3][3].  Partials are
// [chunk][cout][cin][9] (wgrad_simt_kernel) or, with tap_major, [chunk][9][cout][cin] (wgrad_wgmma_kernel).
__global__ void wgrad_reduce_kernel(const double* __restrict__ partial, int chunks, int cout, int cin, int tap_major,
                                    double post, const float* __restrict__ dscale, float* __restrict__ dw) {
  const double inv = post / (dscale != nullptr ? static_cast<double>(dscale[0]) : 1.0);
  const size_t n = static_cast<size_t>(cout) * cin * 9;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t j = tap_major ? (i % 9) * cout * cin + i / 9 : i;
    double s = 0.0;
    for (int k = 0; k < chunks; ++k) s += partial[static_cast<size_t>(k) * n + j];
    dw[i] = static_cast<float>(s * inv);
  }
}

// W [cout][cin][3][3] -> W' [cin][cout][3][3] with W'[ci][co][ky][kx] = W[co][ci][2-ky][2-kx]: conv3x3(dY, W') = dX
__global__ void flip_transpose_weight_kernel(const float* __restrict__ w, float* __restrict__ wt, int cout, int cin) {
  const int n = cout * cin * 9;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int tap = i % 9, ci = (i / 9) % cin, co = i / (9 * cin);
    wt[(static_cast<size_t>(ci) * cout + co) * 9 + (8 - tap)] = w[i];
  }
}

// ------------------------------------------------------------------ adjoint of the align-corners bilinear upsample
// d [B][H][W][256] (times *dscale) -> out [B][ch][cw][256]: every condition pixel GATHERS the outputs that read it, with
// the forward's own source indices and weights (lerp_coord, fp32 ratios as ATen computes them) — no atomics.
__global__ void __launch_bounds__(256) up_adjoint_kernel(const float* __restrict__ d, const float* __restrict__ dscale,
                                                         int H, int W, int ch, int cw, float ry, float rx,
                                                         float* __restrict__ out) {
  const int cx = blockIdx.x, cy = blockIdx.y, b = blockIdx.z, c = threadIdx.x;
  // outputs whose source row is cy - 1 or cy: ry * oy in [cy - 1, cy + 1), widened by one row against rounding
  int y_lo = 0, y_hi = H - 1, x_lo = 0, x_hi = W - 1;
  if (ry > 0.f) {
    y_lo = max(0, static_cast<int>(floorf((cy - 1) / ry)) - 1);
    y_hi = min(H - 1, static_cast<int>(ceilf((cy + 1) / ry)) + 1);
  }
  if (rx > 0.f) {
    x_lo = max(0, static_cast<int>(floorf((cx - 1) / rx)) - 1);
    x_hi = min(W - 1, static_cast<int>(ceilf((cx + 1) / rx)) + 1);
  }
  float acc = 0.f;
  for (int oy = y_lo; oy <= y_hi; ++oy) {
    const Lerp1 ly = lerp_coord(ry, oy, ch);
    const float wy = (ly.i0 == cy ? ly.l0 : 0.f) + (ly.i1 == cy ? ly.l1 : 0.f);
    if (ly.i0 != cy && ly.i1 != cy) continue;
    for (int ox = x_lo; ox <= x_hi; ++ox) {
      const Lerp1 lx = lerp_coord(rx, ox, cw);
      if (lx.i0 != cx && lx.i1 != cx) continue;
      const float wx = (lx.i0 == cx ? lx.l0 : 0.f) + (lx.i1 == cx ? lx.l1 : 0.f);
      acc = fmaf(wy * wx, d[((static_cast<size_t>(b) * H + oy) * W + ox) * 256 + c], acc);
    }
  }
  const float inv = dscale != nullptr ? 1.f / dscale[0] : 1.f;
  out[((static_cast<size_t>(b) * ch + cy) * cw + cx) * 256 + c] = acc * inv;
}

// ------------------------------------------------------------------ walk back through the DDIM loop (dd_denoise_backward)
// x_{s+1} = c_x x_s + c_eps eps(x_s):  d_eps = c_eps g,  g <- c_x g + d_noisy.
__global__ void scale_copy_kernel(const float* __restrict__ x, float s, float* __restrict__ out, size_t n) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x)
    out[i] = s * x[i];
}
// g = cx * g + d / *dscale (dscale nullable = 1)
__global__ void latent_grad_step_kernel(float* __restrict__ g, const float* __restrict__ d, const float* __restrict__ dscale,
                                        float cx, size_t n) {
  const float inv = dscale != nullptr ? 1.f / dscale[0] : 1.f;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x)
    g[i] = fmaf(cx, g[i], d[i] * inv);
}
// acc += x / *scale in fp64 (scale nullable = 1; every scale here is a power of two, so the division is exact)
__global__ void acc_add_kernel(double* __restrict__ acc, const float* __restrict__ x, const float* __restrict__ scale,
                               size_t n) {
  const double inv = scale != nullptr ? 1.0 / static_cast<double>(scale[0]) : 1.0;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x)
    acc[i] += static_cast<double>(x[i]) * inv;
}
// time_embedding row of one step: acc_row += sum over images of d_temb[b], in image order (every image uses the row)
__global__ void temb_acc_kernel(double* __restrict__ acc_row, const float* __restrict__ dtemb, int B) {
  double s = 0.0;
  for (int b = 0; b < B; ++b) s += static_cast<double>(dtemb[b * 256 + threadIdx.x]);
  acc_row[threadIdx.x] += s;
}
__global__ void acc_store_kernel(const double* __restrict__ acc, float* __restrict__ out, size_t n) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x)
    out[i] = static_cast<float>(acc[i]);
}

// ------------------------------------------------------------------ decoder backward (reverse of decoder_kernel)
// Forward (kernels.cuh decoder_kernel): u = ConvT4x4/s2/p1(x) + b_t,  v = s (u - mean) + beta  (eval BatchNorm, s = gamma
// rstd; the forward evaluates v with the folded weights),  r = relu(v),  z = conv3x3(r, w_c) + b_c,
// depth = 1 / max(sigmoid(z), eps) - 1.  Reverse:
//   dz = -d_depth e^{-z} where sigmoid(z) >= eps, else 0 (torch.clamp's gradient);
//   dr(q) = sum_tap w_c[tap] dz(q - tap),  dw_c[ci][tap] = sum_q r[ci](q) dz(q - tap),  db_c = sum dz;
//   dv = dr [v > 0];  dbeta = sum dv,  dgamma = sum dv (u - mean) rstd,  du = s dv,  db_t = sum du = s dbeta;
//   dx(i) = sum over the 4 x 4 outputs o = 2 i - 1 + k of W_t[ci][co][k] du[co](o),  dW_t[ci][co][k] = sum_i x[ci](i) du[co](o).
// 16 channels: fp32 CUDA-core kernels.  Every reduction writes fixed per-block fp64 partials that dec_bwd_finish_kernel
// sums in block order.
constexpr int DEC_ACT_PIX = 1024;  // output pixels per block of dec_bwd_act_kernel (4 per thread)
constexpr int DEC_WC_PIX = 4096;   // output pixels per block of dec_bwd_wc_kernel
constexpr int DEC_WT_PIX = 1024;   // latent pixels per block of dec_bwd_wt_kernel
constexpr int DEC_ACT_N = 33;      // partials of dec_bwd_act_kernel: sum dv [16], sum dv * vhat [16], sum dz
constexpr int DEC_GRAD_N = 4096 + 16 + 16 + 16 + 144 + 1;  // the six decoder gradients, reference layouts back to back

struct DecBwdArgs {
  const float* x;   // latent NHWC [B][h][w][16]
  const float* wt;  // folded ConvT weights [ky][kx][ci][co] (the forward's)
  const float* bt;  // folded bias [16]
  const float* wu;  // unfolded ConvT weights [ky][kx][ci][co]
  const float* bu;  // unfolded bias [16]
  const float* bn;  // [3][16]: s = gamma * rstd, running mean, rstd
  const float* wc;  // final conv [tap][ci]
  const float* dz;  // [B][2h][2w]
  float* r;         // [B][2h][2w][16] relu output
  float* du;        // [B][2h][2w][16]
  double* part_act; // [blocks][DEC_ACT_N]
  double* part_wc;  // [blocks][144], column tap * 16 + ci
  double* part_wt;  // [blocks][4096], column ((ky * 4 + kx) * 16 + co) * 16 + ci
  float* dx;        // [B][h][w][16]
  int B, h, w;
};

// dz from the forward's logit z (in place) and d_depth [B][2h][2w]; sigmoid and the clamp test as decoder_kernel does them
__global__ void dec_dz_kernel(float* __restrict__ z, const float* __restrict__ d_depth, size_t n, float eps) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const float zv = z[i];
    const float s = 1.0f / (1.0f + expf(-zv));
    z[i] = s >= eps ? -d_depth[i] * expf(-zv) : 0.f;
  }
}

// One thread per output pixel: u and v again (v in the forward's own FMA order, so the ReLU mask and r are the forward's),
// dr from the 3 x 3 dz neighbourhood, then r, du and the per-block sums of dv, dv * vhat and dz.
__global__ void __launch_bounds__(256) dec_bwd_act_kernel(const DecBwdArgs a) {
  __shared__ __align__(16) float s_wt[4096];
  __shared__ __align__(16) float s_wu[4096];
  __shared__ double s_red[8][DEC_ACT_N];
  for (int i = threadIdx.x; i < 1024; i += 256) {
    reinterpret_cast<float4*>(s_wt)[i] = reinterpret_cast<const float4*>(a.wt)[i];
    reinterpret_cast<float4*>(s_wu)[i] = reinterpret_cast<const float4*>(a.wu)[i];
  }
  __syncthreads();
  const int H = 2 * a.h, W = 2 * a.w;
  const long long N = static_cast<long long>(a.B) * H * W;
  float acc[DEC_ACT_N];
#pragma unroll
  for (int j = 0; j < DEC_ACT_N; ++j) acc[j] = 0.f;
  const long long base = static_cast<long long>(blockIdx.x) * DEC_ACT_PIX;
  for (int k = 0; k < DEC_ACT_PIX / 256; ++k) {
    const long long q = base + k * 256 + threadIdx.x;
    if (q >= N) break;
    const int b = static_cast<int>(q / (static_cast<long long>(H) * W));
    const int Y = static_cast<int>((q / W) % H), X = static_cast<int>(q % W);
    float of[16], ou[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      of[c] = a.bt[c];
      ou[c] = a.bu[c];
    }
    const int ky0 = (Y + 1) & 1, kx0 = (X + 1) & 1;
#pragma unroll
    for (int a2 = 0; a2 < 2; ++a2) {
      const int ky = ky0 + 2 * a2;
      const int iy = (Y + 1 - ky) / 2;
      if (Y + 1 - ky < 0 || iy >= a.h) continue;
#pragma unroll
      for (int b2 = 0; b2 < 2; ++b2) {
        const int kx = kx0 + 2 * b2;
        const int ix = (X + 1 - kx) / 2;
        if (X + 1 - kx < 0 || ix >= a.w) continue;
        const float* lp = a.x + ((static_cast<size_t>(b) * a.h + iy) * a.w + ix) * 16;
        const float* wf = s_wt + (ky * 4 + kx) * 256;
        const float* wn = s_wu + (ky * 4 + kx) * 256;
#pragma unroll
        for (int ci = 0; ci < 16; ++ci) {
          const float v = lp[ci];
#pragma unroll
          for (int c = 0; c < 16; ++c) {
            of[c] = fmaf(v, wf[ci * 16 + c], of[c]);
            ou[c] = fmaf(v, wn[ci * 16 + c], ou[c]);
          }
        }
      }
    }
    float dzn[9];
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const int yy = Y - (tap / 3 - 1), xx = X - (tap % 3 - 1);
      dzn[tap] = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? a.dz[(static_cast<size_t>(b) * H + yy) * W + xx] : 0.f;
    }
    acc[32] += dzn[4];
    float rv[16], duv[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      float dr = 0.f;
#pragma unroll
      for (int tap = 0; tap < 9; ++tap) dr = fmaf(a.wc[tap * 16 + c], dzn[tap], dr);
      const bool on = of[c] > 0.f;
      const float dv = on ? dr : 0.f;
      rv[c] = on ? of[c] : 0.f;
      duv[c] = a.bn[c] * dv;
      acc[c] += dv;
      acc[16 + c] = fmaf(dv, (ou[c] - a.bn[16 + c]) * a.bn[32 + c], acc[16 + c]);
    }
    float4* rp = reinterpret_cast<float4*>(a.r + q * 16);
    float4* dp = reinterpret_cast<float4*>(a.du + q * 16);
#pragma unroll
    for (int c4 = 0; c4 < 4; ++c4) {
      rp[c4] = make_float4(rv[4 * c4], rv[4 * c4 + 1], rv[4 * c4 + 2], rv[4 * c4 + 3]);
      dp[c4] = make_float4(duv[4 * c4], duv[4 * c4 + 1], duv[4 * c4 + 2], duv[4 * c4 + 3]);
    }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < DEC_ACT_N; ++j) {
    double s = static_cast<double>(acc[j]);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) s_red[warp][j] = s;
  }
  __syncthreads();
  if (threadIdx.x < DEC_ACT_N) {
    double s = 0.0;
    for (int w8 = 0; w8 < 8; ++w8) s += s_red[w8][threadIdx.x];
    a.part_act[static_cast<size_t>(blockIdx.x) * DEC_ACT_N + threadIdx.x] = s;
  }
}

// dw_c: thread (tap, ci) = (t / 16, t % 16) walks the block's DEC_WC_PIX output pixels, fp32 for 256 pixels at a time.
__global__ void __launch_bounds__(160) dec_bwd_wc_kernel(const DecBwdArgs a) {
  const int t = threadIdx.x;
  if (t >= 144) return;
  const int tap = t / 16, ci = t % 16, dy = tap / 3 - 1, dx = tap % 3 - 1;
  const int H = 2 * a.h, W = 2 * a.w;
  const long long N = static_cast<long long>(a.B) * H * W;
  const long long q0 = static_cast<long long>(blockIdx.x) * DEC_WC_PIX, q1 = min(N, q0 + DEC_WC_PIX);
  double total = 0.0;
  for (long long s0 = q0; s0 < q1; s0 += 256) {
    float acc = 0.f;
    const long long s1 = min(q1, s0 + 256);
    for (long long q = s0; q < s1; ++q) {
      const int Y = static_cast<int>((q / W) % H), X = static_cast<int>(q % W);
      const int yy = Y - dy, xx = X - dx;
      if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;
      acc = fmaf(a.r[q * 16 + ci], a.dz[q + static_cast<long long>(-dy) * W - dx], acc);
    }
    total += static_cast<double>(acc);
  }
  a.part_wc[static_cast<size_t>(blockIdx.x) * 144 + t] = total;
}

// d_latent: one thread per latent pixel gathers its 4 x 4 output pixels (unfolded weights, transposed to [k][co][ci]).
__global__ void __launch_bounds__(256) dec_bwd_dx_kernel(const DecBwdArgs a) {
  __shared__ __align__(16) float s_w[4096];
  for (int i = threadIdx.x; i < 4096; i += 256) {
    const int k = i / 256, co = (i / 16) % 16, ci = i % 16;
    s_w[i] = a.wu[k * 256 + ci * 16 + co];
  }
  __syncthreads();
  const int H = 2 * a.h, W = 2 * a.w;
  const long long p = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (p >= static_cast<long long>(a.B) * a.h * a.w) return;
  const int b = static_cast<int>(p / (static_cast<long long>(a.h) * a.w));
  const int iy = static_cast<int>((p / a.w) % a.h), ix = static_cast<int>(p % a.w);
  float acc[16];
#pragma unroll
  for (int c = 0; c < 16; ++c) acc[c] = 0.f;
  for (int ky = 0; ky < 4; ++ky) {
    const int Y = 2 * iy - 1 + ky;
    if (Y < 0 || Y >= H) continue;
    for (int kx = 0; kx < 4; ++kx) {
      const int X = 2 * ix - 1 + kx;
      if (X < 0 || X >= W) continue;
      const float4* dp = reinterpret_cast<const float4*>(a.du + ((static_cast<size_t>(b) * H + Y) * W + X) * 16);
      const float* wk = s_w + (ky * 4 + kx) * 256;
#pragma unroll
      for (int c4 = 0; c4 < 4; ++c4) {
        const float4 d4 = dp[c4];
        const float dv[4] = {d4.x, d4.y, d4.z, d4.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float* wr = wk + (4 * c4 + j) * 16;
#pragma unroll
          for (int ci = 0; ci < 16; ++ci) acc[ci] = fmaf(dv[j], wr[ci], acc[ci]);
        }
      }
    }
  }
  float4* op = reinterpret_cast<float4*>(a.dx + p * 16);
#pragma unroll
  for (int c4 = 0; c4 < 4; ++c4) op[c4] = make_float4(acc[4 * c4], acc[4 * c4 + 1], acc[4 * c4 + 2], acc[4 * c4 + 3]);
}

// dW_t: thread (k, co) = (t / 16, t % 16) holds the 16 input channels; the block's latent pixels pass through shared
// memory 64 at a time and are flushed to fp64 after each stage.
__global__ void __launch_bounds__(256) dec_bwd_wt_kernel(const DecBwdArgs a) {
  __shared__ __align__(16) float s_x[64][16];
  const int t = threadIdx.x, k = t / 16, co = t % 16, ky = k / 4, kx = k % 4;
  const int H = 2 * a.h, W = 2 * a.w;
  const long long NP = static_cast<long long>(a.B) * a.h * a.w;
  const long long p0 = static_cast<long long>(blockIdx.x) * DEC_WT_PIX, p1 = min(NP, p0 + DEC_WT_PIX);
  double total[16];
#pragma unroll
  for (int c = 0; c < 16; ++c) total[c] = 0.0;
  for (long long s0 = p0; s0 < p1; s0 += 64) {
    const int n = static_cast<int>(min(64LL, p1 - s0));
    __syncthreads();
    {
      const int lp = t / 4, c4 = t % 4;
      if (lp < n) reinterpret_cast<float4*>(s_x[lp])[c4] = reinterpret_cast<const float4*>(a.x + (s0 + lp) * 16)[c4];
    }
    __syncthreads();
    float acc[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) acc[c] = 0.f;
    for (int j = 0; j < n; ++j) {
      const long long p = s0 + j;
      const int b = static_cast<int>(p / (static_cast<long long>(a.h) * a.w));
      const int iy = static_cast<int>((p / a.w) % a.h), ix = static_cast<int>(p % a.w);
      const int Y = 2 * iy - 1 + ky, X = 2 * ix - 1 + kx;
      if (Y < 0 || Y >= H || X < 0 || X >= W) continue;
      const float d = a.du[((static_cast<size_t>(b) * H + Y) * W + X) * 16 + co];
#pragma unroll
      for (int c4 = 0; c4 < 4; ++c4) {
        const float4 xv = reinterpret_cast<const float4*>(s_x[j])[c4];
        acc[4 * c4] = fmaf(xv.x, d, acc[4 * c4]);
        acc[4 * c4 + 1] = fmaf(xv.y, d, acc[4 * c4 + 1]);
        acc[4 * c4 + 2] = fmaf(xv.z, d, acc[4 * c4 + 2]);
        acc[4 * c4 + 3] = fmaf(xv.w, d, acc[4 * c4 + 3]);
      }
    }
#pragma unroll
    for (int c = 0; c < 16; ++c) total[c] += static_cast<double>(acc[c]);
  }
  double* out = a.part_wt + static_cast<size_t>(blockIdx.x) * 4096 + t * 16;
#pragma unroll
  for (int c = 0; c < 16; ++c) out[c] = total[c];
}

// The six gradients in the reference layouts, each partial column summed over the blocks in block order:
// out[0] ConvT weight [16 ci][16 co][4][4], out[1] its bias, out[2] BN weight, out[3] BN bias, out[4] conv [1][16][3][3],
// out[5] conv bias (each nullable).
struct DecFinishArgs {
  const double* part_act;
  const double* part_wc;
  const double* part_wt;
  int nb_act, nb_wc, nb_wt;
  const float* bn;
  float* out[6];
};
__global__ void dec_bwd_finish_kernel(const DecFinishArgs f) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= DEC_GRAD_N) return;
  double s = 0.0;
  float* dst;
  int o;
  if (i < 4096) {  // [ci][co][ky][kx] <- column ((ky * 4 + kx) * 16 + co) * 16 + ci
    const int ci = i / 256, co = (i / 16) % 16, k = i % 16;
    const int col = (k * 16 + co) * 16 + ci;
    for (int b = 0; b < f.nb_wt; ++b) s += f.part_wt[static_cast<size_t>(b) * 4096 + col];
    dst = f.out[0];
    o = i;
  } else if (i < 4096 + 48) {  // ConvT bias = s * sum dv, BN weight = sum dv * vhat, BN bias = sum dv
    const int j = i - 4096, c = j % 16, which = j / 16;
    const int col = which == 1 ? 16 + c : c;
    for (int b = 0; b < f.nb_act; ++b) s += f.part_act[static_cast<size_t>(b) * DEC_ACT_N + col];
    if (which == 0) s *= static_cast<double>(f.bn[c]);
    dst = which == 0 ? f.out[1] : (which == 1 ? f.out[2] : f.out[3]);  // constant indices: no local-memory copy of f
    o = c;
  } else if (i < 4096 + 48 + 144) {  // [ci][tap] <- column tap * 16 + ci
    const int j = i - 4096 - 48, ci = j / 9, tap = j % 9;
    for (int b = 0; b < f.nb_wc; ++b) s += f.part_wc[static_cast<size_t>(b) * 144 + tap * 16 + ci];
    dst = f.out[4];
    o = j;
  } else {
    for (int b = 0; b < f.nb_act; ++b) s += f.part_act[static_cast<size_t>(b) * DEC_ACT_N + 32];
    dst = f.out[5];
    o = 0;
  }
  if (dst != nullptr) dst[o] = static_cast<float>(s);
}

}  // namespace dd
