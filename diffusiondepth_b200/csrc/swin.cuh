// Swin Transformer pieces that are not GEMMs (the GEMMs run on convgen_wgmma_kernel in "GEMM mode"):
// patch embedding (4x4/s4 conv + LayerNorm), LayerNorm -> fp16 hi/lo planes, 2x2 patch-merge gather + LayerNorm,
// 7x7 (shifted-)window attention with relative-position bias and the reference's finite -100 shift mask,
// per-stage output LayerNorm written straight into the neck's input planes.
// Token stream layout: x fp32 [B*H*W][C] (NHWC flattened), qkv fp32 [M][3C] with the reference's [3][nH][32]
// column interleave.  Restates reference src/model/backbone/swin.py (PatchMerging :64-88, WindowMSA :150-189,
// ShiftWindowMSA :250-325, SwinBlock :426-437, SwinTransformer.forward :756-777) and
// backbone/utils.py:282-302 (PatchEmbedSwin); parity traps: SURVEY.md Appendix C.
#pragma once
#include "kernels.cuh"

namespace dd {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// LayerNorm statistics of one warp's token: v[i] holds channel lane + 32 i, the first C channels real (the others 0).
// Centres v in place (the others stay 0) and returns rstd = 1 / sqrt(var + eps).  The mean in two parts: the fp32 mean
// m0, then the mean mc of v - m0.  A row with a large mean and a small spread (1e3 +- 1e-2) would otherwise lose the
// spread to m0's rounding (~1e-4 there), and a constant row would come out as rounding noise times rsqrt(eps) instead
// of beta; v - m0 is exact for v within a factor 2 of m0.
template <int N>
__device__ __forceinline__ float warp_ln_centre(float (&v)[N], int C, float eps) {
  const int lane = threadIdx.x & 31;
  const float inv_c = 1.f / static_cast<float>(C);
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < N; ++i) s += v[i];
  const float m0 = warp_sum(s) * inv_c;
  float s1 = 0.f;
#pragma unroll
  for (int i = 0; i < N; ++i) {
    v[i] = (lane + 32 * i < C) ? v[i] - m0 : 0.f;
    s1 += v[i];
  }
  const float mc = warp_sum(s1) * inv_c;
  float s2 = 0.f;
#pragma unroll
  for (int i = 0; i < N; ++i) {
    v[i] = (lane + 32 * i < C) ? v[i] - mc : 0.f;
    s2 = fmaf(v[i], v[i], s2);
  }
  return rsqrtf(warp_sum(s2) * inv_c + eps);
}

// ------------------------------------------------------------------ LayerNorm(C) -> scaled fp16 hi/lo planes
// one warp per token; C = 32 * VPT elements (VPT <= 48).  Optionally also writes fp32 NCHW (stage outputs).
template <int C>
__global__ void __launch_bounds__(256) ln_split_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                                       const float* __restrict__ beta, __half* __restrict__ hi,
                                                       __half* __restrict__ lo, float scale, int M, float* nchw_out,
                                                       int HW, int* status) {
  constexpr int VPT = C / 32;
  const int token = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (token >= M) return;
  const float* row = x + static_cast<size_t>(token) * C;
  float v[VPT];
#pragma unroll
  for (int i = 0; i < VPT; ++i) v[i] = row[lane + 32 * i];
  const float rstd = warp_ln_centre(v, C, 1e-5f);
  bool ov = false;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int c = lane + 32 * i;
    const float y = v[i] * rstd * gamma[c] + beta[c];
    __half h, l;
    split_f16(y, scale, h, l, ov);
    hi[static_cast<size_t>(token) * C + c] = h;
    lo[static_cast<size_t>(token) * C + c] = l;
    if (nchw_out) {
      const int b = token / HW, p = token - b * HW;
      nchw_out[(static_cast<size_t>(b) * C + c) * HW + p] = y;
    }
  }
  if (ov) atomicOr(status, 1);
}

// ------------------------------------------------------------------ patch embed: conv 4x4 s4 (3 -> E) + bias + LayerNorm(E)
// rgb fp32 NCHW [B,3,H,W] (zero right/bottom pad to a multiple of 4) -> x fp32 [B*Hp*Wp][E].  One block of E threads =
// PE_TOK consecutive tokens of one token row: their 3 x 4 image rows are 12 contiguous runs of 4 * PE_TOK floats, loaded
// coalesced into shared memory (a per-token gather keeps L1 saturated);
// thread e then holds the 48 weights of output channel e and walks the tokens 8 at a time.
constexpr int PE_TOK = 32;
template <int E>
__global__ void __launch_bounds__(E) patch_embed_kernel(const float* __restrict__ rgb, const float* __restrict__ w,
                                                        const float* __restrict__ bias, const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, float* __restrict__ x, int B, int H,
                                                        int W, int Hp, int Wp) {
  constexpr int TOK = 8;  // tokens per inner group
  __shared__ __align__(16) float patch[PE_TOK][48];  // [token][c*16 + ky*4 + kx]: read back as broadcast float4s
  __shared__ float red[3][TOK][E / 32];  // per-warp sums of v, of v - m0 and of the centred squares
  const int segs = (Wp + PE_TOK - 1) / PE_TOK;
  const int seg = blockIdx.x % segs, py = (blockIdx.x / segs) % Hp, b = blockIdx.x / (segs * Hp);
  const int px0 = seg * PE_TOK;
  for (int i = threadIdx.x; i < 12 * 4 * PE_TOK; i += E) {
    const int xx = i % (4 * PE_TOK), rowi = i / (4 * PE_TOK);  // rowi = c*4 + ky
    const int c = rowi >> 2, ky = rowi & 3;
    const int yy = py * 4 + ky, gx = px0 * 4 + xx;
    float v = 0.f;
    if (yy < H && gx < W) v = rgb[((static_cast<size_t>(b) * 3 + c) * H + yy) * W + gx];
    patch[xx >> 2][c * 16 + ky * 4 + (xx & 3)] = v;
  }
  __syncthreads();
  const int e = threadIdx.x;
  float wr[48];
#pragma unroll
  for (int k = 0; k < 48; ++k) wr[k] = w[e * 48 + k];
  const float be = bias[e], ga = gamma[e], bt = beta[e];
  const int warp = e >> 5, lane = e & 31;
  for (int g0 = 0; g0 < PE_TOK; g0 += TOK) {
    if (px0 + g0 >= Wp) break;  // block-uniform
    float acc[TOK];
#pragma unroll
    for (int tk = 0; tk < TOK; ++tk) {
      float a = be;
#pragma unroll
      for (int k4 = 0; k4 < 12; ++k4) {  // one 16-byte broadcast load feeds four FMAs
        const float4 pv = *reinterpret_cast<const float4*>(&patch[g0 + tk][4 * k4]);
        a = fmaf(pv.x, wr[4 * k4], a);
        a = fmaf(pv.y, wr[4 * k4 + 1], a);
        a = fmaf(pv.z, wr[4 * k4 + 2], a);
        a = fmaf(pv.w, wr[4 * k4 + 3], a);
      }
      acc[tk] = a;
    }
#pragma unroll
    for (int tk = 0; tk < TOK; ++tk) {
      const float s = warp_sum(acc[tk]);
      if (lane == 0) red[0][tk][warp] = s;
    }
    __syncthreads();
    // the mean in two parts, m0 then the mean of acc - m0, as warp_ln_centre takes it; acc is centred in place
#pragma unroll
    for (int tk = 0; tk < TOK; ++tk) {
      float s = 0.f;
#pragma unroll
      for (int wv = 0; wv < E / 32; ++wv) s += red[0][tk][wv];
      acc[tk] -= s * (1.f / E);
      const float s1 = warp_sum(acc[tk]);
      if (lane == 0) red[1][tk][warp] = s1;
    }
    __syncthreads();
#pragma unroll
    for (int tk = 0; tk < TOK; ++tk) {
      float s1 = 0.f;
#pragma unroll
      for (int wv = 0; wv < E / 32; ++wv) s1 += red[1][tk][wv];
      acc[tk] -= s1 * (1.f / E);
      const float s2 = warp_sum(acc[tk] * acc[tk]);
      if (lane == 0) red[2][tk][warp] = s2;
    }
    __syncthreads();
#pragma unroll
    for (int tk = 0; tk < TOK; ++tk) {
      float s2 = 0.f;
#pragma unroll
      for (int wv = 0; wv < E / 32; ++wv) s2 += red[2][tk][wv];
      const float rstd = rsqrtf(s2 * (1.f / E) + 1e-5f);
      const int px = px0 + g0 + tk;
      if (px < Wp) x[(static_cast<size_t>(b) * Hp * Wp + static_cast<size_t>(py) * Wp + px) * E + e] = acc[tk] * rstd * ga + bt;
    }
    __syncthreads();  // red[] is reused by the next group
  }
}

// ------------------------------------------------------------------ patch merging gather + LayerNorm(4C) -> planes
// x [B,H,W,C] -> tokens [B,(H+1)/2,(W+1)/2,4C] with feature index c*4 + ky*2 + kx (nn.Unfold order), zero pad
// for odd H/W, then LayerNorm over 4C.  One warp per output token.
template <int C>
__global__ void __launch_bounds__(256) merge_ln_split_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                                             const float* __restrict__ beta, __half* __restrict__ hi,
                                                             __half* __restrict__ lo, float scale, int B, int H, int W,
                                                             int* status) {
  constexpr int F = 4 * C, VPT = F / 32;
  const int H2 = (H + 1) / 2, W2 = (W + 1) / 2;
  const int M2 = B * H2 * W2;
  const int token = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (token >= M2) return;
  const int b = token / (H2 * W2), r = token % (H2 * W2), oy = r / W2, ox = r % W2;
  float v[VPT];
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int f = lane + 32 * i;
    const int c = f >> 2, ky = (f >> 1) & 1, kx = f & 1;
    const int yy = 2 * oy + ky, xx = 2 * ox + kx;
    v[i] = (yy < H && xx < W) ? x[((static_cast<size_t>(b) * H + yy) * W + xx) * C + c] : 0.f;
  }
  const float rstd = warp_ln_centre(v, F, 1e-5f);
  bool ov = false;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int f = lane + 32 * i;
    const float y = v[i] * rstd * gamma[f] + beta[f];
    __half h, l;
    split_f16(y, scale, h, l, ov);
    hi[static_cast<size_t>(token) * F + f] = h;
    lo[static_cast<size_t>(token) * F + f] = l;
  }
  if (ov) atomicOr(status, 1);
}

// ------------------------------------------------------------------ (shifted) 7x7 window attention, head_dim 32
// One block (64 threads) per (window, head).  The reference pads the *normalised* tokens with zeros before the
// qkv Linear, so a padded token carries q/k/v = the qkv bias; it attends and is attended to (only the shift mask,
// built from 3x3 region ids on the padded map, hides anything).  Output: attention result scattered back to the
// un-rolled, un-padded token positions as fp16 hi/lo planes [M][C] (input of the proj GEMM).
struct AttnArgs {
  const float* qkv;        // [M][3C]
  const float* qkv_bias;   // [3C]
  const float* bias_table; // [169][nH]
  __half* out_hi;
  __half* out_lo;
  float scale_out;
  int B, H, W, C, nH, shift;
  int Hp, Wp, nWx, nWy;
  int* status;
};
__global__ void __launch_bounds__(64) window_attention_kernel(const AttnArgs a) {
  constexpr int WS = 7, N = 49, D = 32;
  __shared__ __align__(16) float sk[N][D];   // read as broadcast float4 rows
  __shared__ __align__(16) float sv[N][D];
  __shared__ float sp[N][N + 1];             // scores / probabilities, one row per query thread
  __shared__ int s_tok[N];                   // source token index or -1 for padding
  __shared__ int s_reg[N];                   // shift-mask region id
  const int head = blockIdx.x % a.nH;
  const int win = blockIdx.x / a.nH;
  const int wx = win % a.nWx, wy = (win / a.nWx) % a.nWy, b = win / (a.nWx * a.nWy);
  const int tid = threadIdx.x;
  if (tid < N) {
    const int iy = tid / WS, ix = tid % WS;
    const int sy = wy * WS + iy, sx = wx * WS + ix;  // coordinates in the rolled, padded frame
    int reg = 0;
    if (a.shift > 0) {
      const int ry = sy < a.Hp - WS ? 0 : (sy < a.Hp - a.shift ? 1 : 2);
      const int rx = sx < a.Wp - WS ? 0 : (sx < a.Wp - a.shift ? 1 : 2);
      reg = ry * 3 + rx;
    }
    const int py = (sy + a.shift) % a.Hp, px = (sx + a.shift) % a.Wp;  // torch.roll(x, -shift)[i] = x[(i+shift) % n]
    s_tok[tid] = (py < a.H && px < a.W) ? (b * a.H + py) * a.W + px : -1;
    s_reg[tid] = reg;
  }
  __syncthreads();
  // k, v rows -> shared (8 lanes x float4 per row)
  for (int i = tid; i < N * (D / 4); i += 64) {
    const int t = i / (D / 4), d4 = i % (D / 4);
    const int tok = s_tok[t];
    const int col = head * D + d4 * 4;
    const float* base = tok >= 0 ? a.qkv + static_cast<size_t>(tok) * 3 * a.C : a.qkv_bias;
    *reinterpret_cast<float4*>(&sk[t][d4 * 4]) = *reinterpret_cast<const float4*>(base + a.C + col);
    *reinterpret_cast<float4*>(&sv[t][d4 * 4]) = *reinterpret_cast<const float4*>(base + 2 * a.C + col);
  }
  // own query row -> registers, pre-scaled by head_dim ** -0.5 (applied to q before q @ k^T, swin.py:163)
  const int i = tid < N ? tid : N - 1;
  float q[D];
  {
    const int tok = s_tok[i];
    const float* base = (tok >= 0 ? a.qkv + static_cast<size_t>(tok) * 3 * a.C : a.qkv_bias) + head * D;
    const float qscale = rsqrtf(static_cast<float>(D));
#pragma unroll
    for (int d4 = 0; d4 < D / 4; ++d4) {
      const float4 t = *reinterpret_cast<const float4*>(base + d4 * 4);
      q[4 * d4] = t.x * qscale;
      q[4 * d4 + 1] = t.y * qscale;
      q[4 * d4 + 2] = t.z * qscale;
      q[4 * d4 + 3] = t.w * qscale;
    }
  }
  __syncthreads();
  if (tid >= N) return;
  const int iy = i / WS, ix = i % WS;
  const int my_reg = s_reg[i];
  float* p = sp[i];
  float mx = -INFINITY;
  for (int j = 0; j < N; ++j) {
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
    for (int d4 = 0; d4 < D / 4; ++d4) {
      const float4 kk = *reinterpret_cast<const float4*>(&sk[j][d4 * 4]);
      s0 = fmaf(q[4 * d4], kk.x, s0);
      s1 = fmaf(q[4 * d4 + 1], kk.y, s1);
      s2 = fmaf(q[4 * d4 + 2], kk.z, s2);
      s3 = fmaf(q[4 * d4 + 3], kk.w, s3);
    }
    float s = (s0 + s1) + (s2 + s3);
    const int jy = j / WS, jx = j - jy * WS;
    const int rel = (iy - jy + WS - 1) * (2 * WS - 1) + (ix - jx + WS - 1);
    s += __ldg(a.bias_table + rel * a.nH + head);
    if (a.shift > 0 && my_reg != s_reg[j]) s += -100.0f;
    p[j] = s;
    mx = fmaxf(mx, s);
  }
  float sum = 0.f;
  for (int j = 0; j < N; ++j) {
    const float e = expf(p[j] - mx);
    p[j] = e;
    sum += e;
  }
  const float inv = 1.f / sum;
  float o[D];
#pragma unroll
  for (int d = 0; d < D; ++d) o[d] = 0.f;
  for (int j = 0; j < N; ++j) {
    const float pj = p[j] * inv;
#pragma unroll
    for (int d4 = 0; d4 < D / 4; ++d4) {
      const float4 vv = *reinterpret_cast<const float4*>(&sv[j][d4 * 4]);
      o[4 * d4] = fmaf(pj, vv.x, o[4 * d4]);
      o[4 * d4 + 1] = fmaf(pj, vv.y, o[4 * d4 + 1]);
      o[4 * d4 + 2] = fmaf(pj, vv.z, o[4 * d4 + 2]);
      o[4 * d4 + 3] = fmaf(pj, vv.w, o[4 * d4 + 3]);
    }
  }
  const int tok = s_tok[i];
  if (tok < 0) return;  // padded query rows are cropped by the reference (:319-320)
  bool ov = false;
  __align__(16) __half hh[D];
  __align__(16) __half ll[D];
#pragma unroll
  for (int d = 0; d < D; ++d) split_f16(o[d], a.scale_out, hh[d], ll[d], ov);
  uint4* dh = reinterpret_cast<uint4*>(a.out_hi + static_cast<size_t>(tok) * a.C + head * D);
  uint4* dl = reinterpret_cast<uint4*>(a.out_lo + static_cast<size_t>(tok) * a.C + head * D);
#pragma unroll
  for (int d = 0; d < 4; ++d) {
    dh[d] = reinterpret_cast<const uint4*>(hh)[d];
    dl[d] = reinterpret_cast<const uint4*>(ll)[d];
  }
  if (ov) atomicOr(a.status, 1);
}


// ------------------------------------------------------------------ (shifted) 7x7 window attention on wgmma
// QK^T and PV as 3-pass fp16-split warpgroup MMAs with fp32 register accumulators; softmax in registers.  One
// persistent CTA (128 threads = one warpgroup) walks PAIRS of (window, head) units — the two units of a pair are two
// consecutive heads of the same window — and after each product thread t owns row t: unit t / 64, query t % 64 (49
// real rows, 15 zero rows).
//   gather   q (pre-scaled by head_dim^-0.5), k, v rows from the fp32 qkv stream (padded tokens carry the qkv bias,
//            exactly as in window_attention_kernel), split into fp16 hi / lo planes and WRITE them into shared memory in
//            the swizzled K-major layouts wgmma reads: Q [128 x 32] and K_u [64 x 32] with 64-byte rows (16-byte chunk
//            c of row r at chunk c ^ ((r >> 1) & 3)), V_u transposed [32 dims x 64 keys] with 128-byte rows (chunk
//            c ^ (r & 7));
//   S        S_u = Q_u K_u^T: 3 passes x 2 K-steps of m64n64k16 per unit;
//   softmax  the accumulators go through a shared-memory staging tile so that each thread holds its row; it adds the
//            relative-position bias and the finite -100 shift mask, takes the softmax over the 49 keys in fp32 and writes
//            P (x 4096) as hi / lo planes [128 x 64], 128-byte rows;
//   O        O_u = P_u V_u: 3 passes x 4 K-steps of m64n32k16 per unit;
//   store    staged again, each thread splits its 32 outputs and writes the proj GEMM's input planes.
// P re-uses the Q / K tiles (they are dead once the S products have completed).  Replaces reference swin.py:150-189 /
// 250-325.
constexpr int WAU_LD_S = 65, WAU_LD_O = 33;  // staging row strides (floats): conflict-free row reads
constexpr int WAU_SMEM = 32768 /*Q + K, then P*/ + 16384 /*Vt*/ + 128 * WAU_LD_S * 4 /*staging*/ + 1024 /*align*/ +
                         1024 /*ctrl*/;
__device__ __forceinline__ void wau_split8(const float* v, float scale, uint4& hi, uint4& lo, bool& ov) {
  __align__(16) __half2 h[4];
  __align__(16) __half2 l[4];
  float amax = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float s0 = v[2 * j] * scale, s1 = v[2 * j + 1] * scale;
    amax = fmaxf(amax, fmaxf(fabsf(s0), fabsf(s1)));
    h[j] = __floats2half2_rn(s0, s1);
    const float2 b = __half22float2(h[j]);
    l[j] = __floats2half2_rn(s0 - b.x, s1 - b.y);
  }
  ov |= !(amax <= 60000.f);
  hi = *reinterpret_cast<const uint4*>(h);
  lo = *reinterpret_cast<const uint4*>(l);
}
__global__ void __launch_bounds__(128, 2) window_attention_wgmma_kernel(const AttnArgs a, int num_pairs) {
  constexpr int WS = 7, N = 49, D = 32;
  constexpr float kP = 4096.f;  // probabilities are split at this scale
  extern __shared__ uint8_t wau_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(wau_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;                 // [plane][128 rows][64 B]
  uint8_t* sK = smem + 16384;         // [unit][plane][64 rows][64 B]
  uint8_t* sP = smem;                 // [plane][128 rows][128 B]: over Q and K, written after the S products have completed
  uint8_t* sV = smem + 32768;         // [unit][plane][32 rows][128 B]
  float* stg = reinterpret_cast<float*>(smem + 49152);          // [128][WAU_LD_S] (S), then [128][WAU_LD_O] (O)
  uint8_t* ctrl = smem + 49152 + 128 * WAU_LD_S * 4;
  int* s_tok = reinterpret_cast<int*>(ctrl);                    // [49] source token or -1
  int* s_reg = s_tok + 64;                                      // [49] shift-mask region id
  const int t = threadIdx.x;
  const int u = t >> 6, i = t & 63;                             // unit within the pair, query row
  const float qscale = rsqrtf(static_cast<float>(D));
  const int heads_half = a.nH >> 1;
  bool ov = false;
  for (int pair = blockIdx.x; pair < num_pairs; pair += gridDim.x) {
    const int hp = pair % heads_half, win = pair / heads_half;
    const int head = 2 * hp + u;
    const int wx = win % a.nWx, wy = (win / a.nWx) % a.nWy, b = win / (a.nWx * a.nWy);
    if (t < N) {
      const int iy = t / WS, ix = t % WS;
      const int sy = wy * WS + iy, sx = wx * WS + ix;  // coordinates in the rolled, padded frame
      int reg = 0;
      if (a.shift > 0) {
        const int ry = sy < a.Hp - WS ? 0 : (sy < a.Hp - a.shift ? 1 : 2);
        const int rx = sx < a.Wp - WS ? 0 : (sx < a.Wp - a.shift ? 1 : 2);
        reg = ry * 3 + rx;
      }
      const int py = (sy + a.shift) % a.Hp, px = (sx + a.shift) % a.Wp;  // torch.roll(x, -shift)[i] = x[(i+shift) % n]
      s_tok[t] = (py < a.H && px < a.W) ? (b * a.H + py) * a.W + px : -1;
      s_reg[t] = reg;
    }
    __syncthreads();
    // ---------------------------------------------------------------- gather + split + swizzled operand writes
    const int tok = i < N ? s_tok[i] : -1;
    {
      const float* base = (tok >= 0 ? a.qkv + static_cast<size_t>(tok) * 3 * a.C : a.qkv_bias) + head * D;
      const uint32_t rq = static_cast<uint32_t>(t), rk = static_cast<uint32_t>(i);
#pragma unroll
      for (int c = 0; c < 4; ++c) {  // 16-byte chunks of 8 dims
        float q8[8], k8[8];
#pragma unroll
        for (int h4 = 0; h4 < 2; ++h4) {
          float4 qa = make_float4(0.f, 0.f, 0.f, 0.f), ka = qa;
          if (i < N) {
            qa = *reinterpret_cast<const float4*>(base + 8 * c + 4 * h4);
            ka = *reinterpret_cast<const float4*>(base + a.C + 8 * c + 4 * h4);
          }
          q8[4 * h4] = qa.x * qscale; q8[4 * h4 + 1] = qa.y * qscale; q8[4 * h4 + 2] = qa.z * qscale; q8[4 * h4 + 3] = qa.w * qscale;
          k8[4 * h4] = ka.x; k8[4 * h4 + 1] = ka.y; k8[4 * h4 + 2] = ka.z; k8[4 * h4 + 3] = ka.w;
        }
        uint4 hi, lo;
        wau_split8(q8, a.scale_out, hi, lo, ov);
        const uint32_t oq = rq * 64 + ((static_cast<uint32_t>(c) ^ ((rq >> 1) & 3u)) << 4);
        *reinterpret_cast<uint4*>(sQ + oq) = hi;
        *reinterpret_cast<uint4*>(sQ + 8192 + oq) = lo;
        wau_split8(k8, a.scale_out, hi, lo, ov);
        const uint32_t ok = rk * 64 + ((static_cast<uint32_t>(c) ^ ((rk >> 1) & 3u)) << 4);
        *reinterpret_cast<uint4*>(sK + u * 8192 + ok) = hi;
        *reinterpret_cast<uint4*>(sK + u * 8192 + 4096 + ok) = lo;
      }
      // V transposed: element (dim d, key i) of unit u -> row d (128 B), 16-byte chunk (i >> 3) ^ (d & 7), half (i & 7)
#pragma unroll
      for (int d4 = 0; d4 < D / 4; ++d4) {
        float4 va = make_float4(0.f, 0.f, 0.f, 0.f);
        if (i < N) va = *reinterpret_cast<const float4*>(base + 2 * a.C + 4 * d4);
        const float vv[4] = {va.x, va.y, va.z, va.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint32_t d = 4 * d4 + j;
          const float sc = vv[j] * a.scale_out;
          ov |= !(fabsf(sc) <= 60000.f);
          const __half h = __float2half_rn(sc);
          const __half l = __float2half_rn(sc - __half2float(h));
          const uint32_t o = d * 128 + (((static_cast<uint32_t>(i) >> 3) ^ (d & 7u)) << 4) + ((static_cast<uint32_t>(i) & 7u) << 1);
          *reinterpret_cast<__half*>(sV + u * 8192 + o) = h;
          *reinterpret_cast<__half*>(sV + u * 8192 + 4096 + o) = l;
        }
      }
    }
    fence_proxy_async();
    __syncthreads();
    // ---------------------------------------------------------------- S_u = Q_u K_u^T  (lo*hi, hi*lo, hi*hi per K-step)
    float pr[64];
    {
      float sacc[2][32];
      wgmma_fence();
      const uint32_t q_hi = smem_u32(sQ), q_lo = q_hi + 8192;
#pragma unroll
      for (int uu = 0; uu < 2; ++uu) {
        const uint32_t k_hi = smem_u32(sK) + uu * 8192, k_lo = k_hi + 4096;
        const uint32_t qo = uu * 64 * 64;
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          wgmma_f16<64>(sacc[uu], wgmma_desc(q_lo + qo + k * 32, 64), wgmma_desc(k_hi + k * 32, 64), k ? 1u : 0u);
          wgmma_f16<64>(sacc[uu], wgmma_desc(q_hi + qo + k * 32, 64), wgmma_desc(k_lo + k * 32, 64), 1u);
          wgmma_f16<64>(sacc[uu], wgmma_desc(q_hi + qo + k * 32, 64), wgmma_desc(k_hi + k * 32, 64), 1u);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(sacc[0]);
      wgmma_fence_regs(sacc[1]);
      stage_acc_cols<64, 64, WAU_LD_S>(sacc[0], stg, 0, 0);
      stage_acc_cols<64, 64, WAU_LD_S>(sacc[1], stg, 64, 0);
      __syncthreads();
      const float inv = 1.f / (a.scale_out * a.scale_out);
#pragma unroll
      for (int j = 0; j < 64; ++j) pr[j] = stg[t * WAU_LD_S + j] * inv;
    }
    // ---------------------------------------------------------------- softmax of row (u, i)
    if (i < N) {
      const int iy = i / WS, ix = i - iy * WS;
      const int my_reg = s_reg[i];
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < N; ++j) {
        const int jy = j / WS, jx = j - jy * WS;
        const int rel = (iy - jy + WS - 1) * (2 * WS - 1) + (ix - jx + WS - 1);
        float sv = pr[j] + __ldg(a.bias_table + rel * a.nH + head);
        if (a.shift > 0 && my_reg != s_reg[j]) sv += -100.0f;
        pr[j] = sv;
        mx = fmaxf(mx, sv);
      }
      float sum = 0.f;
#pragma unroll
      for (int j = 0; j < N; ++j) {
        pr[j] = expf(pr[j] - mx);
        sum += pr[j];
      }
      const float rs = kP / sum;
#pragma unroll
      for (int j = 0; j < N; ++j) pr[j] *= rs;
#pragma unroll
      for (int j = N; j < 64; ++j) pr[j] = 0.f;
    } else {
#pragma unroll
      for (int j = 0; j < 64; ++j) pr[j] = 0.f;
    }
    __syncthreads();  // every thread has read its S row: the staging tile is free again
    {
      const uint32_t rp = static_cast<uint32_t>(t);
      bool dummy = false;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        uint4 hi, lo;
        wau_split8(pr + 8 * c, 1.f, hi, lo, dummy);  // 0 <= P * 4096 <= 4096: always in range
        const uint32_t o = rp * 128 + ((static_cast<uint32_t>(c) ^ (rp & 7u)) << 4);
        *reinterpret_cast<uint4*>(sP + o) = hi;
        *reinterpret_cast<uint4*>(sP + 16384 + o) = lo;
      }
    }
    fence_proxy_async();
    __syncthreads();
    // ---------------------------------------------------------------- O_u = P_u V_u
    {
      float oacc[2][16];
      wgmma_fence();
      const uint32_t p_hi = smem_u32(sP), p_lo = p_hi + 16384;
#pragma unroll
      for (int uu = 0; uu < 2; ++uu) {
        const uint32_t v_hi = smem_u32(sV) + uu * 8192, v_lo = v_hi + 4096;
        const uint32_t po = uu * 64 * 128;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          wgmma_f16<32>(oacc[uu], wgmma_desc(p_lo + po + k * 32, 128), wgmma_desc(v_hi + k * 32, 128), k ? 1u : 0u);
          wgmma_f16<32>(oacc[uu], wgmma_desc(p_hi + po + k * 32, 128), wgmma_desc(v_lo + k * 32, 128), 1u);
          wgmma_f16<32>(oacc[uu], wgmma_desc(p_hi + po + k * 32, 128), wgmma_desc(v_hi + k * 32, 128), 1u);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(oacc[0]);
      wgmma_fence_regs(oacc[1]);
      stage_acc_cols<32, 32, WAU_LD_O>(oacc[0], stg, 0, 0);
      stage_acc_cols<32, 32, WAU_LD_O>(oacc[1], stg, 64, 0);
      __syncthreads();
      if (tok >= 0) {  // padded query rows are cropped by the reference (:319-320); rows >= 49 do not exist
        const float inv = 1.f / (kP * a.scale_out);
        uint4* dh = reinterpret_cast<uint4*>(a.out_hi + static_cast<size_t>(tok) * a.C + head * D);
        uint4* dl = reinterpret_cast<uint4*>(a.out_lo + static_cast<size_t>(tok) * a.C + head * D);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          float o8[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) o8[j] = stg[t * WAU_LD_O + 8 * c + j] * inv;
          uint4 hi, lo;
          wau_split8(o8, a.scale_out, hi, lo, ov);
          dh[c] = hi;
          dl[c] = lo;
        }
      }
    }
    __syncthreads();  // the staging tile and the operand tiles are free for the next pair
  }
  if (ov) atomicOr(a.status, 1);
}

}  // namespace dd
