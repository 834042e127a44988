// The reference's other learned depth codecs (src/model/ops/depth_transform.py), eval-mode BatchNorm folded into the
// weights on the host in fp64, fp32 CUDA-core work like encoder_kernel / decoder_kernel:
//   DD_CODEC_UP2_1X1  DeepDepthTransformWithUpsampling1x1 (:38-64): encoder_1x1; its decoder is decoder_kernel
//   DD_CODEC_UP4      DeepDepthTransformWithUpsamplingX4  (:67-94): encoder_x4, decoder_x4
//   DD_CODEC_FULL     DeepDepthTransform                  (:97-117): encoder_full, decoder_full
// conv_bn_relu = src/model/common.py:45-60 (no conv bias before a BatchNorm, LeakyReLU(0.2)).
// Every fused kernel keeps its intermediates in shared memory as tiles of pixels x 16 channels with a row stride of
// CS = 20 floats (16-byte aligned rows; conflict-free scalar reads across the 8 pixels of a warp at stride 1).
#pragma once
#include <cuda_runtime.h>

namespace dd {

constexpr int CK_CS = 20;

// 3x3 conv, pad 1, stride S, CI -> 16 channels, from one shared-memory tile to another.  Output pixel (my, mx) of the
// OH x OW tile sits at (oy0 + my, ox0 + mx) of a gh x gw grid and reads input tile rows S my + ky, columns S mx + kx
// (the input tile's origin is (S oy0 - 1, S ox0 - 1); it holds zeros outside its own grid).  Outside the output grid
// the result is 0: the next conv's zero padding.  w [9][CI][16], b [16] in shared memory; ACT 0 none, 1 LeakyReLU(0.2).
template <int CI, int ICS, int IW, int OH, int OW, int S, int ACT>
__device__ __forceinline__ void ck_conv3x3(const float* in, float* out, const float* w, const float* b, int oy0,
                                           int ox0, int gh, int gw) {
  for (int i = threadIdx.x; i < OH * OW * 4; i += blockDim.x) {
    const int cq = i & 3, p = i >> 2, my = p / OW, mx = p % OW;
    const int gy = oy0 + my, gx = ox0 + mx;
    float o[4] = {0.f, 0.f, 0.f, 0.f};
    if (gy >= 0 && gy < gh && gx >= 0 && gx < gw) {
      const float4 bb = *reinterpret_cast<const float4*>(b + 4 * cq);
      o[0] = bb.x; o[1] = bb.y; o[2] = bb.z; o[3] = bb.w;
#pragma unroll
      for (int tap = 0; tap < 9; ++tap) {
        const float* ip = in + ((S * my + tap / 3) * IW + S * mx + tap % 3) * ICS;
        const float* wp = w + tap * CI * 16 + 4 * cq;
#pragma unroll
        for (int ci = 0; ci < CI; ++ci) {
          const float v = ip[ci];
          const float4 wv = *reinterpret_cast<const float4*>(wp + ci * 16);
          o[0] = fmaf(v, wv.x, o[0]); o[1] = fmaf(v, wv.y, o[1]); o[2] = fmaf(v, wv.z, o[2]); o[3] = fmaf(v, wv.w, o[3]);
        }
      }
      if (ACT == 1)
#pragma unroll
        for (int j = 0; j < 4; ++j) o[j] = o[j] > 0.f ? o[j] : 0.2f * o[j];
    }
    *reinterpret_cast<float4*>(out + p * CK_CS + 4 * cq) = make_float4(o[0], o[1], o[2], o[3]);
  }
}

// ConvTranspose2d(16, 16, k4, s2, p1) + bias, from one shared-memory tile to another: output (Y, X) = (oy0 + my,
// ox0 + mx) of the 2ih x 2iw grid gathers the input pixels iy = (Y + 1 - ky) / 2 of matching parity inside the ih x iw
// input grid (the input tile's origin is (iy0, ix0)).  0 outside the output grid.  w [ky][kx][ci][co]; ACT 2 = ReLU.
template <int IW, int OH, int OW, int ACT>
__device__ __forceinline__ void ck_convT(const float* in, int iy0, int ix0, int ih, int iw, float* out, int oy0, int ox0,
                                         const float* w, const float* b) {
  for (int i = threadIdx.x; i < OH * OW * 4; i += blockDim.x) {
    const int cq = i & 3, p = i >> 2, my = p / OW, mx = p % OW;
    const int Y = oy0 + my, X = ox0 + mx;
    float o[4] = {0.f, 0.f, 0.f, 0.f};
    if (Y >= 0 && Y < 2 * ih && X >= 0 && X < 2 * iw) {
      const float4 bb = *reinterpret_cast<const float4*>(b + 4 * cq);
      o[0] = bb.x; o[1] = bb.y; o[2] = bb.z; o[3] = bb.w;
#pragma unroll
      for (int a2 = 0; a2 < 2; ++a2) {
        const int ky = ((Y + 1) & 1) + 2 * a2, ny = Y + 1 - ky;
        if (ny < 0 || ny / 2 >= ih) continue;
#pragma unroll
        for (int b2 = 0; b2 < 2; ++b2) {
          const int kx = ((X + 1) & 1) + 2 * b2, nx = X + 1 - kx;
          if (nx < 0 || nx / 2 >= iw) continue;
          const float* ip = in + ((ny / 2 - iy0) * IW + (nx / 2 - ix0)) * CK_CS;
          const float* wp = w + (ky * 4 + kx) * 256 + 4 * cq;
#pragma unroll
          for (int ci = 0; ci < 16; ++ci) {
            const float v = ip[ci];
            const float4 wv = *reinterpret_cast<const float4*>(wp + ci * 16);
            o[0] = fmaf(v, wv.x, o[0]); o[1] = fmaf(v, wv.y, o[1]); o[2] = fmaf(v, wv.z, o[2]); o[3] = fmaf(v, wv.w, o[3]);
          }
        }
      }
      if (ACT == 2)
#pragma unroll
        for (int j = 0; j < 4; ++j) o[j] = fmaxf(o[j], 0.f);
    }
    *reinterpret_cast<float4*>(out + p * CK_CS + 4 * cq) = make_float4(o[0], o[1], o[2], o[3]);
  }
}

// An NHWC latent patch [LH][LW][16] of [B][h][w][16] with origin (ly0, lx0) -> shared memory (zeros outside the grid).
template <int LH, int LW>
__device__ __forceinline__ void ck_load_latent(const float* x, int b, int h, int w, int ly0, int lx0, float* s) {
  for (int i = threadIdx.x; i < LH * LW * 4; i += blockDim.x) {
    const int q = i & 3, lp = i >> 2;
    const int yy = ly0 + lp / LW, xx = lx0 + lp % LW;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (yy >= 0 && yy < h && xx >= 0 && xx < w)
      v = reinterpret_cast<const float4*>(x + ((static_cast<size_t>(b) * h + yy) * w + xx) * 16)[q];
    *reinterpret_cast<float4*>(s + lp * CK_CS + 4 * q) = v;
  }
}

// A depth patch [DH][DW] of [B][1][H][W] with origin (dy0, dx0) -> shared memory (zeros outside the map).
template <int DH, int DW>
__device__ __forceinline__ void ck_load_depth(const float* d, int b, int H, int W, int dy0, int dx0, float* s) {
  for (int i = threadIdx.x; i < DH * DW; i += blockDim.x) {
    const int yy = dy0 + i / DW, xx = dx0 + i % DW;
    s[i] = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? d[(static_cast<size_t>(b) * H + yy) * W + xx] : 0.f;
  }
}

// n floats global -> shared (n a multiple of 4, both 16-byte aligned)
__device__ __forceinline__ void ck_copy(const float* g, float* s, int n) {
  for (int i = threadIdx.x; i < n / 4; i += blockDim.x)
    reinterpret_cast<float4*>(s)[i] = reinterpret_cast<const float4*>(g)[i];
}

// Final 3x3 conv 16 -> 1 over a TH x TW tile of `mid` (row width TW + 2, origin one pixel up-left), then
// depth = 1 / clamp(sigmoid(z), eps) - 1; z is the optional logit.  wc [9][16] and bc in shared memory.
template <int TH, int TW>
__device__ __forceinline__ void ck_final(const float* mid, const float* wc, const float* bc, int b, int Y0, int X0,
                                         int H, int W, float eps, float* logit, float* depth) {
  constexpr int MW = TW + 2;
  for (int i = threadIdx.x; i < TH * TW; i += blockDim.x) {
    const int yy = i / TW, xx = i % TW;
    const int Y = Y0 + yy, X = X0 + xx;
    if (Y >= H || X >= W) continue;
    float z = bc[0];
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const float* mp = mid + ((yy + tap / 3) * MW + xx + tap % 3) * CK_CS;
#pragma unroll
      for (int c4 = 0; c4 < 4; ++c4) {
        const float4 mv = *reinterpret_cast<const float4*>(mp + 4 * c4);
        const float4 wv = *reinterpret_cast<const float4*>(wc + tap * 16 + 4 * c4);
        z = fmaf(mv.x, wv.x, z); z = fmaf(mv.y, wv.y, z); z = fmaf(mv.z, wv.z, z); z = fmaf(mv.w, wv.w, z);
      }
    }
    const size_t o = (static_cast<size_t>(b) * H + Y) * W + X;
    if (logit) logit[o] = z;
    const float s = 1.0f / (1.0f + expf(-z));
    depth[o] = 1.0f / fmaxf(s, eps) - 1.0f;
  }
}

// ------------------------------------------------------------------ folded parameter layouts (device, engine-owned)
// UP2_1X1 encoder: k [16] = conv_transform.1.weight . conv_transform.0.weight (no bias, no BatchNorm: the two 1x1 convs
// compose exactly into one per-channel scale, summed in fp64)
constexpr int CK_E1_K = 0, CK_E1_N = 16;
// UP4 encoder: three conv_bn_relu stages, w [9][ci][16] and b [16] each
constexpr int CK_E4_W1 = 0, CK_E4_B1 = 144, CK_E4_W2 = 160, CK_E4_B2 = 2464, CK_E4_W3 = 2480, CK_E4_B3 = 4784,
              CK_E4_N = 4800;
// UP4 decoder: ConvT 1 (+ bias), ConvT 2 with the BatchNorm folded, final conv [9][16] and its bias (padded to 4)
constexpr int CK_D4_T1 = 0, CK_D4_B1 = 4096, CK_D4_T2 = 4112, CK_D4_B2 = 8208, CK_D4_WC = 8224, CK_D4_BC = 8368,
              CK_D4_N = 8372;
// FULL decoder: conv_bn_relu 16 -> 16 folded, conv_bn 16 -> 1 folded ([9][16], bias padded to 4)
constexpr int CK_DF_W1 = 0, CK_DF_B1 = 2304, CK_DF_WC = 2320, CK_DF_BC = 2464, CK_DF_N = 2468;

struct CodecKindArgs {
  const float* in;     // encoders: depth [B][1][H][W]; decoders: latent NHWC [B][h][w][16]
  const float* p;      // folded parameters (layouts above)
  float* out;          // encoders: latent NCHW [B][16][h][w]; decoders: depth [B][uh][uw]
  float* logit;        // decoders, optional: [B][uh][uw]
  int H, W, h, w;      // encoders: depth map and latent grid; decoders: latent grid in h, w
  float eps;
};

// ------------------------------------------------------------------ UP2_1X1 encoder (t)
// Conv2d(1,16,1) -> Conv2d(16,16,1) -> tanh -> MaxPool2d(3, s2, p1): one thread per latent pixel, 16 channels.  The
// pool's -inf padding never wins: the centre (2y, 2x) of every window is inside the map.
__global__ void __launch_bounds__(256) encoder_1x1_kernel(const CodecKindArgs a) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(a.h) * a.w) return;
  const int b = blockIdx.y, y = static_cast<int>(i / a.w), x = static_cast<int>(i % a.w);
  float k[16], m[16];
#pragma unroll
  for (int c = 0; c < 16; ++c) {
    k[c] = __ldg(a.p + CK_E1_K + c);
    m[c] = -INFINITY;
  }
  for (int dy = -1; dy <= 1; ++dy) {
    const int yy = 2 * y + dy;
    if (yy < 0 || yy >= a.H) continue;
    for (int dx = -1; dx <= 1; ++dx) {
      const int xx = 2 * x + dx;
      if (xx < 0 || xx >= a.W) continue;
      const float d = __ldg(a.in + (static_cast<size_t>(b) * a.H + yy) * a.W + xx);
#pragma unroll
      for (int c = 0; c < 16; ++c) m[c] = fmaxf(m[c], tanhf(d * k[c]));
    }
  }
#pragma unroll
  for (int c = 0; c < 16; ++c) a.out[((static_cast<size_t>(b) * 16 + c) * a.h + y) * a.w + x] = m[c];
}

// ------------------------------------------------------------------ UP4 encoder (t)
// conv_bn_relu(1,16,3,s2) -> conv_bn_relu(16,16,3,s2) -> conv_bn(16,16,3,s1) -> tanh.  One block = 16 x 16 latent
// pixels (grid h = ceil(ceil(H/2)/2)); the 37 x 37 x 16 half-resolution and the 18 x 18 x 16 quarter-resolution
// intermediates stay in shared memory.
constexpr int E4_T = 16, E4_M2 = E4_T + 2, E4_M1 = 2 * E4_M2 + 1, E4_D = 2 * E4_M1 + 1;  // 18, 37, 75
constexpr int E4_SMEM = (E4_D * E4_D + E4_M1 * E4_M1 * CK_CS + E4_M2 * E4_M2 * CK_CS + CK_E4_N) * 4;
__global__ void __launch_bounds__(256) encoder_x4_kernel(const CodecKindArgs a) {
  extern __shared__ __align__(16) float ck_smem[];
  float* s_w = ck_smem;                         // CK_E4_N
  float* s_m1 = s_w + CK_E4_N;                  // [37 * 37][CS]
  float* s_m2 = s_m1 + E4_M1 * E4_M1 * CK_CS;   // [18 * 18][CS]
  float* s_d = s_m2 + E4_M2 * E4_M2 * CK_CS;    // [75 * 75]; reused for the output tile [16][256]
  const int b = blockIdx.z, y0 = blockIdx.y * E4_T, x0 = blockIdx.x * E4_T;
  const int h1 = (a.H + 1) / 2, w1 = (a.W + 1) / 2;
  const int m2y = y0 - 1, m2x = x0 - 1, m1y = 2 * m2y - 1, m1x = 2 * m2x - 1;
  ck_copy(a.p, s_w, CK_E4_N);
  ck_load_depth<E4_D, E4_D>(a.in, b, a.H, a.W, 2 * m1y - 1, 2 * m1x - 1, s_d);
  __syncthreads();
  ck_conv3x3<1, 1, E4_D, E4_M1, E4_M1, 2, 1>(s_d, s_m1, s_w + CK_E4_W1, s_w + CK_E4_B1, m1y, m1x, h1, w1);
  __syncthreads();
  ck_conv3x3<16, CK_CS, E4_M1, E4_M2, E4_M2, 2, 1>(s_m1, s_m2, s_w + CK_E4_W2, s_w + CK_E4_B2, m2y, m2x, a.h, a.w);
  __syncthreads();
  float* s_o = s_d;  // [T * T][CS]: free once conv1 has read the depth patch
  ck_conv3x3<16, CK_CS, E4_M2, E4_T, E4_T, 1, 0>(s_m2, s_o, s_w + CK_E4_W3, s_w + CK_E4_B3, y0, x0, a.h, a.w);
  __syncthreads();
  for (int i = threadIdx.x; i < 16 * E4_T * E4_T; i += blockDim.x) {
    const int c = i / (E4_T * E4_T), p = i % (E4_T * E4_T), y = y0 + p / E4_T, x = x0 + p % E4_T;
    if (y < a.h && x < a.w) a.out[((static_cast<size_t>(b) * 16 + c) * a.h + y) * a.w + x] = tanhf(s_o[p * CK_CS + c]);
  }
}
static_assert(E4_T * E4_T * CK_CS <= E4_D * E4_D, "encoder_x4 output tile exceeds the depth patch it reuses");

// ------------------------------------------------------------------ FULL encoder (t)
// conv_bn_relu(1,16,3,s1) -> conv_bn(16,16,3,s1) -> tanh at the depth map's own resolution.  One block = 16 x 16
// pixels; the 18 x 18 x 16 intermediate stays in shared memory.  Shares encoder_kernel's folded parameters
// (w1 [9][16], b1, w2 [9][16][16], b2), passed as one block laid out like CK_E4_W1 .. CK_E4_B2.
constexpr int EF_T = 16, EF_M = EF_T + 2, EF_D = EF_M + 2;
constexpr int EF_SMEM = (EF_D * EF_D + EF_M * EF_M * CK_CS + EF_T * EF_T * CK_CS + CK_E4_W3) * 4;
__global__ void __launch_bounds__(256) encoder_full_kernel(const CodecKindArgs a) {
  extern __shared__ __align__(16) float ck_smem[];
  float* s_w = ck_smem;                       // CK_E4_W3 (w1, b1, w2, b2)
  float* s_m = s_w + CK_E4_W3;                // [18 * 18][CS]
  float* s_o = s_m + EF_M * EF_M * CK_CS;     // [16 * 16][CS]
  float* s_d = s_o + EF_T * EF_T * CK_CS;     // [20 * 20]
  const int b = blockIdx.z, y0 = blockIdx.y * EF_T, x0 = blockIdx.x * EF_T;
  ck_copy(a.p, s_w, CK_E4_W3);
  ck_load_depth<EF_D, EF_D>(a.in, b, a.H, a.W, y0 - 2, x0 - 2, s_d);
  __syncthreads();
  ck_conv3x3<1, 1, EF_D, EF_M, EF_M, 1, 1>(s_d, s_m, s_w + CK_E4_W1, s_w + CK_E4_B1, y0 - 1, x0 - 1, a.h, a.w);
  __syncthreads();
  ck_conv3x3<16, CK_CS, EF_M, EF_T, EF_T, 1, 0>(s_m, s_o, s_w + CK_E4_W2, s_w + CK_E4_B2, y0, x0, a.h, a.w);
  __syncthreads();
  for (int i = threadIdx.x; i < 16 * EF_T * EF_T; i += blockDim.x) {
    const int c = i / (EF_T * EF_T), p = i % (EF_T * EF_T), y = y0 + p / EF_T, x = x0 + p % EF_T;
    if (y < a.h && x < a.w) a.out[((static_cast<size_t>(b) * 16 + c) * a.h + y) * a.w + x] = tanhf(s_o[p * CK_CS + c]);
  }
}

// ------------------------------------------------------------------ UP4 decoder (inv_t)
// ConvT(16,16,k4,s2,p1)+b -> ConvT(16,16,k4,s2,p1)+b -> BN (folded into the second) -> ReLU -> Conv2d(16,1,3,1,1)+b
// -> z, depth = 1 / clamp(sigmoid(z), eps) - 1.  One block = 16 x 32 pixels of the 4h x 4w map: the 6 x 10 latent
// patch, the 10 x 18 x 16 2x intermediate and the 18 x 34 x 16 4x intermediate stay in shared memory.
constexpr int D4_TH = 16, D4_TW = 32;
constexpr int D4_LH = D4_TH / 4 + 2, D4_LW = D4_TW / 4 + 2, D4_AH = D4_TH / 2 + 2, D4_AW = D4_TW / 2 + 2;
constexpr int D4_MH = D4_TH + 2, D4_MW = D4_TW + 2;
constexpr int D4_SMEM = (CK_D4_N + (D4_LH * D4_LW + D4_AH * D4_AW + D4_MH * D4_MW) * CK_CS) * 4;
__global__ void __launch_bounds__(256) decoder_x4_kernel(const CodecKindArgs a) {
  extern __shared__ __align__(16) float ck_smem[];
  float* s_w = ck_smem;
  float* s_l = s_w + CK_D4_N;
  float* s_a = s_l + D4_LH * D4_LW * CK_CS;
  float* s_m = s_a + D4_AH * D4_AW * CK_CS;
  const int b = blockIdx.z, Y0 = blockIdx.y * D4_TH, X0 = blockIdx.x * D4_TW;
  const int ay0 = Y0 / 2 - 1, ax0 = X0 / 2 - 1, ly0 = Y0 / 4 - 1, lx0 = X0 / 4 - 1;
  ck_copy(a.p, s_w, CK_D4_N);
  ck_load_latent<D4_LH, D4_LW>(a.in, b, a.h, a.w, ly0, lx0, s_l);
  __syncthreads();
  ck_convT<D4_LW, D4_AH, D4_AW, 0>(s_l, ly0, lx0, a.h, a.w, s_a, ay0, ax0, s_w + CK_D4_T1, s_w + CK_D4_B1);
  __syncthreads();
  ck_convT<D4_AW, D4_MH, D4_MW, 2>(s_a, ay0, ax0, 2 * a.h, 2 * a.w, s_m, Y0 - 1, X0 - 1, s_w + CK_D4_T2, s_w + CK_D4_B2);
  __syncthreads();
  ck_final<D4_TH, D4_TW>(s_m, s_w + CK_D4_WC, s_w + CK_D4_BC, b, Y0, X0, 4 * a.h, 4 * a.w, a.eps, a.logit, a.out);
}

// ------------------------------------------------------------------ FULL decoder (inv_t)
// conv_bn_relu(16,16,3,1) -> conv_bn(16,1,3,1) -> z, depth = 1 / clamp(sigmoid(z), eps) - 1, at the latent's own
// resolution.  One block = 8 x 32 pixels; the 12 x 36 latent patch and the 10 x 34 x 16 intermediate stay in shared
// memory.
constexpr int DF_TH = 8, DF_TW = 32;
constexpr int DF_SMEM = (CK_DF_N + ((DF_TH + 4) * (DF_TW + 4) + (DF_TH + 2) * (DF_TW + 2)) * CK_CS) * 4;
__global__ void __launch_bounds__(256) decoder_full_kernel(const CodecKindArgs a) {
  extern __shared__ __align__(16) float ck_smem[];
  float* s_w = ck_smem;
  float* s_l = s_w + CK_DF_N;
  float* s_m = s_l + (DF_TH + 4) * (DF_TW + 4) * CK_CS;
  const int b = blockIdx.z, Y0 = blockIdx.y * DF_TH, X0 = blockIdx.x * DF_TW;
  ck_copy(a.p, s_w, CK_DF_N);
  ck_load_latent<DF_TH + 4, DF_TW + 4>(a.in, b, a.h, a.w, Y0 - 2, X0 - 2, s_l);
  __syncthreads();
  ck_conv3x3<16, CK_CS, DF_TW + 4, DF_TH + 2, DF_TW + 2, 1, 1>(s_l, s_m, s_w + CK_DF_W1, s_w + CK_DF_B1, Y0 - 1, X0 - 1,
                                                               a.h, a.w);
  __syncthreads();
  ck_final<DF_TH, DF_TW>(s_m, s_w + CK_DF_WC, s_w + CK_DF_BC, b, Y0, X0, a.h, a.w, a.eps, a.logit, a.out);
}

}  // namespace dd
