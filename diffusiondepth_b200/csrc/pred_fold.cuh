// convB -> pred.0 of the Swin head's ScheduledCNNRefine as ONE composed 5x5 conv (256 -> 64) on warpgroup MMA, plus
// the border correction that makes it equal the two-conv chain.
//
// UpSample_add's convB (reference src/model/head/ddim_depth_estimate_res_swin_addHAHI.py:326-333, no norm, no
// activation) feeds pred.0 (:352-353) directly, so y5 = pred0(convB(a)) is affine in convA's output a:
//   K5[co][ci][D] = sum_{cm, d + d' = D} Wp0[co][cm][d] WB[cm][ci][d'],   b5 = bp0 + sum_{cm, d} Wp0[co][cm][d] bB[cm]
// (fp64 at dd_finalize_weights).  409,600 MACs per pixel instead of 737,280.
//
// The composition is exact where neither conv pads.  conv5x5_fold_kernel runs K5 on zero-padded a; at a pixel p next
// to the border it then also counts pred.0 taps that land on positions q outside the image, where the chain has zeros:
//   corr(p) = sum_{d: p + d outside} Wp0[d] b_ext(p + d),   b_ext(q) = bB + sum_{d': q + d' inside} WB[d'] a(q + d')
// ring_fix_kernel subtracts corr on the one-pixel ring (fp32 CUDA cores, as composed 1-D edge convs: ~0.5 GMAC per step
// at B = 4, 176 x 608) and writes the ring's GroupNorm partials; the composed kernel's partials cover the interior only.
#pragma once
#include "conv_common.cuh"

namespace dd {

// ---------------------------------------------------------------------------------------------- composed 5x5 conv
// Transposed implicit GEMM: D[64 cout][pixels] = K5 * X^T, so the 64 output channels are the wgmma M and 128 pixels
// the N of an m64n128k16 accumulator (2 / 128 + 1 / 32 B of shared-memory operand per MAC, as the 256 -> 256 halo
// conv, against 2 / 64 + 1 / 32 for pixels-as-M at COUT = 64).  Each consumer warpgroup holds TWO such accumulators,
// one for the even and one for the odd channel chunks, added in fp32 in the epilogue: a tensor-core accumulator loses
// a little at every wgmma that adds into it, and one accumulator over all 16 chunks x 25 taps x 3 passes (1,200
// wgmmas) was about twice as far from fp64 as the convB + pred.0 chain (432 each); two halve that.
//
// Tile: 16 x 16 pixels; consumer warpgroup w owns rows [8 w, 8 w + 8), all 16 columns.  Per 16-channel chunk the
// producer loads ONE halo patch of (16 + 4) x (16 + 4) pixels per plane, stored column-major without swizzle as
// [8-channel group][x][y][8 ch]: the 8 pixels of one column and one warpgroup are a 128-byte core matrix, N-adjacent
// core matrices are one patch column apart (SBO), K-adjacent ones one channel group apart (LBO), and tap (dy, dx) is
// the descriptor start offset dx * column + dy * 16 B.  All 25 taps read the same patch.  The patch is one 5-D TMA
// box {8 ch, y, x, channel group, image}; its out-of-bounds zero fill is the zero padding of a.
// Weights: [chunk][dy][dx][hi / lo][k group][co group][8 co][8 k] fp16, core-matrix order, so one row of five taps
// (20 KB) is one contiguous bulk copy.
constexpr int F5_TH = 16;
constexpr int F5_TW = 16;

struct F5 {
  static constexpr int CIN = 256, COUT = 64, BK = 16, KC = CIN / BK;
  static constexpr int PH = F5_TH + 4, PW = F5_TW + 4;  // patch rows / columns
  static constexpr int XP = PH * 16;                    // bytes per patch column (PH pixels x 8 channels)
  static constexpr int CGP = PW * XP;                   // bytes per 8-channel group
  static constexpr int PLANE = 2 * CGP;                 // one fp16 plane of a chunk
  static constexpr int P_SLOT = 2 * PLANE;              // hi + lo
  static constexpr int P_SLOTS = 3;
  static constexpr int W_PLANE = COUT * BK * 2;         // 64 x 16 fp16
  static constexpr int W_TAP = 2 * W_PLANE;             // hi + lo
  static constexpr int W_SLOT = 5 * W_TAP;              // one row of taps
  static constexpr int W_SLOTS = 6;
  static constexpr int CHP = 32;                        // pixels per epilogue chunk (4 columns of 8)
  static constexpr int LD = COUT + 4;                   // staging row stride (floats): conflict-free accumulator writes
  static constexpr int STAGE_BYTES = 2 * CHP * LD * 4;
  static constexpr int CTRL_BYTES = 1024;               // barriers, GroupNorm scratch [2][2][4][2]
  static constexpr int SMEM_BYTES = P_SLOTS * P_SLOT + W_SLOTS * W_SLOT + CTRL_BYTES + STAGE_BYTES + 1024;
  static constexpr int THREADS = 384;
  static constexpr size_t W_ELEMS = static_cast<size_t>(KC) * 25 * 2 * COUT * BK;  // packed fp16 elements
  static_assert(SMEM_BYTES <= 232448, "exceeds the 227 KB dynamic shared memory limit");
  static_assert(P_SLOT % 1024 == 0 && W_SLOT % 1024 == 0, "ring slots stay 1 KB aligned");
};

struct FoldArgs {
  int B, H, W;
  int tiles_x, tiles_y, num_tiles;
  const __half* w;       // packed K5 (F5::W_ELEMS)
  const float* bias;     // b5 [64]
  float acc_scale;       // 1 / (act_scale * K5 scale)
  float* y32;            // [B*H*W][64]
  double* stats_partial;  // [num_tiles][4][2] fp64 sums, interior pixels only
};

__global__ void __launch_bounds__(F5::THREADS, 1)
conv5x5_fold_kernel(const __grid_constant__ CUtensorMap tmP_hi, const __grid_constant__ CUtensorMap tmP_lo,
                    const FoldArgs p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* p_ring = smem;
  uint8_t* w_ring = smem + F5::P_SLOTS * F5::P_SLOT;
  uint8_t* ctrl = w_ring + F5::W_SLOTS * F5::W_SLOT;
  uint64_t* p_full = reinterpret_cast<uint64_t*>(ctrl);
  uint64_t* p_empty = p_full + F5::P_SLOTS;
  uint64_t* w_full = p_empty + F5::P_SLOTS;
  uint64_t* w_empty = w_full + F5::W_SLOTS;
  double* red = reinterpret_cast<double*>(w_empty + F5::W_SLOTS);  // [2 par][2 wg][4 warps][2]
  float* stage = reinterpret_cast<float*>(ctrl + F5::CTRL_BYTES);

  const int warp = threadIdx.x >> 5;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmP_hi);
    tma_prefetch_desc(&tmP_lo);
    for (int s = 0; s < F5::P_SLOTS; ++s) {
      mbar_init(&p_full[s], 1);
      mbar_init(&p_empty[s], 2);
    }
    for (int s = 0; s < F5::W_SLOTS; ++s) {
      mbar_init(&w_full[s], 1);
      mbar_init(&w_empty[s], 2);
    }
    fence_barrier_init();
  }
  __syncthreads();

  // role split as in conv3x3_halo_kernel: setmaxnreg first in each branch, no merge point before the exit
  if (warp < 4) {
    setmaxnreg_dec<40>();
    if (warp == 0) {
      // ---------------------------------------------------------------- TMA producer: one halo patch per chunk
      const bool leader = elect_one();
      int s = 0;
      uint32_t ph = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const int tx = tile % p.tiles_x, ty = (tile / p.tiles_x) % p.tiles_y, img = tile / (p.tiles_x * p.tiles_y);
        const int x0 = tx * F5_TW, y0 = ty * F5_TH;
        for (int kc = 0; kc < F5::KC; ++kc) {
          mbar_wait(&p_empty[s], ph ^ 1);
          uint8_t* d = p_ring + s * F5::P_SLOT;
          if (leader) {
            mbar_arrive_expect_tx(&p_full[s], F5::P_SLOT);
            tma_load_5d(d, &tmP_hi, &p_full[s], 0, y0 - 2, x0 - 2, 2 * kc, img);
            tma_load_5d(d + F5::PLANE, &tmP_lo, &p_full[s], 0, y0 - 2, x0 - 2, 2 * kc, img);
          }
          __syncwarp();
          if (++s == F5::P_SLOTS) {
            s = 0;
            ph ^= 1;
          }
        }
      }
    } else if (warp == 1) {
      // ---------------------------------------------------------------- bulk-copy producer: one row of taps per slot
      const bool leader = elect_one();
      int s = 0;
      uint32_t ph = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        for (int r = 0; r < F5::KC * 5; ++r) {  // (chunk, dy) in the consumers' order
          mbar_wait(&w_empty[s], ph ^ 1);
          if (leader) {
            mbar_arrive_expect_tx(&w_full[s], F5::W_SLOT);
            bulk_load(w_ring + s * F5::W_SLOT, p.w + static_cast<size_t>(r) * (F5::W_SLOT / 2), F5::W_SLOT, &w_full[s]);
          }
          __syncwarp();
          if (++s == F5::W_SLOTS) {
            s = 0;
            ph ^= 1;
          }
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    // ------------------------------------------------------------------ consumers: MMA + epilogue
    const int wg = (warp >> 2) - 1;
    const int t = threadIdx.x & 127;
    const int q = t >> 5, lane = t & 31;
    const bool signal = (t == 0);
    float* S = stage + wg * F5::CHP * F5::LD;
    int sp = 0, sw = 0, par = 0;
    uint32_t pp = 0, pw = 0;
    float acc0[64], acc1[64];  // even / odd channel chunks

    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      int prev_w = -1, prev_p = -1;  // slots read by the wgmma group still in flight
      auto retire_prev = [&]() {
        mbar_arrive_if(&w_empty[prev_w < 0 ? 0 : prev_w], signal && prev_w >= 0);
        mbar_arrive_if(&p_empty[prev_p < 0 ? 0 : prev_p], signal && prev_p >= 0);
        prev_w = prev_p = -1;
      };
      auto chunk = [&](float(&acc)[64], int kc) {
        mbar_wait(&p_full[sp], pp);
        const uint32_t pb = smem_u32(p_ring + sp * F5::P_SLOT) + wg * 8 * 16;  // this warpgroup's 8 rows
        for (int dy = 0; dy < 5; ++dy) {
          mbar_wait(&w_full[sw], pw);
          const uint32_t wb = smem_u32(w_ring + sw * F5::W_SLOT);
          wgmma_fence();
#pragma unroll
          for (int dx = 0; dx < 5; ++dx) {
            const uint32_t wa = wb + dx * F5::W_TAP;
            const uint32_t xa = pb + dx * F5::XP + dy * 16;
            const uint64_t a_hi = wgmma_desc_plain(wa, 1024, 128);
            const uint64_t a_lo = wgmma_desc_plain(wa + F5::W_PLANE, 1024, 128);
            const uint64_t b_hi = wgmma_desc_plain(xa, F5::CGP, F5::XP);
            const uint64_t b_lo = wgmma_desc_plain(xa + F5::PLANE, F5::CGP, F5::XP);
            wgmma_f16<128>(acc, a_hi, b_lo, (kc >= 2 || dy != 0 || dx != 0) ? 1u : 0u);  // small terms first
            wgmma_f16<128>(acc, a_lo, b_hi, 1u);
            wgmma_f16<128>(acc, a_hi, b_hi, 1u);
          }
          wgmma_commit();
          wgmma_wait<1>();
          retire_prev();
          prev_w = sw;
          if (dy == 4) prev_p = sp;
          if (++sw == F5::W_SLOTS) {
            sw = 0;
            pw ^= 1;
          }
        }
        if (++sp == F5::P_SLOTS) {
          sp = 0;
          pp ^= 1;
        }
      };
      for (int kc = 0; kc < F5::KC; kc += 2) {
        chunk(acc0, kc);
        chunk(acc1, kc + 1);
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc0);
      wgmma_fence_regs(acc1);
      retire_prev();  // the producers refill the rings while this warpgroup drains its accumulator

      // ---------------------------------------------------------------- epilogue
      // d[4 i + e] = D[co0 + 8 (e / 2)][pixel: column i, row 2 (lane % 4) + e % 2 of this warpgroup's 8]; D = acc0 + acc1
      const int tx = tile % p.tiles_x, ty = (tile / p.tiles_x) % p.tiles_y, img = tile / (p.tiles_x * p.tiles_y);
      const int x0 = tx * F5_TW, yw = ty * F5_TH + wg * 8;
      const int co0 = 16 * q + (lane >> 2);  // this thread's output channels: co0 and co0 + 8 (GroupNorm group q)
      const float bias0 = __ldg(p.bias + co0), bias1 = __ldg(p.bias + co0 + 8);
      // as conv3x3_halo_kernel sums: d = v - k in fp32, k = this thread's first interior value, then fp64 sums of v, v^2
      float tk = 0.f, tsum = 0.f, tsq = 0.f;
      int tn = 0;
#pragma unroll
      for (int cj = 0; cj < F5_TW / 4; ++cj) {
        named_bar_sync(2 + wg, 128);  // the previous chunk's staging reads are done
#pragma unroll
        for (int ii = 0; ii < 4; ++ii) {
          const int i = 4 * cj + ii;
          const int x = x0 + i;
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int yl = 2 * (lane & 3) + (e & 1);
            const int y = yw + yl;
            const float v = fmaf(acc0[4 * i + e] + acc1[4 * i + e], p.acc_scale, (e >> 1) ? bias1 : bias0);
            if (x > 0 && x < p.W - 1 && y > 0 && y < p.H - 1) {  // interior; ring_fix_kernel sums the ring
              if (tn++ == 0) tk = v;
              const float d = v - tk;
              tsum += d;
              tsq = fmaf(d, d, tsq);
            }
            S[(ii * 8 + yl) * F5::LD + co0 + 8 * (e >> 1)] = v;
          }
        }
        named_bar_sync(2 + wg, 128);
        // warp q writes staged pixels [8 q, 8 q + 8): two whole 256-byte rows per store instruction
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int n = 8 * q + 2 * k + (lane >> 4);
          const int x = x0 + 4 * cj + (n >> 3), y = yw + (n & 7);
          if (x < p.W && y < p.H) {
            const float4 v = *reinterpret_cast<const float4*>(S + n * F5::LD + 4 * (lane & 15));
            *reinterpret_cast<float4*>(p.y32 + ((static_cast<size_t>(img) * p.H + y) * p.W + x) * F5::COUT +
                                       4 * (lane & 15)) = v;
          }
        }
      }
      // warp q holds exactly GroupNorm group q: warp tree, then the two warpgroups in fixed order
      const double n = tn, kk = tk, ds = tsum;
      double s = fma(n, kk, ds), s2 = fma(n * kk, kk, fma(2.0 * kk, ds, static_cast<double>(tsq)));
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, o);
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
      }
      if (lane == 0) {
        red[((par * 2 + wg) * 4 + q) * 2 + 0] = s;
        red[((par * 2 + wg) * 4 + q) * 2 + 1] = s2;
      }
      named_bar_sync(1, 256);
      const int e = threadIdx.x - 128;
      if (e < 8) {
        const int g = e >> 1, which = e & 1;
        p.stats_partial[(static_cast<size_t>(tile) * 4 + g) * 2 + which] =
            red[((par * 2 + 0) * 4 + g) * 2 + which] + red[((par * 2 + 1) * 4 + g) * 2 + which];
      }
      par ^= 1;  // double-buffered scratch: one barrier per tile is enough
    }
  }
}

// ---------------------------------------------------------------------------------------------- ring correction
// corr(p) cut by the side that each outside position q = p + d lies on.  Above the image (q in row -1) only convB taps
// with d'y = +1 reach an inside pixel, all in row 0, so for p in row 0 the top share is a 1-D 5-tap 256 -> 64 conv of
// a's row 0, zero-padded along the row:
//   T(x) = cT + sum_{D = -2..2} ET[D] a(0, x + D),   ET[D] = sum_{dx + d'x = D} Wp0[-1][dx] WB[+1][d'x],
//   cT = sum_dx Wp0[-1][dx] bB
// and the same for the bottom row (B), the left column (L, along y) and the right column (R).  T and B own every d whose
// row is outside; L and R own only the d whose row is inside, so their zero-padded column convs count the four corner
// positions once too often and a corner fix-up removes that: at p = (0, 0) the left conv's d = (-1, -1) term is
// Wp0[-1][-1] (bB + WB[+1][+1] a(0, 0)), and likewise at the other corners (Wp0[d] WB[-d] a(p) + Wp0[d] bB).  Hence
//   corr(p) = [y = 0] T(x) + [y = h-1] B(x) + [x = 0] (L(y) - [y = 0] C_TL - [y = h-1] C_BL)
//                                            + [x = w-1] (R(y) - [y = 0] C_TR - [y = h-1] C_BR),
// which holds for any h, w >= 1.  The edge kernels and constants are composed in fp64 next to K5 (compose_edge_kernel):
// about 0.5 GMAC per step at B = 4, 176 x 608, against 1.5 for building b_ext at every outside position.
//
// ring_fix_kernel cuts the ring into straight sides, each counted once: top and bottom rows, then the left and right
// columns between them; a latent with h <= 2 (or w <= 2) is all ring and is cut into its rows (columns).  Sides are
// split into segments of at most RING_S pixels.  A segment's own sides (T / B for a row, L / R for a column) are one
// GEMM [pixels x 1280] . [1280 x 64] on a's line under the segment; the few end pixels that also lie on a crossing side
// or a corner add those terms afterwards.
constexpr int RING_S = 16;
constexpr int RING_LINE = RING_S + 4;  // a along a segment and its 2-pixel halo
constexpr int RING_THREADS = 256;
constexpr int RING_KQ = 5 * 256 / 4;  // K rows per quarter of the own-side GEMM
constexpr int RING_SMEM = RING_LINE * 256 * 4 + 4 * RING_S * 64 * 4 + 4 * 64 * 4 + 2 * 256 * 8;
constexpr int EDGE_E = 5 * 256 * 64;  // one side's kernel [tap][ci][co]
constexpr int EDGE_C = 256 * 64;      // one corner's [ci][co]
constexpr int EDGE_ELEMS = 4 * EDGE_E + 4 * EDGE_C + 8 * 64;  // T, B, L, R; TL, TR, BL, BR; their constants [8][64]

struct RingSide {
  int y0, x0, vert, len;
};
__host__ __device__ inline int ring_sides(int H, int W, RingSide* s) {
  int n = 0;
  if (H <= 2) {
    for (int y = 0; y < H; ++y) s[n++] = {y, 0, 0, W};
  } else if (W <= 2) {
    for (int x = 0; x < W; ++x) s[n++] = {0, x, 1, H};
  } else {
    s[n++] = {0, 0, 0, W};
    s[n++] = {H - 1, 0, 0, W};
    s[n++] = {1, 0, 1, H - 2};
    s[n++] = {1, W - 1, 1, H - 2};
  }
  return n;
}
__host__ __device__ inline int ring_segments(int H, int W) {
  RingSide s[4];
  const int n = ring_sides(H, W, s);
  int k = 0;
  for (int i = 0; i < n; ++i) k += (s[i].len + RING_S - 1) / RING_S;
  return k;
}

struct RingArgs {
  int H, W;
  int nseg, blocks_per_img;  // segments per image, spread over blocks_per_img blocks (each a contiguous range)
  const __half* a_hi;        // convA output planes [B][H][W][256], value = (hi + lo) * a_inv_scale
  const __half* a_lo;
  float a_inv_scale;
  const float* edge;         // EDGE_ELEMS fp32 (compose_edge_kernel)
  float* y32;                // [B][H][W][64]: the composed conv's output, corrected in place on the ring
  double* ring_partial;      // [B][blocks_per_img][4][2] GroupNorm fp64 sums of the corrected ring pixels
};

__device__ __forceinline__ bool inside_img(int y, int x, int H, int W) { return y >= 0 && y < H && x >= 0 && x < W; }
// side s (0 T, 1 B, 2 L, 3 R) holds pixel (y, x)
__device__ __forceinline__ bool on_side(int s, int y, int x, int H, int W) {
  return s == 0 ? y == 0 : s == 1 ? y == H - 1 : s == 2 ? x == 0 : x == W - 1;
}

// grid (blocks_per_img, B), RING_THREADS threads
__global__ void __launch_bounds__(RING_THREADS) ring_fix_kernel(const RingArgs p) {
  extern __shared__ float4 ring_smem4[];
  float* line = reinterpret_cast<float*>(ring_smem4);  // [RING_LINE][256]
  float* corr = line + RING_LINE * 256;                // [RING_S][64]
  float* part = corr + RING_S * 64;                    // [3][RING_S][64]: K quarters 1 .. 3, then the corrected outputs
  float* xred = part + 3 * RING_S * 64;                // [4][64] ci-slice sums of an end pixel's extra terms
  double* red = reinterpret_cast<double*>(xred + 4 * 64);  // [2][256]
  const int img = blockIdx.y, t = threadIdx.x;
  const int H = p.H, W = p.W;
  const float* cst = p.edge + 4 * EDGE_E + 4 * EDGE_C;  // [8][64]
  RingSide sd[4];
  ring_sides(H, W, sd);
  const int s_begin = static_cast<int>(static_cast<long long>(p.nseg) * blockIdx.x / p.blocks_per_img);
  const int s_end = static_cast<int>(static_cast<long long>(p.nseg) * (blockIdx.x + 1) / p.blocks_per_img);
  auto a_at = [&](int y, int x, int ci) {
    const size_t o = ((static_cast<size_t>(img) * H + y) * W + x) * 256 + ci;
    return (__half2float(p.a_hi[o]) + __half2float(p.a_lo[o])) * p.a_inv_scale;
  };
  double ts = 0.0, tq = 0.0;  // fp64 per element: the ring is a few pixels per block
  for (int sg = s_begin; sg < s_end; ++sg) {
    int k = sg, si = 0;
    while (k >= (sd[si].len + RING_S - 1) / RING_S) {
      k -= (sd[si].len + RING_S - 1) / RING_S;
      ++si;
    }
    const int n = min(RING_S, sd[si].len - k * RING_S);
    const int ly = sd[si].vert, lx = 1 - ly;  // along the segment
    const int oy = sd[si].y0 + k * RING_S * ly, ox = sd[si].x0 + k * RING_S * lx;
    const int s0 = 2 * ly;                    // the segment's own sides: T / B for a row, L / R for a column
    __syncthreads();  // the previous segment's shared-memory reads are done
    // a along the segment, positions -2 .. RING_S + 1, zero outside the image and past the segment's halo
    for (int i = t; i < RING_LINE * 32; i += RING_THREADS) {
      const int c8 = i & 31, pos = i >> 5;
      const int c = pos - 2, y = oy + c * ly, x = ox + c * lx;
      float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      if (c <= n + 1 && inside_img(y, x, H, W)) {
        const size_t o = ((static_cast<size_t>(img) * H + y) * W + x) * 256 + c8 * 8;
        const uint4 hv = __ldg(reinterpret_cast<const uint4*>(p.a_hi + o));
        const uint4 lv = __ldg(reinterpret_cast<const uint4*>(p.a_lo + o));
        const __half* hh = reinterpret_cast<const __half*>(&hv);
        const __half* ll = reinterpret_cast<const __half*>(&lv);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = (__half2float(hh[j]) + __half2float(ll[j])) * p.a_inv_scale;
      }
      float4* d = reinterpret_cast<float4*>(line + pos * 256 + c8 * 8);
      d[0] = make_float4(v[0], v[1], v[2], v[3]);
      d[1] = make_float4(v[4], v[5], v[6], v[7]);
    }
    __syncthreads();
    // own sides: thread = (K quarter kq, pixels [4 pg, 4 pg + 4), channels [4 cg, 4 cg + 4)), K = 5 taps x 256 in
    // order.  The L2 latency of the weight loads bounds the kernel, so segments are short and K is split four ways:
    // more blocks in flight, each with a shorter serial K loop (32-pixel segments and K halves took 1.5x as long)
    {
      const int kq = t >> 6, cg = t & 15, pg = (t >> 4) & 3;
      float acc[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[i][c] = 0.f;
      for (int s = s0; s < s0 + 2; ++s) {
        if (!on_side(s, oy, ox, H, W)) continue;  // every pixel of a segment is on the same own sides
        const float* E = p.edge + s * EDGE_E + 4 * cg;
#pragma unroll 2
        for (int kk = kq * RING_KQ; kk < (kq + 1) * RING_KQ; kk += 4) {
          const int tap = kk >> 8, ci = kk & 255;
          float4 w[4];
#pragma unroll
          for (int r = 0; r < 4; ++r) w[r] = __ldg(reinterpret_cast<const float4*>(E + (kk + r) * 64));
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float4 av = *reinterpret_cast<const float4*>(line + (4 * pg + i + tap) * 256 + ci);
            acc[i][0] = fmaf(av.w, w[3].x, fmaf(av.z, w[2].x, fmaf(av.y, w[1].x, fmaf(av.x, w[0].x, acc[i][0]))));
            acc[i][1] = fmaf(av.w, w[3].y, fmaf(av.z, w[2].y, fmaf(av.y, w[1].y, fmaf(av.x, w[0].y, acc[i][1]))));
            acc[i][2] = fmaf(av.w, w[3].z, fmaf(av.z, w[2].z, fmaf(av.y, w[1].z, fmaf(av.x, w[0].z, acc[i][2]))));
            acc[i][3] = fmaf(av.w, w[3].w, fmaf(av.z, w[2].w, fmaf(av.y, w[1].w, fmaf(av.x, w[0].w, acc[i][3]))));
          }
        }
      }
      if (kq > 0)
#pragma unroll
        for (int i = 0; i < 4; ++i)
          *reinterpret_cast<float4*>(part + ((kq - 1) * RING_S + 4 * pg + i) * 64 + 4 * cg) =
              make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
      __syncthreads();
      if (kq == 0) {
        float c0[4] = {0.f, 0.f, 0.f, 0.f};
        for (int s = s0; s < s0 + 2; ++s)
          if (on_side(s, oy, ox, H, W))
#pragma unroll
            for (int c = 0; c < 4; ++c) c0[c] += cst[s * 64 + 4 * cg + c];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          float v[4] = {acc[i][0], acc[i][1], acc[i][2], acc[i][3]};
#pragma unroll
          for (int q = 0; q < 3; ++q) {
            const float4 h = *reinterpret_cast<const float4*>(part + (q * RING_S + 4 * pg + i) * 64 + 4 * cg);
            v[0] += h.x;
            v[1] += h.y;
            v[2] += h.z;
            v[3] += h.w;
          }
          *reinterpret_cast<float4*>(corr + (4 * pg + i) * 64 + 4 * cg) =
              make_float4(v[0] + c0[0], v[1] + c0[1], v[2] + c0[2], v[3] + c0[3]);
        }
      }
    }
    __syncthreads();
    // end pixels that also lie on a crossing side: its 5-tap conv across the segment's line, minus the corner terms;
    // thread = (channel co, input-channel slice of 64), slices summed in order
    for (int e = 0; e < 2; ++e) {
      const int j = e == 0 ? (ly ? -oy : -ox) : (ly ? H - 1 - oy : W - 1 - ox);
      if (j < 0 || j >= n || (e == 1 && j == (ly ? -oy : -ox))) continue;
      const int y = oy + j * ly, x = ox + j * lx;
      const int co = t & 63, c0 = (t >> 6) * 64;
      float v = 0.f, cv = 0.f;
      for (int s = 2 - s0; s < 4 - s0; ++s) {
        if (!on_side(s, y, x, H, W)) continue;
        if (t < 64) cv += cst[s * 64 + co];
        const int ay = s >= 2, ax = s < 2;  // direction of side s
        for (int tap = 0; tap < 5; ++tap) {
          const int yy = y + (tap - 2) * ay, xx = x + (tap - 2) * ax;
          if (!inside_img(yy, xx, H, W)) continue;
          const float* E = p.edge + s * EDGE_E + tap * 256 * 64 + co;
          for (int ci = c0; ci < c0 + 64; ++ci) v = fmaf(a_at(yy, xx, ci), __ldg(E + ci * 64), v);
        }
      }
      for (int cn = 0; cn < 4; ++cn) {  // TL, TR, BL, BR
        if (y != ((cn >> 1) ? H - 1 : 0) || x != ((cn & 1) ? W - 1 : 0)) continue;
        if (t < 64) cv -= cst[(4 + cn) * 64 + co];
        const float* C = p.edge + 4 * EDGE_E + cn * EDGE_C + co;
        for (int ci = c0; ci < c0 + 64; ++ci) v = fmaf(-a_at(y, x, ci), __ldg(C + ci * 64), v);
      }
      xred[t] = v;
      __syncthreads();
      if (t < 64) corr[j * 64 + co] += xred[co] + xred[64 + co] + xred[128 + co] + xred[192 + co] + cv;
      __syncthreads();
    }
    // y(p) -= corr(p)
    for (int i = t; i < n * 64; i += RING_THREADS) {
      const int j = i >> 6, co = i & 63;
      float* yp = p.y32 + ((static_cast<size_t>(img) * H + oy + j * ly) * W + ox + j * lx) * 64 + co;
      const float v = *yp - corr[i];
      *yp = v;
      part[i] = v;
    }
    __syncthreads();
    // GroupNorm sums: thread t takes every 4th pixel of channel t % 64
    {
      const int co = t & 63;
      for (int j = t >> 6; j < n; j += 4) {
        const double v = part[j * 64 + co];
        ts += v;
        tq = fma(v, v, tq);
      }
    }
  }
  // GroupNorm partials of this block's ring pixels, summed in a fixed order
  red[t] = ts;
  red[256 + t] = tq;
  __syncthreads();
  if (t < 8) {
    const int g = t >> 1, which = t & 1;
    double s = 0.0;
    for (int pg = 0; pg < 4; ++pg)
      for (int c = 0; c < 16; ++c) s += red[which * 256 + pg * 64 + g * 16 + c];
    p.ring_partial[((static_cast<size_t>(img) * p.blocks_per_img + blockIdx.x) * 4 + g) * 2 + which] = s;
  }
}

// ---------------------------------------------------------------------------------------------- weight composition
// K5 [64][256][25] and b5 in fp64 from the reference-layout fp32 weights (pred.0 [64][256][3][3], convB
// [256][256][3][3]); the cm / tap order of every sum is fixed.
__global__ void compose_fold_kernel(const float* __restrict__ wp, const float* __restrict__ bp,
                                    const float* __restrict__ wb, const float* __restrict__ bb,
                                    double* __restrict__ k5, float* __restrict__ k5_abs, float* __restrict__ b5) {
  const int n = 64 * 256 * 25;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int t5 = i % 25, ci = (i / 25) % 256, co = i / (25 * 256);
    const int Dy = t5 / 5 - 2, Dx = t5 % 5 - 2;
    double s = 0.0;
    for (int cm = 0; cm < 256; ++cm)
      for (int ky = 0; ky < 3; ++ky) {
        const int ey = Dy - (ky - 1);  // convB's tap offset
        if (ey < -1 || ey > 1) continue;
        for (int kx = 0; kx < 3; ++kx) {
          const int ex = Dx - (kx - 1);
          if (ex < -1 || ex > 1) continue;
          s += static_cast<double>(wp[((co * 256 + cm) * 3 + ky) * 3 + kx]) *
               static_cast<double>(wb[((cm * 256 + ci) * 3 + ey + 1) * 3 + ex + 1]);
        }
      }
    k5[i] = s;
    k5_abs[i] = static_cast<float>(fabs(s));
    if (ci == 0 && t5 == 0) {
      double b = bp[co];
      for (int cm = 0; cm < 256; ++cm)
        for (int k = 0; k < 9; ++k) b += static_cast<double>(wp[(co * 256 + cm) * 9 + k]) * static_cast<double>(bb[cm]);
      b5[co] = static_cast<float>(b);
    }
  }
}
// The ring correction's edge kernels, corners and constants (EDGE_ELEMS, ring_fix_kernel's layout) in fp64 from the
// same weights, rounded once to fp32.  Side s pairs pred.0's outer tap row / column with convB's opposite one:
// T = (ky 0, ey 2), B = (ky 2, ey 0), L = (kx 0, ex 2), R = (kx 2, ex 0); tap D + 2 = k + e along the side.  Corner
// (dy, dx) pairs Wp0[d] with WB[-d].
__global__ void compose_edge_kernel(const float* __restrict__ wp, const float* __restrict__ wb,
                                    const float* __restrict__ bb, float* __restrict__ edge) {
  auto P = [&](int co, int cm, int ky, int kx) { return static_cast<double>(wp[((co * 256 + cm) * 3 + ky) * 3 + kx]); };
  auto Q = [&](int cm, int ci, int ey, int ex) { return static_cast<double>(wb[((cm * 256 + ci) * 3 + ey) * 3 + ex]); };
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < EDGE_ELEMS; i += gridDim.x * blockDim.x) {
    const int co = i & 63;
    double s = 0.0;
    if (i < 4 * EDGE_E) {
      const int ci = (i >> 6) & 255, tap = (i >> 14) % 5, side = i / EDGE_E;
      const int o = (side & 1) ? 2 : 0;  // pred.0's outer row / column; convB's is 2 - o
      for (int cm = 0; cm < 256; ++cm)
        for (int k = 0; k < 3; ++k) {
          const int e = tap - k;
          if (e < 0 || e > 2) continue;
          s += side < 2 ? P(co, cm, o, k) * Q(cm, ci, 2 - o, e) : P(co, cm, k, o) * Q(cm, ci, e, 2 - o);
        }
    } else if (i < 4 * EDGE_E + 4 * EDGE_C) {
      const int j = i - 4 * EDGE_E, ci = (j >> 6) & 255, cn = j / EDGE_C;
      const int ky = (cn >> 1) * 2, kx = (cn & 1) * 2;
      for (int cm = 0; cm < 256; ++cm) s += P(co, cm, ky, kx) * Q(cm, ci, 2 - ky, 2 - kx);
    } else {
      const int c = (i - 4 * EDGE_E - 4 * EDGE_C) >> 6;  // sides T, B, L, R, then corners TL, TR, BL, BR
      for (int cm = 0; cm < 256; ++cm) {
        const double b = bb[cm];
        if (c < 4) {
          const int o = (c & 1) ? 2 : 0;
          for (int k = 0; k < 3; ++k) s += (c < 2 ? P(co, cm, o, k) : P(co, cm, k, o)) * b;
        } else {
          s += P(co, cm, ((c - 4) >> 1) * 2, ((c - 4) & 1) * 2) * b;
        }
      }
    }
    edge[i] = static_cast<float>(s);
  }
}
// K5 * scale -> fp16 hi / lo in conv5x5_fold_kernel's packed order
__global__ void pack_fold_kernel(const double* __restrict__ k5, __half* __restrict__ out, double scale) {
  const int n = 64 * 256 * 25;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int t5 = i % 25, ci = (i / 25) % 256, co = i / (25 * 256);
    const double v = k5[i] * scale;
    const __half hi = __float2half_rn(static_cast<float>(v));
    const __half lo = __float2half_rn(static_cast<float>(v - static_cast<double>(__half2float(hi))));
    const int kc = ci / 16, kg = (ci / 8) & 1, k8 = ci & 7;
    const size_t base = static_cast<size_t>((kc * 25 + t5) * 2) * 2;  // [chunk][dy][dx][plane][k group]
    const size_t cm = static_cast<size_t>((co >> 3) * 64 + (co & 7) * 8 + k8);
    out[(base + 0 + kg) * 512 + cm] = hi;
    out[(base + 2 + kg) * 512 + cm] = lo;
  }
}

}  // namespace dd
