// 3x3 / stride 1 / pad 1 convolution as an implicit GEMM on Hopper's warpgroup MMA (wgmma), with ROW-HALO REUSE of
// the activation operand.
//
//   M = 128 output pixels (a 16-row x 8-column patch of one image), N = COUT, K = 9 taps x CIN.
//
// Operands are fp16 hi/lo planes of the fp32 tensors (x = hi + lo, each scaled by a power of two), and every K step
// issues three MMAs  D += A_lo*B_hi ; D += A_hi*B_hi ; D += A_hi*B_lo  so the fp32 accumulator carries ~22
// significant bits per product (SURVEY.md §7.2-1: a single fp16/tf32 pass misses the 1e-3 parity bar after 20 DDIM
// steps, the 3-pass split matches fp32).
//
// Row-halo reuse: per channel chunk the producer fetches three [18 rows][8 cols] column-shifted strips (dx = -1, 0,
// +1) with one 4-D TMA tensor map {C, W, H, B} (TMA's out-of-bounds zero fill *is* the conv's zero padding).  For tap
// (dy, dx) the A operand is strip dx starting dy rows down: its 8-pixel row groups are dense and aligned to the
// swizzle atom, so the canonical K-major wgmma descriptor (SBO = 8 rows) addresses it with no copy.  The activation
// bytes moved per chunk drop from 9 x 128 to 3 x 144 pixel rows.  Weights are pre-packed [tap][COUT][CIN] fp16 hi/lo
// and fetched by a 3-D map with box {BK, COUT, 1}.
//
// Roles: warpgroup 0 = producers (warp 0: A strips, warp 1: B weight tiles; one elected lane issues the copies),
// warpgroups 1 .. NWG = consumers.  Consumer warpgroup w owns all 128 pixels of the tile and output channels
// [w NW, (w + 1) NW) as two 64-row wgmma accumulators in registers.  After the K loop each consumer warp applies
// scale and bias (and the fp16 hi/lo split) to its fragments in registers, writes them once into its own store buffer
// laid out as the NHWC output box (16 pixels x up to 32 channels), and one lane hands the box to a TMA tensor store,
// which clips it at the image's right and bottom edges.  The warps only wait until a buffer has been read out before
// writing it again, never on global memory, and need no warpgroup barrier, so the next tile's MMAs start while the
// stores drain.  GroupNorm partials are summed per pixel from the staged fp32 chunks in column order, then combined
// in a fixed order (bit-reproducible).
// Replaces: the nn.Conv2d calls inside ScheduledCNNRefine (reference
// src/model/head/ddim_depth_estimate_res_swin_addHAHI.py:339-359, UpSample_add :321-333).
#pragma once
#include "conv_common.cuh"

namespace dd {

constexpr int HALO_TH = 16;  // output tile: 16 rows x 8 columns = 128 pixels
constexpr int HALO_TW = 8;
// output channels per TMA store box of the epilogue (the output maps are built with the same box)
constexpr int halo_out_box_c(int cout) { return cout < 32 ? cout : 32; }

template <int CIN, int COUT, int BK>
struct HaloCfg {
  static_assert(BK == 16 || BK == 32, "bad K chunk");
  static_assert((CIN % BK == 0 || CIN < BK) && CIN % 16 == 0, "bad K chunk");
  static constexpr int KC = (CIN + BK - 1) / BK;
  static constexpr int KSTEPS = (CIN < BK ? CIN : BK) / 16;
  static constexpr int ROW_BYTES = BK * 2;
  static constexpr int STRIP_ROWS = (HALO_TH + 2) * HALO_TW;        // 144 pixel rows
  static constexpr int STRIP_BYTES = STRIP_ROWS * ROW_BYTES;        // one plane, one dx
  static constexpr int STRIP_PAD = (STRIP_BYTES + 1023) / 1024 * 1024;
  static constexpr int DX_STRIDE = 2 * STRIP_PAD;                   // planes of one dx: hi, lo
  static constexpr int A_SLOT = 3 * DX_STRIDE;
  static constexpr int A_SLOTS = 2;
  static constexpr int B_TILE = COUT * ROW_BYTES;                   // one plane, one tap, one chunk
  static constexpr int B_TILE_PAD = (B_TILE + 1023) / 1024 * 1024;
  static constexpr int B_SLOT = 2 * B_TILE_PAD;
  // consumer warpgroups: a 64 x NW fp32 accumulator takes NW / 2 registers per thread, two of them (128 rows) NW
  static constexpr int NWG = COUT > 128 ? 2 : 1;
  static constexpr int NW = COUT / NWG;
  static constexpr int THREADS = 128 * (1 + NWG);
  // Epilogue: each consumer warp stores its 16 fragment rows (two image rows of 8 pixels) in boxes of OC channels,
  // OUT_BUFS buffers per warp.  A buffer holds one box as fp32, or as the fp16 hi plane followed by the lo plane; a
  // box row (OC channels of one pixel) is the swizzle span.  The two-warpgroup (256-wide) layers get one buffer per
  // warp (16 KB in all), which leaves room for a third weight slot, so the producer runs two taps ahead of the MMAs.
  static constexpr int OC = halo_out_box_c(COUT);
  static constexpr int OBUF = 16 * OC * 4;
  static constexpr int OUT_BUFS = NWG > 1 ? 1 : 4;
  static_assert(NW % OC == 0 && OC % 8 == 0, "a warp's columns are whole store boxes of whole fragment blocks");
  static constexpr int STAGE_BYTES = NWG * 4 * OUT_BUFS * OBUF;
  static constexpr int CTRL_BYTES = 1024;  // barriers, GroupNorm partials [2][4 NWG][GPW][2] (fp64)
  static constexpr int BUDGET = 227 * 1024 - 1024 - CTRL_BYTES - STAGE_BYTES - A_SLOTS * A_SLOT;
  static constexpr int B_SLOTS_RAW = BUDGET / B_SLOT;
  // Small layers (16->64, 64->16): all 9 x KC weight tiles fit in shared memory -> fetch them ONCE per CTA instead of
  // once per tile.
  static constexpr bool B_RESIDENT = (9 * KC * B_SLOT <= 40 * 1024) && (9 * KC <= B_SLOTS_RAW);
  static constexpr int B_SLOTS = B_RESIDENT ? 9 * KC : (B_SLOTS_RAW > 8 ? 8 : B_SLOTS_RAW);
  static_assert(B_SLOTS >= 2, "B ring too small");
  static_assert(NWG == 1 || B_SLOTS >= 3, "256-wide layers: the producer must be able to run two taps ahead");
  static constexpr int SMEM_BYTES = A_SLOTS * A_SLOT + B_SLOTS * B_SLOT + 1024 + CTRL_BYTES + STAGE_BYTES;
  static_assert(SMEM_BYTES <= 232448, "exceeds the 227 KB dynamic shared memory limit");
  static constexpr int A_TX = 6 * STRIP_BYTES;
  static constexpr int B_TX = 2 * B_TILE;
  static constexpr int GROUP_CH = COUT / 4;  // GroupNorm(4, COUT)
  static constexpr int GPW = NW >= GROUP_CH ? NW / GROUP_CH : 1;  // groups per consumer warpgroup
  static_assert(NW % GROUP_CH == 0, "a warpgroup's columns cover whole GroupNorm groups");
};

template <int CIN, int COUT, int BK, int EPI>
__global__ void __launch_bounds__((HaloCfg<CIN, COUT, BK>::THREADS), 1)
conv3x3_halo_kernel(const __grid_constant__ CUtensorMap tmA_hi, const __grid_constant__ CUtensorMap tmA_lo,
                    const __grid_constant__ CUtensorMap tmB_hi, const __grid_constant__ CUtensorMap tmB_lo,
                    const __grid_constant__ CUtensorMap tmO0, const __grid_constant__ CUtensorMap tmO1,
                    const ConvArgs p) {
  using C = HaloCfg<CIN, COUT, BK>;
  constexpr int NW = C::NW;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* a_ring = smem;
  uint8_t* b_ring = smem + C::A_SLOTS * C::A_SLOT;
  uint8_t* ctrl = b_ring + C::B_SLOTS * C::B_SLOT;
  uint64_t* a_full = reinterpret_cast<uint64_t*>(ctrl);
  uint64_t* a_empty = a_full + C::A_SLOTS;
  uint64_t* b_full = a_empty + C::A_SLOTS;
  uint64_t* b_empty = b_full + C::B_SLOTS;
  double* red = reinterpret_cast<double*>(b_empty + C::B_SLOTS);  // [2][4 NWG][GPW][2]
  uint8_t* stage = ctrl + C::CTRL_BYTES;  // [consumer warp][OUT_BUFS] store buffers

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA_hi);
    tma_prefetch_desc(&tmA_lo);
    tma_prefetch_desc(&tmB_hi);
    tma_prefetch_desc(&tmB_lo);
    tma_prefetch_desc(&tmO0);
    if (EPI == EPI_SPLIT) tma_prefetch_desc(&tmO1);
    // full: one arrive.expect_tx by the producer; empty: one arrive per consumer warpgroup
    for (int s = 0; s < C::A_SLOTS; ++s) {
      mbar_init(&a_full[s], 1);
      mbar_init(&a_empty[s], C::NWG);
    }
    for (int s = 0; s < C::B_SLOTS; ++s) {
      mbar_init(&b_full[s], 1);
      mbar_init(&b_empty[s], C::NWG);
    }
    fence_barrier_init();
  }
  __syncthreads();

  // setmaxnreg sits at the top of each role's branch and the branches only meet again at the exit.  With a merge point
  // after it (one if / else, then the role dispatch) ptxas ignored setmaxnreg (C7507) and the consumers' accumulators
  // spilled at the 168-register launch bound.  The two producer warps need few registers; 24 leave the consumers 240,
  // which the 256-wide statistics epilogue needs to hold its 128 accumulator registers without spilling.
  if (warp < 4) {
    if constexpr (C::NWG > 1) setmaxnreg_dec<24>();
    if (warp == 0) {
      // ---------------------------------------------------------------- TMA producer (A strips).  The WHOLE warp walks
      // the loop (barrier waits and coordinates stay warp-uniform) and one elected lane issues the copies.
      const bool leader = elect_one();
      int sa = 0;
      uint32_t pa = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const int tx = tile % p.tiles_x, ty = (tile / p.tiles_x) % p.tiles_y, img = tile / (p.tiles_x * p.tiles_y);
        const int x0 = tx * HALO_TW, y0 = ty * HALO_TH;
        for (int kc = 0; kc < C::KC; ++kc) {
          mbar_wait(&a_empty[sa], pa ^ 1);
          uint8_t* s = a_ring + sa * C::A_SLOT;
          if (leader) {
            mbar_arrive_expect_tx(&a_full[sa], C::A_TX);
#pragma unroll
            for (int dx = 0; dx < 3; ++dx) {
              tma_load_4d(s + (2 * dx) * C::STRIP_PAD, &tmA_hi, &a_full[sa], kc * BK, x0 + dx - 1, y0 - 1, img);
              tma_load_4d(s + (2 * dx + 1) * C::STRIP_PAD, &tmA_lo, &a_full[sa], kc * BK, x0 + dx - 1, y0 - 1, img);
            }
          }
          __syncwarp();
          if (++sa == C::A_SLOTS) {
            sa = 0;
            pa ^= 1;
          }
        }
      }
    } else if (warp == 1) {
      // ---------------------------------------------------------------- TMA producer (B weight tiles), same structure
      const bool leader = elect_one();
      int sb = 0;
      uint32_t pb = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        if (C::B_RESIDENT && tile != static_cast<int>(blockIdx.x)) break;  // weights stay in their slots after the first tile
        for (int kc = 0; kc < C::KC; ++kc) {
          for (int tap = 0; tap < 9; ++tap) {
            mbar_wait(&b_empty[sb], pb ^ 1);
            uint8_t* s = b_ring + sb * C::B_SLOT;
            if (leader) {
              mbar_arrive_expect_tx(&b_full[sb], C::B_TX);
              tma_load_3d(s, &tmB_hi, &b_full[sb], kc * BK, 0, tap);
              tma_load_3d(s + C::B_TILE_PAD, &tmB_lo, &b_full[sb], kc * BK, 0, tap);
            }
            __syncwarp();
            if (++sb == C::B_SLOTS) {
              sb = 0;
              pb ^= 1;
            }
          }
        }
      }
    }
  } else {
    if constexpr (C::NWG > 1) setmaxnreg_inc<240>();
    // ------------------------------------------------------------------ consumers: MMA + epilogue
    const int wg = (warp >> 2) - 1;  // consumer warpgroup
    const int t = threadIdx.x & 127;
    const int q = t >> 5;
    const bool signal = (t == 0);    // the thread that releases ring slots for its warpgroup
    uint8_t* obufs = stage + wg * 4 * C::OUT_BUFS * C::OBUF;  // this warpgroup's, [warp][OUT_BUFS]
    const int m = t;                 // epilogue statistics: this thread's row (pixel) of the tile
    const int r = m >> 3, c = m & 7;
    const uint32_t b_off = static_cast<uint32_t>(wg * NW);  // first weight row of this warpgroup
    int sa = 0, sb = 0, par = 0, ob = 0;
    uint32_t pa = 0, pb = 0;
    float acc[2][NW / 2];

    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      // ---------------------------------------------------------------- mainloop
      int prev_b = -1, prev_a = -1;  // slots read by the wgmma group still in flight
      auto retire_prev = [&]() {  // predicated arrives: no branch between wgmma issue and wait
        mbar_arrive_if(&b_empty[prev_b < 0 ? 0 : prev_b], signal && prev_b >= 0);
        mbar_arrive_if(&a_empty[prev_a < 0 ? 0 : prev_a], signal && prev_a >= 0);
        prev_b = prev_a = -1;
      };
      {
        for (int kc = 0; kc < C::KC; ++kc) {
          mbar_wait(&a_full[sa], pa);
          const uint32_t a_base = smem_u32(a_ring + sa * C::A_SLOT);
          for (int tap = 0; tap < 9; ++tap) {
            const int dy = tap / 3, dx = tap % 3;
            mbar_wait(&b_full[sb], C::B_RESIDENT ? 0u : pb);  // resident: phase 0 completes once and stays complete
            // strip dx, dy rows down: 8-pixel groups stay dense (8 * ROW_BYTES) and aligned to the swizzle atom
            const uint32_t sa_hi = a_base + dx * C::DX_STRIDE + dy * HALO_TW * C::ROW_BYTES;
            const uint32_t sa_lo = sa_hi + C::STRIP_PAD;
            const uint32_t sb_hi = smem_u32(b_ring + sb * C::B_SLOT) + b_off * C::ROW_BYTES;
            const uint32_t sb_lo = sb_hi + C::B_TILE_PAD;
            wgmma_fence();
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const uint32_t ho = static_cast<uint32_t>(h * 64 * C::ROW_BYTES);
#pragma unroll
              for (int k = 0; k < C::KSTEPS; ++k) {
                const uint64_t a_hi = wgmma_desc(sa_hi + ho + k * 32, C::ROW_BYTES);
                const uint64_t a_lo = wgmma_desc(sa_lo + ho + k * 32, C::ROW_BYTES);
                const uint64_t b_hi = wgmma_desc(sb_hi + k * 32, C::ROW_BYTES);
                const uint64_t b_lo = wgmma_desc(sb_lo + k * 32, C::ROW_BYTES);
                wgmma_f16<NW>(acc[h], a_lo, b_hi, (kc | tap | k) != 0 ? 1u : 0u);  // small terms first
                wgmma_f16<NW>(acc[h], a_hi, b_lo, 1u);
                wgmma_f16<NW>(acc[h], a_hi, b_hi, 1u);
              }
            }
            wgmma_commit();
            wgmma_wait<1>();
            retire_prev();
            if (!C::B_RESIDENT) prev_b = sb;
            if (tap == 8) prev_a = sa;
            if (++sb == C::B_SLOTS) {
              sb = 0;
              pb ^= 1;
            }
          }
          if (++sa == C::A_SLOTS) {
            sa = 0;
            pa ^= 1;
          }
        }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc[0]);
      wgmma_fence_regs(acc[1]);
      retire_prev();  // the producers refill the rings while this warpgroup drains its accumulators

      // ---------------------------------------------------------------- epilogue
      // Warp q holds fragment rows 64 h + 16 q + [0, 16) of accumulator h: image rows y0 + 8 h + 2 q + {0, 1}, all 8
      // columns.  Per OC-column chunk it applies scale + bias (+ the hi/lo split) in registers, writes the chunk once
      // into a store buffer laid out as the NHWC box {OC, 8, 2} (swizzled as the output map), and lane 0 stores it
      // with one TMA tensor store per plane.  The box is clipped to the image, and nobody waits on the global write:
      // before a buffer is written again, lane 0 only waits until the store that last used it has read it out.
      const int tx = tile % p.tiles_x, ty = (tile / p.tiles_x) % p.tiles_y, img = tile / (p.tiles_x * p.tiles_y);
      const int x0 = tx * HALO_TW, y0 = ty * HALO_TH;
      const bool valid = (x0 + c < p.W) && (y0 + r < p.H);
      // E[v^2] - mean^2 cancels (mean / std)^2 of the sums' significant bits, so a group whose mean dominates its
      // spread loses its variance in plain fp32 sums (rstd off by 1e-2 at mean / std = 1000).  Each thread sums its
      // pixel's d = v - k in fp32, k = the pixel's first value in the group (|d| ~ the group's spread), and turns the
      // sums into fp64 sums of v and v^2 once per group.  Thread m reads its pixel back from the staged chunks, in
      // column order.
      float tk[C::GPW], tsum[C::GPW], tsq[C::GPW];
#pragma unroll
      for (int g = 0; g < C::GPW; ++g) tk[g] = tsum[g] = tsq[g] = 0.f;
      bool overflow = false;
      constexpr int SPAN = C::OC * (EPI == EPI_SPLIT ? 2 : 4);  // bytes per box row
      auto swz = [](int a) { return a ^ (((a >> 7) & (SPAN / 16 - 1)) << 4); };  // TMA swizzle of byte offset a
      const int fc = 2 * (lane & 3), fr = lane >> 2;  // fragment column pair within an 8-column block, row within 8
      uint8_t* wbufs = obufs + q * C::OUT_BUFS * C::OBUF;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int yb = y0 + 8 * h + 2 * q;
#pragma unroll
        for (int cc = 0; cc < NW / C::OC; ++cc) {
          const int ch0 = wg * NW + cc * C::OC;
          uint8_t* O = wbufs + ob * C::OBUF;
          if (lane == 0) bulk_wait_group_read<C::OUT_BUFS - 1>();  // the store that last used O has read it
          // one buffer per warp: every thread has also read its statistics out of the buffers
          if constexpr (EPI == EPI_F32_STATS && C::OUT_BUFS == 1) named_bar_sync(2 + wg, 128);
          __syncwarp();
#pragma unroll
          for (int b = 0; b < C::OC / 8; ++b) {
            const int blk = cc * C::OC / 8 + b;
            const float b0 = __ldg(p.bias + ch0 + 8 * b + fc), b1 = __ldg(p.bias + ch0 + 8 * b + fc + 1);
#pragma unroll
            for (int e = 0; e < 2; ++e) {  // fragment rows fr and fr + 8 (stage_acc_cols' layout): image row yb + e
              const float v0 = fmaf(acc[h][4 * blk + 2 * e], p.acc_scale, b0);
              const float v1 = fmaf(acc[h][4 * blk + 2 * e + 1], p.acc_scale, b1);
              const int o = (8 * e + fr) * C::OC + 8 * b + fc;  // element of the box
              if constexpr (EPI == EPI_SPLIT) {
                const float s0 = v0 * p.split_scale, s1 = v1 * p.split_scale;
                const bool rv = (x0 + fr < p.W) && (yb + e < p.H);
                overflow |= rv && (fabsf(s0) > 60000.f || fabsf(s1) > 60000.f);
                const __half h0 = __float2half_rn(s0), h1 = __float2half_rn(s1);
                const __half l0 = __float2half_rn(s0 - __half2float(h0)), l1 = __float2half_rn(s1 - __half2float(h1));
                *reinterpret_cast<__half2*>(O + swz(2 * o)) = __halves2half2(h0, h1);
                *reinterpret_cast<__half2*>(O + C::OBUF / 2 + swz(2 * o)) = __halves2half2(l0, l1);  // lo plane
              } else {
                *reinterpret_cast<float2*>(O + swz(4 * o)) = make_float2(v0, v1);
              }
            }
          }
          fence_proxy_async();  // this thread's buffer writes become visible to the TMA store
          __syncwarp();
          if (lane == 0) {
            tma_store_4d(&tmO0, O, ch0, x0, yb, img);
            if constexpr (EPI == EPI_SPLIT) tma_store_4d(&tmO1, O + C::OBUF / 2, ch0, x0, yb, img);
            bulk_commit_group();
          }
          if constexpr (EPI == EPI_F32_STATS) {
            named_bar_sync(2 + wg, 128);  // every warp's chunk is staged
            if (valid && (m >> 6) == h) {
              const uint8_t* src = obufs + (((m & 63) >> 4) * C::OUT_BUFS + ob) * C::OBUF;  // the warp that holds m
#pragma unroll
              for (int u = 0; u < C::OC / 4; ++u) {
                const float4 f = *reinterpret_cast<const float4*>(src + swz(((m & 15) * C::OC + 4 * u) * 4));
                const float vv[4] = {f.x, f.y, f.z, f.w};
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                  const int col = cc * C::OC + 4 * u + i;
                  const int g = col / C::GROUP_CH;  // compile-time: group within this warpgroup's columns
                  if (col % C::GROUP_CH == 0) tk[g] = vv[i];
                  const float d = vv[i] - tk[g];
                  tsum[g] += d;
                  tsq[g] = fmaf(d, d, tsq[g]);
                }
              }
            }
          }
          if (++ob == C::OUT_BUFS) ob = 0;
        }
      }

      if constexpr (EPI == EPI_F32_STATS) {
        // warp tree -> shared memory -> 8 threads combine the consumer warps in fixed order (deterministic)
        const int cw = wg * 4 + q;  // consumer warp index
#pragma unroll
        for (int k = 0; k < C::GPW; ++k) {  // this warpgroup's groups
          const double n = valid ? C::GROUP_CH : 0, kk = tk[k], ds = tsum[k];
          double s = fma(n, kk, ds), s2 = fma(n * kk, kk, fma(2.0 * kk, ds, static_cast<double>(tsq[k])));
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            s += __shfl_xor_sync(0xffffffffu, s, o);
            s2 += __shfl_xor_sync(0xffffffffu, s2, o);
          }
          if (lane == 0) {
            red[((par * 4 * C::NWG + cw) * C::GPW + k) * 2 + 0] = s;
            red[((par * 4 * C::NWG + cw) * C::GPW + k) * 2 + 1] = s2;
          }
        }
        named_bar_sync(1, 128 * C::NWG);
        const int e = threadIdx.x - 128;
        if (e < 8) {
          const int g = e >> 1, which = e & 1;
          const int w0 = C::NWG > 1 ? (g / C::GPW) * 4 : 0, k = C::NWG > 1 ? g % C::GPW : g;  // the group's warps
          double tt = 0.0;
#pragma unroll
          for (int w = 0; w < 4 * C::NWG; ++w)
            if (C::NWG == 1 || (w >= w0 && w < w0 + 4)) tt += red[((par * 4 * C::NWG + w) * C::GPW + k) * 2 + which];
          p.stats_partial[(static_cast<size_t>(tile) * 4 + g) * 2 + which] = tt;
        }
        par ^= 1;  // double-buffered scratch: one barrier per tile is enough
      }
      if constexpr (EPI == EPI_SPLIT) {
        if (overflow) atomicOr(p.status, 1);
      }
    }
    if (lane == 0) bulk_wait_group<0>();  // each warp's store buffers stay valid until its last stores have completed
  }
}

}  // namespace dd
