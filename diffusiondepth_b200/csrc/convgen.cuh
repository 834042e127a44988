// General convolution (1x1 or 3x3, zero pad, stride 1 or 2) + per-channel shift (+activation, +addend) on the warpgroup
// MMA (wgmma), used
// for the step-invariant producers: HAHI neck (1x1 / 3x3 ConvModules with eval-BN folded, channel-concatenated
// inputs) and the FPN (3x3 laterals, 2x2/s2 transposed convs as a 1x1 GEMM with a pixel-shuffle epilogue).
// Same machinery as conv3x3_halo_kernel (3-pass fp16 hi/lo split, TMA-staged swizzled tiles, register accumulators,
// warp-specialised persistent CTA) with runtime shapes:
//   M = 128 pixels (8x16 patch), N tile = NT output channels, K = taps x (cin0 + cin1) in chunks of 32 channels,
//   the K range may be fed from two source tensors (torch.cat([a, b], dim=1) never materialises).
// Replaces (reference): mmcv ConvModule calls in src/model/necks/hahi.py:165-276 and the FPN in
// src/model/head/ddim_depth_estimate_res_swin_addHAHI.py:112-122.
#pragma once
#include "conv_common.cuh"

namespace dd {

struct GenConvArgs {
  int B, H, W;
  int tiles_x, tiles_y, m_tiles, n_tiles;
  int kc0, kc1;       // GEN_BK-channel chunks taken from source 0, then source 1 (ceil: a partial last chunk is completed
                      // with zeros by TMA's out-of-bounds fill, on the activation AND the weight side)
  int c0_ch;          // real channel count of source 0 = weight K offset of source 1's first channel
  int taps;           // 1 (1x1) or 9 (3x3, pad 1)
  int ld_out, ch_off; // output rows are ld_out channels wide and this layer writes [ch_off, ch_off + cout) of them: branches
                      // of a concatenation write straight into the concatenated tensor (ld_out = cout, ch_off = 0 otherwise;
                      // not combined with `shuffle`).  The residual `add32` is always dense [pixel][cout].
  int cout;           // total output channels (any multiple of 8; n_tiles = ceil(cout / NT), columns >= cout are dropped)
  const float* shift; // [cout] bias / folded BN shift
  float acc_scale;
  int relu;           // activation: 0 none, 1 ReLU, 2 exact (erf) GELU, 3 Hardswish x * relu6(x + 3) / 6
  int m_valid;        // > 0: GEMM mode (B = 1, W = 16): only "pixels" (tokens) with index < m_valid are stored
  int stride;         // 1 or 2: input pixel of output (y, x), tap (dy, dx) is (stride*y + dy, stride*x + dx); the A tensor
                      // maps are then built with elementStrides = stride so one box still delivers 8 x 16 pixels
  int add_first;      // 1: addend is added BEFORE the activation (ResNet residual), 0: after it (FPN top-down add)
  int shuffle;        // 1: ConvTranspose2d(k=2,s=2): channel n = q*(cout/4)+c goes to pixel (2y+q/2, 2x+q%2), channel c
  float* y32;         // optional fp32 NHWC output
  const float* add32; // optional fp32 NHWC addend (indexed like y32), added after the ReLU
  __half* out_hi;     // optional fp16 hi/lo planes of the output (indexed like y32)
  __half* out_lo;
  float split_scale;
  int* status;
};

// K chunk of the producer convs / GEMMs: 64 channels = 128-byte operand rows (128-byte swizzle): half the TMA row
// requests and barrier round trips per byte of 32-channel chunks.
constexpr int GEN_BK = 64;

// Columns of one consumer unit of an NT-wide work item: 128 x NT items split into two units of NT / 2 columns when
// 128 x NT fp32 accumulators would not fit one warpgroup's registers.  Also the row count of the weight maps' boxes.
constexpr int gen_unit_cols(int nt) { return nt > 128 ? nt / 2 : nt; }

template <int NT>
struct GenCfg {
  static constexpr int BK = GEN_BK;
  static constexpr int ROW_BYTES = BK * 2;
  // one unit: all 128 rows of the tile and NW columns (NW registers of accumulators per consumer thread)
  static constexpr int NW = gen_unit_cols(NT);
  static constexpr int UNITS = NT / NW;  // units per work item
  static constexpr int A_BYTES = TILE_M * ROW_BYTES;  // 16 KB per plane
  static constexpr int B_BYTES = NW * ROW_BYTES;
  static constexpr int STAGE_BYTES = 2 * (A_BYTES + B_BYTES);  // one unit's K chunk
  static constexpr int THREADS = 384;  // producer warpgroup + two consumer warpgroups taking units in turn
  static constexpr int LD = 20;  // staging row stride (floats): 16 columns + 4, rows stay 16-byte aligned
  static constexpr int STAGING_BYTES = 2 * 128 * LD * 4;
  static constexpr int STAGES_RAW = (227 * 1024 - 1024 - 512 - STAGING_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 6 ? 6 : STAGES_RAW;
  static_assert(STAGES >= 3, "stage too large");
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 512 + STAGING_BYTES;
  static_assert(SMEM_BYTES <= 232448, "exceeds the 227 KB dynamic shared memory limit");
  static_assert(NW % 16 == 0 && NT <= 256, "bad N tile");  // instantiated: 64, 128, 192, 256
};

// Warp roles: warp 0 = TMA producer of the activation planes, warp 1 = of the weight planes; warpgroups 1 and 2 =
// consumers.  The CTA's work items are cut into units (128 rows x NW columns, UNITS per item) and numbered in order;
// consumer warpgroup w takes the units j with j % 2 == w: wgmma mainloop, then the epilogue of the unit, drained 16
// columns at a time through a shared-memory staging tile that hands each thread one ROW (pixel / token) of the chunk.
// The producers fill the stage ring unit after unit, and a pair of named barriers hands the tensor cores from unit j's
// mainloop to unit j + 1's: one warpgroup's epilogue runs under the other's MMAs, and every consumer finds the ring
// position of its unit (j * k_iters) filled in order.
template <int NT>
__global__ void __launch_bounds__((GenCfg<NT>::THREADS), 1)
convgen_wgmma_kernel(const __grid_constant__ CUtensorMap tmA0_hi, const __grid_constant__ CUtensorMap tmA0_lo,
                     const __grid_constant__ CUtensorMap tmA1_hi, const __grid_constant__ CUtensorMap tmA1_lo,
                     const __grid_constant__ CUtensorMap tmB_hi, const __grid_constant__ CUtensorMap tmB_lo,
                     const GenConvArgs p) {
  using C = GenCfg<NT>;
  constexpr int NW = C::NW;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + C::STAGES * C::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + C::STAGES;
  float* stage_f = reinterpret_cast<float*>(smem + C::STAGES * C::STAGE_BYTES + 512);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int kc_total = p.kc0 + p.kc1;
  const int k_iters = p.taps * kc_total;
  const int num_work = p.m_tiles * p.n_tiles;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA0_hi);
    tma_prefetch_desc(&tmA0_lo);
    tma_prefetch_desc(&tmB_hi);
    tma_prefetch_desc(&tmB_lo);
    for (int s = 0; s < C::STAGES; ++s) {
      mbar_init(&full_bar[s], 2);        // two producers (activation planes / weight planes) arrive per stage
      mbar_init(&empty_bar[s], 1);       // the one consumer warpgroup of the stage's unit
    }
    fence_barrier_init();
  }
  __syncthreads();
  auto stage_ptr = [&](int s) { return smem + s * C::STAGE_BYTES; };

  // setmaxnreg at the top of each role's branch, branches meeting only at the exit (see conv3x3_halo_kernel)
  if (warp < 4) {
    setmaxnreg_dec<40>();
    if (warp == 0 || warp == 1) {
      // two TMA producers; the whole warp walks the loop, one elected lane issues (consecutive UTMALDGs)
      const bool act = (warp == 0);
      const bool leader = elect_one();
      int stage = 0;
      uint32_t phase = 0;
      for (int work = blockIdx.x; work < num_work; work += gridDim.x) {
        const int nt = work % p.n_tiles;  // n fastest: neighbours share the A patch in L2
        const int mt = work / p.n_tiles;
        const int tx = mt % p.tiles_x, ty = (mt / p.tiles_x) % p.tiles_y, img = mt / (p.tiles_x * p.tiles_y);
        const int x0 = tx * TILE_W, y0 = ty * TILE_H;
        // the item's units one after the other; each loads its own copy of the A tile (an L2 hit after the first)
        for (int u = 0; u < C::UNITS; ++u) {
        for (int tap = 0; tap < p.taps; ++tap) {
          const int dy = p.taps == 9 ? tap / 3 - 1 : 0, dx = p.taps == 9 ? tap % 3 - 1 : 0;
          for (int kc = 0; kc < kc_total; ++kc) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            uint8_t* s = stage_ptr(stage);
            const int ax = x0 * p.stride + dx, ay = y0 * p.stride + dy;
            // weight K coordinate of this chunk: source 1's channels start right after source 0's REAL channels
            const int kw = kc < p.kc0 ? kc * C::BK : p.c0_ch + (kc - p.kc0) * C::BK;
            if (leader) {
              if (!act) {
                mbar_arrive_expect_tx(&full_bar[stage], 2 * C::B_BYTES);
                tma_load_3d(s + 2 * C::A_BYTES, &tmB_hi, &full_bar[stage], kw, nt * NT + u * C::NW, tap);
                tma_load_3d(s + 2 * C::A_BYTES + C::B_BYTES, &tmB_lo, &full_bar[stage], kw, nt * NT + u * C::NW, tap);
              } else if (kc < p.kc0) {
                mbar_arrive_expect_tx(&full_bar[stage], 2 * C::A_BYTES);
                tma_load_4d(s, &tmA0_hi, &full_bar[stage], kc * C::BK, ax, ay, img);
                tma_load_4d(s + C::A_BYTES, &tmA0_lo, &full_bar[stage], kc * C::BK, ax, ay, img);
              } else {
                mbar_arrive_expect_tx(&full_bar[stage], 2 * C::A_BYTES);
                tma_load_4d(s, &tmA1_hi, &full_bar[stage], (kc - p.kc0) * C::BK, ax, ay, img);
                tma_load_4d(s + C::A_BYTES, &tmA1_lo, &full_bar[stage], (kc - p.kc0) * C::BK, ax, ay, img);
              }
            }
            __syncwarp();
            if (++stage == C::STAGES) {
              stage = 0;
              phase ^= 1;
            }
          }
        }
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    const int wg = (warp >> 2) - 1;
    const int t = threadIdx.x & 127;
    const int q = t >> 5;
    const int m = t;
    const int r = m >> 4, c = m & 15;
    float* S = stage_f + wg * 128 * C::LD;
    float* T = S + q * 32 * C::LD;  // this warp's 32 rows
    bool overflow = false;
    const int cq = p.cout >> 2;
    float acc[2][NW / 2];
    int unit = -1;  // index of the CTA's current unit
    for (int work = blockIdx.x; work < num_work; work += gridDim.x) {
    for (int u = 0; u < C::UNITS; ++u) {
      if (((++unit) & 1) != wg) continue;
      // ---------------------------------------------------------------- mainloop
      if (unit > 0) named_bar_sync(4 + wg, 256);  // the previous unit has issued its MMAs
      int stage = (unit * k_iters) % C::STAGES;
      uint32_t phase = ((unit * k_iters) / C::STAGES) & 1;
      int prev = -1;
      for (int it = 0; it < k_iters; ++it) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa_hi = smem_u32(stage_ptr(stage));
        const uint32_t sa_lo = sa_hi + C::A_BYTES;
        const uint32_t sb_hi = sa_hi + 2 * C::A_BYTES;
        const uint32_t sb_lo = sb_hi + C::B_BYTES;
        wgmma_fence();
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint32_t ho = static_cast<uint32_t>(h * 64 * C::ROW_BYTES);
#pragma unroll
          for (int k = 0; k < C::BK / 16; ++k) {
            const uint64_t a_hi = wgmma_desc(sa_hi + ho + k * 32, C::ROW_BYTES);
            const uint64_t a_lo = wgmma_desc(sa_lo + ho + k * 32, C::ROW_BYTES);
            const uint64_t b_hi = wgmma_desc(sb_hi + k * 32, C::ROW_BYTES);
            const uint64_t b_lo = wgmma_desc(sb_lo + k * 32, C::ROW_BYTES);
            wgmma_f16<NW>(acc[h], a_lo, b_hi, (it | k) != 0 ? 1u : 0u);  // small terms first
            wgmma_f16<NW>(acc[h], a_hi, b_lo, 1u);
            wgmma_f16<NW>(acc[h], a_hi, b_hi, 1u);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();
        mbar_arrive_if(&empty_bar[prev < 0 ? 0 : prev], t == 0 && prev >= 0);  // predicated: no branch before the wait
        prev = stage;
        if (++stage == C::STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      if (u + 1 < C::UNITS || work + static_cast<int>(gridDim.x) < num_work)
        named_bar_arrive(4 + (wg ^ 1), 256);  // the next unit (the other warpgroup's) may issue its MMAs
      wgmma_wait<0>();
      wgmma_fence_regs(acc[0]);
      wgmma_fence_regs(acc[1]);
      mbar_arrive_if(&empty_bar[prev < 0 ? 0 : prev], t == 0 && prev >= 0);

      // ---------------------------------------------------------------- epilogue
      //   fp32-only outputs: the staging tile re-distributes the chunk so that a lane holds one float4 of a row and 4
      //     lanes cover the row's 64 bytes: every global access is a full 64-byte segment;
      //   plane outputs (fp16 hi / lo for the next GEMM): row-per-thread, 32 contiguous bytes per row and plane.
      const int nt = work % p.n_tiles;
      const int mt = work / p.n_tiles;
      const int tx = mt % p.tiles_x, ty = (mt / p.tiles_x) % p.tiles_y, img = mt / (p.tiles_x * p.tiles_y);
      const int x = tx * TILE_W + c, y = ty * TILE_H + r;
      const bool valid = (x < p.W) && (y < p.H) && (p.m_valid <= 0 || (y * p.W + x) < p.m_valid);
      const uint32_t vmask = __ballot_sync(0xffffffffu, valid);
      // element offset of this lane's row at channel 0 (non-shuffle) -- fits 32 bits for every tensor we produce
      const uint32_t row_base = static_cast<uint32_t>(((static_cast<size_t>(img) * p.H + y) * p.W + x) * p.cout);
      const uint32_t row_out = static_cast<uint32_t>(((static_cast<size_t>(img) * p.H + y) * p.W + x) * p.ld_out + p.ch_off);
      const bool xpose_path = (p.out_hi == nullptr);
#pragma unroll
      for (int ci = 0; ci < NW / 16; ++ci) {
        const int n0 = nt * NT + u * NW + ci * 16;
        if (n0 >= p.cout) break;  // columns past the last real output channel (cout not a multiple of NT): zero weights
        const int nvalid = p.cout - n0;  // >= 8, multiple of 8; < 16 only in the last chunk of such a layer
        named_bar_sync(2 + wg, 128);  // the previous chunk's staging reads are done
        stage_acc_cols<NW, 16, C::LD>(acc[0], S, 0, ci * 2);
        stage_acc_cols<NW, 16, C::LD>(acc[1], S, 64, ci * 2);
        named_bar_sync(2 + wg, 128);
        uint32_t o_lane;
        if (p.shuffle) {
          const int sub = n0 / cq, cc = n0 - sub * cq;
          o_lane = static_cast<uint32_t>(
              ((static_cast<size_t>(img) * (2 * p.H) + (2 * y + (sub >> 1))) * (2 * p.W) + (2 * x + (sub & 1))) * cq + cc);
        } else {
          o_lane = row_base + static_cast<uint32_t>(n0);
        }
        const uint32_t o_out = p.shuffle ? o_lane : row_out + static_cast<uint32_t>(n0);  // where the outputs go
        if (xpose_path) {
          const int sl = lane & 3;  // this lane's float4 slot: channels n0 + 4 sl .. + 3
          const bool col_ok = 4 * sl < nvalid;
          const float4 sh = __ldg(reinterpret_cast<const float4*>(p.shift + n0) + sl);  // shift[] is padded to n_tiles * NT
          uint32_t o[4], oo[4];
          float4 ad[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) {  // rows (lane >> 2) + 8 k: issue the addend loads before any store
            const int row = (lane >> 2) + 8 * k;
            o[k] = __shfl_sync(0xffffffffu, o_lane, row) + 4 * sl;
            oo[k] = __shfl_sync(0xffffffffu, o_out, row) + 4 * sl;
            ad[k] = (p.add32 && col_ok && ((vmask >> row) & 1u)) ? __ldg(reinterpret_cast<const float4*>(p.add32 + o[k]))
                                                                  : make_float4(0.f, 0.f, 0.f, 0.f);
          }
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int row = (lane >> 2) + 8 * k;
            if (!((vmask >> row) & 1u) || !col_ok) continue;
            const float4 a4 = *reinterpret_cast<const float4*>(T + row * C::LD + 4 * sl);
            float tt[4] = {fmaf(a4.x, p.acc_scale, sh.x), fmaf(a4.y, p.acc_scale, sh.y), fmaf(a4.z, p.acc_scale, sh.z),
                           fmaf(a4.w, p.acc_scale, sh.w)};
            const float av[4] = {ad[k].x, ad[k].y, ad[k].z, ad[k].w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              if (p.add_first) tt[j] += av[j];
              if (p.relu == 1) tt[j] = fmaxf(tt[j], 0.f);
              else if (p.relu == 2) tt[j] = 0.5f * tt[j] * (1.f + erff(tt[j] * 0.70710678118654752f));
              else if (p.relu == 3) tt[j] = tt[j] * fminf(fmaxf(tt[j] + 3.f, 0.f), 6.f) * (1.f / 6.f);
              if (!p.add_first) tt[j] += av[j];
            }
            if (p.y32) *reinterpret_cast<float4*>(p.y32 + oo[k]) = make_float4(tt[0], tt[1], tt[2], tt[3]);
          }
        } else if (valid) {
          // row-per-thread path (fp16 plane outputs: 32 contiguous bytes per row and plane)
          float v[16];
#pragma unroll
          for (int j4 = 0; j4 < 4; ++j4) {
            const float4 sh = __ldg(reinterpret_cast<const float4*>(p.shift + n0) + j4);
            const float4 a4 = *reinterpret_cast<const float4*>(S + m * C::LD + 4 * j4);
            v[4 * j4] = fmaf(a4.x, p.acc_scale, sh.x);
            v[4 * j4 + 1] = fmaf(a4.y, p.acc_scale, sh.y);
            v[4 * j4 + 2] = fmaf(a4.z, p.acc_scale, sh.z);
            v[4 * j4 + 3] = fmaf(a4.w, p.acc_scale, sh.w);
          }
          if (p.add32 && p.add_first) {
#pragma unroll
            for (int j4 = 0; j4 < 4; ++j4) {
              if (4 * j4 < nvalid) {
                const float4 a = __ldg(reinterpret_cast<const float4*>(p.add32 + o_lane) + j4);
                v[4 * j4] += a.x; v[4 * j4 + 1] += a.y; v[4 * j4 + 2] += a.z; v[4 * j4 + 3] += a.w;
              }
            }
          }
          if (p.relu == 1) {
#pragma unroll
            for (int j = 0; j < 16; ++j) v[j] = fmaxf(v[j], 0.f);
          } else if (p.relu == 2) {
#pragma unroll
            for (int j = 0; j < 16; ++j) v[j] = 0.5f * v[j] * (1.f + erff(v[j] * 0.70710678118654752f));
          } else if (p.relu == 3) {
#pragma unroll
            for (int j = 0; j < 16; ++j) v[j] = v[j] * fminf(fmaxf(v[j] + 3.f, 0.f), 6.f) * (1.f / 6.f);
          }
          if (p.add32 && !p.add_first) {
#pragma unroll
            for (int j4 = 0; j4 < 4; ++j4) {
              if (4 * j4 < nvalid) {
                const float4 a = __ldg(reinterpret_cast<const float4*>(p.add32 + o_lane) + j4);
                v[4 * j4] += a.x; v[4 * j4 + 1] += a.y; v[4 * j4 + 2] += a.z; v[4 * j4 + 3] += a.w;
              }
            }
          }
          if (p.y32) {
            float4* d4 = reinterpret_cast<float4*>(p.y32 + o_out);
#pragma unroll
            for (int j = 0; j < 4; ++j)
              if (4 * j < nvalid) d4[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
          }
          // split two channels at a time (one packed fp32 -> fp16x2 conversion each way); the range check is one running
          // max instead of a compare per element
          __align__(16) __half2 hi[8];
          __align__(16) __half2 lo[8];
          float amax = 0.f;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float s0 = v[2 * j] * p.split_scale, s1 = v[2 * j + 1] * p.split_scale;
            amax = fmaxf(amax, fmaxf(fabsf(s0), fabsf(s1)));
            hi[j] = __floats2half2_rn(s0, s1);
            const float2 back = __half22float2(hi[j]);
            lo[j] = __floats2half2_rn(s0 - back.x, s1 - back.y);
          }
          overflow |= !(amax <= 60000.f);  // also catches NaN
          uint4* dh = reinterpret_cast<uint4*>(p.out_hi + o_out);
          uint4* dl = reinterpret_cast<uint4*>(p.out_lo + o_out);
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            if (8 * j < nvalid) {
              dh[j] = reinterpret_cast<const uint4*>(hi)[j];
              dl[j] = reinterpret_cast<const uint4*>(lo)[j];
            }
          }
        }
      }
    }
    }
    if (overflow) atomicOr(p.status, 1);
  }
}

// fp32 NCHW [B][C][P] -> fp16 hi/lo NHWC planes [B][P][C] (scaled): backbone feature maps entering the neck
__global__ void nchw_to_nhwc_split_kernel(const float* __restrict__ in, __half* __restrict__ hi, __half* __restrict__ lo,
                                          int C, int P, float scale, int* status) {
  __shared__ float t[32][33];
  const int b = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const float* src = in + static_cast<size_t>(b) * C * P;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, pp = p0 + threadIdx.x;
    t[i][threadIdx.x] = (c < C && pp < P) ? src[static_cast<size_t>(c) * P + pp] : 0.f;
  }
  __syncthreads();
  bool ov = false;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int pp = p0 + i, c = c0 + threadIdx.x;
    if (pp < P && c < C) {
      const float s = t[threadIdx.x][i] * scale;
      ov |= fabsf(s) > 60000.f;
      const __half h = __float2half_rn(s);
      const size_t o = (static_cast<size_t>(b) * P + pp) * C + c;
      hi[o] = h;
      lo[o] = __float2half_rn(s - __half2float(h));
    }
  }
  if (ov) atomicOr(status, 1);
}

// rgb fp32 NCHW [B,3,H,W] -> fp16 hi/lo NHWC planes [B,H,W,GEN_BK] (channels 3.. zero): first ResNet conv input
__global__ void rgb_to_planes_kernel(const float* __restrict__ rgb, __half* __restrict__ hi, __half* __restrict__ lo,
                                     int B, int HW, float scale, int* status) {
  const size_t n = static_cast<size_t>(B) * HW;
  bool ov = false;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n * GEN_BK;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % GEN_BK);
    const size_t px = i / GEN_BK;
    float v = 0.f;
    if (c < 3) {
      const size_t b = px / HW, p = px % HW;
      v = rgb[(b * 3 + c) * HW + p] * scale;
    }
    ov |= fabsf(v) > 60000.f;
    const __half h = __float2half_rn(v);
    hi[i] = h;
    lo[i] = __float2half_rn(v - __half2float(h));
  }
  if (ov) atomicOr(status, 1);
}

// F.adaptive_avg_pool2d on fp32 NHWC: in [B,IH,IW,C] -> out [B,OH,OW,C]; window of output i = [floor(i*I/O), ceil((i+1)*I/O))
__global__ void adaptive_avg_pool_nhwc_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int IH, int IW,
                                              int OH, int OW, int C) {
  const size_t n = static_cast<size_t>(B) * OH * OW * C;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % C);
    const size_t px = i / C;
    const int ox = static_cast<int>(px % OW), oy = static_cast<int>((px / OW) % OH), b = static_cast<int>(px / (static_cast<size_t>(OW) * OH));
    const int ys = (oy * IH) / OH, ye = ((oy + 1) * IH + OH - 1) / OH;
    const int xs = (ox * IW) / OW, xe = ((ox + 1) * IW + OW - 1) / OW;
    float s = 0.f;
    for (int y = ys; y < ye; ++y)
      for (int x = xs; x < xe; ++x) s += in[((static_cast<size_t>(b) * IH + y) * IW + x) * C + c];
    out[i] = s / static_cast<float>((ye - ys) * (xe - xs));
  }
}

// w [COUT][CIN][kh][kw] (conv) -> scaled fp16 hi/lo [tap][COUT][CIN] with a per-output-channel factor folded in
// (eval-BatchNorm scale).  transposed=1: w is ConvTranspose2d(k=2,s=2) [CIN][CO][2][2] and becomes a 1-tap
// [4*CO][CIN] matrix, row n = (ky*2+kx)*CO + co.
// cin_pad >= cin: output rows are cin_pad wide (extra input channels must be pre-zeroed by the caller)
__global__ void pack_gen_weight_kernel(const float* __restrict__ w, const float* __restrict__ ch_scale,
                                       __half* __restrict__ hi, __half* __restrict__ lo, int cout, int cin, int taps,
                                       int transposed, float scale, int cin_pad = 0) {
  const int n = cout * cin * taps;
  const int cp = cin_pad > 0 ? cin_pad : cin;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float v, f;
    size_t o;
    if (!transposed) {
      const int tap = i % taps, ci = (i / taps) % cin, co = i / (taps * cin);
      v = w[i];
      f = ch_scale ? ch_scale[co] : 1.f;
      o = (static_cast<size_t>(tap) * cout + co) * cp + ci;
    } else {
      const int co4 = cout / 4;  // here cout = 4*CO, taps == 1, n = cin*CO*4
      const int kk = i % 4, co = (i / 4) % co4, ci = i / (4 * co4);
      v = w[i];
      f = ch_scale ? ch_scale[co] : 1.f;
      o = (static_cast<size_t>(kk) * co4 + co) * cin + ci;
    }
    const float s = v * f * scale;
    const __half h = __float2half_rn(s);
    hi[o] = h;
    lo[o] = __float2half_rn(s - __half2float(h));
  }
}
// max |w * ch_scale[co]| for the power-of-two weight scale (*out zeroed before the launch; see absmax_kernel)
__global__ void absmax_scaled_kernel(const float* __restrict__ w, const float* __restrict__ ch_scale, int n, int per_co,
                                     int co_mod, int transposed, float* __restrict__ out) {
  __shared__ float sm[256];
  float m = 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int co = transposed ? (i / 4) % co_mod : i / per_co;
    const float v = fabsf(w[i] * (ch_scale ? ch_scale[co] : 1.f));
    m = (v > m || v != v) ? v : m;
  }
  sm[threadIdx.x] = m;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      const float o = sm[threadIdx.x + s];
      if (o > sm[threadIdx.x] || o != o) sm[threadIdx.x] = o;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) atomicMax(reinterpret_cast<unsigned int*>(out), __float_as_uint(sm[0]));
}

}  // namespace dd
