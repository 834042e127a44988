// Definitions shared by the 3x3 convolution kernels (conv_halo.cuh: warpgroup MMA; kernels.cuh: the fp32 CUDA-core
// check path): tile geometry, epilogue modes, launch arguments and the FP8-correction operand planes.
#pragma once
#include <cuda_fp8.h>

#include "ptx.cuh"

namespace dd {

// FP8-correction operand planes (conv_halo.cuh, F8): with s = the tensor's power-of-two pre-scale,
//   hi = fp16(s v),  a8 = e4m3(s v / 4),  l8 = e4m3((s v - hi) * 512)        (saturating conversions)
// |s v| must stay below 4 * 448 for a8 not to saturate: reported through the status word like an fp16 overflow.
constexpr float kF8ActDiv = 0.25f, kF8LoMul = 512.f, kF8ActMax = 4.f * 448.f;
__device__ __forceinline__ uint16_t e4m3x2(float a, float b) {  // low byte = a
  return static_cast<uint16_t>(__nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, __NV_E4M3));
}

constexpr int TILE_H = 8;
constexpr int TILE_W = 16;
constexpr int TILE_M = TILE_H * TILE_W;  // 128

enum EpiMode : int {
  EPI_F32_STATS = 0,  // y fp32 NHWC + per-(tile, group) fp64 sum / sum-of-squares for the consumer GroupNorm
  EPI_SPLIT = 1,      // y -> scaled fp16 hi/lo planes (input of the next conv; no norm in between)
  EPI_F32 = 2         // y fp32 NHWC only
};

struct ConvArgs {
  int B, H, W;
  int tiles_x, tiles_y, num_tiles;
  const float* bias;       // [COUT]
  float acc_scale;         // 1 / (act_scale * weight_scale): undoes the power-of-two operand scaling
  float* y32;              // [B*H*W][COUT]                       (EPI_F32*)
  double* stats_partial;   // [num_tiles][4][2]                   (EPI_F32_STATS)
  __half* out_hi;          // [B*H*W][COUT]                       (EPI_SPLIT)
  __half* out_lo;
  uint8_t* out_a8;         // non-null (EPI_SPLIT): write the e4m3 planes a8 / l8 instead of the fp16 lo plane
  uint8_t* out_l8;
  float split_scale;       // power-of-two scale applied before the fp16 split of the output
  int* status;             // bit0 set if an fp16 operand would overflow
};

}  // namespace dd
