// Definitions shared by the 3x3 convolution kernels (conv_halo.cuh: warpgroup MMA; kernels.cuh: the fp32 CUDA-core
// check path): tile geometry, epilogue modes and launch arguments.
#pragma once
#include "ptx.cuh"

namespace dd {

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
  float split_scale;       // power-of-two scale applied before the fp16 split of the output
  int* status;             // bit0 set if an fp16 operand would overflow
};

}  // namespace dd
