// The batch statistics of every training-mode BatchNorm (codec_train.cuh, producer_train.cuh).  Two passes over the
// pre-BN values u: pass 1 sums u, pass 2 sums d = u - m and d^2 with m = the pass-1 mean rounded to fp32, so the variance
// is a mean of squared deviations (no E[u^2] - mean^2 cancellation when |mean| >> std) and sum d corrects the rounding
// of m.  Each statistics kernel writes fixed fp64 partials per block, laid out [blocks][2][C] (sum d of the C channels,
// then sum d^2), summed in block order: bit-reproducible.  Across ranks (dd_set_bn_allgather) each pass's totals are
// gathered with the local item count and summed in rank order; the kernels then divide by the global count *cnt
// instead of their own n (cnt null: n).
#pragma once

namespace dd {

// out[c] = sum over blocks, in block order, of part[b * stride + c], c < ncols (one thread per column).  count > 0:
// out[ncols] = count as well, the row a cross-rank gather sends (the launch then covers ncols + 1 threads).
__global__ void part_colsum_kernel(const double* __restrict__ part, int nblk, int stride, int ncols,
                                   double* __restrict__ out, long long count) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c == ncols && count > 0) out[c] = static_cast<double>(count);
  if (c >= ncols) return;
  double s = 0.0;
  for (int b = 0; b < nblk; ++b) s += part[static_cast<size_t>(b) * stride + c];
  out[c] = s;
}

// out[j] = rows[0][j] + rows[1][j] + ... + rows[R - 1][j], added in rank order, j < cols: the gathered per-rank totals
// of a cross-rank BatchNorm (count last), so every rank folds the same union-batch statistics, bit for bit.
__global__ void __launch_bounds__(256) bn_rank_sum_kernel(const double* __restrict__ rows, int R, int cols,
                                                          double* __restrict__ out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= cols) return;
  double s = rows[j];
  for (int r = 1; r < R; ++r) s += rows[static_cast<size_t>(r) * cols + j];
  out[j] = s;
}

// What a fold reads: the pass-1 totals sum1 [C], the pass-2 partials part [nblk][2][C] (across ranks the union batch's
// totals, nblk = 1), and the item count N = *cnt, or n when cnt is null.
struct BnFoldIn {
  const double *sum1, *part;
  int nblk;
  long long n;
  const double* cnt;
};

// One channel's batch statistics, as every fold takes them.
struct BnBatchStats {
  double mean;          // batch mean of u: fp32(sum1 / N) + sum d / N
  double var;           // batch variance: sum d^2 / N - (sum d / N)^2, at least 0
  double scale;         // gamma / sqrt(var + 1e-5), the host fold's formula; callers round it to fp32 once
  double var_unbiased;  // N / (N - 1) var (N = 1: var), the record's, which the running update reads
};
__device__ __forceinline__ BnBatchStats bn_batch_stats(const BnFoldIn& in, int C, int c, const float* gamma) {
  double d1 = 0.0, d2 = 0.0;
  for (int b = 0; b < in.nblk; ++b) {
    d1 += in.part[(static_cast<size_t>(b) * 2) * C + c];
    d2 += in.part[(static_cast<size_t>(b) * 2 + 1) * C + c];
  }
  const double nn = in.cnt ? *in.cnt : static_cast<double>(in.n);
  const double dm = d1 / nn;  // mean of d: the rounding of the shift
  BnBatchStats r;
  r.mean = static_cast<double>(static_cast<float>(in.sum1[c] / nn)) + dm;
  r.var = fmax(d2 / nn - dm * dm, 0.0);
  r.scale = static_cast<double>(gamma[c]) / sqrt(r.var + 1e-5);
  r.var_unbiased = nn > 1.0 ? r.var * nn / (nn - 1.0) : r.var;
  return r;
}

}  // namespace dd
