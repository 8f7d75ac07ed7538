// Binary-classification metrics (include/b2kmeans.h "binary evaluation"): areaUnderROC or areaUnderPR of M models from
// their scores [M][n] and the label bits pos [n], as Spark's BinaryClassificationMetrics defines them, with the whole
// ordered list of distinct scores taken as one partition.  Per model:
//   keys    k_bin_keys: an order-preserving 64-bit key of each score, inverted so that an ascending sort is descending.
//   sort    CUB radix sort of (key, label bit): the rows in descending score order, NaN first.
//   runs    k_bin_flags, then two integer inclusive scans: run[i] = the distinct scores up to row i, cpos[i] = the
//           positives up to row i.  Exact.
//   points  k_bin_points: the last row of each curve point (a distinct score, or numBins' group of g of them) writes the
//           point's cumulative (true positives, rows) at its index.  Each index has one writer.
//   area    k_bin_area: each CTA sums the trapezoids of a fixed range of the curve's segments and reduces them in a fixed
//           order; k_bin_fold adds the CTAs' partials in CTA order.
// Nothing uses atomics, and the grids depend on n and the device alone: two calls on the same input give the same bits.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <string>
#include <vector>

#include "b2k_internal.cuh"

namespace {

constexpr int BN_NT = 256;

int grid_of(b2k_ctx* ctx, int64_t n) {
  return (int)std::max<int64_t>(1, std::min<int64_t>((n + BN_NT - 1) / BN_NT, 8 * (int64_t)ctx->sm_count));
}

// Java's Double.compare order (-0.0 below +0.0; every NaN one value, above +inf) as an unsigned key, then inverted.
__device__ __forceinline__ unsigned long long desc_key(double v) {
  unsigned long long u = isnan(v) ? 0x7ff8000000000000ull : (unsigned long long)__double_as_longlong(v);
  u = (u >> 63) ? ~u : (u | 0x8000000000000000ull);
  return ~u;
}

__global__ void __launch_bounds__(BN_NT) k_bin_keys(const double* __restrict__ s, int n,
                                                   unsigned long long* __restrict__ key) {
  for (int i = blockIdx.x * BN_NT + threadIdx.x; i < n; i += gridDim.x * BN_NT) key[i] = desc_key(s[i]);
}

// start[i] = 1 where sorted row i begins a run of equal keys; lab[i] = its label bit (int, for the scan).
__global__ void __launch_bounds__(BN_NT) k_bin_flags(const unsigned long long* __restrict__ key,
                                                    const uint8_t* __restrict__ pos, int n, int* __restrict__ start,
                                                    int* __restrict__ lab) {
  for (int i = blockIdx.x * BN_NT + threadIdx.x; i < n; i += gridDim.x * BN_NT) {
    start[i] = i == 0 || key[i] != key[i - 1];
    lab[i] = pos[i];
  }
}

// Distinct scores per point: numBins' grouping g = D / num_bins when that is >= 2, else 1 (no down-sampling).
__device__ __forceinline__ int group_size(int D, int num_bins) {
  const int g = num_bins > 0 ? D / num_bins : 0;
  return g >= 2 ? g : 1;
}

__global__ void __launch_bounds__(BN_NT) k_bin_points(const int* __restrict__ run, const int* __restrict__ cpos, int n,
                                                     int num_bins, int* __restrict__ tp, int* __restrict__ rows) {
  const int g = group_size(run[n - 1], num_bins);
  for (int i = blockIdx.x * BN_NT + threadIdx.x; i < n; i += gridDim.x * BN_NT) {
    const int p = (run[i] - 1) / g;
    if (i == n - 1 || (run[i + 1] - 1) / g != p) {
      tp[p] = cpos[i];
      rows[p] = i + 1;
    }
  }
}

// The curve's points: ROC (0, 0), (FPR, TPR) per point, (1, 1); PR (0, precision of the first point), (recall,
// precision) per point.  FPR = FP / N (0 when N = 0), TPR = recall = TP / P (0 when P = 0), precision = TP / (TP + FP)
// (1 when TP + FP = 0), as Spark's FalsePositiveRate, Recall and Precision.
struct Curve {
  const int* tp;
  const int* rows;
  int np;
  double P, N;
  bool roc;
  __device__ __forceinline__ double2 at(int j) const {
    if (roc && j == np + 1) return make_double2(1.0, 1.0);
    if (roc && j == 0) return make_double2(0.0, 0.0);
    const int p = j == 0 ? 0 : j - 1;
    const double t = tp[p], f = rows[p] - tp[p];
    const double recall = P == 0.0 ? 0.0 : t / P;
    if (roc) return make_double2(N == 0.0 ? 0.0 : f / N, recall);
    const double prec = t + f == 0.0 ? 1.0 : t / (t + f);
    return make_double2(j == 0 ? 0.0 : recall, prec);
  }
};

// part[blockIdx.x] = the sum of the trapezoids (x1 - x0) (y1 + y0) / 2 of segments [s0, s1) of this CTA.
__global__ void __launch_bounds__(BN_NT) k_bin_area(const int* __restrict__ run, const int* __restrict__ cpos, int n,
                                                   int num_bins, int roc, const int* __restrict__ tp,
                                                   const int* __restrict__ rows, double* __restrict__ part) {
  __shared__ double red[BN_NT];
  const int D = run[n - 1], g = group_size(D, num_bins);
  const double P = cpos[n - 1];
  const Curve c{tp, rows, (D + g - 1) / g, P, (double)n - P, roc != 0};
  const int64_t segs = c.np + (roc ? 1 : 0), per = (segs + gridDim.x - 1) / gridDim.x;
  const int64_t s0 = min(segs, per * blockIdx.x), s1 = min(segs, s0 + per);
  double acc = 0.0;
  for (int64_t j = s0 + threadIdx.x; j < s1; j += BN_NT) {
    const double2 a = c.at((int)j), b = c.at((int)j + 1);
    acc += (b.x - a.x) * (b.y + a.y) / 2.0;
  }
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int o = BN_NT / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) part[blockIdx.x] = red[0];
}

// out[mi] = the partials of model mi in CTA order
__global__ void k_bin_fold(const double* __restrict__ part, int P, int m, double* __restrict__ out) {
  const int mi = blockIdx.x * blockDim.x + threadIdx.x;
  if (mi >= m) return;
  double t = 0.0;
  for (int s = 0; s < P; ++s) t += part[(size_t)mi * P + s];
  out[mi] = t;
}

}  // namespace

int b2k_eval_binary_impl(b2k_ctx* ctx, const double* scores, const uint8_t* pos, int64_t n, int m, int num_bins,
                         int metric, double* out, cudaStream_t s) {
  if (n < 1) return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_eval_binary: the metrics need at least one row");
  if (n > INT32_MAX)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "b2k_eval_binary supports at most 2^31 - 1 rows, got " +
                                                  std::to_string(n));
  const int ni = (int)n;
  const int grid = grid_of(ctx, n), area_grid = grid_of(ctx, n + 1);
  size_t sort_bytes = 0, scan_bytes = 0;
  B2K_CUDA_OK(ctx, cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (unsigned long long*)nullptr,
                                                   (unsigned long long*)nullptr, (uint8_t*)nullptr, (uint8_t*)nullptr,
                                                   ni, 0, 64, s));
  B2K_CUDA_OK(ctx, cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, (int*)nullptr, (int*)nullptr, ni, s));
  auto layout = [&](B2kLayout& L, unsigned long long** key, unsigned long long** key_s, uint8_t** lab_s, int** start,
                    int** lab, int** run, int** cpos, int** tp, int** rows, double** part, double** folded,
                    void** sort_tmp, void** scan_tmp) {
    *key = L.take<unsigned long long>(n);
    *key_s = L.take<unsigned long long>(n);
    *lab_s = L.take<uint8_t>(n);
    *start = L.take<int>(n);
    *lab = L.take<int>(n);
    *run = L.take<int>(n);
    *cpos = L.take<int>(n);
    *tp = L.take<int>(n);
    *rows = L.take<int>(n);
    *part = L.take<double>((size_t)m * area_grid);
    *folded = L.take<double>(m);
    *sort_tmp = L.take<char>(sort_bytes);
    *scan_tmp = L.take<char>(scan_bytes);
  };
  unsigned long long *key, *key_s;
  uint8_t* lab_s;
  int *start, *lab, *run, *cpos, *tp, *rows;
  double *part, *folded;
  void *sort_tmp, *scan_tmp;
  B2kLayout measure;
  layout(measure, &key, &key_s, &lab_s, &start, &lab, &run, &cpos, &tp, &rows, &part, &folded, &sort_tmp, &scan_tmp);
  DevBuf buf;   // sized by n: held for this call only, not kept in the context's scratch
  char* base = nullptr;
  B2K_TRY(dalloc(ctx, buf, measure.off, s, &base));
  B2kLayout L(base, measure.off);
  layout(L, &key, &key_s, &lab_s, &start, &lab, &run, &cpos, &tp, &rows, &part, &folded, &sort_tmp, &scan_tmp);
  B2K_TRY(L.check(ctx, "binary evaluation"));
  for (int mi = 0; mi < m; ++mi) {
    k_bin_keys<<<grid, BN_NT, 0, s>>>(scores + (size_t)mi * n, ni, key);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    B2K_CUDA_OK(ctx, cub::DeviceRadixSort::SortPairs(sort_tmp, sort_bytes, key, key_s, pos, lab_s, ni, 0, 64, s));
    k_bin_flags<<<grid, BN_NT, 0, s>>>(key_s, lab_s, ni, start, lab);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    B2K_CUDA_OK(ctx, cub::DeviceScan::InclusiveSum(scan_tmp, scan_bytes, start, run, ni, s));
    B2K_CUDA_OK(ctx, cub::DeviceScan::InclusiveSum(scan_tmp, scan_bytes, lab, cpos, ni, s));
    k_bin_points<<<grid, BN_NT, 0, s>>>(run, cpos, ni, num_bins, tp, rows);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    k_bin_area<<<area_grid, BN_NT, 0, s>>>(run, cpos, ni, num_bins, metric == B2K_BINARY_ROC, tp, rows,
                                           part + (size_t)mi * area_grid);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches += 4;
  }
  k_bin_fold<<<(m + 127) / 128, 128, 0, s>>>(part, area_grid, m, folded);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(out, folded, (size_t)m * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  return B2K_OK;
}
