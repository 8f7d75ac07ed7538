// UMAP (sm_90a): b2k_umap_fit and b2k_umap_transform, Euclidean, float32 rows, on one GPU with no collective.
//
//   kNN       b2k_knn_local_impl (b2k_knn.cu's plan, prep, search and refine, without its allgathers).
//   membership k_umap_membership: one thread per row (the bisection is sequential), fp64: rho by local_connectivity, sigma by bisection, the weights.
//   graph     the directed weights as COO keys ((i, j) << 1 | transposed), CUB radix sort, k_umap_combine folds each
//             (i, j) with its transpose into the fuzzy union / intersection mix, a scan compacts the non-zero entries
//             into a CSR with sorted columns.  Supervised: k_umap_labels scales by label agreement and rescales each
//             row to max 1, and the graph is built again as a fuzzy union.
//   schedule  k_umap_schedule: epochs_per_sample = max(w) / w (+inf for a dropped edge), fp64 state per edge.
//   init      random (host, from umap_hash) or spectral (k_umap_spmm + host subspace iteration), then each column
//             rescaled to [0, 10].
//   layout    one launch per epoch, one warp per vertex over its CSR row, reading the positions of the start of the
//             epoch and writing the other buffer: lane-parallel edges for n_components <= 4 (the sums in registers,
//             then a butterfly), lanes over components otherwise.
//   transform k_umap_transform: one warp per query, memberships, the weighted-mean start and every epoch in-kernel.
// Nothing uses atomics: two calls with the same input and seed are bitwise equal, whatever grid_limit is.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cmath>
#include <numeric>
#include <vector>

#include "b2k_internal.cuh"

namespace {

constexpr int U_WARPS = 4;           // warps per block of the per-row kernels
constexpr int U_SMALL_C = 4;         // widths of the lane-parallel-edge layout path
constexpr int SMOOTH_K_ITERS = 64;
constexpr double SMOOTH_K_TOL = 1e-5;
constexpr double MIN_K_DIST_SCALE = 1e-3;

__host__ __device__ __forceinline__ uint64_t umap_mix(uint64_t z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__host__ __device__ __forceinline__ uint64_t umap_hash(uint64_t seed, uint64_t a, uint64_t b, uint64_t c) {
  return umap_mix(umap_mix(umap_mix(umap_mix(seed + 0x9E3779B97F4A7C15ull) ^ a) ^ b) ^ c);
}
__host__ __device__ __forceinline__ double umap_unit(uint64_t h) { return (double)(h >> 11) * 0x1.0p-53; }

// ---- memberships ----
// rho, sigma and w for one row of k (dist, idx) in list order, as tests/umap_oracle.py restates it; self = the row's own
// index (-1: none), whose edge has weight 0 and which the bisection's sum leaves out.  The sigma floor is 1e-3 of the
// row's mean distance when rho > 0 or use_row_mean, else of mean_floor (the mean over every row).
__device__ __forceinline__ void umap_row_membership(const float* dist, const int64_t* idx, int k, int64_t self, double lc,
                                    double mean_floor, bool use_row_mean, double* rho_out, double* sigma_out,
                                    double* w) {
  double rho = 0.0;
  int nz = 0;
  for (int j = 0; j < k; ++j) nz += (double)dist[j] > 0.0;
  const int index = (int)floor(lc);
  const double interp = lc - (double)index;
  if (nz >= lc) {
    // the index-th and (index + 1)-th non-zero distances, in list order
    double prev = 0.0, at = 0.0;
    int c = 0;
    for (int j = 0; j < k; ++j) {
      const double v = (double)dist[j];
      if (v > 0.0) {
        ++c;
        if (c == index) prev = v;
        if (c == index + 1) at = v;
      }
    }
    if (index > 0) {
      rho = prev;
      if (interp > SMOOTH_K_TOL) rho += interp * (at - prev);
    } else {
      rho = interp * at;
    }
  } else if (nz > 0) {
    for (int j = 0; j < k; ++j) rho = fmax(rho, (double)dist[j]);
  }
  const double target = log2((double)k);
  double lo = 0.0, hi = INFINITY, mid = 1.0;
  for (int it = 0; it < SMOOTH_K_ITERS; ++it) {
    double psum = 0.0;
    for (int j = 0; j < k; ++j) {
      if (idx[j] == self) continue;
      const double dd = (double)dist[j] - rho;
      psum += dd > 0.0 ? exp(-(dd / mid)) : 1.0;
    }
    if (fabs(psum - target) < SMOOTH_K_TOL) break;
    if (psum > target) {
      hi = mid;
      mid = (lo + hi) / 2.0;
    } else {
      lo = mid;
      mid = hi == INFINITY ? mid * 2.0 : (lo + hi) / 2.0;
    }
  }
  double row_mean = 0.0;
  for (int j = 0; j < k; ++j) row_mean += (double)dist[j];
  row_mean /= (double)k;
  const double floor_v = MIN_K_DIST_SCALE * (rho > 0.0 || use_row_mean ? row_mean : mean_floor);
  if (mid < floor_v) mid = floor_v;
  *rho_out = rho;
  *sigma_out = mid;
  for (int j = 0; j < k; ++j) {
    const double dd = (double)dist[j] - rho;
    w[j] = idx[j] == self ? 0.0 : (dd <= 0.0 || mid == 0.0) ? 1.0 : exp(-(dd / mid));
  }
}

__global__ void __launch_bounds__(256) k_umap_row_sums(const float* __restrict__ dist, int64_t n, int k,
                                                       double* __restrict__ sums) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    double s = 0.0;
    for (int j = 0; j < k; ++j) s += (double)dist[i * k + j];
    sums[i] = s;
  }
}

__global__ void __launch_bounds__(128) k_umap_membership(const float* __restrict__ dist, const int64_t* __restrict__ idx,
                                                         int64_t n, int k, double lc, double mean_all,
                                                         double* __restrict__ rho, double* __restrict__ sigma,
                                                         double* __restrict__ P) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    umap_row_membership(dist + i * k, idx + i * k, k, i, lc, mean_all, false, rho + i, sigma + i, P + i * k);
}

// ---- graph ----
// COO -> keys ((row << 32 | col) << 1 | t): t = 0 is w_ij at (i, j), t = 1 its transpose at (j, i)
__global__ void __launch_bounds__(256) k_umap_coo_keys(const int64_t* __restrict__ rows, int64_t rows_per,
                                                       const int64_t* __restrict__ cols, const double* __restrict__ vals,
                                                       int64_t m, uint64_t* __restrict__ keys,
                                                       double* __restrict__ kv) {
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < m; e += (int64_t)gridDim.x * blockDim.x) {
    const uint64_t i = rows ? (uint64_t)rows[e] : (uint64_t)(e / rows_per);
    const uint64_t j = (uint64_t)cols[e];
    keys[2 * e] = ((i << 32) | j) << 1;
    keys[2 * e + 1] = (((j << 32) | i) << 1) | 1u;
    kv[2 * e] = vals[e];
    kv[2 * e + 1] = vals[e];
  }
}

// per sorted key: w of its (i, j) at the pair's first key, 0 elsewhere; keep = w > 0
__global__ void __launch_bounds__(256) k_umap_combine(const uint64_t* __restrict__ keys, const double* __restrict__ kv,
                                                      int64_t m, double mix, double* __restrict__ w,
                                                      int* __restrict__ keep) {
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < m; e += (int64_t)gridDim.x * blockDim.x) {
    const uint64_t pk = keys[e] >> 1;
    double v = 0.0;
    if (e == 0 || (keys[e - 1] >> 1) != pk) {
      double a = 0.0, b = 0.0;
      (keys[e] & 1u ? b : a) = kv[e];
      if (e + 1 < m && (keys[e + 1] >> 1) == pk) (keys[e + 1] & 1u ? b : a) = kv[e + 1];
      const double ab = a * b;
      v = mix * (a + b - ab) + (1.0 - mix) * ab;
    }
    w[e] = v;
    keep[e] = v > 0.0;
  }
}

__global__ void __launch_bounds__(256) k_umap_compact(const uint64_t* __restrict__ keys, const double* __restrict__ w,
                                                      const int* __restrict__ keep, const int* __restrict__ pos,
                                                      int64_t m, int64_t* __restrict__ rows,
                                                      int32_t* __restrict__ cols, double* __restrict__ vals) {
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < m; e += (int64_t)gridDim.x * blockDim.x) {
    if (!keep[e]) continue;
    const uint64_t pk = keys[e] >> 1;
    rows[pos[e]] = (int64_t)(pk >> 32);
    cols[pos[e]] = (int32_t)(pk & 0xffffffffu);
    vals[pos[e]] = w[e];
  }
}

// indptr[r] = first entry of row >= r (binary search of the sorted rows)
__global__ void __launch_bounds__(256) k_umap_indptr(const int64_t* __restrict__ rows, int64_t nnz, int64_t n,
                                                     int64_t* __restrict__ indptr) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r <= n; r += (int64_t)gridDim.x * blockDim.x) {
    int64_t lo = 0, hi = nnz;
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (rows[mid] < r) lo = mid + 1;
      else hi = mid;
    }
    indptr[r] = lo;
  }
}

// supervised: w *= exp(-1) for an unknown label (-1) at either end, exp(-5) for two different labels; then each row
// divided by its largest weight.  Writes the COO (row, col, value) of the next fuzzy union.
__global__ void __launch_bounds__(U_WARPS * 32) k_umap_labels(const int64_t* __restrict__ indptr,
                                                              const int32_t* __restrict__ cols,
                                                              const double* __restrict__ vals,
                                                              const int32_t* __restrict__ labels, int64_t n,
                                                              int64_t* __restrict__ rows_out,
                                                              int64_t* __restrict__ cols_out,
                                                              double* __restrict__ vals_out) {
  const int lane = threadIdx.x & 31;
  for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n;
       i += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    const int32_t li = labels[i];
    double mx = 0.0;
    for (int64_t p = indptr[i] + lane; p < indptr[i + 1]; p += 32) {
      const int32_t lj = labels[cols[p]];
      const double f = (li == -1 || lj == -1) ? exp(-1.0) : li != lj ? exp(-5.0) : 1.0;
      const double v = vals[p] * f;
      vals_out[p] = v;
      mx = fmax(mx, v);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    for (int64_t p = indptr[i] + lane; p < indptr[i + 1]; p += 32) {
      vals_out[p] = vals_out[p] / mx;
      rows_out[p] = i;
      cols_out[p] = cols[p];
    }
  }
}

// ---- schedule ----
__global__ void __launch_bounds__(256) k_umap_schedule(const double* __restrict__ w, int64_t nnz, double wmax,
                                                       int n_epochs, int neg_rate, double* __restrict__ eps,
                                                       double* __restrict__ next, double* __restrict__ next_neg,
                                                       double* __restrict__ epn) {
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += (int64_t)gridDim.x * blockDim.x) {
    const double s = w[e] < wmax / (double)n_epochs ? INFINITY : wmax / w[e];
    eps[e] = s;
    next[e] = s;
    epn[e] = s / (double)neg_rate;
    next_neg[e] = s / (double)neg_rate;
  }
}

// ---- the layout's per-edge arithmetic (umap-learn's optimize_layout_euclidean) ----
struct UmapCoef {
  float a, b, gamma;
};
__device__ __forceinline__ float clip4(float v) { return fminf(fmaxf(v, -4.f), 4.f); }
__device__ __forceinline__ float attr_coef(float d2, const UmapCoef& k) {
  if (!(d2 > 0.f)) return 0.f;
  return (-2.f * k.a * k.b * powf(d2, k.b - 1.f)) / (k.a * powf(d2, k.b) + 1.f);
}
// 0 when d2 == 0: the callers then move each component by 4, branching on d2 itself
__device__ __forceinline__ float rep_coef(float d2, const UmapCoef& k) {
  if (!(d2 > 0.f)) return 0.f;
  return (2.f * k.gamma * k.b) / ((0.001f + d2) * (k.a * powf(d2, k.b) + 1.f));
}
// negatives drawn by a due edge at epoch e: the edge's schedule advanced in place (the caller owns the edge)
__device__ __forceinline__ int due_negatives(double* next, double* next_neg, const double* eps, const double* epn,
                                             int64_t p, int e) {
  next[p] += eps[p];
  const int nneg = max(0, (int)(((double)e - next_neg[p]) / epn[p]));
  next_neg[p] += (double)nneg * epn[p];
  return nneg;
}

struct LayoutArgs {
  const int64_t* indptr;
  const int32_t* cols;
  const double* eps;
  const double* epn;
  double* next;
  double* next_neg;
  const float* Y;   // positions at the start of the epoch [n][C]
  float* Yn;        // positions after it
  int64_t n;
  int e;
  float alpha;
  UmapCoef k;
  uint64_t seed;
};

// n_components = C <= 4: lane-parallel edges, sums in registers, a butterfly across the warp
template <int C>
__global__ void __launch_bounds__(U_WARPS * 32) k_umap_layout_small(LayoutArgs a) {
  const int lane = threadIdx.x & 31;
  for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < a.n;
       i += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    float yi[C], acc[C];
#pragma unroll
    for (int c = 0; c < C; ++c) {
      yi[c] = a.Y[i * C + c];
      acc[c] = 0.f;
    }
    for (int64_t p = a.indptr[i] + lane; p < a.indptr[i + 1]; p += 32) {
      if (!(a.next[p] <= (double)a.e)) continue;
      const int64_t j = a.cols[p];
      float yj[C], d2 = 0.f;
#pragma unroll
      for (int c = 0; c < C; ++c) {
        yj[c] = a.Y[j * C + c];
        const float df = yi[c] - yj[c];
        d2 += df * df;
      }
      const float ga = attr_coef(d2, a.k);
      // the edge moves i as its head, and its transpose (j, i), due in the same epoch, moves i as its tail by as much
#pragma unroll
      for (int c = 0; c < C; ++c) acc[c] += 2.f * clip4(ga * (yi[c] - yj[c]));
      const int nneg = due_negatives(a.next, a.next_neg, a.eps, a.epn, p, a.e);
      for (int q = 0; q < nneg; ++q) {
        const int64_t kk = (int64_t)(umap_hash(a.seed, (uint64_t)a.e, (uint64_t)p, (uint64_t)q) % (uint64_t)a.n);
        if (kk == i) continue;
        float yk[C], r2 = 0.f;
#pragma unroll
        for (int c = 0; c < C; ++c) {
          yk[c] = a.Y[kk * C + c];
          const float df = yi[c] - yk[c];
          r2 += df * df;
        }
        const float gr = rep_coef(r2, a.k);
#pragma unroll
        for (int c = 0; c < C; ++c) acc[c] += r2 > 0.f ? clip4(gr * (yi[c] - yk[c])) : 4.f;
      }
    }
#pragma unroll
    for (int c = 0; c < C; ++c) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], o);
    }
    if (lane < C) {
      float v = 0.f, y = 0.f;
#pragma unroll
      for (int c = 0; c < C; ++c)
        if (c == lane) v = acc[c], y = yi[c];
      a.Yn[i * C + lane] = y + a.alpha * v;
    }
  }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// any n_components <= 128: lanes over components (component lane + 32 t), the row's edges in order
__global__ void __launch_bounds__(U_WARPS * 32) k_umap_layout_wide(LayoutArgs a, int C) {
  const int lane = threadIdx.x & 31;
  for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < a.n;
       i += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    float yi[4], acc[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int c = lane + 32 * t;
      yi[t] = c < C ? a.Y[i * C + c] : 0.f;
      acc[t] = 0.f;
    }
    for (int64_t p = a.indptr[i]; p < a.indptr[i + 1]; ++p) {
      if (!(a.next[p] <= (double)a.e)) continue;
      const int64_t j = a.cols[p];
      float yj[4], d2 = 0.f;
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const int c = lane + 32 * t;
        yj[t] = c < C ? a.Y[j * C + c] : 0.f;
        d2 += (yi[t] - yj[t]) * (yi[t] - yj[t]);
      }
      d2 = warp_sum(d2);
      const float ga = attr_coef(d2, a.k);
#pragma unroll
      for (int t = 0; t < 4; ++t) acc[t] += 2.f * clip4(ga * (yi[t] - yj[t]));
      __syncwarp();
      int nneg = 0;
      if (lane == 0) nneg = due_negatives(a.next, a.next_neg, a.eps, a.epn, p, a.e);
      nneg = __shfl_sync(0xffffffffu, nneg, 0);
      for (int q = 0; q < nneg; ++q) {
        const int64_t kk = (int64_t)(umap_hash(a.seed, (uint64_t)a.e, (uint64_t)p, (uint64_t)q) % (uint64_t)a.n);
        if (kk == i) continue;
        float yk[4], r2 = 0.f;
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const int c = lane + 32 * t;
          yk[t] = c < C ? a.Y[kk * C + c] : 0.f;
          r2 += (yi[t] - yk[t]) * (yi[t] - yk[t]);
        }
        r2 = warp_sum(r2);
        const float gr = rep_coef(r2, a.k);
#pragma unroll
        for (int t = 0; t < 4; ++t) acc[t] += r2 > 0.f ? clip4(gr * (yi[t] - yk[t])) : 4.f;
      }
    }
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int c = lane + 32 * t;
      if (c < C) a.Yn[i * C + c] = yi[t] + a.alpha * acc[t];
    }
  }
}

// ---- spectral init: Z = (M Y + Y) / 2 with M = D^-1/2 W D^-1/2, fp64, one warp per row, lanes over columns ----
__global__ void __launch_bounds__(U_WARPS * 32) k_umap_spmm(const int64_t* __restrict__ indptr,
                                                            const int32_t* __restrict__ cols,
                                                            const double* __restrict__ w,
                                                            const double* __restrict__ dinv, const double* __restrict__ Y,
                                                            int64_t n, int m, double* __restrict__ Z) {
  const int lane = threadIdx.x & 31;
  for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n;
       i += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    for (int c0 = 0; c0 < m; c0 += 32) {
      const int c = c0 + lane;
      double s = 0.0;
      for (int64_t p = indptr[i]; p < indptr[i + 1]; ++p)
        if (c < m) s += w[p] * dinv[cols[p]] * Y[(int64_t)cols[p] * m + c];
      if (c < m) Z[i * m + c] = 0.5 * (dinv[i] * s + Y[i * m + c]);
    }
  }
}

// ---- transform: one warp per query, lanes over components; edge state in shared memory ----
struct TransformArgs {
  const float* Yt;       // training embedding [n_train][C]
  const float* dist;     // [nq][k]
  const int64_t* idx;    // [nq][k]
  const float* Q;        // [nq][d] (finiteness only)
  float* out;            // [nq][C]
  int64_t nq, n_train;
  int k, d, C, n_epochs, neg_rate;
  double lc;
  float lr;
  UmapCoef kc;
  uint64_t seed;
};

__global__ void __launch_bounds__(U_WARPS * 32) k_umap_transform(TransformArgs a) {
  extern __shared__ double sm[];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  double* wt = sm + (size_t)w * 5 * a.k;   // weight, eps, epn, next, next_neg per edge
  double* eps = wt + a.k;
  double* epn = eps + a.k;
  double* next = epn + a.k;
  double* nneg_at = next + a.k;
  for (int64_t q = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; q < a.nq;
       q += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    const float* dq = a.dist + q * a.k;
    const int64_t* iq = a.idx + q * a.k;
    bool bad = false;
    for (int f = lane; f < a.d; f += 32) bad |= !isfinite(a.Q[q * a.d + f]);
    bad = __any_sync(0xffffffffu, bad);
    if (bad) {
      for (int c = lane; c < a.C; c += 32) a.out[q * a.C + c] = __int_as_float(0x7fc00000);
      continue;
    }
    if (lane == 0) {
      double rho, sigma;
      umap_row_membership(dq, iq, a.k, -1, a.lc, 0.0, true, &rho, &sigma, wt);
      double wmax = 0.0;
      for (int j = 0; j < a.k; ++j) wmax = fmax(wmax, wt[j]);
      for (int j = 0; j < a.k; ++j) {
        const double s = wt[j] < wmax / (double)max(a.n_epochs, 1) ? INFINITY : wmax / wt[j];
        eps[j] = s;
        next[j] = s;
        epn[j] = a.neg_rate > 0 ? s / (double)a.neg_rate : INFINITY;
        nneg_at[j] = epn[j];
      }
    }
    __syncwarp();
    // start: the weight-normalised mean of the neighbours' embeddings, in fp64, neighbour order
    float yi[4];
    double wsum = 0.0;
    for (int j = 0; j < a.k; ++j) wsum += wt[j];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int c = lane + 32 * t;
      double s = 0.0;
      if (c < a.C)
        for (int j = 0; j < a.k; ++j) s += wt[j] * (double)a.Yt[iq[j] * a.C + c];
      yi[t] = c < a.C ? (float)(s / wsum) : 0.f;
    }
    const uint64_t key0 = (uint64_t)iq[0] * (uint64_t)a.n_train;
    for (int e = 0; e < a.n_epochs; ++e) {
      const float alpha = (float)((double)a.lr * (1.0 - (double)e / (double)a.n_epochs));
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
      for (int j = 0; j < a.k; ++j) {
        if (!(next[j] <= (double)e)) continue;
        const int64_t tj = iq[j];
        float yj[4], d2 = 0.f;
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const int c = lane + 32 * t;
          yj[t] = c < a.C ? a.Yt[tj * a.C + c] : 0.f;
          d2 += (yi[t] - yj[t]) * (yi[t] - yj[t]);
        }
        d2 = warp_sum(d2);
        const float ga = attr_coef(d2, a.kc);
#pragma unroll
        for (int t = 0; t < 4; ++t) acc[t] += clip4(ga * (yi[t] - yj[t]));
        __syncwarp();
        int nneg = 0;
        if (lane == 0) nneg = due_negatives(next, nneg_at, eps, epn, j, e);
        __syncwarp();
        nneg = __shfl_sync(0xffffffffu, nneg, 0);
        for (int r = 0; r < nneg; ++r) {
          const int64_t kk = (int64_t)(umap_hash(a.seed, (uint64_t)e, key0 + (uint64_t)tj, (uint64_t)r) %
                                       (uint64_t)a.n_train);
          float yk[4], r2 = 0.f;
#pragma unroll
          for (int t = 0; t < 4; ++t) {
            const int c = lane + 32 * t;
            yk[t] = c < a.C ? a.Yt[kk * a.C + c] : 0.f;
            r2 += (yi[t] - yk[t]) * (yi[t] - yk[t]);
          }
          r2 = warp_sum(r2);
          const float gr = rep_coef(r2, a.kc);
#pragma unroll
          for (int t = 0; t < 4; ++t) acc[t] += r2 > 0.f ? clip4(gr * (yi[t] - yk[t])) : 4.f;
        }
      }
#pragma unroll
      for (int t = 0; t < 4; ++t) yi[t] += alpha * acc[t];
    }
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int c = lane + 32 * t;
      if (c < a.C) a.out[q * a.C + c] = yi[t];
    }
    __syncwarp();
  }
}

__global__ void __launch_bounds__(256) k_umap_count_bad(const float* __restrict__ X, int64_t m,
                                                        int64_t* __restrict__ part) {
  int64_t c = 0;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < m; e += (int64_t)gridDim.x * blockDim.x)
    c += !isfinite(X[e]);
  __shared__ int64_t s[256];
  s[threadIdx.x] = c;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) part[blockIdx.x] = s[0];
}

// the last fit's graph and init, read back by b2k_umap_graph
struct UmapGraph {
  int64_t n = 0, k = 0, nnz = 0;
  int C = 0;
  std::vector<int64_t> knn_idx, indptr;
  std::vector<float> knn_dist, init;
  std::vector<int32_t> indices;
  std::vector<double> weights, eps, rho, sigma, ritz_values, ritz_vectors;
};

unsigned grid_for(const b2k_ctx* ctx, int64_t work, int per_block) {
  int64_t g = (work + per_block - 1) / per_block;
  int cap = ctx->sm_count * 16;
  if (ctx->grid_limit > 0) cap = std::min(cap, ctx->grid_limit);
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>(g, cap));
}

struct Events {
  cudaEvent_t ev[5] = {};
  Events() {
    for (auto& e : ev) cudaEventCreate(&e);
  }
  ~Events() {
    for (auto& e : ev) cudaEventDestroy(e);
  }
  double ms(int a, int b) const {
    float t = 0.f;
    cudaEventElapsedTime(&t, ev[a], ev[b]);
    return (double)t;
  }
};

// COO (rows, or row = e / rows_per when rows is NULL; cols; vals) of m entries -> sorted CSR of the mix of each (i, j)
// with its transpose, zeros dropped.  The CSR arrays are cudaMalloc'd here and owned by the caller's vectors of
// device pointers (freed by the caller).
struct DevCsr {
  int64_t* indptr = nullptr;
  int64_t* rows = nullptr;
  int32_t* cols = nullptr;
  double* vals = nullptr;
  int64_t nnz = 0;
  void release() {
    cudaFree(indptr);
    cudaFree(rows);
    cudaFree(cols);
    cudaFree(vals);
    *this = DevCsr();
  }
};

int symmetrise(b2k_ctx* ctx, const int64_t* rows, int64_t rows_per, const int64_t* cols, const double* vals, int64_t m,
               int64_t n, double mix, DevCsr* out, cudaStream_t s) {
  const int64_t m2 = 2 * m;
  uint64_t *keys = nullptr, *keys_s = nullptr;
  double *kv = nullptr, *kv_s = nullptr, *w = nullptr;
  int *keep = nullptr, *pos = nullptr;
  size_t sort_bytes = 0, scan_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, keys, keys_s, kv, kv_s, m2, 0, 64, s);
  cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, keep, pos, m2, s);
  char* tmp = nullptr;
  B2K_TRY(b2k_scratch_layout(ctx, "UMAP graph", [&](B2kLayout& L) -> int {
    keys = L.take<uint64_t>(m2);
    keys_s = L.take<uint64_t>(m2);
    kv = L.take<double>(m2);
    kv_s = L.take<double>(m2);
    w = L.take<double>(m2);
    keep = L.take<int>(m2 + 1);
    pos = L.take<int>(m2 + 1);
    tmp = L.take<char>(std::max(sort_bytes, scan_bytes));
    return B2K_OK;
  }));
  const unsigned g = grid_for(ctx, m2, 256);
  k_umap_coo_keys<<<g, 256, 0, s>>>(rows, rows_per, cols, vals, m, keys, kv);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  B2K_CUDA_OK(ctx, cub::DeviceRadixSort::SortPairs(tmp, sort_bytes, keys, keys_s, kv, kv_s, m2, 0, 64, s));
  k_umap_combine<<<g, 256, 0, s>>>(keys_s, kv_s, m2, mix, w, keep);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  B2K_CUDA_OK(ctx, cudaMemsetAsync(keep + m2, 0, sizeof(int), s));
  B2K_CUDA_OK(ctx, cub::DeviceScan::ExclusiveSum(tmp, scan_bytes, keep, pos, m2 + 1, s));
  int nnz = 0;
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(&nnz, pos + m2, sizeof(int), cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  out->release();
  out->nnz = nnz;
  B2K_CUDA_OK(ctx, cudaMalloc(&out->indptr, (size_t)(n + 1) * 8));
  B2K_CUDA_OK(ctx, cudaMalloc(&out->rows, (size_t)std::max(nnz, 1) * 8));
  B2K_CUDA_OK(ctx, cudaMalloc(&out->cols, (size_t)std::max(nnz, 1) * 4));
  B2K_CUDA_OK(ctx, cudaMalloc(&out->vals, (size_t)std::max(nnz, 1) * 8));
  k_umap_compact<<<g, 256, 0, s>>>(keys_s, w, keep, pos, m2, out->rows, out->cols, out->vals);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  k_umap_indptr<<<grid_for(ctx, n + 1, 256), 256, 0, s>>>(out->rows, nnz, n, out->indptr);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches += 6;
  return B2K_OK;
}

int check_params(b2k_ctx* ctx, const char* who, const b2k_umap_params& p, int64_t n_items) {
  auto bad = [&](const std::string& m) { return b2k_fail(ctx, B2K_ERR_INVALID, std::string(who) + ": " + m); };
  if (p.n_neighbors < 1 || p.n_neighbors > n_items || p.n_neighbors > B2K_KNN_MAX_K)
    return bad("n_neighbors = " + std::to_string(p.n_neighbors) + " must be in [1, min(rows, 1024)]");
  if (p.n_components < 1 || p.n_components > 100)
    return bad("n_components = " + std::to_string(p.n_components) + " must be in [1, 100]");
  if (p.negative_sample_rate < 0) return bad("negative_sample_rate must be >= 0");
  if (!(p.local_connectivity >= 0.0) || !std::isfinite(p.local_connectivity))
    return bad("local_connectivity must be finite and >= 0");
  if (!(p.set_op_mix_ratio >= 0.0 && p.set_op_mix_ratio <= 1.0)) return bad("set_op_mix_ratio must be in [0, 1]");
  if (!std::isfinite(p.learning_rate) || !std::isfinite(p.repulsion_strength) || !(p.a > 0.0) || !(p.b > 0.0) ||
      !std::isfinite(p.a) || !std::isfinite(p.b))
    return bad("learning_rate, repulsion_strength, a and b must be finite, a and b > 0");
  return B2K_OK;
}

int count_bad(b2k_ctx* ctx, const float* X, int64_t m, int64_t* out, cudaStream_t s) {
  int64_t* part = nullptr;
  const unsigned g = grid_for(ctx, m, 256);
  B2K_TRY(b2k_scratch_layout(ctx, "UMAP input check", [&](B2kLayout& L) -> int {
    part = L.take<int64_t>(g);
    return B2K_OK;
  }));
  k_umap_count_bad<<<g, 256, 0, s>>>(X, m, part);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  std::vector<int64_t> h(g);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(h.data(), part, g * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  *out = std::accumulate(h.begin(), h.end(), (int64_t)0);
  ctx->stats.kernel_launches++;
  return B2K_OK;
}

// orthonormalise the m columns of Y [n][m] in place (modified Gram-Schmidt, twice), after removing v0
void orthonormalise(std::vector<double>& Y, int64_t n, int m, const std::vector<double>& v0) {
  for (int pass = 0; pass < 2; ++pass)
    for (int c = 0; c < m; ++c) {
      double dv = 0.0;
      for (int64_t i = 0; i < n; ++i) dv += v0[i] * Y[i * m + c];
      for (int64_t i = 0; i < n; ++i) Y[i * m + c] -= dv * v0[i];
      for (int c2 = 0; c2 < c; ++c2) {
        double dp = 0.0;
        for (int64_t i = 0; i < n; ++i) dp += Y[i * m + c2] * Y[i * m + c];
        for (int64_t i = 0; i < n; ++i) Y[i * m + c] -= dp * Y[i * m + c2];
      }
      double nn = 0.0;
      for (int64_t i = 0; i < n; ++i) nn += Y[i * m + c] * Y[i * m + c];
      nn = nn > 0.0 ? 1.0 / std::sqrt(nn) : 0.0;
      for (int64_t i = 0; i < n; ++i) Y[i * m + c] *= nn;
    }
}

int components(const std::vector<int64_t>& indptr, const std::vector<int32_t>& cols, int64_t n) {
  std::vector<int64_t> parent(n);
  std::iota(parent.begin(), parent.end(), 0);
  auto find = [&](int64_t x) {
    while (parent[x] != x) x = parent[x] = parent[parent[x]];
    return x;
  };
  for (int64_t i = 0; i < n; ++i)
    for (int64_t p = indptr[i]; p < indptr[i + 1]; ++p) {
      const int64_t a = find(i), b = find(cols[p]);
      if (a != b) parent[std::max(a, b)] = std::min(a, b);
    }
  int c = 0;
  for (int64_t i = 0; i < n; ++i) c += find(i) == i;
  return c;
}

constexpr int SPECTRAL_MAX_ITERS = 300;
constexpr double SPECTRAL_TOL = 1e-8;

// The C leading non-trivial eigenvectors of M = D^-1/2 W D^-1/2 by block subspace iteration on (M + I) / 2.
int spectral(b2k_ctx* ctx, const DevCsr& G, const UmapGraph& H, int C, uint64_t seed, std::vector<double>* vec,
             std::vector<double>* val, double* resid, cudaStream_t s) {
  const int64_t n = H.n;
  const int m = (int)std::min<int64_t>(C + 4, n - 1);
  std::vector<double> deg(n, 0.0), dinv(n), v0(n);
  for (int64_t i = 0; i < n; ++i)
    for (int64_t p = H.indptr[i]; p < H.indptr[i + 1]; ++p) deg[i] += H.weights[p];
  double nv0 = 0.0;
  for (int64_t i = 0; i < n; ++i) {
    dinv[i] = 1.0 / std::sqrt(deg[i]);
    v0[i] = std::sqrt(deg[i]);
    nv0 += deg[i];
  }
  for (auto& v : v0) v /= std::sqrt(nv0);
  std::vector<double> Y((size_t)n * m), Z((size_t)n * m);
  for (int64_t i = 0; i < n; ++i)
    for (int c = 0; c < m; ++c) Y[i * m + c] = 2.0 * umap_unit(umap_hash(seed, 1ull << 41, (uint64_t)i, c)) - 1.0;
  orthonormalise(Y, n, m, v0);
  double *dY = nullptr, *dZ = nullptr, *dD = nullptr;
  B2K_TRY(b2k_scratch_layout(ctx, "UMAP spectral", [&](B2kLayout& L) -> int {
    dY = L.take<double>((size_t)n * m);
    dZ = L.take<double>((size_t)n * m);
    dD = L.take<double>(n);
    return B2K_OK;
  }));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(dD, dinv.data(), n * 8, cudaMemcpyHostToDevice, s));
  auto apply = [&](const std::vector<double>& in, std::vector<double>& out) -> int {
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(dY, in.data(), in.size() * 8, cudaMemcpyHostToDevice, s));
    k_umap_spmm<<<grid_for(ctx, n, U_WARPS), U_WARPS * 32, 0, s>>>(G.indptr, G.cols, G.vals, dD, dY, n, m, dZ);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(out.data(), dZ, out.size() * 8, cudaMemcpyDeviceToHost, s));
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
    return B2K_OK;
  };
  std::vector<double> H2((size_t)m * m), w, V, X((size_t)n * C);
  for (int it = 0;; ++it) {
    B2K_TRY(apply(Y, Z));
    // Rayleigh-Ritz on span(Y): H2 = Y^T Z, eigenpairs in descending order
    for (int a = 0; a < m; ++a)
      for (int b = 0; b < m; ++b) {
        double t = 0.0;
        for (int64_t i = 0; i < n; ++i) t += Y[i * m + a] * Z[i * m + b];
        H2[(size_t)a * m + b] = t;
      }
    for (int a = 0; a < m; ++a)
      for (int b = 0; b < a; ++b) H2[(size_t)a * m + b] = H2[(size_t)b * m + a] = 0.5 * (H2[(size_t)a * m + b] + H2[(size_t)b * m + a]);
    std::vector<double> Hc = H2;
    if (!b2k_sym_eig(Hc, m, w, V)) return b2k_fail(ctx, B2K_ERR_INVALID, "UMAP spectral init: eigensolver failed");
    std::vector<int> ord(m);
    std::iota(ord.begin(), ord.end(), 0);
    std::stable_sort(ord.begin(), ord.end(), [&](int a, int b) { return w[a] > w[b]; });
    // residual of the C Ritz pairs of (M + I) / 2: || Z V - Y V theta || per vector, the largest
    double r = 0.0;
    for (int c = 0; c < C; ++c) {
      const double* v = &V[(size_t)ord[c] * m];
      double rr = 0.0;
      for (int64_t i = 0; i < n; ++i) {
        double zy = 0.0, yy = 0.0;
        for (int b = 0; b < m; ++b) {
          zy += Z[i * m + b] * v[b];
          yy += Y[i * m + b] * v[b];
        }
        X[i * C + c] = yy;
        rr += (zy - w[ord[c]] * yy) * (zy - w[ord[c]] * yy);
      }
      r = std::max(r, std::sqrt(rr));
    }
    if (r < SPECTRAL_TOL || it + 1 >= SPECTRAL_MAX_ITERS) {
      *resid = 2.0 * r;   // of M itself
      val->resize(C);
      for (int c = 0; c < C; ++c) (*val)[c] = 2.0 * w[ord[c]] - 1.0;
      *vec = X;
      return B2K_OK;
    }
    Y.swap(Z);
    orthonormalise(Y, n, m, v0);
  }
}

}  // namespace

int b2k_umap_fit_impl(b2k_ctx* ctx, const float* X, int64_t n, int d, const int32_t* labels,
                      const b2k_umap_params& p, float* embedding_out, double* info_out, cudaStream_t s) {
  const char* who = "b2k_umap_fit";
  if (n < 2) return b2k_fail(ctx, B2K_ERR_INVALID, std::string(who) + ": UMAP needs at least 2 rows, got " +
                                                       std::to_string(n));
  if (n > (int64_t)0x7fffffff) return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, std::string(who) + ": 2^31 rows or more");
  B2K_TRY(check_params(ctx, who, p, n));
  if (p.n_epochs < 1) return b2k_fail(ctx, B2K_ERR_INVALID, std::string(who) + ": n_epochs must be >= 1");
  if (p.init < 0 || p.init > 2) return b2k_fail(ctx, B2K_ERR_INVALID, std::string(who) + ": init must be 0, 1 or 2");
  // the graph's scan positions are int: 2 n k keys, and up to 4 n k in the supervised second fold (nnz <= 2 n k)
  if ((labels ? 4 : 2) * n * p.n_neighbors >= (int64_t)0x7fffffff)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, std::string(who) + ": " + (labels ? "4" : "2") +
                                                  " n n_neighbors must stay below 2^31");
  int64_t nbad = 0;
  B2K_TRY(count_bad(ctx, X, n * d, &nbad, s));
  if (nbad > 0) return b2k_fail(ctx, B2K_ERR_INVALID, std::string(who) + ": UMAP input contains NaN or infinity");
  const int k = p.n_neighbors, C = p.n_components;
  Events ev;
  cudaEventRecord(ev.ev[0], s);
  auto G = std::make_shared<UmapGraph>();
  G->n = n;
  G->k = k;
  G->C = C;
  // ---- kNN and memberships (device buffers cudaMalloc'd for the call: they outlive several scratch layouts) ----
  float* dist = nullptr;
  int64_t* idx = nullptr;
  double *rho = nullptr, *sigma = nullptr, *P = nullptr, *rsum = nullptr;
  struct Frees {
    std::vector<void*> v;
    ~Frees() {
      for (void* q : v) cudaFree(q);
    }
  } fr;
  auto dmalloc = [&](void** q, size_t bytes) -> int {
    B2K_CUDA_OK(ctx, cudaMalloc(q, std::max<size_t>(bytes, 8)));
    fr.v.push_back(*q);
    return B2K_OK;
  };
  B2K_TRY(dmalloc((void**)&dist, (size_t)n * k * 4));
  B2K_TRY(dmalloc((void**)&idx, (size_t)n * k * 8));
  B2K_TRY(dmalloc((void**)&rho, (size_t)n * 8));
  B2K_TRY(dmalloc((void**)&sigma, (size_t)n * 8));
  B2K_TRY(dmalloc((void**)&P, (size_t)n * k * 8));
  B2K_TRY(dmalloc((void**)&rsum, (size_t)n * 8));
  B2K_TRY(b2k_knn_local_impl(ctx, X, n, X, n, d, k, dist, idx, s));
  cudaEventRecord(ev.ev[1], s);
  k_umap_row_sums<<<grid_for(ctx, n, 256), 256, 0, s>>>(dist, n, k, rsum);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  std::vector<double> hs(n);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(hs.data(), rsum, n * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  double mean_all = 0.0;
  for (double v : hs) mean_all += v;
  mean_all /= (double)n * (double)k;
  k_umap_membership<<<grid_for(ctx, n, 128), 128, 0, s>>>(dist, idx, n, k, p.local_connectivity, mean_all, rho, sigma,
                                                          P);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches += 2;
  DevCsr W;
  struct CsrFree {
    DevCsr* c;
    ~CsrFree() { c->release(); }
  } wf{&W};
  B2K_TRY(symmetrise(ctx, nullptr, k, idx, P, n * k, n, p.set_op_mix_ratio, &W, s));
  if (labels) {
    int64_t *r2 = nullptr, *c2 = nullptr;
    double* v2 = nullptr;
    B2K_TRY(dmalloc((void**)&r2, (size_t)W.nnz * 8));
    B2K_TRY(dmalloc((void**)&c2, (size_t)W.nnz * 8));
    B2K_TRY(dmalloc((void**)&v2, (size_t)W.nnz * 8));
    k_umap_labels<<<grid_for(ctx, n, U_WARPS), U_WARPS * 32, 0, s>>>(W.indptr, W.cols, W.vals, labels, n, r2, c2, v2);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
    B2K_TRY(symmetrise(ctx, r2, 0, c2, v2, W.nnz, n, 1.0, &W, s));
  }
  const int64_t nnz = W.nnz;
  G->nnz = nnz;
  G->knn_idx.resize((size_t)n * k);
  G->knn_dist.resize((size_t)n * k);
  G->rho.resize(n);
  G->sigma.resize(n);
  G->indptr.resize(n + 1);
  G->indices.resize(nnz);
  G->weights.resize(nnz);
  G->eps.resize(nnz);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(G->knn_idx.data(), idx, (size_t)n * k * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(G->knn_dist.data(), dist, (size_t)n * k * 4, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(G->rho.data(), rho, n * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(G->sigma.data(), sigma, n * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(G->indptr.data(), W.indptr, (n + 1) * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(G->indices.data(), W.cols, nnz * 4, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(G->weights.data(), W.vals, nnz * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  double wmax = 0.0;
  for (double v : G->weights) wmax = std::max(wmax, v);

  // ---- schedule ----
  double *eps = nullptr, *next = nullptr, *next_neg = nullptr, *epn = nullptr;
  B2K_TRY(dmalloc((void**)&eps, (size_t)nnz * 8));
  B2K_TRY(dmalloc((void**)&next, (size_t)nnz * 8));
  B2K_TRY(dmalloc((void**)&next_neg, (size_t)nnz * 8));
  B2K_TRY(dmalloc((void**)&epn, (size_t)nnz * 8));
  if (nnz > 0) {
    k_umap_schedule<<<grid_for(ctx, nnz, 256), 256, 0, s>>>(W.vals, nnz, wmax, p.n_epochs,
                                                            std::max(p.negative_sample_rate, 1), eps, next, next_neg,
                                                            epn);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
    if (p.negative_sample_rate == 0) {   // no negatives: their next epoch never comes due
      std::vector<double> big(nnz, INFINITY);
      B2K_CUDA_OK(ctx, cudaMemcpyAsync(epn, big.data(), nnz * 8, cudaMemcpyHostToDevice, s));
    }
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(G->eps.data(), eps, nnz * 8, cudaMemcpyDeviceToHost, s));
  }
  cudaEventRecord(ev.ev[2], s);

  // ---- initial layout ----
  std::vector<float> Y0((size_t)n * C);
  int init_used = p.init;
  double resid = 0.0;
  if (p.init == 1) {
    if (components(G->indptr, G->indices, n) > 1 || n <= C + 1) {
      init_used = 0;
    } else {
      std::vector<double> vec, val;
      B2K_TRY(spectral(ctx, W, *G, C, p.seed, &vec, &val, &resid, s));
      G->ritz_values = val;
      G->ritz_vectors = vec;
      double mx = 0.0;
      for (double v : vec) mx = std::max(mx, std::fabs(v));
      const double sc = mx > 0.0 ? 10.0 / mx : 1.0;
      for (size_t e = 0; e < vec.size(); ++e) {
        // N(0, 1e-4) by Box-Muller from two draws of umap_hash
        const double u1 = umap_unit(umap_hash(p.seed, 1ull << 42, e, 0)), u2 = umap_unit(umap_hash(p.seed, 1ull << 42, e, 1));
        const double z = std::sqrt(-2.0 * std::log(1.0 - u1)) * std::cos(2.0 * M_PI * u2);
        Y0[e] = (float)((double)(float)(vec[e] * sc) + 1e-4 * z);
      }
    }
  }
  if (init_used == 0)
    for (size_t e = 0; e < Y0.size(); ++e)
      Y0[e] = (float)(20.0 * umap_unit(umap_hash(p.seed, 1ull << 40, e / C, e % C)) - 10.0);
  if (init_used != 2) {
    for (int c = 0; c < C; ++c) {   // each column to [0, 10]
      double lo = INFINITY, hi = -INFINITY;
      for (int64_t i = 0; i < n; ++i) lo = std::min(lo, (double)Y0[i * C + c]), hi = std::max(hi, (double)Y0[i * C + c]);
      const double span = hi - lo;
      for (int64_t i = 0; i < n; ++i)
        Y0[i * C + c] = (float)(span > 0.0 ? 10.0 * ((double)Y0[i * C + c] - lo) / span : 0.0);
    }
  } else {
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(Y0.data(), embedding_out, Y0.size() * 4, cudaMemcpyDeviceToHost, s));
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  }
  G->init = Y0;
  float* Yb[2] = {nullptr, nullptr};
  B2K_TRY(dmalloc((void**)&Yb[0], Y0.size() * 4));
  B2K_TRY(dmalloc((void**)&Yb[1], Y0.size() * 4));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(Yb[0], Y0.data(), Y0.size() * 4, cudaMemcpyHostToDevice, s));
  cudaEventRecord(ev.ev[3], s);

  // ---- layout: one launch per epoch ----
  const int E = ctx->umap_stop_epochs > 0 ? std::min(ctx->umap_stop_epochs, p.n_epochs) : p.n_epochs;
  LayoutArgs la{};
  la.indptr = W.indptr;
  la.cols = W.cols;
  la.eps = eps;
  la.epn = epn;
  la.next = next;
  la.next_neg = next_neg;
  la.n = n;
  la.k = UmapCoef{(float)p.a, (float)p.b, (float)p.repulsion_strength};
  la.seed = p.seed;
  const unsigned lg = grid_for(ctx, n, U_WARPS);
  for (int e = 0; e < E; ++e) {
    la.Y = Yb[e & 1];
    la.Yn = Yb[(e + 1) & 1];
    la.e = e;
    la.alpha = (float)(p.learning_rate * (1.0 - (double)e / (double)p.n_epochs));
    switch (C) {
      case 1: k_umap_layout_small<1><<<lg, U_WARPS * 32, 0, s>>>(la); break;
      case 2: k_umap_layout_small<2><<<lg, U_WARPS * 32, 0, s>>>(la); break;
      case 3: k_umap_layout_small<3><<<lg, U_WARPS * 32, 0, s>>>(la); break;
      case 4: k_umap_layout_small<4><<<lg, U_WARPS * 32, 0, s>>>(la); break;
      default: k_umap_layout_wide<<<lg, U_WARPS * 32, 0, s>>>(la, C);
    }
    B2K_CUDA_OK(ctx, cudaGetLastError());
  }
  ctx->stats.kernel_launches += E;
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(embedding_out, Yb[E & 1], Y0.size() * 4, cudaMemcpyDeviceToDevice, s));
  cudaEventRecord(ev.ev[4], s);
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  ctx->stats.last_path = C <= U_SMALL_C ? B2K_PATH_FUSED : B2K_PATH_GENERIC;
  ctx->stats.last_n_iter = E;
  ctx->stats.last_finalize_ms = ev.ms(0, 1);   // kNN
  ctx->stats.last_reduce_ms = ev.ms(1, 2);     // graph and schedule
  ctx->stats.last_allreduce_ms = ev.ms(2, 3);  // init
  ctx->stats.last_fused_ms = ev.ms(3, 4);      // layout
  ctx->stats.last_loop_ms = ev.ms(0, 4);
  if (info_out) {
    info_out[0] = (double)n;
    info_out[1] = (double)k;
    info_out[2] = (double)nnz;
    info_out[3] = (double)E;
    info_out[4] = (double)init_used;
    info_out[5] = resid;
    info_out[6] = (double)C;
    info_out[7] = wmax;
  }
  ctx->umap_graph = G;
  return B2K_OK;
}

int b2k_umap_graph_impl(b2k_ctx* ctx, int64_t* knn_idx, float* knn_dist, double* rho, double* sigma, int64_t* indptr,
                        int32_t* indices, double* weights, double* eps, float* init, double* ritz_values,
                        double* ritz_vectors) {
  const UmapGraph* G = static_cast<const UmapGraph*>(ctx->umap_graph.get());
  if (!G) return b2k_fail(ctx, B2K_ERR_STATE, "b2k_umap_graph: no UMAP fitted on this context");
  auto put = [](auto* dst, const auto& v) {
    if (dst) std::copy(v.begin(), v.end(), dst);
  };
  put(knn_idx, G->knn_idx);
  put(knn_dist, G->knn_dist);
  put(rho, G->rho);
  put(sigma, G->sigma);
  put(indptr, G->indptr);
  put(indices, G->indices);
  put(weights, G->weights);
  put(eps, G->eps);
  put(init, G->init);
  put(ritz_values, G->ritz_values);
  put(ritz_vectors, G->ritz_vectors);
  return B2K_OK;
}

int b2k_umap_transform_impl(b2k_ctx* ctx, const float* X_train, const float* Y_train, int64_t n_train, int d,
                            const float* Q, int64_t nq, const b2k_umap_params& p, float* out, cudaStream_t s) {
  const char* who = "b2k_umap_transform";
  if (n_train < 1) return b2k_fail(ctx, B2K_ERR_INVALID, std::string(who) + ": the model has no training rows");
  B2K_TRY(check_params(ctx, who, p, n_train));
  if (p.n_epochs < 0) return b2k_fail(ctx, B2K_ERR_INVALID, std::string(who) + ": n_epochs must be >= 0");
  if (nq == 0) return B2K_OK;
  const int k = p.n_neighbors;
  float* dist = nullptr;
  int64_t* idx = nullptr;
  B2K_CUDA_OK(ctx, cudaMalloc(&dist, (size_t)nq * k * 4));
  struct Free {
    void* a = nullptr;
    void* b = nullptr;
    ~Free() {
      cudaFree(a);
      cudaFree(b);
    }
  } fr{dist, nullptr};
  B2K_CUDA_OK(ctx, cudaMalloc(&idx, (size_t)nq * k * 8));
  fr.b = idx;
  Events ev;
  cudaEventRecord(ev.ev[0], s);
  B2K_TRY(b2k_knn_local_impl(ctx, X_train, n_train, Q, nq, d, k, dist, idx, s));
  cudaEventRecord(ev.ev[1], s);
  TransformArgs a{};
  a.Yt = Y_train;
  a.dist = dist;
  a.idx = idx;
  a.Q = Q;
  a.out = out;
  a.nq = nq;
  a.n_train = n_train;
  a.k = k;
  a.d = d;
  a.C = p.n_components;
  a.n_epochs = p.n_epochs;
  a.neg_rate = p.negative_sample_rate;
  a.lc = p.local_connectivity;
  a.lr = (float)p.learning_rate;
  a.kc = UmapCoef{(float)p.a, (float)p.b, (float)p.repulsion_strength};
  a.seed = p.seed;
  const size_t smem = (size_t)U_WARPS * 5 * k * 8;
  B2K_CUDA_OK(ctx, cudaFuncSetAttribute(k_umap_transform, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_umap_transform<<<grid_for(ctx, nq, U_WARPS), U_WARPS * 32, smem, s>>>(a);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  cudaEventRecord(ev.ev[2], s);
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  ctx->stats.last_finalize_ms = ev.ms(0, 1);
  ctx->stats.last_fused_ms = ev.ms(1, 2);
  ctx->stats.last_loop_ms = ev.ms(0, 2);
  return B2K_OK;
}
