// ALS (alternating least squares collaborative filtering) on sm_90a: Spark's pyspark.ml.recommendation.ALS, its rules
// pinned in include/b2kmeans.h.
//
// Setup (collective): an id/rating check pass, one allgather of the sizes and error flags, the sorted distinct user and
// item ids from per-rank sort-uniques gathered to every rank, then a redistribution of the ratings by chunked
// allgathers: each rank keeps the ratings of the users it owns sorted by (user, item, global row) and of the items it
// owns sorted by (item, user, global row).
// Per half-step: (implicit) Y^T Y of the whole source table by the local generic Gram pass; the normal-equation pass over
// units (one destination, or UNIT ratings of it) writing fp64 partials; the solve pass folding a destination's units in
// order, adding the regularisation and solving by Cholesky in shared memory; an allgather of the solved rows.  No pass
// uses atomics: a fit is bitwise reproducible and, for the same global row order, does not depend on the rank count.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_select.cuh>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>

#include "b2k_internal.cuh"

namespace {

constexpr int ALS_UNIT = 512;                       // ratings per unit of the normal-equation pass
constexpr int ALS_CH = 32;                          // ratings staged in shared memory per step of a unit
constexpr int64_t ALS_GATHER = (int64_t)1 << 22;    // ratings per rank per redistribution round
constexpr size_t ALS_PART_BYTES = (size_t)1 << 30;  // fp64 partials of one batch of units
constexpr int ALS_SOLVE_NT = 128;
constexpr int ALS_REC_WARPS = 8;                    // query rows per CTA of the recommend pass

struct Rec {          // one rating on its way to its owners
  int32_t u, i;       // dense user / item index
  float r;
  int32_t valid;
};
struct OwnRec {       // one rating kept by an owner
  int64_t grow;       // global row: rank offset + local row
  int32_t dst, src;
  float r;
  int32_t pad;
};

__device__ __forceinline__ bool id_ok(double v) {
  return v == v && v >= -2147483648.0 && v <= 2147483647.0 && v == floor(v);
}

// per CTA, the first row (or INT64_MAX) with a bad user id, bad item id and non-finite rating; int32 ids and fp32 ratings
__global__ void __launch_bounds__(256) k_als_check(const double* __restrict__ u, const double* __restrict__ it,
                                                   const float* __restrict__ r, int64_t n, int64_t per,
                                                   int32_t* __restrict__ u32, int32_t* __restrict__ i32,
                                                   float* __restrict__ r32, int64_t* __restrict__ bad) {
  __shared__ int64_t sb[3][256];
  const int64_t r0 = (int64_t)blockIdx.x * per, r1 = min(n, r0 + per);
  int64_t b0 = INT64_MAX, b1 = INT64_MAX, b2 = INT64_MAX;
  for (int64_t j = r0 + threadIdx.x; j < r1; j += blockDim.x) {
    const double a = u[j], b = it[j];
    const float c = r ? r[j] : 1.0f;
    if (!id_ok(a)) b0 = min(b0, j);
    if (!id_ok(b)) b1 = min(b1, j);
    if (!isfinite(c)) b2 = min(b2, j);
    u32[j] = id_ok(a) ? (int32_t)a : 0;
    i32[j] = id_ok(b) ? (int32_t)b : 0;
    r32[j] = c;
  }
  sb[0][threadIdx.x] = b0;
  sb[1][threadIdx.x] = b1;
  sb[2][threadIdx.x] = b2;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w)
      for (int k = 0; k < 3; ++k) sb[k][threadIdx.x] = min(sb[k][threadIdx.x], sb[k][threadIdx.x + w]);
    __syncthreads();
  }
  if (threadIdx.x < 3) bad[blockIdx.x * 3 + threadIdx.x] = sb[threadIdx.x][0];
}

__device__ __forceinline__ int32_t find_id(const int32_t* __restrict__ ids, int64_t m, int32_t v) {
  int64_t lo = 0, hi = m;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (ids[mid] < v) lo = mid + 1;
    else hi = mid;
  }
  return (lo < m && ids[lo] == v) ? (int32_t)lo : -1;
}

// raw ids -> dense indices (every id is present: the maps hold every rank's ids)
__global__ void k_als_dense(int32_t* __restrict__ u, int32_t* __restrict__ it, int64_t n, const int32_t* __restrict__ uid,
                            int64_t nu, const int32_t* __restrict__ iid, int64_t ni) {
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
    u[j] = find_id(uid, nu, u[j]);
    it[j] = find_id(iid, ni, it[j]);
  }
}

__global__ void k_als_pack(const int32_t* __restrict__ u, const int32_t* __restrict__ it, const float* __restrict__ r,
                           int64_t r0, int64_t r1, int64_t G, Rec* __restrict__ out) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= G) return;
  const int64_t row = r0 + j;
  Rec x{0, 0, 0.f, 0};
  if (row < r1) x = Rec{u[row], it[row], r[row], 1};
  out[j] = x;
}

// rounds: slot (q, j) of a gathered round is local row c * G + j of rank q
__global__ void k_als_own(const Rec* __restrict__ g, int R, int64_t G, const int64_t* __restrict__ offs, int64_t c, int64_t u0,
                          int64_t u1, int64_t i0, int64_t i1, OwnRec* __restrict__ ou, OwnRec* __restrict__ oi,
                          uint8_t* __restrict__ fu, uint8_t* __restrict__ fi) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= (int64_t)R * G) return;
  const int q = (int)(k / G);
  const int64_t j = k % G;
  const Rec x = g[k];
  const int64_t grow = offs[q] + c * G + j;
  ou[k] = OwnRec{grow, x.u, x.i, x.r, 0};
  oi[k] = OwnRec{grow, x.i, x.u, x.r, 0};
  fu[k] = x.valid && x.u >= u0 && x.u < u1;
  fi[k] = x.valid && x.i >= i0 && x.i < i1;
}

__global__ void k_als_keys(const OwnRec* __restrict__ rec, const int32_t* __restrict__ perm, int64_t m, int64_t d0,
                           unsigned long long* __restrict__ key, int32_t* __restrict__ idx) {
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < m; j += (int64_t)gridDim.x * blockDim.x) {
    const int32_t p = perm ? perm[j] : (int32_t)j;
    const OwnRec x = rec[p];
    key[j] = perm ? ((unsigned long long)(x.dst - d0) << 31) | (unsigned long long)x.src : (unsigned long long)x.grow;
    idx[j] = p;
  }
}

__global__ void k_als_unpack(const OwnRec* __restrict__ rec, const int32_t* __restrict__ perm, int64_t m, int64_t d0,
                             int32_t* __restrict__ dst, int32_t* __restrict__ src, float* __restrict__ r) {
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < m; j += (int64_t)gridDim.x * blockDim.x) {
    const OwnRec x = rec[perm[j]];
    dst[j] = (int32_t)(x.dst - d0);
    src[j] = x.src;
    r[j] = x.r;
  }
}

// ptr[k] = first rating of local destination k (dst sorted ascending), k in [0, nd]
__global__ void k_als_ptr(const int32_t* __restrict__ dst, int64_t m, int64_t nd, int64_t* __restrict__ ptr) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k <= nd; k += (int64_t)gridDim.x * blockDim.x) {
    int64_t lo = 0, hi = m;
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (dst[mid] < k) lo = mid + 1;
      else hi = mid;
    }
    ptr[k] = lo;
  }
}

// start factors: rank normals keyed by (seed, raw id, j), scaled to unit L2 norm (include/b2kmeans.h)
__global__ void k_als_start(const int32_t* __restrict__ ids, int64_t m, int rank, uint64_t seed, float* __restrict__ F) {
  const int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= m) return;
  const uint64_t base = b2k_splitmix64(seed) ^ (uint64_t)(uint32_t)ids[u];
  float* f = F + u * rank;
  double ss = 0.0;
  for (int j = 0; j < rank; ++j) {
    const uint64_t h = b2k_splitmix64(b2k_splitmix64(base) ^ (uint64_t)j);
    const double u1 = (double)((h >> 11) + 1) * 0x1.0p-53;
    const double u2 = (double)(b2k_splitmix64(h) >> 11) * 0x1.0p-53;
    const float v = (float)(sqrt(-2.0 * log(u1)) * cospi(2.0 * u2));
    f[j] = v;
    ss += (double)v * (double)v;
  }
  const double nrm = sqrt(ss);
  for (int j = 0; j < rank; ++j) f[j] = (float)((double)f[j] / nrm);
}

struct Unit {
  int64_t beg, end;   // ratings [beg, end) of the side's sorted arrays
};

// The normal-equation pass.  A unit's partial: the upper 4 x 4 tiles of A (tile (I, J), I <= J, in row-major order of
// the upper block triangle, 16 entries each, row-major inside), then b [RP], then the count n: PS doubles in all.
// Thread t forms tiles t, t + NT, ...; each entry adds its terms in rating order with fp64 FMA (the fp32 products are
// exact in fp64, so only the order of the additions matters, and it is fixed).
template <int NT, int MAXT, int RPM, bool IMPL>
__global__ void __launch_bounds__(NT) k_als_normal(const float* __restrict__ Y, int rank, int rp,
                                                   const int32_t* __restrict__ src, const float* __restrict__ rat,
                                                   const Unit* __restrict__ units, int nunits, double alpha,
                                                   double* __restrict__ part) {
  __shared__ __align__(16) float ys[ALS_CH][RPM];
  __shared__ double wa[ALS_CH], wb[ALS_CH];
  const int nb = rp >> 2, tri = nb * (nb + 1) / 2;
  const size_t PS = (size_t)tri * 16 + rp + 1;
  int ti[MAXT], tj[MAXT];
#pragma unroll
  for (int k = 0; k < MAXT; ++k) {
    int t = threadIdx.x + k * NT, I = 0;
    if (t >= tri) t = -1;
    if (t >= 0)
      while (t >= nb - I) {
        t -= nb - I;
        ++I;
      }
    ti[k] = t < 0 ? -1 : I;
    tj[k] = t < 0 ? 0 : I + t;
  }
  for (int un = blockIdx.x; un < nunits; un += gridDim.x) {
    const Unit U = units[un];
    double acc[MAXT][4][4];
#pragma unroll
    for (int k = 0; k < MAXT; ++k)
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[k][a][b] = 0.0;
    double bacc = 0.0, cnt = 0.0;
    for (int64_t c0 = U.beg; c0 < U.end; c0 += ALS_CH) {
      const int jn = (int)min((int64_t)ALS_CH, U.end - c0);
      for (int e = threadIdx.x; e < ALS_CH * rp; e += NT) {
        const int j = e / rp, col = e - j * rp;
        ys[j][col] = (j < jn && col < rank) ? Y[(size_t)src[c0 + j] * rank + col] : 0.f;
      }
      if (threadIdx.x < ALS_CH) {
        const int j = threadIdx.x;
        const double r = j < jn ? (double)rat[c0 + j] : 0.0;
        if (IMPL) {
          const double c1 = alpha * fabs(r);
          wa[j] = c1;
          wb[j] = r > 0.0 ? 1.0 + c1 : 0.0;
        } else {
          wa[j] = 1.0;
          wb[j] = r;
        }
      }
      __syncthreads();
      for (int j = 0; j < jn; ++j) {
#pragma unroll
        for (int k = 0; k < MAXT; ++k) {
          if (ti[k] < 0) continue;
          const float4 p = *reinterpret_cast<const float4*>(&ys[j][ti[k] * 4]);
          const float4 q = *reinterpret_cast<const float4*>(&ys[j][tj[k] * 4]);
          double pa[4] = {p.x, p.y, p.z, p.w};
          const double qa[4] = {q.x, q.y, q.z, q.w};
          if (IMPL) {
            const double w = wa[j];
#pragma unroll
            for (int a = 0; a < 4; ++a) pa[a] *= w;
          }
#pragma unroll
          for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int b = 0; b < 4; ++b) acc[k][a][b] = fma(pa[a], qa[b], acc[k][a][b]);
        }
        if ((int)threadIdx.x < rp) bacc = fma(wb[j], (double)ys[j][threadIdx.x], bacc);
        if (threadIdx.x == 0) cnt += IMPL ? (wb[j] > 0.0 ? 1.0 : 0.0) : 1.0;
      }
      __syncthreads();
    }
    double* o = part + (size_t)un * PS;
#pragma unroll
    for (int k = 0; k < MAXT; ++k) {
      if (ti[k] < 0) continue;
      const int t = threadIdx.x + k * NT;
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) o[(size_t)t * 16 + a * 4 + b] = acc[k][a][b];
    }
    if ((int)threadIdx.x < rp) o[(size_t)tri * 16 + threadIdx.x] = bacc;
    if (threadIdx.x == 0) o[(size_t)tri * 16 + rp] = cnt;
  }
}

__device__ __forceinline__ int tile_index(int I, int J, int nb) { return I * nb - I * (I - 1) / 2 + (J - I); }

// The solve pass: one CTA per destination k of [k0, k0 + nd): A (lower triangle) and b from its units' partials folded
// in unit order, (+ Y^T Y), + reg n on the diagonal, Cholesky in shared memory on [A | b], then L^T x = y.  A pivot that
// is not positive (or not finite) sets bad[k]; the row is then written as NaN.
__global__ void __launch_bounds__(ALS_SOLVE_NT) k_als_solve(const double* __restrict__ part, const int64_t* __restrict__ uofs,
                                                            int k0, int nd, int64_t ubase, int rank, int rp,
                                                            const double* __restrict__ YtY, double reg,
                                                            float* __restrict__ out, int32_t* __restrict__ bad) {
  extern __shared__ double A[];   // [rank][rank + 1]: lower triangle of A, column rank = b
  __shared__ double s_n;
  __shared__ int s_bad;
  const int ld = rank + 1, nb = rp >> 2, tri = nb * (nb + 1) / 2;
  const size_t PS = (size_t)tri * 16 + rp + 1;
  for (int kk = blockIdx.x; kk < nd; kk += gridDim.x) {
    const int k = k0 + kk;
    const int64_t u0 = uofs[k] - ubase, u1 = uofs[k + 1] - ubase;
    for (int e = threadIdx.x; e < rank * ld + 1; e += ALS_SOLVE_NT) {
      double s = 0.0;
      if (e < rank * ld) {
        const int i = e / ld, j = e - i * ld;
        if (j == rank) {
          for (int64_t u = u0; u < u1; ++u) s += part[u * PS + (size_t)tri * 16 + i];
        } else if (j <= i) {
          const size_t off = (size_t)tile_index(j >> 2, i >> 2, nb) * 16 + (j & 3) * 4 + (i & 3);
          for (int64_t u = u0; u < u1; ++u) s += part[u * PS + off];
          if (YtY) s += YtY[j * (2 * rank - j + 1) / 2 + (i - j)];   // (j, i) of the packed upper triangle
        }
        A[e] = s;
      } else {
        for (int64_t u = u0; u < u1; ++u) s += part[u * PS + (size_t)tri * 16 + rp];
        s_n = s;
      }
    }
    if (threadIdx.x == 0) s_bad = 0;
    __syncthreads();
    const double lam = reg * s_n;
    for (int i = threadIdx.x; i < rank; i += ALS_SOLVE_NT) A[i * ld + i] += lam;
    __syncthreads();
    for (int c = 0; c < rank; ++c) {
      const double piv = A[c * ld + c];
      if (!(piv > 0.0) || !isfinite(piv)) {
        if (threadIdx.x == 0) s_bad = 1;
        break;
      }
      const double l = sqrt(piv);
      __syncthreads();   // every thread has read the pivot
      for (int i = c + 1 + threadIdx.x; i <= rank; i += ALS_SOLVE_NT) {
        if (i < rank) A[i * ld + c] /= l;
        else A[c * ld + rank] /= l;   // y_c
      }
      if (threadIdx.x == 0) A[c * ld + c] = l;
      __syncthreads();
      const int m = rank - c - 1;
      for (int e = threadIdx.x; e < m * (m + 1); e += ALS_SOLVE_NT) {
        const int i = c + 1 + e / (m + 1), j = c + 1 + e % (m + 1);
        if (j == rank) A[i * ld + rank] -= A[i * ld + c] * A[c * ld + rank];
        else if (j <= i) A[i * ld + j] -= A[i * ld + c] * A[j * ld + c];
      }
      __syncthreads();
    }
    __syncthreads();
    const bool ok = s_bad == 0;
    if (ok) {
      for (int c = rank - 1; c >= 0; --c) {   // L^T x = y, x into column rank
        if (threadIdx.x == 0) A[c * ld + rank] /= A[c * ld + c];
        __syncthreads();
        const double x = A[c * ld + rank];
        for (int i = threadIdx.x; i < c; i += ALS_SOLVE_NT) A[i * ld + rank] -= A[c * ld + i] * x;
        __syncthreads();
      }
    }
    for (int j = threadIdx.x; j < rank; j += ALS_SOLVE_NT)
      out[(size_t)k * rank + j] = ok ? (float)A[j * ld + rank] : __int_as_float(0x7fc00000);
    if (threadIdx.x == 0) bad[k] = ok ? 0 : 1;
    __syncthreads();
  }
}

// count of bad systems (fixed-order block sum)
__global__ void __launch_bounds__(256) k_als_count(const int32_t* __restrict__ bad, int64_t m, double* __restrict__ out) {
  __shared__ int64_t sb[256];
  int64_t c = 0;
  for (int64_t j = threadIdx.x; j < m; j += 256) c += bad[j];
  sb[threadIdx.x] = c;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) sb[threadIdx.x] += sb[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) *out = (double)sb[0];
}

// the prediction: fl32 products added in rank order, no FMA
__device__ __forceinline__ float als_dot(const float* __restrict__ a, const float* __restrict__ b, int rank) {
  float s = 0.f;
  for (int j = 0; j < rank; ++j) s = __fadd_rn(s, __fmul_rn(a[j], b[j]));
  return s;
}

__device__ __forceinline__ int32_t lookup(double v, const int32_t* __restrict__ ids, int64_t m) {
  return id_ok(v) ? find_id(ids, m, (int32_t)v) : -1;
}

__global__ void k_als_predict(const double* __restrict__ u, const double* __restrict__ it, int64_t n, int rank,
                              const int32_t* __restrict__ uid, const float* __restrict__ UF, int64_t nu,
                              const int32_t* __restrict__ iid, const float* __restrict__ IF, int64_t ni,
                              float* __restrict__ out) {
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
    const int32_t a = lookup(u[j], uid, nu), b = lookup(it[j], iid, ni);
    out[j] = (a < 0 || b < 0) ? __int_as_float(0x7fc00000)
                              : als_dot(UF + (size_t)a * rank, IF + (size_t)b * rank, rank);
  }
}

__device__ __forceinline__ bool better(float s1, int32_t i1, float s2, int32_t i2) {
  return s1 > s2 || (s1 == s2 && i1 < i2);
}

// The recommend pass: warp w of a CTA serves query row blockIdx.x * ALS_REC_WARPS + w (grid-stride); the CTA streams
// the targets through shared memory 32 at a time, each lane scores one target, and the warp keeps its row's best n
// sorted (score descending, lower index first) in shared memory.
__global__ void __launch_bounds__(32 * ALS_REC_WARPS, 1) k_als_recommend(const float* __restrict__ Q, int64_t nq,
                                                                      const float* __restrict__ T, int64_t nt, int rank,
                                                                      int n, int32_t* __restrict__ idx_out,
                                                                      float* __restrict__ score_out) {
  extern __shared__ float sm[];
  const int ldt = rank + 1;
  float* tt = sm;                                   // [32][rank + 1]
  float* qq = tt + 32 * ldt;                        // [warps][rank]
  float* ls = qq + ALS_REC_WARPS * rank;            // [warps][n] scores
  int32_t* li = reinterpret_cast<int32_t*>(ls + ALS_REC_WARPS * n);   // [warps][n] indices
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* myq = qq + w * rank;
  float* mys = ls + (size_t)w * n;
  int32_t* myi = li + (size_t)w * n;
  for (int64_t qb = (int64_t)blockIdx.x * ALS_REC_WARPS; qb < nq; qb += (int64_t)gridDim.x * ALS_REC_WARPS) {
    const int64_t q = qb + w;
    const bool live = q < nq;
    for (int j = lane; j < rank; j += 32) myq[j] = live ? Q[q * rank + j] : 0.f;
    int cnt = 0;
    for (int64_t t0 = 0; t0 < nt; t0 += 32) {
      __syncthreads();
      for (int e = threadIdx.x; e < 32 * rank; e += 32 * ALS_REC_WARPS) {
        const int r = e / rank, c = e - r * rank;
        tt[r * ldt + c] = t0 + r < nt ? T[(t0 + r) * rank + c] : 0.f;
      }
      __syncthreads();
      if (!live) continue;
      const int32_t ti = (int32_t)(t0 + lane);
      const bool valid = t0 + lane < nt;
      float sc = 0.f;
      if (valid) {
        const float* tr = tt + lane * ldt;
        for (int j = 0; j < rank; ++j) sc = __fadd_rn(sc, __fmul_rn(myq[j], tr[j]));
      }
      unsigned mask = __ballot_sync(0xffffffffu, valid && (cnt < n || better(sc, ti, mys[n - 1], myi[n - 1])));
      while (mask) {
        const int src = __ffs(mask) - 1;
        mask &= mask - 1;
        const float cs = __shfl_sync(0xffffffffu, sc, src);
        const int32_t ci = __shfl_sync(0xffffffffu, ti, src);
        if (cnt == n && !better(cs, ci, mys[n - 1], myi[n - 1])) continue;
        int pos = 0;
        for (int e = lane; e < cnt; e += 32) pos += better(mys[e], myi[e], cs, ci) ? 1 : 0;
        pos = __reduce_add_sync(0xffffffffu, pos);
        const int top = min(cnt, n - 1) - 1;   // entries [pos, top] move up by one
        for (int hi = top; hi >= pos; hi -= 32) {
          const int e = hi - lane;
          float vs = 0.f;
          int32_t vi = 0;
          const bool mv = e >= pos;
          if (mv) {
            vs = mys[e];
            vi = myi[e];
          }
          __syncwarp();
          if (mv) {
            mys[e + 1] = vs;
            myi[e + 1] = vi;
          }
          __syncwarp();
        }
        if (lane == 0) {
          mys[pos] = cs;
          myi[pos] = ci;
        }
        __syncwarp();
        cnt = min(cnt + 1, n);
      }
    }
    if (live)
      for (int e = lane; e < n; e += 32) {
        idx_out[q * n + e] = e < cnt ? myi[e] : -1;
        score_out[q * n + e] = e < cnt ? mys[e] : __int_as_float(0x7fc00000);
      }
  }
}

void release(DevBuf& b) {
  if (b.p) cudaFreeAsync(b.p, b.s);
  b.p = nullptr;
}

int grid_cap(const b2k_ctx* ctx, int per_sm) {
  int cap = ctx->sm_count * per_sm;
  if (ctx->grid_limit > 0 && ctx->grid_limit < cap) cap = ctx->grid_limit;
  return std::max(1, cap);
}

int blocks_for(int64_t n, int threads = 256) {
  return (int)std::max<int64_t>(1, std::min<int64_t>((n + threads - 1) / threads, 65536));
}

// one side of the ratings as its owner keeps them
struct Side {
  int64_t d0 = 0, nd = 0;     // owned destinations [d0, d0 + nd) (dense)
  int64_t m = 0;              // ratings
  DevBuf src_b, r_b, units_b, uofs_b;
  int32_t* src = nullptr;     // [m] source dense index
  float* r = nullptr;         // [m]
  Unit* units = nullptr;      // [nunits]
  int64_t* uofs = nullptr;    // [nd + 1] first unit of each destination
  std::vector<int64_t> h_uofs;
};

struct Timing {
  cudaEvent_t ev[8] = {};
  bool on = false;
  double normal = 0, solve = 0, gather = 0, gram = 0;
  explicit Timing(bool enable) : on(enable) {
    if (on)
      for (auto& e : ev) cudaEventCreate(&e);
  }
  ~Timing() {
    if (on)
      for (auto& e : ev) cudaEventDestroy(e);
  }
  void mark(int i, cudaStream_t s) {
    if (on) cudaEventRecord(ev[i], s);
  }
  double ms(int a, int b) const {
    float t = 0.f;
    if (on) cudaEventElapsedTime(&t, ev[a], ev[b]);
    return (double)t;
  }
};

// sorted distinct ids over every rank: a local sort-unique, an allgather of the lists (padded to the longest), then a
// sort-unique of their concatenation
int id_map(b2k_ctx* ctx, const int32_t* v, int64_t n, DevBuf& out_b, int32_t** out, int64_t* m_out, cudaStream_t s) {
  const int R = ctx->nranks;
  DevBuf a_b, b_b, tmp_b, cnt_b, g_b, gc_b, ci_b;
  int32_t *a, *b;
  int64_t* cnt;
  int* ci;
  const int64_t nn = std::max<int64_t>(n, 1);
  B2K_TRY(dalloc(ctx, a_b, nn, s, &a));
  B2K_TRY(dalloc(ctx, b_b, nn, s, &b));
  B2K_TRY(dalloc(ctx, cnt_b, 1 + (size_t)R, s, &cnt));
  B2K_TRY(dalloc(ctx, ci_b, 1, s, &ci));
  size_t sb = 0, ub = 0;
  B2K_CUDA_OK(ctx, cub::DeviceRadixSort::SortKeys(nullptr, sb, v, a, (int)nn, 0, 32, s));
  B2K_CUDA_OK(ctx, cub::DeviceSelect::Unique(nullptr, ub, a, b, ci, (int)nn, s));
  char* tmp;
  B2K_TRY(dalloc(ctx, tmp_b, std::max(sb, ub), s, &tmp));
  int64_t local_u = 0;
  if (n > 0) {
    B2K_CUDA_OK(ctx, cub::DeviceRadixSort::SortKeys(tmp, sb, v, a, (int)n, 0, 32, s));
    B2K_CUDA_OK(ctx, cub::DeviceSelect::Unique(tmp, ub, a, b, ci, (int)n, s));
    int c = 0;
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(&c, ci, 4, cudaMemcpyDeviceToHost, s));
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
    local_u = c;
  }
  std::vector<int64_t> counts(R, local_u);
  if (R > 1) {
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(cnt, &local_u, 8, cudaMemcpyHostToDevice, s));
    B2K_TRY(b2k_comm_allgather_i64(ctx, cnt, cnt + 1, 1, s));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(counts.data(), cnt + 1, 8 * (size_t)R, cudaMemcpyDeviceToHost, s));
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  }
  int64_t mx = 0, tot = 0;
  for (int64_t c : counts) {
    mx = std::max(mx, c);
    tot += c;
  }
  int32_t *g, *gc;
  B2K_TRY(dalloc(ctx, g_b, (size_t)std::max<int64_t>(1, mx) * R, s, &g));
  B2K_TRY(dalloc(ctx, gc_b, (size_t)std::max<int64_t>(1, tot), s, &gc));
  if (R > 1) {
    if (local_u > 0)
      B2K_CUDA_OK(ctx, cudaMemcpyAsync(g + (size_t)ctx->rank * mx, b, 4 * local_u, cudaMemcpyDeviceToDevice, s));
    B2K_TRY(b2k_comm_allgather_bytes(ctx, g + (size_t)ctx->rank * mx, g, 4 * (size_t)std::max<int64_t>(1, mx), s));
    int64_t o = 0;
    for (int q = 0; q < R; ++q) {
      if (counts[q] > 0)
        B2K_CUDA_OK(ctx, cudaMemcpyAsync(gc + o, g + (size_t)q * mx, 4 * counts[q], cudaMemcpyDeviceToDevice, s));
      o += counts[q];
    }
  } else if (tot > 0) {
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(gc, b, 4 * tot, cudaMemcpyDeviceToDevice, s));
  }
  B2K_TRY(dalloc(ctx, out_b, (size_t)std::max<int64_t>(1, tot), s, out));
  int64_t m = 0;
  if (tot > 0) {
    DevBuf t2_b, srt_b;
    int32_t* srt;
    B2K_TRY(dalloc(ctx, srt_b, (size_t)tot, s, &srt));
    size_t sb2 = 0, ub2 = 0;
    B2K_CUDA_OK(ctx, cub::DeviceRadixSort::SortKeys(nullptr, sb2, gc, srt, (int)tot, 0, 32, s));
    B2K_CUDA_OK(ctx, cub::DeviceSelect::Unique(nullptr, ub2, srt, *out, ci, (int)tot, s));
    char* t2;
    B2K_TRY(dalloc(ctx, t2_b, std::max(sb2, ub2), s, &t2));
    B2K_CUDA_OK(ctx, cub::DeviceRadixSort::SortKeys(t2, sb2, gc, srt, (int)tot, 0, 32, s));
    B2K_CUDA_OK(ctx, cub::DeviceSelect::Unique(t2, ub2, srt, *out, ci, (int)tot, s));
    int c = 0;
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(&c, ci, 4, cudaMemcpyDeviceToHost, s));
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
    m = c;
  }
  *m_out = m;
  return B2K_OK;
}

// Sort an owner's ratings by (dst, src, global row) and lay out its units.
int build_side(b2k_ctx* ctx, DevBuf& rec_b, int64_t m, Side* S, cudaStream_t s) {
  OwnRec* rec = static_cast<OwnRec*>(rec_b.p);
  S->m = m;
  const int64_t mm = std::max<int64_t>(m, 1);
  DevBuf k1_b, k2_b, i1_b, i2_b, tmp_b, dst_b, ptr_b;
  unsigned long long *k1, *k2;
  int32_t *i1, *i2, *dst;
  B2K_TRY(dalloc(ctx, k1_b, mm, s, &k1));
  B2K_TRY(dalloc(ctx, k2_b, mm, s, &k2));
  B2K_TRY(dalloc(ctx, i1_b, mm, s, &i1));
  B2K_TRY(dalloc(ctx, i2_b, mm, s, &i2));
  size_t tb = 0;
  B2K_CUDA_OK(ctx, cub::DeviceRadixSort::SortPairs(nullptr, tb, k1, k2, i1, i2, (int)mm, 0, 64, s));
  char* tmp;
  B2K_TRY(dalloc(ctx, tmp_b, tb, s, &tmp));
  B2K_TRY(dalloc(ctx, S->src_b, mm, s, &S->src));
  B2K_TRY(dalloc(ctx, S->r_b, mm, s, &S->r));
  B2K_TRY(dalloc(ctx, dst_b, mm, s, &dst));
  if (m > 0) {
    // stable: by global row first, then by (dst, src)
    k_als_keys<<<blocks_for(m), 256, 0, s>>>(rec, nullptr, m, S->d0, k1, i1);
    B2K_CUDA_OK(ctx, cub::DeviceRadixSort::SortPairs(tmp, tb, k1, k2, i1, i2, (int)m, 0, 64, s));
    k_als_keys<<<blocks_for(m), 256, 0, s>>>(rec, i2, m, S->d0, k1, i1);
    B2K_CUDA_OK(ctx, cub::DeviceRadixSort::SortPairs(tmp, tb, k1, k2, i1, i2, (int)m, 0, 62, s));
    k_als_unpack<<<blocks_for(m), 256, 0, s>>>(rec, i2, m, S->d0, dst, S->src, S->r);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches += 3;
  }
  int64_t* ptr;
  B2K_TRY(dalloc(ctx, ptr_b, (size_t)S->nd + 1, s, &ptr));
  k_als_ptr<<<blocks_for(S->nd + 1), 256, 0, s>>>(dst, m, S->nd, ptr);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  std::vector<int64_t> hp((size_t)S->nd + 1);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(hp.data(), ptr, 8 * hp.size(), cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  std::vector<Unit> units;
  S->h_uofs.assign((size_t)S->nd + 1, 0);
  for (int64_t k = 0; k < S->nd; ++k) {
    S->h_uofs[k] = (int64_t)units.size();
    for (int64_t b = hp[k]; b < hp[k + 1]; b += ALS_UNIT) units.push_back(Unit{b, std::min(hp[k + 1], b + ALS_UNIT)});
  }
  S->h_uofs[S->nd] = (int64_t)units.size();
  B2K_TRY(dalloc(ctx, S->units_b, std::max<size_t>(1, units.size()), s, &S->units));
  B2K_TRY(dalloc(ctx, S->uofs_b, (size_t)S->nd + 1, s, &S->uofs));
  if (!units.empty())
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(S->units, units.data(), units.size() * sizeof(Unit), cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(S->uofs, S->h_uofs.data(), 8 * S->h_uofs.size(), cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));   // the host vectors die with this frame
  return B2K_OK;
}

template <int NT, int MAXT, int RPM>
int launch_normal_t(b2k_ctx* ctx, bool impl, const float* Y, int rank, int rp, const Side& S, int u0, int nu,
                    double alpha, double* part, cudaStream_t s) {
  const int grid = std::min(nu, grid_cap(ctx, 8));
  if (impl)
    k_als_normal<NT, MAXT, RPM, true><<<grid, NT, 0, s>>>(Y, rank, rp, S.src, S.r, S.units + u0, nu, alpha, part);
  else
    k_als_normal<NT, MAXT, RPM, false><<<grid, NT, 0, s>>>(Y, rank, rp, S.src, S.r, S.units + u0, nu, alpha, part);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  return B2K_OK;
}

int launch_normal(b2k_ctx* ctx, bool impl, const float* Y, int rank, int rp, const Side& S, int u0, int nu,
                  double alpha, double* part, cudaStream_t s) {
  if (rp <= 16) return launch_normal_t<64, 1, 16>(ctx, impl, Y, rank, rp, S, u0, nu, alpha, part, s);
  if (rp <= 32) return launch_normal_t<64, 1, 32>(ctx, impl, Y, rank, rp, S, u0, nu, alpha, part, s);
  if (rp <= 64) return launch_normal_t<160, 1, 64>(ctx, impl, Y, rank, rp, S, u0, nu, alpha, part, s);
  return launch_normal_t<192, 3, 128>(ctx, impl, Y, rank, rp, S, u0, nu, alpha, part, s);
}

// owners of a dense range of m entries over R ranks: [m q / R, m (q + 1) / R)
inline int64_t own_lo(int64_t m, int q, int R) { return m * q / R; }

// One half-step: solve the destinations of side D from the full source table Ys [ns][rank] into Yd [*][rank], then
// allgather the solved rows so that every rank holds the whole of Yd.
int half_step(b2k_ctx* ctx, const Side& D, int64_t n_dst_total, const float* Ys, int64_t ns, float* Yd, int rank,
              bool impl, double reg, double alpha, double* YtY, double* part, int64_t part_units, int32_t* bad,
              double* nbad_dev, float* gbuf, Timing& tm, const char* what, cudaStream_t s) {
  const int rp = (rank + 3) / 4 * 4;
  tm.mark(0, s);
  if (impl) B2K_TRY(b2k_gram_local_impl(ctx, Ys, ns, rank, YtY, s));
  tm.mark(1, s);
  double t_normal = 0, t_solve = 0;
  int64_t k = 0;
  while (k < D.nd) {   // batches of whole destinations whose units fit the partial buffer
    int64_t k1 = k + 1;
    while (k1 < D.nd && D.h_uofs[k1 + 1] - D.h_uofs[k] <= part_units) ++k1;
    const int64_t u0 = D.h_uofs[k], nu = D.h_uofs[k1] - u0;
    tm.mark(2, s);
    B2K_TRY(launch_normal(ctx, impl, Ys, rank, rp, D, (int)u0, (int)nu, alpha, part, s));
    tm.mark(3, s);
    const size_t smem = ((size_t)rank * (rank + 1)) * 8;
    B2K_CUDA_OK(ctx, cudaFuncSetAttribute(k_als_solve, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int grid = (int)std::min<int64_t>(k1 - k, grid_cap(ctx, 16));
    k_als_solve<<<grid, ALS_SOLVE_NT, smem, s>>>(part, D.uofs, (int)k, (int)(k1 - k), u0, rank, rp, impl ? YtY : nullptr,
                                                 reg, Yd + D.d0 * rank, bad);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
    tm.mark(4, s);
    if (tm.on) {
      B2K_CUDA_OK(ctx, cudaEventSynchronize(tm.ev[4]));
      t_normal += tm.ms(2, 3);
      t_solve += tm.ms(3, 4);
    }
    k = k1;
  }
  k_als_count<<<1, 256, 0, s>>>(bad, D.nd, nbad_dev);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  B2K_TRY(b2k_comm_allreduce_f64(ctx, nbad_dev, 1, s));
  double nbad = 0;
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(&nbad, nbad_dev, 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  if (nbad > 0)
    return b2k_fail(ctx, B2K_ERR_INVALID, "ALS: the normal equations of " + std::to_string((int64_t)nbad) + " " + what +
                                              " are not positive definite (the Cholesky solve failed; regParam = 0 "
                                              "with fewer ratings than rank?)");
  tm.mark(5, s);
  const int R = ctx->nranks;
  if (R > 1) {
    const int64_t mx = (n_dst_total + R - 1) / R + 1;   // most rows a rank owns
    const size_t row = (size_t)rank * 4;
    if (D.nd > 0)
      B2K_CUDA_OK(ctx, cudaMemcpyAsync(gbuf + (size_t)ctx->rank * mx * rank, Yd + D.d0 * rank, row * D.nd,
                                       cudaMemcpyDeviceToDevice, s));
    B2K_TRY(b2k_comm_allgather_bytes(ctx, gbuf + (size_t)ctx->rank * mx * rank, gbuf, row * mx, s));
    for (int q = 0; q < R; ++q) {
      const int64_t lo = own_lo(n_dst_total, q, R), hi = own_lo(n_dst_total, q + 1, R);
      if (hi > lo)
        B2K_CUDA_OK(ctx, cudaMemcpyAsync(Yd + lo * rank, gbuf + (size_t)q * mx * rank, row * (hi - lo),
                                         cudaMemcpyDeviceToDevice, s));
    }
  }
  tm.mark(6, s);
  if (tm.on) {
    B2K_CUDA_OK(ctx, cudaEventSynchronize(tm.ev[6]));
    tm.gram += tm.ms(0, 1);
    tm.normal += t_normal;
    tm.solve += t_solve;
    tm.gather += tm.ms(5, 6);
  }
  return B2K_OK;
}

std::string fmt_value(double v) {
  if (v != v) return "NaN";
  char buf[64];
  if (v == std::floor(v) && std::fabs(v) < 1e18) std::snprintf(buf, sizeof buf, "%.1f", v);
  else std::snprintf(buf, sizeof buf, "%.17g", v);
  return buf;
}

}  // namespace

int b2k_als_fit_impl(b2k_ctx* ctx, const double* users, const double* items, const float* ratings, int64_t n,
                     int rank, int max_iter, double reg_param, int implicit_prefs, double alpha, uint64_t seed,
                     const float* init_user_factors, int64_t init_n_users, int64_t user_cap, int64_t item_cap,
                     int32_t* user_ids_out, float* user_factors_out, int32_t* item_ids_out, float* item_factors_out,
                     int64_t* n_users_out, int64_t* n_items_out, cudaStream_t s) {
  using clk = std::chrono::steady_clock;
  const auto t_begin = clk::now();
  const int R = ctx->nranks, me = ctx->rank;
  const int64_t nn = std::max<int64_t>(n, 1);
  // ---- check and convert the triples; gather sizes and the first bad row of each kind from every rank ----
  DevBuf u_b, i_b, r_b, bad_b, info_b;
  int32_t *u32, *i32;
  float* r32;
  B2K_TRY(dalloc(ctx, u_b, nn, s, &u32));
  B2K_TRY(dalloc(ctx, i_b, nn, s, &i32));
  B2K_TRY(dalloc(ctx, r_b, nn, s, &r32));
  const int nblk = (int)std::max<int64_t>(1, std::min<int64_t>(1024, (n + 255) / 256));
  const int64_t per = std::max<int64_t>(1, (n + nblk - 1) / nblk);
  int64_t* bad;
  B2K_TRY(dalloc(ctx, bad_b, (size_t)nblk * 3, s, &bad));
  std::vector<int64_t> hb((size_t)nblk * 3, INT64_MAX);
  if (n > 0) {
    k_als_check<<<nblk, 256, 0, s>>>(users, items, ratings, n, per, u32, i32, r32, bad);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(hb.data(), bad, 8 * hb.size(), cudaMemcpyDeviceToHost, s));
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  }
  // info per rank: [n, bad kind (-1 none), bad value bits]
  int64_t info[3] = {n, -1, 0};
  for (int kind = 0; kind < 3 && info[1] < 0; ++kind) {
    int64_t row = INT64_MAX;
    for (int b = 0; b < nblk; ++b) row = std::min(row, hb[(size_t)b * 3 + kind]);
    if (row == INT64_MAX) continue;
    info[1] = kind;
    double v = 0;
    if (kind < 2) {
      B2K_CUDA_OK(ctx, cudaMemcpy(&v, (kind == 0 ? users : items) + row, 8, cudaMemcpyDeviceToHost));
    } else {
      float f = 0;
      B2K_CUDA_OK(ctx, cudaMemcpy(&f, ratings + row, 4, cudaMemcpyDeviceToHost));
      v = f;
    }
    std::memcpy(&info[2], &v, 8);
  }
  int64_t* dinfo;
  B2K_TRY(dalloc(ctx, info_b, 3 + 3 * (size_t)R, s, &dinfo));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(dinfo, info, 24, cudaMemcpyHostToDevice, s));
  B2K_TRY(b2k_comm_allgather_i64(ctx, dinfo, dinfo + 3, 3, s));
  std::vector<int64_t> all(3 * (size_t)R);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(all.data(), dinfo + 3, 24 * (size_t)R, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  std::vector<int64_t> offs(R + 1, 0);
  for (int q = 0; q < R; ++q) offs[q + 1] = offs[q] + all[3 * (size_t)q];
  for (int q = 0; q < R; ++q) {
    const int64_t kind = all[3 * (size_t)q + 1];
    if (kind < 0) continue;
    double v;
    std::memcpy(&v, &all[3 * (size_t)q + 2], 8);
    if (kind < 2)
      return b2k_fail(ctx, B2K_ERR_INVALID,
                      std::string("ALS only supports values in Integer range and without fractional part for column ") +
                          (kind == 0 ? "user" : "item") + ". Value " + fmt_value(v) +
                          " was either out of Integer range or contained a fractional part that could not be "
                          "converted.");
    return b2k_fail(ctx, B2K_ERR_INVALID, "ALS only supports finite ratings; rating " + fmt_value(v) +
                                              " is not finite (rank " + std::to_string(q) + ")");
  }
  const int64_t n_total = offs[R];
  if (n_total == 0) return b2k_fail(ctx, B2K_ERR_INVALID, "ALS: the dataset has no ratings");
  if (init_user_factors && init_n_users < 0) return b2k_fail(ctx, B2K_ERR_INVALID, "ALS: bad init_n_users");

  // ---- id maps, caps ----
  DevBuf uid_b, iid_b;
  int32_t *uid, *iid;
  int64_t U = 0, I = 0;
  B2K_TRY(id_map(ctx, u32, n, uid_b, &uid, &U, s));
  B2K_TRY(id_map(ctx, i32, n, iid_b, &iid, &I, s));
  *n_users_out = U;
  *n_items_out = I;
  if (init_user_factors && init_n_users != U)
    return b2k_fail(ctx, B2K_ERR_INVALID, "ALS: the start factors have " + std::to_string(init_n_users) +
                                              " users, the ratings " + std::to_string(U));
  {   // every rank fails together when one rank's output is too small
    DevBuf f_b;
    double* f;
    B2K_TRY(dalloc(ctx, f_b, 1, s, &f));
    const double small = (U > user_cap || I > item_cap) ? 1.0 : 0.0;
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(f, &small, 8, cudaMemcpyHostToDevice, s));
    B2K_TRY(b2k_comm_allreduce_f64(ctx, f, 1, s));
    double any = 0;
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(&any, f, 8, cudaMemcpyDeviceToHost, s));
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
    if (any > 0)
      return b2k_fail(ctx, B2K_ERR_INVALID, "ALS: the outputs hold fewer rows than the " + std::to_string(U) +
                                                " users / " + std::to_string(I) + " items (on some rank)");
  }
  if (n > 0) {
    k_als_dense<<<blocks_for(n), 256, 0, s>>>(u32, i32, n, uid, U, iid, I);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
  }

  // ---- redistribute: each rank keeps the ratings of the users and items it owns ----
  Side US, IS;
  US.d0 = own_lo(U, me, R);
  US.nd = own_lo(U, me + 1, R) - US.d0;
  IS.d0 = own_lo(I, me, R);
  IS.nd = own_lo(I, me + 1, R) - IS.d0;
  {
    int64_t mx = 0;
    for (int q = 0; q < R; ++q) mx = std::max(mx, all[3 * (size_t)q]);
    const int64_t G = std::max<int64_t>(256, std::min<int64_t>(ALS_GATHER, (mx + 255) / 256 * 256));
    const int64_t rounds = (mx + G - 1) / G;
    const size_t slots = (size_t)R * G;
    DevBuf send_b, recv_b, cu_b, ci_b, fu_b, fi_b, sel_b, offs_b, tmp_b, cnt_b, ou_b, oi_b;
    Rec *send, *recv;
    OwnRec *cu, *ci, *sel;
    uint8_t *fu, *fi;
    int64_t* doffs;
    int* cnt;
    B2K_TRY(dalloc(ctx, send_b, (size_t)G, s, &send));
    B2K_TRY(dalloc(ctx, recv_b, slots, s, &recv));
    B2K_TRY(dalloc(ctx, cu_b, slots, s, &cu));
    B2K_TRY(dalloc(ctx, ci_b, slots, s, &ci));
    B2K_TRY(dalloc(ctx, sel_b, slots, s, &sel));
    B2K_TRY(dalloc(ctx, fu_b, slots, s, &fu));
    B2K_TRY(dalloc(ctx, fi_b, slots, s, &fi));
    B2K_TRY(dalloc(ctx, offs_b, (size_t)R + 1, s, &doffs));
    B2K_TRY(dalloc(ctx, cnt_b, 1, s, &cnt));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(doffs, offs.data(), 8 * offs.size(), cudaMemcpyHostToDevice, s));
    size_t tb = 0;
    B2K_CUDA_OK(ctx, cub::DeviceSelect::Flagged(nullptr, tb, cu, fu, sel, cnt, (int)slots, s));
    char* tmp;
    B2K_TRY(dalloc(ctx, tmp_b, tb, s, &tmp));
    // the kept ratings grow by doubling (a rank's share is not known before the rounds)
    DevBuf* ob[2] = {&ou_b, &oi_b};
    int64_t cap[2] = {std::max<int64_t>(1, n_total / R + 1), std::max<int64_t>(1, n_total / R + 1)};
    int64_t kept[2] = {0, 0};
    for (int side = 0; side < 2; ++side) {
      OwnRec* p;
      B2K_TRY(dalloc(ctx, *ob[side], (size_t)cap[side], s, &p));
    }
    for (int64_t c = 0; c < rounds; ++c) {
      k_als_pack<<<(int)(G / 256), 256, 0, s>>>(u32, i32, r32, c * G, n, G, send);
      B2K_CUDA_OK(ctx, cudaGetLastError());
      B2K_TRY(b2k_comm_allgather_bytes(ctx, send, recv, sizeof(Rec) * (size_t)G, s));
      k_als_own<<<(int)(slots / 256), 256, 0, s>>>(recv, R, G, doffs, c, US.d0, US.d0 + US.nd, IS.d0, IS.d0 + IS.nd, cu,
                                                   ci, fu, fi);
      B2K_CUDA_OK(ctx, cudaGetLastError());
      ctx->stats.kernel_launches += 2;
      for (int side = 0; side < 2; ++side) {
        B2K_CUDA_OK(ctx, cub::DeviceSelect::Flagged(tmp, tb, side ? ci : cu, side ? fi : fu, sel, cnt, (int)slots, s));
        int got = 0;
        B2K_CUDA_OK(ctx, cudaMemcpyAsync(&got, cnt, 4, cudaMemcpyDeviceToHost, s));
        B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
        if (kept[side] + got > cap[side]) {
          DevBuf nb;
          OwnRec* p;
          const int64_t nc = std::max(2 * cap[side], kept[side] + got);
          B2K_TRY(dalloc(ctx, nb, (size_t)nc, s, &p));
          if (kept[side] > 0)
            B2K_CUDA_OK(ctx, cudaMemcpyAsync(p, ob[side]->p, sizeof(OwnRec) * kept[side], cudaMemcpyDeviceToDevice, s));
          std::swap(ob[side]->p, nb.p);
          cap[side] = nc;
        }
        if (got > 0)
          B2K_CUDA_OK(ctx, cudaMemcpyAsync(static_cast<OwnRec*>(ob[side]->p) + kept[side], sel, sizeof(OwnRec) * got,
                                           cudaMemcpyDeviceToDevice, s));
        kept[side] += got;
      }
    }
    B2K_TRY(build_side(ctx, ou_b, kept[0], &US, s));
    B2K_TRY(build_side(ctx, oi_b, kept[1], &IS, s));
  }
  for (DevBuf* b : {&u_b, &i_b, &r_b}) release(*b);
  const double t_setup = std::chrono::duration<double, std::milli>(clk::now() - t_begin).count();

  // ---- factor tables, start ----
  DevBuf uf_b, if_b, ytY_b, part_b, bad_b2, nbad_b, g_b;
  float *UF, *IF, *gbuf = nullptr;
  double *YtY, *part, *nbad;
  int32_t* sbad;
  B2K_TRY(dalloc(ctx, uf_b, (size_t)U * rank, s, &UF));
  B2K_TRY(dalloc(ctx, if_b, (size_t)I * rank, s, &IF));
  B2K_TRY(dalloc(ctx, ytY_b, (size_t)rank * (rank + 1) / 2, s, &YtY));
  B2K_TRY(dalloc(ctx, bad_b2, (size_t)std::max<int64_t>(1, std::max(US.nd, IS.nd)), s, &sbad));
  B2K_TRY(dalloc(ctx, nbad_b, 1, s, &nbad));
  if (R > 1) B2K_TRY(dalloc(ctx, g_b, (size_t)R * ((std::max(U, I) + R - 1) / R + 1) * rank, s, &gbuf));
  const int rp = (rank + 3) / 4 * 4;
  const int64_t PS = (int64_t)(rp / 4) * (rp / 4 + 1) / 2 * 16 + rp + 1;
  int64_t max_units = std::max(US.h_uofs.back(), IS.h_uofs.back());
  const int64_t part_units = std::max<int64_t>(1, std::min<int64_t>(max_units, (int64_t)(ALS_PART_BYTES / (8 * PS))));
  int64_t need_units = part_units;   // a single destination's units always fit one batch
  for (const Side* S : {&US, &IS})
    for (int64_t k = 0; k < S->nd; ++k) need_units = std::max(need_units, S->h_uofs[k + 1] - S->h_uofs[k]);
  B2K_TRY(dalloc(ctx, part_b, (size_t)need_units * PS, s, &part));
  if (init_user_factors) {
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(UF, init_user_factors, (size_t)U * rank * 4, cudaMemcpyHostToDevice, s));
  } else {
    k_als_start<<<blocks_for(U, 128), 128, 0, s>>>(uid, U, rank, seed, UF);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
  }

  // ---- iterations: items from users, then users from items ----
  Timing tm(ctx->time_kernels != 0);
  const bool impl = implicit_prefs != 0;
  for (int it = 0; it < max_iter; ++it) {
    B2K_TRY(half_step(ctx, IS, I, UF, U, IF, rank, impl, reg_param, alpha, YtY, part, part_units, sbad, nbad, gbuf, tm,
                      "items", s));
    B2K_TRY(half_step(ctx, US, U, IF, I, UF, rank, impl, reg_param, alpha, YtY, part, part_units, sbad, nbad, gbuf, tm,
                      "users", s));
  }
  if (max_iter == 0) B2K_CUDA_OK(ctx, cudaMemsetAsync(IF, 0, (size_t)I * rank * 4, s));

  // ---- outputs ----
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(user_ids_out, uid, 4 * (size_t)U, cudaMemcpyDeviceToDevice, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(item_ids_out, iid, 4 * (size_t)I, cudaMemcpyDeviceToDevice, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(user_factors_out, UF, 4 * (size_t)U * rank, cudaMemcpyDeviceToDevice, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(item_factors_out, IF, 4 * (size_t)I * rank, cudaMemcpyDeviceToDevice, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  ctx->stats.last_n_iter = max_iter;
  ctx->stats.last_path = B2K_PATH_GENERIC;
  if (tm.on) {
    const double hs = std::max(1, 2 * max_iter);
    ctx->stats.last_fused_ms = tm.normal / hs;
    ctx->stats.last_finalize_ms = tm.solve / hs;
    ctx->stats.last_allreduce_ms = tm.gather / hs;
    ctx->stats.last_reduce_ms = tm.gram / hs;
    ctx->stats.last_probe_ms = t_setup;
    ctx->stats.last_loop_ms = std::chrono::duration<double, std::milli>(clk::now() - t_begin).count();
  }
  return B2K_OK;
}

int b2k_als_predict_impl(b2k_ctx* ctx, const double* users, const double* items, int64_t n, int rank,
                         const int32_t* user_ids, const float* user_factors, int64_t n_users, const int32_t* item_ids,
                         const float* item_factors, int64_t n_items, float* out, cudaStream_t s) {
  if (n == 0) return B2K_OK;
  k_als_predict<<<blocks_for(n), 256, 0, s>>>(users, items, n, rank, user_ids, user_factors, n_users, item_ids,
                                              item_factors, n_items, out);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  return B2K_OK;
}

int b2k_als_recommend_impl(b2k_ctx* ctx, const float* Q, int64_t nq, const float* T, int64_t nt, int rank, int n,
                           int32_t* idx_out, float* score_out, cudaStream_t s) {
  if (nq == 0) return B2K_OK;
  const size_t smem = ((size_t)32 * (rank + 1) + (size_t)ALS_REC_WARPS * rank + (size_t)ALS_REC_WARPS * n * 2) * 4;
  B2K_CUDA_OK(ctx, cudaFuncSetAttribute(k_als_recommend, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int grid = (int)std::min<int64_t>((nq + ALS_REC_WARPS - 1) / ALS_REC_WARPS, grid_cap(ctx, 2));
  k_als_recommend<<<grid, 32 * ALS_REC_WARPS, smem, s>>>(Q, nq, T, nt, rank, n, idx_out, score_out);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  return B2K_OK;
}
