// Silhouette (sm_90a): b2k_silhouette and b2k_silhouette_multi, the metric of Spark's ClusteringEvaluator in its closed
// form, squared Euclidean or cosine, for 1 .. n clusterings (models) of the same rows; b2k_silhouette is the one-model
// case.  Rows y are x (squared Euclidean) or fl32(x / ||x||) with the fp64 norm (cosine: DBSCAN's k_db_normalize rule);
// cosine is then the squared Euclidean silhouette of the y, since ||y - z||^2 = 2 (1 - cos) for unit rows and s is a
// ratio.  Passes:
//
//   ids         per model and rank: a CUB radix sort of (id, row) and a run-length encode -> the local distinct ids
//               ascending, the rows of each (perm) and its row offsets.  Allgather of the sizes, then of the distinct ids
//               (padded to the largest count); the host merges them into the K global ids and maps each local run to its
//               dense index; cid[row] = that index.
//   statistics  per model, one read of X in perm order (k_sil_stats): chunks of SIL_SC sorted rows write, per run they
//               meet, the fp64 sums of y_f and of ||y||^2 as one piece; k_sil_stats_fold adds each run's pieces in chunk
//               order into stat [K][d + 2] = {sum y, sum ||y||^2, N}.  Two integer counters (non-finite values, zero
//               rows) follow; one f64 allreduce.  Then on the device: the shift m = fl32(sum_c sum y / n) (k_sil_shift),
//               and per cluster mu_c, Psi_c = sum ||y||^2 / N_c - ||mu_c||^2 in fp64 and the shifted means fl32(mu_c - m).
//   silhouette  models whose m has the same bits form a shift group; a group's means are packed side by side, and one
//               pass per chunk of at most B2K_SILHOUETTE_MULTI_CHUNK models forms D(i, c) = ||y_i - mu_c||^2 + Psi_c over
//               every cluster c of each model; a = D(i, A) N_A / (N_A - 1), b = min over c != A; s_i; per model,
//               per-CTA fp64 sums of s_i folded in CTA order; one allreduce of [sum s | n] per model.
//     wgmma    (k_sil_wg, 3xTF32): d % 4 == 0, 4 <= d <= 128, 16-byte aligned X.  The tile operand is X itself (TMA);
//              each consumer warp rewrites its 16 rows of the tile in shared memory once per tile as y - m (one fp32
//              rounding) and takes their fp64 norms, so the pipeline of b2k_pair_wg.cuh runs unchanged; the block
//              operand is the hi / lo planes of the shifted means (k_knn_prep over a zero row and the packed means).
//              D = fl32(fl32(n_c - 2 acc) + n_i) + Psi_c in fp32, within the bound of include/b2kmeans.h.
//     generic  (k_sil_generic, SIMT): every shape; D = sum_f (y_f - mu_c,f)^2 + Psi_c in fp64.
// A model's bits do not depend on which models share the call.  No floating-point atomics: integer counters only, every
// fp64 sum in a fixed order for a given grid, so two calls on the same input, rank count and device give the same bits.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_run_length_encode.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "b2k_internal.cuh"

namespace {
#include "b2k_ptx.cuh"
#include "b2k_knn_prep.cuh"
#include "b2k_pair_wg.cuh"

constexpr int SIL_SC = 256;      // sorted rows per statistics chunk
constexpr int ST_NT = 128;       // threads of the statistics kernels (one feature each)
constexpr int SIL_KMAX = B2K_SILHOUETTE_MAX_CLUSTERS;

__device__ __forceinline__ float sil_y(float x, const double* nrm, int64_t row) {
  return nrm != nullptr ? (float)__ddiv_rn((double)x, nrm[row]) : x;
}

// s of one row from its own-cluster and nearest-other mean distances (negative roundings clamp to 0)
__device__ __forceinline__ double sil_s(double d_own, double d_min, double n_own) {
  if (n_own <= 1.0) return 0.0;
  const double a = fmax(d_own, 0.0) * (n_own / (n_own - 1.0));
  const double b = fmax(d_min, 0.0);
  if (a < b) return 1.0 - a / b;
  if (a > b) return b / a - 1.0;
  return 0.0;
}

// ---- ids ----
__global__ void __launch_bounds__(256) k_sil_iota(int32_t* __restrict__ v, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    v[i] = (int32_t)i;
}

// the run of sorted position p: the largest r < nr with roff[r] <= p
__device__ __forceinline__ int sil_run_of(const int64_t* __restrict__ roff, int nr, int64_t p) {
  int lo = 0, hi = nr - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (roff[mid] <= p) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

__global__ void __launch_bounds__(256) k_sil_cid(const int32_t* __restrict__ perm, const int64_t* __restrict__ roff,
                                                 int nr, const int32_t* __restrict__ lmap, int64_t n,
                                                 int32_t* __restrict__ cid) {
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x)
    cid[perm[p]] = lmap[sil_run_of(roff, nr, p)];
}

// ---- statistics ----
// Chunk j = sorted rows [j SIL_SC, (j + 1) SIL_SC); the piece of (chunk j, run r) is row j + r of piece [][d + 1]
// (runs are non-empty, so along the sorted rows every step moves j or r by one): {sum y_f, sum ||y||^2}.  Each thread
// owns one feature per group of ST_NT and adds the chunk's rows in order; ||y||^2 sums over the features of the
// threads (fixed tree) and over the groups (in order).  bad[0] += non-finite values, bad[1] += zero rows (cosine).
template <bool COS>
__global__ void __launch_bounds__(ST_NT) k_sil_stats(const float* __restrict__ X, int64_t n, int d,
                                                     const int32_t* __restrict__ perm,
                                                     const int64_t* __restrict__ roff, int nr,
                                                     double* __restrict__ piece, double* __restrict__ nrm,
                                                     unsigned long long* __restrict__ bad) {
  __shared__ int32_t srow[SIL_SC];
  __shared__ double snrm[SIL_SC];
  __shared__ double red[ST_NT / 32];
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int64_t p0 = (int64_t)blockIdx.x * SIL_SC;
  const int m = (int)min((int64_t)SIL_SC, n - p0);
  for (int i = tid; i < m; i += ST_NT) srow[i] = perm[p0 + i];
  __syncthreads();
  unsigned long long nbad = 0, nzero = 0;
  if (COS) {
    for (int i = tid; i < m; i += ST_NT) {   // k_db_normalize's rule: feature-order fp64 sum, one sqrt
      const float* x = X + (int64_t)srow[i] * d;
      double s = 0.0;
      for (int f = 0; f < d; ++f) s = __dadd_rn(s, __dmul_rn((double)x[f], (double)x[f]));
      const double r = __dsqrt_rn(s);
      snrm[i] = r;
      nrm[srow[i]] = r;
      nzero += r == 0.0;
    }
    __syncthreads();
  }
  const int r0 = sil_run_of(roff, nr, p0);
  for (int f0 = 0; f0 < d; f0 += ST_NT) {
    const int f = f0 + tid;
    const bool fv = f < d;
    int r = r0;
    int64_t rend = roff[r0 + 1];
    double acc = 0.0, q = 0.0;
    auto flush = [&]() {
      double* pc = piece + ((int64_t)blockIdx.x + r) * (d + 1);
      if (fv) pc[f] = acc;
      double t = q;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
      if (lane == 0) red[w] = t;
      __syncthreads();
      if (tid == 0) {
        double s = 0.0;
        for (int k = 0; k < ST_NT / 32; ++k) s += red[k];
        pc[d] = (f0 == 0 ? 0.0 : pc[d]) + s;
      }
      __syncthreads();
    };
    for (int i0 = 0; i0 < m; i0 += 4) {
      float v[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) v[k] = (fv && i0 + k < m) ? X[(int64_t)srow[i0 + k] * d + f] : 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (i0 + k >= m) break;
        if (p0 + i0 + k == rend) {   // uniform over the CTA
          flush();
          ++r;
          rend = roff[r + 1];
          acc = q = 0.0;
        }
        nbad += fv && !isfinite(v[k]);
        const double y = COS ? (double)(float)__ddiv_rn((double)v[k], snrm[i0 + k]) : (double)v[k];
        acc = __dadd_rn(acc, y);
        q = __dadd_rn(q, __dmul_rn(y, y));
      }
    }
    flush();
  }
  if (nbad) atomicAdd(bad, nbad);
  if (nzero) atomicAdd(bad + 1, nzero);
}

// run r's pieces (chunks j0 .. j1) in chunk order -> stat[lmap[r]] = {sum y [d], sum ||y||^2, N}
__global__ void __launch_bounds__(ST_NT) k_sil_stats_fold(const double* __restrict__ piece, const int64_t* __restrict__ roff,
                                                          const int32_t* __restrict__ lmap, int d,
                                                          double* __restrict__ stat) {
  const int r = blockIdx.x;
  const int64_t a = roff[r], b = roff[r + 1];
  const int64_t j0 = a / SIL_SC, j1 = (b - 1) / SIL_SC;
  double* out = stat + (int64_t)lmap[r] * (d + 2);
  for (int e = threadIdx.x; e <= d; e += ST_NT) {
    double s = 0.0;
    for (int64_t j = j0; j <= j1; ++j) s += piece[(j + r) * (d + 1) + e];
    out[e] = s;
  }
  if (threadIdx.x == 0) out[d + 1] = (double)(b - a);
}

__global__ void k_sil_put_counts(const unsigned long long* __restrict__ bad, double* __restrict__ out) {
  if (threadIdx.x < 2) out[threadIdx.x] = (double)bad[threadIdx.x];
}

// m_f = fl32(sum_c sum y_f / n_total): block f, threads over clusters in order, then a fixed tree
__global__ void __launch_bounds__(256) k_sil_shift(const double* __restrict__ stat, int K, int d, double n_total,
                                                   float* __restrict__ shift) {
  __shared__ double red[256];
  const int f = blockIdx.x;
  double s = 0.0;
  for (int c = threadIdx.x; c < K; c += 256) s += stat[(int64_t)c * (d + 2) + f];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) shift[f] = (float)(red[0] / n_total);
}

// per cluster of one model: cnt, mu (fp64), Psi; wgmma: the shifted means fl32(mu - m) into Mz [K][d], fl32(Psi)
__global__ void __launch_bounds__(256) k_sil_means(const double* __restrict__ stat, int K, int d,
                                                   const float* __restrict__ shift, double* __restrict__ cnt,
                                                   double* __restrict__ mu, double* __restrict__ psi,
                                                   float* __restrict__ Mz, float* __restrict__ psi32) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= K) return;
  const double* st = stat + c * (d + 2);
  const double N = st[d + 1];
  double* mu_c = mu != nullptr ? mu + c * d : nullptr;
  float* mz_c = Mz != nullptr ? Mz + c * d : nullptr;
  double m2 = 0.0;
  for (int f = 0; f < d; ++f) {
    const double v = st[f] / N;
    m2 += v * v;
    if (mu_c != nullptr) mu_c[f] = v;
    if (mz_c != nullptr) mz_c[f] = (float)(v - (double)shift[f]);
  }
  const double p = st[d] / N - m2;
  cnt[c] = N;
  psi[c] = p;
  if (psi32 != nullptr) psi32[c] = (float)p;
}

// wgmma: a group's packed means Mz = [zero row; K means]: the zero row, and the k_knn_prep permutation that takes
// plane row c from Mz row c + 1
__global__ void __launch_bounds__(256) k_sil_mperm(int K, int64_t k_pad, int d, float* __restrict__ Mz,
                                                   int32_t* __restrict__ mperm) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c < d) Mz[c] = 0.f;
  if (c < k_pad) mperm[c] = c < K ? (int32_t)(c + 1) : -1;
}

// ---- silhouette pass: the means of several models packed into one column space ----
// A shift group's models are segments [off[j], off[j + 1]) of the packed clusters, in model order, with no padding
// between them (a segment may start inside a block); b2k_silhouette is a group of one model.  A launch serves a chunk
// of at most SIL_MC models; its per (row, model) state lives in shared memory, so its cost does not grow with the
// chunk.  Each (row, cluster) D depends only on the row's tile and that cluster's mean, d_own / d_min are a select and
// a min, and each thread adds its rows' s_i per model in tile order, so a model's bits do not depend on which models
// share the launch.
constexpr int SIL_MC = B2K_SILHOUETTE_MULTI_CHUNK;

struct SilArgs {
  int64_t n;
  int ntiles, d, nm;             // nm: models in this chunk
  int blo, bhi;                  // wgmma: the blocks of means the chunk's segments touch
  const float* X;
  const double* nrm;
  const float* shift;            // wgmma: the group's m [d]
  const float* cnorm;            // wgmma: [packed k_pad]
  const float* psi32;            // wgmma: [packed]
  const double* mu;              // generic: [packed][d]
  const double* psi;             // generic: [packed]
  const double* cnt;             // [packed]
  int off[SIL_MC + 1];           // the chunk's segments, packed columns
  const int32_t* cid[SIL_MC];    // each model's dense cluster of each row [n]
  double* part;                  // per model j, per CTA: part[j grid + CTA]
};

// ---- wgmma ----
constexpr int SIL_OWN = PW_TM * 4 + SIL_MC * PW_TM * 8 + SIL_MC * 64 * 8;   // norms, (d_own, d_min), per-thread sums
template <int NCH>
using SilWgCfg = PairWgCfg<NCH, SIL_OWN>;

__device__ __forceinline__ void sil_bar_consumers() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// Persistent grid, static round-robin over tiles of PW_TM rows; a unit is one tile against the blocks of means the
// chunk touches.  Per model, each thread that adds rows (a quad's first lane) keeps its own sum of s_i; thread j of the
// consumers folds model j's sums in thread order.
template <int NCH, bool COS>
__global__ void __launch_bounds__(PW_NTHREADS, 1)
k_sil_wg(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapHi,
         const __grid_constant__ CUtensorMap mapLo, const __grid_constant__ SilArgs a) {
  using G = SilWgCfg<NCH>;
  constexpr int R = PW_N / 2;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t base = smem_u32(smem_raw);
  const PairWgBars bars = pair_wg_init<G>(base);
  float* snx = reinterpret_cast<float*>(smem_raw + G::OFF_OWN);
  float* st_own = snx + PW_TM;                       // [SIL_MC][PW_TM]
  float* st_min = st_own + SIL_MC * PW_TM;           // [SIL_MC][PW_TM]
  double* sred = reinterpret_cast<double*>(st_min + SIL_MC * PW_TM);   // [SIL_MC][64]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nit = (int)blockIdx.x < a.ntiles ? (a.ntiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;

  if (warp >= 8) {
    if (warp == 8 && elect_one())
      pair_wg_produce<G>(
          base, bars, &mapQ, &mapHi, &mapLo, nit,
          [&](int it) { return PairWgUnit{((int)blockIdx.x + it * (int)gridDim.x) * PW_TM, a.blo, a.bhi}; },
          [](int) { return false; });
    __syncwarp();
    return;
  }

  const int g = warp >> 2, wi = warp & 3;
  const int wr0 = g * 64 + wi * 16;                 // this warp's 16 rows of the tile
  const int rr0 = wr0 + (lane >> 2);                // this thread's rows rr0, rr0 + 8
  const bool lead = (lane & 3) == 0;                 // the quad's four lanes hold the same rows
  double* my_sum = sred + (threadIdx.x >> 2);        // the adding threads in thread order
  if (lead)
    for (int j = 0; j < a.nm; ++j) my_sum[j * 64] = 0.0;
  float acc[R];
  int q = 0;
  for (int it = 0; it < nit; ++it) {
    const int64_t t0 = ((int64_t)blockIdx.x + (int64_t)it * gridDim.x) * PW_TM;
    mbar_wait_nocall(bars.qfull(), (uint32_t)(it & 1));
    // y - m in place (128B swizzle: row r, column cc of chunk c at r 128 + ((cc / 4) ^ (r % 8)) 16 + (cc % 4) 4)
    for (int k = 0; k < 16; ++k) {
      const int r = wr0 + k;
      const int64_t row = t0 + r;
      double s2 = 0.0;
      if (row < a.n) {
        for (int col = lane; col < a.d; col += 32) {
          const int cc = col & 31;
          float* p = reinterpret_cast<float*>(smem_raw + G::OFF_Q + (col >> 5) * G::QBYTES + r * 128 +
                                              ((((cc >> 2) ^ (r & 7))) << 4) + (cc & 3) * 4);
          const float v = sil_y(*p, COS ? a.nrm : nullptr, row) - __ldg(a.shift + col);
          *p = v;
          s2 += (double)v * (double)v;
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s2 += __shfl_xor_sync(0xffffffffu, s2, o);
      if (lane == 0) snx[r] = (float)s2;
    }
    __syncwarp();
    int64_t row[2];
    float nx[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      row[h] = t0 + rr0 + 8 * h;
      nx[h] = snx[rr0 + 8 * h];
      if (lead)
        for (int j = 0; j < a.nm; ++j) {
          st_own[j * PW_TM + rr0 + 8 * h] = -INFINITY;
          st_min[j * PW_TM + rr0 + 8 * h] = INFINITY;
        }
    }
    for (int b = a.blo; b < a.bhi; ++b) {
      pair_wg_block<G>(smem_raw, base, bars, rr0, lane, acc, q);
      // acc[i] is row rr0 + 8 ((i >> 1) & 1), block column 8 (i >> 2) + 2 (lane & 3) + (i & 1)
      const int cb = b * PW_N + 2 * (lane & 3);
      for (int j = 0; j < a.nm; ++j) {   // the segments this block meets (uniform over the CTA)
        const int lo = a.off[j], hi = a.off[j + 1];
        if (hi <= b * PW_N || lo >= (b + 1) * PW_N) continue;
        int own[2];
        float d_own[2], d_min[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          own[h] = row[h] < a.n ? lo + __ldg(a.cid[j] + row[h]) : -1;
          d_own[h] = -INFINITY;
          d_min[h] = INFINITY;
        }
#pragma unroll
        for (int i = 0; i < R; ++i) {
          const int h = (i >> 1) & 1;
          const int c = cb + 8 * (i >> 2) + (i & 1);
          if ((unsigned)(c - lo) >= (unsigned)(hi - lo)) continue;
          const float S = fmaf(-2.f, acc[i], __ldg(a.cnorm + c)) + nx[h];
          const float D = S + __ldg(a.psi32 + c);
          if (c == own[h]) d_own[h] = D;
          else d_min[h] = fminf(d_min[h], D);
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          d_min[h] = fminf(d_min[h], __shfl_xor_sync(0xffffffffu, d_min[h], 1));
          d_min[h] = fminf(d_min[h], __shfl_xor_sync(0xffffffffu, d_min[h], 2));
          d_own[h] = fmaxf(d_own[h], __shfl_xor_sync(0xffffffffu, d_own[h], 1));
          d_own[h] = fmaxf(d_own[h], __shfl_xor_sync(0xffffffffu, d_own[h], 2));
          if (lead) {
            float* po = st_own + j * PW_TM + rr0 + 8 * h;
            float* pm = st_min + j * PW_TM + rr0 + 8 * h;
            *po = fmaxf(*po, d_own[h]);
            *pm = fminf(*pm, d_min[h]);
          }
        }
      }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the rewritten tile before the next TMA write
    __syncwarp();
    if (lane == 0) mbar_arrive(bars.qempty());
    if (lead)
      for (int j = 0; j < a.nm; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (row[h] < a.n) {
            const int own = __ldg(a.cid[j] + row[h]);
            my_sum[j * 64] += sil_s((double)st_own[j * PW_TM + rr0 + 8 * h], (double)st_min[j * PW_TM + rr0 + 8 * h],
                                    __ldg(a.cnt + a.off[j] + own));
          }
  }
  sil_bar_consumers();
  if (threadIdx.x < a.nm) {
    const int j = threadIdx.x;
    double t = 0.0;
    for (int i = 0; i < 64; ++i) t += sred[j * 64 + i];
    a.part[(int64_t)j * gridDim.x + blockIdx.x] = t;
  }
}

// ---- generic: CTA = 64 rows x tiles of 64 of the chunk's packed clusters [off[0], off[nm]); thread (ty, tx) owns rows
// ty + 16 i and clusters tx + 16 j (i, j < 4), fp64 sums over features staged 32 at a time; per model, the first thread
// of each half warp keeps its sum of s_i ----
constexpr int GR = 64, GC = 64, GF = 32, G_NT = 256;
constexpr int SIL_GEN_SMEM = 2 * GF * (GR + 1) * 8 + 2 * SIL_MC * GR * 8 + SIL_MC * 16 * 8;
template <bool COS>
__global__ void __launch_bounds__(G_NT, 1) k_sil_generic(const __grid_constant__ SilArgs a) {
  extern __shared__ __align__(16) uint8_t gsm[];
  double(*xr)[GR + 1] = reinterpret_cast<double(*)[GR + 1]>(gsm);
  double(*mc)[GC + 1] = reinterpret_cast<double(*)[GC + 1]>(gsm + GF * (GR + 1) * 8);
  double* st_own = reinterpret_cast<double*>(gsm + 2 * GF * (GR + 1) * 8);   // [SIL_MC][GR]
  double* st_min = st_own + SIL_MC * GR;                                      // [SIL_MC][GR]
  double* sred = st_min + SIL_MC * GR;                                        // [SIL_MC][16]
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int d = a.d;
  const int cbeg = a.off[0], cend = a.off[a.nm];
  if (tx == 0)
    for (int j = 0; j < a.nm; ++j) sred[j * 16 + ty] = 0.0;
  for (int tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x) {
    int64_t row[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      row[i] = (int64_t)tile * GR + ty + 16 * i;
      if (tx == 0)
        for (int j = 0; j < a.nm; ++j) {
          st_own[j * GR + ty + 16 * i] = -INFINITY;
          st_min[j * GR + ty + 16 * i] = INFINITY;
        }
    }
    for (int c0 = cbeg; c0 < cend; c0 += GC) {
      double acc[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;
      for (int f0 = 0; f0 < d; f0 += GF) {
        __syncthreads();
        for (int e = threadIdx.x; e < GF * GR; e += G_NT) {
          const int r = e / GF, c = e % GF;
          const int64_t gr = (int64_t)tile * GR + r;
          const int f = f0 + c, cl = c0 + r;
          xr[c][r] = (gr < a.n && f < d) ? (double)sil_y(a.X[gr * d + f], COS ? a.nrm : nullptr, gr) : 0.0;
          mc[c][r] = (cl < cend && f < d) ? a.mu[(int64_t)cl * d + f] : 0.0;
        }
        __syncthreads();
        const int fc = min(GF, d - f0);
        for (int c = 0; c < fc; ++c) {
          double vr[4], vc[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) vr[i] = xr[c][ty + 16 * i];
#pragma unroll
          for (int j = 0; j < 4; ++j) vc[j] = mc[c][tx + 16 * j];
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const double t = vr[i] - vc[j];
              acc[i][j] = fma(t, t, acc[i][j]);
            }
        }
      }
      for (int m = 0; m < a.nm; ++m) {   // the segments this tile meets (uniform over the CTA)
        const int lo = a.off[m], hi = a.off[m + 1];
        if (hi <= c0 || lo >= c0 + GC) continue;
        int own[4];
        double d_own[4], d_min[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          own[i] = row[i] < a.n ? lo + a.cid[m][row[i]] : -1;
          d_own[i] = -INFINITY;
          d_min[i] = INFINITY;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int cl = c0 + tx + 16 * j;
          if (cl < lo || cl >= hi) continue;
          const double p = a.psi[cl];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const double D = acc[i][j] + p;
            if (cl == own[i]) d_own[i] = D;
            else d_min[i] = fmin(d_min[i], D);
          }
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
#pragma unroll
          for (int o = 1; o < 16; o <<= 1) {
            d_min[i] = fmin(d_min[i], __shfl_xor_sync(0xffffffffu, d_min[i], o));
            d_own[i] = fmax(d_own[i], __shfl_xor_sync(0xffffffffu, d_own[i], o));
          }
          if (tx == 0) {
            double* po = st_own + m * GR + ty + 16 * i;
            double* pm = st_min + m * GR + ty + 16 * i;
            *po = fmax(*po, d_own[i]);
            *pm = fmin(*pm, d_min[i]);
          }
        }
      }
    }
    if (tx == 0)
      for (int m = 0; m < a.nm; ++m)
#pragma unroll
        for (int i = 0; i < 4; ++i)
          if (row[i] < a.n)
            sred[m * 16 + ty] += sil_s(st_own[m * GR + ty + 16 * i], st_min[m * GR + ty + 16 * i],
                                       a.cnt[a.off[m] + a.cid[m][row[i]]]);
  }
  __syncthreads();
  if (threadIdx.x < a.nm) {
    const int m = threadIdx.x;
    double t = 0.0;
    for (int i = 0; i < 16; ++i) t += sred[m * 16 + i];
    a.part[(int64_t)m * gridDim.x + blockIdx.x] = t;
  }
}

unsigned grid_1d(int64_t n, int sm) {
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, (int64_t)sm * 16));
}
}  // namespace

// One model's cluster ids and statistics: what the silhouette pass needs besides X, and the pass b2k_silhouette runs
struct SilModel {
  int64_t K = 0, n_total = 0;
  bool wg = false;
  DevBuf b_cid, b_nrm, b_stat;
  int32_t* cid = nullptr;   // dense cluster of each row [n]
  double* nrm = nullptr;    // cosine: ||x|| [n]
  double* stat = nullptr;   // [K][d + 2] + 2, allreduced
};

// The ids and statistics passes of one model and every check of b2k_silhouette, in its order.  tm: marks 0 (start) and
// 1 (ids done).
int sil_prepare(b2k_ctx* ctx, const float* X, int64_t n_local, int d, const int64_t* ids, int metric, B2kTimer& tm,
                SilModel& md, cudaStream_t s) {
  const int nr = ctx->nranks;
  const bool cosine = metric == 1;
  const int64_t n = n_local;
  // ---- ids: sort, runs ----
  size_t sort_bytes = 0, rle_bytes = 0, scan_bytes = 0;
  const int ni = (int)std::max<int64_t>(n, 1);
  B2K_CUDA_OK(ctx, cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const int64_t*)nullptr, (int64_t*)nullptr,
                                                   (const int32_t*)nullptr, (int32_t*)nullptr, ni, 0, 64, s));
  B2K_CUDA_OK(ctx, cub::DeviceRunLengthEncode::Encode(nullptr, rle_bytes, (const int64_t*)nullptr, (int64_t*)nullptr,
                                                      (int64_t*)nullptr, (int64_t*)nullptr, ni, s));
  B2K_CUDA_OK(ctx, cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (const int64_t*)nullptr, (int64_t*)nullptr,
                                                 ni + 1, s));
  const size_t tmp_bytes = std::max({sort_bytes, rle_bytes, scan_bytes});
  constexpr int NS = 4;   // n_local, d, distinct ids, X not 16-byte aligned
  int64_t *sz_dev = nullptr, *keys = nullptr, *uniq = nullptr, *rlen = nullptr, *roff = nullptr, *nruns = nullptr;
  int32_t *rows = nullptr, *perm = nullptr, *cid = nullptr;
  double* nrm = nullptr;
  void* tmp = nullptr;
  B2K_TRY(dalloc(ctx, md.b_cid, (size_t)ni, s, &cid));
  if (cosine) B2K_TRY(dalloc(ctx, md.b_nrm, (size_t)ni, s, &nrm));
  B2K_TRY(b2k_scratch_layout(ctx, "silhouette", [&](B2kLayout& L) -> int {
    sz_dev = L.take<int64_t>((size_t)NS * (nr + 1));
    nruns = L.take<int64_t>(1);
    keys = L.take<int64_t>((size_t)ni);
    uniq = L.take<int64_t>((size_t)ni + 1);
    rlen = L.take<int64_t>((size_t)ni + 1);
    roff = L.take<int64_t>((size_t)ni + 2);
    rows = L.take<int32_t>((size_t)ni);
    perm = L.take<int32_t>((size_t)ni);
    tmp = L.take<char>(tmp_bytes);
    return B2K_OK;
  }));
  tm.mark(0, s);
  int64_t kl = 0;
  if (n > 0) {
    k_sil_iota<<<grid_1d(n, ctx->sm_count), 256, 0, s>>>(rows, n);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    size_t b = tmp_bytes;
    B2K_CUDA_OK(ctx, cub::DeviceRadixSort::SortPairs(tmp, b, ids, keys, rows, perm, (int)n, 0, 64, s));
    b = tmp_bytes;
    B2K_CUDA_OK(ctx, cub::DeviceRunLengthEncode::Encode(tmp, b, keys, uniq, rlen, nruns, (int)n, s));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(&kl, nruns, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
    b = tmp_bytes;
    B2K_CUDA_OK(ctx, cub::DeviceScan::ExclusiveSum(tmp, b, rlen, roff, (int)kl + 1, s));
    ctx->stats.kernel_launches += 4;
  }
  const int64_t mine[NS] = {n, d, kl, n > 0 && (reinterpret_cast<uintptr_t>(X) & 15u) != 0};
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(sz_dev, mine, sizeof(mine), cudaMemcpyHostToDevice, s));
  B2K_TRY(b2k_comm_allgather_i64(ctx, sz_dev, sz_dev + NS, NS, s));
  std::vector<int64_t> sz((size_t)NS * nr);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(sz.data(), sz_dev + NS, sz.size() * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  int64_t n_total = 0, k_max = 0, misaligned = 0;
  for (int r = 0; r < nr; ++r) {
    if (sz[NS * r + 1] != sz[1])
      return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_silhouette: d differs between ranks (rank " + std::to_string(r) +
                                                " has d = " + std::to_string(sz[NS * r + 1]) + ", rank 0 has d = " +
                                                std::to_string(sz[1]) + ")");
    n_total += sz[NS * r];
    k_max = std::max(k_max, sz[NS * r + 2]);
    misaligned += sz[NS * r + 3];
  }
  if (metric != 0 && metric != 1)
    return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_silhouette: metric = " + std::to_string(metric) +
                                              " (0 = squaredEuclidean, 1 = cosine)");
  if (n_total == 0) return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_silhouette: no rows on any rank");
  if (n_total > (int64_t)0x7fffffff)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "b2k_silhouette: 2^31 or more rows in all");
  const std::string too_many = "b2k_silhouette: more than " + std::to_string(SIL_KMAX) + " distinct cluster ids";
  if (k_max > SIL_KMAX) return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, too_many);

  // ---- every rank's distinct ids -> the K global ids, ascending; this rank's runs -> dense indices ----
  DevBuf b_ids, b_send;
  int64_t *all_ids = nullptr, *send = nullptr;
  B2K_TRY(dalloc(ctx, b_ids, (size_t)nr * std::max<int64_t>(k_max, 1), s, &all_ids));
  if (nr > 1) {
    B2K_TRY(dalloc(ctx, b_send, (size_t)std::max<int64_t>(k_max, 1), s, &send));   // this rank's ids, padded
    if (kl > 0) B2K_CUDA_OK(ctx, cudaMemcpyAsync(send, uniq, (size_t)kl * 8, cudaMemcpyDeviceToDevice, s));
    B2K_TRY(b2k_comm_allgather_bytes(ctx, send, all_ids, (size_t)std::max<int64_t>(k_max, 1) * 8, s));
  } else if (kl > 0) {
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(all_ids, uniq, (size_t)kl * 8, cudaMemcpyDeviceToDevice, s));
  }
  std::vector<int64_t> got((size_t)nr * std::max<int64_t>(k_max, 1));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(got.data(), all_ids, got.size() * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  std::vector<int64_t> U;
  for (int r = 0; r < nr; ++r)
    U.insert(U.end(), got.begin() + (size_t)r * std::max<int64_t>(k_max, 1),
             got.begin() + (size_t)r * std::max<int64_t>(k_max, 1) + sz[NS * r + 2]);
  std::sort(U.begin(), U.end());
  U.erase(std::unique(U.begin(), U.end()), U.end());
  const int64_t K = (int64_t)U.size();
  if (K > SIL_KMAX) return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, too_many);
  if (K < 2) return b2k_fail(ctx, B2K_ERR_INVALID, "Number of clusters must be greater than one.");
  std::vector<int32_t> lmap_h((size_t)std::max<int64_t>(kl, 1), 0);
  const int64_t* mine_ids = got.data() + (size_t)(nr > 1 ? ctx->rank : 0) * std::max<int64_t>(k_max, 1);
  for (int64_t r = 0; r < kl; ++r)
    lmap_h[r] = (int32_t)(std::lower_bound(U.begin(), U.end(), mine_ids[r]) - U.begin());
  int32_t* lmap = nullptr;
  DevBuf b_lmap;
  B2K_TRY(dalloc(ctx, b_lmap, lmap_h.size(), s, &lmap));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(lmap, lmap_h.data(), lmap_h.size() * 4, cudaMemcpyHostToDevice, s));
  if (n > 0) {
    k_sil_cid<<<grid_1d(n, ctx->sm_count), 256, 0, s>>>(perm, roff, (int)kl, lmap, n, cid);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
  }
  tm.mark(1, s);

  // ---- statistics ----
  const int64_t nch = (n + SIL_SC - 1) / SIL_SC;
  const size_t slen = (size_t)K * (d + 2) + 2;
  DevBuf b_piece;
  double *piece = nullptr, *stat = nullptr;
  B2K_TRY(dalloc(ctx, b_piece, (size_t)std::max<int64_t>(nch + kl, 1) * (d + 1), s, &piece));
  B2K_TRY(dalloc(ctx, md.b_stat, slen, s, &stat));
  unsigned long long* bad = reinterpret_cast<unsigned long long*>(sz_dev);   // the sizes are on the host now
  B2K_CUDA_OK(ctx, cudaMemsetAsync(stat, 0, slen * 8, s));
  B2K_CUDA_OK(ctx, cudaMemsetAsync(bad, 0, 2 * sizeof(unsigned long long), s));
  if (n > 0) {
    if (cosine) k_sil_stats<true><<<(unsigned)nch, ST_NT, 0, s>>>(X, n, d, perm, roff, (int)kl, piece, nrm, bad);
    else k_sil_stats<false><<<(unsigned)nch, ST_NT, 0, s>>>(X, n, d, perm, roff, (int)kl, piece, nrm, bad);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    k_sil_stats_fold<<<(unsigned)kl, ST_NT, 0, s>>>(piece, roff, lmap, d, stat);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches += 2;
  }
  k_sil_put_counts<<<1, 32, 0, s>>>(bad, stat + (size_t)K * (d + 2));
  B2K_CUDA_OK(ctx, cudaGetLastError());
  B2K_TRY(b2k_comm_allreduce_f64(ctx, stat, slen, s));
  double flags[2] = {0.0, 0.0};
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(flags, stat + (size_t)K * (d + 2), sizeof(flags), cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  if (flags[0] > 0) return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_silhouette: features contain NaN or infinity");
  if (cosine && flags[1] > 0)
    return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_silhouette: cosine distance is undefined for a zero row (" +
                                              std::to_string((int64_t)flags[1]) + " such rows)");

  // ---- plan of the silhouette pass ----
  const bool wg_ok = b2k_knn_wg_width(d) && misaligned == 0;   // the same choice on every rank
  if (ctx->kernel_path == B2K_PATH_FUSED && !wg_ok)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "kernel_path=2 requested but the wgmma silhouette pass needs d % 4 == 0, "
                                              "4 <= d <= 128 and 16-byte aligned X (d = " + std::to_string(d) + ")");
  md.wg = wg_ok && ctx->kernel_path != B2K_PATH_GENERIC;
  md.K = K;
  md.n_total = n_total;
  md.cid = cid;
  md.nrm = nrm;
  md.stat = stat;
  return B2K_OK;
}

int b2k_silhouette_impl(b2k_ctx* ctx, const float* X, int64_t n_local, int d, int n_models, const int64_t* const* ids,
                        int metric, double* out, int* failed_model, cudaStream_t s) {
  const bool on = ctx->time_kernels != 0;
  const bool cosine = metric == 1;
  const int64_t n = n_local;
  const int M = n_models;
  double ms_ids = 0.0, ms_stats = 0.0, ms_pass = 0.0, ms_red = 0.0;
  B2kTimer tall(on);
  tall.mark(0, s);

  // ---- per model: ids, statistics and the shift m ----
  std::vector<SilModel> md(M);
  std::vector<DevBuf> b_shift(M);
  std::vector<float*> shift(M, nullptr);
  std::vector<std::vector<float>> shift_h(M, std::vector<float>((size_t)d));
  for (int m = 0; m < M; ++m) {
    B2kTimer tm(on);
    const int rc = sil_prepare(ctx, X, n, d, ids[m], metric, tm, md[m], s);
    if (rc != B2K_OK) {
      if (failed_model != nullptr) *failed_model = m;
      return rc;
    }
    B2K_TRY(dalloc(ctx, b_shift[m], (size_t)d, s, &shift[m]));
    k_sil_shift<<<(unsigned)d, 256, 0, s>>>(md[m].stat, (int)md[m].K, d, (double)md[m].n_total, shift[m]);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(shift_h[m].data(), shift[m], (size_t)d * 4, cudaMemcpyDeviceToHost, s));
    tm.mark(2, s);
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
    ms_ids += tm.ms(0, 1);
    ms_stats += tm.ms(1, 2);
  }
  const bool wg = md[0].wg;   // decided by d, alignment and kernel_path: the same for every model
  int sm = ctx->sm_count;
  if (ctx->grid_limit > 0 && ctx->grid_limit < sm) sm = ctx->grid_limit;
  const int DP = b2k_knn_wg_dp(d);

  // ---- shift groups: models whose m has the same bits share one tile rewrite y - m, so one pass ----
  std::vector<std::vector<int>> groups;
  for (int m = 0; m < M; ++m) {
    bool put = false;
    for (auto& g : groups)
      if (std::memcmp(shift_h[g[0]].data(), shift_h[m].data(), (size_t)d * 4) == 0) {
        g.push_back(m);
        put = true;
        break;
      }
    if (!put) groups.push_back({m});
  }

  int grid = 0;
  int64_t ntiles = 0;
  if (wg) {
    ntiles = (n + PW_TM - 1) / PW_TM;
    grid = (int)std::min<int64_t>(sm, ntiles);
  } else {
    ntiles = (n + GR - 1) / GR;
    grid = (int)std::min<int64_t>(ntiles, (int64_t)sm * (ctx->grid_limit > 0 ? 1 : 8));
  }
  DevBuf b_sum;
  double* sum = nullptr;   // [M][2] = {sum s, n}
  B2K_TRY(dalloc(ctx, b_sum, (size_t)2 * M, s, &sum));
  for (const auto& g : groups) {
    B2kTimer tm(on);
    tm.mark(0, s);
    std::vector<int64_t> off(g.size() + 1, 0);
    for (size_t j = 0; j < g.size(); ++j) off[j + 1] = off[j] + md[g[j]].K;
    const int64_t Kt = off.back();
    const int64_t k_pad = (Kt + PW_N - 1) / PW_N * PW_N;
    DevBuf b_cnt, b_mu, b_psi, b_mz, b_mperm, b_psi32, b_hi, b_lo, b_cn, b_part;
    double *cnt = nullptr, *mu = nullptr, *psi = nullptr, *part = nullptr;
    float *Mz = nullptr, *psi32 = nullptr, *Xhi = nullptr, *Xlo = nullptr, *cnorm = nullptr;
    int32_t* mperm = nullptr;
    B2K_TRY(dalloc(ctx, b_cnt, (size_t)Kt, s, &cnt));
    B2K_TRY(dalloc(ctx, b_psi, (size_t)Kt, s, &psi));
    if (wg) {
      B2K_TRY(dalloc(ctx, b_mz, (size_t)(Kt + 1) * d, s, &Mz));
      B2K_TRY(dalloc(ctx, b_mperm, (size_t)k_pad, s, &mperm));
      B2K_TRY(dalloc(ctx, b_psi32, (size_t)Kt, s, &psi32));
      B2K_TRY(dalloc(ctx, b_hi, (size_t)k_pad * DP, s, &Xhi));
      B2K_TRY(dalloc(ctx, b_lo, (size_t)k_pad * DP, s, &Xlo));
      B2K_TRY(dalloc(ctx, b_cn, (size_t)k_pad, s, &cnorm));
    } else {
      B2K_TRY(dalloc(ctx, b_mu, (size_t)Kt * d, s, &mu));
    }
    for (size_t j = 0; j < g.size(); ++j) {   // model j's means go to Mz rows off[j] + 1 ..
      const SilModel& mj = md[g[j]];
      const int64_t o = off[j];
      k_sil_means<<<(unsigned)((mj.K + 255) / 256), 256, 0, s>>>(
          mj.stat, (int)mj.K, d, shift[g[j]], cnt + o, mu != nullptr ? mu + o * d : nullptr, psi + o,
          Mz != nullptr ? Mz + (o + 1) * d : nullptr, psi32 != nullptr ? psi32 + o : nullptr);
      B2K_CUDA_OK(ctx, cudaGetLastError());
      ctx->stats.kernel_launches++;
    }
    if (wg) {
      k_sil_mperm<<<(unsigned)((std::max<int64_t>(k_pad, d) + 255) / 256), 256, 0, s>>>((int)Kt, k_pad, d, Mz, mperm);
      B2K_CUDA_OK(ctx, cudaGetLastError());
      ctx->stats.kernel_launches++;
    }
    tm.mark(1, s);
    B2K_TRY(dalloc(ctx, b_part, (size_t)std::max(grid, 1) * SIL_MC, s, &part));
    PairWgMaps maps;
    if (wg && grid > 0) {
      B2K_TRY(b2k_knn_prep_launch(ctx, Mz, Kt + 1, d, mperm, k_pad, DP, Xhi, Xlo, cnorm, s));
      B2K_TRY(pair_wg_maps(ctx, X, n, d, Xhi, Xlo, k_pad, DP, &maps));
    }
    for (size_t c0 = 0; c0 < g.size(); c0 += SIL_MC) {
      const int nm = (int)std::min<size_t>(SIL_MC, g.size() - c0);
      SilArgs a{};
      a.n = n;
      a.ntiles = (int)ntiles;
      a.d = d;
      a.nm = nm;
      a.X = X;
      a.nrm = md[g[c0]].nrm;   // every model's norms are the same values of X
      a.shift = shift[g[0]];
      a.cnorm = cnorm;
      a.psi32 = psi32;
      a.mu = mu;
      a.psi = psi;
      a.cnt = cnt;
      for (int j = 0; j <= nm; ++j) a.off[j] = (int)off[c0 + j];
      for (int j = 0; j < nm; ++j) a.cid[j] = md[g[c0 + j]].cid;
      a.blo = (int)(off[c0] / PW_N);
      a.bhi = (int)((off[c0 + nm] + PW_N - 1) / PW_N);
      a.part = part;
      if (grid > 0) {
        if (wg) {
          if (cosine)
            B2K_TRY(pair_wg_launch<SIL_OWN>(
                ctx, DP, [](auto nch) { return k_sil_wg<decltype(nch)::value, true>; }, grid, maps, a, s));
          else
            B2K_TRY(pair_wg_launch<SIL_OWN>(
                ctx, DP, [](auto nch) { return k_sil_wg<decltype(nch)::value, false>; }, grid, maps, a, s));
          ctx->stats.fused_tc_launches++;
        } else {
          const auto k = cosine ? k_sil_generic<true> : k_sil_generic<false>;
          B2K_CUDA_OK(ctx, cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, SIL_GEN_SMEM));
          k<<<(unsigned)grid, G_NT, SIL_GEN_SMEM, s>>>(a);
          B2K_CUDA_OK(ctx, cudaGetLastError());
          ctx->stats.generic_launches++;
        }
        ctx->stats.kernel_launches++;
      }
      for (int j = 0; j < nm; ++j) {
        double* sm_j = sum + 2 * g[c0 + j];
        if (grid > 0) B2K_TRY(b2k_launch_fold_f64(ctx, part + (size_t)j * grid, grid, sm_j, s));
        else B2K_CUDA_OK(ctx, cudaMemsetAsync(sm_j, 0, sizeof(double), s));
      }
    }
    tm.mark(2, s);
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));   // the group's buffers are freed on return of this scope
    ms_stats += tm.ms(0, 1);
    ms_pass += tm.ms(1, 2);
  }
  ctx->stats.last_path = wg ? B2K_PATH_FUSED : B2K_PATH_GENERIC;

  // ---- one [sum s | n] allreduce per model ----
  B2kTimer tr(on);
  tr.mark(0, s);
  const double nd = (double)n;
  std::vector<double> res((size_t)2 * M);
  for (int m = 0; m < M; ++m) {
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(sum + 2 * m + 1, &nd, sizeof(double), cudaMemcpyHostToDevice, s));
    B2K_TRY(b2k_comm_allreduce_f64(ctx, sum + 2 * m, 2, s));
  }
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(res.data(), sum, res.size() * 8, cudaMemcpyDeviceToHost, s));
  tr.mark(1, s);
  tall.mark(1, s);
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  for (int m = 0; m < M; ++m) out[m] = res[2 * m] / res[2 * m + 1];
  if (on) {
    ms_red = tr.ms(0, 1);
    ctx->stats.last_finalize_ms = ms_ids;
    ctx->stats.last_reduce_ms = ms_stats;
    ctx->stats.last_fused_ms = ms_pass;
    ctx->stats.last_allreduce_ms = ms_red;
    ctx->stats.last_loop_ms = tall.ms(0, 1);
  }
  return B2K_OK;
}
