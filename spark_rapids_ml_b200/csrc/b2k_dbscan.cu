// DBSCAN (sm_90a): b2k_dbscan_fit, euclidean or cosine adjacency on float32 rows, decided exactly in fp64.
//
//   sizes    allgather of (n_local, d, non-finite values, zero rows) per rank; every error is decided on those values.
//   rows     allgather of X padded to the largest shard, compacted to Xg [n_total][d] in global row order (one rank:
//            X itself).  Cosine: Y = rows scaled by 1 / ||x|| (fp64 norm, one fp32 rounding) and the fp64 norms.
//   count    counts[i] = |{j : adj(i, j)}| for the local rows i over all rows j, core = counts >= min_samples.
//   cores    allgather of the core flags (n_total bytes).
//   union    over (local row i, core row j) pairs: i core -> lock-free union of i and j in parent[n_total] (the lower root
//            wins, so a root is always its set's lowest row); i not core -> bmin[i] = lowest adjacent core row.
//   merge    compress; allgather of every rank's parent array (nranks * n_total int32); union of every (x, root_r(x));
//            compress.  Every rank then holds the same forest, whose roots are the lowest rows of their components.
//   labels   cluster ids = exclusive prefix count of the core roots; core rows take their root's id, border rows the id
//            of bmin's root, every other row -1.
//
// adj(i, j) is the fp64 rule of include/b2kmeans.h.  Two passes evaluate it:
//   wgmma  (k_db_wg, 3xTF32): d % 4 == 0, 4 <= d <= 128, 16-byte aligned X (one rank).  Rows in the frame of s = global
//          row 0 (k_knn_prep / k_knn_shift_q, shared with k-NN): screen S = n_i + n_j - 2 v_i.v_j.  |S - D| <= B_ij (the
//          bound below), so S < E - B_ij is adjacent, S > E + B_ij is not, and the band between them is decided by the
//          fp64 rule on the caller's rows, inline.
//   generic (k_db_generic, SIMT): every shape; the fp64 rule itself on every pair.
// Labels depend only on the rows in global order: counts are integer sums, the union-find's roots are set minima, and a
// border row's cluster is that of its lowest adjacent core row, so neither the rank count, the shards, the pass nor the
// order of the atomics shows in the output.
#include <algorithm>
#include <cmath>
#include <vector>

#include "b2k_internal.cuh"

namespace {
#include "b2k_ptx.cuh"
#include "b2k_knn_prep.cuh"
#include "b2k_pair_wg.cuh"

constexpr int DB_SMAX = 4096;    // column splits
constexpr int DB_NONE = 0x7fffffff;
constexpr int DB_SNAP = 2 * PW_N * 4 + 2 * PW_N;   // [2][128] column roots, [2][128] column core flags

// d = 128: row tile 64 KB + two column stages 64 KB + snapshots 1.25 KB
template <int NCH>
using DbWgCfg = PairWgCfg<NCH, DB_SNAP>;
static_assert(DbWgCfg<4>::SMEM_BYTES == 128 * 1024 + 1280 + 48, "d = 128 layout");

struct DbArgs {
  int64_t n_local, n_total, row0;
  int ntiles, S, nblk;
  int d, metric;
  float E;                           // threshold of the screen: fl32(eps^2) (euclidean) or fl32(2 eps) (cosine)
  float coef, B0;                    // B_ij = coef (n_i + n_j) + B0
  double eps2;                       // the fp64 rule: eps^2 (euclidean) or eps (cosine)
  const float* X;                    // the caller's rows in global order [n_total][d]
  const double* nrm;                 // cosine: fp64 ||x|| [n_total]
  const float* norms;                // ||v||^2 of the shifted rows, +inf past n_total
  int* counts;                       // count pass: [n_local]
  const uint8_t* core;               // union pass: [n_total]
  const uint8_t* blk_core;           // union pass: column block holds a core row [nblk]
  int* parent;                       // union pass: [n_total]
  int* bmin;                         // union pass: [n_local]
  unsigned long long* stat;          // [2] band pairs decided in fp64, unions attempted (NULL: not collected)
};

// ---- the fp64 rule, in the operation order tests/dbscan_oracle.py restates (no contraction) ----
__device__ __forceinline__ bool db_adjacent(const float* __restrict__ X, const double* __restrict__ nrm, int d,
                                            int metric, double eps2, int64_t i, int64_t j) {
  const float* a = X + i * d;
  const float* b = X + j * d;
  double s = 0.0;
  if (metric == 0) {
    for (int f = 0; f < d; ++f) {
      const double t = __dsub_rn((double)a[f], (double)b[f]);
      s = __dadd_rn(s, __dmul_rn(t, t));
    }
    return s <= eps2;
  }
  for (int f = 0; f < d; ++f) s = __dadd_rn(s, __dmul_rn((double)a[f], (double)b[f]));
  return __dsub_rn(1.0, __ddiv_rn(s, __dmul_rn(nrm[i], nrm[j]))) <= eps2;
}

// ---- lock-free union-find on parent[]: parent[x] <= x always, so the root of a set is its lowest row ----
__device__ __forceinline__ int db_find(int* parent, int x) {
  volatile int* p = parent;
  int px = p[x];
  while (px != x) {
    const int gp = p[px];
    if (gp != px) p[x] = gp;   // path halving: gp is an ancestor of x, and only roots are ever written by atomicCAS
    x = gp;
    px = p[x];
  }
  return x;
}

// unites the sets of a and b; returns the root of the union (the lower of the two roots)
__device__ __forceinline__ int db_unite(int* parent, int a, int b) {
  for (;;) {
    a = db_find(parent, a);
    b = db_find(parent, b);
    if (a == b) return a;
    if (a > b) {
      const int t = a;
      a = b;
      b = t;
    }
    if (atomicCAS(parent + b, b, a) == b) return a;
  }
}

__device__ __forceinline__ void db_bar_consumers() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// Persistent grid, static round-robin over units u = tile * S + split: tile = 128 local rows, split = a range of the
// column blocks of all rows.  Producer and 3xTF32 main loop of b2k_pair_wg.cuh, as k_knn_wg.
// The epilogue decides every (row, column) pair of the block with the screen and, in the band, the fp64 rule:
//   UNION = false  counts adjacent columns per row (integer atomics once per unit);
//   UNION = true   columns that are not core are skipped (so are blocks with no core row, by both roles); for a core
//                  row, pairs whose roots are already equal are skipped before the decision: column roots are
//                  snapshotted into shared memory per block and the row's root is kept in a register, refreshed per
//                  block; both only ever lag the truth by merges, so equal values mean one set.  A non-core row keeps
//                  the lowest adjacent core column and records it with atomicMin once per unit.
template <int NCH, bool UNION>
__global__ void __launch_bounds__(PW_NTHREADS, 1)
k_db_wg(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapHi,
        const __grid_constant__ CUtensorMap mapLo, const DbArgs args) {
  using G = DbWgCfg<NCH>;
  constexpr int R = PW_N / 2;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t base = smem_u32(smem_raw);
  const PairWgBars bars = pair_wg_init<G>(base);
  int* sroot = reinterpret_cast<int*>(smem_raw + G::OFF_OWN);                     // [2][128]
  uint8_t* score = smem_raw + G::OFF_OWN + 2 * PW_N * 4;                          // [2][128]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nunits = args.ntiles * args.S;
  const int nit = (int)blockIdx.x < nunits ? (nunits - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;

  if (warp >= 8) {
    if (warp == 8 && elect_one())
      pair_wg_produce<G>(
          base, bars, &mapQ, &mapHi, &mapLo, nit,
          [&](int it) {
            const int u = (int)blockIdx.x + it * (int)gridDim.x;
            const int tile = u / args.S, split = u % args.S;
            return PairWgUnit{tile * PW_TM, (int)((int64_t)split * args.nblk / args.S),
                              (int)((int64_t)(split + 1) * args.nblk / args.S)};
          },
          [&](int b) { return UNION && !args.blk_core[b]; });   // the consumers skip the same blocks
    __syncwarp();
    return;
  }

  const int g = warp >> 2, wi = warp & 3;
  const int rr0 = g * 64 + wi * 16 + (lane >> 2);   // this thread's rows rr0, rr0 + 8 of the tile
  float acc[R];
  int q = 0, par = 0;
  unsigned long long n_band = 0, n_union = 0;
  for (int it = 0; it < nit; ++it) {
    const int u = (int)blockIdx.x + it * (int)gridDim.x;
    const int tile = u / args.S, split = u % args.S;
    const int b0 = (int)((int64_t)split * args.nblk / args.S), b1 = (int)((int64_t)(split + 1) * args.nblk / args.S);
    int64_t lrow[2], grow[2];
    bool vrow[2], coreI[2] = {false, false};
    float ni[2];
    int cnt[2] = {0, 0}, rootI[2] = {0, 0}, bm[2] = {DB_NONE, DB_NONE};
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      lrow[h] = (int64_t)tile * PW_TM + rr0 + 8 * h;
      grow[h] = args.row0 + lrow[h];
      vrow[h] = lrow[h] < args.n_local;
      ni[h] = vrow[h] ? __ldg(args.norms + grow[h]) : 0.f;
      if (UNION && vrow[h]) {
        coreI[h] = args.core[grow[h]] != 0;
        rootI[h] = (int)grow[h];
      }
    }
    mbar_wait_nocall(bars.qfull(), (uint32_t)(it & 1));
    for (int b = b0; b < b1; ++b) {
      if (UNION && !args.blk_core[b]) continue;   // as the producer
      pair_wg_block<G>(smem_raw, base, bars, rr0, lane, acc, q);
      if (UNION) {   // snapshot of the block's column roots and core flags; double-buffered, one barrier per block
        const int t = threadIdx.x;
        if (t < PW_N) {
          const int64_t col = (int64_t)b * PW_N + t;
          const bool c = col < args.n_total && args.core[col] != 0;
          score[par * PW_N + t] = c;
          sroot[par * PW_N + t] = c ? db_find(args.parent, (int)col) : -1;
        }
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (coreI[h]) rootI[h] = db_find(args.parent, rootI[h]);
        db_bar_consumers();
      }
      // ---- epilogue: acc[i] is row rr0 + 8 ((i >> 1) & 1), block column 8 (i >> 2) + 2 (lane & 3) + (i & 1) ----
      const int cb = 2 * (lane & 3);
      const float* nb = args.norms + (size_t)b * PW_N + cb;
#pragma unroll
      for (int i = 0; i < R; ++i) {
        const int h = (i >> 1) & 1;
        const int cl = 8 * (i >> 2) + cb + (i & 1);
        const int64_t col = (int64_t)b * PW_N + cl;
        if (!vrow[h] || col >= args.n_total) continue;
        if (UNION) {
          if (!score[par * PW_N + cl]) continue;
          if (coreI[h] ? rootI[h] == sroot[par * PW_N + cl] : col >= bm[h]) continue;
        }
        const float nj = __ldg(nb + 8 * (i >> 2) + (i & 1));
        const float S = fmaf(-2.f, acc[i], nj) + ni[h];
        const float r = S - args.E;
        const float B = fmaf(args.coef, ni[h] + nj, args.B0);
        bool adj;
        if (r < -B) {
          adj = true;
        } else if (r > B) {
          adj = false;
        } else {   // the band, and any screen that overflowed: the fp64 rule
          adj = db_adjacent(args.X, args.nrm, args.d, args.metric, args.eps2, grow[h], col);
          ++n_band;
        }
        if (!adj) continue;
        if (!UNION) {
          ++cnt[h];
        } else if (coreI[h]) {
          rootI[h] = db_unite(args.parent, rootI[h], sroot[par * PW_N + cl]);
          ++n_union;
        } else {
          bm[h] = (int)col;
        }
      }
      par ^= 1;
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(bars.qempty());   // every A fragment of this unit has been read
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!UNION) {   // the quad's four lanes hold the same row
        int c = cnt[h];
        c += __shfl_xor_sync(0xffffffffu, c, 1);
        c += __shfl_xor_sync(0xffffffffu, c, 2);
        if (vrow[h] && (lane & 3) == 0 && c) atomicAdd(args.counts + lrow[h], c);
      } else if (vrow[h] && !coreI[h] && bm[h] != DB_NONE) {
        atomicMin(args.bmin + lrow[h], bm[h]);
      }
    }
  }
  if (args.stat != nullptr) {
    if (n_band) atomicAdd(args.stat, n_band);
    if (n_union) atomicAdd(args.stat + 1, n_union);
  }
}

// Generic pass: CTA = 64 local rows x one split of 64-row column tiles; thread (ty, tx) owns rows ty + 16 a and columns
// tx + 16 b (a, b < 4) and forms the fp64 rule's sums in feature order.  The union mode mirrors k_db_wg's epilogue.
constexpr int GR = 64, GCL = 64, GF = 32, G_NTHREADS = 256;
template <bool UNION, bool COS>
__global__ void __launch_bounds__(G_NTHREADS)
k_db_generic(const DbArgs args) {
  __shared__ float xr[GF][GR + 1], xc[GF][GCL + 1];
  __shared__ int sroot[GCL];
  __shared__ uint8_t score[GCL];
  const int tile = blockIdx.x / args.S, split = blockIdx.x % args.S;
  const int64_t nct = (args.n_total + GCL - 1) / GCL;
  const int64_t t0 = split * nct / args.S, t1 = (split + 1) * nct / args.S;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int d = args.d;
  int64_t lrow[4], grow[4];
  bool vrow[4], coreI[4];
  int cnt[4], rootI[4], bm[4];
  double nri[4];
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    lrow[a] = (int64_t)tile * GR + ty + 16 * a;
    grow[a] = args.row0 + lrow[a];
    vrow[a] = lrow[a] < args.n_local;
    coreI[a] = UNION && vrow[a] && args.core[grow[a]] != 0;
    cnt[a] = 0;
    rootI[a] = (int)grow[a];
    bm[a] = DB_NONE;
    nri[a] = (COS && vrow[a]) ? args.nrm[grow[a]] : 0.0;
  }
  unsigned long long n_union = 0;
  for (int64_t t = t0; t < t1; ++t) {
    if (UNION) {
      __syncthreads();
      if (threadIdx.x < GCL) {
        const int64_t col = t * GCL + threadIdx.x;
        const bool c = col < args.n_total && args.core[col] != 0;
        score[threadIdx.x] = c;
        sroot[threadIdx.x] = c ? db_find(args.parent, (int)col) : -1;
      }
      __syncthreads();
      bool any = false;
      for (int e = 0; e < GCL; ++e) any |= score[e] != 0;
      if (!any) continue;   // no core column in this tile
#pragma unroll
      for (int a = 0; a < 4; ++a)
        if (coreI[a]) rootI[a] = db_find(args.parent, rootI[a]);
    }
    double acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;
    for (int f0 = 0; f0 < d; f0 += GF) {
      __syncthreads();
      for (int e = threadIdx.x; e < GF * GR; e += G_NTHREADS) {
        const int r = e / GF, c = e % GF;
        const int64_t lr = (int64_t)tile * GR + r, gc = t * GCL + r;
        xr[c][r] = (lr < args.n_local && f0 + c < d) ? args.X[(args.row0 + lr) * d + f0 + c] : 0.f;
        xc[c][r] = (gc < args.n_total && f0 + c < d) ? args.X[gc * d + f0 + c] : 0.f;
      }
      __syncthreads();
      const int fc = min(GF, d - f0);
      for (int c = 0; c < fc; ++c) {
        double vr[4], vc[4];
#pragma unroll
        for (int a = 0; a < 4; ++a) vr[a] = (double)xr[c][ty + 16 * a];
#pragma unroll
        for (int b = 0; b < 4; ++b) vc[b] = (double)xc[c][tx + 16 * b];
        if (!COS) {
#pragma unroll
          for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int b = 0; b < 4; ++b) {
              const double df = __dsub_rn(vr[a], vc[b]);
              acc[a][b] = __dadd_rn(acc[a][b], __dmul_rn(df, df));
            }
        } else {
#pragma unroll
          for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int b = 0; b < 4; ++b) acc[a][b] = __dadd_rn(acc[a][b], __dmul_rn(vr[a], vc[b]));
        }
      }
    }
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int cl = tx + 16 * b;
      const int64_t col = t * GCL + cl;
      if (col >= args.n_total) continue;
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        if (!vrow[a]) continue;
        if (UNION) {
          if (!score[cl]) continue;
          if (coreI[a] ? rootI[a] == sroot[cl] : col >= bm[a]) continue;
        }
        const bool adj = !COS
                             ? acc[a][b] <= args.eps2
                             : __dsub_rn(1.0, __ddiv_rn(acc[a][b], __dmul_rn(nri[a], args.nrm[col]))) <= args.eps2;
        if (!adj) continue;
        if (!UNION) {
          ++cnt[a];
        } else if (coreI[a]) {
          rootI[a] = db_unite(args.parent, rootI[a], sroot[cl]);
          ++n_union;
        } else {
          bm[a] = (int)col;
        }
      }
    }
  }
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    if (!vrow[a]) continue;
    if (!UNION) {
      if (cnt[a]) atomicAdd(args.counts + lrow[a], cnt[a]);
    } else if (!coreI[a] && bm[a] != DB_NONE) {
      atomicMin(args.bmin + lrow[a], bm[a]);
    }
  }
  if (UNION && args.stat != nullptr && n_union) atomicAdd(args.stat + 1, n_union);
}

// ---- small passes ----
// out[0] += non-finite values, out[1] += rows whose every value is 0 (warp per row)
__global__ void __launch_bounds__(256) k_db_check(const float* __restrict__ X, int64_t n, int d,
                                                  unsigned long long* __restrict__ out) {
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= n) return;
  int bad = 0, nz = 0;
  for (int f = lane; f < d; f += 32) {
    const float v = X[row * d + f];
    bad += !isfinite(v);
    nz += v != 0.f;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    bad += __shfl_xor_sync(0xffffffffu, bad, o);
    nz += __shfl_xor_sync(0xffffffffu, nz, o);
  }
  if (lane == 0) {
    if (bad) atomicAdd(out, (unsigned long long)bad);
    if (nz == 0) atomicAdd(out + 1, 1ull);
  }
}

// cosine: nrm[i] = sqrt of the feature-order fp64 sum of squares; Y[i] = fl32(x / nrm) (thread per row)
__global__ void __launch_bounds__(256) k_db_normalize(const float* __restrict__ X, int64_t n, int d,
                                                      double* __restrict__ nrm, float* __restrict__ Y) {
  const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= n) return;
  const float* x = X + row * d;
  double s = 0.0;
  for (int f = 0; f < d; ++f) s = __dadd_rn(s, __dmul_rn((double)x[f], (double)x[f]));
  const double r = __dsqrt_rn(s);
  nrm[row] = r;
  if (Y != nullptr)
    for (int f = 0; f < d; ++f) Y[row * d + f] = (float)__ddiv_rn((double)x[f], r);
}

__global__ void __launch_bounds__(256) k_db_core(const int* __restrict__ counts, int64_t n, int min_samples,
                                                 uint8_t* __restrict__ core) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    core[i] = counts[i] >= min_samples;
}

// blk[b] = block b of `width` rows holds a core row
__global__ void __launch_bounds__(256) k_db_blk_core(const uint8_t* __restrict__ core, int64_t n, int width,
                                                     int64_t nblk, uint8_t* __restrict__ blk) {
  for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < nblk; b += (int64_t)gridDim.x * blockDim.x) {
    uint8_t any = 0;
    for (int64_t i = b * width; i < n && i < (b + 1) * width; ++i) any |= core[i];
    blk[b] = any;
  }
}

__global__ void __launch_bounds__(256) k_db_init(int* __restrict__ parent, int64_t n, int* __restrict__ bmin,
                                                 int64_t n_local, int* __restrict__ counts) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    parent[i] = (int)i;
    if (i < n_local) {
      bmin[i] = DB_NONE;
      counts[i] = 0;
    }
  }
}

__global__ void __launch_bounds__(256) k_db_compress(int* __restrict__ parent, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    parent[i] = db_find(parent, (int)i);
}

// union of every (x, roots[r][x]) over the gathered parent arrays of all ranks
__global__ void __launch_bounds__(256) k_db_merge(int* __restrict__ parent, const int* __restrict__ roots, int64_t n,
                                                  int nranks) {
  const int64_t m = n * nranks;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < m; e += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(e % n), r = roots[e];
    if (r != x) db_unite(parent, x, r);
  }
}

// cluster ids: chunk c of DB_SCAN rows -> roots of core rows counted, then scanned, then numbered in row order
constexpr int DB_SCAN = 4096;
__device__ __forceinline__ int db_block_excl_scan(int v, int* sh, int* total) {   // 256 threads
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  __syncthreads();
  if (lane == 31) sh[w] = x;
  __syncthreads();
  int off = 0, tot = 0;
  for (int k = 0; k < 8; ++k) {
    if (k < w) off += sh[k];
    tot += sh[k];
  }
  *total = tot;
  return off + x - v;
}

__device__ __forceinline__ bool db_is_root(const int* parent, const uint8_t* core, int64_t x) {
  return core[x] && parent[x] == x;
}

__global__ void __launch_bounds__(256) k_db_chunk_count(const int* __restrict__ parent, const uint8_t* __restrict__ core,
                                                        int64_t n, int* __restrict__ chunk) {
  __shared__ int sh[8];
  const int64_t c0 = (int64_t)blockIdx.x * DB_SCAN;
  int v = 0;
  for (int k = 0; k < DB_SCAN / 256; ++k) {
    const int64_t x = c0 + (int64_t)threadIdx.x * (DB_SCAN / 256) + k;
    v += x < n && db_is_root(parent, core, x);
  }
  int tot;
  db_block_excl_scan(v, sh, &tot);
  if (threadIdx.x == 0) chunk[blockIdx.x] = tot;
}

// one CTA: chunk[0..nc) -> exclusive offsets in place, chunk[nc] = total
__global__ void __launch_bounds__(256) k_db_chunk_scan(int* __restrict__ chunk, int64_t nc) {
  __shared__ int sh[8];
  int carry = 0;
  for (int64_t b = 0; b < nc; b += 256) {
    const int64_t i = b + threadIdx.x;
    const int v = i < nc ? chunk[i] : 0;
    int tot;
    const int ex = db_block_excl_scan(v, sh, &tot);
    __syncthreads();
    if (i < nc) chunk[i] = carry + ex;
    carry += tot;
  }
  if (threadIdx.x == 0) chunk[nc] = carry;
}

__global__ void __launch_bounds__(256) k_db_number(const int* __restrict__ parent, const uint8_t* __restrict__ core,
                                                   int64_t n, const int* __restrict__ chunk, int* __restrict__ cid) {
  __shared__ int sh[8];
  const int64_t c0 = (int64_t)blockIdx.x * DB_SCAN;
  const int64_t x0 = c0 + (int64_t)threadIdx.x * (DB_SCAN / 256);
  int v = 0;
  for (int k = 0; k < DB_SCAN / 256; ++k) v += x0 + k < n && db_is_root(parent, core, x0 + k);
  int tot;
  int id = chunk[blockIdx.x] + db_block_excl_scan(v, sh, &tot);
  for (int k = 0; k < DB_SCAN / 256; ++k) {
    const int64_t x = x0 + k;
    if (x < n && db_is_root(parent, core, x)) cid[x] = id++;
  }
}

__global__ void __launch_bounds__(256) k_db_labels(const int* __restrict__ parent, const uint8_t* __restrict__ core,
                                                   const int* __restrict__ cid, const int* __restrict__ bmin,
                                                   int64_t row0, int64_t n_local, int32_t* __restrict__ labels,
                                                   uint8_t* __restrict__ core_out) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_local; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t g = row0 + i;
    int lab = -1;
    if (core[g]) lab = cid[parent[g]];
    else if (bmin[i] != DB_NONE) lab = cid[parent[bmin[i]]];
    labels[i] = lab;
    if (core_out != nullptr) core_out[i] = core[g];
  }
}

unsigned grid_1d(int64_t n, int sm) { return (unsigned)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, (int64_t)sm * 16)); }
}  // namespace

// The screen's error bound (used by the host below; tests/test_dbscan_cpu.py checks it against a NumPy restatement of the
// screen).  u = 2^-24.  Let v_i = fl32(x_i - s) be the shifted rows, a = v_i, b = v_j, N = ||a||^2 + ||b||^2, and D the
// fp64 rule's value (euclidean).  The screen S = fl32(fl32(n_j - 2 acc) + n_i) differs from D by at most
//   norms     n = fl32(fp64 sum of v^2): |n - ||v||^2| <= 1.0001 u ||v||^2                        -> 1.0001 u N
//   split     a = ah + al + ra with |ah - a| <= 2^-11 |a|, |ra| <= 2^-22 |a| (likewise b); dropping al.bl, ah.rb,
//             al.rb and ra.b costs <= 12.004 u sum |a_f b_f| per dot, twice in S                    -> 12.004 u N
//   wgmma     the tensor cores sum 3 ceil(d/8) blocks of 8 exact tf32 products each into the fp32 accumulator; modelled
//             pessimistically, each block truncates every addend at the largest addend's 2^-22, so a block loses at
//             most 9 * 4u of (its |products| + |accumulator|), and the whole dot <= 36 u (1 + nb) sum |terms|, sum
//             |terms| <= 1.002 sum |a_f b_f| <= 0.501 N; twice in S                                 -> 36.08 u (1 + nb) N
//   epilogue  two fp32 roundings of values <= 3.1 N                                                   -> 6 u N
//   shift     |v - (x - s)| <= u/(1-u) |v| per component, so | ||a - b||^2 - ||x_i - x_j||^2 | <= 2 eps_s ||a - b||
//             + eps_s^2 with eps_s <= u' (||a|| + ||b||)                                              -> 4.001 u N
//   fp64 rule D is ||x_i - x_j||^2 to (d + 3) 2^-53 relative, with ||x_i - x_j||^2 <= 2.0001 N         -> 0.001 u N
// so |S - D| <= (23.02 + 36.08 (1 + nb)) u N, nb = 3 ceil(d/8).  Cosine compares 2 (1 - cos) with E = 2 eps on the
// normalised rows y = fl32(x / ||x||) (then shifted as above): |y_f - x_f/||x||| <= 1.0001 u |x_f|/||x||, which moves
// ||y_i - y_j||^2 from 2 (1 - cos) by at most 8.001 u, and the fp64 rule's own error is below 0.01 u; B0 adds 8.1 u.
// The comparison itself runs in fp32: r = fl32(S - fl32(E)) with |fl32(E) - E| <= u E, so a margin of (1 + u) (B + u E)
// keeps "r < -B'" adjacent and "r > B'" not; the kernel's fp32 B' = fmaf(coef, fl32(n_i + n_j), B0) is at least that
// with coef = (24 + 37 (1 + nb)) u (1 + 2^-10) and B0 = (2.01 u E + [cosine] 8.1 u) (1 + 2^-10).
static void b2k_dbscan_bound(int d, int metric, double E, float* coef, float* B0) {
  const double u = std::ldexp(1.0, -24);
  const double nb = 3.0 * ((d + 7) / 8);
  *coef = (float)((24.0 + 37.0 * (1.0 + nb)) * u * (1.0 + std::ldexp(1.0, -10)));
  *B0 = (float)((2.01 * u * E + (metric == 1 ? 8.1 * u : 0.0)) * (1.0 + std::ldexp(1.0, -10)));
}

int b2k_dbscan_fit_impl(b2k_ctx* ctx, const float* X, int64_t n_local, int d, double eps, int min_samples, int metric,
                        int32_t* labels_out, uint8_t* core_out, int64_t* n_clusters_out, cudaStream_t s) {
  const int nr = ctx->nranks;
  B2kTimer tm(ctx->time_kernels != 0);
  // ---- sizes and input checks of every rank; each error is decided on them, identically on every rank ----
  constexpr int NS = 4;   // n_local, d, non-finite values, zero rows
  int64_t* sz_dev;
  B2K_TRY(b2k_scratch_layout(ctx, "DBSCAN sizes", [&](B2kLayout& L) -> int {
    sz_dev = L.take<int64_t>((size_t)NS * (nr + 1));
    return B2K_OK;
  }));
  const int64_t mine[2] = {n_local, d};
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(sz_dev, mine, sizeof(mine), cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaMemsetAsync(sz_dev + 2, 0, 2 * sizeof(int64_t), s));
  if (n_local > 0) {
    k_db_check<<<(unsigned)((n_local * 32 + 255) / 256), 256, 0, s>>>(X, n_local, d,
                                                                      reinterpret_cast<unsigned long long*>(sz_dev + 2));
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
  }
  B2K_TRY(b2k_comm_allgather_i64(ctx, sz_dev, sz_dev + NS, NS, s));
  std::vector<int64_t> sz((size_t)NS * nr);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(sz.data(), sz_dev + NS, sz.size() * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  int64_t n_total = 0, row0 = 0, n_max = 0, n_bad = 0, n_zero = 0;
  std::vector<int64_t> off(nr + 1, 0);
  for (int r = 0; r < nr; ++r) {
    if (sz[NS * r + 1] != sz[1])
      return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_dbscan_fit: d differs between ranks (rank " + std::to_string(r) +
                                                " has d = " + std::to_string(sz[NS * r + 1]) + ", rank 0 has d = " +
                                                std::to_string(sz[1]) + ")");
    if (r < ctx->rank) row0 += sz[NS * r];
    off[r + 1] = off[r] + sz[NS * r];
    n_total += sz[NS * r];
    n_max = std::max(n_max, sz[NS * r]);
    n_bad += sz[NS * r + 2];
    n_zero += sz[NS * r + 3];
  }
  if (!(std::isfinite(eps) && eps > 0.0))
    return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_dbscan_fit: eps = " + std::to_string(eps) + " must be finite and > 0");
  if (min_samples < 1)
    return b2k_fail(ctx, B2K_ERR_INVALID,
                    "b2k_dbscan_fit: min_samples = " + std::to_string(min_samples) + " must be >= 1");
  if (metric != 0 && metric != 1)
    return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_dbscan_fit: metric = " + std::to_string(metric) +
                                              " (0 = euclidean, 1 = cosine)");
  if (n_total == 0) return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_dbscan_fit: no rows on any rank");
  if (n_total > (int64_t)0x7ffffeff)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "b2k_dbscan_fit: 2^31 - 256 or more rows in all");
  if (n_bad > 0) return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_dbscan_fit: DBSCAN input contains NaN or infinity");
  if (metric == 1 && n_zero > 0)
    return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_dbscan_fit: cosine distance is undefined for a zero row (" +
                                              std::to_string(n_zero) + " such rows)");

  // ---- plan ----
  const double E = metric == 0 ? eps * eps : 2.0 * eps;
  const bool x_aligned = nr > 1 || (reinterpret_cast<uintptr_t>(X) & 15u) == 0;
  const bool wg_ok = b2k_knn_wg_width(d) && x_aligned && E < 1e30;
  if (ctx->kernel_path == B2K_PATH_FUSED && !wg_ok)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "kernel_path=2 requested but the wgmma DBSCAN pass needs d % 4 == 0, "
                                              "4 <= d <= 128 and 16-byte aligned X (d = " + std::to_string(d) + ")");
  const bool wg = wg_ok && ctx->kernel_path != B2K_PATH_GENERIC;
  int sm = ctx->sm_count;
  if (ctx->grid_limit > 0 && ctx->grid_limit < sm) sm = ctx->grid_limit;
  const int DP = b2k_knn_wg_dp(d);
  const int64_t nblk = wg ? (n_total + PW_N - 1) / PW_N : (n_total + GCL - 1) / GCL;
  const int64_t n_pad = ((n_total + PW_N - 1) / PW_N) * PW_N;
  const int64_t ntiles = wg ? (n_local + PW_TM - 1) / PW_TM : (n_local + GR - 1) / GR;
  // column splits: at least about 2 units per SM, at most one block per split
  const int S = (int)std::max<int64_t>(
      1, std::min<int64_t>({(2 * (int64_t)sm + std::max<int64_t>(ntiles, 1) - 1) / std::max<int64_t>(ntiles, 1), nblk,
                            (int64_t)DB_SMAX}));
  const int64_t nc = (n_total + DB_SCAN - 1) / DB_SCAN;
  float *Xpad = nullptr, *Xg = nullptr, *Y = nullptr, *Vs = nullptr, *Xhi = nullptr, *Xlo = nullptr, *norms = nullptr;
  double* nrm = nullptr;
  int *counts = nullptr, *parent = nullptr, *roots = nullptr, *bmin = nullptr, *cid = nullptr, *chunk = nullptr;
  uint8_t *corepad = nullptr, *core = nullptr, *blk = nullptr;
  unsigned long long* stat = nullptr;
  B2K_TRY(b2k_scratch_layout(ctx, "DBSCAN", [&](B2kLayout& L) -> int {
    sz_dev = L.take<int64_t>((size_t)NS * (nr + 1));
    if (nr > 1) {
      Xpad = L.take<float>((size_t)nr * n_max * d, 1024);
      Xg = L.take<float>((size_t)n_total * d, 1024);
      corepad = L.take<uint8_t>((size_t)nr * n_max);
      roots = L.take<int>((size_t)nr * n_total);
    }
    if (metric == 1) {
      nrm = L.take<double>((size_t)n_total);
      if (wg) Y = L.take<float>((size_t)n_total * d, 1024);
    }
    if (wg) {
      Vs = L.take<float>((size_t)std::max<int64_t>(n_local, 1) * d, 1024);
      Xhi = L.take<float>((size_t)n_pad * DP, 1024);
      Xlo = L.take<float>((size_t)n_pad * DP, 1024);
      norms = L.take<float>((size_t)n_pad);
    }
    counts = L.take<int>((size_t)std::max<int64_t>(n_local, 1));
    bmin = L.take<int>((size_t)std::max<int64_t>(n_local, 1));
    core = L.take<uint8_t>((size_t)n_total);
    blk = L.take<uint8_t>((size_t)nblk);
    parent = L.take<int>((size_t)n_total);
    cid = L.take<int>((size_t)n_total);
    chunk = L.take<int>((size_t)nc + 1);
    stat = L.take<unsigned long long>(2);
    return B2K_OK;
  }));
  const unsigned gsm = (unsigned)ctx->sm_count;
  tm.mark(0, s);
  // ---- every rank's rows, in global order ----
  const float* Xall = X;
  if (nr > 1) {
    float* minex = Xpad + (size_t)ctx->rank * n_max * d;
    if (n_local > 0)
      B2K_CUDA_OK(ctx, cudaMemcpyAsync(minex, X, (size_t)n_local * d * 4, cudaMemcpyDeviceToDevice, s));
    B2K_TRY(b2k_comm_allgather_bytes(ctx, minex, Xpad, (size_t)n_max * d * 4, s));
    for (int r = 0; r < nr; ++r)
      if (sz[NS * r] > 0)
        B2K_CUDA_OK(ctx, cudaMemcpyAsync(Xg + (size_t)off[r] * d, Xpad + (size_t)r * n_max * d,
                                         (size_t)sz[NS * r] * d * 4, cudaMemcpyDeviceToDevice, s));
    Xall = Xg;
  }
  k_db_init<<<grid_1d(n_total, gsm), 256, 0, s>>>(parent, n_total, bmin, n_local, counts);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  B2K_CUDA_OK(ctx, cudaMemsetAsync(stat, 0, 2 * sizeof(unsigned long long), s));
  ctx->stats.kernel_launches++;
  if (metric == 1) {
    k_db_normalize<<<(unsigned)((n_total + 255) / 256), 256, 0, s>>>(Xall, n_total, d, nrm, Y);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
  }
  DbArgs a{};
  a.n_local = n_local;
  a.n_total = n_total;
  a.row0 = row0;
  a.ntiles = (int)ntiles;
  a.S = S;
  a.nblk = (int)nblk;
  a.d = d;
  a.metric = metric;
  a.E = (float)E;
  b2k_dbscan_bound(d, metric, E, &a.coef, &a.B0);
  a.eps2 = metric == 0 ? eps * eps : eps;
  a.X = Xall;
  a.nrm = nrm;
  a.counts = counts;
  a.core = core;
  a.blk_core = blk;
  a.parent = parent;
  a.bmin = bmin;
  a.stat = ctx->collect_recheck ? stat : nullptr;
  PairWgMaps maps;
  if (wg) {
    const float* src = metric == 1 ? Y : Xall;   // shifted by its global row 0
    B2K_TRY(b2k_knn_prep_launch(ctx, src, n_total, d, nullptr, n_pad, DP, Xhi, Xlo, norms, s));
    B2K_TRY(b2k_knn_shift_launch(ctx, src + (size_t)row0 * d, n_local, d, src, Vs, s));
    a.norms = norms;
    B2K_TRY(pair_wg_maps(ctx, Vs, std::max<int64_t>(n_local, 1), d, Xhi, Xlo, n_pad, DP, &maps));
  }
  const int grid = (int)std::min<int64_t>(sm, ntiles * S);
  tm.mark(1, s);

  // ---- count pass ----
  if (ntiles > 0) {
    if (wg) {
      B2K_TRY(pair_wg_launch<DB_SNAP>(
          ctx, DP, [](auto nch) { return k_db_wg<decltype(nch)::value, false>; }, grid, maps, a, s));
      ctx->stats.fused_tc_launches++;
    } else {
      if (metric == 1) k_db_generic<false, true><<<(unsigned)(ntiles * S), G_NTHREADS, 0, s>>>(a);
      else k_db_generic<false, false><<<(unsigned)(ntiles * S), G_NTHREADS, 0, s>>>(a);
      B2K_CUDA_OK(ctx, cudaGetLastError());
      ctx->stats.generic_launches++;
    }
    ctx->stats.kernel_launches++;
  }
  ctx->stats.last_path = wg ? B2K_PATH_FUSED : B2K_PATH_GENERIC;
  tm.mark(2, s);

  // ---- core flags of every row ----
  if (nr > 1) {
    uint8_t* minec = corepad + (size_t)ctx->rank * n_max;
    if (n_local > 0) {
      k_db_core<<<grid_1d(n_local, gsm), 256, 0, s>>>(counts, n_local, min_samples, minec);
      B2K_CUDA_OK(ctx, cudaGetLastError());
      ctx->stats.kernel_launches++;
    }
    B2K_TRY(b2k_comm_allgather_bytes(ctx, minec, corepad, (size_t)n_max, s));
    for (int r = 0; r < nr; ++r)
      if (sz[NS * r] > 0)
        B2K_CUDA_OK(ctx, cudaMemcpyAsync(core + off[r], corepad + (size_t)r * n_max, (size_t)sz[NS * r],
                                         cudaMemcpyDeviceToDevice, s));
  } else {
    k_db_core<<<grid_1d(n_local, gsm), 256, 0, s>>>(counts, n_local, min_samples, core);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
  }
  k_db_blk_core<<<grid_1d(nblk, gsm), 256, 0, s>>>(core, n_total, wg ? PW_N : GCL, nblk, blk);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;

  // ---- union pass ----
  if (ntiles > 0) {
    if (wg) {
      B2K_TRY(pair_wg_launch<DB_SNAP>(
          ctx, DP, [](auto nch) { return k_db_wg<decltype(nch)::value, true>; }, grid, maps, a, s));
      ctx->stats.fused_tc_launches++;
    } else {
      if (metric == 1) k_db_generic<true, true><<<(unsigned)(ntiles * S), G_NTHREADS, 0, s>>>(a);
      else k_db_generic<true, false><<<(unsigned)(ntiles * S), G_NTHREADS, 0, s>>>(a);
      B2K_CUDA_OK(ctx, cudaGetLastError());
      ctx->stats.generic_launches++;
    }
    ctx->stats.kernel_launches++;
  }
  tm.mark(3, s);

  // ---- merge of the ranks' forests, cluster numbering, labels ----
  k_db_compress<<<grid_1d(n_total, gsm), 256, 0, s>>>(parent, n_total);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  if (nr > 1) {
    B2K_TRY(b2k_comm_allgather_bytes(ctx, parent, roots, (size_t)n_total * 4, s));
    k_db_merge<<<grid_1d(n_total * nr, gsm), 256, 0, s>>>(parent, roots, n_total, nr);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    k_db_compress<<<grid_1d(n_total, gsm), 256, 0, s>>>(parent, n_total);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches += 2;
  }
  k_db_chunk_count<<<(unsigned)nc, 256, 0, s>>>(parent, core, n_total, chunk);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  k_db_chunk_scan<<<1, 256, 0, s>>>(chunk, nc);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  k_db_number<<<(unsigned)nc, 256, 0, s>>>(parent, core, n_total, chunk, cid);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches += 3;
  if (n_local > 0) {
    k_db_labels<<<grid_1d(n_local, gsm), 256, 0, s>>>(parent, core, cid, bmin, row0, n_local, labels_out, core_out);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
  }
  int ncl = 0;
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(&ncl, chunk + nc, sizeof(int), cudaMemcpyDeviceToHost, s));
  unsigned long long st[2] = {0, 0};
  if (a.stat != nullptr) B2K_CUDA_OK(ctx, cudaMemcpyAsync(st, stat, sizeof(st), cudaMemcpyDeviceToHost, s));
  tm.mark(4, s);
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  *n_clusters_out = ncl;
  if (a.stat != nullptr) {
    ctx->stats.recheck_candidates = (int64_t)st[0];
    ctx->stats.recheck_rows = (int64_t)st[1];
  }
  if (tm.on) {
    ctx->stats.last_finalize_ms = tm.ms(0, 1);   // row allgather + prep
    ctx->stats.last_fused_ms = tm.ms(1, 2);      // count pass
    ctx->stats.last_reduce_ms = tm.ms(2, 3);     // core allgather + union pass
    ctx->stats.last_allreduce_ms = tm.ms(3, 4);  // merge + labels
    ctx->stats.last_loop_ms = tm.ms(0, 4);
  }
  return B2K_OK;
}
