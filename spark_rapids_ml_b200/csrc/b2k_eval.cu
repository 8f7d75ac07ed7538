// Multi-model evaluation (include/b2kmeans.h "evaluation"): one read of a validation X scores M models and reduces
// their metric accumulators on the device.  Replaces the reference's per-batch loop over the models
// (core.py:1572-1693, classification.py:161-282), which reads X once per model and returns per-row outputs.
//
//   labels   k_eval_labels: min, max, least non-integer and non-finite count of y per span (classification).
//   pass     k_eval_linear / k_eval_forest: a CTA stages a tile of rows of X (and y) in shared memory, then evaluates
//            every model of the chunk from the staged tile with the per-row code of its predict kernel (b2k_rows.cuh).
//            Per model and tile: integer counts by shared atomics (order-free), the per-row values (log-loss term or
//            prediction) into shared memory, then one warp per (model, column) reduces them in a fixed order and
//            folds them into the CTA's running accumulators (Chan's merge for the regression moments).
//   fold     k_eval_fold: per model, the CTAs' fp64 partials in CTA order.
//   scores   k_score_linear / k_score_forest (binary evaluation): the same staged tile, but every model's score of
//            every row (element 1 of its rawPrediction) goes to global memory, with the label bit y > 0.5; the curve
//            pass over them is b2k_binary.cu.
// The grid depends on the device and the shape alone, so two calls on the same input give the same bits.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <string>
#include <vector>

#include "b2k_internal.cuh"
#include "b2k_rows.cuh"

namespace {

constexpr int EV_NT = 256;                  // threads per CTA
constexpr int EV_NW = EV_NT / 32;
constexpr int EV_MAX_ROWS = 256;            // rows of one staged tile, at most
constexpr size_t EV_TILE_BYTES = 16384;     // X bytes of one staged tile of the linear pass, at most (one row at least)
constexpr size_t EV_FTILE_BYTES = 32768;    // ... of the forest pass
constexpr size_t EV_SMEM_MAX = 100 * 1024;  // shared memory of one CTA, at most (two CTAs per SM at the cap)
constexpr int EV_MAX_CHUNK = 32;            // models of one chunk, at most
constexpr int EV_RC = 8;                    // classes per register chunk of the logistic kinds (as k_logreg_rows)
constexpr int EV_CTAS_PER_SM = 2;          // CTAs of a pass per SM, at most (the grid; see pass_grid)

// regression accumulators per model: 3 columns (label, label - prediction, prediction) x {n, mean, m2n, m2, l1}
constexpr int NREG = B2K_EVAL_REG_COLS * B2K_EVAL_REG_STATS;

// (na, ma, qa) <- the merge of (na, ma, qa) and (nb, mb, qb): count, mean, centred sum of squares (Chan et al.)
__host__ __device__ __forceinline__ void chan_merge(double& na, double& ma, double& qa, double nb, double mb, double qb) {
  if (nb == 0.0) return;
  if (na == 0.0) {
    na = nb;
    ma = mb;
    qa = qb;
    return;
  }
  const double n = na + nb, dl = mb - ma;
  ma = ma + dl * (nb / n);
  qa = qa + qb + dl * dl * (na * nb / n);
  na = n;
}

__device__ __forceinline__ double warp_sum(double v) {   // fixed xor butterfly: every lane gets the same bits
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- label check: part[span] = {min, max, least non-integer, non-finite count} ----
__global__ void __launch_bounds__(EV_NT) k_eval_labels(const float* __restrict__ y, int64_t n, int64_t span_rows,
                                                       float* __restrict__ part) {
  __shared__ float red[4][EV_NT];
  const int64_t r0 = (int64_t)blockIdx.x * span_rows, r1 = min(n, r0 + span_rows);
  float mn = INFINITY, mx = -INFINITY, ni = INFINITY, bad = 0.f;
  for (int64_t r = r0 + threadIdx.x; r < r1; r += EV_NT) {
    const float v = y[r];
    if (!isfinite(v)) {
      bad += 1.f;
      continue;
    }
    mn = fminf(mn, v);
    mx = fmaxf(mx, v);
    if (v != floorf(v)) ni = fminf(ni, v);
  }
  red[0][threadIdx.x] = mn;
  red[1][threadIdx.x] = mx;
  red[2][threadIdx.x] = ni;
  red[3][threadIdx.x] = bad > 0.f ? 1.f : 0.f;
  __syncthreads();
  for (int o = EV_NT / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      red[0][threadIdx.x] = fminf(red[0][threadIdx.x], red[0][threadIdx.x + o]);
      red[1][threadIdx.x] = fmaxf(red[1][threadIdx.x], red[1][threadIdx.x + o]);
      red[2][threadIdx.x] = fminf(red[2][threadIdx.x], red[2][threadIdx.x + o]);
      red[3][threadIdx.x] = fmaxf(red[3][threadIdx.x], red[3][threadIdx.x + o]);
    }
    __syncthreads();
  }
  if (threadIdx.x < 4) part[(size_t)blockIdx.x * 4 + threadIdx.x] = red[threadIdx.x][0];
}

// ---- the staged tile ----
// Shared memory of one CTA, carved by ev_carve on the host (to size it) and on the device (to place it) alike.
struct EvCarve {
  size_t xs, ys, pr, lc, tf, acc, bytes;
};
__host__ __device__ __forceinline__ EvCarve ev_carve(int TR, int dpad, int m, int C, bool cls) {
  EvCarve c;
  size_t o = 0;
  auto take = [&o](size_t bytes) {
    const size_t at = o;
    o = (o + bytes + 15) & ~(size_t)15;
    return at;
  };
  c.xs = take((size_t)TR * dpad * 4);                         // f32 [TR][dpad], zero past d
  c.ys = take((size_t)TR * 4);                                // f32 [TR]
  c.pr = take((size_t)m * TR * 8);                            // f64 [m][TR]: log-loss term or prediction
  c.lc = take(cls ? (size_t)C * 4 : 0);                       // u32 [C] label counts
  c.tf = take(cls ? (size_t)m * 2 * C * 4 : 0);               // u32 [m][2][C] tp, fp
  c.acc = take((size_t)m * (cls ? 1 : NREG) * 8);             // f64 [m][1 | NREG] running accumulators
  c.bytes = o;
  return c;
}

template <bool VEC>
__device__ __forceinline__ void stage_tile(const float* __restrict__ X, const float* __restrict__ y, int64_t r0, int tr,
                                           int d, int dpad, float* xs, float* ys) {
  if (VEC) {   // dpad == d, 16-byte aligned rows
    const float4* src = reinterpret_cast<const float4*>(X + r0 * d);
    float4* dst = reinterpret_cast<float4*>(xs);
    const int nv = tr * (d / 4);
    for (int i = threadIdx.x; i < nv; i += EV_NT) dst[i] = __ldcs(src + i);
  } else {
    const int tot = tr * dpad;
    for (int i = threadIdx.x; i < tot; i += EV_NT) {
      const int r = i / dpad, c = i - r * dpad;
      xs[i] = c < d ? __ldcs(X + (r0 + r) * d + c) : 0.f;
    }
  }
  for (int i = threadIdx.x; i < tr; i += EV_NT) ys[i] = __ldcs(y + r0 + i);
}

// One row's classification outcome: the predicted class value pv and the label's probability py.
__device__ __forceinline__ void count_row(unsigned* tf, int C, int yc, int pv) {
  if (pv == yc) atomicAdd(&tf[yc], 1u);
  else atomicAdd(&tf[C + pv], 1u);
}

// After a tile's per-row values are in pr: one warp per (model, column) folds them into acc in row order.
template <bool CLS>
__device__ __forceinline__ void reduce_tile(const double* pr, const float* ys, int TR, int tr, int m, double* acc) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int npair = CLS ? m : B2K_EVAL_REG_COLS * m;
  for (int q = warp; q < npair; q += EV_NW) {
    const int mi = CLS ? q : q / B2K_EVAL_REG_COLS, c = CLS ? 0 : q % B2K_EVAL_REG_COLS;
    const double* p = pr + (size_t)mi * TR;
    if (CLS) {
      double s = 0.0;
      for (int r = lane; r < tr; r += 32) s += p[r];
      s = warp_sum(s);
      if (lane == 0) acc[mi] += s;
      continue;
    }
    auto val = [&](int r) {
      const double yy = (double)ys[r];
      return c == 0 ? yy : c == 1 ? yy - p[r] : p[r];
    };
    double s = 0.0;
    for (int r = lane; r < tr; r += 32) s += val(r);
    const double mt = warp_sum(s) * __drcp_rn((double)tr);   // the tile mean to within an ulp: m2n is about it
    double q2 = 0.0, sq = 0.0, ab = 0.0;
    for (int r = lane; r < tr; r += 32) {
      const double v = val(r), dv = v - mt;
      q2 = fma(dv, dv, q2);
      sq = fma(v, v, sq);
      ab += fabs(v);
    }
    q2 = warp_sum(q2);
    sq = warp_sum(sq);
    ab = warp_sum(ab);
    if (lane == 0) {
      double* a = acc + (size_t)mi * NREG + c * B2K_EVAL_REG_STATS;
      chan_merge(a[0], a[1], a[2], (double)tr, mt, q2);
      a[3] += sq;
      a[4] += ab;
    }
  }
}

// The CTA's accumulators out: integer counts to the global counters (atomics, exact), fp64 to its partial slot.
template <bool CLS>
__device__ __forceinline__ void flush_cta(const unsigned* lc, const unsigned* tf, const double* acc, int m, int C,
                                          unsigned long long* labels, unsigned long long* counts, double* part) {
  if (CLS) {
    if (labels)
      for (int i = threadIdx.x; i < C; i += EV_NT)
        if (lc[i]) atomicAdd(labels + i, (unsigned long long)lc[i]);
    for (int i = threadIdx.x; i < m * 2 * C; i += EV_NT)
      if (tf[i]) atomicAdd(counts + i, (unsigned long long)tf[i]);
  }
  const int np = m * (CLS ? 1 : NREG);
  for (int i = threadIdx.x; i < np; i += EV_NT) part[(size_t)blockIdx.x * np + i] = acc[i];
}

template <bool CLS>
__device__ __forceinline__ void init_cta(unsigned* lc, unsigned* tf, double* acc, int m, int C) {
  if (CLS) {
    for (int i = threadIdx.x; i < C; i += EV_NT) lc[i] = 0u;
    for (int i = threadIdx.x; i < m * 2 * C; i += EV_NT) tf[i] = 0u;
  }
  for (int i = threadIdx.x; i < m * (CLS ? 1 : NREG); i += EV_NT) acc[i] = 0.0;
}

// ---- linear kinds ----
struct LinArgs {
  const float* X;
  const float* y;
  int64_t n;
  int d, dpad, L, TR, m, C;
  const int* kind;        // [m] B2K_EVAL_IDENTITY / LOGISTIC / SOFTMAX
  const int* row0;        // [m + 1] first row of each model in W, b
  const double* W;        // [rows][dpad] fp64, zero past d
  const double* b;        // [rows]
  const int* cls0;        // [m + 1] first class value of each model (classification)
  const double* cls;      // class values
  double eps;
  double* slots;          // [grid][EV_NW * 32 / L][kmax] margins of the softmax kind
  int kmax;
  unsigned long long* labels;   // [C] or NULL
  unsigned long long* counts;   // [m][2][C]
  double* part;                 // [grid][m][1 | NREG]
};

// Minimum resident CTAs per SM: the register budget under which ptxas keeps every instantiation free of spills (the
// classification finish, with its exp / log calls, needs more registers than two CTAs per SM leave).
template <bool VEC, bool CLS>
__global__ void __launch_bounds__(EV_NT, CLS ? 1 : 2) k_eval_linear(LinArgs a) {
  extern __shared__ __align__(16) unsigned char ev_smem[];
  const EvCarve cv = ev_carve(a.TR, a.dpad, a.m, a.C, CLS);
  float* xs = reinterpret_cast<float*>(ev_smem + cv.xs);
  float* ys = reinterpret_cast<float*>(ev_smem + cv.ys);
  double* pr = reinterpret_cast<double*>(ev_smem + cv.pr);
  unsigned* lc = reinterpret_cast<unsigned*>(ev_smem + cv.lc);
  unsigned* tf = reinterpret_cast<unsigned*>(ev_smem + cv.tf);
  double* acc = reinterpret_cast<double*>(ev_smem + cv.acc);
  init_cta<CLS>(lc, tf, acc, a.m, a.C);
  const int d = a.d, L = a.L, TR = a.TR;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, sub = lane & (L - 1), grp = lane / L, rpw = 32 / L;
  const int rps = EV_NW * rpw;   // rows of one step of the CTA
  double* slot = a.slots + ((size_t)blockIdx.x * rps + warp * rpw + grp) * a.kmax;
  for (int64_t t0 = (int64_t)blockIdx.x * TR; t0 < a.n; t0 += (int64_t)gridDim.x * TR) {
    const int tr = (int)min((int64_t)TR, a.n - t0);
    __syncthreads();   // the previous tile is consumed
    stage_tile<VEC>(a.X, a.y, t0, tr, d, a.dpad, xs, ys);
    __syncthreads();
    if (CLS && a.labels)
      for (int i = threadIdx.x; i < tr; i += EV_NT) atomicAdd(&lc[(int)ys[i]], 1u);
    for (int mi = 0; mi < a.m; ++mi) {
      const int kind = a.kind[mi], w0 = a.row0[mi], kp = a.row0[mi + 1] - w0;
      const double* Wm = a.W + (size_t)w0 * a.dpad;
      const double* bm = a.b + w0;
      for (int s = warp * rpw; s < tr; s += rps) {
        const int r = s + grp;
        const bool valid = r < tr;
        const B2kRowSmem ld{xs + (size_t)(valid ? r : 0) * a.dpad};
        if (kind == B2K_EVAL_IDENTITY) {   // k_linreg_predict
          double v = 0.0;
          if (valid) v = b2k_linear_lane(ld, d, Wm, sub, L);
          v = b2k_lanes_sum(v, L);
          if (!CLS && sub == 0 && valid) pr[(size_t)mi * TR + r] = bm[0] + v;
          continue;
        }
        // k_logreg_rows: margins per chunk of EV_RC classes; kp == 1 keeps its margin in a register
        double m1 = 0.0;
        for (int k0 = 0; k0 < kp; k0 += EV_RC) {
          double ac[EV_RC];
#pragma unroll
          for (int q = 0; q < EV_RC; ++q) ac[q] = 0.0;
          if (valid) b2k_logistic_lanes<EV_RC>(ld, d, kp, k0, Wm, a.dpad, sub, L, ac);
#pragma unroll
          for (int q = 0; q < EV_RC; ++q) ac[q] = b2k_lanes_sum(ac[q], L);
          if (sub == 0 && valid) {
#pragma unroll
            for (int q = 0; q < EV_RC; ++q) {
              const int k = k0 + q;
              if (k < kp) {
                if (kp == 1) m1 = bm[k] + ac[q];
                else slot[k] = bm[k] + ac[q];
              }
            }
          }
        }
        if (!CLS || sub != 0 || !valid) continue;
        const double* cvals = a.cls + a.cls0[mi];
        const int yc = (int)ys[r];
        int pi;
        double py;
        if (kp == 1) {
          const double p1 = b2k_sigmoid(m1);
          pi = m1 > 0.0 ? 1 : 0;
          py = yc == 0 ? 1.0 - p1 : yc == 1 ? p1 : 0.0;
        } else {
          const B2kArgmax ax = b2k_softmax_argmax(slot, kp);
          pi = ax.am;
          const double sden = b2k_softmax_denominator(slot, kp, ax.mx);
          py = yc < kp ? exp(slot[yc] - ax.mx) / sden : 0.0;
        }
        count_row(tf + (size_t)mi * 2 * a.C, a.C, yc, (int)cvals[pi]);
        pr[(size_t)mi * TR + r] = -log(fmax(py, a.eps));
      }
    }
    __syncthreads();
    reduce_tile<CLS>(pr, ys, TR, tr, a.m, acc);
  }
  __syncthreads();
  flush_cta<CLS>(lc, tf, acc, a.m, a.C, a.labels, a.counts, a.part);
}

// ---- forests ----
struct EvForest {
  int64_t off0;    // first entry of the forest's tree offsets in `off` (T + 1 entries, tree-local node indices)
  int64_t node0;   // first node of the forest in `nodes`
  int64_t val0;    // first value of the forest in `value` ([nodes][V])
  int T, V;
};
struct ForestArgs {
  const float* X;
  const float* y;
  int64_t n;
  int d, dpad, TR, m, C;
  const EvForest* forests;
  const int64_t* off;
  const B2kPNode* nodes;
  const double* value;
  double eps;
  double* slots;   // [grid][EV_NT][vmax] raw sums of the classification forests
  int vmax;
  unsigned long long* labels;
  unsigned long long* counts;
  double* part;
};

template <bool VEC, bool CLS>
__global__ void __launch_bounds__(EV_NT, 2) k_eval_forest(ForestArgs a) {
  extern __shared__ __align__(16) unsigned char ev_smem[];
  const EvCarve cv = ev_carve(a.TR, a.dpad, a.m, a.C, CLS);
  float* xs = reinterpret_cast<float*>(ev_smem + cv.xs);
  float* ys = reinterpret_cast<float*>(ev_smem + cv.ys);
  double* pr = reinterpret_cast<double*>(ev_smem + cv.pr);
  unsigned* lc = reinterpret_cast<unsigned*>(ev_smem + cv.lc);
  unsigned* tf = reinterpret_cast<unsigned*>(ev_smem + cv.tf);
  double* acc = reinterpret_cast<double*>(ev_smem + cv.acc);
  init_cta<CLS>(lc, tf, acc, a.m, a.C);
  const int TR = a.TR, G = EV_NT / TR;                 // G groups of TR threads, one row per thread of a group
  const int r = threadIdx.x % TR, g = threadIdx.x / TR;
  double* raw = a.slots + ((size_t)blockIdx.x * EV_NT + threadIdx.x) * a.vmax;
  for (int64_t t0 = (int64_t)blockIdx.x * TR; t0 < a.n; t0 += (int64_t)gridDim.x * TR) {
    const int tr = (int)min((int64_t)TR, a.n - t0);
    __syncthreads();
    stage_tile<VEC>(a.X, a.y, t0, tr, a.d, a.dpad, xs, ys);
    __syncthreads();
    if (CLS && a.labels)
      for (int i = threadIdx.x; i < tr; i += EV_NT) atomicAdd(&lc[(int)ys[i]], 1u);
    if (g < G && r < tr) {
      const float* x = xs + (size_t)r * a.dpad;
      const B2kFeatSmem xf{x};
      for (int mi = g; mi < a.m; mi += G) {   // k_rf_predict, forest mi
        const EvForest F = a.forests[mi];
        const int64_t* off = a.off + F.off0;
        const double* value = a.value + F.val0;
        const B2kPNode* P = a.nodes + F.node0;
        const int V = F.V;
        double accr = 0.0;
        if (CLS)
          for (int k = 0; k < V; ++k) raw[k] = 0.0;
        for (int t = 0; t < F.T; ++t) {
          const int64_t o = __ldg(off + t);
          const int i = b2k_rf_leaf(P + o, xf);
          const double* v = value + (o + i) * V;
          if (CLS) {
            for (int k = 0; k < V; ++k) raw[k] = __dadd_rn(raw[k], __ldg(v + k));
          } else {
            accr = __dadd_rn(accr, __ldg(v));
          }
        }
        if (CLS) {
          double tot;
          const int best = b2k_rf_class_best(raw, 0, V, tot);
          const int yc = (int)ys[r];
          const double py = yc < V && tot != 0.0 ? __ddiv_rn(raw[yc], tot) : 0.0;
          count_row(tf + (size_t)mi * 2 * a.C, a.C, yc, best);
          pr[(size_t)mi * TR + r] = -log(fmax(py, a.eps));
        } else {
          pr[(size_t)mi * TR + r] = __ddiv_rn(accr, (double)F.T);
        }
      }
    }
    __syncthreads();
    reduce_tile<CLS>(pr, ys, TR, tr, a.m, acc);
  }
  __syncthreads();
  flush_cta<CLS>(lc, tf, acc, a.m, a.C, a.labels, a.counts, a.part);
}

// ---- binary scores ----
// Where the score passes write: row r of model mi at scores[mi * ld + r]; pos[r] = y > 0.5 (NULL: not written).
struct ScoreOut {
  double* scores;
  int64_t ld;
  uint8_t* pos;
};

__device__ __forceinline__ void write_pos(const float* ys, int64_t t0, int tr, uint8_t* pos) {
  if (pos)
    for (int i = threadIdx.x; i < tr; i += EV_NT) pos[t0 + i] = ys[i] > 0.5f ? 1 : 0;
}

// Logistic kinds: rawPrediction[1] of k_logreg_rows, the margin of class 1 (binomial: raw = [-m, m], so m itself).
// Only classes 0 and 1 are formed; each class's FMA chain is the one k_logreg_rows runs, whatever the chunk width.
template <bool VEC>
__global__ void __launch_bounds__(EV_NT, 2) k_score_linear(LinArgs a, ScoreOut o) {
  extern __shared__ __align__(16) unsigned char ev_smem[];
  const EvCarve cv = ev_carve(a.TR, a.dpad, 0, 0, false);
  float* xs = reinterpret_cast<float*>(ev_smem + cv.xs);
  float* ys = reinterpret_cast<float*>(ev_smem + cv.ys);
  const int d = a.d, L = a.L, TR = a.TR;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, sub = lane & (L - 1), grp = lane / L, rpw = 32 / L;
  const int rps = EV_NW * rpw;
  for (int64_t t0 = (int64_t)blockIdx.x * TR; t0 < a.n; t0 += (int64_t)gridDim.x * TR) {
    const int tr = (int)min((int64_t)TR, a.n - t0);
    __syncthreads();
    stage_tile<VEC>(a.X, a.y, t0, tr, d, a.dpad, xs, ys);
    __syncthreads();
    write_pos(ys, t0, tr, o.pos);
    for (int mi = 0; mi < a.m; ++mi) {
      const int w0 = a.row0[mi], kp = a.row0[mi + 1] - w0, c = kp == 1 ? 0 : 1;
      const double* Wm = a.W + (size_t)w0 * a.dpad;
      for (int s = warp * rpw; s < tr; s += rps) {
        const int r = s + grp;
        const bool valid = r < tr;
        double ac[2] = {0.0, 0.0};
        if (valid) b2k_logistic_lanes<2>(B2kRowSmem{xs + (size_t)r * a.dpad}, d, kp, 0, Wm, a.dpad, sub, L, ac);
        const double m = b2k_lanes_sum(c ? ac[1] : ac[0], L);
        if (sub == 0 && valid) o.scores[mi * o.ld + t0 + r] = a.b[w0 + c] + m;
      }
    }
  }
}

// Classification forests: rawPrediction[1] of k_rf_predict, the trees' values of class 1 summed in tree order.
template <bool VEC>
__global__ void __launch_bounds__(EV_NT, 2) k_score_forest(ForestArgs a, ScoreOut o) {
  extern __shared__ __align__(16) unsigned char ev_smem[];
  const EvCarve cv = ev_carve(a.TR, a.dpad, 0, 0, false);
  float* xs = reinterpret_cast<float*>(ev_smem + cv.xs);
  float* ys = reinterpret_cast<float*>(ev_smem + cv.ys);
  const int TR = a.TR, G = EV_NT / TR;
  const int r = threadIdx.x % TR, g = threadIdx.x / TR;
  for (int64_t t0 = (int64_t)blockIdx.x * TR; t0 < a.n; t0 += (int64_t)gridDim.x * TR) {
    const int tr = (int)min((int64_t)TR, a.n - t0);
    __syncthreads();
    stage_tile<VEC>(a.X, a.y, t0, tr, a.d, a.dpad, xs, ys);
    __syncthreads();
    write_pos(ys, t0, tr, o.pos);
    if (g < G && r < tr) {
      const B2kFeatSmem xf{xs + (size_t)r * a.dpad};
      for (int mi = g; mi < a.m; mi += G) {
        const EvForest F = a.forests[mi];
        const int64_t* off = a.off + F.off0;
        const double* value = a.value + F.val0 + 1;
        const B2kPNode* P = a.nodes + F.node0;
        double raw1 = 0.0;
        for (int t = 0; t < F.T; ++t) {
          const int64_t ot = __ldg(off + t);
          raw1 = __dadd_rn(raw1, __ldg(value + (ot + b2k_rf_leaf(P + ot, xf)) * F.V));
        }
        o.scores[mi * o.ld + t0 + r] = raw1;
      }
    }
  }
}

// out [m][1 | NREG] = the CTAs' partials folded in CTA order
template <bool CLS>
__global__ void k_eval_fold(const double* __restrict__ part, int P, int m, double* __restrict__ out) {
  const int mi = blockIdx.x * blockDim.x + threadIdx.x;
  if (mi >= m) return;
  if (CLS) {
    double t = 0.0;
    for (int s = 0; s < P; ++s) t += part[(size_t)s * m + mi];
    out[mi] = t;
    return;
  }
  double a[NREG];
  for (int i = 0; i < NREG; ++i) a[i] = 0.0;
  for (int s = 0; s < P; ++s) {
    const double* p = part + ((size_t)s * m + mi) * NREG;
    for (int c = 0; c < B2K_EVAL_REG_COLS; ++c) {
      double* q = a + c * B2K_EVAL_REG_STATS;
      const double* u = p + c * B2K_EVAL_REG_STATS;
      chan_merge(q[0], q[1], q[2], u[0], u[1], u[2]);
      q[3] += u[3];
      q[4] += u[4];
    }
  }
  for (int i = 0; i < NREG; ++i) out[(size_t)mi * NREG + i] = a[i];
}

std::string num(double v) {
  char b[64];
  std::snprintf(b, sizeof b, "%.17g", v);
  return b;
}

// y's least and largest finite values, least non-integer (inf: none) and whether any value is non-finite (n > 0).
struct LabelStats {
  double mn, mx, ni;
  bool bad;
};
int label_stats(b2k_ctx* ctx, const float* y, int64_t n, LabelStats* st, cudaStream_t s) {
  const int spans = (int)std::max<int64_t>(1, std::min<int64_t>(4 * ctx->sm_count, (n + 1023) / 1024));
  const int64_t span_rows = (n + spans - 1) / spans;
  float* part;
  B2K_TRY(b2k_scratch_layout(ctx, "evaluation labels", [&](B2kLayout& L) -> int {
    part = L.take<float>((size_t)spans * 4);
    return B2K_OK;
  }));
  k_eval_labels<<<spans, EV_NT, 0, s>>>(y, n, span_rows, part);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  std::vector<float> h((size_t)spans * 4);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(h.data(), part, h.size() * 4, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  double mn = INFINITY, mx = -INFINITY, ni = INFINITY, bad = 0.0;
  for (int i = 0; i < spans; ++i) {
    mn = std::min(mn, (double)h[i * 4 + 0]);
    mx = std::max(mx, (double)h[i * 4 + 1]);
    ni = std::min(ni, (double)h[i * 4 + 2]);
    bad = std::max(bad, (double)h[i * 4 + 3]);
  }
  *st = LabelStats{mn, mx, ni, bad > 0.0};
  return B2K_OK;
}

// The label rule of b2k_logreg_labels on y, with its messages; *C = max label + 1 (0 when n == 0).
int check_labels(b2k_ctx* ctx, const float* y, int64_t n, int* C, cudaStream_t s) {
  *C = 0;
  if (n == 0) return B2K_OK;
  LabelStats st;
  B2K_TRY(label_stats(ctx, y, n, &st, s));
  const double mn = st.mn, mx = st.mx, ni = st.ni;
  if (st.bad) return b2k_fail(ctx, B2K_ERR_INVALID, "evaluation: the label holds a NaN or an infinity");
  if (mn < 0.0) return b2k_fail(ctx, B2K_ERR_INVALID, "Labels MUST be in [0, 2147483647), but got " + num(mn));
  if (std::isfinite(ni)) return b2k_fail(ctx, B2K_ERR_INVALID, "Labels MUST be Integers, but got " + num(ni));
  if (mx >= 2147483647.0) return b2k_fail(ctx, B2K_ERR_INVALID, "Labels MUST be in [0, 2147483647), but got " + num(mx));
  if (mx >= (double)B2K_LOGREG_MAX_CLASSES)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "evaluation supports label values below " +
                                                  std::to_string(B2K_LOGREG_MAX_CLASSES) + ", got " + num(mx));
  *C = (int)mx + 1;
  return B2K_OK;
}

// Rows of one tile: TR * dpad * 4 <= tile_bytes (one row at least), a multiple of `step` rows when that allows.
int tile_rows(int dpad, int step, size_t tile_bytes) {
  int tr = (int)std::min<size_t>(EV_MAX_ROWS, std::max<size_t>(1, tile_bytes / ((size_t)dpad * 4)));
  if (tr >= step) tr = tr / step * step;
  return tr;
}

// Grid of a pass: enough CTAs for the tiles, at most EV_CTAS_PER_SM per SM and option grid_limit.  It depends on n, the
// tile (d) and the device alone, not on which models share a chunk, so every model's fp64 partials fold over the same
// CTAs in the same order whatever M and the chunking are.
int pass_grid(b2k_ctx* ctx, const void* kern, size_t smem, int64_t n, int TR, int* grid) {
  int per_sm = 0;
  B2K_CUDA_OK(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  B2K_CUDA_OK(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, EV_NT, smem));
  if (per_sm < 1) return b2k_fail(ctx, B2K_ERR_STATE, "evaluation: a CTA of " + std::to_string(smem) +
                                                          " bytes of shared memory cannot be resident");
  int64_t g = std::min<int64_t>((n + TR - 1) / TR, (int64_t)EV_CTAS_PER_SM * ctx->sm_count);
  if (ctx->grid_limit > 0) g = std::min<int64_t>(g, ctx->grid_limit);
  *grid = (int)std::max<int64_t>(1, g);
  return B2K_OK;
}

// Models [0, m) in chunks: the largest prefix from `first` whose CTA fits EV_SMEM_MAX, at most EV_MAX_CHUNK models.
int chunk_end(int first, int m, int TR, int dpad, int C, bool cls) {
  int e = first + 1;
  while (e < m && e - first < EV_MAX_CHUNK && ev_carve(TR, dpad, e + 1 - first, C, cls).bytes <= EV_SMEM_MAX) ++e;
  return e;
}

// Host outputs of one chunk: counts [mc][2][C] and fp64 [mc][1 | NREG] copied back, then spread into the caller's arrays.
int finish_chunk(b2k_ctx* ctx, bool cls, int first, int mc, int C, int64_t n, int grid, double* part, double* folded,
                 unsigned long long* counts, unsigned long long* labels, int64_t* label_count_out, int64_t* tp_out,
                 int64_t* fp_out, double* loss_out, double* reg_out, cudaStream_t s) {
  const int np = cls ? 1 : NREG;
  auto fold = cls ? k_eval_fold<true> : k_eval_fold<false>;
  fold<<<(mc + 127) / 128, 128, 0, s>>>(part, n > 0 ? grid : 0, mc, folded);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  std::vector<double> f((size_t)mc * np);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(f.data(), folded, f.size() * 8, cudaMemcpyDeviceToHost, s));
  std::vector<unsigned long long> cnt(cls ? (size_t)mc * 2 * C : 0), lab(cls && labels ? C : 0);
  if (cls && C > 0) {
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(cnt.data(), counts, cnt.size() * 8, cudaMemcpyDeviceToHost, s));
    if (labels) B2K_CUDA_OK(ctx, cudaMemcpyAsync(lab.data(), labels, lab.size() * 8, cudaMemcpyDeviceToHost, s));
  }
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  if (!cls) {
    std::copy(f.begin(), f.end(), reg_out + (size_t)first * NREG);
    return B2K_OK;
  }
  for (int i = 0; i < mc; ++i) {
    loss_out[first + i] = f[i];
    for (int c = 0; c < C; ++c) {
      tp_out[(size_t)(first + i) * C + c] = (int64_t)cnt[((size_t)i * 2 + 0) * C + c];
      fp_out[(size_t)(first + i) * C + c] = (int64_t)cnt[((size_t)i * 2 + 1) * C + c];
    }
  }
  if (labels)
    for (int c = 0; c < C; ++c) label_count_out[c] = (int64_t)lab[c];
  return B2K_OK;
}

// The forests' table: F [m] and the totals of tree offsets (off0), nodes (node0) and values (val0) of all forests, and
// the most values of one forest.  Each forest needs n_values >= min_values (and exactly 1 when min_values is 0).
int forest_table(b2k_ctx* ctx, const char* who, int m, int d, int min_values, const int32_t* n_trees,
                 const int32_t* n_values, const int64_t* tree_offsets, const int32_t* feature, std::vector<EvForest>& F,
                 int64_t& off0, int64_t& node0, int64_t& val0, int& vmax) {
  const std::string w = who;
  for (int i = 0; i < m; ++i) {
    if (n_trees[i] < 1 || n_values[i] < std::max(1, min_values) || (min_values == 0 && n_values[i] != 1))
      return b2k_fail(ctx, B2K_ERR_INVALID, w + ": forest " + std::to_string(i) +
                                                (min_values == 2 ? " needs n_trees >= 1 and n_values >= 2"
                                                                 : " needs n_trees >= 1 and n_values >= 1 (1 for "
                                                                   "regression)"));
    const int64_t* off = tree_offsets + off0;
    if (off[0] != 0)
      return b2k_fail(ctx, B2K_ERR_INVALID, w + ": the tree offsets of forest " + std::to_string(i) + " must start at 0");
    for (int t = 0; t < n_trees[i]; ++t)
      if (off[t + 1] <= off[t])
        return b2k_fail(ctx, B2K_ERR_INVALID, w + ": forest " + std::to_string(i) + " has an empty tree");
    F[i] = EvForest{off0, node0, val0, n_trees[i], n_values[i]};
    const int64_t nn = off[n_trees[i]];
    for (int64_t j = 0; j < nn; ++j)
      if (feature[node0 + j] >= d)
        return b2k_fail(ctx, B2K_ERR_INVALID, w + ": a node splits on feature " + std::to_string(feature[node0 + j]) +
                                                  " >= d = " + std::to_string(d));
    off0 += n_trees[i] + 1;
    node0 += nn;
    val0 += nn * n_values[i];
    vmax = std::max(vmax, n_values[i]);
  }
  return B2K_OK;
}

// The binary passes' label rule: y finite (any value; positive when > 0.5).
int check_binary_labels(b2k_ctx* ctx, const float* y, int64_t n, cudaStream_t s) {
  if (n == 0) return B2K_OK;
  LabelStats st;
  B2K_TRY(label_stats(ctx, y, n, &st, s));
  if (st.bad) return b2k_fail(ctx, B2K_ERR_INVALID, "evaluation: the label holds a NaN or an infinity");
  return B2K_OK;
}

}  // namespace

int b2k_eval_linear_scores_impl(b2k_ctx* ctx, const float* X, const float* y, int64_t n, int d, int m,
                                const int32_t* kind, const int32_t* row_offsets, const double* W, const double* b,
                                double* scores, int64_t ld_scores, uint8_t* pos, cudaStream_t s) {
  if (d > B2K_LOGREG_MAX_D)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "evaluation supports d <= " + std::to_string(B2K_LOGREG_MAX_D));
  int nrows = 0;
  for (int i = 0; i < m; ++i) {
    const int kp = row_offsets[i + 1] - row_offsets[i];
    if (!(kind[i] == B2K_EVAL_LOGISTIC ? kp == 1 : kind[i] == B2K_EVAL_SOFTMAX && kp >= 2) || row_offsets[i] != nrows)
      return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_eval_linear_scores: model " + std::to_string(i) +
                                                " has a bad kind or row range (logistic holds 1 row, softmax >= 2)");
    nrows += kp;
  }
  B2K_TRY(check_binary_labels(ctx, y, n, s));
  if (n == 0) return B2K_OK;
  const int dpad = (d + 3) & ~3, L = b2k_row_lanes(d);
  const int TR = tile_rows(dpad, EV_NW * (32 / L), EV_TILE_BYTES);
  const bool vec = d % 4 == 0 && (reinterpret_cast<uintptr_t>(X) & 15u) == 0;
  std::vector<double> Wp((size_t)nrows * dpad, 0.0);
  for (int r = 0; r < nrows; ++r) std::copy(W + (size_t)r * d, W + (size_t)(r + 1) * d, Wp.begin() + (size_t)r * dpad);
  const size_t smem = ev_carve(TR, dpad, 0, 0, false).bytes;
  const void* kern = vec ? (const void*)k_score_linear<true> : (const void*)k_score_linear<false>;
  int grid = 0;
  B2K_TRY(pass_grid(ctx, kern, smem, n, TR, &grid));
  int* row0_d;
  double *W_d, *b_d;
  B2K_TRY(b2k_scratch_layout(ctx, "binary scores", [&](B2kLayout& Ly) -> int {
    row0_d = Ly.take<int>(m + 1);
    W_d = Ly.take<double>((size_t)nrows * dpad);
    b_d = Ly.take<double>(nrows);
    return B2K_OK;
  }));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(row0_d, row_offsets, (m + 1) * 4, cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(W_d, Wp.data(), Wp.size() * 8, cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(b_d, b, (size_t)nrows * 8, cudaMemcpyHostToDevice, s));
  LinArgs a{X, y, n, d, dpad, L, TR, m, 0, nullptr, row0_d, W_d, b_d, nullptr, nullptr, 0.0, nullptr, 1,
            nullptr, nullptr, nullptr};
  const ScoreOut o{scores, ld_scores, pos};
  if (vec) k_score_linear<true><<<grid, EV_NT, smem, s>>>(a, o);
  else k_score_linear<false><<<grid, EV_NT, smem, s>>>(a, o);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  return B2K_OK;
}

int b2k_eval_forest_scores_impl(b2k_ctx* ctx, const float* X, const float* y, int64_t n, int d, int m,
                                const int32_t* n_trees, const int32_t* n_values, const int64_t* tree_offsets,
                                const int32_t* feature, const float* threshold, const int32_t* children,
                                const double* value, double* scores, int64_t ld_scores, uint8_t* pos, cudaStream_t s) {
  std::vector<EvForest> F(m);
  int64_t off0 = 0, node0 = 0, val0 = 0;
  int vmax = 1;
  B2K_TRY(forest_table(ctx, "b2k_eval_forest_scores", m, d, 2, n_trees, n_values, tree_offsets, feature, F, off0,
                       node0, val0, vmax));
  B2K_TRY(check_binary_labels(ctx, y, n, s));
  if (n == 0) return B2K_OK;
  std::vector<B2kPNode> pn((size_t)node0);
  for (int64_t j = 0; j < node0; ++j)
    pn[j] = B2kPNode{feature[j], threshold[j], children[2 * j], children[2 * j + 1]};
  const int dpad = (d + 3) & ~3;
  const int TR = tile_rows(dpad, 1, EV_FTILE_BYTES);
  const bool vec = d % 4 == 0 && (reinterpret_cast<uintptr_t>(X) & 15u) == 0;
  const size_t smem = ev_carve(TR, dpad, 0, 0, false).bytes;
  const void* kern = vec ? (const void*)k_score_forest<true> : (const void*)k_score_forest<false>;
  int grid = 0;
  B2K_TRY(pass_grid(ctx, kern, smem, n, TR, &grid));
  EvForest* F_d;
  int64_t* off_d;
  B2kPNode* nodes_d;
  double* val_d;
  B2K_TRY(b2k_scratch_layout(ctx, "binary scores", [&](B2kLayout& Ly) -> int {
    F_d = Ly.take<EvForest>(m);
    off_d = Ly.take<int64_t>(off0);
    nodes_d = Ly.take<B2kPNode>(node0);
    val_d = Ly.take<double>(val0);
    return B2K_OK;
  }));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(F_d, F.data(), m * sizeof(EvForest), cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(off_d, tree_offsets, off0 * 8, cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(nodes_d, pn.data(), node0 * sizeof(B2kPNode), cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(val_d, value, val0 * 8, cudaMemcpyHostToDevice, s));
  ForestArgs a{X, y, n, d, dpad, TR, m, 0, F_d, off_d, nodes_d, val_d, 0.0, nullptr, 1, nullptr, nullptr, nullptr};
  const ScoreOut o{scores, ld_scores, pos};
  if (vec) k_score_forest<true><<<grid, EV_NT, smem, s>>>(a, o);
  else k_score_forest<false><<<grid, EV_NT, smem, s>>>(a, o);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  return B2K_OK;
}

int b2k_eval_linear_impl(b2k_ctx* ctx, const float* X, const float* y, int64_t n, int d, int m, const int32_t* kind,
                         const int32_t* row_offsets, const double* W, const double* b, const double* class_values,
                         int n_classes, double eps, int64_t* label_count_out, int64_t* tp_out, int64_t* fp_out,
                         double* loss_out, double* reg_out, cudaStream_t s) {
  if (d > B2K_LOGREG_MAX_D)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "evaluation supports d <= " + std::to_string(B2K_LOGREG_MAX_D));
  const bool cls = kind[0] != B2K_EVAL_IDENTITY;
  int nrows = 0, kmax = 1, ncls = 0, max_cls = -1;
  std::vector<int> cls0(m + 1, 0);
  for (int i = 0; i < m; ++i) {
    const int kp = row_offsets[i + 1] - row_offsets[i];
    if ((kind[i] != B2K_EVAL_IDENTITY) != cls || kind[i] < 0 || kind[i] > B2K_EVAL_SOFTMAX ||
        (kind[i] == B2K_EVAL_SOFTMAX ? kp < 2 : kp != 1) || row_offsets[i] != nrows)
      return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_eval_linear: model " + std::to_string(i) +
                                                " has a bad kind or row range (kinds may not mix regression and "
                                                "classification; identity and logistic hold 1 row, softmax >= 2)");
    nrows += kp;
    kmax = std::max(kmax, kp);
    cls0[i] = ncls;
    if (cls) ncls += kp == 1 ? 2 : kp;
  }
  cls0[m] = ncls;
  for (int i = 0; i < ncls; ++i) {
    const double v = class_values[i];
    if (!(v >= 0.0 && v < B2K_LOGREG_MAX_CLASSES && v == std::floor(v)))
      return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_eval_linear: class value " + num(v) + " is not an integer in [0, " +
                                                std::to_string(B2K_LOGREG_MAX_CLASSES) + ")");
    max_cls = std::max(max_cls, (int)v);
  }
  int C = 0;
  if (cls) {
    B2K_TRY(check_labels(ctx, y, n, &C, s));
    C = std::max(C, max_cls + 1);
    if (C != n_classes)
      return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_eval_linear: n_classes must be " + std::to_string(C) +
                                                " (1 + the largest label or class value), got " + std::to_string(n_classes));
    std::fill(label_count_out, label_count_out + C, 0);
    std::fill(tp_out, tp_out + (size_t)m * C, 0);
    std::fill(fp_out, fp_out + (size_t)m * C, 0);
    std::fill(loss_out, loss_out + m, 0.0);
  } else {
    std::fill(reg_out, reg_out + (size_t)m * NREG, 0.0);
  }
  if (n == 0) return B2K_OK;
  const int dpad = (d + 3) & ~3, L = b2k_row_lanes(d);
  const int TR = tile_rows(dpad, EV_NW * (32 / L), EV_TILE_BYTES);
  const bool vec = d % 4 == 0 && (reinterpret_cast<uintptr_t>(X) & 15u) == 0;
  std::vector<double> Wp((size_t)nrows * dpad, 0.0);
  for (int r = 0; r < nrows; ++r) std::copy(W + (size_t)r * d, W + (size_t)(r + 1) * d, Wp.begin() + (size_t)r * dpad);
  const int np = cls ? 1 : NREG;
  for (int first = 0; first < m; ) {
    const int last = chunk_end(first, m, TR, dpad, C, cls), mc = last - first;
    const size_t smem = ev_carve(TR, dpad, mc, C, cls).bytes;
    if (smem > EV_SMEM_MAX)
      return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "evaluation: one model needs " + std::to_string(smem) +
                                                    " bytes of shared memory, above " + std::to_string(EV_SMEM_MAX));
    const void* kern = cls ? (vec ? (const void*)k_eval_linear<true, true> : (const void*)k_eval_linear<false, true>)
                           : (vec ? (const void*)k_eval_linear<true, false> : (const void*)k_eval_linear<false, false>);
    int kmc = 1;
    for (int i = first; i < last; ++i) kmc = std::max(kmc, row_offsets[i + 1] - row_offsets[i]);
    const int rps = EV_NW * (32 / L);
    int grid = 0;
    B2K_TRY(pass_grid(ctx, kern, smem, n, TR, &grid));
    const int w0 = row_offsets[first], nr = row_offsets[last] - w0;
    int *kind_d, *row0_d, *cls0_d;
    double *W_d, *b_d, *cls_d, *slots, *part, *folded;
    unsigned long long *counts, *labels;
    B2K_TRY(b2k_scratch_layout(ctx, "evaluation", [&](B2kLayout& Ly) -> int {
      kind_d = Ly.take<int>(mc);
      row0_d = Ly.take<int>(mc + 1);
      cls0_d = Ly.take<int>(mc + 1);
      W_d = Ly.take<double>((size_t)nr * dpad);
      b_d = Ly.take<double>(nr);
      cls_d = Ly.take<double>(std::max(1, cls0[last] - cls0[first]));
      slots = Ly.take<double>(kmc > 1 ? (size_t)grid * rps * kmc : 1);
      part = Ly.take<double>((size_t)grid * mc * np);
      folded = Ly.take<double>((size_t)mc * np);
      counts = Ly.take<unsigned long long>(cls ? (size_t)mc * 2 * C : 1);
      labels = Ly.take<unsigned long long>(cls ? C : 1);
      return B2K_OK;
    }));
    std::vector<int> r0h(mc + 1), c0h(mc + 1);
    for (int i = 0; i <= mc; ++i) {
      r0h[i] = row_offsets[first + i] - w0;
      c0h[i] = cls0[first + i] - cls0[first];
    }
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(kind_d, kind + first, mc * 4, cudaMemcpyHostToDevice, s));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(row0_d, r0h.data(), (mc + 1) * 4, cudaMemcpyHostToDevice, s));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(cls0_d, c0h.data(), (mc + 1) * 4, cudaMemcpyHostToDevice, s));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(W_d, Wp.data() + (size_t)w0 * dpad, (size_t)nr * dpad * 8, cudaMemcpyHostToDevice, s));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(b_d, b + w0, (size_t)nr * 8, cudaMemcpyHostToDevice, s));
    if (cls0[last] > cls0[first])
      B2K_CUDA_OK(ctx, cudaMemcpyAsync(cls_d, class_values + cls0[first], (size_t)(cls0[last] - cls0[first]) * 8,
                                       cudaMemcpyHostToDevice, s));
    if (cls) {
      B2K_CUDA_OK(ctx, cudaMemsetAsync(counts, 0, (size_t)mc * 2 * C * 8, s));
      B2K_CUDA_OK(ctx, cudaMemsetAsync(labels, 0, (size_t)C * 8, s));
    }
    LinArgs a{X, y, n, d, dpad, L, TR, mc, C, kind_d, row0_d, W_d, b_d, cls0_d, cls_d, eps, slots, kmc,
              cls && first == 0 ? labels : nullptr, counts, part};
    if (cls) {
      if (vec) k_eval_linear<true, true><<<grid, EV_NT, smem, s>>>(a);
      else k_eval_linear<false, true><<<grid, EV_NT, smem, s>>>(a);
    } else {
      if (vec) k_eval_linear<true, false><<<grid, EV_NT, smem, s>>>(a);
      else k_eval_linear<false, false><<<grid, EV_NT, smem, s>>>(a);
    }
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
    B2K_TRY(finish_chunk(ctx, cls, first, mc, C, n, grid, part, folded, counts, first == 0 ? labels : nullptr,
                         label_count_out, tp_out, fp_out, loss_out, reg_out, s));
    first = last;
  }
  return B2K_OK;
}

int b2k_eval_forest_impl(b2k_ctx* ctx, const float* X, const float* y, int64_t n, int d, int m, int classification,
                         const int32_t* n_trees, const int32_t* n_values, const int64_t* tree_offsets,
                         const int32_t* feature, const float* threshold, const int32_t* children, const double* value,
                         int n_classes, double eps, int64_t* label_count_out, int64_t* tp_out, int64_t* fp_out,
                         double* loss_out, double* reg_out, cudaStream_t s) {
  const bool cls = classification != 0;
  std::vector<EvForest> F(m);
  int64_t off0 = 0, node0 = 0, val0 = 0;
  int vmax = 1;
  B2K_TRY(forest_table(ctx, "b2k_eval_forest", m, d, cls ? 1 : 0, n_trees, n_values, tree_offsets, feature, F, off0,
                       node0, val0, vmax));
  int C = 0;
  if (cls) {
    B2K_TRY(check_labels(ctx, y, n, &C, s));
    C = std::max(C, vmax);
    if (C != n_classes)
      return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_eval_forest: n_classes must be " + std::to_string(C) +
                                                " (1 + the largest label, or the most values of a forest), got " +
                                                std::to_string(n_classes));
    std::fill(label_count_out, label_count_out + C, 0);
    std::fill(tp_out, tp_out + (size_t)m * C, 0);
    std::fill(fp_out, fp_out + (size_t)m * C, 0);
    std::fill(loss_out, loss_out + m, 0.0);
  } else {
    std::fill(reg_out, reg_out + (size_t)m * NREG, 0.0);
  }
  if (n == 0) return B2K_OK;
  std::vector<B2kPNode> pn((size_t)node0);
  for (int64_t j = 0; j < node0; ++j)
    pn[j] = B2kPNode{feature[j], threshold[j], children[2 * j], children[2 * j + 1]};
  const int dpad = (d + 3) & ~3;
  const int TR = tile_rows(dpad, 1, EV_FTILE_BYTES);
  const bool vec = d % 4 == 0 && (reinterpret_cast<uintptr_t>(X) & 15u) == 0;
  const int np = cls ? 1 : NREG;
  for (int first = 0; first < m; ) {
    const int last = chunk_end(first, m, TR, dpad, C, cls), mc = last - first;
    const size_t smem = ev_carve(TR, dpad, mc, C, cls).bytes;
    if (smem > EV_SMEM_MAX)
      return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "evaluation: one forest needs " + std::to_string(smem) +
                                                    " bytes of shared memory, above " + std::to_string(EV_SMEM_MAX));
    const void* kern = cls ? (vec ? (const void*)k_eval_forest<true, true> : (const void*)k_eval_forest<false, true>)
                           : (vec ? (const void*)k_eval_forest<true, false> : (const void*)k_eval_forest<false, false>);
    int vmc = 1;
    for (int i = first; i < last; ++i) vmc = std::max(vmc, F[i].V);
    int grid = 0;
    B2K_TRY(pass_grid(ctx, kern, smem, n, TR, &grid));
    const int64_t o0 = F[first].off0, n0 = F[first].node0, v0 = F[first].val0;
    const int64_t o1 = last < m ? F[last].off0 : off0, n1 = last < m ? F[last].node0 : node0,
                  v1 = last < m ? F[last].val0 : val0;
    std::vector<EvForest> Fc(F.begin() + first, F.begin() + last);
    for (auto& f : Fc) {
      f.off0 -= o0;
      f.node0 -= n0;
      f.val0 -= v0;
    }
    EvForest* F_d;
    int64_t* off_d;
    B2kPNode* nodes_d;
    double *val_d, *slots, *part, *folded;
    unsigned long long *counts, *labels;
    B2K_TRY(b2k_scratch_layout(ctx, "evaluation", [&](B2kLayout& Ly) -> int {
      F_d = Ly.take<EvForest>(mc);
      off_d = Ly.take<int64_t>(o1 - o0);
      nodes_d = Ly.take<B2kPNode>(n1 - n0);
      val_d = Ly.take<double>(v1 - v0);
      slots = Ly.take<double>(cls ? (size_t)grid * EV_NT * vmc : 1);
      part = Ly.take<double>((size_t)grid * mc * np);
      folded = Ly.take<double>((size_t)mc * np);
      counts = Ly.take<unsigned long long>(cls ? (size_t)mc * 2 * C : 1);
      labels = Ly.take<unsigned long long>(cls ? C : 1);
      return B2K_OK;
    }));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(F_d, Fc.data(), mc * sizeof(EvForest), cudaMemcpyHostToDevice, s));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(off_d, tree_offsets + o0, (o1 - o0) * 8, cudaMemcpyHostToDevice, s));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(nodes_d, pn.data() + n0, (n1 - n0) * sizeof(B2kPNode), cudaMemcpyHostToDevice, s));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(val_d, value + v0, (v1 - v0) * 8, cudaMemcpyHostToDevice, s));
    if (cls) {
      B2K_CUDA_OK(ctx, cudaMemsetAsync(counts, 0, (size_t)mc * 2 * C * 8, s));
      B2K_CUDA_OK(ctx, cudaMemsetAsync(labels, 0, (size_t)C * 8, s));
    }
    ForestArgs a{X, y, n, d, dpad, TR, mc, C, F_d, off_d, nodes_d, val_d, eps, slots, vmc,
                 cls && first == 0 ? labels : nullptr, counts, part};
    if (cls) {
      if (vec) k_eval_forest<true, true><<<grid, EV_NT, smem, s>>>(a);
      else k_eval_forest<false, true><<<grid, EV_NT, smem, s>>>(a);
    } else {
      if (vec) k_eval_forest<true, false><<<grid, EV_NT, smem, s>>>(a);
      else k_eval_forest<false, false><<<grid, EV_NT, smem, s>>>(a);
    }
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
    B2K_TRY(finish_chunk(ctx, cls, first, mc, C, n, grid, part, folded, counts, first == 0 ? labels : nullptr,
                         label_count_out, tp_out, fp_out, loss_out, reg_out, s));
    first = last;
  }
  return B2K_OK;
}
