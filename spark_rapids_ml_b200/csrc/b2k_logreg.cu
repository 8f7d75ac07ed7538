// Logistic regression (sm_90a): the label pass, the loss-and-gradient passes, the host L-BFGS / OWL-QN and prediction.
//
//   labels   k_logreg_labels: per-CTA counts of the values in [0, 1024), min, max, least non-integer value and the fp64
//            sum, folded in span order; one allgather of every rank's [counts | min | max | non-integer | sum | n], reduced
//            on the host in rank order, so every rank derives the same classes.
//   moments  b2k_colstats_impl (b2k_pca.cu): column sums, then centred squares on mu32, fp64, span-ordered partials.
//   eval     the loss (1/n) sum l(W x + b, y) and its gradient at (W, b), fp64 throughout:
//              fused   k_logreg_eval: a CTA owns a span of rows and stages tiles of them in shared memory; lanes over
//                      rows form the margins from the staged tile, one thread per row forms its residuals r = p - onehot(y)
//                      and loss, threads over (feature, class block) accumulate sum r_k x_j from the same tile.  Each row
//                      of X is read once per evaluation.
//              generic k_logreg_rows writes the residuals of a chunk of rows (capped at 64 MB), then k_logreg_xtr forms
//                      X^T R in k_xty's layout.  Every shape d <= 1024, any class count.
//            Partials [K'][d + 1] (coefficients, then the intercept) + loss, per CTA or span, folded in order; one f64
//            allreduce per evaluation.
//   solve    host, fp64: L-BFGS (memory 10, strong-Wolfe line search of at most 20 evaluations), OWL-QN with an L1 term;
//            stopped on Breeze's rules as MLlib applies them.
//   predict  k_logreg_rows: rawPrediction, probability and prediction in one pass.
// No floating-point atomics: two evaluations of the same input are bitwise equal.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "b2k_internal.cuh"
#include "b2k_rows.cuh"

namespace {

constexpr int LR_THREADS = 256;
constexpr int MAXC = B2K_LOGREG_MAX_CLASSES;
constexpr int LB_W = MAXC + 4;   // label partial: [counts | min | max | least non-integer | sum]

// ------------------------------------------------------------------------------------------------
// label pass
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(LR_THREADS)
k_logreg_labels(const float* __restrict__ y, int64_t n, int64_t span_rows, double* __restrict__ part) {
  __shared__ unsigned int cnt[MAXC];
  __shared__ float mn_s[LR_THREADS], mx_s[LR_THREADS], ni_s[LR_THREADS];
  __shared__ double sum_s[LR_THREADS];
  for (int i = threadIdx.x; i < MAXC; i += LR_THREADS) cnt[i] = 0u;
  __syncthreads();
  const int64_t r0 = (int64_t)blockIdx.x * span_rows, r1 = min(n, r0 + span_rows);
  float mn = INFINITY, mx = -INFINITY, ni = INFINITY;
  double s = 0.0;
  for (int64_t r = r0 + threadIdx.x; r < r1; r += LR_THREADS) {
    const float v = y[r];
    s += (double)v;
    mn = fminf(mn, v);
    mx = fmaxf(mx, v);
    const bool integral = v == floorf(v);
    if (!integral) ni = fminf(ni, v);
    // integer counts: the order of the shared-memory increments does not change them
    if (integral && v >= 0.f && v < (float)MAXC) atomicAdd(&cnt[(int)v], 1u);
  }
  mn_s[threadIdx.x] = mn;
  mx_s[threadIdx.x] = mx;
  ni_s[threadIdx.x] = ni;
  sum_s[threadIdx.x] = s;
  __syncthreads();
  for (int o = LR_THREADS / 2; o > 0; o >>= 1) {   // a fixed tree: the sum's order depends on the span alone
    if (threadIdx.x < o) {
      mn_s[threadIdx.x] = fminf(mn_s[threadIdx.x], mn_s[threadIdx.x + o]);
      mx_s[threadIdx.x] = fmaxf(mx_s[threadIdx.x], mx_s[threadIdx.x + o]);
      ni_s[threadIdx.x] = fminf(ni_s[threadIdx.x], ni_s[threadIdx.x + o]);
      sum_s[threadIdx.x] += sum_s[threadIdx.x + o];
    }
    __syncthreads();
  }
  double* p = part + (size_t)blockIdx.x * LB_W;
  for (int i = threadIdx.x; i < MAXC; i += LR_THREADS) p[i] = (double)cnt[i];
  if (threadIdx.x == 0) {
    p[MAXC] = mn_s[0];
    p[MAXC + 1] = mx_s[0];
    p[MAXC + 2] = ni_s[0];
    p[MAXC + 3] = sum_s[0];
  }
}

// out [LB_W + 1]: the spans folded in order, then n
__global__ void k_logreg_labels_fold(const double* __restrict__ part, int spans, int64_t n, double* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c > LB_W) return;
  if (c == LB_W) {
    out[c] = (double)n;
    return;
  }
  double t = c == MAXC ? INFINITY : c == MAXC + 1 ? -INFINITY : c == MAXC + 2 ? INFINITY : 0.0;
  for (int s = 0; s < spans; ++s) {
    const double v = part[(size_t)s * LB_W + c];
    if (c == MAXC || c == MAXC + 2) t = fmin(t, v);
    else if (c == MAXC + 1) t = fmax(t, v);
    else t += v;
  }
  out[c] = t;
}

// ------------------------------------------------------------------------------------------------
// fused evaluation pass
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void cp_async4(float* smem, const float* gmem) {
  const unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(sa), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

struct EvalArgs {
  const float* X;
  const float* y;
  const int* cmap;     // [MAXC] label value -> class index, -1 = none
  const double* W;     // [kp][d]
  const double* b;     // [kp]
  int64_t n;
  int d, kp, tr;       // tr: rows per staged tile
  int64_t span_rows;   // a multiple of tr
  double* part;        // [grid][rg][kp (d + 1) + 1]
};

__host__ __device__ inline int tile_stride(int d) { return (d & 1) ? d + 2 : d + 1; }   // odd: conflict-free row reads
__host__ __device__ inline int tile_rows(int d) { return d <= 128 ? 64 : d <= 256 ? 32 : d <= 512 ? 16 : 8; }

struct FusedShape {   // derived from (d, kp) alone, identically on host and device
  int nkb, parts, fs_n, items, rg;
};
__host__ __device__ inline FusedShape fused_shape(int d, int kp, int KB, int tr) {
  FusedShape f;
  f.nkb = (kp + KB - 1) / KB;
  f.parts = LR_THREADS / tr;
  f.fs_n = f.nkb >= f.parts ? 1 : f.parts / f.nkb;
  f.items = d * f.nkb;
  f.rg = f.items >= LR_THREADS ? 1 : min(tr, LR_THREADS / f.items);
  return f;
}
__host__ __device__ inline size_t fused_smem(int d, int kp, int KB) {
  const int tr = tile_rows(d);
  const FusedShape f = fused_shape(d, kp, KB, tr);
  const size_t dbl = (size_t)kp * d + kp + (size_t)f.fs_n * tr * kp + 2 * (size_t)tr * kp + tr;
  return dbl * 8 + 2 * (size_t)tr * tile_stride(d) * 4;
}

// Thread roles per tile of tr rows, all from the staged tile x_s [tr][ds]:
//   margins    thread (row = t % tr, part = t / tr): items (class block kb, feature slice fs) of the parts; a slice is a
//              contiguous feature range summed in order, the row's thread then adds b and the slices in order.
//   residuals  thread t < tr: row t's margins -> residuals r_s [tr][kp], loss and intercept sums per row slot.
//   gradient   thread (row group, item = kb * d + j): acc[kk] += r[row][kb KB + kk] x[row][j] over its rows in order.
// The next tile streams into the second buffer (cp.async) while the current one is processed.
template <int KB, int NIT>
__global__ void __launch_bounds__(LR_THREADS, KB == 1 ? 3 : 2) k_logreg_eval(EvalArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int d = a.d, kp = a.kp, tr = a.tr, ds = tile_stride(d);
  const FusedShape fs = fused_shape(d, kp, KB, tr);
  double* w_s = reinterpret_cast<double*>(smem_raw);   // [kp][d]
  double* b_s = w_s + (size_t)kp * d;                   // [kp]
  double* mp_s = b_s + kp;                              // [fs_n][tr][kp] partial margins
  double* r_s = mp_s + (size_t)fs.fs_n * tr * kp;       // [tr][kp]
  double* ib_s = r_s + (size_t)tr * kp;                 // [tr][kp] intercept sums per row slot
  double* ls_s = ib_s + (size_t)tr * kp;                // [tr] loss per row slot
  float* x_buf = reinterpret_cast<float*>(ls_s + tr);   // [2][tr][ds]: the tile in use and the next one
  const int tid = threadIdx.x;
  for (int i = tid; i < kp * d; i += LR_THREADS) w_s[i] = a.W[i];
  for (int i = tid; i < kp; i += LR_THREADS) b_s[i] = a.b[i];
  for (int i = tid; i < tr * kp; i += LR_THREADS) ib_s[i] = 0.0;
  for (int i = tid; i < tr; i += LR_THREADS) ls_s[i] = 0.0;

  const int64_t r0 = (int64_t)blockIdx.x * a.span_rows, r1 = min(a.n, r0 + a.span_rows);
  // staging: the tile is the contiguous range X[t0 * d, (t0 + rows) * d); thread tid copies elements tid + 256 i with
  // 4-byte cp.async into row (e / d), column (e % d) of the padded tile, the indices stepped incrementally
  const int srow = LR_THREADS / d, scol = LR_THREADS % d;
  const int row0 = tid / d, col0 = tid % d;
  auto load_tile = [&](int64_t t0, int rows, float* dst_tile) {
    const int cnt = rows * d;
    const float* src = a.X + t0 * d;
    int row = row0, col = col0;
    for (int f = tid; f < cnt; f += LR_THREADS) {
      cp_async4(dst_tile + row * ds + col, src + f);
      row += srow;
      col += scol;
      if (col >= d) {
        col -= d;
        ++row;
      }
    }
    cp_async_commit();
  };

  // gradient roles
  int item0, rg;
  if (fs.items >= LR_THREADS) {
    item0 = tid;
    rg = 0;
  } else {
    item0 = tid % fs.items;
    rg = tid / fs.items;
  }
  const bool g_active = rg < fs.rg;
  double acc[NIT][KB];
#pragma unroll
  for (int i = 0; i < NIT; ++i)
#pragma unroll
    for (int kk = 0; kk < KB; ++kk) acc[i][kk] = 0.0;

  if (r0 < r1) load_tile(r0, (int)(r1 - r0 < tr ? r1 - r0 : tr), x_buf);
  int buf = 0;
  for (int64_t t0 = r0; t0 < r1; t0 += tr, buf ^= 1) {
    const int rows = (int)(r1 - t0 < tr ? r1 - t0 : tr);
    float* x_s = x_buf + buf * tr * ds;
    __syncthreads();   // the readers of the other buffer (the previous tile) are done
    if (t0 + tr < r1) {
      load_tile(t0 + tr, (int)(r1 - t0 - tr < tr ? r1 - t0 - tr : tr), x_buf + (buf ^ 1) * tr * ds);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();   // this tile is in shared memory for every thread
    {   // margins
      const int row = tid % tr, part = tid / tr;
      const float* xr = x_s + row * ds;
      for (int it = part; it < fs.nkb * fs.fs_n; it += fs.parts) {
        const int kb = it / fs.fs_n, sl = it - kb * fs.fs_n;
        const int j0 = sl * d / fs.fs_n, j1 = (sl + 1) * d / fs.fs_n;
        double m[KB];
#pragma unroll
        for (int kk = 0; kk < KB; ++kk) m[kk] = 0.0;
        for (int j = j0; j < j1; ++j) {
          const double xv = (double)xr[j];
#pragma unroll
          for (int kk = 0; kk < KB; ++kk) {
            const int k = kb * KB + kk;
            if (k < kp) m[kk] = fma(xv, w_s[(size_t)k * d + j], m[kk]);
          }
        }
#pragma unroll
        for (int kk = 0; kk < KB; ++kk) {
          const int k = kb * KB + kk;
          if (k < kp) mp_s[((size_t)sl * tr + row) * kp + k] = m[kk];
        }
      }
    }
    __syncthreads();
    if (tid < tr) {   // residuals, loss, intercept sums
      double* rr = r_s + (size_t)tid * kp;
      if (tid < rows) {
        for (int k = 0; k < kp; ++k) {
          double m = b_s[k];
          for (int sl = 0; sl < fs.fs_n; ++sl) m += mp_s[((size_t)sl * tr + tid) * kp + k];
          rr[k] = m;
        }
        const double l = b2k_row_loss_residual(rr, kp, b2k_class_of(a.y[t0 + tid], a.cmap, MAXC));
        ls_s[tid] += l;
        for (int k = 0; k < kp; ++k) ib_s[(size_t)tid * kp + k] += rr[k];
      }
    }
    __syncthreads();
    if (g_active) {   // X^T R
#pragma unroll
      for (int i = 0; i < NIT; ++i) {
        const int item = item0 + LR_THREADS * i;
        if ((i > 0 && fs.items < LR_THREADS) || item >= fs.items) continue;
        const int kb = item / d, j = item - kb * d;
        for (int row = rg; row < rows; row += fs.rg) {
          const double xv = (double)x_s[row * ds + j];
          const double* rr = r_s + (size_t)row * kp + kb * KB;
#pragma unroll
          for (int kk = 0; kk < KB; ++kk)
            if (kb * KB + kk < kp) acc[i][kk] = fma(rr[kk], xv, acc[i][kk]);
        }
      }
    }
  }
  __syncthreads();
  const int M = kp * (d + 1) + 1;
  double* out = a.part + ((size_t)blockIdx.x * fs.rg + (g_active ? rg : 0)) * M;
  if (g_active) {
#pragma unroll
    for (int i = 0; i < NIT; ++i) {
      const int item = item0 + LR_THREADS * i;
      if ((i > 0 && fs.items < LR_THREADS) || item >= fs.items) continue;
      const int kb = item / d, j = item - kb * d;
#pragma unroll
      for (int kk = 0; kk < KB; ++kk) {
        const int k = kb * KB + kk;
        if (k < kp) out[(size_t)k * (d + 1) + j] = acc[i][kk];
      }
    }
  }
  // intercept sums and loss: row slots folded in order into row group 0's slot, zeros in the others
  double* base = a.part + (size_t)blockIdx.x * fs.rg * M;
  for (int k = tid; k <= kp; k += LR_THREADS) {
    double t = 0.0;
    if (k < kp)
      for (int r = 0; r < tr; ++r) t += ib_s[(size_t)r * kp + k];
    else
      for (int r = 0; r < tr; ++r) t += ls_s[r];
    const size_t idx = k < kp ? (size_t)k * (d + 1) + d : (size_t)M - 1;
    base[idx] = t;
    for (int g = 1; g < fs.rg; ++g) base[(size_t)g * M + idx] = 0.0;
  }
}

// ------------------------------------------------------------------------------------------------
// generic rows kernel (evaluation path and transform)
// ------------------------------------------------------------------------------------------------
// A group of L lanes owns one row, as in k_linreg_predict: lane l accumulates features 4 (l + L i) .. + 3 in order in fp64
// for a chunk of 8 classes, then the group adds its lanes by a fixed xor butterfly.  Lane 0 of the group writes the
// margins, then forms the row's outputs serially over the classes.
//   TRAIN:   R [row][kp] = p - onehot(y), loss [row]
//   PREDICT: raw [row][nout], prob [row][nout], pred [row] (nout = 2 for kp == 1: raw = [-m, m])
constexpr int RC = 8;
template <bool VEC, bool TRAIN>
__global__ void __launch_bounds__(LR_THREADS)
k_logreg_rows(const float* __restrict__ X, int64_t n, int d, int kp, const double* __restrict__ W,
              const double* __restrict__ b, int L, const float* __restrict__ y, const int* __restrict__ cmap,
              double* __restrict__ R, double* __restrict__ loss, const double* __restrict__ cls_val,
              double* __restrict__ raw, double* __restrict__ prob, double* __restrict__ pred) {
  const int lane = threadIdx.x & 31, sub = lane & (L - 1), grp = lane / L, rpw = 32 / L;
  const int64_t warp = ((int64_t)blockIdx.x * LR_THREADS + threadIdx.x) >> 5;
  const int64_t nwarp = ((int64_t)gridDim.x * LR_THREADS) >> 5;
  const int nout = kp == 1 ? 2 : kp;
  for (int64_t rbase = warp * rpw; rbase < n; rbase += nwarp * rpw) {
    const int64_t row = rbase + grp;
    const bool valid = row < n;
    const float* x = X + (valid ? row : 0) * d;
    double* mrow = TRAIN ? R + (valid ? row : 0) * kp : raw + (valid ? row : 0) * nout;
    for (int k0 = 0; k0 < kp; k0 += RC) {
      double acc[RC];
#pragma unroll
      for (int q = 0; q < RC; ++q) acc[q] = 0.0;
      if (valid) b2k_logistic_lanes<RC>(B2kRowLdg<VEC>{x, d}, d, kp, k0, W, d, sub, L, acc);
#pragma unroll
      for (int q = 0; q < RC; ++q) acc[q] = b2k_lanes_sum(acc[q], L);
      if (sub == 0 && valid) {
#pragma unroll
        for (int q = 0; q < RC; ++q) {
          const int k = k0 + q;
          if (k < kp) mrow[(kp == 1 && !TRAIN) ? 1 : k] = b[k] + acc[q];
        }
      }
    }
    if (sub != 0 || !valid) continue;
    if (TRAIN) {
      loss[row] = b2k_row_loss_residual(mrow, kp, b2k_class_of(y[row], cmap, MAXC));
    } else if (kp == 1) {
      const double m = mrow[1];
      const double p1 = b2k_sigmoid(m);
      mrow[0] = -m;
      prob[row * 2 + 0] = 1.0 - p1;
      prob[row * 2 + 1] = p1;
      pred[row] = cls_val[m > 0.0 ? 1 : 0];
    } else {
      const B2kArgmax ax = b2k_softmax_argmax(mrow, kp);
      const double mx = ax.mx;
      const int am = ax.am;
      const double s = b2k_softmax_denominator(mrow, kp, mx);
      for (int k = 0; k < kp; ++k) prob[row * kp + k] = exp(mrow[k] - mx) / s;
      pred[row] = cls_val[am];
    }
  }
}

// part[span][k (d + 1) + c] = sum over the span's rows of R[row][k] x[row][c] (c == d: x = 1, the intercept), and
// part[span][kp (d + 1)] = the span's loss sum.  CTA: 32 columns x 8 row lanes (as k_xty), blockIdx.z = class.
constexpr int XR_TX = 32, XR_TY = 8;
__global__ void __launch_bounds__(XR_TX * XR_TY)
k_logreg_xtr(const float* __restrict__ X, int64_t rows, int d, int kp, const double* __restrict__ R,
             const double* __restrict__ loss, int64_t span_rows, double* __restrict__ part) {
  __shared__ double red[XR_TY][XR_TX];
  const int c = blockIdx.y * XR_TX + threadIdx.x, k = blockIdx.z;
  const int m = kp * (d + 1) + 1;
  const int64_t r0 = (int64_t)blockIdx.x * span_rows, r1 = min(rows, r0 + span_rows);
  double s = 0.0;
  if (c < d) {
#pragma unroll 4
    for (int64_t r = r0 + threadIdx.y; r < r1; r += XR_TY) s = fma(R[r * kp + k], (double)X[r * d + c], s);
  } else if (c == d) {
    for (int64_t r = r0 + threadIdx.y; r < r1; r += XR_TY) s += R[r * kp + k];
  } else if (c == d + 1 && k == 0) {
    for (int64_t r = r0 + threadIdx.y; r < r1; r += XR_TY) s += loss[r];
  }
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0) {
    double t = 0.0;
    for (int q = 0; q < XR_TY; ++q) t += red[q][threadIdx.x];
    double* p = part + (size_t)blockIdx.x * m;
    if (c <= d) p[(size_t)k * (d + 1) + c] = t;
    else if (c == d + 1 && k == 0) p[m - 1] = t;
  }
}

int row_lanes(int d) { return b2k_row_lanes(d); }

// ------------------------------------------------------------------------------------------------
// fused dispatch
// ------------------------------------------------------------------------------------------------
using EvalKernel = void (*)(EvalArgs);
struct FusedPick {
  int KB = 0, NIT = 0;
  EvalKernel kern = nullptr;
};
// The instantiations: classes per thread KB, items (feature, class block) per thread NIT.
FusedPick fused_pick(int d, int kp) {
  FusedPick p;
  if (kp <= 1) { p.KB = 1; p.NIT = 4; }
  else if (kp <= 2) { p.KB = 2; p.NIT = 4; }
  else if (kp <= 4) { p.KB = 4; p.NIT = 4; }
  else if (kp <= 8) { p.KB = 8; p.NIT = 2; }
  else { p.KB = 16; p.NIT = 1; }
  const int nkb = (kp + p.KB - 1) / p.KB;
  if (d > B2K_LOGREG_MAX_D || (int64_t)d * nkb > (int64_t)LR_THREADS * p.NIT) return FusedPick{};
  switch (p.KB) {
    case 1: p.kern = k_logreg_eval<1, 4>; break;
    case 2: p.kern = k_logreg_eval<2, 4>; break;
    case 4: p.kern = k_logreg_eval<4, 4>; break;
    case 8: p.kern = k_logreg_eval<8, 2>; break;
    default: p.kern = k_logreg_eval<16, 1>; break;
  }
  return p;
}

bool fused_fits(const b2k_ctx* ctx, int d, int kp) {
  const FusedPick p = fused_pick(d, kp);
  return p.kern && fused_smem(d, kp, p.KB) <= ctx->smem_optin;
}

std::string num(double v) {   // Python's repr of a float
  if (std::isnan(v)) return "nan";
  if (std::isinf(v)) return v > 0 ? "inf" : "-inf";
  char buf[64];
  for (int p = 1; p <= 17; ++p) {
    snprintf(buf, sizeof buf, "%.*g", p, v);
    if (std::strtod(buf, nullptr) == v) break;
  }
  std::string t(buf);
  if (t.find_first_of(".eni") == std::string::npos) t += ".0";
  return t;
}

bool finite_all(const double* v, size_t m) {
  for (size_t i = 0; i < m; ++i)
    if (!std::isfinite(v[i])) return false;
  return true;
}

// ------------------------------------------------------------------------------------------------
// host optimizer
// ------------------------------------------------------------------------------------------------
constexpr int LBFGS_M = 10;      // memory (the reference's lbfgs_memory)
constexpr int LS_MAX_EVALS = 20; // evaluations per line search (the reference's linesearch_max_iter)
constexpr int FVAL_MEMORY = 20;  // Breeze's history of function values for its convergence rule

double dot(const std::vector<double>& a, const std::vector<double>& b) {
  double s = 0.0;
  for (size_t i = 0; i < a.size(); ++i) s += a[i] * b[i];
  return s;
}
double norm2(const std::vector<double>& a) { return std::sqrt(dot(a, a)); }

struct Objective {
  b2k_logreg_objective fn;
  void* user;
  const double* l1;   // per-coordinate L1 weights or NULL
  int n;
  int evals = 0;
  int status = B2K_OK;
  // smooth value and gradient at x
  bool eval(const std::vector<double>& x, double* f, std::vector<double>* g) {
    ++evals;
    status = fn(user, n, x.data(), f, g->data());
    return status == B2K_OK;
  }
  double l1_term(const std::vector<double>& x) const {
    if (!l1) return 0.0;
    double s = 0.0;
    for (int i = 0; i < n; ++i) s += l1[i] * std::fabs(x[i]);
    return s;
  }
  // OWL-QN pseudo-gradient of f + sum l1 |x|
  void pseudo_grad(const std::vector<double>& x, const std::vector<double>& g, std::vector<double>* pg) const {
    for (int i = 0; i < n; ++i) {
      const double w = l1 ? l1[i] : 0.0;
      if (w == 0.0) (*pg)[i] = g[i];
      else if (x[i] > 0.0) (*pg)[i] = g[i] + w;
      else if (x[i] < 0.0) (*pg)[i] = g[i] - w;
      else if (g[i] + w < 0.0) (*pg)[i] = g[i] + w;
      else if (g[i] - w > 0.0) (*pg)[i] = g[i] - w;
      else (*pg)[i] = 0.0;
    }
  }
};

// cubic minimiser of the interpolant through (a, fa, da) and (b, fb, db), safeguarded into [lo + 0.1 w, hi - 0.1 w]
double interpolate(double a, double fa, double da, double b, double fb, double db) {
  const double lo = std::min(a, b), hi = std::max(a, b), w = hi - lo;
  const double d1 = da + db - 3.0 * (fa - fb) / (a - b);
  const double disc = d1 * d1 - da * db;
  double t = 0.5 * (a + b);
  if (disc >= 0.0) {
    const double d2 = (b > a ? 1.0 : -1.0) * std::sqrt(disc);
    const double den = db - da + 2.0 * d2;
    if (den != 0.0) t = b - (b - a) * (db + d2 - d1) / den;
  }
  if (!std::isfinite(t)) t = 0.5 * (a + b);
  return std::min(std::max(t, lo + 0.1 * w), hi - 0.1 * w);
}

}  // namespace

int b2k_logreg_minimize_impl(b2k_logreg_objective fn, void* user, int n, double* x_io, const double* l1, int max_iter,
                             double tol, int* n_iter_out, int* n_eval_out, double* f_out, std::vector<double>* f_hist) {
  auto fail = [](int code, const std::string& msg) { return b2k_fail(nullptr, code, msg); };
  if (!fn || !x_io || n < 1) return fail(B2K_ERR_INVALID, "b2k_logreg_minimize: NULL objective / x or n < 1");
  if (max_iter < 0) return fail(B2K_ERR_INVALID, "maxIter given invalid value " + std::to_string(max_iter));
  if (!(tol >= 0.0)) return fail(B2K_ERR_INVALID, "tol given invalid value " + num(tol));
  bool owl = false;
  if (l1)
    for (int i = 0; i < n; ++i) {
      if (!(l1[i] >= 0.0) || !std::isfinite(l1[i])) return fail(B2K_ERR_INVALID, "b2k_logreg_minimize: L1 weights must be finite and >= 0");
      owl = owl || l1[i] > 0.0;
    }
  Objective obj{fn, user, owl ? l1 : nullptr, n};
  std::vector<double> x(x_io, x_io + n), g(n), pg(n), dir(n), xn(n), gn(n), pgn(n);
  double f = 0.0;
  if (!obj.eval(x, &f, &g)) return obj.status;
  double F = f + obj.l1_term(x);   // Breeze's adjusted value
  obj.pseudo_grad(x, g, &pg);
  const double F0 = F;
  if (f_hist) f_hist->assign(1, F);
  std::vector<std::vector<double>> S, Y;   // curvature pairs, oldest first
  std::vector<double> fhist{INFINITY};
  int iter = 0;
  auto converged = [&]() {
    if (iter >= max_iter) return true;
    if ((int)fhist.size() >= FVAL_MEMORY &&
        std::fabs(F - *std::max_element(fhist.begin(), fhist.end())) <= tol * std::fabs(F0))
      return true;
    return norm2(pg) <= std::max(tol * std::fabs(F), 1e-8);
  };
  if (!std::isfinite(F)) return fail(B2K_ERR_INVALID, "logistic regression: the objective is not finite at the start");
  while (!converged()) {
    // two-loop recursion on the (pseudo-)gradient
    std::vector<double> q(pg);
    const int m = (int)S.size();
    std::vector<double> alpha(m), rho(m);
    for (int i = m - 1; i >= 0; --i) {
      rho[i] = 1.0 / dot(Y[i], S[i]);
      alpha[i] = rho[i] * dot(S[i], q);
      for (int j = 0; j < n; ++j) q[j] -= alpha[i] * Y[i][j];
    }
    const double gamma = m > 0 ? dot(S[m - 1], Y[m - 1]) / dot(Y[m - 1], Y[m - 1]) : 1.0;
    for (int j = 0; j < n; ++j) q[j] *= gamma;
    for (int i = 0; i < m; ++i) {
      const double beta = rho[i] * dot(Y[i], q);
      for (int j = 0; j < n; ++j) q[j] += S[i][j] * (alpha[i] - beta);
    }
    for (int j = 0; j < n; ++j) dir[j] = -q[j];
    if (owl)   // keep the direction in the orthant the pseudo-gradient descends into
      for (int j = 0; j < n; ++j)
        if (dir[j] * pg[j] >= 0.0) dir[j] = 0.0;
    double dphi0 = dot(dir, pg);
    if (!(dphi0 < 0.0)) {   // not a descent direction: restart from the steepest descent once
      S.clear();
      Y.clear();
      for (int j = 0; j < n; ++j) dir[j] = -pg[j];
      dphi0 = dot(dir, pg);
      if (!(dphi0 < 0.0)) break;
    }
    const double dnorm = norm2(dir);
    bool ok = false;
    double fn_ = 0.0, Fn = 0.0;
    const double c1 = 1e-4, c2 = 0.9;
    const double slack = 4.0 * std::ldexp(1.0, -52) * std::fabs(F);   // rounding of F itself
    if (!owl) {
      // strong-Wolfe line search on phi(a) = f(x + a dir)
      auto at = [&](double a, double* fa, double* da) {
        for (int j = 0; j < n; ++j) xn[j] = x[j] + a * dir[j];
        if (!obj.eval(xn, fa, &gn)) return false;
        *da = dot(gn, dir);
        return true;
      };
      double a = iter == 0 ? 1.0 / dnorm : 1.0;
      double a_prev = 0.0, f_prev = F, d_prev = dphi0;
      int evals = 0;
      double lo = 0, flo = 0, dlo = 0, hi = 0, fhi = 0, dhi = 0;
      bool zoom = false;
      while (evals < LS_MAX_EVALS) {
        double fa, da;
        if (!at(a, &fa, &da)) return obj.status;
        ++evals;
        if (!std::isfinite(fa) || fa > F + c1 * a * dphi0 + slack || (evals > 1 && fa >= f_prev)) {
          lo = a_prev; flo = f_prev; dlo = d_prev; hi = a; fhi = fa; dhi = da;
          zoom = true;
          break;
        }
        if (std::fabs(da) <= -c2 * dphi0) {
          ok = true;
          fn_ = fa;
          break;
        }
        if (da >= 0.0) {
          lo = a; flo = fa; dlo = da; hi = a_prev; fhi = f_prev; dhi = d_prev;
          zoom = true;
          break;
        }
        a_prev = a; f_prev = fa; d_prev = da;
        a *= 2.0;
      }
      while (zoom && !ok && evals < LS_MAX_EVALS) {
        const double aj = std::isfinite(fhi) ? interpolate(lo, flo, dlo, hi, fhi, dhi) : 0.5 * (lo + hi);
        double fa, da;
        if (!at(aj, &fa, &da)) return obj.status;
        ++evals;
        if (!std::isfinite(fa) || fa > F + c1 * aj * dphi0 + slack || fa >= flo) {
          hi = aj; fhi = fa; dhi = da;
        } else {
          if (std::fabs(da) <= -c2 * dphi0) {
            ok = true;
            fn_ = fa;
            break;
          }
          if (da * (hi - lo) >= 0.0) {
            hi = lo; fhi = flo; dhi = dlo;
          }
          lo = aj; flo = fa; dlo = da;
        }
      }
      Fn = fn_;
    } else {
      // OWL-QN: backtracking on the projected step, Armijo on the adjusted value
      double a = iter == 0 ? 0.5 / norm2(pg) : 1.0;
      const double shrink = iter == 0 ? 0.1 : 0.5;
      for (int evals = 0; evals < LS_MAX_EVALS; ++evals) {
        for (int j = 0; j < n; ++j) {
          const double orth = x[j] != 0.0 ? (x[j] > 0.0 ? 1.0 : -1.0) : (pg[j] < 0.0 ? 1.0 : -1.0);
          const double v = x[j] + a * dir[j];
          xn[j] = v * orth > 0.0 ? v : 0.0;
        }
        if (!obj.eval(xn, &fn_, &gn)) return obj.status;
        Fn = fn_ + obj.l1_term(xn);
        double dec = 0.0;
        for (int j = 0; j < n; ++j) dec += pg[j] * (xn[j] - x[j]);
        if (std::isfinite(Fn) && Fn <= F + c1 * dec + slack) {
          ok = true;
          break;
        }
        a *= shrink;
      }
    }
    if (!ok) break;   // Breeze stops on a failed line search; x keeps the last accepted iterate
    std::vector<double> s(n), yv(n);
    for (int j = 0; j < n; ++j) {
      s[j] = xn[j] - x[j];
      yv[j] = gn[j] - g[j];
    }
    if (dot(s, yv) > 0.0) {
      S.push_back(s);
      Y.push_back(yv);
      if ((int)S.size() > LBFGS_M) {
        S.erase(S.begin());
        Y.erase(Y.begin());
      }
    }
    x.swap(xn);
    g.swap(gn);
    f = fn_;
    F = owl ? Fn : f;
    obj.pseudo_grad(x, g, &pg);
    ++iter;
    if (f_hist) f_hist->push_back(F);
    fhist.push_back(F);
    if ((int)fhist.size() > FVAL_MEMORY) fhist.erase(fhist.begin());
  }
  std::copy(x.begin(), x.end(), x_io);
  if (n_iter_out) *n_iter_out = iter;
  if (n_eval_out) *n_eval_out = obj.evals;
  if (f_out) *f_out = F;
  return B2K_OK;
}

// ------------------------------------------------------------------------------------------------
// device drivers
// ------------------------------------------------------------------------------------------------
int b2k_logreg_labels_impl(b2k_ctx* ctx, const float* y, int64_t n, double* classes_out, int64_t* counts_out,
                           int* n_classes_out, int64_t* n_total_out, cudaStream_t s) {
  const int spans = (int)std::max<int64_t>(1, std::min<int64_t>(4 * ctx->sm_count, (n + 1023) / 1024));
  const int64_t span_rows = std::max<int64_t>(1, (n + spans - 1) / spans);
  const size_t W1 = LB_W + 1;
  double *part, *mine, *all;
  B2K_TRY(b2k_scratch_layout(ctx, "logistic regression labels", [&](B2kLayout& L) -> int {
    part = L.take<double>((size_t)spans * LB_W);
    mine = L.take<double>(W1);
    all = L.take<double>(W1 * ctx->nranks);
    return B2K_OK;
  }));
  if (n > 0) {
    k_logreg_labels<<<spans, LR_THREADS, 0, s>>>(y, n, span_rows, part);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
  }
  k_logreg_labels_fold<<<(int)((W1 + 255) / 256), 256, 0, s>>>(part, n > 0 ? spans : 0, n, mine);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  B2K_TRY(b2k_comm_allgather_bytes(ctx, mine, all, W1 * 8, s));
  std::vector<double> h(W1 * ctx->nranks);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(h.data(), all, h.size() * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  // reduce in rank order: identical on every rank
  std::vector<double> cnt(MAXC, 0.0);
  double mn = INFINITY, mx = -INFINITY, ni = INFINITY, sum = 0.0, nt = 0.0;
  for (int r = 0; r < ctx->nranks; ++r) {
    const double* p = &h[(size_t)r * W1];
    if (p[LB_W] == 0.0) continue;
    for (int c = 0; c < MAXC; ++c) cnt[c] += p[c];
    mn = std::min(mn, p[MAXC]);
    mx = std::max(mx, p[MAXC + 1]);
    ni = std::min(ni, p[MAXC + 2]);
    sum += p[MAXC + 3];
    nt += p[LB_W];
  }
  if (nt < 1.0) return b2k_fail(ctx, B2K_ERR_INVALID, "logistic regression needs at least 1 row, got 0");
  if (!std::isfinite(sum)) return b2k_fail(ctx, B2K_ERR_INVALID, "logistic regression: the label holds a NaN or an infinity");
  // the reference checks the sorted classes in order: a negative one first, then a non-integer one
  if (mn < 0.0) return b2k_fail(ctx, B2K_ERR_INVALID, "Labels MUST be in [0, 2147483647), but got " + num(mn));
  if (std::isfinite(ni)) return b2k_fail(ctx, B2K_ERR_INVALID, "Labels MUST be Integers, but got " + num(ni));
  if (mx >= 2147483647.0) return b2k_fail(ctx, B2K_ERR_INVALID, "Labels MUST be in [0, 2147483647), but got " + num(mx));
  if (mx >= (double)MAXC)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "logistic regression supports label values below " + std::to_string(MAXC) +
                                                  " (at most " + std::to_string(MAXC) + " classes), got " + num(mx));
  int k = 0;
  for (int c = 0; c < MAXC; ++c)
    if (cnt[c] > 0.0) {
      if (classes_out) classes_out[k] = (double)c;
      if (counts_out) counts_out[k] = (int64_t)cnt[c];
      ++k;
    }
  *n_classes_out = k;
  if (n_total_out) *n_total_out = (int64_t)nt;
  return B2K_OK;
}

namespace {

// One evaluation: out [kp (d + 1) + 2] = allreduced [sum r x | sum r per class (at k (d + 1) + d) | sum loss | n].
struct EvalCall {
  const float* X;
  const float* y;
  int64_t n;
  int d, kp;
  const std::vector<int>* cmap;
};

int eval_device(b2k_ctx* ctx, const EvalCall& e, const double* W, const double* b, double* out_host, cudaStream_t s) {
  const int d = e.d, kp = e.kp, M = kp * (d + 1) + 1;
  const bool can_fuse = fused_fits(ctx, d, kp);
  if (ctx->kernel_path == B2K_PATH_FUSED && !can_fuse)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "kernel_path=2 requested but the fused logistic pass does not cover d = " +
                                                  std::to_string(d) + " with " + std::to_string(kp) + " margins per row");
  const bool fused = can_fuse && ctx->kernel_path != B2K_PATH_GENERIC;
  const bool vec = d % 4 == 0 && (reinterpret_cast<uintptr_t>(e.X) & 15u) == 0;
  const int64_t n = e.n;
  // plan
  FusedPick fp;
  int grid = 1, P = 1, tr = tile_rows(d);
  int64_t span_rows = tr;
  size_t smem = 0;
  int64_t chunk = 0, nchunk = 0;
  int spans = 1, ncb = 1;
  if (fused) {
    fp = fused_pick(d, kp);
    smem = fused_smem(d, kp, fp.KB);
    B2K_CUDA_OK(ctx, cudaFuncSetAttribute(fp.kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    B2K_CUDA_OK(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fp.kern, LR_THREADS, smem));
    const int64_t tiles = std::max<int64_t>(1, (n + tr - 1) / tr);
    int64_t cap = (int64_t)std::max(1, per_sm) * ctx->sm_count;
    if (ctx->grid_limit > 0 && ctx->grid_limit < cap) cap = ctx->grid_limit;
    const int64_t g0 = std::min<int64_t>(tiles, cap);
    span_rows = (tiles + g0 - 1) / g0 * tr;
    grid = (int)std::max<int64_t>(1, (n + span_rows - 1) / span_rows);
    P = grid * fused_shape(d, kp, fp.KB, tr).rg;
  } else {
    chunk = std::max<int64_t>(1, std::min<int64_t>(std::max<int64_t>(n, 1), (int64_t)(64u << 20) / (8 * (kp + 1))));
    nchunk = std::max<int64_t>(1, (n + chunk - 1) / chunk);
    ncb = (d + 2 + XR_TX - 1) / XR_TX;
    spans = (int)std::max<int64_t>(1, std::min<int64_t>((chunk + 63) / 64, std::max(1, 8 * ctx->sm_count / (ncb * kp))));
    P = (int)(nchunk * spans);
  }
  double *Wd, *bd, *part, *out, *R = nullptr, *loss = nullptr;
  int* cmap;
  B2K_TRY(b2k_scratch_layout(ctx, "logistic regression evaluation", [&](B2kLayout& L) -> int {
    Wd = L.take<double>((size_t)kp * d);
    bd = L.take<double>(kp);
    cmap = L.take<int>(MAXC);
    out = L.take<double>((size_t)M + 1);
    part = L.take<double>((size_t)P * M);
    if (!fused) {
      R = L.take<double>((size_t)chunk * kp);
      loss = L.take<double>((size_t)chunk);
    }
    return B2K_OK;
  }));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(Wd, W, (size_t)kp * d * 8, cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(bd, b, (size_t)kp * 8, cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(cmap, e.cmap->data(), MAXC * 4, cudaMemcpyHostToDevice, s));
  B2kTimer tm(ctx->time_kernels != 0);
  tm.mark(0, s);
  if (n == 0) {
    B2K_CUDA_OK(ctx, cudaMemsetAsync(part, 0, (size_t)P * M * 8, s));
  } else if (fused) {
    EvalArgs a{e.X, e.y, cmap, Wd, bd, n, d, kp, tr, span_rows, part};
    fp.kern<<<grid, LR_THREADS, smem, s>>>(a);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
    ctx->stats.fused_tc_launches++;
  } else {
    const int L = row_lanes(d);
    auto rk = vec ? k_logreg_rows<true, true> : k_logreg_rows<false, true>;
    for (int64_t c = 0; c < nchunk; ++c) {
      const int64_t c0 = c * chunk, rows = std::min<int64_t>(chunk, n - c0);
      const int64_t rpc = (int64_t)(LR_THREADS / 32) * (32 / L);
      const int g = (int)std::max<int64_t>(1, std::min<int64_t>((rows + rpc - 1) / rpc, 8 * ctx->sm_count));
      rk<<<g, LR_THREADS, 0, s>>>(e.X + c0 * d, rows, d, kp, Wd, bd, L, e.y + c0, cmap, R, loss, nullptr, nullptr,
                                  nullptr, nullptr);
      B2K_CUDA_OK(ctx, cudaGetLastError());
      const int64_t sr = std::max<int64_t>(1, (rows + spans - 1) / spans);
      k_logreg_xtr<<<dim3(spans, ncb, kp), dim3(XR_TX, XR_TY), 0, s>>>(e.X + c0 * d, rows, d, kp, R, loss, sr,
                                                                        part + (size_t)c * spans * M);
      B2K_CUDA_OK(ctx, cudaGetLastError());
      ctx->stats.kernel_launches += 2;
      ctx->stats.generic_launches += 2;
    }
  }
  tm.mark(1, s);
  B2K_TRY(b2k_launch_fold_spans(ctx, part, P, M, out, s, n));   // out [M + 1]: the partials in order, then n
  B2K_TRY(b2k_comm_allreduce_f64(ctx, out, (size_t)M + 1, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(out_host, out, ((size_t)M + 1) * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  ctx->stats.last_path = fused ? B2K_PATH_FUSED : B2K_PATH_GENERIC;
  if (tm.on) ctx->stats.last_fused_ms = tm.ms(0, 1);
  return B2K_OK;
}

}  // namespace

std::vector<int> b2k_logreg_class_map(const double* classes, int n_classes) {
  std::vector<int> m(MAXC, -1);
  for (int i = 0; i < n_classes; ++i) {
    const double c = classes[i];
    if (c >= 0.0 && c < MAXC && c == std::floor(c)) m[(int)c] = i;
  }
  return m;
}

int b2k_logreg_eval_impl(b2k_ctx* ctx, const float* X, const float* y, int64_t n, int d, const double* classes,
                         int n_classes, int kp, const double* W, const double* b, double* loss_out, double* grad_out,
                         int64_t* n_total_out, cudaStream_t s) {
  if (d > B2K_LOGREG_MAX_D)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "logistic regression supports d <= " + std::to_string(B2K_LOGREG_MAX_D) +
                                                  ", got d = " + std::to_string(d));
  if (n_classes < 1 || n_classes > MAXC) return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_logreg_eval: bad class count");
  // a row's residuals are indexed by its class: kp must be 1 (binomial) or cover every class (multinomial)
  if (kp != 1 && kp != n_classes)
    return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_logreg_eval: margins per row must be 1 or the class count " +
                                              std::to_string(n_classes) + ", got " + std::to_string(kp));
  const std::vector<int> cm = b2k_logreg_class_map(classes, n_classes);
  EvalCall e{X, y, n, d, kp, &cm};
  const int M = kp * (d + 1) + 1;
  std::vector<double> out((size_t)M + 1);
  B2K_TRY(eval_device(ctx, e, W, b, out.data(), s));
  const double nt = out[M];
  if (nt < 1.0) return b2k_fail(ctx, B2K_ERR_INVALID, "logistic regression needs at least 1 row, got 0");
  *loss_out = out[M - 1] / nt;
  for (int i = 0; i < M - 1; ++i) grad_out[i] = out[i] / nt;
  if (n_total_out) *n_total_out = (int64_t)nt;
  return B2K_OK;
}

int b2k_logreg_check_params(b2k_ctx* ctx, int K, int n_fits, const b2k_logreg_params* prm) {
  if (K < 1 || K > MAXC) return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_logreg_fit: bad class count");
  for (int f = 0; f < n_fits; ++f) {   // the driver-side checks, repeated so a direct caller gets them too
    const b2k_logreg_params& p = prm[f];
    if (p.max_iter < 0) return b2k_fail(ctx, B2K_ERR_INVALID, "maxIter given invalid value " + std::to_string(p.max_iter));
    if (!(p.reg >= 0.0)) return b2k_fail(ctx, B2K_ERR_INVALID, "C or regParam given an invalid or unsupported value " + num(p.reg));
    if (!(p.l1_ratio >= 0.0 && p.l1_ratio <= 1.0))
      return b2k_fail(ctx, B2K_ERR_INVALID, "elasticNetParam given invalid value " + num(p.l1_ratio));
    if (!(p.tol >= 0.0)) return b2k_fail(ctx, B2K_ERR_INVALID, "tol given invalid value " + num(p.tol));
    if (p.family < 0 || p.family > 2) return b2k_fail(ctx, B2K_ERR_INVALID, "family must be auto, binomial or multinomial");
    if (p.family == 1 && K > 2)
      return b2k_fail(ctx, B2K_ERR_INVALID, "Binomial family only supports 1 or 2 outcome classes but found " +
                                                std::to_string(K) + ".");
  }
  return B2K_OK;
}

int b2k_logreg_fit_settings(b2k_ctx* ctx, int d, int64_t n_total, const std::vector<double>& ssq, const double* classes,
                            const int64_t* counts, int n_classes, int n_fits, const b2k_logreg_params* prm,
                            const B2kLogregEval& eval, double* coef_out, double* intercept_out, int* kp_out,
                            int* n_iter_out) {
  const int K = n_classes;
  if (K == 1) {   // one label value: as the reference, no optimisation (after the moments pass, so that bad
                  // features are still reported)
    if (classes[0] != 0.0 && classes[0] != 1.0)
      return b2k_fail(ctx, B2K_ERR_INVALID, "class value must be either 1. or 0. when dataset has one label");
    for (int f = 0; f < n_fits; ++f) {
      std::fill(coef_out + (size_t)f * K * d, coef_out + (size_t)(f + 1) * K * d, 0.0);
      intercept_out[(size_t)f * K] = classes[0] == 1.0 ? INFINITY : -INFINITY;
      kp_out[f] = 1;
      n_iter_out[f] = 0;
    }
    return B2K_OK;
  }
  // sample standard deviations, as MLlib's summarizer (n - 1; 0 for a single row)
  std::vector<double> sigma(d);
  for (int j = 0; j < d; ++j) sigma[j] = n_total > 1 ? std::sqrt(std::max(ssq[j], 0.0) / (double)(n_total - 1)) : 0.0;
  for (int f = 0; f < n_fits; ++f) {
    const b2k_logreg_params& p = prm[f];
    const bool multi = p.family == 2 || (p.family == 0 && K > 2);
    const int kp = multi ? K : 1;
    const bool fi = p.fit_intercept != 0;
    const int nv = kp * d, nth = nv + (fi ? kp : 0);
    const double l2 = p.reg * (1.0 - p.l1_ratio), l1w = p.reg * p.l1_ratio;
    // solver frame: theta = [V (kp x d) | b], W = V / sigma (0 where sigma = 0); the penalty is on V (standardization)
    // or on W
    std::vector<double> inv(d), pen(d);
    for (int j = 0; j < d; ++j) {
      inv[j] = sigma[j] > 0.0 ? 1.0 / sigma[j] : 0.0;
      pen[j] = p.standardization ? (sigma[j] > 0.0 ? 1.0 : 0.0) : inv[j] * inv[j];
    }
    std::vector<double> l1v(nth, 0.0);
    for (int k = 0; k < kp; ++k)
      for (int j = 0; j < d; ++j) l1v[(size_t)k * d + j] = l1w * (p.standardization ? (sigma[j] > 0.0 ? 1.0 : 0.0) : inv[j]);
    std::vector<double> theta(nth, 0.0);
    if (fi) {   // MLlib's start: the log-odds of the class priors
      if (multi) {
        double mean = 0.0;
        for (int k = 0; k < kp; ++k) mean += std::log1p((double)counts[k]);
        mean /= kp;
        for (int k = 0; k < kp; ++k) theta[nv + k] = std::log1p((double)counts[k]) - mean;
      } else {
        theta[nv] = std::log((double)counts[1] / (double)counts[0]);
      }
    }
    struct Fn {
      const B2kLogregEval* eval;
      int d, kp;
      bool fi;
      double l2;
      const std::vector<double>* inv;
      const std::vector<double>* pen;
      std::vector<double> W, b, out;
      int rc;
    } F{&eval, d, kp, fi, l2, &inv, &pen,
        std::vector<double>(nv), std::vector<double>(kp, 0.0), std::vector<double>((size_t)kp * (d + 1) + 2), B2K_OK};
    auto cb = [](void* user, int, const double* th, double* fval, double* grad) -> int {
      Fn& q = *static_cast<Fn*>(user);
      const int d = q.d, kp = q.kp, nv = kp * d;
      for (int k = 0; k < kp; ++k)
        for (int j = 0; j < d; ++j) q.W[(size_t)k * d + j] = th[(size_t)k * d + j] * (*q.inv)[j];
      for (int k = 0; k < kp; ++k) q.b[k] = q.fi ? th[nv + k] : 0.0;
      q.rc = (*q.eval)(kp, q.W.data(), q.b.data(), q.out.data());
      if (q.rc != B2K_OK) return q.rc;
      const int M = kp * (d + 1) + 1;
      const double nt = q.out[M];
      double fv = q.out[M - 1] / nt, reg = 0.0;
      for (int k = 0; k < kp; ++k) {
        for (int j = 0; j < d; ++j) {
          const double v = th[(size_t)k * d + j];
          reg += (*q.pen)[j] * v * v;
          grad[(size_t)k * d + j] = q.out[(size_t)k * (d + 1) + j] / nt * (*q.inv)[j] + q.l2 * (*q.pen)[j] * v;
        }
        if (q.fi) grad[nv + k] = q.out[(size_t)k * (d + 1) + d] / nt;
      }
      *fval = fv + 0.5 * q.l2 * reg;
      return B2K_OK;
    };
    int iters = 0, evals = 0;
    double fend = 0.0;
    const int rc = b2k_logreg_minimize_impl(cb, &F, nth, theta.data(), l1w > 0.0 ? l1v.data() : nullptr, p.max_iter,
                                            p.tol, &iters, &evals, &fend);
    if (rc != B2K_OK) {
      if (F.rc == B2K_OK) ctx->err = b2k_last_error(nullptr);   // the optimizer's own error, not the device's
      return rc;
    }
    double* cf = coef_out + (size_t)f * K * d;
    double* ic = intercept_out + (size_t)f * K;
    std::fill(cf, cf + (size_t)K * d, 0.0);
    std::fill(ic, ic + K, 0.0);
    for (int k = 0; k < kp; ++k) {
      for (int j = 0; j < d; ++j) cf[(size_t)k * d + j] = theta[(size_t)k * d + j] * inv[j];
      ic[k] = fi ? theta[nv + k] : 0.0;
    }
    if (multi) {   // MLlib's centring: intercepts with an intercept, coefficients per feature without a penalty
      if (fi) {
        double m = 0.0;
        for (int k = 0; k < kp; ++k) m += ic[k];
        m /= kp;
        for (int k = 0; k < kp; ++k) ic[k] -= m;
      }
      if (p.reg == 0.0)
        for (int j = 0; j < d; ++j) {
          double m = 0.0;
          for (int k = 0; k < kp; ++k) m += cf[(size_t)k * d + j];
          m /= kp;
          for (int k = 0; k < kp; ++k) cf[(size_t)k * d + j] = sigma[j] > 0.0 ? cf[(size_t)k * d + j] - m : 0.0;
        }
    }
    kp_out[f] = kp;
    n_iter_out[f] = iters;
    ctx->stats.last_n_iter = iters;
  }
  return B2K_OK;
}

int b2k_logreg_fit_impl(b2k_ctx* ctx, const float* X, const float* y, int64_t n, int d, const double* classes,
                        const int64_t* counts, int n_classes, int n_fits, const b2k_logreg_params* prm,
                        double* coef_out, double* intercept_out, int* kp_out, int* n_iter_out, cudaStream_t s) {
  using clk = std::chrono::steady_clock;
  const auto t_begin = clk::now();
  if (d > B2K_LOGREG_MAX_D)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "logistic regression supports d <= " + std::to_string(B2K_LOGREG_MAX_D) +
                                                  ", got d = " + std::to_string(d));
  B2K_TRY(b2k_logreg_check_params(ctx, n_classes, n_fits, prm));
  int64_t n_total = 0;
  std::vector<double> mu, ssq;
  B2K_TRY(b2k_colstats_impl(ctx, "logistic regression", X, n, d, &n_total, &mu, &ssq, s));
  if (!finite_all(mu.data(), d) || !finite_all(ssq.data(), d))
    return b2k_fail(ctx, B2K_ERR_INVALID, "logistic regression: the features hold a NaN or an infinity");
  const std::vector<int> cm = b2k_logreg_class_map(classes, n_classes);
  const B2kLogregEval eval = [&](int kp, const double* W, const double* b, double* out) {
    return eval_device(ctx, EvalCall{X, y, n, d, kp, &cm}, W, b, out, s);
  };
  B2K_TRY(b2k_logreg_fit_settings(ctx, d, n_total, ssq, classes, counts, n_classes, n_fits, prm, eval, coef_out,
                                  intercept_out, kp_out, n_iter_out));
  if (ctx->time_kernels)
    ctx->stats.last_loop_ms = std::chrono::duration<double, std::milli>(clk::now() - t_begin).count();
  return B2K_OK;
}

int b2k_logreg_predict_impl(b2k_ctx* ctx, const float* X, int64_t n, int d, int kp, const double* W, const double* b,
                            const double* class_values, double* raw_out, double* prob_out, double* pred_out,
                            cudaStream_t s) {
  if (d > B2K_LOGREG_MAX_D)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "logistic regression predicts d <= " + std::to_string(B2K_LOGREG_MAX_D));
  if (n == 0) return B2K_OK;
  const int L = row_lanes(d);
  const bool vec = d % 4 == 0 && (reinterpret_cast<uintptr_t>(X) & 15u) == 0;
  auto kern = vec ? k_logreg_rows<true, false> : k_logreg_rows<false, false>;
  const int64_t rpc = (int64_t)(LR_THREADS / 32) * (32 / L);
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((n + rpc - 1) / rpc, 8 * ctx->sm_count));
  kern<<<grid, LR_THREADS, 0, s>>>(X, n, d, kp, W, b, L, nullptr, nullptr, nullptr, nullptr, class_values, raw_out,
                                   prob_out, pred_out);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  return B2K_OK;
}
