// PCA (sm_90a): the covariance passes, the projection kernel of transform and the host eigen step.
//
//   pass 1  k_colsum: fp64 column sums, per-CTA partials over fixed row spans, folded in span order (k_colsum_fold) into
//           [d sums | n]; one f64 allreduce of d + 1 values; the host forms mu = sum / n_total in fp64.
//   pass 2  the Gram matrix G = sum (x - mu32)(x - mu32)^T of the data centred on mu32 = fl32(mu):
//             wgmma path (b2k_gram_wg.cuh, 3xTF32): d % 4 == 0, d <= B2K_PCA_MAX_D, X 16-byte aligned;
//             generic path (k_gram_generic, SIMT, products and sums in fp64): every d <= B2K_PCA_MAX_D;
//           per-CTA fp64 partials folded in a fixed order and mirrored (upper triangle -> both), one f64 allreduce of
//           d * d values.  The host then removes the offset of mu32 from mu exactly:
//           cov = (G - n (mu - mu32)(mu - mu32)^T) / (n - 1).
//   eigen   b2k_pca_finalize_impl (host, fp64): Householder tridiagonalisation + implicit-shift QL, descending order,
//           sign convention, ratios, singular values.
//   transform  k_project: Y = X C^T, fp32 (SIMT; the components stay in shared memory).
// Every sum is formed in an order fixed by (n, d, grid): no atomics, two fits of the same input are bitwise equal.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <numeric>
#include <vector>

#include "b2k_internal.cuh"

namespace {
#include "b2k_ptx.cuh"
#include "b2k_gram_wg.cuh"

constexpr int CS_TX = 32, CS_TY = 8;   // column-sum CTA: 32 columns x 8 row lanes

__global__ void __launch_bounds__(CS_TX * CS_TY)
k_colsum(const float* __restrict__ X, int64_t n, int d, int64_t span_rows, double* __restrict__ part) {
  __shared__ double red[CS_TY][CS_TX];
  const int c = blockIdx.y * CS_TX + threadIdx.x;
  const int64_t r0 = (int64_t)blockIdx.x * span_rows;
  const int64_t r1 = min(n, r0 + span_rows);
  double s = 0.0;
  if (c < d) {
#pragma unroll 4
    for (int64_t r = r0 + threadIdx.y; r < r1; r += CS_TY) s += (double)X[r * d + c];
  }
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && c < d) {
    double t = 0.0;
    for (int y = 0; y < CS_TY; ++y) t += red[y][threadIdx.x];
    part[(size_t)blockIdx.x * d + c] = t;
  }
}

// sums[c] = sum over spans in order; sums[d] = n (the allreduce turns it into n_total)
__global__ void k_colsum_fold(const double* __restrict__ part, int nspan, int d, int64_t n, double* __restrict__ sums) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < d) {
    double t = 0.0;
    for (int s = 0; s < nspan; ++s) t += part[(size_t)s * d + c];
    sums[c] = t;
  } else if (c == d) {
    sums[d] = (double)n;
  }
}

// wgmma path: G[i][j] = G[j][i] = sum over the P CTAs of tile (i / 128, j / 128), in CTA order, for i <= j
__global__ void k_gram_fold_wg(const double* __restrict__ part, int P, int ntile, int nblk, int d, double* __restrict__ G) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)d * d) return;
  const int gi = (int)(idx / d), gj = (int)(idx % d);
  if (gi > gj) return;
  const int I = gi / GW_BLK, J = gj / GW_BLK;
  const int t = I * nblk - I * (I - 1) / 2 + (J - I);
  const size_t e = (size_t)(gi % GW_BLK) * GW_BLK + (gj % GW_BLK);
  double s = 0.0;
  for (int p = 0; p < P; ++p) s += part[((size_t)p * ntile + t) * GW_BLK * GW_BLK + e];
  G[(size_t)gi * d + gj] = s;
  G[(size_t)gj * d + gi] = s;
}

// generic path: 32 x 32 tiles of the upper block triangle (blockIdx.x) over row span blockIdx.y; thread (tx, ty) forms
// entries (ty + 16 a, tx + 16 b) of the tile in fp64 from the fp32 centred values
constexpr int GG_T = 32;
__global__ void __launch_bounds__(256)
k_gram_generic(const float* __restrict__ X, int64_t n, int d, const float* __restrict__ mu, int64_t span_rows,
               double* __restrict__ part) {
  __shared__ float xi[GG_T][GG_T + 1], xj[GG_T][GG_T + 1];
  const int nb = (d + GG_T - 1) / GG_T;
  int t = blockIdx.x, I = 0;
  while (t >= nb - I) {
    t -= nb - I;
    ++I;
  }
  const int J = I + t;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int64_t r0 = (int64_t)blockIdx.y * span_rows;
  const int64_t r1 = min(n, r0 + span_rows);
  double acc[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
  for (int64_t rb = r0; rb < r1; rb += GG_T) {
    for (int e = threadIdx.x; e < GG_T * GG_T; e += 256) {
      const int rr = e / GG_T, cc = e % GG_T;
      const int64_t row = rb + rr;
      const int ci = I * GG_T + cc, cj = J * GG_T + cc;
      xi[rr][cc] = (row < r1 && ci < d) ? X[row * d + ci] - mu[ci] : 0.f;
      xj[rr][cc] = (row < r1 && cj < d) ? X[row * d + cj] - mu[cj] : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int rr = 0; rr < GG_T; ++rr) {
      const double a0 = xi[rr][ty], a1 = xi[rr][ty + 16];
      const double b0 = xj[rr][tx], b1 = xj[rr][tx + 16];
      acc[0][0] = fma(a0, b0, acc[0][0]);
      acc[0][1] = fma(a0, b1, acc[0][1]);
      acc[1][0] = fma(a1, b0, acc[1][0]);
      acc[1][1] = fma(a1, b1, acc[1][1]);
    }
    __syncthreads();
  }
  double* o = part + (size_t)blockIdx.y * d * d;
  for (int a = 0; a < 2; ++a)
    for (int b = 0; b < 2; ++b) {
      const int gi = I * GG_T + ty + 16 * a, gj = J * GG_T + tx + 16 * b;
      if (gi < d && gj < d) o[(size_t)gi * d + gj] = acc[a][b];
    }
}

__global__ void k_gram_fold_generic(const double* __restrict__ part, int S, int d, double* __restrict__ G) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)d * d) return;
  const int gi = (int)(idx / d), gj = (int)(idx % d);
  if (gi > gj) return;
  double s = 0.0;
  for (int sp = 0; sp < S; ++sp) s += part[(size_t)sp * d * d + idx];
  G[(size_t)gi * d + gj] = s;
  G[(size_t)gj * d + gi] = s;
}

// Y[n][k] = X[n][d] . C[k][d]^T.  CTA: PJ_ROWS rows (one per thread) x PJ_KT components (blockIdx.y); the CTA's
// components stay in shared memory transposed, CT[c][j], for its whole run over row tiles; X is staged 32 features at a
// time, transposed, so that each thread reads its own row without bank conflicts.  fp32 FMA in feature order.
constexpr int PJ_ROWS = 256, PJ_KT = 32, PJ_DC = 32;
__global__ void __launch_bounds__(PJ_ROWS)
k_project(const float* __restrict__ X, int64_t n, int d, const float* __restrict__ C, int k, float* __restrict__ Y) {
  extern __shared__ float pj_smem[];
  const int dpad = (d + PJ_DC - 1) / PJ_DC * PJ_DC;
  float* ct = pj_smem;                      // [dpad][PJ_KT]
  float* xs = pj_smem + dpad * PJ_KT;       // [PJ_DC][PJ_ROWS + 1]
  const int j0 = blockIdx.y * PJ_KT;
  for (int e = threadIdx.x; e < dpad * PJ_KT; e += PJ_ROWS) {
    const int c = e / PJ_KT, j = e % PJ_KT;
    ct[e] = (c < d && j0 + j < k) ? C[(size_t)(j0 + j) * d + c] : 0.f;
  }
  const int64_t ntiles = (n + PJ_ROWS - 1) / PJ_ROWS;
  const int kt = min(PJ_KT, k - j0);
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t row0 = tile * PJ_ROWS;
    float acc[PJ_KT];
#pragma unroll
    for (int j = 0; j < PJ_KT; ++j) acc[j] = 0.f;
    for (int c0 = 0; c0 < dpad; c0 += PJ_DC) {
      __syncthreads();   // previous chunk consumed (and, the first time, ct written)
#pragma unroll 8
      for (int i = 0; i < PJ_DC; ++i) {   // a warp reads 32 consecutive features of one row
        const int e = i * PJ_ROWS + threadIdx.x;
        const int rr = e / PJ_DC, cc = e % PJ_DC;
        const int64_t row = row0 + rr;
        xs[cc * (PJ_ROWS + 1) + rr] = (row < n && c0 + cc < d) ? X[row * d + c0 + cc] : 0.f;
      }
      __syncthreads();
#pragma unroll 4
      for (int cc = 0; cc < PJ_DC; ++cc) {
        const float x = xs[cc * (PJ_ROWS + 1) + threadIdx.x];
        const float4* w = reinterpret_cast<const float4*>(ct + (c0 + cc) * PJ_KT);
#pragma unroll
        for (int j4 = 0; j4 < PJ_KT / 4; ++j4) {
          const float4 v = w[j4];
          acc[4 * j4 + 0] = fmaf(x, v.x, acc[4 * j4 + 0]);
          acc[4 * j4 + 1] = fmaf(x, v.y, acc[4 * j4 + 1]);
          acc[4 * j4 + 2] = fmaf(x, v.z, acc[4 * j4 + 2]);
          acc[4 * j4 + 3] = fmaf(x, v.w, acc[4 * j4 + 3]);
        }
      }
    }
    const int64_t row = row0 + threadIdx.x;
    if (row < n) {
      float* y = Y + row * k + j0;
#pragma unroll
      for (int j = 0; j < PJ_KT; ++j)
        if (j < kt) y[j] = acc[j];
    }
  }
}

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

struct Timer {   // CUDA events around the device phases when option time_kernels is set
  cudaEvent_t ev[8] = {};
  bool on = false;
  explicit Timer(bool enable) : on(enable) {
    if (on)
      for (auto& e : ev) cudaEventCreate(&e);
  }
  ~Timer() {
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

// ---------------------------------------------------------------------------------------------------------------------
// host eigen step
// ---------------------------------------------------------------------------------------------------------------------
// A (n x n, row-major, symmetric) = Z^T diag(w) Z: rows of Z are the eigenvectors.  A is destroyed.
//  1. Householder: for k = 0 .. n - 3, H_k = I - 2 v v^T (v a unit vector over indices k + 1 ..) maps column k below the
//     sub-diagonal onto its first entry, and A <- H_k A H_k (the trailing block as A - v w^T - w v^T with
//     w = 2 (A v) - 2 (v^T A v) v).  Z accumulates H_{n-3} ... H_0, so A_in = Z^T T Z with T tridiagonal.
//  2. implicit QL with Wilkinson-type shifts on T; each plane rotation of rows (i, i + 1) of T is applied to rows i and
//     i + 1 of Z.
// Returns false if an eigenvalue needs more than 60 QL sweeps.
bool sym_eig(std::vector<double>& A, int n, std::vector<double>& w, std::vector<double>& Z) {
  Z.assign((size_t)n * n, 0.0);
  for (int i = 0; i < n; ++i) Z[(size_t)i * n + i] = 1.0;
  std::vector<double> v(n), p(n), zs(n);
  auto a = [&](int i, int j) -> double& { return A[(size_t)i * n + j]; };
  for (int k = 0; k + 2 < n; ++k) {
    const int m = n - k - 1, o = k + 1;
    double xn = 0.0;
    for (int i = 0; i < m; ++i) xn += a(o + i, k) * a(o + i, k);
    xn = std::sqrt(xn);
    if (xn == 0.0) continue;
    const double alpha = a(o, k) > 0.0 ? -xn : xn;
    double vn = 0.0;
    for (int i = 0; i < m; ++i) {
      v[i] = a(o + i, k) - (i == 0 ? alpha : 0.0);
      vn += v[i] * v[i];
    }
    vn = std::sqrt(vn);
    if (vn == 0.0) continue;
    for (int i = 0; i < m; ++i) v[i] /= vn;
    double K = 0.0;
    for (int i = 0; i < m; ++i) {
      const double* row = &a(o + i, o);
      double s = 0.0;
      for (int j = 0; j < m; ++j) s += row[j] * v[j];
      p[i] = s;
      K += v[i] * s;
    }
    for (int i = 0; i < m; ++i) p[i] = 2.0 * p[i] - 2.0 * K * v[i];   // w
    for (int i = 0; i < m; ++i) {
      double* row = &a(o + i, o);
      for (int j = 0; j < m; ++j) row[j] -= v[i] * p[j] + p[i] * v[j];
    }
    a(o, k) = a(k, o) = alpha;
    for (int i = 1; i < m; ++i) a(o + i, k) = a(k, o + i) = 0.0;
    // Z <- H_k Z: rows o .. n - 1
    std::fill(zs.begin(), zs.end(), 0.0);
    for (int i = 0; i < m; ++i) {
      const double* zr = &Z[(size_t)(o + i) * n];
      for (int c = 0; c < n; ++c) zs[c] += v[i] * zr[c];
    }
    for (int i = 0; i < m; ++i) {
      double* zr = &Z[(size_t)(o + i) * n];
      const double f = 2.0 * v[i];
      for (int c = 0; c < n; ++c) zr[c] -= f * zs[c];
    }
  }
  w.assign(n, 0.0);
  std::vector<double> e(n, 0.0);
  for (int i = 0; i < n; ++i) w[i] = a(i, i);
  for (int i = 0; i + 1 < n; ++i) e[i] = a(i + 1, i);

  for (int l = 0; l < n; ++l) {
    int iter = 0;
    for (;;) {
      int m = l;
      for (; m < n - 1; ++m) {
        const double dd = std::fabs(w[m]) + std::fabs(w[m + 1]);
        if (std::fabs(e[m]) <= 2.220446049250313e-16 * dd) break;
      }
      if (m == l) break;
      if (++iter > 60) return false;
      double g = (w[l + 1] - w[l]) / (2.0 * e[l]);
      double r = std::hypot(g, 1.0);
      g = w[m] - w[l] + e[l] / (g + std::copysign(r, g));
      double s = 1.0, c = 1.0, pp = 0.0;
      int i = m - 1;
      bool deflated = false;
      for (; i >= l; --i) {
        const double f = s * e[i], b = c * e[i];
        r = std::hypot(f, g);
        e[i + 1] = r;
        if (r == 0.0) {   // underflow: split the matrix here and restart
          w[i + 1] -= pp;
          e[m] = 0.0;
          deflated = true;
          break;
        }
        s = f / r;
        c = g / r;
        g = w[i + 1] - pp;
        r = (w[i] - g) * s + 2.0 * c * b;
        pp = s * r;
        w[i + 1] = g + pp;
        g = c * r - b;
        double* z0 = &Z[(size_t)i * n];
        double* z1 = &Z[(size_t)(i + 1) * n];
        for (int q = 0; q < n; ++q) {
          const double zf = z1[q];
          z1[q] = s * z0[q] + c * zf;
          z0[q] = c * z0[q] - s * zf;
        }
      }
      if (deflated) continue;
      w[l] -= pp;
      e[l] = g;
      e[m] = 0.0;
    }
  }
  return true;
}
}  // namespace

int b2k_pca_finalize_impl(b2k_ctx* ctx, const double* cov, int d, int64_t n_total, int k, double* components_out,
                          double* evr_out, double* sv_out) {
  if (!cov || !components_out || !evr_out || !sv_out)
    return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_pca_finalize: NULL argument");
  if (d < 1 || d > B2K_PCA_MAX_D)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "PCA supports 1 <= d <= " + std::to_string(B2K_PCA_MAX_D) + ", got d = " +
                                                  std::to_string(d));
  if (k < 1) return b2k_fail(ctx, B2K_ERR_INVALID, "PCA: k must be >= 1, got " + std::to_string(k));
  if (k > d)
    return b2k_fail(ctx, B2K_ERR_INVALID, "source vector size " + std::to_string(d) + " must be no less than k=" +
                                              std::to_string(k));
  if (n_total < 2)
    return b2k_fail(ctx, B2K_ERR_INVALID, "PCA needs at least 2 rows, got " + std::to_string(n_total));
  std::vector<double> A((size_t)d * d);
  double trace = 0.0;
  for (int i = 0; i < d; ++i) {
    for (int j = i; j < d; ++j) {
      const double x = cov[(size_t)i * d + j];
      if (!std::isfinite(x)) return b2k_fail(ctx, B2K_ERR_INVALID, "PCA: the covariance has a non-finite entry");
      A[(size_t)i * d + j] = A[(size_t)j * d + i] = x;
    }
    trace += cov[(size_t)i * d + i];
  }
  std::vector<double> w, Z;
  if (!sym_eig(A, d, w, Z)) return b2k_fail(ctx, B2K_ERR_INVALID, "PCA: the eigensolver did not converge");
  std::vector<int> order(d);
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return w[a] > w[b]; });
  for (int i = 0; i < k; ++i) {
    const double* z = &Z[(size_t)order[i] * d];
    int jm = 0;   // largest |value|, lowest index on a tie
    for (int j = 1; j < d; ++j)
      if (std::fabs(z[j]) > std::fabs(z[jm])) jm = j;
    const double sg = z[jm] < 0.0 ? -1.0 : 1.0;
    for (int j = 0; j < d; ++j) components_out[(size_t)i * d + j] = sg * z[j];
    const double lam = std::max(w[order[i]], 0.0);   // a PSD matrix: negative values are rounding
    evr_out[i] = trace > 0.0 ? lam / trace : 0.0;
    sv_out[i] = std::sqrt(lam * (double)(n_total - 1));
  }
  return B2K_OK;
}

int b2k_pca_fit_impl(b2k_ctx* ctx, const float* X, int64_t n, int d, int k, double* mean_out, double* components_out,
                     double* evr_out, double* sv_out, cudaStream_t s) {
  using clk = std::chrono::steady_clock;
  const auto t_begin = clk::now();
  if (!mean_out || !components_out || !evr_out || !sv_out)
    return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_pca_fit: NULL output");
  if (d > B2K_PCA_MAX_D)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "PCA supports d <= " + std::to_string(B2K_PCA_MAX_D) + ", got d = " +
                                                  std::to_string(d));
  if (k < 1) return b2k_fail(ctx, B2K_ERR_INVALID, "PCA: k must be >= 1, got " + std::to_string(k));
  if (k > d)
    return b2k_fail(ctx, B2K_ERR_INVALID, "source vector size " + std::to_string(d) + " must be no less than k=" +
                                              std::to_string(k));
  if (n > (int64_t)0x7fffff00) return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "PCA: more than 2^31 - 256 rows on one rank");
  const bool wg_ok = d % 4 == 0 && (reinterpret_cast<uintptr_t>(X) & 15u) == 0;
  if (ctx->kernel_path == B2K_PATH_FUSED && !wg_ok)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "kernel_path=2 requested but the wgmma Gram pass needs d % 4 == 0 and a "
                                              "16-byte aligned X (d = " + std::to_string(d) + ")");
  const bool wg = wg_ok && ctx->kernel_path != B2K_PATH_GENERIC;
  Timer tm(ctx->time_kernels != 0);

  // ---- plan and scratch ----
  const int ncb = (d + CS_TX - 1) / CS_TX;
  const int64_t nspan_max = std::max<int64_t>(1, (n + 63) / 64);
  const int nspan = (int)std::min<int64_t>(std::max(1, (8 * ctx->sm_count + ncb - 1) / ncb), nspan_max);
  const int64_t span_rows = std::max<int64_t>(1, (n + nspan - 1) / nspan);
  const int nblk = (d + GW_BLK - 1) / GW_BLK, ntile = nblk * (nblk + 1) / 2;
  const int nrange = (int)std::max<int64_t>(1, (n + GW_RANGE - 1) / GW_RANGE);
  int sm = ctx->sm_count;
  if (ctx->grid_limit > 0 && ctx->grid_limit < sm) sm = ctx->grid_limit;
  const int P = std::max(1, std::min(sm / ntile, nrange));   // CTAs per tile
  // generic: row spans of the fp64 partials, at most 64 MB of them
  const size_t dd = (size_t)d * d;
  const int S = (int)std::max<int64_t>(1, std::min<int64_t>({64, (int64_t)((64u << 20) / (dd * 8)), (n + GG_T - 1) / GG_T}));
  const int64_t gspan = std::max<int64_t>(1, (n + S - 1) / S);
  const size_t o_colp = 0;
  const size_t o_sums = align_up(o_colp + (size_t)nspan * d * 8, 256);
  const size_t o_mu = align_up(o_sums + (size_t)(d + 1) * 8, 256);
  const size_t o_G = align_up(o_mu + (size_t)nblk * GW_BLK * 4, 256);
  const size_t o_part = align_up(o_G + dd * 8, 1024);
  const size_t part_bytes = wg ? (size_t)P * ntile * GW_BLK * GW_BLK * 8 : (size_t)S * dd * 8;
  B2K_TRY(b2k_scratch_reserve(ctx, o_part + part_bytes));
  char* sc = static_cast<char*>(ctx->scratch);
  double* colp = reinterpret_cast<double*>(sc + o_colp);
  double* sums = reinterpret_cast<double*>(sc + o_sums);
  float* mu32_dev = reinterpret_cast<float*>(sc + o_mu);
  double* G = reinterpret_cast<double*>(sc + o_G);
  double* part = reinterpret_cast<double*>(sc + o_part);

  // ---- pass 1: column sums, allreduce of [d sums | n] ----
  tm.mark(0, s);
  if (n > 0) {
    k_colsum<<<dim3(nspan, ncb), dim3(CS_TX, CS_TY), 0, s>>>(X, n, d, span_rows, colp);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
  } else {
    B2K_CUDA_OK(ctx, cudaMemsetAsync(colp, 0, (size_t)nspan * d * 8, s));
  }
  k_colsum_fold<<<(d + 1 + 255) / 256, 256, 0, s>>>(colp, nspan, d, n, sums);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  tm.mark(1, s);
  B2K_TRY(b2k_comm_allreduce_f64(ctx, sums, (size_t)d + 1, s));
  tm.mark(2, s);
  std::vector<double> hs(d + 1);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(hs.data(), sums, (size_t)(d + 1) * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  const int64_t n_total = (int64_t)std::llround(hs[d]);
  if (n_total < 2) return b2k_fail(ctx, B2K_ERR_INVALID, "PCA needs at least 2 rows, got " + std::to_string(n_total));
  std::vector<double> mu(d), delta(d);
  std::vector<float> mu32((size_t)nblk * GW_BLK, 0.f);
  for (int c = 0; c < d; ++c) {
    mu[c] = hs[c] / (double)n_total;
    mu32[c] = (float)mu[c];
    delta[c] = mu[c] - (double)mu32[c];
  }
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(mu32_dev, mu32.data(), mu32.size() * 4, cudaMemcpyHostToDevice, s));

  // ---- pass 2: Gram matrix of the data centred on mu32, allreduce ----
  tm.mark(3, s);
  const int fold_blocks = (int)((dd + 255) / 256);
  if (wg) {
    if (n > 0) {
      CUtensorMap map;
      B2K_TRY(b2k_encode_2d(ctx, &map, X, (uint64_t)d, (uint64_t)n, (uint64_t)d * 4, 32, GW_KC,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_256B));
      GramArgs ga;
      ga.n = n;
      ga.d = d;
      ga.nblk = nblk;
      ga.ntile = ntile;
      ga.nrange = nrange;
      ga.mu = mu32_dev;
      ga.part = part;
      B2K_CUDA_OK(ctx, cudaFuncSetAttribute(k_gram_wg, cudaFuncAttributeMaxDynamicSharedMemorySize, GW_SMEM + 1024));
      k_gram_wg<<<P * ntile, GW_NTHREADS, GW_SMEM + 1024, s>>>(map, ga);
      B2K_CUDA_OK(ctx, cudaGetLastError());
      ctx->stats.kernel_launches++;
    } else {
      B2K_CUDA_OK(ctx, cudaMemsetAsync(part, 0, part_bytes, s));
    }
    k_gram_fold_wg<<<fold_blocks, 256, 0, s>>>(part, P, ntile, nblk, d, G);
  } else {
    const int nb = (d + GG_T - 1) / GG_T;
    if (n > 0) {
      k_gram_generic<<<dim3(nb * (nb + 1) / 2, S), 256, 0, s>>>(X, n, d, mu32_dev, gspan, part);
      B2K_CUDA_OK(ctx, cudaGetLastError());
      ctx->stats.kernel_launches++;
      ctx->stats.generic_launches++;
    } else {
      B2K_CUDA_OK(ctx, cudaMemsetAsync(part, 0, part_bytes, s));
    }
    k_gram_fold_generic<<<fold_blocks, 256, 0, s>>>(part, S, d, G);
  }
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  ctx->stats.last_path = wg ? B2K_PATH_FUSED : B2K_PATH_GENERIC;
  tm.mark(4, s);
  B2K_TRY(b2k_comm_allreduce_f64(ctx, G, dd, s));
  tm.mark(5, s);
  std::vector<double> cov(dd);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(cov.data(), G, dd * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));

  // ---- host: exact removal of the mu32 offset, eigen step ----
  const auto t_eig = clk::now();
  const double nt = (double)n_total, inv = 1.0 / (double)(n_total - 1);
  for (int i = 0; i < d; ++i)
    for (int j = 0; j < d; ++j) cov[(size_t)i * d + j] = (cov[(size_t)i * d + j] - nt * delta[i] * delta[j]) * inv;
  B2K_TRY(b2k_pca_finalize_impl(ctx, cov.data(), d, n_total, k, components_out, evr_out, sv_out));
  std::copy(mu.begin(), mu.end(), mean_out);
  const auto t_end = clk::now();
  if (tm.on) {
    ctx->stats.last_reduce_ms = tm.ms(0, 1);
    ctx->stats.last_allreduce_ms = tm.ms(1, 2) + tm.ms(4, 5);
    ctx->stats.last_fused_ms = tm.ms(3, 4);
    ctx->stats.last_finalize_ms = std::chrono::duration<double, std::milli>(t_end - t_eig).count();
    ctx->stats.last_loop_ms = std::chrono::duration<double, std::milli>(t_end - t_begin).count();
  }
  return B2K_OK;
}

int b2k_pca_transform_impl(b2k_ctx* ctx, const float* X, int64_t n, int d, const float* C, int k, float* Y,
                           cudaStream_t s) {
  if (d > B2K_PCA_MAX_D)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "PCA transform supports d <= " + std::to_string(B2K_PCA_MAX_D));
  if (n == 0) return B2K_OK;
  const int dpad = (d + PJ_DC - 1) / PJ_DC * PJ_DC;
  const size_t smem = ((size_t)dpad * PJ_KT + (size_t)PJ_DC * (PJ_ROWS + 1)) * 4;
  B2K_CUDA_OK(ctx, cudaFuncSetAttribute(k_project, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;
  B2K_CUDA_OK(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_project, PJ_ROWS, smem));
  const int gy = (k + PJ_KT - 1) / PJ_KT;
  const int64_t ntiles = (n + PJ_ROWS - 1) / PJ_ROWS;
  const int gx = (int)std::max<int64_t>(1, std::min<int64_t>(ntiles, (int64_t)std::max(1, per_sm) * ctx->sm_count / gy));
  k_project<<<dim3(gx, gy), PJ_ROWS, smem, s>>>(X, n, d, C, k, Y);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  return B2K_OK;
}
