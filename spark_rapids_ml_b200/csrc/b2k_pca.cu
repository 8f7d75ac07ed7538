// PCA (sm_90a): the covariance passes, the projection kernel of transform and the host eigen step.
//
//   pass 1  k_colsum: fp64 column sums, per-CTA partials over the row spans of b2k_row_spans, folded in span order
//           (b2k_launch_fold_spans) into [d sums | n]; one f64 allreduce of d + 1 values; the host forms
//           mu = sum / n_total in fp64.
//   pass 2  the Gram matrix G = sum (x - mu32)(x - mu32)^T of the data centred on mu32 = fl32(mu), by the unweighted pass
//           of b2k_gram.cu (wgmma, 3xTF32, for d % 4 == 0 and a 16-byte aligned X; generic SIMT in fp64 for every d):
//           its upper triangle, d (d + 1) / 2 values, in one f64 allreduce, then unpacked to [d][d] on the device.  The host
//           then removes the offset of mu32 from mu exactly: cov = (G - n (mu - mu32)(mu - mu32)^T) / (n - 1).
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

// part[span][c] = sum (x_c - mu32_c)^2 over the span's rows: k_colsum's layout, the fp32 difference exact in fp64
__global__ void __launch_bounds__(CS_TX * CS_TY)
k_colsq(const float* __restrict__ X, int64_t n, int d, const float* __restrict__ mu, int64_t span_rows,
        double* __restrict__ part) {
  __shared__ double red[CS_TY][CS_TX];
  const int c = blockIdx.y * CS_TX + threadIdx.x;
  const int64_t r0 = (int64_t)blockIdx.x * span_rows;
  const int64_t r1 = min(n, r0 + span_rows);
  double s = 0.0;
  if (c < d) {
    const double m = (double)mu[c];
#pragma unroll 4
    for (int64_t r = r0 + threadIdx.y; r < r1; r += CS_TY) {
      const double t = (double)X[r * d + c] - m;
      s = fma(t, t, s);
    }
  }
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && c < d) {
    double t = 0.0;
    for (int y = 0; y < CS_TY; ++y) t += red[y][threadIdx.x];
    part[(size_t)blockIdx.x * d + c] = t;
  }
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

}  // namespace

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
bool b2k_sym_eig(std::vector<double>& A, int n, std::vector<double>& w, std::vector<double>& Z) {
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
  if (!b2k_sym_eig(A, d, w, Z)) return b2k_fail(ctx, B2K_ERR_INVALID, "PCA: the eigensolver did not converge");
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

int b2k_moments_impl(b2k_ctx* ctx, const char* who, const float* X, const float* y, int64_t n, int d, int64_t min_rows,
                     B2kMoments* m, cudaStream_t s) {
  if (ctx->kernel_path == B2K_PATH_FUSED && !b2k_gram_wg_ok(X, d))
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "kernel_path=2 requested but the wgmma Gram pass needs d % 4 == 0 and a "
                                              "16-byte aligned X (d = " + std::to_string(d) + ")");
  B2kTimer tm(ctx->time_kernels != 0);

  // ---- plan and scratch ----
  const int ncb = (d + CS_TX - 1) / CS_TX;
  const B2kRowSpans xs = b2k_row_spans(ctx, n, ncb);
  const B2kRowSpans ys = b2k_row_spans(ctx, n, 1);   // the label: one column block
  const int xty_spans = y ? b2k_xty_spans(ctx, n, d) : 0;
  const B2kGramPlan gp = b2k_gram_plan(ctx, X, n, d, 1, ctx->kernel_path != B2K_PATH_GENERIC, (size_t)64 << 20);
  const size_t T = gp.out_len, dd = (size_t)d * d;
  const size_t nsum = (size_t)d + (y ? 2 : 1), nmom = T + (y ? (size_t)d + 1 : 0);
  double *colp, *sums, *G, *Gfull, *part, *ycolp = nullptr, *xtyp = nullptr;
  float* mu32_dev;
  B2K_TRY(b2k_scratch_layout(ctx, who, [&](B2kLayout& L) -> int {
    colp = L.take<double>((size_t)xs.spans * d);
    sums = L.take<double>(nsum);
    mu32_dev = L.take<float>(gp.mu_len);
    G = L.take<double>(nmom);   // [d (d + 1) / 2] upper triangle of the Gram (+ [d] X^T y, [1] y^T y)
    Gfull = L.take<double>(dd);
    part = L.take<double>(gp.part_len, 1024);
    if (y) {
      ycolp = L.take<double>((size_t)ys.spans);
      xtyp = L.take<double>((size_t)xty_spans * (d + 1));
    }
    return B2K_OK;
  }));

  // ---- pass 1: column sums, allreduce of [d sums | n] (with a label: [d sums | label sum | n]) ----
  tm.mark(0, s);
  if (n > 0) {
    k_colsum<<<dim3(xs.spans, ncb), dim3(CS_TX, CS_TY), 0, s>>>(X, n, d, xs.span_rows, colp);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
    if (y) {
      k_colsum<<<dim3(ys.spans, 1), dim3(CS_TX, CS_TY), 0, s>>>(y, n, 1, ys.span_rows, ycolp);
      B2K_CUDA_OK(ctx, cudaGetLastError());
      ctx->stats.kernel_launches++;
    }
  } else {
    B2K_CUDA_OK(ctx, cudaMemsetAsync(colp, 0, (size_t)xs.spans * d * 8, s));
    if (y) B2K_CUDA_OK(ctx, cudaMemsetAsync(ycolp, 0, (size_t)ys.spans * 8, s));
  }
  B2K_TRY(b2k_launch_fold_spans(ctx, colp, xs.spans, d, sums, s, n));
  if (y) B2K_TRY(b2k_launch_fold_spans(ctx, ycolp, ys.spans, 1, sums + d, s, n));   // label sum, n
  tm.mark(1, s);
  B2K_TRY(b2k_comm_allreduce_f64(ctx, sums, nsum, s));
  tm.mark(2, s);
  std::vector<double> hs(nsum);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(hs.data(), sums, nsum * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  const int64_t n_total = (int64_t)std::llround(hs[nsum - 1]);
  if (n_total < min_rows)
    return b2k_fail(ctx, B2K_ERR_INVALID, std::string(who) + " needs at least " + std::to_string(min_rows) +
                                              " rows, got " + std::to_string(n_total));
  const int dm = (int)nsum - 1;   // means: d features (+ the label)
  m->n_total = n_total;
  m->mu.assign(dm, 0.0);
  m->delta.assign(dm, 0.0);
  std::vector<float> mu32(gp.mu_len, 0.f);
  float muy32 = 0.f;
  for (int c = 0; c < dm; ++c) {
    m->mu[c] = hs[c] / (double)n_total;
    const float f = (float)m->mu[c];
    if (c < d) mu32[c] = f;
    else muy32 = f;
    m->delta[c] = m->mu[c] - (double)f;
  }
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(mu32_dev, mu32.data(), mu32.size() * 4, cudaMemcpyHostToDevice, s));

  // ---- pass 2: Gram matrix of the data centred on mu32 (and X^T y), allreduce ----
  tm.mark(3, s);
  B2K_TRY(b2k_gram_launch(ctx, gp, X, mu32_dev, nullptr, nullptr, part, G, s));
  ctx->stats.kernel_launches += n > 0 ? 2 : 1;
  if (n > 0 && !gp.wg) ctx->stats.generic_launches++;
  ctx->stats.last_path = gp.wg ? B2K_PATH_FUSED : B2K_PATH_GENERIC;
  tm.mark(4, s);
  if (y) B2K_TRY(b2k_launch_xty(ctx, X, y, n, d, mu32_dev, muy32, xty_spans, xtyp, G + T, s));
  tm.mark(6, s);
  B2K_TRY(b2k_comm_allreduce_f64(ctx, G, nmom, s));
  tm.mark(5, s);
  // the triangle unpacked to [d][d] on the device, then the label's moments
  B2K_TRY(b2k_launch_gram_unpack(ctx, G, d, Gfull, s));
  m->G.resize(dd + (nmom - T));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(m->G.data(), Gfull, dd * 8, cudaMemcpyDeviceToHost, s));
  if (y) B2K_CUDA_OK(ctx, cudaMemcpyAsync(m->G.data() + dd, G + T, (nmom - T) * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  if (tm.on) {
    ctx->stats.last_reduce_ms = tm.ms(0, 1);
    ctx->stats.last_allreduce_ms = tm.ms(1, 2) + tm.ms(6, 5);
    ctx->stats.last_fused_ms = tm.ms(3, 4);
    if (y) ctx->stats.last_finalize_ms = tm.ms(4, 6);
  }
  return B2K_OK;
}

int b2k_colstats_impl(b2k_ctx* ctx, const char* who, const float* X, int64_t n, int d, int64_t* n_total,
                      std::vector<double>* mu, std::vector<double>* ssq, cudaStream_t s) {
  const int ncb = (d + CS_TX - 1) / CS_TX;
  const B2kRowSpans xs = b2k_row_spans(ctx, n, ncb);
  double *colp, *sums, *sq;
  float* mu32_dev;
  B2K_TRY(b2k_scratch_layout(ctx, who, [&](B2kLayout& L) -> int {
    colp = L.take<double>((size_t)xs.spans * d);
    sums = L.take<double>((size_t)d + 1);
    sq = L.take<double>((size_t)d + 1);
    mu32_dev = L.take<float>((size_t)d);
    return B2K_OK;
  }));
  // sums and n, allreduced; then the centred squares on mu32
  if (n > 0) {
    k_colsum<<<dim3(xs.spans, ncb), dim3(CS_TX, CS_TY), 0, s>>>(X, n, d, xs.span_rows, colp);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
  } else {
    B2K_CUDA_OK(ctx, cudaMemsetAsync(colp, 0, (size_t)xs.spans * d * 8, s));
  }
  B2K_TRY(b2k_launch_fold_spans(ctx, colp, xs.spans, d, sums, s, n));
  B2K_TRY(b2k_comm_allreduce_f64(ctx, sums, (size_t)d + 1, s));
  std::vector<double> hs((size_t)d + 1);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(hs.data(), sums, hs.size() * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  const int64_t nt = (int64_t)std::llround(hs[d]);
  if (nt < 1) return b2k_fail(ctx, B2K_ERR_INVALID, std::string(who) + " needs at least 1 row, got 0");
  mu->assign(d, 0.0);
  std::vector<float> mu32(d);
  for (int c = 0; c < d; ++c) {
    (*mu)[c] = hs[c] / (double)nt;
    mu32[c] = (float)(*mu)[c];
  }
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(mu32_dev, mu32.data(), (size_t)d * 4, cudaMemcpyHostToDevice, s));
  if (n > 0) {
    k_colsq<<<dim3(xs.spans, ncb), dim3(CS_TX, CS_TY), 0, s>>>(X, n, d, mu32_dev, xs.span_rows, colp);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
  }
  B2K_TRY(b2k_launch_fold_spans(ctx, colp, xs.spans, d, sq, s));
  B2K_TRY(b2k_comm_allreduce_f64(ctx, sq, (size_t)d, s));
  ssq->assign(d, 0.0);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(ssq->data(), sq, (size_t)d * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  for (int c = 0; c < d; ++c) {   // sum (x - mu)^2 = sum (x - mu32)^2 - n (mu - mu32)^2
    const double dl = (*mu)[c] - (double)mu32[c];
    (*ssq)[c] -= (double)nt * dl * dl;
  }
  *n_total = nt;
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
  B2kMoments m;
  B2K_TRY(b2k_moments_impl(ctx, "PCA", X, nullptr, n, d, 2, &m, s));

  // ---- host: exact removal of the mu32 offset, eigen step ----
  const auto t_eig = clk::now();
  const int64_t n_total = m.n_total;
  const std::vector<double>& delta = m.delta;
  std::vector<double>& cov = m.G;
  const double nt = (double)n_total, inv = 1.0 / (double)(n_total - 1);
  for (int i = 0; i < d; ++i)
    for (int j = 0; j < d; ++j) cov[(size_t)i * d + j] = (cov[(size_t)i * d + j] - nt * delta[i] * delta[j]) * inv;
  B2K_TRY(b2k_pca_finalize_impl(ctx, cov.data(), d, n_total, k, components_out, evr_out, sv_out));
  std::copy(m.mu.begin(), m.mu.end(), mean_out);
  const auto t_end = clk::now();
  if (ctx->time_kernels) {
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

int b2k_gram_local_impl(b2k_ctx* ctx, const float* X, int64_t n, int d, double* G, cudaStream_t s) {
  const B2kGramPlan gp = b2k_gram_plan(ctx, X, n, d, 1, false, (size_t)64 << 20);   // as b2k_moments_impl's generic pass
  double* part;
  float* zero;
  B2K_TRY(b2k_scratch_layout(ctx, "b2k_gram_local", [&](B2kLayout& L) -> int {
    part = L.take<double>(gp.part_len);
    zero = L.take<float>(gp.mu_len);
    return B2K_OK;
  }));
  B2K_CUDA_OK(ctx, cudaMemsetAsync(zero, 0, gp.mu_len * 4, s));
  B2K_TRY(b2k_gram_launch(ctx, gp, X, zero, nullptr, nullptr, part, G, s));
  ctx->stats.kernel_launches += n > 0 ? 2 : 1;
  return B2K_OK;
}
