// Linear regression (sm_90a): the label pass of the moments, the host solver and the prediction kernel.
//
//   moments  b2k_moments_impl (b2k_pca.cu) runs PCA's column-sum and Gram passes on X, k_colsum on y as an [n, 1]
//            matrix, and k_xty below: sum (x - mu32)(y - muy32) and sum (y - muy32)^2, centred, multiplied and summed in
//            fp64 (the fp32 differences are exact there), per-CTA partials over fixed row spans folded in span order.
//            One f64 allreduce of the d (d + 1) / 2 + d + 1 moments (the Gram's upper triangle, X^T y, y^T y); the
//            host then removes the offsets of (mu32, muy32) from the fp64 means exactly.
//   solve    host, fp64, from the moments alone: Cholesky (minimum norm through b2k_sym_eig when a pivot is negligible)
//            for OLS / ridge, cyclic coordinate descent on the covariance for the elastic net.
//   predict  k_linreg_predict: b + sum_j x_j w_j in fp64, in an order fixed by d alone.
// No atomics anywhere: two fits of the same input are bitwise equal.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "b2k_internal.cuh"
#include "b2k_rows.cuh"

namespace {

constexpr int XT_TX = 32, XT_TY = 8;   // k_xty CTA: 32 columns of [X | y] x 8 row lanes, as k_colsum

// part[span][c] for c <= d: column c < d = sum (x_c - mu32_c)(y - muy32), column d = sum (y - muy32)^2
__global__ void __launch_bounds__(XT_TX * XT_TY)
k_xty(const float* __restrict__ X, const float* __restrict__ y, int64_t n, int d, const float* __restrict__ mu,
      float muy, int64_t span_rows, double* __restrict__ part) {
  __shared__ double red[XT_TY][XT_TX];
  const int c = blockIdx.y * XT_TX + threadIdx.x;
  const int64_t r0 = (int64_t)blockIdx.x * span_rows;
  const int64_t r1 = min(n, r0 + span_rows);
  double s = 0.0;
  if (c < d) {
    const float m = mu[c];
#pragma unroll 4
    for (int64_t r = r0 + threadIdx.y; r < r1; r += XT_TY)
      s = fma((double)X[r * d + c] - (double)m, (double)y[r] - (double)muy, s);
  } else if (c == d) {
#pragma unroll 4
    for (int64_t r = r0 + threadIdx.y; r < r1; r += XT_TY) {
      const double t = (double)y[r] - (double)muy;
      s = fma(t, t, s);
    }
  }
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && c <= d) {
    double t = 0.0;
    for (int q = 0; q < XT_TY; ++q) t += red[q][threadIdx.x];
    part[(size_t)blockIdx.x * (d + 1) + c] = t;
  }
}

// out[r] = b + sum_j x_rj w_j.  A group of L lanes (L a power of two, L = 32 from d = 100 on) owns one row: lane l
// accumulates features 4 (l + L i) .. 4 (l + L i) + 3 in order in fp64, then the group adds its lanes by a fixed xor
// butterfly.  VEC reads those four features as one float4 (d % 4 == 0, 16-byte aligned X); the scalar variant reads the
// same features one by one, so both give the same bits, and the order depends on d alone.  A warp reads 32 / L rows of
// one contiguous span: coalesced for every d.  The weights stay in shared memory in fp64, zero-padded to 4.
constexpr int LP_THREADS = 256;
template <bool VEC>
__global__ void __launch_bounds__(LP_THREADS)
k_linreg_predict(const float* __restrict__ X, int64_t n, int d, const double* __restrict__ coef, double b, int L,
                 double* __restrict__ out) {
  extern __shared__ double w_s[];
  const int dpad = (d + 3) & ~3;
  for (int j = threadIdx.x; j < dpad; j += LP_THREADS) w_s[j] = j < d ? coef[j] : 0.0;
  __syncthreads();
  const int lane = threadIdx.x & 31, sub = lane & (L - 1), grp = lane / L, rpw = 32 / L;
  const int64_t warp = ((int64_t)blockIdx.x * LP_THREADS + threadIdx.x) >> 5;
  const int64_t nwarp = ((int64_t)gridDim.x * LP_THREADS) >> 5;
  for (int64_t r0 = warp * rpw; r0 < n; r0 += nwarp * rpw) {
    const int64_t row = r0 + grp;
    double acc = 0.0;
    if (row < n) acc = b2k_linear_lane(B2kRowLdcs<VEC>{X + row * d, d}, d, w_s, sub, L);
    acc = b2k_lanes_sum(acc, L);
    if (sub == 0 && row < n) __stcs(out + row, b + acc);
  }
}

int predict_lanes(int d) { return b2k_row_lanes(d); }

bool finite_all(const double* v, size_t m) {
  for (size_t i = 0; i < m; ++i)
    if (!std::isfinite(v[i])) return false;
  return true;
}

// (A + ridge I) v = c for symmetric A [d][d]: Cholesky, or, when a pivot is <= d eps max diag, the minimum-norm solution
// of the eigendecomposition with eigenvalues <= d eps lambda_max taken as zero.
bool solve_spd_or_min_norm(std::vector<double> A, int d, double ridge, const std::vector<double>& c, std::vector<double>* v) {
  const double eps = std::ldexp(1.0, -52);
  double dmax = 0.0;
  for (int i = 0; i < d; ++i) {
    A[(size_t)i * d + i] += ridge;
    dmax = std::max(dmax, A[(size_t)i * d + i]);
  }
  const double piv_min = d * eps * dmax;
  std::vector<double> Lc(A);
  bool ok = dmax > 0.0;
  for (int j = 0; j < d && ok; ++j) {
    double* lj = &Lc[(size_t)j * d];
    double s = lj[j];
    for (int k = 0; k < j; ++k) s -= lj[k] * lj[k];
    if (!(s > piv_min)) {
      ok = false;
      break;
    }
    lj[j] = std::sqrt(s);
    for (int i = j + 1; i < d; ++i) {
      double* li = &Lc[(size_t)i * d];
      double t = li[j];
      for (int k = 0; k < j; ++k) t -= li[k] * lj[k];
      li[j] = t / lj[j];
    }
  }
  v->assign(d, 0.0);
  if (ok) {
    std::vector<double>& x = *v;
    for (int i = 0; i < d; ++i) {   // L z = c
      double t = c[i];
      for (int k = 0; k < i; ++k) t -= Lc[(size_t)i * d + k] * x[k];
      x[i] = t / Lc[(size_t)i * d + i];
    }
    for (int i = d - 1; i >= 0; --i) {   // L^T x = z
      double t = x[i];
      for (int k = i + 1; k < d; ++k) t -= Lc[(size_t)k * d + i] * x[k];
      x[i] = t / Lc[(size_t)i * d + i];
    }
    return true;
  }
  std::vector<double> w, Z;
  if (!b2k_sym_eig(A, d, w, Z)) return false;
  double lmax = 0.0;
  for (int i = 0; i < d; ++i) lmax = std::max(lmax, w[i]);
  const double thr = d * eps * lmax;
  for (int i = 0; i < d; ++i) {
    if (!(w[i] > thr)) continue;
    const double* z = &Z[(size_t)i * d];
    double p = 0.0;
    for (int j = 0; j < d; ++j) p += z[j] * c[j];
    p /= w[i];
    for (int j = 0; j < d; ++j) (*v)[j] += p * z[j];
  }
  return true;
}

}  // namespace

int b2k_xty_spans(const b2k_ctx* ctx, int64_t n, int d) {
  return b2k_row_spans(ctx, n, (d + 1 + XT_TX - 1) / XT_TX).spans;
}

int b2k_launch_xty(b2k_ctx* ctx, const float* X, const float* y, int64_t n, int d, const float* mu32, float muy32,
                   int spans, double* part, double* out, cudaStream_t s) {
  const int m = d + 1, ncb = (m + XT_TX - 1) / XT_TX;
  if (n > 0) {
    const int64_t span_rows = std::max<int64_t>(1, (n + spans - 1) / spans);
    k_xty<<<dim3(spans, ncb), dim3(XT_TX, XT_TY), 0, s>>>(X, y, n, d, mu32, muy32, span_rows, part);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
  } else {
    B2K_CUDA_OK(ctx, cudaMemsetAsync(part, 0, (size_t)spans * m * 8, s));
  }
  return b2k_launch_fold_spans(ctx, part, spans, m, out, s);
}

int b2k_linreg_moments_impl(b2k_ctx* ctx, const float* X, const float* y, int64_t n, int d, int64_t* n_total_out,
                            double* mean_out, double* moments_out, cudaStream_t s) {
  using clk = std::chrono::steady_clock;
  const auto t_begin = clk::now();
  if (d > B2K_LINREG_MAX_D)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "linear regression supports d <= " + std::to_string(B2K_LINREG_MAX_D) +
                                                  ", got d = " + std::to_string(d));
  if (n > (int64_t)0x7fffff00)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "linear regression: more than 2^31 - 256 rows on one rank");
  B2kMoments m;
  B2K_TRY(b2k_moments_impl(ctx, "linear regression", X, y, n, d, 1, &m, s));
  // NaN / inf in any row reach the allreduced sums: every rank sees them and fails here together
  if (!finite_all(m.mu.data(), m.mu.size()) || !finite_all(m.G.data(), m.G.size()))
    return b2k_fail(ctx, B2K_ERR_INVALID, "linear regression: the features or the label hold a NaN or an infinity");
  const size_t D = (size_t)d + 1, dd = (size_t)d * d;
  const double nt = (double)m.n_total;
  const std::vector<double>& dl = m.delta;
  for (int i = 0; i < d; ++i) {
    for (int j = 0; j < d; ++j) moments_out[i * D + j] = m.G[(size_t)i * d + j] - nt * dl[i] * dl[j];
    moments_out[i * D + d] = moments_out[(size_t)d * D + i] = m.G[dd + i] - nt * dl[i] * dl[d];
  }
  moments_out[(size_t)d * D + d] = m.G[dd + d] - nt * dl[d] * dl[d];
  std::copy(m.mu.begin(), m.mu.end(), mean_out);
  *n_total_out = m.n_total;
  if (ctx->time_kernels)
    ctx->stats.last_loop_ms = std::chrono::duration<double, std::milli>(clk::now() - t_begin).count();
  return B2K_OK;
}

int b2k_linreg_solve_impl(const double* mean, const double* moments, int d, int64_t n_total, double reg,
                          double l1_ratio, int fit_intercept, int standardization, int max_iter, double tol,
                          double* coef_out, double* intercept_out, int* n_iter_out) {
  auto fail = [](int code, const std::string& msg) { return b2k_fail(nullptr, code, msg); };
  if (!mean || !moments || !coef_out || !intercept_out) return fail(B2K_ERR_INVALID, "b2k_linreg_solve: NULL argument");
  if (d < 1) return fail(B2K_ERR_INVALID, "b2k_linreg_solve: d must be >= 1");
  if (d > B2K_LINREG_MAX_D)
    return fail(B2K_ERR_UNSUPPORTED, "linear regression supports d <= " + std::to_string(B2K_LINREG_MAX_D) +
                                         ", got d = " + std::to_string(d));
  if (n_total < 1) return fail(B2K_ERR_INVALID, "linear regression needs at least 1 row, got " + std::to_string(n_total));
  auto num = [](double v) {
    char buf[64];
    for (int p = 1; p <= 17; ++p) {   // the shortest form that reads back as v
      snprintf(buf, sizeof buf, "%.*g", p, v);
      if (std::strtod(buf, nullptr) == v) break;
    }
    std::string t(buf);
    if (t.find_first_of(".eni") == std::string::npos) t += ".0";   // Python's repr of a float
    return t;
  };
  if (!(reg >= 0.0)) return fail(B2K_ERR_INVALID, "regParam given invalid value " + num(reg));
  if (!(l1_ratio >= 0.0 && l1_ratio <= 1.0)) return fail(B2K_ERR_INVALID, "elasticNetParam given invalid value " + num(l1_ratio));
  if (max_iter < 0) return fail(B2K_ERR_INVALID, "maxIter given invalid value " + std::to_string(max_iter));
  if (!(tol >= 0.0)) return fail(B2K_ERR_INVALID, "tol given invalid value " + num(tol));
  const size_t D = (size_t)d + 1;
  if (!finite_all(mean, D) || !finite_all(moments, D * D))
    return fail(B2K_ERR_INVALID, "linear regression: the moments hold a NaN or an infinity");

  const double nt = (double)n_total;
  auto M = [&](int i, int j) { return moments[(size_t)i * D + j]; };   // index d = the label
  std::vector<double> s(d, 1.0);
  double sy = 1.0;
  const double muy = mean[d];
  if (standardization) {
    for (int j = 0; j < d; ++j) {
      const double sd = std::sqrt(std::max(M(j, j), 0.0) / nt);
      s[j] = sd > 0.0 ? sd : 1.0;
    }
    sy = std::sqrt(std::max(M(d, d), 0.0) / nt);
    if (sy == 0.0) {   // a constant label, as MLlib treats it
      if (fit_intercept || muy == 0.0) {
        std::fill(coef_out, coef_out + d, 0.0);
        *intercept_out = fit_intercept ? muy : 0.0;
        if (n_iter_out) *n_iter_out = 0;
        return B2K_OK;
      }
      sy = std::fabs(muy);
    }
  }
  // the solver's frame: A = Z^T Z / n, c = Z^T t / n with z = (x - mu) / s, t = (y - muy) / sy (mu = 0 without an
  // intercept: the second moments about 0 are the centred ones plus n mu mu^T)
  const double cen = fit_intercept ? 0.0 : 1.0;
  std::vector<double> A((size_t)d * d), c(d);
  for (int i = 0; i < d; ++i) {
    for (int j = 0; j < d; ++j) A[(size_t)i * d + j] = (M(i, j) + cen * nt * mean[i] * mean[j]) / nt / (s[i] * s[j]);
    c[i] = (M(i, d) + cen * nt * mean[i] * muy) / nt / (s[i] * sy);
  }
  const double lam = reg / sy, l1 = lam * l1_ratio, l2 = lam * (1.0 - l1_ratio);
  std::vector<double> v(d, 0.0);
  int iters = 0;
  if (reg == 0.0 || l1_ratio == 0.0) {
    if (!solve_spd_or_min_norm(A, d, l2, c, &v)) return fail(B2K_ERR_INVALID, "linear regression: the eigensolver did not converge");
  } else {
    // cyclic coordinate descent from v = 0, features in index order
    while (iters < max_iter) {
      ++iters;
      double dmax = 0.0, vmax = 0.0;
      for (int j = 0; j < d; ++j) {
        const double* aj = &A[(size_t)j * d];
        const double ajj = aj[j];
        double nv = 0.0;
        if (ajj > 0.0) {
          double r = c[j];
          for (int k = 0; k < d; ++k)
            if (k != j) r -= aj[k] * v[k];
          const double st = r > l1 ? r - l1 : (r < -l1 ? r + l1 : 0.0);
          nv = st / (ajj + l2);
        }
        dmax = std::max(dmax, std::fabs(nv - v[j]));
        v[j] = nv;
        vmax = std::max(vmax, std::fabs(nv));
      }
      if (dmax <= tol * vmax) break;
    }
  }
  double b = fit_intercept ? muy : 0.0;
  for (int j = 0; j < d; ++j) {
    coef_out[j] = v[j] * sy / s[j];
    if (fit_intercept) b -= coef_out[j] * mean[j];
  }
  *intercept_out = b;
  if (n_iter_out) *n_iter_out = iters;
  return B2K_OK;
}

int b2k_linreg_predict_impl(b2k_ctx* ctx, const float* X, int64_t n, int d, const double* coef, double intercept,
                            double* out, cudaStream_t s) {
  if (d > B2K_LINREG_MAX_D)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "linear regression predicts d <= " + std::to_string(B2K_LINREG_MAX_D));
  if (n == 0) return B2K_OK;
  const int L = predict_lanes(d);
  const bool vec = d % 4 == 0 && (reinterpret_cast<uintptr_t>(X) & 15u) == 0;
  const size_t smem = (size_t)((d + 3) & ~3) * 8;
  auto kern = vec ? k_linreg_predict<true> : k_linreg_predict<false>;
  int per_sm = 0;
  B2K_CUDA_OK(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, LP_THREADS, smem));
  const int64_t rows_per_cta = (int64_t)(LP_THREADS / 32) * (32 / L);
  const int64_t need = (n + rows_per_cta - 1) / rows_per_cta;
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(need, (int64_t)std::max(1, per_sm) * ctx->sm_count));
  kern<<<grid, LP_THREADS, smem, s>>>(X, n, d, coef, intercept, L, out);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  return B2K_OK;
}
