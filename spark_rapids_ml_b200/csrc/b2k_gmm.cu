// Gaussian mixtures (sm_90a): b2k_gmm_fit (EM, collective) and b2k_gmm_predict (local).
//
// Model: weights w_k, means mu_k, full covariances Sigma_k (fp64, host).  Densities follow Spark's MultivariateGaussian:
// Sigma_k = U diag(lambda) U^T (b2k_sym_eig), tol = EPS lambda_max d, P_k = diag(lambda_j > tol ? lambda_j^-1/2 : 0) U^T,
// log pdf_k(x) = cst_k - ||P_k (x - mu_k)||^2 / 2 with cst_k = -(d log 2 pi + sum_{lambda_j > tol} log lambda_j) / 2.
// Rows are read in the frame of a fixed shift c (fp32): the device forms ||P_k (x - c) - b_k||^2 with b_k = P_k (mu_k - c)
// from the host in fp64.
//
//   E pass   per row and component q_ik; p_ik = w_k exp(cst_k - q_ik / 2) + EPS, r_ik = p_ik / sum_j p_ij (fp64), the
//            row's log sum_j p_ij added to a per-CTA fp64 partial; predict also writes the first argmax.
//              wgmma (k_gmm_e_wg, 3xTF32 on the pair pipeline of b2k_pair_wg.cuh): d % 4 == 0, 4 <= d <= 128, k <= 64,
//              X 16-byte aligned.  The tile is X, rewritten in shared memory as x - c (one fp32 rounding); the blocks
//              are the hi / lo planes of P_k, one 128-row block per component.  The epilogue forms
//              sum_j (D_ij - b_kj)^2 in fp64 per quad and keeps it in shared memory until the row's last component.
//              generic (k_gmm_e_generic, SIMT): every shape; P_k (x - c) in fp64 from the exact fp64 differences.
//   M pass 1 N_k and s_k = sum r_ik (x_i - c) (k_gmm_mom, fp64, folded in span order); one f64 allreduce of
//            [LL | [k][d + 1] (s_k, then N_k)]; the host forms w_k = N_k / n, mu_k = c + s_k / N_k and the centre
//            c_k = fl32(mu_k) of each component, identically on every rank.
//   M pass 2 T_k = sum (r_ik / N_k)(x_i - c_k)(x_i - c_k)^T by the weighted pass of b2k_gram.cu, its upper triangle per
//            component, the weight r_ik / N_k formed in fp64 on the device:
//              wgmma (3xTF32): d % 4 == 0, X 16-byte aligned; x - c_k rounded once to fp32 and scaled by
//              fl32(sqrt(r_ik / N_k)) at the split; grid over (component, tile) so that a row range is read from HBM
//              about once.
//              generic (SIMT): every shape; fp64 products of the exact differences.
//            Every partial is folded in a fixed order.  One f64 allreduce of the triangles; then
//            Sigma_k = T_k - (mu_k - c_k)(mu_k - c_k)^T and one eigendecomposition per component on every rank.
//            Centring each component at its own mean keeps the wgmma pass's error relative to that component's spread,
//            and the weights r / N_k sum to 1, so a component whose r lie below FLT_MIN still has its covariance.
// No atomics: two calls on the same input, rank count and device give the same bits.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "b2k_internal.cuh"

namespace {
#include "b2k_ptx.cuh"
#include "b2k_pair_wg.cuh"

constexpr double GMM_EPS = 2.220446049250313e-16;   // MLlib's EPSILON
constexpr double GMM_LOG_2PI = 1.8378770664093453;
constexpr int GMM_WG_KMAX = 64;                     // components the wgmma E pass keeps per row in shared memory

// The finished row: p_j = w_j exp(cst_j - q_j / 2) + EPS over the row's q (stride qs), r_j = p_j / sum p written to
// r_row, the first argmax to *label (if not NULL); returns log sum p.  Components in index order.
__device__ __forceinline__ double gmm_row(const double* q, int qs, int k, const double* __restrict__ w,
                                          const double* __restrict__ cst, double* __restrict__ r_row,
                                          int32_t* label) {
  double sum = 0.0;
  for (int j = 0; j < k; ++j) sum += fma(__ldg(w + j), exp(__ldg(cst + j) - 0.5 * q[j * qs]), GMM_EPS);
  const double inv = 1.0 / sum;
  double best = -1.0;
  int arg = 0;
  for (int j = 0; j < k; ++j) {
    const double r = fma(__ldg(w + j), exp(__ldg(cst + j) - 0.5 * q[j * qs]), GMM_EPS) * inv;
    r_row[j] = r;
    if (r > best) {
      best = r;
      arg = j;
    }
  }
  if (label != nullptr) *label = arg;
  return log(sum);
}

struct GmmPass {
  int64_t n;
  int d, k;
  const float* X;
  const float* c32;     // [d] the shift
  const double* P;      // generic: [k][d][d]
  const double* b;      // [k][bs]: P_k (mu_k - c), zero past d
  int bs;               // b's row stride: d (generic) or PW_N (wgmma)
  const double* cst;    // [k]
  const double* w;      // [k]
  double* r;            // [n][k]
  int32_t* labels;      // [n] or NULL
  double* part;         // [grid] per-CTA sums of log sum p
};

// ---- generic E pass: a CTA stages GE_ROWS rows as fp64 x - c; GE_LPR lanes per row split the outputs a of P_k (x - c)
// (a = lane + GE_LPR i, each a dot product in feature order), then add their squares by a fixed xor butterfly ----
constexpr int GE_ROWS = 32, GE_NT = 256, GE_LPR = GE_NT / GE_ROWS;
__global__ void __launch_bounds__(GE_NT) k_gmm_e_generic(const GmmPass a) {
  extern __shared__ __align__(16) double ge_sm[];
  double* xs = ge_sm;                               // [GE_ROWS][d]
  double* qs = ge_sm + (size_t)GE_ROWS * a.d;       // [k][GE_ROWS]
  __shared__ double sred[GE_ROWS];
  const int d = a.d, k = a.k;
  const int rl = threadIdx.x / GE_LPR, sub = threadIdx.x % GE_LPR;
  const int64_t ntiles = (a.n + GE_ROWS - 1) / GE_ROWS;
  double my_ll = 0.0;
  for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const int64_t row0 = t * GE_ROWS;
    __syncthreads();
    for (int e = threadIdx.x; e < GE_ROWS * d; e += GE_NT) {
      const int rr = e / d, f = e - rr * d;
      xs[e] = row0 + rr < a.n ? (double)a.X[row0 * d + e] - (double)a.c32[f] : 0.0;
    }
    __syncthreads();
    const double* x = xs + (size_t)rl * d;
    for (int j = 0; j < k; ++j) {
      const double* Pj = a.P + (size_t)j * d * d;
      const double* bj = a.b + (size_t)j * a.bs;
      double q = 0.0;
      for (int o = sub; o < d; o += GE_LPR) {
        const double* pr = Pj + (size_t)o * d;
        double y = 0.0;
        for (int l = 0; l < d; ++l) y = fma(__ldg(pr + l), x[l], y);
        y -= __ldg(bj + o);
        q = fma(y, y, q);
      }
#pragma unroll
      for (int m = 1; m < GE_LPR; m <<= 1) q += __shfl_xor_sync(0xffffffffu, q, m);
      if (sub == 0) qs[j * GE_ROWS + rl] = q;
    }
    const int64_t row = row0 + rl;
    if (sub == 0 && row < a.n)
      my_ll += gmm_row(qs + rl, GE_ROWS, k, a.w, a.cst, a.r + row * k, a.labels != nullptr ? a.labels + row : nullptr);
  }
  if (sub == 0) sred[rl] = my_ll;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < GE_ROWS; ++i) s += sred[i];
    a.part[blockIdx.x] = s;
  }
}

// ---- wgmma E pass ----
constexpr int GE_WG_OWN = GMM_WG_KMAX * PW_TM * 8 + 64 * 8;   // q [k][PW_TM], the adding threads' sums
template <int NCH>
using GmmWgCfg = PairWgCfg<NCH, GE_WG_OWN>;

// Persistent grid, static round-robin over tiles of PW_TM rows; a unit is one tile against the k blocks of P.  A quad's
// four lanes hold the same two rows: its first lane keeps their q, finishes them and adds their log sum p in tile
// order; the CTA folds those sums in thread order.
template <int NCH>
__global__ void __launch_bounds__(PW_NTHREADS, 1)
k_gmm_e_wg(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapHi,
           const __grid_constant__ CUtensorMap mapLo, const __grid_constant__ GmmPass a) {
  using G = GmmWgCfg<NCH>;
  constexpr int R = PW_N / 2;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t base = smem_u32(smem_raw);
  const PairWgBars bars = pair_wg_init<G>(base);
  double* qs = reinterpret_cast<double*>(smem_raw + G::OFF_OWN);   // [k][PW_TM]
  double* sred = qs + GMM_WG_KMAX * PW_TM;                         // [64]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ntiles = (int)((a.n + PW_TM - 1) / PW_TM);
  const int nit = (int)blockIdx.x < ntiles ? (ntiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;

  if (warp >= 8) {
    if (warp == 8 && elect_one())
      pair_wg_produce<G>(
          base, bars, &mapQ, &mapHi, &mapLo, nit,
          [&](int it) { return PairWgUnit{((int)blockIdx.x + it * (int)gridDim.x) * PW_TM, 0, a.k}; },
          [](int) { return false; });
    __syncwarp();
    return;
  }

  const int g = warp >> 2, wi = warp & 3;
  const int wr0 = g * 64 + wi * 16;                 // this warp's 16 rows of the tile
  const int rr0 = wr0 + (lane >> 2);                // this thread's rows rr0, rr0 + 8
  const bool lead = (lane & 3) == 0;
  double my_ll = 0.0;
  float acc[R];
  int q = 0;
  for (int it = 0; it < nit; ++it) {
    const int64_t t0 = ((int64_t)blockIdx.x + (int64_t)it * gridDim.x) * PW_TM;
    mbar_wait_nocall(bars.qfull(), (uint32_t)(it & 1));
    // x - c in place (128B swizzle: row r, column cc of chunk c at r 128 + ((cc / 4) ^ (r % 8)) 16 + (cc % 4) 4)
    for (int kk = 0; kk < 16; ++kk) {
      const int r = wr0 + kk;
      for (int col = lane; col < a.d; col += 32) {
        const int cc = col & 31;
        float* p = reinterpret_cast<float*>(smem_raw + G::OFF_Q + (col >> 5) * G::QBYTES + r * 128 +
                                            (((cc >> 2) ^ (r & 7)) << 4) + (cc & 3) * 4);
        *p = *p - __ldg(a.c32 + col);
      }
    }
    __syncwarp();
    for (int j = 0; j < a.k; ++j) {
      pair_wg_block<G>(smem_raw, base, bars, rr0, lane, acc, q);
      // acc[i] is row rr0 + 8 ((i >> 1) & 1), column 8 (i >> 2) + 2 (lane & 3) + (i & 1) of P_j (x - c)
      const double* bj = a.b + (size_t)j * PW_N + 2 * (lane & 3);
      double qh[2] = {0.0, 0.0};
#pragma unroll
      for (int i = 0; i < R; ++i) {
        const double t = (double)acc[i] - __ldg(bj + 8 * (i >> 2) + (i & 1));
        qh[(i >> 1) & 1] = fma(t, t, qh[(i >> 1) & 1]);
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        qh[h] += __shfl_xor_sync(0xffffffffu, qh[h], 1);
        qh[h] += __shfl_xor_sync(0xffffffffu, qh[h], 2);
      }
      if (lead) {
        qs[j * PW_TM + rr0] = qh[0];
        qs[j * PW_TM + rr0 + 8] = qh[1];
      }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the rewritten tile before the next TMA write
    __syncwarp();
    if (lane == 0) mbar_arrive(bars.qempty());
    if (lead)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t row = t0 + rr0 + 8 * h;
        if (row < a.n)
          my_ll += gmm_row(qs + rr0 + 8 * h, PW_TM, a.k, a.w, a.cst, a.r + row * a.k,
                           a.labels != nullptr ? a.labels + row : nullptr);
      }
  }
  if (lead) sred[threadIdx.x >> 2] = my_ll;
  asm volatile("bar.sync 1, 256;" ::: "memory");
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < 64; ++i) s += sred[i];
    a.part[blockIdx.x] = s;
  }
}

// hi / lo planes of fl32(P_j), block j = rows [128 j, 128 j + 128) x DP columns, zero past d
__global__ void __launch_bounds__(256) k_gmm_planes(const double* __restrict__ P, int k, int d, int DP,
                                                    float* __restrict__ hi, float* __restrict__ lo) {
  const int64_t total = (int64_t)k * PW_N * DP;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int l = (int)(e % DP);
    const int64_t ro = e / DP;
    const int j = (int)(ro / PW_N), o = (int)(ro % PW_N);
    const float v = (o < d && l < d) ? (float)P[((size_t)j * d + o) * d + l] : 0.f;
    const uint32_t hb = rn_tf32_bits(v);
    hi[e] = __uint_as_float(hb);
    lo[e] = __uint_as_float(rn_tf32_bits(v - __uint_as_float(hb)));
  }
}

// ---- moments: part[span][j (d + 1) + f] = sum r_ij (x_f - c_f) (f < d), sum r_ij (f = d), over the span's rows.  A
// CTA owns 32 columns f (threadIdx.x) of a group of MO_JG components (blockIdx.y = column block + blocks * group), so X
// is read k / MO_JG times per pass; each thread adds its rows (threadIdx.y + 8 i) in order, the 8 lanes in order. ----
constexpr int MO_TX = 32, MO_TY = 8, MO_JG = 8;
static_assert(MO_TY == MO_JG, "k_gmm_mom folds component y in lane y");
__global__ void __launch_bounds__(MO_TX * MO_TY)
k_gmm_mom(const float* __restrict__ X, const double* __restrict__ r, int64_t n, int d, int k,
          const float* __restrict__ c32, int64_t span_rows, double* __restrict__ part) {
  __shared__ double red[MO_TY][MO_JG][MO_TX];
  const int m = k * (d + 1);
  const int ncb = (d + 1 + MO_TX - 1) / MO_TX;
  const int f = ((int)blockIdx.y % ncb) * MO_TX + threadIdx.x;
  const int j0 = ((int)blockIdx.y / ncb) * MO_JG;
  const int64_t r0 = (int64_t)blockIdx.x * span_rows;
  const int64_t r1 = min(n, r0 + span_rows);
  double acc[MO_JG];
#pragma unroll
  for (int jj = 0; jj < MO_JG; ++jj) acc[jj] = 0.0;
  if (f <= d) {
    const double c = f < d ? (double)c32[f] : 0.0;
    for (int64_t row = r0 + threadIdx.y; row < r1; row += MO_TY) {
      const double xv = f < d ? (double)X[row * d + f] - c : 1.0;
      const double* rr = r + row * k + j0;
#pragma unroll
      for (int jj = 0; jj < MO_JG; ++jj)
        if (j0 + jj < k) acc[jj] = fma(rr[jj], xv, acc[jj]);
    }
  }
#pragma unroll
  for (int jj = 0; jj < MO_JG; ++jj) red[threadIdx.y][jj][threadIdx.x] = acc[jj];
  __syncthreads();
  const int jj = threadIdx.y;   // MO_TY == MO_JG: lane y folds component j0 + y
  if (f <= d && j0 + jj < k) {
    double t = 0.0;
#pragma unroll
    for (int y = 0; y < MO_TY; ++y) t += red[y][jj][threadIdx.x];
    part[(size_t)blockIdx.x * m + (size_t)(j0 + jj) * (d + 1) + f] = t;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------------------------------------
// The device form of a model in the frame of the shift c: P [k][d][d], b [k][bs], cst [k].  Fails when a covariance is
// not finite, the eigensolver does not converge, or no eigenvalue exceeds the tolerance.
int gmm_prepare(b2k_ctx* ctx, const char* who, int k, int d, const double* mu, const double* cov,
                const std::vector<double>& c, int bs, std::vector<double>* P, std::vector<double>* b,
                std::vector<double>* cst) {
  P->assign((size_t)k * d * d, 0.0);
  b->assign((size_t)k * bs, 0.0);
  cst->assign(k, 0.0);
  std::vector<double> A((size_t)d * d), lam, Z, dm(d);
  for (int j = 0; j < k; ++j) {
    const double* cj = cov + (size_t)j * d * d;
    for (int r = 0; r < d; ++r)
      for (int q = r; q < d; ++q) {
        const double v = cj[(size_t)r * d + q];
        if (!std::isfinite(v))
          return b2k_fail(ctx, B2K_ERR_INVALID, std::string(who) + ": component " + std::to_string(j) +
                                                    " has a non-finite covariance");
        A[(size_t)r * d + q] = A[(size_t)q * d + r] = v;
      }
    for (int f = 0; f < d; ++f) {
      dm[f] = mu[(size_t)j * d + f] - c[f];
      if (!std::isfinite(dm[f]))
        return b2k_fail(ctx, B2K_ERR_INVALID, std::string(who) + ": component " + std::to_string(j) +
                                                  " has a non-finite mean");
    }
    // QL's deflation test is relative to the eigenvalues, so a cluster of (near) zero eigenvalues may not converge:
    // then solve A + s I, s = the largest diagonal entry, whose eigenvalues are all >= s, and shift them back (an
    // absolute error of a few EPS lambda_max, below tol for d >= 8)
    std::vector<double> A0(A);
    if (!b2k_sym_eig(A, d, lam, Z)) {
      double sh = 0.0;
      for (int q = 0; q < d; ++q) sh = std::max(sh, A0[(size_t)q * d + q]);
      for (int q = 0; q < d; ++q) A0[(size_t)q * d + q] += sh;
      if (!b2k_sym_eig(A0, d, lam, Z))
        return b2k_fail(ctx, B2K_ERR_INVALID, std::string(who) + ": the eigensolver did not converge");
      for (int q = 0; q < d; ++q) lam[q] -= sh;
    }
    double lmax = 0.0;
    for (int q = 0; q < d; ++q) lmax = std::max(lmax, lam[q]);
    const double tol = GMM_EPS * lmax * d;
    double logdet = 0.0;
    int rank = 0;
    double* Pj = P->data() + (size_t)j * d * d;
    for (int q = 0; q < d; ++q) {
      if (!(lam[q] > tol)) continue;
      ++rank;
      logdet += std::log(lam[q]);
      const double s = 1.0 / std::sqrt(lam[q]);
      for (int f = 0; f < d; ++f) Pj[(size_t)q * d + f] = s * Z[(size_t)q * d + f];
    }
    if (rank == 0)
      return b2k_fail(ctx, B2K_ERR_INVALID, std::string(who) + ": the covariance of component " + std::to_string(j) +
                                                " has no eigenvalue above the tolerance (no non-zero singular values)");
    (*cst)[j] = -0.5 * (d * GMM_LOG_2PI + logdet);
    for (int q = 0; q < d; ++q) {
      double t = 0.0;
      for (int f = 0; f < d; ++f) t += Pj[(size_t)q * d + f] * dm[f];
      (*b)[(size_t)j * bs + q] = t;
    }
  }
  return B2K_OK;
}

bool gmm_wg_ok(const float* X, int d, int k) {
  return b2k_knn_wg_width(d) && k <= GMM_WG_KMAX && (reinterpret_cast<uintptr_t>(X) & 15u) == 0;
}

// The device buffers of one E pass and its model (laid out by the caller)
struct GmmE {
  bool wg;
  int DP, grid;
  float* c32;
  double *P, *b, *cst, *w, *part;
  float *hi, *lo;
};

int gmm_e_plan(b2k_ctx* ctx, const char* who, const float* X, int64_t n, int d, int k, GmmE* e) {
  const bool ok = gmm_wg_ok(X, d, k);
  if (ctx->kernel_path == B2K_PATH_FUSED && !ok)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, std::string(who) + ": kernel_path=2 requested but the wgmma E pass needs "
                                              "d % 4 == 0, 4 <= d <= 128, k <= 64 and a 16-byte aligned X (d = " +
                                              std::to_string(d) + ", k = " + std::to_string(k) + ")");
  e->wg = ok && ctx->kernel_path != B2K_PATH_GENERIC;
  e->DP = e->wg ? b2k_knn_wg_dp(d) : 0;
  int sm = ctx->sm_count;
  if (ctx->grid_limit > 0 && ctx->grid_limit < sm) sm = ctx->grid_limit;
  const int64_t ntiles = (n + (e->wg ? PW_TM : GE_ROWS) - 1) / (e->wg ? PW_TM : GE_ROWS);
  e->grid = (int)std::min<int64_t>(ntiles, e->wg ? sm : (int64_t)sm * 8);
  return B2K_OK;
}

void gmm_e_take(B2kLayout& L, GmmE& m, int d, int k) {
  const GmmE& e = m;
  m.c32 = L.take<float>((size_t)d);
  m.P = L.take<double>((size_t)k * d * d);
  m.b = L.take<double>((size_t)k * (e.wg ? PW_N : d));
  m.cst = L.take<double>((size_t)k);
  m.w = L.take<double>((size_t)k);
  m.part = L.take<double>((size_t)std::max(1, e.grid));
  m.hi = e.wg ? L.take<float>((size_t)k * PW_N * e.DP, 1024) : nullptr;
  m.lo = e.wg ? L.take<float>((size_t)k * PW_N * e.DP, 1024) : nullptr;
}

// host: the model (w, mu, cov) in the frame of c32 (one eigendecomposition per component), uploaded
int gmm_e_load(b2k_ctx* ctx, const char* who, const GmmE& e, int d, int k, const std::vector<float>& c32,
               const double* w, const double* mu, const double* cov, cudaStream_t s) {
  std::vector<double> c(c32.begin(), c32.end()), P, b, cst;
  B2K_TRY(gmm_prepare(ctx, who, k, d, mu, cov, c, e.wg ? PW_N : d, &P, &b, &cst));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(e.c32, c32.data(), (size_t)d * 4, cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(e.P, P.data(), P.size() * 8, cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(e.b, b.data(), b.size() * 8, cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(e.cst, cst.data(), (size_t)k * 8, cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(e.w, w, (size_t)k * 8, cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));   // P, b and cst die at scope end
  return B2K_OK;
}

// the E pass of the loaded model: r [n][k], labels (or NULL), ll_out (device, 1 double) = the sum of log sum p over the
// rank's rows
int gmm_e_launch(b2k_ctx* ctx, const GmmE& e, const float* X, int64_t n, int d, int k, double* r, int32_t* labels,
                 double* ll_out, cudaStream_t s) {
  GmmPass a{};
  a.n = n;
  a.d = d;
  a.k = k;
  a.X = X;
  a.c32 = e.c32;
  a.P = e.P;
  a.b = e.b;
  a.bs = e.wg ? PW_N : d;
  a.cst = e.cst;
  a.w = e.w;
  a.r = r;
  a.labels = labels;
  a.part = e.part;
  if (e.grid > 0) {
    if (e.wg) {
      const int64_t total = (int64_t)k * PW_N * e.DP;
      k_gmm_planes<<<(unsigned)std::min<int64_t>((total + 255) / 256, 4096), 256, 0, s>>>(e.P, k, d, e.DP, e.hi, e.lo);
      B2K_CUDA_OK(ctx, cudaGetLastError());
      PairWgMaps maps;
      B2K_TRY(pair_wg_maps(ctx, X, n, d, e.hi, e.lo, (int64_t)k * PW_N, e.DP, &maps));
      B2K_TRY(pair_wg_launch<GE_WG_OWN>(ctx, e.DP, [](auto nch) { return k_gmm_e_wg<decltype(nch)::value>; }, e.grid,
                                     maps, a, s));
      ctx->stats.fused_tc_launches++;
      ctx->stats.kernel_launches += 2;
    } else {
      const size_t smem = ((size_t)GE_ROWS * d + (size_t)k * GE_ROWS) * 8;
      B2K_CUDA_OK(ctx, cudaFuncSetAttribute(k_gmm_e_generic, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      k_gmm_e_generic<<<e.grid, GE_NT, smem, s>>>(a);
      B2K_CUDA_OK(ctx, cudaGetLastError());
      ctx->stats.generic_launches++;
      ctx->stats.kernel_launches++;
    }
    B2K_TRY(b2k_launch_fold_f64(ctx, e.part, e.grid, ll_out, s));
  } else {
    B2K_CUDA_OK(ctx, cudaMemsetAsync(ll_out, 0, 8, s));
  }
  ctx->stats.last_path = e.wg ? B2K_PATH_FUSED : B2K_PATH_GENERIC;
  return B2K_OK;
}

int gmm_check_shape(b2k_ctx* ctx, const char* who, int d, int k) {
  if (d > B2K_GMM_MAX_D || k > B2K_GMM_MAX_K || (int64_t)k * d * d > ((int64_t)1 << 24))
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, std::string(who) + " supports d <= " + std::to_string(B2K_GMM_MAX_D) +
                                                  ", k <= " + std::to_string(B2K_GMM_MAX_K) +
                                                  " and k d^2 <= 2^24, got d = " + std::to_string(d) + ", k = " +
                                                  std::to_string(k));
  return B2K_OK;
}

// the shift of predict: fl32 of the mixture's mean sum_k w_k mu_k, a function of the model alone
std::vector<float> gmm_model_shift(int k, int d, const double* w, const double* mu) {
  std::vector<float> c(d);
  for (int f = 0; f < d; ++f) {
    double t = 0.0;
    for (int j = 0; j < k; ++j) t += w[j] * mu[(size_t)j * d + f];
    c[f] = std::isfinite(t) ? (float)t : 0.f;
  }
  return c;
}

}  // namespace

int b2k_gmm_predict_impl(b2k_ctx* ctx, const float* X, int64_t n, int d, int k, const double* weights,
                         const double* means, const double* covs, double* prob_out, int32_t* labels_out,
                         cudaStream_t s) {
  B2K_TRY(gmm_check_shape(ctx, "Gaussian mixture predict", d, k));
  if (n > (int64_t)0x7fffff00)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "Gaussian mixture predict: more than 2^31 - 256 rows");
  GmmE e{};
  B2K_TRY(gmm_e_plan(ctx, "Gaussian mixture predict", X, n, d, k, &e));
  double* ll;
  B2K_TRY(b2k_scratch_layout(ctx, "b2k_gmm_predict", [&](B2kLayout& L) -> int {
    gmm_e_take(L, e, d, k);
    ll = L.take<double>(1);
    return B2K_OK;
  }));
  const std::vector<float> c = gmm_model_shift(k, d, weights, means);
  B2K_TRY(gmm_e_load(ctx, "Gaussian mixture predict", e, d, k, c, weights, means, covs, s));
  B2K_TRY(gmm_e_launch(ctx, e, X, n, d, k, prob_out, labels_out, ll, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));   // the host model arrays were copied from pageable memory
  return B2K_OK;
}

int b2k_gmm_fit_impl(b2k_ctx* ctx, const float* X, int64_t n, int d, int k, std::vector<double> w,
                     std::vector<double> mu, std::vector<double> cov, int max_iter, double tol, double* weights_out,
                     double* means_out, double* covs_out, double* log_likelihood_out, int* n_iter_out,
                     int64_t* cluster_sizes_out, cudaStream_t s) {
  using clk = std::chrono::steady_clock;
  const auto t_begin = clk::now();
  const char* who = "Gaussian mixture";
  B2K_TRY(gmm_check_shape(ctx, who, d, k));
  {   // the conditions that depend on a rank's own X, decided on allreduced flags so that every rank fails together
    double fl[2] = {n > (int64_t)0x7fffff00 ? 1.0 : 0.0,
                    ctx->kernel_path == B2K_PATH_FUSED && !gmm_wg_ok(X, d, k) ? 1.0 : 0.0};
    DevBuf b_fl;
    double* dfl = nullptr;
    B2K_TRY(dalloc(ctx, b_fl, 2, s, &dfl));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(dfl, fl, sizeof fl, cudaMemcpyHostToDevice, s));
    B2K_TRY(b2k_comm_allreduce_f64(ctx, dfl, 2, s));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(fl, dfl, sizeof fl, cudaMemcpyDeviceToHost, s));
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
    if (fl[0] > 0.0)
      return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "Gaussian mixture: more than 2^31 - 256 rows on one rank");
    if (fl[1] > 0.0)
      return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "Gaussian mixture: kernel_path=2 requested but the wgmma E pass needs "
                                                "d % 4 == 0, 4 <= d <= 128, k <= 64 and a 16-byte aligned X on every rank");
  }
  // the shift c = fl32 of the column means; a NaN or an infinity anywhere reaches the allreduced sums on every rank
  int64_t n_total = 0;
  std::vector<double> cm, ssq;
  B2K_TRY(b2k_colstats_impl(ctx, who, X, n, d, &n_total, &cm, &ssq, s));
  for (int f = 0; f < d; ++f)
    if (!std::isfinite(cm[f]) || !std::isfinite(ssq[f]))
      return b2k_fail(ctx, B2K_ERR_INVALID, "Gaussian mixture: the features hold a NaN or an infinity");
  std::vector<float> c32(d);
  for (int f = 0; f < d; ++f) c32[f] = (float)cm[f];

  GmmE e{};
  B2K_TRY(gmm_e_plan(ctx, who, X, n, d, k, &e));
  const int m1 = k * (d + 1);
  const int ncb = (d + 1 + MO_TX - 1) / MO_TX * ((k + MO_JG - 1) / MO_JG);   // column blocks x component groups
  const B2kRowSpans ms = b2k_row_spans(ctx, n, ncb);
  const size_t dd = (size_t)d * d, T = (size_t)d * (d + 1) / 2;
  const B2kGramPlan gp = b2k_gram_plan(ctx, X, n, d, k, ctx->kernel_path != B2K_PATH_GENERIC, (size_t)256 << 20);
  const int cspans = b2k_row_spans(ctx, n, 1).spans;   // of b2k_launch_label_counts
  const size_t nbuf = 1 + (size_t)m1 + gp.out_len;      // [LL | moments [k][d + 1] | upper triangles [k][T]]
  const size_t cstride = gp.mu_len / k;                  // of the Gram pass's centres [k][cstride]
  double *r, *mpart, *gpart, *buf, *cpart, *ginv;
  float* gcen;
  int32_t* labels;
  B2K_TRY(b2k_scratch_layout(ctx, "b2k_gmm_fit", [&](B2kLayout& L) -> int {
    gmm_e_take(L, e, d, k);
    r = L.take<double>((size_t)n * k);
    labels = L.take<int32_t>((size_t)n);
    mpart = L.take<double>((size_t)ms.spans * m1);
    gpart = L.take<double>(gp.part_len, 1024);
    gcen = L.take<float>(gp.mu_len);
    ginv = L.take<double>((size_t)k);
    buf = L.take<double>(nbuf);
    cpart = L.take<double>((size_t)cspans * k);
    return B2K_OK;
  }));
  double* mom = buf + 1;
  double* tri = mom + m1;

  B2kTimer tm(ctx->time_kernels != 0);
  double e_ms = 0.0, m_ms = 0.0, ar_ms = 0.0, host_ms = 0.0;
  std::vector<double> hb(nbuf), cd(c32.begin(), c32.end());
  std::vector<double> hinv(k), dm((size_t)k * d);   // 1 / N_k; mu_k - c_k
  std::vector<float> ck(gp.mu_len, 0.f);            // c_k = fl32(mu_k), zero past d
  double ll = -INFINITY, llp;
  int iter = 0;
  while (iter < max_iter) {
    const auto t_load = clk::now();
    B2K_TRY(gmm_e_load(ctx, who, e, d, k, c32, w.data(), mu.data(), cov.data(), s));
    host_ms += std::chrono::duration<double, std::milli>(clk::now() - t_load).count();
    tm.mark(0, s);
    B2K_TRY(gmm_e_launch(ctx, e, X, n, d, k, r, nullptr, buf, s));
    tm.mark(1, s);
    k_gmm_mom<<<dim3(ms.spans, ncb), dim3(MO_TX, MO_TY), 0, s>>>(X, r, n, d, k, e.c32, ms.span_rows, mpart);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    B2K_TRY(b2k_launch_fold_spans(ctx, mpart, ms.spans, m1, mom, s));
    tm.mark(2, s);
    B2K_TRY(b2k_comm_allreduce_f64(ctx, buf, 1 + (size_t)m1, s));
    tm.mark(3, s);
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(hb.data(), buf, (1 + (size_t)m1) * 8, cudaMemcpyDeviceToHost, s));
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
    // ---- M step, weights and means (fp64, identical on every rank), and the centres of the Gram pass ----
    auto t_host = clk::now();
    llp = ll;
    ll = hb[0];
    const double* hmom = hb.data() + 1;   // [k][d + 1]: sum r (x - c) per feature, then N_j
    for (int j = 0; j < k; ++j) {
      const double Nj = hmom[(size_t)j * (d + 1) + d];
      w[j] = Nj / (double)n_total;
      hinv[j] = 1.0 / Nj;
      for (int f = 0; f < d; ++f) {
        const double mf = cd[f] + hmom[(size_t)j * (d + 1) + f] / Nj;
        mu[(size_t)j * d + f] = mf;
        ck[(size_t)j * cstride + f] = (float)mf;
        dm[(size_t)j * d + f] = mf - (double)(float)mf;
      }
    }
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(gcen, ck.data(), ck.size() * 4, cudaMemcpyHostToDevice, s));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(ginv, hinv.data(), (size_t)k * 8, cudaMemcpyHostToDevice, s));
    host_ms += std::chrono::duration<double, std::milli>(clk::now() - t_host).count();
    tm.mark(4, s);
    B2K_TRY(b2k_gram_launch(ctx, gp, X, gcen, r, ginv, gpart, tri, s));
    if (gp.wg) {
      ctx->stats.fused_tc_launches++;
      ctx->stats.generic_launches++;
    } else {
      ctx->stats.generic_launches += 2;
    }
    ctx->stats.kernel_launches += 3;
    tm.mark(5, s);
    B2K_TRY(b2k_comm_allreduce_f64(ctx, tri, gp.out_len, s));
    tm.mark(6, s);
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(hb.data() + 1 + m1, tri, gp.out_len * 8, cudaMemcpyDeviceToHost, s));
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));   // also keeps ck and hinv alive until their copies are done
    t_host = clk::now();
    if (tm.on) {
      e_ms += tm.ms(0, 1);
      m_ms += tm.ms(1, 2) + tm.ms(4, 5);
      ar_ms += tm.ms(2, 3) + tm.ms(5, 6);
    }
    // ---- M step, covariances: Sigma_k = T_k - (mu_k - c_k)(mu_k - c_k)^T ----
    const double* htri = hmom + m1;
    for (int j = 0; j < k; ++j) {
      const double* tj = htri + (size_t)j * T;
      const double* m = dm.data() + (size_t)j * d;
      double* cj = cov.data() + (size_t)j * dd;
      size_t t = 0;
      for (int a = 0; a < d; ++a)
        for (int b = a; b < d; ++b, ++t) cj[(size_t)a * d + b] = cj[(size_t)b * d + a] = tj[t] - m[a] * m[b];
    }
    ++iter;
    host_ms += std::chrono::duration<double, std::milli>(clk::now() - t_host).count();
    if (std::fabs(ll - llp) <= tol) break;
  }

  // ---- cluster sizes: the predict pass of the final model, allreduced ----
  const std::vector<float> cpred = gmm_model_shift(k, d, w.data(), mu.data());
  B2K_TRY(gmm_e_load(ctx, who, e, d, k, cpred, w.data(), mu.data(), cov.data(), s));
  B2K_TRY(gmm_e_launch(ctx, e, X, n, d, k, r, labels, buf + k, s));   // its log-likelihood lands past the counts
  B2K_TRY(b2k_launch_label_counts(ctx, labels, n, k, cpart, buf, s));
  B2K_TRY(b2k_comm_allreduce_f64(ctx, buf, (size_t)k, s));
  std::vector<double> hc(k);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(hc.data(), buf, (size_t)k * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  for (int j = 0; j < k; ++j) cluster_sizes_out[j] = (int64_t)std::llround(hc[j]);
  std::copy(w.begin(), w.end(), weights_out);
  std::copy(mu.begin(), mu.end(), means_out);
  std::copy(cov.begin(), cov.end(), covs_out);
  *log_likelihood_out = ll;
  *n_iter_out = iter;
  ctx->stats.last_n_iter = iter;
  if (ctx->time_kernels) {
    ctx->stats.last_fused_ms = e_ms;
    ctx->stats.last_reduce_ms = m_ms;
    ctx->stats.last_allreduce_ms = ar_ms;
    ctx->stats.last_finalize_ms = host_ms;
    ctx->stats.last_loop_ms = std::chrono::duration<double, std::milli>(clk::now() - t_begin).count();
  }
  return B2K_OK;
}
