// Sparse logistic regression (sm_90a): MLlib's objective (b2k_logreg.cu) over rows held in CSR.
//
//   check    k_csr_check: one warp per row flags an index outside [0, d), indices that are not strictly increasing and
//            a NaN or an infinity; the flags of every rank are allgathered, so that all ranks fail together.
//   CSC      built once per call, per row chunk (a chunk's residuals R [rows][kp] fp64 stay under
//            B2K_LOGREG_CSR_R_BYTES): k_csr_pack packs each entry's (chunk row, value) into 64 bits, a stable CUB radix
//            sort by column orders them; within a column the rows stay in ascending order.
//   column   k_csc_pass over fixed pieces of CSC_PIECE entries.  Runs of one column inside a piece are summed in entry
//   sums     order and written straight to their column; the first and last runs of a piece go to a carry array, and
//            k_csc_carry folds every column cut by piece boundaries in piece order.  Heavy columns of power-law data are
//            thereby split over many threads.  Used for the moments (sum x and nnz, then sum (x - mu)^2 with the
//            implicit zeros added on the host as (n - nnz) mu^2) and for the gradient sum_rows r_k x_j.
//   eval     per chunk: k_csr_rows (L lanes per row from the mean nnz; margins in fp64 in a fixed order, W gathered
//            through L2; residuals R and the per-row loss; per-CTA sums of R and of the loss, in row order), the CSC
//            pass over R, then one f64 allreduce of [kp (d + 1) | loss | n].
//   predict  k_csr_rows<false>: rawPrediction, probability and prediction, the outputs of b2k_logreg_predict.
// No floating-point atomics: the same input, rank count, device and grid_limit give the same bits.
#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <string>
#include <vector>

#include "b2k_internal.cuh"
#include "b2k_rows.cuh"

namespace {

constexpr int SP_THREADS = 256;
constexpr int MAXC = B2K_LOGREG_MAX_CLASSES;
constexpr int RC = 8;                // classes per margin sweep of a row
constexpr int CSC_PIECE = 128;       // CSC entries per thread of the column sums
constexpr int64_t CHUNK_NNZ_MAX = ((int64_t)1 << 31) - 1 - CSC_PIECE;   // CUB's item count is an int
enum { BAD_INDEX = 1, BAD_ORDER = 2, BAD_VALUE = 4 };

// ------------------------------------------------------------------------------------------------
// validation
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SP_THREADS)
k_csr_check(const int64_t* __restrict__ indptr, const int32_t* __restrict__ idx, const float* __restrict__ val,
            int64_t n, int64_t d, int* __restrict__ flags) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * SP_THREADS + threadIdx.x) >> 5;
  const int64_t nwarp = ((int64_t)gridDim.x * SP_THREADS) >> 5;
  int f = 0;
  for (int64_t r = warp; r < n; r += nwarp) {
    const int64_t p0 = indptr[r], p1 = indptr[r + 1];
    for (int64_t e = p0 + lane; e < p1; e += 32) {
      const int32_t j = idx[e];
      if (j < 0 || (int64_t)j >= d) f |= BAD_INDEX;
      if (e > p0 && idx[e - 1] >= j) f |= BAD_ORDER;
      if (!isfinite(val[e])) f |= BAD_VALUE;
    }
  }
  f = __reduce_or_sync(0xffffffffu, f);
  if (lane == 0 && f) atomicOr(flags, f);   // an integer OR: the result does not depend on the order
}

// ------------------------------------------------------------------------------------------------
// CSC build
// ------------------------------------------------------------------------------------------------
// out [e - e0] = (chunk row) | (value bits << 32) for the entries of rows [0, rows) of the chunk starting at indptr
__global__ void __launch_bounds__(SP_THREADS)
k_csr_pack(const int64_t* __restrict__ indptr, int64_t rows, const float* __restrict__ val, unsigned long long* out) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * SP_THREADS + threadIdx.x) >> 5;
  const int64_t nwarp = ((int64_t)gridDim.x * SP_THREADS) >> 5;
  const int64_t e0 = indptr[0];
  for (int64_t r = warp; r < rows; r += nwarp) {
    const int64_t p0 = indptr[r], p1 = indptr[r + 1];
    for (int64_t e = p0 + lane; e < p1; e += 32)
      out[e - e0] = (unsigned long long)(uint32_t)r | ((unsigned long long)__float_as_uint(val[e]) << 32);
  }
}

// ------------------------------------------------------------------------------------------------
// column sums over the CSC
// ------------------------------------------------------------------------------------------------
// MODE 0: G[k][c] += sum r[row][k] x (kk = kp classes); 1: G[0][c] += sum x, G[1][c] += nnz (kk = 2);
// 2: G[0][c] += sum (x - mu[c])^2 (kk = 1).  Thread (piece p, k): the piece's entries in order; its first run goes to
// carry slot 0, its last run (if it has more than one) to slot 1 (ccol = -1 when it has one run), the others to G.
template <int MODE>
__global__ void __launch_bounds__(SP_THREADS)
k_csc_pass(const uint32_t* __restrict__ col, const uint2* __restrict__ rv, int64_t nnz, int64_t npieces, int kk,
           const double* __restrict__ R, const double* __restrict__ mu, double* __restrict__ G, int64_t ldg,
           int* __restrict__ ccol, double* __restrict__ csum) {
  const int64_t t = (int64_t)blockIdx.x * SP_THREADS + threadIdx.x;
  const int64_t p = t / kk;
  const int k = (int)(t - p * kk);
  if (p >= npieces) return;
  const int64_t e0 = p * CSC_PIECE, e1 = min(nnz, e0 + CSC_PIECE);
  uint32_t cur = col[e0];
  double acc = 0.0;
  bool first = true;
  for (int64_t e = e0; e < e1; ++e) {
    const uint32_t c = col[e];
    if (c != cur) {
      if (first) {
        csum[(p * 2) * kk + k] = acc;
        if (k == 0) ccol[p * 2] = (int)cur;
        first = false;
      } else {
        G[k * ldg + cur] += acc;
      }
      cur = c;
      acc = 0.0;
    }
    const uint2 q = rv[e];
    const double x = (double)__uint_as_float(q.y);
    if (MODE == 0) {
      acc = fma(R[(int64_t)q.x * kk + k], x, acc);
    } else if (MODE == 1) {
      acc += k == 0 ? x : 1.0;
    } else {
      const double dx = x - mu[cur];
      acc = fma(dx, dx, acc);
    }
  }
  if (first) {
    csum[(p * 2) * kk + k] = acc;
    if (k == 0) {
      ccol[p * 2] = (int)cur;
      ccol[p * 2 + 1] = -1;
    }
  } else {
    csum[(p * 2 + 1) * kk + k] = acc;
    if (k == 0) ccol[p * 2 + 1] = (int)cur;
  }
}

// Thread (piece p, k): each run that starts in piece p, plus its continuations at the head of the following pieces, in
// piece order, added to G.
__global__ void __launch_bounds__(SP_THREADS)
k_csc_carry(const int* __restrict__ ccol, const double* __restrict__ csum, int64_t npieces, int kk, double* __restrict__ G,
            int64_t ldg) {
  const int64_t t = (int64_t)blockIdx.x * SP_THREADS + threadIdx.x;
  const int64_t p = t / kk;
  const int k = (int)(t - p * kk);
  if (p >= npieces) return;
  const bool one_run = ccol[p * 2 + 1] < 0;
  for (int s = 0; s < (one_run ? 1 : 2); ++s) {
    const int c = ccol[p * 2 + s];
    if (s == 0 && p > 0) {   // the head run continues a column of the previous piece: that piece's thread folds it
      const int prev = ccol[(p - 1) * 2 + 1] >= 0 ? ccol[(p - 1) * 2 + 1] : ccol[(p - 1) * 2];
      if (prev == c) continue;
    }
    double tot = csum[(p * 2 + s) * kk + k];
    bool reaches_end = s == 1 || one_run;
    for (int64_t q = p + 1; reaches_end && q < npieces && ccol[q * 2] == c; ++q) {
      tot += csum[(q * 2) * kk + k];
      reaches_end = ccol[q * 2 + 1] < 0;
    }
    G[k * ldg + c] += tot;
  }
}

// ------------------------------------------------------------------------------------------------
// rows pass (evaluation and predict)
// ------------------------------------------------------------------------------------------------
struct CsrRowsArgs {
  const int64_t* indptr;   // the chunk's rows: [rows + 1], global entry positions
  const int32_t* idx;
  const float* val;
  int64_t rows;
  int kp, L;
  const double* W;   // class k, feature j at W[k ldk + j ldj]
  int64_t ldk, ldj;
  const double* b;
  int64_t span;   // rows per CTA
  // training
  const float* y;
  const int* cmap;
  double *R, *loss, *part;   // R [rows][kp], loss [rows], part [grid][kp + 1]
  // predict
  const double* cls_val;
  double *raw, *prob, *pred;
};

// A CTA owns rows [span b, span (b + 1)); a group of L lanes forms one row's margins (b2k_csr_lanes) and lane 0 its
// outputs.  TRAIN: R and loss, then the CTA's sums over its rows in row order: part[b][k] = sum R[.][k], part[b][kp] =
// sum loss.  PREDICT: as k_logreg_rows.
template <bool TRAIN>
__global__ void __launch_bounds__(SP_THREADS) k_csr_rows(CsrRowsArgs a) {
  const int L = a.L, kp = a.kp;
  const int lane = threadIdx.x & 31, sub = lane & (L - 1), grp = lane / L, rpw = 32 / L;
  const int64_t r0 = (int64_t)blockIdx.x * a.span, r1 = min(a.rows, r0 + a.span);
  const int nout = kp == 1 ? 2 : kp;
  for (int64_t rbase = r0 + (int64_t)(threadIdx.x >> 5) * rpw; rbase < r1; rbase += (SP_THREADS / 32) * rpw) {
    const int64_t row = rbase + grp;
    const bool valid = row < r1;
    const int64_t p0 = valid ? a.indptr[row] : 0, p1 = valid ? a.indptr[row + 1] : 0;
    double* mrow = TRAIN ? a.R + (valid ? row : 0) * kp : a.raw + (valid ? row : 0) * nout;
    for (int k0 = 0; k0 < kp; k0 += RC) {
      double acc[RC];
#pragma unroll
      for (int q = 0; q < RC; ++q) acc[q] = 0.0;
      b2k_csr_lanes<RC>(a.idx, a.val, p0, p1, kp, k0, a.W, a.ldk, a.ldj, sub, L, acc);
#pragma unroll
      for (int q = 0; q < RC; ++q) acc[q] = b2k_lanes_sum(acc[q], L);
      if (sub == 0 && valid) {
#pragma unroll
        for (int q = 0; q < RC; ++q) {
          const int k = k0 + q;
          if (k < kp) mrow[(kp == 1 && !TRAIN) ? 1 : k] = a.b[k] + acc[q];
        }
      }
    }
    if (sub != 0 || !valid) continue;
    if (TRAIN) {
      a.loss[row] = b2k_row_loss_residual(mrow, kp, b2k_class_of(a.y[row], a.cmap, MAXC));
    } else if (kp == 1) {
      const double m = mrow[1];
      const double p1v = b2k_sigmoid(m);
      mrow[0] = -m;
      a.prob[row * 2 + 0] = 1.0 - p1v;
      a.prob[row * 2 + 1] = p1v;
      a.pred[row] = a.cls_val[m > 0.0 ? 1 : 0];
    } else {
      const B2kArgmax ax = b2k_softmax_argmax(mrow, kp);
      const double s = b2k_softmax_denominator(mrow, kp, ax.mx);
      for (int k = 0; k < kp; ++k) a.prob[row * kp + k] = exp(mrow[k] - ax.mx) / s;
      a.pred[row] = a.cls_val[ax.am];
    }
  }
  if (TRAIN) {
    __syncthreads();   // the CTA's R and loss rows are written
    for (int c = threadIdx.x; c <= kp; c += SP_THREADS) {
      double t = 0.0;
      for (int64_t r = r0; r < r1; ++r) t += c < kp ? a.R[r * kp + c] : a.loss[r];
      a.part[(int64_t)blockIdx.x * (kp + 1) + c] = t;
    }
  }
}

// out[k (d + 1) + d] += sum_b part[b][k], out[kp (d + 1)] += sum_b part[b][kp], the CTAs in order
__global__ void k_csr_rows_fold(const double* __restrict__ part, int grid, int kp, int64_t d, double* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c > kp) return;
  double t = 0.0;
  for (int g = 0; g < grid; ++g) t += part[(int64_t)g * (kp + 1) + c];
  out[c < kp ? (int64_t)c * (d + 1) + d : (int64_t)kp * (d + 1)] += t;
}

// ------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------
int csr_lanes(int64_t n, int64_t nnz) {   // the least power of two covering half the mean row length, at most 32
  const int64_t mean = n > 0 ? (nnz + n - 1) / n : 0;
  int L = 1;
  while (L < 32 && 2 * L < mean) L <<= 1;
  return L;
}

int grid_for(const b2k_ctx* ctx, int64_t items) {
  return (int)std::max<int64_t>(1, std::min<int64_t>((items + SP_THREADS - 1) / SP_THREADS, 16 * ctx->sm_count));
}

std::string sz(int64_t v) { return std::to_string(v); }

int check_caps(b2k_ctx* ctx, int64_t d, int kp) {
  if (d >= ((int64_t)1 << 31))
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "sparse logistic regression supports d < 2^31, got d = " + sz(d));
  if ((int64_t)kp * (d + 1) > B2K_LOGREG_CSR_MAX_PARAMS)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "sparse logistic regression supports kp (d + 1) <= " +
                                                  sz(B2K_LOGREG_CSR_MAX_PARAMS) + ", got " + sz(kp) + " x " +
                                                  sz(d + 1));
  return B2K_OK;
}

struct Chunk {
  int64_t r0, rows, e0, nnz, pieces, csc0;   // csc0: offset of the chunk's CSC in the CSC arrays
};

// The device state of one call: the rows, their CSC per chunk and every buffer the passes use, placed in one scratch
// layout.
struct CsrPlan {
  B2kCsr X;
  int d = 0, kp_max = 1, L = 1, grid_max = 1;
  std::vector<Chunk> chunks;
  int64_t rows_max = 0, nnz_max = 0, pieces_max = 0;
  size_t sort_bytes = 0;
  // device
  int *flags = nullptr, *flags_all = nullptr, *cmap = nullptr, *ccol = nullptr;
  uint32_t* csc_col = nullptr;
  uint2* csc_rv = nullptr;
  unsigned long long* pack = nullptr;
  void* sort_tmp = nullptr;
  double *csum = nullptr, *R = nullptr, *loss = nullptr, *part = nullptr, *W = nullptr, *b = nullptr, *out = nullptr,
         *mu = nullptr;
  double n_local = 0.0;   // source of the n slot of `out`
  std::vector<double> Wt;  // host staging of W in the pass's [d][kp] layout
};

int plan_rows(b2k_ctx* ctx, const B2kCsr& X, int kp_max, CsrPlan* P, cudaStream_t s) {
  P->X = X;
  P->d = (int)X.d;
  P->kp_max = kp_max;
  std::vector<int64_t> ip((size_t)X.n + 1);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(ip.data(), X.indptr, ip.size() * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  if (ip[0] != 0 || ip[X.n] != X.nnz)
    return b2k_fail(ctx, B2K_ERR_INVALID, "sparse logistic regression: indptr must start at 0 and end at nnz = " +
                                              sz(X.nnz));
  for (int64_t r = 0; r < X.n; ++r)
    if (ip[r + 1] < ip[r])
      return b2k_fail(ctx, B2K_ERR_INVALID, "sparse logistic regression: indptr decreases at row " + sz(r));
  const int64_t rows_cap = std::max<int64_t>(1, (int64_t)(B2K_LOGREG_CSR_R_BYTES / (8 * (size_t)kp_max)));
  for (int64_t r0 = 0, csc0 = 0; r0 < X.n;) {
    int64_t r1 = std::min(X.n, r0 + rows_cap);
    while (ip[r1] - ip[r0] > CHUNK_NNZ_MAX && r1 - r0 > 1) r1 = r0 + (r1 - r0) / 2;
    if (ip[r1] - ip[r0] > CHUNK_NNZ_MAX)
      return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "sparse logistic regression: a row holds more than 2^31 entries");
    Chunk c{r0, r1 - r0, ip[r0], ip[r1] - ip[r0], (ip[r1] - ip[r0] + CSC_PIECE - 1) / CSC_PIECE, csc0};
    P->chunks.push_back(c);
    P->rows_max = std::max(P->rows_max, c.rows);
    P->nnz_max = std::max(P->nnz_max, c.nnz);
    P->pieces_max = std::max(P->pieces_max, c.pieces);
    csc0 += c.nnz;
    r0 = r1;
  }
  P->L = csr_lanes(X.n, X.nnz);
  const int64_t rpc = (int64_t)(SP_THREADS / 32) * (32 / P->L);
  int64_t cap = 8 * (int64_t)ctx->sm_count;
  if (ctx->grid_limit > 0 && ctx->grid_limit < cap) cap = ctx->grid_limit;
  P->grid_max = (int)std::max<int64_t>(1, std::min<int64_t>((P->rows_max + rpc - 1) / rpc, cap));
  return B2K_OK;
}

// Places every buffer of the call; `csc` = whether the CSC and the training buffers are needed (not for predict).
int plan_place(b2k_ctx* ctx, CsrPlan* P, bool csc, cudaStream_t s) {
  const int d = P->d, kp = P->kp_max;
  const int64_t M = (int64_t)kp * (d + 1) + 1;
  if (csc && P->nnz_max > 0)
    B2K_CUDA_OK(ctx, cub::DeviceRadixSort::SortPairs(nullptr, P->sort_bytes, (const uint32_t*)nullptr,
                                                     (uint32_t*)nullptr, (const unsigned long long*)nullptr,
                                                     (unsigned long long*)nullptr, (int)P->nnz_max, 0, 32, s));
  return b2k_scratch_layout(ctx, "sparse logistic regression", [&](B2kLayout& Lo) -> int {
    P->flags = Lo.take<int>(1);
    P->flags_all = Lo.take<int>(ctx->nranks);
    if (!csc) return B2K_OK;
    P->csc_col = Lo.take<uint32_t>((size_t)P->X.nnz);
    P->csc_rv = Lo.take<uint2>((size_t)P->X.nnz);
    P->pack = Lo.take<unsigned long long>((size_t)P->nnz_max);
    P->sort_tmp = Lo.take<char>(P->sort_bytes);
    P->ccol = Lo.take<int>((size_t)P->pieces_max * 2);
    P->csum = Lo.take<double>((size_t)P->pieces_max * 2 * std::max(kp, 2));
    P->R = Lo.take<double>((size_t)P->rows_max * kp);
    P->loss = Lo.take<double>((size_t)P->rows_max);
    P->part = Lo.take<double>((size_t)P->grid_max * (kp + 1));
    P->W = Lo.take<double>((size_t)d * kp);
    P->b = Lo.take<double>((size_t)kp);
    P->cmap = Lo.take<int>(MAXC);
    P->out = Lo.take<double>((size_t)std::max<int64_t>(M + 1, 2 * ((int64_t)d + 1) + 1));
    P->mu = Lo.take<double>((size_t)d);
    return B2K_OK;
  });
}

// Device validation of the rows; collective: every rank's flags are allgathered, so that all ranks fail together.  The
// messages are those of the dense path where it has one.
int validate(b2k_ctx* ctx, CsrPlan* P, bool collective, cudaStream_t s) {
  B2K_CUDA_OK(ctx, cudaMemsetAsync(P->flags, 0, sizeof(int), s));
  if (P->X.n > 0) {
    k_csr_check<<<grid_for(ctx, P->X.n * 32), SP_THREADS, 0, s>>>(P->X.indptr, P->X.indices, P->X.values, P->X.n,
                                                                 P->X.d, P->flags);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
  }
  const int nr = collective ? ctx->nranks : 1;
  if (collective) B2K_TRY(b2k_comm_allgather_bytes(ctx, P->flags, P->flags_all, sizeof(int), s));
  else B2K_CUDA_OK(ctx, cudaMemcpyAsync(P->flags_all, P->flags, sizeof(int), cudaMemcpyDeviceToDevice, s));
  std::vector<int> h(nr);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(h.data(), P->flags_all, h.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  int f = 0;
  for (int v : h) f |= v;
  if (f & BAD_INDEX)
    return b2k_fail(ctx, B2K_ERR_INVALID, "sparse features: an index is out of bounds for vectors of size " + sz(P->X.d));
  if (f & BAD_ORDER)
    return b2k_fail(ctx, B2K_ERR_INVALID, "sparse features: the indices of a row must be strictly increasing");
  if (f & BAD_VALUE) return b2k_fail(ctx, B2K_ERR_INVALID, "logistic regression: the features hold a NaN or an infinity");
  return B2K_OK;
}

int build_csc(b2k_ctx* ctx, CsrPlan* P, cudaStream_t s) {
  int bits = 1;
  while (bits < 32 && ((int64_t)1 << bits) < P->X.d) ++bits;
  for (const Chunk& c : P->chunks) {
    if (c.nnz == 0) continue;
    k_csr_pack<<<grid_for(ctx, c.rows * 32), SP_THREADS, 0, s>>>(P->X.indptr + c.r0, c.rows, P->X.values, P->pack);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    size_t tb = P->sort_bytes;
    B2K_CUDA_OK(ctx, cub::DeviceRadixSort::SortPairs(P->sort_tmp, tb, reinterpret_cast<const uint32_t*>(P->X.indices) + c.e0,
                                                     P->csc_col + c.csc0, P->pack,
                                                     reinterpret_cast<unsigned long long*>(P->csc_rv + c.csc0),
                                                     (int)c.nnz, 0, bits, s));
    ctx->stats.kernel_launches += 2;
  }
  return B2K_OK;
}

// G [kk][ldg] += the column sums of one chunk (MODE as k_csc_pass)
template <int MODE>
int column_sums(b2k_ctx* ctx, const CsrPlan& P, const Chunk& c, int kk, const double* R, double* G, int64_t ldg,
                cudaStream_t s) {
  if (c.pieces == 0) return B2K_OK;
  const int64_t threads = c.pieces * kk;
  const int grid = (int)((threads + SP_THREADS - 1) / SP_THREADS);
  k_csc_pass<MODE><<<grid, SP_THREADS, 0, s>>>(P.csc_col + c.csc0, P.csc_rv + c.csc0, c.nnz, c.pieces, kk, R, P.mu, G,
                                               ldg, P.ccol, P.csum);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  k_csc_carry<<<grid, SP_THREADS, 0, s>>>(P.ccol, P.csum, c.pieces, kk, G, ldg);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches += 2;
  return B2K_OK;
}

// Column moments from the CSC: n_total and ssq [d] = sum over all rows (implicit zeros included) of (x - mu)^2.
int moments(b2k_ctx* ctx, CsrPlan* P, int64_t* n_total, std::vector<double>* ssq, cudaStream_t s) {
  const int d = P->d;
  const int64_t ld = (int64_t)d + 1;
  B2K_CUDA_OK(ctx, cudaMemsetAsync(P->out, 0, (size_t)(2 * ld + 1) * 8, s));
  P->n_local = (double)P->X.n;
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(P->out + 2 * ld, &P->n_local, 8, cudaMemcpyHostToDevice, s));
  for (const Chunk& c : P->chunks) B2K_TRY(column_sums<1>(ctx, *P, c, 2, nullptr, P->out, ld, s));
  B2K_TRY(b2k_comm_allreduce_f64(ctx, P->out, (size_t)(2 * ld + 1), s));
  std::vector<double> h((size_t)(2 * ld + 1));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(h.data(), P->out, h.size() * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  const double nt = h[2 * ld];
  std::vector<double> mu(d), nnz(d);
  for (int j = 0; j < d; ++j) {
    mu[j] = h[j] / nt;
    nnz[j] = h[ld + j];
  }
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(P->mu, mu.data(), (size_t)d * 8, cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaMemsetAsync(P->out, 0, (size_t)ld * 8, s));
  for (const Chunk& c : P->chunks) B2K_TRY(column_sums<2>(ctx, *P, c, 1, nullptr, P->out, ld, s));
  B2K_TRY(b2k_comm_allreduce_f64(ctx, P->out, (size_t)d, s));
  ssq->assign(d, 0.0);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(ssq->data(), P->out, (size_t)d * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));   // also: mu (host) has been read
  for (int j = 0; j < d; ++j) (*ssq)[j] += (nt - nnz[j]) * mu[j] * mu[j];
  *n_total = (int64_t)nt;
  return B2K_OK;
}

// One evaluation: out_host [kp (d + 1) + 2] as B2kLogregEval.
int eval_csr(b2k_ctx* ctx, CsrPlan* P, const float* y, int kp, const double* W, const double* b, double* out_host,
             cudaStream_t s) {
  const int d = P->d;
  const int64_t M = (int64_t)kp * (d + 1) + 1;
  P->Wt.resize((size_t)d * kp);
  for (int k = 0; k < kp; ++k)
    for (int j = 0; j < d; ++j) P->Wt[(size_t)j * kp + k] = W[(size_t)k * d + j];
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(P->W, P->Wt.data(), P->Wt.size() * 8, cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(P->b, b, (size_t)kp * 8, cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaMemsetAsync(P->out, 0, (size_t)(M + 1) * 8, s));
  P->n_local = (double)P->X.n;
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(P->out + M, &P->n_local, 8, cudaMemcpyHostToDevice, s));
  B2kTimer tm(ctx->time_kernels != 0);
  double t_rows = 0.0, t_csc = 0.0;
  const int64_t rpc = (int64_t)(SP_THREADS / 32) * (32 / P->L);
  for (const Chunk& c : P->chunks) {
    tm.mark(0, s);
    const int64_t g0 = std::min<int64_t>((c.rows + rpc - 1) / rpc, P->grid_max);
    const int64_t span = (c.rows + g0 - 1) / g0;
    const int grid = (int)((c.rows + span - 1) / span);
    CsrRowsArgs a{P->X.indptr + c.r0, P->X.indices, P->X.values, c.rows, kp, P->L, P->W, 1, kp, P->b, span,
                  y + c.r0, P->cmap, P->R, P->loss, P->part, nullptr, nullptr, nullptr, nullptr};
    k_csr_rows<true><<<grid, SP_THREADS, 0, s>>>(a);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    k_csr_rows_fold<<<(kp + 1 + 255) / 256, 256, 0, s>>>(P->part, grid, kp, d, P->out);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches += 2;
    tm.mark(1, s);
    B2K_TRY(column_sums<0>(ctx, *P, c, kp, P->R, P->out, (int64_t)d + 1, s));
    tm.mark(2, s);
    if (tm.on) {
      B2K_CUDA_OK(ctx, cudaEventSynchronize(tm.ev[2]));
      t_rows += tm.ms(0, 1);
      t_csc += tm.ms(1, 2);
    }
  }
  tm.mark(3, s);
  ctx->stats.generic_launches++;   // one per evaluation, whatever the number of row chunks
  B2K_TRY(b2k_comm_allreduce_f64(ctx, P->out, (size_t)M + 1, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(out_host, P->out, ((size_t)M + 1) * 8, cudaMemcpyDeviceToHost, s));
  tm.mark(4, s);
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  if (tm.on) {
    ctx->stats.last_fused_ms = t_rows;
    ctx->stats.last_reduce_ms = t_csc;
    ctx->stats.last_allreduce_ms = tm.ms(3, 4);
  }
  return B2K_OK;
}

using clk = std::chrono::steady_clock;
double ms_since(clk::time_point t0) { return std::chrono::duration<double, std::milli>(clk::now() - t0).count(); }

// caps, plan, scratch, validation, CSC and class map: what an evaluation or a fit needs before its first evaluation
int prepare(b2k_ctx* ctx, const B2kCsr& X, int kp_max, const double* classes, int n_classes, CsrPlan* P,
            cudaStream_t s) {
  B2K_TRY(check_caps(ctx, X.d, kp_max));
  B2K_TRY(plan_rows(ctx, X, kp_max, P, s));
  B2K_TRY(plan_place(ctx, P, true, s));
  B2K_TRY(validate(ctx, P, true, s));
  const auto t0 = clk::now();
  B2K_TRY(build_csc(ctx, P, s));
  if (ctx->time_kernels) {
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
    ctx->stats.last_finalize_ms = ms_since(t0);
  }
  const std::vector<int> cm = b2k_logreg_class_map(classes, n_classes);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(P->cmap, cm.data(), MAXC * 4, cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));   // cm is read
  return B2K_OK;
}

}  // namespace

int b2k_logreg_eval_csr_impl(b2k_ctx* ctx, const B2kCsr& X, const float* y, const double* classes, int n_classes, int kp,
                             const double* W, const double* b, double* loss_out, double* grad_out, int64_t* n_total_out,
                             cudaStream_t s) {
  if (n_classes < 1 || n_classes > MAXC) return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_logreg_eval_csr: bad class count");
  if (kp != 1 && kp != n_classes)
    return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_logreg_eval_csr: margins per row must be 1 or the class count " +
                                              std::to_string(n_classes) + ", got " + std::to_string(kp));
  CsrPlan P;
  B2K_TRY(prepare(ctx, X, kp, classes, n_classes, &P, s));
  const int64_t M = (int64_t)kp * (X.d + 1) + 1;
  std::vector<double> out((size_t)M + 1);
  B2K_TRY(eval_csr(ctx, &P, y, kp, W, b, out.data(), s));
  const double nt = out[M];
  if (nt < 1.0) return b2k_fail(ctx, B2K_ERR_INVALID, "logistic regression needs at least 1 row, got 0");
  *loss_out = out[M - 1] / nt;
  for (int64_t i = 0; i < M - 1; ++i) grad_out[i] = out[i] / nt;
  if (n_total_out) *n_total_out = (int64_t)nt;
  return B2K_OK;
}

int b2k_logreg_fit_csr_impl(b2k_ctx* ctx, const B2kCsr& X, const float* y, const double* classes, const int64_t* counts,
                            int n_classes, int n_fits, const b2k_logreg_params* prm, double* coef_out,
                            double* intercept_out, int* kp_out, int* n_iter_out, cudaStream_t s) {
  const auto t_begin = clk::now();
  B2K_TRY(b2k_logreg_check_params(ctx, n_classes, n_fits, prm));
  int kp_max = 1;
  for (int f = 0; f < n_fits; ++f)
    if (prm[f].family == 2 || (prm[f].family == 0 && n_classes > 2)) kp_max = n_classes;
  CsrPlan P;
  B2K_TRY(prepare(ctx, X, kp_max, classes, n_classes, &P, s));
  int64_t n_total = 0;
  std::vector<double> ssq;
  const auto t_mom = clk::now();
  B2K_TRY(moments(ctx, &P, &n_total, &ssq, s));
  if (ctx->time_kernels) ctx->stats.last_probe_ms = ms_since(t_mom);
  const B2kLogregEval eval = [&](int kp, const double* W, const double* b, double* out) {
    return eval_csr(ctx, &P, y, kp, W, b, out, s);
  };
  B2K_TRY(b2k_logreg_fit_settings(ctx, P.d, n_total, ssq, classes, counts, n_classes, n_fits, prm, eval, coef_out,
                                  intercept_out, kp_out, n_iter_out));
  if (ctx->time_kernels) ctx->stats.last_loop_ms = ms_since(t_begin);
  return B2K_OK;
}

int b2k_logreg_predict_csr_impl(b2k_ctx* ctx, const B2kCsr& X, int kp, const double* W, const double* b,
                                const double* class_values, double* raw_out, double* prob_out, double* pred_out,
                                cudaStream_t s) {
  B2K_TRY(check_caps(ctx, X.d, kp));
  if (X.n == 0) return B2K_OK;
  CsrPlan P;
  B2K_TRY(plan_rows(ctx, X, kp, &P, s));
  B2K_TRY(plan_place(ctx, &P, false, s));
  B2K_TRY(validate(ctx, &P, false, s));
  const int64_t rpc = (int64_t)(SP_THREADS / 32) * (32 / P.L);
  const int64_t g0 = std::max<int64_t>(1, std::min<int64_t>((X.n + rpc - 1) / rpc, 8 * (int64_t)ctx->sm_count));
  const int64_t span = (X.n + g0 - 1) / g0;
  CsrRowsArgs a{X.indptr, X.indices, X.values, X.n, kp, P.L, W, X.d, 1, b, span, nullptr, nullptr, nullptr, nullptr,
                nullptr, class_values, raw_out, prob_out, pred_out};
  k_csr_rows<false><<<(int)((X.n + span - 1) / span), SP_THREADS, 0, s>>>(a);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  return B2K_OK;
}
