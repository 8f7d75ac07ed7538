// Approximate k-NN, IVF-Flat (sm_90a): b2k_ivf_search, Euclidean distance, float32 rows.  One index over all ranks' items.
//
//   sizes   allgather of (n_items, n_queries, d, non-finite item flag) per rank; every error is decided on them.
//   queries allgather of every rank's queries, padded to the largest count, as b2k_knn_search does.
//   train   (train = 1) global row r is a training row when floor((r + 1) f) > floor(r f); each rank compacts its own
//           (k_ivf_train_rows), an allgather gives every rank the whole subset in global row order, and every rank
//           runs b2k_kmeans_fit on it as one rank (init random, seed B2K_IVF_SEED, n_iters iterations, tol = float32
//           tiny): the nlist centres are identical on every rank and do not depend on the rank count.
//   assign  b2k_kmeans_assign of the local items -> the list of each item (ties to the lowest centre).
//   index   a stable radix sort by (list, local row); each list starts at a whole block of B2K_KNN_WG_BLOCK rows, so no
//           block of the wgmma pass straddles two lists.  perm [n_pad] = the local row at each position (-1 = padding);
//           the wgmma path writes the planes of k_knn_prep through perm.
//   probes  b2k_knn_local_impl of the queries against the centres with k = nprobe: the exact k-NN rule, ties to the
//           lower list.
//   chunks  of queries whose (query, probe) pairs fit IVF_CHUNK_BYTES: the pairs are sorted by list (stable: query
//           order within a list), the query rows gathered in that order (shifted by item row 0 for the wgmma path, as
//           k_knn_shift_q does), one unit per (list, tile of its pairs) ordered by index blocks descending, one scan
//           pass of b2k_knn.cu over that unit table, and the refine of each query's nprobe partial lists through slots.
//   gather  allgather of the candidates; k_knn_merge of each own query in rank order, with the fill rule.
// Nothing uses atomics: two calls with the same input, rank count and device are bitwise equal.
#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <vector>

#include "b2k_internal.cuh"

namespace {
#include "b2k_ptx.cuh"
#include "b2k_knn_prep.cuh"

// Bytes of the gathered query rows, and of the partial lists, of one chunk of queries: each stays under this bound.
constexpr size_t IVF_CHUNK_BYTES = (size_t)256 << 20;

// the training-subset rule: rows [0, r) of the global order hold train_floor(r, f) training rows
__host__ __device__ inline int64_t train_floor(int64_t r, double f) { return (int64_t)floor((double)r * f); }

// flag = 1 when any component of X is not finite (a plain store of the same value by every writer: no atomics)
__global__ void k_ivf_nonfinite(const float* __restrict__ X, int64_t n, int64_t* flag) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    if (!isfinite(X[i])) *flag = 1;
}

// the local training rows, compacted in row order: local row i (global row0 + i) goes to row
// train_floor(row0 + i, f) - train_floor(row0, f)
__global__ void k_ivf_train_rows(const float* __restrict__ X, int64_t n, int d, int64_t row0, double f,
                                 float* __restrict__ out) {
  const int64_t t0 = train_floor(row0, f);
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n * d; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e / d, g = row0 + i;
    const int64_t t = train_floor(g, f);
    if (train_floor(g + 1, f) > t) out[(t - t0) * d + e % d] = X[e];
  }
}

__global__ void k_ivf_iota(int32_t* v, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    v[i] = (int32_t)i;
}

// off [nkeys + 1]: off[l] = first position of key l in the sorted keys [n] (keys in [0, nkeys)), off[nkeys] = n.
// Position i writes the offsets of the keys in (keys[i - 1], keys[i]]: each offset has exactly one writer.
__global__ void k_ivf_offsets(const int32_t* __restrict__ keys, int64_t n, int nkeys, int32_t* __restrict__ off) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += (int64_t)gridDim.x * blockDim.x) {
    const int prev = i == 0 ? -1 : keys[i - 1];
    const int cur = i == n ? nkeys : keys[i];
    for (int l = prev + 1; l <= cur; ++l) off[l] = (int32_t)i;
  }
}

// perm[pos_off[l] + j] = local row of the j-th item of list l (perm holds -1 elsewhere)
__global__ void k_ivf_perm(const int32_t* __restrict__ skeys, const int32_t* __restrict__ svals, int64_t n,
                           const int32_t* __restrict__ item_off, const int32_t* __restrict__ pos_off,
                           int32_t* __restrict__ perm) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int l = skeys[i];
    perm[pos_off[l] + (i - item_off[l])] = svals[i];
  }
}

// pairs of a chunk: pair i = q * nprobe + j has key = the probed list (nlist when the query probed nothing there)
__global__ void k_ivf_pairs(const int64_t* __restrict__ probes, int64_t npairs, int nlist, int32_t* __restrict__ keys,
                            int32_t* __restrict__ vals) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < npairs; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t l = probes[i];
    keys[i] = l >= 0 && l < nlist ? (int32_t)l : nlist;
    vals[i] = (int32_t)i;
  }
}

// slots[pair] = its position in list order, or -1 when its list is empty on this rank (nothing is scanned for it)
__global__ void k_ivf_slots(const int32_t* __restrict__ skeys, const int32_t* __restrict__ svals, int64_t npairs,
                            int nlist, const int32_t* __restrict__ item_off, int32_t* __restrict__ slots) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < npairs; i += (int64_t)gridDim.x * blockDim.x) {
    const int l = skeys[i];
    slots[svals[i]] = l < nlist && item_off[l + 1] > item_off[l] ? (int32_t)i : -1;
  }
}

// Qg [npairs][d]: row i = the query of sorted pair i; shifted by item row 0 (non-finite components -> 0) when S is set
__global__ void k_ivf_gather_q(const float* __restrict__ Q, const int32_t* __restrict__ svals, int64_t npairs,
                               int nprobe, int d, const float* __restrict__ S, float* __restrict__ Qg) {
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < npairs * d;
       e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e / d;
    const int f = (int)(e % d);
    const float v = Q[(int64_t)(svals[i] / nprobe) * d + f];
    Qg[e] = S != nullptr ? knn_shifted_q(v, knn_shift(S, f)) : v;
  }
}

__global__ void k_ivf_narrow(const int64_t* __restrict__ in, int64_t n, int32_t* __restrict__ out) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = (int32_t)in[i];
}

unsigned grid_for(const b2k_ctx* ctx, int64_t n) {
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, (int64_t)ctx->sm_count * 16));
}

int key_bits(int nkeys) {   // radix bits that hold the keys [0, nkeys]
  int b = 1;
  while (b < 31 && (1 << b) <= nkeys) ++b;
  return b;
}

// the training fit runs on every rank alone, over the gathered training subset: no collective inside it
struct OneRankScope {
  b2k_ctx* c;
  int nranks, rank;
  explicit OneRankScope(b2k_ctx* c_) : c(c_), nranks(c_->nranks), rank(c_->rank) {
    c->nranks = 1;
    c->rank = 0;
  }
  ~OneRankScope() {
    c->nranks = nranks;
    c->rank = rank;
  }
};

// per chunk of queries: events after the pair sort and gather and after the scan (option time_kernels)
struct ChunkEvents {
  std::vector<cudaEvent_t> ev;
  ~ChunkEvents() {
    for (auto& e : ev) cudaEventDestroy(e);
  }
  int mark(b2k_ctx* ctx, bool on, cudaStream_t s) {
    if (!on) return B2K_OK;
    ev.emplace_back();
    B2K_CUDA_OK(ctx, cudaEventCreate(&ev.back()));
    B2K_CUDA_OK(ctx, cudaEventRecord(ev.back(), s));
    return B2K_OK;
  }
  double scan_ms() const {
    double t = 0.0;
    for (size_t i = 0; i + 1 < ev.size(); i += 2) {
      float m = 0.f;
      cudaEventElapsedTime(&m, ev[i], ev[i + 1]);
      t += m;
    }
    return t;
  }
};

// runs the build and probe steps on the kernel path each of them chooses; kernel_path applies to the scan alone
struct PathScope {
  b2k_ctx* c;
  int saved;
  explicit PathScope(b2k_ctx* c_) : c(c_), saved(c_->kernel_path) { c->kernel_path = B2K_PATH_AUTO; }
  ~PathScope() { c->kernel_path = saved; }
};
}  // namespace

int b2k_ivf_search_impl(b2k_ctx* ctx, const float* items, int64_t n_items, const int64_t* item_ids,
                        const float* queries, int64_t nq_local, int d, int k, int nlist, int nprobe_in, int n_iters,
                        double train_fraction, int metric, int train, float* centers, int32_t* item_list_out,
                        int32_t* probe_out, float* dist_out, int64_t* idx_out, cudaStream_t s) {
  const char* who = "b2k_ivf_search";
  const int nr = ctx->nranks;
  B2kTimer tm(ctx->time_kernels != 0);
  auto fail = [&](int code, const std::string& m) { return b2k_fail(ctx, code, std::string(who) + ": " + m); };

  // ---- sizes and the non-finite flag of every rank; each error is decided on them, identically on every rank ----
  DevBuf b_sz;
  int64_t* sz_dev;
  B2K_TRY(dalloc(ctx, b_sz, (size_t)4 * (nr + 1), s, &sz_dev));
  const int64_t mine[3] = {n_items, nq_local, d};
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(sz_dev, mine, sizeof(mine), cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaMemsetAsync(sz_dev + 3, 0, 8, s));
  if (n_items > 0) {
    k_ivf_nonfinite<<<grid_for(ctx, n_items * d), 256, 0, s>>>(items, n_items * d, sz_dev + 3);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
  }
  B2K_TRY(b2k_comm_allgather_i64(ctx, sz_dev, sz_dev + 4, 4, s));
  std::vector<int64_t> sz((size_t)4 * nr);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(sz.data(), sz_dev + 4, sz.size() * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  int64_t n_total = 0, row0 = 0, nq_max = 0, nq_total = 0;
  std::vector<int64_t> rank_row0(nr);
  for (int r = 0; r < nr; ++r) {
    if (sz[4 * r + 2] != sz[2])
      return fail(B2K_ERR_INVALID, "d differs between ranks (rank " + std::to_string(r) + " has d = " +
                                       std::to_string(sz[4 * r + 2]) + ", rank 0 has d = " + std::to_string(sz[2]) + ")");
    if (sz[4 * r + 3] != 0)
      return fail(B2K_ERR_INVALID, "an item has a non-finite component (rank " + std::to_string(r) + ")");
    rank_row0[r] = n_total;
    if (r < ctx->rank) row0 += sz[4 * r];
    n_total += sz[4 * r];
    nq_max = std::max(nq_max, sz[4 * r + 1]);
    nq_total += sz[4 * r + 1];
  }
  if (n_total == 0) return fail(B2K_ERR_INVALID, "the index is empty on every rank");
  if (k < 1 || k > n_total)
    return fail(B2K_ERR_INVALID, "k = " + std::to_string(k) + " must satisfy 1 <= k <= " + std::to_string(n_total) +
                                     " (items on all ranks)");
  if (k > B2K_KNN_MAX_K)
    return fail(B2K_ERR_UNSUPPORTED, "k = " + std::to_string(k) + " exceeds " + std::to_string(B2K_KNN_MAX_K));
  if (n_total > (int64_t)0x7fffffff) return fail(B2K_ERR_UNSUPPORTED, "more than 2^31 - 1 items in all");
  if (metric != B2K_IVF_EUCLIDEAN && metric != B2K_IVF_SQEUCLIDEAN)
    return fail(B2K_ERR_INVALID, "unknown metric " + std::to_string(metric));
  if (nlist < 1) return fail(B2K_ERR_INVALID, "nlist = " + std::to_string(nlist) + " must be >= 1");
  if (nprobe_in < 1) return fail(B2K_ERR_INVALID, "nprobe = " + std::to_string(nprobe_in) + " must be >= 1");
  const int nprobe = std::min(nprobe_in, nlist);
  if (nprobe > B2K_KNN_MAX_LISTS)
    return fail(B2K_ERR_UNSUPPORTED, "nprobe = " + std::to_string(nprobe) + " (after clamping to nlist) exceeds " +
                                         std::to_string(B2K_KNN_MAX_LISTS));
  std::vector<int64_t> t_rank(nr);
  if (train) {
    if (!(train_fraction > 0.0 && train_fraction <= 1.0))
      return fail(B2K_ERR_INVALID, "kmeans_trainset_fraction = " + std::to_string(train_fraction) +
                                       " must lie in (0, 1]");
    if (n_iters < 1) return fail(B2K_ERR_INVALID, "kmeans_n_iters = " + std::to_string(n_iters) + " must be >= 1");
    const int64_t t_total = train_floor(n_total, train_fraction);
    if (nlist > t_total)
      return fail(B2K_ERR_INVALID, "nlist = " + std::to_string(nlist) + " exceeds the " + std::to_string(t_total) +
                                       " training rows");
    for (int r = 0; r < nr; ++r)
      t_rank[r] = train_floor(rank_row0[r] + sz[4 * r], train_fraction) - train_floor(rank_row0[r], train_fraction);
  }
  const bool wg_shape = b2k_knn_wg_shape(d, k);
  if (ctx->kernel_path == B2K_PATH_FUSED && !wg_shape)
    return fail(B2K_ERR_UNSUPPORTED, "kernel_path=2 requested but the wgmma scan needs d % 4 == 0, 4 <= d <= 128 and "
                                     "k <= 64 (d = " + std::to_string(d) + ", k = " + std::to_string(k) + ")");
  const bool wg = wg_shape && ctx->kernel_path != B2K_PATH_GENERIC;
  const int DP = b2k_knn_wg_dp(d);
  const int64_t nq_all = nr > 1 ? nq_max * nr : nq_local;
  tm.mark(0, s);

  // ---- queries of every rank ----
  DevBuf b_q;
  const float* Q = queries;
  if (nr > 1 && nq_total > 0) {
    float* Qall;
    B2K_TRY(dalloc(ctx, b_q, (size_t)nq_all * d, s, &Qall));
    float* mineq = Qall + (size_t)ctx->rank * nq_max * d;
    if (nq_local > 0)
      B2K_CUDA_OK(ctx, cudaMemcpyAsync(mineq, queries, (size_t)nq_local * d * 4, cudaMemcpyDeviceToDevice, s));
    if (nq_max > nq_local)
      B2K_CUDA_OK(ctx, cudaMemsetAsync(mineq + (size_t)nq_local * d, 0, (size_t)(nq_max - nq_local) * d * 4, s));
    B2K_TRY(b2k_comm_allgather_bytes(ctx, mineq, Qall, (size_t)nq_max * d * 4, s));
    Q = Qall;
  }
  tm.mark(1, s);

  // ---- centres and the list of every local item (b2k_kmeans_* lay out the scratch themselves) ----
  DevBuf b_lab;
  int32_t* labels = nullptr;
  B2K_TRY(dalloc(ctx, b_lab, (size_t)n_items, s, &labels));
  {
    PathScope ps(ctx);
    if (train) {
      // every rank gathers the whole training subset in global row order and fits it as one rank: ranks with no
      // training row take part, and the centres depend on neither the rank count nor the partitioning
      int64_t t_max = 0, t_total = 0;
      for (int r = 0; r < nr; ++r) {
        t_max = std::max(t_max, t_rank[r]);
        t_total += t_rank[r];
      }
      DevBuf b_train;
      float* Tg;
      B2K_TRY(dalloc(ctx, b_train, (size_t)(nr > 1 ? nr * t_max + t_total : t_total) * d, s, &Tg));
      float* mine_t = nr > 1 ? Tg + (size_t)ctx->rank * t_max * d : Tg;
      if (n_items > 0) {
        k_ivf_train_rows<<<grid_for(ctx, n_items * d), 256, 0, s>>>(items, n_items, d, row0, train_fraction, mine_t);
        B2K_CUDA_OK(ctx, cudaGetLastError());
        ctx->stats.kernel_launches++;
      }
      float* Xt = Tg;
      if (nr > 1) {
        B2K_TRY(b2k_comm_allgather_bytes(ctx, mine_t, Tg, (size_t)t_max * d * 4, s));
        Xt = Tg + (size_t)nr * t_max * d;
        int64_t o = 0;
        for (int r = 0; r < nr; ++r) {
          if (t_rank[r] > 0)
            B2K_CUDA_OK(ctx, cudaMemcpyAsync(Xt + (size_t)o * d, Tg + (size_t)r * t_max * d,
                                             (size_t)t_rank[r] * d * 4, cudaMemcpyDeviceToDevice, s));
          o += t_rank[r];
        }
      }
      OneRankScope one(ctx);
      int n_iter = 0;
      B2K_TRY(b2k_kmeans_fit(ctx, Xt, t_total, d, nlist, B2K_INIT_RANDOM, nullptr, n_iters, (double)FLT_MIN,
                             B2K_IVF_SEED, 0.0, 1, centers, &n_iter, nullptr, reinterpret_cast<uintptr_t>(s)));
    }
    if (n_items > 0)
      B2K_TRY(b2k_kmeans_assign(ctx, items, n_items, d, centers, nlist, labels, nullptr, reinterpret_cast<uintptr_t>(s)));
  }
  if (item_list_out != nullptr && n_items > 0)
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(item_list_out, labels, (size_t)n_items * 4, cudaMemcpyDeviceToDevice, s));

  // ---- the list-ordered index ----
  DevBuf b_idx;
  int32_t *perm = nullptr, *item_off = nullptr, *pos_off_dev = nullptr;
  float *Xhi = nullptr, *Xlo = nullptr, *norms = nullptr;
  std::vector<int32_t> item_off_h((size_t)nlist + 1, 0), pos_off_h((size_t)nlist + 1, 0);
  int64_t n_pad = 0;
  if (n_items > 0) {
    int32_t *keys_s, *vals, *vals_s;
    size_t sort_bytes = 0;
    const int ibits = key_bits(nlist);
    B2K_CUDA_OK(ctx, cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, labels, (int32_t*)nullptr, (int32_t*)nullptr,
                                                     (int32_t*)nullptr, (int)n_items, 0, ibits, s));
    DevBuf b_sort;
    char* tmp;
    B2K_TRY(dalloc(ctx, b_sort, sort_bytes + (size_t)3 * (n_items + 256) * 4 + (size_t)2 * (nlist + 1) * 4 + 1024, s,
                   &tmp));
    B2kLayout L(tmp, sort_bytes + (size_t)3 * (n_items + 256) * 4 + (size_t)2 * (nlist + 1) * 4 + 1024);
    void* sort_tmp = L.take<char>(sort_bytes);
    keys_s = L.take<int32_t>((size_t)n_items);
    vals = L.take<int32_t>((size_t)n_items);
    vals_s = L.take<int32_t>((size_t)n_items);
    item_off = L.take<int32_t>((size_t)nlist + 1);
    pos_off_dev = L.take<int32_t>((size_t)nlist + 1);
    B2K_TRY(L.check(ctx, who));
    k_ivf_iota<<<grid_for(ctx, n_items), 256, 0, s>>>(vals, n_items);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    // LSD radix sort: stable, so each list keeps its items in local row order
    B2K_CUDA_OK(ctx, cub::DeviceRadixSort::SortPairs(sort_tmp, sort_bytes, labels, keys_s, vals, vals_s, (int)n_items, 0,
                                                     ibits, s));
    k_ivf_offsets<<<grid_for(ctx, n_items + 1), 256, 0, s>>>(keys_s, n_items, nlist, item_off);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches += 3;
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(item_off_h.data(), item_off, item_off_h.size() * 4, cudaMemcpyDeviceToHost, s));
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
    for (int l = 0; l < nlist; ++l) {
      const int64_t c = item_off_h[l + 1] - item_off_h[l];
      n_pad += (c + B2K_KNN_WG_BLOCK - 1) / B2K_KNN_WG_BLOCK * B2K_KNN_WG_BLOCK;
      if (n_pad > (int64_t)0x7fffff00) return fail(B2K_ERR_UNSUPPORTED, "more than 2^31 - 256 padded index rows");
      pos_off_h[l + 1] = (int32_t)n_pad;
    }
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(pos_off_dev, pos_off_h.data(), pos_off_h.size() * 4, cudaMemcpyHostToDevice, s));
    char* ib;
    const size_t ib_bytes = (size_t)n_pad * 4 + 1024 + (wg ? (size_t)n_pad * (2 * DP + 1) * 4 + 3 * 1024 : 0);
    B2K_TRY(dalloc(ctx, b_idx, ib_bytes, s, &ib));
    B2kLayout LI(ib, ib_bytes);
    perm = LI.take<int32_t>((size_t)n_pad);
    if (wg) {
      Xhi = LI.take<float>((size_t)n_pad * DP, 1024);
      Xlo = LI.take<float>((size_t)n_pad * DP, 1024);
      norms = LI.take<float>((size_t)n_pad);
    }
    B2K_TRY(LI.check(ctx, who));
    B2K_CUDA_OK(ctx, cudaMemsetAsync(perm, 0xff, (size_t)n_pad * 4, s));
    k_ivf_perm<<<grid_for(ctx, n_items), 256, 0, s>>>(keys_s, vals_s, n_items, item_off, pos_off_dev, perm);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
    if (wg) B2K_TRY(b2k_knn_prep_launch(ctx, items, n_items, d, perm, n_pad, DP, Xhi, Xlo, norms, s));
    // item_off stays in use by k_ivf_slots: keep it apart from the sort buffer, which is freed here
    int32_t* io;
    B2K_TRY(dalloc(ctx, b_lab, (size_t)nlist + 1, s, &io));   // the labels are no longer needed
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(io, item_off_h.data(), item_off_h.size() * 4, cudaMemcpyHostToDevice, s));
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));   // item_off_h and pos_off_h are pageable
    item_off = io;
  }
  tm.mark(2, s);
  if (nq_total == 0) return B2K_OK;

  // ---- probes of every query ----
  DevBuf b_probe;
  char* pb;
  B2K_TRY(dalloc(ctx, b_probe, (size_t)nq_all * nprobe * 12 + 512, s, &pb));
  int64_t* pidx = reinterpret_cast<int64_t*>(pb);
  float* pdist = reinterpret_cast<float*>(pb + (((size_t)nq_all * nprobe * 8 + 255) / 256 * 256));
  {
    PathScope ps(ctx);
    B2K_TRY(b2k_knn_local_impl(ctx, centers, nlist, Q, nq_all, d, nprobe, pdist, pidx, s));
  }
  const int64_t qown0 = nr > 1 ? (int64_t)ctx->rank * nq_max : 0;
  if (probe_out != nullptr && nq_local > 0) {
    k_ivf_narrow<<<grid_for(ctx, nq_local * nprobe), 256, 0, s>>>(pidx + qown0 * nprobe, nq_local * nprobe, probe_out);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
  }
  tm.mark(3, s);

  // ---- chunks of queries: pairs by list, scan, refine ----
  const int64_t qt = wg ? B2K_KNN_WG_QROWS : B2K_KNN_GEN_QROWS;
  const size_t pair_bytes = (size_t)std::max(d * 4, k * 8);
  const int64_t nqc_max =
      std::max<int64_t>(1, std::min<int64_t>(nq_all, (int64_t)(IVF_CHUNK_BYTES / ((size_t)nprobe * pair_bytes))));
  const int64_t P_max = nqc_max * nprobe;
  const int64_t units_max = P_max / qt + nlist + 1;
  const int pbits = key_bits(nlist + 1);
  int32_t *pkeys = nullptr, *pkeys_s = nullptr, *pvals = nullptr, *pvals_s = nullptr, *pair_off = nullptr,
          *slots = nullptr;
  float* Qg = nullptr;
  KnnUnit* units_dev = nullptr;
  int2* part = nullptr;
  KnnCand *cand = nullptr, *cand_all = nullptr;
  void* sort_tmp = nullptr;
  size_t sort_bytes = 0;
  if (n_items > 0)
    B2K_CUDA_OK(ctx, cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (int32_t*)nullptr, (int32_t*)nullptr,
                                                     (int32_t*)nullptr, (int32_t*)nullptr, (int)P_max, 0, pbits, s));
  B2K_TRY(b2k_scratch_layout(ctx, "IVF search", [&](B2kLayout& L) -> int {
    if (n_items > 0) {
      sort_tmp = L.take<char>(sort_bytes);
      pkeys = L.take<int32_t>((size_t)P_max);
      pkeys_s = L.take<int32_t>((size_t)P_max);
      pvals = L.take<int32_t>((size_t)P_max);
      pvals_s = L.take<int32_t>((size_t)P_max);
      pair_off = L.take<int32_t>((size_t)nlist + 2);
      slots = L.take<int32_t>((size_t)P_max);
      Qg = L.take<float>((size_t)P_max * d, 1024);
      units_dev = L.take<KnnUnit>((size_t)units_max);
      part = L.take<int2>((size_t)P_max * k);
    }
    cand = L.take<KnnCand>((size_t)nq_all * k);
    if (nr > 1) cand_all = L.take<KnnCand>((size_t)nr * nq_all * k);
    return B2K_OK;
  }));
  ChunkEvents cev;
  if (n_items == 0) {
    tm.mark(4, s);
    B2K_TRY(b2k_knn_refine_launch(ctx, nullptr, 0, nullptr, nullptr, nq_all, k, Q, items, 0, d, row0, item_ids, cand, s));
  } else {
    tm.mark(4, s);
    std::vector<int32_t> pair_off_h((size_t)nlist + 2);
    std::vector<KnnUnit> units;
    for (int64_t q0 = 0; q0 < nq_all; q0 += nqc_max) {
      const int64_t nqc = std::min(nqc_max, nq_all - q0), P = nqc * nprobe;
      k_ivf_pairs<<<grid_for(ctx, P), 256, 0, s>>>(pidx + q0 * nprobe, P, nlist, pkeys, pvals);
      B2K_CUDA_OK(ctx, cudaGetLastError());
      B2K_CUDA_OK(ctx, cub::DeviceRadixSort::SortPairs(sort_tmp, sort_bytes, pkeys, pkeys_s, pvals, pvals_s, (int)P, 0,
                                                       pbits, s));
      k_ivf_offsets<<<grid_for(ctx, P + 1), 256, 0, s>>>(pkeys_s, P, nlist + 1, pair_off);
      B2K_CUDA_OK(ctx, cudaGetLastError());
      k_ivf_slots<<<grid_for(ctx, P), 256, 0, s>>>(pkeys_s, pvals_s, P, nlist, item_off, slots);
      B2K_CUDA_OK(ctx, cudaGetLastError());
      k_ivf_gather_q<<<grid_for(ctx, P * d), 256, 0, s>>>(Q + q0 * d, pvals_s, P, nprobe, d, wg ? items : nullptr, Qg);
      B2K_CUDA_OK(ctx, cudaGetLastError());
      ctx->stats.kernel_launches += 5;
      B2K_CUDA_OK(ctx, cudaMemcpyAsync(pair_off_h.data(), pair_off, pair_off_h.size() * 4, cudaMemcpyDeviceToHost, s));
      B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
      // one unit per (list, tile of its pairs), the longest index ranges first so that no SM is left with a long list
      // at the end of the pass
      units.clear();
      for (int l = 0; l < nlist; ++l) {
        const int ni = item_off_h[l + 1] - item_off_h[l];
        if (ni == 0) continue;
        for (int64_t t0 = pair_off_h[l]; t0 < pair_off_h[l + 1]; t0 += qt) {
          KnnUnit u;
          u.out0 = t0;
          u.row0 = (int)t0;
          u.nrows = (int)std::min<int64_t>(qt, pair_off_h[l + 1] - t0);
          u.lo = wg ? pos_off_h[l] / B2K_KNN_WG_BLOCK : pos_off_h[l];
          u.hi = wg ? (pos_off_h[l] + ni + B2K_KNN_WG_BLOCK - 1) / B2K_KNN_WG_BLOCK : pos_off_h[l] + ni;
          units.push_back(u);
        }
      }
      std::stable_sort(units.begin(), units.end(),
                       [](const KnnUnit& a, const KnnUnit& b) { return a.hi - a.lo > b.hi - b.lo; });
      if (!units.empty())
        B2K_CUDA_OK(ctx, cudaMemcpyAsync(units_dev, units.data(), units.size() * sizeof(KnnUnit),
                                         cudaMemcpyHostToDevice, s));
      B2K_TRY(cev.mark(ctx, tm.on, s));
      B2K_TRY(b2k_knn_scan_launch(ctx, wg, DP, Qg, P, items, perm, Xhi, Xlo, norms, n_pad, d, k, units_dev,
                                  (int)units.size(), part, s));
      B2K_TRY(cev.mark(ctx, tm.on, s));
      B2K_TRY(b2k_knn_refine_launch(ctx, part, nprobe, slots, perm, nqc, k, Q + q0 * d, items, n_items, d, row0,
                                    item_ids, cand + q0 * k, s));
    }
  }
  ctx->stats.last_path = wg ? B2K_PATH_FUSED : B2K_PATH_GENERIC;
  tm.mark(5, s);

  // ---- candidate allgather, merge of the own queries in rank order ----
  const KnnCand* all = cand;
  if (nr > 1) {
    B2K_TRY(b2k_comm_allgather_bytes(ctx, cand, cand_all, (size_t)nq_all * k * sizeof(KnnCand), s));
    all = cand_all;
  }
  tm.mark(6, s);
  B2K_TRY(b2k_knn_merge_launch(ctx, all, nr, nq_all, qown0, nq_local, k, metric == B2K_IVF_SQEUCLIDEAN, true,
                               dist_out, idx_out, s));
  tm.mark(7, s);
  if (tm.on) {
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
    const double scan = cev.scan_ms();
    ctx->stats.last_finalize_ms = tm.ms(1, 2);                            // build: subset, Lloyd, assign, sort, prep
    ctx->stats.last_probe_ms = tm.ms(2, 3);                               // probe selection
    ctx->stats.last_fused_ms = scan;                                      // scan passes
    ctx->stats.last_reduce_ms = tm.ms(4, 5) - scan + tm.ms(6, 7);         // pairs, gather, refine + merge
    ctx->stats.last_allreduce_ms = tm.ms(0, 1) + tm.ms(5, 6);             // query and candidate all-gathers
    ctx->stats.last_loop_ms = tm.ms(0, 7);
  }
  return B2K_OK;
}
