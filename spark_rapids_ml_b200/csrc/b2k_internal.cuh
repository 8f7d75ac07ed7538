// Internal declarations shared by the translation units of libb2kmeans.so (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <functional>
#include <memory>
#include <string>
#include <vector>

#include "../../include/b2kmeans.h"

// ------------------------------------------------------------------------------------------------
// Device-resident loop state: lets the host enqueue several Lloyd iterations without a D2H sync —
// every hot-loop kernel returns immediately once `done` is set (SURVEY.md §7 step 4).
// ------------------------------------------------------------------------------------------------
struct B2kLoopState {
  int iter;                  // completed iterations
  int done;                  // 1 once shift < tol (or iter == max_iter)
  int max_iter;
  unsigned int blocks_done;  // last-block-done counter of the finalize kernel
  double tol;
  double shift;              // last sum_j ||dc_j||^2
  double cost;               // last sum_i min_j ||x_i - c_j||^2 (w.r.t. the centers of that pass)
  // large-shape kernel: deferred (exactly re-decided) rows / candidate distances evaluated, cumulative over the call
  // (written by k_fix_accum_t; the host's convergence poll reads them to choose the path of the next burst)
  unsigned long long fix_rows_cum;
  unsigned long long fix_cands_cum;
};

// Layout of the reduced buffer R (doubles) that crosses NCCL: [k*d sums | k counts | 1 cost].
static inline size_t b2k_reduced_len(int k, int d) { return (size_t)k * d + k + 1; }

struct B2kNccl;  // opaque (b2k_comm.cu)

struct b2k_ctx {
  int device = 0;
  int sm_count = 0;
  size_t smem_optin = 0;
  std::string err;
  // options
  int kernel_path = B2K_PATH_AUTO;
  int time_kernels = 0;
  int check_every = 4;
  int grid_limit = 0;
  int adaptive_path = 1;         // option "adaptive_path": a Lloyd loop on the large-shape kernel falls back to the generic
                                 // kernels for its remaining iterations when most rows need the exact fix-up
  int lloyd_switched = 0;        // the last lloyd_impl call did so (the fit's inertia pass follows it)
  int near_tie_hint = 0;         // set around the k-means|| candidate passes: prefer exact 128-centre chunks (d <= 128)
  int force_variant_t = 0;       // option "variant_t": route every supported shape through b2k_fused_t.cu (tests)
  int collect_recheck = 0;       // option "collect_recheck": fill stats.recheck_* (costs a stream sync per call)
  int profile_fused = 0;         // record per-role blocked-cycle counters of the fused kernel
  // Row norms of the large-shape kernel, shared by every pass of ONE b2k_kmeans_fit call (k-means|| candidate passes,
  // the Lloyd loop, the inertia pass all see the same immutable X): computed by the first pass, reused by the rest.
  const float* xnorm_scope_X = nullptr;   // non-null only inside b2k_kmeans_fit
  int64_t xnorm_scope_n = 0;
  int xnorm_scope_d = 0;
  void* xnorm_cache = nullptr;            // float2 [xnorm_cache_rows]
  int64_t xnorm_cache_rows = 0;
  int xnorm_cache_valid = 0;
  long long* prof_dev = nullptr;  // [grid][12 warps][8] phase cycle counters (option profile_fused)
  int prof_grid = 0;
  // comm
  B2kNccl* nccl = nullptr;
  int nranks = 1;
  int rank = 0;
  // scratch (device), grown on demand
  void* scratch = nullptr;
  size_t scratch_bytes = 0;
  // pinned staging for ingest (host) + device staging
  void* pinned[2] = {nullptr, nullptr};
  size_t pinned_bytes = 0;
  void* dev_stage[2] = {nullptr, nullptr};
  size_t dev_stage_bytes = 0;
  cudaEvent_t stage_evt[2] = {nullptr, nullptr};
  int stage_next = 0;
  void* copy_pool = nullptr;     // B2kCopyPool (b2k_ingest.cu): helper threads of the pageable -> pinned staging copy
  int ingest_threads = 0;        // option "ingest_threads": threads of that copy (0 = default 4, capped by the CPU quota)
  // pinned host mirror of the loop state (convergence polls)
  B2kLoopState* h_state = nullptr;
  // TMA descriptor encoder (driver entry point, resolved lazily)
  void* encode_tiled = nullptr;
  // random forests (b2k_rf.cu): the forest of the last b2k_rf_fit, read by b2k_rf_forest; test switches
  std::shared_ptr<void> rf_forest;
  int rf_group_nodes = 0;   // option "rf_group_nodes": cap on the nodes of one histogram pass (0 = capacity)
  int rf_flush_tiles = 0;   // option "rf_flush_tiles": tiles per CTA between flushes of the cluster pass (0 = the bound)
  // UMAP (b2k_umap.cu): the graph of the last b2k_umap_fit, read by b2k_umap_graph; option "stop_after_epochs" (tests)
  std::shared_ptr<void> umap_graph;
  int umap_stop_epochs = 0;
  b2k_stats stats{};
};

// The library's counter-based generator (host and device): Gaussian mixtures draw their start rows from it, bisecting
// k-means its split starts, ALS its start factors.
__host__ __device__ inline uint64_t b2k_splitmix64(uint64_t z) {
  z += 0x9e3779b97f4a7c15ull;
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}

// ------------------------------------------------------------------------------------------------
// error helpers
// ------------------------------------------------------------------------------------------------
int b2k_fail(b2k_ctx* ctx, int code, const std::string& msg);
#define B2K_CUDA_OK(ctx, expr)                                                             \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess)                                                                 \
      return b2k_fail((ctx), B2K_ERR_CUDA,                                                 \
                      std::string(#expr) + ": " + cudaGetErrorName(_e) + ": " +            \
                          cudaGetErrorString(_e));                                         \
  } while (0)
#define B2K_TRY(expr)            \
  do {                           \
    int _s = (expr);             \
    if (_s != B2K_OK) return _s; \
  } while (0)

int b2k_scratch_reserve(b2k_ctx* ctx, size_t bytes);
void b2k_copy_pool_destroy(b2k_ctx* ctx);

// Scratch layout: a bump allocator over a device region {base, cap}.  A driver states its takes once and runs them twice:
// with no base to measure (`off` is then the bytes they need), then over the region to place its arrays.  Offsets are
// aligned relative to base: ctx->scratch comes from cudaMalloc (256 B), a nested region starts at a 1 KB boundary.
struct B2kLayout {
  char* base = nullptr;   // nullptr: measure only, no pointer is formed
  size_t cap = 0, off = 0;
  explicit B2kLayout(void* b = nullptr, size_t c = 0) : base(static_cast<char*>(b)), cap(c) {}
  template <typename T>
  T* take(size_t count, size_t align = 256) {
    off = (off + align - 1) / align * align;
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += count * sizeof(T);
    return p;
  }
  // the unused tail from the next `align` boundary on, as the region of a nested call that measured `need` bytes
  B2kLayout tail(size_t need, size_t align = 1024) {
    char* p = take<char>(need, align);
    const size_t start = off - need;
    return base ? B2kLayout(p, start < cap ? cap - start : 0) : B2kLayout();
  }
  int check(b2k_ctx* ctx, const char* who) const {   // after placing: every take stayed inside the region
    if (off <= cap) return B2K_OK;
    return b2k_fail(ctx, B2K_ERR_STATE, std::string(who) + ": scratch layout of " + std::to_string(off) +
                                            " bytes overruns its region of " + std::to_string(cap));
  }
};

// Device buffers owned by one call that outlive the scratch layouts of the calls it makes (stream-ordered allocation).
struct DevBuf {
  void* p = nullptr;
  cudaStream_t s = nullptr;
  ~DevBuf() {
    if (p) cudaFreeAsync(p, s);
  }
};
template <typename T>
int dalloc(b2k_ctx* ctx, DevBuf& b, size_t count, cudaStream_t s, T** out) {
  if (b.p) {
    B2K_CUDA_OK(ctx, cudaFreeAsync(b.p, s));
    b.p = nullptr;
  }
  b.s = s;
  B2K_CUDA_OK(ctx, cudaMallocAsync(&b.p, (count > 0 ? count : 1) * sizeof(T), s));
  *out = static_cast<T*>(b.p);
  return B2K_OK;
}

// Runs `layout` (int(B2kLayout&)) to measure, grows ctx->scratch to that size, then runs it over the scratch to place.
template <typename F>
int b2k_scratch_layout(b2k_ctx* ctx, const char* who, F&& layout) {
  B2kLayout measure;
  B2K_TRY(layout(measure));
  B2K_TRY(b2k_scratch_reserve(ctx, measure.off));
  B2kLayout place(ctx->scratch, ctx->scratch_bytes);
  B2K_TRY(layout(place));
  return place.check(ctx, who);
}

// ------------------------------------------------------------------------------------------------
// generic (any k, d) kernels — b2k_generic.cu
// ------------------------------------------------------------------------------------------------
// cnorm[j] = ||c_j||^2 (fp32 from a double accumulation)
int b2k_launch_center_norms(b2k_ctx* ctx, const float* C, int k, int d, float* cnorm,
                            const B2kLoopState* st, cudaStream_t s);
// labels/mindist (either may be NULL) + optional per-CTA cost partials
int b2k_launch_assign_generic(b2k_ctx* ctx, const float* X, int64_t n, int d, const float* C,
                              const float* cnorm, int k, int32_t* labels, float* mindist,
                              const B2kLoopState* st, cudaStream_t s);
// per-cluster partial sums from labels: partials [P][k*d] f32, counts [P][k] i32; returns P, the partial slots.
int b2k_update_generic_slots(b2k_ctx* ctx, int64_t n, int d, int k);
int b2k_launch_update_generic(b2k_ctx* ctx, const float* X, int64_t n, int d, const int32_t* labels, int k,
                              int P, float* partials, int32_t* counts, const B2kLoopState* st,
                              cudaStream_t s);
// R[k*d+k+1] (double) = fixed-order sum over P partials (+ cost from mindist partial sums)
int b2k_launch_reduce_partials(b2k_ctx* ctx, const float* partials, const int32_t* counts,
                               const double* cost_partials, int P, int Pc, int k, int d, double* R,
                               const B2kLoopState* st, cudaStream_t s);
// C <- R.S / R.w (w == 0 keeps C), shift, iter++, done.  shift_scratch: k doubles.
int b2k_launch_finalize(b2k_ctx* ctx, const double* R, float* C, int k, int d, double* shift_scratch,
                        B2kLoopState* st, cudaStream_t s);
// cost partials: sum of mindist over fixed-size row blocks (deterministic two-level)
int b2k_launch_sum_f32_to_f64(b2k_ctx* ctx, const float* v, int64_t n, double* out /*1*/,
                              double* block_scratch, int nblocks, cudaStream_t s);
int b2k_launch_fold_f64(b2k_ctx* ctx, const double* in, int m, double* out /*1*/, cudaStream_t s);
// The row spans of the fp64 column passes (per-span partials, folded in span order): with ncb column blocks per span,
// spans = min(max(1, ceil(8 SMs / ncb)), max(1, ceil(n / 64))) and span_rows = max(1, ceil(n / spans)).  A function of
// (n, ncb) and the device alone, so every call on the same shape adds in the same order.
struct B2kRowSpans {
  int spans;
  int64_t span_rows;
};
B2kRowSpans b2k_row_spans(const b2k_ctx* ctx, int64_t n, int ncb);
// out[c] = sum over s = 0 .. spans - 1 of part[s m + c], in span order from 0.0 (c < m); with n_tail >= 0 also
// out[m] = n_tail (a row count that an allreduce then turns into the global one)
int b2k_launch_fold_spans(b2k_ctx* ctx, const double* part, int spans, int m, double* out, cudaStream_t s,
                          int64_t n_tail = -1);
// out [m] (fp64) = the rows of labels [n] with each label value 0 .. m - 1, per row span of b2k_row_spans(n, 1) into
// part [spans][m], folded in span order
int b2k_launch_label_counts(b2k_ctx* ctx, const int32_t* labels, int64_t n, int m, double* part, double* out,
                            cudaStream_t s);
int b2k_launch_gather_rows(b2k_ctx* ctx, const float* X, int d, const int64_t* rows_local, int m,
                           float* out, int64_t out_row0, cudaStream_t s);
// chunked assign: md_acc/lab_acc <- (md, lab + base) where md < md_acc
int b2k_launch_merge_chunk(b2k_ctx* ctx, float* md_acc, int32_t* lab_acc, const float* md, const int32_t* lab, int base,
                           int64_t n, const B2kLoopState* st, cudaStream_t s);
// k-means|| helpers
int b2k_launch_bernoulli_pick(b2k_ctx* ctx, const float* mind, int64_t n, int64_t row_offset,
                              double scale /* l/phi */, uint64_t seed, int round, int64_t* picked,
                              int* n_picked, int cap, cudaStream_t s);
int b2k_launch_histogram(b2k_ctx* ctx, const int32_t* labels, int64_t n, int m, double* hist,
                         cudaStream_t s);
int b2k_launch_weighted_update(b2k_ctx* ctx, const float* P, const double* w, const int32_t* lab, int M, int d, int k,
                               float* C, cudaStream_t s);
int b2k_launch_pairwise_sqdist(b2k_ctx* ctx, const float* P, int M, int d, float* D2, cudaStream_t s);

// ------------------------------------------------------------------------------------------------
// wgmma fused assign kernel (b2k_wg.cuh) in two families:
//   variant 0 — b2k_fused_tc.cu: k <= 128, d <= 128 (its compiled instantiations), 3xTF32
//   variant 1 — b2k_fused_t.cu:  k, d <= 256, 1xTF32 screening + exact fix-up of the near-tie rows
// b2k_fused.cu holds what does not depend on the family: the shape rules, the plan, dispatch and the TMA encoder.
// ------------------------------------------------------------------------------------------------
constexpr int B2K_FUSED_TILE_ROWS = 128;   // X rows per tile of the fused kernel (WG_TM)

struct B2kFusedPlan {
  int KP = 0, DP = 0;        // padded cluster count / dimension of the instantiation
  int grid = 0;              // persistent CTAs (variant 1: whole clusters of WG_CL CTAs)
  int variant = 0;           // family, see above
  int P = 0;                 // partial-sum slots a Lloyd pass writes (variant 0: one per CTA; 1: one per cluster + fix-up)
  int Pc = 0;                // cost partials the pass writes (variant 0: grid; variant 1: grid + fix-up CTAs)
  size_t scratch_bytes = 0;  // centre operands/cnorm + partials/counts/cost (+ row norms, fix-up list, variant 1)
  // byte offsets into the plan scratch of what a pass leaves for its caller
  size_t off_partials = 0;   // f32 [P][k][d]
  size_t off_counts = 0;     // i32 [P][k]
  size_t off_cost = 0;       // f64 [Pc]
  size_t off_rstat = 0;      // variant 1: u64 {rows re-decided exactly, candidate distances} since b2k_fused_prepare
  float* partials(void* ps) const { return reinterpret_cast<float*>(static_cast<char*>(ps) + off_partials); }
  int32_t* counts(void* ps) const { return reinterpret_cast<int32_t*>(static_cast<char*>(ps) + off_counts); }
  double* cost_partials(void* ps) const { return reinterpret_cast<double*>(static_cast<char*>(ps) + off_cost); }
  unsigned long long* rstat(void* ps) const {
    return variant == 1 ? reinterpret_cast<unsigned long long*>(static_cast<char*>(ps) + off_rstat) : nullptr;
  }
};
bool b2k_fused_supported(int64_t n, int d, int k, const float* X);
int b2k_fused_plan(b2k_ctx* ctx, int64_t n, int d, int k, B2kFusedPlan* plan);
// Once per fit / lloyd / assign call, before the first b2k_launch_fused on this X (variant 1: row norms; variant 0: no-op)
int b2k_fused_prepare(b2k_ctx* ctx, const B2kFusedPlan& plan, void* plan_scratch, const float* X, int64_t n, int d, int k,
                      cudaStream_t s);
// One fused pass: labels_out and mindist_out (either may be NULL) + partial sums/counts/cost into the plan scratch.
// `do_update` = accumulate partial sums (Lloyd iteration, no min distances) or not (assign/inertia pass); `need_cost` =
// the caller reads the cost partials of an assign pass (variant 0 forms them on every assign pass).
int b2k_launch_fused(b2k_ctx* ctx, const B2kFusedPlan& plan, void* plan_scratch, const float* X, int64_t n, int d,
                     const float* C, int k, int32_t* labels_out, float* mindist_out, bool do_update, bool need_cost,
                     const B2kLoopState* st, cudaStream_t s);
int b2k_encode_2d(b2k_ctx* ctx, CUtensorMap* map, const void* base, uint64_t inner, uint64_t outer,
                  uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer, CUtensorMapL2promotion l2);

// the families (called by b2k_fused.cu only).  *_plan fill the rest of a plan whose grid b2k_fused_plan has set
// (variant 1 rounds it down to whole clusters).
bool b2k_fused_tc_plan(int64_t n, int d, int k, B2kFusedPlan* plan);   // false: no instantiation for (k, d)
int b2k_launch_fused_tc(b2k_ctx* ctx, const B2kFusedPlan& plan, void* plan_scratch, const float* X, int64_t n, int d,
                        const float* C, int k, int32_t* labels_out, float* mindist_out, bool do_update,
                        const B2kLoopState* st, cudaStream_t s);
void b2k_fused_t_plan(const b2k_ctx* ctx, int64_t n, int d, int k, B2kFusedPlan* plan);
int b2k_fused_t_prepare(b2k_ctx* ctx, const B2kFusedPlan& plan, void* plan_scratch, const float* X, int64_t n, int d,
                        int k, cudaStream_t s);
int b2k_launch_fused_t(b2k_ctx* ctx, const B2kFusedPlan& plan, void* plan_scratch, const float* X, int64_t n, int d,
                       const float* C, int k, int32_t* labels_out, float* mindist_out, bool do_update, bool need_cost,
                       const B2kLoopState* st, cudaStream_t s);

// ------------------------------------------------------------------------------------------------
// comm — b2k_comm.cu
// ------------------------------------------------------------------------------------------------
int b2k_comm_allreduce_f64(b2k_ctx* ctx, double* buf, size_t count, cudaStream_t s);
int b2k_comm_allgather_i64(b2k_ctx* ctx, const int64_t* send_dev, int64_t* recv_dev, size_t count_per_rank,
                           cudaStream_t s);
int b2k_comm_allreduce_f32(b2k_ctx* ctx, float* buf, size_t count, cudaStream_t s);
// exact integer sums (the random-forest histograms): every rank gets the same bits whatever the reduction order
int b2k_comm_allreduce_i64(b2k_ctx* ctx, int64_t* buf, size_t count, cudaStream_t s);
// recv [nranks][bytes_per_rank] <- every rank's send; send may be recv's own slot (in place).  One rank: a copy.
int b2k_comm_allgather_bytes(b2k_ctx* ctx, const void* send_dev, void* recv_dev, size_t bytes_per_rank, cudaStream_t s);

// ingest — b2k_ingest.cu (entry point is the C ABI itself)

// ------------------------------------------------------------------------------------------------
// PCA — b2k_pca.cu (the C ABI entry points in b2k_api.cu check their arguments and the partitions, then call these)
// ------------------------------------------------------------------------------------------------
constexpr int B2K_PCA_MAX_D = 1024;   // both Gram paths, the projection kernel and the host eigen step
// The passes PCA and linear regression share (collective): column sums, then the Gram matrix of X centred on the fp32
// means mu32 = fl32(mu), on the path kernel_path selects.  With a label y [n] (else NULL), also the label's sum and, by
// k_xty (b2k_linreg.cu), sum (x - mu32) (y - muy32) and sum (y - muy32)^2.  The offsets are left for the caller to
// remove exactly with delta.  Fails with B2K_ERR_INVALID, on every rank alike, when fewer than min_rows rows exist.
struct B2kMoments {
  int64_t n_total = 0;
  std::vector<double> mu;      // [d] (+ [1] label) means, fp64
  std::vector<double> delta;   // mu - fl32(mu)
  std::vector<double> G;       // [d][d] Gram about mu32 (+ [d] X^T y, [1] y^T y about (mu32, muy32)), allreduced
};
int b2k_moments_impl(b2k_ctx* ctx, const char* who, const float* X, const float* y, int64_t n, int d, int64_t min_rows,
                     B2kMoments* m, cudaStream_t s);
// Symmetric eigendecomposition (Householder + implicit QL): A = Z^T diag(w) Z, rows of Z the eigenvectors; A is
// destroyed.  False if an eigenvalue needs more than 60 QL sweeps.
bool b2k_sym_eig(std::vector<double>& A, int n, std::vector<double>& w, std::vector<double>& Z);
int b2k_pca_fit_impl(b2k_ctx* ctx, const float* X, int64_t n, int d, int k, double* mean_out, double* components_out,
                     double* evr_out, double* sv_out, cudaStream_t s);
// ctx may be NULL (b2k_pca_finalize): errors then go to b2k_last_error(NULL)
int b2k_pca_finalize_impl(b2k_ctx* ctx, const double* cov, int d, int64_t n_total, int k, double* components_out,
                          double* evr_out, double* sv_out);
int b2k_pca_transform_impl(b2k_ctx* ctx, const float* X, int64_t n, int d, const float* C, int k, float* Y,
                           cudaStream_t s);
// G [d (d + 1) / 2] (device, the packed upper triangle of b2k_gram.cu) = X^T X in fp64 over this rank's rows only (no
// collective): the generic Gram pass with a zero mean, its row spans a function of (n, d) alone.  Uses ctx->scratch.
int b2k_gram_local_impl(b2k_ctx* ctx, const float* X, int64_t n, int d, double* G, cudaStream_t s);

// ------------------------------------------------------------------------------------------------
// Gram passes — b2k_gram.cu: G_c = sum_rows f_c r_rc (x - mu_c)(x - mu_c)^T in fp64 for k components, as packed upper
// triangles [k][d (d + 1) / 2] (row-major, i <= j).  Unweighted (r NULL, k = 1): x - mu in fp32; weighted (r [n][k],
// f [k] fp64, mu_c the component's own centre): x - mu_c in fp64 (generic) or rounded once to fp32 and scaled by
// fl32(sqrt(f_c r)) (wgmma).
// ------------------------------------------------------------------------------------------------
bool b2k_gram_wg_ok(const float* X, int d);   // the wgmma pass takes the shape: d % 4 == 0, X 16-byte aligned
struct B2kGramPlan {
  bool wg = false;      // the wgmma pass (else the generic one)
  int64_t n = 0;
  int d = 0, k = 1;
  int grid = 0;         // wgmma: CTAs; generic: CTAs per row span (tiles x k)
  int spans = 0;        // wgmma: CTAs per (component, tile); generic: row spans
  size_t part_len = 0;  // fp64 partials
  size_t mu_len = 0;    // fp32 centres the pass reads, k of them at a stride of mu_len / k (zero past d)
  size_t out_len = 0;   // k d (d + 1) / 2
};
// the pass for (n, d, k): wgmma when allow_wg and b2k_gram_wg_ok; the generic row spans keep their partials within
// part_bytes (at most 64 spans), so that they depend on (n, d, k) alone
B2kGramPlan b2k_gram_plan(const b2k_ctx* ctx, const float* X, int64_t n, int d, int k, bool allow_wg, size_t part_bytes);
// the pass and its fold into tri [out_len]; mu [mu_len], part [part_len], r [n][k] and r_scale [k] (both NULL for the
// unweighted pass).  n == 0: zero partials, folded.  Counts no launches: the callers keep their own stats.
int b2k_gram_launch(b2k_ctx* ctx, const B2kGramPlan& p, const float* X, const float* mu, const double* r,
                    const double* r_scale, double* part, double* tri, cudaStream_t s);
// G [d][d] (device) <- one packed upper triangle, mirrored; counts no launch
int b2k_launch_gram_unpack(b2k_ctx* ctx, const double* tri, int d, double* G, cudaStream_t s);

// ------------------------------------------------------------------------------------------------
// exact k-NN — b2k_knn.cu (the C ABI entry point in b2k_api.cu checks its arguments, then calls this)
// ------------------------------------------------------------------------------------------------
constexpr int B2K_KNN_MAX_K = 1024;   // the generic path's per-query lists; the wgmma path takes k <= 64
int b2k_knn_search_impl(b2k_ctx* ctx, const float* items, int64_t n_items, const int64_t* item_ids,
                        const float* queries, int64_t nq_local, int d, int k, float* dist_out, int64_t* idx_out,
                        cudaStream_t s);
// The same search on one rank with no collective (UMAP's graph and transform): the k nearest of items [n_items, d] for
// each of queries [nq, d] -> sqrt(distance) ascending, ties to the lower row, and the item row.  1 <= k <= n_items.
int b2k_knn_local_impl(b2k_ctx* ctx, const float* items, int64_t n_items, const float* queries, int64_t nq, int d,
                       int k, float* dist_out, int64_t* idx_out, cudaStream_t s);

// The passes of the search that IVF-Flat (b2k_ivf.cu) runs on its own index layout.
constexpr int B2K_KNN_WG_QROWS = 128;   // query rows of a wgmma unit
constexpr int B2K_KNN_WG_BLOCK = 128;   // index rows per block of the wgmma pass (a unit's index range is in blocks)
constexpr int B2K_KNN_GEN_QROWS = 16;   // query rows of a generic unit (its index range is in item rows)
constexpr int B2K_KNN_MAX_LISTS = 256;  // partial lists one refine merges per query
// one candidate of the refined lists that cross NCCL (16 bytes)
struct KnnCand {
  float d;        // exact squared distance, +inf for padding
  int32_t grow;   // global row, INT32_MAX for padding
  int64_t id;     // the user's item id (global row when no ids are given), -1 for padding
};
// One work unit of a search pass: query rows [row0, row0 + nrows) against the index range [lo, hi); row r of the unit
// writes its k best (screen distance bits, index row) to part[out0 + r][k].
struct KnnUnit {
  int64_t out0;
  int row0, nrows;
  int lo, hi;
};
// true when the wgmma pair-distance pipeline (b2k_pair_wg.cuh: k-NN, IVF-Flat, DBSCAN) takes the width (d % 4 == 0,
// 4 <= d <= 128); true when the k-NN wgmma pass takes the shape (that width and k <= 64); the padded width DP they use
bool b2k_knn_wg_width(int d);
bool b2k_knn_wg_shape(int d, int k);
int b2k_knn_wg_dp(int d);
// index planes of x - s for the wgmma pass, s = X row 0: row p of the planes is X row perm[p] (perm NULL: p < n), or
// padding (zeros, +inf norm) where perm[p] < 0 / p >= n
int b2k_knn_prep_launch(b2k_ctx* ctx, const float* X, int64_t n, int d, const int32_t* perm, int64_t n_pad, int DP,
                        float* Xhi, float* Xlo, float* norms, cudaStream_t s);
// Qs = Q - s [nq][d] for the wgmma pass, s = X row 0 as above; d % 4 == 0, Q and Qs 16-byte aligned
int b2k_knn_shift_launch(b2k_ctx* ctx, const float* Q, int64_t nq, int d, const float* X, float* Qs, cudaStream_t s);
// one search pass over a unit table (device, nunits entries).  wgmma: Q = shifted queries [nq][d] (16-byte aligned),
// the planes and norms of b2k_knn_prep_launch; generic: Q unshifted, item row r of the index is X row xperm[r] (xperm
// NULL: r)
int b2k_knn_scan_launch(b2k_ctx* ctx, bool wg, int DP, const float* Q, int64_t nq, const float* X, const int32_t* xperm,
                        const float* Xhi, const float* Xlo, const float* norms, int64_t n_pad, int d, int k,
                        const KnnUnit* units, int nunits, int2* part, cudaStream_t s);
// refine: per query row of Q [nq][d], merge its nl partial lists (list l at part row slots[q * nl + l], -1 = none; slots
// NULL: l * nq + q), map index rows through perm (NULL: identity) to local item rows, recompute exact fp32 distances
// against X and sort by (distance, global row) -> cand [nq][k]
int b2k_knn_refine_launch(b2k_ctx* ctx, const int2* part, int nl, const int32_t* slots, const int32_t* perm, int64_t nq,
                          int k, const float* Q, const float* X, int64_t n_items, int d, int64_t row0,
                          const int64_t* ids, KnnCand* cand, cudaStream_t s);
// merge of own queries [q0, q0 + nq_own) over nranks candidate lists -> distances (sqrt, or squared) and ids; fill: past
// the found items the id is the first entry's id, or INT64_MAX when nothing was found
int b2k_knn_merge_launch(b2k_ctx* ctx, const KnnCand* all, int nranks, int64_t nq_all, int64_t q0, int64_t nq_own, int k,
                         bool squared, bool fill, float* dist_out, int64_t* idx_out, cudaStream_t s);

struct B2kTimer {   // CUDA events around the device phases when option time_kernels is set
  cudaEvent_t ev[12] = {};
  bool on = false;
  explicit B2kTimer(bool enable) : on(enable) {
    if (on)
      for (auto& e : ev) cudaEventCreate(&e);
  }
  ~B2kTimer() {
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

// ------------------------------------------------------------------------------------------------
// silhouette — b2k_silhouette.cu (the C ABI entry points in b2k_api.cu check their arguments, then call this with
// one model or several; on an error of one model's ids or statistics, *failed_model (if not NULL) = that model)
// ------------------------------------------------------------------------------------------------
int b2k_silhouette_impl(b2k_ctx* ctx, const float* X, int64_t n_local, int d, int n_models, const int64_t* const* ids,
                        int metric, double* out, int* failed_model, cudaStream_t s);

// ------------------------------------------------------------------------------------------------
// approximate k-NN (IVF-Flat) — b2k_ivf.cu (the C ABI entry point in b2k_api.cu checks its arguments, then calls this)
// ------------------------------------------------------------------------------------------------
int b2k_ivf_search_impl(b2k_ctx* ctx, const float* items, int64_t n_items, const int64_t* item_ids,
                        const float* queries, int64_t nq_local, int d, int k, int nlist, int nprobe, int n_iters,
                        double train_fraction, int metric, int train, float* centers, int32_t* item_list_out,
                        int32_t* probe_out, float* dist_out, int64_t* idx_out, cudaStream_t s);

// ------------------------------------------------------------------------------------------------
// UMAP — b2k_umap.cu (the C ABI entry points in b2k_api.cu check their arguments, then call these)
// ------------------------------------------------------------------------------------------------
int b2k_umap_fit_impl(b2k_ctx* ctx, const float* X, int64_t n, int d, const int32_t* labels,
                      const b2k_umap_params& p, float* embedding_out, double* info_out, cudaStream_t s);
int b2k_umap_transform_impl(b2k_ctx* ctx, const float* X_train, const float* Y_train, int64_t n_train, int d,
                            const float* Q, int64_t nq, const b2k_umap_params& p, float* out, cudaStream_t s);
int b2k_umap_graph_impl(b2k_ctx* ctx, int64_t* knn_idx, float* knn_dist, double* rho, double* sigma, int64_t* indptr,
                        int32_t* indices, double* weights, double* eps, float* init, double* ritz_values,
                        double* ritz_vectors);

// ------------------------------------------------------------------------------------------------
// DBSCAN — b2k_dbscan.cu (the C ABI entry point in b2k_api.cu checks its arguments, then calls this)
// ------------------------------------------------------------------------------------------------
int b2k_dbscan_fit_impl(b2k_ctx* ctx, const float* X, int64_t n_local, int d, double eps, int min_samples, int metric,
                        int32_t* labels_out, uint8_t* core_out, int64_t* n_clusters_out, cudaStream_t s);

// ------------------------------------------------------------------------------------------------
// random forests — b2k_rf.cu (the C ABI entry points in b2k_api.cu check their arguments, then call these)
// ------------------------------------------------------------------------------------------------
int b2k_rf_fit_impl(b2k_ctx* ctx, const float* X, const float* y, int64_t n_local, int d, const b2k_rf_params& p,
                    int* n_values_out, int64_t* n_nodes_out, double* level_ms_out, int64_t* level_updates_out,
                    cudaStream_t s);
int b2k_rf_forest_impl(b2k_ctx* ctx, int64_t* tree_offsets_out, int32_t* feature_out, float* threshold_out,
                       int32_t* children_out, double* gain_out, int64_t* count_out, double* value_out);
int b2k_rf_predict_impl(b2k_ctx* ctx, const float* X, int64_t n, int d, int n_trees, const int64_t* tree_offsets,
                        const int32_t* feature, const float* threshold, const int32_t* children, const double* value,
                        int n_values, int classification, double* raw_out, double* prob_out, double* pred_out,
                        cudaStream_t s);

// ------------------------------------------------------------------------------------------------
// linear regression — b2k_linreg.cu (the C ABI entry points in b2k_api.cu check their arguments, then call these)
// ------------------------------------------------------------------------------------------------
constexpr int B2K_LINREG_MAX_D = B2K_PCA_MAX_D;   // the moments ride on PCA's Gram passes
// row spans of k_xty's fp64 partials for (n, d): the caller lays out spans * (d + 1) doubles for b2k_launch_xty
int b2k_xty_spans(const b2k_ctx* ctx, int64_t n, int d);
// out [d + 1] = [sum (x - mu32) (y - muy32) | sum (y - muy32)^2], fp64, folded over the spans in order
int b2k_launch_xty(b2k_ctx* ctx, const float* X, const float* y, int64_t n, int d, const float* mu32, float muy32,
                   int spans, double* part, double* out, cudaStream_t s);
int b2k_linreg_moments_impl(b2k_ctx* ctx, const float* X, const float* y, int64_t n, int d, int64_t* n_total_out,
                            double* mean_out, double* moments_out, cudaStream_t s);
int b2k_linreg_solve_impl(const double* mean, const double* moments, int d, int64_t n_total, double reg,
                          double l1_ratio, int fit_intercept, int standardization, int max_iter, double tol,
                          double* coef_out, double* intercept_out, int* n_iter_out);
int b2k_linreg_predict_impl(b2k_ctx* ctx, const float* X, int64_t n, int d, const double* coef, double intercept,
                            double* out, cudaStream_t s);

// ------------------------------------------------------------------------------------------------
// logistic regression — b2k_logreg.cu (the C ABI entry points in b2k_api.cu check their arguments, then call these)
// ------------------------------------------------------------------------------------------------
constexpr int B2K_LOGREG_MAX_D = B2K_PCA_MAX_D;
constexpr int B2K_LOGREG_MAX_CLASSES = 1024;   // label values in [0, 1024): the label pass counts each value
// Column moments (b2k_pca.cu, collective): *n_total, mu [d] = fp64 means, ssq [d] = sum (x - mu)^2, from column sums
// and a pass of squares centred on mu32 = fl32(mu) with the offset removed exactly.  Two f64 allreduces.
int b2k_colstats_impl(b2k_ctx* ctx, const char* who, const float* X, int64_t n, int d, int64_t* n_total,
                      std::vector<double>* mu, std::vector<double>* ssq, cudaStream_t s);
int b2k_logreg_labels_impl(b2k_ctx* ctx, const float* y, int64_t n, double* classes_out, int64_t* counts_out,
                           int* n_classes_out, int64_t* n_total_out, cudaStream_t s);
int b2k_logreg_eval_impl(b2k_ctx* ctx, const float* X, const float* y, int64_t n, int d, const double* classes,
                         int n_classes, int kp, const double* W, const double* b, double* loss_out, double* grad_out,
                         int64_t* n_total_out, cudaStream_t s);
// f_hist (may be NULL): F at the start and at each accepted iterate
int b2k_logreg_minimize_impl(b2k_logreg_objective fn, void* user, int n, double* x_io, const double* l1, int max_iter,
                             double tol, int* n_iter_out, int* n_eval_out, double* f_out,
                             std::vector<double>* f_hist = nullptr);
int b2k_logreg_fit_impl(b2k_ctx* ctx, const float* X, const float* y, int64_t n, int d, const double* classes,
                        const int64_t* counts, int n_classes, int n_fits, const b2k_logreg_params* prm,
                        double* coef_out, double* intercept_out, int* kp_out, int* n_iter_out, cudaStream_t s);
int b2k_logreg_predict_impl(b2k_ctx* ctx, const float* X, int64_t n, int d, int kp, const double* W, const double* b,
                            const double* class_values, double* raw_out, double* prob_out, double* pred_out,
                            cudaStream_t s);
// The parts of a fit that do not depend on the data layout, shared by the dense and the CSR fits.  An evaluation at
// (W [kp][d], b [kp]) returns out [kp (d + 1) + 2] = allreduced [sum r x | sum r per class (at k (d + 1) + d) | sum loss
// | n], the layout of b2k_logreg_eval's pass.
using B2kLogregEval = std::function<int(int kp, const double* W, const double* b, double* out)>;
int b2k_logreg_check_params(b2k_ctx* ctx, int n_classes, int n_fits, const b2k_logreg_params* prm);
std::vector<int> b2k_logreg_class_map(const double* classes, int n_classes);
// Per setting: the solver frame, penalty weights, prior log-odds start, L-BFGS / OWL-QN through `eval`, W = V / sigma and
// MLlib's centring; ssq [d] = the global sum of (x - mu)^2 per feature over n_total rows.
int b2k_logreg_fit_settings(b2k_ctx* ctx, int d, int64_t n_total, const std::vector<double>& ssq, const double* classes,
                            const int64_t* counts, int n_classes, int n_fits, const b2k_logreg_params* prm,
                            const B2kLogregEval& eval, double* coef_out, double* intercept_out, int* kp_out,
                            int* n_iter_out);

// sparse logistic regression — b2k_logreg_sparse.cu.  A rank's rows in CSR: indptr [n + 1] int64 (indptr[0] = 0), indices
// [nnz] int32, values [nnz] f32.
constexpr int64_t B2K_LOGREG_CSR_MAX_PARAMS = (int64_t)1 << 25;   // cap on kp (d + 1): the host L-BFGS state
constexpr size_t B2K_LOGREG_CSR_R_BYTES = (size_t)256 << 20;      // cap on one row chunk's residuals R [rows][kp] fp64
struct B2kCsr {
  const int64_t* indptr;
  const int32_t* indices;
  const float* values;
  int64_t n, nnz, d;
};
int b2k_logreg_eval_csr_impl(b2k_ctx* ctx, const B2kCsr& X, const float* y, const double* classes, int n_classes, int kp,
                             const double* W, const double* b, double* loss_out, double* grad_out, int64_t* n_total_out,
                             cudaStream_t s);
int b2k_logreg_fit_csr_impl(b2k_ctx* ctx, const B2kCsr& X, const float* y, const double* classes, const int64_t* counts,
                            int n_classes, int n_fits, const b2k_logreg_params* prm, double* coef_out,
                            double* intercept_out, int* kp_out, int* n_iter_out, cudaStream_t s);
int b2k_logreg_predict_csr_impl(b2k_ctx* ctx, const B2kCsr& X, int kp, const double* W, const double* b,
                                const double* class_values, double* raw_out, double* prob_out, double* pred_out,
                                cudaStream_t s);

// ------------------------------------------------------------------------------------------------
// Gaussian mixtures — b2k_gmm.cu (the C ABI entry points in b2k_api.cu check their arguments, check the partitions and
// draw the random start, then call these).  w [k], mu [k][d], cov [k][d][d]: the starting model, fp64.
// ------------------------------------------------------------------------------------------------
int b2k_gmm_fit_impl(b2k_ctx* ctx, const float* X, int64_t n, int d, int k, std::vector<double> w,
                     std::vector<double> mu, std::vector<double> cov, int max_iter, double tol, double* weights_out,
                     double* means_out, double* covs_out, double* log_likelihood_out, int* n_iter_out,
                     int64_t* cluster_sizes_out, cudaStream_t s);
int b2k_gmm_predict_impl(b2k_ctx* ctx, const float* X, int64_t n, int d, int k, const double* weights,
                         const double* means, const double* covs, double* prob_out, int32_t* labels_out,
                         cudaStream_t s);

// ------------------------------------------------------------------------------------------------
// bisecting k-means — b2k_bisect.cu (the C ABI entry points in b2k_api.cu check their arguments and the partitions, then
// call these)
// ------------------------------------------------------------------------------------------------
int b2k_bkm_fit_impl(b2k_ctx* ctx, const float* X, int64_t n, int d, int k, int max_iter, double min_divisible,
                     uint64_t seed, int* n_nodes_out, int64_t* node_index_out, double* node_centers_out,
                     int64_t* node_size_out, double* node_cost_out, double* training_cost_out,
                     int64_t* cluster_sizes_out, double* level_ms_out, cudaStream_t s);
int b2k_bkm_predict_impl(b2k_ctx* ctx, const float* X, int64_t n, int d, int n_nodes, const int64_t* node_index,
                         const double* node_centers, int32_t* labels_out, double* cost_out, cudaStream_t s);

// ------------------------------------------------------------------------------------------------
// multilayer perceptron — b2k_mlp.cu (the C ABI entry points in b2k_api.cu check their arguments and the partitions,
// then call these; layers are checked by b2k_mlp_check_layers)
// ------------------------------------------------------------------------------------------------
int b2k_mlp_check_layers(b2k_ctx* ctx, const int* layers, int n_layers, int d);
int64_t b2k_mlp_n_weights(const int* layers, int n_layers);
int b2k_mlp_eval_impl(b2k_ctx* ctx, const float* X, const float* y, int64_t n, const int* layers, int n_layers,
                      const double* weights, double* f_out, double* grad_out, int64_t* n_total_out, cudaStream_t s);
int b2k_mlp_fit_impl(b2k_ctx* ctx, const float* X, const float* y, int64_t n, const int* layers, int n_layers,
                     int solver, int max_iter, double tol, double step_size, uint64_t seed,
                     const double* initial_weights, double* weights_out, double* history_out, int* n_iter_out,
                     cudaStream_t s);
int b2k_mlp_predict_impl(b2k_ctx* ctx, const float* X, int64_t n, const int* layers, int n_layers,
                         const double* weights, double* raw_out, double* prob_out, double* pred_out, cudaStream_t s);

// ------------------------------------------------------------------------------------------------
// ALS — b2k_als.cu (the C ABI entry points in b2k_api.cu check their arguments, then call these)
// ------------------------------------------------------------------------------------------------
int b2k_als_fit_impl(b2k_ctx* ctx, const double* users, const double* items, const float* ratings, int64_t n,
                     int rank, int max_iter, double reg_param, int implicit_prefs, double alpha, uint64_t seed,
                     const float* init_user_factors, int64_t init_n_users, int64_t user_cap, int64_t item_cap,
                     int32_t* user_ids_out, float* user_factors_out, int32_t* item_ids_out, float* item_factors_out,
                     int64_t* n_users_out, int64_t* n_items_out, cudaStream_t s);
int b2k_als_predict_impl(b2k_ctx* ctx, const double* users, const double* items, int64_t n, int rank,
                         const int32_t* user_ids, const float* user_factors, int64_t n_users, const int32_t* item_ids,
                         const float* item_factors, int64_t n_items, float* out, cudaStream_t s);
int b2k_als_recommend_impl(b2k_ctx* ctx, const float* Q, int64_t nq, const float* T, int64_t nt, int rank, int n,
                           int32_t* idx_out, float* score_out, cudaStream_t s);

// ------------------------------------------------------------------------------------------------
// evaluation — b2k_eval.cu (the C ABI entry points in b2k_api.cu check their arguments, then call these)
// ------------------------------------------------------------------------------------------------
int b2k_eval_linear_impl(b2k_ctx* ctx, const float* X, const float* y, int64_t n, int d, int m, const int32_t* kind,
                         const int32_t* row_offsets, const double* W, const double* b, const double* class_values,
                         int n_classes, double eps, int64_t* label_count_out, int64_t* tp_out, int64_t* fp_out,
                         double* loss_out, double* reg_out, cudaStream_t s);
int b2k_eval_forest_impl(b2k_ctx* ctx, const float* X, const float* y, int64_t n, int d, int m, int classification,
                         const int32_t* n_trees, const int32_t* n_values, const int64_t* tree_offsets,
                         const int32_t* feature, const float* threshold, const int32_t* children, const double* value,
                         int n_classes, double eps, int64_t* label_count_out, int64_t* tp_out, int64_t* fp_out,
                         double* loss_out, double* reg_out, cudaStream_t s);
int b2k_eval_linear_scores_impl(b2k_ctx* ctx, const float* X, const float* y, int64_t n, int d, int m,
                                const int32_t* kind, const int32_t* row_offsets, const double* W, const double* b,
                                double* scores, int64_t ld_scores, uint8_t* pos, cudaStream_t s);
int b2k_eval_forest_scores_impl(b2k_ctx* ctx, const float* X, const float* y, int64_t n, int d, int m,
                                const int32_t* n_trees, const int32_t* n_values, const int64_t* tree_offsets,
                                const int32_t* feature, const float* threshold, const int32_t* children,
                                const double* value, double* scores, int64_t ld_scores, uint8_t* pos, cudaStream_t s);
// b2k_binary.cu
int b2k_eval_binary_impl(b2k_ctx* ctx, const double* scores, const uint8_t* pos, int64_t n, int m, int num_bins,
                         int metric, double* out, cudaStream_t s);
