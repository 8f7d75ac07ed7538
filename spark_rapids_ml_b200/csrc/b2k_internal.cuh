// Internal declarations shared by the translation units of libb2kmeans.so (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

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
  b2k_stats stats{};
};

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
// recv [nranks][bytes_per_rank] <- every rank's send; send may be recv's own slot (in place).  One rank: a copy.
int b2k_comm_allgather_bytes(b2k_ctx* ctx, const void* send_dev, void* recv_dev, size_t bytes_per_rank, cudaStream_t s);

// ingest — b2k_ingest.cu (entry point is the C ABI itself)

// ------------------------------------------------------------------------------------------------
// PCA — b2k_pca.cu (the C ABI entry points in b2k_api.cu check their arguments and the partitions, then call these)
// ------------------------------------------------------------------------------------------------
constexpr int B2K_PCA_MAX_D = 1024;   // both Gram paths, the projection kernel and the host eigen step
int b2k_pca_fit_impl(b2k_ctx* ctx, const float* X, int64_t n, int d, int k, double* mean_out, double* components_out,
                     double* evr_out, double* sv_out, cudaStream_t s);
// ctx may be NULL (b2k_pca_finalize): errors then go to b2k_last_error(NULL)
int b2k_pca_finalize_impl(b2k_ctx* ctx, const double* cov, int d, int64_t n_total, int k, double* components_out,
                          double* evr_out, double* sv_out);
int b2k_pca_transform_impl(b2k_ctx* ctx, const float* X, int64_t n, int d, const float* C, int k, float* Y,
                           cudaStream_t s);

// ------------------------------------------------------------------------------------------------
// exact k-NN — b2k_knn.cu (the C ABI entry point in b2k_api.cu checks its arguments, then calls this)
// ------------------------------------------------------------------------------------------------
constexpr int B2K_KNN_MAX_K = 1024;   // the generic path's per-query lists; the wgmma path takes k <= 64
int b2k_knn_search_impl(b2k_ctx* ctx, const float* items, int64_t n_items, const int64_t* item_ids,
                        const float* queries, int64_t nq_local, int d, int k, float* dist_out, int64_t* idx_out,
                        cudaStream_t s);
