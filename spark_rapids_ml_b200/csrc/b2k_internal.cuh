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
  int probe = 0;                 // debug/experiment switch for the fused kernel (0 = normal)
  int adaptive_path = 1;         // option "adaptive_path": a Lloyd loop on the large-shape kernel falls back to the generic
                                 // kernels for its remaining iterations when most rows need the exact fix-up
  int lloyd_switched = 0;
  int near_tie_hint = 0;         // set around the k-means|| candidate passes: prefer exact 128-centre chunks (d <= 128)        // the last lloyd_impl call did so (the fit's inertia pass follows it)
  int force_variant_t = 0;       // option "variant_t": route every supported shape through b2k_fused_t.cu (tests)
  int tma_box_rows = 0;          // option "tma_box_rows": rows per TMA box of b2k_debug_tma_stream (diagnostic; 0 = 128)
  int collect_recheck = 0;       // option "collect_recheck": fill stats.recheck_* (costs a stream sync per call)
  int want_cost = 1;             // assign passes: compute the cost partial (set by assign_impl)
  int profile_fused = 0;         // record per-role blocked-cycle counters of the fused kernel
  // Row norms of the large-shape kernel, shared by every pass of ONE b2k_kmeans_fit call (k-means|| candidate passes,
  // the Lloyd loop, the inertia pass all see the same immutable X): computed by the first pass, reused by the rest.
  const float* xnorm_scope_X = nullptr;   // non-null only inside b2k_kmeans_fit
  int64_t xnorm_scope_n = 0;
  int xnorm_scope_d = 0;
  void* xnorm_cache = nullptr;            // float2 [xnorm_cache_rows]
  int64_t xnorm_cache_rows = 0;
  int xnorm_cache_valid = 0;
  long long* prof_dev = nullptr;  // [grid][18 warps][8]
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
// per-cluster partial sums from labels: partials [P][k*d] f32, counts [P][k] i32; returns P via *P_out.
size_t b2k_update_generic_scratch(b2k_ctx* ctx, int64_t n, int d, int k, int* P_out);
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
// k-means|| helpers
int b2k_launch_min_inplace(b2k_ctx* ctx, float* a, const float* b, int64_t n, cudaStream_t s);
int b2k_launch_bernoulli_pick(b2k_ctx* ctx, const float* mind, int64_t n, int64_t row_offset,
                              double scale /* l/phi */, uint64_t seed, int round, int64_t* picked,
                              int* n_picked, int cap, cudaStream_t s);
int b2k_launch_histogram(b2k_ctx* ctx, const int32_t* labels, int64_t n, int m, double* hist,
                         cudaStream_t s);
int b2k_launch_weighted_update(b2k_ctx* ctx, const float* P, const double* w, const int32_t* lab, int M, int d, int k,
                               float* C, cudaStream_t s);
int b2k_launch_pairwise_sqdist(b2k_ctx* ctx, const float* P, int M, int d, float* D2, cudaStream_t s);

// ------------------------------------------------------------------------------------------------
// wgmma fused assign kernel — b2k_fused_tc.cu / b2k_fused_t.cu (b2k_wg.cuh)
// ------------------------------------------------------------------------------------------------
struct B2kFusedPlan {
  int KP = 0, DP = 0;        // padded cluster count / dimension of the instantiation, 0 = unsupported
  int grid = 0;              // persistent CTAs
  int variant = 0;           // 0: b2k_fused_tc.cu (k <= 128, d <= 128, 3xTF32); 1: b2k_fused_t.cu (k, d <= 256, 1xTF32 + recheck)
  int P = 0;                 // partial-sum slots of the update pass (b2k_update_generic_scratch)
  int Pc = 0;                // cost partials the pass writes (variant 0: grid; variant 1: grid + fix-up CTAs)
  size_t scratch_bytes = 0;  // centre operands/cnorm + partials/counts/cost (+ row norms, variant 1)
};
bool b2k_fused_supported(const b2k_ctx* ctx, int64_t n, int d, int k, const float* X);
int b2k_fused_plan(b2k_ctx* ctx, int64_t n, int d, int k, B2kFusedPlan* plan);
// Once per fit / lloyd / assign call, before the first b2k_launch_fused on this X (variant 1: row norms; variant 0: no-op)
int b2k_fused_prepare(b2k_ctx* ctx, const B2kFusedPlan& plan, void* plan_scratch, const float* X, int64_t n, int d, int k,
                      cudaStream_t s);
// One fused pass: (labels_out, mindist_out optional) + partial sums/counts/cost into plan scratch.
// `do_update` = accumulate partial sums (Lloyd iteration) or labels only (assign/inertia pass).
int b2k_launch_fused(b2k_ctx* ctx, const B2kFusedPlan& plan, void* plan_scratch, const float* X,
                     int64_t n, int d, const float* C, int k, int32_t* labels_out, float* mindist_out,
                     bool do_update, const B2kLoopState* st, cudaStream_t s, const double* prev_counts = nullptr);
// Views into the plan scratch after a fused pass (to feed b2k_launch_reduce_partials)
void b2k_fused_views(const B2kFusedPlan& plan, void* plan_scratch, int64_t n, int k, int d, float** partials,
                     int32_t** counts, double** cost_partials);
// variant 1 diagnostics: {rows re-decided exactly, candidate distances evaluated} since the last b2k_fused_prepare
int b2k_fused_recheck_stats(b2k_ctx* ctx, const B2kFusedPlan& plan, void* plan_scratch, int64_t n, int k, int d,
                            unsigned long long out[2], cudaStream_t s);

// b2k_fused_t.cu (variant 1)
bool b2k_fused_t_supported(const b2k_ctx* ctx, int64_t n, int d, int k, const float* X);
int b2k_fused_t_plan(b2k_ctx* ctx, int64_t n, int d, int k, B2kFusedPlan* plan);
void b2k_fused_t_views(const B2kFusedPlan& plan, void* plan_scratch, int64_t n, int k, int d, float** partials,
                       int32_t** counts, double** cost_partials, unsigned long long** rstat);
int b2k_fused_t_prepare(b2k_ctx* ctx, const B2kFusedPlan& plan, void* plan_scratch, const float* X, int64_t n, int d,
                        int k, cudaStream_t s);
int b2k_launch_fused_t(b2k_ctx* ctx, const B2kFusedPlan& plan, void* plan_scratch, const float* X, int64_t n, int d,
                       const float* C, int k, int32_t* labels_out, float* mindist_out, bool do_update, bool need_cost,
                       const B2kLoopState* st, cudaStream_t s, const double* prev_counts);
int b2k_launch_merge_chunk(b2k_ctx* ctx, float* md_acc, int32_t* lab_acc, const float* md, const int32_t* lab, int base,
                           int64_t n, const B2kLoopState* st, cudaStream_t s);
int b2k_fused_encode_2d(b2k_ctx* ctx, CUtensorMap* map, const void* base, uint64_t inner, uint64_t outer,
                        uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer, int l2_256);

// ------------------------------------------------------------------------------------------------
// comm — b2k_comm.cu
// ------------------------------------------------------------------------------------------------
int b2k_comm_allreduce_f64(b2k_ctx* ctx, double* buf, size_t count, cudaStream_t s);
int b2k_comm_allgather_i64(b2k_ctx* ctx, const int64_t* send_dev, int64_t* recv_dev, size_t count_per_rank,
                           cudaStream_t s);
int b2k_comm_allreduce_f32(b2k_ctx* ctx, float* buf, size_t count, cudaStream_t s);

// ingest — b2k_ingest.cu (entry point is the C ABI itself)
