// C-ABI entry points + host-side driver of the Lloyd loop (see include/b2kmeans.h for the reference
// interfaces each one replaces).  The driver enqueues {fused assign+update | generic assign, update} ->
// fixed-order partial reduce -> NCCL allreduce of one fused f64 buffer -> finalize, several iterations ahead
// of the host; convergence lives on the device (B2kLoopState) and is polled every `check_every` iterations.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <vector>

#include "b2k_internal.cuh"

static std::string g_last_error;  // failures of calls that have no context

int b2k_fail(b2k_ctx* ctx, int code, const std::string& msg) {
  if (ctx) ctx->err = msg;
  else g_last_error = msg;
  return code;
}

extern "C" int b2k_version(void) { return B2K_VERSION; }

extern "C" const char* b2k_last_error(const b2k_ctx* ctx) {
  return ctx ? ctx->err.c_str() : g_last_error.c_str();
}

extern "C" int b2k_ctx_create(int device, b2k_ctx** out) {
  if (!out) return b2k_fail(nullptr, B2K_ERR_INVALID, "b2k_ctx_create: out is NULL");
  *out = nullptr;
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return b2k_fail(nullptr, B2K_ERR_CUDA,
                    std::string("b2k_ctx_create: no CUDA device (") + cudaGetErrorString(e) +
                        "); libb2kmeans has no CPU fallback");
  }
  if (device < 0 || device >= ndev)
    return b2k_fail(nullptr, B2K_ERR_INVALID, "b2k_ctx_create: device index out of range");
  b2k_ctx* ctx = new b2k_ctx();
  ctx->device = device;
  if ((e = cudaSetDevice(device)) != cudaSuccess) {
    delete ctx;
    return b2k_fail(nullptr, B2K_ERR_CUDA, std::string("cudaSetDevice: ") + cudaGetErrorString(e));
  }
  cudaDeviceProp prop;
  if ((e = cudaGetDeviceProperties(&prop, device)) != cudaSuccess) {
    delete ctx;
    return b2k_fail(nullptr, B2K_ERR_CUDA, std::string("cudaGetDeviceProperties: ") + cudaGetErrorString(e));
  }
  if (prop.major != 9 || prop.minor != 0) {
    delete ctx;
    return b2k_fail(nullptr, B2K_ERR_UNSUPPORTED,
                    "libb2kmeans is built for sm_90a (H100) only; device is sm_" + std::to_string(prop.major) +
                        std::to_string(prop.minor));
  }
  ctx->sm_count = prop.multiProcessorCount;
  ctx->smem_optin = prop.sharedMemPerBlockOptin;
  if ((e = cudaHostAlloc((void**)&ctx->h_state, 2 * sizeof(B2kLoopState), cudaHostAllocDefault)) != cudaSuccess) {
    delete ctx;
    return b2k_fail(nullptr, B2K_ERR_CUDA, std::string("cudaHostAlloc: ") + cudaGetErrorString(e));
  }
  *out = ctx;
  return B2K_OK;
}

extern "C" int b2k_ctx_destroy(b2k_ctx* ctx) {
  if (!ctx) return B2K_OK;
  cudaSetDevice(ctx->device);
  if (ctx->nccl) b2k_comm_destroy(ctx);
  b2k_copy_pool_destroy(ctx);
  if (ctx->scratch) cudaFree(ctx->scratch);
  if (ctx->prof_dev) cudaFree(ctx->prof_dev);
  if (ctx->xnorm_cache) cudaFree(ctx->xnorm_cache);
  for (int i = 0; i < 2; ++i) {
    if (ctx->pinned[i]) cudaFreeHost(ctx->pinned[i]);
    if (ctx->dev_stage[i]) cudaFree(ctx->dev_stage[i]);
    if (ctx->stage_evt[i]) cudaEventDestroy(ctx->stage_evt[i]);
  }
  if (ctx->h_state) cudaFreeHost(ctx->h_state);
  delete ctx;
  return B2K_OK;
}

extern "C" int b2k_ctx_set_option(b2k_ctx* ctx, const char* key, int64_t value) {
  if (!ctx || !key) return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_ctx_set_option: NULL argument");
  std::string k(key);
  if (k == "kernel_path") {
    if (value < B2K_PATH_AUTO || value > B2K_PATH_FUSED)
      return b2k_fail(ctx, B2K_ERR_INVALID, "kernel_path must be 0 (auto), 1 (generic) or 2 (fused)");
    ctx->kernel_path = (int)value;
  } else if (k == "time_kernels") {
    ctx->time_kernels = value < 0 ? 0 : (value > 2 ? 2 : (int)value);
  } else if (k == "check_every") {
    if (value < 1) return b2k_fail(ctx, B2K_ERR_INVALID, "check_every must be >= 1");
    ctx->check_every = (int)value;
  } else if (k == "adaptive_path") {
    ctx->adaptive_path = value ? 1 : 0;
  } else if (k == "probe" || k == "pair") {
    // switches of the earlier sm_100a kernels (diagnostic builds, CTA pairs): accepted for compatibility, no effect
    (void)value;
  } else if (k == "variant_t") {
    ctx->force_variant_t = value ? 1 : 0;
  } else if (k == "ingest_threads") {
    if (value < 0 || value > 64) return b2k_fail(ctx, B2K_ERR_INVALID, "ingest_threads must be in [0, 64]");
    b2k_copy_pool_destroy(ctx);
    ctx->ingest_threads = (int)value;
  } else if (k == "collect_recheck") {
    ctx->collect_recheck = value ? 1 : 0;
  } else if (k == "profile_fused") {
    ctx->profile_fused = value ? 1 : 0;
  } else if (k == "grid_limit") {
    if (value < 0) return b2k_fail(ctx, B2K_ERR_INVALID, "grid_limit must be >= 0");
    ctx->grid_limit = (int)value;
  } else {
    return b2k_fail(ctx, B2K_ERR_INVALID, "unknown option: " + k);
  }
  return B2K_OK;
}

extern "C" int b2k_get_stats(const b2k_ctx* ctx, b2k_stats* out) {
  if (!ctx || !out) return B2K_ERR_INVALID;
  *out = ctx->stats;
  return B2K_OK;
}
extern "C" int b2k_reset_stats(b2k_ctx* ctx) {
  if (!ctx) return B2K_ERR_INVALID;
  ctx->stats = b2k_stats{};
  return B2K_OK;
}

int b2k_scratch_reserve(b2k_ctx* ctx, size_t bytes) {
  if (bytes <= ctx->scratch_bytes) return B2K_OK;
  if (ctx->scratch) {
    B2K_CUDA_OK(ctx, cudaDeviceSynchronize());
    B2K_CUDA_OK(ctx, cudaFree(ctx->scratch));
    ctx->scratch = nullptr;
    ctx->scratch_bytes = 0;
  }
  size_t want = bytes + (bytes >> 3) + (1 << 20);
  cudaError_t e = cudaMalloc(&ctx->scratch, want);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return b2k_fail(ctx, B2K_ERR_NOMEM, "scratch cudaMalloc of " + std::to_string(want) + " bytes failed: " +
                                            cudaGetErrorString(e));
  }
  ctx->scratch_bytes = want;
  return B2K_OK;
}

namespace {
int check_shape(b2k_ctx* ctx, const char* who, const void* X, int64_t n, int d, int k) {
  if (!ctx) return b2k_fail(nullptr, B2K_ERR_INVALID, std::string(who) + ": ctx is NULL");
  if (!X || n < 0 || d <= 0 || k <= 0)
    return b2k_fail(ctx, B2K_ERR_INVALID, std::string(who) + ": bad X/n/d/k");
  return B2K_OK;
}

bool use_fused(const b2k_ctx* ctx, int64_t n, int d, int k, const float* X) {
  return ctx->kernel_path != B2K_PATH_GENERIC && b2k_fused_supported(n, d, k, X);
}

// kernel_path = 2 on a shape the fused kernel does not take is an error, not a fall-back to the generic kernels
int check_forced_fused(b2k_ctx* ctx, int64_t n, int d, int k, const float* X) {
  if (ctx->kernel_path != B2K_PATH_FUSED || b2k_fused_supported(n, d, k, X)) return B2K_OK;
  return b2k_fail(ctx, B2K_ERR_UNSUPPORTED,
                  "kernel_path=2 (fused) requested but shape (n=" + std::to_string(n) + ", d=" + std::to_string(d) +
                      ", k=" + std::to_string(k) + ") is outside the fused kernel's instantiations");
}

// stats.recheck_*: the rows the large-shape kernel re-decided exactly since b2k_fused_prepare and the candidate distances
// it evaluated for them (zero for the 3xTF32 kernel, which defers none).  Synchronises the stream.
int fill_recheck_stats(b2k_ctx* ctx, const B2kFusedPlan& plan, void* plan_scratch, cudaStream_t s) {
  unsigned long long rs[2] = {0ull, 0ull};
  if (const unsigned long long* dev = plan.rstat(plan_scratch)) {
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(rs, dev, sizeof(rs), cudaMemcpyDeviceToHost, s));
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  }
  ctx->stats.recheck_rows = (int64_t)rs[0];
  ctx->stats.recheck_candidates = (int64_t)rs[1];
  return B2K_OK;
}

// Scratch footprint of one assign/lloyd call.
struct LoopBuffers {
  B2kLoopState* st;
  double* R;
  double* shift_scratch;
  float* cnorm;
  // generic
  int32_t* labels;
  float* partials;
  int32_t* counts;
  int P;
  // fused
  B2kFusedPlan plan;
  void* plan_scratch;
};

}  // namespace

// ------------------------------------------------------------------------------------------------
// Chunked assignment for cluster counts beyond one fused pass: the centres are cut into chunks of exactly CH (the last
// chunk is [k - CH, k): the overlap is harmless for a min), each chunk runs one fused assign pass that yields the min
// distance and label of every row within the chunk, and k_merge_chunk keeps the smaller distance (strict '<': lowest
// cluster index on ties).  d <= 128: CH = 128, through the 3xTF32 kernel (exact, no fix-up) where it has a KP = 128
// instantiation, i.e. 32 < d <= 128; at d <= 32 the chunks take the large-shape kernel (1xTF32 screening + exact fix-up),
// as every fused pass with 64 < k <= 128 there does.  128 < d <= 256: CH = 256 through the large-shape kernel.  Used for
// k > 256 (assign passes, and Lloyd with the generic label-driven update) and — d <= 128 only — for k > 128 when the
// caller expects near-ties (the k-means|| candidate passes: candidates drawn from one blob are almost equidistant from
// its rows, which is the worst case of the screening kernel and free for the 3xTF32 one).  Replaces the SIMT assign of
// the generic path for d % 4 == 0.
// ------------------------------------------------------------------------------------------------
namespace {
// The path of one assign pass and where it keeps its scratch (assign_layout)
struct AssignScratch {
  int ch = 0;                   // chunk size, 0 = not chunked
  bool fused = false;           // not chunked: one fused pass over every centre, else the generic kernels
  B2kFusedPlan plan;            // chunked, fused
  void* ps = nullptr;           // plan scratch
  int32_t* tmp_lab = nullptr;   // chunked
  float* tmp_md = nullptr;
  int32_t* lab_acc = nullptr;   // used when the caller passes no labels / mindist buffer
  float* md_acc = nullptr;
  float* cnorm = nullptr;       // generic
  double* blocks = nullptr;     // chunked, generic: block sums of the cost
};
// chunk size, 0 = this (d, k) is not chunked
int chunked_assign_ch(const b2k_ctx* ctx, int64_t n, int d, int k, const float* X) {
  if (ctx->kernel_path == B2K_PATH_GENERIC || n <= 0 || d > 256) return 0;
  const int ch = (d <= 128 && !ctx->force_variant_t) ? 128 : 256;
  const bool want = k > 256 || (ch == 128 && k > 128 && ctx->near_tie_hint);
  if (!want || !b2k_fused_supported(n, d, ch, X)) return 0;
  return ch;
}
constexpr int kCostBlocks = 1024;   // block sums of the two-level cost reduction
// Lays out the scratch of one assign pass in L and chooses its path.  own_md: the caller wants the cost and passes no
// mindist buffer (the generic path then keeps its own in md_acc).  A fused or chunked pass starts with b2k_fused_prepare.
int assign_layout(b2k_ctx* ctx, int64_t n, int d, int k, const float* X, bool own_md, B2kLayout& L, AssignScratch* a) {
  if ((a->ch = chunked_assign_ch(ctx, n, d, k, X))) {
    B2K_TRY(b2k_fused_plan(ctx, n, d, a->ch, &a->plan));
    a->tmp_lab = L.take<int32_t>(n);
    a->tmp_md = L.take<float>(n);
    a->lab_acc = L.take<int32_t>(n);
    a->md_acc = L.take<float>(n);
    a->ps = L.take<char>(a->plan.scratch_bytes, 1024);
    a->blocks = L.take<double>(kCostBlocks);
  } else if ((a->fused = use_fused(ctx, n, d, k, X))) {
    B2K_TRY(b2k_fused_plan(ctx, n, d, k, &a->plan));
    a->ps = L.take<char>(a->plan.scratch_bytes, 1024);
  } else {
    a->cnorm = L.take<float>(k);
    if (own_md) a->md_acc = L.take<float>(n > 0 ? n : 1);
    a->blocks = L.take<double>(kCostBlocks);
  }
  return B2K_OK;
}
// raises *bytes to what assign_impl lays out for these arguments (a caller sizes its nested region with the largest)
int assign_need(b2k_ctx* ctx, int64_t n, int d, int k, const float* X, bool own_md, size_t* bytes) {
  B2kLayout measure;
  AssignScratch a;
  B2K_TRY(assign_layout(ctx, n, d, k, X, own_md, measure, &a));
  *bytes = std::max(*bytes, measure.off);
  return B2K_OK;
}
int chunked_assign_run(b2k_ctx* ctx, const AssignScratch& ca, const float* X, int64_t n, int d, const float* C, int k,
                       int32_t* labels, float* mindist, const B2kLoopState* st, cudaStream_t s) {
  int32_t* lab = labels ? labels : ca.lab_acc;
  float* md = mindist ? mindist : ca.md_acc;
  for (int c0 = 0; c0 < k; c0 += ca.ch) {
    const int base = std::min(c0, k - ca.ch);
    const bool first = c0 == 0;
    B2K_TRY(b2k_launch_fused(ctx, ca.plan, ca.ps, X, n, d, C + (size_t)base * d, ca.ch, first ? lab : ca.tmp_lab,
                             first ? md : ca.tmp_md, false, false, st, s));
    if (!first) B2K_TRY(b2k_launch_merge_chunk(ctx, md, lab, ca.tmp_md, ca.tmp_lab, base, n, st, s));
  }
  return B2K_OK;
}
}  // namespace

// ------------------------------------------------------------------------------------------------
// Lloyd loop
// ------------------------------------------------------------------------------------------------
static int lloyd_impl(b2k_ctx* ctx, const float* X, int64_t n, int d, int k, float* C, int max_iter, double tol,
                      int* n_iter_out, double* shift_out, cudaStream_t s) {
  if (max_iter < 0) return b2k_fail(ctx, B2K_ERR_INVALID, "lloyd: max_iter < 0");
  const bool dbg = std::getenv("B2K_DEBUG_TIMING") != nullptr;
  const auto t_entry = std::chrono::steady_clock::now();
  auto since = [&](std::chrono::steady_clock::time_point t0) {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  };
  // k > 256 (d <= 256): the assignment runs in 256-centre chunks on the large-shape kernel, the update stays generic
  const int chunk_ch = k > 256 ? chunked_assign_ch(ctx, n, d, k, X) : 0;
  const bool chunked = chunk_ch != 0;
  if (!chunked) B2K_TRY(check_forced_fused(ctx, n, d, k, X));
  const bool fused = !chunked && use_fused(ctx, n, d, k, X);
  ctx->stats.last_path = (fused || chunked) ? B2K_PATH_FUSED : B2K_PATH_GENERIC;

  LoopBuffers B{};
  if (fused) B2K_TRY(b2k_fused_plan(ctx, n, d, k, &B.plan));
  // The large-shape kernel (1xTF32 screening) hands near-tie rows to an exact fix-up; on data where most rows are
  // near-ties (e.g. uniform noise in 256 dimensions) the generic kernels are several times faster, so the loop may
  // switch to them between bursts.  The choice is local to the rank: both paths fill the same R buffer.
  const bool can_switch = fused && B.plan.variant == 1 && ctx->adaptive_path && ctx->kernel_path == B2K_PATH_AUTO;
  const bool need_generic = !fused || can_switch;
  if (need_generic) B.P = b2k_update_generic_slots(ctx, n, d, k);
  const size_t rlen = b2k_reduced_len(k, d);
  AssignScratch ca;
  B2K_TRY(b2k_scratch_layout(ctx, "lloyd", [&](B2kLayout& L) -> int {
    B.st = L.take<B2kLoopState>(1);
    B.R = L.take<double>(rlen);
    B.shift_scratch = L.take<double>(k);
    B.cnorm = L.take<float>(k);
    if (need_generic) {
      B.labels = L.take<int32_t>(n > 0 ? n : 1);
      B.partials = L.take<float>((size_t)B.P * k * d);
      B.counts = L.take<int32_t>((size_t)B.P * k);
    }
    if (fused) B.plan_scratch = L.take<char>(B.plan.scratch_bytes, 1024);
    if (chunked) B2K_TRY(assign_layout(ctx, n, d, k, X, false, L, &ca));   // takes the chunked path, as chunk_ch says
    return B2K_OK;
  }));

  B2kLoopState init{};
  init.iter = 0;
  init.done = max_iter == 0 ? 1 : 0;
  init.max_iter = max_iter;
  init.blocks_done = 0;
  init.tol = tol;
  init.shift = 0.0;
  init.cost = 0.0;
  init.fix_rows_cum = 0;
  init.fix_cands_cum = 0;
  *ctx->h_state = init;
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(B.st, ctx->h_state, sizeof(B2kLoopState), cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));  // h_state is reused as the D2H mirror below

  // Events are created BEFORE the timed loop (cudaEventCreate inside it showed up in the multi-GPU per-iteration gap).
  // time_kernels = 1: around every fused launch; 2: also after the partial reduce, the allreduce and finalize.
  const int nev_per_it = ctx->time_kernels >= 2 ? 5 : (ctx->time_kernels ? 2 : 0);
  std::vector<cudaEvent_t> ev;
  cudaEvent_t loop0 = nullptr, loop1 = nullptr, poll_ev[2] = {nullptr, nullptr};
  if (ctx->time_kernels) {
    ev.resize((size_t)nev_per_it * (size_t)std::max(max_iter, 0));
    for (auto& e : ev) B2K_CUDA_OK(ctx, cudaEventCreate(&e));
    B2K_CUDA_OK(ctx, cudaEventCreate(&loop0));
    B2K_CUDA_OK(ctx, cudaEventCreate(&loop1));
  }
  B2K_CUDA_OK(ctx, cudaEventCreateWithFlags(&poll_ev[0], cudaEventDisableTiming));
  B2K_CUDA_OK(ctx, cudaEventCreateWithFlags(&poll_ev[1], cudaEventDisableTiming));
  if (fused && max_iter > 0) B2K_TRY(b2k_fused_prepare(ctx, B.plan, B.plan_scratch, X, n, d, k, s));
  if (chunked && max_iter > 0) B2K_TRY(b2k_fused_prepare(ctx, ca.plan, ca.ps, X, n, d, chunk_ch, s));
  if (ctx->time_kernels) B2K_CUDA_OK(ctx, cudaEventRecord(loop0, s));
  const double t_setup = since(t_entry);
  const auto t_loop = std::chrono::steady_clock::now();
  double t_first_burst = 0.0;

  // The host stays one burst ahead of the device: burst b + 1 is enqueued BEFORE the convergence flag of burst b is
  // read back, so a poll never drains the stream (every hot-loop kernel returns at once when `done` is set, which
  // makes an over-enqueued burst free).  The read-backs alternate between two pinned mirrors.
  int launched = 0, slot = 0;
  bool done = (max_iter == 0), have_pending = false;
  bool fused_now = fused;
  int burst_iters[2] = {0, 0};
  unsigned long long seen_rows = 0, seen_cands = 0;
  ctx->stats.path_switch_iter = -1;
  B2kLoopState* mirror = ctx->h_state;
  int last_slot = 0;
  while (!done && launched < max_iter) {
    int burst = std::min(ctx->check_every, max_iter - launched);
    for (int b = 0; b < burst; ++b) {
      cudaEvent_t* e = ctx->time_kernels ? &ev[(size_t)launched * nev_per_it] : nullptr;
      if (fused_now) {
        if (e) B2K_CUDA_OK(ctx, cudaEventRecord(e[0], s));
        B2K_TRY(b2k_launch_fused(ctx, B.plan, B.plan_scratch, X, n, d, C, k, nullptr, nullptr, true, false, B.st, s));
        if (e) B2K_CUDA_OK(ctx, cudaEventRecord(e[1], s));
        B2K_TRY(b2k_launch_reduce_partials(ctx, B.plan.partials(B.plan_scratch), B.plan.counts(B.plan_scratch),
                                           B.plan.cost_partials(B.plan_scratch), B.plan.P, B.plan.Pc, k, d, B.R, B.st, s));
      } else {
        if (e) B2K_CUDA_OK(ctx, cudaEventRecord(e[0], s));
        if (chunked) {
          B2K_TRY(chunked_assign_run(ctx, ca, X, n, d, C, k, B.labels, nullptr, B.st, s));
        } else {
          B2K_TRY(b2k_launch_center_norms(ctx, C, k, d, B.cnorm, B.st, s));
          B2K_TRY(b2k_launch_assign_generic(ctx, X, n, d, C, B.cnorm, k, B.labels, nullptr, B.st, s));
        }
        B2K_TRY(b2k_launch_update_generic(ctx, X, n, d, B.labels, k, B.P, B.partials, B.counts, B.st, s));
        if (e) B2K_CUDA_OK(ctx, cudaEventRecord(e[1], s));
        B2K_TRY(b2k_launch_reduce_partials(ctx, B.partials, B.counts, nullptr, B.P, 0, k, d, B.R, B.st, s));
      }
      if (e && nev_per_it == 5) B2K_CUDA_OK(ctx, cudaEventRecord(e[2], s));
      if (ctx->nranks > 1) B2K_TRY(b2k_comm_allreduce_f64(ctx, B.R, rlen, s));
      if (e && nev_per_it == 5) B2K_CUDA_OK(ctx, cudaEventRecord(e[3], s));
      B2K_TRY(b2k_launch_finalize(ctx, B.R, C, k, d, B.shift_scratch, B.st, s));
      if (e && nev_per_it == 5) B2K_CUDA_OK(ctx, cudaEventRecord(e[4], s));
      ++launched;
    }
    if (t_first_burst == 0.0) t_first_burst = since(t_loop);
    burst_iters[slot] = fused_now ? burst : 0;
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(&mirror[slot], B.st, sizeof(B2kLoopState), cudaMemcpyDeviceToHost, s));
    B2K_CUDA_OK(ctx, cudaEventRecord(poll_ev[slot], s));
    if (have_pending) {   // the flag of the PREVIOUS burst, while this one is already queued
      B2K_CUDA_OK(ctx, cudaEventSynchronize(poll_ev[slot ^ 1]));
      const B2kLoopState& m = mirror[slot ^ 1];
      done = m.done != 0;
      if (can_switch && fused_now && burst_iters[slot ^ 1] > 0 && n > 0) {
        // cost model (k = d = 256): the fix-up costs ~0.14 ns per candidate distance + ~0.85 ns per deferred row; the
        // generic kernels ~6.4 ns per row more than the fused pass (scaled here by k d).  These constants were fitted on
        // the earlier B200 kernels and have not been re-measured on H100: the switch point is unvalidated there.
        const double it = (double)burst_iters[slot ^ 1];
        const double rows_per_row = (double)(m.fix_rows_cum - seen_rows) / it / (double)n;
        const double cands_per_row = (double)(m.fix_cands_cum - seen_cands) / it / (double)n;
        const double generic_extra_ns = 6.4 * ((double)k * (double)d) / 65536.0;
        if (0.14 * cands_per_row + 0.85 * rows_per_row > generic_extra_ns) {
          fused_now = false;
          ctx->stats.path_switch_iter = launched;
        }
      }
      seen_rows = m.fix_rows_cum;
      seen_cands = m.fix_cands_cum;
    }
    last_slot = slot;
    have_pending = true;
    slot ^= 1;
  }
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  if (dbg)
    fprintf(stderr, "[b2k rank %d] lloyd host timing: setup %.3f ms, first burst enqueued after %.3f ms, loop %.3f ms (%d iterations)\n",
            ctx->rank, t_setup, t_first_burst, since(t_loop), launched);
  if (have_pending && last_slot != 0) mirror[0] = mirror[last_slot];   // h_state[0] = the final state
  cudaEventDestroy(poll_ev[0]);
  cudaEventDestroy(poll_ev[1]);
  if (ctx->time_kernels) {
    B2K_CUDA_OK(ctx, cudaEventRecord(loop1, s));
    B2K_CUDA_OK(ctx, cudaEventSynchronize(loop1));
    float ms = 0.f;
    B2K_CUDA_OK(ctx, cudaEventElapsedTime(&ms, loop0, loop1));
    ctx->stats.last_loop_ms = ms;
    double acc = 0.0, acc_red = 0.0, acc_comm = 0.0, acc_fin = 0.0;
    int cnt = 0;
    const int iters_done = ctx->h_state->iter;
    for (int i = 0; i < launched && i < iters_done; ++i) {   // launches after convergence are no-ops
      float m = 0.f;
      cudaEvent_t* e = &ev[(size_t)i * nev_per_it];
      cudaEventElapsedTime(&m, e[0], e[1]);
      acc += m;
      if (nev_per_it == 5) {
        cudaEventElapsedTime(&m, e[1], e[2]); acc_red += m;
        cudaEventElapsedTime(&m, e[2], e[3]); acc_comm += m;
        cudaEventElapsedTime(&m, e[3], e[4]); acc_fin += m;
      }
      ++cnt;
    }
    for (auto& e : ev) cudaEventDestroy(e);
    ctx->stats.last_fused_ms = cnt ? acc / cnt : 0.0;
    ctx->stats.last_reduce_ms = cnt ? acc_red / cnt : 0.0;
    ctx->stats.last_allreduce_ms = cnt ? acc_comm / cnt : 0.0;
    ctx->stats.last_finalize_ms = cnt ? acc_fin / cnt : 0.0;
    cudaEventDestroy(loop0);
    cudaEventDestroy(loop1);
  }
  ctx->stats.last_n_iter = ctx->h_state->iter;
  ctx->lloyd_switched = (fused && !fused_now) ? 1 : 0;
  if (ctx->lloyd_switched) ctx->stats.last_path = B2K_PATH_GENERIC;
  if (fused && ctx->collect_recheck && max_iter > 0) B2K_TRY(fill_recheck_stats(ctx, B.plan, B.plan_scratch, s));
  if (n_iter_out) *n_iter_out = ctx->h_state->iter;
  if (shift_out) *shift_out = ctx->h_state->shift;
  return B2K_OK;
}

extern "C" int b2k_kmeans_lloyd(b2k_ctx* ctx, const float* X, int64_t n_local, int d, int k, float* centers,
                                int max_iter, double tol, int* n_iter_out, double* shift_out, uintptr_t stream) {
  B2K_TRY(check_shape(ctx, "b2k_kmeans_lloyd", X, n_local, d, k));
  if (!centers) return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_kmeans_lloyd: centers is NULL");
  B2K_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  return lloyd_impl(ctx, X, n_local, d, k, centers, max_iter, tol, n_iter_out, shift_out,
                    reinterpret_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------------------------------------
// assign (+ optional total cost): labels/mindist may be NULL.  assign_impl lays out its scratch in the region its caller
// sized with assign_need; it never grows ctx->scratch, which would move memory the caller still holds there.
// ------------------------------------------------------------------------------------------------
static int assign_impl(b2k_ctx* ctx, const float* X, int64_t n, int d, const float* C, int k, int32_t* labels,
                       float* mindist, double* cost_dev /* device, 1 double, may be NULL */, B2kLayout region,
                       cudaStream_t s) {
  AssignScratch a;
  B2K_TRY(assign_layout(ctx, n, d, k, X, cost_dev && !mindist, region, &a));
  if (!a.ch) B2K_TRY(check_forced_fused(ctx, n, d, k, X));
  B2K_TRY(region.check(ctx, "assign"));
  const bool any_fused = a.ch || a.fused;
  ctx->stats.last_path = any_fused ? B2K_PATH_FUSED : B2K_PATH_GENERIC;
  if (any_fused) B2K_TRY(b2k_fused_prepare(ctx, a.plan, a.ps, X, n, d, a.ch ? a.ch : k, s));
  float* md = mindist ? mindist : a.md_acc;
  if (a.ch) {   // chunks of ch centres through a fused assign pass each
    B2K_TRY(chunked_assign_run(ctx, a, X, n, d, C, k, labels, mindist, nullptr, s));
    if (cost_dev) B2K_TRY(b2k_launch_sum_f32_to_f64(ctx, md, n, cost_dev, a.blocks, kCostBlocks, s));
  } else if (a.fused) {
    B2K_TRY(b2k_launch_fused(ctx, a.plan, a.ps, X, n, d, C, k, labels, mindist, false, cost_dev != nullptr, nullptr, s));
    // fold the per-CTA cost partials in index order
    if (cost_dev) B2K_TRY(b2k_launch_fold_f64(ctx, a.plan.cost_partials(a.ps), a.plan.Pc, cost_dev, s));
  } else {
    B2K_TRY(b2k_launch_center_norms(ctx, C, k, d, a.cnorm, nullptr, s));
    B2K_TRY(b2k_launch_assign_generic(ctx, X, n, d, C, a.cnorm, k, labels, md, nullptr, s));
    if (cost_dev) B2K_TRY(b2k_launch_sum_f32_to_f64(ctx, md, n, cost_dev, a.blocks, kCostBlocks, s));
  }
  if (any_fused && ctx->collect_recheck) B2K_TRY(fill_recheck_stats(ctx, a.plan, a.ps, s));
  return B2K_OK;
}

extern "C" int b2k_kmeans_assign(b2k_ctx* ctx, const float* X, int64_t n, int d, const float* centers, int k,
                                 int32_t* labels_out, float* mindist_out, uintptr_t stream) {
  B2K_TRY(check_shape(ctx, "b2k_kmeans_assign", X, n, d, k));
  if (!centers) return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_kmeans_assign: centers is NULL");
  if (n == 0) return B2K_OK;
  B2K_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  size_t need = 0;
  B2K_TRY(assign_need(ctx, n, d, k, X, false, &need));
  B2K_TRY(b2k_scratch_reserve(ctx, need));
  return assign_impl(ctx, X, n, d, centers, k, labels_out, mindist_out, nullptr,
                     B2kLayout(ctx->scratch, ctx->scratch_bytes), reinterpret_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------------------------------------
// initialisers
// ------------------------------------------------------------------------------------------------
namespace {
// global row bookkeeping across ranks
struct Rows {
  std::vector<int64_t> sizes;  // per rank
  int64_t offset = 0;          // this rank's first global row
  int64_t total = 0;
};

int gather_sizes(b2k_ctx* ctx, int64_t n_local, Rows* rows, cudaStream_t s) {
  rows->sizes.assign(ctx->nranks, 0);
  if (ctx->nranks == 1) {
    rows->sizes[0] = n_local;
  } else {
    int64_t *send = nullptr, *recv = nullptr;
    B2K_TRY(b2k_scratch_layout(ctx, "gather_sizes", [&](B2kLayout& L) -> int {
      send = L.take<int64_t>(1);
      recv = L.take<int64_t>(ctx->nranks);
      return B2K_OK;
    }));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(send, &n_local, 8, cudaMemcpyHostToDevice, s));
    B2K_TRY(b2k_comm_allgather_i64(ctx, send, recv, 1, s));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(rows->sizes.data(), recv, 8 * (size_t)ctx->nranks, cudaMemcpyDeviceToHost, s));
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  }
  rows->offset = 0;
  rows->total = 0;
  for (int r = 0; r < ctx->nranks; ++r) {
    if (r < ctx->rank) rows->offset += rows->sizes[r];
    rows->total += rows->sizes[r];
  }
  return B2K_OK;
}

// Reference: core.py:959-962 "A python worker received no data".  With a communicator the decision is taken on the
// allgathered sizes, so that every rank fails together instead of one rank leaving its peers in a collective.
int check_no_empty_partition(b2k_ctx* ctx, const char* who, int64_t n_local, cudaStream_t s) {
  Rows rows;
  B2K_TRY(gather_sizes(ctx, n_local, &rows, s));
  for (int r = 0; r < ctx->nranks; ++r)
    if (rows.sizes[r] == 0)
      return b2k_fail(ctx, B2K_ERR_INVALID, std::string(who) + ": empty partition (rank " + std::to_string(r) +
                                                " has n_local == 0)");
  return B2K_OK;
}

// out[m,d] (device) <- rows with the given sorted GLOBAL indices, identical on every rank.
int fetch_global_rows(b2k_ctx* ctx, const float* X, int64_t n_local, int d, const Rows& rows,
                      const std::vector<int64_t>& gidx, float* out, int64_t* idx_dev, cudaStream_t s) {
  const int m = (int)gidx.size();
  if (m == 0) return B2K_OK;
  B2K_CUDA_OK(ctx, cudaMemsetAsync(out, 0, (size_t)m * d * sizeof(float), s));
  // contiguous run of indices owned by this rank (gidx is sorted)
  int lo = 0;
  while (lo < m && gidx[lo] < rows.offset) ++lo;
  int hi = lo;
  while (hi < m && gidx[hi] < rows.offset + n_local) ++hi;
  if (hi > lo) {
    std::vector<int64_t> local(hi - lo);
    for (int i = lo; i < hi; ++i) local[i - lo] = gidx[i] - rows.offset;
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(idx_dev, local.data(), local.size() * 8, cudaMemcpyHostToDevice, s));
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));  // `local` dies at scope end
    B2K_TRY(b2k_launch_gather_rows(ctx, X, d, idx_dev, hi - lo, out, lo, s));
  }
  if (ctx->nranks > 1) B2K_TRY(b2k_comm_allreduce_f32(ctx, out, (size_t)m * d, s));
  return B2K_OK;
}

std::vector<int64_t> sample_distinct(std::mt19937_64& rng, int64_t total, int m) {
  // Floyd's algorithm: m distinct values in [0,total)
  std::vector<int64_t> chosen;
  chosen.reserve(m);
  for (int64_t j = total - m; j < total; ++j) {
    std::uniform_int_distribution<int64_t> U(0, j);
    int64_t t = U(rng);
    if (std::find(chosen.begin(), chosen.end(), t) == chosen.end()) chosen.push_back(t);
    else chosen.push_back(j);
  }
  std::sort(chosen.begin(), chosen.end());
  return chosen;
}

// Weighted greedy k-means++ on the (small) candidate set — host side, on the candidate-to-candidate squared distances
// D2 [M x M] computed on the device (every k-means++ centre IS a candidate, so the greedy phase is table look-ups:
// k * trials * M instead of k * trials * M * d operations).  Returns the chosen candidate indices; the weighted Lloyd
// refinement that follows runs on the device (init_kmeans_parallel).
void reduce_candidates(const std::vector<float>& D2, const std::vector<double>& wts, int M, int k, std::mt19937_64& rng,
                       std::vector<int64_t>* out) {
  std::vector<double> d2(M), cum(M);
  std::vector<int> chosen;
  chosen.reserve(k);
  // draw i with probability prob[i] / tot from the running sums cum[] (first i with u < cum[i])
  auto pick = [&](double tot) {
    std::uniform_real_distribution<double> U(0.0, tot);
    const double u = U(rng);
    const int i = (int)(std::upper_bound(cum.begin(), cum.end(), u) - cum.begin());
    return std::min(i, M - 1);
  };
  // potential of adding candidate c: sum_i w_i min(d2_i, D2[c][i]); four fixed partial sums (identical on every rank)
  auto potential = [&](int c) {
    const float* row = &D2[(size_t)c * M];
    double p0 = 0, p1 = 0, p2 = 0, p3 = 0;
    int i = 0;
    for (; i + 4 <= M; i += 4) {
      p0 += wts[i] * std::min(d2[i], (double)row[i]);
      p1 += wts[i + 1] * std::min(d2[i + 1], (double)row[i + 1]);
      p2 += wts[i + 2] * std::min(d2[i + 2], (double)row[i + 2]);
      p3 += wts[i + 3] * std::min(d2[i + 3], (double)row[i + 3]);
    }
    for (; i < M; ++i) p0 += wts[i] * std::min(d2[i], (double)row[i]);
    return (p0 + p1) + (p2 + p3);
  };
  double tot = 0;
  for (int i = 0; i < M; ++i) { tot += wts[i]; cum[i] = tot; }
  const int first = pick(tot);
  chosen.push_back(first);
  for (int i = 0; i < M; ++i) d2[i] = (double)D2[(size_t)first * M + i];
  const int trials = 2 + (int)std::log((double)std::max(k, 2));
  for (int j = 1; j < k; ++j) {
    tot = 0;
    for (int i = 0; i < M; ++i) { tot += wts[i] * d2[i]; cum[i] = tot; }
    double best_pot = -1;
    int best_c = 0;
    for (int tr = 0; tr < trials; ++tr) {
      const int c = tot > 0 ? pick(tot) : (int)(rng() % M);
      const double pot = potential(c);
      if (best_pot < 0 || pot < best_pot) { best_pot = pot; best_c = c; }
    }
    chosen.push_back(best_c);
    const float* row = &D2[(size_t)best_c * M];
    for (int i = 0; i < M; ++i) d2[i] = std::min(d2[i], (double)row[i]);
  }
  out->assign(chosen.begin(), chosen.end());
}
}  // namespace

static int init_random(b2k_ctx* ctx, const float* X, int64_t n, int d, int k, uint64_t seed, float* C,
                       cudaStream_t s) {
  Rows rows;
  B2K_TRY(gather_sizes(ctx, n, &rows, s));
  if (rows.total < k)
    return b2k_fail(ctx, B2K_ERR_INVALID, "init=random: fewer rows (" + std::to_string(rows.total) + ") than k");
  std::mt19937_64 rng(seed);
  std::vector<int64_t> gidx = sample_distinct(rng, rows.total, k);
  int64_t* idx_dev = nullptr;
  B2K_TRY(b2k_scratch_layout(ctx, "init=random", [&](B2kLayout& L) -> int {
    idx_dev = L.take<int64_t>(k);
    return B2K_OK;
  }));
  return fetch_global_rows(ctx, X, n, d, rows, gidx, C, idx_dev, s);
}

// Scalable k-means++ (k-means||): the reference forwards init="scalable-k-means++", oversampling_factor=2.0
// (clustering.py:134-136).  Distributional parity only (the reference's own seeded test is xfail).
static int init_kmeans_parallel(b2k_ctx* ctx, const float* X, int64_t n, int d, int k, uint64_t seed,
                                double oversampling, float* C, cudaStream_t s) {
  struct HintGuard {   // the candidate passes are near-tie heavy: see chunked_assign_ch
    b2k_ctx* c;
    explicit HintGuard(b2k_ctx* c_) : c(c_) { c->near_tie_hint = 1; }
    ~HintGuard() { c->near_tie_hint = 0; }
  } hint_guard(ctx);
  const int rounds = 5;
  Rows rows;
  B2K_TRY(gather_sizes(ctx, n, &rows, s));
  if (rows.total < k)
    return b2k_fail(ctx, B2K_ERR_INVALID, "init=k-means||: fewer rows (" + std::to_string(rows.total) + ") than k");
  const double ell = oversampling * k;
  const int cap = (int)std::min<int64_t>(rows.total, (int64_t)(4 * ell) + 64);  // per-round candidate cap
  const int Mmax = 1 + rounds * cap + k;
  size_t nn = (size_t)(n > 0 ? n : 1);
  const size_t per = (size_t)cap + 1;   // [count | cap indices] per rank in the candidate exchange
  // The assign passes below run with 1, m <= cap (a round) or M <= Mmax (the top-up) centres.  Within one path each need
  // grows with the count: the generic path's (taken for every count or none) with k, a fused plan's up to the 128 or 256
  // where the path changes; a chunked pass needs one full chunk's plan, which covers the fused need of any smaller
  // count.  These counts include every point where the path changes, so their needs bound every pass.
  size_t assign_bytes = 0;
  for (int kk : {1, std::min(cap, 128), std::min(cap, 256), cap, Mmax})
    B2K_TRY(assign_need(ctx, n, d, kk, X, false, &assign_bytes));
  int64_t *idx_dev, *xchg;
  int* n_picked_dev;
  double *phi_dev, *blocks, *hist;
  float *mind, *dn, *cand, *newc;
  int32_t *labels, *lab_new;
  B2kLayout assign_region;
  B2K_TRY(b2k_scratch_layout(ctx, "init=k-means||", [&](B2kLayout& L) -> int {
    idx_dev = L.take<int64_t>(cap + 8);
    n_picked_dev = L.take<int>(8);
    phi_dev = L.take<double>(4);
    blocks = L.take<double>(kCostBlocks);
    xchg = L.take<int64_t>(per * (size_t)(ctx->nranks + 1));
    mind = L.take<float>(nn);
    dn = L.take<float>(nn);
    labels = L.take<int32_t>(nn);    // running nearest candidate of every row (global candidate index)
    lab_new = L.take<int32_t>(nn);   // nearest among one round's new candidates
    cand = L.take<float>((size_t)Mmax * d);
    newc = L.take<float>((size_t)cap * d);
    hist = L.take<double>(Mmax);
    assign_region = L.tail(assign_bytes);
    return B2K_OK;
  }));

  std::mt19937_64 rng(seed);
  int M = 0;
  {  // first candidate: one uniformly random row
    std::uniform_int_distribution<int64_t> U(0, rows.total - 1);
    std::vector<int64_t> g{U(rng)};
    B2K_TRY(fetch_global_rows(ctx, X, n, d, rows, g, cand, idx_dev, s));
    M = 1;
    B2K_TRY(assign_impl(ctx, X, n, d, cand, 1, nullptr, mind, phi_dev, assign_region, s));
    B2K_CUDA_OK(ctx, cudaMemsetAsync(labels, 0, nn * 4, s));   // every row is nearest to candidate 0 so far
  }
  std::vector<int64_t> picked_host(cap);
  std::vector<int64_t> counts_host(ctx->nranks);
  for (int r = 0; r < rounds; ++r) {
    double phi = 0;
    if (r > 0) {
      // phi = sum(mind) (deterministic two-level sum)
      B2K_TRY(b2k_launch_sum_f32_to_f64(ctx, mind, n, phi_dev, blocks, kCostBlocks, s));
    }
    if (ctx->nranks > 1) B2K_TRY(b2k_comm_allreduce_f64(ctx, phi_dev, 1, s));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(&phi, phi_dev, 8, cudaMemcpyDeviceToHost, s));
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
    if (!(phi > 0)) break;
    // The pick kernel stores at most cap entries and WHICH ones it keeps on overflow depends on atomic slot order, so an
    // overflowing draw (expected ell picks against cap = 4 ell + 64: essentially never) is repeated with a smaller
    // probability scale: the draw is keyed on (seed, round, global row), so the smaller draw is a subset and the
    // candidate set stays a deterministic function of the seed.
    double scale = ell / phi;
    int np = 0;
    for (int attempt = 0; attempt < 8; ++attempt) {
      B2K_CUDA_OK(ctx, cudaMemsetAsync(n_picked_dev, 0, sizeof(int), s));
      B2K_TRY(b2k_launch_bernoulli_pick(ctx, mind, n, rows.offset, scale, seed, r, idx_dev, n_picked_dev, cap, s));
      B2K_CUDA_OK(ctx, cudaMemcpyAsync(&np, n_picked_dev, sizeof(int), cudaMemcpyDeviceToHost, s));
      B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
      if (np <= cap) break;
      scale *= 0.75 * (double)cap / (double)np;
    }
    np = std::min(np, cap);
    if (np > 0) B2K_CUDA_OK(ctx, cudaMemcpy(picked_host.data(), idx_dev, (size_t)np * 8, cudaMemcpyDeviceToHost));
    std::sort(picked_host.begin(), picked_host.begin() + np);   // slot order -> canonical order
    // exchange: every rank learns every rank's picks (global indices), capped in total
    std::vector<int64_t> all;
    if (ctx->nranks == 1) {
      all.assign(picked_host.begin(), picked_host.begin() + np);
    } else {
      // fixed-size allgather of [count | cap indices] per rank through a dedicated exchange buffer
      int64_t* send = xchg;
      int64_t* recv = send + per;
      std::vector<int64_t> pack(per, 0);
      pack[0] = np;
      std::copy(picked_host.begin(), picked_host.begin() + np, pack.begin() + 1);
      B2K_CUDA_OK(ctx, cudaMemcpyAsync(send, pack.data(), per * 8, cudaMemcpyHostToDevice, s));
      B2K_TRY(b2k_comm_allgather_i64(ctx, send, recv, per, s));
      std::vector<int64_t> got(per * ctx->nranks);
      B2K_CUDA_OK(ctx, cudaMemcpyAsync(got.data(), recv, got.size() * 8, cudaMemcpyDeviceToHost, s));
      B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
      for (int q = 0; q < ctx->nranks; ++q) {
        int64_t c = got[q * per];
        for (int64_t i = 0; i < c; ++i) all.push_back(got[q * per + 1 + i]);
      }
      std::sort(all.begin(), all.end());
    }
    if ((int)all.size() > cap) all.resize(cap);
    if (all.empty()) continue;
    const int m = (int)all.size();
    B2K_TRY(fetch_global_rows(ctx, X, n, d, rows, all, newc, idx_dev, s));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(cand + (size_t)M * d, newc, (size_t)m * d * 4, cudaMemcpyDeviceToDevice, s));
    // nearest among the new candidates, folded into the running (min distance, nearest candidate): strict '<' keeps the
    // earlier candidate on ties, so after the last round `labels` IS the argmin over all candidates — the k-means||
    // weights need no extra pass over X
    B2K_TRY(assign_impl(ctx, X, n, d, newc, m, lab_new, dn, nullptr, assign_region, s));
    B2K_TRY(b2k_launch_merge_chunk(ctx, mind, labels, dn, lab_new, M, n, nullptr, s));
    M += m;
  }
  if (M < k) {  // top up with distinct random rows so that M >= k (tiny inputs): these need one full assignment
    std::vector<int64_t> extra = sample_distinct(rng, rows.total, k - M + 1);
    B2K_TRY(fetch_global_rows(ctx, X, n, d, rows, extra, cand + (size_t)M * d, idx_dev, s));
    M += (int)extra.size();
    B2K_TRY(assign_impl(ctx, X, n, d, cand, M, labels, nullptr, nullptr, assign_region, s));
  }
  // weights = #points closest to each candidate (the running argmin of the rounds)
  B2K_TRY(b2k_launch_histogram(ctx, labels, n, M, hist, s));
  if (ctx->nranks > 1) B2K_TRY(b2k_comm_allreduce_f64(ctx, hist, M, s));
  std::vector<float> P((size_t)M * d);
  std::vector<double> wts(M);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(P.data(), cand, P.size() * 4, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(wts.data(), hist, (size_t)M * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  for (auto& w : wts) w = std::max(w, 1e-12);
  // candidate-to-candidate squared distances on the device (identical on every rank: same candidates, same kernel),
  // greedy weighted k-means++ on the host (table look-ups), then 10 weighted Lloyd steps on the device: the assignment
  // of the M candidates through the same kernels as any other assign pass, the weighted update in fixed order (fp64)
  std::vector<float> D2h((size_t)M * M);
  float *candd, *D2d, *Ck_dev;
  double* wts_dev;
  int32_t* lab_dev;
  int64_t* chosen_dev;
  B2kLayout refine_region;
  // the scratch may move here: only `cand` is needed from here on, and it was copied to P above
  B2K_TRY(b2k_scratch_layout(ctx, "init=k-means|| refinement", [&](B2kLayout& L) -> int {
    candd = L.take<float>((size_t)M * d);
    D2d = L.take<float>((size_t)M * M);
    wts_dev = L.take<double>(M);
    Ck_dev = L.take<float>((size_t)k * d);
    lab_dev = L.take<int32_t>(M);
    chosen_dev = L.take<int64_t>(k);
    // the refinement assigns the candidates candd: null when measuring, 256-byte aligned when placed, so the fused
    // path's 16-byte alignment rule sees the same in both runs
    size_t need = 0;
    B2K_TRY(assign_need(ctx, M, d, k, candd, false, &need));
    refine_region = L.tail(need);
    return B2K_OK;
  }));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(candd, P.data(), P.size() * 4, cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(wts_dev, wts.data(), (size_t)M * 8, cudaMemcpyHostToDevice, s));
  B2K_TRY(b2k_launch_pairwise_sqdist(ctx, candd, M, d, D2d, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(D2h.data(), D2d, D2h.size() * 4, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  std::vector<int64_t> chosen;
  reduce_candidates(D2h, wts, M, k, rng, &chosen);  // same seed + same inputs => identical on every rank
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(chosen_dev, chosen.data(), (size_t)k * 8, cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));  // `chosen` is pageable
  B2K_TRY(b2k_launch_gather_rows(ctx, candd, d, chosen_dev, k, Ck_dev, 0, s));
  for (int it = 0; it < 10; ++it) {
    B2K_TRY(assign_impl(ctx, candd, M, d, Ck_dev, k, lab_dev, nullptr, nullptr, refine_region, s));
    B2K_TRY(b2k_launch_weighted_update(ctx, candd, wts_dev, lab_dev, M, d, k, Ck_dev, s));
  }
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(C, Ck_dev, (size_t)k * d * 4, cudaMemcpyDeviceToDevice, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  return B2K_OK;
}

// ------------------------------------------------------------------------------------------------
// fit
// ------------------------------------------------------------------------------------------------
extern "C" int b2k_kmeans_fit(b2k_ctx* ctx, const float* X, int64_t n_local, int d, int k, int init_mode,
                              const float* init_centers, int max_iter, double tol, uint64_t seed,
                              double oversampling, int n_init, float* centers_out, int* n_iter_out,
                              double* inertia_out, uintptr_t stream) {
  B2K_TRY(check_shape(ctx, "b2k_kmeans_fit", X, n_local, d, k));
  if (!centers_out) return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_kmeans_fit: centers_out is NULL");
  if (n_init != 1)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "b2k_kmeans_fit: n_init must be 1 (the reference forces n_init=1)");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  B2K_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  B2K_TRY(check_no_empty_partition(ctx, "b2k_kmeans_fit", n_local, s));
  struct NormScope {   // see b2k_ctx::xnorm_scope_X
    b2k_ctx* c;
    NormScope(b2k_ctx* c_, const float* X_, int64_t n_, int d_) : c(c_) {
      c->xnorm_scope_X = X_;
      c->xnorm_scope_n = n_;
      c->xnorm_scope_d = d_;
      c->xnorm_cache_valid = 0;
    }
    ~NormScope() {
      c->xnorm_scope_X = nullptr;
      c->xnorm_cache_valid = 0;
    }
  } norm_scope(ctx, X, n_local, d);
  switch (init_mode) {
    case B2K_INIT_ARRAY:
      if (!init_centers) return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_kmeans_fit: init_centers is NULL");
      if (init_centers != centers_out)
        B2K_CUDA_OK(ctx, cudaMemcpyAsync(centers_out, init_centers, (size_t)k * d * 4, cudaMemcpyDeviceToDevice, s));
      break;
    case B2K_INIT_RANDOM:
      B2K_TRY(init_random(ctx, X, n_local, d, k, seed, centers_out, s));
      break;
    case B2K_INIT_KMEANS_PARALLEL:
      B2K_TRY(init_kmeans_parallel(ctx, X, n_local, d, k, seed, oversampling > 0 ? oversampling : 2.0,
                                   centers_out, s));
      break;
    default:
      return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_kmeans_fit: unknown init_mode");
  }
  B2K_TRY(lloyd_impl(ctx, X, n_local, d, k, centers_out, max_iter, tol, n_iter_out, nullptr, s));
  if (inertia_out) {
    // the inertia pass follows the Lloyd loop's choice of path (see lloyd_impl: adaptive_path)
    const int saved_path = ctx->kernel_path;
    if (ctx->lloyd_switched) ctx->kernel_path = B2K_PATH_GENERIC;
    double* cost_dev = nullptr;
    B2kLayout assign_region;
    int rc = b2k_scratch_layout(ctx, "inertia", [&](B2kLayout& L) -> int {
      cost_dev = L.take<double>(1);
      size_t need = 0;
      B2K_TRY(assign_need(ctx, n_local, d, k, X, true, &need));
      assign_region = L.tail(need);
      return B2K_OK;
    });
    if (rc == B2K_OK) rc = assign_impl(ctx, X, n_local, d, centers_out, k, nullptr, nullptr, cost_dev, assign_region, s);
    ctx->kernel_path = saved_path;
    B2K_TRY(rc);
    if (ctx->nranks > 1) B2K_TRY(b2k_comm_allreduce_f64(ctx, cost_dev, 1, s));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(inertia_out, cost_dev, 8, cudaMemcpyDeviceToHost, s));
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  }
  return B2K_OK;
}

// ------------------------------------------------------------------------------------------------
// PCA (b2k_pca.cu)
// ------------------------------------------------------------------------------------------------
extern "C" int b2k_pca_fit(b2k_ctx* ctx, const float* X, int64_t n_local, int d, int k, double* mean_out,
                           double* components_out, double* explained_variance_ratio_out, double* singular_values_out,
                           uintptr_t stream) {
  if (!ctx) return b2k_fail(nullptr, B2K_ERR_INVALID, "b2k_pca_fit: ctx is NULL");
  if (!X || n_local < 0 || d <= 0) return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_pca_fit: bad X/n/d");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  B2K_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  B2K_TRY(check_no_empty_partition(ctx, "b2k_pca_fit", n_local, s));
  return b2k_pca_fit_impl(ctx, X, n_local, d, k, mean_out, components_out, explained_variance_ratio_out,
                          singular_values_out, s);
}

extern "C" int b2k_pca_finalize(const double* cov, int d, int64_t n_total, int k, double* components_out,
                                double* explained_variance_ratio_out, double* singular_values_out) {
  return b2k_pca_finalize_impl(nullptr, cov, d, n_total, k, components_out, explained_variance_ratio_out,
                               singular_values_out);
}

extern "C" int b2k_pca_transform(b2k_ctx* ctx, const float* X, int64_t n, int d, const float* components, int k,
                                 float* out, uintptr_t stream) {
  if (!ctx) return b2k_fail(nullptr, B2K_ERR_INVALID, "b2k_pca_transform: ctx is NULL");
  if (!X || !components || !out || n < 0 || d <= 0 || k <= 0)
    return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_pca_transform: bad X/components/out/n/d/k");
  B2K_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  return b2k_pca_transform_impl(ctx, X, n, d, components, k, out, reinterpret_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------------------------------------
// exact k-NN (b2k_knn.cu)
// ------------------------------------------------------------------------------------------------
extern "C" int b2k_knn_search(b2k_ctx* ctx, const float* items, int64_t n_items_local, const int64_t* item_ids,
                              const float* queries, int64_t n_queries_local, int d, int k, float* distances_out,
                              int64_t* indices_out, uintptr_t stream) {
  if (!ctx) return b2k_fail(nullptr, B2K_ERR_INVALID, "b2k_knn_search: ctx is NULL");
  if (n_items_local < 0 || n_queries_local < 0 || d <= 0 || (n_items_local > 0 && !items) ||
      (n_queries_local > 0 && (!queries || !distances_out || !indices_out)))
    return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_knn_search: bad items/queries/outputs/n/d");
  if (n_items_local > (int64_t)0x7fffff00)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "b2k_knn_search: more than 2^31 - 256 items on one rank");
  B2K_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  return b2k_knn_search_impl(ctx, items, n_items_local, item_ids, queries, n_queries_local, d, k, distances_out,
                             indices_out, reinterpret_cast<cudaStream_t>(stream));
}
