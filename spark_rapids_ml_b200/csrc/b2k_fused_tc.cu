// Fused assign kernel for sm_90a, k <= 128 and d <= 128 (3xTF32 wgmma, b2k_wg.cuh), plus the host side shared with
// b2k_fused_t.cu (TMA descriptors) and the TMA streaming diagnostic.
//
// One Lloyd iteration on this path = k_prep_centers_tc (hi/lo split of the centres, ||c||^2) + ONE wgmma pass over X
// that assigns every row and forms the per-CTA per-cluster partial sums from the same shared-memory tile.
//
// Algorithmic HBM bytes per launch: 4*n*d (X once) [+ 4*n labels / 4*n mindist when requested] + grid * (k*d + k) * 4
// partials.  See DESIGN.md "Kernels".
#include <float.h>
#include <stdio.h>

#include "b2k_internal.cuh"

namespace {

#include "b2k_ptx.cuh"
#include "b2k_wg.cuh"

constexpr int CHUNK = WG_CHUNK;
constexpr int TM = WG_TM;

// ------------------------------------------------------------------------------------------------
// prep: padded hi/lo split of the centers + ||c||^2
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_prep_centers_tc(const float* __restrict__ C, int k, int d, int KP, int DP,
                                                         float* __restrict__ Chi, float* __restrict__ Clo,
                                                         float* __restrict__ cnorm, const B2kLoopState* st) {
  if (st != nullptr && st->done) return;
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (warp >= KP) return;
  double s = 0.0;
  for (int t = lane; t < DP; t += 32) {
    float v = (warp < k && t < d) ? C[(size_t)warp * d + t] : 0.f;
    uint32_t hb = rn_tf32_bits(v);
    float hi = __uint_as_float(hb);
    float lo = v - hi;
    Chi[(size_t)warp * DP + t] = hi;
    Clo[(size_t)warp * DP + t] = __uint_as_float(rn_tf32_bits(lo));
    s += (double)v * (double)v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) cnorm[warp] = warp < k ? (float)s : __int_as_float(0x7f800000);
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int get_encoder(b2k_ctx* ctx, EncodeTiledFn* fn) {
  if (!ctx->encode_tiled) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !p)
      return b2k_fail(ctx, B2K_ERR_CUDA, "cannot resolve cuTensorMapEncodeTiled from the driver");
    ctx->encode_tiled = p;
  }
  *fn = reinterpret_cast<EncodeTiledFn>(ctx->encode_tiled);
  return B2K_OK;
}

int encode_2d(b2k_ctx* ctx, CUtensorMap* map, const void* base, uint64_t inner, uint64_t outer,
              uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer, CUtensorMapL2promotion l2) {
  EncodeTiledFn fn;
  B2K_TRY(get_encoder(ctx, &fn));
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {row_stride_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, l2, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return b2k_fail(ctx, B2K_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r));
  return B2K_OK;
}

}  // namespace
int b2k_fused_encode_2d(b2k_ctx* ctx, CUtensorMap* map, const void* base, uint64_t inner, uint64_t outer,
                        uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer, int l2_256) {
  return encode_2d(ctx, map, base, inner, outer, row_stride_bytes, box_inner, box_outer,
                   l2_256 ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B : CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
}
namespace {
struct Inst {
  int KP, DP;
};
// instantiations compiled into the library
constexpr Inst kInst[] = {{64, 128}, {64, 64}, {64, 32}, {32, 128}, {128, 128}, {128, 64}, {16, 32}, {16, 64}, {32, 64}, {32, 32}, {16, 128}};

bool pick_inst(int d, int k, Inst* out) {
  int DP = (d + CHUNK - 1) / CHUNK * CHUNK;
  if (DP == 96) DP = 128;
  int best = -1;
  for (size_t i = 0; i < sizeof(kInst) / sizeof(kInst[0]); ++i) {
    if (kInst[i].DP == DP && kInst[i].KP >= k) {
      if (best < 0 || kInst[i].KP < kInst[best].KP) best = (int)i;
    }
  }
  if (best < 0) return false;
  *out = kInst[best];
  return true;
}

struct PlanLayout {
  size_t off_chi, off_clo, off_cnorm, off_partials, off_counts, off_cost, total;
};
PlanLayout plan_layout(const B2kFusedPlan& p, int64_t n, int k, int d) {
  auto al = [](size_t v) { return (v + 255) / 256 * 256; };
  PlanLayout L{};
  size_t o = 0;
  L.off_chi = o; o = al(o + (size_t)p.KP * p.DP * 4);
  L.off_clo = o; o = al(o + (size_t)p.KP * p.DP * 4);
  L.off_cnorm = o; o = al(o + (size_t)p.KP * 4);
  L.off_partials = o; o = al(o + (size_t)p.P * k * d * 4);
  L.off_counts = o; o = al(o + (size_t)p.P * k * 4);
  L.off_cost = o; o = al(o + (size_t)p.Pc * 8);
  L.total = o;
  return L;
}
}  // namespace

bool b2k_fused_supported(const b2k_ctx* ctx, int64_t n, int d, int k, const float* X) {
  (void)ctx;
  if (n < 1 || n > (int64_t)0x7fffff00 * 1LL) return false;
  if (d % 4 != 0) return false;                                   // TMA: row pitch must be a multiple of 16 B
  if ((reinterpret_cast<uintptr_t>(X) & 15u) != 0) return false;  // TMA: 16 B aligned base
  Inst in;
  if (pick_inst(d, k, &in)) return true;
  return b2k_fused_t_supported(ctx, n, d, k, X);   // large shapes: b2k_fused_t.cu (k <= 256, d <= 256)
}

int b2k_fused_plan(b2k_ctx* ctx, int64_t n, int d, int k, B2kFusedPlan* plan) {
  Inst in;
  if (!pick_inst(d, k, &in) || ctx->force_variant_t) {
    if (d % 4 == 0 && d <= 256 && k <= 256) return b2k_fused_t_plan(ctx, n, d, k, plan);
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "fused kernel: no instantiation for this (k, d)");
  }
  plan->variant = 0;
  plan->KP = in.KP;
  plan->DP = in.DP;
  int64_t ntiles = (n + TM - 1) / TM;
  int grid = ctx->sm_count;
  if (ctx->grid_limit > 0 && ctx->grid_limit < grid) grid = ctx->grid_limit;
  if (ntiles < grid) grid = (int)ntiles;
  if (grid < 1) grid = 1;
  plan->grid = grid;
  plan->P = grid;   // one partial-sum slot per CTA (the fused update)
  plan->Pc = grid;
  plan->scratch_bytes = plan_layout(*plan, n, k, d).total;
  return B2K_OK;
}

int b2k_fused_prepare(b2k_ctx* ctx, const B2kFusedPlan& plan, void* plan_scratch, const float* X, int64_t n, int d, int k,
                      cudaStream_t s) {
  if (plan.variant == 1) return b2k_fused_t_prepare(ctx, plan, plan_scratch, X, n, d, k, s);
  return B2K_OK;
}

int b2k_fused_recheck_stats(b2k_ctx* ctx, const B2kFusedPlan& plan, void* plan_scratch, int64_t n, int k, int d,
                            unsigned long long out[2], cudaStream_t s) {
  out[0] = out[1] = 0ull;
  if (plan.variant != 1) return B2K_OK;
  float* p;
  int32_t* c;
  double* cp;
  unsigned long long* rs;
  b2k_fused_t_views(plan, plan_scratch, n, k, d, &p, &c, &cp, &rs);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(out, rs, 16, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  return B2K_OK;
}

void b2k_fused_views(const B2kFusedPlan& plan, void* plan_scratch, int64_t n, int k, int d, float** partials,
                     int32_t** counts, double** cost_partials) {
  if (plan.variant == 1) {
    b2k_fused_t_views(plan, plan_scratch, n, k, d, partials, counts, cost_partials, nullptr);
    return;
  }
  PlanLayout L = plan_layout(plan, n, k, d);
  char* b = static_cast<char*>(plan_scratch);
  *partials = reinterpret_cast<float*>(b + L.off_partials);
  *counts = reinterpret_cast<int32_t*>(b + L.off_counts);
  *cost_partials = reinterpret_cast<double*>(b + L.off_cost);
}

int b2k_launch_fused(b2k_ctx* ctx, const B2kFusedPlan& plan, void* plan_scratch, const float* X, int64_t n, int d,
                     const float* C, int k, int32_t* labels_out, float* mindist_out, bool do_update,
                     const B2kLoopState* st, cudaStream_t s, const double* prev_counts) {
  if (plan.variant == 1)
    return b2k_launch_fused_t(ctx, plan, plan_scratch, X, n, d, C, k, labels_out, mindist_out, do_update,
                              !do_update && (mindist_out != nullptr || ctx->want_cost), st, s, prev_counts);
  PlanLayout L = plan_layout(plan, n, k, d);
  char* b = static_cast<char*>(plan_scratch);
  float* Chi = reinterpret_cast<float*>(b + L.off_chi);
  float* Clo = reinterpret_cast<float*>(b + L.off_clo);
  float* cnorm = reinterpret_cast<float*>(b + L.off_cnorm);

  k_prep_centers_tc<<<(plan.KP * 32 + 255) / 256, 256, 0, s>>>(C, k, d, plan.KP, plan.DP, Chi, Clo, cnorm, st);
  ctx->stats.kernel_launches++;
  B2K_CUDA_OK(ctx, cudaGetLastError());

  CUtensorMap mx, mh, ml;
  B2K_TRY(encode_2d(ctx, &mx, X, (uint64_t)d, (uint64_t)n, (uint64_t)d * 4, CHUNK, TM,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B));
  B2K_TRY(encode_2d(ctx, &mh, Chi, (uint64_t)plan.DP, (uint64_t)plan.KP, (uint64_t)plan.DP * 4, CHUNK, (uint32_t)plan.KP,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_128B));
  B2K_TRY(encode_2d(ctx, &ml, Clo, (uint64_t)plan.DP, (uint64_t)plan.KP, (uint64_t)plan.DP * 4, CHUNK, (uint32_t)plan.KP,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_128B));

  WgArgs a{};
  a.n = n;
  a.ntiles = (int)((n + TM - 1) / TM);
  a.k = k;
  a.d = d;
  a.cnorm = cnorm;
  a.labels_out = labels_out;
  a.mind_out = mindist_out;
  a.cost_partials = reinterpret_cast<double*>(b + L.off_cost);
  a.partials = reinterpret_cast<float*>(b + L.off_partials);
  a.counts = reinterpret_cast<int32_t*>(b + L.off_counts);
  a.st = st;
  if (ctx->profile_fused) {
    const size_t pbytes = (size_t)plan.grid * (WG_NTHREADS / 32) * WG_NPROF * sizeof(long long);
    if (ctx->prof_dev == nullptr) B2K_CUDA_OK(ctx, cudaMalloc(&ctx->prof_dev, (size_t)ctx->sm_count * (WG_NTHREADS / 32) * WG_NPROF * sizeof(long long)));
    B2K_CUDA_OK(ctx, cudaMemsetAsync(ctx->prof_dev, 0, pbytes, s));
    ctx->prof_grid = plan.grid;
    a.prof = ctx->prof_dev;
  }
  // a Lloyd pass computes labels + sums (its callers pass no min distance); the other passes compute labels + cost
  if (do_update && mindist_out != nullptr)
    return b2k_fail(ctx, B2K_ERR_INVALID, "fused kernel: a Lloyd pass does not produce min distances");
  const bool need_cost = !do_update;

  int rc = B2K_ERR_UNSUPPORTED;
#define B2K_DISPATCH(KP_, DP_) \
  if (plan.KP == KP_ && plan.DP == DP_) rc = b2k_launch_wg<KP_, DP_ / CHUNK, true>(ctx, plan.grid, mx, mh, ml, a, need_cost, do_update, s);
  B2K_DISPATCH(64, 128)
  B2K_DISPATCH(64, 64)
  B2K_DISPATCH(64, 32)
  B2K_DISPATCH(32, 128)
  B2K_DISPATCH(128, 128)
  B2K_DISPATCH(128, 64)
  B2K_DISPATCH(16, 32)
  B2K_DISPATCH(16, 64)
  B2K_DISPATCH(32, 64)
  B2K_DISPATCH(32, 32)
  B2K_DISPATCH(16, 128)
#undef B2K_DISPATCH
  if (rc == B2K_ERR_UNSUPPORTED) return b2k_fail(ctx, rc, "fused kernel: instantiation missing");
  B2K_TRY(rc);
  ctx->stats.kernel_launches++;
  ctx->stats.fused_tc_launches++;
  (void)prev_counts;
  return B2K_OK;
}

// diagnostics: per-warp phase cycle counters of the last profiled launch of the k, d <= 128 kernel (option
// profile_fused): [grid][WG_NTHREADS / 32][WG_NPROF], phases as in b2k_wg.cuh (WG_P_*)
extern "C" int b2k_get_fused_profile(b2k_ctx* ctx, long long* out, int64_t cap, int* grid_out, int* warps_out) {
  if (!ctx || !out || !grid_out || !warps_out) return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_get_fused_profile: NULL argument");
  if (ctx->prof_dev == nullptr || ctx->prof_grid == 0) return b2k_fail(ctx, B2K_ERR_STATE, "no fused profile recorded");
  const int64_t len = (int64_t)ctx->prof_grid * (WG_NTHREADS / 32) * WG_NPROF;
  if (cap < len) return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_get_fused_profile: output buffer too small");
  B2K_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  B2K_CUDA_OK(ctx, cudaDeviceSynchronize());
  B2K_CUDA_OK(ctx, cudaMemcpy(out, ctx->prof_dev, (size_t)len * sizeof(long long), cudaMemcpyDeviceToHost));
  *grid_out = ctx->prof_grid;
  *warps_out = WG_NTHREADS / 32;
  return B2K_OK;
}

// ------------------------------------------------------------------------------------------------
// diagnostics: TMA streaming microbenchmark.  Persistent CTAs pull X through an nslot x 16 KB shared-memory
// ring with the same 128B-swizzled [128 x 32 f32] boxes as the fused kernel; one consumer warp releases every
// slot `hold` clock cycles after it lands.  Gives the bandwidth the ring can sustain as a function of its depth
// and of how long the pipeline holds a slot (the fused kernel's ceiling; see DESIGN.md).
// ------------------------------------------------------------------------------------------------
namespace {
__global__ void __launch_bounds__(1024, 1) k_tma_stream(const __grid_constant__ CUtensorMap mapX, int ntiles, int nch,
                                                      int nslot, int hold, unsigned long long* sink, int box_rows) {
  const int SLOT_BYTES = box_rows * CHUNK * 4;   // shadows the 16 KB constant: option "tma_box_rows" (diagnostic)
  const int TM = box_rows;
  extern __shared__ uint8_t smem_raw2[];
  const uint32_t base = (smem_u32(smem_raw2) + 1023u) & ~1023u;
  const uint32_t bars = base + (uint32_t)nslot * SLOT_BYTES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < nslot; ++i) {
      mbar_init(bars + 8u * i, 1);
      mbar_init(bars + 8u * (nslot + i), 1);
    }
    mbar_init(bars + 8u * (2 * nslot), 1);        // "never" barrier: extra warps poll it (polling-load experiment)
    *reinterpret_cast<volatile int*>(smem_raw2 + (base - smem_u32(smem_raw2)) + nslot * SLOT_BYTES + 8 * (2 * nslot + 2)) = 0;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  volatile int* stop = reinterpret_cast<volatile int*>(smem_raw2 + (base - smem_u32(smem_raw2)) + nslot * SLOT_BYTES + 8 * (2 * nslot + 2));
  int s = 0;
  uint32_t ph = 0;
  if (warp >= 2) {                                 // spinner warps
    while (*stop == 0) { mbar_try_wait(bars + 8u * (2 * nslot), 0); }
    return;
  }
  if (warp == 0) {
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x)
      for (int c = 0; c < nch; ++c) {
        mbar_wait(bars + 8u * (nslot + s), ph ^ 1u);
        if (elect_one()) {
          mbar_expect_tx(bars + 8u * s, SLOT_BYTES);
          tma_load_2d(base + s * SLOT_BYTES, &mapX, bars + 8u * s, c * CHUNK, tile * TM);
        }
        __syncwarp();
        if (++s == nslot) { s = 0; ph ^= 1u; }
      }
  } else {
    unsigned long long acc = 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x)
      for (int c = 0; c < nch; ++c) {
        mbar_wait(bars + 8u * s, ph);
        if (hold > 0) {
          const long long t0 = clock64();
          while (clock64() - t0 < hold) {}
        }
        acc += lane;
        __syncwarp();
        if (lane == 0) mbar_arrive(bars + 8u * (nslot + s));
        if (++s == nslot) { s = 0; ph ^= 1u; }
      }
    if (acc == 0xdeadbeefULL) sink[0] = acc;
    *stop = 1;
  }
}
}  // namespace

// out_ms receives the device time of one pass over X[n, d] (d multiple of 32) with the given ring depth / hold
extern "C" int b2k_debug_tma_stream(b2k_ctx* ctx, const float* X, int64_t n, int d, int nslot, int hold_cycles,
                                    float* out_ms) {
  const int spinners = hold_cycles < 0 ? -hold_cycles : 0;   // hold < 0: |hold| extra warps polling an mbarrier
  if (hold_cycles < 0) hold_cycles = 0;
  const int box_rows = ctx->tma_box_rows > 0 ? ctx->tma_box_rows : TM;
  if (!ctx || !X || !out_ms || d % CHUNK != 0 || nslot < 1 || nslot * box_rows > 13 * 128)
    return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_debug_tma_stream: bad argument");
  CUtensorMap mx;
  B2K_TRY(encode_2d(ctx, &mx, X, (uint64_t)d, (uint64_t)n, (uint64_t)d * 4, CHUNK, (uint32_t)box_rows, CU_TENSOR_MAP_L2_PROMOTION_L2_256B));
  const int smem = nslot * box_rows * CHUNK * 4 + 2 * nslot * 8 + 1024 + 128;
  B2K_CUDA_OK(ctx, cudaFuncSetAttribute(k_tma_stream, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  B2K_TRY(b2k_scratch_reserve(ctx, 4096));
  cudaEvent_t e0, e1;
  B2K_CUDA_OK(ctx, cudaEventCreate(&e0));
  B2K_CUDA_OK(ctx, cudaEventCreate(&e1));
  const int ntiles = (int)((n + box_rows - 1) / box_rows);
  for (int rep = 0; rep < 2; ++rep) {
    if (rep == 1) B2K_CUDA_OK(ctx, cudaEventRecord(e0, 0));
    k_tma_stream<<<ctx->sm_count, 64 + 32 * spinners, smem, 0>>>(mx, ntiles, d / CHUNK, nslot, hold_cycles,
                                                 static_cast<unsigned long long*>(ctx->scratch), box_rows);
  }
  B2K_CUDA_OK(ctx, cudaEventRecord(e1, 0));
  B2K_CUDA_OK(ctx, cudaEventSynchronize(e1));
  B2K_CUDA_OK(ctx, cudaEventElapsedTime(out_ms, e0, e1));
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  return B2K_OK;
}
