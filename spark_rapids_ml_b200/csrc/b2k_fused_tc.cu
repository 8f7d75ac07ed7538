// Fused assign kernel for sm_90a, k <= 128 and d <= 128 (3xTF32 wgmma, b2k_wg.cuh): variant 0 of the fused kernel, whose
// shape rules, plan and dispatch are in b2k_fused.cu.  This file holds its instantiations, scratch layout and launch.
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

bool b2k_fused_tc_plan(int64_t n, int d, int k, B2kFusedPlan* plan) {
  Inst in;
  if (!pick_inst(d, k, &in)) return false;
  plan->variant = 0;
  plan->KP = in.KP;
  plan->DP = in.DP;
  plan->P = plan->grid;   // one partial-sum slot per CTA (the fused update)
  plan->Pc = plan->grid;
  const PlanLayout L = plan_layout(*plan, n, k, d);
  plan->off_partials = L.off_partials;
  plan->off_counts = L.off_counts;
  plan->off_cost = L.off_cost;
  plan->scratch_bytes = L.total;
  return true;
}

int b2k_launch_fused_tc(b2k_ctx* ctx, const B2kFusedPlan& plan, void* plan_scratch, const float* X, int64_t n, int d,
                        const float* C, int k, int32_t* labels_out, float* mindist_out, bool do_update,
                        const B2kLoopState* st, cudaStream_t s) {
  PlanLayout L = plan_layout(plan, n, k, d);
  char* b = static_cast<char*>(plan_scratch);
  float* Chi = reinterpret_cast<float*>(b + L.off_chi);
  float* Clo = reinterpret_cast<float*>(b + L.off_clo);
  float* cnorm = reinterpret_cast<float*>(b + L.off_cnorm);

  k_prep_centers_tc<<<(plan.KP * 32 + 255) / 256, 256, 0, s>>>(C, k, d, plan.KP, plan.DP, Chi, Clo, cnorm, st);
  ctx->stats.kernel_launches++;
  B2K_CUDA_OK(ctx, cudaGetLastError());

  CUtensorMap mx, mh, ml;
  B2K_TRY(b2k_encode_2d(ctx, &mx, X, (uint64_t)d, (uint64_t)n, (uint64_t)d * 4, CHUNK, TM,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B));
  B2K_TRY(b2k_encode_2d(ctx, &mh, Chi, (uint64_t)plan.DP, (uint64_t)plan.KP, (uint64_t)plan.DP * 4, CHUNK,
                        (uint32_t)plan.KP, CU_TENSOR_MAP_L2_PROMOTION_L2_128B));
  B2K_TRY(b2k_encode_2d(ctx, &ml, Clo, (uint64_t)plan.DP, (uint64_t)plan.KP, (uint64_t)plan.DP * 4, CHUNK,
                        (uint32_t)plan.KP, CU_TENSOR_MAP_L2_PROMOTION_L2_128B));

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
  const bool need_cost = !do_update;   // every assign pass forms the cost partials

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
