// Host side of the wgmma fused assign kernel that does not depend on the shape family: which shapes it takes, the plan
// (family and persistent grid), dispatch to b2k_fused_tc.cu (variant 0) / b2k_fused_t.cu (variant 1) and the TMA
// descriptor encoder both use.  No device code.
#include <algorithm>

#include "b2k_internal.cuh"

bool b2k_fused_supported(int64_t n, int d, int k, const float* X) {
  if (n < 1 || n > (int64_t)0x7fffff00) return false;
  if (d % 4 != 0) return false;                                   // TMA: row pitch must be a multiple of 16 B
  if ((reinterpret_cast<uintptr_t>(X) & 15u) != 0) return false;  // TMA: 16 B aligned base
  return d <= 256 && k <= 256;                                    // variant 1 covers every shape variant 0 does
}

int b2k_fused_plan(b2k_ctx* ctx, int64_t n, int d, int k, B2kFusedPlan* plan) {
  *plan = B2kFusedPlan{};
  const int64_t ntiles = (n + B2K_FUSED_TILE_ROWS - 1) / B2K_FUSED_TILE_ROWS;
  int grid = ctx->sm_count;
  if (ctx->grid_limit > 0 && ctx->grid_limit < grid) grid = ctx->grid_limit;
  if (ntiles < grid) grid = (int)ntiles;
  plan->grid = std::max(grid, 1);
  if (!ctx->force_variant_t && b2k_fused_tc_plan(n, d, k, plan)) return B2K_OK;
  if (d % 4 != 0 || d > 256 || k > 256) return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "fused kernel: no instantiation for this (k, d)");
  b2k_fused_t_plan(ctx, n, d, k, plan);
  return B2K_OK;
}

int b2k_fused_prepare(b2k_ctx* ctx, const B2kFusedPlan& plan, void* plan_scratch, const float* X, int64_t n, int d, int k,
                      cudaStream_t s) {
  if (plan.variant == 1) return b2k_fused_t_prepare(ctx, plan, plan_scratch, X, n, d, k, s);
  return B2K_OK;
}

int b2k_launch_fused(b2k_ctx* ctx, const B2kFusedPlan& plan, void* plan_scratch, const float* X, int64_t n, int d,
                     const float* C, int k, int32_t* labels_out, float* mindist_out, bool do_update, bool need_cost,
                     const B2kLoopState* st, cudaStream_t s) {
  // a Lloyd pass computes labels + sums (its callers pass no min distance); the other passes compute labels + cost
  if (do_update && mindist_out != nullptr)
    return b2k_fail(ctx, B2K_ERR_INVALID, "fused kernel: a Lloyd pass does not produce min distances");
  if (plan.variant == 1)
    return b2k_launch_fused_t(ctx, plan, plan_scratch, X, n, d, C, k, labels_out, mindist_out, do_update, need_cost, st, s);
  return b2k_launch_fused_tc(ctx, plan, plan_scratch, X, n, d, C, k, labels_out, mindist_out, do_update, st, s);
}

// ------------------------------------------------------------------------------------------------
// TMA descriptors: 2D f32 tensor, 128-byte swizzle (the K-major GMMA operand layout of b2k_wg.cuh)
// ------------------------------------------------------------------------------------------------
namespace {
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
}  // namespace

int b2k_encode_2d(b2k_ctx* ctx, CUtensorMap* map, const void* base, uint64_t inner, uint64_t outer,
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
