// Fused assign for LARGE (k, d) on sm_90a — k <= 256, d <= 256 (BASELINE cfg3: k = 256, d = 256) — 1xTF32 screening
// + exact recheck, ONE pass over X per launch.  At k = d = 256 the tf32 centres (256 KB) do not fit in shared memory,
// so every TMA stage carries the X chunk [128 rows x 32 f32] together with the matching centre chunk [256 x 32 f32]
// (L2-resident); the wgmma kernel is shared with b2k_fused_tc.cu (b2k_wg.cuh, THREE = false):
//
//   * 1xTF32 screening: D = x~.c~ (x~: the fp32 words cut to tf32 by the tensor core, c~ = RN_tf32(c)); the epilogue
//     packs (dist' + ||x||^2 + thr, centre) into one ordered 32-bit key per centre and finds the smallest AND second
//     smallest key of every row.  A row whose gap is below the PROVEN bound thr(x) = 2E (see "Bound") is DEFERRED:
//     it goes to the CTA's segment of a fix-up list with the bit mask of every centre within thr of the best, and gets
//     no label from the pass.  k_fix_labels_t then decides those rows exactly (fp32 dot products against the fp32
//     centres, ascending centre order, strict '<' = lowest index on ties).  Rows outside the bound provably have the
//     same argmin in exact arithmetic, so labels match the 3xTF32 / fp32 paths.
//   * update (Lloyd passes): in the same pass, per 8-CTA cluster through distributed shared memory (b2k_wg.cuh);
//     k_fix_accum_t adds the deferred rows to FIX_SLOTS extra partial slots in a fixed order.
//   * assign / inertia passes: the exact min distance sum (x - c)^2 of every decided row (deferred rows: k_fix_labels_t).
//
// Algorithmic HBM bytes per launch: 4*n*d (X once) + 8*n (row norms) + 4*n labels [+ 4*n mindist when requested]
// + 40 B per deferred row + the deferred rows' X once more (k_fix_accum_t).
#include <float.h>
#include <stdio.h>

#include <algorithm>

#include "b2k_internal.cuh"

namespace {

#include "b2k_ptx.cuh"
#include "b2k_wg.cuh"

constexpr int TN = WG_TM;      // X rows per tile
constexpr int CHUNK = WG_CHUNK;

// ------------------------------------------------------------------------------------------------
// prep kernels
// ------------------------------------------------------------------------------------------------
// Ct[256][DP] = centres rounded to nearest tf32, zero padded; cnorm[256] = ||c||^2 (+inf for padding clusters)
__global__ void __launch_bounds__(256) k_prep_centers_t(const float* __restrict__ C, int k, int d, int DP,
                                                        float* __restrict__ Ct, float* __restrict__ cnorm,
                                                        const B2kLoopState* st) {
  if (st != nullptr && st->done) return;
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= 256) return;
  double s = 0.0, e = 0.0;
  for (int t = lane; t < DP; t += 32) {
    const float v = (row < k && t < d) ? C[(size_t)row * d + t] : 0.f;
    const float r = __uint_as_float(rn_tf32_bits(v));
    Ct[(size_t)row * DP + t] = r;
    s += (double)v * (double)v;
    e += ((double)v - (double)r) * ((double)v - (double)r);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    e += __shfl_xor_sync(0xffffffffu, e, o);
  }
  if (lane == 0) {
    cnorm[row] = row < k ? (float)s : __int_as_float(0x7f800000);
    cnorm[256 + row] = row < k ? (float)sqrt(e) : 0.f;   // ||c - c~||: the rounding error of this centre's tf32 operand
  }
}

// One block of 256 threads: the coefficients of the recheck threshold thr(x), see "Bound" below.
//
// Bound.  dist'_j = fl(||c_j||^2 - 2 x~.c~_j) with x~ = x cut to tf32 by the tensor core (dx = x~ - x, ||dx|| measured per
// row by k_row_norms) and c~ = RN_tf32(c) (dc_j = c~_j - c_j, ||dc_j|| measured per centre by k_prep_centers_t):
//   |x~.c~ - x.c| = |dx.c~ + x.dc| <= ||dx|| ||c~|| + ||x|| ||dc||                                    (Cauchy-Schwarz)
// tf32 products are exact in fp32; the fp32 accumulation of d <= 256 terms adds at most d * 2^-23 ||x|| ||c||
// <= 2^-15 ||x|| ||c|| (truncating adder assumed); the final fma and add round twice (2^-23 relative) and the key drops
// 8 mantissa bits (2^-15 relative), relative to the key value ||x - c||^2 + thr <= (||x|| + ||c||)^2 + thr.  With
// Cmax = max_j ||c_j|| (1 + 2^-11), dCmax = max_j ||dc_j||:
//   E(x) <= 2 (||dx|| Cmax + ||x|| dCmax) + ||x|| Cmax 2^-14 + (||x|| + Cmax)^2 2^-14
// Two approximate distances can be off by E each in opposite directions, so the argmin is proven whenever the gap exceeds
// 2E.  Shipped with a 1.25x margin (also covers the fp32 rounding of the norms themselves):
//   thr(x) = T0 ||dx|| + T1 ||x|| + T2 ||x||^2 + T3,
//   T0 = 5 Cmax,  T1 = 5 dCmax + Cmax 2^-12 * 1.25 + Cmax 2^-12 * 1.25,  T2 = 2^-13 * 1.25,  T3 = Cmax^2 2^-13 * 1.25
__global__ void __launch_bounds__(256) k_tables_t(int k, const float* __restrict__ cnorm, float* __restrict__ thr,
                                                  const B2kLoopState* st) {
  if (st != nullptr && st->done) return;
  __shared__ float cmax2[8];
  __shared__ float dcmax[8];
  const int j = threadIdx.x;
  float c2 = j < k ? cnorm[j] : 0.f;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c2 = fmaxf(c2, __shfl_xor_sync(0xffffffffu, c2, o));
  if ((j & 31) == 0) cmax2[j >> 5] = c2;
  float dc = j < k ? cnorm[256 + j] : 0.f;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) dc = fmaxf(dc, __shfl_xor_sync(0xffffffffu, dc, o));
  if ((j & 31) == 0) dcmax[j >> 5] = dc;
  __syncthreads();
  if (j == 0) {
    float m = 0.f, dm = 0.f;
    for (int i = 0; i < 8; ++i) { m = fmaxf(m, cmax2[i]); dm = fmaxf(dm, dcmax[i]); }
    const float cmax = sqrtf(m) * 1.0005f;
    thr[0] = 5.f * cmax;
    thr[1] = 5.f * dm + cmax * 0.0006103515625f;          // 2 * 1.25 * 2^-12
    thr[2] = 0.000152587890625f;                          // 1.25 * 2^-13
    thr[3] = cmax * cmax * 0.000152587890625f;
  }
}

// xnorm[i] = { ||x_i||, ||x_i - trunc_tf32(x_i)|| } (fp32).  One pass over X, once per fit / lloyd / assign call (X is
// immutable during the call).  The second value is the norm of the error the tensor core makes on this row when it cuts
// the fp32 words to tf32 (an upper bound if the hardware rounds instead: |RN error| <= |truncation error| per element).
__global__ void __launch_bounds__(256) k_row_norms(const float* __restrict__ X, int64_t n, int d, float2* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int d4 = d >> 2;
  for (int64_t row = warp0; row < n; row += nwarps) {
    const float4* p = reinterpret_cast<const float4*>(X + row * d);
    float s = 0.f, e = 0.f;
    for (int t = lane; t < d4; t += 32) {
      const float4 v = __ldcs(p + t);
      s = fmaf(v.x, v.x, fmaf(v.y, v.y, fmaf(v.z, v.z, fmaf(v.w, v.w, s))));
      const float ex = v.x - __uint_as_float(__float_as_uint(v.x) & 0xffffe000u);
      const float ey = v.y - __uint_as_float(__float_as_uint(v.y) & 0xffffe000u);
      const float ez = v.z - __uint_as_float(__float_as_uint(v.z) & 0xffffe000u);
      const float ew = v.w - __uint_as_float(__float_as_uint(v.w) & 0xffffe000u);
      e = fmaf(ex, ex, fmaf(ey, ey, fmaf(ez, ez, fmaf(ew, ew, e))));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s += __shfl_xor_sync(0xffffffffu, s, o);
      e += __shfl_xor_sync(0xffffffffu, e, o);
    }
    if (lane == 0) out[row] = make_float2(sqrtf(s) * 1.0000002f, sqrtf(e) * 1.0000002f);   // round up
  }
}

// ------------------------------------------------------------------------------------------------
// fix-up of the deferred rows
// ------------------------------------------------------------------------------------------------
struct FixArgs {
  const float* X;
  int64_t n;
  int d, k;
  const float* C32;            // [k][d]
  const float* cnorm;          // [256] ||c||^2 (fp32 centres)
  int2* list;
  const uint32_t* masks;
  const int32_t* count;
  int nseg, seg_cap, mask_cap;
  int32_t* labels_out;         // or NULL
  float* mind_out;             // or NULL
  int need_cost;
  double* cost_out;            // [gridDim.x] (always written)
  unsigned long long* rstat;   // or NULL
  float* partial;              // k_fix_accum_t: the deferred rows' [FIX_SLOTS][k][d] sums
  int32_t* counts_out;         // and their [FIX_SLOTS][k] counts
  const B2kLoopState* st;
  B2kLoopState* st_w;          // same object: k_fix_accum_t publishes the cumulative fix-up counters to the host's poll
};
constexpr int FIX_WARPS = 8;
constexpr int FIX_MAXP = 256;

// One warp per deferred row: exact argmin over the row's candidates.  d(j) = ||c_j||^2 - 2 x.c_j with the dot product as
// one fp32 FMA chain per lane (columns lane*4 + 128 i) and a fixed 5-level shuffle tree; candidates in ascending
// cluster order with strict '<' (lowest index wins ties).  Entries beyond the mask capacity test every cluster.
__global__ void __launch_bounds__(FIX_WARPS * 32) k_fix_labels_t(const FixArgs f) {
  if (f.st != nullptr && f.st->done) return;
  __shared__ int pre[FIX_MAXP + 1];
  __shared__ double cost_w[FIX_WARPS];
  if (threadIdx.x == 0) {
    int a = 0;
    for (int p = 0; p < f.nseg; ++p) {
      pre[p] = a;
      a += f.count[p];
    }
    pre[f.nseg] = a;
  }
  __syncthreads();
  const int M = pre[f.nseg];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double cost = 0.0;
  unsigned long long ncand = 0;
  for (int i = (int)blockIdx.x * FIX_WARPS + warp; i < M; i += (int)gridDim.x * FIX_WARPS) {
    int p = 0;   // segment of entry i = the number of segments that end at or before i (ends are non-decreasing)
    for (int b0 = 0; b0 < f.nseg; b0 += 32) {
      const int q = b0 + lane;
      p += __popc(__ballot_sync(0xffffffffu, q < f.nseg && pre[q + 1] <= i));
    }
    const int e = i - pre[p];
    int2* ent = f.list + (size_t)p * (size_t)f.seg_cap + e;
    const int64_t row = (int64_t)ent->x;
    uint32_t mw = 0xffffffffu;
    if (e < f.mask_cap && lane < 8) mw = f.masks[((size_t)p * (size_t)f.mask_cap + (size_t)e) * 8u + (uint32_t)lane];
    float4 xv[2];
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      const int cc = lane * 4 + 128 * t;
      xv[t] = cc < f.d ? __ldg(reinterpret_cast<const float4*>(f.X + (size_t)row * f.d + cc)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float best = __int_as_float(0x7f800000);
    int bj = -1;
    for (int pass = 0; pass < 2 && bj < 0; ++pass) {   // pass 1 (every cluster) only if the mask held no valid candidate
      int wi = -1;
      uint32_t bm = 0;
      auto next_cand = [&]() -> int {   // ascending cluster order, -1 at the end (warp-uniform)
        for (;;) {
          while (bm == 0u && wi < 7) {
            ++wi;
            bm = pass == 0 ? __shfl_sync(0xffffffffu, mw, wi) : 0xffffffffu;
          }
          if (bm == 0u) return -1;
          const int j = wi * 32 + (__ffs(bm) - 1);
          bm &= bm - 1;
          if (j < f.k) return j;
          bm = 0u;   // clusters are ascending: nothing valid is left in this word
        }
      };
      for (;;) {   // two candidates per trip: both centre rows' loads are in flight together
        const int ja = next_cand();
        if (ja < 0) break;
        const int jb = next_cand();
        const int jb2 = jb >= 0 ? jb : ja;
        float dota = 0.f, dotb = 0.f;
#pragma unroll
        for (int t = 0; t < 2; ++t) {
          const int cc = lane * 4 + 128 * t;
          if (cc < f.d) {
            const float4 ca = __ldg(reinterpret_cast<const float4*>(f.C32 + (size_t)ja * f.d + cc));
            const float4 cb = __ldg(reinterpret_cast<const float4*>(f.C32 + (size_t)jb2 * f.d + cc));
            dota = fmaf(xv[t].x, ca.x, fmaf(xv[t].y, ca.y, fmaf(xv[t].z, ca.z, fmaf(xv[t].w, ca.w, dota))));
            dotb = fmaf(xv[t].x, cb.x, fmaf(xv[t].y, cb.y, fmaf(xv[t].z, cb.z, fmaf(xv[t].w, cb.w, dotb))));
          }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          dota += __shfl_xor_sync(0xffffffffu, dota, o);
          dotb += __shfl_xor_sync(0xffffffffu, dotb, o);
        }
        const float da = fmaf(-2.f, dota, f.cnorm[ja]);
        if (da < best) { best = da; bj = ja; }
        ++ncand;
        if (jb >= 0) {
          const float db = fmaf(-2.f, dotb, f.cnorm[jb]);
          if (db < best) { best = db; bj = jb; }
          ++ncand;
        }
      }
    }
    if (lane == 0) {
      ent->y = bj;
      if (f.labels_out != nullptr) f.labels_out[row] = bj;
    }
    if (f.need_cost) {   // exact min distance sum (x - c)^2, as the update role computes it for the other rows
      float s2 = 0.f;
#pragma unroll
      for (int t = 0; t < 2; ++t) {
        const int cc = lane * 4 + 128 * t;
        if (cc < f.d) {
          const float4 cv = __ldg(reinterpret_cast<const float4*>(f.C32 + (size_t)bj * f.d + cc));
          const float dx = xv[t].x - cv.x, dy = xv[t].y - cv.y, dz = xv[t].z - cv.z, dw = xv[t].w - cv.w;
          s2 = fmaf(dx, dx, fmaf(dy, dy, fmaf(dz, dz, fmaf(dw, dw, s2))));
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s2 += __shfl_xor_sync(0xffffffffu, s2, o);
      if (lane == 0) {
        if (f.mind_out != nullptr) f.mind_out[row] = s2;
        cost += (double)s2;
      }
    }
  }
  if (lane == 0) cost_w[warp] = cost;
  __syncthreads();
  if (threadIdx.x == 0) {
    double c = 0.0;
    for (int w2 = 0; w2 < FIX_WARPS; ++w2) c += cost_w[w2];
    f.cost_out[blockIdx.x] = c;
  }
  if (f.rstat != nullptr && lane == 0 && ncand != 0ull) atomicAdd(f.rstat + 1, ncand);
}

// One CTA per cluster, thread = column: scans the segments in order, compacts the rows labelled with its cluster into
// shared memory (list order) and adds them with eight row loads in flight — the order of the additions is a fixed
// function of the data (segments in CTA order, entries in tile order), hence deterministic.
constexpr int ACC_CH = 1024;   // entries per scan step (4 per thread)
constexpr int FIX_SLOTS = 4;   // partial-sum slots of the deferred rows: slot q takes the segments p = q (mod 4)
__global__ void __launch_bounds__(256) k_fix_accum_t(const FixArgs f) {
  if (f.st != nullptr && f.st->done) return;
  __shared__ int buf[ACC_CH];
  __shared__ int wsum[8];
  const int j = (int)blockIdx.x;
  const int slot = (int)blockIdx.y;
  const int tid = (int)threadIdx.x, warp = tid >> 5, lane = tid & 31;
  float acc = 0.f;
  int cnt = 0;
  for (int p = slot; p < f.nseg; p += FIX_SLOTS) {
    const int c = f.count[p];
    const int2* seg = f.list + (size_t)p * (size_t)f.seg_cap;
    for (int e0 = 0; e0 < c; e0 += ACC_CH) {
      const int eb = e0 + tid * 4;
      int2 en[4];
      if (eb + 3 < c) {   // 32 contiguous bytes (segment bases are 256-byte aligned)
        const int4 a0 = *reinterpret_cast<const int4*>(seg + eb);
        const int4 a1 = *reinterpret_cast<const int4*>(seg + eb + 2);
        en[0] = make_int2(a0.x, a0.y);
        en[1] = make_int2(a0.z, a0.w);
        en[2] = make_int2(a1.x, a1.y);
        en[3] = make_int2(a1.z, a1.w);
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q) en[q] = eb + q < c ? seg[eb + q] : make_int2(-1, -1);
      }
      int mine = 0;
#pragma unroll
      for (int q = 0; q < 4; ++q) mine += en[q].y == j ? 1 : 0;
      int incl = mine;   // inclusive scan over the warp, then over the 8 warps
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
      }
      if (lane == 31) wsum[warp] = incl;
      __syncthreads();
      int off = incl - mine, total = 0;
#pragma unroll
      for (int w8 = 0; w8 < 8; ++w8) {
        const int v = wsum[w8];
        if (w8 < warp) off += v;
        total += v;
      }
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (en[q].y == j) buf[off++] = en[q].x;
      __syncthreads();
      if (tid < f.d) {
        const float* xc = f.X + tid;
        for (int q = 0; q < total; q += 16) {
          float v[16];
#pragma unroll
          for (int u = 0; u < 16; ++u) v[u] = q + u < total ? __ldg(xc + (size_t)buf[q + u] * f.d) : 0.f;
#pragma unroll
          for (int u = 0; u < 16; ++u) acc += v[u];
        }
      }
      cnt += total;
      __syncthreads();
    }
  }
  if (tid < f.d) f.partial[((size_t)slot * f.k + j) * f.d + tid] = acc;
  if (tid == 0) f.counts_out[(size_t)slot * f.k + j] = cnt;
  if (tid == 0 && j == 0 && slot == 0 && f.st_w != nullptr && f.rstat != nullptr) {
    f.st_w->fix_rows_cum = f.rstat[0];    // complete: the main kernel and k_fix_labels_t have finished
    f.st_w->fix_cands_cum = f.rstat[1];
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
struct TLayout {
  size_t off_ct, off_cnorm, off_thr, off_rstat, off_partials, off_counts, off_cost, off_xnorm, off_fixlist,
      off_fixmask, off_fixcnt, total;
  int nseg, seg_cap, mask_cap;
};
TLayout t_layout(const B2kFusedPlan& p, int64_t n, int k, int d) {
  auto al = [](size_t v) { return (v + 255) / 256 * 256; };
  TLayout L{};
  size_t o = 0;
  L.off_ct = o; o = al(o + (size_t)256 * p.DP * 4);
  L.off_cnorm = o; o = al(o + 512 * 4);
  L.off_thr = o; o = al(o + 16);
  L.off_rstat = o; o = al(o + 16);
  L.off_partials = o; o = al(o + (size_t)p.P * k * d * 4);
  L.off_counts = o; o = al(o + (size_t)p.P * k * 4);
  L.off_cost = o; o = al(o + (size_t)p.Pc * 8);
  L.off_xnorm = o; o = al(o + (size_t)(n > 0 ? n : 1) * 8);
  // deferred-row segments (one per CTA): a CTA can defer every row it sees; candidate masks for the first 1/4 of a
  // segment (entries beyond that are decided against every cluster)
  L.nseg = p.grid;
  const int64_t ntiles = (n + TN - 1) / TN;
  const int64_t nit_max = (ntiles + L.nseg - 1) / L.nseg;
  L.seg_cap = (int)(nit_max * TN);
  L.mask_cap = (int)std::min<int64_t>(L.seg_cap, ((nit_max + 3) / 4) * TN);
  L.off_fixlist = o; o = al(o + (size_t)L.nseg * L.seg_cap * 8);
  L.off_fixmask = o; o = al(o + (size_t)L.nseg * L.mask_cap * 32);
  L.off_fixcnt = o; o = al(o + (size_t)L.nseg * 4);
  L.total = o;
  return L;
}
}  // namespace

bool b2k_fused_t_supported(const b2k_ctx* ctx, int64_t n, int d, int k, const float* X) {
  (void)ctx;
  if (n < 1 || n > (int64_t)0x7fffff00 * 1LL) return false;
  if (d % 4 != 0 || d > 256 || k > 256) return false;
  if ((reinterpret_cast<uintptr_t>(X) & 15u) != 0) return false;
  return true;
}

int b2k_fused_t_plan(b2k_ctx* ctx, int64_t n, int d, int k, B2kFusedPlan* plan) {
  plan->variant = 1;
  plan->KP = 256;
  plan->DP = d <= 128 ? 128 : 256;
  const int64_t ntiles = (n + TN - 1) / TN;
  // whole clusters of WG_CL CTAs (the Lloyd pass sums in clusters); CTAs past the last tile run empty steps
  int grid = ctx->sm_count;
  if (ctx->grid_limit > 0 && ctx->grid_limit < grid) grid = ctx->grid_limit;
  if (ntiles < grid) grid = (int)ntiles;
  grid = grid / WG_CL * WG_CL;
  if (grid < WG_CL) grid = WG_CL;
  plan->grid = grid;
  plan->P = grid / WG_CL + FIX_SLOTS;   // one slot per cluster + the deferred rows' slots (k_fix_accum_t)
  plan->Pc = grid + 8 * ctx->sm_count;        // cost partials: one per CTA + one per k_fix_labels_t CTA
  plan->scratch_bytes = t_layout(*plan, n, k, d).total;
  return B2K_OK;
}

void b2k_fused_t_views(const B2kFusedPlan& plan, void* plan_scratch, int64_t n, int k, int d, float** partials,
                       int32_t** counts, double** cost_partials, unsigned long long** rstat) {
  TLayout L = t_layout(plan, n, k, d);
  char* b = static_cast<char*>(plan_scratch);
  *partials = reinterpret_cast<float*>(b + L.off_partials);
  *counts = reinterpret_cast<int32_t*>(b + L.off_counts);
  *cost_partials = reinterpret_cast<double*>(b + L.off_cost);
  if (rstat) *rstat = reinterpret_cast<unsigned long long*>(b + L.off_rstat);
}

static bool xnorm_in_scope(const b2k_ctx* ctx, const float* X, int64_t n, int d) {
  return ctx->xnorm_scope_X != nullptr && ctx->xnorm_scope_X == X && ctx->xnorm_scope_n == n && ctx->xnorm_scope_d == d;
}

// once per fit / lloyd / assign call: row norms of X into the plan scratch (or, inside b2k_kmeans_fit, once per fit into
// the context's cache); clears the recheck counters
int b2k_fused_t_prepare(b2k_ctx* ctx, const B2kFusedPlan& plan, void* plan_scratch, const float* X, int64_t n, int d,
                        int k, cudaStream_t s) {
  TLayout L = t_layout(plan, n, k, d);
  char* b = static_cast<char*>(plan_scratch);
  B2K_CUDA_OK(ctx, cudaMemsetAsync(b + L.off_rstat, 0, 16, s));
  int blocks = ctx->sm_count * 8;
  float2* dst = reinterpret_cast<float2*>(b + L.off_xnorm);
  if (xnorm_in_scope(ctx, X, n, d)) {   // inside one b2k_kmeans_fit: one norms pass for all of its passes over X
    if (ctx->xnorm_cache_rows < n) {
      if (ctx->xnorm_cache) cudaFree(ctx->xnorm_cache);
      ctx->xnorm_cache = nullptr;
      ctx->xnorm_cache_rows = 0;
      B2K_CUDA_OK(ctx, cudaMalloc(&ctx->xnorm_cache, (size_t)n * sizeof(float2)));
      ctx->xnorm_cache_rows = n;
      ctx->xnorm_cache_valid = 0;
    }
    if (ctx->xnorm_cache_valid) return B2K_OK;
    dst = static_cast<float2*>(ctx->xnorm_cache);
    ctx->xnorm_cache_valid = 1;
  }
  k_row_norms<<<blocks, 256, 0, s>>>(X, n, d, dst);
  ctx->stats.kernel_launches++;
  B2K_CUDA_OK(ctx, cudaGetLastError());
  return B2K_OK;
}

int b2k_launch_fused_t(b2k_ctx* ctx, const B2kFusedPlan& plan, void* plan_scratch, const float* X, int64_t n, int d,
                       const float* C, int k, int32_t* labels_out, float* mindist_out, bool do_update, bool need_cost,
                       const B2kLoopState* st, cudaStream_t s, const double* prev_counts) {
  (void)prev_counts;
  if (ctx->profile_fused)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "profile_fused: this build records no per-role profile");
  TLayout L = t_layout(plan, n, k, d);
  if (L.nseg > FIX_MAXP) return b2k_fail(ctx, B2K_ERR_STATE, "fused_t: more CTAs than the fix-up kernel indexes");
  char* b = static_cast<char*>(plan_scratch);
  float* Ct = reinterpret_cast<float*>(b + L.off_ct);
  float* cnorm = reinterpret_cast<float*>(b + L.off_cnorm);
  float* thr = reinterpret_cast<float*>(b + L.off_thr);
  int32_t* labels = labels_out;

  k_prep_centers_t<<<32, 256, 0, s>>>(C, k, d, plan.DP, Ct, cnorm, st);
  k_tables_t<<<1, 256, 0, s>>>(k, cnorm, thr, st);
  ctx->stats.kernel_launches += 2;
  B2K_CUDA_OK(ctx, cudaGetLastError());

  CUtensorMap mx, mc;
  B2K_TRY(b2k_fused_encode_2d(ctx, &mx, X, (uint64_t)d, (uint64_t)n, (uint64_t)d * 4, CHUNK, TN, 1));
  B2K_TRY(b2k_fused_encode_2d(ctx, &mc, Ct, (uint64_t)plan.DP, 256, (uint64_t)plan.DP * 4, CHUNK, 256, 0));

  WgArgs a{};
  a.n = n;
  a.ntiles = (int)((n + TN - 1) / TN);
  a.k = k;
  a.d = d;
  a.cnorm = cnorm;
  a.labels_out = labels;
  a.mind_out = mindist_out;
  a.cost_partials = reinterpret_cast<double*>(b + L.off_cost);
  a.st = st;
  a.X = X;
  a.C32 = C;
  a.thr = thr;
  a.xnorm = (xnorm_in_scope(ctx, X, n, d) && ctx->xnorm_cache_valid) ? static_cast<const float2*>(ctx->xnorm_cache)
                                                                      : reinterpret_cast<const float2*>(b + L.off_xnorm);
  a.fix_list = reinterpret_cast<int2*>(b + L.off_fixlist);
  a.fix_masks = reinterpret_cast<uint32_t*>(b + L.off_fixmask);
  a.fix_count = reinterpret_cast<int32_t*>(b + L.off_fixcnt);
  a.seg_cap = L.seg_cap;
  a.mask_cap = L.mask_cap;
  a.rstat = reinterpret_cast<unsigned long long*>(b + L.off_rstat);
  a.partials = reinterpret_cast<float*>(b + L.off_partials);
  a.counts = reinterpret_cast<int32_t*>(b + L.off_counts);

  const int rc = plan.DP == 128 ? b2k_launch_wg<256, 4, false>(ctx, plan.grid, mx, mc, mc, a, need_cost, do_update, s)
                                : b2k_launch_wg<256, 8, false>(ctx, plan.grid, mx, mc, mc, a, need_cost, do_update, s);
  B2K_TRY(rc);
  ctx->stats.kernel_launches++;
  ctx->stats.fused_tc_launches++;

  // the deferred rows: exact labels (+ min distance / cost)
  FixArgs f{};
  f.X = X;
  f.n = n;
  f.d = d;
  f.k = k;
  f.C32 = C;
  f.cnorm = cnorm;
  f.list = a.fix_list;
  f.masks = a.fix_masks;
  f.count = a.fix_count;
  f.nseg = L.nseg;
  f.seg_cap = L.seg_cap;
  f.mask_cap = L.mask_cap;
  f.labels_out = labels;
  f.mind_out = mindist_out;
  f.need_cost = need_cost ? 1 : 0;
  f.cost_out = a.cost_partials + plan.grid;
  f.rstat = a.rstat;
  f.partial = a.partials + (size_t)(plan.P - FIX_SLOTS) * k * d;
  f.counts_out = a.counts + (size_t)(plan.P - FIX_SLOTS) * k;
  f.st = st;
  f.st_w = const_cast<B2kLoopState*>(st);
  k_fix_labels_t<<<plan.Pc - plan.grid, FIX_WARPS * 32, 0, s>>>(f);
  ctx->stats.kernel_launches++;
  B2K_CUDA_OK(ctx, cudaGetLastError());
  if (do_update) {   // the deferred rows' contribution to the sums (the last FIX_SLOTS slots)
    k_fix_accum_t<<<dim3((unsigned)k, FIX_SLOTS), 256, 0, s>>>(f);
    ctx->stats.kernel_launches++;
    B2K_CUDA_OK(ctx, cudaGetLastError());
  }
  return B2K_OK;
}
