// Fused assign kernel for sm_90a (H100): wgmma (tf32) distances + argmin, ONE pass over X per launch.  Shared by the two
// shape families (included inside the anonymous namespace of b2k_fused_tc.cu and b2k_fused_t.cu after b2k_ptx.cuh; their
// common host side — shape rules, plan, dispatch, TMA descriptors — is b2k_fused.cu):
//
//   THREE = true  (k <= 128, d <= 128): "3xTF32".  Each consumer thread loads its wgmma A fragments from the X slot,
//                 splits them in registers into x = hi + lo (both round-to-nearest tf32) and accumulates
//                 lo.Chi^T + hi.Clo^T + hi.Chi^T (A from registers): fp32-class dot products.  The centres stay
//                 resident in shared memory when WgCfg::CRES.  argmin in index order with strict '<'
//                 (lowest index wins ties) -> labels (+ min distance ||x||^2 + min_j (||c_j||^2 - 2 x.c_j), cost).
//   THREE = false (k <= 256, d <= 256): 1xTF32 screening + exact recheck (b2k_fused_t.cu "Bound"): dist' of every
//                 centre is packed with its index into an ordered 32-bit key; rows whose two best keys are closer than
//                 the proven bound thr(x) are DEFERRED to the CTA's segment of a fix-up list together with a bit mask
//                 of every centre within thr of the best (k_fix_labels_t decides them exactly).  Other rows get their
//                 label (+ exact min distance sum (x - c)^2 in assign / inertia passes).
//
// UPD (THREE only, Lloyd passes): the same pass also forms the per-cluster sums.  The tile's X chunks stay in shared
// memory until its sums are formed (the A operands are register copies) while the producer fills the next tile's
// slots.  All 8 consumer warps update every tile together: a counting sort orders the 128 rows by (label, row), and
// each warp adds whole runs of equal labels (lane = 4 columns, one 16-byte unit of a row) in registers and then into
// the CTA's shared-memory sums S[KP][DP].  Every sum is formed in a fixed order (deterministic, no atomics); the CTA
// writes S to its partial slot when it ends.  For k or d > 128 (THREE = false) the sums ([256][256] f32 = 256 KB) do
// not fit beside a tile in one CTA, so the kernel runs in clusters of WG_CL = 8 CTAs: after each step every CTA sums
// the centres [32 r, 32 r + 32) over the 8 tiles of the cluster, reading the peers' labels and X rows through
// distributed shared memory (cluster-scope mbarriers order the hand-offs); deferred rows are added by k_fix_accum_t.
// Either way a Lloyd step reads X once.
//
// Roles: warp 8 (of a producer warpgroup) issues TMA into two rings guarded by mbarriers: X chunks [128 rows x 32 f32] (SX slots) and the matching
// centre chunk(s) [KP x 32 f32] (SC stages), all with 128-byte swizzle = K-major GMMA operands.  Warps 0-7 are two
// consumer warpgroups; warpgroup g owns rows [64 g, 64 g + 64) of every 128-row tile and keeps D[64 x KP] in registers
// (KP / 2 per thread).  Persistent grid, static round-robin over tiles: every output is a fixed function of the data.
constexpr int WG_TM = B2K_FUSED_TILE_ROWS;          // rows per tile (two warpgroups x wgmma M = 64)
constexpr int WG_CHUNK = 32;                        // f32 per 128-byte swizzle row = one TMA box / 4 wgmma K steps
constexpr int WG_XBYTES = WG_TM * WG_CHUNK * 4;     // 16 KB: one X slot
constexpr int WG_NTHREADS = 384;                    // 8 consumer warps + a producer warpgroup (one warp issues)
constexpr int WG_SMEM_LIMIT = 227 * 1024;
constexpr int WG_MISC = 7680;   // barriers, ||c||^2, ||x||^2, labels, flag counts, cost, row order, cluster row list
constexpr int WG_M_CNORM = 256, WG_M_XN = 1280, WG_M_LAB = 1792, WG_M_FLAG = 2816, WG_M_COST = 2880, WG_M_SRT = 2944,
              WG_M_LIST = 3584;
// THREE: barriers, ||c||^2 [KP], ||x||^2 [128] (NC) or the row order [128] (UPD) in one area, per-warp label counts
// [8][KP] u8 (UPD), cost
constexpr int WG_MISC3 = 2368;
constexpr int WG_M3_XN = 768, WG_M3_SRT = 768, WG_M3_HIST = 1280, WG_M3_COST = 2304;
constexpr int WG_CL = 8;   // THREE = false, UPD: CTAs per cluster; CTA r sums centres [r KP / 8, (r + 1) KP / 8)
// PROF builds: per-warp cycle counters [grid][WG_NTHREADS / 32][WG_NPROF].  Each mark charges the cycles since the
// previous mark to one phase, so a warp's counters sum to its whole run.  Consumer warps: X wait, centre wait, hand-off
// wait, A load + split, MMA issue + drain, epilogue, sort, column sums.  Producer warp: X slot wait, centre stage wait,
// issue (slot 2).
constexpr int WG_NPROF = 8;
enum { WG_P_WX, WG_P_WC, WG_P_HAND, WG_P_SPLIT, WG_P_MMA, WG_P_EPI, WG_P_SORT, WG_P_SUMS };

template <int KP, int NCH, bool THREE, bool UPD>
struct WgCfg {
  static_assert(KP % 16 == 0 && KP >= 16 && KP <= 256, "KP");
  static_assert(!UPD || !THREE || (KP <= 128 && NCH <= 4), "3xTF32 covers k, d <= 128");
  static constexpr int SROWS = THREE ? KP : KP / WG_CL;     // centres whose sums this CTA keeps
  static constexpr int DP = NCH * WG_CHUNK;
  static constexpr int NB = THREE ? 2 : 1;                  // centre operands per chunk: (hi, lo) or tf32
  static constexpr int CBYTES = KP * WG_CHUNK * 4;          // one centre chunk (multiple of 1 KB)
  static constexpr int CSTAGE = NB * CBYTES;
  static constexpr int MISC = THREE ? WG_MISC3 : WG_MISC;
  static constexpr int SUM_BYTES = UPD ? SROWS * DP * 4 + SROWS * 4 : 0;   // S[SROWS][DP] f32 + counts[SROWS]
  static constexpr int FIXED = SUM_BYTES + MISC;
  static constexpr int XMIN = UPD ? NCH : 2;                            // UPD holds a whole tile until its update
  // THREE: the centres stay resident (all NCH chunks, loaded once per CTA) when the X ring still holds XRES slots: a
  // Lloyd pass sums tile t while the next tile's slots fill, so it wants two tiles of slots
  static constexpr int XRES = UPD ? 2 * NCH : 2;
  static constexpr bool CRES = THREE && (WG_SMEM_LIMIT - FIXED - NCH * CSTAGE) / WG_XBYTES >= XRES;
  // else a ring of centre stages: two when the X ring still holds XMIN slots, else one
  static constexpr int SC = CRES ? 1 : (WG_SMEM_LIMIT - FIXED - 2 * CSTAGE) / WG_XBYTES >= XMIN ? 2 : 1;
  static constexpr int C_BYTES = CRES ? NCH * CSTAGE : SC * CSTAGE;
  static constexpr int SX_RAW = (WG_SMEM_LIMIT - FIXED - C_BYTES) / WG_XBYTES;
  static constexpr int SX = SX_RAW > 12 ? 12 : SX_RAW;
  static_assert(SX >= XMIN && 2 * (SX + SC) * 8 + 16 <= WG_M_CNORM, "ring");
  static constexpr int OFF_X = 0;
  static constexpr int OFF_C = SX * WG_XBYTES;
  static constexpr int OFF_SUM = OFF_C + C_BYTES;
  static constexpr int OFF_MISC = OFF_SUM + (THREE ? (SUM_BYTES + 7) & ~7 : (SUM_BYTES + 1023) & ~1023);
  static constexpr int SMEM_BYTES = OFF_MISC + MISC;
  static_assert(SMEM_BYTES <= WG_SMEM_LIMIT, "smem");
  static_assert(!THREE || WG_M_CNORM + KP * 4 <= WG_M3_XN, "misc");
  static_assert(!THREE || WG_M3_HIST + 8 * KP <= WG_M3_COST, "misc");
};
// BASELINE cfg2's Lloyd pass (k = 64, d = 128) keeps its centres resident: the fixed areas must leave it 8 X slots
static_assert(WgCfg<64, 4, true, true>::CRES, "cfg2 centres no longer resident");

struct WgArgs {
  int64_t n;
  int ntiles;
  int k;
  int d;
  const float* cnorm;           // [KP] ||c||^2, +inf for padding centres
  int32_t* labels_out;          // [n] or NULL
  float* mind_out;              // [n] or NULL
  double* cost_partials;        // [grid]
  float* partials;              // UPD: [grid][k][d] per-CTA sums
  int32_t* counts;              // UPD: [grid][k]
  const B2kLoopState* st;
  // THREE = false only
  const float* X;               // [n][d] (exact min distance of assign / inertia passes)
  const float* C32;             // [k][d] fp32 centres
  const float* thr;             // [4] coefficients of the recheck bound
  const float2* xnorm;          // [n] {||x||, ||x - trunc_tf32(x)||}
  int2* fix_list;               // CTA b appends {row, -1} to fix_list[b * seg_cap ..] in tile order
  uint32_t* fix_masks;          // [grid][mask_cap][8] candidate masks of the first mask_cap entries
  int32_t* fix_count;           // [grid]
  int seg_cap;
  int mask_cap;
  unsigned long long* rstat;    // [2] deferred rows (this kernel), candidates evaluated (k_fix_labels_t) or NULL
  long long* prof;              // PROF: [grid][WG_NTHREADS / 32][WG_NPROF] cycles
};

// merge two (smallest, second smallest) pairs of disjoint key sets
__device__ __forceinline__ void wg_merge2(uint32_t& a1, uint32_t& a2, uint32_t b1, uint32_t b2) {
  const uint32_t lo = min(a1, b1), hi = max(a1, b1);
  a2 = min(hi, min(a2, b2));
  a1 = lo;
}

template <int KP, int NCH, bool THREE, bool NC, bool UPD, bool PROF = false>
__global__ void __launch_bounds__(WG_NTHREADS, 1)
k_wg_assign(const __grid_constant__ CUtensorMap mapX, const __grid_constant__ CUtensorMap mapC0,
            const __grid_constant__ CUtensorMap mapC1, const WgArgs args) {
  using G = WgCfg<KP, NCH, THREE, UPD>;
  constexpr int R = KP / 2;   // accumulator registers per thread
  constexpr int DP = G::DP;
  if (args.st != nullptr && args.st->done) return;

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t base = smem_u32(smem_raw);
  if ((base & 1023u) != 0u) {   // 128B-swizzle atoms (TMA boxes, GMMA descriptors) need 1 KB alignment
    if (threadIdx.x == 0) printf("b2k wgmma: dynamic shared memory base %u is not 1 KB aligned\n", base);
    __trap();
  }
  uint8_t* misc = smem_raw + G::OFF_MISC;
  const uint32_t bars = base + G::OFF_MISC;
  float* cnorm_s = reinterpret_cast<float*>(misc + WG_M_CNORM);
  float* xn_s = reinterpret_cast<float*>(misc + WG_M3_XN);                             // [128] ||x||^2 (THREE, NC)
  int32_t* lab_s = reinterpret_cast<int32_t*>(misc + WG_M_LAB);   // THREE = false: [2][128] labels, -1 = deferred / invalid
  uint8_t* hist_s = misc + WG_M3_HIST;                             // THREE && UPD: [8][KP] rows of each label per warp
  int32_t* flag_s = reinterpret_cast<int32_t*>(misc + WG_M_FLAG);                      // [2][8] deferred rows per warp
  double* cost_s = reinterpret_cast<double*>(misc + (THREE ? WG_M3_COST : WG_M_COST)); // [8]
  uint32_t* srt_s = reinterpret_cast<uint32_t*>(misc + (THREE ? WG_M3_SRT : WG_M_SRT)); // [128] (label << 16 | row) in (label, row) order
  float* sum_s = reinterpret_cast<float*>(smem_raw + G::OFF_SUM); // UPD: [KP][DP] sums, then [KP] counts
  int32_t* cnt_s = reinterpret_cast<int32_t*>(sum_s + G::SROWS * DP);
  uint32_t* list_s = reinterpret_cast<uint32_t*>(misc + WG_M_LIST);  // [8 * 128] cluster rows (centre, CTA, row)
  auto xfull = [&](int s) -> uint32_t { return bars + 8u * (uint32_t)s; };
  auto xempty = [&](int s) -> uint32_t { return bars + 8u * (uint32_t)(G::SX + s); };
  auto cfull = [&](int s) -> uint32_t { return bars + 8u * (uint32_t)(2 * G::SX + s); };
  auto cempty = [&](int s) -> uint32_t { return bars + 8u * (uint32_t)(2 * G::SX + G::SC + s); };
  constexpr bool CLU = UPD && !THREE;   // cluster update through distributed shared memory
  const uint32_t ready_bar = bars + 8u * (uint32_t)(2 * G::SX + 2 * G::SC);   // CLU: the cluster's labels of a step
  const uint32_t done_bar = ready_bar + 8u;                                     // CLU: the cluster has read my step

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  long long pc[WG_NPROF] = {};
  long long tp = PROF ? clock64() : 0;
  auto mark = [&](int ph) {
    if constexpr (PROF) {
      const long long t = clock64();
      pc[ph] += t - tp;
      tp = t;
    }
  };
  auto prof_store = [&]() {
    if constexpr (PROF) {
      long long* o = args.prof + ((size_t)blockIdx.x * (WG_NTHREADS / 32) + warp) * WG_NPROF;
      for (int i = 0; i < WG_NPROF; ++i) o[i] = pc[i];
    }
  };
  if (threadIdx.x == 0) {
    for (int s = 0; s < G::SX; ++s) {
      mbar_init(xfull(s), 1);
      mbar_init(xempty(s), 8);   // every consumer warp releases the slot
    }
    for (int s = 0; s < G::SC; ++s) {
      mbar_init(cfull(s), 1);
      mbar_init(cempty(s), 8);
    }
    if constexpr (CLU) {
      mbar_init(ready_bar, WG_CL);
      mbar_init(done_bar, WG_CL);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int j = threadIdx.x; j < KP; j += WG_NTHREADS) cnorm_s[j] = args.cnorm[j];
  if constexpr (UPD) {
    for (int i = threadIdx.x; i < G::SROWS * DP + G::SROWS; i += WG_NTHREADS) sum_s[i] = 0.f;   // counts: 0 bits
  }
  __syncthreads();
  uint32_t crank = 0;
  if constexpr (CLU) {
    crank = cluster_ctarank();
    cluster_sync_all();   // every CTA's barriers are initialised before the first remote arrival
  }

  // CLU: every CTA of a cluster runs the step count of its first CTA (the largest); a tile past the end is all
  // out-of-range rows (TMA zero-fills it, no row is valid)
  const int b0 = (int)blockIdx.x - (int)crank;
  const int nit = b0 < args.ntiles ? (args.ntiles - 1 - b0) / (int)gridDim.x + 1 : 0;

  if (warp >= 8) {
    // ======================= TMA producer =======================
    // k = d = 256: the producer warpgroup hands registers to the consumers (D[64 x 256] is 128 per thread)
    if constexpr (!THREE) asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp == 8 && elect_one()) {
      tma_prefetch_desc(&mapX);
      tma_prefetch_desc(&mapC0);
      if constexpr (THREE) tma_prefetch_desc(&mapC1);
      if constexpr (G::CRES) {   // every centre chunk, once
        mbar_expect_tx(cfull(0), (uint32_t)(NCH * G::CSTAGE));
        for (int c = 0; c < NCH; ++c) {
          const uint32_t cst = base + (uint32_t)(G::OFF_C + c * G::CSTAGE);
          tma_load_2d(cst, &mapC0, cfull(0), c * WG_CHUNK, 0);
          tma_load_2d(cst + G::CBYTES, &mapC1, cfull(0), c * WG_CHUNK, 0);
        }
      }
      for (int it = 0; it < nit; ++it) {
        const int tile = (int)blockIdx.x + it * (int)gridDim.x;
#pragma unroll 1
        for (int c = 0; c < NCH; ++c) {
          const int q = it * NCH + c;
          const int xs = q % G::SX, cs = q % G::SC;
          mark(WG_P_HAND);
          mbar_wait_nocall(xempty(xs), (uint32_t)((q / G::SX) & 1) ^ 1u);
          mark(WG_P_WX);
          mbar_expect_tx(xfull(xs), (uint32_t)WG_XBYTES);
          tma_load_2d(base + (uint32_t)(G::OFF_X + xs * WG_XBYTES), &mapX, xfull(xs), c * WG_CHUNK, tile * WG_TM);
          if constexpr (!G::CRES) {
            mark(WG_P_HAND);
            mbar_wait_nocall(cempty(cs), (uint32_t)((q / G::SC) & 1) ^ 1u);
            mark(WG_P_WC);
            const uint32_t cst = base + (uint32_t)(G::OFF_C + cs * G::CSTAGE);
            mbar_expect_tx(cfull(cs), (uint32_t)G::CSTAGE);
            tma_load_2d(cst, &mapC0, cfull(cs), c * WG_CHUNK, 0);
            if constexpr (THREE) tma_load_2d(cst + G::CBYTES, &mapC1, cfull(cs), c * WG_CHUNK, 0);
          }
        }
      }
      mark(WG_P_HAND);
      prof_store();
    }
    __syncwarp();
  } else {
    // ======================= consumer warpgroups =======================
    if constexpr (!THREE) asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    const int g = warp >> 2, wi = warp & 3, tw = threadIdx.x & 127;
    float acc[R];
#pragma unroll
    for (int i = 0; i < R; ++i) acc[i] = 0.f;
    double cost = 0.0;
    int seg_cnt = 0;                 // THREE = false: deferred rows of this CTA so far (same in every consumer thread)
    unsigned long long n_flag = 0;
    float thr0 = 0.f, thr1 = 0.f, thr2 = 0.f, thr3 = 0.f;
    if constexpr (!THREE) {
      thr0 = args.thr[0];
      thr1 = args.thr[1];
      thr2 = args.thr[2];
      thr3 = args.thr[3];
    }
    if constexpr (THREE) {
      // A fragments straight from the swizzled X slot: this thread holds rows ar and ar + 8 of the tile (ar = 64 g +
      // 16 wi + lane / 4, so both rows are lane / 4 modulo 8, which selects the 16-byte unit swizzle) and columns
      // lane % 4 and lane % 4 + 4 of each k step of 8
      const uint32_t arow = (uint32_t)(g * 64 + wi * 16 + (lane >> 2)) * 128u + (uint32_t)(lane & 3) * 4u;
      const uint32_t asw = (uint32_t)(lane >> 2);
      // one wgmma group in flight across chunks needs two chunks' A fragments (32 registers each) and a second centre
      // stage; at KP = 128 the accumulators take 64 registers and two chunks' fragments no longer fit
      constexpr bool PIPE = (G::CRES || G::SC > 1) && KP < 128;
      if constexpr (G::CRES) {
        mark(WG_P_EPI);
        if (nit > 0) mbar_wait_nocall(cfull(0), 0u);
        mark(WG_P_WC);
      }
      for (int it = 0; it < nit; ++it) {
        const int tile = (int)blockIdx.x + it * (int)gridDim.x;
        float xnp[4] = {0.f, 0.f, 0.f, 0.f};   // NC: partial ||x||^2 of rows (tw >> 3) + 16 i
#pragma unroll
        for (int c = 0; c < NCH; ++c) {
          const int q = it * NCH + c;
          const int xsl = q % G::SX, csl = q % G::SC;
          const uint32_t xs = base + (uint32_t)(G::OFF_X + xsl * WG_XBYTES);
          const uint32_t cs = base + (uint32_t)(G::OFF_C + (G::CRES ? c : csl) * G::CSTAGE);
          const uint8_t* xp = smem_raw + G::OFF_X + xsl * WG_XBYTES;
          mark(WG_P_EPI);
          mbar_wait_nocall(xfull(xsl), (uint32_t)((q / G::SX) & 1));
          mark(WG_P_WX);
          if constexpr (NC) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const float4 v = lds128(xs + (uint32_t)(g * (WG_XBYTES / 2) + (tw + 128 * i) * 16));
              xnp[i] = fmaf(v.w, v.w, fmaf(v.z, v.z, fmaf(v.y, v.y, fmaf(v.x, v.x, xnp[i]))));
            }
          }
          // x = hi + lo, hi = RN_tf32(x), lo = RN_tf32(x - hi), in registers
          uint32_t ah[WG_CHUNK / 8][4], al[WG_CHUNK / 8][4];
#pragma unroll
          for (int ks = 0; ks < WG_CHUNK / 8; ++ks) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {   // row ar + 8 (e & 1), column 8 ks + lane % 4 + 4 (e >> 1)
              const uint32_t unit = (uint32_t)(2 * ks + (e >> 1));
              const float v = *reinterpret_cast<const float*>(xp + arow + (uint32_t)(e & 1) * 1024u + ((unit ^ asw) << 4));
              ah[ks][e] = rn_tf32_bits(v);
              al[ks][e] = rn_tf32_bits(v - __uint_as_float(ah[ks][e]));
            }
          }
#pragma unroll
          for (int ks = 0; ks < WG_CHUNK / 8; ++ks) {   // every fragment is formed before the wgmma fence
            reg_fence(ah[ks]);
            reg_fence(al[ks]);
          }
          if constexpr (!UPD) {
            __syncwarp();
            if (lane == 0) mbar_arrive(xempty(xsl));   // the operands are in registers: X is no longer read
          }
          mark(WG_P_SPLIT);
          if constexpr (!G::CRES) {
            mbar_wait_nocall(cfull(csl), (uint32_t)((q / G::SC) & 1));
            mark(WG_P_WC);
          }
          wgmma_fence();
#pragma unroll
          for (int ks = 0; ks < WG_CHUNK / 8; ++ks) {
            const uint64_t db = make_kmajor_sw128_desc(cs + ks * 32);
            const uint64_t dbl = make_kmajor_sw128_desc(cs + G::CBYTES + ks * 32);
            wgmma_tf32_rs<KP>(acc, al[ks], db, (c | ks) != 0 ? 1u : 0u);   // small terms first
            wgmma_tf32_rs<KP>(acc, ah[ks], dbl, 1u);
            wgmma_tf32_rs<KP>(acc, ah[ks], db, 1u);
          }
          wgmma_commit();
          if constexpr (PIPE) {
            // one group stays in flight: loading and splitting the next chunk overlaps this chunk's MMAs
            wgmma_wait1();
            if constexpr (!G::CRES) {
              if (c > 0) {
                __syncwarp();
                if (lane == 0) mbar_arrive(cempty((q - 1) % G::SC));
              }
            }
          } else {
            wgmma_wait0();
            if constexpr (!G::CRES) {
              __syncwarp();
              if (lane == 0) mbar_arrive(cempty(csl));
            }
          }
          mark(WG_P_MMA);
        }
        wgmma_wait0();
        if constexpr (PIPE && !G::CRES) {
          __syncwarp();
          if (lane == 0) mbar_arrive(cempty((it * NCH + NCH - 1) % G::SC));
        }
        reg_fence(acc);
        mark(WG_P_MMA);

        // ---- epilogue: thread holds rows rr0 and rr0 + 8 of the tile, columns 8 a + 2 (lane & 3) + e ----
        const int rr0 = g * 64 + wi * 16 + (lane >> 2);
        if constexpr (NC) {
#pragma unroll
          for (int i = 0; i < 4; ++i) {   // the 8 lanes of a row group hold one row's 8 float4 units
            float v = xnp[i];
            v += __shfl_xor_sync(0xffffffffu, v, 1);
            v += __shfl_xor_sync(0xffffffffu, v, 2);
            v += __shfl_xor_sync(0xffffffffu, v, 4);
            if ((lane & 7) == 0) xn_s[g * 64 + (tw >> 3) + 16 * i] = v;
          }
          asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory");
        }
        float best[2] = {__int_as_float(0x7f800000), __int_as_float(0x7f800000)};
        int bj[2] = {0, 0};
#pragma unroll
        for (int i = 0; i < R; ++i) {
          const int h = (i >> 1) & 1;
          const int j = (i >> 2) * 8 + 2 * (lane & 3) + (i & 1);
          const float dist = fmaf(-2.f, acc[i], cnorm_s[j]);
          if (dist < best[h]) { best[h] = dist; bj[h] = j; }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int o = 1; o <= 2; o <<= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best[h], o);
            const int oj = __shfl_xor_sync(0xffffffffu, bj[h], o);
            if (ob < best[h] || (ob == best[h] && oj < bj[h])) { best[h] = ob; bj[h] = oj; }
          }
          const int64_t grow = (int64_t)tile * WG_TM + rr0 + 8 * h;
          if ((lane & 3) == 0) {
            if (grow < args.n) {
              if (args.labels_out != nullptr) args.labels_out[grow] = bj[h];
              if constexpr (NC) {
                const float md = fmaxf(xn_s[rr0 + 8 * h] + best[h], 0.f);
                if (args.mind_out != nullptr) args.mind_out[grow] = md;
                cost += (double)md;
              }
            }
          }
        }
        mark(WG_P_EPI);
        if constexpr (UPD) {
          // ---- per-cluster sums of the tile, from its X chunks still in shared memory, by all 8 consumer warps.  A
          // counting sort puts the valid rows in (label, row) order; each warp then adds whole runs of equal labels.
          // Rows past n take no part.  Every warp passes the first barrier of tile it + 1 only after its sums of tile
          // it, so the read-modify-writes of a row of S stay in tile order, and the counts and the row order are
          // rewritten only after every warp has read them. ----
          // (1) this warp's rows 16 warp + 8 h + q are held by lanes 4 q + h (h < 2); per label: how many, and the
          // rank of each row among them in row order
          const int hq = lane & 3;
          const int64_t grow0 = (int64_t)tile * WG_TM + rr0;
          const uint32_t key = hq == 0   ? (grow0 < args.n ? (uint32_t)bj[0] : (uint32_t)KP)
                               : hq == 1 ? (grow0 + 8 < args.n ? (uint32_t)bj[1] : (uint32_t)KP)
                                         : 0x10000u + (uint32_t)lane;   // lanes 2, 3 of a quad match no other lane
          const bool own = hq < 2 && key < (uint32_t)KP;
          const uint32_t mk = __match_any_sync(0xffffffffu, key);
          const uint32_t lt = (1u << lane) - 1u;
          const int wr = hq == 0 ? __popc(mk & 0x11111111u & lt) : __popc(mk & 0x11111111u) + __popc(mk & 0x22222222u & lt);
          uint8_t* hist = hist_s + warp * KP;
          if (lane < KP / 4) reinterpret_cast<uint32_t*>(hist)[lane] = 0u;
          __syncwarp();
          if (own && wr == 0) hist[key] = (uint8_t)__popc(mk & 0x33333333u);
          mark(WG_P_SORT);
          asm volatile("bar.sync 3, 256;" ::: "memory");   // every warp's counts of the tile
          mark(WG_P_HAND);
          // (2) rank = rows of smaller labels + rows of the same label in lower warps + wr.  Lane j holds labels
          // 4 j .. 4 j + 3 as packed bytes: no byte exceeds the 128 rows of a tile, so the packed sums do not carry.
          uint32_t tot = 0u, pre = 0u;
          if (lane < KP / 4) {
#pragma unroll
            for (int w = 0; w < 8; ++w) {
              const uint32_t v = reinterpret_cast<const uint32_t*>(hist_s + w * KP)[lane];
              tot += v;
              if (w < warp) pre += v;
            }
          }
          const int lsum = (int)((tot * 0x01010101u) >> 24);
          int incl = lsum;
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
          }
          const int nv = __shfl_sync(0xffffffffu, incl, 31);   // valid rows of the tile
          const uint32_t first = tot * 0x01010100u + (uint32_t)(incl - lsum) * 0x01010101u + pre;
          const uint32_t fb = __shfl_sync(0xffffffffu, first, (int)(key >> 2) & 31);
          if (own) srt_s[((fb >> (8 * (key & 3u))) & 0xffu) + (uint32_t)wr] = (key << 16) | (uint32_t)(rr0 + 8 * hq);
          mark(WG_P_SORT);
          asm volatile("bar.sync 3, 256;" ::: "memory");   // row order complete
          mark(WG_P_HAND);
          // (3) warp w adds the runs that start at sorted positions [16 w, 16 w + 16): positions [p0, p1)
          int p0 = 128, p1 = 128;
          {
            const uint4 e4 = *reinterpret_cast<const uint4*>(srt_s + 4 * lane);   // positions 4 lane + i
            const uint32_t ev[4] = {e4.x, e4.y, e4.z, e4.w};
            uint32_t prev = __shfl_up_sync(0xffffffffu, e4.w >> 16, 1);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int p = 4 * lane + i;
              const uint32_t l = ev[i] >> 16;
              if (p < nv && (p == 0 || l != prev)) {
                if (p >= 16 * warp && p0 == 128) p0 = p;
                if (p >= 16 * warp + 16 && p1 == 128) p1 = p;
              }
              prev = l;
            }
            p0 = min(__reduce_min_sync(0xffffffffu, p0), nv);
            p1 = min(__reduce_min_sync(0xffffffffu, p1), nv);
          }
          // lane owns columns 4 lane .. 4 lane + 3: 16-byte unit lane % 8 (swizzled by row % 8) of chunk lane / 8
          const bool act = lane < DP / 4;
          const uint8_t* xbase = smem_raw + G::OFF_X + ((it * NCH + (act ? lane >> 3 : 0)) % G::SX) * WG_XBYTES;
          const uint32_t unit = (uint32_t)(lane & 7);
          float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
          int cur = -1, run = 0;
          auto flush = [&]() {   // one run: S[cur] += a, count += run length
            if (act) {
              float4* sp = reinterpret_cast<float4*>(sum_s + cur * DP) + lane;
              float4 s = *sp;
              s.x += a.x;
              s.y += a.y;
              s.z += a.z;
              s.w += a.w;
              *sp = s;
            }
            if (lane == 0) cnt_s[cur] += run;
          };
#pragma unroll 1
          for (int i0 = p0; i0 < p1; i0 += 8) {   // 8 rows' loads in flight, then the adds in row order
            uint32_t e[8];
            float4 x[8];
#pragma unroll
            for (int v = 0; v < 8; ++v) e[v] = i0 + v < p1 ? srt_s[i0 + v] : 0xffffffffu;
#pragma unroll
            for (int v = 0; v < 8; ++v) {
              const uint32_t r = e[v] & 127u;
              x[v] = *reinterpret_cast<const float4*>(xbase + r * 128u + ((unit ^ (r & 7u)) << 4));
            }
#pragma unroll
            for (int v = 0; v < 8; ++v) {
              if (e[v] == 0xffffffffu) break;
              const int l = (int)(e[v] >> 16);
              if (l != cur) {
                if (cur >= 0) flush();
                cur = l;
                a = make_float4(0.f, 0.f, 0.f, 0.f);
                run = 0;
              }
              a.x += x[v].x;
              a.y += x[v].y;
              a.z += x[v].z;
              a.w += x[v].w;
              ++run;
            }
          }
          if (cur >= 0) flush();
          __syncwarp();
          if (lane == 0) {   // this warp no longer reads the tile's X slots
#pragma unroll
            for (int c = 0; c < NCH; ++c) mbar_arrive(xempty((it * NCH + c) % G::SX));
          }
          mark(WG_P_SUMS);
        }
      }
    } else {
      for (int it = 0; it < nit; ++it) {
        const int tile = (int)blockIdx.x + it * (int)gridDim.x;
        int prev_q = -1;                         // chunk whose wgmma group may still be in flight
#pragma unroll 1
        for (int c = 0; c < NCH; ++c) {
          const int q = it * NCH + c;
          const int xsl = q % G::SX, csl = q % G::SC;
          const uint32_t xs = base + (uint32_t)(G::OFF_X + xsl * WG_XBYTES + g * (WG_XBYTES / 2));   // my 64 rows
          const uint32_t cs = base + (uint32_t)(G::OFF_C + csl * G::CSTAGE);
          mbar_wait_nocall(xfull(xsl), (uint32_t)((q / G::SX) & 1));
          mbar_wait_nocall(cfull(csl), (uint32_t)((q / G::SC) & 1));
          wgmma_fence();
#pragma unroll
          for (int ks = 0; ks < WG_CHUNK / 8; ++ks) {
            const uint64_t da = make_kmajor_sw128_desc(xs + ks * 32);
            const uint64_t db = make_kmajor_sw128_desc(cs + ks * 32);
            const uint32_t sd = (c | ks) != 0 ? 1u : 0u;
            wgmma_tf32<KP>(acc, da, db, sd);
          }
          wgmma_commit();
          // X slots of an updating pass stay until the tile's sums are formed
          if constexpr (G::SC == 1) {
            // the only centre stage is needed by the next chunk: this chunk's group must complete
            wgmma_wait0();
            __syncwarp();
            if (lane == 0) {
              mbar_arrive(cempty(csl));
              if constexpr (!UPD) mbar_arrive(xempty(xsl));
            }
          } else {
            // one group stays in flight: the previous chunk's operands are released while this one runs
            wgmma_wait1();
            if (prev_q >= 0) {
              __syncwarp();
              if (lane == 0) {
                if constexpr (!UPD) mbar_arrive(xempty(prev_q % G::SX));
                mbar_arrive(cempty(prev_q % G::SC));
              }
            }
            prev_q = q;
          }
        }
        if constexpr (G::SC > 1) {
          wgmma_wait0();
          __syncwarp();
          if (lane == 0) {
            if constexpr (!UPD) mbar_arrive(xempty(prev_q % G::SX));
            mbar_arrive(cempty(prev_q % G::SC));
          }
        }
        reg_fence(acc);

        // ---- epilogue: thread holds rows rr0 and rr0 + 8 of the tile, columns 8 a + 2 (lane & 3) + e ----
        const int rr0 = g * 64 + wi * 16 + (lane >> 2);
        // keys: (dist' + ||x||^2 + thr) is a positive float, so its bits order like an unsigned integer; the low 8 bits
        // carry the centre index
        float thr[2], xoff[2];
        bool valid[2];
        int64_t grow[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          grow[h] = (int64_t)tile * WG_TM + rr0 + 8 * h;
          valid[h] = grow[h] < args.n;
          const float2 xq = valid[h] ? __ldg(args.xnorm + grow[h]) : make_float2(0.f, 0.f);
          thr[h] = fmaf(xq.y, thr0, fmaf(xq.x, fmaf(xq.x, thr2, thr1), thr3));
          xoff[h] = fmaf(xq.x, xq.x, thr[h]);
        }
        uint32_t m1[2] = {0xffffffffu, 0xffffffffu}, m2[2] = {0xffffffffu, 0xffffffffu};
#pragma unroll
        for (int i = 0; i < R; ++i) {
          const int h = (i >> 1) & 1;
          const int j = (i >> 2) * 8 + 2 * (lane & 3) + (i & 1);
          const float dist = fmaf(-2.f, acc[i], cnorm_s[j]) + xoff[h];
          const uint32_t key = (__float_as_uint(dist) & 0xffffff00u) | (uint32_t)j;
          wg_merge2(m1[h], m2[h], key, 0xffffffffu);
        }
        bool flag[2];
        int label[2];
        float T[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int o = 1; o <= 2; o <<= 1) {
            const uint32_t r1 = __shfl_xor_sync(0xffffffffu, m1[h], o), r2 = __shfl_xor_sync(0xffffffffu, m2[h], o);
            wg_merge2(m1[h], m2[h], r1, r2);
          }
          label[h] = (int)(m1[h] & 255u);
          const float M1f = __uint_as_float(m1[h] & 0xffffff00u);
          flag[h] = valid[h] && (__uint_as_float(m2[h] & 0xffffff00u) - M1f) < thr[h];
          T[h] = M1f + thr[h];
        }
        const uint32_t b0 = __ballot_sync(0xffffffffu, flag[0] && (lane & 3) == 0);
        const uint32_t b1 = __ballot_sync(0xffffffffu, flag[1] && (lane & 3) == 0);
        const int pb = it & 1;
        if (lane == 0) flag_s[pb * 8 + warp] = __popc(b0) + __popc(b1);
        if ((lane & 3) == 0) {
#pragma unroll
          for (int h = 0; h < 2; ++h) lab_s[pb * WG_TM + rr0 + 8 * h] = (valid[h] && !flag[h]) ? label[h] : -1;
        }
        // candidate masks: every centre whose key lies within thr of the best (a superset of the exact argmin set)
        uint32_t mk[2][KP / 32];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int w = 0; w < KP / 32; ++w) mk[h][w] = 0u;
        if (__any_sync(0xffffffffu, flag[0] || flag[1])) {
#pragma unroll
          for (int i = 0; i < R; ++i) {
            const int h = (i >> 1) & 1;
            const int j = (i >> 2) * 8 + 2 * (lane & 3) + (i & 1);
            const float dist = fmaf(-2.f, acc[i], cnorm_s[j]) + xoff[h];
            if (__uint_as_float(__float_as_uint(dist) & 0xffffff00u) <= T[h]) mk[h][i >> 4] |= 1u << (j & 31);
          }
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int w = 0; w < KP / 32; ++w) {
              mk[h][w] |= __shfl_xor_sync(0xffffffffu, mk[h][w], 1);
              mk[h][w] |= __shfl_xor_sync(0xffffffffu, mk[h][w], 2);
            }
        }
        asm volatile("bar.sync 3, 256;" ::: "memory");   // flag counts and labels of the tile (both warpgroups)
        int pre = 0, total = 0;
#pragma unroll
        for (int w = 0; w < 8; ++w) {
          const int v = flag_s[pb * 8 + w];
          if (w < warp) pre += v;
          total += v;
        }
        if ((lane & 3) == 0) {
          const uint32_t lt = (1u << lane) - 1u;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (flag[h]) {
              const int e = seg_cnt + pre + (h == 0 ? __popc(b0 & lt) : __popc(b0) + __popc(b1 & lt));
              args.fix_list[(size_t)blockIdx.x * (size_t)args.seg_cap + e] = make_int2((int)grow[h], -1);
              if (e < args.mask_cap) {
                uint32_t* dst = args.fix_masks + ((size_t)blockIdx.x * (size_t)args.mask_cap + (size_t)e) * 8u;
#pragma unroll
                for (int w = 0; w < 8; ++w) dst[w] = w < KP / 32 ? mk[h][w < KP / 32 ? w : 0] : 0u;
              }
              ++n_flag;
            } else if (valid[h] && args.labels_out != nullptr) {
              args.labels_out[grow[h]] = label[h];
            }
          }
        }
        seg_cnt += total;
        if constexpr (CLU) {
          // ---- per-cluster sums over the 8 tiles of the cluster's step: this CTA owns centres [crank * SR, + SR) and
          // reads the peers' labels and X rows through distributed shared memory; the deferred rows (label -1) are
          // added by k_fix_accum_t ----
          constexpr int SR = G::SROWS;
          const uint32_t par = (uint32_t)(it & 1);
          if (threadIdx.x == 0) {
            for (int r = 0; r < WG_CL; ++r) mbar_arrive_remote(ready_bar, (uint32_t)r);
          }
          mbar_wait_cluster_nocall(ready_bar, par);
          // the row list, in (source CTA, row) order: consumer warp w scans the labels of CTA w
          const uint32_t lab_src = mapa_u32(smem_u32(lab_s + pb * WG_TM), (uint32_t)warp);
          uint32_t m[4];
          int rel[4], n_my = 0;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int l = ld_cluster_s32(lab_src + 4u * (uint32_t)(lane + 32 * i));
            rel[i] = l - (int)crank * SR;
            m[i] = __ballot_sync(0xffffffffu, l >= 0 && (unsigned)rel[i] < (unsigned)SR);
            n_my += __popc(m[i]);
          }
          if (lane == 0) srt_s[warp] = (uint32_t)n_my;
          asm volatile("bar.sync 3, 256;" ::: "memory");
          int lpos = 0, ltot = 0;
#pragma unroll
          for (int w = 0; w < 8; ++w) {
            const int v = (int)srt_s[w];
            if (w < warp) lpos += v;
            ltot += v;
          }
          const uint32_t lt = (1u << lane) - 1u;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            if ((m[i] >> lane) & 1u)
              list_s[lpos + __popc(m[i] & lt)] = ((uint32_t)rel[i] << 16) | ((uint32_t)warp << 7) | (uint32_t)(lane + 32 * i);
            lpos += __popc(m[i]);
          }
          asm volatile("bar.sync 3, 256;" ::: "memory");
          if (threadIdx.x < DP) {   // thread = column: the rows of each centre added in list order (deterministic)
            const int col = threadIdx.x;
            const uint32_t coff = base + (uint32_t)(G::OFF_X + ((it * NCH + col / WG_CHUNK) % G::SX) * WG_XBYTES + (col % 4) * 4);
            const uint32_t unit = (uint32_t)((col % WG_CHUNK) / 4);
#pragma unroll 1
            for (int i0 = 0; i0 < ltot; i0 += 8) {   // 8 remote loads in flight, then the adds in order
              uint32_t e[8];
              float x[8];
#pragma unroll
              for (int u = 0; u < 8; ++u) e[u] = i0 + u < ltot ? list_s[i0 + u] : 0xffffffffu;
#pragma unroll
              for (int u = 0; u < 8; ++u) {
                const uint32_t row = e[u] & 127u, src = (e[u] >> 7) & 7u;
                x[u] = e[u] != 0xffffffffu ? ld_cluster_f32(mapa_u32(coff + row * 128u + ((unit ^ (row & 7u)) << 4), src))
                                           : 0.f;
              }
#pragma unroll
              for (int u = 0; u < 8; ++u) {
                if (e[u] == 0xffffffffu) continue;
                const int l = (int)(e[u] >> 16);
                sum_s[l * DP + col] += x[u];
                if (col == 0) cnt_s[l] += 1;
              }
            }
          }
          asm volatile("bar.sync 3, 256;" ::: "memory");   // this CTA has read the cluster's step
          if (threadIdx.x == 0) {
            for (int r = 0; r < WG_CL; ++r) mbar_arrive_remote(done_bar, (uint32_t)r);
          }
          mbar_wait_cluster_nocall(done_bar, par);          // ... and every peer has read mine
          __syncwarp();
          if (lane == 0) {
#pragma unroll 1
            for (int c = 0; c < NCH; ++c) mbar_arrive(xempty((it * NCH + c) % G::SX));
          }
        }
        if constexpr (NC) {
          // exact min distance sum (x - c)^2 of the decided rows (k_fix_labels_t handles the deferred ones)
#pragma unroll 1
          for (int r2 = 0; r2 < 16; ++r2) {
            const int row = warp * 16 + r2;
            const int lab = lab_s[pb * WG_TM + row];
            if (lab < 0) continue;
            const int64_t gr = (int64_t)tile * WG_TM + row;
            float sacc = 0.f;
#pragma unroll
            for (int t = 0; t < 2; ++t) {
              const int cc = lane * 4 + 128 * t;
              if (cc < args.d) {
                const float4 xv = __ldg(reinterpret_cast<const float4*>(args.X + (size_t)gr * args.d + cc));
                const float4 cv = __ldg(reinterpret_cast<const float4*>(args.C32 + (size_t)lab * args.d + cc));
                const float dx = xv.x - cv.x, dy = xv.y - cv.y, dz = xv.z - cv.z, dw = xv.w - cv.w;
                sacc = fmaf(dx, dx, fmaf(dy, dy, fmaf(dz, dz, fmaf(dw, dw, sacc))));
              }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) sacc += __shfl_xor_sync(0xffffffffu, sacc, o);
            if (lane == 0) {
              if (args.mind_out != nullptr) args.mind_out[gr] = sacc;
              cost += (double)sacc;
            }
          }
        }
      }
    }
    // per-CTA cost: fixed-order fold (lanes, then the 8 warps after the final barrier)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cost += __shfl_xor_sync(0xffffffffu, cost, o);
    if (lane == 0) cost_s[warp] = cost;
    mark(WG_P_EPI);
    if (lane == 0) prof_store();
    if constexpr (!THREE) {
      if (threadIdx.x == 0) args.fix_count[blockIdx.x] = seg_cnt;
      if (args.rstat != nullptr) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) n_flag += __shfl_xor_sync(0xffffffffu, n_flag, o);
        if (lane == 0 && n_flag != 0ull) atomicAdd(args.rstat + 0, n_flag);
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double c = 0.0;
    for (int w = 0; w < 8; ++w) c += cost_s[w];
    args.cost_partials[blockIdx.x] = c;
  }
  if constexpr (UPD && THREE) {
    const int kd = args.k * args.d;
    float* out = args.partials + (size_t)blockIdx.x * kd;
    for (int i = threadIdx.x; i < kd; i += WG_NTHREADS) out[i] = sum_s[(i / args.d) * DP + i % args.d];
    for (int l = threadIdx.x; l < args.k; l += WG_NTHREADS) args.counts[(size_t)blockIdx.x * args.k + l] = cnt_s[l];
  }
  if constexpr (CLU) {   // partial slot of the cluster, rows [crank * SROWS, + SROWS)
    const size_t slot = (size_t)(blockIdx.x / WG_CL);
    const int l0 = (int)crank * G::SROWS;
    const int nl = min(G::SROWS, args.k - l0);
    for (int i = threadIdx.x; i < nl * args.d; i += WG_NTHREADS)
      args.partials[(slot * args.k + l0) * args.d + i] = sum_s[(i / args.d) * DP + i % args.d];
    for (int l = threadIdx.x; l < nl; l += WG_NTHREADS) args.counts[slot * args.k + l0 + l] = cnt_s[l];
    cluster_sync_all();
  }
}

// a.prof != NULL selects the PROF instantiation (THREE only)
template <int KP, int NCH, bool THREE>
int b2k_launch_wg(b2k_ctx* ctx, int grid, const CUtensorMap& mx, const CUtensorMap& m0, const CUtensorMap& m1,
                  const WgArgs& a, bool need_cost, bool do_update, cudaStream_t s) {
  int smem = 0;
  void (*kern)(CUtensorMap, CUtensorMap, CUtensorMap, WgArgs) = nullptr;
  if (do_update) {
    kern = k_wg_assign<KP, NCH, THREE, false, true>;
    smem = WgCfg<KP, NCH, THREE, true>::SMEM_BYTES;
  } else {
    kern = need_cost ? k_wg_assign<KP, NCH, THREE, true, false> : k_wg_assign<KP, NCH, THREE, false, false>;
    smem = WgCfg<KP, NCH, THREE, false>::SMEM_BYTES;
  }
  if constexpr (THREE) {
    if (a.prof != nullptr) {
      kern = do_update ? k_wg_assign<KP, NCH, THREE, false, true, true>
             : need_cost ? k_wg_assign<KP, NCH, THREE, true, false, true>
                         : k_wg_assign<KP, NCH, THREE, false, false, true>;
    }
  }
  B2K_CUDA_OK(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  if (!THREE && do_update) {   // the update of the 1xTF32 family runs in clusters of WG_CL CTAs
    if (grid % WG_CL != 0) return b2k_fail(ctx, B2K_ERR_STATE, "fused kernel: grid is not a multiple of the cluster size");
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(WG_NTHREADS);
    cfg.dynamicSmemBytes = (size_t)smem;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = WG_CL;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    B2K_CUDA_OK(ctx, cudaLaunchKernelEx(&cfg, kern, mx, m0, m1, a));
  } else {
    kern<<<grid, WG_NTHREADS, smem, s>>>(mx, m0, m1, a);
  }
  B2K_CUDA_OK(ctx, cudaGetLastError());
  return B2K_OK;
}
