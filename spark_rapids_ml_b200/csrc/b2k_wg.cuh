// Fused assign kernel for sm_90a (H100): wgmma (tf32) distances + argmin, ONE pass over X per launch.  Shared by the two
// shape families (included inside the anonymous namespace of b2k_fused_tc.cu and b2k_fused_t.cu after b2k_ptx.cuh):
//
//   THREE = true  (k <= 128, d <= 128): "3xTF32".  Each consumer warpgroup splits its 64 rows of an X chunk in shared
//                 memory into x = hi + lo (both round-to-nearest tf32, in split buffers) and accumulates
//                 lo.Chi^T + hi.Clo^T + hi.Chi^T: fp32-class dot products.  argmin in index order with strict '<'
//                 (lowest index wins ties) -> labels (+ min distance ||x||^2 + min_j (||c_j||^2 - 2 x.c_j), cost).
//   THREE = false (k <= 256, d <= 256): 1xTF32 screening + exact recheck (b2k_fused_t.cu "Bound"): dist' of every
//                 centre is packed with its index into an ordered 32-bit key; rows whose two best keys are closer than
//                 the proven bound thr(x) are DEFERRED to the CTA's segment of a fix-up list together with a bit mask
//                 of every centre within thr of the best (k_fix_labels_t decides them exactly).  Other rows get their
//                 label (+ exact min distance sum (x - c)^2 in assign / inertia passes).
//
// UPD (THREE only, Lloyd passes): the same pass also forms the per-cluster sums.  The tile's X chunks stay in shared
// memory until its labels are known (the A operands are copies: the hi / lo split buffers); the 128 rows are then
// ordered by (label, row), and the thread that owns column c adds each label's run of rows in registers and then into
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
constexpr int WG_TM = 128;                          // rows per tile (two warpgroups x wgmma M = 64)
constexpr int WG_CHUNK = 32;                        // f32 per 128-byte swizzle row = one TMA box / 4 wgmma K steps
constexpr int WG_XBYTES = WG_TM * WG_CHUNK * 4;     // 16 KB: one X slot
constexpr int WG_NTHREADS = 384;                    // 8 consumer warps + a producer warpgroup (one warp issues)
constexpr int WG_SMEM_LIMIT = 227 * 1024;
constexpr int WG_MISC = 7680;   // barriers, ||c||^2, ||x||^2, labels, flag counts, cost, row order, cluster row list
constexpr int WG_M_CNORM = 256, WG_M_XN = 1280, WG_M_LAB = 1792, WG_M_FLAG = 2816, WG_M_COST = 2880, WG_M_SRT = 2944,
              WG_M_LIST = 3584;
constexpr int WG_CL = 8;        // THREE = false, UPD: CTAs per cluster; CTA r sums centres [r KP / 8, (r + 1) KP / 8)

template <int KP, int NCH, bool THREE, bool UPD>
struct WgCfg {
  static_assert(KP % 16 == 0 && KP >= 16 && KP <= 256, "KP");
  static_assert(!UPD || !THREE || (KP <= 128 && NCH <= 4), "3xTF32 covers k, d <= 128");
  static constexpr int SROWS = THREE ? KP : KP / WG_CL;     // centres whose sums this CTA keeps
  static constexpr int DP = NCH * WG_CHUNK;
  static constexpr int NB = THREE ? 2 : 1;                  // centre operands per chunk: (hi, lo) or tf32
  static constexpr int CBYTES = KP * WG_CHUNK * 4;          // one centre chunk (multiple of 1 KB)
  static constexpr int CSTAGE = NB * CBYTES;
  static constexpr int HL_BYTES = THREE ? 2 * WG_XBYTES : 0;            // hi and lo split of one chunk (both warpgroups)
  static constexpr int SUM_BYTES = UPD ? SROWS * DP * 4 + SROWS * 4 : 0;   // S[SROWS][DP] f32 + counts[SROWS]
  static constexpr int FIXED = HL_BYTES + SUM_BYTES + WG_MISC;
  static constexpr int XMIN = UPD ? NCH : 2;                            // UPD holds a whole tile until its update
  // two centre stages when the X ring still holds XMIN slots, else one
  static constexpr int SC = (WG_SMEM_LIMIT - FIXED - 2 * CSTAGE) / WG_XBYTES >= XMIN ? 2 : 1;
  static constexpr int SX_RAW = (WG_SMEM_LIMIT - FIXED - SC * CSTAGE) / WG_XBYTES;
  static constexpr int SX = SX_RAW > 12 ? 12 : SX_RAW;
  static_assert(SX >= XMIN && 2 * (SX + SC) * 8 + 16 <= WG_M_CNORM, "ring");
  static constexpr int OFF_X = 0;
  static constexpr int OFF_C = SX * WG_XBYTES;
  static constexpr int OFF_HL = OFF_C + SC * CSTAGE;
  static constexpr int OFF_SUM = OFF_HL + HL_BYTES;
  static constexpr int OFF_MISC = OFF_SUM + ((SUM_BYTES + 1023) & ~1023);
  static constexpr int SMEM_BYTES = OFF_MISC + WG_MISC;
  static_assert(SMEM_BYTES <= WG_SMEM_LIMIT, "smem");
};

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
};

// merge two (smallest, second smallest) pairs of disjoint key sets
__device__ __forceinline__ void wg_merge2(uint32_t& a1, uint32_t& a2, uint32_t b1, uint32_t b2) {
  const uint32_t lo = min(a1, b1), hi = max(a1, b1);
  a2 = min(hi, min(a2, b2));
  a1 = lo;
}

template <int KP, int NCH, bool THREE, bool NC, bool UPD>
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
  float* xn_s = reinterpret_cast<float*>(misc + WG_M_XN);         // [128] ||x||^2 (THREE)
  int32_t* lab_s = reinterpret_cast<int32_t*>(misc + WG_M_LAB);   // [2][128] labels, -1 = deferred / invalid
  int32_t* flag_s = reinterpret_cast<int32_t*>(misc + WG_M_FLAG); // [2][8] deferred rows per warp
  double* cost_s = reinterpret_cast<double*>(misc + WG_M_COST);   // [8]
  uint32_t* srt_s = reinterpret_cast<uint32_t*>(misc + WG_M_SRT); // [128] (label << 16 | row) in (label, row) order
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
      for (int it = 0; it < nit; ++it) {
        const int tile = (int)blockIdx.x + it * (int)gridDim.x;
#pragma unroll 1
        for (int c = 0; c < NCH; ++c) {
          const int q = it * NCH + c;
          const int xs = q % G::SX, cs = q % G::SC;
          mbar_wait_nocall(xempty(xs), (uint32_t)((q / G::SX) & 1) ^ 1u);
          mbar_expect_tx(xfull(xs), (uint32_t)WG_XBYTES);
          tma_load_2d(base + (uint32_t)(G::OFF_X + xs * WG_XBYTES), &mapX, xfull(xs), c * WG_CHUNK, tile * WG_TM);
          mbar_wait_nocall(cempty(cs), (uint32_t)((q / G::SC) & 1) ^ 1u);
          const uint32_t cst = base + (uint32_t)(G::OFF_C + cs * G::CSTAGE);
          mbar_expect_tx(cfull(cs), (uint32_t)G::CSTAGE);
          tma_load_2d(cst, &mapC0, cfull(cs), c * WG_CHUNK, 0);
          if constexpr (THREE) tma_load_2d(cst + G::CBYTES, &mapC1, cfull(cs), c * WG_CHUNK, 0);
        }
      }
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
    const uint32_t hi_s = base + (uint32_t)(G::OFF_HL + g * (WG_XBYTES / 2));
    const uint32_t lo_s = hi_s + (uint32_t)WG_XBYTES;
    for (int it = 0; it < nit; ++it) {
      const int tile = (int)blockIdx.x + it * (int)gridDim.x;
      float xnp[4] = {0.f, 0.f, 0.f, 0.f};   // THREE && NC: partial ||x||^2 of rows (tw >> 3) + 16 i
      int prev_q = -1;                         // THREE = false: chunk whose wgmma group may still be in flight
#pragma unroll 1
      for (int c = 0; c < NCH; ++c) {
        const int q = it * NCH + c;
        const int xsl = q % G::SX, csl = q % G::SC;
        const uint32_t xs = base + (uint32_t)(G::OFF_X + xsl * WG_XBYTES + g * (WG_XBYTES / 2));   // my 64 rows
        const uint32_t cs = base + (uint32_t)(G::OFF_C + csl * G::CSTAGE);
        mbar_wait_nocall(xfull(xsl), (uint32_t)((q / G::SX) & 1));
        uint32_t a_hi = xs, a_lo = xs;
        if constexpr (THREE) {
          // elementwise split (the swizzled layout is preserved): hi = RN_tf32(x), lo = RN_tf32(x - hi); X stays intact
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const uint32_t off = (uint32_t)(tw + 128 * i) * 16u;
            const float4 v = lds128(xs + off);
            if constexpr (NC) xnp[i] = fmaf(v.w, v.w, fmaf(v.z, v.z, fmaf(v.y, v.y, fmaf(v.x, v.x, xnp[i]))));
            float4 h, l;
            h.x = __uint_as_float(rn_tf32_bits(v.x));
            h.y = __uint_as_float(rn_tf32_bits(v.y));
            h.z = __uint_as_float(rn_tf32_bits(v.z));
            h.w = __uint_as_float(rn_tf32_bits(v.w));
            l.x = __uint_as_float(rn_tf32_bits(v.x - h.x));
            l.y = __uint_as_float(rn_tf32_bits(v.y - h.y));
            l.z = __uint_as_float(rn_tf32_bits(v.z - h.z));
            l.w = __uint_as_float(rn_tf32_bits(v.w - h.w));
            sts128(hi_s + off, h);
            sts128(lo_s + off, l);
          }
          fence_proxy_async();
          asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory");
          if constexpr (!UPD) {
            __syncwarp();
            if (lane == 0) mbar_arrive(xempty(xsl));   // the split buffers are the operands: X is no longer read
          }
          a_hi = hi_s;
          a_lo = lo_s;
        }
        mbar_wait_nocall(cfull(csl), (uint32_t)((q / G::SC) & 1));
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < WG_CHUNK / 8; ++ks) {
          const uint64_t da = make_kmajor_sw128_desc(a_hi + ks * 32);
          const uint64_t db = make_kmajor_sw128_desc(cs + ks * 32);
          const uint32_t sd = (c | ks) != 0 ? 1u : 0u;
          if constexpr (THREE) {
            const uint64_t dal = make_kmajor_sw128_desc(a_lo + ks * 32);
            const uint64_t dbl = make_kmajor_sw128_desc(cs + G::CBYTES + ks * 32);
            wgmma_tf32<KP>(acc, dal, db, sd);   // small terms first
            wgmma_tf32<KP>(acc, da, dbl, 1u);
            wgmma_tf32<KP>(acc, da, db, 1u);
          } else {
            wgmma_tf32<KP>(acc, da, db, sd);
          }
        }
        wgmma_commit();
        // X slots of an updating pass stay until the tile's sums are formed
        if constexpr (THREE || G::SC == 1) {
          // the split buffers / the only centre stage are needed by the next chunk: this chunk's group must complete
          wgmma_wait0();
          __syncwarp();
          if (lane == 0) {
            mbar_arrive(cempty(csl));
            if constexpr (!THREE && !UPD) mbar_arrive(xempty(xsl));
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
      if constexpr (!THREE && G::SC > 1) {
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
      if constexpr (THREE) {
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
            if constexpr (UPD) lab_s[rr0 + 8 * h] = grow < args.n ? bj[h] : -1;
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
        if constexpr (UPD) {
          // ---- per-cluster sums of the tile, from the X chunks still in shared memory ----
          asm volatile("bar.sync 3, 256;" ::: "memory");   // labels of all 128 rows
          if (threadIdx.x < WG_TM) {   // rank of row t in (label, row) order; rows past n sort last
            const int t = threadIdx.x;
            const int mine = lab_s[t] < 0 ? KP : lab_s[t];
            int rank = 0;
#pragma unroll 8
            for (int r = 0; r < WG_TM; ++r) {
              const int o = lab_s[r] < 0 ? KP : lab_s[r];
              rank += (o < mine || (o == mine && r < t)) ? 1 : 0;
            }
            srt_s[rank] = ((uint32_t)(mine < KP ? mine : 0xffff) << 16) | (uint32_t)t;
          }
          asm volatile("bar.sync 3, 256;" ::: "memory");   // row order complete
          if (threadIdx.x < DP) {
            const int col = threadIdx.x;
            // column col of row r: X slot of chunk col / 32, 16-B unit (col % 32) / 4 swizzled by r % 8
            const uint8_t* cbase = smem_raw + G::OFF_X + ((it * NCH + col / WG_CHUNK) % G::SX) * WG_XBYTES + (col % 4) * 4;
            const uint32_t unit = (uint32_t)((col % WG_CHUNK) / 4);
            int cur = -1, run = 0;
            float a = 0.f;
#pragma unroll 1
            for (int i0 = 0; i0 < WG_TM; i0 += 8) {   // 8 rows' loads in flight, then the adds in order
              uint32_t e[8];
              float x[8];
#pragma unroll
              for (int u = 0; u < 8; ++u) e[u] = srt_s[i0 + u];
#pragma unroll
              for (int u = 0; u < 8; ++u) {
                const uint32_t r = e[u] & 0xffffu;
                x[u] = *reinterpret_cast<const float*>(cbase + r * 128u + ((unit ^ (r & 7u)) << 4));
              }
#pragma unroll
              for (int u = 0; u < 8; ++u) {
                const int l = (int)(e[u] >> 16);
                if (l == 0xffff) continue;   // rows past n sort last
                if (l != cur) {
                  if (cur >= 0) {
                    sum_s[cur * DP + col] += a;
                    if (col == 0) cnt_s[cur] += run;
                  }
                  cur = l;
                  a = 0.f;
                  run = 0;
                }
                a += x[u];
                ++run;
              }
            }
            if (cur >= 0) {
              sum_s[cur * DP + col] += a;
              if (col == 0) cnt_s[cur] += run;
            }
          }
          asm volatile("bar.sync 3, 256;" ::: "memory");   // the tile's X slots and labels are consumed
          __syncwarp();
          if (lane == 0) {
#pragma unroll 1
            for (int c = 0; c < NCH; ++c) mbar_arrive(xempty((it * NCH + c) % G::SX));
          }
        }
      } else {
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
