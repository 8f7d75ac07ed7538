// The 3xTF32 pair-distance pipeline of the wgmma passes: exact k-NN (k_knn_wg, b2k_knn.cu) and DBSCAN (k_db_wg,
// b2k_dbscan.cu).  Included inside each translation unit's anonymous namespace, after b2k_ptx.cuh.
//
// A persistent CTA of PW_NTHREADS walks its units: a tile of PW_TM rows (the A operand, shifted as b2k_knn_prep.cuh
// describes) against a range of PW_N-row blocks of the tf32 hi/lo planes.  Warp 8 issues TMA: the unit's tile (NCH
// chunks, once per unit) and its blocks, chunk by chunk, hi and lo planes into a ring of PW_SC stages.  Consumer
// warpgroup g owns rows [64 g, 64 g + 64) of the tile; per block it accumulates lo.Xhi^T + hi.Xlo^T + hi.Xhi^T (A split
// in registers, as the 3xTF32 branch of k_wg_assign) into D[64 x 128].  Each kernel keeps its own epilogue.
// b2k_dbscan_bound proves DBSCAN's screen for exactly this split and this product order.

constexpr int PW_TM = B2K_KNN_WG_QROWS;   // rows per tile (two consumer warpgroups x wgmma M = 64)
constexpr int PW_N = B2K_KNN_WG_BLOCK;    // rows per block (wgmma N)
constexpr int PW_CHUNK = 32;              // f32 per 128-byte swizzle row
constexpr int PW_NTHREADS = 384;          // 8 consumer warps + a producer warpgroup (one warp issues)
constexpr int PW_SC = 2;                  // ring stages of (hi, lo)

// Shared memory: the tile, the ring, then OWN bytes of the kernel's own, then the barriers.
template <int NCH_, int OWN>
struct PairWgCfg {
  static constexpr int NCH = NCH_;
  static constexpr int QBYTES = PW_TM * PW_CHUNK * 4;   // one tile chunk: 16 KB
  static constexpr int CBYTES = PW_N * PW_CHUNK * 4;    // one block chunk plane: 16 KB
  static constexpr int OFF_Q = 0;
  static constexpr int OFF_C = OFF_Q + NCH * QBYTES;
  static constexpr int OFF_OWN = OFF_C + PW_SC * 2 * CBYTES;
  static constexpr int OFF_BAR = OFF_OWN + OWN;
  static constexpr int SMEM_BYTES = OFF_BAR + 8 * (2 + 2 * PW_SC);
  static_assert(OFF_C % 1024 == 0 && CBYTES % 1024 == 0, "swizzle atoms need 1 KB alignment");
  static_assert(SMEM_BYTES + 1024 <= 227 * 1024, "smem");
};

// the mbarriers: tile full / empty, then per ring stage chunk full, then chunk empty
struct PairWgBars {
  uint32_t bars;
  __device__ __forceinline__ uint32_t qfull() const { return bars; }
  __device__ __forceinline__ uint32_t qempty() const { return bars + 8u; }
  __device__ __forceinline__ uint32_t cfull(int s) const { return bars + 16u + 8u * (uint32_t)s; }
  __device__ __forceinline__ uint32_t cempty(int s) const { return bars + 16u + 8u * (uint32_t)(PW_SC + s); }
};

// every thread: checks the base alignment and initialises the barriers (thread 0), then the CTA barrier
template <class G>
__device__ __forceinline__ PairWgBars pair_wg_init(uint32_t base) {
  if ((base & 1023u) != 0u) __trap();   // 128B-swizzle atoms need a 1 KB aligned base
  const PairWgBars bars{base + G::OFF_BAR};
  if (threadIdx.x == 0) {
    mbar_init(bars.qfull(), 1);
    mbar_init(bars.qempty(), 8);
    for (int s = 0; s < PW_SC; ++s) {
      mbar_init(bars.cfull(s), 1);
      mbar_init(bars.cempty(s), 8);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  return bars;
}

// units of a CTA: the tile's first row in the tile operand and the unit's blocks [lo, hi)
struct PairWgUnit {
  int row0, lo, hi;
};

// The producer (one elected lane of warp 8): for it < nit, unit_of(it) -> PairWgUnit; blocks with skip(b) are not
// loaded.  Invariant: the consumers skip exactly the blocks skipped here.  Both sides count the ring's chunks in q, so a
// block skipped on one side only puts the ring's parities out of step and the kernel hangs.
template <class G, class UnitOf, class Skip>
__device__ __forceinline__ void pair_wg_produce(uint32_t base, PairWgBars bars, const CUtensorMap* mapQ,
                                                const CUtensorMap* mapHi, const CUtensorMap* mapLo, int nit,
                                                UnitOf unit_of, Skip skip) {
  tma_prefetch_desc(mapQ);
  tma_prefetch_desc(mapHi);
  tma_prefetch_desc(mapLo);
  int q = 0;
  for (int it = 0; it < nit; ++it) {
    const PairWgUnit un = unit_of(it);
    mbar_wait_nocall(bars.qempty(), (uint32_t)((it & 1) ^ 1));
    mbar_expect_tx(bars.qfull(), (uint32_t)(G::NCH * G::QBYTES));
    for (int c = 0; c < G::NCH; ++c)
      tma_load_2d(base + (uint32_t)(G::OFF_Q + c * G::QBYTES), mapQ, bars.qfull(), c * PW_CHUNK, un.row0);
    for (int b = un.lo; b < un.hi; ++b) {
      if (skip(b)) continue;
#pragma unroll 1
      for (int c = 0; c < G::NCH; ++c, ++q) {
        const int cs = q % PW_SC;
        mbar_wait_nocall(bars.cempty(cs), (uint32_t)((q / PW_SC) & 1) ^ 1u);
        const uint32_t dst = base + (uint32_t)(G::OFF_C + cs * 2 * G::CBYTES);
        mbar_expect_tx(bars.cfull(cs), (uint32_t)(2 * G::CBYTES));
        tma_load_2d(dst, mapHi, bars.cfull(cs), c * PW_CHUNK, b * PW_N);
        tma_load_2d(dst + G::CBYTES, mapLo, bars.cfull(cs), c * PW_CHUNK, b * PW_N);
      }
    }
  }
}

// A consumer thread's next block (after it has waited on qfull for the unit): acc = the 3xTF32 products of tile rows
// rr0 and rr0 + 8 with the block's rows.  acc[i] is row rr0 + 8 ((i >> 1) & 1), block column 8 (i >> 2) + 2 (lane & 3)
// + (i & 1).  q counts the ring's chunks across blocks and units.
template <class G>
__device__ __forceinline__ void pair_wg_block(const uint8_t* smem_raw, uint32_t base, PairWgBars bars, int rr0,
                                              int lane, float (&acc)[PW_N / 2], int& q) {
  const uint32_t arow = (uint32_t)rr0 * 128u + (uint32_t)(lane & 3) * 4u;
  const uint32_t asw = (uint32_t)(lane >> 2);
#pragma unroll
  for (int c = 0; c < G::NCH; ++c, ++q) {
    const int cs = q % PW_SC;
    const uint8_t* xp = smem_raw + G::OFF_Q + c * G::QBYTES;
    const uint32_t cst = base + (uint32_t)(G::OFF_C + cs * 2 * G::CBYTES);
    // v = hi + lo, hi = RN_tf32(v), lo = RN_tf32(v - hi), in registers
    uint32_t ah[PW_CHUNK / 8][4], al[PW_CHUNK / 8][4];
#pragma unroll
    for (int ks = 0; ks < PW_CHUNK / 8; ++ks) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {   // row rr0 + 8 (e & 1), column 8 ks + lane % 4 + 4 (e >> 1)
        const uint32_t unit = (uint32_t)(2 * ks + (e >> 1));
        const float v = *reinterpret_cast<const float*>(xp + arow + (uint32_t)(e & 1) * 1024u + ((unit ^ asw) << 4));
        ah[ks][e] = rn_tf32_bits(v);
        al[ks][e] = rn_tf32_bits(v - __uint_as_float(ah[ks][e]));
      }
    }
#pragma unroll
    for (int ks = 0; ks < PW_CHUNK / 8; ++ks) {
      reg_fence(ah[ks]);
      reg_fence(al[ks]);
    }
    mbar_wait_nocall(bars.cfull(cs), (uint32_t)((q / PW_SC) & 1));
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < PW_CHUNK / 8; ++ks) {
      const uint64_t dh = make_kmajor_sw128_desc(cst + ks * 32);
      const uint64_t dl = make_kmajor_sw128_desc(cst + G::CBYTES + ks * 32);
      wgmma_tf32_rs<PW_N>(acc, al[ks], dh, (c | ks) != 0 ? 1u : 0u);   // small terms first
      wgmma_tf32_rs<PW_N>(acc, ah[ks], dl, 1u);
      wgmma_tf32_rs<PW_N>(acc, ah[ks], dh, 1u);
    }
    wgmma_commit();
    wgmma_wait0();
    __syncwarp();
    if (lane == 0) mbar_arrive(bars.cempty(cs));
  }
  reg_fence(acc);
}

// ---- host ----
struct PairWgMaps {
  CUtensorMap q, hi, lo;
};

// tile operand rows [nq][d] (16-byte aligned) and the hi / lo planes [n_pad][DP] of b2k_knn_prep_launch
int pair_wg_maps(b2k_ctx* ctx, const float* Q, int64_t nq, int d, const float* Xhi, const float* Xlo, int64_t n_pad,
                 int DP, PairWgMaps* m) {
  B2K_TRY(b2k_encode_2d(ctx, &m->q, Q, (uint64_t)d, (uint64_t)nq, (uint64_t)d * 4, PW_CHUNK, PW_TM,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B));
  B2K_TRY(b2k_encode_2d(ctx, &m->hi, Xhi, (uint64_t)DP, (uint64_t)n_pad, (uint64_t)DP * 4, PW_CHUNK, PW_N,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B));
  B2K_TRY(b2k_encode_2d(ctx, &m->lo, Xlo, (uint64_t)DP, (uint64_t)n_pad, (uint64_t)DP * 4, PW_CHUNK, PW_N,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B));
  return B2K_OK;
}

// Launches the instance kern(std::integral_constant<int, NCH>()) for DP = 32 NCH (b2k_knn_wg_dp) on `grid` CTAs, with
// the shared memory of PairWgCfg<NCH, OWN>.
template <int OWN, class Kern, class Args>
int pair_wg_launch(b2k_ctx* ctx, int DP, Kern kern, int grid, const PairWgMaps& m, const Args& a, cudaStream_t s) {
  auto go = [&](auto nch) -> int {
    const int smem = PairWgCfg<decltype(nch)::value, OWN>::SMEM_BYTES;
    const auto k = kern(nch);
    B2K_CUDA_OK(ctx, cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    k<<<grid, PW_NTHREADS, smem, s>>>(m.q, m.hi, m.lo, a);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    return B2K_OK;
  };
  if (DP == 32) return go(std::integral_constant<int, 1>());
  if (DP == 64) return go(std::integral_constant<int, 2>());
  return go(std::integral_constant<int, 4>());
}
