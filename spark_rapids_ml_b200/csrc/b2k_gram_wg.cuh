// Gram matrix of the centred data on wgmma (sm_90a, 3xTF32): G = sum_rows (x - mu)^T (x - mu), the upper block triangle
// of 128 x 128 feature blocks.  Included inside the anonymous namespace of b2k_pca.cu (k_gram_wg) and of b2k_gmm.cu
// (k_gmm_gram_wg) after b2k_ptx.cuh; each defines its kernel over gram_wg_body.
//
// Weighted variant (W = true, Gaussian mixtures): G_c = sum_rows r_rc (x - mu)^T (x - mu) for each component c of a
// row weight table r [n][K] (fp64).  Each row's centred fp32 value is multiplied by fl32(sqrt(fl32(r_rc))) before the
// split, in both operands, so the product carries r_rc.  The grid is a multiple of K * ntile: CTA b owns component
// (b % (K ntile)) / ntile and tile b % ntile, so the K ntile CTAs of one p read the same row range at the same time and
// it is fetched from HBM about once per pass.  W = false is the unweighted pass above, unchanged.
//
// Work: tile t = (I, J), I <= J, is the product of feature block I (wgmma M, 64 per consumer warpgroup) and feature block
// J (wgmma N = 128); the contraction runs over rows.  The grid is a multiple of the tile count: CTA b owns tile
// b % ntile for its whole run and the row ranges p, p + P, p + 2P, ... (p = b / ntile, P = grid / ntile) of GW_RANGE rows
// each.  Every output is a fixed function of (n, d, grid): no atomics, bitwise reproducible.  CTAs of the same p read
// the same rows at the same time, so a row range is fetched from HBM about once and re-read from L2 by the other tiles.
//
// Layout.  tf32 wgmma takes only K-major shared-memory operands, and the contraction index here is the row, while X is
// row-major.  TMA brings [32 rows x 32 features] boxes (128-byte swizzle) of blocks I and J into a ring slot (one chunk =
// 32 rows).  Per chunk the 256 consumer threads read the slot, subtract mu, split x = hi + lo (both round-to-nearest
// tf32) and write hi and lo transposed into K-major 128B-swizzled operand buffers [128 features][32 rows] (block J -> B,
// block I -> A; a diagonal tile writes one block and uses it for both), then fence.proxy.async + a named barrier release
// the slot to the producer.  Two operand stages alternate, so a chunk's writes never meet the previous chunk's wgmma
// reads.  Each warpgroup then accumulates its 64 rows of block I: D += lo_I.hi_J + hi_I.lo_J + hi_I.hi_J, 4 k steps of
// 8 rows, both operands from shared memory.  (The A operand could come from registers, as in k_wg_assign; with the two
// 64-register accumulators below it would not fit the 168 registers a 3-warpgroup CTA gets without spilling.)
// Rows past n and features past d are zeroed by the consumers: TMA zero-fills the part of a box past the edge, but x - mu
// would not be 0, and a box that lies wholly past d is not loaded at all.
//
// Accuracy.  The tensor core adds into its fp32 accumulator with truncation, so its error grows linearly with the
// accumulation length.  Each chunk (32 rows, 12 wgmma) starts from a zero accumulator (scale_d = 0), is added in
// round-to-nearest fp32 into a second register accumulator, and that one is added into the CTA's fp64 partial every
// GW_RANGE rows.  The fp32 error is therefore bounded by 12 truncations plus GW_RANGE / 32 rounded additions, whatever n.
constexpr int GW_BLK = 128;                        // features per block
constexpr int GW_KC = 32;                          // rows per chunk: one 128-byte K-major row of the B operand
constexpr int GW_RANGE = 4096;                     // rows per work unit = fp64 flush interval
constexpr int GW_SX = 3;                           // X ring slots
constexpr int GW_NTHREADS = 288;                   // two consumer warpgroups + one TMA producer warp
constexpr int GW_XHALF = GW_KC * GW_BLK * 4;       // 16 KB: one block of a chunk, 4 boxes of [32 rows x 32 f32]
constexpr int GW_BOX = GW_KC * 32 * 4;             // 4 KB
constexpr int GW_XSLOT = 2 * GW_XHALF;             // blocks I and J
constexpr int GW_BBYTES = GW_BLK * GW_KC * 4;      // 16 KB: one K-major operand [128 features][32 rows]
constexpr int GW_OFF_OP = GW_SX * GW_XSLOT;        // 2 stages x (B hi, B lo, A hi, A lo)
constexpr int GW_OFF_MU = GW_OFF_OP + 8 * GW_BBYTES;
constexpr int GW_OFF_BAR = GW_OFF_MU + 2 * GW_BLK * 4;
constexpr int GW_SMEM = GW_OFF_BAR + 2 * GW_SX * 8;
static_assert(GW_SMEM + 1024 <= 227 * 1024, "smem");

struct GramArgs {
  int64_t n;
  int d;
  int nblk;          // feature blocks, ceil(d / 128)
  int ntile;         // nblk (nblk + 1) / 2
  int nrange;        // ceil(n / GW_RANGE)
  const float* mu;   // [nblk * 128] fp32 mean, 0 past d
  double* part;      // [grid][128][128] fp64 sums of the CTA's tile (rows of block I, columns of block J)
};

__device__ __forceinline__ void gw_tile_ij(int t, int nblk, int* I, int* J) {
  int i = 0;
  while (t >= nblk - i) {
    t -= nblk - i;
    ++i;
  }
  *I = i;
  *J = i + t;
}

struct GramWeights {
  const double* r;   // [n][K] row weights (W = true), else unused
  int K;
};

template <bool W>
__device__ __forceinline__ void gram_wg_body(const CUtensorMap& mapX, const GramArgs args, const GramWeights wt) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // the runtime aligns dynamic shared memory to 16 B only: the host asks for 1 KB more and the kernel aligns itself
  uint8_t* sm = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const uint32_t base = smem_u32(sm);
  const uint32_t bars = base + GW_OFF_BAR;
  auto xfull = [&](int s) -> uint32_t { return bars + 8u * (uint32_t)s; };
  auto xempty = [&](int s) -> uint32_t { return bars + 8u * (uint32_t)(GW_SX + s); };
  float* mu_s = reinterpret_cast<float*>(sm + GW_OFF_MU);   // [0, 128): block I, [128, 256): block J

  const int units = W ? args.ntile * wt.K : args.ntile;   // CTAs that read the same row range
  const int t = (int)blockIdx.x % args.ntile;
  const int comp = W ? ((int)blockIdx.x % units) / args.ntile : 0;
  const int p0 = (int)blockIdx.x / units;
  const int P = (int)gridDim.x / units;
  int I, J;
  gw_tile_ij(t, args.nblk, &I, &J);
  const bool diag = I == J;

  if (threadIdx.x == 0) {
    for (int s = 0; s < GW_SX; ++s) {
      mbar_init(xfull(s), 1);
      mbar_init(xempty(s), 1);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = threadIdx.x; i < 2 * GW_BLK; i += GW_NTHREADS)
    mu_s[i] = args.mu[(i < GW_BLK ? I : J) * GW_BLK + (i & (GW_BLK - 1))];
  __syncthreads();

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (warp == 8) {
    // ======================= TMA producer =======================
    if (elect_one()) {
      tma_prefetch_desc(&mapX);
      // boxes of 32 features that hold at least one feature < d
      const int nbI = min(4, (args.d - I * GW_BLK + 31) / 32), nbJ = diag ? 0 : min(4, (args.d - J * GW_BLK + 31) / 32);
      const uint32_t bytes = (uint32_t)((nbI + nbJ) * GW_BOX);
      int q = 0;
      for (int r = p0; r < args.nrange; r += P) {
        const int64_t row0 = (int64_t)r * GW_RANGE;
        const int nch = (int)((min((int64_t)GW_RANGE, args.n - row0) + GW_KC - 1) / GW_KC);
#pragma unroll 1
        for (int c = 0; c < nch; ++c, ++q) {
          const int xs = q % GW_SX;
          mbar_wait_nocall(xempty(xs), (uint32_t)((q / GW_SX) & 1) ^ 1u);
          mbar_expect_tx(xfull(xs), bytes);
          const uint32_t dst = base + (uint32_t)(xs * GW_XSLOT);
          const int y = (int)(row0 + c * GW_KC);
          for (int bx = 0; bx < nbI; ++bx) tma_load_2d(dst + bx * GW_BOX, &mapX, xfull(xs), I * GW_BLK + bx * 32, y);
          for (int bx = 0; bx < nbJ; ++bx)
            tma_load_2d(dst + GW_XHALF + bx * GW_BOX, &mapX, xfull(xs), J * GW_BLK + bx * 32, y);
        }
      }
    }
    __syncwarp();
    return;
  }

  // ======================= consumer warpgroups =======================
  const int g = warp >> 2, tid = threadIdx.x;   // tid < 256
  // centre, split and transpose one block of the chunk into K-major (hi, lo) operands; a warp handles 32 consecutive
  // features of one group of 4 rows: conflict-free reads, 16-byte stores
  // wrow: W = true, the chunk's first row of the weight table at this CTA's component
  auto stage = [&](const uint8_t* xb, const float* mub, int nvalid, uint32_t dhi, uint32_t dlo, int kv,
                   const double* wrow) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int it = tid + 256 * j;
      const int nf = it & (GW_BLK - 1), k4 = it >> 7;
      uint32_t hi[4], lo[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int k = 4 * k4 + i;
        const float raw = *reinterpret_cast<const float*>(
            xb + (nf >> 5) * GW_BOX + k * 128 + ((((nf & 31) >> 2) ^ (k & 7)) << 4) + (nf & 3) * 4);
        float v = (k < kv && nf < nvalid) ? raw - mub[nf] : 0.f;
        if constexpr (W) v *= k < kv ? sqrtf((float)__ldg(wrow + (int64_t)k * wt.K)) : 0.f;
        hi[i] = rn_tf32_bits(v);
        lo[i] = rn_tf32_bits(v - __uint_as_float(hi[i]));
      }
      const uint32_t off = (uint32_t)(nf * 128 + ((k4 ^ (nf & 7)) << 4));
      asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(dhi + off), "r"(hi[0]), "r"(hi[1]), "r"(hi[2]),
                   "r"(hi[3]) : "memory");
      asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(dlo + off), "r"(lo[0]), "r"(lo[1]), "r"(lo[2]),
                   "r"(lo[3]) : "memory");
    }
  };
  float acc[64], acc2[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = acc2[i] = 0.f;
  double* part = args.part + (size_t)blockIdx.x * GW_BLK * GW_BLK;
  const int wi = warp & 3;
  const int m0 = g * 64 + wi * 16 + (lane >> 2);   // accumulator rows m0, m0 + 8 (features of block I)
  bool first = true;
  int q = 0;
  for (int r = p0; r < args.nrange; r += P) {
    const int64_t row0 = (int64_t)r * GW_RANGE;
    const int nch = (int)((min((int64_t)GW_RANGE, args.n - row0) + GW_KC - 1) / GW_KC);
#pragma unroll 1
    for (int c = 0; c < nch; ++c, ++q) {
      const int xs = q % GW_SX;
      const int kv = (int)min((int64_t)GW_KC, args.n - (row0 + (int64_t)c * GW_KC));   // valid rows of the chunk
      const uint8_t* xI = sm + xs * GW_XSLOT;
      const uint32_t bh = base + (uint32_t)(GW_OFF_OP + (q & 1) * 4 * GW_BBYTES);
      const uint32_t bl = bh + (uint32_t)GW_BBYTES;
      const uint32_t ah = diag ? bh : bl + (uint32_t)GW_BBYTES;
      const uint32_t al = diag ? bl : ah + (uint32_t)GW_BBYTES;
      const double* wrow = W ? wt.r + (row0 + (int64_t)c * GW_KC) * wt.K + comp : nullptr;
      mbar_wait_nocall(xfull(xs), (uint32_t)((q / GW_SX) & 1));
      if (diag) {
        stage(xI, mu_s, args.d - I * GW_BLK, bh, bl, kv, wrow);
      } else {
        stage(xI + GW_XHALF, mu_s + GW_BLK, args.d - J * GW_BLK, bh, bl, kv, wrow);
        stage(xI, mu_s, args.d - I * GW_BLK, ah, al, kv, wrow);
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // operand writes -> visible to wgmma
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (tid == 0) mbar_arrive(xempty(xs));   // every consumer has read the slot
      wgmma_fence();
      const uint32_t arow = (uint32_t)g * 64u * 128u;   // this warpgroup's 64 rows of A
#pragma unroll
      for (int ks = 0; ks < GW_KC / 8; ++ks) {
        const uint64_t dah = make_kmajor_sw128_desc(ah + arow + ks * 32);
        const uint64_t dal = make_kmajor_sw128_desc(al + arow + ks * 32);
        const uint64_t dbh = make_kmajor_sw128_desc(bh + ks * 32);
        const uint64_t dbl = make_kmajor_sw128_desc(bl + ks * 32);
        wgmma_tf32<128>(acc, dal, dbh, ks != 0 ? 1u : 0u);   // small terms first
        wgmma_tf32<128>(acc, dah, dbl, 1u);
        wgmma_tf32<128>(acc, dah, dbh, 1u);
      }
      wgmma_commit();
      wgmma_wait0();
      reg_fence(acc);
#pragma unroll
      for (int i = 0; i < 64; ++i) acc2[i] += acc[i];
    }
    // ---- flush the range into the CTA's fp64 partial: row m of block I, column 8 (i >> 2) + 2 (lane & 3) + (i & 1) ----
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
      const int m = m0 + 8 * ((i >> 1) & 1);
      const int col = 8 * (i >> 2) + 2 * (lane & 3);
      double2* o = reinterpret_cast<double2*>(part + (size_t)m * GW_BLK + col);
      double2 v = first ? make_double2(0.0, 0.0) : *o;
      v.x += (double)acc2[i];
      v.y += (double)acc2[i + 1];
      *o = v;
      acc2[i] = 0.f;
      acc2[i + 1] = 0.f;
    }
    first = false;
  }
}
