// The fp64 Gram passes (sm_90a): G_c = sum_rows f_c r_rc (x - mu_c)(x - mu_c)^T for k components c, as packed upper
// triangles [k][d (d + 1) / 2] (row-major, i <= j).  PCA and linear regression (b2k_moments_impl) and ALS's Y^T Y
// (b2k_gram_local_impl) run the unweighted pass (W = false, k = 1, r = f = 1); Gaussian mixtures the weighted one
// (W = true: r [n][k] fp64 row weights, f [k] fp64 factors, each component about its own centre mu_c).
//
//   wgmma   k_gram_wg<W> (3xTF32): d % 4 == 0, X 16-byte aligned.  Per-CTA fp64 partials of one 128 x 128 tile,
//           folded in CTA order (k_gram_fold_wg).
//   generic k_gram_generic<W> (SIMT, fp64 products and sums): every d.  Per-row-span fp64 partials of every 32 x 32 tile,
//           folded in span order (k_gram_fold_generic).
//   Numerics.  W = false centres in fp32 (x - mu as a float; exact for data near mu); W = true centres in fp64 (the
//   generic pass) or rounds x - mu_c once to fp32 and scales it by fl32(sqrt(fl32(f_c r))) at the split (the wgmma
//   pass), f_c r formed in fp64.
// Every output is a fixed function of (n, d, k, grid): no atomics, bitwise reproducible.
#include <algorithm>
#include <type_traits>

#include "b2k_internal.cuh"

namespace {
#include "b2k_ptx.cuh"

// ---------------------------------------------------------------------------------------------------------------------
// wgmma pass: the upper block triangle of 128 x 128 feature blocks.
//
// Weighted variant (W = true): G_c for each component c of r [n][K], about the component's own centre mu_c.  Each row's
// centred fp32 value is multiplied by fl32(sqrt(fl32(f_c r_rc))) before the split, in both operands, so the product
// carries f_c r_rc.  The caller picks f_c = 1 / N_c: the weights of a component then sum to 1, so a component whose r
// all lie below FLT_MIN keeps its weights in fp32, and G_c is its covariance about mu_c.  The grid is a multiple of
// K * ntile: CTA b owns component (b % (K ntile)) / ntile and tile b % ntile, so the K ntile CTAs of one p read the same
// row range at the same time and it is fetched from HBM about once per pass.
//
// Work: tile t = (I, J), I <= J, is the product of feature block I (wgmma M, 64 per consumer warpgroup) and feature block
// J (wgmma N = 128); the contraction runs over rows.  The grid is a multiple of the tile count: CTA b owns tile
// b % ntile for its whole run and the row ranges p, p + P, p + 2P, ... (p = b / ntile, P = grid / ntile) of GW_RANGE rows
// each.  CTAs of the same p read the same rows at the same time, so a row range is fetched from HBM about once and
// re-read from L2 by the other tiles.
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
// ---------------------------------------------------------------------------------------------------------------------
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
  const float* mu;   // [K][nblk * 128] fp32 centre per component (K = 1 unless W), 0 past d
  double* part;      // [grid][128][128] fp64 sums of the CTA's tile (rows of block I, columns of block J)
};

struct GramWeights {
  const double* r;       // [n][K] row weights (W = true), else unused
  const double* scale;   // [K] per-component factors of r (W = true), else unused
  int K;
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

template <bool W>
__global__ void __launch_bounds__(GW_NTHREADS, 1)
k_gram_wg(const __grid_constant__ CUtensorMap mapX, const GramArgs args, const GramWeights wt) {
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
  const float* mu_c = args.mu + (size_t)comp * args.nblk * GW_BLK;
  for (int i = threadIdx.x; i < 2 * GW_BLK; i += GW_NTHREADS)
    mu_s[i] = mu_c[(i < GW_BLK ? I : J) * GW_BLK + (i & (GW_BLK - 1))];
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
  // wrow: W = true, the chunk's first row of the weight table at this CTA's component, scaled by wsc in fp64
  const double wsc = W ? __ldg(wt.scale + comp) : 1.0;
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
        if constexpr (W) v *= k < kv ? sqrtf((float)(__ldg(wrow + (int64_t)k * wt.K) * wsc)) : 0.f;
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

// entry (gi, gj), gi <= gj, of component comp in the packed upper triangles [k][d (d + 1) / 2]
__device__ __forceinline__ int64_t tri_index(int comp, int gi, int gj, int d) {
  return comp * ((int64_t)d * (d + 1) / 2) + (int64_t)gi * d - (int64_t)gi * (gi - 1) / 2 + (gj - gi);
}

// CTA b = (p k + comp) ntile + t: the P partials of (comp, tile (I, J)) in CTA order -> the upper triangles
__global__ void k_gram_fold_wg(const double* __restrict__ part, int P, int ntile, int nblk, int d, int k,
                               double* __restrict__ tri) {
  const int64_t dd = (int64_t)d * d;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)k * dd) return;
  const int comp = (int)(idx / dd);
  const int gi = (int)((idx % dd) / d), gj = (int)(idx % d);
  if (gi > gj) return;
  const int I = gi / GW_BLK, J = gj / GW_BLK;
  const int t = I * nblk - I * (I - 1) / 2 + (J - I);
  const size_t e = (size_t)(gi % GW_BLK) * GW_BLK + (gj % GW_BLK);
  double s = 0.0;
  for (int p = 0; p < P; ++p) s += part[(((size_t)p * k + comp) * ntile + t) * GW_BLK * GW_BLK + e];
  tri[tri_index(comp, gi, gj, d)] = s;
}

// ---- generic pass: 32 x 32 tiles of the upper block triangle x component (blockIdx.x, tile fastest, so the CTAs of one
// row span run together and read it from L2) x row span (blockIdx.y); thread (tx, ty) forms entries (ty + 16 a,
// tx + 16 b) of the tile in fp64.  W = false stages x - mu in fp32, W = true x - mu_comp (mu [k][d]) in fp64 with the
// row weights r [n][k] times scale [k]. ----
constexpr int GG_T = 32;
template <bool W>
__global__ void __launch_bounds__(256)
k_gram_generic(const float* __restrict__ X, const double* __restrict__ r, int64_t n, int d, int k,
               const float* __restrict__ mu, int64_t span_rows, double* __restrict__ part,
               const double* __restrict__ scale) {
  using T = typename std::conditional<W, double, float>::type;
  __shared__ T xi[GG_T][GG_T + 1], xj[GG_T][GG_T + 1];
  __shared__ double wr[W ? GG_T : 1];
  const int nb = (d + GG_T - 1) / GG_T, ntri = nb * (nb + 1) / 2;
  int t = W ? (int)blockIdx.x % ntri : (int)blockIdx.x, I = 0;
  while (t >= nb - I) {
    t -= nb - I;
    ++I;
  }
  const int J = I + t, comp = W ? (int)blockIdx.x / ntri : 0;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int64_t r0 = (int64_t)blockIdx.y * span_rows;
  const int64_t r1 = min(n, r0 + span_rows);
  double acc[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
  for (int64_t rb = r0; rb < r1; rb += GG_T) {
    for (int e = threadIdx.x; e < GG_T * GG_T; e += 256) {
      const int rr = e / GG_T, cc = e % GG_T;
      const int64_t row = rb + rr;
      const int ci = I * GG_T + cc, cj = J * GG_T + cc;
      if constexpr (W) {
        xi[rr][cc] = (row < r1 && ci < d) ? (double)X[row * d + ci] - (double)mu[(size_t)comp * d + ci] : 0.0;
        xj[rr][cc] = (row < r1 && cj < d) ? (double)X[row * d + cj] - (double)mu[(size_t)comp * d + cj] : 0.0;
      } else {
        xi[rr][cc] = (row < r1 && ci < d) ? X[row * d + ci] - mu[ci] : 0.f;
        xj[rr][cc] = (row < r1 && cj < d) ? X[row * d + cj] - mu[cj] : 0.f;
      }
    }
    if (W && threadIdx.x < GG_T)
      wr[threadIdx.x] = rb + threadIdx.x < r1 ? r[(rb + threadIdx.x) * k + comp] * scale[comp] : 0.0;
    __syncthreads();
#pragma unroll(W ? 4 : 8)
    for (int rr = 0; rr < GG_T; ++rr) {
      double a0 = xi[rr][ty], a1 = xi[rr][ty + 16];
      if constexpr (W) {
        const double w = wr[rr];
        a0 = w * xi[rr][ty];
        a1 = w * xi[rr][ty + 16];
      }
      const double b0 = xj[rr][tx], b1 = xj[rr][tx + 16];
      acc[0][0] = fma(a0, b0, acc[0][0]);
      acc[0][1] = fma(a0, b1, acc[0][1]);
      acc[1][0] = fma(a1, b0, acc[1][0]);
      acc[1][1] = fma(a1, b1, acc[1][1]);
    }
    __syncthreads();
  }
  double* o = part + (W ? (size_t)blockIdx.y * k + comp : (size_t)blockIdx.y) * d * d;
  for (int a = 0; a < 2; ++a)
    for (int b = 0; b < 2; ++b) {
      const int gi = I * GG_T + ty + 16 * a, gj = J * GG_T + tx + 16 * b;
      if (gi < d && gj < d) o[(size_t)gi * d + gj] = acc[a][b];
    }
}

// spans in order -> the upper triangles
__global__ void k_gram_fold_generic(const double* __restrict__ part, int S, int d, int k, double* __restrict__ tri) {
  const int64_t dd = (int64_t)d * d;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)k * dd) return;
  const int comp = (int)(idx / dd);
  const int gi = (int)((idx % dd) / d), gj = (int)(idx % d);
  if (gi > gj) return;
  double s = 0.0;
  for (int sp = 0; sp < S; ++sp) s += part[((size_t)sp * k + comp) * dd + gi * d + gj];
  tri[tri_index(comp, gi, gj, d)] = s;
}

// G [d][d] <- the packed upper triangle, mirrored
__global__ void k_gram_unpack(const double* __restrict__ tri, int d, double* __restrict__ G) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)d * d) return;
  const int i = (int)(idx / d), j = (int)(idx % d);
  G[idx] = tri[tri_index(0, min(i, j), max(i, j), d)];
}

}  // namespace

int b2k_launch_gram_unpack(b2k_ctx* ctx, const double* tri, int d, double* G, cudaStream_t s) {
  k_gram_unpack<<<(unsigned)(((int64_t)d * d + 255) / 256), 256, 0, s>>>(tri, d, G);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  return B2K_OK;
}

bool b2k_gram_wg_ok(const float* X, int d) { return d % 4 == 0 && (reinterpret_cast<uintptr_t>(X) & 15u) == 0; }

B2kGramPlan b2k_gram_plan(const b2k_ctx* ctx, const float* X, int64_t n, int d, int k, bool allow_wg,
                          size_t part_bytes) {
  B2kGramPlan p;
  p.wg = allow_wg && b2k_gram_wg_ok(X, d);
  p.n = n;
  p.d = d;
  p.k = k;
  const size_t dd = (size_t)d * d;
  p.out_len = (size_t)k * d * (d + 1) / 2;
  if (p.wg) {
    const int nblk = (d + GW_BLK - 1) / GW_BLK, ntile = nblk * (nblk + 1) / 2;
    const int nrange = (int)std::max<int64_t>(1, (n + GW_RANGE - 1) / GW_RANGE);
    int sm = ctx->sm_count;
    if (ctx->grid_limit > 0 && ctx->grid_limit < sm) sm = ctx->grid_limit;
    p.spans = std::max(1, std::min(sm / (ntile * k), nrange));   // CTAs per (component, tile)
    p.grid = p.spans * ntile * k;
    p.part_len = (size_t)p.grid * GW_BLK * GW_BLK;
    p.mu_len = (size_t)k * nblk * GW_BLK;
  } else {
    // row spans of the fp64 partials, at most part_bytes of them: a function of (n, d, k) alone
    p.spans = (int)std::max<int64_t>(
        1, std::min<int64_t>({64, (int64_t)(part_bytes / ((size_t)k * dd * 8)), (n + GG_T - 1) / GG_T}));
    const int nb = (d + GG_T - 1) / GG_T;
    p.grid = nb * (nb + 1) / 2 * k;
    p.part_len = (size_t)p.spans * k * dd;
    p.mu_len = (size_t)k * d;
  }
  return p;
}

int b2k_gram_launch(b2k_ctx* ctx, const B2kGramPlan& p, const float* X, const float* mu, const double* r,
                    const double* r_scale, double* part, double* tri, cudaStream_t s) {
  const int64_t n = p.n;
  const int d = p.d, k = p.k;
  const bool W = r != nullptr;
  const unsigned fold_blocks = (unsigned)(((int64_t)k * d * d + 255) / 256);
  if (n == 0) B2K_CUDA_OK(ctx, cudaMemsetAsync(part, 0, p.part_len * 8, s));
  if (p.wg) {
    const int nblk = (d + GW_BLK - 1) / GW_BLK, ntile = nblk * (nblk + 1) / 2;
    if (n > 0) {
      CUtensorMap map;
      B2K_TRY(b2k_encode_2d(ctx, &map, X, (uint64_t)d, (uint64_t)n, (uint64_t)d * 4, 32, GW_KC,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_256B));
      const GramArgs ga{n, d, nblk, ntile, (int)std::max<int64_t>(1, (n + GW_RANGE - 1) / GW_RANGE), mu, part};
      auto kern = W ? k_gram_wg<true> : k_gram_wg<false>;
      B2K_CUDA_OK(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, GW_SMEM + 1024));
      kern<<<p.grid, GW_NTHREADS, GW_SMEM + 1024, s>>>(map, ga, GramWeights{r, r_scale, k});
      B2K_CUDA_OK(ctx, cudaGetLastError());
    }
    k_gram_fold_wg<<<fold_blocks, 256, 0, s>>>(part, p.spans, ntile, nblk, d, k, tri);
  } else {
    if (n > 0) {
      const int64_t span_rows = std::max<int64_t>(1, (n + p.spans - 1) / p.spans);
      auto kern = W ? k_gram_generic<true> : k_gram_generic<false>;
      kern<<<dim3(p.grid, p.spans), 256, 0, s>>>(X, r, n, d, k, mu, span_rows, part, r_scale);
      B2K_CUDA_OK(ctx, cudaGetLastError());
    }
    k_gram_fold_generic<<<fold_blocks, 256, 0, s>>>(part, p.spans, d, k, tri);
  }
  B2K_CUDA_OK(ctx, cudaGetLastError());
  return B2K_OK;
}
