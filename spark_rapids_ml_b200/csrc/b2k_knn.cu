// Exact k-NN (sm_90a): b2k_knn_search, Euclidean distance, float32 rows.
//
//   sizes   allgather of (n_items, n_queries, d) per rank; every size error is decided on the gathered values.
//   queries allgather of every rank's queries, padded to the largest count: Q [nranks * nq_max][d].
//   search  over the local index for every query, in work units = (tile of queries, index split):
//             wgmma path (k_knn_wg, 3xTF32): d % 4 == 0, 4 <= d <= 128, k <= 64, 16-byte aligned queries;
//               k_knn_prep writes the index as zero-padded tf32 hi/lo planes [n_pad][DP] and ||x||^2 (+inf padding).
//               Screening distance ||x||^2 - 2 q.x; each row keeps its k best (screen, local row) in shared memory.
//             generic path (k_knn_generic, SIMT): every other shape with k <= 1024; direct sum (q - x)^2.
//           Each unit writes its rows' lists to part [S][nq_all][k].
//   refine  k_knn_refine: per query, merge the S lists in split order, recompute the exact fp32 distance
//           sum_f (q_f - x_f)^2 (feature order) of the k survivors, re-sort by (exact distance, global row), map rows
//           to ids -> cand [nq_all][k].
//   gather  allgather of cand; k_knn_merge merges each own query's nranks lists in rank order -> sqrt(distance), id.
// Nothing uses atomics: two calls with the same input, rank count and device are bitwise equal.
#include <algorithm>
#include <vector>

#include "b2k_internal.cuh"

namespace {
#include "b2k_ptx.cuh"

// one candidate of the refined lists that cross NCCL (16 bytes)
struct KnnCand {
  float d;        // exact squared distance, +inf for padding
  int32_t grow;   // global row, INT32_MAX for padding
  int64_t id;     // the user's item id (global row when no ids are given), -1 for padding
};
static_assert(sizeof(KnnCand) == 16, "KnnCand crosses NCCL as 16 bytes");

__device__ __forceinline__ bool key_less(float da, int ra, float db, int rb) { return da < db || (da == db && ra < rb); }

// list entry in shared memory: (screen distance bits, local row), kept sorted ascending; (+inf, INT_MAX) = empty
__device__ __forceinline__ void list_insert(int2* L, int k, float d, int r) {
  const int2 last = L[k - 1];
  if (!key_less(d, r, __int_as_float(last.x), last.y)) return;
  int p = k - 1;
  while (p > 0) {
    const int2 e = L[p - 1];
    if (!key_less(d, r, __int_as_float(e.x), e.y)) break;
    L[p] = e;
    --p;
  }
  L[p] = make_int2(__float_as_int(d), r);
}

constexpr int KW_TM = 128;                  // queries per tile (two consumer warpgroups x wgmma M = 64)
constexpr int KW_N = 128;                   // index rows per block (wgmma N)
constexpr int KW_CHUNK = 32;                // f32 per 128-byte swizzle row
constexpr int KW_KMAX = 64;                 // largest k of the wgmma path
constexpr int KW_NTHREADS = 384;            // 8 consumer warps + a producer warpgroup (one warp issues)
constexpr int KW_SMAX = 256;                // index splits (the merge keeps 8 list heads per lane)

template <int NCH>
struct KnnWgCfg {
  static constexpr int DP = NCH * KW_CHUNK;
  static constexpr int QBYTES = KW_TM * KW_CHUNK * 4;   // one query chunk: 16 KB
  static constexpr int CBYTES = KW_N * KW_CHUNK * 4;    // one index chunk plane: 16 KB
  static constexpr int SC = 2;                           // index stages of (hi, lo)
  static constexpr int OFF_Q = 0;
  static constexpr int OFF_C = OFF_Q + NCH * QBYTES;
  static constexpr int OFF_L = OFF_C + SC * 2 * CBYTES;
  static constexpr int LBYTES = KW_TM * KW_KMAX * 8;    // [128][64] (screen distance, row)
  static constexpr int OFF_BAR = OFF_L + LBYTES;
  static constexpr int SMEM_BYTES = OFF_BAR + 8 * (2 + 2 * SC);
  static_assert(OFF_C % 1024 == 0 && CBYTES % 1024 == 0, "swizzle atoms need 1 KB alignment");
  static_assert(SMEM_BYTES + 1024 <= 227 * 1024, "smem");
};
// d = 128: query tile 64 KB + two index stages 64 KB + lists 64 KB
static_assert(KnnWgCfg<4>::SMEM_BYTES == 192 * 1024 + 48, "cfg5 layout");

struct KnnArgs {
  int64_t nq;                // query rows (all ranks, padded)
  int ntiles;                // query tiles
  int S;                     // index splits
  int nblk;                  // index blocks of KW_N rows
  int k;
  int64_t n_items;           // local index rows
  const float* norms;        // [nblk * KW_N] ||x||^2, +inf past n_items
  int2* part;                // [S][nq][k] (screen distance bits, local row)
};

__global__ void __launch_bounds__(256) k_knn_prep(const float* __restrict__ X, int64_t n, int d, int64_t n_pad, int DP,
                                                  float* __restrict__ Xhi, float* __restrict__ Xlo,
                                                  float* __restrict__ norms) {
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= n_pad) return;
  double s = 0.0;
  for (int t = lane; t < DP; t += 32) {
    const float v = (row < n && t < d) ? X[row * d + t] : 0.f;
    const uint32_t hb = rn_tf32_bits(v);
    Xhi[row * DP + t] = __uint_as_float(hb);
    Xlo[row * DP + t] = __uint_as_float(rn_tf32_bits(v - __uint_as_float(hb)));
    s += (double)v * (double)v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) norms[row] = row < n ? (float)s : __int_as_float(0x7f800000);
}

// Persistent grid, static round-robin over units u = tile * S + split.  Warp 8 issues TMA: the unit's query tile
// (NCH chunks, once per unit) and the split's index blocks, chunk by chunk, hi and lo planes into a ring of SC stages.
// Consumer warpgroup g owns queries [64 g, 64 g + 64) of the tile; per block it accumulates lo.Xhi^T + hi.Xlo^T +
// hi.Xhi^T (A = the query split in registers, as the 3xTF32 branch of k_wg_assign) into D[64 x 128].  The epilogue
// screens ||x||^2 - 2 q.x against each row's current k-th best (a register threshold replicated over the row's quad);
// the quad's lanes insert the candidates under it in turn.
template <int NCH>
__global__ void __launch_bounds__(KW_NTHREADS, 1)
k_knn_wg(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapHi,
         const __grid_constant__ CUtensorMap mapLo, const KnnArgs args) {
  using G = KnnWgCfg<NCH>;
  constexpr int R = KW_N / 2;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t base = smem_u32(smem_raw);
  if ((base & 1023u) != 0u) __trap();   // 128B-swizzle atoms need a 1 KB aligned base
  const uint32_t bars = base + G::OFF_BAR;
  const uint32_t qfull = bars, qempty = bars + 8u;
  auto cfull = [&](int s) -> uint32_t { return bars + 16u + 8u * (uint32_t)s; };
  auto cempty = [&](int s) -> uint32_t { return bars + 16u + 8u * (uint32_t)(G::SC + s); };
  int2* lists = reinterpret_cast<int2*>(smem_raw + G::OFF_L);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    mbar_init(qfull, 1);
    mbar_init(qempty, 8);
    for (int s = 0; s < G::SC; ++s) {
      mbar_init(cfull(s), 1);
      mbar_init(cempty(s), 8);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int nunits = args.ntiles * args.S;
  const int nit = (int)blockIdx.x < nunits ? (nunits - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  const int k = args.k;

  if (warp >= 8) {
    if (warp == 8 && elect_one()) {
      tma_prefetch_desc(&mapQ);
      tma_prefetch_desc(&mapHi);
      tma_prefetch_desc(&mapLo);
      int q = 0;
      for (int it = 0; it < nit; ++it) {
        const int u = (int)blockIdx.x + it * (int)gridDim.x;
        const int tile = u / args.S, split = u % args.S;
        const int b0 = (int)((int64_t)split * args.nblk / args.S), b1 = (int)((int64_t)(split + 1) * args.nblk / args.S);
        mbar_wait_nocall(qempty, (uint32_t)((it & 1) ^ 1));
        mbar_expect_tx(qfull, (uint32_t)(NCH * G::QBYTES));
        for (int c = 0; c < NCH; ++c)
          tma_load_2d(base + (uint32_t)(G::OFF_Q + c * G::QBYTES), &mapQ, qfull, c * KW_CHUNK, tile * KW_TM);
        for (int b = b0; b < b1; ++b) {
#pragma unroll 1
          for (int c = 0; c < NCH; ++c, ++q) {
            const int cs = q % G::SC;
            mbar_wait_nocall(cempty(cs), (uint32_t)((q / G::SC) & 1) ^ 1u);
            const uint32_t dst = base + (uint32_t)(G::OFF_C + cs * 2 * G::CBYTES);
            mbar_expect_tx(cfull(cs), (uint32_t)(2 * G::CBYTES));
            tma_load_2d(dst, &mapHi, cfull(cs), c * KW_CHUNK, b * KW_N);
            tma_load_2d(dst + G::CBYTES, &mapLo, cfull(cs), c * KW_CHUNK, b * KW_N);
          }
        }
      }
    }
    __syncwarp();
    return;
  }

  const int g = warp >> 2, wi = warp & 3;
  const int rr0 = g * 64 + wi * 16 + (lane >> 2);   // this thread's rows rr0, rr0 + 8 of the tile
  const uint32_t arow = (uint32_t)rr0 * 128u + (uint32_t)(lane & 3) * 4u;
  const uint32_t asw = (uint32_t)(lane >> 2);
  int2* L[2] = {lists + (size_t)rr0 * KW_KMAX, lists + (size_t)(rr0 + 8) * KW_KMAX};
  float acc[R];
  int q = 0;
  for (int it = 0; it < nit; ++it) {
    const int u = (int)blockIdx.x + it * (int)gridDim.x;
    const int tile = u / args.S, split = u % args.S;
    const int b0 = (int)((int64_t)split * args.nblk / args.S), b1 = (int)((int64_t)(split + 1) * args.nblk / args.S);
    for (int e = lane & 3; e < k; e += 4) {
      L[0][e] = make_int2(0x7f800000, 0x7fffffff);
      L[1][e] = make_int2(0x7f800000, 0x7fffffff);
    }
    __syncwarp();
    float thr[2] = {__int_as_float(0x7f800000), __int_as_float(0x7f800000)};
    mbar_wait_nocall(qfull, (uint32_t)(it & 1));
    for (int b = b0; b < b1; ++b) {
#pragma unroll
      for (int c = 0; c < NCH; ++c, ++q) {
        const int cs = q % G::SC;
        const uint8_t* xp = smem_raw + G::OFF_Q + c * G::QBYTES;
        const uint32_t cst = base + (uint32_t)(G::OFF_C + cs * 2 * G::CBYTES);
        // q = hi + lo, hi = RN_tf32(q), lo = RN_tf32(q - hi), in registers
        uint32_t ah[KW_CHUNK / 8][4], al[KW_CHUNK / 8][4];
#pragma unroll
        for (int ks = 0; ks < KW_CHUNK / 8; ++ks) {
#pragma unroll
          for (int e = 0; e < 4; ++e) {   // row rr0 + 8 (e & 1), column 8 ks + lane % 4 + 4 (e >> 1)
            const uint32_t unit = (uint32_t)(2 * ks + (e >> 1));
            const float v = *reinterpret_cast<const float*>(xp + arow + (uint32_t)(e & 1) * 1024u + ((unit ^ asw) << 4));
            ah[ks][e] = rn_tf32_bits(v);
            al[ks][e] = rn_tf32_bits(v - __uint_as_float(ah[ks][e]));
          }
        }
#pragma unroll
        for (int ks = 0; ks < KW_CHUNK / 8; ++ks) {
          reg_fence(ah[ks]);
          reg_fence(al[ks]);
        }
        mbar_wait_nocall(cfull(cs), (uint32_t)((q / G::SC) & 1));
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < KW_CHUNK / 8; ++ks) {
          const uint64_t dh = make_kmajor_sw128_desc(cst + ks * 32);
          const uint64_t dl = make_kmajor_sw128_desc(cst + G::CBYTES + ks * 32);
          wgmma_tf32_rs<KW_N>(acc, al[ks], dh, (c | ks) != 0 ? 1u : 0u);   // small terms first
          wgmma_tf32_rs<KW_N>(acc, ah[ks], dl, 1u);
          wgmma_tf32_rs<KW_N>(acc, ah[ks], dh, 1u);
        }
        wgmma_commit();
        wgmma_wait0();
        __syncwarp();
        if (lane == 0) mbar_arrive(cempty(cs));
      }
      reg_fence(acc);
      // ---- epilogue: acc[i] is row rr0 + 8 ((i >> 1) & 1), block column 8 (i >> 2) + 2 (lane & 3) + (i & 1) ----
      const float* nb = args.norms + (size_t)b * KW_N + 2 * (lane & 3);
      bool cand = false;
#pragma unroll
      for (int i = 0; i < R; ++i) {
        const float dist = fmaf(-2.f, acc[i], __ldg(nb + 8 * (i >> 2) + (i & 1)));
        acc[i] = dist;
        cand |= dist <= thr[(i >> 1) & 1] && dist < __int_as_float(0x7f800000);   // padding rows have +inf
      }
      if (__any_sync(0xffffffffu, cand)) {
#pragma unroll 1
        for (int t = 0; t < 4; ++t) {   // the quad's lanes insert in turn: each row list has one writer at a time
          if ((lane & 3) == t && cand) {
#pragma unroll
            for (int i = 0; i < R; ++i) {
              const int h = (i >> 1) & 1;
              if (acc[i] <= thr[h] && acc[i] < __int_as_float(0x7f800000)) {
                list_insert(L[h], k, acc[i], b * KW_N + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1));
                thr[h] = __int_as_float(L[h][k - 1].x);
              }
            }
          }
          __syncwarp();
        }
        thr[0] = __int_as_float(L[0][k - 1].x);
        thr[1] = __int_as_float(L[1][k - 1].x);
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(qempty);   // every A fragment of this unit has been read
    for (int h = 0; h < 2; ++h) {
      const int64_t qrow = (int64_t)tile * KW_TM + rr0 + 8 * h;
      if (qrow < args.nq) {
        int2* o = args.part + ((size_t)split * args.nq + qrow) * k;
        for (int e = lane & 3; e < k; e += 4) o[e] = L[h][e];
      }
    }
    __syncwarp();
  }
}

// generic search: CTA = GQ queries x one index split; thread (qi = tid / 8, il = tid % 8) forms the exact fp32 sums
// (q - x)^2 in feature order of items il + 8 u (u < 8) of each 64-item tile; the 8 threads of a query insert in turn
constexpr int GQ = 16, GN = 64, GC = 32, G_NTHREADS = 128;
__global__ void __launch_bounds__(G_NTHREADS, 1)
k_knn_generic(const float* __restrict__ Q, int64_t nq, const float* __restrict__ X, int64_t n_items, int d, int k,
              int S, int2* __restrict__ part) {
  extern __shared__ int2 gl[];   // [GQ][k]
  __shared__ float qs[GQ][GC + 1], xs[GN][GC + 1];
  const int tile = blockIdx.x / S, split = blockIdx.x % S;
  const int64_t ntx = (n_items + GN - 1) / GN;
  const int64_t t0 = split * ntx / S, t1 = (split + 1) * ntx / S;
  const int qi = threadIdx.x >> 3, il = threadIdx.x & 7;
  const int64_t qrow = (int64_t)tile * GQ + qi;
  int2* L = gl + (size_t)qi * k;
  for (int e = il; e < k; e += 8) L[e] = make_int2(0x7f800000, 0x7fffffff);
  __syncwarp();
  float thr = __int_as_float(0x7f800000);
  for (int64_t t = t0; t < t1; ++t) {
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int f0 = 0; f0 < d; f0 += GC) {
      __syncthreads();
      for (int e = threadIdx.x; e < GQ * GC; e += G_NTHREADS) {
        const int r = e / GC, c = e % GC;
        const int64_t qr = (int64_t)tile * GQ + r;
        qs[r][c] = (qr < nq && f0 + c < d) ? Q[qr * d + f0 + c] : 0.f;
      }
      for (int e = threadIdx.x; e < GN * GC; e += G_NTHREADS) {
        const int r = e / GC, c = e % GC;
        const int64_t xr = t * GN + r;
        xs[r][c] = (xr < n_items && f0 + c < d) ? X[xr * d + f0 + c] : 0.f;
      }
      __syncthreads();
      const int fc = min(GC, d - f0);
      for (int c = 0; c < fc; ++c) {
        const float qv = qs[qi][c];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const float df = qv - xs[il + 8 * u][c];
          acc[u] = fmaf(df, df, acc[u]);
        }
      }
    }
    const int nv = n_items - t * GN < GN ? (int)(n_items - t * GN) : GN;   // valid items of the tile
    bool cand = false;
#pragma unroll
    for (int u = 0; u < 8; ++u) cand |= il + 8 * u < nv && acc[u] <= thr;
    if (__any_sync(0xffffffffu, cand)) {
#pragma unroll 1
      for (int r = 0; r < 8; ++r) {
        if (il == r && cand) {
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            if (il + 8 * u < nv && acc[u] <= thr) {
              list_insert(L, k, acc[u], (int)(t * GN + il + 8 * u));
              thr = __int_as_float(L[k - 1].x);
            }
          }
        }
        __syncwarp();
      }
      thr = __int_as_float(L[k - 1].x);
    }
  }
  if (qrow < nq) {
    int2* o = part + ((size_t)split * nq + qrow) * k;
    for (int e = il; e < k; e += 8) o[e] = L[e];
  }
}

// Warp-wide merge of nl sorted lists (nl <= 8 * 32): lane l holds the heads of lists l, l + 32, ...; each of the k
// rounds takes the smallest head (key (d, r), then list order) and advances that list.  head(list, pos, &d, &r);
// emit(t, list, pos) runs on the lane that holds the winning list.
template <typename Head, typename Emit>
__device__ __forceinline__ void warp_merge(int nl, int k, Head head, Emit emit) {
  const int lane = threadIdx.x & 31;
  int pos[KW_SMAX / 32];
#pragma unroll
  for (int j = 0; j < KW_SMAX / 32; ++j) pos[j] = 0;
  for (int t = 0; t < k; ++t) {
    float bd = __int_as_float(0x7f800000);
    int br = 0x7fffffff, bl = 0x7fffffff;
#pragma unroll
    for (int j = 0; j < KW_SMAX / 32; ++j) {
      const int l = lane + 32 * j;
      if (l < nl && pos[j] < k) {
        float dd;
        int rr;
        head(l, pos[j], &dd, &rr);
        if (key_less(dd, rr, bd, br) || (dd == bd && rr == br && l < bl)) {
          bd = dd;
          br = rr;
          bl = l;
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float od = __shfl_xor_sync(0xffffffffu, bd, o);
      const int orr = __shfl_xor_sync(0xffffffffu, br, o), ol = __shfl_xor_sync(0xffffffffu, bl, o);
      if (key_less(od, orr, bd, br) || (od == bd && orr == br && ol < bl)) {
        bd = od;
        br = orr;
        bl = ol;
      }
    }
#pragma unroll
    for (int j = 0; j < KW_SMAX / 32; ++j)
      if (lane + 32 * j == bl) {   // the owner of the winning list emits its head (every list holds k entries)
        emit(t, bl, pos[j]);
        ++pos[j];
      }
    __syncwarp();
  }
}

// refine: warp per query row of Q.  Survivors = the k smallest (screen, local row) of the S lists; their exact fp32
// distances are recomputed in feature order and the list re-sorted by (exact distance, global row, survivor position).
constexpr int RF_WARPS = 4;
__global__ void __launch_bounds__(RF_WARPS * 32)
k_knn_refine(const int2* __restrict__ part, int S, int64_t nq, int k, const float* __restrict__ Q,
             const float* __restrict__ X, int64_t n_items, int d, int64_t row0, const int64_t* __restrict__ ids,
             KnnCand* __restrict__ cand) {
  extern __shared__ int rf_smem[];   // per warp: rows [k] (int), then exact distances [k] (float)
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t qrow = (int64_t)blockIdx.x * RF_WARPS + w;
  if (qrow >= nq) return;
  int* rows = rf_smem + (size_t)w * 2 * k;
  float* ex = reinterpret_cast<float*>(rows + k);
  if (S == 0) {
    for (int t = lane; t < k; t += 32) rows[t] = -1;
  } else {
    warp_merge(
        S, k,
        [&](int l, int p, float* dd, int* rr) {
          const int2 e = part[((size_t)l * nq + qrow) * k + p];
          *dd = __int_as_float(e.x);
          *rr = e.y;
        },
        [&](int t, int l, int p) {
          const int2 e = part[((size_t)l * nq + qrow) * k + p];
          rows[t] = e.y < n_items && e.y >= 0 ? e.y : -1;
        });
  }
  __syncwarp();
  const float* q = Q + qrow * d;
  for (int t = lane; t < k; t += 32) {
    const int r = rows[t];
    float s = __int_as_float(0x7f800000);
    if (r >= 0) {
      const float* x = X + (int64_t)r * d;
      s = 0.f;
      for (int f = 0; f < d; ++f) {
        const float df = q[f] - x[f];
        s = fmaf(df, df, s);
      }
    }
    ex[t] = s;
  }
  __syncwarp();
  for (int t = lane; t < k; t += 32) {
    const int r = rows[t];
    const float dt = ex[t];
    const int gt = r >= 0 ? (int)(row0 + r) : 0x7fffffff;
    int rank = 0;
    for (int v = 0; v < k; ++v) {
      const int rv = rows[v];
      const int gv = rv >= 0 ? (int)(row0 + rv) : 0x7fffffff;
      const float dv = ex[v];
      rank += key_less(dv, gv, dt, gt) || (dv == dt && gv == gt && v < t);
    }
    KnnCand c;
    c.d = dt;
    c.grow = gt;
    c.id = r < 0 ? -1 : (ids != nullptr ? ids[r] : row0 + r);
    cand[qrow * k + rank] = c;
  }
}

// merge: warp per own query qi; list r = all[r][q0 + qi][0, k) for r < nranks, in rank order
__global__ void __launch_bounds__(RF_WARPS * 32)
k_knn_merge(const KnnCand* __restrict__ all, int nranks, int64_t nq_all, int64_t q0, int64_t nq_own, int k,
            float* __restrict__ dist_out, int64_t* __restrict__ idx_out) {
  const int w = threadIdx.x >> 5;
  const int64_t qi = (int64_t)blockIdx.x * RF_WARPS + w;
  if (qi >= nq_own) return;
  auto at = [&](int l, int p) -> const KnnCand& { return all[((size_t)l * nq_all + q0 + qi) * k + p]; };
  warp_merge(
      nranks, k,
      [&](int l, int p, float* dd, int* rr) {
        const KnnCand& c = at(l, p);
        *dd = c.d;
        *rr = c.grow;
      },
      [&](int t, int l, int p) {
        const KnnCand& c = at(l, p);
        dist_out[qi * k + t] = sqrtf(c.d);
        idx_out[qi * k + t] = c.id;
      });
}

struct Timer {   // CUDA events around the device phases when option time_kernels is set
  cudaEvent_t ev[7] = {};
  bool on = false;
  explicit Timer(bool enable) : on(enable) {
    if (on)
      for (auto& e : ev) cudaEventCreate(&e);
  }
  ~Timer() {
    if (on)
      for (auto& e : ev) cudaEventDestroy(e);
  }
  void mark(int i, cudaStream_t s) {
    if (on) cudaEventRecord(ev[i], s);
  }
  double ms(int a, int b) const {
    float t = 0.f;
    if (on) cudaEventElapsedTime(&t, ev[a], ev[b]);
    return (double)t;
  }
};

template <int NCH>
int launch_wg(b2k_ctx* ctx, int grid, const CUtensorMap& mq, const CUtensorMap& mh, const CUtensorMap& ml,
              const KnnArgs& a, cudaStream_t s) {
  const int smem = KnnWgCfg<NCH>::SMEM_BYTES;
  B2K_CUDA_OK(ctx, cudaFuncSetAttribute(k_knn_wg<NCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  k_knn_wg<NCH><<<grid, KW_NTHREADS, smem, s>>>(mq, mh, ml, a);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  return B2K_OK;
}
}  // namespace

int b2k_knn_search_impl(b2k_ctx* ctx, const float* items, int64_t n_items, const int64_t* item_ids,
                        const float* queries, int64_t nq_local, int d, int k, float* dist_out, int64_t* idx_out,
                        cudaStream_t s) {
  const int nr = ctx->nranks;
  Timer tm(ctx->time_kernels != 0);
  // ---- sizes of every rank; each error is decided on them, identically on every rank ----
  int64_t* sz_dev;
  B2K_TRY(b2k_scratch_layout(ctx, "kNN sizes", [&](B2kLayout& L) -> int {
    sz_dev = L.take<int64_t>((size_t)3 * (nr + 1));
    return B2K_OK;
  }));
  const int64_t mine[3] = {n_items, nq_local, d};
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(sz_dev, mine, sizeof(mine), cudaMemcpyHostToDevice, s));
  B2K_TRY(b2k_comm_allgather_i64(ctx, sz_dev, sz_dev + 3, 3, s));
  std::vector<int64_t> sz((size_t)3 * nr);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(sz.data(), sz_dev + 3, sz.size() * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  int64_t n_total = 0, row0 = 0, nq_max = 0, nq_total = 0;
  for (int r = 0; r < nr; ++r) {
    if (sz[3 * r + 2] != d)
      return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_knn_search: d differs between ranks (rank " + std::to_string(r) +
                                                " has d = " + std::to_string(sz[3 * r + 2]) + ")");
    if (r < ctx->rank) row0 += sz[3 * r];
    n_total += sz[3 * r];
    nq_max = std::max(nq_max, sz[3 * r + 1]);
    nq_total += sz[3 * r + 1];
  }
  if (n_total == 0) return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_knn_search: the index is empty on every rank");
  if (k < 1 || k > n_total)
    return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_knn_search: k = " + std::to_string(k) + " must satisfy 1 <= k <= " +
                                              std::to_string(n_total) + " (items on all ranks)");
  if (k > B2K_KNN_MAX_K)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "b2k_knn_search: k = " + std::to_string(k) + " exceeds " +
                                                  std::to_string(B2K_KNN_MAX_K));
  if (n_total > (int64_t)0x7fffffff)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "b2k_knn_search: more than 2^31 - 1 items in all");
  if (nq_total == 0) return B2K_OK;

  // ---- plan ----
  const int64_t nq_all = nr > 1 ? nq_max * nr : nq_local;
  const bool q_aligned = nr > 1 || (reinterpret_cast<uintptr_t>(queries) & 15u) == 0;
  const bool wg_ok = d % 4 == 0 && d >= 4 && d <= 128 && k <= KW_KMAX && q_aligned;
  if (ctx->kernel_path == B2K_PATH_FUSED && !wg_ok)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "kernel_path=2 requested but the wgmma kNN pass needs d % 4 == 0, "
                                              "4 <= d <= 128, k <= 64 and 16-byte aligned queries (d = " +
                                                  std::to_string(d) + ", k = " + std::to_string(k) + ")");
  const bool wg = wg_ok && ctx->kernel_path != B2K_PATH_GENERIC;
  int sm = ctx->sm_count;
  if (ctx->grid_limit > 0 && ctx->grid_limit < sm) sm = ctx->grid_limit;
  const int DP = d <= 32 ? 32 : d <= 64 ? 64 : 128;
  const int64_t nblk = (n_items + KW_N - 1) / KW_N;
  const int64_t n_pad = nblk * KW_N;
  const int64_t qt = wg ? KW_TM : GQ;
  const int64_t ntiles = (nq_all + qt - 1) / qt;
  const int64_t item_tiles = wg ? nblk : (n_items + GN - 1) / GN;
  // splits of the index: at least about 2 units per SM, at most one tile of the index per split
  const int S = n_items == 0 ? 0
                             : (int)std::max<int64_t>(1, std::min<int64_t>({(2 * sm + ntiles - 1) / ntiles, item_tiles,
                                                                             (int64_t)KW_SMAX}));
  float *Qall = nullptr, *Xhi = nullptr, *Xlo = nullptr, *norms = nullptr;
  int2* part = nullptr;
  KnnCand *cand = nullptr, *cand_all = nullptr;
  B2K_TRY(b2k_scratch_layout(ctx, "kNN", [&](B2kLayout& L) -> int {
    sz_dev = L.take<int64_t>((size_t)3 * (nr + 1));
    if (nr > 1) Qall = L.take<float>((size_t)nq_all * d, 1024);
    if (wg && n_items > 0) {
      Xhi = L.take<float>((size_t)n_pad * DP, 1024);
      Xlo = L.take<float>((size_t)n_pad * DP, 1024);
      norms = L.take<float>((size_t)n_pad);
    }
    part = L.take<int2>((size_t)std::max(S, 1) * nq_all * k);
    cand = L.take<KnnCand>((size_t)nq_all * k);
    if (nr > 1) cand_all = L.take<KnnCand>((size_t)nr * nq_all * k);
    return B2K_OK;
  }));
  const float* Q = queries;
  tm.mark(0, s);
  if (nr > 1) {
    float* mineq = Qall + (size_t)ctx->rank * nq_max * d;
    if (nq_local > 0)
      B2K_CUDA_OK(ctx, cudaMemcpyAsync(mineq, queries, (size_t)nq_local * d * 4, cudaMemcpyDeviceToDevice, s));
    if (nq_max > nq_local)
      B2K_CUDA_OK(ctx, cudaMemsetAsync(mineq + (size_t)nq_local * d, 0, (size_t)(nq_max - nq_local) * d * 4, s));
    B2K_TRY(b2k_comm_allgather_bytes(ctx, mineq, Qall, (size_t)nq_max * d * 4, s));
    Q = Qall;
  }
  tm.mark(1, s);

  // ---- search of the local index for every query ----
  if (n_items > 0) {
    if (wg) {
      k_knn_prep<<<(unsigned)((n_pad * 32 + 255) / 256), 256, 0, s>>>(items, n_items, d, n_pad, DP, Xhi, Xlo, norms);
      B2K_CUDA_OK(ctx, cudaGetLastError());
      ctx->stats.kernel_launches++;
    }
    tm.mark(2, s);
    if (wg) {
      CUtensorMap mq, mh, ml;
      B2K_TRY(b2k_encode_2d(ctx, &mq, Q, (uint64_t)d, (uint64_t)nq_all, (uint64_t)d * 4, KW_CHUNK, KW_TM,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_256B));
      B2K_TRY(b2k_encode_2d(ctx, &mh, Xhi, (uint64_t)DP, (uint64_t)n_pad, (uint64_t)DP * 4, KW_CHUNK, KW_N,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_256B));
      B2K_TRY(b2k_encode_2d(ctx, &ml, Xlo, (uint64_t)DP, (uint64_t)n_pad, (uint64_t)DP * 4, KW_CHUNK, KW_N,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_256B));
      KnnArgs a{};
      a.nq = nq_all;
      a.ntiles = (int)ntiles;
      a.S = S;
      a.nblk = (int)nblk;
      a.k = k;
      a.n_items = n_items;
      a.norms = norms;
      a.part = part;
      const int grid = (int)std::min<int64_t>(sm, ntiles * S);
      if (DP == 32) B2K_TRY(launch_wg<1>(ctx, grid, mq, mh, ml, a, s));
      else if (DP == 64) B2K_TRY(launch_wg<2>(ctx, grid, mq, mh, ml, a, s));
      else B2K_TRY(launch_wg<4>(ctx, grid, mq, mh, ml, a, s));
      ctx->stats.fused_tc_launches++;
    } else {
      const size_t smem = (size_t)GQ * k * sizeof(int2);
      B2K_CUDA_OK(ctx, cudaFuncSetAttribute(k_knn_generic, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      k_knn_generic<<<(unsigned)(ntiles * S), G_NTHREADS, smem, s>>>(Q, nq_all, items, n_items, d, k, S, part);
      B2K_CUDA_OK(ctx, cudaGetLastError());
      ctx->stats.generic_launches++;
    }
    ctx->stats.kernel_launches++;
  } else {
    tm.mark(2, s);
  }
  ctx->stats.last_path = wg ? B2K_PATH_FUSED : B2K_PATH_GENERIC;
  tm.mark(3, s);

  // ---- refine, candidate allgather, merge of the own queries in rank order ----
  const size_t rf_smem = (size_t)RF_WARPS * 2 * k * 4;
  B2K_CUDA_OK(ctx, cudaFuncSetAttribute(k_knn_refine, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rf_smem));
  k_knn_refine<<<(unsigned)((nq_all + RF_WARPS - 1) / RF_WARPS), RF_WARPS * 32, rf_smem, s>>>(
      part, S, nq_all, k, Q, items, n_items, d, row0, item_ids, cand);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  tm.mark(4, s);
  const KnnCand* all = cand;
  if (nr > 1) {
    B2K_TRY(b2k_comm_allgather_bytes(ctx, cand, cand_all, (size_t)nq_all * k * sizeof(KnnCand), s));
    all = cand_all;
  }
  tm.mark(5, s);
  if (nq_local > 0) {
    k_knn_merge<<<(unsigned)((nq_local + RF_WARPS - 1) / RF_WARPS), RF_WARPS * 32, 0, s>>>(
        all, nr, nq_all, nr > 1 ? (int64_t)ctx->rank * nq_max : 0, nq_local, k, dist_out, idx_out);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
  }
  tm.mark(6, s);
  if (tm.on) {
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
    ctx->stats.last_finalize_ms = tm.ms(1, 2);                  // prep
    ctx->stats.last_fused_ms = tm.ms(2, 3);                     // search
    ctx->stats.last_reduce_ms = tm.ms(3, 4) + tm.ms(5, 6);      // refine + merge
    ctx->stats.last_allreduce_ms = tm.ms(0, 1) + tm.ms(4, 5);   // query and candidate all-gathers
    ctx->stats.last_loop_ms = tm.ms(0, 6);
  }
  return B2K_OK;
}
