// Exact k-NN (sm_90a): b2k_knn_search, Euclidean distance, float32 rows.
//
//   sizes   allgather of (n_items, n_queries, d) per rank; every size error is decided on the gathered values.
//   queries allgather of every rank's queries, padded to the largest count: Q [nranks * nq_max][d].
//   search  over the local index for every query, in work units = (tile of queries, index split), given to the passes
//           as a unit table {query rows, index range, output row} that IVF-Flat (b2k_ivf.cu) fills with its own units:
//             wgmma path (k_knn_wg, 3xTF32): d % 4 == 0, 4 <= d <= 128, k <= 64, 16-byte aligned queries;
//               everything in the frame of s = local item row 0 (non-finite components -> 0): k_knn_prep writes the
//               index as zero-padded tf32 hi/lo planes of x - s [n_pad][DP] and ||x - s||^2 (+inf padding),
//               k_knn_shift_q writes Qs = Q - s [nq][d].  Screening distance ||x - s||^2 - 2 (q - s).(x - s); each
//               row keeps its k best (screen, local row) in shared memory.
//             generic path (k_knn_generic, SIMT): every other shape with k <= 1024; direct sum (q - x)^2.
//           Each unit writes its rows' lists to part [S][nq_all][k].
//   refine  k_knn_refine: per query, merge the S lists in split order, recompute the exact fp32 distance
//           sum_f (q_f - x_f)^2 (feature order, from the caller's unshifted rows) of the k survivors, re-sort by
//           (exact distance, global row), map rows to ids -> cand [nq_all][k].
//   gather  allgather of cand; k_knn_merge merges each own query's nranks lists in rank order -> sqrt(distance), id.
// Nothing uses atomics: two calls with the same input, rank count and device are bitwise equal.
#include <algorithm>
#include <vector>

#include "b2k_internal.cuh"

namespace {
#include "b2k_ptx.cuh"
#include "b2k_pair_wg.cuh"

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

constexpr int KW_KMAX = 64;                 // largest k of the wgmma path
constexpr int KW_SMAX = B2K_KNN_MAX_LISTS;  // index splits (the merge keeps 8 list heads per lane)
constexpr int KW_LBYTES = PW_TM * KW_KMAX * 8;   // row lists [128][64] (screen distance bits, row)

// d = 128: query tile 64 KB + two index stages 64 KB + lists 64 KB
template <int NCH>
using KnnWgCfg = PairWgCfg<NCH, KW_LBYTES>;
static_assert(KnnWgCfg<4>::SMEM_BYTES == 192 * 1024 + 48, "cfg5 layout");

struct KnnArgs {
  const KnnUnit* units;      // [nunits], index ranges in blocks of PW_N rows
  int nunits;
  int k;
  const float* norms;        // [blocks * PW_N] ||x - s||^2, +inf on padding rows
  int2* part;                // rows of k (screen distance bits, index row)
};

#include "b2k_knn_prep.cuh"

// Persistent grid, static round-robin over the unit table; producer and main loop of b2k_pair_wg.cuh.  Q, X and the
// norms all come shifted by s.  The epilogue screens ||x - s||^2 - 2 (q - s).(x - s) against each row's current k-th
// best (a register threshold replicated over the row's quad); the quad's lanes insert the candidates under it in turn.
template <int NCH>
__global__ void __launch_bounds__(PW_NTHREADS, 1)
k_knn_wg(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapHi,
         const __grid_constant__ CUtensorMap mapLo, const KnnArgs args) {
  using G = KnnWgCfg<NCH>;
  constexpr int R = PW_N / 2;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t base = smem_u32(smem_raw);
  const PairWgBars bars = pair_wg_init<G>(base);
  int2* lists = reinterpret_cast<int2*>(smem_raw + G::OFF_OWN);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nunits = args.nunits;
  const int nit = (int)blockIdx.x < nunits ? (nunits - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  const int k = args.k;

  if (warp >= 8) {
    if (warp == 8 && elect_one())
      pair_wg_produce<G>(
          base, bars, &mapQ, &mapHi, &mapLo, nit,
          [&](int it) {
            const KnnUnit un = args.units[(int)blockIdx.x + it * (int)gridDim.x];
            return PairWgUnit{un.row0, un.lo, un.hi};
          },
          [](int) { return false; });
    __syncwarp();
    return;
  }

  const int g = warp >> 2, wi = warp & 3;
  const int rr0 = g * 64 + wi * 16 + (lane >> 2);   // this thread's rows rr0, rr0 + 8 of the tile
  int2* L[2] = {lists + (size_t)rr0 * KW_KMAX, lists + (size_t)(rr0 + 8) * KW_KMAX};
  float acc[R];
  int q = 0;
  for (int it = 0; it < nit; ++it) {
    const KnnUnit un = args.units[(int)blockIdx.x + it * (int)gridDim.x];
    for (int e = lane & 3; e < k; e += 4) {
      L[0][e] = make_int2(0x7f800000, 0x7fffffff);
      L[1][e] = make_int2(0x7f800000, 0x7fffffff);
    }
    __syncwarp();
    float thr[2] = {__int_as_float(0x7f800000), __int_as_float(0x7f800000)};
    mbar_wait_nocall(bars.qfull(), (uint32_t)(it & 1));
    for (int b = un.lo; b < un.hi; ++b) {
      pair_wg_block<G>(smem_raw, base, bars, rr0, lane, acc, q);
      // ---- epilogue: acc[i] is row rr0 + 8 ((i >> 1) & 1), block column 8 (i >> 2) + 2 (lane & 3) + (i & 1) ----
      const float* nb = args.norms + (size_t)b * PW_N + 2 * (lane & 3);
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
                list_insert(L[h], k, acc[i], b * PW_N + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1));
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
    if (lane == 0) mbar_arrive(bars.qempty());   // every A fragment of this unit has been read
    for (int h = 0; h < 2; ++h) {
      const int r = rr0 + 8 * h;
      if (r < un.nrows) {
        int2* o = args.part + (size_t)(un.out0 + r) * k;
        for (int e = lane & 3; e < k; e += 4) o[e] = L[h][e];
      }
    }
    __syncwarp();
  }
}

// generic search: CTA = one unit of GQ queries x an item row range; thread (qi = tid / 8, il = tid % 8) forms the exact
// fp32 sums (q - x)^2 in feature order of items il + 8 u (u < 8) of each 64-item tile; the 8 threads of a query insert
// in turn
constexpr int GQ = B2K_KNN_GEN_QROWS, GN = 64, GC = 32, G_NTHREADS = 128;
__global__ void __launch_bounds__(G_NTHREADS, 1)
k_knn_generic(const float* __restrict__ Q, const float* __restrict__ X, const int32_t* __restrict__ xperm, int d, int k,
              const KnnUnit* __restrict__ units, int2* __restrict__ part) {
  extern __shared__ int2 gl[];   // [GQ][k]
  __shared__ float qs[GQ][GC + 1], xs[GN][GC + 1];
  const KnnUnit un = units[blockIdx.x];
  const int qi = threadIdx.x >> 3, il = threadIdx.x & 7;
  int2* L = gl + (size_t)qi * k;
  for (int e = il; e < k; e += 8) L[e] = make_int2(0x7f800000, 0x7fffffff);
  __syncwarp();
  float thr = __int_as_float(0x7f800000);
  for (int64_t t = un.lo; t < un.hi; t += GN) {
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int f0 = 0; f0 < d; f0 += GC) {
      __syncthreads();
      for (int e = threadIdx.x; e < GQ * GC; e += G_NTHREADS) {
        const int r = e / GC, c = e % GC;
        qs[r][c] = (r < un.nrows && f0 + c < d) ? Q[(int64_t)(un.row0 + r) * d + f0 + c] : 0.f;
      }
      for (int e = threadIdx.x; e < GN * GC; e += G_NTHREADS) {
        const int r = e / GC, c = e % GC;
        const int64_t xr = t + r;
        xs[r][c] = (xr < un.hi && f0 + c < d) ? X[(xperm != nullptr ? (int64_t)xperm[xr] : xr) * d + f0 + c] : 0.f;
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
    const int nv = un.hi - t < GN ? (int)(un.hi - t) : GN;   // valid items of the tile
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
              list_insert(L, k, acc[u], (int)(t + il + 8 * u));
              thr = __int_as_float(L[k - 1].x);
            }
          }
        }
        __syncwarp();
      }
      thr = __int_as_float(L[k - 1].x);
    }
  }
  if (qi < un.nrows) {
    int2* o = part + (size_t)(un.out0 + qi) * k;
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

// refine: warp per query row of Q.  Survivors = the k smallest (screen, local row) of the nl lists; their exact fp32
// distances are recomputed in feature order and the list re-sorted by (exact distance, global row, survivor position).
// A list is sorted by (screen, index row), and index rows order as local rows within one list, so each list is also
// sorted by (screen, local row) and the merge may key on the local row.
constexpr int RF_WARPS = 4;
__global__ void __launch_bounds__(RF_WARPS * 32)
k_knn_refine(const int2* __restrict__ part, int nl, const int32_t* __restrict__ slots, const int32_t* __restrict__ perm,
             int64_t nq, int k, const float* __restrict__ Q, const float* __restrict__ X, int64_t n_items, int d,
             int64_t row0, const int64_t* __restrict__ ids, KnnCand* __restrict__ cand) {
  extern __shared__ int rf_smem[];   // per warp: rows [k] (int), then exact distances [k] (float)
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t qrow = (int64_t)blockIdx.x * RF_WARPS + w;
  if (qrow >= nq) return;
  int* rows = rf_smem + (size_t)w * 2 * k;
  float* ex = reinterpret_cast<float*>(rows + k);
  // entry p of list l as (screen bits, local row); a missing list reads as empty
  auto entry = [&](int l, int p) -> int2 {
    const int64_t sl = slots != nullptr ? (int64_t)slots[qrow * nl + l] : (int64_t)l * nq + qrow;
    if (sl < 0) return make_int2(0x7f800000, 0x7fffffff);
    int2 e = part[(size_t)sl * k + p];
    if (perm != nullptr && e.y >= 0 && e.y != 0x7fffffff) e.y = perm[e.y];
    return e;
  };
  if (nl == 0) {
    for (int t = lane; t < k; t += 32) rows[t] = -1;
  } else {
    warp_merge(
        nl, k,
        [&](int l, int p, float* dd, int* rr) {
          const int2 e = entry(l, p);
          *dd = __int_as_float(e.x);
          *rr = e.y;
        },
        [&](int t, int l, int p) {
          const int2 e = entry(l, p);
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
            bool squared, bool fill, float* __restrict__ dist_out, int64_t* idx_out) {
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
        dist_out[qi * k + t] = squared ? c.d : sqrtf(c.d);
        // entry 0 was written by its lane before warp_merge's __syncwarp
        idx_out[qi * k + t] = !fill || c.grow != 0x7fffffff ? c.id : t == 0 ? INT64_MAX : idx_out[qi * k];
      });
}

// The local search: plan, prep, search and refine of queries Q [nq][d] against this rank's items, with no collective.
struct KnnLocal {
  bool wg = false;
  int DP = 0, S = 0;
  int64_t nblk = 0, n_pad = 0, ntiles = 0;
  float *Qs = nullptr, *Xhi = nullptr, *Xlo = nullptr, *norms = nullptr;
  KnnUnit* units = nullptr;
  int2* part = nullptr;
};

int knn_local_plan(b2k_ctx* ctx, int64_t n_items, int64_t nq, int d, int k, bool q_aligned, KnnLocal* p) {
  const bool wg_ok = b2k_knn_wg_shape(d, k) && q_aligned;
  if (ctx->kernel_path == B2K_PATH_FUSED && !wg_ok)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "kernel_path=2 requested but the wgmma kNN pass needs d % 4 == 0, "
                                              "4 <= d <= 128, k <= 64 and 16-byte aligned queries (d = " +
                                                  std::to_string(d) + ", k = " + std::to_string(k) + ")");
  p->wg = wg_ok && ctx->kernel_path != B2K_PATH_GENERIC;
  int sm = ctx->sm_count;
  if (ctx->grid_limit > 0 && ctx->grid_limit < sm) sm = ctx->grid_limit;
  p->DP = b2k_knn_wg_dp(d);
  p->nblk = (n_items + PW_N - 1) / PW_N;
  p->n_pad = p->nblk * PW_N;
  const int64_t qt = p->wg ? PW_TM : GQ;
  p->ntiles = (nq + qt - 1) / qt;
  const int64_t item_tiles = p->wg ? p->nblk : (n_items + GN - 1) / GN;
  // splits of the index: at least about 2 units per SM, at most one tile of the index per split
  p->S = n_items == 0 ? 0
                      : (int)std::max<int64_t>(1, std::min<int64_t>({(2 * sm + p->ntiles - 1) / p->ntiles, item_tiles,
                                                                     (int64_t)KW_SMAX}));
  return B2K_OK;
}

void knn_local_take(B2kLayout& L, KnnLocal* p, int64_t n_items, int64_t nq, int d, int k) {
  if (p->wg && n_items > 0) {
    p->Qs = L.take<float>((size_t)nq * d, 1024);
    p->Xhi = L.take<float>((size_t)p->n_pad * p->DP, 1024);
    p->Xlo = L.take<float>((size_t)p->n_pad * p->DP, 1024);
    p->norms = L.take<float>((size_t)p->n_pad);
  }
  p->units = L.take<KnnUnit>((size_t)std::max<int64_t>(p->ntiles * p->S, 1));
  p->part = L.take<int2>((size_t)std::max(p->S, 1) * nq * k);
}

// marks 2 (after prep), 3 (after search) and 4 (after refine) of tm
int knn_local_run(b2k_ctx* ctx, const KnnLocal& p, const float* items, int64_t n_items, const int64_t* item_ids,
                  const float* Q, int64_t nq, int d, int k, int64_t row0, KnnCand* cand, B2kTimer& tm, cudaStream_t s) {
  // ---- search of the local index for every query ----
  if (n_items > 0) {
    // units u = tile * S + split: a tile of queries against one split of the index
    const int64_t qt = p.wg ? PW_TM : GQ, ntx = p.wg ? p.nblk : (n_items + GN - 1) / GN;
    std::vector<KnnUnit> units((size_t)(p.ntiles * p.S));
    for (int64_t tile = 0; tile < p.ntiles; ++tile)
      for (int split = 0; split < p.S; ++split) {
        KnnUnit& u = units[(size_t)(tile * p.S + split)];
        u.row0 = (int)(tile * qt);
        u.nrows = (int)std::min<int64_t>(qt, nq - tile * qt);
        u.out0 = (int64_t)split * nq + tile * qt;
        const int64_t t0 = split * ntx / p.S, t1 = (split + 1) * ntx / p.S;
        u.lo = p.wg ? (int)t0 : (int)(t0 * GN);
        u.hi = p.wg ? (int)t1 : (int)std::min<int64_t>(t1 * GN, n_items);
      }
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(p.units, units.data(), units.size() * sizeof(KnnUnit), cudaMemcpyHostToDevice, s));
    if (p.wg) {
      B2K_TRY(b2k_knn_prep_launch(ctx, items, n_items, d, nullptr, p.n_pad, p.DP, p.Xhi, p.Xlo, p.norms, s));
      B2K_TRY(b2k_knn_shift_launch(ctx, Q, nq, d, items, p.Qs, s));
    }
    tm.mark(2, s);
    B2K_TRY(b2k_knn_scan_launch(ctx, p.wg, p.DP, p.wg ? p.Qs : Q, nq, items, nullptr, p.Xhi, p.Xlo, p.norms, p.n_pad, d,
                                k, p.units, (int)units.size(), p.part, s));
  } else {
    tm.mark(2, s);
  }
  ctx->stats.last_path = p.wg ? B2K_PATH_FUSED : B2K_PATH_GENERIC;
  tm.mark(3, s);

  // ---- refine ----
  B2K_TRY(b2k_knn_refine_launch(ctx, p.part, p.S, nullptr, nullptr, nq, k, Q, items, n_items, d, row0, item_ids, cand,
                                s));
  tm.mark(4, s);
  return B2K_OK;
}
}  // namespace

bool b2k_knn_wg_width(int d) { return d % 4 == 0 && d >= 4 && d <= 128; }
bool b2k_knn_wg_shape(int d, int k) { return b2k_knn_wg_width(d) && k <= KW_KMAX; }
int b2k_knn_wg_dp(int d) { return d <= 32 ? 32 : d <= 64 ? 64 : 128; }

int b2k_knn_prep_launch(b2k_ctx* ctx, const float* X, int64_t n, int d, const int32_t* perm, int64_t n_pad, int DP,
                        float* Xhi, float* Xlo, float* norms, cudaStream_t s) {
  if (n_pad == 0) return B2K_OK;
  k_knn_prep<<<(unsigned)((n_pad * 32 + 255) / 256), 256, 0, s>>>(X, n, d, perm, n_pad, DP, Xhi, Xlo, norms);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  return B2K_OK;
}

int b2k_knn_shift_launch(b2k_ctx* ctx, const float* Q, int64_t nq, int d, const float* X, float* Qs, cudaStream_t s) {
  if (nq == 0) return B2K_OK;
  const int64_t n4 = nq * d / 4;
  k_knn_shift_q<<<(unsigned)std::min<int64_t>((n4 + 255) / 256, (int64_t)ctx->sm_count * 16), 256, 0, s>>>(
      reinterpret_cast<const float4*>(Q), n4, d, X, reinterpret_cast<float4*>(Qs));
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  return B2K_OK;
}

int b2k_knn_scan_launch(b2k_ctx* ctx, bool wg, int DP, const float* Q, int64_t nq, const float* X, const int32_t* xperm,
                        const float* Xhi, const float* Xlo, const float* norms, int64_t n_pad, int d, int k,
                        const KnnUnit* units, int nunits, int2* part, cudaStream_t s) {
  if (nunits == 0) return B2K_OK;
  if (wg) {
    PairWgMaps maps;
    B2K_TRY(pair_wg_maps(ctx, Q, nq, d, Xhi, Xlo, n_pad, DP, &maps));
    KnnArgs a{};
    a.units = units;
    a.nunits = nunits;
    a.k = k;
    a.norms = norms;
    a.part = part;
    int sm = ctx->sm_count;
    if (ctx->grid_limit > 0 && ctx->grid_limit < sm) sm = ctx->grid_limit;
    const int grid = std::min(sm, nunits);
    B2K_TRY(pair_wg_launch<KW_LBYTES>(
        ctx, DP, [](auto nch) { return k_knn_wg<decltype(nch)::value>; }, grid, maps, a, s));
    ctx->stats.fused_tc_launches++;
  } else {
    // The attribute is per function and process-wide, so it is set for the largest k: ranks running as threads of one
    // process, at different k, never lower it under each other's launches.
    const size_t smem = (size_t)GQ * k * sizeof(int2);
    B2K_CUDA_OK(ctx, cudaFuncSetAttribute(k_knn_generic, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)((size_t)GQ * B2K_KNN_MAX_K * sizeof(int2))));
    k_knn_generic<<<(unsigned)nunits, G_NTHREADS, smem, s>>>(Q, X, xperm, d, k, units, part);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.generic_launches++;
  }
  ctx->stats.kernel_launches++;
  return B2K_OK;
}

int b2k_knn_refine_launch(b2k_ctx* ctx, const int2* part, int nl, const int32_t* slots, const int32_t* perm, int64_t nq,
                          int k, const float* Q, const float* X, int64_t n_items, int d, int64_t row0,
                          const int64_t* ids, KnnCand* cand, cudaStream_t s) {
  if (nq == 0) return B2K_OK;
  const size_t rf_smem = (size_t)RF_WARPS * 2 * k * 4;
  B2K_CUDA_OK(ctx, cudaFuncSetAttribute(k_knn_refine, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        RF_WARPS * 2 * B2K_KNN_MAX_K * 4));   // the largest k, as for k_knn_generic
  k_knn_refine<<<(unsigned)((nq + RF_WARPS - 1) / RF_WARPS), RF_WARPS * 32, rf_smem, s>>>(
      part, nl, slots, perm, nq, k, Q, X, n_items, d, row0, ids, cand);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  return B2K_OK;
}

int b2k_knn_merge_launch(b2k_ctx* ctx, const KnnCand* all, int nranks, int64_t nq_all, int64_t q0, int64_t nq_own, int k,
                         bool squared, bool fill, float* dist_out, int64_t* idx_out, cudaStream_t s) {
  if (nq_own == 0) return B2K_OK;
  k_knn_merge<<<(unsigned)((nq_own + RF_WARPS - 1) / RF_WARPS), RF_WARPS * 32, 0, s>>>(
      all, nranks, nq_all, q0, nq_own, k, squared, fill, dist_out, idx_out);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  return B2K_OK;
}

int b2k_knn_search_impl(b2k_ctx* ctx, const float* items, int64_t n_items, const int64_t* item_ids,
                        const float* queries, int64_t nq_local, int d, int k, float* dist_out, int64_t* idx_out,
                        cudaStream_t s) {
  const int nr = ctx->nranks;
  B2kTimer tm(ctx->time_kernels != 0);
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
    // judged against rank 0's d, on gathered values only: every rank reports the same rank and the same message
    if (sz[3 * r + 2] != sz[2])
      return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_knn_search: d differs between ranks (rank " + std::to_string(r) +
                                                " has d = " + std::to_string(sz[3 * r + 2]) + ", rank 0 has d = " +
                                                std::to_string(sz[2]) + ")");
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
  KnnLocal lp;
  B2K_TRY(knn_local_plan(ctx, n_items, nq_all, d, k, q_aligned, &lp));
  float* Qall = nullptr;
  KnnCand *cand = nullptr, *cand_all = nullptr;
  B2K_TRY(b2k_scratch_layout(ctx, "kNN", [&](B2kLayout& L) -> int {
    sz_dev = L.take<int64_t>((size_t)3 * (nr + 1));
    if (nr > 1) Qall = L.take<float>((size_t)nq_all * d, 1024);
    knn_local_take(L, &lp, n_items, nq_all, d, k);
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
  B2K_TRY(knn_local_run(ctx, lp, items, n_items, item_ids, Q, nq_all, d, k, row0, cand, tm, s));

  // ---- candidate allgather, merge of the own queries in rank order ----
  const KnnCand* all = cand;
  if (nr > 1) {
    B2K_TRY(b2k_comm_allgather_bytes(ctx, cand, cand_all, (size_t)nq_all * k * sizeof(KnnCand), s));
    all = cand_all;
  }
  tm.mark(5, s);
  B2K_TRY(b2k_knn_merge_launch(ctx, all, nr, nq_all, nr > 1 ? (int64_t)ctx->rank * nq_max : 0, nq_local, k, false,
                               false, dist_out, idx_out, s));
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

int b2k_knn_local_impl(b2k_ctx* ctx, const float* items, int64_t n_items, const float* queries, int64_t nq, int d,
                       int k, float* dist_out, int64_t* idx_out, cudaStream_t s) {
  if (nq == 0) return B2K_OK;
  B2kTimer tm(false);
  KnnLocal lp;
  B2K_TRY(knn_local_plan(ctx, n_items, nq, d, k, (reinterpret_cast<uintptr_t>(queries) & 15u) == 0, &lp));
  KnnCand* cand = nullptr;
  B2K_TRY(b2k_scratch_layout(ctx, "kNN local", [&](B2kLayout& L) -> int {
    knn_local_take(L, &lp, n_items, nq, d, k);
    cand = L.take<KnnCand>((size_t)nq * k);
    return B2K_OK;
  }));
  B2K_TRY(knn_local_run(ctx, lp, items, n_items, nullptr, queries, nq, d, k, 0, cand, tm, s));
  return b2k_knn_merge_launch(ctx, cand, 1, nq, 0, nq, k, false, false, dist_out, idx_out, s);
}
