// Random forests (include/b2kmeans.h "random forests"): every tree grows level by level from exact integer histograms
// of all ranks' rows.  Passes: a finite check, the sample select and its allgather, k_rf_bin (X -> uint8 bins), then per
// level and node group k_rf_hist_cluster (or k_rf_hist_generic), one int64 allreduce, the host split choice and
// k_rf_route.  k_rf_predict walks a flat forest for transform.
#include <cooperative_groups.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <vector>

#include "b2k_internal.cuh"
#include "b2k_rows.cuh"

namespace cg = cooperative_groups;

namespace {

constexpr int RF_CL = 8;                     // CTAs per cluster of the histogram pass
constexpr int RF_NT = 256;                   // threads per CTA of every kernel here
constexpr int64_t RF_FLUSH_ROWS = 1LL << 28; // rows a cluster may add between flushes: 12 (the weight cap) * 2^28 < 2^32,
                                             // so no u32 count can wrap; the u64 label sums then hold |S| <= 2^52.6
constexpr size_t RF_STAGE_MAX = 64 * 1024;   // bytes of one staged tile of the cluster pass

// The hash and the bootstrap draw of include/b2kmeans.h ("random forests"), on the host and the device alike.
__host__ __device__ __forceinline__ uint64_t rf_mix(uint64_t z) {
  z ^= z >> 30;
  z *= B2K_RF_MIX1;
  z ^= z >> 27;
  z *= B2K_RF_MIX2;
  return z ^ (z >> 31);
}
__host__ __device__ __forceinline__ uint64_t b2k_rf_hash(uint64_t seed, uint64_t stream, uint64_t tree,
                                                         uint64_t index) {
  return rf_mix(rf_mix(rf_mix(seed + stream * B2K_RF_GOLDEN) + tree * B2K_RF_GOLDEN) + index * B2K_RF_GOLDEN);
}
__device__ __forceinline__ int b2k_rf_poisson(uint32_t u) {
  const uint32_t cdf[B2K_RF_POISSON_CAP] = B2K_RF_POISSON_CDF;
  int k = 0;
  while (k < B2K_RF_POISSON_CAP && u >= cdf[k]) ++k;
  return k;
}

unsigned grid_for(int64_t work, int sm) {
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>((work + RF_NT - 1) / RF_NT, (int64_t)sm * 8));
}

// ---- checks: non-finite values of X and y, max |y| (as float bits: ordered like the values for |y| >= 0) ----
__global__ void __launch_bounds__(RF_NT) k_rf_check(const float* __restrict__ X, const float* __restrict__ y, int64_t n,
                                                    int d, unsigned long long* __restrict__ out /* bad X, bad y, max */) {
  unsigned long long bx = 0, by = 0;
  unsigned int mx = 0;
  const int64_t nd = n * d;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nd; i += (int64_t)gridDim.x * blockDim.x)
    bx += isfinite(X[i]) ? 0 : 1;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = y[i];
    if (!isfinite(v)) by++;
    else mx = max(mx, __float_as_uint(fabsf(v)));
  }
  for (int o = 16; o > 0; o >>= 1) {
    bx += __shfl_xor_sync(0xffffffffu, bx, o);
    by += __shfl_xor_sync(0xffffffffu, by, o);
    mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if ((threadIdx.x & 31) == 0) {
    if (bx) atomicAdd(out, bx);
    if (by) atomicAdd(out + 1, by);
    if (mx) atomicMax(out + 2, (unsigned long long)mx);
  }
}

// ---- sample select: rows with h(seed, SAMPLE, 0, row0 + r) < thr; count, then copy (order-free: sorted later) ----
__global__ void __launch_bounds__(RF_NT) k_rf_sample(const float* __restrict__ X, int64_t n, int d, int64_t row0,
                                                     uint64_t seed, uint64_t thr, int all, float* __restrict__ out,
                                                     unsigned long long* __restrict__ count) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    if (!all && b2k_rf_hash(seed, B2K_RF_SAMPLE, 0, (uint64_t)(row0 + r)) >= thr) continue;
    const unsigned long long slot = atomicAdd(count, 1ull);
    if (out != nullptr)
      for (int f = 0; f < d; ++f) out[slot * d + f] = X[r * d + f] + 0.0f;   // -0.0 -> +0.0
  }
}

// ---- k_rf_bin: bins [n][d] uint8 = #{thresholds of feature f < x}, binary search over thresholds in shared memory
// (SMEM) or through L1 ----
template <bool SMEM>
__global__ void __launch_bounds__(RF_NT) k_rf_bin(const float* __restrict__ X, int64_t n, int d,
                                                  const float* __restrict__ thr /* [d][TS] */, int TS,
                                                  const int* __restrict__ nthr, uint8_t* __restrict__ bins) {
  extern __shared__ float sthr[];
  const float* T = thr;
  if constexpr (SMEM) {
    for (int i = threadIdx.x; i < d * TS; i += blockDim.x) sthr[i] = thr[i];
    __syncthreads();
    T = sthr;
  }
  const int64_t nd = n * d;
  for (int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4; i0 < nd; i0 += (int64_t)gridDim.x * blockDim.x * 4) {
    float v[4];
    if (i0 + 4 <= nd && (reinterpret_cast<uintptr_t>(X + i0) & 15) == 0) {
      const float4 q = __ldcs(reinterpret_cast<const float4*>(X + i0));
      v[0] = q.x, v[1] = q.y, v[2] = q.z, v[3] = q.w;
    } else {
      for (int u = 0; u < 4; ++u) v[u] = i0 + u < nd ? X[i0 + u] : 0.f;
    }
    uint32_t packed = 0;
    int f = (int)(i0 % d);
    for (int u = 0; u < 4; ++u) {
      const float* t = T + (size_t)f * TS;
      int lo = 0, hi = __ldg(nthr + f);
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (t[mid] < v[u]) lo = mid + 1;
        else hi = mid;
      }
      packed |= (uint32_t)lo << (8 * u);
      if (++f == d) f = 0;
    }
    if (i0 + 4 <= nd && (reinterpret_cast<uintptr_t>(bins + i0) & 3) == 0) {
      *reinterpret_cast<uint32_t*>(bins + i0) = packed;
    } else {
      for (int u = 0; u < 4 && i0 + u < nd; ++u) bins[i0 + u] = (uint8_t)(packed >> (8 * u));
    }
  }
}

// ---- per (tree, row): bootstrap weight, node (0 = the tree's root at level 0), label on its integer grid ----
__global__ void __launch_bounds__(RF_NT) k_rf_init(const float* __restrict__ y, int64_t n, int T, int64_t row0,
                                                   uint64_t seed, int bootstrap, int regression, double yscale,
                                                   uint8_t* __restrict__ wt, int32_t* __restrict__ nid,
                                                   int32_t* __restrict__ lab, unsigned long long* __restrict__ pairs) {
  unsigned long long cnt = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n * T; i += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(i / n);
    const int64_t r = i - (int64_t)t * n;
    const int w = bootstrap ? b2k_rf_poisson((uint32_t)(b2k_rf_hash(seed, B2K_RF_BOOT, t, (uint64_t)(row0 + r)) >> 32))
                            : 1;
    wt[i] = (uint8_t)w;
    nid[i] = w > 0 ? t : -1;   // level 0 lists the roots in tree order
    cnt += w > 0;
    if (t == 0) lab[r] = regression ? __double2int_rn((double)y[r] * yscale) : (int32_t)y[r];
  }
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(pairs, cnt);
}

struct HistArgs {
  const uint8_t* bins;     // [n][d]
  const int32_t* nid;      // [T][n] level node or -1
  const uint8_t* wt;       // [T][n]
  const int32_t* lab;      // [n] class index or y_q
  const int32_t* subset;   // [level nodes][k] features of each node
  unsigned long long* H;   // [group nodes][k][B][V] int64 (two's complement in u64)
  int64_t n;
  int d, T, k, B, V, g0, g1, regression;
};

// One (row, tree) update of the group's histogram: add(word index, value) for each of the node's k feature slots.
template <typename Add>
__device__ __forceinline__ void rf_update(const HistArgs& a, int node, int w, int lab, const uint8_t* brow, Add add) {
  const int* sub = a.subset + (size_t)node * a.k;
  const int64_t base = (int64_t)(node - a.g0) * a.k;
  for (int s = 0; s < a.k; ++s) {
    const int b = brow[__ldg(sub + s)];
    const int64_t idx = ((base + s) * a.B + b) * a.V;
    if (a.regression) {
      add(idx, (unsigned long long)w);
      add(idx + 1, (unsigned long long)(long long)(w * lab));
    } else {
      add(idx + lab, (unsigned long long)w);
    }
  }
}

// The generic pass: every update is an int64 atomic on the global histogram.
__global__ void __launch_bounds__(RF_NT) k_rf_hist_generic(HistArgs a) {
  const int64_t total = a.n * a.T;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int node = a.nid[i];
    if (node < a.g0 || node >= a.g1) continue;
    const int64_t r = i % a.n;
    rf_update(a, node, a.wt[i], a.lab[r], a.bins + r * a.d,
              [&](int64_t idx, unsigned long long v) { atomicAdd(a.H + idx, v); });
  }
}

// The cluster pass.  The group's histogram (words [0, words)) is sharded over the cluster's CTAs: CTA q owns words
// [q wpc, (q + 1) wpc) in its shared memory (Word = u32 counts, or u64 for regression's {W, S}).  Each CTA stages tiles
// of TR rows (bins for all d features, node and weight for all T trees, labels) and adds every update into the owning
// CTA's shared memory with a remote shared atomic.  Every `flush_tiles` tiles per CTA (at most RF_FLUSH_ROWS rows per
// cluster), the cluster synchronises and each CTA adds its nonzero words into the global int64 histogram and clears them.
template <typename Word>
__global__ void __launch_bounds__(RF_NT) k_rf_hist_cluster(HistArgs a, int64_t words, int wpc, int TR, int flush_tiles) {
  cg::cluster_group cl = cg::this_cluster();
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Word* hist = reinterpret_cast<Word*>(smem_raw);
  unsigned char* stage = smem_raw + (((size_t)wpc * sizeof(Word) + 15) / 16) * 16;
  uint8_t* sb = stage;                                                          // [TR][d]
  int32_t* sn = reinterpret_cast<int32_t*>(stage + (((size_t)TR * a.d + 15) / 16) * 16);   // [T][TR]
  int32_t* sl = sn + (size_t)a.T * TR;                                          // [TR]
  uint8_t* sw = reinterpret_cast<uint8_t*>(sl + TR);                            // [T][TR]
  const unsigned q = cl.block_rank();
  const int64_t my0 = (int64_t)q * wpc;
  for (int i = threadIdx.x; i < wpc; i += blockDim.x) hist[i] = 0;
  const int64_t ntiles = (a.n + TR - 1) / TR;
  const int64_t stride = gridDim.x;
  // every CTA of a cluster runs the same number of rounds (the cluster's first CTA has the most tiles)
  const int64_t first = (int64_t)blockIdx.x - q;
  const int64_t max_tiles = first < ntiles ? (ntiles - first + stride - 1) / stride : 0;
  const int64_t rounds = (max_tiles + flush_tiles - 1) / flush_tiles;
  cl.sync();
  int64_t tile = blockIdx.x;
  for (int64_t rd = 0; rd < rounds; ++rd) {
    for (int j = 0; j < flush_tiles && tile < ntiles; ++j, tile += stride) {
      const int64_t r0 = tile * TR;
      const int rows = a.n - r0 < TR ? (int)(a.n - r0) : TR;
      __syncthreads();   // the previous tile's updates have read the stage
      for (int i = threadIdx.x; i < rows * a.d; i += blockDim.x) sb[i] = a.bins[r0 * a.d + i];
      for (int i = threadIdx.x; i < a.T * TR; i += blockDim.x) {
        const int t = i / TR, r = i - t * TR;
        const int64_t g = (int64_t)t * a.n + r0 + r;
        sn[i] = r < rows ? a.nid[g] : -1;
        sw[i] = r < rows ? a.wt[g] : 0;
      }
      for (int i = threadIdx.x; i < rows; i += blockDim.x) sl[i] = a.lab[r0 + i];
      __syncthreads();
      for (int i = threadIdx.x; i < a.T * TR; i += blockDim.x) {
        const int node = sn[i];
        if (node < a.g0 || node >= a.g1) continue;
        const int r = i % TR;
        rf_update(a, node, sw[i], sl[r], sb + (size_t)r * a.d, [&](int64_t idx, unsigned long long v) {
          const unsigned u = (unsigned)idx;   // < words <= RF_CL wpc, far below 2^32
          const unsigned owner = u / (unsigned)wpc;
          Word* dst = cl.map_shared_rank(hist, owner);
          atomicAdd(dst + (u - owner * (unsigned)wpc), (Word)v);
        });
      }
    }
    cl.sync();   // every update of this round has landed
    for (int i = threadIdx.x; i < wpc && my0 + i < words; i += blockDim.x) {
      const Word v = hist[i];
      if (v != 0) {
        atomicAdd(a.H + my0 + i, (unsigned long long)v);
        hist[i] = 0;
      }
    }
    cl.sync();   // cleared before the next round adds
  }
}

// ---- route every (tree, row) of this level to its node on the next level, or -1 ----
struct RouteInfo {
  int32_t feature;   // -1: no further histogram for this node's rows
  int32_t bin;       // left: bin <= this
  int32_t left;      // next-level index of the left child or -1 (its rows need no histogram)
  int32_t right;
};
__global__ void __launch_bounds__(RF_NT) k_rf_route(const uint8_t* __restrict__ bins, int64_t n, int d, int T,
                                                    const uint8_t* __restrict__ wt, const RouteInfo* __restrict__ info,
                                                    int32_t* __restrict__ nid, unsigned long long* __restrict__ pairs) {
  unsigned long long cnt = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n * T; i += (int64_t)gridDim.x * blockDim.x) {
    const int node = nid[i];
    if (node < 0) continue;
    const RouteInfo ri = info[node];
    int next = -1;
    if (ri.feature >= 0) {
      const int64_t r = i % n;
      next = bins[r * d + ri.feature] <= ri.bin ? ri.left : ri.right;
    }
    nid[i] = next;
    cnt += next >= 0 && wt[i] > 0;
  }
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(pairs, cnt);
}

// ---- prediction ----
using PNode = B2kPNode;
template <bool SMEM>
__global__ void __launch_bounds__(RF_NT) k_rf_predict(const float* __restrict__ X, int64_t n, int d, int T,
                                                      const int64_t* __restrict__ off, const PNode* __restrict__ nodes,
                                                      int64_t n_nodes, const double* __restrict__ value, int V, int cls,
                                                      double* __restrict__ raw, double* __restrict__ prob,
                                                      double* __restrict__ pred) {
  extern __shared__ PNode snodes[];
  const PNode* P = nodes;
  if constexpr (SMEM) {
    for (int64_t i = threadIdx.x; i < n_nodes; i += blockDim.x) snodes[i] = nodes[i];
    __syncthreads();
    P = snodes;
  }
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    const float* x = X + r * d;
    double acc = 0.0;
    if (cls)
      for (int k = 0; k < V; ++k) raw[r * V + k] = 0.0;
    for (int t = 0; t < T; ++t) {
      const PNode* tree = P + __ldg(off + t);
      const int i = b2k_rf_leaf(tree, B2kFeatLdg{x});
      const int64_t o = __ldg(off + t);
      const double* v = value + (o + i) * V;
      if (cls) {
        for (int k = 0; k < V; ++k) raw[r * V + k] = __dadd_rn(raw[r * V + k], __ldg(v + k));
      } else {
        acc = __dadd_rn(acc, __ldg(v));
      }
    }
    if (cls) {
      double tot = 0.0;   // b2k_rf_class_best's order, kept inline: the call form spills here
      int best = 0;
      for (int k = 0; k < V; ++k) {
        const double a = raw[r * V + k];
        tot = __dadd_rn(tot, a);
        if (a > raw[r * V + best]) best = k;
      }
      for (int k = 0; k < V; ++k) prob[r * V + k] = tot != 0.0 ? __ddiv_rn(raw[r * V + k], tot) : 0.0;
      pred[r] = (double)best;
    } else {
      pred[r] = __ddiv_rn(acc, (double)T);
    }
  }
}

// ---- host: thresholds, feature subsets, impurities and the split choice (bit-exact with tests/rf_oracle.py) ----
float mid32(float a, float b) {
  const float t = (float)(((double)a + (double)b) / 2.0);
  return t == b ? a : t;
}

void thresholds_of(std::vector<float>& s /* the feature's sample, sorted in place */, int max_bins,
                   std::vector<float>* out) {
  out->clear();
  std::sort(s.begin(), s.end());
  const int64_t m = (int64_t)s.size();
  std::vector<float> v;
  for (int64_t i = 0; i < m; ++i)
    if (i == 0 || s[i] != s[i - 1]) v.push_back(s[i]);
  if ((int64_t)v.size() <= max_bins) {
    for (size_t i = 0; i + 1 < v.size(); ++i) out->push_back(mid32(v[i], v[i + 1]));
    return;
  }
  for (int j = 1; j < max_bins; ++j) {
    const int64_t p = (int64_t)j * m / max_bins;
    const float t = mid32(s[p - 1], s[p]);
    if (out->empty() || out->back() != t) out->push_back(t);
  }
}

void feature_subset(uint64_t seed, int tree, int64_t heap, int d, int k, std::vector<int>& perm, int* out) {
  for (int j = 0; j < d; ++j) perm[j] = j;
  if (k < d)
    for (int j = 0; j < k; ++j) {
      const uint64_t h = b2k_rf_hash(seed, B2K_RF_FEAT, (uint64_t)tree, (uint64_t)heap * (uint64_t)d + (uint64_t)j);
      const int r = j + (int)(h % (uint64_t)(d - j));
      std::swap(perm[j], perm[r]);
    }
  std::copy(perm.begin(), perm.begin() + k, out);
  std::sort(out, out + k);
}

// The products and sums below must round once each.  They run on the host, built for the x86-64 baseline, which has no
// fused multiply-add to contract them into.
double rf_log2(double p) {
  int e = 0;
  double m = std::frexp(p, &e);
  if (m < 0.7071067811865476) {
    m = m * 2.0;
    e = e - 1;
  }
  const double z = (m - 1.0) / (m + 1.0);
  const double z2 = z * z;
  double a = 1.0 / 25.0;
  for (int i = 11; i >= 0; --i) {
    a = a * z2;
    a = a + 1.0 / (double)(2 * i + 1);
  }
  double l = z * a;
  l = l * 2.0;
  l = l * 1.4426950408889634;
  return l + (double)e;
}

double impurity(int imp, const int64_t* c, int V, int64_t N) {
  const double Nd = (double)N;
  double s = 0.0;
  for (int k = 0; k < V; ++k) {
    if (c[k] == 0) continue;
    const double p = (double)c[k] / Nd;
    if (imp == 0) {
      const double pp = p * p;
      s = s + pp;
    } else {
      const double t = p * rf_log2(p);
      s = s - t;
    }
  }
  return imp == 0 ? 1.0 - s : s;
}

double class_gain(double imp_p, int imp, const int64_t* cl, const int64_t* cr, int V, int64_t NL, int64_t NR,
                  int64_t N) {
  const double il = impurity(imp, cl, V, NL), ir = impurity(imp, cr, V, NR);
  const double a = (double)NL / (double)N, b = (double)NR / (double)N;
  const double t1 = a * il, t2 = b * ir;
  const double g = imp_p - t1;
  return g - t2;
}

double var_gain(int64_t SL, int64_t WL, int64_t S, int64_t W, double q2) {
  const __int128 D = (__int128)SL * W - (__int128)S * WL;
  double g = (double)D;
  g = g * g;
  const double den = (double)WL * (double)(W - WL);
  g = g / den;
  g = g / (double)W;
  g = g / (double)W;
  return g * q2;
}

struct Node {   // one node of a tree under construction
  int32_t feature = -1;
  float threshold = 0.f;
  int32_t left = -1, right = -1;
  double gain = 0.0;
  int64_t count = 0;
  std::vector<int64_t> stat;   // classification: c_k; regression: {W, S}
  int64_t heap = 1;
  int depth = 0;
};

struct Forest {
  int V = 1;
  std::vector<int64_t> off;
  std::vector<int32_t> feature, children;
  std::vector<float> threshold;
  std::vector<double> gain, value;
  std::vector<int64_t> count;
};

struct Timer {
  bool on;
  std::vector<cudaEvent_t> ev;
  explicit Timer(bool enable) : on(enable) {}
  ~Timer() {
    for (auto e : ev) cudaEventDestroy(e);
  }
  int mark(cudaStream_t s) {   // index of a new event recorded on s (-1 when off)
    if (!on) return -1;
    cudaEvent_t e;
    cudaEventCreate(&e);
    cudaEventRecord(e, s);
    ev.push_back(e);
    return (int)ev.size() - 1;
  }
  double ms(int a, int b) const {
    float t = 0.f;
    if (on && a >= 0 && b >= 0) cudaEventElapsedTime(&t, ev[a], ev[b]);
    return (double)t;
  }
};

double since(std::chrono::steady_clock::time_point t0) {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

}  // namespace

int b2k_rf_fit_impl(b2k_ctx* ctx, const float* X, const float* y, int64_t n, int d, const b2k_rf_params& p,
                    int* n_values_out, int64_t* n_nodes_out, double* level_ms_out, int64_t* level_updates_out,
                    cudaStream_t s) {
  const auto t_entry = std::chrono::steady_clock::now();
  const int nr = ctx->nranks;
  Timer tm(ctx->time_kernels != 0);
  double ms_hist = 0.0, ms_allreduce = 0.0;
  // ---- sizes and checks of every rank; every error is decided on them, identically on every rank ----
  constexpr int NS = 5;   // n_local, d, non-finite X, non-finite y, max |y| bits
  DevBuf b_sz;
  int64_t* sz_dev;
  B2K_TRY(dalloc(ctx, b_sz, (size_t)NS * (nr + 1), s, &sz_dev));
  const int64_t mine[2] = {n, d};
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(sz_dev, mine, sizeof(mine), cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaMemsetAsync(sz_dev + 2, 0, 3 * sizeof(int64_t), s));
  if (n > 0) {
    k_rf_check<<<grid_for(n * d, ctx->sm_count), RF_NT, 0, s>>>(X, y, n, d,
                                                               reinterpret_cast<unsigned long long*>(sz_dev + 2));
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
  }
  B2K_TRY(b2k_comm_allgather_i64(ctx, sz_dev, sz_dev + NS, NS, s));
  std::vector<int64_t> sz((size_t)NS * nr);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(sz.data(), sz_dev + NS, sz.size() * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  if (p.max_depth < 0) return b2k_fail(ctx, B2K_ERR_INVALID, "maxDepth given invalid value " + std::to_string(p.max_depth));
  if (p.max_bins < 2 || p.max_bins > B2K_RF_MAX_BINS)
    return b2k_fail(ctx, B2K_ERR_INVALID, "maxBins given invalid value " + std::to_string(p.max_bins));
  if (p.max_depth > B2K_RF_MAX_DEPTH)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "maxDepth " + std::to_string(p.max_depth) + " > 16 is not supported");
  if (p.n_trees < 1) return b2k_fail(ctx, B2K_ERR_INVALID, "numTrees given invalid value " + std::to_string(p.n_trees));
  if (p.min_instances < 1)
    return b2k_fail(ctx, B2K_ERR_INVALID, "minInstancesPerNode given invalid value " + std::to_string(p.min_instances));
  if (!(std::isfinite(p.min_info_gain) && p.min_info_gain >= 0.0))
    return b2k_fail(ctx, B2K_ERR_INVALID, "minInfoGain given invalid value " + std::to_string(p.min_info_gain));
  if (p.impurity < 0 || p.impurity > 2)
    return b2k_fail(ctx, B2K_ERR_INVALID, "impurity given invalid value " + std::to_string(p.impurity));
  if (p.features_per_node < 1 || p.features_per_node > d)
    return b2k_fail(ctx, B2K_ERR_INVALID, "features per node " + std::to_string(p.features_per_node) +
                                              " outside [1, d = " + std::to_string(d) + "]");
  int64_t n_total = 0, row0 = 0, bad_x = 0, bad_y = 0;
  uint32_t ymax_bits = 0;
  for (int r = 0; r < nr; ++r) {
    const int64_t* q = &sz[(size_t)NS * r];
    if (q[0] == 0)
      return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_rf_fit: empty partition (rank " + std::to_string(r) +
                                                " has n_local == 0)");
    if (q[1] != sz[1])
      return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_rf_fit: d differs between ranks (rank " + std::to_string(r) +
                                                " has d = " + std::to_string(q[1]) + ", rank 0 has d = " +
                                                std::to_string(sz[1]) + ")");
    if (r < ctx->rank) row0 += q[0];
    n_total += q[0];
    bad_x += q[2];
    bad_y += q[3];
    ymax_bits = std::max(ymax_bits, (uint32_t)q[4]);
  }
  if (bad_x || bad_y) return b2k_fail(ctx, B2K_ERR_INVALID, "RandomForest input contains NaN or infinity");
  const bool regression = p.impurity == 2;
  const int T = p.n_trees, k = p.features_per_node;
  int V = 2;   // histogram words per (node, slot, bin)
  int n_values = 1;
  double yscale = 1.0, q2 = 1.0, qv = 1.0;
  if (!regression) {
    std::vector<double> cls(B2K_LOGREG_MAX_CLASSES);
    std::vector<int64_t> cnt(B2K_LOGREG_MAX_CLASSES);
    int ncls = 0;
    int64_t nt = 0;
    B2K_TRY(b2k_logreg_labels_impl(ctx, y, n, cls.data(), cnt.data(), &ncls, &nt, s));
    n_values = V = (int)cls[ncls - 1] + 1;
  } else if (ymax_bits != 0) {
    float ym;
    std::memcpy(&ym, &ymax_bits, 4);
    int e = 0;
    const double m = std::frexp((double)ym, &e);   // 2^(e-1) <= ym < 2^e
    if (m == 0.5) e -= 1;                           // now 2^(e-1) < ym <= 2^e
    yscale = std::ldexp(1.0, 24 - e);
    qv = std::ldexp(1.0, e - 24);
    q2 = qv * qv;
  }
  // ---- sample, thresholds ----
  const double M = std::max<double>((double)p.max_bins * p.max_bins, 10000.0);
  const bool all_rows = M >= (double)n_total;
  const uint64_t thr_h = all_rows ? ~0ull : (uint64_t)std::ldexp(M / (double)n_total, 64);
  DevBuf b_cnt, b_sample, b_gath;
  unsigned long long* cnt_dev;
  B2K_TRY(dalloc(ctx, b_cnt, 4, s, &cnt_dev));
  B2K_CUDA_OK(ctx, cudaMemsetAsync(cnt_dev, 0, 4 * 8, s));
  k_rf_sample<<<grid_for(n, ctx->sm_count), RF_NT, 0, s>>>(X, n, d, row0, p.seed, thr_h, all_rows, nullptr, cnt_dev);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  std::vector<int64_t> scnt(nr);
  {
    int64_t* g;
    DevBuf b_g;
    B2K_TRY(dalloc(ctx, b_g, (size_t)nr, s, &g));
    B2K_TRY(b2k_comm_allgather_i64(ctx, reinterpret_cast<int64_t*>(cnt_dev), g, 1, s));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(scnt.data(), g, 8 * (size_t)nr, cudaMemcpyDeviceToHost, s));
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  }
  const int64_t smax = *std::max_element(scnt.begin(), scnt.end());
  float *sample, *gath;
  B2K_TRY(dalloc(ctx, b_sample, (size_t)std::max<int64_t>(smax, 1) * d, s, &sample));
  B2K_TRY(dalloc(ctx, b_gath, (size_t)std::max<int64_t>(smax, 1) * d * nr, s, &gath));
  B2K_CUDA_OK(ctx, cudaMemsetAsync(cnt_dev, 0, 8, s));
  k_rf_sample<<<grid_for(n, ctx->sm_count), RF_NT, 0, s>>>(X, n, d, row0, p.seed, thr_h, all_rows, sample, cnt_dev);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches += 2;
  B2K_TRY(b2k_comm_allgather_bytes(ctx, sample, gath, (size_t)std::max<int64_t>(smax, 1) * d * 4, s));
  std::vector<float> hs((size_t)std::max<int64_t>(smax, 1) * d * nr);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(hs.data(), gath, hs.size() * 4, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  int64_t m_total = 0;
  for (int r = 0; r < nr; ++r) m_total += scnt[r];
  std::vector<std::vector<float>> thr(d);
  int nb_max = 1;
  {
    std::vector<float> col((size_t)m_total);
    for (int f = 0; f < d; ++f) {
      size_t o = 0;
      for (int r = 0; r < nr; ++r)
        for (int64_t i = 0; i < scnt[r]; ++i) col[o++] = hs[((size_t)r * std::max<int64_t>(smax, 1) + i) * d + f];
      thresholds_of(col, p.max_bins, &thr[f]);
      nb_max = std::max(nb_max, (int)thr[f].size() + 1);
    }
  }
  const int TS = std::max(1, p.max_bins - 1);
  std::vector<float> thr_flat((size_t)d * TS, 0.f);
  std::vector<int> nthr(d);
  for (int f = 0; f < d; ++f) {
    nthr[f] = (int)thr[f].size();
    std::copy(thr[f].begin(), thr[f].end(), thr_flat.begin() + (size_t)f * TS);
  }
  const double ms_edges = since(t_entry);
  // ---- bins ----
  DevBuf b_thr, b_nthr, b_bins, b_wt, b_nid, b_lab, b_pairs;
  float* thr_dev;
  int* nthr_dev;
  uint8_t *bins, *wt;
  int32_t *nid, *lab;
  unsigned long long* pairs_dev;
  B2K_TRY(dalloc(ctx, b_thr, thr_flat.size(), s, &thr_dev));
  B2K_TRY(dalloc(ctx, b_nthr, (size_t)d, s, &nthr_dev));
  B2K_TRY(dalloc(ctx, b_bins, (size_t)n * d, s, &bins));
  B2K_TRY(dalloc(ctx, b_wt, (size_t)n * T, s, &wt));
  B2K_TRY(dalloc(ctx, b_nid, (size_t)n * T, s, &nid));
  B2K_TRY(dalloc(ctx, b_lab, (size_t)n, s, &lab));
  B2K_TRY(dalloc(ctx, b_pairs, (size_t)B2K_RF_MAX_DEPTH + 2, s, &pairs_dev));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(thr_dev, thr_flat.data(), thr_flat.size() * 4, cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(nthr_dev, nthr.data(), (size_t)d * 4, cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaMemsetAsync(pairs_dev, 0, 8 * (B2K_RF_MAX_DEPTH + 2), s));
  const int ev_bin0 = tm.mark(s);
  {
    const size_t smem = thr_flat.size() * 4;
    const unsigned g = grid_for((n * d + 3) / 4, ctx->sm_count);
    if (smem <= 96 * 1024) {
      B2K_CUDA_OK(ctx, cudaFuncSetAttribute(k_rf_bin<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      k_rf_bin<true><<<g, RF_NT, smem, s>>>(X, n, d, thr_dev, TS, nthr_dev, bins);
    } else {
      k_rf_bin<false><<<g, RF_NT, 0, s>>>(X, n, d, thr_dev, TS, nthr_dev, bins);
    }
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
  }
  const int ev_bin1 = tm.mark(s);
  k_rf_init<<<grid_for(n * T, ctx->sm_count), RF_NT, 0, s>>>(y, n, T, row0, p.seed, p.bootstrap, regression, yscale, wt,
                                                             nid, lab, pairs_dev);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  // ---- histogram pass plan: words per node, the cluster's capacity, node groups ----
  const int B = nb_max;
  const int64_t node_words = (int64_t)k * B * V;
  const size_t word_bytes = regression ? 8 : 4;
  int TR = 128;
  auto stage_bytes = [&](int tr) {
    return (((size_t)tr * d + 15) / 16) * 16 + (size_t)tr * T * 5 + (size_t)tr * 4 + 16;
  };
  while (TR > 8 && stage_bytes(TR) > RF_STAGE_MAX) TR /= 2;
  const size_t stage = stage_bytes(TR);
  const size_t optin = ctx->smem_optin ? ctx->smem_optin : 227 * 1024;
  const int64_t wpc_cap = stage + 1024 <= optin ? (int64_t)((optin - stage - 1024) / word_bytes) : 0;
  const bool cluster_fits = stage <= RF_STAGE_MAX && node_words <= wpc_cap * RF_CL;
  if (ctx->kernel_path == B2K_PATH_FUSED && !cluster_fits)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "b2k_rf_fit: one node's histogram (" + std::to_string(node_words) +
                                                  " words) exceeds the cluster pass");
  const bool use_cluster = cluster_fits && ctx->kernel_path != B2K_PATH_GENERIC;
  ctx->stats.last_path = use_cluster ? B2K_PATH_FUSED : B2K_PATH_GENERIC;
  int64_t group_cap = use_cluster ? (wpc_cap * RF_CL) / node_words
                                  : std::max<int64_t>(1, ((int64_t)1 << 24) / std::max<int64_t>(node_words, 1));
  if (ctx->rf_group_nodes > 0) group_cap = std::min<int64_t>(group_cap, ctx->rf_group_nodes);
  DevBuf b_H, b_sub, b_route;
  unsigned long long* H;
  B2K_TRY(dalloc(ctx, b_H, (size_t)(group_cap * node_words), s, &H));
  int grid_cl = 0;
  int flush_tiles = 1;
  if (use_cluster) {
    const size_t smem_cl = ((wpc_cap * word_bytes + 15) / 16) * 16 + stage;
    auto kern = regression ? (void*)k_rf_hist_cluster<unsigned long long> : (void*)k_rf_hist_cluster<unsigned int>;
    B2K_CUDA_OK(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cl));
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(RF_CL);
    cfg.blockDim = dim3(RF_NT);
    cfg.dynamicSmemBytes = smem_cl;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = RF_CL;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int nclusters = 0;
    B2K_CUDA_OK(ctx, cudaOccupancyMaxActiveClusters(&nclusters, kern, &cfg));
    grid_cl = std::max(1, nclusters) * RF_CL;
    if (ctx->grid_limit > 0) grid_cl = std::max(RF_CL, std::min(grid_cl, ctx->grid_limit / RF_CL * RF_CL));
    flush_tiles = (int)std::max<int64_t>(1, RF_FLUSH_ROWS / ((int64_t)RF_CL * TR));
    if (ctx->rf_flush_tiles > 0) flush_tiles = std::min(flush_tiles, ctx->rf_flush_tiles);
  }
  // ---- trees, level by level ----
  std::vector<std::vector<Node>> trees(T);
  std::vector<std::pair<int, int>> level;   // (tree, node) of this level's nodes that need a histogram, in order
  for (int t = 0; t < T; ++t) {
    trees[t].emplace_back();
    level.emplace_back(t, 0);
  }
  std::vector<int> perm(d);
  std::vector<int64_t> hbuf;
  const int64_t min_inst = p.min_instances;
  int levels = 0;
  int64_t passes = 0, ar_bytes = 0;
  if (level_ms_out) std::fill(level_ms_out, level_ms_out + p.max_depth + 1, 0.0);
  std::vector<int64_t> pairs_h((size_t)B2K_RF_MAX_DEPTH + 2, 0);
  // a node needs a histogram when it may still split: below max depth, of weight >= 2 min_instances and not pure; the
  // root always gets one (its statistics come from it)
  auto may_split = [&](const Node& nd) {
    if (nd.depth >= p.max_depth || nd.count < 2 * min_inst) return false;
    if (!regression) {
      int nz = 0;
      for (int c = 0; c < V; ++c) nz += nd.stat[c] > 0;
      if (nz <= 1) return false;
    }
    return true;
  };
  for (int depth = 0; !level.empty(); ++depth) {
    ++levels;
    const int nl = (int)level.size();
    std::vector<int32_t> sub((size_t)nl * k);
    for (int i = 0; i < nl; ++i) {
      const Node& nd = trees[level[i].first][level[i].second];
      feature_subset(p.seed, level[i].first, nd.heap, d, k, perm, &sub[(size_t)i * k]);
    }
    int32_t* sub_dev;
    B2K_TRY(dalloc(ctx, b_sub, sub.size(), s, &sub_dev));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(sub_dev, sub.data(), sub.size() * 4, cudaMemcpyHostToDevice, s));
    std::vector<RouteInfo> route(nl, RouteInfo{-1, 0, -1, -1});
    std::vector<std::pair<int, int>> next;
    double ms_level = 0.0;
    for (int g0 = 0; g0 < nl; g0 += (int)group_cap) {
      const int g1 = (int)std::min<int64_t>(nl, g0 + group_cap);
      const int64_t words = (int64_t)(g1 - g0) * node_words;
      B2K_CUDA_OK(ctx, cudaMemsetAsync(H, 0, (size_t)words * 8, s));
      HistArgs a{bins, nid, wt, lab, sub_dev, H, n, d, T, k, B, V, g0, g1, regression ? 1 : 0};
      const int e0 = tm.mark(s);
      if (use_cluster) {
        const int wpc = (int)((words + RF_CL - 1) / RF_CL);
        const size_t smem_cl = ((wpc_cap * word_bytes + 15) / 16) * 16 + stage;
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = dim3((unsigned)grid_cl);
        cfg.blockDim = dim3(RF_NT);
        cfg.dynamicSmemBytes = smem_cl;
        cfg.stream = s;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = RF_CL;
        attr[0].val.clusterDim.y = 1;
        attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        if (regression)
          B2K_CUDA_OK(ctx, cudaLaunchKernelEx(&cfg, k_rf_hist_cluster<unsigned long long>, a, words, wpc, TR, flush_tiles));
        else
          B2K_CUDA_OK(ctx, cudaLaunchKernelEx(&cfg, k_rf_hist_cluster<unsigned int>, a, words, wpc, TR, flush_tiles));
        ctx->stats.fused_tc_launches++;
      } else {
        k_rf_hist_generic<<<grid_for(n * T, ctx->sm_count), RF_NT, 0, s>>>(a);
        ctx->stats.generic_launches++;
      }
      B2K_CUDA_OK(ctx, cudaGetLastError());
      ctx->stats.kernel_launches++;
      const int e1 = tm.mark(s);
      B2K_TRY(b2k_comm_allreduce_i64(ctx, reinterpret_cast<int64_t*>(H), (size_t)words, s));
      const int e2 = tm.mark(s);
      ++passes;
      ar_bytes += nr > 1 ? words * 8 : 0;
      hbuf.resize((size_t)words);
      B2K_CUDA_OK(ctx, cudaMemcpyAsync(hbuf.data(), H, (size_t)words * 8, cudaMemcpyDeviceToHost, s));
      B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
      ms_hist += tm.ms(e0, e1);
      ms_level += tm.ms(e0, e1);
      ms_allreduce += tm.ms(e1, e2);
      // ---- the split of each node of the group ----
      for (int i = g0; i < g1; ++i) {
        const int t = level[i].first;
        std::vector<Node>& tree = trees[t];
        const int ni = level[i].second;
        const int64_t* h = hbuf.data() + (size_t)(i - g0) * node_words;
        if (ni == 0 && depth == 0) {   // the root's statistics: any slot's bins sum to them
          tree[0].stat.assign(V, 0);
          for (int b = 0; b < B; ++b)
            for (int v = 0; v < V; ++v) tree[0].stat[v] += h[(size_t)b * V + v];
          if (regression) tree[0].count = tree[0].stat[0];
          else {
            tree[0].count = 0;
            for (int v = 0; v < V; ++v) tree[0].count += tree[0].stat[v];
          }
          if (!may_split(tree[0])) continue;
        }
        const Node nd = tree[ni];
        const int64_t N = nd.count;
        double imp_p = 0.0;
        if (!regression) imp_p = impurity(p.impurity, nd.stat.data(), V, N);
        double best = -INFINITY;
        int bs = -1, bb = -1;
        std::vector<int64_t> left(V), right(V), bestl(V);
        for (int sl = 0; sl < k; ++sl) {
          const int f = sub[(size_t)i * k + sl];
          std::fill(left.begin(), left.end(), 0);
          for (int b = 0; b < nthr[f]; ++b) {   // candidate b: left = bins 0..b
            for (int v = 0; v < V; ++v) left[v] += h[((size_t)sl * B + b) * V + v];
            int64_t NL = 0;
            if (regression) NL = left[0];
            else
              for (int v = 0; v < V; ++v) NL += left[v];
            const int64_t NR = N - NL;
            if (NL < min_inst || NR < min_inst) continue;
            double g;
            if (regression) {
              g = var_gain(left[1], NL, nd.stat[1], N, q2);
            } else {
              for (int v = 0; v < V; ++v) right[v] = nd.stat[v] - left[v];
              g = class_gain(imp_p, p.impurity, left.data(), right.data(), V, NL, NR, N);
            }
            if (g > best) {
              best = g;
              bs = sl;
              bb = b;
              bestl = left;
            }
          }
        }
        if (bs < 0 || !(best > 0.0) || best < p.min_info_gain) continue;   // a leaf
        const int f = sub[(size_t)i * k + bs];
        Node L, R;
        L.stat = bestl;
        R.stat.resize(V);
        for (int v = 0; v < V; ++v) R.stat[v] = nd.stat[v] - bestl[v];
        if (regression) {
          L.count = L.stat[0];
          R.count = R.stat[0];
        } else {
          L.count = R.count = 0;
          for (int v = 0; v < V; ++v) L.count += L.stat[v], R.count += R.stat[v];
        }
        L.depth = R.depth = nd.depth + 1;
        L.heap = 2 * nd.heap;
        R.heap = 2 * nd.heap + 1;
        const int li = (int)tree.size();
        tree[ni].feature = f;
        tree[ni].threshold = thr[f][bb];
        tree[ni].gain = best;
        tree[ni].left = li;
        tree[ni].right = li + 1;
        tree.push_back(L);
        tree.push_back(R);
        route[i].feature = f;
        route[i].bin = bb;
        if (may_split(tree[li])) {
          route[i].left = (int)next.size();
          next.emplace_back(t, li);
        }
        if (may_split(tree[li + 1])) {
          route[i].right = (int)next.size();
          next.emplace_back(t, li + 1);
        }
      }
    }
    if (level_ms_out && depth <= p.max_depth) level_ms_out[depth] = ms_level;
    if (next.empty()) break;
    // `level` is ordered by tree, so `next` (created in that order) is too
    RouteInfo* route_dev;
    B2K_TRY(dalloc(ctx, b_route, (size_t)nl, s, &route_dev));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(route_dev, route.data(), (size_t)nl * sizeof(RouteInfo), cudaMemcpyHostToDevice, s));
    k_rf_route<<<grid_for(n * T, ctx->sm_count), RF_NT, 0, s>>>(bins, n, d, T, wt, route_dev, nid, pairs_dev + depth + 1);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
    level = next;
  }
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(pairs_h.data(), pairs_dev, pairs_h.size() * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  if (level_updates_out) {
    std::vector<int64_t> pu(pairs_h.begin(), pairs_h.begin() + p.max_depth + 1);
    int64_t* pd;
    DevBuf b_pu;
    B2K_TRY(dalloc(ctx, b_pu, pu.size(), s, &pd));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(pd, pu.data(), pu.size() * 8, cudaMemcpyHostToDevice, s));
    B2K_TRY(b2k_comm_allreduce_i64(ctx, pd, pu.size(), s));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(pu.data(), pd, pu.size() * 8, cudaMemcpyDeviceToHost, s));
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
    for (int l = 0; l <= p.max_depth; ++l) level_updates_out[l] = l < levels ? pu[l] * k : 0;
  }
  // ---- the flat forest ----
  auto F = std::make_shared<Forest>();
  F->V = n_values;
  F->off.push_back(0);
  for (int t = 0; t < T; ++t) {
    for (const Node& nd : trees[t]) {
      F->feature.push_back(nd.feature);
      F->threshold.push_back(nd.feature >= 0 ? nd.threshold : 0.f);
      F->children.push_back(nd.left);
      F->children.push_back(nd.right);
      F->gain.push_back(nd.feature >= 0 ? nd.gain : 0.0);
      F->count.push_back(nd.count);
      for (int v = 0; v < n_values; ++v) {
        double val = 0.0;
        if (nd.count > 0) val = regression ? ((double)nd.stat[1] * qv) / (double)nd.count
                                           : (double)nd.stat[v] / (double)nd.count;
        F->value.push_back(val);
      }
    }
    F->off.push_back((int64_t)F->feature.size());
  }
  ctx->rf_forest = F;
  *n_values_out = n_values;
  *n_nodes_out = F->off.back();
  ctx->stats.last_n_iter = levels;
  ctx->stats.recheck_rows = passes;
  ctx->stats.recheck_candidates = ar_bytes;
  if (ctx->time_kernels) {
    ctx->stats.last_finalize_ms = ms_edges;
    ctx->stats.last_reduce_ms = tm.ms(ev_bin0, ev_bin1);
    ctx->stats.last_fused_ms = ms_hist;
    ctx->stats.last_allreduce_ms = ms_allreduce;
    ctx->stats.last_loop_ms = since(t_entry);
  }
  return B2K_OK;
}

int b2k_rf_forest_impl(b2k_ctx* ctx, int64_t* off_out, int32_t* feature_out, float* threshold_out,
                       int32_t* children_out, double* gain_out, int64_t* count_out, double* value_out) {
  const Forest* F = static_cast<const Forest*>(ctx->rf_forest.get());
  if (!F) return b2k_fail(ctx, B2K_ERR_STATE, "b2k_rf_forest: no forest fitted on this context");
  std::copy(F->off.begin(), F->off.end(), off_out);
  std::copy(F->feature.begin(), F->feature.end(), feature_out);
  std::copy(F->threshold.begin(), F->threshold.end(), threshold_out);
  std::copy(F->children.begin(), F->children.end(), children_out);
  std::copy(F->gain.begin(), F->gain.end(), gain_out);
  std::copy(F->count.begin(), F->count.end(), count_out);
  std::copy(F->value.begin(), F->value.end(), value_out);
  return B2K_OK;
}

int b2k_rf_predict_impl(b2k_ctx* ctx, const float* X, int64_t n, int d, int T, const int64_t* off, const int32_t* feature,
                        const float* threshold, const int32_t* children, const double* value, int V, int cls,
                        double* raw, double* prob, double* pred, cudaStream_t s) {
  if (n == 0) return B2K_OK;
  int64_t n_nodes = 0;
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(&n_nodes, off + T, 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  std::vector<int32_t> f((size_t)n_nodes), ch((size_t)n_nodes * 2);
  std::vector<float> t((size_t)n_nodes);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(f.data(), feature, f.size() * 4, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(ch.data(), children, ch.size() * 4, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(t.data(), threshold, t.size() * 4, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  std::vector<PNode> pn((size_t)n_nodes);
  for (int64_t i = 0; i < n_nodes; ++i) {
    if (f[i] >= d) return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_rf_predict: a node splits on feature " +
                                                             std::to_string(f[i]) + " >= d = " + std::to_string(d));
    pn[i] = PNode{f[i], t[i], ch[2 * i], ch[2 * i + 1]};
  }
  DevBuf b_nodes;
  PNode* nodes = nullptr;
  B2K_TRY(dalloc(ctx, b_nodes, pn.size(), s, &nodes));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(nodes, pn.data(), pn.size() * sizeof(PNode), cudaMemcpyHostToDevice, s));
  const size_t smem = pn.size() * sizeof(PNode);
  const unsigned g = grid_for(n, ctx->sm_count);
  if (smem <= 48 * 1024) {
    k_rf_predict<true><<<g, RF_NT, smem, s>>>(X, n, d, T, off, nodes, n_nodes, value, V, cls, raw, prob, pred);
  } else {
    k_rf_predict<false><<<g, RF_NT, 0, s>>>(X, n, d, T, off, nodes, n_nodes, value, V, cls, raw, prob, pred);
  }
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));   // the staged nodes are freed at scope end
  return B2K_OK;
}
