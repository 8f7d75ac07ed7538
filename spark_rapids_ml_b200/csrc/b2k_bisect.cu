// Bisecting k-means (sm_90a): b2k_bkm_fit (collective) and b2k_bkm_predict (local).  Semantics: include/b2kmeans.h.
//
// Rows stay where they are in X; a permutation perm of the rank's rows keeps each active node's rows contiguous (its
// segment), in two int32 buffers used in turn.  Per level the host lists the dividing nodes (slots) and cuts their
// segments into units of at most S rows.  Then, with no host synchronisation until the level ends:
//   k_bkm_split     per unit: the fp64 parent and child centres in shared memory, the rows read through perm (float4
//                   when d % 4 == 0) and staged in shared memory; each row's side (the nearer live child, ties left)
//                   and, when partials are on, the unit's [2][n, S2, S1[d]] about the parent centre p, rows in order.
//   k_bkm_fold      per (slot, side, column): the slot's units in unit order -> the allreduce buffer.
//   allreduce       one f64 allreduce of [slots][2][d + 2].
//   k_bkm_centres   centre = p + S1 / n, cost = max(S2 - ||S1||^2 / n, 0); a child with n = 0 has dropped out.
// After maxIter iterations, one split pass without partials gives the final sides, and k_bkm_count / k_bkm_scan /
// k_bkm_scatter partition each dividing segment stably into [left | right] through per-unit counts and a scan in unit
// order.  The host then reads the child summaries once and decides the next level.
//   k_bkm_predict   tree descent, warp per row: the leaf and (optionally) the squared distance to its centre.
// No atomics anywhere: two calls on the same input, rank count and device give the same bits.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <map>
#include <string>
#include <vector>

#include "b2k_internal.cuh"

namespace {

constexpr double BKM_EPS = 2.220446049250313e-16;   // MLlib's EPSILON
constexpr int BKM_LEVEL_LIMIT = 63;                 // Spark's LEVEL_LIMIT: levels 1 .. 62
constexpr int BS_NT = 256;                          // threads of the split pass
constexpr int BS_STAGE = 8192;                      // floats of X a split CTA stages at once
constexpr int BS_MAX_R = 256;                       // rows a split CTA stages at once
constexpr int BKM_UNITS_PER_SM = 16;                // units per SM a level aims at (bounds the fold's length)
constexpr int BKM_MIN_SPAN = 256;                   // fewest rows of a unit (but the last of a segment)

struct BkmUnit {
  int32_t pos0;    // first position in perm
  int32_t nrows;
  int32_t slot;    // dividing node of the level
  int32_t pad;
};

struct BkmSplit {
  const float* X;
  int d, R;                // R: rows staged per chunk
  const int32_t* perm;     // [n] node-ordered rows
  const BkmUnit* units;
  int nunits;
  const double* parent;    // [slots][d]
  const double* child;     // [slots][2][d]
  const double* summ;      // [slots][2][2] (n, cost): a child with n = 0 takes no rows
  uint8_t* side;           // [n] by position: 0 left, 1 right
  double* part;            // [nunits][2][d + 2] or NULL (level-end reassignment)
};

__host__ __device__ inline size_t bkm_split_smem(int d, int R, bool partials) {
  const size_t dd = (size_t)(d + 1) / 2 * 2;   // keeps every region 16-byte aligned
  return (3 * dd + (partials ? 2 * dd : 0) + (size_t)(R + 1) / 2 * 2) * 8 + (size_t)R * d * 4 + (size_t)R * 4 + R;
}

template <bool VEC>
__global__ void __launch_bounds__(BS_NT) k_bkm_split(const BkmSplit a) {
  extern __shared__ __align__(16) double bs_sm[];
  const int d = a.d, R = a.R;
  const size_t dd = (size_t)(d + 1) / 2 * 2;
  const bool parts = a.part != nullptr;
  double* cp = bs_sm;
  double* c0 = cp + dd;
  double* c1 = c0 + dd;
  double* acc = c1 + dd;                            // [2][dd] when parts
  double* sd2 = acc + (parts ? 2 * dd : 0);         // [R] ||x - p||^2
  float* xs = reinterpret_cast<float*>(sd2 + (R + 1) / 2 * 2);   // [R][d]
  int32_t* rows = reinterpret_cast<int32_t*>(xs + (size_t)R * d);
  uint8_t* sside = reinterpret_cast<uint8_t*>(rows + R);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  int cur = -1;
  for (int u = blockIdx.x; u < a.nunits; u += gridDim.x) {
    const BkmUnit un = a.units[u];
    __syncthreads();   // the previous unit's partials are written
    if (un.slot != cur) {
      cur = un.slot;
      const double* p = a.parent + (size_t)cur * d;
      const double* c = a.child + (size_t)cur * 2 * d;
      for (int f = tid; f < d; f += BS_NT) {
        cp[f] = p[f];
        c0[f] = c[f];
        c1[f] = c[d + f];
      }
    }
    const bool live0 = a.summ[(size_t)cur * 4 + 0] > 0.0, live1 = a.summ[(size_t)cur * 4 + 2] > 0.0;
    if (parts)
      for (int f = tid; f < d; f += BS_NT) acc[f] = acc[dd + f] = 0.0;
    double n0 = 0.0, n1 = 0.0, q0 = 0.0, q1 = 0.0;   // thread BS_NT - 1: the unit's counts and S2 per side
    for (int r0 = 0; r0 < un.nrows; r0 += R) {
      const int m = min(R, un.nrows - r0);
      __syncthreads();
      for (int t = tid; t < m; t += BS_NT) rows[t] = a.perm[un.pos0 + r0 + t];
      __syncthreads();
      if (VEC) {
        const int d4 = d >> 2;
        const float4* X4 = reinterpret_cast<const float4*>(a.X);
        float4* xs4 = reinterpret_cast<float4*>(xs);
        for (int e = tid; e < m * d4; e += BS_NT) {
          const int r = e / d4, c = e - r * d4;
          xs4[e] = __ldg(X4 + (int64_t)rows[r] * d4 + c);
        }
      } else {
        for (int e = tid; e < m * d; e += BS_NT) {
          const int r = e / d, c = e - r * d;
          xs[e] = __ldg(a.X + (int64_t)rows[r] * d + c);
        }
      }
      __syncthreads();
      // sides: a warp per row, lanes over the features in order, then a fixed xor butterfly
      for (int r = warp; r < m; r += BS_NT / 32) {
        const float* x = xs + (size_t)r * d;
        double s0 = 0.0, s1 = 0.0, sp = 0.0;
        for (int f = lane; f < d; f += 32) {
          const double v = (double)x[f];
          const double e0 = v - c0[f], e1 = v - c1[f], ep = v - cp[f];
          s0 = fma(e0, e0, s0);
          s1 = fma(e1, e1, s1);
          sp = fma(ep, ep, sp);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          s0 += __shfl_xor_sync(0xffffffffu, s0, o);
          s1 += __shfl_xor_sync(0xffffffffu, s1, o);
          sp += __shfl_xor_sync(0xffffffffu, sp, o);
        }
        if (lane == 0) {
          const uint8_t sd = live0 && live1 ? (uint8_t)(s1 < s0) : (uint8_t)!live0;
          sside[r] = sd;
          sd2[r] = sp;
          a.side[un.pos0 + r0 + r] = sd;
        }
      }
      if (!parts) continue;
      __syncthreads();
      for (int f = tid; f < d; f += BS_NT) {
        double a0 = acc[f], a1 = acc[dd + f];
        const double pf = cp[f];
        for (int r = 0; r < m; ++r) {
          const double v = (double)xs[(size_t)r * d + f] - pf;
          if (sside[r]) a1 += v;
          else a0 += v;
        }
        acc[f] = a0;
        acc[dd + f] = a1;
      }
      if (tid == BS_NT - 1)
        for (int r = 0; r < m; ++r) {
          if (sside[r]) {
            n1 += 1.0;
            q1 += sd2[r];
          } else {
            n0 += 1.0;
            q0 += sd2[r];
          }
        }
    }
    if (!parts) continue;
    __syncthreads();
    double* o = a.part + (size_t)u * 2 * (d + 2);
    for (int f = tid; f < d; f += BS_NT) {
      o[2 + f] = acc[f];
      o[d + 2 + 2 + f] = acc[dd + f];
    }
    if (tid == BS_NT - 1) {
      o[0] = n0;
      o[1] = q0;
      o[d + 2] = n1;
      o[d + 3] = q1;
    }
  }
}

// buf[slot][side][c] = sum over the slot's units in unit order of part[u][side][c]; thread (x, y) of block (slot * 2 +
// side, column block) adds units ustart + y, + 8, ... in order, then lane y = 0 adds the 8 sums in y order
constexpr int BF_TX = 32, BF_TY = 8;
__global__ void __launch_bounds__(BF_TX * BF_TY)
k_bkm_fold(const double* __restrict__ part, const int32_t* __restrict__ ustart, int d, double* __restrict__ buf) {
  __shared__ double red[BF_TY][BF_TX];
  const int w = d + 2;
  const int c = blockIdx.y * BF_TX + threadIdx.x;
  const int slot = blockIdx.x >> 1, side = blockIdx.x & 1;
  const int u0 = ustart[slot], u1 = ustart[slot + 1];
  double t = 0.0;
  if (c < w)
    for (int u = u0 + threadIdx.y; u < u1; u += BF_TY) t += part[((size_t)u * 2 + side) * w + c];
  red[threadIdx.y][threadIdx.x] = t;
  __syncthreads();
  if (threadIdx.y == 0 && c < w) {
    double s = 0.0;
#pragma unroll
    for (int y = 0; y < BF_TY; ++y) s += red[y][threadIdx.x];
    buf[((size_t)slot * 2 + side) * w + c] = s;
  }
}

// block = slot, warp = side: centre, cost and n of the child from the allreduced sums
__global__ void __launch_bounds__(64)
k_bkm_centres(const double* __restrict__ buf, const double* __restrict__ parent, int d, double* __restrict__ child,
              double* __restrict__ summ) {
  const int slot = blockIdx.x, side = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const double* b = buf + ((size_t)slot * 2 + side) * (d + 2);
  const double n = b[0];
  double* sm = summ + ((size_t)slot * 2 + side) * 2;
  if (!(n > 0.0)) {   // no rows: the child drops out (its centre is left as it was and never read again)
    if (lane == 0) sm[0] = sm[1] = 0.0;
    return;
  }
  const double* p = parent + (size_t)slot * d;
  double* c = child + ((size_t)slot * 2 + side) * d;
  double q = 0.0;
  for (int f = lane; f < d; f += 32) {
    const double s1 = b[2 + f];
    q = fma(s1, s1, q);
    c[f] = p[f] + s1 / n;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  if (lane == 0) {
    sm[0] = n;
    sm[1] = fmax(b[1] - q / n, 0.0);
  }
}

// ---- stable partition of the dividing segments by the final sides ----
__global__ void __launch_bounds__(256)
k_bkm_count(const BkmUnit* __restrict__ units, int nunits, const uint8_t* __restrict__ side, int32_t* __restrict__ nl) {
  __shared__ int32_t red[8];
  for (int u = blockIdx.x; u < nunits; u += gridDim.x) {
    const BkmUnit un = units[u];
    int c = 0;
    for (int r = threadIdx.x; r < un.nrows; r += 256) c += side[un.pos0 + r] == 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
      int t = 0;
      for (int w = 0; w < 8; ++w) t += red[w];
      nl[u] = t;
    }
  }
}

// thread = slot: the first left and right position of each of its units, in unit order; nleft[slot] = its left rows
__global__ void k_bkm_scan(const BkmUnit* __restrict__ units, const int32_t* __restrict__ ustart, int nslots,
                           const int32_t* __restrict__ nl, int32_t* __restrict__ loff, int32_t* __restrict__ roff,
                           int32_t* __restrict__ nleft) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= nslots) return;
  const int u0 = ustart[slot], u1 = ustart[slot + 1];
  int L = 0;
  for (int u = u0; u < u1; ++u) L += nl[u];
  nleft[slot] = L;
  if (u0 == u1) return;
  int lo = units[u0].pos0, ro = units[u0].pos0 + L;
  for (int u = u0; u < u1; ++u) {
    loff[u] = lo;
    roff[u] = ro;
    lo += nl[u];
    ro += units[u].nrows - nl[u];
  }
}

__global__ void __launch_bounds__(256)
k_bkm_scatter(const BkmUnit* __restrict__ units, int nunits, const uint8_t* __restrict__ side,
              const int32_t* __restrict__ loff, const int32_t* __restrict__ roff, const int32_t* __restrict__ perm_in,
              int32_t* __restrict__ perm_out) {
  __shared__ int32_t wl[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int u = blockIdx.x; u < nunits; u += gridDim.x) {
    const BkmUnit un = units[u];
    int lo = loff[u], ro = roff[u];
    for (int r0 = 0; r0 < un.nrows; r0 += 256) {
      const int r = r0 + threadIdx.x;
      const bool in = r < un.nrows;
      const bool left = in && side[un.pos0 + r] == 0;
      const unsigned bl = __ballot_sync(0xffffffffu, left);
      __syncthreads();
      if (lane == 0) wl[warp] = __popc(bl);
      __syncthreads();
      int before = 0, total = 0;
      for (int w = 0; w < 8; ++w) {
        before += w < warp ? wl[w] : 0;
        total += wl[w];
      }
      const int lrank = before + __popc(bl & ((1u << lane) - 1u));
      if (in) {
        const int pos = un.pos0 + r;
        const int dst = left ? lo + lrank : ro + (r - r0) - lrank;
        perm_out[dst] = perm_in[pos];
      }
      lo += total;
      ro += min(256, un.nrows - r0) - total;
    }
  }
}

__global__ void k_bkm_iota(int32_t* __restrict__ perm, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    perm[i] = (int32_t)i;
}

// ---- predict: a warp per row descends the tree (node 0 the root); kid [nn][2] node positions or -1, leaf [nn] the
// leaf number or -1 ----
__device__ __forceinline__ double bkm_dist(const float* __restrict__ x, const double* __restrict__ c, int d, int lane) {
  double s = 0.0;
  for (int f = lane; f < d; f += 32) {
    const double e = (double)__ldg(x + f) - c[f];
    s = fma(e, e, s);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  return s;
}

__global__ void __launch_bounds__(256)
k_bkm_predict(const float* __restrict__ X, int64_t n, int d, const double* __restrict__ centers,
              const int2* __restrict__ kid, const int32_t* __restrict__ leaf, int32_t* __restrict__ labels,
              double* __restrict__ cost) {
  const int lane = threadIdx.x & 31;
  const int64_t wpb = blockDim.x >> 5;
  for (int64_t row = (int64_t)blockIdx.x * wpb + (threadIdx.x >> 5); row < n; row += (int64_t)gridDim.x * wpb) {
    const float* x = X + row * d;
    int p = 0;
    double d2 = -1.0;   // the squared distance to node p, when known
    while (leaf[p] < 0) {
      const int2 k2 = kid[p];
      if (k2.x >= 0 && k2.y >= 0) {
        const double dl = bkm_dist(x, centers + (size_t)k2.x * d, d, lane);
        const double dr = bkm_dist(x, centers + (size_t)k2.y * d, d, lane);
        p = dl <= dr ? k2.x : k2.y;
        d2 = dl <= dr ? dl : dr;
      } else {
        p = k2.x >= 0 ? k2.x : k2.y;
        d2 = -1.0;
      }
    }
    if (cost != nullptr && d2 < 0.0) d2 = bkm_dist(x, centers + (size_t)p * d, d, lane);
    if (lane == 0) {
      labels[row] = leaf[p];
      if (cost != nullptr) cost[row] = d2;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------------------------------------
int bkm_check_shape(b2k_ctx* ctx, const char* who, int d, int k) {
  if (d > B2K_BKM_MAX_D || k > B2K_BKM_MAX_K || (int64_t)k * d > ((int64_t)1 << 24))
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, std::string(who) + " supports d <= " + std::to_string(B2K_BKM_MAX_D) +
                                                  ", k <= " + std::to_string(B2K_BKM_MAX_K) + " and k d <= 2^24, got d = " +
                                                  std::to_string(d) + ", k = " + std::to_string(k));
  return B2K_OK;
}

int bkm_split_rows(int d) { return std::max(1, std::min(BS_MAX_R, BS_STAGE / d)); }

// The descent table of a node list: kid [nn] (left, right positions or -1), leaf [nn] (depth-first leaf number or -1);
// *n_leaves.  Fails unless the indices are distinct, >= 1, include the root and every non-root's parent.
int bkm_tree(b2k_ctx* ctx, const char* who, int nn, const int64_t* index, std::vector<int2>* kid,
             std::vector<int32_t>* leaf, int* n_leaves) {
  std::map<int64_t, int> pos;
  for (int i = 0; i < nn; ++i) {
    if (index[i] < 1 || !pos.emplace(index[i], i).second)
      return b2k_fail(ctx, B2K_ERR_INVALID, std::string(who) + ": node indices must be distinct and >= 1");
  }
  if (!pos.count(1)) return b2k_fail(ctx, B2K_ERR_INVALID, std::string(who) + ": the node list has no root (index 1)");
  kid->assign(nn, make_int2(-1, -1));
  leaf->assign(nn, -1);
  for (const auto& e : pos) {
    if (e.first == 1) continue;
    auto it = pos.find(e.first / 2);
    if (it == pos.end())
      return b2k_fail(ctx, B2K_ERR_INVALID, std::string(who) + ": node " + std::to_string(e.first) + " has no parent");
    if (e.first % 2 == 0) (*kid)[it->second].x = e.second;
    else (*kid)[it->second].y = e.second;
  }
  int nl = 0;
  std::vector<int> stack{pos[1]};
  while (!stack.empty()) {
    const int p = stack.back();
    stack.pop_back();
    const int2 c = (*kid)[p];
    if (c.x < 0 && c.y < 0) (*leaf)[p] = nl++;
    if (c.y >= 0) stack.push_back(c.y);
    if (c.x >= 0) stack.push_back(c.x);
  }
  *n_leaves = nl;
  return B2K_OK;
}

struct BkmTreeDev {
  double* centers;
  int2* kid;
  int32_t* leaf;
};

int bkm_tree_upload(b2k_ctx* ctx, const BkmTreeDev& t, int nn, int d, const double* centers,
                    const std::vector<int2>& kid, const std::vector<int32_t>& leaf, cudaStream_t s) {
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(t.centers, centers, (size_t)nn * d * 8, cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(t.kid, kid.data(), (size_t)nn * sizeof(int2), cudaMemcpyHostToDevice, s));
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(t.leaf, leaf.data(), (size_t)nn * 4, cudaMemcpyHostToDevice, s));
  return B2K_OK;
}

int bkm_predict_launch(b2k_ctx* ctx, const BkmTreeDev& t, const float* X, int64_t n, int d, int32_t* labels,
                       double* cost, cudaStream_t s) {
  if (n == 0) return B2K_OK;
  int sm = ctx->sm_count;
  if (ctx->grid_limit > 0 && ctx->grid_limit < sm) sm = ctx->grid_limit;
  const int grid = (int)std::min<int64_t>((n + 7) / 8, (int64_t)sm * 8);
  k_bkm_predict<<<grid, 256, 0, s>>>(X, n, d, t.centers, t.kid, t.leaf, labels, cost);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  ctx->stats.generic_launches++;
  return B2K_OK;
}

struct BkmNode {
  double n, cost;
  std::vector<double> c;
  int64_t seg0 = 0, seglen = 0;   // the rank's segment of the node's rows in perm (active nodes)
};

// Device times of one level, by the phase that ends at each mark (option time_kernels)
struct BkmMarks {
  bool on;
  std::vector<cudaEvent_t> ev;
  std::vector<int> cat;
  explicit BkmMarks(bool enable) : on(enable) {}
  ~BkmMarks() {
    for (auto e : ev) cudaEventDestroy(e);
  }
  void mark(int c, cudaStream_t s) {
    if (!on) return;
    cudaEvent_t e;
    cudaEventCreate(&e);
    cudaEventRecord(e, s);
    ev.push_back(e);
    cat.push_back(c);
  }
  // after a synchronise: adds each interval to acc[cat] and returns the span of the marks
  double drain(double* acc) {
    double total = 0.0;
    for (size_t i = 1; i < ev.size(); ++i) {
      float t = 0.f;
      cudaEventElapsedTime(&t, ev[i - 1], ev[i]);
      acc[cat[i]] += t;
      total += t;
    }
    for (auto e : ev) cudaEventDestroy(e);
    ev.clear();
    cat.clear();
    return total;
  }
};
enum { BKM_T_START = 0, BKM_T_SPLIT = 1, BKM_T_REDUCE = 2, BKM_T_ALLREDUCE = 3 };

}  // namespace

int b2k_bkm_predict_impl(b2k_ctx* ctx, const float* X, int64_t n, int d, int n_nodes, const int64_t* node_index,
                         const double* node_centers, int32_t* labels_out, double* cost_out, cudaStream_t s) {
  const char* who = "bisecting k-means predict";
  if (d > B2K_BKM_MAX_D || n_nodes > 2 * B2K_BKM_MAX_K - 1)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, std::string(who) + " supports d <= " + std::to_string(B2K_BKM_MAX_D) +
                                                  " and at most " + std::to_string(2 * B2K_BKM_MAX_K - 1) + " nodes");
  std::vector<int2> kid;
  std::vector<int32_t> leaf;
  int nl = 0;
  B2K_TRY(bkm_tree(ctx, who, n_nodes, node_index, &kid, &leaf, &nl));
  for (size_t i = 0; i < (size_t)n_nodes * d; ++i)
    if (!std::isfinite(node_centers[i])) return b2k_fail(ctx, B2K_ERR_INVALID, std::string(who) + ": a non-finite centre");
  BkmTreeDev t{};
  B2K_TRY(b2k_scratch_layout(ctx, "b2k_bkm_predict", [&](B2kLayout& L) -> int {
    t.centers = L.take<double>((size_t)n_nodes * d);
    t.kid = L.take<int2>((size_t)n_nodes);
    t.leaf = L.take<int32_t>((size_t)n_nodes);
    return B2K_OK;
  }));
  B2K_TRY(bkm_tree_upload(ctx, t, n_nodes, d, node_centers, kid, leaf, s));
  B2K_TRY(bkm_predict_launch(ctx, t, X, n, d, labels_out, cost_out, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));   // the host tables were copied from pageable memory
  return B2K_OK;
}

int b2k_bkm_fit_impl(b2k_ctx* ctx, const float* X, int64_t n, int d, int k, int max_iter, double min_divisible,
                     uint64_t seed, int* n_nodes_out, int64_t* node_index_out, double* node_centers_out,
                     int64_t* node_size_out, double* node_cost_out, double* training_cost_out,
                     int64_t* cluster_sizes_out, double* level_ms_out, cudaStream_t s) {
  using clk = std::chrono::steady_clock;
  const auto t_begin = clk::now();
  const char* who = "bisecting k-means";
  B2K_TRY(bkm_check_shape(ctx, who, d, k));
  {   // the row cap depends on a rank's own X: decided on an allreduced flag so that every rank fails together
    double fl = n > (int64_t)INT32_MAX ? 1.0 : 0.0;
    DevBuf b_fl;
    double* dfl = nullptr;
    B2K_TRY(dalloc(ctx, b_fl, 1, s, &dfl));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(dfl, &fl, 8, cudaMemcpyHostToDevice, s));
    B2K_TRY(b2k_comm_allreduce_f64(ctx, dfl, 1, s));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(&fl, dfl, 8, cudaMemcpyDeviceToHost, s));
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
    if (fl > 0.0) return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "bisecting k-means: more than 2^31 - 1 rows on one rank");
  }
  // the root: fp64 column means and centred squares; a NaN or an infinity anywhere reaches them on every rank
  int64_t n_total = 0;
  std::vector<double> mu, ssq;
  B2K_TRY(b2k_colstats_impl(ctx, who, X, n, d, &n_total, &mu, &ssq, s));
  double root_cost = 0.0;
  for (int f = 0; f < d; ++f) {
    if (!std::isfinite(mu[f]) || !std::isfinite(ssq[f]))
      return b2k_fail(ctx, B2K_ERR_INVALID, "bisecting k-means: the features hold a NaN or an infinity");
    root_cost += ssq[f];
  }
  const int64_t min_size = min_divisible >= 1.0 ? (int64_t)std::ceil(min_divisible)
                                                : (int64_t)std::ceil(min_divisible * (double)n_total);

  const int kd = k - 1;                                               // most nodes one level divides
  const int umax = BKM_UNITS_PER_SM * ctx->sm_count + kd;             // most units of one level
  const int R = bkm_split_rows(d);
  const size_t w = (size_t)d + 2;
  const int nn_max = 2 * k - 1;
  int32_t *perm[2], *ustart, *nl, *loff, *roff, *nleft, *labels;
  uint8_t* side;
  BkmUnit* units;
  double *parent, *child, *summ, *buf, *part, *spart;
  BkmTreeDev tree{};
  const int cspans = b2k_row_spans(ctx, n, 1).spans;   // of b2k_launch_label_counts
  B2K_TRY(b2k_scratch_layout(ctx, "b2k_bkm_fit", [&](B2kLayout& L) -> int {
    perm[0] = L.take<int32_t>((size_t)n);
    perm[1] = L.take<int32_t>((size_t)n);
    side = L.take<uint8_t>((size_t)n);
    units = L.take<BkmUnit>((size_t)umax);
    ustart = L.take<int32_t>((size_t)kd + 1);
    nl = L.take<int32_t>((size_t)umax);
    loff = L.take<int32_t>((size_t)umax);
    roff = L.take<int32_t>((size_t)umax);
    nleft = L.take<int32_t>((size_t)kd);
    parent = L.take<double>((size_t)kd * d);
    child = L.take<double>((size_t)kd * 2 * d);
    summ = L.take<double>((size_t)kd * 4);
    buf = L.take<double>((size_t)kd * 2 * w);
    part = L.take<double>((size_t)umax * 2 * w);
    tree.centers = L.take<double>((size_t)nn_max * d);
    tree.kid = L.take<int2>((size_t)nn_max);
    tree.leaf = L.take<int32_t>((size_t)nn_max);
    labels = L.take<int32_t>((size_t)n);
    spart = L.take<double>((size_t)cspans * k + k);
    return B2K_OK;
  }));
  const bool vec = d % 4 == 0 && (reinterpret_cast<uintptr_t>(X) & 15u) == 0;
  const size_t smem_p = bkm_split_smem(d, R, true), smem_s = bkm_split_smem(d, R, false);
  auto split_fn = vec ? k_bkm_split<true> : k_bkm_split<false>;
  B2K_CUDA_OK(ctx, cudaFuncSetAttribute(split_fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_p));
  int per_sm = 0;
  B2K_CUDA_OK(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, split_fn, BS_NT, smem_p));
  int gsm = ctx->sm_count;
  if (ctx->grid_limit > 0 && ctx->grid_limit < gsm) gsm = ctx->grid_limit;
  const int split_cap = std::max(1, ctx->grid_limit > 0 ? gsm : per_sm * gsm);
  {
    const unsigned g = (unsigned)std::min<int64_t>(std::max<int64_t>(1, (n + 255) / 256), (int64_t)ctx->sm_count * 8);
    k_bkm_iota<<<g, 256, 0, s>>>(perm[0], n);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
  }

  std::map<int64_t, BkmNode> nodes;
  nodes[1] = BkmNode{(double)n_total, root_cost, mu, 0, n};
  std::vector<int64_t> active{1};
  int64_t need = k - 1;
  int level = 1, cur = 0;
  BkmMarks marks(ctx->time_kernels != 0);
  double acc_ms[4] = {0.0, 0.0, 0.0, 0.0}, host_ms = 0.0;
  std::vector<BkmUnit> hu;
  std::vector<int32_t> hus, hnleft;
  std::vector<double> hpar, hchild, hsumm;
  while (!active.empty() && need > 0 && level < BKM_LEVEL_LIMIT) {
    const auto t_host = clk::now();
    std::vector<std::pair<int64_t, int64_t>> divisible;   // (-n, index)
    for (int64_t i : active) {
      const BkmNode& nd = nodes[i];
      if (nd.n >= (double)min_size && nd.cost > BKM_EPS * nd.n) divisible.emplace_back(-(int64_t)nd.n, i);
    }
    if (divisible.empty()) break;
    if ((int64_t)divisible.size() > need) {
      std::sort(divisible.begin(), divisible.end());
      divisible.resize((size_t)need);
    }
    std::vector<int64_t> div;
    for (const auto& e : divisible) div.push_back(e.second);
    std::sort(div.begin(), div.end());
    const int ns = (int)div.size();
    // units of at most S rows over the dividing segments, and the split starts c -/+ 1e-4 ||c|| u
    int64_t rows_div = 0;
    for (int64_t i : div) rows_div += nodes[i].seglen;
    const int64_t S = std::max<int64_t>(BKM_MIN_SPAN, (rows_div + (int64_t)BKM_UNITS_PER_SM * ctx->sm_count - 1) /
                                                          ((int64_t)BKM_UNITS_PER_SM * ctx->sm_count));
    hu.clear();
    hus.assign(ns + 1, 0);
    hpar.assign((size_t)ns * d, 0.0);
    hchild.assign((size_t)ns * 2 * d, 0.0);
    hsumm.assign((size_t)ns * 4, 1.0);   // both children live at the start
    for (int j = 0; j < ns; ++j) {
      const BkmNode& nd = nodes[div[j]];
      hus[j] = (int32_t)hu.size();
      for (int64_t r = 0; r < nd.seglen; r += S)
        hu.push_back(BkmUnit{(int32_t)(nd.seg0 + r), (int32_t)std::min<int64_t>(S, nd.seglen - r), j, 0});
      double nrm = 0.0;
      for (int f = 0; f < d; ++f) nrm += nd.c[f] * nd.c[f];
      const double l = 1e-4 * std::sqrt(nrm);
      const uint64_t z = b2k_splitmix64(seed ^ b2k_splitmix64((uint64_t)div[j]));
      for (int f = 0; f < d; ++f) {
        const double u = (double)(b2k_splitmix64(z + (uint64_t)f) >> 11) * 0x1.0p-53;
        hpar[(size_t)j * d + f] = nd.c[f];
        hchild[((size_t)j * 2) * d + f] = nd.c[f] - l * u;
        hchild[((size_t)j * 2 + 1) * d + f] = nd.c[f] + l * u;
      }
    }
    hus[ns] = (int32_t)hu.size();
    const int nu = (int)hu.size();
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(units, hu.data(), std::max<size_t>(1, hu.size()) * sizeof(BkmUnit),
                                     cudaMemcpyHostToDevice, s));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(ustart, hus.data(), hus.size() * 4, cudaMemcpyHostToDevice, s));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(parent, hpar.data(), hpar.size() * 8, cudaMemcpyHostToDevice, s));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(child, hchild.data(), hchild.size() * 8, cudaMemcpyHostToDevice, s));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(summ, hsumm.data(), hsumm.size() * 8, cudaMemcpyHostToDevice, s));
    host_ms += std::chrono::duration<double, std::milli>(clk::now() - t_host).count();

    BkmSplit a{};
    a.X = X;
    a.d = d;
    a.R = R;
    a.perm = perm[cur];
    a.units = units;
    a.nunits = nu;
    a.parent = parent;
    a.child = child;
    a.summ = summ;
    a.side = side;
    const int sgrid = std::max(1, std::min(nu, split_cap));
    const dim3 fgrid((unsigned)(2 * ns), (unsigned)((w + BF_TX - 1) / BF_TX));
    marks.mark(BKM_T_START, s);
    for (int it = 0; it < max_iter; ++it) {
      a.part = part;
      if (nu > 0) {
        split_fn<<<sgrid, BS_NT, smem_p, s>>>(a);
        B2K_CUDA_OK(ctx, cudaGetLastError());
      }
      marks.mark(BKM_T_SPLIT, s);
      k_bkm_fold<<<fgrid, dim3(BF_TX, BF_TY), 0, s>>>(part, ustart, d, buf);
      B2K_CUDA_OK(ctx, cudaGetLastError());
      marks.mark(BKM_T_REDUCE, s);
      B2K_TRY(b2k_comm_allreduce_f64(ctx, buf, (size_t)ns * 2 * w, s));
      marks.mark(BKM_T_ALLREDUCE, s);
      k_bkm_centres<<<ns, 64, 0, s>>>(buf, parent, d, child, summ);
      B2K_CUDA_OK(ctx, cudaGetLastError());
      marks.mark(BKM_T_REDUCE, s);
      ctx->stats.kernel_launches += 3;
      ctx->stats.generic_launches += 3;
    }
    // level end: the final sides, then the stable partition into [left | right] per dividing segment
    a.part = nullptr;
    if (nu > 0) {
      split_fn<<<sgrid, BS_NT, smem_s, s>>>(a);
      B2K_CUDA_OK(ctx, cudaGetLastError());
    }
    marks.mark(BKM_T_SPLIT, s);
    const int pgrid = std::max(1, std::min(nu, gsm * 8));
    if (nu > 0) {
      k_bkm_count<<<pgrid, 256, 0, s>>>(units, nu, side, nl);
      B2K_CUDA_OK(ctx, cudaGetLastError());
    }
    k_bkm_scan<<<(ns + 127) / 128, 128, 0, s>>>(units, ustart, ns, nl, loff, roff, nleft);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    if (nu > 0) {
      k_bkm_scatter<<<pgrid, 256, 0, s>>>(units, nu, side, loff, roff, perm[cur], perm[cur ^ 1]);
      B2K_CUDA_OK(ctx, cudaGetLastError());
    }
    marks.mark(BKM_T_REDUCE, s);
    ctx->stats.kernel_launches += 4;
    ctx->stats.generic_launches += 4;
    hnleft.resize(ns);
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(hsumm.data(), summ, hsumm.size() * 8, cudaMemcpyDeviceToHost, s));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(hchild.data(), child, hchild.size() * 8, cudaMemcpyDeviceToHost, s));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(hnleft.data(), nleft, (size_t)ns * 4, cudaMemcpyDeviceToHost, s));
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
    const double lvl_ms = marks.drain(acc_ms);
    if (level_ms_out != nullptr) level_ms_out[level - 1] = lvl_ms;
    const auto t_next = clk::now();
    cur ^= 1;
    std::vector<int64_t> next;
    for (int j = 0; j < ns; ++j) {
      const BkmNode& pn = nodes[div[j]];
      const int64_t seg[2][2] = {{pn.seg0, hnleft[j]}, {pn.seg0 + hnleft[j], pn.seglen - hnleft[j]}};
      for (int sd = 0; sd < 2; ++sd) {
        const double cn = hsumm[((size_t)j * 2 + sd) * 2];
        if (!(cn > 0.0)) continue;
        const int64_t ci = 2 * div[j] + sd;
        const double* cc = hchild.data() + ((size_t)j * 2 + sd) * d;
        nodes[ci] = BkmNode{cn, hsumm[((size_t)j * 2 + sd) * 2 + 1], std::vector<double>(cc, cc + d), seg[sd][0],
                            seg[sd][1]};
        next.push_back(ci);
      }
    }
    std::sort(next.begin(), next.end());
    active.swap(next);
    need -= ns;
    ++level;
    host_ms += std::chrono::duration<double, std::milli>(clk::now() - t_next).count();
  }

  // the tree in depth-first order, left first
  const auto t_tree = clk::now();
  std::vector<int64_t> order;
  {
    std::vector<int64_t> stack{1};
    while (!stack.empty()) {
      const int64_t i = stack.back();
      stack.pop_back();
      order.push_back(i);
      if (nodes.count(2 * i + 1)) stack.push_back(2 * i + 1);
      if (nodes.count(2 * i)) stack.push_back(2 * i);
    }
  }
  const int nn = (int)order.size();
  std::vector<double> hc((size_t)nn * d);
  double tcost = 0.0;
  for (int p = 0; p < nn; ++p) {
    const BkmNode& nd = nodes[order[p]];
    node_index_out[p] = order[p];
    node_size_out[p] = (int64_t)std::llround(nd.n);
    node_cost_out[p] = nd.cost;
    std::copy(nd.c.begin(), nd.c.end(), hc.begin() + (size_t)p * d);
    if (!nodes.count(2 * order[p]) && !nodes.count(2 * order[p] + 1)) tcost += nd.cost;
  }
  std::copy(hc.begin(), hc.end(), node_centers_out);
  *n_nodes_out = nn;
  *training_cost_out = tcost;
  std::vector<int2> kid;
  std::vector<int32_t> leaf;
  int nleaves = 0;
  B2K_TRY(bkm_tree(ctx, who, nn, order.data(), &kid, &leaf, &nleaves));
  host_ms += std::chrono::duration<double, std::milli>(clk::now() - t_tree).count();

  // cluster sizes: the predict pass over the training rows, counted per leaf and allreduced
  B2K_TRY(bkm_tree_upload(ctx, tree, nn, d, hc.data(), kid, leaf, s));
  B2K_TRY(bkm_predict_launch(ctx, tree, X, n, d, labels, nullptr, s));
  double* sizes = spart + (size_t)cspans * k;
  B2K_TRY(b2k_launch_label_counts(ctx, labels, n, nleaves, spart, sizes, s));
  B2K_TRY(b2k_comm_allreduce_f64(ctx, sizes, (size_t)nleaves, s));
  std::vector<double> hsz(nleaves);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(hsz.data(), sizes, (size_t)nleaves * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  for (int j = 0; j < nleaves; ++j) cluster_sizes_out[j] = (int64_t)std::llround(hsz[j]);
  for (int j = nleaves; j < k; ++j) cluster_sizes_out[j] = 0;
  ctx->stats.last_n_iter = level - 1;
  ctx->stats.last_path = B2K_PATH_GENERIC;
  if (ctx->time_kernels) {
    ctx->stats.last_fused_ms = acc_ms[BKM_T_SPLIT];
    ctx->stats.last_reduce_ms = acc_ms[BKM_T_REDUCE];
    ctx->stats.last_allreduce_ms = acc_ms[BKM_T_ALLREDUCE];
    ctx->stats.last_finalize_ms = host_ms;
    ctx->stats.last_loop_ms = std::chrono::duration<double, std::milli>(clk::now() - t_begin).count();
  }
  return B2K_OK;
}
