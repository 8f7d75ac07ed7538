// Multilayer perceptron classification (sm_90a): one loss-and-gradient evaluation per solver step, the fit loop
// (L-BFGS through b2k_logreg_minimize_impl, or MLlib's full-batch gradient descent) and prediction.
//
// An evaluation runs the rows in chunks of R rows (mlp_chunk_rows: the activations of a chunk take at most
// MLP_CHUNK_BYTES, so at the benchmark shapes a chunk stays in L2 between its passes).  Per chunk:
//   forward   layer l = 1 .. L-1: a_l = sigmoid(a_{l-1} W_l^T + b_l); layer L: z = a_{L-1} W_L^T + b_L
//   softmax   k_mlp_softmax: per row the loss -log softmax(z)_y (fp64, row maximum removed) and delta_L = p - onehot(y),
//             written over z
//   backward  layer l = L .. 1: the cross-Gram sum_rows [a_{l-1} | 1]^T delta_l into fp64 partials of fixed row units
//             (MLP_GRAM_ROWS rows), then (l > 1) delta_{l-1} = (delta_l W_l) (.) a_{l-1} (1 - a_{l-1}) written over a_{l-1}
//   fold      k_mlp_fold adds the chunk's unit partials, in unit order, into the evaluation's fp64 total
// then one f64 allreduce of [gradient (Spark's flat layout) | loss | rows].
//
// Two implementations of the products (MlpGemm, one descriptor for all four modes):
//   wgmma  k_mlp_wg<NB, GRAM>: a CTA is one warpgroup; a work item is a 64 x NB output tile (GRAM: of one 512-row
//          unit).
//          Per 32-wide K chunk the operands are loaded from global memory, split x = hi + lo (both round-to-nearest
//          tf32) and written K-major, 128-byte swizzled; D += lo.hi + hi.lo + hi.hi from a zero accumulator, added in
//          round-to-nearest fp32 into a second accumulator (3xTF32, the discipline of b2k_gram.cu).  Activations and
//          deltas are fp32 in the chunk buffers; the weights are uploaded as fp32 in the orientation each product reads
//          K-contiguous (forward: W_l as [numOut][numIn]; backward: Spark's layout, [numIn][numOut]).
//   simt   k_mlp_simt<TA, TB>: one thread per output, fp64 products and sums; activations and deltas fp64.
// Work items are fixed functions of the shape: a CTA's share of them changes with the grid, the bits of each output do
// not.  No atomics: an evaluation is bitwise reproducible for the same input, rank count and device.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "b2k_internal.cuh"

namespace {
#include "b2k_ptx.cuh"

constexpr int MLP_UNIT = 4096;                    // a chunk is a multiple of this many rows
// rows of one cross-Gram work unit (fp64 flush interval): small enough that a chunk's Gram has work for every SM
constexpr int MLP_GRAM_ROWS = 512;
static_assert(MLP_UNIT % MLP_GRAM_ROWS == 0, "a chunk holds whole Gram units");
constexpr size_t MLP_CHUNK_BYTES = (size_t)32 << 20;
constexpr int MT = 64;                            // output rows of a wgmma tile (one warpgroup)
constexpr int KC = 32;                            // K chunk: one 128-byte K-major operand row
constexpr int WG_THREADS = 128;
constexpr int SIMT_THREADS = 256;

enum MlpMode { MODE_FWD = 0, MODE_AFF = 1, MODE_BWD = 2, MODE_GRAM = 3 };

// out(m, n) = sum_k A(m, k) B(n, k), A(m, k) = A[m a_sm + k a_sk] (m == ones_m: 1 for every valid k), B likewise.
//   FWD  out[m ldo + n] = sigmoid(. + bias[n])       AFF  out[m ldo + n] = . + bias[n]
//   BWD  out[m ldo + n] = . * a (1 - a), a = out[m ldo + n] before the write (delta written over the activation)
//   GRAM k runs over the rows of unit u = [u MLP_GRAM_ROWS, min(K, (u + 1) MLP_GRAM_ROWS)); part[u part_ld + m N + n] = .
struct MlpGemm {
  int mode;
  const void* A;
  int64_t a_sm, a_sk;
  int64_t ones_m;
  const void* B;
  int64_t b_sn, b_sk;
  int64_t M, N, K;
  const double* bias;
  void* out;
  int64_t ldo;
  double* part;
  int64_t part_ld;
};

__device__ __forceinline__ double mlp_sigmoid(double v) { return 1.0 / (1.0 + exp(-v)); }

// ---------------------------------------------------------------------------------------------------------------------
// wgmma path
// ---------------------------------------------------------------------------------------------------------------------
// Operand tile [rows][32 k] of fp32 source values -> tf32 hi / lo planes, K-major SW128 (element (r, k) at r * 128 +
// ((k / 4 ^ r % 8) * 16) + (k % 4) * 4).  KCONT: the source is contiguous in k (a thread reads 4 consecutive k of one
// row, float4 when `vec`), else contiguous in m (a thread reads one m at 4 consecutive k; neighbours read neighbours).
template <bool KCONT>
__device__ __forceinline__ void mlp_stage(uint32_t dhi, uint32_t dlo, const float* __restrict__ src, int64_t sm,
                                          int64_t sk, int64_t m0, int64_t mv, int64_t ones_m, int rows, int64_t k0,
                                          int64_t kv, bool vec) {
  for (int idx = threadIdx.x; idx < rows * 8; idx += WG_THREADS) {
    const int r = KCONT ? idx >> 3 : idx % rows;
    const int k4 = KCONT ? idx & 7 : idx / rows;
    const int64_t m = m0 + r, kb = k0 + 4 * k4;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (m == ones_m) {
#pragma unroll
      for (int i = 0; i < 4; ++i) v[i] = kb + i < kv ? 1.f : 0.f;
    } else if (m < mv) {
      const float* p = src + m * sm + kb * sk;
      if (KCONT && vec && kb + 3 < kv) {
        const float4 q = __ldg(reinterpret_cast<const float4*>(p));
        v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i)
          if (kb + i < kv) v[i] = __ldg(p + i * sk);
      }
    }
    uint32_t hi[4], lo[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      hi[i] = rn_tf32_bits(v[i]);
      lo[i] = rn_tf32_bits(v[i] - __uint_as_float(hi[i]));
    }
    const uint32_t off = (uint32_t)(r * 128 + ((k4 ^ (r & 7)) << 4));
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(dhi + off), "r"(hi[0]), "r"(hi[1]), "r"(hi[2]),
                 "r"(hi[3]) : "memory");
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(dlo + off), "r"(lo[0]), "r"(lo[1]), "r"(lo[2]),
                 "r"(lo[3]) : "memory");
  }
}

template <int NB>
constexpr int wg_smem() { return 1024 + 2 * MT * 128 + 2 * NB * 128; }

// Row products (GRAM = false: both operands K-contiguous) or the cross-Gram (GRAM = true: both M/N-contiguous).
template <int NB, bool GRAM>
__global__ void __launch_bounds__(WG_THREADS) k_mlp_wg(const MlpGemm g) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* sm = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const uint32_t ahi = smem_u32(sm), alo = ahi + MT * 128, bhi = alo + MT * 128, blo = bhi + NB * 128;
  const float* A = static_cast<const float*>(g.A);
  const float* B = static_cast<const float*>(g.B);
  const int64_t tm = (g.M + MT - 1) / MT, tn = (g.N + NB - 1) / NB;
  const int64_t units = GRAM ? (g.K + MLP_GRAM_ROWS - 1) / MLP_GRAM_ROWS : 1;
  const int64_t items = units * tm * tn;
  const bool avec = !GRAM && (g.a_sm & 3) == 0 && (reinterpret_cast<uintptr_t>(A) & 15u) == 0;
  const bool bvec = !GRAM && (g.b_sn & 3) == 0 && (reinterpret_cast<uintptr_t>(B) & 15u) == 0;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float acc[NB / 2], acc2[NB / 2];
  for (int64_t it = blockIdx.x; it < items; it += gridDim.x) {
    const int64_t u = it / (tm * tn), rest = it % (tm * tn);
    const int64_t mt = rest / tn, nt = rest % tn;
    const int64_t k_lo = GRAM ? u * MLP_GRAM_ROWS : 0, k_hi = GRAM ? min(g.K, k_lo + MLP_GRAM_ROWS) : g.K;
#pragma unroll
    for (int i = 0; i < NB / 2; ++i) acc2[i] = 0.f;
    for (int64_t k0 = k_lo; k0 < k_hi; k0 += KC) {
      __syncthreads();   // the previous chunk's wgmma reads are complete in every warp
      mlp_stage<!GRAM>(ahi, alo, A, g.a_sm, g.a_sk, mt * MT, g.M, g.ones_m, MT, k0, k_hi, avec);
      mlp_stage<!GRAM>(bhi, blo, B, g.b_sn, g.b_sk, nt * NB, g.N, -1, NB, k0, k_hi, bvec);
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncthreads();
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < KC / 8; ++ks) {
        const uint64_t dah = make_kmajor_sw128_desc(ahi + ks * 32), dal = make_kmajor_sw128_desc(alo + ks * 32);
        const uint64_t dbh = make_kmajor_sw128_desc(bhi + ks * 32), dbl = make_kmajor_sw128_desc(blo + ks * 32);
        wgmma_tf32<NB>(acc, dal, dbh, ks != 0 ? 1u : 0u);   // small terms first
        wgmma_tf32<NB>(acc, dah, dbl, 1u);
        wgmma_tf32<NB>(acc, dah, dbh, 1u);
      }
      wgmma_commit();
      wgmma_wait0();
      reg_fence(acc);
#pragma unroll
      for (int i = 0; i < NB / 2; ++i) acc2[i] += acc[i];
    }
    // accumulator i of this lane: row 16 warp + lane / 4 + 8 ((i >> 1) & 1), column 8 (i >> 2) + 2 (lane & 3) + (i & 1)
#pragma unroll
    for (int i = 0; i < NB / 2; ++i) {
      const int64_t m = mt * MT + 16 * warp + (lane >> 2) + 8 * ((i >> 1) & 1);
      const int64_t n = nt * NB + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
      if (m >= g.M || n >= g.N) continue;
      if constexpr (GRAM) {
        g.part[u * g.part_ld + m * g.N + n] = (double)acc2[i];
      } else {
        float* o = static_cast<float*>(g.out) + m * g.ldo + n;
        if (g.mode == MODE_FWD) *o = (float)mlp_sigmoid((double)acc2[i] + g.bias[n]);
        else if (g.mode == MODE_AFF) *o = (float)((double)acc2[i] + g.bias[n]);
        else {
          const float a = *o;
          *o = acc2[i] * (a * (1.f - a));
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// generic fp64 path
// ---------------------------------------------------------------------------------------------------------------------
template <typename TA, typename TB>
__global__ void __launch_bounds__(SIMT_THREADS) k_mlp_simt(const MlpGemm g) {
  const TA* A = static_cast<const TA*>(g.A);
  const TB* B = static_cast<const TB*>(g.B);
  const bool gram = g.mode == MODE_GRAM;
  const int64_t units = gram ? (g.K + MLP_GRAM_ROWS - 1) / MLP_GRAM_ROWS : 1;
  const int64_t total = units * g.M * g.N;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    // n fastest: neighbouring threads read neighbouring weights (rows) or deltas (Gram)
    const int64_t u = t / (g.M * g.N), rest = t % (g.M * g.N);
    const int64_t m = rest / g.N, n = rest % g.N;
    const int64_t k_lo = gram ? u * MLP_GRAM_ROWS : 0, k_hi = gram ? min(g.K, k_lo + MLP_GRAM_ROWS) : g.K;
    double s = 0.0;
    for (int64_t k = k_lo; k < k_hi; ++k) {
      const double a = m == g.ones_m ? 1.0 : (double)A[m * g.a_sm + k * g.a_sk];
      s += a * (double)B[n * g.b_sn + k * g.b_sk];
    }
    if (gram) {
      g.part[u * g.part_ld + m * g.N + n] = s;
    } else {
      double* o = static_cast<double*>(g.out) + m * g.ldo + n;
      if (g.mode == MODE_FWD) *o = mlp_sigmoid(s + g.bias[n]);
      else if (g.mode == MODE_AFF) *o = s + g.bias[n];
      else *o = s * (*o * (1.0 - *o));
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// row passes shared by both paths
// ---------------------------------------------------------------------------------------------------------------------
// Per row: loss_rows[r] = log sum exp(z - max) - (z_y - max) and delta = softmax(z) - onehot(y) written over z.
template <typename T>
__global__ void __launch_bounds__(SIMT_THREADS) k_mlp_softmax(T* __restrict__ z, int64_t ld, const float* __restrict__ y,
                                                              int64_t rows, int C, double* __restrict__ loss_rows) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (int64_t)gridDim.x * blockDim.x) {
    T* zr = z + r * ld;
    double mx = -INFINITY;
    for (int c = 0; c < C; ++c) mx = fmax(mx, (double)zr[c]);
    double s = 0.0;
    for (int c = 0; c < C; ++c) s += exp((double)zr[c] - mx);
    const int yc = (int)y[r];
    loss_rows[r] = log(s) - ((double)zr[yc] - mx);
    for (int c = 0; c < C; ++c) zr[c] = (T)(exp((double)zr[c] - mx) / s - (c == yc ? 1.0 : 0.0));
  }
}

// part[u part_ld + loss_at] = sum of the loss of unit u's rows: 256 strided per-thread sums, then a fixed tree.
__global__ void __launch_bounds__(SIMT_THREADS) k_mlp_loss_units(const double* __restrict__ loss_rows, int64_t rows,
                                                                 double* __restrict__ part, int64_t part_ld,
                                                                 int64_t loss_at) {
  __shared__ double sh[SIMT_THREADS];
  const int64_t r0 = (int64_t)blockIdx.x * MLP_GRAM_ROWS, r1 = min(rows, r0 + MLP_GRAM_ROWS);
  double s = 0.0;
  for (int64_t r = r0 + threadIdx.x; r < r1; r += SIMT_THREADS) s += loss_rows[r];
  sh[threadIdx.x] = s;
  __syncthreads();
  for (int w = SIMT_THREADS / 2; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) sh[threadIdx.x] += sh[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) part[blockIdx.x * part_ld + loss_at] = sh[0];
}

// total[j] += sum over units u (in order) of part[u part_ld + j], j < m
__global__ void k_mlp_fold(const double* __restrict__ part, int64_t units, int64_t part_ld, int64_t m,
                           double* __restrict__ total) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= m) return;
  double s = total[j];
  for (int64_t u = 0; u < units; ++u) s += part[u * part_ld + j];
  total[j] = s;
}

// rawPrediction = z, probability = softmax(z), prediction = first argmax of z
template <typename T>
__global__ void __launch_bounds__(SIMT_THREADS) k_mlp_predict_rows(const T* __restrict__ z, int64_t ld, int64_t rows,
                                                                   int C, double* __restrict__ raw,
                                                                   double* __restrict__ prob,
                                                                   double* __restrict__ pred) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (int64_t)gridDim.x * blockDim.x) {
    const T* zr = z + r * ld;
    double mx = -INFINITY;
    int am = 0;
    for (int c = 0; c < C; ++c) {
      const double v = (double)zr[c];
      raw[r * C + c] = v;
      if (v > mx) {
        mx = v;
        am = c;
      }
    }
    double s = 0.0;
    for (int c = 0; c < C; ++c) s += exp((double)zr[c] - mx);
    for (int c = 0; c < C; ++c) prob[r * C + c] = exp((double)zr[c] - mx) / s;
    pred[r] = (double)am;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------------------------------------
int64_t ld4(int w) { return ((int64_t)w + 3) & ~(int64_t)3; }

struct Net {
  std::vector<int> w;   // layer widths w[0] = d .. w[L] = C
  int L = 0;
  std::vector<int64_t> off;   // flat offset of layer l's block (l = 1 .. L), off[L + 1] = P
  int64_t P = 0;
  explicit Net(const int* layers, int n_layers) : w(layers, layers + n_layers), L(n_layers - 1), off(n_layers + 1, 0) {
    for (int l = 1; l <= L; ++l) off[l + 1] = off[l] + (int64_t)w[l] * (w[l - 1] + 1);
    P = off[L + 1];
  }
};

int64_t chunk_rows(const Net& net, int64_t n, size_t es) {
  size_t per_row = 8;   // the row's loss
  for (int l = 1; l <= net.L; ++l) per_row += es * (size_t)ld4(net.w[l]);
  int64_t R = std::max<int64_t>(1, (int64_t)(MLP_CHUNK_BYTES / per_row / MLP_UNIT)) * MLP_UNIT;
  return std::min<int64_t>(R, std::max<int64_t>(1, (n + MLP_UNIT - 1) / MLP_UNIT) * MLP_UNIT);
}

int nb_for(int64_t n) { return n <= 16 ? 16 : n <= 32 ? 32 : n <= 64 ? 64 : 128; }

template <int NB, bool GRAM>
int launch_wg_nb(b2k_ctx* ctx, const MlpGemm& g, cudaStream_t s) {
  const int64_t units = GRAM ? (g.K + MLP_GRAM_ROWS - 1) / MLP_GRAM_ROWS : 1;
  const int64_t items = units * ((g.M + MT - 1) / MT) * ((g.N + NB - 1) / NB);
  constexpr int smem = wg_smem<NB>();
  B2K_CUDA_OK(ctx, cudaFuncSetAttribute(k_mlp_wg<NB, GRAM>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  int per_sm = 0;
  B2K_CUDA_OK(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_mlp_wg<NB, GRAM>, WG_THREADS, smem));
  int64_t cap = (int64_t)std::max(1, per_sm) * ctx->sm_count;
  if (ctx->grid_limit > 0 && ctx->grid_limit < cap) cap = ctx->grid_limit;
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(items, cap));
  k_mlp_wg<NB, GRAM><<<grid, WG_THREADS, smem, s>>>(g);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  ctx->stats.fused_tc_launches++;
  return B2K_OK;
}

int launch_wg(b2k_ctx* ctx, const MlpGemm& g, cudaStream_t s) {
  const int nb = nb_for(g.N);
  if (g.mode == MODE_GRAM) {
    if (nb == 16) return launch_wg_nb<16, true>(ctx, g, s);
    if (nb == 32) return launch_wg_nb<32, true>(ctx, g, s);
    if (nb == 64) return launch_wg_nb<64, true>(ctx, g, s);
    return launch_wg_nb<128, true>(ctx, g, s);
  }
  if (nb == 16) return launch_wg_nb<16, false>(ctx, g, s);
  if (nb == 32) return launch_wg_nb<32, false>(ctx, g, s);
  if (nb == 64) return launch_wg_nb<64, false>(ctx, g, s);
  return launch_wg_nb<128, false>(ctx, g, s);
}

template <typename TA, typename TB>
int launch_simt_t(b2k_ctx* ctx, const MlpGemm& g, cudaStream_t s) {
  const int64_t units = g.mode == MODE_GRAM ? (g.K + MLP_GRAM_ROWS - 1) / MLP_GRAM_ROWS : 1;
  const int64_t total = units * g.M * g.N;
  int64_t cap = 8 * (int64_t)ctx->sm_count;
  if (ctx->grid_limit > 0 && ctx->grid_limit < cap) cap = ctx->grid_limit;
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((total + SIMT_THREADS - 1) / SIMT_THREADS, cap));
  k_mlp_simt<TA, TB><<<grid, SIMT_THREADS, 0, s>>>(g);
  B2K_CUDA_OK(ctx, cudaGetLastError());
  ctx->stats.kernel_launches++;
  ctx->stats.generic_launches++;
  return B2K_OK;
}

// The device state of one call: the path, the weights in both orientations, the chunk buffers and the partials.
struct MlpRun {
  b2k_ctx* ctx;
  const Net& net;
  const float* X;
  int64_t n;
  bool wg;
  size_t es;       // bytes per activation: 4 (wgmma) or 8 (generic)
  int64_t R;       // rows per chunk
  void* Wf;        // forward orientation [numOut][numIn] per layer at off[l] (fp32 or fp64)
  void* Wb;        // Spark's layout (fp32 or fp64)
  double* bias;    // fp64, Spark's layout (the biases of layer l at off[l] + numIn numOut)
  std::vector<void*> act;   // act[l] [R][ld4(w[l])], l = 1 .. L
  double* loss_rows;
  double* part;    // [R / MLP_GRAM_ROWS][P + 1]
  double* total;   // [P + 2]: gradient sums, loss sum, rows

  // a_is_x: the A operand is X (fp32 on both paths); every other operand is a chunk buffer or weights
  int gemm(const MlpGemm& g, bool a_is_x, cudaStream_t s) {
    if (wg) return launch_wg(ctx, g, s);
    if (a_is_x) return launch_simt_t<float, double>(ctx, g, s);
    return launch_simt_t<double, double>(ctx, g, s);
  }
  const void* wf(int l) const { return static_cast<const char*>(Wf) + net.off[l] * es; }
  const void* wb(int l) const { return static_cast<const char*>(Wb) + net.off[l] * es; }
  const double* b(int l) const { return bias + net.off[l] + (int64_t)net.w[l] * net.w[l - 1]; }

  // forward of rows [r0, r0 + rows): activations of layers 1 .. L-1 and z of layer L
  int forward(int64_t r0, int64_t rows, cudaStream_t s) {
    for (int l = 1; l <= net.L; ++l) {
      const bool first = l == 1;
      MlpGemm g{};
      g.mode = l < net.L ? MODE_FWD : MODE_AFF;
      g.A = first ? static_cast<const void*>(X + r0 * net.w[0]) : act[l - 1];
      g.a_sm = first ? net.w[0] : ld4(net.w[l - 1]);
      g.a_sk = 1;
      g.ones_m = -1;
      g.B = wf(l);
      g.b_sn = net.w[l - 1];
      g.b_sk = 1;
      g.M = rows;
      g.N = net.w[l];
      g.K = net.w[l - 1];
      g.bias = b(l);
      g.out = act[l];
      g.ldo = ld4(net.w[l]);
      B2K_TRY(gemm(g, first, s));
    }
    return B2K_OK;
  }

  // one chunk of an evaluation: forward, softmax, then per layer the cross-Gram and the backward product
  int chunk(const float* y, int64_t r0, int64_t rows, cudaStream_t s) {
    B2K_TRY(forward(r0, rows, s));
    const int C = net.w[net.L];
    const int g1 = (int)std::max<int64_t>(1, std::min<int64_t>((rows + SIMT_THREADS - 1) / SIMT_THREADS, 8 * ctx->sm_count));
    if (wg) k_mlp_softmax<float><<<g1, SIMT_THREADS, 0, s>>>(static_cast<float*>(act[net.L]), ld4(C), y + r0, rows, C, loss_rows);
    else k_mlp_softmax<double><<<g1, SIMT_THREADS, 0, s>>>(static_cast<double*>(act[net.L]), ld4(C), y + r0, rows, C, loss_rows);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    const int64_t units = (rows + MLP_GRAM_ROWS - 1) / MLP_GRAM_ROWS;
    k_mlp_loss_units<<<(int)units, SIMT_THREADS, 0, s>>>(loss_rows, rows, part, net.P + 1, net.P);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches += 2;
    for (int l = net.L; l >= 1; --l) {
      const bool first = l == 1;
      MlpGemm g{};
      g.mode = MODE_GRAM;   // G[i][o] = sum_rows [a_{l-1} | 1]_i delta_l,o at off[l] + i numOut + o
      g.A = first ? static_cast<const void*>(X + r0 * net.w[0]) : act[l - 1];
      g.a_sm = 1;
      g.a_sk = first ? net.w[0] : ld4(net.w[l - 1]);
      g.ones_m = net.w[l - 1];
      g.B = act[l];
      g.b_sn = 1;
      g.b_sk = ld4(net.w[l]);
      g.M = net.w[l - 1] + 1;
      g.N = net.w[l];
      g.K = rows;
      g.part = part + net.off[l];
      g.part_ld = net.P + 1;
      B2K_TRY(gemm(g, first, s));
      if (first) break;
      MlpGemm h{};
      h.mode = MODE_BWD;   // delta_{l-1} = (delta_l W_l) (.) a (1 - a), over a_{l-1}
      h.A = act[l];
      h.a_sm = ld4(net.w[l]);
      h.a_sk = 1;
      h.ones_m = -1;
      h.B = wb(l);
      h.b_sn = net.w[l];
      h.b_sk = 1;
      h.M = rows;
      h.N = net.w[l - 1];
      h.K = net.w[l];
      h.out = act[l - 1];
      h.ldo = ld4(net.w[l - 1]);
      B2K_TRY(gemm(h, false, s));
    }
    k_mlp_fold<<<(int)((net.P + 1 + 255) / 256), 256, 0, s>>>(part, units, net.P + 1, net.P + 1, total);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
    return B2K_OK;
  }
};

// The wgmma envelope: rows of X 16-byte aligned (d % 4 == 0 and X aligned).  Every other legal shape runs generic.
bool wg_supported(int d, const float* X) { return d % 4 == 0 && (reinterpret_cast<uintptr_t>(X) & 15u) == 0; }

// Chooses the path, lays out the scratch and uploads the weights.  A collective call (evaluation, fit) decides the path
// on an allreduced flag, since the envelope depends on each rank's own X pointer: either every rank runs wgmma or none
// does, and kernel_path=2 outside the envelope on any rank fails on every rank.  Prediction is local.
int mlp_setup(b2k_ctx* ctx, const Net& net, const float* X, int64_t n, bool collective, MlpRun* run, cudaStream_t s) {
  bool can = wg_supported(net.w[0], X);
  if (collective && ctx->nranks > 1) {
    double fl = can ? 0.0 : 1.0;
    DevBuf b_fl;
    double* dfl = nullptr;
    B2K_TRY(dalloc(ctx, b_fl, 1, s, &dfl));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(dfl, &fl, sizeof fl, cudaMemcpyHostToDevice, s));
    B2K_TRY(b2k_comm_allreduce_f64(ctx, dfl, 1, s));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(&fl, dfl, sizeof fl, cudaMemcpyDeviceToHost, s));
    B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
    can = fl == 0.0;
  }
  if (ctx->kernel_path == B2K_PATH_FUSED && !can)
    return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "kernel_path=2 requested but the wgmma multilayer perceptron pass needs "
                                              "d % 4 == 0 and 16-byte aligned rows on every rank, got d = " +
                                              std::to_string(net.w[0]));
  run->wg = can && ctx->kernel_path != B2K_PATH_GENERIC;
  run->es = run->wg ? 4 : 8;
  run->R = chunk_rows(net, n, run->es);
  run->X = X;
  run->n = n;
  const int64_t units = run->R / MLP_GRAM_ROWS;
  run->act.assign(net.L + 1, nullptr);
  return b2k_scratch_layout(ctx, "multilayer perceptron", [&](B2kLayout& Lo) -> int {
    run->Wf = Lo.take<char>((size_t)net.P * run->es);
    run->Wb = Lo.take<char>((size_t)net.P * run->es);
    run->bias = Lo.take<double>((size_t)net.P);
    for (int l = 1; l <= net.L; ++l) run->act[l] = Lo.take<char>((size_t)run->R * ld4(net.w[l]) * run->es);
    run->loss_rows = collective ? Lo.take<double>((size_t)run->R) : nullptr;
    run->part = collective ? Lo.take<double>((size_t)units * (net.P + 1)) : nullptr;
    run->total = collective ? Lo.take<double>((size_t)net.P + 2) : nullptr;
    return B2K_OK;
  });
}

int upload_weights(b2k_ctx* ctx, MlpRun& run, const double* w, cudaStream_t s) {
  const Net& net = run.net;
  std::vector<double> wf((size_t)net.P);
  for (int l = 1; l <= net.L; ++l) {   // forward orientation [o][i] from Spark's (o, i) at i numOut + o
    const int no = net.w[l], ni = net.w[l - 1];
    const double* src = w + net.off[l];
    double* dst = wf.data() + net.off[l];
    for (int o = 0; o < no; ++o)
      for (int i = 0; i < ni; ++i) dst[(size_t)o * ni + i] = src[(size_t)i * no + o];
    for (int o = 0; o < no; ++o) dst[(size_t)no * ni + o] = src[(size_t)no * ni + o];
  }
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(run.bias, w, (size_t)net.P * 8, cudaMemcpyHostToDevice, s));
  if (run.es == 8) {
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(run.Wf, wf.data(), (size_t)net.P * 8, cudaMemcpyHostToDevice, s));
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(run.Wb, w, (size_t)net.P * 8, cudaMemcpyHostToDevice, s));
    return B2K_OK;
  }
  // pageable sources: each copy has read its buffer when it returns
  std::vector<float> f32((size_t)net.P);
  for (int64_t j = 0; j < net.P; ++j) f32[j] = (float)wf[j];
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(run.Wf, f32.data(), (size_t)net.P * 4, cudaMemcpyHostToDevice, s));
  for (int64_t j = 0; j < net.P; ++j) f32[j] = (float)w[j];
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(run.Wb, f32.data(), (size_t)net.P * 4, cudaMemcpyHostToDevice, s));
  return B2K_OK;
}

// One evaluation at w (host f64, Spark's layout): *F = (1/n) sum loss, grad [P] = its gradient, *n_total.
int mlp_eval_device(MlpRun& run, const float* y, const double* w, double* F, double* grad, int64_t* n_total,
                    double* dev_ms, cudaStream_t s) {
  b2k_ctx* ctx = run.ctx;
  const Net& net = run.net;
  for (int64_t j = 0; j < net.P; ++j)
    if (!std::isfinite(w[j])) return b2k_fail(ctx, B2K_ERR_INVALID, "multilayer perceptron: a weight is not finite");
  B2K_TRY(upload_weights(ctx, run, w, s));
  B2K_CUDA_OK(ctx, cudaMemsetAsync(run.total, 0, (size_t)(net.P + 2) * 8, s));
  B2kTimer tm(ctx->time_kernels != 0);
  tm.mark(0, s);
  for (int64_t r0 = 0; r0 < run.n; r0 += run.R) B2K_TRY(run.chunk(y, r0, std::min(run.R, run.n - r0), s));
  tm.mark(1, s);
  const double nl = (double)run.n;
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(run.total + net.P + 1, &nl, 8, cudaMemcpyHostToDevice, s));
  B2K_TRY(b2k_comm_allreduce_f64(ctx, run.total, (size_t)net.P + 2, s));
  std::vector<double> h((size_t)net.P + 2);
  B2K_CUDA_OK(ctx, cudaMemcpyAsync(h.data(), run.total, h.size() * 8, cudaMemcpyDeviceToHost, s));
  B2K_CUDA_OK(ctx, cudaStreamSynchronize(s));
  ctx->stats.nccl_allreduces += ctx->nranks > 1 ? 1 : 0;
  ctx->stats.last_path = run.wg ? B2K_PATH_FUSED : B2K_PATH_GENERIC;
  if (tm.on) *dev_ms += tm.ms(0, 1);
  const double nt = h[net.P + 1];
  bool finite = std::isfinite(h[net.P]);
  for (int64_t j = 0; j < net.P && finite; ++j) finite = std::isfinite(h[j]);
  if (!finite) return b2k_fail(ctx, B2K_ERR_INVALID, "multilayer perceptron: the features hold a NaN or an infinity");
  *F = h[net.P] / nt;
  for (int64_t j = 0; j < net.P; ++j) grad[j] = h[j] / nt;
  if (n_total) *n_total = (int64_t)nt;
  return B2K_OK;
}

std::string fnum(double v) {
  char b[64];
  std::snprintf(b, sizeof b, "%.17g", v);
  return b;
}

// The labels: b2k_logreg_labels' rules (integers in [0, 1024), decided on gathered values), then every class < C.
int check_labels(b2k_ctx* ctx, const float* y, int64_t n, int C, cudaStream_t s) {
  std::vector<double> cls(B2K_LOGREG_MAX_CLASSES);
  std::vector<int64_t> cnt(B2K_LOGREG_MAX_CLASSES);
  int k = 0;
  B2K_TRY(b2k_logreg_labels_impl(ctx, y, n, cls.data(), cnt.data(), &k, nullptr, s));
  if (k > 0 && cls[k - 1] >= (double)C)
    return b2k_fail(ctx, B2K_ERR_INVALID, "multilayer perceptron: labels must be in [0, " + std::to_string(C) +
                                              ") for the " + std::to_string(C) + " outputs of the last layer, got " +
                                              fnum(cls[k - 1]));
  return B2K_OK;
}

struct FitObjective {
  MlpRun* run;
  const float* y;
  double* dev_ms;
  cudaStream_t s;
};

int fit_objective(void* user, int n, const double* x, double* f, double* grad) {
  FitObjective* o = static_cast<FitObjective*>(user);
  (void)n;
  return mlp_eval_device(*o->run, o->y, x, f, grad, nullptr, o->dev_ms, o->s);
}

}  // namespace

int b2k_mlp_check_layers(b2k_ctx* ctx, const int* layers, int n_layers, int d) {
  if (!layers || n_layers < 2)
    return b2k_fail(ctx, B2K_ERR_INVALID, "multilayer perceptron: layers must have at least 2 entries");
  for (int i = 0; i < n_layers; ++i)
    if (layers[i] < 1)
      return b2k_fail(ctx, B2K_ERR_INVALID, "multilayer perceptron: every layer width must be >= 1, got " +
                                                std::to_string(layers[i]) + " at " + std::to_string(i));
  for (int i = 0; i < n_layers; ++i)
    if (layers[i] > B2K_MLP_MAX_WIDTH)
      return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "multilayer perceptron supports layer widths <= " +
                                                    std::to_string(B2K_MLP_MAX_WIDTH) + ", got " +
                                                    std::to_string(layers[i]));
  if (layers[0] != d)
    return b2k_fail(ctx, B2K_ERR_INVALID, "multilayer perceptron: layers[0] = " + std::to_string(layers[0]) +
                                              " must equal the feature count " + std::to_string(d));
  return B2K_OK;
}

int64_t b2k_mlp_n_weights(const int* layers, int n_layers) { return Net(layers, n_layers).P; }

int b2k_mlp_eval_impl(b2k_ctx* ctx, const float* X, const float* y, int64_t n, const int* layers, int n_layers,
                      const double* weights, double* f_out, double* grad_out, int64_t* n_total_out, cudaStream_t s) {
  const Net net(layers, n_layers);
  B2K_TRY(check_labels(ctx, y, n, net.w[net.L], s));
  MlpRun run{ctx, net};
  B2K_TRY(mlp_setup(ctx, net, X, n, true, &run, s));
  double ms = 0.0;
  B2K_TRY(mlp_eval_device(run, y, weights, f_out, grad_out, n_total_out, &ms, s));
  if (ctx->time_kernels) ctx->stats.last_fused_ms = ms;
  return B2K_OK;
}

int b2k_mlp_fit_impl(b2k_ctx* ctx, const float* X, const float* y, int64_t n, const int* layers, int n_layers,
                     int solver, int max_iter, double tol, double step_size, uint64_t seed,
                     const double* initial_weights, double* weights_out, double* history_out, int* n_iter_out,
                     cudaStream_t s) {
  using clk = std::chrono::steady_clock;
  const auto t_begin = clk::now();
  const Net net(layers, n_layers);
  B2K_TRY(check_labels(ctx, y, n, net.w[net.L], s));
  std::vector<double> w((size_t)net.P);
  if (initial_weights) {
    std::copy(initial_weights, initial_weights + net.P, w.begin());
  } else {   // (u 4.8 - 2.4) / sqrt(numIn), u = splitmix64(seed ^ splitmix64(j)) / 2^64 at 53 bits
    for (int l = 1; l <= net.L; ++l) {
      const double sc = 1.0 / std::sqrt((double)net.w[l - 1]);
      for (int64_t j = net.off[l]; j < net.off[l + 1]; ++j) {
        const double u = (double)(b2k_splitmix64(seed ^ b2k_splitmix64((uint64_t)j)) >> 11) * 0x1.0p-53;
        w[j] = (u * 4.8 - 2.4) * sc;
      }
    }
  }
  MlpRun run{ctx, net};
  B2K_TRY(mlp_setup(ctx, net, X, n, true, &run, s));
  double ms = 0.0;
  std::vector<double> hist;
  if (solver == B2K_MLP_LBFGS) {
    FitObjective obj{&run, y, &ms, s};
    if (net.P > INT32_MAX) return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "multilayer perceptron: too many weights");
    ctx->err.clear();
    const int rc = b2k_logreg_minimize_impl(fit_objective, &obj, (int)net.P, w.data(), nullptr, max_iter, tol, nullptr,
                                            nullptr, nullptr, &hist);
    if (rc != B2K_OK) {
      // an evaluation's error is in ctx; the minimiser's own goes to the context-free slot
      if (ctx->err.empty()) ctx->err = b2k_last_error(nullptr);
      return rc;
    }
  } else {   // MLlib's GradientDescent with SimpleUpdater, full batch
    std::vector<double> g((size_t)net.P), wn((size_t)net.P);
    for (int t = 1; t <= max_iter; ++t) {
      double F = 0.0;
      B2K_TRY(mlp_eval_device(run, y, w.data(), &F, g.data(), nullptr, &ms, s));
      hist.push_back(F);
      const double step = step_size / std::sqrt((double)t);
      double dd = 0.0, nn = 0.0;
      for (int64_t j = 0; j < net.P; ++j) {
        wn[j] = w[j] - step * g[j];
        dd += (wn[j] - w[j]) * (wn[j] - w[j]);
        nn += wn[j] * wn[j];
      }
      w.swap(wn);
      if (std::sqrt(dd) < tol * std::max(std::sqrt(nn), 1.0)) break;
    }
  }
  std::copy(w.begin(), w.end(), weights_out);
  const int nh = (int)std::min<size_t>(hist.size(), (size_t)max_iter + 1);
  std::copy(hist.begin(), hist.begin() + nh, history_out);
  *n_iter_out = nh;
  ctx->stats.last_n_iter = nh;
  if (ctx->time_kernels) {
    ctx->stats.last_fused_ms = ms;
    ctx->stats.last_loop_ms = std::chrono::duration<double, std::milli>(clk::now() - t_begin).count();
  }
  return B2K_OK;
}

int b2k_mlp_predict_impl(b2k_ctx* ctx, const float* X, int64_t n, const int* layers, int n_layers,
                         const double* weights, double* raw_out, double* prob_out, double* pred_out, cudaStream_t s) {
  const Net net(layers, n_layers);
  for (int64_t j = 0; j < net.P; ++j)
    if (!std::isfinite(weights[j])) return b2k_fail(ctx, B2K_ERR_INVALID, "multilayer perceptron: a weight is not finite");
  if (n == 0) return B2K_OK;
  MlpRun run{ctx, net};
  B2K_TRY(mlp_setup(ctx, net, X, n, false, &run, s));
  B2K_TRY(upload_weights(ctx, run, weights, s));
  const int C = net.w[net.L];
  for (int64_t r0 = 0; r0 < n; r0 += run.R) {
    const int64_t rows = std::min(run.R, n - r0);
    B2K_TRY(run.forward(r0, rows, s));
    const int g1 = (int)std::max<int64_t>(1, std::min<int64_t>((rows + SIMT_THREADS - 1) / SIMT_THREADS, 8 * ctx->sm_count));
    if (run.wg)
      k_mlp_predict_rows<float><<<g1, SIMT_THREADS, 0, s>>>(static_cast<const float*>(run.act[net.L]), ld4(C), rows, C,
                                                            raw_out + r0 * C, prob_out + r0 * C, pred_out + r0);
    else
      k_mlp_predict_rows<double><<<g1, SIMT_THREADS, 0, s>>>(static_cast<const double*>(run.act[net.L]), ld4(C), rows,
                                                             C, raw_out + r0 * C, prob_out + r0 * C, pred_out + r0);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
  }
  ctx->stats.last_path = run.wg ? B2K_PATH_FUSED : B2K_PATH_GENERIC;
  return B2K_OK;
}
