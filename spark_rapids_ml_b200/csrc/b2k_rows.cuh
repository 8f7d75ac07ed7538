// Per-row prediction code shared by the predict kernels (k_linreg_predict, k_logreg_rows, k_csr_rows, k_rf_predict) and
// the multi-model evaluation pass (b2k_eval.cu).  One definition keeps a model's per-row prediction bit-identical in both:
// the same lane split, the same fp64 FMA order and xor butterfly, the same tree walk and __dadd_rn order.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

// Lanes per row of the linear kinds: the least power of two covering ceil(d / 4), at most 32.
__host__ __device__ __forceinline__ int b2k_row_lanes(int d) {
  int L = 1;
  while (L < 32 && 4 * L < d) L <<= 1;
  return L;
}

// Loaders of the features k .. k + 3 of one row, 0 past d.  VEC reads one float4 (d % 4 == 0, 16-byte aligned row).
template <bool VEC>
struct B2kRowLdcs {   // global, streaming
  const float* x;
  int d;
  __device__ __forceinline__ float4 operator()(int k) const {
    if (VEC) return __ldcs(reinterpret_cast<const float4*>(x + k));
    float4 v;
    v.x = __ldcs(x + k);
    v.y = k + 1 < d ? __ldcs(x + k + 1) : 0.f;
    v.z = k + 2 < d ? __ldcs(x + k + 2) : 0.f;
    v.w = k + 3 < d ? __ldcs(x + k + 3) : 0.f;
    return v;
  }
};
template <bool VEC>
struct B2kRowLdg {   // global, read-only path
  const float* x;
  int d;
  __device__ __forceinline__ float4 operator()(int k) const {
    if (VEC) return __ldg(reinterpret_cast<const float4*>(x + k));
    float4 v;
    v.x = __ldg(x + k);
    v.y = k + 1 < d ? __ldg(x + k + 1) : 0.f;
    v.z = k + 2 < d ? __ldg(x + k + 2) : 0.f;
    v.w = k + 3 < d ? __ldg(x + k + 3) : 0.f;
    return v;
  }
};
struct B2kRowSmem {   // a staged row in shared memory, zero-padded to a multiple of 4, 16-byte aligned
  const float* x;
  __device__ __forceinline__ float4 operator()(int k) const { return *reinterpret_cast<const float4*>(x + k); }
};

// Identity model: lane `sub` of the row's L lanes accumulates features 4 (sub + L i) .. + 3 in order in fp64 against w
// (fp64, zero-padded to a multiple of 4, 16-byte aligned).
template <class LD>
__device__ __forceinline__ double b2k_linear_lane(const LD& ld, int d, const double* w, int sub, int L) {
  double acc = 0.0;
#pragma unroll 4
  for (int k = 4 * sub; k < d; k += 4 * L) {
    const float4 v = ld(k);
    const double2 w01 = *reinterpret_cast<const double2*>(w + k);
    const double2 w23 = *reinterpret_cast<const double2*>(w + k + 2);
    acc = fma((double)v.x, w01.x, acc);
    acc = fma((double)v.y, w01.y, acc);
    acc = fma((double)v.z, w23.x, acc);
    acc = fma((double)v.w, w23.y, acc);
  }
  return acc;
}

// The row's L lanes add their partials by a fixed xor butterfly (every lane of the warp takes part).
__device__ __forceinline__ double b2k_lanes_sum(double acc, int L) {
  for (int o = L >> 1; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  return acc;
}

// Logistic kinds: the partial margins of classes k0 .. k0 + RC - 1 (< kp) of W [kp][ld_w], features as above; a
// weight past d is never read.
template <int RC, class LD>
__device__ __forceinline__ void b2k_logistic_lanes(const LD& ld, int d, int kp, int k0, const double* __restrict__ W,
                                                   int ld_w, int sub, int L, double (&acc)[RC]) {
  for (int j = 4 * sub; j < d; j += 4 * L) {
    const float4 v = ld(j);
#pragma unroll
    for (int q = 0; q < RC; ++q) {
      const int k = k0 + q;
      if (k < kp) {
        const double* w = W + (size_t)k * ld_w + j;
        acc[q] = fma((double)v.x, __ldg(w), acc[q]);
        if (j + 1 < d) acc[q] = fma((double)v.y, __ldg(w + 1), acc[q]);
        if (j + 2 < d) acc[q] = fma((double)v.z, __ldg(w + 2), acc[q]);
        if (j + 3 < d) acc[q] = fma((double)v.w, __ldg(w + 3), acc[q]);
      }
    }
  }
}

// Sparse rows (CSR): lane `sub` of the row's L lanes accumulates entries p0 + sub + L i in order in fp64 for the classes
// k0 .. k0 + RC - 1 (< kp), the weight of class k and feature j at W[k ldk + j ldj] (gathered through L2).
template <int RC>
__device__ __forceinline__ void b2k_csr_lanes(const int32_t* __restrict__ idx, const float* __restrict__ val, int64_t p0,
                                              int64_t p1, int kp, int k0, const double* __restrict__ W, int64_t ldk,
                                              int64_t ldj, int sub, int L, double (&acc)[RC]) {
  for (int64_t e = p0 + sub; e < p1; e += L) {
    const int64_t j = __ldg(idx + e);
    const double v = (double)__ldg(val + e);
#pragma unroll
    for (int q = 0; q < RC; ++q) {
      const int k = k0 + q;
      if (k < kp) acc[q] = fma(v, __ldg(W + k * ldk + j * ldj), acc[q]);
    }
  }
}

// Training: m [kp] margins in, r [kp] = p - onehot(c) out (c = -1: no class); returns the row's loss.
__device__ __forceinline__ double b2k_row_loss_residual(double* m, int kp, int c) {
  if (kp == 1) {
    const double x = m[0], yy = c == 1 ? 1.0 : 0.0;
    const double e = exp(-fabs(x));
    const double p = x >= 0.0 ? 1.0 / (1.0 + e) : e / (1.0 + e);
    m[0] = p - yy;
    return fmax(x, 0.0) + log1p(e) - yy * x;
  }
  double mx = m[0];
  for (int k = 1; k < kp; ++k) mx = fmax(mx, m[k]);
  double s = 0.0;
  for (int k = 0; k < kp; ++k) s += exp(m[k] - mx);
  const double lse = mx + log(s);
  const double loss = lse - (c >= 0 ? m[c] : 0.0);
  for (int k = 0; k < kp; ++k) m[k] = exp(m[k] - lse) - (k == c ? 1.0 : 0.0);
  return loss;
}

// The class index of label v: cmap [maxc] maps an integral label in [0, maxc) to its class, -1 = none.
__device__ __forceinline__ int b2k_class_of(float v, const int* __restrict__ cmap, int maxc) {
  return (v >= 0.f && v < (float)maxc && v == floorf(v)) ? cmap[(int)v] : -1;
}

// Binomial: the probability of class 1 at margin m.
__device__ __forceinline__ double b2k_sigmoid(double m) {
  const double e = exp(-fabs(m));
  return m >= 0.0 ? 1.0 / (1.0 + e) : e / (1.0 + e);
}

// Multinomial: the largest margin and its class (the lowest on a tie), then the softmax denominator.
struct B2kArgmax {
  double mx;
  int am;
};
__device__ __forceinline__ B2kArgmax b2k_softmax_argmax(const double* m, int kp) {
  B2kArgmax o{m[0], 0};
  for (int k = 1; k < kp; ++k)
    if (m[k] > o.mx) {
      o.mx = m[k];
      o.am = k;
    }
  return o;
}
__device__ __forceinline__ double b2k_softmax_denominator(const double* m, int kp, double mx) {
  double s = 0.0;
  for (int k = 0; k < kp; ++k) s += exp(m[k] - mx);
  return s;
}

// Random forests: a node of the flat forest, and the leaf (tree-local index) a row reaches; xf(f) is feature f.
struct B2kPNode {
  int32_t f;
  float t;
  int32_t l, r;
};
struct B2kFeatLdg {   // feature f of a row in global memory
  const float* x;
  __device__ __forceinline__ float operator()(int f) const { return __ldg(x + f); }
};
struct B2kFeatSmem {   // ... of a staged row in shared memory
  const float* x;
  __device__ __forceinline__ float operator()(int f) const { return x[f]; }
};
template <class XF>
__device__ __forceinline__ int b2k_rf_leaf(const B2kPNode* tree, XF xf) {
  int i = 0;
  for (int f = tree[0].f; f >= 0; f = tree[i].f) i = xf(f) <= tree[i].t ? tree[i].l : tree[i].r;
  return i;
}
// Classification, over the row's sums raw[o .. o + V - 1]: tot = their sum in k order; returns argmax_k (the lowest k
// on a tie).
__device__ __forceinline__ int b2k_rf_class_best(const double* __restrict__ raw, int64_t o, int V, double& tot) {
  tot = 0.0;
  int best = 0;
  for (int k = 0; k < V; ++k) {
    const double a = raw[o + k];
    tot = __dadd_rn(tot, a);
    if (a > raw[o + best]) best = k;
  }
  return best;
}
