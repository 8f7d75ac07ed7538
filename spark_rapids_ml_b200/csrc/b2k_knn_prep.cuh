// The shifted-frame prep of the wgmma distance screens (exact k-NN in b2k_knn.cu, DBSCAN in b2k_dbscan.cu).
// Included inside each translation unit's anonymous namespace, after b2k_ptx.cuh.

// The wgmma pass screens in the frame of the shift point s = item row 0 with every non-finite component replaced by 0
// (a NaN or inf there would otherwise reach every item): the screen ||x - s||^2 - 2 (q - s).(x - s) orders the items as
// ||q - x||^2 does, and its fp32 rounding scales with the data's spread rather than its distance from the origin.
__device__ __forceinline__ float knn_shift(const float* __restrict__ X, int f) {
  const float v = X[f];
  return isfinite(v) ? v : 0.f;
}

// index planes of x - s (rounded once to fp32), zero-padded to [n_pad][DP], and ||x - s||^2 of those same values.
// Plane row p holds X row perm[p] (perm NULL: row p); rows with perm[p] < 0 or p >= n are padding (+inf norm).
__global__ void __launch_bounds__(256) k_knn_prep(const float* __restrict__ X, int64_t n, int d,
                                                  const int32_t* __restrict__ perm, int64_t n_pad, int DP,
                                                  float* __restrict__ Xhi, float* __restrict__ Xlo,
                                                  float* __restrict__ norms) {
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= n_pad) return;
  const int64_t src = perm != nullptr ? (int64_t)perm[row] : row < n ? row : -1;
  double s = 0.0;
  for (int t = lane; t < DP; t += 32) {
    const float v = (src >= 0 && t < d) ? X[src * d + t] - knn_shift(X, t) : 0.f;
    const uint32_t hb = rn_tf32_bits(v);
    Xhi[row * DP + t] = __uint_as_float(hb);
    Xlo[row * DP + t] = __uint_as_float(rn_tf32_bits(v - __uint_as_float(hb)));
    s += (double)v * (double)v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) norms[row] = src >= 0 ? (float)s : __int_as_float(0x7f800000);
}

// q - s as the wgmma pass reads it.  rn_tf32_bits carries out of the mantissa for NaNs whose payload fills its top bits,
// so the device's canonical NaN 0x7fffffff would split into hi = lo = -0 and a NaN query would be screened as finite;
// 0x7fc00000 stays NaN as hi.  (An item needs no such care: its NaN norm makes its screen NaN.)
__device__ __forceinline__ float knn_shifted_q(float q, float s) {
  const float v = q - s;
  return isnan(v) ? __int_as_float(0x7fc00000) : v;
}

// Qs = Q - s for the wgmma pass, [nq][d] with d % 4 == 0 and both buffers 16-byte aligned
__global__ void __launch_bounds__(256) k_knn_shift_q(const float4* __restrict__ Q, int64_t n4, int d,
                                                     const float* __restrict__ X, float4* __restrict__ Qs) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const int f = (int)(i * 4 % d);
    const float4 q = Q[i];
    Qs[i] = make_float4(knn_shifted_q(q.x, knn_shift(X, f)), knn_shifted_q(q.y, knn_shift(X, f + 1)),
                        knn_shifted_q(q.z, knn_shift(X, f + 2)), knn_shifted_q(q.w, knn_shift(X, f + 3)));
  }
}
