// Per-partition Arrow-batch -> device ingest (replaces the reference's host-side stacking
// `np.array(list(pdf[alias.data]))` core.py:916, multi-column np.array(pdf[cols]) core.py:910, the second host
// copy `_concat_and_free` utils.py:358-400 and cuML's input_to_cuml_array H2D).  The batch's Arrow value
// buffer goes host -> pinned staging -> HBM once, and a coalesced/vectorised kernel converts (f64/int -> f32)
// or transposes (d scalar columns -> row-major rows) straight into the reserved [n_max, d] matrix.
#include <string.h>
#include <unistd.h>

#include <atomic>
#include <chrono>
#include <condition_variable>
#include <mutex>
#include <thread>
#include <vector>

#include "b2k_internal.cuh"

// The pageable -> pinned staging copy is the bound of the Arrow-batch ingest (one host thread moves ~17-20 GB/s, the PCIe
// Gen5 link 55 GB/s): a few helper threads split every copy.  Helpers spin for a short while after a job (batches arrive
// every few hundred microseconds during a partition's ingest) and block on a condition variable when idle.
struct B2kCopyPool {
  struct Job { char* dst; const char* src; size_t bytes; };
  std::vector<std::thread> workers;
  std::mutex mu;
  std::condition_variable cv;
  std::atomic<uint64_t> generation{0};
  std::atomic<int> pending{0};
  std::atomic<bool> stop{false};
  Job job{nullptr, nullptr, 0};
  int nthreads = 1;   // helpers + the caller

  static void slice(const Job& j, int part, int parts, char** d, const char** s, size_t* n) {
    const size_t per = ((j.bytes / parts) + 4095) & ~(size_t)4095;
    const size_t lo = std::min(j.bytes, per * (size_t)part);
    const size_t hi = part == parts - 1 ? j.bytes : std::min(j.bytes, per * (size_t)(part + 1));
    *d = j.dst + lo; *s = j.src + lo; *n = hi - lo;
  }
  void worker(int id) {
    uint64_t seen = 0;
    for (;;) {
      // spin briefly for the next job, then sleep
      auto t0 = std::chrono::steady_clock::now();
      while (generation.load(std::memory_order_acquire) == seen && !stop.load(std::memory_order_relaxed)) {
        if (std::chrono::steady_clock::now() - t0 > std::chrono::microseconds(400)) {
          std::unique_lock<std::mutex> lk(mu);
          cv.wait(lk, [&] { return generation.load(std::memory_order_acquire) != seen || stop.load(); });
          break;
        }
      }
      if (stop.load()) return;
      seen = generation.load(std::memory_order_acquire);
      char* d; const char* s; size_t n;
      slice(job, id, nthreads, &d, &s, &n);
      if (n) memcpy(d, s, n);
      pending.fetch_sub(1, std::memory_order_acq_rel);
    }
  }
  explicit B2kCopyPool(int n) : nthreads(n) {
    for (int i = 1; i < n; ++i) workers.emplace_back([this, i] { worker(i); });
  }
  ~B2kCopyPool() {
    { std::lock_guard<std::mutex> lk(mu); stop.store(true); }
    cv.notify_all();
    for (auto& t : workers) t.join();
  }
  void copy(void* dst, const void* src, size_t bytes) {
    if (nthreads <= 1 || bytes < ((size_t)512 << 10)) { memcpy(dst, src, bytes); return; }
    job = Job{static_cast<char*>(dst), static_cast<const char*>(src), bytes};
    pending.store(nthreads - 1, std::memory_order_release);
    { std::lock_guard<std::mutex> lk(mu); generation.fetch_add(1, std::memory_order_acq_rel); }
    cv.notify_all();
    char* d; const char* s; size_t n;
    slice(job, 0, nthreads, &d, &s, &n);
    if (n) memcpy(d, s, n);
    while (pending.load(std::memory_order_acquire) != 0) { /* helpers finish within microseconds of the caller */ }
  }
};

void b2k_copy_pool_destroy(b2k_ctx* ctx) {
  delete static_cast<B2kCopyPool*>(ctx->copy_pool);
  ctx->copy_pool = nullptr;
}

namespace {
constexpr size_t STAGE_BYTES = (size_t)64 << 20;

B2kCopyPool* copy_pool(b2k_ctx* ctx) {
  if (!ctx->copy_pool) {
    int n = ctx->ingest_threads;
    if (n <= 0) {   // default: 4, capped by the CPUs this process may use (affinity, cgroup quota)
      long cpus = sysconf(_SC_NPROCESSORS_ONLN);
      FILE* f = fopen("/sys/fs/cgroup/cpu.max", "r");
      if (f) {
        char q[64] = {0};
        long period = 0;
        if (fscanf(f, "%63s %ld", q, &period) == 2 && strcmp(q, "max") != 0 && period > 0) {
          long quota = atol(q) / period;
          if (quota >= 1 && quota < cpus) cpus = quota;
        }
        fclose(f);
      }
      n = (int)std::max(1L, std::min(4L, cpus / 2));
    }
    ctx->copy_pool = new B2kCopyPool(n);
  }
  return static_cast<B2kCopyPool*>(ctx->copy_pool);
}

__host__ __device__ inline size_t dtype_size(int t) {
  switch (t) {
    case B2K_F32: return 4;
    case B2K_F64: return 8;
    case B2K_I8: return 1;
    case B2K_I16: return 2;
    case B2K_I32: return 4;
    case B2K_I64: return 8;
  }
  return 0;
}

template <typename T>
__device__ __forceinline__ float to_f32(T v) { return (float)v; }

// contiguous convert: 4 elements per thread, 16 B stores
template <typename T>
__global__ void __launch_bounds__(256) k_convert_rows(const T* __restrict__ src, float* __restrict__ dst,
                                                      size_t count) {
  size_t i4 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  size_t stride = (size_t)gridDim.x * blockDim.x * 4;
  const bool aligned = ((reinterpret_cast<uintptr_t>(dst) & 15) == 0);
  for (; i4 < count; i4 += stride) {
    if (i4 + 4 <= count && aligned) {
      float4 o;
      o.x = to_f32(src[i4]);
      o.y = to_f32(src[i4 + 1]);
      o.z = to_f32(src[i4 + 2]);
      o.w = to_f32(src[i4 + 3]);
      *reinterpret_cast<float4*>(dst + i4) = o;
    } else {
      for (size_t e = i4; e < count && e < i4 + 4; ++e) dst[e] = to_f32(src[e]);
    }
  }
}

// columnar [d][rows] (each column contiguous) -> row-major rows: 32x32 shared-memory tile transpose,
// coalesced on both sides.
template <typename T>
__global__ void __launch_bounds__(256) k_transpose_cols(const T* __restrict__ src, int64_t rows, int d,
                                                        float* __restrict__ dst /* [rows][d] */) {
  __shared__ float tile[32][33];
  int64_t r0 = (int64_t)blockIdx.x * 32;
  int c0 = blockIdx.y * 32;
  int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 8 rows of threads
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int c = c0 + ty + 8 * i;
    int64_t r = r0 + tx;
    float v = 0.f;
    if (c < d && r < rows) v = to_f32(src[(size_t)c * rows + r]);
    tile[ty + 8 * i][tx] = v;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int64_t r = r0 + ty + 8 * i;
    int c = c0 + tx;
    if (r < rows && c < d) dst[(size_t)r * d + c] = tile[tx][ty + 8 * i];
  }
}

template <typename T>
int launch_convert(b2k_ctx* ctx, const void* src, float* dst, size_t count, cudaStream_t s) {
  size_t threads = (count + 3) / 4;
  size_t blocks = (threads + 255) / 256;
  size_t cap = (size_t)ctx->sm_count * 16;
  if (blocks > cap) blocks = cap;
  if (blocks == 0) return B2K_OK;
  k_convert_rows<T><<<(unsigned)blocks, 256, 0, s>>>(static_cast<const T*>(src), dst, count);
  ctx->stats.kernel_launches++;
  B2K_CUDA_OK(ctx, cudaGetLastError());
  return B2K_OK;
}
template <typename T>
int launch_transpose(b2k_ctx* ctx, const void* src, int64_t rows, int d, float* dst, cudaStream_t s) {
  dim3 grid((unsigned)((rows + 31) / 32), (unsigned)((d + 31) / 32));
  k_transpose_cols<T><<<grid, 256, 0, s>>>(static_cast<const T*>(src), rows, d, dst);
  ctx->stats.kernel_launches++;
  B2K_CUDA_OK(ctx, cudaGetLastError());
  return B2K_OK;
}

int ensure_staging(b2k_ctx* ctx) {
  if (ctx->pinned[0]) return B2K_OK;
  for (int i = 0; i < 2; ++i) {
    B2K_CUDA_OK(ctx, cudaHostAlloc(&ctx->pinned[i], STAGE_BYTES, cudaHostAllocDefault));
    B2K_CUDA_OK(ctx, cudaMalloc(&ctx->dev_stage[i], STAGE_BYTES));
    B2K_CUDA_OK(ctx, cudaEventCreateWithFlags(&ctx->stage_evt[i], cudaEventDisableTiming));
  }
  ctx->pinned_bytes = STAGE_BYTES;
  ctx->dev_stage_bytes = STAGE_BYTES;
  return B2K_OK;
}

bool host_ptr_is_pinned(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeHost;
}

int convert_dispatch(b2k_ctx* ctx, int dt, const void* src, float* dst, size_t count, cudaStream_t s) {
  switch (dt) {
    case B2K_F32: return launch_convert<float>(ctx, src, dst, count, s);
    case B2K_F64: return launch_convert<double>(ctx, src, dst, count, s);
    case B2K_I8: return launch_convert<int8_t>(ctx, src, dst, count, s);
    case B2K_I16: return launch_convert<int16_t>(ctx, src, dst, count, s);
    case B2K_I32: return launch_convert<int32_t>(ctx, src, dst, count, s);
    case B2K_I64: return launch_convert<int64_t>(ctx, src, dst, count, s);
  }
  return b2k_fail(ctx, B2K_ERR_INVALID, "ingest: unknown src_dtype");
}
int transpose_dispatch(b2k_ctx* ctx, int dt, const void* src, int64_t rows, int d, float* dst, cudaStream_t s) {
  switch (dt) {
    case B2K_F32: return launch_transpose<float>(ctx, src, rows, d, dst, s);
    case B2K_F64: return launch_transpose<double>(ctx, src, rows, d, dst, s);
    case B2K_I8: return launch_transpose<int8_t>(ctx, src, rows, d, dst, s);
    case B2K_I16: return launch_transpose<int16_t>(ctx, src, rows, d, dst, s);
    case B2K_I32: return launch_transpose<int32_t>(ctx, src, rows, d, dst, s);
    case B2K_I64: return launch_transpose<int64_t>(ctx, src, rows, d, dst, s);
  }
  return b2k_fail(ctx, B2K_ERR_INVALID, "ingest: unknown src_dtype");
}
// One staged batch of Spark vector rows -> CSR rows: a warp per row; row i's entries go to positions vo[i] - vo[0] of
// the batch (its values' offsets), a dense row (type 1) gets the column indices 0 .. len - 1.
template <typename T>
__global__ void __launch_bounds__(256)
k_csr_ingest(const int8_t* __restrict__ type, const int32_t* __restrict__ io, const int32_t* __restrict__ iv,
             const int32_t* __restrict__ vo, const T* __restrict__ vv, int64_t rows, int64_t nnz0,
             int64_t* __restrict__ indptr, int32_t* __restrict__ indices, float* __restrict__ values) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarp = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < rows; r += nwarp) {
    const int64_t p = vo[r] - vo[0], len = vo[r + 1] - vo[r], ip = io[r] - io[0];
    const bool dense = type[r] == 1;
    for (int64_t e = lane; e < len; e += 32) {
      indices[nnz0 + p + e] = dense ? (int32_t)e : iv[ip + e];
      values[nnz0 + p + e] = to_f32(vv[p + e]);
    }
    if (lane == 0) indptr[r + 1] = nnz0 + p + len;
  }
}
}  // namespace

extern "C" int b2k_ingest_csr_append(b2k_ctx* ctx, int64_t* indptr, int32_t* indices, float* values, int64_t n_max,
                                     int64_t nnz_max, int64_t d, int64_t row0, int64_t nnz0, const int8_t* type,
                                     const int32_t* size, const int32_t* idx_offsets, const int32_t* idx_values,
                                     const int32_t* val_offsets, const void* val_values, int val_dtype, int64_t n_b,
                                     uintptr_t stream, int64_t* nnz_written) {
  if (!ctx) return b2k_fail(nullptr, B2K_ERR_INVALID, "b2k_ingest_csr_append: ctx is NULL");
  if (nnz_written) *nnz_written = 0;
  if (!indptr || !indices || !values || n_b < 0 || row0 < 0 || nnz0 < 0 || row0 + n_b > n_max || d < 1 ||
      (n_b > 0 && (!type || !size || !idx_offsets || !idx_values || !val_offsets || !val_values)))
    return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_ingest_csr_append: bad destination/source/d/row range");
  if (val_dtype != B2K_F32 && val_dtype != B2K_F64)
    return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_ingest_csr_append: values must be f32 or f64");
  if (n_b == 0) return B2K_OK;
  // the row widths, as the dense ingest checks them: a sparse row's size and a dense row's length must be d, and a
  // sparse row holds as many indices as values
  for (int64_t i = 0; i < n_b; ++i) {
    const int64_t nv = (int64_t)val_offsets[i + 1] - val_offsets[i], ni = (int64_t)idx_offsets[i + 1] - idx_offsets[i];
    if (type[i] != 0 && type[i] != 1)
      return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_ingest_csr_append: row " + std::to_string(i) + " has vector type " +
                                                std::to_string((int)type[i]) + " (0 sparse, 1 dense)");
    const int64_t width = type[i] == 0 ? (int64_t)size[i] : nv;
    if (width != d)
      return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_ingest_csr_append: row " + std::to_string(i) + " has size " +
                                                std::to_string(width) + ", expected " + std::to_string(d));
    if (type[i] == 0 && ni != nv)
      return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_ingest_csr_append: row " + std::to_string(i) + " has " +
                                                std::to_string(ni) + " indices and " + std::to_string(nv) + " values");
  }
  const int64_t nnz_b = (int64_t)val_offsets[n_b] - val_offsets[0];
  if (nnz0 + nnz_b > nnz_max) return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_ingest_csr_append: nnz_max exceeded");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  B2K_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  B2K_TRY(ensure_staging(ctx));
  const size_t es = dtype_size(val_dtype);
  // rows [r, r1) per staging slot: type | index offsets | value offsets | indices | values, each 16-byte aligned
  auto al = [](size_t b) { return (b + 15) & ~(size_t)15; };
  auto bytes = [&](int64_t r, int64_t r1) {
    const int64_t ni = (int64_t)idx_offsets[r1] - idx_offsets[r], nv = (int64_t)val_offsets[r1] - val_offsets[r];
    return al(r1 - r) + 2 * al(4 * (size_t)(r1 - r + 1)) + al(4 * (size_t)ni) + al(es * (size_t)nv);
  };
  for (int64_t r = 0; r < n_b;) {
    int64_t r1 = n_b;
    while (r1 > r + 1 && bytes(r, r1) > STAGE_BYTES) r1 = r + (r1 - r) / 2;
    if (bytes(r, r1) > STAGE_BYTES)
      return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "b2k_ingest_csr_append: one row exceeds the staging buffer");
    const int64_t rows = r1 - r;
    const int64_t ni = (int64_t)idx_offsets[r1] - idx_offsets[r], nv = (int64_t)val_offsets[r1] - val_offsets[r];
    const int b = ctx->stage_next;
    ctx->stage_next ^= 1;
    B2K_CUDA_OK(ctx, cudaEventSynchronize(ctx->stage_evt[b]));   // the previous use of this slot has drained
    char* pin = static_cast<char*>(ctx->pinned[b]);
    char* dev = static_cast<char*>(ctx->dev_stage[b]);
    size_t off = 0;
    const size_t o_type = off; memcpy(pin + off, type + r, rows); off += al(rows);
    const size_t o_io = off; memcpy(pin + off, idx_offsets + r, 4 * (rows + 1)); off += al(4 * (rows + 1));
    const size_t o_vo = off; memcpy(pin + off, val_offsets + r, 4 * (rows + 1)); off += al(4 * (rows + 1));
    const size_t o_iv = off; copy_pool(ctx)->copy(pin + off, idx_values + idx_offsets[r], 4 * (size_t)ni); off += al(4 * ni);
    const size_t o_vv = off;
    copy_pool(ctx)->copy(pin + off, static_cast<const char*>(val_values) + es * (size_t)val_offsets[r], es * (size_t)nv);
    off += al(es * nv);
    B2K_CUDA_OK(ctx, cudaMemcpyAsync(dev, pin, off, cudaMemcpyHostToDevice, s));
    const int64_t at = nnz0 + (int64_t)val_offsets[r] - val_offsets[0];
    const unsigned grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>((rows + 7) / 8, 16 * ctx->sm_count));
    auto tp = reinterpret_cast<const int8_t*>(dev + o_type);
    auto io = reinterpret_cast<const int32_t*>(dev + o_io);
    auto vo = reinterpret_cast<const int32_t*>(dev + o_vo);
    auto iv = reinterpret_cast<const int32_t*>(dev + o_iv);
    if (val_dtype == B2K_F64)
      k_csr_ingest<double><<<grid, 256, 0, s>>>(tp, io, iv, vo, reinterpret_cast<const double*>(dev + o_vv), rows, at,
                                                indptr + row0 + r, indices, values);
    else
      k_csr_ingest<float><<<grid, 256, 0, s>>>(tp, io, iv, vo, reinterpret_cast<const float*>(dev + o_vv), rows, at,
                                               indptr + row0 + r, indices, values);
    B2K_CUDA_OK(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
    B2K_CUDA_OK(ctx, cudaEventRecord(ctx->stage_evt[b], s));
    r = r1;
  }
  if (nnz_written) *nnz_written = nnz_b;
  return B2K_OK;
}

extern "C" int b2k_ingest_append(b2k_ctx* ctx, float* dst, int64_t n_max, int d, int64_t row0, const void* values,
                                 const int32_t* offsets, int64_t n_b, int src_dtype, int layout,
                                 uintptr_t stream, int64_t* rows_written) {
  if (!ctx) return b2k_fail(nullptr, B2K_ERR_INVALID, "b2k_ingest_append: ctx is NULL");
  if (rows_written) *rows_written = 0;
  if (!dst || !values || d <= 0 || n_b < 0 || row0 < 0 || row0 + n_b > n_max)
    return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_ingest_append: bad dst/values/d/row range");
  const size_t es = dtype_size(src_dtype);
  if (es == 0) return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_ingest_append: unknown src_dtype");
  if (n_b == 0) return B2K_OK;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  B2K_CUDA_OK(ctx, cudaSetDevice(ctx->device));

  if (layout == B2K_LAYOUT_ROWS) {
    size_t first = 0;
    if (offsets) {
      // the reference's stacking fails on ragged rows (np.array of unequal lists); so do we, loudly.
      first = (size_t)offsets[0];
      for (int64_t i = 0; i < n_b; ++i) {
        if (offsets[i + 1] - offsets[i] != d)
          return b2k_fail(ctx, B2K_ERR_INVALID,
                          "b2k_ingest_append: row " + std::to_string(i) + " has length " +
                              std::to_string(offsets[i + 1] - offsets[i]) + ", expected " + std::to_string(d));
      }
    }
    const char* src = static_cast<const char*>(values) + first * es;
    const size_t total = (size_t)n_b * d;
    float* out = dst + (size_t)row0 * d;
    const bool pinned_src = host_ptr_is_pinned(src);
    if (pinned_src && src_dtype == B2K_F32) {
      // zero-staging path: the caller's buffer is already page-locked
      B2K_CUDA_OK(ctx, cudaMemcpyAsync(out, src, total * 4, cudaMemcpyHostToDevice, s));
    } else {
      B2K_TRY(ensure_staging(ctx));
      size_t per = STAGE_BYTES / es;
      per -= per % 4;
      for (size_t done = 0; done < total; done += per) {
        size_t cnt = total - done < per ? total - done : per;
        int b = ctx->stage_next;
        ctx->stage_next ^= 1;
        B2K_CUDA_OK(ctx, cudaEventSynchronize(ctx->stage_evt[b]));  // previous use of this slot has drained
        const void* hsrc = src + done * es;
        if (!pinned_src) {
          copy_pool(ctx)->copy(ctx->pinned[b], hsrc, cnt * es);
          hsrc = ctx->pinned[b];
        }
        if (src_dtype == B2K_F32) {
          B2K_CUDA_OK(ctx, cudaMemcpyAsync(out + done, hsrc, cnt * 4, cudaMemcpyHostToDevice, s));
        } else {
          B2K_CUDA_OK(ctx, cudaMemcpyAsync(ctx->dev_stage[b], hsrc, cnt * es, cudaMemcpyHostToDevice, s));
          B2K_TRY(convert_dispatch(ctx, src_dtype, ctx->dev_stage[b], out + done, cnt, s));
        }
        B2K_CUDA_OK(ctx, cudaEventRecord(ctx->stage_evt[b], s));
      }
    }
  } else if (layout == B2K_LAYOUT_COLUMNS) {
    const void* const* cols = static_cast<const void* const*>(values);
    for (int c = 0; c < d; ++c)
      if (!cols[c]) return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_ingest_append: NULL column pointer");
    B2K_TRY(ensure_staging(ctx));
    int64_t rows_per = (int64_t)(STAGE_BYTES / ((size_t)d * es));
    rows_per -= rows_per % 32;
    if (rows_per < 32) return b2k_fail(ctx, B2K_ERR_UNSUPPORTED, "b2k_ingest_append: d too large for staging");
    for (int64_t r = 0; r < n_b; r += rows_per) {
      int64_t cnt = n_b - r < rows_per ? n_b - r : rows_per;
      int b = ctx->stage_next;
      ctx->stage_next ^= 1;
      B2K_CUDA_OK(ctx, cudaEventSynchronize(ctx->stage_evt[b]));
      char* pin = static_cast<char*>(ctx->pinned[b]);
      for (int c = 0; c < d; ++c)
        memcpy(pin + (size_t)c * cnt * es, static_cast<const char*>(cols[c]) + (size_t)r * es, (size_t)cnt * es);
      B2K_CUDA_OK(ctx, cudaMemcpyAsync(ctx->dev_stage[b], pin, (size_t)d * cnt * es, cudaMemcpyHostToDevice, s));
      B2K_TRY(transpose_dispatch(ctx, src_dtype, ctx->dev_stage[b], cnt, d, dst + (size_t)(row0 + r) * d, s));
      B2K_CUDA_OK(ctx, cudaEventRecord(ctx->stage_evt[b], s));
    }
  } else {
    return b2k_fail(ctx, B2K_ERR_INVALID, "b2k_ingest_append: unknown layout");
  }
  if (rows_written) *rows_written = n_b;
  return B2K_OK;
}
