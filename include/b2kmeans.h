/*
 * b2kmeans.h — C ABI of libb2kmeans.so: the H100-native (sm_90a) KMeans Lloyd-loop and PCA backend that
 * replaces the cuML calls on spark-rapids-ml's distributed KMeans.fit() and PCA.fit() paths.
 *
 * Reference interfaces each entry point stands in for (paths relative to the reference repo
 * NVIDIA/spark-rapids-ml @ c51743bb, python/src/spark_rapids_ml/):
 *
 *   b2k_ctx_create/destroy      core.py:390-407 (_set_gpu_device) + cuml_context.py:68 (Handle)
 *   b2k_comm_unique_id          cuml_context.py:75-81   (nccl.get_unique_id on rank 0)
 *   b2k_comm_init               cuml_context.py:123-131 (nccl.init + inject_comms_on_handle)
 *   b2k_comm_destroy / _abort   cuml_context.py:158-175 (destroy, or abort when an exception is in flight)
 *   b2k_ingest_append           core.py:907-941 (per-Arrow-batch np.array(list(...))) +
 *                               utils.py:358-400 (_concat_and_free) + utils.py:452-522 (reserved buffer)
 *   b2k_kmeans_fit              clustering.py:383-425 (KMeansMG(handle, **cuml_init).fit(X) and the
 *                               cluster_centers_/n_iter_/inertia_ attribute reads)
 *   b2k_kmeans_lloyd            the Lloyd loop inside the above (EXTERNAL cuML: minClusterAndDistance,
 *                               reduce_rows_by_key, allreduce x2, divide, convergence) — also the unit
 *                               bench.py times as one "step" per iteration
 *   b2k_kmeans_assign           clustering.py:582-602 (KMeans.predict with injected cluster_centers_)
 *   b2k_pca_fit                 feature.py:196-242 (PCAMG(handle, **cuml_init).fit(...) and the mean_/components_/
 *                               explained_variance_ratio_/singular_values_ attribute reads)
 *   b2k_pca_finalize            the eigen step inside the above (EXTERNAL cuML: eigendecomposition of the covariance,
 *                               sign flip, explained variance ratio, singular values)
 *   b2k_pca_transform           feature.py:398-451 (PCAMG.transform with injected components_, mean added back)
 *   b2k_knn_search              knn.py:662-804 (NearestNeighborsMG(handle).kneighbors(...) and the row -> id mapping
 *                               of NearestNeighborsModel.kneighbors' fit function)
 *   b2k_linreg_moments          regression.py:546-607 (the passes over the data of LinearRegressionMG / RidgeMG / CDMG)
 *   b2k_linreg_solve            the solvers inside them (normal equations, coordinate descent) and the rescaling
 *   b2k_linreg_predict          regression.py:800-862 (LinearRegressionModel's transform: cuML predict)
 *   b2k_logreg_labels           classification.py:1075-1103 (the classes cuML finds and the label checks after them)
 *   b2k_logreg_eval             one loss-and-gradient evaluation of cuML's qn solver behind LogisticRegressionMG
 *   b2k_logreg_minimize         cuML's qn solver (L-BFGS / OWL-QN) itself
 *   b2k_logreg_fit              classification.py:984-1171 (LogisticRegressionMG.fit per param map, rescaling, centring)
 *   b2k_logreg_predict          classification.py:1455-1553 (LogisticRegressionModel's transform)
 *   b2k_ingest_csr_append       core.py:193-264, 507-521 (_read_csr_matrix_from_unwrapped_spark_vec: Spark vector rows
 *                               -> a per-partition scipy CSR matrix, the default with enable_sparse_data_optim=None)
 *   b2k_logreg_eval_csr         one evaluation of cuML's qn solver on the CSR input of classification.py:1038-1060
 *   b2k_logreg_fit_csr          classification.py:998-1171 with the CSR matrix (LogisticRegressionMG.fit on sparse rows)
 *   b2k_logreg_predict_csr      classification.py:1455-1553 on sparse rows (cuML predict on a CSR matrix)
 *   b2k_dbscan_fit              clustering.py:1049-1186 (DBSCANModel's fit function: cuML DBSCANMG(handle).fit_predict
 *                               over NCCL + UCX, labels gathered on rank 0)
 *   b2k_rf_fit / b2k_rf_forest  tree.py:343-527 (the per-worker cuML RandomForest fits and the treelite models they
 *                               return), classification.py:285-676, regression.py:865-1147
 *   b2k_rf_predict              tree.py:670- (the model's transform: cuML's forest inference over treelite)
 *   b2k_umap_fit / _graph       umap.py:1009-1065 (UMAP's fit function: cuML UMAP(...).fit on one partition)
 *   b2k_umap_transform          umap.py:1449-1551 (UMAPModel's transform: cuML UMAP.transform)
 *   b2k_ivf_search              knn.py:1406-1692 (ApproximateNearestNeighborsModel.kneighbors with algorithm "ivfflat":
 *                               the cuVS IVF-Flat build and search per partition and the top-k aggregation)
 *   b2k_silhouette              none: the reference has no clustering evaluator (its DBSCAN benchmark collects the
 *                               frame and calls scikit-learn's silhouette_score); stands in for Spark's
 *                               pyspark.ml.evaluation.ClusteringEvaluator (metricName "silhouette")
 *   b2k_gmm_fit / _predict      none: the reference has no Gaussian mixture; stands in for Spark's
 *                               pyspark.ml.clustering.GaussianMixture (fit and GaussianMixtureModel.transform)
 *   b2k_bkm_fit / _predict      none: the reference has no bisecting k-means; stands in for Spark's
 *                               pyspark.ml.clustering.BisectingKMeans (fit and BisectingKMeansModel.transform /
 *                               computeCost)
 *   b2k_mlp_eval / _fit /       none: the reference has no multilayer perceptron; stands in for Spark's
 *     _predict                  pyspark.ml.classification.MultilayerPerceptronClassifier (fit and the model's transform)
 *   b2k_als_fit / _predict /    none: the reference has no recommender; stands in for Spark's
 *     _recommend                pyspark.ml.recommendation.ALS (fit, ALSModel.transform and the recommendFor* calls)
 *   b2k_silhouette_multi        none: the reference tunes KMeans with pyspark's CrossValidator, scoring each model on
 *                               the CPU; here one device pass scores every model of a param grid
 *
 * Conventions
 *   - Plain C, no exceptions across the boundary: every call returns a b2k_status; the message for the
 *     last failure on a context is b2k_last_error(ctx) (ctx == NULL: last failure of a call that has no
 *     context, e.g. b2k_ctx_create).
 *   - All device pointers are BORROWED from the caller (torch tensors on the Python side); the library owns
 *     only its scratch, TMA descriptors, pinned staging and the NCCL communicator, all inside the ctx.
 *   - `stream` is a cudaStream_t passed as uintptr_t (0 = legacy default stream).  All device work is
 *     enqueued on it.  Calls that return host values (fit, lloyd, pca_fit) synchronise that stream before returning.
 *   - One context per process per GPU; NOT thread-safe (callers are single-threaded Spark Python workers).
 *   - There is no CPU fallback: without a CUDA device every compute entry point fails with B2K_ERR_CUDA.
 */
#ifndef B2KMEANS_H_
#define B2KMEANS_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2K_VERSION 100 /* 0.1.0 */
#define B2K_UNIQUE_ID_BYTES 128

typedef struct b2k_ctx b2k_ctx;

typedef enum b2k_status {
  B2K_OK = 0,
  B2K_ERR_INVALID = 1,     /* bad argument */
  B2K_ERR_CUDA = 2,        /* CUDA runtime/driver error (message has the cudaError string) */
  B2K_ERR_NCCL = 3,        /* NCCL error or libnccl not loadable */
  B2K_ERR_UNSUPPORTED = 4, /* shape/dtype/layout not supported by the requested kernel path */
  B2K_ERR_STATE = 5,       /* e.g. comm already initialised / not initialised */
  B2K_ERR_NOMEM = 6
} b2k_status;

/* cuml_init["init"] after the reference's param mapping (clustering.py:86-98,134): "scalable-k-means++"
 * (Spark "k-means||"), "random", or an injected array (used by every parity test). */
typedef enum b2k_init_mode {
  B2K_INIT_ARRAY = 0,
  B2K_INIT_RANDOM = 1,
  B2K_INIT_KMEANS_PARALLEL = 2
} b2k_init_mode;

typedef enum b2k_dtype {
  B2K_F32 = 0,
  B2K_F64 = 1,
  B2K_I8 = 2,
  B2K_I16 = 3,
  B2K_I32 = 4,
  B2K_I64 = 5
} b2k_dtype;

/* Host layouts the Spark->worker Arrow stream delivers (core.py:907-916):
 *   ROWS    : one contiguous [n_b, d] row-major values buffer — the child buffer of an Arrow
 *             list<T>/fixed_size_list<T> column; `offsets` (n_b+1 int32, may be NULL for fixed_size_list)
 *             is validated for a constant row length d.
 *   COLUMNS : d separate scalar columns; `values` is a const void* const[d] array of column buffers. */
typedef enum b2k_layout { B2K_LAYOUT_ROWS = 0, B2K_LAYOUT_COLUMNS = 1 } b2k_layout;

/* Values for the "kernel_path" option. AUTO picks the wgmma fused kernel when the shape fits it. */
typedef enum b2k_kernel_path {
  B2K_PATH_AUTO = 0,
  B2K_PATH_GENERIC = 1, /* SIMT fp32 tiles: any (k, d) */
  B2K_PATH_FUSED = 2    /* TMA + wgmma fused assign (+ deterministic update pass) (3xTF32 for k, d <= 128; 1xTF32 screening + exact
                           recheck for k, d <= 256); fails with UNSUPPORTED otherwise */
} b2k_kernel_path;

/* Per-fit statistics (b2k_get_stats): what ran, for tests and bench.py's gpu_launches claim. */
typedef struct b2k_stats {
  int64_t kernel_launches;     /* kernels of this library launched since ctx creation / last reset */
  int64_t fused_tc_launches;   /* ... of which the wgmma fused assign kernel */
  int64_t generic_launches;    /* ... of which generic assign/update kernels */
  int64_t nccl_allreduces;     /* collectives issued */
  int32_t last_path;           /* b2k_kernel_path actually used by the last fit/lloyd/assign */
  int32_t last_n_iter;
  double last_fused_ms;        /* mean device time of the fused kernel over the last lloyd call (CUDA events
                                  on the caller's stream; 0 unless option "time_kernels" is 1) */
  double last_loop_ms;         /* device time of the whole last Lloyd loop (same condition) */
  double last_reduce_ms;       /* option "time_kernels" = 2: mean device time per iteration of the partial fold, ... */
  double last_allreduce_ms;    /* ... of the NCCL allreduce of the [k*d+k+1] buffer (0 on one rank), ... */
  double last_finalize_ms;     /* ... and of finalize */
  int64_t recheck_rows;        /* large-shape kernel (k, d <= 256: 1xTF32 screening): rows of the last lloyd/assign call
                                  whose approximate margin was below the proven error bound and were re-decided
                                  exactly (summed over its passes; 0 unless option "collect_recheck" is 1) */
  int64_t recheck_candidates;  /* ... exact candidate distances evaluated for them */
  int64_t path_switch_iter;    /* iteration from which the last Lloyd loop left the large-shape wgmma kernel for the
                                  generic kernels because most rows needed the exact fix-up (option "adaptive_path",
                                  default 1; only with kernel_path = auto); -1 = it did not */
  double last_probe_ms;        /* b2k_ivf_search with option "time_kernels" != 0: the probe selection (device time) */
} b2k_stats;
/* b2k_pca_fit reuses the fields: last_path = the Gram pass that ran (B2K_PATH_FUSED = wgmma, B2K_PATH_GENERIC = SIMT);
 * with option "time_kernels" != 0, last_reduce_ms = the column-sum pass, last_fused_ms = the Gram pass, last_allreduce_ms
 * = both allreduces (device times, CUDA events), last_finalize_ms = the host eigen step and last_loop_ms = the whole call
 * (host clock). */

int b2k_version(void);
const char* b2k_last_error(const b2k_ctx* ctx);

int b2k_ctx_create(int device, b2k_ctx** out);
int b2k_ctx_destroy(b2k_ctx* ctx);
/* Options:
 *   "kernel_path"      b2k_kernel_path
 *   "time_kernels"     0/1/2: CUDA events around every fused launch; 2 = also around the partial fold, the allreduce and
 *                      finalize
 *   "check_every"      iterations between host convergence polls, default 4
 *   "grid_limit"       cap on persistent CTAs, 0 = #SMs; also caps the CTAs of the fused logistic pass (0 = as many as
 *                      fit on every SM at once)
 *   "variant_t"        1 = route every shape with k, d <= 256 through the large-shape kernel b2k_fused_t.cu; default 0 =
 *                      only shapes the 3xTF32 kernel does not cover
 *   "collect_recheck"  1 = lloyd/assign synchronise and fill b2k_stats.recheck_*
 *   "adaptive_path"    see b2k_stats.path_switch_iter
 *   "ingest_threads"   host threads of the pageable -> pinned staging copy of b2k_ingest_append; 0 = default: 4, capped
 *                      by half of the CPUs the process may use
 *   "rf_group_nodes"   b2k_rf_fit: cap on the nodes of one histogram pass, 0 = as many as fit (tests)
 *   "rf_flush_tiles"   b2k_rf_fit: cap on the tiles a CTA of the cluster pass adds between flushes, 0 = the bound (tests)
 *   "profile_fused"    0/1; the k, d <= 128 fused kernel runs a separately compiled instantiation that records per-warp
 *                      phase cycle counters, read back with b2k_get_fused_profile; the large-shape kernel rejects it
 *                      with B2K_ERR_UNSUPPORTED
 *   "probe", "pair"    accepted and ignored (switches of earlier builds) */
int b2k_ctx_set_option(b2k_ctx* ctx, const char* key, int64_t value);
int b2k_get_stats(const b2k_ctx* ctx, b2k_stats* out);
/* Diagnostics: per-warp phase cycle counters of the last fused launch made with option profile_fused (k, d <= 128
 * kernel): out[grid][warps][8] int64 (cap = capacity of out in elements), *grid_out and *warps_out (= 12) set.
 * Consumer warps 0-7: X wait, centre wait, hand-off wait, A load + split, MMA issue + drain, epilogue, sort, column
 * sums; producer warp 8: X slot wait, centre stage wait, issue.  A warp's counters sum to its whole run.
 * B2K_ERR_STATE when no profiled launch was made. */
int b2k_get_fused_profile(b2k_ctx* ctx, long long* out, int64_t cap, int* grid_out, int* warps_out);
int b2k_reset_stats(b2k_ctx* ctx);

/* ---- communicator (NCCL over NVLink; one rank per process per GPU).  libnccl is loaded at the first call: the library
 * named by the environment variable B2K_NCCL_LIB when it is set (failing to load it is B2K_ERR_NCCL), else
 * libnccl.so.2. ---- */
int b2k_comm_unique_id(char out[B2K_UNIQUE_ID_BYTES]); /* rank 0 only */
int b2k_comm_init(b2k_ctx* ctx, int nranks, int rank, const char uid[B2K_UNIQUE_ID_BYTES]);
int b2k_comm_destroy(b2k_ctx* ctx);
int b2k_comm_abort(b2k_ctx* ctx); /* callable after a CUDA/NCCL error; never blocks on peers */

/* ---- ingest: host Arrow batch -> rows [row0, row0+n_b) of the device matrix dst[n_max, d] (f32, row-major).
 * Stages through pinned memory, converts/transposes on the device (coalesced, vectorised).  Rejects a
 * non-constant row length.  *rows_written receives n_b.  Asynchronous with respect to the host except for
 * the staging copy; ordered on `stream`. ---- */
int b2k_ingest_append(b2k_ctx* ctx, float* dst, int64_t n_max, int d, int64_t row0, const void* values,
                      const int32_t* offsets, int64_t n_b, int src_dtype, int layout, uintptr_t stream,
                      int64_t* rows_written);

/* ---- sparse ingest (stands in for core.py:193-264, 507-521, the reference's CSR build from Spark vectors): one Arrow
 * batch of a Spark VectorUDT column (struct<type: tinyint, size: int, indices: array<int>, values: array<double>>),
 * given by its child buffers, appended as rows [row0, row0 + n_b) and entries [nnz0, nnz0 + nnz_b) of a device CSR
 * (indptr int64 [n_max + 1], indices int32 and values f32 [nnz_max]).  type [n_b] int8 (0 sparse, 1 dense), size [n_b]
 * int32 (read for sparse rows only), idx_offsets / val_offsets [n_b + 1] int32 and their child buffers idx_values int32
 * and val_values (B2K_F64 or B2K_F32, rounded to f32); offsets index the whole child buffers, as Arrow's do.  A dense
 * row becomes the entries 0 .. d - 1; stored zeros stay entries.  indptr[row0 + i + 1] is written for each row; the
 * caller sets indptr[0] = 0.  Errors (B2K_ERR_INVALID), as the dense ingest checks row widths: a sparse row's size or a
 * dense row's length other than d, a sparse row whose index count differs from its value count, a type other than
 * 0 / 1; these fail on the ingesting rank only.  Index range, order and finiteness are checked on the device by the
 * calls that read the rows.  Stages through the pinned buffers of
 * b2k_ingest_append; *nnz_written = nnz_b.  Ordered on `stream`. ---- */
int b2k_ingest_csr_append(b2k_ctx* ctx, int64_t* indptr, int32_t* indices, float* values, int64_t n_max,
                          int64_t nnz_max, int64_t d, int64_t row0, int64_t nnz0, const int8_t* type, const int32_t* size,
                          const int32_t* idx_offsets, const int32_t* idx_values, const int32_t* val_offsets,
                          const void* val_values, int val_dtype, int64_t n_b, uintptr_t stream, int64_t* nnz_written);

/* ---- fit: init + Lloyd loop + (optional) inertia against the final centers.
 *   X              device f32 [n_local, d] row-major (this rank's partition)
 *   init_centers   device f32 [k, d] when init_mode == B2K_INIT_ARRAY (identical on all ranks), else NULL
 *   tol            stop when sum_j ||c_j_new - c_j_old||^2 < tol; the caller maps tol==0 to float32 tiny
 *                  exactly as the reference does (clustering.py:113-123)
 *   n_init         must be 1 (the reference forces n_init=1, clustering.py:316-319)
 *   centers_out    device f32 [k, d]
 *   n_iter_out, inertia_out   host; inertia_out may be NULL (skips the extra assign pass)
 * Collective across the communicator when one is initialised: every rank must call it.  An empty partition on any
 * rank (n_local == 0, X may then be NULL) fails on every rank together. ---- */
int b2k_kmeans_fit(b2k_ctx* ctx, const float* X, int64_t n_local, int d, int k, int init_mode,
                   const float* init_centers, int max_iter, double tol, uint64_t seed, double oversampling,
                   int n_init, float* centers_out, int* n_iter_out, double* inertia_out, uintptr_t stream);

/* ---- the Lloyd loop alone, in place on device centers[k,d]: at most max_iter iterations of
 * {assign + per-cluster partial sums (one pass over X), allreduce(sum,count), finalize, convergence}.
 * shift_out (host, may be NULL) receives the last sum_j||dc_j||^2.  Collective like b2k_kmeans_fit: its sizes are
 * allgathered first, so an empty partition on any rank (n_local == 0, X may then be NULL) fails on every rank together
 * instead of running a loop whose allreduces would need every rank. ---- */
int b2k_kmeans_lloyd(b2k_ctx* ctx, const float* X, int64_t n_local, int d, int k, float* centers,
                     int max_iter, double tol, int* n_iter_out, double* shift_out, uintptr_t stream);

/* ---- assign-only (KMeansModel.transform / predict): labels_out device int32 [n]; mindist_out device f32 [n]
 * or NULL.  Ties -> lowest center index. Asynchronous on `stream`. ---- */
int b2k_kmeans_assign(b2k_ctx* ctx, const float* X, int64_t n, int d, const float* centers, int k,
                      int32_t* labels_out, float* mindist_out, uintptr_t stream);

/* ---- PCA ----
 * Shapes: 1 <= k <= d <= 1024.  The Gram pass runs on wgmma (3xTF32, fp64 partials every 4096 rows) when d % 4 == 0 and X is
 * 16-byte aligned, else on the generic SIMT kernel (fp64 products and sums); option "kernel_path" = B2K_PATH_GENERIC
 * forces the generic kernel, B2K_PATH_FUSED fails with B2K_ERR_UNSUPPORTED where the wgmma pass cannot run.  d > 1024:
 * B2K_ERR_UNSUPPORTED.
 *
 * fit: X device f32 [n_local, d] row-major.  Host f64 outputs: mean_out [d] = sum x / n_total (fp64), components_out
 * [k][d] = eigenvectors of the covariance (x - mean)^T (x - mean) / (n_total - 1) by descending eigenvalue, each signed
 * so that its largest-|value| element (lowest index on a tie) is positive; explained_variance_ratio_out [k] = lambda_i /
 * trace(covariance); singular_values_out [k] = sqrt(lambda_i (n_total - 1)).  Eigenvalues below 0 (rounding) count as 0.
 * Zero total variance (constant features) is not an error: the ratios and singular values are 0 and the components are
 * the first k unit vectors.  Errors: k < 1, k > d ("source vector size d must be no less than k"), n_total < 2, an
 * empty partition on any rank (X may then be NULL; every rank fails together).  Collective across the communicator when one is initialised; synchronises `stream`
 * before returning.  Bitwise reproducible for the same input, rank count and device. */
int b2k_pca_fit(b2k_ctx* ctx, const float* X, int64_t n_local, int d, int k, double* mean_out, double* components_out,
                double* explained_variance_ratio_out, double* singular_values_out, uintptr_t stream);
/* The eigen step of b2k_pca_fit alone, on the host (no context, no device): cov [d][d] f64 (only the upper triangle is
 * read), outputs as above.  Errors through b2k_last_error(NULL). */
int b2k_pca_finalize(const double* cov, int d, int64_t n_total, int k, double* components_out,
                     double* explained_variance_ratio_out, double* singular_values_out);
/* out [n][k] f32 = X [n][d] . components^T (components device f32 [k][d]); no mean is subtracted, as in Spark's
 * PCAModel.  fp32 accumulation in feature order.  Asynchronous on `stream`. */
int b2k_pca_transform(b2k_ctx* ctx, const float* X, int64_t n, int d, const float* components, int k, float* out,
                      uintptr_t stream);

/* ---- exact k-NN (Euclidean) ----
 * Stands in for knn.py:662-804 (NearestNeighborsModel.kneighbors' fit function: cuML NearestNeighborsMG.kneighbors
 * over NCCL, then the row -> id mapping).
 *   items      device f32 [n_items_local, d] row-major: this rank's part of the index
 *   item_ids   device int64 [n_items_local] or NULL (ids = global rows: rank 0's rows in order, then rank 1's, ...)
 *   queries    device f32 [n_queries_local, d]
 *   outputs    device [n_queries_local][k]: distances_out f32 = sqrt of the exact fp32 sum_f (q_f - x_f)^2 in feature
 *              order, ascending; indices_out int64 = ids.  Ties of the reported distance: lowest global row first.
 * Search on all ranks' items for every rank's queries.  The pass runs on wgmma (3xTF32 screening distances, exact
 * recompute of the survivors) when d % 4 == 0, 4 <= d <= 128, k <= 64 and the queries are 16-byte aligned, else on the
 * generic SIMT kernel (exact fp32 distances); k > 1024: B2K_ERR_UNSUPPORTED.  Option "kernel_path" as for PCA.
 * Errors, decided on the allgathered sizes so that every rank fails together: k < 1, k > n_items_total, no item on any
 * rank, d differing between ranks.  Ranks with no items or no queries are legal.  Collective across the communicator
 * when one is initialised (allgathers of the sizes, the queries and the candidate lists); synchronises `stream` once
 * after the size allgather.  Bitwise reproducible for the same input, rank count and device.
 * Stats: last_path = the search pass that ran; with option "time_kernels" != 0, last_finalize_ms = the index prep
 * (wgmma path), last_fused_ms = the search pass, last_reduce_ms = refine + merge, last_allreduce_ms = both allgathers,
 * last_loop_ms = the whole call after the size allgather (device times, CUDA events). */
int b2k_knn_search(b2k_ctx* ctx, const float* items, int64_t n_items_local, const int64_t* item_ids,
                   const float* queries, int64_t n_queries_local, int d, int k, float* distances_out,
                   int64_t* indices_out, uintptr_t stream);

/* ---- approximate k-NN: IVF-Flat (Euclidean) ----
 * Stands in for knn.py:1406-1692 (ApproximateNearestNeighborsModel.kneighbors, algorithm "ivfflat").  Arguments as for
 * b2k_knn_search, plus:
 *   nlist, nprobe  lists of the index and lists probed per query; nprobe is clamped to nlist
 *   n_iters, train_fraction   the Lloyd run of the coarse quantizer (train = 1)
 *   metric         B2K_IVF_EUCLIDEAN (distance) or B2K_IVF_SQEUCLIDEAN (the squared fp32 sum)
 *   centers        device f32 [nlist, d]: used as given when train = 0; with train = 1 it receives the trained centres
 *   item_list_out  device int32 [n_items_local] or NULL: the list of each local item
 *   probe_out      device int32 [n_queries_local][nprobe (clamped)] or NULL: the lists each query probes, nearest first
 *                  (-1 where a query with a NaN component probes nothing)
 * One index over all ranks' items, so that for fixed centres the result depends neither on the rank count nor on how
 * the rows are partitioned:
 *   - Training subset: global row r (rank 0's rows in order, then rank 1's, ...) is a training row when
 *     floor((r + 1) f) > floor(r f), f = train_fraction in (0, 1].  The training rows of all ranks are allgathered
 *     in global row order and every rank runs b2k_kmeans_fit on them as one rank: init B2K_INIT_RANDOM with seed
 *     B2K_IVF_SEED, max_iter = n_iters, tol = float32 tiny.  Ranks without a training row take part; the centres do not
 *     depend on the rank count.  Each rank holds (ranks + 1) x the largest rank's training rows meanwhile.
 *     nlist <= training rows.
 *   - Lists: each item goes to its nearest centre by b2k_kmeans_assign (ties to the lowest centre).
 *   - Probes: per query, the nprobe nearest centres under the exact k-NN rule (ties to the lower list).
 *   - Result: per query, the exact k-NN result of b2k_knn_search over the items of its probed lists (fp32 distance
 *     recomputed, sorted by (distance, global row)).  With nprobe = nlist it is b2k_knn_search's result.
 *   - Fewer than k items found: the remaining distances are +inf and their ids the first entry's id, or INT64_MAX when
 *     nothing was found.  A query with a NaN component finds nothing.
 * The scan runs on wgmma (3xTF32 screening, exact recompute of the survivors) under b2k_knn_search's conditions, else on
 * the generic SIMT kernel; option "kernel_path" selects the scan pass only (the build and probe steps choose their own).
 * Errors, decided on allgathered sizes and flags so that every rank fails together: those of b2k_knn_search; an item
 * with a non-finite component (B2K_ERR_INVALID); nlist < 1; nprobe < 1; nprobe > 256 after clamping
 * (B2K_ERR_UNSUPPORTED); an unknown metric.  Collective across the communicator when one is initialised; synchronises
 * `stream`.  Nothing uses atomics: bitwise reproducible for the same input, rank count and device.
 * Stats: last_path = the scan pass that ran; with option "time_kernels" != 0, last_finalize_ms = the build (subset,
 * Lloyd, assign, sort and prep), last_probe_ms = the probe selection, last_fused_ms = the scan passes, last_reduce_ms =
 * the pair sort and query gather, refine and merge, last_allreduce_ms = both allgathers, last_loop_ms = the whole call
 * after the size allgather (device times, CUDA events). */
#define B2K_IVF_SEED 20240613ULL
typedef enum b2k_ivf_metric { B2K_IVF_EUCLIDEAN = 0, B2K_IVF_SQEUCLIDEAN = 1 } b2k_ivf_metric;
int b2k_ivf_search(b2k_ctx* ctx, const float* items, int64_t n_items_local, const int64_t* item_ids,
                   const float* queries, int64_t n_queries_local, int d, int k, int nlist, int nprobe, int n_iters,
                   double train_fraction, int metric, int train, float* centers, int32_t* item_list_out,
                   int32_t* probe_out, float* distances_out, int64_t* indices_out, uintptr_t stream);

/* ---- linear regression (squared loss: OLS, ridge, lasso, elastic net) ----
 * Stands in for regression.py:546-607 (LinearRegressionMG / RidgeMG / CDMG on the standardized data, then the
 * coefficients scaled back).  Every fit needs only the centred second moments of [X | y], so one moments pass serves
 * any number of solver settings.
 *
 * moments (collective): X device f32 [n_local, d], y device f32 [n_local], 1 <= d <= 1024 (d > 1024:
 * B2K_ERR_UNSUPPORTED).  Host outputs: *n_total_out = rows over all ranks; mean_out [d + 1] = fp64 means of [X | y];
 * moments_out [d + 1][d + 1] = sum (v - mean)(v - mean)^T over the rows v = [x | y], fp64.  Column sums of X and of y,
 * then the Gram pass of PCA on X (wgmma or generic, chosen as for b2k_pca_fit, option "kernel_path" likewise) and k_xty
 * for X^T y and y^T y, all centred on the fp32 means; the host removes that offset exactly.  Errors, decided on
 * allreduced values so that every rank fails together: an empty partition on any rank (X and y may then be NULL); a NaN
 * or an infinity in X or y (B2K_ERR_INVALID).  Synchronises `stream`.  Bitwise reproducible for the same input, rank
 * count and device.  Stats: last_path = the Gram pass that ran; with option "time_kernels" != 0, last_reduce_ms = the column-sum pass,
 * last_fused_ms = the Gram pass, last_finalize_ms = the k_xty pass, last_allreduce_ms = both allreduces (device times)
 * and last_loop_ms = the whole call (host clock). */
int b2k_linreg_moments(b2k_ctx* ctx, const float* X, const float* y, int64_t n_local, int d, int64_t* n_total_out,
                       double* mean_out, double* moments_out, uintptr_t stream);
/* The solver, on the host (no context, no device), from the outputs of b2k_linreg_moments.  With mu = mean[0..d),
 * muy = mean[d], population standard deviations sigma_j = sqrt(moments[j][j] / n_total) (sigma_y likewise):
 *   centring   fit_intercept: mu, muy; else 0 and 0 (scaled, not centred)
 *   scales     standardization: s_j = sigma_j (1 where sigma_j = 0), s_y = sigma_y; else 1
 *   problem    z = (x - mu) / s, t = (y - muy) / s_y, lambda' = reg / s_y; minimise
 *              (1/2n) sum (t - z.v)^2 + lambda' (l1_ratio |v|_1 + (1 - l1_ratio)/2 |v|^2)
 *   result     coef_out [d] = v_j s_y / s_j; *intercept_out = muy - coef.mu with an intercept, else 0
 * reg == 0 or l1_ratio == 0: Cholesky of A + lambda' (1 - l1_ratio) I (A = Z^T Z / n); when a pivot is <= d 2^-52 max
 * diag, the minimum-norm solution of its eigendecomposition (eigenvalues <= d 2^-52 lambda_max count as 0); *n_iter_out
 * = 0.  Otherwise cyclic coordinate descent from v = 0 in feature order, soft-thresholding at lambda' l1_ratio, stopped
 * after a sweep with max |dv| <= tol max |v| or after max_iter sweeps; *n_iter_out = the sweeps.  A constant label under
 * standardization: coef = 0 and intercept = muy (0 without an intercept) when fit_intercept or muy == 0, else s_y = |muy|.
 * Errors (B2K_ERR_INVALID, through b2k_last_error(NULL)): reg < 0, l1_ratio outside [0, 1], max_iter < 0, tol < 0,
 * n_total < 1, non-finite inputs; d > 1024: B2K_ERR_UNSUPPORTED.  n_iter_out may be NULL. */
int b2k_linreg_solve(const double* mean, const double* moments, int d, int64_t n_total, double reg, double l1_ratio,
                     int fit_intercept, int standardization, int max_iter, double tol, double* coef_out,
                     double* intercept_out, int* n_iter_out);
/* out [n] f64 = intercept + sum_j X[i][j] coef[j] (coef device f64 [d]), accumulated in fp64 in an order fixed by d
 * alone.  Asynchronous on `stream`. */
int b2k_linreg_predict(b2k_ctx* ctx, const float* X, int64_t n, int d, const double* coef, double intercept, double* out,
                       uintptr_t stream);

/* ---- logistic regression (binomial and multinomial, L2 / L1 / elastic net, MLlib's objective) ----
 * With K' = 1 (binomial) or K (multinomial) margins per row, coefficients W [K'][d] and intercepts b [K'], the fit
 * minimises (1/n) sum_i l(W x_i + b, y_i) + reg ((1 - l1_ratio)/2 |V|^2 + l1_ratio |V|_1), where l is the logistic loss
 * max(m, 0) + log1p(exp(-|m|)) - y m (binomial) or the softmax cross-entropy (log-sum-exp with the row maximum taken
 * out), the intercepts are not penalised, and V = W diag(sigma) with standardization, else V = W.  sigma are the sample
 * (n - 1) standard deviations of the features, MLlib's convention; a feature with sigma = 0 gets a coefficient of 0.
 * Labels are the class values: integers in [0, 1024); classes = the sorted distinct label values.
 *
 * b2k_logreg_labels (collective) stands in for the class discovery of classification.py:1075-1103 (cuML's
 * LogisticRegressionMG.fit and the label checks after it).  One pass over y [n_local] (device f32) and one allgather.
 * Outputs (host): classes_out [<= 1024] f64, counts_out [<= 1024] rows per class, *n_classes_out, *n_total_out.
 * Errors, decided on the gathered values so that every rank fails together (B2K_ERR_INVALID unless noted): an empty
 * partition on any rank; a NaN or an infinity; "Labels MUST be in [0, 2147483647), but got v" (v the least label,
 * the first sorted class the reference reports); "Labels MUST be Integers, but got v"; a label
 * >= 1024 (B2K_ERR_UNSUPPORTED).  Synchronises `stream`. */
int b2k_logreg_labels(b2k_ctx* ctx, const float* y, int64_t n_local, double* classes_out, int64_t* counts_out,
                      int* n_classes_out, int64_t* n_total_out, uintptr_t stream);
/* b2k_logreg_eval (collective) stands in for one loss-and-gradient evaluation inside cuML's qn solver: the loss
 * (1/n) sum l and its gradient (no penalty) at W [kp][d], b [kp] (host f64), over X [n_local, d] and y [n_local] (device
 * f32).  classes [n_classes] are the class values (b2k_logreg_labels); a row whose label is not one of them counts as no
 * class.  kp = 1: the binomial loss with class index 1 the positive class.  Outputs (host): *loss_out, grad_out
 * [kp][d + 1] = (1/n) sum r_k x_j, then (1/n) sum r_k in column d; *n_total_out (may be NULL).  The fused pass
 * (k_logreg_eval) runs where its accumulators and its shared memory fit: a class block of KB = 1, 2, 4, 8 or 16 (the
 * least >= K', at most 16) and d * ceil(K'/KB) <= 256 NIT (NIT = 4 for KB <= 4, 2 for KB = 8, 1 for KB = 16), i.e.
 * K' <= 4 at every d <= 1024, K' <= 8 at d <= 512, K' <= 16 at d <= 256, K' <= 32 at d <= 128 and so on, while its
 * shared memory fits the device's opt-in limit (which alone bounds K' at small d); elsewhere the generic rows + X^T R
 * passes.  Option "kernel_path" as for PCA, option "grid_limit" caps the fused pass's CTAs; stats.last_path reports the
 * pass; with "time_kernels", last_fused_ms = its device time.  Errors: an empty
 * partition; d > 1024 (B2K_ERR_UNSUPPORTED).  Synchronises `stream`.  Bitwise reproducible for the same input, rank
 * count and device. */
int b2k_logreg_eval(b2k_ctx* ctx, const float* X, const float* y, int64_t n_local, int d, const double* classes,
                    int n_classes, int kp, const double* W, const double* b, double* loss_out, double* grad_out,
                    int64_t* n_total_out, uintptr_t stream);
/* Objective of b2k_logreg_minimize: the smooth part f(x) and its gradient at x [n]; nonzero return aborts the
 * minimisation with that status. */
typedef int (*b2k_logreg_objective)(void* user, int n, const double* x, double* f, double* grad);
/* b2k_logreg_minimize (host only, no device) stands in for cuML's qn solver (L-BFGS / OWL-QN): minimises f(x) + sum_i
 * l1[i] |x_i| from x [n] (in: the start, out: the result); l1 may be NULL.  L-BFGS with memory 10 and a strong-Wolfe
 * line search (c1 = 1e-4, c2 = 0.9) of at most 20 evaluations, first step 1/|d|; OWL-QN (any l1[i] > 0): the
 * pseudo-gradient, orthant-projected steps and a backtracking line search of at most 20 evaluations.  Stops on Breeze's
 * rules as MLlib applies them: iterations == max_iter; |F - max of the last 20 F| <= tol |F_0|; |pseudo-gradient| <=
 * max(tol |F|, 1e-8); or a failed line search (x keeps the last accepted iterate).  F is the value with the L1 term.
 * Outputs: *n_iter_out, *n_eval_out, *f_out (each may be NULL).  Errors through b2k_last_error(NULL): max_iter < 0,
 * tol < 0, a negative or non-finite l1 weight, a non-finite start value. */
int b2k_logreg_minimize(b2k_logreg_objective fn, void* user, int n, double* x, const double* l1, int max_iter,
                        double tol, int* n_iter_out, int* n_eval_out, double* f_out);
typedef struct b2k_logreg_params {
  double reg;              /* regParam >= 0 */
  double l1_ratio;         /* elasticNetParam in [0, 1] */
  double tol;              /* >= 0 */
  int32_t max_iter;        /* >= 0 */
  int32_t fit_intercept;   /* 0 / 1 */
  int32_t standardization; /* 0 / 1 */
  int32_t family;          /* 0 auto (binomial for 2 classes), 1 binomial, 2 multinomial */
} b2k_logreg_params;
/* b2k_logreg_fit (collective) stands in for classification.py:984-1171 (LogisticRegressionMG.fit per param map, the
 * rescaling and the intercept centring).  classes / counts / n_classes from b2k_logreg_labels.  One column-moments
 * pass (sums, then centred squares, fp64), then per setting params[f]: L-BFGS / OWL-QN through b2k_logreg_eval in the
 * solver frame theta = [V | b], intercepts started at MLlib's log-odds of the priors; then W = V / sigma, and for
 * multinomial fits the intercepts centred over the classes (with an intercept) and, when reg == 0, the coefficients
 * centred per feature.  Outputs (host), per setting f: coef_out [f][K][d] (rows past kp_out[f] zero), intercept_out
 * [f][K], kp_out[f] = K' and n_iter_out[f] = iterations.  One class (0 or 1): zero coefficients, intercept +inf (class 1)
 * or -inf, 0 iterations; another single class value is an error.  Errors (B2K_ERR_INVALID): those of the params
 * ("maxIter given invalid value -1", "C or regParam given an invalid or unsupported value -1.0", ...), "Binomial family
 * only supports 1 or 2 outcome classes but found K.", an empty partition, a NaN or an infinity in X; d > 1024:
 * B2K_ERR_UNSUPPORTED.  Synchronises `stream`; bitwise reproducible for the same input, rank count and device.
 * stats.last_n_iter = the last setting's iterations; with "time_kernels", last_loop_ms = the whole call. */
int b2k_logreg_fit(b2k_ctx* ctx, const float* X, const float* y, int64_t n_local, int d, const double* classes,
                   const int64_t* counts, int n_classes, int n_fits, const b2k_logreg_params* params, double* coef_out,
                   double* intercept_out, int* kp_out, int* n_iter_out, uintptr_t stream);
/* b2k_logreg_predict stands in for classification.py:1455-1553 (LogisticRegressionModel's transform): margins m = W x +
 * b in fp64 (W device f64 [kp][d], b device f64 [kp]); with nout = 2 for kp = 1, else kp: raw_out [n][nout] = [-m, m]
 * or the margins, prob_out [n][nout] = [1 - s, s] (s the sigmoid) or the softmax, pred_out [n] = class_values[argmax]
 * (class_values device f64 [nout]; binomial: m > 0).  Asynchronous on `stream`. */
int b2k_logreg_predict(b2k_ctx* ctx, const float* X, int64_t n, int d, int kp, const double* W, const double* b,
                       const double* class_values, double* raw_out, double* prob_out, double* pred_out,
                       uintptr_t stream);

/* ---- sparse logistic regression: the objective, classes, label rules, optimiser, stopping rules, start and centring of
 * b2k_logreg_fit, over rows in CSR: indptr [n_local + 1] int64 (indptr[0] = 0, indptr[n_local] = nnz_local), indices
 * [nnz] int32, values [nnz] f32 (device); y [n_local] f32.  sigma counts the implicit zeros (sample deviations over all n
 * rows); standardization scales and never centres, so a CSR fit and a dense fit of the same matrix solve the same
 * problem and differ only by summation order.  All arithmetic fp64.  Caps (B2K_ERR_UNSUPPORTED): d < 2^31 and
 * kp (d + 1) <= 2^25 (the host L-BFGS state holds about 20 vectors of that length).  Collective errors (every rank fails
 * together, B2K_ERR_INVALID): an empty partition; "sparse features: an index is out of bounds for vectors of size d";
 * "sparse features: the indices of a row must be strictly increasing"; "logistic regression: the features hold a NaN
 * or an infinity".  The CSC copy is built once per call: rows are split into chunks whose residuals R [rows][kp] fp64
 * stay under 256 MB, each chunk sorted by column with a stable radix sort.  One evaluation = per chunk a rows pass
 * (margins, residuals, loss) and a CSC pass over fixed ranges of entries (columns cut at range boundaries are carried
 * and folded in range order), then one f64 allreduce.  No floating-point atomics: bitwise reproducible for the same
 * input, rank count, device and option "grid_limit" (which caps the rows pass's CTAs).  stats.generic_launches counts
 * the evaluations (+1 each, whatever the number of row chunks).  With "time_kernels":
 * last_fused_ms = the rows passes, last_reduce_ms = the CSC passes, last_allreduce_ms = the allreduce and read-back of
 * the last evaluation; last_finalize_ms = the CSC build, last_probe_ms = the moments pass (fit), last_loop_ms = the whole
 * fit.  Synchronise `stream`.
 *
 * b2k_logreg_eval_csr (collective) stands in for one evaluation of cuML's qn solver on the reference's CSR input
 * (classification.py:1038-1060): outputs as b2k_logreg_eval (grad_out [kp][d + 1]); builds its own CSC (for tests and
 * diagnostics).  b2k_logreg_fit_csr (collective) stands in for classification.py:998-1171 on sparse rows: outputs as
 * b2k_logreg_fit; the CSC, the validation and the moments pass (sum x and nnz per column, one allreduce, then
 * sum over the entries of (x - mu)^2 plus (n - nnz) mu^2, a second allreduce) serve all n_fits settings. */
int b2k_logreg_eval_csr(b2k_ctx* ctx, const int64_t* indptr, const int32_t* indices, const float* values,
                        int64_t n_local, int64_t nnz_local, int64_t d, const float* y, const double* classes,
                        int n_classes, int kp, const double* W, const double* b, double* loss_out, double* grad_out,
                        int64_t* n_total_out, uintptr_t stream);
int b2k_logreg_fit_csr(b2k_ctx* ctx, const int64_t* indptr, const int32_t* indices, const float* values,
                       int64_t n_local, int64_t nnz_local, int64_t d, const float* y, const double* classes,
                       const int64_t* counts, int n_classes, int n_fits, const b2k_logreg_params* params,
                       double* coef_out, double* intercept_out, int* kp_out, int* n_iter_out, uintptr_t stream);
/* b2k_logreg_predict_csr stands in for classification.py:1455-1553 on sparse rows: the outputs of b2k_logreg_predict
 * (W device f64 [kp][d], b, class_values as there) for n CSR rows, margins summed in fp64 by the rows pass's code.  The
 * caps and the index / order / finiteness checks above apply (not collective).  Synchronises `stream` when it checks. */
int b2k_logreg_predict_csr(b2k_ctx* ctx, const int64_t* indptr, const int32_t* indices, const float* values, int64_t n,
                           int64_t nnz, int64_t d, int kp, const double* W, const double* b, const double* class_values,
                           double* raw_out, double* prob_out, double* pred_out, uintptr_t stream);

/* ---- DBSCAN (euclidean or cosine) ----
 * Stands in for clustering.py:1049-1186 (DBSCANModel's fit function: cuML DBSCANMG.fit_predict).  Semantics, with the
 * rows in global order (rank 0's rows in order, then rank 1's, ...):
 *   adjacency  rows i and j are adjacent when dist(i, j) <= eps, evaluated in fp64 from the float32 values:
 *              metric 0 (euclidean): sum_f ((double)x_if - (double)x_jf)^2 <= eps^2 (eps^2 formed in fp64);
 *              metric 1 (cosine):    1 - x_i.x_j / (|x_i| |x_j|) <= eps, |x| = sqrt(sum_f x_f^2), all in fp64;
 *              every sum in feature order, every operation rounded once (no fused multiply-add).  A row is adjacent to
 *              itself.
 *   core       a row with >= min_samples adjacent rows, itself included.
 *   clusters   the connected components of the graph of core rows, numbered 0..C-1 by their lowest global row.
 *   border     a non-core row with an adjacent core row takes the cluster of the adjacent core row of lowest global row
 *              (order-free; scikit-learn's expansion order can give a row that touches two clusters the other one).
 *   noise      every other row: -1.
 * Outputs (device, this rank's rows): labels_out int32 [n_local], core_out uint8 [n_local] (may be NULL); host:
 * *n_clusters_out = C.  Every rank ends up holding all rows (allgather of X padded to the largest shard: n_total d 4
 * bytes, plus 2 n_total DP 4 bytes of tf32 planes on the wgmma pass, DP = 32, 64 or 128), one parent array per rank of
 * the others (nranks n_total 4 bytes) and n_total bytes of core flags.
 * Passes: a count pass, then a union pass over core columns (lock-free union-find, lowest root wins).  They run on
 * wgmma (3xTF32 screen with a proven error bound, pairs inside the bound decided by the fp64 rule) when d % 4 == 0,
 * 4 <= d <= 128 and X is 16-byte aligned, else on the generic SIMT pass (the fp64 rule on every pair).  Options
 * "kernel_path" and "grid_limit" as for b2k_knn_search.
 * Errors, decided on allgathered values so that every rank fails together (B2K_ERR_INVALID unless noted): eps not
 * finite or <= 0; min_samples < 1; metric not 0 or 1; no row on any rank; d differing between ranks; "DBSCAN input
 * contains NaN or infinity"; cosine with a zero row; 2^31 - 256 rows or more (B2K_ERR_UNSUPPORTED).  A rank with no rows
 * is legal (X and labels_out may then be NULL).  Collective; synchronises `stream`.  The labels and core flags depend
 * only on the rows in global order: not on the rank count, the shard boundaries, the pass or the order of atomics.
 * Stats: last_path = the pass that ran; with option "time_kernels" != 0, last_finalize_ms = row allgather and prep,
 * last_fused_ms = the count pass, last_reduce_ms = core allgather and the union pass, last_allreduce_ms = merge and
 * labels, last_loop_ms = all of them (device times, CUDA events); with option "collect_recheck" = 1,
 * recheck_candidates = pairs of the wgmma pass decided by the fp64 rule and recheck_rows = unions attempted. */
int b2k_dbscan_fit(b2k_ctx* ctx, const float* X, int64_t n_local, int d, double eps, int min_samples, int metric,
                   int32_t* labels_out, uint8_t* core_out, int64_t* n_clusters_out, uintptr_t stream);

/* ---- random forests (classification: gini / entropy; regression: variance) ----
 * Stands in for tree.py / classification.py:285-676 / regression.py:865-1147 (cuML's RandomForest*MG fits on each
 * worker's partition).  Unlike the reference, every tree is grown from the histograms of ALL ranks' rows, level by
 * level, with one int64 allreduce per histogram pass (MLlib's design), so the forest depends only on the rows in global
 * order (rank 0's rows, then rank 1's, ...) and the params: not on the rank count, the shard boundaries, the pass or the
 * order of atomics.  Semantics (tests/rf_oracle.py restates them in NumPy):
 *   hash       h(seed, stream, tree, index), SplitMix64's finaliser chained (below); streams B2K_RF_BOOT,
 *              B2K_RF_SAMPLE, B2K_RF_FEAT.
 *   bootstrap  bootstrap = 1: row r of tree t has weight w = Poisson(1) drawn by inverse CDF from u = h(seed, BOOT, t,
 *              r) >> 32 against B2K_RF_POISSON_CDF (below), capped at 12; else w = 1.  Every statistic is an integer
 *              sum of w.
 *   thresholds row r is in the sample iff h(seed, SAMPLE, 0, r) < (uint64)ldexp(f, 64), f = M / n_total with M =
 *              max(max_bins^2, 10000) (every row when M >= n_total).  Per feature, the sample values (-0.0 read as +0.0)
 *              sorted: s_0 <= ... <= s_{m-1}, distinct values v_0 < ... < v_{u-1}.  mid(a, b) = fl32(((double)a +
 *              (double)b) / 2), replaced by a when it equals b.  u <= max_bins: thresholds mid(v_i, v_{i+1}), i < u - 1;
 *              else mid(s_{p-1}, s_p) at p = floor(j m / max_bins), j = 1..max_bins-1, duplicates dropped.  A feature has
 *              nthr <= max_bins - 1 ascending thresholds t_0 < t_1 < ... and nthr + 1 bins; bin(x) = #{thresholds < x}
 *              in float32, so x <= t_b <=> bin(x) <= b: training routes rows by bin, prediction by threshold, alike.
 *   features   each node draws features_per_node features of d: a partial Fisher-Yates shuffle of 0..d-1 whose step j
 *              swaps slot j with slot j + h(seed, FEAT, t, heap d + j) % (d - j), heap the node's heap index (root 1,
 *              children 2 heap and 2 heap + 1); the first features_per_node slots, sorted ascending.
 *   statistics classification: per class c_k = sum w (N = sum_k c_k).  Regression: labels on a fixed-point grid, y_q =
 *              rint(y 2^(24-e)) with 2^(e-1) < max|y| <= 2^e over all ranks (q = 2^(e-24); q = 1 when max|y| = 0), so
 *              that W = sum w and S = sum w y_q are exact integers: labels are resolved to max|y| 2^-24, a deliberate
 *              semantic.
 *   gain       fp64, each operation rounded once (no fused multiply-add), in this order:
 *                gini     s = 0; s = s + p_k p_k over k ascending (p_k = c_k / N); imp = 1 - s
 *                entropy  s = 0; s = s - p_k L(p_k) over k ascending with c_k > 0; imp = s, where L = b2k_rf_log2 below
 *                         (written in + - * / only, so the host and NumPy agree bit for bit)
 *                gain     a = N_L / N; b = N_R / N; g = (imp - a imp_L) - b imp_R
 *                variance D = S_L W - S W_L (exact, 128-bit); g = (double)D; g = g g; g = g / (W_L W_R); g = g / W;
 *                         g = g / W; g = g q^2   (= the variance reduction of y; the sum of y^2 cancels)
 *              A candidate (feature, bin b: left = bin <= b) is valid when both sides weigh >= min_instances.  The best
 *              has the highest gain; ties go to the lowest feature, then the lowest bin.  A node is a leaf when its
 *              depth is max_depth, it is pure (one class; classification), it has no valid candidate, or the best gain
 *              is <= 0 or below min_info_gain (MLlib's rule).
 *   values     classification: c_k / N for k < n_values (n_values = max label + 1); regression: ((double)S q) / W.  A
 *              node of weight 0 (a root whose bootstrap drew no row) has value 0.  Every node carries its value.
 *   numbering  per tree, breadth first: the root is node 0; the nodes of one level, in order, append their children
 *              (left, then right).
 * b2k_rf_fit (collective): X device f32 [n_local, d], y device f32 [n_local] (class values 0, 1, ... or targets).
 * Histograms hold (tree, node, feature slot, bin) x {c_0..c_{C-1} | W, S} of the nodes of one level.  Passes: a finite
 * check and an allgather of the sizes; the label pass of b2k_logreg_labels (classification; its label rules apply); the
 * sample select and an allgather of the sample; the host sort and thresholds; k_rf_bin (X -> uint8 bins, n_local d
 * bytes); per level and node group, one histogram pass, one int64 allreduce, the host split choice, then k_rf_route.
 * The histogram pass runs on an 8-CTA thread-block cluster that shards the group's histogram over its CTAs' shared
 * memory (u32 counts, u64 label sums, remote shared atomics, flushed with int64 global atomics at least every
 * 2^28 rows per cluster, option "rf_flush_tiles" lowers that for tests); node groups are sized to the cluster's shared
 * memory.  Where one node's histogram exceeds it, the generic pass adds every update with int64 global atomics.  Option
 * "kernel_path" = B2K_PATH_GENERIC forces the generic pass, B2K_PATH_FUSED fails with B2K_ERR_UNSUPPORTED where the
 * cluster pass cannot run; option "grid_limit" caps the CTAs; option "rf_group_nodes" caps the nodes of one group.
 * Outputs: *n_values_out = C (classification) or 1; *n_nodes_out = nodes of the forest, read with b2k_rf_forest;
 * level_ms_out [max_depth + 1] (may be NULL; needs "time_kernels") = device time of each level's histogram passes;
 * level_updates_out [max_depth + 1] (may be NULL) = (row, tree, feature slot) updates with w > 0 of each level, all
 * ranks.  Errors, decided on gathered values so that every rank fails together (B2K_ERR_INVALID unless noted):
 * "maxDepth given invalid value -1", "maxBins given invalid value -1" (max_bins outside [2, 256]), n_trees < 1,
 * min_instances < 1, min_info_gain < 0 or not finite, features_per_node outside [1, d], impurity outside 0..2, max_depth
 * > 16 (B2K_ERR_UNSUPPORTED), an empty partition on any rank, d differing between ranks, "RandomForest input contains NaN
 * or infinity", and the label rules of b2k_logreg_labels (classification).  Synchronises `stream`.
 * Stats: last_path = the histogram pass that ran; last_n_iter = levels; recheck_rows = histogram passes;
 * recheck_candidates = bytes allreduced by them; with "time_kernels": last_finalize_ms = checks, labels, sample, sort
 * and thresholds (host clock), last_reduce_ms = k_rf_bin, last_fused_ms = every histogram pass, last_allreduce_ms =
 * their allreduces (device times), last_loop_ms = the whole call (host clock). */
#define B2K_RF_MAX_DEPTH 16
#define B2K_RF_MAX_BINS 256
#define B2K_RF_BOOT 1
#define B2K_RF_SAMPLE 2
#define B2K_RF_FEAT 3
#define B2K_RF_POISSON_CAP 12
/* The hash, in uint64 wrap-around arithmetic, with G = B2K_RF_GOLDEN:
 *   mix(z)                           z ^= z >> 30; z *= B2K_RF_MIX1; z ^= z >> 27; z *= B2K_RF_MIX2; z ^= z >> 31
 *   h(seed, stream, tree, index)   = mix(mix(mix(seed + stream G) + tree G) + index G)
 * The bootstrap weight of u (the top 32 bits of h) is the least k with u < B2K_RF_POISSON_CDF[k] (floor(2^32 CDF(k))
 * of Poisson(1), k = 0..11), else B2K_RF_POISSON_CAP. */
#define B2K_RF_GOLDEN 0x9E3779B97F4A7C15ull
#define B2K_RF_MIX1 0xBF58476D1CE4E5B9ull
#define B2K_RF_MIX2 0x94D049BB133111EBull
#define B2K_RF_POISSON_CDF                                                                                         \
  {1580030168u, 3160060337u, 3950075421u, 4213413783u, 4279248373u, 4292415291u, 4294609777u, 4294923276u,         \
   4294962463u, 4294966817u, 4294967252u, 4294967292u}
typedef struct b2k_rf_params {
  int32_t n_trees;           /* >= 1 */
  int32_t max_depth;         /* 0..16 */
  int32_t max_bins;          /* 2..256 */
  int32_t min_instances;     /* >= 1 (minInstancesPerNode, in bootstrap weight) */
  int32_t features_per_node; /* 1..d (featureSubsetStrategy resolved by the caller) */
  int32_t bootstrap;         /* 0 / 1 */
  int32_t impurity;          /* 0 gini, 1 entropy (classification); 2 variance (regression) */
  int32_t reserved;          /* 0 */
  double min_info_gain;      /* >= 0 */
  uint64_t seed;
} b2k_rf_params;
int b2k_rf_fit(b2k_ctx* ctx, const float* X, const float* y, int64_t n_local, int d, const b2k_rf_params* params,
               int* n_values_out, int64_t* n_nodes_out, double* level_ms_out, int64_t* level_updates_out,
               uintptr_t stream);
/* The forest of the context's last successful b2k_rf_fit, host outputs (V = *n_values_out): tree_offsets_out [T + 1]
 * (tree t is nodes [off_t, off_t+1)); per node: feature_out (-1 for a leaf), threshold_out (go left when x <= t),
 * children_out [2] (tree-local indices, -1 for a leaf), gain_out (0 for a leaf), count_out (N or W), value_out [V]. */
int b2k_rf_forest(b2k_ctx* ctx, int64_t* tree_offsets_out, int32_t* feature_out, float* threshold_out,
                  int32_t* children_out, double* gain_out, int64_t* count_out, double* value_out);
/* Prediction (k_rf_predict) over X [n, d] with a forest in device arrays laid out as b2k_rf_forest's output (any
 * tree-local child indices; nodes staged in shared memory when the forest fits, else read through L1/L2).
 * classification = 1: raw_out [n][V] = sum of the leaves' values in tree order (fp64), prob_out [n][V] = raw / sum_k raw
 * (0 when that sum is 0), pred_out [n] = argmax_k raw (lowest k on a tie).  classification = 0: pred_out [n] = sum of
 * the leaves' values in tree order / T; raw_out and prob_out unused (may be NULL).  Asynchronous on `stream`. */
int b2k_rf_predict(b2k_ctx* ctx, const float* X, int64_t n, int d, int n_trees, const int64_t* tree_offsets,
                   const int32_t* feature, const float* threshold, const int32_t* children, const double* value,
                   int n_values, int classification, double* raw_out, double* prob_out, double* pred_out,
                   uintptr_t stream);
/* L(p) of the entropy above, p in (0, 1]: p = m 2^E (frexp; m < 0.7071067811865476: m = 2m, E = E - 1), z = (m - 1)
 * / (m + 1), z2 = z z, a = 1.0 / 25; a = a z2 + 1.0 / (2i + 1) for i = 11..0; L = ((z a) 2) 1.4426950408889634 + E. */

/* ---- evaluation (b2k_eval.cu): M models scored on one validation set in one read of X ----
 * Replaces the reference's multi-model transform-and-evaluate loop (python core.py:1572-1693, classification.py:161-282),
 * which reads X once per model per batch and hands every row's outputs to the host metric code.  Here a CTA stages a
 * tile of rows of X [n, d] (device f32, row-major) and y [n] (device f32) in shared memory and evaluates every model from
 * it, so X is read from HBM once per call, whatever M is, unless the models' accumulators exceed one CTA's shared memory
 * (at most 32 models, or fewer for large n_classes, per chunk); the call then splits the models into chunks, one read of
 * X each, with the same results.
 * Each model's per-row prediction has exactly the bits its own predict entry point writes (b2k_linreg_predict,
 * b2k_logreg_predict, b2k_rf_predict): the per-row code is one definition, shared.
 * Classification (n_classes = C = 1 + max(the largest label, the largest class value a model can predict); the labels
 * must follow b2k_logreg_labels' rule and its messages: integers in [0, 1024); n == 0 gives C from the models alone):
 *   label_count_out [C]  rows per label value
 *   tp_out [M][C]        rows whose prediction equals their label, by label
 *   fp_out [M][C]        rows whose prediction differs from their label, by the predicted class value
 *   loss_out [M]         sum over rows of -log(max(p_y, eps)) in fp64, p_y = the model's probability vector at index y
 *                        (as the probability column transform() writes it; 0 when y is past its end)
 * Regression: reg_out [M][3][5], for the columns (label, label - prediction, prediction) in fp64:
 *   {count, mean, m2n = sum (x - mean)^2, m2 = sum x^2, l1 = sum |x|}.  Per tile, mean and m2n are formed about the
 *   tile's mean; tiles, then CTAs in CTA order, merge by Chan's update (n = na + nb, delta = mb - ma, mean = ma + delta
 *   nb / n, m2n = m2n_a + m2n_b + delta^2 na nb / n), so a label with a large offset keeps its precision.
 * Integer counts are summed with atomics (exact, order-free); fp64 sums use per-CTA partials folded in CTA order.  The
 * grid depends on the device, the shape and option "grid_limit" alone: two calls on the same input give the same bits.
 * n == 0 is legal and gives zero accumulators.  The work runs on `stream`; the call returns once the accumulators are
 * copied to the host (it synchronises `stream`). */
#define B2K_EVAL_IDENTITY 0 /* linear regression: b + x . w */
#define B2K_EVAL_LOGISTIC 1 /* binomial logistic regression (one row of W; class values [2]) */
#define B2K_EVAL_SOFTMAX 2  /* multinomial logistic regression (K' >= 2 rows of W; class values [K']) */
#define B2K_EVAL_REG_COLS 3
#define B2K_EVAL_REG_STATS 5
/* M linear models, all identity (regression) or all logistic / softmax (classification, mixed K' allowed).  Host
 * arrays: kind [M]; row_offsets [M + 1] (model i owns rows row_offsets[i] .. row_offsets[i + 1] - 1 of W and b,
 * row_offsets[0] = 0); W [rows][d] fp64; b [rows] fp64; class_values (classification) = per model, in order, the class
 * value of each prediction index (2 for logistic, K' for softmax: prediction = class_values[argmax]).  d <= 1024. */
int b2k_eval_linear(b2k_ctx* ctx, const float* X, const float* y, int64_t n, int d, int n_models, const int32_t* kind,
                    const int32_t* row_offsets, const double* W, const double* b, const double* class_values,
                    int n_classes, double eps, int64_t* label_count_out, int64_t* tp_out, int64_t* fp_out,
                    double* loss_out, double* reg_out, uintptr_t stream);
/* M forests in b2k_rf_predict's layout, concatenated, host arrays: n_trees [M], n_values [M] (V; 1 for regression),
 * tree_offsets [sum (T_i + 1)] (each forest's own offsets, starting at 0), then per node, all forests' nodes in order:
 * feature, threshold, children [2] (tree-local) and value [V_i].  Forests may differ in trees, depth and bins.
 * classification = 1: prediction = argmax of the summed leaf values, p = raw / sum raw (as b2k_rf_predict). */
int b2k_eval_forest(b2k_ctx* ctx, const float* X, const float* y, int64_t n, int d, int n_models, int classification,
                    const int32_t* n_trees, const int32_t* n_values, const int64_t* tree_offsets,
                    const int32_t* feature, const float* threshold, const int32_t* children, const double* value,
                    int n_classes, double eps, int64_t* label_count_out, int64_t* tp_out, int64_t* fp_out,
                    double* loss_out, double* reg_out, uintptr_t stream);

/* ---- binary evaluation (b2k_eval.cu scores, b2k_binary.cu curve): areaUnderROC / areaUnderPR of M models ----
 * Semantics: Spark's BinaryClassificationEvaluator / BinaryClassificationMetrics with unit weights
 * (tests/binary_oracle.py restates them in fp64 NumPy):
 *   score    element 1 of the model's rawPrediction; a row is positive when its label > 0.5, else negative.
 *   curve    the rows grouped by distinct score in descending order, in the order of Java's Double.compare (-0.0 below
 *            +0.0; NaN one value, above +inf); each distinct score carries its (positives, negatives).  numBins > 0
 *            with D distinct scores: g = D / numBins (integer division); when g >= 2, each run of g consecutive distinct
 *            scores is one point (the last run may be shorter), else every distinct score is a point.  Spark groups per
 *            partition of its sorted RDD; here the whole ordered list is one partition.  Cumulative counts give each
 *            point's TP and FP; P and N are the totals.
 *   ROC      (0, 0), then (FPR, TPR) = (FP / N, TP / P) per point, then (1, 1).
 *   PR       (0, precision of the first point), then (recall, precision) = (TP / P, TP / (TP + FP)) per point.
 *   area     the sum of the trapezoids (x1 - x0) (y1 + y0) / 2 over consecutive points, fp64.
 *   guards   FPR = 0 when N = 0, recall = TPR = 0 when P = 0, precision = 1 when TP + FP = 0: the rules of Spark's
 *            FalsePositiveRate, Recall and Precision in BinaryClassificationMetricComputers.  So a single-class set has
 *            areaUnderROC 0 (all negative) or 1 (all positive), and areaUnderPR 0 (all negative) or 1 (all positive).
 *            These guards are the one point of this statement not yet checked against Spark's sources.
 * The score passes stage tiles of X [n, d] and y [n] (device f32) as b2k_eval_linear / b2k_eval_forest do, and write
 * each model's score of row r to scores[i * ld_scores + r] (device f64) with the bits its own predict entry point writes
 * at rawPrediction[r][1], and pos[r] = y[r] > 0.5 (device u8; may be NULL).  y must be finite.  Both return after
 * enqueueing the pass on `stream` (the label check synchronises it first).  Models as b2k_eval_linear takes them, all of
 * kind B2K_EVAL_LOGISTIC or B2K_EVAL_SOFTMAX (class values are not needed) ... */
int b2k_eval_linear_scores(b2k_ctx* ctx, const float* X, const float* y, int64_t n, int d, int n_models,
                           const int32_t* kind, const int32_t* row_offsets, const double* W, const double* b,
                           double* scores, int64_t ld_scores, uint8_t* pos, uintptr_t stream);
/* ... and forests as b2k_eval_forest takes them, classification, each with n_values >= 2. */
int b2k_eval_forest_scores(b2k_ctx* ctx, const float* X, const float* y, int64_t n, int d, int n_models,
                           const int32_t* n_trees, const int32_t* n_values, const int64_t* tree_offsets,
                           const int32_t* feature, const float* threshold, const int32_t* children,
                           const double* value, double* scores, int64_t ld_scores, uint8_t* pos, uintptr_t stream);
/* out [M] (host) = the metric of each model from scores [M][n] and pos [n] (device), 1 <= n < 2^31, num_bins >= 0.  Per
 * model: a radix sort of (score key, label bit), integer scans for the distinct scores and positives, then the
 * trapezoids, whose fp64 partials fold in a fixed order.  No atomics: two calls on the same input give the same bits.
 * Device memory of about 50 n bytes is allocated for the call.  Synchronises `stream`. */
#define B2K_BINARY_ROC 0
#define B2K_BINARY_PR 1
int b2k_eval_binary(b2k_ctx* ctx, const double* scores, const uint8_t* pos, int64_t n, int n_models, int num_bins,
                    int metric, double* out, uintptr_t stream);

/* ---- silhouette (b2k_silhouette.cu): Spark's ClusteringEvaluator, metricName "silhouette" ----
 * b2k_silhouette is the one-model case of b2k_silhouette_multi below: the same passes with n_models = 1, and its errors
 * without the "model 0: " prefix.  No reference interface: Spark computes it in closed form (ClusteringEvaluator /
 * SquaredEuclideanSilhouette / CosineSilhouette); tests/silhouette_oracle.py restates the rule in fp64 NumPy.  X device
 * f32 [n_local][d] (this rank's rows), cluster_ids device int64 [n_local] (any values; -1 is a cluster like any other),
 * metric 0 squaredEuclidean or 1 cosine; *out (host) = the metric.  Rule, over the rows of all ranks (n rows, clusters =
 * the distinct ids):
 *   rows     y = x (metric 0), or y = fl32(x / |x|) with |x| = sqrt of the feature-order fp64 sum of squares (metric 1,
 *            DBSCAN's rule), so that ||y_i - y_j||^2 = 2 (1 - cos) up to the rounding of y.
 *   D(i, c)  = the mean of ||y_i - y_j||^2 over the members j of cluster c (all of them) = ||y_i - mu_c||^2 + Psi_c, mu_c
 *            the mean of c's rows and Psi_c = sum_{j in c} ||y_j - mu_c||^2 / N_c.
 *   s_i      row i in cluster A: 0 if N_A = 1; else a = D(i, A) N_A / (N_A - 1), b = min_{c != A} D(i, c), s_i = 1 - a/b
 *            (a < b), b/a - 1 (a > b), 0 (a = b).  The metric is sum_i s_i / n.  (Cosine's s equals Spark's: the
 *            factor 2 cancels in a / b.)  = scikit-learn's silhouette_score, metric "sqeuclidean" or "cosine".
 * Spark forms D as ||x||^2 + sum ||y||^2 / N - 2 x.sum y / N, which cancels on offset data; here D is formed in a frame
 * shifted by the global mean (wgmma) or as a sum of fp64 squared differences (generic).
 * Passes: the cluster ids (per-rank CUB sort-unique, allgather of the counts and values, host merge; K <= 65536), one
 * statistics pass over X (fp64 per-cluster sums of y and ||y||^2, fixed-order folds, one f64 allreduce of K (d + 2) + 2
 * values), then the silhouette pass: wgmma (3xTF32 products of the tile rows y - m with the shifted means fl32(mu_c - m),
 * m = fl32(the global mean of y)) when d % 4 == 0, 4 <= d <= 128 and X is 16-byte aligned on every rank, else the
 * generic SIMT pass (fp64).  Option "kernel_path" = B2K_PATH_GENERIC forces the generic pass, B2K_PATH_FUSED fails with
 * B2K_ERR_UNSUPPORTED where wgmma cannot run; option "grid_limit" caps the CTAs of the silhouette pass.
 * Error bound (wgmma; the generic pass is inside it too): u = 2^-24, nb = 3 ceil(d / 8), N_ic = ||y_i - m||^2 +
 * ||mu_c - m||^2.  The fp32 screen of b2k_dbscan_fit (norms, split, wgmma model, epilogue, shift) gives
 * (23.02 + 36.08 (1 + nb)) u N_ic for ||y'_i - mu'_c||^2; the rounding of mu'_c = fl32(mu_c - m) is inside its shift term,
 * and the fp32 add of fl32(Psi_c) costs 2 u (3.1 N_ic + Psi_c).  Psi_c in fp64 (sums over at most L_c = 256 + d + N_c +
 * 8 sequential adds per term): |dPsi_c| <= (3 L_c + d + 6) 2^-53 Q_c / N_c, Q_c = sum ||y||^2 over c.  Cosine adds 8.1 u
 * (the rounding of y).  So |D~ - D| <= delta(i, c) = (31.3 + 36.08 (1 + nb)) u N_ic + 2.01 u Psi_c + |dPsi_c| (+ 8.1 u).
 * With da = delta(i, A) N_A / (N_A - 1) and db = max_{c != A} delta(i, c), s_i lies in [s(a + da, b - db), s(a - da,
 * b + db)] (s falls with a and rises with b; arguments clamp at 0); the metric is within beta = the mean of the
 * half-widths (+ (n + 8) 2^-53) of the exact value.
 * Errors, decided on allgathered or allreduced values so that every rank fails together (B2K_ERR_INVALID unless noted):
 * metric not 0 or 1; no row on any rank; d differing between ranks; "Number of clusters must be greater than one." (fewer
 * than 2 distinct ids); more than 65536 distinct ids (B2K_ERR_UNSUPPORTED); a NaN or infinite feature; cosine with a
 * zero row.  A rank with no rows takes part (X and cluster_ids may then be NULL).  Collective; synchronises `stream`.
 * Deterministic: no floating-point atomics, every fp64 sum in a fixed order, so two calls with the same input, rank
 * count and device give the same bits, and every rank gets the same value.
 * Stats: last_path = the silhouette pass that ran; with option "time_kernels" != 0, last_finalize_ms = the cluster ids,
 * last_reduce_ms = the statistics pass, its allreduce and the means, last_fused_ms = the silhouette pass (with the
 * means' planes), last_allreduce_ms = the final allreduce, last_loop_ms = the whole call (device times, CUDA events). */
#define B2K_SILHOUETTE_MAX_CLUSTERS 65536
int b2k_silhouette(b2k_ctx* ctx, const float* X, int64_t n_local, int d, const int64_t* cluster_ids, int metric,
                   double* out, uintptr_t stream);
/* b2k_silhouette_multi: the silhouette of n_models >= 1 clusterings of the same rows in one call.  cluster_ids is a host
 * array of n_models device int64 [n_local] arrays; out (host) [n_models].  A model's bits do not depend on which models
 * share the call: out[m] has exactly the bits that b2k_silhouette(ctx, X, n_local, d, cluster_ids[m], metric, ...)
 * returns, for any rank count, grid_limit and kernel_path.
 * Per model: the ids and statistics passes of b2k_silhouette and its shift m.  Models whose m has the same bits form a
 * shift group; a group's shifted means are packed one model after another into shared blocks of 128 (wgmma) or tiles
 * of 64 (generic), and one silhouette pass per chunk of at most B2K_SILHOUETTE_MULTI_CHUNK models scores all of them in
 * one read of X.  Stats: fused_tc_launches / generic_launches grow by one per (group, chunk); with "time_kernels",
 * last_finalize_ms / last_reduce_ms / last_fused_ms are the ids, statistics and silhouette passes summed over models
 * and groups.  Errors: those of b2k_silhouette, prefixed with "model m: " for the first model that fails (every rank
 * fails together); n_models < 1 is B2K_ERR_INVALID.  Collective; synchronises `stream`. */
#define B2K_SILHOUETTE_MULTI_CHUNK 16
int b2k_silhouette_multi(b2k_ctx* ctx, const float* X, int64_t n_local, int d, int n_models,
                         const int64_t* const* cluster_ids, int metric, double* out, uintptr_t stream);

/* ---- UMAP (euclidean) ----
 * b2k_umap_fit stands in for umap.py:1009-1065 (the fit function: cuML UMAP(...).fit on the rows coalesced to one
 * partition), b2k_umap_transform for umap.py:1449-1551 (UMAPModel's transform: cuML UMAP.transform against the model's
 * raw data and embedding).  Both run on one GPU and make no collective call.
 * Semantics (McInnes, Healy & Melville 2018; tests/umap_oracle.py restates each step in fp64 NumPy):
 *   kNN        exact Euclidean k-NN of the rows against themselves, k = n_neighbors (1 <= k <= n), ties to the lower row;
 *              the row itself is recognised by its index.
 *   membership per row, fp64: rho = the local_connectivity-th non-zero distance (interpolated for a fraction; the
 *              largest when fewer); sigma by 64 bisection steps on sum_{j != self} exp(-max(0, d_j - rho) / sigma)
 *              = log2(k), tolerance 1e-5, floored at 1e-3 times the row's mean distance (rho > 0) or the mean of all
 *              distances (rho == 0); w_ij = exp(-max(0, d_ij - rho_i) / sigma_i), 1 at or below rho, 0 for the self edge.
 *   graph      W = mix (P + P^T - P o P^T) + (1 - mix) P o P^T, mix = set_op_mix_ratio: CSR, columns ascending, no zeros.
 *   labels     (optional int32 [n], -1 unknown) w_ij *= exp(-1) if either label is unknown, exp(-5) if they differ; each
 *              row divided by its largest weight; then W = W + W^T - W o W^T.
 *   schedule   edges with w < max(w) / n_epochs never fire; epochs_per_sample = max(w) / w, per negative sample that
 *              over negative_sample_rate, state in fp64.
 *   init       0: uniform [-10, 10] from umap_hash; 1: the n_components leading non-trivial eigenvectors of
 *              D^-1/2 W D^-1/2 (block subspace iteration, SpMM on the device, fp64 Rayleigh-Ritz on the host), scaled
 *              to max |.| = 10 plus N(0, 1e-4) noise, or 0 when the graph has more than one connected component; both
 *              then rescaled per column to [0, 10].  2: embedding_out holds the start on entry, used as it is.
 *   layout     epochs e = 0 .. n_epochs - 1, alpha = learning_rate (1 - e / n_epochs); an edge is due when its next
 *              epoch <= e.  Due edge (i, j): attraction -2ab d2^(b-1) / (a d2^b + 1) (y_i - y_j) per component clipped to
 *              +-4, on i and (negated) on j; then floor((e - next_neg) / epn) negatives k = umap_hash(seed, e, edge, q)
 *              mod n, each (k != i) repelling i by 2 gamma b / ((0.001 + d2)(a d2^b + 1)) (y_i - y_k) clipped to +-4,
 *              or 4 per component when d2 = 0.  Every update reads the positions of the start of the epoch; a vertex
 *              moves by alpha times the fixed-order sum of its contributions.  Positions are fp32.
 * params: n_epochs >= 1 (resolved by the caller); option "stop_after_epochs" = E > 0 stops the layout after E epochs.
 * info_out (may be NULL) [8]: n, k, nnz of W, epochs run, init used (0 random, 1 spectral, 2 given), Ritz residual
 * max ||M x - theta x|| of the spectral init, n_components, max(w).  Stats: last_finalize_ms = kNN, last_reduce_ms =
 * graph and schedule, last_allreduce_ms = init, last_fused_ms = layout (device times); last_path 2 for the
 * lane-parallel-edge layout (n_components <= 4), 1 otherwise.  Errors (B2K_ERR_INVALID): n < 2, a non-finite value in
 * X ("UMAP input contains NaN or infinity"), a parameter out of range. */
typedef struct b2k_umap_params {
  int32_t n_neighbors;
  int32_t n_components;         /* 1 .. 100 */
  int32_t n_epochs;
  int32_t init;                 /* 0 random, 1 spectral, 2 given (fit only) */
  int32_t negative_sample_rate;
  int32_t reserved;
  double local_connectivity;
  double set_op_mix_ratio;
  double learning_rate;
  double repulsion_strength;
  double a, b;
  uint64_t seed;
} b2k_umap_params;
int b2k_umap_fit(b2k_ctx* ctx, const float* X, int64_t n, int d, const int32_t* labels, const b2k_umap_params* params,
                 float* embedding_out, double* info_out, uintptr_t stream);
/* The last fit's intermediates, host arrays, any may be NULL: knn_idx [n][k], knn_dist [n][k], rho [n], sigma [n],
 * indptr [n + 1], indices [nnz], weights [nnz], epochs_per_sample [nnz] (+inf: never fires), init [n][C] (the start of
 * the layout), ritz_values [C] and ritz_vectors [n][C] (spectral init only). */
int b2k_umap_graph(b2k_ctx* ctx, int64_t* knn_idx, float* knn_dist, double* rho, double* sigma, int64_t* indptr,
                   int32_t* indices, double* weights, double* epochs_per_sample, float* init, double* ritz_values,
                   double* ritz_vectors);
/* Each query row: its k exact neighbours among X_train [n_train][d]; memberships as above with no self edge and the
 * sigma floor from the row's own mean; the edges with w < max_row(w) / n_epochs never fire, epochs_per_sample =
 * max_row(w) / w; start = the w-weighted mean of the neighbours' embedding rows (fp64); then n_epochs epochs (0 allowed)
 * moving the query only, negatives k = umap_hash(seed, e, idx_0 n_train + idx_j, q) mod n_train (idx_0 the nearest
 * neighbour, idx_j the edge's), all in one kernel.  A row's result depends on that row alone.  A query with a non-finite
 * component gets a NaN row. */
int b2k_umap_transform(b2k_ctx* ctx, const float* X_train, const float* embedding, int64_t n_train, int d, const float* Q,
                       int64_t nq, const b2k_umap_params* params, float* out, uintptr_t stream);

/* ---- Gaussian mixtures (full covariances, EM) ----
 * Stands in for pyspark.ml.clustering.GaussianMixture (the reference has no Gaussian mixture).  Model: weights w_k,
 * means mu_k, covariances Sigma_k, fp64.  Densities follow Spark's MultivariateGaussian, so a singular covariance is
 * legal: Sigma_k = U diag(lambda) U^T, tol = EPS max(lambda) d with EPS = 2.220446e-16, P_k = diag(lambda_j > tol ?
 * lambda_j^-1/2 : 0) U^T and log pdf_k(x) = -(d log 2 pi + sum_{lambda_j > tol} log lambda_j) / 2 - ||P_k (x - mu_k)||^2
 * / 2; a covariance with no eigenvalue above tol is an error.
 *
 * b2k_gmm_fit (collective): X device f32 [n_local, d].  E-step per row: p_ik = w_k pdf_k(x_i) + EPS (MLlib's EM),
 * r_ik = p_ik / sum_j p_ij, LL = sum_i log sum_j p_ij over all rows of all ranks.  M-step: N_k = sum_i r_ik,
 * w_k = N_k / n, mu_k = sum r_ik x_i / N_k, Sigma_k = sum r_ik (x_i - mu_k)(x_i - mu_k)^T / N_k; the device sums are
 * taken about c = fl32(column means) and the host removes c in fp64.  One f64 allreduce per iteration.  Stops when
 * iter == max_iter or |LL - LL_prev| <= tol; *log_likelihood_out = the LL of the last E-step (-inf when max_iter = 0).
 * init_mode B2K_INIT_ARRAY: the start is init_weights [k], init_means [k][d], init_covs [k][d][d] (host f64);
 * B2K_INIT_RANDOM: weights 1/k, and component i takes the mean and the biased per-feature variance (a diagonal
 * covariance) of global rows g_{5i} .. g_{5i+4}, g_j = splitmix64(seed ^ splitmix64(j)) mod n_total, the global row
 * order being rank 0's rows, then rank 1's, and so on (splitmix64: z += 0x9e3779b97f4a7c15, z = (z ^ z >> 30)
 * 0xbf58476d1ce4e5b9, z = (z ^ z >> 27) 0x94d049bb133111eb, z ^ z >> 31).  Outputs (host): weights_out [k], means_out
 * [k][d], covs_out [k][d][d], *n_iter_out, cluster_sizes_out [k] = argmax counts of b2k_gmm_predict with the final
 * model over all ranks.  E pass on wgmma (3xTF32) for d % 4 == 0, 4 <= d <= 128, k <= 64 and a 16-byte aligned X,
 * else on a generic fp64 SIMT pass; option "kernel_path" = B2K_PATH_GENERIC forces the generic pass, B2K_PATH_FUSED
 * fails with B2K_ERR_UNSUPPORTED where wgmma cannot run (decided on every rank together).  The weighted Gram pass of the
 * M-step runs on wgmma (3xTF32, fp64 partials) for d % 4 == 0 and a 16-byte aligned X, else on an fp64 SIMT pass, and
 * kernel_path = B2K_PATH_GENERIC forces that pass too; the moments pass is fp64 SIMT.  Errors, decided on allgathered or
 * allreduced values so that every rank fails together (B2K_ERR_INVALID unless noted): an empty partition on any rank;
 * a NaN or an infinity in X; k < 2; k > n_total; d < 1; max_iter < 0; tol < 0; a covariance with no eigenvalue above
 * tol; d > 256, k > 256 or k d^2 > 2^24, more than 2^31 - 256 rows on a rank (B2K_ERR_UNSUPPORTED).  Synchronises `stream`.  Bitwise reproducible for the
 * same input, rank count and device.  Stats: last_path = the E pass that ran; last_n_iter; with option "time_kernels"
 * != 0, last_fused_ms = the E passes, last_reduce_ms = the M passes, last_allreduce_ms = the allreduces (device times,
 * summed over the iterations), last_finalize_ms = the host updates (the eigendecompositions and the model uploads
 * included) and last_loop_ms = the whole call (host clock). */
#define B2K_GMM_MAX_D 256
#define B2K_GMM_MAX_K 256
int b2k_gmm_fit(b2k_ctx* ctx, const float* X, int64_t n_local, int d, int k, int init_mode, const double* init_weights,
                const double* init_means, const double* init_covs, int max_iter, double tol, uint64_t seed,
                double* weights_out, double* means_out, double* covs_out, double* log_likelihood_out, int* n_iter_out,
                int64_t* cluster_sizes_out, uintptr_t stream);
/* Local (no collective): per row of X [n, d] the probabilities prob_out [n][k] (device f64, r_ik of the E-step above)
 * and labels_out [n] (device int32, the first argmax), with the model weights [k], means [k][d], covs [k][d][d] (host
 * f64).  Rows are read about fl32(sum_k w_k mu_k), so a row's result depends on that row and the model alone.  Same
 * passes, bounds and errors as b2k_gmm_fit's E-step.  Synchronises `stream`. */
int b2k_gmm_predict(b2k_ctx* ctx, const float* X, int64_t n, int d, int k, const double* weights, const double* means,
                    const double* covs, double* prob_out, int32_t* labels_out, uintptr_t stream);

/* ---- bisecting k-means (euclidean) ----
 * Stands in for pyspark.ml.clustering.BisectingKMeans (the reference has no bisecting k-means), whose rules are restated
 * here so that no Spark source is needed.
 *
 * Nodes: the root is 1, the children of i are 2i (left) and 2i + 1 (right).  A node's summary is its row count n, its
 * centre (the fp64 mean of its rows) and its cost (the sum of squared distances of its rows to that centre).
 * minSize = ceil(min_divisible) when min_divisible >= 1, else ceil(min_divisible n_total).
 * Levels: level 1 starts with the root as the only active node and need = k - 1.  While there are active nodes,
 * need > 0 and level < 63: a node is divisible when n >= minSize and cost > EPS n (EPS = 2.220446049250313e-16); when
 * more than `need` nodes are divisible the `need` largest by n divide, ties to the lower index (Spark breaks ties in
 * hash-map order, which is not reproduced); when none is, every active node becomes a leaf and the loop ends.
 * Split start: a node i with centre c starts its children at c - l u and c + l u, l = 1e-4 ||c||_2, u_j =
 * (splitmix64(splitmix64(seed ^ splitmix64(i)) + j) >> 11) 2^-53 (splitmix64 as for b2k_gmm_fit), so the start
 * depends on neither the order of the splits nor the rank count.  Spark draws from java.util.Random(seed) in map order:
 * the start differs from Spark's for the same seed (deliberate).
 * Iterations: max_iter per level.  Each reassigns every row of every dividing node to the nearer of that node's live
 * children (fp64 sums of (x_j - c_j)^2 from the fp32 row, ties to the left) and recomputes the children's summaries; a
 * child left with no rows drops out for the rest of the level.  The device sums are taken about the parent's centre p:
 * S1 = sum (x - p), S2 = sum ||x - p||^2, centre = p + S1 / n, cost = max(S2 - ||S1||^2 / n, 0) in fp64 (Spark forms
 * sumSq - n ||c||^2, equal in exact arithmetic but cancelling on offset data: a deliberate difference).  The root's
 * summary comes from the fp64 column means and centred squares.
 * Level end: every row of a dividing node is reassigned once more with the final centres (the assignment the next level
 * starts from); the stored child summaries stay those of the last iteration (Spark's order).  The children with rows
 * become the active nodes; every other node is inactive; need drops by the number of nodes divided, even when a child
 * came out empty, so the model can have fewer than k leaves (also when k > n_total, which is legal).
 * Leaves are numbered 0, 1, ... in depth-first order, left first.  Predict: from the root, move to the nearer existing
 * child (the fp64 rule above, ties left) until a leaf; a node with one child passes to it.
 *
 * b2k_bkm_fit (collective): X device f32 [n_local, d].  Outputs (host): *n_nodes_out; per node in depth-first order
 * (at most 2k - 1) node_index_out, node_centers_out [n_nodes][d] (fp64), node_size_out, node_cost_out;
 * *training_cost_out = the sum of the leaf costs; cluster_sizes_out [k] = per leaf the rows b2k_bkm_predict sends
 * there over all ranks, zero past the leaf count; level_ms_out [B2K_BKM_MAX_LEVELS] (or NULL) = each level's device time
 * with option "time_kernels".  Errors, decided on allgathered or allreduced values so that every rank fails together
 * (B2K_ERR_INVALID unless noted): an empty partition on any rank; a NaN or an infinity in X; k < 2; max_iter < 1;
 * min_divisible <= 0 (or not finite); d < 1; d > B2K_BKM_MAX_D, k > B2K_BKM_MAX_K, k d > 2^24 or more than 2^31 - 1
 * rows on a rank (B2K_ERR_UNSUPPORTED).  Synchronises `stream`.  No atomics: bitwise reproducible for the same input,
 * rank count and device (option "grid_limit", which caps the split pass's CTAs, does not change the result).  Stats:
 * last_n_iter = the levels run; with option "time_kernels" != 0, last_fused_ms = the split passes, last_reduce_ms =
 * the fold, centre and partition passes, last_allreduce_ms = the allreduces (device times, CUDA events),
 * last_finalize_ms = the host's level decisions and last_loop_ms = the whole call (host clock). */
#define B2K_BKM_MAX_D 4096
#define B2K_BKM_MAX_K 65536
#define B2K_BKM_MAX_LEVELS 62
int b2k_bkm_fit(b2k_ctx* ctx, const float* X, int64_t n_local, int d, int k, int max_iter, double min_divisible,
                uint64_t seed, int* n_nodes_out, int64_t* node_index_out, double* node_centers_out,
                int64_t* node_size_out, double* node_cost_out, double* training_cost_out, int64_t* cluster_sizes_out,
                double* level_ms_out, uintptr_t stream);
/* Local (no collective): per row of X [n, d] the leaf reached by descent (labels_out, device int32) and, when cost_out
 * is not NULL, the squared distance to that leaf's centre (device f64), for the tree of n_nodes nodes node_index [n_nodes]
 * with centres node_centers [n_nodes][d] (host, any order; the indices must be distinct, include 1 and every non-root's
 * parent).  Errors: a bad node list or a non-finite centre (B2K_ERR_INVALID); d > B2K_BKM_MAX_D or more than
 * 2 B2K_BKM_MAX_K - 1 nodes (B2K_ERR_UNSUPPORTED).  Synchronises `stream`. */
int b2k_bkm_predict(b2k_ctx* ctx, const float* X, int64_t n, int d, int n_nodes, const int64_t* node_index,
                    const double* node_centers, int32_t* labels_out, double* cost_out, uintptr_t stream);

/* ---- multilayer perceptron classification ----
 * Stands in for pyspark.ml.classification.MultilayerPerceptronClassifier (the reference has none); its rules are restated
 * here so that no Spark source is needed.
 *
 * Topology: layers [n_layers] = [d, h_1, ..., h_{L-1}, C], n_layers >= 2, every entry >= 1 (B2K_ERR_INVALID) and at most
 * B2K_MLP_MAX_WIDTH (B2K_ERR_UNSUPPORTED); layers[0] must equal d, C = layers[L] is the class count.  Every layer is
 * affine, z_l = W_l a_{l-1} + b_l (a_0 = x); hidden layers apply the sigmoid a_l = 1 / (1 + exp(-z_l)); the last layer's
 * z_L goes to the softmax with cross-entropy loss.
 * Weights (Spark's flat layout, fp64): for l = 1 .. L in order, W_l (numOut x numIn, column-major: element (o, i) at
 * offset i numOut + o), then its numOut biases; P = sum_l numOut_l (numIn_l + 1) values in all.  So a Spark model's
 * weights can be used as they are.
 * Objective: F(w) = (1/n) sum_rows -log softmax(z_L)_y, the log-sum-exp with the row maximum removed; no regularisation.
 * Gradient: delta_L = p - onehot(y), delta_l = (W_{l+1}^T delta_{l+1}) (.) a_l (1 - a_l), dW_l = (1/n) sum delta_l
 * a_{l-1}^T, db_l = (1/n) sum delta_l.
 * Labels: integers in [0, C), checked by b2k_logreg_labels' pass and rules ("Labels MUST be Integers, but got v", ...)
 * plus a max label < C check, decided on gathered values: every rank fails together.  Spark truncates a fractional
 * label; rejecting it is a deliberate difference.
 * Loss weighting: Spark averages the loss within blockSize blocks and then across blocks; here the average is over
 * rows, so blockSize has no effect (deliberate).
 *
 * Device passes: the rows run in chunks whose fp32 (wgmma) or fp64 (generic) activations take at most 32 MB (rows per
 * chunk: the largest multiple of 4096 within 2^25 / (8 + es sum_{l >= 1} ceil4(layers[l])), es = 4 or 8, at least 4096).
 * The products run on wgmma (3xTF32: fp32-accurate products, fp32 activations and deltas) when d % 4 == 0 and X is
 * 16-byte aligned on every rank (the wgmma envelope, decided on an allreduced flag; any widths up to B2K_MLP_MAX_WIDTH),
 * else on a generic fp64 SIMT path (fp64 products, activations and sums); option "kernel_path" = B2K_PATH_GENERIC
 * forces the generic path, B2K_PATH_FUSED fails with B2K_ERR_UNSUPPORTED outside the envelope.  The gradient sums are
 * formed per fixed 512-row unit of a rank's rows (in fp32 on the wgmma path: 32-row chunks added in round-to-nearest
 * fp32; in fp64 on the generic path), and the units are folded in order in fp64: no atomics, bitwise reproducible for
 * the same input, rank count and device, whatever option "grid_limit" (a cap on the CTAs of every pass) is.  Across
 * rank counts the unit boundaries move with the shards: the generic path's gradient agrees with one rank's to about
 * 1e-12 of |grad F|, the wgmma path's to about 1e-6 of |grad F| (the fp32 unit sums); F agrees to about 1e-12 on both
 * (its per-row losses are fp64 and row-local).
 *
 * b2k_mlp_eval (collective): X device f32 [n_local, d], y device f32 [n_local], weights host f64 [P].  Outputs (host):
 * *f_out = F, grad_out [P] = its gradient in the flat layout, *n_total_out (may be NULL).  One label pass, one f64
 * allreduce; synchronises `stream`.  Errors (B2K_ERR_INVALID unless noted, every rank together): an empty partition on
 * any rank; a NaN or an infinity in X; a non-finite weight; the layer and label rules; kernel_path=2 outside the envelope
 * (B2K_ERR_UNSUPPORTED).  Stats: last_path; with option "time_kernels", last_fused_ms = the device passes.
 *
 * b2k_mlp_fit (collective): solver B2K_MLP_LBFGS: b2k_logreg_minimize's L-BFGS (l1 = NULL) with max_iter and tol;
 * B2K_MLP_GD: MLlib's full-batch GradientDescent with SimpleUpdater, w_t = w_{t-1} - (step_size / sqrt(t)) grad F(w_{t-1}),
 * t = 1 .. max_iter, stopping early when ||w_t - w_{t-1}|| < tol max(||w_t||, 1).  The start is initial_weights [P] when
 * not NULL, else weight j of layer l is (u_j 4.8 - 2.4) / sqrt(numIn_l), u_j = (splitmix64(seed ^ splitmix64(j)) >> 11)
 * 2^-53 (splitmix64 as for b2k_gmm_fit), so it depends on neither the rank count nor the partitioning.  Spark draws
 * from XORShiftRandom: the start differs from Spark's for the same seed (deliberate).  Outputs (host): weights_out [P];
 * history_out [max_iter + 1] = F at each accepted iterate (L-BFGS: the start, then each iteration; GD: the point of each
 * step, before its update, as MLlib records it); *n_iter_out = the entries written.  Errors: those of b2k_mlp_eval;
 * max_iter < 0; tol < 0; step_size <= 0 (GD); an unknown solver.  Stats: last_n_iter; with "time_kernels",
 * last_fused_ms = the device passes of every evaluation and last_loop_ms = the whole call (host clock).
 *
 * b2k_mlp_predict (local, asynchronous on `stream`; the weights are copied before it returns): per row of X [n, d]
 * raw_out [n][C] = z_L, prob_out [n][C] = softmax(z_L), pred_out [n] = the first argmax of z_L (device f64).  Same
 * paths; errors: the layer rules, a non-finite weight, kernel_path=2 outside the envelope. */
#define B2K_MLP_MAX_WIDTH 1024
typedef enum b2k_mlp_solver { B2K_MLP_LBFGS = 0, B2K_MLP_GD = 1 } b2k_mlp_solver;
int b2k_mlp_eval(b2k_ctx* ctx, const float* X, const float* y, int64_t n_local, const int32_t* layers, int n_layers,
                 const double* weights, double* f_out, double* grad_out, int64_t* n_total_out, uintptr_t stream);
int b2k_mlp_fit(b2k_ctx* ctx, const float* X, const float* y, int64_t n_local, const int32_t* layers, int n_layers,
                int solver, int max_iter, double tol, double step_size, uint64_t seed, const double* initial_weights,
                double* weights_out, double* history_out, int* n_iter_out, uintptr_t stream);
int b2k_mlp_predict(b2k_ctx* ctx, const float* X, int64_t n, const int32_t* layers, int n_layers, const double* weights,
                    double* raw_out, double* prob_out, double* pred_out, uintptr_t stream);

/* ---- ALS (alternating least squares collaborative filtering) ----
 * Stands in for pyspark.ml.recommendation.ALS (the reference has none); its rules are restated here so that no Spark
 * source is needed.
 *
 * Input: per rank, n_local (user, item, rating) triples.  users / items are device f64 [n_local] (any numeric column,
 * cast): each value must be integral and inside int32, else B2K_ERR_INVALID with Spark's message ("ALS only supports
 * values in Integer range and without fractional part for column user. Value v was either out of Integer range or
 * contained a fractional part that could not be converted.").  ratings is device f32 [n_local], or NULL for every rating
 * 1.0; a non-finite rating is B2K_ERR_INVALID.  Duplicate (user, item) pairs are all kept, each a separate rating.  The
 * sizes and the first bad value of every rank are allgathered first, so every error fails on every rank.  A rank may
 * hold no ratings; the whole dataset may not be empty.
 * Indexing: users are the sorted distinct user ids over all ranks (dense index u), items likewise (dense index i).
 * Start: without init_user_factors, user u's factor is x_j = fl32(v_j / sqrt(sum_j v_j^2)) (the sum in fp64, in j order),
 * v_j = fl32(sqrt(-2 ln u1) cos(2 pi u2)) for j < rank, where h = splitmix64(splitmix64(splitmix64(seed) ^ id) ^ j)
 * (id the raw user id as uint32, splitmix64 as for b2k_gmm_fit), u1 = ((h >> 11) + 1) 2^-53, u2 = (splitmix64(h) >> 11)
 * 2^-53.  Spark draws from XORShiftRandom per block: the start differs from Spark's for the same seed (deliberate), and
 * depends on neither the rank count nor the partitioning.  The item factors need no start.
 * Iteration (max_iter >= 0 times, Spark's order): solve every item from the user factors, then every user from the item
 * factors.  For destination d over its ratings (s, r), with source factors y_s:
 *   explicit: A = sum y_s y_s^T, b = sum r y_s, n = #ratings;
 *   implicit: c1 = alpha |r|, A = Y^T Y + sum c1 y_s y_s^T, b = sum_{r > 0} (1 + c1) y_s, n = #{r > 0}, Y^T Y the Gram of
 *   every source factor;
 *   then (A + reg_param n I) x = b by Cholesky, accumulated and solved in fp64 from the fp32 factors, x stored as fp32.
 *   A system that is not positive definite (reg_param = 0 with fewer ratings than rank, say) fails on every rank
 *   (B2K_ERR_INVALID), as Spark's solver fails.  With max_iter = 0 the item factors are zero.
 * Distribution: rank q owns users [U q / R, U (q + 1) / R) and items likewise.  The ratings travel by chunked allgathers
 * (2^22 per rank per round); each rank keeps those of its users sorted by (user, item, global row) and of its items by
 * (item, user, global row), global row = the rank's offset + local row.  Per rank the fit holds: the n_local triples
 * (12 B each, freed after the redistribution), both full factor tables ((U + I) rank 4 B), its own ratings twice (12 B
 * each, plus 24 B each and the sort buffers while it sorts them), one round's buffers (R 2^22 x 88 B at most) and at most
 * 1 GB of fp64 unit partials (more only when one destination needs more).  Each half-step every rank holds the whole
 * source table, forms Y^T Y over all of it (no allreduce: the result does not depend on the rank count), solves the
 * destinations it owns and allgathers them.  No pass uses atomics: the factors are bitwise identical for the same input
 * on any rank count and any option "grid_limit" (a cap on the CTAs of the normal-equation and solve passes).
 * Device passes: the normal-equation pass runs over units of at most 512 ratings of one destination; each unit sums the
 * upper triangle of A, b and n in fp64 FMA (the fp32 products are exact in fp64, so only the order of the additions
 * matters, and it is the rating order), a long destination spanning several units that the solve pass folds in unit
 * order; Y^T Y comes from the local generic Gram pass; the solve pass runs one CTA per destination on [A | b] in shared
 * memory.  1 <= rank <= B2K_ALS_MAX_RANK, else B2K_ERR_UNSUPPORTED.
 *
 * b2k_als_fit (collective): outputs on the device, sized by the caller: user_ids_out [user_cap] i32, user_factors_out
 * [user_cap][rank] f32, item_ids_out [item_cap], item_factors_out [item_cap][rank]; *n_users_out = U and *n_items_out = I
 * (host), set also when a cap is too small (then B2K_ERR_INVALID on every rank, so a caller can size and call again).
 * init_user_factors (host f32 [init_n_users][rank], in sorted user-id order; NULL: the seeded start) must have
 * init_n_users == U.  Errors also: max_iter < 0, reg_param < 0 or not finite, alpha < 0 or not finite (implicit).
 * Synchronises `stream`.  Stats: last_n_iter; with option "time_kernels": last_fused_ms, last_finalize_ms,
 * last_allreduce_ms and last_reduce_ms = the mean device time per half-step of the normal-equation pass, the solve pass,
 * the factor allgather and the Y^T Y pass; last_probe_ms = the setup (check, id maps, redistribution, sorts) and
 * last_loop_ms = the whole call (host clock).
 *
 * b2k_als_predict (local, asynchronous on `stream`): out [n] f32 = for each (users[j], items[j]) (device f64) the fp32
 * dot product s = fl32(s + fl32(u_k v_k)) in k order of the user's and the item's factors, looked up in the sorted id
 * maps (device i32 [n_users] / [n_items] with their factor tables); NaN when either id is unknown, fractional or outside
 * int32.
 *
 * b2k_als_recommend (local, asynchronous): for each query row q of Q [nq][rank] (device f32), the n best rows of T
 * [nt][rank] by the same dot product, score descending, the lower row first on a tie: idx_out [nq][n] i32 (-1 past nt)
 * and score_out [nq][n] f32 (NaN past nt).  1 <= n <= B2K_ALS_MAX_N. */
#define B2K_ALS_MAX_RANK 128
#define B2K_ALS_MAX_N 1024
int b2k_als_fit(b2k_ctx* ctx, const double* users, const double* items, const float* ratings, int64_t n_local,
                int rank, int max_iter, double reg_param, int implicit_prefs, double alpha, uint64_t seed,
                const float* init_user_factors, int64_t init_n_users, int64_t user_cap, int64_t item_cap,
                int32_t* user_ids_out, float* user_factors_out, int32_t* item_ids_out, float* item_factors_out,
                int64_t* n_users_out, int64_t* n_items_out, uintptr_t stream);
int b2k_als_predict(b2k_ctx* ctx, const double* users, const double* items, int64_t n, int rank,
                    const int32_t* user_ids, const float* user_factors, int64_t n_users, const int32_t* item_ids,
                    const float* item_factors, int64_t n_items, float* out, uintptr_t stream);
int b2k_als_recommend(b2k_ctx* ctx, const float* Q, int64_t nq, const float* T, int64_t nt, int rank, int n,
                      int32_t* idx_out, float* score_out, uintptr_t stream);

#ifdef __cplusplus
}
#endif
#endif /* B2KMEANS_H_ */
