"""ctypes binding of libb2kmeans.so (the C ABI declared in include/b2kmeans.h).

PyTorch tensors are used only as device-memory containers: every call hands raw addresses and the
current CUDA stream to the library, which trusts them, so Context takes every device address through
Context._dev after checking the tensor behind it.  There is NO fallback: if the shared library
is missing or no CUDA device is present, the compute entry points raise.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np

_PKG_DIR = os.path.dirname(os.path.abspath(__file__))
# B2K_LIB loads another build of the same library instead of the in-tree one
LIB_PATH = os.environ.get("B2K_LIB") or os.path.join(_PKG_DIR, "libb2kmeans.so")
CSRC_DIR = os.path.join(_PKG_DIR, "csrc")

B2K_OK = 0
INIT_ARRAY, INIT_RANDOM, INIT_KMEANS_PARALLEL = 0, 1, 2
PATH_AUTO, PATH_GENERIC, PATH_FUSED = 0, 1, 2
LAYOUT_ROWS, LAYOUT_COLUMNS = 0, 1
UNIQUE_ID_BYTES = 128

_DTYPE_CODES = {
    np.dtype("float32"): 0,
    np.dtype("float64"): 1,
    np.dtype("int8"): 2,
    np.dtype("int16"): 3,
    np.dtype("int32"): 4,
    np.dtype("int64"): 5,
}

# every symbol include/b2kmeans.h declares (tests check the library exports exactly these)
EXPORTED_SYMBOLS = (
    "b2k_version",
    "b2k_last_error",
    "b2k_ctx_create",
    "b2k_ctx_destroy",
    "b2k_ctx_set_option",
    "b2k_get_stats",
    "b2k_get_fused_profile",
    "b2k_reset_stats",
    "b2k_comm_unique_id",
    "b2k_comm_init",
    "b2k_comm_destroy",
    "b2k_comm_abort",
    "b2k_ingest_append",
    "b2k_kmeans_fit",
    "b2k_kmeans_lloyd",
    "b2k_kmeans_assign",
    "b2k_pca_fit",
    "b2k_pca_finalize",
    "b2k_pca_transform",
    "b2k_knn_search",
    "b2k_ivf_search",
    "b2k_linreg_moments",
    "b2k_linreg_solve",
    "b2k_linreg_predict",
    "b2k_logreg_labels",
    "b2k_logreg_eval",
    "b2k_logreg_minimize",
    "b2k_logreg_fit",
    "b2k_logreg_predict",
    "b2k_ingest_csr_append",
    "b2k_logreg_eval_csr",
    "b2k_logreg_fit_csr",
    "b2k_logreg_predict_csr",
    "b2k_dbscan_fit",
    "b2k_rf_fit",
    "b2k_rf_forest",
    "b2k_rf_predict",
    "b2k_eval_linear",
    "b2k_eval_forest",
    "b2k_eval_linear_scores",
    "b2k_eval_forest_scores",
    "b2k_eval_binary",
    "b2k_umap_fit",
    "b2k_umap_graph",
    "b2k_umap_transform",
    "b2k_silhouette",
    "b2k_silhouette_multi",
    "b2k_gmm_fit",
    "b2k_gmm_predict",
    "b2k_bkm_fit",
    "b2k_bkm_predict",
    "b2k_mlp_eval",
    "b2k_mlp_fit",
    "b2k_mlp_predict",
    "b2k_als_fit",
    "b2k_als_predict",
    "b2k_als_recommend",
)

ALS_MAX_RANK = 128   # B2K_ALS_MAX_RANK
ALS_MAX_N = 1024     # B2K_ALS_MAX_N

MLP_SOLVERS = {"l-bfgs": 0, "gd": 1}   # b2k_mlp_solver

BKM_MAX_LEVELS = 62   # B2K_BKM_MAX_LEVELS

EVAL_KINDS = {"identity": 0, "logistic": 1, "softmax": 2}
BINARY_METRICS = {"areaUnderROC": 0, "areaUnderPR": 1}
SILHOUETTE_METRICS = {"squaredEuclidean": 0, "cosine": 1}

FAMILY_CODES = {"auto": 0, "binomial": 1, "multinomial": 2}
METRIC_CODES = {"euclidean": 0, "cosine": 1}
IMPURITY_CODES = {"gini": 0, "entropy": 1, "variance": 2}
# int (*)(void* user, int n, const double* x, double* f, double* grad)
LOGREG_OBJECTIVE = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_double),
                                    ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double))


class B2KError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"libb2kmeans error {code}: {msg}")
        self.code = code


def _u64(seed: int) -> int:
    """A seed as the library's uint64_t (a negative seed wraps as in C)."""
    return int(seed) & 0xFFFFFFFFFFFFFFFF


def _dims(shape: Sequence[Optional[int]]) -> str:
    return "[" + ", ".join("*" if s is None else str(s) for s in shape) + "]"


def _host(a: Any, dtype: Any, shape: Sequence[Optional[int]], name: str) -> np.ndarray:
    """a as a C-contiguous host array of dtype, once its shape is checked against `shape` (None: any extent).  The
    caller keeps the array alive while the library reads it through .ctypes.data."""
    arr = np.ascontiguousarray(a, dtype=dtype)
    if arr.ndim != len(shape) or any(s is not None and e != s for e, s in zip(arr.shape, shape)):
        raise ValueError(f"{name} must be a {arr.dtype} array {_dims(shape)}, got shape {list(arr.shape)}")
    return arr


class LogregParams(ctypes.Structure):
    _fields_ = [
        ("reg", ctypes.c_double),
        ("l1_ratio", ctypes.c_double),
        ("tol", ctypes.c_double),
        ("max_iter", ctypes.c_int32),
        ("fit_intercept", ctypes.c_int32),
        ("standardization", ctypes.c_int32),
        ("family", ctypes.c_int32),
    ]


class RfParams(ctypes.Structure):
    _fields_ = [
        ("n_trees", ctypes.c_int32),
        ("max_depth", ctypes.c_int32),
        ("max_bins", ctypes.c_int32),
        ("min_instances", ctypes.c_int32),
        ("features_per_node", ctypes.c_int32),
        ("bootstrap", ctypes.c_int32),
        ("impurity", ctypes.c_int32),
        ("reserved", ctypes.c_int32),
        ("min_info_gain", ctypes.c_double),
        ("seed", ctypes.c_uint64),
    ]


class UmapParams(ctypes.Structure):
    _fields_ = [
        ("n_neighbors", ctypes.c_int32),
        ("n_components", ctypes.c_int32),
        ("n_epochs", ctypes.c_int32),
        ("init", ctypes.c_int32),
        ("negative_sample_rate", ctypes.c_int32),
        ("reserved", ctypes.c_int32),
        ("local_connectivity", ctypes.c_double),
        ("set_op_mix_ratio", ctypes.c_double),
        ("learning_rate", ctypes.c_double),
        ("repulsion_strength", ctypes.c_double),
        ("a", ctypes.c_double),
        ("b", ctypes.c_double),
        ("seed", ctypes.c_uint64),
    ]


UMAP_INIT_CODES = {"random": 0, "spectral": 1, "given": 2}


def umap_params(n_neighbors: int = 15, n_components: int = 2, n_epochs: int = 200, init: str = "spectral",
                negative_sample_rate: int = 5, local_connectivity: float = 1.0, set_op_mix_ratio: float = 1.0,
                learning_rate: float = 1.0, repulsion_strength: float = 1.0, a: float = 1.577, b: float = 0.895,
                seed: int = 0) -> UmapParams:
    """b2k_umap_params from keyword values (n_epochs resolved by the caller)."""
    return UmapParams(int(n_neighbors), int(n_components), int(n_epochs), UMAP_INIT_CODES[init],
                      int(negative_sample_rate), 0, float(local_connectivity), float(set_op_mix_ratio),
                      float(learning_rate), float(repulsion_strength), float(a), float(b), _u64(seed))


class Stats(ctypes.Structure):
    _fields_ = [
        ("kernel_launches", ctypes.c_int64),
        ("fused_tc_launches", ctypes.c_int64),
        ("generic_launches", ctypes.c_int64),
        ("nccl_allreduces", ctypes.c_int64),
        ("last_path", ctypes.c_int32),
        ("last_n_iter", ctypes.c_int32),
        ("last_fused_ms", ctypes.c_double),
        ("last_loop_ms", ctypes.c_double),
        ("last_reduce_ms", ctypes.c_double),
        ("last_allreduce_ms", ctypes.c_double),
        ("last_finalize_ms", ctypes.c_double),
        ("recheck_rows", ctypes.c_int64),
        ("recheck_candidates", ctypes.c_int64),
        ("path_switch_iter", ctypes.c_int64),
        ("last_probe_ms", ctypes.c_double),
    ]


def build(verbose: bool = False) -> str:
    """Compile libb2kmeans.so for sm_90a with nvcc (cross-compiles without a GPU)."""
    cmd = ["make", "-C", CSRC_DIR, "-j", "8"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("building libb2kmeans.so failed:\n" + res.stdout + "\n" + res.stderr)
    if verbose:
        print(res.stdout)
    return LIB_PATH


_lib: Optional[ctypes.CDLL] = None


def load_library() -> ctypes.CDLL:
    """Load (never build) the in-tree shared library; raises loudly when it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise FileNotFoundError(
            f"{LIB_PATH} not found. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make -C spark_rapids_ml_b200/csrc`). There is no CPU/PyTorch fallback for the KMeans path."
        )
    L = ctypes.CDLL(LIB_PATH, mode=ctypes.RTLD_GLOBAL)
    vp, i32, i64, u64, f64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_uint64, ctypes.c_double
    L.b2k_version.restype = i32
    L.b2k_last_error.restype = ctypes.c_char_p
    L.b2k_last_error.argtypes = [vp]
    L.b2k_ctx_create.argtypes = [i32, ctypes.POINTER(vp)]
    L.b2k_ctx_destroy.argtypes = [vp]
    L.b2k_ctx_set_option.argtypes = [vp, ctypes.c_char_p, i64]
    L.b2k_get_stats.argtypes = [vp, ctypes.POINTER(Stats)]
    L.b2k_reset_stats.argtypes = [vp]
    L.b2k_get_fused_profile.argtypes = [vp, vp, i64, ctypes.POINTER(i32), ctypes.POINTER(i32)]
    L.b2k_comm_unique_id.argtypes = [ctypes.c_char_p]
    L.b2k_comm_init.argtypes = [vp, i32, i32, ctypes.c_char_p]
    L.b2k_comm_destroy.argtypes = [vp]
    L.b2k_comm_abort.argtypes = [vp]
    L.b2k_ingest_append.argtypes = [vp, vp, i64, i32, i64, vp, vp, i64, i32, i32, ctypes.c_size_t,
                                    ctypes.POINTER(i64)]
    L.b2k_kmeans_fit.argtypes = [vp, vp, i64, i32, i32, i32, vp, i32, f64, u64, f64, i32, vp,
                                 ctypes.POINTER(i32), ctypes.POINTER(f64), ctypes.c_size_t]
    L.b2k_kmeans_lloyd.argtypes = [vp, vp, i64, i32, i32, vp, i32, f64, ctypes.POINTER(i32),
                                   ctypes.POINTER(f64), ctypes.c_size_t]
    L.b2k_kmeans_assign.argtypes = [vp, vp, i64, i32, vp, i32, vp, vp, ctypes.c_size_t]
    L.b2k_pca_fit.argtypes = [vp, vp, i64, i32, i32, vp, vp, vp, vp, ctypes.c_size_t]
    L.b2k_pca_finalize.argtypes = [vp, i32, i64, i32, vp, vp, vp]
    L.b2k_pca_transform.argtypes = [vp, vp, i64, i32, vp, i32, vp, ctypes.c_size_t]
    L.b2k_knn_search.argtypes = [vp, vp, i64, vp, vp, i64, i32, i32, vp, vp, ctypes.c_size_t]
    L.b2k_ivf_search.argtypes = [vp, vp, i64, vp, vp, i64, i32, i32, i32, i32, i32, f64, i32, i32, vp, vp, vp, vp, vp,
                                 ctypes.c_size_t]
    L.b2k_linreg_moments.argtypes = [vp, vp, vp, i64, i32, ctypes.POINTER(i64), vp, vp, ctypes.c_size_t]
    L.b2k_linreg_solve.argtypes = [vp, vp, i32, i64, f64, f64, i32, i32, i32, f64, vp, ctypes.POINTER(f64),
                                   ctypes.POINTER(i32)]
    L.b2k_linreg_predict.argtypes = [vp, vp, i64, i32, vp, f64, vp, ctypes.c_size_t]
    L.b2k_logreg_labels.argtypes = [vp, vp, i64, vp, vp, ctypes.POINTER(i32), ctypes.POINTER(i64), ctypes.c_size_t]
    L.b2k_logreg_eval.argtypes = [vp, vp, vp, i64, i32, vp, i32, i32, vp, vp, ctypes.POINTER(f64), vp,
                                  ctypes.POINTER(i64), ctypes.c_size_t]
    L.b2k_logreg_minimize.argtypes = [LOGREG_OBJECTIVE, vp, i32, vp, vp, i32, f64, ctypes.POINTER(i32),
                                      ctypes.POINTER(i32), ctypes.POINTER(f64)]
    L.b2k_logreg_fit.argtypes = [vp, vp, vp, i64, i32, vp, vp, i32, i32, ctypes.POINTER(LogregParams), vp, vp, vp, vp,
                                 ctypes.c_size_t]
    L.b2k_logreg_predict.argtypes = [vp, vp, i64, i32, i32, vp, vp, vp, vp, vp, vp, ctypes.c_size_t]
    L.b2k_ingest_csr_append.argtypes = [vp, vp, vp, vp, i64, i64, i64, i64, i64, vp, vp, vp, vp, vp, vp, i32, i64,
                                        ctypes.c_size_t, ctypes.POINTER(i64)]
    L.b2k_logreg_eval_csr.argtypes = [vp, vp, vp, vp, i64, i64, i64, vp, vp, i32, i32, vp, vp, ctypes.POINTER(f64), vp,
                                      ctypes.POINTER(i64), ctypes.c_size_t]
    L.b2k_logreg_fit_csr.argtypes = [vp, vp, vp, vp, i64, i64, i64, vp, vp, vp, i32, i32, ctypes.POINTER(LogregParams),
                                     vp, vp, vp, vp, ctypes.c_size_t]
    L.b2k_logreg_predict_csr.argtypes = [vp, vp, vp, vp, i64, i64, i64, i32, vp, vp, vp, vp, vp, vp, ctypes.c_size_t]
    L.b2k_dbscan_fit.argtypes = [vp, vp, i64, i32, f64, i32, i32, vp, vp, ctypes.POINTER(i64), ctypes.c_size_t]
    L.b2k_rf_fit.argtypes = [vp, vp, vp, i64, i32, ctypes.POINTER(RfParams), ctypes.POINTER(i32), ctypes.POINTER(i64),
                             vp, vp, ctypes.c_size_t]
    L.b2k_rf_forest.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp]
    L.b2k_rf_predict.argtypes = [vp, vp, i64, i32, i32, vp, vp, vp, vp, vp, i32, i32, vp, vp, vp, ctypes.c_size_t]
    L.b2k_eval_linear.argtypes = [vp, vp, vp, i64, i32, i32, vp, vp, vp, vp, vp, i32, f64, vp, vp, vp, vp, vp,
                                  ctypes.c_size_t]
    L.b2k_eval_forest.argtypes = [vp, vp, vp, i64, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, i32, f64, vp, vp, vp, vp,
                                  vp, ctypes.c_size_t]
    L.b2k_eval_linear_scores.argtypes = [vp, vp, vp, i64, i32, i32, vp, vp, vp, vp, vp, i64, vp, ctypes.c_size_t]
    L.b2k_eval_forest_scores.argtypes = [vp, vp, vp, i64, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, i64, vp,
                                         ctypes.c_size_t]
    L.b2k_eval_binary.argtypes = [vp, vp, vp, i64, i32, i32, i32, vp, ctypes.c_size_t]
    L.b2k_umap_fit.argtypes = [vp, vp, i64, i32, vp, ctypes.POINTER(UmapParams), vp, vp, ctypes.c_size_t]
    L.b2k_umap_graph.argtypes = [vp] + [vp] * 11
    L.b2k_umap_transform.argtypes = [vp, vp, vp, i64, i32, vp, i64, ctypes.POINTER(UmapParams), vp, ctypes.c_size_t]
    L.b2k_silhouette.argtypes = [vp, vp, i64, i32, vp, i32, ctypes.POINTER(f64), ctypes.c_size_t]
    L.b2k_silhouette_multi.argtypes = [vp, vp, i64, i32, i32, vp, i32, vp, ctypes.c_size_t]
    L.b2k_gmm_fit.argtypes = [vp, vp, i64, i32, i32, i32, vp, vp, vp, i32, f64, u64, vp, vp, vp, ctypes.POINTER(f64),
                              ctypes.POINTER(i32), vp, ctypes.c_size_t]
    L.b2k_gmm_predict.argtypes = [vp, vp, i64, i32, i32, vp, vp, vp, vp, vp, ctypes.c_size_t]
    L.b2k_bkm_fit.argtypes = [vp, vp, i64, i32, i32, i32, f64, u64, ctypes.POINTER(i32), vp, vp, vp, vp,
                              ctypes.POINTER(f64), vp, vp, ctypes.c_size_t]
    L.b2k_bkm_predict.argtypes = [vp, vp, i64, i32, i32, vp, vp, vp, vp, ctypes.c_size_t]
    L.b2k_mlp_eval.argtypes = [vp, vp, vp, i64, vp, i32, vp, ctypes.POINTER(f64), vp, ctypes.POINTER(i64),
                               ctypes.c_size_t]
    L.b2k_mlp_fit.argtypes = [vp, vp, vp, i64, vp, i32, i32, i32, f64, f64, u64, vp, vp, vp, ctypes.POINTER(i32),
                              ctypes.c_size_t]
    L.b2k_mlp_predict.argtypes = [vp, vp, i64, vp, i32, vp, vp, vp, vp, ctypes.c_size_t]
    L.b2k_als_fit.argtypes = [vp, vp, vp, vp, i64, i32, i32, f64, i32, f64, u64, vp, i64, i64, i64, vp, vp, vp, vp,
                              ctypes.POINTER(i64), ctypes.POINTER(i64), ctypes.c_size_t]
    L.b2k_als_predict.argtypes = [vp, vp, vp, i64, i32, vp, vp, i64, vp, vp, i64, vp, ctypes.c_size_t]
    L.b2k_als_recommend.argtypes = [vp, vp, i64, vp, i64, i32, i32, vp, vp, ctypes.c_size_t]
    for name in EXPORTED_SYMBOLS:
        if name not in ("b2k_last_error",):
            getattr(L, name).restype = i32
    _lib = L
    return L


def comm_unique_id() -> bytes:
    """NCCL unique id (rank 0 only) — mirrors nccl.get_unique_id() in cuml_context.py:77."""
    L = load_library()
    buf = ctypes.create_string_buffer(UNIQUE_ID_BYTES)
    rc = L.b2k_comm_unique_id(buf)
    if rc != B2K_OK:
        raise B2KError(rc, (L.b2k_last_error(None) or b"").decode())
    return buf.raw


def pca_finalize(cov: np.ndarray, n_total: int, k: int) -> Dict[str, np.ndarray]:
    """The host eigen step of b2k_pca_fit alone (no device): cov [d, d] float64 -> components_ [k, d],
    explained_variance_ratio_ [k], singular_values_ [k] (float64)."""
    L = load_library()
    cov = np.ascontiguousarray(cov, dtype=np.float64)
    if cov.ndim != 2 or cov.shape[0] != cov.shape[1]:
        raise ValueError("cov must be a square matrix")
    d = int(cov.shape[0])
    kk = max(int(k), 0)
    comp = np.zeros((kk, d), dtype=np.float64)
    evr = np.zeros(kk, dtype=np.float64)
    sv = np.zeros(kk, dtype=np.float64)
    rc = L.b2k_pca_finalize(cov.ctypes.data, d, int(n_total), int(k), comp.ctypes.data, evr.ctypes.data, sv.ctypes.data)
    if rc != B2K_OK:
        raise B2KError(rc, (L.b2k_last_error(None) or b"").decode())
    return {"components_": comp, "explained_variance_ratio_": evr, "singular_values_": sv}


def linreg_solve(mean: np.ndarray, moments: np.ndarray, n_total: int, reg: float = 0.0, l1_ratio: float = 0.0,
                 fit_intercept: bool = True, standardization: bool = True, max_iter: int = 100,
                 tol: float = 1e-6) -> Tuple[np.ndarray, float, int]:
    """b2k_linreg_solve (host only): the fit from the outputs of Context.linreg_moments -> (coef [d] float64,
    intercept, coordinate-descent sweeps)."""
    L = load_library()
    mean = _host(mean, np.float64, (None,), "mean")
    d = int(mean.shape[0]) - 1
    moments = _host(moments, np.float64, (d + 1, d + 1), "moments")
    coef = np.zeros(max(d, 0), dtype=np.float64)
    b = ctypes.c_double(0.0)
    it = ctypes.c_int(0)
    rc = L.b2k_linreg_solve(mean.ctypes.data, moments.ctypes.data, d, int(n_total), float(reg), float(l1_ratio),
                            int(bool(fit_intercept)), int(bool(standardization)), int(max_iter), float(tol),
                            coef.ctypes.data, ctypes.byref(b), ctypes.byref(it))
    if rc != B2K_OK:
        raise B2KError(rc, (L.b2k_last_error(None) or b"").decode())
    return coef, float(b.value), int(it.value)


def logreg_minimize(fun: Any, x0: np.ndarray, l1: Optional[np.ndarray] = None, max_iter: int = 100,
                    tol: float = 1e-6) -> Tuple[np.ndarray, int, int, float]:
    """b2k_logreg_minimize (host only): minimise fun(x) -> (f, grad) plus sum l1 |x| from x0 -> (x, iterations,
    evaluations, final value with the L1 term).  An exception raised by fun aborts the minimisation and is re-raised."""
    L = load_library()
    x = np.array(x0, dtype=np.float64, copy=True)
    n = int(x.shape[0])
    l1a = None if l1 is None else _host(l1, np.float64, (n,), "l1")
    err: list = []

    def _cb(_user: Any, m: int, xp: Any, fp: Any, gp: Any) -> int:
        try:
            f, g = fun(np.ctypeslib.as_array(xp, shape=(m,)).copy())
            fp[0] = float(f)
            np.ctypeslib.as_array(gp, shape=(m,))[:] = np.asarray(g, dtype=np.float64)
            return 0
        except Exception as e:  # noqa: BLE001 - handed back to the caller below
            err.append(e)
            return 1

    cb = LOGREG_OBJECTIVE(_cb)
    it, ev, fv = ctypes.c_int(0), ctypes.c_int(0), ctypes.c_double(0.0)
    rc = L.b2k_logreg_minimize(cb, None, n, x.ctypes.data, l1a.ctypes.data if l1a is not None else None,
                               int(max_iter), float(tol), ctypes.byref(it), ctypes.byref(ev), ctypes.byref(fv))
    if err:
        raise err[0]
    if rc != B2K_OK:
        raise B2KError(rc, (L.b2k_last_error(None) or b"").decode())
    return x, int(it.value), int(ev.value), float(fv.value)


def _stream_handle(torch_mod: Any, device: Any) -> int:
    return int(torch_mod.cuda.current_stream(device).cuda_stream)


class Context:
    """One library context per process per GPU (reference: one Spark barrier task per GPU)."""

    def __init__(self, device: int = 0):
        import torch

        self._torch = torch
        self._L = load_library()
        self.device_index = int(device)
        self.device = torch.device("cuda", self.device_index)
        h = ctypes.c_void_p()
        rc = self._L.b2k_ctx_create(self.device_index, ctypes.byref(h))
        if rc != B2K_OK:
            raise B2KError(rc, (self._L.b2k_last_error(None) or b"").decode())
        self._h = h
        self.nranks = 1
        self.rank = 0

    # -- plumbing ---------------------------------------------------------------------------
    def _check(self, rc: int) -> None:
        if rc != B2K_OK:
            raise B2KError(rc, (self._L.b2k_last_error(self._h) or b"").decode())

    def _stream(self) -> int:
        return _stream_handle(self._torch, self.device)

    def _invoke(self, fn: str, *args: Any, after: Tuple[Any, ...] = ()) -> int:
        """The status of the stream-ordered entry point fn(ctx, *args, stream, *after), called on this context's device
        with its current stream."""
        with self._torch.cuda.device(self.device):
            return getattr(self._L, fn)(self._h, *args, self._stream(), *after)

    def _call(self, fn: str, *args: Any, after: Tuple[Any, ...] = ()) -> None:
        self._check(self._invoke(fn, *args, after=after))

    def _dev(self, x: Any, dtype: Any, shape: Sequence[Optional[int]], name: str, optional: bool = False
             ) -> Optional[int]:
        """The device address of x, once x is checked to be a contiguous `dtype` tensor of `shape` (None: any extent)
        on this context's device; None when optional and x is None.  The library trusts every address it receives, so
        no tensor reaches it any other way."""
        if x is None and optional:
            return None
        t = self._torch
        if not (isinstance(x, t.Tensor) and x.device == self.device and x.dtype == dtype and x.is_contiguous()
                and x.dim() == len(shape) and all(s is None or e == s for e, s in zip(x.shape, shape))):
            got = (f"{'' if x.is_contiguous() else 'a non-contiguous '}{x.dtype} {list(x.shape)} on {x.device}"
                   if isinstance(x, t.Tensor) else type(x).__name__)
            raise ValueError(f"{name} must be a contiguous {dtype} tensor {_dims(shape)} on {self.device}, got {got}")
        return x.data_ptr()

    def _empty(self, shape: Sequence[int], dtype: Any) -> Tuple[Any, int]:
        """A new output tensor on this device and its address."""
        x = self._torch.empty(tuple(shape), dtype=dtype, device=self.device)
        return x, self._dev(x, dtype, shape, "output")

    def _check_X(self, X: Any, name: str = "X") -> Tuple[int, int, int]:
        """(address, n, d) of the float32 rows X [n, d]."""
        p = self._dev(X, self._torch.float32, (None, None), name)
        return p, int(X.shape[0]), int(X.shape[1])

    def close(self) -> None:
        if getattr(self, "_h", None) is not None and self._h:
            self._L.b2k_ctx_destroy(self._h)
            self._h = None

    def __enter__(self) -> "Context":
        return self

    def __exit__(self, *exc: Any) -> None:
        self.close()

    def __del__(self) -> None:  # best effort
        try:
            self.close()
        except Exception:
            pass

    def set_option(self, key: str, value: int) -> None:
        self._check(self._L.b2k_ctx_set_option(self._h, key.encode(), int(value)))

    def stats(self) -> Dict[str, Any]:
        st = Stats()
        self._check(self._L.b2k_get_stats(self._h, ctypes.byref(st)))
        return {f: getattr(st, f) for f, _ in Stats._fields_}

    def fused_profile(self) -> "np.ndarray":
        """[grid, warps, 8] int64 cycle counters of the last fused launch (needs option profile_fused=1)."""
        buf = np.zeros(1024 * 32 * 8, dtype=np.int64)
        g, w = ctypes.c_int(0), ctypes.c_int(0)
        self._check(self._L.b2k_get_fused_profile(self._h, buf.ctypes.data, buf.size, ctypes.byref(g), ctypes.byref(w)))
        return buf[: g.value * w.value * 8].reshape(g.value, w.value, 8)

    def reset_stats(self) -> None:
        self._check(self._L.b2k_reset_stats(self._h))

    # -- comm -------------------------------------------------------------------------------
    def comm_init(self, nranks: int, rank: int, uid: bytes) -> None:
        if len(uid) != UNIQUE_ID_BYTES:
            raise ValueError(f"uid must hold the {UNIQUE_ID_BYTES} bytes of comm_unique_id(), got {len(uid)}")
        self._check(self._L.b2k_comm_init(self._h, int(nranks), int(rank), uid))
        self.nranks, self.rank = int(nranks), int(rank)

    def comm_destroy(self) -> None:
        self._check(self._L.b2k_comm_destroy(self._h))
        self.nranks, self.rank = 1, 0

    def comm_abort(self) -> None:
        self._check(self._L.b2k_comm_abort(self._h))
        self.nranks, self.rank = 1, 0

    # -- ingest -----------------------------------------------------------------------------
    def ingest_rows(self, dst: Any, row0: int, values: np.ndarray, d: int,
                    offsets: Optional[np.ndarray] = None, n_rows: Optional[int] = None) -> int:
        """Append a contiguous [n_b, d] host value buffer (Arrow list child buffer) at dst[row0:].  Row i is
        values[offsets[i]:offsets[i + 1]] when offsets are given (a sliced list array starts past 0).  A page-locked
        `values` is read by the device asynchronously: it must stay unchanged until the current stream has passed
        this call."""
        code = _DTYPE_CODES.get(values.dtype)
        if code is None:
            raise TypeError(f"unsupported source dtype {values.dtype}")
        if not values.flags.c_contiguous:
            raise ValueError("values must be a C-contiguous host array")
        dp = self._dev(dst, self._torch.float32, (None, int(d)), "dst")
        if offsets is not None:
            offsets = _host(offsets, np.int32, (None,), "offsets")
            # the library reads values[offsets[0]:offsets[-1]] and checks only each row's width against d
            if offsets.shape[0] < 1 or offsets[0] < 0 or offsets[-1] > values.size:
                ends = offsets[[0, -1]].tolist() if offsets.size else "none"
                raise ValueError(f"offsets must be n_b + 1 >= 1 positions within the {values.size} values, "
                                 f"got first and last {ends}")
            n_b = offsets.shape[0] - 1
        else:
            n_b = int(n_rows) if n_rows is not None else values.size // d
            # without offsets nothing downstream can see a wrong row width: a batch whose rows are not `d` wide would make
            # the C side read past the buffer (narrower) or silently re-shape it (wider)
            if values.size != n_b * d:
                raise ValueError(f"feature batch holds {values.size} values for {n_b} rows of width {d}: "
                                 "row width differs from the expected dimension")
        wrote = ctypes.c_int64(0)
        self._call("b2k_ingest_append", dp, int(dst.shape[0]), int(d), int(row0), values.ctypes.data,
                   offsets.ctypes.data if offsets is not None else None, int(n_b), code, LAYOUT_ROWS,
                   after=(ctypes.byref(wrote),))
        return int(wrote.value)

    def ingest_pinned_tensor(self, dst: Any, row0: int, src: Any) -> int:
        """Append a (pinned) host torch tensor [n_b, d] f32.  A pinned `src` is copied to dst by the device
        asynchronously, with no staging copy: it must stay unchanged until the current stream has passed this call."""
        t = self._torch
        if not (isinstance(src, t.Tensor) and src.device.type == "cpu" and src.dtype == t.float32 and src.dim() == 2
                and src.is_contiguous()):
            raise ValueError("src must be a contiguous float32 host tensor [n_b, d]")
        n_b, d = int(src.shape[0]), int(src.shape[1])
        dp = self._dev(dst, t.float32, (None, d), "dst")
        wrote = ctypes.c_int64(0)
        self._call("b2k_ingest_append", dp, int(dst.shape[0]), d, int(row0), src.data_ptr(), None, n_b, 0, LAYOUT_ROWS,
                   after=(ctypes.byref(wrote),))
        return int(wrote.value)

    def ingest_columns(self, dst: Any, row0: int, columns: Sequence[np.ndarray]) -> int:
        """Append d scalar host columns (multi-column feature layout, core.py:910)."""
        d = len(columns)
        dt = columns[0].dtype
        code = _DTYPE_CODES.get(dt)
        if code is None:
            raise TypeError(f"unsupported source dtype {dt}")
        n_b = int(columns[0].shape[0])
        cols = [np.ascontiguousarray(c) for c in columns]
        for c in cols:
            if c.dtype != dt or c.shape != (n_b,):
                raise ValueError("columns must share dtype and length")
        dp = self._dev(dst, self._torch.float32, (None, d), "dst")
        ptrs = (ctypes.c_void_p * d)(*[c.ctypes.data for c in cols])
        wrote = ctypes.c_int64(0)
        self._call("b2k_ingest_append", dp, int(dst.shape[0]), d, int(row0), ctypes.addressof(ptrs), None, n_b, code,
                   LAYOUT_COLUMNS, after=(ctypes.byref(wrote),))
        self._torch.cuda.current_stream(self.device).synchronize()  # cols/ptrs must outlive the staging copies
        return int(wrote.value)

    # -- compute ----------------------------------------------------------------------------
    def kmeans_fit(self, X: Any, k: int, *, init: Any = "scalable-k-means++", max_iter: int = 300,
                   tol: float = 1e-4, seed: int = 0, oversampling_factor: float = 2.0, n_init: int = 1,
                   compute_inertia: bool = True) -> Dict[str, Any]:
        """KMeansMG(**cuml_init).fit(X) equivalent.  Returns dict(cluster_centers_ [k,d] cuda tensor,
        n_iter_, inertia_)."""
        t = self._torch
        Xp, n, d = self._check_X(X)
        if isinstance(init, str):
            mode = {"scalable-k-means++": INIT_KMEANS_PARALLEL, "k-means||": INIT_KMEANS_PARALLEL,
                    "random": INIT_RANDOM}.get(init)
            if mode is None:
                raise ValueError(f"unknown init {init!r}")
            init_p = None
        else:
            keep = t.as_tensor(init, dtype=t.float32, device=self.device).contiguous()
            init_p = self._dev(keep, t.float32, (int(k), d), "init")
            mode = INIT_ARRAY
        centers, cp = self._empty((int(k), d), t.float32)
        n_iter = ctypes.c_int(0)
        inertia = ctypes.c_double(0.0)
        self._call("b2k_kmeans_fit", Xp, n, d, int(k), mode, init_p, int(max_iter), float(tol), _u64(seed),
                   float(oversampling_factor), int(n_init), cp, ctypes.byref(n_iter),
                   ctypes.byref(inertia) if compute_inertia else None)
        return {"cluster_centers_": centers, "n_iter_": int(n_iter.value),
                "inertia_": float(inertia.value) if compute_inertia else None}

    def kmeans_lloyd(self, X: Any, centers: Any, max_iter: int, tol: float) -> Tuple[int, float]:
        """Lloyd loop in place on `centers` (cuda f32 [k,d]); returns (n_iter, last shift)."""
        Xp, n, d = self._check_X(X)
        cp = self._dev(centers, self._torch.float32, (None, d), "centers")
        n_iter = ctypes.c_int(0)
        shift = ctypes.c_double(0.0)
        self._call("b2k_kmeans_lloyd", Xp, n, d, int(centers.shape[0]), cp, int(max_iter), float(tol),
                   ctypes.byref(n_iter), ctypes.byref(shift))
        return int(n_iter.value), float(shift.value)

    def kmeans_assign(self, X: Any, centers: Any, want_mindist: bool = False) -> Tuple[Any, Any]:
        """KMeans.predict equivalent: int32 labels (and optionally squared min distances)."""
        t = self._torch
        Xp, n, d = self._check_X(X)
        C = t.as_tensor(centers, dtype=t.float32, device=self.device).contiguous()
        cp = self._dev(C, t.float32, (None, d), "centers")
        labels, lp = self._empty((n,), t.int32)
        md, mp = self._empty((n,), t.float32) if want_mindist else (None, None)
        self._call("b2k_kmeans_assign", Xp, n, d, cp, int(C.shape[0]), lp, mp)
        t.cuda.current_stream(self.device).synchronize()  # C (a temporary) must outlive the kernels
        return labels, md

    def pca_fit(self, X: Any, k: int) -> Dict[str, np.ndarray]:
        """PCAMG(n_components=k).fit(X) equivalent (collective when a communicator is initialised).  Returns host float64
        arrays: mean_ [d], components_ [k, d], explained_variance_ratio_ [k], singular_values_ [k]."""
        Xp, n, d = self._check_X(X)
        kk = max(int(k), 0)
        mean = np.zeros(d, dtype=np.float64)
        comp = np.zeros((kk, d), dtype=np.float64)
        evr = np.zeros(kk, dtype=np.float64)
        sv = np.zeros(kk, dtype=np.float64)
        self._call("b2k_pca_fit", Xp, n, d, int(k), mean.ctypes.data, comp.ctypes.data, evr.ctypes.data, sv.ctypes.data)
        return {"mean_": mean, "components_": comp, "explained_variance_ratio_": evr, "singular_values_": sv}

    def pca_transform(self, X: Any, components: Any) -> Any:
        """PCAModel.transform equivalent: X [n, d] . components^T -> float32 CUDA tensor [n, k] (no mean subtracted)."""
        t = self._torch
        Xp, n, d = self._check_X(X)
        C = t.as_tensor(components, dtype=t.float32, device=self.device).contiguous()
        cp = self._dev(C, t.float32, (None, d), "components")
        k = int(C.shape[0])
        out, op = self._empty((n, k), t.float32)
        self._call("b2k_pca_transform", Xp, n, d, cp, k, op)
        t.cuda.current_stream(self.device).synchronize()  # C (possibly a temporary) must outlive the kernel
        return out

    def knn_search(self, items: Any, queries: Any, k: int, item_ids: Any = None) -> Tuple[Any, Any]:
        """NearestNeighborsMG.kneighbors equivalent (collective when a communicator is initialised): the k nearest of all
        ranks' items for each of this rank's queries.  items [n_items, d] and queries [n_q, d] are float32 CUDA tensors
        (either may have 0 rows), item_ids an int64 CUDA tensor [n_items] or None (ids = global rows).  Returns CUDA
        tensors distances float32 [n_q, k] (Euclidean, ascending) and indices int64 [n_q, k] (ids)."""
        t = self._torch
        ip, n, d = self._check_X(items, "items")
        qp, nq, dq = self._check_X(queries, "queries")
        if dq != d:
            raise ValueError(f"queries have {dq} features, items {d}")
        idp = self._dev(item_ids, t.int64, (n,), "item_ids", optional=True)
        kk = max(int(k), 0)
        dist, dp = self._empty((nq, kk), t.float32)
        idx, xp = self._empty((nq, kk), t.int64)
        self._call("b2k_knn_search", ip, n, idp, qp, nq, d, int(k), dp, xp)
        return dist, idx

    IVF_METRICS = {"euclidean": 0, "l2": 0, "sqeuclidean": 1}

    def ivf_search(self, items: Any, queries: Any, k: int, nlist: int, nprobe: int, item_ids: Any = None,
                   centers: Any = None, n_iters: int = 20, train_fraction: float = 0.5, metric: str = "euclidean",
                   return_lists: bool = False) -> Tuple[Any, ...]:
        """IVF-Flat search (b2k_ivf_search; collective when a communicator is initialised): the k nearest items of each
        of this rank's queries among the items of its nprobe nearest lists.  Arguments as for knn_search; centers is a
        float32 CUDA tensor [nlist, d] used as given, or None to train them on all ranks' items.  Returns (distances,
        indices, centers) as CUDA tensors, plus (item lists int32 [n_items], probes int32 [n_q, min(nprobe, nlist)])
        with return_lists."""
        t = self._torch
        ip, n, d = self._check_X(items, "items")
        qp, nq, dq = self._check_X(queries, "queries")
        if dq != d:
            raise ValueError(f"queries have {dq} features, items {d}")
        if metric not in self.IVF_METRICS:
            raise ValueError(f"metric {metric!r} is not supported by IVF-Flat (supported: {sorted(self.IVF_METRICS)})")
        idp = self._dev(item_ids, t.int64, (n,), "item_ids", optional=True)
        train = centers is None
        self._dev(centers, t.float32, (int(nlist), d), "centers", optional=True)
        nl = max(int(nlist), 1)
        kk = max(int(k), 0)
        npr = max(min(int(nprobe), nl), 0)
        if train:
            C, Cp = self._empty((nl, d), t.float32)
        else:
            C = centers.clone()
            Cp = self._dev(C, t.float32, (int(nlist), d), "centers")
        dist, dp = self._empty((nq, kk), t.float32)
        idx, xp = self._empty((nq, kk), t.int64)
        lists, lp = self._empty((n,), t.int32) if return_lists else (None, None)
        probes, pp = self._empty((nq, npr), t.int32) if return_lists else (None, None)
        self._call("b2k_ivf_search", ip, n, idp, qp, nq, d, int(k), int(nlist), int(nprobe), int(n_iters),
                   float(train_fraction), self.IVF_METRICS[metric], int(train), Cp, lp, pp, dp, xp)
        return (dist, idx, C, lists, probes) if return_lists else (dist, idx, C)

    def linreg_moments(self, X: Any, y: Any) -> Tuple[int, np.ndarray, np.ndarray]:
        """The passes over the data of a linear regression fit (collective when a communicator is initialised): X [n, d]
        and y [n] float32 CUDA tensors -> (n_total, mean [d + 1], centred moments [d + 1, d + 1] of [X | y]), host
        float64."""
        Xp, n, d = self._check_X(X)
        yp = self._dev(y, self._torch.float32, (n,), "y")
        n_total = ctypes.c_int64(0)
        mean = np.zeros(d + 1, dtype=np.float64)
        mom = np.zeros((d + 1, d + 1), dtype=np.float64)
        self._call("b2k_linreg_moments", Xp, yp, n, d, ctypes.byref(n_total), mean.ctypes.data, mom.ctypes.data)
        return int(n_total.value), mean, mom

    def linreg_predict(self, X: Any, coef: Any, intercept: float) -> Any:
        """intercept + X . coef, accumulated in fp64 -> float64 CUDA tensor [n]."""
        t = self._torch
        Xp, n, d = self._check_X(X)
        w = t.as_tensor(coef, dtype=t.float64, device=self.device).contiguous()
        wp = self._dev(w, t.float64, (d,), "coef")
        out, op = self._empty((n,), t.float64)
        self._call("b2k_linreg_predict", Xp, n, d, wp, float(intercept), op)
        t.cuda.current_stream(self.device).synchronize()  # w (possibly a temporary) must outlive the kernel
        return out

    # -- Gaussian mixtures ------------------------------------------------------------------
    def gmm_fit(self, X: Any, k: int, *, init: Optional[Tuple[Any, Any, Any]] = None, max_iter: int = 100,
                tol: float = 0.01, seed: int = 0) -> Dict[str, Any]:
        """GaussianMixture.fit (b2k_gmm_fit, collective when a communicator is initialised).  init = None draws the
        start from `seed`, or (weights [k], means [k, d], covariances [k, d, d]) starts from those values.  Returns host
        float64 arrays weights [k], means [k, d], covs [k, d, d], int64 cluster_sizes [k], and log_likelihood, n_iter."""
        Xp, n, d = self._check_X(X)
        kk = max(int(k), 0)
        init_p: List[Optional[int]] = [None, None, None]
        if init is not None:
            iw = _host(np.ravel(init[0]), np.float64, (kk,), "init weights")
            im = _host(init[1], np.float64, (kk, d), "init means")
            ic = _host(init[2], np.float64, (kk, d, d), "init covariances")
            init_p = [iw.ctypes.data, im.ctypes.data, ic.ctypes.data]
        w = np.zeros(kk, dtype=np.float64)
        mu = np.zeros((kk, d), dtype=np.float64)
        cov = np.zeros((kk, d, d), dtype=np.float64)
        sizes = np.zeros(kk, dtype=np.int64)
        ll = ctypes.c_double(0.0)
        n_iter = ctypes.c_int(0)
        self._call("b2k_gmm_fit", Xp, n, d, int(k), INIT_RANDOM if init is None else INIT_ARRAY, *init_p, int(max_iter),
                   float(tol), _u64(seed), w.ctypes.data, mu.ctypes.data, cov.ctypes.data, ctypes.byref(ll),
                   ctypes.byref(n_iter), sizes.ctypes.data)
        return {"weights": w, "means": mu, "covs": cov, "cluster_sizes": sizes, "log_likelihood": float(ll.value),
                "n_iter": int(n_iter.value)}

    def gmm_predict(self, X: Any, weights: Any, means: Any, covs: Any) -> Tuple[Any, Any]:
        """Per row of X: the float64 probabilities [n, k] and the int32 argmax [n] of a Gaussian mixture (CUDA
        tensors)."""
        t = self._torch
        Xp, n, d = self._check_X(X)
        w = _host(np.ravel(weights), np.float64, (None,), "weights")
        k = int(w.shape[0])
        mu = _host(means, np.float64, (k, d), "means")
        cov = _host(covs, np.float64, (k, d, d), "covs")
        prob, pp = self._empty((n, k), t.float64)
        labels, lp = self._empty((n,), t.int32)
        self._call("b2k_gmm_predict", Xp, n, d, k, w.ctypes.data, mu.ctypes.data, cov.ctypes.data, pp, lp)
        return prob, labels

    # -- bisecting k-means -------------------------------------------------------------------
    def bkm_fit(self, X: Any, k: int, *, max_iter: int = 20, min_divisible: float = 1.0, seed: int = 0
                ) -> Dict[str, Any]:
        """BisectingKMeans.fit (b2k_bkm_fit, collective when a communicator is initialised).  Returns the tree in
        depth-first order as host arrays node_index int64 [m], centers float64 [m, d], sizes int64 [m], costs float64
        [m]; training_cost; cluster_sizes int64 [leaves]; n_levels; level_ms float64 [n_levels] (zeros unless option
        time_kernels is set)."""
        Xp, n, d = self._check_X(X)
        kk = max(int(k), 1)
        m = 2 * kk - 1
        idx = np.zeros(m, dtype=np.int64)
        cen = np.zeros((m, max(d, 1)), dtype=np.float64)
        sizes = np.zeros(m, dtype=np.int64)
        costs = np.zeros(m, dtype=np.float64)
        csz = np.zeros(kk, dtype=np.int64)
        lms = np.zeros(BKM_MAX_LEVELS, dtype=np.float64)
        nn = ctypes.c_int(0)
        tc = ctypes.c_double(0.0)
        self._call("b2k_bkm_fit", Xp, n, d, int(k), int(max_iter), float(min_divisible), _u64(seed), ctypes.byref(nn),
                   idx.ctypes.data, cen.ctypes.data, sizes.ctypes.data, costs.ctypes.data, ctypes.byref(tc),
                   csz.ctypes.data, lms.ctypes.data)
        nn = int(nn.value)
        idx, cen = idx[:nn], cen.reshape(-1)[: nn * d].reshape(nn, d)
        ids = set(idx.tolist())
        n_leaves = sum(1 for i in ids if 2 * i not in ids and 2 * i + 1 not in ids)
        levels = int(self.stats()["last_n_iter"])
        return {"node_index": idx, "centers": cen, "sizes": sizes[:nn], "costs": costs[:nn],
                "training_cost": float(tc.value), "cluster_sizes": csz[:n_leaves], "n_levels": levels,
                "level_ms": lms[:levels]}

    def bkm_predict(self, X: Any, node_index: Any, node_centers: Any, *, with_cost: bool = False
                    ) -> Tuple[Any, Optional[Any]]:
        """Per row of X the int32 leaf (depth-first number) reached by descent and, with with_cost, the float64
        squared distance to that leaf's centre (CUDA tensors; the cost is None otherwise)."""
        t = self._torch
        Xp, n, d = self._check_X(X)
        idx = _host(np.ravel(node_index), np.int64, (None,), "node_index")
        cen = _host(node_centers, np.float64, (idx.shape[0], d), "node_centers")
        labels, lp = self._empty((n,), t.int32)
        cost, cp = self._empty((n,), t.float64) if with_cost else (None, None)
        self._call("b2k_bkm_predict", Xp, n, d, int(idx.shape[0]), idx.ctypes.data, cen.ctypes.data, lp, cp)
        return labels, cost

    # -- multilayer perceptron ----------------------------------------------------------------
    @staticmethod
    def _mlp_layers(layers: Sequence[int], d: int) -> Tuple[np.ndarray, int]:
        lay = np.ascontiguousarray([int(v) for v in layers], dtype=np.int32)
        if lay.size >= 1 and int(lay[0]) != d:
            raise ValueError(f"layers[0] = {int(lay[0])} must equal the feature count {d}")
        P = sum(int(lay[i]) * (int(lay[i - 1]) + 1) for i in range(1, lay.size))
        return lay, P

    def mlp_eval(self, X: Any, y: Any, layers: Sequence[int], weights: Any) -> Tuple[float, np.ndarray, int]:
        """One loss-and-gradient evaluation (collective): F(w) and its gradient [P] in Spark's flat layout, n_total."""
        Xp, n, d = self._check_X(X)
        yp = self._dev(y, self._torch.float32, (n,), "y")
        lay, P = self._mlp_layers(layers, d)
        w = _host(np.ravel(weights), np.float64, (P,), "weights")
        f = ctypes.c_double(0.0)
        g = np.zeros(P, dtype=np.float64)
        nt = ctypes.c_int64(0)
        self._call("b2k_mlp_eval", Xp, yp, n, lay.ctypes.data, int(lay.size), w.ctypes.data, ctypes.byref(f),
                   g.ctypes.data, ctypes.byref(nt))
        return float(f.value), g, int(nt.value)

    def mlp_fit(self, X: Any, y: Any, layers: Sequence[int], *, solver: str = "l-bfgs", max_iter: int = 100,
                tol: float = 1e-6, step_size: float = 0.03, seed: int = 0, initial_weights: Any = None
                ) -> Dict[str, Any]:
        """MultilayerPerceptronClassifier.fit (b2k_mlp_fit, collective) -> weights [P], objective_history, n_iter."""
        Xp, n, d = self._check_X(X)
        yp = self._dev(y, self._torch.float32, (n,), "y")
        lay, P = self._mlp_layers(layers, d)
        if solver not in MLP_SOLVERS:
            raise ValueError(f"solver must be one of {sorted(MLP_SOLVERS)}, got {solver!r}")
        w0 = None if initial_weights is None else _host(np.ravel(initial_weights), np.float64, (P,), "initialWeights")
        w = np.zeros(P, dtype=np.float64)
        hist = np.zeros(max(int(max_iter), 0) + 1, dtype=np.float64)
        it = ctypes.c_int(0)
        self._call("b2k_mlp_fit", Xp, yp, n, lay.ctypes.data, int(lay.size), MLP_SOLVERS[solver], int(max_iter),
                   float(tol), float(step_size), _u64(seed), w0.ctypes.data if w0 is not None else None, w.ctypes.data,
                   hist.ctypes.data, ctypes.byref(it))
        return {"weights": w, "objective_history": hist[: it.value].copy(), "n_iter": int(it.value)}

    def mlp_predict(self, X: Any, layers: Sequence[int], weights: Any) -> Tuple[Any, Any, Any]:
        """rawPrediction [n, C], probability [n, C] and prediction [n] as float64 CUDA tensors."""
        t = self._torch
        Xp, n, d = self._check_X(X)
        lay, P = self._mlp_layers(layers, d)
        w = _host(np.ravel(weights), np.float64, (P,), "weights")
        C = int(lay[-1]) if lay.size else 0
        raw, rp = self._empty((n, C), t.float64)
        prob, pp = self._empty((n, C), t.float64)
        pred, dp = self._empty((n,), t.float64)
        self._call("b2k_mlp_predict", Xp, n, lay.ctypes.data, int(lay.size), w.ctypes.data, rp, pp, dp)
        return raw, prob, pred

    # -- ALS ------------------------------------------------------------------------------------
    def als_fit(self, users: Any, items: Any, ratings: Any, *, rank: int = 10, max_iter: int = 10,
                reg_param: float = 0.1, implicit_prefs: bool = False, alpha: float = 1.0, seed: int = 0,
                init_user_factors: Any = None) -> Dict[str, Any]:
        """ALS.fit (b2k_als_fit, collective): users / items float64 and ratings float32 (or None: every rating 1.0)
        CUDA tensors of this rank's triples -> user_ids [U] int32, user_factors [U, rank] float32, item_ids [I],
        item_factors [I, rank] (CUDA tensors, sorted by id).  init_user_factors: [U, rank] float32 in user-id order."""
        t = self._torch
        up = self._dev(users, t.float64, (None,), "users")
        n = int(users.shape[0])
        ip = self._dev(items, t.float64, (n,), "items")
        rp = self._dev(ratings, t.float32, (n,), "ratings", optional=True)
        w0, nw = None, 0
        if init_user_factors is not None:
            w0 = _host(init_user_factors, np.float32, (None, int(rank)), "init_user_factors")
            nw = int(w0.shape[0])
        nu, ni = ctypes.c_int64(0), ctypes.c_int64(0)
        cap_u = cap_i = max(min(n, 1 << 20), nw, 1)
        for _ in range(2):   # a cap too small fails on every rank with the sizes set: every rank calls again with them
            uid, uidp = self._empty((max(cap_u, 1),), t.int32)
            uf, ufp = self._empty((max(cap_u, 1), int(rank)), t.float32)
            iid, iidp = self._empty((max(cap_i, 1),), t.int32)
            itf, itfp = self._empty((max(cap_i, 1), int(rank)), t.float32)
            rc = self._invoke("b2k_als_fit", up if n else None, ip if n else None, rp if n else None, n, int(rank),
                              int(max_iter), float(reg_param), int(bool(implicit_prefs)), float(alpha), _u64(seed),
                              w0.ctypes.data if w0 is not None else None, nw, cap_u, cap_i, uidp, ufp, iidp, itfp,
                              ctypes.byref(nu), ctypes.byref(ni))
            if rc != B2K_OK and (self._L.b2k_last_error(self._h) or b"").startswith(b"ALS: the outputs hold fewer"):
                cap_u, cap_i = max(cap_u, nu.value), max(cap_i, ni.value)
                continue
            self._check(rc)
            break
        U, I = int(nu.value), int(ni.value)
        return {"user_ids": uid[:U], "user_factors": uf[:U], "item_ids": iid[:I], "item_factors": itf[:I]}

    def als_predict(self, users: Any, items: Any, user_ids: Any, user_factors: Any, item_ids: Any,
                    item_factors: Any) -> Any:
        """ALSModel.transform's prediction (b2k_als_predict): float32 [n], NaN for an unknown id."""
        t = self._torch
        up = self._dev(users, t.float64, (None,), "users")
        n = int(users.shape[0])
        ip = self._dev(items, t.float64, (n,), "items")
        uidp = self._dev(user_ids, t.int32, (None,), "user_ids")
        nu = int(user_ids.shape[0])
        ufp = self._dev(user_factors, t.float32, (nu, None), "user_factors")
        rank = int(user_factors.shape[1])
        iidp = self._dev(item_ids, t.int32, (None,), "item_ids")
        ni = int(item_ids.shape[0])
        ifp = self._dev(item_factors, t.float32, (ni, rank), "item_factors")
        out, op = self._empty((n,), t.float32)
        self._call("b2k_als_predict", up, ip, n, rank, uidp, ufp, nu, iidp, ifp, ni, op)
        return out

    def als_recommend(self, Q: Any, T: Any, n: int) -> Tuple[Any, Any]:
        """The n best rows of T [nt, rank] for each row of Q [nq, rank] (b2k_als_recommend): row indices [nq, n] int32
        (-1 past nt) and scores [nq, n] float32, score descending, the lower row first on a tie."""
        t = self._torch
        qp = self._dev(Q, t.float32, (None, None), "Q")
        nq, rank = int(Q.shape[0]), int(Q.shape[1])
        tp = self._dev(T, t.float32, (None, rank), "T")
        nt = int(T.shape[0])
        idx, xp = self._empty((nq, int(n)), t.int32)
        sc, sp = self._empty((nq, int(n)), t.float32)
        self._call("b2k_als_recommend", qp if nq else None, nq, tp if nt else None, nt, rank, int(n), xp, sp)
        return idx, sc

    # -- logistic regression ----------------------------------------------------------------
    def logreg_labels(self, y: Any) -> Tuple[np.ndarray, np.ndarray, int]:
        """The label pass (collective): y [n] float32 CUDA tensor -> (classes float64 [K], counts int64 [K], n_total)."""
        yp = self._dev(y, self._torch.float32, (None,), "y")
        cls = np.zeros(1024, dtype=np.float64)
        cnt = np.zeros(1024, dtype=np.int64)
        k, nt = ctypes.c_int(0), ctypes.c_int64(0)
        self._call("b2k_logreg_labels", yp, int(y.shape[0]), cls.ctypes.data, cnt.ctypes.data, ctypes.byref(k),
                   ctypes.byref(nt))
        return cls[: k.value].copy(), cnt[: k.value].copy(), int(nt.value)

    @staticmethod
    def _logreg_W(W: Any, b: Any, d: int) -> Tuple[np.ndarray, np.ndarray, int]:
        """Host float64 W [kp, d] and b [kp] of a logistic model, and kp."""
        W = _host(W, np.float64, (None, d), "W")
        kp = int(W.shape[0])
        return W, _host(b, np.float64, (kp,), "b"), kp

    def _logreg_eval(self, fn: str, data: Sequence[Any], d: int, classes: Sequence[float], W: Any, b: Any
                     ) -> Tuple[float, np.ndarray, np.ndarray, int]:
        """logreg_eval through the entry point fn; data: its (checked) arguments before classes."""
        cls = _host(classes, np.float64, (None,), "classes")
        W, b, kp = self._logreg_W(W, b, d)
        loss = ctypes.c_double(0.0)
        grad = np.zeros((kp, d + 1), dtype=np.float64)
        nt = ctypes.c_int64(0)
        self._call(fn, *data, cls.ctypes.data, int(cls.size), kp, W.ctypes.data, b.ctypes.data, ctypes.byref(loss),
                   grad.ctypes.data, ctypes.byref(nt))
        return float(loss.value), grad[:, :d].copy(), grad[:, d].copy(), int(nt.value)

    def _logreg_fit(self, fn: str, data: Sequence[Any], d: int, classes: np.ndarray, counts: np.ndarray,
                    settings: Sequence[Dict[str, Any]]) -> List[Tuple[np.ndarray, np.ndarray, int]]:
        """logreg_fit through the entry point fn; data: its (checked) arguments before classes."""
        cls = _host(classes, np.float64, (None,), "classes")
        K, m = int(cls.size), len(settings)
        cnt = _host(counts, np.int64, (K,), "counts")
        prm = (LogregParams * m)(*[LogregParams(float(s["reg"]), float(s["l1_ratio"]), float(s["tol"]),
                                                int(s["max_iter"]), int(bool(s["fit_intercept"])),
                                                int(bool(s["standardization"])), FAMILY_CODES[s["family"]])
                                   for s in settings])
        coef = np.zeros((m, K, d), dtype=np.float64)
        icpt = np.zeros((m, K), dtype=np.float64)
        kp = np.zeros(m, dtype=np.int32)
        it = np.zeros(m, dtype=np.int32)
        self._call(fn, *data, cls.ctypes.data, cnt.ctypes.data, K, m, prm, coef.ctypes.data, icpt.ctypes.data,
                   kp.ctypes.data, it.ctypes.data)
        return [(coef[f, : kp[f]].copy(), icpt[f, : kp[f]].copy(), int(it[f])) for f in range(m)]

    def _logreg_model(self, W: Any, b: Any, class_values: Sequence[float], d: int
                      ) -> Tuple[int, List[Any], List[Any]]:
        """nout, the device copies of W [kp, d], b [kp] and class_values [nout] of a logistic model (nout = 2 for a
        binomial W [1, d]), and the predict entry points' arguments kp, W, b, class values."""
        t = self._torch
        W, b, kp = self._logreg_W(W, b, d)
        nout = 2 if kp == 1 else kp
        cv = _host(class_values, np.float64, (nout,), "class_values")
        dev = [t.as_tensor(a, device=self.device) for a in (W, b, cv)]
        return nout, dev, [kp] + [self._dev(x, t.float64, x.shape, name)
                                  for x, name in zip(dev, ("W", "b", "class_values"))]

    def logreg_eval(self, X: Any, y: Any, classes: Sequence[float], W: np.ndarray, b: np.ndarray
                    ) -> Tuple[float, np.ndarray, np.ndarray, int]:
        """One loss-and-gradient evaluation (collective): (1/n) sum loss and its gradient at W [kp, d], b [kp] (no
        penalty) -> (loss, dW [kp, d], db [kp], n_total)."""
        Xp, n, d = self._check_X(X)
        yp = self._dev(y, self._torch.float32, (n,), "y")
        return self._logreg_eval("b2k_logreg_eval", (Xp, yp, n, d), d, classes, W, b)

    def logreg_fit(self, X: Any, y: Any, classes: np.ndarray, counts: np.ndarray, settings: Sequence[Dict[str, Any]]
                   ) -> List[Tuple[np.ndarray, np.ndarray, int]]:
        """Fits (collective), one per setting dict (reg, l1_ratio, tol, max_iter, fit_intercept, standardization,
        family) from one column-moments pass -> [(coef [kp, d], intercept [kp], iterations)]."""
        Xp, n, d = self._check_X(X)
        yp = self._dev(y, self._torch.float32, (n,), "y")
        return self._logreg_fit("b2k_logreg_fit", (Xp, yp, n, d), d, classes, counts, settings)

    def logreg_predict(self, X: Any, W: Any, b: Any, class_values: Sequence[float]) -> Tuple[Any, Any, Any]:
        """rawPrediction [n, nout], probability [n, nout] and prediction [n] as float64 CUDA tensors (nout = 2 for a
        binomial W [1, d])."""
        t = self._torch
        Xp, n, d = self._check_X(X)
        nout, (Wd, bd, cv), model = self._logreg_model(W, b, class_values, d)
        raw, rp = self._empty((n, nout), t.float64)
        prob, pp = self._empty((n, nout), t.float64)
        pred, dp = self._empty((n,), t.float64)
        self._call("b2k_logreg_predict", Xp, n, d, *model, rp, pp, dp)
        t.cuda.current_stream(self.device).synchronize()  # Wd, bd, cv (temporaries) must outlive the kernel
        return raw, prob, pred

    # -- sparse logistic regression: rows as a device CSR (indptr int64 [n + 1], indices int32, values float32) --------
    def _check_csr(self, X: Any, d: int) -> Tuple[List[int], int, int]:
        """The addresses of the CSR triple X = (indptr [n + 1], indices [nnz], values [nnz]) of width d, n and nnz."""
        t = self._torch
        indptr, indices, values = X
        ptrs = [self._dev(indptr, t.int64, (None,), "indptr"), self._dev(indices, t.int32, (None,), "indices")]
        nnz = int(indices.shape[0])
        ptrs.append(self._dev(values, t.float32, (nnz,), "values"))
        if indptr.shape[0] < 1:
            raise ValueError("indptr must hold n + 1 >= 1 offsets")
        if int(d) < 1:
            raise ValueError("d must be >= 1")
        return ptrs, int(indptr.shape[0]) - 1, nnz

    def ingest_csr(self, indptr: Any, indices: Any, values: Any, d: int, row0: int, nnz0: int, type_: np.ndarray,
                   size: np.ndarray, idx_offsets: np.ndarray, idx_values: np.ndarray, val_offsets: np.ndarray,
                   val_values: np.ndarray) -> int:
        """Append one batch of Spark vector rows, given by the Arrow child buffers of its struct column, at rows
        [row0, row0 + n_b) and entries [nnz0, ...) of the device CSR -> the batch's entry count."""
        code = _DTYPE_CODES.get(val_values.dtype)
        if code not in (0, 1):
            raise TypeError(f"unsupported vector value dtype {val_values.dtype}")
        ptrs, n_max, nnz_max = self._check_csr((indptr, indices, values), d)
        tp = _host(type_, np.int8, (None,), "type")
        n_b = int(tp.shape[0])
        arrs = [tp, _host(size, np.int32, (n_b,), "size"), _host(idx_offsets, np.int32, (n_b + 1,), "idx_offsets"),
                _host(idx_values, np.int32, (None,), "idx_values"),
                _host(val_offsets, np.int32, (n_b + 1,), "val_offsets"),
                _host(val_values, val_values.dtype, (None,), "val_values")]
        wrote = ctypes.c_int64(0)
        self._call("b2k_ingest_csr_append", *ptrs, n_max, nnz_max, int(d), int(row0), int(nnz0),
                   *[a.ctypes.data for a in arrs], code, n_b, after=(ctypes.byref(wrote),))
        return int(wrote.value)

    def logreg_eval_csr(self, X: Any, d: int, y: Any, classes: Sequence[float], W: np.ndarray, b: np.ndarray
                        ) -> Tuple[float, np.ndarray, np.ndarray, int]:
        """logreg_eval on CSR rows X = (indptr, indices, values) of width d (collective; builds its own CSC)."""
        ptrs, n, nnz = self._check_csr(X, d)
        yp = self._dev(y, self._torch.float32, (n,), "y")
        return self._logreg_eval("b2k_logreg_eval_csr", (*ptrs, n, nnz, int(d), yp), int(d), classes, W, b)

    def logreg_fit_csr(self, X: Any, d: int, y: Any, classes: np.ndarray, counts: np.ndarray,
                       settings: Sequence[Dict[str, Any]]) -> List[Tuple[np.ndarray, np.ndarray, int]]:
        """logreg_fit on CSR rows X = (indptr, indices, values) of width d: one CSC and one moments pass for every
        setting (collective)."""
        ptrs, n, nnz = self._check_csr(X, d)
        yp = self._dev(y, self._torch.float32, (n,), "y")
        return self._logreg_fit("b2k_logreg_fit_csr", (*ptrs, n, nnz, int(d), yp), int(d), classes, counts, settings)

    def logreg_predict_csr(self, X: Any, d: int, W: Any, b: Any, class_values: Sequence[float]
                           ) -> Tuple[Any, Any, Any]:
        """logreg_predict on CSR rows X = (indptr, indices, values) of width d."""
        t = self._torch
        ptrs, n, nnz = self._check_csr(X, d)
        nout, (Wd, bd, cv), model = self._logreg_model(W, b, class_values, int(d))
        raw, rp = self._empty((n, nout), t.float64)
        prob, pp = self._empty((n, nout), t.float64)
        pred, dp = self._empty((n,), t.float64)
        self._call("b2k_logreg_predict_csr", *ptrs, n, nnz, int(d), *model, rp, pp, dp)
        t.cuda.current_stream(self.device).synchronize()  # Wd, bd, cv (temporaries) must outlive the kernel
        return raw, prob, pred

    # -- DBSCAN -----------------------------------------------------------------------------
    def dbscan_fit(self, X: Any, eps: float, min_samples: int, metric: str = "euclidean") -> Tuple[Any, Any, int]:
        """DBSCAN over all ranks' rows (collective when a communicator is initialised): X [n, d] float32 CUDA tensor (may
        have 0 rows) -> (labels int32 [n], core flags bool [n], both CUDA tensors for this rank's rows, and the number of
        clusters).  metric is "euclidean" or "cosine"."""
        t = self._torch
        Xp, n, d = self._check_X(X)
        if metric not in METRIC_CODES:
            raise ValueError(f"metric must be one of {sorted(METRIC_CODES)}, got {metric!r}")
        labels, lp = self._empty((n,), t.int32)
        core, cp = self._empty((n,), t.uint8)
        ncl = ctypes.c_int64(0)
        self._call("b2k_dbscan_fit", Xp, n, d, float(eps), int(min_samples), METRIC_CODES[metric], lp, cp,
                   ctypes.byref(ncl))
        return labels, core.bool(), int(ncl.value)

    # -- silhouette -------------------------------------------------------------------------
    def silhouette(self, X: Any, cluster_ids: Any, distance_measure: str = "squaredEuclidean") -> float:
        """b2k_silhouette over all ranks' rows (collective when a communicator is initialised): X [n, d] float32 and
        cluster_ids [n] int64 CUDA tensors (n may be 0) -> Spark's silhouette, the same value on every rank.
        distance_measure is "squaredEuclidean" or "cosine"."""
        Xp, n, d = self._check_X(X)
        if distance_measure not in SILHOUETTE_METRICS:
            raise ValueError(f"distance_measure must be one of {sorted(SILHOUETTE_METRICS)}, got {distance_measure!r}")
        ip = self._dev(cluster_ids, self._torch.int64, (n,), "cluster_ids")
        out = ctypes.c_double(0.0)
        self._call("b2k_silhouette", Xp, n, d, ip, SILHOUETTE_METRICS[distance_measure], ctypes.byref(out))
        return float(out.value)

    def silhouette_multi(self, X: Any, ids_list: Sequence[Any], distance_measure: str = "squaredEuclidean") -> List[float]:
        """b2k_silhouette_multi: the silhouette of several clusterings of the same rows (collective when a communicator
        is initialised).  X [n, d] float32 and each of ids_list [n] int64 CUDA tensors -> one value per clustering,
        each with the bits Context.silhouette returns for it; one device pass over X serves the models whose shifts
        agree."""
        Xp, n, d = self._check_X(X)
        if distance_measure not in SILHOUETTE_METRICS:
            raise ValueError(f"distance_measure must be one of {sorted(SILHOUETTE_METRICS)}, got {distance_measure!r}")
        ids_list = list(ids_list)
        if not ids_list:
            raise ValueError("ids_list must hold at least one cluster-id tensor")
        M = len(ids_list)
        ptrs = (ctypes.c_void_p * M)(*[self._dev(ids, self._torch.int64, (n,), f"ids_list[{j}]")
                                       for j, ids in enumerate(ids_list)])
        out = (ctypes.c_double * M)()
        self._call("b2k_silhouette_multi", Xp, n, d, M, ptrs, SILHOUETTE_METRICS[distance_measure], out)
        return [float(v) for v in out]

    # -- random forests ---------------------------------------------------------------------
    def rf_fit(self, X: Any, y: Any, *, n_trees: int = 20, max_depth: int = 5, max_bins: int = 32,
               min_instances: int = 1, features_per_node: Optional[int] = None, bootstrap: bool = True,
               impurity: str = "gini", min_info_gain: float = 0.0, seed: int = 0) -> Dict[str, Any]:
        """A random forest over all ranks' rows (collective when a communicator is initialised): X [n, d] and y [n]
        float32 CUDA tensors (either may have 0 rows on a rank that then fails with every other).  impurity "gini" or
        "entropy" (classification, y the class values) or "variance" (regression).  Returns host arrays:
        tree_offsets int64 [T + 1], feature int32 [N] (-1 for a leaf), threshold float32 [N], children int32 [N, 2],
        gain float64 [N], count int64 [N], value float64 [N, V], and n_values V, level_ms [max_depth + 1] (with option
        time_kernels), level_updates [max_depth + 1]."""
        Xp, n, d = self._check_X(X)
        yp = self._dev(y, self._torch.float32, (n,), "y")
        if impurity not in IMPURITY_CODES:
            raise ValueError(f"impurity must be one of {sorted(IMPURITY_CODES)}, got {impurity!r}")
        prm = RfParams(int(n_trees), int(max_depth), int(max_bins), int(min_instances),
                       int(d if features_per_node is None else features_per_node), int(bool(bootstrap)),
                       IMPURITY_CODES[impurity], 0, float(min_info_gain), _u64(seed))
        nv, nn = ctypes.c_int(0), ctypes.c_int64(0)
        L = max(int(max_depth), 0) + 1
        lms = np.zeros(L, dtype=np.float64)
        lup = np.zeros(L, dtype=np.int64)
        self._call("b2k_rf_fit", Xp, yp, n, d, ctypes.byref(prm), ctypes.byref(nv), ctypes.byref(nn), lms.ctypes.data,
                   lup.ctypes.data)
        V, N, T = int(nv.value), int(nn.value), int(n_trees)
        out = {"tree_offsets": np.zeros(T + 1, dtype=np.int64), "feature": np.zeros(N, dtype=np.int32),
               "threshold": np.zeros(N, dtype=np.float32), "children": np.zeros((N, 2), dtype=np.int32),
               "gain": np.zeros(N, dtype=np.float64), "count": np.zeros(N, dtype=np.int64),
               "value": np.zeros((N, V), dtype=np.float64)}
        self._check(self._L.b2k_rf_forest(self._h, *[out[key].ctypes.data for key in
                                                     ("tree_offsets", "feature", "threshold", "children", "gain",
                                                      "count", "value")]))
        out.update(n_values=V, level_ms=lms, level_updates=lup)
        return out

    def rf_predict(self, X: Any, forest: Dict[str, Any], classification: bool) -> Tuple[Any, Any, Any]:
        """k_rf_predict over X [n, d] with a forest laid out as rf_fit's output -> float64 CUDA tensors rawPrediction
        [n, V], probability [n, V] and prediction [n] (classification; prediction = the class index), or (None, None,
        prediction [n]) for regression."""
        t = self._torch
        Xp, n, d = self._check_X(X)
        host = {key: np.ascontiguousarray(forest[key], dtype=dt) for key, dt in
                (("tree_offsets", np.int64), ("feature", np.int32), ("threshold", np.float32), ("children", np.int32),
                 ("value", np.float64))}
        T, V = int(host["tree_offsets"].size) - 1, int(host["value"].shape[1])
        dev = {key: t.as_tensor(a, device=self.device) for key, a in host.items()}
        ptrs = [self._dev(x, x.dtype, x.shape, key) for key, x in dev.items()]
        raw, rp = self._empty((n, V), t.float64) if classification else (None, None)
        prob, pp = self._empty((n, V), t.float64) if classification else (None, None)
        pred, dp = self._empty((n,), t.float64)
        self._call("b2k_rf_predict", Xp, n, d, T, *ptrs, V, int(bool(classification)), rp, pp, dp)
        return raw, prob, pred

    # -- evaluation -------------------------------------------------------------------------
    def _eval_out(self, m: int, C: int, classification: bool) -> Dict[str, np.ndarray]:
        if classification:
            return {"label_count": np.zeros(max(C, 1), dtype=np.int64), "tp": np.zeros((m, max(C, 1)), dtype=np.int64),
                    "fp": np.zeros((m, max(C, 1)), dtype=np.int64), "loss": np.zeros(m, dtype=np.float64)}
        return {"reg": np.zeros((m, 3, 5), dtype=np.float64)}

    def _eval_result(self, out: Dict[str, np.ndarray], n: int, C: int, classification: bool) -> Dict[str, Any]:
        if classification:
            return {"n": n, "label_count": out["label_count"][:C].copy(), "tp": out["tp"][:, :C].copy(),
                    "fp": out["fp"][:, :C].copy(), "loss": out["loss"]}
        return {"n": n, "reg": out["reg"]}

    def eval_linear(self, X: Any, y: Any, models: Sequence[Dict[str, Any]], eps: float = 1e-15) -> Dict[str, Any]:
        """b2k_eval_linear: M linear models scored on (X [n, d], y [n]) float32 CUDA tensors in one read of X.  Each
        model is a dict: kind ("identity", "logistic" or "softmax"), W [K', d], b [K'] and, for the logistic kinds,
        class_values [2 or K'].  Returns host arrays: classification {n, label_count [C], tp [M, C], fp [M, C],
        loss [M]} (C = 1 + the largest label or class value), regression {n, reg [M, 3, 5]} (columns label,
        label - prediction, prediction; stats count, mean, m2n, m2, l1)."""
        Xp, n, d = self._check_X(X)
        yp = self._dev(y, self._torch.float32, (n,), "y")
        m = len(models)
        kinds, rows, W, b = self._linear_table(models, d)
        classification = bool(kinds[0] != 0)
        cv = (np.ascontiguousarray(np.concatenate([np.asarray(md["class_values"], dtype=np.float64).reshape(-1)
                                                   for md in models])) if classification else np.zeros(1))
        C = self._eval_classes(y, n, int(cv.max()) + 1 if classification and cv.size else 0) if classification else 0
        out = self._eval_out(m, C, classification)
        self._call("b2k_eval_linear", Xp, yp, n, d, m, kinds.ctypes.data, rows.ctypes.data, W.ctypes.data,
                   b.ctypes.data, cv.ctypes.data, C, float(eps), *self._eval_ptrs(out, classification))
        return self._eval_result(out, n, C, classification)

    def eval_forest(self, X: Any, y: Any, forests: Sequence[Dict[str, Any]], classification: bool,
                    eps: float = 1e-15) -> Dict[str, Any]:
        """b2k_eval_forest: M forests (each laid out as rf_fit's output) scored on (X, y) in one read of X.  Returns
        what eval_linear returns."""
        Xp, n, d = self._check_X(X)
        yp = self._dev(y, self._torch.float32, (n,), "y")
        m = len(forests)
        nt, nv, *arrays = self._forest_table(forests)
        C = self._eval_classes(y, n, int(nv.max())) if classification else 0
        out = self._eval_out(m, C, classification)
        self._call("b2k_eval_forest", Xp, yp, n, d, m, int(bool(classification)), nt.ctypes.data, nv.ctypes.data,
                   *[a.ctypes.data for a in arrays], C, float(eps), *self._eval_ptrs(out, classification))
        return self._eval_result(out, n, C, classification)

    @staticmethod
    def _linear_table(models: Sequence[Dict[str, Any]], d: int) -> Tuple[np.ndarray, ...]:
        """kind [M], row_offsets [M + 1], W [rows, d] and b [rows] of b2k_eval_linear's model arguments."""
        kinds = np.array([EVAL_KINDS[md["kind"]] for md in models], dtype=np.int32)
        Ws = [np.ascontiguousarray(md["W"], dtype=np.float64).reshape(-1, d) for md in models]
        rows = np.zeros(len(models) + 1, dtype=np.int32)
        rows[1:] = np.cumsum([w.shape[0] for w in Ws])
        W = np.ascontiguousarray(np.concatenate(Ws, axis=0))
        b = np.ascontiguousarray(np.concatenate([np.asarray(md["b"], dtype=np.float64).reshape(-1) for md in models]))
        return kinds, rows, W, b

    @staticmethod
    def _forest_table(forests: Sequence[Dict[str, Any]]) -> Tuple[np.ndarray, ...]:
        """n_trees, n_values, tree_offsets, feature, threshold, children and value of b2k_eval_forest's arguments."""
        offs = [np.ascontiguousarray(f["tree_offsets"], dtype=np.int64) for f in forests]
        vals = [np.ascontiguousarray(f["value"], dtype=np.float64) for f in forests]
        nt = np.array([o.size - 1 for o in offs], dtype=np.int32)
        nv = np.array([v.shape[1] for v in vals], dtype=np.int32)
        off = np.ascontiguousarray(np.concatenate(offs))
        feat = np.ascontiguousarray(np.concatenate([np.asarray(f["feature"], dtype=np.int32) for f in forests]))
        thr = np.ascontiguousarray(np.concatenate([np.asarray(f["threshold"], dtype=np.float32) for f in forests]))
        ch = np.ascontiguousarray(np.concatenate([np.asarray(f["children"], dtype=np.int32).reshape(-1, 2)
                                                  for f in forests]))
        val = np.ascontiguousarray(np.concatenate([v.reshape(-1) for v in vals]))
        return nt, nv, off, feat, thr, ch, val

    # -- binary evaluation ------------------------------------------------------------------
    def binary_buffers(self, n_models: int, n: int) -> Tuple[Any, Any]:
        """Device buffers of the binary scores of n_models models over n rows: scores [M, n] float64 and pos [n] uint8.
        Their n x M x 9 bytes are checked against the device's free memory first."""
        t = self._torch
        need = int(n) * int(n_models) * 9
        free, _ = t.cuda.mem_get_info(self.device)
        if need > free:
            raise MemoryError(f"binary evaluation: the scores of {n_models} models over {n} rows need {need} bytes of "
                              f"device memory, and {free} are free; evaluate fewer rows or fewer models at once")
        return (t.empty((int(n_models), int(n)), dtype=t.float64, device=self.device),
                t.empty((int(n),), dtype=t.uint8, device=self.device))

    def _binary_out(self, scores: Any, pos: Any, m: Optional[int], row0: int, n: int) -> Tuple[int, int, int]:
        """The addresses of column row0 of scores [m, N] float64 and of pos[row0] in pos [N] uint8, and N, once rows
        [row0, row0 + n) are checked to lie inside both."""
        t = self._torch
        sp = self._dev(scores, t.float64, (m, None), "scores")
        N = int(scores.shape[1])
        pp = self._dev(pos, t.uint8, (N,), "pos")
        if not (0 <= row0 and row0 + n <= N):
            raise ValueError(f"scores and pos must hold rows [{row0}, {row0 + n}), and hold {N}")
        return sp + 8 * row0, pp + row0, N

    def binary_scores_linear(self, X: Any, y: Any, models: Sequence[Dict[str, Any]], scores: Any, pos: Any,
                             row0: int = 0) -> None:
        """b2k_eval_linear_scores: scores[i, row0 + r] = rawPrediction[r][1] of logistic model i (kind "logistic" or
        "softmax", as eval_linear takes them) on (X [n, d], y [n]), pos[row0 + r] = y[r] > 0.5; one read of X."""
        Xp, n, d = self._check_X(X)
        yp = self._dev(y, self._torch.float32, (n,), "y")
        m = len(models)
        sp, pp, N = self._binary_out(scores, pos, m, row0, n)
        kinds, rows, W, b = self._linear_table(models, d)
        self._call("b2k_eval_linear_scores", Xp, yp, n, d, m, kinds.ctypes.data, rows.ctypes.data, W.ctypes.data,
                   b.ctypes.data, sp, N, pp)

    def binary_scores_forest(self, X: Any, y: Any, forests: Sequence[Dict[str, Any]], scores: Any, pos: Any,
                             row0: int = 0) -> None:
        """b2k_eval_forest_scores: as binary_scores_linear for classification forests (rf_fit's layout, >= 2 values)."""
        Xp, n, d = self._check_X(X)
        yp = self._dev(y, self._torch.float32, (n,), "y")
        m = len(forests)
        sp, pp, N = self._binary_out(scores, pos, m, row0, n)
        nt, nv, *arrays = self._forest_table(forests)
        self._call("b2k_eval_forest_scores", Xp, yp, n, d, m, nt.ctypes.data, nv.ctypes.data,
                   *[a.ctypes.data for a in arrays], sp, N, pp)

    def eval_binary(self, scores: Any, pos: Any, num_bins: int, metric: str) -> np.ndarray:
        """b2k_eval_binary: areaUnderROC or areaUnderPR of each row of scores [M, n] with the label bits pos [n]
        (Spark's BinaryClassificationMetrics with numBins, the whole list of distinct scores as one partition)."""
        sp, pp, N = self._binary_out(scores, pos, None, 0, 0)
        m = int(scores.shape[0])
        out = np.zeros(m, dtype=np.float64)
        self._call("b2k_eval_binary", sp, pp, N, m, int(num_bins), BINARY_METRICS[metric], out.ctypes.data)
        return out

    def _eval_classes(self, y: Any, n: int, c_models: int) -> int:
        """C = 1 + max(the largest label, the models' largest class); a bad label is reported by the pass itself."""
        if n == 0:
            return c_models
        t = self._torch
        finite = t.isfinite(y)
        mx = float(y[finite].max().item()) if bool(finite.any().item()) else 0.0
        return max(c_models, int(mx) + 1 if 0 <= mx < 1024 and mx == int(mx) else 1)

    @staticmethod
    def _eval_ptrs(out: Dict[str, np.ndarray], classification: bool) -> List[Any]:
        if classification:
            return [out["label_count"].ctypes.data, out["tp"].ctypes.data, out["fp"].ctypes.data,
                    out["loss"].ctypes.data, None]
        return [None, None, None, None, out["reg"].ctypes.data]

    # -- UMAP -------------------------------------------------------------------------------
    def umap_fit(self, X: Any, params: UmapParams, labels: Any = None, init: Any = None) -> Tuple[Any, Dict[str, Any]]:
        """b2k_umap_fit on one GPU: X [n, d] float32 CUDA tensor, labels an int32 CUDA tensor [n] (-1 unknown) or None,
        init a float32 [n, C] start (params.init must then be 2).  Returns (embedding float32 CUDA tensor [n, C],
        info dict: n, k, nnz, epochs, init_used, ritz_residual, max_weight)."""
        t = self._torch
        Xp, n, d = self._check_X(X)
        C = int(params.n_components)
        lp = self._dev(labels, t.int32, (n,), "labels", optional=True)
        start = None if init is None else t.as_tensor(init, dtype=t.float32, device=self.device).reshape(n, C)
        emb, ep = self._empty((n, max(C, 1)), t.float32)
        if start is not None:
            emb.copy_(start)
        info = np.zeros(8, dtype=np.float64)
        self._call("b2k_umap_fit", Xp, n, d, lp, ctypes.byref(params), ep, info.ctypes.data)
        keys = ("n", "k", "nnz", "epochs", "init_used", "ritz_residual", "n_components", "max_weight")
        out = {key: (float(v) if key in ("ritz_residual", "max_weight") else int(v)) for key, v in zip(keys, info)}
        return emb, out

    def umap_graph(self, info: Dict[str, Any]) -> Dict[str, np.ndarray]:
        """The intermediates of the last umap_fit (b2k_umap_graph) as host arrays, sized from its info dict."""
        n, k, nnz, C = info["n"], info["k"], info["nnz"], info["n_components"]
        g = {"knn_idx": np.zeros((n, k), np.int64), "knn_dist": np.zeros((n, k), np.float32),
             "rho": np.zeros(n), "sigma": np.zeros(n), "indptr": np.zeros(n + 1, np.int64),
             "indices": np.zeros(nnz, np.int32), "weights": np.zeros(nnz), "epochs_per_sample": np.zeros(nnz),
             "init": np.zeros((n, C), np.float32), "ritz_values": np.zeros(C), "ritz_vectors": np.zeros((n, C))}
        self._check(self._L.b2k_umap_graph(self._h, *[g[key].ctypes.data for key in
                                                      ("knn_idx", "knn_dist", "rho", "sigma", "indptr", "indices",
                                                       "weights", "epochs_per_sample", "init", "ritz_values",
                                                       "ritz_vectors")]))
        return g

    def umap_transform(self, X_train: Any, embedding: Any, Q: Any, params: UmapParams) -> Any:
        """b2k_umap_transform: Q [nq, d] against the model (X_train [n, d], embedding [n, C], float32 CUDA tensors) ->
        float32 CUDA tensor [nq, C]; params.n_epochs is the transform's epoch count."""
        t = self._torch
        Xp, n, d = self._check_X(X_train, "X_train")
        qp, nq, dq = self._check_X(Q, "Q")
        C = int(params.n_components)
        if dq != d:
            raise ValueError(f"Q has {dq} features, the model {d}")
        ep = self._dev(embedding, t.float32, (n, C), "embedding")
        out, op = self._empty((nq, C), t.float32)
        self._call("b2k_umap_transform", Xp, ep, n, d, qp, nq, ctypes.byref(params), op)
        return out
