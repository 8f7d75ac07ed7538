"""Child process of tests/test_gpu_ranks.py: R ranks as threads of this process, all on cuda:0, talking through the
in-process NCCL stand-in (tests/fake_nccl, loaded by the library through B2K_NCCL_LIB).  Runs every case of one area
and pickles, per case, each rank's outputs or error text, the collectives the stand-in saw per rank, and the one-rank
result on the concatenated rows.

    python tests/_ranks_child.py <area> <R> <out.pkl>

The data generators and shard splits are plain NumPy, so the parent imports this module to rebuild the same inputs
for its oracles.
"""
from __future__ import annotations

import ctypes
import os
import pickle
import sys
import threading
import time
import traceback

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
FAKE_NCCL = os.path.join(HERE, "fake_nccl", "libfake_nccl.so")

KMEANS_SHAPES = [(64, 128), (256, 256), (16, 6)]   # fused 3xTF32, large-shape, generic
PCA_DS = [128, 130, 1020]                           # wgmma, generic, wgmma with 36 tiles and a ragged block
LINREG_DS = [1, 20, 128, 1024]
KNN_INT = [("w16", 16, 10, 2), ("g7", 7, 10, 1), ("g7k100", 7, 100, 1)]   # (name, d, k, kernel_path)


# ---- shards: uneven row splits; R = 3 ends with a rank smaller than one tile ----
def sizes(n, R, tiny=7):
    if R == 2:
        a = n * 6 // 10
        return [a, n - a]
    big = (n - tiny) * 6 // 10
    return [big, n - tiny - big, tiny]


def split(A, sz):
    out, o = [], 0
    for s in sz:
        out.append(A[o:o + s])
        o += s
    return out


def pca_sizes(R):   # a rank of n = 1 (mod 4096) and one of fewer than 32 rows
    return [8193, 17] if R == 2 else [12289, 4000, 7]


def knn_sizes(R, n, nq):   # items [big, 0, small] and queries [0, some, rest] at R = 3
    if R == 2:
        return [n * 2 // 3, n - n * 2 // 3], [nq * 2 // 5, nq - nq * 2 // 5]
    return [n * 3 // 4, 0, n - n * 3 // 4], [0, nq * 2 // 5, nq - nq * 2 // 5]


# ---- data ----
def blobs(n, d, k, seed):
    sys.path.insert(0, ROOT)
    from oracle import kmeans_oracle as ko

    X, ctr = ko.make_blobs(n, d, k, seed=seed)
    C0 = (ctr + 0.25 * np.random.default_rng(seed + 1).normal(size=ctr.shape)).astype(np.float32)
    return X, C0


def pca_data(n, d, seed):   # a decaying spectrum (tests/test_gpu_pca.py _data "random")
    rng = np.random.default_rng(seed)
    Q, _ = np.linalg.qr(rng.normal(size=(d, d)))
    X = (rng.normal(size=(n, d)) * (1.0 / np.sqrt(1.0 + np.arange(d)))) @ Q.T + 0.1 * rng.normal(size=d)
    return X.astype(np.float32)


def linreg_data(n, d, seed):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, d)).astype(np.float32)
    y = (X.astype(np.float64) @ rng.normal(size=d) + 1.5 + 0.3 * rng.normal(size=n)).astype(np.float32)
    return X, y


def logreg_eval_data(n, d, kp, seed):
    rng = np.random.default_rng(seed)
    K = max(kp, 2)
    X = rng.normal(size=(n, d)).astype(np.float32)
    y = rng.integers(0, K, size=n).astype(np.float32)
    return X, y, np.arange(K, dtype=np.float64), rng.normal(size=(kp, d)) / np.sqrt(d), rng.normal(size=kp)


def logreg_fit_data(n, d, K, seed):
    rng = np.random.default_rng(seed)
    X = (rng.normal(size=(n, d)) * (1 + np.arange(d) % 3)).astype(np.float32)
    W = rng.normal(size=(K, d)) / np.sqrt(d)
    y = (X.astype(np.float64) @ W.T + rng.gumbel(size=(n, K))).argmax(1).astype(np.float32)
    return X, y


def labels_data(R):
    """Labels in {0, 1, 2} everywhere and class 5 only in the last rank's rows."""
    n = 3000
    y = np.random.default_rng(11).integers(0, 3, size=n).astype(np.float32)
    sz = sizes(n, R)
    y[n - sz[-1] + 2:n - sz[-1] + 4] = 5.0
    return y, sz


def knn_int_data(d, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(-3, 4, size=(3000, d)).astype(np.int64), rng.integers(-3, 4, size=(100, d)).astype(np.int64)


def knn_float_data():
    rng = np.random.default_rng(21)
    return rng.normal(size=(4000, 128)).astype(np.float32), rng.normal(size=(200, 128)).astype(np.float32)


LOGREG_SETTING = {"reg": 0.01, "l1_ratio": 0.0, "tol": 1e-12, "max_iter": 1000, "fit_intercept": True,
                  "standardization": True, "family": "auto"}


# ---- the cases of each area: name -> (per-rank inputs, one-rank inputs or None, fn(ctx, inputs) -> outputs) ----
def _np(t):
    return t.detach().cpu().numpy()


def _kmeans_cases(R):
    cases = {}
    for k, d in KMEANS_SHAPES:
        X, C0 = blobs(20000, d, k, seed=k + d)
        parts = [{"X": p, "C0": C0} for p in split(X, sizes(len(X), R))]

        def fit(ctx, a, k=k):
            out = ctx.kmeans_fit(a["X"], k, init=a["C0"], max_iter=8, tol=1e-4)
            lab, _ = ctx.kmeans_assign(a["X"], out["cluster_centers_"])
            return {"C": _np(out["cluster_centers_"]), "n_iter": out["n_iter_"], "inertia": out["inertia_"],
                    "labels": _np(lab), "path": ctx.stats()["last_path"]}

        def lloyd(ctx, a):
            C = a["C0"].clone()
            n_it, shift = ctx.kmeans_lloyd(a["X"], C, 8, 1e-4)
            lab, _ = ctx.kmeans_assign(a["X"], C)
            return {"C": _np(C), "n_iter": n_it, "shift": shift, "labels": _np(lab), "path": ctx.stats()["last_path"]}

        cases[f"fit_{k}_{d}"] = (parts, {"X": X, "C0": C0}, fit)
        cases[f"lloyd_{k}_{d}"] = (parts, {"X": X, "C0": C0}, lloyd)
    X, _ = blobs(20000, 128, 64, seed=192)
    parts = [{"X": p} for p in split(X, sizes(len(X), R))]
    for init, seed in (("random", 5), ("k-means||", 7)):
        def f(ctx, a, init=init, seed=seed):
            out = ctx.kmeans_fit(a["X"], 64, init=init, max_iter=0, seed=seed)
            return {"C": _np(out["cluster_centers_"]), "n_iter": out["n_iter_"]}

        cases[f"init_{init}"] = (parts, {"X": X}, f)
    return cases


def _pca_cases(R):
    cases = {}
    for d in PCA_DS:
        X = pca_data(sum(pca_sizes(R)), d, seed=d)

        def f(ctx, a, d=d):
            out = ctx.pca_fit(a["X"], d)
            out["path"] = ctx.stats()["last_path"]
            return out

        cases[f"pca_{d}"] = ([{"X": p} for p in split(X, pca_sizes(R))], {"X": X}, f)
    return cases


def _linreg_cases(R):
    cases = {}
    for d in LINREG_DS:
        X, y = linreg_data(20000 if d < 1024 else 6000, d, seed=d)
        sz = sizes(len(X), R, tiny=1)
        parts = [{"X": a, "y": b} for a, b in zip(split(X, sz), split(y, sz))]
        for path in ([1, 2] if d % 4 == 0 else [1]):
            def f(ctx, a, path=path):
                ctx.set_option("kernel_path", path)
                n, mean, mom = ctx.linreg_moments(a["X"], a["y"])
                return {"n": n, "mean": mean, "mom": mom, "path": ctx.stats()["last_path"]}

            cases[f"moments_{d}_p{path}"] = (parts, {"X": X, "y": y}, f)
    return cases


def _logreg_cases(R):
    cases = {}
    y, sz = labels_data(R)

    def labels(ctx, a):
        cls, cnt, nt = ctx.logreg_labels(a["y"])
        return {"classes": cls, "counts": cnt, "n": nt}

    cases["labels"] = ([{"y": p} for p in split(y, sz)], {"y": y}, labels)
    for kp in (1, 4):
        X, y, classes, W, b = logreg_eval_data(5000, 64, kp, seed=40 + kp)
        sz = sizes(len(X), R)
        parts = [{"X": p, "y": q} for p, q in zip(split(X, sz), split(y, sz))]
        for path in (1, 2):
            def ev(ctx, a, path=path, classes=classes, W=W, b=b):
                ctx.set_option("kernel_path", path)
                loss, gW, gb, nt = ctx.logreg_eval(a["X"], a["y"], classes, W, b)
                return {"loss": loss, "gW": gW, "gb": gb, "n": nt, "path": ctx.stats()["last_path"]}

            cases[f"eval_k{kp}_p{path}"] = (parts, {"X": X, "y": y}, ev)
    for K in (2, 4):
        X, y = logreg_fit_data(4000, 12, K, seed=K + 50)
        sz = sizes(len(X), R)
        parts = [{"X": p, "y": q} for p, q in zip(split(X, sz), split(y, sz))]

        def fit(ctx, a):
            cls, cnt, _ = ctx.logreg_labels(a["y"])
            (W, b, it), = ctx.logreg_fit(a["X"], a["y"], cls, cnt, [LOGREG_SETTING])
            return {"W": W, "b": b, "it": it}

        cases[f"fit_K{K}"] = (parts, {"X": X, "y": y}, fit)
    return cases


def _knn_cases(R):
    cases = {}
    for name, d, k, path in KNN_INT:
        Xi, Qi = knn_int_data(d, seed=d + k)
        X, Q = Xi.astype(np.float32), Qi.astype(np.float32)
        isz, qsz = knn_sizes(R, len(X), len(Q))
        for with_ids in (False, True):
            ids = (7 * np.arange(len(X)) + 5).astype(np.int64)
            parts = [{"X": a, "Q": q, "ids": i} for a, q, i in zip(split(X, isz), split(Q, qsz), split(ids, isz))]

            def f(ctx, a, k=k, path=path, with_ids=with_ids):
                ctx.set_option("kernel_path", path)
                dist, idx = ctx.knn_search(a["X"], a["Q"], k, a["ids"] if with_ids else None)
                return {"dist": _np(dist), "idx": _np(idx), "path": ctx.stats()["last_path"]}

            cases[f"int_{name}_{'ids' if with_ids else 'rows'}"] = (parts, None, f)
    X, Q = knn_float_data()
    isz, qsz = knn_sizes(R, len(X), len(Q))

    def ff(ctx, a):
        dist, idx = ctx.knn_search(a["X"], a["Q"], 16)
        return {"dist": _np(dist), "idx": _np(idx)}

    cases["float_128"] = ([{"X": a, "Q": q} for a, q in zip(split(X, isz), split(Q, qsz))], None, ff)
    return cases


EMPTY_RANK = 1   # the rank holding an empty partition in the failure cases


def _fail_cases(R):
    cases = {}
    X, C0 = blobs(3000, 8, 4, seed=3)
    y = (np.arange(len(X)) % 2).astype(np.float32)
    sz = sizes(len(X), R)
    sz_e = list(sz)
    sz_e[0] += sz_e[EMPTY_RANK]
    sz_e[EMPTY_RANK] = 0
    parts = [{"X": a, "y": b, "C0": C0} for a, b in zip(split(X, sz_e), split(y, sz_e))]
    s = dict(LOGREG_SETTING, max_iter=5)
    ops = {
        "kmeans_fit": lambda ctx, a: ctx.kmeans_fit(a["X"], 4, init=a["C0"], max_iter=3),
        "kmeans_lloyd": lambda ctx, a: ctx.kmeans_lloyd(a["X"], a["C0"].clone(), 3, 0.0),
        "pca_fit": lambda ctx, a: ctx.pca_fit(a["X"], 2),
        "linreg_moments": lambda ctx, a: ctx.linreg_moments(a["X"], a["y"]),
        "logreg_labels": lambda ctx, a: ctx.logreg_labels(a["y"]),
        "logreg_eval": lambda ctx, a: ctx.logreg_eval(a["X"], a["y"], [0.0, 1.0], np.zeros((1, 8)), np.zeros(1)),
        "logreg_fit": lambda ctx, a: ctx.logreg_fit(a["X"], a["y"], np.array([0.0, 1.0]), np.array([1500, 1500]), [s]),
    }
    for name, op in ops.items():
        cases[f"empty_{name}"] = (parts, None, lambda ctx, a, op=op: op(ctx, a) and {})
    bad = R - 1   # the rank with the faulty row
    ok_parts = [{"X": a, "y": b} for a, b in zip(split(X, sz), split(y, sz))]

    def with_bad(key, row, value):
        p = [dict(q) for q in ok_parts]
        v = p[bad][key].copy()
        v[row] = value
        p[bad][key] = v
        return p

    cases["nan_linreg"] = (with_bad("X", (3, 2), np.nan), None, lambda ctx, a: ctx.linreg_moments(a["X"], a["y"]) and {})
    cases["label_negative"] = (with_bad("y", 2, -1.0), None, lambda ctx, a: ctx.logreg_labels(a["y"]) and {})
    cases["label_fraction"] = (with_bad("y", 2, 0.5), None, lambda ctx, a: ctx.logreg_labels(a["y"]) and {})
    Xk = np.random.default_rng(4).normal(size=(300, 8)).astype(np.float32)
    kp = [{"X": a, "Q": a[:5]} for a in split(Xk, sizes(len(Xk), R))]
    kd = [dict(q) for q in kp]
    kd[bad] = {"X": kd[bad]["X"][:, :7].copy(), "Q": kd[bad]["Q"][:, :7].copy()}
    cases["knn_d_differs"] = (kd, None, lambda ctx, a: ctx.knn_search(a["X"], a["Q"], 3) and {})
    cases["knn_k_too_large"] = (kp, None, lambda ctx, a: ctx.knn_search(a["X"], a["Q"], 301) and {})
    return cases


AREAS = {"kmeans": _kmeans_cases, "pca": _pca_cases, "linreg": _linreg_cases, "logreg": _logreg_cases,
         "knn": _knn_cases, "fail": _fail_cases}


# ---- running ranks ----
def _fake():
    L = ctypes.CDLL(FAKE_NCCL)
    L.b2kFakeNcclTrace.restype = ctypes.c_longlong
    L.b2kFakeNcclTrace.argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.c_char_p, ctypes.c_longlong]
    L.b2kFakeNcclGroupError.restype = ctypes.c_longlong
    L.b2kFakeNcclGroupError.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_longlong]
    return L


def _read(call):
    buf = ctypes.create_string_buffer(1 << 20)
    n = call(buf, len(buf))
    assert 0 <= n < len(buf), n
    return buf.value.decode()


def _to_device(torch, a):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in a.items()}


def run_ranks(R, parts, fn):
    """Runs fn(ctx, inputs) on R rank threads -> (outputs or None per rank, error text or None per rank, the stand-in's
    trace per rank, the group's error, seconds)."""
    import torch

    from spark_rapids_ml_b200 import _native

    uid = _native.comm_unique_id()   # on this thread, before any rank thread: nccl_api()'s first call is not thread-safe
    dev = [_to_device(torch, p) for p in parts]
    streams = [torch.cuda.Stream() for _ in range(R)]
    torch.cuda.synchronize()
    outs, errs = [None] * R, [None] * R

    def rank(r):
        ctx = None
        try:
            ctx = _native.Context(0)
            with torch.cuda.stream(streams[r]):
                ctx.comm_init(R, r, uid)
                outs[r] = fn(ctx, dev[r])
                streams[r].synchronize()
        except Exception as e:  # noqa: BLE001 - reported to the parent
            errs[r] = str(e) or traceback.format_exc()
        finally:
            if ctx is not None:
                ctx.close()   # destroys the communicator; never aborts it, so a stranded peer shows as a timeout

    t0 = time.monotonic()
    th = [threading.Thread(target=rank, args=(r,)) for r in range(R)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    secs = time.monotonic() - t0
    L = _fake()
    trace = [_read(lambda b, c, r=r: L.b2kFakeNcclTrace(uid, r, b, c)) for r in range(R)]
    gerr = _read(lambda b, c: L.b2kFakeNcclGroupError(uid, b, c))
    return outs, errs, trace, gerr, secs


def run_single(one, fn):
    import torch

    from spark_rapids_ml_b200 import _native

    with _native.Context(0) as ctx:
        return fn(ctx, _to_device(torch, one))


# ---- the stand-in itself, through ctypes on CUDA tensors ----
NCCL_UINT8, NCCL_INT64, NCCL_FLOAT32, NCCL_FLOAT64, NCCL_SUM = 1, 4, 7, 8, 0


class _Uid(ctypes.Structure):
    _fields_ = [("internal", ctypes.c_char * 128)]


def _nccl():
    L = ctypes.CDLL(FAKE_NCCL)
    vp = ctypes.c_void_p
    L.ncclGetUniqueId.argtypes = [ctypes.POINTER(_Uid)]
    L.ncclCommInitRank.argtypes = [ctypes.POINTER(vp), ctypes.c_int, _Uid, ctypes.c_int]
    L.ncclAllReduce.argtypes = [vp, vp, ctypes.c_size_t, ctypes.c_int, ctypes.c_int, vp, vp]
    L.ncclAllGather.argtypes = [vp, vp, ctypes.c_size_t, ctypes.c_int, vp, vp]
    L.ncclCommDestroy.argtypes = [vp]
    L.ncclCommAbort.argtypes = [vp]
    L.ncclGetErrorString.restype = ctypes.c_char_p
    L.ncclGetErrorString.argtypes = [ctypes.c_int]
    return L


def _group(L, R, body):
    """body(r, comm, stream) on R threads of one fresh group -> per rank (value, error text or None, seconds)."""
    import torch

    uid = _Uid()
    assert L.ncclGetUniqueId(ctypes.byref(uid)) == 0
    streams = [torch.cuda.Stream() for _ in range(R)]
    torch.cuda.synchronize()
    res = [None] * R

    def run(r):
        comm = ctypes.c_void_p()
        t0 = time.monotonic()
        rc = L.ncclCommInitRank(ctypes.byref(comm), R, uid, r)
        if rc != 0:
            res[r] = (None, L.ncclGetErrorString(rc).decode(), time.monotonic() - t0)
            return
        with torch.cuda.stream(streams[r]):
            val, rc, aborted = body(r, comm, streams[r])
        err = L.ncclGetErrorString(rc).decode() if rc != 0 else None
        res[r] = (val, err, time.monotonic() - t0)
        if not aborted:
            L.ncclCommDestroy(comm)

    th = [threading.Thread(target=run, args=(r,)) for r in range(R)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    return res


def shim_checks(R):
    import torch

    L = _nccl()
    out = {}
    rng = np.random.default_rng(R)
    # allreduce: values over 16 decades, so that the order of the sum shows in the bits
    ins = {np.float32: [(rng.normal(size=1000) * 10.0 ** rng.integers(-8, 8, size=1000)).astype(np.float32)
                        for _ in range(R)],
           np.float64: [rng.normal(size=1000) * 10.0 ** rng.integers(-8, 8, size=1000) for _ in range(R)]}
    dt = {np.float32: NCCL_FLOAT32, np.float64: NCCL_FLOAT64}
    dev = {t: [torch.from_numpy(a).cuda() for a in v] for t, v in ins.items()}
    outp = [torch.zeros(1000, dtype=torch.float64, device="cuda") for _ in range(R)]

    def allreduce(r, comm, s):
        got = {}
        for t in (np.float32, np.float64):   # in place, as the library calls it
            x = dev[t][r]
            rc = L.ncclAllReduce(x.data_ptr(), x.data_ptr(), 1000, dt[t], NCCL_SUM, comm, s.cuda_stream)
            if rc:
                return got, rc, False
            got[t.__name__] = x.cpu().numpy()
        src = torch.from_numpy(ins[np.float64][r]).cuda()   # out of place
        rc = L.ncclAllReduce(src.data_ptr(), outp[r].data_ptr(), 1000, NCCL_FLOAT64, NCCL_SUM, comm, s.cuda_stream)
        got["out_of_place"] = outp[r].cpu().numpy()
        return got, rc, False

    out["allreduce"] = {"inputs": {t.__name__: v for t, v in ins.items()}, "ranks": _group(L, R, allreduce)}

    def allgather(r, comm, s):
        mine = np.arange(5, dtype=np.int64) + 100 * r
        recv = torch.full((R * 5,), -1, dtype=torch.int64, device="cuda")
        recv[5 * r:5 * r + 5] = torch.from_numpy(mine).cuda()   # in place: send is the rank's own slot of recv
        rc = L.ncclAllGather(recv.data_ptr() + 40 * r, recv.data_ptr(), 5, NCCL_INT64, comm, s.cuda_stream)
        if rc:
            return None, rc, False
        src = torch.from_numpy(mine.view(np.uint8).copy()).cuda()
        recv2 = torch.zeros(R * 40, dtype=torch.uint8, device="cuda")
        rc = L.ncclAllGather(src.data_ptr(), recv2.data_ptr(), 40, NCCL_UINT8, comm, s.cuda_stream)
        return {"in_place": recv.cpu().numpy(), "out_of_place": recv2.cpu().numpy().view(np.int64)}, rc, False

    out["allgather"] = {"ranks": _group(L, R, allgather)}
    buf = [torch.zeros(8, dtype=torch.float64, device="cuda") for _ in range(R)]

    def mismatch(r, comm, s):   # the last rank reduces one value more
        b = buf[r]
        return None, L.ncclAllReduce(b.data_ptr(), b.data_ptr(), 4 + (r == R - 1), NCCL_FLOAT64, NCCL_SUM, comm,
                                     s.cuda_stream), False

    out["mismatch"] = {"ranks": _group(L, R, mismatch)}

    def missing(r, comm, s):   # the last rank never enters the collective
        if r == R - 1:
            return None, 0, False
        b = buf[r]
        return None, L.ncclAllReduce(b.data_ptr(), b.data_ptr(), 4, NCCL_FLOAT64, NCCL_SUM, comm, s.cuda_stream), False

    os.environ["B2K_FAKE_NCCL_TIMEOUT_S"] = "2"
    try:
        out["timeout"] = {"ranks": _group(L, R, missing)}
    finally:
        os.environ["B2K_FAKE_NCCL_TIMEOUT_S"] = "20"

    def abort(r, comm, s):   # the last rank aborts while its peers wait in a collective
        if r == R - 1:
            time.sleep(0.5)
            return None, L.ncclCommAbort(comm), True
        b = buf[r]
        return None, L.ncclAllReduce(b.data_ptr(), b.data_ptr(), 4, NCCL_FLOAT64, NCCL_SUM, comm, s.cuda_stream), False

    out["abort"] = {"ranks": _group(L, R, abort)}
    return out


def main(area, R, out_path):
    import torch

    sys.path.insert(0, ROOT)
    if area == "shim":
        with open(out_path, "wb") as f:
            pickle.dump(shim_checks(R), f)
        return
    res = {"empty_ptr": torch.empty((0, 8), dtype=torch.float32, device="cuda").data_ptr()}
    for name, (parts, one, fn) in AREAS[area](R).items():
        try:
            outs, errs, trace, gerr, secs = run_ranks(R, parts, fn)
            single = run_single(one, fn) if one is not None else None
            res[name] = {"outs": outs, "errs": errs, "trace": trace, "group_error": gerr, "secs": secs,
                         "single": single}
        except Exception:  # noqa: BLE001 - a harness failure is the parent's to report
            res[name] = {"harness_error": traceback.format_exc()}
    with open(out_path, "wb") as f:
        pickle.dump(res, f)


if __name__ == "__main__":
    main(sys.argv[1], int(sys.argv[2]), sys.argv[3])
