"""The multi-rank paths on one GPU: every estimator's collective code at R = 2 and R = 3 ranks with uneven shards, run
as threads of a child interpreter through the in-process NCCL stand-in of tests/fake_nccl (real NCCL refuses two
ranks on one device).  The child is tests/_ranks_child.py; it runs all cases of one area per (area, R) and hands back
each rank's outputs or error text, the collectives the stand-in saw per rank, and the one-rank result on the
concatenated rows.  B2K_NCCL_LIB is set in the child only, so this process keeps real NCCL.

Every case checks that the ranks' replicated outputs are bitwise identical, that the stand-in saw the same collective
sequence on every rank, that the result meets its oracle's bound, and that it is close to the one-rank result.  The
stand-in sums in rank order and NCCL in its own, so comparisons with one rank use tolerances NCCL also meets; they are
bitwise only where the design implies it: init="random" and k-means|| (picks keyed on the global row, exact weights)
and k-NN on integer data (every distance exact, ties broken by global row).
"""
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import _ranks_child as child
import logreg_oracle as lo
from oracle import kmeans_oracle as ko

pytestmark = pytest.mark.gpu

CHILD = os.path.join(child.HERE, "_ranks_child.py")
CHILD_TIMEOUT_S = 600   # one child runs every case of an area
RENDEZVOUS_TIMEOUT_S = 20
RANKS = [2, 3]
_RUNS = {}


def _run(area, R):
    """The child's results for (area, R), run once per session."""
    key = (area, R)
    if key not in _RUNS:
        _RUNS[key] = _spawn(area, R)
    res = _RUNS[key]
    if isinstance(res, str):
        pytest.fail(res)
    return res


def _spawn(area, R):
    if not os.path.exists(child.FAKE_NCCL):
        return (f"{child.FAKE_NCCL} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(or `make -C tests/fake_nccl`)")
    env = dict(os.environ, B2K_NCCL_LIB=child.FAKE_NCCL, B2K_FAKE_NCCL_TIMEOUT_S=str(RENDEZVOUS_TIMEOUT_S))
    if sys.flags.no_user_site:
        env["PYTHONNOUSERSITE"] = "1"
    with tempfile.TemporaryDirectory() as td:
        out = os.path.join(td, "out.pkl")
        try:
            p = subprocess.run([sys.executable, CHILD, area, str(R), out], env=env, cwd=child.ROOT,
                               capture_output=True, text=True, timeout=CHILD_TIMEOUT_S)
        except subprocess.TimeoutExpired as e:   # subprocess.run has killed the child
            return f"{area} R={R}: the child timed out after {CHILD_TIMEOUT_S} s\n{(e.stderr or '')[-4000:]}"
        if p.returncode != 0 or not os.path.exists(out):
            return f"{area} R={R}: the child failed (exit {p.returncode})\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}"
        with open(out, "rb") as f:
            return pickle.load(f)


def _bits(v):
    if isinstance(v, np.ndarray):
        return (v.dtype.str, v.shape, v.tobytes())
    if isinstance(v, float):
        return np.float64(v).tobytes()
    return v


def _case(area, R, name, replicated=()):
    """One case's results after the checks every case shares: no rank failed, no collective failed, the same
    collective sequence on every rank, and bitwise-identical `replicated` outputs."""
    c = _run(area, R)[name]
    assert "harness_error" not in c, c.get("harness_error")
    assert c["errs"] == [None] * R, c["errs"]
    assert c["group_error"] == "", c["group_error"]
    assert c["trace"][0] and all(t == c["trace"][0] for t in c["trace"]), c["trace"]
    for key in replicated:
        assert all(_bits(o[key]) == _bits(c["outs"][0][key]) for o in c["outs"]), f"ranks differ in {key}"
    return c


def _case_failing(area, R, name):
    """Every rank raised the same message, and none waited out the stand-in's timeout."""
    c = _run(area, R)[name]
    assert "harness_error" not in c, c.get("harness_error")
    errs = c["errs"]
    assert all(e is not None for e in errs), errs
    assert all(e == errs[0] for e in errs), errs
    assert "timed out" not in c["group_error"] and "fake NCCL" not in errs[0], (c["group_error"], errs[0])
    assert c["secs"] < RENDEZVOUS_TIMEOUT_S / 2, c["secs"]
    return errs[0]


# ---- 1. the stand-in itself ----
@pytest.mark.parametrize("R", RANKS)
def test_stand_in_allreduce_sums_in_rank_order(R):
    res = _run("shim", R)["allreduce"]
    for t, outs in (("float32", "float32"), ("float64", "float64"), ("float64", "out_of_place")):
        acc = res["inputs"][t][0].copy()
        for a in res["inputs"][t][1:]:
            acc = acc + a   # one left-to-right sum in the dtype's own arithmetic
        for r, (val, err, _) in enumerate(res["ranks"]):
            assert err is None, err
            assert val[outs].tobytes() == acc.tobytes(), (t, outs, r)


@pytest.mark.parametrize("R", RANKS)
def test_stand_in_allgather_in_and_out_of_place(R):
    want = np.concatenate([np.arange(5, dtype=np.int64) + 100 * r for r in range(R)])
    for val, err, _ in _run("shim", R)["allgather"]["ranks"]:
        assert err is None, err
        np.testing.assert_array_equal(val["in_place"], want)
        np.testing.assert_array_equal(val["out_of_place"], want)


@pytest.mark.parametrize("R", RANKS)
def test_stand_in_reports_a_sequence_mismatch_on_every_rank(R):
    for val, err, _ in _run("shim", R)["mismatch"]["ranks"]:
        assert err is not None and "sequence mismatch at rendezvous #0" in err, err
        assert f"rank {R - 1} AllReduce(dtype 8, count 5)" in err and "rank 0 AllReduce(dtype 8, count 4)" in err, err


@pytest.mark.parametrize("R", RANKS)
def test_stand_in_times_out_naming_the_missing_rank(R):
    ranks = _run("shim", R)["timeout"]["ranks"]
    assert ranks[R - 1][1] is None
    for val, err, secs in ranks[:-1]:
        assert err is not None and "timed out after 2 s" in err and f"missing ranks: {R - 1}" in err, err
        assert 1.9 <= secs < 10, secs


@pytest.mark.parametrize("R", RANKS)
def test_stand_in_abort_wakes_the_waiters(R):
    ranks = _run("shim", R)["abort"]["ranks"]
    assert ranks[R - 1][1] is None
    for val, err, secs in ranks[:-1]:
        assert err is not None and f"communicator aborted by rank {R - 1}" in err, err
        assert secs < 10, secs


# ---- 2. KMeans ----
@pytest.mark.parametrize("R", RANKS)
@pytest.mark.parametrize("kind", ["fit", "lloyd"])
@pytest.mark.parametrize("k,d", child.KMEANS_SHAPES)
def test_kmeans_lloyd_matches_the_oracle(R, kind, k, d):
    """Array init, 8 iterations: the per-iteration allreduce of [sums | counts | cost] against the oracle's Lloyd loop
    over the same shards, through b2k_kmeans_fit and b2k_kmeans_lloyd."""
    c = _case("kmeans", R, f"{kind}_{k}_{d}", ["C", "n_iter", "inertia" if kind == "fit" else "shift"])
    X, C0 = child.blobs(20000, d, k, seed=k + d)
    ref = ko.lloyd(child.split(X, child.sizes(len(X), R)), C0, 8, 1e-4)
    o = c["outs"][0]
    assert o["path"] == (1 if d % 4 else 2)
    assert o["n_iter"] == ref["n_iter"] == c["single"]["n_iter"]
    assert ko.max_center_rel_err(o["C"], ref["centers"]) <= 1e-5
    assert ko.max_center_rel_err(o["C"], c["single"]["C"]) <= 1e-5
    labels = np.concatenate([x["labels"] for x in c["outs"]])
    cmp = ko.compare_labels(X, o["C"], labels)
    assert cmp["n_mismatch_outside_margin"] == 0, cmp
    if kind == "fit":
        assert abs(o["inertia"] - ref["inertia"]) <= 1e-3 * ref["inertia"]


@pytest.mark.parametrize("R", RANKS)
@pytest.mark.parametrize("init", ["random", "k-means||"])
def test_kmeans_init_is_bitwise_the_one_rank_init(R, init):
    """max_iter = 0 returns the initial centres.  init="random" draws global rows and fetches them with an allreduce of
    zero-filled rows; k-means|| keys its Bernoulli picks on (seed, round, global row) and weighs the candidates with an
    exact histogram: both must give the one-rank centres bit for bit."""
    c = _case("kmeans", R, f"init_{init}", ["C", "n_iter"])
    o = c["outs"][0]
    assert o["n_iter"] == 0
    assert o["C"].tobytes() == c["single"]["C"].tobytes()
    if init == "random":
        X, _ = child.blobs(20000, 128, 64, seed=192)
        rows = {r.tobytes() for r in X}
        assert all(r.tobytes() in rows for r in o["C"])


# ---- 3. PCA ----
@pytest.fixture(scope="module")
def ctx():
    from spark_rapids_ml_b200 import _native

    with _native.Context(0) as c:
        yield c


@pytest.mark.parametrize("R", RANKS)
@pytest.mark.parametrize("d", child.PCA_DS)
def test_pca_matches_the_oracle(ctx, R, d):
    from test_gpu_pca import _check_against_oracle

    keys = ["mean_", "components_", "explained_variance_ratio_", "singular_values_"]
    c = _case("pca", R, f"pca_{d}", keys + ["path"])
    X = child.pca_data(sum(child.pca_sizes(R)), d, seed=d)
    o = c["outs"][0]
    assert o["path"] == (1 if d % 4 else 2)
    _check_against_oracle(X, o, d, ctx)
    s = c["single"]
    assert np.abs(o["singular_values_"] - s["singular_values_"]).max() <= 2e-5 * s["singular_values_"][0]
    assert np.abs(o["mean_"] - s["mean_"]).max() <= 2e-6 * np.abs(s["mean_"]).max()


# ---- 4. linear regression ----
def _check_moments(X, y, n, mean, M, path):
    """tests/test_gpu_linreg.py _check_moments' bounds, against fp64 moments of the concatenated rows."""
    from test_gpu_linreg import EPS

    d = X.shape[1]
    V = np.concatenate([X.astype(np.float64), y.astype(np.float64)[:, None]], 1)
    m_ref = V.mean(0)
    C = V - m_ref
    M_ref, S = C.T @ C, np.abs(C).T @ np.abs(C)
    assert n == X.shape[0]
    np.testing.assert_allclose(mean, m_ref, rtol=1e-12, atol=1e-12 * np.abs(m_ref).max())
    G, G_ref = M[:d, :d], M_ref[:d, :d]
    if path == 2:
        assert np.abs(G - G_ref).max() <= EPS[2] * np.abs(G_ref).max()
    else:
        assert (np.abs(G - G_ref) <= (2.0 ** -23 + n * 2.0 ** -53) * S[:d, :d]).all()
    cs = np.sqrt(np.outer(np.diag(M_ref), np.diag(M_ref)))[d]
    assert (np.abs(M[d] - M_ref[d]) <= 1e-10 * cs).all()
    assert np.array_equal(M, M.T)


@pytest.mark.parametrize("R", RANKS)
@pytest.mark.parametrize("d,path", [(d, p) for d in child.LINREG_DS for p in ([1, 2] if d % 4 == 0 else [1])])
def test_linreg_moments_match_the_oracle(R, d, path):
    """Two f64 allreduces in b2k_moments_impl: [sums | label sum | n], then the Gram, X^T y and y^T y; R = 3 ends with
    a rank of one row."""
    c = _case("linreg", R, f"moments_{d}_p{path}", ["n", "mean", "mom"])
    X, y = child.linreg_data(20000 if d < 1024 else 6000, d, seed=d)
    assert [o["path"] for o in c["outs"]] == [path] * R
    o, s = c["outs"][0], c["single"]
    _check_moments(X, y, o["n"], o["mean"], o["mom"], path)
    _check_moments(X, y, s["n"], s["mean"], s["mom"], path)


# ---- 5. logistic regression ----
@pytest.mark.parametrize("R", RANKS)
def test_logreg_labels_count_exactly(R):
    """The label pass's allgather, reduced in rank order: a class held only by the last rank is found and counted."""
    c = _case("logreg", R, "labels", ["classes", "counts", "n"])
    y, _ = child.labels_data(R)
    cls, cnt = np.unique(y.astype(np.float64), return_counts=True)
    o = c["outs"][0]
    np.testing.assert_array_equal(o["classes"], cls)
    np.testing.assert_array_equal(o["counts"], cnt)
    assert o["n"] == len(y) and 5.0 in cls


@pytest.mark.parametrize("R", RANKS)
@pytest.mark.parametrize("kp", [1, 4])
@pytest.mark.parametrize("path", [1, 2])
def test_logreg_eval_within_the_round_off_bound(R, kp, path):
    c = _case("logreg", R, f"eval_k{kp}_p{path}", ["loss", "gW", "gb", "n"])
    X, y, classes, W, b = child.logreg_eval_data(5000, 64, kp, seed=40 + kp)
    assert [o["path"] for o in c["outs"]] == [path] * R
    ref = lo.loss_grad(X, np.searchsorted(classes, y.astype(np.float64)), W, b)
    bd = lo.eval_bound(X, W, b)
    for o in (c["outs"][0], c["single"]):
        assert o["n"] == len(X)
        assert abs(o["loss"] - ref[0]) <= bd["loss"]
        assert np.all(np.abs(o["gW"] - ref[1]) <= bd["dW"])
        assert np.all(np.abs(o["gb"] - ref[2]) <= bd["db"])


@pytest.mark.parametrize("R", RANKS)
@pytest.mark.parametrize("K", [2, 4])
def test_logreg_fit_is_rank_identical_and_optimal(R, K):
    """Every rank runs the optimiser on the same allreduced values: the models are bitwise equal and optimal."""
    c = _case("logreg", R, f"fit_K{K}", ["W", "b", "it"])
    X, y = child.logreg_fit_data(4000, 12, K, seed=K + 50)
    o, s = c["outs"][0], c["single"]
    P = lo.Problem(X, y, child.LOGREG_SETTING["reg"], 0.0)
    assert P.residual(np.concatenate([(o["W"] * P.sig).ravel(), o["b"]])) <= 1e-8
    assert np.abs(o["W"] - s["W"]).max() <= 1e-6 * max(1.0, np.abs(s["W"]).max())
    assert np.abs(o["b"] - s["b"]).max() <= 1e-6 * max(1.0, np.abs(s["b"]).max())


# ---- 6. exact k-NN ----
@pytest.mark.parametrize("R", RANKS)
@pytest.mark.parametrize("name,d,k,path", child.KNN_INT)
@pytest.mark.parametrize("ids", ["rows", "ids"])
def test_knn_integer_data_is_exact(R, name, d, k, path, ids):
    """Integer data in [-3, 3]: every distance is exact and ties are many, so the ids must be the oracle's, ties broken
    by global row, on every rank's queries, including ranks with no items or no queries."""
    from test_gpu_knn_exact import _int_oracle

    c = _case("knn", R, f"int_{name}_{ids}")
    Xi, Qi = child.knn_int_data(d, seed=d + k)
    ref_d, ref_i = _int_oracle(Xi, Qi, k)
    if ids == "ids":
        ref_i = 7 * ref_i + 5
    _, qsz = child.knn_sizes(R, len(Xi), len(Qi))
    q0 = 0
    for r, o in enumerate(c["outs"]):
        assert o["dist"].shape == (qsz[r], k)
        np.testing.assert_array_equal(o["idx"], ref_i[q0:q0 + qsz[r]], err_msg=f"rank {r}")
        np.testing.assert_array_equal(o["dist"].view(np.uint32), ref_d[q0:q0 + qsz[r]].view(np.uint32))
        if qsz[r]:
            assert o["path"] == path
        q0 += qsz[r]


@pytest.mark.parametrize("R", RANKS)
def test_knn_float_data_meets_the_parity_rule(R):
    import knn_oracle

    c = _case("knn", R, "float_128")
    X, Q = child.knn_float_data()
    dist = np.concatenate([o["dist"] for o in c["outs"]])
    idx = np.concatenate([o["idx"] for o in c["outs"]])
    bad = knn_oracle.compare(X, Q, 16, dist, idx)
    assert bad["n_outside_margin"] == 0, bad


# ---- 7. every rank fails together ----
EMPTY_OPS = ["kmeans_fit", "kmeans_lloyd", "pca_fit", "linreg_moments", "logreg_labels", "logreg_eval", "logreg_fit"]


@pytest.mark.parametrize("R", RANKS)
def test_an_empty_cuda_tensor_has_a_null_data_pointer(R):
    """The premise of the empty-partition cases: torch hands the library NULL for an empty CUDA tensor."""
    assert _run("fail", R)["empty_ptr"] == 0


@pytest.mark.parametrize("R", RANKS)
@pytest.mark.parametrize("op", EMPTY_OPS)
def test_empty_partition_fails_on_every_rank(R, op):
    err = _case_failing("fail", R, f"empty_{op}")
    assert f"b2k_{op}: empty partition (rank {child.EMPTY_RANK} has n_local == 0)" in err, err


@pytest.mark.parametrize("R", RANKS)
@pytest.mark.parametrize("name,msg", [
    ("nan_linreg", "linear regression: the features or the label hold a NaN or an infinity"),
    ("label_negative", "Labels MUST be in [0, 2147483647), but got -1"),
    ("label_fraction", "Labels MUST be Integers, but got 0.5"),
    ("knn_k_too_large", "k = 301 must satisfy 1 <= k <= 300 (items on all ranks)"),
])
def test_bad_data_on_one_rank_fails_on_every_rank(R, name, msg):
    err = _case_failing("fail", R, name)
    assert msg in err, err


@pytest.mark.parametrize("R", RANKS)
def test_knn_d_differing_between_ranks_fails_on_every_rank(R):
    err = _case_failing("fail", R, "knn_d_differs")
    assert f"d differs between ranks (rank {R - 1} has d = 7, rank 0 has d = 8)" in err, err
