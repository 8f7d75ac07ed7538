"""GPU parity tests proper: the CUDA path through the C ABI vs the fp64 oracle on identical seeded inputs,
the committed golden fixtures, and the reference's known-answer vectors.

Parity rule (SURVEY.md 8c / BASELINE.json north_star): labels bit-exact except rows whose fp64 margin
(d2-d1)/max(d1,||x||^2) is below 1e-6 (fp32 ordering noise; n_mismatch_outside_margin must be 0);
centroids within 1e-4 relative.
"""
import glob
import json
import os

import numpy as np
import pytest

from oracle import kmeans_oracle as ko

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
TAU = 1e-6
CENTER_RTOL = 1e-4
PATHS = {"generic": 1, "tcgen05": 2}


@pytest.fixture(scope="module")
def ctx():
    from spark_rapids_ml_b200 import _native

    c = _native.Context(0)
    yield c
    c.close()


def _dev(x):
    import torch

    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _supported(path, d, k):
    if path == "generic":
        return True
    return d % 4 == 0 and d <= 256 and k <= 256


@pytest.mark.parametrize("path", ["generic", "tcgen05"])
@pytest.mark.parametrize("n,d,k,gen", [
    (4096, 128, 64, "blobs"),
    (5000, 128, 64, "uniform"),     # near-tie stress + ragged last tile
    (1000, 32, 8, "blobs"),
    (777, 64, 16, "uniform"),
    (130, 20, 5, "blobs"),          # d not a multiple of 32
    (64, 4, 3, "uniform"),
    (1, 8, 1, "uniform"),           # single row, single center
    (3000, 100, 40, "blobs"),
])
def test_assign_matches_oracle(ctx, path, n, d, k, gen):
    if not _supported(path, d, k):
        pytest.skip("shape outside the fused kernel's instantiations")
    ctx.set_option("kernel_path", PATHS[path])
    X = ko.make_blobs(n, d, k, seed=7)[0] if gen == "blobs" else ko.make_uniform(n, d, seed=7)
    rng = np.random.default_rng(3)
    C = X[rng.choice(n, size=k, replace=(n < k))].copy() + (0.01 if gen == "uniform" else 0.0)
    labels, md = ctx.kmeans_assign(_dev(X), _dev(C), want_mindist=True)
    st = ctx.stats()
    assert st["last_path"] == PATHS[path]
    cmp = ko.compare_labels(X, C, labels.cpu().numpy(), tau=TAU)
    assert cmp["n_mismatch_outside_margin"] == 0, cmp
    _, md_o, _ = ko.assign(X, C)
    xn = (X.astype(np.float64) ** 2).sum(1)
    np.testing.assert_allclose(md.cpu().numpy(), md_o, rtol=2e-4, atol=2e-5 * float(xn.max()) + 1e-6)


@pytest.mark.parametrize("path", ["generic", "tcgen05"])
def test_tie_break_lowest_index_and_duplicate_centers(ctx, path):
    ctx.set_option("kernel_path", PATHS[path])
    d, k = 32, 8
    X = ko.make_uniform(512, d, seed=1)
    C = np.repeat(X[:1], k, axis=0).copy()      # all centers identical -> every row must pick index 0
    labels, _ = ctx.kmeans_assign(_dev(X), _dev(C))
    assert int(labels.max()) == 0
    C2 = X[:k].copy()
    C2[5] = C2[2]                                # duplicate pair: index 5 must never win
    labels, _ = ctx.kmeans_assign(_dev(X), _dev(C2))
    assert int((labels == 5).sum()) == 0


@pytest.mark.parametrize("path", ["generic", "tcgen05"])
@pytest.mark.parametrize("fixture", sorted(glob.glob(os.path.join(GOLD, "lloyd_golden_*.npz"))),
                         ids=os.path.basename)
def test_lloyd_golden_fixtures(ctx, path, fixture):
    g = np.load(fixture)
    X, C0 = g["X"], g["C0"]
    n, d = X.shape
    k = C0.shape[0]
    if not _supported(path, d, k):
        pytest.skip("shape outside the fused kernel's instantiations")
    ctx.set_option("kernel_path", PATHS[path])
    out = ctx.kmeans_fit(_dev(X), k, init=C0, max_iter=int(g["max_iter"]),
                         tol=ko.map_tol(float(g["tol"])))
    Cg = out["cluster_centers_"].cpu().numpy()
    assert out["n_iter_"] == int(g["n_iter"])
    assert ko.max_center_rel_err(Cg, g["centers"]) <= CENTER_RTOL
    assert abs(out["inertia_"] - float(g["inertia"])) <= 1e-4 * float(g["inertia"])
    labels, _ = ctx.kmeans_assign(_dev(X), out["cluster_centers_"])
    cmp = ko.compare_labels(X, Cg, labels.cpu().numpy(), tau=TAU)
    assert cmp["n_mismatch_outside_margin"] == 0, cmp
    if "blobs" in fixture:  # well separated: bit-exact against the oracle's own run
        np.testing.assert_array_equal(labels.cpu().numpy(), g["labels"])


@pytest.mark.parametrize("path", ["generic", "tcgen05"])
def test_reference_known_answers(ctx, path):
    """python/tests/test_kmeans.py:202-249 and :420-526 toy results, from every non-degenerate init."""
    cases = json.load(open(os.path.join(GOLD, "kmeans_known_answers.json")))["cases"]
    ctx.set_option("kernel_path", PATHS[path])
    for case in cases:
        X = np.array(case["data"], dtype=np.float32)
        Xp = np.zeros((4, 4), dtype=np.float32)   # pad d=2 -> 4 so the TMA path (d % 4 == 0) also runs
        Xp[:, :2] = X
        exp = np.array(case["expected_sorted_centers"])
        ok = 0
        for a in range(4):
            for b in range(a + 1, 4):
                C0 = Xp[[a, b]].copy()
                ref = ko.lloyd([Xp], C0, case["max_iter"], case["tol"])
                out = ctx.kmeans_fit(_dev(Xp), 2, init=C0, max_iter=case["max_iter"],
                                     tol=ko.map_tol(case["tol"]))
                Cg = out["cluster_centers_"].cpu().numpy()
                np.testing.assert_allclose(Cg, ref["centers"], rtol=1e-6, atol=1e-7)
                assert out["n_iter_"] == ref["n_iter"]
                if np.allclose(np.array(sorted(Cg[:, :2].tolist())), exp, rtol=max(case["rel_tol"], 1e-7)):
                    ok += 1
                    lab = ctx.kmeans_assign(_dev(Xp), out["cluster_centers_"])[0].cpu().numpy()
                    for p, q in case["same_label_pairs"]:
                        assert lab[p] == lab[q]
                    for p, q in case["diff_label_pairs"]:
                        assert lab[p] != lab[q]
        assert ok >= 4


@pytest.mark.parametrize("path", ["generic", "tcgen05"])
def test_empty_cluster_keeps_center_and_stops(ctx, path):
    ctx.set_option("kernel_path", PATHS[path])
    X = np.array([[0, 0, 0, 0], [0, 1, 0, 0], [1, 0, 0, 0], [1, 1, 0, 0]], dtype=np.float32)
    C0 = np.array([[0.5, 0.5, 0, 0], [0.5, 0.5, 0, 0], [100, 100, 0, 0]], dtype=np.float32)
    out = ctx.kmeans_fit(_dev(X), 3, init=C0, max_iter=3, tol=1e-4)
    C = out["cluster_centers_"].cpu().numpy()
    np.testing.assert_array_equal(C[1], C0[1])
    np.testing.assert_array_equal(C[2], C0[2])
    assert out["n_iter_"] == 1


@pytest.mark.parametrize("path", ["generic", "tcgen05"])
def test_lloyd_convergence_semantics(ctx, path):
    """n_iter, early stop on sum||dc||^2 < tol, max_iter cap, tol=0 -> float32 tiny (clustering.py:113-123)."""
    ctx.set_option("kernel_path", PATHS[path])
    X, _ = ko.make_blobs(6000, 32, 8, seed=21)
    C0 = X[:8].copy()
    for max_iter, tol in [(3, 1e-4), (50, 1e-2), (50, 0.0), (1, 1e-4)]:
        ref = ko.lloyd([X], C0, max_iter, tol)
        for ce in (1, 4):
            ctx.set_option("check_every", ce)
            out = ctx.kmeans_fit(_dev(X), 8, init=C0, max_iter=max_iter, tol=ko.map_tol(tol))
            assert out["n_iter_"] == ref["n_iter"], (max_iter, tol, ce)
            assert ko.max_center_rel_err(out["cluster_centers_"].cpu().numpy(), ref["centers"]) <= CENTER_RTOL
    ctx.set_option("check_every", 4)


@pytest.mark.parametrize("path", ["generic", "tcgen05"])
def test_large_shape_properties(ctx, path):
    """BASELINE cfg2-shaped slice (d=128, k=64) at a size the oracle cannot check row by row quickly:
    size-independent properties — counts sum to n, one Lloyd step == oracle step on the partial sums implied by
    the device labels, determinism (bitwise identical reruns), idempotence at a fixed point."""
    import torch

    ctx.set_option("kernel_path", PATHS[path])
    n, d, k = 1_000_003, 128, 64
    g = torch.Generator(device="cuda").manual_seed(5)
    ctr = (torch.rand((k, d), generator=g, device="cuda") * 20 - 10)
    z = torch.randint(0, k, (n,), generator=g, device="cuda")
    X = (ctr[z] + torch.randn((n, d), generator=g, device="cuda")).contiguous()
    C0 = X[:k].clone()
    labels, md = ctx.kmeans_assign(X, C0, want_mindist=True)
    assert int(labels.min()) >= 0 and int(labels.max()) < k
    # device labels -> torch fp64 partial sums -> expected next centers
    C1 = C0.clone()
    n_it, shift = ctx.kmeans_lloyd(X, C1, 1, 0.0)
    assert n_it == 1
    S = torch.zeros((k, d), dtype=torch.float64, device="cuda").index_add_(0, labels.long(), X.double())
    w = torch.bincount(labels.long(), minlength=k).double()
    exp = torch.where(w[:, None] > 0, S / w.clamp(min=1)[:, None], C0.double()).float()
    rel = ((C1 - exp).double().norm(dim=1) / exp.double().norm(dim=1)).max().item()
    assert rel <= 1e-5, rel
    assert abs(shift - float(((exp - C0).double() ** 2).sum())) <= 1e-4 * shift + 1e-12
    # determinism
    C2 = C0.clone()
    ctx.kmeans_lloyd(X, C2, 1, 0.0)
    assert torch.equal(C1, C2)
    # run to convergence from a near-optimal start, then one more step is a fixed point (idempotence)
    C3 = (ctr + 0.3 * torch.randn((k, d), generator=g, device="cuda")).contiguous()
    n_conv, _ = ctx.kmeans_lloyd(X, C3, 60, 1e-12)
    assert n_conv < 60
    C4 = C3.clone()
    _, shift2 = ctx.kmeans_lloyd(X, C4, 1, 0.0)
    assert shift2 <= 1e-10
    # spot-check 20k rows of the final labelling against the oracle
    idx = torch.randperm(n, generator=g, device="cuda")[:20000]
    lab, _ = ctx.kmeans_assign(X[idx].contiguous(), C3)
    cmp = ko.compare_labels(X[idx].cpu().numpy(), C3.cpu().numpy(), lab.cpu().numpy(), tau=TAU)
    assert cmp["n_mismatch_outside_margin"] == 0, cmp


def test_init_modes_statistical(ctx):
    """random / k-means|| are validated by final inertia against the oracle's own initialisers
    (the reference's seeded test is xfail: python/tests/test_kmeans.py:332,355)."""
    ctx.set_option("kernel_path", 0)
    X, _ = ko.make_blobs(20000, 16, 10, seed=9)
    best_o = min(ko.lloyd([X], ko.init_kmeans_parallel([X], 10, s), 50, 1e-6)["inertia"] for s in range(3))
    best_g = min(ctx.kmeans_fit(_dev(X), 10, init="scalable-k-means++", max_iter=50, tol=1e-6, seed=s)["inertia_"]
                 for s in range(3))
    assert best_g <= 1.10 * best_o
    out = ctx.kmeans_fit(_dev(X), 10, init="random", max_iter=1, tol=1e-6, seed=4)
    assert out["cluster_centers_"].shape == (10, 16)
    a = ctx.kmeans_fit(_dev(X), 10, init="random", max_iter=5, tol=1e-6, seed=4)
    b = ctx.kmeans_fit(_dev(X), 10, init="random", max_iter=5, tol=1e-6, seed=4)
    np.testing.assert_array_equal(a["cluster_centers_"].cpu().numpy(), b["cluster_centers_"].cpu().numpy())


def test_kmeans_parallel_init_large_k(ctx):
    """k-means|| with k >= 1024 (its scratch comes from one arena sized from the candidate cap: a fixed 64 KB control
    region used to overlap the min-distance array from k ~ 1008 on): the seeding must find (nearly) every blob."""
    import torch

    ctx.set_option("kernel_path", 0)
    n, d, k = 200_000, 32, 1024
    g = torch.Generator(device="cuda").manual_seed(2)
    ctr = torch.rand((k, d), generator=g, device="cuda") * 20 - 10
    X = (ctr[torch.randint(0, k, (n,), generator=g, device="cuda")] + 0.2 * torch.randn((n, d), generator=g, device="cuda")).contiguous()
    a = ctx.kmeans_fit(X, k, init="scalable-k-means++", max_iter=5, tol=1e-6, seed=1)
    b = ctx.kmeans_fit(X, k, init="scalable-k-means++", max_iter=5, tol=1e-6, seed=1)
    ideal = n * d * 0.04                     # sigma^2 * d per row if every blob has its own centre
    assert a["inertia_"] <= 6.0 * ideal, (a["inertia_"], ideal)   # a random start leaves ~1/e of the blobs without a centre: >> this
    np.testing.assert_array_equal(a["cluster_centers_"].cpu().numpy(), b["cluster_centers_"].cpu().numpy())   # seeded: reproducible


def test_ingest_layouts(ctx):
    import torch

    rng = np.random.default_rng(0)
    n, d = 2500, 24
    dst = torch.zeros((n, d), dtype=torch.float32, device="cuda")
    A = rng.normal(size=(1000, d)).astype(np.float32)
    B = rng.normal(size=(900, d))                      # float64 list<double> batch
    Ccols = [rng.integers(-5, 5, size=600).astype(np.int32) for _ in range(d)]  # integer scalar columns
    off = (np.arange(1001) * d).astype(np.int32)
    assert ctx.ingest_rows(dst, 0, A.reshape(-1), d, offsets=off) == 1000
    assert ctx.ingest_rows(dst, 1000, B.reshape(-1), d) == 900
    assert ctx.ingest_columns(dst, 1900, Ccols) == 600
    torch.cuda.synchronize()
    exp = np.concatenate([A, B.astype(np.float32), np.stack(Ccols, 1).astype(np.float32)])
    np.testing.assert_array_equal(dst.cpu().numpy(), exp)
    bad = off.copy()
    bad[5] += 1
    from spark_rapids_ml_b200._native import B2KError

    with pytest.raises(B2KError):
        ctx.ingest_rows(dst, 0, A.reshape(-1), d, offsets=bad)   # ragged rows are rejected
    with pytest.raises(B2KError):
        ctx.ingest_rows(dst, 2000, A.reshape(-1), d, offsets=off)  # would overflow the reserved matrix


def test_errors_are_loud(ctx):
    from spark_rapids_ml_b200._native import B2KError
    import torch

    X = torch.zeros((16, 6), device="cuda")
    ctx.set_option("kernel_path", 2)
    with pytest.raises(B2KError):      # d % 4 != 0 cannot take the TMA path and must not silently fall back
        ctx.kmeans_assign(X, torch.zeros((2, 6), device="cuda"))
    ctx.set_option("kernel_path", 0)
    with pytest.raises(B2KError):
        ctx.kmeans_fit(X, 2, init="random", n_init=3)
    with pytest.raises(B2KError):
        ctx.kmeans_fit(X, 32, init="random")   # fewer rows than k


def test_baseline_config_shapes(ctx):
    """BASELINE.json configs[0] (k=8, n=100k, d=32: full size) and configs[2] (k=256, d=256: a 20k-row slice of the
    per-GPU partition) against the oracle from an injected init; 'auto' path selection: both take a wgmma kernel
    (cfg1 the 3xTF32 one, cfg3 the large-shape 1xTF32 + recheck one, tests/test_gpu_large.py)."""
    ctx.set_option("kernel_path", 0)
    for (n, d, k, iters, want_path) in [(100_000, 32, 8, 6, 2), (20_000, 256, 256, 3, 2)]:
        X, _ = ko.make_blobs(n, d, k, seed=17)
        C0 = X[:k].copy()
        ref = ko.lloyd([X], C0, iters, -1.0)
        out = ctx.kmeans_fit(_dev(X), k, init=C0, max_iter=iters, tol=-1.0)
        assert ctx.stats()["last_path"] in (1, 2)
        Cg = out["cluster_centers_"].cpu().numpy()
        labels, _ = ctx.kmeans_assign(_dev(X), out["cluster_centers_"])
        assert ctx.stats()["last_path"] == want_path
        cmp = ko.compare_labels(X, Cg, labels.cpu().numpy(), tau=TAU)
        assert cmp["n_mismatch_outside_margin"] == 0, cmp
        # trajectories agree unless an admissible (< 1e-6 margin) tie row sent them apart: check one exact step instead
        C1, _, _ = ko.lloyd_iteration([X], C0)
        one = ctx.kmeans_fit(_dev(X), k, init=C0, max_iter=1, tol=-1.0)["cluster_centers_"].cpu().numpy()
        lab0, _, margin0 = ko.assign(X, C0)
        if margin0.min() > 1e-5:
            assert ko.max_center_rel_err(one, C1) <= CENTER_RTOL
            assert ko.max_center_rel_err(Cg, ref["centers"]) <= 1e-3


def test_baseline_cfg2_full_size_every_row(ctx):
    """BASELINE configs[1] at its real size (k=64, n=10 M, d=128, one GPU): every row's label and min distance against an
    fp64 PyTorch restatement on the device, one Lloyd step against the fp64 sums of those labels, bitwise determinism."""
    import torch
    from _fullsize import check_every_row, check_one_step, make_blobs

    ctx.set_option("kernel_path", 2)
    X, C = make_blobs(10_000_000, 128, 64, seed=21)
    r = check_every_row(ctx, X, C)
    assert r["outside_margin"] == 0, {k: v for k, v in r.items() if k != "labels"}
    assert r["worst_mindist_rel_err"] <= 2e-4, r["worst_mindist_rel_err"]
    rel, same = check_one_step(ctx, X, C, r["labels"])
    assert rel <= 1e-5 and same, (rel, same)
    del X
    torch.cuda.empty_cache()
