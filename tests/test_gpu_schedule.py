"""The persistent fused kernels in steady state, and the paths the other GPU tests leave at their edges.

Every fused kernel runs a persistent grid (one CTA per SM, static round-robin over 128-row tiles: tile t runs on CTA
t mod grid) and feeds it through TMA rings whose mbarrier phase bit flips each time a ring wraps.  The X ring holds at
most 12 slots (WgCfg::SX in csrc/b2k_wg.cuh), i.e. at most 12 tiles per turn, so slot reuse, the parity expression and
the shared-memory sums accumulating over many tiles only run once a CTA has more than 12 tiles.  Option `grid_limit`
caps the grid: at n = 20011 (157 tiles, a ragged last one) a grid of 1, 3 or 7 CTAs gives 157, 53 or 23 tiles per CTA,
and 3 and 7 give the CTAs unequal counts.  Per-row results do not depend on the schedule, so labels and min distances
must be bitwise equal to the full grid's; a Lloyd step must match the fp64 sums of the device's labels and be bitwise
reproducible at each grid.

Also here: the screening kernel's fix-up of entries past its mask capacity, the inertia identity of every family, the
generic kernels on the shapes only they take (d > 256, d % 4 != 0, a misaligned X, the CW = 32 and atomic updates), the
PCA Gram pass at tiny and ragged row counts with one CTA per tile, the projection kernel against an elementwise bound,
and the profiled build of the 3xTF32 kernel.
"""
import contextlib

import numpy as np
import pytest

import pca_oracle as po

pytestmark = pytest.mark.gpu
TILE = 128          # B2K_FUSED_TILE_ROWS
N = 20011           # 157 tiles, the last one ragged
MAX_RING = 12       # most tiles one turn of an X ring holds (WgCfg::SX <= 12, one chunk per tile at DP = 32)
STEP_RTOL = 1e-5
CFG2_ROWS_PER_CTA = 2048
DEFAULTS = {"kernel_path": 0, "grid_limit": 0, "variant_t": 0, "profile_fused": 0, "collect_recheck": 0}
# (k, d) -> (KP, DP): every 3xTF32 instantiation of csrc/b2k_fused_tc.cu kInst, as in test_gpu_update.py
TC_SHAPES = [(5, 20), (16, 64), (12, 128), (32, 32), (24, 60), (32, 128), (48, 32), (64, 64), (64, 128), (100, 64),
             (128, 128)]


@pytest.fixture(scope="module")
def ctx():
    from spark_rapids_ml_b200 import _native

    c = _native.Context(0)
    yield c
    c.close()


@contextlib.contextmanager
def _options(ctx, **kw):
    try:
        for key, v in kw.items():
            ctx.set_option(key, v)
        yield
    finally:
        for key in kw:
            ctx.set_option(key, DEFAULTS[key])


def _cdiv(a, b):
    return -(-a // b)


def _sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def _tc_grid(n, grid_limit):
    """the persistent grid of the 3xTF32 kernel (b2k_fused_plan)"""
    ntiles = _cdiv(n, TILE)
    g = _sm_count() if grid_limit == 0 else min(grid_limit, _sm_count())
    return max(min(g, ntiles), 1)


def _t_grid(n, grid_limit):
    """the screening kernel rounds the grid to whole 8-CTA clusters, at least one (b2k_fused_t_plan)"""
    return max(_tc_grid(n, grid_limit) // 8 * 8, 8)


def _step_rtol(labels, k, grid, per=1):
    """Tolerance of one Lloyd step.  A CTA (per = 1) or an 8-CTA cluster (per = 8) adds each cluster's rows into fp32
    sums over all of its tiles, so the rounding error of a centre grows with m, the most rows of one cluster that one
    such accumulator takes (tile t runs on CTA t mod grid).  1e-5 holds up to cfg2's per-CTA load (2048 rows); beyond it
    the tolerance grows linearly with m, as the error bound of an fp32 sum does."""
    import torch

    owner = (torch.arange(labels.shape[0], device=labels.device) // TILE) % grid // per
    m = int(torch.bincount(owner * k + labels.long()).max())
    return STEP_RTOL * max(1.0, m / CFG2_ROWS_PER_CTA), m


def _blobs(n, d, k, seed):
    from _fullsize import make_blobs

    return make_blobs(n, d, k, seed)


def _uniform(n, d, k, seed):
    """rows uniform in the unit cube; centres drawn from the rows and pulled three quarters of the way to its middle, so
    that the distances of a row to all centres are close: most rows are near-ties for the screening kernel"""
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    X = torch.rand((n, d), generator=g, device="cuda")
    return X, (0.5 + 0.25 * (X[torch.randperm(n, generator=g, device="cuda")[:k]] - 0.5)).contiguous()


def _check_labels(ctx, X, C):
    from _fullsize import check_every_row

    r = check_every_row(ctx, X, C)
    assert r["outside_margin"] == 0, {key: v for key, v in r.items() if key != "labels"}
    assert r["worst_mindist_rel_err"] <= 2e-4, r["worst_mindist_rel_err"]
    return r["labels"]


# ---------------------------------------------------------------------------------------------------------------------
# 3xTF32 kernel: every instantiation, far past one turn of its rings
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k,d", TC_SHAPES)
def test_tc_every_instantiation_past_the_ring(ctx, k, d):
    import torch

    from _fullsize import check_one_step

    X, C = _blobs(N, d, k, seed=k * 1000 + d + 7)
    ntiles = _cdiv(N, TILE)
    with _options(ctx, kernel_path=2):
        labels = _check_labels(ctx, X, C)
        lab0, md0 = ctx.kmeans_assign(X, C, want_mindist=True)
        assert torch.equal(lab0, labels)
    for gl in (0, 1, 3, 7):
        grid = _tc_grid(N, gl)
        if gl:
            assert _cdiv(ntiles, grid) > MAX_RING, (gl, grid)
        with _options(ctx, kernel_path=2, grid_limit=gl):
            lab, md = ctx.kmeans_assign(X, C, want_mindist=True)
            assert ctx.stats()["last_path"] == 2
            assert torch.equal(lab, lab0), (gl, int((lab != lab0).sum()))
            assert torch.equal(md, md0), gl
            before = ctx.stats()["fused_tc_launches"]
            rel, same = check_one_step(ctx, X, C, lab0)
            assert ctx.stats()["last_path"] == 2 and ctx.stats()["fused_tc_launches"] > before
            tol, m = _step_rtol(lab0, k, grid)
            assert rel <= tol, {"grid_limit": gl, "rel": rel, "tol": tol, "m": m}
            assert same, f"two runs of one Lloyd step differ at grid_limit = {gl}"


# ---------------------------------------------------------------------------------------------------------------------
# screening kernel (variant 1): both instantiations, the cluster update and the fix-up past the mask capacity
# ---------------------------------------------------------------------------------------------------------------------
def _mask_overflow_floor(n, grid):
    """nseg * mask_cap of t_layout (csrc/b2k_fused_t.cu): the most deferred rows that can all carry a candidate mask"""
    ntiles = _cdiv(n, TILE)
    nit_max = _cdiv(ntiles, grid)
    mask_cap = min(nit_max * TILE, _cdiv(nit_max, 4) * TILE)
    return grid * mask_cap


@pytest.mark.parametrize("gen", ["blobs", "uniform"])
@pytest.mark.parametrize("k,d", [(256, 256), (200, 160), (64, 128)])
def test_screening_past_the_ring(ctx, k, d, gen):
    """DP = 256 and DP = 128 (forced with variant_t).  At n = 20 * 128 - 37 and grid 16 the first cluster runs two
    steps and half of its CTAs run an empty second step."""
    import torch

    from _fullsize import check_one_step

    make = _blobs if gen == "blobs" else _uniform
    for n in (N, 20 * TILE - 37):
        X, C = make(n, d, k, seed=k + d + n)
        with _options(ctx, kernel_path=2, variant_t=1):
            labels = _check_labels(ctx, X, C)
            lab0, md0 = ctx.kmeans_assign(X, C, want_mindist=True)
            assert torch.equal(lab0, labels)
        for gl in (0, 8, 16):
            grid = _t_grid(n, gl)
            if gl == 8 and n == N:
                assert _cdiv(_cdiv(n, TILE), grid) > MAX_RING, grid
            with _options(ctx, kernel_path=2, variant_t=1, collect_recheck=1, grid_limit=gl):
                lab, md = ctx.kmeans_assign(X, C, want_mindist=True)
                st = ctx.stats()
                assert st["last_path"] == 2
                assert torch.equal(lab, lab0), (n, gl, int((lab != lab0).sum()))
                assert torch.equal(md, md0), (n, gl)
                if gen == "uniform" and n == N and gl == 8:
                    # more deferred rows than every segment's masks can hold: some entry took the every-cluster fix-up
                    floor = _mask_overflow_floor(n, grid)
                    assert st["recheck_rows"] > floor, (st["recheck_rows"], floor)
                rel, same = check_one_step(ctx, X, C, lab0)
                assert ctx.stats()["last_path"] == 2
                tol, m = _step_rtol(lab0, k, grid, per=8)
                assert rel <= tol, {"n": n, "grid_limit": gl, "rel": rel, "tol": tol, "m": m}
                assert same, f"two runs of one Lloyd step differ at n = {n}, grid_limit = {gl}"


# ---------------------------------------------------------------------------------------------------------------------
# inertia: the fixed-order fp64 sum of exactly the min distances kmeans_assign returns
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("family,k,d,opts", [
    ("3xtf32", 64, 128, {"kernel_path": 2}),
    ("3xtf32", 5, 20, {"kernel_path": 2}),
    ("screening", 256, 256, {"kernel_path": 2}),
    ("screening", 64, 128, {"kernel_path": 2, "variant_t": 1}),
    ("chunked", 300, 64, {}),
    ("generic", 64, 128, {"kernel_path": 1}),
    ("generic", 20, 260, {}),
])
def test_inertia_is_the_sum_of_the_min_distances(ctx, family, k, d, opts):
    """fit(init=C0, max_iter=0) runs no Lloyd step, so its inertia is the cost of C0: every family adds exactly the fp32
    min distance it writes for a row, and only the fp64 fold order differs from a plain sum of kmeans_assign's."""
    gen = _uniform if family == "screening" else _blobs
    X, C = gen(N, d, k, seed=k * 7 + d)
    for gl in (0, 8):
        with _options(ctx, grid_limit=gl, **opts):
            out = ctx.kmeans_fit(X, k, init=C, max_iter=0)
            assert out["n_iter_"] == 0
            assert ctx.stats()["last_path"] == (1 if family == "generic" else 2)
            _, md = ctx.kmeans_assign(X, C, want_mindist=True)
        s = float(md.double().sum())
        assert abs(out["inertia_"] - s) <= 1e-12 * s, (gl, out["inertia_"], s)


# ---------------------------------------------------------------------------------------------------------------------
# generic kernels, on the shapes only they take
# ---------------------------------------------------------------------------------------------------------------------
def _smem_optin():
    import torch

    return getattr(torch.cuda.get_device_properties(0), "shared_memory_per_block_optin", None)


@pytest.mark.parametrize("n,d,k,path", [
    (N, 260, 40, 0),        # d > 256
    (N, 384, 40, 0),
    (10007, 1000, 24, 0),
    (N, 130, 32, 0),        # d % 4 != 0
    (N, 257, 32, 0),
    (N, 16, 500, 1),        # 448 < k <= 1753: the CW = 32 update
    (N, 16, 1800, 1),       # k >= 1754: the atomic update
])
def test_generic_path_where_only_it_runs(ctx, n, d, k, path):
    from _fullsize import check_one_step

    X, C = _blobs(n, d, k, seed=d * 31 + k)
    optin = _smem_optin()
    if optin is not None and path == 1:   # plan_update (b2k_generic.cu): S[k][CW] f32 + counts[k] in optin - 1 KB
        cap = optin - 1024
        cw = 128 if k * (128 * 4 + 4) <= cap else 32 if k * (32 * 4 + 4) <= cap else 0
        assert cw == (32 if k == 500 else 0), (k, cap, cw)
    with _options(ctx, kernel_path=path):
        _check_labels(ctx, X, C)
        assert ctx.stats()["last_path"] == 1
        labels, _ = ctx.kmeans_assign(X, C)
        rel, same = check_one_step(ctx, X, C, labels)
        assert ctx.stats()["last_path"] == 1
        assert rel <= STEP_RTOL, rel
        if k < 1754:   # the atomic update adds in arrival order: not bitwise reproducible (DESIGN.md section 4.2)
            assert same, "two runs of one Lloyd step differ"


def _misaligned(X):
    """a contiguous copy of X that starts 4 bytes past a 16-byte boundary"""
    import torch

    buf = torch.empty(X.numel() + 4, dtype=X.dtype, device=X.device)
    off = (4 - (buf.data_ptr() // 4) % 4) % 4 + 1      # one float past an aligned element
    Xm = buf[off:off + X.numel()].view(X.shape)
    Xm.copy_(X)
    assert Xm.is_contiguous() and Xm.data_ptr() % 16 == 4
    return Xm


def _check_cov(X, out):
    """the covariance reconstructed from a k = d fit against the fp64 NumPy covariance"""
    n = X.shape[0]
    C = out["components_"]
    lam = out["singular_values_"] ** 2 / (n - 1)
    cov = C.T @ np.diag(lam) @ C
    ref = po.covariance(X)
    err, scale = float(np.abs(cov - ref).max()), float(np.abs(ref).max())
    assert err <= 1e-5 * scale, (err, scale)
    np.testing.assert_allclose(out["mean_"], X.astype(np.float64).mean(0), rtol=1e-6,
                               atol=1e-6 * float(np.abs(X).max()))


def test_misaligned_x_takes_the_generic_kernels(ctx):
    """a 16-byte-misaligned X cannot be a TMA source: auto runs the generic kernels, kernel_path = 2 fails loudly"""
    import torch

    from _fullsize import check_one_step
    from spark_rapids_ml_b200._native import B2KError

    n, d, k = N, 64, 32
    X0, C = _blobs(n, d, k, seed=77)
    X = _misaligned(X0)
    _check_labels(ctx, X, C)
    assert ctx.stats()["last_path"] == 1
    labels, _ = ctx.kmeans_assign(X, C)
    rel, same = check_one_step(ctx, X, C, labels)
    assert ctx.stats()["last_path"] == 1
    assert rel <= STEP_RTOL and same, (rel, same)
    with _options(ctx, kernel_path=2):
        with pytest.raises(B2KError):
            ctx.kmeans_assign(X, C)
        with pytest.raises(B2KError):
            ctx.kmeans_lloyd(X, C.clone(), 1, 0.0)
    Xp = _misaligned(torch.from_numpy(_pca_data(5000, 128, seed=3)).cuda())
    out = ctx.pca_fit(Xp, 128)
    assert ctx.stats()["last_path"] == 1
    _check_cov(Xp.cpu().numpy(), out)
    with _options(ctx, kernel_path=2):
        with pytest.raises(B2KError):
            ctx.pca_fit(Xp, 4)


# ---------------------------------------------------------------------------------------------------------------------
# PCA: the wgmma Gram pass at tiny and ragged row counts, one CTA per tile; the projection kernel
# ---------------------------------------------------------------------------------------------------------------------
def _pca_data(n, d, seed):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, d)) * (1.0 / np.sqrt(1.0 + np.arange(d))) + rng.normal(size=d)
    return X.astype(np.float32)


def _gram_ctas_per_tile(n, d, grid_limit):
    """P of b2k_pca_fit_impl: CTAs per 128 x 128 feature tile of the upper triangle"""
    nblk = _cdiv(d, 128)
    ntile = nblk * (nblk + 1) // 2
    nrange = max(1, _cdiv(n, 4096))
    sm = _sm_count() if grid_limit == 0 else min(grid_limit, _sm_count())
    return max(1, min(sm // ntile, nrange)), ntile, nrange


@pytest.mark.parametrize("n", [2, 3, 33, 4097, 3 * 4096 + 1])
def test_pca_gram_tiny_and_ragged_row_counts(ctx, n):
    """d = 132: a ragged second feature block in the off-diagonal tile; n <= 3 has a degenerate spectrum, so only the
    covariance is checked"""
    import torch

    d = 132
    X = _pca_data(n, d, seed=n)
    ntile = _gram_ctas_per_tile(n, d, 0)[1]
    for gl in (0, ntile):
        with _options(ctx, grid_limit=gl):
            out = ctx.pca_fit(torch.from_numpy(X).cuda(), d)
        assert ctx.stats()["last_path"] == 2
        if gl:
            assert _gram_ctas_per_tile(n, d, gl)[0] == 1
        _check_cov(X, out)


@pytest.mark.parametrize("d,n", [(132, 40000), (1020, 20000)])
def test_pca_gram_one_cta_per_tile(ctx, d, n):
    """grid_limit = the tile count: P = 1, so one CTA flushes every 4096-row range of its tile into its fp64 partial"""
    import torch

    X = _pca_data(n, d, seed=d)
    ntile = _gram_ctas_per_tile(n, d, 0)[1]
    P, _, nrange = _gram_ctas_per_tile(n, d, ntile)
    assert P == 1 and nrange > 1
    with _options(ctx, grid_limit=ntile):
        out = ctx.pca_fit(torch.from_numpy(X).cuda(), d)
    assert ctx.stats()["last_path"] == 2
    _check_cov(X, out)


@pytest.mark.parametrize("d", [4, 33, 1024])
@pytest.mark.parametrize("k", [1, 33, 64, 100])
def test_projection_elementwise_bound(ctx, k, d):
    """Y = X C^T of k_project as an fp32 FMA chain over d features: |Y - X C^T| <= 2 d 2^-24 (|X| |C|^T), in fp64.
    k > 32 spans several grid.y blocks of 32 components, n = 1, 255 and 257 the edges of a 256-row tile."""
    import torch

    g = torch.Generator(device="cuda").manual_seed(k * 10 + d)
    C = torch.randn((k, d), generator=g, device="cuda")
    C = (C / C.norm(dim=1, keepdim=True)).contiguous()
    for n in (1, 255, 257, 100_003):
        X = (torch.randn((n, d), generator=g, device="cuda") * 3.0 + 1.0).contiguous()
        Y = ctx.pca_transform(X, C)
        assert Y.shape == (n, k)
        X64, C64 = X.double(), C.double()
        err = (Y.double() - X64 @ C64.T).abs()
        bound = 2.0 * d * 2.0 ** -24 * (X64.abs() @ C64.abs().T)
        assert bool((err <= bound).all()), (n, float((err - bound).max()))
        del X, Y, X64, err, bound


# ---------------------------------------------------------------------------------------------------------------------
# the profiled build of the 3xTF32 kernel (option profile_fused, DESIGN.md section 6)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k,d", [(5, 20), (64, 128), (128, 128)])
def test_profiled_build_changes_no_result(ctx, k, d):
    import torch

    from spark_rapids_ml_b200._native import B2KError

    X, C = _blobs(N, d, k, seed=k + d)
    res = {}
    for prof in (0, 1):
        with _options(ctx, kernel_path=2, profile_fused=prof):
            lab, md = ctx.kmeans_assign(X, C, want_mindist=True)
            C1 = C.clone()
            ctx.kmeans_lloyd(X, C1, 1, 0.0)
            assert ctx.stats()["last_path"] == 2
            if prof:
                counters = ctx.fused_profile()
                assert counters.shape[0] == _tc_grid(N, 0) and (counters.sum(axis=(1, 2)) > 0).all()
        res[prof] = (lab, md, C1)
    for a, b in zip(res[0], res[1]):
        assert torch.equal(a, b)
    with _options(ctx, kernel_path=2, variant_t=1, profile_fused=1):
        with pytest.raises(B2KError) as e:
            ctx.kmeans_assign(X, C)
    assert e.value.code == 4   # B2K_ERR_UNSUPPORTED: the screening kernel has no profiled build
