"""b2k_gmm_fit at R = 2 and 3 ranks on one GPU through the in-process NCCL stand-in (child: tests/_ranks_child_gmm.py):
the seeded start is bitwise the one-rank start, the fit agrees with the one-rank fit within the E pass's tolerance and
is the same on every rank; a component with no support fits on every rank of an uneven split; an empty partition fails
on every rank with one message."""
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import _ranks_child as child
import _ranks_child_gmm as gmm_child

pytestmark = pytest.mark.gpu

CHILD = os.path.join(child.HERE, "_ranks_child_gmm.py")
RENDEZVOUS_TIMEOUT_S = 20
_RUNS = {}


def _run(R):
    if R not in _RUNS:
        if not os.path.exists(child.FAKE_NCCL):
            pytest.fail(f"{child.FAKE_NCCL} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'`")
        env = dict(os.environ, B2K_NCCL_LIB=child.FAKE_NCCL, B2K_FAKE_NCCL_TIMEOUT_S=str(RENDEZVOUS_TIMEOUT_S))
        if sys.flags.no_user_site:
            env["PYTHONNOUSERSITE"] = "1"
        with tempfile.TemporaryDirectory() as td:
            out = os.path.join(td, "out.pkl")
            p = subprocess.run([sys.executable, CHILD, "gmm", str(R), out], env=env, cwd=child.ROOT,
                               capture_output=True, text=True, timeout=600)
            if p.returncode != 0 or not os.path.exists(out):
                pytest.fail(f"R={R}: the child failed (exit {p.returncode})\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}")
            with open(out, "rb") as f:
                _RUNS[R] = pickle.load(f)
    return _RUNS[R]


@pytest.mark.parametrize("R", [2, 3])
@pytest.mark.parametrize("name,d,k,path", gmm_child.GMM_CASES)
def test_start_bitwise_and_fit_within_tolerance(R, name, d, k, path):
    c = _run(R)[name]
    assert "harness_error" not in c, c.get("harness_error")
    assert c["errs"] == [None] * R, c["errs"]
    one = c["single"]
    for o in c["outs"]:
        for key in ("weights", "means", "covs"):
            np.testing.assert_array_equal(o["start"][key], one["start"][key])
        for key in ("weights", "means", "covs", "cluster_sizes"):
            np.testing.assert_array_equal(o["fit"][key], c["outs"][0]["fit"][key])
        assert o["fit"]["log_likelihood"] == c["outs"][0]["fit"]["log_likelihood"]
    f, s = c["outs"][0]["fit"], one["fit"]
    atol = 1e-3 if path == 0 else 1e-9
    np.testing.assert_allclose(f["weights"], s["weights"], atol=atol)
    np.testing.assert_allclose(f["means"], s["means"], atol=10 * atol)
    np.testing.assert_allclose(f["covs"], s["covs"], atol=10 * atol)
    assert abs(f["log_likelihood"] - s["log_likelihood"]) <= atol * abs(s["log_likelihood"])
    assert f["cluster_sizes"].sum() == 3000


def test_dead_component_at_two_ranks():
    # the E pass is the generic one (d = 132) and reads each row alone, so the ranks and the one-rank run differ only in
    # the order of the fp64 sums and in the wgmma Gram's row ranges: each covariance is within 1e-5 of its component's
    # spread (tests/test_gpu_gram.py) on both sides
    c = _run(2)["dead"]
    assert "harness_error" not in c, c.get("harness_error")
    assert c["errs"] == [None, None], c["errs"]
    f = c["outs"][0]["fit"]
    for o in c["outs"]:
        for key in ("weights", "means", "covs", "cluster_sizes"):
            np.testing.assert_array_equal(o["fit"][key], f[key])
    s = c["single"]["fit"]
    assert f["n_iter"] == s["n_iter"] == 1
    np.testing.assert_allclose(f["weights"], s["weights"], rtol=1e-9, atol=0)
    np.testing.assert_allclose(f["means"], s["means"], rtol=0, atol=1e-9)
    for j in range(3):
        spread = np.diag(s["covs"][j]).max()
        assert np.abs(f["covs"][j] - s["covs"][j]).max() <= 2e-5 * spread, j
    lam = np.linalg.eigvalsh(f["covs"][2])
    assert lam.max() > 0 and lam.min() >= -1e-6 * lam.max(), (lam.min(), lam.max())   # PSD within the Gram's bound
    assert f["weights"][2] < 1e-80
    assert f["cluster_sizes"].sum() == 3 * 4096 + 5


@pytest.mark.parametrize("R", [2, 3])
def test_empty_partition_fails_on_every_rank(R):
    c = _run(R)["empty"]
    assert "harness_error" not in c, c.get("harness_error")
    errs = c["errs"]
    assert all(e is not None for e in errs) and all(e == errs[0] for e in errs), errs
    assert "empty partition (rank 1" in errs[0], errs[0]
    assert c["secs"] < RENDEZVOUS_TIMEOUT_S / 2, c["secs"]
