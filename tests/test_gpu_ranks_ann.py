"""IVF-Flat at R = 2 and 3 ranks on one GPU through the in-process NCCL stand-in (child: tests/_ranks_child_ann.py):
uneven shards, a rank with no items, a rank with no queries, ranks that hold nothing.  With injected centres the
result on integer data is bitwise the one-rank result; with trained centres every rank holds the same centres, bitwise
equal to the one-rank fit, and the result meets the oracle; errors fail on every rank with one message."""
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import _ranks_child as child
import _ranks_child_ann as ann_child
import ann_oracle as ao

pytestmark = pytest.mark.gpu

CHILD = os.path.join(child.HERE, "_ranks_child_ann.py")
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
            p = subprocess.run([sys.executable, CHILD, "ann", str(R), out], env=env, cwd=child.ROOT,
                               capture_output=True, text=True, timeout=600)
            if p.returncode != 0 or not os.path.exists(out):
                pytest.fail(f"R={R}: the child failed (exit {p.returncode})\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}")
            with open(out, "rb") as f:
                _RUNS[R] = pickle.load(f)
    return _RUNS[R]


def _case(R, name):
    c = _run(R)[name]
    assert "harness_error" not in c, c.get("harness_error")
    assert c["errs"] == [None] * R, c["errs"]
    assert c["group_error"] == "", c["group_error"]
    assert c["trace"][0] and all(t == c["trace"][0] for t in c["trace"]), c["trace"]
    for key in ("centers",):
        assert all(o[key].tobytes() == c["outs"][0][key].tobytes() for o in c["outs"]), f"ranks differ in {key}"
    return c


def _cat(c, key):
    return np.concatenate([o[key] for o in c["outs"]])


@pytest.mark.parametrize("R", [2, 3])
@pytest.mark.parametrize("name", ["w16", "g7"])
def test_injected_centres_integer_data_match_one_rank_bitwise(R, name):
    c = _case(R, f"int_{name}")
    s = c["single"]
    for key in ("dist", "idx", "lists", "probes"):
        got = _cat(c, key)
        assert got.tobytes() == s[key].tobytes(), key


@pytest.mark.parametrize("R", [2, 3])
@pytest.mark.parametrize("name", ["uneven", "query_only"])
def test_trained_centres_identical_on_every_rank_and_to_one_rank(R, name):
    c = _case(R, f"trained_{name}")
    s = c["single"]
    assert c["outs"][0]["centers"].tobytes() == s["centers"].tobytes()
    X, Q = ann_child.blobs_data()
    dist, idx, lists, probes = (_cat(c, key) for key in ("dist", "idx", "lists", "probes"))
    C = s["centers"]
    assert ao.check_lists(X, C, lists) == 0
    assert ao.check_probes(C, Q, probes) == 0
    assert ao.check_result(X, Q, 8, lists, probes, dist, idx) == {"n_outside_margin": 0, "n_fill": 0}
    # the same centres and lists: the result is the one-rank result up to the screen's shift point
    np.testing.assert_array_equal(lists, s["lists"])
    np.testing.assert_array_equal(probes, s["probes"])


@pytest.mark.parametrize("R", [2, 3])
@pytest.mark.parametrize("name,msg", [("nonfinite_item", "non-finite component"),
                                      ("nlist_too_large", "nlist = 2001 exceeds the 2000 training rows")])
def test_errors_fail_on_every_rank(R, name, msg):
    c = _run(R)[name]
    assert "harness_error" not in c, c.get("harness_error")
    errs = c["errs"]
    assert all(e is not None for e in errs) and all(e == errs[0] for e in errs), errs
    assert msg in errs[0], errs[0]
    assert c["secs"] < RENDEZVOUS_TIMEOUT_S / 2, c["secs"]
