"""Random forests' multi-rank path on one GPU: R = 2 and 3 ranks as threads of a child interpreter
(tests/_ranks_child_rf.py) through the in-process NCCL stand-in, with uneven shards and a rank of a few rows.  Every
rank's forest must be byte-identical to the one-rank forest on the concatenated rows (and to the oracle); an empty rank,
a NaN and a bad label on one rank must fail on every rank with the same message."""
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import _ranks_child as rc
import _ranks_child_rf as child
import rf_oracle as ro

pytestmark = pytest.mark.gpu

CHILD = os.path.join(child.HERE, "_ranks_child_rf.py")
CHILD_TIMEOUT_S = 600
RENDEZVOUS_TIMEOUT_S = 20
RANKS = [2, 3]
_RUNS = {}
SPECS = {s[0]: s for s in child.case_specs()}


def _run(R):
    if R not in _RUNS:
        _RUNS[R] = _spawn(R)
    res = _RUNS[R]
    if isinstance(res, str):
        pytest.fail(res)
    return res


def _spawn(R):
    if not os.path.exists(rc.FAKE_NCCL):
        return f"{rc.FAKE_NCCL} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'`"
    env = dict(os.environ, B2K_NCCL_LIB=rc.FAKE_NCCL, B2K_FAKE_NCCL_TIMEOUT_S=str(RENDEZVOUS_TIMEOUT_S))
    if sys.flags.no_user_site:
        env["PYTHONNOUSERSITE"] = "1"
    with tempfile.TemporaryDirectory() as td:
        out = os.path.join(td, "out.pkl")
        try:
            p = subprocess.run([sys.executable, CHILD, str(R), out], env=env, cwd=rc.ROOT, capture_output=True,
                               text=True, timeout=CHILD_TIMEOUT_S)
        except subprocess.TimeoutExpired as e:
            return f"R={R}: the child timed out after {CHILD_TIMEOUT_S} s\n{(e.stderr or '')[-4000:]}"
        if p.returncode != 0 or not os.path.exists(out):
            return f"R={R}: the child failed (exit {p.returncode})\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}"
        with open(out, "rb") as f:
            return pickle.load(f)


@pytest.mark.parametrize("R", RANKS)
@pytest.mark.parametrize("name", list(SPECS))
def test_ranks_equal_one_rank_bytewise(R, name):
    c = _run(R)[name]
    assert "harness_error" not in c, c.get("harness_error")
    assert c["errs"] == [None] * R, c["errs"]
    assert c["group_error"] == "", c["group_error"]
    assert c["trace"][0] and all(t == c["trace"][0] for t in c["trace"]), c["trace"]
    one = c["single"]
    for o in c["outs"]:
        assert o["bits"] == one["bits"]
        assert o["path"] == one["path"]
    _, X, y, kw, _, _ = SPECS[name]
    okw = dict(kw)
    okw["impurity_name"] = okw.pop("impurity", "gini")
    assert child._forest_json(ro.fit(X, y, **okw)) == one["bits"]


@pytest.mark.parametrize("R", RANKS)
@pytest.mark.parametrize("name, msg", [("fail_nan", "RandomForest input contains NaN or infinity"),
                                       ("fail_label", "Labels MUST be Integers"),
                                       ("fail_empty_rank", "empty partition")])
def test_every_rank_fails_together(R, name, msg):
    c = _run(R)[name]
    assert "harness_error" not in c, c.get("harness_error")
    errs = c["errs"]
    assert all(e is not None for e in errs), errs
    assert all(e == errs[0] for e in errs), errs
    assert msg in errs[0], errs[0]
    assert "timed out" not in c["group_error"], c["group_error"]
    assert c["secs"] < RENDEZVOUS_TIMEOUT_S / 2, c["secs"]
