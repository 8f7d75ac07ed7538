"""The pyspark branch of the Spark<->worker boundary (SURVEY.md 8b "B1"), checked without a pyspark / JVM: a fresh
interpreter imports the library with tests/fake_pyspark on sys.path (HAVE_PYSPARK = True) and runs fit / transform on a
recording fake pyspark DataFrame.  What must hold (reference call sites in parentheses):

  * KMeans IS a pyspark.ml.Estimator with pyspark Params, KMeansModel a pyspark.ml.Model
  * fit: select/cast of the feature column, VectorUDT -> vector_to_array (core.py:523-525), repartition(num_workers),
    mapInPandas(_train_udf, schema).rdd.barrier().mapPartitions(...).collect() (core.py:1005-1013), the worker takes its
    context from pyspark.BarrierTaskContext.get(), local mode derived from the session's master URL
  * transform: pandas_udf("int") over struct(features) appended with withColumn (core.py:1846-1878)

CPU version: the device pieces of the worker (GPU selection, CumlContext, the device row appender, the fit function)
are replaced by host stand-ins — the WIRING is what is under test.  GPU version: nothing is replaced."""
import json
import os
import subprocess
import sys
import textwrap

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = os.path.join(ROOT, "tests", "fake_pyspark")

_COMMON = '''
import sys, json
import numpy as np
import pyspark
from pyspark import CALLS
from pyspark.sql import DataFrame
import spark_rapids_ml_b200.sparkshim as shim
assert shim.HAVE_PYSPARK
from spark_rapids_ml_b200.clustering import KMeans, KMeansModel
import pyspark.ml, pyspark.ml.param
assert issubclass(KMeans, pyspark.ml.Estimator) and issubclass(KMeansModel, pyspark.ml.Model)
assert isinstance(KMeans().getParam("k"), pyspark.ml.param.Param)
sess = shim.LocalSession()
rng = np.random.default_rng(0)
ctr = rng.uniform(-10, 10, size=(4, 8))
X = (ctr[rng.integers(0, 4, size=600)] + 0.05 * rng.normal(size=(600, 8)))
'''

_CPU_STUBS = '''
import pandas as pd
import spark_rapids_ml_b200.core as core
import spark_rapids_ml_b200.common.cuml_context as cc

class HostAppender:
    def __init__(self, ctx, d, first_capacity=0):
        self.d, self.rows_ = d, []
    def append_values(self, values, offsets, n_b):
        lo = int(offsets[0]) if offsets is not None else 0
        self.rows_.append(np.asarray(values[lo:lo + n_b * self.d], dtype=np.float32).reshape(n_b, self.d))
    def append_columns(self, cols):
        self.rows_.append(np.stack(cols, 1).astype(np.float32))
    def finish(self):
        return np.concatenate(self.rows_)

class HostContext:
    def __init__(self, *a, **k): self.handle, self._loop = object(), None
    def __enter__(self): return self
    def __exit__(self, *a): return None

core.DeviceRowAppender = HostAppender
cc.CumlContext = HostContext
core._CumlCommon._set_gpu_device = staticmethod(lambda context, is_local, is_transform=False: 0)

def host_fit_func(self, dataset, extra_params=None):
    def fit(inputs, params):
        Xh = inputs[0][0]
        k = params[core.param_alias.cuml_init]["n_clusters"]
        C = Xh[:k].astype(np.float64)
        for _ in range(5):
            lab = ((Xh[:, None, :] - C[None]) ** 2).sum(-1).argmin(1)
            C = np.stack([Xh[lab == j].mean(0) if (lab == j).any() else C[j] for j in range(k)])
        return {"chunk_id": [0], "cluster_centers_": [C.tolist()], "n_cols": [Xh.shape[1]], "dtype": ["float32"]}
    return fit
KMeans._get_cuml_fit_func = host_fit_func

class HostModel:
    def __init__(self, C): self.C = C
    def close(self): pass

def host_transform_func(self, dataset, eval_metric_info=None):
    C = np.asarray(self.cluster_centers_)
    def construct(gpu=0): return HostModel(C)
    def transform(model, dfs):
        out = []
        for df in dfs:
            col = df[core.alias.data] if hasattr(df, "columns") and core.alias.data in df.columns else df
            A = np.array([np.asarray(r, dtype=np.float64) for r in col])
            out.append((((A[:, None, :] - model.C[None]) ** 2).sum(-1).argmin(1).astype("int32"),))
        return out
    transform.row_bytes = 4 * C.shape[1]
    return construct, transform, None
KMeansModel._get_cuml_transform_func = host_transform_func
'''

_BODY = '''
results = {}
for kind in ("array<float>", "array<double>", "vector"):
    del CALLS[:]
    Xs = X.astype(np.float32) if kind == "array<float>" else X
    local = sess.from_numpy(Xs, col="features", num_partitions=2)
    df = DataFrame(local, vector_cols=("features",) if kind == "vector" else ())
    model = KMeans(k=4, maxIter=5, initMode="random", seed=1, num_workers=1).setFeaturesCol("features").fit(df)
    fit_calls = [c[0] for c in CALLS]
    C = np.array(model.cluster_centers_)
    del CALLS[:]
    out = model.transform(df)
    tr_calls = [c[0] for c in CALLS]
    pred = np.array([r["prediction"] for r in out.collect()])
    truth = ((X[:, None, :] - C[None]) ** 2).sum(-1).argmin(1)
    results[kind] = {"fit_calls": fit_calls, "transform_calls": tr_calls, "pred_ok": bool((pred == truth).all()),
                     "n_centers": int(C.shape[0]), "pred_col": "prediction" in out.columns}
print("RESULT " + json.dumps(results))
'''


def _run(script: str) -> dict:
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([FAKE, ROOT, env.get("PYTHONPATH", "")])
    res = subprocess.run([sys.executable, "-c", textwrap.dedent(script)], env=env, capture_output=True, text=True,
                         timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
    line = [l for l in res.stdout.splitlines() if l.startswith("RESULT ")][-1]
    return json.loads(line[len("RESULT "):])


def _check(results: dict) -> None:
    for kind, r in results.items():
        fc = r["fit_calls"]
        # the reference's fit plan, in order
        i_map, i_bar, i_mp, i_col = (fc.index(x) for x in ("mapInPandas", "rdd.barrier", "rdd.mapPartitions", "rdd.collect"))
        assert fc.index("select") < fc.index("repartition") < i_map < i_bar < i_mp < i_col, (kind, fc)
        assert "BarrierTaskContext.get" in fc, (kind, fc)          # the worker asked pyspark for its barrier context
        assert ("vector_to_array" in fc) == (kind == "vector"), (kind, fc)
        tc = r["transform_calls"]
        assert tc.index("pandas_udf") < tc.index("withColumn"), (kind, tc)
        assert ("vector_to_array" in tc) == (kind == "vector"), (kind, tc)
        assert r["pred_ok"] and r["pred_col"] and r["n_centers"] == 4, (kind, r)


def test_pyspark_branch_wiring_with_grouped_host_stand_ins():
    _check(_run(_COMMON + _CPU_STUBS + _BODY))


@pytest.mark.gpu
def test_pyspark_branch_end_to_end_on_gpu():
    """Same plan, nothing replaced: the worker function ingests the Arrow batches on the device and calls libb2kmeans."""
    _check(_run(_COMMON + _BODY))


_PERSIST = '''
import os, tempfile
from pyspark import SparkContext
SparkContext._active_spark_context = SparkContext()      # a live SparkContext: persistence goes through pyspark.ml.util
import pyspark.ml.util as U
root = tempfile.mkdtemp()
km = KMeans(k=4, maxIter=9, seed=2, num_workers=1).setFeaturesCol("f")
del CALLS[:]
w = km.write()
assert isinstance(w, U.MLWriter)
w.overwrite().save(os.path.join(root, "est"))
est_calls = [c[0] for c in CALLS]
km2 = KMeans.load(os.path.join(root, "est"))
m = KMeansModel(cluster_centers_=[[0.0, 1.0], [2.0, 3.0]], n_cols=2, dtype="float32")
m._set(featuresCol="f")
del CALLS[:]
m.write().overwrite().save(os.path.join(root, "model"))
model_calls = [c[0] for c in CALLS]
del CALLS[:]
r = KMeansModel.read()
assert isinstance(r, U.MLReader)
m2 = r.load(os.path.join(root, "model"))
load_calls = [c[0] for c in CALLS]
# what the Spark-side writer left on disk is also what the local reader accepts (and the reference's layout)
SparkContext._active_spark_context = None
m3 = KMeansModel.load(os.path.join(root, "model"))
print("RESULT " + json.dumps({
    "est_calls": est_calls, "model_calls": model_calls, "load_calls": load_calls,
    "est_ok": km2.uid == km.uid and km2.getK() == 4 and km2.getMaxIter() == 9 and km2.getFeaturesCol() == "f"
              and km2.cuml_params["n_clusters"] == 4,
    "model_ok": m2.uid == m.uid and m2.cluster_centers_ == m.cluster_centers_ and m2.getFeaturesCol() == "f",
    "local_reads_spark_layout": m3.uid == m.uid and m3.cluster_centers_ == m.cluster_centers_,
    "files": sorted(os.listdir(os.path.join(root, "model"))),
}))
'''

_INSTALL = '''
import pyspark.ml.clustering as stock_mod
StockKMeans = stock_mod.KMeans
import spark_rapids_ml_b200.install as inst
from pyspark.ml.clustering import KMeans as K1, KMeansModel as M1, BisectingKMeans as B1
import pyspark.ml.clustering as proxied
import pyspark.ml
from pyspark.ml.clustering import _sibling_lookup
res = {
    "user_import_is_accelerated": K1 is KMeans and M1 is KMeansModel,
    "attribute_access_is_accelerated": proxied.KMeans is KMeans and pyspark.ml.clustering.KMeans is KMeans,
    "other_names_untouched": getattr(B1, "stock", False) is True,
    "pyspark_ml_itself_sees_stock": _sibling_lookup() is StockKMeans,
    "this_package_sees_stock": inst._called_from_library.__module__ == "spark_rapids_ml_b200.install",
    "missing_attr_raises": False,
}
try:
    proxied.NoSuchThing
except AttributeError:
    res["missing_attr_raises"] = True
inst.install()                                   # idempotent
res["idempotent"] = proxied is sys.modules["pyspark.ml.clustering"]
inst.uninstall()
res["uninstall_restores"] = sys.modules["pyspark.ml.clustering"].KMeans is StockKMeans
# python -m spark_rapids_ml_b200 script.py: the script's plain pyspark import is the accelerated class
import os, tempfile, subprocess
d = tempfile.mkdtemp()
with open(os.path.join(d, "user_script.py"), "w") as f:
    f.write("import sys\\nfrom pyspark.ml.clustering import KMeans\\nprint('SCRIPT', KMeans.__module__, sys.argv[1:])\\n")
out = subprocess.run([sys.executable, "-m", "spark_rapids_ml_b200", os.path.join(d, "user_script.py"), "a", "b"],
                     capture_output=True, text=True, env=os.environ)
res["runner_output"] = [l for l in out.stdout.splitlines() if l.startswith("SCRIPT")] or [out.stderr[-300:]]
print("RESULT " + json.dumps(res))
'''


def test_pyspark_branch_persistence_goes_through_mlwriter():
    r = _run(_COMMON + _PERSIST)
    assert r["est_calls"][:2] == ["MLWriter.save", "DefaultParamsWriter.saveMetadata"], r
    mc = r["model_calls"]
    assert mc.index("DefaultParamsWriter.saveMetadata") < mc.index("rdd.saveAsTextFile"), r
    assert mc.count("rdd.saveAsTextFile") == 2 and "sc.parallelize" in mc, r          # metadata + data
    lc = r["load_calls"]
    assert lc.index("DefaultParamsReader.loadMetadata") < lc.index("DefaultParamsReader.getAndSetParams"), r
    assert "sc.textFile" in lc, r
    assert r["est_ok"] and r["model_ok"] and r["local_reads_spark_layout"] and r["files"] == ["data", "metadata"], r


def test_install_proxy_swaps_kmeans_for_user_code_only():
    r = _run(_COMMON + _INSTALL)
    for key in ("user_import_is_accelerated", "attribute_access_is_accelerated", "other_names_untouched",
                "pyspark_ml_itself_sees_stock", "missing_attr_raises", "idempotent", "uninstall_restores"):
        assert r[key] is True, (key, r)
    assert r["runner_output"] == ["SCRIPT spark_rapids_ml_b200.clustering ['a', 'b']"], r


_RETRY = '''
import logging
records = []
class H(logging.Handler):
    def emit(self, r): records.append(r.getMessage())
logging.getLogger().addHandler(H())
local = sess.from_numpy(X.astype(np.float32), col="features", num_partitions=3)
df = DataFrame(local).coalesce(1)                  # same partition count as num_workers: no repartition before the stage
del CALLS[:]
est = KMeans(k=4, maxIter=5, initMode="random", seed=1, num_workers=1).setFeaturesCol("features")
est.logger.addHandler(H())
model = est.fit(df)
calls = [c[0] for c in CALLS]
print("RESULT " + json.dumps({"calls": calls, "n_centers": len(model.cluster_centers_),
                              "warned": any("Retrying with repartitioning" in m for m in records)}))
'''


def test_barrier_rdd_chain_error_is_retried_after_repartition():
    """reference core.py:1245-1257 / tests/test_kmeans.py:285-310: a coalesced input makes Spark refuse the barrier stage;
    the estimator logs the warning and fits the repartitioned dataset."""
    r = _run(_COMMON + _CPU_STUBS + _RETRY)
    c = r["calls"]
    assert c.count("mapInPandas") == 2 and c.count("rdd.collect") == 2, r
    first_collect = c.index("rdd.collect")
    assert "repartition" in c[first_collect:] and "repartition" not in c[:first_collect], r
    assert r["warned"] and r["n_centers"] == 4, r


_STAGE = '''
import pyspark.sql as ps
ps.CLUSTER_CONF = {"spark.master": "spark://head:7077", "spark.executor.cores": "8",
                   "spark.executor.resource.gpu.amount": "1", "spark.task.resource.gpu.amount": "0.125"}
local = sess.from_numpy(X.astype(np.float32), col="features", num_partitions=1)
del CALLS[:]
# a cluster master: the GPU comes from the task's resources, as under a real scheduler
import pyspark
pyspark.TaskContext.resources = lambda self: {"gpu": type("R", (), {"addresses": ["0"]})()}
model = KMeans(k=4, maxIter=5, initMode="random", seed=1, num_workers=1).setFeaturesCol("features").fit(DataFrame(local))
calls = [(c[0], c[1]) for c in CALLS if c[0] in ("rdd.barrier", "rdd.mapPartitions", "rdd.withResources", "rdd.collect")]
print("RESULT " + json.dumps({"calls": calls, "n_centers": len(model.cluster_centers_)}))
'''


def test_training_stage_gets_its_own_resource_profile_on_a_cluster():
    """reference core.py:693-740: on a standalone cluster the barrier stage is submitted with a task resource profile
    (more than half of the executor's cores + one GPU) between mapPartitions and collect."""
    r = _run(_COMMON + _CPU_STUBS + _STAGE)
    names = [c[0] for c in r["calls"]]
    assert names == ["rdd.barrier", "rdd.mapPartitions", "rdd.withResources", "rdd.collect"], r
    assert r["calls"][2][1] == {"cpus": 5, "gpu": 1.0} and r["n_centers"] == 4, r
