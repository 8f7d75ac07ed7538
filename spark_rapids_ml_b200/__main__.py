"""`python -m spark_rapids_ml_b200 script.py [args...]` or `python -m spark_rapids_ml_b200 -m module [args...]`: run a
Python program with the no-import-change mode of install.py switched on, so that its `pyspark.ml.clustering.KMeans`
is this package's.  Reference: python/src/spark_rapids_ml/__main__.py."""
import argparse
import runpy
import sys


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog="python -m spark_rapids_ml_b200",
                                 description="Run a program with pyspark.ml.clustering.KMeans replaced by this package.")
    ap.add_argument("-m", dest="module", default=None, help="run a module as __main__ (like python -m)")
    ap.add_argument("rest", nargs=argparse.REMAINDER, help="script path (unless -m) followed by its arguments")
    ns = ap.parse_args(argv)
    if ns.module is None and not ns.rest:
        ap.print_help()
        return 1
    from . import install  # noqa: F401  (the import installs the proxies)

    if ns.module is not None:
        sys.argv[:] = [ns.module] + ns.rest
        runpy.run_module(ns.module, run_name="__main__", alter_sys=True)
    else:
        sys.argv[:] = ns.rest
        runpy.run_path(ns.rest[0], run_name="__main__")
    return 0


if __name__ == "__main__":
    sys.exit(main())
