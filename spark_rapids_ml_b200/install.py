"""No-import-change mode: after `import spark_rapids_ml_b200.install`, user code that says
`from pyspark.ml.clustering import KMeans` (or KMeansModel, or `from pyspark.ml.feature import PCA` / PCAModel) receives
this package's accelerated classes; every other attribute of those modules, and every access made from inside pyspark.ml
or from this package itself, still resolves to pyspark's own module.  Reference behaviour:
python/src/spark_rapids_ml/install.py:21-81 (a proxy module per pyspark.ml sub-module whose __getattr__ looks at the
calling file); only the sub-modules of the paths this package accelerates have an entry (SURVEY.md 8 f-4, f-1).

`python -m spark_rapids_ml_b200 script.py [args]` / `-m module [args]` runs a script with this mode on
(reference: python/src/spark_rapids_ml/__main__.py).
"""
from __future__ import annotations

import importlib
import os
import sys
import types
from typing import Any, Dict, Tuple

ACCELERATED: Dict[str, Tuple[str, ...]] = {"clustering": ("KMeans", "KMeansModel"), "feature": ("PCA", "PCAModel")}

_PKG_DIR = os.path.dirname(os.path.abspath(__file__))


class _PysparkMlProxy(types.ModuleType):
    """Stands in for pyspark.ml.<name> in sys.modules."""

    def __init__(self, name: str, original: types.ModuleType, accelerated: types.ModuleType, names: Tuple[str, ...]):
        super().__init__(original.__name__, original.__doc__)
        self.__dict__["_b2k_name"] = name
        self.__dict__["_b2k_original"] = original
        self.__dict__["_b2k_accelerated"] = accelerated
        self.__dict__["_b2k_names"] = frozenset(names)

    def __getattr__(self, attr: str) -> Any:   # only reached for names not in the proxy's own __dict__
        d = self.__dict__
        if attr in d["_b2k_names"] and not _called_from_library(sys._getframe(1)):
            return getattr(d["_b2k_accelerated"], attr)
        try:
            return getattr(d["_b2k_original"], attr)
        except AttributeError:
            raise AttributeError(f"module '{d['_b2k_original'].__name__}' has no attribute '{attr}'") from None

    def __dir__(self) -> Any:
        return dir(self.__dict__["_b2k_original"])


def _called_from_library(frame: Any) -> bool:
    """True when the attribute is being looked up by pyspark.ml itself or by this package (which must keep seeing the
    stock classes: e.g. pyspark.ml.pipeline / tuning import their siblings, and this package subclasses them)."""
    # `from m import X` runs the lookup inside importlib's machinery: skip those frames to find the importing file
    while frame is not None and frame.f_code.co_filename.startswith("<frozen importlib"):
        frame = frame.f_back
    if frame is None:
        return False
    path = os.path.abspath(frame.f_code.co_filename).replace(os.sep, "/")
    return "/pyspark/ml/" in path or path.startswith(_PKG_DIR.replace(os.sep, "/") + "/")


def install() -> None:
    """Idempotent."""
    for name, names in ACCELERATED.items():
        full = f"pyspark.ml.{name}"
        current = sys.modules.get(full)
        if isinstance(current, _PysparkMlProxy):
            continue
        original = current if current is not None else importlib.import_module(full)
        accelerated = importlib.import_module(f"{__package__}.{name}")
        proxy = _PysparkMlProxy(name, original, accelerated, names)
        sys.modules[full] = proxy
        parent = sys.modules.get("pyspark.ml")
        if parent is not None:
            setattr(parent, name, proxy)   # `import pyspark.ml.clustering as c` / `pyspark.ml.clustering.KMeans`


def uninstall() -> None:
    for name in ACCELERATED:
        full = f"pyspark.ml.{name}"
        current = sys.modules.get(full)
        if isinstance(current, _PysparkMlProxy):
            original = current.__dict__["_b2k_original"]
            sys.modules[full] = original
            parent = sys.modules.get("pyspark.ml")
            if parent is not None:
                setattr(parent, name, original)


install()
