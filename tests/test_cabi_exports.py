"""CPU-side checks of the drop-in boundary: the C-ABI library loads without a GPU, exports every symbol
include/b2kmeans.h declares, and fails loudly (no fallback) when there is no CUDA device."""
import ctypes
import os
import re

import pytest

from spark_rapids_ml_b200 import _native

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_symbols():
    src = open(os.path.join(ROOT, "include", "b2kmeans.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b2k_[a-z0-9_]+)\s*\(", src)))


def test_header_and_binding_agree():
    assert _header_symbols() == sorted(_native.EXPORTED_SYMBOLS)


def test_library_loads_and_exports_every_symbol():
    assert os.path.exists(_native.LIB_PATH), "run __graft_entry__.build() first"
    L = _native.load_library()
    for name in _header_symbols():
        assert hasattr(L, name), name
    assert L.b2k_version() == 100


def test_no_cpu_fallback_without_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    L = _native.load_library()
    h = ctypes.c_void_p()
    rc = L.b2k_ctx_create(0, ctypes.byref(h))
    assert rc != 0
    assert b"no CPU fallback" in L.b2k_last_error(None)
    with pytest.raises(_native.B2KError):
        _native.Context(0)


def test_product_never_imports_oracle():
    """The oracle is test infrastructure: nothing under spark_rapids_ml_b200/ may reference it."""
    pkg = os.path.join(ROOT, "spark_rapids_ml_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in txt and "from oracle" not in txt, f
                assert "kmeans_oracle" not in txt, f


# The header is kept by hand in three places: the prototypes, the argtypes load_library() sets and the Structures that
# mirror its structs.  ctypes converts each argument by its argtypes entry, so a disagreement passes a value of the
# wrong width or a pointer to the wrong layout without any error.
_INTS = {"int": (4, True), "int32_t": (4, True), "int64_t": (8, True), "uint64_t": (8, False), "size_t": (8, False),
         "uintptr_t": (8, False)}
_POINTEE_SIZES = {"char": 1, "int8_t": 1, "uint8_t": 1, "int": 4, "int32_t": 4, "float": 4, "int64_t": 8,
                  "long long": 8, "double": 8}
_STRUCTS = {"b2k_stats": _native.Stats, "b2k_logreg_params": _native.LogregParams, "b2k_rf_params": _native.RfParams,
            "b2k_umap_params": _native.UmapParams}
_FIELD_TYPES = {"int32_t": ctypes.c_int32, "int64_t": ctypes.c_int64, "uint64_t": ctypes.c_uint64,
                "double": ctypes.c_double}


def _header():
    src = open(os.path.join(ROOT, "include", "b2kmeans.h")).read()
    return re.sub(r"/\*.*?\*/", "", src, flags=re.S)


def _params(arglist):
    """(base type, pointer depth) of each parameter of a C parameter list; an array parameter is a pointer."""
    out = []
    for p in arglist.split(","):
        p = " ".join(p.split())
        if p in ("", "void"):
            continue
        m = re.fullmatch(r"(.*?)\s*\b\w+\s*(\[[^\]]*\])?", p)
        typ = m.group(1).replace("const", " ")
        out.append((" ".join(typ.replace("*", " ").split()), typ.count("*") + (m.group(2) is not None)))
    return out


def _agrees(ctype, base, depth):
    """Whether the ctypes type converts a C parameter of base type `base` behind `depth` pointers without change."""
    if depth == 0:
        if base in _INTS:
            size, signed = _INTS[base]
            return (issubclass(ctype, ctypes._SimpleCData) and ctype._type_ in "bBhHiIlLqQ"
                    and ctypes.sizeof(ctype) == size and (ctype(-1).value < 0) == signed)
        if base == "double":
            return ctype is ctypes.c_double
        return base == "b2k_logreg_objective" and ctype is _native.LOGREG_OBJECTIVE
    if ctype is ctypes.c_void_p or (ctype is ctypes.c_char_p and base == "char" and depth == 1):
        return True
    if not issubclass(ctype, ctypes._Pointer):
        return False
    if depth > 1:
        return ctypes.sizeof(ctype._type_) == ctypes.sizeof(ctypes.c_void_p)
    if base in _STRUCTS:
        return ctype._type_ is _STRUCTS[base]
    return base in _POINTEE_SIZES and ctypes.sizeof(ctype._type_) == _POINTEE_SIZES[base]


def test_argtypes_agree_with_the_header_prototypes():
    L = _native.load_library()
    protos = re.findall(r"^(int|const char\s*\*)\s*(b2k_\w+)\s*\(([^)]*)\)\s*;", _header(), flags=re.M)
    assert sorted(name for _, name, _ in protos) == sorted(_native.EXPORTED_SYMBOLS)
    for ret, name, arglist in protos:
        fn = getattr(L, name)
        assert fn.restype is (ctypes.c_int if ret == "int" else ctypes.c_char_p), name
        params = _params(arglist)
        argtypes = fn.argtypes or ()
        assert len(argtypes) == len(params), name
        for i, (ctype, (base, depth)) in enumerate(zip(argtypes, params)):
            assert _agrees(ctype, base, depth), f"{name} parameter {i}: {base}{'*' * depth} bound as {ctype}"


def test_logreg_objective_agrees_with_its_typedef():
    m = re.search(r"typedef\s+int\s*\(\s*\*\s*b2k_logreg_objective\s*\)\s*\(([^)]*)\)\s*;", _header())
    params = _params(m.group(1))
    assert _native.LOGREG_OBJECTIVE._restype_ is ctypes.c_int
    assert len(_native.LOGREG_OBJECTIVE._argtypes_) == len(params)
    for ctype, (base, depth) in zip(_native.LOGREG_OBJECTIVE._argtypes_, params):
        assert _agrees(ctype, base, depth), (base, depth, ctype)


def test_structures_agree_with_the_header_structs():
    structs = dict(re.findall(r"typedef\s+struct\s+(\w+)\s*\{(.*?)\}\s*\1\s*;", _header(), flags=re.S))
    assert sorted(structs) == sorted(_STRUCTS)
    for name, body in structs.items():
        fields = []
        for decl in filter(None, (" ".join(s.split()) for s in body.split(";"))):
            typ, names = decl.split(" ", 1)
            fields += [(f.strip(), _FIELD_TYPES[typ]) for f in names.split(",")]
        got = [(f, t) for f, t in _STRUCTS[name]._fields_]
        assert [f for f, _ in got] == [f for f, _ in fields], name
        for (f, want), (_, have) in zip(fields, got):
            assert have is want, f"{name}.{f}: {have} for {want}"
