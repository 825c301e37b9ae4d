"""The C-ABI library loads and exports every symbol include/svsb200.h declares (no GPU needed)."""
import ctypes
import os
import re

import pytest

from conftest import ROOT


def header_symbols():
    text = open(os.path.join(ROOT, "include", "svsb200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(svsb200_[a-z0-9_]+)\s*\(", text)))


def header_prototypes():
    """{symbol: (return type, [parameter declarations])} of include/svsb200.h; ``(void)`` has no parameters."""
    text = open(os.path.join(ROOT, "include", "svsb200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    protos = {}
    for m in re.finditer(r"(\w+\**)\s*\**\s*\b(svsb200_[a-z0-9_]+)\s*\(", text):
        params, depth, i = [""], 1, m.end()
        while depth:   # split at the top-level commas: a parameter may be a function pointer
            ch = text[i]
            depth += {"(": 1, ")": -1}.get(ch, 0)
            if ch == "," and depth == 1:
                params.append("")
            elif depth:
                params[-1] += ch
            i += 1
        params = [" ".join(p.split()) for p in params]
        ret = text[m.start():m.end()].split(m.group(2))[0].strip()
        protos[m.group(2)] = (ret, [] if params == ["void"] else params)
    return protos


def test_header_declares_the_expected_surface():
    syms = header_symbols()
    for name in ("svsb200_index_create", "svsb200_search", "svsb200_search_device", "svsb200_merge_topk_device",
                 "svsb200_get_counters", "svsb200_last_error", "svsb200_ivf_plan", "svsb200_ivf_group_plan"):
        assert name in syms


def test_library_exports_every_declared_symbol():
    from scalablevectorsearch_b200 import _lib
    lib = _lib.lib()
    missing = [s for s in header_symbols() if not hasattr(lib, s)]
    assert not missing, f"libsvsb200.so lacks {missing}"
    assert sorted(_lib.SYMBOLS) == header_symbols(), "python binding list out of sync with the header"
    assert lib.svsb200_version() == 201


def test_abi_table_matches_the_header_prototypes():
    """Every entry of the binding's ABI table has one argtype per parameter of its prototype, a pointer type exactly
    where the parameter is a pointer, and the prototype's return type (no library needed)."""
    from scalablevectorsearch_b200 import _lib
    returns = {"int": ctypes.c_int, "size_t": ctypes.c_size_t, "uint64_t": ctypes.c_uint64, "char*": ctypes.c_char_p,
               "void": None}
    protos = header_prototypes()
    assert sorted(_lib.ABI) == sorted(protos)
    for name, (restype, argtypes) in _lib.ABI.items():
        ret, params = protos[name]
        assert len(argtypes) == len(params), f"{name}: {len(argtypes)} argtypes for {len(params)} parameters"
        assert restype is returns[ret], name
        for i, (t, p) in enumerate(zip(argtypes, params)):
            pointer = t in (ctypes.c_void_p, ctypes.c_char_p) or issubclass(t, (ctypes._Pointer, ctypes._CFuncPtr))
            assert pointer == ("*" in p), f"{name} parameter {i} ({p}) is bound as {t.__name__}"


def test_no_cpu_fallback_without_a_device():
    """Without a CUDA device index creation must fail loudly (never silently compute on the CPU)."""
    import numpy as np
    from scalablevectorsearch_b200 import DistanceType, Svsb200Error, Vamana, _lib
    if _lib.lib().svsb200_device_count() > 0:
        pytest.skip("a CUDA device is present")
    data = np.zeros((4, 8), dtype=np.float32)
    graph = np.zeros((4, 3), dtype=np.uint32)
    with pytest.raises(Svsb200Error, match="no CUDA device"):
        Vamana.from_arrays(data, graph, 0, DistanceType.L2)


def test_product_never_touches_the_oracle():
    """The product path must not import, link or load anything under oracle/."""
    pkg = os.path.join(ROOT, "scalablevectorsearch_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                text = open(os.path.join(dirpath, f), errors="replace").read()
                assert "oracle" not in text.lower() or f in ("synthetic.py",) and False, \
                    f"{os.path.join(dirpath, f)} mentions the oracle"
    out = os.popen(f"ldd {os.path.join(pkg, 'libsvsb200.so')}").read()
    assert "oracle" not in out and "svsref" not in out


def test_oracle_library_exports_every_declared_symbol():
    """The checker's own header and shared object must agree (a declared-but-undefined function only shows up when a
    GPU test first calls it)."""
    from oracle.bindings import OracleLib
    OracleLib()   # builds oracle/liboracle.so on demand
    header = open(os.path.join(ROOT, "oracle", "vamana_oracle.h")).read()
    names = set(re.findall(r"\b(oracle_[a-z0-9_]+)\s*\(", header))
    assert len(names) > 10
    lib = ctypes.CDLL(os.path.join(ROOT, "oracle", "liboracle.so"))
    missing = [n for n in sorted(names) if not hasattr(lib, n)]
    assert not missing, missing
