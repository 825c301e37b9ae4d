"""Stored-row access at the C ABI, without a GPU: svsb200_index_distances and svsb200_index_reconstruct exist in the
header, the library and the binding's table, and their argument refusals come before any device is touched."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import ROOT

NAMES = ("svsb200_index_distances", "svsb200_index_reconstruct")


def test_entry_points_are_declared_and_exported():
    from scalablevectorsearch_b200 import _lib
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "svsb200.h")).read(), flags=re.S)
    lib = _lib.lib()
    for name in NAMES:
        assert re.search(rf"\b{name}\s*\(", text), name
        assert name in _lib.ABI and hasattr(lib, name), name


def test_null_arguments_are_refused_before_any_device():
    from scalablevectorsearch_b200 import Svsb200Error, _lib
    lib = _lib.lib()
    q = np.zeros(8, dtype=np.float32)
    ids = np.zeros(1, dtype=np.uint64)
    out = np.full(8, 7.0, dtype=np.float32)
    with pytest.raises(Svsb200Error, match="svsb200_index_distances: NULL index"):
        _lib.check(lib.svsb200_index_distances(None, q.ctypes.data, 0, 1, ids.ctypes.data, out.ctypes.data))
    with pytest.raises(Svsb200Error, match="svsb200_index_reconstruct: NULL index"):
        _lib.check(lib.svsb200_index_reconstruct(None, ids.ctypes.data, 1, out.ctypes.data))
    assert (out == 7.0).all()


def test_unknown_query_dtype_is_refused_first():
    from scalablevectorsearch_b200 import Svsb200Error, _lib
    lib = _lib.lib()
    q = np.zeros(8, dtype=np.float32)
    ids = np.zeros(1, dtype=np.uint64)
    out = np.full(1, 7.0, dtype=np.float32)
    for qdtype in (-1, 4, 99):
        with pytest.raises(Svsb200Error, match="svsb200_index_distances: bad query dtype"):
            _lib.check(lib.svsb200_index_distances(None, q.ctypes.data, qdtype, 1, ids.ctypes.data, out.ctypes.data))
    assert out[0] == 7.0


def test_runtime_demo_is_built_with_the_runtime_library():
    """dynamic_vamana_demo is part of cpp/Makefile's `all`, next to the other runtime demos."""
    text = open(os.path.join(ROOT, "scalablevectorsearch_b200", "cpp", "Makefile")).read()
    all_line = text[text.index("all:"):text.index("\n$(OUT)/search_index_gpu")]
    assert "$(OUT)/dynamic_vamana_demo" in all_line
