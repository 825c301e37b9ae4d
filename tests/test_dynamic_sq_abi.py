"""The dynamic Vamana index over SQ codes at the C ABI, without a GPU: its two entry points exist in the header and
the library, and their argument checks refuse bad input before any device is touched."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import ROOT

NAMES = ("svsb200_dynamic_create_sq", "svsb200_dynamic_build_sq")
BAD_PARAMS = ((0.0, 0.0), (-1.0, 0.0), (float("nan"), 0.0), (float("inf"), 0.0), (0.1, float("inf")),
              (0.1, float("nan")))


def test_entry_points_are_declared_and_exported():
    from scalablevectorsearch_b200 import _lib
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "svsb200.h")).read(), flags=re.S)
    lib = _lib.lib()
    for name in NAMES:
        assert re.search(rf"\b{name}\s*\(", text), name
        assert name in _lib.ABI and hasattr(lib, name), name


def _create(codes, code_type, scale, bias, ids):
    from scalablevectorsearch_b200 import _lib
    n, dim = codes.shape
    graph = np.zeros((n, 9), dtype=np.uint32)
    out = C.c_void_p()
    _lib.check(_lib.lib().svsb200_dynamic_create_sq(codes.ctypes.data, code_type, n, dim, scale, bias, graph.ctypes.data,
                                                    9, 0, 0, ids.ctypes.data, 0, C.byref(out)))


def _build(codes, code_type, scale, bias, ids):
    from scalablevectorsearch_b200 import _lib
    n, dim = codes.shape
    out = C.c_void_p()
    _lib.check(_lib.lib().svsb200_dynamic_build_sq(codes.ctypes.data, code_type, n, dim, 0, scale, bias, 0.0, 8, 16, 0, 0,
                                                   ids.ctypes.data, 0, C.byref(out)))


@pytest.mark.parametrize("call,who", [(_create, "svsb200_dynamic_create_sq"), (_build, "svsb200_dynamic_build_sq")])
def test_refusals_before_any_device(call, who):
    """A bad code type, a scale or bias an SQ index cannot hold, and repeated or reserved ids, each named, on a machine
    with or without a device (these checks come first)."""
    from scalablevectorsearch_b200 import Svsb200Error
    codes = np.random.default_rng(0).integers(-100, 100, (64, 20)).astype(np.int8)
    ids = np.arange(64, dtype=np.uint64)
    for code_type in (0, 1, 4):   # float32, float16, not a type
        with pytest.raises(Svsb200Error, match=f"{who}: codes must be int8 or uint8"):
            call(codes, code_type, 0.1, 0.0, ids)
    for scale, bias in BAD_PARAMS:
        with pytest.raises(Svsb200Error, match=f"{who}: the SQ scale must be finite and positive"):
            call(codes, 2, scale, bias, ids)
    repeated = ids.copy()
    repeated[5] = repeated[6]
    with pytest.raises(Svsb200Error, match="repeat"):
        call(codes, 3, 0.1, 0.0, repeated)
    reserved = ids.copy()
    reserved[3] = np.uint64(2**64 - 1)
    with pytest.raises(Svsb200Error, match="reserved"):
        call(codes, 2, 0.1, 0.0, reserved)


def test_python_refuses_codes_of_the_wrong_type():
    from scalablevectorsearch_b200 import DynamicVamana, VamanaBuildParameters
    x = np.zeros((8, 4), dtype=np.float32)
    with pytest.raises(TypeError, match="SQ codes"):
        DynamicVamana.from_arrays(x, np.zeros((8, 3), dtype=np.uint32), 0, sq=(0.1, 0.0))
    with pytest.raises(TypeError, match="SQ codes"):
        DynamicVamana.build(VamanaBuildParameters(graph_max_degree=2, window_size=4), x, sq=(0.1, 0.0))
