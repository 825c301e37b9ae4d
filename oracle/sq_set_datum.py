"""ctypes wrapper of ``_ref/libsvsref_sq_set_datum.so`` (ref/sq_set_datum_capi.cpp): the reference's own
``SQDataset<int8_t / uint8_t>::set_datum`` behind a test-only façade.  TEST INFRASTRUCTURE ONLY (see README.md)."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libsvsref_sq_set_datum.so")
CODE_TYPES = {np.dtype(np.int8): 2, np.dtype(np.uint8): 3}


class RefSQSetDatum:
    """float32 rows stored into an SQDataset with a given scale and bias, as the reference encodes an add."""

    def __init__(self, path: str = PATH):
        self.lib = C.CDLL(path)
        self.lib.svsref_sq_set_datum_last_error.restype = C.c_char_p
        sz, vp = C.c_size_t, C.c_void_p
        self.lib.svsref_sq_set_datum.argtypes = [vp, sz, sz, C.c_int, C.c_float, C.c_float, vp]

    @staticmethod
    def available() -> bool:
        return os.path.exists(PATH)

    def set_datum(self, data, code_dtype, scale: float, bias: float) -> np.ndarray:
        """-> the codes [n, dim] of ``code_dtype``."""
        x = np.ascontiguousarray(data, dtype=np.float32)
        codes = np.empty(x.shape, dtype=code_dtype)
        rc = self.lib.svsref_sq_set_datum(x.ctypes.data, x.shape[0], x.shape[1], CODE_TYPES[np.dtype(code_dtype)],
                                          float(scale), float(bias), codes.ctypes.data)
        if rc:
            raise RuntimeError(self.lib.svsref_sq_set_datum_last_error().decode())
        return codes
