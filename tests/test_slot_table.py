"""The slot rules of the dynamic indexes (scalablevectorsearch_b200/csrc/slots.h), without a GPU: the header is compiled
with the host C++ compiler behind tests/slot_table_shim.cpp and held to the pure-Python models the GPU tests use --
tests/dynamic_flat_model.py's SlotModel for the dynamic flat (and Vamana) rule, tests/dynamic_ivf_model.py's slots for
the dynamic IVF rule -- after every step of their mutation scripts, to the Vamana index's soft delete by hand, and to
the refusals' messages, which leave the table as it was."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from dynamic_flat_model import EMPTY, RESERVED, VALID, SlotModel, mutation_script
from dynamic_ivf_model import DynamicIVFModel

DELETED = 2
HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "scalablevectorsearch_b200", "csrc")


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    cxx = next((c for c in (os.environ.get("CXX"), "c++", "g++", "clang++") if c and shutil.which(c)), None)
    if cxx is None:
        pytest.skip("no C++ compiler on the PATH")
    so = str(tmp_path_factory.mktemp("slots") / "libslot_table.so")
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-Wall", "-shared", "-fPIC", "-I", CSRC,
                           os.path.join(HERE, "slot_table_shim.cpp"), "-o", so])
    l = C.CDLL(so)
    vp, sz, i32 = C.c_void_p, C.c_size_t, C.c_int
    l.st_last_error.restype = C.c_char_p
    l.st_new.restype = vp
    l.st_free.argtypes = [vp]
    l.st_assign.argtypes = [vp, vp, sz]
    l.st_add.argtypes = [vp, vp, sz, i32, i32, vp]
    l.st_delete.argtypes = [vp, vp, sz, C.c_uint8]
    l.st_compact.argtypes = [vp]
    for name in ("st_num_slots", "st_size", "st_first_empty"):
        getattr(l, name).restype, getattr(l, name).argtypes = sz, [vp]
    l.st_export.argtypes = [vp, vp, vp]
    l.st_ids.argtypes = [vp, vp, C.POINTER(sz)]
    l.st_has_id.argtypes = [vp, C.c_uint64, C.POINTER(i32)]
    return l


class Refused(Exception):
    pass


class Table:
    """One SlotTable; `ivf` selects the dynamic IVF index's add rule."""

    def __init__(self, lib, ids, ivf=False):
        self.lib, self.ivf = lib, ivf
        self.t = lib.st_new()
        self._check(lib.st_assign(self.t, self._ids(ids).ctypes.data, len(ids)))

    def __del__(self):
        self.lib.st_free(self.t)

    @staticmethod
    def _ids(ids):
        return np.ascontiguousarray(np.atleast_1d(np.asarray(ids, dtype=np.uint64)))

    def _check(self, rc):
        if rc:
            raise Refused(self.lib.st_last_error().decode())

    def add(self, ids, reuse_empty=False):
        ids = self._ids(ids)
        slots = np.zeros(len(ids), dtype=np.uint64)
        self._check(self.lib.st_add(self.t, ids.ctypes.data, len(ids), int(reuse_empty), int(self.ivf), slots.ctypes.data))
        return slots.tolist()

    def delete(self, ids, to=EMPTY):
        ids = self._ids(ids)
        self._check(self.lib.st_delete(self.t, ids.ctypes.data, len(ids), to))

    def compact(self):
        self.lib.st_compact(self.t)

    @property
    def first_empty(self):
        return self.lib.st_first_empty(self.t)

    @property
    def size(self):
        return self.lib.st_size(self.t)

    def export(self):
        n = self.lib.st_num_slots(self.t)
        status, ext = np.empty(n, dtype=np.uint8), np.empty(n, dtype=np.uint64)
        self.lib.st_export(self.t, status.ctypes.data, ext.ctypes.data)
        return status, ext

    def all_ids(self):
        n = C.c_size_t(self.size)
        out = np.empty(n.value, dtype=np.uint64)
        self._check(self.lib.st_ids(self.t, out.ctypes.data, C.byref(n)))
        return out[: n.value]

    def has_id(self, id):
        out = C.c_int()
        self._check(self.lib.st_has_id(self.t, id, C.byref(out)))
        return bool(out.value)

    def state(self):
        status, ext = self.export()
        return status.tolist(), ext.tolist(), self.first_empty, self.size


@pytest.mark.parametrize("n0,seed", [(0, 1), (40, 2), (300, 3)])
def test_flat_rule_follows_the_slot_model(lib, n0, seed):
    ids = 3 * np.arange(n0, dtype=np.uint64) + 1
    table, model = Table(lib, ids), SlotModel(ids)

    def agree(step):
        status, ext = table.export()
        want_status, want_ext = model.export()
        assert np.array_equal(status, want_status) and np.array_equal(ext, want_ext), step
        assert table.first_empty == model.first_empty, step
        assert np.array_equal(table.all_ids(), model.live_ids()), step

    agree("create")
    for step in mutation_script(model, n0, seed):
        if step[0] == "delete":
            table.delete(step[1])
            model.delete(step[1])
        elif step[0] == "add":
            _, _, new, reuse = step
            assert table.add(new, reuse) == model.add(new, reuse_empty=reuse), step[:1]
        else:
            table.compact()
            model.compact()
        agree(step[0])


def test_ivf_rule_follows_the_dynamic_ivf_model(lib):
    rng = np.random.default_rng(7)
    n0 = 50
    ids = rng.choice(10**6, size=n0, replace=False).astype(np.uint64)
    model = DynamicIVFModel.assemble(None, 0, np.zeros((1, 2), np.float32), np.zeros((n0, 2), np.float32), ids,
                                     assignments=np.zeros(n0, dtype=np.int64))
    model.nearest_cluster = lambda rows: np.zeros(len(rows), dtype=np.int64)   # (the clusters do not bear on slots)
    table = Table(lib, ids, ivf=True)
    fresh = iter(range(2 * 10**6, 3 * 10**6, 7))

    def add(count, reuse):
        new = np.array([next(fresh) for _ in range(count)], dtype=np.uint64)
        got = table.add(new, reuse)
        assert got == model.add(np.zeros((count, 2), np.float32), new, reuse_empty=reuse)
        return got

    def agree():
        status, ext = table.export()
        want_status, want_ext, _ = model.export()
        assert np.array_equal(status, want_status) and np.array_equal(ext, want_ext)
        assert np.array_equal(table.all_ids(), model.all_ids())

    for _ in range(3):
        live = model.all_ids()
        gone = rng.choice(live, size=len(live) // 5, replace=False)
        table.delete(gone)
        model.delete(gone)
        agree()
        assert add(4, False)[0] == len(model.valid) - 4   # appended although Empty slots exist
        agree()
        add(len(gone) + 3, True)                          # the Empty slots from slot 0, then appended
        agree()
        table.delete(model.all_ids()[::3])
        model.delete(model.all_ids()[::3])
        table.compact()
        model.compact()
        agree()


def test_soft_delete_keeps_ids_and_first_empty(lib):
    t = Table(lib, [10, 11, 12, 13, 14, 15])
    t.delete([13, 11], to=DELETED)
    status, ext = t.export()
    assert status.tolist() == [VALID, DELETED, VALID, DELETED, VALID, VALID]
    assert ext.tolist() == [10, 11, 12, 13, 14, 15] and t.first_empty == 6 and t.size == 4
    assert not t.has_id(11) and t.has_id(12) and t.all_ids().tolist() == [10, 12, 14, 15]
    assert t.add([20]) == [6] and t.add([21], reuse_empty=True) == [7]   # Deleted slots are never reused
    t.delete([10])                                                      # Empty: reused from slot 0
    assert t.first_empty == 0 and t.add([22], reuse_empty=True) == [0]
    with pytest.raises(Refused, match="External ID 13 does not exist!"):
        t.delete([13], to=DELETED)


def test_refusals_leave_the_table_unchanged(lib):
    for ids, msg in (([1, RESERVED], "t: external id 2^64 - 1 is reserved"),
                     ([1, 2, 1], "t: External IDs contain repeat elements!")):
        with pytest.raises(Refused) as e:
            Table(lib, ids)
        assert str(e.value) == msg
    t = Table(lib, [1, 2, 3, 4])
    t.delete([2])
    before = t.state()
    cases = [
        (lambda: t.add([7, RESERVED]), "t: external id 2^64 - 1 is reserved"),
        (lambda: t.add([7, 8, 7]), "t: External IDs contain repeat elements!"),
        (lambda: t.add([7, 3]), "t: External ID 3 already exists!"),
        (lambda: t.delete([1, 9]), "t: External ID 9 does not exist!"),
        (lambda: t.delete([1, 1]), "t: External ID 1 does not exist!"),
        (lambda: t.delete([2]), "t: External ID 2 does not exist!"),
    ]
    for call, msg in cases:
        with pytest.raises(Refused) as e:
            call()
        assert str(e.value) == msg
        assert t.state() == before
    n = C.c_size_t(2)
    out = np.empty(2, dtype=np.uint64)
    assert lib.st_ids(t.t, out.ctypes.data, C.byref(n)) == 1
    assert lib.st_last_error().decode() == "t: output too small"
    assert t.state() == before
