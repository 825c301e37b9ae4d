"""Work split of the flat search for a given k (svsb200_flat_plan_k, csrc/flat.cu): the same as svsb200_flat_plan for
k <= 25, and for the deep lists of a flat index (26 <= k <= 121, more than 256 queries) one list of 129 entries per
query and piece, within what the rescoring kernel holds; deep-k batches of at most 256 queries report the scan
(no lists, no CTAs).  No GPU needed."""
import ctypes as C

import numpy as np
import pytest

CMAX, BM, BN, DEEP = 1024, 128, 256, 129

SHAPES = [
    (10_000, 1_000_000, 148), (100, 1_000_000, 148), (700, 1_000_000, 148), (1, 300, 148), (129, 257, 148),
    (1100, 40_000, 148), (600, 30_000, 148), (100_000, 12_500_000, 148), (5000, 999, 148), (10_000, 1_000_000, 132),
    (513, 100_000, 7), (4096, 65_536, 1), (256, 1_000_000, 132), (257, 1_000_000, 132),
]


def plan(nq, n, sms):
    from scalablevectorsearch_b200 import _lib
    lib = _lib.lib()
    ctas, share, lists = C.c_uint32(), C.c_uint32(), C.c_uint32()
    _lib.check(lib.svsb200_flat_plan(nq, n, sms, C.byref(ctas), C.byref(share), C.byref(lists), None))
    seg = np.zeros(ctas.value // share.value + 1, dtype=np.uint64)
    _lib.check(lib.svsb200_flat_plan(nq, n, sms, C.byref(ctas), C.byref(share), C.byref(lists), seg.ctypes.data))
    return ctas.value, share.value, lists.value, seg


def plan_k(nq, n, k, sms):
    from scalablevectorsearch_b200 import _lib
    lib = _lib.lib()
    ctas, share, lists, entries = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint32()
    out = (C.byref(ctas), C.byref(share), C.byref(lists), C.byref(entries))
    _lib.check(lib.svsb200_flat_plan_k(nq, n, k, sms, *out, None))
    if entries.value == 0:
        return ctas.value, share.value, lists.value, entries.value, None
    seg = np.zeros(ctas.value // share.value + 1, dtype=np.uint64)
    _lib.check(lib.svsb200_flat_plan_k(nq, n, k, sms, *out, seg.ctypes.data))
    return ctas.value, share.value, lists.value, entries.value, seg


def pieces(seg, ngroups, ntiles):
    first = np.searchsorted(seg, np.arange(ngroups, dtype=np.uint64) * ntiles, side="right") - 1
    last = np.searchsorted(seg, (np.arange(ngroups, dtype=np.uint64) + 1) * ntiles - 1, side="right") - 1
    return int((last - first + 1).max())


@pytest.mark.parametrize("nq,n,sms", SHAPES)
@pytest.mark.parametrize("k", [1, 10, 25])
def test_shallow_k_is_the_existing_plan(nq, n, sms, k):
    ctas, share, lists, entries, seg = plan_k(nq, n, k, sms)
    c0, s0, l0, seg0 = plan(nq, n, sms)
    assert (ctas, share, lists, entries) == (c0, s0, l0, 33)
    assert np.array_equal(seg, seg0)


@pytest.mark.parametrize("nq,n,sms", SHAPES)
@pytest.mark.parametrize("k", [26, 100, 121])
def test_deep_lists_partition_the_tiles_and_fit(nq, n, sms, k):
    ctas, share, lists, entries, seg = plan_k(nq, n, k, sms)
    if nq <= 256:   # batches of one or two query tiles run the scan at deep k
        assert (ctas, share, lists, entries) == (0, 0, 0, 0)
        return
    assert entries == DEEP
    mtiles, ntiles = -(-nq // BM), -(-n // BN)
    assert share == (4 if mtiles >= 8 else 2 if mtiles >= 4 else 1) and ctas % share == 0
    assert 1 <= ctas <= max(sms, share)
    nseg, ngroups = ctas // share, -(-mtiles // share)
    total = ngroups * ntiles
    assert seg[0] == 0 and seg[-1] == total and len(seg) == nseg + 1
    runs = np.diff(seg.astype(np.int64))
    assert runs.min() >= 1 and runs.max() - runs.min() <= 1
    # one list per query and piece, all of them within the rescoring kernel's candidates
    assert pieces(seg, ngroups, ntiles) == lists and lists * DEEP <= CMAX
    # the largest admissible number of segments: one more would cut a query tile into too many pieces
    if nseg < max(1, sms // share) and nseg < total:
        more = np.array([total * b // (nseg + 1) for b in range(nseg + 2)], dtype=np.uint64)
        assert pieces(more, ngroups, ntiles) * DEEP > CMAX


def test_plan_k_rejects_bad_arguments():
    from scalablevectorsearch_b200 import _lib
    lib = _lib.lib()
    a = C.c_uint32()
    out = (C.byref(a), C.byref(a), C.byref(a), C.byref(a))
    assert lib.svsb200_flat_plan_k(10, 1000, 0, 148, *out, None) != 0
    assert lib.svsb200_flat_plan_k(10, 1000, 122, 148, *out, None) != 0
    assert b"flat_plan_k" in lib.svsb200_last_error()
    assert lib.svsb200_flat_plan_k(0, 1000, 10, 148, *out, None) != 0
    assert lib.svsb200_flat_plan_k(10, 1000, 10, 0, *out, None) != 0
    assert lib.svsb200_flat_plan_k(10, 1000, 121, 148, *out, None) == 0
