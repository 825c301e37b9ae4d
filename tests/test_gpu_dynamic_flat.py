"""The dynamic flat index (svsb200_dynamic_flat_*, Python DynamicFlat) on the GPU.

After every step of the mutation script of tests/dynamic_flat_model.py its search must equal a static Flat over the live
rows in slot order, ids mapped through the exported external ids: ids and distance bits.  Both Flat handles are exact,
so this holds on every route (tensor-core GEMM, fallback, scan) whichever route each of them takes.  Also: no fallback
where the error bound proves every query, no deleted id on any route, the fp16 bound's Xmax taken over the Valid rows
only, edge cases, errors that change nothing, and agreement with the reference's own DynamicFlatIndex."""
import itertools

import numpy as np
import pytest

from conftest import GOLDEN, bits
from dynamic_flat_model import RESERVED, SlotModel, mutation_script, pool_size, run_script

pytestmark = pytest.mark.gpu

METRICS = {"l2": 0, "ip": 1, "cosine": 2}
KS = (1, 10, 25, 100, 121, 200)
QTYPES = {np.float32: (np.float32, np.float16), np.float16: (np.float32, np.float16), np.int8: (np.int8, np.float32),
          np.uint8: (np.uint8, np.float32)}


def _data(dtype, n, nq, dim=96):
    """Clustered unit vectors (float rows), or their integer codes (int8 / uint8 rows), and queries."""
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    base, queries = clustered_unit_vectors(n, nq, dim)
    if dtype == np.uint8:
        lo, hi = float(min(base.min(), queries.min())), float(max(base.max(), queries.max()))
        f = lambda v: np.rint((v - lo) * (255.0 / (hi - lo))).astype(np.uint8)   # noqa: E731
        return f(base), f(queries)
    if dtype == np.int8:
        m = float(max(abs(base).max(), abs(queries).max()))
        f = lambda v: np.rint(v * (127.0 / m)).astype(np.int8)   # noqa: E731
        return f(base), f(queries)
    return base.astype(dtype), queries


def _queries(q, qtype):
    return q if q.dtype == qtype else q.astype(qtype)


def _dyn(x, ids, metric):
    from scalablevectorsearch_b200 import DistanceType, DynamicFlat
    return DynamicFlat.build(x, ids, DistanceType(METRICS[metric]))


def _live_flat(pool, model, metric):
    """search(q, k) of a static Flat over the live rows in slot order, its row numbers mapped to the live slots'
    external ids."""
    from scalablevectorsearch_b200 import DistanceType, Flat
    live, ext = model.live_payload(), model.live_ids()
    flat = Flat(pool[live], DistanceType(METRICS[metric])) if len(live) else None

    def search(q, k):
        if flat is None:
            pad = -np.inf if metric != "l2" else np.inf
            return np.full((q.shape[0], k), RESERVED, dtype=np.uint64), np.full((q.shape[0], k), pad, dtype=np.float32)
        ids, d = flat.search(q, k)
        out = np.full(ids.shape, RESERVED, dtype=np.uint64)
        ok = ids != np.uint64(RESERVED)
        out[ok] = ext[ids[ok].astype(np.int64)]
        return out, d
    return search


def _expected(pool, model, metric, q, k):
    return _live_flat(pool, model, metric)(q, k)


def _assert_equal(index, pool, model, metric, q, k, what, live_flat=None):
    got_i, got_d = index.search(q, k)
    want_i, want_d = (live_flat or _live_flat(pool, model, metric))(q, k)
    assert np.array_equal(got_i, want_i), (what, k, q.shape, q.dtype)
    assert np.array_equal(bits(got_d), bits(want_d)), (what, k, q.shape, q.dtype)


def _device_call(index, q, k, stream=None):
    import torch
    dq = torch.from_numpy(np.ascontiguousarray(q)).cuda()
    ids = torch.empty((q.shape[0], k), dtype=torch.int64, device="cuda")
    d = torch.empty((q.shape[0], k), dtype=torch.float32, device="cuda")
    s = stream or torch.cuda.current_stream()
    with torch.cuda.stream(s):
        fb = index.search_device(dq.data_ptr(), q.dtype, q.shape[0], k, ids.data_ptr(), d.data_ptr(),
                                 stream=s.cuda_stream or 1)
    torch.cuda.synchronize()
    return ids.cpu().numpy().view(np.uint64), d.cpu().numpy(), fb


def _apply(index, model, pool, step):
    if step[0] == "delete":
        index.delete(step[1])
        model.delete(step[1])
    elif step[0] == "add":
        _, rows, ids, reuse = step
        got = index.add(pool[rows], ids, reuse_empty=reuse)
        assert got.tolist() == model.add(ids, reuse_empty=reuse, payload=rows), step[:1]
    else:
        index.compact()
        model.compact()
    status, ext = index.export()
    want_status, want_ext = model.export()
    assert np.array_equal(status, want_status) and np.array_equal(ext, want_ext), step[:1]
    assert index.size == len(model.live_slots()) and index.num_slots == len(model.status)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("searched_first", [True, False], ids=["tiles-built", "tiles-unbuilt"])
@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
@pytest.mark.parametrize("dtype", [np.float32, np.float16, np.int8, np.uint8], ids=["f32", "f16", "i8", "u8"])
def test_equals_static_flat_over_live_rows_through_the_script(dtype, metric, searched_first):
    """nq 200 and 300: both sides of the 256-query deep-k rule; k up to 200 (the scan)."""
    n0 = 2000
    pool, queries = _data(dtype, pool_size(n0), 300)
    ids = 3 * np.arange(n0, dtype=np.uint64) + 1
    index, model = _dyn(pool[:n0], ids, metric), SlotModel(ids, payload=range(n0))

    def check(what):
        live_flat = _live_flat(pool, model, metric)
        for qt in QTYPES[dtype]:
            q = _queries(queries, qt)
            for k in KS:
                for nq in (200, 300):
                    _assert_equal(index, pool, model, metric, q[:nq], k, what, live_flat)

    if searched_first:
        check("build")
    for i, step in enumerate(mutation_script(model, n0, seed=7)):
        _apply(index, model, pool, step)
        # tiles-unbuilt: the first search comes after the deletions and the first adds
        if searched_first or i >= 2:
            check(step[0])


@pytest.mark.timeout(600)
@pytest.mark.parametrize("metric", ["l2", "ip"])
@pytest.mark.parametrize("dtype", [np.float32, np.float16, np.int8, np.uint8], ids=["f32", "f16", "i8", "u8"])
def test_no_fallback_where_the_bound_proves_every_query(dtype, metric):
    """Clustered unit vectors on the fp16 path, integer rows (far below 2^24) on the integer path: zero fallbacks
    after every step."""
    n0 = 4000
    pool, queries = _data(dtype, pool_size(n0), 300)
    ids = 3 * np.arange(n0, dtype=np.uint64) + 1
    index, model = _dyn(pool[:n0], ids, metric), SlotModel(ids, payload=range(n0))
    qtypes = (np.float32,) if dtype in (np.float32, np.float16) else (dtype,)
    # (lazily: each step is drawn from the model's state after the previous one)
    for step in itertools.chain([("build",)], mutation_script(model, n0, seed=3)):
        if step[0] != "build":
            _apply(index, model, pool, step)
        for qt in qtypes:
            q = _queries(queries, qt)
            for k in (10, 100):
                gi, gd, fb = _device_call(index, q, k)
                assert fb == 0, (step[0], k, fb)
                wi, wd = _expected(pool, model, metric, q, k)
                assert np.array_equal(gi, wi) and np.array_equal(bits(gd), bits(wd)), (step[0], k)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("route", ["gemm", "fallback", "scan"])
def test_deleted_ids_never_come_back(route):
    """Delete each query's exact top k, search again: no deleted id on the GEMM route (no fallback), on the fallback
    route (a live row with an element >= 65520 makes every fp16 bound infinite) or on the scan (k = 200)."""
    n0, nq = 6000, 20
    pool, queries = _data(np.float32, n0 + 1, nq)
    if route == "fallback":
        pool[n0, 0] = 70000.0
    rows = n0 + 1 if route == "fallback" else n0
    ids = 3 * np.arange(rows, dtype=np.uint64) + 1
    index, model = _dyn(pool[:rows], ids, "l2"), SlotModel(ids, payload=range(rows))
    k = 200 if route == "scan" else 10
    first, _, _ = _device_call(index, queries, k)
    gone = np.unique(first.ravel())
    index.delete(gone)
    model.delete(gone)
    got, gd, fb = _device_call(index, queries, k)
    assert not np.isin(got, gone).any()
    assert fb == (0 if route == "gemm" else nq)
    want, wd = _expected(pool, model, "l2", queries, k)
    assert np.array_equal(got, want) and np.array_equal(bits(gd), bits(wd))


@pytest.mark.timeout(600)
def test_xmax_is_taken_over_the_valid_rows():
    """float32 rows, one with an element >= 65520: every query falls back while it is live, none right after it is
    deleted (before any compact), and none after rows are added again."""
    n0 = 5000
    pool, queries = _data(np.float32, n0 + 300, 300)
    pool[17, 5] = 65520.0
    ids = 3 * np.arange(n0, dtype=np.uint64) + 1
    index, model = _dyn(pool[:n0], ids, "l2"), SlotModel(ids, payload=range(n0))
    more = 3 * np.arange(300, dtype=np.uint64) + 2
    for step, want_fb in ((None, 300), (("delete", ids[17:18]), 0), (("add", np.arange(n0, n0 + 300), more, False), 0)):
        if step:
            _apply(index, model, pool, step)
        for k in (10, 100):
            gi, gd, fb = _device_call(index, queries, k)
            assert fb == want_fb, (step and step[0], k, fb)
            wi, wd = _expected(pool, model, "l2", queries, k)
            assert np.array_equal(gi, wi) and np.array_equal(bits(gd), bits(wd))


@pytest.mark.timeout(300)
@pytest.mark.parametrize("metric", ["l2", "ip"])
def test_edge_cases(metric):
    from scalablevectorsearch_b200 import DistanceType, DynamicFlat
    pool, queries = _data(np.float32, 3000, 300, dim=32)
    # created empty, then filled
    index = DynamicFlat.build(np.zeros((0, 32), np.float32), np.zeros(0, np.uint64), DistanceType(METRICS[metric]))
    model = SlotModel([])
    assert index.size == 0 and index.num_slots == 0
    _assert_equal(index, pool, model, metric, queries, 10, "empty")
    ids = 2 * np.arange(2000, dtype=np.uint64) + 5
    _apply(index, model, pool, ("add", np.arange(2000), ids, False))
    for k in (10, 100):
        _assert_equal(index, pool, model, metric, queries, k, "filled")
    # k above the live count: rows padded
    _apply(index, model, pool, ("delete", ids[5:]))
    _assert_equal(index, pool, model, metric, queries, 10, "k > live")
    # everything deleted: every row padded
    _apply(index, model, pool, ("delete", ids[:5]))
    gi, gd = index.search(queries, 10)
    assert (gi == np.uint64(RESERVED)).all() and (gd == (np.inf if metric == "l2" else -np.inf)).all()
    # back again, and search_device on a caller stream == search
    _apply(index, model, pool, ("add", np.arange(2000, 3000), ids[:1000], True))
    import torch
    stream = torch.cuda.Stream()
    for k in (10, 100, 200):
        si, sd = index.search(queries, k)
        di, dd, _ = _device_call(index, queries, k, stream=stream)
        assert np.array_equal(si, di) and np.array_equal(bits(sd), bits(dd)), k
        _assert_equal(index, pool, model, metric, queries, k, "re-added")


@pytest.mark.timeout(300)
def test_errors_leave_the_index_unchanged():
    from scalablevectorsearch_b200 import Svsb200Error
    pool, queries = _data(np.float32, 1500, 50, dim=32)
    ids = 3 * np.arange(1000, dtype=np.uint64) + 1
    index = _dyn(pool[:1000], ids, "l2")
    index.delete(ids[:10])
    before = index.export(), index.size, index.num_slots, index.search(queries, 10)
    bad = [
        lambda: index.add(pool[1000:1002], [ids[20], 99999]),                 # present
        lambda: index.add(pool[1000:1002], [88888, 88888]),                   # repeated
        lambda: index.add(pool[1000:1001], [RESERVED]),                       # reserved
        lambda: index.add(pool[1000:1002].astype(np.float16), [77, 78]),      # wrong dtype
        lambda: index.delete([ids[0]]),                                       # already deleted
        lambda: index.delete([ids[30], 424242]),                              # unknown
        lambda: index.delete([ids[30], ids[30]]),                             # repeated
    ]
    for f in bad:
        with pytest.raises(Svsb200Error):
            f()
        after = index.export(), index.size, index.num_slots, index.search(queries, 10)
        assert all(np.array_equal(a, b) for a, b in zip(before[0], after[0])) and before[1:3] == after[1:3]
        assert np.array_equal(before[3][0], after[3][0]) and np.array_equal(bits(before[3][1]), bits(after[3][1]))
    assert index.has_id(ids[30]) and not index.has_id(ids[0])
    assert index.all_ids().tolist() == ids[10:].tolist()


def _tie_free_equal(got_i, got_d, ref_i, ref_d):
    """Distances bit-equal; id sets equal outside the tie group at the k-th distance."""
    assert np.array_equal(bits(got_d), bits(ref_d))
    for gi, ri, d in zip(got_i, ref_i, got_d):
        keep = d != d[-1]
        assert set(gi[keep].tolist()) == set(ri[keep].tolist())


@pytest.mark.timeout(900)
@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
def test_agrees_with_the_reference_dynamic_flat_index(metric, reflib):
    """The reference's test dataset through the same script on the reference's DynamicFlatIndex (oracle/_ref façade)
    and on the GPU: identical slots, status and external ids after every step, distances bit-equal, ids equal
    outside the tie group at the k-th distance."""
    from oracle.dynamic_flat import RefDynamicFlatLib
    if not RefDynamicFlatLib.available():
        pytest.skip("oracle/_ref/libsvsref_dynamic_flat.so not built")
    z = np.load(f"{GOLDEN}/test_dataset.npz")
    pool, queries = z["data"].astype(np.float32), z["queries"].astype(np.float32)[:100]
    n0 = 6000
    assert pool_size(n0) <= pool.shape[0]
    ids = 3 * np.arange(n0, dtype=np.uint64) + 1
    ref = RefDynamicFlatLib().dynamic_flat(pool[:n0], ids, metric)
    gpu = _dyn(pool[:n0], ids, metric)
    model = SlotModel(ids, payload=range(n0))

    class Both:
        def add(self, pts, ids, reuse_empty):
            a = ref.add(pts, ids, reuse_empty)
            b = gpu.add(pts, ids, reuse_empty)
            assert np.array_equal(a, b)
            return b

        def delete(self, ids):
            ref.delete(ids)
            gpu.delete(ids)

        def compact(self):
            ref.compact()
            gpu.compact()

    def check(step):
        rs, re = ref.export()
        gs, ge = gpu.export()
        assert np.array_equal(rs, gs) and np.array_equal(re, ge), step[:1]
        for k in (10, 100):
            _tie_free_equal(*gpu.search(queries, k), *ref.search(queries, k))

    check(("build",))
    run_script(Both(), model, pool, n0, seed=11, check=check)
