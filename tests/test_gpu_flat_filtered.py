"""The filtered exact search of Flat and DynamicFlat (svsb200_flat_index_search_filtered, svsb200_dynamic_flat_search_filtered)
held to its defining identity: the result equals the unfiltered search of a Flat built from the allowed rows in
ascending id (slot) order, ids mapped back, distance bits equal, only the padding's distance changed to +inf.  Masks are
chosen on both sides of the sparse route's threshold, with filter_route as witness."""
import ctypes as C

import numpy as np
import pytest

from conftest import bits

pytestmark = pytest.mark.gpu

PAD = np.uint64(2**64 - 1)
METRICS = {"l2": 0, "ip": 1, "cosine": 2}


def _flat(x, metric):
    from scalablevectorsearch_b200 import DistanceType, Flat
    return Flat(x, DistanceType(METRICS[metric]))


def _expected(x, q, metric, rows, k, ids_of=None):
    """The unfiltered search over the rows `rows` (ascending), ids mapped back through `rows` (then `ids_of`)."""
    nq = q.shape[0]
    ids = np.full((nq, k), PAD, dtype=np.uint64)
    d = np.full((nq, k), np.inf, dtype=np.float32)
    if len(rows):
        si, sd = _flat(x[rows], metric).search(q, k)
        real = si != PAD
        mapped = rows[si[real].astype(np.int64)]
        ids[real] = mapped if ids_of is None else ids_of[mapped]
        d[real] = sd[real]
    return ids, d


def _same(got, want, tag):
    gi, gd = got[0], got[1]
    wi, wd = want
    assert np.array_equal(gi, wi), f"{tag}: ids differ in {np.count_nonzero(gi != wi)} entries"
    assert np.array_equal(bits(gd), bits(wd)), f"{tag}: distance bits differ"


def _data(n, nq, dim, dtype, seed=0):
    rng = np.random.default_rng(seed)
    if dtype in (np.int8, np.uint8):
        lo, hi = (-128, 128) if dtype == np.int8 else (0, 256)
        return rng.integers(lo, hi, (n, dim)).astype(dtype), rng.integers(lo, hi, (nq, dim)).astype(dtype)
    return rng.standard_normal((n, dim)).astype(dtype), rng.standard_normal((nq, dim)).astype(dtype)


def _masks(n, rng):
    m = {"all": np.ones(n, bool), "none": np.zeros(n, bool)}
    one = np.zeros(n, bool)
    one[31] = True
    m["bit31"] = one
    last = np.zeros(n, bool)
    last[n - 1] = True
    m["last_word"] = last
    for f in (0.5, 0.05, 0.01, 0.001):
        m[f"rand{f}"] = rng.random(n) < f
    tiles = rng.random(n) < 0.5
    tiles[256:768] = False   # whole 256-row tiles cleared
    m["tiles_cleared"] = tiles
    return m


def _check(x, q, metric, mask, k, tag):
    from scalablevectorsearch_b200.flat import filter_route
    flat = _flat(x, metric)
    ids, d, found, allowed = flat.search_filtered(q, k, mask, with_counts=True)
    rows = np.flatnonzero(mask)
    assert allowed == len(rows), tag
    assert (found == min(k, len(rows))).all(), tag
    _same((ids, d), _expected(x, q, metric, rows, k), tag)
    return filter_route(x.shape[0], len(rows))


TYPES = [(np.float32, np.float32), (np.float32, np.float16), (np.float16, np.float32), (np.float16, np.float16),
         (np.int8, np.int8), (np.uint8, np.uint8), (np.int8, np.float32), (np.uint8, np.float32)]


@pytest.mark.parametrize("rt,qt", TYPES, ids=lambda t: np.dtype(t).name)
@pytest.mark.parametrize("metric", ["l2", "ip"])
def test_types_metrics_and_masks(rt, qt, metric):
    n, dim = 3000, 40
    x, _ = _data(n, 1, dim, rt, seed=1)
    _, q = _data(1, 300, dim, qt, seed=2)
    rng = np.random.default_rng(3)
    routes = set()
    for name, mask in _masks(n, rng).items():
        for k in (1, 10, 26):
            routes.add(_check(x, q, metric, mask, k, f"{name} k={k}"))
    assert routes == {"sparse", "dense"}


@pytest.mark.parametrize("k", [1, 10, 25, 26, 100, 121, 122, 1024])
@pytest.mark.parametrize("nq", [1, 256, 257])
def test_k_and_batch(k, nq):
    n, dim = 4096, 24
    x, q = _data(n, nq, dim, np.float32, seed=k + nq)
    rng = np.random.default_rng(k)
    for frac in (0.5, 0.01):
        _check(x, q, "l2", rng.random(n) < frac, k, f"frac={frac}")


def test_large_batch_both_routes():
    n, dim = 20_000, 32
    x, q = _data(n, 10_000, dim, np.float32, seed=7)
    rng = np.random.default_rng(8)
    assert _check(x, q, "l2", rng.random(n) < 0.3, 10, "dense") == "dense"
    assert _check(x, q, "ip", rng.random(n) < 0.005, 100, "sparse") == "sparse"


def test_cosine_and_around_512():
    n, dim = 3000, 16
    x, q = _data(n, 300, dim, np.float32, seed=9)
    for a in (511, 512, 513):
        mask = np.zeros(n, bool)
        mask[np.random.default_rng(a).choice(n, a, replace=False)] = True
        for metric in ("l2", "cosine"):
            _check(x, q, metric, mask, 10, f"{metric} A={a}")


def test_threshold_both_sides():
    from scalablevectorsearch_b200.flat import filter_route
    n = 6400
    x, q = _data(n, 300, 32, np.float32, seed=11)
    t = n // 64
    for a, want in ((t, "sparse"), (t + 1, "dense")):
        mask = np.zeros(n, bool)
        mask[np.random.default_rng(a).choice(n, a, replace=False)] = True
        assert filter_route(n, a) == want
        assert _check(x, q, "l2", mask, 10, f"A={a}") == want


def test_fp16_overflow_rows_take_the_masked_scan():
    import flat_range_fixtures as F
    for metric in ("l2", "ip"):
        x, q, z = F.data_overflow(metric, nq=300)
        mask = np.random.default_rng(1).random(x.shape[0]) < 0.6
        mask[z] = True
        _check(x, q, metric, mask, 10, f"overflow {metric}")


def test_integer_rows_in_the_2_24_regime():
    n, dim = 2048, 512
    rng = np.random.default_rng(12)
    x = rng.integers(200, 256, (n, dim)).astype(np.uint8)
    q = rng.integers(0, 60, (300, dim)).astype(np.uint8)
    _check(x, q, "l2", rng.random(n) < 0.5, 10, "u8 2^24")


def _device(index_fn, q, k, words, stream):
    import torch
    dq = torch.from_numpy(np.ascontiguousarray(q)).cuda()
    db = torch.from_numpy(words.view(np.int32).copy()).cuda()
    ids = torch.empty((q.shape[0], k), dtype=torch.int64, device="cuda")
    d = torch.empty((q.shape[0], k), dtype=torch.float32, device="cuda")
    fb = index_fn(dq.data_ptr(), q.dtype, q.shape[0], k, db.data_ptr(), ids.data_ptr(), d.data_ptr(),
                  stream=stream.cuda_stream)
    return ids, d, fb, (dq, db)


def test_two_streams_with_different_masks():
    import torch
    from scalablevectorsearch_b200._lib import _bitmap
    n = 8192
    x, q = _data(n, 2000, 32, np.float32, seed=13)
    flat = _flat(x, "l2")
    rng = np.random.default_rng(14)
    masks = [rng.random(n) < 0.4, rng.random(n) < 0.003]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    outs = [_device(flat.search_filtered_device, q, 10, _bitmap(m, n), s) for m, s in zip(masks, streams)]
    torch.cuda.synchronize()
    for m, (ids, d, _, _) in zip(masks, outs):
        _same((ids.cpu().numpy().view(np.uint64), d.cpu().numpy()), _expected(x, q, "l2", np.flatnonzero(m), 10), "stream")


def test_refusals():
    from scalablevectorsearch_b200 import _lib
    x, q = _data(600, 4, 16, np.float32)
    flat = _flat(x, "l2")
    lib = _lib.lib()
    ids = np.empty((4, 10), np.uint64)
    d = np.empty((4, 10), np.float32)
    words = _lib._bitmap(np.ones(600, bool), 600)
    assert lib.svsb200_flat_index_search_filtered(flat._h, q.ctypes.data, 0, 4, 10, None, ids.ctypes.data, d.ctypes.data,
                                                  None) != 0
    for k in (0, 1025):
        with pytest.raises(_lib.Svsb200Error):
            flat.search_filtered(q, k, np.ones(600, bool))
    with pytest.raises(_lib.Svsb200Error):   # int8 queries over float rows, even with nothing allowed
        flat.search_filtered(q.astype(np.int8), 10, np.zeros(600, bool))
    assert words.shape == (19,)


def test_unfiltered_search_unchanged_in_the_same_run():
    x, q = _data(5000, 300, 32, np.float32, seed=15)
    flat = _flat(x, "l2")
    before = flat.search(q, 10)
    flat.search_filtered(q, 10, np.random.default_rng(0).random(5000) < 0.5)
    flat.search_filtered(q, 10, np.random.default_rng(0).random(5000) < 0.001)
    after = flat.search(q, 10)
    _same(after, before, "unfiltered")


# ---- DynamicFlat ----
def _dyn_expected(dyn, rows_by_id, q, metric, slot_mask, k):
    status, ext = dyn.export()
    slots = np.flatnonzero(slot_mask & (status == 1))
    x = np.stack([rows_by_id[int(e)] for e in ext[slots]]) if len(slots) else np.zeros((0, q.shape[1]), np.float32)
    ids = np.full((q.shape[0], k), PAD, dtype=np.uint64)
    d = np.full((q.shape[0], k), np.inf, dtype=np.float32)
    if len(slots):
        si, sd = _flat(x, metric).search(q, k)
        real = si != PAD
        ids[real] = ext[slots][si[real].astype(np.int64)]
        d[real] = sd[real]
    return ids, d, len(slots)


@pytest.mark.parametrize("metric", ["l2", "ip"])
@pytest.mark.parametrize("dtype", [np.float32, np.int8])
def test_dynamic_flat_through_mutations(metric, dtype):
    from scalablevectorsearch_b200 import DistanceType, DynamicFlat
    rng = np.random.default_rng(16)
    n, dim = 4000, 32
    x, q = _data(n + 1000, 300, dim, dtype, seed=17)
    qs = [q, q.astype(np.float32)] if dtype == np.int8 else [q]
    ids = np.arange(n, dtype=np.uint64) * 3 + 1
    rows = {int(i): x[j] for j, i in enumerate(ids)}
    dyn = DynamicFlat.build(x[:n], ids, DistanceType(METRICS[metric]))

    def check(tag):
        status, _ = dyn.export()
        for frac in (0.7, 0.01, 0.0):
            mask = rng.random(len(status)) < frac
            mask[status == 0] = True   # Empty slots' bits set: ignored
            for qq in qs:
                for k in (10, 100):
                    gi, gd, found, allowed = dyn.search_filtered(qq, k, mask, with_counts=True)
                    wi, wd, a = _dyn_expected(dyn, rows, qq, metric, mask, k)
                    assert allowed == a, tag
                    _same((gi, gd), (wi, wd), f"{tag} frac={frac} k={k}")

    check("built")
    dyn.delete(ids[rng.choice(n, 1500, replace=False)])
    check("deleted")
    new = np.arange(500, dtype=np.uint64) * 3 + 2
    dyn.add(x[n:n + 500], new, reuse_empty=True)
    rows.update({int(i): x[n + j] for j, i in enumerate(new)})
    check("reuse_empty")
    dyn.compact()
    check("compacted")


def test_dynamic_delete_right_after_a_device_search():
    import torch
    from scalablevectorsearch_b200 import DistanceType, DynamicFlat
    from scalablevectorsearch_b200._lib import _bitmap
    n = 6000
    x, q = _data(n, 2000, 32, np.float32, seed=18)
    ids = np.arange(n, dtype=np.uint64)
    rows = {int(i): x[i] for i in ids}
    dyn = DynamicFlat.build(x, ids, DistanceType.L2)
    rng = np.random.default_rng(19)
    for frac in (0.5, 0.005):
        mask = rng.random(dyn.num_slots) < frac
        want = _dyn_expected(dyn, rows, q, "l2", mask, 10)
        s = torch.cuda.Stream()
        gi, gd, _, keep = _device(dyn.search_filtered_device, q, 10, _bitmap(mask, dyn.num_slots), s)
        victims = np.flatnonzero(mask & (dyn.export()[0] == 1))[:50].astype(np.uint64)
        dyn.delete(victims)   # no synchronisation: the mutation waits for the search
        torch.cuda.synchronize()
        _same((gi.cpu().numpy().view(np.uint64), gd.cpu().numpy()), want[:2], f"frac={frac}")
        for v in victims:
            rows.pop(int(v))
