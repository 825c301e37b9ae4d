"""The filtered flat search's contract (include/svsb200.h, svsb200_flat_index_search_filtered), restated in numpy and
checked against brute force on hand-made cases, and its route function (svsb200_flat_filter_plan) pinned at and around
its threshold.  No GPU needed.

The model: the exact top k over the allowed rows (a dynamic flat index: allowed AND Valid slots, Empty slots' bits
ignored), ordered by (distance, id), min(k, A) real entries and the rest all-ones ids with +inf for every metric."""
import ctypes as C

import numpy as np
import pytest

PAD = np.uint64(2**64 - 1)


def bitmap(mask):
    from scalablevectorsearch_b200._lib import _bitmap
    return _bitmap(mask, len(mask))


def allowed_rows(words, n, status=None):
    """Rows whose bit (word i / 32, bit i % 32) is set, i < n, and (status given) whose slot is Valid (1)."""
    i = np.arange(n)
    ok = ((words[i >> 5] >> (i & 31).astype(np.uint32)) & 1).astype(bool)
    return np.flatnonzero(ok if status is None else ok & (status == 1))


def distances(x, q, metric):
    x64, q64 = x.astype(np.float64), q.astype(np.float64)
    if metric == "l2":
        d = ((q64[:, None, :] - x64[None, :, :]) ** 2).sum(-1)
    else:
        d = q64 @ x64.T
        if metric == "cosine":
            d = d / np.linalg.norm(q64, axis=1)[:, None] / np.linalg.norm(x64, axis=1)[None, :]
    return d.astype(np.float32)


def model(dist, words, k, metric, status=None, ext_ids=None):
    """(ids, dists) of the filtered search over the precomputed distances dist[nq, n]."""
    nq, n = dist.shape
    rows = allowed_rows(words, n, status)
    ids = np.full((nq, k), PAD, dtype=np.uint64)
    out = np.full((nq, k), np.inf, dtype=np.float32)
    key = -dist if metric != "l2" else dist
    for qi in range(nq):
        order = rows[np.lexsort((rows, key[qi, rows]))][:k]
        ids[qi, : len(order)] = order if ext_ids is None else ext_ids[order]
        out[qi, : len(order)] = dist[qi, order]
    return ids, out


def brute(dist, allowed, k, metric):
    """First principles: sort every allowed (distance, id) pair and cut at k."""
    nq = dist.shape[0]
    ids = np.full((nq, k), PAD, dtype=np.uint64)
    out = np.full((nq, k), np.inf, dtype=np.float32)
    for qi in range(nq):
        pairs = sorted((float(dist[qi, i]) * (1 if metric == "l2" else -1), int(i)) for i in allowed)
        for j, (_, i) in enumerate(pairs[:k]):
            ids[qi, j], out[qi, j] = i, dist[qi, i]
    return ids, out


def _case(n=100, nq=4, dim=8, seed=0):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((n, dim)).astype(np.float32), rng.standard_normal((nq, dim)).astype(np.float32)


@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
@pytest.mark.parametrize("allowed", [[], [3], [31], [99], [0, 31, 32, 63, 64, 99], list(range(0, 100, 7)),
                                     list(range(100))])
@pytest.mark.parametrize("k", [1, 5, 15])
def test_model_is_the_exact_top_k_over_the_allowed_rows(metric, allowed, k):
    x, q = _case()
    dist = distances(x, q, metric)
    mask = np.zeros(100, dtype=bool)
    mask[allowed] = True
    ids, d = model(dist, bitmap(mask), k, metric)
    bi, bd = brute(dist, np.array(allowed, dtype=np.int64), k, metric)
    assert np.array_equal(ids, bi) and np.array_equal(d.view(np.uint32), bd.view(np.uint32))
    found = min(k, len(allowed))
    assert (ids[:, found:] == PAD).all() and np.isposinf(d[:, found:]).all()   # +inf padding for every metric
    assert (ids[:, :found] != PAD).all()


def test_ties_are_broken_by_id():
    x = np.zeros((64, 4), dtype=np.float32)
    x[::2] = 1.0   # two groups of 32 equal rows
    q = np.ones((2, 4), dtype=np.float32)
    mask = np.ones(64, dtype=bool)
    mask[[0, 10]] = False
    for metric in ("l2", "ip"):
        ids, _ = model(distances(x, q, metric), bitmap(mask), 8, metric)
        assert list(ids[0]) == [2, 4, 6, 8, 12, 14, 16, 18]


@pytest.mark.parametrize("n", [1, 31, 32, 33, 64, 65, 1000])
def test_bitmap_words_and_bits(n):
    rng = np.random.default_rng(n)
    mask = rng.random(n) < 0.3
    mask[-1] = True
    words = bitmap(mask)
    assert words.dtype == np.uint32 and len(words) == (n + 31) // 32
    assert np.array_equal(allowed_rows(words, n), np.flatnonzero(mask))
    if n > 31:   # bit 31 of a full word
        m = np.zeros(n, dtype=bool)
        m[31] = True
        assert bitmap(m)[0] == np.uint32(1 << 31)


def test_bits_past_n_are_ignored():
    words = np.array([0xFFFFFFFF, 0xFFFFFFFF], dtype=np.uint32)
    assert np.array_equal(allowed_rows(words, 40), np.arange(40))


def test_slot_bitmap_ignores_empty_slots():
    """DynamicFlat: the bitmap is over slots; an Empty slot's bit never lets it through, and ids are external."""
    x, q = _case(n=70)
    status = np.ones(70, dtype=np.uint8)
    status[[1, 31, 69]] = 0
    ext = np.arange(70, dtype=np.uint64) * 10 + 5
    ext[status == 0] = PAD
    mask = np.ones(70, dtype=bool)   # Empty slots' bits set
    mask[[2, 40]] = False
    dist = distances(x, q, "l2")
    ids, d = model(dist, bitmap(mask), 70, "l2", status, ext)
    live = np.flatnonzero(mask & (status == 1))
    assert (ids[:, : len(live)] != PAD).all() and (ids[:, len(live):] == PAD).all()
    assert set(ids[0, : len(live)].tolist()) == set(ext[live].tolist())
    bi, bd = brute(dist, live, 70, "l2")
    assert np.array_equal(d.view(np.uint32), bd.view(np.uint32))
    assert np.array_equal(ids[:, : len(live)], ext[bi[:, : len(live)].astype(np.int64)])


def route(n, allowed):
    from scalablevectorsearch_b200.flat import filter_route
    return filter_route(n, allowed)


@pytest.mark.parametrize("n", [64, 1000, 4096, 1_000_000, 1_000_037])
def test_route_threshold(n):
    t = n // 64   # the sparse route takes at most n / 64 allowed rows
    assert route(n, 0) == "sparse"
    assert route(n, t) == "sparse"
    assert route(n, t + 1) == "dense"
    assert route(n, n) == "dense"
    if t > 0:
        assert route(n, t - 1) == "sparse"


def test_route_refuses_more_allowed_than_rows():
    from scalablevectorsearch_b200 import _lib
    out = C.c_int()
    assert _lib.lib().svsb200_flat_filter_plan(10, 11, C.byref(out)) != 0
    assert _lib.lib().svsb200_flat_filter_plan(10, 10, None) != 0
