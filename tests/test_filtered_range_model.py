"""The host model of the filtered and range searches (tests/filtered_range_model.py) against first principles.

Driven by an exact brute-force ``plain`` (every row, ordered by (distance, id)) the model has answers that can be
written down without it: the k nearest allowed rows, every row inside the radius, and list lengths computed by hand.
Stub ``plain`` functions cover what an exact search cannot show: the 16384 cap on a large index, lists that change
with their length (as a graph search's do) and searches that are exhausted early."""
import numpy as np
import pytest

from filtered_range_model import LIST_CAP, PAD, filtered, ranged

N, DIM = 2000, 12


def exact_plain(x, greater, reachable=None, calls=None):
    """Exact search over the rows of ``x`` (those in ``reachable`` only, when given): best first, ties by id."""
    rows = np.arange(len(x)) if reachable is None else np.asarray(reachable)

    def plain(queries, kk, window, capacity):
        assert window == capacity == max(window, kk)
        if calls is not None:
            calls.append((len(queries), kk, window))
        ids = np.full((len(queries), kk), PAD, dtype=np.uint64)
        dists = np.full((len(queries), kk), -np.inf if greater else np.inf, dtype=np.float32)
        for i, q in enumerate(queries):
            d = distances(x[rows], q, greater)
            order = np.lexsort((rows, -d if greater else d))[:kk]
            ids[i, :len(order)] = rows[order]
            dists[i, :len(order)] = d[order]
        return ids, dists

    return plain


def distances(x, q, greater):
    d = (x @ q) if greater else ((x - q) ** 2).sum(1)
    return d.astype(np.float32)


def ranking(x, q, greater):
    d = distances(x, q, greater)
    return np.lexsort((np.arange(len(x)), -d if greater else d)), d


@pytest.fixture(scope="module")
def rows():
    rng = np.random.default_rng(0)
    # small integers: exact in float32 and full of distance ties
    return rng.integers(-4, 5, (N, DIM)).astype(np.float32), rng.integers(-4, 5, (9, DIM)).astype(np.float32)


@pytest.mark.parametrize("greater", [False, True])
@pytest.mark.parametrize("share", [1.0, 0.3, 0.02])
def test_filtered_is_the_k_nearest_allowed_rows(rows, greater, share):
    x, q = rows
    allowed = np.random.default_rng(1).random(N) < share
    k = 10
    ids, dists, found, lengths = filtered(exact_plain(x, greater), q, k, 16, allowed, N)
    assert (found == k).all() and ids.dtype == np.uint64 and dists.dtype == np.float32
    for i in range(len(q)):
        order, d = ranking(x, q[i], greater)
        want = order[allowed[order]][:k]
        assert ids[i].tolist() == want.tolist()
        assert np.array_equal(dists[i], d[want])
    assert (lengths[0] == 16) and (len(lengths) > 2) == (share == 0.02)


@pytest.mark.parametrize("first,want_lengths", [(0, [64]), (63, [64, 256]), (100, [64, 256]), (1014, [64, 256, 1024]),
                                                (1015, [64, 256, 1024, N])])
def test_filtered_growth_sequence(rows, first, want_lengths):
    """k = 10 members at ranks first .. first + 9 of one query: the list grows x4 from max(k, window) = 64 until it
    holds all ten, and is clipped to n."""
    x, q = rows
    order, d = ranking(x, q[0], False)
    allowed = np.zeros(N, dtype=bool)
    allowed[order[first:first + 10]] = True
    ids, dists, found, lengths = filtered(exact_plain(x, False), q[:1], 10, 64, allowed, N)
    assert lengths == want_lengths
    assert found.tolist() == [10] and ids[0].tolist() == order[first:first + 10].tolist()
    assert np.array_equal(dists[0], d[order[first:first + 10]])


@pytest.mark.parametrize("greater", [False, True])
def test_filtered_short_rows_are_padded_with_plus_infinity(rows, greater):
    x, q = rows
    allowed = np.zeros(N, dtype=bool)
    allowed[[5, 900, 1999]] = True
    ids, dists, found, lengths = filtered(exact_plain(x, greater), q, 10, 64, allowed, N)
    assert lengths == [64, 256, 1024, N]
    assert (found == 3).all()
    assert all(sorted(r[:3].tolist()) == [5, 900, 1999] for r in ids)
    assert (ids[:, 3:] == PAD).all() and np.isposinf(dists[:, 3:]).all()
    # nothing allowed: the list still grows to the whole index, every row is padding
    ids, dists, found, lengths = filtered(exact_plain(x, greater), q, 4, 64, np.zeros(N, dtype=bool), N)
    assert lengths == [64, 256, 1024, N] and (found == 0).all() and (ids == PAD).all() and np.isposinf(dists).all()


def test_filtered_k_above_window_and_k_above_n(rows):
    x, q = rows
    calls = []
    allowed = np.ones(N, dtype=bool)
    ids, dists, found, lengths = filtered(exact_plain(x, False, calls=calls), q, 50, 8, allowed, N)
    assert lengths == [50] and calls == [(len(q), 50, 50)] and (found == 50).all()
    # window above the list: the search window is max(window, kk), the list stays k long
    calls.clear()
    filtered(exact_plain(x, False, calls=calls), q, 1, 1, allowed, N)
    filtered(exact_plain(x, False, calls=calls), q, 5, 40, allowed, N)
    assert calls == [(len(q), 1, 1), (len(q), 40, 40)]
    # a nine-row index asked for twenty: one list of nine, the rest padding
    small = x[:9]
    ids, dists, found, lengths = filtered(exact_plain(small, False), q, 20, 4, np.ones(9, dtype=bool), 9)
    assert lengths == [9] and (found == 9).all() and (ids[:, 9:] == PAD).all() and np.isposinf(dists[:, 9:]).all()
    assert all(sorted(r[:9].tolist()) == list(range(9)) for r in ids)


def test_an_exhausted_search_is_not_grown(rows):
    """Three reachable rows: the first list already holds padding, so a longer one cannot hold more members."""
    x, q = rows
    plain = exact_plain(x, False, reachable=[3, 40, 700])
    allowed = np.zeros(N, dtype=bool)
    allowed[[40, 41, 42]] = True
    ids, dists, found, lengths = filtered(plain, q, 5, 64, allowed, N)
    assert lengths == [64] and (found == 1).all() and (ids[:, 0] == 40).all() and (ids[:, 1:] == PAD).all()
    res, lengths = ranged(plain, q, np.inf, 64, N, False)
    assert lengths == [64] and all(sorted(i.tolist()) == [3, 40, 700] for i, _ in res)


@pytest.mark.parametrize("greater", [False, True])
def test_ranged_is_every_row_strictly_inside_the_radius(rows, greater):
    x, q = rows
    order, d = ranking(x, q[0], greater)
    # a tie group: the radius equal to its distance shuts the whole group out, the next float lets all of it in
    at = d[order[300]]
    for radius in (at, np.nextafter(at, np.float32(-np.inf if greater else np.inf)), d[order[0]]):
        res, lengths = ranged(exact_plain(x, greater), q, radius, 64, N, greater)
        for i in range(len(q)):
            o, di = ranking(x, q[i], greater)
            want = o[(di[o] > radius) if greater else (di[o] < radius)]
            assert res[i][0].tolist() == want.tolist() and np.array_equal(res[i][1], di[want])
            assert len(want) < lengths[-1] or lengths[-1] == N
    # strict: the radius at a query's best distance returns nothing for it
    assert len(ranged(exact_plain(x, greater), q[:1], d[order[0]], 64, N, greater)[0][0][0]) == 0
    # everything inside: the list reaches the whole index and every row comes back in order
    res, lengths = ranged(exact_plain(x, greater), q[:2], -np.inf if greater else np.inf, 64, N, greater)
    assert lengths == [64, 256, 1024, N]
    assert res[0][0].tolist() == order.tolist() and np.array_equal(res[0][1], d[order])


def test_ranged_growth_small_indexes_and_nan(rows):
    x, q = rows
    order, d = ranking(x, q[0], False)
    # exactly 16 rows inside: the first list (max(window, 16) = 16) is full of them, so one more is needed
    r16 = d[order[16]]
    inside = int((d < r16).sum())
    res, lengths = ranged(exact_plain(x, False), q[:1], r16, 1, N, False)
    assert lengths == ([16, 64] if inside >= 16 else [16]) and len(res[0][0]) == inside
    res, lengths = ranged(exact_plain(x, False), q[:1], d[order[200]], 1, N, False)
    assert lengths[:3] == [16, 64, 256] and len(res[0][0]) == int((d < d[order[200]]).sum())
    # fewer than 16 rows: one list of n
    res, lengths = ranged(exact_plain(x[:9], False), q, np.inf, 1, 9, False)
    assert lengths == [9] and all(len(i) == 9 for i, _ in res)
    for greater in (False, True):
        res, lengths = ranged(exact_plain(x, greater), q, np.nan, 64, N, greater)
        assert lengths == [64] and all(len(i) == 0 and len(dd) == 0 for i, dd in res)


def stub_plain(n, seed):
    """A search over a synthetic index of n rows that is never exhausted: random ids, sorted random distances, both
    drawn afresh for every list length (a graph search's list is not a prefix of its longer lists either)."""
    def plain(queries, kk, window, capacity):
        rng = np.random.default_rng(seed + kk)
        ids = np.stack([rng.permutation(n)[:kk] for _ in queries]).astype(np.uint64)
        dists = np.sort(rng.random((len(queries), kk)).astype(np.float32), axis=1)
        return ids, dists
    return plain


def test_lists_stop_growing_at_the_cap():
    n = 100000
    q = np.zeros((2, 4), dtype=np.float32)
    none = np.zeros(n, dtype=bool)
    assert filtered(stub_plain(n, 0), q, 10, 64, none, n)[3] == [64, 256, 1024, 4096, LIST_CAP]
    # the cap is tested before the step: a list below it grows once more, past it
    assert filtered(stub_plain(n, 0), q, 10, 10, none, n)[3] == [10, 40, 160, 640, 2560, 10240, 40960]
    assert filtered(stub_plain(n, 0), q, 10, 30000, none, n)[3] == [30000]
    assert ranged(stub_plain(n, 0), q, 2.0, 1, n, False)[1] == [16, 64, 256, 1024, 4096, LIST_CAP]
    assert ranged(stub_plain(n, 0), q, -1.0, 100, n, True)[1] == [100, 400, 1600, 6400, 25600]
    assert ranged(stub_plain(n, 0), q, 0.0, 100, n, False)[1] == [100]


def test_every_row_of_a_mixed_batch_comes_from_the_last_list():
    """Query 0 has its k members in the first list, query 1 does not: the batch is run again and query 0's row is
    rewritten from the longer list, whose leading members are different ones."""
    n, k = 5000, 4
    q = np.zeros((2, 4), dtype=np.float32)
    plain = stub_plain(n, 7)
    first, _ = plain(q, 64, 64, 64)
    last, last_d = plain(q, 256, 256, 256)
    allowed = np.zeros(n, dtype=bool)
    taken = np.concatenate([first[1], first[0]])
    allowed[first[0, [1, 5, 9, 30]].astype(np.int64)] = True        # four members in query 0's first list ...
    allowed[np.setdiff1d(last[0], taken)[:k].astype(np.int64)] = True   # ... four others in its second ...
    allowed[np.setdiff1d(last[1], taken)[:k].astype(np.int64)] = True   # ... query 1: none in the first, four in the second
    assert int(allowed[first[0].astype(np.int64)].sum()) == k and not allowed[first[1].astype(np.int64)].any()
    ids, dists, found, lengths = filtered(plain, q, k, 64, allowed, n)
    assert lengths == [64, 256]
    for i in range(2):
        at = np.flatnonzero(allowed[last[i].astype(np.int64)])[:k]
        assert ids[i, :len(at)].tolist() == last[i, at].tolist() and np.array_equal(dists[i, :len(at)], last_d[i, at])
        assert found[i] == len(at) and (ids[i, len(at):] == PAD).all()
    assert ids[0].tolist() != first[0, [1, 5, 9, 30]].tolist()
    assert found[1] == k
