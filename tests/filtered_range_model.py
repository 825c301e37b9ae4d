"""Host model of the filtered and range searches (svsb200_search_filtered / svsb200_range_search), in plain numpy.

Both procedures are a loop around a plain graph search that is trusted on its own: run the whole batch with a result
list of ``kk`` entries per query (search window = capacity = max(window, kk)), look at every query's list, and run
the batch again with a list four times as long while some query could still gain from it.  The model restates that
loop from the contract in include/svsb200.h; the plain search is handed in as

    plain(queries, kk, window, capacity) -> (ids uint64[nq, kk], dists float32[nq, kk])

with rows sorted best first and short rows padded with id = all-ones.  Each function also returns the list lengths
it went through, so that a test can assert which case it hit (growth, the whole index, the cap).
"""
import numpy as np

PAD = np.uint64(0xFFFFFFFFFFFFFFFF)
LIST_CAP = 16384   # a list this long (or longer) is never grown again


def _grow(plain, queries, kk, window, n, unfinished):
    """Runs the batch with lists of kk, 4 kk, 16 kk, ... entries until no row is unfinished, the list holds the whole
    index or has reached the cap.  Returns the last lists and the lengths tried."""
    lengths = []
    while True:
        kk = min(kk, n)
        w = max(window, kk)
        ids, dists = plain(queries, kk, w, w)
        ids = np.asarray(ids, dtype=np.uint64).reshape(len(queries), kk)
        dists = np.asarray(dists, dtype=np.float32).reshape(len(queries), kk)
        lengths.append(kk)
        if not any(unfinished(i, d) for i, d in zip(ids, dists)) or kk >= n or kk >= LIST_CAP:
            return ids, dists, lengths
        kk *= 4


def filtered(plain, queries, k, window, allowed, n):
    """The first k results, in result order, whose id is set in ``allowed`` (bool[n]).

    Returns (ids uint64[nq, k], dists float32[nq, k], found uint32[nq], lengths).  A query is unfinished while it has
    fewer than k members and its list is full (no padding: a longer list could hold more).  Every row is taken from
    the last list of the batch.  Short rows are padded with all-ones / +inf whatever the metric."""
    allowed = np.asarray(allowed, dtype=bool)
    assert allowed.shape == (n,)

    def members(ids):
        valid = ids != PAD
        keep = np.zeros(len(ids), dtype=bool)
        keep[valid] = allowed[ids[valid].astype(np.int64)]
        return keep

    def unfinished(ids, dists):
        return int(members(ids).sum()) < k and not (ids == PAD).any()

    ids, dists, lengths = _grow(plain, queries, max(k, window), window, n, unfinished)
    nq = len(queries)
    out_ids = np.full((nq, k), PAD, dtype=np.uint64)
    out_dists = np.full((nq, k), np.inf, dtype=np.float32)
    found = np.zeros(nq, dtype=np.uint32)
    for q in range(nq):
        at = np.flatnonzero(members(ids[q]))[:k]
        found[q] = len(at)
        out_ids[q, :len(at)] = ids[q, at]
        out_dists[q, :len(at)] = dists[q, at]
    return out_ids, out_dists, found, lengths


def ranged(plain, queries, radius, window, n, greater):
    """Per query, the leading results strictly inside the radius: d < radius, or d > radius when ``greater`` (inner
    product, cosine).  Returns ([(ids, dists)] per query, lengths).  A query is unfinished while its whole list is
    inside the radius and full.  A NaN radius compares false either way: every row is empty after one list."""
    radius = np.float32(radius)

    def count(ids, dists):
        inside = (dists > radius) if greater else (dists < radius)
        stop = np.flatnonzero(~((ids != PAD) & inside))
        return int(stop[0]) if len(stop) else len(ids)

    def unfinished(ids, dists):
        return count(ids, dists) == len(ids)

    ids, dists, lengths = _grow(plain, queries, max(window, 16), window, n, unfinished)
    rows = []
    for q in range(len(queries)):
        c = count(ids[q], dists[q])
        rows.append((ids[q, :c].copy(), dists[q, :c].copy()))
    return rows, lengths
