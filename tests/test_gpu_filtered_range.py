"""Filtered and range search on the GPU against the exact host model of tests/filtered_range_model.py.

Every check is an equality: ids (uint64), distance bits, ``found`` and counts, between the C ABI (through
``Vamana.search_filtered`` / ``range_search``) and the model driven by a plain search that is already held bit for
bit elsewhere -- the oracle's for the static index (test_gpu_parity.py), the dynamic index's own ``search`` for the
dynamic one (test_gpu_dynamic.py).  The model reports the list lengths it went through, and the cases that are meant
to grow, reach the whole index or stop after one list assert that they did."""
import numpy as np
import pytest

from conftest import bits, knn_graph
from filtered_range_model import PAD, filtered, ranged

pytestmark = pytest.mark.gpu

METRICS = {"l2": 0, "ip": 1, "cosine": 2}
PAIRS = ["f32_f32", "f16_f16", "f32_f16", "f32_i8", "i8_i8", "u8_u8"]


def make_index(data, graph, ep, metric, **kw):
    from scalablevectorsearch_b200 import DistanceType, Vamana
    return Vamana.from_arrays(data, graph, ep, DistanceType(METRICS[metric]), **kw)


def launches():
    from scalablevectorsearch_b200 import _lib
    return int(_lib.lib().svsb200_launch_count())


def check_filtered(index, plain, q, k, window, allowed, tag, n=None, offset=0):
    """search_filtered == the model, bit for bit.  Returns (ids, dists, found, list lengths of the model)."""
    n = index.size if n is None else n
    index.search_window_size = window
    ids, dists, found = index.search_filtered(q, k, allowed)
    wi, wd, wf, lengths = filtered(plain, q, k, window, allowed, n)
    wi = np.where(wi == PAD, PAD, wi + np.uint64(offset))
    assert found.dtype == np.uint32 and np.array_equal(found, wf), f"{tag}: found differs"
    assert ids.dtype == np.uint64 and np.array_equal(ids, wi), f"{tag}: ids differ"
    assert np.array_equal(bits(dists), bits(wd)), f"{tag}: distance bits differ"
    return ids, dists, found, lengths


def check_ranged(index, plain, q, radius, window, greater, tag, n=None, offset=0):
    """range_search == the model: per query the same number of results, the same ids and distance bits."""
    n = index.size if n is None else n
    index.search_window_size = window
    got = index.range_search(q, radius)
    want, lengths = ranged(plain, q, radius, window, n, greater)
    assert len(got) == len(want) == len(q)
    for i, ((gi, gd), (wi, wd)) in enumerate(zip(got, want)):
        assert len(gi) == len(wi) == len(gd), f"{tag} query {i}: {len(gi)} results, {len(wi)} expected"
        assert np.array_equal(gi, wi + np.uint64(offset)), f"{tag} query {i}: ids differ"
        assert np.array_equal(bits(gd), bits(wd)), f"{tag} query {i}: distance bits differ"
    return want, lengths


def worse(d, greater):
    """The next float32 on the far side of d: a radius that admits exactly the results at distance d and better."""
    return np.nextafter(np.float32(d), np.float32(-np.inf if greater else np.inf))


class Pair:
    """A GPU index and the oracle's index over the same bytes."""

    def __init__(self, index, want, queries, metric):
        self.index, self.want, self.q, self.metric = index, want, queries, metric
        self.greater = metric != "l2"
        self.plain = want.search
        self.n = index.size


@pytest.fixture(scope="module")
def static(dataset, oracle):
    """(metric, storage) -> Pair over the committed dataset, built once per module."""
    made = {}

    def get(metric, kind):
        if (metric, kind) in made:
            return made[(metric, kind)]
        g, ep = dataset.graph, dataset.entry_point
        if kind.startswith("sq_"):       # sq_<code>_<query type>: the oracle's codes, scale and bias on both sides
            _, code, qt = kind.split("_")
            base = made.get((metric, "sqbase_" + code))
            if base is None:
                want, codes, scale, bias = oracle.sq_index(dataset.data, g, ep, metric, np.dtype(code))
                base = made[(metric, "sqbase_" + code)] = (make_index(codes, g, ep, metric, sq=(scale, bias)), want)
            q = dataset.queries * np.float32(0.37) + np.float32(1.5)
            pair = Pair(base[0], base[1], q.astype(np.float16) if qt == "f16" else q, metric)
        else:
            q, x = dataset.variant(kind)
            pair = Pair(make_index(x, g, ep, metric), oracle.index(x, g, ep, metric), q, metric)
        made[(metric, kind)] = pair
        return pair

    return get


@pytest.fixture(scope="module")
def masks(dataset):
    n = dataset.data.shape[0]
    rng = np.random.default_rng(0)
    return {"all": np.ones(n, dtype=bool), "30%": rng.random(n) < 0.3, "1%": rng.random(n) < 0.01,
            "none": np.zeros(n, dtype=bool)}


# ---- static index, filtered -------------------------------------------------------------------------------------

@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
@pytest.mark.parametrize("kind", PAIRS + ["sq_int8_f32", "sq_int8_f16", "sq_uint8_f32", "sq_uint8_f16"])
def test_filtered_every_metric_and_row_type(static, masks, metric, kind):
    p = static(metric, kind)
    _, _, found, lengths = check_filtered(p.index, p.plain, p.q[:66], 10, 32, masks["30%"], f"{metric} {kind}")
    assert (found == 10).all() and lengths[0] == 32


@pytest.mark.parametrize("metric", ["l2", "ip"])
def test_filtered_lvq8(oracle, metric):
    from scalablevectorsearch_b200 import lvq8_compress
    dim, n = 100, 3000
    rng = np.random.default_rng(dim)
    centres = rng.standard_normal((20, dim)).astype(np.float32)
    x = (centres[rng.integers(0, 20, n)] + 0.3 * rng.standard_normal((n, dim))).astype(np.float32)
    q = (centres[rng.integers(0, 20, 50)] + 0.3 * rng.standard_normal((50, dim))).astype(np.float32)
    graph = knn_graph(x, 32, rng)
    rows, mean = lvq8_compress(x)
    index = make_index(rows, graph, 7, metric, lvq8=(dim, mean))
    want = oracle.lvq8_index(rows, dim, mean, graph, 7, metric)
    for share in (0.3, 0.02):
        allowed = rng.random(n) < share
        for qq in (q, q.astype(np.float16)):
            lengths = check_filtered(index, want.search, qq, 8, 16, allowed, f"lvq8 {metric} {share} {qq.dtype}")[3]
            assert len(lengths) >= (3 if share == 0.02 else 1)
    check_ranged(index, want.search, q[:8], want.search(q[:1], 64, 64, 64)[1][0, 40], 8, metric != "l2", f"lvq8 {metric}")


@pytest.mark.parametrize("metric", ["l2", "ip"])
def test_filtered_selectivity(dataset, static, masks, metric):
    from scalablevectorsearch_b200 import SearchBufferConfig
    p = static(metric, "f32_f32")
    k, window = 10, 64
    # everything allowed: the plain search's first k on a list of max(k, window)
    ids, dists, found, lengths = check_filtered(p.index, p.plain, p.q[:40], k, window, masks["all"], "all")
    p.index.search_parameters.buffer_config = SearchBufferConfig(window, window)
    pi, pd = p.index.search(p.q[:40], window)
    assert lengths == [window] and (found == k).all()
    assert np.array_equal(ids, pi[:, :k]) and np.array_equal(bits(dists), bits(pd[:, :k]))
    # 1 %: the list grows at least twice
    _, _, found, lengths = check_filtered(p.index, p.plain, p.q[:24], k, window, masks["1%"], "1%")
    assert len(lengths) >= 3 and lengths[:3] == [64, 256, 1024] and (found == k).all()
    # a short window: lists of 10, 40, 160 -- far from exact, so a different length gives different rows
    lengths = check_filtered(p.index, p.plain, p.q[:200], k, 10, masks["30%"], "30% w10")[3]
    assert lengths[:2] == [10, 40]
    # three allowed ids, the entry point among them: the list reaches the whole index and rows stay short
    whole = p.plain(p.q[:1], p.n, p.n, p.n)[0][0]
    whole = whole[whole != PAD].astype(np.int64)
    three = np.zeros(p.n, dtype=bool)
    three[[dataset.entry_point, whole[len(whole) // 2], whole[-1]]] = True     # query 0's farthest reachable row
    ids, dists, found, lengths = check_filtered(p.index, p.plain, p.q[:4], k, window, three, "three")
    assert lengths == [64, 256, 1024, 4096, p.n] and (found == 3).all()
    assert (ids[:, 3:] == PAD).all() and np.isposinf(dists[:, 3:]).all()    # +inf for inner product as well
    # nothing allowed
    ids, dists, found, lengths = check_filtered(p.index, p.plain, p.q[:3], 3, window, masks["none"], "none")
    assert lengths[-1] == p.n and (found == 0).all() and (ids == PAD).all() and np.isposinf(dists).all()
    # one allowed id, k = 1 on a list of min(n, 4096): how the runtime's get_distance reads one row's distance
    one = np.zeros(p.n, dtype=bool)
    one[777] = True
    ids, dists, found, lengths = check_filtered(p.index, p.plain, p.q[:3], 1, min(p.n, 4096), one, "one")
    assert lengths[0] == 4096 and (found == 1).all() and (ids == 777).all()


@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_filtered_mixed_batch_rows_come_from_the_last_list(static, metric):
    """Most queries have their k members in the first list; one query's members are out of its reach, so the batch
    is run again and every row is rewritten from the longer list."""
    p = static(metric, "f32_f32")
    q, k, window = p.q[:21], 10, 10
    first, _ = p.plain(q, window, window, window)
    far, _ = p.plain(q[20:21], 40, 40, 40)
    allowed = np.zeros(p.n, dtype=bool)
    allowed[first[:20].astype(np.int64).ravel()] = True      # queries 0..19: all ten of the first list
    allowed[far[0, 8:].astype(np.int64)] = True              # query 20: the tail of its second list,
    allowed[first[20].astype(np.int64)] = False              # none of its first
    ids, dists, found, lengths = check_filtered(p.index, p.plain, q, k, window, allowed, f"mixed {metric}")
    assert lengths == [10, 40] and (found == k).all()
    in_first = allowed[first.astype(np.int64)].sum(1)
    done = np.flatnonzero(in_first == k)
    assert len(done) >= 10 and in_first[20] == 0
    # the rows of the queries that were done are the longer list's: it is a better search, so some of them changed
    assert not np.array_equal(ids[done], first[done])


@pytest.fixture(scope="module")
def ragged(oracle):
    """n = 1501 (a bitmap whose last word holds 29 bits), dim = 100 (masked tail)."""
    rng = np.random.default_rng(1501)
    n, dim = 1501, 100
    x = rng.standard_normal((n, dim)).astype(np.float32)
    q = rng.standard_normal((133, dim)).astype(np.float32)
    graph = knn_graph(x, 32, rng)
    return {m: Pair(make_index(x, graph, 3, m), oracle.index(x, graph, 3, m), q, m) for m in ("l2", "ip")}


@pytest.mark.parametrize("metric", ["l2", "ip"])
def test_filtered_bitmap_edges_and_shapes(ragged, metric):
    p = ragged[metric]
    n = p.n
    edge = np.zeros(n, dtype=bool)
    edge[1472:] = True            # the partial last word
    edge[31::32] = True           # bit 31 of every full word
    for nq in (1, 3, 5, 133):     # four queries per block: full and partial blocks
        _, _, found, lengths = check_filtered(p.index, p.plain, p.q[:nq], 10, 16, edge, f"edge nq{nq}")
        assert len(lengths) >= 2
    last = np.zeros(n, dtype=bool)
    last[1472:] = True
    ids, _, found, lengths = check_filtered(p.index, p.plain, p.q[:9], 40, 16, last, "last word")
    assert lengths[-1] == n and (found == 29).all() and all(sorted(r[:29].tolist()) == list(range(1472, 1501)) for r in ids)
    rng = np.random.default_rng(2)
    half = rng.random(n) < 0.5
    assert check_filtered(p.index, p.plain, p.q, 50, 8, half, "k above window")[3][0] == 50
    assert check_filtered(p.index, p.plain, p.q, 1, 1, half, "k1 w1")[3][0] == 1
    # k above n: one list of n, rows padded past the members
    _, _, found, lengths = check_filtered(p.index, p.plain, p.q[:5], 1600, 8, half, "k above n")
    assert lengths == [n] and (found == int(half.sum())).all()


def small_graph():
    rng = np.random.default_rng(3)
    x = rng.standard_normal((50, 16)).astype(np.float32)
    q = rng.standard_normal((7, 16)).astype(np.float32)
    graph = np.zeros((50, 5), dtype=np.uint32)
    graph[0, :3] = (2, 1, 2)      # 0 -> {1, 2}; 1 and 2 have no out-edges
    graph[7, :2] = (1, 7)         # a self-loop elsewhere
    return x, q, graph


@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
def test_exhausted_searches_stop_after_one_list(oracle, metric):
    """Three, one and one reachable rows: found = the reachable allowed rows, the rest padding, and no second list --
    the call launches as many kernels as one whose queries all finish on the first list."""
    x, q, graph = small_graph()
    everything = np.ones(50, dtype=bool)
    for ep, reachable in ((0, [0, 1, 2]), (1, [1]), (7, [7])):
        index = make_index(x, graph, ep, metric)
        want = oracle.index(x, graph, ep, metric)
        for generic in (0, 1):
            index.set_option("generic_kernel", generic)
            tag = f"{metric} ep{ep} generic{generic}"
            before = launches()
            ids, dists, found, lengths = check_filtered(index, want.search, q, 5, 4, everything, tag)
            exhausted = launches() - before
            assert lengths == [5] and (found == len(reachable)).all()
            assert all(sorted(r[:f].tolist()) == reachable for r, f in zip(ids, found))
            assert (ids[:, len(reachable):] == PAD).all() and np.isposinf(dists[:, len(reachable):]).all()
            before = launches()
            _, _, found, lengths = check_filtered(index, want.search, q, 1, 5, everything, tag + " k1")
            assert lengths == [5] and (found == 1).all() and launches() - before == exhausted
            # only unreachable rows allowed, and one reachable row among unreachable ones
            mask = np.ones(50, dtype=bool)
            mask[reachable] = False
            before = launches()
            _, _, found, lengths = check_filtered(index, want.search, q, 5, 4, mask, tag + " unreachable")
            assert lengths == [5] and (found == 0).all() and launches() - before == exhausted
            mask[reachable[-1]] = True
            assert (check_filtered(index, want.search, q, 5, 4, mask, tag + " one")[2] == 1).all()
            # range search: everything reachable is inside, the list is not grown either
            before = launches()
            res, lengths = check_ranged(index, want.search, q, np.inf if metric == "l2" else -np.inf, 4, metric != "l2", tag)
            grown = launches() - before
            assert lengths == [16] and all(sorted(i.tolist()) == reachable for i, _ in res)
            before = launches()
            check_ranged(index, want.search, q, -np.inf if metric == "l2" else np.inf, 4, metric != "l2", tag + " empty")
            assert launches() - before == grown


@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
def test_both_kernels(static, masks, metric):
    p = static(metric, "f32_f32")
    _, dist = p.plain(p.q[:1], 256, 256, 256)
    try:
        for generic in (0, 1):
            p.index.set_option("generic_kernel", generic)
            check_filtered(p.index, p.plain, p.q[:37], 10, 20, masks["30%"], f"{metric} generic{generic}")
            assert p.index.get_option("last_kernel") == 1 - generic
            lengths = check_filtered(p.index, p.plain, p.q[:13], 10, 20, masks["1%"], f"{metric} 1% generic{generic}")[3]
            assert len(lengths) >= 3
            lengths = check_ranged(p.index, p.plain, p.q[:13], dist[0, 100], 20, p.greater, f"{metric} generic{generic}")[1]
            assert len(lengths) >= 2 and p.index.get_option("last_kernel") == 1 - generic
    finally:
        p.index.set_option("generic_kernel", 0)


def test_wide_graph_rows_take_the_generic_kernel(oracle):
    rng = np.random.default_rng(11)
    n, dim = 1200, 32
    x = rng.standard_normal((n, dim)).astype(np.float32)
    q = rng.standard_normal((30, dim)).astype(np.float32)
    graph = knn_graph(x, 140, rng)
    index = make_index(x, graph, 1, "l2")
    want = oracle.index(x, graph, 1, "l2")
    lengths = check_filtered(index, want.search, q, 10, 16, rng.random(n) < 0.05, "R140")[3]
    assert index.get_option("last_kernel") == 0 and len(lengths) >= 2
    d = want.search(q[:1], 64, 64, 64)[1]
    assert len(check_ranged(index, want.search, q, d[0, 30], 16, False, "R140 range")[1]) >= 2


# ---- static index, range ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
@pytest.mark.parametrize("kind", ["f32_f32", "i8_i8", "u8_u8", "sq_int8_f32"])
def test_range_radii_from_the_result_list(static, metric, kind):
    """Radii taken from query 0's own sorted distances; the data is integer valued, so ties at the radius are real."""
    p = static(metric, kind)
    q = p.q[:5]
    d = p.plain(q[:1], 256, 256, 256)[1][0]
    for window in (1, 64):
        tag = f"{metric} {kind} w{window}"
        first = max(window, 16)
        # the best distance any of the queries reaches on the first list of this window, and the query that reaches it
        top = p.plain(q, first, first, first)[1][:, 0]
        j = int(np.argmax(top) if p.greater else np.argmin(top))
        res, lengths = check_ranged(p.index, p.plain, q, top[j], window, p.greater, tag + " d0")
        assert lengths == [first] and len(res[j][0]) == 0        # strict: a result at the radius is not inside it
        res, lengths = check_ranged(p.index, p.plain, q, worse(top[j], p.greater), window, p.greater, tag + " d0+")
        assert lengths == [first] and len(res[j][0]) >= 1 and (res[j][1] == top[j]).all()
        check_ranged(p.index, p.plain, q, d[20], window, p.greater, tag + " d20")
    res, lengths = check_ranged(p.index, p.plain, q, d[200], 1, p.greater, f"{metric} {kind} d200")
    assert lengths[:3] == [16, 64, 256] and len(res[0][0]) >= 150


@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
def test_range_everything_nothing_and_nan(static, metric):
    p = static(metric, "f32_f32")
    q = p.q[:3]
    far = np.float32(-np.inf if p.greater else np.inf)
    res, lengths = check_ranged(p.index, p.plain, q, far, 64, p.greater, f"{metric} everything")
    assert lengths == [64, 256, 1024, 4096, p.n]
    whole = p.plain(q, p.n, p.n, p.n)[0]
    for (ids, dd), row in zip(res, whole):
        assert np.array_equal(ids, row[row != PAD]) and len(ids) > 9000
        assert (np.diff(dd) <= 0).all() if p.greater else (np.diff(dd) >= 0).all()
    # nothing inside, and a NaN radius (neither comparison holds): empty rows after one list, no growth
    before = launches()
    res, lengths = check_ranged(p.index, p.plain, q, -far, 64, p.greater, f"{metric} nothing")
    one_list = launches() - before
    assert lengths == [64] and all(len(i) == 0 for i, _ in res)
    before = launches()
    res, lengths = check_ranged(p.index, p.plain, q, np.nan, 64, p.greater, f"{metric} nan")
    assert lengths == [64] and all(len(i) == 0 for i, _ in res) and launches() - before == one_list


def test_range_negative_inner_product_radius(static):
    p = static("ip", "f32_f32")
    ids, d = p.plain(p.q[:4], p.n, p.n, p.n)
    radius = np.float32(-1000.0)
    reachable = (ids != PAD).sum(1)
    res, lengths = check_ranged(p.index, p.plain, p.q[:4], radius, 64, True, "ip negative radius")
    assert lengths[-1] == p.n
    # the radius cuts every query's list: thousands inside, and reachable rows left outside
    assert all(1000 < len(i) < r and (dd > radius).all() for (i, dd), r in zip(res, reachable))


@pytest.mark.parametrize("metric", ["l2", "ip"])
def test_range_on_the_ragged_set(ragged, metric):
    p = ragged[metric]
    d = p.plain(p.q[:1], 256, 256, 256)[1][0]
    for radius in (d[0], worse(d[0], p.greater), d[20], d[200], np.float32(-np.inf if p.greater else np.inf)):
        for window in (1, 40):
            check_ranged(p.index, p.plain, p.q[:11], radius, window, p.greater, f"ragged {metric} r{radius} w{window}")
    lengths = check_ranged(p.index, p.plain, p.q[:129], d[60], 16, p.greater, f"ragged {metric} nq129")[1]
    assert len(lengths) >= 2


# ---- shards -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("metric", ["l2", "ip"])
def test_filtered_and_range_search_on_a_shard(dataset, oracle, metric):
    """The second shard of a two-shard ShardedVamana (rows 7100 .. 9999 of the dataset): its bitmap is over its own
    2900 rows, the ids that come back carry the shard's offset."""
    from scalablevectorsearch_b200 import ShardedVamana
    rng = np.random.default_rng(5)
    cut = 7100
    parts = [dataset.data[:cut], dataset.data[cut:]]
    graphs = [knn_graph(x, 24, rng) for x in parts]
    shards = [make_index(x, g, 5, metric) for x, g in zip(parts, graphs)]
    ShardedVamana(shards, [0, cut])      # sets the shards' id offsets
    shard, n = shards[1], len(parts[1])
    want = oracle.index(parts[1], graphs[1], 5, metric)
    q = dataset.queries[:50]
    # the first shard's offset is zero: ids as they are
    check_filtered(shards[0], oracle.index(parts[0], graphs[0], 5, metric).search, q, 10, 32, rng.random(cut) < 0.3,
                   f"shard 0 {metric}")
    for name, allowed in (("30%", rng.random(n) < 0.3), ("2%", rng.random(n) < 0.02), ("all", np.ones(n, dtype=bool)),
                          ("none", np.zeros(n, dtype=bool))):
        ids, _, found, _ = check_filtered(shard, want.search, q[:50 if name != "none" else 3], 10, 32, allowed,
                                          f"shard {metric} {name}", offset=cut)
        assert (ids[ids != PAD] >= cut).all() and (found == (0 if name == "none" else 10)).all()
    d = want.search(q[:1], 256, 256, 256)[1][0]
    for radius in (d[0], worse(d[0], metric != "l2"), d[100]):
        check_ranged(shard, want.search, q[:8], radius, 32, metric != "l2", f"shard {metric} r{radius}", offset=cut)


# ---- dynamic index ----------------------------------------------------------------------------------------------

class Dynamic:
    """A DynamicVamana and the plain search the model trusts: the index's own ``search`` on a (w, w) buffer, with
    external ids mapped back to slots so that the model can test them against a mask over slots."""

    def __init__(self, index, metric):
        self.index, self.greater = index, metric != "l2"
        self.refresh()

    def refresh(self):
        _, self.status, self.ext, self.entry_point = self.index.export()
        self.n = len(self.status)
        order = np.argsort(self.ext[self.status == 1])
        self._sorted_ext = self.ext[self.status == 1][order]
        self._sorted_slot = np.flatnonzero(self.status == 1)[order]

    def plain(self, q, kk, window, capacity):
        from scalablevectorsearch_b200 import SearchBufferConfig
        self.index.search_parameters.buffer_config = SearchBufferConfig(window, capacity)
        ids, dists = self.index.search(q, kk)
        slots = np.full(ids.shape, PAD, dtype=np.uint64)
        at = np.searchsorted(self._sorted_ext, ids[ids != PAD])
        assert np.array_equal(self._sorted_ext[at], ids[ids != PAD]), "the plain search returned an id that is not Valid"
        slots[ids != PAD] = self._sorted_slot[at]
        return slots, dists

    def check_filtered(self, q, k, window, allowed, tag):
        self.index.search_window_size = window
        ids, dists, found = self.index.search_filtered(q, k, allowed)
        wi, wd, wf, lengths = filtered(self.plain, q, k, window, allowed & (self.status == 1), self.n)
        wi[wi != PAD] = self.ext[wi[wi != PAD].astype(np.int64)]
        assert np.array_equal(found, wf), f"{tag}: found differs"
        assert np.array_equal(ids, wi), f"{tag}: ids differ"
        assert np.array_equal(bits(dists), bits(wd)), f"{tag}: distance bits differ"
        return ids, dists, found, lengths

    def check_ranged(self, q, radius, window, tag):
        self.index.search_window_size = window
        got = self.index.range_search(q, radius)
        want, lengths = ranged(self.plain, q, radius, window, self.n, self.greater)
        for i, ((gi, gd), (wi, wd)) in enumerate(zip(got, want)):
            assert len(gi) == len(wi), f"{tag} query {i}: {len(gi)} results, {len(wi)} expected"
            assert np.array_equal(gi, self.ext[wi.astype(np.int64)]), f"{tag} query {i}: ids differ"
            assert np.array_equal(bits(gd), bits(wd)), f"{tag} query {i}: distance bits differ"
        return want, lengths

    def battery(self, q, tag):
        """Every filtered and range case on the index as it stands."""
        rng = np.random.default_rng(9)
        n, k, window = self.n, 10, 32
        valid = self.status == 1
        ids, _, found, lengths = self.check_filtered(q, k, window, np.ones(n, dtype=bool), tag + " all")
        assert lengths == [window] and (found == k).all()
        self.check_filtered(q, k, window, rng.random(n) < 0.3, tag + " 30%")
        _, _, found, lengths = self.check_filtered(q[:12], k, window, rng.random(n) < 0.01, tag + " 1%")
        assert len(lengths) >= 3 and (found == k).all()
        # only slots that are not Valid: nothing comes back, though every one of them is set in the mask
        ids, dists, found, lengths = self.check_filtered(q[:3], k, window, ~valid, tag + " not valid")
        assert (found == 0).all() and (ids == PAD).all() and np.isposinf(dists).all()
        # Valid slots at 5 % plus every slot that is not Valid
        mask = ~valid | (rng.random(n) < 0.05)
        ids, _, found, _ = self.check_filtered(q, k, window, mask, tag + " mixed")
        live = set(self.ext[valid & mask].tolist())
        assert (found == k).all() and all(int(i) in live for i in ids.ravel())
        d = self.plain(q[:1], 256, 256, 256)[1][0]
        res, _ = self.check_ranged(q[:8], d[0], window, tag + " d0")
        assert len(res[0][0]) == 0
        res, _ = self.check_ranged(q[:8], worse(d[0], self.greater), window, tag + " d0+")
        assert len(res[0][0]) >= 1
        self.check_ranged(q[:8], d[20], 1, tag + " d20")
        lengths = self.check_ranged(q[:8], d[200], window, tag + " d200")[1]
        assert len(lengths) >= 3
        res, lengths = self.check_ranged(q[:2], -np.inf if self.greater else np.inf, window, tag + " everything")
        # the list grows until it holds padding: every reachable Valid row is inside
        assert len(lengths) >= 4 and lengths[-1] >= min(n, valid.sum()) and all(len(i) > 0.9 * valid.sum() for i, _ in res)
        assert all(len(i) == 0 for i, _ in self.check_ranged(q[:3], np.nan, window, tag + " nan")[0])


@pytest.mark.parametrize("metric,dtype,frac", [("l2", np.float32, 0.2), ("ip", np.float16, 0.6), ("ip", np.float32, 0.2),
                                               ("l2", np.float16, 0.6)])
def test_dynamic_filtered_and_range(dataset, metric, dtype, frac):
    from test_gpu_dynamic import make_index as make_dynamic
    rng = np.random.default_rng(int(frac * 10))
    index, data, ext, valid = make_dynamic(dataset, metric, dtype, frac, rng, delete_entry=True)
    q = dataset.queries[:16].astype(np.float32)
    dyn = Dynamic(index, metric)
    assert dyn.status[dataset.entry_point] == 2 and np.array_equal(dyn.status == 1, valid)
    dyn.battery(q, f"{metric} {np.dtype(dtype).name} {frac}")
    # Empty and Deleted slots side by side: consolidate, then delete some more
    index.consolidate()
    index.delete(rng.choice(index.all_ids(), 500, replace=False))
    dyn.refresh()
    assert (dyn.status == 0).any() and (dyn.status == 2).sum() == 500
    dyn.battery(q, f"{metric} {np.dtype(dtype).name} {frac} empty+deleted")
    index.consolidate()
    index.compact()
    dyn.refresh()
    assert dyn.n == index.size and (dyn.status == 1).all()
    dyn.battery(q, f"{metric} {np.dtype(dtype).name} {frac} compacted")
