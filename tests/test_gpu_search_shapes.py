"""Every kernel shape the search dispatch can choose, against the oracle, ids and distance bits.

* the exhaustive scan over every row kind (plain pairs, SQ codes, LVQ-8 rows) at each dimension class the distance code
  switches on (tails, static 96 / 128, generic, split), k from 1 to 1024, split and un-split batches, n < k padding --
  and a float64 layer that recomputes each returned distance from the operands the kernel sees and bounds its rounding
  error, so that the SQ and LVQ-8 paths are held to something other than their own restatement;
* the tuning knobs that never change results (rows_in_flight, warps_per_cta, ctas_per_sm, no_split, filter_tag16,
  host_chunks), each against the oracle, with the kernel the setting selects asserted;
* the visited filter at its exactness boundary: the n at which the lean kernel doubles its sets and the generic kernel
  falls back to 32-bit entries;
* compressed and integer rows at wide and ragged dimensions on both kernels;
* the LVQ-8 encoder against float64, including the float16 range edges it refuses.
"""
import numpy as np
import pytest

from conftest import bits, knn_graph

pytestmark = pytest.mark.gpu

METRICS = {"l2": 0, "ip": 1, "cosine": 2}
U = 2.0 ** -24
ALL_ONES = np.uint64(0xFFFFFFFFFFFFFFFF)
WINDOWS = ((8, 8, 8), (33, 97, 20), (130, 300, 50))   # (window, capacity, k)


def make_index(data, graph, ep, metric, **kw):
    from scalablevectorsearch_b200 import DistanceType, Vamana
    return Vamana.from_arrays(data, graph, ep, DistanceType(METRICS[metric]), **kw)


def search(index, queries, k, window, capacity):
    from scalablevectorsearch_b200 import SearchBufferConfig
    index.search_parameters.buffer_config = SearchBufferConfig(window, capacity)
    return index.search(queries, k)


def assert_same(got, want_ids, want_dists, tag):
    ids, dists = got
    assert np.array_equal(ids.astype(np.uint64), want_ids.astype(np.uint64)), f"{tag}: neighbour ids differ"
    assert np.array_equal(bits(dists), bits(want_dists)), f"{tag}: distances differ (bit-exact bar)"


def f16(x):
    """float16 copy with subnormals flushed: the scalar float16 -> float conversion of the SQ and cosine query
    preparation flushes them, and the float64 layer below works on the values the kernel sees."""
    h = np.asarray(x, dtype=np.float32).astype(np.float16)
    h[np.abs(h) < np.float16(2.0 ** -14)] = 0
    return h


def launches():
    from scalablevectorsearch_b200 import _lib
    return int(_lib.lib().svsb200_launch_count())


# ------------------------------------------------------------------------------------------------------------------
# Row kinds: data, queries, the oracle's distances and the float64 model of every returned distance
# ------------------------------------------------------------------------------------------------------------------
PLAIN = ["f32_f32", "f32_f16", "f16_f16", "f16_f32", "f32_i8", "i8_i8", "f32_u8", "u8_u8"]
SQ = ["sq_i8_f32", "sq_i8_f16", "sq_u8_f32", "sq_u8_f16"]
LVQ = ["lvq8_f32", "lvq8_f16"]
KINDS = PLAIN + SQ + LVQ


def kind_metrics(kind):
    return ["l2", "ip"] if kind.startswith("lvq8") else ["l2", "ip", "cosine"]


def _floats(rng, shape, coarse, scale=1.0):
    x = rng.standard_normal(shape) * scale
    return np.round(x * 2) / 2 if coarse else x


def _nonzero_rows(x):
    """Cosine of a zero-norm row is NaN, which is out of scope here: give such rows a first element."""
    x = np.array(x)
    zero = ~np.any(x != 0, axis=1)
    x[zero, 0] = 1
    return x


class Kind:
    """One row kind over n x dim data: the index, its queries, the oracle's distances and the float64 layer."""

    def __init__(self, name, n, dim, nq, rng, coarse, oracle):
        self.name, self.dim = name, dim
        self.sq = self.lvq = None
        if name in PLAIN:
            qt, dt = name.split("_")
            self.x = _nonzero_rows(self._draw(dt, (n, dim), rng, coarse))
            self.q = _nonzero_rows(self._draw(qt, (nq, dim), rng, coarse))
            self.rows = self.x
        elif name in SQ:
            # codes, scale and bias from the oracle's SQDataset::compress (pinned against the reference)
            _, ct, qt = name.split("_")
            self.code = np.int8 if ct == "i8" else np.uint8
            self.x = (_floats(rng, (n, dim), coarse, 2.0) + 0.3).astype(np.float32)
            _, self.rows, scale, bias = oracle.sq_index(self.x, np.zeros((n, 2), np.uint32), 0, "l2", self.code)
            self.sq = (np.float32(scale), np.float32(bias))
            q = _floats(rng, (nq, dim), coarse, 2.0) + 0.3
            self.q = f16(q) if qt == "f16" else q.astype(np.float32)
        else:
            from scalablevectorsearch_b200 import lvq8_compress
            qt = name.split("_")[1]
            self.x = _floats(rng, (n, dim), coarse).astype(np.float32) + np.float32(0.5)
            self.rows, self.mean = lvq8_compress(self.x)
            assert np.array_equal(self.rows, oracle.lvq8_compress(self.x, self.mean)), f"{name} d{dim}: encoder bytes"
            self.lvq = (dim, self.mean)
            q = _floats(rng, (nq, dim), coarse) + 0.5
            self.q = f16(q) if qt == "f16" else q.astype(np.float32)

    @staticmethod
    def _draw(t, shape, rng, coarse):
        if t == "i8":
            return rng.integers(-128, 128, shape).astype(np.int8)
        if t == "u8":
            return rng.integers(0, 256, shape).astype(np.uint8)
        x = _floats(rng, shape, coarse, 3.0 if coarse else 1.0)
        return f16(x) if t == "f16" else x.astype(np.float32)

    def index(self, graph, ep, metric):
        return make_index(self.rows, graph, ep, metric, sq=self.sq, lvq8=self.lvq)

    def oracle_index(self, oracle, graph, ep, metric):
        if self.sq is not None:
            index, codes, _, _ = oracle.sq_index(self.x, graph, ep, metric, self.code)
            assert np.array_equal(codes, self.rows)
            return index
        if self.lvq is not None:
            return oracle.lvq8_index(self.rows, self.dim, self.mean, graph, ep, metric)
        return oracle.index(self.rows, graph, ep, metric)

    def oracle_distances(self, oracle, metric, i):
        if self.sq is not None:
            return oracle.sq_distance_rows(metric, self.q[i], self.rows, *self.sq)
        if self.lvq is not None:
            return oracle.lvq8_distance_rows(metric, self.q[i], self.rows, self.dim, self.mean)
        return oracle.distance_rows(metric, self.q[i], self.rows)

    # ---- float64 layer ------------------------------------------------------------------------------------------
    def _operands(self, i, ids):
        """(query, rows) as float64: the operands the kernel's float tree sees."""
        q = self.q[i].astype(np.float64)
        if self.lvq is not None:
            off = (self.dim + 3) // 4 * 4
            r = self.rows[ids]
            d16 = r[:, off:off + 2].copy().view(np.float16)[:, 0].astype(np.float64)
            l16 = r[:, off + 2:off + 4].copy().view(np.float16)[:, 0].astype(np.float64)
            # decode fma(delta16, c, lower16): the product and sum are exact in float64, then one rounding to fp32
            y = (d16[:, None] * r[:, :self.dim] + l16[:, None]).astype(np.float32).astype(np.float64)
            return q, y
        if self.sq is not None:
            scale, bias = self.sq
            # cosine decompresses scale * c + bias in fp32, one rounding per operation (scalar.h:44-46)
            y = (scale * self.rows[ids].astype(np.float32) + bias).astype(np.float64)
            return q, y
        return q, self.rows[ids].astype(np.float64)

    def check_float64(self, metric, i, ids, d32, tag):
        """|d32 - d64| <= (dim + 8) 2^-24 sum|terms| * 1.01 for every returned (id, distance); SQ L2 is exact."""
        keep = ids != ALL_ONES
        ids, d32 = ids[keep].astype(np.int64), d32[keep].astype(np.float64)
        if len(ids) == 0:
            return
        gamma = (self.dim + 8) * U * 1.01
        if self.sq is not None and metric == "l2":
            scale, bias = self.sq
            lo, hi = (-128, 127) if self.rows.dtype == np.int8 else (0, 255)
            v = self.q[i].astype(np.float32)
            t = ((v - bias) / scale).astype(np.float64)                    # fp32 subtract and divide, as compress does
            qc = np.clip(np.sign(t) * np.floor(np.abs(t) + 0.5), lo, hi)   # roundf: half away from zero
            l2 = ((self.rows[ids].astype(np.int64) - qc.astype(np.int64)) ** 2).sum(1)
            want = np.float32(scale * scale) * l2.astype(np.float32)
            assert np.array_equal(bits(d32.astype(np.float32)), bits(want)), f"{tag}: SQ L2 is not scale^2 * int L2"
            return
        if self.sq is not None and metric == "ip":
            scale, bias = (float(s) for s in self.sq)
            q, c = self.q[i].astype(np.float64), self.rows[ids].astype(np.float64)
            d64 = (q * (scale * c + bias)).sum(1)
            terms = (np.abs(q) * (np.abs(scale * c) + abs(bias))).sum(1)
            err = np.abs(d32 - d64)
            assert np.all(err <= gamma * terms), f"{tag}: SQ MIP off float64 by {np.max(err / np.maximum(terms, 1e-300))}"
            return
        q, y = self._operands(i, ids)
        if self.lvq is not None and metric == "l2":
            q = (self.q[i].astype(np.float32) - self.mean).astype(np.float64)   # fl32(q - mean), once per query
        if metric == "l2":
            t = (q[None, :] - y) ** 2
            d64, terms = t.sum(1), t.sum(1)
            bound = gamma * terms
        elif metric == "ip":
            t = q[None, :] * y
            d64, terms = t.sum(1), np.abs(t).sum(1)
            if self.lvq is not None:
                m = q * self.mean.astype(np.float64)
                d64, terms = d64 + m.sum(), terms + np.abs(m).sum()
            bound = gamma * terms
        else:
            t = q[None, :] * y
            norms = np.sqrt((y * y).sum(1)) * np.sqrt((q * q).sum())
            d64 = t.sum(1) / norms
            bound = gamma * (np.abs(t).sum(1) / norms + 2 * np.abs(d64))
        err = np.abs(d32 - d64)
        bad = ~(err <= bound)
        assert not np.any(bad), f"{tag}: off float64 by {err[bad][:4]} > {bound[bad][:4]}"


def expected_topk(kind, oracle, metric, k):
    """Oracle distances ordered by (key, id), padded with all-ones ids and +-inf past n."""
    nq, n = kind.q.shape[0], kind.rows.shape[0]
    ids = np.full((nq, k), ALL_ONES, dtype=np.uint64)
    dists = np.full((nq, k), np.inf if metric == "l2" else -np.inf, dtype=np.float32)
    for i in range(nq):
        d = kind.oracle_distances(oracle, metric, i)
        order = np.lexsort((np.arange(n), d if metric == "l2" else -d))[:k]
        ids[i, :len(order)] = order
        dists[i, :len(order)] = d[order]
    return ids, dists


def exhaustive(index, q, k):
    import torch
    nq = q.shape[0]
    dq = torch.from_numpy(np.ascontiguousarray(q)).cuda()
    ids = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    dists = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    index.exhaustive_device(dq.data_ptr(), q.dtype, nq, k, ids.data_ptr(), dists.data_ptr(),
                            stream=torch.cuda.current_stream().cuda_stream or 1)
    torch.cuda.synchronize()
    return ids.cpu().numpy().view(np.uint64), dists.cpu().numpy()


def check_exhaustive(kind, oracle, metric, k, tag, no_split=False):
    graph = np.zeros((kind.rows.shape[0], 2), dtype=np.uint32)
    index = kind.index(graph, 0, metric)
    if no_split:
        index.set_option("no_split", 1)
    got = exhaustive(index, kind.q, k)
    want = expected_topk(kind, oracle, metric, k)
    assert_same(got, *want, tag)
    for i in range(kind.q.shape[0]):
        kind.check_float64(metric, i, got[0][i], got[1][i], f"{tag} q{i}")


# ------------------------------------------------------------------------------------------------------------------
# a + b. The exhaustive scan over every row kind, every metric, every dimension class
# ------------------------------------------------------------------------------------------------------------------
DIM_CLASSES = [(1, False), (3, False), (17, False), (96, False), (128, False), (223, False), (256, False),
               (300, False), (768, False), (300, True)]   # (dim, no_split)
K_CYCLE = (12, 100, 1, 1024)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("dim,no_split", DIM_CLASSES)
def test_exhaustive_scan_every_row_kind(oracle, kind, dim, no_split):
    """Ids and distance bits equal the oracle's top k by (distance, id), and every distance is within its rounding
    bound of float64.  Half the cases use coarse-grid data (exact ties); k and nq rotate over the cases."""
    case = KINDS.index(kind) * len(DIM_CLASSES) + DIM_CLASSES.index((dim, no_split))
    k, nq = K_CYCLE[case % 4], (1 if case % 3 == 0 else 40)
    rng = np.random.default_rng(1000 + case)
    kd = Kind(kind, 1500, dim, nq, rng, coarse=(case // 4) % 2 == 0, oracle=oracle)
    for metric in kind_metrics(kind):
        check_exhaustive(kd, oracle, metric, k, f"{kind} d{dim} {metric} k{k} nq{nq} no_split{int(no_split)}",
                         no_split)


@pytest.mark.parametrize("kind", ["f32_f32", "f16_f16", "i8_i8", "u8_u8", "sq_i8_f32", "sq_u8_f16", "lvq8_f32"])
def test_exhaustive_scan_pads_when_n_is_below_k(oracle, kind):
    """n = 50 < k = 100: the first 50 entries are the whole dataset in (distance, id) order, the rest all-ones ids
    with +inf (L2) / -inf (MIP, cosine)."""
    rng = np.random.default_rng(7)
    kd = Kind(kind, 50, 20, 5, rng, coarse=True, oracle=oracle)
    for metric in kind_metrics(kind):
        check_exhaustive(kd, oracle, metric, 100, f"{kind} {metric} n50 k100")


@pytest.mark.parametrize("kind", ["f32_f32", "sq_i8_f32"])
def test_exhaustive_scan_unsplit_batch(oracle, kind):
    """A batch of 32 x SM count queries fills the GPU on its own, so the scan runs without cutting the rows into
    ranges (no merge launch) -- and still gives the oracle's top k."""
    import torch
    nq = 32 * torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.default_rng(17)
    kd = Kind(kind, 2000, 40, nq, rng, coarse=True, oracle=oracle)
    graph = np.zeros((2000, 2), dtype=np.uint32)
    for metric in ("l2", "ip"):
        index = kd.index(graph, 0, metric)
        small = kd.q[:40]
        exhaustive(index, small, 12)                      # warm: scratch, module loads
        l0 = launches()
        exhaustive(index, small, 12)
        split_launches = launches() - l0
        l0 = launches()
        got = exhaustive(index, kd.q, 12)
        assert launches() - l0 == split_launches - 1, "a full batch still cut the rows into ranges"
        assert_same(got, *expected_topk(kd, oracle, metric, 12), f"{kind} {metric} nq{nq}")


# ------------------------------------------------------------------------------------------------------------------
# c. The knobs that never change results
# ------------------------------------------------------------------------------------------------------------------
_EXPECTED = {}


def _knob_set(name, dataset):
    """(data, queries, graph, entry point, metric) of the three knob datasets: the reference's test dataset (L2) and
    2000 x 300 float32 (MIP) / float16 (cosine) rows with a degree-32 kNN graph."""
    if name == "ref":
        return dataset.data, dataset.queries, dataset.graph, dataset.entry_point, "l2"
    rng = np.random.default_rng(300)
    x = rng.standard_normal((2000, 300)).astype(np.float32)
    q = rng.standard_normal((1000, 300)).astype(np.float32)
    graph = knn_graph(x, 32, rng)
    if name == "d300_f16":
        return x.astype(np.float16), q.astype(np.float16), graph, 5, "cosine"
    return x, q, graph, 5, "ip"


def _expected(oracle, dataset, name, window, capacity, k):
    key = (name, window, capacity, k)
    if key not in _EXPECTED:
        x, q, graph, ep, metric = _knob_set(name, dataset)
        _EXPECTED[key] = oracle.index(x, graph, ep, metric).search(q, k, window, capacity)
    return _EXPECTED[key]


def _knob_index(dataset, name):
    x, q, graph, ep, metric = _knob_set(name, dataset)
    return make_index(x, graph, ep, metric), q


def _check_knob(index, q, oracle, dataset, name, options, lean, tag):
    for opt, val in options.items():
        index.set_option(opt, val)
    for window, capacity, k in WINDOWS:
        wi, wd = _expected(oracle, dataset, name, window, capacity, k)
        got = search(index, q, k, window, capacity)
        assert_same(got, wi, wd, f"{name} {tag} w{window} c{capacity}")
        if lean is not None:
            assert index.get_option("last_kernel") == int(lean), f"{name} {tag}: wrong kernel"


KNOB_SETS = ["ref", "d300_f32", "d300_f16"]


@pytest.mark.parametrize("name", KNOB_SETS)
def test_rows_in_flight_and_warps_per_cta(oracle, dataset, name):
    """The generic kernel with one or two rows per pass (and one row with unsplit wide rows), and 1, 3 or 8 queries
    per CTA."""
    index, q = _knob_index(dataset, name)
    for rows in (1, 2):
        _check_knob(index, q, oracle, dataset, name, {"generic_kernel": 1, "rows_in_flight": rows}, False,
                    f"rows_in_flight {rows}")
    if name != "ref":
        _check_knob(index, q, oracle, dataset, name, {"no_split": 1, "rows_in_flight": 1}, False,
                    "rows_in_flight 1 no_split")
        index.set_option("no_split", 0)
    index.set_option("rows_in_flight", 0)
    for warps in (1, 3, 8):
        _check_knob(index, q, oracle, dataset, name, {"generic_kernel": 1, "warps_per_cta": warps}, False,
                    f"warps_per_cta {warps}")


@pytest.mark.parametrize("name", KNOB_SETS)
def test_ctas_per_sm_and_filter_tag16(oracle, dataset, name):
    """One or 32 CTAs per SM on both kernels; direct-mapped 32-bit filter entries on the generic kernel."""
    index, q = _knob_index(dataset, name)
    for generic in (0, 1):
        for ctas in (1, 32):
            _check_knob(index, q, oracle, dataset, name, {"generic_kernel": generic, "ctas_per_sm": ctas}, not generic,
                        f"generic {generic} ctas_per_sm {ctas}")
    index.set_option("ctas_per_sm", 0)
    _check_knob(index, q, oracle, dataset, name, {"generic_kernel": 0, "filter_tag16": 0}, False, "filter_tag16 0")


@pytest.mark.parametrize("name", KNOB_SETS)
def test_host_chunks(oracle, dataset, name):
    """A host batch cut into 1, 2 or 16 pieces gives the same rows, for batches of 1, 3, 17 and 5000 queries."""
    index, q = _knob_index(dataset, name)
    for chunks in (1, 2, 16):
        index.set_option("host_chunks", chunks)
        for window, capacity, k in WINDOWS:
            wi, wd = _expected(oracle, dataset, name, window, capacity, k)
            for nq in (1, 3, 17, 5000):
                reps = (nq + len(q) - 1) // len(q)
                qq = np.concatenate([q] * reps)[:nq]
                got = search(index, qq, k, window, capacity)
                assert_same(got, np.concatenate([wi] * reps)[:nq], np.concatenate([wd] * reps)[:nq],
                            f"{name} host_chunks {chunks} nq{nq} w{window}")


# ------------------------------------------------------------------------------------------------------------------
# d. The visited filter at its exactness boundary
# ------------------------------------------------------------------------------------------------------------------
def _band_graph(n, rng, band=12, extra=8):
    """Degree 32: the 2 x band nearest ids (random ids where the band leaves [0, n)) plus `extra` random long edges."""
    offs = np.concatenate([np.arange(-band, 0), np.arange(1, band + 1)])
    nb = np.arange(n, dtype=np.int64)[:, None] + offs[None, :]
    rnd = rng.integers(0, n, (n, 2 * band + extra))
    rnd = np.where(rnd == np.arange(n)[:, None], (rnd + n // 2) % n, rnd)
    nb = np.where((nb < 0) | (nb >= n), rnd[:, :2 * band], nb)
    graph = np.empty((n, 2 * band + extra + 1), dtype=np.uint32)
    graph[:, 0] = 2 * band + extra
    graph[:, 1:] = np.concatenate([nb, rnd[:, 2 * band:]], axis=1)
    return graph


def _boundary_case(n, seed):
    """dim 8 rows increasing with the id, queries among the top ids, entry points near the top: every result row holds
    the eight highest ids, the ones whose filter tag would reach the 0xFFFF "empty" mark without the host's rule.  The
    top id's only in-edge is the first neighbour of the entry point expanded first (n - 20), so the filter is asked about
    it once, while its set still holds the empty marks: a tag equal to the mark would hide it for good (met again later,
    after its set had filled up, it would pass)."""
    rng = np.random.default_rng(seed)
    x = (rng.random((n, 8)) * 0.01).astype(np.float32)
    x[:, 0] = np.arange(n, dtype=np.float32) * np.float32(2.0 ** -4)
    q = (rng.random((64, 8)) * 0.01).astype(np.float32)
    q[:, 0] = (n - 1 - rng.random(64) * 6).astype(np.float32) * np.float32(2.0 ** -4)
    graph = _band_graph(n, rng)
    adj = graph[:, 1:]
    rows, cols = np.nonzero(adj == n - 1)
    adj[rows, cols] = np.where(rows == 0, 1, 0)
    adj[n - 20, 0] = n - 1
    return x, q, graph, [n - 40, n - 30, n - 20]


@pytest.mark.parametrize("generic,slots,n", [(False, 64, 524280), (False, 64, 524281),
                                             (True, 8, 262140), (True, 8, 262141)])
def test_visited_filter_boundary(oracle, generic, slots, n):
    x, q, graph, eps = _boundary_case(n, n)
    index = make_index(x, graph, eps[0], "l2")
    index.set_entry_points(eps)
    want = oracle.index(x, graph, eps[0], "l2")
    want.set_entry_points(eps)
    index.set_option("generic_kernel", int(generic))
    for window, capacity in ((16, 16), (40, 64)):
        wi, wd = want.search(q, 16, window, capacity)
        assert all(np.isin(np.arange(n - 8, n), row).all() for row in wi), "every row must hold the top eight ids"
        for filt in (slots, 0):
            index.set_option("visited_filter_slots", filt)
            got = search(index, q, 16, window, capacity)
            assert index.get_option("last_kernel") == int(filt != 0 and not generic)
            assert_same(got, wi, wd, f"n{n} slots {filt} generic {int(generic)} w{window}")


# ------------------------------------------------------------------------------------------------------------------
# e (+ c's no_split). Integer, SQ and LVQ-8 rows at wide and ragged dimensions, on both kernels
# ------------------------------------------------------------------------------------------------------------------
COMPRESSED_KINDS = ["f32_i8", "i8_i8", "f32_u8", "u8_u8", "sq_i8_f32", "sq_i8_f16", "sq_u8_f32", "sq_u8_f16",
                    "lvq8_f32", "lvq8_f16"]
GRAPH_CASES = ([(kind, dim) for kind in COMPRESSED_KINDS for dim in (17, 100, 300, 768)] +
               [(kind, dim) for kind in ("f32_f32", "f16_f16", "f16_f32") for dim in (256, 300, 768)] +
               [(kind, 256) for kind in ("sq_u8_f32", "lvq8_f32")])


@pytest.mark.parametrize("kind,dim", GRAPH_CASES)
def test_graph_search_wide_and_ragged(oracle, kind, dim):
    """Graph search vs the oracle on the lean and the generic kernel, and with no_split at dim >= 256 (wide float rows
    -- plain, SQ MIP / cosine, LVQ-8 -- kept on the narrow mapping instead of float_rows_split)."""
    rng = np.random.default_rng(dim * 31 + KINDS.index(kind))
    kd = Kind(kind, 1200, dim, 100, rng, coarse=dim % 2 == 0, oracle=oracle)
    graph = knn_graph(kd.x.astype(np.float32), 24, rng)
    for metric in kind_metrics(kind):
        index = kd.index(graph, 3, metric)
        want = kd.oracle_index(oracle, graph, 3, metric)
        for no_split in ((0, 1) if dim >= 256 else (0,)):
            index.set_option("no_split", no_split)
            for generic in (0, 1):
                index.set_option("generic_kernel", generic)
                for window, capacity, k in WINDOWS[:2]:
                    got = search(index, kd.q, k, window, capacity)
                    assert index.get_option("last_kernel") == 1 - generic
                    assert_same(got, *want.search(kd.q, k, window, capacity),
                                f"{kind} d{dim} {metric} no_split{no_split} generic{generic} w{window}")


# ------------------------------------------------------------------------------------------------------------------
# 3. The LVQ-8 encoder against float64, and at float16's range edges
# ------------------------------------------------------------------------------------------------------------------
H_MAX = 65504.0          # largest finite float16
H_INF_AT = 65520.0       # float16 rounds to +inf from here (round to nearest even)


def check_lvq8_encoding(x, mean, rows, tag):
    """Per element: the code is the nearest point of the row's stored grid {fp32(delta16 c + lower16)} (the
    neighbouring code only where (r - lower16) / delta16 is within fp32 rounding of a midpoint), and the decode is
    within 0.5 delta16 + |lower - lower16| + 255 |delta - delta16| + 2 ulp of the residual.  Padding bytes are 0."""
    n, dim = x.shape
    off = (dim + 3) // 4 * 4
    r = (x.astype(np.float32) - mean.astype(np.float32)).astype(np.float64)
    d16 = rows[:, off:off + 2].copy().view(np.float16)[:, 0].astype(np.float64)
    l16 = rows[:, off + 2:off + 4].copy().view(np.float16)[:, 0].astype(np.float64)
    codes = rows[:, :dim].astype(np.int64)
    with np.errstate(invalid="ignore"):     # inf * 0 is the NaN this looks for
        dec = (d16[:, None] * codes + l16[:, None]).astype(np.float32).astype(np.float64)
    assert np.all(np.isfinite(dec)), f"{tag}: rows decode to {np.unique(dec[~np.isfinite(dec)])}"
    assert np.all(rows[:, dim:off] == 0) and np.all(rows[:, off + 4:] == 0), f"{tag}: padding bytes are not 0"
    lo, hi = r.min(1), r.max(1)
    delta = (hi - lo) / 255
    mag = np.abs(r) + np.abs(l16)[:, None] + 255 * d16[:, None]
    ulp2 = 2 * np.spacing(mag.astype(np.float32)).astype(np.float64)
    bound = (0.5 * d16 + np.abs(lo - l16) + 255 * np.abs(delta - d16))[:, None] + ulp2
    err = np.abs(dec - r)
    bad = ~(err <= bound)
    assert not np.any(bad), f"{tag}: decode error {err[bad][:4]} above {bound[bad][:4]} for residuals {r[bad][:4]}"
    zero = d16 == 0
    assert np.all(codes[zero] == 0), f"{tag}: codes of a zero delta16 must be 0"
    if np.any(~zero):
        rr, cc, dd, ll = r[~zero], codes[~zero], d16[~zero, None], l16[~zero, None]
        grid = (dd[:, :, None] * np.arange(256)[None, None, :] + ll[:, :, None]).astype(np.float32).astype(np.float64)
        best = np.argmin(np.abs(grid - rr[:, :, None]), axis=2)
        t = (rr - ll) / dd
        near_mid = np.abs(t - np.floor(t) - 0.5) <= 8 * U * (np.abs(t) + (np.abs(rr) + np.abs(ll)) / dd)
        ok = (cc == best) | ((np.abs(cc - best) == 1) & near_mid)
        assert np.all(ok), f"{tag}: codes {cc[~ok][:4]} are not the nearest grid points {best[~ok][:4]}"


def _encode(fn):
    try:
        return fn(), None
    except Exception as e:     # the GPU raises Svsb200Error, the oracle RuntimeError
        return None, e


def _row(dim, lo, hi, rng):
    """A row of `dim` residuals spanning exactly [lo, hi] (float32), the others in between."""
    v = lo + (hi - lo) * rng.random(dim)
    v[0], v[-1] = lo, hi
    return v.astype(np.float32)


def _lvq8_cases(rng):
    """(tag, x, mean, first refused row or None)."""
    z = lambda d: np.zeros(d, np.float32)  # noqa: E731
    cases = []
    x = np.full((3, 17), 3.25, np.float32)
    cases.append(("constant rows", x, z(17), None))
    cases.append(("rows equal to the mean", x, x[0].copy(), None))
    for tag, rng_hi in (("range just below 255 x 65504", 255 * H_MAX * (1 - 2.0 ** -12)),
                        ("range just above 255 x 65504 (delta16 = 65504)", 255 * H_MAX * (1 + 2.0 ** -13))):
        cases.append((tag, np.stack([_row(40, 0.0, rng_hi, rng), _row(40, -60000.0, rng_hi - 60000.0, rng)]), z(40), None))
    cases.append(("lower just inside -65504", np.stack([_row(24, -H_MAX + 0.5, -H_MAX + 900, rng)]), z(24), None))
    cases.append(("lower just outside -65504 (lower16 = -65504)", np.stack([_row(24, -65510.0, -60000.0, rng)]), z(24),
                  None))
    cases.append(("rows on one side of the mean", np.stack([_row(33, 2.0, 9.0, rng), _row(33, -9.0, -2.0, rng)]),
                  z(33), None))
    cases.append(("delta in float16 subnormals", np.stack([_row(20, 0.0, 255 * 3e-6, rng),
                                                          _row(20, 1.0, 1.0 + 255 * 2.0 ** -20, rng)]), z(20), None))
    cases.append(("delta16 = 0", np.stack([_row(20, 0.0, 255 * 1e-8, rng)]), z(20), None))
    for d in (1, 3, 5):
        cases.append((f"dim {d}", (rng.standard_normal((6, d)) * 2).astype(np.float32), z(d), None))
    ok = (rng.standard_normal((4, 12))).astype(np.float32)
    for tag, bad in (("range at 255 x 65520", lambda v: v.__setitem__(slice(None), _row(12, 0.0, 255 * H_INF_AT, rng))),
                     ("range above 255 x 65520", lambda v: v.__setitem__(slice(None), _row(12, -1e7, 255 * H_INF_AT, rng))),
                     ("lower at -65520", lambda v: v.__setitem__(slice(None), _row(12, -H_INF_AT, 0.0, rng))),
                     ("lower below -65520", lambda v: v.__setitem__(slice(None), _row(12, -7e4, 0.0, rng))),
                     ("NaN element", lambda v: v.__setitem__(4, np.nan)),
                     ("+inf element", lambda v: v.__setitem__(4, np.inf)),
                     ("-inf element", lambda v: v.__setitem__(0, -np.inf))):
        x = ok.copy()
        bad(x[2])
        bad(x[3])
        cases.append((tag, x, z(12), 2))
    return cases


def test_lvq8_encoder_against_float64(oracle):
    """The GPU encoder and the oracle write the same bytes, within the float64 bound; rows whose residuals or float16
    constants are not finite are refused by both, naming the first such row."""
    from scalablevectorsearch_b200 import lvq8_compress
    rng = np.random.default_rng(12)
    for tag, x, mean, refused in _lvq8_cases(rng):
        for who, fn in (("gpu", lambda: lvq8_compress(x, mean)[0]), ("oracle", lambda: oracle.lvq8_compress(x, mean))):
            rows, err = _encode(fn)
            if err is None:
                check_lvq8_encoding(x, mean, rows, f"{who} {tag}")
            assert (err is None) == (refused is None), f"{who} {tag}: {err!r}"
            if refused is not None:
                assert f"row {refused} " in str(err), f"{who} {tag}: {err}"
        if refused is None:
            assert np.array_equal(lvq8_compress(x, mean)[0], oracle.lvq8_compress(x, mean)), f"{tag}: bytes differ"
