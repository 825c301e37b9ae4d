"""The GPU graph builder held to the reference's adjacency rows wherever the reference itself is deterministic.

The reference's builder (index/vamana/vamana_build.h) works in rounds of several nodes, and inside a round its result
depends on thread timing: add_reverse_edges walks a node's row while the round's other nodes append to it.  A round of
one node is exact, and so is every fixture below, which the CPU premise test checks by running the reference with
1 and 8 threads:
  * static builds of n <= 40 (one node per round): every row, in order, and the entry point;
  * sequences of `add` calls of at most 40 points (one node per round) on the dynamic index: every slot's row, in
    order, its status and the entry point, after every call;
  * large adds into an existing graph (hundreds of nodes per round): the neighbour SET of every slot.  The order in
    which reverse edges are appended to a row that does not overflow is the order in which the round's nodes reach
    it, in the reference as on the GPU.
Whole static builds with many nodes per round stay on the recall bar (tests/test_gpu_build.py)."""
import numpy as np
import pytest

from conftest import knn_graph

METRIC = {"l2": 0, "ip": 1, "cosine": 2}
PREMISE_THREADS = (1, 8)


def gaussian(n, dim, dtype, seed):
    return np.random.default_rng(seed).standard_normal((n, dim)).astype(np.float32).astype(dtype)


def rows(graph):
    return [tuple(r[1:1 + r[0]].tolist()) for r in graph]


def first_difference(got, want, as_sets=False):
    """(slot, got row, wanted row) of the first slot whose rows differ, or None."""
    for v, (a, b) in enumerate(zip(got, want)):
        if (set(a) != set(b)) if as_sets else (a != b):
            return v, a, b
    if len(got) != len(want):
        return min(len(got), len(want)), "(missing)", "(missing)"
    return None


def ref_threads():
    from oracle.bindings import effective_cpus
    return min(8, effective_cpus())


# ---------------------------------------------------------------- static builds, one node per round

# id, metric, dtype, n, R, window, max_candidate_pool_size, prune_to, alpha (0 / None: the defaults)
STATIC = [
    ("l2-f32", "l2", np.float32, 40, 6, 12, 0, 0, None),
    ("ip-f32", "ip", np.float32, 40, 6, 12, 0, 0, None),
    ("cosine-f32", "cosine", np.float32, 40, 6, 12, 0, 0, None),
    ("l2-f16", "l2", np.float16, 40, 8, 16, 0, 0, None),
    ("ip-f16", "ip", np.float16, 37, 8, 16, 0, 0, None),
    ("cosine-f16", "cosine", np.float16, 40, 8, 16, 0, 0, None),
    ("l2-prune_to", "l2", np.float32, 40, 8, 16, 0, 5, None),
    ("ip-prune_to", "ip", np.float32, 40, 8, 16, 0, 6, None),
    ("l2-small-pool", "l2", np.float32, 40, 8, 16, 10, 0, None),
    ("cosine-small-pool-prune_to", "cosine", np.float16, 40, 4, 12, 6, 3, None),
    ("l2-alpha", "l2", np.float32, 40, 6, 12, 0, 0, 1.5),
    ("ip-alpha", "ip", np.float32, 33, 7, 12, 0, 0, 0.85),
]
STATIC_IDS = [s[0] for s in STATIC]


def static_data(case):
    _, _, dtype, n, *_ = case
    return gaussian(n, 20, dtype, seed=n * 7 + case[4])


def static_ref(reflib, case, threads):
    _, metric, _, _, R, window, mc, prune_to, alpha = case
    return reflib.build(static_data(case), metric, R, window, alpha, mc or None, prune_to or None, threads=threads)


def static_gpu(case):
    from scalablevectorsearch_b200 import DistanceType, VamanaBuildParameters, build_graph
    _, metric, _, _, R, window, mc, prune_to, alpha = case
    params = VamanaBuildParameters(alpha=alpha or 0.0, graph_max_degree=R, window_size=window,
                                   max_candidate_pool_size=mc, prune_to=prune_to)
    return build_graph(static_data(case), DistanceType(METRIC[metric]), params)


# ---------------------------------------------------------------- dynamic index: sequences of mutations

def medoid(x):
    x = x.astype(np.float64)
    return int(np.argmin(((x - x.mean(0)) ** 2).sum(1)))


def random_regular(n, R, seed):
    """Every row R distinct random neighbours: a poor graph, on which a search expands somewhat more nodes than its
    window."""
    rng = np.random.default_rng(seed)
    graph = np.zeros((n, R + 1), dtype=np.uint32)
    graph[:, 0] = R
    for v in range(n):
        nb = rng.choice(n - 1, R, replace=False)
        graph[v, 1:] = nb + (nb >= v)
    return graph


def chain(total, n0, dim, dtype, R, seed):
    """Rows spread along a line (plus a little noise) and a band graph over the first n0 of them in line order, each
    row linked to its R/2 predecessors and R/2 successors, entered at one end.  A search walks the band towards the
    query, and every node it expands on the way is later pushed out of the window by closer ones: it expands up to
    window + n0 / (R/2) nodes, far more than its window."""
    rng = np.random.default_rng(seed)
    direction = rng.standard_normal(dim)
    direction /= np.linalg.norm(direction)
    t = rng.uniform(0.0, 100.0, total)
    data = (t[:, None] * direction[None, :] + 0.05 * rng.standard_normal((total, dim))).astype(np.float32).astype(dtype)
    order = np.argsort(t[:n0], kind="stable")
    graph = np.zeros((n0, R + 1), dtype=np.uint32)
    for pos, v in enumerate(order):
        lo = max(0, min(pos - R // 2, n0 - 1 - R))
        nb = [int(u) for u in order[lo:lo + R + 1] if u != v][:R]
        graph[v, 0] = len(nb)
        graph[v, 1:1 + len(nb)] = nb
    return data, graph, int(order[0])


class Dyn:
    """One dynamic scenario: a base graph over the first n0 rows, then a list of mutations.
    ops: ("add", count, reuse_empty) takes the next `count` rows (external id = row); ("delete", count) deletes
    `count` random present ids; ("consolidate",)."""

    def __init__(self, name, metric, dtype, R, window, n0, ops, base="knn", dim=20, alpha=None, max_candidates=None,
                 prune_to=None, seed=0):
        self.name, self.metric, self.dtype, self.R, self.window, self.n0 = name, metric, dtype, R, window, n0
        self.ops, self.base, self.dim, self.seed = ops, base, dim, seed
        self.alpha, self.max_candidates, self.prune_to = alpha, max_candidates, prune_to
        total = n0 + sum(op[1] for op in ops if op[0] == "add")
        self.data = gaussian(total, dim, dtype, seed=1000 + seed)
        self.ep = medoid(self.data[:n0])
        if n0 == 1:
            self.graph = np.zeros((1, R + 1), dtype=np.uint32)
        elif base == "random":
            self.graph = random_regular(n0, R, seed)
        elif base == "chain":
            self.data, self.graph, self.ep = chain(total, n0, dim, dtype, R, seed)
        else:
            self.graph = knn_graph(self.data[:n0], R, np.random.default_rng(seed))

    def __repr__(self):
        return self.name

    def parameters(self):
        """(alpha, window, max_candidates, prune_to) as the GPU index resolves them (0 / None: its defaults)."""
        alpha = self.alpha if self.alpha is not None else (1.2 if self.metric == "l2" else 0.95)
        max_candidates = self.max_candidates or min(3 * self.window, 512)
        prune_to = self.prune_to or (self.R - 4 if self.R >= 16 else self.R)
        return np.float32(alpha), self.window, max_candidates, prune_to

    def run(self, index):
        """Drives `index` (GPU or reference: same methods) through the ops; yields (op, export) after each."""
        rng = np.random.default_rng(self.seed + 7)
        nxt = self.n0
        present = list(range(self.n0))
        for op in self.ops:
            if op[0] == "add":
                ids = np.arange(nxt, nxt + op[1], dtype=np.uint64)
                index.add(self.data[nxt:nxt + op[1]], ids, reuse_empty=op[2])
                present += ids.tolist()
                nxt += op[1]
            elif op[0] == "delete":
                gone = rng.choice(len(present), op[1], replace=False)
                index.delete(np.array([present[i] for i in gone], dtype=np.uint64))
                present = [p for i, p in enumerate(present) if i not in set(gone.tolist())]
            else:
                index.consolidate()
            yield op, index.export()

    def reference(self, refdyn, threads):
        alpha, window, mc, prune_to = self.parameters()
        return refdyn.dynamic(self.data[:self.n0], self.graph, self.ep, np.arange(self.n0, dtype=np.uint64),
                              self.metric, alpha, window, mc, prune_to, threads=threads)

    def gpu(self):
        from scalablevectorsearch_b200 import DistanceType, DynamicVamana
        index = DynamicVamana.from_arrays(self.data[:self.n0], self.graph, self.ep, np.arange(self.n0, dtype=np.uint64),
                                          DistanceType(METRIC[self.metric]))
        alpha, window, mc, prune_to = self.parameters()
        index.alpha, index.construction_window_size, index.max_candidates, index.prune_to = alpha, window, mc, prune_to
        assert (index.alpha, index.construction_window_size, index.max_candidates, index.prune_to) == \
            (alpha, window, mc, prune_to)
        return index


def compare(scenario, got_states, want_states, as_sets):
    """Status, entry point and every slot's row after every call; the first difference is reported."""
    for call, ((op, got), (_, want)) in enumerate(zip(got_states, want_states)):
        g_graph, g_status, _, g_ep = got
        r_graph, r_status, _, r_ep = want
        where = f"{scenario.name}: call {call} {op}"
        assert np.array_equal(g_status, r_status), f"{where}: status differs at slot " \
            f"{int(np.flatnonzero(g_status != r_status)[0]) if len(g_status) == len(r_status) else 'count'}"
        assert g_ep == r_ep, f"{where}: entry point {g_ep} != {r_ep}"
        diff = first_difference(rows(g_graph), rows(r_graph), as_sets)
        ndiff = sum((set(a) != set(b)) if as_sets else (a != b) for a, b in zip(rows(g_graph), rows(r_graph)))
        assert diff is None, f"{where}: {ndiff} slots differ; first slot {diff[0]}: gpu {diff[1]} vs reference {diff[2]}"


ONE_NODE_ROUNDS = [
    *[Dyn(f"{m}-{np.dtype(t).name}-R32", m, t, 32, 64, 1000, [("add", 40, False), ("add", 40, False), ("add", 25, False)],
          seed=i)
      for i, (m, t) in enumerate([(m, t) for m in ("l2", "ip", "cosine") for t in (np.float32, np.float16)])],
    Dyn("l2-f32-R128-window352", "l2", np.float32, 128, 352, 1000, [("add", 40, False), ("add", 33, False)], seed=10),
    Dyn("cosine-f16-R128-window352", "cosine", np.float16, 128, 352, 1000, [("add", 40, False)], seed=11),
    # poor base graphs: the inserts' searches expand more nodes than the window, up to several times as many on the
    # band graphs (test_poor_graph_fixtures_expand_past_the_history_room), and the whole search history is the pool
    Dyn("l2-f32-R128-window352-band-graph", "l2", np.float32, 128, 352, 12000, [("add", 40, False), ("add", 40, False)],
        base="chain", seed=12),
    Dyn("l2-f16-R32-window448-band-graph", "l2", np.float16, 32, 448, 12000, [("add", 40, False)], base="chain", seed=14),
    Dyn("ip-f32-R32-window64-random-graph", "ip", np.float32, 32, 64, 3000, [("add", 40, False)], base="random", seed=13),
    # Empty slots reused after delete + consolidate, then growth past the current capacity
    *[Dyn(f"{m}-{np.dtype(t).name}-reuse-and-grow", m, t, 32, 64, 1000,
          [("add", 40, False), ("delete", 60), ("consolidate",), ("add", 40, True), ("add", 40, True), ("add", 40, False)],
          seed=20 + i)
      for i, (m, t) in enumerate([("l2", np.float32), ("ip", np.float16), ("cosine", np.float32)])],
    # non-default mutation parameters
    Dyn("l2-f32-alpha-pool-prune_to", "l2", np.float32, 32, 48, 1000, [("add", 40, False), ("add", 40, False)],
        alpha=1.1, max_candidates=40, prune_to=24, seed=30),
    Dyn("cosine-f32-alpha-pool-prune_to", "cosine", np.float32, 32, 48, 1000, [("add", 40, False), ("add", 40, False)],
        alpha=0.9, max_candidates=50, prune_to=20, seed=31),
    Dyn("ip-f16-R8-pool-prune_to", "ip", np.float16, 8, 24, 500, [("add", 40, False), ("add", 40, False)],
        max_candidates=12, prune_to=6, seed=32),
]

LARGE_ROUNDS = [
    # 24 000 points into a 1-row index: 40 rounds of 600; in the first, every new node links to the entry point, which
    # receives 600 reverse edges at once
    Dyn("l2-f32-one-row-plus-24000", "l2", np.float32, 32, 64, 1, [("add", 24000, False)], seed=40),
    # a few thousand points into a built base: 40 rounds of 75 and 100
    Dyn("l2-f32-base2000-plus-3000", "l2", np.float32, 32, 64, 2000, [("add", 3000, False)], seed=41),
    Dyn("cosine-f16-base3000-plus-4000", "cosine", np.float16, 32, 64, 3000, [("add", 4000, False)], seed=42),
]


@pytest.fixture(scope="module")
def refdyn(reflib):
    from oracle.dynamic import RefDynamicLib
    if not RefDynamicLib.available():
        pytest.skip("oracle/_ref/libsvsref_dynamic.so not built (needs /root/reference)")
    return RefDynamicLib()


# ---------------------------------------------------------------- the premise (CPU, reference only)

@pytest.mark.parametrize("case", STATIC, ids=STATIC_IDS)
def test_premise_reference_static_build_is_deterministic(reflib, case):
    (g1, ep1), (g8, ep8) = (static_ref(reflib, case, t) for t in PREMISE_THREADS)
    diff = first_difference(rows(g8), rows(g1))
    assert ep1 == ep8 and diff is None, f"premise broken for static fixture {case[0]}: {diff}"


@pytest.mark.parametrize("scenario", ONE_NODE_ROUNDS + LARGE_ROUNDS, ids=repr)
def test_premise_reference_dynamic_is_deterministic(refdyn, scenario):
    as_sets = scenario in LARGE_ROUNDS
    runs = [list(scenario.run(scenario.reference(refdyn, t))) for t in PREMISE_THREADS]
    try:
        compare(scenario, runs[1], runs[0], as_sets)
    except AssertionError as e:
        raise AssertionError(f"premise broken for dynamic fixture {scenario.name} (1 vs 8 reference threads): {e}")


def test_poor_graph_fixtures_expand_past_the_history_room(oracle):
    """The band-graph fixtures do what they are there for: the first insert's searches (greedy search over the base
    graph, the C oracle's hop count) expand more nodes than 512 - R, the room a 512-entry pool leaves for the history
    next to the node's own row."""
    for s in ONE_NODE_ROUNDS:
        if s.base != "chain":
            continue
        index = oracle.index(s.data[:s.n0].astype(np.float32), s.graph, s.ep, s.metric)
        hops, _ = index.counts(s.data[s.n0:s.n0 + 40].astype(np.float32), s.window)
        assert hops.max() > 512 - s.R, (s.name, int(hops.max()))


# ---------------------------------------------------------------- the GPU against the reference

@pytest.mark.gpu
@pytest.mark.parametrize("case", STATIC, ids=STATIC_IDS)
def test_static_one_node_rounds_match_the_reference_rows(reflib, case):
    g_graph, g_ep = static_gpu(case)
    r_graph, r_ep = static_ref(reflib, case, ref_threads())
    assert g_ep == r_ep, (g_ep, r_ep)
    diff = first_difference(rows(g_graph), rows(r_graph))
    assert diff is None, f"{case[0]}: first row that differs {diff[0]}: gpu {diff[1]} vs reference {diff[2]}"


@pytest.mark.gpu
@pytest.mark.parametrize("scenario", ONE_NODE_ROUNDS, ids=repr)
def test_dynamic_one_node_rounds_match_the_reference_rows(refdyn, scenario):
    compare(scenario, scenario.run(scenario.gpu()), scenario.run(scenario.reference(refdyn, ref_threads())), False)


@pytest.mark.gpu
@pytest.mark.parametrize("scenario", LARGE_ROUNDS, ids=repr)
def test_dynamic_large_rounds_match_the_reference_neighbour_sets(refdyn, scenario):
    compare(scenario, scenario.run(scenario.gpu()), scenario.run(scenario.reference(refdyn, ref_threads())), True)


def test_static_build_refuses_a_candidate_pool_above_512():
    """The builder's candidate pool holds 512 entries: an explicit max_candidate_pool_size above that is refused, as
    the dynamic index refuses max_candidates > 512, instead of being clamped.  The check runs before any device work.
    (The default, 3 * window_size, is clamped to 512 on both paths.)"""
    from scalablevectorsearch_b200 import DistanceType, Svsb200Error, VamanaBuildParameters, build_graph
    data = gaussian(64, 20, np.float32, seed=0)
    with pytest.raises(Svsb200Error, match="512"):
        build_graph(data, DistanceType.L2, VamanaBuildParameters(graph_max_degree=8, window_size=16,
                                                                  max_candidate_pool_size=513))
