"""The GPU graph builder on int8 and uint8 rows, held to the same bar as on float32 / float16
(tests/test_gpu_build_exact.py, tests/test_gpu_build.py).

The reference builds SimpleData<int8_t / uint8_t> with the datum itself as the query (index/vamana/extensions.h), so
every distance of the build is int x int: exact int32 sums for L2 and inner product, and for cosine the integer sum
over a_norm * sqrt(float(|y|^2)), where a_norm is distance::norm's sequential fp32 sum.  So the bar is:
  * static builds of n <= 40 (one node per round): every row, in order, and the entry point equal the reference's,
    including data drawn from a narrow range (exact distance ties everywhere), dimensions that are not a multiple of 16
    and uint8 rows whose sum x*x passes 2^24, where the order of the norm's fp32 sum changes its value;
  * on integer data whose sums stay below 2^24 the integer build equals the float32 build of the same values;
  * whole builds: recall equivalence with the reference's builder."""
import numpy as np
import pytest

from conftest import recall_at_k

METRIC = {"l2": 0, "ip": 1, "cosine": 2}
PREMISE_THREADS = (1, 8)

# id, metric, dtype, n, dim, (lo, hi) value range, R, window, max_candidate_pool_size, prune_to, alpha
STATIC = [
    ("l2-i8", "l2", np.int8, 40, 20, (-127, 127), 6, 12, 0, 0, None),
    ("ip-i8", "ip", np.int8, 40, 20, (-127, 127), 6, 12, 0, 0, None),
    ("cosine-i8", "cosine", np.int8, 40, 20, (-127, 127), 6, 12, 0, 0, None),
    ("l2-u8", "l2", np.uint8, 40, 20, (0, 255), 8, 16, 0, 0, None),
    ("ip-u8", "ip", np.uint8, 37, 20, (0, 255), 8, 16, 0, 0, None),
    ("cosine-u8", "cosine", np.uint8, 40, 20, (0, 255), 8, 16, 0, 0, None),
    ("l2-i8-ties", "l2", np.int8, 40, 20, (-3, 3), 8, 16, 0, 0, None),
    ("ip-i8-ties", "ip", np.int8, 40, 20, (-3, 3), 6, 12, 0, 0, None),
    ("cosine-i8-ties", "cosine", np.int8, 40, 20, (-3, 3), 6, 12, 0, 0, None),
    ("l2-u8-ties", "l2", np.uint8, 40, 20, (0, 3), 7, 12, 0, 0, None),
    ("cosine-u8-ties", "cosine", np.uint8, 40, 20, (1, 3), 8, 16, 0, 0, None),
    ("l2-i8-dim100-prune_to", "l2", np.int8, 40, 100, (-127, 127), 8, 16, 0, 5, None),
    ("ip-u8-dim100-prune_to", "ip", np.uint8, 40, 100, (0, 255), 8, 16, 0, 6, None),
    ("l2-u8-small-pool", "l2", np.uint8, 40, 20, (0, 255), 8, 16, 10, 0, None),
    ("cosine-i8-small-pool-prune_to", "cosine", np.int8, 40, 20, (-127, 127), 4, 12, 6, 3, None),
    ("l2-i8-alpha", "l2", np.int8, 40, 20, (-127, 127), 6, 12, 0, 0, 1.5),
    ("ip-u8-alpha", "ip", np.uint8, 33, 20, (0, 255), 7, 12, 0, 0, 0.85),
    ("cosine-i8-ties-alpha", "cosine", np.int8, 40, 20, (-3, 3), 6, 12, 0, 0, 0.9),
    # sum x*x > 2^24 in every row: the norm's sequential fp32 sum rounds
    ("cosine-u8-dim300", "cosine", np.uint8, 40, 300, (232, 255), 8, 16, 0, 0, None),
    ("l2-u8-dim300", "l2", np.uint8, 40, 300, (232, 255), 8, 16, 0, 0, None),
]
STATIC_IDS = [s[0] for s in STATIC]
# sums below 2^24: the float32 builder computes the same distances exactly
BELOW_2_24 = [s for s in STATIC if s[4] * max(abs(s[5][0]), abs(s[5][1])) ** 2 < 1 << 24]


def static_data(case):
    _, _, dtype, n, dim, (lo, hi), R, *_ = case
    return np.random.default_rng(n * 7 + R + dim).integers(lo, hi + 1, (n, dim)).astype(dtype)


def parameters(case):
    from scalablevectorsearch_b200 import VamanaBuildParameters
    *_, R, window, mc, prune_to, alpha = case
    return VamanaBuildParameters(alpha=alpha or 0.0, graph_max_degree=R, window_size=window,
                                 max_candidate_pool_size=mc, prune_to=prune_to)


def static_gpu(case, data=None):
    from scalablevectorsearch_b200 import DistanceType, build_graph
    return build_graph(static_data(case) if data is None else data, DistanceType(METRIC[case[1]]), parameters(case))


def static_ref(refint, case, threads):
    _, metric, *_, R, window, mc, prune_to, alpha = case
    return refint.build(static_data(case), metric, R, window, alpha, mc or None, prune_to or None, threads=threads)


def rows(graph):
    return [tuple(r[1:1 + r[0]].tolist()) for r in graph]


def first_difference(got, want):
    for v, (a, b) in enumerate(zip(got, want)):
        if a != b:
            return v, a, b
    return None


def ref_threads():
    from oracle.bindings import effective_cpus
    return min(8, effective_cpus())


@pytest.fixture(scope="module")
def refint(reflib):
    """The reference's builder over int8 / uint8 rows (oracle/_ref/libsvsref_int.so)."""
    from oracle.build_int import RefIntBuildLib
    if not RefIntBuildLib.available():
        pytest.skip("oracle/_ref/libsvsref_int.so not built (needs /root/reference)")
    return RefIntBuildLib()


@pytest.fixture(scope="module")
def vnni(reflib, refint):
    """The reference computes int x int distances exactly only on its AVX-512 VNNI path; without it, it falls back
    to the float tree."""
    if not reflib.avx512vnni():
        pytest.skip("host lacks AVX-512 VNNI: the reference would take its float fallback for integer rows")
    return refint


# ---------------------------------------------------------------- CPU

@pytest.mark.parametrize("case", STATIC, ids=STATIC_IDS)
def test_premise_reference_static_int_build_is_deterministic(vnni, case):
    (g1, ep1), (g8, ep8) = (static_ref(vnni, case, t) for t in PREMISE_THREADS)
    diff = first_difference(rows(g8), rows(g1))
    assert ep1 == ep8 and diff is None, f"premise broken for static fixture {case[0]}: {diff}"


def test_dim300_fixtures_need_the_sequential_norm():
    """The dim-300 uint8 rows pass 2^24 in sum x*x, and for some of them distance::norm's sequential fp32 sum differs
    from float(sum x*x): the fixture tells the two orders apart."""
    for case in STATIC:
        if case[4] != 300:
            continue
        x = static_data(case).astype(np.int64)
        exact = (x * x).sum(1)
        assert exact.min() > 1 << 24, case[0]
        sequential = np.cumsum((x * x).astype(np.float32), axis=1, dtype=np.float32)[:, -1]
        assert (sequential != exact.astype(np.float32)).any(), case[0]


def test_integer_sums_of_the_equivalence_fixtures_stay_below_2_24():
    for case in BELOW_2_24:
        x = static_data(case).astype(np.int64)
        assert (x * x).sum(1).max() < 1 << 24, case[0]


def test_dynamic_index_refuses_integer_data():
    """The dynamic index stays float32 / float16: its consolidation orders equal distances by id where the reference
    leaves them unspecified, and integer distances tie constantly."""
    import ctypes as C

    from scalablevectorsearch_b200 import DistanceType, DynamicVamana, Svsb200Error, VamanaBuildParameters, _lib
    data = np.zeros((64, 16), dtype=np.int8)
    with pytest.raises(TypeError):
        DynamicVamana.build(VamanaBuildParameters(graph_max_degree=8, window_size=16), data)
    with pytest.raises(TypeError):
        DynamicVamana.from_arrays(data, np.zeros((64, 9), dtype=np.uint32), 0)
    lib = _lib.lib()
    for dtype in (np.int8, np.uint8):
        x = data.astype(dtype)
        handle = C.c_void_p()
        with pytest.raises(Svsb200Error, match="float32 / float16"):
            _lib.check(lib.svsb200_dynamic_build(x.ctypes.data, 2 if dtype == np.int8 else 3, 64, 16,
                                                 int(DistanceType.L2), 0.0, 8, 16, 0, 0, None, 0, C.byref(handle)))


@pytest.mark.parametrize("dtype", [np.int8, np.uint8])
def test_int_build_refuses_a_candidate_pool_above_512(dtype):
    from scalablevectorsearch_b200 import DistanceType, Svsb200Error, VamanaBuildParameters, build_graph
    data = np.random.default_rng(0).integers(0, 100, (64, 20)).astype(dtype)
    with pytest.raises(Svsb200Error, match="512"):
        build_graph(data, DistanceType.L2, VamanaBuildParameters(graph_max_degree=8, window_size=16,
                                                                  max_candidate_pool_size=513))


# ---------------------------------------------------------------- GPU

@pytest.mark.gpu
@pytest.mark.parametrize("case", STATIC, ids=STATIC_IDS)
def test_static_int_build_matches_the_reference_rows(vnni, case):
    g_graph, g_ep = static_gpu(case)
    r_graph, r_ep = static_ref(vnni, case, ref_threads())
    assert g_ep == r_ep, (g_ep, r_ep)
    diff = first_difference(rows(g_graph), rows(r_graph))
    assert diff is None, f"{case[0]}: first row that differs {diff[0]}: gpu {diff[1]} vs reference {diff[2]}"


@pytest.mark.gpu
@pytest.mark.parametrize("case", BELOW_2_24, ids=[s[0] for s in BELOW_2_24])
def test_int_build_equals_the_float32_build_of_the_same_values(case):
    g_int, ep_int = static_gpu(case)
    g_f32, ep_f32 = static_gpu(case, static_data(case).astype(np.float32))
    assert ep_int == ep_f32
    diff = first_difference(rows(g_int), rows(g_f32))
    assert diff is None, f"{case[0]}: first row that differs {diff[0]}: int {diff[1]} vs float32 {diff[2]}"


def _search(data, graph, ep, metric, queries, window):
    from scalablevectorsearch_b200 import DistanceType, SearchBufferConfig, Vamana
    index = Vamana.from_arrays(data, graph, ep, DistanceType(METRIC[metric]))
    index.search_parameters.buffer_config = SearchBufferConfig(window)
    return index.search(queries, 10)


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
def test_int8_build_on_reference_dataset_matches_reference_builder_recall(refint, metric):
    """The reference's 10k x 128 int8 test dataset in its native type, R = 32, window 64: the GPU graph against the
    reference builder's graph, both searched with int8 queries by the bit-exact search."""
    import os

    from conftest import GOLDEN
    from scalablevectorsearch_b200 import DistanceType, VamanaBuildParameters, build_graph
    z = np.load(os.path.join(GOLDEN, "test_dataset.npz"))
    X, Q, gt = z["data"], z["queries"], z[f"gt_{metric}"]
    assert X.dtype == np.int8 and Q.dtype == np.int8
    alpha = 1.2 if metric == "l2" else 0.95
    g_gpu, ep_gpu = build_graph(X, DistanceType(METRIC[metric]),
                                VamanaBuildParameters(alpha=alpha, graph_max_degree=32, window_size=64))
    g_ref, ep_ref = refint.build(X, metric, 32, 64, alpha=alpha, threads=ref_threads())
    assert ep_gpu == ep_ref, "medoid entry point differs from the reference's"
    for window in (10, 30):
        r_gpu = recall_at_k(_search(X, g_gpu, ep_gpu, metric, Q, window)[0], gt)
        r_ref = recall_at_k(_search(X, g_ref, ep_ref, metric, Q, window)[0], gt)
        assert r_gpu >= r_ref - 0.01, (metric, window, r_gpu, r_ref)
    d_gpu, d_ref = g_gpu[:, 0].mean(), g_ref[:, 0].mean()
    assert 0.8 * d_ref <= d_gpu <= 1.25 * d_ref, (d_gpu, d_ref)


def clustered_uint8(n, nq, dim):
    """The bench's clustered unit vectors, mapped affinely onto 0..255 (queries clipped to that range)."""
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    base, queries = clustered_unit_vectors(n, nq, dim)
    lo, hi = float(base.min()), float(base.max())

    def q8(x):
        return np.clip(np.rint((x - lo) * (255.0 / (hi - lo))), 0, 255).astype(np.uint8)
    return q8(base), q8(queries)


@pytest.mark.gpu
def test_uint8_build_and_search_end_to_end(refint, oracle):
    """Vamana.build on 30k x 96 clustered uint8 rows, then search with uint8 and float32 queries: recall@10 against
    brute force at least the reference builder's minus 0.01, and ids and distance bits equal to the C oracle's."""
    from scalablevectorsearch_b200 import DistanceType, SearchBufferConfig, Vamana, VamanaBuildParameters
    base, queries = clustered_uint8(30_000, 500, 96)
    index = Vamana.build(VamanaBuildParameters(graph_max_degree=64, window_size=128), base, DistanceType.L2)
    index.search_parameters.buffer_config = SearchBufferConfig(64)
    ids, _ = index.search(queries, 10)
    x, q = base.astype(np.int64), queries.astype(np.int64)
    d = (q * q).sum(1)[:, None] + (x * x).sum(1)[None, :] - 2 * q @ x.T
    gt = np.argsort(d, axis=1, kind="stable")[:, :10]
    g_ref, ep_ref = refint.build(base, "l2", 64, 128, alpha=1.2, threads=ref_threads())
    r_gpu = recall_at_k(ids, gt)
    r_ref = recall_at_k(_search(base, g_ref, ep_ref, "l2", queries, 64)[0], gt)
    assert r_gpu >= r_ref - 0.01 and r_gpu > 0.9, (r_gpu, r_ref)

    # the built graph, searched by the GPU and by the C oracle: same ids, same distance bits
    from scalablevectorsearch_b200 import build_graph
    graph, ep = build_graph(base, DistanceType.L2, VamanaBuildParameters(graph_max_degree=64, window_size=128))
    built = Vamana.from_arrays(base, graph, ep, DistanceType.L2)
    built.search_parameters.buffer_config = SearchBufferConfig(64)
    want = oracle.index(base, graph, ep, "l2")
    for qs in (queries[:200], queries[:200].astype(np.float32)):
        got_ids, got_d = built.search(qs, 10)
        want_ids, want_d = want.search(qs, 10, 64, 64)
        assert np.array_equal(got_ids.astype(np.uint64), want_ids), qs.dtype
        assert np.array_equal(got_d.view(np.uint32), want_d.view(np.uint32)), qs.dtype


@pytest.mark.gpu
def test_dynamic_add_refuses_integer_points():
    from scalablevectorsearch_b200 import DynamicVamana, Svsb200Error, VamanaBuildParameters
    data = np.random.default_rng(1).standard_normal((200, 16)).astype(np.float32)
    index = DynamicVamana.build(VamanaBuildParameters(graph_max_degree=8, window_size=16), data)
    for dtype in (np.int8, np.uint8):
        with pytest.raises(Svsb200Error, match="dtype"):
            index.add(np.ones((4, 16), dtype=dtype), np.arange(1000, 1004, dtype=np.uint64))
    assert index.size == 200
