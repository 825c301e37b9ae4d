"""The GPU graph builder over SQ codes (svsb200_build_vamana_sq, Vamana.build(..., sq=)), held to the bar of the other
builds (tests/test_gpu_build_int.py), and the runtime VamanaIndex with SQI8 storage.

The reference builds SQDataset<int8_t / uint8_t> with each datum as its own query through DecompressionAdaptor
(tests/build_sq_fixtures.py restates that distance; tests/test_build_sq_model.py pins it to the reference).  So:
  * static builds of n <= 40 (one node per round): every row, in order, and the entry point equal the reference's,
    for int8 and uint8 codes and the three metrics, including narrow code ranges (ties), dimension 100 and a bias so
    large against the scale that the L2 round trip moves codes;
  * with a power-of-two scale and an exact round trip, the SQ L2 build is the int8 / uint8 build of the same codes;
  * whole builds on the reference's test dataset: recall equivalence with the reference's SQ builder;
  * a GPU-built SQ index, searched on the GPU, equals the C oracle's search over the same graph and codes."""
import os
import subprocess

import numpy as np
import pytest

import build_sq_fixtures as F
from conftest import GOLDEN, ROOT, recall_at_k

METRIC = F.METRIC


def parameters(case):
    from scalablevectorsearch_b200 import VamanaBuildParameters
    *_, R, window, mc, prune_to, alpha = case
    return VamanaBuildParameters(alpha=alpha or 0.0, graph_max_degree=R, window_size=window,
                                 max_candidate_pool_size=mc, prune_to=prune_to)


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
def refsq(reflib):
    from oracle.build_sq import RefSQBuildLib
    if not RefSQBuildLib.available():
        pytest.skip("oracle/_ref/libsvsref_sq_build.so not built (needs /root/reference)")
    if not reflib.avx512vnni():
        pytest.skip("host lacks AVX-512 VNNI: the reference would take its float fallback for integer rows")
    return RefSQBuildLib()


# ---------------------------------------------------------------- CPU

def test_sq_build_refusals():
    """Codes that are not int8 / uint8, a scale or bias an SQ index cannot hold, and svsb200_build_vamana's own
    refusals, each with an error that names the cause."""
    import ctypes as C

    from scalablevectorsearch_b200 import DistanceType, Svsb200Error, VamanaBuildParameters, _lib, build_graph
    lib = _lib.lib()
    codes = np.random.default_rng(0).integers(-100, 100, (64, 20)).astype(np.int8)
    graph = np.empty((64, 9), dtype=np.uint32)
    ep = C.c_uint32()

    def raw(code_type, scale, bias, pool=0):
        _lib.check(lib.svsb200_build_vamana_sq(codes.ctypes.data, code_type, 64, 20, 0, scale, bias, 0.0, 8, 16, pool, 0,
                                               0, graph.ctypes.data, C.byref(ep)))
    for code_type in (0, 1):   # float32, float16
        with pytest.raises(Svsb200Error, match="svsb200_build_vamana_sq: codes must be int8 or uint8"):
            raw(code_type, 0.1, 0.0)
    for scale, bias in ((0.0, 0.0), (-1.0, 0.0), (float("nan"), 0.0), (float("inf"), 0.0), (0.1, float("inf")),
                        (0.1, float("nan"))):
        with pytest.raises(Svsb200Error, match="svsb200_build_vamana_sq: the SQ scale must be finite and positive"):
            raw(2, scale, bias)
    with pytest.raises(Svsb200Error, match="svsb200_build_vamana_sq: max_candidate_pool_size above 512"):
        raw(2, 0.1, 0.0, pool=513)
    with pytest.raises(TypeError, match="SQ codes are int8 or uint8"):
        build_graph(codes.astype(np.float32), DistanceType.L2, VamanaBuildParameters(graph_max_degree=8, window_size=16),
                    sq=(0.1, 0.0))


# ---------------------------------------------------------------- GPU

@pytest.mark.gpu
@pytest.mark.parametrize("case", F.STATIC, ids=F.STATIC_IDS)
def test_static_sq_build_matches_the_reference_rows(refsq, case):
    from scalablevectorsearch_b200 import DistanceType, build_graph
    codes, scale, bias = F.static_codes(case)
    metric, R, window, mc, prune_to, alpha = case[1], *case[-5:]
    g_graph, g_ep = build_graph(codes, DistanceType(METRIC[metric]), parameters(case), sq=(scale, bias))
    r_graph, r_ep = refsq.build(codes, scale, bias, metric, R, window, alpha, mc or None, prune_to or None,
                                threads=ref_threads())
    assert g_ep == r_ep, (g_ep, r_ep)
    diff = first_difference(rows(g_graph), rows(r_graph))
    assert diff is None, f"{case[0]}: first row that differs {diff[0]}: gpu {diff[1]} vs reference {diff[2]}"


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,scale,bias", [(np.int8, 0.25, -3.0), (np.uint8, 2.0**-7, 0.5), (np.int8, 4.0, 0.0)])
def test_power_of_two_sq_l2_build_equals_the_integer_build(dtype, scale, bias):
    """scale a power of two and every decompressed value exact: the round trip returns the codes, and scale^2 times the
    integer L2 orders every pair as the integer L2 does, so the SQ L2 build is the integer build of the same codes."""
    from scalablevectorsearch_b200 import DistanceType, VamanaBuildParameters, build_graph
    lo, hi = (-128, 127) if dtype == np.int8 else (0, 255)
    for n, dim, R, window in ((40, 20, 6, 12), (40, 100, 8, 16), (37, 33, 8, 16)):
        codes = np.random.default_rng(n + dim).integers(lo, hi + 1, (n, dim)).astype(dtype)
        assert F.round_trip_moves(codes, scale, bias) == 0
        p = VamanaBuildParameters(graph_max_degree=R, window_size=window)
        g_sq, ep_sq = build_graph(codes, DistanceType.L2, p, sq=(scale, bias))
        g_int, ep_int = build_graph(codes, DistanceType.L2, p)
        assert ep_sq == ep_int
        diff = first_difference(rows(g_sq), rows(g_int))
        assert diff is None, f"n={n} dim={dim}: first row that differs {diff[0]}: sq {diff[1]} vs int {diff[2]}"


def _dataset_codes():
    from scalablevectorsearch_b200.ivf import sq_compress
    z = np.load(os.path.join(GOLDEN, "test_dataset.npz"))
    X = z["data"].astype(np.float32)
    codes, scale, bias = sq_compress(X)
    return z, X, codes, scale, bias


def _sq_search(codes, graph, ep, metric, scale, bias, queries, window):
    from scalablevectorsearch_b200 import DistanceType, SearchBufferConfig, Vamana
    index = Vamana.from_arrays(codes, graph, ep, DistanceType(METRIC[metric]), sq=(scale, bias))
    index.search_parameters.buffer_config = SearchBufferConfig(window)
    return index.search(queries, 10)


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
def test_sq_build_on_reference_dataset_matches_reference_builder_recall(refsq, metric):
    """The reference's 10k x 128 test dataset compressed to int8 codes by sq_compress, R = 32, window 64: the GPU SQ
    graph against the reference's SQ-built graph, both searched with float32 queries by the SQ search."""
    from scalablevectorsearch_b200 import DistanceType, VamanaBuildParameters, build_graph
    z, _, codes, scale, bias = _dataset_codes()
    Q, gt = z["queries"].astype(np.float32), z[f"gt_{metric}"]
    alpha = 1.2 if metric == "l2" else 0.95
    g_gpu, ep_gpu = build_graph(codes, DistanceType(METRIC[metric]),
                                VamanaBuildParameters(alpha=alpha, graph_max_degree=32, window_size=64),
                                sq=(scale, bias))
    g_ref, ep_ref = refsq.build(codes, scale, bias, metric, 32, 64, alpha=alpha, threads=ref_threads())
    assert ep_gpu == ep_ref, "medoid entry point differs from the reference's"
    for window in (10, 30):
        r_gpu = recall_at_k(_sq_search(codes, g_gpu, ep_gpu, metric, scale, bias, Q, window)[0], gt)
        r_ref = recall_at_k(_sq_search(codes, g_ref, ep_ref, metric, scale, bias, Q, window)[0], gt)
        assert r_gpu >= r_ref - 0.01, (metric, window, r_gpu, r_ref)
    d_gpu, d_ref = g_gpu[:, 0].mean(), g_ref[:, 0].mean()
    assert 0.8 * d_ref <= d_gpu <= 1.25 * d_ref, (d_gpu, d_ref)


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
def test_gpu_built_sq_index_search_equals_the_oracle(oracle, metric):
    """Vamana.build(..., sq=) on the test dataset's sq_compress codes, searched on the GPU: ids and distance bits equal
    the C oracle's SQ search over the same graph and codes."""
    from scalablevectorsearch_b200 import DistanceType, SearchBufferConfig, Vamana, VamanaBuildParameters
    z, X, codes, scale, bias = _dataset_codes()
    index = Vamana.build(VamanaBuildParameters(graph_max_degree=32, window_size=64), codes, DistanceType(METRIC[metric]),
                         sq=(scale, bias))
    from scalablevectorsearch_b200 import build_graph
    graph, ep = build_graph(codes, DistanceType(METRIC[metric]), VamanaBuildParameters(graph_max_degree=32, window_size=64),
                            sq=(scale, bias))
    built = Vamana.from_arrays(codes, graph, ep, DistanceType(METRIC[metric]), sq=(scale, bias))
    built.search_parameters.buffer_config = SearchBufferConfig(24, 40)
    want, o_codes, o_scale, o_bias = oracle.sq_index(X, graph, ep, metric)
    assert np.array_equal(o_codes, codes) and (o_scale, o_bias) == (scale, bias)
    q = z["queries"].astype(np.float32)[:256]
    got_ids, got_d = built.search(q, 10)
    want_ids, want_d = want.search(q, 10, 24, 40)
    assert np.array_equal(got_ids.astype(np.uint64), want_ids)
    assert np.array_equal(got_d.view(np.uint32), want_d.view(np.uint32))
    # Vamana.build(..., sq=) is the same SQ index: its search over the codes is as good as the assembled one's
    gt = z[f"gt_{metric}"][:256]
    index.search_parameters.buffer_config = SearchBufferConfig(24, 40)
    assert recall_at_k(index.search(q, 10)[0], gt) >= recall_at_k(got_ids, gt) - 0.01


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["l2", "ip"])
def test_runtime_vamana_sq_demo_matches_the_python_path(tmp_path, metric):
    """cpp/vamana_sq_demo, written against the reference's runtime headers only (VamanaIndex with StorageKind::SQI8),
    prints what sq_compress + Vamana.build(..., sq=) give for the same rows and parameters: search, IDFilter search,
    range search, reconstruct_at and get_distance.  check_storage_kind(SQI8) is 0 and constant rows, which have no SQ
    scale, are an add status RUNTIME_ERROR (5).  n = 40 keeps the build one node per round, so both sides build the
    same graph."""
    from scalablevectorsearch_b200 import DistanceType, SearchBufferConfig, Vamana, VamanaBuildParameters
    from scalablevectorsearch_b200.ivf import sq_compress
    exe = os.path.join(ROOT, "scalablevectorsearch_b200", "cpp", "_build", "vamana_sq_demo")
    if not os.path.exists(exe):
        pytest.skip("vamana_sq_demo not built (needs the reference's runtime headers at build time)")
    n, dim, nq, k, R, W = 40, 24, 12, 5, 8, 16
    rng = np.random.default_rng(5)
    x = rng.standard_normal((n, dim)).astype(np.float32)
    q = rng.standard_normal((nq, dim)).astype(np.float32)
    codes, scale, bias = sq_compress(x)
    index = Vamana.build(VamanaBuildParameters(graph_max_degree=R, window_size=W), codes,
                         DistanceType(METRIC[metric]), sq=(scale, bias))
    index.search_parameters.buffer_config = SearchBufferConfig(2 * k)
    ids, dists = index.search(q, k)
    radius = float(np.median(dists[:, 2]))
    x.tofile(tmp_path / "x.f32")
    q.tofile(tmp_path / "q.f32")
    out = subprocess.run([exe, str(tmp_path / "x.f32"), str(n), str(dim), str(tmp_path / "q.f32"), str(nq), str(k),
                          str(METRIC[metric]), str(R), str(W), repr(radius)], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    got = {}
    for line in out.stdout.splitlines():
        tag, *rest = line.split()
        got.setdefault(tag, []).append(rest)
    assert got["storage_sqi8"] == [["0"]]
    assert got["constant"] == [["5"]]

    def pairs(tag):
        return (np.array([int(r[0]) for r in got[tag]], dtype=np.uint64).reshape(nq, k),
                np.array([float(r[1]) for r in got[tag]]).astype(np.float32).reshape(nq, k))
    r_ids, r_d = pairs("search")
    assert np.array_equal(r_ids, ids) and np.array_equal(r_d.view(np.uint32), dists.view(np.uint32))
    f_ids, f_d, _ = index.search_filtered(q, k, np.arange(n) % 3 == 0)
    r_ids, r_d = pairs("filtered")
    assert np.array_equal(r_ids, f_ids) and np.array_equal(r_d.view(np.uint32), f_d.view(np.uint32))
    want = [(qi, int(i), np.float32(d)) for qi, (ii, dd) in enumerate(index.range_search(q, radius)) for i, d in zip(ii, dd)]
    assert [(int(a), int(b), np.float32(float(c))) for a, b, c in got.get("range", [])] == want
    back = np.array([float(r[0]) for r in got["reconstruct"]], dtype=np.float32).reshape(4, dim)
    assert np.array_equal(back.view(np.uint32), F.decompress(codes[:4], scale, bias).view(np.uint32))
    for r in got["distance"]:
        i = int(r[0])
        s_ids, s_d, found = index.search_filtered(q[:1], 1, np.arange(n) == i)
        assert found[0] == 1 and int(s_ids[0, 0]) == i
        assert np.float32(float(r[1])).view(np.uint32) == s_d[0, 0].view(np.uint32), i
    graph_bytes, _ = (int(v) for v in got["memory"][0])
    assert graph_bytes == n * (R + 1) * 4
