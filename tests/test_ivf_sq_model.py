"""The SQ IVF model (tests/ivf_sq_model.py) without a GPU: its compression against the C oracle's SQDataset::compress and
the reference's own (through its IVF façade, oracle/ivf_sq.mk), bit for bit, and its L2 / MIP / cosine distances against
the oracle's SQ index, whose SQ distances are held to the reference's goldens."""
import os

import numpy as np
import pytest

import ivf_sq_model as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def oracle():
    from oracle.bindings import OracleLib
    if not OracleLib.available():
        import subprocess
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "oracle"])
    return OracleLib()


def oracle_compress(oracle, x, dtype):
    graph = np.zeros((x.shape[0], 2), dtype=np.uint32)
    index, codes, scale, bias = oracle.sq_index(x, graph, 0, "l2", code_dtype=dtype)
    index.close()
    return codes, scale, bias


def datasets():
    z = np.load(os.path.join(ROOT, "tests", "golden", "test_dataset.npz"))
    rng = np.random.default_rng(3)
    edges = rng.standard_normal((301, 37)).astype(np.float32)
    edges[0, :4] = [edges.min() - 1, edges.max() + 1, -0.0, 0.0]
    halves = (np.arange(-300, 300, dtype=np.float32) * 0.5).reshape(40, 15)   # ties at the rounding midpoints
    zero_min = np.abs(rng.standard_normal((50, 9))).astype(np.float32)
    zero_min[3, 2], zero_min[7, 1] = -0.0, 0.0                                # the first zero is negative
    return {"reference": z["data"].astype(np.float32), "edges": edges, "halves": halves, "zero_min": zero_min}


@pytest.mark.parametrize("dtype", [np.int8, np.uint8])
@pytest.mark.parametrize("name", ["reference", "edges", "halves", "zero_min"])
def test_compression_equals_the_oracle(oracle, name, dtype):
    x = datasets()[name]
    codes, scale, bias = S.compress(x, dtype)
    want_codes, want_scale, want_bias = oracle_compress(oracle, x, dtype)
    assert np.float32(scale).view(np.uint32) == np.float32(want_scale).view(np.uint32)
    assert np.float32(bias).view(np.uint32) == np.float32(want_bias).view(np.uint32)
    assert np.array_equal(codes, want_codes)


@pytest.mark.parametrize("dtype", [np.int8, np.uint8])
@pytest.mark.parametrize("metric", [0, 1, 2])
def test_distances_equal_the_oracle_sq_index(oracle, metric, dtype):
    # a complete graph with a window of n makes the oracle's greedy search score every row
    rng = np.random.default_rng(1)
    x = rng.standard_normal((200, 48)).astype(np.float32)
    q = rng.standard_normal((5, 48)).astype(np.float32) * 1.5   # values past the data's range clamp
    graph = np.zeros((200, 200), dtype=np.uint32)
    graph[:, 0] = 199
    for i in range(200):
        graph[i, 1:] = [j for j in range(200) if j != i]
    index, codes, scale, bias = oracle.sq_index(x, graph, 0, ("l2", "ip", "cosine")[metric], code_dtype=dtype)
    ids, dists = index.search(q, 200, 200)
    index.close()
    for i in range(q.shape[0]):
        d = S.distances(oracle, metric, q[i], codes, scale, bias)
        assert np.array_equal(d[ids[i].astype(np.int64)].view(np.uint32), dists[i].view(np.uint32))


# ---- the model against the reference's own IVF index over SQ rows (oracle/ivf_sq.mk façade) ----

@pytest.fixture(scope="module")
def ref_ivf_sq():
    from oracle.ivf_sq import RefIVFSQ
    if not RefIVFSQ.available():
        pytest.skip("oracle/_ref/libsvsref_ivf_sq.so not built (needs the reference at build time)")
    return RefIVFSQ()


def test_compression_equals_the_reference(ref_ivf_sq):
    # the reference's own SQDataset<int8_t / uint8_t>::compress, through its IVF façade
    z = np.load(os.path.join(ROOT, "tests", "golden", "test_dataset.npz"))
    for x in (z["data"].astype(np.float32), datasets()["edges"], datasets()["zero_min"]):
        assign = np.zeros(x.shape[0], dtype=np.uint32)
        for dtype in (np.int8, np.uint8):
            _, _, rcodes, rscale, rbias = ref_ivf_sq.search(x, dtype, 0, x[:1], assign, x[:1], 1, 1)
            codes, scale, bias = S.compress(x, dtype)
            assert np.float32(scale).view(np.uint32) == np.float32(rscale).view(np.uint32)
            assert np.float32(bias).view(np.uint32) == np.float32(rbias).view(np.uint32)
            assert np.array_equal(codes, rcodes)
