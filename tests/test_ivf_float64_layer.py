"""The float64 layer of tests/test_gpu_ivf_shapes.py on the CPU: it accepts the models' own (oracle) results for the
GPU file's fixtures, and rejects them after a change its bound says is too large -- a distance moved by 2^-10 of the
magnitudes its bound scales, one integer step of an SQ L2 sum, a returned row swapped for a farther one, a row
assigned to its farthest centroid.  So the bound is neither wrong nor vacuous before any GPU run.  No GPU needed."""
import numpy as np
import pytest

import float64_layer as F64
import ivf_model as M
import test_gpu_ivf_shapes as G

CASES = [  # (dim, rows dtype, queries dtype, metric, SQ code)
    (128, np.float32, np.float32, 0, None), (385, np.float16, np.float32, 1, None), (769, np.float32, np.float16, 2, None),
    (3073, np.float16, np.float16, 0, None), (200, np.float32, np.float32, 0, np.int8),
    (6161, np.float32, np.float16, 0, np.uint8), (3072, np.float32, np.float32, 1, np.int8),
    (3072, np.float32, np.float32, 2, np.uint8),
]


def _rejects(fn):
    with pytest.raises(AssertionError):
        fn()


@pytest.mark.parametrize("dim,dtype,qdtype,metric,code", CASES)
def test_layer_accepts_the_model_and_rejects_perturbations(oracle, dim, dtype, qdtype, metric, code):
    case = G.Case(dim, dtype, qdtype, metric, 300, 8, 4, seed=dim + metric, sq_code=code)
    for P in (case.C, 2):
        ids, dists = case.model(oracle, case.q, 10, P)
        layer = (case.rows, case.sq, metric, case.cent, case.assign, case.q)
        G.float64_layer(oracle, *layer, (ids, dists), P, "model")
    ids, dists = case.model(oracle, case.q, 10, case.C)   # every row a candidate
    rows = F64.Rows(case.rows, case.sq)
    name = G.NAME[metric]
    i, q = 0, case.q[0]
    if code is not None and metric == 0:
        # one integer step of the first row's sum: fl32(fl32(scale^2) * fl32(sum + 1))
        qc = F64.sq_l2_query_codes(q, case.rows.dtype, *case.sq)
        s = int(((case.rows[int(ids[i, 0])].astype(np.int64) - qc) ** 2).sum())
        assert s + 1 < 2 ** 24, "the step must survive the float32 conversion"
        scale = np.float32(case.sq[0])
        bad = dists[i].copy()
        bad[0] = np.float32(scale * scale) * np.float32(s + 1)
        assert bad[0] != dists[i, 0]
    else:
        # 2^-10 of the magnitudes the bound scales (sum |terms|; for cosine relative to the norms): far past
        # (dim + 8) 2^-24 of them, and past 2^-10 of the distance itself wherever the sum cancels
        _, bound = rows.reference(name, q, ids[i, :1])
        bad = dists[i].copy()
        bad[0] = np.float32(bad[0] + 2.0 ** -10 * bound[0] / F64.gamma(dim))
    rows.check_distances(name, q, ids[i], dists[i], "model")
    _rejects(lambda: rows.check_distances(name, q, ids[i], bad, "perturbed"))
    # a returned row swapped for the candidate farthest away in float64
    cand = np.arange(case.rows.shape[0])
    d64, _ = rows.reference(name, q, cand)
    far = cand[np.argmax(d64 if metric == 0 else -d64)]
    assert far not in ids[i]
    swapped = ids[i].copy()
    swapped[0] = far
    rows.check_set(name, q, ids[i], cand, "model")
    _rejects(lambda: rows.check_set(name, q, swapped, cand, "swapped"))


@pytest.mark.parametrize("dim,metric", [(33, 0), (33, 1), (200, 2)])
def test_assignment_check(oracle, dim, metric):
    x = G.rows_of(np.random.default_rng(dim), 500, dim, np.float32, 8)
    cent, assign = M.kmeans(oracle, x, metric, 20, 2, 0.5, dim)
    F64.check_assignment(G.NAME[metric], x, cent, assign, "model")
    d, _ = F64.float_tree(G.NAME[metric], x[0].astype(np.float64), cent.astype(np.float64))
    bad = assign.copy()
    bad[0] = np.argmax(d if metric == 0 else -d)
    _rejects(lambda: F64.check_assignment(G.NAME[metric], x, cent, bad, "moved"))
