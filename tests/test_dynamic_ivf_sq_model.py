"""The numpy model of the SQ dynamic IVF index (tests/dynamic_ivf_sq_model.py) without a GPU: the slot rules over codes
on a hand-made script, the add refusals, equalities with the static SQ model (an unmutated index, an assembled prefix
filled by float32 adds, an empty index filled by one add), and the add encoder held bit for bit to the reference's own
SQDataset::set_datum (through a test-only façade, oracle/sq_set_datum.mk)."""
import numpy as np
import pytest

import ivf_model as M
import ivf_sq_model as S
from dynamic_ivf_model import NONE32, RESERVED, Refused
from dynamic_ivf_sq_model import DynamicIVFSQModel


def _two_clusters(oracle, metric=0, dtype=np.int8):
    """Six rows in two well separated clusters (rows 0, 2, 4 near centroid 0; 1, 3, 5 near centroid 1), ids 10-15."""
    cent = np.array([[0.0, 0.0], [10.0, 10.0]], dtype=np.float32)
    x = np.array([[0, 1], [10, 11], [1, 0], [11, 10], [1, 1], [9, 9]], dtype=np.float32)
    codes, scale, bias = S.compress(x, dtype)
    a = np.array([0, 1, 0, 1, 0, 1], dtype=np.uint32)
    return DynamicIVFSQModel.assemble(oracle, metric, cent, codes, np.arange(10, 16), scale, bias, a), x, codes


def test_script_over_codes(oracle):
    m, x, codes = _two_clusters(oracle)
    assert m.stored == [[0, 2, 4], [1, 3, 5]]
    m.delete([11, 12])
    slots = m.add(np.array([[0.5, 0.5], [10.5, 10.5]], dtype=np.float32), [20, 21], reuse_empty=True)
    assert slots == [1, 2]
    status, ext, cluster = m.export()
    assert list(status) == [1] * 6 and list(ext) == [10, 20, 21, 13, 14, 15]
    assert list(cluster) == [0, 0, 1, 1, 0, 1]
    assert m.stored == [[0, None, 4, 1], [None, 3, 5, 2]]
    assert np.array_equal(m.rows[1], S.encode(np.array([0.5, 0.5], np.float32), np.int8, m.scale, m.bias))
    m.delete([10])
    m.compact()
    assert list(m.all_ids()) == [20, 21, 13, 14, 15]
    assert m.stored == [[3, 0], [2, 4, 1]]
    ids, d = m.search(np.array([[0.2, 0.2]], dtype=np.float32), 3, 1)
    assert set(ids[0]) == {20, 14} | {RESERVED}
    assert ids[0, 2] == RESERVED and np.isinf(d[0, 2])


def test_add_refusals_change_nothing(oracle):
    m, x, codes = _two_clusters(oracle)
    before = [a.copy() for a in m.export()]
    for bad in (x[:1].astype(np.float16), codes[:1], np.array([[np.nan, 0]], np.float32),
                np.array([[np.inf, 0]], np.float32)):
        with pytest.raises(Refused):
            m.add(bad, [99])
        for a, b in zip(m.export(), before):
            assert np.array_equal(a, b)
    with pytest.raises(Refused, match="assignments"):
        DynamicIVFSQModel.assemble(oracle, 0, m.centroids, codes, np.arange(6), m.scale, m.bias)


def test_clamped_adds(oracle):
    m, x, _ = _two_clusters(oracle, dtype=np.uint8)
    far = np.array([[-100.0, 1000.0]], dtype=np.float32)
    m.add(far, [50])
    assert list(m.rows[6]) == [0, 255]


def _data(seed, n=600, dim=12):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((n, dim)).astype(np.float32), rng.standard_normal((7, dim)).astype(np.float32)


@pytest.mark.parametrize("metric", [0, 1, 2])
@pytest.mark.parametrize("dtype", [np.int8, np.uint8])
def test_equalities_with_the_static_sq_model(oracle, metric, dtype):
    x, q = _data(metric + 10)
    C = 9
    cent = x[::67][:C].copy()
    codes, scale, bias = S.compress(x, dtype)
    near = M.nearest(oracle, metric, x, cent, 1)[:, 0].astype(np.uint32)
    given = (near + np.arange(x.shape[0]) % 2).astype(np.uint32) % C   # assignments other than the nearest
    n0 = 400
    # 2: unmutated, ids 0 .. n-1
    unmutated = DynamicIVFSQModel.assemble(oracle, metric, cent, codes, np.arange(600), scale, bias, given)
    # 3: the first n0 codes assembled, the remaining rows added as float32
    prefix = DynamicIVFSQModel.assemble(oracle, metric, cent, codes[:n0], np.arange(n0), scale, bias, given[:n0])
    prefix.add(x[n0:], np.arange(n0, 600))
    mixed = np.concatenate([given[:n0], near[n0:]])
    # 4: empty, filled by one add
    empty = DynamicIVFSQModel.assemble(oracle, metric, cent, codes[:0], [], scale, bias)
    empty.add(x, np.arange(600))
    for n_probes in (1, 4, C):
        for k in (1, 10, 100):
            want = S.search(oracle, metric, codes, scale, bias, cent, given, q, k, n_probes)
            got = unmutated.search(q, k, n_probes)
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32))
            want = S.search(oracle, metric, codes, scale, bias, cent, mixed, q, k, n_probes)
            got = prefix.search(q, k, n_probes)
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32))
            want = S.search(oracle, metric, S.encode(x, dtype, scale, bias), scale, bias, cent, near, q, k, n_probes)
            got = empty.search(q, k, n_probes)
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32))


# ---- the add encoder against the reference's own SQDataset::set_datum (oracle/sq_set_datum.mk façade) ----

@pytest.fixture(scope="module")
def ref_set_datum():
    from oracle.sq_set_datum import RefSQSetDatum
    if not RefSQSetDatum.available():
        pytest.skip("oracle/_ref/libsvsref_sq_set_datum.so not built (needs the reference at build time)")
    return RefSQSetDatum()


@pytest.mark.parametrize("dtype", [np.int8, np.uint8])
def test_add_encoder_equals_the_reference_set_datum(ref_set_datum, dtype):
    rng = np.random.default_rng(5)
    base = rng.standard_normal((200, 16)).astype(np.float32)
    _, scale, bias = S.compress(base, dtype)
    s, b = np.float32(scale), np.float32(bias)
    lo, hi = S.RANGE[np.dtype(dtype)]
    # exact .5 midpoints: x = bias + (j + 0.5) scale wherever that lands on a float32 midpoint, and its neighbours
    j = np.arange(lo - 3, hi + 3, dtype=np.float32)
    mid = (b + (j + np.float32(0.5)) * s).astype(np.float32)
    mids = np.concatenate([mid, np.nextafter(mid, np.float32(np.inf)), np.nextafter(mid, np.float32(-np.inf))])
    edges = np.array([-0.0, 0.0, b, -b, 1e30, -1e30, np.float32(3.4e38), np.float32(-3.4e38),
                      base.min() - 5, base.max() + 5], dtype=np.float32)
    wide = rng.standard_normal(16 * 64).astype(np.float32) * 8   # well beyond both ends of the range
    x = np.concatenate([base.reshape(-1), mids, edges, wide])
    x = np.concatenate([x, np.zeros((-x.size) % 16, np.float32)]).reshape(-1, 16)
    want = ref_set_datum.set_datum(x, dtype, scale, bias)
    with np.errstate(over="ignore"):   # (values near float32's ends divide to +-inf, which clamps)
        got = S.encode(x, dtype, scale, bias)
    assert np.array_equal(got, want)
    assert (got == lo).any() and (got == hi).any()   # both ends clamp
