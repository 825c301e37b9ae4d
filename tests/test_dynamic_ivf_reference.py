"""The dynamic IVF model (tests/dynamic_ivf_model.py) against the reference's own DynamicIVFIndex behind a test-only
façade (oracle/dynamic_ivf.mk, oracle/ref/dynamic_ivf_capi.cpp), no GPU.

On the reference's test dataset and three metrics, through a mutation script: the slots every add returns and the
external ids in slot order equal the reference's at every step; searches are compared after assembly, after deletes
and after compaction (in between, the reference's added entries are wrong, below): at n_probes = C the distance bits
are equal and the ids equal up to the order inside tie groups, and with fewer probes recall@10 against the model's
exact result agrees within the allowance of the static IVF comparison (the reference ranks centroids from its GEMM).

Three tests pin where the reference's add_points departs from its documented intent, which this project follows
(DESIGN.md §16), so that a fix in the reference is noticed."""
import os

import numpy as np
import pytest

import ivf_model as M
from dynamic_ivf_model import RESERVED, DynamicIVFModel


@pytest.fixture(scope="module")
def ref_cls():
    from oracle.dynamic_ivf import RefDynamicIVF
    if not RefDynamicIVF.available():
        pytest.skip("oracle/_ref/libsvsref_dynamic_ivf.so not built (needs the reference at build time)")
    return RefDynamicIVF


@pytest.fixture(scope="module")
def dataset():
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "test_dataset.npz"))
    return z["data"].astype(np.float32), z["queries"].astype(np.float32)


def _same_up_to_kth_ties(ids_a, d_a, ids_b, d_b):
    """Distance bits equal everywhere; the same ids at every distance above the k-th (a tie group compares as a set)."""
    assert np.array_equal(d_a.view(np.uint32), d_b.view(np.uint32))
    for ia, ib, d in zip(ids_a, ids_b, d_a):
        for v in np.unique(d[d != d[-1]]):
            assert set(ia[d == v].tolist()) == set(ib[d == v].tolist())


def _compare(model, ref, q, C, what):
    mi, md = model.search(q, 10, C)
    ri, rd = ref.search(q, 10, C)
    _same_up_to_kth_ties(mi, md, ri, rd)
    exact = mi

    def recall(ids):
        return float(np.mean([len(set(a.tolist()) & set(b.tolist())) / 10 for a, b in zip(ids, exact)]))

    for n_probes in (2, 8):
        mi, _ = model.search(q, 10, n_probes)
        ri, _ = ref.search(q, 10, n_probes)
        print(f"{what}, n_probes {n_probes}: recall model {recall(mi):.4f} reference {recall(ri):.4f}, "
              f"{int((mi != ri).any(1).sum())} of {len(q)} queries with different ids")
        assert abs(recall(mi) - recall(ri)) <= 0.005, what


@pytest.mark.parametrize("metric", [0, 1, 2])
def test_model_equals_the_reference_through_a_mutation_script(oracle, ref_cls, dataset, metric):
    x, q = dataset
    C = 32
    cent, assign = M.kmeans(oracle, x[:8000], metric, C, 3, 0.1, 1)
    rng = np.random.default_rng(metric)
    ids = rng.permutation(10**6)[:10000].astype(np.uint64)
    model = DynamicIVFModel.assemble(oracle, metric, cent, x[:8000], ids[:8000], assign)
    ref = ref_cls(x[:8000], ids[:8000], metric, cent, assign)
    assert np.array_equal(model.all_ids(), ref.all_ids())
    _compare(model, ref, q, C, "assembled")
    gone = rng.choice(ids[:8000], 2000, replace=False)
    model.delete(gone)
    ref.delete(gone)
    assert np.array_equal(model.all_ids(), ref.all_ids())
    _compare(model, ref, q, C, "deleted")
    for lo, hi, reuse in ((8000, 8500, False), (8500, 9700, True), (9700, 10000, False)):
        assert model.add(x[lo:hi], ids[lo:hi], reuse) == ref.add(x[lo:hi], ids[lo:hi], reuse)
        assert np.array_equal(model.all_ids(), ref.all_ids())
    model.compact()
    ref.compact()
    assert np.array_equal(model.all_ids(), ref.all_ids())
    _compare(model, ref, q, C, "compacted")


def _six_rows(ref_cls, oracle):
    """Six rows in two clusters (rows 0, 2, 4 near centroid 0; 1, 3, 5 near centroid 1), ids 10-15."""
    cent = np.array([[0, 0], [10, 10]], np.float32)
    x = np.array([[0, 1], [10, 11], [1, 0], [11, 10], [1, 1], [9, 9]], np.float32)
    a = np.array([0, 1, 0, 1, 0, 1], np.uint32)
    return (ref_cls(x, np.arange(10, 16), 0, cent, a), DynamicIVFModel.assemble(oracle, 0, cent, x, np.arange(10, 16), a),
            x)


def test_reference_defect_an_added_row_comes_back_under_slot_zeros_id(ref_cls, oracle):
    ref, model, _ = _six_rows(ref_cls, oracle)
    p = np.array([[0.5, 0.5]], np.float32)
    for index in (ref, model):
        index.delete([11])
        assert index.add(p, [20]) == [6]
    ri, rd = ref.search(p, 1, 1)
    assert ri[0, 0] == 10 and rd[0, 0] == 0.0     # the new row (distance 0) under slot 0's id
    mi, md = model.search(p, 1, 1)
    assert mi[0, 0] == 20 and md[0, 0] == 0.0


def test_reference_defect_a_reused_slot_brings_back_the_deleted_row(ref_cls, oracle):
    ref, model, x = _six_rows(ref_cls, oracle)
    p = np.array([[0.5, 0.5]], np.float32)
    for index in (ref, model):
        index.delete([11])
        assert index.add(p, [20], True) == [1]
    ri, rd = ref.search(x[1:2], 1, 1)                # the deleted row's own vector, probing its old cluster
    assert ri[0, 0] == 20 and rd[0, 0] == 0.0
    mi, md = model.search(x[1:2], 1, 1)
    assert mi[0, 0] == 13 and md[0, 0] == 2.0
    ref.compact()                                    # compaction repairs the reference
    model.compact()
    _same_up_to_kth_ties(*model.search(x, 3, 2), *ref.search(x, 3, 2))


def test_reference_defect_short_results_are_padded_with_slot_zero(ref_cls, oracle):
    ref, model, x = _six_rows(ref_cls, oracle)
    ri, rd = ref.search(x[:1], 4, 1)                 # the probed cluster holds 3 rows
    assert ri[0, 3] == 10 and rd[0, 3] == 0.0
    mi, md = model.search(x[:1], 4, 1)
    assert mi[0, 3] == RESERVED and md[0, 3] == np.inf
