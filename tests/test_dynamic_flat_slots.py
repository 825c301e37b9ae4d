"""The slot rules of the dynamic flat index, without a GPU: the pure-Python model of tests/dynamic_flat_model.py by hand,
and against the reference's own DynamicFlatIndex (oracle/_ref façade) through the mutation script the GPU tests run.
Slots returned by add, status, external ids and first_empty_ must agree after every step."""
import numpy as np
import pytest

from dynamic_flat_model import EMPTY, RESERVED, VALID, SlotModel, pool_size, run_script


def test_model_first_empty_rules_by_hand():
    m = SlotModel([10, 11, 12, 13, 14, 15])
    assert m.first_empty == 6
    m.delete([13, 11])
    assert m.first_empty == 1                       # min(first_empty, slot)
    assert m.add([20], reuse_empty=False) == [1]    # scans from first_empty
    assert m.first_empty == 2
    assert m.add([21, 22]) == [3, 6]                # the remaining Empty slot, then growth
    assert m.first_empty == 7
    assert m.add([23, 24], reuse_empty=True) == [7, 8]
    m.delete([10])
    assert m.first_empty == 0
    m.compact()
    assert m.live_ids().tolist() == [20, 12, 21, 14, 15, 22, 23, 24] and m.first_empty == 8
    status, ext = m.export()
    assert (status == VALID).all() and ext.tolist() == m.live_ids().tolist()


def test_model_refuses_without_changing():
    m = SlotModel([1, 2, 3])
    before = (m.export(), m.first_empty)
    for bad in ([1], [7, 7], [RESERVED]):
        with pytest.raises(ValueError):
            m.add(bad)
    for bad in ([9], [2, 2]):
        with pytest.raises(KeyError):
            m.delete(bad)
    after = (m.export(), m.first_empty)
    assert all(np.array_equal(a, b) for a, b in zip(before[0], after[0])) and before[1] == after[1]
    m.delete([2])
    assert m.export()[0].tolist() == [VALID, EMPTY, VALID]


def _reflib():
    from oracle.dynamic_flat import RefDynamicFlatLib
    if not RefDynamicFlatLib.available():
        pytest.skip("oracle/_ref/libsvsref_dynamic_flat.so not built (needs /root/reference)")
    return RefDynamicFlatLib()


@pytest.mark.parametrize("dtype", [np.float32, np.int8])
def test_reference_follows_the_model(dtype):
    lib = _reflib()
    n0 = 300
    rng = np.random.default_rng(3)
    pool = (rng.standard_normal((pool_size(n0), 8)) * 20).astype(dtype)
    ids = 3 * np.arange(n0, dtype=np.uint64) + 1
    ref = lib.dynamic_flat(pool[:n0], ids, "l2", threads=2)
    model = SlotModel(ids, payload=range(n0))

    def check(step):
        status, ext = ref.export()
        want_status, want_ext = model.export()
        assert np.array_equal(status, want_status), step[:1]
        assert np.array_equal(ext, want_ext), step[:1]
        assert np.array_equal(ref.all_ids(), model.live_ids()), step[:1]

    check(("build",))
    run_script(ref, model, pool, n0, seed=1, check=check)
    assert len(model.status) == model.first_empty == ref.size
