"""The SQ graph builder's distance model against the reference, without a GPU.

tests/build_sq_fixtures.py restates the distance the reference's builder uses over SQDataset<int8_t / uint8_t>
(DecompressionAdaptor over the compressed distance): datum i decompressed to float32, then prepared and measured as
the SQ search prepares and measures a float32 query.  Here that model reproduces the reference's own values bit for
bit on every fixture, pair by pair, and the reference's SQ builds of n <= 40 do not depend on its thread count, which
is what lets tests/test_gpu_build_sq.py compare rows exactly."""
import numpy as np
import pytest

import build_sq_fixtures as F

PREMISE_THREADS = (1, 8)


@pytest.fixture(scope="module")
def refsq(reflib):
    """The reference's builder over SQ codes (oracle/_ref/libsvsref_sq_build.so); its distances are the AVX-512
    ones the C oracle restates, and its integer L2 is exact on the VNNI path only."""
    from oracle.build_sq import RefSQBuildLib
    if not RefSQBuildLib.available():
        pytest.skip("oracle/_ref/libsvsref_sq_build.so not built (needs /root/reference)")
    if not reflib.avx512vnni():
        pytest.skip("host lacks AVX-512 VNNI: the reference would take its float fallback for integer rows")
    return RefSQBuildLib()


@pytest.mark.parametrize("case", F.STATIC, ids=F.STATIC_IDS)
def test_build_distance_model_equals_the_reference(refsq, oracle, case):
    codes, scale, bias = F.static_codes(case)
    metric, n = case[1], codes.shape[0]
    pairs = np.array([(i, j) for i in range(n) for j in range(n)], dtype=np.uint32)
    want = refsq.distance(codes, scale, bias, metric, pairs).reshape(n, n)
    got = np.stack([F.build_distances(oracle, metric, codes, scale, bias, i) for i in range(n)])
    bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
    assert bad.size == 0, f"{case[0]}: {len(bad)} pairs differ, first {tuple(bad[0])}: {got[tuple(bad[0])]} vs {want[tuple(bad[0])]}"


@pytest.mark.parametrize("case", F.MOVING, ids=[c[0] for c in F.MOVING])
def test_moving_fixtures_move_codes_in_the_l2_round_trip(case):
    """The bias is large against the scale: the decompressed float loses bits, so compressing it again does not
    always return the datum's codes, and the L2 build measures from the moved codes."""
    codes, scale, bias = F.static_codes(case)
    assert F.round_trip_moves(codes, scale, bias) > 0, case[0]


def test_other_fixtures_keep_their_codes():
    for case in F.STATIC:
        if case not in F.MOVING:
            codes, scale, bias = F.static_codes(case)
            assert F.round_trip_moves(codes, scale, bias) == 0, case[0]


@pytest.mark.parametrize("case", F.STATIC, ids=F.STATIC_IDS)
def test_premise_reference_static_sq_build_is_deterministic(refsq, case):
    codes, scale, bias = F.static_codes(case)
    _, metric, *_, R, window, mc, prune_to, alpha = case
    (g1, ep1), (g8, ep8) = (refsq.build(codes, scale, bias, metric, R, window, alpha, mc or None, prune_to or None,
                                        threads=t) for t in PREMISE_THREADS)
    assert ep1 == ep8 and np.array_equal(g1, g8), f"premise broken for static fixture {case[0]}"
