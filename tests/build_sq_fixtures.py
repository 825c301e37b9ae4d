"""The SQ graph builder's fixtures and its numpy distance model (include/svsb200.h, svsb200_build_vamana_sq), shared
by tests/test_build_sq_model.py (no GPU) and tests/test_gpu_build_sq.py.

The reference builds SQDataset<int8_t / uint8_t> through DecompressionAdaptor: datum i is decompressed to float32 as
scale * c + bias (each operation rounded on its own) and becomes the query of the SQ search's compressed distance,
whose model is tests/ivf_sq_model.py's ``distances``."""
from __future__ import annotations

import numpy as np

import ivf_sq_model as SQ

METRIC = {"l2": 0, "ip": 1, "cosine": 2}

# id, metric, code dtype, n, dim, codes (lo, hi), scale, bias, R, window, max_candidate_pool_size, prune_to, alpha.
# scale None: scale and bias of SQDataset::compress over float rows drawn from [-1, 1).  "moving": a bias large
# against the scale, so that decompressing and compressing again moves some codes.
STATIC = [
    ("l2-i8", "l2", np.int8, 40, 20, None, None, None, 6, 12, 0, 0, None),
    ("ip-i8", "ip", np.int8, 40, 20, None, None, None, 6, 12, 0, 0, None),
    ("cosine-i8", "cosine", np.int8, 40, 20, None, None, None, 6, 12, 0, 0, None),
    ("l2-u8", "l2", np.uint8, 40, 20, None, None, None, 8, 16, 0, 0, None),
    ("ip-u8", "ip", np.uint8, 37, 20, None, None, None, 8, 16, 0, 0, None),
    ("cosine-u8", "cosine", np.uint8, 40, 20, None, None, None, 8, 16, 0, 0, None),
    ("l2-i8-ties", "l2", np.int8, 40, 20, (-3, 3), 0.37, 0.11, 8, 16, 0, 0, None),
    ("ip-i8-ties", "ip", np.int8, 40, 20, (-3, 3), 0.37, 0.11, 6, 12, 0, 0, None),
    ("cosine-u8-ties", "cosine", np.uint8, 40, 20, (1, 3), 0.37, 0.11, 8, 16, 0, 0, None),
    ("l2-u8-dim100-prune_to", "l2", np.uint8, 40, 100, None, None, None, 8, 16, 0, 5, None),
    ("ip-i8-dim100", "ip", np.int8, 40, 100, None, None, None, 8, 16, 0, 0, None),
    ("cosine-u8-dim100-small-pool", "cosine", np.uint8, 40, 100, None, None, None, 4, 12, 6, 3, None),
    ("l2-i8-moving", "l2", np.int8, 40, 20, (-128, 127), 2e-5, 300.7, 6, 12, 0, 0, None),
    ("l2-u8-moving", "l2", np.uint8, 40, 20, (0, 255), 2e-5, -300.7, 8, 16, 0, 0, None),
    ("ip-i8-moving", "ip", np.int8, 40, 20, (-128, 127), 2e-5, 300.7, 6, 12, 0, 0, None),
    ("cosine-u8-moving", "cosine", np.uint8, 40, 20, (0, 255), 2e-5, -300.7, 8, 16, 0, 0, None),
    ("l2-i8-alpha", "l2", np.int8, 40, 20, None, None, None, 6, 12, 0, 0, 1.5),
    ("cosine-i8-alpha", "cosine", np.int8, 33, 20, None, None, None, 7, 12, 0, 0, 0.85),
]
STATIC_IDS = [s[0] for s in STATIC]
MOVING = [s for s in STATIC if s[0].endswith("moving")]


def static_codes(case):
    """(codes, scale, bias) of a fixture, float32 scale and bias."""
    _, _, dtype, n, dim, rng_, scale, bias, R, *_ = case
    rng = np.random.default_rng(n * 7 + R + dim)
    if scale is None:
        return SQ.compress(rng.uniform(-1, 1, (n, dim)).astype(np.float32), dtype)
    lo, hi = rng_
    return rng.integers(lo, hi + 1, (n, dim)).astype(dtype), float(np.float32(scale)), float(np.float32(bias))


def decompress(codes: np.ndarray, scale: float, bias: float) -> np.ndarray:
    """detail::decompress: scale * c + bias, each operation rounded to float32."""
    return ((np.float32(scale) * codes.astype(np.float32)).astype(np.float32) + np.float32(bias)).astype(np.float32)


def round_trip_moves(codes: np.ndarray, scale: float, bias: float) -> int:
    """Codes that EuclideanCompressed::fix_argument's compression of the decompressed datum does not return."""
    return int((SQ.encode(decompress(codes, scale, bias), codes.dtype, scale, bias) != codes).sum())


def build_distances(oracle, metric: str, codes: np.ndarray, scale: float, bias: float, i: int) -> np.ndarray:
    """The build's distance from datum i (its own query) to every datum."""
    return SQ.distances(oracle, METRIC[metric], decompress(codes[i], scale, bias), codes, scale, bias)
