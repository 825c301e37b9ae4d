"""Builds flat_gt100.npz: the reference's 100-deep ground truth of its test dataset (data/test_dataset/
groundtruth_{euclidean,mip,cosine}.ivecs, 1000 queries x 100 ids each, over the 10 000 rows of test_dataset.npz),
stored as uint16.  Run once where the reference's sources are; the tests read only the npz.

    python tests/golden/make_flat_gt.py /path/to/reference
"""
import os
import sys

import numpy as np


def read_ivecs(path):
    raw = np.fromfile(path, dtype=np.int32)
    dim = int(raw[0])
    rows = raw.reshape(-1, dim + 1)
    assert (rows[:, 0] == dim).all()
    return rows[:, 1:]


def main(ref):
    out = {}
    for name, key in (("euclidean", "l2"), ("mip", "ip"), ("cosine", "cosine")):
        gt = read_ivecs(os.path.join(ref, "data", "test_dataset", f"groundtruth_{name}.ivecs"))
        assert gt.shape == (1000, 100) and gt.min() >= 0 and gt.max() < 10_000
        out[key] = gt.astype(np.uint16)
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "flat_gt100.npz"), **out)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/root/reference")
