import os

import numpy as np

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load_real_pair():
    """The real-imagery fixture (tests/golden/make_golden_real_pair.py), stored in three files of less than 1 MB each."""
    z = {}
    for name in ("real_pair", "real_pair_rectified_ref", "real_pair_rectified_disp"):
        z.update(np.load(os.path.join(GOLD, name + ".npz")))
    return z


def same(a, b):
    """bit-equality with NaN == NaN"""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape:
        return False
    if a.dtype.kind == "f":
        return bool(np.all((a == b) | (np.isnan(a) & np.isnan(b))))
    return bool(np.array_equal(a, b))


def nmismatch(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype.kind == "f":
        return int((~((a == b) | (np.isnan(a) & np.isnan(b)))).sum())
    return int((a != b).sum())
