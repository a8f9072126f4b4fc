"""The host builder of the DCT coefficient tables (s2pb_dct_coefficients, the code dct_tables and the streamed K-panels use) against
the dense formulas evaluated one coefficient at a time with the C library's cos / sin (Python's math module), bit for bit, at widths
below, at and above the 8192 px of the tables the device keeps once per width.  No device needed."""
import math
import os

import numpy as np
import pytest

from s2p_b200 import _lib

pytestmark = pytest.mark.skipif(not os.path.exists(_lib.LIB_PATH), reason="libs2pb200.so is not built")

PI = 3.14159265358979323846264338327950288


def dense(kind, n, r, c):
    """the coefficient as the reference's DCT stand-in writes it (oracle/shim/fftw_shim.c): kind 0 REDFT10 [k][j], 1 REDFT01 [i][k],
    2 RODFT01 [i][k]"""
    if kind == 0:
        return 2.0 * math.cos(PI * (c + 0.5) * r / n)
    if kind == 1:
        return 1.0 if c == 0 else 2.0 * math.cos(PI * c * (r + 0.5) / n)
    return ((-1.0 if r & 1 else 1.0) if c == n - 1 else 2.0 * math.sin(PI * (c + 1) * (r + 0.5) / n))


@pytest.mark.parametrize("n", [2, 17, 1000, 8192, 8193, 12288, 16384])
@pytest.mark.parametrize("kind", [0, 1, 2])
def test_blocks_equal_the_dense_formula(kind, n):
    from s2p_b200.engine import dct_coefficients
    rng = np.random.default_rng(n * 3 + kind)
    # a block at each corner and one inside, so that the first and last row and column are covered
    starts = {(0, 0), (max(0, n - 40), max(0, n - 40)), (0, max(0, n - 40))}
    starts.add((int(rng.integers(0, max(1, n - 40))), int(rng.integers(0, max(1, n - 40)))))
    for r0, c0 in starts:
        rows, cols = range(r0, min(n, r0 + 40)), range(c0, min(n, c0 + 40))
        got = dct_coefficients(kind, n, rows, cols)
        want = np.array([[dense(kind, n, r, c) for c in cols] for r in rows])
        assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), "n %d block (%d, %d)" % (n, r0, c0)


def test_panel_of_many_rows_equals_the_formula():
    """a panel built on the thread pool (rows split between threads) equals the formula in every row"""
    from s2p_b200.engine import dct_coefficients
    n = 9000
    got = dct_coefficients(0, n, range(0, n), range(4096, 4112))
    rows = np.random.default_rng(1).integers(0, n, 64)
    want = np.array([[dense(0, n, int(r), c) for c in range(4096, 4112)] for r in rows])
    assert np.array_equal(got[rows].view(np.uint64), want.view(np.uint64))


def test_arguments():
    from s2p_b200.engine import S2pbError, dct_coefficients
    for kind, n, rows, cols in ((3, 10, range(0, 1), range(0, 1)), (0, 0, range(0, 0), range(0, 0)),
                                (0, 10, range(5, 11), range(0, 1)), (1, 10, range(0, 1), range(9, 12))):
        with pytest.raises(S2pbError) as e:
            dct_coefficients(kind, n, rows, cols)
        assert e.value.code == _lib.ERR_ARG
