"""The census cost volume is stored as 8-bit codes (finite costs 0..127, csrc/agg_kernel.cuh).  s2pb_aggregate still takes
integer costs up to 2048: a volume whose costs fit the codes runs on them, one with a larger cost goes through the
float-cost flavour with unit weights.  Both must equal the oracle bit for bit."""
import numpy as np
import pytest

from s2p_b200.synth import make_pair
from util import nmismatch, same

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("tsgm", [1, 2, 3, 4])
@pytest.mark.parametrize("scale", [5, 11])      # census 5x5 costs are 0..24: x 5 stays within the codes (<= 120), x 11 does not (<= 264)
def test_aggregate_scaled_integer_costs(engine, oracle, tsgm, scale):
    h, w, dmin, dmax = 45, 70, -10, 13
    ref, sec, _ = make_pair(h, w, dmin, dmax, seed=5)
    lo, hi = np.full((h, w), dmin, np.int32), np.full((h, w), dmax, np.int32)
    lo[20:24, 30:50] = dmin
    hi[20:24, 30:50] = dmin + 1
    D = dmax - dmin + 1
    C = oracle.port.costvolume(ref, sec, lo, hi, dmin, D, 5) * np.float32(scale)
    assert np.nanmax(np.where(np.isinf(C), np.nan, C)) > (127 if scale == 11 else 24)
    So, do, co, fo = oracle.port.aggregate(C, lo, hi, dmin, 8.0, 32.0, 8, tsgm)
    Sg, dg, cg, fg = engine.aggregate(C, lo, hi, dmin, 8.0, 32.0, 8, tsgm)
    assert same(dg, do), "integer WTA index differs at %d pixels" % nmismatch(dg, do)
    assert same(fg, fo), "consensus differs at %d pixels" % nmismatch(fg, fo)
    assert same(Sg, So), "aggregated volume differs at %d voxels" % nmismatch(Sg, So)
    assert same(cg, co)
