"""The two-stage pruned WTA (wta_pruned2_kernel, DESIGN.md 3.2: pass 0 read where C <= T, passes 1-7 where L_0 <= T or
C <= L_q[d0]) against wta_kernel on the same device, on the cases of test_gpu_wta_prune.py: disparity, confidence, mask and
right disparity bit for bit, NaNs included.  S2PB_WTA_PRUNE is read when a context is created: 2 (the default) selects
the two-stage kernel, 0 wta_kernel."""
import os

import numpy as np
import pytest

from s2p_b200.synth import make_pair
from test_gpu_wta_prune import CASES, _same_bits, _tile

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engines():
    from s2p_b200.engine import Engine
    old = os.environ.get("S2PB_WTA_PRUNE")
    made = []
    try:
        for v in ("2", "0"):
            os.environ["S2PB_WTA_PRUNE"] = v
            made.append(Engine(0))
    finally:
        if old is None:
            os.environ.pop("S2PB_WTA_PRUNE", None)
        else:
            os.environ["S2PB_WTA_PRUNE"] = old
    yield made
    for e in made:
        e.close()


@pytest.mark.parametrize("kind,shape,dmin,dmax,kw", CASES)
def test_two_stage_wta_equals_full_wta(engines, kind, shape, dmin, dmax, kw):
    from s2p_b200.engine import default_params
    h, w = shape
    ref, sec = _tile(kind, h, w, dmin, dmax, seed=h + w)
    p = default_params("mgm", **kw)
    new, old = (e.mgm(ref, sec, dmin, dmax, p, want_right=True) for e in engines)
    for k in ("disp", "conf", "disp_right"):
        assert _same_bits(new[k], old[k]), "%s differs at %d pixels" % (k, int((new[k].view(np.int32) != old[k].view(np.int32)).sum()))
    assert np.array_equal(new["mask"], old["mask"])


def test_two_stage_wta_equals_full_wta_in_mgm_multi(engines):
    """every pyramid level and the half-pixel pass (ZOOMFACTOR 2) go through the same WTA"""
    from s2p_b200.engine import default_params
    ref, sec, _ = make_pair(130, 170, -14, 16, seed=5, nan_border=0.06)
    p = default_params("mgm_multi")
    new, old = (e.mgm(ref, sec, -14, 16, p, want_right=True) for e in engines)
    for k in ("disp", "conf", "disp_right"):
        assert _same_bits(new[k], old[k]), k


def test_two_stage_wta_on_a_tile_of_many_warps(engines):
    """a tile with more pixels than the grid has warps: every warp runs its three-pixel-deep pipeline through several rounds
    and its tail (the last pixels of a warp, whose successors are past the end)"""
    from s2p_b200.engine import default_params
    ref, sec, _ = make_pair(256, 384, -64, 63, seed=11, nan_border=0.03)
    p = default_params("mgm")
    new, old = (e.mgm(ref, sec, -64, 63, p, want_right=True) for e in engines)
    for k in ("disp", "conf", "disp_right"):
        assert _same_bits(new[k], old[k]), k
