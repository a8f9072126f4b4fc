"""The WTA that reads only the labels that can still win (wta_pruned_kernel, DESIGN.md 3.2: pass 0 read where C <= T,
passes 1-7 where L_0 <= T or C <= L_q[d0]) against wta_kernel on the same device: disparity, confidence, mask and right
disparity bit for bit, NaNs included.  S2PB_WTA_PRUNE is read when a context is created: unset selects the pruned kernel,
0 wta_kernel, so the two engines of this module differ in nothing else."""
import os

import numpy as np
import pytest

from s2p_b200.synth import make_pair

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engines():
    from s2p_b200.engine import Engine
    old = os.environ.get("S2PB_WTA_PRUNE")
    made = []
    try:
        os.environ.pop("S2PB_WTA_PRUNE", None)
        made.append(Engine(0))                  # the default: wta_pruned_kernel
        os.environ["S2PB_WTA_PRUNE"] = "0"
        made.append(Engine(0))                  # wta_kernel
    finally:
        if old is None:
            os.environ.pop("S2PB_WTA_PRUNE", None)
        else:
            os.environ["S2PB_WTA_PRUNE"] = old
    yield made
    for e in made:
        e.close()


def _tile(kind, h, w, dmin, dmax, seed):
    if kind == "constant":                      # every cost equal: nothing can be pruned
        return np.full((h, w), 100.0, np.float32), np.full((h, w), 100.0, np.float32)
    if kind == "ties":                          # a texture of period 4: many labels tie at the minimum
        row = np.tile(np.array([10, 200, 90, 1500], np.float32), w // 4 + 2)
        ref = np.tile(row[:w], (h, 1))
        return ref.copy(), np.tile(row[1:w + 1], (h, 1)).copy()
    ref, sec, _ = make_pair(h, w, dmin, dmax, seed=seed, nan_border=0.05 if kind == "nodata" else 0.0)
    return ref, sec


def _same_bits(a, b):
    return np.array_equal(a.view(np.int32), b.view(np.int32))


CASES = [
    # kind, shape, dmin, dmax, parameter overrides                      labels per lane of the left slab
    ("clean", (40, 64), -12, 11, {}),                                   # 1
    ("nodata", (40, 64), -12, 11, {}),
    ("clean", (36, 90), -20, 30, {}),                                   # 2
    ("clean", (40, 130), -64, 63, {}),                                  # 4
    ("nodata", (33, 140), -64, 63, {}),                                 # 4 left, 5 right (wta_kernel serves that view)
    ("clean", (24, 260), -128, 127, {}),                                # 8
    ("nodata", (24, 260), -120, 120, {}),                               # 8
    ("constant", (30, 140), -64, 63, {}),
    ("ties", (30, 140), -64, 63, {}),
    ("ties", (30, 140), -64, 63, dict(refine=2)),
    ("clean", (40, 130), -64, 63, dict(tsgm=1)),
    ("clean", (40, 130), -64, 63, dict(tsgm=2)),
    ("clean", (40, 130), -64, 63, dict(tsgm=4)),
    ("nodata", (40, 130), -64, 63, dict(census_win=3)),                 # scaled costs: the bound rounds
    ("nodata", (40, 130), -64, 63, dict(census_win=7)),
    ("clean", (40, 130), -64, 63, dict(census_win=3, tsgm=4, fix_overcount=0)),
    ("nodata", (40, 130), -64, 63, dict(fix_overcount=0)),
    ("clean", (40, 130), -64, 63, dict(refine=0, median=0, lr_mode=0)),
]


@pytest.mark.parametrize("kind,shape,dmin,dmax,kw", CASES)
def test_pruned_wta_equals_full_wta(engines, kind, shape, dmin, dmax, kw):
    from s2p_b200.engine import default_params
    h, w = shape
    ref, sec = _tile(kind, h, w, dmin, dmax, seed=h + w)
    p = default_params("mgm", **kw)
    new, old = (e.mgm(ref, sec, dmin, dmax, p, want_right=True) for e in engines)
    for k in ("disp", "conf", "disp_right"):
        assert _same_bits(new[k], old[k]), "%s differs at %d pixels" % (k, int((new[k].view(np.int32) != old[k].view(np.int32)).sum()))
    assert np.array_equal(new["mask"], old["mask"])


def test_pruned_wta_equals_full_wta_in_mgm_multi(engines):
    """every pyramid level and the half-pixel pass (ZOOMFACTOR 2) go through the same WTA"""
    from s2p_b200.engine import default_params
    ref, sec, _ = make_pair(130, 170, -14, 16, seed=5, nan_border=0.06)
    p = default_params("mgm_multi")
    new, old = (e.mgm(ref, sec, -14, 16, p, want_right=True) for e in engines)
    for k in ("disp", "conf", "disp_right"):
        assert _same_bits(new[k], old[k]), k


def test_pruned_wta_on_a_tile_of_many_warps(engines):
    """a tile with more pixels than the grid has warps: every warp runs its three-pixel-deep pipeline through several rounds
    and its tail (the last pixels of a warp, whose successors are past the end)"""
    from s2p_b200.engine import default_params
    ref, sec, _ = make_pair(256, 384, -64, 63, seed=11, nan_border=0.03)
    p = default_params("mgm")
    new, old = (e.mgm(ref, sec, -64, 63, p, want_right=True) for e in engines)
    for k in ("disp", "conf", "disp_right"):
        assert _same_bits(new[k], old[k]), k
