"""The entry points that take host buffers borrow their device scratch from the context's pool, which keeps buffers between
calls.  A reused buffer still holds another call's data, and a call that fails on its arguments must still give its buffers
back.  Every result here is compared with the oracle, bit for bit where the stage's own test is."""
import ctypes

import numpy as np
import pytest

from s2p_b200.synth import make_pair
from util import nmismatch, same

pytestmark = pytest.mark.gpu
H, W, DMIN, DMAX = 41, 67, -9, 10
D = DMAX - DMIN + 1


def _cc_input(h, w, seed):
    """piecewise-constant levels 6 apart with noise and 15 % NaN: many components, most of them smaller than 25 px"""
    rng = np.random.default_rng(seed)
    a = (rng.integers(0, 4, size=(h, w)) * 6).astype(np.float32) + rng.normal(0, 0.5, (h, w)).astype(np.float32)
    a[rng.random((h, w)) < 0.15] = np.nan
    return a


@pytest.mark.parametrize("h,w", [(60, 80), (120, 160), (300, 500)])
def test_remove_small_cc(engine, oracle, h, w):
    a = _cc_input(h, w, seed=h)
    want = oracle.port.remove_small_cc(a, 25)
    assert np.isnan(want).sum() > np.isnan(a).sum()
    got = engine.remove_small_cc(a, 25)
    assert same(got, want), "%d px differ" % nmismatch(got, want)


def _ranges(seed):
    """the full range with a ragged block, so that the volumes hold labels outside a pixel's range"""
    rng = np.random.default_rng(seed)
    lo, hi = np.full((H, W), DMIN, np.int32), np.full((H, W), DMAX, np.int32)
    y, x = rng.integers(0, H - 6), rng.integers(0, W - 20)
    lo[y:y + 5, x:x + 18] = DMIN + 2
    hi[y:y + 5, x:x + 18] = DMIN + 5
    return lo, hi


def _assert_same(name, got, want):
    for k, (g, o) in enumerate(zip(got, want)):
        assert same(g, o), "%s: output %d differs at %d elements" % (name, k, nmismatch(g, o))


def _stage(name, k, engine, oracle):
    """One call of the entry point `name` on the k-th seeded input (the same shape for every k), checked against the oracle."""
    nodata = name in ("census", "median", "rejection_mask")      # the cost and aggregation stages take NaN-free images
    ref, sec, gt = make_pair(H, W, DMIN, DMAX, seed=70 + k, nan_border=0.05 if nodata else 0.0)
    lo, hi = _ranges(k)
    rng = np.random.default_rng(k)
    if name == "census":
        _assert_same(name, [engine.census(ref, 5)], [oracle.port.census(ref, 5)])
    elif name == "costvolume":
        _assert_same(name, [engine.costvolume(ref, sec, lo, hi, DMIN, D, 5)], [oracle.port.costvolume(ref, sec, lo, hi, DMIN, D, 5)])
    elif name == "costvolume_dist":
        _assert_same(name, [engine.costvolume(ref, sec, lo, hi, DMIN, D, 5, cost="ncc")],
                     [oracle.port.costvolume(ref, sec, lo, hi, DMIN, D, 5, cost="ncc")])
    elif name == "aggregate":
        C = oracle.port.costvolume(ref, sec, lo, hi, DMIN, D, 5)
        _assert_same(name, engine.aggregate(C, lo, hi, DMIN, 8.0, 32.0, 8, 3), oracle.port.aggregate(C, lo, hi, DMIN, 8.0, 32.0, 8, 3))
    elif name == "aggregate_w":
        C = oracle.port.costvolume(ref, sec, lo, hi, DMIN, D, 5, cost="btad")
        wgt = rng.uniform(0.2, 1.0, (H, W)).astype(np.float32)
        _assert_same(name, engine.aggregate(C, lo, hi, DMIN, 12.0, 48.0, 8, 3, weights=wgt, general=True),
                     oracle.port.aggregate(C, lo, hi, DMIN, 12.0, 48.0, 8, 3, weights=wgt))
    elif name == "median":
        _assert_same(name, [engine.median(ref, 2)], [oracle.port.median(ref, 2)])
    elif name == "remove_small_cc":
        a = _cc_input(H, W, seed=k)
        _assert_same(name, [engine.remove_small_cc(a, 25)], [oracle.port.remove_small_cc(a, 25)])
    elif name == "rejection_mask":
        d = gt + rng.uniform(-0.7, 0.7, gt.shape).astype(np.float32)
        d[rng.random(d.shape) < 0.1] = np.nan
        _assert_same(name, [engine.rejection_mask(d, ref, sec)], [oracle.port.rejection_mask(d, ref, sec)])
    elif name == "erode_mask":
        # the inputs of test_fusion.py's erosion test: the reference's outputs are recorded for them
        radius = (2, 3)[k]
        m = (np.random.default_rng(radius).random((61, 83)) > 0.15).astype(np.uint8)
        live = (lambda: {"eroded": oracle.ref_disk_erosion(m.astype(np.float32), radius).astype(np.uint8)}) if oracle.have_ref_morsi() else None
        assert oracle.digest(engine.erode_mask(m, radius)) == oracle.recorded(oracle.call_key("morsi", (radius,), [m]), live)["eroded"]
    elif name == "disp_to_lonlatalt":
        # the inputs of test_triangulation.py (recorded likewise), with and without the direct RPC model
        from s2p_b200.triangulation import disp_to_lonlatalt
        from test_triangulation import _assert_close, _geometry, _rpc
        r = np.random.default_rng(5)
        rpc1, rpc2 = _rpc(1, bool(k)), _rpc(2, bool(k))
        disp = r.normal(0, 6, (60, 90)).astype(np.float32)
        mask = (r.random((60, 90)) > 0.2).astype(np.float32)
        H1, H2, bbx = _geometry()
        mo = (r.random((int(bbx[3] - bbx[2]) + 1, int(bbx[1] - bbx[0]) + 1)) > 0.1).astype(np.float32)
        want, werr = oracle.ref_disp_to_lonlatalt_sampled(disp, mask, mo, H1, H2, rpc1, rpc2, bbx)
        got, gerr = disp_to_lonlatalt(disp, mask, mo, H1, H2, rpc1, rpc2, bbx, engine=engine)
        _assert_close(want, werr, got, gerr, 0.3)
    else:
        raise ValueError(name)


STAGES = ["census", "costvolume", "costvolume_dist", "aggregate", "aggregate_w", "median", "remove_small_cc", "rejection_mask",
          "erode_mask", "disp_to_lonlatalt"]


@pytest.mark.parametrize("name", STAGES)
def test_reused_scratch_holds_no_stale_data(engine, oracle, name):
    """Two calls on different inputs of one shape, with a call of another entry point between them: the second call gets
    pooled buffers that hold the data of both earlier calls."""
    other = STAGES[(STAGES.index(name) + 1) % len(STAGES)]
    _stage(name, 0, engine, oracle)
    _stage(other, 0, engine, oracle)
    _stage(name, 1, engine, oracle)


def test_argument_errors_give_their_scratch_back(engine, oracle):
    """Calls that fail with S2PB_ERR_ARG after they have taken scratch, each followed by the same call with valid arguments."""
    from oracle import fusion_oracle as F
    from s2p_b200 import _lib
    from s2p_b200.engine import S2pbError
    from test_gpu_homography import CASES, REL_TOL, _src

    ref, sec, _ = make_pair(H, W, DMIN, DMAX, seed=80)
    lo, hi = _ranges(80)
    bad = hi.copy()
    bad[H // 2, W // 2] = DMAX + 1
    with pytest.raises(S2pbError) as e:
        engine.costvolume(ref, sec, lo, bad, DMIN, D, 5)
    assert e.value.code == _lib.ERR_ARG
    _assert_same("costvolume", [engine.costvolume(ref, sec, lo, hi, DMIN, D, 5)], [oracle.port.costvolume(ref, sec, lo, hi, DMIN, D, 5)])

    src = _src()
    with pytest.raises(S2pbError) as e:          # the output's pre-image lies left of the source: an empty region of interest
        engine.homography(src, np.array([[1.0, 0, 1e5], [0, 1, 0], [0, 0, 1]]), 256, 200)
    assert e.value.code == _lib.ERR_ARG
    want = oracle.ref_homography_sampled(src, CASES["rot10"], 256, 200)
    got = engine.homography(src, CASES["rot10"], 256, 200)
    assert int((want.nan != np.isnan(got)).sum()) <= 2
    g = want.values_of(got)
    both = np.isfinite(want.val) & np.isfinite(g)
    assert both.any() and np.abs(want.val[both] - g[both]).max() <= REL_TOL * np.nanmax(np.abs(src))

    rng = np.random.default_rng(3)
    maps = [rng.normal(100, 5, (H, W)).astype(np.float32) for _ in range(3)]
    offsets = [0.5, 1.5, 2.5]
    out = np.empty((H, W), np.float32)
    ptrs = (ctypes.c_void_p * 3)(maps[0].ctypes.data, None, maps[2].ctypes.data)
    rc = engine._L.s2pb_merge_n(engine._ctx, ptrs, (ctypes.c_double * 3)(*offsets), 3, W, H, 0, 3.0,
                                out.ctypes.data_as(ctypes.POINTER(ctypes.c_float)))
    assert rc == _lib.ERR_ARG
    got = engine.merge_n(maps, offsets, "average_if_close", threshold=3, sub_f32=True)
    assert same(got, F.merge_port(maps, offsets, "average_if_close", 3, sub_f32=True))
