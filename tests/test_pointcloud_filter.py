"""The 3D outlier filter of triangulation (count_3d_neighbors, remove_isolated_3d_points, filter_xyz; c/disp_to_h.c:143-230,
s2p/triangulation.py:275-343) against the reference's own functions (oracle/_ref/libdisp_to_h_ref.so live, or the
digests recorded from it in tests/golden/pointcloud_ref_outputs.json) and against a numpy restatement
(tests/pointcloud_oracle.py).  Every comparison is bit for bit.

Without a device: the restatement, in particular the reading of the reference's repeated sweeps as reachability, is
pinned to the reference, and every GPU case below has a reference output.  On the GPU: counts, rejection, the rounding
of the distance, real imagery and the drop-in adapter."""
import sys
import types

import numpy as np
import pytest

import pointcloud_oracle as P
from oracle.oracle import digest

gpu = pytest.mark.gpu


# ---------------------------------------------------------------- cases

def _cloud(name):
    """the clouds of the cases, by name (seeded)"""
    if name == "small":
        return P.utm_cloud(40, 53, 1)
    if name == "small_nanborder":
        return P.utm_cloud(40, 53, 2, nan_border=2)
    if name == "tile":
        return P.utm_cloud(131, 257, 3)
    if name == "tile_nanborder":
        return P.utm_cloud(131, 257, 4, nan_border=3)
    if name == "row":
        return P.utm_cloud(1, 700, 5)
    if name == "column":
        return P.utm_cloud(700, 1, 6)
    if name == "tiny":
        return P.utm_cloud(37, 61, 7)
    if name == "full":
        return P.utm_cloud(1024, 1024, 8)
    if name == "serpentine":
        return P.serpentine()
    if name == "pins":
        return P.rounding_pins()[0]
    raise KeyError(name)


_clouds = {}


def cloud(name):
    if name not in _clouds:
        _clouds[name] = _cloud(name)
    return _clouds[name].copy()


# (cloud, r, p): tile-unaligned shapes, 1xN and Nx1, p from 0 to the shared-memory limit of one CTA and past it
# (a 16x16 tile with a halo of p stages (16 + 2p)^2 x 24 bytes: p = 20 needs the opt-in above 48 KB, p = 45 does not fit
# the 227 KB of an H100 and reads through L1 / L2), empty windows, a window wider than the image
GPU_COUNTS = ([(c, r, p) for c in ("tile", "row", "column") for r in (0.5, 5.0) for p in (0, 1, 3, 10)] +
              [("tile", 5.0, 20), ("tile", 5.0, 40), ("tile", 5.0, 45), ("tile_nanborder", 5.0, 3),
               ("tile_nanborder", 0.5, 10), ("tiny", 5.0, -1), ("tiny", 5.0, 300), ("tiny", 0.0, 2), ("full", 5.0, 10)])
# (cloud, r, p, n, q)
GPU_REMOVALS = ([("tile", 5.0, 5, n, q) for q in (0, 1, 2) for n in (0, 1, 5, 50)] +
                [("tile", 0.5, 3, 5, 1), ("tile_nanborder", 5.0, 10, 50, 1), ("tile", 5.0, 3, 5, -1)] +
                [("serpentine", 5.0, 3, 5, q) for q in (0, 1, 2)] + [("tile", 5.0, 10, 50, 1), ("full", 5.0, 10, 50, 1)])
# (cloud, r, p, n, q) where the restatement runs too
CPU_REMOVALS = ([("small", 5.0, 3, n, q) for q in (0, 1, 2) for n in (-2, 0, 1, 5, 30, 50)] +
                [("small", 0.5, 3, 5, q) for q in (0, 1, 2)] + [("small_nanborder", 5.0, 2, 20, 1), ("small", 5.0, 2, 1000, 1)] +
                [("serpentine", 5.0, 3, 5, q) for q in (0, 1, 2)])
CPU_COUNTS = [(c, r, p) for c in ("small", "small_nanborder") for r in (0.5, 5.0) for p in (-1, 0, 1, 3, 10)] + [("pins", 5.0, 1)]


def _id(case):
    return "-".join(str(x) for x in case)


# ---------------------------------------------------------------- without a device

@pytest.mark.parametrize("case", CPU_COUNTS, ids=_id)
def test_restated_counts_match_reference(case):
    name, r, p = case
    xyz = cloud(name)
    assert digest(P.count_restated(xyz, r, p)) == P.ref_count_output(xyz, r, p)


@pytest.mark.parametrize("case", CPU_REMOVALS, ids=_id)
def test_reachability_matches_reference_sweeps(case):
    """the reference's sweeps until nothing changes == saving exactly what a chain of close rejected points joins to a
    kept point"""
    name, r, p, n, q = case
    xyz = cloud(name)
    assert digest(P.remove_restated(xyz, r, p, n, q)) == P.ref_remove_output(xyz, r, p, n, q)


def test_cases_cover_what_they_claim():
    small = cloud("small")
    assert P.reference_sweeps(cloud("serpentine"), 5.0, 3, 5, 1) > 100        # many sweeps, one step of the chain each
    out = P.remove_restated(cloud("serpentine"), 5.0, 3, 5, 1)
    assert np.isnan(out).all(axis=2).sum() > 200 and np.isfinite(out[-5, :]).all()    # the chain itself survives
    assert np.isnan(P.remove_restated(small, 5.0, 2, 1000, 1)).all()                   # everything rejected
    assert np.array_equal(np.isnan(P.remove_restated(small, 5.0, 3, 0, 1)), np.isnan(small))   # nothing rejected
    part = np.isnan(small).any(axis=2) & ~np.isnan(small).all(axis=2)
    assert part.any()                                                                  # points with one NaN coordinate
    assert np.isnan(P.remove_restated(small, 5.0, 3, 1, 1)[part]).all()                # ... count 0 and go entirely


def test_rounding_pins_classify_as_designed():
    """each pin pair is close under the reference build's distance and not under the named wrong one, or the reverse;
    the reference library's own counts agree (live, or through the recorded digest)"""
    xyz, kinds = P.rounding_pins()
    alt = P.pin_alternatives(xyz)
    for k, kind in enumerate(kinds):
        assert alt["ours"][k] != alt[kind][k], (k, kind)
    assert sorted(set(kinds)) == ["double", "float_xyz", "unfused"]
    assert len(set(alt["ours"].tolist())) == 2                                        # both answers occur
    want = np.ones((2, len(kinds)), np.int32) + alt["ours"][None, :]
    assert digest(want) == P.ref_count_output(xyz, 5.0, 1)


def test_every_gpu_case_has_a_reference_output():
    for name, r, p in GPU_COUNTS:
        P.ref_count_output(cloud(name), r, p)
    for name, r, p, n, q in GPU_REMOVALS:
        P.ref_remove_output(cloud(name), r, p, n, q)


def test_argument_checks():
    """what the reference's ndpointer(c_double, shape=(h, w, 3)) argument types refuse, refused before any device call"""
    from s2p_b200.engine import Engine
    from s2p_b200.triangulation import _check_cloud
    good = np.zeros((4, 5, 3))
    assert Engine._cloud(good) is good
    with pytest.raises(TypeError):
        Engine._cloud(good.astype(np.float32))
    with pytest.raises(ValueError):
        Engine._cloud(np.zeros((4, 5, 2)))
    with pytest.raises(ValueError):
        Engine._cloud(np.zeros((4, 15)))
    _check_cloud(good, 5, 4)
    for bad in (good.astype(np.float32), good[:, ::-1], np.zeros((5, 4, 3)), good.tolist()):
        with pytest.raises(TypeError):
            _check_cloud(bad, 5, 4)


# ---------------------------------------------------------------- on the GPU

@gpu
@pytest.mark.parametrize("case", GPU_COUNTS, ids=_id)
def test_counts_match_reference(engine, case):
    name, r, p = case
    xyz = cloud(name)
    got = engine.count_3d_neighbors(xyz, r, p)
    assert got.dtype == np.int32 and got.shape == xyz.shape[:2]
    assert digest(got) == P.ref_count_output(xyz, r, p)


@gpu
def test_counts_rounding_pins(engine):
    xyz, kinds = P.rounding_pins()
    got = engine.count_3d_neighbors(xyz, 5.0, 1)
    assert np.array_equal(got[0] - 1, P.pin_alternatives(xyz)["ours"].astype(np.int32))
    assert digest(got) == P.ref_count_output(xyz, 5.0, 1)


@gpu
@pytest.mark.parametrize("case", GPU_REMOVALS, ids=_id)
def test_removal_matches_reference(engine, case):
    name, r, p, n, q = case
    xyz = cloud(name)
    before = np.isnan(xyz).any(axis=2)
    got = engine.remove_isolated_3d_points(xyz, r, p, n, q)
    assert got is xyz                                                     # in place
    removed = np.isnan(got).any(axis=2) & ~before
    assert np.isnan(got[removed]).all()                                   # all three coordinates
    assert digest(got) == P.ref_remove_output(cloud(name), r, p, n, q)


@gpu
def test_python_interface_in_place(engine):
    """as s2p's own functions: a C-contiguous float64 cloud is filtered in place, any other is left as it is"""
    from s2p_b200 import triangulation as T
    xyz = cloud("tile")
    want = P.ref_remove_output(cloud("tile"), 5.0, 5, 50, 1)
    a = xyz.copy()
    assert T.remove_isolated_3d_points(a, 5.0, 5, 50, engine=engine) is None
    assert digest(a) == want
    f = np.asfortranarray(xyz)
    T.remove_isolated_3d_points(f, 5.0, 5, 50, engine=engine)
    assert digest(f) == digest(xyz)
    b = xyz.copy()
    T.filter_xyz(b, 5.0, 50, 0.5, engine=engine)                          # p = ceil(5 / 0.5) = 10, q = 1
    assert digest(b) == P.ref_remove_output(xyz, 5.0, 10, 50, 1)
    assert digest(T.count_3d_neighbors(xyz, 5.0, 3, engine=engine)) == P.ref_count_output(xyz, 5.0, 3)
    with pytest.raises(TypeError):
        T.count_3d_neighbors(xyz.astype(np.float32), 5.0, 3, engine=engine)
    empty = np.zeros((0, 7, 3))
    assert T.count_3d_neighbors(empty, 5.0, 3, engine=engine).shape == (0, 7)
    T.remove_isolated_3d_points(empty, 5.0, 3, 5, engine=engine)


def _real_cloud(engine):
    """The reference's Pleiades pair (tests/golden/real_pair*.npz) triangulated by the engine, lon / lat mapped to metres by
    a fixed equirectangular projection about the RPC's offset, moved to UTM-like magnitudes and rounded to the millimetre
    (so that the cloud, which keys the recorded reference output, does not depend on the last bits of the triangulation)."""
    from s2p_b200.triangulation import disp_to_lonlatalt, rpc_from_geotiff_tag
    from util import load_real_pair
    z = load_real_pair()
    rpc1, rpc2 = rpc_from_geotiff_tag(z["rpc1"]), rpc_from_geotiff_tag(z["rpc2"])
    disp = z["rectified_disp"]
    mask = np.isfinite(disp).astype(np.float32)
    lla, _ = disp_to_lonlatalt(np.nan_to_num(disp), mask, np.ones((1024, 1024), np.float32), z["H1"], z["H2"], rpc1, rpc2,
                               (0.0, 1023.0, 0.0, 1023.0), engine=engine)
    lat0, lon0 = float(z["rpc1"][4]), float(z["rpc1"][5])
    m = 6378137.0 * np.pi / 180.0
    x = 340000.0 + (lla[..., 0] - lon0) * m * np.cos(np.radians(lat0))
    y = 7660000.0 + (lla[..., 1] - lat0) * m
    return np.round(np.stack([x, y, lla[..., 2]], axis=2), 3)


@gpu
def test_real_pair(engine):
    xyz = _real_cloud(engine)
    assert 0.5 < np.isfinite(xyz).all(axis=2).mean() < 1
    p = int(np.ceil(5 / 0.5))                                             # filter_xyz at a Pleiades GSD of 0.5 m
    want_c, want = P.ref_count_output(xyz, 5.0, p), P.ref_remove_output(xyz, 5.0, p, 50, 1)
    assert digest(engine.count_3d_neighbors(xyz, 5.0, p)) == want_c
    got = engine.remove_isolated_3d_points(xyz.copy(), 5.0, p, 50, 1)
    assert digest(got) == want
    removed = np.isnan(got).any(axis=2) & ~np.isnan(xyz).any(axis=2)
    assert removed.any()


@gpu
def test_drop_in_adapter(engine, monkeypatch):
    """s2p's own calls (s2p/triangulation.py:293-299,324-328) through the adapter install() puts in place of its library"""
    import ctypes
    from numpy.ctypeslib import ndpointer
    from s2p_b200 import triangulation as T
    original = ctypes.CDLL(P.REF_LIB) if P.have_ref() else types.SimpleNamespace(stereo_corresp_to_lonlatalt=object())
    mod = types.ModuleType("s2p.triangulation")
    mod.lib = original
    pkg = types.ModuleType("s2p")
    pkg.triangulation = mod
    monkeypatch.setitem(sys.modules, "s2p", pkg)
    monkeypatch.setitem(sys.modules, "s2p.triangulation", mod)
    assert T.install() is mod and isinstance(mod.lib, T._LibAdapter)
    lib = mod.lib
    assert lib.stereo_corresp_to_lonlatalt is original.stereo_corresp_to_lonlatalt
    xyz = cloud("tile")
    h, w = xyz.shape[:2]
    r, p, n, q = 5.0, np.ceil(5.0 / 0.5).astype(int), 50, 1
    lib.count_3d_neighbors.argtypes = (ndpointer(dtype=ctypes.c_int, shape=(h, w)), ndpointer(dtype=ctypes.c_double, shape=(h, w, 3)),
                                       ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_int)
    out = np.zeros((h, w), dtype="int32")
    lib.count_3d_neighbors(out, np.ascontiguousarray(xyz), w, h, r, p)
    assert np.array_equal(out, engine.count_3d_neighbors(xyz, r, p))
    assert digest(out) == P.ref_count_output(xyz, r, p)
    lib.remove_isolated_3d_points.argtypes = (ndpointer(dtype=ctypes.c_double, shape=(h, w, 3)),
                                              ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_int, ctypes.c_int, ctypes.c_int)
    a = np.ascontiguousarray(xyz.copy())
    lib.remove_isolated_3d_points(a, w, h, r, p, n, q)
    assert digest(a) == digest(engine.remove_isolated_3d_points(xyz.copy(), r, p, n, q)) == P.ref_remove_output(xyz, r, p, n, q)
    r64 = 5.0000001                                                       # rounded to float32 on the way, as c_float does
    lib.count_3d_neighbors(out, xyz, w, h, r64, p)
    assert np.array_equal(out, engine.count_3d_neighbors(xyz, np.float32(r64), p))
