"""The localisation of a height map on the GPU (s2pb_height_map_to_xyz, csrc/triangulation_kernels.cuh) and the
height_map_to_xyz drop-in built on it.

The contract: lon / lat within 1e-9 degree of the reference's own rpc_localization (the tolerance of test_triangulation.py),
the third coordinate the input height bit for bit, NaN in all three exactly where the height is NaN, and, where the camera
iterates, every point projected back within the iteration's own stopping test (squared normalised residual <= 1e-18).
Projected to UTM: within 2e-4 m of the oracle's lon / lat carried through the exact map of tests/utm_oracle.py (1e-9 degree
is at most 1.2e-4 m on the ground, plus the projection's 1e-6 m)."""
import sys
import types

import numpy as np
import pytest

import dsm_oracle as D
import localization_oracle as LO
import utm_oracle as U
from util import same

pytestmark = pytest.mark.gpu

TOL_DEG = 1e-9
TOL_UTM = 2e-4
ZONE = 31                     # EPSG:32631, the expected DSM's CRS


def _check_zone0(got, heights, rpc, ox, oy, want):
    nan = np.isnan(heights)
    assert got.shape == heights.shape + (3,) and got.dtype == np.float64
    assert np.array_equal(np.isnan(got).all(axis=2), nan) and np.isfinite(got[~nan]).all()
    assert same(got[..., 2], heights.astype(np.float64))
    ok = ~want.nan.ravel()[want.idx]
    assert ok.sum() > 0.7 * len(want.idx)
    assert np.abs(want.values_of(got[..., :2])[ok] - want.val[ok]).max() < TOL_DEG
    if not np.isfinite(rpc.numx[0]):            # no direct polynomials: every point comes out of the iteration
        rows, cols = np.nonzero(~nan)
        r2 = LO.residual2(rpc, cols + ox, rows + oy, heights[~nan], got[~nan][:, 0], got[~nan][:, 1])
        assert r2.max() <= LO.STOP


@pytest.mark.parametrize("name", ["synthetic_iterative", "synthetic_direct", "triplet"])
def test_localisation_matches_rpc_localization(engine, name):
    heights, rpc, ox, oy, want = LO.ref_sampled(name)
    before = engine.kernel_launches()
    got = engine.height_map_to_xyz(heights, rpc, ox, oy)
    assert engine.kernel_launches() == before + 1
    _check_zone0(got, heights, rpc, ox, oy, want)


def test_utm_on_the_triplet(engine):
    heights, rpc, ox, oy, want = LO.ref_sampled("triplet")
    before = engine.kernel_launches()
    got = engine.height_map_to_xyz(heights, rpc, ox, oy, ZONE, False)
    assert engine.kernel_launches() == before + 2
    nan = np.isnan(heights)
    assert np.array_equal(np.isnan(got).all(axis=2), nan) and np.isfinite(got[~nan]).all()
    assert same(got[..., 2], heights.astype(np.float64))
    ok = ~want.nan.ravel()[want.idx]
    lonlat = want.val[ok]
    lla = np.column_stack([lonlat, np.zeros(len(lonlat))])
    mine = want.values_of(got)[ok]
    assert np.abs(mine[:, :2] - U.restate(lla, ZONE, False)[:, :2]).max() < TOL_UTM
    pick = np.linspace(0, len(lonlat) - 1, 24).astype(int)
    assert np.abs(mine[pick, :2] - U.truth_array(lonlat[pick], ZONE, False)).max() < TOL_UTM
    # the projection is the one s2pb_lonlat_to_utm runs, applied to the zone-0 output on the device
    assert same(got, engine.lonlat_to_utm(engine.height_map_to_xyz(heights, rpc, ox, oy), ZONE, False))


def test_engine_arguments(engine):
    from s2p_b200._lib import ERR_ARG, S2pbError
    heights, rpc, ox, oy = LO.cases()["synthetic_iterative"]
    for zone in (-1, 61):
        with pytest.raises(S2pbError) as e:
            engine.height_map_to_xyz(heights, rpc, ox, oy, zone)
        assert e.value.code == ERR_ARG
    with pytest.raises(ValueError):
        engine.height_map_to_xyz(heights.ravel(), rpc, ox, oy)
    one = engine.height_map_to_xyz(heights[:1, :1], rpc, ox, oy)
    assert same(one, engine.height_map_to_xyz(heights, rpc, ox, oy)[:1, :1])


# ---------------------------------------------------------------- the drop-in

def _tiff(tmp_path, heights, name="height_map.tif"):
    from s2p_b200 import rasterio_compat
    path = str(tmp_path / name)
    rasterio_compat.write_float_tiff(path, heights)
    return path


def test_drop_in_reads_the_file(engine, tmp_path):
    from s2p_b200.triangulation import height_map_to_xyz
    t = LO.triplet()
    rpc = LO.triplet_rpc()
    path = _tiff(tmp_path, t["heights"])
    ox, oy = t["off"]
    got = height_map_to_xyz(path, rpc, int(ox), int(oy), "epsg:32631", engine=engine)
    assert same(got, engine.height_map_to_xyz(t["heights"], rpc, ox, oy, ZONE, False))
    for crs in (None, "EPSG:4979", 4326):
        assert same(height_map_to_xyz(path, rpc, ox, oy, crs, engine=engine), engine.height_map_to_xyz(t["heights"], rpc, ox, oy))


def test_drop_in_keeps_a_float64_map(engine, tmp_path):
    """a float64 height map keeps its bits: the third coordinate is the stored value, not its float32 rounding"""
    import cv2
    from s2p_b200.triangulation import height_map_to_xyz
    heights, rpc, ox, oy = LO.cases()["synthetic_iterative"]
    z = heights.astype(np.float64) + 1e-6 / 3
    path = str(tmp_path / "height_map64.tif")
    assert cv2.imwrite(path, z)
    got = height_map_to_xyz(path, rpc, ox, oy, engine=engine)
    assert same(got[..., 2], z) and not same(got[..., 2], z.astype(np.float32).astype(np.float64))
    assert same(got, engine.height_map_to_xyz(z, rpc, ox, oy))


def test_drop_in_other_crs_without_pyproj(engine, tmp_path, monkeypatch):
    from s2p_b200._lib import ERR_UNSUPPORTED, S2pbError
    from s2p_b200.triangulation import height_map_to_xyz
    heights, rpc, ox, oy = LO.cases()["synthetic_iterative"]
    path = _tiff(tmp_path, heights)
    monkeypatch.setitem(sys.modules, "s2p", None)                   # s2p (and so its pyproj wrappers) not importable
    with pytest.raises(S2pbError) as e:
        height_map_to_xyz(path, rpc, ox, oy, "epsg:32631+5773", engine=engine)
    assert e.value.code == ERR_UNSUPPORTED


def test_drop_in_other_crs_through_pyproj(engine, tmp_path, monkeypatch):
    """a target the device does not serve: the GPU's lon, lat, alt go through s2p.geographiclib's pyproj calls, as in the
    reference (s2p/triangulation.py:207-213)"""
    from s2p_b200.triangulation import height_map_to_xyz
    heights, rpc, ox, oy = LO.cases()["synthetic_iterative"]
    path = _tiff(tmp_path, heights)
    calls = []

    def pyproj_transform(x, y, in_crs, out_crs, z=None):
        calls.append((x.copy(), y.copy(), in_crs, out_crs, z.copy()))
        return x * 2.0, y - 1.0, z + 3.0

    geo = types.ModuleType("s2p.geographiclib")
    geo.pyproj_crs = lambda p: "crs(%s)" % p
    geo.pyproj_transform = pyproj_transform
    pkg = types.ModuleType("s2p")
    pkg.geographiclib = geo
    monkeypatch.setitem(sys.modules, "s2p", pkg)
    monkeypatch.setitem(sys.modules, "s2p.geographiclib", geo)
    lla = engine.height_map_to_xyz(heights, rpc, ox, oy)
    xyz = height_map_to_xyz(path, rpc, ox, oy, "epsg:32631+5773", engine=engine)
    assert len(calls) == 1
    x, y, in_crs, out_crs, z = calls[0]
    assert in_crs == "crs(epsg:4979)" and out_crs == "epsg:32631+5773"
    flat = lla.reshape(-1, 3)
    assert same(x, flat[:, 0]) and same(y, flat[:, 1]) and same(z, flat[:, 2])
    assert same(xyz, np.stack([lla[..., 0] * 2.0, lla[..., 1] - 1.0, lla[..., 2] + 3.0], axis=2))


def test_installed_height_map_to_xyz_is_the_drop_in(engine, tmp_path, monkeypatch):
    from s2p_b200 import triangulation as T
    original = object()
    mod = types.ModuleType("s2p.triangulation")
    mod.lib = types.SimpleNamespace()
    mod.height_map_to_xyz = original
    pkg = types.ModuleType("s2p")
    pkg.triangulation = mod
    monkeypatch.setitem(sys.modules, "s2p", pkg)
    monkeypatch.setitem(sys.modules, "s2p.triangulation", mod)
    assert T.install() is mod and T.install() is mod
    assert mod.height_map_to_xyz is T.height_map_to_xyz and mod._s2pb_original_height_map_to_xyz is original
    t = LO.triplet()
    rpc = LO.triplet_rpc()
    got = mod.height_map_to_xyz(_tiff(tmp_path, t["heights"]), rpc, 400, 400, _Crs(32631))
    assert same(got, engine.height_map_to_xyz(t["heights"], rpc, 400, 400, ZONE, False))


class _Crs:
    """what the drop-in reads from a pyproj.CRS"""
    def __init__(self, code):
        self.code = code

    def to_epsg(self):
        return self.code


# ---------------------------------------------------------------- non-convergence

def _no_preimage_camera():
    """normalised col = lon^2 + 0.5 lon - height, row = lat (scale 100, no offsets): pixel (col, row) at height z has a
    preimage only where col / 100 - z / 100 >= -1/16, the minimum of the quadratic"""
    from s2p_b200.triangulation import RPCStruct
    r = RPCStruct()
    for k in range(20):
        r.numx[k] = r.denx[k] = r.numy[k] = r.deny[k] = np.nan
    r.inumx[7], r.inumx[1], r.inumx[3], r.idenx[0] = 1.0, 0.5, -1.0, 1.0
    r.inumy[2], r.ideny[0] = 1.0, 1.0
    for i in range(3):
        r.scale[i], r.iscale[i] = 100.0, 1.0
    r.delta = 1.0
    return r


def test_non_convergence_is_an_error(engine, tmp_path):
    from s2p_b200._lib import ERR_ARG, S2pbError
    from s2p_b200.triangulation import height_map_to_xyz
    rpc = _no_preimage_camera()
    z = np.zeros((8, 16))
    z[3, 5] = -50.0                                              # col 5: 0.05 + 0.5 < 1/16 below the minimum
    rows, cols = np.indices(z.shape)
    # on the CPU restatement: that pixel never meets the stopping test, and stays finite; every other one converges
    lon, lat, converged = LO.localize(rpc, cols, rows, z, maxit=5000)
    assert np.array_equal(~converged.reshape(z.shape), z != 0) and np.isfinite(lon).all() and np.isfinite(lat).all()
    with pytest.raises(S2pbError) as e:
        engine.height_map_to_xyz(z, rpc, 0, 0)
    assert e.value.code == ERR_ARG and "1 pixel" in str(e.value)
    with pytest.raises(S2pbError) as e:
        height_map_to_xyz(_tiff(tmp_path, z), rpc, 0, 0, "epsg:32631", engine=engine)
    assert e.value.code == ERR_ARG
    # without that pixel the same camera localises every point, as the restatement does
    z[3, 5] = np.nan
    got = engine.height_map_to_xyz(z, rpc, 0, 0)
    ok = ~np.isnan(z)
    lon, lat, converged = LO.localize(rpc, cols[ok], rows[ok], z[ok])
    assert converged.all()
    assert np.abs(got[ok][:, 0] - lon).max() < TOL_DEG and np.abs(got[ok][:, 1] - lat).max() < TOL_DEG
    assert LO.residual2(rpc, cols[ok], rows[ok], z[ok], got[ok][:, 0], got[ok][:, 1]).max() <= LO.STOP


# ---------------------------------------------------------------- georeferencing, end to end

def test_triplet_lands_on_the_expected_dsm(engine):
    """The fixture crop localised into EPSG:32631 and rasterised by s2pb_plyflatten on the grid of the expected DSM's window.
    The DSM comes from both pairs' merged, filtered heights and the crop is one height map, so they differ; the statistics of
    that difference were computed on the CPU (oracle localisation, tests/dsm_oracle.py) when the fixture was made.  The GPU's
    points are within 2e-4 m of the oracle's, so only a point within that distance of a cell edge can change cell: the
    common cells within 0.5 %, the median within 1 cm and the 99th percentile within 5 cm of the recorded values."""
    from s2p_b200 import _lib
    t = LO.triplet()
    xyz = engine.height_map_to_xyz(t["heights"], LO.triplet_rpc(), t["off"][0], t["off"][1], ZONE, False)
    pts = xyz.reshape(-1, 3)
    pts = np.ascontiguousarray(pts[np.isfinite(pts).all(axis=1)])
    win = t["dsm"]
    xoff, yoff, r = float(t["dsm_xoff"]), float(t["dsm_yoff"]), float(t["dsm_res"])
    ysize, xsize = win.shape
    assert (D.cells(pts[:, 0], pts[:, 1], xoff, yoff, r, xsize, ysize) >= 0).all()         # the footprint is inside the window
    records = pts.view(np.uint8).reshape(len(pts), 24)
    got = engine.plyflatten([records], 24, [(0, _lib.PLY_F64), (8, _lib.PLY_F64), (16, _lib.PLY_F64)], xoff, yoff, r, xsize,
                            ysize)[..., 0]
    both = np.isfinite(got) & np.isfinite(win)
    dz = np.abs(got[both].astype(np.float64) - win[both])
    assert abs(both.sum() - int(t["dz_cells"])) <= 0.005 * int(t["dz_cells"])
    assert abs(np.median(dz) - float(t["dz_median"])) <= 0.01
    assert abs(np.percentile(dz, 99) - float(t["dz_p99"])) <= 0.05
