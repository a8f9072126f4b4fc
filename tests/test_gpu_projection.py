"""WGS84 -> UTM on the GPU (csrc/projection_kernels.cuh) and the disp_to_xyz drop-in built on it.

The contract: x and y within 1e-6 m of the 50-digit truth of tests/utm_oracle.py, z bit for bit the altitude that comes in
(disp_to_lonlatalt's), the same NaN mask.  The float64 restatement of the kernel is within 1e-7 m of the truth
(tests/test_utm_oracle.py), so every point is held to 9e-7 m of the restatement, and a subset to 1e-6 m of the truth itself."""
import sys
import types

import numpy as np
import pytest

import utm_oracle as U
from util import same

pytestmark = pytest.mark.gpu

TOL_RESTATE = 9e-7
TOL_TRUTH = 1e-6


def _check(got, lla, zone, south, ntruth=0):
    want = U.restate(lla, zone, south)
    nan_got, nan_want = np.isnan(got), np.isnan(want)
    assert np.array_equal(nan_got, nan_want)
    fin = np.isfinite(want[..., 0])
    assert np.array_equal(np.isposinf(got), np.isposinf(want))
    assert same(got[..., 2][fin], lla[..., 2][fin])                              # the altitude passes through, bit for bit
    assert np.abs(got[..., :2][fin] - want[..., :2][fin]).max(initial=0) <= TOL_RESTATE
    if ntruth:
        pts = lla[fin].reshape(-1, 3)
        pick = np.linspace(0, len(pts) - 1, min(ntruth, len(pts))).astype(int)
        t = U.truth_array(pts[pick, :2], zone, south)
        assert np.abs(got[fin].reshape(-1, 3)[pick, :2] - t).max() <= TOL_TRUTH


def _points(seed, zone, n=4096):
    rng = np.random.default_rng(seed)
    lon0 = U.lon0_of(zone)
    p = np.stack([lon0 + rng.uniform(-4.0, 4.0, n), rng.uniform(-80.0, 84.0, n), rng.uniform(-500.0, 9000.0, n)], axis=1)
    edges = [[lon0 - 3.0, 0.0, 1.0], [lon0 + 3.0, 0.0, 2.0], [lon0 - 3.0, -80.0, 3.0], [lon0 + 3.0, 84.0, 4.0],
             [lon0, 0.0, 5.0], [lon0, -80.0, 6.0], [lon0, 84.0, 7.0], [lon0 + 4.0, 45.0, 8.0], [lon0 - 4.0, -45.0, 9.0]]
    return np.concatenate([p, np.array(edges)])


@pytest.mark.parametrize("zone,south", [(1, False), (1, True), (17, False), (31, True), (40, True), (60, False), (60, True)])
def test_lonlat_to_utm_matches_the_oracle(engine, zone, south):
    lla = _points(zone * 2 + south, zone)
    got = engine.lonlat_to_utm(lla, zone, south)
    assert got.shape == lla.shape and got.dtype == np.float64
    _check(got, lla, zone, south, ntruth=64)


def test_lonlat_to_utm_nan_domain_and_wrap(engine):
    lla = np.array([[57.0, -21.0, 100.0], [np.nan, -21.0, 1.0], [57.0, np.nan, 1.0], [57.0, -21.0, np.nan],
                    [np.nan, np.nan, np.nan], [57.0, 91.0, 3.0], [57.0, -90.5, 3.0],
                    [57.0 + 360.0, -21.0, 4.0], [57.0 - 360.0, -21.0, 5.0]])
    got = engine.lonlat_to_utm(lla, 40, True)
    _check(got, lla, 40, True)
    assert np.isnan(got[1:5]).all() and np.isposinf(got[5:7]).all()
    assert np.abs(got[7:, :2] - got[0, :2]).max() < 1e-6
    # zone 1 next to the antimeridian, from both sides
    lla = np.array([[179.5, 10.0, 0.0], [-179.5, 10.0, 0.0], [-177.0, -10.0, 0.0]])
    _check(engine.lonlat_to_utm(lla, 1, False), lla, 1, False, ntruth=3)


def test_lonlat_to_utm_shapes_and_arguments(engine):
    from s2p_b200._lib import ERR_ARG, S2pbError
    lla = _points(5, 31, 300).reshape(3, 103, 3)
    _check(engine.lonlat_to_utm(lla, 31, False), lla, 31, False)
    assert engine.lonlat_to_utm(np.zeros((0, 3)), 31, False).shape == (0, 3)
    for zone in (0, 61, -1):
        with pytest.raises(S2pbError) as e:
            engine.lonlat_to_utm(lla, zone, False)
        assert e.value.code == ERR_ARG
    with pytest.raises(ValueError):
        engine.lonlat_to_utm(np.zeros((4, 2)), 31, False)
    before = engine.kernel_launches()
    engine.lonlat_to_utm(lla, 31, False)
    assert engine.kernel_launches() == before + 1


def _real():
    from s2p_b200.triangulation import rpc_from_geotiff_tag
    from util import load_real_pair
    z = load_real_pair()
    disp = z["rectified_disp"]
    args = dict(rpc1=rpc_from_geotiff_tag(z["rpc1"]), rpc2=rpc_from_geotiff_tag(z["rpc2"]), H1=z["H1"], H2=z["H2"],
                disp=np.nan_to_num(disp), mask_rect=np.isfinite(disp).astype(np.float32), img_bbx=(0.0, 1023.0, 0.0, 1023.0),
                mask_orig=np.ones((1024, 1024), np.float32))
    return args


class _Crs:
    """what the drop-in reads from a pyproj.CRS"""
    def __init__(self, code):
        self.code = code

    def to_epsg(self):
        return self.code


@pytest.mark.parametrize("out_crs", [None, "epsg:4979", "EPSG:4326", "epsg:32740", 32740, _Crs(32740)])
def test_disp_to_xyz_real_pair(engine, out_crs):
    from s2p_b200.projection import utm_target
    from s2p_b200.triangulation import disp_to_lonlatalt, disp_to_xyz
    a = _real()
    lla, lerr = disp_to_lonlatalt(a["disp"], a["mask_rect"], a["mask_orig"], a["H1"], a["H2"], a["rpc1"], a["rpc2"],
                                  a["img_bbx"], engine=engine)
    assert 0.5 < np.isfinite(lla[..., 0]).mean() < 1
    before = engine.kernel_launches()
    xyz, err = disp_to_xyz(a["rpc1"], a["rpc2"], a["H1"], a["H2"], a["disp"], a["mask_rect"], a["img_bbx"], a["mask_orig"],
                           out_crs=out_crs, engine=engine)
    zone, south = utm_target(out_crs)
    assert engine.kernel_launches() == before + (2 if zone else 1)
    assert xyz.shape == lla.shape and xyz.dtype == np.float64 and err.dtype == np.float32
    assert same(err, lerr)
    if not zone:
        assert same(xyz, lla)
    else:
        assert (zone, south) == (40, True)
        _check(xyz, lla, zone, south, ntruth=48)
        fin = np.isfinite(xyz[..., 0])
        assert 7.6e6 < xyz[..., 1][fin].min() and xyz[..., 1][fin].max() < 7.7e6          # about 21 S
        assert 2e5 < xyz[..., 0][fin].min() and xyz[..., 0][fin].max() < 8e5


def test_disp_to_xyz_pointing_correction(engine):
    from s2p_b200.triangulation import disp_to_xyz
    a = _real()
    A = np.array([[1.000186, 0.000156, 0.518804], [0.000040, 1.000032, 0.109895], [0.0, 0.0, 1.0]])
    got, gerr = disp_to_xyz(a["rpc1"], a["rpc2"], a["H1"], a["H2"], a["disp"], a["mask_rect"], a["img_bbx"], a["mask_orig"],
                            A=A, out_crs="epsg:32740", engine=engine)
    want, werr = engine.disp_to_xyz(a["disp"], a["mask_rect"], a["mask_orig"], a["H1"], np.dot(a["H2"], np.linalg.inv(A)),
                                    a["rpc1"], a["rpc2"], a["img_bbx"], 40, True)
    assert same(got, want) and same(gerr, werr)


def test_disp_to_xyz_engine_arguments(engine):
    from s2p_b200._lib import ERR_ARG, S2pbError
    a = _real()
    for zone in (-1, 61):
        with pytest.raises(S2pbError) as e:
            engine.disp_to_xyz(a["disp"], a["mask_rect"], a["mask_orig"], a["H1"], a["H2"], a["rpc1"], a["rpc2"], a["img_bbx"],
                               zone, True)
        assert e.value.code == ERR_ARG
    with pytest.raises(ValueError):
        engine.disp_to_xyz(a["disp"], a["mask_rect"][:-1], a["mask_orig"], a["H1"], a["H2"], a["rpc1"], a["rpc2"],
                           a["img_bbx"])


def test_disp_to_xyz_other_crs_without_pyproj(engine, monkeypatch):
    from s2p_b200._lib import ERR_UNSUPPORTED, S2pbError
    from s2p_b200.triangulation import disp_to_xyz
    monkeypatch.setitem(sys.modules, "s2p", None)                   # s2p (and so its pyproj wrappers) not importable
    a = _real()
    with pytest.raises(S2pbError) as e:
        disp_to_xyz(a["rpc1"], a["rpc2"], a["H1"], a["H2"], a["disp"], a["mask_rect"], a["img_bbx"], a["mask_orig"],
                    out_crs="epsg:32740+5773", engine=engine)
    assert e.value.code == ERR_UNSUPPORTED


def test_disp_to_xyz_other_crs_through_pyproj(engine, monkeypatch):
    """a target the device does not serve: the GPU's lon, lat, alt go through s2p.geographiclib's pyproj calls, as in the
    reference (s2p/triangulation.py:147-160)"""
    from s2p_b200.triangulation import disp_to_lonlatalt, disp_to_xyz
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
    a = _real()
    lla, _ = disp_to_lonlatalt(a["disp"], a["mask_rect"], a["mask_orig"], a["H1"], a["H2"], a["rpc1"], a["rpc2"], a["img_bbx"],
                               engine=engine)
    xyz, _ = disp_to_xyz(a["rpc1"], a["rpc2"], a["H1"], a["H2"], a["disp"], a["mask_rect"], a["img_bbx"], a["mask_orig"],
                         out_crs="epsg:32740+5773", engine=engine)
    assert len(calls) == 1
    x, y, in_crs, out_crs, z = calls[0]
    assert in_crs == "crs(epsg:4979)" and out_crs == "epsg:32740+5773"
    flat = lla.reshape(-1, 3)
    assert same(x, flat[:, 0]) and same(y, flat[:, 1]) and same(z, flat[:, 2])
    assert same(xyz, np.stack([lla[..., 0] * 2.0, lla[..., 1] - 1.0, lla[..., 2] + 3.0], axis=2))


def test_installed_disp_to_xyz_is_the_drop_in(engine, monkeypatch):
    from s2p_b200 import triangulation as T
    original = object()
    mod = types.ModuleType("s2p.triangulation")
    mod.lib = types.SimpleNamespace()
    mod.disp_to_xyz = original
    pkg = types.ModuleType("s2p")
    pkg.triangulation = mod
    monkeypatch.setitem(sys.modules, "s2p", pkg)
    monkeypatch.setitem(sys.modules, "s2p.triangulation", mod)
    assert T.install() is mod and T.install() is mod
    assert mod.disp_to_xyz is T.disp_to_xyz and mod._s2pb_original_disp_to_xyz is original
    a = _real()
    xyz, err = mod.disp_to_xyz(a["rpc1"], a["rpc2"], a["H1"], a["H2"], a["disp"], a["mask_rect"], a["img_bbx"], a["mask_orig"],
                               out_crs=_Crs(32740))
    want, werr = engine.disp_to_xyz(a["disp"], a["mask_rect"], a["mask_orig"], a["H1"], a["H2"], a["rpc1"], a["rpc2"],
                                    a["img_bbx"], 40, True)
    assert same(xyz, want) and same(err, werr)
