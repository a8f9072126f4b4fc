"""Heights above the EGM96 geoid on the GPU (S2PB_ZONE_EGM96, csrc/projection_kernels.cuh): the clouds of disp_to_xyz and
height_map_to_xyz, the PLY calls, the tile calls and the tile steps with s2p's `out_geoid` target, on seeded synthetic global
grids (within +-100 m) and the real-RPC fixtures.

The contract: x and y bit for bit those of the same call without the geoid, z within 1e-6 m of the ellipsoidal z minus the
restatement's N (tests/geoid_oracle.py), the same NaN mask.  Parity with PROJ itself is checked only where pyproj and
us_nga_egm96_15.tif are both installed."""
import os
import sys

import numpy as np
import pytest

import geoid_oracle as G
from util import same

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(int(np.__version__.split(".")[0]) < 2, reason="the device reproduces NumPy >= 2's casting")]

TOL = 1e-6
R, PW, N = 5.0, 10, 50


def _flag():
    from s2p_b200._lib import ZONE_EGM96
    return ZONE_EGM96


@pytest.fixture(scope="module")
def grid():
    return G.smooth_grid(11)


def _real():
    from test_gpu_ply import _real as real
    return real()


def _check(got, base, ell, grid):
    """got: the cloud with the geoid; base: the same call without it; ell: its (lon, lat, alt)"""
    assert np.array_equal(np.isnan(got), np.isnan(base))
    assert same(got[..., :2], base[..., :2])
    fin = np.isfinite(base[..., 0])
    want = G.shift(ell[fin], grid)[:, 2]
    assert np.abs(got[..., 2][fin] - want).max(initial=0) <= TOL
    assert np.abs(got[..., 2][fin] - base[..., 2][fin]).max() > 1.0          # the shift did happen


@pytest.mark.parametrize("zone,south", [(40, True), (0, False)])
def test_disp_to_xyz(engine, grid, zone, south):
    a = _real()
    args = (a["disp"], a["mask_rect"], a["mask_orig"], a["H1"], a["H2"], a["rpc1"], a["rpc2"], a["img_bbx"])
    engine.set_geoid(grid)
    lla, err0 = engine.disp_to_xyz(*args, 0, False)
    base, err1 = engine.disp_to_xyz(*args, zone, south)
    k0 = engine.kernel_launches()
    got, err = engine.disp_to_xyz(*args, zone | _flag(), south)
    assert engine.kernel_launches() - k0 == 2                   # triangulation, then one projection kernel
    assert same(err, err1) and 0.5 < np.isfinite(got[..., 0]).mean() < 1
    _check(got, base, lla, grid)


@pytest.mark.parametrize("zone,south", [(31, False), (0, False)])
def test_height_map_to_xyz(engine, grid, zone, south):
    from test_gpu_ply import _triplet
    heights, rpc, ox, oy, _ = _triplet()
    engine.set_geoid(grid)
    lla = engine.height_map_to_xyz(heights, rpc, ox, oy, 0, False)
    base = engine.height_map_to_xyz(heights, rpc, ox, oy, zone, south)
    got = engine.height_map_to_xyz(heights, rpc, ox, oy, zone | _flag(), south)
    _check(got, base, lla, grid)


def test_lonlat_to_utm_wrap_and_domain(engine, grid):
    engine.set_geoid(grid)
    lla = np.array([[179.9, 10.0, 5.0], [-180.1, -10.0, 5.0], [177.0, 89.99, 1.0], [-177.0, -90.0, 1.0], [177.0, 91.0, 1.0],
                    [np.nan, 1.0, 1.0], [177.0, 0.0, np.nan]])
    base = engine.lonlat_to_utm(lla, 60, False)
    got = engine.lonlat_to_utm(lla, 60 | _flag(), False)
    assert same(got[:4, :2], base[:4, :2])
    assert np.abs(got[:4, 2] - G.shift(lla[:4], grid)[:, 2]).max() <= TOL
    assert np.isposinf(got[4]).all() and np.isnan(got[5:]).all()


@pytest.mark.parametrize("zone", [40, 0])
def test_zero_and_constant_grids(engine, zone):
    a = _real()
    args = (a["disp"], a["mask_rect"], a["mask_orig"], a["H1"], a["H2"], a["rpc1"], a["rpc2"], a["img_bbx"])
    base, _ = engine.disp_to_xyz(*args, zone, True)
    engine.set_geoid(G.smooth_grid(0, constant=0.0))
    got, _ = engine.disp_to_xyz(*args, zone | _flag(), True)
    assert same(got, base)
    c = np.float32(-23.47)
    engine.set_geoid(G.smooth_grid(0, constant=c))
    got, _ = engine.disp_to_xyz(*args, zone | _flag(), True)
    want = base.copy()
    want[..., 2] -= np.float64(c)
    assert same(got, want)


@pytest.mark.parametrize("filt", [True, False])
def test_ply_calls_equal_the_stepwise_calls(engine, grid, filt):
    from s2p_b200.engine import Engine
    a = _real()
    r, p, n = (R, PW, N) if filt else (0.0, 0, 0)
    engine.set_geoid(grid)
    cloud = (a["disp"], a["mask_rect"], a["mask_orig"], a["H1"], a["H2"], a["rpc1"], a["rpc2"], a["img_bbx"], 40 | _flag(), True)
    xyz, _ = engine.disp_to_xyz(*cloud)
    if filt:
        engine.remove_isolated_3d_points(xyz, R, PW, N, 1)
    want = engine.ply_records(xyz, engine.stretch_8bit(a["colors"]), a["conf"])
    got = engine.disp_to_ply(*cloud, r=r, p=p, n=n, colors=a["colors"], confidence=a["conf"])
    assert len(got) > 1000 and got.tobytes() == want.tobytes()
    # the clr form: the warped colours in float32
    clr, hc = a["colors"].astype(np.float32), np.eye(3)
    warped = engine.homography(clr[0], hc, a["disp"].shape[1], a["disp"].shape[0])
    want = engine.ply_records_typed(xyz, warped[None], a["conf"])
    got = engine.disp_to_ply_clr(*cloud, r=r, p=p, n=n, clr=clr, hc=hc, confidence=a["conf"])
    assert got.dtype == Engine.ply_dtype(1, True, np.float32) and got.tobytes() == want.tobytes()
    # the height map's calls
    from test_gpu_ply import _triplet
    heights, rpc, ox, oy, colors = _triplet()
    xyz = engine.height_map_to_xyz(heights, rpc, ox, oy, 31 | _flag(), False)
    if filt:
        engine.remove_isolated_3d_points(xyz, R, PW, N, 1)
    want = engine.ply_records(xyz, engine.stretch_8bit(colors))
    got = engine.height_map_to_ply(heights, rpc, ox, oy, 31 | _flag(), False, r=r, p=p, n=n, colors=colors)
    assert len(got) > 1000 and got.tobytes() == want.tobytes()
    want = engine.ply_records_typed(xyz, colors)
    got = engine.height_map_to_ply_clr(heights, rpc, ox, oy, 31 | _flag(), False, r=r, p=p, n=n, colors=colors)
    assert got.tobytes() == want.tobytes()


@pytest.mark.parametrize("filt", [True, False])
def test_tile_calls_equal_the_stepwise_calls(engine, grid, filt):
    from test_gpu_pair_tile import _params, _real as pair_real
    from test_gpu_tristereo_tile import _colours, _triplet_maps
    r, p, n = (R, PW, N) if filt else (0.0, 0, 0)
    engine.set_geoid(grid)
    t = pair_real()
    rec, out = engine.pair_tile_to_ply(t["src1"], t["H1"], t["src2"], t["H2"], t["w"], t["h"], t["dmin"], t["dmax"], t["mask_orig"],
                                       t["H_ref"], t["H_sec"], t["rpc1"], t["rpc2"], t["bbx"], 40 | _flag(), True,
                                       params=_params(engine, "mgm"), erode_radius=2, r=r, p=p, n=n, confidence=True,
                                       want=("rect1", "disp", "conf", "mask"))
    want = engine.disp_to_ply(out["disp"], out["mask"], t["mask_orig"], t["H_ref"], t["H_sec"], t["rpc1"], t["rpc2"], t["bbx"],
                              40 | _flag(), True, r=r, p=p, n=n, colors=out["rect1"][None], confidence=out["conf"])
    assert len(rec) > 1000 and rec.tobytes() == want.tobytes()
    maps, offsets, rpc, ox, oy = _triplet_maps(2, seed=3)
    colours = _colours(maps[0].shape, "stretch")
    rec, out = engine.heights_tile_to_ply(maps, offsets, rpc, ox, oy, 31 | _flag(), False, cargarse_basura=True, sub_f32=False,
                                          r=r, p=p, n=n, want=("merged",), **colours)
    want = engine.height_map_to_ply(out["merged"].astype(np.float64), rpc, ox, oy, 31 | _flag(), False, r=r, p=p, n=n,
                                    colors=colours["colors"])
    assert len(rec) > 100 and rec.tobytes() == want.tobytes()


@pytest.fixture
def egm96_file(tmp_path, monkeypatch, grid):
    """grid as the us_nga_egm96_15.tif of the only PROJ data directory searched"""
    d = tmp_path / "proj"
    d.mkdir()
    G.write_grid_tiff(str(d / "us_nga_egm96_15.tif"), grid.values, grid.lon0, grid.lat0, grid.dlon, grid.dlat)
    monkeypatch.setenv("PROJ_DATA", str(d))
    monkeypatch.setitem(sys.modules, "pyproj", None)
    return d


def test_disp_to_xyz_drop_in_with_the_grid_file(engine, grid, egm96_file):
    from s2p_b200.triangulation import disp_to_xyz
    a = _real()
    xyz, _ = disp_to_xyz(a["rpc1"], a["rpc2"], a["H1"], a["H2"], a["disp"], a["mask_rect"], a["img_bbx"], a["mask_orig"],
                         out_crs="EPSG:32740+5773", engine=engine)
    lla, _ = engine.disp_to_xyz(a["disp"], a["mask_rect"], a["mask_orig"], a["H1"], a["H2"], a["rpc1"], a["rpc2"], a["img_bbx"])
    base, _ = engine.disp_to_xyz(a["disp"], a["mask_rect"], a["mask_orig"], a["H1"], a["H2"], a["rpc1"], a["rpc2"], a["img_bbx"],
                                 40, True)
    _check(xyz, base, lla, grid)


@pytest.mark.parametrize("clean", [False, True])
def test_pair_tile_with_out_geoid(engine, tmp_path, monkeypatch, egm96_file, clean):
    from s2p_b200 import fused
    from test_gpu_pair_tile import PT, _tile_setup

    def setup(name):
        s2p, tile, cfg = _tile_setup(tmp_path, monkeypatch, "mgm", clean, name=name)
        cfg["out_crs"] = "epsg:32740+5773"
        return s2p, tile
    s2p, stepwise_tile = setup("stepwise")
    s2p.rectification_pair(stepwise_tile, 1)
    s2p.stereo_matching(stepwise_tile, 1)
    s2p.disparity_to_ply(stepwise_tile)
    s2p, tile = setup("fused")
    fused.pair_tile(tile, engine=engine)
    assert s2p.calls == ["rectification_pair"]
    want, got = PT.files(stepwise_tile["dir"]), PT.files(tile["dir"])
    assert sorted(got) == sorted(want) and "cloud.ply" in got
    for name in want:
        assert got[name] == want[name], name
    assert b"comment projection: CRS epsg:32740+5773\n" in got["cloud.ply"]


@pytest.mark.parametrize("clean", [False, True])
def test_heights_tile_with_out_geoid(engine, tmp_path, monkeypatch, egm96_file, clean):
    from s2p_b200 import fused
    from test_gpu_tristereo_tile import TC, _heights_setup

    def setup(name):
        s2p, tile = _heights_setup(tmp_path, monkeypatch, True, clean, False, name)
        sys.modules["s2p.config"].cfg["out_crs"] = "epsg:32631+5773"
        return s2p, tile
    s2p, stepwise_tile = setup("stepwise")
    s2p.heights_to_ply(stepwise_tile)
    assert s2p.calls == ["heights_to_ply", "heights_fusion"]
    s2p, tile = setup("fused")
    fused.heights_tile(tile, engine=engine)
    assert s2p.calls == []
    want, got = TC.files(stepwise_tile["dir"]), TC.files(tile["dir"])
    assert sorted(got) == sorted(want) and "cloud.ply" in got
    for name in want:
        assert got[name] == want[name], name


def test_errors(engine, grid):
    from s2p_b200._lib import ERR_ARG, S2pbError
    a = _real()
    args = (a["disp"], a["mask_rect"], a["mask_orig"], a["H1"], a["H2"], a["rpc1"], a["rpc2"], a["img_bbx"])
    F = _flag()

    def refused(call):
        with pytest.raises(S2pbError) as e:
            call()
        assert e.value.code == ERR_ARG

    engine.set_geoid(None)
    refused(lambda: engine.disp_to_xyz(*args, 40 | F, True))                 # the flag without a grid
    refused(lambda: engine.lonlat_to_utm(np.zeros((2, 3)), 31 | F))
    engine.set_geoid(grid)
    for zone in (0x200 | 40, 0x80 | 40, 61 | F, -1, -1 & ~F, 0x101 << 1):     # other bits, zones outside 0..60
        refused(lambda: engine.disp_to_xyz(*args, zone, True))
    refused(lambda: engine.lonlat_to_utm(np.zeros((2, 3)), F))                # zone 0 is not a UTM zone
    from s2p_b200.projection import GeoidGrid
    v = grid.values
    for bad in (GeoidGrid(v[:, :100], -180.0, 90.0, 0.25, 0.25), GeoidGrid(v[:-4], -180.0, 90.0, 0.25, 0.25),
                GeoidGrid(v, -180.0, 89.0, 0.25, 0.25), GeoidGrid(v, -180.0, 90.0, -0.25, 0.25), GeoidGrid(v[:1], -180.0, 90.0, 0.25, 0.25)):
        refused(lambda: engine.set_geoid(bad))
    # a refused grid leaves the one held in place
    got, _ = engine.disp_to_xyz(*args, 40 | F, True)
    lla, _ = engine.disp_to_xyz(*args)
    base, _ = engine.disp_to_xyz(*args, 40, True)
    _check(got, base, lla, grid)


def test_pyproj_parity_where_installed(engine):
    """EPSG:4979 -> 32740+5773 by pyproj with PROJ's own us_nga_egm96_15.tif, where both are installed (they are not on every
    test machine; the test then skips)"""
    pyproj = pytest.importorskip("pyproj")
    from s2p_b200.projection import egm96_grid, utm_target
    if egm96_grid() is None:
        pytest.skip("no us_nga_egm96_15.tif that the device reads")
    a = _real()
    args = (a["disp"], a["mask_rect"], a["mask_orig"], a["H1"], a["H2"], a["rpc1"], a["rpc2"], a["img_bbx"])
    lla, _ = engine.disp_to_xyz(*args)
    got, _ = engine.disp_to_xyz(*args, *utm_target("epsg:32740+5773", engine))
    fin = np.isfinite(lla[..., 0])
    t = pyproj.Transformer.from_crs("epsg:4979", "epsg:32740+5773", always_xy=True)
    x, y, z = t.transform(lla[..., 0][fin], lla[..., 1][fin], lla[..., 2][fin])
    assert np.abs(got[..., 0][fin] - x).max() < 1e-6 and np.abs(got[..., 1][fin] - y).max() < 1e-6
    assert np.abs(got[..., 2][fin] - z).max() < 1e-6
