"""CPU tests of the EGM96 output heights: the restated bilinear rule checked by hand, the parsing of the compound targets, the
grid locator and reader against grid files written here, the fall-through decisions of the tile steps with s2p's
`out_geoid` on, and the C ABI's argument errors that need no device."""
import ctypes
import os
import re
import sys
import types

import numpy as np
import pytest

import geoid_oracle as G
from test_pair_tile_host import tile_env  # noqa: F401  (the fixture of the two-view tile)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _grid(values, lon0=-180.0, lat0=90.0, step=1.0):
    from s2p_b200.projection import GeoidGrid
    return GeoidGrid(np.asarray(values, np.float32), lon0, lat0, step, step)


def _ramp():
    """360 x 181 nodes at 1 degree, node (i, j) = i + 1000 j"""
    return _grid(np.arange(360)[None, :] + 1000.0 * np.arange(181)[:, None])


def test_rule_by_hand():
    g = _ramp()
    N = lambda lon, lat: float(G.undulation(g, np.array([lon]), np.array([lat]))[0])
    assert N(-180.0, 90.0) == 0.0 and N(-170.0, 80.0) == 10.0 + 10000.0          # nodes
    assert N(-169.5, 80.0) == 10.5 + 10000.0                                    # on a row, between two nodes
    assert N(-170.0, 79.5) == 10.0 + 10500.0                                    # on a column
    assert N(-169.75, 79.25) == 10.25 + 10750.0                                 # inside a cell
    assert N(179.5, 0.0) == 0.5 * (359 + 0) + 90000.0                           # the cell across the antimeridian
    assert N(-180.25, 0.0) == N(179.75, 0.0) == 0.25 * 359 + 0.75 * 0 + 90000.0
    assert N(180.0, 0.0) == N(-180.0, 0.0) == N(540.0, 0.0) == 90000.0          # longitude wraps modulo 360
    assert N(0.0, -90.0) == 180.0 + 180000.0                                    # the last row
    c = _grid(np.full((181, 360), 17.3, np.float32))
    rng = np.random.default_rng(0)
    lon, lat = rng.uniform(-400, 400, 1000), rng.uniform(-90, 90, 1000)
    assert (G.undulation(c, lon, lat) == np.float64(np.float32(17.3))).all()  # a constant grid is its constant everywhere


def test_shift_keeps_nan_points():
    g = _ramp()
    lla = np.array([[-170.0, 80.0, 5.0], [np.nan, 1.0, 2.0], [1.0, np.nan, 2.0], [1.0, 2.0, np.nan]])
    out = G.shift(lla, g)
    assert out[0].tolist() == [-170.0, 80.0, 5.0 - 10010.0]
    assert np.isnan(out[1:]).all()


class _Crs:
    def __init__(self, code, subs=None):
        self.code, self.sub_crs_list = code, subs or []

    def to_epsg(self):
        return self.code


@pytest.fixture
def proj_dir(tmp_path, monkeypatch):
    """an empty PROJ data directory, the only place searched (pyproj made unimportable)"""
    d = tmp_path / "proj"
    d.mkdir()
    monkeypatch.setenv("PROJ_DATA", str(d))
    monkeypatch.delenv("PROJ_LIB", raising=False)
    monkeypatch.setitem(sys.modules, "pyproj", None)
    return d


def _write_egm96(d, **kw):
    g = G.smooth_grid(1, step=2.0)
    G.write_grid_tiff(str(d / "us_nga_egm96_15.tif"), g.values, g.lon0, g.lat0, g.dlon, g.dlat, **kw)
    return g


def test_crs_parsing_without_a_grid(proj_dir):
    from s2p_b200.projection import unserved_reason, utm_target
    assert utm_target(None) == (0, False) and utm_target("epsg:4326") == (0, False)
    assert utm_target(" EPSG:32740 ") == (40, True) and utm_target(_Crs(32631)) == (31, False)
    for crs in ("epsg:32631+5773", "EPSG:32740+5773", "epsg:4326+5773", _Crs(None, [_Crs(32631), _Crs(5773)])):
        assert utm_target(crs) is None
        assert "us_nga_egm96_15.tif" in unserved_reason(crs)
    assert "not a UTM zone" in unserved_reason("epsg:2154")


def test_crs_parsing_with_a_grid(proj_dir):
    from s2p_b200._lib import ZONE_EGM96
    from s2p_b200.projection import utm_target
    _write_egm96(proj_dir)
    assert utm_target("epsg:32631+5773") == (31 | ZONE_EGM96, False)
    assert utm_target(" Epsg:32760+5773") == (60 | ZONE_EGM96, True)
    assert utm_target("epsg:32601+5773") == (1 | ZONE_EGM96, False)
    assert utm_target("EPSG:4326+5773") == (ZONE_EGM96, False)
    assert utm_target(_Crs(None, [_Crs(32740), _Crs(5773)])) == (40 | ZONE_EGM96, True)
    assert utm_target(_Crs(None, [_Crs(4326), _Crs(5773)])) == (ZONE_EGM96, False)
    # still as before without a vertical part
    assert utm_target("epsg:32631") == (31, False) and utm_target(4979) == (0, False)
    for crs in ("epsg:32631+3855", "epsg:4979+5773", "epsg:2154+5773", "epsg:32661+5773", "epsg:32700+5773", "epsg:32631+",
                "epsg:32631+5773+1", "32631+5773", _Crs(None, [_Crs(32631), _Crs(3855)]), _Crs(None, [_Crs(32631), _Crs(None)]),
                _Crs(None, [_Crs(32631)])):
        assert utm_target(crs) is None, crs


def test_grid_registered_on_the_engine(proj_dir):
    from s2p_b200.projection import egm96_grid, utm_target

    class Eng:
        grids = []

        def set_geoid(self, grid):
            self.grids.append(grid)
    _write_egm96(proj_dir)
    e = Eng()
    utm_target("epsg:32631+5773", e)
    utm_target("epsg:32631", e)
    assert len(e.grids) == 1 and e.grids[0] is egm96_grid()          # read once per file version


@pytest.mark.parametrize("kw", [dict(), dict(pixel_is_area=False), dict(compression=1, predictor=1), dict(predictor=2),
                                dict(tile=(64, 32)), dict(tile=(48, 16), predictor=1, compression=1),
                                dict(metadata={"interpolation_method": "bilinear", "TYPE": "VERTICAL_OFFSET_GEOGRAPHIC_TO_VERTICAL"})])
def test_reader_round_trip(tmp_path, kw):
    from s2p_b200.projection import read_geoid_grid
    g = G.smooth_grid(2, step=1.5)
    path = str(tmp_path / "g.tif")
    G.write_grid_tiff(path, g.values, g.lon0, g.lat0, g.dlon, g.dlat, **kw)
    r = read_geoid_grid(path)
    assert r.values.dtype == np.float32 and r.values.tobytes() == g.values.tobytes()
    assert (r.lon0, r.lat0, r.dlon, r.dlat) == (g.lon0, g.lat0, g.dlon, g.dlat)


def test_locator_search_order(tmp_path, monkeypatch):
    from s2p_b200.projection import egm96_grid, locate_egm96
    a, b, c = (tmp_path / n for n in "abc")
    for d in (a, b, c):
        d.mkdir()
    monkeypatch.delenv("PROJ_DATA", raising=False)
    monkeypatch.setenv("PROJ_LIB", os.pathsep.join([str(a), str(b)]))
    pyproj = types.ModuleType("pyproj")
    pyproj.datadir = types.SimpleNamespace(get_data_dir=lambda: str(c), get_user_data_dir=lambda: str(c / "user"))
    monkeypatch.setitem(sys.modules, "pyproj", pyproj)
    assert locate_egm96() is None and egm96_grid() is None
    _write_egm96(c)
    assert locate_egm96() == str(c / "us_nga_egm96_15.tif")                 # pyproj's data directory
    _write_egm96(b)
    assert locate_egm96() == str(b / "us_nga_egm96_15.tif")                 # PROJ_LIB before pyproj
    monkeypatch.setenv("PROJ_DATA", str(a))
    assert locate_egm96() == str(c / "us_nga_egm96_15.tif")                 # PROJ_DATA replaces PROJ_LIB
    assert egm96_grid() is not None


@pytest.mark.parametrize("case", ["missing", "regional", "subgrids", "bicubic", "nodata", "area_short"])
def test_grids_not_served(proj_dir, case):
    from s2p_b200.projection import GeoidGridError, egm96_grid, read_geoid_grid, utm_target
    path = proj_dir / "us_nga_egm96_15.tif"
    g = G.smooth_grid(3, step=2.0)
    if case == "missing":
        (proj_dir / "cache.db").write_bytes(b"")          # PROJ's network cache holds grids, not grid files
    elif case == "regional":
        G.write_grid_tiff(str(path), g.values[:, :150], g.lon0, g.lat0, g.dlon, g.dlat)
    elif case == "subgrids":
        G.write_grid_tiff(str(path), g.values, g.lon0, g.lat0, g.dlon, g.dlat, extra_image=True)
    elif case == "bicubic":
        G.write_grid_tiff(str(path), g.values, g.lon0, g.lat0, g.dlon, g.dlat, metadata={"interpolation_method": "bicubic"})
    elif case == "nodata":
        v = g.values.copy()
        v[3, 4] = -32768
        G.write_grid_tiff(str(path), v, g.lon0, g.lat0, g.dlon, g.dlat, nodata=-32768)
    elif case == "area_short":                            # cell centres from 89 to -89: the poles are outside
        G.write_grid_tiff(str(path), g.values[:-1], g.lon0, g.lat0 - 1.0, g.dlon, g.dlat, pixel_is_area=True)
    assert egm96_grid() is None and utm_target("epsg:32631+5773") is None
    if case != "missing":
        with pytest.raises(GeoidGridError):
            read_geoid_grid(str(path))


def _cfg(n_images, out_crs):
    img = dict(img="a.tif", clr=None, rpcm=None)
    return dict(images=[dict(img) for _ in range(n_images)], matching_algorithm="mgm", out_crs=out_crs, fusion_operator="average_if_close")


def test_fall_through_reasons_with_out_geoid(proj_dir, monkeypatch):
    from s2p_b200 import cloud, fused
    monkeypatch.setattr(cloud, "numpy_stretch_is_float64", lambda: True)
    for crs in ("epsg:32631+5773", "epsg:4326+5773"):
        assert "us_nga_egm96_15.tif" in fused.fall_through_reason(_cfg(2, crs))
        assert "us_nga_egm96_15.tif" in fused.heights_tile_fall_through_reason(_cfg(3, crs))
    _write_egm96(proj_dir)
    for crs in ("epsg:32631+5773", "epsg:4326+5773"):
        assert fused.fall_through_reason(_cfg(2, crs)) is None
        assert fused.heights_tile_fall_through_reason(_cfg(3, crs)) is None
    assert "not a UTM zone" in fused.fall_through_reason(_cfg(2, "epsg:32631+3855"))
    assert "not a UTM zone" in fused.heights_tile_fall_through_reason(_cfg(3, "epsg:2154+5773"))


def test_pair_tile_passes_the_geoid_zone(tile_env, proj_dir):
    from s2p_b200 import fused
    from s2p_b200._lib import ZONE_EGM96
    from s2p_b200.projection import egm96_grid
    from test_pair_tile_host import RecordingEngine

    class Eng(RecordingEngine):
        def set_geoid(self, grid):
            self.grid = grid

        def pair_tile_to_ply(self, *args, **kw):
            self.zone = args[14:16]
            return RecordingEngine.pair_tile_to_ply(self, *args, **kw)
    _write_egm96(proj_dir)
    s2p, tile, cfg, steps = tile_env("mgm", True, out_crs="epsg:32631+5773")
    eng = Eng()
    fused.pair_tile(tile, engine=eng)
    assert s2p.calls == ["rectification_pair"] and eng.grid is egm96_grid() and eng.zone == (31 | ZONE_EGM96, False)
    with open(os.path.join(tile["dir"], "cloud.ply"), "rb") as f:
        assert b"comment projection: CRS epsg:32631+5773\n" in f.read()


def test_abi_flag_and_arguments_without_a_device():
    from s2p_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "s2pb200.h")).read()
    assert int(re.search(r"#define S2PB_ZONE_EGM96 (0x[0-9a-fA-F]+)", hdr).group(1), 16) == _lib.ZONE_EGM96 == 0x100
    L = _lib.lib()
    grid = np.zeros((181, 360), np.float32)
    fp = grid.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
    assert L.s2pb_set_geoid(None, fp, 360, 181, -180.0, 90.0, 1.0, 1.0) == _lib.ERR_ARG
    assert L.s2pb_set_geoid(None, None, 0, 0, 0.0, 0.0, 0.0, 0.0) == _lib.ERR_ARG
    out = np.zeros(3)
    dp = out.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    assert L.s2pb_lonlat_to_utm(None, dp, dp, 1, 31 | _lib.ZONE_EGM96, 0) == _lib.ERR_ARG
