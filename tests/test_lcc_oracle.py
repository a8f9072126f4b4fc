"""The maps of S2PB_ZONE_PROJ on the CPU: the float64 restatements of tests/lcc_oracle.py against 50-digit truths (Lambert
conic conformal 2SP by IOGP Guidance Note 7-2, transverse Mercator on GRS80 by the UTM truth of tests/utm_oracle.py with
the ellipsoid as a parameter), and the reading of the new output CRSs (s2p_b200.projection.output_target)."""
import ctypes
import os
import re
import sys

import mpmath as mp
import numpy as np
import pytest

import lcc_oracle as L
import utm_oracle as U

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-6
LCC_CODES = [2154] + list(range(3942, 3951))
TM_CODES = list(range(25828, 25839))


def _proj(code):
    from s2p_b200.projection import PROJECTED
    return PROJECTED[code]


def _grid(proj, lon_half, lat_lo, lat_hi, nlon, nlat):
    lons = np.linspace(proj.lon0 - lon_half, proj.lon0 + lon_half, nlon)
    lats = np.linspace(lat_lo, lat_hi, nlat)
    return np.array([(a, b) for a in lons for b in lats])


def _with_alt(ll):
    return np.concatenate([ll, np.zeros((len(ll), 1))], axis=1)


def test_epsg_parameters():
    """the table against the EPSG dataset's entries (GRS 1980: a 6378137, 1/f 298.257222101)"""
    from s2p_b200 import _lib
    P = _proj(2154)
    assert P == (_lib.PROJ_LCC, 6378137.0, 298.257222101, 3.0, 46.5, 49.0, 44.0, 0.0, 700000.0, 6600000.0)
    for lat in range(42, 51):
        assert _proj(3900 + lat) == (_lib.PROJ_LCC, 6378137.0, 298.257222101, 3.0, lat, lat - 0.75, lat + 0.75, 0.0, 1700000.0,
                                     1200000.0 + (lat - 42) * 1000000.0)
    for zone in range(28, 39):
        assert _proj(25800 + zone) == (_lib.PROJ_TM, 6378137.0, 298.257222101, 6.0 * zone - 183.0, 0.0, 0.0, 0.0, 0.9996,
                                       500000.0, 0.0)
    from s2p_b200.projection import PROJECTED
    assert sorted(PROJECTED) == sorted(LCC_CODES + TM_CODES)


def test_lcc_truth_guidance_note_example():
    """Guidance Note 7-2's worked example of LCC 2SP: NAD27 / Texas South Central on Clarke 1866 (a 6378206.400 m,
    1/f 294.9786982), false origin 27 50' N 99 W at (2 000 000, 0) US survey feet, parallels 28 23' N and 30 17' N; the point
    28 30' N 96 W is at E 2 963 503.91, N 254 759.80 US survey feet"""
    from s2p_b200.projection import Projection
    ft = 1200 / 3937
    texas = Projection(L.LCC, 6378206.4, 294.9786982, -99.0, 27 + 50 / 60, 28 + 23 / 60, 30 + 17 / 60, 0.0, 2000000.0 * ft, 0.0)
    x, y = L.lcc_truth(-96.0, 28.5, texas)
    assert abs(float(x) / ft - 2963503.91) < 0.005 and abs(float(y) / ft - 254759.80) < 0.005
    got = L.lcc_restate(np.array([[-96.0, 28.5, 0.0]]), texas)[0]
    assert abs(got[0] - float(x)) < TOL and abs(got[1] - float(y)) < TOL


def test_lcc_truth_facts():
    """the false origin maps to (x0, y0); the scale is 1 on both standard parallels; easting antisymmetric about lon0"""
    P = _proj(2154)
    x, y = L.lcc_truth(P.lon0, P.lat0, P)
    assert abs(x - P.x0) < mp.mpf("1e-30") and abs(y - P.y0) < mp.mpf("1e-20")
    with mp.workdps(L.DPS):
        _, e2, _ = L._ell(P.a, P.rf)
        h = mp.mpf("1e-9")
        for lat in (P.lat1, P.lat2):               # northing against the meridian arc: scale 1 on the standard parallels
            y1 = L.lcc_truth(P.lon0, mp.mpf(lat) - h, P)[1]
            y2 = L.lcc_truth(P.lon0, mp.mpf(lat) + h, P)[1]
            phi = mp.mpf(lat) * mp.pi / 180
            rho_m = P.a * (1 - e2) / (1 - e2 * mp.sin(phi) ** 2) ** mp.mpf(1.5)
            k = (y2 - y1) / (rho_m * 2 * h * mp.pi / 180)
            assert abs(k - 1) < mp.mpf("1e-15")
        k = (L.lcc_truth(P.lon0, mp.mpf(46) + h, P)[1] - L.lcc_truth(P.lon0, mp.mpf(46) - h, P)[1]) / (
            P.a * (1 - e2) / (1 - e2 * mp.sin(46 * mp.pi / 180) ** 2) ** mp.mpf(1.5) * 2 * h * mp.pi / 180)
        assert k < 1 - mp.mpf("1e-6")              # and below 1 between them
        xe, ye = L.lcc_truth(P.lon0 + 7.25, 43.0, P)
        xw, yw = L.lcc_truth(P.lon0 - 7.25, 43.0, P)
        assert abs((xe - P.x0) + (xw - P.x0)) < mp.mpf("1e-20") and abs(ye - yw) < mp.mpf("1e-20")


@pytest.mark.parametrize("code", LCC_CODES)
def test_lcc_restatement_within_1e6_m_of_the_truth(code):
    """a dense grid over the CRS's area of use (France, about 9.9 W to 10.4 E, 41.2 N to 51.6 N) and well beyond it:
    30 degrees either side of the central meridian, from 30 S to 85 N"""
    P = _proj(code)
    ll = np.concatenate([_grid(P, 10.0, 40.0, 52.0, 21, 25), _grid(P, 30.0, -30.0, 85.0, 13, 24)])
    got = L.lcc_restate(_with_alt(ll), P)
    assert np.isfinite(got).all()
    assert np.abs(got[:, :2] - L.truth_array(ll, P)).max() < TOL


@pytest.mark.parametrize("code", [25828, 25832, 25838])
def test_tm_grs80_restatement_within_1e6_m_of_the_truth(code):
    """the ETRS89 zones: 4 degrees either side of the central meridian (a zone and its overlap) from 80 S to 84 N, and 3
    degrees beyond on a coarser grid"""
    P = _proj(code)
    ll = np.concatenate([_grid(P, 4.0, 34.0, 72.0, 17, 20), _grid(P, 7.0, -80.0, 84.0, 8, 14)])
    got = L.tm_restate(_with_alt(ll), P)
    assert np.isfinite(got).all()
    assert np.abs(got[:, :2] - L.truth_array(ll, P)).max() < TOL


def test_tm_machinery_is_the_utm_oracle_on_wgs84():
    """on WGS84 the generalised TM statements are utm_oracle's: the restatement bit for bit, the truth to 1e-9 m (utm_oracle
    takes 1/f as the decimal 298.257223563, the generalised truth as the float64 the host computes with)"""
    from s2p_b200.projection import Projection
    for zone, south in ((31, False), (40, True)):
        P = Projection(L.TM, 6378137.0, 298.257223563, U.lon0_of(zone), 0.0, 0.0, 0.0, 0.9996, 500000.0, 1e7 if south else 0.0)
        assert L.tm_coefficients(6378137.0, 1 / 298.257223563, 0.9996) == U.coefficients()
        rng = np.random.default_rng(zone)
        p = np.stack([U.lon0_of(zone) + rng.uniform(-5, 5, 50), rng.uniform(-80, 84, 50), rng.uniform(-100, 100, 50)], axis=1)
        assert L.tm_restate(p, P).tobytes() == U.restate(p, zone, south).tobytes()
        for lo, la in p[:4, :2]:
            x, y = L.tm_truth(lo, la, P)
            xu, yu = U.truth(lo, la, zone, south)
            assert abs(x - xu) < mp.mpf("1e-9") and abs(y - yu) < mp.mpf("1e-9")


def test_grs80_and_wgs84_differ():
    """the ellipsoid is a parameter: GRS80 and WGS84 differ by about 0.1 mm in 1/f, far below a metre but far above 1e-6 m"""
    P = _proj(25831)
    W = P._replace(rf=298.257223563)
    a = L.tm_truth(3.0 + 2.5, 60.0, P)
    b = L.tm_truth(3.0 + 2.5, 60.0, W)
    assert 1e-5 < abs(float(a[1] - b[1])) < 1.0


def test_lcc_nan_inf_poles_and_altitude():
    P = _proj(2154)
    p = np.array([[3.0, 46.5, 123.456], [np.nan, 45.0, 1.0], [3.0, np.nan, 1.0], [3.0, 45.0, np.nan], [3.0, 91.0, 5.0],
                  [3.0, -90.0, 5.0], [40.0, 90.0, 7.0], [3.0 + 360.0 - 1.0, 45.0, -7.0]])
    out = L.lcc_restate(p, P)
    assert out[0, 2] == 123.456 and np.abs(out[0, :2] - [P.x0, P.y0]).max() < 1e-6
    assert np.isnan(out[1:4]).all()
    assert np.isposinf(out[4:6]).all()                    # |lat| > 90, the south pole away from the cone
    assert out[6, 0] == P.x0 and out[6, 1] == P.y0 + L.lcc_params(P)[3] and out[6, 2] == 7.0       # the north pole: the apex
    assert np.abs(out[7, :2] - L.lcc_restate(np.array([[2.0, 45.0, -7.0]]), P)[0, :2]).max() < 1e-6


class _Crs:
    def __init__(self, code, subs=None):
        self.code = code
        if subs is not None:
            self.sub_crs_list = subs

    def to_epsg(self):
        return self.code


@pytest.fixture
def no_grid(tmp_path, monkeypatch):
    """an empty PROJ data directory, and a pyproj whose transformations agree with the device's maps"""
    d = tmp_path / "proj"
    d.mkdir()
    monkeypatch.setenv("PROJ_DATA", str(d))
    monkeypatch.delenv("PROJ_LIB", raising=False)
    monkeypatch.setitem(sys.modules, "pyproj", L.fake_pyproj())
    return d


def test_served_only_where_proj_agrees(no_grid, monkeypatch):
    """without pyproj (s2p's own path needs it too), or with a PROJ whose operation moves the points (a datum shift), the
    targets fall through as before; PROJ is asked once per code and pyproj module"""
    from s2p_b200 import projection
    from s2p_b200._lib import ZONE_PROJ
    assert projection.output_target("epsg:2154") == (ZONE_PROJ, False)
    assert projection.output_target("epsg:2154") == (ZONE_PROJ, False)
    assert sys.modules["pyproj"].calls == [("epsg:4979", "epsg:2154")]
    monkeypatch.setitem(sys.modules, "pyproj", None)
    for crs in ("epsg:2154", "epsg:25832", "epsg:3950+5773"):
        assert projection.output_target(crs) is None
        r = projection.unserved_reason(crs)
        assert "not a UTM zone" in r and "pyproj" in r
    monkeypatch.setitem(sys.modules, "pyproj", L.fake_pyproj(shift=0.3))
    assert projection.output_target("epsg:25832") is None
    monkeypatch.setitem(sys.modules, "pyproj", L.fake_pyproj(shift=1e-5))          # rounding-sized differences
    assert projection.output_target("epsg:25832") == (ZONE_PROJ, False)
    monkeypatch.setitem(sys.modules, "pyproj", L.fake_pyproj(codes={2154: _proj(2154)._replace(lat0=46.0)}))
    assert projection.output_target("epsg:2154") is None                            # another definition of the CRS
    assert projection.output_target("epsg:3942") is None                            # PROJ without the code


def test_numpy_map_of_the_check():
    """map_lonlat, the package's float64 map that PROJ is compared with, against the truths at the reference points"""
    from s2p_b200.projection import PROJECTED, _reference_points, map_lonlat
    for code in (2154, 3942, 3950, 25828, 25838):
        P = PROJECTED[code]
        lon, lat = _reference_points(P)
        x, y = map_lonlat(P, lon, lat)
        want = L.truth_array(np.stack([lon, lat], 1), P)
        assert np.abs(x - want[:, 0]).max() < 1e-6 and np.abs(y - want[:, 1]).max() < 1e-6


def test_output_target_parsing(no_grid):
    from s2p_b200._lib import ZONE_PROJ
    from s2p_b200.projection import output_target, utm_target
    P = (ZONE_PROJ, False)
    for crs in ("epsg:2154", "EPSG:2154", " Epsg:3942 ", 3950, np.int64(25828), "epsg:25838", _Crs(25832), _Crs(2154)):
        assert output_target(crs) == P, crs
        assert utm_target(crs) is None, crs                      # utm_target keeps to WGS84
    # WGS84 and its UTM zones as before
    assert output_target(None) == (0, False) and output_target("epsg:4979") == (0, False)
    assert output_target("epsg:32631") == (31, False) and output_target(_Crs(32740)) == (40, True)
    # boundaries and neighbours that fall through
    for crs in (25827, "epsg:25839", "epsg:3941", "epsg:3951", "epsg:2153", "epsg:2155", "epsg:26915", "epsg:27572",
                "epsg:3857", "epsg:28354", "epsg:2154+3855", "epsg:2154+", "2154", "+proj=lcc", _Crs(None),
                _Crs(None, [_Crs(2154)]),
                _Crs(None, [_Crs(2154), _Crs(3855)]), True):
        assert output_target(crs) is None, crs


def test_output_target_with_egm96(no_grid):
    from s2p_b200._lib import ZONE_EGM96, ZONE_PROJ
    from s2p_b200.projection import output_target, unserved_reason
    import geoid_oracle as G
    for crs in ("EPSG:25832+5773", "epsg:2154+5773", _Crs(None, [_Crs(3945), _Crs(5773)])):
        assert output_target(crs) is None
        assert "us_nga_egm96_15.tif" in unserved_reason(crs)
    g = G.smooth_grid(1, step=2.0)
    G.write_grid_tiff(str(no_grid / "us_nga_egm96_15.tif"), g.values, g.lon0, g.lat0, g.dlon, g.dlat)
    for crs in ("EPSG:25832+5773", "epsg:2154+5773", _Crs(None, [_Crs(3945), _Crs(5773)])):
        assert output_target(crs) == (ZONE_PROJ | ZONE_EGM96, False), crs
    for crs in ("epsg:25839+5773", "epsg:3941+5773", "epsg:27572+5773"):
        assert output_target(crs) is None


def test_registered_on_the_engine(no_grid):
    from s2p_b200.projection import output_target

    class Eng:
        def __init__(self):
            self.calls = []

        def set_projection(self, proj):
            self.calls.append(("proj", proj))

        def set_geoid(self, grid):
            self.calls.append(("geoid", grid))
    e = Eng()
    output_target("epsg:3944", e)
    assert e.calls == [("proj", _proj(3944))]
    e = Eng()
    output_target("epsg:32631", e)
    output_target("epsg:27572", e)
    output_target("epsg:2154+5773", e)                           # no grid: nothing registered
    assert e.calls == []


def test_unserved_reasons(no_grid):
    from s2p_b200.projection import unserved_reason
    for crs in ("epsg:27572", "epsg:25839", "epsg:3951"):
        r = unserved_reason(crs)
        assert "not a UTM zone" in r and "ETRS89" in r and "RGF93" in r


def _cfg(n_images, out_crs):
    img = dict(img="a.tif", clr=None, rpcm=None)
    return dict(images=[dict(img) for _ in range(n_images)], matching_algorithm="mgm", out_crs=out_crs,
                fusion_operator="average_if_close")


def test_fall_through_reasons(no_grid, monkeypatch):
    from s2p_b200 import cloud, fused
    monkeypatch.setattr(cloud, "numpy_stretch_is_float64", lambda: True)
    for crs in ("epsg:2154", "epsg:25832", "EPSG:3942", 3950):
        assert fused.fall_through_reason(_cfg(2, crs)) is None
        assert fused.heights_tile_fall_through_reason(_cfg(3, crs)) is None
        assert fused.pair_heights_fall_through_reason(_cfg(3, crs)) is None
    for crs in ("epsg:25827", "epsg:3951", "epsg:27572"):
        assert "RGF93" in fused.fall_through_reason(_cfg(2, crs))
        assert "RGF93" in fused.heights_tile_fall_through_reason(_cfg(3, crs))
    assert "us_nga_egm96_15.tif" in fused.fall_through_reason(_cfg(2, "epsg:2154+5773"))


def test_abi_without_a_device():
    from s2p_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "s2pb200.h")).read()
    assert int(re.search(r"#define S2PB_ZONE_PROJ (0x[0-9a-fA-F]+)", hdr).group(1), 16) == _lib.ZONE_PROJ == 0x200
    assert int(re.search(r"#define S2PB_PROJ_TM (\d+)", hdr).group(1)) == _lib.PROJ_TM
    assert int(re.search(r"#define S2PB_PROJ_LCC (\d+)", hdr).group(1)) == _lib.PROJ_LCC
    body = re.search(r"typedef struct s2pb_projection \{(.*?)\} s2pb_projection;", hdr, re.S).group(1)
    fields = [f for line in re.findall(r"(?:int32_t|double)\s+([\w, ]+);", body) for f in re.split(r",\s*", line)]
    assert fields == [f for f, _ in _lib.Projection._fields_]
    L_ = _lib.lib()
    from s2p_b200.engine import _projection
    p = _projection(_proj(2154))
    out = np.zeros(3)
    dp = out.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    assert L_.s2pb_set_projection(None, ctypes.byref(p)) == _lib.ERR_ARG
    assert L_.s2pb_lonlat_to_proj(None, dp, dp, 1, ctypes.byref(p)) == _lib.ERR_ARG
    assert L_.s2pb_lonlat_to_utm(None, dp, dp, 1, _lib.ZONE_PROJ, 0) == _lib.ERR_ARG
