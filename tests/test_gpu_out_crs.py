"""The ETRS89 UTM zones (EPSG 25828-25838) and the RGF93 v1 Lambert grids (2154, 3942-3950) on the GPU (S2PB_ZONE_PROJ,
csrc/projection_kernels.cuh): s2pb_lonlat_to_proj, the clouds of disp_to_xyz and height_map_to_xyz, the PLY and tile calls
and the tile steps, on the real-RPC fixtures.

The contract: x and y within 1e-6 m of the float64 restatement (tests/lcc_oracle.py) applied to the device's own WGS84
(lon, lat), the same NaN and +inf masks; z bit for bit the WGS84 call's, or the EGM96 call's with +5773.  The drop-ins and
tile steps serve these CRSs only where PROJ agrees with the device's maps (projection.proj_agrees); there a stand-in pyproj
that runs the restatement plays PROJ.  Parity with PROJ itself is not checked here (it needs pyproj)."""
import sys

import numpy as np
import pytest

import geoid_oracle as G
import lcc_oracle as L
from util import same

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(int(np.__version__.split(".")[0]) < 2, reason="the device reproduces NumPy >= 2's casting")]

TOL = 1e-6
R, PW, N = 5.0, 10, 50
CODES = [2154] + list(range(3942, 3951)) + list(range(25828, 25839))


def _proj(code):
    from s2p_b200.projection import PROJECTED
    return PROJECTED[code]


def _zone():
    from s2p_b200._lib import ZONE_PROJ
    return ZONE_PROJ


def _egm96():
    from s2p_b200._lib import ZONE_EGM96
    return ZONE_EGM96


def _real():
    from test_gpu_ply import _real as real
    return real()


def _cloud_args(a):
    return (a["disp"], a["mask_rect"], a["mask_orig"], a["H1"], a["H2"], a["rpc1"], a["rpc2"], a["img_bbx"])


def _check(got, lla, proj):
    """got: the cloud in proj; lla: the same call's WGS84 cloud"""
    want = L.restate(lla, proj)
    assert np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(np.isposinf(got), np.isposinf(want))
    fin = np.isfinite(want[..., 0])
    assert fin.mean() > 0.5
    assert np.abs(got[..., :2][fin] - want[..., :2][fin]).max() <= TOL
    assert same(got[..., 2], lla[..., 2])


@pytest.mark.parametrize("code", CODES)
def test_lonlat_to_proj(engine, code):
    P = _proj(code)
    rng = np.random.default_rng(code)
    n = 20000
    # TM: the whole sphere of latitudes; LCC: up to 60 S, where the radius on the side away from the cone reaches 1e8 m
    # (closer to that pole it grows as exp(-n psi) and a few ulps of psi exceed 1e-6 m)
    lat_lo = -89.9 if P.method == L.TM else -60.0
    lla = np.stack([P.lon0 + rng.uniform(-40, 40, n), rng.uniform(lat_lo, 89.9, n), rng.uniform(-500, 5000, n)], axis=1)
    lla[:2000, 0] = P.lon0 + rng.uniform(-8, 8, 2000)             # the area of use
    lla[:2000, 1] = rng.uniform(40, 55, 2000) if P.method == L.LCC else rng.uniform(34, 72, 2000)
    special = np.array([[P.lon0, 90.0, 1.0], [P.lon0 + 10, -90.0, 2.0], [P.lon0, 91.0, 3.0], [P.lon0, -90.5, 3.0],
                        [np.nan, 45.0, 1.0], [3.0, np.nan, 1.0], [3.0, 45.0, np.nan], [P.lon0 + 359.0, 45.0, 4.0],
                        [P.lon0 - 181.0, 45.0, 5.0], [P.lon0 + 89.0, 1.0, 6.0], [np.inf, 45.0, 1.0]])
    lla = np.concatenate([lla, special])
    got = engine.lonlat_to_proj(lla, P)
    want = L.restate(lla, P)
    assert np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(np.isposinf(got), np.isposinf(want))
    fin = np.isfinite(want[:, 0])
    assert np.abs(got[fin, :2] - want[fin, :2]).max() <= TOL
    assert same(got[fin, 2], lla[fin, 2])


@pytest.mark.parametrize("code", [2154, 3942, 3950, 25828, 25831, 25838])
def test_disp_to_xyz(engine, code):
    a = _real()
    args = _cloud_args(a)
    engine.set_projection(_proj(code))
    lla, err0 = engine.disp_to_xyz(*args, 0, False)
    k0 = engine.kernel_launches()
    got, err = engine.disp_to_xyz(*args, _zone(), False)
    assert engine.kernel_launches() - k0 == 2                   # triangulation, then one projection kernel
    assert same(err, err0)
    _check(got, lla, _proj(code))


@pytest.mark.parametrize("code", [2154, 3945, 25831, 25832])
def test_height_map_to_xyz(engine, code):
    from test_gpu_ply import _triplet
    heights, rpc, ox, oy, _ = _triplet()
    engine.set_projection(_proj(code))
    lla = engine.height_map_to_xyz(heights, rpc, ox, oy, 0, False)
    got = engine.height_map_to_xyz(heights, rpc, ox, oy, _zone(), False)
    _check(got, lla, _proj(code))


@pytest.mark.parametrize("code", [2154, 25832])
def test_egm96_heights(engine, code):
    """+5773: x and y those of the call without the geoid, z that of the WGS84 call with it, bit for bit"""
    a = _real()
    args = _cloud_args(a)
    engine.set_geoid(G.smooth_grid(11))
    engine.set_projection(_proj(code))
    base, _ = engine.disp_to_xyz(*args, _zone(), False)
    geo, _ = engine.disp_to_xyz(*args, _egm96(), False)
    got, _ = engine.disp_to_xyz(*args, _zone() | _egm96(), False)
    assert same(got[..., :2], base[..., :2]) and same(got[..., 2], geo[..., 2])
    from test_gpu_ply import _triplet
    heights, rpc, ox, oy, _ = _triplet()
    base = engine.height_map_to_xyz(heights, rpc, ox, oy, _zone(), False)
    geo = engine.height_map_to_xyz(heights, rpc, ox, oy, _egm96(), False)
    got = engine.height_map_to_xyz(heights, rpc, ox, oy, _zone() | _egm96(), False)
    assert same(got[..., :2], base[..., :2]) and same(got[..., 2], geo[..., 2])


@pytest.mark.parametrize("code", [2154, 25832])
def test_ply_calls_equal_the_stepwise_calls(engine, code):
    from test_gpu_ply import _triplet
    a = _real()
    engine.set_projection(_proj(code))
    cloud = _cloud_args(a) + (_zone(), False)
    xyz, _ = engine.disp_to_xyz(*cloud)
    engine.remove_isolated_3d_points(xyz, R, PW, N, 1)
    want = engine.ply_records(xyz, engine.stretch_8bit(a["colors"]), a["conf"])
    got = engine.disp_to_ply(*cloud, r=R, p=PW, n=N, colors=a["colors"], confidence=a["conf"])
    assert len(got) > 1000 and got.tobytes() == want.tobytes()
    clr, hc = a["colors"].astype(np.float32), np.eye(3)
    warped = engine.homography(clr[0], hc, a["disp"].shape[1], a["disp"].shape[0])
    want = engine.ply_records_typed(xyz, warped[None], a["conf"])
    got = engine.disp_to_ply_clr(*cloud, r=R, p=PW, n=N, clr=clr, hc=hc, confidence=a["conf"])
    assert got.tobytes() == want.tobytes()
    heights, rpc, ox, oy, colors = _triplet()
    xyz = engine.height_map_to_xyz(heights, rpc, ox, oy, _zone(), False)
    engine.remove_isolated_3d_points(xyz, R, PW, N, 1)
    want = engine.ply_records(xyz, engine.stretch_8bit(colors))
    got = engine.height_map_to_ply(heights, rpc, ox, oy, _zone(), False, r=R, p=PW, n=N, colors=colors)
    assert len(got) > 1000 and got.tobytes() == want.tobytes()
    want = engine.ply_records_typed(xyz, colors)
    got = engine.height_map_to_ply_clr(heights, rpc, ox, oy, _zone(), False, r=R, p=PW, n=N, colors=colors)
    assert got.tobytes() == want.tobytes()


@pytest.mark.parametrize("code", [2154, 25832])
def test_tile_calls_equal_the_stepwise_calls(engine, code):
    from test_gpu_pair_tile import _params, _real as pair_real
    from test_gpu_tristereo_tile import _colours, _triplet_maps
    engine.set_projection(_proj(code))
    t = pair_real()
    rec, out = engine.pair_tile_to_ply(t["src1"], t["H1"], t["src2"], t["H2"], t["w"], t["h"], t["dmin"], t["dmax"], t["mask_orig"],
                                       t["H_ref"], t["H_sec"], t["rpc1"], t["rpc2"], t["bbx"], _zone(), False,
                                       params=_params(engine, "mgm"), erode_radius=2, r=R, p=PW, n=N, confidence=True,
                                       want=("rect1", "disp", "conf", "mask"))
    want = engine.disp_to_ply(out["disp"], out["mask"], t["mask_orig"], t["H_ref"], t["H_sec"], t["rpc1"], t["rpc2"], t["bbx"],
                              _zone(), False, r=R, p=PW, n=N, colors=out["rect1"][None], confidence=out["conf"])
    assert len(rec) > 1000 and rec.tobytes() == want.tobytes()
    maps, offsets, rpc, ox, oy = _triplet_maps(2, seed=3)
    colours = _colours(maps[0].shape, "stretch")
    rec, out = engine.heights_tile_to_ply(maps, offsets, rpc, ox, oy, _zone(), False, cargarse_basura=True, sub_f32=False,
                                          r=R, p=PW, n=N, want=("merged",), **colours)
    want = engine.height_map_to_ply(out["merged"].astype(np.float64), rpc, ox, oy, _zone(), False, r=R, p=PW, n=N,
                                    colors=colours["colors"])
    assert len(rec) > 100 and rec.tobytes() == want.tobytes()


@pytest.mark.parametrize("crs", ["epsg:2154", "EPSG:25832"])
@pytest.mark.parametrize("clean", [False, True])
def test_pair_tile_step(engine, tmp_path, monkeypatch, crs, clean):
    from s2p_b200 import fused
    from test_gpu_pair_tile import PT, _tile_setup

    monkeypatch.setitem(sys.modules, "pyproj", L.fake_pyproj())      # a PROJ that agrees with the device's maps

    def setup(name):
        s2p, tile, cfg = _tile_setup(tmp_path, monkeypatch, "mgm", clean, name=name)
        cfg["out_crs"] = crs
        assert fused.fall_through_reason(cfg) is None
        return s2p, tile
    s2p, stepwise_tile = setup("stepwise")
    s2p.rectification_pair(stepwise_tile, 1)
    s2p.stereo_matching(stepwise_tile, 1)
    s2p.disparity_to_ply(stepwise_tile)
    assert s2p.calls == ["rectification_pair", "stereo_matching", "disparity_to_ply"]
    s2p, tile = setup("fused")
    fused.pair_tile(tile, engine=engine)
    assert s2p.calls == ["rectification_pair"]
    want, got = PT.files(stepwise_tile["dir"]), PT.files(tile["dir"])
    assert sorted(got) == sorted(want) and "cloud.ply" in got
    for name in want:
        assert got[name] == want[name], name
    assert b"comment projection: CRS %s\n" % crs.encode() in got["cloud.ply"]


@pytest.mark.parametrize("crs", ["epsg:2154", "epsg:25831"])
@pytest.mark.parametrize("clean", [False, True])
def test_heights_tile_step(engine, tmp_path, monkeypatch, crs, clean):
    from s2p_b200 import fused
    from test_gpu_tristereo_tile import TC, _heights_setup

    monkeypatch.setitem(sys.modules, "pyproj", L.fake_pyproj())

    def setup(name):
        s2p, tile = _heights_setup(tmp_path, monkeypatch, True, clean, False, name)
        cfg = sys.modules["s2p.config"].cfg
        cfg["out_crs"] = crs
        assert fused.heights_tile_fall_through_reason(cfg) is None
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
    assert b"comment projection: CRS %s\n" % crs.encode() in got["cloud.ply"]


def test_drop_ins(engine, monkeypatch):
    from s2p_b200.triangulation import disp_to_xyz
    monkeypatch.setitem(sys.modules, "pyproj", L.fake_pyproj())
    a = _real()
    xyz, _ = disp_to_xyz(a["rpc1"], a["rpc2"], a["H1"], a["H2"], a["disp"], a["mask_rect"], a["img_bbx"], a["mask_orig"],
                         out_crs="epsg:3946", engine=engine)
    lla, _ = engine.disp_to_xyz(*_cloud_args(a))
    _check(xyz, lla, _proj(3946))


def test_errors(engine):
    from s2p_b200._lib import ERR_ARG, S2pbError
    a = _real()
    args = _cloud_args(a)
    F, E = _zone(), _egm96()

    def refused(call):
        with pytest.raises(S2pbError) as e:
            call()
        assert e.value.code == ERR_ARG
    engine.set_projection(None)
    refused(lambda: engine.disp_to_xyz(*args, F, False))                      # the flag without a projection
    engine.set_geoid(None)
    engine.set_projection(_proj(2154))
    refused(lambda: engine.disp_to_xyz(*args, F | E, False))                  # EGM96 without a grid
    refused(lambda: engine.disp_to_xyz(*args, F, True))                       # a nonzero south
    for zone in (F | 31, F | 0x80, F | 0x400, -1):                            # a UTM zone or another bit with the flag
        refused(lambda: engine.disp_to_xyz(*args, zone, False))
    from test_gpu_ply import _triplet
    heights, rpc, ox, oy, _ = _triplet()
    refused(lambda: engine.height_map_to_xyz(heights, rpc, ox, oy, F, True))
    refused(lambda: engine.lonlat_to_utm(np.zeros((2, 3)), F))                # the UTM entry point takes no projection
    P = _proj(2154)
    for bad in (P._replace(method=0), P._replace(method=3), P._replace(a=-1.0), P._replace(rf=1.0), P._replace(lat1=90.0),
                P._replace(lat1=-44.0), P._replace(lat0=-90.0), P._replace(lat0=91.0), P._replace(x0=np.nan),
                _proj(25832)._replace(lat0=1.0), _proj(25832)._replace(k0=0.0), _proj(25832)._replace(lon0=np.inf)):
        refused(lambda: engine.set_projection(bad))
        refused(lambda: engine.lonlat_to_proj(np.zeros((1, 3)), bad))
    # a refused projection leaves the one held in place
    got, _ = engine.disp_to_xyz(*args, F, False)
    lla, _ = engine.disp_to_xyz(*args)
    _check(got, lla, P)
