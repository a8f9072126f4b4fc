"""CPU tests of s2p_b200.fused.pair_heights and heights_tile's host side, with an engine that records its calls: the files a
tri-stereo tile is left with (clean_intermediate or not, pairs 1 and 2), the outputs asked of the device, the confidence-file rule,
the fall-through decisions and the errors; the float64 height-map writer; and the ctypes mirror of s2pb_heights_tile against the
C header."""
import os
import subprocess

import numpy as np
import pytest

import tristereo_cases as TC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, H, DMIN, DMAX = 40, 30, -5.0, 5.0
TILE = (3, 2, 24, 20)
H1 = np.array([[1.0, 0.0, -3.0], [0.0, 1.0, -2.0], [0.0, 0.0, 1.0]])
H2 = np.array([[1.0, 0.01, -4.0], [0.0, 1.0, -2.5], [0.0, 0.0, 1.0]])


class RecordingEngine:
    """pair_tile_to_height_map's and heights_tile_to_ply's contracts without a device"""

    def __init__(self, error=None):
        self.calls, self.error = [], error

    def _maybe_fail(self):
        from s2p_b200.engine import S2pbError
        if self.error is not None:
            raise S2pbError(self.error, "refused")

    def pair_tile_to_height_map(self, src1, H1, src2, H2, w, h, dmin, dmax, mask_orig, H_ref, H_sec, rpc1, rpc2, tile, **kw):
        self.calls.append(dict(kw, kind="pair", dmin=dmin, dmax=dmax, w=w, h=h, tile=tuple(tile), H_sec=H_sec))
        self._maybe_fail()
        out = {k: np.ones((h, w), np.uint8 if k == "mask" else np.float32) for k in kw["want"]}
        return np.full((tile[3], tile[2]), 7.25, np.float64), out

    def heights_tile_to_ply(self, maps, offsets, rpc, off_x, off_y, zone=0, south=False, **kw):
        from s2p_b200.engine import Engine
        self.calls.append(dict(kw, kind="heights", maps=maps, offsets=offsets, off=(off_x, off_y), zone=zone, south=south))
        self._maybe_fail()
        h, w = maps[0].shape
        out = {}
        if "merged" in kw["want"]:
            out["merged"] = np.full((h, w), 3.5, np.float32)
        if "cleaned" in kw["want"]:
            out["cleaned"] = [np.full((h, w), 1.5 + k, np.float32) for k in range(len(maps))]
        nb = 1 if kw.get("clr") is not None or kw.get("colors") is not None else 0
        return np.zeros(3, Engine.ply_dtype(nb, False)), out


@pytest.fixture
def tri_env(tmp_path, monkeypatch):
    """-> make(algo, clean, **cfg overrides) -> (s2p stub, tile, cfg, calls of the stand-ins)"""
    from s2p_b200 import rasterio_compat as rio
    from s2p_b200.triangulation import rpc_from_geotiff_tag
    from util import load_real_pair
    z = load_real_pair()
    rng = np.random.default_rng(0)
    imgs = [str(tmp_path / ("img%d.tif" % k)) for k in (1, 2, 3)]
    for f in imgs:
        rio.write_float_tiff(f, rng.random((H + 10, W + 10)).astype(np.float32))
    for i in (1, 2):
        np.savetxt(str(tmp_path / ("global_pointing_pair_%d.txt" % i)), np.eye(3) if i == 1 else np.diag([1.0, 1.0, 2.0]))
        np.savetxt(str(tmp_path / ("global_mean_height_pair_%d.txt" % i)), [10.0 * i])
    rpcs = [rpc_from_geotiff_tag(z["rpc1"]), rpc_from_geotiff_tag(z["rpc2"]), rpc_from_geotiff_tag(z["rpc2"])]

    def make(algo, clean, nimages=3, **over):
        steps = []
        cfg = TC.cfg_for(tmp_path, imgs[:nimages], rpcs[:nimages], algo, clean)
        cfg.update(over)
        s2p = TC.stub_s2p(monkeypatch, cfg, H1, H2, W, H, DMIN, DMAX,
                          lambda out, im, Hm, w, h: steps.append(("warp", out)),
                          lambda im1, im2, disp, mask, *a, **k: (steps.append(("match",)),     # the files the step reads next
                                                                 rio.write_float_tiff(disp, np.zeros((H, W), np.float32)),
                                                                 rio.write_mask_png(mask, np.ones((H, W), np.uint8))),
                          lambda out, msk, r: steps.append(("erode", r)),
                          height_map=lambda *a, **k: steps.append(("height_map",)) or np.zeros((TILE[3], TILE[2])),
                          write_height_map=lambda path, a: steps.append(("write_height_map", path)),
                          heights_to_ply=lambda tile: steps.append(("heights_to_ply",)))
        tile = TC.make_tile(tmp_path, "tile_%s_%d" % (algo, clean), TILE, nimages - 1)
        return s2p, tile, cfg, steps
    return make


CONF = {"mgm": "rectified_disp_confidence.tif", "mgm_multi": "rectified_disp_confidence.tif",
        "mgm_multi_lsd": "rectified_disp.tif.confidence.tif", "sgbm": None}


@pytest.mark.parametrize("i", [1, 2])
@pytest.mark.parametrize("clean", [False, True])
@pytest.mark.parametrize("algo", sorted(CONF))
def test_pair_heights_files_left(tri_env, algo, clean, i):
    from s2p_b200 import fused, rasterio_compat as rio
    s2p, tile, cfg, steps = tri_env(algo, clean)
    eng = RecordingEngine()
    fused.pair_heights(tile, i, engine=eng)
    assert s2p.calls == ["rectification_pair"] and steps == []      # the warps were intercepted, nothing else ran
    left = set(TC.files(tile["dir"]))
    p, other = "pair_%d/" % i, "pair_%d/" % (3 - i)
    conf = {p + CONF[algo]} if CONF[algo] else set()
    untouched = {"mask.png", other + "pointing.txt", other + "sift_matches.txt"}
    if clean:
        assert left == untouched | {p + "height_map.tif"} | conf
    else:
        assert left == untouched | {p + f for f in ("pointing.txt", "sift_matches.txt", "H_ref.txt", "H_sec.txt", "disp_min_max.txt",
                                                    "rectified_ref.tif", "rectified_sec.tif", "rectified_disp.tif",
                                                    "rectified_mask.png", "height_map.tif")} | conf
    (call,) = eng.calls
    assert set(call["want"]) == (set() if clean else {"rect1", "rect2", "disp", "mask"}) | ({"conf"} if conf else set())
    assert call["erode_radius"] == 2 and (call["dmin"], call["dmax"]) == (DMIN, DMAX) and call["tile"] == TILE
    assert (call["weights"] is not None) == (algo == "mgm_multi_lsd")
    # H_sec carries pair i's pointing correction
    A = np.eye(3) if i == 1 else np.diag([1.0, 1.0, 2.0])
    assert np.allclose(call["H_sec"], np.dot(np.round(H2, 6), np.linalg.inv(A)), rtol=0, atol=1e-12)
    # the height map is float64, as common.rasterio_write writes the array triangulation.height_map returns
    hm = rio.read_band_stored(os.path.join(tile["dir"], p + "height_map.tif"))
    assert hm.dtype == np.float64 and hm.shape == (TILE[3], TILE[2]) and (hm == 7.25).all()


def _pair_maps(tile, n, dtype=np.float64):
    from s2p_b200 import rasterio_compat as rio
    for k in range(1, n + 1):
        os.makedirs(os.path.join(tile["dir"], "pair_%d" % k), exist_ok=True)
        m = np.full((TILE[3], TILE[2]), 100.0 + k, dtype)
        if dtype == np.float64:
            rio.write_float64_tiff(os.path.join(tile["dir"], "pair_%d" % k, "height_map.tif"), m)
        else:
            rio.write_float_tiff(os.path.join(tile["dir"], "pair_%d" % k, "height_map.tif"), m)


@pytest.mark.parametrize("basura", [False, True])
@pytest.mark.parametrize("clean", [False, True])
def test_heights_tile_files_left(tri_env, clean, basura):
    from s2p_b200 import fused, rasterio_compat as rio
    s2p, tile, cfg, steps = tri_env("mgm", clean, cargarse_basura=basura)
    _pair_maps(tile, 2)
    eng = RecordingEngine()
    fused.heights_tile(tile, engine=eng)
    assert s2p.calls == [] and steps == []
    left = set(TC.files(tile["dir"]))
    junk = {"pair_%d/%s" % (i, f) for i in (1, 2) for f in ("pointing.txt", "sift_matches.txt")}
    if clean:
        assert left == junk | {"cloud.ply"}
    else:
        assert left == junk | {"cloud.ply", "mask.png", "height_map.tif", "pair_1/height_map.tif", "pair_2/height_map.tif"}
    (call,) = eng.calls
    assert set(call["want"]) == (set() if clean else {"merged"} | ({"cleaned"} if basura else set()))
    assert call["cargarse_basura"] == basura and call["averaging"] == "average_if_close" and call["threshold"] == 3.0
    assert [m.dtype for m in call["maps"]] == [np.float64] * 2 and [float(o) for o in call["offsets"]] == [10.0, 20.0]
    assert call["off"] == TILE[:2] and call["zone"] == 40 and call["south"]
    assert call["colors"] is not None and call["clr"] is None
    if not clean:
        merged = rio.read_band_stored(os.path.join(tile["dir"], "height_map.tif"))
        assert (merged == 3.5).all()
        p1 = rio.read_band_stored(os.path.join(tile["dir"], "pair_1", "height_map.tif"))
        # the cleaned maps replace the pair maps in float32; without the cleaning they stay as they were
        assert (p1.dtype, float(p1[0, 0])) == ((np.float32, 1.5) if basura else (np.float64, 101.0))


def test_heights_tile_reads_float32_maps_as_float32(tri_env):
    from s2p_b200 import fused
    _, tile, _, _ = tri_env("mgm", False, cargarse_basura=False)
    _pair_maps(tile, 2, np.float32)
    eng = RecordingEngine()
    fused.heights_tile(tile, engine=eng)
    assert [m.dtype for m in eng.calls[0]["maps"]] == [np.float32] * 2


def test_heights_tile_missing_map_raises(tri_env):
    from s2p_b200 import fused
    _, tile, _, _ = tri_env("mgm", False)
    _pair_maps(tile, 1)
    eng = RecordingEngine()
    with pytest.raises(Exception):
        fused.heights_tile(tile, engine=eng)
    assert not eng.calls and not os.path.exists(os.path.join(tile["dir"], "cloud.ply"))


@pytest.mark.parametrize("case", ["two_views", "algo"])
def test_pair_heights_fall_through_runs_the_three_steps(tri_env, case):
    from s2p_b200 import fused
    s2p, tile, cfg, steps = tri_env("tvl1" if case == "algo" else "mgm", False, nimages=2 if case == "two_views" else 3)
    assert fused.pair_heights_fall_through_reason(cfg)
    eng = RecordingEngine()
    fused.pair_heights(tile, 1, engine=eng)
    assert not eng.calls
    assert s2p.calls == ["rectification_pair", "stereo_matching", "disparity_to_height"]
    assert [s[0] for s in steps] == ["warp", "warp", "match", "erode", "height_map", "write_height_map"]


def test_pair_heights_ignores_crs_colours_and_numpy(tri_env, monkeypatch, tmp_path):
    from s2p_b200 import cloud, fused
    _, _, cfg, _ = tri_env("mgm", False, out_crs="epsg:2154")
    cfg["images"][0]["clr"] = str(tmp_path / "missing.tif")
    monkeypatch.setattr(cloud, "numpy_stretch_is_float64", lambda: False)
    for algo in CONF:
        cfg["matching_algorithm"] = algo
        assert fused.pair_heights_fall_through_reason(cfg) is None


@pytest.mark.parametrize("case", ["crs", "numpy1", "clr", "colours", "operator", "maps"])
def test_heights_tile_fall_through_runs_heights_to_ply(tri_env, monkeypatch, tmp_path, case):
    from s2p_b200 import cloud, fused, rasterio_compat as rio
    over = {"crs": {"out_crs": "epsg:2154"}, "operator": {"fusion_operator": "np.std"}}.get(case, {})
    s2p, tile, cfg, steps = tri_env("mgm", False, **over)
    _pair_maps(tile, 2)
    if case == "numpy1":
        monkeypatch.setattr(cloud, "numpy_stretch_is_float64", lambda: False)
    if case == "clr":
        cfg["images"][0]["clr"] = str(tmp_path / "missing.tif")
    if case == "colours":                   # int32 colours: not a type the device stretches as the reference does
        cfg["images"][0]["img"] = str(tmp_path / "int.png")
        rio.write_mask_png(cfg["images"][0]["img"], np.ones((H + 10, W + 10), np.uint8))
        monkeypatch.setattr(cloud, "_colours_ok", lambda c: False)
    if case == "maps":
        cfg["images"] += [dict(cfg["images"][1]) for _ in range(15)]
    assert bool(fused.heights_tile_fall_through_reason(cfg)) == (case in ("crs", "numpy1", "operator", "maps"))
    eng = RecordingEngine()
    fused.heights_tile(tile, engine=eng)
    assert not eng.calls
    assert s2p.calls == ["heights_to_ply"] and steps == [("heights_to_ply",)]


def test_heights_tile_serves_every_fusion_operator(tri_env):
    from s2p_b200 import fused
    from s2p_b200.engine import Engine
    _, _, cfg, _ = tri_env("mgm", False)
    for op in list(Engine.FUSION_OPS) + ["numpy.nanmedian"]:
        cfg["fusion_operator"] = op
        assert fused.heights_tile_fall_through_reason(cfg) is None, op
    cfg["images"] += [dict(cfg["images"][1]) for _ in range(14)]        # 16 maps
    assert fused.heights_tile_fall_through_reason(cfg) is None


def test_heights_tile_typed_clr_colours(tri_env, tmp_path):
    from s2p_b200 import fused, rasterio_compat as rio
    _, tile, cfg, _ = tri_env("mgm", False)
    _pair_maps(tile, 2)
    clr = str(tmp_path / "clr.png")
    rio.write_mask_png(clr, np.arange((H + 10) * (W + 10)).reshape(H + 10, W + 10).astype(np.uint8))
    cfg["images"][0]["clr"] = clr
    eng = RecordingEngine()
    fused.heights_tile(tile, engine=eng)
    (call,) = eng.calls
    x, y, w, h = TILE
    assert call["colors"] is None and call["clr"].dtype == np.uint8 and call["clr"].shape == (1, h, w)
    assert np.array_equal(call["clr"][0], rio.read_stored(clr)[0, y:y + h, x:x + w])


def test_pair_heights_timeout_raises_timeout_expired(tri_env):
    from s2p_b200 import _lib, fused
    _, tile, _, _ = tri_env("mgm", False)
    with pytest.raises(subprocess.TimeoutExpired):
        fused.pair_heights(tile, 2, engine=RecordingEngine(_lib.ERR_TIMEOUT))
    assert not os.path.exists(os.path.join(tile["dir"], "pair_2", "height_map.tif"))


def test_pair_heights_other_errors_raise_called_process_error(tri_env):
    from s2p_b200 import _lib, fused
    _, tile, _, _ = tri_env("sgbm", True)
    with pytest.raises(subprocess.CalledProcessError):
        fused.pair_heights(tile, 1, engine=RecordingEngine(_lib.ERR_ARG))


def test_pair_heights_unsupported_replays_the_steps(tri_env):
    from s2p_b200 import _lib, fused
    s2p, tile, _, steps = tri_env("sgbm", True)
    fused.pair_heights(tile, 2, engine=RecordingEngine(_lib.ERR_UNSUPPORTED))
    assert s2p.calls == ["rectification_pair", "stereo_matching", "disparity_to_height"]
    pair = os.path.join(tile["dir"], "pair_2")
    assert steps == [("warp", os.path.join(pair, "rectified_ref.tif")), ("warp", os.path.join(pair, "rectified_sec.tif")),
                     ("match",), ("erode", 2), ("height_map",), ("write_height_map", os.path.join(pair, "height_map.tif"))]


def test_heights_tile_unsupported_runs_heights_to_ply(tri_env):
    from s2p_b200 import _lib, fused
    s2p, tile, _, steps = tri_env("mgm", False)
    _pair_maps(tile, 2)
    fused.heights_tile(tile, engine=RecordingEngine(_lib.ERR_UNSUPPORTED))
    assert s2p.calls == ["heights_to_ply"] and not os.path.exists(os.path.join(tile["dir"], "cloud.ply"))


def test_pair_heights_oversize_range_raises_before_the_device(tri_env):
    from s2p_b200 import fused
    from s2p_b200.block_matching import MaxDisparityRangeError
    _, tile, _, _ = tri_env("mgm", False, max_disp_range=4)
    eng = RecordingEngine()
    with pytest.raises(MaxDisparityRangeError):
        fused.pair_heights(tile, 1, engine=eng)
    assert not eng.calls


def test_float64_height_map_writer(tmp_path):
    """the pair's height map keeps its float64 bits and its NaN through the file"""
    from s2p_b200 import rasterio_compat as rio
    a = np.random.default_rng(3).normal(300.0, 40.0, (17, 23))
    a[4, 5] = np.nan
    f = str(tmp_path / "height_map.tif")
    rio.write_float64_tiff(f, a)
    b = rio.read_band_stored(f)
    assert b.dtype == np.float64 and np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(a[~np.isnan(a)], b[~np.isnan(b)])


def test_heights_tile_struct_matches_the_header(tmp_path):
    """the ctypes mirror of s2pb_heights_tile has the C struct's size and field offsets (gcc on the public header)"""
    import ctypes
    from s2p_b200 import _lib
    names = [f[0] for f in _lib.HeightsTile._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "s2pb200.h"\nint main(void) {\n'
                   '    printf("%zu\\n", sizeof(s2pb_heights_tile));\n    printf("%d\\n", S2PB_MAX_FUSION);\n' +
                   "".join('    printf("%%zu\\n", offsetof(s2pb_heights_tile, %s));\n' % n for n in names) + "    return 0;\n}\n")
    exe = tmp_path / "layout"
    r = subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [ctypes.sizeof(_lib.HeightsTile), _lib.MAX_FUSION] + [getattr(_lib.HeightsTile, n).offset for n in names]
