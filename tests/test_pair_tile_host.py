"""CPU tests of s2p_b200.fused.pair_tile's host side, with an engine that records its calls: the files a two-view tile is left
with (clean_intermediate or not), the confidence-column rule, the erosion radius, the fall-through decisions and the errors; and
the ctypes mirror of s2pb_pair_tile against the C header."""
import os
import subprocess

import numpy as np
import pytest

import pair_tile_cases as PT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, H, DMIN, DMAX = 40, 30, -5.0, 5.0
H1 = np.array([[1.0, 0.0, -3.0], [0.0, 1.0, -2.0], [0.0, 0.0, 1.0]])
H2 = np.array([[1.0, 0.01, -4.0], [0.0, 1.0, -2.5], [0.0, 0.0, 1.0]])


class RecordingEngine:
    """pair_tile_to_ply's contract without a device: constant intermediates, three records"""

    def __init__(self, error=None):
        self.calls, self.error = [], error

    @staticmethod
    def sgbm_params(**kw):
        from s2p_b200.engine import Engine
        return Engine.sgbm_params(**kw)

    def pair_tile_to_ply(self, src1, H1, src2, H2, w, h, dmin, dmax, mask_orig, *args, **kw):
        from s2p_b200.engine import Engine, S2pbError
        self.calls.append(dict(kw, dmin=dmin, dmax=dmax, w=w, h=h))
        if self.error is not None:
            raise S2pbError(self.error, "refused")
        out = {k: np.ones((h, w), np.uint8 if k == "mask" else np.float32) for k in kw["want"]}
        return np.zeros(3, Engine.ply_dtype(1, kw["confidence"])), out


@pytest.fixture
def tile_env(tmp_path, monkeypatch):
    """-> make(algo, clean, **cfg overrides) -> (s2p stub, tile, cfg, calls of the stand-ins)"""
    from s2p_b200 import rasterio_compat as rio
    from s2p_b200.triangulation import rpc_from_geotiff_tag
    from util import load_real_pair
    z = load_real_pair()
    rng = np.random.default_rng(0)
    img1, img2 = str(tmp_path / "img1.tif"), str(tmp_path / "img2.tif")
    rio.write_float_tiff(img1, rng.random((H + 10, W + 10)).astype(np.float32))
    rio.write_float_tiff(img2, rng.random((H + 10, W + 10)).astype(np.float32))
    np.savetxt(str(tmp_path / "global_pointing_pair_1.txt"), np.eye(3))
    rpc1, rpc2 = rpc_from_geotiff_tag(z["rpc1"]), rpc_from_geotiff_tag(z["rpc2"])

    def make(algo, clean, **over):
        steps = []
        cfg = PT.cfg_for(tmp_path, img1, img2, rpc1, rpc2, algo, clean)
        cfg.update(over)
        s2p = PT.stub_s2p(monkeypatch, cfg, H1, H2, W, H, DMIN, DMAX,
                          lambda out, im, Hm, w, h: steps.append(("warp", out)),
                          lambda *a, **k: steps.append(("match",)),
                          lambda out, msk, r: steps.append(("erode", r)),
                          lambda tile: steps.append(("ply",)))
        tile = PT.make_tile(tmp_path, "tile_%s_%d" % (algo, clean), (H, W))
        return s2p, tile, cfg, steps
    return make


CONF = {"mgm": "pair_1/rectified_disp_confidence.tif", "mgm_multi": "pair_1/rectified_disp_confidence.tif",
        "mgm_multi_lsd": "pair_1/rectified_disp.tif.confidence.tif", "sgbm": None}


@pytest.mark.parametrize("clean", [False, True])
@pytest.mark.parametrize("algo", sorted(CONF))
def test_files_left_and_confidence_column(tile_env, algo, clean):
    from s2p_b200 import fused
    s2p, tile, cfg, steps = tile_env(algo, clean)
    eng = RecordingEngine()
    fused.pair_tile(tile, engine=eng)
    assert s2p.calls == ["rectification_pair"] and steps == []      # the warps were intercepted, nothing else ran
    left = set(PT.files(tile["dir"]))
    conf = {CONF[algo]} if CONF[algo] else set()
    if clean:
        assert left == {"cloud.ply"} | conf
    else:
        assert left == {"mask.png", "cloud.ply", "pair_1/pointing.txt", "pair_1/sift_matches.txt", "pair_1/H_ref.txt",
                        "pair_1/H_sec.txt", "pair_1/disp_min_max.txt", "pair_1/rectified_ref.tif", "pair_1/rectified_sec.tif",
                        "pair_1/rectified_disp.tif", "pair_1/rectified_mask.png"} | conf
    (call,) = eng.calls
    # only the rasters that stay are asked for
    assert set(call["want"]) == (set() if clean else {"rect1", "rect2", "disp", "mask"}) | ({"conf"} if conf else set())
    # the PLY gets a confidence column when disparity_to_ply finds rectified_disp_confidence.tif
    assert call["confidence"] == (algo in ("mgm", "mgm_multi"))
    with open(os.path.join(tile["dir"], "cloud.ply"), "rb") as f:
        assert (b"property float confidence" in f.read()) == (algo in ("mgm", "mgm_multi"))
    assert call["erode_radius"] == 2 and (call["dmin"], call["dmax"]) == (DMIN, DMAX)
    assert (call["weights"] is not None) == (algo == "mgm_multi_lsd")


def test_erosion_radius():
    from s2p_b200.fused import erosion_radius
    assert [erosion_radius(r) for r in (0, 1, 1.9, 2, 2.7, 5)] == [0, 0, 0, 2, 2, 5]


@pytest.mark.parametrize("case", ["crs", "algo", "clr", "numpy1"])
def test_fall_through_runs_the_three_steps(tile_env, monkeypatch, tmp_path, case):
    from s2p_b200 import cloud, fused
    over = {"crs": {"out_crs": "epsg:2154"}, "algo": {"matching_algorithm": "tvl1"}, "numpy1": {}, "clr": {}}[case]
    s2p, tile, cfg, steps = tile_env("mgm", False, **over)
    if case == "clr":
        cfg["images"][0]["clr"] = str(tmp_path / "missing.tif")
    if case == "numpy1":
        monkeypatch.setattr(cloud, "numpy_stretch_is_float64", lambda: False)
    assert fused.fall_through_reason(cfg)
    eng = RecordingEngine()
    fused.pair_tile(tile, engine=eng)
    assert not eng.calls
    assert s2p.calls == ["rectification_pair", "stereo_matching", "disparity_to_ply"]
    assert [s[0] for s in steps] == ["warp", "warp", "match", "erode", "ply"]


def test_served_configurations_do_not_fall_through(tile_env):
    from s2p_b200 import fused
    for algo in CONF:
        _, _, cfg, _ = tile_env(algo, False)
        assert fused.fall_through_reason(cfg) is None
        cfg["out_crs"] = "epsg:4326"
        assert fused.fall_through_reason(cfg) is None
        cfg["images"].append(dict(cfg["images"][1]))
        assert fused.fall_through_reason(cfg)


def test_timeout_raises_timeout_expired(tile_env):
    from s2p_b200 import _lib, fused
    _, tile, _, _ = tile_env("mgm", False)
    with pytest.raises(subprocess.TimeoutExpired):
        fused.pair_tile(tile, engine=RecordingEngine(_lib.ERR_TIMEOUT))
    assert not os.path.exists(os.path.join(tile["dir"], "cloud.ply"))


def test_other_errors_raise_called_process_error(tile_env):
    from s2p_b200 import _lib, fused
    _, tile, _, _ = tile_env("sgbm", True)
    with pytest.raises(subprocess.CalledProcessError):
        fused.pair_tile(tile, engine=RecordingEngine(_lib.ERR_ARG))


def test_unsupported_tile_replays_the_steps(tile_env):
    """a tile the device refuses as unsupported goes through the steps after the rectification: its warps, then the matcher
    step and the cloud step, whose own error (or tool) decides"""
    from s2p_b200 import _lib, fused
    s2p, tile, _, steps = tile_env("sgbm", True)
    fused.pair_tile(tile, engine=RecordingEngine(_lib.ERR_UNSUPPORTED))
    assert s2p.calls == ["rectification_pair", "stereo_matching", "disparity_to_ply"]
    pair = os.path.join(tile["dir"], "pair_1")
    assert steps == [("warp", os.path.join(pair, "rectified_ref.tif")), ("warp", os.path.join(pair, "rectified_sec.tif")),
                     ("match",), ("erode", 2), ("ply",)]


def test_oversize_range_raises_before_the_device(tile_env):
    from s2p_b200 import fused
    from s2p_b200.block_matching import MaxDisparityRangeError
    _, tile, _, _ = tile_env("mgm", False, max_disp_range=4)
    eng = RecordingEngine()
    with pytest.raises(MaxDisparityRangeError):
        fused.pair_tile(tile, engine=eng)
    assert not eng.calls


def test_pair_tile_struct_matches_the_header(tmp_path):
    """the ctypes mirror of s2pb_pair_tile has the C struct's size and field offsets (gcc on the public header)"""
    import ctypes
    from s2p_b200 import _lib
    names = [f[0] for f in _lib.PairTile._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "s2pb200.h"\nint main(void) {\n'
                   '    printf("%zu\\n", sizeof(s2pb_pair_tile));\n' +
                   "".join('    printf("%%zu\\n", offsetof(s2pb_pair_tile, %s));\n' % n for n in names) + "    return 0;\n}\n")
    exe = tmp_path / "layout"
    r = subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [ctypes.sizeof(_lib.PairTile)] + [getattr(_lib.PairTile, n).offset for n in names]
