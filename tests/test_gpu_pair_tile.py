"""A two-view tile from its source crops to its point cloud in one device call (csrc/pair_tile.cu, Engine.pair_tile_to_ply,
s2p_b200.fused.pair_tile), bit for bit with the stepwise path:

- the records and every intermediate of s2pb_pair_tile_to_ply against homography x 2 -> mgm / sgbm -> erode_mask ->
  disp_to_ply[_clr] on the engine, on the real Pleiades pair and on seeded synthetic pairs with no-data strips, for the four
  matchers, the filter on and off, erosion radius 0 and 2, the 8-bit stretch and 1- and 3-band clr colours, with and without
  the confidence column;
- fused.pair_tile on a tile directory under a stub s2p package against the three step drop-ins in sequence: the same files,
  byte for byte, with clean_intermediate on and off; the timeout and the oversize range.
"""
import os
import subprocess

import numpy as np
import pytest

import pair_tile_cases as PT
from util import same

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(int(np.__version__.split(".")[0]) < 2, reason="the device reproduces NumPy >= 2's casting")]

R, PW, N = 5.0, 10, 50          # filter_xyz(r = 5 m, n = 50) at a GSD of 0.5 m
ZONE, SOUTH = 40, True


def _shift(Hm, xy):
    return np.asarray(Hm, np.float64) @ np.array([[1, 0, xy[0]], [0, 1, xy[1]], [0, 0, 1.0]])


def _real():
    """the fixture's crops with their crop-compensated homographies on [-41, 30], H_ref / H_sec as their text files hold them"""
    from s2p_b200.triangulation import rpc_from_geotiff_tag
    from util import load_real_pair
    z = load_real_pair()
    h, w = z["rectified_ref"].shape
    return dict(src1=z["crop1"].astype(np.float32), src2=z["crop2"].astype(np.float32), H1=_shift(z["H1"], z["xy1"]),
                H2=_shift(z["H2"], z["xy2"]), w=w, h=h, dmin=-41, dmax=30, H_ref=z["H1"], H_sec=z["H2"],
                rpc1=rpc_from_geotiff_tag(z["rpc1"]), rpc2=rpc_from_geotiff_tag(z["rpc2"]), mask_orig=np.ones((1024, 1024), np.float32),
                bbx=(0.0, 1023.0, 0.0, 1023.0))


def _synthetic(seed):
    """seeded sources with no-data strips (s2p_b200.synth), each warped by a small affine map onto 200 x 150"""
    from s2p_b200.synth import make_pair
    a = _real()
    ref, sec, _ = make_pair(170, 230, -12, 11, seed=seed, nan_border=0.04)
    rng = np.random.default_rng(seed)
    H1 = np.array([[1.0, 0.002 * rng.standard_normal(), -6.5], [0.0, 1.0, -5.25], [0.0, 0.0, 1.0]])
    H2 = np.array([[1.0, 0.0, -7.0], [0.003 * rng.standard_normal(), 1.0, -5.0], [0.0, 0.0, 1.0]])
    return dict(a, src1=ref, src2=sec, H1=H1, H2=H2, w=200, h=150, dmin=-12, dmax=11, H_ref=np.round(H1, 6), H_sec=np.round(H2, 6))


def _params(engine, algo):
    from s2p_b200.block_matching import SGBM_ARGS, matcher_params
    return engine.sgbm_params(**SGBM_ARGS) if algo == "sgbm" else matcher_params(algo, 0)


def _stepwise(engine, t, algo, weights, erode, filt, colours, conf):
    """the existing calls in sequence, with the conversions of s2p's file round trips (float32 TIFF, 0/1 PNG read as uint8)"""
    rect1 = engine.homography(t["src1"], t["H1"], t["w"], t["h"])
    rect2 = engine.homography(t["src2"], t["H2"], t["w"], t["h"])
    if algo == "sgbm":
        m = engine.sgbm(rect1, rect2, t["dmin"], t["dmax"], _params(engine, algo))
    else:
        m = engine.mgm(rect1, rect2, t["dmin"], t["dmax"], _params(engine, algo), want_right=True, weights=weights)
    mask = engine.erode_mask(m["mask"], erode) if erode else m["mask"]
    r, p, n = (R, PW, N) if filt else (0.0, 0, 0)
    cloud = (m["disp"], mask, t["mask_orig"], t["H_ref"], t["H_sec"], t["rpc1"], t["rpc2"], t["bbx"], ZONE, SOUTH)
    confidence = m["conf"] if conf else None
    if colours == "stretch":
        rec = engine.disp_to_ply(*cloud, r=r, p=p, n=n, colors=rect1[None], confidence=confidence)
    else:
        rec = engine.disp_to_ply_clr(*cloud, r=r, p=p, n=n, clr=colours[0], hc=colours[1], confidence=confidence)
    return rec, dict(m, rect1=rect1, rect2=rect2, mask=mask)


def _clr(t, nbands):
    """a clr crop of nbands float32 planes (the reference crop and two functions of it) and the homography that warps it"""
    c = t["src1"]
    return np.stack([c, 0.5 * c + 3.0, np.sqrt(np.abs(c))][:nbands]).astype(np.float32), t["H1"]


CASES = [  # (tile, algo, filter, erosion radius, colours, confidence column)
    ("real", "mgm", True, 2, "stretch", True),
    ("real", "mgm_multi", True, 2, "stretch", True),
    ("real", "mgm_multi_lsd", True, 2, "stretch", False),
    ("real", "sgbm", True, 2, "stretch", False),
    ("real", "mgm", False, 0, "stretch", False),
    ("real", "mgm_multi", True, 2, 1, True),
    ("real", "mgm", False, 2, 3, False),
    ("synth0", "mgm", True, 2, "stretch", True),
    ("synth1", "mgm_multi", False, 0, 3, True),
    ("synth2", "mgm_multi_lsd", True, 2, 1, False),
    ("synth3", "sgbm", False, 2, "stretch", False),
    ("synth4", "sgbm", True, 0, 3, False),
]


@pytest.mark.parametrize("tile,algo,filt,erode,colours,conf", CASES, ids=["-".join(map(str, c)) for c in CASES])
def test_records_and_intermediates_equal_the_stepwise_calls(engine, tile, algo, filt, erode, colours, conf):
    t = _real() if tile == "real" else _synthetic(int(tile[5:]))
    weights = None
    if algo == "mgm_multi_lsd":       # weights that are not all 1, so that their path through the call shows
        rng = np.random.default_rng(7)
        weights = tuple(rng.uniform(0.25, 1.0, (t["h"], t["w"])).astype(np.float32) for _ in range(2))
    cl = colours if colours == "stretch" else _clr(t, colours)
    want_rec, want = _stepwise(engine, t, algo, weights, erode, filt, cl, conf)
    names = ("rect1", "rect2", "disp", "mask") + (() if algo == "sgbm" else ("conf", "disp_right"))
    r, p, n = (R, PW, N) if filt else (0.0, 0, 0)
    rec, out = engine.pair_tile_to_ply(t["src1"], t["H1"], t["src2"], t["H2"], t["w"], t["h"], t["dmin"], t["dmax"], t["mask_orig"],
                                       t["H_ref"], t["H_sec"], t["rpc1"], t["rpc2"], t["bbx"], ZONE, SOUTH,
                                       params=_params(engine, algo), weights=weights, erode_radius=erode, r=r, p=p, n=n,
                                       clr=None if colours == "stretch" else cl[0], hc=None if colours == "stretch" else cl[1],
                                       confidence=conf, want=names)
    assert 0 < len(want_rec) < t["w"] * t["h"]
    assert rec.dtype == want_rec.dtype and rec.tobytes() == want_rec.tobytes()
    for k in names:
        assert same(out[k], want[k]), k
    # nothing asked, nothing copied back; the records stay the same
    rec2, out2 = engine.pair_tile_to_ply(t["src1"], t["H1"], t["src2"], t["H2"], t["w"], t["h"], t["dmin"], t["dmax"], t["mask_orig"],
                                         t["H_ref"], t["H_sec"], t["rpc1"], t["rpc2"], t["bbx"], ZONE, SOUTH,
                                         params=_params(engine, algo), weights=weights, erode_radius=erode, r=r, p=p, n=n,
                                         clr=None if colours == "stretch" else cl[0], hc=None if colours == "stretch" else cl[1],
                                         confidence=conf)
    assert out2 == {} and rec2.tobytes() == rec.tobytes()


def test_arguments(engine):
    from s2p_b200._lib import ERR_ARG, S2pbError
    t = _real()
    call = lambda **kw: engine.pair_tile_to_ply(t["src1"], t["H1"], t["src2"], t["H2"], t["w"], t["h"], t["dmin"], t["dmax"],
                                                t["mask_orig"], t["H_ref"], t["H_sec"], t["rpc1"], t["rpc2"], t["bbx"], ZONE, SOUTH, **kw)
    for kw in (dict(params=engine.sgbm_params(), confidence=True), dict(params=engine.sgbm_params(), want=("conf",)),
               dict(erode_radius=1.0), dict(erode_radius=65.0), dict(clr=np.zeros((2, 8, 8), np.float32), hc=np.eye(3))):
        with pytest.raises(S2pbError) as e:
            call(**kw)
        assert e.value.code == ERR_ARG, kw


# ------------------------------------------------------------------ the tile step on a tile directory

def _tile_setup(tmp_path, monkeypatch, algo, clean, clr=False, t=None, name="fused"):
    """(stub s2p, tile, cfg) for a tile of the real pair: source images as files, the three steps as the drop-ins run them"""
    from s2p_b200 import block_matching, cloud, common, masking, rasterio_compat as rio
    t = t or _real()
    img1, img2 = str(tmp_path / "img_01.tif"), str(tmp_path / "img_02.tif")
    if not os.path.exists(img1):
        rio.write_float_tiff(img1, t["src1"])
        rio.write_float_tiff(img2, t["src2"])
        rio.write_float_tiff_bands(str(tmp_path / "clr.tif"), list(_clr(t, 3)[0]))
        np.savetxt(str(tmp_path / "global_pointing_pair_1.txt"), np.eye(3))
    cfg = PT.cfg_for(tmp_path, img1, img2, t["rpc1"], t["rpc2"], algo, clean, str(tmp_path / "clr.tif") if clr else None)
    s2p = PT.stub_s2p(monkeypatch, cfg, t["H1"], t["H2"], t["w"], t["h"], float(t["dmin"]), float(t["dmax"]), common.image_apply_homography,
                      block_matching.compute_disparity_map, masking.erosion, cloud.disparity_to_ply)
    return s2p, PT.make_tile(tmp_path, name, (1024, 1024)), cfg


@pytest.mark.parametrize("clean", [False, True])
@pytest.mark.parametrize("algo,clr", [("mgm", False), ("mgm_multi", True), ("mgm_multi_lsd", False), ("sgbm", False)])
def test_pair_tile_leaves_the_files_of_the_three_steps(engine, tmp_path, monkeypatch, algo, clr, clean):
    from s2p_b200 import fused
    s2p, stepwise_tile, _ = _tile_setup(tmp_path, monkeypatch, algo, clean, clr, name="stepwise")
    s2p.rectification_pair(stepwise_tile, 1)
    s2p.stereo_matching(stepwise_tile, 1)
    s2p.disparity_to_ply(stepwise_tile)
    s2p, tile, _ = _tile_setup(tmp_path, monkeypatch, algo, clean, clr)
    k0 = engine.kernel_launches()
    fused.pair_tile(tile, engine=engine)
    assert engine.kernel_launches() > k0
    assert s2p.calls == ["rectification_pair"]
    want, got = PT.files(stepwise_tile["dir"]), PT.files(tile["dir"])
    assert sorted(got) == sorted(want)
    for name in want:
        assert got[name] == want[name], name
    assert "cloud.ply" in got and (not clean or len(got) <= 2)


def test_pair_tile_timeout(engine, tmp_path, monkeypatch):
    """a matcher over its time limit raises subprocess.TimeoutExpired, as compute_disparity_map does, and writes no cloud"""
    from s2p_b200 import fused
    from s2p_b200.synth import make_pair
    ref, sec, _ = make_pair(512, 512, -100, 100, seed=1)
    t = dict(_real(), src1=ref, src2=sec, H1=np.eye(3), H2=np.eye(3), w=512, h=512, dmin=-100, dmax=100)
    _, tile, cfg = _tile_setup(tmp_path, monkeypatch, "mgm", False, t=t)
    cfg["mgm_timeout"] = 0.001
    with pytest.raises(subprocess.TimeoutExpired):
        fused.pair_tile(tile, engine=engine)
    assert not os.path.exists(os.path.join(tile["dir"], "cloud.ply"))
    # the engine stays usable
    cfg["mgm_timeout"] = 600
    fused.pair_tile(tile, engine=engine)
    assert os.path.exists(os.path.join(tile["dir"], "cloud.ply"))


def test_pair_tile_oversize_range(engine, tmp_path, monkeypatch):
    from s2p_b200 import fused
    from s2p_b200.block_matching import MaxDisparityRangeError
    _, tile, cfg = _tile_setup(tmp_path, monkeypatch, "mgm", False)
    cfg["max_disp_range"] = 50
    k0 = engine.kernel_launches()
    with pytest.raises(MaxDisparityRangeError):
        fused.pair_tile(tile, engine=engine)
    assert engine.kernel_launches() == k0
