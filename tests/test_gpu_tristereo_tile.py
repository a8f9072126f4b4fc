"""A tri-stereo tile from its source crops to its point cloud in two device calls (csrc/pair_tile.cu, csrc/heights_tile.cu,
Engine.pair_tile_to_height_map / heights_tile_to_ply, s2p_b200.fused.pair_heights / heights_tile), bit for bit with the stepwise
path:

- s2pb_pair_tile_to_height_map against homography x 2 -> mgm / sgbm -> erode_mask -> height_map on the engine: the heights, their
  NaN set and every intermediate, for the four matchers and erosion radius 0 and 2, on the real Pleiades pair and on seeded
  synthetic pairs with no-data strips;
- s2pb_heights_tile_to_ply against cargarse_basura -> merge_n -> height_map_to_ply[_clr] with the cleaning, and against a NumPy
  restatement of s2p.fusion.merge_n on the float64 maps -> height_map_to_ply[_clr] without it, for every operator, 2 and 3 maps,
  the stretch colours and a typed clr window;
- fused.pair_heights and fused.heights_tile on tile directories under a stub s2p package against the step drop-ins in sequence:
  the same files, byte for byte, with clean_intermediate on and off; the matcher's timeout.
"""
import os
import subprocess

import numpy as np
import pytest

import tristereo_cases as TC
from util import same

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(int(np.__version__.split(".")[0]) < 2, reason="the device reproduces NumPy >= 2's casting")]

R, PW, N = 5.0, 10, 50          # filter_xyz(r = 5 m, n = 50) at a GSD of 0.5 m
POINTING = np.array([[1.000186, 0.000156, 0.518804], [0.000040, 1.000032, 0.109895], [0.0, 0.0, 1.0]])


def _shift(Hm, xy):
    return np.asarray(Hm, np.float64) @ np.array([[1, 0, xy[0]], [0, 1, xy[1]], [0, 0, 1.0]])


def _real():
    """the fixture's crops with their crop-compensated homographies on [-41, 30], the tile (500, 150, 350, 350) of the
    reference image with a hole in its mask, H_sec with the reference's pointing correction"""
    from s2p_b200.triangulation import rpc_from_geotiff_tag
    from util import load_real_pair
    z = load_real_pair()
    h, w = z["rectified_ref"].shape
    mo = np.ones((350, 350), np.uint8)
    mo[100:140, 200:260] = 0
    return dict(src1=z["crop1"].astype(np.float32), src2=z["crop2"].astype(np.float32), H1=_shift(z["H1"], z["xy1"]),
                H2=_shift(z["H2"], z["xy2"]), w=w, h=h, dmin=-41, dmax=30, H_ref=z["H1"], H_sec=np.dot(z["H2"], np.linalg.inv(POINTING)),
                rpc1=rpc_from_geotiff_tag(z["rpc1"]), rpc2=rpc_from_geotiff_tag(z["rpc2"]), mask_orig=mo, tile=(500, 150, 350, 350),
                Hr1=z["H1"], Hr2=z["H2"], xy1=tuple(int(v) for v in z["xy1"]), xy2=tuple(int(v) for v in z["xy2"]))


def _synthetic(seed):
    """seeded sources with no-data strips (s2p_b200.synth), each warped by a small affine map onto 200 x 150, triangulated with
    the real pair's cameras on a tile inside the sources"""
    from s2p_b200.synth import make_pair
    a = _real()
    ref, sec, _ = make_pair(170, 230, -12, 11, seed=seed, nan_border=0.04)
    rng = np.random.default_rng(seed)
    H1 = np.array([[1.0, 0.002 * rng.standard_normal(), -6.5], [0.0, 1.0, -5.25], [0.0, 0.0, 1.0]])
    H2 = np.array([[1.0, 0.0, -7.0], [0.003 * rng.standard_normal(), 1.0, -5.0], [0.0, 0.0, 1.0]])
    mo = (rng.random((120, 160)) > 0.02).astype(np.uint8)
    return dict(a, src1=ref, src2=sec, H1=H1, H2=H2, w=200, h=150, dmin=-12, dmax=11, mask_orig=mo, tile=(10, 8, 160, 120),
                H_ref=np.round(H1, 6), H_sec=np.dot(np.round(H2, 6), np.linalg.inv(POINTING)), Hr1=H1, Hr2=H2, xy1=(0, 0), xy2=(0, 0))


def _params(engine, algo):
    from s2p_b200.block_matching import SGBM_ARGS, matcher_params
    return engine.sgbm_params(**SGBM_ARGS) if algo == "sgbm" else matcher_params(algo, 0)


def _weights(t, algo):
    if algo != "mgm_multi_lsd":
        return None
    rng = np.random.default_rng(7)       # weights that are not all 1, so that their path through the call shows
    return tuple(rng.uniform(0.25, 1.0, (t["h"], t["w"])).astype(np.float32) for _ in range(2))


PAIR_CASES = [  # (pair, algo, erosion radius)
    ("real", "mgm", 2), ("real", "mgm_multi", 0), ("real", "mgm_multi_lsd", 2), ("real", "sgbm", 2), ("real", "mgm", 0),
    ("synth0", "mgm", 2), ("synth1", "mgm_multi", 2), ("synth2", "mgm_multi_lsd", 0), ("synth3", "sgbm", 0), ("synth4", "sgbm", 2),
]


@pytest.mark.parametrize("pair,algo,erode", PAIR_CASES, ids=["-".join(map(str, c)) for c in PAIR_CASES])
def test_pair_height_map_equals_the_stepwise_calls(engine, pair, algo, erode):
    t = _real() if pair == "real" else _synthetic(int(pair[5:]))
    weights = _weights(t, algo)
    rect1 = engine.homography(t["src1"], t["H1"], t["w"], t["h"])
    rect2 = engine.homography(t["src2"], t["H2"], t["w"], t["h"])
    if algo == "sgbm":
        m = engine.sgbm(rect1, rect2, t["dmin"], t["dmax"], _params(engine, algo))
    else:
        m = engine.mgm(rect1, rect2, t["dmin"], t["dmax"], _params(engine, algo), want_right=True, weights=weights)
    mask = engine.erode_mask(m["mask"], erode) if erode else m["mask"]
    x, y, tw, th = t["tile"]
    want_h = engine.height_map(x, y, tw, th, t["rpc1"], t["rpc2"], t["H_ref"], t["H_sec"], m["disp"], mask, t["mask_orig"])
    want = dict(m, rect1=rect1, rect2=rect2, mask=mask)

    names = ("rect1", "rect2", "disp", "mask") + (() if algo == "sgbm" else ("conf", "disp_right"))
    args = (t["src1"], t["H1"], t["src2"], t["H2"], t["w"], t["h"], t["dmin"], t["dmax"], t["mask_orig"], t["H_ref"], t["H_sec"],
            t["rpc1"], t["rpc2"], t["tile"])
    got_h, out = engine.pair_tile_to_height_map(*args, params=_params(engine, algo), weights=weights, erode_radius=erode, want=names)
    assert got_h.dtype == np.float64 and got_h.shape == (th, tw)
    assert np.array_equal(np.isnan(got_h), np.isnan(want_h))
    assert np.isfinite(got_h).any() and np.isnan(got_h).any()
    assert got_h.tobytes() == want_h.tobytes()
    for k in names:
        assert same(out[k], want[k]), k
    got2, out2 = engine.pair_tile_to_height_map(*args, params=_params(engine, algo), weights=weights, erode_radius=erode)
    assert out2 == {} and got2.tobytes() == got_h.tobytes()


def test_pair_height_map_arguments(engine):
    from s2p_b200._lib import ERR_ARG, ERR_UNSUPPORTED, S2pbError
    t = _real()
    args = lambda **o: tuple(dict(t, **o)[k] for k in ("src1", "H1", "src2", "H2", "w", "h", "dmin", "dmax", "mask_orig", "H_ref",
                                                       "H_sec", "rpc1", "rpc2", "tile"))
    for o, kw, code in ((dict(), dict(params=engine.sgbm_params(), want=("conf",)), ERR_ARG),
                        (dict(), dict(erode_radius=1.0), ERR_ARG),
                        (dict(H_ref=np.array([[1.0, 0, 0], [0, 1, 0], [1e-9, 0, 1]])), dict(), ERR_ARG),
                        (dict(h=1), dict(), ERR_UNSUPPORTED)):
        with pytest.raises(S2pbError) as e:
            engine.pair_tile_to_height_map(*args(**o), **kw)
        assert e.value.code == code, (o, kw)


# ------------------------------------------------------------------ the heights of a tile to its cloud

def _triplet_maps(nmaps, seed, crop=(slice(100, 220), slice(100, 260))):
    """nmaps float64 height maps around a window of the triplet's merged map, each with its own offset, noise, NaN holes and
    small raised islands that the cleaning removes, and their seeded offsets"""
    import localization_oracle as LO
    t = LO.triplet()
    base = t["heights"][crop].astype(np.float64)
    rng = np.random.default_rng(seed)
    offsets = list(rng.uniform(-3.0, 3.0, nmaps))
    maps = []
    for k in range(nmaps):
        m = base + offsets[k] + rng.normal(0.0, 0.7, base.shape) + rng.uniform(-1e-3, 1e-3, base.shape)
        m[rng.random(base.shape) < 0.03] = np.nan
        i, j = rng.integers(10, base.shape[0] - 20), rng.integers(10, base.shape[1] - 20)
        m[i:i + 6, j:j + 8] = np.nan                        # a hole
        i, j = rng.integers(10, base.shape[0] - 20), rng.integers(10, base.shape[1] - 20)
        m[i:i + 5, j:j + 5] += 40.0                         # an island
        maps.append(m)
    rpc = LO.triplet_rpc()
    return maps, [np.array(o) for o in offsets], rpc, float(t["off"][0]) + crop[1].start, float(t["off"][1]) + crop[0].start


def _colours(shape, kind, seed=4):
    rng = np.random.default_rng(seed)
    if kind == "stretch":
        return dict(colors=rng.integers(100, 3000, (3,) + shape).astype(np.uint16))
    return dict(clr=rng.integers(0, 60000, (1,) + shape).astype(np.uint16))


def _to_ply(engine, merged, rpc, ox, oy, colours):
    args = (merged.astype(np.float64), rpc, ox, oy, 31, False)
    if "clr" in colours:
        return engine.height_map_to_ply_clr(*args, r=R, p=PW, n=N, colors=colours["clr"])
    return engine.height_map_to_ply(*args, r=R, p=PW, n=N, colors=colours["colors"])


def _fusion_ops():
    from s2p_b200.engine import Engine
    return sorted(Engine.FUSION_OPS)


HEIGHTS_CASES = [(op, nmaps, basura) for op in _fusion_ops() for nmaps in (2, 3) for basura in (True, False)]


@pytest.mark.parametrize("op,nmaps,basura", HEIGHTS_CASES, ids=["%s-%d-%s" % (o, k, "basura" if b else "raw") for o, k, b in HEIGHTS_CASES])
def test_heights_tile_equals_the_stepwise_path(engine, op, nmaps, basura):
    k = HEIGHTS_CASES.index((op, nmaps, basura))
    maps, offsets, rpc, ox, oy = _triplet_maps(nmaps, seed=k)
    colours = _colours(maps[0].shape, "stretch" if k % 2 else "clr")
    thr = 1.5
    if basura:
        cleaned = [engine.cargarse_basura(m) for m in maps]
        merged = engine.merge_n(cleaned, offsets, op, thr, sub_f32=False)
    else:
        merged = TC.merge_n_numpy(maps, offsets, op, thr)
        # the float32 route, which rounds each map before the subtraction, would not give this map
        assert not same(engine.merge_n([m.astype(np.float32) for m in maps], offsets, op, thr, sub_f32=False), merged)
    want = _to_ply(engine, merged, rpc, ox, oy, colours)
    rec, out = engine.heights_tile_to_ply(maps, offsets, rpc, ox, oy, 31, False, cargarse_basura=basura, averaging=op, threshold=thr,
                                          sub_f32=False, r=R, p=PW, n=N, want=("merged",) + (("cleaned",) if basura else ()),
                                          **colours)
    assert same(out["merged"], merged)
    assert np.isfinite(merged).mean() > 0.3
    if basura:
        assert len(out["cleaned"]) == nmaps and all(same(a, b) for a, b in zip(out["cleaned"], cleaned))
        assert all((np.isnan(c) & ~np.isnan(m)).any() for c, m in zip(cleaned, maps))       # the cleaning removed something
    assert 0 < len(want) and rec.dtype == want.dtype and rec.tobytes() == want.tobytes()


def test_heights_tile_float32_maps(engine):
    """float32 maps merge as s2pb_merge_n merges them"""
    maps, offsets, rpc, ox, oy = _triplet_maps(3, seed=99)
    maps = [m.astype(np.float32) for m in maps]
    merged = engine.merge_n(maps, offsets, "average_if_close", 1.5, sub_f32=False)
    rec, out = engine.heights_tile_to_ply(maps, offsets, rpc, ox, oy, 31, False, threshold=1.5, sub_f32=False, r=R, p=PW, n=N,
                                          want=("merged",), **_colours(maps[0].shape, "stretch"))
    assert same(out["merged"], merged)
    assert rec.tobytes() == _to_ply(engine, merged, rpc, ox, oy, _colours(maps[0].shape, "stretch")).tobytes()


# ------------------------------------------------------------------ the tile steps on tile directories

def _canvas(src, xy):
    """the source crop at its place in an image of zeros, which is all the warp reads of the original image"""
    a = np.zeros((xy[1] + src.shape[0], xy[0] + src.shape[1]), np.float32)
    a[xy[1]:, xy[0]:] = src
    return a


def _pair_setup(tmp_path, monkeypatch, algo, clean, t, name):
    """(stub s2p, tile, cfg) of a three-image run on the real pair (image 3 = image 2, pair 2 with its own pointing): source
    images as files, the steps as the drop-ins run them"""
    from s2p_b200 import block_matching, common, masking, rasterio_compat as rio, triangulation
    img1, img2 = str(tmp_path / "img_01.tif"), str(tmp_path / "img_02.tif")
    if not os.path.exists(img1):
        rio.write_float_tiff(img1, _canvas(t["src1"], t["xy1"]))
        rio.write_float_tiff(img2, _canvas(t["src2"], t["xy2"]))
        np.savetxt(str(tmp_path / "global_pointing_pair_1.txt"), np.eye(3))
        np.savetxt(str(tmp_path / "global_pointing_pair_2.txt"), POINTING)
    cfg = TC.cfg_for(tmp_path, [img1, img2, img2], [t["rpc1"], t["rpc2"], t["rpc2"]], algo, clean)
    s2p = TC.stub_s2p(monkeypatch, cfg, t["Hr1"], t["Hr2"], t["w"], t["h"], float(t["dmin"]), float(t["dmax"]), common.image_apply_homography,
                      block_matching.compute_disparity_map, masking.erosion, height_map=triangulation.height_map,
                      write_height_map=rio.write_float64_tiff)
    tile = TC.make_tile(tmp_path, name, t["tile"], 2)
    rio.write_mask_png(os.path.join(tile["dir"], "mask.png"), t["mask_orig"])
    return s2p, tile, cfg


@pytest.mark.parametrize("clean", [False, True])
@pytest.mark.parametrize("algo,i", [("mgm", 1), ("mgm_multi_lsd", 2), ("sgbm", 2)])
def test_pair_heights_leaves_the_files_of_the_three_steps(engine, tmp_path, monkeypatch, algo, i, clean):
    from s2p_b200 import fused
    t = _real()
    s2p, stepwise_tile, _ = _pair_setup(tmp_path, monkeypatch, algo, clean, t, "stepwise")
    s2p.rectification_pair(stepwise_tile, i)
    s2p.stereo_matching(stepwise_tile, i)
    s2p.disparity_to_height(stepwise_tile, i)
    s2p, tile, _ = _pair_setup(tmp_path, monkeypatch, algo, clean, t, "fused")
    k0 = engine.kernel_launches()
    fused.pair_heights(tile, i, engine=engine)
    assert engine.kernel_launches() > k0
    assert s2p.calls == ["rectification_pair"]
    want, got = TC.files(stepwise_tile["dir"]), TC.files(tile["dir"])
    assert sorted(got) == sorted(want)
    for name in want:
        assert got[name] == want[name], name
    assert "pair_%d/height_map.tif" % i in got


def test_pair_heights_timeout(engine, tmp_path, monkeypatch):
    """a matcher over its time limit raises subprocess.TimeoutExpired, as compute_disparity_map does, and writes no height map"""
    from s2p_b200 import fused
    from s2p_b200.synth import make_pair
    ref, sec, _ = make_pair(512, 512, -100, 100, seed=1)
    t = dict(_real(), src1=ref, src2=sec, Hr1=np.eye(3), Hr2=np.eye(3), xy1=(0, 0), xy2=(0, 0), w=512, h=512, dmin=-100, dmax=100)
    _, tile, cfg = _pair_setup(tmp_path, monkeypatch, "mgm", False, t, "fused")
    cfg["mgm_timeout"] = 0.001
    with pytest.raises(subprocess.TimeoutExpired):
        fused.pair_heights(tile, 1, engine=engine)
    assert not os.path.exists(os.path.join(tile["dir"], "pair_1", "height_map.tif"))


def _heights_setup(tmp_path, monkeypatch, basura, clean, clr, name):
    """(stub s2p, tile) of a three-image tile whose pair height maps are float64 files, heights_to_ply the cloud drop-in over the
    stub's heights_fusion (cargarse_basura and merge_n drop-ins with the cleaning, the NumPy restatement of merge_n without)"""
    import cv2
    from s2p_b200 import cloud, common, fusion, rasterio_compat as rio
    maps, offsets, rpc, ox, oy = _triplet_maps(2, seed=5)
    h, w = maps[0].shape
    x, y = int(ox), int(oy)
    img = str(tmp_path / "img.tif")
    if not os.path.exists(img):
        full = np.zeros((3, y + h + 5, x + w + 5), np.uint16)
        full[:, y:y + h, x:x + w] = _colours((h, w), "stretch")["colors"]
        assert cv2.imwrite(img, np.ascontiguousarray(np.moveaxis(full, 0, 2)[..., ::-1]))
        assert cv2.imwrite(str(tmp_path / "clr.tif"), full[0])
        for k, o in enumerate(offsets):
            np.savetxt(str(tmp_path / ("global_mean_height_pair_%d.txt" % (k + 1))), [o])
    cfg = TC.cfg_for(tmp_path, [img, img, img], [rpc, rpc, rpc], "mgm", clean, basura=basura,
                     clr=str(tmp_path / "clr.tif") if clr else None)
    cfg.update(out_crs="epsg:32631", fusion_thresh=1.5)
    s2p = TC.stub_s2p(monkeypatch, cfg, np.eye(3), np.eye(3), 8, 8, -1.0, 1.0, None, None, None,
                      cargarse_basura=common.cargarse_basura, merge_n=fusion.merge_n if basura else TC.merge_n_file,
                      heights_to_ply=cloud.heights_to_ply)
    tile = TC.make_tile(tmp_path, name, (x, y, w, h), 2)
    for k, m in enumerate(maps):
        rio.write_float64_tiff(os.path.join(tile["dir"], "pair_%d" % (k + 1), "height_map.tif"), m)
    return s2p, tile


@pytest.mark.parametrize("clean", [False, True])
@pytest.mark.parametrize("basura,clr", [(True, False), (False, False), (True, True)])
def test_heights_tile_leaves_the_files_of_heights_to_ply(engine, tmp_path, monkeypatch, basura, clr, clean):
    from s2p_b200 import fused
    s2p, stepwise_tile = _heights_setup(tmp_path, monkeypatch, basura, clean, clr, "stepwise")
    s2p.heights_to_ply(stepwise_tile)
    assert s2p.calls == ["heights_to_ply", "heights_fusion"]
    s2p, tile = _heights_setup(tmp_path, monkeypatch, basura, clean, clr, "fused")
    k0 = engine.kernel_launches()
    fused.heights_tile(tile, engine=engine)
    assert engine.kernel_launches() > k0 and s2p.calls == []
    want, got = TC.files(stepwise_tile["dir"]), TC.files(tile["dir"])
    assert sorted(got) == sorted(want)
    for name in want:
        assert got[name] == want[name], name
    assert "cloud.ply" in got and (not clean or "height_map.tif" not in got)
