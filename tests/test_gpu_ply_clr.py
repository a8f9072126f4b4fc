"""The tile's point cloud coloured from a `clr` image in its own type (csrc/cloud.cu, s2p_b200/cloud.py), bit for bit with the
reference's writer restated in tests/ply_oracle.py:

- s2pb_ply_records_typed for the eight PLY colour types, 1, 3 and 4 bands, with and without confidence;
- s2pb_disp_to_ply_clr against Engine.homography of each band of the crop, then the writer;
- s2pb_height_map_to_ply_clr against height_map_to_xyz, the filter, then the writer;
- the step drop-ins on a tile directory with a multi-band clr TIFF, their fall-throughs, and the ushort-coloured cloud
  through the DSM rasterisation.
"""
import os
import sys

import numpy as np
import pytest

import dsm_oracle as D
import dsm_typed_oracle as DT
import ply_oracle as P
from test_gpu_ply import N, PW, R, _cfg, _real, _stub_s2p, _triplet
from util import same

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(int(np.__version__.split(".")[0]) < 2, reason="the device reproduces NumPy >= 2's casting")]

TYPES = [np.int8, np.uint8, np.int16, np.uint16, np.int32, np.uint32, np.float32, np.float64]
PLY_NAMES = dict(zip(TYPES, ["char", "uchar", "short", "ushort", "int", "uint", "float", "double"]))
COMMENTS = ["created by S2P", "projection: CRS epsg:32740"]


def _colours(rng, dtype, shape):
    """seeded colours over the whole range of an integer type; normal floats with NaN, ±inf and signed zeros"""
    if np.dtype(dtype).kind in "iu":
        info = np.iinfo(dtype)
        return rng.integers(info.min, int(info.max) + 1, shape, dtype=np.int64).astype(dtype)
    c = rng.normal(0, 1e3, shape).astype(dtype)
    flat = c.reshape(-1)
    flat[rng.random(flat.size) < 0.1] = np.nan
    flat[:4] = [np.inf, -np.inf, 0.0, -0.0]
    return c


def _cloud(rng, h, w):
    xyz = rng.normal(0, 1e5, (h, w, 3))
    for k, bad in enumerate((np.nan, np.inf, -np.inf)):
        xyz[rng.random((h, w)) < 0.1, k] = bad
    return xyz


def _same_records(got, want):
    assert got.dtype == want.dtype
    assert got.tobytes() == want.tobytes()


@pytest.mark.parametrize("dtype", TYPES, ids=[np.dtype(t).name for t in TYPES])
def test_typed_records_equal_the_writer(engine, dtype):
    """every band count, with and without confidence; 37 x 131 points span several CTA tiles with ragged ends"""
    rng = np.random.default_rng(np.dtype(dtype).num)
    for h, w in ((13, 17), (37, 131)):
        xyz = _cloud(rng, h, w)
        for nb in (1, 3, 4):
            col = _colours(rng, dtype, (nb, h, w))
            for conf in (None, rng.random((h, w)).astype(np.float32)):
                _same_records(engine.ply_records_typed(xyz, col, conf), P.ply_records_literal(xyz, col, conf))
    assert len(engine.ply_records_typed(np.full((3, 5, 3), np.nan), _colours(rng, dtype, (3, 3, 5)))) == 0


def _records(xyz, colors, confidence):
    """the writer's records, vectorised, for colours of any type (ply_records_literal at a million points is slow)"""
    pts = xyz.reshape(-1, 3)
    keep = np.all(np.isfinite(pts), axis=1)
    nb = colors.shape[0]
    rec = np.empty(int(keep.sum()), P.ply_dtype(nb, confidence is not None, colors.dtype))
    for k, name in enumerate("xyz"):
        rec[name] = pts[keep, k]
    c = colors.reshape(nb, -1)[:, keep]
    for k, name in enumerate(("red", "green", "blue", "ir")[:max(nb, 3)]):
        rec[name] = c[0 if nb == 1 else k]
    if confidence is not None:
        rec["confidence"] = confidence.ravel()[keep]
    return rec


def test_typed_records_many_points(engine):
    """a million points: every record width at every byte alignment over hundreds of CTA tiles"""
    rng = np.random.default_rng(5)
    xyz = _cloud(rng, 1000, 1037)
    small = _cloud(rng, 37, 131)
    for dtype in (np.int16, np.uint32, np.float32, np.float64):
        for nb in (1, 4):
            col = _colours(rng, dtype, (nb, 1000, 1037))
            for conf in (None, rng.random((1000, 1037)).astype(np.float32)):
                sc = None if conf is None else conf[:37, :131]
                _same_records(_records(small, col[:, :37, :131], sc), P.ply_records_literal(small, col[:, :37, :131], sc))
                _same_records(engine.ply_records_typed(xyz, col, conf), _records(xyz, col, conf))


def test_typed_records_arguments(engine):
    from s2p_b200._lib import ERR_ARG, S2pbError
    for nb in (2, 5):
        with pytest.raises(S2pbError) as e:
            engine.ply_records_typed(np.zeros((2, 2, 3)), np.zeros((nb, 2, 2), np.uint16))
        assert e.value.code == ERR_ARG
    for bad in (np.int64, np.uint64, np.float16, np.bool_):
        with pytest.raises(TypeError):
            engine.ply_records_typed(np.zeros((2, 2, 3)), np.zeros((3, 2, 2), bad))
    import ctypes
    n = ctypes.c_int64(0)
    xyz, col, out = np.zeros(3), np.zeros(3, np.uint8), np.zeros(64, np.uint8)
    for t in (3, 7, 15, 21, -1):
        rc = engine._L.s2pb_ply_records_typed(engine._ctx, xyz.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), 1, col.ctypes.data,
                                              3, t, None, out.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)), ctypes.byref(n))
        assert rc == ERR_ARG, t


def _clr_source(seed, nb=3, side=700):
    """seeded 12-bit planes; at 700 x 700 the warp of the real pair's tile leaves the image (columns 414 to 935)"""
    return np.random.default_rng(seed).integers(0, 4096, (nb, side, side)).astype(np.uint16)


def _crop(src, H, w, h):
    """what common.homography_crop reads from a file holding src"""
    from s2p_b200.common import needed_roi
    x, y, rw, rh = needed_roi(H, w, h)
    rw, rh = rw + min(x, 0), rh + min(y, 0)
    x, y = max(x, 0), max(y, 0)
    rw, rh = min(rw, src.shape[2] - x), min(rh, src.shape[1] - y)
    Hc = np.asarray(H, np.float64) @ np.array([[1, 0, x], [0, 1, y], [0, 0, 1]], np.float64)
    return np.ascontiguousarray(src[:, y:y + rh, x:x + rw], np.float32), Hc


@pytest.mark.parametrize("nb,with_conf", [(1, False), (3, True), (4, False), (4, True)])
def test_disp_to_ply_clr_equals_the_composition(engine, nb, with_conf):
    a = _real()
    h, w = a["disp"].shape
    crop, hc = _crop(_clr_source(nb, nb), a["H1"], w, h)
    conf = a["conf"] if with_conf else None
    xyz, _ = engine.disp_to_xyz(a["disp"], a["mask_rect"], a["mask_orig"], a["H1"], a["H2"], a["rpc1"], a["rpc2"], a["img_bbx"],
                                40, True)
    engine.remove_isolated_3d_points(xyz, R, PW, N, 1)
    colours = np.stack([engine.homography(b, hc, w, h) for b in crop])
    assert np.isnan(colours).any() and np.isfinite(colours).any()
    want = P.ply_records_literal(xyz, colours, conf)
    got = engine.disp_to_ply_clr(a["disp"], a["mask_rect"], a["mask_orig"], a["H1"], a["H2"], a["rpc1"], a["rpc2"], a["img_bbx"],
                                 40, True, r=R, p=PW, n=N, clr=crop, hc=hc, confidence=conf)
    assert 1000 < len(want) and np.isnan(want["red"]).any()
    _same_records(got, want)


def test_disp_to_ply_clr_arguments(engine):
    from s2p_b200._lib import ERR_ARG, S2pbError
    a = _real()
    h, w = a["disp"].shape
    args = (a["disp"], a["mask_rect"], a["mask_orig"], a["H1"], a["H2"], a["rpc1"], a["rpc2"], a["img_bbx"], 40, True)
    crop, hc = _crop(_clr_source(0, 2), a["H1"], w, h)
    with pytest.raises(S2pbError) as e:
        engine.disp_to_ply_clr(*args, clr=crop, hc=hc)
    assert e.value.code == ERR_ARG
    crop, hc = _crop(_clr_source(0, 1), a["H1"], w, h)
    with pytest.raises(S2pbError) as e:                       # the crop lies wholly outside the warp's domain
        engine.disp_to_ply_clr(*args, clr=crop, hc=np.asarray(hc) @ np.array([[1, 0, 1e5], [0, 1, 0], [0, 0, 1]]))
    assert e.value.code == ERR_ARG


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.int16, np.float32], ids=["uint8", "uint16", "int16", "float32"])
def test_height_map_to_ply_clr_equals_the_composition(engine, dtype):
    heights, rpc, ox, oy, _ = _triplet()
    rng = np.random.default_rng(3)
    xyz = engine.height_map_to_xyz(heights, rpc, ox, oy, 31, False)
    engine.remove_isolated_3d_points(xyz, R, PW, N, 1)
    for nb in (1, 3, 4):
        colors = _colours(rng, dtype, (nb,) + heights.shape)
        want = P.ply_records_literal(xyz, colors)
        got = engine.height_map_to_ply_clr(heights, rpc, ox, oy, 31, False, r=R, p=PW, n=N, colors=colors)
        assert len(want) > 1000
        _same_records(got, want)


# ------------------------------------------------------------------ the step drop-ins on a tile directory

def _write_uint16(path, planes):
    """a multi-band uint16 TIFF, as the heights test writes its image"""
    import cv2
    a = planes[0] if len(planes) == 1 else np.moveaxis(planes, 0, 2)[..., ::-1]
    assert cv2.imwrite(path, np.ascontiguousarray(a))


def _pair_tile(tmp_path, a, ref_shape=None):
    from s2p_b200 import rasterio_compat
    d = tmp_path / "tile"
    (d / "pair_1").mkdir(parents=True)
    np.savetxt(str(d / "pair_1" / "H_ref.txt"), a["H1"])
    np.savetxt(str(d / "pair_1" / "H_sec.txt"), a["H2"])
    np.savetxt(str(tmp_path / "global_pointing_pair_1.txt"), np.eye(3))
    rasterio_compat.write_float_tiff(str(d / "pair_1" / "rectified_disp.tif"), a["disp"])
    ref = a["colors"][0] if ref_shape is None else np.zeros(ref_shape, np.float32)
    rasterio_compat.write_float_tiff(str(d / "pair_1" / "rectified_ref.tif"), ref)
    rasterio_compat.write_float_tiff(str(d / "pair_1" / "rectified_disp_confidence.tif"), a["conf"])
    rasterio_compat.write_mask_png(str(d / "pair_1" / "rectified_mask.png"), a["mask_rect"])
    rasterio_compat.write_mask_png(str(d / "mask.png"), a["mask_orig"])
    return d


def test_disparity_to_ply_clr_drop_in(engine, tmp_path, monkeypatch):
    from s2p_b200 import cloud, common, rasterio_compat, rasterization
    a = _real()
    h, w = a["disp"].shape
    d = _pair_tile(tmp_path, a)
    clr = str(tmp_path / "clr.tif")
    _write_uint16(clr, _clr_source(7))
    cfg = _cfg(tmp_path, rpcm=a["rpc1"])
    cfg["images"][1]["rpcm"] = a["rpc2"]
    cfg["images"][0]["clr"] = clr
    calls = []
    s2p = _stub_s2p(monkeypatch, cfg, disparity_to_ply=lambda tile: calls.append(tile))
    cloud.install()
    tile = {"dir": str(d), "coordinates": (0, 0, 1023, 1023)}
    s2p.disparity_to_ply(tile)
    assert not calls

    # the reference's path: the warp into a temporary TIFF, read back, then the writer
    warped = str(tmp_path / "colors.tif")
    common.image_apply_homography(warped, clr, a["H1"], w, h)
    colours = np.stack([rasterio_compat.read_window(warped, 0, 0, w, h, k + 1) for k in range(3)])
    xyz, _ = engine.disp_to_xyz(a["disp"], a["mask_rect"], a["mask_orig"], a["H1"], a["H2"], a["rpc1"], a["rpc2"],
                                (0, 1023, 0, 1023), 40, True)
    engine.remove_isolated_3d_points(xyz, R, PW, N, 1)
    rec = P.ply_records_literal(xyz, colours, a["conf"])
    with open(str(d / "cloud.ply"), "rb") as f:
        assert f.read() == P.ply_header(len(rec), COMMENTS, 3, True, "float") + rec.tobytes()
    back = rasterization.read_ply(str(d / "cloud.ply"))
    assert back.records.tobytes() == rec.tobytes()


def test_disparity_to_ply_clr_falls_through(engine, tmp_path, monkeypatch):
    """a clr image with 2 bands, and a rectified reference whose size is not the disparity's, go to the original step"""
    from s2p_b200 import cloud
    a = _real()
    h, w = a["disp"].shape
    clr2 = str(tmp_path / "clr2.tif")
    from PIL import Image
    Image.fromarray(np.zeros((50, 60, 2), np.uint8), "LA").save(clr2)
    for clr, ref_shape in ((clr2, None), (None, (h + 1, w))):
        sub = tmp_path / ("case%d" % (ref_shape is None))
        sub.mkdir()
        d = _pair_tile(sub, a, ref_shape)
        if clr is None:
            clr = str(sub / "clr.tif")
            _write_uint16(clr, _clr_source(1, 1, 600))
        cfg = _cfg(sub, rpcm=a["rpc1"])
        cfg["images"][1]["rpcm"] = a["rpc2"]
        cfg["images"][0]["clr"] = clr
        calls = []
        s2p = _stub_s2p(monkeypatch, cfg, disparity_to_ply=lambda tile: calls.append(tile))
        cloud.install()
        s2p.disparity_to_ply({"dir": str(d), "coordinates": (0, 0, 1023, 1023)})
        assert len(calls) == 1 and not (d / "cloud.ply").exists()


def _heights_tile(tmp_path, monkeypatch, clr, fused):
    from s2p_b200 import cloud, rasterio_compat
    heights, rpc, ox, oy, colors = _triplet()
    h, w = heights.shape
    x, y = int(ox), int(oy)
    d = tmp_path / "tile"
    d.mkdir(exist_ok=True)
    img = str(tmp_path / "img.tif")
    _write_uint16(img, np.zeros((3, y + h + 5, x + w + 5), np.uint16))

    def heights_fusion(tile):
        rasterio_compat.write_float_tiff(os.path.join(tile["dir"], "height_map.tif"), heights)
        fused.append(tile)

    cfg = _cfg(tmp_path, rpcm=rpc, img=img)
    cfg["out_crs"] = "epsg:32631"
    cfg["images"][0]["clr"] = clr
    calls = []
    s2p = _stub_s2p(monkeypatch, cfg, heights_to_ply=lambda tile: calls.append(tile), heights_fusion=heights_fusion)
    cloud.install()
    return s2p, d, (x, y, w, h), calls


def test_heights_to_ply_clr_drop_in_and_dsm(engine, tmp_path, monkeypatch):
    """the ushort cloud of a 12-bit clr image, then its DSM through the device with the plyflatten package absent"""
    from s2p_b200 import rasterization
    heights, rpc, ox, oy, colors = _triplet()
    h, w = heights.shape
    x, y = int(ox), int(oy)
    full = np.zeros((3, y + h + 5, x + w + 5), np.uint16)
    full[:, y:y + h, x:x + w] = colors
    clr = str(tmp_path / "clr.tif")
    _write_uint16(clr, full)
    fused = []
    s2p, d, coords, calls = _heights_tile(tmp_path, monkeypatch, clr, fused)
    s2p.heights_to_ply({"dir": str(d), "coordinates": coords})
    assert len(fused) == 1 and not calls

    xyz = engine.height_map_to_xyz(heights, rpc, x, y, 31, False)
    engine.remove_isolated_3d_points(xyz, R, PW, N, 1)
    rec = P.ply_records_literal(xyz, colors)
    ply = str(d / "cloud.ply")
    with open(ply, "rb") as f:
        assert f.read() == P.ply_header(len(rec), ["created by S2P", "projection: CRS epsg:32631"], 3, False, "ushort") + rec.tobytes()

    monkeypatch.setitem(sys.modules, "plyflatten", None)          # the device must read the ushort colours itself
    raster, profile = rasterization.plyflatten_from_plyfiles_list([ply], resolution=0.5, engine=engine)
    types = [D.F64] * 3 + [DT.U16] * 3
    pts = DT.columns(rec.view(np.uint8).reshape(len(rec), -1), list(rec.dtype.names), types)
    roi = D.roi_s2p(pts[:, 0], pts[:, 1], 0.5)
    want = D.plyflatten([pts], *roi[:2], 0.5, *roi[2:])
    assert raster.shape == want.shape == (roi[3], roi[2], 4)
    assert same(raster, want)
    assert np.isfinite(raster[..., 1:]).any()


def test_heights_to_ply_clr_falls_through(engine, tmp_path, monkeypatch):
    """a clr image that does not open, whose window has 2 bands, or of a type plyfile does not write goes to the original
    step, before heights_fusion"""
    from s2p_b200 import cloud
    read_stored = cloud.rasterio_compat.read_stored
    cases = [(str(tmp_path / "missing.tif"), None),
             (str(tmp_path / "img.tif"), lambda a: a[:2]),
             (str(tmp_path / "img.tif"), lambda a: a.astype(np.int64)),
             (str(tmp_path / "img.tif"), lambda a: a.astype(np.uint64)),
             (str(tmp_path / "img.tif"), lambda a: a.astype(np.float16))]
    for k, (clr, change) in enumerate(cases):
        if change is not None:
            monkeypatch.setattr(cloud.rasterio_compat, "read_stored",
                                lambda p, window=None, change=change: change(read_stored(p, window)))
        fused = []
        s2p, d, coords, calls = _heights_tile(tmp_path, monkeypatch, clr, fused)
        s2p.heights_to_ply({"dir": str(d), "coordinates": coords})
        assert len(calls) == 1 and not fused and not (d / "cloud.ply").exists(), k
        monkeypatch.setattr(cloud.rasterio_compat, "read_stored", read_stored)
