"""The tile's point cloud on the GPU (csrc/cloud_kernels.cuh, csrc/cloud.cu, s2p_b200/cloud.py), bit for bit:

- s2pb_stretch_8bit against np.nanpercentile + s2p's expression;
- s2pb_ply_records against the restated writer (tests/ply_oracle.py);
- s2pb_disp_to_ply / s2pb_height_map_to_ply against disp_to_xyz / height_map_to_xyz -> remove_isolated_3d_points -> the
  restated writer, with the kernels each call launches counted;
- the step drop-ins on a tile directory under a stub s2p package, against the file the composition writes.
"""
import os
import sys
import types
import warnings

import numpy as np
import pytest

import ply_oracle as P
from test_ply_host import CASES, CLOUDS

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(int(np.__version__.split(".")[0]) < 2, reason="the device reproduces NumPy >= 2's casting")]

SELECT, PACK = 8, 3          # launches of the radix select (4 digits x 2 kernels) and of count + scan + pack


def _numpy_stretch(img, p=1):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return P.stretch_8bit_reference(img, p)


@pytest.mark.parametrize("name", sorted(CASES))
def test_stretch_equals_numpy(engine, name):
    img = CASES[name]
    assert np.array_equal(engine.stretch_8bit(img), _numpy_stretch(img))


def test_stretch_percentages_and_arguments(engine):
    from s2p_b200._lib import ERR_ARG, S2pbError
    img = CASES["nan_b3"]
    for p in (0, 0.5, 10, 50):
        assert np.array_equal(engine.stretch_8bit(img, p), _numpy_stretch(img, p)), p
    for p in (-1, 100.5, float("nan")):
        with pytest.raises(S2pbError) as e:
            engine.stretch_8bit(img, p)
        assert e.value.code == ERR_ARG


@pytest.mark.parametrize("name", sorted(CLOUDS))
def test_records_equal_the_writer(engine, name):
    xyz, col, conf = CLOUDS[name]
    got = engine.ply_records(xyz, col, conf)
    want = P.ply_records_literal(xyz, col, conf)
    assert got.dtype == want.dtype and got.tobytes() == want.tobytes()


def test_records_many_points(engine):
    """several CTA tiles and every record length at every byte alignment"""
    rng = np.random.default_rng(5)
    xyz = rng.normal(0, 1, (1000, 1037, 3))
    xyz[rng.random((1000, 1037)) < 0.37, rng.integers(0, 3)] = np.nan
    for nb in (0, 1, 3, 4):
        col = rng.integers(0, 256, (nb, 1000, 1037)).astype(np.uint8) if nb else None
        for conf in (None, rng.random((1000, 1037)).astype(np.float32)):
            assert engine.ply_records(xyz, col, conf).tobytes() == P.ply_records(xyz, col, conf).tobytes()


def test_records_arguments(engine):
    from s2p_b200._lib import ERR_ARG, S2pbError
    for nb in (2, 5):
        with pytest.raises(S2pbError) as e:
            engine.ply_records(np.zeros((2, 2, 3)), np.zeros((nb, 2, 2), np.uint8))
        assert e.value.code == ERR_ARG
    assert len(engine.ply_records(np.zeros((0, 3)))) == 0


def _real():
    from s2p_b200.triangulation import rpc_from_geotiff_tag
    from util import load_real_pair
    z = load_real_pair()
    disp = z["rectified_disp"]
    rng = np.random.default_rng(1)
    return dict(rpc1=rpc_from_geotiff_tag(z["rpc1"]), rpc2=rpc_from_geotiff_tag(z["rpc2"]), H1=z["H1"], H2=z["H2"],
                disp=np.nan_to_num(disp), mask_rect=np.isfinite(disp).astype(np.float32), img_bbx=(0.0, 1023.0, 0.0, 1023.0),
                mask_orig=np.ones((1024, 1024), np.float32), colors=z["rectified_ref"][None],
                conf=rng.random(disp.shape).astype(np.float32))


R, PW, N = 5.0, 10, 50          # filter_xyz(r = 5 m, n = 50) at a GSD of 0.5 m: p = ceil(5 / 0.5)


@pytest.mark.parametrize("with_conf", [False, True])
def test_disp_to_ply_equals_the_composition(engine, with_conf):
    a = _real()
    conf = a["conf"] if with_conf else None
    k0 = engine.kernel_launches()
    xyz, _ = engine.disp_to_xyz(a["disp"], a["mask_rect"], a["mask_orig"], a["H1"], a["H2"], a["rpc1"], a["rpc2"], a["img_bbx"],
                                40, True)
    k1 = engine.kernel_launches()
    engine.remove_isolated_3d_points(xyz, R, PW, N, 1)
    k2 = engine.kernel_launches()
    want = P.ply_records(xyz, _numpy_stretch(a["colors"]), conf)
    got = engine.disp_to_ply(a["disp"], a["mask_rect"], a["mask_orig"], a["H1"], a["H2"], a["rpc1"], a["rpc2"], a["img_bbx"],
                             40, True, r=R, p=PW, n=N, colors=a["colors"], confidence=conf)
    k3 = engine.kernel_launches()
    assert 1000 < len(want) < xyz.shape[0] * xyz.shape[1]
    assert got.dtype == want.dtype and got.tobytes() == want.tobytes()
    assert k3 - k2 == (k1 - k0) + (k2 - k1) + SELECT + PACK


def test_disp_to_ply_without_filter(engine):
    a = _real()
    xyz, _ = engine.disp_to_xyz(a["disp"], a["mask_rect"], a["mask_orig"], a["H1"], a["H2"], a["rpc1"], a["rpc2"], a["img_bbx"],
                                40, True)
    k0 = engine.kernel_launches()
    got = engine.disp_to_ply(a["disp"], a["mask_rect"], a["mask_orig"], a["H1"], a["H2"], a["rpc1"], a["rpc2"], a["img_bbx"],
                             40, True, colors=a["colors"])
    assert engine.kernel_launches() - k0 == 2 + SELECT + PACK        # triangulation and projection, no filter
    assert got.tobytes() == P.ply_records(xyz, _numpy_stretch(a["colors"])).tobytes()


def _triplet():
    import localization_oracle as LO
    t = LO.triplet()
    rng = np.random.default_rng(2)
    return t["heights"], LO.triplet_rpc(), float(t["off"][0]), float(t["off"][1]), \
        rng.integers(100, 3000, (3,) + t["heights"].shape).astype(np.uint16)


def test_height_map_to_ply_equals_the_composition(engine):
    heights, rpc, ox, oy, colors = _triplet()
    k0 = engine.kernel_launches()
    xyz = engine.height_map_to_xyz(heights, rpc, ox, oy, 31, False)
    k1 = engine.kernel_launches()
    engine.remove_isolated_3d_points(xyz, R, PW, N, 1)
    k2 = engine.kernel_launches()
    want = P.ply_records(xyz, _numpy_stretch(colors))
    got = engine.height_map_to_ply(heights, rpc, ox, oy, 31, False, r=R, p=PW, n=N, colors=colors)
    k3 = engine.kernel_launches()
    assert len(want) > 1000
    assert got.dtype == want.dtype and got.tobytes() == want.tobytes()
    assert k3 - k2 == (k1 - k0) + (k2 - k1) + SELECT + PACK


# ------------------------------------------------------------------ the step drop-ins on a tile directory

def _stub_s2p(monkeypatch, cfg, **steps):
    s2p = types.ModuleType("s2p")
    config = types.ModuleType("s2p.config")
    config.cfg = cfg
    s2p.config = config
    for k, v in steps.items():
        setattr(s2p, k, v)
    monkeypatch.setitem(sys.modules, "s2p", s2p)
    monkeypatch.setitem(sys.modules, "s2p.config", config)
    return s2p


def _cfg(tmp_path, **images):
    return {"out_dir": str(tmp_path), "out_crs": "epsg:32740", "gsd": 0.5, "3d_filtering_r": R, "3d_filtering_n": N,
            "clean_intermediate": False, "images": [dict(images, clr=None), {"rpcm": None, "clr": None}]}


def test_disparity_to_ply_drop_in(engine, tmp_path, monkeypatch):
    from s2p_b200 import cloud, rasterio_compat, rasterization
    a = _real()
    d = tmp_path / "tile"
    (d / "pair_1").mkdir(parents=True)
    np.savetxt(str(d / "pair_1" / "H_ref.txt"), a["H1"])
    np.savetxt(str(d / "pair_1" / "H_sec.txt"), a["H2"])
    np.savetxt(str(tmp_path / "global_pointing_pair_1.txt"), np.eye(3))
    rasterio_compat.write_float_tiff(str(d / "pair_1" / "rectified_disp.tif"), a["disp"])
    rasterio_compat.write_float_tiff(str(d / "pair_1" / "rectified_ref.tif"), a["colors"][0])
    rasterio_compat.write_float_tiff(str(d / "pair_1" / "rectified_disp_confidence.tif"), a["conf"])
    rasterio_compat.write_mask_png(str(d / "pair_1" / "rectified_mask.png"), a["mask_rect"])
    rasterio_compat.write_mask_png(str(d / "mask.png"), a["mask_orig"])
    cfg = _cfg(tmp_path, rpcm=a["rpc1"])
    cfg["images"][1]["rpcm"] = a["rpc2"]
    calls = []
    s2p = _stub_s2p(monkeypatch, cfg, disparity_to_ply=lambda tile: calls.append(tile))
    cloud.install()
    tile = {"dir": str(d), "coordinates": (0, 0, 1023, 1023)}
    s2p.disparity_to_ply(tile)
    assert not calls

    xyz, _ = engine.disp_to_xyz(a["disp"], a["mask_rect"], a["mask_orig"], a["H1"], np.dot(a["H2"], np.linalg.inv(np.eye(3))),
                                a["rpc1"], a["rpc2"], (0, 1023, 0, 1023), 40, True)
    engine.remove_isolated_3d_points(xyz, R, PW, N, 1)
    rec = P.ply_records(xyz, _numpy_stretch(a["colors"]), a["conf"])
    comments = ["created by S2P", "projection: CRS epsg:32740"]
    with open(str(d / "cloud.ply"), "rb") as f:
        assert f.read() == P.ply_header(len(rec), comments, 1, True) + rec.tobytes()
    back = rasterization.read_ply(str(d / "cloud.ply"))
    assert back.comments == comments and back.records.tobytes() == rec.tobytes()

    # an output CRS the device does not serve, and a clr image, go to the original step
    for key, value in (("out_crs", "epsg:2154"), ("clr", "colors.tif")):
        if key == "clr":
            cfg["images"][0]["clr"] = value
        else:
            cfg[key] = value
        s2p.disparity_to_ply(tile)
    assert len(calls) == 2


def test_heights_to_ply_drop_in(engine, tmp_path, monkeypatch):
    import cv2
    from s2p_b200 import cloud, rasterio_compat
    heights, rpc, ox, oy, colors = _triplet()
    h, w = heights.shape
    x, y = int(ox), int(oy)
    d = tmp_path / "tile"
    d.mkdir()
    full = np.zeros((3, y + h + 5, x + w + 5), np.uint16)
    full[:, y:y + h, x:x + w] = colors
    img = str(tmp_path / "img.tif")
    assert cv2.imwrite(img, np.ascontiguousarray(np.moveaxis(full, 0, 2)[..., ::-1]))
    fused = []

    def heights_fusion(tile):
        rasterio_compat.write_float_tiff(os.path.join(tile["dir"], "height_map.tif"), heights)
        fused.append(tile)

    cfg = _cfg(tmp_path, rpcm=rpc, img=img)
    cfg["out_crs"] = "epsg:32631"
    s2p = _stub_s2p(monkeypatch, cfg, heights_to_ply=lambda tile: None, heights_fusion=heights_fusion)
    cloud.install()
    s2p.heights_to_ply({"dir": str(d), "coordinates": (x, y, w, h)})
    assert len(fused) == 1

    xyz = engine.height_map_to_xyz(heights, rpc, x, y, 31, False)
    engine.remove_isolated_3d_points(xyz, R, PW, N, 1)
    rec = P.ply_records(xyz, _numpy_stretch(colors))
    with open(str(d / "cloud.ply"), "rb") as f:
        assert f.read() == P.ply_header(len(rec), ["created by S2P", "projection: CRS epsg:32631"], 3) + rec.tobytes()
