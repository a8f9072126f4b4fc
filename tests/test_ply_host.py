"""CPU checks of the point-cloud step's restatements (tests/ply_oracle.py) and of the PLY writer (s2p_b200/cloud.py).

- The stretch as the device forms it (two order statistics per percentile and numpy's _lerp) equals
  np.nanpercentile + s2p's expression bit for bit.
- The vectorised records equal the reference's tuple path byte for byte.
- write_ply's header equals the header of s2p's own writer output (tests/golden/cloud_ply_header.txt).
"""
import os
import warnings

import numpy as np
import pytest

import ply_oracle as P
from util import GOLD

pytestmark = pytest.mark.skipif(int(np.__version__.split(".")[0]) < 2, reason="the device reproduces NumPy >= 2's casting")


def stretch_cases():
    """name -> image (bands, h, w): seeded, with NaN, infinities, ties, constant and all-NaN images, uint16 and float32"""
    rng = np.random.default_rng(7)
    out = {}
    for n in (1, 2, 3, 7, 99, 100, 101, 1000, 4099, 10 ** 6):
        out["f32_%d" % n] = rng.normal(300.0, 80.0, (1, 1, n)).astype(np.float32)
    for nb in (1, 3, 4):
        out["u16_b%d" % nb] = rng.integers(0, 65536, (nb, 61, 47)).astype(np.uint16)
        out["u8_b%d" % nb] = rng.integers(0, 256, (nb, 33, 29)).astype(np.uint8)
        a = rng.normal(0.0, 1e3, (nb, 64, 80)).astype(np.float32)
        a[rng.random(a.shape) < 0.3] = np.nan
        out["nan_b%d" % nb] = a
        out["ties_b%d" % nb] = rng.integers(0, 5, (nb, 50, 50)).astype(np.float32)
    b = rng.normal(0.0, 1.0, (3, 40, 40)).astype(np.float32)
    b[rng.random(b.shape) < 0.05] = np.inf
    b[rng.random(b.shape) < 0.05] = -np.inf
    b[rng.random(b.shape) < 0.05] = np.nan
    out["inf"] = b
    out["mostly_inf"] = np.where(rng.random((1, 30, 30)) < 0.995, np.inf, 1.0).astype(np.float32)
    out["constant"] = np.full((3, 20, 20), 17.25, np.float32)
    out["all_nan"] = np.full((1, 9, 9), np.nan, np.float32)
    one = np.full((1, 10, 10), np.nan, np.float32)
    one[0, 3, 4] = 5.0
    out["one_value"] = one
    out["big_range"] = np.array([[[-3e38, 3e38, 0.0, 1.0]]], np.float32)
    out["u16_full_tile"] = rng.integers(200, 1400, (1, 1024, 1024)).astype(np.uint16)
    return out


CASES = stretch_cases()


@pytest.mark.parametrize("name", sorted(CASES))
def test_stretch_restatement_equals_numpy(name):
    img = CASES[name]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        want = P.stretch_8bit_reference(img)
        a, b = np.nanpercentile(img, (1, 99))
    ra, rb = P.percentiles(img)
    assert (ra == a or (np.isnan(ra) and np.isnan(a))) and (rb == b or (np.isnan(rb) and np.isnan(b)))
    assert np.array_equal(P.stretch_8bit(img), want)


def test_stretch_other_percentages():
    rng = np.random.default_rng(3)
    img = rng.normal(0, 1, (3, 31, 17)).astype(np.float32)
    for p in (0, 0.5, 2, 10, 25, 50):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            want = P.stretch_8bit_reference(img, p)
        assert np.array_equal(P.stretch_8bit(img, p), want), p


def clouds():
    """name -> (xyz (h, w, 3) float64, colours (nbands, h, w) uint8 or None, confidence (h, w) float32 or None)"""
    rng = np.random.default_rng(11)
    out = {}
    for bad in ("nan", "inf", "-inf"):
        for k in range(3):
            xyz = rng.normal(0, 1e5, (13, 17, 3))
            sel = rng.random((13, 17)) < 0.2
            xyz[sel, k] = float(bad)
            for nb in (0, 1, 3, 4):
                col = rng.integers(0, 256, (nb, 13, 17)).astype(np.uint8) if nb else None
                out["%s%d_b%d" % (bad, k, nb)] = (xyz, col, None)
                out["%s%d_b%d_conf" % (bad, k, nb)] = (xyz, col, rng.random((13, 17)).astype(np.float32))
    empty = np.full((4, 5, 3), np.nan)
    out["no_point"] = (empty, rng.integers(0, 256, (3, 4, 5)).astype(np.uint8), None)
    out["no_point_conf"] = (empty, rng.integers(0, 256, (1, 4, 5)).astype(np.uint8), np.ones((4, 5), np.float32))
    return out


CLOUDS = clouds()


@pytest.mark.parametrize("name", sorted(CLOUDS))
def test_records_equal_the_tuple_path(name):
    xyz, col, conf = CLOUDS[name]
    got = P.ply_records(xyz, col, conf)
    want = P.ply_records_literal(xyz, col, conf)
    assert got.dtype == want.dtype
    assert got.tobytes() == want.tobytes()


def test_refused_band_counts_raise_alike():
    xyz = np.zeros((2, 2, 3))
    for nb in (2, 5):
        col = np.zeros((nb, 2, 2), np.uint8)
        with pytest.raises(Exception) as e1:
            P.ply_records_literal(xyz, col)
        with pytest.raises(Exception) as e2:
            P.ply_records(xyz, col)
        assert type(e1.value) is type(e2.value)


def test_engine_dtype_is_the_writer_dtype():
    from s2p_b200.engine import Engine
    for nb in (0, 1, 3, 4):
        for conf in (False, True):
            assert Engine.ply_dtype(nb, conf) == P.ply_dtype(nb, conf)
            assert Engine.ply_dtype(nb, conf).itemsize == 24 + (4 if nb == 4 else 3 if nb else 0) + 4 * conf


def test_header_equals_the_reference_writer_output():
    from s2p_b200 import cloud
    with open(os.path.join(GOLD, "cloud_ply_header.txt"), "rb") as f:
        want = f.read()
    records = np.zeros(120764, P.ply_dtype(3, False))
    got = cloud.ply_header(records, ["created by S2P", "projection: CRS epsg:32740"])
    assert got == want
    assert got == P.ply_header(120764, ["created by S2P", "projection: CRS epsg:32740"])


@pytest.mark.parametrize("nb,conf", [(0, False), (1, True), (3, True), (4, False), (4, True)])
def test_write_ply_reads_back(tmp_path, nb, conf):
    from s2p_b200 import cloud, rasterization
    xyz, col, c = CLOUDS["nan1_b%d%s" % (nb, "_conf" if conf else "")]
    rec = P.ply_records(xyz, col, c)
    path = str(tmp_path / "cloud.ply")
    cloud.write_ply(path, rec, ["created by S2P", "projection: CRS epsg:32631"])
    with open(path, "rb") as f:
        data = f.read()
    hdr = P.ply_header(len(rec), ["created by S2P", "projection: CRS epsg:32631"], nb, conf)
    assert data == hdr + rec.tobytes()
    back = rasterization.read_ply(path)
    assert back.comments == ["created by S2P", "projection: CRS epsg:32631"]
    assert back.records.tobytes() == rec.tobytes()


def test_install_tolerates_a_package_without_the_steps(monkeypatch):
    import sys
    import types
    from s2p_b200 import cloud
    stub = types.ModuleType("s2p")
    monkeypatch.setitem(sys.modules, "s2p", stub)
    cloud.install()
    assert not hasattr(stub, "disparity_to_ply")
    stub.disparity_to_ply = lambda tile: "orig"
    stub.heights_to_ply = lambda tile: "orig_h"
    cloud.install()
    cloud.install()
    assert stub.disparity_to_ply is cloud.disparity_to_ply and stub.heights_to_ply is cloud.heights_to_ply
    assert stub._s2pb_original_disparity_to_ply(None) == "orig" and stub._s2pb_original_heights_to_ply(None) == "orig_h"
