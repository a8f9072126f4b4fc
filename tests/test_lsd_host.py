"""The regularity weights of algo == 'mgm_multi_lsd' (s2p/block_matching.py:199-217).

The reference's pipeline `qauto IM | lsd - - | cut | pview segments W H | plambda - "255 x - 255 / 2 pow 0.1 fmax"`
writes 1 at every pixel whatever the image: qauto writes its 8-bit image into the pipe as NPY, lsd reads only PGM and
stops, pview draws no segment and the weight law maps 0 to 1.  These tests pin that with the tools built in place
(oracle/lsd.mk) where they are, and with their recorded output (tests/golden/lsd_weights.npz) everywhere, and check
that block_matching.lsd_weight_map gives the same weights without starting a process."""
import subprocess

import numpy as np
import pytest

import lsd_cases as C
from oracle import oracle as O
from oracle import lsd_oracle as L

REC = C.recorded()
NAMES = sorted(C.CASES)
have_ref = pytest.mark.skipif(not L.have_ref_lsd(), reason="oracle/_ref/{qauto,lsd,pview,plambda} not built")


def test_golden_covers_the_cases():
    assert sorted(REC) == NAMES
    for name in NAMES:
        assert REC[name]["digest"] == O.digest(C.CASES[name]()), "%s: the case's image changed since it was recorded" % name


@pytest.mark.parametrize("name", NAMES)
def test_recorded_pipeline_writes_ones(name):
    r, img = REC[name], C.CASES[name]()
    assert r["status"] == 0, "the shell reports plambda's status, and plambda succeeds"
    assert r["qauto_head"] == b"\x93NUMPY", "qauto writes NPY into a pipe"
    assert r["lsd_out"] == "" and "not a PGM file" in r["lsd_err"]
    assert r["weights"].dtype == np.float32 and r["weights"].shape == img.shape
    assert np.all(r["weights"] == 1.0)


def test_lsd_finds_segments_in_a_pgm():
    """The empty lsd output is the format, not the images: given qauto's output as a PGM file, lsd finds segments on
    every real image and every image with lines."""
    for name in ("crop1", "crop2", "rectified", "crop1_reflect_1024", "lines_0", "lines_45", "lines_90",
                 "lines_generic", "dense_parallel", "nan_border", "odd_size", "pair_ref", "pair_sec"):
        assert REC[name]["pgm_segments"] > 0, name


@have_ref
@pytest.mark.parametrize("name", NAMES)
def test_pipeline_against_golden(name):
    r, rec = L.ref_lsd_pipeline(C.CASES[name]()), REC[name]
    assert r["status"] == rec["status"]
    assert r["qauto_out"][:6] == rec["qauto_head"]
    assert r["lsd_out"] == rec["lsd_out"] and r["lsd_err"] == rec["lsd_err"]
    assert r["weights"].tobytes() == rec["weights"].tobytes()


@have_ref
def test_lsd_on_pgm_against_golden():
    assert len(L.ref_lsd_on_pgm(C.CASES["crop1"]()).splitlines()) == REC["crop1"]["pgm_segments"]


@pytest.mark.parametrize("name", NAMES)
def test_lsd_weight_map_matches_the_pipeline(name, tmp_path, monkeypatch):
    from s2p_b200 import block_matching as bm, rasterio_compat as rio

    def no_process(*a, **k):
        raise AssertionError("lsd_weight_map started a process")
    monkeypatch.setattr(subprocess, "Popen", no_process)
    im = str(tmp_path / "rectified_ref.tif")
    rio.write_float_tiff(im, C.CASES[name]())
    w = bm.lsd_weight_map(im)
    assert w.dtype == np.float32 and w.tobytes() == REC[name]["weights"].tobytes()


def test_lsd_weight_map_unreadable_image_raises(tmp_path):
    """The reference reads the image's size with rasterio before the pipeline, so a missing file raises there."""
    from s2p_b200 import block_matching as bm
    with pytest.raises(Exception):
        bm.lsd_weight_map(str(tmp_path / "missing.tif"))
