"""compute_disparity_map(algo='mgm_multi_lsd') with the weight maps the reference's pipeline writes
(tests/test_lsd_host.py): no process, no tool on PATH, and the files of the matcher fed the recorded weights."""
import subprocess

import numpy as np
import pytest

import lsd_cases as C
from util import same

pytestmark = pytest.mark.gpu


def test_dropin_mgm_multi_lsd_starts_no_process(engine, tmp_path, monkeypatch):
    from s2p_b200 import block_matching as bm, rasterio_compat as rio
    dmin, dmax = -14, 11
    ref, sec = C.CASES["pair_ref"](), C.CASES["pair_sec"]()
    im1, im2 = str(tmp_path / "rectified_ref.tif"), str(tmp_path / "rectified_sec.tif")
    disp, mask = str(tmp_path / "rectified_disp.tif"), str(tmp_path / "rectified_mask.png")
    rio.write_float_tiff(im1, ref)
    rio.write_float_tiff(im2, sec)
    empty = tmp_path / "bin"
    empty.mkdir()
    monkeypatch.setenv("PATH", str(empty))

    def no_process(*a, **k):
        raise AssertionError("compute_disparity_map started a process")
    monkeypatch.setattr(subprocess, "Popen", no_process)
    assert bm.compute_disparity_map(im1, im2, disp, mask, "mgm_multi_lsd", dmin, dmax) is None
    monkeypatch.undo()

    rec = C.recorded()
    weights = (rec["pair_ref"]["weights"], rec["pair_sec"]["weights"])
    out = engine.mgm(rio.read_band(im1), rio.read_band(im2), dmin, dmax, bm.matcher_params("mgm_multi_lsd", 600),
                     want_mask=True, weights=weights)
    assert same(rio.read_band(disp), out["disp"])
    assert same(rio.read_band(disp + ".confidence.tif"), out["conf"])
    assert np.array_equal(rio.read_band(mask), out["mask"])
