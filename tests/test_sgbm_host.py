"""Host-side logic of the `sgbm` matcher (no GPU): the routing of compute_disparity_map, the ctypes mirror of
s2pb_sgbm_params, the qauto thresholds against what the reference binary prints, its determinism with zeroed allocations,
and the recorded digests the GPU tests fall back on."""
import json
import os
import re

import numpy as np
import pytest

import sgbm_oracle as SO
from s2p_b200 import _lib, block_matching as bm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_params_mirror_header():
    hdr = open(os.path.join(ROOT, "include", "s2pb200.h")).read()
    body = re.search(r"typedef struct s2pb_sgbm_params \{(.*?)\} s2pb_sgbm_params;", hdr, re.S).group(1)
    fields = re.findall(r"int32_t\s+(\w+);", body)
    assert fields == [f for f, _ in _lib.SgbmParams._fields_]
    assert "s2pb_sgbm" in _lib.exported_symbols() and "s2pb_sgbm_default_params" in _lib.exported_symbols()
    for name in ("s2pb_sgbm", "s2pb_sgbm_default_params"):
        assert re.search(r"\b%s\(" % name, hdr)


def test_s2p_arguments():
    assert bm.SGBM_ARGS == dict(win=3, P1=8, P2=32, lr_diff=1)


def test_sgbm_with_bounds_goes_to_the_engine(monkeypatch, tmp_path):
    calls = []

    class FakeEngine:
        def sgbm_params(self, **kw):
            return kw

        def sgbm(self, a, b, dmin, dmax, params, want_mask):
            calls.append((a.shape, dmin, dmax, params, want_mask))
            return dict(disp=np.zeros(a.shape, np.float32), mask=np.ones(a.shape, np.uint8))

    written = []
    monkeypatch.setattr(bm, "get_engine", lambda: FakeEngine())
    monkeypatch.setattr(bm.rio, "image_size", lambda p: (50, 20))
    monkeypatch.setattr(bm.rio, "read_band", lambda p: np.zeros((20, 50), np.float32))
    monkeypatch.setattr(bm.rio, "write_float_tiff", lambda p, a: written.append(p))
    monkeypatch.setattr(bm.rio, "write_mask_png", lambda p, a: written.append(p))
    bm.compute_disparity_map("a.tif", "b.tif", "d.tif", "m.png", "sgbm", -7.5, 3.2)
    assert calls == [((20, 50), -8, 4, bm.SGBM_ARGS, True)]
    assert written == ["d.tif", "m.png"]                 # no _confidence.tif, as the reference
    # a range wider than the image is shrunk around its centre first (s2p/block_matching.py:62-68)
    bm.compute_disparity_map("a.tif", "b.tif", "d.tif", "m.png", "sgbm", -100, 100)
    assert calls[-1][1:3] == (-25, 25)
    with pytest.raises(bm.MaxDisparityRangeError):
        bm.compute_disparity_map("a.tif", "b.tif", "d.tif", "m.png", "sgbm", -10, 10, max_disp_range=5)


def test_sgbm_with_a_none_bound_falls_through(monkeypatch):
    monkeypatch.setattr(bm, "get_engine", lambda: pytest.fail("the engine must not run without both bounds"))
    monkeypatch.setattr(bm, "_original_compute_disparity_map", lambda: None)
    for lo, hi in ((None, 5), (-5, None), (None, None)):
        with pytest.raises(NotImplementedError):
            bm.compute_disparity_map("a", "b", "c", "d", "sgbm", lo, hi)
    seen = []
    monkeypatch.setattr(bm, "_original_compute_disparity_map", lambda: (lambda *a: seen.append(a)))
    bm.compute_disparity_map("a", "b", "c", "d", "sgbm", None, 5)
    assert seen and seen[0][4] == "sgbm" and seen[0][5] is None


def test_qauto_restatement_matches_the_binary():
    if not SO.have_ref():
        pytest.skip("oracle/_ref/sgbm not built")
    for name in ("base_96x160", "nan_border", "constant", "real_inputs"):
        a, b, dmin, dmax, win, P1, P2, lr = SO.case(name)
        r = SO.run_ref(a, b, dmin, dmax, win, P1, P2, lr)
        lo, hi = SO.qauto_thresholds(a)
        assert r["rminmax"] == (float("%g" % lo), float("%g" % hi)), name


def test_recorded_thresholds_match_the_restatement():
    db = json.load(open(SO.RECORDED))
    assert sorted(db) == sorted(SO.CASES)
    for name, rec in db.items():
        lo, hi = SO.qauto_thresholds(SO.case(name)[0])
        assert rec["rminmax"] == [float("%g" % lo), float("%g" % hi)], name


def test_oracle_is_deterministic_with_zeroed_allocations():
    if not SO.have_ref():
        pytest.skip("oracle/_ref/sgbm not built")
    a, b, dmin, dmax, win, P1, P2, lr = SO.case("odd_37x61")
    one = SO.run_ref(a, b, dmin, dmax, win, P1, P2, lr)["disp"]
    two = SO.run_ref(a, b, dmin, dmax, win, P1, P2, lr)["disp"]
    assert np.array_equal(np.isnan(one), np.isnan(two)) and np.array_equal(one[np.isfinite(one)], two[np.isfinite(two)])


def test_recorded_digests_match_the_live_oracle():
    if not (SO.have_ref() and SO.O.have_ref_mask()):
        pytest.skip("oracle/_ref not built")
    db = json.load(open(SO.RECORDED))
    for name in ("base_96x160", "constant", "speckle"):
        assert SO.ref_digests(name) == db[name], name
