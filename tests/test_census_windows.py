"""Every census window s2p can ask for (census_ncc_win 2 to 11) on the CPU: the oracle of tests/census_window_oracle.py against the
reference binaries, bit for bit, and the rule that decides which windows the device matcher serves."""
import os

import numpy as np
import pytest

import census_window_oracle as CW
from s2p_b200.synth import make_pair
from util import GOLD, nmismatch, same


def _needs_ref(oracle, binary="mgm"):
    if not os.access(os.path.join(oracle.REF_DIR, binary), os.X_OK):
        pytest.skip("oracle/_ref/%s is not built (the reference's sources are absent)" % binary)


def _check(ours, ref):
    d, c, dr = ours
    assert same(d, ref["disp"]), "%d px differ" % nmismatch(d, ref["disp"])
    assert same(c, ref["conf"]) and same(dr, ref["dispR"])


@pytest.mark.parametrize("nanb", [0.0, 0.05])
@pytest.mark.parametrize("win", [2, 4, 6, 8, 9, 10, 11])
def test_mgm_oracle_matches_reference(oracle, win, nanb):
    """`mgm` with CENSUS_NCC_WIN = win, on a clean pair and on one with no-data strips (the DCT round trip does work)"""
    _needs_ref(oracle)
    ref, sec, _ = make_pair(40, 88, -10, 9, seed=win, nan_border=nanb)
    P = oracle.mgm_params(census_win=win)
    _check(CW.mgm(ref, sec, -10, 9, P), oracle.run_ref(ref, sec, -10, 9, P, threads=1))


@pytest.mark.parametrize("win", [9, 11])
def test_mgm_multi_oracle_matches_reference(oracle, win):
    _needs_ref(oracle, "mgm_multi")
    ref, sec, _ = make_pair(64, 120, -10, 9, seed=win, nan_border=0.03)
    P = oracle.mgm_multi_params(census_win=win)
    _check(CW.mgm_multi(ref, sec, -10, 9, P), oracle.run_ref(ref, sec, -10, 9, P, threads=1))


@pytest.mark.parametrize("win", [4, 9])
def test_ncc_window_matches_reference(oracle, win):
    """NCC's n is the number of taps, (2 (win / 2) + 1)^2, also for even windows"""
    _needs_ref(oracle)
    ref, sec, _ = make_pair(40, 88, -10, 9, seed=30 + win, nan_border=0.03)
    P = oracle.mgm_params(census_win=win, cost=oracle.COSTS.index("ncc"))
    _check(CW.mgm(ref, sec, -10, 9, P), oracle.run_ref(ref, sec, -10, 9, P, threads=1))


@pytest.mark.parametrize("win", [4, 9])
def test_mindiff_window_matches_reference(oracle, win):
    """MINDIFF takes win itself, with the asymmetric window of the even ones"""
    _needs_ref(oracle)
    ref, sec, _ = make_pair(40, 88, -10, 9, seed=40 + win, nan_border=0.03)
    P = oracle.mgm_params(census_win=win, mindiff=1.0)
    _check(CW.mgm(ref, sec, -10, 9, P), oracle.run_ref(ref, sec, -10, 9, P, threads=1))


def test_oracle_reproduces_golden(oracle):
    """tests/golden/census_windows.npz (make_golden_census_windows.py: the reference binary at win 4, 9 and 11)"""
    g = np.load(os.path.join(GOLD, "census_windows.npz"))
    for win in g["wins"]:
        d, c, dr = CW.mgm(g["ref"], g["sec"], int(g["dmin"]), int(g["dmax"]), oracle.mgm_params(census_win=int(win)))
        assert same(d, g["disp_%d" % win]) and same(c, g["conf_%d" % win]) and same(dr, g["dispR_%d" % win]), win


def test_code_bits_and_channels():
    """census_tools.cc:76-99: side 2 (win / 2) + 1, side^2 - 1 bits, ceil(bits / 32) channels"""
    bits = {w: CW.census_bits(w) for w in range(2, 12)}
    assert bits == {2: 8, 3: 8, 4: 24, 5: 24, 6: 48, 7: 48, 8: 80, 9: 80, 10: 120, 11: 120}
    ref, _, _ = make_pair(9, 13, -2, 2, seed=1)
    assert CW.census_codes(ref, 11).shape == (15, 9, 13)


# ------------------------------------------------------------------ which windows the device serves, and the drop-ins

def test_census_window_served():
    from s2p_b200.engine import census_window_served
    assert [w for w in range(-1, 20) if census_window_served(w)] == list(range(2, 12))


class _FakeEngine:
    def __init__(self):
        self.wins = []

    def mgm(self, a, b, dmin, dmax, params, want_mask=True, weights=None):
        self.wins.append(params.census_win)
        return dict(disp=np.zeros_like(a), conf=np.zeros_like(a), mask=np.zeros(a.shape, np.uint8))


@pytest.mark.parametrize("algo", ["mgm", "mgm_multi"])
def test_compute_disparity_map_routes_by_window(monkeypatch, algo):
    """windows 2 to 11 go to the engine, 1 and 12 to s2p's own compute_disparity_map"""
    from s2p_b200 import block_matching as bm
    from s2p_b200.config import cfg
    eng, fell = _FakeEngine(), []
    monkeypatch.setattr(bm, "get_engine", lambda: eng)
    monkeypatch.setattr(bm, "_original_compute_disparity_map", lambda: (lambda *a: fell.append(cfg["census_ncc_win"])))
    monkeypatch.setattr(bm.rio, "image_size", lambda path: (16, 8))
    monkeypatch.setattr(bm.rio, "read_band", lambda path: np.ones((8, 16), np.float32))
    monkeypatch.setattr(bm.rio, "write_float_tiff", lambda path, a: None)
    monkeypatch.setattr(bm.rio, "write_mask_png", lambda path, a: None)
    for win in (2, 9, 11, 1, 12):
        monkeypatch.setitem(cfg, "census_ncc_win", win)
        assert bm.compute_disparity_map("a.tif", "b.tif", "d.tif", "m.png", algo, -4, 4) is None
    assert eng.wins == [2, 9, 11] and fell == [1, 12]


def test_compute_disparity_map_unserved_window_without_s2p(monkeypatch):
    from s2p_b200 import block_matching as bm
    from s2p_b200.config import cfg
    monkeypatch.setattr(bm, "_original_compute_disparity_map", lambda: None)
    monkeypatch.setitem(cfg, "census_ncc_win", 13)
    with pytest.raises(NotImplementedError, match="census_ncc_win 13"):
        bm.compute_disparity_map("a.tif", "b.tif", "d.tif", "m.png", "mgm", -4, 4)


def _cfg(nimages, algo, win):
    return {"images": [{"img": "im%d.tif" % i, "rpcm": None, "clr": None} for i in range(nimages)], "matching_algorithm": algo,
            "census_ncc_win": win, "out_crs": "epsg:32631"}


@pytest.mark.parametrize("reason", ["fall_through_reason", "pair_heights_fall_through_reason"])
def test_fused_reasons_name_unserved_windows(reason):
    from s2p_b200 import fused
    f, n = getattr(fused, reason), 2 if reason == "fall_through_reason" else 3
    for win in (1, 12):
        assert "census_ncc_win %d is not served" % win in (f(_cfg(n, "mgm", win)) or "")
        assert "census_ncc_win %d is not served" % win in (f(_cfg(n, "mgm_multi_lsd", win)) or "")
    for win in (2, 9, 11):
        assert "census_ncc_win" not in (f(_cfg(n, "mgm", win)) or "")
    assert "census_ncc_win" not in (f(_cfg(n, "sgbm", 12)) or "")      # sgbm has no census window
