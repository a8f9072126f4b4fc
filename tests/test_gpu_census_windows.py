"""Every census window s2p can ask for (census_ncc_win 2 to 11) on the device, bit for bit against the oracle of
tests/census_window_oracle.py (pinned to the reference binaries by tests/test_census_windows.py) or the reference's recorded
outputs."""
import os

import numpy as np
import pytest

import census_window_oracle as CW
from s2p_b200 import _lib
from s2p_b200.engine import Engine, S2pbError, default_params, workspace_bytes
from s2p_b200.synth import make_pair
from util import GOLD, nmismatch, same

pytestmark = pytest.mark.gpu


def _orc(oracle, p):
    """the oracle's parameters of an engine parameter block"""
    return oracle.mgm_params(**{f: getattr(p, f) for f, _ in oracle.OrcParams._fields_ if f != "dct_shift"})


def _check(out, ref, oracle, im1, im2):
    d, c, dr = ref
    assert same(out["disp"], d), "%d px differ" % nmismatch(out["disp"], d)
    assert same(out["conf"], c) and same(out["disp_right"], dr)
    if out.get("mask") is not None:
        assert np.array_equal(out["mask"], oracle.port.rejection_mask(d, im1, im2))


@pytest.mark.parametrize("nanb", [0.0, 0.05])
@pytest.mark.parametrize("win", list(range(2, 12)))
def test_mgm_every_window(engine, oracle, win, nanb):
    ref, sec, _ = make_pair(50, 120, -9, 10, seed=win, nan_border=nanb)
    p = default_params("mgm", census_win=win)
    out = engine.mgm(ref, sec, -9, 10, p, want_right=True)
    _check(out, CW.mgm(ref, sec, -9, 10, _orc(oracle, p)), oracle, ref, sec)


@pytest.mark.parametrize("win", [2, 4, 7, 8, 9, 11])
def test_mgm_more_than_512_labels(engine, oracle, win):
    """the chunk-skipping cost, aggregation and WTA kernels"""
    ref, sec, _ = make_pair(24, 400, -300, 299, seed=win, nan_border=0.03)
    p = default_params("mgm", census_win=win)
    out = engine.mgm(ref, sec, -300, 299, p, want_right=True)
    _check(out, CW.mgm(ref, sec, -300, 299, _orc(oracle, p)), oracle, ref, sec)


@pytest.mark.parametrize("win", [9, 11])
@pytest.mark.parametrize("algo", ["mgm_multi", "mgm_multi_lsd"])
def test_mgm_multi(engine, oracle, algo, win):
    """mgm_multi with its half-pixel pass; mgm_multi_lsd's weights select the float-cost flavour"""
    ref, sec, _ = make_pair(96, 150, -12, 12, seed=win, nan_border=0.03)
    p = default_params(algo, census_win=win)
    weights = None
    if algo == "mgm_multi_lsd":
        rng = np.random.default_rng(win)
        weights = tuple(rng.uniform(0.25, 1.0, ref.shape).astype(np.float32) for _ in range(2))
    out = engine.mgm(ref, sec, -12, 12, p, want_right=True, weights=weights)
    wl, wr = weights if weights else (None, None)
    _check(out, CW.mgm_multi(ref, sec, -12, 12, _orc(oracle, p), wl, wr), oracle, ref, sec)


@pytest.mark.parametrize("win", [9, 11])
def test_costvolume(engine, oracle, win):
    h, w, dmin, dmax = 30, 90, -14, 13
    ref, sec, _ = make_pair(h, w, dmin, dmax, seed=win)
    lo, hi = np.full((h, w), dmin, np.int32), np.full((h, w), dmax, np.int32)
    lo[4:9, 10:40] = dmin + 3
    D = dmax - dmin + 1
    C = engine.costvolume(ref, sec, lo, hi, dmin, D, win=win)
    assert same(C, CW.costvolume(ref, sec, lo, hi, dmin, D, win))


def test_folded_equals_resident_at_11(oracle):
    h, w, dmin, dmax = 64, 160, -20, 19
    ref, sec, _ = make_pair(h, w, dmin, dmax, seed=11)
    p = default_params("mgm", census_win=11)
    outs = []
    with Engine(0) as eng:
        for folded in (False, True):
            eng.set_workspace_limit(workspace_bytes(w, h, dmax - dmin + 1, folded=True) if folded else 0)
            before = eng.folded_calls()
            outs.append(eng.mgm(ref, sec, dmin, dmax, p, want_right=True))
            assert (eng.folded_calls() > before) == folded
    for k in ("disp", "conf", "mask", "disp_right"):
        assert same(outs[0][k], outs[1][k]), k
    _check(outs[1], CW.mgm(ref, sec, dmin, dmax, _orc(oracle, p)), oracle, ref, sec)


@pytest.mark.parametrize("win", [8, 11])
def test_window_adds_no_workspace(oracle, win):
    """a tile whose workspace limit is exactly s2pb_workspace_bytes runs resident: the second code words need no bytes of their own"""
    h, w, dmin, dmax = 64, 160, -20, 19
    ref, sec, _ = make_pair(h, w, dmin, dmax, seed=win)
    p = default_params("mgm", census_win=win)
    with Engine(0) as eng:
        eng.set_workspace_limit(workspace_bytes(w, h, dmax - dmin + 1))
        out = eng.mgm(ref, sec, dmin, dmax, p, want_right=True)
        assert eng.folded_calls() == 0
    _check(out, CW.mgm(ref, sec, dmin, dmax, _orc(oracle, p)), oracle, ref, sec)


def test_wta_prune_off_equals_default_at_9():
    ref, sec, _ = make_pair(70, 140, -16, 15, seed=9, nan_border=0.02)
    p = default_params("mgm", census_win=9)
    old = os.environ.get("S2PB_WTA_PRUNE")
    outs = []
    try:
        for v in (None, "0"):
            if v is None:
                os.environ.pop("S2PB_WTA_PRUNE", None)
            else:
                os.environ["S2PB_WTA_PRUNE"] = v
            with Engine(0) as eng:
                outs.append(eng.mgm(ref, sec, -16, 15, p, want_right=True))
    finally:
        if old is None:
            os.environ.pop("S2PB_WTA_PRUNE", None)
        else:
            os.environ["S2PB_WTA_PRUNE"] = old
    for k in ("disp", "conf", "mask", "disp_right"):
        assert same(outs[0][k], outs[1][k]), k


def test_golden_reference_outputs(engine):
    """tests/golden/census_windows.npz: the reference binary at win 4, 9 and 11"""
    g = np.load(os.path.join(GOLD, "census_windows.npz"))
    for win in g["wins"]:
        out = engine.mgm(g["ref"], g["sec"], int(g["dmin"]), int(g["dmax"]), default_params("mgm", census_win=int(win)),
                         want_right=True)
        assert same(out["disp"], g["disp_%d" % win]), "win %d: %d px differ" % (win, nmismatch(out["disp"], g["disp_%d" % win]))
        assert same(out["conf"], g["conf_%d" % win]) and same(out["disp_right"], g["dispR_%d" % win])


def test_refused_windows(engine):
    ref, sec, _ = make_pair(20, 40, -4, 4, seed=0)
    for win, code in ((12, _lib.ERR_UNSUPPORTED), (25, _lib.ERR_UNSUPPORTED), (1, _lib.ERR_ARG), (0, _lib.ERR_ARG)):
        with pytest.raises(S2pbError) as e:
            engine.mgm(ref, sec, -4, 4, default_params("mgm", census_win=win))
        assert e.value.code == code, win
        lo, hi = np.full(ref.shape, -4, np.int32), np.full(ref.shape, 4, np.int32)
        with pytest.raises(S2pbError) as e:
            engine.costvolume(ref, sec, lo, hi, -4, 9, win=win)
        assert e.value.code == code, win
    with pytest.raises(S2pbError) as e:          # s2pb_census keeps its 3 / 5 / 7 contract
        engine.census(ref, 9)
    assert e.value.code == _lib.ERR_ARG
