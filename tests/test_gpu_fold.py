"""The folded workspace layout (DESIGN.md section 3.6): every test caps the workspace just below the resident size of its tile, so
that the matcher runs folded, checks that it did (Engine.folded_calls), and holds the results to the oracle or to the resident
layout on the same device, bit for bit."""
import subprocess
from contextlib import contextmanager

import numpy as np
import pytest

from s2p_b200 import _lib
from s2p_b200.engine import Engine, S2pbError, default_params, workspace_bytes
from s2p_b200.synth import make_pair
from util import nmismatch, same

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


def below_resident(w, h, nlabels, ndir=8, cost_bytes=1):
    """a limit one byte below the resident workspace of a single-scale tile whose hull is nlabels wide"""
    return workspace_bytes(w, h, nlabels, ndir, cost_bytes) - 1


@contextmanager
def limited(e, nbytes, min_folded=1):
    """run under a workspace limit; at least min_folded calls must run folded"""
    before = e.folded_calls()
    e.set_workspace_limit(nbytes)
    try:
        yield
    finally:
        e.set_workspace_limit(0)
    assert e.folded_calls() - before >= min_folded, "the call did not run in the folded layout"


def check_mgm(e, oracle, ref, sec, dmin, dmax, kw=None, cost_bytes=1, mask=False):
    kw = kw or {}
    h, w = ref.shape
    with limited(e, below_resident(w, h, dmax - dmin + 1, kw.get("ndir", 8), cost_bytes)):
        out = e.mgm(ref, sec, dmin, dmax, default_params("mgm", **kw), want_mask=mask, want_right=True)
    d, c, dr = oracle.port.mgm(ref, sec, dmin, dmax, oracle.mgm_params(**kw))
    assert same(out["disp"], d), "disparity differs at %d px" % nmismatch(out["disp"], d)
    assert same(out["conf"], c), "confidence differs at %d px" % nmismatch(out["conf"], c)
    assert same(out["disp_right"], dr)
    if mask:
        assert np.array_equal(out["mask"], oracle.port.rejection_mask(d, ref, sec))


# the shapes of test_gpu_parity.py::test_mgm_end_to_end: 1 to 16 labels per lane, no-data, a positive range
@pytest.mark.parametrize("shape,dmin,dmax,nanb,seed", [
    ((64, 96), -12, 11, 0.0, 1), ((50, 81), -20, 30, 0.0, 2), ((40, 130), -64, 63, 0.0, 3), ((33, 140), -64, 63, 0.06, 4),
    ((30, 200), -90, 70, 0.0, 5), ((24, 260), -128, 127, 0.0, 6), ((70, 45), 3, 19, 0.05, 7), ((20, 400), -150, 150, 0.0, 8),
    ((18, 520), -250, 249, 0.03, 9)])
def test_fold_end_to_end(eng, oracle, shape, dmin, dmax, nanb, seed):
    h, w = shape
    ref, sec, _ = make_pair(h, w, dmin, dmax, seed=seed, nan_border=nanb)
    check_mgm(eng, oracle, ref, sec, dmin, dmax, mask=True)


@pytest.mark.parametrize("kw", [dict(tsgm=1), dict(tsgm=2), dict(tsgm=3), dict(tsgm=4), dict(ndir=2), dict(ndir=4),
                                dict(census_win=3), dict(census_win=7), dict(median=0, lr_mode=0, refine=0), dict(median=2),
                                dict(mindiff=1.0), dict(ndir=2, tsgm=4, census_win=7)])
def test_fold_options(eng, oracle, kw):
    h, w, dmin, dmax = 48, 90, -9, 14
    ref, sec, _ = make_pair(h, w, dmin, dmax, seed=21, nan_border=0.04)
    check_mgm(eng, oracle, ref, sec, dmin, dmax, kw)


@pytest.mark.parametrize("dmin,dmax,tsgm", [(-300, 299, 3), (-20, 560, 4), (-700, 450, 2)])
def test_fold_more_than_512_labels(eng, oracle, dmin, dmax, tsgm):
    ref, sec, _ = make_pair(37, 640, dmin, dmax, seed=dmax, nan_border=0.03)
    check_mgm(eng, oracle, ref, sec, dmin, dmax, dict(tsgm=tsgm))


def test_fold_weighted_float_costs(eng, oracle):
    """the float-cost flavour (another distance) folds too"""
    h, w, dmin, dmax = 57, 100, -12, 17
    ref, sec, _ = make_pair(h, w, dmin, dmax, seed=41)
    with limited(eng, below_resident(w, h, dmax - dmin + 1, cost_bytes=4)):
        out = eng.mgm(ref, sec, dmin, dmax, default_params("mgm", cost="ad", P1=12.0, P2=48.0), want_right=True)
    d, c, dr = oracle.port.mgm(ref, sec, dmin, dmax, oracle.mgm_params(cost=oracle.COSTS.index("ad"), P1=12.0, P2=48.0))
    assert same(out["disp"], d) and same(out["conf"], c) and same(out["disp_right"], dr)


def tightest(e, call, w, h, ndir=8, cost_bytes=1):
    """call() under the smallest of a ladder of limits it runs with -- the folded size of a w x h tile of 32, 64, ... 2048 labels --
    so that every pyramid level that folds at all does; -> (its result, the calls that ran folded)"""
    for D in range(32, 2049, 32):
        before = e.folded_calls()
        e.set_workspace_limit(workspace_bytes(w, h, D, ndir, cost_bytes, folded=True))
        try:
            out = call()
        except S2pbError as x:
            if x.code != _lib.ERR_NOMEM:
                raise
            continue
        finally:
            e.set_workspace_limit(0)
        n = e.folded_calls() - before
        assert n >= 1, "no call ran in the folded layout"
        return out, n
    raise AssertionError("no limit of the ladder lets the call run")


def mgm_calls(w, h, scales=6, subpix=2):
    """mgm calls of mgm_multi: one per pyramid level, plus the half-pixel pass"""
    n = 1
    while n - 1 < scales and max(w, h) > 100 and min(w, h) > 50:
        w, h, n = (w + 1) // 2, (h + 1) // 2, n + 1
    return n + (subpix > 1)


def test_fold_mgm_multi_level_hull_wider_than_512_labels(eng, oracle):
    h, w, dmin, dmax = 123, 191, -128, 61
    kw = dict(ndir=2, tsgm=4, census_win=3, P1=8.0, P2=48.0, median=1, lr_mode=0)
    p = default_params("mgm_multi", **kw)
    for seed, nanb in ((5, 0.05), (6, 0.0)):
        ref, sec, _ = make_pair(h, w, dmin, dmax, seed=seed, nan_border=nanb)
        out, _ = tightest(eng, lambda: eng.mgm(ref, sec, dmin, dmax, p, want_right=True), w, h, ndir=2)
        d, c, dr = oracle.port.mgm_multi(ref, sec, dmin, dmax, oracle.mgm_multi_params(**kw))
        assert same(out["disp"], d), "%d px differ" % nmismatch(out["disp"], d)
        assert same(out["conf"], c) and same(out["disp_right"], dr)


@pytest.mark.parametrize("shape,dmin,dmax,nanb,seed,kw", [
    ((120, 160), -20, 20, 0.0, 1, dict()), ((130, 170), -14, 16, 0.06, 5, dict()), ((110, 150), -12, 18, 0.0, 4, dict(lr_mode=2)),
    ((230, 260), -40, 40, 0.0, 3, dict(scales=3))])
def test_fold_mgm_multi(eng, oracle, shape, dmin, dmax, nanb, seed, kw):
    """the levels whose resident workspace exceeds the limit fold, the coarse ones stay resident: results as the oracle's"""
    h, w = shape
    ref, sec, _ = make_pair(h, w, dmin, dmax, seed=seed, nan_border=nanb)
    d, c, dr = oracle.port.mgm_multi(ref, sec, dmin, dmax, oracle.mgm_multi_params(**kw))
    p = default_params("mgm_multi", **kw)
    before = eng.folded_calls()
    eng.mgm(ref, sec, dmin, dmax, p)
    assert eng.folded_calls() == before, "no limit: every level runs resident"
    out, n = tightest(eng, lambda: eng.mgm(ref, sec, dmin, dmax, p, want_right=True), w, h)
    assert n < mgm_calls(w, h, p.scales, p.subpix), "some levels fold and the others do not"
    assert same(out["conf"], c), "consensus differs at %d px" % nmismatch(out["conf"], c)
    assert same(out["disp"], d), "%d px differ" % nmismatch(out["disp"], d)
    assert same(out["disp_right"], dr)


def test_fold_mgm_multi_lsd(eng, oracle):
    from test_gpu_distances import _weights
    h, w, dmin, dmax = 130, 190, -21, 16
    ref, sec, _ = make_pair(h, w, dmin, dmax, seed=51)
    wl, wr = _weights((h, w), 3, 0.75), _weights((h, w), 4, 0.75)
    p = default_params("mgm_multi_lsd", subpix=1)
    out, _ = tightest(eng, lambda: eng.mgm(ref, sec, dmin, dmax, p, want_right=True, weights=(wl, wr)), w, h, cost_bytes=4)
    d, c, dr = oracle.port.mgm_multi(ref, sec, dmin, dmax, oracle.mgm_multi_params(P1=12.0, P2=48.0, median=1, subpix=1), wl, wr)
    assert same(out["conf"], c) and same(out["disp"], d) and same(out["disp_right"], dr)


@pytest.mark.parametrize("algo,shape,dmin,dmax,nanb", [
    ("mgm", (70, 110), -12, 12, 0.05), ("mgm", (37, 640), -300, 299, 0.03), ("mgm_multi", (120, 160), -20, 20, 0.0)])
def test_fold_pkr_confidence(eng, oracle, algo, shape, dmin, dmax, nanb):
    h, w = shape
    ref, sec, _ = make_pair(h, w, dmin, dmax, seed=h + w, nan_border=nanb)
    multi = algo == "mgm_multi"
    call = lambda: eng.mgm(ref, sec, dmin, dmax, default_params(algo), want_right=True, want_pkr=True)  # noqa: E731
    if multi:
        out, _ = tightest(eng, call, w, h)
    else:
        with limited(eng, below_resident(w, h, dmax - dmin + 1)):
            out = call()
    P = oracle.mgm_multi_params() if multi else oracle.mgm_params()
    d, c, dr, pl, pr = oracle.port.mgm_pkr(ref, sec, dmin, dmax, P, multi=multi)
    assert same(out["disp"], d) and same(out["conf"], c) and same(out["disp_right"], dr)
    assert same(out["pkr_left"], pl), "%d px differ" % nmismatch(out["pkr_left"], pl)
    assert same(out["pkr_right"], pr)


@pytest.mark.parametrize("dmin,dmax,nanb", [(-64, 63, 0.0), (-64, 63, 0.05), (-256, 255, 0.0)])
def test_fold_matches_resident_1024(eng, dmin, dmax, nanb):
    ref, sec, _ = make_pair(1024, 1024, dmin, dmax, seed=7, nan_border=nanb)
    p = default_params("mgm")
    a = eng.mgm(ref, sec, dmin, dmax, p, want_right=True)
    with limited(eng, below_resident(1024, 1024, dmax - dmin + 1)):
        b = eng.mgm(ref, sec, dmin, dmax, p, want_right=True)
    for k in ("disp", "conf", "mask", "disp_right"):
        assert same(a[k], b[k]), "%s differs at %d px" % (k, nmismatch(a[k], b[k]))


def test_neither_layout_fits(eng, tmp_path, monkeypatch):
    ref, sec, _ = make_pair(40, 60, -8, 8, seed=3)
    eng.set_workspace_limit(1)
    try:
        with pytest.raises(S2pbError) as e:
            eng.mgm(ref, sec, -8, 8, default_params("mgm"))
        assert e.value.code == _lib.ERR_NOMEM and "folded" in str(e.value)
        # the drop-in raises CalledProcessError, as for any other failure of the engine
        from s2p_b200 import block_matching as bm, rasterio_compat as rio
        monkeypatch.setattr(bm, "get_engine", lambda: eng)
        im1, im2 = str(tmp_path / "a.tif"), str(tmp_path / "b.tif")
        rio.write_float_tiff(im1, ref)
        rio.write_float_tiff(im2, sec)
        with pytest.raises(subprocess.CalledProcessError):
            bm.compute_disparity_map(im1, im2, str(tmp_path / "d.tif"), str(tmp_path / "m.png"), "mgm", -8, 8)
    finally:
        eng.set_workspace_limit(0)
