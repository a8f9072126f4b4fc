"""The engine's `sgbm` matcher against the reference binary (3rdparty/sgbm compiled in place as oracle/_ref/sgbm, run with
MALLOC_PERTURB_=255, i.e. with the margins of its crop trick zero), live or through the digests recorded in
tests/golden/sgbm_ref_outputs.json: identical NaN masks, identical values (all multiples of 1/16), and the rejection mask
of the reference's own plambda / backflow chain, bit for bit."""
import os
import subprocess

import numpy as np
import pytest

import sgbm_oracle as SO
from oracle import oracle as O
from util import same

pytestmark = pytest.mark.gpu


def _run(engine, name):
    a, b, dmin, dmax, win, P1, P2, lr = SO.case(name)
    out = engine.sgbm(a, b, dmin, dmax, engine.sgbm_params(win=win, P1=P1, P2=P2, lr_diff=lr))
    return a, b, dmin, dmax, out


@pytest.mark.parametrize("name", sorted(SO.CASES))
def test_sgbm_matches_reference(engine, name):
    a, b, dmin, dmax, out = _run(engine, name)
    d = out["disp"]
    fin = d[np.isfinite(d)]
    assert np.array_equal(fin * 16, np.round(fin * 16)), "disparities are not multiples of 1/16"
    ref = SO.ref_digests(name)
    if SO.have_ref():                                    # a readable diff before the digest comparison
        r = SO.run_ref(a, b, dmin, dmax, *SO.CASES[name][3:])["disp"]
        nanmis = int((np.isnan(r) != np.isnan(d)).sum())
        both = np.isfinite(r) & np.isfinite(d)
        bad = np.argwhere((np.isnan(r) != np.isnan(d)) | (both & (r != d)))
        assert len(bad) == 0, "%s: NaN masks differ on %d px, values on %d px, first at (y, x) %s" % (
            name, nanmis, int((r[both] != d[both]).sum()), bad[:6].tolist())
    assert O.digest(d) == ref["disp"]
    assert O.digest(out["mask"]) == ref["mask"]
    assert int(np.isfinite(d).sum()) == ref["valid"]


def test_sgbm_cases_are_not_trivial():
    """the seeded tiles exercise the filters: most pixels valid on the textured tiles, some rejected everywhere"""
    if not SO.have_ref():
        pytest.skip("counts come from the live reference")
    for name in ("base_96x160", "speckle", "real_inputs"):
        a, b, dmin, dmax, win, P1, P2, lr = SO.case(name)
        r = SO.run_ref(a, b, dmin, dmax, win, P1, P2, lr)["disp"]
        v = np.isfinite(r).mean()
        assert 0.3 < v < 0.999, (name, v)


def test_sgbm_all_nan(engine):
    """undefined in the reference (it reads an empty sort); the engine returns all NaN and a zero mask"""
    a = np.full((30, 50), np.nan, np.float32)
    out = engine.sgbm(a, a, -5, 5)
    assert np.isnan(out["disp"]).all() and not out["mask"].any()


def test_sgbm_argument_errors(engine):
    from s2p_b200._lib import ERR_ARG, ERR_UNSUPPORTED, S2pbError
    a, b = SO.case("odd_37x61")[:2]
    for dmin, dmax, kw, code in ((5, 5, {}, ERR_ARG), (6, 5, {}, ERR_ARG), (-5, 5, dict(win=4), ERR_ARG),
                                 (-5, 5, dict(win=0), ERR_ARG), (-2100, 5, {}, ERR_UNSUPPORTED),
                                 (-5, 5, dict(win=15, P2=32), ERR_UNSUPPORTED),
                                 (-5, 5, dict(P2=5000), ERR_UNSUPPORTED)):
        with pytest.raises(S2pbError) as e:
            engine.sgbm(a, b, dmin, dmax, engine.sgbm_params(**kw))
        assert e.value.code == code, (dmin, dmax, kw)


def test_sgbm_real_pair_rectified(engine):
    """the real Pleiades pair of tests/golden/real_pair*.npz, rectified by the engine's warp, against the live reference"""
    if not (SO.have_ref() and O.have_ref_mask()):
        pytest.skip("oracle/_ref/sgbm not built")
    from util import load_real_pair
    z = load_real_pair()
    comp = lambda Hm, xy: np.asarray(Hm, np.float64) @ np.array([[1, 0, xy[0]], [0, 1, xy[1]], [0, 0, 1.0]])
    h, w = z["rectified_ref"].shape
    a = engine.homography(z["crop1"].astype(np.float32), comp(z["H1"], z["xy1"]), w, h)
    b = engine.homography(z["crop2"].astype(np.float32), comp(z["H2"], z["xy2"]), w, h)
    out = engine.sgbm(a, b, -40, 40)
    r = SO.run_ref(a, b, -40, 40)["disp"]
    assert same(out["disp"], r)
    assert np.array_equal(out["mask"], O.ref_rejection_mask(r, a, b))
    assert np.isfinite(r).mean() > 0.1


def test_sgbm_drop_in_writes_the_reference_files(engine, tmp_path):
    """compute_disparity_map(..., 'sgbm', dmin, dmax) writes the disparity TIFF and mask PNG of `sgbm ... 3 8 32 1` +
    create_rejection_mask, and no confidence file"""
    from s2p_b200 import block_matching as bm, rasterio_compat as rio
    a, b = SO.case("base_96x160")[:2]
    p1, p2, pd, pm = (str(tmp_path / n) for n in ("im1.tif", "im2.tif", "disp.tif", "mask.png"))
    rio.write_float_tiff(p1, a)
    rio.write_float_tiff(p2, b)
    bm.compute_disparity_map(p1, p2, pd, pm, "sgbm", -20.3, 11.2)
    assert sorted(os.listdir(tmp_path)) == ["disp.tif", "im1.tif", "im2.tif", "mask.png"]
    d, m = rio.read_band(pd), rio.read_band(pm)
    ref = SO.ref_digests("base_96x160")            # bounds floor / ceil to [-21, 12]: not the case's range
    want = engine.sgbm(a, b, -21, 12)
    assert same(d, want["disp"]) and np.array_equal(m, want["mask"])
    if SO.have_ref() and O.have_ref_mask():
        r = SO.run_ref(a, b, -21, 12)["disp"]
        assert same(d, r) and np.array_equal(m, O.ref_rejection_mask(r, a, b))
    assert ref["disp"]
    with pytest.raises(subprocess.CalledProcessError):
        bm.compute_disparity_map(p1, p2, pd, pm, "sgbm", 5, 5)
