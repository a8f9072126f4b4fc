"""Tiles wider than the DCT tables the device keeps once per width (8192 px), and mgm_multi tiles wider than 4000 px, bit for bit
with the CPU port of the matcher (oracle/liboracle.so) and, where oracle/_ref is built, with the reference binaries themselves:

- `mgm` at 8193 and 12000 px, `mgm_multi` and `mgm_multi_lsd` (with weights) at 4001, 6000 and 8193 px, with no-data rows and
  columns so that the round trip of the matched image transforms rows: disparity, confidence, right disparity and mask;
- the tables streamed in K-panels (table limit 0) against the same tiles with resident tables;
- the folded workspace layout at 8193 px;
- s2pb_rectify_match and s2pb_pair_tile_to_ply on a wide tile against their stepwise calls, and the drop-in
  compute_disparity_map on a wide tile.
The tiles are short (16 to 24 rows) so that the CPU side stays cheap.
"""
import numpy as np
import pytest

from s2p_b200.engine import Engine, default_params
from s2p_b200.synth import make_pair
from util import nmismatch, same

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def streamed():
    """an engine that streams every table of rows wider than 8192 px"""
    e = Engine(0)
    e.set_dct_table_limit(0)
    yield e
    e.close()


def nodata(ref, sec, seed):
    """no-data strips at the left of the reference and the right of the secondary view, and a no-data row and a few no-data
    columns in each (the round trip then transforms rows of both).  (make_pair's nan_border blanks whole rows of a short tile.)"""
    rng = np.random.default_rng(seed)
    h, w = ref.shape
    ref[:, :40] = np.nan
    sec[:, w - 40:] = np.nan
    for im in (ref, sec):
        im[rng.integers(0, h)] = np.nan
        im[:, rng.integers(0, w, 5)] = np.nan
    return ref, sec


def wide_pair(h, w, dmin, dmax, seed):
    ref, sec, _ = make_pair(h, w, dmin, dmax, seed=seed)
    return nodata(ref, sec, seed)


def weights(shape, seed):
    rng = np.random.default_rng(seed)
    return tuple(rng.uniform(0.25, 1.0, shape).astype(np.float32) for _ in range(2))


def reference(oracle, algo, ref, sec, dmin, dmax, wts=None):
    """-> (disp, conf, disp_right) of the CPU port, checked against the reference binary where it is built"""
    multi = algo != "mgm"
    kw = dict(P1=12.0, P2=48.0, median=1) if algo == "mgm_multi_lsd" else {}
    P = oracle.mgm_multi_params(**kw) if multi else oracle.mgm_params()
    wl, wr = wts if wts else (None, None)
    d, c, dr = (oracle.port.mgm_multi if multi else oracle.port.mgm)(ref, sec, dmin, dmax, P, wl, wr)
    if oracle.have_ref():
        r = oracle.run_ref(ref, sec, dmin, dmax, P, threads=1, wl=wl, wr=wr)
        assert same(r["disp"], d) and same(r["conf"], c) and same(r["dispR"], dr), "the port differs from the reference binary"
    return d, c, dr


def check(out, oracle, ref, sec, d, c, dr):
    assert np.isfinite(d).mean() > 0.5, "a tile the matcher mostly rejects tells little"
    assert same(out["disp"], d), "disparity differs at %d px" % nmismatch(out["disp"], d)
    assert same(out["conf"], c), "confidence differs at %d px" % nmismatch(out["conf"], c)
    assert same(out["disp_right"], dr), "right disparity differs at %d px" % nmismatch(out["disp_right"], dr)
    assert np.array_equal(out["mask"], oracle.port.rejection_mask(d, ref, sec))


CASES = [("mgm", 8193, 16, -12, 11), ("mgm", 12000, 16, -9, 6),
         ("mgm_multi", 4001, 20, -10, 9), ("mgm_multi", 6000, 20, -8, 7), ("mgm_multi", 8193, 16, -8, 7),
         ("mgm_multi_lsd", 4001, 20, -10, 9), ("mgm_multi_lsd", 6000, 20, -8, 7), ("mgm_multi_lsd", 8193, 16, -8, 7)]


@pytest.mark.parametrize("algo,w,h,dmin,dmax", CASES, ids=["%s-%d" % (c[0], c[1]) for c in CASES])
def test_wide_tile_matches_the_reference(eng, streamed, oracle, algo, w, h, dmin, dmax):
    ref, sec = wide_pair(h, w, dmin, dmax, seed=w)
    wts = weights((h, w), w) if algo == "mgm_multi_lsd" else None
    d, c, dr = reference(oracle, algo, ref, sec, dmin, dmax, wts)
    out = eng.mgm(ref, sec, dmin, dmax, default_params(algo), want_right=True, weights=wts)
    check(out, oracle, ref, sec, d, c, dr)
    if w > 8192:            # the same tile with every table streamed in panels
        check(streamed.mgm(ref, sec, dmin, dmax, default_params(algo), want_right=True, weights=wts), oracle, ref, sec, d, c, dr)


def test_streamed_round_trip_without_nodata(eng, streamed):
    """no row needs the round trip: nothing is streamed, and the results are those of the resident tables"""
    ref, sec, _ = make_pair(16, 9000, -6, 5, seed=3)
    p = default_params("mgm")
    a, b = eng.mgm(ref, sec, -6, 5, p, want_right=True), streamed.mgm(ref, sec, -6, 5, p, want_right=True)
    for k in ("disp", "conf", "mask", "disp_right"):
        assert same(a[k], b[k]), k


def test_streamed_with_ragged_columns(eng, streamed):
    """no-data in many columns: the inverse product streams the rows of its table of all those columns"""
    ref, sec, _ = make_pair(24, 8300, -7, 8, seed=5)
    rng = np.random.default_rng(5)
    for im in (ref, sec):
        im[rng.random(im.shape) < 0.02] = np.nan
    for algo in ("mgm", "mgm_multi"):
        p = default_params(algo)
        a, b = eng.mgm(ref, sec, -7, 8, p, want_right=True), streamed.mgm(ref, sec, -7, 8, p, want_right=True)
        for k in ("disp", "conf", "mask", "disp_right"):
            assert same(a[k], b[k]), "%s: %s differs at %d px" % (algo, k, nmismatch(a[k], b[k]))


def test_wide_tile_folded(oracle):
    """a wide tile in the folded layout, its tables streamed because the workspace limit also caps them"""
    from test_gpu_fold import below_resident
    h, w, dmin, dmax = 16, 8193, -12, 11
    ref, sec = wide_pair(h, w, dmin, dmax, seed=77)
    d, c, dr = reference(oracle, "mgm", ref, sec, dmin, dmax)
    with Engine(0) as e:
        e.set_workspace_limit(below_resident(w, h, dmax - dmin + 1))
        out = e.mgm(ref, sec, dmin, dmax, default_params("mgm"), want_right=True)
        assert e.folded_calls() >= 1
    check(out, oracle, ref, sec, d, c, dr)


def test_rectify_match_wide_equals_its_two_steps(eng):
    ref, sec, _ = make_pair(24, 8400, -10, 9, seed=11)
    ref, sec = nodata(ref, sec, 11)
    H1 = np.array([[1.0, 0.0005, -3.5], [0.0, 1.0, -1.25], [0.0, 0.0, 1.0]])
    H2 = np.array([[1.0, 0.0, -4.0], [0.0007, 1.0, -1.0], [0.0, 0.0, 1.0]])
    w, h = 8300, 20
    for algo in ("mgm", "mgm_multi"):
        p = default_params(algo)
        r1, r2 = eng.homography(ref, H1, w, h), eng.homography(sec, H2, w, h)
        want = eng.mgm(r1, r2, -10, 9, p, want_right=True)
        got = eng.rectify_match(ref, H1, sec, H2, w, h, -10, 9, p, want_right=True)
        for k in ("disp", "conf", "mask", "disp_right"):
            assert same(got[k], want[k]), "%s: %s" % (algo, k)


def test_pair_tile_to_ply_wide_equals_the_stepwise_calls(eng):
    from test_gpu_pair_tile import R, PW, N, SOUTH, ZONE, _params, _real, _stepwise
    a = _real()
    ref, sec, _ = make_pair(30, 8400, -12, 11, seed=13)
    ref, sec = nodata(ref, sec, 13)
    H1 = np.array([[1.0, 0.0004, -6.5], [0.0, 1.0, -5.25], [0.0, 0.0, 1.0]])
    H2 = np.array([[1.0, 0.0, -7.0], [0.0006, 1.0, -5.0], [0.0, 0.0, 1.0]])
    t = dict(a, src1=ref, src2=sec, H1=H1, H2=H2, w=8300, h=20, dmin=-12, dmax=11, H_ref=np.round(H1, 6), H_sec=np.round(H2, 6))
    for algo in ("mgm", "mgm_multi"):
        want_rec, want = _stepwise(eng, t, algo, None, 2, True, "stretch", True)
        names = ("rect1", "rect2", "disp", "mask", "conf", "disp_right")
        rec, out = eng.pair_tile_to_ply(t["src1"], t["H1"], t["src2"], t["H2"], t["w"], t["h"], t["dmin"], t["dmax"], t["mask_orig"],
                                        t["H_ref"], t["H_sec"], t["rpc1"], t["rpc2"], t["bbx"], ZONE, SOUTH, params=_params(eng, algo),
                                        erode_radius=2, r=R, p=PW, n=N, confidence=True, want=names)
        assert rec.dtype == want_rec.dtype and rec.tobytes() == want_rec.tobytes(), algo
        for k in names:
            assert same(out[k], want[k]), "%s: %s" % (algo, k)


def test_drop_in_serves_a_wide_tile(eng, tmp_path, monkeypatch):
    """compute_disparity_map runs a tile wider than 8192 px on the engine instead of raising"""
    from s2p_b200 import block_matching as bm, rasterio_compat as rio
    ref, sec = wide_pair(16, 8200, -6, 5, seed=17)
    monkeypatch.setattr(bm, "get_engine", lambda: eng)
    im1, im2 = str(tmp_path / "a.tif"), str(tmp_path / "b.tif")
    rio.write_float_tiff(im1, ref)
    rio.write_float_tiff(im2, sec)
    for algo in ("mgm", "mgm_multi"):
        disp, mask = str(tmp_path / ("d_%s.tif" % algo)), str(tmp_path / ("m_%s.png" % algo))
        bm.compute_disparity_map(im1, im2, disp, mask, algo, -6, 5)
        want = eng.mgm(ref, sec, -6, 5, bm.matcher_params(algo, 600))
        assert same(rio.read_band(disp), want["disp"]), algo
