"""The float-cost flavour (the distances ad, sd, ncc, btad, btsd and / or the -wl / -wr regularity weights) on slabs wider
than 512 slots, served by the chunk-skipping cost, aggregation and WTA kernels (agg_chunked.cuh): algo mgm with a wide
disparity range, and mgm_multi whose level hulls exceed 512 labels.  The reference has no label limit
(mgm_costvolume.cc:63-72); the oracle these tests compare with is pinned to its binary at such widths
(tests/test_oracle_wide_general.py)."""
import numpy as np
import pytest

from s2p_b200.synth import make_pair
from util import nmismatch, same

pytestmark = pytest.mark.gpu


def _weights(shape, seed, ones=0.6):
    rng = np.random.default_rng(seed)
    x = rng.uniform(0, 255, shape)
    w = np.maximum(((255 - x) / 255) ** 2, 0.1).astype(np.float32)
    w[rng.random(shape) < ones] = 1.0
    return w


# 600 / 581 labels: a slab in (512, 1024] (8 warps per CTA); 1151 / 1101 / 1151 labels: a slab in (1024, 2048] (2 warps)
@pytest.mark.parametrize("cost,weighted,tsgm,ndir,dmin,dmax,nanb", [
    ("ad", True, 3, 8, -300, 299, 0.03),
    ("sd", False, 1, 8, -20, 560, 0.0),
    ("ncc", True, 2, 4, -300, 299, 0.0),
    ("census", True, 1, 4, -300, 299, 0.03),
    ("btad", True, 4, 8, -700, 450, 0.03),
    ("btsd", False, 4, 4, -600, 500, 0.0),
    ("census", True, 3, 8, -700, 450, 0.0),
    ("ad", False, 2, 8, -700, 450, 0.03),
])
def test_mgm_general_more_than_512_labels(engine, oracle, cost, weighted, tsgm, ndir, dmin, dmax, nanb):
    from s2p_b200.engine import default_params
    h, w = 37, 640
    ref, sec, _ = make_pair(h, w, dmin, dmax, seed=dmax + tsgm, nan_border=nanb)
    wts = (_weights((h, w), 7), _weights((h, w), 8)) if weighted else None
    kw = dict(tsgm=tsgm, ndir=ndir, P1=12.0, P2=48.0)
    out = engine.mgm(ref, sec, dmin, dmax, default_params("mgm", cost=cost, **kw), want_right=True, weights=wts)
    d, c, dr = oracle.port.mgm(ref, sec, dmin, dmax, oracle.mgm_params(cost=oracle.COSTS.index(cost), **kw), *(wts or (None, None)))
    assert same(out["disp"], d), "disparity differs at %d px" % nmismatch(out["disp"], d)
    assert same(out["conf"], c), "consensus differs at %d px" % nmismatch(out["conf"], c)
    assert same(out["disp_right"], dr), "right disparity differs at %d px" % nmismatch(out["disp_right"], dr)


@pytest.mark.parametrize("cost,dmin,dmax", [
    ("census", -300, 260),      # ZOOM = 1 levels of 561+ labels with weights
    ("ad", -128, 61),           # the inputs of test_mgm_multi_level_hull_wider_than_512_labels: a half-pixel pass wider than 512
])
def test_mgm_multi_lsd_hull_wider_than_512_labels(engine, oracle, cost, dmin, dmax):
    """mgm_multi with the flags and weights of algo == 'mgm_multi_lsd' (see test_gpu_distances.py::test_mgm_multi_lsd for the
    standard: the ZOOM = 1 result and the consensus exact, the half-pixel disparity to the 2e-3 tolerance)"""
    from s2p_b200.engine import default_params
    h, w = 123, 191
    for seed, nanb in ((5, 0.05), (6, 0.0)):
        ref, sec, _ = make_pair(h, w, dmin, dmax, seed=seed, nan_border=nanb)
        wl, wr = _weights((h, w), 3 + seed, 0.75), _weights((h, w), 4 + seed, 0.75)
        for subpix in (1, 2):
            out = engine.mgm(ref, sec, dmin, dmax, default_params("mgm_multi_lsd", subpix=subpix, cost=cost), want_right=True,
                             weights=(wl, wr))
            d, c, dr = oracle.port.mgm_multi(ref, sec, dmin, dmax, oracle.mgm_multi_params(
                P1=12.0, P2=48.0, median=1, subpix=subpix, cost=oracle.COSTS.index(cost)), wl, wr)
            assert same(out["conf"], c), "consensus differs at %d px" % nmismatch(out["conf"], c)
            if subpix == 1:
                assert same(out["disp"], d), "disparity differs at %d px" % nmismatch(out["disp"], d)
                assert same(out["disp_right"], dr)
            else:
                both = np.isfinite(d) & np.isfinite(out["disp"])
                assert (np.isnan(d) != np.isnan(out["disp"])).mean() < 2e-3
                assert (np.abs(d[both] - out["disp"][both]) > 0.25).mean() < 2e-3


def test_dropin_mgm_multi_lsd_more_than_512_labels(engine, oracle, tmp_path, monkeypatch):
    """compute_disparity_map(algo='mgm_multi_lsd') on a 561-label range writes its three files instead of raising"""
    from s2p_b200 import block_matching as bm, rasterio_compat as rio
    h, w, dmin, dmax = 70, 620, -300, 260
    ref, sec, _ = make_pair(h, w, dmin, dmax, seed=72, nan_border=0.02)
    im1, im2 = str(tmp_path / "rectified_ref.tif"), str(tmp_path / "rectified_sec.tif")
    disp, mask = str(tmp_path / "rectified_disp.tif"), str(tmp_path / "rectified_mask.png")
    rio.write_float_tiff(im1, ref)
    rio.write_float_tiff(im2, sec)
    wmap = {im1: _weights((h, w), 9, 0.8), im2: _weights((h, w), 10, 0.8)}
    monkeypatch.setattr(bm, "lsd_weight_map", lambda path: wmap[path])
    assert bm.compute_disparity_map(im1, im2, disp, mask, "mgm_multi_lsd", dmin, dmax) is None
    d, c, _ = oracle.port.mgm_multi(ref, sec, dmin, dmax, oracle.mgm_multi_params(P1=12.0, P2=48.0, median=1),
                                    wmap[im1], wmap[im2])
    assert same(rio.read_band(disp + ".confidence.tif"), c)
    got = rio.read_band(disp)
    both = np.isfinite(d) & np.isfinite(got)
    assert (np.isnan(d) != np.isnan(got)).mean() < 2e-3 and (np.abs(d[both] - got[both]) > 0.25).mean() < 2e-3
    assert set(np.unique(rio.read_band(mask))) <= {0, 1}
