"""The oracle of the height-map localisation (tests/localization_oracle.py) and the tri-stereo fixture, checked on the CPU:
the reference's rpc_localization meets its own stopping test on the real camera when its output is projected back by the
numpy polynomials, and the numpy restatement of the iteration agrees with it."""
import os

import numpy as np
import pytest

import localization_oracle as LO


def _finite_samples(name):
    heights, rpc, ox, oy, want = LO.ref_sampled(name)
    rows, cols = np.divmod(want.idx, heights.shape[1])
    z = heights.ravel()[want.idx].astype(np.float64)
    ok = ~np.isnan(z)
    return rpc, cols[ok] + ox, rows[ok] + oy, z[ok], want.val[ok]


def test_rpc_localization_meets_its_stopping_test_on_the_real_camera():
    """img_02.tif's camera has ground->image polynomials only, so every pixel goes through the iteration of c/rpc.c:378-411"""
    rpc, cols, rows, z, ll = _finite_samples("triplet")
    assert not np.isfinite(rpc.numx[0])
    assert len(z) > 1000 and np.isfinite(ll).all()
    r2 = LO.residual2(rpc, cols, rows, z, ll[:, 0], ll[:, 1])
    assert r2.max() <= LO.STOP


@pytest.mark.parametrize("name", ["triplet", "synthetic_iterative"])
def test_numpy_restatement_matches_rpc_localization(name):
    rpc, cols, rows, z, ll = _finite_samples(name)
    lon, lat, converged = LO.localize(rpc, cols, rows, z)
    assert converged.all()
    assert np.abs(lon - ll[:, 0]).max() < 1e-9 and np.abs(lat - ll[:, 1]).max() < 1e-9


def test_triplet_fixture():
    t = LO.triplet()
    assert os.path.getsize(LO.TRIPLET) < 512 * 1024
    assert t["rpc"].shape == (92,) and t["heights"].dtype == np.float32 and t["heights"].shape == (200, 200)
    assert tuple(t["off"]) == (400.0, 400.0)                    # (250, 250) into the map of the ROI at (150, 150)
    assert 0.05 < np.isnan(t["heights"]).mean() < 0.3
    # the window lies on the expected DSM's 0.5 m grid (tiepoint 698053.031, 4792984.069)
    assert float(t["dsm_res"]) == 0.5
    for v, o in ((t["dsm_xoff"], 698053.031), (t["dsm_yoff"], 4792984.069)):
        assert abs((float(v) - o) / 0.5 - round((float(v) - o) / 0.5)) < 1e-6
    assert 0.5 < np.isfinite(t["dsm"]).mean()
    assert 0 < float(t["dz_median"]) < float(t["dz_p99"]) and int(t["dz_cells"]) > 20000
