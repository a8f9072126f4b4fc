"""The rectification warp (`s2pb_homography`) against the float64 restatement of tests/warp_oracle.py, on the cases of
tests/warp_cases.py: ROI sides on both sides of every change of prefilter kernel and segment count, sample points on the
borders, odd output sizes, the anti-aliasing branch at 3 to 63 taps and every position of its unfiltered tail, and sources
with NaN and +-Inf.  Tolerance K * 2^-24 * max|spline coefficient| (tests/warp_cases.py says how K was set); NaN and
infinity masks identical."""
import numpy as np
import pytest

import warp_cases as C
import warp_oracle as W

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", sorted(C.CASES))
def test_warp_matches_oracle(engine, name):
    want, st = C.oracle_run(name)
    src, H, ow, oh = C.case(name)
    got = engine.homography(src, H, ow, oh)
    C.assert_matches_oracle(got, want, st["max_coef"])


@pytest.mark.parametrize("name", sorted(C.TINY))
def test_tiny_spline_image_is_refused(engine, name):
    """Below 4 samples a side the prefilter and the border formula would index outside the image, and the reference
    produces no image (tests/test_warp_oracle.py): the engine refuses with S2PB_ERR_ARG."""
    from s2p_b200._lib import ERR_ARG, S2pbError
    src, H, ow, oh = C.case(name, C.TINY)
    with pytest.raises(W.WarpError):
        W.warp(src, H, ow, oh)
    with pytest.raises(S2pbError) as e:
        engine.homography(src, H, ow, oh)
    assert e.value.code == ERR_ARG and "spline" in str(e.value)


def test_dropin_refuses_a_tiny_roi(engine, tmp_path):
    """The drop-in reports a tiny ROI as the binary's failure, as it does an empty one."""
    import subprocess
    from s2p_b200 import common, rasterio_compat as rio
    im = str(tmp_path / "im.tif")
    rio.write_float_tiff(im, np.array(C.source(60, 60, 0)))
    with pytest.raises(subprocess.CalledProcessError):
        common.image_apply_homography(str(tmp_path / "out.tif"), im, C.affine(1, 1, 10.5, 10), 1, 9)
