"""Warps at the line lengths, borders and output sizes where the rectification warp's kernels change behaviour, shared by
tests/test_warp_oracle.py (the oracle on the CPU) and tests/test_gpu_warp_oracle.py (the engine against the oracle).

* ROI sides 4-7 and around every multiple of 32 up to 321 on each axis: the sequential prefilter below 128 samples, the
  segmented one (64-sample segments, 32-sample warm-up) above, with a last segment of 1, 2, 31, 32 or 33 samples.  The
  matrices are dyadic translations and x2 zooms, so the sample coordinates are exact.
* Sample points on the borders: px == w (valid), px just above w (NaN), px in [0, 0.5) (xi = -1), px just below 0 (NaN).
* Output sizes that are not multiples of the 32 x 8 block, 1 x 1 included.
* The anti-aliasing branch with 3 to 63 taps and every tw mod 4 (the unfiltered tail of the vertical pass starts at jlim).
* Sources with NaN (zeroed before the prefilter) and with +-Inf (spread by the recursions, segment by segment).
* TINY: spline images with a side below 4 (the ROI, or the anti-aliasing intermediate), which the engine refuses.

Tolerance of the engine: |engine - oracle| <= K * 2^-24 * max|spline coefficient| on every finite pixel, the maximum taken over
the case's spline images.  The oracle run in float32 departs from the float64 oracle by at most 11.2 such units over CASES
(the largest, border_zoom2_both_edges; most cases stay within 2-7); K is four times that."""
import functools

import numpy as np

import warp_oracle as W

K = 45
UNIT = 2.0 ** -24
FLOAT32_SPREAD = 11.2           # units, measured as described above; tests/test_warp_oracle.py keeps it true

ROI_SIDES = [4, 5, 6, 7, 31, 32, 33, 63, 64, 65, 127, 128, 129, 130, 159, 160, 161, 191, 192, 193, 255, 256, 257, 321]


@functools.lru_cache(maxsize=None)
def source(h, w, seed, special=None):
    """A smooth 12-bit image; special = "nan": a NaN block and isolated NaN, "inf": those plus +Inf and -Inf pixels."""
    from s2p_b200.synth import _blur
    rng = np.random.default_rng(seed)
    a = _blur(rng.integers(0, 4096, size=(h, w)).astype(np.float64), 0.8).astype(np.float32)
    if special:
        a[h // 3:h // 3 + 12, w // 5:w // 5 + 15] = np.nan
        a[rng.integers(0, h, 6), rng.integers(0, w, 6)] = np.nan
    if special == "inf":        # one of each next to a border
        a[17, w // 2], a[h - 30, w // 4], a[5, w - 2] = np.inf, np.inf, np.inf
        a[h - 2, 33], a[h // 2, 2 * w // 3] = -np.inf, -np.inf
    a.setflags(write=False)
    return a


def affine(sx, sy, tx, ty):
    """H whose inverse maps output (j, i) to source (sx j + tx, sy i + ty); exact for dyadic arguments."""
    return np.array([[1.0 / sx, 0, -tx / sx], [0, 1.0 / sy, -ty / sy], [0, 0, 1.0]])


def _roi_case(k):
    """ROI of ROI_SIDES[k] columns and ROI_SIDES[k + 12] rows, by a translation of (7.375, 5.625) or a x2 zoom."""
    w, h = ROI_SIDES[k], ROI_SIDES[(k + 12) % len(ROI_SIDES)]
    if k % 2:
        return (340, 340, k), affine(1, 1, 7.375, 5.625), w - 1, h - 1, (w, h)
    return (340, 340, k), affine(0.5, 0.5, 6.25, 9.75), 2 * (w - 1), 2 * (h - 1), (w, h)


# name -> ((source h, w, seed[, special]), H, ow, oh, the ROI's (w, h) where the case is built for it)
CASES = {"roi_%dx%d" % (ROI_SIDES[k], ROI_SIDES[(k + 12) % 24]): _roi_case(k) for k in range(len(ROI_SIDES))}
CASES.update({
    "border_px_eq_w": ((150, 140, 1), affine(1, 1, 0.5, 0.5), 142, 152, (140, 150)),          # px = w at the last column and row
    "border_px_above_w": ((150, 140, 1), affine(1, 1, 0.5 + 2.0 ** -12, 0.5 + 2.0 ** -12), 142, 152, (140, 150)),
    "border_px_below_half": ((150, 140, 2), affine(1, 1, -0.25, -0.375), 139, 149, (139, 149)),
    "border_px_below_zero": ((150, 140, 2), affine(1, 1, -0.5 - 2.0 ** -12, -0.5 - 2.0 ** -12), 140, 150, (140, 150)),
    "border_zoom2_both_edges": ((90, 200, 3), affine(0.5, 0.5, -0.75, -1.25), 404, 184, (200, 90)),
    "out_1x1_aa": ((60, 60, 4), affine(4, 4, 10, 12), 1, 1, (4, 4)),
    "out_33x9": ((60, 80, 5), affine(1, 1, 3.125, 7.875), 33, 9, (34, 10)),
    "out_257x201": ((260, 300, 6), affine(1, 1, 11.5, 20.25), 257, 201, (258, 202)),
    "out_257x201_rot": ((300, 340, 6), np.array([[0.985, -0.17, 30], [0.17, 0.985, -20], [0, 0, 1.0]]), 257, 201, None),
    "out_257x201_persp": ((300, 340, 7), np.array([[1.1, 0.03, -10], [0.01, 1.05, 5], [1e-4, -2e-4, 1.0]]), 257, 201, None),
    "nan_sequential": ((120, 110, 8, "nan"), affine(1, 1, 2.375, 3.625), 100, 96, None),
    "nan_inf_sequential": ((120, 110, 8, "inf"), affine(1, 1, 2.375, 3.625), 100, 96, None),
    "nan_inf_segmented": ((300, 340, 9, "inf"), affine(0.5, 0.5, 0.25, 0.75), 600, 560, (301, 281)),
    "nan_inf_aa": ((300, 340, 10, "inf"), affine(2, 2, 0, 0), 150, 140, None),
    "nan_aa": ((300, 340, 10, "nan"), affine(2, 2, 0, 0), 150, 140, None),
})
for _z, _ow, _oh in ((1.1, 41, 37), (1.25, 38, 30), (1.5, 30, 33), (2, 25, 26), (3, 22, 20), (4, 21, 23), (6, 19, 18),
                     (8, 13, 11), (9.6, 14, 12), (9.7, 20, 17), (9.7, 18, 19)):
    CASES["aa_zoom%g_%dx%d" % (_z, _ow, _oh)] = ((400, 400, int(_z * 10)), affine(_z, _z, 0, 0), _ow, _oh, None)
CASES["aa_anisotropic"] = ((300, 400, 11), affine(3, 1.25, 0, 0), 50, 60, None)
CASES["aa_rotated"] = ((360, 400, 12), np.array([[0.45, -0.1, 60], [0.1, 0.45, 20], [0, 0, 1.0]]), 150, 140, None)

TINY = {   # name -> ((source h, w, seed), H, ow, oh)
    "roi_1x1": ((60, 60, 0), affine(1, 1, 10, 10), 1, 1),
    "roi_2x9": ((60, 60, 0), affine(1, 1, 10.5, 10), 1, 9),
    "roi_9x3": ((60, 60, 0), affine(1, 1, 10, 10.5), 9, 2),
    "roi_clipped_to_3": ((60, 60, 0), affine(1, 1, 57, 10), 8, 8),       # the source ends three columns into the ROI
    "aa_1x1": ((60, 60, 0), affine(1.25, 1.25, 10, 10), 1, 1),
}


def case(name, table=CASES):
    key, H, ow, oh = table[name][:4]
    return source(*key), H, ow, oh


def oracle_run(name, dtype=np.float64):
    """-> (oracle output, stats) of a case"""
    src, H, ow, oh = case(name)
    st = {}
    return W.warp(src, H, ow, oh, dtype, st), st


def assert_matches_oracle(got, want, max_coef, k=K):
    """Identical NaN, +Inf and -Inf masks; |got - want| <= k units elsewhere."""
    assert got.shape == want.shape
    assert np.array_equal(np.isnan(got), np.isnan(want)), "%d NaN-mask mismatches" % int((np.isnan(got) != np.isnan(want)).sum())
    for f in (np.isposinf, np.isneginf):
        assert np.array_equal(f(got), f(want)), "%d %s mismatches" % (int((f(got) != f(want)).sum()), f.__name__)
    fin = np.isfinite(want)
    if fin.any():
        d = np.where(fin, np.abs(got.astype(np.float64) - want), -1.0)
        at = np.unravel_index(np.argmax(d), d.shape)
        assert d[at] <= k * UNIT * max_coef, "max |engine - oracle| = %g = %.1f units of 2^-24 max|coef| at (row, col) %s, tolerance %d" % (
            d[at], d[at] / (UNIT * max_coef), at, k)
