"""The float64 restatement of the rectification warp (tests/warp_oracle.py), pinned to truths that do not depend on it or on
the engine: the textbook prefilter recursion, the closed-form order-5 B-spline, the reproduction of polynomials, and the
reference's own resampler."""
import math
import os
import subprocess

import numpy as np
import pytest

import warp_cases as C
import warp_oracle as W


def _textbook_prefilter(line):
    """The two-pole prefilter of one line, written out: causal start with the whole-sample mirror over the full line, causal
    recursion, anticausal start from the last two causal values, anticausal recursion; lambda applied once."""
    x = np.asarray(line, np.float64) * W.LAMBDA
    n = len(x)
    for z in W.POLES:
        c = np.empty(n)
        c[0] = (x[0] + z ** (n - 1) * x[n - 1] + sum((z ** k + z ** (2 * n - 2 - k)) * x[k] for k in range(1, n - 1))) / (1 - z ** (2 * n - 2))
        for k in range(1, n):
            c[k] = x[k] + z * c[k - 1]
        d = np.empty(n)
        d[n - 1] = z / (z * z - 1) * (c[n - 1] + z * c[n - 2])
        for k in range(n - 2, -1, -1):
            d[k] = z * (d[k + 1] - c[k])
        x = d
    return x


@pytest.mark.parametrize("lengths", [range(4, 130), range(130, 260), range(260, 400)], ids=["4-129", "130-259", "260-399"])
def test_prefilter_equals_the_sequential_recursion(lengths):
    """At every length, both forms of the oracle's prefilter (sequential, and segmented from 128 samples on) equal the
    recursion written out, to 1e-9 of the largest coefficient: the segments' warm-up errs by |z0|^32 ~ 2e-12, and the last
    coefficient of a 64k + 1 line is covered like any other."""
    rng = np.random.default_rng(1)
    for n in lengths:
        a = rng.uniform(-100, 4096, (n, 3))
        want = np.stack([_textbook_prefilter(a[:, k]) for k in range(3)], 1)
        for segmented in (False, True):
            got = W.prefilter_lines(a, segmented=segmented)
            assert np.abs(got - want).max() <= 1e-9 * np.abs(want).max(), (n, segmented)


def _beta5(x):
    """The centred order-5 B-spline, from its definition as a sum of truncated powers."""
    x = np.asarray(x, np.float64)
    return sum((-1) ** k * math.comb(6, k) * np.maximum(x + 3 - k, 0) ** 5 for k in range(7)) / 120


def test_weights_are_the_order5_bspline():
    """init_spline5 in float64 is the B-spline itself; formed in float32, as the kernel forms them, the weights lose up to
    6e-5 to the cancellation of the formula, and the oracle keeps that rounding."""
    t = np.concatenate([np.linspace(0, 1, 1001, endpoint=False), [2.0 ** -20, 0.5 - 2.0 ** -24]])
    exact = W.bspline5_weights(t, np.float64)
    for k in range(6):                               # w[5 - k] weighs sample xi - 2 + k, at distance t + 2 - k
        assert np.abs(exact[5 - k] - _beta5(t + 2 - k)).max() < 1e-13
    assert np.abs(exact.sum(0) - 1).max() < 1e-13
    f32 = W.bspline5_weights(t.astype(np.float32))
    assert f32.dtype == np.float32
    err = np.abs(f32.astype(np.float64) - W.bspline5_weights(t.astype(np.float32).astype(np.float64), np.float64)).max()
    assert 1e-6 < err < 6e-5


def _cubic(x, y):
    u, v = x - 130, y - 100
    return u ** 3 - 2 * u * u * v + 3 * u * v * v - v ** 3 + 50 * u * u - 40 * u * v + 60 * v * v + 1000 * u - 700 * v + 5e5


POLY_CASES = {
    "shift": C.affine(1, 1, 10.375, 20.625),
    "zoom2": C.affine(0.5, 0.5, 15.25, 20.75),
    "zoom2_x_shift_y": C.affine(0.5, 1, 12.25, 3.375),
    "rot10": np.array([[0.985, -0.174, 30], [0.174, 0.985, -40], [0, 0, 1.0]]),
    "rot_zoom_in": np.array([[1.69, 0.17, -60], [-0.17, 1.69, 20], [0, 0, 1.0]]),
    "perspective": np.array([[1.3, 0.03, -10], [0.01, 1.2, 5], [1e-4, -2e-4, 1.0]]),
}


@pytest.mark.parametrize("name", sorted(POLY_CASES))
def test_interior_reproduces_a_cubic(name):
    """Order-5 B-spline interpolation reproduces polynomials of degree <= 5.  A cubic image (exact in float32) warped with
    exact weights equals the cubic at the kernel's sample points, 30 pixels or more inside the ROI (where the boundary
    extension's effect has decayed), to 1e-9 of its range.  The engine's 6-digit poles cost 6e-12 of that."""
    h, w = 200, 260
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    src = _cubic(xx, yy)
    assert np.array_equal(src.astype(np.float32), src)
    H, ow, oh = POLY_CASES[name], 200, 150
    st = {}
    out = W.warp(src.astype(np.float32), H, ow, oh, stats=st, exact_weights=True)
    assert "aa" not in st
    x0, y0, rw, rh, Hc = W.needed_roi(H, w, h, ow, oh)
    x, y, _, _ = W.sample_coords(W.invert33(Hc), ow, oh)
    x, y = x.astype(np.float64), y.astype(np.float64)
    inside = (x > 30) & (x < rw - 31) & (y > 30) & (y < rh - 31)
    assert inside.sum() > 2000
    err = np.abs(out[inside] - _cubic(x[inside] + x0, y[inside] + y0)).max()
    assert err <= 1e-9 * np.abs(src).max(), err / np.abs(src).max()


def test_cases_reach_the_edges():
    """tests/warp_cases.py covers what its docstring promises."""
    rois = {}
    for name, c in C.CASES.items():
        src, H, ow, oh = C.case(name)
        x, y, w, h, _ = W.needed_roi(H, src.shape[1], src.shape[0], ow, oh)
        if c[4] is not None:
            assert (w, h) == c[4], name
        rois[name] = (w, h)
    for L in C.ROI_SIDES:
        assert any(w == L for w, _ in rois.values()) and any(h == L for _, h in rois.values()), L
    assert {(1, 1), (33, 9), (257, 201)} <= {c[2:4] for c in C.CASES.values()}
    taps, tails = set(), set()
    for name in C.CASES:
        if name.startswith("aa_"):
            aa = C.oracle_run(name)[1]["aa"]
            taps |= {g["ks"] for g in aa}
            tails |= {g["tw"] % 4 for g in aa}
    assert {3, 63} <= taps and len(taps) >= 8 and tails == {0, 1, 2, 3}, (sorted(taps), tails)
    _, H, ow, oh = C.case("border_px_eq_w")
    x, y, px, py = W.sample_coords(W.invert33(W.needed_roi(H, 140, 150, ow, oh)[4]), ow, oh)
    assert (px == 140).any() and (px > 140).any() and (py == 150).any()
    _, H, ow, oh = C.case("border_px_above_w")
    _, _, px, _ = W.sample_coords(W.invert33(W.needed_roi(H, 140, 150, ow, oh)[4]), ow, oh)
    assert ((px > 140) & (px < 140.001)).any()
    _, H, ow, oh = C.case("border_px_below_half")
    _, _, px, _ = W.sample_coords(W.invert33(W.needed_roi(H, 140, 150, ow, oh)[4]), ow, oh)
    assert ((px >= 0) & (px < 0.5)).any()
    for name in ("nan_inf_sequential", "nan_inf_segmented"):
        out = C.oracle_run(name)[0]
        assert np.isnan(out).any(), name
    assert np.isfinite(C.oracle_run("nan_inf_segmented")[0]).mean() > 0.05       # the infinities stay local to their segments
    for name in C.TINY:
        src, H, ow, oh = C.case(name, C.TINY)
        with pytest.raises(W.WarpError):
            W.warp(src, H, ow, oh)


def test_float32_spread_is_what_the_tolerance_assumes():
    """The oracle in float32 stays within FLOAT32_SPREAD units of the float64 oracle on every case, with identical NaN and
    infinity masks: the tolerance of tests/test_gpu_warp_oracle.py is four times that."""
    worst = 0.0
    for name in sorted(C.CASES):
        want, st = C.oracle_run(name)
        got, _ = C.oracle_run(name, np.float32)
        C.assert_matches_oracle(got, want, st["max_coef"], k=C.FLOAT32_SPREAD)
        fin = np.isfinite(want)
        if fin.any():
            worst = max(worst, np.abs(got[fin] - want[fin]).max() / (C.UNIT * st["max_coef"]))
    assert C.K >= 4 * worst and worst > 0.5 * C.FLOAT32_SPREAD, worst


def test_oracle_agrees_with_the_reference(oracle):
    """On the cases of tests/test_gpu_homography.py, the oracle is within that file's tolerance of the reference's own
    resampler (live where oracle/_ref is built, its recorded samples elsewhere)."""
    from test_gpu_homography import CASES, REL_TOL, _src
    src = _src()
    for name, H in sorted(CASES.items()):
        want = oracle.ref_homography_sampled(src, H, 256, 200)
        got = W.warp(src, H, 256, 200)
        nan_diff = int((want.nan != np.isnan(got)).sum())
        assert nan_diff <= max(2, got.size // 5000), (name, nan_diff)
        g = want.values_of(got)
        both = np.isfinite(want.val) & np.isfinite(g)
        assert both.any()
        assert np.abs(want.val[both] - g[both]).max() <= REL_TOL * np.nanmax(np.abs(src)), name


def test_reference_refuses_a_tiny_roi(oracle, tmp_path):
    """The reference cannot warp a spline image with a side below 4: prepareSpline's `i < height - 4` wraps around in
    size_t and it reads outside the image.  Recorded outcome: each TINY case ends on SIGSEGV without writing an output,
    while a 4 x 4 ROI warps.  The engine refuses these cases with S2PB_ERR_ARG."""
    if not oracle.have_ref_homography():
        pytest.skip("oracle/_ref/homography_ref is not built")
    exe = os.path.join(oracle.REF_DIR, "homography_ref")
    a = str(tmp_path / "src.pfm")
    oracle.write_pfm(a, np.array(C.source(60, 60, 0)))
    for name, (key, H, ow, oh) in sorted(C.TINY.items()) + [("roi_4x4", ((60, 60, 0), C.affine(1, 1, 10, 10), 4, 4))]:
        out = str(tmp_path / (name + ".pfm"))
        r = subprocess.run([exe, a, " ".join(repr(float(v)) for v in H.ravel()), out, str(ow), str(oh)], capture_output=True, timeout=120)
        if name == "roi_4x4":
            assert r.returncode == 0 and os.path.exists(out)
        else:
            assert r.returncode != 0 and not os.path.exists(out), (name, r.returncode)
