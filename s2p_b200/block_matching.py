"""Drop-in for ``s2p.block_matching`` (boundary #1 of SURVEY.md section 8b).

``compute_disparity_map`` keeps the reference's signature, file contract and exceptions
(s2p/block_matching.py:35-336) but, for ``algo in {'mgm', 'mgm_multi', 'mgm_multi_lsd'}``, runs the H100 engine
through the C ABI instead of spawning the ``mgm`` / ``mgm_multi`` binaries and the three
``plambda`` / ``backflow`` processes of ``create_rejection_mask`` (and, for ``mgm_multi_lsd``, the two five-command
weight-map pipelines, see ``lsd_weight_map``).  The matcher serves ``census_ncc_win`` 2 to 11; any other window goes to s2p as well.  ``algo == 'sgbm'`` with both
disparity bounds given (as s2p always passes them) runs the engine's bit-exact restatement of the
``sgbm`` binary with s2p's arguments (win 3, P1 8, P2 32, lr 1) and writes no confidence file, as the
reference does.  Any other ``algo`` (and ``sgbm`` with a bound of None) is handed to the original s2p
implementation when that package is importable.

    disp  -> float32 TIFF, NaN = rejected
    '<disp stem>_confidence.tif' -> float32 TIFF, consensus 0..nb_directions (read at s2p/__init__.py:263-265)
    mask  -> 8-bit PNG, 0 rejected / 1 accepted

``install()`` swaps the function into an importable ``s2p`` so that ``s2p/__init__.py`` and
``s2p/parallel.py`` run unchanged.
"""
import os
import subprocess

import numpy as np

from . import _lib, rasterio_compat as rio
from .config import cfg
from .engine import S2pbError, census_window_served, default_params, get_engine

try:  # share the exception class with a real s2p so that its `except` clauses keep matching
    from s2p.block_matching import MaxDisparityRangeError  # pragma: no cover
except Exception:
    class MaxDisparityRangeError(Exception):
        pass

_NATIVE = ("mgm", "mgm_multi", "mgm_multi_lsd")
SGBM_ARGS = dict(win=3, P1=8, P2=32, lr_diff=1)    # `sgbm ... dmin dmax 3 8 32 1`, s2p/block_matching.py:116-134


def disparity_bounds(width, disp_min, disp_max, max_disp_range=None):
    """The reference's treatment of the requested range (s2p/block_matching.py:62-84):
    a range wider than the image is shrunk around its centre, bounds are floored / ceiled to
    integers, and a range above ``max_disp_range`` raises MaxDisparityRangeError."""
    if disp_min is not None and disp_max is not None and disp_max - disp_min > width:
        mid = 0.5 * (disp_min + disp_max)
        disp_min, disp_max = int(mid - 0.5 * width), int(mid + 0.5 * width)
    if disp_min is not None:
        disp_min = int(np.floor(disp_min))
    if disp_max is not None:
        disp_max = int(np.ceil(disp_max))
    if max_disp_range is not None and disp_max - disp_min > max_disp_range:
        raise MaxDisparityRangeError(
            "Disparity range [{}, {}] greater than {}".format(disp_min, disp_max, max_disp_range))
    return disp_min, disp_max


def matcher_params(algo, timeout):
    """cfg -> s2pb_mgm_params, field for field what the reference passes as argv / environment
    (s2p/block_matching.py:155-186 for 'mgm', :269-308 for 'mgm_multi')."""
    p = default_params(algo)
    p.census_win = int(cfg["census_ncc_win"])
    p.ndir = int(cfg["mgm_nb_directions"])
    p.lr_mode = int(cfg["mgm_leftright_control"])
    p.lr_tau = float(cfg["mgm_leftright_threshold"])
    p.mindiff = float(cfg["mgm_mindiff_control"])
    if algo in ("mgm_multi", "mgm_multi_lsd"):
        mult = float(cfg["stereo_regularity_multiplier"])
        base = (12.0, 48.0) if algo == "mgm_multi_lsd" else (8.0, 32.0)     # s2p/block_matching.py:236-237,284-285
        p.P1, p.P2 = base[0] * mult, base[1] * mult
        p.remove_small_cc = int(cfg["stereo_speckle_filter"])
    p.timeout_ms = int(1000 * timeout) if timeout else 0
    return p


def confidence_path(disp, algo="mgm"):
    if algo == "mgm_multi_lsd":                     # s2p/block_matching.py:238
        return disp + ".confidence.tif"
    return "{}_confidence.tif".format(os.path.splitext(disp)[0])


def lsd_weight_map(im):
    """Regularity weights of 'mgm_multi_lsd' for one rectified image: what the reference's host pipeline
    (s2p/block_matching.py:199-218: qauto | lsd | cut | pview segments | plambda "255 x - 255 / 2 pow 0.1 fmax")
    writes, without starting it.  That is 1 at every pixel, whatever the image: qauto writes into its pipe in NPY, the
    format iio gives a stream without a file name; lsd reads only PGM and exits; pview draws no segment on its zero
    image, and the weight law maps 0 to 1.  /bin/sh reports the status of plambda, so the reference goes on
    (DESIGN.md section 3.4).  -> float32 (h, w)."""
    width, height = rio.image_size(im)
    return np.ones((height, width), np.float32)


def _original_compute_disparity_map():
    """s2p's own implementation (the one install() replaced, if it did), or None when s2p is not importable."""
    try:
        from s2p import block_matching as original  # pragma: no cover
    except Exception:
        return None
    fn = getattr(original, "_s2pb_original_compute_disparity_map", original.compute_disparity_map)
    return None if fn is compute_disparity_map else fn


def compute_disparity_map(im1, im2, disp, mask, algo, disp_min=None, disp_max=None, timeout=600,
                          max_disp_range=None, extra_params=""):
    """Same contract as s2p.block_matching.compute_disparity_map (see the module docstring).

    Raises MaxDisparityRangeError, subprocess.TimeoutExpired (``timeout`` seconds exceeded, as
    ``common.run(timeout=)`` does for the mgm binaries) or subprocess.CalledProcessError.
    """
    if algo == "sgbm" and disp_min is not None and disp_max is not None:
        return _sgbm(im1, im2, disp, mask, disp_min, disp_max, max_disp_range)
    if algo not in _NATIVE or not census_window_served(cfg["census_ncc_win"]):
        fn = _original_compute_disparity_map()
        if fn is None:
            what = ("algo %r" % algo) if algo not in _NATIVE else ("census_ncc_win %r" % cfg["census_ncc_win"])
            raise NotImplementedError("%s is not served by the H100 engine and the s2p package "
                                      "is not importable to fall through to" % what)
        return fn(im1, im2, disp, mask, algo, disp_min, disp_max, timeout, max_disp_range, extra_params)

    width, _ = rio.image_size(im1)
    disp_min, disp_max = disparity_bounds(width, disp_min, disp_max, max_disp_range)
    if disp_min is None or disp_max is None:       # the binaries' own default, main_mgm.cc:137-138
        disp_min = -30 if disp_min is None else disp_min
        disp_max = 30 if disp_max is None else disp_max

    cmd = ["s2pb200:%s" % algo, "-r", str(disp_min), "-R", str(disp_max), im1, im2, disp]
    print("\nRUN: %s" % " ".join(cmd))
    a, b = rio.read_band(im1), rio.read_band(im2)
    if a.shape != b.shape:
        raise subprocess.CalledProcessError(1, cmd, output="rectified images differ in size")
    try:
        weights = (lsd_weight_map(im1), lsd_weight_map(im2)) if algo == "mgm_multi_lsd" else None
        out = get_engine().mgm(a, b, disp_min, disp_max, matcher_params(algo, timeout), want_mask=True, weights=weights)
    except S2pbError as e:
        if e.code == _lib.ERR_TIMEOUT:
            raise subprocess.TimeoutExpired(cmd, timeout) from e
        # everything else (no device, a shape the engine does not serve, ...) fails loudly: there is no CPU path
        raise subprocess.CalledProcessError(-e.code, cmd, output=str(e)) from e
    rio.write_float_tiff(disp, out["disp"])
    rio.write_float_tiff(confidence_path(disp, algo), out["conf"])
    rio.write_mask_png(mask, out["mask"])


def _sgbm(im1, im2, disp, mask, disp_min, disp_max, max_disp_range):
    """The reference's 'sgbm' branch (s2p/block_matching.py:116-134): the binary, then create_rejection_mask."""
    width, _ = rio.image_size(im1)
    disp_min, disp_max = disparity_bounds(width, disp_min, disp_max, max_disp_range)
    cmd = ["s2pb200:sgbm", im1, im2, disp, str(disp_min), str(disp_max)] + [str(v) for v in SGBM_ARGS.values()]
    print("\nRUN: %s" % " ".join(cmd))
    a, b = rio.read_band(im1), rio.read_band(im2)
    if a.shape != b.shape:
        raise subprocess.CalledProcessError(1, cmd, output="rectified images differ in size")
    eng = get_engine()
    try:
        out = eng.sgbm(a, b, disp_min, disp_max, eng.sgbm_params(**SGBM_ARGS), want_mask=True)
    except S2pbError as e:
        raise subprocess.CalledProcessError(-e.code, cmd, output=str(e)) from e
    rio.write_float_tiff(disp, out["disp"])
    rio.write_mask_png(mask, out["mask"])


def install():
    """Route an importable ``s2p`` to this engine without touching its sources."""
    import s2p.block_matching as original
    if not hasattr(original, "_s2pb_original_compute_disparity_map"):
        original._s2pb_original_compute_disparity_map = original.compute_disparity_map
    original.compute_disparity_map = compute_disparity_map
    return original
