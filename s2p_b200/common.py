"""Drop-in for ``s2p.common.image_apply_homography`` (boundary #2 of SURVEY.md section 8b).

``rectification.rectify_pair`` (s2p/rectification.py:281-382) is host algebra on 3x3 matrices and at most a
few hundred points; its only heavy work is the two calls ``common.image_apply_homography(out, im, H, w, h)``
(:379-380), each of which spawns the ``homography`` binary (s2p/common.py:159-180).  This module keeps that
function's signature and file contract and runs the H100 warp instead.  ``install()`` swaps it into an
importable ``s2p`` so that ``rectify_pair`` and ``s2p/__init__.py:276`` use it unchanged.
"""
import subprocess

import numpy as np

from . import rasterio_compat as rio
from .engine import S2pbError, get_engine


def needed_roi(H, w, h):
    """Source rectangle (x, y, w, h) that the output domain [0,w] x [0,h] pulls from: pre-image of the four
    corners, integer bounding box (3rdparty/homography/main.cpp:29-55)."""
    Hi = np.linalg.inv(np.asarray(H, dtype=np.float64).reshape(3, 3))
    c = np.array([[0, 0, 1], [w, 0, 1], [w, h, 1], [0, h, 1]], dtype=np.float64).T
    p = Hi @ c
    p = p[:2] / p[2]
    x0, y0 = int(np.floor(p[0].min())), int(np.floor(p[1].min()))
    return x0, y0, int(np.ceil(p[0].max() - x0)), int(np.ceil(p[1].max() - y0))


def image_apply_homography(out, im, H, w, h):
    """Same contract as s2p.common.image_apply_homography: ``out`` is written as a float32 TIFF of
    exactly ``w`` x ``h`` pixels with out(x) = im(H^-1 x), NaN outside the source."""
    H = np.asarray(H, dtype=np.float64).reshape(3, 3)
    cmd = ["s2pb200:homography", im, "-h", " ".join(str(x) for x in H.flatten()), out, "%d" % w, "%d" % h]
    print("\nRUN: %s" % " ".join(cmd))
    # read only the part of the source the output needs (the reference does the same through GDAL RasterIO,
    # main.cpp:112-149), and move the crop's origin into the homography
    sw, sh = rio.image_size(im)
    x, y, rw, rh = needed_roi(H, w, h)
    if x < 0:
        rw += x
        x = 0
    if y < 0:
        rh += y
        y = 0
    rw, rh = min(rw, sw - x), min(rh, sh - y)
    if rw <= 0 or rh <= 0:
        raise subprocess.CalledProcessError(1, cmd, output="ERROR: empty roi")
    Hc = H @ np.array([[1, 0, x], [0, 1, y], [0, 0, 1]], dtype=np.float64)
    res = []
    try:
        for band in range(1, rio.band_count(im) + 1):      # every band, like the binary (main.cpp loops over GetRasterCount):
            src = rio.read_window(im, x, y, rw, rh, band)  # s2p/__init__.py:276 warps the colour image through this function
            res.append(get_engine().homography(src, Hc, w, h))
    except S2pbError as e:
        raise subprocess.CalledProcessError(-e.code, cmd, output=str(e)) from e
    rio.write_float_tiff_bands(out, res)


def install():
    """Route an importable ``s2p`` to this warp without touching its sources."""
    import s2p.common as original
    if not hasattr(original, "_s2pb_original_image_apply_homography"):
        original._s2pb_original_image_apply_homography = original.image_apply_homography
    original.image_apply_homography = image_apply_homography
    return original
