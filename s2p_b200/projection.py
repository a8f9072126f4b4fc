"""The output coordinate systems of ``s2p.triangulation.disp_to_xyz`` that the GPU serves.

s2p triangulates to WGS84 (lon, lat, alt), EPSG:4979, and projects the cloud to ``out_crs`` with pyproj
(s2p/triangulation.py:147-160); when the configuration leaves ``out_crs`` unset it becomes the UTM zone of the ROI
(s2p/initialization.py:133-141).  The device projects to the UTM zones of WGS84, EPSG 32601-32660 (north) and 32701-32760
(south), with PROJ's exact transverse Mercator (``csrc/projection_kernels.cuh``).  No output CRS, 4979 and 4326 leave
(lon, lat, alt) as they are, as pyproj does.  Any other target -- a compound CRS with a geoid height such as
``epsg:32740+5773``, another datum, another projection -- goes through the reference's pyproj code when it is importable,
and raises ``S2pbError`` with ``ERR_UNSUPPORTED`` otherwise.

A target is read without pyproj: an ``"epsg:NNNN"`` string (any case), an int, or any object with ``.to_epsg()`` (a
``pyproj.CRS``).
"""
import re

import numpy as np

from . import _lib
from .engine import get_engine

GEOGRAPHIC = (4979, 4326)


def epsg_of(crs):
    """the EPSG code of crs, or None when it is not one the code can be read from"""
    if isinstance(crs, (int, np.integer)) and not isinstance(crs, bool):
        return int(crs)
    if isinstance(crs, str):
        m = re.fullmatch(r"\s*epsg:(\d+)\s*", crs, re.IGNORECASE)
        return int(m.group(1)) if m else None
    to_epsg = getattr(crs, "to_epsg", None)
    if callable(to_epsg):
        code = to_epsg()
        return None if code is None else int(code)
    return None


def utm_target(crs):
    """-> (zone, south) for the targets the device serves: (0, False) when the cloud stays in (lon, lat, alt) -- no
    output CRS (s2p's `if out_crs and ...`), EPSG 4979 or 4326 -- and (zone, south) for EPSG 326zz / 327zz; None for any
    other target"""
    if not crs:
        return 0, False
    code = epsg_of(crs)
    if code in GEOGRAPHIC:
        return 0, False
    if code is not None and (32601 <= code <= 32660 or 32701 <= code <= 32760):
        return code % 100, code > 32700
    return None


def lonlat_to_utm(lonlatalt, zone, south=False, engine=None):
    """(..., 3) float64 (lon, lat in degrees, alt) -> (..., 3) float64 (easting, northing, alt) in UTM zone `zone` of WGS84"""
    return (engine or get_engine()).lonlat_to_utm(lonlatalt, zone, south)


def pyproj_original(lonlatalt, out_crs):
    """The reference's change of coordinates (s2p/triangulation.py:147-160) for the targets the device does not serve:
    s2p.geographiclib's pyproj wrappers when they are importable, S2pbError(ERR_UNSUPPORTED) otherwise."""
    try:
        from s2p import geographiclib
        in_crs = geographiclib.pyproj_crs("epsg:4979")
    except ImportError:
        raise _lib.S2pbError(_lib.ERR_UNSUPPORTED, "output CRS %r: only WGS84 (EPSG 4979, 4326) and its UTM zones are projected on "
                             "the device, and s2p.geographiclib (pyproj) is not importable" % (out_crs,)) from None
    if not (out_crs and out_crs != in_crs):
        return lonlatalt
    h, w = lonlatalt.shape[:2]
    lla = lonlatalt.reshape(-1, 3)
    x, y, z = geographiclib.pyproj_transform(lla[:, 0], lla[:, 1], in_crs, out_crs, lla[:, 2])
    return np.column_stack((x, y, z)).reshape(h, w, 3).astype(np.float64)
