"""Drop-in for the native half of ``s2p.triangulation.disp_to_xyz`` (SURVEY.md section 8f rank 2).

The reference triangulates through ``lib/disp_to_h.so`` loaded with ctypes (s2p/triangulation.py:18-20) and calls
``lib.disp_to_lonlatalt(lonlatalt, err, dispx, dispy, msk, w, h, msk_orig, ww, hh, H1, H2, byref(rpc1),
byref(rpc2), bbx)`` (:134-143).  ``s2pb_disp_to_xyz`` takes the same argument list (plus the context, then the output
zone, 0 for lon, lat, alt) and ``RPCStruct`` below has the layout of the reference's ``struct rpc`` / ``RPCStruct``;
``install()`` swaps the library handle of an importable ``s2p.triangulation`` for an adapter that forwards the very same
call.

The 3D outlier filter of the same library, ``count_3d_neighbors`` and ``remove_isolated_3d_points`` (c/disp_to_h.c:143-230),
which ``filter_xyz`` runs on the cloud of a tile (s2p/triangulation.py:275-343), goes through the adapter too.

``disp_to_xyz`` (s2p/triangulation.py:85-162) triangulates and projects the cloud to its output CRS in one device call
(``s2pb_disp_to_xyz``) when that CRS is WGS84, one of its UTM zones, an ETRS89 UTM zone or an RGF93 v1 Lambert grid
(``projection.output_target``); ``install()`` replaces the reference's
function with it.

``height_map`` (s2p/triangulation.py:346-389), the tri-stereo step that triangulates a pair and resamples the altitude onto the
tile grid, runs as one device call (``s2pb_height_map``); ``install()`` replaces the reference's function with it.

``height_map_to_xyz`` (s2p/triangulation.py:165-217), which localises the merged tri-stereo height map with the reference
image's camera and projects it to the output CRS, runs as one device call (``s2pb_height_map_to_xyz``) for the same targets
as ``disp_to_xyz``; ``install()`` replaces the reference's function with it.
"""
import ctypes
from ctypes import c_double

import numpy as np

from . import projection
from .engine import get_engine


class RPCStruct(ctypes.Structure):
    """``struct rpc`` (c/rpc.h:14-32), field for field as in s2p/triangulation.py:23-40."""
    _fields_ = [("numx", c_double * 20), ("denx", c_double * 20), ("numy", c_double * 20), ("deny", c_double * 20),
                ("scale", c_double * 3), ("offset", c_double * 3),
                ("inumx", c_double * 20), ("idenx", c_double * 20), ("inumy", c_double * 20), ("ideny", c_double * 20),
                ("iscale", c_double * 3), ("ioffset", c_double * 3),
                ("dmval", c_double * 4), ("imval", c_double * 4), ("delta", c_double)]


def rpc_from_geotiff_tag(tag, delta=1.0):
    """RPCStruct from the 92 doubles of a GeoTIFF RPCCoefficientTag (50844): [err_bias, err_rand, line_off, samp_off, lat_off,
    long_off, height_off, line_scale, samp_scale, lat_scale, long_scale, height_scale, line_num[20], line_den[20], samp_num[20],
    samp_den[20]] -- filled the way s2p/triangulation.py:42-83 fills its structure from an rpcm model read from the same
    tag: only the ground->image polynomials exist, the other direction is NaN (the library then iterates, c/rpc.c:378-411)."""
    t = [float(x) for x in tag]
    if len(t) != 92:
        raise ValueError("an RPCCoefficientTag holds 92 doubles, got %d" % len(t))
    r = RPCStruct()
    line_off, samp_off, lat_off, lon_off, h_off, line_sc, samp_sc, lat_sc, lon_sc, h_sc = t[2:12]
    r.offset[0], r.offset[1], r.offset[2] = samp_off, line_off, h_off
    r.ioffset[0], r.ioffset[1], r.ioffset[2] = lon_off, lat_off, h_off
    r.scale[0], r.scale[1], r.scale[2] = samp_sc, line_sc, h_sc
    r.iscale[0], r.iscale[1], r.iscale[2] = lon_sc, lat_sc, h_sc
    for i in range(20):
        r.inumy[i], r.ideny[i], r.inumx[i], r.idenx[i] = t[12 + i], t[32 + i], t[52 + i], t[72 + i]
        r.numx[i] = r.denx[i] = r.numy[i] = r.deny[i] = float("nan")
    r.delta = delta
    return r


def disp_to_lonlatalt(disp, mask_rect, mask_orig, H1, H2, rpc1, rpc2, img_bbx, dispy=None, engine=None):
    """numpy-level call: -> (lonlatalt (h, w, 3) float64, err (h, w) float32).
    rpc1 / rpc2: any ctypes structure with the layout of ``RPCStruct`` (the reference's own class works)."""
    return (engine or get_engine()).disp_to_xyz(disp, mask_rect, mask_orig, H1, H2, rpc1, rpc2, img_bbx, zone=0, dispy=dispy)


def disp_to_xyz(rpc1, rpc2, H1, H2, disp, mask_rect, img_bbx, mask_orig, A=None, out_crs=None, engine=None):
    """s2p.triangulation.disp_to_xyz (s2p/triangulation.py:85-162): -> (xyz (h, w, 3) float64 in the coordinates of
    out_crs, err (h, w) float32).  rpc1 / rpc2 are wrapped as the reference wraps them (``RPCStruct(rpc)``); ctypes
    structures pass as they are.  No out_crs, EPSG 4979 / 4326, the UTM zones of WGS84 and ETRS89 and the RGF93 v1 Lambert
    grids, and those with EGM96 heights (+5773) when the grid is found, run on the device in one call; any other out_crs is triangulated on the device and projected by the reference's pyproj code (``projection``)."""
    r1, r2 = _rpc_struct(rpc1), _rpc_struct(rpc2)
    if A is not None:                                       # pointing correction (s2p/triangulation.py:114-115)
        H2 = np.dot(H2, np.linalg.inv(A))
    eng = engine or get_engine()
    target = projection.output_target(out_crs, eng)
    if target is None:
        lla, err = disp_to_lonlatalt(disp, mask_rect, mask_orig, H1, H2, r1, r2, img_bbx, engine=eng)
        return projection.pyproj_original(lla, out_crs), err
    return eng.disp_to_xyz(disp, mask_rect, mask_orig, H1, H2, r1, r2, img_bbx, *target)


def height_map_to_xyz(heights, rpc, off_x=0, off_y=0, out_crs=None, engine=None):
    """s2p.triangulation.height_map_to_xyz (s2p/triangulation.py:165-217): -> (h, w, 3) float64, every pixel of the height
    map at ``heights`` (a raster file; band 1, read in its stored dtype) localised by the camera ``rpc`` at image pixel
    (col + off_x, row + off_y) and its height, in the coordinates of out_crs.  rpc is wrapped as the reference wraps it
    (``RPCStruct(rpc)``); ctypes structures pass as they are.  NaN heights give NaN in all three coordinates (the reference
    leaves lon and lat undefined there).  No out_crs, EPSG 4979 / 4326, the UTM zones of WGS84 and ETRS89 and the RGF93 v1
    Lambert grids, and those with EGM96 heights (+5773) when the grid is found, run on the device in one call; any other out_crs is localised on the device and projected by the reference's pyproj code (``projection``)."""
    from . import rasterio_compat
    h_map = rasterio_compat.read_band_stored(heights)
    r = _rpc_struct(rpc)
    eng = engine or get_engine()
    target = projection.output_target(out_crs, eng)
    if target is None:
        return projection.pyproj_original(eng.height_map_to_xyz(h_map, r, off_x, off_y), out_crs)
    return eng.height_map_to_xyz(h_map, r, off_x, off_y, *target)


def height_map(x, y, w, h, rpc1, rpc2, H1, H2, disp, mask, mask_orig, A=None, engine=None):
    """s2p.triangulation.height_map (s2p/triangulation.py:346-389): -> (h, w) float64 altitudes on the grid of the tile
    (x, y, w, h) of the reference image, NaN where the rectified map has no height within one pixel.  rpc1 / rpc2 are
    the camera models, wrapped as disp_to_xyz wraps them (``RPCStruct(rpc)``); ctypes structures pass as they are."""
    return (engine or get_engine()).height_map(x, y, w, h, _rpc_struct(rpc1), _rpc_struct(rpc2), H1, H2, disp, mask, mask_orig, A)


def _rpc_struct(rpc):
    if isinstance(rpc, ctypes.Structure):
        return rpc
    import s2p.triangulation as reference          # its RPCStruct reads an rpcm.RPCModel (s2p/triangulation.py:42-83)
    return reference.RPCStruct(rpc)


def count_3d_neighbors(xyz, r, p, engine=None):
    """s2p.triangulation.count_3d_neighbors: -> (h, w) int32, per point the number of points of its (2p+1)^2 window
    (clipped at the border, itself included) closer than r units."""
    return (engine or get_engine()).count_3d_neighbors(xyz, r, p)


def remove_isolated_3d_points(xyz, r, p, n, q=1, engine=None):
    """s2p.triangulation.remove_isolated_3d_points: NaN into the points with fewer than n neighbours closer than r in
    their (2p+1)^2 window, except those joined to a kept point by a chain of close points within (2q+1)^2 windows.
    In place on np.ascontiguousarray(xyz), as the reference: a C-contiguous float64 xyz is modified, another is not."""
    (engine or get_engine()).remove_isolated_3d_points(xyz, r, p, n, q)


def filter_xyz(xyz, r, n, img_gsd, engine=None):
    """s2p.triangulation.filter_xyz: remove_isolated_3d_points with p = ceil(r / img_gsd) and q = 1."""
    p = np.ceil(r / img_gsd).astype(int)
    remove_isolated_3d_points(xyz, r, p, n, engine=engine)


class _LibAdapter:
    """Stands in for ``s2p.triangulation.lib``: ``disp_to_lonlatalt``, ``count_3d_neighbors`` and
    ``remove_isolated_3d_points`` go to the GPU, anything else to the original.  Each takes the positional arguments of
    the library function and writes into the arrays it is given."""

    def __init__(self, original):
        self._original = original

        def call(lonlatalt, err, dispx, dispy, msk, w, h, msk_orig, ww, hh, ha, hb, rpca, rpcb, bbx):
            out, e = disp_to_lonlatalt(dispx, msk, msk_orig, ha, hb, rpca._obj, rpcb._obj, bbx, dispy=dispy)
            lonlatalt[...] = out
            err[...] = e

        def count(out, xyz, w, h, r, p):
            _check_cloud(xyz, w, h)
            out[...] = count_3d_neighbors(xyz, np.float32(r), p)

        def remove(xyz, w, h, r, p, n, q):
            _check_cloud(xyz, w, h)
            remove_isolated_3d_points(xyz, np.float32(r), p, n, q)

        # s2p assigns .argtypes before calling (s2p/triangulation.py:118,293,324)
        for name, fn in (("disp_to_lonlatalt", call), ("count_3d_neighbors", count), ("remove_isolated_3d_points", remove)):
            fn.argtypes = None
            setattr(self, name, fn)

    def __getattr__(self, name):
        return getattr(self._original, name)


def _check_cloud(xyz, w, h):
    """what the ndpointer(c_double, shape=(h, w, 3)) argument type s2p assigns would check, and that xyz is the memory
    the library would write to"""
    if not isinstance(xyz, np.ndarray) or xyz.dtype != np.float64 or xyz.shape != (h, w, 3) or not xyz.flags.c_contiguous:
        raise TypeError("expecting a C-contiguous float64 array of shape (%d, %d, 3)" % (h, w))


def install():
    import s2p.triangulation as original
    if not isinstance(original.lib, _LibAdapter):
        original.lib = _LibAdapter(original.lib)
    if hasattr(original, "disp_to_xyz"):
        if not hasattr(original, "_s2pb_original_disp_to_xyz"):
            original._s2pb_original_disp_to_xyz = original.disp_to_xyz
        original.disp_to_xyz = disp_to_xyz
    if hasattr(original, "height_map"):
        if not hasattr(original, "_s2pb_original_height_map"):
            original._s2pb_original_height_map = original.height_map
        original.height_map = height_map
    if hasattr(original, "height_map_to_xyz"):
        if not hasattr(original, "_s2pb_original_height_map_to_xyz"):
            original._s2pb_original_height_map_to_xyz = original.height_map_to_xyz
        original.height_map_to_xyz = height_map_to_xyz
    return original
