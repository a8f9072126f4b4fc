"""Drop-in for the native half of ``s2p.triangulation.disp_to_xyz`` (SURVEY.md section 8f rank 2).

The reference triangulates through ``lib/disp_to_h.so`` loaded with ctypes (s2p/triangulation.py:18-20) and calls
``lib.disp_to_lonlatalt(lonlatalt, err, dispx, dispy, msk, w, h, msk_orig, ww, hh, H1, H2, byref(rpc1),
byref(rpc2), bbx)`` (:134-143).  ``s2pb_disp_to_lonlatalt`` takes the same argument list (plus the context) and
``RPCStruct`` below has the layout of the reference's ``struct rpc`` / ``RPCStruct``; ``install()`` swaps the
library handle of an importable ``s2p.triangulation`` for an adapter that forwards the very same call.

The 3D outlier filter of the same library, ``count_3d_neighbors`` and ``remove_isolated_3d_points`` (c/disp_to_h.c:143-230),
which ``filter_xyz`` runs on the cloud of a tile (s2p/triangulation.py:275-343), goes through the adapter too.
"""
import ctypes
from ctypes import c_double

import numpy as np

from . import _lib
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
    eng = engine or get_engine()
    dispx = np.ascontiguousarray(disp, np.float32)
    h, w = dispx.shape
    dy = np.zeros((h, w), np.float32) if dispy is None else np.ascontiguousarray(dispy, np.float32)
    msk = np.ascontiguousarray(mask_rect, np.float32)
    mo = np.ascontiguousarray(mask_orig, np.float32)
    hh, ww = mo.shape
    out = np.zeros((h, w, 3), np.float64)
    err = np.zeros((h, w), np.float32)
    fp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
    dp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    Ha = np.ascontiguousarray(np.asarray(H1, np.float64).reshape(9))
    Hb = np.ascontiguousarray(np.asarray(H2, np.float64).reshape(9))
    bb = np.ascontiguousarray(np.asarray(img_bbx, np.float32).reshape(4))
    L = _lib.lib()
    _lib.check(L.s2pb_disp_to_lonlatalt(eng._ctx, dp(out), fp(err), fp(dispx), fp(dy), fp(msk), w, h, fp(mo), ww, hh,
                                        dp(Ha), dp(Hb), ctypes.cast(ctypes.pointer(rpc1), ctypes.c_void_p),
                                        ctypes.cast(ctypes.pointer(rpc2), ctypes.c_void_p), fp(bb)))
    return out, err


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
    return original
