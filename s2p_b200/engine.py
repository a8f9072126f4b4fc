"""numpy-level handle on the H100 stereo engine (one context per process and GPU).

``Engine.mgm`` is the in-memory equivalent of what s2p obtains from the `mgm`
subprocess plus ``create_rejection_mask`` (s2p/block_matching.py:18-32,155-188):
rectified pair in, (disparity, consensus confidence, rejection mask) out.
CUDA is initialised lazily in the calling process, so a forked
``multiprocessing`` worker (s2p/parallel.py:80) creates its own context.
"""
import ctypes
import operator
import os

import numpy as np

from . import _lib
from ._lib import MgmParams, S2pbError, SgbmParams  # noqa: F401  (re-exported)


def default_params(algo="mgm", **overrides):
    """What s2p sets for ``algo`` ('mgm', 'mgm_multi', 'mgm_multi_lsd'), then the overrides; ``cost`` may be the
    reference's ``-t`` name ('census', 'ad', 'sd', 'ncc', 'btad', 'btsd') or its S2PB_COST_* index."""
    p = MgmParams()
    _lib.check(_lib.lib().s2pb_default_params(algo.encode(), ctypes.byref(p)))
    for k, v in overrides.items():
        if not hasattr(p, k):
            raise TypeError("unknown matcher parameter %r" % k)
        if k == "cost" and isinstance(v, str):
            if v not in _lib.COSTS:
                raise ValueError("unknown distance %r (one of %s)" % (v, ", ".join(_lib.COSTS)))
            v = _lib.COSTS.index(v)
        setattr(p, k, v)
    return p


def census_window_served(win):
    """Whether the device matcher serves CENSUS_NCC_WIN = ``win`` (s2p's ``census_ncc_win``): 2 to 11, windows of side 3 to 11.
    The reference takes win / 2 as the radius of any win; win <= 1 gives codes of no bit (every cost 0 / 0) and from 12 on the
    popcount no longer fits the 8-bit cost codes, so those windows go to the reference's own binaries."""
    return 2 <= int(win) <= 11


def device_count():
    return _lib.lib().s2pb_device_count()


def workspace_bytes(w, h, nlabels, ndir=8, cost_bytes=1, folded=False):
    """Bytes of one workspace for a w x h tile whose slab holds ``nlabels`` labels, in the resident or the folded layout
    (s2pb_workspace_bytes; no device needed).  ``cost_bytes``: 1 for census codes, 4 for the other distances or the weights."""
    r = _lib.lib().s2pb_workspace_bytes(int(w), int(h), int(nlabels), int(ndir), int(cost_bytes), int(bool(folded)))
    _lib.check(int(r) if r < 0 else 0)
    return int(r)


def workspace_layout(w, h, nlabels, ndir=8, cost_bytes=1, limit=0):
    """'resident' or 'folded': the layout a workspace limit of ``limit`` bytes (0: none) selects for that tile; raises S2pbError
    (S2PB_ERR_NOMEM) when neither fits (s2pb_workspace_layout)."""
    r = _lib.lib().s2pb_workspace_layout(int(w), int(h), int(nlabels), int(ndir), int(cost_bytes), int(limit))
    _lib.check(r if r < 0 else 0)
    return "folded" if r == 1 else "resident"


def dct_coefficients(kind, n, rows, cols):
    """The engine's DCT coefficient table ``kind`` (0 REDFT10, 1 REDFT01, 2 RODFT01) for rows of n pixels, on the row range
    ``rows`` and the column range ``cols`` (Python ranges of step 1), float64 (s2pb_dct_coefficients; no device needed)."""
    out = np.empty((len(rows), len(cols)), np.float64)
    r0 = rows.start if len(rows) else 0
    c0 = cols.start if len(cols) else 0
    _lib.check(_lib.lib().s2pb_dct_coefficients(int(kind), int(n), int(r0), len(rows), int(c0), len(cols),
                                                out.ctypes.data_as(ctypes.POINTER(ctypes.c_double))))
    return out


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _fp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))


def _dp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))


def _u8(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8))


def _ip(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))


def _mat3(H):
    """a 3x3 matrix as 9 contiguous float64 (the pointer keeps its array alive)"""
    return _dp(np.ascontiguousarray(np.asarray(H, np.float64).reshape(9)))


def _rpc(rpc):
    """a ctypes structure with the layout of ``triangulation.RPCStruct``, as the ``const s2pb_rpc *`` of the C ABI"""
    return ctypes.cast(ctypes.pointer(rpc), ctypes.c_void_p)


def _projection(proj):
    """projection.Projection (any object with its fields) as the ``s2pb_projection`` of the C ABI"""
    return _lib.Projection(*(getattr(proj, name) for name, _ in _lib.Projection._fields_))


class Engine:
    def __init__(self, device=0):
        L = _lib.lib()
        self._L = L
        self._ctx = L.s2pb_create(int(device))
        if not self._ctx:
            raise S2pbError(_lib.ERR_CUDA, L.s2pb_last_error().decode("utf-8", "replace"))
        self.device = int(device)

    def close(self):
        if getattr(self, "_ctx", None):
            self._L.s2pb_destroy(self._ctx)
            self._ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    # ------------------------------------------------------------------ matcher
    def mgm(self, im1, im2, dmin, dmax, params=None, want_mask=True, want_right=False, weights=None, want_pkr=False):
        """-> dict(disp, conf, mask[, disp_right][, pkr_left, pkr_right]) for one rectified pair (host arrays).
        ``weights`` = (wl, wr): the regularity weight images of ``-wl`` / ``-wr`` (mgm_multi_lsd).
        ``want_pkr``: also the peak-ratio confidence images of ``-confidence_pkrL`` / ``-confidence_pkrR``."""
        p = params or default_params("mgm")
        im1, im2 = _f32(im1), _f32(im2)
        if im1.shape != im2.shape or im1.ndim != 2:
            raise ValueError("im1 and im2 must be 2-D arrays of the same shape")
        h, w = im1.shape
        wl = wr = None
        if weights is not None:
            wl, wr = _f32(weights[0]), _f32(weights[1])
            if wl.shape != im1.shape or wr.shape != im1.shape:
                raise ValueError("the weight images must have the shape of the rectified images")
        disp = np.empty((h, w), np.float32)
        conf = np.empty((h, w), np.float32)
        mask = np.empty((h, w), np.uint8) if want_mask else None
        right = np.empty((h, w), np.float32) if want_right else None
        if want_pkr:
            if weights is not None:
                raise NotImplementedError("PKR images with regularity weights")
            pl, pr = np.empty((h, w), np.float32), np.empty((h, w), np.float32)
            _lib.check(self._L.s2pb_mgm_pkr(
                self._ctx, _fp(im1), _fp(im2), w, h, int(dmin), int(dmax), ctypes.byref(p), _fp(disp), _fp(conf),
                _u8(mask) if want_mask else None, _fp(right) if want_right else None, _fp(pl), _fp(pr)))
            out = dict(disp=disp, conf=conf, mask=mask, pkr_left=pl, pkr_right=pr)
            if want_right:
                out["disp_right"] = right
            return out
        _lib.check(self._L.s2pb_mgm_weighted(
            self._ctx, _fp(im1), _fp(im2), w, h, int(dmin), int(dmax), ctypes.byref(p),
            _fp(wl) if wl is not None else None, _fp(wr) if wr is not None else None, _fp(disp), _fp(conf),
            _u8(mask) if want_mask else None, _fp(right) if want_right else None))
        out = dict(disp=disp, conf=conf, mask=mask)
        if want_right:
            out["disp_right"] = right
        return out

    # ------------------------------------------------------------------ sgbm
    @staticmethod
    def sgbm_params(**overrides):
        """What s2p passes to the `sgbm` binary (win 3, P1 8, P2 32, lr_diff 1), then the overrides."""
        p = SgbmParams()
        _lib.check(_lib.lib().s2pb_sgbm_default_params(ctypes.byref(p)))
        for k, v in overrides.items():
            if not hasattr(p, k):
                raise TypeError("unknown sgbm parameter %r" % k)
            setattr(p, k, int(v))
        return p

    def sgbm(self, im1, im2, dmin, dmax, params=None, want_mask=True):
        """-> dict(disp, mask): what `sgbm im1 im2 disp cost dmin dmax win P1 P2 lr` writes (NaN = rejected), then
        create_rejection_mask on the float inputs (mask None when ``want_mask`` is false).  No confidence image."""
        p = params or self.sgbm_params()
        im1, im2 = _f32(im1), _f32(im2)
        if im1.shape != im2.shape or im1.ndim != 2:
            raise ValueError("im1 and im2 must be 2-D arrays of the same shape")
        h, w = im1.shape
        disp = np.empty((h, w), np.float32)
        mask = np.empty((h, w), np.uint8) if want_mask else None
        _lib.check(self._L.s2pb_sgbm(self._ctx, _fp(im1), _fp(im2), w, h, int(dmin), int(dmax), ctypes.byref(p), _fp(disp),
                                     _u8(mask) if want_mask else None))
        return dict(disp=disp, mask=mask)

    def mgm_batch(self, refs, secs, dmin, dmax, params=None, want_mask=True, out=None):
        """n same-shaped pairs pipelined over the context's workspaces (s2pb_reserve first for overlap).
        ``out`` = optional (disp, conf, mask) lists of preallocated C-contiguous arrays.  Page-locked arrays (e.g.
        numpy views of torch pinned tensors), on either side, are DMA'd directly instead of being staged."""
        p = params or default_params("mgm")
        n = len(refs)
        refs = [_f32(a) for a in refs]
        secs = [_f32(a) for a in secs]
        h, w = refs[0].shape
        if out is not None:
            disp, conf, mask = out
            want_mask = mask is not None
            for xs, dt in ((disp, np.float32), (conf, np.float32)) + (((mask, np.uint8),) if want_mask else ()):
                if len(xs) != n or any(x.shape != (h, w) or x.dtype != dt or not x.flags.c_contiguous for x in xs):
                    raise ValueError("out arrays must be %d C-contiguous (h, w) arrays of %s" % (n, np.dtype(dt).name))
        else:
            disp = [np.empty((h, w), np.float32) for _ in range(n)]
            conf = [np.empty((h, w), np.float32) for _ in range(n)]
            mask = [np.empty((h, w), np.uint8) for _ in range(n)] if want_mask else None
        arr = lambda xs: (ctypes.c_void_p * n)(*[x.ctypes.data for x in xs])
        _lib.check(self._L.s2pb_mgm_batch(self._ctx, n, arr(refs), arr(secs), w, h, int(dmin), int(dmax), ctypes.byref(p),
                                          arr(disp), arr(conf), arr(mask) if want_mask else None))
        return disp, conf, mask

    def mgm_device(self, slot, d_im1, d_im2, w, h, dmin, dmax, params, d_disp, d_conf=0, d_mask=0, d_right=0,
                   nodata_hint=-1, stream=0):
        """Device pointers in and out (integers, e.g. torch ``tensor.data_ptr()``); asynchronous on the slot's
        stream (or ``stream``).  nodata_hint: 0 = no NaN in the images, 2 = the secondary image may hold NaN,
        -1 = let the library look (one stream synchronisation)."""
        _lib.check(self._L.s2pb_mgm_device(self._ctx, int(slot), d_im1, d_im2, int(w), int(h), int(dmin), int(dmax),
                                           ctypes.byref(params), d_disp, d_conf or None, d_mask or None, d_right or None,
                                           int(nodata_hint), stream or None))

    def reserve(self, nslots, w, h, nlabels):
        _lib.check(self._L.s2pb_reserve(self._ctx, int(nslots), int(w), int(h), int(nlabels)))

    def sync(self):
        _lib.check(self._L.s2pb_sync(self._ctx))

    def last_timings(self, slot=0):
        ms = (ctypes.c_float * len(_lib.T_NAMES))()
        _lib.check(self._L.s2pb_last_timings(self._ctx, int(slot), ms))
        return dict(zip(_lib.T_NAMES, [float(x) for x in ms]))

    def set_workspace_limit(self, nbytes):
        """Cap each workspace of this engine at ``nbytes`` (0: no cap).  A tile whose resident workspace exceeds the cap runs in the
        folded layout, with the same results (s2pb_set_workspace_limit)."""
        _lib.check(self._L.s2pb_set_workspace_limit(self._ctx, int(nbytes)))

    def set_dct_table_limit(self, nbytes):
        """Keep the DCT tables of rows wider than 8192 px on the device up to ``nbytes`` in all (default 8 GiB, and no more
        than the workspace limit when one is set); wider tables are streamed in panels, with the same results
        (s2pb_set_dct_table_limit)."""
        _lib.check(self._L.s2pb_set_dct_table_limit(self._ctx, int(nbytes)))

    def folded_calls(self):
        """matcher calls (pyramid levels of mgm_multi included) that ran in the folded layout"""
        return int(self._L.s2pb_folded_calls(self._ctx))

    def kernel_launches(self):
        return int(self._L.s2pb_kernel_launches(self._ctx))

    # ------------------------------------------------------------------ rectification warp
    def homography(self, src, H, w, h, out=None):
        """out(x) = src(H^-1 x) on [0,w] x [0,h]: what `homography im -h "..." out w h` computes
        (s2p/common.py:159-180), order-5 B-spline with the reference's anti-aliasing rule."""
        src = _f32(src)
        if src.ndim != 2:
            raise ValueError("src must be a 2-D array")
        if out is None:
            out = np.empty((int(h), int(w)), np.float32)
        elif out.shape != (int(h), int(w)) or out.dtype != np.float32 or not out.flags.c_contiguous:
            raise ValueError("out must be a C-contiguous float32 array of shape (h, w)")     # e.g. a page-locked buffer: DMA'd directly
        _lib.check(self._L.s2pb_homography(self._ctx, _fp(src), src.shape[1], src.shape[0], _mat3(H), _fp(out), int(w), int(h)))
        return out

    def rectify_match(self, src1, H1, src2, H2, w, h, dmin, dmax, params=None, want_rect=True, want_right=False):
        """rectify_pair's two warps + compute_disparity_map in one call, the rectified pair staying on the device
        (s2p/__init__.py:147-155,184-190).  -> dict(disp, conf, mask[, rect1, rect2][, disp_right])"""
        src1, src2 = _f32(src1), _f32(src2)
        p = params or default_params("mgm")
        w, h = int(w), int(h)
        out = dict(disp=np.empty((h, w), np.float32), conf=np.empty((h, w), np.float32), mask=np.empty((h, w), np.uint8))
        if want_rect:
            out["rect1"], out["rect2"] = np.empty((h, w), np.float32), np.empty((h, w), np.float32)
        if want_right:
            out["disp_right"] = np.empty((h, w), np.float32)
        nul = ctypes.POINTER(ctypes.c_float)()
        _lib.check(self._L.s2pb_rectify_match(
            self._ctx, _fp(src1), src1.shape[1], src1.shape[0], _mat3(H1), _fp(src2), src2.shape[1], src2.shape[0], _mat3(H2), w, h,
            int(dmin), int(dmax), ctypes.byref(p), _fp(out["rect1"]) if want_rect else nul, _fp(out["rect2"]) if want_rect else nul,
            _fp(out["disp"]), _fp(out["conf"]), _u8(out["mask"]), _fp(out["disp_right"]) if want_right else nul))
        return out

    # ------------------------------------------------------------------ n-view merge
    FUSION_OPS = {"average_if_close": 0, "np.nanmedian": 1, "np.nanmean": 2, "np.nanmin": 3, "np.nanmax": 4,
                  "np.median": 5, "np.mean": 6, "np.min": 7, "np.max": 8, "np.amin": 7, "np.amax": 8}
    FUSE_SUB_F32 = 0x100

    @staticmethod
    def numpy_subtracts_in_float32():
        """How `f.read(1) - offsets[i]` (s2p/fusion.py:49: float32 raster minus the 0-d float64 array np.loadtxt returned)
        is evaluated by the NumPy in this environment: float32 under value-based casting (NumPy < 2), float64 under NEP 50."""
        return (np.zeros(1, np.float32) - np.array(1.5)).dtype == np.float32

    def merge_n(self, rasters, offsets, averaging="average_if_close", threshold=1.0, sub_f32=None):
        """Pixelwise merge of n equally sized rasters (s2p/fusion.py:25-68) -> float32 array.
        sub_f32: subtract the offsets in float32 (NumPy < 2 semantics) or float64; None = what this NumPy does."""
        if averaging.startswith("numpy."):
            averaging = "np." + averaging[6:]
        if averaging not in self.FUSION_OPS:
            raise NotImplementedError("averaging operator %r (supported: %s)" % (averaging, ", ".join(sorted(self.FUSION_OPS))))
        if sub_f32 is None:
            sub_f32 = self.numpy_subtracts_in_float32()
        rs = [_f32(r) for r in rasters]
        n = len(rs)
        h, w = rs[0].shape
        ptrs = (ctypes.c_void_p * n)(*[r.ctypes.data for r in rs])
        offs = (ctypes.c_double * n)(*[float(o) for o in offsets])
        out = np.empty((h, w), np.float32)
        _lib.check(self._L.s2pb_merge_n(self._ctx, ptrs, offs, n, w, h, self.FUSION_OPS[averaging] | (self.FUSE_SUB_F32 if sub_f32 else 0), float(threshold), _fp(out)))
        return out

    def erode_mask(self, mask, radius=2):
        """`morsi diskR erosion` of a 0/1 mask (s2p/masking.py:87-97)."""
        m = np.ascontiguousarray(mask, dtype=np.uint8)
        h, w = m.shape
        out = np.empty_like(m)
        _lib.check(self._L.s2pb_erode_mask(self._ctx, _u8(m), _u8(out), w, h, float(radius)))
        return out

    # ------------------------------------------------------------------ 3D outlier filter of triangulation
    @staticmethod
    def _cloud(xyz):
        """The array the reference's ctypes call receives, np.ascontiguousarray(xyz), with the checks its
        ndpointer(c_double, shape=(h, w, 3)) argument type makes."""
        a = np.ascontiguousarray(xyz)
        if a.ndim != 3 or a.shape[2] != 3:
            raise ValueError("expecting a 3-channels image with shape (h, w, 3), got shape %s" % (a.shape,))
        if a.dtype != np.float64:
            raise TypeError("the point cloud must be float64, got %s" % a.dtype)
        return a

    def count_3d_neighbors(self, xyz, r, p):
        """-> (h, w) int32: per point, the points of its (2p+1)^2 window closer than r (c/disp_to_h.c:152-174).
        r is rounded to float32, as the reference's c_float argument is."""
        a = self._cloud(xyz)
        h, w = a.shape[:2]
        out = np.zeros((h, w), np.int32)
        if a.size:
            _lib.check(self._L.s2pb_count_3d_neighbors(self._ctx, _ip(out), _dp(a), w, h, float(r), operator.index(p)))
        return out

    def remove_isolated_3d_points(self, xyz, r, p, n, q=1):
        """NaN into the isolated points of np.ascontiguousarray(xyz), in place (c/disp_to_h.c:177-230): a C-contiguous
        float64 xyz is itself modified.  -> that array."""
        a = self._cloud(xyz)
        h, w = a.shape[:2]
        if not a.flags.writeable:
            raise ValueError("the point cloud is read-only")
        if a.size:
            _lib.check(self._L.s2pb_remove_isolated_3d_points(self._ctx, _dp(a), w, h, float(r), operator.index(p),
                                                               operator.index(n), operator.index(q)))
        return a

    # ------------------------------------------------------------------ triangulation into output coordinates
    @staticmethod
    def _triangulation(disp, mask_rect, mask_orig, H1, H2, rpc1, rpc2, img_bbx, zone, south, dispy):
        """-> (h, w) of the rectified map and s2pb_disp_to_xyz's arguments from dispx to south, checked and converted"""
        dispx, msk, mo = _f32(disp), _f32(mask_rect), _f32(mask_orig)
        if dispx.ndim != 2 or msk.shape != dispx.shape or mo.ndim != 2:
            raise ValueError("disp and mask_rect must be 2-D arrays of the same shape, and mask_orig a 2-D array")
        h, w = dispx.shape
        dy = np.zeros((h, w), np.float32) if dispy is None else _f32(dispy)
        if dy.shape != dispx.shape:
            raise ValueError("dispy must have the shape of disp")
        bb = np.ascontiguousarray(np.asarray(img_bbx, np.float32).reshape(4))
        return (h, w), (_fp(dispx), _fp(dy), _fp(msk), w, h, _fp(mo), mo.shape[1], mo.shape[0], _mat3(H1), _mat3(H2), _rpc(rpc1),
                        _rpc(rpc2), _fp(bb), int(zone), int(bool(south)))

    @staticmethod
    def _localisation(heights, rpc, off_x, off_y, zone, south):
        """-> (h, w) of the height map and s2pb_height_map_to_xyz's arguments from heights to south, checked and converted"""
        z = np.ascontiguousarray(heights, np.float64)
        if z.ndim != 2:
            raise ValueError("expecting a 2-D height map, got shape %s" % (z.shape,))
        h, w = z.shape
        return (h, w), (_dp(z), w, h, _rpc(rpc), float(off_x), float(off_y), int(zone), int(bool(south)))

    def disp_to_xyz(self, disp, mask_rect, mask_orig, H1, H2, rpc1, rpc2, img_bbx, zone=0, south=False, dispy=None):
        """disp_to_lonlatalt and the projection to UTM zone `zone` (1..60; 0: lon, lat, alt as they are; with _lib.ZONE_EGM96
        OR'ed in, heights above the geoid of set_geoid) in one device call
        -> (xyz (h, w, 3) float64, err (h, w) float32).  rpc1 / rpc2: ctypes structures with the layout of
        ``triangulation.RPCStruct``; H2 already carries the pointing correction."""
        (h, w), args = self._triangulation(disp, mask_rect, mask_orig, H1, H2, rpc1, rpc2, img_bbx, zone, south, dispy)
        xyz = np.empty((h, w, 3), np.float64)
        err = np.empty((h, w), np.float32)
        _lib.check(self._L.s2pb_disp_to_xyz(self._ctx, _dp(xyz), _fp(err), *args))
        return xyz, err

    def set_geoid(self, grid):
        """Hold ``grid`` (projection.GeoidGrid, or None to drop it) on the device for the zones with _lib.ZONE_EGM96 OR'ed in,
        which every cloud, tile and projection method then takes: heights above the geoid, z - N(lon, lat) (s2pb_set_geoid).
        Uploads only when the grid is not the one the engine already holds."""
        if grid is getattr(self, "_geoid", None):
            return
        if grid is None:
            _lib.check(self._L.s2pb_set_geoid(self._ctx, None, 0, 0, 0.0, 0.0, 0.0, 0.0))
        else:
            v = _f32(grid.values)
            if v.ndim != 2:
                raise ValueError("the geoid grid must be a 2-D array")
            _lib.check(self._L.s2pb_set_geoid(self._ctx, _fp(v), v.shape[1], v.shape[0], float(grid.lon0), float(grid.lat0),
                                              float(grid.dlon), float(grid.dlat)))
        self._geoid = grid

    def set_projection(self, proj):
        """Hold ``proj`` (projection.Projection, or None to drop it) on the context for the zone _lib.ZONE_PROJ, which every
        cloud and tile method then takes: the map of that projection instead of a UTM zone (s2pb_set_projection)."""
        if proj == getattr(self, "_projection", None):
            return
        _lib.check(self._L.s2pb_set_projection(self._ctx, None if proj is None else ctypes.byref(_projection(proj))))
        self._projection = proj

    def lonlat_to_proj(self, lonlatalt, proj):
        """(..., 3) float64 (lon, lat in degrees, alt) -> (..., 3) float64 (x, y, alt) in the map ``proj``
        (projection.Projection; s2pb_lonlat_to_proj).  NaN in any coordinate gives NaN in all three, a point the map cannot
        project +inf in all three."""
        a = np.ascontiguousarray(lonlatalt, np.float64)
        if a.ndim < 1 or a.shape[-1] != 3:
            raise ValueError("expecting points of three coordinates, got shape %s" % (a.shape,))
        out = np.empty_like(a)
        _lib.check(self._L.s2pb_lonlat_to_proj(self._ctx, _dp(out), _dp(a), a.size // 3, ctypes.byref(_projection(proj))))
        return out

    def lonlat_to_utm(self, lonlatalt, zone, south=False):
        """(..., 3) float64 (lon, lat in degrees, alt) -> (..., 3) float64 (easting, northing, alt) in UTM zone `zone` (1..60)
        of WGS84, north or south (EPSG 326zz / 327zz); with _lib.ZONE_EGM96 OR'ed into the zone, alt - N(lon, lat) in the geoid
        of set_geoid.  NaN in any coordinate gives NaN in all three."""
        a = np.ascontiguousarray(lonlatalt, np.float64)
        if a.ndim < 1 or a.shape[-1] != 3:
            raise ValueError("expecting points of three coordinates, got shape %s" % (a.shape,))
        out = np.empty_like(a)
        _lib.check(self._L.s2pb_lonlat_to_utm(self._ctx, _dp(out), _dp(a), a.size // 3, int(zone), int(bool(south))))
        return out

    def height_map_to_xyz(self, heights, rpc, off_x, off_y, zone=0, south=False):
        """The localisation of every pixel of a (h, w) height map and the projection to UTM zone `zone` (1..60; 0: lon, lat,
        alt as they are; _lib.ZONE_EGM96 as in disp_to_xyz) in one device call -> (h, w, 3) float64.  Pixel (i, j) is image pixel (j + off_x, i + off_y) of the
        camera ``rpc`` (a ctypes structure with the layout of ``triangulation.RPCStruct``); its third coordinate is the height
        converted to float64.  NaN heights give NaN in all three.  Pixels whose localisation does not converge raise
        S2pbError(ERR_ARG)."""
        (h, w), args = self._localisation(heights, rpc, off_x, off_y, zone, south)
        xyz = np.empty((h, w, 3), np.float64)
        _lib.check(self._L.s2pb_height_map_to_xyz(self._ctx, _dp(xyz), *args))
        return xyz

    # ------------------------------------------------------------------ the tile's point cloud as PLY records
    # numpy colour types -> S2PB_PLY_*: the eight plyfile writes
    PLY_COLOR_TYPES = {np.dtype(np.int8): _lib.PLY_I8, np.dtype(np.uint8): _lib.PLY_U8, np.dtype("<i2"): _lib.PLY_I16,
                       np.dtype("<u2"): _lib.PLY_U16, np.dtype("<i4"): _lib.PLY_I32, np.dtype("<u4"): _lib.PLY_U32,
                       np.dtype("<f4"): _lib.PLY_F32, np.dtype("<f8"): _lib.PLY_F64}

    @staticmethod
    def ply_dtype(nbands=3, confidence=False, color_dtype=np.uint8):
        """The packed record write_to_ply writes: x, y, z float64, red, green, blue (and ir with 4 bands) of color_dtype
        (little-endian) when there are colours (1, 3 or 4 bands), confidence float32 when asked."""
        d = [("x", "<f8"), ("y", "<f8"), ("z", "<f8")]
        if nbands:
            c = np.dtype(color_dtype).newbyteorder("<")
            d += [("red", c), ("green", c), ("blue", c)] + ([("ir", c)] if nbands == 4 else [])
        if confidence:
            d += [("confidence", "<f4")]
        return np.dtype(d)

    @classmethod
    def _typed(cls, colors, shape):
        """(nbands, h, w) or (h, w) colour planes of one of the eight PLY types -> C-contiguous little-endian (nbands, h, w)
        planes, nbands and their S2PB_PLY_* type"""
        c = np.asarray(colors)
        c = c[None] if c.ndim == 2 else c
        if c.ndim != 3 or c.shape[1:] != tuple(shape):
            raise ValueError("expecting colour planes of shape (nbands, %d, %d), got %s" % (shape[0], shape[1], c.shape))
        dt = c.dtype.newbyteorder("<")
        if dt not in cls.PLY_COLOR_TYPES:
            raise TypeError("PLY colours must be one of int8, uint8, int16, uint16, int32, uint32, float32, float64; got %s" % c.dtype)
        return np.ascontiguousarray(c, dt), c.shape[0], cls.PLY_COLOR_TYPES[dt]

    @staticmethod
    def _bands(colors, shape):
        """(nbands, h, w) or (h, w) colour planes -> C-contiguous (nbands, h, w) float32 and nbands (0 for None)"""
        if colors is None:
            return None, 0
        c = np.asarray(colors)
        c = c[None] if c.ndim == 2 else c
        if c.ndim != 3 or c.shape[1:] != tuple(shape):
            raise ValueError("expecting colour planes of shape (nbands, %d, %d), got %s" % (shape[0], shape[1], c.shape))
        return np.ascontiguousarray(c, np.float32), c.shape[0]

    def _records(self, call, npix, nbands, confidence, color_dtype=np.uint8):
        dt = self.ply_dtype(nbands, confidence, color_dtype)
        buf = np.empty(npix * dt.itemsize, np.uint8)
        n = ctypes.c_int64(0)
        _lib.check(call(_u8(buf), ctypes.byref(n)))
        return np.frombuffer(buf[:n.value * dt.itemsize].tobytes(), dt)

    def stretch_8bit(self, img, p=1):
        """common.linear_stretching_and_quantization_8bit(img, p) bit for bit (NumPy >= 2) on the device: the
        percentiles run over every value of img together -> uint8 of img's shape.  img must convert to float32 exactly."""
        a = np.ascontiguousarray(img, np.float32)
        out = np.empty(a.shape, np.uint8)
        _lib.check(self._L.s2pb_stretch_8bit(self._ctx, _fp(a), a.size, float(p), _u8(out)))
        return out

    def ply_records(self, xyz, colors=None, confidence=None):
        """The vertex records write_to_ply writes for the cloud xyz (..., 3) float64: its points with three finite coordinates,
        in order, with the uint8 colours (nbands, ...) and the float32 confidence (...) of those points -> structured array of
        ply_dtype(nbands, confidence is not None)."""
        a = np.ascontiguousarray(xyz, np.float64)
        if a.ndim < 1 or a.shape[-1] != 3:
            raise ValueError("expecting points of three coordinates, got shape %s" % (a.shape,))
        n = a.size // 3
        nb, col = 0, None
        if colors is not None:
            col = np.ascontiguousarray(colors, np.uint8).reshape(-1, n) if n else np.zeros((np.shape(colors)[0], 0), np.uint8)
            nb = col.shape[0]
        conf = None if confidence is None else np.ascontiguousarray(confidence, np.float32).reshape(n)
        call = lambda out, cnt: self._L.s2pb_ply_records(self._ctx, _dp(a), n, _u8(col) if nb else None, nb,
                                                         _fp(conf) if conf is not None else None, out, cnt)
        return self._records(call, n, nb, conf is not None)

    def disp_to_ply(self, disp, mask_rect, mask_orig, H1, H2, rpc1, rpc2, img_bbx, zone=0, south=False, r=0.0, p=0, n=0,
                    colors=None, stretch_p=1, confidence=None, dispy=None):
        """disp_to_xyz, the 3D filter (remove_isolated_3d_points(r, p, n, q=1); off when r == 0 or n == 0), the 8-bit stretch of
        the colour planes (nbands, h, w) and the records of ply_records in one device call -> structured array."""
        (h, w), args = self._triangulation(disp, mask_rect, mask_orig, H1, H2, rpc1, rpc2, img_bbx, zone, south, dispy)
        bands, nb = self._bands(colors, (h, w))
        conf = None if confidence is None else _f32(confidence).reshape(h, w)
        call = lambda out, cnt: self._L.s2pb_disp_to_ply(
            self._ctx, *args, float(r), operator.index(p), operator.index(n), _fp(bands) if nb else None, nb, float(stretch_p),
            _fp(conf) if conf is not None else None, out, cnt)
        return self._records(call, h * w, nb, conf is not None)

    def height_map_to_ply(self, heights, rpc, off_x, off_y, zone=0, south=False, r=0.0, p=0, n=0, colors=None, stretch_p=1):
        """height_map_to_xyz, the 3D filter, the 8-bit stretch of the colour planes and the records of ply_records in one device
        call -> structured array (no confidence)."""
        (h, w), args = self._localisation(heights, rpc, off_x, off_y, zone, south)
        bands, nb = self._bands(colors, (h, w))
        call = lambda out, cnt: self._L.s2pb_height_map_to_ply(
            self._ctx, *args, float(r), operator.index(p), operator.index(n), _fp(bands) if nb else None, nb, float(stretch_p),
            out, cnt)
        return self._records(call, h * w, nb, False)

    def ply_records_typed(self, xyz, colors=None, confidence=None):
        """ply_records with colours of any of the eight PLY types, copied as they are: colors (nbands, ...) keeps its dtype in
        the records (a clr image's own type, as write_to_ply writes it) -> structured array of
        ply_dtype(nbands, confidence is not None, colors.dtype)."""
        a = np.ascontiguousarray(xyz, np.float64)
        if a.ndim < 1 or a.shape[-1] != 3:
            raise ValueError("expecting points of three coordinates, got shape %s" % (a.shape,))
        n = a.size // 3
        nb, col, ptype, cdt = 0, None, _lib.PLY_U8, np.uint8
        if colors is not None:
            c = np.asarray(colors)
            col, nb, ptype = self._typed(c.reshape(c.shape[0], 1, n), (1, n))
            cdt = col.dtype
        conf = None if confidence is None else np.ascontiguousarray(confidence, np.float32).reshape(n)
        call = lambda out, cnt: self._L.s2pb_ply_records_typed(self._ctx, _dp(a), n, col.ctypes.data if nb else None, nb, ptype,
                                                               _fp(conf) if conf is not None else None, out, cnt)
        return self._records(call, n, nb, conf is not None, cdt)

    def disp_to_ply_clr(self, disp, mask_rect, mask_orig, H1, H2, rpc1, rpc2, img_bbx, zone=0, south=False, r=0.0, p=0, n=0,
                        clr=None, hc=None, confidence=None, dispy=None):
        """disp_to_ply with the colours of a clr image: clr (nbands, ch, cw) is the crop of that image which the warp of the
        rectified reference needs, hc the reference's homography with the crop's origin folded in (common.homography_crop).
        Every band is warped onto the disparity's grid on the device as homography(band, hc, w, h) warps it, and the records
        get float32 colours -> structured array of ply_dtype(nbands, confidence is not None, np.float32)."""
        (h, w), args = self._triangulation(disp, mask_rect, mask_orig, H1, H2, rpc1, rpc2, img_bbx, zone, south, dispy)
        c = _f32(clr)
        c = c[None] if c.ndim == 2 else c
        if c.ndim != 3:
            raise ValueError("expecting clr planes of shape (nbands, ch, cw), got %s" % (c.shape,))
        nb, ch, cw = c.shape
        conf = None if confidence is None else _f32(confidence).reshape(h, w)
        call = lambda out, cnt: self._L.s2pb_disp_to_ply_clr(
            self._ctx, *args, float(r), operator.index(p), operator.index(n), _fp(c), cw, ch, nb, _mat3(hc),
            _fp(conf) if conf is not None else None, out, cnt)
        return self._records(call, h * w, nb, conf is not None, np.float32)

    PAIR_TILE_OUTPUTS = ("rect1", "rect2", "disp", "conf", "mask", "disp_right")

    @staticmethod
    def _pair_tile(src1, H1, src2, H2, w, h, dmin, dmax, mask_orig, H_ref, H_sec, rpc1, rpc2, params, weights, erode_radius, want):
        """-> (PairTile with the fields of the warps, the matcher, the erosion, msk_orig, the cameras, ha and hb filled; the arrays
        its pointers refer to)"""
        src1, src2, mo = _f32(src1), _f32(src2), _f32(mask_orig)
        if src1.ndim != 2 or src2.ndim != 2 or mo.ndim != 2:
            raise ValueError("src1, src2 and mask_orig must be 2-D arrays")
        unknown = set(want) - set(Engine.PAIR_TILE_OUTPUTS)
        if unknown:
            raise ValueError("unknown outputs %s (one of %s)" % (sorted(unknown), ", ".join(Engine.PAIR_TILE_OUTPUTS)))
        keep = [src1, src2, mo]
        t = _lib.PairTile()
        t.src1, t.sw1, t.sh1, t.src2, t.sw2, t.sh2 = _fp(src1), src1.shape[1], src1.shape[0], _fp(src2), src2.shape[1], src2.shape[0]
        t.w, t.h, t.dmin, t.dmax = w, h, int(dmin), int(dmax)
        params = params if params is not None else default_params("mgm")
        if isinstance(params, SgbmParams):
            t.matcher, t.sgbm = _lib.MATCHER_SGBM, params
        else:
            t.matcher, t.mgm = _lib.MATCHER_MGM, params
        if weights is not None:
            wl, wr = _f32(weights[0]), _f32(weights[1])
            if wl.shape != (h, w) or wr.shape != (h, w):
                raise ValueError("the weight images must have the shape of the rectified images")
            t.wl, t.wr = _fp(wl), _fp(wr)
            keep += [wl, wr]
        t.erode_radius = float(erode_radius)
        t.msk_orig, t.mw, t.mh = _fp(mo), mo.shape[1], mo.shape[0]
        t.rpc1, t.rpc2 = _rpc(rpc1), _rpc(rpc2)
        for name, H in (("H1", H1), ("H2", H2), ("ha", H_ref), ("hb", H_sec)):
            getattr(t, name)[:] = [float(v) for v in np.asarray(H, np.float64).reshape(9)]
        return t, keep

    def _pair_outputs(self, want, h, w):
        """the host arrays of the intermediates named in ``want`` and the pointer arguments from rect1 to disp_right"""
        out = {k: np.empty((h, w), np.uint8 if k == "mask" else np.float32) for k in self.PAIR_TILE_OUTPUTS if k in want}
        ptr = lambda k, conv: conv(out[k]) if k in out else None
        return out, (ptr("rect1", _fp), ptr("rect2", _fp), ptr("disp", _fp), ptr("conf", _fp), ptr("mask", _u8), ptr("disp_right", _fp))

    PAIR_TILE_OUTPUTS = ("rect1", "rect2", "disp", "conf", "mask", "disp_right")

    def pair_tile_to_ply(self, src1, H1, src2, H2, w, h, dmin, dmax, mask_orig, H_ref, H_sec, rpc1, rpc2, img_bbx, zone=0, south=False,
                         params=None, weights=None, erode_radius=0, r=0.0, p=0, n=0, stretch_p=1, clr=None, hc=None,
                         confidence=False, want=()):
        """A two-view tile from its source crops to its cloud's records in one device call (s2pb_pair_tile_to_ply): homography
        of src1 by H1 and of src2 by H2 onto w x h, the matcher (``params``: MgmParams, or SgbmParams for sgbm; ``weights`` =
        (wl, wr) for mgm_multi_lsd) on [dmin, dmax], the erosion of its mask (erode_radius 0: none), then disp_to_ply on the
        disparity and the eroded mask (H_ref, H_sec: the triangulation's homographies, H_sec with the pointing correction)
        coloured by the stretch of the rectified reference, or by the clr crop (nbands, ch, cw) warped by hc, with the
        confidence column when ``confidence``.  -> (records, dict of the intermediates named in ``want``, a subset of
        PAIR_TILE_OUTPUTS)."""
        w, h = int(w), int(h)
        t, keep = self._pair_tile(src1, H1, src2, H2, w, h, dmin, dmax, mask_orig, H_ref, H_sec, rpc1, rpc2, params, weights,
                                  erode_radius, want)
        t.bbox[:] = [float(v) for v in np.asarray(img_bbx, np.float32).reshape(4)]
        t.zone, t.south = int(zone), int(bool(south))
        t.r, t.p, t.n, t.pct = float(r), operator.index(p), operator.index(n), float(stretch_p)
        nb, cdt = 1, np.uint8
        if clr is not None:
            c = _f32(clr)
            c = c[None] if c.ndim == 2 else c
            if c.ndim != 3:
                raise ValueError("expecting clr planes of shape (nbands, ch, cw), got %s" % (c.shape,))
            nb, cdt = c.shape[0], np.float32
            t.clr, t.clr_bands, t.ch, t.cw = _fp(c), c.shape[0], c.shape[1], c.shape[2]
            t.hc[:] = [float(v) for v in np.asarray(hc, np.float64).reshape(9)]
        t.with_conf = int(bool(confidence))
        out, ptrs = self._pair_outputs(want, h, w)
        call = lambda rec, cnt: self._L.s2pb_pair_tile_to_ply(self._ctx, ctypes.byref(t), rec, cnt, *ptrs)
        records = self._records(call, h * w, nb, bool(confidence), cdt)
        return records, out

    def pair_tile_to_height_map(self, src1, H1, src2, H2, w, h, dmin, dmax, mask_orig, H_ref, H_sec, rpc1, rpc2, tile, params=None,
                                weights=None, erode_radius=0, want=()):
        """One pair of a tri-stereo tile from its source crops to its height map in one device call
        (s2pb_pair_tile_to_height_map): the warps, the matcher and the erosion of pair_tile_to_ply, then height_map on the
        disparity and the eroded mask for the tile (x, y, tw, th) of the reference image (H_ref: H_ref.txt; H_sec: H_sec.txt
        times the inverse of the pointing correction).  -> ((th, tw) float64 heights, dict of the intermediates named in
        ``want``, a subset of PAIR_TILE_OUTPUTS)."""
        w, h = int(w), int(h)
        x, y, tw, th = (int(v) for v in tile)
        t, keep = self._pair_tile(src1, H1, src2, H2, w, h, dmin, dmax, mask_orig, H_ref, H_sec, rpc1, rpc2, params, weights,
                                  erode_radius, want)
        heights = np.empty((th, tw), np.float64)
        out, ptrs = self._pair_outputs(want, h, w)
        _lib.check(self._L.s2pb_pair_tile_to_height_map(self._ctx, ctypes.byref(t), x, y, tw, th, _dp(heights), *ptrs))
        return heights, out

    HEIGHTS_TILE_OUTPUTS = ("cleaned", "merged")

    def heights_tile_to_ply(self, maps, offsets, rpc, off_x, off_y, zone=0, south=False, cargarse_basura=False,
                            averaging="average_if_close", threshold=1.0, sub_f32=None, r=0.0, p=0, n=0, colors=None, stretch_p=1,
                            clr=None, want=()):
        """A tri-stereo tile from its pairs' height maps to its cloud's records in one device call (s2pb_heights_tile_to_ply):
        with ``cargarse_basura``, each map rounded to float32 and cleaned as cargarse_basura cleans it; then merge_n of the
        maps (the cleaned ones, else as they are: float32 maps as float32, any other type as float64, which every stored
        height type converts to exactly) with ``offsets``, ``averaging`` and ``threshold``; then height_map_to_ply of the merged
        map coloured by the stretch of the float32 planes ``colors`` (as height_map_to_ply) or by the typed planes ``clr`` (as
        height_map_to_ply_clr).  sub_f32: as merge_n.  -> (records, dict of the intermediates named in ``want``: 'cleaned',
        the list of cleaned float32 maps, and 'merged', the merged float32 map)."""
        unknown = set(want) - set(self.HEIGHTS_TILE_OUTPUTS)
        if unknown:
            raise ValueError("unknown outputs %s (one of %s)" % (sorted(unknown), ", ".join(self.HEIGHTS_TILE_OUTPUTS)))
        if "cleaned" in want and not cargarse_basura:
            raise ValueError("the cleaned maps exist with cargarse_basura only")
        if averaging.startswith("numpy."):
            averaging = "np." + averaging[6:]
        if averaging not in self.FUSION_OPS:
            raise NotImplementedError("averaging operator %r (supported: %s)" % (averaging, ", ".join(sorted(self.FUSION_OPS))))
        if sub_f32 is None:
            sub_f32 = self.numpy_subtracts_in_float32()
        maps = [np.asarray(m) for m in maps]
        if not maps or len(maps) != len(offsets):
            raise ValueError("%d maps, %d offsets" % (len(maps), len(offsets)))
        if len(maps) > _lib.MAX_FUSION:
            raise NotImplementedError("at most %d height maps can be merged, got %d" % (_lib.MAX_FUSION, len(maps)))
        if any(m.ndim != 2 or m.shape != maps[0].shape for m in maps):
            raise ValueError("the height maps must be 2-D arrays of the same shape")
        f32 = all(m.dtype == np.float32 for m in maps)
        maps = [np.ascontiguousarray(m, np.float32 if f32 else np.float64) for m in maps]
        h, w = maps[0].shape
        t = _lib.HeightsTile()
        t.n_maps, t.w, t.h, t.map_type = len(maps), w, h, _lib.PLY_F32 if f32 else _lib.PLY_F64
        for k, m in enumerate(maps):
            t.maps[k], t.offsets[k] = m.ctypes.data, float(offsets[k])
        t.cargarse_basura = int(bool(cargarse_basura))
        t.op, t.threshold = self.FUSION_OPS[averaging] | (self.FUSE_SUB_F32 if sub_f32 else 0), float(threshold)
        t.rpc, t.off_x, t.off_y, t.zone, t.south = _rpc(rpc), float(off_x), float(off_y), int(zone), int(bool(south))
        t.r, t.p, t.n = float(r), operator.index(p), operator.index(n)
        if clr is not None:
            if colors is not None:
                raise ValueError("colors (stretched) or clr (typed), not both")
            col, nb, t.color_type = self._typed(clr, (h, w))
            cdt = col.dtype
        else:
            col, nb = self._bands(colors, (h, w))
            cdt, t.stretch, t.pct = np.uint8, 1, float(stretch_p)
        t.colors, t.nbands = (col.ctypes.data if nb else None), nb
        out = {}
        cleaned = None
        if "cleaned" in want:
            out["cleaned"] = [np.empty((h, w), np.float32) for _ in maps]
            cleaned = (_lib._f * len(maps))(*[_fp(c) for c in out["cleaned"]])
        if "merged" in want:
            out["merged"] = np.empty((h, w), np.float32)
        call = lambda rec, cnt: self._L.s2pb_heights_tile_to_ply(self._ctx, ctypes.byref(t), rec, cnt, cleaned,
                                                                 _fp(out["merged"]) if "merged" in out else None)
        records = self._records(call, h * w, nb, False, cdt)
        return records, out

    def height_map_to_ply_clr(self, heights, rpc, off_x, off_y, zone=0, south=False, r=0.0, p=0, n=0, colors=None):
        """height_map_to_ply with the colours of a clr image: the planes (nbands, h, w) keep their dtype (one of the eight PLY
        types) in the records -> structured array of ply_dtype(nbands, False, colors.dtype)."""
        (h, w), args = self._localisation(heights, rpc, off_x, off_y, zone, south)
        col, nb, ptype = self._typed(colors, (h, w))
        call = lambda out, cnt: self._L.s2pb_height_map_to_ply_clr(
            self._ctx, *args, float(r), operator.index(p), operator.index(n), col.ctypes.data, nb, ptype, out, cnt)
        return self._records(call, h * w, nb, False, col.dtype)

    # ------------------------------------------------------------------ DSM rasterisation
    def plyflatten(self, clouds, record_bytes, columns, xoff, yoff, resolution, xsize, ysize):
        """plyflatten with radius 0 and no sigma on the roi (xoff, yoff, xsize, ysize) -> (ysize, xsize, len(columns) - 2)
        float32, NaN where no point fell.  clouds: in order, each the raw vertex records of a binary little-endian PLY as a
        C-contiguous host array of record_bytes-byte records (any dtype), or a (device pointer, npoints) pair.  columns:
        (byte offset, _lib.PLY_* type) of x, y, then of each channel."""
        ptrs, counts, keep = [], [], []
        for c in clouds:
            if isinstance(c, tuple):
                ptr, npts = int(c[0]), operator.index(c[1])
            else:
                a = np.ascontiguousarray(c)
                if a.nbytes % record_bytes:
                    raise ValueError("%d bytes of records are not a whole number of %d-byte records" % (a.nbytes, record_bytes))
                keep.append(a)
                ptr, npts = a.ctypes.data, a.nbytes // record_bytes
            ptrs.append(ptr if npts else None)
            counts.append(npts)
        n = len(ptrs)
        cols = (_lib.PlyColumn * len(columns))(*[_lib.PlyColumn(int(o), int(t)) for o, t in columns])
        out = np.empty((int(ysize), int(xsize), max(len(columns) - 2, 0)), np.float32)
        _lib.check(self._L.s2pb_plyflatten(self._ctx, n, (ctypes.c_void_p * n)(*ptrs), (ctypes.c_int64 * n)(*counts),
                                           int(record_bytes), cols, len(columns), float(xoff), float(yoff), float(resolution),
                                           int(xsize), int(ysize), _fp(out)))
        return out

    # ------------------------------------------------------------------ global DSM
    TILE_STREAM_MAX = 262175        # bytes of a 256 x 256 float32 tile's zlib stream in stored blocks, the longest one

    def mosaic_deflate(self, sources, offsets, W, H, band_rows=0):
        """rasterio.merge(method='first') of the float32 rasters `sources` (2-D host arrays, NaN = nodata) placed at the
        destination (column, row) `offsets` onto a W x H raster, and the zlib streams of its 256 x 256 GeoTIFF tiles after
        PREDICTOR=2 -> (data, sizes): data uint8, the streams back to back in row-major tile order; sizes int32, each stream's
        bytes.  band_rows: tile rows per device band, 0 = automatic."""
        srcs = [np.ascontiguousarray(s, dtype=np.float32) for s in sources]
        if any(s.ndim != 2 for s in srcs):
            raise ValueError("every source must be a 2-D raster")
        if len(offsets) != len(srcs):
            raise ValueError("%d sources, %d offsets" % (len(srcs), len(offsets)))
        n = len(srcs)
        ntiles = -(-int(W) // 256) * -(-int(H) // 256)
        data = np.empty(ntiles * self.TILE_STREAM_MAX, np.uint8)
        sizes = np.empty(ntiles, np.int32)
        ptrs = (ctypes.c_void_p * max(n, 1))(*[s.ctypes.data for s in srcs])
        ws = (ctypes.c_int32 * max(n, 1))(*[s.shape[1] for s in srcs])
        hs = (ctypes.c_int32 * max(n, 1))(*[s.shape[0] for s in srcs])
        cx = (ctypes.c_int64 * max(n, 1))(*[operator.index(o[0]) for o in offsets])
        cy = (ctypes.c_int64 * max(n, 1))(*[operator.index(o[1]) for o in offsets])
        _lib.check(self._L.s2pb_mosaic_deflate(self._ctx, n, ptrs, ws, hs, cx, cy, int(W), int(H), operator.index(band_rows),
                                               _u8(data), data.size, sizes.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))))
        return data[:int(sizes.sum(dtype=np.int64))], sizes

    def deflate_blocks(self, raster, band_rows=0):
        """the tile streams of mosaic_deflate for one (H, W) float32 raster at offset (0, 0) -> (data, sizes)"""
        a = np.ascontiguousarray(raster, dtype=np.float32)
        H, W = a.shape
        ntiles = -(-W // 256) * -(-H // 256)
        data = np.empty(ntiles * self.TILE_STREAM_MAX, np.uint8)
        sizes = np.empty(ntiles, np.int32)
        _lib.check(self._L.s2pb_deflate_blocks(self._ctx, _fp(a), W, H, operator.index(band_rows), _u8(data), data.size,
                                               sizes.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))))
        return data[:int(sizes.sum(dtype=np.int64))], sizes

    # ------------------------------------------------------------------ tri-stereo height maps
    def height_map(self, x, y, w, h, rpc1, rpc2, H1, H2, disp, mask, mask_orig, A=None):
        """s2p.triangulation.height_map on the device -> (h, w) float64 heights on the tile grid.
        rpc1 / rpc2: ctypes structures with the layout of ``triangulation.RPCStruct``.  ``A``: the pointing correction, applied
        on the host as the reference does (H2 <- np.dot(H2, np.linalg.inv(A))) before the call."""
        disp, msk, mo = _f32(disp), _f32(mask), _f32(mask_orig)
        if disp.ndim != 2 or msk.shape != disp.shape or mo.ndim != 2:
            raise ValueError("disp and mask must be 2-D arrays of the same shape, and mask_orig a 2-D array")
        Hb = np.asarray(H2, np.float64).reshape(3, 3)
        if A is not None:
            Hb = np.dot(Hb, np.linalg.inv(np.asarray(A, np.float64).reshape(3, 3)))
        out = np.empty((int(h), int(w)), np.float64)
        ny, nx = disp.shape
        _lib.check(self._L.s2pb_height_map(self._ctx, _dp(out), _fp(disp), _fp(msk), nx, ny, _fp(mo), mo.shape[1], mo.shape[0],
                                           int(x), int(y), int(w), int(h), _mat3(H1), _mat3(Hb), _rpc(rpc1), _rpc(rpc2)))
        return out

    def resample_heights(self, z, H, w, h):
        """The resampling stage of height_map alone: affine_transform(nan_to_num(z).T, H, output_shape=(w, h), order=1).T
        with its NaN restoration, z a float64 map on the rectified grid -> (h, w) float64."""
        z = np.ascontiguousarray(z, np.float64)
        if z.ndim != 2:
            raise ValueError("z must be a 2-D array")
        out = np.empty((int(h), int(w)), np.float64)
        _lib.check(self._L.s2pb_resample_heights(self._ctx, _dp(z), z.shape[1], z.shape[0], _mat3(H), _dp(out), int(w), int(h)))
        return out

    def cargarse_basura(self, img):
        """s2p.common.cargarse_basura on an image -> float32 array.  The image is rounded to float32 first, as the
        reference's tools read it."""
        img = _f32(img)
        if img.ndim != 2:
            raise ValueError("img must be a 2-D array")
        h, w = img.shape
        out = np.empty_like(img)
        _lib.check(self._L.s2pb_cargarse_basura(self._ctx, _fp(img), _fp(out), w, h))
        return out

    # ------------------------------------------------------------------ stages (parity tests)
    def census(self, img, win=5):
        img = _f32(img)
        h, w = img.shape
        out = np.empty((h, w), np.uint64)
        _lib.check(self._L.s2pb_census(self._ctx, _fp(img), w, h, win, out.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64))))
        return out

    def costvolume(self, u, v, lo, hi, gmin, D, win=5, cost=None):
        """cost=None: the census / 8-bit cost path of the hot matcher; otherwise one of _lib.COSTS through the general path."""
        u, v = _f32(u), _f32(v)
        h, w = u.shape
        lo = np.ascontiguousarray(lo, np.int32)
        hi = np.ascontiguousarray(hi, np.int32)
        C = np.empty((h, w, D), np.float32)
        if cost is None:
            _lib.check(self._L.s2pb_costvolume(self._ctx, _fp(u), _fp(v), w, h, _ip(lo), _ip(hi), int(gmin), int(D), win, _fp(C)))
        else:
            ci = _lib.COSTS.index(cost) if isinstance(cost, str) else int(cost)
            _lib.check(self._L.s2pb_costvolume_dist(self._ctx, _fp(u), _fp(v), w, h, _ip(lo), _ip(hi), int(gmin), int(D), win, ci,
                                                    _fp(C)))
        return C

    def aggregate(self, C, lo, hi, gmin, P1=8.0, P2=32.0, ndir=8, tsgm=3, fix_overcount=1, want_S=True, weights=None,
                  general=False):
        """general / weights: the float-cost aggregation flavour (any costs, optional per-pixel weight image)."""
        C = _f32(C)
        h, w, D = C.shape
        lo = np.ascontiguousarray(lo, np.int32)
        hi = np.ascontiguousarray(hi, np.int32)
        S = np.empty_like(C) if want_S else None
        disp = np.empty((h, w), np.float32)
        cost = np.empty((h, w), np.float32)
        conf = np.empty((h, w), np.float32)
        if general or weights is not None:
            wgt = _f32(weights) if weights is not None else None
            _lib.check(self._L.s2pb_aggregate_w(self._ctx, _fp(C), _ip(lo), _ip(hi), w, h, int(gmin), D, P1, P2, ndir, tsgm,
                                                fix_overcount, _fp(wgt) if wgt is not None else None,
                                                _fp(S) if want_S else None, _fp(disp), _fp(cost), _fp(conf)))
        else:
            _lib.check(self._L.s2pb_aggregate(self._ctx, _fp(C), _ip(lo), _ip(hi), w, h, int(gmin), D, P1, P2, ndir, tsgm,
                                              fix_overcount, _fp(S) if want_S else None, _fp(disp), _fp(cost), _fp(conf)))
        return S, disp, cost, conf

    def median(self, img, radius=1):
        img = _f32(img)
        h, w = img.shape
        out = np.empty_like(img)
        _lib.check(self._L.s2pb_median(self._ctx, _fp(img), _fp(out), w, h, radius))
        return out

    def remove_small_cc(self, img, minarea=25):
        img = _f32(img)
        h, w = img.shape
        out = np.empty_like(img)
        _lib.check(self._L.s2pb_remove_small_cc(self._ctx, _fp(img), _fp(out), w, h, int(minarea)))
        return out

    def rejection_mask(self, disp, im1, im2):
        disp, im1, im2 = _f32(disp), _f32(im1), _f32(im2)
        h, w = disp.shape
        mask = np.empty((h, w), np.uint8)
        _lib.check(self._L.s2pb_rejection_mask(self._ctx, _fp(disp), _fp(im1), _fp(im2), w, h, _u8(mask)))
        return mask


_engines = {}


def get_engine(device=None):
    """Per-process, per-device singleton.  ``device=None`` picks a GPU from the
    multiprocessing worker identity (worker k -> GPU k mod n_gpu), which is how the
    s2p process pool (s2p/parallel.py:80-98) is spread over the GPUs of a box."""
    if device is None:
        device = int(os.environ.get("S2PB_DEVICE", -1))
        if device < 0:
            import multiprocessing
            ident = multiprocessing.current_process()._identity
            n = max(1, device_count())
            device = (ident[0] - 1) % n if ident else 0
    key = (os.getpid(), device)
    if key not in _engines:
        eng = Engine(device)
        # S2PB_WORKSPACE_LIMIT (GiB per workspace): the setting reaches s2p's pool workers through their environment
        limit = os.environ.get("S2PB_WORKSPACE_LIMIT")
        if limit:
            eng.set_workspace_limit(int(float(limit) * 2 ** 30))
        _engines[key] = eng
    return _engines[key]
