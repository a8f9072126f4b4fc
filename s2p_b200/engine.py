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
from ._lib import MgmParams, S2pbError  # noqa: F401  (re-exported)


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


def device_count():
    return _lib.lib().s2pb_device_count()


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _fp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))


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
                mask.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)) if want_mask else None,
                _fp(right) if want_right else None, _fp(pl), _fp(pr)))
            out = dict(disp=disp, conf=conf, mask=mask, pkr_left=pl, pkr_right=pr)
            if want_right:
                out["disp_right"] = right
            return out
        _lib.check(self._L.s2pb_mgm_weighted(
            self._ctx, _fp(im1), _fp(im2), w, h, int(dmin), int(dmax), ctypes.byref(p),
            _fp(wl) if wl is not None else None, _fp(wr) if wr is not None else None, _fp(disp), _fp(conf),
            mask.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)) if want_mask else None,
            _fp(right) if want_right else None))
        out = dict(disp=disp, conf=conf, mask=mask)
        if want_right:
            out["disp_right"] = right
        return out

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

    def kernel_launches(self):
        return int(self._L.s2pb_kernel_launches(self._ctx))

    # ------------------------------------------------------------------ rectification warp
    def homography(self, src, H, w, h, out=None):
        """out(x) = src(H^-1 x) on [0,w] x [0,h]: what `homography im -h "..." out w h` computes
        (s2p/common.py:159-180), order-5 B-spline with the reference's anti-aliasing rule."""
        src = _f32(src)
        if src.ndim != 2:
            raise ValueError("src must be a 2-D array")
        Hm = np.ascontiguousarray(np.asarray(H, dtype=np.float64).reshape(9))
        if out is None:
            out = np.empty((int(h), int(w)), np.float32)
        elif out.shape != (int(h), int(w)) or out.dtype != np.float32 or not out.flags.c_contiguous:
            raise ValueError("out must be a C-contiguous float32 array of shape (h, w)")     # e.g. a page-locked buffer: DMA'd directly
        _lib.check(self._L.s2pb_homography(self._ctx, _fp(src), src.shape[1], src.shape[0],
                                           Hm.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), _fp(out), int(w), int(h)))
        return out

    def rectify_match(self, src1, H1, src2, H2, w, h, dmin, dmax, params=None, want_rect=True, want_right=False):
        """rectify_pair's two warps + compute_disparity_map in one call, the rectified pair staying on the device
        (s2p/__init__.py:147-155,184-190).  -> dict(disp, conf, mask[, rect1, rect2][, disp_right])"""
        src1, src2 = _f32(src1), _f32(src2)
        p = params or default_params("mgm")
        w, h = int(w), int(h)
        dp = lambda a: np.ascontiguousarray(np.asarray(a, dtype=np.float64).reshape(9)).ctypes.data_as(ctypes.POINTER(ctypes.c_double))
        Ha, Hb = np.ascontiguousarray(np.asarray(H1, np.float64).reshape(9)), np.ascontiguousarray(np.asarray(H2, np.float64).reshape(9))
        out = dict(disp=np.empty((h, w), np.float32), conf=np.empty((h, w), np.float32), mask=np.empty((h, w), np.uint8))
        if want_rect:
            out["rect1"], out["rect2"] = np.empty((h, w), np.float32), np.empty((h, w), np.float32)
        if want_right:
            out["disp_right"] = np.empty((h, w), np.float32)
        nul = ctypes.POINTER(ctypes.c_float)()
        _lib.check(self._L.s2pb_rectify_match(
            self._ctx, _fp(src1), src1.shape[1], src1.shape[0], Ha.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
            _fp(src2), src2.shape[1], src2.shape[0], Hb.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), w, h, int(dmin), int(dmax),
            ctypes.byref(p), _fp(out["rect1"]) if want_rect else nul, _fp(out["rect2"]) if want_rect else nul, _fp(out["disp"]),
            _fp(out["conf"]), out["mask"].ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)), _fp(out["disp_right"]) if want_right else nul))
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
        u8 = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8))
        _lib.check(self._L.s2pb_erode_mask(self._ctx, u8(m), u8(out), w, h, float(radius)))
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
            _lib.check(self._L.s2pb_count_3d_neighbors(self._ctx, out.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)),
                                                        a.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), w, h, float(r),
                                                        operator.index(p)))
        return out

    def remove_isolated_3d_points(self, xyz, r, p, n, q=1):
        """NaN into the isolated points of np.ascontiguousarray(xyz), in place (c/disp_to_h.c:177-230): a C-contiguous
        float64 xyz is itself modified.  -> that array."""
        a = self._cloud(xyz)
        h, w = a.shape[:2]
        if not a.flags.writeable:
            raise ValueError("the point cloud is read-only")
        if a.size:
            _lib.check(self._L.s2pb_remove_isolated_3d_points(self._ctx, a.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), w, h,
                                                               float(r), operator.index(p), operator.index(n), operator.index(q)))
        return a

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
        ip = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))
        if cost is None:
            _lib.check(self._L.s2pb_costvolume(self._ctx, _fp(u), _fp(v), w, h, ip(lo), ip(hi), int(gmin), int(D), win, _fp(C)))
        else:
            ci = _lib.COSTS.index(cost) if isinstance(cost, str) else int(cost)
            _lib.check(self._L.s2pb_costvolume_dist(self._ctx, _fp(u), _fp(v), w, h, ip(lo), ip(hi), int(gmin), int(D), win, ci, _fp(C)))
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
        ip = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))
        if general or weights is not None:
            wgt = _f32(weights) if weights is not None else None
            _lib.check(self._L.s2pb_aggregate_w(self._ctx, _fp(C), ip(lo), ip(hi), w, h, int(gmin), D, P1, P2, ndir, tsgm,
                                                fix_overcount, _fp(wgt) if wgt is not None else None,
                                                _fp(S) if want_S else None, _fp(disp), _fp(cost), _fp(conf)))
        else:
            _lib.check(self._L.s2pb_aggregate(self._ctx, _fp(C), ip(lo), ip(hi), w, h, int(gmin), D, P1, P2, ndir, tsgm,
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
        _lib.check(self._L.s2pb_rejection_mask(self._ctx, _fp(disp), _fp(im1), _fp(im2), w, h,
                                               mask.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8))))
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
        _engines[key] = Engine(device)
    return _engines[key]
