"""The reference matcher at every census window s2p can ask for (CENSUS_NCC_WIN 2 to 11), as a CPU oracle for the tests.

oracle/mgm_oracle.c keeps one 64-bit word per census code and takes the code's bits from win * win, which is right for the odd
windows up to 7.  The reference takes any win: the radius is win / 2 (mgm_costvolume.cc:109), a code has side^2 - 1 bits in
ceil(bits / 32) float channels nch (census_tools.cc:38-99), and a label costs popcount * (25 / win^2) / nch
(mgm_costvolume.h:86-92).  Here the census cost volume is restated with codes of up to 120 bits in numpy; every other stage of
`mgm` and `mgm_multi` is the C restatement's own exported function (liboracle.so), called in the order orc_view, orc_mgm_call_w,
orc_mgm_w, orc_recursive and orc_mgm_multi_w call them.  The other distances take the window only as NCC's half width and as
MINDIFF's window, which the C restatement already follows for every win: ``mgm`` / ``mgm_multi`` hand them to it.
"""
import ctypes

import numpy as np

from oracle import oracle as O

_POPC8 = np.array([bin(i).count("1") for i in range(256)], np.uint8)


def census_bits(win):
    side = 2 * (int(win) // 2) + 1
    return side * side - 1


def census_codes(img, win):
    """census_tools.cc:38-57: -> uint8 [nbytes, h, w], the code's bits (centre < neighbour, row-major window order, centre
    skipped, 0 outside the image) packed 8 to a byte"""
    img = np.asarray(img, np.float32)
    h, w = img.shape
    r = int(win) // 2
    pad = np.full((h + 2 * r, w + 2 * r), np.nan, np.float32)
    pad[r:r + h, r:r + w] = img
    bits = [img < pad[r + j:r + j + h, r + i:r + i + w] for j in range(-r, r + 1) for i in range(-r, r + 1) if i or j]
    return np.packbits(np.stack(bits), axis=0)


def costvolume(u, v, lo, hi, gmin, D, win, zoom=1, dct_shift=1):
    """orc_costvolume_census with codes of any width: [h, w, D] float32, +INF outside each pixel's [lo, hi]"""
    u = np.ascontiguousarray(u, np.float32)
    h, w = u.shape
    cu = census_codes(u, win)
    cv = []
    for z in range(zoom):                      # alloc_prefiltered_fourier_subpix_interp, mgm_costvolume.cc:50-60
        t = np.empty_like(u)
        O.lib().orc_shift(O._p(np.ascontiguousarray(v, np.float32)), O._p(t), w, h, ctypes.c_float(z / zoom), dct_shift)
        cv.append(census_codes(t, win))
    nch = (census_bits(win) // 8 + 3) // 4
    ratio = np.float64(np.float32(25.0 / (float(win) * win)))
    lo = lo.reshape(h, w)
    hi = hi.reshape(h, w)
    C = np.full((h, w, D), np.inf, np.float32)
    xs = np.arange(w)[None, :]
    anyfin = np.zeros((h, w), bool)
    for k in range(D):
        o = gmin + k
        qx = xs + o // zoom                    # floor(o / zoom), goodmod(o, zoom): mgm_costvolume.cc:145-154
        ok = (qx >= 0) & (qx < w)
        qc = np.clip(qx, 0, w - 1)
        r = _POPC8[cu ^ cv[o % zoom][:, :, qc[0]]].sum(axis=0, dtype=np.int64)
        e = np.where(ok, ((r * 1.0) * ratio / nch).astype(np.float32), np.float32(np.inf))
        inr = (o >= lo) & (o <= hi)
        C[:, :, k] = np.where(inr, e, np.inf)
        anyfin |= inr & ok
    for k in range(D):                         # no finite label in the range: the whole range is 0 (:166-171)
        o = gmin + k
        C[:, :, k] = np.where(~anyfin & (o >= lo) & (o <= hi), 0, C[:, :, k])
    return C


def _i32(a):
    return np.ascontiguousarray(a, np.int32)


def _view(u, v, dmin_i, dmax_i, P, zoom, wgt):
    """orc_view (census): -> disp, cost, conf"""
    L = O.lib()
    h, w = u.shape
    n = w * h
    lo, hi = np.empty(n, np.int32), np.empty(n, np.int32)
    L.orc_ranges(O._p(O._f32(dmin_i)), O._p(O._f32(dmax_i)), n, zoom, O._p(lo, ctypes.c_int), O._p(hi, ctypes.c_int))
    gmin, D = int(lo.min()), int(hi.max() - lo.min() + 1)
    C = costvolume(u, v, lo, hi, gmin, D, P.census_win, zoom, P.dct_shift)
    S = np.empty_like(C)
    disp, cost, conf = (np.empty((h, w), np.float32) for _ in range(3))
    P1 = np.float32(P.P1) / np.float32(zoom)                     # mgm_multiscale.cc:194-202
    L.orc_aggregate_w(O._p(C), O._p(lo, ctypes.c_int), O._p(hi, ctypes.c_int), w, h, gmin, D, ctypes.c_float(P1),
                      ctypes.c_float(P.P2), P.ndir, P.tsgm, P.fix_overcount, O._p(O._f32(wgt)) if wgt is not None else None,
                      O._p(S), O._p(disp), O._p(cost), O._p(conf))
    L.orc_refine(O._p(S), O._p(lo, ctypes.c_int), O._p(hi, ctypes.c_int), n, gmin, D, P.refine, O._p(disp), O._p(cost))
    return disp / np.float32(zoom), cost, conf


def _mgm_call(u, v, a, b, c, d, P, zoom, wl, wr):
    """orc_mgm_call_w: -> dl, dr, confL"""
    L = O.lib()
    h, w = u.shape
    dl, _, confL = _view(u, v, a, b, P, zoom, wl)
    dr, cr, _ = _view(v, u, c, d, P, zoom, wr)
    if P.median:
        dl, dr = O.port.median(dl, P.median), O.port.median(dr, P.median)
    dl, dr = np.ascontiguousarray(dl), np.ascontiguousarray(dr)
    if P.mindiff >= 0:
        L.orc_mindiff(O._p(dl), O._p(np.ascontiguousarray(cr)), w, h, P.census_win, ctypes.c_float(P.mindiff))
    if P.lr_mode == 1:
        tl, tr = dl.copy(), dr.copy()
        L.orc_lrcheck(O._p(dr), w, h, O._p(tl), w, ctypes.c_float(P.lr_tau))
        L.orc_lrcheck(O._p(dl), w, h, O._p(tr), w, ctypes.c_float(P.lr_tau))
    if P.remove_small_cc > 0:
        dl, dr = O.port.remove_small_cc(dl, P.remove_small_cc, 5.0), O.port.remove_small_cc(dr, P.remove_small_cc, 5.0)
    return dl, dr, confL


def _inputs(im1, im2, dmin, dmax):
    """main_mgm.cc:172-216 / main_mgm_multi.cc:160-196: NaN-free images and the four bound images"""
    im1, im2 = O._f32(im1), O._f32(im2)
    u = np.where(np.isfinite(im1), im1, 0).astype(np.float32)
    v = np.where(np.isfinite(im2), im2, 0).astype(np.float32)
    n1, n2 = np.isnan(im1), np.isnan(im2)
    a = np.full(im1.shape, dmin, np.float32)
    b = np.where(n1, dmin + 1, dmax).astype(np.float32)
    c = np.where(n2, dmin, -dmax).astype(np.float32)
    d = np.where(n2, dmin + 1, -dmin).astype(np.float32)
    return u, v, a, b, c, d


def mgm(im1, im2, dmin, dmax, P, wl=None, wr=None):
    """-> disp, conf, dispR: the `mgm` binary, as oracle.port.mgm"""
    if P.cost != 0:
        return O.port.mgm(im1, im2, dmin, dmax, P, wl, wr)
    u, v, a, b, c, d = _inputs(im1, im2, dmin, dmax)
    if wl is None or wr is None:
        wl = wr = None
    dl, dr, conf = _mgm_call(u, v, a, b, c, d, P, 1, wl, wr)
    return np.where(np.isnan(im1), np.nan, dl).astype(np.float32), conf, np.where(np.isnan(im2), np.nan, dr).astype(np.float32)


def _ds(img, sigma=0.8):
    h, w = img.shape
    out = np.empty(((h + 1) // 2, (w + 1) // 2), np.float32)
    O.lib().orc_downsample2x(O._p(O._f32(img)), w, h, ctypes.c_float(sigma), O._p(out))
    return out


def _ds_disp(img, is_max):
    h, w = img.shape
    out = np.empty(((h + 1) // 2, (w + 1) // 2), np.float32)
    O.lib().orc_downsample2x_disp(O._p(O._f32(img)), w, h, int(is_max), O._p(out))
    return out


def _update(disp, dmin_i, dmax_i, prev_min, prev_max, slack, radius):
    h, w = disp.shape
    ph, pw = prev_min.shape
    dmin_i, dmax_i = O._f32(dmin_i).copy(), O._f32(dmax_i).copy()
    O.lib().orc_update_dmin_dmax(O._p(O._f32(disp)), w, h, O._p(dmin_i), O._p(dmax_i), O._p(O._f32(prev_min)),
                                 O._p(O._f32(prev_max)), pw, ph, slack, radius)
    return dmin_i, dmax_i


def _upsample(sdisp, dmin, dmax):
    sh, sw = sdisp.shape
    h, w = dmin.shape
    dmin, dmax = O._f32(dmin).copy(), O._f32(dmax).copy()
    O.lib().orc_upsample2x_disp(O._p(O._f32(sdisp)), sw, sh, O._p(dmin), O._p(dmax), w, h)
    return dmin, dmax


def _recursive(u, v, a, b, c, d, P, zoom, numscales, scale, wl, wr):
    """orc_recursive: -> dl, dr, confL (a..d are updated in place by the coarser levels, as in the C code)"""
    h, w = u.shape
    if max(w, h) > 100 and min(w, h) > 50 and scale < numscales:
        swl, swr = (_ds(wl), _ds(wr)) if wl is not None and wr is not None else (None, None)
        sdl, sdr, _ = _recursive(_ds(u), _ds(v), _ds_disp(a, 0), _ds_disp(b, 1), _ds_disp(c, 0), _ds_disp(d, 1), P, zoom,
                                 numscales, scale + 1, swl, swr)
        a[:], b[:] = _upsample(sdl, a, b)
        c[:], d[:] = _upsample(sdr, c, d)
    return _mgm_call(u, v, a, b, c, d, P, zoom, wl, wr)


def mgm_multi(im1, im2, dmin, dmax, P, wl=None, wr=None):
    """-> disp, conf, dispR: the `mgm_multi` binary, as oracle.port.mgm_multi"""
    if P.cost != 0:
        return O.port.mgm_multi(im1, im2, dmin, dmax, P, wl, wr)
    L = O.lib()
    u, v, a, b, c, d = _inputs(im1, im2, dmin, dmax)
    h, w = u.shape
    if wl is None or wr is None:
        wl = wr = None
    dl, dr, conf = _recursive(u, v, a, b, c, d, P, 1, P.scales, 0, wl, wr)
    if P.subpix > 1:                                             # main_mgm_multi.cc:203-209, without the weight images
        a, b = _update(dl, a, b, a, b, 2, 4)
        c, d = _update(dr, c, d, c, d, 2, 4)
        dl, dr, _ = _recursive(u, v, a, b, c, d, P, P.subpix, 0, 0, None, None)
    if P.lr_mode == 2:
        tl, tr = dl.copy(), dr.copy()
        dl, dr = np.ascontiguousarray(dl), np.ascontiguousarray(dr)
        L.orc_lrcheck(O._p(dr), w, h, O._p(tl), w, ctypes.c_float(P.lr_tau))
        L.orc_lrcheck(O._p(dl), w, h, O._p(tr), w, ctypes.c_float(P.lr_tau))
    im1, im2 = O._f32(im1), O._f32(im2)
    return np.where(np.isnan(im1), np.nan, dl).astype(np.float32), conf, np.where(np.isnan(im2), np.nan, dr).astype(np.float32)
