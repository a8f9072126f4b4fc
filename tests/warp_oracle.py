"""The rectification warp restated in NumPy, as the engine defines it (s2p_b200/csrc/warp.cu, homography_kernels.cuh).

Test infrastructure.  Every step is written from the engine's definitions, vectorised across lines and pixels:
  * the needed ROI: pre-image of the output corners through the adjugate inverse, floor / ceil, clipped to the source;
  * NaN -> 0 on the spline image, infinities kept;
  * the two-pole prefilter along rows, then along columns.  A line shorter than 2 * SEG samples runs the sequential recursion
    (`spline_columns_kernel`: full-length initForward, exact initBackward); a longer one runs in SEG-sample segments with a
    WARM-sample zero-state warm-up on both sides (`spline_segments_kernel`).  For finite data the two agree to |z0|^WARM of a
    coefficient; the segmented form is kept because it decides where an infinity spreads;
  * the order-5 B-spline weights and the half-sample symmetric extension.  The weights are formed in float32 as the kernel
    forms them (their formula cancels: up to 6e-5 away from the exact weights), unless exact_weights is set;
  * the sample coordinates: invert33 (multiplication by 1/det), (x, y) in double, px = (float)(x + 0.5), NaN unless
    0 <= px <= w and 0 <= py <= h;
  * the anti-aliasing branch: min_zoom_out, the intermediate of tw x th pixels, the Gaussian with float32 taps as the host
    computes them, replicated borders, the unfiltered tail of the vertical pass from column jlim, and the NaN mask of the
    true homography.
`dtype` is the precision of the image arithmetic (np.float64, or np.float32 to measure the rounding spread of a float32
implementation); the coordinates are always formed as the kernel forms them.
A spline image with a side below MIN_SIDE raises WarpError, as the engine returns S2PB_ERR_ARG there."""
import math

import numpy as np

POLES = (-0.430575, -0.0430963)
LAMBDA = 1.430575 * (1.0 + 1.0 / 0.430575) * 1.0430963 * (1.0 + 1.0 / 0.0430963)
SEG, WARM = 64, 32          # segment and warm-up lengths of spline_segments_kernel
INIT_TERMS = 48             # terms of the first segment's initForward
MIN_SIDE = 4
MAX_TAPS = 64


class WarpError(ValueError):
    """The engine refuses this warp (S2PB_ERR_ARG, or S2PB_ERR_UNSUPPORTED for a filter beyond MAX_TAPS)."""


def invert33(m):
    """Homography inverse as the kernels receive it: the adjugate times 1/det, in double, in the engine's order."""
    m = [float(v) for v in np.asarray(m, np.float64).ravel()]
    det = 1.0 / (m[0] * m[4] * m[8] - m[0] * m[5] * m[7] - m[1] * m[3] * m[8] + m[1] * m[5] * m[6] + m[2] * m[3] * m[7] -
                 m[2] * m[4] * m[6])
    return [det * (m[4] * m[8] - m[5] * m[7]), det * (m[2] * m[7] - m[1] * m[8]), det * (m[1] * m[5] - m[2] * m[4]),
            det * (m[5] * m[6] - m[3] * m[8]), det * (m[0] * m[8] - m[2] * m[6]), det * (m[2] * m[3] - m[0] * m[5]),
            det * (m[3] * m[7] - m[4] * m[6]), det * (m[1] * m[6] - m[0] * m[7]), det * (m[0] * m[4] - m[1] * m[3])]


def invert_homography(i):
    """The adjugate divided by det, which the ROI uses."""
    i = [float(v) for v in np.asarray(i, np.float64).ravel()]
    det = i[0] * i[4] * i[8] + i[2] * i[3] * i[7] + i[1] * i[5] * i[6] - i[2] * i[4] * i[6] - i[1] * i[3] * i[8] - i[0] * i[5] * i[7]
    return [(i[4] * i[8] - i[5] * i[7]) / det, (i[2] * i[7] - i[1] * i[8]) / det, (i[1] * i[5] - i[2] * i[4]) / det,
            (i[5] * i[6] - i[3] * i[8]) / det, (i[0] * i[8] - i[2] * i[6]) / det, (i[2] * i[3] - i[0] * i[5]) / det,
            (i[3] * i[7] - i[4] * i[6]) / det, (i[1] * i[6] - i[0] * i[7]) / det, (i[0] * i[4] - i[1] * i[3]) / det]


def needed_roi(H, sw, sh, dw, dh):
    """-> (x, y, w, h, Hc): the source window the output needs and H composed with the window's offset."""
    Hi = invert_homography(H)
    px, py = [], []
    for cx, cy in ((0.0, 0.0), (float(dw), 0.0), (float(dw), float(dh)), (0.0, float(dh))):
        z = Hi[6] * cx + Hi[7] * cy + Hi[8]
        px.append((Hi[0] * cx + Hi[1] * cy + Hi[2]) / z)
        py.append((Hi[3] * cx + Hi[4] * cy + Hi[5]) / z)
    mnx, mxx, mny, mxy = min(px), max(px), min(py), max(py)
    if not all(math.isfinite(v) for v in (mnx, mxx, mny, mxy)) or min(mnx, mny) < -1e9 or max(mxx, mxy) > 1e9:
        raise WarpError("degenerate matrix")
    x, y = math.floor(mnx), math.floor(mny)
    w, h = math.ceil(mxx - x), math.ceil(mxy - y)
    if x < 0:
        w, x = w + x, 0
    if y < 0:
        h, y = h + y, 0
    w, h = min(w, sw - x), min(h, sh - y)
    if w <= 0 or h <= 0:
        raise WarpError("empty roi")
    Hm = [float(v) for v in np.asarray(H, np.float64).ravel()]
    T = [1.0, 0.0, float(x), 0.0, 1.0, float(y), 0.0, 0.0, 1.0]
    Hc = [Hm[3 * r] * T[q] + Hm[3 * r + 1] * T[3 + q] + Hm[3 * r + 2] * T[6 + q] for r in range(3) for q in range(3)]
    return x, y, w, h, Hc


# ---------------------------------------------------------------- prefilter

def _sequential_pole(v, pz, dt):
    """One pole of spline_columns_kernel on lines along axis 0, in place."""
    L = v.shape[0]
    zn = dt(pz)
    zk, iz, z2k = pz, 1.0 / pz, pz ** (L - 1)
    s = v[0] + dt(z2k) * v[L - 1]
    z2k = z2k * z2k * iz
    for k in range(1, L - 1):
        s = s + dt(zk + z2k) * v[k]
        zk *= pz
        z2k *= iz
    v[0] = s / dt(1.0 - zk * zk)
    for k in range(1, L):
        v[k] = zn * v[k - 1] + v[k]
    v[L - 1] = dt(pz / (pz * pz - 1.0)) * (dt(pz) * v[L - 2] + v[L - 1])
    for k in range(L - 2, -1, -1):
        v[k] = zn * (v[k + 1] - v[k])


def _segmented_pole(v, pz, dt):
    """One pole of spline_segments_kernel on lines along axis 0 -> new array."""
    L = v.shape[0]
    zn = dt(pz)
    out = np.empty_like(v)
    c0 = dt(pz / (pz * pz - 1.0))
    for s in range(0, L, SEG):
        e, e2 = min(s + SEG, L), min(s + SEG + WARM, L)
        if s == 0:
            state, zk = v[0].copy(), pz
            for k in range(1, min(L - 2, INIT_TERMS) + 1):
                state = state + dt(zk) * v[k]
                zk *= pz
        else:
            state = np.zeros_like(v[0])
            for k in range(s - WARM, s + 1):
                state = zn * state + v[k]
        f = [state]
        for k in range(s + 1, e2):
            state = zn * state + v[k]
            f.append(state)
        if e2 == L:
            # exact start from the last two forward values, written by the segment that holds both of them
            prev = f[L - 2 - s] if L - 2 >= s else np.zeros_like(v[0])
            b = c0 * (dt(pz) * prev + f[L - 1 - s])
            if s <= L - 2 < e:
                out[L - 1] = b
            for k in range(L - 2, s - 1, -1):
                b = zn * (b - f[k - s])
                if k < e:
                    out[k] = b
        else:
            b = np.zeros_like(v[0])
            for k in range(e2 - 1, s - 1, -1):
                b = zn * (b - f[k - s])
                if k < e:
                    out[k] = b
    return out


def prefilter_lines(a, dtype=np.float64, segmented=True):
    """The two-pole prefilter of every line along axis 0 (lambda applied with the first pole) -> new array of `dtype`."""
    dt = np.dtype(dtype).type
    v = np.array(a, dtype=dt) * dt(LAMBDA)
    L = v.shape[0]
    if L < MIN_SIDE:
        raise WarpError("a spline line of %d samples" % L)
    for pz in POLES:
        if segmented and L >= 2 * SEG:
            v = _segmented_pole(v, pz, dt)
        else:
            _sequential_pole(v, pz, dt)
    return v


def prefilter(img, dtype=np.float64, segmented=True):
    """prepareSpline as the engine runs it: NaN -> 0, then along rows, then along columns."""
    a = np.array(img, dtype=dtype)
    a[np.isnan(a)] = 0
    a = prefilter_lines(a.T, dtype, segmented).T
    return prefilter_lines(a, dtype, segmented)


# ---------------------------------------------------------------- interpolation

def bspline5_weights(t, dtype=np.float32):
    """init_spline5 in `dtype` (float32: bit for bit the kernel's weights) -> (6, n); w[5 - k] weighs sample xi - 2 + k."""
    dt = np.dtype(dtype).type
    t = np.asarray(t, dt)
    ak = [dt(1.0 / 120.0), dt(-0.05), dt(0.125), dt(-1.0 / 6.0), dt(0.125), dt(-0.05)]
    p = []
    for k in range(6):
        u = t + dt(k)
        u2 = u * u
        p.append(u2 * u2 * u)
    return np.stack([sum(p[k] * ak[m - k] for k in range(m + 1)) for m in range(6)])


def symi(x, n):
    return np.where(x < 0, -x - 1, np.where(x >= n, 2 * n - x - 1, x))


def sample_coords(Hinv, ow, oh):
    """The kernel's sample points of an ow x oh output: -> (x, y) float32 positions in the spline image (px - 0.5f) and
    px, py (the float32 values tested against the image's extent)."""
    j, i = np.meshgrid(np.arange(ow, dtype=np.float64), np.arange(oh, dtype=np.float64))
    m = Hinv
    xd = m[0] * j + m[1] * i + m[2]
    yd = m[3] * j + m[4] * i + m[5]
    zd = m[6] * j + m[7] * i + m[8]
    with np.errstate(divide="ignore", invalid="ignore"):
        xd, yd = xd / zd, yd / zd
        px, py = (xd + 0.5).astype(np.float32), (yd + 0.5).astype(np.float32)
    return px - np.float32(0.5), py - np.float32(0.5), px, py


def interpolate(coef, Hinv, ow, oh, dtype=np.float64, exact_weights=False):
    """spline_warp_kernel: the coefficients `coef` (h x w) sampled at Hinv (j, i, 1) -> (oh, ow), NaN outside [0,w] x [0,h]."""
    dt = np.dtype(dtype).type
    h, w = coef.shape
    x, y, px, py = sample_coords(Hinv, ow, oh)
    valid = (px >= 0) & (px <= w) & (py >= 0) & (py <= h)
    out = np.full((oh, ow), np.nan, dt)
    x, y = x[valid], y[valid]
    xi = np.where(x < 0, -1, np.floor(x)).astype(np.int64)
    yi = np.where(y < 0, -1, np.floor(y)).astype(np.int64)
    wdt = np.float64 if exact_weights else np.float32
    cx = bspline5_weights(x - xi.astype(np.float32), wdt)[::-1].astype(dt)      # cx[k] weighs column xi - 2 + k
    cy = bspline5_weights(y - yi.astype(np.float32), wdt)[::-1].astype(dt)
    off = np.arange(-2, 4)[:, None]
    xx, yy = symi(xi[None] + off, w), symi(yi[None] + off, h)
    c = np.asarray(coef, dt)
    with np.errstate(invalid="ignore", over="ignore"):
        acc = np.zeros(xi.shape, dt)
        for a in range(6):
            row = np.zeros(xi.shape, dt)
            for b in range(6):
                row = row + c[yy[a], xx[b]] * cx[b]
            acc = acc + cy[a] * row
    out[valid] = acc
    return out


# ---------------------------------------------------------------- anti-aliasing

def min_zoom_out(m, w, h):
    """getMinZoomOut as the host computes it: the smallest singular value of H's Jacobian at the four corners, float32, <= 1."""
    m = [float(v) for v in np.asarray(m, np.float64).ravel()]

    def sv(px, py):
        X = (m[0] * px + m[1] * py + m[2], m[3] * px + m[4] * py + m[5], m[6] * px + m[7] * py + m[8])
        z = 1.0 / X[2]
        x, y = z * X[0], z * X[1]
        a, b, c, d = z * (m[0] - m[6] * x), z * (m[1] - m[7] * x), z * (m[3] - m[6] * y), z * (m[4] - m[7] * y)
        return np.float32(math.sqrt(0.5 * (a * a + b * b + c * c + d * d -
                                           math.sqrt((a * a + b * b - c * c - d * d) * (a * a + b * b - c * c - d * d) +
                                                     4.0 * (a * c + b * d) * (a * c + b * d)))))
    r = np.fmin(sv(0.0, float(h)), sv(float(w), float(h)))
    r = np.fmin(sv(float(w), 0.0), r)
    r = np.fmin(sv(0.0, 0.0), r)
    return np.fmin(np.float32(1), r)


def aa_geometry(M, w, h, ow, oh):
    """-> None when the warp of a w x h image through M needs no anti-aliasing, else
    dict(zoom_out, zoom_in, tw, th, taps (float32), jlim)."""
    zoom_out = min_zoom_out(M, w, h)
    if not zoom_out < 1:
        return None
    zoom_in = np.float32(1) / zoom_out
    tw = math.ceil(float(np.float32(ow) * zoom_in) * 1.5)
    th = math.ceil(float(np.float32(oh) * zoom_in) * 1.5)
    f = np.float32
    sigma = f(0.8) * np.sqrt(zoom_in * zoom_in - f(1))
    ks = int(f(8) * sigma + f(1))
    ks = ks + 1 - ks % 2 if ks > 3 else 3
    taps = None
    if ks <= MAX_TAPS:
        x = (np.arange(ks) - ks // 2).astype(np.float32)
        taps = np.exp(-x * x / (f(2) * sigma * sigma)).astype(np.float32)
        s = f(0)
        for t in taps:
            s = f(s + t)
        taps = (taps / s).astype(np.float32)
    jlim = 0
    while jlim < tw - 4:
        jlim += 4
    return dict(zoom_out=zoom_out, zoom_in=zoom_in, tw=tw, th=th, ks=ks, taps=taps, jlim=jlim)


def gaussian(a, taps, jlim, dtype=np.float64):
    """gauss_rows_kernel then gauss_cols_kernel: replicated borders; from column jlim the vertical pass keeps row max(y - half, 0)."""
    dt = np.dtype(dtype).type
    h, w = a.shape
    half = len(taps) // 2
    k = np.asarray(taps, dt)
    r = np.zeros_like(a)
    cols = np.arange(w)
    for q in range(len(taps)):
        r = r + k[q] * a[:, np.clip(cols + q - half, 0, w - 1)]
    rows = np.arange(h)
    c = np.zeros_like(r)
    for q in range(len(taps)):
        c = c + k[q] * r[np.clip(rows + q - half, 0, h - 1)]
    c[:, jlim:] = r[np.maximum(rows - half, 0)][:, jlim:]
    return c


# ---------------------------------------------------------------- the warp

def map_image(src, M, ow, oh, dtype=np.float64, use_aa=True, depth=0, stats=None, exact_weights=False):
    """mapImage on the ROI `src` (h x w, already cropped) through M -> (oh, ow) of `dtype`.
    `stats`, a dict, collects max_coef (the largest |spline coefficient| of every spline image) and the anti-aliasing geometry."""
    dt = np.dtype(dtype).type
    if depth > 6:
        raise WarpError("anti-aliasing recursion does not settle")
    stats = {} if stats is None else stats
    h, w = src.shape
    aa = aa_geometry(M, w, h, ow, oh) if use_aa else None
    if aa is not None:
        tw, th = aa["tw"], aa["th"]
        if tw < 1 or th < 1 or tw * th > 1 << 31:
            raise WarpError("degenerate zoom")
    else:
        tw, th = w, h
    if tw < MIN_SIDE or th < MIN_SIDE:
        raise WarpError("a %d x %d spline image" % (tw, th))
    if aa is not None:
        if aa["taps"] is None:
            raise WarpError("a %d-tap anti-aliasing filter" % aa["ks"])
        stats.setdefault("aa", []).append(aa)
        zi = float(aa["zoom_in"])
        Mz = [zi * float(v) for v in np.asarray(M, np.float64).ravel()[:6]] + [float(v) for v in np.asarray(M, np.float64).ravel()[6:]]
        with np.errstate(invalid="ignore", over="ignore"):
            img = gaussian(map_image(src, Mz, tw, th, dtype, True, depth + 1, stats, exact_weights), aa["taps"], aa["jlim"], dtype)
        zo = float(aa["zoom_out"])
        Mw = [zo, 0.0, 0.0, 0.0, zo, 0.0, 0.0, 0.0, 1.0]
    else:
        img, Mw = np.asarray(src, dt), M
    with np.errstate(invalid="ignore", over="ignore"):
        coef = prefilter(img, dtype)
    fin = np.isfinite(coef)
    stats["max_coef"] = max(stats.get("max_coef", 0.0), float(np.abs(coef[fin]).max()) if fin.any() else 0.0)
    out = interpolate(coef, invert33(Mw), ow, oh, dtype, exact_weights)
    if aa is not None:
        Ht = invert33(M)
        j, i = np.meshgrid(np.arange(ow, dtype=np.float64), np.arange(oh, dtype=np.float64))
        x, y, z = Ht[0] * j + Ht[1] * i + Ht[2], Ht[3] * j + Ht[4] * i + Ht[5], Ht[6] * j + Ht[7] * i + Ht[8]
        with np.errstate(divide="ignore", invalid="ignore"):
            x, y = x / z, y / z
            out[(x < 0) | (x >= w) | (y < 0) | (y >= h)] = np.nan
    return out


def warp(src, H, ow, oh, dtype=np.float64, stats=None, exact_weights=False):
    """`homography src -h H out ow oh` as the engine computes it -> (oh, ow) of `dtype`; raises WarpError where the engine
    returns an error.  `stats` as in map_image, plus the ROI (x, y, w, h)."""
    stats = {} if stats is None else stats
    src = np.asarray(src, np.float32)
    x, y, w, h, Hc = needed_roi(H, src.shape[1], src.shape[0], ow, oh)
    stats["roi"] = (x, y, w, h)
    return map_image(src[y:y + h, x:x + w], Hc, ow, oh, dtype, True, 0, stats, exact_weights)
