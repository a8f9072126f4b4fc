"""TEST INFRASTRUCTURE ONLY -- what the 3D outlier filter of triangulation (count_3d_neighbors, remove_isolated_3d_points,
c/disp_to_h.c:143-230) is checked against:

* the reference's own functions in oracle/_ref/libdisp_to_h_ref.so (c/disp_to_h.c compiled in place by oracle/Makefile),
  live where that library is built, otherwise through the digests of their outputs recorded in
  tests/golden/pointcloud_ref_outputs.json (S2PB_RECORD_REF=1 with the library built rewrites the entries that run);
* a plain numpy restatement: exact counts (the reference build's fused float arithmetic emulated, ties near r*r resolved
  with fractions) and the rejection as reachability: a rejected point is kept iff a chain of "close and within the
  q-window" links through rejected points joins it to a point that was never rejected;
* the seeded clouds the tests use.
"""
import ctypes
import json
import os
from collections import deque
from fractions import Fraction

import numpy as np

from oracle import oracle as O

REF_LIB = os.path.join(O.REF_DIR, "libdisp_to_h_ref.so")
RECORDED = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pointcloud_ref_outputs.json")


def have_ref():
    return os.path.exists(REF_LIB)


# ---------------------------------------------------------------- the reference library

def _ref():
    return ctypes.CDLL(REF_LIB)


def _cloud(xyz):
    a = np.ascontiguousarray(xyz, np.float64)
    assert a.ndim == 3 and a.shape[2] == 3
    return a


def ref_count_3d_neighbors(xyz, r, p):
    a = _cloud(xyz)
    h, w = a.shape[:2]
    out = np.zeros((h, w), np.int32)
    _ref().count_3d_neighbors(out.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), a.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                              w, h, ctypes.c_float(r), int(p))
    return out


def ref_remove_isolated_3d_points(xyz, r, p, n, q=1):
    """-> a filtered copy of xyz"""
    a = _cloud(xyz).copy()
    h, w = a.shape[:2]
    _ref().remove_isolated_3d_points(a.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), w, h, ctypes.c_float(r), int(p), int(n), int(q))
    return a


_db = None


def recorded(key, live):
    """live: a callable running the reference -> array, or None where the library is not built.  -> digest of its output."""
    global _db
    if _db is None:
        _db = json.load(open(RECORDED)) if os.path.exists(RECORDED) else {}
    if live is None:
        if key not in _db:
            raise LookupError("no recorded output of the reference for %s (record it where oracle/_ref is built: S2PB_RECORD_REF=1)" % key)
        return _db[key]
    out = O.digest(live())
    if os.environ.get("S2PB_RECORD_REF") == "1" and _db.get(key) != out:
        _db[key] = out
        merged = json.load(open(RECORDED)) if os.path.exists(RECORDED) else {}
        merged[key] = out
        with open(RECORDED, "w") as f:
            json.dump(merged, f, indent=0, sort_keys=True)
    return out


def _r32(r):
    return float(np.float32(r))          # what a c_float argument holds


def ref_count_output(xyz, r, p):
    """digest of the reference's count_3d_neighbors(xyz, r, p)"""
    key = O.call_key("count_3d_neighbors", (_r32(r), int(p)), [xyz])
    return recorded(key, (lambda: ref_count_3d_neighbors(xyz, r, p)) if have_ref() else None)


def ref_remove_output(xyz, r, p, n, q):
    """digest of the cloud the reference's remove_isolated_3d_points(xyz, r, p, n, q) leaves"""
    key = O.call_key("remove_isolated_3d_points", (_r32(r), int(p), int(n), int(q)), [xyz])
    return recorded(key, (lambda: ref_remove_isolated_3d_points(xyz, r, p, n, q)) if have_ref() else None)


# ---------------------------------------------------------------- numpy restatement

def _round_f32(v):
    """a Fraction rounded to the nearest float32 (ties to even; normal range)"""
    if v == 0:
        return v
    a = abs(v)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1                                           # 2^e <= |v| < 2^(e+1)
    ulp = Fraction(2) ** (e - 23)
    return round(v / ulp) * ulp


def _exact_sqdist(x, y, z):
    """fmaf(z, z, fmaf(x, x, y*y)) of three float32 values, as a Fraction"""
    X, Y, Z = Fraction(float(x)), Fraction(float(y)), Fraction(float(z))
    return _round_f32(Z * Z + _round_f32(X * X + _round_f32(Y * Y)))


def close(a, b, r):
    """squared_distance_between_3d_points(a, b) < r*r, elementwise over (..., 3) float64 arrays, as the reference build
    evaluates it: differences in double rounded to float, then fmaf(z, z, fmaf(x, x, y*y)) in float.  float32 products are
    exact in float64, so only the rounding of the two float64 sums to float32 can differ from fmaf (double rounding); the
    pairs where that could change the answer lie next to r*r and are recomputed exactly."""
    rr = np.float32(r) * np.float32(r)
    d = np.asarray(a, np.float64) - np.asarray(b, np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        x, y, z = (d[..., k].astype(np.float32) for k in range(3))
        inner = (x.astype(np.float64) ** 2 + (y * y).astype(np.float64)).astype(np.float32)
        dd = (z.astype(np.float64) ** 2 + inner.astype(np.float64)).astype(np.float32)
        out = dd < rr
        near = (np.abs(dd.astype(np.float64) - float(rr)) <= float(rr) * 2.0 ** -19) & ~((x == 0) & (y == 0) & (z == 0))
    for i in zip(*np.nonzero(near)):
        out[i] = _exact_sqdist(x[i], y[i], z[i]) < Fraction(float(rr))
    return out


def _shifted_pairs(h, w, di, dj):
    """slices (centre, neighbour) of the centres whose neighbour at offset (di, dj) lies in the image"""
    cy, cx = slice(max(0, -di), min(h, h - di)), slice(max(0, -dj), min(w, w - dj))
    ny_, nx_ = slice(cy.start + di, cy.stop + di), slice(cx.start + dj, cx.stop + dj)
    return (cy, cx), (ny_, nx_)


def count_restated(xyz, r, p):
    xyz = _cloud(xyz)
    h, w = xyz.shape[:2]
    out = np.zeros((h, w), np.int32)
    p = min(int(p), max(h, w))
    for di in range(-p, p + 1):
        for dj in range(-p, p + 1):
            c, u = _shifted_pairs(h, w, di, dj)
            if c[0].start < c[0].stop and c[1].start < c[1].stop:
                out[c] += close(xyz[u], xyz[c], r)
    return out


def remove_restated(xyz, r, p, n, q=1):
    """-> a filtered copy of xyz: breadth-first search from the kept points through close rejected points of the q-window"""
    xyz = _cloud(xyz)
    out = xyz.copy()
    h, w = xyz.shape[:2]
    if n <= 0:
        return out
    rejected = count_restated(xyz, r, p) < n
    q = min(int(q), max(h, w))
    links = []                                             # (di, dj, close[y, x] of (y, x) and (y + di, x + dj))
    for di in range(-q, q + 1):
        for dj in range(-q, q + 1):
            m = np.zeros((h, w), bool)
            c, u = _shifted_pairs(h, w, di, dj)
            if c[0].start < c[0].stop and c[1].start < c[1].stop:
                m[c] = close(xyz[c], xyz[u], r)
            links.append((di, dj, m))
    saved = np.zeros((h, w), bool)
    todo = deque()
    for di, dj, m in links:                                # rejected points with a close kept point in their window
        c, u = _shifted_pairs(h, w, di, dj)
        hit = np.zeros((h, w), bool)
        hit[c] = m[c] & rejected[c] & ~rejected[u]
        for y, x in zip(*np.nonzero(hit & ~saved)):
            saved[y, x] = True
            todo.append((y, x))
    while todo:
        y, x = todo.popleft()
        for di, dj, m in links:
            yy, xx = y + di, x + dj
            if 0 <= yy < h and 0 <= xx < w and m[y, x] and rejected[yy, xx] and not saved[yy, xx]:
                saved[yy, xx] = True
                todo.append((yy, xx))
    out[rejected & ~saved] = np.nan
    return out


def reference_sweeps(xyz, r, p, n, q=1):
    """number of sweeps the reference's loop makes (c/disp_to_h.c:196-220) on xyz: a plain restatement of that loop"""
    xyz = _cloud(xyz)
    h, w = xyz.shape[:2]
    rejected = count_restated(xyz, r, p) < n
    sweeps, more = 0, True
    while more:
        more, sweeps = False, sweeps + 1
        for y, x in zip(*np.nonzero(rejected)):            # raster order
            for yy in range(max(0, y - q), min(h, y + q + 1)):
                hit = False
                for xx in range(max(0, x - q), min(w, x + q + 1)):
                    if not rejected[yy, xx] and close(xyz[y, x][None], xyz[yy, xx][None], r)[0]:
                        rejected[y, x], more, hit = False, True, True
                        break
                if hit:
                    break
    return sweeps


# ---------------------------------------------------------------- clouds

def utm_cloud(h, w, seed, gsd=0.5, outliers=0.03, holes=True, nan_border=0):
    """A gridded cloud at UTM scale (easting ~3.5e5 m, northing ~7.66e6 m): a smooth surface sampled every gsd metres with
    centimetre noise, a fraction of outliers (single points and small clumps, 6 to 80 m off the surface), NaN holes
    (rectangles, single points, points with one NaN coordinate) and an optional NaN border."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    X = 350000.0 + gsd * xx + rng.normal(0, 0.05, (h, w))
    Y = 7660000.0 - gsd * yy + rng.normal(0, 0.05, (h, w))
    Z = 120.0 + 8.0 * np.sin(xx / 37.0) + 5.0 * np.cos(yy / 23.0) + rng.normal(0, 0.3, (h, w))
    k = rng.random((h, w)) < outliers
    Z[k] += rng.choice([-1.0, 1.0], k.sum()) * rng.uniform(6, 80, k.sum())
    for _ in range(max(1, h * w // 4000)):                 # clumps: rejected together, close to one another
        y0, x0 = rng.integers(0, max(1, h - 3)), rng.integers(0, max(1, w - 3))
        Z[y0:y0 + 3, x0:x0 + 3] += rng.uniform(10, 40)
    xyz = np.stack([X, Y, Z], axis=2)
    if holes:
        for _ in range(max(1, h * w // 8000)):
            y0, x0 = rng.integers(0, h), rng.integers(0, w)
            xyz[y0:y0 + rng.integers(1, 12), x0:x0 + rng.integers(1, 12)] = np.nan
        xyz[rng.random((h, w)) < 0.01] = np.nan
        one = rng.random((h, w)) < 0.005
        xyz[one, rng.integers(0, 3)] = np.nan
    if nan_border:
        b = nan_border
        xyz[:b], xyz[-b:], xyz[:, :b], xyz[:, -b:] = np.nan, np.nan, np.nan, np.nan
    return xyz


def serpentine(h=24, w=30, r=5.0, seed=0):
    """An inlier blob in the bottom-right corner and a chain of points that leaves it and snakes up the grid, every other
    row, right to left then left to right.  Consecutive chain points are 0.8 r apart in 3D, any other two at least
    1.6 r, so with p = 3 and n = 5 every chain point but the first is rejected and only the chain saves it; the reference
    needs a sweep per step against its scan order.  Everything else is scattered far apart."""
    rng = np.random.default_rng(seed)
    xyz = np.stack([rng.uniform(0, 1e5, (h, w)), rng.uniform(0, 1e5, (h, w)), rng.uniform(2e5, 3e5, (h, w))], axis=2)
    xyz[..., 0] += 350000.0
    xyz[..., 1] += 7660000.0
    B = np.array([360000.0, 7670000.0, 500.0])
    xyz[h - 4:, w - 4:] = B + rng.normal(0, 0.02 * r, (4, 4, 3))
    path, y = [], h - 5
    while y >= 0:                                          # rows h-5, h-7, ...: right to left, up, left to right, up, ...
        cols = range(w - 1, -1, -1) if ((h - 5 - y) // 2) % 2 == 0 else range(w)
        path += [(y, x) for x in cols]
        if y - 1 >= 0:
            path.append((y - 1, path[-1][1]))
        y -= 2
    for k, (y, x) in enumerate(path):
        xyz[y, x] = B + np.array([0.8 * r * (k + 1), 0.0, 0.0])
    return xyz


def rounding_pins(seed=0, per_kind=4):
    """-> (xyz of shape (2, K, 3), kinds): column k holds a pair of points (rows 0 and 1) whose squared distance lies next
    to r*r = 25, 1000 m from every other column, so count[0, k] = 1 + [the pair is close] at r = 5, p = 1.  The pairs are
    chosen so that a wrong distance classifies them the other way:
      "unfused":   the float sum without FMA contraction, (x*x + y*y) + z*z;
      "double":    the differences kept in double, the squares summed in double;
      "float_xyz": the coordinates rounded to float before the differences (at 5e6 m, where a float step is 0.5 m)."""
    rng = np.random.default_rng(seed)
    r, rr = 5.0, np.float32(25.0)
    pairs, kinds = [], []
    m = 40000
    # small coordinates: a - b is the float32 vector itself, so only the sum's rounding is at stake
    v = rng.normal(size=(m, 3))
    v = (v / np.linalg.norm(v, axis=1)[:, None] * r * (1 + rng.uniform(-2e-7, 2e-7, (m, 1)))).astype(np.float32)
    a = np.zeros((m, 3))
    ours = close(a, a - v.astype(np.float64), r)
    unfused = ((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2]) < rr
    for i in np.nonzero(ours != unfused)[0][:per_kind]:
        pairs.append((a[i], a[i] - v[i].astype(np.float64)))
        kinds.append("unfused")
    # near 5e6 m: the differences are exact in double and round to float
    a = 5e6 + rng.uniform(0, 1000, (m, 3))
    d = rng.normal(size=(m, 3))
    d = d / np.linalg.norm(d, axis=1)[:, None] * r * (1 + rng.uniform(-3e-7, 3e-7, (m, 1)))
    b = a - d
    ours = close(a, b, r)
    dbl = ((a - b) ** 2).sum(axis=1) < float(rr)
    f32 = close(a.astype(np.float32).astype(np.float64), b.astype(np.float32).astype(np.float64), r)
    for alt, name in ((dbl, "double"), (f32, "float_xyz")):
        for i in np.nonzero(ours != alt)[0][:per_kind]:
            pairs.append((a[i], b[i]))
            kinds.append(name)
    K = len(pairs)
    xyz = np.zeros((2, K, 3))
    for k, (pa, pb) in enumerate(pairs):
        off = np.array([1000.0 * k, 0.0, 0.0]) if abs(pa[0]) < 1e6 else np.array([0.0, 1000.0 * k, 0.0])
        xyz[0, k], xyz[1, k] = pa + off, pb + off
    return xyz, kinds


def pin_alternatives(xyz):
    """per column of a rounding_pins cloud: is the pair close under (ours, unfused, double, float_xyz)"""
    a, b = xyz[0], xyz[1]
    rr = np.float32(25.0)
    v = (a - b).astype(np.float32)
    return dict(ours=close(a, b, 5.0),
                unfused=((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2]) < rr,
                double=((a - b) ** 2).sum(axis=1) < float(rr),
                float_xyz=close(a.astype(np.float32).astype(np.float64), b.astype(np.float32).astype(np.float64), 5.0))
