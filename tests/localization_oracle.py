"""TEST INFRASTRUCTURE ONLY -- what the localisation of a height map (s2p.triangulation.height_map_to_xyz,
s2p/triangulation.py:165-217) is checked against:

* the reference's own rpc_localization (c/rpc.c:469; eval_rpc: the direct polynomials when the model has them, the
  iteration of c/rpc.c:378-411 otherwise), from oracle/_ref/libdisp_to_h_ref.so (c/disp_to_h.c + c/rpc.c compiled in place
  by oracle/Makefile), called pixel by pixel through ctypes.  Where that library is not built (it needs the reference's
  sources), what it returned for the cases below when they were recorded: tests/golden/localization_ref_samples.npz, the
  NaN mask and lon / lat on a seeded sample of pixels, written by tests/golden/make_golden_triplet.py;
* a numpy evaluation of the ground->image polynomials in the monomial order of csrc/triangulation_kernels.cuh, which
  projects a localised point back into the image: the normalised residual is what the iteration stops on (<= 1e-18 squared);
* a numpy restatement of that iteration, vectorised over the pixels (the non-convergence case is checked on it first, and
  scripts/height_map_to_xyz_probe.py times it as a one-core stand-in for rpcm);
* the real tri-stereo fixture, tests/golden/triplet.npz (tests/golden/make_golden_triplet.py).
"""
import ctypes
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libdisp_to_h_ref.so")
TRIPLET = os.path.join(HERE, "golden", "triplet.npz")
RECORDED = os.path.join(HERE, "golden", "localization_ref_samples.npz")
SAMPLE = 2048
STOP = 1e-18                  # the iteration's test on the squared normalised residual (c/rpc.c:397)
MAXIT = 1000                  # the device's cap on that iteration


# ---------------------------------------------------------------- the reference's rpc_localization

def have_ref():
    return os.path.exists(REF_LIB)


_ref = None


def _lib():
    global _ref
    if _ref is None:
        _ref = ctypes.CDLL(REF_LIB)
        _ref.rpc_localization.restype = None
        _ref.rpc_localization.argtypes = [ctypes.POINTER(ctypes.c_double), ctypes.c_void_p, ctypes.POINTER(ctypes.c_double)]
    return _ref


def ref_localization(rpc, cols, rows, alts):
    """rpc_localization(lonlat, rpc, (col, row, alt)) point by point -> (lon, lat) float64 arrays"""
    L = _lib()
    cols, rows, alts = (np.asarray(a, np.float64).ravel() for a in (cols, rows, alts))
    lon, lat = np.empty(len(cols)), np.empty(len(cols))
    ijh, ll = (ctypes.c_double * 3)(), (ctypes.c_double * 2)()
    p = ctypes.cast(ctypes.pointer(rpc), ctypes.c_void_p)
    for k in range(len(cols)):
        ijh[0], ijh[1], ijh[2] = cols[k], rows[k], alts[k]
        L.rpc_localization(ll, p, ijh)
        lon[k], lat[k] = ll[0], ll[1]
    return lon, lat


def ref_height_map_to_xyz(heights, rpc, off_x, off_y):
    """height_map_to_xyz with out_crs None, localised by the reference's library -> (h, w, 3) float64; NaN in all three
    where the height is NaN (the reference leaves lon / lat undefined there, and every later step drops such rows)"""
    z = np.asarray(heights)
    h, w = z.shape
    rows, cols = np.indices((h, w))
    ok = ~np.isnan(z)
    out = np.full((h, w, 3), np.nan)
    out[ok, 0], out[ok, 1] = ref_localization(rpc, cols[ok] + off_x, rows[ok] + off_y, z[ok])
    out[ok, 2] = z[ok]
    return out


# ---------------------------------------------------------------- numpy evaluation of the camera

def _monomials(u, v, w):
    """(20, n): 1 u v w uv uw vw uu vv ww uvw uuu uvv uww uuv vvv vww uuw vvw www (csrc/triangulation_kernels.cuh)"""
    return np.stack([np.ones_like(u), u, v, w, u * v, u * w, v * w, u * u, v * v, w * w, u * v * w, u * u * u, u * v * v,
                     u * w * w, u * u * v, v * v * v, v * w * w, u * u * w, v * v * w, w * w * w])


def _coef(rpc, name):
    return np.array(getattr(rpc, name)[:], np.float64)


def _ground_to_image_n(rpc, ln, lt, w):
    """normalised (lon, lat, height) -> normalised (col, row), the reference's eval_nrpci"""
    m = _monomials(ln, lt, w)
    return (_coef(rpc, "inumx") @ m) / (_coef(rpc, "idenx") @ m), (_coef(rpc, "inumy") @ m) / (_coef(rpc, "ideny") @ m)


def residual2(rpc, cols, rows, alts, lon, lat):
    """the squared normalised distance between image pixel (col, row) and the projection of (lon, lat, alt): the quantity
    the localisation iterates on, with lon / lat normalised back from the output"""
    xn = (np.asarray(cols, np.float64) - rpc.offset[0]) / rpc.scale[0]
    yn = (np.asarray(rows, np.float64) - rpc.offset[1]) / rpc.scale[1]
    w = (np.asarray(alts, np.float64) - rpc.offset[2]) / rpc.scale[2]
    px, py = _ground_to_image_n(rpc, (np.asarray(lon) - rpc.ioffset[0]) / rpc.iscale[0],
                                (np.asarray(lat) - rpc.ioffset[1]) / rpc.iscale[1], w)
    return (xn - px) ** 2 + (yn - py) ** 2


def localize(rpc, cols, rows, alts, maxit=MAXIT):
    """numpy restatement of the localisation of a model without direct polynomials (c/rpc.c:378-411 with the device's cap),
    vectorised over the points -> (lon, lat, converged): converged is False where the cap was reached without the test
    being met"""
    xn = (np.asarray(cols, np.float64).ravel() - rpc.offset[0]) / rpc.scale[0]
    yn = (np.asarray(rows, np.float64).ravel() - rpc.offset[1]) / rpc.scale[1]
    w = (np.asarray(alts, np.float64).ravel() - rpc.offset[2]) / rpc.scale[2]
    delta = rpc.delta if rpc.delta else 1.0
    n = len(xn)
    ln, lt, eps = np.full(n, -delta), np.full(n, -delta), np.full(n, 2 * delta)
    f = lambda a, b, c: _ground_to_image_n(rpc, a, b, c)
    x0, y0 = f(ln, lt, w)
    x1, y1 = f(ln + eps, lt, w)
    x2, y2 = f(ln, lt + eps, w)
    live = np.arange(n)
    done = np.zeros(n, bool)
    with np.errstate(all="ignore"):
        for _ in range(maxit + 1):
            ux, uy = xn[live] - x0, yn[live] - y0
            go = ux * ux + uy * uy > STOP
            done[live[~go]] = True
            if not go.any():
                break
            if _ == maxit:
                break
            live, ux, uy, e = live[go], ux[go], uy[go], eps[live[go]]
            x0, y0, x1, y1, x2, y2 = x0[go], y0[go], x1[go], y1[go], x2[go], y2[go]
            e1x, e1y, e2x, e2y = x1 - x0, y1 - y0, x2 - x0, y2 - y0
            det = e1x * e2y - e1y * e2x
            ln[live] += (e2y * ux - e2x * uy) / det * e
            lt[live] += (-e1y * ux + e1x * uy) / det * e
            eps[live] = 0.1
            wl = w[live]
            x0, y0 = f(ln[live], lt[live], wl)
            x1, y1 = f(ln[live] + 0.1, lt[live], wl)
            x2, y2 = f(ln[live], lt[live] + 0.1, wl)
    return ln * rpc.iscale[0] + rpc.ioffset[0], lt * rpc.iscale[1] + rpc.ioffset[1], done


# ---------------------------------------------------------------- cases

def synthetic_rpc(seed, with_direct):
    """the synthetic camera of tests/test_triangulation.py"""
    from test_triangulation import _rpc
    return _rpc(seed, with_direct)


def synthetic_heights(seed, h=48, w=80):
    """heights around the synthetic camera's height offset (100 m), a few NaN"""
    rng = np.random.default_rng(seed)
    z = (100.0 + rng.normal(0.0, 150.0, (h, w))).astype(np.float32)
    z[rng.random((h, w)) < 0.05] = np.nan
    return z


def triplet():
    """the real tri-stereo fixture -> dict: rpc (92 doubles of img_02.tif's RPCCoefficientTag), heights (float32 crop of
    expected_output/triplet/height_map.tif), off (its origin in img_02.tif), dsm / dsm_xoff / dsm_yoff / dsm_res (the expected
    DSM's window over the crop's footprint, EPSG:32631), dz_median / dz_p99 (|dz| between the two, computed when the fixture
    was made)"""
    return dict(np.load(TRIPLET))


def triplet_rpc():
    from s2p_b200.triangulation import rpc_from_geotiff_tag
    return rpc_from_geotiff_tag(triplet()["rpc"])


def cases():
    """name -> (heights, rpc, off_x, off_y): the cases with a recorded reference output"""
    t = triplet()
    return {
        "synthetic_iterative": (synthetic_heights(1), synthetic_rpc(1, False), 4180.0, 3290.0),
        "synthetic_direct": (synthetic_heights(2), synthetic_rpc(2, True), 4180.0, 3290.0),
        "triplet": (t["heights"], triplet_rpc(), float(t["off"][0]), float(t["off"][1])),
    }


def case_key(name, heights, rpc, off_x, off_y):
    from oracle import oracle as O
    return O.call_key("rpc_localization:" + name, (bytes(rpc).hex(), float(off_x), float(off_y)), [heights])


def sample_of(nan, seed=0):
    npix = nan.size
    return np.sort(np.random.default_rng(seed).choice(npix, min(SAMPLE, npix), replace=False))


def record(name):
    """-> {key/...: array} of one case, run live"""
    heights, rpc, ox, oy = cases()[name]
    out = ref_height_map_to_xyz(heights, rpc, ox, oy)
    nan = np.isnan(heights)
    idx = sample_of(nan)
    key = case_key(name, heights, rpc, ox, oy)
    return {key + "/nan": np.packbits(nan.ravel()), key + "/idx": idx, key + "/val": out.reshape(-1, 3)[idx, :2]}


def ref_sampled(name):
    """-> (heights, rpc, off_x, off_y, Sampled lon / lat): every pixel live where oracle/_ref is built, else the recorded
    sample"""
    from oracle import oracle as O
    heights, rpc, ox, oy = cases()[name]
    nan = np.isnan(heights)
    if have_ref():
        out = ref_height_map_to_xyz(heights, rpc, ox, oy)
        return heights, rpc, ox, oy, O.Sampled(out.shape, nan, np.arange(nan.size), out.reshape(-1, 3)[:, :2])
    key = case_key(name, heights, rpc, ox, oy)
    db = np.load(RECORDED)
    if key + "/idx" not in db:
        raise LookupError("no recorded output of rpc_localization for %s (tests/golden/make_golden_triplet.py records it)" % key)
    rec_nan = np.unpackbits(db[key + "/nan"])[:nan.size].reshape(nan.shape).astype(bool)
    assert np.array_equal(rec_nan, nan)
    return heights, rpc, ox, oy, O.Sampled(heights.shape + (2,), nan, db[key + "/idx"], db[key + "/val"])
