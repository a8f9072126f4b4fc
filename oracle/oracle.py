"""TEST INFRASTRUCTURE ONLY -- Python handles on the CPU oracle.

Two things live here:

* ``port``: ctypes bindings of ``oracle/liboracle.so`` (our plain-C restatement,
  ``oracle/mgm_oracle.c``);
* ``run_ref_mgm`` / ``run_ref_mgm_multi``: drive the UNMODIFIED reference binaries
  ``oracle/_ref/mgm`` and ``oracle/_ref/mgm_multi`` (built by ``oracle/Makefile`` from
  the sources under /root/reference, never copied) through PFM files with exactly the
  argv/environment s2p uses (s2p/block_matching.py:155-186,269-308).

Only tests/, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline /
``--impl reference`` legs may import this module.  The product package ``s2p_b200``
never does.
"""
import ctypes
import hashlib
import json
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(HERE, "_ref")
LIB_PATH = os.path.join(HERE, "liboracle.so")


class OrcParams(ctypes.Structure):
    _fields_ = [
        ("ndir", ctypes.c_int), ("tsgm", ctypes.c_int), ("census_win", ctypes.c_int),
        ("P1", ctypes.c_float), ("P2", ctypes.c_float), ("median", ctypes.c_int),
        ("lr_mode", ctypes.c_int), ("lr_tau", ctypes.c_float), ("mindiff", ctypes.c_float),
        ("remove_small_cc", ctypes.c_int), ("subpix", ctypes.c_int), ("scales", ctypes.c_int),
        ("refine", ctypes.c_int), ("fix_overcount", ctypes.c_int), ("dct_shift", ctypes.c_int),
        ("cost", ctypes.c_int),
    ]


COSTS = ("census", "ad", "sd", "ncc", "btad", "btsd")   # -t, index = OrcParams.cost


def mgm_params(**kw):
    """Defaults = what s2p sets for algo == 'mgm' (s2p/block_matching.py:155-186).  dct_shift=1: the matched image goes
    through the reference's DCT round trip even at shift 0 (mgm_costvolume.cc:23-60), like the binary; 0 = identity."""
    d = dict(ndir=8, tsgm=3, census_win=5, P1=8.0, P2=32.0, median=1, lr_mode=1, lr_tau=1.0,
             mindiff=-1.0, remove_small_cc=0, subpix=1, scales=-1, refine=1, fix_overcount=1,
             dct_shift=1, cost=0)
    d.update(kw)
    return OrcParams(**d)


def mgm_multi_params(**kw):
    """Defaults = what s2p sets for algo == 'mgm_multi' (s2p/block_matching.py:269-308)."""
    d = dict(ndir=8, tsgm=4, census_win=5, P1=8.0, P2=32.0, median=0, lr_mode=1, lr_tau=1.0,
             mindiff=-1.0, remove_small_cc=25, subpix=2, scales=6, refine=1, fix_overcount=1,
             dct_shift=1, cost=0)
    d.update(kw)
    return OrcParams(**d)


_lib = None


def build():
    """(Re)build liboracle.so and, when /root/reference is present, oracle/_ref."""
    subprocess.run(["make", "-s", "-C", HERE, "all"], check=True)


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            build()
        _lib = ctypes.CDLL(LIB_PATH)
    return _lib


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _p(a, t=ctypes.c_float):
    return a.ctypes.data_as(ctypes.POINTER(t))


class port:
    """numpy-level wrappers around the C restatement."""

    @staticmethod
    def census(img, win=5):
        img = _f32(img)
        h, w = img.shape
        out = np.zeros((h, w), np.uint64)
        lib().orc_census(_p(img), w, h, win, _p(out, ctypes.c_uint64))
        return out

    @staticmethod
    def costvolume(u, v, lo, hi, gmin, D, win=5, zoom=1, dct_shift=1, cost=0):
        """cost: index into COSTS, or its name"""
        u, v = _f32(u), _f32(v)
        h, w = u.shape
        lo = np.ascontiguousarray(lo, np.int32)
        hi = np.ascontiguousarray(hi, np.int32)
        C = np.empty((h, w, D), np.float32)
        ci = COSTS.index(cost) if isinstance(cost, str) else int(cost)
        lib().orc_costvolume(_p(u), _p(v), w, h, _p(lo, ctypes.c_int), _p(hi, ctypes.c_int),
                             gmin, D, win, zoom, dct_shift, ci, _p(C))
        return C

    @staticmethod
    def aggregate(C, lo, hi, gmin, P1=8.0, P2=32.0, ndir=8, tsgm=3, fix_overcount=1, weights=None):
        C = _f32(C)
        h, w, D = C.shape
        lo = np.ascontiguousarray(lo, np.int32)
        hi = np.ascontiguousarray(hi, np.int32)
        S = np.empty_like(C)
        disp = np.empty((h, w), np.float32)
        cost = np.empty((h, w), np.float32)
        conf = np.empty((h, w), np.float32)
        wgt = _f32(weights) if weights is not None else None
        lib().orc_aggregate_w(_p(C), _p(lo, ctypes.c_int), _p(hi, ctypes.c_int), w, h, gmin, D,
                              ctypes.c_float(P1), ctypes.c_float(P2), ndir, tsgm, fix_overcount,
                              _p(wgt) if wgt is not None else None, _p(S), _p(disp), _p(cost), _p(conf))
        return S, disp, cost, conf

    @staticmethod
    def mgm(im1, im2, dmin, dmax, params=None, wl=None, wr=None):
        """-> disp (left), conf, dispR : the `mgm` binary from memory to memory (wl, wr = -wl / -wr weights)."""
        return port._run("orc_mgm_w", params or mgm_params(), im1, im2, dmin, dmax, wl, wr)

    @staticmethod
    def mgm_multi(im1, im2, dmin, dmax, params=None, wl=None, wr=None):
        """-> disp (left), conf, dispR : the `mgm_multi` binary from memory to memory."""
        return port._run("orc_mgm_multi_w", params or mgm_multi_params(), im1, im2, dmin, dmax, wl, wr)

    @staticmethod
    def _run(fn, params, im1, im2, dmin, dmax, wl, wr):
        im1, im2 = _f32(im1), _f32(im2)
        h, w = im1.shape
        disp = np.empty((h, w), np.float32)
        conf = np.empty((h, w), np.float32)
        dispR = np.empty((h, w), np.float32)
        if wl is not None and wr is not None:
            wl, wr = _f32(wl), _f32(wr)
            pw = (_p(wl), _p(wr))
        else:
            pw = (None, None)
        getattr(lib(), fn)(_p(im1), _p(im2), w, h, int(dmin), int(dmax), ctypes.byref(params), pw[0], pw[1],
                           _p(disp), _p(conf), _p(dispR))
        return disp, conf, dispR

    @staticmethod
    def mgm_pkr(im1, im2, dmin, dmax, params=None, multi=False):
        """-> disp, conf, dispR, pkrL, pkrR: as `mgm` / `mgm_multi` with -confidence_pkrL / -confidence_pkrR"""
        im1, im2 = _f32(im1), _f32(im2)
        h, w = im1.shape
        out = [np.empty((h, w), np.float32) for _ in range(5)]
        lib().orc_mgm_pkr(_p(im1), _p(im2), w, h, int(dmin), int(dmax), ctypes.byref(params or (mgm_multi_params() if multi else mgm_params())),
                          1 if multi else 0, *[_p(o) for o in out])
        return tuple(out)

    @staticmethod
    def rejection_mask(disp, im1, im2):
        disp, im1, im2 = _f32(disp), _f32(im1), _f32(im2)
        h, w = disp.shape
        mask = np.empty((h, w), np.uint8)
        lib().orc_rejection_mask(_p(disp), _p(im1), _p(im2), w, h, _p(mask, ctypes.c_uint8))
        return mask

    @staticmethod
    def remove_small_cc(img, minarea=25, thr=5.0):
        img = _f32(img)
        h, w = img.shape
        out = np.empty_like(img)
        lib().orc_remove_small_cc(w, h, _p(img), _p(out), int(minarea), ctypes.c_float(thr))
        return out

    @staticmethod
    def median(img, radius=1):
        img = _f32(img)
        h, w = img.shape
        out = np.empty_like(img)
        lib().orc_median(_p(img), _p(out), w, h, radius)
        return out


# ---------------------------------------------------------------- PFM + ref binaries

def write_pfm(path, a):
    """Single-band little-endian PFM in iio's convention: rows in memory order, NO vertical
    flip (iio.c:2049-2071 reads and :3124-3137 writes the raster as is)."""
    a = _f32(a)
    h, w = a.shape
    with open(path, "wb") as f:
        f.write(b"Pf\n%d %d\n-1.0\n" % (w, h))
        f.write(a.tobytes())


def read_pfm(path):
    with open(path, "rb") as f:
        assert f.readline().strip() == b"Pf"
        w, h = map(int, f.readline().split())
        scale = float(f.readline())
        a = np.frombuffer(f.read(), dtype="<f4" if scale < 0 else ">f4").reshape(h, w)
    return np.ascontiguousarray(a).astype(np.float32)


def have_ref():
    return os.access(os.path.join(REF_DIR, "mgm"), os.X_OK)


def _env(params, threads):
    e = os.environ.copy()
    e["OMP_NUM_THREADS"] = str(threads)
    e["CENSUS_NCC_WIN"] = str(params.census_win)
    e["TSGM"] = str(params.tsgm)
    e["TESTLRRL"] = str(params.lr_mode)
    e["TESTLRRL_TAU"] = repr(float(params.lr_tau))
    e["MINDIFF"] = str(int(params.mindiff)) if params.mindiff < 0 else repr(float(params.mindiff))
    e["MEDIAN"] = str(params.median)
    e["REMOVESMALLCC"] = str(params.remove_small_cc)
    e["SUBPIX"] = str(params.subpix)
    e["TSGM_FIX_OVERCOUNT"] = str(params.fix_overcount)
    return e


_REFINE = {0: "none", 1: "vfit", 2: "parabola"}


def run_ref(im1, im2, dmin, dmax, params, threads=1, extra_env=None, workdir=None, binary=None, wl=None, wr=None, want_pkr=False):
    """Run oracle/_ref/mgm (params.scales < 0) or mgm_multi on in-memory images.
    -> dict(disp, conf, dispR, seconds).  OMP_NUM_THREADS=1 is the parity oracle."""
    import time
    binary = binary or ("mgm" if params.scales < 0 else "mgm_multi")
    exe = os.path.join(REF_DIR, binary)
    tmp = workdir or tempfile.mkdtemp(prefix="s2pb_ref_")
    a, b = os.path.join(tmp, "ref.pfm"), os.path.join(tmp, "sec.pfm")
    d, c, r = (os.path.join(tmp, n) for n in ("disp.pfm", "conf.pfm", "dispR.pfm"))
    write_pfm(a, im1)
    write_pfm(b, im2)
    argv = [exe, "-r", str(int(dmin)), "-R", str(int(dmax))]
    if binary == "mgm_multi":
        argv += ["-S", str(params.scales)]
    argv += ["-s", _REFINE[params.refine], "-t", COSTS[params.cost], "-O", str(params.ndir),
             "-P1", repr(float(params.P1)), "-P2", repr(float(params.P2))]
    if wl is not None and wr is not None:
        pl, pr = os.path.join(tmp, "wl.pfm"), os.path.join(tmp, "wr.pfm")
        write_pfm(pl, wl)
        write_pfm(pr, wr)
        argv += ["-wl", pl, "-wr", pr]
    pk = [os.path.join(tmp, n) for n in ("pkrL.pfm", "pkrR.pfm")]
    if want_pkr:
        argv += ["-confidence_pkrL", pk[0], "-confidence_pkrR", pk[1]]
    argv += ["-confidence_consensusL", c, "-Rd", r, a, b, d]
    env = _env(params, threads)
    if extra_env:
        env.update(extra_env)
    t0 = time.perf_counter()
    subprocess.run(argv, env=env, check=True, stdout=subprocess.DEVNULL, cwd=tmp)
    dt = time.perf_counter() - t0
    out = dict(disp=read_pfm(d), conf=read_pfm(c), dispR=read_pfm(r), seconds=dt, workdir=tmp)
    if want_pkr:
        out["pkrL"], out["pkrR"] = read_pfm(pk[0]), read_pfm(pk[1])
    return out


def have_ref_mask():
    return os.access(os.path.join(REF_DIR, "backflow"), os.X_OK) and os.access(os.path.join(REF_DIR, "plambda"), os.X_OK)


def ref_rejection_mask(disp, im1, im2, workdir=None):
    """create_rejection_mask (s2p/block_matching.py:18-32) with the reference's own programs (oracle/_ref/{plambda,backflow} =
    c/plambda.c, c/backflow.c compiled in place), the same three commands, through PFM files.  -> uint8 0/1 mask."""
    tmp = workdir or tempfile.mkdtemp(prefix="s2pb_mask_")
    d, a, b = (os.path.join(tmp, n) for n in ("disp.pfm", "im1.pfm", "im2.pfm"))
    t1, t2, m = (os.path.join(tmp, n) for n in ("tmp1.pfm", "tmp2.pfm", "mask.pfm"))
    write_pfm(d, disp)
    write_pfm(a, im1)
    write_pfm(b, im2)
    pl, bf = os.path.join(REF_DIR, "plambda"), os.path.join(REF_DIR, "backflow")
    run = lambda argv: subprocess.run(argv, check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    run([pl, d, "x 0 join", "-o", t1])
    run([bf, t1, b, t2])
    run([pl, d, a, t2, "x isfinite y isfinite z isfinite and and vmul", "-o", m])
    out = read_pfm(m)
    assert np.all((out == 0) | (out == 1))
    return out.astype(np.uint8)


def read_costvolume_dump(path):
    """DUMP_COSTVOLUME=1 format (mgm_costvolume.cc:222-234): int nx, ny, ndisp, dmin; floats."""
    with open(path, "rb") as f:
        nx, ny, nd, dmin = np.frombuffer(f.read(16), np.int32)
        vol = np.frombuffer(f.read(), np.float32).reshape(ny, nx, nd)
    return vol, int(dmin)


def run_ref_homography(src, H, w, h, binary="homography_ref", workdir=None):
    """Run the reference resampler (oracle/_ref/homography_ref: the unmodified LibHomography sources behind
    oracle/homography_harness.cpp) on an in-memory image.  -> float32 (h, w) array."""
    exe = os.path.join(REF_DIR, binary)
    tmp = workdir or tempfile.mkdtemp(prefix="s2pb_hom_")
    a, b = os.path.join(tmp, "src.pfm"), os.path.join(tmp, "out.pfm")
    write_pfm(a, src)
    hs = " ".join(repr(float(x)) for x in np.asarray(H, dtype=np.float64).ravel())
    subprocess.run([exe, a, hs, b, str(int(w)), str(int(h))], check=True, stdout=subprocess.DEVNULL)
    return read_pfm(b)


def have_ref_homography():
    return os.access(os.path.join(REF_DIR, "homography_ref"), os.X_OK)


def ref_disk_erosion(mask, radius=2.0):
    """The reference's `morsi diskR erosion` (oracle/_ref/libmorsi_ref.so = c/morsi.c compiled in place)."""
    L = ctypes.CDLL(os.path.join(REF_DIR, "libmorsi_ref.so"))
    x = _f32(mask)
    h, w = x.shape
    y = np.empty_like(x)
    rc = L.s2pb_ref_disk_erosion(_p(y), _p(x), w, h, ctypes.c_float(radius))
    if rc:
        raise ValueError("radius must be > 1")
    return y


def have_ref_morsi():
    return os.path.exists(os.path.join(REF_DIR, "libmorsi_ref.so"))


def ref_disp_to_lonlatalt(disp, mask_rect, mask_orig, H1, H2, rpc1, rpc2, img_bbx):
    """The reference's lib/disp_to_h.so entry point (oracle/_ref/libdisp_to_h_ref.so = c/disp_to_h.c + c/rpc.c
    compiled in place), called the way s2p/triangulation.py:118-143 calls it."""
    L = ctypes.CDLL(os.path.join(REF_DIR, "libdisp_to_h_ref.so"))
    dispx = _f32(disp)
    h, w = dispx.shape
    dispy = np.zeros((h, w), np.float32)
    msk, mo = _f32(mask_rect), _f32(mask_orig)
    hh, ww = mo.shape
    out = np.zeros((h, w, 3), np.float64)
    err = np.zeros((h, w), np.float32)
    Ha = np.ascontiguousarray(np.asarray(H1, np.float64).reshape(9))
    Hb = np.ascontiguousarray(np.asarray(H2, np.float64).reshape(9))
    bb = np.ascontiguousarray(np.asarray(img_bbx, np.float32).reshape(4))
    L.disp_to_lonlatalt(_p(out, ctypes.c_double), _p(err), _p(dispx), _p(dispy), _p(msk), w, h, _p(mo), ww, hh,
                        _p(Ha, ctypes.c_double), _p(Hb, ctypes.c_double), ctypes.byref(rpc1), ctypes.byref(rpc2), _p(bb))
    return out, err


def have_ref_triangulation():
    return os.path.exists(os.path.join(REF_DIR, "libdisp_to_h_ref.so"))


# ---------------------------------------------------------------- recorded outputs of the reference programs
#
# Where oracle/_ref is built, the reference programs run live.  Elsewhere (oracle/_ref needs the reference's sources) the
# comparisons use what those programs produced when their outputs were recorded, keyed by a digest of the program, its
# arguments and its inputs:
#   tests/golden/ref_outputs.json   per call, a digest of every output (the bit-exact comparisons)
#   tests/golden/ref_samples.npz    per call and output, the NaN mask and the values on a fixed, seeded sample of pixels (the
#                                   comparisons with a tolerance)
# S2PB_RECORD_REF=1 with oracle/_ref built rewrites the entries of the calls that run.

GOLDEN = os.path.join(os.path.dirname(HERE), "tests", "golden")
RECORDED = os.path.join(GOLDEN, "ref_outputs.json")
RECORDED_SAMPLES = os.path.join(GOLDEN, "ref_samples.npz")
SAMPLE = 512
_recorded_db = None


def digest(a):
    """Digest of an array's values with every NaN alike and -0 == +0: equal digests <=> tests/util.same."""
    a = np.ascontiguousarray(a)
    if a.dtype.kind == "f":
        a = np.where(np.isnan(a), np.nan, a + a.dtype.type(0)).astype(a.dtype)
    return hashlib.sha256(("%s%s" % (a.dtype.str, a.shape)).encode() + a.tobytes()).hexdigest()[:32]


def call_key(program, args, inputs):
    h = hashlib.sha256(repr((program, args)).encode())
    for x in inputs:
        h.update(digest(x).encode())
    return "%s:%s" % (program, h.hexdigest()[:24])


def params_tuple(params):
    return tuple(getattr(params, f) for f, _ in params._fields_)


def _db():
    global _recorded_db
    if _recorded_db is None:
        exact = json.load(open(RECORDED)) if os.path.exists(RECORDED) else {}
        samples = dict(np.load(RECORDED_SAMPLES)) if os.path.exists(RECORDED_SAMPLES) else {}
        _recorded_db = (exact, samples)
    return _recorded_db


def _missing(key):
    return LookupError("no recorded output of the reference for %s (record it where oracle/_ref is built: S2PB_RECORD_REF=1)" % key)


def recorded(key, live):
    """live: a callable running the reference -> {name: array}, or None when the program is not built.
    -> {name: digest} (compare with digest(ours))."""
    exact, _ = _db()
    if live is None:
        if key not in exact:
            raise _missing(key)
        return exact[key]
    out = {k: digest(v) for k, v in live().items()}
    if os.environ.get("S2PB_RECORD_REF") == "1":
        exact[key] = out
        merged = json.load(open(RECORDED)) if os.path.exists(RECORDED) else {}     # (other processes may have recorded too)
        merged[key] = out
        with open(RECORDED, "w") as f:
            json.dump(merged, f, indent=0, sort_keys=True)
    return out


class Sampled:
    """A reference output kept as its NaN mask and its values on a fixed sample of pixels (all pixels when run live)."""

    def __init__(self, shape, nan, idx, val):
        self.shape, self.nan, self.idx, self.val = tuple(shape), nan, idx, val

    def values_of(self, ours):
        """ours, flattened over the pixels (a trailing axis of another shape is kept), at the sampled pixels"""
        ours = np.asarray(ours)
        npix = int(np.prod(self.nan.shape))
        return ours.reshape(npix, -1)[self.idx].reshape((len(self.idx),) + ours.shape[self.nan.ndim:])


def recorded_sampled(key, live):
    """As recorded(), for the comparisons with a tolerance: -> {name: Sampled}.  The NaN mask is over the first two axes."""
    _, samples = _db()
    if live is not None:
        out = {}
        for k, v in live().items():
            v = np.asarray(v)
            nan = np.isnan(v) if v.ndim == 2 else np.isnan(v).any(axis=tuple(range(2, v.ndim)))
            npix = nan.size
            out[k] = Sampled(v.shape, nan, np.arange(npix), v.reshape((npix,) + v.shape[2:]))
            if os.environ.get("S2PB_RECORD_REF") == "1":
                idx = np.sort(np.random.default_rng(0).choice(npix, min(SAMPLE, npix), replace=False))
                samples["%s/%s/shape" % (key, k)] = np.array(v.shape)
                samples["%s/%s/nan" % (key, k)] = np.packbits(nan.ravel())
                samples["%s/%s/idx" % (key, k)] = idx
                samples["%s/%s/val" % (key, k)] = v.reshape((npix,) + v.shape[2:])[idx]
        if os.environ.get("S2PB_RECORD_REF") == "1":
            np.savez_compressed(RECORDED_SAMPLES, **samples)
        return out
    names = sorted({n.split("/")[-2] for n in samples if n.startswith(key + "/")})
    if not names:
        raise _missing(key)
    out = {}
    for k in names:
        g = lambda f: samples["%s/%s/%s" % (key, k, f)]
        shape = tuple(int(s) for s in g("shape"))
        nan = np.unpackbits(g("nan"))[:shape[0] * shape[1]].reshape(shape[:2]).astype(bool)
        out[k] = Sampled(shape, nan, g("idx"), g("val"))
    return out


def ref_mgm_outputs(im1, im2, dmin, dmax, params, wl=None, wr=None, want_pkr=False, binary=None):
    """run_ref at OMP_NUM_THREADS=1, live or recorded -> {disp, conf, dispR[, pkrL, pkrR]: digest}"""
    binary = binary or ("mgm" if params.scales < 0 else "mgm_multi")
    ins = [im1, im2] + ([wl, wr] if wl is not None else [])
    key = call_key(binary, (int(dmin), int(dmax), params_tuple(params), want_pkr), ins)
    names = ("disp", "conf", "dispR") + (("pkrL", "pkrR") if want_pkr else ())
    live = None
    if os.access(os.path.join(REF_DIR, binary), os.X_OK):
        def live():
            r = run_ref(im1, im2, dmin, dmax, params, threads=1, binary=binary, wl=wl, wr=wr, want_pkr=want_pkr)
            return {k: r[k] for k in names}
    return recorded(key, live)


def ref_homography_sampled(src, H, w, h):
    """run_ref_homography, live or recorded -> Sampled"""
    key = call_key("homography", (tuple(np.asarray(H, np.float64).ravel().tolist()), int(w), int(h)), [src])
    return recorded_sampled(key, (lambda: {"out": run_ref_homography(src, H, w, h)}) if have_ref_homography() else None)["out"]


def ref_disp_to_lonlatalt_sampled(disp, mask_rect, mask_orig, H1, H2, rpc1, rpc2, img_bbx):
    """ref_disp_to_lonlatalt, live or recorded -> (Sampled lon/lat/alt, Sampled reprojection error)"""
    rpcs = tuple(bytes(r).hex() for r in (rpc1, rpc2))
    args = (tuple(np.asarray(H1, np.float64).ravel().tolist()), tuple(np.asarray(H2, np.float64).ravel().tolist()), rpcs,
            tuple(float(x) for x in img_bbx))
    key = call_key("disp_to_lonlatalt", args, [disp, mask_rect, mask_orig])
    live = None
    if have_ref_triangulation():
        def live():
            out, err = ref_disp_to_lonlatalt(disp, mask_rect, mask_orig, H1, H2, rpc1, rpc2, img_bbx)
            return {"lonlatalt": out, "err": err}
    r = recorded_sampled(key, live)
    return r["lonlatalt"], r["err"]


def ref_rejection_mask_output(disp, im1, im2):
    """ref_rejection_mask, live or recorded -> digest of the mask"""
    key = call_key("plambda+backflow", (), [disp, im1, im2])
    return recorded(key, (lambda: {"mask": ref_rejection_mask(disp, im1, im2)}) if have_ref_mask() else None)["mask"]
