"""TEST INFRASTRUCTURE ONLY -- what the engine's `sgbm` matcher is checked against:

* the reference binary oracle/_ref/sgbm (3rdparty/sgbm compiled in place by oracle/sgbm.mk), run with
  MALLOC_PERTURB_=255 so that the never-initialised margins of its crop trick are zero, live where it is built;
* otherwise the digests of its outputs recorded in tests/golden/sgbm_ref_outputs.json (S2PB_RECORD_REF=1 with the binary
  built rewrites the entries that run);
* a numpy restatement of its qauto thresholds;
* the seeded tiles the tests use.
"""
import json
import os
import re
import subprocess
import tempfile
import time

import numpy as np

from oracle import oracle as O
from s2p_b200.synth import make_pair

REF_BIN = os.path.join(O.REF_DIR, "sgbm")
RECORDED = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sgbm_ref_outputs.json")
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def have_ref():
    return os.access(REF_BIN, os.X_OK)


def run_ref(im1, im2, dmin, dmax, win=3, P1=8, P2=32, lr=1, perturb="255"):
    """`sgbm im1 im2 disp cost dmin dmax win P1 P2 lr` -> dict(disp, rminmax, seconds).  perturb=None: plain malloc."""
    tmp = tempfile.mkdtemp(prefix="s2pb_sgbm_")
    a, b, d, c = (os.path.join(tmp, n) for n in ("im1.pfm", "im2.pfm", "disp.pfm", "cost.pfm"))
    O.write_pfm(a, im1)
    O.write_pfm(b, im2)
    env = os.environ.copy()
    env.pop("MALLOC_PERTURB_", None)
    if perturb is not None:
        env["MALLOC_PERTURB_"] = perturb
    t0 = time.perf_counter()
    r = subprocess.run([REF_BIN, a, b, d, c] + [str(int(v)) for v in (dmin, dmax, win, P1, P2, lr)], env=env,
                       check=True, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, cwd=tmp)
    dt = time.perf_counter() - t0
    m = re.search(r"qauto: rminmax = (\S+) (\S+)", r.stderr.decode())
    out = dict(disp=O.read_pfm(d), rminmax=(float(m.group(1)), float(m.group(2))), seconds=dt)
    for f in os.listdir(tmp):
        os.remove(os.path.join(tmp, f))
    os.rmdir(tmp)
    return out


def qauto_thresholds(x):
    """numpy restatement of get_rminmax (sgbm.cpp:30-42)"""
    t = np.sort(np.asarray(x, np.float32)[~np.isnan(x)].ravel())
    rb = t.size // 200
    return float(t[rb]), float(t[t.size - 1 - rb])


# ---------------------------------------------------------------- the seeded cases

def _pair(h, w, dmin, dmax, seed, nan_border=0.0):
    a, b, _ = make_pair(h, w, dmin, dmax, seed=seed, nan_border=nan_border)
    return a, b


def _speckled(h, w, seed):
    """texture with flat patches and small islands: the speckle and uniqueness filters both fire"""
    a, b = _pair(h, w, -12, 4, seed)
    rng = np.random.default_rng(seed + 7)
    for _ in range(12):
        y, x = rng.integers(0, h - 8), rng.integers(0, w - 8)
        a[y:y + 6, x:x + 6] = a[y, x]
        b[y:y + 6, x:x + 6] = b[y, x]
    a[h // 3:h // 3 + 20, :] = np.float32(a.mean())
    b[h // 3:h // 3 + 20, :] = np.float32(a.mean())
    return a, b


def _real():
    z = np.load(os.path.join(GOLD, "real_inputs.npz"))
    return z["ref"], z["sec"]


# name -> (im1, im2 factory, dmin, dmax, win, P1, P2, lr)
CASES = {
    "base_96x160": (lambda: _pair(96, 160, -20, 12, 0), -20, 12, 3, 8, 32, 1),
    "odd_37x61": (lambda: _pair(37, 61, -9, 6, 1), -9, 6, 3, 8, 32, 1),
    "three_rows": (lambda: _pair(3, 80, -5, 5, 2), -5, 5, 3, 8, 32, 1),
    "three_rows_win7": (lambda: _pair(3, 70, -5, 5, 3), -5, 5, 7, 8, 32, 1),
    "narrow_3": (lambda: _pair(40, 3, -3, 3, 4), -3, 3, 3, 8, 32, 1),
    "all_negative": (lambda: _pair(64, 120, -30, -10, 5), -30, -10, 3, 8, 32, 1),
    "all_positive": (lambda: _pair(64, 120, 8, 27, 6), 8, 27, 3, 8, 32, 1),
    "straddle_not16": (lambda: _pair(72, 130, -7, 13, 7), -7, 13, 3, 8, 32, 1),
    "exact16": (lambda: _pair(50, 90, -8, 8, 8), -8, 8, 3, 8, 32, 1),
    "win1": (lambda: _pair(60, 100, -10, 10, 9), -10, 10, 1, 8, 32, 1),
    "win5_p": (lambda: _pair(60, 100, -10, 10, 10), -10, 10, 5, 20, 90, 1),
    "win7": (lambda: _pair(60, 100, -10, 10, 11), -10, 10, 7, 8, 32, 1),
    "lr0": (lambda: _pair(60, 100, -10, 10, 12), -10, 10, 3, 8, 32, 0),
    "lr3": (lambda: _pair(60, 100, -10, 10, 12), -10, 10, 3, 8, 32, 3),
    "p_default_rule": (lambda: _pair(60, 100, -10, 10, 13), -10, 10, 3, 0, 0, 1),
    "nan_border": (lambda: _pair(80, 120, -15, 9, 14, nan_border=0.1), -15, 9, 3, 8, 32, 1),
    "constant": (lambda: (np.full((40, 70), 17.5, np.float32), np.full((40, 70), 17.5, np.float32)), -6, 6, 3, 8, 32, 1),
    "speckle": (lambda: _speckled(90, 140, 15), -12, 4, 3, 8, 32, 1),
    "real_inputs": (_real, -20, 20, 3, 8, 32, 1),
}


def case(name):
    f, dmin, dmax, win, P1, P2, lr = CASES[name]
    a, b = f()
    return np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32), dmin, dmax, win, P1, P2, lr


_db = None


def ref_digests(name):
    """-> dict(disp, mask digests, rminmax) of the reference on case `name`: live where oracle/_ref is built, else recorded."""
    global _db
    if _db is None:
        _db = json.load(open(RECORDED)) if os.path.exists(RECORDED) else {}
    if not (have_ref() and O.have_ref_mask()):
        if name not in _db:
            raise LookupError("no recorded output of the reference for %s (record it where oracle/_ref is built: S2PB_RECORD_REF=1)" % name)
        return _db[name]
    a, b, dmin, dmax, win, P1, P2, lr = case(name)
    r = run_ref(a, b, dmin, dmax, win, P1, P2, lr)
    out = dict(disp=O.digest(r["disp"]), mask=O.digest(O.ref_rejection_mask(r["disp"], a, b)), rminmax=list(r["rminmax"]),
               valid=int(np.isfinite(r["disp"]).sum()))
    if os.environ.get("S2PB_RECORD_REF") == "1" and _db.get(name) != out:
        _db[name] = out
        merged = json.load(open(RECORDED)) if os.path.exists(RECORDED) else {}
        merged[name] = out
        with open(RECORDED, "w") as f:
            json.dump(merged, f, indent=0, sort_keys=True)
    return out
