"""Fuzz the CUDA matcher (through the C ABI) against the CPU oracle on random shapes, ranges and parameters:
mgm and mgm_multi, every distance, weights, MINDIFF, all refinements.  Needs an H100.
usage: python scripts/fuzz_gpu.py [N] [seed]"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from oracle import oracle as O
from s2p_b200.engine import Engine, default_params
from s2p_b200.synth import make_pair

N = int(sys.argv[1]) if len(sys.argv) > 1 else 50
rng = np.random.default_rng(int(sys.argv[2]) if len(sys.argv) > 2 else 0)
eng = Engine(0)


def differ(a, b):
    return int((~((a == b) | (np.isnan(a) & np.isnan(b)))).sum())


bad = 0
for it in range(N):
    multi = rng.random() < 0.3
    h, w = (int(rng.integers(101, 150)), int(rng.integers(101, 200))) if multi else (int(rng.integers(2, 70)), int(rng.integers(2, 300)))
    dmin = int(rng.integers(-200, 50))
    dmax = dmin + int(rng.integers(1, min(700 if it % 7 == 0 else 480, max(2, 3 * w))))      # every 7th case may exceed 512 labels
    kw = dict(ndir=int(rng.choice([2, 4, 8])), tsgm=int(rng.integers(1, 5)), census_win=int(rng.choice([3, 5, 7])),
              P1=float(rng.choice([8.0, 12.0, 5.5])), P2=float(rng.choice([32.0, 48.0, 41.0])), median=int(rng.integers(0, 3)),
              lr_mode=int(rng.integers(0, 2)), refine=int(rng.choice([0, 1, 1, 2])), cost=int(rng.choice([0, 0, 0, 1, 2, 3, 4, 5])),
              mindiff=float(rng.choice([-1.0, -1.0, 1.0])))
    nanb = float(rng.choice([0.0, 0.0, 0.05]))
    if multi:
        kw.update(subpix=int(rng.choice([1, 2])), scales=int(rng.choice([1, 3, 6])), remove_small_cc=int(rng.choice([0, 25])),
                  lr_mode=int(rng.integers(0, 3)))
        if dmax - dmin > 200:
            dmax = dmin + 200
    ref, sec, _ = make_pair(h, w, dmin, dmax, seed=int(rng.integers(1 << 30)), nan_border=nanb)
    wts = None
    if rng.random() < 0.4:
        def wt():
            x = rng.uniform(0, 255, (h, w))
            a = np.maximum(((255 - x) / 255) ** 2, 0.1).astype(np.float32)
            a[rng.random((h, w)) < 0.6] = 1.0
            return a
        wts = (wt(), wt())
    P = (O.mgm_multi_params if multi else O.mgm_params)(**kw)
    d, c, dr = (O.port.mgm_multi if multi else O.port.mgm)(ref, sec, dmin, dmax, P, *(wts or (None, None)))
    try:
        # timeout_ms: a deadlocked persistent kernel is drained through the abort flag instead of hanging the box
        out = eng.mgm(ref, sec, dmin, dmax, default_params("mgm_multi" if multi else "mgm", timeout_ms=20000, **kw), want_right=True,
                      weights=wts)
    except Exception as e:
        print(it, "engine refused:", e, (h, w), dmin, dmax, kw, flush=True)
        continue
    n = (differ(out["disp"], d), differ(out["conf"], c), differ(out["disp_right"], dr))
    ok = not any(n)                       # bit-exact everywhere, the half-pixel pass of mgm_multi included (round 2)
    if not ok:
        bad += 1
    if any(n):
        print(it, "DIFF" if ok else "MISMATCH", n, "multi" if multi else "mgm", (h, w), dmin, dmax, kw, "weights" if wts else "", "nan", nanb, flush=True)
print("done: %d cases, %d failing" % (N, bad))
