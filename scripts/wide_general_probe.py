"""Times one 768x532 mgm_multi_lsd tile with a 256-label range (weights of the LSD kind), and the same tile with the ad
distance, whose half-pixel pass runs the float-cost flavour on a slab wider than 512 slots (the chunk-skipping kernels).
Prints the card, its power limit and the median of the timed calls.
usage: python scripts/wide_general_probe.py [repeats]"""
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from s2p_b200.engine import Engine, default_params
from s2p_b200.synth import make_pair


def weights(shape, seed, ones=0.75):
    rng = np.random.default_rng(seed)
    w = np.maximum(((255 - rng.uniform(0, 255, shape)) / 255) ** 2, 0.1).astype(np.float32)
    w[rng.random(shape) < ones] = 1.0
    return w


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown")
    h, w, dmin, dmax = 532, 768, -128, 127
    ref, sec, _ = make_pair(h, w, dmin, dmax, seed=5, nan_border=0.02)
    wts = (weights((h, w), 1), weights((h, w), 2))
    with Engine(0) as eng:
        for cost in ("census", "ad"):
            p = default_params("mgm_multi_lsd", cost=cost)
            eng.mgm(ref, sec, dmin, dmax, p, weights=wts)          # warm-up: workspaces, module loads
            ts = []
            for _ in range(reps):
                t = time.perf_counter()
                out = eng.mgm(ref, sec, dmin, dmax, p, weights=wts)     # returns host arrays: ends in a device synchronise
                ts.append(time.perf_counter() - t)
            print("mgm_multi_lsd %dx%d, %d labels, cost %s: %.1f ms per tile (median of %d; min %.1f), %.1f %% valid" % (
                w, h, dmax - dmin + 1, cost, 1e3 * statistics.median(ts), reps, 1e3 * min(ts), 100.0 * np.isfinite(out["disp"]).mean()))


if __name__ == "__main__":
    main()
