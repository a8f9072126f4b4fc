"""Stage timings of the matcher per census window (census_ncc_win), on the C2 shape: one 1024 x 1024 tile, 128 labels.

For `mgm` at win 5, 7, 9 and 11 it prints the medians over the timed calls of the s2pb_last_timings stages (census, cost,
aggregate, WTA, total; device events); for `mgm_multi` at 9, which records no stage events, the host wall time of a call that
ends in a device synchronisation.  The census and the cost grow with the window (9 and 11 carry a second 64-bit code word);
the aggregation and the WTA read the same 8-bit cost codes whatever the window.

    python scripts/census_window_probe.py [--iters 10] [--warmup 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from s2p_b200.engine import Engine, default_params  # noqa: E402
from s2p_b200.synth import make_pair  # noqa: E402

STAGES = ("census", "cost", "aggregate", "wta", "total")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # pragma: no cover
        q = "unknown (%s)" % e
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--size", type=int, default=1024)
    a = ap.parse_args()
    n, dmin, dmax = a.size, -64, 63
    ref, sec, _ = make_pair(n, n, dmin, dmax, seed=0)
    print(json.dumps({"card": card(), "shape": [n, n], "labels": dmax - dmin + 1}), flush=True)
    with Engine(0) as eng:
        for algo, win in [("mgm", 5), ("mgm", 7), ("mgm", 9), ("mgm", 11), ("mgm_multi", 9)]:
            p = default_params(algo, census_win=win)
            rows, wall = [], []
            for it in range(a.warmup + a.iters):
                t = time.perf_counter()
                eng.mgm(ref, sec, dmin, dmax, p)
                dt = (time.perf_counter() - t) * 1e3
                if it < a.warmup:
                    continue
                wall.append(dt)
                if algo == "mgm":
                    rows.append(eng.last_timings())
            res = {"algo": algo, "win": win, "wall_ms": round(float(np.median(wall)), 3)}
            for s in STAGES:
                vals = [r[k] for r in rows for k in r if k.startswith(s)]
                if vals:
                    res[s + "_ms"] = round(float(np.median(vals)), 3)
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
