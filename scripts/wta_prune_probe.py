#!/usr/bin/env python3
"""The WTA stage of one C2 tile (1024 x 1024, 128 labels) alone on the device, without and with pruning (DESIGN.md 3.2, 6).

The library records CUDA events around the two WTA launches of a tile (left and right view); this script runs the tile serially,
nothing else on the device, N times after a warm-up, with S2PB_WTA_PRUNE=0 and unset (the default) in turn, twice (the switch is
read when the context is created), and sets the bytes the kernel requests -- the sector fractions of scripts/wta_prune_model.py
on a strip of the same pair -- against the time.  Prints the card's name, power limit and SM clock from the same process.

    python scripts/wta_prune_probe.py [--n 20] [--nan-border 0.05]
"""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=20)
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--nan-border", type=float, default=0.0)
    a = ap.parse_args()
    import wta_prune_model as M
    from s2p_b200.engine import Engine, default_params
    from s2p_b200.synth import make_pair
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("device:", q.stdout.strip() or q.stderr.strip())
    dmin, dmax = -64, 63
    ref, sec, _ = make_pair(a.size, a.size, dmin, dmax, seed=0, nan_border=a.nan_border)
    npix = a.size * a.size
    nbytes = {"0": 0.0, "default": 0.0}
    for view in "LR":
        C, S = M.strip_volumes(0, a.size, (300, 396), dmin, dmax, a.nan_border, view)
        DP = C.shape[-1]
        full = npix * (8 * 4 * DP + DP)
        nbytes["0"] += full
        if DP % 32 or DP // 32 not in (1, 2, 4, 8):          # interleaved labels per lane: wta_kernel serves the view
            nbytes["default"] += full
            print("view %s: %d slots, not pruned" % (view, DP))
            continue
        f2, _ = M.two_stage_fractions(C, S)
        nbytes["default"] += M.requested_bytes(npix, DP, f2)
        print("view %s: %d slots, sector fraction per pass %s (mean %.3f)" % (
            view, DP, " ".join("%.3f" % x for x in f2), np.mean(f2)))
    p = default_params("mgm")
    outs = []
    for sw in ("0", "default", "0", "default"):
        if sw == "default":
            os.environ.pop("S2PB_WTA_PRUNE", None)
        else:
            os.environ["S2PB_WTA_PRUNE"] = sw
        eng = Engine(0)
        for _ in range(3):
            out = eng.mgm(ref, sec, dmin, dmax, p, want_right=True)
        t = []
        for _ in range(a.n):
            out = eng.mgm(ref, sec, dmin, dmax, p, want_right=True)
            t.append(eng.last_timings())
        eng.close()
        outs.append(out)
        wta = np.array([x["wta"] for x in t])
        agg = np.array([x["aggregate"] for x in t])
        print("S2PB_WTA_PRUNE %s: wta %.3f ms (min %.3f, max %.3f), aggregate %.3f ms, %.2f GB requested -> %.2f TB/s" % (
            sw, wta.mean(), wta.min(), wta.max(), agg.mean(), nbytes[sw] / 1e9, nbytes[sw] / 1e9 / wta.mean()), flush=True)
    same = all(np.array_equal(outs[0][k].view(np.int32), o[k].view(np.int32)) for o in outs[1:] for k in ("disp", "conf", "disp_right"))
    print("outputs identical:", same)
    return 0 if same else 1


if __name__ == "__main__":
    sys.exit(main())
