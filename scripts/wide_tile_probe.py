"""Wide tiles on the device: the DCT tables of rows of 4096 to 16384 px and the matcher on such tiles, with the tables resident and
streamed in K-panels.

For each width: the host build of one n x n table (s2pb_dct_coefficients, on the engine's thread pool) and its upload from pageable
memory; then, for each label count, the wall clock of one `mgm` and one `mgm_multi` call on a seeded tile with no-data borders (so
that the round trip transforms rows), once on an engine that keeps every table resident and once on one that streams every table
of rows wider than 8192 px (up to 8192 px both engines keep the tables resident).  The first call of each engine at a width builds
and uploads its tables and is reported apart; the figures are medians of the calls after it.  Outputs of the two engines are
checked bit for bit.

    python scripts/wide_tile_probe.py [--rows 128] [--labels 64 256] [--widths 4096 8192 12288 16384] [--reps 3] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from s2p_b200.engine import Engine, dct_coefficients, default_params  # noqa: E402
from s2p_b200.synth import make_pair  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def wall(call):
    t = time.perf_counter()
    out = call()               # the engine's host calls return after their stream has synchronised
    return out, 1e3 * (time.perf_counter() - t)


def table_build(n):
    import torch
    _, host_ms = wall(lambda: dct_coefficients(0, n, range(n), range(n)))
    t = dct_coefficients(0, n, range(n), range(n))
    torch.cuda.synchronize()
    s = time.perf_counter()
    d = torch.from_numpy(t).to("cuda")
    torch.cuda.synchronize()
    up_ms = 1e3 * (time.perf_counter() - s)
    del d
    return host_ms, up_ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=128)
    ap.add_argument("--labels", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--widths", type=int, nargs="+", default=[4096, 8192, 12288, 16384])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for wide_tile_probe.json (default: print only)")
    a = ap.parse_args()
    res = dict(card=card(), host_threads=os.cpu_count(), rows=a.rows, widths=[])
    print(res["card"], "host threads", os.cpu_count(), flush=True)
    for w in a.widths:
        host_ms, up_ms = table_build(w)
        row = dict(width=w, table_host_ms=host_ms, table_upload_ms=up_ms, calls=[])
        print("width %d: one table %.0f MiB, host build %.1f ms, upload %.1f ms" % (w, w * w * 8 / 2 ** 20, host_ms, up_ms), flush=True)
        resident, streamed = Engine(0), Engine(0)
        resident.set_dct_table_limit(64 << 30)
        streamed.set_dct_table_limit(0)
        for D in a.labels:
            dmin = -(D // 2)
            dmax = dmin + D - 1
            ref, sec, _ = make_pair(a.rows, w, dmin, dmax, seed=w + D, nan_border=0.02)
            for algo in ("mgm", "mgm_multi"):
                p = default_params(algo)
                rec = dict(algo=algo, labels=D)
                for name, e in (("resident", resident), ("streamed", streamed)):
                    out, first = wall(lambda: e.mgm(ref, sec, dmin, dmax, p, want_right=True))
                    ms = sorted(wall(lambda: e.mgm(ref, sec, dmin, dmax, p, want_right=True))[1] for _ in range(a.reps))
                    rec[name + "_first_ms"], rec[name + "_ms"] = first, ms[len(ms) // 2]
                    rec[name + "_out"] = out
                same = all(np.array_equal(rec["resident_out"][k], rec["streamed_out"][k], equal_nan=True)
                           for k in ("disp", "conf", "mask", "disp_right"))
                del rec["resident_out"], rec["streamed_out"]
                rec["identical"] = bool(same)
                row["calls"].append(rec)
                print("  %-9s %4d labels: resident %.1f ms (first %.1f), streamed %.1f ms (first %.1f), identical %s" % (
                    algo, D, rec["resident_ms"], rec["resident_first_ms"], rec["streamed_ms"], rec["streamed_first_ms"], same),
                    flush=True)
        resident.close()
        streamed.close()
        res["widths"].append(row)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "wide_tile_probe.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
