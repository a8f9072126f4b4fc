"""Timing of the engine's `sgbm` matcher on a seeded 1024 x 1024 tile with 128 labels (s2p's `-100 28 3 8 32 1`):
host-to-host time of Engine.sgbm (images in host memory, disparity and mask back), the per-kernel breakdown from
torch.profiler in a separate run, and the reference binary (oracle/_ref/sgbm, one host core, MALLOC_PERTURB_=255) on the same
tile, whose output must be identical.  Prints one JSON line (and writes it to --out).

    python scripts/sgbm_probe.py [--size 1024] [--dmin -100] [--dmax 28] [--reps 10] [--out PATH]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clk = [s.strip() for s in q.split(",")]
        return dict(gpu=name, power_limit=power, max_sm_clock=clk)
    except Exception as e:                      # the timing stands without it, but says so
        return dict(gpu="unknown (%s)" % e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--dmin", type=int, default=-100)
    ap.add_argument("--dmax", type=int, default=28)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()

    from s2p_b200.engine import Engine
    from s2p_b200.synth import make_pair
    import sgbm_oracle as SO
    n = a.size
    im1, im2, _ = make_pair(n, n, a.dmin, a.dmax, seed=3, nan_border=0.02)
    res = dict(tile="%dx%d" % (n, n), dmin=a.dmin, dmax=a.dmax, labels=(a.dmax - a.dmin + 15) // 16 * 16, **gpu_info())
    with Engine(0) as eng:
        p = eng.sgbm_params()
        out = eng.sgbm(im1, im2, a.dmin, a.dmax, p)            # warm-up: module load, pooled buffers
        ts = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            out = eng.sgbm(im1, im2, a.dmin, a.dmax, p)
            ts.append(time.perf_counter() - t0)
        res["host_to_host_ms"] = dict(median=1e3 * float(np.median(ts)), min=1e3 * min(ts), max=1e3 * max(ts), reps=a.reps)
        res["valid_fraction"] = float(np.isfinite(out["disp"]).mean())
        try:
            import torch
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(3):
                    eng.sgbm(im1, im2, a.dmin, a.dmax, p)
                torch.cuda.synchronize()
            per = {}
            for ev in prof.events():
                if ev.device_type.name == "CUDA":
                    k = ev.name.split("(")[0].replace("void s2pb::", "").replace("s2pb::", "")
                    per[k] = per.get(k, 0.0) + ev.device_time / 1e3 / 3
            res["kernel_ms"] = {k: round(v, 3) for k, v in sorted(per.items(), key=lambda kv: -kv[1])}
            res["kernel_total_ms"] = round(sum(v for k, v in per.items() if "Memcpy" not in k and "Memset" not in k), 3)
        except Exception as e:
            res["kernel_ms"] = "profiler unavailable: %s" % e
    if SO.have_ref():
        r = SO.run_ref(im1, im2, a.dmin, a.dmax)
        res["reference_s"] = r["seconds"]
        res["identical_to_reference"] = bool(np.array_equal(np.isnan(r["disp"]), np.isnan(out["disp"])) and
                                             np.array_equal(r["disp"][np.isfinite(r["disp"])], out["disp"][np.isfinite(out["disp"])]))
        res["speedup_vs_reference"] = r["seconds"] / (res["host_to_host_ms"]["median"] / 1e3)
    else:
        res["reference_s"] = "not measured (oracle/_ref/sgbm not built)"
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
