"""The 3D outlier filter of triangulation (filter_xyz at r = 5 m, n = 50, p = 10, q = 1) on a seeded 1024x1024 UTM-scale
cloud with a few percent outliers and NaN holes: host-to-host time of remove_isolated_3d_points, per-kernel times from a
separate torch.profiler run, the reference library on one host core (when oracle/_ref is built), the card and its power
limit, and whether the two outputs are identical.  One JSON line on stdout; --trace DIR also writes the profiler's table.

    python scripts/pointcloud_probe.py [--reps 50] [--trace DIR]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

from s2p_b200.engine import Engine  # noqa: E402
import pointcloud_oracle as P  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, check=True).stdout.strip().split(", ")
        return q[0], q[1]
    except Exception:
        return "unknown", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--trace", default=None)
    a = ap.parse_args()
    r, n, p, q = 5.0, 50, 10, 1
    xyz = P.utm_cloud(1024, 1024, 8)
    eng = Engine(0)
    out = eng.remove_isolated_3d_points(xyz.copy(), r, p, n, q)             # warm-up (and pooled buffers)
    work = [xyz.copy() for _ in range(a.reps)]
    t = []
    for w in work:
        t0 = time.perf_counter()
        eng.remove_isolated_3d_points(w, r, p, n, q)                         # synchronous: returns with the host array written
        t.append(time.perf_counter() - t0)
    t = np.array(t) * 1e3
    tc = []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        eng.count_3d_neighbors(xyz, r, p)
        tc.append(time.perf_counter() - t0)
    tc = np.array(tc) * 1e3

    import torch
    from torch.profiler import ProfilerActivity, profile
    w = xyz.copy()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            w[...] = xyz
            eng.remove_isolated_3d_points(w, r, p, n, q)
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.key_averages():
        dt = getattr(e, "device_time_total", None)
        if dt is None:
            dt = e.cuda_time_total
        if dt > 0 and e.count > 0:
            kernels[e.key[:80]] = round(dt / e.count / 1e3, 4)               # ms per call
    if a.trace:
        os.makedirs(a.trace, exist_ok=True)
        with open(os.path.join(a.trace, "pointcloud_profile.txt"), "w") as f:
            f.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=30))

    res = {"workload": "remove_isolated_3d_points, 1024x1024 UTM-scale cloud, r=5 n=50 p=10 q=1",
           "gpu_host_to_host_ms": {"median": round(float(np.median(t)), 3), "min": round(float(t.min()), 3),
                                   "max": round(float(t.max()), 3), "reps": a.reps},
           "gpu_count_host_to_host_ms": {"median": round(float(np.median(tc)), 3), "min": round(float(tc.min()), 3)},
           "kernel_ms_per_call": kernels, "card": card()[0], "power_limit": card()[1],
           "removed_points": int((np.isnan(out).any(axis=2) & ~np.isnan(xyz).any(axis=2)).sum())}
    if P.have_ref():
        os.environ["OMP_NUM_THREADS"] = "1"
        t0 = time.perf_counter()
        ref = P.ref_remove_isolated_3d_points(xyz, r, p, n, q)
        res["reference_one_core_s"] = round(time.perf_counter() - t0, 3)
        t0 = time.perf_counter()
        refc = P.ref_count_3d_neighbors(xyz, r, p)
        res["reference_count_one_core_s"] = round(time.perf_counter() - t0, 3)
        from oracle.oracle import digest
        res["identical_to_reference"] = digest(ref) == digest(out) and all(digest(x) == digest(ref) for x in work)
        res["counts_identical_to_reference"] = bool(np.array_equal(refc, eng.count_3d_neighbors(xyz, r, p)))
    else:
        res["reference_one_core_s"] = "not measured (oracle/_ref is not built)"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
