"""height_map_to_xyz into UTM on the shape s2p gives it: a 1024x1024 merged height map in the frame of the reference's
triplet camera (img_02.tif's RPCs, from tests/golden/triplet.npz, ground->image polynomials only, so every pixel runs the
iteration of c/rpc.c:378-411), seeded about the camera's height offset with a few percent NaN, localised and projected to
EPSG:32631.

Times, host buffers in and out, each call ending in a device synchronise, median of --reps after a warm-up:
  * `height_map_to_xyz` with zone 31 north: localisation and projection in one device call;
  * the same with zone 0 (lon, lat, alt);
  * the numpy float64 restatement of the localisation (tests/localization_oracle.py) and of the projection
    (tests/utm_oracle.py) on one host core, once.  It stands in for the reference's host path (rpcm's localisation, then
    pyproj), which is not installed here: the reference's own time is not measured.
Compares the GPU cloud with the restatement on the same inputs, and reads the card and its power limit in the same run.
One JSON line on stdout.

    python scripts/height_map_to_xyz_probe.py [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

os.environ.setdefault("OMP_NUM_THREADS", "1")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import localization_oracle as LO  # noqa: E402
import utm_oracle as U  # noqa: E402
from s2p_b200.engine import Engine  # noqa: E402

ZONE, SOUTH = 31, False


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, check=True).stdout.strip().split(", ")
        return q[0], q[1]
    except Exception:
        return "unknown", "unknown"


def inputs(side, seed=0, nan_fraction=0.03):
    rpc = LO.triplet_rpc()
    rng = np.random.default_rng(seed)
    z = (rpc.offset[2] + rng.normal(0.0, 30.0, (side, side))).astype(np.float32)
    z[rng.random((side, side)) < nan_fraction] = np.nan
    return z, rpc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--side", type=int, default=1024)
    a = ap.parse_args()
    z, rpc = inputs(a.side)
    eng = Engine(0)
    utm_call = lambda: eng.height_map_to_xyz(z, rpc, 0, 0, ZONE, SOUTH)
    lla_call = lambda: eng.height_map_to_xyz(z, rpc, 0, 0)
    xyz = utm_call()                                                       # warm-up: module load, pooled buffers
    lla = lla_call()

    def timed(fn, reps):
        t = []
        for _ in range(reps):
            t0 = time.perf_counter()
            fn()                                                           # synchronous: returns with the results on the host
            t.append(time.perf_counter() - t0)
        return np.array(t) * 1e3

    t_utm = timed(utm_call, a.reps)
    t_lla = timed(lla_call, a.reps)
    ok = ~np.isnan(z)
    rows, cols = np.nonzero(ok)
    t0 = time.perf_counter()
    lon, lat, converged = LO.localize(rpc, cols, rows, z[ok])
    t_loc = time.perf_counter() - t0
    host = np.full(z.shape + (3,), np.nan)
    host[ok] = np.column_stack([lon, lat, z[ok].astype(np.float64)])
    t0 = time.perf_counter()
    host_utm = U.restate(host, ZONE, SOUTH)
    t_proj = time.perf_counter() - t0
    name, power = card()
    med = lambda t: round(float(np.median(t)), 3)
    res = {"workload": "height_map_to_xyz %dx%d to EPSG:32631, host buffers in and out" % (a.side, a.side),
           "points": int(z.size), "valid_points": int(ok.sum()),
           "height_map_to_xyz_utm_ms": med(t_utm),
           "height_map_to_xyz_lonlat_ms": med(t_lla),
           "numpy_restatement_one_core_ms": round((t_loc + t_proj) * 1e3, 1),
           "numpy_restatement_note": "stand-in for rpcm localisation + pyproj on one core; the reference itself: not measured",
           "reps": a.reps,
           "restatement_converged": bool(converged.all()),
           "same_nan_mask": bool(np.array_equal(np.isnan(xyz), np.isnan(host_utm))),
           "max_abs_dlonlat_deg": float(np.abs(lla[ok][:, :2] - host[ok][:, :2]).max()),
           "max_abs_dxy_m": float(np.abs(xyz[ok][:, :2] - host_utm[ok][:, :2]).max()),
           "card": name, "power_limit": power}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
