"""disp_to_xyz into UTM on the shape s2p gives it: a 1024x1024 rectified disparity map of the reference's Pleiades pair
(its camera models and rectifying homographies from tests/golden/real_pair*.npz, a seeded disparity field about its
disparities), projected to EPSG:32740.

Times, host buffers in and out, each call ending in a device synchronise, median of --reps after a warm-up:
  * `disp_to_xyz` with zone 40 south: triangulation and projection in one device call;
  * `disp_to_lonlatalt` alone, the numpy float64 projection of tests/utm_oracle.py on one host core, and their sum (the
    host-projection path this call replaces, with the restatement standing in for pyproj, which is not installed here
    and was not measured);
  * `lonlat_to_utm` alone, host to host.
Compares the GPU cloud with disp_to_lonlatalt + the numpy projection on the same inputs, and reads the card and its power
limit in the same run.  One JSON line on stdout.

    python scripts/projection_probe.py [--reps 20]
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

import utm_oracle as U  # noqa: E402
from s2p_b200.engine import Engine  # noqa: E402
from s2p_b200.triangulation import disp_to_lonlatalt, rpc_from_geotiff_tag  # noqa: E402
from util import load_real_pair  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, check=True).stdout.strip().split(", ")
        return q[0], q[1]
    except Exception:
        return "unknown", "unknown"


def inputs(side, seed=0):
    z = load_real_pair()
    d = z["rectified_disp"]
    rng = np.random.default_rng(seed)
    disp = (np.nanmedian(d) + rng.normal(0.0, np.nanstd(d), (side, side))).astype(np.float32)
    return dict(disp=disp, mask_rect=np.ones((side, side), np.float32), mask_orig=np.ones((1, 1), np.float32),
                H1=z["H1"], H2=z["H2"], rpc1=rpc_from_geotiff_tag(z["rpc1"]), rpc2=rpc_from_geotiff_tag(z["rpc2"]),
                img_bbx=(-1e6, 1e6, -1e6, 1e6))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--side", type=int, default=1024)
    a = ap.parse_args()
    zone, south = 40, True
    x = inputs(a.side)
    eng = Engine(0)
    xyz_call = lambda: eng.disp_to_xyz(x["disp"], x["mask_rect"], x["mask_orig"], x["H1"], x["H2"], x["rpc1"], x["rpc2"],
                                       x["img_bbx"], zone, south)
    lla_call = lambda: disp_to_lonlatalt(x["disp"], x["mask_rect"], x["mask_orig"], x["H1"], x["H2"], x["rpc1"], x["rpc2"],
                                         x["img_bbx"], engine=eng)
    xyz, err = xyz_call()                                                  # warm-up: module load, pooled buffers
    lla, lerr = lla_call()
    eng.lonlat_to_utm(lla, zone, south)

    def timed(fn, reps):
        t = []
        for _ in range(reps):
            t0 = time.perf_counter()
            fn()                                                           # synchronous: returns with the results on the host
            t.append(time.perf_counter() - t0)
        return np.array(t) * 1e3

    t_xyz = timed(xyz_call, a.reps)
    t_lla = timed(lla_call, a.reps)
    t_utm = timed(lambda: eng.lonlat_to_utm(lla, zone, south), a.reps)
    t_np = timed(lambda: U.restate(lla, zone, south), max(3, a.reps // 4))
    host = U.restate(lla, zone, south)
    fin = np.isfinite(host[..., 0])
    name, power = card()
    med = lambda t: round(float(np.median(t)), 3)
    res = {"workload": "disp_to_xyz %dx%d to EPSG:32740, host buffers in and out" % (a.side, a.side),
           "points": int(a.side * a.side), "valid_points": int(fin.sum()),
           "disp_to_xyz_ms": med(t_xyz),
           "disp_to_lonlatalt_ms": med(t_lla),
           "numpy_projection_one_core_ms": med(t_np),
           "disp_to_lonlatalt_plus_numpy_ms": round(med(t_lla) + med(t_np), 3),
           "lonlat_to_utm_ms": med(t_utm),
           "reps": a.reps,
           "same_nan_mask": bool(np.array_equal(np.isnan(xyz), np.isnan(host))),
           "z_bit_equal": bool(np.array_equal(xyz[..., 2][fin].view(np.uint64), lla[..., 2][fin].view(np.uint64))),
           "err_bit_equal": bool(np.array_equal(err.view(np.uint32), lerr.view(np.uint32))),
           "max_abs_dxy_m": float(np.abs(xyz[..., :2][fin] - host[..., :2][fin]).max()),
           "card": name, "power_limit": power}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
