"""The pair path's last per-tile step (disparity_to_ply) on a 1024x1024 tile with about 10^6 points: the real pair's cameras
and rectifying homographies (tests/golden/real_pair*.npz) with its rectified disparity and reference image tiled to 1024x1024,
EPSG:32740, filter r = 5 m, n = 50 at a GSD of 0.5 m, one colour band and a confidence image.

Times, host buffers in and out, each call ending in a device synchronise, median of --reps after a warm-up:
  * `disp_to_ply`: triangulation, projection, filter, stretch and records in one device call;
  * today's path with the drop-ins installed: `disp_to_xyz` and `remove_isolated_3d_points` on the device, then the
    stretch (np.nanpercentile) and s2p's writer (one Python tuple per point, tests/ply_oracle.py) on the host;
  * the writer's host time alone (the tuple path and the file write; plyfile's own write is replaced by a raw dump).
Checks that both paths give the same records, and reads the card and its power limit in the same run.  One JSON line.

    python scripts/ply_probe.py [--reps 10] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

os.environ.setdefault("OMP_NUM_THREADS", "1")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import ply_oracle as P  # noqa: E402
from s2p_b200 import cloud  # noqa: E402
from s2p_b200.engine import Engine  # noqa: E402
from s2p_b200.triangulation import rpc_from_geotiff_tag  # noqa: E402
from util import load_real_pair  # noqa: E402

R, PW, N, ZONE, SOUTH = 5.0, 10, 50, 40, True


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def inputs(side=1024):
    z = load_real_pair()
    disp = np.nan_to_num(z["rectified_disp"])
    tile = lambda a: np.ascontiguousarray(np.tile(a, (side // a.shape[0] + 1, side // a.shape[1] + 1))[:side, :side])
    rng = np.random.default_rng(0)
    return dict(disp=tile(disp), mask_rect=np.ones((side, side), np.float32), mask_orig=np.ones((1024, 1024), np.float32),
                H1=z["H1"], H2=z["H2"], rpc1=rpc_from_geotiff_tag(z["rpc1"]), rpc2=rpc_from_geotiff_tag(z["rpc2"]),
                bbx=(0.0, 1023.0, 0.0, 1023.0), colors=tile(z["rectified_ref"])[None],
                conf=rng.random((side, side)).astype(np.float32))


def timed(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)) * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    a = inputs()
    eng = Engine(0)
    tmp = tempfile.mkdtemp()
    path = os.path.join(tmp, "cloud.ply")
    comments = ["created by S2P", "projection: CRS epsg:32740"]

    def chained():
        rec = eng.disp_to_ply(a["disp"], a["mask_rect"], a["mask_orig"], a["H1"], a["H2"], a["rpc1"], a["rpc2"], a["bbx"],
                              ZONE, SOUTH, r=R, p=PW, n=N, colors=a["colors"], confidence=a["conf"])
        cloud.write_ply(path, rec, comments)
        return rec

    def writer(xyz, colors):
        rec = P.ply_records_literal(xyz, colors, a["conf"])
        with open(path, "wb") as f:
            f.write(P.ply_header(len(rec), comments, 1, True))
            f.write(rec.tobytes())
        return rec

    def today():
        xyz, _ = eng.disp_to_xyz(a["disp"], a["mask_rect"], a["mask_orig"], a["H1"], a["H2"], a["rpc1"], a["rpc2"], a["bbx"],
                                 ZONE, SOUTH)
        a["finite"] = int(np.isfinite(xyz).all(axis=2).sum())
        eng.remove_isolated_3d_points(xyz, R, PW, N, 1)
        return writer(xyz, P.stretch_8bit_reference(a["colors"])), xyz

    t_chain, rec = timed(chained, args.reps)
    t_today, (want, xyz) = timed(today, max(1, args.reps // 5))
    colors = P.stretch_8bit_reference(a["colors"])
    t_writer, _ = timed(lambda: writer(xyz, colors), max(1, args.reps // 5))
    res = dict(card=card(), tile=list(a["disp"].shape), points=a["finite"], kept=len(rec),
               record_bytes=rec.dtype.itemsize, chained_ms=round(t_chain, 3), today_ms=round(t_today, 3),
               writer_host_ms=round(t_writer, 3), identical=rec.tobytes() == want.tobytes())
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "ply_probe.json"), "w") as f:
            f.write(line + "\n")
    eng.close()


if __name__ == "__main__":
    main()
