"""Cost of the EGM96 step (S2PB_ZONE_EGM96) on a C2-sized tile (1024 x 1024, 128 labels): disp_to_ply and pair_tile_to_ply
with and without the geoid, alternated, host clock around each synchronous call, median of REPS.  Prints the card's name and
power limit with the times; the grid is a seeded synthetic global 15' grid (tests/geoid_oracle.py).  Writes nothing."""
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import numpy as np  # noqa: E402

import geoid_oracle as G  # noqa: E402
from s2p_b200._lib import ZONE_EGM96  # noqa: E402
from s2p_b200.block_matching import matcher_params  # noqa: E402
from s2p_b200.engine import Engine  # noqa: E402
from s2p_b200.synth import make_pair  # noqa: E402
from s2p_b200.triangulation import rpc_from_geotiff_tag  # noqa: E402
from util import load_real_pair  # noqa: E402

REPS = int(os.environ.get("REPS", 15))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "nvidia-smi unavailable"


def timed(fn):
    t = time.perf_counter()
    fn()
    return (time.perf_counter() - t) * 1e3


def main():
    fx = load_real_pair()
    rpc1, rpc2 = rpc_from_geotiff_tag(fx["rpc1"]), rpc_from_geotiff_tag(fx["rpc2"])
    n, dmin, dmax = 1024, -64, 63
    ref, sec, _ = make_pair(n, n, dmin, dmax, seed=0)
    eye, mo, bbx = np.eye(3), np.ones((n, n), np.float32), (0.0, float(n - 1), 0.0, float(n - 1))
    eng = Engine(0)
    eng.set_geoid(G.smooth_grid(5))
    p = matcher_params("mgm", 0)
    zone, south = 40, True

    def tile(zn):
        return eng.pair_tile_to_ply(ref, eye, sec, eye, n, n, dmin, dmax, mo, fx["H1"], fx["H2"], rpc1, rpc2, bbx, zn, south, params=p,
                                    erode_radius=2, r=5.0, p=10, n=50, confidence=True, want=("disp", "mask", "conf"))

    _, out = tile(zone)

    def cloud(zn):
        return eng.disp_to_ply(out["disp"], out["mask"], mo, fx["H1"], fx["H2"], rpc1, rpc2, bbx, zn, south, r=5.0, p=10, n=50,
                               colors=ref[None], confidence=out["conf"])

    npts = (len(cloud(zone)), len(cloud(zone | ZONE_EGM96)))
    times = {k: [] for k in ("disp_to_ply", "disp_to_ply+egm96", "pair_tile", "pair_tile+egm96")}
    for _ in range(2):                                          # warm-up of every shape
        cloud(zone), cloud(zone | ZONE_EGM96), tile(zone), tile(zone | ZONE_EGM96)
    for _ in range(REPS):
        times["disp_to_ply"].append(timed(lambda: cloud(zone)))
        times["disp_to_ply+egm96"].append(timed(lambda: cloud(zone | ZONE_EGM96)))
        times["pair_tile"].append(timed(lambda: tile(zone)))
        times["pair_tile+egm96"].append(timed(lambda: tile(zone | ZONE_EGM96)))
    print("card (name, power limit, max SM clock):", card())
    print("tile %dx%d, %d labels, %d repetitions alternated; points kept without / with the geoid: %d / %d"
          % ((n, n, dmax - dmin + 1, REPS) + npts))
    for k, v in times.items():
        print("%-18s median %8.2f ms  min %8.2f ms  max %8.2f ms" % (k, statistics.median(v), min(v), max(v)))
    eng.close()


if __name__ == "__main__":
    main()
