"""Cost of a tile at out_crs = epsg:2154 (RGF93 v1 / Lambert-93) on a C2-sized tile (1024 x 1024, 128 labels), host clock
around each synchronous call, median of REPS, alternated:
- pair_tile_2154: s2pb_pair_tile_to_ply with S2PB_ZONE_PROJ, the whole tile in one device call;
- pair_tile_utm: the same call at UTM zone 31N, the same work with the UTM map;
- fall_through_floor: what the path a 2154 tile took before cannot do without: the triangulation to (lon, lat, alt) on the
  device (s2pb_disp_to_xyz, zone 0) and the Lambert map of that cloud in float64 numpy on one host core
  (tests/lcc_oracle.py), which stands in for pyproj; the separate rectification and matching steps, pyproj's own overhead,
  the CPU filter and the PLY writing are not counted, so the old path costs more than this.
Prints the card's name and power limit with the times.  Writes nothing."""
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import numpy as np  # noqa: E402

import lcc_oracle as L  # noqa: E402
from s2p_b200 import projection  # noqa: E402
from s2p_b200._lib import ZONE_PROJ  # noqa: E402
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
    p = matcher_params("mgm", 0)
    eng.set_projection(projection.PROJECTED[2154])
    lambert = (ZONE_PROJ, False)

    def tile(zone, south):
        return eng.pair_tile_to_ply(ref, eye, sec, eye, n, n, dmin, dmax, mo, fx["H1"], fx["H2"], rpc1, rpc2, bbx, zone, south,
                                    params=p, erode_radius=2, r=5.0, p=10, n=50, confidence=True, want=("disp", "mask", "conf"))

    rec, out = tile(*lambert)

    def floor():
        lla, _ = eng.disp_to_xyz(out["disp"], out["mask"], mo, fx["H1"], fx["H2"], rpc1, rpc2, bbx)
        return L.lcc_restate(lla, projection.PROJECTED[2154])

    runs = {"pair_tile_2154": lambda: tile(*lambert), "pair_tile_utm": lambda: tile(31, False), "fall_through_floor": floor}
    times = {k: [] for k in runs}
    for _ in range(2):                                          # warm-up of every shape
        for fn in runs.values():
            fn()
    for _ in range(REPS):
        for k, fn in runs.items():
            times[k].append(timed(fn))
    print("card (name, power limit, max SM clock):", card())
    print("tile %dx%d, %d labels, %d repetitions alternated; points kept at 2154: %d" % (n, n, dmax - dmin + 1, REPS, len(rec)))
    for k, v in times.items():
        print("%-20s median %8.2f ms  min %8.2f ms  max %8.2f ms" % (k, statistics.median(v), min(v), max(v)))
    eng.close()


if __name__ == "__main__":
    main()
