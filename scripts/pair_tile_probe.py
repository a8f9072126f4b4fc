"""Per-tile wall clock of steps 3 to 5 of a two-view run (rectification_pair, stereo_matching, disparity_to_ply) by three paths,
on tile directories in a local temporary directory, under the stub s2p package of the tests (tests/pair_tile_cases.py: s2p's
step functions around fixed homographies and range instead of rectify_pair's algebra):

  * `stepwise`: the three steps through the drop-ins, every hand-off through files (the two warps write the rectified TIFFs,
    the matcher reads them and writes the disparity, confidence and mask, the erosion rewrites the mask, the cloud step reads
    them back);
  * `rectify_and_match`: fused.rectify_and_match for steps 3 and 4 (warps and matcher in one device call, the same files out),
    then the erosion and disparity_to_ply through files;
  * `pair_tile`: fused.pair_tile, one device call from the source images to cloud.ply.

Tiles: the real Pleiades pair of tests/golden/real_pair*.npz (503 x 425, [-41, 30]) and a C2-size synthetic tile (1024 x 1024, 128
labels, seeded sources warped by a translation).  Algo mgm, s2p's defaults otherwise (msk_erosion 2, no 3D filter), EPSG:32740,
clean_intermediate off and on.  Each figure is the median over --reps runs after one warm-up, the three paths alternating within
a run; every run starts from a fresh tile directory made outside the timed region.  The paths must leave the same cloud.ply,
byte for byte.  Reads the card and its power limit in the same run; one JSON line.

    python scripts/pair_tile_probe.py [--reps 7] [--out DIR]
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

os.environ.setdefault("OMP_NUM_THREADS", "1")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402

import pair_tile_cases as PT  # noqa: E402
from ply_probe import card  # noqa: E402
from s2p_b200 import block_matching, cloud, common, fused, masking, rasterio_compat as rio  # noqa: E402
from s2p_b200.engine import get_engine  # noqa: E402
from s2p_b200.synth import make_pair  # noqa: E402
from s2p_b200.triangulation import rpc_from_geotiff_tag  # noqa: E402
from util import load_real_pair  # noqa: E402


class _Modules:
    """the setitem of pytest's monkeypatch, for PT.stub_s2p outside pytest"""
    def setitem(self, d, k, v):
        d[k] = v


def tiles():
    z = load_real_pair()
    shift = lambda Hm, xy: np.asarray(Hm, np.float64) @ np.array([[1, 0, xy[0]], [0, 1, xy[1]], [0, 0, 1.0]])
    h, w = z["rectified_ref"].shape
    real = dict(src1=z["crop1"].astype(np.float32), src2=z["crop2"].astype(np.float32), H1=shift(z["H1"], z["xy1"]),
                H2=shift(z["H2"], z["xy2"]), w=w, h=h, dmin=-41, dmax=30)
    ref, sec, _ = make_pair(1040, 1040, -64, 63, seed=0)
    T = np.array([[1.0, 0.0, -8.0], [0.0, 1.0, -8.0], [0.0, 0.0, 1.0]])
    c2 = dict(src1=ref, src2=sec, H1=T, H2=T, w=1024, h=1024, dmin=-64, dmax=63)
    return dict(real=real, c2=c2), rpc_from_geotiff_tag(z["rpc1"]), rpc_from_geotiff_tag(z["rpc2"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    eng = get_engine()
    tmp = tempfile.mkdtemp()
    ts, rpc1, rpc2 = tiles()
    res = dict(card=card(), algo="mgm", reps=args.reps)
    for name, t in ts.items():
        img1, img2 = os.path.join(tmp, name + "_1.tif"), os.path.join(tmp, name + "_2.tif")
        rio.write_float_tiff(img1, t["src1"])
        rio.write_float_tiff(img2, t["src2"])
        for clean in (False, True):
            cfg = PT.cfg_for(tmp, img1, img2, rpc1, rpc2, "mgm", clean)
            cfg["3d_filtering_r"] = cfg["3d_filtering_n"] = None
            np.savetxt(os.path.join(tmp, "global_pointing_pair_1.txt"), np.eye(3))
            s2p = PT.stub_s2p(_Modules(), cfg, t["H1"], t["H2"], t["w"], t["h"], float(t["dmin"]), float(t["dmax"]),
                              common.image_apply_homography, block_matching.compute_disparity_map, masking.erosion,
                              cloud.disparity_to_ply)

            def stepwise(tile):
                s2p.rectification_pair(tile, 1)
                s2p.stereo_matching(tile, 1)
                s2p.disparity_to_ply(tile)

            def rectify_and_match(tile):
                calls = []
                s2p.common.image_apply_homography = lambda *a: calls.append(a)
                try:
                    s2p.rectification_pair(tile, 1)
                finally:
                    s2p.common.image_apply_homography = common.image_apply_homography
                (o1, i1, Ha, w, h), (o2, i2, Hb, _, _) = calls
                pair = os.path.join(tile["dir"], "pair_1")
                dmin, dmax = np.loadtxt(os.path.join(pair, "disp_min_max.txt"))
                disp, mask = os.path.join(pair, "rectified_disp.tif"), os.path.join(pair, "rectified_mask.png")
                fused.rectify_and_match(o1, o2, disp, mask, i1, i2, Ha, Hb, w, h, "mgm", dmin, dmax, cfg["mgm_timeout"])
                masking.erosion(mask, mask, cfg["msk_erosion"])
                if clean:
                    os.remove(o2)
                    os.remove(os.path.join(pair, "disp_min_max.txt"))
                s2p.disparity_to_ply(tile)

            def pair_tile(tile):
                fused.pair_tile(tile, engine=eng)

            paths = dict(stepwise=stepwise, rectify_and_match=rectify_and_match, pair_tile=pair_tile)
            times = {k: [] for k in paths}
            clouds = {}
            for rep in range(args.reps + 1):
                for k, fn in paths.items():
                    tile = PT.make_tile(tmp, "%s_%s_%d_%d" % (name, k, clean, rep), (1024, 1024))
                    t0 = time.perf_counter()
                    fn(tile)
                    dt = time.perf_counter() - t0
                    if rep:
                        times[k].append(dt)
                    with open(os.path.join(tile["dir"], "cloud.ply"), "rb") as f:
                        clouds[k] = f.read()
                    shutil.rmtree(tile["dir"])
            key = "%s_%s" % (name, "clean" if clean else "keep")
            res[key] = {k: round(float(np.median(v)) * 1e3, 2) for k, v in times.items()}
            res[key]["identical"] = len(set(clouds.values())) == 1
    shutil.rmtree(tmp)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "pair_tile_probe.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
