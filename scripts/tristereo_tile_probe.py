"""Per-tile wall clock of steps 3 to 5d of a three-image run by two paths, on tile directories in a local temporary directory,
under the stub s2p package of the tests (tests/tristereo_cases.py: s2p's step functions around fixed homographies and range instead
of rectify_pair's algebra):

  * `stepwise`: for pairs 1 and 2, rectification_pair, stereo_matching and disparity_to_height through the drop-ins, every
    hand-off through files; then heights_to_ply (the cloud drop-in) with its heights_fusion (the cargarse_basura and merge_n
    drop-ins), which reads the pair height maps back;
  * `fused`: fused.pair_heights for pairs 1 and 2, then fused.heights_tile: two device calls per pair and tile.

Steps 5b and 5c (mean_heights, global_mean_heights), the barrier across tiles, are left out: both paths read the same fixed
global_mean_height_pair_k.txt.  Image 3 is image 2, its pair with its own pointing correction.

Tiles: the real Pleiades pair of tests/golden/real_pair*.npz (503 x 425 rectified, [-41, 30], the tile (500, 150, 350, 350))
and a C2-size synthetic tile (1024 x 1024 rectified, 128 labels, seeded sources warped by a translation, the tile
(8, 8, 1000, 1000)).  Algo mgm, s2p's defaults otherwise (msk_erosion 2, cargarse_basura on, average_if_close with threshold 3,
no 3D filter), EPSG:32740, clean_intermediate off and on.  Each figure is the median over --reps runs after one warm-up, the
paths alternating within a run; every run starts from a fresh tile directory made outside the timed region.  The paths must
leave the same cloud.ply, byte for byte.  Reads the card and its power limit in the same run; one JSON line.

    python scripts/tristereo_tile_probe.py [--reps 7] [--out DIR]
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

import tristereo_cases as TC  # noqa: E402
from ply_probe import card  # noqa: E402
from s2p_b200 import block_matching, cloud, common, fused, fusion, masking, rasterio_compat as rio, triangulation  # noqa: E402
from s2p_b200.engine import get_engine  # noqa: E402
from s2p_b200.synth import make_pair  # noqa: E402
from s2p_b200.triangulation import rpc_from_geotiff_tag  # noqa: E402
from util import load_real_pair  # noqa: E402

POINTING = np.array([[1.000186, 0.000156, 0.518804], [0.000040, 1.000032, 0.109895], [0.0, 0.0, 1.0]])


class _Modules:
    """the setitem of pytest's monkeypatch, for TC.stub_s2p outside pytest"""
    def setitem(self, d, k, v):
        d[k] = v


def _canvas(src, xy):
    a = np.zeros((xy[1] + src.shape[0], xy[0] + src.shape[1]), np.float32)
    a[xy[1]:, xy[0]:] = src
    return a


def tiles():
    z = load_real_pair()
    h, w = z["rectified_ref"].shape
    real = dict(img1=_canvas(z["crop1"].astype(np.float32), z["xy1"]), img2=_canvas(z["crop2"].astype(np.float32), z["xy2"]),
                H1=z["H1"], H2=z["H2"], w=w, h=h, dmin=-41, dmax=30, tile=(500, 150, 350, 350))
    ref, sec, _ = make_pair(1040, 1040, -64, 63, seed=0)
    T = np.array([[1.0, 0.0, -8.0], [0.0, 1.0, -8.0], [0.0, 0.0, 1.0]])
    c2 = dict(img1=ref, img2=sec, H1=T, H2=T, w=1024, h=1024, dmin=-64, dmax=63, tile=(8, 8, 1000, 1000))
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
    np.savetxt(os.path.join(tmp, "global_pointing_pair_1.txt"), np.eye(3))
    np.savetxt(os.path.join(tmp, "global_pointing_pair_2.txt"), POINTING)
    for name, t in ts.items():
        img1, img2 = os.path.join(tmp, name + "_1.tif"), os.path.join(tmp, name + "_2.tif")
        rio.write_float_tiff(img1, t["img1"])
        rio.write_float_tiff(img2, t["img2"])
        x, y, tw, th = t["tile"]
        mask = np.ones((th, tw), np.uint8)
        mask[th // 3:th // 3 + 20, tw // 2:tw // 2 + 30] = 0
        for clean in (False, True):
            cfg = TC.cfg_for(tmp, [img1, img2, img2], [rpc1, rpc2, rpc2], "mgm", clean)
            cfg.update({"3d_filtering_r": None, "3d_filtering_n": None, "fusion_thresh": 3})
            s2p = TC.stub_s2p(_Modules(), cfg, t["H1"], t["H2"], t["w"], t["h"], float(t["dmin"]), float(t["dmax"]),
                              common.image_apply_homography, block_matching.compute_disparity_map, masking.erosion,
                              height_map=triangulation.height_map, write_height_map=rio.write_float64_tiff,
                              cargarse_basura=common.cargarse_basura, merge_n=fusion.merge_n, heights_to_ply=cloud.heights_to_ply)

            def stepwise(tile):
                for i in (1, 2):
                    s2p.rectification_pair(tile, i)
                    s2p.stereo_matching(tile, i)
                    s2p.disparity_to_height(tile, i)
                s2p.heights_to_ply(tile)

            def tristereo(tile):
                for i in (1, 2):
                    fused.pair_heights(tile, i, engine=eng)
                fused.heights_tile(tile, engine=eng)

            # the global mean heights of the tile's pairs (steps 5b and 5c, run once here, outside the timed region)
            tile = TC.make_tile(tmp, "%s_offsets_%d" % (name, clean), t["tile"], 2)
            rio.write_mask_png(os.path.join(tile["dir"], "mask.png"), mask)
            for i in (1, 2):
                fused.pair_heights(tile, i, engine=eng)
                hm = rio.read_band_stored(os.path.join(tile["dir"], "pair_%d" % i, "height_map.tif"))
                np.savetxt(os.path.join(tmp, "global_mean_height_pair_%d.txt" % i), [np.nanmean(hm)])
            shutil.rmtree(tile["dir"])

            paths = dict(stepwise=stepwise, fused=tristereo)
            times = {k: [] for k in paths}
            clouds = {}
            for rep in range(args.reps + 1):
                for k, fn in paths.items():
                    tile = TC.make_tile(tmp, "%s_%s_%d_%d" % (name, k, clean, rep), t["tile"], 2)
                    rio.write_mask_png(os.path.join(tile["dir"], "mask.png"), mask)
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
            res[key]["points"] = int(clouds["fused"].split(b"element vertex ")[1].split(b"\n")[0])
    shutil.rmtree(tmp)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "tristereo_tile_probe.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
