"""The pair path's last per-tile step (disparity_to_ply) with a `clr` image on a 1024x1024 tile: the real pair's cameras and
rectifying homographies (tests/golden/real_pair*.npz) with its rectified disparity tiled to 1024x1024, EPSG:32740, filter
r = 5 m, n = 50 at a GSD of 0.5 m, a confidence image, and a seeded 3-band uint16 clr image of 2000x2000 written as a TIFF.

Times, each ending in a device synchronise, median of --reps after a warm-up:
  * `clr`: the crop of the clr image the warp needs (common.homography_crop), then `disp_to_ply_clr` (triangulation,
    projection, filter, the warp of every band and the float32 records in one device call) and the file write;
  * `clr_call`: the same without reading the crop (the device call and the file write);
  * the path it replaces: the warp drop-in (common.image_apply_homography) writing its temporary TIFF, that TIFF read back,
    `disp_to_xyz` and `remove_isolated_3d_points` on the device, then s2p's writer (one Python tuple per point,
    tests/ply_oracle.py) and the file write.
Checks that both paths give the same records, and reads the card and its power limit in the same run.  One JSON line.

    python scripts/clr_ply_probe.py [--reps 10] [--out DIR]
"""
import argparse
import json
import os
import sys
import tempfile
import time

os.environ.setdefault("OMP_NUM_THREADS", "1")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402

import ply_oracle as P  # noqa: E402
from ply_probe import N, PW, R, SOUTH, ZONE, card, inputs, timed  # noqa: E402
from s2p_b200 import cloud, common, rasterio_compat  # noqa: E402
from s2p_b200.engine import Engine  # noqa: E402


def clr_image(path, side=2000, seed=0):
    import cv2
    planes = np.random.default_rng(seed).integers(0, 4096, (3, side, side)).astype(np.uint16)
    if not cv2.imwrite(path, np.ascontiguousarray(np.moveaxis(planes, 0, 2)[..., ::-1])):
        raise IOError("cv2.imwrite failed for %s" % path)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    a = inputs()
    h, w = a["disp"].shape
    eng = Engine(0)
    tmp = tempfile.mkdtemp()
    path = os.path.join(tmp, "cloud.ply")
    clr = os.path.join(tmp, "clr.tif")
    warped = os.path.join(tmp, "colors.tif")
    clr_image(clr)
    comments = ["created by S2P", "projection: CRS epsg:32740"]
    cloud_args = (a["disp"], a["mask_rect"], a["mask_orig"], a["H1"], a["H2"], a["rpc1"], a["rpc2"], a["bbx"], ZONE, SOUTH)

    def device():
        crop, hc = common.homography_crop(clr, a["H1"], w, h, ["homography", clr])
        rec = eng.disp_to_ply_clr(*cloud_args, r=R, p=PW, n=N, clr=crop, hc=hc, confidence=a["conf"])
        cloud.write_ply(path, rec, comments)
        return rec

    def replaced():
        common.image_apply_homography(warped, clr, a["H1"], w, h)
        colors = rasterio_compat.read_stored(warped)
        xyz, _ = eng.disp_to_xyz(*cloud_args)
        eng.remove_isolated_3d_points(xyz, R, PW, N, 1)
        rec = P.ply_records_literal(xyz, colors, a["conf"])
        with open(path, "wb") as f:
            f.write(P.ply_header(len(rec), comments, 3, True, "float"))
            f.write(rec.tobytes())
        return rec

    crop, hc = common.homography_crop(clr, a["H1"], w, h, ["homography", clr])

    def call():
        rec = eng.disp_to_ply_clr(*cloud_args, r=R, p=PW, n=N, clr=crop, hc=hc, confidence=a["conf"])
        cloud.write_ply(path, rec, comments)
        return rec

    t_call, _ = timed(call, args.reps)
    t_device, rec = timed(device, args.reps)
    t_replaced, want = timed(replaced, max(1, args.reps // 5))
    res = dict(card=card(), tile=[h, w], clr="3 x 2000 x 2000 uint16", kept=len(rec), record_bytes=rec.dtype.itemsize,
               nan_colours=int(np.isnan(rec["red"]).sum()), clr_ms=round(t_device, 3), clr_call_ms=round(t_call, 3),
               replaced_ms=round(t_replaced, 3),
               identical=rec.dtype == want.dtype and rec.tobytes() == want.tobytes())
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "clr_ply_probe.json"), "w") as f:
            f.write(line + "\n")
    eng.close()


if __name__ == "__main__":
    main()
