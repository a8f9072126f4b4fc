"""Writes tests/golden/triplet.npz and tests/golden/localization_ref_samples.npz from fixtures the reference ships for its own
tests: the tri-stereo height map and DSM of its triplet run (tests/data/expected_output/triplet/{height_map,dsm}.tif) and the
camera of that run's reference image (tests/data/input_triplet/img_02.tif, RPCCoefficientTag).

* height_map.tif is 700 x 700 float32 in the frame of input_triplet/config.json's ROI, (x, y) = (150, 150) on img_02.tif,
  the first image of the configuration and so the reference image.  A CROP x CROP crop of it is kept with its origin in
  img_02.tif, (150 + CX, 150 + CY).
* dsm.tif is 0.5 m, EPSG:32631, tiepoint (698053.031, 4792984.069).  The window of it that the crop's footprint covers is kept,
  with its origin.
* The offset is confirmed here: the crop, localised by the reference's own rpc_localization (tests/localization_oracle.py),
  projected to UTM 31N (tests/utm_oracle.py) and rasterised on the window's grid (tests/dsm_oracle.py), falls inside the
  window, and there it shares more cells with the DSM, with a narrower spread of dz, than the same crop given an origin 4 or
  150 pixels away.  The median and 99th percentile of |dz| over the cells both have are stored.  They are not zero: the DSM
  was made from the merged, filtered heights of both pairs, and the height map is one stage earlier.  At the time of writing:
  30 716 common cells, |dz| median 2.314 m, p99 3.514 m; dz itself has median -2.314 m (the height map lies below the DSM)
  and a median absolute deviation of 0.317 m about it.
* For the machines where oracle/_ref is not built, what rpc_localization returns for the cases of
  tests/localization_oracle.py is recorded on a seeded sample of pixels.
    python tests/golden/make_golden_triplet.py        (after __graft_entry__.build() has built oracle/_ref)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
REF = "/root/reference/tests/data"
ROI = (150, 150)
CX, CY, CROP = 250, 250, 200
DSM_X0, DSM_Y0, DSM_RES = 698053.031, 4792984.069, 0.5
ZONE, SOUTH = 31, False
MARGIN = 4


def localise_utm(heights, rpc, off_x, off_y):
    import localization_oracle as LO
    import utm_oracle as U
    lla = LO.ref_height_map_to_xyz(heights, rpc, off_x, off_y)
    return U.restate(lla, ZONE, SOUTH)


def rasterise(xyz, xoff, yoff, xsize, ysize):
    import dsm_oracle as D
    pts = xyz.reshape(-1, 3)
    pts = pts[np.isfinite(pts).all(axis=1)]
    return D.plyflatten([pts], xoff, yoff, DSM_RES, xsize, ysize)[..., 0]


def dz_stats(a, b):
    """-> (common cells, median |dz|, 99th percentile of |dz|, median dz, median |dz - median dz|), dz = a - b"""
    both = np.isfinite(a) & np.isfinite(b)
    d = a[both].astype(np.float64) - b[both]
    m = float(np.median(d))
    return int(both.sum()), float(np.median(np.abs(d))), float(np.percentile(np.abs(d), 99)), m, float(np.median(np.abs(d - m)))


def main():
    import localization_oracle as LO
    from PIL import Image
    from s2p_b200 import rasterio_compat as rio
    from s2p_b200.triangulation import rpc_from_geotiff_tag
    assert LO.have_ref(), "oracle/_ref is not built"
    with Image.open(os.path.join(REF, "input_triplet", "img_02.tif")) as im:
        tag = np.array(im.tag_v2[50844], np.float64)
    assert tag.size == 92
    rpc = rpc_from_geotiff_tag(tag)
    hmap = rio.read_band_stored(os.path.join(REF, "expected_output", "triplet", "height_map.tif"))
    dsm = rio.read_band_stored(os.path.join(REF, "expected_output", "triplet", "dsm.tif"))
    assert hmap.dtype == np.float32 and hmap.shape == (700, 700) and dsm.dtype == np.float32
    crop = np.ascontiguousarray(hmap[CY:CY + CROP, CX:CX + CROP])
    off = (ROI[0] + CX, ROI[1] + CY)
    xyz = localise_utm(crop, rpc, *off)
    fin = np.isfinite(xyz).all(axis=2)
    x, y = xyz[fin][:, 0], xyz[fin][:, 1]
    # the DSM window over the footprint, MARGIN cells wider on every side
    c0, c1 = int(np.floor((x.min() - DSM_X0) / DSM_RES)) - MARGIN, int(np.floor((x.max() - DSM_X0) / DSM_RES)) + MARGIN + 1
    r0, r1 = int(np.floor((DSM_Y0 - y.max()) / DSM_RES)) - MARGIN, int(np.floor((DSM_Y0 - y.min()) / DSM_RES)) + MARGIN + 1
    assert 0 <= c0 and c1 <= dsm.shape[1] and 0 <= r0 and r1 <= dsm.shape[0], "the footprint leaves the DSM"
    win = np.ascontiguousarray(dsm[r0:r1, c0:c1])
    xoff, yoff = DSM_X0 + c0 * DSM_RES, DSM_Y0 - r0 * DSM_RES
    got = rasterise(xyz, xoff, yoff, win.shape[1], win.shape[0])
    n, med, p99, bias, spread = dz_stats(got, win)
    print("crop %dx%d at (%d, %d) of img_02.tif, %.1f %% NaN; DSM window %dx%d at (%d, %d)" % (
        CROP, CROP, off[0], off[1], 100 * np.isnan(crop).mean(), win.shape[1], win.shape[0], c0, r0))
    line = "origin %+4d %+4d px: %5d common cells, |dz| median %.4f m, p99 %.4f m; dz median %+.4f m, spread %.4f m"
    print(line % (0, 0, n, med, p99, bias, spread))
    # the same crop with another origin: fewer common cells and a wider spread of dz about its median
    for dx, dy in ((-150, -150), (-4, -4), (-4, 0), (-4, 4), (0, -4), (0, 4), (4, -4), (4, 0), (4, 4)):
        other = dz_stats(rasterise(localise_utm(crop, rpc, off[0] + dx, off[1] + dy), xoff, yoff, win.shape[1], win.shape[0]), win)
        print(line % ((dx, dy) + other))
        assert other[0] < n and other[4] > spread, "another origin fits the DSM as well"
    np.savez_compressed(os.path.join(HERE, "triplet.npz"), rpc=tag, heights=crop, off=np.array(off, np.float64), dsm=win,
                        dsm_xoff=np.float64(xoff), dsm_yoff=np.float64(yoff), dsm_res=np.float64(DSM_RES),
                        dz_median=np.float64(med), dz_p99=np.float64(p99), dz_cells=np.int64(n))
    samples = {}
    for name in sorted(LO.cases()):
        samples.update(LO.record(name))
        print("recorded rpc_localization:%s" % name)
    np.savez_compressed(LO.RECORDED, **samples)


if __name__ == "__main__":
    main()
