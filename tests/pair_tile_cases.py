"""A stub ``s2p`` package for s2p_b200.fused.pair_tile, shared by the CPU and GPU tests of the pair tile.

s2p itself is not importable here (rasterio, rpcm), so its per-tile steps of a two-view run are restated: ``rectification_pair``
with fixed homographies and range in place of ``rectify_pair``'s algebra, but with its two ``common.image_apply_homography``
calls, its text files and its cleaning (s2p/__init__.py:102-164); ``stereo_matching`` (:166-196) around the matcher and erosion
given; ``disparity_to_ply`` is the one given.
"""
import os
import sys
import types

import numpy as np


def stub_s2p(monkeypatch, cfg, H1, H2, w, h, disp_min, disp_max, image_apply_homography, compute_disparity_map, erosion,
             disparity_to_ply):
    s2p = types.ModuleType("s2p")
    config = types.ModuleType("s2p.config")
    config.cfg = cfg
    common = types.ModuleType("s2p.common")
    common.image_apply_homography = image_apply_homography
    s2p.config, s2p.common = config, common
    s2p.calls = []

    def remove(path):
        if os.path.exists(path):
            os.remove(path)

    def rectification_pair(tile, i):
        s2p.calls.append("rectification_pair")
        out_dir = os.path.join(tile['dir'], 'pair_{}'.format(i))
        # rectify_pair warps through the module attribute, as s2p/rectification.py:379-380 does
        s2p.common.image_apply_homography(os.path.join(out_dir, 'rectified_ref.tif'), cfg['images'][0]['img'], H1, w, h)
        s2p.common.image_apply_homography(os.path.join(out_dir, 'rectified_sec.tif'), cfg['images'][i]['img'], H2, w, h)
        np.savetxt(os.path.join(out_dir, 'H_ref.txt'), H1, fmt='%12.6f')
        np.savetxt(os.path.join(out_dir, 'H_sec.txt'), H2, fmt='%12.6f')
        np.savetxt(os.path.join(out_dir, 'disp_min_max.txt'), [disp_min, disp_max], fmt='%3.1f')
        if cfg['clean_intermediate']:
            remove(os.path.join(out_dir, 'pointing.txt'))
            remove(os.path.join(out_dir, 'sift_matches.txt'))

    def stereo_matching(tile, i):
        s2p.calls.append("stereo_matching")
        out_dir = os.path.join(tile['dir'], 'pair_{}'.format(i))
        rect1, rect2 = os.path.join(out_dir, 'rectified_ref.tif'), os.path.join(out_dir, 'rectified_sec.tif')
        mask = os.path.join(out_dir, 'rectified_mask.png')
        dmin, dmax = np.loadtxt(os.path.join(out_dir, 'disp_min_max.txt'))
        compute_disparity_map(rect1, rect2, os.path.join(out_dir, 'rectified_disp.tif'), mask, cfg['matching_algorithm'], dmin, dmax,
                              timeout=cfg['mgm_timeout'], max_disp_range=cfg['max_disp_range'])
        erosion(mask, mask, cfg['msk_erosion'])
        if cfg['clean_intermediate']:
            if len(cfg['images']) > 2:
                remove(rect1)
            remove(rect2)
            remove(os.path.join(out_dir, 'disp_min_max.txt'))

    def step_disparity_to_ply(tile):
        s2p.calls.append("disparity_to_ply")
        return disparity_to_ply(tile)

    s2p.rectification_pair, s2p.stereo_matching, s2p.disparity_to_ply = rectification_pair, stereo_matching, step_disparity_to_ply
    monkeypatch.setitem(sys.modules, "s2p", s2p)
    monkeypatch.setitem(sys.modules, "s2p.config", config)
    monkeypatch.setitem(sys.modules, "s2p.common", common)
    return s2p


def cfg_for(out_dir, img1, img2, rpc1, rpc2, algo, clean, clr=None):
    return {"out_dir": str(out_dir), "out_crs": "epsg:32740", "gsd": 0.5, "3d_filtering_r": 5.0, "3d_filtering_n": 50,
            "clean_intermediate": clean, "matching_algorithm": algo, "mgm_timeout": 600, "max_disp_range": None,
            "msk_erosion": 2, "images": [{"img": img1, "rpcm": rpc1, "clr": clr}, {"img": img2, "rpcm": rpc2, "clr": None}]}


def make_tile(root, name, mask_shape):
    """a tile directory with the files the earlier steps leave: the tile's mask, the pair's pointing and SIFT matches"""
    from s2p_b200 import rasterio_compat as rio
    d = os.path.join(str(root), name)
    os.makedirs(os.path.join(d, "pair_1"))
    rio.write_mask_png(os.path.join(d, "mask.png"), np.ones(mask_shape, np.uint8))
    np.savetxt(os.path.join(d, "pair_1", "pointing.txt"), np.eye(3))
    np.savetxt(os.path.join(d, "pair_1", "sift_matches.txt"), np.zeros((2, 4)))
    return {"dir": d, "coordinates": (0, 0, mask_shape[1] - 1, mask_shape[0] - 1), "neighborhood_dirs": []}


def files(d):
    """{path relative to d: bytes} of every file under d"""
    out = {}
    for root, _, names in os.walk(d):
        for n in names:
            p = os.path.join(root, n)
            with open(p, "rb") as f:
                out[os.path.relpath(p, d)] = f.read()
    return out
