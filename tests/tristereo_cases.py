"""A stub ``s2p`` package for s2p_b200.fused.pair_heights and heights_tile, shared by the CPU and GPU tests of the tri-stereo tile.

s2p itself is not importable here, so its per-tile steps of a run with three or more images are restated for pair i:
``rectification_pair`` and ``stereo_matching`` as pair_tile_cases restates them; ``disparity_to_height`` (s2p/__init__.py:199-239)
around the height map and its writer given; ``heights_fusion`` (:355-385) around the cleaning and the merge given; ``heights_to_ply``
is the one given, which runs ``s2p.heights_fusion`` itself when it is the cloud drop-in.
"""
import os

import numpy as np

import pair_tile_cases as PT


def stub_s2p(monkeypatch, cfg, H1, H2, w, h, disp_min, disp_max, image_apply_homography, compute_disparity_map, erosion,
             height_map=None, write_height_map=None, cargarse_basura=None, merge_n=None, heights_to_ply=None):
    s2p = PT.stub_s2p(monkeypatch, cfg, H1, H2, w, h, disp_min, disp_max, image_apply_homography, compute_disparity_map, erosion,
                      lambda tile: None)
    del s2p.disparity_to_ply

    def remove(path):
        if os.path.exists(path):
            os.remove(path)

    def disparity_to_height(tile, i):
        from s2p_b200 import rasterio_compat as rio
        s2p.calls.append("disparity_to_height")
        out_dir = os.path.join(tile['dir'], 'pair_{}'.format(i))
        x, y, tw, th = tile['coordinates']
        H_ref = os.path.join(out_dir, 'H_ref.txt')
        H_sec = os.path.join(out_dir, 'H_sec.txt')
        disp = os.path.join(out_dir, 'rectified_disp.tif')
        mask = os.path.join(out_dir, 'rectified_mask.png')
        pointing = os.path.join(cfg['out_dir'], 'global_pointing_pair_{}.txt'.format(i))
        hm = height_map(x, y, tw, th, cfg['images'][0]['rpcm'], cfg['images'][i]['rpcm'], np.loadtxt(H_ref), np.loadtxt(H_sec),
                        rio.read_stored(disp).squeeze(), rio.read_stored(mask).squeeze(),
                        rio.read_stored(os.path.join(tile['dir'], 'mask.png')).squeeze(), A=np.loadtxt(pointing))
        write_height_map(os.path.join(out_dir, 'height_map.tif'), hm)          # common.rasterio_write
        if cfg['clean_intermediate']:
            for f in (H_ref, H_sec, disp, mask):
                remove(f)

    def heights_fusion(tile):
        s2p.calls.append("heights_fusion")
        maps = [os.path.join(tile['dir'], 'pair_%d' % (k + 1), 'height_map.tif') for k in range(len(cfg['images']) - 1)]
        if cfg['cargarse_basura']:
            for f in maps:
                cargarse_basura(f, f)
        offsets = [np.loadtxt(os.path.join(cfg['out_dir'], 'global_mean_height_pair_{}.txt'.format(k + 1)))
                   for k in range(len(cfg['images']) - 1)]
        merge_n(os.path.join(tile['dir'], 'height_map.tif'), maps, offsets, averaging=cfg['fusion_operator'],
                threshold=cfg['fusion_thresh'])
        if cfg['clean_intermediate']:
            for f in maps:
                remove(f)

    def step_heights_to_ply(tile):
        s2p.calls.append("heights_to_ply")
        return heights_to_ply(tile)

    s2p.disparity_to_height, s2p.heights_fusion, s2p.heights_to_ply = disparity_to_height, heights_fusion, step_heights_to_ply
    return s2p


def cfg_for(out_dir, imgs, rpcs, algo, clean, basura=True, operator="average_if_close", clr=None):
    cfg = PT.cfg_for(out_dir, imgs[0], imgs[1], rpcs[0], rpcs[1], algo, clean, clr)
    cfg["images"] += [{"img": im, "rpcm": rpc, "clr": None} for im, rpc in zip(imgs[2:], rpcs[2:])]
    cfg.update(cargarse_basura=basura, fusion_operator=operator, fusion_thresh=3.0)
    return cfg


def make_tile(root, name, coordinates, npairs):
    """a tile directory with the files the earlier steps leave: the tile's mask, each pair's pointing and SIFT matches"""
    from s2p_b200 import rasterio_compat as rio
    d = os.path.join(str(root), name)
    _, _, w, h = coordinates
    for i in range(1, npairs + 1):
        os.makedirs(os.path.join(d, "pair_%d" % i))
        np.savetxt(os.path.join(d, "pair_%d" % i, "pointing.txt"), np.eye(3))
        np.savetxt(os.path.join(d, "pair_%d" % i, "sift_matches.txt"), np.zeros((2, 4)))
    rio.write_mask_png(os.path.join(d, "mask.png"), np.ones((h, w), np.uint8))
    return {"dir": d, "coordinates": tuple(coordinates), "neighborhood_dirs": []}


def merge_n_numpy(maps, offsets, averaging, threshold):
    """s2p.fusion.merge_n's arithmetic (s2p/fusion.py:44-66) on maps as rasterio reads them: the stack in float64, minus each
    offset, the operator through np.apply_along_axis, plus np.mean(offsets), stored as float32"""
    def average_if_close(x, threshold):
        if np.nanmax(x) - np.nanmin(x) > threshold:
            return np.nan
        return np.nanmedian(x)

    h, w = maps[0].shape
    x = np.empty((h, w, len(maps)))
    for i, m in enumerate(maps):
        x[:, :, i] = m - offsets[i]
    if averaging.startswith(('np.', 'numpy.')):
        avg = np.apply_along_axis(getattr(np, averaging.split('.')[1]), axis=2, arr=x)
    else:
        avg = np.apply_along_axis(average_if_close, 2, x, threshold)
    avg += np.mean(offsets)
    return np.asarray(avg).astype('float32')


def merge_n_file(output, inputs, offsets, averaging='average_if_close', threshold=1):
    """merge_n_numpy with s2p.fusion.merge_n's file contract, written as the s2p_b200.fusion drop-in writes its result"""
    import shutil
    from s2p_b200 import rasterio_compat as rio
    avg = merge_n_numpy([rio.read_band_stored(f) for f in inputs], offsets, averaging, threshold)
    shutil.copy(inputs[0], output)
    rio.overwrite_band(output, avg)


def files(d):
    return PT.files(d)
