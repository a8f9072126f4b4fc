"""Opt-in fusion of pipeline steps 3 and 4 (SURVEY.md section 8f rank 3): rectify the pair and match it in ONE call, the
rectified images staying on the device between the two.

In the reference, `rectification_pair` (s2p/__init__.py:147-155) writes `rectified_ref.tif` / `rectified_sec.tif` through two
`homography` subprocesses, and `stereo_matching` (s2p/__init__.py:184-190) reads them back in another worker process to
run `mgm`.  The two steps run in different `multiprocessing.Pool`s (s2p/parallel.py:80), so device memory cannot be handed
from one to the other without changing s2p/__init__.py; the drop-ins of `common.py` and `block_matching.py` therefore keep the
file hand-off.  A pipeline that calls both steps from the same worker can use `rectify_and_match` instead: same files out
(rectified pair, disparity, confidence, mask), bit-identical to the two-step path, one TIFF decode and two host<->device
round trips fewer per tile.  INTEGRATION.md shows the ten lines of s2p/__init__.py this replaces.

With two images, `pair_tile` goes further: steps 3, 4 and 5 of a tile (rectification_pair, stereo_matching, disparity_to_ply)
in one device call from the source images to cloud.ply, the intermediates written only where s2p keeps them (INTEGRATION.md
section 2b).  With three or more, `pair_heights` runs steps 3, 4 and 5a of one pair (rectification_pair, stereo_matching,
disparity_to_height) in one device call down to the pair's height map, and `heights_tile` step 5d (heights_to_ply with its
heights_fusion) in another, from the pairs' height maps to cloud.ply.
"""
import os
import shutil
import subprocess

import numpy as np

from . import _lib, cloud, common, projection, rasterio_compat as rio, triangulation
from .block_matching import _NATIVE, SGBM_ARGS, confidence_path, disparity_bounds, matcher_params
from .common import needed_roi
from .engine import Engine, S2pbError, census_window_served, get_engine


def _crop(im, H, w, h):
    """the part of image file `im` the warp needs (s2p_b200.common.image_apply_homography does the same), crop-compensated H"""
    H = np.asarray(H, dtype=np.float64).reshape(3, 3)
    sw, sh = rio.image_size(im)
    x, y, rw, rh = needed_roi(H, w, h)
    if x < 0:
        rw += x
        x = 0
    if y < 0:
        rh += y
        y = 0
    rw, rh = min(rw, sw - x), min(rh, sh - y)
    if rw <= 0 or rh <= 0:
        raise subprocess.CalledProcessError(1, ["s2pb200:homography", im], output="ERROR: empty roi")
    return rio.read_window(im, x, y, rw, rh), H @ np.array([[1, 0, x], [0, 1, y], [0, 0, 1]], dtype=np.float64)


def rectify_and_match(out1, out2, disp, mask, im1, im2, H1, H2, w, h, algo, disp_min, disp_max, timeout=600, max_disp_range=None):
    """image_apply_homography(out1, im1, H1, w, h); image_apply_homography(out2, im2, H2, w, h);
    compute_disparity_map(out1, out2, disp, mask, algo, disp_min, disp_max, timeout, max_disp_range) -- in one device call."""
    if algo not in _NATIVE or algo == "mgm_multi_lsd":
        raise NotImplementedError("the fused path serves algo 'mgm' and 'mgm_multi'")
    disp_min, disp_max = disparity_bounds(w, disp_min, disp_max, max_disp_range)
    src1, H1c = _crop(im1, H1, w, h)
    src2, H2c = _crop(im2, H2, w, h)
    cmd = ["s2pb200:rectify+%s" % algo, im1, im2, disp]
    print("\nRUN: %s" % " ".join(cmd))
    try:
        out = get_engine().rectify_match(src1, H1c, src2, H2c, w, h, disp_min, disp_max, matcher_params(algo, timeout))
    except S2pbError as e:
        if e.code == _lib.ERR_TIMEOUT:
            raise subprocess.TimeoutExpired(cmd, timeout) from e
        raise subprocess.CalledProcessError(-e.code, cmd, output=str(e)) from e
    rio.write_float_tiff(out1, out["rect1"])
    rio.write_float_tiff(out2, out["rect2"])
    rio.write_float_tiff(disp, out["disp"])
    rio.write_float_tiff(confidence_path(disp, algo), out["conf"])
    rio.write_mask_png(mask, out["mask"])


# ------------------------------------------------------------------ steps 3 to 5 of a two-view tile in one device call

SERVED = ("mgm", "mgm_multi", "mgm_multi_lsd", "sgbm")
CONFIDENCE_COLUMN = ("mgm", "mgm_multi")    # the algos whose confidence file disparity_to_ply finds at `extra`


def fall_through_reason(cfg):
    """Why ``pair_tile`` runs the three steps instead of the device call for this configuration, or None."""
    if len(cfg['images']) != 2:
        return "not a two-view run"
    if cfg['matching_algorithm'] not in SERVED:
        return "algo %r is not served" % cfg['matching_algorithm']
    window = _window_unserved(cfg)
    if window:
        return window
    if projection.output_target(cfg['out_crs']) is None:
        return projection.unserved_reason(cfg['out_crs'])
    if not cloud.numpy_stretch_is_float64():
        return "NumPy < 2 stretches the colours in float32"
    clr = cfg['images'][0]['clr']
    if clr and not cloud._clr_bands_ok(clr):
        return "the clr image does not open with 1, 3 or 4 bands"
    return None


def _window_unserved(cfg):
    """the reason when the matcher's census window (the mgm algos' CENSUS_NCC_WIN; s2p's default is 5) is one the device does
    not serve, or None"""
    win = cfg.get('census_ncc_win', 5)
    if cfg['matching_algorithm'] in _NATIVE and not census_window_served(win):
        return "census_ncc_win %r is not served" % win
    return None


def erosion_radius(radius):
    """masking.erosion's radius as the device call takes it: nothing happens below 2 (s2p/masking.py:87-97)"""
    return int(radius) if radius >= 2 else 0


def _stepwise(s2p, tile):
    s2p.rectification_pair(tile, 1)
    s2p.stereo_matching(tile, 1)
    s2p.disparity_to_ply(tile)


def _rectify(s2p, tile, i):
    """s2p's own ``rectification_pair(tile, i)`` with its two ``common.image_apply_homography`` calls recorded instead of run
    -> (the recorded calls (out, im, H, w, h), the warp they would have run)"""
    import s2p.common as s2p_common
    calls = []
    saved = s2p_common.image_apply_homography
    s2p_common.image_apply_homography = lambda out, im, H, ww, hh: calls.append((out, im, H, ww, hh))
    try:
        s2p.rectification_pair(tile, i)
    finally:
        s2p_common.image_apply_homography = saved
    if len(calls) != 2 or calls[0][3:] != calls[1][3:]:
        raise RuntimeError("rectify_pair did not warp its two images the way s2p/rectification.py:379-380 does")
    return calls, saved


def _matcher_inputs(cfg, calls, pair_dir):
    """What stereo_matching hands to the matcher of the pair in pair_dir, read without the rectified files: -> (src1, H1c, src2,
    H2c, w, h, disp_min, disp_max, params, weights).  Raises MaxDisparityRangeError before any image is read."""
    (_, im1, H1, w, h), (_, im2, H2, _, _) = calls
    algo = cfg['matching_algorithm']
    disp_min, disp_max = np.loadtxt(os.path.join(pair_dir, 'disp_min_max.txt'))
    disp_min, disp_max = disparity_bounds(w, disp_min, disp_max, cfg['max_disp_range'])
    src1, H1c = _crop(im1, H1, w, h)
    src2, H2c = _crop(im2, H2, w, h)
    if algo == "sgbm":
        params, weights = Engine.sgbm_params(**SGBM_ARGS), None
    else:
        params = matcher_params(algo, cfg['mgm_timeout'])
        weights = (np.ones((h, w), np.float32),) * 2 if algo == "mgm_multi_lsd" else None     # block_matching.lsd_weight_map
    return src1, H1c, src2, H2c, w, h, disp_min, disp_max, params, weights


def _pointing_corrected(pair_dir, out_dir, i):
    """(H_ref, H_sec . A^-1) of pair i, from its text files and global_pointing_pair_i.txt (s2p/triangulation.py:114-115)"""
    H_ref = np.loadtxt(os.path.join(pair_dir, 'H_ref.txt'))
    H_sec = np.dot(np.loadtxt(os.path.join(pair_dir, 'H_sec.txt')),
                   np.linalg.inv(np.loadtxt(os.path.join(out_dir, 'global_pointing_pair_{}.txt'.format(i)))))
    return H_ref, H_sec


def pair_tile(tile, engine=None):
    """``rectification_pair(tile, 1)``, ``stereo_matching(tile, 1)`` and ``disparity_to_ply(tile)`` of a two-view run
    (s2p/__init__.py:102-318) with one device call between the rectification's host algebra and cloud.ply.

    ``rectification_pair`` itself runs -- pointing, SIFT matches and those of the neighbours, ``rectify_pair``'s algebra, the text
    files it writes and removes -- with its two ``common.image_apply_homography`` calls intercepted; then ``s2pb_pair_tile_to_ply``
    warps, matches, erodes and triangulates, and only the files the three steps leave are written, byte for byte: with
    ``clean_intermediate`` none of the rasters that ``stereo_matching`` and ``disparity_to_ply`` would delete.  The three steps
    run instead whenever ``fall_through_reason`` gives one, and when the device refuses the tile as unsupported.  Raises
    MaxDisparityRangeError before any device work and subprocess.TimeoutExpired as ``compute_disparity_map`` does."""
    import s2p
    from s2p.config import cfg
    if fall_through_reason(cfg):
        return _stepwise(s2p, tile)

    calls, saved = _rectify(s2p, tile, 1)
    (rect1, im1, _, _, _), (rect2, im2, _, _, _) = calls
    out_dir = tile['dir']
    pair_dir = os.path.join(out_dir, 'pair_1')
    algo = cfg['matching_algorithm']
    clean = cfg['clean_intermediate']
    src1, H1c, src2, H2c, w, h, disp_min, disp_max, params, weights = _matcher_inputs(cfg, calls, pair_dir)
    eng = engine or get_engine()
    x, y, tw, th = tile['coordinates']
    H_ref, H_sec = _pointing_corrected(pair_dir, cfg['out_dir'], 1)
    mask_orig = os.path.join(out_dir, 'mask.png')
    r, p, n = cloud._filter_args(cfg)
    clr, hc = None, None
    ply_file = os.path.join(out_dir, 'cloud.ply')
    if cfg['images'][0]['clr']:
        im = cfg['images'][0]['clr']
        clr, hc = common.homography_crop(im, H_ref, w, h, common.homography_cmd("<colours of %s>" % ply_file, im, H_ref, w, h))
    conf_file = confidence_path(os.path.join(pair_dir, 'rectified_disp.tif'), algo) if algo != "sgbm" else None
    want = () if clean else ("rect1", "rect2", "disp", "mask")
    if conf_file:
        want += ("conf",)

    cmd = ["s2pb200:rectify+%s+ply" % algo, im1, im2, ply_file]
    print("\nRUN: %s" % " ".join(cmd))
    try:
        records, out = eng.pair_tile_to_ply(
            src1, H1c, src2, H2c, w, h, disp_min, disp_max, rio.read_stored(mask_orig).squeeze(), H_ref, H_sec,
            triangulation._rpc_struct(cfg['images'][0]['rpcm']), triangulation._rpc_struct(cfg['images'][1]['rpcm']),
            (x, x + tw, y, y + th), *projection.output_target(cfg['out_crs'], eng), params=params, weights=weights,
            erode_radius=erosion_radius(cfg['msk_erosion']), r=r, p=p, n=n, clr=clr, hc=hc,
            confidence=algo in CONFIDENCE_COLUMN, want=want)
    except S2pbError as e:
        if e.code == _lib.ERR_TIMEOUT:
            raise subprocess.TimeoutExpired(cmd, cfg['mgm_timeout']) from e
        if e.code == _lib.ERR_UNSUPPORTED:      # the steps' own handling of the tile (their error or the original tool)
            for out_file, im, H, ww, hh in calls:
                saved(out_file, im, H, ww, hh)
            s2p.stereo_matching(tile, 1)
            return s2p.disparity_to_ply(tile)
        raise subprocess.CalledProcessError(-e.code, cmd, output=str(e)) from e

    if not clean:
        rio.write_float_tiff(rect1, out["rect1"])
        rio.write_float_tiff(rect2, out["rect2"])
        rio.write_float_tiff(os.path.join(pair_dir, 'rectified_disp.tif'), out["disp"])
        rio.write_mask_png(os.path.join(pair_dir, 'rectified_mask.png'), out["mask"])
    if conf_file:
        rio.write_float_tiff(conf_file, out["conf"])
    cloud.write_ply(ply_file, records, cloud._comments(cfg))
    if clean:
        for f in ('disp_min_max.txt', 'H_ref.txt', 'H_sec.txt'):
            cloud._remove(os.path.join(pair_dir, f))
        cloud._remove(mask_orig)


# ------------------------------------------------------------------ steps 3 to 5 of a tri-stereo tile in two device calls

def pair_heights_fall_through_reason(cfg):
    """Why ``pair_heights`` runs the three steps instead of the device call for this configuration, or None.  Nothing in
    these steps depends on the output CRS, the colours or the NumPy version."""
    if len(cfg['images']) <= 2:
        return "not a tri-stereo run"
    if cfg['matching_algorithm'] not in SERVED:
        return "algo %r is not served" % cfg['matching_algorithm']
    return _window_unserved(cfg)


def pair_heights(tile, i, engine=None):
    """``rectification_pair(tile, i)``, ``stereo_matching(tile, i)`` and ``disparity_to_height(tile, i)`` of pair i of a run
    with three or more images (s2p/__init__.py:102-239) with one device call between the rectification's host algebra and
    the pair's height map.

    ``rectification_pair`` runs as in ``pair_tile``, with its two warps intercepted; then ``s2pb_pair_tile_to_height_map``
    warps, matches, erodes and triangulates the pair onto the tile's grid, and only the files the three steps leave are
    written, byte for byte: pair_i/height_map.tif in float64 as ``common.rasterio_write`` writes it, and, without
    ``clean_intermediate``, the rectified pair, the disparity, its confidence and the eroded mask; with it, only the height map
    and the confidence file, which the cleaning of these steps keeps.  The tile's mask.png stays for the other pairs and
    step 5d.  The three steps run instead whenever ``pair_heights_fall_through_reason`` gives one, and when the device refuses
    the pair as unsupported.  Raises MaxDisparityRangeError before any device work and subprocess.TimeoutExpired as
    ``compute_disparity_map`` does."""
    import s2p
    from s2p.config import cfg
    if pair_heights_fall_through_reason(cfg):
        s2p.rectification_pair(tile, i)
        s2p.stereo_matching(tile, i)
        return s2p.disparity_to_height(tile, i)

    calls, saved = _rectify(s2p, tile, i)
    (rect1, im1, _, _, _), (rect2, im2, _, _, _) = calls
    out_dir = tile['dir']
    pair_dir = os.path.join(out_dir, 'pair_{}'.format(i))
    algo = cfg['matching_algorithm']
    clean = cfg['clean_intermediate']
    src1, H1c, src2, H2c, w, h, disp_min, disp_max, params, weights = _matcher_inputs(cfg, calls, pair_dir)
    eng = engine or get_engine()
    H_ref, H_sec = _pointing_corrected(pair_dir, cfg['out_dir'], i)
    height_map = os.path.join(pair_dir, 'height_map.tif')
    conf_file = confidence_path(os.path.join(pair_dir, 'rectified_disp.tif'), algo) if algo != "sgbm" else None
    want = () if clean else ("rect1", "rect2", "disp", "mask")
    if conf_file:
        want += ("conf",)

    cmd = ["s2pb200:rectify+%s+height" % algo, im1, im2, height_map]
    print("\nRUN: %s" % " ".join(cmd))
    try:
        heights, out = eng.pair_tile_to_height_map(
            src1, H1c, src2, H2c, w, h, disp_min, disp_max, rio.read_stored(os.path.join(out_dir, 'mask.png')).squeeze(), H_ref,
            H_sec, triangulation._rpc_struct(cfg['images'][0]['rpcm']), triangulation._rpc_struct(cfg['images'][i]['rpcm']),
            tile['coordinates'], params=params, weights=weights, erode_radius=erosion_radius(cfg['msk_erosion']), want=want)
    except S2pbError as e:
        if e.code == _lib.ERR_TIMEOUT:
            raise subprocess.TimeoutExpired(cmd, cfg['mgm_timeout']) from e
        if e.code == _lib.ERR_UNSUPPORTED:      # the steps' own handling of the pair (their error or the original tool)
            for out_file, im, H, ww, hh in calls:
                saved(out_file, im, H, ww, hh)
            s2p.stereo_matching(tile, i)
            return s2p.disparity_to_height(tile, i)
        raise subprocess.CalledProcessError(-e.code, cmd, output=str(e)) from e

    if not clean:
        rio.write_float_tiff(rect1, out["rect1"])
        rio.write_float_tiff(rect2, out["rect2"])
        rio.write_float_tiff(os.path.join(pair_dir, 'rectified_disp.tif'), out["disp"])
        rio.write_mask_png(os.path.join(pair_dir, 'rectified_mask.png'), out["mask"])
    if conf_file:
        rio.write_float_tiff(conf_file, out["conf"])
    rio.write_float64_tiff(height_map, heights)
    if clean:
        for f in ('disp_min_max.txt', 'H_ref.txt', 'H_sec.txt'):
            cloud._remove(os.path.join(pair_dir, f))


def _fusion_operator(name):
    return "np." + name[6:] if name.startswith("numpy.") else name


def heights_tile_fall_through_reason(cfg):
    """Why ``heights_tile`` hands the tile to ``s2p.heights_to_ply`` for this configuration, or None (the colours are looked
    at in ``heights_tile``, as ``cloud.heights_to_ply`` looks at them)."""
    if projection.output_target(cfg['out_crs']) is None:
        return projection.unserved_reason(cfg['out_crs'])
    if not cloud.numpy_stretch_is_float64():
        return "NumPy < 2 stretches the colours in float32"
    if _fusion_operator(cfg['fusion_operator']) not in Engine.FUSION_OPS:
        return "fusion operator %r is not served" % cfg['fusion_operator']
    if len(cfg['images']) - 1 > _lib.MAX_FUSION:
        return "more than %d height maps" % _lib.MAX_FUSION
    return None


def heights_tile(tile, engine=None):
    """``heights_to_ply(tile)`` of a run with three or more images, its ``heights_fusion`` included (s2p/__init__.py:355-429),
    in one device call from the pairs' height maps to cloud.ply.

    The n-1 pair_k/height_map.tif are read in the type they are stored in (float64 as ``pair_heights`` and s2p's
    ``disparity_to_height`` write them) with the global_mean_height_pair_k.txt offsets; ``s2pb_heights_tile_to_ply`` cleans them
    (``cargarse_basura``), merges them (``merge_n``, a float64 map subtracted from its offset in float64 as s2p/fusion.py:49
    does) and localises, filters, colours and packs the merged map.  Then the files the step leaves are written, byte for
    byte as the drop-ins write them: the cleaned pair maps (float32, each with its own metadata), height_map.tif (a copy of the
    first pair map with the merged band) and cloud.ply; with ``clean_intermediate`` only cloud.ply, and the pair maps and the
    tile's mask.png are removed.  ``s2p.heights_to_ply`` runs instead whenever ``heights_tile_fall_through_reason`` gives
    one, when the colours are ones ``cloud.heights_to_ply`` hands to the original, and when the device refuses the tile as
    unsupported.  A missing pair map raises, as the reference's merge_n does."""
    import s2p
    from s2p.config import cfg
    if heights_tile_fall_through_reason(cfg):
        return s2p.heights_to_ply(tile)
    out_dir = tile['dir']
    x, y, w, h = tile['coordinates']
    clr = cfg['images'][0]['clr']
    if clr:
        colors = cloud._clr_window(clr, (x, y, w, h))
        if colors is None:
            return s2p.heights_to_ply(tile)
    else:
        colors = rio.read_stored(cfg['images'][0]['img'], window=(x, y, w, h))
        if not cloud._colours_ok(colors):
            return s2p.heights_to_ply(tile)

    nmaps = len(cfg['images']) - 1
    height_maps = [os.path.join(out_dir, 'pair_%d' % (k + 1), 'height_map.tif') for k in range(nmaps)]
    maps = [rio.read_band_stored(f) for f in height_maps]
    offsets = [np.loadtxt(os.path.join(cfg['out_dir'], 'global_mean_height_pair_{}.txt'.format(k + 1))) for k in range(nmaps)]
    basura, clean = bool(cfg['cargarse_basura']), cfg['clean_intermediate']
    want = () if clean else ("merged",) + (("cleaned",) if basura else ())
    r, p, n = cloud._filter_args(cfg)
    ply_file = os.path.join(out_dir, 'cloud.ply')
    eng = engine or get_engine()
    try:
        records, out = eng.heights_tile_to_ply(
            maps, offsets, triangulation._rpc_struct(cfg['images'][0]['rpcm']), x, y, *projection.output_target(cfg['out_crs'], eng),
            cargarse_basura=basura, averaging=_fusion_operator(cfg['fusion_operator']), threshold=cfg['fusion_thresh'], r=r, p=p,
            n=n, colors=None if clr else colors, clr=colors if clr else None, want=want)
    except S2pbError as e:
        if e.code == _lib.ERR_UNSUPPORTED:      # the step's own handling of the tile (its error or the original tools)
            return s2p.heights_to_ply(tile)
        raise

    if not clean:
        if basura:                              # in place, as heights_fusion runs cargarse_basura(img, img)
            for f, m in zip(height_maps, out["cleaned"]):
                rio.write_float_tiff_like(f, m, f)
        height_map = os.path.join(out_dir, 'height_map.tif')
        shutil.copy(height_maps[0], height_map)  # keeps the metadata of the first input (s2p/fusion.py:64)
        rio.overwrite_band(height_map, out["merged"])
    cloud.write_ply(ply_file, records, cloud._comments(cfg))
    if clean:
        for f in height_maps:
            cloud._remove(f)
        cloud._remove(os.path.join(out_dir, 'mask.png'))
