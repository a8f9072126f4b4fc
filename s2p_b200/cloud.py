"""The last per-tile step of s2p on the GPU: ``disparity_to_ply`` (s2p/__init__.py:242-318) and ``heights_to_ply`` (:388-429).

Each step computes a cloud (``disp_to_xyz`` / ``height_map_to_xyz``), filters it (``filter_xyz``), colours it with
``common.linear_stretching_and_quantization_8bit`` and writes it with ``triangulation.write_to_ply``.  Here the whole chain
runs as one device call (``s2pb_disp_to_ply`` / ``s2pb_height_map_to_ply``) and only the records of the kept points come
back; ``write_ply`` puts them behind the header s2p's writer (s2p/ply.py:24-69, through plyfile) writes.

With a ``clr`` image (``cfg['images'][0]['clr']``) the reference writes that image's colours in their own type, without the
stretch: for the pair, the float32 warp of the image onto the rectified reference's grid (s2p/__init__.py:270-280), which
runs on the device inside the same call (``s2pb_disp_to_ply_clr``) from the crop the warp reads (``common.homography_crop``),
with no temporary file; for tri-stereo, the tile's window of the image in its stored type (:404-406,
``s2pb_height_map_to_ply_clr``).

The steps fall through to the original when the device path would not write the reference's file:
- an output CRS other than WGS84, its UTM zones, the ETRS89 UTM zones and the RGF93 v1 Lambert grids, with or without EGM96
  heights (those only where the grid is found; ``projection.output_target``; the original then uses the installed
  ``disp_to_xyz`` / filter drop-ins);
- NumPy < 2, whose casting rules make the stretch float32;
- colours whose band count the reference refuses, or whose type does not convert exactly to float32 (the original raises or
  stretches them itself);
- a ``clr`` image that cannot be opened (the original raises its own error), whose band count is not 1, 3 or 4, whose type
  plyfile does not write (e.g. int64, uint64, float16), or whose warp or window does not have the shape of the tile's map.

``install()`` replaces ``s2p.disparity_to_ply`` and ``s2p.heights_to_ply`` and keeps the originals as
``s2p._s2pb_original_*``.
"""
import os

import numpy as np

from . import common, projection, rasterio_compat, triangulation
from .engine import get_engine

# the property types plyfile writes, by numpy type
_PLY_TYPES = {"<f8": "double", "<f4": "float", "|u1": "uchar", "|i1": "char", "<i2": "short", "<u2": "ushort", "<i4": "int",
              "<u4": "uint"}
_STRETCHABLE = (np.uint8, np.uint16, np.float32)      # convert to float32 exactly; numpy subtracts their neighbours exactly


def ply_header(records, comments=()):
    """the header plyfile writes for one binary little-endian vertex element with the fields of records.dtype"""
    lines = ["ply", "format binary_little_endian 1.0"] + ["comment %s" % c for c in comments]
    lines.append("element vertex %d" % len(records))
    for name in records.dtype.names:
        lines.append("property %s %s" % (_PLY_TYPES[records.dtype[name].str], name))
    lines.append("end_header")
    return ("\n".join(lines) + "\n").encode("ascii")


def write_ply(path, records, comments=()):
    """The file ply.write_3d_point_cloud_to_ply writes (s2p/ply.py:24-69) for the structured vertex records ``records``
    (Engine.ply_dtype): the header, then the records as they lie in memory."""
    records = np.ascontiguousarray(records)
    with open(path, "wb") as f:
        f.write(ply_header(records, comments))
        f.write(records.tobytes())


def numpy_stretch_is_float64():
    """NumPy >= 2 forms the stretch in float64 (NEP 50), which is what the device reproduces"""
    return int(np.__version__.split(".")[0]) >= 2


def _remove(path):
    """s2p.common.remove"""
    try:
        os.remove(path)
    except OSError:
        pass


def _filter_args(cfg):
    """(r, p, n) of `if r and n: filter_xyz(xyz, r, n, cfg['gsd'])`; n = 0 turns the filter off"""
    r, n = cfg['3d_filtering_r'], cfg['3d_filtering_n']
    if r and n:
        return float(r), int(np.ceil(r / cfg['gsd']).astype(int)), int(n)
    return 0.0, 0, 0


def _colours_ok(colors):
    return colors.ndim == 3 and colors.shape[0] in (1, 3, 4) and colors.dtype.type in _STRETCHABLE


def _clr_bands_ok(path):
    """the clr image opens and has 1, 3 or 4 bands"""
    try:
        return rasterio_compat.band_count(path) in (1, 3, 4)
    except Exception:
        return False


def _clr_window(path, window):
    """the window (x, y, w, h) of the clr image in its stored type, or None when the device cannot write its colours as the
    reference does: the image does not open, or its band count, type or window shape is not one write_to_ply writes"""
    try:
        colors = rasterio_compat.read_stored(path, window=window)
    except Exception:
        return None
    ok = (colors.ndim == 3 and colors.shape[0] in (1, 3, 4) and colors.shape[1:] == (window[3], window[2]) and
          colors.dtype.newbyteorder("<").str in _PLY_TYPES)
    return colors if ok else None


def _comments(cfg):
    return ["created by S2P", "projection: {}".format("CRS {}".format(cfg['out_crs']))]


def disparity_to_ply(tile, engine=None):
    """s2p.disparity_to_ply (s2p/__init__.py:242-318): the tile's cloud.ply from the pair's disparity map in one device call."""
    import s2p
    from s2p.config import cfg
    original = getattr(s2p, "_s2pb_original_disparity_to_ply", None)
    target = projection.output_target(cfg['out_crs'])
    clr = cfg['images'][0]['clr']
    if original is not None and (target is None or not numpy_stretch_is_float64() or (clr and not _clr_bands_ok(clr))):
        return original(tile)
    out_dir = tile['dir']
    ply_file = os.path.join(out_dir, 'cloud.ply')
    x, y, w, h = tile['coordinates']
    rpc1 = cfg['images'][0]['rpcm']
    rpc2 = cfg['images'][1]['rpcm']

    print('triangulating tile {} {}...'.format(x, y))
    H_ref = os.path.join(out_dir, 'pair_1', 'H_ref.txt')
    H_sec = os.path.join(out_dir, 'pair_1', 'H_sec.txt')
    pointing = os.path.join(cfg['out_dir'], 'global_pointing_pair_1.txt')
    disp = os.path.join(out_dir, 'pair_1', 'rectified_disp.tif')
    extra = os.path.join(out_dir, 'pair_1', 'rectified_disp_confidence.tif')
    if not os.path.exists(extra):    # confidence file not always generated
        extra = ''
    mask_rect = os.path.join(out_dir, 'pair_1', 'rectified_mask.png')
    mask_orig = os.path.join(out_dir, 'mask.png')

    rectified_ref = os.path.join(out_dir, 'pair_1', 'rectified_ref.tif')
    colors = None
    if clr:
        # the colours of the clr image warped onto the grid of rectified_ref.tif (s2p/__init__.py:270-280)
        ww, hh = rasterio_compat.image_size(rectified_ref)
    else:
        colors = rasterio_compat.read_stored(rectified_ref)
        if original is not None and not _colours_ok(colors):
            return original(tile)
    disp_img = rasterio_compat.read_stored(disp).squeeze()
    if original is not None and clr and disp_img.shape != (hh, ww):
        return original(tile)
    mask_rect_img = rasterio_compat.read_stored(mask_rect).squeeze()
    mask_orig_img = rasterio_compat.read_stored(mask_orig).squeeze()
    confidence = rasterio_compat.read_stored(extra).squeeze() if extra else None

    H1 = np.loadtxt(H_ref)
    H2 = np.dot(np.loadtxt(H_sec), np.linalg.inv(np.loadtxt(pointing)))   # pointing correction (s2p/triangulation.py:114-115)
    r, p, n = _filter_args(cfg)
    eng = engine or get_engine()
    cloud = (disp_img, mask_rect_img, mask_orig_img, H1, H2, triangulation._rpc_struct(rpc1), triangulation._rpc_struct(rpc2),
             (x, x + w, y, y + h), *projection.output_target(cfg['out_crs'], eng))
    if clr:
        crop, hc = common.homography_crop(clr, H1, ww, hh, common.homography_cmd("<colours of %s>" % ply_file, clr, H1, ww, hh))
        records = eng.disp_to_ply_clr(*cloud, r=r, p=p, n=n, clr=crop, hc=hc, confidence=confidence)
    else:
        records = eng.disp_to_ply(*cloud, r=r, p=p, n=n, colors=colors, confidence=confidence)
    write_ply(ply_file, records, _comments(cfg))

    if cfg['clean_intermediate']:
        _remove(H_ref)
        _remove(H_sec)
        _remove(disp)
        _remove(mask_rect)
        _remove(mask_orig)
        _remove(os.path.join(out_dir, 'pair_1', 'rectified_ref.tif'))


def heights_to_ply(tile, engine=None):
    """s2p.heights_to_ply (s2p/__init__.py:388-429): heights_fusion, then the tile's cloud.ply from the merged height map in
    one device call."""
    import s2p
    from s2p.config import cfg
    original = getattr(s2p, "_s2pb_original_heights_to_ply", None)
    target = projection.output_target(cfg['out_crs'])
    if original is not None and (target is None or not numpy_stretch_is_float64()):
        return original(tile)
    out_dir = tile['dir']
    x, y, w, h = tile['coordinates']
    clr = cfg['images'][0]['clr']
    if clr:
        colors = _clr_window(clr, (x, y, w, h))
        if colors is None:
            if original is not None:
                return original(tile)
            raise ValueError("%s: the device does not write the colours of this image" % clr)
    else:
        colors = rasterio_compat.read_stored(cfg['images'][0]['img'], window=(x, y, w, h))
        if original is not None and not _colours_ok(colors):
            return original(tile)

    # merge the n-1 height maps of the tile (n = nb of images)
    s2p.heights_fusion(tile)

    plyfile = os.path.join(out_dir, 'cloud.ply')
    height_map = os.path.join(out_dir, 'height_map.tif')
    heights = rasterio_compat.read_band_stored(height_map)
    r, p, n = _filter_args(cfg)
    eng = engine or get_engine()
    cloud = (heights, triangulation._rpc_struct(cfg['images'][0]['rpcm']), x, y, *projection.output_target(cfg['out_crs'], eng))
    if clr:
        records = eng.height_map_to_ply_clr(*cloud, r=r, p=p, n=n, colors=colors)
    else:
        records = eng.height_map_to_ply(*cloud, r=r, p=p, n=n, colors=colors)
    write_ply(plyfile, records, _comments(cfg))

    if cfg['clean_intermediate']:
        _remove(height_map)
        _remove(os.path.join(out_dir, 'mask.png'))


def install():
    import s2p
    for name, fn in (("disparity_to_ply", disparity_to_ply), ("heights_to_ply", heights_to_ply)):
        if not hasattr(s2p, name):
            continue
        if not hasattr(s2p, "_s2pb_original_" + name):
            setattr(s2p, "_s2pb_original_" + name, getattr(s2p, name))
        setattr(s2p, name, fn)
    return s2p
