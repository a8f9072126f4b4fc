"""The last per-tile step of s2p on the GPU: ``disparity_to_ply`` (s2p/__init__.py:242-318) and ``heights_to_ply`` (:388-429).

Each step computes a cloud (``disp_to_xyz`` / ``height_map_to_xyz``), filters it (``filter_xyz``), colours it with
``common.linear_stretching_and_quantization_8bit`` and writes it with ``triangulation.write_to_ply``.  Here the whole chain
runs as one device call (``s2pb_disp_to_ply`` / ``s2pb_height_map_to_ply``) and only the records of the kept points come
back; ``write_ply`` puts them behind the header s2p's writer (s2p/ply.py:24-69, through plyfile) writes.

The steps fall through to the original when the device path would not write the reference's file:
- an output CRS other than WGS84 and its UTM zones (the original then uses the installed ``disp_to_xyz`` / filter drop-ins);
- NumPy < 2, whose casting rules make the stretch float32;
- a ``clr`` image: the reference then writes the colours in that image's own type (float32 properties for the pair path's
  warped image), which the uint8 records do not hold;
- colours whose band count the reference refuses, or whose type does not convert exactly to float32 (the original raises or
  stretches them itself).

``install()`` replaces ``s2p.disparity_to_ply`` and ``s2p.heights_to_ply`` and keeps the originals as
``s2p._s2pb_original_*``.
"""
import os

import numpy as np

from . import projection, rasterio_compat, triangulation
from .engine import get_engine

_PLY_TYPES = {"<f8": "double", "<f4": "float", "|u1": "uchar"}
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


def _comments(cfg):
    return ["created by S2P", "projection: {}".format("CRS {}".format(cfg['out_crs']))]


def disparity_to_ply(tile, engine=None):
    """s2p.disparity_to_ply (s2p/__init__.py:242-318): the tile's cloud.ply from the pair's disparity map in one device call."""
    import s2p
    from s2p.config import cfg
    original = getattr(s2p, "_s2pb_original_disparity_to_ply", None)
    target = projection.utm_target(cfg['out_crs'])
    if original is not None and (target is None or cfg['images'][0]['clr'] or not numpy_stretch_is_float64()):
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

    colors = rasterio_compat.read_stored(os.path.join(out_dir, 'pair_1', 'rectified_ref.tif'))
    if original is not None and not _colours_ok(colors):
        return original(tile)
    disp_img = rasterio_compat.read_stored(disp).squeeze()
    mask_rect_img = rasterio_compat.read_stored(mask_rect).squeeze()
    mask_orig_img = rasterio_compat.read_stored(mask_orig).squeeze()
    confidence = rasterio_compat.read_stored(extra).squeeze() if extra else None

    H2 = np.dot(np.loadtxt(H_sec), np.linalg.inv(np.loadtxt(pointing)))   # pointing correction (s2p/triangulation.py:114-115)
    r, p, n = _filter_args(cfg)
    records = (engine or get_engine()).disp_to_ply(
        disp_img, mask_rect_img, mask_orig_img, np.loadtxt(H_ref), H2, triangulation._rpc_struct(rpc1),
        triangulation._rpc_struct(rpc2), (x, x + w, y, y + h), *target, r=r, p=p, n=n, colors=colors, confidence=confidence)
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
    target = projection.utm_target(cfg['out_crs'])
    if original is not None and (target is None or cfg['images'][0]['clr'] or not numpy_stretch_is_float64()):
        return original(tile)
    out_dir = tile['dir']
    x, y, w, h = tile['coordinates']
    colors = rasterio_compat.read_stored(cfg['images'][0]['img'], window=(x, y, w, h))
    if original is not None and not _colours_ok(colors):
        return original(tile)

    # merge the n-1 height maps of the tile (n = nb of images)
    s2p.heights_fusion(tile)

    plyfile = os.path.join(out_dir, 'cloud.ply')
    height_map = os.path.join(out_dir, 'height_map.tif')
    heights = rasterio_compat.read_band_stored(height_map)
    r, p, n = _filter_args(cfg)
    records = (engine or get_engine()).height_map_to_ply(heights, triangulation._rpc_struct(cfg['images'][0]['rpcm']), x, y,
                                                         *target, r=r, p=p, n=n, colors=colors)
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
