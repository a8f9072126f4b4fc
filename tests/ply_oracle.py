"""NumPy restatements of the last step of a tile (``disparity_to_ply`` / ``heights_to_ply``) as the device forms it.

- ``stretch_8bit``: common.linear_stretching_and_quantization_8bit (s2p/common.py:284-297) from two order statistics per
  percentile and numpy's ``_lerp``, the way ``sgbm_select_kernel`` (rule kOrdLinear) and ``stretch_8bit`` in
  cloud_kernels.cuh form it.
- ``ply_records``: the vertex records triangulation.write_to_ply writes (s2p/triangulation.py:392-429 ->
  s2p/ply.py:24-69), vectorised.
- ``ply_records_literal``: the same through the reference's own sequence of numpy calls, one Python tuple per point, without
  plyfile (its writer dumps the structured array as it stands for a binary little-endian file).
"""
import numpy as np


def _linear(n, q):
    """numpy's 'linear' method for n sorted values: (previous rank, next rank, gamma), as _get_indexes and _get_gamma."""
    vi = np.float64(n - 1) * np.float64(q)
    if vi >= n - 1:
        return n - 1, n - 1, vi + 1.0
    f = np.floor(vi)
    return int(f), int(f) + 1, vi - f


def _lerp(a, b, t):
    """numpy's _lerp for float32 neighbours: their difference in float32, the rest in float64"""
    d = np.float64(np.float32(b) - np.float32(a))
    if t >= 0.5:
        return np.float64(b) - d * (1.0 - t)
    return np.float64(a) + d * t


def percentiles(img, p=1):
    """(a, b) = np.nanpercentile(img, (p, 100 - p)) from order statistics: the kernel's formula"""
    v = np.sort(np.asarray(img, np.float32).ravel())
    v = v[~np.isnan(v)]
    n = v.size
    if n == 0:
        return np.nan, np.nan
    out = []
    for q in (p / 100.0, (100.0 - p) / 100.0):
        i, j, g = _linear(n, q)
        out.append(_lerp(v[i], v[j], g))
    return out[0], out[1]


def stretch_8bit(img, p=1):
    """the kernel's stretch: clip as numpy's float loop (max then min, NaN propagates), then the expression in float64"""
    a, b = percentiles(img, p)
    x = np.asarray(img, np.float32).astype(np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        t = np.where(np.isnan(x), x, np.where(x > a, x, a))
        c = np.where(np.isnan(t), t, np.where(t < b, t, b))
        v = np.rint(255.0 * (c - a) / (b - a))
    out = np.zeros(v.shape, np.uint8)
    ok = ~np.isnan(v)
    out[ok] = v[ok].astype(np.uint8)
    return out


def stretch_8bit_reference(img, p=1):
    """s2p/common.py:296-297 as written"""
    a, b = np.nanpercentile(img, (p, 100 - p))
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.round(255 * (np.clip(img, a, b) - a) / (b - a)).astype(np.uint8)


def ply_dtype(nbands=3, confidence=False, color_dtype=np.uint8):
    d = [("x", "<f8"), ("y", "<f8"), ("z", "<f8")]
    if nbands:
        c = np.dtype(color_dtype).newbyteorder("<")
        d += [("red", c), ("green", c), ("blue", c)] + ([("ir", c)] if nbands == 4 else [])
    if confidence:
        d += [("confidence", "<f4")]
    return np.dtype(d)


def ply_records(xyz, colors=None, confidence=None):
    """write_to_ply's records, vectorised: xyz (h, w, 3), colors (nbands, h, w) uint8, confidence (h, w) or None"""
    pts = np.asarray(xyz, np.float64).reshape(-1, 3)
    keep = np.all(np.isfinite(pts), axis=1)
    nb = 0 if colors is None else np.shape(colors)[0]
    if nb not in (0, 1, 3, 4):
        raise Exception('Error: colors must have either 1, 3 or 4 channels')
    rec = np.empty(int(keep.sum()), ply_dtype(nb, confidence is not None))
    for k, name in enumerate("xyz"):
        rec[name] = pts[keep, k]
    if nb:
        c = np.asarray(colors).reshape(nb, -1)[:, keep]
        for k, name in enumerate(("red", "green", "blue", "ir")[:max(nb, 3)]):
            rec[name] = c[0 if nb == 1 else k]
    if confidence is not None:
        rec["confidence"] = np.asarray(confidence).ravel()[keep].astype(np.float32)
    return rec


def ply_records_literal(xyz, colors=None, confidence=None):
    """s2p/triangulation.py:405-429 and s2p/ply.py:42-66 line for line, with the confidence image given as an array (the
    reference reads it from a file with rasterio): the structured array plyfile writes"""
    xyz_list = xyz.reshape(-1, 3)
    valid = np.all(np.isfinite(xyz_list), axis=1)
    colors_list = colors.transpose(1, 2, 0).reshape(-1, colors.shape[0])[valid] if colors is not None else None
    if confidence is not None:
        extra_list = confidence.flatten()[valid].astype(np.float32)
        extra_names = ['confidence']
    else:
        extra_list, extra_names = None, None
    coordinates = xyz_list[valid]
    points = coordinates
    dtypes = [('x', coordinates.dtype), ('y', coordinates.dtype), ('z', coordinates.dtype)]
    if colors_list is not None:
        c = colors_list
        if c.shape[1] == 1:
            c = np.column_stack([c] * 3)
        elif c.shape[1] not in [3, 4]:
            raise Exception('Error: colors must have either 1, 3 or 4 channels')
        points = np.column_stack((points, c))
        dtypes += [('red', c.dtype), ('green', c.dtype), ('blue', c.dtype)]
        if c.shape[1] == 4:
            dtypes += [('ir', c.dtype)]
    if extra_list is not None:
        points = np.column_stack((points, extra_list))
        dtypes += [(s, extra_list.dtype) for s in extra_names]
    tuples = [tuple(x) for x in points]
    return np.asarray(tuples, dtype=dtypes)


def ply_header(n, comments, nbands=3, confidence=False, color_type="uchar"):
    """the header plyfile writes for write_to_ply's vertex element"""
    lines = ["ply", "format binary_little_endian 1.0"] + ["comment " + c for c in comments]
    lines += ["element vertex %d" % n, "property double x", "property double y", "property double z"]
    if nbands:
        lines += ["property %s %s" % (color_type, c) for c in ("red", "green", "blue", "ir")[:4 if nbands == 4 else 3]]
    if confidence:
        lines += ["property float confidence"]
    return ("\n".join(lines + ["end_header"]) + "\n").encode("ascii")
