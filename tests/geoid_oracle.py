"""The EGM96 step of the compound output CRS (csrc/projection_kernels.cuh, geoid_undulation) restated in float64 numpy, seeded
smooth global grids, and a minimal GeoTIFF writer for grid files like PROJ's us_nga_egm96_15.tif (no GDAL needed)."""
import struct
import zlib

import numpy as np


def undulation(grid, lon, lat):
    """N(lon, lat) for arrays of |lat| <= 90 and finite lon: the kernel's rule, operation for operation"""
    g = np.asarray(grid.values, np.float32)
    h, w = g.shape
    lon, lat = np.asarray(lon, np.float64), np.asarray(lat, np.float64)
    t = np.fmod(lon - grid.lon0, 360.0)
    t = np.where(t < 0.0, t + 360.0, t)
    x, y = t / grid.dlon, (grid.lat0 - lat) / grid.dlat
    i = np.minimum(np.floor(x).astype(np.int64), w - 1)
    j = np.clip(np.floor(y).astype(np.int64), 0, h - 1)
    fx, fy = x - i, y - j
    i2 = np.where(i + 1 < w, i + 1, 0)
    j2 = np.minimum(j + 1, h - 1)
    a, b = g[j, i].astype(np.float64), g[j, i2].astype(np.float64)
    c, d = g[j2, i].astype(np.float64), g[j2, i2].astype(np.float64)
    top, bottom = a + fx * (b - a), c + fx * (d - c)
    return top + fy * (bottom - top)


def shift(lla, grid):
    """(lon, lat, alt) -> (lon, lat, alt - N) where the point is finite; NaN stays NaN"""
    out = np.array(lla, np.float64)
    ok = np.isfinite(out).all(axis=-1)
    out[..., 2][ok] = out[..., 2][ok] - undulation(grid, out[..., 0][ok], out[..., 1][ok])
    out[~ok] = np.nan
    return out


def smooth_grid(seed, step=0.25, amplitude=100.0, constant=None):
    """a global north-up grid at `step` degrees (node-registered: 360 / step columns from -180, rows from 90 to -90): a
    seeded sum of low-order waves within +-amplitude metres, or `constant` everywhere"""
    from s2p_b200.projection import GeoidGrid
    w, h = int(round(360 / step)), int(round(180 / step)) + 1
    lon = np.radians(-180.0 + step * np.arange(w))[None, :]
    lat = np.radians(90.0 - step * np.arange(h))[:, None]
    if constant is not None:
        v = np.full((h, w), constant, np.float32)
    else:
        rng = np.random.default_rng(seed)
        v = np.zeros((h, w))
        for _ in range(8):
            m, k = rng.integers(1, 7), rng.integers(0, 7)
            v += rng.uniform(-1, 1) * np.cos(m * lon + rng.uniform(0, 2 * np.pi)) * np.cos(lat) ** k * np.sin(k * lat + rng.uniform(0, 6))
        v = (amplitude * v / np.abs(v).max()).astype(np.float32)
    return GeoidGrid(v, -180.0, 90.0, step, step)


def _tag(tag, typ, values):
    fmt = {2: "s", 3: "H", 4: "I", 12: "d"}[typ]
    if typ == 2:
        raw = values.encode("latin-1") + b"\0"
        return tag, typ, len(raw), raw
    return tag, typ, len(values), struct.pack("<" + fmt * len(values), *values)


def _encode(rows, predictor):
    """the bytes of float32 rows (r, w) under a TIFF predictor"""
    if predictor == 1:
        return rows.astype("<f4").tobytes()
    if predictor == 2:
        u = rows.astype("<f4").view("<u4")
        d = u.copy()
        d[:, 1:] = u[:, 1:] - u[:, :-1]
        return d.tobytes()
    b = rows.astype(">f4").view(np.uint8).reshape(rows.shape[0], rows.shape[1], 4).transpose(0, 2, 1).reshape(rows.shape[0], -1)
    d = b.copy()
    d[:, 1:] = b[:, 1:] - b[:, :-1]
    return d.tobytes()


def write_grid_tiff(path, values, lon0, lat0, dlon, dlat, pixel_is_area=True, compression=8, predictor=3, tile=None,
                    metadata=None, nodata=None, extra_image=False):
    """A little-endian GeoTIFF of one float32 band with the georeferencing GDAL writes for a north-up grid whose node (i, j)
    lies at (lon0 + i dlon, lat0 - j dlat): pixel scale, one tie point and GeoKeys (geographic, PixelIsArea or PixelIsPoint).
    tile: (tw, th) for a tiled file, else one row per strip.  metadata: {name: value} of the GDAL_METADATA tag.
    extra_image: a second IFD (as subgrids or overviews make)."""
    v = np.asarray(values, np.float32)
    h, w = v.shape
    tw, th = tile if tile else (w, 1)
    blocks = []
    for r0 in range(0, h, th):
        for c0 in range(0, w, tw):
            b = np.full((th if tile else min(th, h - r0), tw), 0, np.float32)
            part = v[r0:r0 + th, c0:c0 + tw]
            b[:part.shape[0], :part.shape[1]] = part
            raw = _encode(b, predictor)
            blocks.append(zlib.compress(raw) if compression == 8 else raw)
    half = 0.5 if pixel_is_area else 0.0
    tags = [_tag(256, 4, [w]), _tag(257, 4, [h]), _tag(258, 3, [32]), _tag(259, 3, [compression]), _tag(262, 3, [1]),
            _tag(277, 3, [1]), _tag(284, 3, [1]), _tag(339, 3, [3]),
            _tag(33550, 12, [dlon, dlat, 0.0]), _tag(33922, 12, [0.0, 0.0, 0.0, lon0 - half * dlon, lat0 + half * dlat, 0.0]),
            _tag(34735, 3, [1, 1, 0, 3, 1024, 0, 1, 2, 1025, 0, 1, 1 if pixel_is_area else 2, 2048, 0, 1, 4326])]
    if predictor != 1:
        tags.append(_tag(317, 3, [predictor]))
    if metadata:
        items = "".join('<Item name="%s">%s</Item>' % kv for kv in metadata.items())
        tags.append(_tag(42112, 2, "<GDALMetadata>%s</GDALMetadata>" % items))
    if nodata is not None:
        tags.append(_tag(42113, 2, str(nodata)))
    data = bytearray(b"II*\0\0\0\0\0")
    offsets = []
    for b in blocks:
        offsets.append(len(data))
        data += b
    counts = [len(b) for b in blocks]
    if tile:
        tags += [_tag(322, 3, [tw]), _tag(323, 3, [th]), _tag(324, 4, offsets), _tag(325, 4, counts)]
    else:
        tags += [_tag(273, 4, offsets), _tag(278, 4, [th]), _tag(279, 4, counts)]
    tags.sort()

    def ifd(tags, next_off_at_end):
        nonlocal data
        entries = []
        for tag, typ, count, raw in tags:
            if len(raw) <= 4:
                entries.append(struct.pack("<HHI", tag, typ, count) + raw.ljust(4, b"\0"))
            else:
                if len(data) % 2:
                    data += b"\0"
                entries.append(struct.pack("<HHII", tag, typ, count, len(data)))
                data += raw
        if len(data) % 2:
            data += b"\0"
        at = len(data)
        data += struct.pack("<H", len(entries)) + b"".join(entries) + b"\0\0\0\0"
        return at

    first = ifd(tags, False)
    struct.pack_into("<I", data, 4, first)
    if extra_image:
        second = ifd([_tag(256, 4, [1]), _tag(257, 4, [1]), _tag(258, 3, [32])], False)
        struct.pack_into("<I", data, first + 2 + 12 * len(tags), second)
    with open(path, "wb") as f:
        f.write(bytes(data))
