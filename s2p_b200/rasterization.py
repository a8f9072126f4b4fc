"""Drop-in for ``plyflatten_from_plyfiles_list``, the rasterisation of point clouds into a DSM that ``plys_to_dsm`` runs on
each tile's cloud and its neighbours' (s2p/__init__.py:432-476).

The clouds' vertex records go to the device as they lie in the files (``s2pb_plyflatten``), where each point is placed in
its cell and every cell averages its points in order, bit for bit the reference's float accumulation.  Radius > 0, a sigma
(the Gaussian splat) and PLY files other than binary little-endian with double, float and uchar vertex properties go to the
original ``plyflatten`` package when it is importable; otherwise they raise ``S2pbError`` with ``ERR_UNSUPPORTED``.  The
colour properties (red, green, blue, ir) may also have the integer types s2p writes for a ``clr`` image in its own type
(char, short, ushort, int, uint; e.g. ushort for a 12-bit product); like every property they are read as float64.

``install()`` replaces the name ``plyflatten_from_plyfiles_list`` in the ``s2p`` package, which imports it by name
(s2p/__init__.py:31), and keeps the original as ``s2p._s2pb_original_plyflatten_from_plyfiles_list``.
"""
import re

import numpy as np

from . import _lib
from .engine import get_engine

# PLY property type names -> (_lib.PLY_* code, little-endian numpy type)
_TYPES = {"double": (_lib.PLY_F64, "<f8"), "float64": (_lib.PLY_F64, "<f8"),
          "float": (_lib.PLY_F32, "<f4"), "float32": (_lib.PLY_F32, "<f4"),
          "uchar": (_lib.PLY_U8, "u1"), "uint8": (_lib.PLY_U8, "u1")}
# ... and the integer types of the colour properties only
_COLOUR_TYPES = {"char": (_lib.PLY_I8, "i1"), "int8": (_lib.PLY_I8, "i1"),
                 "short": (_lib.PLY_I16, "<i2"), "int16": (_lib.PLY_I16, "<i2"),
                 "ushort": (_lib.PLY_U16, "<u2"), "uint16": (_lib.PLY_U16, "<u2"),
                 "int": (_lib.PLY_I32, "<i4"), "int32": (_lib.PLY_I32, "<i4"),
                 "uint": (_lib.PLY_U32, "<u4"), "uint32": (_lib.PLY_U32, "<u4")}
_COLOURS = ("red", "green", "blue", "ir")


class UnsupportedPly(ValueError):
    """A PLY file this reader does not take: ASCII or big-endian, another vertex property type, or list properties."""


class PlyCloud:
    """The vertex element of a binary little-endian PLY file.  records: (n, record_bytes) uint8, as in the file;
    names / types: the vertex properties in file order (types as _lib.PLY_* codes); comments: the header's comments."""

    def __init__(self, records, names, types, comments):
        self.records, self.names, self.types, self.comments = records, names, types, comments

    @property
    def dtype(self):
        """packed structured dtype of a record"""
        codes = {c: t for c, t in list(_TYPES.values()) + list(_COLOUR_TYPES.values())}
        return np.dtype({"names": self.names, "formats": [codes[t] for t in self.types]})

    @property
    def columns(self):
        """(byte offset, _lib.PLY_* type) of each property"""
        d = self.dtype
        return [(d.fields[n][1], t) for n, t in zip(self.names, self.types)]

    def column(self, k):
        """property k of every point as float64, as numpy's astype(np.float64) gives it"""
        return self.records.view(self.dtype)[self.names[k]].reshape(-1).astype(np.float64)


def read_ply(path):
    """-> PlyCloud.  Raises UnsupportedPly for the files the GPU path does not read, ValueError for malformed ones."""
    with open(path, "rb") as f:
        if f.readline().rstrip(b"\r\n") != b"ply":
            raise ValueError("%s is not a PLY file" % path)
        fmt, comments, elements = None, [], []
        while True:
            line = f.readline()
            if not line:
                raise ValueError("%s: the header has no end_header" % path)
            words = line.decode("ascii", "replace").split()
            if not words:
                continue
            if words[0] == "end_header":
                break
            if words[0] == "format":
                fmt = words[1] if len(words) > 1 else None
            elif words[0] == "comment":
                comments.append(line.decode("ascii", "replace").rstrip("\r\n")[len("comment "):])
            elif words[0] == "element" and len(words) == 3:
                elements.append((words[1], int(words[2]), []))
            elif words[0] == "property" and elements:
                elements[-1][2].append(words[1:])
            elif words[0] != "obj_info":
                raise ValueError("%s: unexpected header line %r" % (path, line))
        if fmt != "binary_little_endian":
            raise UnsupportedPly("%s: format %s (binary_little_endian only)" % (path, fmt))
        if not elements or elements[0][0] != "vertex":
            raise UnsupportedPly("%s: the vertex element is not the first one" % path)
        _, n, props = elements[0]
        names, types = [], []
        for p in props:
            t = _TYPES.get(p[0]) or (_COLOUR_TYPES.get(p[0]) if len(p) == 2 and p[1] in _COLOURS else None)
            if len(p) != 2 or t is None:
                raise UnsupportedPly("%s: vertex property %s (double, float and uchar, and integer colours, only)" %
                                     (path, " ".join(p)))
            types.append(t[0])
            names.append(p[1])
        cloud = PlyCloud(None, names, types, comments)
        rb = cloud.dtype.itemsize
        records = np.fromfile(f, dtype=np.uint8, count=n * rb)
        if records.size != n * rb:
            raise ValueError("%s: %d vertex records announced, %d bytes found" % (path, n, records.size))
        cloud.records = records.reshape(n, rb)
        return cloud


def roi_of(clouds, resolution):
    """(xoff, yoff, xsize, ysize): the grid of unit `resolution` that holds every point, by the formulas of plys_to_dsm
    (s2p/__init__.py:449-457) in float64 numpy"""
    r = resolution
    x = np.concatenate([c.column(0) for c in clouds])
    y = np.concatenate([c.column(1) for c in clouds])
    xmin, xmax, ymin, ymax = np.min(x), np.max(x), np.min(y), np.max(y)
    xoff = np.floor(xmin / r) * r
    xsize = int(1 + np.floor((xmax - xoff) / r))
    yoff = np.ceil(ymax / r) * r
    ysize = int(1 - np.floor((ymin - yoff) / r))
    return xoff, yoff, xsize, ysize


def crs_of(comments):
    """the `epsg:NNNN` of a `projection: CRS epsg:NNNN` comment (what s2p writes, s2p/__init__.py write_to_ply), or None"""
    for c in comments:
        m = re.match(r"\s*projection:\s*CRS\s+(\S+)", c)
        if m:
            return m.group(1)
    return None


def profile_of(crs, xoff, yoff, resolution):
    """crs, transform, tiled and nodata of the raster: rasterio objects when rasterio is importable, plain values
    (the crs string, the transform's six coefficients a, b, c, d, e, f) otherwise"""
    r = float(resolution)
    coeffs = (r, 0.0, float(xoff), 0.0, -r, float(yoff))
    try:
        import rasterio
    except ImportError:
        return {"crs": crs, "transform": coeffs, "tiled": True, "nodata": float("nan")}
    return {"crs": rasterio.crs.CRS.from_string(crs) if crs else None, "transform": rasterio.Affine(*coeffs),
            "tiled": True, "nodata": float("nan")}


def _original(clouds, resolution, radius, roi, sigma, why):
    try:
        from plyflatten import plyflatten_from_plyfiles_list as original
    except ImportError:
        raise _lib.S2pbError(_lib.ERR_UNSUPPORTED, "%s, and the plyflatten package is not installed" % why) from None
    return original(clouds, resolution, radius=radius, roi=roi, sigma=sigma)


def plyflatten_from_plyfiles_list(clouds, resolution, radius=0, roi=None, sigma=None, engine=None):
    """-> (raster, profile): raster (ysize, xsize, nprops - 2) float32, channel k the mean of vertex property k + 2 (after x
    and y) over the points of each cell, NaN where none fell; profile: crs, transform, tiled and nodata.  roi = (xoff, yoff,
    xsize, ysize), or None for the grid of unit `resolution` that holds every point."""
    if radius != 0 or sigma is not None:
        return _original(clouds, resolution, radius, roi, sigma, "radius %r, sigma %r: the Gaussian splat" % (radius, sigma))
    try:
        plys = [read_ply(c) for c in clouds]
    except UnsupportedPly as e:
        return _original(clouds, resolution, radius, roi, sigma, str(e))
    if not plys:
        raise ValueError("no cloud to rasterise")
    layout = (plys[0].names, plys[0].types)
    if any((p.names, p.types) != layout for p in plys[1:]):
        return _original(clouds, resolution, radius, roi, sigma, "clouds with different vertex properties")
    xoff, yoff, xsize, ysize = roi if roi is not None else roi_of(plys, resolution)
    raster = (engine or get_engine()).plyflatten([p.records for p in plys], plys[0].dtype.itemsize, plys[0].columns,
                                                 xoff, yoff, resolution, xsize, ysize)
    return raster, profile_of(crs_of(plys[0].comments), xoff, yoff, resolution)


def install():
    import s2p
    if not hasattr(s2p, "_s2pb_original_plyflatten_from_plyfiles_list"):
        s2p._s2pb_original_plyflatten_from_plyfiles_list = s2p.plyflatten_from_plyfiles_list
    s2p.plyflatten_from_plyfiles_list = plyflatten_from_plyfiles_list
    return s2p
