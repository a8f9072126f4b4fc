"""The output coordinate systems of ``s2p.triangulation.disp_to_xyz`` that the GPU serves.

s2p triangulates to WGS84 (lon, lat, alt), EPSG:4979, and projects the cloud to ``out_crs`` with pyproj
(s2p/triangulation.py:147-160); when the configuration leaves ``out_crs`` unset it becomes the UTM zone of the ROI, and with
``out_geoid`` that zone with heights above the EGM96 geoid, ``epsg:326zz+5773`` (s2p/initialization.py:133-141).  The device
projects to the UTM zones of WGS84, EPSG 32601-32660 (north) and 32701-32760 (south), with PROJ's exact transverse Mercator
(``csrc/projection_kernels.cuh``).  No output CRS, 4979 and 4326 leave (lon, lat, alt) as they are, as pyproj does.

The device also projects to the ETRS89 UTM zones 28N-38N (EPSG 25828-25838) and to RGF93 v1 / Lambert-93 (2154) and its nine
conic zones CC42-CC50 (3942-3950), the national grids s2p's users in Europe and France set most often (``PROJECTED``, the one
table of their map parameters, with ``S2PB_ZONE_PROJ``).  All of them are on GRS80, and their datums reach WGS84 through the
null transformations "ETRS89 to WGS 84 (1)" and "RGF93 v1 to WGS 84 (1)" of the EPSG dataset, the operation PROJ applies
where no grid applies: the cloud is the pure map of the triangulated (lon, lat) and the altitude passes through, as for UTM.
They are served where PROJ itself agrees (``proj_agrees``): pyproj is importable and its transformation from EPSG:4979 of
reference points over the area of use lands within 1 mm of the same map (``map_lonlat``), the altitude unchanged.  A PROJ
whose database or grids apply another operation, or no pyproj (which the reference's own path needs too), keeps the
reference's path.

The compound targets 326zz+5773, 327zz+5773 and 4326+5773 (and those grids +5773) differ from those only in z: PROJ
subtracts the EGM96 undulation N(lon, lat), interpolated bilinearly in its grid ``us_nga_egm96_15.tif``, from the ellipsoidal
height.  The device does the
same (``S2PB_ZONE_EGM96``) with the grid file PROJ would open, found by ``locate_egm96`` and read by ``read_geoid_grid``
without GDAL; where there is no such file, or it is not a global north-up float32 grid interpolated bilinearly, the target is
not served.  Any target not served -- those, another geoid, datum or projection -- goes through the reference's pyproj code
when it is importable, and raises ``S2pbError`` with ``ERR_UNSUPPORTED`` otherwise.

A target is read without pyproj: an ``"epsg:NNNN"`` or ``"epsg:NNNN+VVVV"`` string (any case), an int, or any object with
``.to_epsg()`` (a ``pyproj.CRS``), a compound one by the codes of its ``sub_crs_list``.
"""
import collections
import os
import re
import struct
import xml.etree.ElementTree as ET
import zlib

import numpy as np

from . import _lib
from .engine import get_engine

GEOGRAPHIC = (4979, 4326)


def epsg_of(crs):
    """the EPSG code of crs, or None when it is not one the code can be read from"""
    if isinstance(crs, (int, np.integer)) and not isinstance(crs, bool):
        return int(crs)
    if isinstance(crs, str):
        m = re.fullmatch(r"\s*epsg:(\d+)\s*", crs, re.IGNORECASE)
        return int(m.group(1)) if m else None
    to_epsg = getattr(crs, "to_epsg", None)
    if callable(to_epsg):
        code = to_epsg()
        return None if code is None else int(code)
    return None


def _codes(crs):
    """(horizontal EPSG code, vertical EPSG code or None) of a truthy crs, or None when they cannot be read"""
    if isinstance(crs, str):
        m = re.fullmatch(r"\s*epsg:(\d+)(?:\+(\d+))?\s*", crs, re.IGNORECASE)
        return (int(m.group(1)), int(m.group(2)) if m.group(2) else None) if m else None
    subs = getattr(crs, "sub_crs_list", None)
    if subs:                                    # a compound pyproj.CRS: to_epsg() gives None
        codes = [epsg_of(c) for c in subs]
        return tuple(codes) if len(codes) == 2 and None not in codes else None
    code = epsg_of(crs)
    return None if code is None else (code, None)


def _zone_of(code):
    """(zone, south) of EPSG 326zz / 327zz, None for another code"""
    if 32601 <= code <= 32660 or 32701 <= code <= 32760:
        return code % 100, code > 32700
    return None


def utm_target(crs, engine=None):
    """-> (zone, south) for the targets the device serves: (0, False) when the cloud stays in (lon, lat, alt) -- no
    output CRS (s2p's `if out_crs and ...`), EPSG 4979 or 4326 -- and (zone, south) for EPSG 326zz / 327zz; the same with
    _lib.ZONE_EGM96 OR'ed into the zone for 4326+5773, 326zz+5773 and 327zz+5773 when ``egm96_grid()`` finds the grid, which
    is then registered on ``engine`` (when given) for the call that takes the zone; None for any other target"""
    if not crs:
        return 0, False
    codes = _codes(crs)
    if codes is None:
        return None
    code, vertical = codes
    target = (0, False) if code in GEOGRAPHIC else _zone_of(code)
    if vertical is None or target is None:
        return target
    if vertical != EGM96_HEIGHT or code != 4326 and target[0] == 0:
        return None
    grid = egm96_grid()
    if grid is None:
        return None
    if engine is not None:
        engine.set_geoid(grid)
    return target[0] | _lib.ZONE_EGM96, target[1]


# ------------------------------------------------------------------ the other projected targets (S2PB_ZONE_PROJ)

Projection = collections.namedtuple("Projection", "method a rf lon0 lat0 lat1 lat2 k0 x0 y0")
Projection.__doc__ = """the fields of s2pb_projection: method _lib.PROJ_TM or _lib.PROJ_LCC, the ellipsoid (semi-major axis a in
metres, inverse flattening rf), the origin (lon0, lat0), the standard parallels lat1, lat2 (LCC), the scale k0 (TM), degrees,
and the false easting and northing x0, y0 in metres"""

GRS80 = (6378137.0, 298.257222101)          # EPSG:7019 GRS 1980, the ellipsoid of ETRS89 (EPSG:6258) and RGF93 v1 (EPSG:6171)


def _etrs89_utm(zone):
    """EPSG 25800 + zone, ETRS89 / UTM zone zoneN: Transverse Mercator (EPSG method 9807), latitude of natural origin 0,
    longitude 6 zone - 183, scale 0.9996, false easting 500 000 m, false northing 0"""
    return Projection(_lib.PROJ_TM, *GRS80, 6.0 * zone - 183.0, 0.0, 0.0, 0.0, 0.9996, 500000.0, 0.0)


def _rgf93_cc(lat):
    """EPSG 3900 + lat, RGF93 v1 / CC<lat>: Lambert Conic Conformal (2SP) (EPSG method 9802), false origin (3 E, lat N) at
    (1 700 000, 1 200 000 + (lat - 42) 1 000 000) m, standard parallels lat - 0.75 and lat + 0.75"""
    return Projection(_lib.PROJ_LCC, *GRS80, 3.0, float(lat), lat - 0.75, lat + 0.75, 0.0, 1700000.0,
                      1200000.0 + (lat - 42) * 1000000.0)


# EPSG code -> the map the device runs for it (the single rule of which projected CRSs other than WGS84 UTM are served)
PROJECTED = {
    **{25800 + zone: _etrs89_utm(zone) for zone in range(28, 39)},
    # EPSG:2154 RGF93 v1 / Lambert-93: LCC 2SP, false origin (3 E, 46.5 N) at (700 000, 6 600 000) m, parallels 49 and 44
    2154: Projection(_lib.PROJ_LCC, *GRS80, 3.0, 46.5, 49.0, 44.0, 0.0, 700000.0, 6600000.0),
    **{3900 + lat: _rgf93_cc(lat) for lat in range(42, 51)},
}


# ------------------------------------------------------------------ PROJ's consent

def map_lonlat(proj, lon, lat):
    """(x, y) in metres of (lon, lat) in degrees by the map proj in float64 numpy: the Lambert conic conformal of lcc_forward,
    or the transverse Mercator of utm_forward (Krueger's series to order n^6, the coefficients of projection.cu's tm_params).
    For the agreement check below; the device's maps are pinned to 50-digit truths by the tests."""
    lon, lat = np.asarray(lon, np.float64), np.asarray(lat, np.float64)
    f = 1.0 / proj.rf
    lam = np.radians(lon - proj.lon0)
    lam = lam - 2 * np.pi * np.floor((lam + np.pi) / (2 * np.pi))
    phi = np.radians(lat)
    if proj.method == _lib.PROJ_LCC:
        e = np.sqrt(f * (2.0 - f))
        m = lambda p: np.cos(p) / np.sqrt(1.0 - (e * np.sin(p)) ** 2)                          # noqa: E731
        psi = lambda p: np.arcsinh(np.tan(p)) - e * np.arctanh(e * np.sin(p))                  # noqa: E731
        p1, p2, p0 = np.radians(proj.lat1), np.radians(proj.lat2), np.radians(proj.lat0)
        n = np.sin(p1) if proj.lat1 == proj.lat2 else (np.log(m(p1)) - np.log(m(p2))) / (psi(p2) - psi(p1))
        aF = proj.a * m(p1) * np.exp(n * psi(p1)) / n
        rho, theta = aF * np.exp(-n * psi(phi)), n * lam
        return proj.x0 + rho * np.sin(theta), proj.y0 + aF * np.exp(-n * psi(p0)) - rho * np.cos(theta)
    n = f / (2.0 - f)
    cbg = [n * (-2 + n * (2 / 3 + n * (4 / 3 + n * (-82 / 45 + n * (32 / 45 + n * 4642 / 4725))))),
           n ** 2 * (5 / 3 + n * (-16 / 15 + n * (-13 / 9 + n * (904 / 315 + n * -1522 / 945)))),
           n ** 3 * (-26 / 15 + n * (34 / 21 + n * (8 / 5 + n * -12686 / 2835))),
           n ** 4 * (1237 / 630 + n * (-12 / 5 + n * -24832 / 14175)), n ** 5 * (-734 / 315 + n * 109598 / 31185),
           n ** 6 * 444337 / 155925]
    gtu = [n * (1 / 2 + n * (-2 / 3 + n * (5 / 16 + n * (41 / 180 + n * (-127 / 288 + n * 7891 / 37800))))),
           n ** 2 * (13 / 48 + n * (-3 / 5 + n * (557 / 1440 + n * (281 / 630 + n * -1983433 / 1935360)))),
           n ** 3 * (61 / 240 + n * (-103 / 140 + n * (15061 / 26880 + n * 167603 / 181440))),
           n ** 4 * (49561 / 161280 + n * (-179 / 168 + n * 6601661 / 7257600)), n ** 5 * (34729 / 80640 + n * -3418889 / 1995840),
           n ** 6 * 212378941 / 319334400]
    chi = phi + sum(c * np.sin(2 * (k + 1) * phi) for k, c in enumerate(cbg))
    zeta = np.arctan2(np.sin(chi), np.cos(chi) * np.cos(lam)) + 1j * np.arcsinh(
        np.sin(lam) * np.cos(chi) / np.hypot(np.sin(chi), np.cos(chi) * np.cos(lam)))
    zeta = zeta + sum(c * np.sin(2 * (k + 1) * zeta) for k, c in enumerate(gtu))
    qa = proj.a * proj.k0 / (1 + n) * (1 + n ** 2 / 4 + n ** 4 / 64 + n ** 6 / 256)
    return proj.x0 + qa * zeta.imag, proj.y0 + qa * zeta.real


AGREE_M = 1e-3      # PROJ against map_lonlat: far above rounding, far below any datum shift ETRS89 / RGF93 v1 could have


def _reference_points(proj):
    """3 x 3 (lon, lat) over the CRS's area of use, degrees"""
    if proj.method == _lib.PROJ_LCC:
        lons, lats = (-4.0, 3.0, 9.0), (proj.lat0 - 2.0, proj.lat0, proj.lat0 + 2.0)
    else:
        lons, lats = (proj.lon0 - 3.0, proj.lon0, proj.lon0 + 3.0), (36.0, 50.0, 70.0)
    lon, lat = np.meshgrid(lons, lats)
    return lon.ravel(), lat.ravel()


_consent = {}


def proj_agrees(code):
    """Whether PROJ, through pyproj, takes EPSG:4979 to EPSG ``code`` of PROJECTED as the device does: its transformation of
    reference points over the area of use within AGREE_M of map_lonlat in x and y, the altitude unchanged.  The device
    serves these CRSs only then, so that a PROJ whose database or grids would apply another operation (a datum shift) keeps the
    reference's path; without pyproj the reference's path cannot run either, and the steps fall through as before.  Asked
    once per code and pyproj module."""
    try:
        import pyproj
    except ImportError:
        return False
    key = (code, pyproj)
    if key not in _consent:
        proj = PROJECTED[code]
        lon, lat = _reference_points(proj)
        h = np.linspace(-100.0, 4000.0, lon.size)
        try:
            t = pyproj.Transformer.from_crs("epsg:4979", "epsg:%d" % code, always_xy=True)
            x, y, z = (np.asarray(v, np.float64) for v in t.transform(lon, lat, h))
        except Exception:       # pyproj's errors (CRSError, ProjError) and a PROJ without the code
            _consent[key] = False
        else:
            wx, wy = map_lonlat(proj, lon, lat)
            _consent[key] = bool(np.all(np.abs(x - wx) <= AGREE_M) and np.all(np.abs(y - wy) <= AGREE_M) and
                                 np.all(np.abs(z - h) <= 1e-6))
    return _consent[key]


def output_target(crs, engine=None):
    """The zone argument of the device's cloud calls for crs -> (zone, south): utm_target's for WGS84 and its UTM zones;
    (_lib.ZONE_PROJ, False) for a code of PROJECTED that proj_agrees with, whose map is then registered on ``engine`` (when
    given); either with _lib.ZONE_EGM96 OR'ed in for a +5773 target when ``egm96_grid()`` finds the grid, registered as
    utm_target registers it; None for any other target"""
    target = utm_target(crs, engine)
    if target is not None:
        return target
    codes = _codes(crs)
    if codes is None or codes[0] not in PROJECTED or codes[1] not in (None, EGM96_HEIGHT) or not proj_agrees(codes[0]):
        return None
    zone = _lib.ZONE_PROJ
    if codes[1] == EGM96_HEIGHT:
        grid = egm96_grid()
        if grid is None:
            return None
        if engine is not None:
            engine.set_geoid(grid)
        zone |= _lib.ZONE_EGM96
    if engine is not None:
        engine.set_projection(PROJECTED[codes[0]])
    return zone, False


def unserved_reason(crs):
    """why output_target(crs) is None, for the fall-through messages"""
    codes = _codes(crs)
    if codes and codes[0] in PROJECTED and codes[1] in (None, EGM96_HEIGHT) and not proj_agrees(codes[0]):
        return ("output CRS %r is not a UTM zone of WGS84, and the device serves it as an ETRS89 / RGF93 v1 grid only where pyproj "
                "is importable and PROJ's own transformation from EPSG:4979 agrees with the device's map" % (crs,))
    if codes and codes[1] == EGM96_HEIGHT and (codes[0] == 4326 or _zone_of(codes[0]) or codes[0] in PROJECTED):
        return "output CRS %r needs the EGM96 grid %s, which was not found or is not one the device reads" % (crs, EGM96_FILE)
    return ("output CRS %r is not a UTM zone of WGS84, nor an ETRS89 UTM zone (EPSG 25828-25838) or RGF93 v1 Lambert grid "
            "(2154, 3942-3950)" % (crs,))


# ------------------------------------------------------------------ the EGM96 grid

EGM96_HEIGHT = 5773                 # EGM96 height, the vertical CRS of s2p's out_geoid targets
EGM96_FILE = "us_nga_egm96_15.tif"  # the grid PROJ uses for it (PROJ-data)

GeoidGrid = collections.namedtuple("GeoidGrid", "values lon0 lat0 dlon dlat")
GeoidGrid.__doc__ = """values: (h, w) float32 undulations in metres, row 0 northernmost; node (i, j) at (lon0 + i dlon, lat0 - j dlat)
degrees (s2pb_set_geoid)"""


class GeoidGridError(ValueError):
    """a grid file the device does not serve, and why"""


def proj_data_dirs():
    """the directories searched for a grid, in order: PROJ_DATA (or, when it is unset, PROJ_LIB), each a path list, then
    pyproj's data directory and its user data directory when pyproj is importable"""
    env = os.environ.get("PROJ_DATA") or os.environ.get("PROJ_LIB") or ""
    dirs = [d for d in env.split(os.pathsep) if d]
    try:
        from pyproj import datadir
    except ImportError:
        return dirs
    for get in (datadir.get_data_dir, datadir.get_user_data_dir):
        try:
            dirs.append(get())
        except Exception:       # pyproj raises DataDirError when it has no data directory
            pass
    return dirs


def locate_egm96():
    """the path of the first us_nga_egm96_15.tif of proj_data_dirs(), or None (a grid held only in PROJ's network cache
    is not a file there)"""
    for d in proj_data_dirs():
        path = os.path.join(d, EGM96_FILE)
        if os.path.isfile(path):
            return path
    return None


_grids = {}


def egm96_grid():
    """the GeoidGrid of locate_egm96()'s file, read once per file version, or None when there is no file or
    read_geoid_grid refuses it"""
    path = locate_egm96()
    if path is None:
        return None
    st = os.stat(path)
    key = (path, st.st_mtime_ns, st.st_size)
    if key not in _grids:
        try:
            _grids[key] = read_geoid_grid(path)
        except (GeoidGridError, OSError, zlib.error):
            _grids[key] = None
    return _grids[key]


_TIFF_TYPES = {1: "B", 2: "s", 3: "H", 4: "I", 5: "II", 6: "b", 7: "B", 8: "h", 9: "i", 10: "ii", 11: "f", 12: "d"}


def _tiff_tags(data):
    """-> (byte order, {tag: values}) of the first IFD of a classic TIFF; GeoidGridError for another layout"""
    if data[:4] not in (b"II*\0", b"MM\0*"):
        raise GeoidGridError("not a classic TIFF")
    bo = "<" if data[:2] == b"II" else ">"
    (off,) = struct.unpack_from(bo + "I", data, 4)
    (n,) = struct.unpack_from(bo + "H", data, off)
    tags = {}
    for k in range(n):
        tag, typ, count, value = struct.unpack_from(bo + "HHI4s", data, off + 2 + 12 * k)
        if typ not in _TIFF_TYPES:
            continue
        fmt = _TIFF_TYPES[typ]
        size = struct.calcsize(bo + fmt) * count
        raw = value if size <= 4 else data[struct.unpack(bo + "I", value)[0]:][:size]
        if typ == 2:
            tags[tag] = raw[:count].split(b"\0")[0].decode("latin-1")
        else:
            v = struct.unpack(bo + fmt * count, raw[:size])
            tags[tag] = [v[i] / v[i + 1] for i in range(0, len(v), 2)] if typ in (5, 10) else list(v)
    (nxt,) = struct.unpack_from(bo + "I", data, off + 2 + 12 * n)
    if nxt:
        raise GeoidGridError("more than one image (subgrids or overviews)")
    return bo, tags


def _undo_predictor(block, predictor, bo, width):
    """the float32 samples of one decompressed strip or tile whose rows hold `width` samples"""
    if predictor == 1:
        return np.frombuffer(block, bo + "f4")
    if predictor == 2:                  # libtiff's horizontal differencing of 32-bit words
        return np.cumsum(np.frombuffer(block, bo + "u4").reshape(-1, width), axis=1, dtype=np.uint32).view(np.float32).ravel()
    if predictor == 3:                  # floating-point predictor: byte planes, most significant first, differenced per row
        b = np.cumsum(np.frombuffer(block, np.uint8).reshape(-1, width * 4), axis=1, dtype=np.uint8)
        return np.ascontiguousarray(b.reshape(-1, 4, width).transpose(0, 2, 1)).view(">f4").ravel()
    raise GeoidGridError("predictor %d" % predictor)


def _tiff_samples(data, bo, tags):
    """-> (h, w) float32 of a single-band float32 TIFF, strips or tiles, uncompressed or deflate"""
    w, h = tags[256][0], tags[257][0]
    if tags.get(277, [1])[0] != 1 or tags.get(258, [0])[0] != 32 or tags.get(339, [1])[0] != 3:
        raise GeoidGridError("not a single-band float32 raster")
    compression, predictor = tags.get(259, [1])[0], tags.get(317, [1])[0]
    if compression not in (1, 8, 32946):
        raise GeoidGridError("compression %d" % compression)
    tiled = 322 in tags
    bw, bh = (tags[322][0], tags[323][0]) if tiled else (w, tags.get(278, [h])[0])
    offsets, counts = (tags[324], tags[325]) if tiled else (tags[273], tags[279])
    across = -(-w // bw)
    out = np.empty((-(-h // bh) * bh, across * bw), np.float32)
    for k, (o, c) in enumerate(zip(offsets, counts)):
        block = data[o:o + c]
        if compression != 1:
            block = zlib.decompress(block)
        rows = min(bh, h - (k // across) * bh) if not tiled else bh
        v = _undo_predictor(block[:rows * bw * 4], predictor, bo, bw).reshape(rows, bw)
        r0, c0 = (k // across) * bh, (k % across) * bw
        out[r0:r0 + rows, c0:c0 + bw] = v
    return out[:h, :w]


def _gdal_items(xml):
    """{(name, role): text} of a GDAL_METADATA tag"""
    if not xml:
        return {}
    return {(it.get("name"), it.get("role")): (it.text or "").strip() for it in ET.fromstring(xml).iter("Item")}


def read_geoid_grid(path):
    """The GeoidGrid of a PROJ vertical-offset grid file, a GeoTIFF, read without GDAL.  GeoidGridError unless it is one
    single-band float32 image (classic TIFF; strips or tiles; uncompressed or deflate, any predictor), north-up (pixel scale
    and one tie point), global (360 degrees of longitude, 90 to -90), with finite values other than its nodata value, no
    scale or offset, and PROJ's bilinear interpolation (GDAL metadata item interpolation_method absent or 'bilinear')."""
    with open(path, "rb") as f:
        data = f.read()
    bo, tags = _tiff_tags(data)
    items = _gdal_items(tags.get(42112))
    method = items.get(("interpolation_method", None), "bilinear")
    if method.lower() != "bilinear":
        raise GeoidGridError("interpolation_method %s" % method)
    if float(items.get(("SCALE", "scale"), 1)) != 1 or float(items.get(("OFFSET", "offset"), 0)) != 0:
        raise GeoidGridError("a scale or offset")
    if 34264 in tags or 33550 not in tags or len(tags.get(33922, ())) != 6:
        raise GeoidGridError("not a north-up grid with one tie point")
    keys = tags.get(34735, [])
    geokeys = {keys[i]: keys[i + 3] for i in range(4, len(keys) - 3, 4) if keys[i + 1] == 0}
    if geokeys.get(1024, 2) != 2:
        raise GeoidGridError("not a geographic grid")
    sx, sy = tags[33550][:2]
    I, J, _, X, Y, _ = tags[33922]
    if not (sx > 0 and sy > 0):
        raise GeoidGridError("not north-up")
    half = 0.5 if geokeys.get(1025, 1) == 1 else 0.0          # PixelIsArea: the nodes are the pixels' centres
    values = _tiff_samples(data, bo, tags)
    h, w = values.shape
    grid = GeoidGrid(np.ascontiguousarray(values), X + (half - I) * sx, Y - (half - J) * sy, float(sx), float(sy))
    eps = 1e-9
    if w * grid.dlon < 360 - eps or grid.lat0 < 90 - eps or grid.lat0 - (h - 1) * grid.dlat > -90 + eps:
        raise GeoidGridError("not a global grid")
    nodata = tags.get(42113)
    if not np.isfinite(values).all() or (nodata and (values == np.float32(float(nodata))).any()):
        raise GeoidGridError("nodata nodes")
    return grid


def lonlat_to_utm(lonlatalt, zone, south=False, engine=None):
    """(..., 3) float64 (lon, lat in degrees, alt) -> (..., 3) float64 (easting, northing, alt) in UTM zone `zone` of WGS84"""
    return (engine or get_engine()).lonlat_to_utm(lonlatalt, zone, south)


def pyproj_original(lonlatalt, out_crs):
    """The reference's change of coordinates (s2p/triangulation.py:147-160) for the targets output_target does not serve:
    s2p.geographiclib's pyproj wrappers when they are importable, S2pbError(ERR_UNSUPPORTED) otherwise."""
    try:
        from s2p import geographiclib
        in_crs = geographiclib.pyproj_crs("epsg:4979")
    except ImportError:
        raise _lib.S2pbError(_lib.ERR_UNSUPPORTED, "output CRS %r: only WGS84 (EPSG 4979, 4326), its UTM zones, the ETRS89 UTM zones "
                             "and the RGF93 v1 Lambert grids, with EGM96 heights when %s is found, are projected on the device, "
                             "and s2p.geographiclib (pyproj) is not importable" % (out_crs, EGM96_FILE)) from None
    if not (out_crs and out_crs != in_crs):
        return lonlatalt
    h, w = lonlatalt.shape[:2]
    lla = lonlatalt.reshape(-1, 3)
    x, y, z = geographiclib.pyproj_transform(lla[:, 0], lla[:, 1], in_crs, out_crs, lla[:, 2])
    return np.column_stack((x, y, z)).reshape(h, w, 3).astype(np.float64)
