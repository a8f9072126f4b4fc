"""Single-band raster I/O for the drop-in boundary.

The reference exchanges tile rasters as files (SURVEY.md section 8b): rectified images are
float32 GeoTIFFs written through rasterio, the matcher binary writes plain float32 TIFFs with
iio and ``plambda`` writes the mask as an 8-bit PNG.  rasterio is used when it is importable
(as in a real s2p installation); otherwise Pillow / OpenCV read and write the same files.
"""
import numpy as np

try:  # pragma: no cover - depends on the installation
    import rasterio
    _HAVE_RASTERIO = True
except Exception:  # ImportError or a broken GDAL
    rasterio = None
    _HAVE_RASTERIO = False


def read_band(path):
    """-> 2-D float32 array (first band), NaN preserved."""
    if _HAVE_RASTERIO:
        with rasterio.open(path, "r") as f:
            return np.ascontiguousarray(f.read(1).astype(np.float32))
    return np.ascontiguousarray(_read_all(path)[0])


def read_band_stored(path):
    """-> 2-D array of the first band in the dtype it is stored in (rasterio's ``read(1)``): a float64 raster keeps its
    bits, where read_band rounds to float32."""
    if _HAVE_RASTERIO:
        with rasterio.open(path, "r") as f:
            return np.ascontiguousarray(f.read(1))
    import cv2
    a = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    if a is not None and a.ndim == 2:
        return np.ascontiguousarray(a)
    from PIL import Image
    with Image.open(path) as im:
        a = np.array(im)
    return np.ascontiguousarray(a if a.ndim == 2 else a[..., 0])


def _read_all(path):
    """-> float32 array (bands, h, w) without rasterio"""
    try:
        from PIL import Image
        with Image.open(path) as im:
            a = np.array(im)
    except Exception:
        import cv2
        a = cv2.imread(path, cv2.IMREAD_UNCHANGED)
        if a is None:
            raise
        if a.ndim == 3:
            a = a[..., ::-1]          # OpenCV stores BGR
    a = a[None] if a.ndim == 2 else np.moveaxis(a, 2, 0)
    return np.ascontiguousarray(a.astype(np.float32))


def read_stored(path, window=None):
    """-> (bands, h, w) array in the dtype the raster stores (rasterio's ``read()``); window = (x, y, w, h) or None"""
    if _HAVE_RASTERIO:
        with rasterio.open(path, "r") as f:
            if window is None:
                return np.ascontiguousarray(f.read())
            x, y, w, h = window
            return np.ascontiguousarray(f.read(window=((y, y + h), (x, x + w))))
    import cv2
    a = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    if a is None:
        from PIL import Image
        with Image.open(path) as im:
            a = np.array(im)
    elif a.ndim == 3:
        a = a[..., ::-1]              # OpenCV stores BGR
    a = a[None] if a.ndim == 2 else np.moveaxis(a, 2, 0)
    if window is not None:
        x, y, w, h = window
        a = a[:, y:y + h, x:x + w]
    return np.ascontiguousarray(a)


def band_count(path):
    if _HAVE_RASTERIO:
        with rasterio.open(path, "r") as f:
            return f.count
    return _read_all(path).shape[0]


def read_window(path, x, y, w, h, band=1):
    """-> float32 array of the w x h window at (x, y) of band `band` (1-based, as in GDAL)."""
    if _HAVE_RASTERIO:
        from rasterio.windows import Window
        with rasterio.open(path, "r") as f:
            return np.ascontiguousarray(f.read(band, window=Window(x, y, w, h)).astype(np.float32))
    if band == 1:
        return np.ascontiguousarray(read_band(path)[y:y + h, x:x + w])
    return np.ascontiguousarray(_read_all(path)[band - 1, y:y + h, x:x + w])


def image_size(path):
    """-> (width, height)"""
    if _HAVE_RASTERIO:
        with rasterio.open(path, "r") as f:
            return f.width, f.height
    try:
        from PIL import Image
        with Image.open(path) as im:
            return im.size
    except Exception:            # e.g. a multi-band float TIFF, which Pillow does not decode
        a = _read_all(path)
        return a.shape[2], a.shape[1]


def write_float_tiff(path, a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    if _HAVE_RASTERIO:
        h, w = a.shape
        with rasterio.open(path, "w", driver="GTiff", height=h, width=w, count=1, dtype="float32") as f:
            f.write(a, 1)
        return
    from PIL import Image
    Image.fromarray(a, mode="F").save(path, format="TIFF")


def write_float64_tiff(path, a):
    """Single-band float64 raster, as common.rasterio_write writes the float64 height map of a pair (s2p/common.py:125-156:
    rasterio with the profile driver, count, width, height and dtype only); without rasterio a plain float64 TIFF."""
    a = np.ascontiguousarray(a, dtype=np.float64)
    if _HAVE_RASTERIO:
        h, w = a.shape
        with rasterio.Env():
            with rasterio.open(path, "w", driver="GTiff", count=1, width=w, height=h, dtype=a.dtype) as f:
                f.write(a[None])
                f.update_tags()
        return
    import cv2
    if not cv2.imwrite(path, a):
        raise IOError("cv2.imwrite failed for %s" % path)


def write_float_tiff_like(path, a, template):
    """Single-band float32 raster at `path` with the metadata (CRS, transform, ...) of the raster `template`, which may be
    `path` itself; without rasterio a plain float32 TIFF."""
    a = np.ascontiguousarray(a, dtype=np.float32)
    if not _HAVE_RASTERIO:
        return write_float_tiff(path, a)
    with rasterio.open(template, "r") as f:
        profile = f.profile
    profile.update(driver="GTiff", dtype="float32", count=1, height=a.shape[0], width=a.shape[1])
    with rasterio.open(path, "w", **profile) as f:
        f.write(a, 1)


def write_float_tiff_bands(path, bands):
    """float32 TIFF with one band per array of `bands` (what the reference's `homography` writes for a colour image,
    3rdparty/homography/main.cpp: one RasterIO per band)."""
    bands = [np.ascontiguousarray(b, dtype=np.float32) for b in bands]
    if len(bands) == 1:
        return write_float_tiff(path, bands[0])
    if _HAVE_RASTERIO:
        h, w = bands[0].shape
        with rasterio.open(path, "w", driver="GTiff", height=h, width=w, count=len(bands), dtype="float32") as f:
            for k, b in enumerate(bands):
                f.write(b, k + 1)
        return
    import cv2
    if len(bands) not in (3, 4):
        raise ValueError("writing a %d-band float TIFF needs rasterio" % len(bands))
    a = np.stack(bands[:3][::-1] + bands[3:], axis=2)      # OpenCV stores BGR(A)
    if not cv2.imwrite(path, a):
        raise IOError("cv2.imwrite failed for %s" % path)


def write_mask_png(path, m):
    """uint8 0/1 mask, as plambda writes it (s2p/block_matching.py:32)."""
    m = np.ascontiguousarray(m, dtype=np.uint8)
    if _HAVE_RASTERIO:
        h, w = m.shape
        with rasterio.open(path, "w", driver="PNG", height=h, width=w, count=1, dtype="uint8") as f:
            f.write(m, 1)
        return
    from PIL import Image
    Image.fromarray(m, mode="L").save(path, format="PNG")


def overwrite_band(path, a):
    """Replace the content of the (single) band of an existing raster, keeping its metadata
    (rasterio 'r+' as in s2p/fusion.py:65-66; without rasterio the file is rewritten as a plain TIFF)."""
    a = np.ascontiguousarray(a, dtype=np.float32)
    if _HAVE_RASTERIO:
        with rasterio.open(path, "r+") as f:
            f.write(np.asarray([a]).astype("float32"))
        return
    write_float_tiff(path, a)
