"""ctypes binding of ``libs2pb200.so`` (C ABI in ``include/s2pb200.h``).

Loaded the way the reference loads its own native helpers (``ctypes.CDLL`` on a
library shipped next to the package: s2p/triangulation.py:18-20, s2p/sift.py:25-26).
There is no Python/numpy fallback: if the library is missing or no CUDA device is
visible, the calls raise.
"""
import ctypes
import os
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_longlong, c_uint8, c_uint64, c_void_p

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("S2PB200_LIB") or os.path.join(HERE, "libs2pb200.so")   # the override serves A/B kernel experiments

OK, ERR_CUDA, ERR_ARG, ERR_TIMEOUT, ERR_NOMEM, ERR_UNSUPPORTED = 0, -1, -2, -3, -4, -5
T_NAMES = ("census", "cost", "aggregate", "wta", "post", "total")


class MgmParams(ctypes.Structure):
    """Mirror of ``s2pb_mgm_params``."""
    _fields_ = [
        ("ndir", c_int32), ("tsgm", c_int32), ("census_win", c_int32), ("P1", c_float), ("P2", c_float),
        ("median", c_int32), ("lr_mode", c_int32), ("lr_tau", c_float), ("mindiff", c_float),
        ("remove_small_cc", c_int32), ("subpix", c_int32), ("scales", c_int32), ("refine", c_int32),
        ("fix_overcount", c_int32), ("timeout_ms", c_int32), ("cost", c_int32),
    ]


class SgbmParams(ctypes.Structure):
    """Mirror of ``s2pb_sgbm_params``: the `sgbm` binary's argv after dmin dmax."""
    _fields_ = [("win", c_int32), ("P1", c_int32), ("P2", c_int32), ("lr_diff", c_int32)]


class PairTile(ctypes.Structure):
    """Mirror of ``s2pb_pair_tile``: the inputs of s2pb_pair_tile_to_ply and s2pb_pair_tile_to_height_map."""
    _fields_ = [
        ("src1", POINTER(c_float)), ("src2", POINTER(c_float)), ("sw1", c_int32), ("sh1", c_int32), ("sw2", c_int32),
        ("sh2", c_int32), ("H1", c_double * 9), ("H2", c_double * 9), ("w", c_int32), ("h", c_int32), ("dmin", c_int32),
        ("dmax", c_int32), ("matcher", c_int32), ("mgm", MgmParams), ("sgbm", SgbmParams), ("wl", POINTER(c_float)),
        ("wr", POINTER(c_float)), ("erode_radius", c_float), ("msk_orig", POINTER(c_float)), ("mw", c_int32), ("mh", c_int32),
        ("bbox", c_float * 4), ("rpc1", c_void_p), ("rpc2", c_void_p), ("ha", c_double * 9), ("hb", c_double * 9),
        ("zone", c_int32), ("south", c_int32), ("r", c_float), ("p", c_int32), ("n", c_int32), ("pct", c_double),
        ("clr", POINTER(c_float)), ("cw", c_int32), ("ch", c_int32), ("clr_bands", c_int32), ("hc", c_double * 9),
        ("with_conf", c_int32),
    ]


MATCHER_MGM, MATCHER_SGBM = 0, 1     # S2PB_MATCHER_*
ZONE_EGM96 = 0x100                   # S2PB_ZONE_EGM96
ZONE_PROJ = 0x200                    # S2PB_ZONE_PROJ
PROJ_TM, PROJ_LCC = 1, 2             # S2PB_PROJ_*


class Projection(ctypes.Structure):
    """Mirror of ``s2pb_projection``: a map projection for S2PB_ZONE_PROJ (angles in degrees, lengths in metres)."""
    _fields_ = [("method", c_int32), ("a", c_double), ("rf", c_double), ("lon0", c_double), ("lat0", c_double), ("lat1", c_double),
                ("lat2", c_double), ("k0", c_double), ("x0", c_double), ("y0", c_double)]
MAX_FUSION = 16                      # S2PB_MAX_FUSION


class HeightsTile(ctypes.Structure):
    """Mirror of ``s2pb_heights_tile``: the inputs of s2pb_heights_tile_to_ply."""
    _fields_ = [
        ("n_maps", c_int32), ("w", c_int32), ("h", c_int32), ("map_type", c_int32), ("maps", c_void_p * MAX_FUSION),
        ("offsets", c_double * MAX_FUSION), ("cargarse_basura", c_int32), ("op", c_int32), ("threshold", c_double),
        ("rpc", c_void_p), ("off_x", c_double), ("off_y", c_double), ("zone", c_int32), ("south", c_int32), ("r", c_float),
        ("p", c_int32), ("n", c_int32), ("colors", c_void_p), ("nbands", c_int32), ("color_type", c_int32), ("stretch", c_int32),
        ("pct", c_double),
    ]


class PlyColumn(ctypes.Structure):
    """Mirror of ``s2pb_ply_column``: byte offset of a vertex property in a PLY record and its PLY_* type."""
    _fields_ = [("offset", c_int32), ("type", c_int32)]


PLY_F64, PLY_F32, PLY_U8 = 0, 1, 2     # S2PB_PLY_*
PLY_I8, PLY_I16, PLY_U16, PLY_I32, PLY_U32 = 16, 17, 18, 19, 20

COSTS = ("census", "ad", "sd", "ncc", "btad", "btsd")   # S2PB_COST_* = index; the reference's `-t` names


class S2pbError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("s2pb200 error %d: %s" % (code, msg))
        self.code = code


_lib = None
_f = POINTER(c_float)

_SIGNATURES = {
    "s2pb_version": (c_int, []),
    "s2pb_last_error": (c_char_p, []),
    "s2pb_device_count": (c_int, []),
    "s2pb_create": (c_void_p, [c_int]),
    "s2pb_destroy": (None, [c_void_p]),
    "s2pb_default_params": (c_int, [c_char_p, POINTER(MgmParams)]),
    "s2pb_mgm": (c_int, [c_void_p, _f, _f, c_int, c_int, c_int, c_int, POINTER(MgmParams), _f, _f, POINTER(c_uint8), _f]),
    "s2pb_mgm_weighted": (c_int, [c_void_p, _f, _f, c_int, c_int, c_int, c_int, POINTER(MgmParams), _f, _f, _f, _f,
                                  POINTER(c_uint8), _f]),
    "s2pb_mgm_pkr": (c_int, [c_void_p, _f, _f, c_int, c_int, c_int, c_int, POINTER(MgmParams), _f, _f, POINTER(c_uint8), _f, _f, _f]),
    "s2pb_mgm_device": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int, POINTER(MgmParams),
                                c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "s2pb_mgm_batch": (c_int, [c_void_p, c_int, POINTER(c_void_p), POINTER(c_void_p), c_int, c_int, c_int, c_int,
                               POINTER(MgmParams), POINTER(c_void_p), POINTER(c_void_p), POINTER(c_void_p)]),
    "s2pb_reserve": (c_int, [c_void_p, c_int, c_int, c_int, c_int]),
    "s2pb_num_slots": (c_int, [c_void_p]),
    "s2pb_sync": (c_int, [c_void_p]),
    "s2pb_set_workspace_limit": (c_int, [c_void_p, c_longlong]),
    "s2pb_workspace_bytes": (c_longlong, [c_int, c_int, c_int, c_int, c_int, c_int]),
    "s2pb_workspace_layout": (c_int, [c_int, c_int, c_int, c_int, c_int, c_longlong]),
    "s2pb_folded_calls": (c_longlong, [c_void_p]),
    "s2pb_set_dct_table_limit": (c_int, [c_void_p, c_longlong]),
    "s2pb_dct_coefficients": (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, POINTER(c_double)]),
    "s2pb_homography": (c_int, [c_void_p, _f, c_int, c_int, POINTER(c_double), _f, c_int, c_int]),
    "s2pb_rectify_match": (c_int, [c_void_p, _f, c_int, c_int, POINTER(c_double), _f, c_int, c_int, POINTER(c_double), c_int, c_int,
                                   c_int, c_int, POINTER(MgmParams), _f, _f, _f, _f, POINTER(c_uint8), _f]),
    "s2pb_sgbm_default_params": (c_int, [POINTER(SgbmParams)]),
    "s2pb_sgbm": (c_int, [c_void_p, _f, _f, c_int, c_int, c_int, c_int, POINTER(SgbmParams), _f, POINTER(c_uint8)]),
    "s2pb_merge_n": (c_int, [c_void_p, POINTER(c_void_p), POINTER(c_double), c_int, c_int, c_int, c_int, c_double, _f]),
    "s2pb_disp_to_xyz": (c_int, [c_void_p, POINTER(c_double), _f, _f, _f, _f, c_int, c_int, _f, c_int, c_int,
                                 POINTER(c_double), POINTER(c_double), c_void_p, c_void_p, _f, c_int, c_int]),
    "s2pb_lonlat_to_utm": (c_int, [c_void_p, POINTER(c_double), POINTER(c_double), c_int64, c_int, c_int]),
    "s2pb_set_geoid": (c_int, [c_void_p, _f, c_int, c_int, c_double, c_double, c_double, c_double]),
    "s2pb_set_projection": (c_int, [c_void_p, POINTER(Projection)]),
    "s2pb_lonlat_to_proj": (c_int, [c_void_p, POINTER(c_double), POINTER(c_double), c_int64, POINTER(Projection)]),
    "s2pb_height_map_to_xyz": (c_int, [c_void_p, POINTER(c_double), POINTER(c_double), c_int, c_int, c_void_p, c_double, c_double,
                                       c_int, c_int]),
    "s2pb_height_map": (c_int, [c_void_p, POINTER(c_double), _f, _f, c_int, c_int, _f, c_int, c_int, c_int, c_int, c_int, c_int,
                                POINTER(c_double), POINTER(c_double), c_void_p, c_void_p]),
    "s2pb_resample_heights": (c_int, [c_void_p, POINTER(c_double), c_int, c_int, POINTER(c_double), POINTER(c_double), c_int, c_int]),
    "s2pb_cargarse_basura": (c_int, [c_void_p, _f, _f, c_int, c_int]),
    "s2pb_count_3d_neighbors": (c_int, [c_void_p, POINTER(c_int32), POINTER(c_double), c_int, c_int, c_float, c_int]),
    "s2pb_remove_isolated_3d_points": (c_int, [c_void_p, POINTER(c_double), c_int, c_int, c_float, c_int, c_int, c_int]),
    "s2pb_stretch_8bit": (c_int, [c_void_p, _f, c_int64, c_double, POINTER(c_uint8)]),
    "s2pb_ply_records": (c_int, [c_void_p, POINTER(c_double), c_int64, POINTER(c_uint8), c_int, _f, POINTER(c_uint8), POINTER(c_int64)]),
    "s2pb_disp_to_ply": (c_int, [c_void_p, _f, _f, _f, c_int, c_int, _f, c_int, c_int, POINTER(c_double), POINTER(c_double), c_void_p,
                                 c_void_p, _f, c_int, c_int, c_float, c_int, c_int, _f, c_int, c_double, _f, POINTER(c_uint8),
                                 POINTER(c_int64)]),
    "s2pb_height_map_to_ply": (c_int, [c_void_p, POINTER(c_double), c_int, c_int, c_void_p, c_double, c_double, c_int, c_int, c_float,
                                       c_int, c_int, _f, c_int, c_double, POINTER(c_uint8), POINTER(c_int64)]),
    "s2pb_ply_records_typed": (c_int, [c_void_p, POINTER(c_double), c_int64, c_void_p, c_int, c_int, _f, POINTER(c_uint8),
                                       POINTER(c_int64)]),
    "s2pb_disp_to_ply_clr": (c_int, [c_void_p, _f, _f, _f, c_int, c_int, _f, c_int, c_int, POINTER(c_double), POINTER(c_double),
                                     c_void_p, c_void_p, _f, c_int, c_int, c_float, c_int, c_int, _f, c_int, c_int, c_int,
                                     POINTER(c_double), _f, POINTER(c_uint8), POINTER(c_int64)]),
    "s2pb_height_map_to_ply_clr": (c_int, [c_void_p, POINTER(c_double), c_int, c_int, c_void_p, c_double, c_double, c_int, c_int,
                                           c_float, c_int, c_int, c_void_p, c_int, c_int, POINTER(c_uint8), POINTER(c_int64)]),
    "s2pb_plyflatten": (c_int, [c_void_p, c_int, POINTER(c_void_p), POINTER(c_int64), c_int, POINTER(PlyColumn), c_int, c_double,
                                c_double, c_double, c_int, c_int, _f]),
    "s2pb_mosaic_deflate": (c_int, [c_void_p, c_int, POINTER(c_void_p), POINTER(c_int32), POINTER(c_int32), POINTER(c_int64),
                                    POINTER(c_int64), c_int, c_int, c_int, POINTER(c_uint8), c_int64, POINTER(c_int32)]),
    "s2pb_deflate_blocks": (c_int, [c_void_p, _f, c_int, c_int, c_int, POINTER(c_uint8), c_int64, POINTER(c_int32)]),
    "s2pb_pair_tile_to_ply": (c_int, [c_void_p, POINTER(PairTile), POINTER(c_uint8), POINTER(c_int64), _f, _f, _f, _f, POINTER(c_uint8),
                                      _f]),
    "s2pb_pair_tile_to_height_map": (c_int, [c_void_p, POINTER(PairTile), c_int, c_int, c_int, c_int, POINTER(c_double), _f, _f, _f, _f,
                                             POINTER(c_uint8), _f]),
    "s2pb_heights_tile_to_ply": (c_int, [c_void_p, POINTER(HeightsTile), POINTER(c_uint8), POINTER(c_int64), POINTER(_f), _f]),
    "s2pb_erode_mask": (c_int, [c_void_p, POINTER(c_uint8), POINTER(c_uint8), c_int, c_int, c_float]),
    "s2pb_census": (c_int, [c_void_p, _f, c_int, c_int, c_int, POINTER(c_uint64)]),
    "s2pb_costvolume": (c_int, [c_void_p, _f, _f, c_int, c_int, POINTER(c_int32), POINTER(c_int32), c_int, c_int, c_int, _f]),
    "s2pb_costvolume_dist": (c_int, [c_void_p, _f, _f, c_int, c_int, POINTER(c_int32), POINTER(c_int32), c_int, c_int, c_int,
                                     c_int, _f]),
    "s2pb_aggregate_w": (c_int, [c_void_p, _f, POINTER(c_int32), POINTER(c_int32), c_int, c_int, c_int, c_int, c_float, c_float,
                                 c_int, c_int, c_int, _f, _f, _f, _f, _f]),
    "s2pb_aggregate": (c_int, [c_void_p, _f, POINTER(c_int32), POINTER(c_int32), c_int, c_int, c_int, c_int, c_float, c_float,
                               c_int, c_int, c_int, _f, _f, _f, _f]),
    "s2pb_median": (c_int, [c_void_p, _f, _f, c_int, c_int, c_int]),
    "s2pb_remove_small_cc": (c_int, [c_void_p, _f, _f, c_int, c_int, c_int]),
    "s2pb_rejection_mask": (c_int, [c_void_p, _f, _f, _f, c_int, c_int, POINTER(c_uint8)]),
    "s2pb_last_timings": (c_int, [c_void_p, c_int, _f]),
    "s2pb_kernel_launches": (c_longlong, [c_void_p]),
}


def exported_symbols():
    """Every symbol include/s2pb200.h declares (checked by the CPU test-suite)."""
    return sorted(_SIGNATURES)


def lib():
    """Load the shared library (no CUDA call happens at load time)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                "%s not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "or `make -C s2p_b200/csrc` (there is no CPU fallback)" % LIB_PATH)
        _lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(_lib, name)
            fn.restype = res
            fn.argtypes = args
    return _lib


def check(code):
    if code != OK:
        raise S2pbError(code, lib().s2pb_last_error().decode("utf-8", "replace"))
