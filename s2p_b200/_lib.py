"""ctypes binding of ``libs2pb200.so`` (C ABI in ``include/s2pb200.h``).

Loaded the way the reference loads its own native helpers (``ctypes.CDLL`` on a
library shipped next to the package: s2p/triangulation.py:18-20, s2p/sift.py:25-26).
There is no Python/numpy fallback: if the library is missing or no CUDA device is
visible, the calls raise.
"""
import ctypes
import os
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_int32, c_longlong, c_uint8, c_uint64, c_void_p

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
    "s2pb_homography": (c_int, [c_void_p, _f, c_int, c_int, POINTER(c_double), _f, c_int, c_int]),
    "s2pb_rectify_match": (c_int, [c_void_p, _f, c_int, c_int, POINTER(c_double), _f, c_int, c_int, POINTER(c_double), c_int, c_int,
                                   c_int, c_int, POINTER(MgmParams), _f, _f, _f, _f, POINTER(c_uint8), _f]),
    "s2pb_merge_n": (c_int, [c_void_p, POINTER(c_void_p), POINTER(c_double), c_int, c_int, c_int, c_int, c_double, _f]),
    "s2pb_disp_to_lonlatalt": (c_int, [c_void_p, POINTER(c_double), _f, _f, _f, _f, c_int, c_int, _f, c_int, c_int,
                                       POINTER(c_double), POINTER(c_double), c_void_p, c_void_p, _f]),
    "s2pb_count_3d_neighbors": (c_int, [c_void_p, POINTER(c_int32), POINTER(c_double), c_int, c_int, c_float, c_int]),
    "s2pb_remove_isolated_3d_points": (c_int, [c_void_p, POINTER(c_double), c_int, c_int, c_float, c_int, c_int, c_int]),
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
