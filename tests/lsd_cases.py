"""The images on which the weight maps of algo == 'mgm_multi_lsd' are checked, and the recorded oracle for them
(tests/golden/lsd_weights.npz, written by tests/golden/make_golden_lsd.py where oracle/_ref is built)."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")
RECORDED = os.path.join(GOLDEN, "lsd_weights.npz")
if os.path.dirname(HERE) not in sys.path:
    sys.path.insert(0, os.path.dirname(HERE))


def _real(key):
    return np.load(os.path.join(GOLDEN, "real_pair.npz"))[key].astype(np.float32)


def _lines(h, w, angle_deg, spacing, seed, noise=2.0):
    """Bright bands at ``angle_deg`` every ``spacing`` pixels on a noisy 12-bit-like background."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    t = np.deg2rad(angle_deg)
    d = x * np.sin(t) - y * np.cos(t)
    img = 300.0 + 900.0 * (np.mod(d, spacing) < spacing / 2) + rng.normal(0.0, noise, (h, w))
    return img.astype(np.float32)


def _nan_border(img, b):
    img = img.copy()
    img[:b], img[-b:], img[:, :b], img[:, -b:] = np.nan, np.nan, np.nan, np.nan
    return img


def _mostly_nan(h, w, seed):
    img = np.full((h, w), np.nan, np.float32)
    img[: h // 8, : w // 8] = np.random.default_rng(seed).uniform(0, 1000, (h // 8, w // 8))
    return img


def _pair():
    """The tile of tests/test_gpu_lsd.py::test_dropin_mgm_multi_lsd_starts_no_process"""
    from s2p_b200.synth import make_pair
    return make_pair(110, 160, -14, 11, seed=71)[:2]


CASES = {
    "crop1": lambda: _real("crop1"),
    "crop2": lambda: _real("crop2"),
    "rectified": lambda: np.load(os.path.join(GOLDEN, "real_pair_rectified_ref.npz"))["rectified_ref"],
    "crop1_reflect_1024": lambda: np.pad(_real("crop1"), ((0, 1024 - 597), (0, 1024 - 537)), mode="reflect"),
    "lines_0": lambda: _lines(96, 128, 0.0, 16, 1),
    "lines_45": lambda: _lines(96, 128, 45.0, 16, 2),
    "lines_90": lambda: _lines(96, 128, 90.0, 16, 3),
    "lines_generic": lambda: _lines(101, 77, 23.7, 13, 4),
    "dense_parallel": lambda: _lines(64, 64, 61.3, 4, 5),
    "noise": lambda: np.random.default_rng(6).uniform(0, 4095, (83, 97)).astype(np.float32),
    "nan_border": lambda: _nan_border(_lines(90, 110, 12.5, 11, 7), 9),
    "constant": lambda: np.full((48, 40), 517.0, np.float32),
    "one_wide": lambda: _lines(57, 1, 30.0, 9, 8),
    "two_wide": lambda: _lines(57, 2, 30.0, 9, 9),
    "odd_size": lambda: _lines(37, 211, 100.0, 7, 10),
    "mostly_nan": lambda: _mostly_nan(80, 96, 11),
    "pair_ref": lambda: _pair()[0],
    "pair_sec": lambda: _pair()[1],
}


def recorded():
    """-> {case: {field: value}} from the golden file."""
    z = np.load(RECORDED)
    out = {}
    for k in z.files:
        name, field = k.split("/")
        v = z[k]
        out.setdefault(name, {})[field] = v.item() if v.ndim == 0 else v
    return out
