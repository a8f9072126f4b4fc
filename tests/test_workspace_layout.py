"""The workspace arithmetic of the two layouts (s2pb_workspace_bytes) against an independent restatement of them, and the rule
that picks one (s2pb_workspace_layout).  No device needed."""
import pytest

from s2p_b200 import _lib
from s2p_b200.engine import workspace_bytes, workspace_layout

LPLS = (1, 2, 3, 4, 5, 6, 8, 12, 16)     # register-resident widths (labels per lane); wider slabs: 32-label chunks


def _slots(D):
    for n in LPLS:
        if 32 * n >= D:
            return 32 * n
    return 32 * -(-D // 32)


def _band_lines(DP, gen):
    """scanlines per band of the kernel that aggregates a slab of DP slots"""
    if DP <= 512:
        return 16
    if gen:
        return 8 if DP <= 1024 else 2
    return 8 if DP <= 1024 else 4


def restated(w, h, D, ndir, cost_bytes, folded):
    DP, npix = _slots(D), w * h
    sizes = []
    for _view in range(2):
        sizes += [npix * 4, npix * 2, npix * 2, npix * 8, npix * 4, npix * 8, (h + w) * 4 + w + 16, h * 4, 256]
        sizes.append(npix * DP * cost_bytes)                           # costs
        if folded:
            nw = _band_lines(DP, cost_bytes == 4)
            boundary = max(-(-h // nw) * w, -(-w // nw) * h)           # one scanline per band, larger scan geometry
            sizes += [npix * DP * 4, boundary * DP * 4] + [npix * 2] * ndir + [npix * 4] * ndir
        else:
            sizes += [npix * DP * 4, npix * 4] * ndir                  # pass volumes and their minima
        sizes += [8 * ((max(w, h) + 1) // 2) * 4] + [npix * 4] * 4     # progress; disp, cost, conf, tmp
    sizes += [256, 256, npix * 8]
    return sum(-(-s // 256) * 256 for s in sizes)


SHAPES = [(96, 160, 48, 8, 1), (900, 820, 400, 8, 1), (2100, 2020, 400, 8, 1), (2048, 2048, 512, 8, 1),
          (640, 37, 600, 8, 1), (517, 333, 1100, 4, 1), (300, 200, 2048, 2, 1), (300, 200, 700, 8, 4),
          (300, 200, 1500, 8, 4), (1000, 1000, 100, 8, 4), (45, 70, 24, 2, 1), (2, 2, 1, 8, 1)]


@pytest.mark.parametrize("w,h,D,ndir,cb", SHAPES)
@pytest.mark.parametrize("folded", [False, True])
def test_workspace_bytes_restated(w, h, D, ndir, cb, folded):
    assert workspace_bytes(w, h, D, ndir, cb, folded) == restated(w, h, D, ndir, cb, folded)


def test_folded_is_far_smaller():
    # 2048 x 2048 x 512 labels: ~142 GB resident, ~22.5 GB folded
    res, fold = workspace_bytes(2048, 2048, 512), workspace_bytes(2048, 2048, 512, folded=True)
    assert 140e9 < res < 145e9 and 22e9 < fold < 23.5e9
    assert workspace_bytes(2100, 2020, 400) > 80 * 2 ** 30 > workspace_bytes(2100, 2020, 400, folded=True)


@pytest.mark.parametrize("w,h,D,ndir,cb", SHAPES)
def test_selection_rule(w, h, D, ndir, cb):
    res, fold = restated(w, h, D, ndir, cb, False), restated(w, h, D, ndir, cb, True)
    assert fold < res
    for limit in (0, res + 1, res, res - 1, (res + fold) // 2, fold + 1, fold, fold - 1, 1):
        if limit == 0 or res <= limit:
            assert workspace_layout(w, h, D, ndir, cb, limit) == "resident"
        elif fold <= limit:
            assert workspace_layout(w, h, D, ndir, cb, limit) == "folded"
        else:
            with pytest.raises(_lib.S2pbError) as e:
                workspace_layout(w, h, D, ndir, cb, limit)
            assert e.value.code == _lib.lib().s2pb_workspace_layout(w, h, D, ndir, cb, limit) == -4   # S2PB_ERR_NOMEM


@pytest.mark.parametrize("args", [(1, 5, 10, 8, 1), (5, 5, 0, 8, 1), (5, 5, 10, 3, 1), (5, 5, 10, 8, 2), (5, 5, 2049, 8, 1)])
def test_workspace_bytes_rejects(args):
    with pytest.raises(_lib.S2pbError):
        workspace_bytes(*args)
