"""Boundary #2 (SURVEY.md section 8b): ``s2p.rectification.rectify_pair``.

Everything in ``rectify_pair`` except the two image warps is 3x3 algebra on at most a few hundred points
(s2p/rectification.py:281-378: virtual matches from the RPCs, affine fundamental matrix, rectifying
similarities, disparity range) and needs s2p's own geometry modules (rpcm, estimation, rpc_utils); it stays
the reference's numpy code.  Only ``common.image_apply_homography`` (:379-380) is heavy, and
``s2p_b200.common`` replaces it.  ``rectify_pair`` below therefore is the reference's function running with the
H100 warp installed.  ``rectify_pair_and_match`` goes one step further: the same host algebra, then both warps AND the matcher in
one device call, the rectified pair never leaving the GPU (the opt-in of INTEGRATION.md section 2b).
"""
from . import common


def rectify_pair(im1, im2, rpc1, rpc2, x, y, w, h, out1, out2, A=None, sift_matches=None, method="rpc",
                 hmargin=0, vmargin=0):
    """Same signature and return value (H1, H2, disp_min, disp_max) as s2p.rectification.rectify_pair."""
    try:
        import s2p.rectification as original
    except Exception as e:  # pragma: no cover - depends on the installation
        raise NotImplementedError("rectify_pair's geometry lives in the s2p package (rpcm, estimation, rpc_utils), "
                                  "which is not importable here; s2p_b200.common.image_apply_homography is the "
                                  "part this engine replaces") from e
    common.install()
    return original.rectify_pair(im1, im2, rpc1, rpc2, x, y, w, h, out1, out2, A, sift_matches, method, hmargin, vmargin)


def rectify_pair_and_match(im1, im2, rpc1, rpc2, x, y, w, h, out1, out2, disp, mask, algo, A=None, sift_matches=None, method="rpc",
                           hmargin=0, vmargin=0, timeout=600, max_disp_range=None):
    """Steps 3 and 4 of a tile in one device call (SURVEY.md section 8f rank 3): the reference's own ``rectify_pair`` computes
    the homographies, the output size and the disparity range exactly as it always does -- its two
    ``common.image_apply_homography`` calls (s2p/rectification.py:379-380) are intercepted instead of executed -- then
    ``fused.rectify_and_match`` warps both images into the matcher's device inputs and matches them there.  Writes ``out1``,
    ``out2``, ``disp``, its confidence and ``mask`` like ``rectify_pair`` followed by ``compute_disparity_map``; returns what
    ``rectify_pair`` returns: (H1, H2, disp_min, disp_max)."""
    try:
        import s2p.common as s2p_common
        import s2p.rectification as original
    except Exception as e:  # pragma: no cover - depends on the installation
        raise NotImplementedError("rectify_pair's geometry lives in the s2p package, which is not importable here") from e
    from . import fused
    calls = []
    saved = s2p_common.image_apply_homography
    s2p_common.image_apply_homography = lambda out, im, H, ww, hh: calls.append((out, im, H, ww, hh))
    try:
        H1, H2, disp_min, disp_max = original.rectify_pair(im1, im2, rpc1, rpc2, x, y, w, h, out1, out2, A, sift_matches, method,
                                                           hmargin, vmargin)
    finally:
        s2p_common.image_apply_homography = saved
    if len(calls) != 2 or calls[0][3:] != calls[1][3:]:
        raise RuntimeError("rectify_pair did not warp its two images the way s2p/rectification.py:379-380 does")
    (o1, i1, Ha, ww, hh), (o2, i2, Hb, _, _) = calls
    fused.rectify_and_match(o1, o2, disp, mask, i1, i2, Ha, Hb, ww, hh, algo, disp_min, disp_max, timeout, max_disp_range)
    return H1, H2, disp_min, disp_max


def install():
    """Patch an importable s2p: both boundaries (matcher and warp) and the two "next" rows already served
    (mask erosion, n-view merge) go to the H100 engine, and so do the triangulation steps, the tile's point cloud and the DSM rasterisation."""
    from . import block_matching, cloud, fusion, masking, rasterization, triangulation
    common.install()
    block_matching.install()
    masking.install()
    fusion.install()
    triangulation.install()
    rasterization.install()
    cloud.install()
