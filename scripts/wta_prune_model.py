#!/usr/bin/env python3
"""How much of the pass volumes the WTA has to read when it prunes by the exact bound S[d] >= C[d] (DESIGN.md 3.2).

For the census flavour with unit weights every message of the aggregation is >= 0, so L_p[d] >= C[d] for every pass and
S[d] >= C[d].  With S[d0] of any probe slot d0 known, only the survivors {d : C[d] <= S[d0]} can hold the winner or a
pass minimum; dilated by one slot they also hold the three values of the sub-pixel fit.  This script counts, on the CPU
oracle's C and S of the benchmark's own pairs, which 16-byte lane pieces, 32-byte sectors and 64-byte sector pairs of a
pixel's 128-slot pass vector hold a (dilated) survivor, and asserts on every pixel that winner and fit values from the
survivors alone equal those from the full vector.  `check_claims` with pass volumes does the same for the eight pass arg-minima with pass
volumes from a plain numpy restatement of the scan (small strips only: it is a per-pixel Python loop).

The two-stage mask (`two_stage`) reads pass 0 whole and passes 1-7 only where L_0[d] <= S[d0] (dilated) or
C[d] <= L_q[d0]; `--two-stage` counts it per pass with those pass volumes and gives the bytes the kernel requests (slow:
minutes per strip and view).

    python scripts/wta_prune_model.py [--rows 300:396] [--seeds 0,1] [--size 1024] [--views LR] [--two-stage]
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

INF = np.float32(np.inf)
# mgm_core.cc:884-891: neighbour offsets (dx, dy) of each pass, then inc_x, inc_y, row_major
PASSES = [
    (((-1, 0), (0, -1), (-1, -1), (1, -1)), 1, 1, 1), (((1, 0), (0, 1), (1, 1), (-1, 1)), 0, 0, 1),
    (((0, 1), (-1, 0), (-1, 1), (-1, -1)), 1, 0, 0), (((0, -1), (1, 0), (1, -1), (1, 1)), 0, 1, 0),
    (((-1, -1), (1, -1), (0, -1), (1, 0)), 0, 1, 1), (((1, -1), (1, 1), (1, 0), (0, 1)), 0, 0, 0),
    (((1, 1), (-1, 1), (0, 1), (-1, 0)), 1, 0, 1), (((-1, 1), (-1, -1), (-1, 0), (0, -1)), 1, 1, 0),
]


def pass_volumes(C, P1=8.0, P2=32.0, tsgm=3):
    """The eight L_p of a cost volume C [h][w][D] (+INF outside a pixel's range), unit weights, in float32 and in the
    reference's operation order (update_cost2, mgm_core.cc:46-70)."""
    h, w, D = C.shape
    P1, P2, div = np.float32(P1), np.float32(P2), np.float32(2 if tsgm == 2 else tsgm)
    out = []
    pad = np.full(1, INF, np.float32)
    for nb, inc_x, inc_y, row_major in PASSES:
        L = np.full_like(C, INF)
        for jj in range(h if row_major else w):
            for ii in range(w if row_major else h):
                x, y = (ii, jj) if row_major else (jj, ii)
                if not inc_x:
                    x = w - 1 - x
                if not inc_y:
                    y = h - 1 - y
                if any(not (0 <= x + dx < w and 0 <= y + dy < h) for dx, dy in nb):
                    L[y, x] = C[y, x]
                    continue
                e = np.zeros(D, np.float32)
                for dx, dy in nb[:tsgm]:
                    Lq = L[y + dy, x + dx]
                    mq = Lq.min()
                    side = np.minimum(np.concatenate((pad, Lq[:-1])), np.concatenate((Lq[1:], pad)))
                    t = np.minimum(np.minimum(Lq, side + P1), mq + P2) - mq
                    e = e + (t / div if tsgm == 2 else t)
                L[y, x] = C[y, x] + (e if tsgm == 2 else e / div)
        out.append(L)
    return out


def sum_passes(Ls, C, fix_overcount=1):
    S = np.zeros_like(C)
    for L in Ls:
        S = S + L
    if fix_overcount:                      # fma(-7, C, S): exact in double for the integer census costs; NaN where C is +INF
        with np.errstate(invalid="ignore"):
            S = (S.astype(np.float64) - 7.0 * C.astype(np.float64)).astype(np.float32)
    return S


def first_min(S):
    """first strict minimum over the finite S (mgm_core.cc:1044-1048) -> slot [h][w]"""
    return np.argmin(np.where(np.isfinite(S), S, INF), axis=-1)


def probe_value(C, S, rule):
    """S at the probe slot(s) of every pixel -> [h][w].  'cmin': first arg-minimum of C; 'best': the true minimum of S;
    'cmin+prev': the smaller of 'cmin' and S at the winner of the pixel on the left when that slot is finite here."""
    if rule == "best":
        return np.take_along_axis(S, first_min(S)[..., None], -1)[..., 0]
    t = np.take_along_axis(S, np.argmin(C, axis=-1)[..., None], -1)[..., 0]
    if rule == "cmin+prev":
        k = first_min(S)
        prev = np.concatenate((k[:, :1], k[:, :-1]), axis=1)
        t2 = np.take_along_axis(S, prev[..., None], -1)[..., 0]
        t = np.minimum(t, np.where(np.isfinite(t2), t2, INF))
    return t


def dilate(s):
    d = s.copy()
    d[..., 1:] |= s[..., :-1]
    d[..., :-1] |= s[..., 1:]
    return d


def survivors(C, T):
    """{d : C[d] <= T} dilated by one slot on each side, clipped to the slab.  T is taken 2^-16 wider, like the kernel's:
    the scaled costs of census 3x3 / 7x7 round in the sums (the integer costs of 5x5 do not)."""
    s = C <= (T * np.float32(1 + 2.0 ** -16))[..., None]
    return s, dilate(s)


def two_stage(C, T, Ls):
    """The slots each pass is read on by the two-stage WTA (wta_pruned_kernel) -> eight [h][w][D] masks.  Pass 0: every
    slot (the kernel requests it with the probe).  Passes 1-7: {d : L_0[d] <= T}, dilated (S >= L_0 like S >= C, same
    slack), and {d : C[d] <= L_q[d0]} with d0 the probe slot (first arg-minimum of C): every arg-minimum of L_q lies there."""
    d1 = dilate(Ls[0] <= (T * np.float32(1 + 2.0 ** -16))[..., None])
    k0 = np.argmin(C, axis=-1)[..., None]
    return [np.ones(C.shape, bool)] + [d1 | (C <= np.take_along_axis(L, k0, -1)) for L in Ls[1:]]


def check_claims(C, S, dil, Ls=None):
    """winner, fit values and (with the pass volumes) the eight last arg-minima from the survivors only equal those from
    the full vectors, on every pixel.  A slot with C = +INF has L_p = +INF whether it is read or not.  dil: one mask for
    every pass, or a list of eight (two_stage): a slot missed by any pass sums to +INF."""
    per_pass = isinstance(dil, (list, tuple))
    dils = [d | np.isinf(C) for d in (dil if per_pass else [dil] * 8)]
    dil = np.logical_and.reduce(dils)
    Sp = np.where(dil, S, INF)
    k = first_min(S)
    assert np.array_equal(first_min(Sp), k), "winner differs"
    D = S.shape[-1]
    for o in (-1, 0, 1):
        kk = np.clip(k + o, 0, D - 1)
        a = np.take_along_axis(S, kk[..., None], -1)
        b = np.take_along_axis(Sp, kk[..., None], -1)
        assert np.array_equal(a, b, equal_nan=True), "fit value %+d differs" % o
    for L, dq in zip(Ls or (), dils):
        Lp = np.where(dq, L, INF)
        last = lambda V: D - 1 - np.argmax((V == V.min(-1, keepdims=True))[..., ::-1], axis=-1)
        assert np.array_equal(last(L), last(Lp)), "pass arg-minimum differs"


def fractions(C, S, rule):
    """-> dict of requested fractions of one view (probes not included)"""
    T = probe_value(C, S, rule)
    s, d = survivors(C, T)
    check_claims(C, S, d)
    h, w, D = C.shape
    cmax = np.where(np.isfinite(C), C, -INF).max(-1)
    return dict(survivors=s.mean(), piece16=d.reshape(h, w, D // 4, 4).any(-1).mean(),
                sector32=d.reshape(h, w, D // 8, 8).any(-1).mean(), pair64=d.reshape(h, w, D // 16, 16).any(-1).mean(),
                unpruned=(T >= cmax).mean())


def strip_volumes(seed, size, rows, dmin, dmax, nan_border, view):
    from oracle import oracle as O
    from s2p_b200.synth import make_pair
    ref, sec, _ = make_pair(size, size, dmin, dmax, seed=seed, nan_border=nan_border)
    ref, sec = ref[rows[0]:rows[1]], sec[rows[0]:rows[1]]
    nl, nr = np.isnan(ref), np.isnan(sec)
    u, v = np.where(nl, 0, ref).astype(np.float32), np.where(nr, 0, sec).astype(np.float32)
    if view == "L":
        lo, hi = np.full(u.shape, dmin, np.int32), np.where(nl, dmin + 1, dmax).astype(np.int32)
    else:                                   # main_mgm.cc:207,214-216
        u, v = v, u
        lo, hi = np.where(nr, dmin, -dmax).astype(np.int32), np.where(nr, dmin + 1, -dmin).astype(np.int32)
    gmin = int(lo.min())
    D = int(hi.max()) - gmin + 1
    C = O.port.costvolume(u, v, lo, hi, gmin, D, 5)
    S = O.port.aggregate(C, lo, hi, gmin, 8.0, 32.0, 8, 3)[0]
    Dp = -(-D // 32) * 32                   # the slab: +INF padding up to a multiple of 32 slots
    padw = ((0, 0), (0, 0), (0, Dp - D))
    return np.pad(C, padw, constant_values=INF), np.pad(S, padw, constant_values=INF)


RULES = (("cmin", 1), ("best", 1), ("cmin+prev", 2))


def sector_fraction(d):
    h, w, D = d.shape
    return d.reshape(h, w, D // 8, 8).any(-1).mean()


def requested_bytes(npix, DP, f):
    """bytes wta_pruned_kernel requests for a view of npix pixels and DP slots: the 32-byte sectors of the eight passes
    (fractions f), one probe sector per pass, the codes"""
    return npix * (sum(f) * 4 * DP + 8 * 32 + DP)


def two_stage_fractions(C, S):
    """-> (per-pass 32-byte sector fractions of the two-stage mask, that of the one-stage mask), probes not included; checks
    winner, fit and the eight arg-minima of the two-stage mask on every pixel"""
    Ls = pass_volumes(C)
    fin = np.isfinite(S)
    assert np.array_equal(sum_passes(Ls, C)[fin], S[fin]), "numpy pass volumes do not sum to the oracle's S"
    T = probe_value(C, S, "cmin")
    masks = two_stage(C, T, Ls)
    check_claims(C, S, masks, Ls)
    return [sector_fraction(d) for d in masks], sector_fraction(survivors(C, T)[1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", default="300:396")
    ap.add_argument("--seeds", default="0")
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--views", default="LR")
    ap.add_argument("--two-stage", action="store_true", help="per-pass sector fractions of the two-stage mask")
    a = ap.parse_args()
    rows = tuple(int(x) for x in a.rows.split(":"))
    if a.two_stage:
        # GB: what the kernel requests for the whole size x size view at the strip's fractions
        print("| tile | view | C <= T, every pass | pass 0 | passes 1-7 | mean of 8 | mean + probes | GB per view |")
        print("|---|---|---|---|---|---|---|---|")
        for nanb in (0.0, 0.05):
            for seed in (int(s) for s in a.seeds.split(",")):
                for view in a.views:
                    C, S = strip_volumes(seed, a.size, rows, -64, 63, nanb, view)
                    f, f1 = two_stage_fractions(C, S)
                    print("| seed %d%s | %s | %.3f | %.3f | %.3f-%.3f | %.3f | %.3f | %.2f |" % (
                        seed, " nodata" if nanb else "", view, f1, f[0], min(f[1:]), max(f[1:]), np.mean(f),
                        np.mean(f) + 1 / (C.shape[-1] // 8), requested_bytes(a.size * a.size, C.shape[-1], f) / 1e9),
                        flush=True)
        return
    # "unpruned pixels": S[d0] >= the largest finite C, recognisable before any mask work -- they read every sector
    print("| tile | view | probe | survivors | 16 B pieces | 32 B sectors | 64 B pairs | unpruned pixels | sectors + probes |")
    print("|---|---|---|---|---|---|---|---|---|")
    for nanb in (0.0, 0.05):
        for seed in (int(s) for s in a.seeds.split(",")):
            for view in a.views:
                C, S = strip_volumes(seed, a.size, rows, -64, 63, nanb, view)
                nsec = C.shape[-1] // 8
                for rule, nprobe in RULES:
                    f = fractions(C, S, rule)
                    # a probe requests one 32-byte sector per pass (an upper bound: the probe slot is a survivor itself, so the
                    # bulk loads request the same sector again)
                    print("| seed %d%s | %s | %s | %.3f | %.3f | %.3f | %.3f | %.3f | %.3f |" % (
                        seed, " nodata" if nanb else "", view, rule, f["survivors"], f["piece16"], f["sector32"], f["pair64"],
                        f["unpruned"], f["sector32"] + nprobe / nsec), flush=True)


if __name__ == "__main__":
    main()
