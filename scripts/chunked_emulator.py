"""CPU emulation of run_band_chunked (s2p_b200/csrc/agg_chunked.cuh), index for index: ring slots, guards, meta,
staging slots, the 4-byte range words, the previous band's ring.  Warps run one after the other inside a step and
bands one after the other, so this checks the kernel's indexing and masking logic, not its synchronisation.  The
sum of the emulated pass volumes is compared with the oracle's aggregated volume (bit for bit).
EMU_GENERAL=1 replays the general flavour (GEN): float costs, a weight image, penalties P*w rounded as the kernel does,
with the kernel's warps and pipeline depth for the slab (ck_warps / ck_stage).
usage: python scripts/chunked_emulator.py [DP] [h] [w] [tsgm] [seed]"""
import os
import sys
from fractions import Fraction

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from oracle import oracle as O

F = np.float32
INF = F(np.inf)
W_, RING, STAGE, R0, PAD, PUBLISH = 16, 4, 4, 8, 4, 8
if os.environ.get("EMU_WARPS"):          # the configurations of the slabs wider than 512 slots: 8 warps / 2 stages, 4 warps / 2 stages
    W_ = int(os.environ["EMU_WARPS"])
    STAGE = int(os.environ.get("EMU_STAGE", 2))
    R0 = 2 * STAGE
FIXED = os.environ.get("EMU_BUGGY") != "1"      # EMU_BUGGY=1 reproduces the first version of the kernel (chunk-edge bug)
GENERAL = os.environ.get("EMU_GENERAL") == "1"


def fma32(a, b, c):
    """fmaf on float32 values: a*b is exact in float64, and the float64 sum rounds to the float32 result unless it lands on
    a float32 midpoint (low 29 bits of the float64 = 1 followed by zeros); those few are redone exactly"""
    a, b, c = np.broadcast_arrays(np.atleast_1d(np.asarray(a, F)), np.atleast_1d(np.asarray(b, F)), np.atleast_1d(np.asarray(c, F)))
    r64 = a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)
    r = r64.astype(F)
    tie = (r64.view(np.uint64) & np.uint64(0x1FFFFFFF)) == np.uint64(0x10000000)
    if tie.any():
        for i in zip(*np.nonzero(tie)):
            x = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
            if x != Fraction(float(r64[i])):
                lo_, hi_ = np.nextafter(F(r64[i]), F(-np.inf)), np.nextafter(F(r64[i]), F(np.inf))
                lo_, hi_ = (lo_, r[i]) if r[i] > r64[i] else (r[i], hi_)
                r[i] = lo_ if x < Fraction(float(r64[i])) else hi_
    return r if r.size > 1 else r[0]


def fill_pass(p, w, h):
    W, H = w, h
    t = [(h, w, 0, w, 1, 0), (h, w, (H - 1) * W + (W - 1), -w, -1, 0), (w, h, (H - 1) * W, 1, -w, 0), (w, h, W - 1, -1, w, 0),
         (h, w, W - 1, w, -1, 1), (w, h, (H - 1) * W + (W - 1), -1, -w, 1), (h, w, (H - 1) * W, -w, 1, 1), (w, h, 0, 1, w, 1)][p]
    return dict(nS=t[0], nI=t[1], base=t[2], strideS=t[3], strideI=t[4], type=t[5])


def run_pass(pd, C, lo_img, hi_img, gmin, DP, tsgm, P1, P2, L, Lmin, W=None):
    """C: [npix, DP] float32 costs (the census slab's values), lo_img / hi_img: int16 [npix] labels, W: float32 [npix] weights
    (GENERAL only, None = unweighted).  Fills L [npix, DP], Lmin [npix]."""
    TYPE = pd["type"]
    useA = True if TYPE == 0 else tsgm == 4
    useCn = tsgm >= 2 if TYPE == 0 else tsgm >= 3
    useB = tsgm >= 3 if TYPE == 0 else tsgm >= 2
    useE = tsgm == 4 if TYPE == 0 else True
    usePrev = useCn or useB or useE
    SKEW, LEAD = (2, 1) if useE else (1, 0)
    S = STAGE - 1
    NC, VS = DP // 32, DP + 2 * PAD
    nI, nS, sI, sS = pd["nI"], pd["nS"], pd["strideI"], pd["strideS"]
    lane = np.arange(32)
    lo_words = lo_img.view(np.uint32) if lo_img.size % 2 == 0 else np.concatenate([lo_img, [0]]).astype(np.int16).view(np.uint32)
    hi_words = hi_img.view(np.uint32) if hi_img.size % 2 == 0 else np.concatenate([hi_img, [0]]).astype(np.int16).view(np.uint32)
    nbands = (nS + W_ - 1) // W_
    for band in range(nbands):
        ring = np.full((W_, RING, VS), F(777.0), F)           # stale values must never matter
        meta = np.zeros((W_, RING, 3), np.float64)
        r0 = np.full((R0, VS), F(555.0), F)
        r0m = np.zeros(R0, F)
        r0[:, :PAD] = INF
        r0[:, PAD + DP:] = INF
        cst = np.full((W_, STAGE, DP), F(333.0), F)
        rng = np.zeros((W_, STAGE, 2), np.uint32)
        wst = np.full((W_, STAGE), F(999.0), F)
        r0rng = np.zeros((R0, 2), np.uint32)
        st = []
        for k in range(W_):
            s = band * W_ + k
            live = s < nS
            rowbase = pd["base"] + s * sS
            st.append(dict(s=s, live=live, rowbase=rowbase, prev=usePrev and live and s > 0, jc=0, pidx=rowbase, jp=0, upix=rowbase,
                           outpix=rowbase, prevbase=rowbase - sS))

        def range_words(k, j):
            w = st[k]
            if w["live"] and j < nI:
                q = w["rowbase"] + j * sI
                return int(lo_words[(q * 2 & ~3) // 4]), int(hi_words[(q * 2 & ~3) // 4])
            return 0, 0
        for k in range(W_):
            st[k]["nw"] = [range_words(k, 0), range_words(k, 1), range_words(k, 2)]

        def stage_mine(k):
            w = st[k]
            if w["live"] and w["jc"] < nI:
                slot = w["jc"] & (STAGE - 1)
                sh = (w["pidx"] & 1) * 16
                s16 = lambda v: v - 65536 if v >= 32768 else v
                ea = (s16((w["nw"][0][0] >> sh) & 0xffff) - gmin) >> 5
                eb = (s16((w["nw"][0][1] >> sh) & 0xffff) - gmin) >> 5
                cst[k, slot, 32 * ea:32 * (eb + 1)] = C[w["pidx"], 32 * ea:32 * (eb + 1)]      # only the chunks of the span
                rng[k, slot, 0] = lo_words[(w["pidx"] * 2 & ~3) // 4]
                rng[k, slot, 1] = hi_words[(w["pidx"] * 2 & ~3) // 4]
                if W is not None:
                    wst[k, slot] = W[w["pidx"]]
                w["pidx"] += sI
            w["jc"] += 1
            w["nw"] = [w["nw"][1], w["nw"][2], range_words(k, w["jc"] + 2)]

        def stage_prevband(k):
            w = st[k]
            if k == 0 and w["prev"]:
                if w["jp"] < nI:
                    slot = w["jp"] & (R0 - 1)
                    q = w["prevbase"] + w["jp"] * sI
                    r0[slot, PAD:PAD + DP] = L[q]
                    r0m[slot] = Lmin[q]
                    r0rng[slot, 0] = lo_words[(q * 2 & ~3) // 4]
                    r0rng[slot, 1] = hi_words[(q * 2 & ~3) // 4]
                w["jp"] += 1

        def nb_at(k, j, mine):
            if mine:
                slot = j & (RING - 1)
                return ring[k, slot], F(meta[k, slot, 0]), int(meta[k, slot, 1]), int(meta[k, slot, 2])
            if k == 0:
                slot = j & (R0 - 1)
                qpix = st[0]["prevbase"] + j * sI
                sh = (qpix & 1) * 16
                s16 = lambda v: v - 65536 if v >= 32768 else v
                qlo, qhi = s16((int(r0rng[slot, 0]) >> sh) & 0xffff), s16((int(r0rng[slot, 1]) >> sh) & 0xffff)
                assert qlo == lo_img[qpix] and qhi == hi_img[qpix], "previous-band range word mismatch"
                ea, eb = (qlo - gmin) >> 5, (qhi - gmin) >> 5
                r0[slot, PAD + 32 * ea - 1] = INF
                r0[slot, PAD + 32 * (eb + 1)] = INF
                return r0[slot], r0m[slot], ea, eb
            slot = j & (RING - 1)
            return ring[k - 1, slot], F(meta[k - 1, slot, 0]), int(meta[k - 1, slot, 1]), int(meta[k - 1, slot, 2])

        def term(n, e, kk, ordn, wv, P1w):
            v, m, ea, eb = n
            a, c0, b = np.full(32, INF, F), np.full(32, INF, F), np.full(32, INF, F)
            if ea <= e <= eb:
                a, c0, b = v[PAD + kk - 1], v[PAD + kk], v[PAD + kk + 1]
            elif FIXED and e == ea - 1:          # lane 31's right neighbour is the first element of the neighbour's span
                b[31] = v[PAD + kk[31] + 1]
            elif FIXED and e == eb + 1:          # lane 0's left neighbour is the last element of its span
                a[0] = v[PAD + kk[0] - 1]
            if GENERAL:        # P1*w: mul then add for the 1st / 2nd neighbour of the list, fma for the 3rd / 4th; P2*w: fma
                v1 = fma32(F(P1), wv, np.minimum(a, b)) if ordn >= 2 else np.minimum(a, b) + P1w
                return np.minimum(np.minimum(c0, v1), fma32(F(P2), wv, m)) - m
            v1 = np.minimum(a, b) + F(P1)
            return np.minimum(np.minimum(c0, v1), m + F(P2)) - m

        for k in range(W_):
            if LEAD == 1:
                stage_prevband(k)
            for _ in range(S):
                stage_mine(k)
                stage_prevband(k)
        for t in range(nI + (W_ - 1) * SKEW):
            for k in range(W_):
                w = st[k]
                i = t - k * SKEW
                act = w["live"] and 0 <= i < nI
                if i >= 0:
                    stage_mine(k)
                    stage_prevband(k)
                if not act:
                    continue
                slot = i & (STAGE - 1)
                sh = (w["upix"] & 1) * 16
                s16 = lambda v: v - 65536 if v >= 32768 else v          # (int)(short)
                plo = s16((int(rng[k, slot, 0]) >> sh) & 0xffff)
                phi = s16((int(rng[k, slot, 1]) >> sh) & 0xffff)
                assert plo == lo_img[w["upix"]] and phi == hi_img[w["upix"]], "range word mismatch"
                ea, eb = (plo - gmin) >> 5, (phi - gmin) >> 5
                border = w["s"] == 0 or i == 0 or i == nI - 1
                if not border:
                    nA = nb_at(k, i - 1, True)
                    nB = nb_at(k, i - 1, False) if useB else None
                    nC = nb_at(k, i, False) if useCn else None
                    nE = nb_at(k, i + 1, False) if useE else None
                mine = ring[k, i & (RING - 1)]
                lm = np.full(32, INF, F)
                wv = wst[k, slot] if W is not None else F(1.0)
                P1w = F(P1) * wv
                outv = L[w["outpix"]].copy()
                for e in range(NC):
                    kk = 32 * e + lane
                    if ea <= e <= eb:
                        c = cst[k, slot, kk]
                        Lv = c.copy()
                        if not border:
                            if TYPE == 0:         # the reference's neighbour list: A, Cn, B, E
                                acc = term(nA, e, kk, 0, wv, P1w)
                                if tsgm == 2:
                                    acc = acc * F(0.5)
                                if useCn:
                                    tt = term(nC, e, kk, 1, wv, P1w)
                                    acc = acc + (tt * F(0.5) if tsgm == 2 else tt)
                                if useB:
                                    acc = acc + term(nB, e, kk, 2, wv, P1w)
                                if useE:
                                    acc = acc + term(nE, e, kk, 3, wv, P1w)
                            else:                 # E, B, Cn, A
                                acc = term(nE, e, kk, 0, wv, P1w)
                                if tsgm == 2:
                                    acc = acc * F(0.5)
                                if useB:
                                    tt = term(nB, e, kk, 1, wv, P1w)
                                    acc = acc + (tt * F(0.5) if tsgm == 2 else tt)
                                if useCn:
                                    acc = acc + term(nC, e, kk, 2, wv, P1w)
                                if useA:
                                    acc = acc + term(nA, e, kk, 3, wv, P1w)
                            if tsgm == 3:
                                acc = acc / F(3)
                            if tsgm == 4:
                                acc = acc * F(0.25)
                            Lv = c + acc
                        mine[PAD + kk] = Lv
                        lm = np.minimum(lm, Lv)
                        outv[kk] = Lv
                m = lm.min()
                mine[PAD + 32 * ea - 1] = INF
                mine[PAD + 32 * (eb + 1)] = INF
                meta[k, i & (RING - 1)] = (m, ea, eb)
                L[w["outpix"]] = outv
                Lmin[w["outpix"]] = m          # (the kernel only writes it for the band-closing scanline)
                w["outpix"] += sI
                w["upix"] += sI


def main():
    global W_, STAGE, R0
    a = [int(x) for x in sys.argv[1:6]] + [512, 40, 48, 3, 0][len(sys.argv) - 1:]
    DP, h, w, tsgm, seed = a
    if GENERAL and not os.environ.get("EMU_WARPS"):      # ck_warps / ck_stage of the general flavour
        W_, STAGE = (8 if DP <= 1024 else 2), 2
        R0 = 2 * STAGE
    rng_ = np.random.default_rng(seed)
    npix = h * w
    gmin = -DP // 2
    # label ranges: most pixels narrow around a smooth surface, some with the full range (as next to rejected pixels)
    yy, xx = np.mgrid[0:h, 0:w]
    centre = (gmin + DP // 2 + 0.3 * DP * np.sin(xx / 9.0) * np.cos(yy / 7.0)).astype(int)
    lo = np.clip(centre - rng_.integers(8, 20, (h, w)), gmin, gmin + DP - 1)
    hi = np.clip(centre + rng_.integers(8, 20, (h, w)), gmin, gmin + DP - 1)
    wide = rng_.random((h, w)) < 0.12
    lo[wide], hi[wide] = gmin, gmin + DP - 1
    lo, hi = lo.astype(np.int32), hi.astype(np.int32)
    C = np.full((h, w, DP), np.inf, np.float32)
    vals = rng_.integers(0, 25, (h, w, DP)).astype(np.float32)
    Wimg = None
    P1, P2 = 8.0, 32.0
    if GENERAL:        # costs with fractions (as ad / btad / ncc give), LSD-like weights, penalties whose products are inexact
        vals = rng_.uniform(0, 40, (h, w, DP)).astype(np.float32)
        Wimg = np.maximum(rng_.uniform(0, 1, (h, w)) ** 2, 0.1).astype(np.float32)
        Wimg[rng_.random((h, w)) < 0.5] = 1.0
        P1, P2 = 12.0, 48.0
    k = np.arange(DP)[None, None, :] + gmin
    inr = (k >= lo[..., None]) & (k <= hi[..., None])
    C[inr] = vals[inr]
    So, do, co, fo = O.port.aggregate(C, lo, hi, gmin, P1, P2, 8, tsgm, weights=Wimg)
    Cf = C.reshape(npix, DP)
    lo16, hi16 = lo.reshape(-1).astype(np.int16), hi.reshape(-1).astype(np.int16)
    Ls = []
    for p in range(8):
        L = np.full((npix, DP), np.float32(-1.0), np.float32)
        Lmin = np.zeros(npix, np.float32)
        run_pass(fill_pass(p, w, h), Cf, lo16, hi16, gmin, DP, tsgm, P1, P2, L, Lmin, None if Wimg is None else Wimg.reshape(-1))
        Ls.append(L)
        print("pass", p, "done", flush=True)
    Ssum = np.zeros((npix, DP), np.float32)
    for L in Ls:
        Ssum = Ssum + L
    Ssum = (np.float64(-7.0) * Cf.astype(np.float64) + Ssum.astype(np.float64)).astype(np.float32)     # fmaf(-7, C, S)
    So = So.reshape(npix, DP)
    ok = (Ssum == So) | (np.isnan(Ssum) & np.isnan(So)) | (~inr.reshape(npix, DP))
    print("%sDP %d %dx%d tsgm %d (%d warps, %d stages): %d of %d in-range voxels differ" % (
        "general, " if GENERAL else "", DP, w, h, tsgm, W_, STAGE, int((~ok).sum()), int(inr.sum())))
    # chunks outside a pixel's span are never written in the emulated global volume (the chunk-skipping WTA never reads them)
    ea, eb = (lo.reshape(-1) - gmin) >> 5, (hi.reshape(-1) - gmin) >> 5
    e_of = (np.arange(DP) >> 5)[None, :]
    outside = (e_of < ea[:, None]) | (e_of > eb[:, None])
    print("skipped chunks untouched:", bool(np.all(Ls[0][outside] == np.float32(-1.0))))
    if os.environ.get("EMU_WTA", "1") == "1":
        main_wta(DP, h, w, tsgm, seed, Ls, Cf, lo.reshape(-1), hi.reshape(-1), gmin, Wimg, P1, P2)


def vfit3(v0, v1, v2):
    """vfit3 of mgm_kernels.cuh (refine.h:70-92 with the fused minimum value) -> (vmin, xmin), float32"""
    if v1 > v0 and v1 > v2:
        return v1, F(0)
    slope = v2 - v1
    if (v2 - v1) < (v0 - v1):
        slope = v0 - v1
    xmin = (v0 - v2) / (F(2) * slope)
    vmin = F(np.float64(xmin - F(1)) * np.float64(slope) + np.float64(v2))       # fmaf
    return vmin, xmin


def wta_chunked(Ls, Cf, lo, hi, gmin, DP, ndir=8, refine=1):
    """wta_chunked_kernel of mgm_kernels.cuh, lane by lane: only the chunks of a pixel's span are read."""
    npix = Cf.shape[0]
    disp, conf = np.zeros(npix, F), np.zeros(npix, F)
    lane = np.arange(32)
    for p in range(npix):
        slo, shi = int(lo[p]) - gmin, int(hi[p]) - gmin
        ea, eb = slo >> 5, shi >> 5
        pm = np.full((ndir, 32), INF, F)
        pa = np.full((ndir, 32), -1, np.int64)
        best, bidx = np.full(32, INF, F), np.full(32, 0x7fffffff, np.int64)
        sS = np.full(DP, F(12345.0), F)
        for e in range(ea, eb + 1):
            kk = 32 * e + lane
            s = np.zeros(32, F)
            for d in range(ndir):
                v = Ls[d][p, kk]
                lt, eq = v < pm[d], v == pm[d]
                pa[d] = np.where(lt | eq, kk, pa[d])
                pm[d] = np.where(lt, v, pm[d])
                s = s + v
            with np.errstate(invalid="ignore"):
                s = (np.float64(-(ndir - 1)) * Cf[p, kk].astype(np.float64) + s.astype(np.float64)).astype(F)
            take = np.isfinite(s) & (best > s)
            best, bidx = np.where(take, s, best), np.where(take, kk, bidx)
            sS[kk] = s
        am = []
        for d in range(ndir):
            md = pm[d].min()
            am.append(int(np.where(pm[d] == md, pa[d], -1).max()))
        m = best.min()
        kbest = int(np.where((best == m) & (bidx != 0x7fffffff), bidx, 0x7fffffff).min())
        if kbest > DP - 1:
            kbest = 0
        o = gmin + kbest
        minP = F(o)
        conf[p] = sum(1 for d in range(ndir) if am[d] == kbest)
        if refine and kbest - 1 >= slo and kbest + 2 <= shi:
            v0, v1, v2 = sS[kbest - 1], sS[kbest], sS[kbest + 1]
            ml, dx = vfit3(v0, v1, v2)
            mlr, dxr = vfit3(v2, v1, v0)
            minP = F(o) + dx
            if mlr < ml:
                minP = F(o) - dxr
        disp[p] = minP
    return disp, conf


def main_wta(DP, h, w, tsgm, seed, Ls, Cf, lo, hi, gmin, Wimg=None, P1=8.0, P2=32.0):
    """compare the emulated chunk-skipping WTA (on the emulated pass volumes, garbage outside the spans) with the oracle"""
    import ctypes
    npix = h * w
    C3 = Cf.reshape(h, w, DP)
    So, do, co, fo = O.port.aggregate(C3, lo.reshape(h, w), hi.reshape(h, w), gmin, P1, P2, 8, tsgm, weights=Wimg)
    d_ref, c_ref = do.reshape(-1).copy(), co.reshape(-1).copy()
    lo32, hi32 = np.ascontiguousarray(lo, np.int32), np.ascontiguousarray(hi, np.int32)
    pf = lambda a, t=ctypes.c_float: a.ctypes.data_as(ctypes.POINTER(t))
    O.lib().orc_refine(pf(np.ascontiguousarray(So)), pf(lo32, ctypes.c_int), pf(hi32, ctypes.c_int), npix, gmin, DP, 1, pf(d_ref), pf(c_ref))
    d, cf = wta_chunked(Ls, Cf, lo, hi, gmin, DP)
    print("chunk-skipping WTA: %d disparities and %d confidences of %d differ" % (int((d != d_ref).sum()), int((cf != fo.reshape(-1)).sum()), npix))


if __name__ == "__main__":
    main()
