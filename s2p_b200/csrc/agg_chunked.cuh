// agg_chunked.cuh -- the MGM aggregation for slabs wider than 512 slots, which the register-resident kernel of agg_kernel.cuh
// cannot hold: a level of mgm_multi whose label hull exceeds 512 labels, or `mgm` with more than 512 labels.  It computes only
// the 32-label chunks that hold each pixel's label range, which is what it was first written for: volumes whose pixels use a
// small part of the slab, i.e. the fine levels of mgm_multi.
//
// Why.  update_dmin_dmax gives most pixels of a fine level 17..40 labels but hands the parent's full range to every
// pixel next to a rejected one, so the dense slab spans up to 512 labels while the mean range is ~65
// (scripts/range_width_analysis.py: 666 Mvoxel dense, 135 Mvoxel ragged, 164 Mvoxel for a lock-step band that only
// touches the 32-label chunks its 16 pixels need).  The register-resident kernel of agg_kernel.cuh cannot skip work:
// a lane owns LPL consecutive slots, so a narrow pixel idles most lanes instead of most instructions.
//
// How.  Same band / skew / barrier structure, same global layout, same arithmetic, but
//   * chunk-major mapping: element e of lane l is slot 32*e + l, so a whole 32-label chunk is skipped by a
//     warp-uniform branch; a pixel only computes the chunks [ea, eb] that hold its label range;
//   * one scanline per warp (16 warps per CTA) and the neighbours' vectors live in SHARED memory, read with
//     offsets -1 / 0 / +1 (no shuffles, no register windows); every stored vector carries its chunk span and an
//     +INF guard on both sides of the span, chunks of a neighbour outside its span read as +INF;
//   * the chunks a pixel does not compute are left untouched in the global L volume (the chunk-skipping WTA of
//     mgm_kernels.cuh never reads them; the band hand-off carries the previous band's spans as well).
// The label range of a pixel only enters through its span; slots of an active chunk outside the range hold +INF
// costs and therefore +INF results, exactly as in the dense kernel.
// GEN: the general flavour (float costs, per-pixel weights): f32 costs and the current pixel's weight are staged instead of
// u8 codes, and the penalties are scaled by the weight with the rounding of recurse2 (agg_kernel.cuh).
// Status: scripts/chunked_emulator.py replays this file's indexing on the CPU (ring slots, guards, staging slots,
// range words, previous-band ring) and equals the oracle bit for bit for every TSGM and slab width; it found the
// chunk-edge case of term() below (a neighbour whose span starts right after / ends right before my chunk), which
// the first GPU run showed as 1.5 % differing pixels on the 512-slot level.  The corrected kernel is bit-identical on the
// GPU (tests/test_gpu_parity.py) but not faster than the dense kernel on ragged levels (DESIGN.md section 3.3), so slabs of
// up to 512 slots stay with the dense kernel.
#pragma once
#include "agg_kernel.cuh"

namespace s2pb {

constexpr int kCkWarps = 16;       // scanlines per band = warps per CTA for census slabs of up to 512 slots; wider slabs run
                                   // with fewer warps so that the rings and the staged costs still fit shared memory (ck_warps)
constexpr int kCkThreads = kCkWarps * 32;
constexpr int kCkRing = 4;         // ring slots per scanline (a reader is at most 3 pixels behind the writer)
constexpr int kCkStage = 4;        // cp.async pipeline depth in pixel steps (2 for the slabs wider than 512 slots)
constexpr int kCkPad = 4;          // floats of +INF guard before and after a stored vector (keeps 16-byte alignment)
// slots of the previous band's scanline for a pipeline depth of `stage` (> stage + 1: pixel 0 is staged ahead)
__host__ __device__ constexpr int ck_r0(int stage) { return 2 * stage; }
// warps per CTA (= scanlines per band) and pipeline depth for a slab of DP slots.  GEN stages four times the cost bytes:
// 8 warps at <= 1024 slots take ~215 KB of shared memory, 4 warps at 2048 slots would take ~230 KB, so 2 run there.
__host__ __device__ inline int ck_warps(int DP, bool gen) { return gen ? (DP <= 1024 ? 8 : 2) : DP <= 512 ? 16 : DP <= 1024 ? 8 : 4; }
__host__ __device__ inline int ck_stage(int DP, bool gen) { return (DP <= 512 && !gen) ? 4 : 2; }

struct ChunkedParams {
    AggParams A;
    const short *lo[kMaxPV], *hi[kMaxPV];   // per pass-view: the view's per-pixel label range
    int gmin[kMaxPV];                       // ... and the label of slot 0
    int DP;                                 // slots per pixel (multiple of 32, <= 2048)
};
// the folded layout (FoldView, agg_kernel.cuh): one pass index per launch; bands of ck_warps scanlines index the boundary buffer
struct ChunkedFoldParams : ChunkedParams {
    FoldView fv[kMaxPV];
    int first;
};
template <bool FOLD> using ChunkedArgs = typename std::conditional<FOLD, ChunkedFoldParams, ChunkedParams>::type;

// shared memory carve-up for a run-time DP
struct CkSmem {
    int DP, vstride;                        // vstride = DP + 2 * kCkPad floats per stored vector
    size_t ring_off, meta_off, r0_off, r0m_off, cst_off, rng_off, r0rng_off, wst_off, bytes;
    __host__ __device__ CkSmem(int dp, int warps, int stage, bool gen) : DP(dp), vstride(dp + 2 * kCkPad)
    {
        const int r0n = ck_r0(stage);
        ring_off = 0;                                                               // float [warps][ring][vstride]
        meta_off = ring_off + sizeof(float) * warps * kCkRing * vstride;            // float min, int ea, int eb per slot
        r0_off = meta_off + 12 * warps * kCkRing;                                   // float [r0n][vstride]
        r0m_off = r0_off + sizeof(float) * r0n * vstride;                           // float [r0n]
        cst_off = (r0m_off + sizeof(float) * r0n + 15) / 16 * 16;                   // u8 | float (GEN) [warps][stage][DP] (costs)
        rng_off = cst_off + (gen ? sizeof(float) : sizeof(uint8_t)) * warps * stage * dp;   // 2 words per (warp, stage): lo, hi
        r0rng_off = rng_off + 8 * warps * stage;                                    // 2 words per previous-band slot
        wst_off = r0rng_off + 8 * r0n;                                              // float [warps][stage] (GEN: weights)
        bytes = wst_off + (gen ? sizeof(float) * warps * stage : 0);
    }
};

template <int TSGM, int TYPE, bool SCALED, int STAGE, bool GEN, bool FOLD>
__device__ __forceinline__ void run_band_chunked(const PassDesc &pd, const FoldView &fv, int first, const short *__restrict__ lo_img,
                                                 const short *__restrict__ hi_img, int gmin, int DP, int band, float P1, float P2,
                                                 const float *__restrict__ lut, const int *abort_flag, unsigned char *smem)
{
    constexpr bool useA = (TYPE == 0) ? true : (TSGM == 4);
    constexpr bool useCn = (TYPE == 0) ? (TSGM >= 2) : (TSGM >= 3);
    constexpr bool useB = (TYPE == 0) ? (TSGM >= 3) : (TSGM >= 2);
    constexpr bool useE = (TYPE == 0) ? (TSGM == 4) : true;
    constexpr bool usePrev = useCn || useB || useE;
    constexpr int SKEW = useE ? 2 : 1;
    constexpr int LEAD = useE ? 1 : 0;
    constexpr int kCkStage = STAGE, kCkR0 = ck_r0(STAGE);    // (shadow the defaults: this instantiation's pipeline depth)
    constexpr int S = kCkStage - 1;
    const int kCkWarps = (int)(blockDim.x >> 5);             // scanlines per band
    const CkSmem SM(DP, kCkWarps, STAGE, GEN);
    using CT = typename std::conditional<GEN, float, uint8_t>::type;     // stored cost element
    constexpr int CB = (int)sizeof(CT);
    const int NC = DP >> 5, VS = SM.vstride;
    const int nI = pd.nI;
    const int nsteps = nI + (kCkWarps - 1) * SKEW;
    const int lane = threadIdx.x & 31, k = threadIdx.x >> 5;

    const int s = band * kCkWarps + k;                       // my scanline
    const bool live = s < pd.nS;
    const long long strideI = pd.strideI;
    const bool prev = usePrev && live && s > 0;
    const bool from_r0 = (k == 0);
    const bool publish = live && (k == kCkWarps - 1) && (s + 1 < pd.nS);
    const long long rowbase = pd.base + (long long)s * pd.strideS;

    const unsigned smem_s = (unsigned)__cvta_generic_to_shared(smem);
    float *ring = reinterpret_cast<float *>(smem + SM.ring_off);
    float *meta = reinterpret_cast<float *>(smem + SM.meta_off);
    float *r0 = reinterpret_cast<float *>(smem + SM.r0_off);
    float *r0m = reinterpret_cast<float *>(smem + SM.r0m_off);
    const CT *cst = reinterpret_cast<const CT *>(smem + SM.cst_off) + (size_t)k * kCkStage * DP;
    const float *wst = reinterpret_cast<const float *>(smem + SM.wst_off) + k * kCkStage;      // GEN only
    const bool weighted = GEN && pd.W != nullptr;
    const unsigned *rng = reinterpret_cast<const unsigned *>(smem + SM.rng_off) + k * kCkStage * 2;
    const unsigned *r0rng = reinterpret_cast<const unsigned *>(smem + SM.r0rng_off);
    float *myring = ring + (size_t)k * kCkRing * VS;
    float *mymeta = meta + k * kCkRing * 3;
    const float *srcring = from_r0 ? r0 : ring + (size_t)(k - 1) * kCkRing * VS;
    const float *srcmeta = meta + (k - 1) * kCkRing * 3;     // unused when from_r0
    const int srcmask = from_r0 ? (kCkR0 - 1) : (kCkRing - 1);

    // guards of the previous-band slots: the copies only ever write [kCkPad, kCkPad + DP)
    if (from_r0) {
        for (int q = lane; q < kCkR0 * 2 * kCkPad; q += 32) {
            const int slot = q / (2 * kCkPad), j = q % (2 * kCkPad);
            r0[slot * VS + (j < kCkPad ? j : DP + j)] = S2PB_INF;
        }
    }
    __syncwarp();

    // ---- staging: my scanline's costs and range words; (warp 0) the previous band's vectors and minima
    const char *csrc = reinterpret_cast<const char *>(pd.C) + rowbase * (long long)(DP * CB);
    const long long cstep = strideI * (DP * CB);
    const unsigned cdst = smem_s + (unsigned)SM.cst_off + (unsigned)(k * kCkStage * DP * CB);
    const unsigned rdst = smem_s + (unsigned)SM.rng_off + (unsigned)(k * kCkStage * 8);
    const unsigned wdst = smem_s + (unsigned)SM.wst_off + (unsigned)(k * kCkStage * 4);
    long long pidx = rowbase;                                // pixel index of the pixel to stage next
    int jc = 0;
    // chunk span of the pixels about to be staged: their range words are fetched with plain (L2-resident, warp-uniform)
    // loads two stagings ahead and wait in registers, so that only the chunks of the span are copied
    auto range_words = [&](int j, unsigned &wl, unsigned &wh) {
        wl = wh = 0;
        if (live && j < nI) {
            const long long q = rowbase + (long long)j * strideI;
            wl = __ldg(reinterpret_cast<const unsigned *>(reinterpret_cast<const char *>(lo_img) + ((q * 2) & ~3LL)));
            wh = __ldg(reinterpret_cast<const unsigned *>(reinterpret_cast<const char *>(hi_img) + ((q * 2) & ~3LL)));
        }
    };
    unsigned nl0, nh0, nl1, nh1, nl2, nh2;                    // words of pixels jc, jc + 1, jc + 2
    range_words(0, nl0, nh0); range_words(1, nl1, nh1); range_words(2, nl2, nh2);
    const bool stage_prev = prev && from_r0;
    const long long prevbase = rowbase - pd.strideS;
    // (FOLD: the previous band's closing scanline is stored contiguously in the boundary buffer)
    const char *psrc = FOLD ? reinterpret_cast<const char *>(fv.Lb + (long long)(band > 0 ? band - 1 : 0) * nI * DP)
                            : reinterpret_cast<const char *>(pd.L + prevbase * DP);
    const float *pmsrc = pd.Lmin + prevbase;
    const long long lstepb = (FOLD ? 1 : strideI) * (long long)(DP * 4);
    const unsigned r0_s = smem_s + (unsigned)SM.r0_off, r0m_s = smem_s + (unsigned)SM.r0m_off, r0rng_s = smem_s + (unsigned)SM.r0rng_off;
    long long ppix = prevbase;                               // pixel index of the previous-band pixel to stage next
    const int *prev_progress = (band > 0) ? pd.progress + (band - 1) : nullptr;
    int jp = 0, avail = 0;

    auto stage_mine = [&]() {
        if (live && jc < nI) {
            const unsigned slot = (unsigned)(jc & (kCkStage - 1));
            const int sh = (int)((pidx & 1) * 16);
            const int ea = ((int)(short)((nl0 >> sh) & 0xffff) - gmin) >> 5, eb = ((int)(short)((nh0 >> sh) & 0xffff) - gmin) >> 5;
            for (int c = 2 * CB * ea + lane; c <= 2 * CB * eb + 2 * CB - 1; c += 32)     // a chunk of 32 costs = 2 * CB 16-byte pieces
                cp_async16_s(cdst + slot * (unsigned)(DP * CB) + 16 * c, csrc + 16 * c);
            // the 4-byte words that hold lo[pidx] and hi[pidx] (2-byte elements): the half is picked at use time
            if (lane == 0) cp_async4_s(rdst + slot * 8, reinterpret_cast<const char *>(lo_img) + ((pidx * 2) & ~3LL));
            if (lane == 1) cp_async4_s(rdst + slot * 8 + 4, reinterpret_cast<const char *>(hi_img) + ((pidx * 2) & ~3LL));
            if (weighted && lane == 2) cp_async4_s(wdst + slot * 4, pd.W + pidx);
            csrc += cstep;
            pidx += strideI;
        }
        jc++;
        nl0 = nl1; nh0 = nh1; nl1 = nl2; nh1 = nh2;
        range_words(jc + 2, nl2, nh2);
    };
    auto stage_prevband = [&]() {
        if (stage_prev) {
            if (jp < nI) {
                int spins = 0;
                while (avail < jp + 1) {
                    avail = ld_acquire(prev_progress);
                    if (((++spins) & 1023) == 0 && *(volatile const int *)abort_flag) break;
                }
                const unsigned slot = (unsigned)(jp & (kCkR0 - 1));
                for (int c = lane; c < DP / 4; c += 32) cp_async16_s(r0_s + (slot * VS + kCkPad) * 4 + 16 * c, psrc + 16 * c);
                if (lane == 0) cp_async4_s(r0m_s + slot * 4, pmsrc);
                if (lane == 1) cp_async4_s(r0rng_s + slot * 8, reinterpret_cast<const char *>(lo_img) + ((ppix * 2) & ~3LL));
                if (lane == 2) cp_async4_s(r0rng_s + slot * 8 + 4, reinterpret_cast<const char *>(hi_img) + ((ppix * 2) & ~3LL));
                psrc += lstepb;
                pmsrc += strideI;
                ppix += strideI;
            }
            jp++;
        }
    };

    float *out = (FOLD ? fv.S : pd.L) + rowbase * DP;        // FOLD: the running sum S instead of L_p
    float *lmin_out = pd.Lmin + rowbase;
    float *lb_out = FOLD ? fv.Lb + (long long)band * nI * DP : nullptr;    // FOLD: the band-closing scanline's vectors
    short *am_out = FOLD ? fv.am + rowbase : nullptr;
    long long upix = rowbase;                                // pixel index of the pixel computed next (for the range halves)

    // one neighbour's contribution for slot kk of chunk e: update_costW, mgm_core.cc:92-121
    struct Nb { const float *v; float m; int ea, eb; };
    auto nb_at = [&](int j, bool mine) {
        Nb n;
        if (mine) {                     // my own previous pixel
            const int slot = j & (kCkRing - 1);
            n.v = myring + slot * VS + kCkPad;
            n.m = mymeta[slot * 3]; n.ea = __float_as_int(mymeta[slot * 3 + 1]); n.eb = __float_as_int(mymeta[slot * 3 + 2]);
        } else if (from_r0) {           // previous band: the whole vector was copied, only its span is meaningful
            const int slot = j & srcmask;
            float *v = r0 + slot * VS + kCkPad;
            const long long qpix = prevbase + (long long)j * strideI;
            const int sh = (int)((qpix & 1) * 16);
            const int qlo = (int)(short)((r0rng[slot * 2] >> sh) & 0xffff), qhi = (int)(short)((r0rng[slot * 2 + 1] >> sh) & 0xffff);
            n.ea = (qlo - gmin) >> 5; n.eb = (qhi - gmin) >> 5;
            if (lane == 0) { v[32 * n.ea - 1] = S2PB_INF; v[32 * (n.eb + 1)] = S2PB_INF; }     // guards (the copy brought whatever the chunks next to the span hold)
            __syncwarp();
            n.v = v;
            n.m = r0m[slot];
        } else {
            const int slot = j & srcmask;
            n.v = srcring + slot * VS + kCkPad;
            n.m = srcmeta[slot * 3]; n.ea = __float_as_int(srcmeta[slot * 3 + 1]); n.eb = __float_as_int(srcmeta[slot * 3 + 2]);
        }
        return n;
    };
    // GEN: the penalties scaled by the current pixel's weight wv as recurse2 rounds them: P2*w + m is an fma, P1*w + x is
    // an fma for the 3rd / 4th neighbour of the reference's list (ord 2, 3) and mul then add (P1w) for the 1st / 2nd
    float wv = 1.f, P1w = P1;
    auto term = [&](const Nb &n, int e, int kk, auto ord_c) {
        float a = S2PB_INF, b = S2PB_INF, c0 = S2PB_INF;
        if (e >= n.ea && e <= n.eb) { a = n.v[kk - 1]; c0 = n.v[kk]; b = n.v[kk + 1]; }      // the guards make the span edges +INF
        else if (e == n.ea - 1) { if (lane == 31) b = n.v[kk + 1]; }     // my last slot's right neighbour is the first slot of its span
        else if (e == n.eb + 1) { if (lane == 0) a = n.v[kk - 1]; }      // my first slot's left neighbour is the last slot of its span
        if constexpr (GEN) {
            const float v1 = (decltype(ord_c)::value >= 2) ? __fmaf_rn(P1, wv, fminf(a, b)) : __fadd_rn(fminf(a, b), P1w);
            return fmin3f(c0, v1, __fmaf_rn(P2, wv, n.m)) - n.m;
        } else {
            const float v1 = fminf(a, b) + P1;
            return fmin3f(c0, v1, n.m + P2) - n.m;
        }
    };
    using o0 = std::integral_constant<int, 0>; using o1 = std::integral_constant<int, 1>;
    using o2 = std::integral_constant<int, 2>; using o3 = std::integral_constant<int, 3>;

    // prologue: S groups in flight
    if (LEAD == 1) stage_prevband();
    for (int g = 0; g < S; g++) { stage_mine(); stage_prevband(); cp_async_commit(); }

    for (int t = 0; t < nsteps; t++) {
        const int i = t - k * SKEW;
        const bool act = live && i >= 0 && i < nI;
        if (i >= 0) { stage_mine(); stage_prevband(); }
        cp_async_commit();
        if (act) {
            cp_async_wait<S>();
            __syncwarp();
            const int slot = i & (kCkStage - 1);
            const unsigned wl = rng[slot * 2], wh = rng[slot * 2 + 1];
            const int sh = (int)((upix & 1) * 16);
            const int plo = (int)(short)((wl >> sh) & 0xffff), phi = (int)(short)((wh >> sh) & 0xffff);
            const int ea = (plo - gmin) >> 5, eb = (phi - gmin) >> 5;          // my chunk span
            const bool border = (s == 0) || (i == 0) || (i == nI - 1);
            Nb nA, nB, nC, nE;
            if (!border) {
                nA = nb_at(i - 1, true);
                if (useB) nB = nb_at(i - 1, false);
                if (useCn) nC = nb_at(i, false);
                if (useE) nE = nb_at(i + 1, false);
            }
            const CT *cp = cst + (size_t)slot * DP;
            float *mine = myring + (i & (kCkRing - 1)) * VS + kCkPad;
            float lm = S2PB_INF;
            int la = -1;                                     // FOLD: my last slot attaining lm
            if (weighted) { wv = wst[slot]; P1w = __fmul_rn(P1, wv); }
            for (int e = 0; e < NC; e++) {
                const int kk = 32 * e + lane;
                float L = S2PB_INF;
                if (e >= ea && e <= eb) {
                    const float sv = (FOLD && !first) ? __ldcg(out + kk) : 0.f;     // FOLD: S so far (0 before pass 0)
                    float c;
                    if constexpr (GEN) c = cp[kk];
                    else {
                        c = cost_decode(cp[kk]);
                        if (SCALED) { if (c >= 0.f && c < (float)kCostLut) c = lut[(int)c]; }
                    }
                    L = c;
                    if (!border) {
                        float acc;
                        // the neighbours in the order of the reference's list: type 0 = A, Cn, B, E ; type 1 = E, B, Cn, A
                        if constexpr (TYPE == 0) {
                            acc = term(nA, e, kk, o0{});
                            if (TSGM == 2) acc *= 0.5f;
                            if (useCn) { float tt = term(nC, e, kk, o1{}); acc += (TSGM == 2) ? tt * 0.5f : tt; }
                            if (useB) acc += term(nB, e, kk, o2{});
                            if (useE) acc += term(nE, e, kk, o3{});
                        } else {
                            acc = term(nE, e, kk, o0{});
                            if (TSGM == 2) acc *= 0.5f;
                            if (useB) { float tt = term(nB, e, kk, o1{}); acc += (TSGM == 2) ? tt * 0.5f : tt; }
                            if (useCn) acc += term(nC, e, kk, o2{});
                            if (useA) acc += term(nA, e, kk, o3{});
                        }
                        if constexpr (TSGM == 3) acc = div3_exact(acc);
                        if constexpr (TSGM == 4) acc = acc * 0.25f;
                        L = c + acc;
                    }
                    mine[kk] = L;
                    if constexpr (FOLD) {
                        // S + L_p in pass order, as the WTA adds; the arg-minimum rule of the chunked WTA (wta_chunked_kernel)
                        if (L <= lm) la = kk;
                        lm = fminf(lm, L);
                        out[kk] = __fadd_rn(sv, L);
                        if (publish) lb_out[kk] = L;
                    } else {
                        lm = fminf(lm, L);
                        out[kk] = L;
                    }
                }
            }
            const float m = warp_min_f32(lm);
            if constexpr (FOLD) {
                const int a = __reduce_max_sync(0xffffffffu, lm == m ? la : -1);
                if (lane == 0) *am_out = (short)a;
                am_out += strideI;
                lb_out += DP;
            }
            if (lane == 0) {
                mine[32 * ea - 1] = S2PB_INF;                  // guards on both sides of the span
                mine[32 * (eb + 1)] = S2PB_INF;
                float *mt = mymeta + (i & (kCkRing - 1)) * 3;
                mt[0] = m; mt[1] = __int_as_float(ea); mt[2] = __int_as_float(eb);
                if (publish) *lmin_out = m;
            }
            out += strideI * DP;
            lmin_out += strideI;
            upix += strideI;
            if (publish && (((i + 1) % kPublish) == 0 || i == nI - 1)) {
                __syncwarp();
                if (lane == 0) st_release(pd.progress + band, i + 1);
            }
        }
        __syncthreads();
    }
    cp_async_wait<0>();
}

// FOLD: the folded layout (ChunkedFoldParams), as in aggregate_kernel
template <int TSGM, bool SCALED, int STAGE, bool GEN, bool FOLD = false>
__global__ void __launch_bounds__(kCkThreads) aggregate_chunked_kernel(const __grid_constant__ ChunkedArgs<FOLD> P)
{
    extern __shared__ __align__(16) unsigned char smem[];
    __shared__ int s_item;
    const int kCkWarps = (int)(blockDim.x >> 5);
    // bands of kCkWarps scanlines here (the dense kernel's bands hold kNW): recompute the counts
    int maxBands = 0;
    for (int v = 0; v < P.A.nPV; v++) { const int nb = (P.A.pv[v].nS + kCkWarps - 1) / kCkWarps; if (nb > maxBands) maxBands = nb; }
    const int total = maxBands * P.A.nPV;
    for (;;) {
        if (threadIdx.x == 0) s_item = atomicAdd(P.A.next_item, 1);
        __syncthreads();
        const int item = s_item;
        __syncthreads();
        if (item >= total) return;
        const int band = item / P.A.nPV, pvi = item - band * P.A.nPV;
        const PassDesc &pd = P.A.pv[pvi];
        if (band >= (pd.nS + kCkWarps - 1) / kCkWarps) continue;
        FoldView fv{};
        int first = 0;
        if constexpr (FOLD) { fv = P.fv[pvi]; first = P.first; }
        if (pd.type == 0) run_band_chunked<TSGM, 0, SCALED, STAGE, GEN, FOLD>(pd, fv, first, P.lo[pvi], P.hi[pvi], P.gmin[pvi], P.DP, band, P.A.P1, P.A.P2, P.A.lut, P.A.abort_flag, smem);
        else run_band_chunked<TSGM, 1, SCALED, STAGE, GEN, FOLD>(pd, fv, first, P.lo[pvi], P.hi[pvi], P.gmin[pvi], P.DP, band, P.A.P1, P.A.P2, P.A.lut, P.A.abort_flag, smem);
    }
}

}  // namespace s2pb
