// mgm_kernels.cuh -- census, cost volume, WTA / sub-pixel and image-space post-filter kernels.
// Layout, reference citations and numerical conventions: see the header of agg_kernel.cuh.
#pragma once
#include "agg_kernel.cuh"

namespace s2pb {

// ------------------------------------------------------------------ census

// census_tools.cc:38-57: neighbours in row-major window order, centre skipped,
// bit = (centre < neighbour), out-of-image neighbour compares as NaN -> 0.
// NW = census_words(win): 2 for the codes of more than 64 bits (sides 9 and 11), shifted through the pair (codes_hi : codes);
// the Hamming distance does not depend on where a bit sits as long as both codes put it in the same place.
template <int NW>
__global__ void census_kernel(const float *__restrict__ img, int w, int h, int r, uint64_t *__restrict__ codes, uint64_t *__restrict__ codes_hi)
{
    int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    float c = img[(size_t)y * w + x];
    uint64_t code = 0, hi = 0;
    for (int j = -r; j <= r; j++)
        for (int i = -r; i <= r; i++) {
            if (i == 0 && j == 0) continue;
            int xx = x + i, yy = y + j;
            unsigned bit = 0;
            if (xx >= 0 && xx < w && yy >= 0 && yy < h) bit = c < img[(size_t)yy * w + xx];
            if constexpr (NW == 2) census_push(code, hi, bit);
            else code = (code << 1) | bit;
        }
    codes[(size_t)y * w + x] = code;
    if constexpr (NW == 2) codes_hi[(size_t)y * w + x] = hi;
}

// main_mgm.cc:172-173,178,207,210-216: NaN -> 0 and the per-pixel label range of one view.
// `sentinel` is the reference's dmin (sic, for BOTH views) used for no-data pixels.
__global__ void prepare_view_kernel(const float *__restrict__ in, int n, int lo_all, int hi_all, int sentinel,
                                    float *__restrict__ clean, short *__restrict__ lo, short *__restrict__ hi)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float v = in[i];
    bool isn = isnan(v);
    clean[i] = isfinite(v) ? v : 0.f;
    lo[i] = (short)(isn ? sentinel : lo_all);
    hi[i] = (short)(isn ? sentinel + 1 : hi_all);
}

// does the image hold a NaN?  (a no-data pixel of the secondary image widens the right view's label hull: mgm_enqueue in
// s2pb200.cu)
__global__ void has_nan_kernel(const float *__restrict__ in, int n, int *flag)
{
    bool f = false;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) f |= isnan(in[i]);
    if (__any_sync(0xffffffffu, f) && (threadIdx.x & 31) == 0) *(volatile int *)flag = 1;
}

// ------------------------------------------------------------------ cost volume

// One warp per pixel.  mgm_costvolume.cc:140-172: label o of pixel (x,y) compares census
// codes cu(x,y) and cv(x+o,y); +INF when x+o is outside; if no label of the pixel's range is
// finite, the whole range is set to 0.  Slots outside [lo,hi] stay +INF.
// With ZOOMFACTOR = 2 (mgm_costvolume.cc:145-154) label o compares cu(x) with the census of the matched image
// shifted by (o mod 2)/2 pixel, at column x + floor(o/2): cv = shift 0, cv1 = shift 1/2.
// BITS, the width of the census codes: 32 when they fit the low words (3x3 and 5x5 windows: 8 and 24 bits), so one POPC on
// those does it; 64 (7x7: 48 bits); 128 (9x9 and 11x11: 80 and 120 bits), the second words in cuh / cvh / cv1h.
// The Hamming distance is stored as its 8-bit code (agg_kernel.cuh), four labels per 32-bit word, with no conversion
// instruction on the quarter-rate pipe that POPC uses.
template <int LPL, bool ZOOM2, int BITS>
__global__ void cost_kernel(const uint64_t *__restrict__ cu, const uint64_t *__restrict__ cv, const uint64_t *__restrict__ cv1,
                            int w, int h,
                            const short *__restrict__ lo, const short *__restrict__ hi, int gmin, uint8_t *__restrict__ C,
                            const uint64_t *__restrict__ cuh, const uint64_t *__restrict__ cvh, const uint64_t *__restrict__ cv1h)
{
    constexpr int DP = 32 * LPL;
    int lane = threadIdx.x & 31;
    size_t npix = (size_t)w * h;
    size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
    for (size_t p = warp; p < npix; p += nwarps) {
        int x = (int)(p % w);
        size_t row = p - x;
        const uint64_t a = cu[p], ah = BITS == 128 ? cuh[p] : 0;
        const int l = lo[p], hgh = hi[p];
        unsigned cnt[LPL];                   // Hamming distance where the label has one, else 0
        unsigned okm = 0, inm = 0;           // bit e: label e has a distance / lies in the pixel's range
#pragma unroll
        for (int e = 0; e < LPL; e++) {
            const int o = gmin + lane * LPL + e;
            cnt[e] = 0;
            if (o >= l && o <= hgh) {
                inm |= 1u << e;
                int q = x + o;
                const uint64_t *codes = cv, *codes_hi = cvh;
                if (ZOOM2) { q = x + (o >> 1); if (o & 1) { codes = cv1; codes_hi = cv1h; } }     // floor(o/2), goodmod(o,2)
                if (q >= 0 && q < w) {
                    if constexpr (BITS == 32) cnt[e] = __popc((unsigned)a ^ reinterpret_cast<const unsigned *>(codes)[2 * (row + q)]);
                    else cnt[e] = __popcll(a ^ codes[row + q]);
                    if constexpr (BITS == 128) cnt[e] += __popcll(ah ^ codes_hi[row + q]);
                    okm |= 1u << e;
                }
            }
        }
        // no label of the range has a distance: the whole range is 0 (mgm_costvolume.cc:166-171); cnt is 0 there already
        const unsigned fin = __any_sync(0xffffffffu, okm != 0) ? okm : inm;
        st_cost<LPL>(C + p * DP + lane * LPL, cost_pack<LPL>(cnt, fin));     // 4 codes per 32-bit word
    }
}

// The same volume for 32-bit census codes (3x3 / 5x5 windows) at full-pixel labels, one warp per strip of 32 consecutive pixels
// of a row.  cost_kernel reads every code through its own 8-byte load at a lane stride of 8*LPL bytes: LPL loads of 8 L1
// wavefronts each per pixel, and that -- not POPC, not issue -- is its bound (0.225 ms per C2 view whatever the arithmetic).  Here
// the strip's 32 + DP matched-image codes are staged once in shared memory, in four copies shifted by 0..3 words, so that pixel i
// reads its lane's LPL consecutive codes from copy i & 3 with aligned 16- / 8-byte loads (4 wavefronts for 512 bytes); the
// pixel's own code and range come from registers of lane i by shuffle.  The range test is against warp-uniform bounds clamped
// to the image, which also answers "does any label of the range have a distance" without a vote.  Same values as cost_kernel.
constexpr int kCostStripThreads = 128;
template <int LPL>
__global__ void __launch_bounds__(kCostStripThreads) cost_strip_kernel(const uint64_t *__restrict__ cu, const uint64_t *__restrict__ cv, int w, int h,
                                                                       const short *__restrict__ lo, const short *__restrict__ hi, int gmin,
                                                                       uint8_t *__restrict__ C)
{
    constexpr int DP = 32 * LPL, T = 32, NW = T + DP, CS = NW + 4;
    __shared__ __align__(16) unsigned codes[kCostStripThreads / 32][4][CS];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int spr = (w + T - 1) / T, total = h * spr;
    const int gw = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), nw = (int)((gridDim.x * blockDim.x) >> 5);
    unsigned (*mine)[CS] = codes[wib];
    for (int strip = gw; strip < total; strip += nw) {
        const int y = strip / spr, x0 = (strip - y * spr) * T;
        const size_t row = (size_t)y * w;
        __syncwarp();                                         // the previous strip's reads are done
        for (int j = lane; j < NW; j += 32) {
            const int q = x0 + gmin + j;
            const unsigned c = (q >= 0 && q < w) ? reinterpret_cast<const unsigned *>(cv)[2 * (row + q)] : 0u;
#pragma unroll
            for (int sft = 0; sft < 4; sft++)
                if (j - sft >= 0) mine[sft][j - sft] = c;     // copy sft: word k = code k + sft
        }
        const int xi = x0 + lane;
        unsigned a_i = 0;
        int l_i = 0, h_i = -1;
        if (xi < w) { a_i = reinterpret_cast<const unsigned *>(cu)[2 * (row + xi)]; l_i = lo[row + xi]; h_i = hi[row + xi]; }
        __syncwarp();
        const int npx = (w - x0 < T) ? w - x0 : T;
        uint8_t *dst = C + (row + x0) * DP + lane * LPL;
        for (int i = 0; i < npx; i++, dst += DP) {
            const unsigned a = __shfl_sync(0xffffffffu, a_i, i);
            const int l = __shfl_sync(0xffffffffu, l_i, i), hgh = __shfl_sync(0xffffffffu, h_i, i);
            const int x = x0 + i;
            int flo = l > -x ? l : -x, fhi = hgh < w - 1 - x ? hgh : w - 1 - x;       // labels of the range whose column is in the image
            const bool none = flo > fhi;                       // no such label: the whole range is 0 (mgm_costvolume.cc:166-171)
            if (none) { flo = l; fhi = hgh; }
            const unsigned *src = &mine[i & 3][(i & ~3) + lane * LPL];
            unsigned cw[LPL];
            if constexpr (LPL % 4 == 0) {
#pragma unroll
                for (int q = 0; q < LPL / 4; q++) {
                    const uint4 t = reinterpret_cast<const uint4 *>(src)[q];
                    cw[4 * q] = t.x; cw[4 * q + 1] = t.y; cw[4 * q + 2] = t.z; cw[4 * q + 3] = t.w;
                }
            } else if constexpr (LPL % 2 == 0) {
#pragma unroll
                for (int q = 0; q < LPL / 2; q++) {
                    const uint2 t = reinterpret_cast<const uint2 *>(src)[q];
                    cw[2 * q] = t.x; cw[2 * q + 1] = t.y;
                }
            } else {
#pragma unroll
                for (int e = 0; e < LPL; e++) cw[e] = src[e];
            }
            unsigned cnt[LPL], fin = 0;
#pragma unroll
            for (int e = 0; e < LPL; e++) {
                const int o = gmin + lane * LPL + e;
                cnt[e] = none ? 0u : (unsigned)__popc(a ^ cw[e]);
                if (o >= flo && o <= fhi) fin |= 1u << e;
            }
            st_cost<LPL>(dst, cost_pack<LPL>(cnt, fin));
        }
    }
}

// ------------------------------------------------------------------ general cost volume (float32)

// The other distances of the reference's table (mgm_costvolume.h:25-57,96-180) on one channel, plus census through
// the scaling table, written as a float32 slab for the general aggregation flavour.  Arithmetic follows the
// reference build operation by operation (fmas where gcc contracts them; the NCC quotient in double): the
// restatement in oracle/mgm_oracle.c is pinned bit for bit against the reference binary for every distance.
enum { kCostCensus = 0, kCostAD, kCostSD, kCostNCC, kCostBTAD, kCostBTSD };
struct CostGenParams {
    const float *u, *v0, *v1;          // this view's image; matched image; matched image shifted by 1/2 px (ZOOMFACTOR 2)
    const uint64_t *cu, *cv0, *cv1;    // census codes of the same three (cost == census)
    const float *lut;                  // census: popcount -> cost (mgm_costvolume.h:90-91)
    const float2 *su, *sv0, *sv1;      // ncc: per-pixel window (mean, variance) of the same three images (ncc_stats_kernel)
    const short *lo, *hi;
    int w, h, gmin, cost, win, zoom;
    float *C;
    const uint64_t *cuh, *cv0h, *cv1h; // the second words of the census codes of more than 64 bits (census_words(win) = 2), else null
};

__device__ __forceinline__ float bt_cost(const float *__restrict__ u, const float *__restrict__ v, int w, size_t row, int x, int qx)
{   // BTAD, mgm_costvolume.h:96-124
    const float IL = u[row + x];
    float ILp = IL, ILm = IL;
    if (x < w - 1) ILp = (IL + u[row + x + 1]) * 0.5f;       // "/2.0" in double then back to float: exact halving
    if (x >= 1) ILm = (IL + u[row + x - 1]) * 0.5f;
    const float IR = v[row + qx];
    float IRp = IR, IRm = IR;
    if (qx < w - 1) IRp = (IR + v[row + qx + 1]) * 0.5f;
    if (qx >= 1) IRm = (IR + v[row + qx - 1]) * 0.5f;
    const float IminR = fminf(IRm, fminf(IRp, IR)), ImaxR = fmaxf(IRm, fmaxf(IRp, IR));
    const float IminL = fminf(ILm, fminf(ILp, IL)), ImaxL = fmaxf(ILm, fmaxf(ILp, IL));
    const float dLR = fmaxf(0.f, fmaxf(IL - ImaxR, IminR - IL));
    const float dRL = fmaxf(0.f, fmaxf(IR - ImaxL, IminL - IR));
    return fabsf(fminf(dLR, dRL));
}
// computeC_clippedNCC, mgm_costvolume.h:152-180.  The window sums of one image (mu = sum v / n, s = sum v*v / n,
// accumulated x-major with the reference build's fmas) depend on the pixel only, not on the label: they are computed
// once per image by ncc_stats_kernel as (mu, s - mu*mu); the cost kernel is left with the cross term.
__global__ void ncc_stats_kernel(const float *__restrict__ img, int w, int h, int hw, float2 *__restrict__ st)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    float2 r = make_float2(0.f, 0.f);
    if (x - hw >= 0 && x + hw < w && y - hw >= 0 && y + hw < h) {      // else: never read (the cost is +INF)
        float mu = 0.f, s = 0.f;
        for (int i = -hw; i <= hw; i++)
            for (int j = -hw; j <= hw; j++) {
                const float v = img[(size_t)(y + j) * w + x + i];
                mu += v;
                s = fmaf(v, v, s);
            }
        const float n = (float)((2 * hw + 1) * (2 * hw + 1));
        mu = __fdiv_rn(mu, n);
        s = __fdiv_rn(s, n);
        r = make_float2(mu, fmaf(-mu, mu, s));
    }
    st[(size_t)y * w + x] = r;
}
__device__ __forceinline__ float ncc_finish(float prod, float n, float2 a, float2 b)
{
    prod = __fdiv_rn(prod, n);
    const float num = fmaf(-a.x, b.x, prod);
    const float den = a.y * b.y;
    const double dd = (0.0000001 > (double)den) ? 0.0000001 : (double)den;
    const float ncc = (float)((double)num / sqrt(dd));
    float cl = (ncc < 1.f) ? ncc : 1.f;
    cl = (0.f > cl) ? 0.f : cl;
    return (1.f - cl) * 64.f;
}

// The costs of LPL labels of one pixel for one lane, label o0 + e in element e: +INF outside [l, hgh] or where the matched
// column (or an NCC tap) leaves the image.  -> whether one of them is finite (the caller applies the all-invalid rule).
template <int LPL>
__device__ __forceinline__ bool cost_gen_labels(const CostGenParams &P, size_t p, int x, int y, int l, int hgh, int o0, float (&c)[LPL])
{
    const int w = P.w, hw = P.win / 2;
    const size_t row = p - x;
    bool anyfinite = false;
    if (P.cost == kCostNCC) {
        // cross term of every label of this lane at once: the taps run in the reference's order (x-major) for each
        // label, the reference image's tap is loaded once per tap instead of once per tap and label
        int q[LPL];
        const float *vq[LPL];
        bool ok[LPL];
        const bool pin = x - hw >= 0 && x + hw < w && y - hw >= 0 && y + hw < P.h;
#pragma unroll
        for (int e = 0; e < LPL; e++) {
            const int o = o0 + e;
            q[e] = x + o;
            bool half = false;
            if (P.zoom == 2) { q[e] = x + (o >> 1); half = (o & 1) != 0; }
            vq[e] = half ? P.v1 : P.v0;
            c[e] = S2PB_INF;
            const bool inrange = o >= l && o <= hgh && q[e] >= 0 && q[e] < w;          // else the slot stays +INF
            ok[e] = inrange && pin && q[e] - hw >= 0 && q[e] + hw < w;                  // else a tap is outside: +INF
            if (ok[e]) c[e] = 0.f;
        }
        for (int i = -hw; i <= hw; i++)
            for (int j = -hw; j <= hw; j++) {
                const size_t r = (size_t)(y + j) * w;
                const float ut = pin ? P.u[r + x + i] : 0.f;
#pragma unroll
                for (int e = 0; e < LPL; e++)
                    if (ok[e]) c[e] = fmaf(ut, vq[e][r + q[e] + i], c[e]);
            }
        const float n = (float)((2 * hw + 1) * (2 * hw + 1));        // the taps (mgm_costvolume.h:152-180)
        const float2 sa = pin ? P.su[p] : make_float2(0.f, 0.f);
#pragma unroll
        for (int e = 0; e < LPL; e++)
            if (ok[e]) {
                const float2 sb = (vq[e] == P.v1 ? P.sv1 : P.sv0)[row + q[e]];
                c[e] = ncc_finish(c[e], n, sa, sb);
                if (isfinite(c[e])) anyfinite = true;
            }
    } else
#pragma unroll
    for (int e = 0; e < LPL; e++) {
        const int o = o0 + e;
        float val = S2PB_INF;
        if (o >= l && o <= hgh) {
            int q = x + o;
            bool half = false;
            if (P.zoom == 2) { q = x + (o >> 1); half = (o & 1) != 0; }       // floor(o/2), goodmod(o,2)
            if (q >= 0 && q < w) {
                if (P.cost == kCostCensus) {
                    const uint64_t *codes = half ? P.cv1 : P.cv0;
                    int r = __popcll(P.cu[p] ^ codes[row + q]);
                    if (P.cuh) r += __popcll(P.cuh[p] ^ (half ? P.cv1h : P.cv0h)[row + q]);
                    val = P.lut[r];
                } else {
                    const float *v = half ? P.v1 : P.v0;
                    if (P.cost == kCostBTAD || P.cost == kCostBTSD) {
                        const float b = bt_cost(P.u, v, w, row, x, q);
                        val = (P.cost == kCostBTAD) ? b : b * b;
                    } else {
                        float d = P.u[p] - v[row + q];
                        d = (d > -d) ? d : -d;
                        val = (P.cost == kCostAD) ? d : d * d;
                    }
                }
                if (isfinite(val)) anyfinite = true;
            }
        }
        c[e] = val;
    }
    return anyfinite;
}

// one warp per pixel, lanes over labels (slot k <-> label gmin + k), like cost_kernel
template <int LPL>
__global__ void cost_gen_kernel(const CostGenParams P)
{
    constexpr int DP = 32 * LPL;
    const int lane = threadIdx.x & 31, w = P.w;
    const size_t npix = (size_t)w * P.h;
    size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
    for (size_t p = warp; p < npix; p += nwarps) {
        const int x = (int)(p % w), y = (int)(p / w);
        const int l = P.lo[p], hgh = P.hi[p];
        float c[LPL];
        const bool anyfinite = cost_gen_labels<LPL>(P, p, x, y, l, hgh, P.gmin + lane * LPL, c);
        if (!__any_sync(0xffffffffu, anyfinite)) {        // mgm_costvolume.cc:166-171
#pragma unroll
            for (int e = 0; e < LPL; e++) {
                const int o = P.gmin + lane * LPL + e;
                if (o >= l && o <= hgh) c[e] = 0.f;
            }
        }
        st_vec<LPL>(P.C + p * DP + lane * LPL, c);
    }
}
// float slab <-> dense float volume (stage-level API)
__global__ void pad_cost_kernel(const float *__restrict__ Cin, size_t npix, int D, int DP, float *__restrict__ C)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npix * DP) return;
    size_t p = i / DP; int k = (int)(i % DP);
    C[i] = k < D ? Cin[p * D + k] : S2PB_INF;
}
__global__ void unpad_cost_kernel(const float *__restrict__ C, size_t npix, int D, int DP, float *__restrict__ Cout)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npix * D) return;
    size_t p = i / D; int k = (int)(i % D);
    Cout[i] = C[p * DP + k];
}

// Companion of agg_chunked.cuh (slabs wider than 512 slots): the census cost volume written only on the 32-slot
// chunks [ea, eb] that hold a pixel's label range (slot 32*e + lane); the chunk-skipping aggregation and WTA never
// read the others.  Same values as cost_kernel on those chunks, including +INF on the slots of an active chunk that
// lie outside the range and the all-invalid -> 0 rule (mgm_costvolume.cc:166-171).
// BITS: 64, or 128 with the codes' second words in cuh / cvh / cv1h (as cost_kernel).
template <bool ZOOM2, int BITS>
__global__ void cost_chunked_kernel(const uint64_t *__restrict__ cu, const uint64_t *__restrict__ cv, const uint64_t *__restrict__ cv1,
                                    int w, int h, const short *__restrict__ lo, const short *__restrict__ hi, int gmin, int DP,
                                    uint8_t *__restrict__ C, const uint64_t *__restrict__ cuh, const uint64_t *__restrict__ cvh,
                                    const uint64_t *__restrict__ cv1h)
{
    const int lane = threadIdx.x & 31;
    const size_t npix = (size_t)w * h;
    size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
    for (size_t p = warp; p < npix; p += nwarps) {
        const int x = (int)(p % w);
        const size_t row = p - x;
        const uint64_t a = cu[p], ah = BITS == 128 ? cuh[p] : 0;
        const int l = lo[p], hgh = hi[p];
        const int ea = (l - gmin) >> 5, eb = (hgh - gmin) >> 5;
        uint8_t *dst = C + p * DP;
        bool anyfinite = false;
        for (int e = ea; e <= eb; e++) {
            const int o = gmin + 32 * e + lane;
            unsigned cnt = 0;
            bool ok = false;
            if (o >= l && o <= hgh) {
                int q = x + o;
                const uint64_t *codes = cv, *codes_hi = cvh;
                if (ZOOM2) { q = x + (o >> 1); if (o & 1) { codes = cv1; codes_hi = cv1h; } }
                if (q >= 0 && q < w) {
                    cnt = __popcll(a ^ codes[row + q]);
                    if constexpr (BITS == 128) cnt += __popcll(ah ^ codes_hi[row + q]);
                    ok = anyfinite = true;
                }
            }
            dst[32 * e + lane] = (uint8_t)cost_encode(cnt, ok);
        }
        if (!__any_sync(0xffffffffu, anyfinite)) {
            for (int e = ea; e <= eb; e++) {
                const int o = gmin + 32 * e + lane;
                if (o >= l && o <= hgh) dst[32 * e + lane] = (uint8_t)cost_encode(0, true);
            }
        }
    }
}

// The same for the general flavour: cost_gen_kernel's float costs, written only on the chunks [ea, eb] of each pixel's span
// (slot 32*e + lane), +INF on the slots of an active chunk outside the range; the other chunks are left untouched.
__global__ void cost_gen_chunked_kernel(const CostGenParams P, int DP)
{
    const int lane = threadIdx.x & 31, w = P.w;
    const size_t npix = (size_t)w * P.h;
    size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
    for (size_t p = warp; p < npix; p += nwarps) {
        const int x = (int)(p % w), y = (int)(p / w);
        const int l = P.lo[p], hgh = P.hi[p];
        const int ea = (l - P.gmin) >> 5, eb = (hgh - P.gmin) >> 5;
        float *dst = P.C + p * DP;
        bool anyfinite = false;
        for (int e = ea; e <= eb; e++) {
            float c[1];
            if (cost_gen_labels<1>(P, p, x, y, l, hgh, P.gmin + 32 * e + lane, c)) anyfinite = true;
            dst[32 * e + lane] = c[0];
        }
        if (!__any_sync(0xffffffffu, anyfinite)) {        // mgm_costvolume.cc:166-171
            for (int e = ea; e <= eb; e++) {
                const int o = P.gmin + 32 * e + lane;
                if (o >= l && o <= hgh) dst[32 * e + lane] = 0.f;
            }
        }
    }
}

// float volume (stage-level API; integer costs in [0, kCostMaxCode] or +INF) -> code slab with +INF padding, and back
__global__ void pack_cost_kernel(const float *__restrict__ Cin, size_t npix, int D, int DP, uint8_t *__restrict__ C)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npix * DP) return;
    size_t p = i / DP; int k = (int)(i % DP);
    C[i] = cost_encode_f(k < D ? Cin[p * D + k] : S2PB_INF);
}
__global__ void unpack_cost_kernel(const uint8_t *__restrict__ C, size_t npix, int D, int DP, const float *__restrict__ lut,
                                   float *__restrict__ Cout)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npix * D) return;
    size_t p = i / D; int k = (int)(i % D);
    Cout[i] = cost_value(C[p * DP + k], lut);
}

// ------------------------------------------------------------------ WTA + consensus + sub-pixel

struct WtaParams {
    const float *L[kMaxPasses];
    const void *C;            // u8 code slab, or float slab for the general flavour (GEN)
    const short *lo, *hi;     // per-pixel label range (labels, not slots)
    const float *lut;
    int ndir, gmin, fix_overcount, refine;
    float inv_zoom_div;       // ZOOMFACTOR (disparity is divided by it, mgm_multiscale.cc:253)
    size_t npix;
    float *S;                 // optional [npix][D] dense output (stage API / PKR), D = Dout
    int Dout;
    float *disp, *cost, *conf;
    float *pkr;               // optional: peak-ratio confidence (compute_PKR_confidence, mgm_costvolume.cc:199-214)
};

// PKR of one pixel from its lane-distributed S: second minimum over the slots of the pixel's range more than 2 away from the
// winner, divided by max(first minimum, 0.01) in double like the reference's `secondmin / fmax(firstmin, 0.01)`
__device__ __forceinline__ float pkr_ratio(float secondmin, float firstmin)
{
    return (float)((double)secondmin / fmax((double)firstmin, 0.01));
}

__device__ __forceinline__ void vfit3(float v0, float v1, float v2, float &vmin, float &xmin)
{   // refine.h:70-92
    if ((v1 > v0) && (v1 > v2)) { vmin = v1; xmin = 0.f; return; }
    float slope = v2 - v1;
    if ((v2 - v1) < (v0 - v1)) slope = v0 - v1;
    xmin = __fdiv_rn(v0 - v2, 2.f * slope);
    vmin = fmaf(xmin - 1.f, slope, v2);     // one fma in the reference build (pinned: oracle/mgm_oracle.c, scripts/fuzz_oracle.py)
}
__device__ __forceinline__ void parabola3(float v0, float v1, float v2, float &vmin, float &xmin)
{   // refine.h:40-68
    if (v1 > v0 && v1 > v2) { xmin = 0.f; vmin = v1; return; }
    float c = v1;
    float b = __fdiv_rn(v2 - v0, 2.f);
    float a = __fdiv_rn(v2 - 2.f * v1 + v0, 2.f);
    float x = __fdiv_rn(-b, 2.f * a);
    if (x > 1.f) x = 1.f;
    if (x < -1.f) x = -1.f;
    vmin = fmaf(fmaf(a, x, b), x, c);       // two fmas in the reference build
    xmin = x;
}

// The end of every WTA pixel: the sub-pixel fit around the winning slot kbest (V-fit / parabola on sS[kbest-1..kbest+1] when
// o-1 >= plo and o+2 <= phi, mgm_refine.h:67-84) and the disp / cost / conf stores.  o = gmin + kbest, the winning label;
// minP = (float)o and minL = S at kbest, formed by the caller as soon as it knows kbest (formed after its S and PKR stores
// instead, they cost the register-capped WTA kernels stack); confi: the passes whose last arg-minimum is kbest; plo, phi: the
// pixel's label range.  The closing __syncwarp lets the warp's next pixel reuse sS.
__device__ __forceinline__ void wta_store(const WtaParams &P, size_t p, int lane, const float *sS, int kbest, int o, float minP,
                                          float minL, int confi, int plo, int phi)
{
    if (P.refine != 0 && lane == 0) {
        if (o - 1 >= plo && o + 2 <= phi) {
            const float v0 = sS[kbest - 1], v1 = sS[kbest], v2 = sS[kbest + 1];
            float dx = 0.f, dxr = 0.f, ml = minL, mlr = minP;
            if (P.refine == 1) { vfit3(v0, v1, v2, ml, dx); vfit3(v2, v1, v0, mlr, dxr); }
            else { parabola3(v0, v1, v2, ml, dx); parabola3(v2, v1, v0, mlr, dxr); }
            minP = (float)o + dx;
            minL = ml;
            if (mlr < ml) { minP = (float)o - dxr; minL = mlr; }
        }
    }
    if (lane == 0) {
        P.disp[p] = __fdiv_rn(minP, P.inv_zoom_div);
        if (P.cost) P.cost[p] = minL;
        if (P.conf) P.conf[p] = (float)confi;
    }
    __syncwarp();
}

// One warp per pixel: S = (L0+L1+...+L_{ndir-1}) - (ndir-1) C in pass order (dvec.cc:110-118,
// mgm_core.cc:1041-1042), first strict minimum over finite S (:1044-1048), consensus (:1054-1057),
// V-fit / parabola on S[o-1..o+1] when o-1 >= lo and o+2 <= hi (mgm_refine.h:67-84).

// Which slots a lane of the WTA warp owns.  The sums are element-wise, so the WTA is free to choose: blocked (lane*LPL + e, one
// 8-/16-byte request per lane) when LPL is a multiple of 4 or is 2, interleaved (32*e + lane, LPL 4-byte requests of 128 contiguous
// bytes) for LPL = 3, 5, 6 -- a blocked lane stride of 12/20/24 bytes makes every request touch all of the pixel's 32-byte sectors
// (3-5x the L2->SM traffic of LPL 4/8/16).
// Both enumerate a lane's slots in ascending order, which is all the first-/last-minimum rules below need.
template <int LPL> struct WtaMap {
    static constexpr bool interleaved = (LPL == 3 || LPL == 5 || LPL == 6);
    static __device__ __forceinline__ int slot(int lane, int e) { return interleaved ? 32 * e + lane : lane * LPL + e; }
};
template <int LPL> __device__ __forceinline__ void wta_ld_pass(const float *px, int lane, float (&v)[LPL])
{
    if constexpr (WtaMap<LPL>::interleaved) {
#pragma unroll
        for (int e = 0; e < LPL; e++) v[e] = __ldcg(px + 32 * e + lane);
    } else ld_vec_cg<LPL>(px + lane * LPL, v);
}

// one pass' vector of this pixel: add it to S, note the LAST slot attaining the pass minimum (mgm_core.cc:1015-1019)
template <int LPL> __device__ __forceinline__ int wta_add_pass(const float (&v)[LPL], int lane, float (&s)[LPL])
{
    float lm = v[0];
#pragma unroll
    for (int e = 1; e < LPL; e++) lm = fminf(lm, v[e]);
    const float md = warp_min_f32(lm);
    int a = -1;
#pragma unroll
    for (int e = 0; e < LPL; e++) { if (v[e] == md) a = WtaMap<LPL>::slot(lane, e); s[e] += v[e]; }
    return __reduce_max_sync(0xffffffffu, a);
}
// everything after the sums: overcount fix, winner, consensus, sub-pixel fit, outputs.  sSrow: DP floats of shared memory
template <int LPL>
__device__ __forceinline__ void wta_finish(const WtaParams &P, size_t p, int lane, float (&s)[LPL], const int (&am)[kMaxPasses],
                                           const float (&c)[LPL], float *sSrow, int plo, int phi)
{   // plo, phi: the pixel's label range, loaded by the caller ahead of the sums (off the dependent chain of the pixel)
    constexpr int DP = 32 * LPL;
    float best = S2PB_INF;
    int bidx = 0x7fffffff;
#pragma unroll
    for (int e = 0; e < LPL; e++) {
        if (P.fix_overcount == 1) s[e] = fmaf(-(float)(P.ndir - 1), c[e], s[e]);
        if (isfinite(s[e]) && best > s[e]) { best = s[e]; bidx = WtaMap<LPL>::slot(lane, e); }
    }
    const float m = warp_min_f32(best);
    int cand = (best == m && bidx != 0x7fffffff) ? bidx : 0x7fffffff;
    int kbest = __reduce_min_sync(0xffffffffu, cand);         // first slot attaining the minimum
    if (kbest > DP - 1) kbest = 0;                            // unreachable: a pixel always has a finite S
    // every pixel has at least one finite S (its range always holds a finite cost)
    const int o = P.gmin + kbest;
    float minP = (float)o, minL = m;

    int confi = 0;
#pragma unroll
    for (int d = 0; d < kMaxPasses; d++) confi += (am[d] == kbest) ? 1 : 0;

    if (P.S != nullptr || P.refine != 0) {
        __syncwarp();
#pragma unroll
        for (int e = 0; e < LPL; e++) sSrow[WtaMap<LPL>::slot(lane, e)] = s[e];
        __syncwarp();
    }
    if (P.S != nullptr) {
        const int lo = plo - P.gmin, hi = phi - P.gmin;
        for (int kk = lane; kk < P.Dout; kk += 32)
            P.S[p * P.Dout + kk] = (kk >= lo && kk <= hi) ? sSrow[kk] : S2PB_INF;
    }
    if (P.pkr != nullptr) {
        const int lo = plo - P.gmin, hi = phi - P.gmin;
        float sec = S2PB_INF;
#pragma unroll
        for (int e = 0; e < LPL; e++) {
            const int kk = WtaMap<LPL>::slot(lane, e);
            if (kk >= lo && kk <= hi && abs(kk - kbest) > 2) sec = fminf(sec, s[e]);
        }
        sec = warp_min_f32(sec);
        if (lane == 0) P.pkr[p] = pkr_ratio(sec, m);
    }
    wta_store(P, p, lane, sSrow, kbest, o, minP, minL, confi, plo, phi);
}

// 128-thread CTAs capped at 64 registers for LPL <= 4: one of them still fits on an SM next to the two resident
// CTAs of the (issue-bound) aggregation kernel of the NEXT tile (2 x 256 x 112 + 128 x 64 = the 64 K registers of an SM), so this
// memory-bound kernel overlaps it.
constexpr int kWtaThreads = 128;
// NDIR: the number of passes when it is known at compile time (8: every s2p configuration), 0 = read P.ndir.  With a run-time
// count every pass sits behind its own branch and the eight (minimum -> compare -> last index) reductions of a pixel run one
// after the other; with NDIR = 8 they are straight-line code the scheduler interleaves.
template <int LPL, bool GEN, int NDIR>
__device__ __forceinline__ void wta_pixels(const WtaParams &P, float *sSrow)
{
    constexpr int DP = 32 * LPL;
    const int ndir = NDIR ? NDIR : P.ndir;
    const int lane = threadIdx.x & 31;
    size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
    for (size_t p = warp; p < P.npix; p += nwarps) {
        float s[LPL];
        int am[kMaxPasses];
#pragma unroll
        for (int e = 0; e < LPL; e++) s[e] = 0.f;
        // the pixel's range and (census flavour) its costs are requested first: they are consumed last, and a warp's pixel is one
        // dependent chain -- next to the aggregation kernel only four warps per SM run this kernel, so its rate there is
        // 1 / chain length, and every global load that waits at the end of the chain is ~1000 cycles of it
        const int plo = __ldg(P.lo + p), phi = __ldg(P.hi + p);
        constexpr bool early_cost = !GEN && !WtaMap<LPL>::interleaved && LPL <= 8;      // (wider: no registers to spare)
        CostPack<early_cost ? LPL : 1> cpk;
        if constexpr (early_cost) cpk = ld_cost<LPL, true>(reinterpret_cast<const uint8_t *>(P.C) + p * DP + lane * LPL);
        // the passes' vectors are requested four at a time before any is consumed (memory-level parallelism
        // within the register budget that lets this kernel share an SM with the aggregation kernel)
#pragma unroll
        for (int g = 0; g < kMaxPasses; g += 4) {
            float v[4][LPL];
#pragma unroll
            for (int q = 0; q < 4; q++)
                if (g + q < ndir) wta_ld_pass<LPL>(P.L[g + q] + p * DP, lane, v[q]);
#pragma unroll
            for (int q = 0; q < 4; q++) {
                am[g + q] = -1;
                if (g + q < ndir) am[g + q] = wta_add_pass<LPL>(v[q], lane, s);
            }
        }
        float c[LPL];
        if constexpr (GEN) wta_ld_pass<LPL>(reinterpret_cast<const float *>(P.C) + p * DP, lane, c);
        else if constexpr (WtaMap<LPL>::interleaved) {
            const uint8_t *cp = reinterpret_cast<const uint8_t *>(P.C) + p * DP + lane;
#pragma unroll
            for (int e = 0; e < LPL; e++) c[e] = cost_value(__ldg(cp + 32 * e), P.lut);
        } else {
            // (one code at a time: the packed decoder's temporaries cost this register-capped kernel spills)
            CostPack<LPL> cp;
            if constexpr (early_cost) cp = cpk;
            else cp = ld_cost<LPL, true>(reinterpret_cast<const uint8_t *>(P.C) + p * DP + lane * LPL);
#pragma unroll
            for (int e = 0; e < LPL; e++) c[e] = cost_value(cost_code(cp, e), P.lut);
        }
        wta_finish<LPL>(P, p, lane, s, am, c, sSrow, plo, phi);
    }
}
template <int LPL, bool GEN>
__global__ void __launch_bounds__(kWtaThreads) __maxnreg__((LPL <= 4) ? 64 : 128) wta_kernel(const WtaParams P)
{
    __shared__ float sS[kWtaThreads / 32][32 * LPL];
    float *sSrow = sS[threadIdx.x >> 5];
    if (P.ndir == kMaxPasses) wta_pixels<LPL, GEN, kMaxPasses>(P, sSrow);
    else wta_pixels<LPL, GEN, 0>(P, sSrow);
}

// The WTA of the folded layout (FoldView, agg_kernel.cuh): the aggregation has summed S in pass order and recorded each pass's
// last arg-minimum, so a pixel reads its S vector, its costs (for the overcount fix) and one short per pass, and ends in
// wta_finish as wta_kernel does -- the same winner, consensus, sub-pixel fit, PKR and outputs.
struct FoldPlanes {
    const float *S;                     // [npix][DP]
    const short *am[kMaxPasses];        // [npix] per pass (passes >= ndir: unused)
};
// a pixel's costs in the WTA's slot mapping (WtaMap)
template <int LPL, bool GEN> __device__ __forceinline__ void wta_ld_cost(const WtaParams &P, size_t p, int lane, float (&c)[LPL])
{
    constexpr int DP = 32 * LPL;
    if constexpr (GEN) wta_ld_pass<LPL>(reinterpret_cast<const float *>(P.C) + p * DP, lane, c);
    else if constexpr (WtaMap<LPL>::interleaved) {
        const uint8_t *cp = reinterpret_cast<const uint8_t *>(P.C) + p * DP + lane;
#pragma unroll
        for (int e = 0; e < LPL; e++) c[e] = cost_value(__ldg(cp + 32 * e), P.lut);
    } else {
        const CostPack<LPL> cp = ld_cost<LPL, true>(reinterpret_cast<const uint8_t *>(P.C) + p * DP + lane * LPL);
#pragma unroll
        for (int e = 0; e < LPL; e++) c[e] = cost_value(cost_code(cp, e), P.lut);
    }
}
template <int LPL, bool GEN>
__global__ void __launch_bounds__(kWtaThreads) wta_fold_kernel(const WtaParams P, const FoldPlanes F)
{
    constexpr int DP = 32 * LPL;
    __shared__ float sS[kWtaThreads / 32][DP];
    float *sSrow = sS[threadIdx.x >> 5];
    const int lane = threadIdx.x & 31;
    const short *amp = F.am[0];                   // lanes 0 .. ndir-1: the arg-minimum plane of pass `lane`
#pragma unroll
    for (int q = 1; q < kMaxPasses; q++) if (lane == q) amp = F.am[q];
    const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
    for (size_t p = warp; p < P.npix; p += nwarps) {
        const int plo = __ldg(P.lo + p), phi = __ldg(P.hi + p);
        const int a = lane < P.ndir ? __ldg(amp + p) : -1;
        float s[LPL], c[LPL];
        wta_ld_pass<LPL>(F.S + p * DP, lane, s);
        wta_ld_cost<LPL, GEN>(P, p, lane, c);
        int am[kMaxPasses];
#pragma unroll
        for (int d = 0; d < kMaxPasses; d++) am[d] = __shfl_sync(0xffffffffu, a, d);
        wta_finish<LPL>(P, p, lane, s, am, c, sSrow, plo, phi);
    }
}

// The same WTA reading only the labels that can still win (DESIGN.md 3.2).  Census flavour, unit weights: every message of
// the aggregation is >= 0, so L_p[d] >= C[d] in every pass, S[d] >= C[d] and S[d] >= L_0[d].  With T = S[d0] of one probe
// slot d0 (any slot gives a valid bound; the first slot holding the pixel's smallest cost code is the probe), a slot with
// L_0[d] > T is neither the winner nor a tie for it.  Pass 0 is read whole.  Passes 1-7 are read only where L_0[d] <= T,
// dilated by one slot (the sub-pixel fit reads S[k-1], S[k+1]), or where C[d] <= L_q[d0]: a pass-q arg-minimum d* has
// C[d*] <= L_q[d*] = min L_q <= L_q[d0], so every pass's consensus slot is read.  Lanes 0-7 hold L_q[d0] from the probe.
// L_q >= C holds without rounding (L_q = fl(C + x), x >= 0), so that term needs no slack.  The other slots of passes 1-7 read
// +INF, which is what the sums, minima and comparisons of wta_finish make of a slot that cannot win.  Outputs are those of
// wta_kernel bit for bit.  Eight passes, blocked slots, no dense S and no PKR image (both read slots that cannot win).
//
// A pixel's dependent chain is codes -> probe -> passes 1-7.  Pass 0 is requested with the probe: masking it by C <= T would
// wait on the probe, one more round trip per pixel, to skip about 37 % of its sectors.  A warp works three pixels deep:
// pixel p+1's probe and whole pass 0 are requested before p's passes 1-7, and pixel p+2's codes and range one pixel ahead of
// its probe.  Passes 1-7 are requested together (all seven fit in flight under the 64-register cap), so a pixel waits on one
// round trip.
template <int LPL> __device__ __forceinline__ unsigned wta_probe_key(const CostPack<LPL> &cp, int lane)
{   // (smallest code << 9) | first slot holding it
    unsigned key = 0xffffffffu;
#pragma unroll
    for (int e = 0; e < LPL; e++) key = min(key, (cost_code(cp, e) << 9) | (unsigned)(lane * LPL + e));
    return __reduce_min_sync(0xffffffffu, key);
}
// S of the probe slot from lanes 0-7's L_p[d0], with wta_finish's arithmetic: passes added in order, then the overcount fix
__device__ __forceinline__ float wta_probe_sum(const WtaParams &P, float pv, unsigned key)
{
    float t = 0.f;
#pragma unroll
    for (int q = 0; q < kMaxPasses; q++) t += __shfl_sync(0xffffffffu, pv, q);
    if (P.fix_overcount == 1) t = fmaf(-(float)(kMaxPasses - 1), cost_value(key >> 9, P.lut), t);
    return t;
}
// m: which of the lane's LPL slots can still win.  The lane requests its slots when one of them or a neighbour of one (the
// sub-pixel fit reads S[k-1], S[k+1]) is in m; the dilation across lanes is two shuffles.  (A pixel always has a finite S at
// its probe; were it not so, nothing is pruned.)
template <int LPL> __device__ __forceinline__ bool wta_lane_reads(unsigned m, int lane, float T)
{
    const unsigned left = __shfl_up_sync(0xffffffffu, m, 1), right = __shfl_down_sync(0xffffffffu, m, 1);
    return m != 0 || (lane > 0 && ((left >> (LPL - 1)) & 1u)) || (lane < 31 && (right & 1u)) || !(T < S2PB_INF);
}
template <int LPL> __device__ __forceinline__ void wta_ld_pass_if(const float *px, int lane, bool ld, float (&v)[LPL])
{
#pragma unroll
    for (int e = 0; e < LPL; e++) v[e] = S2PB_INF;
    if (ld) wta_ld_pass<LPL>(px, lane, v);
}
__device__ __forceinline__ unsigned wta_range(const WtaParams &P, unsigned p)
{
    return ((unsigned)(unsigned short)__ldg(P.lo + p)) | ((unsigned)(unsigned short)__ldg(P.hi + p) << 16);
}
// the widths wta_pruned_kernel serves (launch_wta in s2pb200.cu picks it): blocked slots, codes held in registers
__host__ __device__ constexpr bool wta_pruned_width(int LPL) { return LPL == 1 || LPL == 2 || LPL == 4 || LPL == 8; }
template <int LPL>
__global__ void __launch_bounds__(kWtaThreads) __maxnreg__((LPL <= 4) ? 64 : 128) wta_pruned_kernel(const WtaParams P)
{
    static_assert(wta_pruned_width(LPL) && !WtaMap<LPL>::interleaved, "blocked slots, codes held in registers");
    constexpr int DP = 32 * LPL;
    __shared__ float sS[kWtaThreads / 32][DP];
    float *sSrow = sS[threadIdx.x >> 5];
    const int lane = threadIdx.x & 31;
    // (32-bit pixel counters and the range in one word: the state of three pixels shares the register cap)
    const unsigned warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
    const unsigned npix = (unsigned)P.npix;
    if (warp >= npix) return;
    const float *probe = P.L[0];                 // lanes 0-7: the pass this lane probes
#pragma unroll
    for (int q = 1; q < kMaxPasses; q++) if (lane == q) probe = P.L[q];
    const uint8_t *codes = reinterpret_cast<const uint8_t *>(P.C) + lane * LPL;
    // pixel p: range, codes, probe values and pass 0 requested; pixel p1: range and codes requested
    unsigned p = warp;
    unsigned range = wta_range(P, p);
    CostPack<LPL> cpk = ld_cost<LPL, true>(codes + (size_t)p * DP);
    unsigned key = wta_probe_key<LPL>(cpk, lane);
    float pv = lane < kMaxPasses ? __ldcg(probe + (size_t)p * DP + (key & 511u)) : 0.f;
    float v0[LPL];
    wta_ld_pass<LPL>(P.L[0] + (size_t)p * DP, lane, v0);
    unsigned p1 = p + nwarps;
    unsigned range1 = range;
    CostPack<LPL> cpk1 = cpk;
    if (p1 < npix) { range1 = wta_range(P, p1); cpk1 = ld_cost<LPL, true>(codes + (size_t)p1 * DP); }
    for (;;) {
        const bool more1 = p1 < npix;
        const unsigned p2 = p1 + nwarps;
        unsigned range2 = range1;
        CostPack<LPL> cpk2 = cpk1;
        unsigned key1 = 0;
        float pv1 = 0.f, v01[LPL];
        if (more1) {
            if (p2 < npix) { range2 = wta_range(P, p2); cpk2 = ld_cost<LPL, true>(codes + (size_t)p2 * DP); }
            key1 = wta_probe_key<LPL>(cpk1, lane);
            if (lane < kMaxPasses) pv1 = __ldcg(probe + (size_t)p1 * DP + (key1 & 511u));
            wta_ld_pass<LPL>(P.L[0] + (size_t)p1 * DP, lane, v01);
        }
        // the integer costs of census 5x5 make S >= L_0 exact; the scaled costs of 3x3 / 7x7 round in the eight additions and the
        // overcount fix, by less than 2^-18 of S in all, so the bound is taken 2^-16 wider
        const float T = wta_probe_sum(P, pv, key) * (1.f + 1.f / 65536.f);
        float s[LPL];
        int am[kMaxPasses];
#pragma unroll
        for (int e = 0; e < LPL; e++) s[e] = 0.f;
        am[0] = wta_add_pass<LPL>(v0, lane, s);
        unsigned m = 0;
        float cmin = S2PB_INF;
#pragma unroll
        for (int e = 0; e < LPL; e++) {
            if (v0[e] <= T) m |= 1u << e;
            cmin = fminf(cmin, cost_value(cost_code(cpk, e), P.lut));
        }
        const bool ld = wta_lane_reads<LPL>(m, lane, T);
        // (every lane takes part in the shuffles: no short-circuit around them)
        unsigned ldq = 0;
#pragma unroll
        for (int q = 1; q < kMaxPasses; q++) if (cmin <= __shfl_sync(0xffffffffu, pv, q)) ldq |= 1u << q;
        float v[kMaxPasses - 1][LPL];
#pragma unroll
        for (int q = 1; q < kMaxPasses; q++) wta_ld_pass_if<LPL>(P.L[q] + (size_t)p * DP, lane, ld || ((ldq >> q) & 1u), v[q - 1]);
#pragma unroll
        for (int q = 1; q < kMaxPasses; q++) am[q] = wta_add_pass<LPL>(v[q - 1], lane, s);
        float c[LPL];
#pragma unroll
        for (int e = 0; e < LPL; e++) c[e] = cost_value(cost_code(cpk, e), P.lut);
        wta_finish<LPL>(P, p, lane, s, am, c, sSrow, (short)(range & 0xffffu), (short)(range >> 16));
        if (!more1) break;
        p = p1; p1 = p2; range = range1; range1 = range2; cpk = cpk1; cpk1 = cpk2; key = key1; pv = pv1;
#pragma unroll
        for (int e = 0; e < LPL; e++) v0[e] = v01[e];
    }
}

// Companion of agg_chunked.cuh (slabs wider than 512 slots): the same WTA for
// slabs whose pixels use few of their 32-label chunks.  A warp owns a pixel and only reads the chunks [ea, eb] that hold its
// label range (slot 32*e + lane), so a 40-label pixel of a 512-slot slab reads 2 x 128 B per pass instead of 2 KB.
// Per lane it keeps, for every pass, the running minimum and the LAST slot attaining it, and for S the running
// first minimum; S itself goes to shared memory for the sub-pixel fit.  Same arithmetic as wta_kernel<LPL, GEN>.
// FOLD: the folded layout's WTA (F): S is read as the aggregation summed it, and each pass's arg-minimum from its plane.
template <bool GEN, bool FOLD = false>
__global__ void __launch_bounds__(kWtaThreads) wta_chunked_kernel(const WtaParams P, int DP, const FoldPlanes F)
{
    extern __shared__ float sS_all[];                    // [warps][DP]
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    float *sS = sS_all + (size_t)wib * DP;
    size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
    for (size_t p = warp; p < P.npix; p += nwarps) {
        const int lo = P.lo[p] - P.gmin, hi = P.hi[p] - P.gmin;      // slots
        const int ea = lo >> 5, eb = hi >> 5;
        float pm[kMaxPasses];
        int pa[kMaxPasses];
#pragma unroll
        for (int d = 0; d < kMaxPasses; d++) { pm[d] = S2PB_INF; pa[d] = -1; }
        float best = S2PB_INF;
        int bidx = 0x7fffffff;
        for (int e = ea; e <= eb; e++) {
            const int kk = 32 * e + lane;
            float s = 0.f;
            if constexpr (FOLD) s = __ldcg(F.S + p * DP + kk);
            else {
#pragma unroll
                for (int d = 0; d < kMaxPasses; d++)
                    if (d < P.ndir) {
                        const float v = __ldcg(P.L[d] + p * DP + kk);
                        if (v < pm[d]) { pm[d] = v; pa[d] = kk; } else if (v == pm[d]) pa[d] = kk;
                        s += v;
                    }
            }
            const float c = GEN ? reinterpret_cast<const float *>(P.C)[p * DP + kk]
                                : cost_value(reinterpret_cast<const uint8_t *>(P.C)[p * DP + kk], P.lut);
            if (P.fix_overcount == 1) s = fmaf(-(float)(P.ndir - 1), c, s);
            if (isfinite(s) && best > s) { best = s; bidx = kk; }
            sS[kk] = s;
        }
        // per pass: the LAST slot of the whole vector attaining its minimum (mgm_core.cc:1015-1019)
        int confi_src[kMaxPasses];
#pragma unroll
        for (int d = 0; d < kMaxPasses; d++) {
            confi_src[d] = -1;
            if (d < P.ndir) {
                if constexpr (FOLD) confi_src[d] = __ldg(F.am[d] + p);
                else {
                    const float md = warp_min_f32(pm[d]);
                    confi_src[d] = __reduce_max_sync(0xffffffffu, (pm[d] == md) ? pa[d] : -1);
                }
            }
        }
        const float m = warp_min_f32(best);
        int kbest = __reduce_min_sync(0xffffffffu, (best == m && bidx != 0x7fffffff) ? bidx : 0x7fffffff);
        if (kbest > DP - 1) kbest = 0;
        const int o = P.gmin + kbest;
        float minP = (float)o, minL = m;
        int confi = 0;
#pragma unroll
        for (int d = 0; d < kMaxPasses; d++) confi += (confi_src[d] == kbest) ? 1 : 0;
        __syncwarp();
        if (P.pkr != nullptr) {
            float sec = S2PB_INF;
            for (int e = ea; e <= eb; e++) {
                const int kk = 32 * e + lane;
                if (kk >= lo && kk <= hi && abs(kk - kbest) > 2) sec = fminf(sec, sS[kk]);
            }
            sec = warp_min_f32(sec);
            if (lane == 0) P.pkr[p] = pkr_ratio(sec, m);
        }
        wta_store(P, p, lane, sS, kbest, o, minP, minL, confi, P.gmin + lo, P.gmin + hi);
    }
}

// ------------------------------------------------------------------ image-space post filters

// median_filter, img_tools.h:204-238: window clipped to the image, NaN skipped, element
// size/2 of the sorted values; pixel unchanged when the window holds no value.
__global__ void median_kernel(const float *__restrict__ in, float *__restrict__ out, int w, int h, int radius)
{
    int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    float v[25];
    int n = 0;
    for (int j = -radius; j <= radius; j++) {
        int yy = y + j;
        if (yy < 0 || yy >= h) continue;
        for (int i = -radius; i <= radius; i++) {
            int xx = x + i;
            if (xx < 0 || xx >= w) continue;
            float t = in[(size_t)yy * w + xx];
            if (!isnan(t)) {   // insertion sort
                int q = n++;
                while (q > 0 && v[q - 1] > t) { v[q] = v[q - 1]; q--; }
                v[q] = t;
            }
        }
    }
    out[(size_t)y * w + x] = n ? v[n / 2] : in[(size_t)y * w + x];
}

// leftright_test, stereo_utils.cc:9-32: `out` = `dx` with the pixels failing the test set to NaN;
// `other` is the other view's disparity BEFORE its own test (mgm_multiscale.cc:322-327).
__global__ void lrcheck_kernel(const float *__restrict__ dx, const float *__restrict__ other, float *__restrict__ out,
                               int w, int h, float tau)
{
    int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    size_t i = (size_t)y * w + x;
    float d = dx[i], r = d;
    float t = (float)x + d;
    if (!isfinite(t)) r = __int_as_float(0x7fc00000);
    else {
        float rt = roundf(t);
        if (rt < (float)w && rt >= 0.f) {
            int Lx = (int)rt;
            float Rx = (float)Lx + other[(size_t)y * w + Lx];
            if (fabs((double)(Rx - (float)x)) > (double)tau) r = __int_as_float(0x7fc00000);
        } else r = __int_as_float(0x7fc00000);
    }
    out[i] = r;
}

// mindiff, stereo_utils.cc:93-124: inside the image minus a border of half a window, a pixel whose disparity
// differs by more than tau from the disparity of the window's lowest-cost finite pixel becomes NaN.  `corr` is
// the OTHER view's refined cost image, indexed with this view's coordinates, exactly as the reference does
// (mgm_multiscale.cc:318-319).  Window scan: x offset outer, y offset inner, strict comparison.
__global__ void mindiff_kernel(const float *__restrict__ disp, const float *__restrict__ corr, float *__restrict__ out,
                               int w, int h, int win, float tau)
{
    int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const int wl = win / 2, wr = (win % 2 == 0) ? win / 2 - 1 : win / 2;
    const size_t o = (size_t)y * w + x;
    float d = disp[o];
    if (y >= wl && y < h - wr && x >= wl && x < w - wr) {
        float mincorr = S2PB_INF, mindisp = 0.f;
        for (int i = -wl; i <= wr; i++)
            for (int j = -wl; j <= wr; j++) {
                const size_t q = (size_t)(y + j) * w + (x + i);
                const float c = corr[q], dd = disp[q];
                if (mincorr > c && isfinite(dd)) { mincorr = c; mindisp = dd; }
            }
        if (fabsf(d - mindisp) > tau) d = __int_as_float(0x7fc00000);
    }
    out[o] = d;
}

// main_mgm.cc:231-236 : no-data pixels of the view's own image get NaN
__global__ void nan_restore_kernel(float *__restrict__ d, const float *__restrict__ orig, int n)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && isnan(orig[i])) d[i] = __int_as_float(0x7fc00000);
}

__device__ __forceinline__ float cubic1(const float v[4], float x)
{   // c/bicubic.c:8-13 -- double arithmetic through the literals, result narrowed to float
    double xd = x;
    return (float)((double)v[1] + 0.5 * xd * ((double)v[2] - (double)v[0]
                   + xd * (2.0 * v[0] - 5.0 * v[1] + 4.0 * v[2] - (double)v[3]
                   + xd * (3.0 * ((double)v[1] - (double)v[2]) + (double)v[3] - (double)v[0]))));
}
// create_rejection_mask (s2p/block_matching.py:18-32): backflow samples im2 at (x+d, y) with the
// zero-boundary bicubic of c/bicubic.c:69-96, mask = finite(disp) & finite(im1) & finite(sample).
__global__ void rejection_mask_kernel(const float *__restrict__ disp, const float *__restrict__ im1,
                                      const float *__restrict__ im2, int w, int h, uint8_t *__restrict__ mask)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= w || j >= h) return;
    size_t idx = (size_t)j * w + i;
    float d = disp[idx];
    float x = ((float)i + d) - 1.f, y = (float)j - 1.f;
    float r;
    if (!isfinite(x)) r = x;
    else {
        int ix = (int)floorf(x), iy = (int)floorf(y);
        float vv[4];
        for (int ii = 0; ii < 4; ii++) {
            float col[4];
            for (int jj = 0; jj < 4; jj++) {
                int sx = ix + ii, sy = iy + jj;
                col[jj] = (sx < 0 || sx >= w || sy < 0 || sy >= h) ? 0.f : im2[(size_t)sy * w + sx];
            }
            vv[ii] = cubic1(col, y - (float)iy);
        }
        r = cubic1(vv, x - (float)ix);
    }
    mask[idx] = (isfinite(d) && isfinite(im1[idx]) && isfinite(r)) ? 1 : 0;
}


// masking.erosion (s2p/masking.py:87-97 -> `morsi diskR erosion`, c/morsi.c:54-66,280-298): minimum over the
// discrete disk {(i,j) : hypot(i,j) < R}; samples outside the image are NaN for the reference's fmin, i.e. ignored.
__global__ void erode_mask_kernel(const uint8_t *__restrict__ in, uint8_t *__restrict__ out, int w, int h, float radius)
{
    int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const int r = (int)radius + 1;
    unsigned v = 255;
    for (int i = -r; i <= r; i++)
        for (int j = -r; j <= r; j++) {
            if (!(hypot((double)i, (double)j) < (double)radius)) continue;
            int xx = x + i, yy = y + j;
            if (xx < 0 || xx >= w || yy < 0 || yy >= h) continue;
            v = min(v, (unsigned)in[(size_t)yy * w + xx]);
        }
    out[(size_t)y * w + x] = (uint8_t)v;
}

}  // namespace s2pb
