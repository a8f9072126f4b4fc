// sgbm_kernels.cuh -- s2p's `sgbm` matcher (3rdparty/sgbm: sgbm.cpp + OpenCV 2's StereoSGBM with fullDP = 1) on the GPU.
//
// Every step is integer arithmetic and reproduces the reference bit for bit (DESIGN.md section 3.5):
//   qauto thresholds  -> radix select of two order statistics of the non-NaN floats of im1
//   quantisation      -> both images into a zero-padded 8-bit pair (the wrapper's crop trick, margins zero)
//   pixel cost        -> x-Sobel through clipTab, Birchfield-Tomasi on (Sobel, intensity/4), one block per row
//   window cost       -> SAD box sum with the reference's clamped indices and its two untouched regions
//   aggregation       -> 8 scanline passes, one warp per scanline, labels across lanes; S = min(sum of L, SHRT_MAX)
//   WTA               -> first minimum, uniqueness, parabola with C division, right view by packed atomicMin, LR check
//   post-filters      -> 3x3 median (replicated border), speckle filter by union-find, crop and -d/16
// Coordinates: X = column of the padded images (width `wp`), x = X - minX1 = column of the cost volume (width `w1`).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "union_find.cuh"
#include "order_stats.h"

namespace s2pb {

constexpr int kSgbmMaxCost = 32767;        // SHRT_MAX, the reference's MAX_COST and the int16 saturation value
constexpr int kSgbmFtzero = 63;            // max(preFilterCap = 63, 15) | 1
constexpr int kSgbmUniqueness = 10;        // uniquenessRatio
constexpr int kSgbmSpeckleWindow = 50;     // speckleWindowSize
constexpr int kSgbmSpeckleRange = 16;      // speckleRange 1, times DISP_SCALE
constexpr int kSgbmPixMax = 2 * kSgbmFtzero + (255 >> 2);   // largest per-pixel BT cost: Sobel channel + intensity >> 2

typedef OrderStats SgbmState;

// float -> unsigned key with the order of the floats (-0 sorts before +0; the two quantise alike)
__device__ __forceinline__ unsigned sgbm_key(float f)
{
    const unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float sgbm_unkey(unsigned k)
{
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// one 8-bit digit of every order statistic (digit 3 = most significant); hist[kOrdMaxRanks][256], zeroed by the caller.
// Before the first pass every prefix is 0 and the mask keeps no bit, so all ranks count every value.
__global__ void sgbm_hist_kernel(const float *__restrict__ im, int n, int digit, const SgbmState *__restrict__ st,
                                 unsigned *__restrict__ hist)
{
    __shared__ unsigned h[kOrdMaxRanks][256];
    for (int i = threadIdx.x; i < kOrdMaxRanks * 256; i += blockDim.x) h[i >> 8][i & 255] = 0;
    __syncthreads();
    const int shift = 8 * digit;
    const unsigned hi_mask = digit == 3 ? 0u : (0xffffffffu << (shift + 8));
    const int nr = digit == 3 ? 1 : st->nranks;      // the first pass: one histogram of all values serves every rank
    unsigned p[kOrdMaxRanks];
    for (int r = 0; r < kOrdMaxRanks; r++) p[r] = st->prefix[r];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float f = im[i];
        if (isnan(f)) continue;
        const unsigned k = sgbm_key(f), b = (k >> shift) & 255u;
#pragma unroll
        for (int r = 0; r < kOrdMaxRanks; r++)
            if (r < nr && (k & hi_mask) == p[r]) atomicAdd(&h[r][b], 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kOrdMaxRanks * 256; i += blockDim.x)
        if (h[i >> 8][i & 255]) atomicAdd(hist + i, h[i >> 8][i & 255]);
}

// numpy's 'linear' quantile q of n sorted values (numpy/lib/_function_base_impl.py: _quantile with get_virtual_index
// (n - 1) * q, _get_indexes, _get_gamma): the ranks of the two neighbours and the weight gamma
__device__ __forceinline__ void ord_linear_ranks(unsigned n, double q, unsigned &prev, unsigned &next, double &gamma)
{
    const double vi = __dmul_rn((double)(n - 1), q);
    if (vi >= (double)(n - 1)) {             // index -1 for both: the largest value; gamma = vi - (-1)
        prev = next = n - 1;
        gamma = __dadd_rn(vi, 1.0);
    } else {
        const double f = floor(vi);
        prev = (unsigned)f; next = prev + 1;
        gamma = __dsub_rn(vi, f);
    }
}

// numpy's _lerp(a, b, t) for float32 (or narrower) a and b: b - a in the inputs' type, everything else in double
__device__ __forceinline__ double ord_lerp(float a, float b, double t)
{
    const double d = (double)__fsub_rn(b, a);
    if (t >= 0.5) return __dsub_rn((double)b, __dmul_rn(d, __dsub_rn(1.0, t)));
    return __dadd_rn((double)a, __dmul_rn(d, t));
}

// one thread: the digit's bucket for every rank.  After digit 0 the prefixes are the keys of the order statistics.
// kOrdQauto (get_rminmax, sgbm.cpp:30-42): rb = N/200, rmin = tx[rb], rmax = tx[N-1-rb] of the sorted non-NaN values.
// kOrdLinear: the floor and ceiling ranks of the virtual index of q[0] and q[1], then their interpolation into lo and hi.
__global__ void sgbm_select_kernel(int digit, int rule, double q0, double q1, SgbmState *st, unsigned *hist)
{
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    if (digit == 3) {
        st->rule = rule; st->q[0] = q0; st->q[1] = q1;
        unsigned n = 0;
        for (int b = 0; b < 256; b++) n += hist[b];
        st->n = (int)n;
        if (st->rule == kOrdQauto) {
            const unsigned rb = n / 200;
            st->nranks = 2;
            st->rank[0] = rb;
            st->rank[1] = n ? n - 1 - rb : 0;
        } else {
            st->nranks = 4;
            double g;
            for (int k = 0; k < 2; k++) ord_linear_ranks(n ? n : 1, st->q[k], st->rank[2 * k], st->rank[2 * k + 1], g);
        }
        for (int r = 0; r < kOrdMaxRanks; r++) st->prefix[r] = 0;
        for (int r = 1; r < st->nranks; r++)                     // the first pass counted every value once, for rank 0
            for (int b = 0; b < 256; b++) hist[r * 256 + b] = hist[b];
    }
    for (int r = 0; r < st->nranks; r++) {
        unsigned cum = 0, b = 0;
        for (; b < 255; b++) {
            if (st->rank[r] < cum + hist[r * 256 + b]) break;
            cum += hist[r * 256 + b];
        }
        st->prefix[r] |= b << (8 * digit);
        st->rank[r] -= cum;
    }
    for (int i = 0; i < kOrdMaxRanks * 256; i++) hist[i] = 0;
    if (digit == 0) {
        for (int r = 0; r < st->nranks; r++) st->v[r] = sgbm_unkey(st->prefix[r]);
        st->rmin = st->v[0]; st->rmax = st->v[1];
        if (st->rule == kOrdLinear) {
            const double nan = __longlong_as_double(0x7ff8000000000000ll);
            double g[2];
            unsigned pr, nx;
            for (int k = 0; k < 2; k++) ord_linear_ranks(st->n ? (unsigned)st->n : 1u, st->q[k], pr, nx, g[k]);
            st->lo = st->n ? ord_lerp(st->v[0], st->v[1], g[0]) : nan;
            st->hi = st->n ? ord_lerp(st->v[2], st->v[3], g[1]) : nan;
        }
    }
}

// qauto / qeasy (sgbm.cpp:44-71) into the padded 8-bit images: g = floor(255 * (x - rmin) / (rmax - rmin)) in float,
// clamped to [0, 255]; a NaN (input, or 0/0 when rmax == rmin) converts to 0 as on x86.  Margins are zero.
__global__ void sgbm_quantize_kernel(const float *__restrict__ im1, const float *__restrict__ im2, int w, int h, int off,
                                     int wp, const SgbmState *__restrict__ st, uint8_t *__restrict__ q1,
                                     uint8_t *__restrict__ q2)
{
    const int X = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (X >= wp) return;
    const int x = X - off;
    uint8_t a = 0, b = 0;
    if (x >= 0 && x < w && st->n > 0) {
        const float lo = st->rmin, span = __fsub_rn(st->rmax, st->rmin);
        const float f[2] = {im1[(size_t)y * w + x], im2[(size_t)y * w + x]};
        uint8_t o[2];
        for (int k = 0; k < 2; k++) {
            float g = floorf(__fdiv_rn(__fmul_rn(255.f, __fsub_rn(f[k], lo)), span));
            if (g < 0.f) g = 0.f;
            if (g > 255.f) g = 255.f;
            o[k] = isnan(g) ? 0 : (uint8_t)g;
        }
        a = o[0]; b = o[1];
    }
    q1[(size_t)y * wp + X] = a;
    q2[(size_t)y * wp + X] = b;
}

// Geometry of one computeDisparitySGBM call (stereosgbm.cpp:328-341, 121-123), shared by the host and the kernels.
struct SgbmGeom {
    int wp, h;              // padded width, height
    int minD, D;            // labels minD .. minD+D-1 (OpenCV convention: img1(X) ~ img2(X - d))
    int minX1, w1;          // cost-volume columns X = minX1 .. minX1+w1-1
    int minX2, w2;          // columns of the min/max buffers of calcPixelCostBT
    int SW2, SH2, P1, P2;
};

// calcPixelCostBT (stereosgbm.cpp:115-280) for row y, one block.  The reference reads its per-row byte buffer
// (v0 | v1 | prow1 x 2 channels | prow2 x 2 channels, followed by never-written bytes and preceded by disp2ptr, which is
// still zero while pass 1 computes costs) at indices that leave the valid ranges for the labels that look past an image
// border.  This kernel lays out the same bytes in shared memory and reads them with the same index arithmetic, so those
// costs match as well; bytes outside the written ranges are zero (the allocation is zeroed; DESIGN.md section 4).
__device__ __forceinline__ int sgbm_byte(const uint8_t *vv, const uint8_t *prow, int nvv, int nprow, int off)
{
    if (off < 0) return 0;
    if (off < nvv) return vv[off];
    off -= nvv;
    return off < nprow ? prow[off] : 0;
}
__global__ void sgbm_pixcost_kernel(const uint8_t *__restrict__ q1, const uint8_t *__restrict__ q2, SgbmGeom g,
                                    short *__restrict__ pix)
{
    extern __shared__ uint8_t sgbm_rowbuf[];
    const int y = blockIdx.x, wp = g.wp, nvv = 2 * g.w2, nprow = 4 * wp;
    uint8_t *prow = sgbm_rowbuf, *vv0 = sgbm_rowbuf + nprow, *vv1 = vv0 + nvv;     // prow1 c0, prow1 c1, prow2 c0, prow2 c1; v0|v1 per channel
    const uint8_t *r1 = q1 + (size_t)y * wp, *r2 = q2 + (size_t)y * wp;
    const uint8_t *n1 = q1 + (size_t)(y > 0 ? y - 1 : y) * wp, *s1 = q1 + (size_t)(y < g.h - 1 ? y + 1 : y) * wp;
    const uint8_t *n2 = q2 + (size_t)(y > 0 ? y - 1 : y) * wp, *s2 = q2 + (size_t)(y < g.h - 1 ? y + 1 : y) * wp;
    for (int x = threadIdx.x; x < wp; x += blockDim.x) {
        uint8_t a0 = kSgbmFtzero, a1 = kSgbmFtzero, b0 = kSgbmFtzero, b1 = kSgbmFtzero;   // tab[0] at both ends
        if (x >= 1 && x < wp - 1) {
            const int sa = (r1[x + 1] - r1[x - 1]) * 2 + n1[x + 1] - n1[x - 1] + s1[x + 1] - s1[x - 1];
            const int sb = (r2[x + 1] - r2[x - 1]) * 2 + n2[x + 1] - n2[x - 1] + s2[x + 1] - s2[x - 1];
            a0 = (uint8_t)(min(max(sa, -kSgbmFtzero), kSgbmFtzero) + kSgbmFtzero);
            b0 = (uint8_t)(min(max(sb, -kSgbmFtzero), kSgbmFtzero) + kSgbmFtzero);
            a1 = r1[x];
            b1 = r2[x];
        }
        prow[x] = a0;
        prow[wp + x] = a1;
        prow[2 * wp + (wp - 1 - x)] = b0;                    // the right row is stored reversed
        prow[3 * wp + (wp - 1 - x)] = b1;
    }
    __syncthreads();
    for (int c = 0; c < 2; c++) {                            // min / max of the half-pixel neighbourhood of the right row
        const uint8_t *p2 = prow + 2 * wp + c * wp;
        uint8_t *vv = c ? vv1 : vv0;
        for (int x = g.minX2 + threadIdx.x; x < g.minX2 + g.w2; x += blockDim.x) {
            const int v = p2[x];
            const int vl = x > 0 ? (v + p2[x - 1]) / 2 : v, vr = x < wp - 1 ? (v + p2[x + 1]) / 2 : v;
            vv[x - g.minX2] = (uint8_t)min(min(vl, vr), v);
            vv[x - g.minX2 + g.w2] = (uint8_t)max(max(vl, vr), v);
        }
    }
    __syncthreads();
    const size_t n = (size_t)g.w1 * g.D;
    short *out = pix + (size_t)y * n;
    for (size_t i = threadIdx.x; i < n; i += blockDim.x) {
        const int xi = (int)(i / g.D), di = (int)(i - (size_t)xi * g.D);
        const int x = xi + g.minX1, d = di + g.minD;
        int cost = 0;
        for (int c = 0; c < 2; c++) {
            const uint8_t *p1 = prow + c * wp, *vv = c ? vv1 : vv0;
            const int u = p1[x];
            const int ul = x > 0 ? (u + p1[x - 1]) / 2 : u, ur = x < wp - 1 ? (u + p1[x + 1]) / 2 : u;
            const int u0 = min(min(ul, ur), u), u1 = max(max(ul, ur), u);
            const int j = wp - 1 - x + d;                    // reversed right column x - d
            const int v = sgbm_byte(vv, prow, nvv, nprow, nvv + 2 * wp + c * wp + j);
            const int v0 = sgbm_byte(vv, prow, nvv, nprow, j - g.minX2);
            const int v1 = sgbm_byte(vv, prow, nvv, nprow, j - g.minX2 + g.w2);
            const int c0 = max(max(0, u - v1), v0 - u), c1 = max(max(0, v - u1), u0 - v);
            cost += min(c0, c1) >> (c ? 2 : 0);
        }
        out[i] = (short)cost;
    }
}

// The SAD window (stereosgbm.cpp:392-516): C = P2 + the (2*SW2+1) x (2*SH2+1) sum of the pixel costs with clamped row and
// column indices.  The reference pre-adds P2 to the first row of its volume only and never writes column 0 of the other
// rows nor the last SH2 rows (there the window's lower edge leaves the image): those keep the allocation's zero.
__global__ void sgbm_window_kernel(const short *__restrict__ pix, SgbmGeom g, short *__restrict__ C)
{
    const size_t n = (size_t)g.w1 * g.D;
    const int y = blockIdx.y;
    short *out = C + (size_t)y * n;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int x = (int)(i / g.D), d = (int)(i - (size_t)x * g.D);
        int s = 0;
        if (y == 0 || (x > 0 && y + g.SH2 < g.h)) {
            s = g.P2;
            for (int dy = -g.SH2; dy <= g.SH2; dy++) {
                const short *row = pix + (size_t)min(max(y + dy, 0), g.h - 1) * n + d;
                for (int dx = -g.SW2; dx <= g.SW2; dx++) s += row[(size_t)min(max(x + dx, 0), g.w1 - 1) * g.D];
            }
        }
        out[i] = (short)s;
    }
}

// One of the 8 scanline passes (stereosgbm.cpp:524-661): a warp walks one line of the volume in steps (sx, sy), labels
// across the lanes, the previous pixel's L in shared memory with SHRT_MAX sentinels at d = -1 and d = D; a predecessor
// outside the volume has L = 0 and min L = 0 (the reference's memset borders).  Every L lies in [C - P2, C] and is exact
// in int32 (host bound, DESIGN.md section 3.5): where C carries P2 all 8 L of a pixel are >= 0, where C = 0 they are all
// in [-P2, 0], so S = min(S + L, SHRT_MAX) is the reference's saturating sum in any order.
__global__ void sgbm_path_kernel(const short *__restrict__ C, SgbmGeom g, int sx, int sy, short *__restrict__ S)
{
    extern __shared__ int sgbm_lbuf[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, D = g.D, W = g.w1, H = g.h;
    int *prev = sgbm_lbuf + (size_t)wib * 2 * (D + 2), *cur = prev + (D + 2);
    const int line = blockIdx.x * (blockDim.x >> 5) + wib;
    int x, y;
    if (sy == 0) {
        if (line >= H) return;
        x = sx > 0 ? 0 : W - 1; y = line;
    } else if (sx == 0) {
        if (line >= W) return;
        x = line; y = sy > 0 ? 0 : H - 1;
    } else {
        if (line >= W + H - 1) return;
        if (line < W) { x = line; y = sy > 0 ? 0 : H - 1; }
        else { x = sx > 0 ? 0 : W - 1; y = (sy > 0 ? 0 : H - 1) + sy * (line - W + 1); }
    }
    for (int d = lane; d < D + 2; d += 32) {
        prev[d] = (d == 0 || d == D + 1) ? kSgbmMaxCost : 0;
        cur[d] = (d == 0 || d == D + 1) ? kSgbmMaxCost : 0;
    }
    __syncwarp();
    int minPrev = 0;
    for (; x >= 0 && x < W && y >= 0 && y < H; x += sx, y += sy) {
        const size_t base = ((size_t)y * W + x) * D;
        const int delta = minPrev + g.P2;
        int m = kSgbmMaxCost;
        for (int d = lane; d < D; d += 32) {
            const int lp = min(min(prev[d + 1], delta), min(prev[d], prev[d + 2]) + g.P1);
            const int L = C[base + d] + lp - delta;
            cur[d + 1] = L;
            m = min(m, L);
            S[base + d] = (short)min(S[base + d] + L, kSgbmMaxCost);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = min(m, __shfl_xor_sync(0xffffffffu, m, o));
        minPrev = m;
        __syncwarp();
        int *t = prev; prev = cur; cur = t;
    }
}

// Right-view candidate of the reference's descending-x loop (stereosgbm.cpp:782-786: strict `>`, so the largest x wins a
// tie): the smallest packed (minS + 32768, 0xFFFFFFFF - x) per right column.  S is negative where C = 0.
constexpr unsigned long long kSgbmNoMatch = ~0ull;

// WTA of one pixel per warp (stereosgbm.cpp:672-800): the first minimum of S below SHRT_MAX (none: bestDisp = -1),
// the uniqueness test, the parabola with C integer division, and the right view's candidate.
__global__ void sgbm_wta_kernel(const short *__restrict__ S, SgbmGeom g, short *__restrict__ disp1,
                                unsigned long long *__restrict__ d2key)
{
    const int lane = threadIdx.x & 31;
    const size_t pw = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (pw >= (size_t)g.w1 * g.h) return;
    const int y = (int)(pw / g.w1), x = (int)(pw - (size_t)y * g.w1), D = g.D;
    const short *Sp = S + pw * D;
    unsigned best = 0xffffffffu;                              // (S + 32768) << 16 | d
    for (int d = lane; d < D; d += 32) {
        const int s = Sp[d];
        if (s < kSgbmMaxCost) best = min(best, ((unsigned)(s + 32768) << 16) | (unsigned)d);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
    const int minS = best == 0xffffffffu ? kSgbmMaxCost : (int)(best >> 16) - 32768;
    const int bestDisp = best == 0xffffffffu ? -1 : (int)(best & 0xffffu);
    bool reject = false;
    for (int d = lane; d < D; d += 32)
        if (Sp[d] * (100 - kSgbmUniqueness) < minS * 100 && abs(bestDisp - d) > 1) reject = true;
    if (__any_sync(0xffffffffu, reject) || lane != 0) return;
    int d = bestDisp;
    const int X = x + g.minX1, x2 = X - d - g.minD;
    if (x2 >= 0)                                              // x2 < 0: outside the reference's disp2 buffers (DESIGN.md section 4)
        atomicMin(d2key + (size_t)y * g.wp + x2, ((unsigned long long)(minS + 32768) << 32) | (0xffffffffu - (unsigned)x));
    if (0 < d && d < D - 1) {
        const int sm1 = Sp[d - 1], sp1 = Sp[d + 1], s0 = Sp[d];
        const int denom2 = max(sm1 + sp1 - 2 * s0, 1);
        d = d * 16 + ((sm1 - sp1) * 16 + denom2) / (denom2 * 2);
    } else d *= 16;
    disp1[(size_t)y * g.wp + X] = (short)(d + g.minD * 16);
}

__global__ void sgbm_fill_kernel(short *__restrict__ p, size_t n, short v)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v;
}

// LR check (stereosgbm.cpp:802-816) with disp12MaxDiff = lr, the right view decoded from the packed candidates
__global__ void sgbm_lr_kernel(short *__restrict__ disp1, const unsigned long long *__restrict__ d2key, SgbmGeom g, int lr)
{
    const int xi = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (xi >= g.w1) return;
    const int X = xi + g.minX1, invalid = (g.minD - 1) * 16;
    short *row = disp1 + (size_t)y * g.wp;
    const int d1 = row[X];
    if (d1 == invalid) return;
    const unsigned long long *k = d2key + (size_t)y * g.wp;
    auto disp2 = [&](int c) -> int {
        const unsigned long long key = k[c];
        if (key == kSgbmNoMatch) return invalid;
        const int x = (int)(0xffffffffu - (unsigned)(key & 0xffffffffu));
        return x + g.minX1 - c;                               // d + minD of the winning pixel
    };
    const int d0 = d1 >> 4, dc = (d1 + 15) >> 4;
    const int xa = X - d0, xb = X - dc;
    if (0 <= xa && xa < g.wp && disp2(xa) >= g.minD && abs(disp2(xa) - d0) > lr &&
        0 <= xb && xb < g.wp && disp2(xb) >= g.minD && abs(disp2(xb) - dc) > lr)
        row[X] = (short)invalid;
}

__device__ __forceinline__ void sgbm_sort2(int &a, int &b) { const int t = min(a, b); b = max(a, b); a = t; }
// medianBlur(disp, disp, 3) on int16 (smooth.cpp:224-270): replicated border, the reference's sorting network
__global__ void sgbm_median_kernel(const short *__restrict__ in, int w, int h, short *__restrict__ out)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const int xm = max(x - 1, 0), xp = min(x + 1, w - 1);
    const short *r0 = in + (size_t)max(y - 1, 0) * w, *r1 = in + (size_t)y * w, *r2 = in + (size_t)min(y + 1, h - 1) * w;
    int p0 = r0[xm], p1 = r0[x], p2 = r0[xp], p3 = r1[xm], p4 = r1[x], p5 = r1[xp], p6 = r2[xm], p7 = r2[x], p8 = r2[xp];
    sgbm_sort2(p1, p2); sgbm_sort2(p4, p5); sgbm_sort2(p7, p8); sgbm_sort2(p0, p1);
    sgbm_sort2(p3, p4); sgbm_sort2(p6, p7); sgbm_sort2(p1, p2); sgbm_sort2(p4, p5);
    sgbm_sort2(p7, p8); sgbm_sort2(p0, p3); sgbm_sort2(p5, p8); sgbm_sort2(p4, p7);
    sgbm_sort2(p3, p6); sgbm_sort2(p1, p4); sgbm_sort2(p2, p5); sgbm_sort2(p4, p7);
    sgbm_sort2(p4, p2); sgbm_sort2(p6, p4); sgbm_sort2(p4, p2);
    out[(size_t)y * w + x] = (short)p4;
}

// filterSpeckles (stereosgbm.cpp:869-983): 4-connected components of the pixels != newVal whose neighbours differ by at
// most kSgbmSpeckleRange.  The relation is symmetric, so the components do not depend on the reference's scan order.
__global__ void sgbm_speckle_init_kernel(const short *__restrict__ d, int n, int newVal, int *__restrict__ lab,
                                         int *__restrict__ area)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { lab[i] = d[i] != newVal ? i : -1; area[i] = 0; }
}
__global__ void sgbm_speckle_link_kernel(const short *__restrict__ d, int w, int h, int newVal, int *lab)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const int i = y * w + x, a = d[i];
    if (a == newVal) return;
    if (x + 1 < w && d[i + 1] != newVal && abs(a - d[i + 1]) <= kSgbmSpeckleRange) uf_union(lab, i, i + 1);
    if (y + 1 < h && d[i + w] != newVal && abs(a - d[i + w]) <= kSgbmSpeckleRange) uf_union(lab, i, i + w);
}
// speckles -> newVal, then the crop of sgbm.cpp:210 and its conversion (sgbm.cpp:221-234): -d/16, NaN for newVal.
// An image without a single valid pixel (undefined in the reference) comes out all NaN.
__global__ void sgbm_output_kernel(const short *__restrict__ d, const int *__restrict__ lab, const int *__restrict__ area,
                                   int wp, int off, int w, int h, int newVal, const SgbmState *__restrict__ st,
                                   float *__restrict__ out)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const int i = y * wp + x + off, r = lab[i];
    int v = d[i];
    if (r >= 0 && area[r] <= kSgbmSpeckleWindow) v = newVal;
    out[(size_t)y * w + x] = (v == newVal || st->n == 0) ? __int_as_float(0x7fc00000) : -(float)v * 0.0625f;
}

}  // namespace s2pb
