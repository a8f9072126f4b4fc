// homography_kernels.cuh -- the rectification warp (SURVEY.md row a13): order-5 B-spline resampling of an
// image through a homography, with the reference's anti-aliasing rule.
//
// Behavioural reference, paths under $REF/3rdparty/homography ($REF: the root of the s2p sources): LibHomography/Homography.cpp:50-168
// (mapImage), Splines.cpp:26-121 (prefilter), :125-211 (36-tap interpolation), :215-227 (weights),
// :234-399 (recursions), LibImages/LibImages.cpp:506-687 (Gaussian of the anti-aliasing branch).
// The reference is float32 with SSE; built with -O3 -march=native its result depends on FMA contraction
// (two builds of the same sources differ by up to 6e-5 of the dynamic range), so parity for this stage is a
// stated tolerance (tests/test_gpu_homography.py), not bit equality.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace s2pb {

// NaN -> 0 (prepareSpline, Splines.cpp:34-45; isNumber is x == x, so infinities stay)
__global__ void nan_to_zero_kernel(float *a, size_t n)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { float v = a[i]; if (!(v == v)) a[i] = 0.f; }
}

__global__ void transpose_kernel(const float *__restrict__ in, int w, int h, float *__restrict__ out)
{   // out[x][y] = in[y][x]
    __shared__ float t[32][33];
    int x = blockIdx.x * 32 + threadIdx.x, y0 = blockIdx.y * 32;
    for (int k = threadIdx.y; k < 32; k += blockDim.y)
        if (x < w && y0 + k < h) t[k][threadIdx.x] = in[(size_t)(y0 + k) * w + x];
    __syncthreads();
    int ox = blockIdx.y * 32 + threadIdx.x, oy0 = blockIdx.x * 32;
    for (int k = threadIdx.y; k < 32; k += blockDim.y)
        if (ox < h && oy0 + k < w) out[(size_t)(oy0 + k) * h + ox] = t[threadIdx.x][k];
}

// applySpline (Splines.cpp:234-270) down every column of a w x h image, one thread per column (coalesced across
// the warp): scale by lambda, then for each of the two poles a forward and a backward recursion whose start values
// come from initForward (:315-340, a full-length weighted sum) and initBackward (:375-384).  The recursions are
// sequential in k, exactly as in the reference; rows are moved in register blocks of kSplineBlk so that the
// global-memory latency is paid once per block instead of once per row.
constexpr int kSplineBlk = 16;
__global__ void spline_columns_kernel(float *__restrict__ a, int w, int h, float lambda, double z0, double z1)
{
    int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= w) return;
    float *v = a + x;
    const size_t st = (size_t)w;
    float buf[kSplineBlk];
    for (int n = 0; n < 2; n++) {
        const double pz = n == 0 ? z0 : z1;
        const float zn = (float)pz;
        // every applySpline call scales the line by lambda first; the second pole sees the line already scaled
        const float scale = n == 0 ? lambda : 1.f;
        // initForward: sum = v[0] + z^(h-1) v[h-1] + sum_k (z^k + z^(2h-2-k)) v[k]
        double zk = pz, iz = 1.0 / pz, z2k = pow(pz, (double)(h - 1));
        float sum = v[0] * scale + (float)z2k * (v[(size_t)(h - 1) * st] * scale);
        z2k = z2k * z2k * iz;
        for (int k0 = 1; k0 < h - 1; k0 += kSplineBlk) {
            const int m = min(kSplineBlk, h - 1 - k0);
#pragma unroll
            for (int q = 0; q < kSplineBlk; q++) if (q < m) buf[q] = v[(size_t)(k0 + q) * st] * scale;
#pragma unroll
            for (int q = 0; q < kSplineBlk; q++)
                if (q < m) { sum = fmaf((float)(zk + z2k), buf[q], sum); zk *= pz; z2k *= iz; }
        }
        sum = __fdiv_rn(sum, (float)(1.0 - zk * zk));
        // forward recursion (also applies the scale of the first pole in place)
        v[0] = sum;
        for (int k0 = 1; k0 < h; k0 += kSplineBlk) {
            const int m = min(kSplineBlk, h - k0);
#pragma unroll
            for (int q = 0; q < kSplineBlk; q++) if (q < m) buf[q] = v[(size_t)(k0 + q) * st] * scale;
#pragma unroll
            for (int q = 0; q < kSplineBlk; q++) if (q < m) { sum = fmaf(zn, sum, buf[q]); buf[q] = sum; }
#pragma unroll
            for (int q = 0; q < kSplineBlk; q++) if (q < m) v[(size_t)(k0 + q) * st] = buf[q];
        }
        // initBackward + backward recursion
        sum = (float)(pz / (pz * pz - 1.0)) * fmaf((float)pz, v[(size_t)(h - 2) * st], v[(size_t)(h - 1) * st]);
        v[(size_t)(h - 1) * st] = sum;
        for (int k0 = h - 2; k0 >= 0; k0 -= kSplineBlk) {
            const int m = min(kSplineBlk, k0 + 1);
#pragma unroll
            for (int q = 0; q < kSplineBlk; q++) if (q < m) buf[q] = v[(size_t)(k0 - q) * st];
#pragma unroll
            for (int q = 0; q < kSplineBlk; q++) if (q < m) { sum = zn * (sum - buf[q]); buf[q] = sum; }
#pragma unroll
            for (int q = 0; q < kSplineBlk; q++) if (q < m) v[(size_t)(k0 - q) * st] = buf[q];
        }
    }
}

// The same prefilter, one pole per launch, parallel ALONG the line as well: the poles are small (|z| = 0.43 and
// 0.043), so the state of either recursion forgets its past at the rate |z|^k -- below 2e-12 after kSplineWarm = 32
// samples, five orders of magnitude under float32 resolution.  A thread therefore owns kSplineSeg consecutive
// samples of one column: it runs the forward recursion from a zero state kSplineWarm samples early (the first
// segment starts from initForward's weighted sum instead, whose terms beyond 48 samples are below half an ulp),
// keeps the forward values of its segment plus kSplineWarm more in registers, and runs the backward recursion from
// a zero state that far beyond its end (the last segment from initBackward's exact start value).  w x (h / 64)
// threads instead of w, and no global-memory latency chain: the 2250-column anti-aliasing case drops from 3.6 ms
// per launch to tens of microseconds.  Out of place (in -> out); lines shorter than 2 * kSplineSeg use the
// sequential kernel above.  Both kernels need lines of kSplineMinSide samples at least (map_image refuses shorter ones).
constexpr int kSplineSeg = 64, kSplineWarm = 32, kSplineMinSide = 4;
__global__ void __launch_bounds__(128) spline_segments_kernel(const float *__restrict__ in, float *__restrict__ out, int w, int h,
                                                             float scale, double pz)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= w) return;
    const int s = blockIdx.y * kSplineSeg;
    const int e = min(s + kSplineSeg, h);            // my samples: [s, e)
    const int e2 = min(e + kSplineWarm, h);          // forward values kept for [s, e2)
    const float zn = (float)pz;
    const float *v = in + x;
    const size_t st = (size_t)w;
    float f[kSplineSeg + kSplineWarm];
    float state;
    if (s == 0) {            // initForward (Splines.cpp:315-340): v[0] + sum_k z^k v[k] (+ mirrored terms, < 1e-20 here)
        double zk = pz;
        state = v[0] * scale;
        const int K = min(h - 2, 48);
        for (int k = 1; k <= K; k++) { state = fmaf((float)zk, v[(size_t)k * st] * scale, state); zk *= pz; }
    } else {                 // zero state kSplineWarm samples early, then the recursion proper
        state = 0.f;
#pragma unroll 8
        for (int k = s - kSplineWarm; k < s; k++) state = fmaf(zn, state, v[(size_t)k * st] * scale);
        state = fmaf(zn, state, v[(size_t)s * st] * scale);
    }
    f[0] = state;
#pragma unroll
    for (int q = 1; q < kSplineSeg + kSplineWarm; q++) {
        if (s + q < e2) state = fmaf(zn, state, v[(size_t)(s + q) * st] * scale);
        f[q] = state;
    }
    // backward: y[k] = z (y[k+1] - f[k]); exact start at the end of the line, zero state beyond an interior segment
    float b;
    float *o = out + x;
    if (e2 == h) {
        // initBackward (Splines.cpp:375-384) from the last two forward values
        float last = 0.f, prev = 0.f;
#pragma unroll
        for (int q = 0; q < kSplineSeg + kSplineWarm; q++) { if (s + q == h - 1) last = f[q]; if (s + q == h - 2) prev = f[q]; }
        b = (float)(pz / (pz * pz - 1.0)) * fmaf((float)pz, prev, last);
        // o[h-1] is written by the segment that holds h-2, the only one with both values: when h = 64k + 1 the last
        // segment is the single sample h-1, and its forward value at h-2 (prev) would be missing
        if (s <= h - 2 && h - 2 < e) o[(size_t)(h - 1) * st] = b;
#pragma unroll
        for (int q = kSplineSeg + kSplineWarm - 1; q >= 0; q--) {
            const int k = s + q;
            if (k <= h - 2) { b = zn * (b - f[q]); if (k < e) o[(size_t)k * st] = b; }
        }
    } else {
        b = 0.f;
#pragma unroll
        for (int q = kSplineSeg + kSplineWarm - 1; q >= 0; q--) {
            b = zn * (b - f[q]);
            if (q < kSplineSeg) o[(size_t)(s + q) * st] = b;      // s + q < e always holds for an interior segment
        }
    }
}

__device__ __forceinline__ float pow5f(float x) { float x2 = x * x; return x2 * x2 * x; }
__device__ __forceinline__ void init_spline5(float w[6], float t)
{   // Splines.cpp:215-227
    const float ak[6] = {(float)(1. / 120.), (float)-0.05, (float)0.125, (float)(-1. / 6.), (float)0.125, (float)-0.05};
    const float p0 = pow5f(t), p1 = pow5f(t + 1), p2 = pow5f(t + 2), p3 = pow5f(t + 3), p4 = pow5f(t + 4), p5 = pow5f(t + 5);
    w[0] = p0 * ak[0];
    w[1] = p0 * ak[1] + p1 * ak[0];
    w[2] = p0 * ak[2] + p1 * ak[1] + p2 * ak[0];
    w[3] = p0 * ak[3] + p1 * ak[2] + p2 * ak[1] + p3 * ak[0];
    w[4] = p0 * ak[4] + p1 * ak[3] + p2 * ak[2] + p3 * ak[1] + p4 * ak[0];
    w[5] = p0 * ak[5] + p1 * ak[4] + p2 * ak[3] + p3 * ak[2] + p4 * ak[1] + p5 * ak[0];
}
__device__ __forceinline__ int symi(int x, int w) { return x < 0 ? -x - 1 : (x >= w ? 2 * w - x - 1 : x); }

struct Mat9 { double m[9]; };

// The per-pixel loop of mapImage (Homography.cpp:125-135) + interpolateSpline (Splines.cpp:125-211):
// (x, y) = Hinv (j, i, 1) in double, sampled at (x + 0.5, y + 0.5) converted to float; outside [0,w] x [0,h] -> NaN.
__global__ void spline_warp_kernel(const float *__restrict__ coef, int w, int h, Mat9 Hinv, float *__restrict__ out, int ow, int oh)
{
    int j = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y * blockDim.y + threadIdx.y;
    if (j >= ow || i >= oh) return;
    double xd = Hinv.m[0] * j + Hinv.m[1] * i + Hinv.m[2];
    double yd = Hinv.m[3] * j + Hinv.m[4] * i + Hinv.m[5];
    double zd = Hinv.m[6] * j + Hinv.m[7] * i + Hinv.m[8];
    xd = xd / zd; yd = yd / zd;
    const float px = (float)(xd + 0.5), py = (float)(yd + 0.5);
    float r;
    if (px < 0.f || px > (float)w || py < 0.f || py > (float)h || !(px == px) || !(py == py)) r = __int_as_float(0x7fc00000);
    else {
        const float x = px - 0.5f, y = py - 0.5f;
        const int xi = x < 0 ? -1 : (int)x, yi = y < 0 ? -1 : (int)y;
        float cx[6], cy[6];
        init_spline5(cx, x - (float)xi);
        init_spline5(cy, y - (float)yi);
        if (xi >= 2 && xi < w - 3 && yi >= 2 && yi < h - 3) {
            // interior: the reference's SSE grouping -- four columns xi-2..xi+1 accumulated over the rows, weighted
            // by cx[5..2] at the end, plus the two remaining columns summed row by row
            float c0 = 0.f, c1 = 0.f, c2 = 0.f, c3 = 0.f, value = 0.f;
#pragma unroll
            for (int d = 0; d < 6; d++) {
                const float *row = coef + (size_t)(yi - 2 + d) * w + xi;
                const float wy = cy[5 - d];
                const float t0 = wy * row[-2], t1 = wy * row[-1], t2 = wy * row[0], t3 = wy * row[1];
                c0 = d == 0 ? t0 : c0 + t0; c1 = d == 0 ? t1 : c1 + t1; c2 = d == 0 ? t2 : c2 + t2; c3 = d == 0 ? t3 : c3 + t3;
                const float tt = wy * (row[2] * cx[1] + row[3] * cx[0]);
                value = d == 0 ? tt : value + tt;
            }
            r = value + cx[5] * c0 + cx[4] * c1 + cx[3] * c2 + cx[2] * c3;
        } else {
            float value = 0.f;
            for (int d = -2; d <= 3; d++) {
                int yy = yi + d;
                yy = yy < 0 ? -yy - 1 : (yy >= h ? 2 * h - yy - 1 : yy);
                const float *row = coef + (size_t)yy * w;
                value += cy[3 - d] * (row[symi(xi - 2, w)] * cx[5] + row[symi(xi - 1, w)] * cx[4] + row[symi(xi, w)] * cx[3] +
                                      row[symi(xi + 1, w)] * cx[2] + row[symi(xi + 2, w)] * cx[1] + row[symi(xi + 3, w)] * cx[0]);
            }
            r = value;
        }
    }
    out[(size_t)i * ow + j] = r;
}

// anti-aliasing branch: the NaN mask of the TRUE homography goes back on (Homography.cpp:139-167)
__global__ void warp_mask_kernel(float *__restrict__ out, int ow, int oh, Mat9 Hinv, int w, int h)
{
    int j = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y * blockDim.y + threadIdx.y;
    if (j >= ow || i >= oh) return;
    double x = Hinv.m[0] * j + Hinv.m[1] * i + Hinv.m[2];
    double y = Hinv.m[3] * j + Hinv.m[4] * i + Hinv.m[5];
    double z = Hinv.m[6] * j + Hinv.m[7] * i + Hinv.m[8];
    x /= z; y /= z;
    if (x < 0 || x >= w || y < 0 || y >= h) out[(size_t)i * ow + j] = __int_as_float(0x7fc00000);
}

// Image::convolveGaussian (LibImages.cpp:506-687): separable, borders replicated.
struct GaussKernel { float k[64]; int size; };
__global__ void gauss_rows_kernel(const float *__restrict__ in, float *__restrict__ out, int w, int h, GaussKernel K)
{
    int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const int half = K.size / 2;
    const float *row = in + (size_t)y * w;
    float v = 0.f;
    for (int k = 0; k < K.size; k++) { int xx = min(max(x + k - half, 0), w - 1); v += K.k[k] * row[xx]; }
    out[(size_t)y * w + x] = v;
}
// vertical pass; columns at and beyond `jlim` reproduce the reference's scalar tail, which stores the
// UNFILTERED buffer entry col[i] = row max(i - half, 0) instead of the filtered value (LibImages.cpp:655-670)
__global__ void gauss_cols_kernel(const float *__restrict__ in, float *__restrict__ out, int w, int h, GaussKernel K, int jlim)
{
    int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const int half = K.size / 2;
    float v;
    if (x >= jlim) v = in[(size_t)max(y - half, 0) * w + x];
    else {
        v = 0.f;
        for (int k = 0; k < K.size; k++) { int yy = min(max(y + k - half, 0), h - 1); v += K.k[k] * in[(size_t)yy * w + x]; }
    }
    out[(size_t)y * w + x] = v;
}

}  // namespace s2pb
