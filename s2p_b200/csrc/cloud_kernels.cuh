// cloud_kernels.cuh -- the last per-tile step of s2p: the kept points of a cloud packed into the vertex records of the PLY
// file that s2p.triangulation.write_to_ply writes (s2p/triangulation.py:392-429, s2p/ply.py:24-69), with the colours of
// common.linear_stretching_and_quantization_8bit (s2p/common.py:284-297) formed on the fly.
//
//   stretch   -> a, b = np.nanpercentile(img, (p, 100 - p)) by the radix select of sgbm_kernels.cuh (rule kOrdLinear, run by sgbm.cu), then
//                round(255 * (clip(v, a, b) - a) / (b - a)) in double, NaN -> 0 (DESIGN.md section 3.4)
//   keep      -> x, y and z finite (np.all(np.isfinite(xyz), axis=1)): one count per CTA tile, one exclusive scan of the counts
//   pack      -> each CTA stages its records in shared memory at the byte offset they have in the output modulo 16, then
//                writes the 16-byte chunks that lie wholly inside its range with 16-byte stores and the two ragged ends
//                byte by byte, so neighbouring CTAs never store to the same byte
// A record is x, y, z float64, then red, green, blue (and ir), then confidence float32, packed without padding.  The colours
// are either stretched to uint8, or copied byte for byte from colour planes of one PLY type of 1, 2, 4 or 8 bytes (a `clr`
// image's own type: float colours keep their bits, NaN included).  Records of up to kPlyMaxRecord bytes are packed by CTAs of
// kPlyTile points; wider ones (up to kPlyMaxWide) by CTAs of half as many, so that the stage stays within static shared memory.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "order_stats.h"

namespace s2pb {

constexpr int kPlyThreads = 256;
constexpr int kPlyPer = 4;                               // points per thread
constexpr int kPlyTile = kPlyThreads * kPlyPer;          // points per CTA
constexpr int kPlyMaxRecord = 32;                        // 24 + 4 uint8 colours + 4 confidence
constexpr int kPlyPerWide = 2;                           // points per thread of the wide records
constexpr int kPlyMaxWide = 60;                          // 24 + 4 float64 colours + 4 confidence

// one value of common.linear_stretching_and_quantization_8bit with the bounds a, b (float64, as numpy forms them):
// np.clip as its float loop does it (max then min, a NaN operand propagates), then the expression in double, np.round
// (half to even) and astype(uint8) (NaN -> 0; every other value lies in [0, 255])
__device__ __forceinline__ uint8_t stretch_8bit(float f, double a, double b)
{
    const double x = (double)f;
    const double t = isnan(x) ? x : (x > a ? x : a);
    const double c = isnan(t) ? t : (t < b ? t : b);
    const double v = rint(__ddiv_rn(__dmul_rn(255.0, __dsub_rn(c, a)), __dsub_rn(b, a)));
    return isnan(v) ? 0 : (uint8_t)(int)v;
}

// the stretched image on its own (s2pb_stretch_8bit): n values, bounds from the select
__global__ void stretch_8bit_kernel(const float *__restrict__ im, size_t n, const OrderStats *__restrict__ os,
                                    uint8_t *__restrict__ out)
{
    const double a = os->lo, b = os->hi;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        out[i] = stretch_8bit(im[i], a, b);
}

__device__ __forceinline__ bool ply_keep(const double *__restrict__ xyz, size_t i)
{
    return isfinite(xyz[3 * i]) && isfinite(xyz[3 * i + 1]) && isfinite(xyz[3 * i + 2]);
}

// kept points of each CTA tile of kPlyThreads * Per points
template <int Per>
__global__ void __launch_bounds__(kPlyThreads) ply_count_kernel(const double *__restrict__ xyz, size_t n, int *__restrict__ counts)
{
    const size_t base = (size_t)blockIdx.x * (kPlyThreads * Per);
    int c = 0;
#pragma unroll
    for (int k = 0; k < Per; k++) {
        const size_t i = base + k * kPlyThreads + threadIdx.x;
        c += i < n && ply_keep(xyz, i);
    }
    c = __reduce_add_sync(0xffffffffu, c);
    __shared__ int ws[kPlyThreads / 32];
    if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        int s = 0;
        for (int w = 0; w < kPlyThreads / 32; w++) s += ws[w];
        counts[blockIdx.x] = s;
    }
}

// inclusive scan of one value per thread of the CTA (blockDim.x == 1024)
__device__ __forceinline__ long long block_scan_1024(long long v, long long *ws)
{
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const long long u = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += u;
    }
    if (lane == 31) ws[wid] = v;
    __syncthreads();
    if (wid == 0) {
        long long s = ws[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const long long u = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += u;
        }
        ws[lane] = s;
    }
    __syncthreads();
    const long long r = v + (wid ? ws[wid - 1] : 0);
    __syncthreads();
    return r;
}

// one CTA of 1024 threads: offsets[k] = counts[0] + ... + counts[k-1] (the tiles in row-major order), *total = the sum
__global__ void __launch_bounds__(1024) ply_scan_kernel(const int *__restrict__ counts, int ntiles, long long *__restrict__ offsets,
                                                        long long *__restrict__ total)
{
    __shared__ long long ws[32];
    __shared__ long long chunk;
    long long base = 0;
    for (int b = 0; b < ntiles; b += 1024) {
        const int i = b + threadIdx.x;
        const long long v = i < ntiles ? counts[i] : 0;
        const long long inc = block_scan_1024(v, ws);
        if (i < ntiles) offsets[i] = base + inc - v;
        if (threadIdx.x == 1023) chunk = inc;
        __syncthreads();
        base += chunk;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = base;
}

struct PlyPackParams {
    const double *xyz;          // n points of three float64
    size_t n;
    const long long *offsets;   // per CTA tile: the kept points before it (ply_scan_kernel)
    int nbands;                 // 0 (no colour), 1 (grey, written three times), 3 or 4
    int cb;                     // bytes of one colour value: 1, 2, 4 or 8 (1 when stretched)
    const uint8_t *colors;      // nbands planes of n values of cb bytes, copied as they are, or null: ...
    const float *bands;         // ... nbands planes of n float32, stretched to uint8 with the bounds of *os
    const OrderStats *os;
    const float *conf;          // n float32, or null (no confidence property)
    int rb;                     // record bytes
    uint8_t *out;               // the records of the kept points, in point order
};

__device__ __forceinline__ void put_bytes(uint8_t *dst, const void *src, int nb)
{
    const uint8_t *s = (const uint8_t *)src;
    for (int k = 0; k < nb; k++) dst[k] = s[k];
}

// CTA tiles of kPlyThreads * Per points with records of at most MaxRecord bytes: <kPlyPer, kPlyMaxRecord> or
// <kPlyPerWide, kPlyMaxWide>
template <int Per, int MaxRecord>
__global__ void __launch_bounds__(kPlyThreads) ply_pack_kernel(const PlyPackParams P)
{
    __shared__ __align__(16) uint8_t stage[kPlyThreads * Per * MaxRecord + 16];
    __shared__ int ws[kPlyThreads / 32 + 1];
    const size_t base = (size_t)blockIdx.x * (kPlyThreads * Per);
    const size_t gstart = (size_t)P.offsets[blockIdx.x] * P.rb;
    const int shift = (int)(gstart & 15);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int ncol = P.nbands == 4 ? 4 : P.nbands ? 3 : 0;
    double a = 0.0, b = 0.0;
    if (!P.colors && P.nbands) { a = P.os->lo; b = P.os->hi; }
    int before = 0;                                          // kept points of this tile in earlier rounds
    for (int k = 0; k < Per; k++) {
        const size_t i = base + (size_t)k * kPlyThreads + threadIdx.x;
        const bool keep = i < P.n && ply_keep(P.xyz, i);
        // rank of this point among the kept ones of the round: warp ballot, then the warps before it
        const unsigned m = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) ws[wid] = __popc(m);
        __syncthreads();
        if (threadIdx.x == 0) {
            int s = 0;
            for (int w = 0; w < kPlyThreads / 32; w++) { const int c = ws[w]; ws[w] = s; s += c; }
            ws[kPlyThreads / 32] = s;
        }
        __syncthreads();
        if (keep) {
            const int j = before + ws[wid] + __popc(m & ((1u << lane) - 1));
            uint8_t *r = stage + shift + (size_t)j * P.rb;
            put_bytes(r, P.xyz + 3 * i, 24);
            if (ncol && P.colors) {
                for (int q = 0; q < ncol; q++) {
                    const int band = P.nbands == 1 ? 0 : q;
                    put_bytes(r + 24 + q * P.cb, P.colors + ((size_t)band * P.n + i) * P.cb, P.cb);
                }
            } else if (ncol) {
                uint8_t c[4];
                for (int q = 0; q < ncol; q++) {
                    const int band = P.nbands == 1 ? 0 : q;
                    c[q] = stretch_8bit(P.bands[(size_t)band * P.n + i], a, b);
                }
                put_bytes(r + 24, c, ncol);
            }
            if (P.conf) put_bytes(r + 24 + ncol * P.cb, P.conf + i, 4);
        }
        before += ws[kPlyThreads / 32];
        __syncthreads();
    }
    // the tile's bytes [gstart, gend): whole 16-byte chunks by 16-byte stores, the ragged ends byte by byte
    const size_t gend = gstart + (size_t)before * P.rb;
    const size_t A = (gstart + 15) & ~(size_t)15, B = gend & ~(size_t)15;
    const size_t g0 = gstart & ~(size_t)15;                  // stage[g - g0] holds byte g
    if (A < B) {
        for (size_t g = A + 16 * (size_t)threadIdx.x; g < B; g += 16 * kPlyThreads)
            *(uint4 *)(P.out + g) = *(const uint4 *)(stage + (g - g0));
        for (size_t g = gstart + threadIdx.x; g < A; g += kPlyThreads) P.out[g] = stage[g - g0];
        for (size_t g = B + threadIdx.x; g < gend; g += kPlyThreads) P.out[g] = stage[g - g0];
    } else {
        for (size_t g = gstart + threadIdx.x; g < gend; g += kPlyThreads) P.out[g] = stage[g - g0];
    }
}

}  // namespace s2pb
