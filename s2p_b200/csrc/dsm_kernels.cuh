// Rasterisation of point clouds into a DSM: plyflatten_from_plyfiles_list with radius 0 and no sigma, the last step of
// s2p's plys_to_dsm (s2p/__init__.py:432-476).  Points arrive as the raw vertex records of binary little-endian PLY files
// and are converted on the device.  Per cell and channel the reference accumulates, in point order,
// acc = (float)((double)acc + 1.0 * v) with a float acc, and cnt += 1.0f; the cell's value is acc / cnt in float, NaN where no
// point fell.  Float atomics would reorder that fold, so the points are sorted by cell instead (a stable radix sort over the
// cell key, the point index riding along) and each cell's run is folded by one thread, in point order.
#pragma once
#include <cstdint>

#include "../../include/s2pb200.h"

namespace s2pb {

constexpr int kDsmMaxCols = 16;                  // x, y and up to 14 channels

struct DsmParams {
    const uint8_t *rec;                          // all clouds' records back to back, record_bytes each
    uint32_t n;                                  // points
    int rb;                                      // record_bytes
    int ncols;                                   // x, y, then the channels
    int off[kDsmMaxCols], type[kDsmMaxCols];     // byte offset in the record and S2PB_PLY_* type of each property
    double xoff, yoff, r;
    int xsize, ysize;
    uint32_t ncells;                             // xsize * ysize: also the key of a skipped point, so skipped points sort last
};

// one property of a record as float64 (exact for every type the descriptor allows); records are packed, so byte loads
__device__ __forceinline__ double dsm_load(const uint8_t *p, int type)
{
    if (type == S2PB_PLY_U8) return (double)p[0];
    if (type == S2PB_PLY_F32 || type == S2PB_PLY_I32 || type == S2PB_PLY_U32) {
        const uint32_t u = (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24;
        return type == S2PB_PLY_F32 ? (double)__uint_as_float(u) : type == S2PB_PLY_U32 ? (double)u : (double)(int32_t)u;
    }
    if (type == S2PB_PLY_I8) return (double)(int8_t)p[0];
    if (type == S2PB_PLY_U16 || type == S2PB_PLY_I16) {
        const uint16_t u = (uint16_t)(p[0] | p[1] << 8);
        return type == S2PB_PLY_U16 ? (double)u : (double)(int16_t)u;
    }
    unsigned long long u = 0;
#pragma unroll
    for (int b = 7; b >= 0; b--) u = u << 8 | p[b];
    return __longlong_as_double((long long)u);
}

// the cell of each point: (floor((x - xoff) / r), floor((yoff - y) / r)) in double; outside the raster or a NaN coordinate:
// the sentinel ncells.  floor, not truncation, for -1 < (x - xoff) / r < 0 (DESIGN.md section 4).
__global__ void dsm_key_kernel(const DsmParams P, uint32_t *key, uint32_t *idx)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    const uint8_t *rec = P.rec + (size_t)i * P.rb;
    const double x = dsm_load(rec + P.off[0], P.type[0]), y = dsm_load(rec + P.off[1], P.type[1]);
    const double fx = floor(__ddiv_rn(__dsub_rn(x, P.xoff), P.r)), fy = floor(__ddiv_rn(__dsub_rn(P.yoff, y), P.r));
    uint32_t k = P.ncells;
    if (fx >= 0.0 && fx < (double)P.xsize && fy >= 0.0 && fy < (double)P.ysize)     // false for NaN
        k = (uint32_t)fy * (uint32_t)P.xsize + (uint32_t)fx;
    key[i] = k;
    idx[i] = i;
}

__global__ void dsm_fill_nan_kernel(float *raster, size_t n)
{
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        raster[i] = __int_as_float(0x7fc00000);
}

// One thread per sorted point; the first point of each cell's run folds the whole run, channel by channel, in point order
// (the stable sort kept it), and writes the cell's channel-last values.  Cells without points keep the NaN of the fill.
__global__ void dsm_fold_kernel(const DsmParams P, const uint32_t *key, const uint32_t *idx, float *raster)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    const uint32_t k = key[i];
    if (k == P.ncells || (i > 0 && key[i - 1] == k)) return;
    uint32_t end = i + 1;
    while (end < P.n && key[end] == k) end++;
    const int nch = P.ncols - 2;
    for (int c = 0; c < nch; c++) {
        const int off = P.off[c + 2], type = P.type[c + 2];
        float acc = 0.f, cnt = 0.f;
        for (uint32_t j = i; j < end; j++) {
            const double v = dsm_load(P.rec + (size_t)idx[j] * P.rb + off, type);
            acc = __double2float_rn(__dadd_rn((double)acc, __dmul_rn(1.0, v)));     // float += (float weight 1) * double
            cnt = __fadd_rn(cnt, 1.f);                                              // saturates at 2^24, as the reference's
        }
        raster[(size_t)k * nch + c] = __fdiv_rn(acc, cnt);
    }
}

}  // namespace s2pb
