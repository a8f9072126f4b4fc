// dct_kernels.cuh -- the DCT round trip the reference applies to the MATCHED image of every cost volume, bit for bit.
//
// Behavioural reference: shift() (3rdparty/mgm_multi/mgm_costvolume.cc:23-43) sends the matched image through
// image_shear (shear.c:28-101): per row REDFT10, /n, phase factors cos(ka) / sin(ka) with a = -(pi/n) q, REDFT01 +
// RODFT01, out = 0.5 (sym + antisym) cast to float -- even for q = 0 (mgm_costvolume.cc:50-60, `us[0]`), where it is
// the identity up to double rounding.  That rounding is invisible after the cast back to float32 EXCEPT on pixels that
// are (nearly) zero relative to their row: no-data pixels (NaN -> 0, main_mgm.cc:172-173) come back as +-1e-13-ish
// noise, and the census transform then compares noise with noise.  Two reference builds that differ only in the
// summation order of their DCT agree with each other within rounding-noise statistics, but the identity does not
// (scripts/nodata_spread.py), so the engine reproduces the round trip with the reference's own arithmetic:
//   * transforms are dense matrix products in double, terms added in ascending index order, multiply and add rounded
//     separately (what the oracle build's DCT does; real fftw builds use other orders and differ among themselves);
//   * the coefficient tables are computed on the HOST with libm's cos / sin (device cos differs in the last bit);
//   * q = 0: only rows that hold a pixel with |x| <= rowmax * n * 2^-24 are transformed, and only those pixels are
//     replaced; every other pixel provably returns to its float32 value (margin > 10x over 1e6 random rows,
//     tests/test_oracle.py::test_roundtrip_flag_rule), so a tile without no-data costs one pass over its pixels;
//   * q = 1/2 (SUBPIX = 2 of mgm_multi): every row, both inverse transforms.
// Nothing here is translated from the reference; the transforms are FFTW's published definitions (REDFT10, REDFT01,
// RODFT01, unnormalised).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace s2pb {

// per-image bookkeeping of the round trip, in device memory (so that nothing has to synchronise with the host)
struct RtState {
    int nrows;       // rows that need the transform
    int ncols;       // columns that hold a flagged pixel in any of those rows
    int pad[2];
};

// One block per image row: copy the row to `rt`, find rowmax, flag the pixels that the round trip may change and append
// the row to the list when it has any.  A row of zeros returns exact zeros and is skipped.
__global__ void rt_flag_kernel(const float *__restrict__ img, int w, int h, float *__restrict__ rt, RtState *st, int *__restrict__ rowlist,
                               float *__restrict__ rowthr, unsigned char *__restrict__ colflag)
{
    const int row = blockIdx.x;
    const float *src = img + (size_t)row * w;
    float *dst = rt + (size_t)row * w;
    __shared__ float red[32];
    float m = 0.f;
    for (int i = threadIdx.x; i < w; i += blockDim.x) { float v = src[i]; dst[i] = v; m = fmaxf(m, fabsf(v)); }
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x < 32) {
        m = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
        for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (threadIdx.x == 0) red[0] = m;
    }
    __syncthreads();
    const float rowmax = red[0];
    const float thr = rowmax * ((float)w * (1.f / 16777216.f));
    bool any = false;
    if (rowmax > 0.f)
        for (int i = threadIdx.x; i < w; i += blockDim.x)
            if (fabsf(src[i]) <= thr) { any = true; colflag[i] = 1; }      // (every writer stores the same value)
    const int cnt = __syncthreads_or(any ? 1 : 0);
    if (threadIdx.x == 0) {
        rowthr[row] = (cnt && rowmax > 0.f) ? thr : -1.f;
        if (cnt && rowmax > 0.f) rowlist[atomicAdd(&st->nrows, 1)] = row;
    }
}

// Y[r][o] = (sum_{i=0}^{n-1} T[o][i] * X[r][i]) * scale-by-division, r over the listed rows (or all rows when
// rowlist == nullptr).  The sum runs in ascending i with separately rounded multiply and add, from 0.0, like a plain C
// loop compiled without contraction.  T is [n][n] row-major.  64 outputs x 32 rows per block of 128 threads, 4 x 4 per
// thread: a thread's four T values and four X values of one i are two 16-byte shared loads each, i.e. four loads per
// sixteen multiply-add pairs (a 4 x 2 tile with 8-byte loads needs six per eight and is bound by them).  512 work items on a
// 1024 x 1024 image for the 132 SMs.
// IN = float (image rows) or double.  DIVN: divide the sum by n (the forward transform's normalisation, shear.c:62-63).
// `mul` (optional, [n]): the output is multiplied by mul[o] (the phase factor cos(o a));
// `mul2`/`Y2` (optional): a second output Y2[r][o-1] = y * mul2[o] for o >= 1 and Y2[r][n-1] = 0 (the antisymmetric
// part's input, shear.c:71-79).
constexpr int kGemmThreads = 128, kGemmTO = 64, kGemmTR = 32, kGemmTK = 16;
// one tile product: acc[qa][qb] += Ts[kk][gemm_out(tx, qa)] * Xs[kk][4 ty + qb] for kk < kmax, in ascending kk.  A thread's four
// outputs are two adjacent pairs 32 apart (2 tx, 2 tx + 1, 32 + 2 tx, 33 + 2 tx): the lanes' 16-byte loads are then contiguous
// (a 4-consecutive mapping strides them by 32 bytes: two wavefronts per load).
__device__ __forceinline__ int gemm_out(int tx, int qa) { return (qa < 2) ? 2 * tx + qa : 32 + 2 * tx + (qa - 2); }
__device__ __forceinline__ void gemm_tile_fp64(const double (*Ts)[kGemmTO + 2], const double (*Xs)[kGemmTR + 2], int kmax, int tx, int ty,
                                               double (&acc)[4][4])
{
    for (int kk = 0; kk < kmax; kk++) {
        const double2 a01 = *reinterpret_cast<const double2 *>(&Ts[kk][2 * tx]), a23 = *reinterpret_cast<const double2 *>(&Ts[kk][32 + 2 * tx]);
        const double2 b01 = *reinterpret_cast<const double2 *>(&Xs[kk][4 * ty]), b23 = *reinterpret_cast<const double2 *>(&Xs[kk][4 * ty + 2]);
        const double a[4] = {a01.x, a01.y, a23.x, a23.y}, b[4] = {b01.x, b01.y, b23.x, b23.y};
#pragma unroll
        for (int qa = 0; qa < 4; qa++)
#pragma unroll
            for (int qb = 0; qb < 4; qb++) acc[qa][qb] = __dadd_rn(acc[qa][qb], __dmul_rn(a[qa], b[qb]));
    }
}
template <typename IN, bool DIVN>
__global__ void __launch_bounds__(kGemmThreads) dct_gemm_kernel(const double *__restrict__ T, const IN *__restrict__ X, int n, int nrows_all,
                                                                const RtState *st, const int *__restrict__ rowlist,
                                                                double *__restrict__ Y, const double *__restrict__ mul,
                                                                const double *__restrict__ mul2, double *__restrict__ Y2)
{
    constexpr int TO = kGemmTO, TR = kGemmTR, TK = kGemmTK;
    __shared__ __align__(16) double Ts[TK][TO + 2];
    __shared__ __align__(16) double Xs[TK][TR + 2];
    __shared__ int rows_s[TR];
    const int nrows = rowlist ? st->nrows : nrows_all;
    const int otiles = (n + TO - 1) / TO, rtiles = (nrows + TR - 1) / TR;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;         // outputs gemm_out(tx, 0..3), rows 4 ty .. +3
    for (int item = blockIdx.x; item < otiles * rtiles; item += gridDim.x) {
        const int o0 = (item % otiles) * TO, r0 = (item / otiles) * TR;
        __syncthreads();
        if (threadIdx.x < TR) {
            const int rr = r0 + threadIdx.x;
            rows_s[threadIdx.x] = rr < nrows ? (rowlist ? rowlist[rr] : rr) : -1;
        }
        double acc[4][4];
#pragma unroll
        for (int qa = 0; qa < 4; qa++)
#pragma unroll
            for (int qb = 0; qb < 4; qb++) acc[qa][qb] = 0.0;
        // T tile: 64 outputs x 16 inputs, thread t holds output (t >> 1), inputs 8 (t & 1) .. +7; X tile: 32 rows x 16 inputs, thread t
        // holds row (t >> 2), inputs 4 (t & 3) .. +3.  The next tile's values are fetched into registers before the current tile's
        // product, so the global-load latency hides behind 16 x 32 FP64 instructions instead of standing between two barriers.
        __syncthreads();                                             // rows_s is visible
        const int to = o0 + (threadIdx.x >> 1), tkk = 8 * (threadIdx.x & 1);
        const int xrow = rows_s[threadIdx.x >> 2], xkk = 4 * (threadIdx.x & 3);
        double tv[8], xv[4];
        auto fetch = [&](int k0) {
#pragma unroll
            for (int q = 0; q < 8; q++) { const int k = k0 + tkk + q; tv[q] = (to < n && k < n) ? T[(size_t)to * n + k] : 0.0; }
#pragma unroll
            for (int q = 0; q < 4; q++) { const int k = k0 + xkk + q; xv[q] = (xrow >= 0 && k < n) ? (double)X[(size_t)xrow * n + k] : 0.0; }
        };
        fetch(0);
        for (int k0 = 0; k0 < n; k0 += TK) {
            __syncthreads();                                         // the previous product is done with the tiles
#pragma unroll
            for (int q = 0; q < 8; q++) Ts[tkk + q][threadIdx.x >> 1] = tv[q];
#pragma unroll
            for (int q = 0; q < 4; q++) Xs[xkk + q][threadIdx.x >> 2] = xv[q];
            __syncthreads();
            if (k0 + TK < n) fetch(k0 + TK);
            gemm_tile_fp64(Ts, Xs, (n - k0 < TK) ? n - k0 : TK, tx, ty, acc);
        }
#pragma unroll
        for (int qb = 0; qb < 4; qb++) {
            const int row = rows_s[4 * ty + qb];
            if (row < 0) continue;
#pragma unroll
            for (int qa = 0; qa < 4; qa++) {
                const int o = o0 + gemm_out(tx, qa);
                if (o >= n) continue;
                double y = acc[qa][qb];
                if (DIVN) y = __ddiv_rn(y, (double)n);
                if (Y2) {
                    if (o >= 1) Y2[(size_t)row * n + o - 1] = __dmul_rn(y, mul2[o]);
                    if (o == n - 1) Y2[(size_t)row * n + n - 1] = 0.0;
                }
                Y[(size_t)row * n + o] = mul ? __dmul_rn(y, mul[o]) : y;
            }
        }
    }
}

// the columns that hold a flagged pixel, compacted (one block; the order is irrelevant)
__global__ void rt_collist_kernel(const unsigned char *__restrict__ colflag, int w, RtState *st, int *__restrict__ collist)
{
    __shared__ int count;
    if (threadIdx.x == 0) count = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < w; i += blockDim.x)
        if (colflag[i]) collist[atomicAdd(&count, 1)] = i;
    __syncthreads();
    if (threadIdx.x == 0) st->ncols = count;
}

// q = 0, inverse: rt[r][i] = (float)(0.5 * (sum_k T01[i][k] Y[r][k] + 0.0)) for the FLAGGED pixels of the listed rows (the
// antisymmetric part is identically +0: its inputs are Y[k] sin(0) = +-0).  The same tiled product as dct_gemm_kernel, over
// the listed rows x the listed columns only -- a no-data margin is a few percent of the columns, so the inverse costs a few
// percent of the forward transform; with a ragged mask the column list grows towards the full width and the cost towards
// that of the forward one.  T01 is [n][n] row-major (output pixel, coefficient).
__global__ void __launch_bounds__(kGemmThreads) rt_inverse_gemm_kernel(const double *__restrict__ T01, const double *__restrict__ Y, int n,
                                                                       const RtState *st, const int *__restrict__ rowlist, const int *__restrict__ collist,
                                                                       const float *__restrict__ rowthr, const float *__restrict__ img, float *__restrict__ rt)
{
    constexpr int TO = kGemmTO, TR = kGemmTR, TK = kGemmTK;
    __shared__ __align__(16) double Ts[TK][TO + 2];
    __shared__ __align__(16) double Xs[TK][TR + 2];
    __shared__ int rows_s[TR], cols_s[TO];
    const int nrows = st->nrows, ncols = st->ncols;
    const int otiles = (ncols + TO - 1) / TO, rtiles = (nrows + TR - 1) / TR;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    for (int item = blockIdx.x; item < otiles * rtiles; item += gridDim.x) {
        const int o0 = (item % otiles) * TO, r0 = (item / otiles) * TR;
        __syncthreads();
        if (threadIdx.x < TR) rows_s[threadIdx.x] = (r0 + (int)threadIdx.x < nrows) ? rowlist[r0 + threadIdx.x] : -1;
        else if (threadIdx.x < TR + TO) { const int q = threadIdx.x - TR; cols_s[q] = (o0 + q < ncols) ? collist[o0 + q] : -1; }
        double acc[4][4];
#pragma unroll
        for (int qa = 0; qa < 4; qa++)
#pragma unroll
            for (int qb = 0; qb < 4; qb++) acc[qa][qb] = 0.0;
        __syncthreads();                                             // rows_s, cols_s are visible
        const int tcol = cols_s[threadIdx.x >> 1], tkk = 8 * (threadIdx.x & 1);
        const int xrow = rows_s[threadIdx.x >> 2], xkk = 4 * (threadIdx.x & 3);
        double tv[8], xv[4];
        auto fetch = [&](int k0) {                                   // (register prefetch of the next tiles, as in dct_gemm_kernel)
#pragma unroll
            for (int q = 0; q < 8; q++) { const int k = k0 + tkk + q; tv[q] = (tcol >= 0 && k < n) ? T01[(size_t)tcol * n + k] : 0.0; }
#pragma unroll
            for (int q = 0; q < 4; q++) { const int k = k0 + xkk + q; xv[q] = (xrow >= 0 && k < n) ? Y[(size_t)xrow * n + k] : 0.0; }
        };
        fetch(0);
        for (int k0 = 0; k0 < n; k0 += TK) {
            __syncthreads();
#pragma unroll
            for (int q = 0; q < 8; q++) Ts[tkk + q][threadIdx.x >> 1] = tv[q];
#pragma unroll
            for (int q = 0; q < 4; q++) Xs[xkk + q][threadIdx.x >> 2] = xv[q];
            __syncthreads();
            if (k0 + TK < n) fetch(k0 + TK);
            gemm_tile_fp64(Ts, Xs, (n - k0 < TK) ? n - k0 : TK, tx, ty, acc);
        }
#pragma unroll
        for (int qb = 0; qb < 4; qb++) {
            const int row = rows_s[4 * ty + qb];
            if (row < 0) continue;
            const float thr = rowthr[row];
#pragma unroll
            for (int qa = 0; qa < 4; qa++) {
                const int col = cols_s[gemm_out(tx, qa)];
                if (col < 0) continue;
                const size_t p = (size_t)row * n + col;
                if (fabsf(img[p]) <= thr) rt[p] = (float)__dmul_rn(0.5, __dadd_rn(acc[qa][qb], 0.0));
            }
        }
    }
}

// q != 0: out = (float)(0.5 * (sym + antisym)) on every pixel (shear.c:88-89)
__global__ void dct_combine_kernel(const double *__restrict__ sym, const double *__restrict__ anti, size_t n, float *__restrict__ out)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (float)__dmul_rn(0.5, __dadd_rn(sym[i], anti[i]));
}

// census of the image and of its round-tripped copy in one pass; when no row needed the transform the second code is
// the first (saves the second evaluation on tiles without no-data)
__global__ void census_pair_kernel(const float *__restrict__ img, const float *__restrict__ rt, const RtState *st, int w, int h, int r,
                                   uint64_t *__restrict__ codes, uint64_t *__restrict__ codes_rt)
{
    int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const bool both = st->nrows > 0;
    float c = img[(size_t)y * w + x], c2 = both ? rt[(size_t)y * w + x] : 0.f;
    uint64_t code = 0, code2 = 0;
    for (int j = -r; j <= r; j++)
        for (int i = -r; i <= r; i++) {
            if (i == 0 && j == 0) continue;
            int xx = x + i, yy = y + j;
            unsigned bit = 0, bit2 = 0;
            if (xx >= 0 && xx < w && yy >= 0 && yy < h) {
                bit = c < img[(size_t)yy * w + xx];
                if (both) bit2 = c2 < rt[(size_t)yy * w + xx];
            }
            code = (code << 1) | bit;
            code2 = (code2 << 1) | bit2;
        }
    codes[(size_t)y * w + x] = code;
    codes_rt[(size_t)y * w + x] = both ? code2 : code;
}

}  // namespace s2pb
