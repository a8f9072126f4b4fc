// raster.cu -- the rasters of s2p's last steps: the n-view merge (section 8f) and the DSM rasterisation of plys_to_dsm.
#include "host.h"
#include "fusion_kernels.cuh"
#include "dsm_kernels.cuh"

#include <cub/device/device_radix_sort.cuh>

#include <cmath>
#include <cstring>

// ------------------------------------------------------------------ n-view merge (section 8f)

static_assert(S2PB_MAX_FUSION == kMaxFusion, "the public bound on the merged maps is the merge kernel's");

// what the merge refuses: n outside 1..kMaxFusion, an operator code (S2PB_FUSE_SUB_F32 aside) it does not know
int fusion_args_ok(int n, int op)
{
    if (n < 1) return fail(S2PB_ERR_ARG, "bad argument");
    if (n > kMaxFusion) return fail(S2PB_ERR_UNSUPPORTED, "at most %d rasters can be merged", kMaxFusion);
    op &= ~S2PB_FUSE_SUB_F32;
    if (op < FUSE_AVERAGE_IF_CLOSE || op >= FUSE_OP_COUNT) return fail(S2PB_ERR_ARG, "unknown averaging operator %d", op);
    return S2PB_OK;
}

// merge_n of n device rasters of npix float32 (f64: float64) values into the float32 d_out, after fusion_args_ok
void fusion_enqueue(s2pb_ctx *ctx, cudaStream_t st, const void *const *d_in, bool f64, const double *offsets, int n, size_t npix,
                    int op, double threshold, float *d_out)
{
    FusionParams P;
    memset(&P, 0, sizeof P);
    double s = 0;
    for (int k = 0; k < n; k++) {
        P.in[k] = d_in[k];
        P.offset[k] = offsets[k];
        s += offsets[k];                     // np.mean of a short list: plain left-to-right sum / n
    }
    P.n = n; P.op = op & ~S2PB_FUSE_SUB_F32; P.sub_f32 = (op & S2PB_FUSE_SUB_F32) ? 1 : 0; P.threshold = threshold;
    P.mean_offset = s / n; P.npix = npix; P.out = d_out;
    launch(ctx, f64 ? fusion_kernel<double> : fusion_kernel<float>, (unsigned)((npix + 255) / 256), 256, 0, st, P);
}

extern "C" int s2pb_merge_n(s2pb_ctx *ctx, const float *const *inputs, const double *offsets, int n, int w, int h, int op,
                            double threshold, float *out)
{
    if (!ctx || !inputs || !offsets || !out || w < 1 || h < 1) return fail(S2PB_ERR_ARG, "bad argument");
    if (int rc = fusion_args_ok(n, op)) return rc;
    const size_t npix = (size_t)w * h;
    HostCall L(ctx, "the merge");
    float *o = L.take<float>(npix * 4);
    const void *d_in[kMaxFusion] = {};
    for (int k = 0; k < n; k++) {
        if (!inputs[k]) return fail(S2PB_ERR_ARG, "null raster %d", k);
        d_in[k] = L.upload(inputs[k], npix * 4);
    }
    if (int rc = L.error()) return rc;
    fusion_enqueue(ctx, L.st, d_in, false, offsets, n, npix, op, threshold, o);
    CK(cudaGetLastError());
    L.download(out, o, npix * 4);
    return L.finish();
}

// ------------------------------------------------------------------ DSM rasterisation (plys_to_dsm)

// bits of the largest key, ncells: the radix sort looks at no more
static int key_bits(uint32_t ncells) { int b = 1; while (b < 32 && (ncells >> b)) b++; return b; }

// plyflatten with radius 0 and no sigma (dsm_kernels.cuh): upload the clouds' records back to back, key each point by its
// cell, stable radix sort by key, fold each cell's run in point order into the NaN-filled raster.
extern "C" int s2pb_plyflatten(s2pb_ctx *ctx, int nclouds, const void *const *records, const int64_t *npoints, int record_bytes,
                               const s2pb_ply_column *cols, int ncols, double xoff, double yoff, double resolution, int xsize,
                               int ysize, float *raster)
{
    if (!ctx || nclouds < 0 || (nclouds > 0 && (!records || !npoints)) || !cols || !raster || record_bytes < 1 || ncols < 3 ||
        !(resolution > 0.0) || !std::isfinite(resolution) || xsize < 1 || ysize < 1)
        return fail(S2PB_ERR_ARG, "bad argument");
    if (ncols > kDsmMaxCols) return fail(S2PB_ERR_UNSUPPORTED, "at most %d PLY properties, got %d", kDsmMaxCols, ncols);
    DsmParams P;
    memset(&P, 0, sizeof P);
    for (int c = 0; c < ncols; c++) {
        const int size = ply_type_bytes(cols[c].type);
        if (!size) return fail(S2PB_ERR_ARG, "column %d: unknown type %d", c, cols[c].type);
        if (cols[c].offset < 0 || cols[c].offset + size > record_bytes)
            return fail(S2PB_ERR_ARG, "column %d: bytes [%d, %d) outside a %d-byte record", c, cols[c].offset, cols[c].offset + size,
                        record_bytes);
        P.off[c] = cols[c].offset;
        P.type[c] = cols[c].type;
    }
    int64_t n = 0;
    for (int k = 0; k < nclouds; k++) {
        if (npoints[k] < 0 || (npoints[k] > 0 && !records[k])) return fail(S2PB_ERR_ARG, "cloud %d: bad records or count", k);
        n += npoints[k];
        if (n > INT32_MAX) return fail(S2PB_ERR_UNSUPPORTED, "at most 2^31 - 1 points in all");
    }
    const uint64_t ncells = (uint64_t)xsize * (uint64_t)ysize;
    if (ncells >= 0xFFFFFFFFull) return fail(S2PB_ERR_UNSUPPORTED, "a %dx%d raster: at most 2^32 - 2 cells", xsize, ysize);
    const int nch = ncols - 2;
    P.n = (uint32_t)n; P.rb = record_bytes; P.ncols = ncols;
    P.xoff = xoff; P.yoff = yoff; P.r = resolution; P.xsize = xsize; P.ysize = ysize; P.ncells = (uint32_t)ncells;
    HostCall L(ctx, "the DSM rasterisation");
    const size_t out_bytes = (size_t)ncells * nch * 4;
    float *d_raster = L.take<float>(out_bytes);
    const int bits = key_bits(P.ncells);
    size_t sort_bytes = 0;
    uint8_t *d_rec = nullptr;
    uint32_t *key = nullptr, *idx = nullptr, *key_s = nullptr, *idx_s = nullptr;
    void *sort_tmp = nullptr;
    if (n > 0) {
        CK(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint32_t *)nullptr, (uint32_t *)nullptr,
                                           (const uint32_t *)nullptr, (uint32_t *)nullptr, (int)n, 0, bits, L.st));
        d_rec = L.take<uint8_t>((size_t)n * record_bytes);
        key = L.take<uint32_t>((size_t)n * 4); idx = L.take<uint32_t>((size_t)n * 4);
        key_s = L.take<uint32_t>((size_t)n * 4); idx_s = L.take<uint32_t>((size_t)n * 4);
        sort_tmp = L.take<void>(sort_bytes);
    }
    if (int rc = L.error()) return rc;
    launch(ctx, dsm_fill_nan_kernel, (unsigned)std::min<size_t>((out_bytes / 4 + 255) / 256, 65536), 256, 0, L.st, d_raster, out_bytes / 4);
    CK(cudaGetLastError());
    if (n > 0) {
        size_t at = 0;
        for (int k = 0; k < nclouds; k++) {               // host (pageable or page-locked) or device records, by unified addressing
            const size_t bytes = (size_t)npoints[k] * record_bytes;
            if (bytes) CK(cudaMemcpyAsync(d_rec + at, records[k], bytes, cudaMemcpyDefault, L.st));
            at += bytes;
        }
        P.rec = d_rec;
        const unsigned g = (unsigned)((n + 255) / 256);
        launch(ctx, dsm_key_kernel, g, 256, 0, L.st, P, key, idx);
        CK(cudaGetLastError());
        CK(cub::DeviceRadixSort::SortPairs(sort_tmp, sort_bytes, key, key_s, idx, idx_s, (int)n, 0, bits, L.st));
        ctx->launches++;                                  // the radix sort counts as one launch, whatever CUB runs for it
        launch(ctx, dsm_fold_kernel, g, 256, 0, L.st, P, key_s, idx_s, d_raster);
        CK(cudaGetLastError());
    }
    L.download(raster, d_raster, out_bytes);
    return L.finish();
}
