// cloud.cu -- the tile's point cloud as PLY records (cloud_kernels.cuh): the colours of
// common.linear_stretching_and_quantization_8bit, or of a clr image in its own type, and the vertex records of
// triangulation.write_to_ply, alone or at the end of disparity_to_ply / heights_to_ply's triangulation and 3D filter on one stream.
#include "host.h"
#include "cloud_kernels.cuh"

// bytes of one record: x, y, z float64, 3 colours (1 or 3 bands) or 4 (4 bands) of cb bytes, confidence float32
static int record_bytes(int nbands, int cb, bool conf) { return 24 + (nbands == 4 ? 4 : nbands ? 3 : 0) * cb + (conf ? 4 : 0); }

static bool bands_ok(int nbands) { return nbands == 0 || nbands == 1 || nbands == 3 || nbands == 4; }

// np.nanpercentile(img, (pct, 100 - pct)) of the n values of d_im into d_os (order_stats_bytes())
static int stretch_bounds_enqueue(s2pb_ctx *ctx, cudaStream_t st, const float *d_im, size_t n, double pct, OrderStats *d_os)
{
    return launch_order_stats(ctx, st, d_im, (int)n, kOrdLinear, pct / 100.0, (100.0 - pct) / 100.0, d_os);
}

// The kept points of the device cloud d_xyz (n points) packed into d_out; their number into *d_total.  Colours: d_colors
// (nbands planes of values of cb bytes, copied) or, when it is null, d_bands (nbands float32 planes) stretched to uint8 with
// the bounds of d_os.  Records wider than kPlyMaxRecord bytes go through the wide kernels' smaller CTA tiles.
static int pack_enqueue(s2pb_ctx *ctx, HostCall &L, const double *d_xyz, size_t n, int nbands, const uint8_t *d_colors, int cb,
                        const float *d_bands, const OrderStats *d_os, const float *d_conf, uint8_t *d_out, long long *d_total)
{
    const int rb = record_bytes(nbands, d_colors ? cb : 1, d_conf != nullptr);
    const bool wide = rb > kPlyMaxRecord;
    const int tile = wide ? kPlyThreads * kPlyPerWide : kPlyTile;
    const int ntiles = (int)((n + tile - 1) / tile);
    int *d_counts = L.take<int>((size_t)ntiles * 4);
    long long *d_offsets = L.take<long long>((size_t)ntiles * 8);
    if (int rc = L.error()) return rc;
    launch(ctx, wide ? ply_count_kernel<kPlyPerWide> : ply_count_kernel<kPlyPer>, ntiles, kPlyThreads, 0, L.st, d_xyz, n, d_counts);
    launch(ctx, ply_scan_kernel, 1, 1024, 0, L.st, d_counts, ntiles, d_offsets, d_total);
    PlyPackParams P;
    P.xyz = d_xyz; P.n = n; P.offsets = d_offsets; P.nbands = nbands; P.cb = d_colors ? cb : 1; P.colors = d_colors;
    P.bands = d_bands; P.os = d_os; P.conf = d_conf; P.rb = rb; P.out = d_out;
    launch(ctx, wide ? ply_pack_kernel<kPlyPerWide, kPlyMaxWide> : ply_pack_kernel<kPlyPer, kPlyMaxRecord>, ntiles, kPlyThreads, 0,
           L.st, P);
    CK(cudaGetLastError());
    return S2PB_OK;
}

// the number of records, then only their bytes come back
static int download_records(HostCall &L, const long long *d_total, const uint8_t *d_out, int rb, uint8_t *records, int64_t *npoints)
{
    long long total = 0;
    L.download(&total, d_total, 8);
    if (int rc = L.finish()) return rc;
    *npoints = total;
    if (total) L.download(records, d_out, (size_t)total * rb);
    return L.finish();
}

extern "C" int s2pb_stretch_8bit(s2pb_ctx *ctx, const float *img, int64_t n, double pct, uint8_t *out)
{
    if (!ctx || n < 0 || (n && (!img || !out))) return fail(S2PB_ERR_ARG, "bad argument");
    if (!(pct >= 0.0 && pct <= 100.0)) return fail(S2PB_ERR_ARG, "percentiles must be in the range [0, 100] (got %g)", pct);
    if (n > INT32_MAX) return fail(S2PB_ERR_UNSUPPORTED, "at most 2^31 - 1 values");
    if (n == 0) return S2PB_OK;
    HostCall L(ctx, "the 8-bit stretch");
    float *d_im = L.upload(img, (size_t)n * 4);
    OrderStats *d_os = L.take<OrderStats>(order_stats_bytes());
    uint8_t *d_out = L.take<uint8_t>((size_t)n);
    if (int rc = L.error()) return rc;
    if (int rc = stretch_bounds_enqueue(ctx, L.st, d_im, (size_t)n, pct, d_os)) return rc;
    launch(ctx, stretch_8bit_kernel, (unsigned)std::min<int64_t>((n + 255) / 256, (int64_t)ctx->sm_count * 16), 256, 0, L.st, d_im,
           (size_t)n, d_os, d_out);
    CK(cudaGetLastError());
    L.download(out, d_out, (size_t)n);
    return L.finish();
}

extern "C" int s2pb_ply_records(s2pb_ctx *ctx, const double *xyz, int64_t n, const uint8_t *colors, int nbands, const float *conf,
                                uint8_t *records, int64_t *npoints)
{
    if (!ctx || !npoints || n < 0 || (n && (!xyz || !records || (nbands && !colors)))) return fail(S2PB_ERR_ARG, "bad argument");
    if (!bands_ok(nbands)) return fail(S2PB_ERR_ARG, "colors must have either 1, 3 or 4 channels (got %d)", nbands);
    if (n > INT32_MAX) return fail(S2PB_ERR_UNSUPPORTED, "at most 2^31 - 1 points");
    *npoints = 0;
    if (n == 0) return S2PB_OK;
    HostCall L(ctx, "the PLY records");
    const size_t np = (size_t)n;
    const int rb = record_bytes(nbands, 1, conf != nullptr);
    double *d_xyz = L.upload(xyz, np * 24);
    uint8_t *d_col = nbands ? L.upload(colors, np * nbands) : nullptr;
    float *d_conf = conf ? L.upload(conf, np * 4) : nullptr;
    uint8_t *d_out = L.take<uint8_t>(np * rb);
    long long *d_total = L.take<long long>(8);
    if (int rc = L.error()) return rc;
    if (int rc = pack_enqueue(ctx, L, d_xyz, np, nbands, d_col, 1, nullptr, nullptr, d_conf, d_out, d_total)) return rc;
    return download_records(L, d_total, d_out, rb, records, npoints);
}

// nbands 1, 3 or 4 and a known colour type: the colours of a clr image
int typed_colours_ok(int nbands, int color_type)
{
    if (nbands != 1 && nbands != 3 && nbands != 4) return fail(S2PB_ERR_ARG, "colors must have either 1, 3 or 4 channels (got %d)", nbands);
    if (!ply_type_bytes(color_type)) return fail(S2PB_ERR_ARG, "unknown PLY colour type %d", color_type);
    return S2PB_OK;
}

extern "C" int s2pb_ply_records_typed(s2pb_ctx *ctx, const double *xyz, int64_t n, const void *colors, int nbands, int color_type,
                                      const float *conf, uint8_t *records, int64_t *npoints)
{
    if (!ctx || !npoints || n < 0 || (n && (!xyz || !records || (nbands && !colors)))) return fail(S2PB_ERR_ARG, "bad argument");
    if (!bands_ok(nbands)) return fail(S2PB_ERR_ARG, "colors must have either 1, 3 or 4 channels (got %d)", nbands);
    const int cb = ply_type_bytes(color_type);
    if (!cb) return fail(S2PB_ERR_ARG, "unknown PLY colour type %d", color_type);
    if (n > INT32_MAX) return fail(S2PB_ERR_UNSUPPORTED, "at most 2^31 - 1 points");
    *npoints = 0;
    if (n == 0) return S2PB_OK;
    HostCall L(ctx, "the PLY records");
    const size_t np = (size_t)n;
    const int rb = record_bytes(nbands, cb, conf != nullptr);
    double *d_xyz = L.upload(xyz, np * 24);
    uint8_t *d_col = nbands ? L.upload((const uint8_t *)colors, np * nbands * cb) : nullptr;
    float *d_conf = conf ? L.upload(conf, np * 4) : nullptr;
    uint8_t *d_out = L.take<uint8_t>(np * rb);
    long long *d_total = L.take<long long>(8);
    if (int rc = L.error()) return rc;
    if (int rc = pack_enqueue(ctx, L, d_xyz, np, nbands, d_col, cb, nullptr, nullptr, d_conf, d_out, d_total)) return rc;
    return download_records(L, d_total, d_out, rb, records, npoints);
}

// The common tail of the steps on device inputs: filter, colours, records.  Colours: d_typed (nbands device planes of cb-byte
// values, copied as they are) or, when it is null, the device float32 planes d_bands stretched with pct.
int cloud_tail_device(s2pb_ctx *ctx, HostCall &L, double *d_xyz, int nx, int ny, float r, int p, int n, const float *d_bands,
                      int nbands, double pct, const uint8_t *d_typed, int cb, const float *d_conf, uint8_t *records, int64_t *npoints)
{
    const size_t npix = (size_t)nx * ny;
    const int rb = record_bytes(nbands, d_typed ? cb : 1, d_conf != nullptr);
    int *d_work = (r != 0.f && n > 0) ? L.take<int>(npix * 12) : nullptr;
    OrderStats *d_os = d_bands ? L.take<OrderStats>(order_stats_bytes()) : nullptr;
    uint8_t *d_out = L.take<uint8_t>(npix * rb);
    long long *d_total = L.take<long long>(8);
    if (int rc = L.error()) return rc;
    if (d_work) {
        if (int rc = remove_isolated_enqueue(ctx, L.st, d_xyz, nx, ny, r, p, n, 1, d_work)) return rc;
    }
    if (d_bands) {
        if (int rc = stretch_bounds_enqueue(ctx, L.st, d_bands, npix * nbands, pct, d_os)) return rc;
    }
    if (int rc = pack_enqueue(ctx, L, d_xyz, npix, nbands, d_typed, cb, d_bands, d_os, d_conf, d_out, d_total)) return rc;
    return download_records(L, d_total, d_out, rb, records, npoints);
}

// The common tail of the steps with host inputs: the float32 planes `bands` (when d_typed is null) and conf go to the device first.
static int cloud_tail(s2pb_ctx *ctx, HostCall &L, double *d_xyz, int nx, int ny, float r, int p, int n, const float *bands,
                      int nbands, double pct, const uint8_t *d_typed, int cb, const float *conf, uint8_t *records, int64_t *npoints)
{
    const size_t npix = (size_t)nx * ny;
    float *d_bands = nbands && !d_typed ? L.upload(bands, npix * nbands * 4) : nullptr;
    float *d_conf = conf ? L.upload(conf, npix * 4) : nullptr;
    return cloud_tail_device(ctx, L, d_xyz, nx, ny, r, p, n, d_bands, nbands, pct, d_typed, cb, d_conf, records, npoints);
}

// the arguments of the tail, checked before the cloud is made; the cloud's own step checks the rest
int tail_args_ok(s2pb_ctx *ctx, int nx, int ny, const float *bands, int nbands, double pct, uint8_t *records,
                        int64_t *npoints)
{
    if (!ctx || nx < 1 || ny < 1 || !records || !npoints || (nbands && !bands)) return fail(S2PB_ERR_ARG, "bad argument");
    if (!bands_ok(nbands)) return fail(S2PB_ERR_ARG, "colors must have either 1, 3 or 4 channels (got %d)", nbands);
    if (!(pct >= 0.0 && pct <= 100.0)) return fail(S2PB_ERR_ARG, "percentiles must be in the range [0, 100] (got %g)", pct);
    if ((size_t)nx * ny * std::max(nbands, 1) > INT32_MAX) return fail(S2PB_ERR_UNSUPPORTED, "at most 2^31 - 1 points and colour values");
    return S2PB_OK;
}

extern "C" int s2pb_disp_to_ply(s2pb_ctx *ctx, const float *dispx, const float *dispy, const float *msk, int nx, int ny,
                                const float *msk_orig, int w, int h, const double ha[9], const double hb[9], const s2pb_rpc *rpca,
                                const s2pb_rpc *rpcb, const float bbox[4], int zone, int south, float r, int p, int n,
                                const float *bands, int nbands, double pct, const float *conf, uint8_t *records, int64_t *npoints)
{
    if (int rc = tail_args_ok(ctx, nx, ny, bands, nbands, pct, records, npoints)) return rc;
    *npoints = 0;
    HostCall L(ctx, "the tile's cloud");
    double *d_xyz = nullptr;
    float *d_err = nullptr;
    if (int rc = triangulated_cloud(ctx, L, dispx, dispy, msk, nx, ny, msk_orig, w, h, ha, hb, rpca, rpcb, bbox, zone, south, &d_xyz,
                                    &d_err))
        return rc;
    return cloud_tail(ctx, L, d_xyz, nx, ny, r, p, n, bands, nbands, pct, nullptr, 1, conf, records, npoints);
}

extern "C" int s2pb_height_map_to_ply(s2pb_ctx *ctx, const double *heights, int w, int h, const s2pb_rpc *rpc, double off_x,
                                      double off_y, int zone, int south, float r, int p, int n, const float *bands, int nbands,
                                      double pct, uint8_t *records, int64_t *npoints)
{
    if (int rc = tail_args_ok(ctx, w, h, bands, nbands, pct, records, npoints)) return rc;
    *npoints = 0;
    HostCall L(ctx, "the tile's cloud");
    double *d_xyz = nullptr;
    if (int rc = localised_cloud(ctx, L, heights, w, h, rpc, off_x, off_y, zone, south, &d_xyz)) return rc;
    return cloud_tail(ctx, L, d_xyz, w, h, r, p, n, bands, nbands, pct, nullptr, 1, nullptr, records, npoints);
}

extern "C" int s2pb_disp_to_ply_clr(s2pb_ctx *ctx, const float *dispx, const float *dispy, const float *msk, int nx, int ny,
                                    const float *msk_orig, int w, int h, const double ha[9], const double hb[9], const s2pb_rpc *rpca,
                                    const s2pb_rpc *rpcb, const float bbox[4], int zone, int south, float r, int p, int n,
                                    const float *clr, int cw, int ch, int nbands, const double hc[9], const float *conf,
                                    uint8_t *records, int64_t *npoints)
{
    if (int rc = tail_args_ok(ctx, nx, ny, clr, nbands, 0.0, records, npoints)) return rc;
    if (int rc = typed_colours_ok(nbands, S2PB_PLY_F32)) return rc;
    if (!hc || cw < 1 || ch < 1) return fail(S2PB_ERR_ARG, "bad argument");
    *npoints = 0;
    HostCall L(ctx, "the tile's cloud");
    double *d_xyz = nullptr;
    float *d_err = nullptr;
    if (int rc = triangulated_cloud(ctx, L, dispx, dispy, msk, nx, ny, msk_orig, w, h, ha, hb, rpca, rpcb, bbox, zone, south, &d_xyz,
                                    &d_err))
        return rc;
    // each band as s2pb_homography warps it, into the plane the records read its colours from
    const size_t npix = (size_t)nx * ny;
    float *d_col = L.take<float>(npix * nbands * 4);
    if (int rc = L.error()) return rc;
    for (int b = 0; b < nbands; b++)
        if (int rc = warp_host_to_device(ctx, L, L.st, clr + (size_t)b * cw * ch, cw, ch, hc, d_col + (size_t)b * npix, nx, ny))
            return rc;
    return cloud_tail(ctx, L, d_xyz, nx, ny, r, p, n, nullptr, nbands, 0.0, (const uint8_t *)d_col, 4, conf, records, npoints);
}

extern "C" int s2pb_height_map_to_ply_clr(s2pb_ctx *ctx, const double *heights, int w, int h, const s2pb_rpc *rpc, double off_x,
                                          double off_y, int zone, int south, float r, int p, int n, const void *colors, int nbands,
                                          int color_type, uint8_t *records, int64_t *npoints)
{
    if (int rc = tail_args_ok(ctx, w, h, (const float *)colors, nbands, 0.0, records, npoints)) return rc;
    if (int rc = typed_colours_ok(nbands, color_type)) return rc;
    *npoints = 0;
    HostCall L(ctx, "the tile's cloud");
    const int cb = ply_type_bytes(color_type);
    uint8_t *d_col = L.upload((const uint8_t *)colors, (size_t)w * h * nbands * cb);
    if (int rc = L.error()) return rc;
    double *d_xyz = nullptr;
    if (int rc = localised_cloud(ctx, L, heights, w, h, rpc, off_x, off_y, zone, south, &d_xyz)) return rc;
    return cloud_tail(ctx, L, d_xyz, w, h, r, p, n, nullptr, nbands, 0.0, d_col, cb, nullptr, records, npoints);
}
