// heights_tile.cu -- a tri-stereo tile from its pairs' height maps to the records of cloud.ply in one call: heights_fusion
// (cargarse_basura of each map, merge_n) and heights_to_ply's localisation, filter and records chained on one stream, the
// maps staying on the device (s2p/__init__.py:355-429).
#include "host.h"

// out[i] = (Out)in[i]: a float64 map rounded to the float32 the reference's tools read (cargarse_basura), and the merged
// float32 map converted exactly to the float64 heights the localisation reads
template <typename In, typename Out>
__global__ void convert_kernel(const In *__restrict__ in, Out *__restrict__ out, size_t n)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (Out)in[i];
}

template <typename In, typename Out>
static void launch_convert(s2pb_ctx *ctx, cudaStream_t st, const In *in, Out *out, size_t n)
{
    launch(ctx, convert_kernel<In, Out>, (unsigned)((n + 255) / 256), 256, 0, st, in, out, n);
}

// what the stages would refuse that can be seen before the first launch
static int heights_tile_args_ok(s2pb_ctx *ctx, const s2pb_heights_tile *t, uint8_t *records, int64_t *npoints, float *const *cleaned)
{
    if (!ctx || !t || t->w < 1 || t->h < 1) return fail(S2PB_ERR_ARG, "bad argument");
    if (t->map_type != S2PB_PLY_F32 && t->map_type != S2PB_PLY_F64) return fail(S2PB_ERR_ARG, "height maps are float32 or float64");
    if (int rc = fusion_args_ok(t->n_maps, t->op)) return rc;
    for (int k = 0; k < t->n_maps; k++)
        if (!t->maps[k]) return fail(S2PB_ERR_ARG, "null raster %d", k);
    if (cleaned && !t->cargarse_basura) return fail(S2PB_ERR_ARG, "the cleaned maps exist with cargarse_basura only");
    if (t->cargarse_basura) {
        if (int rc = basura_args_ok(t->w, t->h)) return rc;
    }
    if (int rc = localised_cloud_args_ok(ctx, t->w, t->h, t->rpc, t->zone, t->south)) return rc;
    if (t->stretch) return tail_args_ok(ctx, t->w, t->h, (const float *)t->colors, t->nbands, t->pct, records, npoints);
    if (int rc = tail_args_ok(ctx, t->w, t->h, (const float *)t->colors, t->nbands, 0.0, records, npoints)) return rc;
    return typed_colours_ok(t->nbands, t->color_type);
}

extern "C" int s2pb_heights_tile_to_ply(s2pb_ctx *ctx, const s2pb_heights_tile *t, uint8_t *records, int64_t *npoints,
                                        float *const *cleaned, float *merged)
{
    if (int rc = heights_tile_args_ok(ctx, t, records, npoints, cleaned)) return rc;
    *npoints = 0;
    const int w = t->w, h = t->h, n = t->n_maps;
    const size_t npix = (size_t)w * h;
    const bool f64 = t->map_type == S2PB_PLY_F64;
    HostCall L(ctx, "the heights tile");
    const void *d_in[S2PB_MAX_FUSION] = {};
    for (int k = 0; k < n; k++) d_in[k] = L.upload((const uint8_t *)t->maps[k], npix * (f64 ? 8 : 4));
    float *d_merged = L.take<float>(npix * 4);
    double *d_z = L.take<double>(npix * 8);
    if (int rc = L.error()) return rc;

    // heights_fusion: cargarse_basura of each map on its float32 rounding, then merge_n on the cleaned maps or the stored ones
    bool merge_f64 = f64;
    if (t->cargarse_basura) {
        float *d_round = f64 ? L.take<float>(npix * 4) : nullptr, *d_m = L.take<float>(npix * 4);
        int *lab = L.take<int>(npix * 4), *area = L.take<int>(npix * 4);
        float *d_clean[S2PB_MAX_FUSION] = {};
        for (int k = 0; k < n; k++) d_clean[k] = L.take<float>(npix * 4);
        if (int rc = L.error()) return rc;
        for (int k = 0; k < n; k++) {
            const float *src = (const float *)d_in[k];
            if (f64) {
                launch_convert(ctx, L.st, (const double *)d_in[k], d_round, npix);
                src = d_round;
            }
            if (int rc = basura_enqueue(ctx, L.st, src, d_clean[k], w, h, d_m, lab, area)) return rc;
            if (cleaned && cleaned[k]) L.download(cleaned[k], d_clean[k], npix * 4);
            d_in[k] = d_clean[k];
        }
        merge_f64 = false;
    }
    fusion_enqueue(ctx, L.st, d_in, merge_f64, t->offsets, n, npix, t->op, t->threshold, d_merged);
    if (merged) L.download(merged, d_merged, npix * 4);

    // heights_to_ply: the merged map as float64 heights, localised, filtered, coloured and packed
    launch_convert(ctx, L.st, (const float *)d_merged, d_z, npix);
    CK(cudaGetLastError());
    const int nb = t->nbands;
    const float *d_bands = nullptr;
    const uint8_t *d_typed = nullptr;
    const int cb = t->stretch ? 1 : ply_type_bytes(t->color_type);
    if (nb && t->stretch) d_bands = L.upload((const float *)t->colors, npix * nb * 4);
    else if (nb) d_typed = L.upload((const uint8_t *)t->colors, npix * nb * cb);
    if (int rc = L.error()) return rc;
    double *d_xyz = nullptr;
    if (int rc = localised_cloud_device(ctx, L, d_z, w, h, t->rpc, t->off_x, t->off_y, t->zone, t->south, &d_xyz)) return rc;
    return cloud_tail_device(ctx, L, d_xyz, w, h, t->r, t->p, t->n, d_bands, nb, t->stretch ? t->pct : 0.0, d_typed, cb, nullptr,
                             records, npoints);
}
