// projection.cu -- the change of coordinates of s2p.triangulation.disp_to_xyz: WGS84 (lon, lat, alt) -> UTM, and the EGM96
// geoid heights of the compound targets (EPSG:326zz+5773, 327zz+5773, 4326+5773).
#include "host.h"

#include <cmath>

// The coefficients of projection_kernels.cuh for UTM zone `zone` (1..60) of WGS84, in double.  The series in the third
// flattening n are those of Karney (2011), eq. (35) for alpha (Krueger's series, ellipsoid <- sphere) and the conformal-latitude
// series of Engsager and Poder (2007), both to order n^6, as PROJ evaluates them for its exact transverse Mercator.
static UtmParams utm_params(int zone, bool south)
{
    const double a = 6378137.0, f = 1.0 / 298.257223563, k0 = 0.9996;
    const double n = f / (2.0 - f);
    UtmParams P;
    double np = n;
    P.cbg[0] = n * (-2 + n * (2 / 3.0 + n * (4 / 3.0 + n * (-82 / 45.0 + n * (32 / 45.0 + n * (4642 / 4725.0))))));
    P.gtu[0] = n * (0.5 + n * (-2 / 3.0 + n * (5 / 16.0 + n * (41 / 180.0 + n * (-127 / 288.0 + n * (7891 / 37800.0))))));
    np *= n;
    P.cbg[1] = np * (5 / 3.0 + n * (-16 / 15.0 + n * (-13 / 9.0 + n * (904 / 315.0 + n * (-1522 / 945.0)))));
    P.gtu[1] = np * (13 / 48.0 + n * (-3 / 5.0 + n * (557 / 1440.0 + n * (281 / 630.0 + n * (-1983433 / 1935360.0)))));
    np *= n;
    P.cbg[2] = np * (-26 / 15.0 + n * (34 / 21.0 + n * (8 / 5.0 + n * (-12686 / 2835.0))));
    P.gtu[2] = np * (61 / 240.0 + n * (-103 / 140.0 + n * (15061 / 26880.0 + n * (167603 / 181440.0))));
    np *= n;
    P.cbg[3] = np * (1237 / 630.0 + n * (-12 / 5.0 + n * (-24832 / 14175.0)));
    P.gtu[3] = np * (49561 / 161280.0 + n * (-179 / 168.0 + n * (6601661 / 7257600.0)));
    np *= n;
    P.cbg[4] = np * (-734 / 315.0 + n * (109598 / 31185.0));
    P.gtu[4] = np * (34729 / 80640.0 + n * (-3418889 / 1995840.0));
    np *= n;
    P.cbg[5] = np * (444337 / 155925.0);
    P.gtu[5] = np * (212378941 / 319334400.0);
    // k0 times the rectifying radius A = a / (1 + n) (1 + n^2 / 4 + n^4 / 64 + n^6 / 256 + ...)
    const double n2 = n * n;
    P.qa = a * (k0 / (1 + n) * (1 + n2 * (1 / 4.0 + n2 * (1 / 64.0 + n2 / 256.0))));
    P.lon0 = 6.0 * zone - 183.0;
    P.x0 = 500000.0;
    P.y0 = south ? 10000000.0 : 0.0;
    return P;
}

int cloud_crs_ok(const s2pb_ctx *ctx, int zone, bool zone0)
{
    const int utm = zone & ~S2PB_ZONE_EGM96;
    if (utm < (zone0 ? 0 : 1) || utm > 60)
        return fail(S2PB_ERR_ARG, "zone %d: a UTM zone 1 to 60%s, optionally OR S2PB_ZONE_EGM96", zone, zone0 ? ", or 0 for lon, lat" : "");
    if ((zone & S2PB_ZONE_EGM96) && !ctx->geoid.g) return fail(S2PB_ERR_ARG, "S2PB_ZONE_EGM96 on a context without a geoid grid");
    return S2PB_OK;
}

int launch_cloud_project(s2pb_ctx *ctx, cudaStream_t st, int zone, bool south, const double *d_in, double *d_out, size_t n)
{
    const int utm = zone & ~S2PB_ZONE_EGM96;
    const bool geoid = (zone & S2PB_ZONE_EGM96) != 0;
    if (n == 0 || (!utm && !geoid)) return S2PB_OK;
    const unsigned b = 256;
    const dim3 g((unsigned)((n + b - 1) / b));
    const UtmParams P = utm_params(utm, south);
    if (!geoid) launch(ctx, cloud_project_kernel<true, false>, g, dim3(b), 0, st, P, ctx->geoid, d_in, d_out, (long long)n);
    else if (utm) launch(ctx, cloud_project_kernel<true, true>, g, dim3(b), 0, st, P, ctx->geoid, d_in, d_out, (long long)n);
    else launch(ctx, cloud_project_kernel<false, true>, g, dim3(b), 0, st, P, ctx->geoid, d_in, d_out, (long long)n);
    CK(cudaGetLastError());
    return S2PB_OK;
}

extern "C" int s2pb_lonlat_to_utm(s2pb_ctx *ctx, double *xyz, const double *lonlatalt, int64_t n, int zone, int south)
{
    if (!ctx || n < 0 || (n > 0 && (!xyz || !lonlatalt))) return fail(S2PB_ERR_ARG, "bad argument");
    if (int rc = cloud_crs_ok(ctx, zone, false)) return rc;
    if (n == 0) return S2PB_OK;
    const size_t bytes = (size_t)n * 24;
    HostCall L(ctx, "the projection");
    double *d = L.upload(lonlatalt, bytes);
    if (int rc = L.error()) return rc;
    int rc = launch_cloud_project(ctx, L.st, zone, south != 0, d, d, (size_t)n);
    if (rc != S2PB_OK) return rc;
    L.download(xyz, d, bytes);
    return L.finish();
}

void geoid_free(s2pb_ctx *ctx)
{
    if (ctx->geoid.g) cudaFree((void *)ctx->geoid.g);
    ctx->geoid = GeoidGrid{};
}

// The grid must be global (GeoidGrid): no point of a cloud falls outside it.
extern "C" int s2pb_set_geoid(s2pb_ctx *ctx, const float *grid, int w, int h, double lon0, double lat0, double dlon, double dlat)
{
    if (!ctx) return fail(S2PB_ERR_ARG, "bad argument");
    CK(cudaSetDevice(ctx->device));
    if (!grid) {
        geoid_free(ctx);
        return S2PB_OK;
    }
    if (w < 2 || h < 2 || (int64_t)w * h > INT32_MAX || !std::isfinite(lon0) || !std::isfinite(lat0) || !(dlon > 0.0) ||
        !(dlat > 0.0) || !std::isfinite(dlon) || !std::isfinite(dlat))
        return fail(S2PB_ERR_ARG, "bad geoid grid: %d x %d nodes, origin (%g, %g), spacing (%g, %g)", w, h, lon0, lat0, dlon, dlat);
    const double eps = 1e-9;
    if (w * dlon < 360.0 - eps || lat0 < 90.0 - eps || lat0 - (h - 1) * dlat > -90.0 + eps)
        return fail(S2PB_ERR_ARG, "the geoid grid is not global: %d x %d nodes from (%g, %g) by (%g, %g) degrees", w, h, lon0, lat0,
                    dlon, dlat);
    const size_t bytes = (size_t)w * h * sizeof(float);
    float *d = nullptr;
    if (cudaMalloc(&d, bytes) != cudaSuccess) {
        cudaGetLastError();
        return fail(S2PB_ERR_NOMEM, "cudaMalloc of %zu bytes failed for the geoid grid", bytes);
    }
    if (cudaError_t e = cudaMemcpy(d, grid, bytes, cudaMemcpyHostToDevice)) {
        cudaFree(d);
        return fail(S2PB_ERR_CUDA, "copy of the geoid grid failed: %s", cudaGetErrorString(e));
    }
    geoid_free(ctx);
    ctx->geoid = GeoidGrid{d, w, h, lon0, lat0, dlon, dlat};
    return S2PB_OK;
}
