// projection.cu -- the change of coordinates of s2p.triangulation.disp_to_xyz: WGS84 (lon, lat, alt) -> UTM, the ETRS89 UTM
// zones and the RGF93 Lambert grids (S2PB_ZONE_PROJ), and the EGM96 geoid heights of the compound targets (EPSG:326zz+5773,
// 327zz+5773, 4326+5773, and those grids +5773).
#include "host.h"

#include <cmath>

// The coefficients of projection_kernels.cuh's transverse Mercator with scale k0 on the ellipsoid (a, f), in double.  The
// series in the third flattening n are those of Karney (2011), eq. (35) for alpha (Krueger's series, ellipsoid <- sphere) and
// the conformal-latitude series of Engsager and Poder (2007), both to order n^6, as PROJ evaluates them for its exact
// transverse Mercator.
static UtmParams tm_params(double a, double f, double k0, double lon0, double x0, double y0)
{
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
    P.lon0 = lon0;
    P.x0 = x0;
    P.y0 = y0;
    return P;
}

// UTM zone `zone` (1..60) of WGS84
static UtmParams utm_params(int zone, bool south)
{
    return tm_params(6378137.0, 1.0 / 298.257223563, 0.9996, 6.0 * zone - 183.0, 500000.0, south ? 10000000.0 : 0.0);
}

// The constants of lcc_forward (EPSG method 9802, IOGP Guidance Note 7-2 sec. 3.1.1.1), in double, with t = exp(-psi):
// m(phi) = cos phi / sqrt(1 - e^2 sin^2 phi); n = (ln m1 - ln m2) / (psi2 - psi1) (sin phi1 when the parallels coincide);
// F = m1 exp(n psi1) / n; r_F = a F exp(-n psi_F), 0 at the pole the cone opens to.
static LccParams lcc_params(const s2pb_projection &p)
{
    const double d2r = 0.017453292519943295, f = 1.0 / p.rf, e2 = f * (2.0 - f), e = std::sqrt(e2);
    auto m = [&](double phi) { const double s = std::sin(phi); return std::cos(phi) / std::sqrt(1.0 - e2 * s * s); };
    auto psi = [&](double phi) { return std::asinh(std::tan(phi)) - e * std::atanh(e * std::sin(phi)); };
    const double phi1 = p.lat1 * d2r, phi2 = p.lat2 * d2r, phi0 = p.lat0 * d2r;
    LccParams P;
    P.lon0 = p.lon0;
    P.e = e;
    P.n = p.lat1 == p.lat2 ? std::sin(phi1) : (std::log(m(phi1)) - std::log(m(phi2))) / (psi(phi2) - psi(phi1));
    P.aF = p.a * (m(phi1) * std::exp(P.n * psi(phi1)) / P.n);
    P.rho0 = std::fabs(p.lat0) == 90.0 ? 0.0 : P.aF * std::exp(-(P.n * psi(phi0)));
    P.x0 = p.x0;
    P.y0 = p.y0;
    return P;
}

// *proj checked (the rules of s2pb_set_projection) into the kernel's map and parameters
static int projection_map(const s2pb_projection *proj, MapKind *kind, MapParams *P)
{
    if (!proj) return fail(S2PB_ERR_ARG, "bad argument");
    const s2pb_projection &p = *proj;
    if (p.method != S2PB_PROJ_TM && p.method != S2PB_PROJ_LCC) return fail(S2PB_ERR_ARG, "unknown projection method %d", p.method);
    const bool tm = p.method == S2PB_PROJ_TM;
    const double vals[] = {p.a, p.rf, p.lon0, p.lat0, p.x0, p.y0, tm ? p.k0 : p.lat1, tm ? 0.0 : p.lat2};
    for (double v : vals)
        if (!std::isfinite(v)) return fail(S2PB_ERR_ARG, "a projection parameter is not finite");
    if (!(p.a > 0.0) || !(p.rf > 1.0)) return fail(S2PB_ERR_ARG, "ellipsoid a = %g, 1/f = %g", p.a, p.rf);
    if (tm) {
        if (!(p.k0 > 0.0) || p.lat0 != 0.0)
            return fail(S2PB_ERR_ARG, "transverse Mercator: k0 = %g must be > 0 and lat0 = %g must be 0", p.k0, p.lat0);
        *kind = MapKind::kTm;
        P->tm = tm_params(p.a, 1.0 / p.rf, p.k0, p.lon0, p.x0, p.y0);
        return S2PB_OK;
    }
    if (!(std::fabs(p.lat1) < 90.0) || !(std::fabs(p.lat2) < 90.0) || p.lat1 == -p.lat2 || !(std::fabs(p.lat0) <= 90.0) ||
        (std::fabs(p.lat0) == 90.0 && (p.lat0 > 0.0) != (p.lat1 + p.lat2 > 0.0)))
        return fail(S2PB_ERR_ARG, "Lambert conic: parallels %g and %g, false origin latitude %g", p.lat1, p.lat2, p.lat0);
    *kind = MapKind::kLcc;
    P->lcc = lcc_params(p);
    return S2PB_OK;
}

extern "C" int s2pb_set_projection(s2pb_ctx *ctx, const s2pb_projection *proj)
{
    if (!ctx) return fail(S2PB_ERR_ARG, "bad argument");
    if (!proj) {
        ctx->proj_kind = MapKind::kNone;
        return S2PB_OK;
    }
    MapKind kind;
    MapParams P;
    if (int rc = projection_map(proj, &kind, &P)) return rc;
    ctx->proj_kind = kind;
    ctx->proj = P;
    return S2PB_OK;
}

int cloud_crs_ok(const s2pb_ctx *ctx, int zone, int south, bool zone0)
{
    if (zone0 && (zone & S2PB_ZONE_PROJ)) {
        if (zone & ~(S2PB_ZONE_PROJ | S2PB_ZONE_EGM96))
            return fail(S2PB_ERR_ARG, "zone %#x: S2PB_ZONE_PROJ takes no UTM zone, only S2PB_ZONE_EGM96", zone);
        if (ctx->proj_kind == MapKind::kNone) return fail(S2PB_ERR_ARG, "S2PB_ZONE_PROJ on a context without a projection");
        if (south) return fail(S2PB_ERR_ARG, "S2PB_ZONE_PROJ with south = %d: the projection holds its false northing", south);
    } else {
        const int utm = zone & ~S2PB_ZONE_EGM96;
        if (utm < (zone0 ? 0 : 1) || utm > 60)
            return fail(S2PB_ERR_ARG, "zone %d: a UTM zone 1 to 60%s, optionally OR S2PB_ZONE_EGM96", zone,
                        zone0 ? ", or 0 for lon, lat, or S2PB_ZONE_PROJ" : "");
    }
    if ((zone & S2PB_ZONE_EGM96) && !ctx->geoid.g) return fail(S2PB_ERR_ARG, "S2PB_ZONE_EGM96 on a context without a geoid grid");
    return S2PB_OK;
}

// cloud_project_kernel<kind, geoid> over n points
static int launch_map(s2pb_ctx *ctx, cudaStream_t st, MapKind kind, const MapParams &P, bool geoid, const double *d_in,
                      double *d_out, size_t n)
{
    const unsigned b = 256;
    const dim3 g((unsigned)((n + b - 1) / b));
    auto go = [&](auto kernel, const auto &arg) {
        launch(ctx, kernel, g, dim3(b), 0, st, arg, ctx->geoid, d_in, d_out, (long long)n);
    };
    switch (kind) {
    case MapKind::kTm:
        geoid ? go(cloud_project_kernel<MapKind::kTm, true>, P.tm) : go(cloud_project_kernel<MapKind::kTm, false>, P.tm);
        break;
    case MapKind::kLcc:
        geoid ? go(cloud_project_kernel<MapKind::kLcc, true>, P.lcc) : go(cloud_project_kernel<MapKind::kLcc, false>, P.lcc);
        break;
    case MapKind::kNone: go(cloud_project_kernel<MapKind::kNone, true>, P.tm); break;
    }
    CK(cudaGetLastError());
    return S2PB_OK;
}

int launch_cloud_project(s2pb_ctx *ctx, cudaStream_t st, int zone, bool south, const double *d_in, double *d_out, size_t n)
{
    const bool geoid = (zone & S2PB_ZONE_EGM96) != 0;
    if (zone & S2PB_ZONE_PROJ) return n ? launch_map(ctx, st, ctx->proj_kind, ctx->proj, geoid, d_in, d_out, n) : S2PB_OK;
    const int utm = zone & ~S2PB_ZONE_EGM96;
    if (n == 0 || (!utm && !geoid)) return S2PB_OK;
    MapParams P;
    P.tm = utm_params(utm, south);
    return launch_map(ctx, st, utm ? MapKind::kTm : MapKind::kNone, P, geoid, d_in, d_out, n);
}

extern "C" int s2pb_lonlat_to_utm(s2pb_ctx *ctx, double *xyz, const double *lonlatalt, int64_t n, int zone, int south)
{
    if (!ctx || n < 0 || (n > 0 && (!xyz || !lonlatalt))) return fail(S2PB_ERR_ARG, "bad argument");
    if (int rc = cloud_crs_ok(ctx, zone, south, false)) return rc;
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

extern "C" int s2pb_lonlat_to_proj(s2pb_ctx *ctx, double *xyz, const double *lonlatalt, int64_t n, const s2pb_projection *proj)
{
    if (!ctx || n < 0 || (n > 0 && (!xyz || !lonlatalt))) return fail(S2PB_ERR_ARG, "bad argument");
    MapKind kind;
    MapParams P;
    if (int rc = projection_map(proj, &kind, &P)) return rc;
    if (n == 0) return S2PB_OK;
    const size_t bytes = (size_t)n * 24;
    HostCall L(ctx, "the projection");
    double *d = L.upload(lonlatalt, bytes);
    if (int rc = L.error()) return rc;
    int rc = launch_map(ctx, L.st, kind, P, false, d, d, (size_t)n);
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
