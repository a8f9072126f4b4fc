// projection_kernels.cuh -- WGS84 (lon, lat, alt) -> UTM (easting, northing, alt), forward, one thread per point; the
// Lambert conic conformal map of the French grids (lcc_forward below); and the EGM96 geoid heights of a compound target such
// as EPSG:326zz+5773 (GeoidGrid below).
//
// The map is the one PROJ runs for `+proj=utm` unless `+approx` is given: the "exact" transverse Mercator of Poder and
// Engsager (K. Engsager, K. Poder, "A highly accurate world wide algorithm for the transverse Mercator mapping (almost)",
// XXIII ICA conference, 2007), i.e. Krueger's series in the third flattening n carried to order n^6, in the form and with
// the coefficients of C. F. F. Karney, "Transverse Mercator with an accuracy of a few nanometers", J. Geodesy 85 (2011)
// 475-485, eqs. (7)-(11) and (35).  Within 4000 km of the central meridian its error is a few nanometres (Karney, sec. 4).
// Four steps per point:
//   1. geodetic latitude phi -> conformal (Gaussian) latitude chi = phi + sum_k cbg[k] sin(2 k phi), a Clenshaw sum;
//   2. the spherical transverse Mercator of (chi, lambda): xi' = atan2(sin chi, cos chi cos lambda),
//      eta' = asinh(sin lambda cos chi / hypot(sin chi, cos chi cos lambda))  (Karney eq. 10);
//   3. Krueger's series xi + i eta = zeta' + sum_k gtu[k] sin(2 k zeta'), zeta' = xi' + i eta', by a complex Clenshaw sum whose
//      sin / cos 2xi' and sinh / cosh 2eta' come from the quantities of step 2 without further transcendental calls;
//   4. scale by k0 times the rectifying radius and add the false easting / northing.
// The coefficients depend on the ellipsoid only; the host computes them in double (projection.cu) and they travel as a
// __grid_constant__ kernel parameter, in the constant bank, as the triangulation kernels pass their camera models.  The same
// map on GRS80 gives the ETRS89 UTM zones (EPSG 25828-25838): only the coefficients, qa and the origin differ.
#pragma once
#include <cuda_runtime.h>

namespace s2pb {

constexpr int kUtmOrder = 6;              // order of both series, in n

struct UtmParams {
    double cbg[kUtmOrder];                // geodetic -> conformal latitude: chi - phi = sum_k cbg[k] sin(2 (k+1) phi)
    double gtu[kUtmOrder];                // Krueger's alpha_1..alpha_6: spherical -> ellipsoidal normalised TM
    double lon0;                          // central meridian, degrees: 6 zone - 183
    double qa;                            // a k0 A: metres per unit of the normalised (xi, eta)
    double x0, y0;                        // false easting, false northing, metres
};

// (lon, lat) in degrees -> (x, y) in metres, in this operation order (tests/utm_oracle.py restates it in numpy).
// Points outside the projection's domain -- |lat| > 90, or so far from the central meridian that |eta| > 2.623395162778,
// Engsager's bound -- give +inf, as PROJ flags a point it cannot project with HUGE_VAL.
__device__ __forceinline__ void utm_forward(const UtmParams &P, double lon, double lat, double &x, double &y)
{
    const double d2r = 0.017453292519943295;      // pi / 180
    double lam = (lon - P.lon0) * d2r;
    if (fabs(lam) > 3.141592653589793) lam -= 6.283185307179586 * floor((lam + 3.141592653589793) / 6.283185307179586);
    const double phi = lat * d2r;
    // 1. conformal latitude: Clenshaw on sin(2 k phi), k = 1..6
    const double s2 = sin(2.0 * phi), c2 = cos(2.0 * phi), tc2 = 2.0 * c2;
    double h1 = P.cbg[kUtmOrder - 1], h2 = 0.0, h = h1;
    for (int k = kUtmOrder - 2; k >= 0; k--) {
        h = -h2 + tc2 * h1 + P.cbg[k];
        h2 = h1;
        h1 = h;
    }
    const double chi = phi + h * s2;
    // 2. spherical transverse Mercator
    const double sc = sin(chi), cc = cos(chi), sl = sin(lam), cl = cos(lam);
    const double ccl = cc * cl;
    const double xip = atan2(sc, ccl);
    const double inv_d = 1.0 / hypot(sc, ccl);    // 1 / cos(asin(cos chi sin lambda)) = cosh eta'
    const double sinh_e = sl * cc * inv_d;        // sinh eta'
    const double etap = asinh(sinh_e);
    // 3. Krueger: sin 2xi' = 2 sin xi' cos xi', cos 2xi' = 2 cos^2 xi' - 1, sinh 2eta' = 2 sinh eta' cosh eta',
    //    cosh 2eta' = 2 cosh^2 eta' - 1, with sin xi' = sc inv_d, cos xi' = ccl inv_d, cosh eta' = inv_d
    const double two_inv_d = 2.0 * inv_d;
    const double two_inv_d2 = two_inv_d * inv_d;
    const double t = ccl * two_inv_d2;
    const double sin2x = sc * t, cos2x = ccl * t - 1.0;
    const double sinh2e = sinh_e * two_inv_d, cosh2e = two_inv_d2 - 1.0;
    // complex Clenshaw on sin(2 k zeta'): multiplier 2 cos(2 zeta') = r + i q, final factor sin(2 zeta') = sr + i si
    const double r = 2.0 * cos2x * cosh2e, q = -2.0 * sin2x * sinh2e;
    double hr = P.gtu[kUtmOrder - 1], hi = 0.0, hr1 = 0.0, hi1 = 0.0, hr2, hi2;
    for (int k = kUtmOrder - 2; k >= 0; k--) {
        hr2 = hr1; hi2 = hi1; hr1 = hr; hi1 = hi;
        hr = -hr2 + r * hr1 - q * hi1 + P.gtu[k];
        hi = -hi2 + q * hr1 + r * hi1;
    }
    const double sr = sin2x * cosh2e, si = cos2x * sinh2e;
    const double xi = xip + (sr * hr - si * hi);
    const double eta = etap + (sr * hi + si * hr);
    // 4. metres
    if (!(fabs(lat) <= 90.0) || fabs(eta) > 2.623395162778) {
        x = y = __longlong_as_double(0x7ff0000000000000LL);
        return;
    }
    x = P.qa * eta + P.x0;
    y = P.qa * xi + P.y0;
}

// The Lambert conic conformal map with two standard parallels (EPSG method 9802, IOGP Guidance Note 7-2 sec. 3.1.1.1) of
// RGF93 v1 / Lambert-93 (EPSG:2154) and the nine zones CC42-CC50 (EPSG 3942-3950), on GRS80.  With the isometric latitude
// psi(phi) = asinh(tan phi) - e atanh(e sin phi), the note's t(phi) is exp(-psi), so the radius r = a F t^n is a F exp(-n psi).
// The host computes the cone constant n, a F and r_F = a F t(phi_F)^n (projection.cu).
struct LccParams {
    double lon0;                          // longitude of the false origin, degrees
    double e;                             // first eccentricity
    double n;                             // cone constant
    double aF;                            // a F, metres
    double rho0;                          // r_F: radius at the latitude of the false origin, metres
    double x0, y0;                        // easting, northing at the false origin, metres
};

// (lon, lat) in degrees -> (x, y) in metres, in this operation order (tests/lcc_oracle.py restates it in numpy):
//   lam = (lon - lon0) d2r, reduced to [-pi, pi] as utm_forward reduces it; phi = lat d2r;
//   psi = asinh(tan phi) - e atanh(e sin phi);  rho = aF exp(-(n psi));  theta = n lam;
//   x = x0 + rho sin theta;  y = y0 + (rho0 - rho cos theta).
// A pole (| |phi| - pi/2 | < 1e-10 rad) is the apex of the cone, rho = 0, on the side the cone opens to (phi n > 0); on the
// other side, and for |lat| > 90, the point cannot be projected and gives +inf, as PROJ flags it with HUGE_VAL.
__device__ __forceinline__ void lcc_forward(const LccParams &P, double lon, double lat, double &x, double &y)
{
    const double d2r = 0.017453292519943295;      // pi / 180
    double lam = (lon - P.lon0) * d2r;
    if (fabs(lam) > 3.141592653589793) lam -= 6.283185307179586 * floor((lam + 3.141592653589793) / 6.283185307179586);
    const double phi = lat * d2r;
    const bool pole = fabs(fabs(phi) - 1.5707963267948966) < 1e-10;
    if (!(fabs(lat) <= 90.0) || (pole && phi * P.n <= 0.0)) {
        x = y = __longlong_as_double(0x7ff0000000000000LL);
        return;
    }
    double rho = 0.0;
    if (!pole) {
        const double psi = asinh(tan(phi)) - P.e * atanh(P.e * sin(phi));
        rho = P.aF * exp(-(P.n * psi));
    }
    const double theta = P.n * lam;
    x = P.x0 + rho * sin(theta);
    y = P.y0 + (P.rho0 - rho * cos(theta));
}

// The map of a cloud's output CRS: which one is a template parameter of cloud_project_kernel, and its parameters, which the
// host keeps in the union MapParams, travel as the struct of that map (MapArg), so that the UTM instantiations take the
// UtmParams they always took.
enum class MapKind { kNone, kTm, kLcc };
union MapParams {
    UtmParams tm;                         // kTm (and kNone): utm_forward (WGS84 UTM, ETRS89 UTM)
    LccParams lcc;                        // kLcc: lcc_forward
};
template <MapKind kMap> struct MapArgOf { using type = UtmParams; };
template <> struct MapArgOf<MapKind::kLcc> { using type = LccParams; };
template <MapKind kMap> using MapArg = typename MapArgOf<kMap>::type;
__device__ __forceinline__ void map_forward(const UtmParams &P, double lon, double lat, double &x, double &y)
{
    utm_forward(P, lon, lat, x, y);
}
__device__ __forceinline__ void map_forward(const LccParams &P, double lon, double lat, double &x, double &y)
{
    lcc_forward(P, lon, lat, x, y);
}

// The vertical datum of a cloud: heights above the EGM96 geoid instead of the WGS84 ellipsoid, H = h - N(lon, lat), the
// step PROJ's `+proj=vgridshift` runs for a target such as EPSG:326zz+5773.  N is interpolated bilinearly in a float32 grid
// of h rows of w nodes: node (i, j) lies at (lon0 + i dlon, lat0 - j dlat), row 0 northernmost.  The grid is global: it spans
// at least 360 degrees of longitude, which wraps (column w - 1 is followed by column 0), and every latitude from 90 to -90.
struct GeoidGrid {
    const float *g;                       // h * w nodes, row-major; device memory
    int w, h;
    double lon0, lat0;                    // node (0, 0), degrees
    double dlon, dlat;                    // node spacing, degrees, both > 0
};

// N(lon, lat) for |lat| <= 90 and a finite lon: bilinear in the four float32 nodes around the point, in float64, as two
// interpolations along the row and one across (tests/geoid_oracle.py restates it in numpy).  This form gives a node's value
// at the node and a constant grid's value everywhere exactly; it differs from PROJ's sum of four weighted nodes by rounding
// only.  The last row stands in for the row below it, as PROJ clamps it.
__device__ __forceinline__ double geoid_undulation(const GeoidGrid &G, double lon, double lat)
{
    double t = fmod(lon - G.lon0, 360.0);
    if (t < 0.0) t += 360.0;
    const double x = t / G.dlon, y = (G.lat0 - lat) / G.dlat;
    const int i = min((int)floor(x), G.w - 1), j = max(0, min((int)floor(y), G.h - 1));
    const double fx = x - i, fy = y - j;
    const int i2 = i + 1 < G.w ? i + 1 : 0, j2 = min(j + 1, G.h - 1);
    const double a = G.g[(size_t)j * G.w + i], b = G.g[(size_t)j * G.w + i2];
    const double c = G.g[(size_t)j2 * G.w + i], d = G.g[(size_t)j2 * G.w + i2];
    const double top = a + fx * (b - a), bottom = c + fx * (d - c);
    return top + fy * (bottom - top);
}

// out[i] = (x, y, z) of in[i] = (lon, lat, alt), n points of three doubles; in == out is allowed.  kMap: (x, y) the map of
// (lon, lat) (kTm: utm_forward, kLcc: lcc_forward), kNone: (lon, lat) as they are; kGeoid: z = alt - N(lon,
// lat) in float64, else alt.  A point with a NaN coordinate becomes NaN in all three; a point outside the domain (of the map,
// or |lat| > 90 / an infinite lon for the geoid) becomes +inf in all three.
template <MapKind kMap, bool kGeoid>
__global__ void cloud_project_kernel(const __grid_constant__ MapArg<kMap> P, const __grid_constant__ GeoidGrid G, const double *in,
                                     double *out, long long n)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double lon = in[3 * i], lat = in[3 * i + 1], alt = in[3 * i + 2];
    double x, y, z = alt;
    if (isnan(lon) || isnan(lat) || isnan(alt)) {
        x = y = z = __longlong_as_double(0x7ff8000000000000LL);
    } else {
        bool outside = false;
        if constexpr (kMap != MapKind::kNone) {
            map_forward(P, lon, lat, x, y);
            outside = isinf(x);
        } else {
            x = lon;
            y = lat;
        }
        if (kGeoid && !outside) {
            if (fabs(lat) <= 90.0 && isfinite(lon)) z = alt - geoid_undulation(G, lon, lat);
            else outside = true;
        }
        if (outside) x = y = z = __longlong_as_double(0x7ff0000000000000LL);
    }
    out[3 * i] = x;
    out[3 * i + 1] = y;
    out[3 * i + 2] = z;
}

}  // namespace s2pb
