// triangulation_kernels.cuh -- disparity -> (lon, lat, alt) by RPC ray intersection (SURVEY.md section 8f rank 2).
//
// Behavioural reference (what the numbers must agree with, to 1e-9 degree / 1e-6 m): disp_to_lonlatalt, c/disp_to_h.c:70-141,
// which searches the height at which the ray of pixel a, projected into image b, passes closest to the matched pixel
// (rpc_height, c/rpc.c:480-515), with the RPC camera model of c/rpc.c:279-462 -- four cubic polynomials in three
// normalised variables per direction, the ground->image direction always present, the image->ground direction either
// given or obtained by a Newton iteration on the other one (:378-411).
//
// The organisation is ours.  One thread owns one pixel and works on the problem's actual structure:
//   * a cubic in (x, y, z) is kept as a cubic in z with coefficients in (x, y): Z-FORM.  Image a's pixel is FIXED during
//     the height search, so its four polynomials collapse once per pixel into 4 x 4 numbers and every later evaluation
//     at a new height is four Horner steps instead of 4 x 20 products;
//   * where all three variables move (projection into image b, Newton steps) the 19 non-constant monomials are formed
//     ONCE per point and shared by the four polynomials of that point (the reference rebuilds them for each);
//   * both camera models travel as __grid_constant__ kernel parameters, i.e. in the constant bank: every coefficient read
//     is a broadcast, no thread keeps a coefficient in a register.
// Sums run in another order than the reference's left-to-right 20-term loop, which itself depends on the FMA contraction
// of the -O3 -march=native build; both effects are ~1e-16 relative, nine orders below the tolerance.
#pragma once
#include <cuda_runtime.h>

namespace s2pb {

struct RpcModel {            // same layout as `struct rpc` (c/rpc.h:14-32) / s2p.triangulation.RPCStruct
    double numx[20], denx[20], numy[20], deny[20], scale[3], offset[3];
    double inumx[20], idenx[20], inumy[20], ideny[20], iscale[3], ioffset[3];
    double dmval[4], imval[4];
    double delta;
};

// Monomial table of the RPC00B cubic in the reference's variable order (c/rpc.c:279-297: the first argument plays "lig",
// the second "col"): index -> (power of first, power of second, power of third argument)
//   0:1  1:u  2:v  3:w  4:uv  5:uw  6:vw  7:uu  8:vv  9:ww  10:uvw  11:uuu  12:uvv  13:uww  14:uuv  15:vvv  16:vww  17:uuw  18:vvw  19:www
// with u = first argument, v = second, w = third (height).
struct Mono { double u, v, w, uv, uw, vw, uu, vv, ww, uvw, uuu, uvv, uww, uuv, vvv, vww, uuw, vvw, www; };
__device__ __forceinline__ Mono monomials(double u, double v, double w)
{
    Mono m;
    m.u = u; m.v = v; m.w = w;
    m.uv = u * v; m.uw = u * w; m.vw = v * w; m.uu = u * u; m.vv = v * v; m.ww = w * w;
    m.uvw = m.uv * w; m.uuu = m.uu * u; m.uvv = m.uv * v; m.uww = m.uw * w; m.uuv = m.uu * v;
    m.vvv = m.vv * v; m.vww = m.vw * w; m.uuw = m.uu * w; m.vvw = m.vv * w; m.www = m.ww * w;
    return m;
}
__device__ __forceinline__ double dot20(const double *c, const Mono &m)
{
    double r = c[0];
    r = fma(c[1], m.u, r);    r = fma(c[2], m.v, r);    r = fma(c[3], m.w, r);    r = fma(c[4], m.uv, r);
    r = fma(c[5], m.uw, r);   r = fma(c[6], m.vw, r);   r = fma(c[7], m.uu, r);   r = fma(c[8], m.vv, r);
    r = fma(c[9], m.ww, r);   r = fma(c[10], m.uvw, r); r = fma(c[11], m.uuu, r); r = fma(c[12], m.uvv, r);
    r = fma(c[13], m.uww, r); r = fma(c[14], m.uuv, r); r = fma(c[15], m.vvv, r); r = fma(c[16], m.vww, r);
    r = fma(c[17], m.uuw, r); r = fma(c[18], m.vvw, r); r = fma(c[19], m.www, r);
    return r;
}
// one point through the four polynomials of one direction: (numx / denx, numy / deny)
__device__ __forceinline__ void ratio_pair(const double *numx, const double *denx, const double *numy, const double *deny,
                                           double u, double v, double w, double &rx, double &ry)
{
    const Mono m = monomials(u, v, w);
    rx = dot20(numx, m) / dot20(denx, m);
    ry = dot20(numy, m) / dot20(deny, m);
}
// Z-form of one polynomial at fixed (u, v): p(w) = z[0] + z[1] w + z[2] w^2 + z[3] w^3
__device__ __forceinline__ void zform(const double *c, double u, double v, double (&z)[4])
{
    const double uu = u * u, vv = v * v, uv = u * v;
    z[0] = c[0] + c[1] * u + c[2] * v + c[4] * uv + c[7] * uu + c[8] * vv + c[11] * (uu * u) + c[12] * (uv * v) + c[14] * (uu * v) + c[15] * (vv * v);
    z[1] = c[3] + c[5] * u + c[6] * v + c[10] * uv + c[17] * uu + c[18] * vv;
    z[2] = c[9] + c[13] * u + c[16] * v;
    z[3] = c[19];
}
__device__ __forceinline__ double horner3(const double (&z)[4], double w) { return fma(fma(fma(z[3], w, z[2]), w, z[1]), w, z[0]); }

// The camera of image a seen from one of its pixels: the pixel is fixed, only the height varies.
// With the image->ground polynomials (direct model) it is four z-forms; without them the reference inverts the
// ground->image polynomials by Newton steps from a fixed start (c/rpc.c:378-411), which needs the full evaluation.
struct PixelRay {
    bool direct;
    double zx[4], zdx[4], zy[4], zdy[4];     // direct: z-forms of numx, denx, numy, deny at the normalised pixel
    double xn, yn;                           // iterative: the normalised pixel
};
__device__ __forceinline__ PixelRay make_ray(const RpcModel &a, double x, double y)
{
    PixelRay r;
    r.xn = (x - a.offset[0]) / a.scale[0];
    r.yn = (y - a.offset[1]) / a.scale[1];
    r.direct = isfinite(a.numx[0]);
    if (r.direct) { zform(a.numx, r.xn, r.yn, r.zx); zform(a.denx, r.xn, r.yn, r.zdx); zform(a.numy, r.xn, r.yn, r.zy); zform(a.deny, r.xn, r.yn, r.zdy); }
    return r;
}
// ground point (lon, lat) of the pixel at height z.  -> false when the iteration stopped at its cap of 1000 steps without
// meeting the reference's stopping test (the reference would loop on); a NaN residual leaves the loop as in c/rpc.c.
__device__ bool ray_at(const RpcModel &a, const PixelRay &r, double z, double &lon, double &lat)
{
    const double w = (z - a.offset[2]) / a.scale[2];
    double ln, lt;
    bool converged = true;
    if (r.direct) {
        ln = horner3(r.zx, w) / horner3(r.zdx, w);
        lt = horner3(r.zy, w) / horner3(r.zdy, w);
    } else {
        // Newton on the ground->image polynomials with one-sided differences, the reference's start point and steps
        double delta = 1.0;
        if (a.delta) delta = a.delta;
        ln = -delta; lt = -delta;
        double eps = 2 * delta;
        double x0, y0, x1, y1, x2, y2;
        ratio_pair(a.inumx, a.idenx, a.inumy, a.ideny, ln, lt, w, x0, y0);
        ratio_pair(a.inumx, a.idenx, a.inumy, a.ideny, ln + eps, lt, w, x1, y1);
        ratio_pair(a.inumx, a.idenx, a.inumy, a.ideny, ln, lt + eps, w, x2, y2);
        int it = 0;
        for (; it < 1000; it++) {                 // (the reference loops until convergence; it takes a handful of steps)
            const double ux = r.xn - x0, uy = r.yn - y0;
            if (!(ux * ux + uy * uy > 1e-18)) break;
            const double e1x = x1 - x0, e1y = y1 - y0, e2x = x2 - x0, e2y = y2 - y0;
            const double det = e1x * e2y - e1y * e2x;
            ln += (e2y * ux - e2x * uy) / det * eps;
            lt += (-e1y * ux + e1x * uy) / det * eps;
            eps = 0.1;
            ratio_pair(a.inumx, a.idenx, a.inumy, a.ideny, ln, lt, w, x0, y0);
            ratio_pair(a.inumx, a.idenx, a.inumy, a.ideny, ln + eps, lt, w, x1, y1);
            ratio_pair(a.inumx, a.idenx, a.inumy, a.ideny, ln, lt + eps, w, x2, y2);
        }
        if (it == 1000) {                         // at the cap: the point of the last step has not been tested yet
            const double ux = r.xn - x0, uy = r.yn - y0;
            converged = !(ux * ux + uy * uy > 1e-18);
        }
    }
    lon = ln * a.iscale[0] + a.ioffset[0];
    lat = lt * a.iscale[1] + a.ioffset[1];
    return converged;
}
// ground point -> pixel of image b
__device__ __forceinline__ void project(const RpcModel &b, double lon, double lat, double z, double &x, double &y)
{
    double px, py;
    ratio_pair(b.inumx, b.idenx, b.inumy, b.ideny, (lon - b.ioffset[0]) / b.iscale[0], (lat - b.ioffset[1]) / b.iscale[1],
               (z - b.ioffset[2]) / b.iscale[2], px, py);
    x = px * b.scale[0] + b.offset[0];
    y = py * b.scale[1] + b.offset[1];
}

struct TriParams {
    const float *dispx, *dispy, *msk, *msk_orig;
    int nx, ny, w, h;
    double ha_inv[9], hb_inv[9];
    RpcModel rpca, rpcb;                      // by value: they live in the constant bank with the other kernel parameters
    float col_min, col_max, row_min, row_max;
    double *lonlatalt;
    float *err;
};
__device__ __forceinline__ void hom_apply(double &y0, double &y1, const double *h, double x0, double x1)
{
    const double z = h[6] * x0 + h[7] * x1 + h[8];
    y0 = (h[0] * x0 + h[1] * x1 + h[2]) / z;
    y1 = (h[3] * x0 + h[4] * x1 + h[5]) / z;
}
__global__ void __maxnreg__(120) triangulate_kernel(const __grid_constant__ TriParams P)
{
    const int col = blockIdx.x * blockDim.x + threadIdx.x, row = blockIdx.y * blockDim.y + threadIdx.y;
    if (col >= P.nx || row >= P.ny) return;
    const size_t pix = (size_t)row * P.nx + col;
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    double o0 = nan, o1 = nan, o2 = nan;
    float oe = __int_as_float(0x7fc00000);
    if (P.msk[pix] != 0.f) {
        double pa0, pa1;
        hom_apply(pa0, pa1, P.ha_inv, (double)col, (double)row);             // the pixel of image a behind this rectified pixel
        const double r0 = round(pa0), r1 = round(pa1);
        bool ok = !(r0 < P.col_min || r0 > P.col_max || r1 < P.row_min || r1 > P.row_max);     // image-domain bounding box
        if (ok) {
            const int x = (int)((float)(int)r0 - P.col_min), y = (int)((float)(int)r1 - P.row_min);
            if (x < P.w && y < P.h && P.msk_orig[(size_t)y * P.w + x] == 0.f) ok = false;       // image-domain mask
        }
        if (ok) {
            double qb0, qb1;
            hom_apply(qb0, qb1, P.hb_inv, (double)col + (double)P.dispx[pix], (double)row + (double)P.dispy[pix]);   // its match in image b
            const PixelRay ray = make_ray(P.rpca, pa0, pa1);
            // height search: project the ray's points at h and h + 1 into image b, move h by the matched pixel's abscissa on
            // that segment (at most 100 times, until the move is below 1e-5 m); the residual distance is the error
            double h = 0, e = 0;
            for (int t = 0; t < 100; t++) {
                double lon, lat, p0, p1, q0, q1;
                ray_at(P.rpca, ray, h, lon, lat);
                project(P.rpcb, lon, lat, h, p0, p1);
                ray_at(P.rpca, ray, h + 1, lon, lat);
                project(P.rpcb, lon, lat, h + 1, q0, q1);
                const double a0 = q0 - p0, a1 = q1 - p1, b0 = qb0 - p0, b1 = qb1 - p1;
                const double lambda = (a0 * b0 + a1 * b1) / (a0 * a0 + a1 * a1);
                e = hypot(p0 + lambda * a0 - qb0, p1 + lambda * a1 - qb1);
                h += lambda;
                if (fabs(lambda) < 0.00001) break;
            }
            ray_at(P.rpca, ray, h, o0, o1);
            o2 = h; oe = (float)e;
        }
    }
    P.lonlatalt[3 * pix + 0] = o0;
    P.lonlatalt[3 * pix + 1] = o1;
    P.lonlatalt[3 * pix + 2] = o2;
    P.err[pix] = oe;
}

// Localisation of a height map (s2p.triangulation.height_map_to_xyz, s2p/triangulation.py:165-217): pixel (i, j) of a w x h
// map with height z is the ground point of image pixel (j + off_x, i + off_y) at height z (rpc_localization, c/rpc.c:469),
// written as (lon, lat, z).  A NaN height gives NaN in all three; a pixel whose iteration hits its cap is counted in *capped.
struct HeightMapParams {
    const double *heights;
    int w, h;
    double off_x, off_y;
    RpcModel rpc;                             // by value: the constant bank
    double *xyz;
    int *capped;
};
__global__ void height_map_to_xyz_kernel(const __grid_constant__ HeightMapParams P)
{
    const int col = blockIdx.x * blockDim.x + threadIdx.x, row = blockIdx.y * blockDim.y + threadIdx.y;
    if (col >= P.w || row >= P.h) return;
    const size_t pix = (size_t)row * P.w + col;
    const double z = P.heights[pix];
    double lon = z, lat = z;                  // NaN stays NaN
    if (!isnan(z)) {
        const PixelRay ray = make_ray(P.rpc, (double)col + P.off_x, (double)row + P.off_y);
        if (!ray_at(P.rpc, ray, z, lon, lat)) atomicAdd(P.capped, 1);
    }
    P.xyz[3 * pix + 0] = lon;
    P.xyz[3 * pix + 1] = lat;
    P.xyz[3 * pix + 2] = z;
}

}  // namespace s2pb
