// warp.cu -- the rectification warp: `homography` (3rdparty/homography) from host memory to host or device memory.
#include "host.h"
#include "homography_kernels.cuh"

#include <cmath>

static void invert33(const double m[9], double o[9])
{   // Homography.cpp:281-303
    const double det = 1.0 / (m[0] * m[4] * m[8] - m[0] * m[5] * m[7] - m[1] * m[3] * m[8] + m[1] * m[5] * m[6] + m[2] * m[3] * m[7] -
                              m[2] * m[4] * m[6]);
    o[0] = det * (m[4] * m[8] - m[5] * m[7]); o[1] = det * (m[2] * m[7] - m[1] * m[8]); o[2] = det * (m[1] * m[5] - m[2] * m[4]);
    o[3] = det * (m[5] * m[6] - m[3] * m[8]); o[4] = det * (m[0] * m[8] - m[2] * m[6]); o[5] = det * (m[2] * m[3] - m[0] * m[5]);
    o[6] = det * (m[3] * m[7] - m[4] * m[6]); o[7] = det * (m[1] * m[6] - m[0] * m[7]); o[8] = det * (m[0] * m[4] - m[1] * m[3]);
}
// adjugate over determinant: invert_homography of c/disp_to_h.c:26-42, also the ROI inverse of 3rdparty/homography/main.cpp.
// It rounds differently from invert33, which multiplies by 1/det as Homography.cpp does.
void invert_homography(const double i[9], double o[9])
{
    const double det = i[0] * i[4] * i[8] + i[2] * i[3] * i[7] + i[1] * i[5] * i[6] - i[2] * i[4] * i[6] - i[1] * i[3] * i[8] - i[0] * i[5] * i[7];
    o[0] = (i[4] * i[8] - i[5] * i[7]) / det; o[1] = (i[2] * i[7] - i[1] * i[8]) / det; o[2] = (i[1] * i[5] - i[2] * i[4]) / det;
    o[3] = (i[5] * i[6] - i[3] * i[8]) / det; o[4] = (i[0] * i[8] - i[2] * i[6]) / det; o[5] = (i[2] * i[3] - i[0] * i[5]) / det;
    o[6] = (i[3] * i[7] - i[4] * i[6]) / det; o[7] = (i[1] * i[6] - i[0] * i[7]) / det; o[8] = (i[0] * i[4] - i[1] * i[3]) / det;
}
static float min_sv_jacobian(const double m[9], double px, double py)
{   // getMinSVJacob, Homography.cpp:174-198
    const double X[3] = {m[0] * px + m[1] * py + m[2], m[3] * px + m[4] * py + m[5], m[6] * px + m[7] * py + m[8]};
    const double z = 1.0 / X[2], x = z * X[0], y = z * X[1];
    const double a = z * (m[0] - m[6] * x), b = z * (m[1] - m[7] * x), c = z * (m[3] - m[6] * y), d = z * (m[4] - m[7] * y);
    return (float)sqrt(0.5 * (a * a + b * b + c * c + d * d -
                              sqrt((a * a + b * b - c * c - d * d) * (a * a + b * b - c * c - d * d) + 4.0 * (a * c + b * d) * (a * c + b * d))));
}
static float min_zoom_out(const double m[9], size_t w, size_t h)
{   // getMinZoomOut, Homography.cpp:203-212
    float r = std::fmin(min_sv_jacobian(m, 0, (double)h), min_sv_jacobian(m, (double)w, (double)h));
    r = std::fmin(min_sv_jacobian(m, (double)w, 0), r);
    r = std::fmin(min_sv_jacobian(m, 0, 0), r);
    return std::fmin(1.f, r);
}

// mapImage (Homography.cpp:50-168) on device images; recursive through the anti-aliasing branch.
static int map_image(s2pb_ctx *ctx, ScratchLease &L, cudaStream_t st, const float *d_src, int w, int h, const double M[9],
                     float *d_out, int ow, int oh, bool use_aa, int depth)
{
    if (depth > 6) return fail(S2PB_ERR_ARG, "homography: anti-aliasing recursion does not settle");
    dim3 b2(32, 8);
    const float zoomOut = use_aa ? min_zoom_out(M, (size_t)w, (size_t)h) : 1.f;
    const bool useZ = zoomOut < 1.f;
    double matZ[9] = {0};
    float *tmp, *scratch;
    const float zoomIn = 1.0f / zoomOut;
    int tw = w, th = h;                        // the spline image: the source, or the anti-aliasing intermediate
    if (useZ) {
        tw = (int)std::ceil((size_t)ow * zoomIn * 1.5);
        th = (int)std::ceil((size_t)oh * zoomIn * 1.5);
        if (tw < 1 || th < 1 || (size_t)tw * th > ((size_t)1 << 31)) return fail(S2PB_ERR_ARG, "homography: degenerate zoom %g", (double)zoomIn);
    }
    // Below 4 samples a side the prefilter's initBackward and the border formula's single reflection index outside the
    // image, and the reference produces no image (prepareSpline's `i < height - 4` wraps around in size_t).
    if (tw < kSplineMinSide || th < kSplineMinSide)
        return fail(S2PB_ERR_ARG, "homography: the %s is %d x %d pixels; the order-5 spline needs %d x %d at least",
                    useZ ? "anti-aliasing intermediate" : "region of interest", tw, th, kSplineMinSide, kSplineMinSide);
    if (useZ) {
        for (int k = 0; k < 6; k++) matZ[k] = zoomIn * M[k];
        for (int k = 6; k < 9; k++) matZ[k] = M[k];
        tmp = L.take<float>((size_t)tw * th * 4);
        scratch = L.take<float>((size_t)tw * th * 4);
        if (!tmp || !scratch) return L.nomem("the warp");
        int rc = map_image(ctx, L, st, d_src, w, h, matZ, tmp, tw, th, true, depth + 1);
        if (rc != S2PB_OK) return rc;
        // Gaussian of sigma = 0.8 sqrt(zoomIn^2 - 1) (Homography.cpp:101-102, LibImages.cpp:506-687)
        const float sigma = 0.8f * std::sqrt(zoomIn * zoomIn - 1.f);
        GaussKernel K;
        int ks = (int)(8.f * sigma + 1.f);
        ks = ks > 3 ? ks + 1 - ks % 2 : 3;
        if (ks > 64) return fail(S2PB_ERR_UNSUPPORTED, "homography: zoom-out of %g needs a %d-tap anti-aliasing filter (64 supported)", (double)zoomIn, ks);
        K.size = ks;
        float sum = 0.f;
        for (int i = 0; i < ks; i++) { const float x = (float)(i - ks / 2); K.k[i] = std::exp(-x * x / (2.f * sigma * sigma)); sum += K.k[i]; }
        for (int i = 0; i < ks; i++) K.k[i] /= sum;
        int jlim = 0;
        while (jlim < tw - 4) jlim += 4;       // first column of the reference's scalar tail
        launch(ctx, gauss_rows_kernel, grid2d(tw, th, b2), b2, 0, st, tmp, scratch, tw, th, K);
        launch(ctx, gauss_cols_kernel, grid2d(tw, th, b2), b2, 0, st, scratch, tmp, tw, th, K, jlim);
        matZ[0] = zoomOut; matZ[1] = 0; matZ[2] = 0; matZ[3] = 0; matZ[4] = zoomOut; matZ[5] = 0; matZ[6] = 0; matZ[7] = 0; matZ[8] = 1;
    } else {
        tmp = L.take<float>((size_t)w * h * 4);
        scratch = L.take<float>((size_t)w * h * 4);
        if (!tmp || !scratch) return L.nomem("the warp");
        CK(cudaMemcpyAsync(tmp, d_src, (size_t)w * h * 4, cudaMemcpyDeviceToDevice, st));
    }
    // prepareSpline (Splines.cpp:26-121): NaN -> 0, 2-pole prefilter along rows, then along columns
    const size_t n = (size_t)tw * th;
    const float lambda = (float)(1.430575 * (1.0 + 1.0 / 0.430575) * 1.0430963 * (1.0 + 1.0 / 0.0430963));
    const double z0 = -0.430575, z1 = -0.0430963;
    launch(ctx, nan_to_zero_kernel, (unsigned)((n + 255) / 256), 256, 0, st, tmp, n);
    dim3 bt(32, 8);
    // prefilter along x (on the transposed image) then along y; `a` holds the data, `b` is the other buffer
    auto prefilter = [&](float *a, float *b, int lw, int lh) {      // columns of an lw x lh image, result back in a
        if (lh >= 2 * kSplineSeg) {
            dim3 g((lw + 127) / 128, (lh + kSplineSeg - 1) / kSplineSeg);
            launch(ctx, spline_segments_kernel, g, 128, 0, st, a, b, lw, lh, lambda, z0);
            launch(ctx, spline_segments_kernel, g, 128, 0, st, b, a, lw, lh, 1.f, z1);
        } else {
            launch(ctx, spline_columns_kernel, (lw + 31) / 32, 32, 0, st, a, lw, lh, lambda, z0, z1);
        }
    };
    launch(ctx, transpose_kernel, dim3((tw + 31) / 32, (th + 31) / 32), bt, 0, st, tmp, tw, th, scratch);
    prefilter(scratch, tmp, th, tw);                                                // rows of the image
    launch(ctx, transpose_kernel, dim3((th + 31) / 32, (tw + 31) / 32), bt, 0, st, scratch, th, tw, tmp);
    prefilter(tmp, scratch, tw, th);
    Mat9 Hi;
    invert33(useZ ? matZ : M, Hi.m);
    launch(ctx, spline_warp_kernel, grid2d(ow, oh, b2), b2, 0, st, tmp, tw, th, Hi, d_out, ow, oh);
    if (useZ) {
        Mat9 Ht;
        invert33(M, Ht.m);
        launch(ctx, warp_mask_kernel, grid2d(ow, oh, b2), b2, 0, st, d_out, ow, oh, Ht, w, h);
    }
    CK(cudaGetLastError());
    return S2PB_OK;
}

// The part of `homography im -h "..." out w h` (3rdparty/homography/main.cpp:65-177) between reading and writing: needed
// region of the host image `src`, upload of that region only, crop compensation of H, warp into the DEVICE image d_out.
// Asynchronous on `st`; its scratch comes from the caller's lease.
int warp_host_to_device(s2pb_ctx *ctx, ScratchLease &L, cudaStream_t st, const float *src, int sw, int sh, const double H[9],
                        float *d_out, int dw, int dh)
{
    // needed ROI of the source: pre-image of the output corners, integer bounding box, clipped (main.cpp:29-55,94-127)
    double Hi[9];
    invert_homography(H, Hi);
    const double cx[4] = {0, (double)dw, (double)dw, 0}, cy[4] = {0, 0, (double)dh, (double)dh};
    double px[4], py[4];
    for (int k = 0; k < 4; k++) {
        double z = Hi[6] * cx[k] + Hi[7] * cy[k] + Hi[8];
        px[k] = (Hi[0] * cx[k] + Hi[1] * cy[k] + Hi[2]) / z;
        py[k] = (Hi[3] * cx[k] + Hi[4] * cy[k] + Hi[5]) / z;
    }
    double mnx = px[0], mxx = px[0], mny = py[0], mxy = py[0];
    for (int k = 1; k < 4; k++) { if (px[k] < mnx) mnx = px[k]; if (px[k] > mxx) mxx = px[k]; if (py[k] < mny) mny = py[k]; if (py[k] > mxy) mxy = py[k]; }
    if (!(std::isfinite(mnx) && std::isfinite(mxx) && std::isfinite(mny) && std::isfinite(mxy))) return fail(S2PB_ERR_ARG, "homography: degenerate matrix");
    if (mnx < -1e9 || mny < -1e9 || mxx > 1e9 || mxy > 1e9) return fail(S2PB_ERR_ARG, "homography: region of interest out of range");
    int x = (int)std::floor(mnx), y = (int)std::floor(mny), w = (int)std::ceil(mxx - x), h = (int)std::ceil(mxy - y);
    if (x < 0) { w += x; x = 0; }
    if (y < 0) { h += y; y = 0; }
    if (x + w > sw) w = sw - x;
    if (y + h > sh) h = sh - y;
    if (w <= 0 || h <= 0) return fail(S2PB_ERR_ARG, "ERROR: empty roi");
    const double T[9] = {1, 0, (double)x, 0, 1, (double)y, 0, 0, 1};
    double Hc[9];
    for (int r = 0; r < 3; r++) for (int q = 0; q < 3; q++) Hc[3 * r + q] = H[3 * r] * T[q] + H[3 * r + 1] * T[3 + q] + H[3 * r + 2] * T[6 + q];
    float *roi = L.take<float>((size_t)w * h * 4);
    if (!roi) return L.nomem("the warp");
    CK(cudaMemcpy2DAsync(roi, (size_t)w * 4, src + (size_t)y * sw + x, (size_t)sw * 4, (size_t)w * 4, (size_t)h, cudaMemcpyHostToDevice, st));
    return map_image(ctx, L, st, roi, w, h, Hc, d_out, dw, dh, true, 0);
}

// `homography im -h "..." out w h` (3rdparty/homography/main.cpp:65-177) from memory to memory
extern "C" int s2pb_homography(s2pb_ctx *ctx, const float *src, int sw, int sh, const double H[9], float *dst, int dw, int dh)
{
    if (!ctx || !src || !H || !dst || sw < 1 || sh < 1 || dw < 1 || dh < 1) return fail(S2PB_ERR_ARG, "bad argument");
    HostCall L(ctx, "the warp");
    float *out = L.take<float>((size_t)dw * dh * 4);
    if (int rc = L.error()) return rc;
    int rc = warp_host_to_device(ctx, L, L.st, src, sw, sh, H, out, dw, dh);
    if (rc != S2PB_OK) return rc;
    L.download(dst, out, (size_t)dw * dh * 4);
    return L.finish();
}
