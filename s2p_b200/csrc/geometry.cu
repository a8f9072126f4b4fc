// geometry.cu -- triangulation (section 8f), the tri-stereo height maps and the 3D outlier filter of triangulation.
#include "host.h"
#include "triangulation_kernels.cuh"
#include "heightmap_kernels.cuh"
#include "pointcloud_kernels.cuh"

#include <cstring>

// ------------------------------------------------------------------ triangulation (section 8f)

static_assert(sizeof(s2pb_rpc) == sizeof(RpcModel), "s2pb_rpc must have the layout of the reference's struct rpc");

// disp_to_lonlatalt (c/disp_to_h.c:70-141) on device buffers: lonlatalt nx*ny*3 doubles, err nx*ny floats
static int triangulate_enqueue(s2pb_ctx *ctx, cudaStream_t st, const float *d_dx, const float *d_dy, const float *d_m, int nx,
                               int ny, const float *d_mo, int w, int h, const double ha[9], const double hb[9],
                               const s2pb_rpc *rpca, const s2pb_rpc *rpcb, const float bbox[4], double *d_out, float *d_err)
{
    TriParams P;
    memset(&P, 0, sizeof P);
    P.dispx = d_dx; P.dispy = d_dy; P.msk = d_m; P.msk_orig = d_mo;
    P.nx = nx; P.ny = ny; P.w = w; P.h = h;
    invert_homography(ha, P.ha_inv);
    invert_homography(hb, P.hb_inv);
    memcpy(&P.rpca, rpca, sizeof(RpcModel)); memcpy(&P.rpcb, rpcb, sizeof(RpcModel));      // kernel parameters: constant bank
    P.col_min = bbox[0]; P.col_max = bbox[1]; P.row_min = bbox[2]; P.row_max = bbox[3];
    P.lonlatalt = d_out; P.err = d_err;
    dim3 b2(32, 4);
    launch(ctx, triangulate_kernel, grid2d(nx, ny, b2), b2, 0, st, P);
    CK(cudaGetLastError());
    return S2PB_OK;
}

int triangulated_cloud_device(s2pb_ctx *ctx, HostCall &L, const float *d_dx, const float *d_dy, const float *d_m, int nx, int ny,
                              const float *d_mo, int w, int h, const double ha[9], const double hb[9], const s2pb_rpc *rpca,
                              const s2pb_rpc *rpcb, const float bbox[4], int zone, int south, double **d_xyz, float **d_err)
{
    const size_t npix = (size_t)nx * ny;
    *d_xyz = L.take<double>(npix * 24);
    *d_err = L.take<float>(npix * 4);
    if (int rc = L.error()) return rc;
    int rc = triangulate_enqueue(ctx, L.st, d_dx, d_dy, d_m, nx, ny, d_mo, w, h, ha, hb, rpca, rpcb, bbox, *d_xyz, *d_err);
    if (rc == S2PB_OK) rc = launch_cloud_project(ctx, L.st, zone, south != 0, *d_xyz, *d_xyz, npix);
    return rc;
}

int triangulated_cloud_args_ok(const s2pb_ctx *ctx, int nx, int ny, int w, int h, const double ha[9], const double hb[9],
                               const s2pb_rpc *rpca, const s2pb_rpc *rpcb, const float bbox[4], int zone, int south)
{
    if (!ha || !hb || !rpca || !rpcb || !bbox || nx < 1 || ny < 1 || w < 1 || h < 1) return fail(S2PB_ERR_ARG, "bad argument");
    return cloud_crs_ok(ctx, zone, south, true);
}

int triangulated_cloud(s2pb_ctx *ctx, HostCall &L, const float *dispx, const float *dispy, const float *msk, int nx, int ny,
                       const float *msk_orig, int w, int h, const double ha[9], const double hb[9], const s2pb_rpc *rpca,
                       const s2pb_rpc *rpcb, const float bbox[4], int zone, int south, double **d_xyz, float **d_err)
{
    if (!dispx || !dispy || !msk || !msk_orig) return fail(S2PB_ERR_ARG, "bad argument");
    if (int rc = triangulated_cloud_args_ok(ctx, nx, ny, w, h, ha, hb, rpca, rpcb, bbox, zone, south)) return rc;
    const size_t npix = (size_t)nx * ny, nm = (size_t)w * h;
    float *d_dx = L.upload(dispx, npix * 4), *d_dy = L.upload(dispy, npix * 4), *d_m = L.upload(msk, npix * 4);
    float *d_mo = L.upload(msk_orig, nm * 4);
    return triangulated_cloud_device(ctx, L, d_dx, d_dy, d_m, nx, ny, d_mo, w, h, ha, hb, rpca, rpcb, bbox, zone, south, d_xyz, d_err);
}

// s2p.triangulation.disp_to_xyz (s2p/triangulation.py:85-162) with a UTM, another projected (S2PB_ZONE_PROJ) or no output
// CRS, heights optionally above EGM96: disp_to_lonlatalt, then the projection (projection.cu) in place on the device cloud;
// only the projected cloud and the error come back.
extern "C" int s2pb_disp_to_xyz(s2pb_ctx *ctx, double *xyz, float *err, const float *dispx, const float *dispy, const float *msk,
                                int nx, int ny, const float *msk_orig, int w, int h, const double ha[9], const double hb[9],
                                const s2pb_rpc *rpca, const s2pb_rpc *rpcb, const float bbox[4], int zone, int south)
{
    if (!ctx || !xyz || !err) return fail(S2PB_ERR_ARG, "bad argument");
    HostCall L(ctx, "the triangulation");
    double *d_xyz = nullptr;
    float *d_err = nullptr;
    if (int rc = triangulated_cloud(ctx, L, dispx, dispy, msk, nx, ny, msk_orig, w, h, ha, hb, rpca, rpcb, bbox, zone, south, &d_xyz,
                                    &d_err))
        return rc;
    const size_t npix = (size_t)nx * ny;
    L.download(xyz, d_xyz, npix * 24);
    L.download(err, d_err, npix * 4);
    return L.finish();
}

int localised_cloud_device(s2pb_ctx *ctx, HostCall &L, const double *d_z, int w, int h, const s2pb_rpc *rpc, double off_x,
                           double off_y, int zone, int south, double **d_xyz)
{
    const size_t npix = (size_t)w * h;
    *d_xyz = L.take<double>(npix * 24);
    int *d_capped = L.take<int>(4);
    if (int rc = L.error()) return rc;
    CK(cudaMemsetAsync(d_capped, 0, 4, L.st));
    HeightMapParams P;
    memset(&P, 0, sizeof P);
    P.heights = d_z; P.w = w; P.h = h; P.off_x = off_x; P.off_y = off_y;
    memcpy(&P.rpc, rpc, sizeof(RpcModel));
    P.xyz = *d_xyz; P.capped = d_capped;
    const dim3 b2(32, 4);
    launch(ctx, height_map_to_xyz_kernel, grid2d(w, h, b2), b2, 0, L.st, P);
    CK(cudaGetLastError());
    if (int rc = launch_cloud_project(ctx, L.st, zone, south != 0, *d_xyz, *d_xyz, npix)) return rc;
    int capped = 0;
    L.download(&capped, d_capped, 4);
    if (int rc = L.finish()) return rc;
    if (capped) return fail(S2PB_ERR_ARG, "the localisation of %d pixel(s) did not converge in 1000 steps", capped);
    return S2PB_OK;
}

int localised_cloud_args_ok(const s2pb_ctx *ctx, int w, int h, const s2pb_rpc *rpc, int zone, int south)
{
    if (!rpc || w < 1 || h < 1) return fail(S2PB_ERR_ARG, "bad argument");
    return cloud_crs_ok(ctx, zone, south, true);
}

int localised_cloud(s2pb_ctx *ctx, HostCall &L, const double *heights, int w, int h, const s2pb_rpc *rpc, double off_x,
                    double off_y, int zone, int south, double **d_xyz)
{
    if (!heights) return fail(S2PB_ERR_ARG, "bad argument");
    if (int rc = localised_cloud_args_ok(ctx, w, h, rpc, zone, south)) return rc;
    double *d_z = L.upload(heights, (size_t)w * h * 8);
    return localised_cloud_device(ctx, L, d_z, w, h, rpc, off_x, off_y, zone, south, d_xyz);
}

// s2p.triangulation.height_map_to_xyz (s2p/triangulation.py:165-217) with a UTM, another projected or no output CRS, heights optionally above
// EGM96: every pixel of the height map localised by the camera, then the projection (projection.cu) in place on the device
// cloud.
extern "C" int s2pb_height_map_to_xyz(s2pb_ctx *ctx, double *xyz, const double *heights, int w, int h, const s2pb_rpc *rpc,
                                      double off_x, double off_y, int zone, int south)
{
    if (!ctx || !xyz) return fail(S2PB_ERR_ARG, "bad argument");
    HostCall L(ctx, "the localisation");
    double *d_xyz = nullptr;
    if (int rc = localised_cloud(ctx, L, heights, w, h, rpc, off_x, off_y, zone, south, &d_xyz)) return rc;
    L.download(xyz, d_xyz, (size_t)w * h * 24);
    return L.finish();
}

// ------------------------------------------------------------------ tri-stereo height maps (section 8f)

// affine_transform(nan_to_num(z).T, H, output_shape=(w, h), order=1).T with the NaN restoration of height_map
// (heightmap_kernels.cuh), z on the device with `zstride` doubles per pixel
static int resample_heights_enqueue(s2pb_ctx *ctx, cudaStream_t st, const double *z, int zstride, int zw, int zh, const double H[9],
                                    double *out, int w, int h)
{
    ResampleParams P;
    memset(&P, 0, sizeof P);
    P.z = z; P.zstride = zstride; P.zw = zw; P.zh = zh;
    for (int k = 0; k < 6; k++) P.H[k] = H[k];
    P.w = w; P.h = h; P.out = out;
    const dim3 b2(32, 8);
    launch(ctx, heightmap_resample_kernel, grid2d(w, h, b2), b2, 0, st, P);
    CK(cudaGetLastError());
    return S2PB_OK;
}

// scipy.ndimage.affine_transform refuses a homogeneous matrix whose last row is not exactly (0, 0, 1)
static bool affine_last_row(const double H[9]) { return H[6] == 0.0 && H[7] == 0.0 && H[8] == 1.0; }

extern "C" int s2pb_resample_heights(s2pb_ctx *ctx, const double *z, int zw, int zh, const double H[9], double *out, int w, int h)
{
    if (!ctx || !z || !H || !out || zw < 1 || zh < 1 || w < 1 || h < 1) return fail(S2PB_ERR_ARG, "bad argument");
    if (!affine_last_row(H)) return fail(S2PB_ERR_ARG, "the last row of the matrix is not (0, 0, 1)");
    const size_t nz = (size_t)zw * zh, npix = (size_t)w * h;
    HostCall L(ctx, "the height resampling");
    double *d_z = L.upload(z, nz * 8), *d_out = L.take<double>(npix * 8);
    if (int rc = L.error()) return rc;
    int rc = resample_heights_enqueue(ctx, L.st, d_z, 1, zw, zh, H, d_out, w, h);
    if (rc != S2PB_OK) return rc;
    L.download(out, d_out, npix * 8);
    return L.finish();
}

// s2p.triangulation.height_map (s2p/triangulation.py:346-389) with p = 1: triangulate inside the bounding box
// float32(x-1, x+w+2, y-1, y+h+2) against mask_orig padded by one row / column of ones, keep the altitude on the device
// and resample it onto the tile grid through H1 * T(x, y).
// H1 * T(x, y): the first two columns are H1's, the third H1 (x, y, 1)^T summed left to right
static void tile_homography(const double H1[9], int x, int y, double H[9])
{
    memcpy(H, H1, 9 * sizeof(double));
    for (int r = 0; r < 3; r++) H[3 * r + 2] = H1[3 * r] * x + H1[3 * r + 1] * y + H1[3 * r + 2];
}

int height_map_args_ok(int nx, int ny, int mw, int mh, int x, int y, int w, int h, const double H1[9], const double H2[9],
                       const s2pb_rpc *rpc1, const s2pb_rpc *rpc2)
{
    if (!H1 || !H2 || !rpc1 || !rpc2 || nx < 1 || ny < 1 || mw < 1 || mh < 1 || w < 1 || h < 1)
        return fail(S2PB_ERR_ARG, "bad argument");
    if (nx < 2 || ny < 2) return fail(S2PB_ERR_UNSUPPORTED, "a %dx%d rectified map (the reference squeezes it to 1-D)", nx, ny);
    double H[9];
    tile_homography(H1, x, y, H);
    if (!affine_last_row(H)) return fail(S2PB_ERR_ARG, "the last row of H1 * T(x, y) is not (0, 0, 1)");
    return S2PB_OK;
}

int height_map_device(s2pb_ctx *ctx, HostCall &L, const float *d_dx, const float *d_m, int nx, int ny, const float *d_mo0, int mw,
                      int mh, int x, int y, int w, int h, const double H1[9], const double H2[9], const s2pb_rpc *rpc1,
                      const s2pb_rpc *rpc2, double *d_out)
{
    double H[9];
    tile_homography(H1, x, y, H);
    const float bbox[4] = {(float)(x - 1), (float)(x + w + 2), (float)(y - 1), (float)(y + h + 2)};
    const size_t npix = (size_t)nx * ny, pw = (size_t)mw + 2, ph = (size_t)mh + 2;
    float *d_dy = L.take<float>(npix * 4), *d_mo = L.take<float>(pw * ph * 4), *d_err = L.take<float>(npix * 4);
    double *d_xyz = L.take<double>(npix * 24);
    if (int rc = L.error()) return rc;
    CK(cudaMemsetAsync(d_dy, 0, npix * 4, L.st));
    const dim3 b2(32, 8);
    launch(ctx, pad_ones_kernel, grid2d((int)pw, (int)ph, b2), b2, 0, L.st, d_mo0, mw, mh, d_mo);
    int rc = triangulate_enqueue(ctx, L.st, d_dx, d_dy, d_m, nx, ny, d_mo, (int)pw, (int)ph, H1, H2, rpc1, rpc2, bbox, d_xyz, d_err);
    if (rc == S2PB_OK) rc = resample_heights_enqueue(ctx, L.st, d_xyz + 2, 3, nx, ny, H, d_out, w, h);
    return rc;
}

// s2p.triangulation.height_map (s2p/triangulation.py:346-389) with p = 1: triangulate inside the bounding box
// float32(x-1, x+w+2, y-1, y+h+2) against mask_orig padded by one row / column of ones, keep the altitude on the device
// and resample it onto the tile grid through H1 * T(x, y).
extern "C" int s2pb_height_map(s2pb_ctx *ctx, double *out, const float *disp, const float *msk, int nx, int ny,
                               const float *mask_orig, int mw, int mh, int x, int y, int w, int h, const double H1[9],
                               const double H2[9], const s2pb_rpc *rpc1, const s2pb_rpc *rpc2)
{
    if (!ctx || !out || !disp || !msk || !mask_orig) return fail(S2PB_ERR_ARG, "bad argument");
    if (int rc = height_map_args_ok(nx, ny, mw, mh, x, y, w, h, H1, H2, rpc1, rpc2)) return rc;
    const size_t npix = (size_t)nx * ny;
    HostCall L(ctx, "the height map");
    float *d_dx = L.upload(disp, npix * 4), *d_m = L.upload(msk, npix * 4);
    float *d_mo0 = L.upload(mask_orig, (size_t)mw * mh * 4);
    double *d_out = L.take<double>((size_t)w * h * 8);
    if (int rc = L.error()) return rc;
    if (int rc = height_map_device(ctx, L, d_dx, d_m, nx, ny, d_mo0, mw, mh, x, y, w, h, H1, H2, rpc1, rpc2, d_out)) return rc;
    L.download(out, d_out, (size_t)w * h * 8);
    return L.finish();
}

// s2p.common.cargarse_basura (s2p/common.py:251-262) on the float32 image its tools read: 5x5 min / max and plambda in one
// kernel, then remove_small_cc(200, 5)
int basura_args_ok(int w, int h)
{
    if (w < 2 || h < 2) return fail(S2PB_ERR_UNSUPPORTED, "a %dx%d image: the reference's morphoop reads outside it", w, h);
    if ((size_t)w * h > INT32_MAX) return fail(S2PB_ERR_UNSUPPORTED, "at most 2^31 - 1 pixels");
    return S2PB_OK;
}

int basura_enqueue(s2pb_ctx *ctx, cudaStream_t st, const float *d_in, float *d_out, int w, int h, float *d_m, int *lab, int *area)
{
    const dim3 bb(kBasuraTx, kBasuraTy);
    launch(ctx, basura_minmax_kernel, grid2d(w, h, bb), bb, 0, st, d_in, w, h, d_m);
    CK(cudaGetLastError());
    return launch_remove_small_cc(ctx, d_m, d_out, w, h, 200, 5.f, lab, area, st);
}

extern "C" int s2pb_cargarse_basura(s2pb_ctx *ctx, const float *in, float *out, int w, int h)
{
    if (!ctx || !in || !out || w < 1 || h < 1) return fail(S2PB_ERR_ARG, "bad argument");
    if (int rc = basura_args_ok(w, h)) return rc;
    const size_t npix = (size_t)w * h;
    HostCall L(ctx, "cargarse_basura");
    float *a = L.upload(in, npix * 4), *m = L.take<float>(npix * 4), *b = L.take<float>(npix * 4);
    int *lab = L.take<int>(npix * 4), *area = L.take<int>(npix * 4);
    if (int rc = L.error()) return rc;
    if (int rc = basura_enqueue(ctx, L.st, a, b, w, h, m, lab, area)) return rc;
    L.download(out, b, npix * 4);
    return L.finish();
}

// ------------------------------------------------------------------ 3D outlier filter of triangulation (section 8f)

// count_3d_neighbors (c/disp_to_h.c:152-174) of a device cloud into a device count image
static int pc_count_enqueue(s2pb_ctx *ctx, cudaStream_t st, const double *xyz, int nx, int ny, float r, int p, int *count)
{
    if (p < 0) { CK(cudaMemsetAsync(count, 0, (size_t)nx * ny * 4, st)); return S2PB_OK; }     // empty windows
    p = std::min(p, std::max(nx, ny));                                  // a wider window is the whole image
    const long long side = kPcTile + 2LL * p;
    const size_t smem = (size_t)std::min<long long>(side, nx) * std::min<long long>(side, ny) * 24;    // one CTA's clipped footprint
    int optin = 0;
    CK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, ctx->device));
    const dim3 b(kPcTile, kPcTile), g = grid2d(nx, ny, b);
    if (smem <= (size_t)optin) {
        CK(cudaFuncSetAttribute(pc_count_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        launch(ctx, pc_count_kernel<true>, g, b, smem, st, xyz, nx, ny, r, p, count);
    } else {
        launch(ctx, pc_count_kernel<false>, g, b, 0, st, xyz, nx, ny, r, p, count);
    }
    CK(cudaGetLastError());
    return S2PB_OK;
}

// Same argument list as the reference's count_3d_neighbors (c/disp_to_h.c:152), plus the context.
extern "C" int s2pb_count_3d_neighbors(s2pb_ctx *ctx, int32_t *count, const double *xyz, int nx, int ny, float r, int p)
{
    if (!ctx || !count || !xyz || nx < 1 || ny < 1) return fail(S2PB_ERR_ARG, "bad argument");
    const size_t npix = (size_t)nx * ny;
    if (npix > INT32_MAX) return fail(S2PB_ERR_UNSUPPORTED, "at most 2^31 - 1 points");
    HostCall L(ctx, "the point cloud");
    double *d_xyz = L.upload(xyz, npix * 24);
    int *d_count = L.take<int>(npix * 4);
    if (int rc = L.error()) return rc;
    int rc = pc_count_enqueue(ctx, L.st, d_xyz, nx, ny, r, p, d_count);
    if (rc != S2PB_OK) return rc;
    L.download(count, d_count, npix * 4);
    return L.finish();
}

// remove_isolated_3d_points on a device cloud of nx * ny < 2^31 points with n > 0; d_work: 3 * nx * ny ints of scratch
int remove_isolated_enqueue(s2pb_ctx *ctx, cudaStream_t st, double *d_xyz, int nx, int ny, float r, int p, int n, int q, int *d_work)
{
    const size_t npix = (size_t)nx * ny;
    int *d_count = d_work, *d_lab = d_work + npix, *d_saved = d_work + 2 * npix;
    int rc = pc_count_enqueue(ctx, st, d_xyz, nx, ny, r, p, d_count);
    if (rc != S2PB_OK) return rc;
    const unsigned g1 = (unsigned)((npix + 255) / 256);
    const dim3 b2(32, 8), g2 = grid2d(nx, ny, b2);
    launch(ctx, pc_label_kernel, g1, 256, 0, st, d_count, (int)npix, n, d_lab, d_saved);
    if (q >= 0) {                                                       // q < 0: empty windows, nothing is saved
        q = std::min(q, std::max(nx, ny));
        launch(ctx, pc_link_kernel, g2, b2, 0, st, d_xyz, nx, ny, r, q, d_lab);
        cc_flatten(ctx, (int)npix, d_lab, st);
        launch(ctx, pc_mark_kernel, g2, b2, 0, st, d_xyz, nx, ny, r, q, d_lab, d_saved);
    }
    launch(ctx, pc_reject_kernel, g1, 256, 0, st, (int)npix, d_lab, d_saved, d_xyz);
    CK(cudaGetLastError());
    return S2PB_OK;
}

// Same argument list as the reference's remove_isolated_3d_points (c/disp_to_h.c:177-184), plus the context; in place on
// the host cloud.  Rejection by count, then the closure of the reference's "mercy" sweeps as connected components
// (pointcloud_kernels.cuh): label, link, flatten, mark the saved components, NaN the rest.
extern "C" int s2pb_remove_isolated_3d_points(s2pb_ctx *ctx, double *xyz, int nx, int ny, float r, int p, int n, int q)
{
    if (!ctx || !xyz || nx < 1 || ny < 1) return fail(S2PB_ERR_ARG, "bad argument");
    const size_t npix = (size_t)nx * ny;
    if (npix > INT32_MAX) return fail(S2PB_ERR_UNSUPPORTED, "at most 2^31 - 1 points");
    if (n <= 0) return S2PB_OK;                                         // a count is never negative: nothing is rejected
    HostCall L(ctx, "the point cloud");
    double *d_xyz = L.upload(xyz, npix * 24);
    int *d_work = L.take<int>(npix * 12);
    if (int rc = L.error()) return rc;
    if (int rc = remove_isolated_enqueue(ctx, L.st, d_xyz, nx, ny, r, p, n, q, d_work)) return rc;
    L.download(xyz, d_xyz, npix * 24);
    return L.finish();
}
