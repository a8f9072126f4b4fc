// pair_tile.cu -- one pair of a tile from its source crops on, in one call: rectify_pair's two warps and the matcher with its
// rejection mask chained on one stream (rectify_and_match, all of s2pb_rectify_match), then masking.erosion (pair_match) and,
// for a two-view tile, disparity_to_ply down to the records of cloud.ply, or, for a pair of a tri-stereo tile,
// disparity_to_height down to the pair's height map; the intermediates stay on the device (s2p/__init__.py:102-318).
#include "host.h"

// the eroded 0/1 mask as the float32 image disparity_to_ply hands to the triangulation (a PNG read back as uint8, then float32)
__global__ void mask_to_float_kernel(const uint8_t *__restrict__ in, float *__restrict__ out, size_t n)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (float)in[i];
}

// what the warps, the matcher and the erosion would refuse that can be seen before the first launch
// (with_conf: the confidence column is asked for)
static int pair_match_args_ok(const s2pb_pair_tile *t, const float *conf, const float *disp_right, bool with_conf)
{
    if (!t->src1 || !t->src2 || !t->msk_orig || t->sw1 < 1 || t->sh1 < 1 || t->sw2 < 1 || t->sh2 < 1 || t->w < 1 || t->h < 1 ||
        t->mw < 1 || t->mh < 1)
        return fail(S2PB_ERR_ARG, "bad argument");
    if (t->matcher != S2PB_MATCHER_MGM && t->matcher != S2PB_MATCHER_SGBM) return fail(S2PB_ERR_ARG, "unknown matcher %d", t->matcher);
    if (t->matcher == S2PB_MATCHER_SGBM && (conf || disp_right || with_conf || t->wl || t->wr))
        return fail(S2PB_ERR_ARG, "sgbm has no confidence, right disparity or weight images");
    if ((t->wl == nullptr) != (t->wr == nullptr)) return fail(S2PB_ERR_ARG, "the weight images come in pairs (-wl and -wr)");
    if (t->erode_radius != 0.f) {
        if (int rc = erode_radius_ok(t->erode_radius)) return rc;
    }
    return S2PB_OK;
}

// The device results of a pair's front half (w*h each, scratch of the call)
struct PairMatch {
    const float *rect1;       // the rectified reference
    const float *disp, *conf; // the disparity and, with MGM, its confidence
    uint8_t *mask;            // the rejection mask
    const float *dispR;       // MGM's right disparity, when asked for
    const float *msk;         // pair_match: the eroded 0/1 mask as float32
};

// rectify_pair's two warps and the matcher (t->matcher) with its rejection mask, on L's stream: the buffers come from L, the
// rectified pair is copied back when rect1 / rect2 are not null (in flight on L.st), and MGM waits for its stream through its
// timeout.  want_right: MGM's right disparity.
static int rectify_and_match(s2pb_ctx *ctx, HostCall &L, const s2pb_pair_tile *t, float *rect1, float *rect2, bool want_right,
                             PairMatch *m)
{
    const int w = t->w, h = t->h;
    const size_t npix = (size_t)w * h;
    const bool mgm = t->matcher == S2PB_MATCHER_MGM;
    float *d_r1 = L.take<float>(npix * 4), *d_r2 = L.take<float>(npix * 4), *d_disp = L.take<float>(npix * 4);
    float *d_conf = mgm ? L.take<float>(npix * 4) : nullptr, *d_dispR = want_right ? L.take<float>(npix * 4) : nullptr;
    uint8_t *d_mask = L.take<uint8_t>(npix);
    const float *d_wl = t->wl ? L.upload(t->wl, npix * 4) : nullptr, *d_wr = t->wr ? L.upload(t->wr, npix * 4) : nullptr;
    if (int rc = L.error()) return rc;

    // rectification_pair: both warps straight into the matcher's inputs
    if (int rc = warp_host_to_device(ctx, L, L.st, t->src1, t->sw1, t->sh1, t->H1, d_r1, w, h)) return rc;
    if (int rc = warp_host_to_device(ctx, L, L.st, t->src2, t->sw2, t->sh2, t->H2, d_r2, w, h)) return rc;
    if (rect1) L.download(rect1, d_r1, npix * 4);
    if (rect2) L.download(rect2, d_r2, npix * 4);

    // stereo_matching: the matcher and its rejection mask
    if (mgm) {
        if (int rc = mgm_match_device(ctx, L.st, d_r1, d_r2, w, h, t->dmin, t->dmax, &t->mgm, d_wl, d_wr, d_disp, d_conf, d_mask,
                                      d_dispR))
            return rc;
    } else if (int rc = sgbm_enqueue(ctx, L, d_r1, d_r2, w, h, t->dmin, t->dmax, &t->sgbm, d_disp, d_mask)) {
        return rc;
    }
    m->rect1 = d_r1; m->disp = d_disp; m->conf = d_conf; m->mask = d_mask; m->dispR = d_dispR; m->msk = nullptr;
    return S2PB_OK;
}

// Steps 3 and 4 of a tile in one call (s2p/__init__.py:147-155 rectify_pair's two warps, :184-190 compute_disparity_map): both
// images are warped straight into the matcher's device inputs and matched there; the rectified pair never travels through
// files or host memory unless the caller asks for a copy (rect1 / rect2).
extern "C" int s2pb_rectify_match(s2pb_ctx *ctx, const float *src1, int sw1, int sh1, const double H1[9],
                                  const float *src2, int sw2, int sh2, const double H2[9], int w, int h, int dmin, int dmax,
                                  const s2pb_mgm_params *p, float *rect1, float *rect2, float *disp, float *conf, uint8_t *mask,
                                  float *disp_right)
{
    if (!ctx || !src1 || !src2 || !H1 || !H2 || !p || !disp || !conf || sw1 < 1 || sh1 < 1 || sw2 < 1 || sh2 < 1 ||
        w < 1 || h < 1)
        return fail(S2PB_ERR_ARG, "bad argument");
    s2pb_pair_tile t = {};
    t.src1 = src1; t.sw1 = sw1; t.sh1 = sh1; std::copy(H1, H1 + 9, t.H1);
    t.src2 = src2; t.sw2 = sw2; t.sh2 = sh2; std::copy(H2, H2 + 9, t.H2);
    t.w = w; t.h = h; t.dmin = dmin; t.dmax = dmax;
    t.matcher = S2PB_MATCHER_MGM; t.mgm = *p;
    const size_t npix = (size_t)w * h;
    HostCall L(ctx, "the rectified pair");
    PairMatch m;
    if (int rc = rectify_and_match(ctx, L, &t, rect1, rect2, disp_right != nullptr, &m)) return rc;
    L.download(disp, m.disp, npix * 4);
    L.download(conf, m.conf, npix * 4);
    if (mask) L.download(mask, m.mask, npix);
    if (disp_right) L.download(disp_right, m.dispR, npix * 4);
    return L.finish();
}

// rectify_and_match, then masking.erosion of the mask and its float32 copy (m->msk): the intermediates named by non-null host
// pointers are copied back (in flight on L.st)
static int pair_match(s2pb_ctx *ctx, HostCall &L, const s2pb_pair_tile *t, float *rect1, float *rect2, float *disp, float *conf,
                      uint8_t *mask, float *disp_right, PairMatch *m)
{
    const int w = t->w, h = t->h;
    const size_t npix = (size_t)w * h;
    const bool erode = t->erode_radius != 0.f;
    if (int rc = rectify_and_match(ctx, L, t, rect1, rect2, disp_right != nullptr, m)) return rc;
    uint8_t *d_eroded = erode ? L.take<uint8_t>(npix) : m->mask;
    float *d_msk = L.take<float>(npix * 4);
    if (int rc = L.error()) return rc;
    if (erode) launch_erode_mask(ctx, m->mask, d_eroded, w, h, t->erode_radius, L.st);
    launch(ctx, mask_to_float_kernel, (unsigned)((npix + 255) / 256), 256, 0, L.st, d_eroded, d_msk, npix);
    CK(cudaGetLastError());
    if (disp) L.download(disp, m->disp, npix * 4);
    if (conf) L.download(conf, m->conf, npix * 4);
    if (mask) L.download(mask, d_eroded, npix);
    if (disp_right) L.download(disp_right, m->dispR, npix * 4);
    m->msk = d_msk;
    return S2PB_OK;
}

// what the stages of s2pb_pair_tile_to_ply would refuse that can be seen before the first launch
static int pair_tile_args_ok(s2pb_ctx *ctx, const s2pb_pair_tile *t, uint8_t *records, int64_t *npoints, const float *conf,
                             const float *disp_right)
{
    if (!ctx || !t) return fail(S2PB_ERR_ARG, "bad argument");
    if (int rc = pair_match_args_ok(t, conf, disp_right, t->with_conf != 0)) return rc;
    if (int rc = triangulated_cloud_args_ok(ctx, t->w, t->h, t->mw, t->mh, t->ha, t->hb, t->rpc1, t->rpc2, t->bbox, t->zone, t->south))
        return rc;
    if (t->clr) {
        if (int rc = tail_args_ok(ctx, t->w, t->h, t->clr, t->clr_bands, 0.0, records, npoints)) return rc;
        if (int rc = typed_colours_ok(t->clr_bands, S2PB_PLY_F32)) return rc;
        if (t->cw < 1 || t->ch < 1) return fail(S2PB_ERR_ARG, "bad argument");
        return S2PB_OK;
    }
    return tail_args_ok(ctx, t->w, t->h, nullptr, 0, t->pct, records, npoints);      // colours: the call's own rectified reference
}

extern "C" int s2pb_pair_tile_to_ply(s2pb_ctx *ctx, const s2pb_pair_tile *t, uint8_t *records, int64_t *npoints, float *rect1,
                                     float *rect2, float *disp, float *conf, uint8_t *mask, float *disp_right)
{
    if (int rc = pair_tile_args_ok(ctx, t, records, npoints, conf, disp_right)) return rc;
    *npoints = 0;
    const int w = t->w, h = t->h;
    const size_t npix = (size_t)w * h;
    HostCall L(ctx, "the pair tile");
    PairMatch m;
    if (int rc = pair_match(ctx, L, t, rect1, rect2, disp, conf, mask, disp_right, &m)) return rc;

    // disparity_to_ply: the cloud, its colours and its records
    float *d_dy = L.take<float>(npix * 4);
    const float *d_mo = L.upload(t->msk_orig, (size_t)t->mw * t->mh * 4);
    if (int rc = L.error()) return rc;
    CK(cudaMemsetAsync(d_dy, 0, npix * 4, L.st));
    double *d_xyz = nullptr;
    float *d_err = nullptr;
    if (int rc = triangulated_cloud_device(ctx, L, m.disp, d_dy, m.msk, w, h, d_mo, t->mw, t->mh, t->ha, t->hb, t->rpc1, t->rpc2,
                                           t->bbox, t->zone, t->south, &d_xyz, &d_err))
        return rc;
    const float *d_cc = t->with_conf ? m.conf : nullptr;
    if (!t->clr) return cloud_tail_device(ctx, L, d_xyz, w, h, t->r, t->p, t->n, m.rect1, 1, t->pct, nullptr, 1, d_cc, records, npoints);
    float *d_col = L.take<float>(npix * t->clr_bands * 4);
    if (int rc = L.error()) return rc;
    for (int b = 0; b < t->clr_bands; b++)
        if (int rc = warp_host_to_device(ctx, L, L.st, t->clr + (size_t)b * t->cw * t->ch, t->cw, t->ch, t->hc, d_col + (size_t)b * npix,
                                         w, h))
            return rc;
    return cloud_tail_device(ctx, L, d_xyz, w, h, t->r, t->p, t->n, nullptr, t->clr_bands, 0.0, (const uint8_t *)d_col, 4, d_cc,
                             records, npoints);
}

extern "C" int s2pb_pair_tile_to_height_map(s2pb_ctx *ctx, const s2pb_pair_tile *t, int x, int y, int tw, int th, double *heights,
                                            float *rect1, float *rect2, float *disp, float *conf, uint8_t *mask, float *disp_right)
{
    if (!ctx || !t || !heights) return fail(S2PB_ERR_ARG, "bad argument");
    if (int rc = pair_match_args_ok(t, conf, disp_right, false)) return rc;
    if (int rc = height_map_args_ok(t->w, t->h, t->mw, t->mh, x, y, tw, th, t->ha, t->hb, t->rpc1, t->rpc2)) return rc;
    HostCall L(ctx, "the pair's height map");
    PairMatch m;
    if (int rc = pair_match(ctx, L, t, rect1, rect2, disp, conf, mask, disp_right, &m)) return rc;

    // disparity_to_height: triangulation.height_map on the device disparity and eroded mask
    const float *d_mo = L.upload(t->msk_orig, (size_t)t->mw * t->mh * 4);
    double *d_out = L.take<double>((size_t)tw * th * 8);
    if (int rc = L.error()) return rc;
    if (int rc = height_map_device(ctx, L, m.disp, m.msk, t->w, t->h, d_mo, t->mw, t->mh, x, y, tw, th, t->ha, t->hb, t->rpc1,
                                   t->rpc2, d_out))
        return rc;
    L.download(heights, d_out, (size_t)tw * th * 8);
    return L.finish();
}
