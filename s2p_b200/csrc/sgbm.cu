// sgbm.cu -- s2p's `sgbm` matcher (3rdparty/sgbm, sgbm_kernels.cuh).
#include "host.h"
#include "sgbm_kernels.cuh"

extern "C" int s2pb_sgbm_default_params(s2pb_sgbm_params *p)
{
    if (!p) return fail(S2PB_ERR_ARG, "null params");
    p->win = 3; p->P1 = 8; p->P2 = 32; p->lr_diff = 1;       // what s2p passes: s2p/block_matching.py:116-134
    return S2PB_OK;
}

size_t order_stats_bytes() { return sizeof(OrderStats) + kOrdMaxRanks * 256 * sizeof(unsigned); }

// The radix select of sgbm_kernels.cuh: four passes of one 8-bit digit over the n values of d_x, every rank at once.
int launch_order_stats(s2pb_ctx *ctx, cudaStream_t st, const float *d_x, int n, int rule, double q0, double q1, OrderStats *d_os)
{
    unsigned *d_hist = (unsigned *)(d_os + 1);
    CK(cudaMemsetAsync(d_os, 0, order_stats_bytes(), st));
    const int hblocks = (int)std::max<size_t>(1, std::min<size_t>(((size_t)n + 255) / 256, (size_t)ctx->sm_count * 4));
    for (int digit = 3; digit >= 0; digit--) {
        launch(ctx, sgbm_hist_kernel, hblocks, 256, 0, st, d_x, n, digit, d_os, d_hist);
        launch(ctx, sgbm_select_kernel, 1, 32, 0, st, digit, rule, q0, q1, d_os, d_hist);
    }
    CK(cudaGetLastError());
    return S2PB_OK;
}

// The whole `sgbm im1 im2 disp cost dmin dmax win P1 P2 lr` run followed by create_rejection_mask, enqueued on the call's
// stream.  d_im1 / d_im2 / d_disp: w*h float32, d_mask: w*h uint8 or null, all from L, which is checked before the first launch.
// S2PB_ERR_ARG / S2PB_ERR_UNSUPPORTED for what s2pb_sgbm refuses, before anything is enqueued.
int sgbm_enqueue(s2pb_ctx *ctx, HostCall &L, const float *d_im1, const float *d_im2, int w, int h, int dmin, int dmax,
                 const s2pb_sgbm_params *p, float *d_disp, uint8_t *d_mask)
{
    if (dmin >= dmax) return fail(S2PB_ERR_ARG, "mindisp(%d) > maxdisp(%d)", -dmax, -dmin);     // sgbm.cpp:174-177
    if (p->win < 1 || p->win % 2 == 0) return fail(S2PB_ERR_ARG, "SADWindowSize must be odd and positive (got %d)", p->win);
    const cudaStream_t st = L.st;
    // sgbm.cpp:166-192: OpenCV's convention is the opposite of s2p's; the label count is rounded up to a multiple of 16
    const int mindisp = -dmax, maxdisp = -dmin;
    const int ND = (maxdisp - mindisp + 15) / 16 * 16;
    SgbmGeom g;
    g.minD = mindisp; g.D = ND;
    const int maxD = g.minD + ND;
    g.wp = w + std::max(-mindisp, 0) + std::max(maxdisp, 0);         // the crop trick, sgbm.cpp:204-207
    g.h = h;
    const int off = std::max(maxdisp, 0);
    g.minX1 = std::max(-maxD, 0);
    const int maxX1 = g.wp + std::min(g.minD, 0);
    g.w1 = maxX1 - g.minX1;
    g.minX2 = std::max(g.minX1 - maxD, 0);
    g.w2 = std::min(maxX1 - g.minD, g.wp) - g.minX2;
    g.SW2 = g.SH2 = p->win / 2;
    g.P1 = p->P1 > 0 ? p->P1 : 2;                                      // stereosgbm.cpp:333-334
    g.P2 = std::max(p->P2 > 0 ? p->P2 : 5, g.P1 + 1);
    const int lr = p->lr_diff > 0 ? p->lr_diff : 1;
    const int invalid = (g.minD - 1) * 16;

    if ((long long)invalid < -32768 || (long long)maxD * 16 > 32767)
        return fail(S2PB_ERR_UNSUPPORTED, "disparity range [%d,%d] does not fit the reference's int16 disparities (x16)", dmin, dmax);
    // every L is in [C - P2, C]: min L + P2 must stay an int16, and 8 L of a zero-cost pixel must not reach -32768
    // (DESIGN.md section 3.5)
    if ((long long)p->win * p->win * kSgbmPixMax + 2LL * g.P2 > kSgbmMaxCost || g.P2 > 4096)
        return fail(S2PB_ERR_UNSUPPORTED, "win %d with P2 %d can overflow the reference's int16 path costs "
                    "(needs win^2 * %d + 2 * P2 <= 32767 and P2 <= 4096)", p->win, g.P2, kSgbmPixMax);
    const bool any = g.w1 > 0;                                         // else every pixel is invalid (stereosgbm.cpp:347-351)
    size_t pix_smem = 4 * (size_t)g.wp + 4 * (size_t)std::max(g.w2, 0);
    const size_t path_smem = 4 * 2 * ((size_t)ND + 2) * sizeof(int);
    if (any) {
        if (g.w1 <= g.SW2) return fail(S2PB_ERR_UNSUPPORTED, "a %d px wide cost volume is narrower than the half window %d", g.w1, g.SW2);
        // bytes calcPixelCostBT reads around its row buffer: at most 4 * width before it (disp2ptr, disp2cost, zero while
        // the costs are computed) and below 16 * width after it (its own never-written tail)
        const long long jmin = (long long)g.wp - maxX1 + g.minD, jmax = (long long)g.wp - 1 - g.minX1 + maxD - 1;
        if (jmin - g.minX2 < -4LL * g.wp || 2LL * g.w2 + 3LL * g.wp + jmax >= 16LL * g.wp)
            return fail(S2PB_ERR_UNSUPPORTED, "disparity range [%d,%d] reads outside the reference's row buffers", dmin, dmax);
        if (pix_smem > 227 * 1024 || path_smem > 227 * 1024)
            return fail(S2PB_ERR_UNSUPPORTED, "a %d px wide, %d label tile needs more shared memory than an SM has", g.wp, ND);
    }
    const size_t npix = (size_t)w * h, ppix = (size_t)g.wp * h;
    if (ppix > INT32_MAX) return fail(S2PB_ERR_UNSUPPORTED, "at most 2^31 - 1 padded pixels");
    const size_t vol = any ? (size_t)h * g.w1 * ND : 0;

    SgbmState *d_st = L.take<SgbmState>(order_stats_bytes());
    uint8_t *q1 = L.take<uint8_t>(ppix), *q2 = L.take<uint8_t>(ppix);
    short *pix = any ? L.take<short>(vol * 2) : nullptr, *C = any ? L.take<short>(vol * 2) : nullptr;
    short *disp1 = L.take<short>(ppix * 2), *dmed = L.take<short>(ppix * 2);
    unsigned long long *d2key = L.take<unsigned long long>(ppix * 8);
    int *lab = L.take<int>(ppix * 4), *area = L.take<int>(ppix * 4);
    if (int rc = L.error()) return rc;

    // qauto thresholds: the two order statistics of get_rminmax
    if (int rc = launch_order_stats(ctx, st, d_im1, (int)npix, kOrdQauto, 0.0, 0.0, d_st)) return rc;
    launch(ctx, sgbm_quantize_kernel, dim3((g.wp + 255) / 256, h), 256, 0, st, d_im1, d_im2, w, h, off, g.wp, d_st, q1, q2);
    launch(ctx, sgbm_fill_kernel, std::max(1, (int)std::min<size_t>((ppix + 255) / 256, 4096)), 256, 0, st, disp1, ppix, (short)invalid);
    if (any) {
        CK(cudaFuncSetAttribute(sgbm_pixcost_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pix_smem));
        CK(cudaFuncSetAttribute(sgbm_path_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)path_smem));
        launch(ctx, sgbm_pixcost_kernel, h, 256, pix_smem, st, q1, q2, g, pix);
        const size_t rowel = (size_t)g.w1 * ND;
        launch(ctx, sgbm_window_kernel, dim3((unsigned)std::min<size_t>((rowel + 255) / 256, 1024), h), 256, 0, st, pix, g, C);
        short *S = pix;                                                  // the pixel costs are dead once C is formed
        CK(cudaMemsetAsync(S, 0, vol * 2, st));
        // pass 1 (top-down: predecessors left, up-left, up, up-right) and pass 2 (bottom-up, the mirrored four)
        static const int steps[8][2] = {{1, 0}, {1, 1}, {0, 1}, {-1, 1}, {-1, 0}, {1, -1}, {0, -1}, {-1, -1}};
        for (auto &s : steps) {
            const int nlines = s[1] == 0 ? h : s[0] == 0 ? g.w1 : g.w1 + h - 1;
            launch(ctx, sgbm_path_kernel, (nlines + 3) / 4, 128, path_smem, st, C, g, s[0], s[1], S);
        }
        CK(cudaMemsetAsync(d2key, 0xff, ppix * 8, st));
        const size_t nw = (size_t)g.w1 * h;
        launch(ctx, sgbm_wta_kernel, (unsigned)((nw + 7) / 8), 256, 0, st, S, g, disp1, d2key);
        launch(ctx, sgbm_lr_kernel, dim3((g.w1 + 255) / 256, h), 256, 0, st, disp1, d2key, g, lr);
    }
    const dim3 b2(32, 8);
    const unsigned g1 = (unsigned)((ppix + 255) / 256);
    launch(ctx, sgbm_median_kernel, grid2d(g.wp, h, b2), b2, 0, st, disp1, g.wp, h, dmed);
    launch(ctx, sgbm_speckle_init_kernel, g1, 256, 0, st, dmed, (int)ppix, invalid, lab, area);
    launch(ctx, sgbm_speckle_link_kernel, grid2d(g.wp, h, b2), b2, 0, st, dmed, g.wp, h, invalid, lab);
    cc_flatten(ctx, (int)ppix, lab, st);
    cc_area(ctx, (int)ppix, lab, area, st);
    launch(ctx, sgbm_output_kernel, grid2d(w, h, b2), b2, 0, st, dmed, lab, area, g.wp, off, w, h, invalid, d_st, d_disp);
    if (d_mask) launch_rejection_mask(ctx, d_disp, d_im1, d_im2, w, h, d_mask, st);
    CK(cudaGetLastError());
    return S2PB_OK;
}

// `sgbm im1 im2 disp cost dmin dmax win P1 P2 lr` + create_rejection_mask from host buffers (pageable or page-locked)
extern "C" int s2pb_sgbm(s2pb_ctx *ctx, const float *im1, const float *im2, int w, int h, int dmin, int dmax,
                         const s2pb_sgbm_params *p, float *disp, uint8_t *mask)
{
    if (!ctx || !im1 || !im2 || !p || !disp || w < 1 || h < 1) return fail(S2PB_ERR_ARG, "bad argument");
    const size_t npix = (size_t)w * h;
    HostCall L(ctx, "sgbm");
    float *d_im1 = L.upload(im1, npix * 4), *d_im2 = L.upload(im2, npix * 4), *d_disp = L.take<float>(npix * 4);
    uint8_t *d_mask = mask ? L.take<uint8_t>(npix) : nullptr;
    int rc = sgbm_enqueue(ctx, L, d_im1, d_im2, w, h, dmin, dmax, p, d_disp, d_mask);
    if (rc != S2PB_OK) return rc;
    L.download(disp, d_disp, npix * 4);
    if (mask) L.download(mask, d_mask, npix);
    return L.finish();
}
