// s2pb200.cu -- context, workspace, the matcher and its stage entry points of the C ABI declared in include/s2pb200.h.
//
// Host-side orchestration of the kernels in mgm_kernels.cuh.  The sequence of stages mirrors
// what one `mgm` process does for one tile (main_mgm.cc:167-262 -> mgm_call,
// mgm_multiscale.cc:161-335 in the reference) followed by create_rejection_mask
// (s2p/block_matching.py:18-32).  There is no CPU fallback in this file.  The other entry points are in warp.cu,
// geometry.cu, sgbm.cu and raster.cu; host.h holds what they share with this file.
#include "host.h"
#include "mgm_kernels.cuh"
#include "multiscale_kernels.cuh"
#include "dct_kernels.cuh"
#include "agg_dispatch.h"
#include "agg_chunked.cuh"

#include <chrono>
#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <optional>
#include <thread>
#include <type_traits>

// ------------------------------------------------------------------ errors

thread_local std::string g_err;
int fail(int code, const char *fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}

// ------------------------------------------------------------------ context

// stride of the per-pass progress counters: bands hold kNW scanlines in the register-resident kernel, but as few as 2 in the
// chunk-skipping kernel on float-cost slabs wider than 1024 slots (agg_chunked.cuh, ck_warps)
static int max_bands(int w, int h) { return ((w > h ? w : h) + 1) / 2; }

// Scanlines of the boundary buffer of the folded layout: one per band of the pass, for the larger of the two scan geometries
// (rows: h scanlines of w pixels; columns: w of h).  A band holds kNW scanlines in the register-resident kernel and ck_warps in
// the chunk-skipping one, which serves the slabs wider than 512 slots (wide_slab).
static size_t boundary_pixels(int w, int h, int DP, bool gen)
{
    const int nw = DP > 512 ? ck_warps(DP, gen) : kNW;
    const size_t rows = (size_t)((h + nw - 1) / nw) * w, cols = (size_t)((w + nw - 1) / nw) * h;
    return rows > cols ? rows : cols;
}

// The workspace of one slot, in the resident layout (eight pass volumes per view) or the folded one (the running sum S, the
// boundary buffer and one arg-minimum plane per pass, DESIGN.md section 3.6).  Carves one allocation; called with
// allocate=false to size it (s.bytes).
static int slot_layout(Slot &s, int w, int h, int DP, int ndir, int cbytes, bool folded, bool allocate)
{
    size_t npix = (size_t)w * h, off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
    char *b = (char *)s.base;
    int mb = max_bands(w, h);
    for (int vi = 0; vi < 2; vi++) {
        ViewWS &v = s.v[vi];
        size_t o;
        o = take(npix * 4); if (allocate) v.img = (float *)(b + o);
        o = take(npix * 2); if (allocate) v.lo = (short *)(b + o);
        o = take(npix * 2); if (allocate) v.hi = (short *)(b + o);
        o = take(npix * 8); if (allocate) v.census = (uint64_t *)(b + o);
        o = take(npix * 4); if (allocate) v.rt = (float *)(b + o);
        o = take(npix * 8); if (allocate) v.census_rt = (uint64_t *)(b + o);
        o = take(((size_t)h + w) * 4 + w + 16); if (allocate) v.rowlist = (int *)(b + o);      // rows, then columns, then column flags
        o = take((size_t)h * 4); if (allocate) v.rowthr = (float *)(b + o);
        o = take(256); if (allocate) v.rtstate = (RtState *)(b + o);
        o = take(npix * DP * cbytes); if (allocate) v.C = (void *)(b + o);
        for (int p = 0; p < kMaxPasses; p++) { v.L[p] = nullptr; v.am[p] = nullptr; }
        v.S = v.Lb = nullptr;
        if (folded) {
            o = take(npix * DP * 4); if (allocate) v.S = (float *)(b + o);
            o = take(boundary_pixels(w, h, DP, cbytes == 4) * DP * 4); if (allocate) v.Lb = (float *)(b + o);
            for (int p = 0; p < ndir; p++) { o = take(npix * 2); if (allocate) v.am[p] = (short *)(b + o); }
        }
        for (int p = 0; p < ndir; p++) {
            if (!folded) { o = take(npix * DP * 4); if (allocate) v.L[p] = (float *)(b + o); }
            o = take(npix * 4); if (allocate) v.Lmin[p] = (float *)(b + o);
        }
        o = take((size_t)kMaxPasses * mb * 4); if (allocate) v.progress = (int *)(b + o);
        o = take(npix * 4); if (allocate) v.disp = (float *)(b + o);
        o = take(npix * 4); if (allocate) v.cost = (float *)(b + o);
        o = take(npix * 4); if (allocate) v.conf = (float *)(b + o);
        o = take(npix * 4); if (allocate) v.tmp = (float *)(b + o);
    }
    size_t o;
    o = take(256); if (allocate) s.next_item = (int *)(b + o);
    // the popcount -> cost table (kCostLut floats) runs on into the head of Ydct (256 bytes or more), which only the round trips
    // at the start of mgm_call use: mgm_call uploads the table after them
    static_assert(kCostLut * sizeof(float) <= 512, "the cost table overflows lut + the head of Ydct");
    o = take(256); if (allocate) s.lut = (float *)(b + o);
    o = take(npix * 8); if (allocate) s.Ydct = (double *)(b + o);
    if (!allocate) s.bytes = off;
    return 0;
}

// device-side staging of the host-buffer API (inputs, outputs); separate from the workspace because
// mgm_multi re-carves the workspace at every pyramid level
static int slot_io_ensure(Slot &s, size_t npix)
{
    if (s.io_pix >= npix) return S2PB_OK;
    if (s.io_base) { CK(cudaStreamSynchronize(s.stream)); CK(cudaFree(s.io_base)); s.io_base = nullptr; s.io_pix = 0; }
    size_t stride = align_up(npix * 4, 256);
    cudaError_t e = cudaMalloc((void **)&s.io_base, stride * 8);
    if (e != cudaSuccess) { cudaGetLastError(); return fail(S2PB_ERR_NOMEM, "I/O staging of %zu bytes: %s", stride * 8, cudaGetErrorString(e)); }
    s.d_in[0] = (float *)s.io_base; s.d_in[1] = (float *)(s.io_base + stride);
    s.d_disp = (float *)(s.io_base + 2 * stride); s.d_conf = (float *)(s.io_base + 3 * stride);
    s.d_dispR = (float *)(s.io_base + 4 * stride); s.d_mask = (uint8_t *)(s.io_base + 5 * stride);
    s.d_w[0] = (float *)(s.io_base + 6 * stride); s.d_w[1] = (float *)(s.io_base + 7 * stride);
    s.io_pix = npix;
    return S2PB_OK;
}

static size_t layout_bytes(int w, int h, int DP, int ndir, int cbytes, bool folded)
{
    Slot probe;
    slot_layout(probe, w, h, DP, ndir, cbytes, folded, false);
    return probe.bytes;
}

// The layout a workspace limit (0: none) selects: 0 resident when it is within the limit, else 1 folded when that is, else -1
// (slot_ensure also falls back to the folded layout when the resident one's allocation fails)
static bool fits(size_t bytes, size_t limit) { return limit == 0 || bytes <= limit; }
static int plan_layout(size_t resident, size_t folded, size_t limit)
{
    return fits(resident, limit) ? 0 : fits(folded, limit) ? 1 : -1;
}

// s.base holds at least `bytes` afterwards, or false (nothing allocated; the CUDA error in *err)
static int slot_alloc(Slot &s, size_t bytes, cudaError_t *err)
{
    *err = cudaSuccess;
    if (s.base && bytes <= s.bytes) return S2PB_OK;
    if (s.base) { CK(cudaStreamSynchronize(s.stream)); CK(cudaFree(s.base)); s.base = nullptr; s.bytes = 0; }
    *err = cudaMalloc(&s.base, bytes);
    if (*err != cudaSuccess) { cudaGetLastError(); s.base = nullptr; s.bytes = 0; return S2PB_OK; }
    s.bytes = bytes;
    return S2PB_OK;
}

// Size the slot's workspace for a tile and carve it.  The resident layout when it is within the context's workspace limit
// (s2pb_set_workspace_limit) and its allocation succeeds, else the folded one (allow_fold: the matcher's calls; the stage entry
// points run resident only), else S2PB_ERR_NOMEM naming both sizes.
static int slot_ensure(s2pb_ctx *ctx, Slot &s, int w, int h, int DP, int ndir, int cbytes = 1, bool allow_fold = true)
{
    const size_t limit = ctx->ws_limit;
    const size_t res = layout_bytes(w, h, DP, ndir, cbytes, false), fold = layout_bytes(w, h, DP, ndir, cbytes, true);
    if (s.base && limit != 0 && s.bytes > limit) {        // allocated before the limit was lowered: give it back
        CK(cudaStreamSynchronize(s.stream)); CK(cudaFree(s.base)); s.base = nullptr; s.bytes = 0;
    }
    const int plan = plan_layout(res, fold, limit);
    cudaError_t e = cudaErrorMemoryAllocation;
    bool folded = false;
    int rc;
    if (plan == 0 && (rc = slot_alloc(s, res, &e)) != S2PB_OK) return rc;
    if (plan >= 0 && e != cudaSuccess && allow_fold) {
        folded = true;
        if ((rc = slot_alloc(s, fold, &e)) != S2PB_OK) return rc;
    }
    if (e != cudaSuccess) {
        char why[128];
        if (!fits(allow_fold ? fold : res, limit)) snprintf(why, sizeof why, "the workspace limit is %.2f GiB", limit / 1073741824.0);
        else snprintf(why, sizeof why, "%s", cudaGetErrorString(e));
        return fail(S2PB_ERR_NOMEM, "workspace for a %dx%dx%d tile does not fit: %.2f GiB resident, %.2f GiB folded%s: %s",
                    w, h, DP, res / 1073741824.0, fold / 1073741824.0, allow_fold ? "" : " (not available here)", why);
    }
    s.w = w; s.h = h; s.DP = DP; s.ndir = ndir; s.cbytes = cbytes; s.folded = folded;
    size_t keep = s.bytes;
    slot_layout(s, w, h, DP, ndir, cbytes, folded, true);
    s.bytes = keep;
    return S2PB_OK;
}

static int slot_host_ensure(Slot &s, size_t npix)
{
    if (s.h_pix >= npix) return S2PB_OK;
    if (s.h_in[0]) { cudaFreeHost(s.h_in[0]); s.h_in[0] = nullptr; }
    // one pinned block: 2 inputs, disp, conf, dispR (float) + mask (u8)
    char *p = nullptr;
    CK(cudaMallocHost((void **)&p, npix * (5 * 4 + 1) + 1024));
    s.h_in[0] = (float *)p;
    s.h_in[1] = s.h_in[0] + npix;
    s.h_disp = s.h_in[1] + npix;
    s.h_conf = s.h_disp + npix;
    s.h_dispR = s.h_conf + npix;
    s.h_mask = (uint8_t *)(s.h_dispR + npix);
    s.h_pix = npix;
    return S2PB_OK;
}

static int slot_init(s2pb_ctx *ctx, Slot &s)
{
    s.abort = ctx->abort_words + (&s - ctx->slots.data());
    CK(cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&s.stream2, cudaStreamNonBlocking));
    CK(cudaMalloc((void **)&s.d_small, 256));
    CK(cudaEventCreateWithFlags(&s.fork, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&s.join, cudaEventDisableTiming));
    for (auto &e : s.ev) CK(cudaEventCreate(&e));
    CK(cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming));
    return S2PB_OK;
}

// ------------------------------------------------------------------ library / context entry points

extern "C" int s2pb_version(void) { return S2PB_VERSION; }
extern "C" const char *s2pb_last_error(void) { return g_err.c_str(); }

extern "C" int s2pb_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

extern "C" s2pb_ctx *s2pb_create(int device)
{
    int n = s2pb_device_count();
    if (n <= 0) { fail(S2PB_ERR_CUDA, "no CUDA device is visible: this library has no CPU path"); return nullptr; }
    if (device < 0 || device >= n) { fail(S2PB_ERR_ARG, "device %d out of range [0,%d)", device, n); return nullptr; }
    if (cudaSetDevice(device) != cudaSuccess) { fail(S2PB_ERR_CUDA, "cudaSetDevice(%d) failed", device); return nullptr; }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) { fail(S2PB_ERR_CUDA, "cudaGetDeviceProperties failed"); return nullptr; }
    if (prop.major != 9 || prop.minor != 0) {
        fail(S2PB_ERR_UNSUPPORTED, "device %d is sm_%d%d; this library carries sm_90a code only", device, prop.major, prop.minor);
        return nullptr;
    }
    s2pb_ctx *ctx = new s2pb_ctx;
    ctx->device = device;
    ctx->sm_count = prop.multiProcessorCount;
    if (const char *e = getenv("S2PB_WTA_PRUNE")) ctx->wta_prune = atoi(e) != 0;
    if (cudaHostAlloc((void **)&ctx->abort_words, 64 * sizeof(int), cudaHostAllocMapped) != cudaSuccess) {
        fail(S2PB_ERR_CUDA, "cudaHostAlloc failed"); delete ctx; return nullptr;
    }
    for (int i = 0; i < 64; i++) ctx->abort_words[i] = 0;
    ctx->slots.reserve(64);
    ctx->slots.resize(1);
    if (slot_init(ctx, ctx->slots[0]) != S2PB_OK) { delete ctx; return nullptr; }
    // function attributes are per device: every context sets them for its own (not once per process)
    if (agg_configure() != 0 || agg_chunked_configure() != 0 ||
        cudaFuncSetAttribute(wta_chunked_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * 2048 * 4) != cudaSuccess ||
        cudaFuncSetAttribute(wta_chunked_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * 2048 * 4) != cudaSuccess ||
        cudaFuncSetAttribute(wta_chunked_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * 2048 * 4) != cudaSuccess ||
        cudaFuncSetAttribute(wta_chunked_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * 2048 * 4) != cudaSuccess) {
        fail(S2PB_ERR_CUDA, "cudaFuncSetAttribute failed for the aggregation kernels"); delete ctx; return nullptr;
    }
    return ctx;
}

extern "C" void s2pb_destroy(s2pb_ctx *ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    for (auto &s : ctx->slots) {
        if (s.stream) cudaStreamSynchronize(s.stream);
        if (s.base) cudaFree(s.base);
        if (s.arena) cudaFree(s.arena);
        if (s.io_base) cudaFree(s.io_base);
        if (s.d_small) cudaFree(s.d_small);
        if (s.h_in[0]) cudaFreeHost(s.h_in[0]);
        for (auto &e : s.ev) if (e) cudaEventDestroy(e);
        if (s.done) cudaEventDestroy(s.done);
        if (s.fork) cudaEventDestroy(s.fork);
        if (s.join) cudaEventDestroy(s.join);
        if (s.stream2) { cudaStreamSynchronize(s.stream2); cudaStreamDestroy(s.stream2); }
        if (s.stream) cudaStreamDestroy(s.stream);
    }
    for (auto &b : ctx->pool) cudaFree(b.p);
    for (auto &t : ctx->dct) for (double *q : {t.T10, t.T01, t.TR01, t.mc, t.ms}) if (q) cudaFree(q);
    for (auto &s : ctx->slots) {
        Slot::DctStream &S = s.dcts;
        if (S.copy) { cudaStreamSynchronize(S.copy); cudaStreamDestroy(S.copy); }
        for (int b = 0; b < 2; b++) {
            if (S.h[b]) cudaFreeHost(S.h[b]);
            if (S.d[b]) cudaFree(S.d[b]);
            if (S.copied[b]) cudaEventDestroy(S.copied[b]);
            if (S.consumed[b]) cudaEventDestroy(S.consumed[b]);
        }
        if (S.acc) cudaFree(S.acc);
    }
    geoid_free(ctx);
    if (ctx->abort_words) cudaFreeHost(ctx->abort_words);
    delete ctx;
}

extern "C" int s2pb_default_params(const char *algo, s2pb_mgm_params *p)
{
    if (!algo || !p) return fail(S2PB_ERR_ARG, "null argument");
    memset(p, 0, sizeof *p);
    p->ndir = 8; p->census_win = 5; p->P1 = 8.f; p->P2 = 32.f; p->lr_mode = 1; p->lr_tau = 1.f;
    p->mindiff = -1.f; p->refine = 1; p->fix_overcount = 1; p->timeout_ms = 0;
    if (!strcmp(algo, "mgm")) {          // s2p/block_matching.py:155-186
        p->tsgm = 3; p->median = 1; p->remove_small_cc = 0; p->subpix = 1; p->scales = -1;
    } else if (!strcmp(algo, "mgm_multi")) {   // s2p/block_matching.py:269-308 ; TSGM default 4 (mgm_multiscale.cc:120)
        p->tsgm = 4; p->median = 0; p->remove_small_cc = 25; p->subpix = 2; p->scales = 6;
    } else if (!strcmp(algo, "mgm_multi_lsd")) {   // s2p/block_matching.py:191-266 (the caller supplies the LSD weight maps)
        p->tsgm = 4; p->median = 1; p->remove_small_cc = 25; p->subpix = 2; p->scales = 6; p->P1 = 12.f; p->P2 = 48.f;
    } else return fail(S2PB_ERR_ARG, "unknown algo '%s'", algo);
    return S2PB_OK;
}

extern "C" int s2pb_num_slots(const s2pb_ctx *ctx) { return ctx ? (int)ctx->slots.size() : 0; }
extern "C" long long s2pb_kernel_launches(const s2pb_ctx *ctx) { return ctx ? ctx->launches.load() : 0LL; }
extern "C" long long s2pb_folded_calls(const s2pb_ctx *ctx) { return ctx ? ctx->folded_calls.load() : 0LL; }

extern "C" int s2pb_set_workspace_limit(s2pb_ctx *ctx, long long bytes)
{
    if (!ctx || bytes < 0) return fail(S2PB_ERR_ARG, "bad argument");
    ctx->ws_limit = (size_t)bytes;
    return S2PB_OK;
}

extern "C" int s2pb_sync(s2pb_ctx *ctx)
{
    if (!ctx) return fail(S2PB_ERR_ARG, "null context");
    CK(cudaSetDevice(ctx->device));
    for (auto &s : ctx->slots) if (s.stream) CK(cudaStreamSynchronize(s.stream));
    return S2PB_OK;
}

static int ensure_slots(s2pb_ctx *ctx, int nslots)
{
    // slots may be requested from several host threads (one per workspace for mgm_multi); the vector's capacity is reserved at
    // creation so that references to existing slots stay valid while it grows
    if (nslots > 64) return fail(S2PB_ERR_ARG, "at most 64 workspaces per context");
    std::lock_guard<std::mutex> lock(ctx->dct_mu);
    while ((int)ctx->slots.size() < nslots) {
        ctx->slots.emplace_back();
        int r = slot_init(ctx, ctx->slots.back());
        if (r != S2PB_OK) return r;
    }
    return S2PB_OK;
}

// ------------------------------------------------------------------ matcher calls and timeouts

using Deadline = std::optional<std::chrono::steady_clock::time_point>;

// One call into the matcher: what its entry point decides once and every stage of the call reads.  Calls on different slots
// may run at once from different host threads, so nothing of a call is kept on the context.
struct MatchCall {
    Slot &s;                                   // the workspace
    cudaStream_t st;                           // the stream the call is enqueued on: the slot's, or the caller's
    Deadline deadline;                         // none: the call waits without a timeout
    const float *wl = nullptr, *wr = nullptr;  // device weight images (-wl / -wr) at full resolution, both or neither
    float *pkr[2] = {nullptr, nullptr};        // device destinations of the PKR images of the two views, or none
};

// The timeout contract (timeout_ms -> S2PB_ERR_TIMEOUT -> subprocess.TimeoutExpired upstream) counts from the API
// entry: every host-side wait of a matcher call goes through sync_or_timeout, also the per-level read-backs of mgm_multi.
static Deadline deadline_after(long long timeout_ms)
{
    if (timeout_ms <= 0) return std::nullopt;
    return std::chrono::steady_clock::now() + std::chrono::milliseconds(timeout_ms);
}
// stop everything that is in flight on any slot (s2pb_mgm_batch, which drives them all, on an error): raise every slot's abort
// word (the persistent aggregation kernels drain), wait for every slot stream -- some of them DMA into the caller's buffers --
// then clear the words
static void drain_all(s2pb_ctx *ctx)
{
    for (auto &s : ctx->slots) *(volatile int *)s.abort = 1;
    for (auto &s : ctx->slots) { cudaStreamSynchronize(s.stream); cudaStreamSynchronize(s.stream2); }
    for (auto &s : ctx->slots) *(volatile int *)s.abort = 0;
}
// Wait for the call's stream.  Past the deadline, only the call's own slot is stopped: its abort word is raised until the
// call's stream and the slot's streams have drained, so calls on other slots run on undisturbed.
static int sync_or_timeout(const MatchCall &c)
{
    if (!c.deadline) { CK(cudaStreamSynchronize(c.st)); return S2PB_OK; }
    for (;;) {
        cudaError_t e = cudaStreamQuery(c.st);
        if (e == cudaSuccess) return S2PB_OK;
        if (e != cudaErrorNotReady) return fail(S2PB_ERR_CUDA, "stream failed: %s", cudaGetErrorString(e));
        if (std::chrono::steady_clock::now() > *c.deadline) {
            *(volatile int *)c.s.abort = 1;
            for (cudaStream_t q : {c.st, c.s.stream, c.s.stream2}) cudaStreamSynchronize(q);
            *(volatile int *)c.s.abort = 0;
            return fail(S2PB_ERR_TIMEOUT, "matcher exceeded its timeout");
        }
        std::this_thread::sleep_for(std::chrono::microseconds(100));
    }
}

// Is another workspace's aggregation queued or running?  (ev[3] of a slot is recorded right after its aggregation; an event that
// was never recorded reads as complete.)  A racy answer is harmless: it only picks the grid size.
static bool other_aggregation_pending(s2pb_ctx *ctx, const Slot &me)
{
    const size_t n = ctx->slots.size();
    for (size_t k = 0; k < n; k++) {
        const Slot &o = ctx->slots[k];
        if (&o == &me || !o.ev[3]) continue;
        if (cudaEventQuery(o.ev[3]) == cudaErrorNotReady) return true;
    }
    return false;
}

// ------------------------------------------------------------------ stage launchers

// CENSUS_NCC_WIN: the reference takes any win and uses win / 2 as the radius (mgm_costvolume.cc:109).  win <= 1 gives codes
// of no bit, whose cost is 0 / 0; from 12 on (side 13) the popcount overflows the 8-bit cost codes (agg_kernel.cuh)
static int census_win_ok(int win)
{
    if (win < 2) return fail(S2PB_ERR_ARG, "census window must be at least 2 (got %d)", win);
    if (win > 11) return fail(S2PB_ERR_UNSUPPORTED, "census windows wider than 11 are not supported (got %d)", win);
    return S2PB_OK;
}

static int check_params(const s2pb_mgm_params *p, int w, int h, int dmin, int dmax)
{
    if (!p) return fail(S2PB_ERR_ARG, "null params");
    int rc;
    if (w < 2 || h < 2) return fail(S2PB_ERR_ARG, "image too small (%dx%d)", w, h);
    if (dmax <= dmin) return fail(S2PB_ERR_ARG, "need dmin < dmax (got %d, %d)", dmin, dmax);
    if (p->ndir != 2 && p->ndir != 4 && p->ndir != 8) return fail(S2PB_ERR_ARG, "ndir must be 2, 4 or 8");
    if (p->tsgm < 1 || p->tsgm > 4) return fail(S2PB_ERR_ARG, "tsgm must be 1..4");
    rc = census_win_ok(p->census_win);
    if (rc != S2PB_OK) return rc;
    if (p->median < 0 || p->median > 2) return fail(S2PB_ERR_ARG, "median radius must be 0..2");
    if (p->refine < 0 || p->refine > 2) return fail(S2PB_ERR_ARG, "refine must be 0 (none), 1 (vfit) or 2 (parabola)");
    if (p->subpix != 1 && p->subpix != 2) return fail(S2PB_ERR_UNSUPPORTED, "SUBPIX must be 1 or 2");
    if (p->scales < 0 && p->subpix != 1) return fail(S2PB_ERR_ARG, "SUBPIX=2 only exists in mgm_multi (scales >= 0)");
    if (p->scales < 0 && p->remove_small_cc > 0) return fail(S2PB_ERR_UNSUPPORTED, "REMOVESMALLCC is only wired into the mgm_multi path");
    if (p->lr_mode < 0 || p->lr_mode > 2) return fail(S2PB_ERR_ARG, "TESTLRRL must be 0, 1 or 2");
    if (p->scales < 0 && p->lr_mode == 2) return fail(S2PB_ERR_ARG, "TESTLRRL=2 only exists in mgm_multi");
    // pixel indices of the pyramid, the label ranges and the post filters are 32-bit
    if ((long long)w * h > INT_MAX) return fail(S2PB_ERR_UNSUPPORTED, "tiles of more than 2^31 - 1 pixels are not supported (%dx%d)", w, h);
    if (abs(dmin) > 16000 || abs(dmax) > 16000) return fail(S2PB_ERR_ARG, "disparity bounds out of the int16 label range");
    if (p->cost < 0 || p->cost >= S2PB_COST_COUNT) return fail(S2PB_ERR_ARG, "cost must be one of S2PB_COST_* (got %d)", p->cost);
    return S2PB_OK;
}

// cost LUT for scaled census costs: cost(r) = (float)((double)r * ratio / nch), mgm_costvolume.h:90-91.  The code's bits and
// its float channels nch come from the window's side (census_tools.cc:76-99), the ratio 25 / win^2 from win itself.
static bool cost_lut(int win, float lut[kCostLut])
{
    const int nbits = census_bits(win), nch = (nbits / 8 + 3) / 4;
    const float ratio = (float)(5 * 5 / ((double)win * win));
    bool identity = true;
    for (int r = 0; r < kCostLut; r++) {
        float fr = (float)r;
        lut[r] = (float)((double)fr * 1.0 * (double)ratio / nch);
        if (lut[r] != fr) identity = false;
    }
    return !identity;
}

// Label hull of each view (main_mgm.cc:178,207,210-216).  The no-data sentinel range [dmin, dmin+1]
// always lies inside the left hull; on the right view it only matters when the secondary image
// really holds no-data pixels, and then it may stick out of [-dmax, -dmin].
static void plan_labels(int dmin, int dmax, bool sec_has_nodata, int gminv[2], int gmaxv[2])
{
    gminv[0] = dmin; gmaxv[0] = dmax;
    gminv[1] = -dmax; gmaxv[1] = -dmin;
    if (sec_has_nodata) {
        if (dmin < gminv[1]) gminv[1] = dmin;
        if (dmin + 1 > gmaxv[1]) gmaxv[1] = dmin + 1;
    }
}

// Labels per lane of a slab of D labels (DP = 32 LPL slots): the narrowest register-resident width up to 512 labels, else
// ceil(D / 32) 32-slot chunks for the chunk-skipping kernels (wide_slab), up to 2048 labels.
static int slab_lpl(int D, int *lpl)
{
#define FITS(n) if (32 * n >= D) { *lpl = n; return S2PB_OK; }
    S2PB_FOR_EACH_LPL(FITS)
#undef FITS
    if (D > 2048) return fail(S2PB_ERR_UNSUPPORTED, "a slab of %d labels: at most 2048 are supported", D);
    *lpl = (D + 31) / 32;
    return S2PB_OK;
}

// the workspace arithmetic of a w x h tile of D labels, for the C ABI (no device): slot_layout of the slab slab_lpl gives
static int workspace_args(int w, int h, int D, int ndir, int cost_bytes, int *DP)
{
    if (w < 2 || h < 2 || D < 1) return fail(S2PB_ERR_ARG, "bad tile shape %dx%d, %d labels", w, h, D);
    if (ndir != 2 && ndir != 4 && ndir != 8) return fail(S2PB_ERR_ARG, "ndir must be 2, 4 or 8");
    if (cost_bytes != 1 && cost_bytes != 4) return fail(S2PB_ERR_ARG, "cost_bytes must be 1 (census codes) or 4 (float costs)");
    int LPL, rc = slab_lpl(D, &LPL);
    if (rc != S2PB_OK) return rc;
    *DP = 32 * LPL;
    return S2PB_OK;
}
extern "C" long long s2pb_workspace_bytes(int w, int h, int D, int ndir, int cost_bytes, int folded)
{
    int DP, rc = workspace_args(w, h, D, ndir, cost_bytes, &DP);
    if (rc != S2PB_OK) return rc;
    return (long long)layout_bytes(w, h, DP, ndir, cost_bytes, folded != 0);
}
extern "C" int s2pb_workspace_layout(int w, int h, int D, int ndir, int cost_bytes, long long limit)
{
    int DP, rc = workspace_args(w, h, D, ndir, cost_bytes, &DP);
    if (rc != S2PB_OK) return rc;
    if (limit < 0) return fail(S2PB_ERR_ARG, "negative limit");
    const int plan = plan_layout(layout_bytes(w, h, DP, ndir, cost_bytes, false), layout_bytes(w, h, DP, ndir, cost_bytes, true), (size_t)limit);
    return plan >= 0 ? plan : fail(S2PB_ERR_NOMEM, "neither layout fits the limit");
}

static void fill_pass(PassDesc &pd, int pass, int w, int h)
{
    const long long W = w, H = h;
    switch (pass) {   // scan coordinates of the table at mgm_core.cc:884-891 (see SURVEY.md appendix B)
    case 0: pd.nS = h; pd.nI = w; pd.base = 0;                     pd.strideS = w;  pd.strideI = 1;  pd.type = 0; break;
    case 1: pd.nS = h; pd.nI = w; pd.base = (H - 1) * W + (W - 1); pd.strideS = -w; pd.strideI = -1; pd.type = 0; break;
    case 2: pd.nS = w; pd.nI = h; pd.base = (H - 1) * W;           pd.strideS = 1;  pd.strideI = -w; pd.type = 0; break;
    case 3: pd.nS = w; pd.nI = h; pd.base = W - 1;                 pd.strideS = -1; pd.strideI = w;  pd.type = 0; break;
    case 4: pd.nS = h; pd.nI = w; pd.base = W - 1;                 pd.strideS = w;  pd.strideI = -1; pd.type = 1; break;
    case 5: pd.nS = w; pd.nI = h; pd.base = (H - 1) * W + (W - 1); pd.strideS = -1; pd.strideI = -w; pd.type = 1; break;
    case 6: pd.nS = h; pd.nI = w; pd.base = (H - 1) * W;           pd.strideS = -w; pd.strideI = 1;  pd.type = 1; break;
    default: pd.nS = w; pd.nI = h; pd.base = 0;                    pd.strideS = 1;  pd.strideI = w;  pd.type = 1; break;
    }
    pd.nBands = (pd.nS + kNW - 1) / kNW;
}

// A slab wider than 512 slots (more labels than the register-resident kernels hold) goes through the chunk-skipping cost,
// aggregation and WTA kernels (agg_chunked.cuh), which run with any width up to 2048 slots: the reference has no such limit
// (mgm_costvolume.cc:63-72 allocates one vector per pixel of its own length).  Both flavours: census codes and float costs.
static bool wide_slab(int LPL) { return 32 * LPL > 512; }

// Enqueue the MGM aggregation of `nviews` views of slot s, from view first_view, on stream st.  The resident layout: ONE persistent
// launch carrying the ndir passes of the views.  The folded layout (s.folded): ndir launches in pass order, launch p carrying pass p
// of the views; each adds its pass into the views' S, so the order of the launches is the order of the sum.  Each pass has its own
// progress counters, reset once; the item queue is reset before every launch.
// general: the float-cost flavour; wgt[vi] = that view's weight image or nullptr (general only)
// gminv: label of slot 0 per view (read by the chunk-skipping kernel only)
// ctas_per_sm > 0 caps the persistent CTAs per SM of a resident launch (agg_launch); the folded launches take no cap
static int launch_aggregate(s2pb_ctx *ctx, Slot &s, int nviews, int w, int h, int LPL, float P1, float P2, int ndir, int tsgm,
                            const float *lut, cudaStream_t st, bool general = false, const float *const *wgt = nullptr,
                            const int *gminv = nullptr, int first_view = 0, int ctas_per_sm = 0)
{
    const int mb = max_bands(w, h), sm = ctx->sm_count;
    int *counter = s.next_item + 16 * first_view;          // two launches may be in flight at once: one work counter each
    for (int vi = first_view; vi < first_view + nviews; vi++) CK(cudaMemsetAsync(s.v[vi].progress, 0, (size_t)kMaxPasses * mb * 4, st));
    const int passes = s.folded ? 1 : ndir;                // per launch
    for (int p0 = 0; p0 < ndir; p0 += passes) {
        AggFoldParams F;                      // a resident launch takes its AggParams part,
        ChunkedFoldParams Q;                  // and a resident chunk-skipping one this one's ChunkedParams part
        memset(&F, 0, sizeof F);
        memset(&Q, 0, sizeof Q);
        AggParams &P = F;
        for (int vi = first_view; vi < first_view + nviews; vi++)
            for (int p = p0; p < p0 + passes; p++) {
                // slot_layout leaves null what the other layout holds: L_p in the folded layout, the FoldView in the resident one
                const int q = P.nPV++;
                PassDesc &pd = P.pv[q];
                fill_pass(pd, p, w, h);
                pd.C = s.v[vi].C; pd.L = s.v[vi].L[p]; pd.Lmin = s.v[vi].Lmin[p];
                pd.W = (general && wgt) ? wgt[vi] : nullptr;
                pd.progress = s.v[vi].progress + (size_t)p * mb;
                if (pd.nBands > P.maxBands) P.maxBands = pd.nBands;
                Q.fv[q] = F.fv[q] = FoldView{s.v[vi].S, s.v[vi].Lb, s.v[vi].am[p]};
                Q.lo[q] = s.v[vi].lo; Q.hi[q] = s.v[vi].hi; Q.gmin[q] = gminv ? gminv[vi] : 0;
            }
        P.P1 = P1; P.P2 = P2; P.next_item = counter; P.abort_flag = s.abort; P.lut = general ? nullptr : lut;
        P.general = general ? 1 : 0;
        Q.first = F.first = p0 == 0;
        CK(cudaMemsetAsync(counter, 0, 4, st));
        int r;
        if (wide_slab(LPL)) {
            Q.A = P;
            Q.DP = 32 * LPL;
            r = s.folded ? agg_chunked_launch<true>(tsgm, Q, sm, st) : agg_chunked_launch<false>(tsgm, Q, sm, st);
        } else {
            r = s.folded ? agg_launch<true>(LPL, tsgm, F, sm, st) : agg_launch<false>(LPL, tsgm, F, sm, st, ctas_per_sm);
        }
        if (r == -2)
            return fail(S2PB_ERR_UNSUPPORTED, "no %s%s aggregation kernel serves a slab of %d slots with TSGM %d%s",
                        s.folded ? "folded " : "", wide_slab(LPL) ? "chunk-skipping" : "register-resident", 32 * LPL, tsgm,
                        general ? " (float costs)" : "");
        if (r != 0) return fail(S2PB_ERR_CUDA, "aggregation launch failed: %s", cudaGetErrorString(cudaGetLastError()));
        ctx->launches++;
    }
    return S2PB_OK;
}

// f(std::integral_constant<int, LPL>()): the instantiation for a register-resident width LPL
template <class F> static int with_lpl(int LPL, F &&f)
{
    switch (LPL) {
#define CASE(n) case n: f(std::integral_constant<int, n>()); return S2PB_OK;
    S2PB_FOR_EACH_LPL(CASE)
#undef CASE
    }
    return fail(S2PB_ERR_UNSUPPORTED, "unsupported labels-per-lane %d", LPL);
}

// census 3x3 / 5x5 up to 8 labels per lane: the strip-staged kernel; wider windows, the half-pixel pass and 12 / 16 labels per
// lane: the per-pixel one, for codes of `bits` bits (cost_kernel's BITS)
template <int LPL> static void launch_cost_t(s2pb_ctx *ctx, const CostGenParams &G, int bits, uint8_t *C, cudaStream_t st)
{
    const int sm = ctx->sm_count;
    auto go = [&](auto kernel) { launch(ctx, kernel, sm * 8, 256, 0, st, G.cu, G.cv0, G.cv1, G.w, G.h, G.lo, G.hi, G.gmin, C, G.cuh, G.cv0h, G.cv1h); };
    if (G.zoom == 2) {
        if (bits == 32) go(cost_kernel<LPL, true, 32>);
        else if (bits == 64) go(cost_kernel<LPL, true, 64>);
        else go(cost_kernel<LPL, true, 128>);
    } else if (bits == 64) go(cost_kernel<LPL, false, 64>);
    else if (bits == 128) go(cost_kernel<LPL, false, 128>);
    else if constexpr (LPL <= 8) launch(ctx, cost_strip_kernel<LPL>, sm * 16, kCostStripThreads, 0, st, G.cu, G.cv0, G.w, G.h, G.lo, G.hi, G.gmin, C);
    else go(cost_kernel<LPL, false, 32>);
}

// The cost volume of one view into G.C.  general: float costs of G.cost (census through G.lut included); else the 8-bit census
// codes of G.cu against G.cv0 (G.cv1 at odd labels when G.zoom = 2), read as bytes from G.C, where G.win <= 5 leaves the high
// half of a code zero and G.win >= 8 puts its second word in G.cuh / G.cv0h / G.cv1h.  A wide slab (wide_slab) is written only
// on the chunks of each pixel's span.
static int launch_cost(s2pb_ctx *ctx, int LPL, bool general, const CostGenParams &G, cudaStream_t st)
{
    const int sm = ctx->sm_count;
    uint8_t *C8 = (uint8_t *)G.C;
    int rc = S2PB_OK;
    if (wide_slab(LPL)) {
        if (general) launch(ctx, cost_gen_chunked_kernel, sm * 8, 256, 0, st, G, 32 * LPL);
        else {
            auto go = [&](auto kernel) { launch(ctx, kernel, sm * 8, 256, 0, st, G.cu, G.cv0, G.cv1, G.w, G.h, G.lo, G.hi, G.gmin, 32 * LPL, C8, G.cuh, G.cv0h, G.cv1h); };
            const bool wide = census_words(G.win) == 2;
            if (G.zoom == 2) { if (wide) go(cost_chunked_kernel<true, 128>); else go(cost_chunked_kernel<true, 64>); }
            else if (wide) go(cost_chunked_kernel<false, 128>);
            else go(cost_chunked_kernel<false, 64>);
        }
    } else if (general) {
        rc = with_lpl(LPL, [&](auto k) { constexpr int K = decltype(k)::value; launch(ctx, cost_gen_kernel<K>, sm * 8, 256, 0, st, G); });
    } else {
        rc = with_lpl(LPL, [&](auto k) {
            constexpr int K = decltype(k)::value;
            launch_cost_t<K>(ctx, G, G.win <= 5 ? 32 : census_words(G.win) == 2 ? 128 : 64, C8, st);
        });
    }
    if (rc != S2PB_OK) return rc;
    CK(cudaGetLastError());
    return S2PB_OK;
}

template <int LPL> static void launch_wta_t(s2pb_ctx *ctx, const WtaParams &P, const FoldPlanes *F, cudaStream_t st, bool general,
                                            bool pruned)
{
    const int sm = ctx->sm_count;
    if (F) {
        if (general) launch(ctx, wta_fold_kernel<LPL, true>, sm * 16, kWtaThreads, 0, st, P, *F);
        else launch(ctx, wta_fold_kernel<LPL, false>, sm * 16, kWtaThreads, 0, st, P, *F);
        return;
    }
    if constexpr (wta_pruned_width(LPL))
        if (pruned) { launch(ctx, wta_pruned_kernel<LPL>, sm * 16, kWtaThreads, 0, st, P); return; }
    if (general) launch(ctx, wta_kernel<LPL, true>, sm * 16, kWtaThreads, 0, st, P);
    else launch(ctx, wta_kernel<LPL, false>, sm * 16, kWtaThreads, 0, st, P);
}
// The WTA of view vi of slot s.  A wide slab without a dense S: wta_chunked_kernel.  In the folded layout, S and the arg-minimum
// planes of the view instead of its pass volumes: wta_fold_kernel, or wta_chunked_kernel's FOLD instantiation on a wide slab; no
// dense S output (the stage entry points run resident).  In the resident layout, the census flavour's eight-pass WTA without a
// dense S or PKR output, on the widths wta_pruned_kernel serves: that kernel, which reads only the labels that can still win,
// unless the context was created with S2PB_WTA_PRUNE=0 (s2pb_ctx::wta_prune).  Everything else: wta_kernel.
static int launch_wta(s2pb_ctx *ctx, const Slot &s, int vi, int LPL, const WtaParams &P, cudaStream_t st, bool general)
{
    const int sm = ctx->sm_count;
    FoldPlanes F;
    memset(&F, 0, sizeof F);
    if (s.folded) {
        F.S = s.v[vi].S;
        for (int d = 0; d < kMaxPasses; d++) F.am[d] = s.v[vi].am[d];
    }
    int rc = S2PB_OK;
    if (P.S == nullptr && wide_slab(LPL)) {
        const int DP = 32 * LPL;
        const size_t smem = (size_t)(kWtaThreads / 32) * DP * sizeof(float);
        auto go = [&](auto kernel) { launch(ctx, kernel, sm * 16, kWtaThreads, smem, st, P, DP, F); };
        if (s.folded && general) go(wta_chunked_kernel<true, true>);
        else if (s.folded) go(wta_chunked_kernel<false, true>);
        else if (general) go(wta_chunked_kernel<true>);
        else go(wta_chunked_kernel<false>);
    } else {
        const bool pruned = ctx->wta_prune && !general && P.ndir == kMaxPasses && P.S == nullptr && P.pkr == nullptr &&
                            wta_pruned_width(LPL);
        rc = with_lpl(LPL, [&](auto k) {
            constexpr int K = decltype(k)::value;
            launch_wta_t<K>(ctx, P, s.folded ? &F : nullptr, st, general, pruned);
        });
    }
    if (rc != S2PB_OK) return rc;
    CK(cudaGetLastError());
    return S2PB_OK;
}

static void fill_wta(WtaParams &P, const ViewWS &v, int ndir, int gmin, const s2pb_mgm_params *p, const float *lut, size_t npix)
{
    memset(&P, 0, sizeof P);
    P.pkr = nullptr;
    for (int d = 0; d < ndir; d++) P.L[d] = v.L[d];
    P.C = v.C; P.lo = v.lo; P.hi = v.hi; P.lut = lut;
    P.ndir = ndir; P.gmin = gmin; P.fix_overcount = p->fix_overcount; P.refine = p->refine;
    P.inv_zoom_div = 1.f; P.npix = npix; P.S = nullptr; P.Dout = 0;
    P.disp = v.disp; P.cost = v.cost; P.conf = v.conf;
}

// ------------------------------------------------------------------ the matched image's DCT round trip (dct_kernels.cuh)

// Coefficient tables for rows of n pixels, computed on the host (libm, like the reference's DCT: device cos / sin differ in the
// last bit).  FFTW's unnormalised definitions, each table [output][input] row-major:
//   REDFT10  Y[k] = sum_j 2 cos(pi (j + 1/2) k / n) X[j]
//   REDFT01  Y[i] = X[0] + sum_{k>=1} 2 cos(pi k (i + 1/2) / n) X[k]
//   RODFT01  Y[i] = (-1)^i X[n-1] + sum_{k<n-1} 2 sin(pi (k + 1) (i + 1/2) / n) X[k]
// Up to kDctDenseWidth they are kept on the device, once per width, whatever they take (1.5 GiB at 8192 with the half shift).
// Wider rows keep a table resident while the context's resident wide tables stay within its table budget (dct_budget), and
// stream it in K-panels otherwise.  Either way every product runs through dct_gemm_kernel (dct_product): a resident table is
// one panel.
constexpr int kDctDenseWidth = 8192;
enum DctKind { kDctT10 = 0, kDctT01 = 1, kDctTR01 = 2 };

static double dct_coef(int kind, int n, int r, int c)
{
    const double pi = 3.14159265358979323846264338327950288;
    if (kind == kDctT10) return 2.0 * cos(pi * (c + 0.5) * r / n);
    if (kind == kDctT01) return (c == 0) ? 1.0 : 2.0 * cos(pi * c * (r + 0.5) / n);
    return (c == n - 1) ? ((r & 1) ? -1.0 : 1.0) : 2.0 * sin(pi * (c + 1) * (r + 0.5) / n);
}

// dst[q][c - c0] = coefficient (rows[q], c) of table `kind` (rows == nullptr: row q), c in [c0, c0 + ncols), on a pool of host
// threads (one block of rows each)
static void dct_fill(int kind, int n, const int *rows, int nrows, int c0, int ncols, double *dst)
{
    auto work = [=](int q0, int q1) {
        for (int q = q0; q < q1; q++) {
            const int r = rows ? rows[q] : q;
            double *o = dst + (size_t)q * ncols;
            for (int c = 0; c < ncols; c++) o[c] = dct_coef(kind, n, r, c0 + c);
        }
    };
    const long long terms = (long long)nrows * ncols;
    int nt = (int)std::min<long long>(std::max(1u, std::thread::hardware_concurrency()), std::min<long long>(64, terms / 65536 + 1));
    nt = std::min(nt, nrows);
    if (nt <= 1) { work(0, nrows); return; }
    std::vector<std::thread> pool;
    for (int t = 0; t < nt; t++) pool.emplace_back(work, (int)((long long)nrows * t / nt), (int)((long long)nrows * (t + 1) / nt));
    for (auto &th : pool) th.join();
}

extern "C" int s2pb_dct_coefficients(int kind, int n, int row0, int nrows, int col0, int ncols, double *out)
{
    if (kind < kDctT10 || kind > kDctTR01 || n < 1 || !out || row0 < 0 || nrows < 0 || col0 < 0 || ncols < 0 || row0 + nrows > n ||
        col0 + ncols > n)
        return fail(S2PB_ERR_ARG, "bad argument");
    std::vector<int> rows(nrows);
    for (int q = 0; q < nrows; q++) rows[q] = row0 + q;
    dct_fill(kind, n, rows.data(), nrows, col0, ncols, out);
    return S2PB_OK;
}

extern "C" int s2pb_set_dct_table_limit(s2pb_ctx *ctx, long long bytes)
{
    if (!ctx || bytes < 0) return fail(S2PB_ERR_ARG, "bad argument");
    std::lock_guard<std::mutex> lock(ctx->dct_mu);
    ctx->dct_limit = (size_t)bytes;
    return S2PB_OK;
}

// the device bytes the context may hold in resident tables wider than kDctDenseWidth: its table limit, and no more than its
// workspace limit when one is set
static size_t dct_budget(const s2pb_ctx *ctx)
{
    return ctx->ws_limit ? std::min(ctx->dct_limit, ctx->ws_limit) : ctx->dct_limit;
}

// The tables of rows of n pixels (half: with what the half-pixel shift of SUBPIX = 2 needs, RODFT01 and the phase factors
// cos(k a), sin(k a), a = (pi / n) * (-1/2), shear.c:66-79).  Above kDctDenseWidth a table that the budget or the device
// cannot hold stays null: the caller streams it.
static int dct_tables(s2pb_ctx *ctx, int n, bool half, const s2pb_ctx::DctTab **out)
{
    std::lock_guard<std::mutex> lock(ctx->dct_mu);
    s2pb_ctx::DctTab *t = nullptr;
    for (auto &e : ctx->dct) if (e.n == n) t = &e;
    if (!t) { ctx->dct.push_back({n, nullptr, nullptr, nullptr, nullptr, nullptr}); t = &ctx->dct.back(); }
    const bool wide = n > kDctDenseWidth;
    const size_t nn = (size_t)n * n;
    std::vector<double> h;
    auto upload = [&](double **dst, size_t count) -> int {
        cudaError_t e = cudaMalloc((void **)dst, count * sizeof(double));
        if (e != cudaSuccess) { cudaGetLastError(); *dst = nullptr; return fail(S2PB_ERR_NOMEM, "DCT table of %zu bytes: %s", count * 8, cudaGetErrorString(e)); }
        CK(cudaMemcpy(*dst, h.data(), count * sizeof(double), cudaMemcpyHostToDevice));
        return S2PB_OK;
    };
    auto table = [&](double **dst, int kind) -> int {
        if (*dst) return S2PB_OK;
        if (wide && ctx->dct_wide_bytes + nn * 8 > dct_budget(ctx)) return S2PB_OK;       // streamed
        h.resize(nn);
        dct_fill(kind, n, nullptr, n, 0, n, h.data());
        int rc = upload(dst, nn);
        if (!wide || rc == S2PB_ERR_CUDA) return rc;
        if (*dst) ctx->dct_wide_bytes += nn * 8;
        return S2PB_OK;                                                                      // (out of memory: streamed)
    };
    int rc;
    if ((rc = table(&t->T10, kDctT10)) != S2PB_OK) return rc;
    if ((rc = table(&t->T01, kDctT01)) != S2PB_OK) return rc;
    if (half && (rc = table(&t->TR01, kDctTR01)) != S2PB_OK) return rc;
    if (half && !t->mc) {
        const float q = 0.5f, translation = -q;                  // shift() passes (0., -q) as floats, mgm_costvolume.cc:35
        const double tt = 0 * 0.0f + translation, a = (M_PI / n) * tt;
        h.resize(n);
        for (int k = 0; k < n; k++) h[k] = cos(k * a);
        if ((rc = upload(&t->mc, n)) != S2PB_OK) return rc;
        for (int k = 0; k < n; k++) h[k] = sin(k * a);
        if ((rc = upload(&t->ms, n)) != S2PB_OK) return rc;
    }
    *out = t;
    return S2PB_OK;
}

// Columns per K-panel of a table streamed for rows of n pixels: panels of about 64 MiB, a multiple of the products' K tile
static int dct_panel_cols(int n)
{
    const size_t cols = ((size_t)64 << 20) / 8 / (size_t)n / kGemmTK * kGemmTK;
    return (int)std::max<size_t>(kGemmTK, std::min<size_t>(cols, (size_t)n));
}

// the staging of slot s's streamed products for panels of `panel` doubles and, when acc_pix > 0, that many running sums
static int dct_stream_ensure(Slot &s, size_t panel, size_t acc_pix)
{
    Slot::DctStream &S = s.dcts;
    if (!S.copy) {
        CK(cudaStreamCreateWithFlags(&S.copy, cudaStreamNonBlocking));
        for (int b = 0; b < 2; b++) {
            CK(cudaEventCreateWithFlags(&S.copied[b], cudaEventDisableTiming));
            CK(cudaEventCreateWithFlags(&S.consumed[b], cudaEventDisableTiming));
        }
    }
    // the buffers are replaced only after the products that read them: each panel's product records consumed[b]
    if (S.panel < panel || S.acc_pix < acc_pix)
        for (int b = 0; b < 2; b++) { CK(cudaEventSynchronize(S.consumed[b])); CK(cudaEventSynchronize(S.copied[b])); }
    if (S.panel < panel) {
        for (int b = 0; b < 2; b++) {
            if (S.h[b]) { cudaFreeHost(S.h[b]); S.h[b] = nullptr; }
            if (S.d[b]) { cudaFree(S.d[b]); S.d[b] = nullptr; }
        }
        S.panel = 0;
        for (int b = 0; b < 2; b++) {
            if (cudaMallocHost((void **)&S.h[b], panel * 8) != cudaSuccess || cudaMalloc((void **)&S.d[b], panel * 8) != cudaSuccess) {
                cudaGetLastError();
                return fail(S2PB_ERR_NOMEM, "staging of the streamed DCT tables (2 x %zu bytes pinned and on the device)", panel * 8);
            }
        }
        S.panel = panel;
    }
    if (S.acc_pix < acc_pix) {
        if (S.acc) { CK(cudaFree(S.acc)); S.acc = nullptr; S.acc_pix = 0; }
        if (cudaMalloc((void **)&S.acc, acc_pix * 8) != cudaSuccess) {
            cudaGetLastError();
            return fail(S2PB_ERR_NOMEM, "running sums of the streamed DCT round trip (%zu bytes)", acc_pix * 8);
        }
        S.acc_pix = acc_pix;
    }
    return S2PB_OK;
}

// One product through table `kind` for rows of n pixels, restricted to the table rows `rows` (nullptr: all n; nrows of them):
// product(P, ldp, listed, k0, k1) multiplies by the panel P of the table's inputs [k0, k1) (dct_gemm_kernel).  A resident
// table T is one panel, product(T, n, false, 0, n).  A streamed one (T null) goes in K-panels of the listed rows: panel p is
// built on the host into staging buffer p % 2 while the device multiplies panel p - 1, uploaded on the slot's copy stream once
// the product of panel p - 2 is done with device buffer p % 2, and multiplied on st.  Returns once the last panel is enqueued.
template <class F>
static int dct_product(Slot &s, cudaStream_t st, const double *T, int kind, int n, const int *rows, int nrows, F &&product)
{
    if (T) {
        product(T, n, false, 0, n);
        return S2PB_OK;
    }
    const int kp = dct_panel_cols(n);
    int rc = dct_stream_ensure(s, (size_t)nrows * kp, 0);
    if (rc != S2PB_OK) return rc;
    Slot::DctStream &S = s.dcts;
    for (int k0 = 0, p = 0; k0 < n; k0 += kp, p++) {
        const int b = p & 1, k1 = std::min(n, k0 + kp);
        CK(cudaEventSynchronize(S.copied[b]));                   // the upload of panel p - 2 has left the staging buffer
        dct_fill(kind, n, rows, nrows, k0, k1 - k0, S.h[b]);
        CK(cudaStreamWaitEvent(S.copy, S.consumed[b], 0));       // the product of panel p - 2 is done with the device buffer
        CK(cudaMemcpyAsync(S.d[b], S.h[b], (size_t)nrows * (k1 - k0) * 8, cudaMemcpyHostToDevice, S.copy));
        CK(cudaEventRecord(S.copied[b], S.copy));
        CK(cudaStreamWaitEvent(st, S.copied[b], 0));
        product((const double *)S.d[b], k1 - k0, rows != nullptr, k0, k1);
        CK(cudaEventRecord(S.consumed[b], st));
    }
    CK(cudaGetLastError());
    return S2PB_OK;
}

// rt = shift(img, 0) of the reference: see dct_kernels.cuh.  Asynchronous with resident tables; when no row needs it the
// kernels return at once.  A streamed table (rows wider than kDctDenseWidth) first waits for the row and column lists: with no
// listed row nothing is streamed, and the inverse streams the listed columns' rows of its table only.
// Y: [h][w] doubles of scratch.  rowlist: room for h + w ints and w bytes (row list, column list, column flags).
static int round_trip_zero(s2pb_ctx *ctx, Slot &s, const float *img, int w, int h, float *rt, RtState *state, int *rowlist, float *rowthr,
                           double *Y, cudaStream_t st)
{
    int *collist = rowlist + h;
    unsigned char *colflag = reinterpret_cast<unsigned char *>(collist + w);
    const s2pb_ctx::DctTab *t;
    int rc = dct_tables(ctx, w, false, &t);
    if (rc != S2PB_OK) return rc;
    CK(cudaMemsetAsync(state, 0, sizeof(RtState), st));
    CK(cudaMemsetAsync(colflag, 0, (size_t)w, st));
    launch(ctx, rt_flag_kernel, h, 256, 0, st, img, w, h, rt, state, rowlist, rowthr, colflag);
    launch(ctx, rt_collist_kernel, 1, 1024, 0, st, colflag, w, state, collist);
    RtState hs{};
    std::vector<int> cols;
    if (!t->T10 || !t->T01) {
        cols.resize(w);
        CK(cudaMemcpyAsync(&hs, state, sizeof hs, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(cols.data(), collist, (size_t)w * 4, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        if (hs.nrows == 0) return S2PB_OK;
    }
    const int g = ctx->sm_count * 4;
    rc = dct_product(s, st, t->T10, kDctT10, w, nullptr, w, [&](const double *P, int ldp, bool listed, int k0, int k1) {
        launch(ctx, dct_gemm_kernel<float, true, false>, g, kGemmThreads, 0, st, P, ldp, listed, k0, k1, img, w, h, state, rowlist, nullptr,
               Y, k0 == 0, k1 == w, Y, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
    });
    if (rc != S2PB_OK) return rc;
    if (!t->T01 && (rc = dct_stream_ensure(s, 0, (size_t)w * h)) != S2PB_OK) return rc;
    rc = dct_product(s, st, t->T01, kDctT01, w, cols.data(), hs.ncols, [&](const double *P, int ldp, bool listed, int k0, int k1) {
        launch(ctx, dct_gemm_kernel<double, false, true>, g, kGemmThreads, 0, st, P, ldp, listed, k0, k1, (const double *)Y, w, 0, state,
               rowlist, collist, s.dcts.acc, k0 == 0, k1 == w, nullptr, nullptr, nullptr, nullptr, rowthr, img, rt);
    });
    CK(cudaGetLastError());
    return rc;
}

// out = shift(img, 1/2) of the reference (SUBPIX = 2).  scratch: 4 x [h][w] doubles.
static int shift_half(s2pb_ctx *ctx, Slot &s, const float *img, int w, int h, float *out, double *scratch, cudaStream_t st)
{
    const s2pb_ctx::DctTab *t;
    int rc = dct_tables(ctx, w, true, &t);
    if (rc != S2PB_OK) return rc;
    const size_t npix = (size_t)w * h;
    double *ck = scratch, *sk = scratch + npix, *sym = scratch + 2 * npix, *anti = scratch + 3 * npix;
    const int g = ctx->sm_count * 4;
    rc = dct_product(s, st, t->T10, kDctT10, w, nullptr, w, [&](const double *P, int ldp, bool listed, int k0, int k1) {
        launch(ctx, dct_gemm_kernel<float, true, false>, g, kGemmThreads, 0, st, P, ldp, listed, k0, k1, img, w, h, nullptr, nullptr, nullptr,
               ck, k0 == 0, k1 == w, ck, (const double *)t->mc, (const double *)t->ms, sk, nullptr, nullptr, nullptr);
    });
    if (rc != S2PB_OK) return rc;
    const double *inv_tab[2] = {t->T01, t->TR01};
    const double *inv_in[2] = {ck, sk};
    double *inv_out[2] = {sym, anti};
    for (int i = 0; i < 2; i++) {
        rc = dct_product(s, st, inv_tab[i], i ? kDctTR01 : kDctT01, w, nullptr, w, [&](const double *P, int ldp, bool listed, int k0, int k1) {
            launch(ctx, dct_gemm_kernel<double, false, false>, g, kGemmThreads, 0, st, P, ldp, listed, k0, k1, inv_in[i], w, h, nullptr,
                   nullptr, nullptr, inv_out[i], k0 == 0, k1 == w, inv_out[i], nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
        });
        if (rc != S2PB_OK) return rc;
    }
    launch(ctx, dct_combine_kernel, (unsigned)((npix + 255) / 256), 256, 0, st, sym, anti, npix, out);
    CK(cudaGetLastError());
    return S2PB_OK;
}

// ------------------------------------------------------------------ mgm_call and mgm_multi (device level)

static int arena_reset(Slot &s, size_t need)
{
    if (need > s.arena_cap) {
        if (s.arena) { CK(cudaStreamSynchronize(s.stream)); CK(cudaFree(s.arena)); s.arena = nullptr; s.arena_cap = 0; }
        cudaError_t e = cudaMalloc((void **)&s.arena, need);
        if (e != cudaSuccess) { cudaGetLastError(); return fail(S2PB_ERR_NOMEM, "pyramid arena of %zu bytes: %s", need, cudaGetErrorString(e)); }
        s.arena_cap = need;
    }
    s.arena_off = 0;
    return S2PB_OK;
}
template <class T> static T *arena_take(Slot &s, size_t n)
{
    size_t o = s.arena_off;
    s.arena_off = align_up(o + n * sizeof(T), 256);
    return s.arena_off <= s.arena_cap ? (T *)(s.arena + o) : nullptr;
}

struct Level {
    int w, h;
    float *u, *v;                          // NaN-free images
    float *dminL, *dmaxL, *dminR, *dmaxR;  // per-pixel disparity bounds (pixels, float)
    float *dl, *dr, *conf;                 // results of this level's mgm_call
    float *wl = nullptr, *wr = nullptr;    // regularity weights of this level (-wl / -wr), or none
};

static GaussTaps gauss_taps(float sigma)
{   // mgm_multiscale.cc:66-71
    GaussTaps T;
    for (int j = 0; j < 10; j++)
        for (int i = 0; i < 10; i++) {
            float a = i - 4 - .5, b = j - 4 - .5;
            double sq = a * a + b * b;
            T.g[i + j * 10] = (float)exp(-sq / (2.0 * sigma * sigma));
        }
    return T;
}

// remove_small_cc on a device image (in -> out), scratch: two int images; thr: the intensity threshold of a link
int launch_remove_small_cc(s2pb_ctx *ctx, const float *in, float *out, int w, int h, int minarea, float thr, int *lab, int *area,
                           cudaStream_t st)
{
    int n = w * h;
    dim3 b2(32, 8);
    launch(ctx, cc_init_kernel, (n + 255) / 256, 256, 0, st, in, n, lab, area);
    launch(ctx, cc_rows_kernel, (h + 3) / 4, 128, 0, st, in, w, h, thr, lab);                 // one warp per row
    launch(ctx, cc_link_kernel, grid2d(w, h, b2), b2, 0, st, in, w, h, thr, lab);
    launch(ctx, cc_flatten_kernel, (n + 255) / 256, 256, 0, st, n, lab);
    launch(ctx, cc_area_kernel, (n + 255) / 256, 256, 0, st, n, lab, area);
    launch(ctx, cc_filter_kernel, (n + 255) / 256, 256, 0, st, in, n, lab, area, minarea, out);
    CK(cudaGetLastError());
    return S2PB_OK;
}
// its union-find passes over n labels, for the 3D filter and sgbm
void cc_flatten(s2pb_ctx *ctx, int n, int *lab, cudaStream_t st)
{
    launch(ctx, cc_flatten_kernel, (unsigned)(((size_t)n + 255) / 256), 256, 0, st, n, lab);
}
void cc_area(s2pb_ctx *ctx, int n, const int *lab, int *area, cudaStream_t st)
{
    launch(ctx, cc_area_kernel, (unsigned)(((size_t)n + 255) / 256), 256, 0, st, n, lab, area);
}

// S2PB_TRACE=1: synchronise and report after every stage of mgm_call; 2: report only (debugging aid)
static int trace_mode() { static int t = -1; if (t < 0) { const char *e = getenv("S2PB_TRACE"); t = e ? atoi(e) : 0; } return t; }
#define TRACE(st, ...) do { if (trace_mode()) { cudaError_t e_ = trace_mode() == 1 ? cudaStreamSynchronize(st) : cudaSuccess; \
    fprintf(stderr, "[s2pb] " __VA_ARGS__); fprintf(stderr, " -> %s\n", cudaGetErrorString(e_)); fflush(stderr); } } while (0)

// the float-cost flavour: a distance other than census, or the regularity weights of both views (-wl / -wr)
static bool general_flavour(const s2pb_mgm_params *p, const float *const wgt[2])
{
    return p->cost != S2PB_COST_CENSUS || (wgt[0] && wgt[1]);
}

// One mgm_call (mgm_multiscale.cc:161-335) on the workspace of c's slot, which slot_ensure has sized for the wider slab, on c's
// stream; the PKR images go to c.pkr.
//   img:   the NaN-free images; lo / hi: each view's per-pixel label range; gminv: the label of each view's slot 0
//   LPLv:  labels per lane of each view's slab (wide_slab: the chunk-skipping kernels)
//   zoom:  ZOOMFACTOR, 1 or 2 (labels of half pixels: SUBPIX = 2); wgt: the views' weight images, or none
//   outL / outR: the destinations of the left-right check; outR == nullptr: the right map is not wanted, it goes to a free
//   scratch image of the slot, returned in outR
//   timed (single scale): record s.ev[1..4] after the stages (s2pb_last_timings), and size the aggregation's grid by
//   whether another slot's aggregation is in flight (other_aggregation_pending reads those events)
// Enqueues only: no host synchronisation (except S2PB_TRACE=1).
static int mgm_call(s2pb_ctx *ctx, const MatchCall &c, int w, int h, const float *const img[2], short *const lo[2],
                    short *const hi[2], const int gminv[2], const int LPLv[2], int zoom, const float *const wgt[2],
                    const s2pb_mgm_params *p, float *outL, float *&outR, bool timed)
{
    Slot &s = c.s; const cudaStream_t st = c.st;
    const bool general = general_flavour(p, wgt);
    const bool census = p->cost == S2PB_COST_CENSUS, ncc = p->cost == S2PB_COST_NCC;
    const size_t npix = (size_t)w * h;
    dim3 b2(32, 8);
    int rc;
    // codes of more than 64 bits (census_words): the second words of each view's two codes go to the head of the view's last pass
    // volume (resident) or of its S (folded), 16 bytes a pixel of a region of at least 128 that the aggregation writes only
    // after the cost stage has read them
    const bool wide = census && census_words(p->census_win) == 2;
    uint64_t *hi_words[2] = {nullptr, nullptr};
    if (wide)
        for (int vi = 0; vi < 2; vi++) hi_words[vi] = (uint64_t *)(s.folded ? s.v[vi].S : s.v[vi].L[p->ndir - 1]);
    // ---- census of both images and of the copies the other view matches against
    for (int vi = 0; vi < 2; vi++) {
        ViewWS &v = s.v[vi];
        v.lo = lo[vi]; v.hi = hi[vi];
        // v.rt = shift(img[vi], 0): the reference's DCT round trip (mgm_costvolume.cc:50-60)
        rc = round_trip_zero(ctx, s, img[vi], w, h, v.rt, v.rtstate, v.rowlist, v.rowthr, s.Ydct, st);
        if (rc != S2PB_OK) return rc;
        if (census && wide)
            launch(ctx, census_pair_kernel<2>, grid2d(w, h, b2), b2, 0, st, img[vi], v.rt, v.rtstate, w, h, p->census_win / 2, v.census,
                   v.census_rt, hi_words[vi], hi_words[vi] + npix);
        else if (census)
            launch(ctx, census_pair_kernel<1>, grid2d(w, h, b2), b2, 0, st, img[vi], v.rt, v.rtstate, w, h, p->census_win / 2, v.census,
                   v.census_rt, nullptr, nullptr);
        if (ncc) {     // window statistics in the (then unused) census buffers: 8 B / pixel
            launch(ctx, ncc_stats_kernel, grid2d(w, h, b2), b2, 0, st, img[vi], w, h, p->census_win / 2, (float2 *)v.census);
            launch(ctx, ncc_stats_kernel, grid2d(w, h, b2), b2, 0, st, v.rt, w, h, p->census_win / 2, (float2 *)v.census_rt);
        }
    }
    // ZOOMFACTOR 2: shf[vi] = shift(img[vi], 1/2) (kept for the image-domain distances) and its census, in the pyramid arena
    // (mgm_multi_enqueue sizes it for two full-size mgm_calls: the half-pixel pass, second words included, takes less than one)
    float *shf[2] = {nullptr, nullptr};
    uint64_t *cen_half[2] = {nullptr, nullptr}, *cen_half_hi[2] = {nullptr, nullptr};
    if (zoom == 2) {
        for (int vi = 0; vi < 2; vi++) {
            shf[vi] = arena_take<float>(s, npix); cen_half[vi] = arena_take<uint64_t>(s, npix);
            if (wide) cen_half_hi[vi] = arena_take<uint64_t>(s, npix);
        }
        double *scratch = arena_take<double>(s, npix * 4);
        if (!scratch) return fail(S2PB_ERR_NOMEM, "pyramid arena exhausted");
        for (int vi = 0; vi < 2; vi++) {
            rc = shift_half(ctx, s, img[vi], w, h, shf[vi], scratch, st);
            if (rc != S2PB_OK) return rc;
            if (census && wide) launch(ctx, census_kernel<2>, grid2d(w, h, b2), b2, 0, st, shf[vi], w, h, p->census_win / 2, cen_half[vi], cen_half_hi[vi]);
            else if (census) launch(ctx, census_kernel<1>, grid2d(w, h, b2), b2, 0, st, shf[vi], w, h, p->census_win / 2, cen_half[vi], nullptr);
            if (ncc) launch(ctx, ncc_stats_kernel, grid2d(w, h, b2), b2, 0, st, shf[vi], w, h, p->census_win / 2, (float2 *)cen_half[vi]);
        }
    }
    // the round trips are done with Ydct, whose head the cost table takes (slot_layout)
    float lut_h[kCostLut];
    const float *lut = nullptr;
    if (cost_lut(p->census_win, lut_h) || general) { CK(cudaMemcpyAsync(s.lut, lut_h, sizeof lut_h, cudaMemcpyHostToDevice, st)); lut = s.lut; }
    CK(cudaGetLastError());
    if (timed) CK(cudaEventRecord(s.ev[1], st));
    // ---- cost volumes: view 0 = left reference, view 1 = right reference (mgm_multiscale.cc:222,270)
    for (int vi = 0; vi < 2; vi++) {
        const ViewWS &v = s.v[vi], &o = s.v[1 - vi];
        CostGenParams G;
        memset(&G, 0, sizeof G);
        G.u = img[vi]; G.v0 = o.rt; G.v1 = shf[1 - vi];
        G.cu = v.census; G.cv0 = o.census_rt; G.cv1 = cen_half[1 - vi];
        if (wide) { G.cuh = hi_words[vi]; G.cv0h = hi_words[1 - vi] + npix; G.cv1h = cen_half_hi[1 - vi]; }
        G.su = (const float2 *)G.cu; G.sv0 = (const float2 *)G.cv0; G.sv1 = (const float2 *)G.cv1;
        G.lut = s.lut; G.lo = lo[vi]; G.hi = hi[vi];
        G.w = w; G.h = h; G.gmin = gminv[vi]; G.cost = p->cost; G.win = p->census_win; G.zoom = zoom;
        G.C = (float *)v.C;
        rc = launch_cost(ctx, LPLv[vi], general, G, st);
        if (rc != S2PB_OK) return rc;
    }
    if (timed) CK(cudaEventRecord(s.ev[2], st));
    TRACE(st, "  census + cost");
    // ---- 8-pass MGM of both views (mgm_multiscale.cc:194-202: P1 / ZOOMFACTOR) in one launch_aggregate, or two when the views'
    // slabs differ in width; in the folded layout (slot_ensure) each is a launch per pass
    const float P1 = p->P1 / (float)zoom;
    if (s.folded) ctx->folded_calls++;
    if (LPLv[0] == LPLv[1]) {
        // With another tile's aggregation queued or running (tiles in flight) the launch takes one CTA per SM instead of two, so
        // two tiles' aggregations share the SMs: a pass is a chain of bands, two CTAs per SM on 16 pass-views run it twice as
        // many bands deep as one CTA per SM does, and a good part of each launch is the chain filling and draining.  (This
        // policy was chosen by measurement on the GPU the engine was first written for and has not been re-measured on the H100.)
        rc = launch_aggregate(ctx, s, 2, w, h, LPLv[0], P1, p->P2, p->ndir, p->tsgm, lut, st, general, wgt, gminv, 0,
                              timed && other_aggregation_pending(ctx, s) ? 1 : 0);
    } else {
        // one launch per view, side by side: each takes one persistent CTA per SM (a chain of bands per pass limits what a single
        // view can keep busy: alone, 8 passes fill the GPU no better than 16 do), the right view on the slot's second stream
        CK(cudaEventRecord(s.fork, st));
        CK(cudaStreamWaitEvent(s.stream2, s.fork, 0));
        rc = launch_aggregate(ctx, s, 1, w, h, LPLv[0], P1, p->P2, p->ndir, p->tsgm, lut, st, general, wgt, gminv, 0, 1);
        if (rc == S2PB_OK) rc = launch_aggregate(ctx, s, 1, w, h, LPLv[1], P1, p->P2, p->ndir, p->tsgm, lut, s.stream2, general, wgt, gminv, 1, 1);
        CK(cudaEventRecord(s.join, s.stream2));
        CK(cudaStreamWaitEvent(st, s.join, 0));
    }
    if (rc != S2PB_OK) return rc;
    if (timed) CK(cudaEventRecord(s.ev[3], st));
    TRACE(st, "  aggregate");
    // ---- WTA + consensus + sub-pixel
    for (int vi = 0; vi < 2; vi++) {
        WtaParams W;
        fill_wta(W, s.v[vi], p->ndir, gminv[vi], p, lut, npix);
        W.inv_zoom_div = (float)zoom;
        W.pkr = c.pkr[vi];
        rc = launch_wta(ctx, s, vi, LPLv[vi], W, st, general);
        if (rc != S2PB_OK) return rc;
    }
    if (timed) CK(cudaEventRecord(s.ev[4], st));
    TRACE(st, "  wta");
    // ---- post filters (mgm_multiscale.cc:310-334)
    float *dl = s.v[0].disp, *dr = s.v[1].disp, *xl = s.v[0].tmp, *xr = s.v[1].tmp;
    if (p->median > 0) {
        launch(ctx, median_kernel, grid2d(w, h, b2), b2, 0, st, dl, xl, w, h, p->median);
        launch(ctx, median_kernel, grid2d(w, h, b2), b2, 0, st, dr, xr, w, h, p->median);
        float *t = dl; dl = xl; xl = t; t = dr; dr = xr; xr = t;
    }
    if (p->mindiff >= 0) {      // mgm_multiscale.cc:318-319: only the left map, against the right view's cost image
        launch(ctx, mindiff_kernel, grid2d(w, h, b2), b2, 0, st, dl, s.v[1].cost, xl, w, h, p->census_win, p->mindiff);
        float *t = dl; dl = xl; xl = t;
    }
    if (!outR) outR = xr;
    if (p->lr_mode == 1) {
        launch(ctx, lrcheck_kernel, grid2d(w, h, b2), b2, 0, st, dr, dl, outR, w, h, p->lr_tau);
        launch(ctx, lrcheck_kernel, grid2d(w, h, b2), b2, 0, st, dl, dr, outL, w, h, p->lr_tau);
    } else {
        CK(cudaMemcpyAsync(outL, dl, npix * 4, cudaMemcpyDeviceToDevice, st));
        CK(cudaMemcpyAsync(outR, dr, npix * 4, cudaMemcpyDeviceToDevice, st));
    }
    CK(cudaGetLastError());
    TRACE(st, "  median / lr");
    return S2PB_OK;
}

// One mgm_call of a pyramid level: the label ranges of both views from the level's bounds, one slab for both views
// sized by the wider hull, then the speckle filter (mgm_multiscale.cc:328-334).  Weighted by the level's weight maps when the
// call has weight images.
static int mgm_call_level(s2pb_ctx *ctx, const MatchCall &c, Level &L, int zoom, const s2pb_mgm_params *p)
{
    Slot &s = c.s; const cudaStream_t st = c.st;
    const bool weighted = c.wl && c.wr;
    const int w = L.w, h = L.h, n = w * h;
    const float *wgt[2] = {weighted ? L.wl : nullptr, weighted ? L.wr : nullptr};
    const bool general = general_flavour(p, wgt);
    const size_t npix = (size_t)n;
    // ---- integer label ranges of both views and their hulls (one host round trip: the layout depends on them)
    short *lo[2], *hi[2];
    for (int vi = 0; vi < 2; vi++) { lo[vi] = arena_take<short>(s, npix); hi[vi] = arena_take<short>(s, npix); }
    float *tl = arena_take<float>(s, npix), *tr = arena_take<float>(s, npix);
    int *lab = arena_take<int>(s, npix), *area = arena_take<int>(s, npix);
    if (!area) return fail(S2PB_ERR_NOMEM, "pyramid arena exhausted");
    // hull accumulators live in device memory (atomics on mapped host memory need PCIe atomics); copied back once
    int *d_hull = s.d_small;
    const int hull_init[4] = {0x7fffffff, (int)0x80000000, 0x7fffffff, (int)0x80000000};
    CK(cudaMemcpyAsync(d_hull, hull_init, sizeof hull_init, cudaMemcpyHostToDevice, st));
    launch(ctx, label_ranges_kernel, (n + 255) / 256, 256, 0, st, L.dminL, L.dmaxL, n, (float)zoom, lo[0], hi[0], d_hull);
    launch(ctx, label_ranges_kernel, (n + 255) / 256, 256, 0, st, L.dminR, L.dmaxR, n, (float)zoom, lo[1], hi[1], d_hull + 2);
    CK(cudaGetLastError());
    int hull[4];
    CK(cudaMemcpyAsync(hull, d_hull, sizeof hull, cudaMemcpyDeviceToHost, st));
    int rc = sync_or_timeout(c);
    if (rc != S2PB_OK) return rc;
    int gminv[2] = {hull[0], hull[2]}, gmaxv[2] = {hull[1], hull[3]};
    int D = 0;
    for (int vi = 0; vi < 2; vi++) {
        if (gminv[vi] < -16000 || gmaxv[vi] > 16000) return fail(S2PB_ERR_ARG, "label range out of the int16 domain");
        int d = gmaxv[vi] - gminv[vi] + 1; if (d > D) D = d;
    }
    int LPL;
    rc = slab_lpl(D, &LPL);
    if (rc != S2PB_OK) return rc;
    rc = slot_ensure(ctx, s, w, h, 32 * LPL, p->ndir, general ? 4 : 1);
    if (rc != S2PB_OK) return rc;
    TRACE(st, "level %dx%d zoom %d: hull L [%d,%d] R [%d,%d] -> LPL %d%s", w, h, zoom, gminv[0], gmaxv[0], gminv[1], gmaxv[1], LPL,
          general ? " (general flavour)" : "");
    const float *img[2] = {L.u, L.v};
    const int LPLv[2] = {LPL, LPL};
    const bool cc = p->remove_small_cc > 0;
    float *lrL = cc ? tl : L.dl, *lrR = cc ? tr : L.dr;
    rc = mgm_call(ctx, c, w, h, img, lo, hi, gminv, LPLv, zoom, wgt, p, lrL, lrR, false);
    if (rc != S2PB_OK) return rc;
    if (cc) {
        rc = launch_remove_small_cc(ctx, lrL, L.dl, w, h, p->remove_small_cc, 5.f, lab, area, st);   // mgm_multiscale.cc:332-333
        if (rc != S2PB_OK) return rc;
        rc = launch_remove_small_cc(ctx, lrR, L.dr, w, h, p->remove_small_cc, 5.f, lab, area, st);
        if (rc != S2PB_OK) return rc;
    }
    TRACE(st, "  remove_small_cc");
    CK(cudaMemcpyAsync(L.conf, s.v[0].conf, npix * 4, cudaMemcpyDeviceToDevice, st));
    CK(cudaGetLastError());
    return S2PB_OK;
}

// main() of mgm_multi (main_mgm_multi.cc:88-256) + recursive_multiscale (mgm_multiscale.cc:339-410)
static int mgm_multi_enqueue(s2pb_ctx *ctx, const MatchCall &call, const float *d_im1, const float *d_im2, int w, int h, int dmin,
                             int dmax, const s2pb_mgm_params *p, float *d_disp, float *d_conf, uint8_t *d_mask, float *d_dispR)
{
    Slot &s = call.s; const cudaStream_t st = call.st;
    const int n = w * h;
    dim3 b2(32, 8);
    const bool weighted = call.wl && call.wr;
    // pyramid shape: downsample while max > 100, min > 50 and scale < -S (mgm_multiscale.cc:362)
    std::vector<Level> lv(1);
    lv[0].w = w; lv[0].h = h;
    while ((int)lv.size() - 1 < p->scales) {
        const Level &c = lv.back();
        if (!((c.w > c.h ? c.w : c.h) > 100 && (c.w < c.h ? c.w : c.h) > 50)) break;
        Level nx; nx.w = (c.w + 1) / 2; nx.h = (c.h + 1) / 2;
        lv.push_back(nx);
    }
    size_t need = 0;
    for (auto &L : lv) need += (size_t)L.w * L.h * 4 * 11 + 11 * 256;
    need += (size_t)n * (4 * 12 + 2 * 4 + 8 * 2 + 4 * 2 + 8 * 4) * 2 + (1 << 20);     // scratch of the mgm_calls (two at full size)
    int rc = arena_reset(s, need);
    if (rc != S2PB_OK) return rc;
    for (auto &L : lv) {
        size_t m = (size_t)L.w * L.h;
        L.u = arena_take<float>(s, m); L.v = arena_take<float>(s, m);
        L.dminL = arena_take<float>(s, m); L.dmaxL = arena_take<float>(s, m);
        L.dminR = arena_take<float>(s, m); L.dmaxR = arena_take<float>(s, m);
        L.dl = arena_take<float>(s, m); L.dr = arena_take<float>(s, m); L.conf = arena_take<float>(s, m);
        if (!L.conf) return fail(S2PB_ERR_NOMEM, "pyramid arena exhausted");
        if (weighted) {
            L.wl = arena_take<float>(s, m); L.wr = arena_take<float>(s, m);
            if (!L.wr) return fail(S2PB_ERR_NOMEM, "pyramid arena exhausted");
        }
    }
    if (weighted) {
        CK(cudaMemcpyAsync(lv[0].wl, call.wl, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
        CK(cudaMemcpyAsync(lv[0].wr, call.wr, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
    }
    s.timed = false;
    // level 0: NaN -> 0, initial bounds (main_mgm_multi.cc:160-196; the sentinel for no-data is dmin in both views)
    launch(ctx, init_ranges_kernel, (n + 255) / 256, 256, 0, st, d_im1, n, (float)dmin, (float)dmax, (float)dmin, lv[0].u, lv[0].dminL, lv[0].dmaxL);
    launch(ctx, init_ranges_kernel, (n + 255) / 256, 256, 0, st, d_im2, n, (float)-dmax, (float)-dmin, (float)dmin, lv[0].v, lv[0].dminR, lv[0].dmaxR);
    const GaussTaps T = gauss_taps(0.8f);
    for (size_t l = 0; l + 1 < lv.size(); l++) {
        Level &a = lv[l], &b = lv[l + 1];
        dim3 g = grid2d(b.w, b.h, b2);
        launch(ctx, downsample2x_kernel, g, b2, 0, st, a.u, a.w, a.h, T, b.u, b.w, b.h);
        launch(ctx, downsample2x_kernel, g, b2, 0, st, a.v, a.w, a.h, T, b.v, b.w, b.h);
        if (weighted) {                        // the weight maps follow the pyramid, mgm_multiscale.cc:375-378
            launch(ctx, downsample2x_kernel, g, b2, 0, st, a.wl, a.w, a.h, T, b.wl, b.w, b.h);
            launch(ctx, downsample2x_kernel, g, b2, 0, st, a.wr, a.w, a.h, T, b.wr, b.w, b.h);
        }
        launch(ctx, downsample2x_disp_kernel, g, b2, 0, st, a.dminL, a.w, a.h, 0, b.dminL, b.w, b.h);
        launch(ctx, downsample2x_disp_kernel, g, b2, 0, st, a.dmaxL, a.w, a.h, 1, b.dmaxL, b.w, b.h);
        launch(ctx, downsample2x_disp_kernel, g, b2, 0, st, a.dminR, a.w, a.h, 0, b.dminR, b.w, b.h);
        launch(ctx, downsample2x_disp_kernel, g, b2, 0, st, a.dmaxR, a.w, a.h, 1, b.dmaxR, b.w, b.h);
    }
    CK(cudaGetLastError());
    const size_t arena_mark = s.arena_off;
    for (int l = (int)lv.size() - 1; l >= 0; l--) {
        Level &L = lv[l];
        if (l + 1 < (int)lv.size()) {          // upsample2x_disp (mgm_multiscale.cc:36-48): slack 8, radius 4, then zoom_nn x2
            Level &c = lv[l + 1];
            s.arena_off = arena_mark;
            size_t m = (size_t)c.w * c.h;
            float *omin = arena_take<float>(s, m), *omax = arena_take<float>(s, m);
            const float *disp2[2] = {c.dl, c.dr};
            float *fmin[2] = {L.dminL, L.dminR}, *fmax[2] = {L.dmaxL, L.dmaxR};
            for (int vi = 0; vi < 2; vi++) {
                launch(ctx, update_ranges_kernel, grid2d(c.w, c.h, b2), b2, 0, st, disp2[vi], 2.f, c.w, c.h, nullptr, nullptr, fmin[vi], fmax[vi],
                                                                       L.w, L.h, 8.f, 4, omin, omax);
                launch(ctx, zoom2_kernel, grid2d(L.w, L.h, b2), b2, 0, st, omin, c.w, fmin[vi], L.w, L.h);
                launch(ctx, zoom2_kernel, grid2d(L.w, L.h, b2), b2, 0, st, omax, c.w, fmax[vi], L.w, L.h);
            }
            CK(cudaGetLastError());
        }
        s.arena_off = arena_mark;
        rc = mgm_call_level(ctx, call, L, 1, p);
        if (rc != S2PB_OK) return rc;
    }
    Level &L0 = lv[0];
    if (d_conf) CK(cudaMemcpyAsync(d_conf, L0.conf, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));   // the ZOOM=1 call's consensus
    if (p->subpix > 1) {                       // main_mgm_multi.cc:203-209: bounds = result +-2 over 9x9, labels = half pixels
        s.arena_off = arena_mark;
        float *a = arena_take<float>(s, n), *b = arena_take<float>(s, n), *c = arena_take<float>(s, n), *d = arena_take<float>(s, n);
        const size_t mark2 = s.arena_off;
        launch(ctx, update_ranges_kernel, grid2d(w, h, b2), b2, 0, st, L0.dl, 1.f, w, h, L0.dminL, L0.dmaxL, L0.dminL, L0.dmaxL, w, h, 2.f, 4, a, b);
        launch(ctx, update_ranges_kernel, grid2d(w, h, b2), b2, 0, st, L0.dr, 1.f, w, h, L0.dminR, L0.dmaxR, L0.dminR, L0.dmaxR, w, h, 2.f, 4, c, d);
        L0.dminL = a; L0.dmaxL = b; L0.dminR = c; L0.dmaxR = d;
        s.arena_off = mark2;
        MatchCall half = call;        // fresh `param` without the weight images (main_mgm_multi.cc:207), and with its own img_dict:
        half.wl = half.wr = nullptr; half.pkr[0] = half.pkr[1] = nullptr;     // the PKR images written are the ZOOM = 1 call's
        rc = mgm_call_level(ctx, half, L0, p->subpix, p);
        if (rc != S2PB_OK) return rc;
    }
    float *outL = d_disp;
    if (p->lr_mode == 2) {                     // main_mgm_multi.cc:212-217
        s.arena_off = arena_mark;
        float *tr = arena_take<float>(s, n);
        launch(ctx, lrcheck_kernel, grid2d(w, h, b2), b2, 0, st, L0.dr, L0.dl, tr, w, h, p->lr_tau);
        launch(ctx, lrcheck_kernel, grid2d(w, h, b2), b2, 0, st, L0.dl, L0.dr, outL, w, h, p->lr_tau);
        if (d_dispR) CK(cudaMemcpyAsync(d_dispR, tr, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
    } else {
        CK(cudaMemcpyAsync(outL, L0.dl, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
        if (d_dispR) CK(cudaMemcpyAsync(d_dispR, L0.dr, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
    }
    launch(ctx, nan_restore_kernel, (n + 255) / 256, 256, 0, st, outL, d_im1, n);
    if (d_dispR) launch(ctx, nan_restore_kernel, (n + 255) / 256, 256, 0, st, d_dispR, d_im2, n);
    if (d_mask) launch_rejection_mask(ctx, outL, d_im1, d_im2, w, h, d_mask, st);
    CK(cudaGetLastError());
    return S2PB_OK;
}

// ------------------------------------------------------------------ the matcher (device level)

static int mgm_enqueue(s2pb_ctx *ctx, const MatchCall &c, const float *d_im1, const float *d_im2, int w, int h, int dmin, int dmax,
                       const s2pb_mgm_params *p, float *d_disp, float *d_conf, uint8_t *d_mask, float *d_dispR, int nodata_hint)
{
    if (p->scales >= 0) return mgm_multi_enqueue(ctx, c, d_im1, d_im2, w, h, dmin, dmax, p, d_disp, d_conf, d_mask, d_dispR);
    Slot &s = c.s; const cudaStream_t st = c.st;
    const float *wgt[2] = {c.wl, c.wr};
    const bool general = general_flavour(p, wgt);
    const size_t npix = (size_t)w * h;
    const int n = (int)npix;
    if (nodata_hint < 0) {     // unknown: look (costs one stream synchronisation)
        int *flag = s.d_small + 16;      // this slot's own word (several slots may ask at once)
        CK(cudaMemsetAsync(flag, 0, 4, st));
        launch(ctx, has_nan_kernel, ctx->sm_count * 4, 256, 0, st, d_im2, n, flag);
        int hflag = 0;
        CK(cudaMemcpyAsync(&hflag, flag, 4, cudaMemcpyDeviceToHost, st));
        int rs = sync_or_timeout(c);
        if (rs != S2PB_OK) return rs;
        nodata_hint = hflag ? 3 : 0;
    }
    // each view's slab is sized on its own: a no-data pixel in the secondary image widens only the right view's hull (by one
    // label when |dmin| > dmax), and each view's kernels run at that view's own width -- the volumes are [H][W][32 LPL_view]
    // inside buffers sized for the wider view
    int gminv[2], gmaxv[2], LPLv[2], rc;
    plan_labels(dmin, dmax, (nodata_hint & 2) != 0, gminv, gmaxv);
    for (int vi = 0; vi < 2; vi++)
        if ((rc = slab_lpl(gmaxv[vi] - gminv[vi] + 1, &LPLv[vi])) != S2PB_OK) return rc;
    const int LPL = LPLv[0] > LPLv[1] ? LPLv[0] : LPLv[1];
    rc = slot_ensure(ctx, s, w, h, 32 * LPL, p->ndir, general ? 4 : 1);
    if (rc != S2PB_OK) return rc;
    const float *im[2] = {d_im1, d_im2};
    s.timed = true;
    CK(cudaEventRecord(s.ev[0], st));
    // ---- NaN-free copies of both images and their label ranges
    for (int vi = 0; vi < 2; vi++) {
        int lo_all = vi == 0 ? dmin : -dmax, hi_all = vi == 0 ? dmax : -dmin;
        launch(ctx, prepare_view_kernel, (n + 255) / 256, 256, 0, st, im[vi], n, lo_all, hi_all, dmin, s.v[vi].img, s.v[vi].lo, s.v[vi].hi);
    }
    const float *img[2] = {s.v[0].img, s.v[1].img};
    short *lo[2] = {s.v[0].lo, s.v[1].lo}, *hi[2] = {s.v[0].hi, s.v[1].hi};
    float *outL = d_disp, *outR = d_dispR;
    rc = mgm_call(ctx, c, w, h, img, lo, hi, gminv, LPLv, 1, wgt, p, outL, outR, true);
    if (rc != S2PB_OK) return rc;
    // ---- no-data restore (main_mgm.cc:231-236), mask
    launch(ctx, nan_restore_kernel, (n + 255) / 256, 256, 0, st, outL, d_im1, n);
    launch(ctx, nan_restore_kernel, (n + 255) / 256, 256, 0, st, outR, d_im2, n);
    if (d_conf) CK(cudaMemcpyAsync(d_conf, s.v[0].conf, npix * 4, cudaMemcpyDeviceToDevice, st));
    if (d_mask) launch_rejection_mask(ctx, outL, d_im1, d_im2, w, h, d_mask, st);
    CK(cudaGetLastError());
    CK(cudaEventRecord(s.ev[5], st));
    return S2PB_OK;
}

extern "C" int s2pb_mgm_device(s2pb_ctx *ctx, int slot, const float *d_im1, const float *d_im2, int w, int h, int dmin, int dmax,
                               const s2pb_mgm_params *p, float *d_disp, float *d_conf, uint8_t *d_mask, float *d_disp_right,
                               int nodata_hint, void *stream)
{
    if (!ctx || !d_im1 || !d_im2 || !d_disp) return fail(S2PB_ERR_ARG, "null argument");
    int rc = check_params(p, w, h, dmin, dmax);
    if (rc != S2PB_OK) return rc;
    CK(cudaSetDevice(ctx->device));
    if (slot < 0) return fail(S2PB_ERR_ARG, "negative slot");
    rc = ensure_slots(ctx, slot + 1);
    if (rc != S2PB_OK) return rc;
    Slot &s = ctx->slots[slot];
    const MatchCall c{s, stream ? (cudaStream_t)stream : s.stream, deadline_after(p->timeout_ms)};
    rc = mgm_enqueue(ctx, c, d_im1, d_im2, w, h, dmin, dmax, p, d_disp, d_conf, d_mask, d_disp_right, nodata_hint);
    if (rc != S2PB_OK) return rc;
    if (c.deadline) return sync_or_timeout(c);
    return S2PB_OK;
}

// true when `p` is page-locked host memory known to CUDA (cudaHostAlloc / cudaHostRegister, e.g. a torch pinned
// tensor): such buffers are used for the DMA directly instead of being staged through the slot's pinned block
static bool is_pinned_host(const void *p)
{
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost;
}

// stage the inputs of one tile through pinned memory and enqueue everything on the stream of c, the slot's own; wl / wr: host
// weight images, both or neither
static int mgm_host_enqueue(s2pb_ctx *ctx, const MatchCall &c, const float *im1, const float *im2, int w, int h, int dmin,
                            int dmax, const s2pb_mgm_params *p, bool want_mask, bool want_right, float *o_disp, float *o_conf,
                            uint8_t *o_mask, const float *wl = nullptr, const float *wr = nullptr)
{
    Slot &s = c.s;
    size_t npix = (size_t)w * h;
    int rc = slot_host_ensure(s, npix);
    if (rc != S2PB_OK) return rc;
    // copy into the pinned staging block (unless the caller's buffers are page-locked already), noticing no-data
    // pixels of the secondary image on the way
    const float *src1 = im1, *src2 = im2;
    if (!is_pinned_host(im1)) { memcpy(s.h_in[0], im1, npix * 4); src1 = s.h_in[0]; }
    bool sec_nodata = false;
    {
        const bool pinned2 = is_pinned_host(im2);
        float *dst = s.h_in[1];
        unsigned acc = 0;
        if (pinned2) { for (size_t i = 0; i < npix; i++) { float v = im2[i]; acc |= (unsigned)(v != v); } }
        else { for (size_t i = 0; i < npix; i++) { float v = im2[i]; dst[i] = v; acc |= (unsigned)(v != v); } src2 = dst; }
        sec_nodata = acc != 0;
    }
    rc = slot_io_ensure(s, npix);
    if (rc != S2PB_OK) return rc;
    CK(cudaMemcpyAsync(s.d_in[0], src1, npix * 4, cudaMemcpyHostToDevice, s.stream));
    CK(cudaMemcpyAsync(s.d_in[1], src2, npix * 4, cudaMemcpyHostToDevice, s.stream));
    MatchCall cw = c;
    if (wl && wr) {        // not a hot path: plain (driver-staged) copies of the caller's weight images
        CK(cudaMemcpyAsync(s.d_w[0], wl, npix * 4, cudaMemcpyHostToDevice, s.stream));
        CK(cudaMemcpyAsync(s.d_w[1], wr, npix * 4, cudaMemcpyHostToDevice, s.stream));
        cw.wl = s.d_w[0]; cw.wr = s.d_w[1];
    }
    rc = mgm_enqueue(ctx, cw, s.d_in[0], s.d_in[1], w, h, dmin, dmax, p, s.d_disp, s.d_conf, want_mask ? s.d_mask : nullptr,
                     want_right ? s.d_dispR : nullptr, sec_nodata ? 2 : 0);
    if (rc != S2PB_OK) return rc;
    // results go straight into the caller's buffers when those are page-locked (o_* != nullptr), else to the staging block
    s.direct_out = o_disp && o_conf && is_pinned_host(o_disp) && is_pinned_host(o_conf) && (!want_mask || (o_mask && is_pinned_host(o_mask)));
    CK(cudaMemcpyAsync(s.direct_out ? o_disp : s.h_disp, s.d_disp, npix * 4, cudaMemcpyDeviceToHost, s.stream));
    CK(cudaMemcpyAsync(s.direct_out ? o_conf : s.h_conf, s.d_conf, npix * 4, cudaMemcpyDeviceToHost, s.stream));
    if (want_mask) CK(cudaMemcpyAsync(s.direct_out ? o_mask : s.h_mask, s.d_mask, npix, cudaMemcpyDeviceToHost, s.stream));
    if (want_right) CK(cudaMemcpyAsync(s.h_dispR, s.d_dispR, npix * 4, cudaMemcpyDeviceToHost, s.stream));
    CK(cudaEventRecord(s.done, s.stream));
    return S2PB_OK;
}

// after the slot's stream has finished: the results of mgm_host_enqueue that went to the staging block, into the caller's buffers
static void copy_staged_outputs(const Slot &s, size_t npix, float *disp, float *conf, uint8_t *mask)
{
    if (s.direct_out) return;
    memcpy(disp, s.h_disp, npix * 4);
    memcpy(conf, s.h_conf, npix * 4);
    if (mask) memcpy(mask, s.h_mask, npix);
}

// s2pb_mgm, s2pb_mgm_weighted and s2pb_mgm_pkr: one tile from host buffers on slot 0.  wl / wr: host weight images or null;
// pkr_left / pkr_right: host destinations of the PKR images, or null.
static int mgm_host(s2pb_ctx *ctx, const float *im1, const float *im2, int w, int h, int dmin, int dmax, const s2pb_mgm_params *p,
                    const float *wl, const float *wr, float *disp, float *conf, uint8_t *mask, float *disp_right, float *pkr_left,
                    float *pkr_right)
{
    if (!ctx || !im1 || !im2 || !disp || !conf) return fail(S2PB_ERR_ARG, "null argument");
    if ((wl == nullptr) != (wr == nullptr)) return fail(S2PB_ERR_ARG, "the weight images come in pairs (-wl and -wr)");
    int rc = check_params(p, w, h, dmin, dmax);
    if (rc != S2PB_OK) return rc;
    const size_t npix = (size_t)w * h;
    // the lease holds the device PKR images, and waits for slot 0's stream on every return: after an error nothing may still
    // DMA into the caller's buffers
    HostCall L(ctx, "the PKR images");
    Slot &s = ctx->slots[0];
    MatchCall c{s, s.stream, deadline_after(p->timeout_ms)};
    if (pkr_left) { c.pkr[0] = L.take<float>(npix * 4); c.pkr[1] = L.take<float>(npix * 4); }
    if ((rc = L.error()) != S2PB_OK) return rc;
    rc = mgm_host_enqueue(ctx, c, im1, im2, w, h, dmin, dmax, p, mask != nullptr, disp_right != nullptr, disp, conf, mask, wl, wr);
    if (rc == S2PB_OK) rc = sync_or_timeout(c);
    if (rc != S2PB_OK) return rc;
    copy_staged_outputs(s, npix, disp, conf, mask);
    if (disp_right) memcpy(disp_right, s.h_dispR, npix * 4);
    if (pkr_left) { L.download(pkr_left, c.pkr[0], npix * 4); L.download(pkr_right, c.pkr[1], npix * 4); }
    return L.finish();
}

extern "C" int s2pb_mgm(s2pb_ctx *ctx, const float *im1, const float *im2, int w, int h, int dmin, int dmax,
                        const s2pb_mgm_params *p, float *disp, float *conf, uint8_t *mask, float *disp_right)
{
    return mgm_host(ctx, im1, im2, w, h, dmin, dmax, p, nullptr, nullptr, disp, conf, mask, disp_right, nullptr, nullptr);
}

extern "C" int s2pb_mgm_weighted(s2pb_ctx *ctx, const float *im1, const float *im2, int w, int h, int dmin, int dmax,
                                 const s2pb_mgm_params *p, const float *wl, const float *wr,
                                 float *disp, float *conf, uint8_t *mask, float *disp_right)
{
    return mgm_host(ctx, im1, im2, w, h, dmin, dmax, p, wl, wr, disp, conf, mask, disp_right, nullptr, nullptr);
}

// `mgm ... -confidence_pkrL f -confidence_pkrR g` (main_mgm.cc:147,250-262; mgm_multi likewise): s2pb_mgm plus the peak-ratio
// confidence images of both views.  s2p never asks for them (s2p/block_matching.py:167-183); the matcher's option surface does.
extern "C" int s2pb_mgm_pkr(s2pb_ctx *ctx, const float *im1, const float *im2, int w, int h, int dmin, int dmax,
                            const s2pb_mgm_params *p, float *disp, float *conf, uint8_t *mask, float *disp_right,
                            float *pkr_left, float *pkr_right)
{
    if (!pkr_left || !pkr_right) return fail(S2PB_ERR_ARG, "null argument");
    return mgm_host(ctx, im1, im2, w, h, dmin, dmax, p, nullptr, nullptr, disp, conf, mask, disp_right, pkr_left, pkr_right);
}

extern "C" int s2pb_reserve(s2pb_ctx *ctx, int nslots, int w, int h, int nlabels)
{
    if (!ctx || nslots < 1) return fail(S2PB_ERR_ARG, "bad argument");
    CK(cudaSetDevice(ctx->device));
    int LPL;
    int rc = slab_lpl(nlabels, &LPL);
    if (rc != S2PB_OK) return rc;
    rc = ensure_slots(ctx, nslots);
    if (rc != S2PB_OK) return rc;
    for (int i = 0; i < nslots; i++) {
        rc = slot_ensure(ctx, ctx->slots[i], w, h, 32 * LPL, 8);
        if (rc != S2PB_OK) return rc;
        rc = slot_host_ensure(ctx->slots[i], (size_t)w * h);
        if (rc != S2PB_OK) return rc;
        rc = slot_io_ensure(ctx->slots[i], (size_t)w * h);
        if (rc != S2PB_OK) return rc;
    }
    return S2PB_OK;
}

extern "C" int s2pb_mgm_batch(s2pb_ctx *ctx, int n, const float *const *im1, const float *const *im2, int w, int h, int dmin,
                              int dmax, const s2pb_mgm_params *p, float *const *disp, float *const *conf, uint8_t *const *mask)
{
    if (!ctx || n < 0 || !im1 || !im2 || !disp || !conf) return fail(S2PB_ERR_ARG, "null argument");
    int rc = check_params(p, w, h, dmin, dmax);
    if (rc != S2PB_OK) return rc;
    CK(cudaSetDevice(ctx->device));
    const int ns = (int)ctx->slots.size();
    const size_t npix = (size_t)w * h;
    const Deadline deadline = deadline_after(p->timeout_ms * (long long)(n > 0 ? n : 1));   // the per-tile timeout times the number of tiles
    auto call = [&](int si) { Slot &s = ctx->slots[si]; return MatchCall{s, s.stream, deadline}; };
    if (p->scales >= 0 && ns > 1 && n > 1) {
        // mgm_multi reads a label hull back at every pyramid level, so a tile's enqueue blocks its host thread: one thread per
        // workspace keeps several tiles in flight (their kernels overlap on the device, each on its slot's stream)
        const int T = (ns < n ? ns : n) < 4 ? (ns < n ? ns : n) : 4;     // (a C3-sized tile holds 13 GiB of volumes at its widest level)
        std::vector<int> codes(T, S2PB_OK);
        std::vector<std::string> errs(T);
        std::atomic<bool> stop{false};
        std::vector<std::thread> th;
        for (int k = 0; k < T; k++)
            th.emplace_back([&, k]() {
                cudaSetDevice(ctx->device);
                const MatchCall c = call(k);
                for (int t = k; t < n && !stop.load(); t += T) {
                    int r = mgm_host_enqueue(ctx, c, im1[t], im2[t], w, h, dmin, dmax, p, mask && mask[t], false, disp[t], conf[t],
                                             mask ? mask[t] : nullptr);
                    if (r == S2PB_OK) r = sync_or_timeout(c);
                    if (r != S2PB_OK) { codes[k] = r; errs[k] = g_err; stop.store(true); break; }
                    copy_staged_outputs(c.s, npix, disp[t], conf[t], mask ? mask[t] : nullptr);
                }
            });
        for (auto &t : th) t.join();
        for (int k = 0; k < T; k++)
            if (codes[k] != S2PB_OK) { drain_all(ctx); g_err = errs[k]; return codes[k]; }
        return S2PB_OK;
    }
    std::vector<int> inflight(ns, -1);
    auto collect = [&](int si) -> int {
        int t = inflight[si];
        if (t < 0) return S2PB_OK;
        int r = sync_or_timeout(call(si));
        if (r != S2PB_OK) return r;
        copy_staged_outputs(ctx->slots[si], npix, disp[t], conf[t], mask ? mask[t] : nullptr);
        inflight[si] = -1;
        return S2PB_OK;
    };
    // on any error the other slots still have kernels and copies in flight, some of them into the caller's page-locked
    // buffers: stop and wait for all of them before returning (the caller may free its arrays right away)
    auto bail = [&](int code) -> int { std::string keep = g_err; drain_all(ctx); g_err = keep; return code; };
    for (int t = 0; t < n; t++) {
        int si = t % ns;
        rc = collect(si);
        if (rc != S2PB_OK) return bail(rc);
        rc = mgm_host_enqueue(ctx, call(si), im1[t], im2[t], w, h, dmin, dmax, p, mask && mask[t], false, disp[t], conf[t],
                              mask ? mask[t] : nullptr);
        if (rc != S2PB_OK) return bail(rc);
        inflight[si] = t;
    }
    for (int k = 0; k < ns; k++) {
        rc = collect((n + k) % ns);
        if (rc != S2PB_OK) return bail(rc);
    }
    return S2PB_OK;
}

extern "C" int s2pb_last_timings(s2pb_ctx *ctx, int slot, float ms[S2PB_T_COUNT])
{
    if (!ctx || slot < 0 || slot >= (int)ctx->slots.size() || !ms) return fail(S2PB_ERR_ARG, "bad argument");
    Slot &s = ctx->slots[slot];
    if (!s.timed) return fail(S2PB_ERR_ARG, "no timed call on this slot yet");
    CK(cudaSetDevice(ctx->device));
    CK(cudaEventSynchronize(s.ev[5]));
    for (int i = 0; i < 5; i++) CK(cudaEventElapsedTime(&ms[i], s.ev[i], s.ev[i + 1]));
    CK(cudaEventElapsedTime(&ms[S2PB_T_TOTAL], s.ev[0], s.ev[5]));
    return S2PB_OK;
}

// ------------------------------------------------------------------ stage-level entry points (host buffers)

// the stage entry points take the matched image as the caller has it and apply the reference's round trip themselves
// (allocate_and_fill_sgm_costvolume does, mgm_costvolume.cc:94): *rt = shift(dv, 0)
static int stage_round_trip(s2pb_ctx *ctx, ScratchLease &L, const float *dv, int w, int h, cudaStream_t st, float **rt)
{
    size_t npix = (size_t)w * h;
    // aux: row list [h] + column list [w] + column flags [w bytes], then the per-row thresholds [h], then the state
    const size_t lists = ((size_t)h + w) * 4 + ((size_t)w + 15) / 16 * 16;
    float *out = L.take<float>(npix * 4);
    char *aux = L.take<char>(lists + (size_t)h * 4 + 256);
    double *Y = L.take<double>(npix * 8);
    if (!out || !aux || !Y) return L.nomem("the round trip");
    int rc = round_trip_zero(ctx, ctx->slots[0], dv, w, h, out, (RtState *)(aux + lists + (size_t)h * 4), (int *)aux, (float *)(aux + lists), Y, st);
    if (rc != S2PB_OK) return rc;
    *rt = out;
    return S2PB_OK;
}

extern "C" int s2pb_census(s2pb_ctx *ctx, const float *img, int w, int h, int win, uint64_t *codes)
{
    if (!ctx || !img || !codes || w < 1 || h < 1) return fail(S2PB_ERR_ARG, "bad argument");
    if (win != 3 && win != 5 && win != 7) return fail(S2PB_ERR_ARG, "census window must be 3, 5 or 7");
    size_t npix = (size_t)w * h;
    HostCall L(ctx, "the census");
    float *a = L.upload(img, npix * 4);
    uint64_t *b = L.take<uint64_t>(npix * 8);
    if (int rc = L.error()) return rc;
    dim3 b2(32, 8);
    launch(ctx, census_kernel<1>, grid2d(w, h, b2), b2, 0, L.st, a, w, h, win / 2, b, nullptr);
    CK(cudaGetLastError());
    L.download(codes, b, npix * 8);
    return L.finish();
}

// the int16 label ranges of a host-buffer call, uploaded through its protocol: the caller checks L.error() after this
static int upload_ranges(HostCall &L, const int32_t *lo, const int32_t *hi, size_t npix, int gmin, int D, short **dlo, short **dhi)
{
    std::vector<short> a(npix), b(npix);
    for (size_t i = 0; i < npix; i++) {
        if (lo[i] < gmin || hi[i] > gmin + D - 1 || lo[i] > hi[i]) return fail(S2PB_ERR_ARG, "range of pixel %zu outside the volume", i);
        a[i] = (short)lo[i]; b[i] = (short)hi[i];
    }
    *dlo = L.upload(a.data(), npix * 2);
    *dhi = L.upload(b.data(), npix * 2);
    CK(cudaStreamSynchronize(L.st));         // a and b go on return
    return S2PB_OK;
}

// The [h][w][D] cost volume of u against the round trip of v: through the 8-bit census codes of the hot matcher (codes, with
// cost = census), or through the general path's `cost` (S2PB_COST_*).
static int stage_costvolume(s2pb_ctx *ctx, const float *u, const float *v, int w, int h, const int32_t *lo, const int32_t *hi,
                            int gmin, int D, int win, int cost, bool codes, float *C)
{
    if (!ctx || !u || !v || !lo || !hi || !C || w < 1 || h < 1 || D < 1) return fail(S2PB_ERR_ARG, "bad argument");
    int rc = census_win_ok(win);
    if (rc != S2PB_OK) return rc;
    if (cost < 0 || cost >= S2PB_COST_COUNT) return fail(S2PB_ERR_ARG, "cost must be one of S2PB_COST_*");
    int LPL;
    rc = slab_lpl(D, &LPL);               // the stage entry points run the register-resident kernels only
    if (rc == S2PB_OK && wide_slab(LPL)) rc = fail(S2PB_ERR_UNSUPPORTED, "the stage entry points take at most 512 labels, not %d", D);
    if (rc != S2PB_OK) return rc;
    const int DP = 32 * LPL;
    size_t npix = (size_t)w * h, tot = npix * D;
    float lut_h[kCostLut];
    const bool scaled = cost_lut(win, lut_h);
    const bool wide = cost == S2PB_COST_CENSUS && census_words(win) == 2;
    HostCall L(ctx, "the cost volume");
    float *du = L.upload(u, npix * 4), *dv = L.upload(v, npix * 4);
    // census codes (their second words after the first npix when wide) or NCC window statistics
    uint64_t *cu = L.take<uint64_t>(npix * 8 * (wide ? 2 : 1)), *cv = L.take<uint64_t>(npix * 8 * (wide ? 2 : 1));
    void *dC = L.take<void>(npix * DP * (codes ? 1 : 4));
    float *dCf = L.take<float>(tot * 4), *dlut = L.upload(lut_h, sizeof lut_h);
    short *dlo, *dhi;
    rc = upload_ranges(L, lo, hi, npix, gmin, D, &dlo, &dhi);
    if (rc == S2PB_OK) rc = L.error();
    if (rc != S2PB_OK) return rc;
    float *rt = nullptr;
    rc = stage_round_trip(ctx, L, dv, w, h, L.st, &rt);
    if (rc != S2PB_OK) return rc;
    dim3 b2(32, 8);
    if (wide) {
        launch(ctx, census_kernel<2>, grid2d(w, h, b2), b2, 0, L.st, du, w, h, win / 2, cu, cu + npix);
        launch(ctx, census_kernel<2>, grid2d(w, h, b2), b2, 0, L.st, rt, w, h, win / 2, cv, cv + npix);
    } else if (cost == S2PB_COST_CENSUS) {
        launch(ctx, census_kernel<1>, grid2d(w, h, b2), b2, 0, L.st, du, w, h, win / 2, cu, nullptr);
        launch(ctx, census_kernel<1>, grid2d(w, h, b2), b2, 0, L.st, rt, w, h, win / 2, cv, nullptr);
    }
    if (cost == S2PB_COST_NCC) {
        launch(ctx, ncc_stats_kernel, grid2d(w, h, b2), b2, 0, L.st, du, w, h, win / 2, (float2 *)cu);
        launch(ctx, ncc_stats_kernel, grid2d(w, h, b2), b2, 0, L.st, rt, w, h, win / 2, (float2 *)cv);
    }
    CostGenParams G;
    memset(&G, 0, sizeof G);
    G.u = du; G.v0 = rt; G.cu = cu; G.cv0 = cv;
    if (wide) { G.cuh = cu + npix; G.cv0h = cv + npix; }
    G.su = (float2 *)cu; G.sv0 = (float2 *)cv;
    G.lut = dlut; G.lo = dlo; G.hi = dhi;
    G.w = w; G.h = h; G.gmin = gmin; G.cost = cost; G.win = win; G.zoom = 1; G.C = (float *)dC;
    rc = launch_cost(ctx, LPL, !codes, G, L.st);
    if (rc != S2PB_OK) return rc;
    if (codes) launch(ctx, unpack_cost_kernel, (unsigned)((tot + 255) / 256), 256, 0, L.st, (uint8_t *)dC, npix, D, DP, scaled ? dlut : nullptr, dCf);
    else launch(ctx, unpad_cost_kernel, (unsigned)((tot + 255) / 256), 256, 0, L.st, (float *)dC, npix, D, DP, dCf);
    CK(cudaGetLastError());
    L.download(C, dCf, tot * 4);
    return L.finish();
}

extern "C" int s2pb_costvolume(s2pb_ctx *ctx, const float *u, const float *v, int w, int h, const int32_t *lo, const int32_t *hi,
                               int gmin, int D, int win, float *C)
{
    return stage_costvolume(ctx, u, v, w, h, lo, hi, gmin, D, win, S2PB_COST_CENSUS, true, C);
}

extern "C" int s2pb_costvolume_dist(s2pb_ctx *ctx, const float *u, const float *v, int w, int h, const int32_t *lo, const int32_t *hi,
                                    int gmin, int D, int win, int cost, float *C)
{
    return stage_costvolume(ctx, u, v, w, h, lo, hi, gmin, D, win, cost, false, C);
}

// Aggregation and WTA of the host cost volume C [h][w][D]: with 8-bit cost codes in the slab, or in the float-cost flavour
// (general) with an optional weight image.
static int stage_aggregate(s2pb_ctx *ctx, const float *C, const int32_t *lo, const int32_t *hi, int w, int h, int gmin, int D,
                           float P1, float P2, int ndir, int tsgm, int fix_overcount, bool general, const float *weights,
                           float *S, float *disp, float *cost, float *conf)
{
    if (!ctx || !C || !lo || !hi || !disp || w < 2 || h < 2 || D < 1) return fail(S2PB_ERR_ARG, "bad argument");
    if (ndir != 2 && ndir != 4 && ndir != 8) return fail(S2PB_ERR_ARG, "ndir must be 2, 4 or 8");
    if (tsgm < 1 || tsgm > 4) return fail(S2PB_ERR_ARG, "tsgm must be 1..4");
    int LPL, rc = slab_lpl(D, &LPL);      // the stage entry points run the register-resident kernels only
    if (rc == S2PB_OK && wide_slab(LPL)) rc = fail(S2PB_ERR_UNSUPPORTED, "the stage entry points take at most 512 labels, not %d", D);
    if (rc != S2PB_OK) return rc;
    const int DP = 32 * LPL;
    size_t npix = (size_t)w * h, tot = npix * D;
    if (!general) {
        // the device slab stores 8-bit cost codes (agg_kernel.cuh): integers up to kCostMaxCode.  Larger integer costs take the
        // float-cost flavour, which with unit weights computes the same values.
        for (size_t i = 0; i < tot; i++) {
            float c = C[i];
            if (!(c == INFINITY || (c >= 0.f && c <= 2048.f && c == floorf(c))))
                return fail(S2PB_ERR_UNSUPPORTED, "cost %g at %zu is not an integer in [0,2048] or +inf", c, i);
            if (c > (float)kCostMaxCode && c != INFINITY) general = true;
        }
    }
    HostCall L(ctx, "the aggregation");
    float *dCf = L.upload(C, tot * 4);
    float *dS = S ? L.take<float>(tot * 4) : nullptr;
    float *dW = weights ? L.upload(weights, npix * 4) : nullptr;
    short *dlo, *dhi;
    rc = upload_ranges(L, lo, hi, npix, gmin, D, &dlo, &dhi);
    if (rc == S2PB_OK) rc = L.error();
    if (rc != S2PB_OK) return rc;
    Slot &s = ctx->slots[0];          // the workspace of slot 0 holds the slab
    rc = slot_ensure(ctx, s, w, h, DP, ndir, general ? 4 : 1, false);
    if (rc != S2PB_OK) return rc;
    size_t totp = npix * DP;
    if (general) launch(ctx, pad_cost_kernel, (unsigned)((totp + 255) / 256), 256, 0, L.st, dCf, npix, D, DP, (float *)s.v[0].C);
    else launch(ctx, pack_cost_kernel, (unsigned)((totp + 255) / 256), 256, 0, L.st, dCf, npix, D, DP, (uint8_t *)s.v[0].C);
    CK(cudaGetLastError());
    const float *wgt[2] = {dW, nullptr};
    rc = launch_aggregate(ctx, s, 1, w, h, LPL, P1, P2, ndir, tsgm, nullptr, L.st, general, wgt);
    if (rc != S2PB_OK) return rc;
    s2pb_mgm_params prm;
    s2pb_default_params("mgm", &prm);
    prm.fix_overcount = fix_overcount; prm.refine = 0;
    WtaParams W;
    fill_wta(W, s.v[0], ndir, gmin, &prm, nullptr, npix);
    W.lo = dlo; W.hi = dhi;
    W.S = dS; W.Dout = D;
    rc = launch_wta(ctx, s, 0, LPL, W, L.st, general);
    if (rc != S2PB_OK) return rc;
    L.download(disp, s.v[0].disp, npix * 4);
    if (cost) L.download(cost, s.v[0].cost, npix * 4);
    if (conf) L.download(conf, s.v[0].conf, npix * 4);
    if (S) L.download(S, dS, tot * 4);
    return L.finish();
}

extern "C" int s2pb_aggregate_w(s2pb_ctx *ctx, const float *C, const int32_t *lo, const int32_t *hi, int w, int h, int gmin, int D,
                                float P1, float P2, int ndir, int tsgm, int fix_overcount, const float *weights,
                                float *S, float *disp, float *cost, float *conf)
{
    return stage_aggregate(ctx, C, lo, hi, w, h, gmin, D, P1, P2, ndir, tsgm, fix_overcount, true, weights, S, disp, cost, conf);
}

extern "C" int s2pb_aggregate(s2pb_ctx *ctx, const float *C, const int32_t *lo, const int32_t *hi, int w, int h, int gmin, int D,
                              float P1, float P2, int ndir, int tsgm, int fix_overcount, float *S, float *disp, float *cost, float *conf)
{
    return stage_aggregate(ctx, C, lo, hi, w, h, gmin, D, P1, P2, ndir, tsgm, fix_overcount, false, nullptr, S, disp, cost, conf);
}

extern "C" int s2pb_median(s2pb_ctx *ctx, const float *in, float *out, int w, int h, int radius)
{
    if (!ctx || !in || !out || w < 1 || h < 1 || radius < 0 || radius > 2) return fail(S2PB_ERR_ARG, "bad argument");
    size_t npix = (size_t)w * h;
    HostCall L(ctx, "the median");
    float *a = L.upload(in, npix * 4), *b = L.take<float>(npix * 4);
    if (int rc = L.error()) return rc;
    dim3 b2(32, 8);
    launch(ctx, median_kernel, grid2d(w, h, b2), b2, 0, L.st, a, b, w, h, radius);
    CK(cudaGetLastError());
    L.download(out, b, npix * 4);
    return L.finish();
}

extern "C" int s2pb_remove_small_cc(s2pb_ctx *ctx, const float *in, float *out, int w, int h, int minarea)
{
    if (!ctx || !in || !out || w < 2 || h < 2) return fail(S2PB_ERR_ARG, "bad argument");
    size_t npix = (size_t)w * h;
    HostCall L(ctx, "remove_small_cc");
    float *a = L.upload(in, npix * 4), *b = L.take<float>(npix * 4);
    int *lab = L.take<int>(npix * 4), *area = L.take<int>(npix * 4);
    if (int rc = L.error()) return rc;
    int rc = launch_remove_small_cc(ctx, a, b, w, h, minarea, 5.f, lab, area, L.st);
    if (rc != S2PB_OK) return rc;
    L.download(out, b, npix * 4);
    return L.finish();
}

int erode_radius_ok(float radius)
{
    if (!(radius > 1.f) || radius > 64.f) return fail(S2PB_ERR_ARG, "disk radius must be in (1, 64]");   // build_disk, c/morsi.c:282
    return S2PB_OK;
}

void launch_erode_mask(s2pb_ctx *ctx, const uint8_t *in, uint8_t *out, int w, int h, float radius, cudaStream_t st)
{
    dim3 b2(32, 8);
    launch(ctx, erode_mask_kernel, grid2d(w, h, b2), b2, 0, st, in, out, w, h, radius);
}

extern "C" int s2pb_erode_mask(s2pb_ctx *ctx, const uint8_t *in, uint8_t *out, int w, int h, float radius)
{
    if (!ctx || !in || !out || w < 1 || h < 1) return fail(S2PB_ERR_ARG, "bad argument");
    if (int rc = erode_radius_ok(radius)) return rc;
    size_t npix = (size_t)w * h;
    HostCall L(ctx, "the mask erosion");
    uint8_t *a = L.upload(in, npix), *b = L.take<uint8_t>(npix);
    if (int rc = L.error()) return rc;
    launch_erode_mask(ctx, a, b, w, h, radius, L.st);
    CK(cudaGetLastError());
    L.download(out, b, npix);
    return L.finish();
}

// create_rejection_mask (s2p/block_matching.py:18-32) of a device disparity map
void launch_rejection_mask(s2pb_ctx *ctx, const float *disp, const float *im1, const float *im2, int w, int h, uint8_t *mask,
                           cudaStream_t st)
{
    dim3 b2(32, 8);
    launch(ctx, rejection_mask_kernel, grid2d(w, h, b2), b2, 0, st, disp, im1, im2, w, h, mask);
}

extern "C" int s2pb_rejection_mask(s2pb_ctx *ctx, const float *disp, const float *im1, const float *im2, int w, int h, uint8_t *mask)
{
    if (!ctx || !disp || !im1 || !im2 || !mask || w < 1 || h < 1) return fail(S2PB_ERR_ARG, "bad argument");
    size_t npix = (size_t)w * h;
    HostCall L(ctx, "the rejection mask");
    float *a = L.upload(disp, npix * 4), *b = L.upload(im1, npix * 4), *c = L.upload(im2, npix * 4);
    uint8_t *m = L.take<uint8_t>(npix);
    if (int rc = L.error()) return rc;
    launch_rejection_mask(ctx, a, b, c, w, h, m, L.st);
    CK(cudaGetLastError());
    L.download(mask, m, npix);
    return L.finish();
}

// ------------------------------------------------------------------ the matcher of pair_tile.cu

// The matcher of s2pb_mgm_weighted between device buffers on slot 0 (st is that slot's stream, as HostCall's): the deadline counts
// from here, and the call waits for the stream through the timeout.
int mgm_match_device(s2pb_ctx *ctx, cudaStream_t st, const float *d_im1, const float *d_im2, int w, int h, int dmin, int dmax,
                     const s2pb_mgm_params *p, const float *d_wl, const float *d_wr, float *d_disp, float *d_conf, uint8_t *d_mask,
                     float *d_dispR)
{
    if (int rc = check_params(p, w, h, dmin, dmax)) return rc;
    const MatchCall c{ctx->slots[0], st, deadline_after(p->timeout_ms), d_wl, d_wr};
    int rc = mgm_enqueue(ctx, c, d_im1, d_im2, w, h, dmin, dmax, p, d_disp, d_conf, d_mask, d_dispR, -1);
    if (rc != S2PB_OK) return rc;
    return sync_or_timeout(c);
}
