// s2pb200.cu -- context, workspace and the C ABI declared in include/s2pb200.h.
//
// Host-side orchestration of the kernels in mgm_kernels.cuh.  The sequence of stages mirrors
// what one `mgm` process does for one tile (main_mgm.cc:167-262 -> mgm_call,
// mgm_multiscale.cc:161-335 in the reference) followed by create_rejection_mask
// (s2p/block_matching.py:18-32).  There is no CPU fallback in this file.
#include "../../include/s2pb200.h"
#include "mgm_kernels.cuh"
#include "multiscale_kernels.cuh"
#include "dct_kernels.cuh"
#include "homography_kernels.cuh"
#include "fusion_kernels.cuh"
#include "triangulation_kernels.cuh"
#include "pointcloud_kernels.cuh"
#include "sgbm_kernels.cuh"
#include "agg_dispatch.h"
#include "agg_chunked.cuh"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <list>
#include <mutex>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <string>
#include <thread>
#include <vector>

using namespace s2pb;

// ------------------------------------------------------------------ errors

static thread_local std::string g_err;
static int fail(int code, const char *fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}
#define CK(call)                                                                                     \
    do {                                                                                             \
        cudaError_t e_ = (call);                                                                     \
        if (e_ != cudaSuccess)                                                                       \
            return fail(S2PB_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

// ------------------------------------------------------------------ context

struct ViewWS {
    float *img;            // NaN-free copy
    float *rt;             // ... after the reference's DCT round trip (what the OTHER view's cost volume matches against)
    uint64_t *census_rt;   // census (or NCC window statistics) of rt
    int *rowlist;          // rows the round trip had to transform
    float *rowthr;         // per row: pixels with |x| <= rowthr are recomputed (-1: none)
    RtState *rtstate;
    short *lo, *hi;        // per-pixel label range
    uint64_t *census;
    void *C;               // [H][W][DP] costs: u8 codes (census popcounts, agg_kernel.cuh) or float (general flavour)
    float *L[kMaxPasses];
    float *Lmin[kMaxPasses];
    int *progress;         // [kMaxPasses][maxBands]
    float *disp, *cost, *conf, *tmp;
};
struct Slot {
    void *base = nullptr;
    size_t bytes = 0;
    int w = 0, h = 0, DP = 0, ndir = 0;
    int cbytes = 1;               // bytes per stored cost: 1 = 8-bit census codes, 4 = float (general flavour)
    ViewWS v[2];
    int *next_item = nullptr;
    float *lut = nullptr;
    double *Ydct = nullptr;       // [H][W] DCT coefficients of the rows in flight (dct_kernels.cuh)
    // staging for the host-buffer API
    float *d_in[2] = {nullptr, nullptr};
    float *d_w[2] = {nullptr, nullptr};           // -wl / -wr weight images of s2pb_mgm_weighted
    float *d_disp = nullptr, *d_conf = nullptr, *d_dispR = nullptr;
    uint8_t *d_mask = nullptr;
    char *io_base = nullptr;
    size_t io_pix = 0;
    float *h_in[2] = {nullptr, nullptr};          // pinned
    float *h_disp = nullptr, *h_conf = nullptr, *h_dispR = nullptr;
    uint8_t *h_mask = nullptr;
    size_t h_pix = 0;
    // bump arena for the pyramid of mgm_multi (images, range images, per-level results)
    char *arena = nullptr;
    size_t arena_cap = 0, arena_off = 0;
    int *d_small = nullptr;           // 64 words of device memory of this slot's own (hull accumulators of mgm_multi)
    cudaStream_t stream = nullptr;
    cudaStream_t stream2 = nullptr;   // the right view's aggregation when the two views' slabs differ in width (runs beside the left one)
    cudaEvent_t fork = nullptr, join = nullptr;
    cudaEvent_t ev[S2PB_T_COUNT + 1] = {};
    cudaEvent_t done = nullptr;
    bool timed = false;
    bool direct_out = false;      // the last host-API call wrote its results straight into the caller's pinned buffers
};
struct s2pb_ctx {
    int device = 0;
    int sm_count = 132;
    std::vector<Slot> slots;
    int *abort_flag = nullptr;     // pinned + mapped: the host raises it on timeout
    int *scratch_flag = nullptr;   // pinned + mapped: device -> host one-word answers
    int *d_scratch = nullptr;      // 64 words of device memory (hull accumulators of mgm_multi)
    std::atomic<long long> launches{0};   // (mgm_multi tiles of a batch are enqueued from several host threads)
    // destination of the PKR images of s2pb_mgm_pkr (device, per view), or null: every mgm_call writes them, the last one stays
    float *pkr_dst[2] = {nullptr, nullptr};
    // deadline of the matcher call in flight (timeout_ms counted from the API entry; has_deadline = false: none)
    std::chrono::steady_clock::time_point deadline;
    bool has_deadline = false;
    // DCT coefficient tables of the matched image's round trip, one entry per image width (dct_tables)
    struct DctTab { int n; double *T10, *T01, *TR01, *mc, *ms; };
    std::list<DctTab> dct;          // a list: entries stay put while other host threads hold pointers to them
    std::mutex dct_mu;
    // scratch pool of the host-buffer entry points: device buffers are kept between calls (a cudaMalloc / cudaFree pair per
    // call costs more than the merge or the warp itself).  Borrowed through a ScratchLease only.  It has no lock, so nothing
    // that s2pb_mgm_batch's worker threads run may take from it.
    struct PoolBuf { void *p; size_t bytes; bool used; };
    std::vector<PoolBuf> pool;
};

static size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// smallest idle pooled buffer that is large enough, else a new allocation; when that fails the idle buffers are given back
// to the device and the allocation is tried once more (nullptr when out of memory)
static void *pool_take(s2pb_ctx *ctx, size_t bytes)
{
    int best = -1;
    for (int i = 0; i < (int)ctx->pool.size(); i++)
        if (!ctx->pool[i].used && ctx->pool[i].bytes >= bytes && (best < 0 || ctx->pool[i].bytes < ctx->pool[best].bytes)) best = i;
    if (best >= 0) { ctx->pool[best].used = true; return ctx->pool[best].p; }
    void *p = nullptr;
    size_t want = align_up(bytes ? bytes : 1, (size_t)1 << 20);
    if (cudaMalloc(&p, want) != cudaSuccess) {
        cudaGetLastError();
        // an idle buffer is safe to free: the lease that held it waited for its stream before handing it back
        std::vector<s2pb_ctx::PoolBuf> held;
        for (auto &b : ctx->pool) if (b.used) held.push_back(b); else cudaFree(b.p);
        ctx->pool.swap(held);
        if (cudaMalloc(&p, want) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    }
    ctx->pool.push_back({p, want, true});
    return p;
}

// The device scratch of one host-buffer call, borrowed from the pool.  `st` is the stream the call runs on.  The destructor
// waits for that stream, then hands back only the buffers this lease took, on every return path: after any return no kernel
// or copy still touches the scratch or the caller's buffers, and leases nest.  Success paths still end in a checked
// cudaStreamSynchronize of their own, which is where an asynchronous error is reported.
class ScratchLease {
public:
    ScratchLease(s2pb_ctx *ctx, cudaStream_t st) : ctx_(ctx), st_(st) {}
    ScratchLease(const ScratchLease &) = delete;
    ScratchLease &operator=(const ScratchLease &) = delete;
    ~ScratchLease()
    {
        cudaStreamSynchronize(st_);
        for (auto &b : ctx_->pool)
            if (std::find(taken_.begin(), taken_.end(), b.p) != taken_.end()) b.used = false;
    }
    // nullptr when the device is out of memory; the caller then returns nomem()
    template <class T> T *take(size_t bytes)
    {
        void *p = pool_take(ctx_, bytes);
        if (p) taken_.push_back(p);
        else if (!failed_) failed_ = bytes ? bytes : 1;
        return (T *)p;
    }
    int nomem(const char *what) const { return fail(S2PB_ERR_NOMEM, "cudaMalloc of %zu bytes failed for %s", failed_, what); }

private:
    s2pb_ctx *ctx_;
    cudaStream_t st_;
    std::vector<void *> taken_;
    size_t failed_ = 0;       // size of the first request that failed
};

static int lpl_for(int D)
{
    static const int opts[] = {1, 2, 3, 4, 5, 6, 8, 12, 16};
    for (int o : opts) if (32 * o >= D) return o;
    return -1;
}
// stride of the per-pass progress counters: bands hold kNW scanlines in the register-resident kernel, but as few as 2 in the
// chunk-skipping kernel on float-cost slabs wider than 1024 slots (agg_chunked.cuh, ck_warps)
static int max_bands(int w, int h) { return ((w > h ? w : h) + 1) / 2; }

static int slot_layout(Slot &s, int w, int h, int DP, int ndir, int cbytes, bool allocate)
{
    // carve one allocation; called first with allocate=false to size it
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
        for (int p = 0; p < ndir; p++) {
            o = take(npix * DP * 4); if (allocate) v.L[p] = (float *)(b + o);
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

static int slot_ensure(s2pb_ctx *ctx, Slot &s, int w, int h, int DP, int ndir, int cbytes = 1)
{
    Slot probe;
    slot_layout(probe, w, h, DP, ndir, cbytes, false);
    if (!s.base || probe.bytes > s.bytes) {
        if (s.base) { CK(cudaStreamSynchronize(s.stream)); CK(cudaFree(s.base)); s.base = nullptr; }
        cudaError_t e = cudaMalloc(&s.base, probe.bytes);
        if (e != cudaSuccess) {
            cudaGetLastError();
            s.base = nullptr; s.bytes = 0;
            return fail(S2PB_ERR_NOMEM, "workspace of %.2f GiB for a %dx%dx%d tile does not fit: %s",
                        probe.bytes / 1073741824.0, w, h, DP, cudaGetErrorString(e));
        }
        s.bytes = probe.bytes;
    }
    s.w = w; s.h = h; s.DP = DP; s.ndir = ndir; s.cbytes = cbytes;
    size_t keep = s.bytes;
    slot_layout(s, w, h, DP, ndir, cbytes, true);
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
    if (cudaHostAlloc((void **)&ctx->abort_flag, 16 * sizeof(int), cudaHostAllocMapped) != cudaSuccess) {
        fail(S2PB_ERR_CUDA, "cudaHostAlloc failed"); delete ctx; return nullptr;
    }
    ctx->scratch_flag = ctx->abort_flag + 8;
    for (int i = 0; i < 16; i++) ctx->abort_flag[i] = 0;
    if (cudaMalloc((void **)&ctx->d_scratch, 256) != cudaSuccess) { fail(S2PB_ERR_CUDA, "cudaMalloc failed"); delete ctx; return nullptr; }
    ctx->slots.reserve(64);
    ctx->slots.resize(1);
    if (slot_init(ctx, ctx->slots[0]) != S2PB_OK) { delete ctx; return nullptr; }
    // function attributes are per device: every context sets them for its own (not once per process)
    if (agg_configure() != 0 || agg_chunked_configure() != 0 ||
        cudaFuncSetAttribute(wta_chunked_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * 2048 * 4) != cudaSuccess ||
        cudaFuncSetAttribute(wta_chunked_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * 2048 * 4) != cudaSuccess) {
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
    if (ctx->abort_flag) cudaFreeHost(ctx->abort_flag);
    if (ctx->d_scratch) cudaFree(ctx->d_scratch);
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

// ------------------------------------------------------------------ timeouts

// The timeout contract (timeout_ms -> S2PB_ERR_TIMEOUT -> subprocess.TimeoutExpired upstream) counts from the API
// entry: every host-side wait of a matcher call goes through sync_or_timeout, also the per-level read-backs of mgm_multi.
static void set_deadline(s2pb_ctx *ctx, long long timeout_ms)
{
    ctx->has_deadline = timeout_ms > 0;
    if (ctx->has_deadline) ctx->deadline = std::chrono::steady_clock::now() + std::chrono::milliseconds(timeout_ms);
}
// stop everything that is in flight on any slot: raise the abort flag (the persistent aggregation kernels drain), wait
// for every slot stream -- some of them DMA into the caller's buffers -- then clear the flag
static void drain_all(s2pb_ctx *ctx, bool abort)
{
    if (abort) *(volatile int *)ctx->abort_flag = 1;
    for (auto &s : ctx->slots) if (s.stream) cudaStreamSynchronize(s.stream);
    if (abort) *(volatile int *)ctx->abort_flag = 0;
}
static int sync_or_timeout(s2pb_ctx *ctx, cudaStream_t st)
{
    if (!ctx->has_deadline) { CK(cudaStreamSynchronize(st)); return S2PB_OK; }
    for (;;) {
        cudaError_t e = cudaStreamQuery(st);
        if (e == cudaSuccess) return S2PB_OK;
        if (e != cudaErrorNotReady) return fail(S2PB_ERR_CUDA, "stream failed: %s", cudaGetErrorString(e));
        if (std::chrono::steady_clock::now() > ctx->deadline) {
            drain_all(ctx, true);
            cudaStreamSynchronize(st);
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

static dim3 grid2d(int w, int h, dim3 b) { return dim3((w + b.x - 1) / b.x, (h + b.y - 1) / b.y); }

static int check_params(const s2pb_mgm_params *p, int w, int h, int dmin, int dmax)
{
    if (!p) return fail(S2PB_ERR_ARG, "null params");
    if (w < 2 || h < 2) return fail(S2PB_ERR_ARG, "image too small (%dx%d)", w, h);
    if (dmax <= dmin) return fail(S2PB_ERR_ARG, "need dmin < dmax (got %d, %d)", dmin, dmax);
    if (p->ndir != 2 && p->ndir != 4 && p->ndir != 8) return fail(S2PB_ERR_ARG, "ndir must be 2, 4 or 8");
    if (p->tsgm < 1 || p->tsgm > 4) return fail(S2PB_ERR_ARG, "tsgm must be 1..4");
    if (p->census_win != 3 && p->census_win != 5 && p->census_win != 7) return fail(S2PB_ERR_ARG, "census_win must be 3, 5 or 7");
    if (p->median < 0 || p->median > 2) return fail(S2PB_ERR_ARG, "median radius must be 0..2");
    if (p->refine < 0 || p->refine > 2) return fail(S2PB_ERR_ARG, "refine must be 0 (none), 1 (vfit) or 2 (parabola)");
    if (p->subpix != 1 && p->subpix != 2) return fail(S2PB_ERR_UNSUPPORTED, "SUBPIX must be 1 or 2");
    if (p->scales < 0 && p->subpix != 1) return fail(S2PB_ERR_ARG, "SUBPIX=2 only exists in mgm_multi (scales >= 0)");
    if (p->scales < 0 && p->remove_small_cc > 0) return fail(S2PB_ERR_UNSUPPORTED, "REMOVESMALLCC is only wired into the mgm_multi path");
    if (p->lr_mode < 0 || p->lr_mode > 2) return fail(S2PB_ERR_ARG, "TESTLRRL must be 0, 1 or 2");
    if (p->scales < 0 && p->lr_mode == 2) return fail(S2PB_ERR_ARG, "TESTLRRL=2 only exists in mgm_multi");
    if (p->scales >= 0 && w > 4000) return fail(S2PB_ERR_UNSUPPORTED, "mgm_multi tiles wider than 4000 px are not supported");
    if (abs(dmin) > 16000 || abs(dmax) > 16000) return fail(S2PB_ERR_ARG, "disparity bounds out of the int16 label range");
    if (p->cost < 0 || p->cost >= S2PB_COST_COUNT) return fail(S2PB_ERR_ARG, "cost must be one of S2PB_COST_* (got %d)", p->cost);
    return S2PB_OK;
}

// cost LUT for scaled census costs: cost(r) = (float)((double)r * ratio / nch), mgm_costvolume.h:90-91
static bool cost_lut(int win, float lut[64])
{
    int nbits = win * win - 1, nch = (nbits / 8 + 3) / 4;
    const float ratio = (float)(5 * 5 / ((double)win * win));
    bool identity = true;
    for (int r = 0; r < 64; r++) {
        float fr = (float)r;
        lut[r] = (float)((double)fr * 1.0 * (double)ratio / nch);
        if (lut[r] != fr) identity = false;
    }
    return !identity;
}

// Label hull of each view (main_mgm.cc:178,207,210-216).  The no-data sentinel range [dmin, dmin+1]
// always lies inside the left hull; on the right view it only matters when the secondary image
// really holds no-data pixels, and then it may stick out of [-dmax, -dmin].
static int plan_labels(int dmin, int dmax, bool sec_has_nodata, int gminv[2], int gmaxv[2])
{
    gminv[0] = dmin; gmaxv[0] = dmax;
    gminv[1] = -dmax; gmaxv[1] = -dmin;
    if (sec_has_nodata) {
        if (dmin < gminv[1]) gminv[1] = dmin;
        if (dmin + 1 > gmaxv[1]) gmaxv[1] = dmin + 1;
    }
    int D = 0;
    for (int vi = 0; vi < 2; vi++) { int d = gmaxv[vi] - gminv[vi] + 1; if (d > D) D = d; }
    return lpl_for(D);
}
// labels per lane of ONE view's slab.  The views may differ: a no-data pixel in the secondary image widens only the right
// view's hull (by one label when |dmin| > dmax), and each view's kernels run at that view's own width -- the volumes are
// [H][W][32 LPL_view] inside buffers sized for the wider view.
static int view_lpl(const int gminv[2], const int gmaxv[2], int vi) { return lpl_for(gmaxv[vi] - gminv[vi] + 1); }

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

// Enqueue the 8-pass aggregation of `nviews` views of slot s in ONE persistent launch.
// general: the float-cost flavour; wgt[vi] = that view's weight image or nullptr (general only)
// gminv: label of slot 0 per view (read by the chunk-skipping kernel only)
static int launch_aggregate(s2pb_ctx *ctx, Slot &s, int nviews, int w, int h, int LPL, float P1, float P2, int ndir, int tsgm,
                            const float *lut, cudaStream_t st, bool general = false, const float *const *wgt = nullptr,
                            const int *gminv = nullptr, int first_view = 0, int ctas_per_sm = 0)
{
    AggParams P;
    memset(&P, 0, sizeof P);
    int mb = max_bands(w, h);
    P.nPV = 0; P.maxBands = 0;
    for (int vi = first_view; vi < first_view + nviews; vi++) {
        CK(cudaMemsetAsync(s.v[vi].progress, 0, (size_t)kMaxPasses * mb * 4, st));
        for (int p = 0; p < ndir; p++) {
            PassDesc &pd = P.pv[P.nPV++];
            fill_pass(pd, p, w, h);
            pd.C = s.v[vi].C; pd.L = s.v[vi].L[p]; pd.Lmin = s.v[vi].Lmin[p];
            pd.W = (general && wgt) ? wgt[vi] : nullptr;
            pd.progress = s.v[vi].progress + (size_t)p * mb;
            if (pd.nBands > P.maxBands) P.maxBands = pd.nBands;
        }
    }
    int *counter = s.next_item + 16 * first_view;          // two launches may be in flight at once: one work counter each
    P.P1 = P1; P.P2 = P2; P.next_item = counter; P.abort_flag = ctx->abort_flag; P.lut = general ? nullptr : lut;
    P.general = general ? 1 : 0;
    CK(cudaMemsetAsync(counter, 0, 4, st));
    if (wide_slab(LPL)) {
        ChunkedParams Q;
        memset(&Q, 0, sizeof Q);
        Q.A = P;
        Q.DP = 32 * LPL;
        int q = 0;
        for (int vi = first_view; vi < first_view + nviews; vi++)
            for (int p = 0; p < ndir; p++, q++) { Q.lo[q] = s.v[vi].lo; Q.hi[q] = s.v[vi].hi; Q.gmin[q] = gminv[vi]; }
        int rr = agg_chunked_launch(tsgm, Q, ctx->sm_count, st);
        if (rr == 0) { ctx->launches++; return S2PB_OK; }
        if (rr != -2) return fail(S2PB_ERR_CUDA, "chunked aggregation launch failed: %s", cudaGetErrorString(cudaGetLastError()));
    }
    int r = agg_launch(LPL, tsgm, P, ctx->sm_count, st, ctas_per_sm);
    if (r == -2) return fail(S2PB_ERR_UNSUPPORTED, "no aggregation kernel for %d labels per lane", LPL);
    if (r != 0) return fail(S2PB_ERR_CUDA, "aggregation launch failed: %s", cudaGetErrorString(cudaGetLastError()));
    ctx->launches++;
    return S2PB_OK;
}

// S2PB_COST_STRIP=0: the per-pixel cost kernel for every shape (A/B)
static bool cost_strip_enabled() { static int v = -1; if (v < 0) { const char *e = getenv("S2PB_COST_STRIP"); v = e ? atoi(e) : 1; } return v != 0; }
template <int LPL> static void launch_cost_t(const uint64_t *cu, const uint64_t *cv, const uint64_t *cv1, int zoom, bool narrow, int w, int h,
                                             const short *lo, const short *hi, int gmin, uint8_t *C, int sm, cudaStream_t st)
{
    if constexpr (LPL <= 8) {
        if (zoom != 2 && narrow && cost_strip_enabled()) { cost_strip_kernel<LPL><<<sm * 16, kCostStripThreads, 0, st>>>(cu, cv, w, h, lo, hi, gmin, C); return; }
    }
    if (zoom == 2) {
        if (narrow) cost_kernel<LPL, true, true><<<sm * 8, 256, 0, st>>>(cu, cv, cv1, w, h, lo, hi, gmin, C);
        else cost_kernel<LPL, true, false><<<sm * 8, 256, 0, st>>>(cu, cv, cv1, w, h, lo, hi, gmin, C);
    } else {
        if (narrow) cost_kernel<LPL, false, true><<<sm * 8, 256, 0, st>>>(cu, cv, cv1, w, h, lo, hi, gmin, C);
        else cost_kernel<LPL, false, false><<<sm * 8, 256, 0, st>>>(cu, cv, cv1, w, h, lo, hi, gmin, C);
    }
}
template <int LPL> static void launch_wta_t(const WtaParams &P, int sm, cudaStream_t st, bool general)
{
    if (general) wta_kernel<LPL, true><<<sm * 16, kWtaThreads, 0, st>>>(P);
    else wta_kernel<LPL, false><<<sm * 16, kWtaThreads, 0, st>>>(P);
}
template <int LPL> static void launch_cost_gen_t(const CostGenParams &P, int sm, cudaStream_t st)
{
    cost_gen_kernel<LPL><<<sm * 8, 256, 0, st>>>(P);
}
#define LPL_SWITCH(LPL, CALL)                                                             \
    switch (LPL) {                                                                        \
    case 1: { constexpr int K = 1; CALL; } break;   case 2: { constexpr int K = 2; CALL; } break;   \
    case 3: { constexpr int K = 3; CALL; } break;   case 4: { constexpr int K = 4; CALL; } break;   \
    case 5: { constexpr int K = 5; CALL; } break;   case 6: { constexpr int K = 6; CALL; } break;   \
    case 8: { constexpr int K = 8; CALL; } break;   case 12: { constexpr int K = 12; CALL; } break; \
    case 16: { constexpr int K = 16; CALL; } break;                                        \
    default: return fail(S2PB_ERR_UNSUPPORTED, "unsupported labels-per-lane %d", LPL);     \
    }

// census_win: the census window the codes were made with (3 and 5 leave the high word of a code zero)
static int launch_cost(s2pb_ctx *ctx, int LPL, int census_win, const uint64_t *cu, const uint64_t *cv, int w, int h, const short *lo, const short *hi,
                       int gmin, void *C, cudaStream_t st, const uint64_t *cv1 = nullptr, int zoom = 1)
{
    const bool narrow = census_win <= 5;
    LPL_SWITCH(LPL, launch_cost_t<K>(cu, cv, cv1, zoom, narrow, w, h, lo, hi, gmin, (uint8_t *)C, ctx->sm_count, st));
    CK(cudaGetLastError());
    ctx->launches++;
    return S2PB_OK;
}
static int launch_cost_gen(s2pb_ctx *ctx, int LPL, const CostGenParams &P, cudaStream_t st)
{
    LPL_SWITCH(LPL, launch_cost_gen_t<K>(P, ctx->sm_count, st));
    CK(cudaGetLastError());
    ctx->launches++;
    return S2PB_OK;
}
static int launch_wta(s2pb_ctx *ctx, int LPL, const WtaParams &P, cudaStream_t st, bool general = false)
{
    if (P.S == nullptr && wide_slab(LPL)) {
        const int DP = 32 * LPL;
        const size_t smem = (size_t)(kWtaThreads / 32) * DP * sizeof(float);
        if (general) wta_chunked_kernel<true><<<ctx->sm_count * 16, kWtaThreads, smem, st>>>(P, DP);
        else wta_chunked_kernel<false><<<ctx->sm_count * 16, kWtaThreads, smem, st>>>(P, DP);
        CK(cudaGetLastError());
        ctx->launches++;
        return S2PB_OK;
    }
    LPL_SWITCH(LPL, launch_wta_t<K>(P, ctx->sm_count, st, general));
    CK(cudaGetLastError());
    ctx->launches++;
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

// Coefficient tables for rows of n pixels, computed once per width on the host (libm, like the reference's DCT) and
// kept on the device.  FFTW's unnormalised definitions:
//   REDFT10  Y[k] = sum_j 2 cos(pi (j + 1/2) k / n) X[j]
//   REDFT01  Y[i] = X[0] + sum_{k>=1} 2 cos(pi k (i + 1/2) / n) X[k]
//   RODFT01  Y[i] = (-1)^i X[n-1] + sum_{k<n-1} 2 sin(pi (k + 1) (i + 1/2) / n) X[k]
// half = true adds what the half-pixel shift of SUBPIX = 2 needs (both inverse tables row-major and the phase factors
// cos(k a), sin(k a), a = (pi / n) * (-1/2), shear.c:66-79).
static int dct_tables(s2pb_ctx *ctx, int n, bool half, const s2pb_ctx::DctTab **out)
{
    if (n > 8192) return fail(S2PB_ERR_UNSUPPORTED, "tiles wider than 8192 px are not supported (DCT tables of %d x %d doubles)", n, n);
    std::lock_guard<std::mutex> lock(ctx->dct_mu);
    s2pb_ctx::DctTab *t = nullptr;
    for (auto &e : ctx->dct) if (e.n == n) t = &e;
    if (!t) { ctx->dct.push_back({n, nullptr, nullptr, nullptr, nullptr, nullptr}); t = &ctx->dct.back(); }
    const double pi = 3.14159265358979323846264338327950288;
    const size_t nn = (size_t)n * n;
    std::vector<double> h;
    auto upload = [&](double **dst, size_t count) -> int {
        cudaError_t e = cudaMalloc((void **)dst, count * sizeof(double));
        if (e != cudaSuccess) { cudaGetLastError(); *dst = nullptr; return fail(S2PB_ERR_NOMEM, "DCT table of %zu bytes: %s", count * 8, cudaGetErrorString(e)); }
        CK(cudaMemcpy(*dst, h.data(), count * sizeof(double), cudaMemcpyHostToDevice));
        return S2PB_OK;
    };
    int rc;
    if (!t->T10) {
        h.resize(nn);
        for (int k = 0; k < n; k++)
            for (int j = 0; j < n; j++) h[(size_t)k * n + j] = 2.0 * cos(pi * (j + 0.5) * k / n);
        if ((rc = upload(&t->T10, nn)) != S2PB_OK) return rc;
    }
    if (!t->T01) {
        h.resize(nn);
        for (int i = 0; i < n; i++)
            for (int k = 0; k < n; k++) h[(size_t)i * n + k] = (k == 0) ? 1.0 : 2.0 * cos(pi * k * (i + 0.5) / n);
        if ((rc = upload(&t->T01, nn)) != S2PB_OK) return rc;
    }
    if (half && !t->TR01) {
        h.resize(nn);
        for (int i = 0; i < n; i++)
            for (int k = 0; k < n; k++) h[(size_t)i * n + k] = (k == n - 1) ? ((i & 1) ? -1.0 : 1.0) : 2.0 * sin(pi * (k + 1) * (i + 0.5) / n);
        if ((rc = upload(&t->TR01, nn)) != S2PB_OK) return rc;
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

// rt = shift(img, 0) of the reference: see dct_kernels.cuh.  Asynchronous; when no row needs it the kernels return at once.
// Y: [h][w] doubles of scratch.  rowlist: room for h + w ints and w bytes (row list, column list, column flags).
static int round_trip_zero(s2pb_ctx *ctx, const float *img, int w, int h, float *rt, RtState *state, int *rowlist, float *rowthr,
                           double *Y, cudaStream_t st)
{
    int *collist = rowlist + h;
    unsigned char *colflag = reinterpret_cast<unsigned char *>(collist + w);
    const s2pb_ctx::DctTab *t;
    int rc = dct_tables(ctx, w, false, &t);
    if (rc != S2PB_OK) return rc;
    CK(cudaMemsetAsync(state, 0, sizeof(RtState), st));
    CK(cudaMemsetAsync(colflag, 0, (size_t)w, st));
    rt_flag_kernel<<<h, 256, 0, st>>>(img, w, h, rt, state, rowlist, rowthr, colflag);
    rt_collist_kernel<<<1, 1024, 0, st>>>(colflag, w, state, collist);
    dct_gemm_kernel<float, true><<<ctx->sm_count * 4, kGemmThreads, 0, st>>>(t->T10, img, w, h, state, rowlist, Y, nullptr, nullptr, nullptr);
    rt_inverse_gemm_kernel<<<ctx->sm_count * 4, kGemmThreads, 0, st>>>(t->T01, Y, w, state, rowlist, collist, rowthr, img, rt);
    ctx->launches += 4;
    CK(cudaGetLastError());
    return S2PB_OK;
}

// out = shift(img, 1/2) of the reference (SUBPIX = 2).  scratch: 4 x [h][w] doubles.
static int shift_half(s2pb_ctx *ctx, const float *img, int w, int h, float *out, double *scratch, cudaStream_t st)
{
    const s2pb_ctx::DctTab *t;
    int rc = dct_tables(ctx, w, true, &t);
    if (rc != S2PB_OK) return rc;
    const size_t npix = (size_t)w * h;
    double *ck = scratch, *sk = scratch + npix, *sym = scratch + 2 * npix, *anti = scratch + 3 * npix;
    const int g = ctx->sm_count * 4;
    dct_gemm_kernel<float, true><<<g, kGemmThreads, 0, st>>>(t->T10, img, w, h, nullptr, nullptr, ck, t->mc, t->ms, sk);
    dct_gemm_kernel<double, false><<<g, kGemmThreads, 0, st>>>(t->T01, ck, w, h, nullptr, nullptr, sym, nullptr, nullptr, nullptr);
    dct_gemm_kernel<double, false><<<g, kGemmThreads, 0, st>>>(t->TR01, sk, w, h, nullptr, nullptr, anti, nullptr, nullptr, nullptr);
    dct_combine_kernel<<<(unsigned)((npix + 255) / 256), 256, 0, st>>>(sym, anti, npix, out);
    ctx->launches += 4;
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
// device weight images at full resolution, both or neither (s2pb_mgm_weighted)
struct MgmExtra { const float *wl = nullptr, *wr = nullptr; };

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

// remove_small_cc on a device image (in -> out), scratch: two int images
static int launch_remove_small_cc(s2pb_ctx *ctx, const float *in, float *out, int w, int h, int minarea, int *lab, int *area, cudaStream_t st)
{
    int n = w * h;
    dim3 b2(32, 8);
    cc_init_kernel<<<(n + 255) / 256, 256, 0, st>>>(in, n, lab, area);
    cc_rows_kernel<<<(h + 3) / 4, 128, 0, st>>>(in, w, h, 5.f, lab);                 // one warp per row
    cc_link_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(in, w, h, 5.f, lab);
    cc_flatten_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, lab);
    cc_area_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, lab, area);
    cc_filter_kernel<<<(n + 255) / 256, 256, 0, st>>>(in, n, lab, area, minarea, out);
    ctx->launches += 6;
    CK(cudaGetLastError());
    return S2PB_OK;
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

// One mgm_call (mgm_multiscale.cc:161-335) on the slot's workspace, which slot_ensure has sized for the wider slab.
//   img:   the NaN-free images; lo / hi: each view's per-pixel label range; gminv: the label of each view's slot 0
//   LPLv:  labels per lane of each view's slab (wide_slab: the chunk-skipping kernels)
//   zoom:  ZOOMFACTOR, 1 or 2 (labels of half pixels: SUBPIX = 2); wgt: the views' weight images, or none
//   outL / outR: the destinations of the left-right check; outR == nullptr: the right map is not wanted, it goes to a free
//   scratch image of the slot, returned in outR
//   timed (single scale): record s.ev[1..4] after the stages (s2pb_last_timings), and size the aggregation's grid by
//   whether another slot's aggregation is in flight (other_aggregation_pending reads those events)
// Enqueues only: no host synchronisation (except S2PB_TRACE=1).
static int mgm_call(s2pb_ctx *ctx, Slot &s, int w, int h, const float *const img[2], short *const lo[2], short *const hi[2],
                    const int gminv[2], const int LPLv[2], int zoom, const float *const wgt[2], const s2pb_mgm_params *p,
                    float *outL, float *&outR, cudaStream_t st, bool timed)
{
    const bool general = general_flavour(p, wgt);
    const bool census = p->cost == S2PB_COST_CENSUS, ncc = p->cost == S2PB_COST_NCC;
    const size_t npix = (size_t)w * h;
    dim3 b2(32, 8);
    int rc;
    float lut_h[64];
    const float *lut = nullptr;
    if (cost_lut(p->census_win, lut_h) || general) { CK(cudaMemcpyAsync(s.lut, lut_h, sizeof lut_h, cudaMemcpyHostToDevice, st)); lut = s.lut; }
    // ---- census of both images and of the copies the other view matches against
    for (int vi = 0; vi < 2; vi++) {
        ViewWS &v = s.v[vi];
        v.lo = lo[vi]; v.hi = hi[vi];
        // v.rt = shift(img[vi], 0): the reference's DCT round trip (mgm_costvolume.cc:50-60)
        rc = round_trip_zero(ctx, img[vi], w, h, v.rt, v.rtstate, v.rowlist, v.rowthr, s.Ydct, st);
        if (rc != S2PB_OK) return rc;
        if (census) {
            census_pair_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(img[vi], v.rt, v.rtstate, w, h, p->census_win / 2, v.census, v.census_rt);
            ctx->launches++;
        }
        if (ncc) {     // window statistics in the (then unused) census buffers: 8 B / pixel
            ncc_stats_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(img[vi], w, h, p->census_win / 2, (float2 *)v.census);
            ncc_stats_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(v.rt, w, h, p->census_win / 2, (float2 *)v.census_rt);
            ctx->launches += 2;
        }
    }
    // ZOOMFACTOR 2: shf[vi] = shift(img[vi], 1/2) (kept for the image-domain distances) and its census, in the pyramid arena
    float *shf[2] = {nullptr, nullptr};
    uint64_t *cen_half[2] = {nullptr, nullptr};
    if (zoom == 2) {
        for (int vi = 0; vi < 2; vi++) { shf[vi] = arena_take<float>(s, npix); cen_half[vi] = arena_take<uint64_t>(s, npix); }
        double *scratch = arena_take<double>(s, npix * 4);
        if (!scratch) return fail(S2PB_ERR_NOMEM, "pyramid arena exhausted");
        for (int vi = 0; vi < 2; vi++) {
            rc = shift_half(ctx, img[vi], w, h, shf[vi], scratch, st);
            if (rc != S2PB_OK) return rc;
            if (census) { census_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(shf[vi], w, h, p->census_win / 2, cen_half[vi]); ctx->launches++; }
            if (ncc) { ncc_stats_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(shf[vi], w, h, p->census_win / 2, (float2 *)cen_half[vi]); ctx->launches++; }
        }
    }
    CK(cudaGetLastError());
    if (timed) CK(cudaEventRecord(s.ev[1], st));
    // ---- cost volumes: view 0 = left reference, view 1 = right reference (mgm_multiscale.cc:222,270)
    for (int vi = 0; vi < 2; vi++) {
        const ViewWS &v = s.v[vi], &o = s.v[1 - vi];
        if (general) {
            CostGenParams G;
            memset(&G, 0, sizeof G);
            G.u = img[vi]; G.v0 = o.rt; G.v1 = shf[1 - vi];
            G.cu = v.census; G.cv0 = o.census_rt; G.cv1 = cen_half[1 - vi];
            G.su = (const float2 *)G.cu; G.sv0 = (const float2 *)G.cv0; G.sv1 = (const float2 *)G.cv1;
            G.lut = s.lut; G.lo = lo[vi]; G.hi = hi[vi];
            G.w = w; G.h = h; G.gmin = gminv[vi]; G.cost = p->cost; G.win = p->census_win; G.zoom = zoom;
            G.C = (float *)v.C;
            if (wide_slab(LPLv[vi])) {         // only the chunks of each pixel's span
                cost_gen_chunked_kernel<<<ctx->sm_count * 8, 256, 0, st>>>(G, 32 * LPLv[vi]);
                ctx->launches++;
                rc = cudaGetLastError() == cudaSuccess ? S2PB_OK : fail(S2PB_ERR_CUDA, "cost_gen_chunked_kernel launch failed");
            } else {
                rc = launch_cost_gen(ctx, LPLv[vi], G, st);
            }
        } else if (wide_slab(LPLv[vi])) {      // only the chunks of each pixel's span
            if (zoom == 2) cost_chunked_kernel<true><<<ctx->sm_count * 8, 256, 0, st>>>(v.census, o.census_rt, cen_half[1 - vi], w, h,
                                                                                  lo[vi], hi[vi], gminv[vi], 32 * LPLv[vi], (uint8_t *)v.C);
            else cost_chunked_kernel<false><<<ctx->sm_count * 8, 256, 0, st>>>(v.census, o.census_rt, nullptr, w, h,
                                                                               lo[vi], hi[vi], gminv[vi], 32 * LPLv[vi], (uint8_t *)v.C);
            ctx->launches++;
            rc = cudaGetLastError() == cudaSuccess ? S2PB_OK : fail(S2PB_ERR_CUDA, "cost_chunked_kernel launch failed");
        } else {
            rc = launch_cost(ctx, LPLv[vi], p->census_win, v.census, o.census_rt, w, h, lo[vi], hi[vi], gminv[vi], v.C, st,
                             cen_half[1 - vi], zoom);
        }
        if (rc != S2PB_OK) return rc;
    }
    if (timed) CK(cudaEventRecord(s.ev[2], st));
    TRACE(st, "  census + cost");
    // ---- 8-pass MGM of both views (mgm_multiscale.cc:194-202: P1 / ZOOMFACTOR) in one persistent launch, or two when the
    // views' slabs differ in width
    const float P1 = p->P1 / (float)zoom;
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
        W.pkr = ctx->pkr_dst[vi];
        rc = launch_wta(ctx, LPLv[vi], W, st, general);
        if (rc != S2PB_OK) return rc;
    }
    if (timed) CK(cudaEventRecord(s.ev[4], st));
    TRACE(st, "  wta");
    // ---- post filters (mgm_multiscale.cc:310-334)
    float *dl = s.v[0].disp, *dr = s.v[1].disp, *xl = s.v[0].tmp, *xr = s.v[1].tmp;
    if (p->median > 0) {
        median_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(dl, xl, w, h, p->median);
        median_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(dr, xr, w, h, p->median);
        ctx->launches += 2;
        float *t = dl; dl = xl; xl = t; t = dr; dr = xr; xr = t;
    }
    if (p->mindiff >= 0) {      // mgm_multiscale.cc:318-319: only the left map, against the right view's cost image
        mindiff_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(dl, s.v[1].cost, xl, w, h, p->census_win, p->mindiff);
        ctx->launches++;
        float *t = dl; dl = xl; xl = t;
    }
    if (!outR) outR = xr;
    if (p->lr_mode == 1) {
        lrcheck_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(dr, dl, outR, w, h, p->lr_tau);
        lrcheck_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(dl, dr, outL, w, h, p->lr_tau);
        ctx->launches += 2;
    } else {
        CK(cudaMemcpyAsync(outL, dl, npix * 4, cudaMemcpyDeviceToDevice, st));
        CK(cudaMemcpyAsync(outR, dr, npix * 4, cudaMemcpyDeviceToDevice, st));
    }
    CK(cudaGetLastError());
    TRACE(st, "  median / lr");
    return S2PB_OK;
}

// One mgm_call of a pyramid level: the label ranges of both views from the level's bounds, one slab for both views
// sized by the wider hull, then the speckle filter (mgm_multiscale.cc:328-334).
static int mgm_call_level(s2pb_ctx *ctx, Slot &s, Level &L, int zoom, const s2pb_mgm_params *p, cudaStream_t st, bool weighted)
{
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
    label_ranges_kernel<<<(n + 255) / 256, 256, 0, st>>>(L.dminL, L.dmaxL, n, (float)zoom, lo[0], hi[0], d_hull);
    label_ranges_kernel<<<(n + 255) / 256, 256, 0, st>>>(L.dminR, L.dmaxR, n, (float)zoom, lo[1], hi[1], d_hull + 2);
    ctx->launches += 2;
    CK(cudaGetLastError());
    int hull[4];
    CK(cudaMemcpyAsync(hull, d_hull, sizeof hull, cudaMemcpyDeviceToHost, st));
    int rc = sync_or_timeout(ctx, st);
    if (rc != S2PB_OK) return rc;
    int gminv[2] = {hull[0], hull[2]}, gmaxv[2] = {hull[1], hull[3]};
    int D = 0;
    for (int vi = 0; vi < 2; vi++) {
        if (gminv[vi] < -16000 || gmaxv[vi] > 16000) return fail(S2PB_ERR_ARG, "label range out of the int16 domain");
        int d = gmaxv[vi] - gminv[vi] + 1; if (d > D) D = d;
    }
    int LPL = lpl_for(D);
    if (LPL < 0) {      // hull wider than 512 labels: slab of ceil(D / 32) chunks through the chunk-skipping kernels
        LPL = (D + 31) / 32;
        if (LPL > 64) return fail(S2PB_ERR_UNSUPPORTED, "a %dx%d level needs %d labels in its volume; 2048 are supported", w, h, D);
    }
    rc = slot_ensure(ctx, s, w, h, 32 * LPL, p->ndir, general ? 4 : 1);
    if (rc != S2PB_OK) return rc;
    TRACE(st, "level %dx%d zoom %d: hull L [%d,%d] R [%d,%d] -> LPL %d%s", w, h, zoom, gminv[0], gmaxv[0], gminv[1], gmaxv[1], LPL,
          general ? " (general flavour)" : "");
    const float *img[2] = {L.u, L.v};
    const int LPLv[2] = {LPL, LPL};
    const bool cc = p->remove_small_cc > 0;
    float *lrL = cc ? tl : L.dl, *lrR = cc ? tr : L.dr;
    rc = mgm_call(ctx, s, w, h, img, lo, hi, gminv, LPLv, zoom, wgt, p, lrL, lrR, st, false);
    if (rc != S2PB_OK) return rc;
    if (cc) {
        rc = launch_remove_small_cc(ctx, lrL, L.dl, w, h, p->remove_small_cc, lab, area, st);
        if (rc != S2PB_OK) return rc;
        rc = launch_remove_small_cc(ctx, lrR, L.dr, w, h, p->remove_small_cc, lab, area, st);
        if (rc != S2PB_OK) return rc;
    }
    TRACE(st, "  remove_small_cc");
    CK(cudaMemcpyAsync(L.conf, s.v[0].conf, npix * 4, cudaMemcpyDeviceToDevice, st));
    CK(cudaGetLastError());
    return S2PB_OK;
}

// main() of mgm_multi (main_mgm_multi.cc:88-256) + recursive_multiscale (mgm_multiscale.cc:339-410)
static int mgm_multi_enqueue(s2pb_ctx *ctx, Slot &s, const float *d_im1, const float *d_im2, int w, int h, int dmin, int dmax,
                             const s2pb_mgm_params *p, float *d_disp, float *d_conf, uint8_t *d_mask, float *d_dispR, cudaStream_t st,
                             const MgmExtra *x)
{
    const int n = w * h;
    dim3 b2(32, 8);
    const bool weighted = x && x->wl && x->wr;
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
        CK(cudaMemcpyAsync(lv[0].wl, x->wl, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
        CK(cudaMemcpyAsync(lv[0].wr, x->wr, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
    }
    s.timed = false;
    // level 0: NaN -> 0, initial bounds (main_mgm_multi.cc:160-196; the sentinel for no-data is dmin in both views)
    init_ranges_kernel<<<(n + 255) / 256, 256, 0, st>>>(d_im1, n, (float)dmin, (float)dmax, (float)dmin, lv[0].u, lv[0].dminL, lv[0].dmaxL);
    init_ranges_kernel<<<(n + 255) / 256, 256, 0, st>>>(d_im2, n, (float)-dmax, (float)-dmin, (float)dmin, lv[0].v, lv[0].dminR, lv[0].dmaxR);
    ctx->launches += 2;
    const GaussTaps T = gauss_taps(0.8f);
    for (size_t l = 0; l + 1 < lv.size(); l++) {
        Level &a = lv[l], &b = lv[l + 1];
        dim3 g = grid2d(b.w, b.h, b2);
        downsample2x_kernel<<<g, b2, 0, st>>>(a.u, a.w, a.h, T, b.u, b.w, b.h);
        downsample2x_kernel<<<g, b2, 0, st>>>(a.v, a.w, a.h, T, b.v, b.w, b.h);
        if (weighted) {                        // the weight maps follow the pyramid, mgm_multiscale.cc:375-378
            downsample2x_kernel<<<g, b2, 0, st>>>(a.wl, a.w, a.h, T, b.wl, b.w, b.h);
            downsample2x_kernel<<<g, b2, 0, st>>>(a.wr, a.w, a.h, T, b.wr, b.w, b.h);
            ctx->launches += 2;
        }
        downsample2x_disp_kernel<<<g, b2, 0, st>>>(a.dminL, a.w, a.h, 0, b.dminL, b.w, b.h);
        downsample2x_disp_kernel<<<g, b2, 0, st>>>(a.dmaxL, a.w, a.h, 1, b.dmaxL, b.w, b.h);
        downsample2x_disp_kernel<<<g, b2, 0, st>>>(a.dminR, a.w, a.h, 0, b.dminR, b.w, b.h);
        downsample2x_disp_kernel<<<g, b2, 0, st>>>(a.dmaxR, a.w, a.h, 1, b.dmaxR, b.w, b.h);
        ctx->launches += 6;
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
                update_ranges_kernel<<<grid2d(c.w, c.h, b2), b2, 0, st>>>(disp2[vi], 2.f, c.w, c.h, nullptr, nullptr, fmin[vi], fmax[vi],
                                                                       L.w, L.h, 8.f, 4, omin, omax);
                zoom2_kernel<<<grid2d(L.w, L.h, b2), b2, 0, st>>>(omin, c.w, fmin[vi], L.w, L.h);
                zoom2_kernel<<<grid2d(L.w, L.h, b2), b2, 0, st>>>(omax, c.w, fmax[vi], L.w, L.h);
                ctx->launches += 3;
            }
            CK(cudaGetLastError());
        }
        s.arena_off = arena_mark;
        rc = mgm_call_level(ctx, s, L, 1, p, st, weighted);
        if (rc != S2PB_OK) return rc;
    }
    Level &L0 = lv[0];
    if (d_conf) CK(cudaMemcpyAsync(d_conf, L0.conf, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));   // the ZOOM=1 call's consensus
    if (p->subpix > 1) {                       // main_mgm_multi.cc:203-209: bounds = result +-2 over 9x9, labels = half pixels
        s.arena_off = arena_mark;
        float *a = arena_take<float>(s, n), *b = arena_take<float>(s, n), *c = arena_take<float>(s, n), *d = arena_take<float>(s, n);
        const size_t mark2 = s.arena_off;
        update_ranges_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(L0.dl, 1.f, w, h, L0.dminL, L0.dmaxL, L0.dminL, L0.dmaxL, w, h, 2.f, 4, a, b);
        update_ranges_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(L0.dr, 1.f, w, h, L0.dminR, L0.dmaxR, L0.dminR, L0.dmaxR, w, h, 2.f, 4, c, d);
        ctx->launches += 2;
        L0.dminL = a; L0.dmaxL = b; L0.dminR = c; L0.dmaxR = d;
        s.arena_off = mark2;
        float *keep[2] = {ctx->pkr_dst[0], ctx->pkr_dst[1]};          // ... and with its own img_dict: the PKR images written are the ZOOM = 1 call's
        ctx->pkr_dst[0] = ctx->pkr_dst[1] = nullptr;
        rc = mgm_call_level(ctx, s, L0, p->subpix, p, st, false);   // fresh `param` without the weight images (main_mgm_multi.cc:207)
        ctx->pkr_dst[0] = keep[0]; ctx->pkr_dst[1] = keep[1];
        if (rc != S2PB_OK) return rc;
    }
    float *outL = d_disp;
    if (p->lr_mode == 2) {                     // main_mgm_multi.cc:212-217
        s.arena_off = arena_mark;
        float *tr = arena_take<float>(s, n);
        lrcheck_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(L0.dr, L0.dl, tr, w, h, p->lr_tau);
        lrcheck_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(L0.dl, L0.dr, outL, w, h, p->lr_tau);
        ctx->launches += 2;
        if (d_dispR) CK(cudaMemcpyAsync(d_dispR, tr, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
    } else {
        CK(cudaMemcpyAsync(outL, L0.dl, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
        if (d_dispR) CK(cudaMemcpyAsync(d_dispR, L0.dr, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
    }
    nan_restore_kernel<<<(n + 255) / 256, 256, 0, st>>>(outL, d_im1, n);
    ctx->launches++;
    if (d_dispR) { nan_restore_kernel<<<(n + 255) / 256, 256, 0, st>>>(d_dispR, d_im2, n); ctx->launches++; }
    if (d_mask) { rejection_mask_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(outL, d_im1, d_im2, w, h, d_mask); ctx->launches++; }
    CK(cudaGetLastError());
    return S2PB_OK;
}

// ------------------------------------------------------------------ the matcher (device level)

static int mgm_enqueue(s2pb_ctx *ctx, Slot &s, const float *d_im1, const float *d_im2, int w, int h, int dmin, int dmax,
                       const s2pb_mgm_params *p, float *d_disp, float *d_conf, uint8_t *d_mask, float *d_dispR, cudaStream_t st,
                       int nodata_hint, const MgmExtra *x = nullptr)
{
    if (p->scales >= 0) return mgm_multi_enqueue(ctx, s, d_im1, d_im2, w, h, dmin, dmax, p, d_disp, d_conf, d_mask, d_dispR, st, x);
    const float *wgt[2] = {x ? x->wl : nullptr, x ? x->wr : nullptr};
    const bool general = general_flavour(p, wgt);
    const size_t npix = (size_t)w * h;
    const int n = (int)npix;
    if (nodata_hint < 0) {     // unknown: look (costs one stream synchronisation)
        int *flag = s.d_small + 16;      // this slot's own word (several slots may ask at once)
        CK(cudaMemsetAsync(flag, 0, 4, st));
        has_nan_kernel<<<ctx->sm_count * 4, 256, 0, st>>>(d_im2, n, flag);
        ctx->launches++;
        int hflag = 0;
        CK(cudaMemcpyAsync(&hflag, flag, 4, cudaMemcpyDeviceToHost, st));
        int rs = sync_or_timeout(ctx, st);
        if (rs != S2PB_OK) return rs;
        nodata_hint = hflag ? 3 : 0;
    }
    int gminv[2], gmaxv[2];
    plan_labels(dmin, dmax, (nodata_hint & 2) != 0, gminv, gmaxv);
    int LPLv[2] = {view_lpl(gminv, gmaxv, 0), view_lpl(gminv, gmaxv, 1)};
    for (int vi = 0; vi < 2; vi++)
        if (LPLv[vi] < 0) {      // more than 512 labels: chunk-skipping kernels on a slab of ceil(D / 32) chunks
            LPLv[vi] = (gmaxv[vi] - gminv[vi] + 32) / 32;
            if (LPLv[vi] > 64)
                return fail(S2PB_ERR_UNSUPPORTED, "disparity range [%d,%d] needs more than the 2048 labels supported", dmin, dmax);
        }
    const int LPL = LPLv[0] > LPLv[1] ? LPLv[0] : LPLv[1];
    int rc = slot_ensure(ctx, s, w, h, 32 * LPL, p->ndir, general ? 4 : 1);
    if (rc != S2PB_OK) return rc;
    const float *im[2] = {d_im1, d_im2};
    dim3 b2(32, 8);
    s.timed = true;
    CK(cudaEventRecord(s.ev[0], st));
    // ---- NaN-free copies of both images and their label ranges
    for (int vi = 0; vi < 2; vi++) {
        int lo_all = vi == 0 ? dmin : -dmax, hi_all = vi == 0 ? dmax : -dmin;
        prepare_view_kernel<<<(n + 255) / 256, 256, 0, st>>>(im[vi], n, lo_all, hi_all, dmin, s.v[vi].img, s.v[vi].lo, s.v[vi].hi);
        ctx->launches++;
    }
    const float *img[2] = {s.v[0].img, s.v[1].img};
    short *lo[2] = {s.v[0].lo, s.v[1].lo}, *hi[2] = {s.v[0].hi, s.v[1].hi};
    float *outL = d_disp, *outR = d_dispR;
    rc = mgm_call(ctx, s, w, h, img, lo, hi, gminv, LPLv, 1, wgt, p, outL, outR, st, true);
    if (rc != S2PB_OK) return rc;
    // ---- no-data restore (main_mgm.cc:231-236), mask
    nan_restore_kernel<<<(n + 255) / 256, 256, 0, st>>>(outL, d_im1, n);
    nan_restore_kernel<<<(n + 255) / 256, 256, 0, st>>>(outR, d_im2, n);
    ctx->launches += 2;
    if (d_conf) CK(cudaMemcpyAsync(d_conf, s.v[0].conf, npix * 4, cudaMemcpyDeviceToDevice, st));
    if (d_mask) {
        rejection_mask_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(outL, d_im1, d_im2, w, h, d_mask);
        ctx->launches++;
    }
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
    cudaStream_t st = stream ? (cudaStream_t)stream : s.stream;
    set_deadline(ctx, p->timeout_ms);
    rc = mgm_enqueue(ctx, s, d_im1, d_im2, w, h, dmin, dmax, p, d_disp, d_conf, d_mask, d_disp_right, st, nodata_hint);
    if (rc != S2PB_OK) return rc;
    if (p->timeout_ms > 0) return sync_or_timeout(ctx, st);
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

// stage the inputs of one tile through pinned memory and enqueue everything on the slot's stream
static int mgm_host_enqueue(s2pb_ctx *ctx, Slot &s, const float *im1, const float *im2, int w, int h, int dmin, int dmax,
                            const s2pb_mgm_params *p, bool want_mask, bool want_right,
                            float *o_disp = nullptr, float *o_conf = nullptr, uint8_t *o_mask = nullptr,
                            const float *wl = nullptr, const float *wr = nullptr)
{
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
    MgmExtra x;
    if (wl && wr) {        // not a hot path: plain (driver-staged) copies of the caller's weight images
        CK(cudaMemcpyAsync(s.d_w[0], wl, npix * 4, cudaMemcpyHostToDevice, s.stream));
        CK(cudaMemcpyAsync(s.d_w[1], wr, npix * 4, cudaMemcpyHostToDevice, s.stream));
        x.wl = s.d_w[0]; x.wr = s.d_w[1];
    }
    rc = mgm_enqueue(ctx, s, s.d_in[0], s.d_in[1], w, h, dmin, dmax, p, s.d_disp, s.d_conf, want_mask ? s.d_mask : nullptr,
                     want_right ? s.d_dispR : nullptr, s.stream, sec_nodata ? 2 : 0, &x);
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

extern "C" int s2pb_mgm(s2pb_ctx *ctx, const float *im1, const float *im2, int w, int h, int dmin, int dmax,
                        const s2pb_mgm_params *p, float *disp, float *conf, uint8_t *mask, float *disp_right)
{
    return s2pb_mgm_weighted(ctx, im1, im2, w, h, dmin, dmax, p, nullptr, nullptr, disp, conf, mask, disp_right);
}

extern "C" int s2pb_mgm_weighted(s2pb_ctx *ctx, const float *im1, const float *im2, int w, int h, int dmin, int dmax,
                                 const s2pb_mgm_params *p, const float *wl, const float *wr,
                                 float *disp, float *conf, uint8_t *mask, float *disp_right)
{
    if (!ctx || !im1 || !im2 || !disp || !conf) return fail(S2PB_ERR_ARG, "null argument");
    if ((wl == nullptr) != (wr == nullptr)) return fail(S2PB_ERR_ARG, "the weight images come in pairs (-wl and -wr)");
    int rc = check_params(p, w, h, dmin, dmax);
    if (rc != S2PB_OK) return rc;
    CK(cudaSetDevice(ctx->device));
    Slot &s = ctx->slots[0];
    set_deadline(ctx, p->timeout_ms);
    rc = mgm_host_enqueue(ctx, s, im1, im2, w, h, dmin, dmax, p, mask != nullptr, disp_right != nullptr, disp, conf, mask, wl, wr);
    if (rc != S2PB_OK) { cudaStreamSynchronize(s.stream); return rc; }      // nothing may still DMA into the caller's buffers
    rc = sync_or_timeout(ctx, s.stream);
    if (rc != S2PB_OK) return rc;
    size_t npix = (size_t)w * h;
    copy_staged_outputs(s, npix, disp, conf, mask);
    if (disp_right) memcpy(disp_right, s.h_dispR, npix * 4);
    return S2PB_OK;
}

// `mgm ... -confidence_pkrL f -confidence_pkrR g` (main_mgm.cc:147,250-262; mgm_multi likewise): s2pb_mgm plus the peak-ratio
// confidence images of both views.  s2p never asks for them (s2p/block_matching.py:167-183); the matcher's option surface does.
extern "C" int s2pb_mgm_pkr(s2pb_ctx *ctx, const float *im1, const float *im2, int w, int h, int dmin, int dmax,
                            const s2pb_mgm_params *p, float *disp, float *conf, uint8_t *mask, float *disp_right,
                            float *pkr_left, float *pkr_right)
{
    if (!ctx || !pkr_left || !pkr_right) return fail(S2PB_ERR_ARG, "null argument");
    CK(cudaSetDevice(ctx->device));
    const size_t npix = (size_t)w * h;
    cudaStream_t st = ctx->slots[0].stream;
    ScratchLease L(ctx, st);
    float *d0 = L.take<float>(npix * 4), *d1 = L.take<float>(npix * 4);
    if (!d0 || !d1) return L.nomem("the PKR images");
    ctx->pkr_dst[0] = d0; ctx->pkr_dst[1] = d1;
    int rc = s2pb_mgm_weighted(ctx, im1, im2, w, h, dmin, dmax, p, nullptr, nullptr, disp, conf, mask, disp_right);
    ctx->pkr_dst[0] = ctx->pkr_dst[1] = nullptr;
    if (rc == S2PB_OK) {
        cudaError_t e = cudaMemcpyAsync(pkr_left, d0, npix * 4, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(pkr_right, d1, npix * 4, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) rc = fail(S2PB_ERR_CUDA, "copy of the PKR images failed: %s", cudaGetErrorString(e));
    }
    return rc;
}

extern "C" int s2pb_reserve(s2pb_ctx *ctx, int nslots, int w, int h, int nlabels)
{
    if (!ctx || nslots < 1) return fail(S2PB_ERR_ARG, "bad argument");
    CK(cudaSetDevice(ctx->device));
    int LPL = lpl_for(nlabels);
    if (LPL < 0) LPL = (nlabels + 31) / 32;
    if (LPL > 64) return fail(S2PB_ERR_UNSUPPORTED, "too many labels");
    int rc = ensure_slots(ctx, nslots);
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
    set_deadline(ctx, p->timeout_ms * (long long)(n > 0 ? n : 1));       // the per-tile timeout times the number of tiles
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
                Slot &s = ctx->slots[k];
                for (int t = k; t < n && !stop.load(); t += T) {
                    int r = mgm_host_enqueue(ctx, s, im1[t], im2[t], w, h, dmin, dmax, p, mask && mask[t], false, disp[t], conf[t],
                                             mask ? mask[t] : nullptr);
                    if (r == S2PB_OK) r = sync_or_timeout(ctx, s.stream);
                    if (r != S2PB_OK) { codes[k] = r; errs[k] = g_err; stop.store(true); break; }
                    copy_staged_outputs(s, npix, disp[t], conf[t], mask ? mask[t] : nullptr);
                }
            });
        for (auto &t : th) t.join();
        for (int k = 0; k < T; k++)
            if (codes[k] != S2PB_OK) { drain_all(ctx, true); g_err = errs[k]; return codes[k]; }
        return S2PB_OK;
    }
    std::vector<int> inflight(ns, -1);
    auto collect = [&](int si) -> int {
        Slot &s = ctx->slots[si];
        int t = inflight[si];
        if (t < 0) return S2PB_OK;
        int r = sync_or_timeout(ctx, s.stream);
        if (r != S2PB_OK) return r;
        copy_staged_outputs(s, npix, disp[t], conf[t], mask ? mask[t] : nullptr);
        inflight[si] = -1;
        return S2PB_OK;
    };
    // on any error the other slots still have kernels and copies in flight, some of them into the caller's page-locked
    // buffers: stop and wait for all of them before returning (the caller may free its arrays right away)
    auto bail = [&](int code) -> int { std::string keep = g_err; drain_all(ctx, true); g_err = keep; return code; };
    for (int t = 0; t < n; t++) {
        int si = t % ns;
        rc = collect(si);
        if (rc != S2PB_OK) return bail(rc);
        rc = mgm_host_enqueue(ctx, ctx->slots[si], im1[t], im2[t], w, h, dmin, dmax, p, mask && mask[t], false, disp[t], conf[t],
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
    int rc = round_trip_zero(ctx, dv, w, h, out, (RtState *)(aux + lists + (size_t)h * 4), (int *)aux, (float *)(aux + lists), Y, st);
    if (rc != S2PB_OK) return rc;
    *rt = out;
    return S2PB_OK;
}

extern "C" int s2pb_census(s2pb_ctx *ctx, const float *img, int w, int h, int win, uint64_t *codes)
{
    if (!ctx || !img || !codes || w < 1 || h < 1) return fail(S2PB_ERR_ARG, "bad argument");
    if (win != 3 && win != 5 && win != 7) return fail(S2PB_ERR_ARG, "census window must be 3, 5 or 7");
    CK(cudaSetDevice(ctx->device));
    size_t npix = (size_t)w * h;
    cudaStream_t st = ctx->slots[0].stream;
    ScratchLease L(ctx, st);
    float *a = L.take<float>(npix * 4);
    uint64_t *b = L.take<uint64_t>(npix * 8);
    if (!a || !b) return L.nomem("the census");
    CK(cudaMemcpyAsync(a, img, npix * 4, cudaMemcpyHostToDevice, st));
    dim3 b2(32, 8);
    census_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(a, w, h, win / 2, b);
    ctx->launches++;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(codes, b, npix * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return S2PB_OK;
}

static int upload_ranges(ScratchLease &L, const int32_t *lo, const int32_t *hi, size_t npix, int gmin, int D, cudaStream_t st,
                         short **dlo, short **dhi)
{
    std::vector<short> a(npix), b(npix);
    for (size_t i = 0; i < npix; i++) {
        if (lo[i] < gmin || hi[i] > gmin + D - 1 || lo[i] > hi[i]) return fail(S2PB_ERR_ARG, "range of pixel %zu outside the volume", i);
        a[i] = (short)lo[i]; b[i] = (short)hi[i];
    }
    *dlo = L.take<short>(npix * 2);
    *dhi = L.take<short>(npix * 2);
    if (!*dlo || !*dhi) return L.nomem("the label ranges");
    CK(cudaMemcpyAsync(*dlo, a.data(), npix * 2, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(*dhi, b.data(), npix * 2, cudaMemcpyHostToDevice, st));
    CK(cudaStreamSynchronize(st));
    return S2PB_OK;
}

// The [h][w][D] cost volume of u against the round trip of v: through the 8-bit census codes of the hot matcher (codes, with
// cost = census), or through the general path's `cost` (S2PB_COST_*).
static int stage_costvolume(s2pb_ctx *ctx, const float *u, const float *v, int w, int h, const int32_t *lo, const int32_t *hi,
                            int gmin, int D, int win, int cost, bool codes, float *C)
{
    if (!ctx || !u || !v || !lo || !hi || !C || w < 1 || h < 1 || D < 1) return fail(S2PB_ERR_ARG, "bad argument");
    if (win != 3 && win != 5 && win != 7) return fail(S2PB_ERR_ARG, "window must be 3, 5 or 7");
    if (cost < 0 || cost >= S2PB_COST_COUNT) return fail(S2PB_ERR_ARG, "cost must be one of S2PB_COST_*");
    CK(cudaSetDevice(ctx->device));
    int LPL = lpl_for(D);
    if (LPL < 0) return fail(S2PB_ERR_UNSUPPORTED, "too many labels");
    const int DP = 32 * LPL;
    size_t npix = (size_t)w * h, tot = npix * D;
    cudaStream_t st = ctx->slots[0].stream;
    ScratchLease L(ctx, st);
    float *du = L.take<float>(npix * 4), *dv = L.take<float>(npix * 4);
    uint64_t *cu = L.take<uint64_t>(npix * 8), *cv = L.take<uint64_t>(npix * 8);      // census codes or NCC window statistics
    void *dC = L.take<void>(npix * DP * (codes ? 1 : 4));
    float *dCf = L.take<float>(tot * 4), *dlut = L.take<float>(256);
    if (!du || !dv || !cu || !cv || !dC || !dCf || !dlut) return L.nomem("the cost volume");
    short *dlo, *dhi;
    int rc = upload_ranges(L, lo, hi, npix, gmin, D, st, &dlo, &dhi);
    if (rc != S2PB_OK) return rc;
    CK(cudaMemcpyAsync(du, u, npix * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(dv, v, npix * 4, cudaMemcpyHostToDevice, st));
    float *rt = nullptr;
    rc = stage_round_trip(ctx, L, dv, w, h, st, &rt);
    if (rc != S2PB_OK) return rc;
    float lut_h[64];
    const bool scaled = cost_lut(win, lut_h);
    CK(cudaMemcpyAsync(dlut, lut_h, 256, cudaMemcpyHostToDevice, st));
    dim3 b2(32, 8);
    if (cost == S2PB_COST_CENSUS) {
        census_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(du, w, h, win / 2, cu);
        census_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(rt, w, h, win / 2, cv);
        ctx->launches += 2;
    }
    if (cost == S2PB_COST_NCC) {
        ncc_stats_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(du, w, h, win / 2, (float2 *)cu);
        ncc_stats_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(rt, w, h, win / 2, (float2 *)cv);
        ctx->launches += 2;
    }
    if (codes) {
        rc = launch_cost(ctx, LPL, win, cu, cv, w, h, dlo, dhi, gmin, dC, st);
        if (rc != S2PB_OK) return rc;
        unpack_cost_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>((uint8_t *)dC, npix, D, DP, scaled ? dlut : nullptr, dCf);
    } else {
        CostGenParams G;
        memset(&G, 0, sizeof G);
        G.u = du; G.v0 = rt; G.cu = cu; G.cv0 = cv;
        G.su = (float2 *)cu; G.sv0 = (float2 *)cv;
        G.lut = dlut; G.lo = dlo; G.hi = dhi;
        G.w = w; G.h = h; G.gmin = gmin; G.cost = cost; G.win = win; G.zoom = 1; G.C = (float *)dC;
        rc = launch_cost_gen(ctx, LPL, G, st);
        if (rc != S2PB_OK) return rc;
        unpad_cost_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>((float *)dC, npix, D, DP, dCf);
    }
    ctx->launches++;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(C, dCf, tot * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return S2PB_OK;
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
    CK(cudaSetDevice(ctx->device));
    int LPL = lpl_for(D);
    if (LPL < 0) return fail(S2PB_ERR_UNSUPPORTED, "too many labels");
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
    Slot &s = ctx->slots[0];
    cudaStream_t st = s.stream;
    int rc = slot_ensure(ctx, s, w, h, DP, ndir, general ? 4 : 1);
    if (rc != S2PB_OK) return rc;
    ScratchLease L(ctx, st);
    float *dCf = L.take<float>(tot * 4);
    float *dS = S ? L.take<float>(tot * 4) : nullptr;
    float *dW = weights ? L.take<float>(npix * 4) : nullptr;
    if (!dCf || (S && !dS) || (weights && !dW)) return L.nomem("the aggregation");
    if (weights) CK(cudaMemcpyAsync(dW, weights, npix * 4, cudaMemcpyHostToDevice, st));
    short *dlo, *dhi;
    rc = upload_ranges(L, lo, hi, npix, gmin, D, st, &dlo, &dhi);
    if (rc != S2PB_OK) return rc;
    CK(cudaMemcpyAsync(dCf, C, tot * 4, cudaMemcpyHostToDevice, st));
    size_t totp = npix * DP;
    if (general) pad_cost_kernel<<<(unsigned)((totp + 255) / 256), 256, 0, st>>>(dCf, npix, D, DP, (float *)s.v[0].C);
    else pack_cost_kernel<<<(unsigned)((totp + 255) / 256), 256, 0, st>>>(dCf, npix, D, DP, (uint8_t *)s.v[0].C);
    ctx->launches++;
    CK(cudaGetLastError());
    const float *wgt[2] = {dW, nullptr};
    rc = launch_aggregate(ctx, s, 1, w, h, LPL, P1, P2, ndir, tsgm, nullptr, st, general, wgt);
    if (rc != S2PB_OK) return rc;
    s2pb_mgm_params prm;
    s2pb_default_params("mgm", &prm);
    prm.fix_overcount = fix_overcount; prm.refine = 0;
    WtaParams W;
    fill_wta(W, s.v[0], ndir, gmin, &prm, nullptr, npix);
    W.lo = dlo; W.hi = dhi;
    W.S = dS; W.Dout = D;
    rc = launch_wta(ctx, LPL, W, st, general);
    if (rc != S2PB_OK) return rc;
    CK(cudaMemcpyAsync(disp, s.v[0].disp, npix * 4, cudaMemcpyDeviceToHost, st));
    if (cost) CK(cudaMemcpyAsync(cost, s.v[0].cost, npix * 4, cudaMemcpyDeviceToHost, st));
    if (conf) CK(cudaMemcpyAsync(conf, s.v[0].conf, npix * 4, cudaMemcpyDeviceToHost, st));
    if (S) CK(cudaMemcpyAsync(S, dS, tot * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return S2PB_OK;
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
    CK(cudaSetDevice(ctx->device));
    size_t npix = (size_t)w * h;
    cudaStream_t st = ctx->slots[0].stream;
    ScratchLease L(ctx, st);
    float *a = L.take<float>(npix * 4), *b = L.take<float>(npix * 4);
    if (!a || !b) return L.nomem("the median");
    CK(cudaMemcpyAsync(a, in, npix * 4, cudaMemcpyHostToDevice, st));
    dim3 b2(32, 8);
    median_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(a, b, w, h, radius);
    ctx->launches++;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out, b, npix * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return S2PB_OK;
}

extern "C" int s2pb_remove_small_cc(s2pb_ctx *ctx, const float *in, float *out, int w, int h, int minarea)
{
    if (!ctx || !in || !out || w < 2 || h < 2) return fail(S2PB_ERR_ARG, "bad argument");
    CK(cudaSetDevice(ctx->device));
    size_t npix = (size_t)w * h;
    cudaStream_t st = ctx->slots[0].stream;
    ScratchLease L(ctx, st);
    float *a = L.take<float>(npix * 4), *b = L.take<float>(npix * 4);
    int *lab = L.take<int>(npix * 4), *area = L.take<int>(npix * 4);
    if (!a || !b || !lab || !area) return L.nomem("remove_small_cc");
    CK(cudaMemcpyAsync(a, in, npix * 4, cudaMemcpyHostToDevice, st));
    int rc = launch_remove_small_cc(ctx, a, b, w, h, minarea, lab, area, st);
    if (rc != S2PB_OK) return rc;
    CK(cudaMemcpyAsync(out, b, npix * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return S2PB_OK;
}

extern "C" int s2pb_erode_mask(s2pb_ctx *ctx, const uint8_t *in, uint8_t *out, int w, int h, float radius)
{
    if (!ctx || !in || !out || w < 1 || h < 1) return fail(S2PB_ERR_ARG, "bad argument");
    if (!(radius > 1.f) || radius > 64.f) return fail(S2PB_ERR_ARG, "disk radius must be in (1, 64]");   // build_disk, c/morsi.c:282
    CK(cudaSetDevice(ctx->device));
    size_t npix = (size_t)w * h;
    cudaStream_t st = ctx->slots[0].stream;
    ScratchLease L(ctx, st);
    uint8_t *a = L.take<uint8_t>(npix), *b = L.take<uint8_t>(npix);
    if (!a || !b) return L.nomem("the mask erosion");
    CK(cudaMemcpyAsync(a, in, npix, cudaMemcpyHostToDevice, st));
    dim3 b2(32, 8);
    erode_mask_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(a, b, w, h, radius);
    ctx->launches++;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out, b, npix, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return S2PB_OK;
}

extern "C" int s2pb_rejection_mask(s2pb_ctx *ctx, const float *disp, const float *im1, const float *im2, int w, int h, uint8_t *mask)
{
    if (!ctx || !disp || !im1 || !im2 || !mask || w < 1 || h < 1) return fail(S2PB_ERR_ARG, "bad argument");
    CK(cudaSetDevice(ctx->device));
    size_t npix = (size_t)w * h;
    cudaStream_t st = ctx->slots[0].stream;
    ScratchLease L(ctx, st);
    float *a = L.take<float>(npix * 4), *b = L.take<float>(npix * 4), *c = L.take<float>(npix * 4);
    uint8_t *m = L.take<uint8_t>(npix);
    if (!a || !b || !c || !m) return L.nomem("the rejection mask");
    CK(cudaMemcpyAsync(a, disp, npix * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(b, im1, npix * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(c, im2, npix * 4, cudaMemcpyHostToDevice, st));
    dim3 b2(32, 8);
    rejection_mask_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(a, b, c, w, h, m);
    ctx->launches++;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(mask, m, npix, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return S2PB_OK;
}

// ------------------------------------------------------------------ rectification warp

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
static void invert_homography(const double i[9], double o[9])
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
    int tw = w, th = h;
    if (useZ) {
        const float zoomIn = 1.0f / zoomOut;
        tw = (int)std::ceil((size_t)ow * zoomIn * 1.5);
        th = (int)std::ceil((size_t)oh * zoomIn * 1.5);
        if (tw < 1 || th < 1 || (size_t)tw * th > ((size_t)1 << 31)) return fail(S2PB_ERR_ARG, "homography: degenerate zoom %g", (double)zoomIn);
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
        gauss_rows_kernel<<<grid2d(tw, th, b2), b2, 0, st>>>(tmp, scratch, tw, th, K);
        gauss_cols_kernel<<<grid2d(tw, th, b2), b2, 0, st>>>(scratch, tmp, tw, th, K, jlim);
        ctx->launches += 2;
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
    nan_to_zero_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(tmp, n);
    dim3 bt(32, 8);
    // prefilter along x (on the transposed image) then along y; `a` holds the data, `b` is the other buffer
    auto prefilter = [&](float *a, float *b, int lw, int lh) {      // columns of an lw x lh image, result back in a
        if (lh >= 2 * kSplineSeg) {
            dim3 g((lw + 127) / 128, (lh + kSplineSeg - 1) / kSplineSeg);
            spline_segments_kernel<<<g, 128, 0, st>>>(a, b, lw, lh, lambda, z0);
            spline_segments_kernel<<<g, 128, 0, st>>>(b, a, lw, lh, 1.f, z1);
            ctx->launches += 2;
        } else {
            spline_columns_kernel<<<(lw + 31) / 32, 32, 0, st>>>(a, lw, lh, lambda, z0, z1);
            ctx->launches++;
        }
    };
    transpose_kernel<<<dim3((tw + 31) / 32, (th + 31) / 32), bt, 0, st>>>(tmp, tw, th, scratch);
    prefilter(scratch, tmp, th, tw);                                                // rows of the image
    transpose_kernel<<<dim3((th + 31) / 32, (tw + 31) / 32), bt, 0, st>>>(scratch, th, tw, tmp);
    prefilter(tmp, scratch, tw, th);
    Mat9 Hi;
    invert33(useZ ? matZ : M, Hi.m);
    spline_warp_kernel<<<grid2d(ow, oh, b2), b2, 0, st>>>(tmp, tw, th, Hi, d_out, ow, oh);
    ctx->launches += 4;
    if (useZ) {
        Mat9 Ht;
        invert33(M, Ht.m);
        warp_mask_kernel<<<grid2d(ow, oh, b2), b2, 0, st>>>(d_out, ow, oh, Ht, w, h);
        ctx->launches++;
    }
    CK(cudaGetLastError());
    return S2PB_OK;
}

// The part of `homography im -h "..." out w h` (3rdparty/homography/main.cpp:65-177) between reading and writing: needed
// region of the host image `src`, upload of that region only, crop compensation of H, warp into the DEVICE image d_out.
// Asynchronous on `st`; its scratch comes from the caller's lease.
static int warp_host_to_device(s2pb_ctx *ctx, ScratchLease &L, cudaStream_t st, const float *src, int sw, int sh, const double H[9],
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
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->slots[0].stream;
    ScratchLease L(ctx, st);
    float *out = L.take<float>((size_t)dw * dh * 4);
    if (!out) return L.nomem("the warp");
    int rc = warp_host_to_device(ctx, L, st, src, sw, sh, H, out, dw, dh);
    if (rc != S2PB_OK) return rc;
    CK(cudaMemcpyAsync(dst, out, (size_t)dw * dh * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
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
    if (!ctx || !src1 || !src2 || !H1 || !H2 || !disp || !conf || sw1 < 1 || sh1 < 1 || sw2 < 1 || sh2 < 1) return fail(S2PB_ERR_ARG, "bad argument");
    int rc = check_params(p, w, h, dmin, dmax);
    if (rc != S2PB_OK) return rc;
    CK(cudaSetDevice(ctx->device));
    Slot &s = ctx->slots[0];
    cudaStream_t st = s.stream;
    const size_t npix = (size_t)w * h;
    rc = slot_io_ensure(s, npix);
    if (rc != S2PB_OK) return rc;
    set_deadline(ctx, p->timeout_ms);
    ScratchLease L(ctx, st);
    rc = warp_host_to_device(ctx, L, st, src1, sw1, sh1, H1, s.d_in[0], w, h);
    if (rc == S2PB_OK) rc = warp_host_to_device(ctx, L, st, src2, sw2, sh2, H2, s.d_in[1], w, h);
    if (rc != S2PB_OK) return rc;
    if (rect1) CK(cudaMemcpyAsync(rect1, s.d_in[0], npix * 4, cudaMemcpyDeviceToHost, st));
    if (rect2) CK(cudaMemcpyAsync(rect2, s.d_in[1], npix * 4, cudaMemcpyDeviceToHost, st));
    rc = mgm_enqueue(ctx, s, s.d_in[0], s.d_in[1], w, h, dmin, dmax, p, s.d_disp, s.d_conf, mask ? s.d_mask : nullptr,
                     disp_right ? s.d_dispR : nullptr, st, -1);
    if (rc != S2PB_OK) return rc;
    CK(cudaMemcpyAsync(disp, s.d_disp, npix * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(conf, s.d_conf, npix * 4, cudaMemcpyDeviceToHost, st));
    if (mask) CK(cudaMemcpyAsync(mask, s.d_mask, npix, cudaMemcpyDeviceToHost, st));
    if (disp_right) CK(cudaMemcpyAsync(disp_right, s.d_dispR, npix * 4, cudaMemcpyDeviceToHost, st));
    return sync_or_timeout(ctx, st);
}

// ------------------------------------------------------------------ n-view merge (section 8f)

extern "C" int s2pb_merge_n(s2pb_ctx *ctx, const float *const *inputs, const double *offsets, int n, int w, int h, int op,
                            double threshold, float *out)
{
    if (!ctx || !inputs || !offsets || !out || n < 1 || w < 1 || h < 1) return fail(S2PB_ERR_ARG, "bad argument");
    if (n > kMaxFusion) return fail(S2PB_ERR_UNSUPPORTED, "at most %d rasters can be merged", kMaxFusion);
    const int sub_f32 = (op & S2PB_FUSE_SUB_F32) ? 1 : 0;
    op &= ~S2PB_FUSE_SUB_F32;
    if (op < FUSE_AVERAGE_IF_CLOSE || op >= FUSE_OP_COUNT) return fail(S2PB_ERR_ARG, "unknown averaging operator %d", op);
    CK(cudaSetDevice(ctx->device));
    const size_t npix = (size_t)w * h;
    cudaStream_t st = ctx->slots[0].stream;
    ScratchLease L(ctx, st);
    float *in = L.take<float>(npix * 4 * n), *o = L.take<float>(npix * 4);
    if (!in || !o) return L.nomem("the merge");
    FusionParams P;
    memset(&P, 0, sizeof P);
    double s = 0;
    for (int k = 0; k < n; k++) {
        if (!inputs[k]) return fail(S2PB_ERR_ARG, "null raster %d", k);
        P.in[k] = in + npix * k;
        CK(cudaMemcpyAsync((void *)P.in[k], inputs[k], npix * 4, cudaMemcpyHostToDevice, st));
        P.offset[k] = offsets[k];
        s += offsets[k];                     // np.mean of a short list: plain left-to-right sum / n
    }
    P.n = n; P.op = op; P.sub_f32 = sub_f32; P.threshold = threshold; P.mean_offset = s / n; P.npix = npix; P.out = o;
    fusion_kernel<<<(unsigned)((npix + 255) / 256), 256, 0, st>>>(P);
    ctx->launches++;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out, o, npix * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return S2PB_OK;
}

// ------------------------------------------------------------------ triangulation (section 8f)

static_assert(sizeof(s2pb_rpc) == sizeof(RpcModel), "s2pb_rpc must have the layout of the reference's struct rpc");

// Same argument list as the reference's ctypes entry point disp_to_lonlatalt (c/disp_to_h.c:70-76), plus the context.
extern "C" int s2pb_disp_to_lonlatalt(s2pb_ctx *ctx, double *lonlatalt, float *err, const float *dispx, const float *dispy,
                                      const float *msk, int nx, int ny, const float *msk_orig, int w, int h, const double ha[9],
                                      const double hb[9], const s2pb_rpc *rpca, const s2pb_rpc *rpcb, const float bbox[4])
{
    if (!ctx || !lonlatalt || !err || !dispx || !dispy || !msk || !msk_orig || !ha || !hb || !rpca || !rpcb || !bbox || nx < 1 ||
        ny < 1 || w < 1 || h < 1)
        return fail(S2PB_ERR_ARG, "bad argument");
    CK(cudaSetDevice(ctx->device));
    const size_t npix = (size_t)nx * ny, nm = (size_t)w * h;
    cudaStream_t st = ctx->slots[0].stream;
    ScratchLease L(ctx, st);
    float *d_dx = L.take<float>(npix * 4), *d_dy = L.take<float>(npix * 4), *d_m = L.take<float>(npix * 4), *d_mo = L.take<float>(nm * 4);
    double *d_out = L.take<double>(npix * 24);
    float *d_err = L.take<float>(npix * 4);
    if (!d_dx || !d_dy || !d_m || !d_mo || !d_out || !d_err) return L.nomem("the triangulation");
    CK(cudaMemcpyAsync(d_dx, dispx, npix * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_dy, dispy, npix * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_m, msk, npix * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_mo, msk_orig, nm * 4, cudaMemcpyHostToDevice, st));
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
    triangulate_kernel<<<grid2d(nx, ny, b2), b2, 0, st>>>(P);
    ctx->launches++;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(lonlatalt, d_out, npix * 24, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(err, d_err, npix * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return S2PB_OK;
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
        pc_count_kernel<true><<<g, b, smem, st>>>(xyz, nx, ny, r, p, count);
    } else {
        pc_count_kernel<false><<<g, b, 0, st>>>(xyz, nx, ny, r, p, count);
    }
    ctx->launches++;
    CK(cudaGetLastError());
    return S2PB_OK;
}

// Same argument list as the reference's count_3d_neighbors (c/disp_to_h.c:152), plus the context.
extern "C" int s2pb_count_3d_neighbors(s2pb_ctx *ctx, int32_t *count, const double *xyz, int nx, int ny, float r, int p)
{
    if (!ctx || !count || !xyz || nx < 1 || ny < 1) return fail(S2PB_ERR_ARG, "bad argument");
    const size_t npix = (size_t)nx * ny;
    if (npix > INT32_MAX) return fail(S2PB_ERR_UNSUPPORTED, "at most 2^31 - 1 points");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->slots[0].stream;
    ScratchLease L(ctx, st);
    double *d_xyz = L.take<double>(npix * 24);
    int *d_count = L.take<int>(npix * 4);
    if (!d_xyz || !d_count) return L.nomem("the point cloud");
    CK(cudaMemcpyAsync(d_xyz, xyz, npix * 24, cudaMemcpyHostToDevice, st));
    int rc = pc_count_enqueue(ctx, st, d_xyz, nx, ny, r, p, d_count);
    if (rc != S2PB_OK) return rc;
    CK(cudaMemcpyAsync(count, d_count, npix * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
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
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->slots[0].stream;
    ScratchLease L(ctx, st);
    double *d_xyz = L.take<double>(npix * 24);
    int *d_count = L.take<int>(npix * 4), *d_lab = L.take<int>(npix * 4), *d_saved = L.take<int>(npix * 4);
    if (!d_xyz || !d_count || !d_lab || !d_saved) return L.nomem("the point cloud");
    CK(cudaMemcpyAsync(d_xyz, xyz, npix * 24, cudaMemcpyHostToDevice, st));
    int rc = pc_count_enqueue(ctx, st, d_xyz, nx, ny, r, p, d_count);
    if (rc != S2PB_OK) return rc;
    const unsigned g1 = (unsigned)((npix + 255) / 256);
    const dim3 b2(32, 8), g2 = grid2d(nx, ny, b2);
    pc_label_kernel<<<g1, 256, 0, st>>>(d_count, (int)npix, n, d_lab, d_saved);
    ctx->launches++;
    if (q >= 0) {                                                       // q < 0: empty windows, nothing is saved
        q = std::min(q, std::max(nx, ny));
        pc_link_kernel<<<g2, b2, 0, st>>>(d_xyz, nx, ny, r, q, d_lab);
        cc_flatten_kernel<<<g1, 256, 0, st>>>((int)npix, d_lab);
        pc_mark_kernel<<<g2, b2, 0, st>>>(d_xyz, nx, ny, r, q, d_lab, d_saved);
        ctx->launches += 3;
    }
    pc_reject_kernel<<<g1, 256, 0, st>>>((int)npix, d_lab, d_saved, d_xyz);
    ctx->launches++;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(xyz, d_xyz, npix * 24, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return S2PB_OK;
}

// ------------------------------------------------------------------ sgbm (3rdparty/sgbm, sgbm_kernels.cuh)

extern "C" int s2pb_sgbm_default_params(s2pb_sgbm_params *p)
{
    if (!p) return fail(S2PB_ERR_ARG, "null params");
    p->win = 3; p->P1 = 8; p->P2 = 32; p->lr_diff = 1;       // what s2p passes: s2p/block_matching.py:116-134
    return S2PB_OK;
}

// The whole `sgbm im1 im2 disp cost dmin dmax win P1 P2 lr` run followed by create_rejection_mask, enqueued on `st`.
// d_im1 / d_im2 / d_disp: w*h float32, d_mask: w*h uint8 or null.  Its scratch comes from the caller's lease.
static int sgbm_enqueue(s2pb_ctx *ctx, ScratchLease &L, cudaStream_t st, const float *d_im1, const float *d_im2, int w, int h, int dmin,
                        int dmax, const s2pb_sgbm_params *p, float *d_disp, uint8_t *d_mask)
{
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

    SgbmState *d_st = L.take<SgbmState>(sizeof(SgbmState) + 512 * 4);
    unsigned *d_hist = (unsigned *)(d_st + 1);
    uint8_t *q1 = L.take<uint8_t>(ppix), *q2 = L.take<uint8_t>(ppix);
    short *pix = any ? L.take<short>(vol * 2) : nullptr, *C = any ? L.take<short>(vol * 2) : nullptr;
    short *disp1 = L.take<short>(ppix * 2), *dmed = L.take<short>(ppix * 2);
    unsigned long long *d2key = L.take<unsigned long long>(ppix * 8);
    int *lab = L.take<int>(ppix * 4), *area = L.take<int>(ppix * 4);
    if (!d_st || !q1 || !q2 || (any && (!pix || !C)) || !disp1 || !dmed || !d2key || !lab || !area) return L.nomem("the sgbm volumes");

    // qauto thresholds: four radix digits of both order statistics
    CK(cudaMemsetAsync(d_st, 0, sizeof(SgbmState) + 512 * 4, st));
    const int hblocks = (int)std::min<size_t>((npix + 255) / 256, (size_t)ctx->sm_count * 4);
    for (int digit = 3; digit >= 0; digit--) {
        sgbm_hist_kernel<<<hblocks, 256, 0, st>>>(d_im1, (int)npix, digit, d_st, d_hist);
        sgbm_select_kernel<<<1, 32, 0, st>>>(digit, d_st, d_hist);
        ctx->launches += 2;
    }
    sgbm_quantize_kernel<<<dim3((g.wp + 255) / 256, h), 256, 0, st>>>(d_im1, d_im2, w, h, off, g.wp, d_st, q1, q2);
    sgbm_fill_kernel<<<std::max(1, (int)std::min<size_t>((ppix + 255) / 256, 4096)), 256, 0, st>>>(disp1, ppix, (short)invalid);
    ctx->launches += 2;
    if (any) {
        CK(cudaFuncSetAttribute(sgbm_pixcost_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pix_smem));
        CK(cudaFuncSetAttribute(sgbm_path_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)path_smem));
        sgbm_pixcost_kernel<<<h, 256, pix_smem, st>>>(q1, q2, g, pix);
        const size_t rowel = (size_t)g.w1 * ND;
        sgbm_window_kernel<<<dim3((unsigned)std::min<size_t>((rowel + 255) / 256, 1024), h), 256, 0, st>>>(pix, g, C);
        short *S = pix;                                                  // the pixel costs are dead once C is formed
        CK(cudaMemsetAsync(S, 0, vol * 2, st));
        ctx->launches += 2;
        // pass 1 (top-down: predecessors left, up-left, up, up-right) and pass 2 (bottom-up, the mirrored four)
        static const int steps[8][2] = {{1, 0}, {1, 1}, {0, 1}, {-1, 1}, {-1, 0}, {1, -1}, {0, -1}, {-1, -1}};
        for (auto &s : steps) {
            const int nlines = s[1] == 0 ? h : s[0] == 0 ? g.w1 : g.w1 + h - 1;
            sgbm_path_kernel<<<(nlines + 3) / 4, 128, path_smem, st>>>(C, g, s[0], s[1], S);
            ctx->launches++;
        }
        CK(cudaMemsetAsync(d2key, 0xff, ppix * 8, st));
        const size_t nw = (size_t)g.w1 * h;
        sgbm_wta_kernel<<<(unsigned)((nw + 7) / 8), 256, 0, st>>>(S, g, disp1, d2key);
        sgbm_lr_kernel<<<dim3((g.w1 + 255) / 256, h), 256, 0, st>>>(disp1, d2key, g, lr);
        ctx->launches += 2;
    }
    const dim3 b2(32, 8);
    const unsigned g1 = (unsigned)((ppix + 255) / 256);
    sgbm_median_kernel<<<grid2d(g.wp, h, b2), b2, 0, st>>>(disp1, g.wp, h, dmed);
    sgbm_speckle_init_kernel<<<g1, 256, 0, st>>>(dmed, (int)ppix, invalid, lab, area);
    sgbm_speckle_link_kernel<<<grid2d(g.wp, h, b2), b2, 0, st>>>(dmed, g.wp, h, invalid, lab);
    cc_flatten_kernel<<<g1, 256, 0, st>>>((int)ppix, lab);
    cc_area_kernel<<<g1, 256, 0, st>>>((int)ppix, lab, area);
    sgbm_output_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(dmed, lab, area, g.wp, off, w, h, invalid, d_st, d_disp);
    ctx->launches += 6;
    if (d_mask) { rejection_mask_kernel<<<grid2d(w, h, b2), b2, 0, st>>>(d_disp, d_im1, d_im2, w, h, d_mask); ctx->launches++; }
    CK(cudaGetLastError());
    return S2PB_OK;
}

// `sgbm im1 im2 disp cost dmin dmax win P1 P2 lr` + create_rejection_mask from host buffers (pageable or page-locked)
extern "C" int s2pb_sgbm(s2pb_ctx *ctx, const float *im1, const float *im2, int w, int h, int dmin, int dmax,
                         const s2pb_sgbm_params *p, float *disp, uint8_t *mask)
{
    if (!ctx || !im1 || !im2 || !p || !disp || w < 1 || h < 1) return fail(S2PB_ERR_ARG, "bad argument");
    if (dmin >= dmax) return fail(S2PB_ERR_ARG, "mindisp(%d) > maxdisp(%d)", -dmax, -dmin);     // sgbm.cpp:174-177
    if (p->win < 1 || p->win % 2 == 0) return fail(S2PB_ERR_ARG, "SADWindowSize must be odd and positive (got %d)", p->win);
    const size_t npix = (size_t)w * h;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->slots[0].stream;
    ScratchLease L(ctx, st);
    float *d_im1 = L.take<float>(npix * 4), *d_im2 = L.take<float>(npix * 4), *d_disp = L.take<float>(npix * 4);
    uint8_t *d_mask = mask ? L.take<uint8_t>(npix) : nullptr;
    if (!d_im1 || !d_im2 || !d_disp || (mask && !d_mask)) return L.nomem("the sgbm images");
    CK(cudaMemcpyAsync(d_im1, im1, npix * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_im2, im2, npix * 4, cudaMemcpyHostToDevice, st));
    int rc = sgbm_enqueue(ctx, L, st, d_im1, d_im2, w, h, dmin, dmax, p, d_disp, d_mask);
    if (rc != S2PB_OK) return rc;
    CK(cudaMemcpyAsync(disp, d_disp, npix * 4, cudaMemcpyDeviceToHost, st));
    if (mask) CK(cudaMemcpyAsync(mask, d_mask, npix, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return S2PB_OK;
}
