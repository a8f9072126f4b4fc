// host.h -- host-side state and helpers shared by the translation units of the C ABI (not a public header).
//
// s2pb200.cu owns the context, the slots, the matcher and the matcher's stage entry points; warp.cu, geometry.cu, projection.cu,
// sgbm.cu, raster.cu, cloud.cu, mosaic.cu, pair_tile.cu and heights_tile.cu each hold one family of entry points.  Every kernel header that defines a non-template kernel is included by one of
// those files only, so that its kernels are compiled once; the few launchers another file needs are declared at the end.
#pragma once
#include "../../include/s2pb200.h"
#include "agg_kernel.cuh"          // kMaxPasses
#include "projection_kernels.cuh"  // GeoidGrid

#include <cuda_runtime.h>
#include <algorithm>
#include <atomic>
#include <list>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

namespace s2pb { struct RtState; struct OrderStats; }
using namespace s2pb;            // every file that includes this one launches the kernels of namespace s2pb

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
    float *L[kMaxPasses];  // resident layout: one volume per pass
    float *S;              // folded layout (FoldView, agg_kernel.cuh): the running sum of the passes [H][W][DP],
    float *Lb;             // ... the band-closing scanlines of the pass in flight,
    short *am[kMaxPasses]; // ... and each pass's last arg-minimum [H][W]
    float *Lmin[kMaxPasses];
    int *progress;         // [kMaxPasses][maxBands]
    float *disp, *cost, *conf, *tmp;
};
struct Slot {
    void *base = nullptr;
    size_t bytes = 0;
    int w = 0, h = 0, DP = 0, ndir = 0;
    int cbytes = 1;               // bytes per stored cost: 1 = 8-bit census codes, 4 = float (general flavour)
    bool folded = false;          // the workspace holds the folded layout (slot_ensure picks it when the resident one does not fit)
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
    int *abort = nullptr;         // this slot's word of s2pb_ctx::abort_words: a timeout of a call on this slot raises it
    bool timed = false;
    bool direct_out = false;      // the last host-API call wrote its results straight into the caller's pinned buffers
    // K-panels of the DCT tables that are not resident (dct_tables, dct_product; a resident table is multiplied as one panel):
    // two pinned staging buffers and two device panels of `panel` doubles each, the copy stream and its events, and the running
    // sums of the round trip's inverse product (acc_pix doubles); allocated on first use
    struct DctStream {
        double *h[2] = {nullptr, nullptr}, *d[2] = {nullptr, nullptr};
        size_t panel = 0;
        cudaStream_t copy = nullptr;
        cudaEvent_t copied[2] = {}, consumed[2] = {};
        double *acc = nullptr;
        size_t acc_pix = 0;
    } dcts;
};
struct s2pb_ctx {
    int device = 0;
    int sm_count = 132;
    bool wta_prune = true;         // S2PB_WTA_PRUNE (read when the context is created): 0 wta_kernel for every shape, the
                                   // same-device reference of wta_pruned_kernel (DESIGN.md 3.2); unset or any other value prunes
    std::vector<Slot> slots;
    // pinned + mapped, one word per slot (Slot::abort; at most 64 slots): the persistent aggregation kernels of a slot stop
    // waiting on band hand-offs while its word is raised, so a timed-out call drains without touching other slots' calls
    int *abort_words = nullptr;
    std::atomic<long long> launches{0};   // (mgm_multi tiles of a batch are enqueued from several host threads)
    size_t ws_limit = 0;                  // s2pb_set_workspace_limit: bytes per workspace, 0 = none
    std::atomic<long long> folded_calls{0};   // mgm_calls that ran in the folded layout (s2pb_folded_calls)
    // DCT coefficient tables of the matched image's round trip, one entry per image width (dct_tables); every product runs
    // through dct_gemm_kernel, a table held here as one panel, a null table (only above kDctDenseWidth) streamed in K-panels
    struct DctTab { int n; double *T10, *T01, *TR01, *mc, *ms; };
    size_t dct_limit = (size_t)8 << 30;   // s2pb_set_dct_table_limit: device bytes of resident tables above kDctDenseWidth
    size_t dct_wide_bytes = 0;            // ... held now
    std::list<DctTab> dct;          // a list: entries stay put while other host threads hold pointers to them
    std::mutex dct_mu;
    // scratch pool of the host-buffer entry points: device buffers are kept between calls (a cudaMalloc / cudaFree pair per
    // call costs more than the merge or the warp itself).  Borrowed through a ScratchLease only.  It has no lock, so nothing
    // that s2pb_mgm_batch's worker threads run may take from it.
    struct PoolBuf { void *p; size_t bytes; bool used; };
    std::vector<PoolBuf> pool;
    GeoidGrid geoid{};              // s2pb_set_geoid: the EGM96 grid of S2PB_ZONE_EGM96 (geoid.g null: none), owned
    MapKind proj_kind = MapKind::kNone;   // s2pb_set_projection: the map of S2PB_ZONE_PROJ (kNone: none) and its parameters
    MapParams proj{};
};

// nothing declared from here on is part of the library's exported interface
#pragma GCC visibility push(hidden)

// ------------------------------------------------------------------ errors

extern thread_local std::string g_err;
int fail(int code, const char *fmt, ...);
#define CK(call)                                                                                     \
    do {                                                                                             \
        cudaError_t e_ = (call);                                                                     \
        if (e_ != cudaSuccess)                                                                       \
            return fail(S2PB_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

// ------------------------------------------------------------------ scratch of the host-buffer entry points

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// smallest idle pooled buffer that is large enough, else a new allocation; when that fails the idle buffers are given back
// to the device and the allocation is tried once more (nullptr when out of memory)
inline void *pool_take(s2pb_ctx *ctx, size_t bytes)
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

// The protocol of an entry point that works on host buffers: it runs on slot 0's stream of the context's device and borrows
// its scratch through the lease it is.  take() and upload() (scratch holding a copy of a host buffer) keep the first failure
// and do nothing after it; the caller returns error() if it is set before its first launch, downloads its results and returns
// finish(), the checked synchronisation of the stream.
class HostCall : public ScratchLease {
public:
    const cudaStream_t st;
    // what: the call's scratch, as the message of a failed allocation names it
    HostCall(s2pb_ctx *ctx, const char *what) : ScratchLease(ctx, ctx->slots[0].stream), st(ctx->slots[0].stream), what_(what)
    {
        keep(cudaSetDevice(ctx->device), "cudaSetDevice");
    }
    template <class T> T *take(size_t bytes)
    {
        T *p = rc_ != S2PB_OK ? nullptr : ScratchLease::take<T>(bytes);
        if (!p && rc_ == S2PB_OK) rc_ = nomem(what_);
        return p;
    }
    template <class T> T *upload(const T *src, size_t bytes)
    {
        T *p = take<T>(bytes);
        if (p) keep(cudaMemcpyAsync(p, src, bytes, cudaMemcpyHostToDevice, st), "host-to-device copy");
        return p;
    }
    void download(void *dst, const void *src, size_t bytes)
    {
        if (rc_ == S2PB_OK) keep(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, st), "device-to-host copy");
    }
    int error() const { return rc_; }
    int finish()
    {
        if (rc_ != S2PB_OK) return rc_;
        CK(cudaStreamSynchronize(st));
        return S2PB_OK;
    }

private:
    void keep(cudaError_t e, const char *what)
    {
        if (e != cudaSuccess && rc_ == S2PB_OK) rc_ = fail(S2PB_ERR_CUDA, "%s failed: %s", what, cudaGetErrorString(e));
    }
    const char *what_;
    int rc_ = S2PB_OK;        // the first failure
};

// ------------------------------------------------------------------ launches

// kernel k<<<grid, block, smem, st>>>(args...), counted in s2pb_kernel_launches
template <class... P, class... A>
inline void launch(s2pb_ctx *ctx, void (*k)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A &&...args)
{
    k<<<grid, block, smem, st>>>(std::forward<A>(args)...);
    ctx->launches++;
}

inline dim3 grid2d(int w, int h, dim3 b) { return dim3((w + b.x - 1) / b.x, (h + b.y - 1) / b.y); }

// bytes of a value of PLY property type S2PB_PLY_*, 0 for an unknown type
inline int ply_type_bytes(int type)
{
    switch (type) {
    case S2PB_PLY_F64: return 8;
    case S2PB_PLY_F32: case S2PB_PLY_I32: case S2PB_PLY_U32: return 4;
    case S2PB_PLY_I16: case S2PB_PLY_U16: return 2;
    case S2PB_PLY_U8: case S2PB_PLY_I8: return 1;
    default: return 0;
    }
}

// ------------------------------------------------------------------ shared between the translation units

// s2pb200.cu: remove_small_cc and the union-find passes it shares with the 3D filter and sgbm (multiscale_kernels.cuh), and
// create_rejection_mask (mgm_kernels.cuh)
int launch_remove_small_cc(s2pb_ctx *ctx, const float *in, float *out, int w, int h, int minarea, float thr, int *lab, int *area,
                           cudaStream_t st);
void cc_flatten(s2pb_ctx *ctx, int n, int *lab, cudaStream_t st);
void cc_area(s2pb_ctx *ctx, int n, const int *lab, int *area, cudaStream_t st);
void launch_rejection_mask(s2pb_ctx *ctx, const float *disp, const float *im1, const float *im2, int w, int h, uint8_t *mask,
                           cudaStream_t st);
// s2pb200.cu: morsi's disk erosion of a device mask (erode_radius_ok: the radii s2pb_erode_mask accepts); the matcher of
// s2pb_mgm_weighted between device buffers on slot 0, st being that slot's stream (the deadline of p->timeout_ms counts from the
// call, which waits for st through it: S2PB_ERR_TIMEOUT); d_wl / d_wr: device weight images or null
int erode_radius_ok(float radius);
void launch_erode_mask(s2pb_ctx *ctx, const uint8_t *in, uint8_t *out, int w, int h, float radius, cudaStream_t st);
int mgm_match_device(s2pb_ctx *ctx, cudaStream_t st, const float *d_im1, const float *d_im2, int w, int h, int dmin, int dmax,
                     const s2pb_mgm_params *p, const float *d_wl, const float *d_wr, float *d_disp, float *d_conf, uint8_t *d_mask,
                     float *d_dispR);
// projection.cu: the output CRS of a cloud, `zone` and `south` as the C ABI takes them (a UTM zone, 0 for none when zone0 is
// true, or S2PB_ZONE_PROJ with south 0 when zone0 is true and the context holds a projection; optionally with S2PB_ZONE_EGM96
// when it holds a geoid grid): its check, and the projection of n device points (lon, lat, alt) to it, in place when
// d_in == d_out (nothing to launch for zone 0 without the geoid)
int cloud_crs_ok(const s2pb_ctx *ctx, int zone, int south, bool zone0);
int launch_cloud_project(s2pb_ctx *ctx, cudaStream_t st, int zone, bool south, const double *d_in, double *d_out, size_t n);
// the context's geoid grid back to the device (s2pb_destroy, s2pb_set_geoid)
void geoid_free(s2pb_ctx *ctx);
// geometry.cu: the two clouds of a host call, each from host buffers into scratch of L after the checks of its arguments, then
// projected in place to the output CRS `zone` (launch_cloud_project).  triangulated_cloud: disp_to_lonlatalt of s2pb_disp_to_xyz's inputs, *d_xyz
// nx*ny*3 doubles and *d_err nx*ny floats, still in flight on L.st.  localised_cloud: s2pb_height_map_to_xyz's localisation,
// *d_xyz w*h*3 doubles, complete on return (the pixels whose iteration hit its cap are an error).  remove_isolated_3d_points
// (n > 0; d_work: 3 * nx * ny ints) on device buffers.
int triangulated_cloud(s2pb_ctx *ctx, HostCall &L, const float *dispx, const float *dispy, const float *msk, int nx, int ny,
                       const float *msk_orig, int w, int h, const double ha[9], const double hb[9], const s2pb_rpc *rpca,
                       const s2pb_rpc *rpcb, const float bbox[4], int zone, int south, double **d_xyz, float **d_err);
// triangulated_cloud_device: the same from device disparities and masks, after triangulated_cloud_args_ok checked the rest.
int triangulated_cloud_args_ok(const s2pb_ctx *ctx, int nx, int ny, int w, int h, const double ha[9], const double hb[9], const s2pb_rpc *rpca,
                               const s2pb_rpc *rpcb, const float bbox[4], int zone, int south);
int triangulated_cloud_device(s2pb_ctx *ctx, HostCall &L, const float *d_dx, const float *d_dy, const float *d_m, int nx, int ny,
                              const float *d_mo, int w, int h, const double ha[9], const double hb[9], const s2pb_rpc *rpca,
                              const s2pb_rpc *rpcb, const float bbox[4], int zone, int south, double **d_xyz, float **d_err);
int localised_cloud(s2pb_ctx *ctx, HostCall &L, const double *heights, int w, int h, const s2pb_rpc *rpc, double off_x,
                    double off_y, int zone, int south, double **d_xyz);
// localised_cloud_device: the same from device heights d_z, after localised_cloud_args_ok checked the rest.
int localised_cloud_args_ok(const s2pb_ctx *ctx, int w, int h, const s2pb_rpc *rpc, int zone, int south);
int localised_cloud_device(s2pb_ctx *ctx, HostCall &L, const double *d_z, int w, int h, const s2pb_rpc *rpc, double off_x,
                           double off_y, int zone, int south, double **d_xyz);
// s2pb_height_map from the device disparity d_dx and mask d_m (nx*ny) and the unpadded device mask_orig d_mo0 (mw*mh) into the
// device heights d_out (w*h), in flight on L.st, after height_map_args_ok checked its arguments.
int height_map_args_ok(int nx, int ny, int mw, int mh, int x, int y, int w, int h, const double H1[9], const double H2[9],
                       const s2pb_rpc *rpc1, const s2pb_rpc *rpc2);
int height_map_device(s2pb_ctx *ctx, HostCall &L, const float *d_dx, const float *d_m, int nx, int ny, const float *d_mo0, int mw,
                      int mh, int x, int y, int w, int h, const double H1[9], const double H2[9], const s2pb_rpc *rpc1,
                      const s2pb_rpc *rpc2, double *d_out);
// s2pb_cargarse_basura of a device w*h float32 image into d_out (d_m: w*h floats, lab and area: w*h ints of scratch), after
// basura_args_ok
int basura_args_ok(int w, int h);
int basura_enqueue(s2pb_ctx *ctx, cudaStream_t st, const float *d_in, float *d_out, int w, int h, float *d_m, int *lab, int *area);
int remove_isolated_enqueue(s2pb_ctx *ctx, cudaStream_t st, double *d_xyz, int nx, int ny, float r, int p, int n, int q, int *d_work);
// sgbm.cu: order statistics of the non-NaN values of n device floats by radix select (sgbm_kernels.cuh) into d_os, which
// holds order_stats_bytes(); rule kOrdQauto (qauto's thresholds) or kOrdLinear (numpy's 'linear' quantiles q0 and q1)
size_t order_stats_bytes();
int launch_order_stats(s2pb_ctx *ctx, cudaStream_t st, const float *d_x, int n, int rule, double q0, double q1, OrderStats *d_os);
// the `sgbm` run and its rejection mask on device buffers of L (see s2pb_sgbm for what it refuses)
int sgbm_enqueue(s2pb_ctx *ctx, HostCall &L, const float *d_im1, const float *d_im2, int w, int h, int dmin, int dmax,
                 const s2pb_sgbm_params *p, float *d_disp, uint8_t *d_mask);
// cloud.cu: the checks of the cloud steps' tail arguments (colours, pct, records) and of a clr image's bands and type, and the
// tail itself on device inputs -- 3D filter, colours (d_typed planes of cb-byte values copied, else the float32 planes d_bands
// stretched with pct), confidence (nullable) -- down to the records and their number in host memory, synchronised
int tail_args_ok(s2pb_ctx *ctx, int nx, int ny, const float *bands, int nbands, double pct, uint8_t *records, int64_t *npoints);
int typed_colours_ok(int nbands, int color_type);
int cloud_tail_device(s2pb_ctx *ctx, HostCall &L, double *d_xyz, int nx, int ny, float r, int p, int n, const float *d_bands,
                      int nbands, double pct, const uint8_t *d_typed, int cb, const float *d_conf, uint8_t *records, int64_t *npoints);
// raster.cu: s2pb_merge_n's checks of n and op, and its merge of n device rasters (float32, or float64 when f64) into d_out
int fusion_args_ok(int n, int op);
void fusion_enqueue(s2pb_ctx *ctx, cudaStream_t st, const void *const *d_in, bool f64, const double *offsets, int n, size_t npix,
                    int op, double threshold, float *d_out);
// warp.cu
void invert_homography(const double i[9], double o[9]);
int warp_host_to_device(s2pb_ctx *ctx, ScratchLease &L, cudaStream_t st, const float *src, int sw, int sh, const double H[9],
                        float *d_out, int dw, int dh);

#pragma GCC visibility pop
