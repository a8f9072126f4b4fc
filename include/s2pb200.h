/* s2pb200.h -- C ABI of the H100-native stereo engine that drops in behind s2p.
 *
 * Plain C, plain pointers and sizes, no torch / numpy types.  The library
 * (s2p_b200/libs2pb200.so, sources in s2p_b200/csrc/) is loaded with
 * ctypes.CDLL exactly like the reference loads its own native helpers
 * (s2p/triangulation.py:18-20, s2p/sift.py:25-26).  INTEGRATION.md shows the
 * binding a maintainer of the reference would add.
 *
 * What each entry point replaces in the reference (paths relative to the root of the s2p sources):
 *
 *   s2pb_mgm()           the `mgm` / `mgm_multi` subprocess + the three
 *                        plambda/backflow subprocesses of create_rejection_mask
 *                        (s2p/block_matching.py:18-32,155-188,269-310;
 *                         3rdparty/mgm_multi/main_mgm.cc:80-266,
 *                         main_mgm_multi.cc:88-256)
 *   s2pb_homography()    the `homography` subprocess run by
 *                        common.image_apply_homography (s2p/common.py:159-180;
 *                        3rdparty/homography/main.cpp:65-177)
 *   s2pb_mgm_batch()     the per-(tile,pair) fan-out of stereo_matching through
 *                        parallel.launch_calls (s2p/__init__.py:166-196,586-591)
 *   s2pb_sgbm()          the `sgbm` subprocess (OpenCV 2's StereoSGBM, 3rdparty/sgbm) + create_rejection_mask
 *                        (s2p/block_matching.py:116-134)
 *
 * Conventions: all images are single-band, row-major, C-contiguous float32,
 * NaN = no data.  Disparity d at ref pixel (x,y) means the match is at
 * (x+d, y) in the secondary image.  Every function returns S2PB_OK (0) or a
 * negative error code; s2pb_last_error() gives the message (thread local).
 * There is no CPU fallback: without a CUDA device every compute call fails with
 * S2PB_ERR_CUDA.
 */
#ifndef S2PB200_H
#define S2PB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define S2PB_VERSION 101

enum {
    S2PB_OK = 0,
    S2PB_ERR_CUDA = -1,      /* CUDA runtime / kernel failure, or no device          */
    S2PB_ERR_ARG = -2,       /* invalid argument (the reference would exit non-zero)  */
    S2PB_ERR_TIMEOUT = -3,   /* params.timeout_ms exceeded -> subprocess.TimeoutExpired */
    S2PB_ERR_NOMEM = -4,     /* tile does not fit the device workspace                */
    S2PB_ERR_UNSUPPORTED = -5
};

/* Matcher parameters.  In the reference these travel as argv + environment
 * "smart parameters" (3rdparty/mgm_multi/smartparameter.h:27-51); the comment
 * on each field names the flag it mirrors. */
typedef struct s2pb_mgm_params {
    int32_t ndir;            /* -O           number of scan passes: 2, 4 or 8            */
    int32_t tsgm;            /* TSGM         neighbours mixed per pass: 1..4             */
    int32_t census_win;      /* CENSUS_NCC_WIN  census window side: 3, 5 or 7            */
    float   P1;              /* -P1                                                       */
    float   P2;              /* -P2                                                       */
    int32_t median;          /* MEDIAN       radius of the median post-filter, 0 = off    */
    int32_t lr_mode;         /* TESTLRRL     0 off, 1 per scale, 2 once at the end        */
    float   lr_tau;          /* TESTLRRL_TAU                                              */
    float   mindiff;         /* MINDIFF      < 0 = off                                    */
    int32_t remove_small_cc; /* REMOVESMALLCC  0 = off                                    */
    int32_t subpix;          /* SUBPIX       1, or 2 for the half-pixel pass (mgm_multi)  */
    int32_t scales;          /* -S           < 0: single-scale `mgm`; >= 0: `mgm_multi`   */
    int32_t refine;          /* -s           0 none, 1 vfit, 2 parabola                   */
    int32_t fix_overcount;   /* TSGM_FIX_OVERCOUNT                                        */
    int32_t timeout_ms;      /* <= 0: none.  mirrors common.run(timeout=) for mgm*        */
    int32_t cost;            /* -t           S2PB_COST_*: census (what s2p passes), ad, sd, ncc, btad, btsd */
} s2pb_mgm_params;

/* -t: the distances of the reference's table (3rdparty/mgm_multi/mgm_costvolume.h:186-197).  census uses the
 * census prefilter (mgm_costvolume.cc:98-102), the others work on the images; ncc's window is census_win. */
enum { S2PB_COST_CENSUS = 0, S2PB_COST_AD, S2PB_COST_SD, S2PB_COST_NCC, S2PB_COST_BTAD, S2PB_COST_BTSD, S2PB_COST_COUNT };

typedef struct s2pb_ctx s2pb_ctx;   /* one per (process, GPU); not thread safe */

/* ---- library / context ---------------------------------------------------- */
int          s2pb_version(void);
const char  *s2pb_last_error(void);
int          s2pb_device_count(void);               /* 0 if no usable CUDA device */
/* CUDA is initialised here, never at load time, so a forked multiprocessing
 * worker (s2p/parallel.py:80) can create its context after the fork. */
s2pb_ctx    *s2pb_create(int device);
void         s2pb_destroy(s2pb_ctx *ctx);
/* algo = "mgm" or "mgm_multi": the values s2p sets at s2p/block_matching.py:155-186,269-308 */
int          s2pb_default_params(const char *algo, s2pb_mgm_params *p);

/* ---- the matcher ----------------------------------------------------------- */
/* Host buffers in, host buffers out (H2D/D2H inside).  disp, conf: w*h float32;
 * mask: w*h uint8 (0 rejected / 1 accepted) or NULL; disp_right: w*h or NULL.
 * Up to 2048 labels per view's volume (an mgm_multi level: its label hull), for every distance, with or without
 * weights; wider volumes fail with S2PB_ERR_UNSUPPORTED.
 * Buffers may be pageable or page-locked (cudaHostAlloc / cudaHostRegister): page-locked
 * ones are used for the DMA directly, pageable ones are staged through the library's own
 * pinned block. */
int s2pb_mgm(s2pb_ctx *ctx, const float *im1, const float *im2, int w, int h,
             int dmin, int dmax, const s2pb_mgm_params *p,
             float *disp, float *conf, uint8_t *mask, float *disp_right);

/* s2pb_mgm with the regularity weight images of `-wl` / `-wr` (main_mgm.cc:139-140,219-222; what
 * algo == 'mgm_multi_lsd' passes, s2p/block_matching.py:191-266): wl, wr = w*h float32 each, both or neither.
 * Every penalty of pixel p is multiplied by w(p) (mgm_weights.h:92-110, mgm_core.cc:981-992); in mgm_multi the
 * weight maps follow the pyramid (mgm_multiscale.cc:375-378) and the half-pixel pass runs unweighted
 * (main_mgm_multi.cc:207). */
int s2pb_mgm_weighted(s2pb_ctx *ctx, const float *im1, const float *im2, int w, int h,
                      int dmin, int dmax, const s2pb_mgm_params *p, const float *wl, const float *wr,
                      float *disp, float *conf, uint8_t *mask, float *disp_right);

/* `mgm ... -confidence_pkrL f -confidence_pkrR g` (3rdparty/mgm_multi/main_mgm.cc:147,250-262, main_mgm_multi.cc likewise):
 * s2pb_mgm plus the peak-ratio confidence of both views (compute_PKR_confidence, mgm_costvolume.cc:199-214: second minimum of
 * the aggregated cost more than 2 labels away from the winner, over max(first minimum, 0.01)).  With scales >= 0 the images
 * are those of the full-resolution ZOOM = 1 call, as in mgm_multi.  s2p itself never requests them. */
int s2pb_mgm_pkr(s2pb_ctx *ctx, const float *im1, const float *im2, int w, int h, int dmin, int dmax,
                 const s2pb_mgm_params *p, float *disp, float *conf, uint8_t *mask, float *disp_right,
                 float *pkr_left, float *pkr_right);

/* Same, device pointers on both sides, enqueued on `stream` (a cudaStream_t
 * passed as void*, NULL = the context's own stream) and NOT synchronised when
 * timeout_ms <= 0.  `slot` selects one of the context's workspaces
 * (0 <= slot < s2pb_num_slots) so that several tiles can be in flight.
 * nodata_hint: bit 1 = the secondary image may hold NaN pixels (the reference
 * then gives them the label range [dmin, dmin+1], main_mgm.cc:214-216, which can
 * widen the right view's volume); 0 = neither image holds NaN; < 0 = unknown, the
 * library inspects the image (one stream synchronisation). */
int s2pb_mgm_device(s2pb_ctx *ctx, int slot, const float *d_im1, const float *d_im2,
                    int w, int h, int dmin, int dmax, const s2pb_mgm_params *p,
                    float *d_disp, float *d_conf, uint8_t *d_mask, float *d_disp_right,
                    int nodata_hint, void *stream);

/* n independent tiles of identical shape, pipelined over the context's slots
 * (staging or direct DMA as above, H2D / compute / D2H of different tiles overlap).
 * Arrays of n host pointers.  For the multi-scale algorithms (scales >= 0), which read a
 * label hull back at every pyramid level, the tiles are driven by one host thread per
 * workspace inside the call (at most four); a context may also be used from several
 * caller threads as long as each uses its own slot. */
int s2pb_mgm_batch(s2pb_ctx *ctx, int n, const float *const *im1, const float *const *im2,
                   int w, int h, int dmin, int dmax, const s2pb_mgm_params *p,
                   float *const *disp, float *const *conf, uint8_t *const *mask);

/* Reserve `nslots` workspaces for tiles up to w x h x (dmax-dmin+1) labels.
 * Optional: s2pb_mgm* grow the workspace on demand. */
int s2pb_reserve(s2pb_ctx *ctx, int nslots, int w, int h, int nlabels);
int s2pb_num_slots(const s2pb_ctx *ctx);
int s2pb_sync(s2pb_ctx *ctx);

/* ---- the `sgbm` matcher (3rdparty/sgbm/sgbm.cpp + stereosgbm.cpp) ----------------- */
/* The binary's argv after dmin dmax (`sgbm im1 im2 disp cost dmin dmax win P1 P2 lr`).  What it hardcodes stays
 * constant: fullDP, preFilterCap 63, uniquenessRatio 10, speckle window 50 and range 1, median 3x3. */
typedef struct s2pb_sgbm_params {
    int32_t win;             /* SADwindow    odd window side                                      */
    int32_t P1;              /* P1           <= 0: 2 (stereosgbm.cpp:334)                         */
    int32_t P2;              /* P2           <= 0: 5; at least P1 + 1                             */
    int32_t lr_diff;         /* LRdiff       disp12MaxDiff; <= 0: 1                               */
} s2pb_sgbm_params;
/* what s2p passes: win 3, P1 8, P2 32, lr_diff 1 */
int s2pb_sgbm_default_params(s2pb_sgbm_params *p);
/* Bit for bit the disparity the `sgbm` binary writes (NaN = rejected; the padding of its crop trick taken as zero),
 * then the rejection mask of s2pb_mgm.  disp: w*h float32; mask: w*h uint8 or NULL.  Host buffers, pageable or
 * page-locked; synchronous.  S2PB_ERR_ARG: dmin >= dmax or an even / non-positive win, as the binary.
 * S2PB_ERR_UNSUPPORTED: disparities x16 outside int16, or win^2 * 189 + 2 * P2 > 32767 or P2 > 4096 (int16 path costs). */
int s2pb_sgbm(s2pb_ctx *ctx, const float *im1, const float *im2, int w, int h, int dmin, int dmax,
              const s2pb_sgbm_params *p, float *disp, uint8_t *mask);

/* ---- rectification warp ---------------------------------------------------- */
/* dst(j,i) = src sampled at H^-1 (j,i,1), order-5 B-spline with the reference's
 * anti-aliasing rule (3rdparty/homography/LibHomography/Homography.cpp:50-168). */
int s2pb_homography(s2pb_ctx *ctx, const float *src, int sw, int sh,
                    const double H[9], float *dst, int dw, int dh);

/* ---- steps 3 + 4 of a tile without leaving the device (SURVEY.md section 8f rank 3) ---- */
/* rectify_pair's two warps (s2p/rectification.py:379-380 -> common.image_apply_homography) followed by
 * compute_disparity_map (s2p/__init__.py:184-190) in one call: src1 / src2 are the (crops of the) original images, H1 / H2
 * the rectifying homographies in their pixel coordinates; both are warped into the matcher's device inputs and matched there.
 * rect1 / rect2 (nullable): host copies of the rectified pair, for the files later steps read.  Results are identical to
 * s2pb_homography x 2 followed by s2pb_mgm. */
int s2pb_rectify_match(s2pb_ctx *ctx, const float *src1, int sw1, int sh1, const double H1[9],
                       const float *src2, int sw2, int sh2, const double H2[9], int w, int h, int dmin, int dmax,
                       const s2pb_mgm_params *p, float *rect1, float *rect2, float *disp, float *conf, uint8_t *mask,
                       float *disp_right);

/* ---- n-view merge (a "next" row of SURVEY.md section 8f) ---------------------- */
/* s2p.fusion.merge_n (s2p/fusion.py:25-68) from memory to memory: out = op_k(inputs[k] - offsets[k]) +
 * mean(offsets), pixelwise in float64, stored as float32.  op: 0 average_if_close (NaN when
 * nanmax - nanmin > threshold, else nanmedian; s2p/fusion.py:16-23), 1 nanmedian, 2 nanmean, 3 nanmin, 4 nanmax,
 * 5 median, 6 mean, 7 min, 8 max (the reducers s2p/fusion.py:31-36 names).  OR-ing S2PB_FUSE_SUB_F32 into op performs
 * the subtraction in float32, which is what `f.read(1) - offsets[i]` does under NumPy < 2 (value-based casting of
 * the 0-d float64 offset); without it the subtraction is in float64 (NumPy >= 2). */
#define S2PB_FUSE_SUB_F32 0x100
int s2pb_merge_n(s2pb_ctx *ctx, const float *const *inputs, const double *offsets, int n, int w, int h,
                 int op, double threshold, float *out);

/* ---- triangulation (a "next" row of SURVEY.md section 8f) --------------------- */
/* Rational polynomial camera model: the reference's `struct rpc` (c/rpc.h:14-32) field for field, which is also
 * the layout of s2p.triangulation.RPCStruct (s2p/triangulation.py:23-40). */
typedef struct s2pb_rpc {
    double numx[20], denx[20], numy[20], deny[20], scale[3], offset[3];
    double inumx[20], idenx[20], inumy[20], ideny[20], iscale[3], ioffset[3];
    double dmval[4], imval[4];
    double delta;
} s2pb_rpc;
/* Same argument list as lib/disp_to_h.so's disp_to_lonlatalt (c/disp_to_h.c:70-76), which
 * s2p.triangulation.disp_to_xyz calls through ctypes (s2p/triangulation.py:118-143), plus the context. */
int s2pb_disp_to_lonlatalt(s2pb_ctx *ctx, double *lonlatalt, float *err, const float *dispx, const float *dispy,
                           const float *msk, int nx, int ny, const float *msk_orig, int w, int h,
                           const double ha[9], const double hb[9], const s2pb_rpc *rpca, const s2pb_rpc *rpcb,
                           const float orig_img_bounding_box[4]);

/* The 3D outlier filter of s2p.triangulation.filter_xyz (s2p/triangulation.py:275-343): same argument lists as
 * lib/disp_to_h.so's count_3d_neighbors and remove_isolated_3d_points (c/disp_to_h.c:152-230), plus the context.
 * xyz: nx*ny points of three doubles, row-major.  count[y*nx+x] = number of points of the (2p+1)^2 window, clipped at
 * the border, whose squared distance (differences in double, rounded to float, summed in float) is < r*r.
 * remove_isolated_3d_points rejects the points with count < n, saves every rejected point joined to a kept one by a chain
 * of close points within (2q+1)^2 windows, and writes NaN into the three coordinates of the rest, in place.
 * Synchronous on the context's stream. */
int s2pb_count_3d_neighbors(s2pb_ctx *ctx, int32_t *count, const double *xyz, int nx, int ny, float r, int p);
int s2pb_remove_isolated_3d_points(s2pb_ctx *ctx, double *xyz, int nx, int ny, float r, int p, int n, int q);

/* masking.erosion (s2p/masking.py:87-97 = `morsi diskR erosion`, c/morsi.c:54-66,280-298) on a 0/1 mask */
int s2pb_erode_mask(s2pb_ctx *ctx, const uint8_t *in, uint8_t *out, int w, int h, float radius);

/* ---- stage-level entry points (host buffers; used by the parity tests) ----- */
/* census_tools.cc:127-153.  codes: w*h uint64, first neighbour in the top bit. */
int s2pb_census(s2pb_ctx *ctx, const float *img, int w, int h, int win, uint64_t *codes);
/* mgm_costvolume.cc:74-174.  lo/hi: per-pixel label range (int32, inclusive);
 * C: w*h*D float32, slot k <-> label gmin+k, +INF outside the range / image. */
int s2pb_costvolume(s2pb_ctx *ctx, const float *u, const float *v, int w, int h,
                    const int32_t *lo, const int32_t *hi, int gmin, int D, int win, float *C);
/* Same for any distance (cost = S2PB_COST_*; win = census or ncc window): mgm_costvolume.h:25-180. */
int s2pb_costvolume_dist(s2pb_ctx *ctx, const float *u, const float *v, int w, int h,
                         const int32_t *lo, const int32_t *hi, int gmin, int D, int win, int cost, float *C);
/* mgm_core.cc:829-1074 on a caller-supplied volume, D <= 512.  S (nullable): w*h*D. */
int s2pb_aggregate(s2pb_ctx *ctx, const float *C, const int32_t *lo, const int32_t *hi,
                   int w, int h, int gmin, int D, float P1, float P2, int ndir, int tsgm,
                   int fix_overcount, float *S, float *disp, float *cost, float *conf);
/* Same through the general aggregation flavour: any float costs, optional per-pixel weights (w*h, nullable). */
int s2pb_aggregate_w(s2pb_ctx *ctx, const float *C, const int32_t *lo, const int32_t *hi,
                     int w, int h, int gmin, int D, float P1, float P2, int ndir, int tsgm,
                     int fix_overcount, const float *weights, float *S, float *disp, float *cost, float *conf);
/* img_tools.h:204-238 */
int s2pb_median(s2pb_ctx *ctx, const float *in, float *out, int w, int h, int radius);
/* remove_small_cc.c:9-73 with the intensity threshold 5 of mgm_multiscale.cc:332-333 */
int s2pb_remove_small_cc(s2pb_ctx *ctx, const float *in, float *out, int w, int h, int minarea);
/* s2p/block_matching.py:18-32 (plambda + backflow + plambda) */
int s2pb_rejection_mask(s2pb_ctx *ctx, const float *disp, const float *im1, const float *im2,
                        int w, int h, uint8_t *mask);

/* ---- instrumentation -------------------------------------------------------- */
enum { S2PB_T_CENSUS = 0, S2PB_T_COST, S2PB_T_AGGREGATE, S2PB_T_WTA, S2PB_T_POST, S2PB_T_TOTAL, S2PB_T_COUNT };
/* CUDA-event milliseconds of the stages of the last s2pb_mgm / s2pb_mgm_device
 * call on `slot` (valid after the stream has been synchronised). */
int s2pb_last_timings(s2pb_ctx *ctx, int slot, float ms[S2PB_T_COUNT]);
/* number of kernels this library has launched since the context was created */
long long s2pb_kernel_launches(const s2pb_ctx *ctx);

#ifdef __cplusplus
}
#endif
#endif /* S2PB200_H */
