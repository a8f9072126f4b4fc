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
 *   s2pb_cargarse_basura() the morphoop / plambda / remove_small_cc subprocesses of
 *                        common.cargarse_basura (s2p/common.py:251-262)
 *   s2pb_disp_to_xyz()   s2p.triangulation.disp_to_xyz with a WGS84 / UTM output CRS: the lib/disp_to_h.so call and the
 *                        pyproj change of coordinates (s2p/triangulation.py:85-162)
 *   s2pb_height_map_to_xyz() s2p.triangulation.height_map_to_xyz with a WGS84 / UTM output CRS: rpcm's localisation
 *                        of every pixel of the merged height map and the pyproj change of coordinates
 *                        (s2p/triangulation.py:165-217)
 *   s2pb_plyflatten()    plyflatten_from_plyfiles_list with radius 0 (the external plyflatten package) in plys_to_dsm
 *                        (s2p/__init__.py:432-476)
 *   s2pb_disp_to_ply()   disparity_to_ply's cloud after its inputs are read (s2p/__init__.py:242-318): disp_to_xyz, filter_xyz,
 *                        linear_stretching_and_quantization_8bit (s2p/common.py:284-297) and the vertex records of write_to_ply
 *                        (s2p/triangulation.py:392-429, s2p/ply.py:24-69)
 *   s2pb_height_map_to_ply() the same for heights_to_ply after heights_fusion (s2p/__init__.py:388-429), from height_map_to_xyz
 *   s2pb_disp_to_ply_clr(), s2pb_height_map_to_ply_clr() the same two steps with a clr image: its colours in its own type,
 *                        warped on the device for the pair (s2p/__init__.py:270-280), the raw window for tri-stereo (:404-406)
 *   s2pb_mosaic_deflate() global_dsm's rasterio.merge of the tile DSMs and the deflate of its GeoTIFF tiles
 *                        (s2p/__init__.py:479-525)
 *   s2pb_sgbm()          the `sgbm` subprocess (OpenCV 2's StereoSGBM, 3rdparty/sgbm) + create_rejection_mask
 *                        (s2p/block_matching.py:116-134)
 *   s2pb_pair_tile_to_ply() rectification_pair, stereo_matching and disparity_to_ply of a two-view tile (s2p/__init__.py:102-318)
 *                        in one call, from the source crops to the records of cloud.ply
 *   s2pb_pair_tile_to_height_map() rectification_pair, stereo_matching and disparity_to_height of one pair of a tri-stereo
 *                        tile (s2p/__init__.py:102-239) in one call, from the source crops to the pair's height map
 *   s2pb_heights_tile_to_ply() heights_to_ply of a tri-stereo tile, its heights_fusion included (s2p/__init__.py:355-429), in
 *                        one call, from the pairs' height maps to the records of cloud.ply
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
    int32_t census_win;      /* CENSUS_NCC_WIN  2..11: side 2*(win/2)+1; <= 1 ARG, >= 12 UNSUPPORTED */
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
 * passed as void*, NULL = the slot's own stream) and NOT synchronised when
 * timeout_ms <= 0.  `slot` selects one of the context's workspaces
 * (0 <= slot < s2pb_num_slots) so that several tiles can be in flight.  A slot
 * owns its workspace, its streams and its abort word; a call that exceeds its
 * timeout raises only its own slot's abort word and waits for its stream and
 * the slot's streams, so calls on other slots are not disturbed.
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
 * caller threads as long as each uses its own slot.  The timeout is the per-tile
 * timeout_ms times n for the whole batch; on any error or timeout every slot is
 * aborted and drained before the call returns. */
int s2pb_mgm_batch(s2pb_ctx *ctx, int n, const float *const *im1, const float *const *im2,
                   int w, int h, int dmin, int dmax, const s2pb_mgm_params *p,
                   float *const *disp, float *const *conf, uint8_t *const *mask);

/* Reserve `nslots` workspaces for tiles up to w x h x (dmax-dmin+1) labels.
 * Optional: s2pb_mgm* grow the workspace on demand. */
int s2pb_reserve(s2pb_ctx *ctx, int nslots, int w, int h, int nlabels);
int s2pb_num_slots(const s2pb_ctx *ctx);
int s2pb_sync(s2pb_ctx *ctx);

/* ---- workspace layouts ------------------------------------------------------------
 * Every mgm call of a matcher (the single-scale call, each mgm_multi level including the half-pixel one) runs in one of two
 * workspace layouts.  The resident layout keeps one f32 volume per scan pass and view (about 33 bytes per voxel and view with
 * census codes).  The folded layout keeps the running sum of the passes instead, plus a buffer of band-closing scanlines and
 * one int16 arg-minimum plane per pass (about 5.25 bytes per voxel and view), and runs the passes one after the other.  Both
 * give the same results, bit for bit.  A call uses the resident layout when it is within the context's workspace limit and
 * its allocation succeeds, else the folded one; when that does not fit either, S2PB_ERR_NOMEM names both sizes.  The stage
 * entry points (s2pb_aggregate, s2pb_aggregate_w) run resident only. */
/* The limit in bytes for each workspace of the context (s2pb_reserve, one per slot); 0 = none (the default), which keeps the
 * resident layout wherever its allocation succeeds.  It lets several processes share a GPU.  S2PB_ERR_ARG: bytes < 0. */
int s2pb_set_workspace_limit(s2pb_ctx *ctx, long long bytes);
/* Bytes of the workspace of a w x h tile whose slab holds D labels (the hull dmax - dmin + 1 of a single-scale call; the
 * slab is rounded up as the kernels round it), ndir passes, cost_bytes 1 (census codes) or 4 (float costs: the other
 * distances, or the -wl / -wr weights), in the resident (folded = 0) or folded layout.  No device needed.  A negative S2PB_ERR_*
 * code for arguments the matcher does not serve. */
long long s2pb_workspace_bytes(int w, int h, int D, int ndir, int cost_bytes, int folded);
/* The layout a workspace limit (bytes, 0 = none) selects for that tile: 0 resident, 1 folded, S2PB_ERR_NOMEM for neither.
 * No device needed; an allocation failure of the resident layout also falls back to the folded one at run time. */
int s2pb_workspace_layout(int w, int h, int D, int ndir, int cost_bytes, long long limit);
/* number of mgm calls the context has run in the folded layout */
long long s2pb_folded_calls(const s2pb_ctx *ctx);
/* ---- DCT coefficient tables ---------------------------------------------------------
 * The matched image's DCT round trip (and the half-pixel shift of mgm_multi) multiplies each image row by n x n double tables
 * computed on the host with libm.  Up to 8192 px they stay on the device once per width.  Wider rows keep a table there while
 * the context's tables of such widths stay within this limit -- and within the workspace limit, when one is set -- and
 * otherwise stream it in K-panels through pinned staging buffers, with the same results, bit for bit.  Default 8 GiB;
 * 0 streams every table of rows wider than 8192 px.  Tables already on the device stay.  S2PB_ERR_ARG: bytes < 0. */
int s2pb_set_dct_table_limit(s2pb_ctx *ctx, long long bytes);
/* out[r][c] (nrows x ncols, row-major) = the coefficients (row0 + r, col0 + c) of a table for rows of n pixels, as the engine
 * computes them: kind 0 REDFT10 [k][j] = 2 cos(pi (j + 1/2) k / n), 1 REDFT01 [i][k] = 1 for k = 0, else 2 cos(pi k (i + 1/2) / n),
 * 2 RODFT01 [i][k] = (-1)^i for k = n - 1, else 2 sin(pi (k + 1) (i + 1/2) / n).  No device needed. */
int s2pb_dct_coefficients(int kind, int n, int row0, int nrows, int col0, int ncols, double *out);

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
 * anti-aliasing rule (3rdparty/homography/LibHomography/Homography.cpp:50-168).
 * S2PB_ERR_ARG for an empty region of interest, and for a spline image (the region of interest, or
 * the anti-aliasing intermediate) with a side below 4 pixels, which the reference cannot warp either. */
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
/* s2p.triangulation.disp_to_xyz (s2p/triangulation.py:85-162) for an output CRS of WGS84 / UTM (EPSG 32601-32660 north,
 * 32701-32760 south) in one call: the argument list of lib/disp_to_h.so's disp_to_lonlatalt (c/disp_to_h.c:70-76), which
 * s2p.triangulation.disp_to_xyz calls through ctypes (s2p/triangulation.py:118-143), plus the context, then the UTM zone
 * (1..60, or 0: the output is lon, lat, alt as disp_to_lonlatalt writes them) and south (non-zero: false northing
 * 10 000 000 m).  The cloud is triangulated and projected as s2pb_lonlat_to_utm projects it on the device; xyz (nx*ny*3
 * float64) and err (nx*ny float32) come back.
 * S2PB_ERR_ARG: a null pointer, a size below 1, a zone outside 0..60 (S2PB_ZONE_EGM96 and S2PB_ZONE_PROJ aside). */
int s2pb_disp_to_xyz(s2pb_ctx *ctx, double *xyz, float *err, const float *dispx, const float *dispy, const float *msk, int nx,
                     int ny, const float *msk_orig, int w, int h, const double ha[9], const double hb[9], const s2pb_rpc *rpca,
                     const s2pb_rpc *rpcb, const float orig_img_bounding_box[4], int zone, int south);
/* EPSG:4979 -> UTM zone `zone` (1..60) of WGS84, north (EPSG 326zz) or south (south != 0, EPSG 327zz), for n points of
 * three float64 (lon and lat in degrees, alt), host buffers (xyz may be lonlatalt).  The exact transverse Mercator that PROJ
 * runs for +proj=utm (Poder / Engsager, Krueger's series to order n^6; Karney 2011), k0 = 0.9996, central meridian
 * 6 zone - 183, false easting 500 000 m.  The altitude passes through.  A point with a NaN coordinate becomes NaN in all
 * three; a point outside the projection's domain (|lat| > 90, or too far from the central meridian) +inf in all three.
 * Within 1e-6 m of the exact map.  S2PB_ERR_ARG: a null pointer with n > 0, n < 0, a zone outside 1..60 (S2PB_ZONE_EGM96
 * aside). */
int s2pb_lonlat_to_utm(s2pb_ctx *ctx, double *xyz, const double *lonlatalt, int64_t n, int zone, int south);

/* Heights above the EGM96 geoid (EPSG:5773), the vertical datum of s2p's `out_geoid` targets EPSG:326zz+5773 / 327zz+5773
 * (and EPSG:4326+5773 for zone 0).  OR S2PB_ZONE_EGM96 into the `zone` argument of s2pb_disp_to_xyz, s2pb_lonlat_to_utm,
 * s2pb_height_map_to_xyz and the PLY calls, or into the zone field of s2pb_pair_tile and s2pb_heights_tile: every point then
 * gets z = z - N(lon, lat) in float64, N interpolated in the context's geoid grid at the point's WGS84 longitude and
 * latitude, before the UTM map (which leaves x and y as they are without the flag).  The cloud's 3D filter runs on the
 * shifted cloud.  Bilinear rule: node (i, j) lies at (lon0 + i dlon, lat0 - j dlat); for x = ((lon - lon0) mod 360) / dlon
 * and y = (lat0 - lat) / dlat, i = floor(x), j = floor(y) (at most h - 1), fx = x - i, fy = y - j, column i + 1 is column 0
 * past the last one and row j + 1 the last row past it; from the float32 nodes a = (i, j), b = (i+1, j), c = (i, j+1),
 * d = (i+1, j+1), in float64, t = a + fx (b - a), u = c + fx (d - c), N = t + fy (u - t): PROJ's bilinear vgridshift on a
 * grid such as us_nga_egm96_15.tif up to rounding, exact at the nodes and on a constant grid.  A NaN point stays NaN in all three coordinates; a point with
 * |lat| > 90 becomes +inf in all three.  S2PB_ERR_ARG: the flag on a context without a grid; any bit other than the flag
 * or a zone outside the call's range once the flag is removed. */
#define S2PB_ZONE_EGM96 0x100
/* Upload the geoid grid of S2PB_ZONE_EGM96 to the context's device, replacing the one it holds (grid NULL: drop it).  grid:
 * h rows of w float32 node values in metres, row 0 northernmost, node (i, j) at (lon0 + i dlon, lat0 - j dlat) degrees.  The
 * grid must be global: w dlon >= 360 (longitude wraps), lat0 >= 90 and lat0 - (h - 1) dlat <= -90.  Synchronous.
 * S2PB_ERR_ARG: w or h below 2, w * h above 2^31 - 1, a non-finite origin, a spacing that is not positive and finite, a grid
 * that is not global.  S2PB_ERR_NOMEM: the grid does not fit the device. */
int s2pb_set_geoid(s2pb_ctx *ctx, const float *grid, int w, int h, double lon0, double lat0, double dlon, double dlat);

/* Map projections other than the UTM zones of WGS84, for output CRSs whose datum reaches WGS84 through a null
 * transformation, so that the cloud is the map of the triangulated WGS84 (lon, lat) and the altitude passes through: the
 * ETRS89 UTM zones (EPSG 25828-25838, S2PB_PROJ_TM on GRS80) and RGF93 v1 / Lambert-93 and CC42-CC50 (EPSG 2154,
 * 3942-3950, S2PB_PROJ_LCC on GRS80).  Angles in degrees, lengths in metres.
 *   S2PB_PROJ_TM: transverse Mercator, the map of s2pb_lonlat_to_utm on the given ellipsoid, central meridian lon0, scale k0,
 *     false easting x0 and northing y0; lat0 must be 0 (northings count from the equator); lat1 and lat2 are not read.
 *   S2PB_PROJ_LCC: Lambert conic conformal with two standard parallels lat1 and lat2 (EPSG method 9802), false origin
 *     (lon0, lat0) at (x0, y0); k0 is not read.  lat1 == lat2 gives the one-parallel cone.  In this operation order, with
 *     psi(phi) = asinh(tan phi) - e atanh(e sin phi) and the host's n, a F and r_F (IOGP Guidance Note 7-2, 3.1.1.1):
 *     lam = lon - lon0 reduced to [-180, 180], rho = a F exp(-(n psi)), theta = n lam, x = x0 + rho sin theta,
 *     y = y0 + (r_F - rho cos theta).  A pole on the side the cone opens to maps to the apex (rho = 0); the other pole
 *     gives +inf in all three coordinates. */
#define S2PB_PROJ_TM 1
#define S2PB_PROJ_LCC 2
typedef struct s2pb_projection {
    int32_t method;              /* S2PB_PROJ_TM or S2PB_PROJ_LCC */
    double a, rf;                /* ellipsoid: semi-major axis, inverse flattening */
    double lon0, lat0;           /* natural origin (TM) or false origin (LCC) */
    double lat1, lat2;           /* standard parallels (LCC) */
    double k0;                   /* scale factor on the central meridian (TM) */
    double x0, y0;               /* false easting and northing */
} s2pb_projection;
/* OR S2PB_ZONE_PROJ, instead of a UTM zone, into the `zone` argument of s2pb_disp_to_xyz, s2pb_height_map_to_xyz and the PLY
 * calls, or into the zone field of s2pb_pair_tile and s2pb_heights_tile: every point of that call then goes through the
 * context's projection (s2pb_set_projection).  S2PB_ZONE_EGM96 may be OR'ed in too (heights above the geoid, then the map).
 * S2PB_ERR_ARG: the flag on a context without a projection, with a nonzero south, or with any bit other than S2PB_ZONE_EGM96. */
#define S2PB_ZONE_PROJ 0x200
/* Hold *proj on the context for S2PB_ZONE_PROJ, replacing the one it holds (proj NULL: drop it).  Nothing is uploaded.
 * S2PB_ERR_ARG: an unknown method; a, rf, k0 (TM), an angle, x0 or y0 not finite; a <= 0, rf <= 1; TM: k0 <= 0 or lat0 != 0;
 * LCC: a standard parallel outside (-90, 90), lat1 == -lat2 (no cone), |lat0| > 90, lat0 the pole the cone does not reach.
 * A refused projection leaves the one held in place. */
int s2pb_set_projection(s2pb_ctx *ctx, const s2pb_projection *proj);
/* EPSG:4979 -> the map *proj (checked as s2pb_set_projection checks it) for n points of three float64 (lon and lat in degrees,
 * alt), host buffers (xyz may be lonlatalt).  The altitude passes through.  A point with a NaN coordinate becomes NaN in all
 * three; a point the map cannot project (|lat| > 90, outside the TM domain of s2pb_lonlat_to_utm, the LCC pole away from
 * the cone) +inf in all three.  S2PB_ERR_ARG: a null pointer with n > 0, n < 0, a refused projection. */
int s2pb_lonlat_to_proj(s2pb_ctx *ctx, double *xyz, const double *lonlatalt, int64_t n, const s2pb_projection *proj);

/* ---- tri-stereo height maps (s2p/__init__.py disparity_to_height and heights_fusion) ---- */
/* s2p.triangulation.height_map (s2p/triangulation.py:346-389) in one call.  disp, msk: the rectified disparity and mask,
 * nx*ny float32; mask_orig: the tile's mask as s2p reads it, mw*mh float32, unpadded (padded here by one row and column of
 * ones); (x, y, w, h): the tile in the reference image; H1, H2: the rectifying homographies, H2 with the pointing correction
 * already applied (H2 * A^-1, which the Python drop-in computes with numpy as the reference does).
 * Triangulates as s2pb_disp_to_xyz with zone 0 inside the bounding box float32(x-1, x+w+2, y-1, y+h+2), keeps the altitude on
 * the device and writes out (h*w float64, row-major) = affine_transform(nan_to_num(alt).T, H1 * T(x, y),
 * output_shape=(w, h), order=1).T, NaN on the 3x3 dilation of the nearest-neighbour transform of isnan(alt).T (see
 * s2pb_resample_heights).  The third column of H1 * T(x, y) is summed left to right, H1[r][0]*x + H1[r][1]*y + H1[r][2].
 * S2PB_ERR_ARG: the last row of H1 * T(x, y) is not (0, 0, 1), which scipy refuses.
 * S2PB_ERR_UNSUPPORTED: nx or ny below 2 (the reference squeezes such a map to one dimension and fails). */
int s2pb_height_map(s2pb_ctx *ctx, double *out, const float *disp, const float *msk, int nx, int ny, const float *mask_orig,
                    int mw, int mh, int x, int y, int w, int h, const double H1[9], const double H2[9], const s2pb_rpc *rpc1,
                    const s2pb_rpc *rpc2);
/* The resampling stage of s2pb_height_map alone, on a zw*zh float64 map z: scipy.ndimage.affine_transform(nan_to_num(z).T,
 * H, output_shape=(w, h), order=1, mode='constant', cval=0).T bit for bit, then NaN where
 * the 3x3 dilation (zero border) of affine_transform(isnan(z).T, H, output_shape=(w, h), order=0).T is set.
 * S2PB_ERR_ARG: the last row of H is not (0, 0, 1), which scipy refuses. */
int s2pb_resample_heights(s2pb_ctx *ctx, const double *z, int zw, int zh, const double H[9], double *out, int w, int h);
/* s2p.common.cargarse_basura (s2p/common.py:251-262) on a w*h float32 image: NaN where the 5x5 max and min of the
 * non-NaN values (c/morphoop.c, mirrored border) differ by more than 5, then remove_small_cc with area 200 and intensity
 * threshold 5 (components of area <= 200 become NaN).  Bit for bit the output of the reference's six commands.
 * S2PB_ERR_UNSUPPORTED: w or h below 2 (the reference's morphoop reads outside the image). */
int s2pb_cargarse_basura(s2pb_ctx *ctx, const float *in, float *out, int w, int h);
/* s2p.triangulation.height_map_to_xyz (s2p/triangulation.py:165-217), which heights_to_ply runs on the merged height map,
 * for an output CRS of WGS84 / UTM in one call.  heights: w*h float64, row-major (a float32 map converts exactly); rpc: the
 * camera of the reference image; (off_x, off_y): where the map's origin lies in that image.  Pixel (i, j) with height z
 * becomes the ground point of image pixel (j + off_x, i + off_y) at height z (rpc_localization, c/rpc.c:469: the direct
 * polynomials when the model has them, the iteration of c/rpc.c:378-411 otherwise), then UTM zone `zone` (1..60; 0: lon,
 * lat, alt as they are) north or south (south != 0) as s2pb_lonlat_to_utm projects it; xyz (w*h*3 float64) comes back.
 * The third coordinate is z bit for bit.  A NaN height gives NaN in all three (the reference leaves lon and lat undefined
 * there); an iteration whose residual turns NaN stops, as the reference's does, with a NaN lon and lat.
 * S2PB_ERR_ARG: a null pointer, a size below 1, a zone outside 0..60 (S2PB_ZONE_EGM96 and S2PB_ZONE_PROJ aside), or pixels whose iteration did not meet the
 * reference's stopping test within 1000 steps (the reference would not return; the message gives their number). */
int s2pb_height_map_to_xyz(s2pb_ctx *ctx, double *xyz, const double *heights, int w, int h, const s2pb_rpc *rpc, double off_x,
                           double off_y, int zone, int south);

/* The 3D outlier filter of s2p.triangulation.filter_xyz (s2p/triangulation.py:275-343): same argument lists as
 * lib/disp_to_h.so's count_3d_neighbors and remove_isolated_3d_points (c/disp_to_h.c:152-230), plus the context.
 * xyz: nx*ny points of three doubles, row-major.  count[y*nx+x] = number of points of the (2p+1)^2 window, clipped at
 * the border, whose squared distance (differences in double, rounded to float, summed in float) is < r*r.
 * remove_isolated_3d_points rejects the points with count < n, saves every rejected point joined to a kept one by a chain
 * of close points within (2q+1)^2 windows, and writes NaN into the three coordinates of the rest, in place.
 * Synchronous on the context's stream. */
int s2pb_count_3d_neighbors(s2pb_ctx *ctx, int32_t *count, const double *xyz, int nx, int ny, float r, int p);
int s2pb_remove_isolated_3d_points(s2pb_ctx *ctx, double *xyz, int nx, int ny, float r, int p, int n, int q);

/* ---- the tile's point cloud (s2p/__init__.py disparity_to_ply and heights_to_ply) ---- */
/* common.linear_stretching_and_quantization_8bit(img, pct) (s2p/common.py:284-297) of n float32 values (every band of the image
 * together; a uint8 or uint16 image converts exactly) bit for bit with NumPy >= 2: a, b = np.nanpercentile(img, (pct, 100 - pct))
 * by numpy's 'linear' method (float64 quantiles pct / 100 and (100 - pct) / 100, virtual index (N - 1) q over the N non-NaN values,
 * the neighbours' difference in float32, the rest of the interpolation in float64), then out = round_half_even(255 * (clip(v, a, b)
 * - a) / (b - a)) in float64 as uint8, NaN -> 0 (a constant or all-NaN image gives 0 everywhere).
 * S2PB_ERR_ARG: a null pointer with n > 0, n < 0, pct outside [0, 100].  S2PB_ERR_UNSUPPORTED: n > 2^31 - 1. */
int s2pb_stretch_8bit(s2pb_ctx *ctx, const float *img, int64_t n, double pct, uint8_t *out);
/* The vertex records write_to_ply writes for a cloud (s2p/triangulation.py:392-429 -> ply.write_3d_point_cloud_to_ply): the points
 * of xyz (n points of three float64) whose three coordinates are finite, in order, each packed as x, y, z float64, then, with
 * nbands = 1, 3 or 4 colour planes (n uint8 each; one band is written three times), red, green, blue (and ir) uint8, then, with conf
 * (n float32, nullable), confidence float32: 24 + {0, 3, 4} + {0, 4} bytes, no padding.  records holds n such records; *npoints
 * gets the number written.  S2PB_ERR_ARG: a null pointer, n < 0, nbands not 0, 1, 3 or 4 (the reference raises).
 * S2PB_ERR_UNSUPPORTED: n > 2^31 - 1. */
int s2pb_ply_records(s2pb_ctx *ctx, const double *xyz, int64_t n, const uint8_t *colors, int nbands, const float *conf,
                     uint8_t *records, int64_t *npoints);
/* disparity_to_ply's cloud (s2p/__init__.py:242-318) in one call: s2pb_disp_to_xyz's argument list without its outputs, then
 * the 3D filter (remove_isolated_3d_points with r, p, n and q = 1 on the projected cloud, as filter_xyz; off when r == 0 or
 * n <= 0), nbands colour planes of nx*ny float32 stretched as s2pb_stretch_8bit stretches them with pct, an optional nx*ny
 * float32 confidence image, and the records of s2pb_ply_records (records: nx*ny records).  Only the npoints records come back.
 * S2PB_ERR_ARG: as s2pb_disp_to_xyz and s2pb_ply_records, pct outside [0, 100].
 * S2PB_ERR_UNSUPPORTED: more than 2^31 - 1 points or colour values. */
int s2pb_disp_to_ply(s2pb_ctx *ctx, const float *dispx, const float *dispy, const float *msk, int nx, int ny, const float *msk_orig,
                     int w, int h, const double ha[9], const double hb[9], const s2pb_rpc *rpca, const s2pb_rpc *rpcb,
                     const float orig_img_bounding_box[4], int zone, int south, float r, int p, int n, const float *bands,
                     int nbands, double pct, const float *conf, uint8_t *records, int64_t *npoints);
/* heights_to_ply's cloud after heights_fusion (s2p/__init__.py:388-429) in one call: s2pb_height_map_to_xyz's argument list
 * without its output, then the filter, colours (w*h planes) and records of s2pb_disp_to_ply, without confidence.
 * S2PB_ERR_ARG: as s2pb_height_map_to_xyz (non-converging localisations included) and s2pb_disp_to_ply. */
int s2pb_height_map_to_ply(s2pb_ctx *ctx, const double *heights, int w, int h, const s2pb_rpc *rpc, double off_x, double off_y,
                           int zone, int south, float r, int p, int n, const float *bands, int nbands, double pct,
                           uint8_t *records, int64_t *npoints);

/* PLY property types: the eight plyfile writes, as double, float, uchar, char, short, ushort, int and uint */
enum { S2PB_PLY_F64 = 0, S2PB_PLY_F32 = 1, S2PB_PLY_U8 = 2 };
enum { S2PB_PLY_I8 = 16, S2PB_PLY_I16 = 17, S2PB_PLY_U16 = 18, S2PB_PLY_I32 = 19, S2PB_PLY_U32 = 20 };

/* The tile's point cloud coloured from the image cfg['images'][0]['clr']: the colours keep that image's type, as s2p writes
 * them (s2p/__init__.py:270-280 and :404-406), and are copied into the records as they are, without a stretch.
 *
 * s2pb_ply_records with colour planes of any S2PB_PLY_* type: colors holds nbands planes of n values of color_type,
 * little-endian, copied byte for byte (NaN colours included) into red, green, blue (and ir) of that type:
 * 24 + {0, 3, 4} * {1, 2, 4, 8} + {0, 4} bytes per record, at most 60, no padding.
 * S2PB_ERR_ARG: as s2pb_ply_records, and an unknown color_type. */
int s2pb_ply_records_typed(s2pb_ctx *ctx, const double *xyz, int64_t n, const void *colors, int nbands, int color_type,
                           const float *conf, uint8_t *records, int64_t *npoints);
/* disparity_to_ply with a clr image (s2p/__init__.py:270-280) in one call: s2pb_disp_to_ply's cloud and filter, with float
 * colours warped on the device.  clr: nbands float32 planes of the cw*ch crop of the clr image that the warp of the rectified
 * reference needs; hc: H_ref with the crop's origin folded in (H_ref . [[1, 0, x], [0, 1, y], [0, 0, 1]]).  Each band is
 * warped into nx*ny as s2pb_homography(band, cw, ch, hc, ..., nx, ny) warps it (NaN outside the source), and the float
 * colours and the optional confidence are packed as s2pb_ply_records_typed packs them.
 * S2PB_ERR_ARG: as s2pb_disp_to_ply and s2pb_homography, nbands not 1, 3 or 4. */
int s2pb_disp_to_ply_clr(s2pb_ctx *ctx, const float *dispx, const float *dispy, const float *msk, int nx, int ny,
                         const float *msk_orig, int w, int h, const double ha[9], const double hb[9], const s2pb_rpc *rpca,
                         const s2pb_rpc *rpcb, const float orig_img_bounding_box[4], int zone, int south, float r, int p, int n,
                         const float *clr, int cw, int ch, int nbands, const double hc[9], const float *conf, uint8_t *records,
                         int64_t *npoints);
/* heights_to_ply with a clr image (s2p/__init__.py:404-406) after heights_fusion in one call: s2pb_height_map_to_ply's cloud and
 * filter, then the records of s2pb_ply_records_typed with the colours (nbands planes of w*h values of color_type: the clr
 * window in its stored type).  S2PB_ERR_ARG: as s2pb_height_map_to_ply, nbands not 1, 3 or 4, an unknown color_type. */
int s2pb_height_map_to_ply_clr(s2pb_ctx *ctx, const double *heights, int w, int h, const s2pb_rpc *rpc, double off_x,
                               double off_y, int zone, int south, float r, int p, int n, const void *colors, int nbands,
                               int color_type, uint8_t *records, int64_t *npoints);

/* ---- DSM rasterisation (s2p/__init__.py plys_to_dsm) -------------------------- */
/* One vertex property of a binary little-endian PLY record: its byte offset in the record and its type (S2PB_PLY_*). */
typedef struct s2pb_ply_column {
    int32_t offset;
    int32_t type;            /* S2PB_PLY_* */
} s2pb_ply_column;
/* plyflatten_from_plyfiles_list(clouds, resolution, radius=0, roi=(xoff, yoff, xsize, ysize), sigma=None), which
 * plys_to_dsm runs on a tile's cloud and its neighbours' (s2p/__init__.py:432-476).  records[k]: the npoints[k] vertex records
 * of cloud k, record_bytes each, as they lie in the file; host memory (pageable or page-locked) or device memory, NULL when
 * npoints[k] == 0.  cols[0], cols[1]: x and y; cols[2..ncols-1]: the raster's channels, in that order.  Every property is
 * read as float64 (exactly, for every type).  A point falls in cell (floor((x - xoff) / resolution), floor((yoff - y) / resolution)), in double; points
 * outside the raster or with a NaN coordinate are skipped.  Per cell and channel, over the clouds in order and each cloud's
 * points in order: acc = (float)((double)acc + 1.0 * v) from 0.0f, cnt += 1.0f; raster[(j * xsize + i) * (ncols - 2) + c] =
 * acc / cnt in float, NaN where no point fell.  Deterministic.  Synchronous on the context's stream.
 * S2PB_ERR_ARG: a null pointer, npoints < 0, ncols < 3, resolution not positive and finite, xsize or ysize < 1, a column
 * outside the record or of an unknown type.
 * S2PB_ERR_UNSUPPORTED: more than 2^31 - 1 points in all, xsize * ysize >= 2^32 - 1, or more than 16 columns. */
int s2pb_plyflatten(s2pb_ctx *ctx, int nclouds, const void *const *records, const int64_t *npoints, int record_bytes,
                    const s2pb_ply_column *cols, int ncols, double xoff, double yoff, double resolution, int xsize, int ysize,
                    float *raster);

/* global_dsm (s2p/__init__.py:479-525): rasterio.merge(method='first') of the tile DSMs onto a W x H destination, written as
 * the tiles of a GeoTIFF with 256 x 256 tiles, PREDICTOR=2 and COMPRESS=DEFLATE.  Source k: src_w[k] x src_h[k] row-major
 * float32 in host memory (pageable or page-locked), NaN = nodata, its pixel (0, 0) at destination column col_off[k] and row
 * row_off[k] (either may be negative; the part outside the destination is clipped).  Each destination pixel is the first
 * non-NaN value, over the sources in order, among those that cover it; NaN where none does (other values, -0.0 and +-inf
 * included, keep their bits).  Tile (i, j), in row-major tile order, is the 256 x 256 window at (256 i, 256 j), NaN past the
 * raster's edge; its bytes after libtiff's horizontal differencing of 32-bit words within each tile row (horDiff32) are
 * compressed into one zlib stream (0x78 0x9C, deflate, Adler-32), or into stored blocks when those are shorter.
 * out: the streams back to back in tile order; block_sizes[t]: stream t's bytes (ceil(W / 256) * ceil(H / 256) of them).
 * The destination is processed in bands of band_rows tile rows (0: as many as a fixed device budget holds), two in flight;
 * only the sources' rows a band covers go to the device with it.  Synchronous.
 * S2PB_ERR_ARG: a null pointer, a size below 1, an offset beyond +-2^30, band_rows < 0, or out_capacity smaller than the
 * streams.  S2PB_ERR_NOMEM: a band's scratch does not fit the device. */
int s2pb_mosaic_deflate(s2pb_ctx *ctx, int nsrc, const float *const *srcs, const int *src_w, const int *src_h,
                        const int64_t *col_off, const int64_t *row_off, int W, int H, int band_rows, uint8_t *out,
                        int64_t out_capacity, int32_t *block_sizes);
/* The tile streams of s2pb_mosaic_deflate for one W x H raster (host memory) at offset (0, 0). */
int s2pb_deflate_blocks(s2pb_ctx *ctx, const float *raster, int W, int H, int band_rows, uint8_t *out, int64_t out_capacity,
                        int32_t *block_sizes);

/* masking.erosion (s2p/masking.py:87-97 = `morsi diskR erosion`, c/morsi.c:54-66,280-298) on a 0/1 mask */
int s2pb_erode_mask(s2pb_ctx *ctx, const uint8_t *in, uint8_t *out, int w, int h, float radius);

/* ---- a two-view tile from its source images to its point cloud (s2p.main steps 3 to 5 with two images) ---------- */
enum { S2PB_MATCHER_MGM = 0, S2PB_MATCHER_SGBM = 1 };
/* The inputs of s2pb_pair_tile_to_ply and s2pb_pair_tile_to_height_map, stage by stage.  Host pointers. */
typedef struct s2pb_pair_tile {
    /* rectify_pair's two warps: the crops of the two images and their rectifying homographies with the crops' origins folded in */
    const float *src1, *src2;
    int32_t sw1, sh1, sw2, sh2;
    double H1[9], H2[9];
    int32_t w, h;                /* the rectified size */
    int32_t dmin, dmax;          /* the matcher's range, as compute_disparity_map hands it to the matcher */
    /* the matcher */
    int32_t matcher;             /* S2PB_MATCHER_MGM (mgm, mgm_multi, mgm_multi_lsd by mgm.scales and wl / wr) or _SGBM */
    s2pb_mgm_params mgm;
    s2pb_sgbm_params sgbm;
    const float *wl, *wr;        /* MGM: the -wl / -wr weight images (w*h float32), both or neither */
    float erode_radius;          /* masking.erosion of the mask: 0 none, else a disk radius in (1, 64] */
    /* disparity_to_ply's cloud: s2pb_disp_to_ply's arguments from msk_orig to south, and the filter's r, p, n */
    const float *msk_orig;
    int32_t mw, mh;
    float bbox[4];
    const s2pb_rpc *rpc1, *rpc2;
    double ha[9], hb[9];         /* H_ref and H_sec . A^-1 as disparity_to_ply reads them */
    int32_t zone, south;
    float r;
    int32_t p, n;
    /* the colours: the rectified reference stretched with pct, or, when clr is not null, clr_bands float32 planes of the cw x ch
     * crop of the clr image warped by hc as s2pb_disp_to_ply_clr warps them */
    double pct;
    const float *clr;
    int32_t cw, ch, clr_bands;
    double hc[9];
    int32_t with_conf;           /* MGM: the confidence column */
} s2pb_pair_tile;
/* s2pb_homography x 2 -> s2pb_mgm_weighted or s2pb_sgbm -> s2pb_erode_mask when erode_radius > 0 -> s2pb_disp_to_ply, or
 * s2pb_disp_to_ply_clr with a clr crop, on the disparity, the eroded mask as float32 and a zero dispy, in one call: the rectified pair, the
 * disparity, the confidence and the mask stay on the device between the stages, and the records and every intermediate are
 * those of that sequence, bit for bit.  records: w*h records of the record size of the colours and the confidence; *npoints
 * gets the number written.  Nullable host copies of the intermediates (w*h each): rect1, rect2, disp, conf (MGM), mask (0/1,
 * after the erosion), disp_right (MGM).  Errors as the calls of the sequence, S2PB_ERR_TIMEOUT from the MGM matcher included;
 * S2PB_ERR_ARG also for conf, disp_right or with_conf with sgbm.  Synchronous. */
int s2pb_pair_tile_to_ply(s2pb_ctx *ctx, const s2pb_pair_tile *t, uint8_t *records, int64_t *npoints, float *rect1, float *rect2,
                          float *disp, float *conf, uint8_t *mask, float *disp_right);

/* ---- a tri-stereo tile from its source images to its point cloud (s2p.main steps 3 to 5 with three or more images) ---- */
/* One pair i of the tile: s2pb_homography x 2 -> s2pb_mgm_weighted or s2pb_sgbm -> s2pb_erode_mask when erode_radius > 0 ->
 * s2pb_height_map on the disparity and the eroded mask as float32, in one call, with the intermediates on the device.  It
 * reads the warp fields of t (src1 to h), the matcher fields (dmin to wr), erode_radius, msk_orig, mw, mh, rpc1, rpc2, and
 * ha = H_ref as H_ref.txt holds it and hb = H_sec . A^-1 (the pointing correction applied), s2pb_height_map's H1 and H2.  It
 * ignores the cloud-only fields: bbox, zone, south, r, p, n, pct, clr, cw, ch, clr_bands, hc and with_conf.  (x, y, w, h): the
 * tile in the reference image; heights: w*h float64, the pair's height map.  The heights, their NaN set and every
 * intermediate are those of that sequence, bit for bit.  Nullable host copies of the intermediates (t->w * t->h each): rect1,
 * rect2, disp, conf (MGM), mask (0/1, after the erosion), disp_right (MGM).  Errors as the calls of the sequence: S2PB_ERR_TIMEOUT
 * from the MGM matcher, S2PB_ERR_UNSUPPORTED for a rectified size below 2 x 2, and S2PB_ERR_ARG also for conf or disp_right
 * with sgbm.  Synchronous. */
int s2pb_pair_tile_to_height_map(s2pb_ctx *ctx, const s2pb_pair_tile *t, int x, int y, int w, int h, double *heights, float *rect1,
                                 float *rect2, float *disp, float *conf, uint8_t *mask, float *disp_right);
#define S2PB_MAX_FUSION 16
/* The inputs of s2pb_heights_tile_to_ply, stage by stage.  Host pointers. */
typedef struct s2pb_heights_tile {
    /* heights_fusion: n_maps (1..S2PB_MAX_FUSION) w*h height maps of the pairs, all of map_type (S2PB_PLY_F32 or S2PB_PLY_F64) as
     * they are stored, their offsets (the global mean heights), cargarse_basura, and merge_n's operator (the op codes of
     * s2pb_merge_n, S2PB_FUSE_SUB_F32 included) and threshold */
    int32_t n_maps, w, h, map_type;
    const void *maps[S2PB_MAX_FUSION];
    double offsets[S2PB_MAX_FUSION];
    int32_t cargarse_basura, op;
    double threshold;
    /* height_map_to_xyz: the reference image's camera, the tile's origin in that image, the output UTM zone (0: lon, lat, alt;
     * S2PB_ZONE_PROJ instead: the context's projection; S2PB_ZONE_EGM96 may be OR'ed in) */
    const s2pb_rpc *rpc;
    double off_x, off_y;
    int32_t zone, south;
    /* the filter of filter_xyz (off when r == 0 or n <= 0) */
    float r;
    int32_t p, n;
    /* the colours: nbands (0, 1, 3 or 4) planes of w*h values; stretch != 0: float32 stretched with pct as
     * s2pb_height_map_to_ply stretches them; else values of PLY type color_type copied as s2pb_height_map_to_ply_clr copies them */
    const void *colors;
    int32_t nbands, color_type, stretch;
    double pct;
} s2pb_heights_tile;
/* heights_fusion then heights_to_ply's cloud (s2p/__init__.py:355-429) in one call: with cargarse_basura, each map rounded to
 * float32 (as the reference's tools read a float64 map) and cleaned as s2pb_cargarse_basura cleans it, then merged by
 * s2pb_merge_n's rule; without it the maps are merged in their stored type, a float64 map subtracted from its offset in float64
 * without a rounding first (as s2p/fusion.py:49 does with the float64 array rasterio reads).  The merged float32 map, converted
 * to float64 exactly, goes through s2pb_height_map_to_ply (stretch) or s2pb_height_map_to_ply_clr (typed colours).  records: w*h
 * records of the record size of the colours; *npoints gets the number written.  Nullable host copies of the intermediates:
 * cleaned (null, or n_maps nullable pointers to w*h float32: each cleaned map, with cargarse_basura only) and merged (w*h
 * float32).  Errors as the calls of the sequence: S2PB_ERR_UNSUPPORTED for more than S2PB_MAX_FUSION maps, or a map below
 * 2 x 2 with cargarse_basura; S2PB_ERR_ARG also for a map_type other than float32 / float64, or cleaned without
 * cargarse_basura.  Synchronous. */
int s2pb_heights_tile_to_ply(s2pb_ctx *ctx, const s2pb_heights_tile *t, uint8_t *records, int64_t *npoints, float *const *cleaned,
                             float *merged);

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
