// multiscale_kernels.cuh -- the extra stages of `mgm_multi` (SURVEY.md row a11).
//
// Behavioural reference, paths under $REF/3rdparty/mgm_multi ($REF: the root of the s2p sources): mgm_multiscale.cc:16-117
// (zoom_nn, upsample2x_disp, downsample2x, downsample2x_disp), stereo_utils.cc:134-175
// (update_dmin_dmax), remove_small_cc.c:9-73, shear.c:28-101 + mgm_costvolume.cc:23-60 (DCT shift).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace s2pb {

// downsample2x (mgm_multiscale.cc:57-95): 10x10 Gaussian taps centred between pixels (CX = 4),
// renormalised over the in-image taps; y outer / x inner accumulation, `acc += u*g` contracted to one
// fma exactly as gcc does for the reference at -O3 -march=native.
struct GaussTaps { float g[100]; };
__global__ void downsample2x_kernel(const float *__restrict__ u, int nx, int ny, GaussTaps T, float *__restrict__ out, int onx, int ony)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= onx || j >= ony) return;
    float acc = 0.f, norm = 0.f;
    for (int y = 0; y < 10; y++) {
        int yy = j * 2 + y - 4;
        for (int x = 0; x < 10; x++) {
            int xx = i * 2 + x - 4;
            if (xx >= 0 && yy >= 0 && xx < nx && yy < ny) {
                float gg = T.g[x + y * 10];
                acc = fmaf(u[(size_t)yy * nx + xx], gg, acc);
                norm += gg;
            }
        }
    }
    out[(size_t)j * onx + i] = __fdiv_rn(acc, norm);
}

// downsample2x_disp (mgm_multiscale.cc:98-117): 2x2 min / max pooling of the range images, halved
__global__ void downsample2x_disp_kernel(const float *__restrict__ u, int nx, int ny, int is_max, float *__restrict__ out, int onx, int ony)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= onx || j >= ony) return;
    float vmin = __int_as_float(0x7f800000), vmax = __int_as_float(0xff800000);
    for (int k = 0; k < 2; k++)
        for (int l = 0; l < 2; l++) {
            int x = 2 * i + k, y = 2 * j + l;
            if (x < nx && y < ny) { float t = u[(size_t)y * nx + x]; vmin = fminf(vmin, t); vmax = fmaxf(vmax, t); }
        }
    out[(size_t)j * onx + i] = (is_max ? vmax : vmin) * 0.5f;
}

// update_dmin_dmax (stereo_utils.cc:134-175).  disp, dminI/dmaxI (in) and omin/omax (out) are nx x ny;
// the fall-back images dminP/dmaxP are pnx x pny and are read at disp's coordinates clamped to THEIR size.
__global__ void update_ranges_kernel(const float *__restrict__ disp, float scale, int nx, int ny, const float *__restrict__ dminI,
                                     const float *__restrict__ dmaxI, const float *__restrict__ dminP, const float *__restrict__ dmaxP,
                                     int pnx, int pny, float slack, int radius, float *__restrict__ omin, float *__restrict__ omax)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= nx || j >= ny) return;
    float dmin = __int_as_float(0x7f800000), dmax = __int_as_float(0xff800000);
    for (int dj = -radius; dj <= radius; dj++)
        for (int di = -radius; di <= radius; di++) {
            int x = min(max(i + di, 0), nx - 1), y = min(max(j + dj, 0), ny - 1);
            float v = disp[(size_t)y * nx + x] * scale;         // upsample2x_disp doubles the coarse disparity first
            if (isfinite(v)) { dmin = fminf(dmin, v - slack); dmax = fmaxf(dmax, v + slack); }
            else {
                int px = min(max(i + di, 0), pnx - 1), py = min(max(j + dj, 0), pny - 1);
                dmin = fminf(dmin, dminP[(size_t)py * pnx + px]);
                dmax = fmaxf(dmax, dmaxP[(size_t)py * pnx + px]);
            }
        }
    size_t o = (size_t)j * nx + i;
    if (isfinite(dmin)) { omin[o] = dmin; omax[o] = dmax; }
    else { omin[o] = dminI ? dminI[o] : 0.f; omax[o] = dmaxI ? dmaxI[o] : 0.f; }
}

// zoom_nn by 2 (mgm_multiscale.cc:16-31)
__global__ void zoom2_kernel(const float *__restrict__ in, int inx, float *__restrict__ out, int nx, int ny)
{
    int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= nx || y >= ny) return;
    out[(size_t)y * nx + x] = in[(size_t)(y / 2) * inx + x / 2];
}

// first-level range images of one view (main_mgm_multi.cc:160-196)
__global__ void init_ranges_kernel(const float *__restrict__ img, int n, float lo_all, float hi_all, float sentinel,
                                   float *__restrict__ clean, float *__restrict__ dmin, float *__restrict__ dmax)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float v = img[i];
    bool isn = isnan(v);
    clean[i] = isfinite(v) ? v : 0.f;
    dmin[i] = isn ? sentinel : lo_all;
    dmax[i] = isn ? sentinel + 1.f : hi_all;
}

// float range images -> integer label ranges of one mgm_call (allocate_costvolume, mgm_costvolume.cc:63-72,
// after the scaling by ZOOMFACTOR of mgm_multiscale.cc:218-219) and their hull (hull[0] = min lo, hull[1] = max hi)
__global__ void label_ranges_kernel(const float *__restrict__ dmin, const float *__restrict__ dmax, int n, float zoom,
                                    short *__restrict__ lo, short *__restrict__ hi, int *hull)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    int l = 0x7fffffff, h = (int)0x80000000;
    if (i < n) {
        l = (int)floorf(dmin[i] * zoom);
        h = (int)ceilf(dmax[i] * zoom);
        lo[i] = (short)l; hi[i] = (short)h;
    }
    l = __reduce_min_sync(0xffffffffu, l);
    h = __reduce_max_sync(0xffffffffu, h);
    if ((threadIdx.x & 31) == 0) { atomicMin(hull, l); atomicMax(hull + 1, h); }
}

// ---- remove_small_cc (remove_small_cc.c:9-73): union-find over the 4-neighbour links the reference makes
// (only from pixels with i < w-1 and j < h-1; |difference| < threshold; NaN never joins), then every
// component with area <= minarea becomes NaN.  Any union-find yields the same partition.
__device__ __forceinline__ int uf_find(const int *lab, int a)
{   // read-only chase: parents only ever move towards smaller roots, so this terminates under concurrent unions
    while (true) { int p = ((const volatile int *)lab)[a]; if (p == a) return a; a = p; }
}
__device__ __forceinline__ void uf_union(int *lab, int a, int b)
{
    while (true) {
        a = uf_find(lab, a); b = uf_find(lab, b);
        if (a == b) return;
        if (a < b) { int t = a; a = b; b = t; }                            // a > b: hang the larger root below the smaller
        int old = atomicCAS(lab + a, a, b);
        if (old == a) return;
    }
}
__global__ void cc_init_kernel(const float *__restrict__ in, int n, int *__restrict__ lab, int *__restrict__ area)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { lab[i] = isnan(in[i]) ? -1 : i; area[i] = 0; }
}
// horizontal links: one warp per row.  A valid pixel whose left neighbour is invalid or not close starts a run; every
// pixel of a run is labelled with the run's first pixel, found by a running maximum of the start indices (an inclusive
// warp scan per 32-pixel chunk plus a carry) -- no atomics.  (The reference makes no horizontal link in the last row.)
__global__ void cc_rows_kernel(const float *__restrict__ in, int w, int h, float thr, int *lab)
{
    const int j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (j >= h - 1) return;
    const float *row = in + (size_t)j * w;
    int *l = lab + (size_t)j * w;
    int carry = -1;
    for (int i0 = 0; i0 < w; i0 += 32) {
        const int i = i0 + lane;
        const float a = i < w ? row[i] : __int_as_float(0x7fc00000);
        const bool valid = !isnan(a);
        float left = __shfl_up_sync(0xffffffffu, a, 1);
        if (lane == 0) left = i0 > 0 ? row[i0 - 1] : __int_as_float(0x7fc00000);
        const bool linked = valid && !isnan(left) && fabs((double)(left - a)) < (double)thr;
        int s = (valid && !linked) ? i : -1;                   // index of the run start at or before me, within the chunk
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const int o = __shfl_up_sync(0xffffffffu, s, d); if (lane >= d && o > s) s = o; }
        if (carry > s) s = carry;
        if (valid && i < w) l[i] = j * w + s;                  // a valid pixel always has a start at or before it
        carry = __shfl_sync(0xffffffffu, s, 31);
    }
}
// vertical links (none in the last column, as in the reference): union of the two runs' roots.  When the column to the
// left carries the same vertical link and both pixels continue their left neighbours' runs, the union is implied.
__global__ void cc_link_kernel(const float *__restrict__ in, int w, int h, float thr, int *lab)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= w - 1 || j >= h - 1) return;
    const int p0 = j * w + i, p2 = p0 + w;
    const float a = in[p0], b = in[p2];
    if (isnan(a) || isnan(b)) return;
    if (!(fabs((double)(a - b)) < (double)thr)) return;
    if (i > 0 && j + 1 < h - 1) {                              // row j+1 has horizontal links only if it is not the last row
        const float al = in[p0 - 1], bl = in[p2 - 1];
        if (!isnan(al) && !isnan(bl) && fabs((double)(al - bl)) < (double)thr &&
            fabs((double)(al - a)) < (double)thr && fabs((double)(bl - b)) < (double)thr) return;
    }
    uf_union(lab, p0, p2);
}
// every pixel points straight at its root (no unions run concurrently with this pass)
__global__ void cc_flatten_kernel(int n, int *lab)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && lab[i] >= 0) lab[i] = uf_find(lab, i);
}
// component areas: one atomic per distinct root and warp (a big component would otherwise serialise on one counter)
__global__ void cc_area_kernel(int n, const int *__restrict__ lab, int *area)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x, lane = threadIdx.x & 31;
    const int r = i < n ? lab[i] : -1;                         // flattened: the root itself
    const unsigned same = __match_any_sync(0xffffffffu, r);
    if (r >= 0 && lane == __ffs(same) - 1) atomicAdd(area + r, __popc(same));
}
__global__ void cc_filter_kernel(const float *__restrict__ in, int n, const int *__restrict__ lab, const int *__restrict__ area,
                                 int minarea, float *__restrict__ out)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int r = lab[i];                                      // flattened by cc_flatten_kernel
    out[i] = (r >= 0 && area[r] <= minarea) ? __int_as_float(0x7fc00000) : in[i];
}

}  // namespace s2pb
