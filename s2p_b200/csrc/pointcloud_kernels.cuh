// pointcloud_kernels.cuh -- the 3D outlier filter of triangulation: count_3d_neighbors and remove_isolated_3d_points
// (c/disp_to_h.c:143-230), which s2p.triangulation.filter_xyz runs on the (h, w, 3) cloud of a tile.
//
// Counting: one thread per pixel compares its point with every point of its (2p+1)^2 window, clipped at the image border.
// A CTA stages its 16x16 tile plus the p-halo in shared memory as three double arrays (SoA: 24-byte AoS records would
// put the lanes of a warp on conflicting banks); when the halo does not fit, the same loop reads the neighbours through
// L1 / L2 instead.  Both give the same integer: the loop, the distance and the comparison are the same.
//
// Rejection: the reference rejects the points with count < n, then sweeps the grid until no sweep changes anything,
// un-rejecting each rejected point that has a close, non-rejected point in its (2q+1)^2 window.  The distance is
// symmetric bit for bit and un-rejecting only goes one way, so the sweeps end on an order-free set: a rejected point is
// saved iff a chain of "close and within the q-window" links through rejected points joins it to a point that was never
// rejected.  Here that is a connected-components pass over the rejected pixels (union_find.cuh, flattened by
// remove_small_cc's cc_flatten_kernel), bounded work where the sweeps need as many passes as the longest chain against the
// scan order.
#pragma once
#include <cuda_runtime.h>
#include "union_find.cuh"

namespace s2pb {

constexpr int kPcTile = 16;        // CTA tile of the count kernel: kPcTile x kPcTile pixels, one thread each

// squared_distance_between_3d_points (c/disp_to_h.c:143-149) as the reference's build evaluates it: the differences in
// double, each rounded to float, then y*y and two fused multiply-adds (gcc contracts x*x + y*y + z*z into
// fma(z, z, fma(x, x, y*y))).  Rounding is explicit, whatever -fmad says.  Symmetric: float(a - b) == -float(b - a).
__device__ __forceinline__ float pc_sqdist(double ax, double ay, double az, double bx, double by, double bz)
{
    const float x = __double2float_rn(__dsub_rn(ax, bx));
    const float y = __double2float_rn(__dsub_rn(ay, by));
    const float z = __double2float_rn(__dsub_rn(az, bz));
    return __fmaf_rn(z, z, __fmaf_rn(x, x, __fmul_rn(y, y)));
}
__device__ __forceinline__ bool pc_has_nan(double a, double b, double c) { return isnan(a) || isnan(b) || isnan(c); }

// count[y][x] = #{ points u of the clipped (2p+1)^2 window with d(u, centre) < r*r }  (count_3d_neighbors, :152-174).
// 0 <= p <= max(nx, ny) (the host clamps: a wider window is the whole image).  kStaged: the CTA's window footprint,
// clipped to the image, sits in dynamic shared memory (the host checks that it fits).  A centre with a NaN coordinate
// makes every distance NaN, so its count is 0 without the loop.
template <bool kStaged>
__global__ void __launch_bounds__(kPcTile * kPcTile) pc_count_kernel(const double *__restrict__ xyz, int nx, int ny, float r, int p,
                                                                     int *__restrict__ count)
{
    extern __shared__ double pc_sm[];
    const int x0 = blockIdx.x * kPcTile, y0 = blockIdx.y * kPcTile;
    const int x = x0 + threadIdx.x, y = y0 + threadIdx.y;
    const int sx0 = max(x0 - p, 0), sy0 = max(y0 - p, 0);
    const int sw = min(x0 + kPcTile - 1 + p, nx - 1) - sx0 + 1, sh = min(y0 + kPcTile - 1 + p, ny - 1) - sy0 + 1;
    const double *sX = pc_sm, *sY = pc_sm + sw * sh, *sZ = pc_sm + 2 * sw * sh;
    if (kStaged) {
        for (int k = threadIdx.y * kPcTile + threadIdx.x; k < sw * sh; k += kPcTile * kPcTile) {
            const int i = k / sw, j = k - i * sw;
            const double *u = xyz + 3 * ((size_t)(sy0 + i) * nx + sx0 + j);
            pc_sm[k] = u[0]; pc_sm[sw * sh + k] = u[1]; pc_sm[2 * sw * sh + k] = u[2];
        }
        __syncthreads();
    }
    if (x >= nx || y >= ny) return;
    const size_t pix = (size_t)y * nx + x;
    const double vx = xyz[3 * pix], vy = xyz[3 * pix + 1], vz = xyz[3 * pix + 2];
    const float rr = __fmul_rn(r, r);
    int c = 0;
    if (!pc_has_nan(vx, vy, vz)) {
        const int i0 = max(y - p, 0), i1 = min(y + p, ny - 1), j0 = max(x - p, 0), j1 = min(x + p, nx - 1);
        for (int i = i0; i <= i1; i++) {
            if (kStaged) {
                const int row = (i - sy0) * sw - sx0;
#pragma unroll 4
                for (int j = j0; j <= j1; j++)
                    c += pc_sqdist(sX[row + j], sY[row + j], sZ[row + j], vx, vy, vz) < rr;
            } else {
                const double *u = xyz + 3 * (size_t)i * nx;
#pragma unroll 4
                for (int j = j0; j <= j1; j++)
                    c += pc_sqdist(__ldg(u + 3 * j), __ldg(u + 3 * j + 1), __ldg(u + 3 * j + 2), vx, vy, vz) < rr;
            }
        }
    }
    count[pix] = c;
}

// rejected pixels (count < n) start as their own union-find roots, kept ones are -1; no root is saved yet
__global__ void pc_label_kernel(const int *__restrict__ count, int npix, int n, int *__restrict__ lab, int *__restrict__ saved)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npix) return;
    lab[i] = count[i] < n ? i : -1;
    saved[i] = 0;
}

// joins every close pair of rejected pixels within the q-window, each pair once: from the earlier pixel in raster order
// to the later half of its window.  Rejected stays rejected here, so the sign of lab[] is stable under the unions.
__global__ void pc_link_kernel(const double *__restrict__ xyz, int nx, int ny, float r, int q, int *lab)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= nx || y >= ny) return;
    const int i = y * nx + x;
    if (lab[i] < 0) return;
    const double vx = xyz[3 * (size_t)i], vy = xyz[3 * (size_t)i + 1], vz = xyz[3 * (size_t)i + 2];
    if (pc_has_nan(vx, vy, vz)) return;                      // a NaN point is close to nothing
    const float rr = __fmul_rn(r, r);
    for (int yy = y; yy <= min(y + q, ny - 1); yy++)
        for (int xx = yy == y ? x + 1 : max(x - q, 0); xx <= min(x + q, nx - 1); xx++) {
            const int j = yy * nx + xx;
            if (lab[j] >= 0 && pc_sqdist(vx, vy, vz, xyz[3 * (size_t)j], xyz[3 * (size_t)j + 1], xyz[3 * (size_t)j + 2]) < rr)
                uf_union(lab, i, j);
        }
}

// after cc_flatten_kernel: the component of every rejected pixel with a close, kept pixel in its q-window is saved
__global__ void pc_mark_kernel(const double *__restrict__ xyz, int nx, int ny, float r, int q, const int *__restrict__ lab,
                               int *__restrict__ saved)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= nx || y >= ny) return;
    const int i = y * nx + x, root = lab[i];
    if (root < 0) return;
    const double vx = xyz[3 * (size_t)i], vy = xyz[3 * (size_t)i + 1], vz = xyz[3 * (size_t)i + 2];
    if (pc_has_nan(vx, vy, vz)) return;
    const float rr = __fmul_rn(r, r);
    for (int yy = max(y - q, 0); yy <= min(y + q, ny - 1); yy++)
        for (int xx = max(x - q, 0); xx <= min(x + q, nx - 1); xx++) {
            const int j = yy * nx + xx;
            if (lab[j] < 0 && pc_sqdist(vx, vy, vz, xyz[3 * (size_t)j], xyz[3 * (size_t)j + 1], xyz[3 * (size_t)j + 2]) < rr) {
                saved[root] = 1;
                return;
            }
        }
}

// the rejected points of unsaved components become NaN, all three coordinates
__global__ void pc_reject_kernel(int npix, const int *__restrict__ lab, const int *__restrict__ saved, double *__restrict__ xyz)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npix) return;
    const int root = lab[i];
    if (root < 0 || saved[root]) return;
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    xyz[3 * (size_t)i] = nan; xyz[3 * (size_t)i + 1] = nan; xyz[3 * (size_t)i + 2] = nan;
}

}  // namespace s2pb
