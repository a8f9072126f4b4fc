// fusion_kernels.cuh -- n-view height-map merge (SURVEY.md section 8f, rank 1).
//
// Behavioural reference: s2p/fusion.py:16-68.  merge_n stacks n float32 rasters as float64, subtracts one
// offset per raster, reduces every pixel's n values with an operator ('average_if_close': NaN when
// nanmax - nanmin > threshold, else nanmedian; or any np.* reducer named in the config), adds the mean offset and
// stores float32.  The reference runs the operator through np.apply_along_axis, i.e. one Python call per pixel; here
// it is one thread per pixel in float64.
//
// Which NumPy the reference runs under matters for `f.read(1) - offsets[i]` (float32 raster minus the 0-d float64
// array np.loadtxt returned, s2p/__init__.py:371-374): NumPy >= 2 (NEP 50) subtracts in float64, NumPy < 2
// (value-based casting) in float32.  `sub_f32` selects the latter; the Python drop-in asks the NumPy it runs under.
// Sums follow NumPy's pairwise scheme (8 accumulators from 8 values on), so np.mean / np.nanmean agree for every n.
//
// The rasters are read in the type they are stored in (fusion_kernel<float> or <double>): a float64 height map, which
// triangulation.height_map returns and common.rasterio_write keeps, is subtracted in float64 without a rounding to float32
// first, as `f.read(1) - offsets[i]` does with the float64 array rasterio returns for it (under any NumPy).
#pragma once
#include <cuda_runtime.h>

namespace s2pb {

constexpr int kMaxFusion = 16;
enum { FUSE_AVERAGE_IF_CLOSE = 0, FUSE_NANMEDIAN = 1, FUSE_NANMEAN = 2, FUSE_NANMIN = 3, FUSE_NANMAX = 4,
       FUSE_MEDIAN = 5, FUSE_MEAN = 6, FUSE_MIN = 7, FUSE_MAX = 8, FUSE_OP_COUNT = 9 };
struct FusionParams {
    const void *in[kMaxFusion];   // float or double rasters, as the kernel's instantiation reads them
    double offset[kMaxFusion];
    int n, op, sub_f32;
    double threshold, mean_offset;
    size_t npix;
    float *out;
};

// np.add.reduce over a short contiguous double vector (numpy/core/src/umath/loops_utils.h, pairwise_sum): plain loop
// below 8 values, else 8 running sums combined as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)) and the remainder added last
__device__ __forceinline__ double np_sum(const double *a, int n)
{
    if (n < 8) {
        double r = 0.0;            // numpy starts from -0.0; the difference cannot survive the + mean_offset below
        for (int i = 0; i < n; i++) r += a[i];
        return r;
    }
    double r[8];
    for (int j = 0; j < 8; j++) r[j] = a[j];
    int i = 8;
    for (; i < n - (n % 8); i += 8)
        for (int j = 0; j < 8; j++) r[j] += a[i + j];
    double res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; i++) res += a[i];
    return res;
}

// one stored value minus its offset, in float64 (sub_f32: in float32, NumPy < 2's rule for a float32 raster)
__device__ __forceinline__ double fusion_input(float in, double offset, int sub_f32)
{
    return sub_f32 ? (double)(in - (float)offset) : (double)in - offset;
}
__device__ __forceinline__ double fusion_input(double in, double offset, int) { return in - offset; }

template <typename T>
__global__ void fusion_kernel(const FusionParams P)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.npix) return;
    double v[kMaxFusion], a[kMaxFusion];
    int m = 0;
    for (int k = 0; k < P.n; k++) {
        const double x = fusion_input(static_cast<const T *>(P.in[k])[i], P.offset[k], P.sub_f32);
        a[k] = x;
        if (x == x) {                       // insertion sort of the non-NaN values
            int q = m++;
            while (q > 0 && v[q - 1] > x) { v[q] = v[q - 1]; q--; }
            v[q] = x;
        }
    }
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    double r = nan;
    const bool nanaware = P.op <= FUSE_NANMAX;
    if (m > 0 && (nanaware || m == P.n)) {  // the plain reducers return NaN as soon as one value is NaN
        const double mn = v[0], mx = v[m - 1];
        const double med = (m & 1) ? v[m / 2] : 0.5 * (v[m / 2 - 1] + v[m / 2]);   // mean of the two middle values
        switch (P.op) {
        case FUSE_AVERAGE_IF_CLOSE: r = (mx - mn > P.threshold) ? nan : med; break;
        case FUSE_NANMEDIAN: case FUSE_MEDIAN: r = med; break;
        case FUSE_NANMEAN: case FUSE_MEAN:
            for (int k = 0; k < P.n; k++) if (a[k] != a[k]) a[k] = 0.0;            // np.nanmean: NaN -> 0, sum, / count
            r = np_sum(a, P.n) / (double)m;
            break;
        case FUSE_NANMIN: case FUSE_MIN: r = mn; break;
        default: r = mx; break;
        }
    }
    P.out[i] = (float)(r + P.mean_offset);
}

}  // namespace s2pb
