// union_find.cuh -- the lock-free union-find of remove_small_cc (multiscale_kernels.cuh), shared with the other stages that
// label connected components (pointcloud_kernels.cuh, sgbm_kernels.cuh).  Device functions only: this header defines no
// kernel, so any translation unit may include it.
#pragma once
#include <cuda_runtime.h>

namespace s2pb {

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

}  // namespace s2pb
