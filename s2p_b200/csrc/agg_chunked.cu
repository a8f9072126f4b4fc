// agg_chunked.cu -- instantiations and launcher of the chunk-skipping aggregation (agg_chunked.cuh).
#include "agg_chunked.cuh"
#include "agg_dispatch.h"

namespace s2pb {

static constexpr int kCkMaxSmem = 224 * 1024;      // dynamic part: the 227 KB opt-in limit minus the static shared memory of the kernel

int agg_chunked_configure()
{
    cudaError_t e = cudaSuccess;
#define CFG(T, S) e = cudaFuncSetAttribute(aggregate_chunked_kernel<T, S, 4, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kCkMaxSmem); if (e) return -1; \
                  e = cudaFuncSetAttribute(aggregate_chunked_kernel<T, S, 2, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kCkMaxSmem); if (e) return -1;
    CFG(1, false) CFG(2, false) CFG(3, false) CFG(4, false) CFG(1, true) CFG(2, true) CFG(3, true) CFG(4, true)
#undef CFG
#define CFG_GEN(T) e = cudaFuncSetAttribute(aggregate_chunked_kernel<T, false, 2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kCkMaxSmem); if (e) return -1;
    CFG_GEN(1) CFG_GEN(2) CFG_GEN(3) CFG_GEN(4)
#undef CFG_GEN
    return 0;
}

// 0 ok, -1 CUDA error, -2 this shape is not served (the caller then uses the dense kernel)
int agg_chunked_launch(int tsgm, const ChunkedParams &P, int sm_count, cudaStream_t st)
{
    if (P.DP < 32 || P.DP > 2048 || (P.DP & 31)) return -2;
    const bool gen = P.A.general != 0;          // float costs (and weights): no cost table, pipeline depth 2 (ck_stage)
    const int warps = ck_warps(P.DP, gen), stage = ck_stage(P.DP, gen);
    const CkSmem SM(P.DP, warps, stage, gen);
    if (SM.bytes > (size_t)kCkMaxSmem) return -2;
    int maxBands = 0;
    for (int v = 0; v < P.A.nPV; v++) { const int nb = (P.A.pv[v].nS + warps - 1) / warps; if (nb > maxBands) maxBands = nb; }
    const int total = maxBands * P.A.nPV;
    const int per_sm = (int)(kCkMaxSmem / (SM.bytes + 1024)) >= 2 ? 2 : 1;      // 512-thread CTAs: at most two per SM
    int grid = sm_count * per_sm;
    if (grid > total) grid = total;
    const bool scaled = P.A.lut != nullptr;
    const int threads = warps * 32;
#define GO2(T, ST) do { if (scaled) aggregate_chunked_kernel<T, true, ST, false><<<grid, threads, SM.bytes, st>>>(P); \
                        else aggregate_chunked_kernel<T, false, ST, false><<<grid, threads, SM.bytes, st>>>(P); } while (0)
#define GO(T) do { if (gen) aggregate_chunked_kernel<T, false, 2, true><<<grid, threads, SM.bytes, st>>>(P); \
                   else if (stage == 4) GO2(T, 4); else GO2(T, 2); } while (0)
    switch (tsgm) {
    case 1: GO(1); break;
    case 2: GO(2); break;
    case 3: GO(3); break;
    case 4: GO(4); break;
    default: return -2;
    }
#undef GO
#undef GO2
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

}  // namespace s2pb
