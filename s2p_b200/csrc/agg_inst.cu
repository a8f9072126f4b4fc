// agg_inst.cu -- instantiates aggregate_kernel<S2PB_LPL, TSGM, SCALED, GEN> for TSGM = 1..4: census popcounts,
// census through the scaling table (windows 3 / 7), and the general flavour (float costs / weights).
#include "agg_dispatch.h"
#ifndef S2PB_LPL
#error "compile with -DS2PB_LPL=<labels per lane>"
#endif

namespace s2pb {

static constexpr int kLPL = S2PB_LPL;
static constexpr size_t kSmem = AggSmem<kLPL, false>::bytes, kSmemGen = AggSmem<kLPL, true>::bytes;

template <> int agg_configure_lpl<kLPL>()
{
    cudaError_t e = cudaSuccess;
#define CFG(T, S, G) e = cudaFuncSetAttribute(aggregate_kernel<kLPL, T, S, G>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(G ? kSmemGen : kSmem)); if (e) return -1; \
    if (kLPL > 4 && AggOcc<kLPL, T>::ctas == 2) { /* two CTAs of up to 113 KB: ask for the largest shared-memory carve-out */ \
        e = cudaFuncSetAttribute(aggregate_kernel<kLPL, T, S, G>, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared); if (e) return -1; }
    CFG(1, false, false) CFG(2, false, false) CFG(3, false, false) CFG(4, false, false)
    CFG(1, true, false) CFG(2, true, false) CFG(3, true, false) CFG(4, true, false)
    CFG(1, false, true) CFG(2, false, true) CFG(3, false, true) CFG(4, false, true)
#undef CFG
    return 0;
}

template <> int agg_launch_lpl<kLPL>(int tsgm, const AggParams &P, int sm_count, cudaStream_t st, int ctas_per_sm)
{
    // persistent CTAs, one (or two) per SM; bands are pulled from a global queue in dependency order
    const int total = P.maxBands * P.nPV;
    dim3 block(kAggThreads);
    const bool scaled = P.lut != nullptr;
#define GO(T) do { int per = AggOcc<kLPL, T>::ctas; if (ctas_per_sm > 0 && ctas_per_sm < per) per = ctas_per_sm; \
                   int grid = sm_count * per; if (grid > total) grid = total; \
                   if (P.general) aggregate_kernel<kLPL, T, false, true><<<grid, block, kSmemGen, st>>>(P); \
                   else if (scaled) aggregate_kernel<kLPL, T, true, false><<<grid, block, kSmem, st>>>(P); \
                   else aggregate_kernel<kLPL, T, false, false><<<grid, block, kSmem, st>>>(P); } while (0)
    switch (tsgm) {
    case 1: GO(1); break;
    case 2: GO(2); break;
    case 3: GO(3); break;
    case 4: GO(4); break;
    default: return -2;
    }
#undef GO
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

}  // namespace s2pb
static_assert(s2pb::AggSmem<S2PB_LPL, false>::bytes <= 227 * 1024 && s2pb::AggSmem<S2PB_LPL, true>::bytes <= 227 * 1024,
              "aggregation CTA exceeds the 227 KB of shared memory of an sm_90 SM");
