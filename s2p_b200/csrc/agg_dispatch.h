// agg_dispatch.h -- host-side dispatch to the per-LPL instantiations of aggregate_kernel.
// Each agg_inst.cu object (compiled with -DS2PB_LPL=n) carries the four TSGM variants for one
// labels-per-lane value, so the instantiations build in parallel.
#pragma once
#include "agg_kernel.cuh"

namespace s2pb {
// The register-resident widths, in labels per lane (up to 512 labels).  The Makefile's LPLS builds one agg_inst object per entry.
#define S2PB_FOR_EACH_LPL(X) X(1) X(2) X(3) X(4) X(5) X(6) X(8) X(12) X(16)

template <int LPL, bool FOLD> int agg_launch_lpl(int tsgm, const AggArgs<FOLD> &P, int sm_count, cudaStream_t st, int ctas_per_sm);
template <int LPL> int agg_configure_lpl();
int agg_configure();                                   // 0 ok
// FOLD: the folded layout (AggFoldParams), one pass index of one or both views.
// ctas_per_sm > 0 caps the persistent CTAs per SM (two launches meant to share the SMs); 0 ok, -1 CUDA error, -2 unsupported
template <bool FOLD> int agg_launch(int LPL, int tsgm, const AggArgs<FOLD> &P, int sm_count, cudaStream_t st, int ctas_per_sm = 0);
// chunk-skipping aggregation of slabs wider than 512 slots (agg_chunked.cuh); 0 ok, -1 CUDA error, -2 shape not served
struct ChunkedParams;
struct ChunkedFoldParams;
int agg_chunked_configure();
// P: ChunkedArgs<FOLD> of agg_chunked.cuh, spelled out so that this header need not include the kernel
template <bool FOLD> int agg_chunked_launch(int tsgm, const std::conditional_t<FOLD, ChunkedFoldParams, ChunkedParams> &P, int sm_count,
                                            cudaStream_t st);
}  // namespace s2pb
