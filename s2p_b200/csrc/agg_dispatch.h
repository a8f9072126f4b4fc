// agg_dispatch.h -- host-side dispatch to the per-LPL instantiations of aggregate_kernel.
// Each agg_inst.cu object (compiled with -DS2PB_LPL=n) carries the four TSGM variants for one
// labels-per-lane value, so the instantiations build in parallel.
#pragma once
#include "agg_kernel.cuh"

namespace s2pb {
// The register-resident widths, in labels per lane (up to 512 labels).  The Makefile's LPLS builds one agg_inst object per entry.
#define S2PB_FOR_EACH_LPL(X) X(1) X(2) X(3) X(4) X(5) X(6) X(8) X(12) X(16)

template <int LPL> int agg_launch_lpl(int tsgm, const AggParams &P, int sm_count, cudaStream_t st, int ctas_per_sm);
template <int LPL> int agg_fold_launch_lpl(int tsgm, const AggFoldParams &P, int sm_count, cudaStream_t st);
template <int LPL> int agg_configure_lpl();
int agg_configure();                                   // 0 ok
// ctas_per_sm > 0 caps the persistent CTAs per SM (two launches meant to share the SMs); 0 ok, -1 CUDA error, -2 unsupported
int agg_launch(int LPL, int tsgm, const AggParams &P, int sm_count, cudaStream_t st, int ctas_per_sm = 0);
// the folded layout (AggFoldParams): one pass index of one or both views; same return codes
int agg_fold_launch(int LPL, int tsgm, const AggFoldParams &P, int sm_count, cudaStream_t st);
// chunk-skipping aggregation of slabs wider than 512 slots (agg_chunked.cuh); 0 ok, -1 CUDA error, -2 shape not served
struct ChunkedParams;
struct ChunkedFoldParams;
int agg_chunked_configure();
int agg_chunked_launch(int tsgm, const ChunkedParams &P, int sm_count, cudaStream_t st);
int agg_chunked_fold_launch(int tsgm, const ChunkedFoldParams &P, int sm_count, cudaStream_t st);
}  // namespace s2pb
