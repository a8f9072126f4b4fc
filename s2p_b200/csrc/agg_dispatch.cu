// agg_dispatch.cu -- run-time switch over the labels-per-lane instantiations.
#include "agg_dispatch.h"

namespace s2pb {

#define DECL(n) template <> int agg_configure_lpl<n>();
S2PB_FOR_EACH_LPL(DECL)
#undef DECL

int agg_configure()
{
#define CFG(n) if (agg_configure_lpl<n>() != 0) return -1;
    S2PB_FOR_EACH_LPL(CFG)
#undef CFG
    return 0;
}

template <bool FOLD> int agg_launch(int LPL, int tsgm, const AggArgs<FOLD> &P, int sm_count, cudaStream_t st, int ctas_per_sm)
{
    switch (LPL) {
#define CASE(n) case n: return agg_launch_lpl<n, FOLD>(tsgm, P, sm_count, st, ctas_per_sm);
    S2PB_FOR_EACH_LPL(CASE)
#undef CASE
    default: return -2;
    }
}
template int agg_launch<false>(int, int, const AggParams &, int, cudaStream_t, int);
template int agg_launch<true>(int, int, const AggFoldParams &, int, cudaStream_t, int);

}  // namespace s2pb
