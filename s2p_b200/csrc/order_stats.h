// order_stats.h -- the state of the radix select of sgbm_kernels.cuh (sgbm_hist_kernel / sgbm_select_kernel), which
// sgbm.cu runs for qauto's thresholds and for the 8-bit stretch of the point-cloud colours (launch_order_stats, host.h).
#pragma once

namespace s2pb {

// Order statistics of the non-NaN floats of a buffer by radix select: four passes of 8-bit digits on order-preserving keys,
// every wanted rank at once.  The ranks follow from the count n, which the first pass finds, by one of two rules.
constexpr int kOrdMaxRanks = 4;
enum { kOrdQauto = 0, kOrdLinear = 1 };
struct OrderStats {
    unsigned prefix[kOrdMaxRanks];   // key bits found so far, per rank
    unsigned rank[kOrdMaxRanks];     // ... rank still to find below that prefix
    int n;                           // number of non-NaN values
    int nranks;
    int rule;                        // kOrdQauto, kOrdLinear
    double q[2];                     // kOrdLinear: the two quantiles
    float v[kOrdMaxRanks];           // after the last pass: the order statistics
    float rmin, rmax;                // kOrdQauto: qauto's thresholds
    double lo, hi;                   // kOrdLinear: the two quantiles of numpy's 'linear' method (NaN when n == 0)
};

}  // namespace s2pb
