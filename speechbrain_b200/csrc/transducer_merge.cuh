// Arg-max and log-sum-exp partials of the transducer search (transducer.cu), host- and device-callable so that a CPU
// test can check them on non-finite logits.
//
// The order is torch.max's: NaN ranks above every number (the first NaN wins), equal values keep the smaller index.  It
// is a strict total order on (value, index), so any merge order (the kernel's lane-strided scan, shuffle tree and
// cross-CTA fold) picks the same element.  The decision follows the reference, which takes torch.max of the LOG-PROBS:
// when the row's maximum is not finite (a NaN or +inf logit, or every logit -inf), log_softmax makes every entry NaN
// and the reference picks index 0.  The token indexes the U table, so it never leaves [0, V) whatever the inputs.
#pragma once
#include <climits>
#include <cmath>

#ifdef __CUDACC__
#define TD_HD __host__ __device__ __forceinline__
#else
#define TD_HD inline
#endif

namespace sbk {
namespace td {

constexpr int NO_ARG = INT_MAX;   // arg-max of an empty slice

// does (x, ix) come before (m, im) in torch.max's order?
TD_HD bool argmax_before(float x, int ix, float m, int im) {
    const bool nx = x != x, nm = m != m;
    if (nx != nm) return nx;
    if (!nx && x != m) return x > m;
    return ix < im;
}

// fold the partial (m2, a2, s2) = (max, arg-max, sum exp(x - max)) into (m, a, s)
TD_HD void lse_merge(float& m, int& a, float& s, float m2, int a2, float s2) {
    if (a2 == NO_ARG) return;
    if (a == NO_ARG) { m = m2; a = a2; s = s2; return; }
    const bool take = argmax_before(m2, a2, m, a);
    const float M = take ? m2 : m;
    s = s * expf(m - M) + s2 * expf(m2 - M);
    if (take) a = a2;
    m = M;
}

// the token of a decision from the merged (max, arg-max): index 0 when the maximum is not finite, as the reference's
// arg-max of an all-NaN log-prob row
TD_HD int decision(float m, int a, int V) {
    return (m != m || m == INFINITY || m == -INFINITY || a < 0 || a >= V) ? 0 : a;
}

}  // namespace td
}  // namespace sbk
