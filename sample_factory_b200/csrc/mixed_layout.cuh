// Layout of a Tuple action space whose members are Discrete(n) or 1-D Box(d) spaces (TupleActionDistribution,
// action_distributions.py:197-286, with ActionParameterizationDefault, actor_critic.py:43-53): member k owns
//   params  columns [pofs, pofs + n)  (Discrete: logits)  or  [pofs, pofs + 2d)  ([means | log_std], torch.chunk(., 2))
//   actions columns [aofs, aofs + 1)  (the index, as a float)  or  [aofs, aofs + d)
//   noise   columns [nofs, nofs + n)  (Exp(1) per logit)      or  [nofs, nofs + d)  (N(0,1) per dimension)
// in member order (calc_num_action_parameters / calc_num_actions, action_distributions.py:16-44).
#pragma once
#include "common.cuh"

namespace sfb {

constexpr int kMixedMaxHeads = 8;
constexpr int kMixedMaxRows = 1024;
enum { kMixedCategorical = 0, kMixedGaussian = 1 };

struct MixedLayout {
    int K;
    int kind[kMixedMaxHeads];
    int size[kMixedMaxHeads];
    int pofs[kMixedMaxHeads], aofs[kMixedMaxHeads], nofs[kMixedMaxHeads];
    int A, W, Wn;   // params / actions / noise row widths
};

// builds the layout from the host arrays of the C ABI and checks it against A = rows of distribution_linear
static inline int make_mixed_layout(MixedLayout& ml, int A, int num_heads, const int32_t* kinds, const int32_t* sizes,
                                    const char* who) {
    SFB_CHECK_ARG(num_heads >= 1 && num_heads <= kMixedMaxHeads && kinds && sizes, "%s: 1 <= number of members <= %d", who,
                  kMixedMaxHeads);
    ml = MixedLayout{};
    ml.K = num_heads;
    int p = 0, a = 0, n = 0;
    for (int k = 0; k < num_heads; ++k) {
        SFB_CHECK_ARG(kinds[k] == kMixedCategorical || kinds[k] == kMixedGaussian,
                      "%s: member %d has kind %d (0 = categorical, 1 = Gaussian)", who, k, kinds[k]);
        SFB_CHECK_ARG(sizes[k] >= 1, "%s: member %d is empty", who, k);
        ml.kind[k] = kinds[k];
        ml.size[k] = sizes[k];
        ml.pofs[k] = p;
        ml.aofs[k] = a;
        ml.nofs[k] = n;
        const bool cat = kinds[k] == kMixedCategorical;
        p += cat ? sizes[k] : 2 * sizes[k];
        a += cat ? 1 : sizes[k];
        n += sizes[k];
    }
    SFB_CHECK_ARG(p == A && A <= kMixedMaxRows,
                  "%s: the members need %d distribution_linear rows, got A = %d (at most %d)", who, p, A, kMixedMaxRows);
    ml.A = p;
    ml.W = a;
    ml.Wn = n;
    return 0;
}

}  // namespace sfb
