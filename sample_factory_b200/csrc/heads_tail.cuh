// The distribution tail of the policy heads and the action layout it walks.  row_tail samples every action space from
// a row held in registers (heads_wide.cu: stored params rows of any width); heads_row_tail is the same math on one
// element per lane for the narrow heads (heads.cu stand-alone kernels, and gemm_tc.cu, whose fused GEMM finishes the
// heads in its last-arriving CTA).
#pragma once
#include <curand_kernel.h>

#include "common.cuh"
#include "mixed_layout.cuh"

namespace sfb {

// A Box with adaptive_stddev=0: one learned log-stddev vector instead of a log-stddev half of the params row
enum { kMixedGaussianLearned = 2 };

// The action space as the tail walks it: the members of mixed_layout.cuh (a Discrete space is one categorical member,
// a Tuple of Discretes one per head, a Box one Gaussian member), where each member writes its env actions, the
// learned-stddev fields of a Box, and the calling thread's sampling mode.
struct ActionLayout {
    MixedLayout m;                      // m.A = rows of distribution_linear (the elements of a row the tail reads)
    void* env[kMixedMaxHeads];          // per member: int32 [rows, stride] (categorical) or float32 [rows, stride]; may be null
    int env_stride[kMixedMaxHeads];
    const float* learned_log_std; float tanh_scale;   // kMixedGaussianLearned (action_parameterization.py:64-78)
    // sampling mode (sfb200_set_sampling_mode): action_mask[row * mask_stride + a] == 0 forbids action a of a plain
    // Discrete space (masked_softmax / masked_log_softmax, action_distributions.py:84-95); deterministic = argmax of the
    // probabilities / the Gaussian means instead of a draw (enjoy.py:165-171 eval_deterministic)
    const uint8_t* action_mask; int64_t mask_stride; int deterministic;
};

struct HeadsOut {
    float* values; int64_t values_stride;
    float* logits; int64_t logits_stride;     // the params rows: logits / [means | log_std]
    float* actions_f32; int64_t actions_stride;
    float* log_prob; int64_t log_prob_stride;
    float* pv_out; int64_t pv_stride;
    ActionLayout lay;
};

// Fills out.lay for one action space of the C ABI and applies the calling host thread's sampling mode
// (sfb200_set_sampling_mode).  space: 0 Discrete(A); 1 Tuple of Discrete(sizes[k]); 2 Box(act_dim) with its log-stddev
// in the row (adaptive_stddev) or learned; 3 Tuple of Discrete / Box members (kinds, sizes).  env_actions is the env
// action buffer of spaces 0-2, env_members the per-member buffers of space 3.  who prefixes the error messages.
int make_heads_layout(HeadsOut& out, int space, int A, int num_heads, const int32_t* kinds, const int32_t* sizes,
                      int act_dim, int adaptive_stddev, const float* learned_log_std, float tanh_scale, void* env_actions,
                      void* const* env_members, const char* who);

constexpr float kStddevMin = 1e-4f, kStddevMax = 1e4f;   // action_distributions.py:291-292
constexpr float kHalfLog2Pi = 0.91893853320467274178f;   // log(sqrt(2 pi))

// argmax of (best, idx) pairs over an aligned group of G lanes (G = 32: the warp), first index on ties
template <int G = 32>
__device__ __forceinline__ void argmax_first(float& best, int& idx) {   // torch.multinomial(p, 1) == argmax(p / q)
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
        if (ob > best || (ob == best && oi < idx)) { best = ob; idx = oi; }
    }
}

// Draw number i of a row's noise: the explicit noise[i] if given, else Philox subsequence i at `offset`.
// Exp(1) for the categorical race (curand_uniform is in (0, 1]), N(0, 1) for a Gaussian.
__device__ __forceinline__ float exp1_draw(const float* __restrict__ noise, int64_t i, uint64_t seed, uint64_t offset) {
    if (noise) return noise[i];
    curandStatePhilox4_32_10_t st;
    curand_init(seed, (unsigned long long)i, offset, &st);
    return fmaxf(-logf(curand_uniform(&st)), 1.0e-30f);
}
__device__ __forceinline__ float normal_draw(const float* __restrict__ noise, int64_t i, uint64_t seed, uint64_t offset) {
    if (noise) return noise[i];
    curandStatePhilox4_32_10_t st;
    curand_init(seed, (unsigned long long)i, offset, &st);
    return curand_normal(&st);
}

// CategoricalActionDistribution (action_distributions.py:110-148) of one row on an aligned group of G lanes, as
// heads_row_tail runs it on a warp: the lane holding logit a (a < A, at group position (a + 1) % G) passes x = the logit
// and its index a; the other lanes pass a >= A.  draw: sample with draw number row_draw0 + a (exp1_draw); otherwise
// q = 1.  Returns the sampled index on every lane of the group, and its log-prob (:145-148) in lp.
// The reductions are xor butterflies from G/2 down to 1.  G = 8 gives the bits of the 32-lane warp for up to 8 logits:
// on 32 lanes (logit a on lane a + 1) the xor-16 and xor-8 steps only add exact zeros or take the max with -inf, after
// which lane (a + 1) % 8 holds logit a -- the layout of an 8-lane group -- and the xor-4, 2, 1 steps associate the same
// terms.
template <int G>
__device__ __forceinline__ int categorical_draw(float x_in, int a, int A, bool draw, const float* __restrict__ noise,
                                                int64_t row_draw0, uint64_t seed, uint64_t offset, float& lp) {
    const bool is_logit = a < A;
    const float x = is_logit ? x_in : -INFINITY;
    float m = x;
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    const float e = is_logit ? expf(x - m) : 0.f;
    float s = e;
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float p = __fdiv_rn(e, s);                    // softmax :116
    const float logp = (x - m) - logf(s);               // log_softmax :125
    const float q = (is_logit && draw) ? exp1_draw(noise, row_draw0 + a, seed, offset) : 1.f;
    // torch.multinomial(p, 1, True) == argmax(p / q) (first index on ties)
    float best = is_logit ? __fdiv_rn(p, q) : -INFINITY;
    int idx = is_logit ? a : 0x7fffffff;
    argmax_first<G>(best, idx);
    lp = __shfl_sync(0xffffffffu, logp, (idx + 1) & (G - 1), G);
    return idx;
}

// Slot k of lane l holds element (32k + l - S) mod 32*LPL of the row.  S = 1 leaves lane 0 free for the value: up to
// 31 elements sit on lane a+1, and a row of exactly 32*LPL elements puts the last one in slot 0.  The slot map fixes
// which terms every lane-local sum and warp reduction adds in which order, so it fixes the bits of the results.
template <int LPL, int S>
__device__ __forceinline__ int slot_elem(int k, int lane) {
    return (k * 32 + lane - S) & (32 * LPL - 1);
}

// The distribution tail of one row held in registers, x[k] = element slot_elem(k, lane) (elements >= out.lay.m.A are
// never read).  Per member: CategoricalActionDistribution (action_distributions.py:110-148, with the optional mask of a
// plain Discrete space) or ContinuousActionDistribution (:290-323); log_prob is the sum over the members (:231-241).
// Noise and Philox subsequences are indexed row * Wn + nofs + j.  Elements outside a member contribute -inf to maxima
// and an exact 0 to sums.  The adaptive log-stddev of a Gaussian member comes from the partner lane at LPL = 1 and from
// the stored params row (out.logits) otherwise; a learned-stddev row is completed in out.logits.
// Returns the index sampled for the last categorical member (a plain Discrete space's action), -1 if none.
template <int LPL, int S>
__device__ __forceinline__ int row_tail(const float (&x)[LPL], int lane, int64_t row, const HeadsOut& out,
                                        const float* __restrict__ noise, uint64_t seed, uint64_t offset, float pv) {
    const ActionLayout& L = out.lay;
    float lp_total = 0.f;
    int act = -1;
#pragma unroll 1
    for (int s = 0; s < L.m.K; ++s) {
        const int po = L.m.pofs[s], n = L.m.size[s], no = L.m.nofs[s], ao = L.m.aofs[s];
        if (L.m.kind[s] == kMixedCategorical) {
            if (out.actions_f32 == nullptr) continue;   // values / logits only (warp-uniform)
            const bool masked = L.action_mask != nullptr;
            bool ok[LPL];
            // the logit of slot k; masked_softmax / masked_log_softmax :84-95: a forbidden logit gets -1e9 added
            auto logit = [&](int k) {
                const bool in = (unsigned)(slot_elem<LPL, S>(k, lane) - po) < (unsigned)n;
                return in ? ((masked && !ok[k]) ? __fadd_rn(x[k], -1.0e9f) : x[k]) : -INFINITY;
            };
            float mloc = -INFINITY;
#pragma unroll
            for (int k = 0; k < LPL; ++k) {
                const int j = slot_elem<LPL, S>(k, lane) - po;
                ok[k] = (unsigned)j < (unsigned)n && (!masked || L.action_mask[row * L.mask_stride + j] != 0);
                mloc = k == 0 ? logit(k) : fmaxf(mloc, logit(k));
            }
            const float m = warp_max(mloc);
            float p[LPL], sl = 0.f;
#pragma unroll
            for (int k = 0; k < LPL; ++k) {
                p[k] = ((unsigned)(slot_elem<LPL, S>(k, lane) - po) < (unsigned)n) ? expf(logit(k) - m) : 0.f;
                sl += p[k];
            }
            const float sum = warp_sum(sl);
            const float logs = logf(sum);
#pragma unroll
            for (int k = 0; k < LPL; ++k) p[k] = __fdiv_rn(p[k], sum);             // softmax :116
            if (masked) {
                float ps = 0.f;
#pragma unroll
                for (int k = 0; k < LPL; ++k) {
                    p[k] = __fmul_rn(p[k], ok[k] ? 1.f : 0.f);                     // :88
                    ps += p[k];
                }
                const float den = __fadd_rn(warp_sum(ps), 1.0e-13f);               // :89
                bool any = false;
#pragma unroll
                for (int k = 0; k < LPL; ++k) {
                    p[k] = __fdiv_rn(p[k], den);
                    any |= p[k] > 0.f;
                }
                if (__ballot_sync(0xffffffffu, any) == 0u)                         // :137-140 nothing allowed: uniform
#pragma unroll
                    for (int k = 0; k < LPL; ++k) p[k] = 1.0e-6f;
            }
            // one row element per lane: the log-prob of every slot is formed before the draw, so that m and logs die
            // before the Philox state is live (log_softmax :125)
            const float logp1 = LPL == 1 ? (logit(0) - m) - logs : 0.f;
            float best = -INFINITY;
            int idx = 0x7fffffff;
#pragma unroll
            for (int k = 0; k < LPL; ++k) {
                const int j = slot_elem<LPL, S>(k, lane) - po;
                if ((unsigned)j >= (unsigned)n) continue;
                const float q = L.deterministic ? 1.f : exp1_draw(noise, row * L.m.Wn + no + j, seed, offset);
                const float r = __fdiv_rn(p[k], q);
                if (k == 0 || r > best || (r == best && j < idx)) { best = r; idx = j; }
            }
            argmax_first(best, idx);
            const int q = (po + idx + S) & (32 * LPL - 1);                          // the slot of the chosen logit
            float mine = logp1;
#pragma unroll
            for (int k = 0; k < LPL; ++k)
                if (LPL > 1 && k == (q >> 5)) mine = (logit(k) - m) - logs;
            lp_total += __shfl_sync(0xffffffffu, mine, q & 31);                     // log_prob :145-148
            if (lane == 0) {
                out.actions_f32[row * out.actions_stride + ao] = (float)idx;
                if (L.env[s]) static_cast<int32_t*>(L.env[s])[row * L.env_stride[s]] = idx;
            }
            act = idx;
        } else {
            const bool learned = L.m.kind[s] == kMixedGaussianLearned;
            float* pr = out.logits ? out.logits + row * out.logits_stride : nullptr;
            // the log-stddev of a dimension sits n elements after its mean: on lane + n at LPL = 1
            const float partner = (LPL == 1 && !learned) ? __shfl_sync(0xffffffffu, x[0], (lane + n) & 31) : 0.f;
            float lps = 0.f;
#pragma unroll
            for (int k = 0; k < LPL; ++k) {
                const int j = slot_elem<LPL, S>(k, lane) - po;
                if ((unsigned)j >= (unsigned)n) continue;
                float mean = x[k], log_std;
                if (!learned) {
                    log_std = LPL == 1 ? partner : pr[po + n + j];
                } else {
                    log_std = L.learned_log_std[j];
                    if (L.tanh_scale > 0.f) mean = tanhf(__fdiv_rn(mean, L.tanh_scale)) * L.tanh_scale;
                    if (pr) {            // the params row the reference returns: tanh-scaled means, the repeated vector
                        pr[po + j] = mean;
                        pr[po + n + j] = log_std;
                    }
                }
                if (out.actions_f32 == nullptr) continue;   // distribution parameters only (warp-uniform)
                const float sd = clampf(expf(log_std), kStddevMin, kStddevMax);
                const float eps = L.deterministic ? 0.f : normal_draw(noise, row * L.m.Wn + no + j, seed, offset);
                // Normal.sample(): eps * std + mean, product and sum rounded separately (SURVEY App.C)
                const float a = __fadd_rn(__fmul_rn(eps, sd), mean);
                const float d = a - mean;
                lps += -(d * d) / (2.f * (sd * sd)) - logf(sd) - kHalfLog2Pi;      // normal.py:84-94
                out.actions_f32[row * out.actions_stride + ao + j] = a;
                if (L.env[s]) static_cast<float*>(L.env[s])[row * L.env_stride[s] + j] = a;
            }
            if (out.actions_f32 == nullptr) continue;
            lp_total += warp_sum(lps);                                              // Independent(.., 1)
        }
    }
    if (out.actions_f32 == nullptr) return -1;
    if (lane == 0) {
        if (out.log_prob) out.log_prob[row * out.log_prob_stride] = lp_total;
        if (out.pv_out) out.pv_out[row * out.pv_stride] = pv;
    }
    return act;
}

// The narrow heads (up to 31 distribution_linear rows) keep a straight-line tail per space on the S = 1, LPL = 1 map of
// row_tail, bit for bit the same results: the stand-alone kernels inline it several times per warp and the fused step
// tail and GEMM epilogue sit at tight register budgets, where the member loop of row_tail spills.

// ContinuousActionDistribution on the lanes: lane j in 1..act_dim owns action dimension j-1.  Stored `logits` are the
// distribution parameters [means | log_std] (2*act_dim floats) exactly as the reference's action_parameterization returns
// them (tanh-scaled means and the repeated learned vector when adaptive_stddev=False, action_parameterization.py:64-78).
__device__ __forceinline__ void gaussian_row_tail(float mine, int lane, int64_t row, const HeadsOut& out,
                                                  const float* __restrict__ noise, uint64_t seed, uint64_t offset,
                                                  float pv) {
    const ActionLayout& L = out.lay;
    const int Ad = L.m.size[0];
    const bool is_dim = lane >= 1 && lane <= Ad;
    float mean = mine, log_std;
    if (L.m.kind[0] == kMixedGaussian) {
        const int src = lane + Ad;
        log_std = __shfl_sync(0xffffffffu, mine, src < 32 ? src : 31);
    } else {
        log_std = is_dim ? L.learned_log_std[lane - 1] : 0.f;
        if (L.tanh_scale > 0.f) mean = tanhf(__fdiv_rn(mine, L.tanh_scale)) * L.tanh_scale;
    }
    if (out.logits && is_dim) {
        out.logits[row * out.logits_stride + (lane - 1)] = mean;
        out.logits[row * out.logits_stride + Ad + (lane - 1)] = log_std;
    }
    if (out.actions_f32 == nullptr) return;   // values / distribution parameters only (warp-uniform)
    const float sd = clampf(expf(log_std), kStddevMin, kStddevMax);
    const float eps = (is_dim && !L.deterministic) ? normal_draw(noise, row * Ad + (lane - 1), seed, offset) : 0.f;
    // Normal.sample(): eps * std + mean, product and sum rounded separately (SURVEY App.C)
    const float a = __fadd_rn(__fmul_rn(eps, sd), mean);
    const float d = a - mean;
    const float lpj = is_dim ? (-(d * d) / (2.f * (sd * sd)) - logf(sd) - kHalfLog2Pi) : 0.f;   // normal.py:84-94
    const float lp = warp_sum(lpj);                                                              // Independent(.., 1)
    if (is_dim) {
        out.actions_f32[row * out.actions_stride + (lane - 1)] = a;
        if (L.env[0]) static_cast<float*>(L.env[0])[row * Ad + (lane - 1)] = a;
    }
    if (lane == 0) {
        if (out.log_prob) out.log_prob[row * out.log_prob_stride] = lp;
        if (out.pv_out) out.pv_out[row * out.pv_stride] = pv;
    }
}

// TupleActionDistribution on the lanes: every head runs the categorical recipe on its own lane range; actions_f32 gets K
// floats per row (one index per head), env_actions K int32, log_prob the sum over the heads (:231-241).
__device__ __forceinline__ void tuple_row_tail(float mine, int lane, int A, int64_t row, const HeadsOut& out,
                                               const float* __restrict__ noise, uint64_t seed, uint64_t offset, float pv) {
    const ActionLayout& L = out.lay;
    const bool is_logit = lane >= 1 && lane <= A;
    const float q = (is_logit && !L.deterministic) ? exp1_draw(noise, row * A + (lane - 1), seed, offset) : 1.f;
    float lp_total = 0.f;
    int start = 0;
    const int K = L.m.K;
    for (int k = 0; k < K; ++k) {
        const int n = L.m.size[k];
        const bool in_seg = (lane - 1) >= start && (lane - 1) < start + n;
        const float x = in_seg ? mine : -INFINITY;
        const float m = warp_max(x);
        const float e = in_seg ? expf(x - m) : 0.f;
        const float s = warp_sum(e);
        const float p = __fdiv_rn(e, s);
        const float logp = (x - m) - logf(s);
        float best = in_seg ? __fdiv_rn(p, q) : -INFINITY;
        int idx = in_seg ? (lane - 1 - start) : 0x7fffffff;
        argmax_first(best, idx);
        lp_total += __shfl_sync(0xffffffffu, logp, start + idx + 1);
        if (lane == 0) {
            out.actions_f32[row * out.actions_stride + k] = (float)idx;
            if (L.env[0]) static_cast<int32_t*>(L.env[0])[row * K + k] = idx;
        }
        start += n;
    }
    if (lane == 0) {
        if (out.log_prob) out.log_prob[row * out.log_prob_stride] = lp_total;
        if (out.pv_out) out.pv_out[row * out.pv_stride] = pv;
    }
}

// Lane a of the warp holds output a of one row (0 = value, 1..A = logits, bias included): store them and, in sampling
// mode, run CategoricalActionDistribution (action_distributions.py:110-148) on the lanes.
// Returns the sampled action index of a plain Discrete space (the same value in every lane), -1 otherwise.
__device__ __forceinline__ int heads_row_tail(float mine, int lane, int A, int64_t row, const HeadsOut& out,
                                              const float* __restrict__ noise, uint64_t seed, uint64_t offset, float pv) {
    const ActionLayout& L = out.lay;
    if (lane == 0) out.values[row * out.values_stride] = mine;
    if (L.m.kind[0] != kMixedCategorical) {
        gaussian_row_tail(mine, lane, row, out, noise, seed, offset, pv);
        return -1;
    }
    const bool is_logit = lane >= 1 && lane <= A;
    if (out.logits && is_logit) out.logits[row * out.logits_stride + (lane - 1)] = mine;
    if (out.actions_f32 == nullptr) return -1;   // values / logits only (warp-uniform)
    if (L.m.K > 1) {
        tuple_row_tail(mine, lane, A, row, out, noise, seed, offset, pv);
        return -1;
    }

    const bool masked = L.action_mask != nullptr;
    const float mk = (masked && is_logit && L.action_mask[row * L.mask_stride + (lane - 1)] != 0) ? 1.f : 0.f;
    // masked_softmax / masked_log_softmax :84-95: a forbidden logit gets -1e9 added (an allowed one -0.0: unchanged)
    const float x = is_logit ? ((masked && mk == 0.f) ? __fadd_rn(mine, -1.0e9f) : mine) : -INFINITY;
    const float m = warp_max(x);
    const float e = is_logit ? expf(x - m) : 0.f;
    const float s = warp_sum(e);
    float p = __fdiv_rn(e, s);                          // softmax :116
    const float logp = (x - m) - logf(s);               // log_softmax :125
    if (masked) {
        p = __fmul_rn(p, mk);                                              // :88
        p = __fdiv_rn(p, __fadd_rn(warp_sum(p), 1.0e-13f));                // :89
        if (__ballot_sync(0xffffffffu, p > 0.f) == 0u) p = 1.0e-6f;        // :137-140 nothing allowed: uniform fallback
    }
    const float q = (is_logit && !L.deterministic) ? exp1_draw(noise, row * A + (lane - 1), seed, offset) : 1.f;
    // torch.multinomial(p, 1, True) == argmax(p / q) (first index on ties)
    float best = is_logit ? __fdiv_rn(p, q) : -INFINITY;
    int idx = is_logit ? (lane - 1) : 0x7fffffff;
    argmax_first(best, idx);
    const float lp = __shfl_sync(0xffffffffu, logp, idx + 1);   // log_prob :145-148
    if (lane == 0) {
        out.actions_f32[row * out.actions_stride] = (float)idx;
        if (L.env[0]) static_cast<int32_t*>(L.env[0])[row] = idx;
        if (out.log_prob) out.log_prob[row * out.log_prob_stride] = lp;
        if (out.pv_out) out.pv_out[row * out.pv_stride] = pv;
    }
    return idx;
}

// partial head dot products left by the fused GEMM epilogue: part[p][row][kHeadPartPad]
constexpr int kHeadPartPad = 12;

// everything the finishing step of the heads needs besides the partials
struct HeadsFinish {
    HeadsOut out;
    const float* bv;
    const float* ba;
    const float* noise;
    uint64_t seed, offset_host;
    const int64_t* offset_dev;
    const float* pv_scalar;
};

// one warp finishes one row: fixed-order sum of the P partials (deterministic) + bias, then the distribution tail
__device__ __forceinline__ int heads_finish_row(const float* __restrict__ part, int P, int64_t rows, int64_t row, int lane,
                                                const HeadsFinish& f, float pv, uint64_t offset) {
    const int A = f.out.lay.m.A;
    float mine = 0.f;
    if (lane <= A) {
        for (int p = 0; p < P; ++p) mine += part[((int64_t)p * rows + row) * kHeadPartPad + lane];
    }
    mine += (lane == 0) ? f.bv[0] : (lane <= A ? f.ba[lane - 1] : 0.f);
    return heads_row_tail(mine, lane, A, row, f.out, f.noise, f.seed, offset, pv);
}

}  // namespace sfb
