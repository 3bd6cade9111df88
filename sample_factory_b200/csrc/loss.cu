// PPO loss, forward and backward fused (algo/learning/learner.py:586-657, :431-477), plus the per-minibatch advantage
// statistics (:646-647) and the action-ratio pre-pass V-trace needs (:588-594).  One thread per sample; every input
// is read exactly once (HBM-bound, ~(2A+9)*4 B read + (A+1)*4 B written per sample).
#include <type_traits>

#include "common.cuh"
#include "mixed_layout.cuh"

namespace sfb {

constexpr int kLossMaxBlocks = 1024;
constexpr float kStdMin = 1e-4f, kStdMax = 1e4f;          // action_distributions.py:291-292
constexpr float kHalfLog2PiL = 0.91893853320467274178f;   // log(sqrt(2 pi))
constexpr int kNumPart = 12;
// partial-sum slots
enum { P_PL = 0, P_VL, P_ENT, P_KL, P_KLMAX, P_RDEV, P_RMIN, P_RMAX, P_CLIPPED, P_VSUM, P_COUNT, P_SKL };

template <int AMAX>
__device__ __forceinline__ void load_row(const float* __restrict__ p, int A, float (&out)[AMAX]) {
    if ((A & 3) == 0 && ((reinterpret_cast<uintptr_t>(p) & 15u) == 0)) {
#pragma unroll
        for (int a = 0; a < AMAX; a += 4) {
            if (a < A) {
                const float4 v = *reinterpret_cast<const float4*>(p + a);
                out[a] = v.x; out[a + 1] = v.y; out[a + 2] = v.z; out[a + 3] = v.w;
            }
        }
    } else {
#pragma unroll
        for (int a = 0; a < AMAX; ++a)
            if (a < A) out[a] = p[a];
    }
}

template <int AMAX>
__device__ __forceinline__ void store_row(float* __restrict__ p, int A, const float (&v)[AMAX]) {
    if ((A & 3) == 0 && ((reinterpret_cast<uintptr_t>(p) & 15u) == 0)) {
#pragma unroll
        for (int a = 0; a < AMAX; a += 4)
            if (a < A) *reinterpret_cast<float4*>(p + a) = make_float4(v[a], v[a + 1], v[a + 2], v[a + 3]);
    } else {
#pragma unroll
        for (int a = 0; a < AMAX; ++a)
            if (a < A) p[a] = v[a];
    }
}

// log_softmax / softmax of one row held in registers (action_distributions.py:116,125)
template <int AMAX>
__device__ __forceinline__ void row_softmax(const float (&l)[AMAX], int A, float (&p)[AMAX], float (&logp)[AMAX]) {
    float m = -INFINITY;
#pragma unroll
    for (int a = 0; a < AMAX; ++a)
        if (a < A) m = fmaxf(m, l[a]);
    float s = 0.f;
#pragma unroll
    for (int a = 0; a < AMAX; ++a)
        if (a < A) { p[a] = expf(l[a] - m); s += p[a]; }
    const float logs = logf(s);
#pragma unroll
    for (int a = 0; a < AMAX; ++a)
        if (a < A) { logp[a] = (l[a] - m) - logs; p[a] = __fdiv_rn(p[a], s); }
}

template <int AMAX>
__global__ void __launch_bounds__(256) action_ratio_kernel(const float* __restrict__ logits, int A,
                                                           const float* __restrict__ actions,
                                                           const float* __restrict__ lp_old, int64_t batch,
                                                           float* __restrict__ ratio) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= batch) return;
    float l[AMAX], p[AMAX], logp[AMAX];
    load_row<AMAX>(logits + i * A, A, l);
    row_softmax<AMAX>(l, A, p, logp);
    const int act = (int)actions[i];
    float lp = 0.f;
#pragma unroll
    for (int a = 0; a < AMAX; ++a)
        if (a < A && a == act) lp = logp[a];
    ratio[i] = clampf(expf(lp - lp_old[i]), 0.05f, 20.0f);   // learner.py:589-592
}

// ---- advantage statistics -------------------------------------------------------------------------------------------
__device__ __forceinline__ double block_sum(double v, double* sm) {
    v = warp_sum(v);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) sm[w] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x < 32) {
        t = (threadIdx.x < (blockDim.x >> 5)) ? sm[threadIdx.x] : 0.0;
        t = warp_sum(t);
    }
    return t;   // valid in warp 0
}
__device__ __forceinline__ double block_max(double v, double* sm) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    __syncthreads();
    if (lane == 0) sm[w] = v;
    __syncthreads();
    double t = -INFINITY;
    if (threadIdx.x < 32) {
        t = (threadIdx.x < (blockDim.x >> 5)) ? sm[threadIdx.x] : -INFINITY;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t = fmax(t, __shfl_xor_sync(0xffffffffu, t, o));
    }
    return t;
}

__global__ void __launch_bounds__(256) adv_stats_partial_kernel(const float* __restrict__ adv,
                                                                const uint8_t* __restrict__ valids, int64_t batch,
                                                                double* __restrict__ part) {
    __shared__ double sm[8];
    double c = 0.0, s = 0.0, ss = 0.0;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < batch; i += (int64_t)gridDim.x * blockDim.x) {
        if (valids[i]) {
            const double a = (double)adv[i];
            c += 1.0; s += a; ss += a * a;
        }
    }
    c = block_sum(c, sm); s = block_sum(s, sm); ss = block_sum(ss, sm);
    if (threadIdx.x == 0) { part[blockIdx.x * 3 + 0] = c; part[blockIdx.x * 3 + 1] = s; part[blockIdx.x * 3 + 2] = ss; }
}

__device__ __forceinline__ void adv_finalize(double c, double s, double ss, double* stats) {
    const double mean = c > 0.0 ? s / c : 0.0;
    // torch.std_mean default: unbiased (n-1).  With one valid sample (or none) torch gives NaN, which would reach every
    // weight; here the stddev is 0, clamped to 1e-7 by the loss, so the normalised advantage and the policy gradient are
    // 0 while the value, exploration and KL terms still train (a deliberate deviation, DESIGN section 7)
    const double var = c > 1.0 ? (ss - s * mean) / (c - 1.0) : 0.0;
    stats[SFB200_LS_NUM_VALID] = c;
    stats[SFB200_LS_ADV_MEAN] = (double)(float)mean;
    stats[SFB200_LS_ADV_STD] = (double)(float)sqrt(var > 0.0 ? var : 0.0);
}

__global__ void adv_stats_finalize_kernel(const double* __restrict__ part, int nblocks, double* __restrict__ stats,
                                          double* __restrict__ dp_partials) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    double c = 0.0, s = 0.0, ss = 0.0;
    for (int b = 0; b < nblocks; ++b) { c += part[b * 3]; s += part[b * 3 + 1]; ss += part[b * 3 + 2]; }
    if (dp_partials) { dp_partials[0] = c; dp_partials[1] = s; dp_partials[2] = ss; }
    adv_finalize(c, s, ss, stats);
}
__global__ void adv_stats_from_partials_kernel(const double* __restrict__ dp, double* __restrict__ stats) {
    if (threadIdx.x == 0 && blockIdx.x == 0) adv_finalize(dp[0], dp[1], dp[2], stats);
}

// ---- the loss ---------------------------------------------------------------------------------------------------------
// distribution-independent pieces shared by the categorical and the Gaussian kernels
struct PpoAcc {
    double s_pl = 0, s_vl = 0, s_ent = 0, s_kl = 0, s_rdev = 0, s_clip = 0, s_v = 0, s_cnt = 0, s_skl = 0;
    double m_kl = -INFINITY, m_rmin = -INFINITY /* holds -min */, m_rmax = -INFINITY;
};

// _policy_loss :431-439 given log_prob of the stored action under the new distribution.  Returns d(loss)/d(log_prob).
__device__ __forceinline__ float ppo_policy_terms(float lp, float lp_old, float adv, float adv_mean, float adv_std,
                                                  float clip_lo, float clip_hi, float w, PpoAcc& acc) {
    const float ratio_raw = expf(lp - lp_old);                          // :589
    const float ratio = clampf(ratio_raw, 0.05f, 20.0f);                // :592
    const float advn = __fdiv_rn(__fsub_rn(adv, adv_mean), adv_std);    // :647
    const float rc = clampf(ratio, clip_lo, clip_hi);
    const float s1 = ratio * advn, s2 = rc * advn;
    acc.s_pl = fminf(s1, s2);
    const bool in_window = ratio >= clip_lo && ratio <= clip_hi;
    const float g_ratio = (in_window || s1 < s2) ? -advn : 0.f;         // d(-min)/d ratio (ties split evenly)
    const float dratio_dlp = (ratio_raw >= 0.05f && ratio_raw <= 20.0f) ? ratio_raw : 0.f;
    // summaries :843-923
    acc.s_rdev = fabsf(1.f - ratio);
    acc.m_rmin = -(double)ratio;
    acc.m_rmax = ratio;
    acc.s_clip = (ratio < clip_lo ? 1.0 : 0.0) + (ratio > clip_hi ? 1.0 : 0.0);
    return w * g_ratio * dratio_dlp;
}

// _value_loss :441-459.  Returns d(loss)/d(value).
__device__ __forceinline__ float ppo_value_terms(float v, float vo, float R, float clip_value, float w, float c_val,
                                                 PpoAcc& acc) {
    const float diff = v - vo;
    const float vc = vo + clampf(diff, -clip_value, clip_value);
    const float l1 = (v - R) * (v - R), l2 = (vc - R) * (vc - R);
    acc.s_vl = fmaxf(l1, l2);
    const bool inside = diff >= -clip_value && diff <= clip_value;
    const float g1 = 2.f * (v - R), g2 = inside ? 2.f * (vc - R) : 0.f;
    const float gv = (l1 > l2) ? g1 : ((l2 > l1) ? g2 : 0.5f * (g1 + g2));
    return w * c_val * gv;
}

// the minibatch constants every loss kernel starts from: advantage mean / std and the gradient weight grad_scale / n_valid
struct PpoW {
    float adv_mean, adv_std, w;
};
__device__ __forceinline__ PpoW ppo_weights(const double* __restrict__ stats, float grad_scale) {
    const double n_valid = stats[SFB200_LS_NUM_VALID];
    PpoW pw;
    pw.adv_mean = (float)stats[SFB200_LS_ADV_MEAN];
    pw.adv_std = fmaxf((float)stats[SFB200_LS_ADV_STD], 1e-7f);   // clamp_min :647
    pw.w = n_valid > 0.0 ? (float)((double)grad_scale / n_valid) : 0.f;
    return pw;
}

__device__ __forceinline__ void ppo_store_partials(const PpoAcc& a, double* __restrict__ part, double* sm) {
    double* my = part + (int64_t)blockIdx.x * kNumPart;
    double t;
    t = block_sum(a.s_pl, sm);   if (threadIdx.x == 0) my[P_PL] = t;
    t = block_sum(a.s_vl, sm);   if (threadIdx.x == 0) my[P_VL] = t;
    t = block_sum(a.s_ent, sm);  if (threadIdx.x == 0) my[P_ENT] = t;
    t = block_sum(a.s_kl, sm);   if (threadIdx.x == 0) my[P_KL] = t;
    t = block_max(a.m_kl, sm);   if (threadIdx.x == 0) my[P_KLMAX] = t;
    t = block_sum(a.s_rdev, sm); if (threadIdx.x == 0) my[P_RDEV] = t;
    t = block_max(a.m_rmin, sm); if (threadIdx.x == 0) my[P_RMIN] = t;
    t = block_max(a.m_rmax, sm); if (threadIdx.x == 0) my[P_RMAX] = t;
    t = block_sum(a.s_clip, sm); if (threadIdx.x == 0) my[P_CLIPPED] = t;
    t = block_sum(a.s_v, sm);    if (threadIdx.x == 0) my[P_VSUM] = t;
    t = block_sum(a.s_cnt, sm);  if (threadIdx.x == 0) my[P_COUNT] = t;
    t = block_sum(a.s_skl, sm);  if (threadIdx.x == 0) my[P_SKL] = t;
}

template <int AMAX>
__global__ void __launch_bounds__(256) ppo_loss_kernel(
    const float* __restrict__ logits, const float* __restrict__ values, int A, const float* __restrict__ actions,
    const float* __restrict__ lp_old, const float* __restrict__ v_old, const float* __restrict__ adv,
    const float* __restrict__ targets, const uint8_t* __restrict__ valids, const float* __restrict__ logits_old,
    int64_t batch, float clip_lo, float clip_hi, float clip_value, float c_ent, int expl_mode, float c_val, float c_kl,
    float grad_scale, float* __restrict__ dlogits, float* __restrict__ dvalues, const double* __restrict__ stats,
    double* __restrict__ part) {
    __shared__ double sm[8];
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const PpoW pw = ppo_weights(stats, grad_scale);
    const float adv_mean = pw.adv_mean, adv_std = pw.adv_std, w = pw.w;
    PpoAcc acc;

    if (i < batch) {
        const float v = values[i];
        acc.s_v = v;
        float dl[AMAX];
#pragma unroll
        for (int a = 0; a < AMAX; ++a) dl[a] = 0.f;
        float dv = 0.f;
        if (valids[i]) {
            acc.s_cnt = 1.0;
            float l[AMAX], p[AMAX], logp[AMAX];
            load_row<AMAX>(logits + i * A, A, l);
            row_softmax<AMAX>(l, A, p, logp);
            const int act = (int)actions[i];                                   // .long() :146
            float lp = 0.f;
#pragma unroll
            for (int a = 0; a < AMAX; ++a)
                if (a < A && a == act) lp = logp[a];
            const float g_lp = ppo_policy_terms(lp, lp_old[i], adv[i], adv_mean, adv_std, clip_lo, clip_hi, w, acc);
            // entropy :150-152, :473-477
            float H = 0.f;
#pragma unroll
            for (int a = 0; a < AMAX; ++a)
                if (a < A) H -= logp[a] * p[a];
            acc.s_ent = H;
            // symmetric KL to the uniform prior (action_distributions.py:168-177), the alternative exploration loss
            // (learner.py:479-486):  0.5 * (sum_a p_a (logp_a - log u) + sum_a u (log u - logp_a)),  u = 1/A
            const float u = 1.f / (float)A, log_u = -logf((float)A);
            float S1 = 0.f, S2 = 0.f;
            if (expl_mode == 1) {
#pragma unroll
                for (int a = 0; a < AMAX; ++a)
                    if (a < A) { S1 += p[a] * (logp[a] - log_u); S2 += u * (log_u - logp[a]); }
                acc.s_skl = 0.5f * (S1 + S2);
            }
            // KL(new || old) :154-158
            float kl = 0.f;
            float lq[AMAX];
            if (logits_old) {
                float lo[AMAX], po[AMAX];
                load_row<AMAX>(logits_old + i * A, A, lo);
                row_softmax<AMAX>(lo, A, po, lq);
#pragma unroll
                for (int a = 0; a < AMAX; ++a)
                    if (a < A) kl += p[a] * (logp[a] - lq[a]);
                acc.s_kl = kl;
                acc.m_kl = kl;
            }
            const float we = w * c_ent, wk = (logits_old ? w * c_kl : 0.f);
#pragma unroll
            for (int a = 0; a < AMAX; ++a) {
                if (a < A) {
                    float g = g_lp * ((a == act ? 1.f : 0.f) - p[a]);
                    if (expl_mode == 1) g += we * 0.5f * (p[a] * ((logp[a] - log_u) - S1) + p[a] - u);   // +c * d skl / d l_a
                    else g += we * p[a] * (logp[a] + H);                                                    // -c * d H / d l_a
                    if (logits_old) g += wk * p[a] * ((logp[a] - lq[a]) - kl);
                    dl[a] = g;
                }
            }
            dv = ppo_value_terms(v, v_old[i], targets[i], clip_value, w, c_val, acc);
        }
        store_row<AMAX>(dlogits + i * A, A, dl);
        dvalues[i] = dv;
    }
    ppo_store_partials(acc, part, sm);
}


// Tuple of independent categorical heads (TupleActionDistribution, action_distributions.py:197-286): log-prob, entropy,
// KL and the symmetric KL are sums over the heads; every head normalises over its own logit segment.
struct Segs {
    int n;
    int len[8];
};

template <int AMAX>
__device__ __forceinline__ void row_softmax_segs(const float (&l)[AMAX], const Segs& sg, float (&p)[AMAX],
                                                 float (&logp)[AMAX]) {
    int start = 0;
    for (int k = 0; k < sg.n; ++k) {
        const int end = start + sg.len[k];
        float m = -INFINITY;
#pragma unroll
        for (int a = 0; a < AMAX; ++a)
            if (a >= start && a < end) m = fmaxf(m, l[a]);
        float s = 0.f;
#pragma unroll
        for (int a = 0; a < AMAX; ++a)
            if (a >= start && a < end) { p[a] = expf(l[a] - m); s += p[a]; }
        const float logs = logf(s);
#pragma unroll
        for (int a = 0; a < AMAX; ++a)
            if (a >= start && a < end) { logp[a] = (l[a] - m) - logs; p[a] = __fdiv_rn(p[a], s); }
        start = end;
    }
}

template <int AMAX>
__global__ void __launch_bounds__(256) ppo_loss_tuple_kernel(
    const float* __restrict__ logits, const float* __restrict__ values, int A, Segs sg, const float* __restrict__ actions,
    const float* __restrict__ lp_old, const float* __restrict__ v_old, const float* __restrict__ adv,
    const float* __restrict__ targets, const uint8_t* __restrict__ valids, const float* __restrict__ logits_old,
    int64_t batch, float clip_lo, float clip_hi, float clip_value, float c_ent, int expl_mode, float c_val, float c_kl,
    float grad_scale, float* __restrict__ dlogits, float* __restrict__ dvalues, const double* __restrict__ stats,
    double* __restrict__ part) {
    __shared__ double sm[8];
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const PpoW pw = ppo_weights(stats, grad_scale);
    const float adv_mean = pw.adv_mean, adv_std = pw.adv_std, w = pw.w;
    PpoAcc acc;

    if (i < batch) {
        const float v = values[i];
        acc.s_v = v;
        float dl[AMAX];
#pragma unroll
        for (int a = 0; a < AMAX; ++a) dl[a] = 0.f;
        float dv = 0.f;
        if (valids[i]) {
            acc.s_cnt = 1.0;
            float l[AMAX], p[AMAX], logp[AMAX], lq[AMAX];
            load_row<AMAX>(logits + i * A, A, l);
            row_softmax_segs<AMAX>(l, sg, p, logp);
            if (logits_old) {
                float lo[AMAX], po[AMAX];
                load_row<AMAX>(logits_old + i * A, A, lo);
                row_softmax_segs<AMAX>(lo, sg, po, lq);
            }
            // per-head terms
            float lp = 0.f, Htot = 0.f, kltot = 0.f, skltot = 0.f;
            float segH[8], segKL[8], segS1[8];
            int act_idx[8];
            int start = 0;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                segH[k] = 0.f; segKL[k] = 0.f; segS1[k] = 0.f; act_idx[k] = -1;
                if (k < sg.n) {
                    const int n = sg.len[k], end = start + n;
                    act_idx[k] = start + (int)actions[i * sg.n + k];
                    const float u = 1.f / (float)n, log_u = -logf((float)n);
                    float S2 = 0.f;
#pragma unroll
                    for (int a = 0; a < AMAX; ++a) {
                        if (a >= start && a < end) {
                            if (a == act_idx[k]) lp += logp[a];
                            segH[k] -= logp[a] * p[a];
                            if (logits_old) segKL[k] += p[a] * (logp[a] - lq[a]);
                            segS1[k] += p[a] * (logp[a] - log_u);
                            S2 += u * (log_u - logp[a]);
                        }
                    }
                    Htot += segH[k];
                    kltot += segKL[k];
                    skltot += 0.5f * (segS1[k] + S2);
                    start = end;
                }
            }
            const float g_lp = ppo_policy_terms(lp, lp_old[i], adv[i], adv_mean, adv_std, clip_lo, clip_hi, w, acc);
            acc.s_ent = Htot;
            if (expl_mode == 1) acc.s_skl = skltot;
            if (logits_old) { acc.s_kl = kltot; acc.m_kl = kltot; }
            const float we = w * c_ent, wk = (logits_old ? w * c_kl : 0.f);
            start = 0;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                if (k < sg.n) {
                    const int n = sg.len[k], end = start + n;
                    const float u = 1.f / (float)n, log_u = -logf((float)n);
#pragma unroll
                    for (int a = 0; a < AMAX; ++a) {
                        if (a >= start && a < end) {
                            float g = g_lp * ((a == act_idx[k] ? 1.f : 0.f) - p[a]);
                            if (expl_mode == 1) g += we * 0.5f * (p[a] * ((logp[a] - log_u) - segS1[k]) + p[a] - u);
                            else g += we * p[a] * (logp[a] + segH[k]);
                            if (logits_old) g += wk * p[a] * ((logp[a] - lq[a]) - segKL[k]);
                            dl[a] = g;
                        }
                    }
                    start = end;
                }
            }
            dv = ppo_value_terms(v, v_old[i], targets[i], clip_value, w, c_val, acc);
        }
        store_row<AMAX>(dlogits + i * A, A, dl);
        dvalues[i] = dv;
    }
    ppo_store_partials(acc, part, sm);
}

template <int AMAX>
__global__ void __launch_bounds__(256) action_ratio_tuple_kernel(const float* __restrict__ logits, int A, Segs sg,
                                                                 const float* __restrict__ actions,
                                                                 const float* __restrict__ lp_old, int64_t batch,
                                                                 float* __restrict__ ratio) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= batch) return;
    float l[AMAX], p[AMAX], logp[AMAX];
    load_row<AMAX>(logits + i * A, A, l);
    row_softmax_segs<AMAX>(l, sg, p, logp);
    float lp = 0.f;
    int start = 0;
    for (int k = 0; k < sg.n; ++k) {
        const int idx = start + (int)actions[i * sg.n + k];
#pragma unroll
        for (int a = 0; a < AMAX; ++a)
            if (a == idx) lp += logp[a];
        start += sg.len[k];
    }
    ratio[i] = clampf(expf(lp - lp_old[i]), 0.05f, 20.0f);
}

// Diagonal Gaussian policy (ContinuousActionDistribution, action_distributions.py:290-323; torch Normal / kl formulas):
// params rows are [means | log_std] (2*Ad floats, the layout of `action_logits`), actions rows Ad floats.
//   log_prob = sum_j -(a-m)^2 / (2 sd^2) - log sd - log sqrt(2 pi),  sd = clamp(exp(log_std), 1e-4, 1e4)
//   entropy  = sum_j 0.5 + 0.5 log(2 pi) + log sd
//   KL(new || old) = sum_j 0.5 (r + t - 1 - log r),  r = (sd/sd_old)^2,  t = ((m - m_old)/sd_old)^2
// Gradients go to the distribution_linear outputs: adaptive stddev -> dlogits [B, 2*Ad] = [d means | d log_std];
// learned stddev -> dlogits [B, Ad] = d means * (1 - (m/tanh_scale)^2) (tanh-squashed means) and dlogstd [B, Ad], which
// the caller column-sums into the learned vector's gradient.  The clamp passes gradient inside [1e-4, 1e4] only.
template <int AH>
__device__ __forceinline__ void gauss_load(const float* __restrict__ row, int Ad, float (&m)[AH], float (&s)[AH]) {
#pragma unroll
    for (int j = 0; j < AH; ++j)
        if (j < Ad) { m[j] = row[j]; s[j] = row[Ad + j]; }
}

template <int AH>
__global__ void __launch_bounds__(256) ppo_loss_gauss_kernel(
    const float* __restrict__ params, const float* __restrict__ values, int Ad, int adaptive, float tanh_scale,
    const float* __restrict__ actions, const float* __restrict__ lp_old, const float* __restrict__ v_old,
    const float* __restrict__ adv, const float* __restrict__ targets, const uint8_t* __restrict__ valids,
    const float* __restrict__ params_old, int64_t batch, float clip_lo, float clip_hi, float clip_value, float c_ent,
    float c_val, float c_kl, float grad_scale, float* __restrict__ dlogits, float* __restrict__ dlogstd,
    float* __restrict__ dvalues, const double* __restrict__ stats, double* __restrict__ part) {
    __shared__ double sm[8];
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const PpoW pw = ppo_weights(stats, grad_scale);
    const float adv_mean = pw.adv_mean, adv_std = pw.adv_std, w = pw.w;
    PpoAcc acc;

    if (i < batch) {
        const float v = values[i];
        acc.s_v = v;
        float dm[AH], ds[AH];
#pragma unroll
        for (int j = 0; j < AH; ++j) { dm[j] = 0.f; ds[j] = 0.f; }
        float dv = 0.f;
        if (valids[i]) {
            acc.s_cnt = 1.0;
            float m[AH], s[AH], sd[AH], dlt[AH];
            gauss_load<AH>(params + i * 2 * Ad, Ad, m, s);
            float lp = 0.f, H = 0.f;
#pragma unroll
            for (int j = 0; j < AH; ++j) {
                if (j < Ad) {
                    sd[j] = clampf(expf(s[j]), kStdMin, kStdMax);
                    dlt[j] = actions[i * Ad + j] - m[j];
                    const float lsd = logf(sd[j]);
                    lp += -(dlt[j] * dlt[j]) / (2.f * (sd[j] * sd[j])) - lsd - kHalfLog2PiL;
                    H += 0.5f + kHalfLog2PiL + lsd;     // 0.5 + 0.5 log(2 pi) + log sd
                }
            }
            const float g_lp = ppo_policy_terms(lp, lp_old[i], adv[i], adv_mean, adv_std, clip_lo, clip_hi, w, acc);
            acc.s_ent = H;
            const float we = w * c_ent, wk = (params_old ? w * c_kl : 0.f);
            float mo[AH], so[AH];
            float kl = 0.f;
            if (params_old) gauss_load<AH>(params_old + i * 2 * Ad, Ad, mo, so);
#pragma unroll
            for (int j = 0; j < AH; ++j) {
                if (j < Ad) {
                    const float ex = expf(s[j]);
                    const float in_range = (ex >= kStdMin && ex <= kStdMax) ? 1.f : 0.f;
                    const float inv_var = 1.f / (sd[j] * sd[j]);
                    float gm = g_lp * dlt[j] * inv_var;
                    float gs = g_lp * (dlt[j] * dlt[j] * inv_var - 1.f) - we;
                    if (params_old) {
                        const float sdo = clampf(expf(so[j]), kStdMin, kStdMax);
                        const float q = sd[j] / sdo, r = q * q;
                        const float dq = (m[j] - mo[j]) / sdo;
                        kl += 0.5f * (r + dq * dq - 1.f - logf(r));
                        gm += wk * dq / sdo;
                        gs += wk * (r - 1.f);
                    }
                    gs *= in_range;
                    if (!adaptive && tanh_scale > 0.f) {
                        const float tq = m[j] / tanh_scale;      // m = tanh(z/ts)*ts -> dm/dz = 1 - tanh^2
                        gm *= (1.f - tq * tq);
                    }
                    dm[j] = gm;
                    ds[j] = gs;
                }
            }
            if (params_old) { acc.s_kl = kl; acc.m_kl = kl; }
            dv = ppo_value_terms(v, v_old[i], targets[i], clip_value, w, c_val, acc);
        }
        float* drow = dlogits + i * (adaptive ? 2 * Ad : Ad);
#pragma unroll
        for (int j = 0; j < AH; ++j) {
            if (j < Ad) {
                drow[j] = dm[j];
                if (adaptive) drow[Ad + j] = ds[j];
                else dlogstd[i * Ad + j] = ds[j];
            }
        }
        dvalues[i] = dv;
    }
    ppo_store_partials(acc, part, sm);
}

template <int AH>
__global__ void __launch_bounds__(256) action_ratio_gauss_kernel(const float* __restrict__ params, int Ad,
                                                                 const float* __restrict__ actions,
                                                                 const float* __restrict__ lp_old, int64_t batch,
                                                                 float* __restrict__ ratio) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= batch) return;
    float m[AH], s[AH];
    gauss_load<AH>(params + i * 2 * Ad, Ad, m, s);
    float lp = 0.f;
#pragma unroll
    for (int j = 0; j < AH; ++j) {
        if (j < Ad) {
            const float sd = clampf(expf(s[j]), kStdMin, kStdMax);
            const float d = actions[i * Ad + j] - m[j];
            lp += -(d * d) / (2.f * (sd * sd)) - logf(sd) - kHalfLog2PiL;
        }
    }
    ratio[i] = clampf(expf(lp - lp_old[i]), 0.05f, 20.0f);
}

__global__ void __launch_bounds__(256) ppo_loss_finalize_kernel(const double* __restrict__ part, int nblocks,
                                                                int64_t batch, float c_ent, int expl_mode, float c_val,
                                                                float c_kl, double* __restrict__ stats) {
    __shared__ double sm[8];
    double acc[kNumPart];
#pragma unroll
    for (int k = 0; k < kNumPart; ++k) acc[k] = (k == P_KLMAX || k == P_RMIN || k == P_RMAX) ? -INFINITY : 0.0;
    for (int b = threadIdx.x; b < nblocks; b += blockDim.x) {
#pragma unroll
        for (int k = 0; k < kNumPart; ++k) {
            const double v = part[(int64_t)b * kNumPart + k];
            if (k == P_KLMAX || k == P_RMIN || k == P_RMAX) acc[k] = fmax(acc[k], v);
            else acc[k] += v;
        }
    }
#pragma unroll
    for (int k = 0; k < kNumPart; ++k) {
        if (k == P_KLMAX || k == P_RMIN || k == P_RMAX) acc[k] = block_max(acc[k], sm);
        else acc[k] = block_sum(acc[k], sm);
    }
    if (threadIdx.x == 0) {
        const double n = stats[SFB200_LS_NUM_VALID];
        const double inv = n > 0.0 ? 1.0 / n : 0.0;
        const double pl = -acc[P_PL] * inv;
        const double vl = (double)c_val * acc[P_VL] * inv;
        // entropy bonus :473-477, or +coeff * min(mean symmetric KL, 30) :479-486 (the gradient assumes the clamp inactive:
        // a mean symmetric KL above 30 needs probabilities below e^-60)
        double el = -(double)c_ent * acc[P_ENT] * inv;
        if (expl_mode == 1) {
            double skl = acc[P_SKL] * inv;
            if (!isfinite(skl)) skl = 0.0;
            el = (double)c_ent * (skl < 30.0 ? skl : 30.0);
        }
        const double kl = (double)c_kl * acc[P_KL] * inv;
        stats[SFB200_LS_POLICY_LOSS] = pl;
        stats[SFB200_LS_VALUE_LOSS] = vl;
        stats[SFB200_LS_EXPLORATION_LOSS] = el;
        stats[SFB200_LS_KL_LOSS] = kl;
        stats[SFB200_LS_KL_OLD_MEAN] = acc[P_KL] * inv;
        stats[SFB200_LS_KL_OLD_MAX] = acc[P_KLMAX];
        stats[SFB200_LS_ENTROPY_MEAN] = acc[P_ENT] * inv;
        stats[SFB200_LS_RATIO_MEAN_ABS_DEV] = acc[P_RDEV] * inv;
        stats[SFB200_LS_RATIO_MIN] = -acc[P_RMIN];
        stats[SFB200_LS_RATIO_MAX] = acc[P_RMAX];
        stats[SFB200_LS_FRACTION_CLIPPED] = acc[P_CLIPPED] * inv;
        stats[SFB200_LS_VALUE_MEAN] = batch > 0 ? acc[P_VSUM] / (double)batch : 0.0;
        stats[SFB200_LS_TOTAL_LOSS] = pl + vl + el + kl;
    }
}

// ---- rows wider than 32 (up to kWideMax): one warp per sample -----------------------------------------------------
// Lane l holds elements l, l+32, ... of a row (LPL per lane).  A block still covers 256 consecutive samples (8 warps x 32
// rows) and lane r of a warp keeps the statistics of the warp's r-th sample, so ppo_store_partials sees the same thread ->
// sample map as the thread-per-sample kernels above: same partial slots, same fixed-order reduction, same workspace.
constexpr int kWideMax = 1024;

template <int LPL>
__device__ __forceinline__ void wide_load(const float* __restrict__ p, int n, int lane, float (&v)[LPL]) {
#pragma unroll
    for (int k = 0; k < LPL; ++k) v[k] = (k * 32 + lane < n) ? p[k * 32 + lane] : 0.f;
}
template <int LPL>
__device__ __forceinline__ void wide_store(float* __restrict__ p, int n, int lane, const float (&v)[LPL]) {
#pragma unroll
    for (int k = 0; k < LPL; ++k)
        if (k * 32 + lane < n) p[k * 32 + lane] = v[k];
}
// element a of a row spread over the warp
template <int LPL>
__device__ __forceinline__ float wide_get(const float (&v)[LPL], int a, int lane) {
    float mine = 0.f;
#pragma unroll
    for (int k = 0; k < LPL; ++k)
        if (k == (a >> 5)) mine = v[k];
    return __shfl_sync(0xffffffffu, mine, a & 31);
}
// softmax / log_softmax over the elements [lo, hi) of a row (row_softmax / row_softmax_segs); other slots untouched
template <int LPL>
__device__ __forceinline__ void wide_softmax(const float (&l)[LPL], int lo, int hi, int lane, float (&p)[LPL],
                                             float (&logp)[LPL]) {
    float m = -INFINITY;
#pragma unroll
    for (int k = 0; k < LPL; ++k) {
        const int a = k * 32 + lane;
        if (a >= lo && a < hi) m = fmaxf(m, l[k]);
    }
    m = warp_max(m);
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < LPL; ++k) {
        const int a = k * 32 + lane;
        if (a >= lo && a < hi) { p[k] = expf(l[k] - m); s += p[k]; }
    }
    s = warp_sum(s);
    const float logs = logf(s);
#pragma unroll
    for (int k = 0; k < LPL; ++k) {
        const int a = k * 32 + lane;
        if (a >= lo && a < hi) { logp[k] = (l[k] - m) - logs; p[k] = __fdiv_rn(p[k], s); }
    }
}


template <int LPL>
__global__ void __launch_bounds__(256) ppo_loss_wide_kernel(
    const float* __restrict__ logits, const float* __restrict__ values, int A, const float* __restrict__ actions,
    const float* __restrict__ lp_old, const float* __restrict__ v_old, const float* __restrict__ adv,
    const float* __restrict__ targets, const uint8_t* __restrict__ valids, const float* __restrict__ logits_old,
    int64_t batch, float clip_lo, float clip_hi, float clip_value, float c_ent, int expl_mode, float c_val, float c_kl,
    float grad_scale, float* __restrict__ dlogits, float* __restrict__ dvalues, const double* __restrict__ stats,
    double* __restrict__ part) {
    __shared__ double sm[8];
    const int lane = threadIdx.x & 31;
    const PpoW pw = ppo_weights(stats, grad_scale);
    const float adv_mean = pw.adv_mean, adv_std = pw.adv_std, w = pw.w;
    PpoAcc acc;   // statistics of sample blockIdx.x * 256 + threadIdx.x
    const int64_t base = blockIdx.x * (int64_t)blockDim.x + (threadIdx.x & ~31);
    for (int r = 0; r < 32; ++r) {
        const int64_t i = base + r;
        if (i >= batch) break;   // warp-uniform
        PpoAcc t;
        const float v = values[i];
        t.s_v = v;
        float dl[LPL];
#pragma unroll
        for (int k = 0; k < LPL; ++k) dl[k] = 0.f;
        float dv = 0.f;
        if (valids[i]) {
            t.s_cnt = 1.0;
            float l[LPL], p[LPL], logp[LPL], lq[LPL];
            wide_load<LPL>(logits + i * A, A, lane, l);
            wide_softmax<LPL>(l, 0, A, lane, p, logp);
            const int act = (int)actions[i];
            const float lp = wide_get<LPL>(logp, act, lane);
            const float g_lp = ppo_policy_terms(lp, lp_old[i], adv[i], adv_mean, adv_std, clip_lo, clip_hi, w, t);
            const float u = 1.f / (float)A, log_u = -logf((float)A);
            float h = 0.f, s1 = 0.f, s2 = 0.f;
#pragma unroll
            for (int k = 0; k < LPL; ++k) {
                if (k * 32 + lane < A) {
                    h -= logp[k] * p[k];
                    s1 += p[k] * (logp[k] - log_u);
                    s2 += u * (log_u - logp[k]);
                }
            }
            const float H = warp_sum(h);
            t.s_ent = H;
            float S1 = 0.f;
            if (expl_mode == 1) {
                S1 = warp_sum(s1);
                t.s_skl = 0.5f * (S1 + warp_sum(s2));
            }
            float kl = 0.f;
            if (logits_old) {
                float lo[LPL], po[LPL];
                wide_load<LPL>(logits_old + i * A, A, lane, lo);
                wide_softmax<LPL>(lo, 0, A, lane, po, lq);
                float klp = 0.f;
#pragma unroll
                for (int k = 0; k < LPL; ++k)
                    if (k * 32 + lane < A) klp += p[k] * (logp[k] - lq[k]);
                kl = warp_sum(klp);
                t.s_kl = kl;
                t.m_kl = kl;
            }
            const float we = w * c_ent, wk = (logits_old ? w * c_kl : 0.f);
#pragma unroll
            for (int k = 0; k < LPL; ++k) {
                const int a = k * 32 + lane;
                if (a < A) {
                    float g = g_lp * ((a == act ? 1.f : 0.f) - p[k]);
                    if (expl_mode == 1) g += we * 0.5f * (p[k] * ((logp[k] - log_u) - S1) + p[k] - u);
                    else g += we * p[k] * (logp[k] + H);
                    if (logits_old) g += wk * p[k] * ((logp[k] - lq[k]) - kl);
                    dl[k] = g;
                }
            }
            dv = ppo_value_terms(v, v_old[i], targets[i], clip_value, w, c_val, t);
        }
        wide_store<LPL>(dlogits + i * A, A, lane, dl);
        if (lane == 0) dvalues[i] = dv;
        if (lane == r) acc = t;
    }
    ppo_store_partials(acc, part, sm);
}

template <int LPL>
__global__ void __launch_bounds__(256) ppo_loss_tuple_wide_kernel(
    const float* __restrict__ logits, const float* __restrict__ values, int A, Segs sg, const float* __restrict__ actions,
    const float* __restrict__ lp_old, const float* __restrict__ v_old, const float* __restrict__ adv,
    const float* __restrict__ targets, const uint8_t* __restrict__ valids, const float* __restrict__ logits_old,
    int64_t batch, float clip_lo, float clip_hi, float clip_value, float c_ent, int expl_mode, float c_val, float c_kl,
    float grad_scale, float* __restrict__ dlogits, float* __restrict__ dvalues, const double* __restrict__ stats,
    double* __restrict__ part) {
    __shared__ double sm[8];
    const int lane = threadIdx.x & 31;
    const PpoW pw = ppo_weights(stats, grad_scale);
    const float adv_mean = pw.adv_mean, adv_std = pw.adv_std, w = pw.w;
    PpoAcc acc;   // statistics of sample blockIdx.x * 256 + threadIdx.x
    const int64_t base = blockIdx.x * (int64_t)blockDim.x + (threadIdx.x & ~31);
    for (int r = 0; r < 32; ++r) {
        const int64_t i = base + r;
        if (i >= batch) break;
        PpoAcc t;
        const float v = values[i];
        t.s_v = v;
        float dl[LPL];
#pragma unroll
        for (int k = 0; k < LPL; ++k) dl[k] = 0.f;
        float dv = 0.f;
        if (valids[i]) {
            t.s_cnt = 1.0;
            float l[LPL], p[LPL], logp[LPL], lq[LPL];
#pragma unroll
            for (int k = 0; k < LPL; ++k) { p[k] = 0.f; logp[k] = 0.f; lq[k] = 0.f; }
            wide_load<LPL>(logits + i * A, A, lane, l);
            float lo[LPL], po[LPL];
            if (logits_old) wide_load<LPL>(logits_old + i * A, A, lane, lo);
            float lp = 0.f, Htot = 0.f, kltot = 0.f, skltot = 0.f;
            float segH[8], segKL[8], segS1[8];
            int act_idx[8];
            int start = 0;
            for (int s = 0; s < sg.n; ++s) {
                const int end = start + sg.len[s];
                wide_softmax<LPL>(l, start, end, lane, p, logp);
                if (logits_old) wide_softmax<LPL>(lo, start, end, lane, po, lq);
                act_idx[s] = start + (int)actions[i * sg.n + s];
                lp += wide_get<LPL>(logp, act_idx[s], lane);
                const float u = 1.f / (float)sg.len[s], log_u = -logf((float)sg.len[s]);
                float h = 0.f, klp = 0.f, s1 = 0.f, s2 = 0.f;
#pragma unroll
                for (int k = 0; k < LPL; ++k) {
                    const int a = k * 32 + lane;
                    if (a >= start && a < end) {
                        h -= logp[k] * p[k];
                        if (logits_old) klp += p[k] * (logp[k] - lq[k]);
                        s1 += p[k] * (logp[k] - log_u);
                        s2 += u * (log_u - logp[k]);
                    }
                }
                segH[s] = warp_sum(h);
                segKL[s] = warp_sum(klp);
                segS1[s] = warp_sum(s1);
                Htot += segH[s];
                kltot += segKL[s];
                skltot += 0.5f * (segS1[s] + warp_sum(s2));
                start = end;
            }
            const float g_lp = ppo_policy_terms(lp, lp_old[i], adv[i], adv_mean, adv_std, clip_lo, clip_hi, w, t);
            t.s_ent = Htot;
            if (expl_mode == 1) t.s_skl = skltot;
            if (logits_old) { t.s_kl = kltot; t.m_kl = kltot; }
            const float we = w * c_ent, wk = (logits_old ? w * c_kl : 0.f);
            start = 0;
            for (int s = 0; s < sg.n; ++s) {
                const int end = start + sg.len[s];
                const float u = 1.f / (float)sg.len[s], log_u = -logf((float)sg.len[s]);
#pragma unroll
                for (int k = 0; k < LPL; ++k) {
                    const int a = k * 32 + lane;
                    if (a >= start && a < end) {
                        float g = g_lp * ((a == act_idx[s] ? 1.f : 0.f) - p[k]);
                        if (expl_mode == 1) g += we * 0.5f * (p[k] * ((logp[k] - log_u) - segS1[s]) + p[k] - u);
                        else g += we * p[k] * (logp[k] + segH[s]);
                        if (logits_old) g += wk * p[k] * ((logp[k] - lq[k]) - segKL[s]);
                        dl[k] = g;
                    }
                }
                start = end;
            }
            dv = ppo_value_terms(v, v_old[i], targets[i], clip_value, w, c_val, t);
        }
        wide_store<LPL>(dlogits + i * A, A, lane, dl);
        if (lane == 0) dvalues[i] = dv;
        if (lane == r) acc = t;
    }
    ppo_store_partials(acc, part, sm);
}

template <int LPL>
__global__ void __launch_bounds__(256) ppo_loss_gauss_wide_kernel(
    const float* __restrict__ params, const float* __restrict__ values, int Ad, int adaptive, float tanh_scale,
    const float* __restrict__ actions, const float* __restrict__ lp_old, const float* __restrict__ v_old,
    const float* __restrict__ adv, const float* __restrict__ targets, const uint8_t* __restrict__ valids,
    const float* __restrict__ params_old, int64_t batch, float clip_lo, float clip_hi, float clip_value, float c_ent,
    float c_val, float c_kl, float grad_scale, float* __restrict__ dlogits, float* __restrict__ dlogstd,
    float* __restrict__ dvalues, const double* __restrict__ stats, double* __restrict__ part) {
    __shared__ double sm[8];
    const int lane = threadIdx.x & 31;
    const PpoW pw = ppo_weights(stats, grad_scale);
    const float adv_mean = pw.adv_mean, adv_std = pw.adv_std, w = pw.w;
    PpoAcc acc;   // statistics of sample blockIdx.x * 256 + threadIdx.x
    const int64_t base = blockIdx.x * (int64_t)blockDim.x + (threadIdx.x & ~31);
    for (int r = 0; r < 32; ++r) {
        const int64_t i = base + r;
        if (i >= batch) break;
        PpoAcc t;
        const float v = values[i];
        t.s_v = v;
        float dm[LPL], ds[LPL];
#pragma unroll
        for (int k = 0; k < LPL; ++k) { dm[k] = 0.f; ds[k] = 0.f; }
        float dv = 0.f;
        if (valids[i]) {
            t.s_cnt = 1.0;
            float m[LPL], s[LPL], a_[LPL], sd[LPL], dlt[LPL];
            wide_load<LPL>(params + i * 2 * Ad, Ad, lane, m);
            wide_load<LPL>(params + i * 2 * Ad + Ad, Ad, lane, s);
            wide_load<LPL>(actions + i * Ad, Ad, lane, a_);
            float lpp = 0.f, hp = 0.f;
#pragma unroll
            for (int k = 0; k < LPL; ++k) {
                sd[k] = clampf(expf(s[k]), kStdMin, kStdMax);
                dlt[k] = a_[k] - m[k];
                if (k * 32 + lane < Ad) {
                    const float lsd = logf(sd[k]);
                    lpp += -(dlt[k] * dlt[k]) / (2.f * (sd[k] * sd[k])) - lsd - kHalfLog2PiL;
                    hp += 0.5f + kHalfLog2PiL + lsd;
                }
            }
            const float lp = warp_sum(lpp);
            const float g_lp = ppo_policy_terms(lp, lp_old[i], adv[i], adv_mean, adv_std, clip_lo, clip_hi, w, t);
            t.s_ent = warp_sum(hp);
            const float we = w * c_ent, wk = (params_old ? w * c_kl : 0.f);
            float mo[LPL], so[LPL];
            if (params_old) {
                wide_load<LPL>(params_old + i * 2 * Ad, Ad, lane, mo);
                wide_load<LPL>(params_old + i * 2 * Ad + Ad, Ad, lane, so);
            }
            float klp = 0.f;
#pragma unroll
            for (int k = 0; k < LPL; ++k) {
                if (k * 32 + lane < Ad) {
                    const float ex = expf(s[k]);
                    const float in_range = (ex >= kStdMin && ex <= kStdMax) ? 1.f : 0.f;
                    const float inv_var = 1.f / (sd[k] * sd[k]);
                    float gm = g_lp * dlt[k] * inv_var;
                    float gs = g_lp * (dlt[k] * dlt[k] * inv_var - 1.f) - we;
                    if (params_old) {
                        const float sdo = clampf(expf(so[k]), kStdMin, kStdMax);
                        const float q = sd[k] / sdo, rr = q * q;
                        const float dq = (m[k] - mo[k]) / sdo;
                        klp += 0.5f * (rr + dq * dq - 1.f - logf(rr));
                        gm += wk * dq / sdo;
                        gs += wk * (rr - 1.f);
                    }
                    gs *= in_range;
                    if (!adaptive && tanh_scale > 0.f) {
                        const float tq = m[k] / tanh_scale;
                        gm *= (1.f - tq * tq);
                    }
                    dm[k] = gm;
                    ds[k] = gs;
                }
            }
            if (params_old) {
                const float kl = warp_sum(klp);
                t.s_kl = kl;
                t.m_kl = kl;
            }
            dv = ppo_value_terms(v, v_old[i], targets[i], clip_value, w, c_val, t);
        }
        float* drow = dlogits + i * (adaptive ? 2 * Ad : Ad);
        wide_store<LPL>(drow, Ad, lane, dm);
        wide_store<LPL>(adaptive ? drow + Ad : dlogstd + i * Ad, Ad, lane, ds);
        if (lane == 0) dvalues[i] = dv;
        if (lane == r) acc = t;
    }
    ppo_store_partials(acc, part, sm);
}

// action-ratio pre-pass of V-trace for wide rows: one warp per sample
template <int LPL>
__global__ void __launch_bounds__(256) action_ratio_wide_kernel(const float* __restrict__ logits, int A, Segs sg,
                                                                const float* __restrict__ actions,
                                                                const float* __restrict__ lp_old, int64_t batch,
                                                                float* __restrict__ ratio) {
    const int lane = threadIdx.x & 31;
    const int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    if (i >= batch) return;   // warp-uniform
    float l[LPL], p[LPL], logp[LPL];
    wide_load<LPL>(logits + i * A, A, lane, l);
    float lp = 0.f;
    int start = 0;
    for (int s = 0; s < sg.n; ++s) {   // (a plain Discrete space is one segment)
        const int end = start + sg.len[s];
        wide_softmax<LPL>(l, start, end, lane, p, logp);
        lp += wide_get<LPL>(logp, start + (int)actions[i * sg.n + s], lane);
        start = end;
    }
    if (lane == 0) ratio[i] = clampf(expf(lp - lp_old[i]), 0.05f, 20.0f);
}

template <int LPL>
__global__ void __launch_bounds__(256) action_ratio_gauss_wide_kernel(const float* __restrict__ params, int Ad,
                                                                      const float* __restrict__ actions,
                                                                      const float* __restrict__ lp_old, int64_t batch,
                                                                      float* __restrict__ ratio) {
    const int lane = threadIdx.x & 31;
    const int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    if (i >= batch) return;
    float m[LPL], s[LPL], a_[LPL];
    wide_load<LPL>(params + i * 2 * Ad, Ad, lane, m);
    wide_load<LPL>(params + i * 2 * Ad + Ad, Ad, lane, s);
    wide_load<LPL>(actions + i * Ad, Ad, lane, a_);
    float lpp = 0.f;
#pragma unroll
    for (int k = 0; k < LPL; ++k) {
        if (k * 32 + lane < Ad) {
            const float sd = clampf(expf(s[k]), kStdMin, kStdMax);
            const float d = a_[k] - m[k];
            lpp += -(d * d) / (2.f * (sd * sd)) - logf(sd) - kHalfLog2PiL;
        }
    }
    const float lp = warp_sum(lpp);
    if (lane == 0) ratio[i] = clampf(expf(lp - lp_old[i]), 0.05f, 20.0f);
}

// ---- Tuple of Discrete and Box members (mixed_layout.cuh): one warp per sample at every width --------------------
// Log-prob, entropy and KL are sums over the members; a categorical member normalises over its own logits, a Gaussian
// member uses the formulas of ppo_loss_gauss_kernel with its [means | log_std] columns.  Slot k of lane l holds params
// column k*32 + l; a Gaussian slot reads its partner column (log_std of a mean, mean of a log_std) from memory.
template <int LPL>
__device__ __forceinline__ float mixed_log_prob(const float* __restrict__ prow, const float* __restrict__ arow,
                                                const MixedLayout& ml, int lane, const float (&l)[LPL], float (&p)[LPL],
                                                float (&logp)[LPL], float (&segH)[kMixedMaxHeads], int (&act_idx)[kMixedMaxHeads],
                                                float& Htot) {
    float lp = 0.f, lpg = 0.f, hg = 0.f;
    Htot = 0.f;
    for (int s = 0; s < ml.K; ++s) {
        const int po = ml.pofs[s], n = ml.size[s];
        if (ml.kind[s] == kMixedCategorical) {
            wide_softmax<LPL>(l, po, po + n, lane, p, logp);
            act_idx[s] = po + (int)arow[ml.aofs[s]];
            lp += wide_get<LPL>(logp, act_idx[s], lane);
            float h = 0.f;
#pragma unroll
            for (int k = 0; k < LPL; ++k) {
                const int a = k * 32 + lane;
                if (a >= po && a < po + n) h -= logp[k] * p[k];
            }
            segH[s] = warp_sum(h);
            Htot += segH[s];
        } else {
#pragma unroll
            for (int k = 0; k < LPL; ++k) {
                const int a = k * 32 + lane;
                if (a >= po && a < po + n) {
                    const float sd = clampf(expf(prow[a + n]), kStdMin, kStdMax);
                    const float d = arow[ml.aofs[s] + a - po] - l[k];
                    const float lsd = logf(sd);
                    lpg += -(d * d) / (2.f * (sd * sd)) - lsd - kHalfLog2PiL;
                    hg += 0.5f + kHalfLog2PiL + lsd;
                }
            }
        }
    }
    Htot += warp_sum(hg);
    return lp + warp_sum(lpg);
}

template <int LPL>
__global__ void __launch_bounds__(256) ppo_loss_mixed_kernel(
    const float* __restrict__ params, const float* __restrict__ values, const MixedLayout ml,
    const float* __restrict__ actions, const float* __restrict__ lp_old, const float* __restrict__ v_old,
    const float* __restrict__ adv, const float* __restrict__ targets, const uint8_t* __restrict__ valids,
    const float* __restrict__ params_old, int64_t batch, float clip_lo, float clip_hi, float clip_value, float c_ent,
    float c_val, float c_kl, float grad_scale, float* __restrict__ dlogits, float* __restrict__ dvalues,
    const double* __restrict__ stats, double* __restrict__ part) {
    __shared__ double sm[8];
    const int lane = threadIdx.x & 31;
    const PpoW pw = ppo_weights(stats, grad_scale);
    const float adv_mean = pw.adv_mean, adv_std = pw.adv_std, w = pw.w;
    PpoAcc acc;   // statistics of sample blockIdx.x * 256 + threadIdx.x
    const int64_t base = blockIdx.x * (int64_t)blockDim.x + (threadIdx.x & ~31);
    const int A = ml.A;
    for (int r = 0; r < 32; ++r) {
        const int64_t i = base + r;
        if (i >= batch) break;   // warp-uniform
        PpoAcc t;
        const float v = values[i];
        t.s_v = v;
        float dl[LPL];
#pragma unroll
        for (int k = 0; k < LPL; ++k) dl[k] = 0.f;
        float dv = 0.f;
        if (valids[i]) {
            t.s_cnt = 1.0;
            const float* prow = params + i * A;
            const float* orow = params_old ? params_old + i * A : nullptr;
            const float* arow = actions + i * ml.W;
            float l[LPL], p[LPL], logp[LPL], lo[LPL], po_[LPL], lq[LPL];
#pragma unroll
            for (int k = 0; k < LPL; ++k) { p[k] = 0.f; logp[k] = 0.f; po_[k] = 0.f; lq[k] = 0.f; }
            wide_load<LPL>(prow, A, lane, l);
            float segH[kMixedMaxHeads], segKL[kMixedMaxHeads];
            int act_idx[kMixedMaxHeads];
            float Htot;
            const float lp = mixed_log_prob<LPL>(prow, arow, ml, lane, l, p, logp, segH, act_idx, Htot);
            float kltot = 0.f;
            if (orow) {
                wide_load<LPL>(orow, A, lane, lo);
                float klg = 0.f;
                for (int s = 0; s < ml.K; ++s) {
                    const int po = ml.pofs[s], n = ml.size[s];
                    if (ml.kind[s] == kMixedCategorical) {
                        wide_softmax<LPL>(lo, po, po + n, lane, po_, lq);
                        float klp = 0.f;
#pragma unroll
                        for (int k = 0; k < LPL; ++k) {
                            const int a = k * 32 + lane;
                            if (a >= po && a < po + n) klp += p[k] * (logp[k] - lq[k]);
                        }
                        segKL[s] = warp_sum(klp);
                        kltot += segKL[s];
                    } else {
#pragma unroll
                        for (int k = 0; k < LPL; ++k) {
                            const int a = k * 32 + lane;
                            if (a >= po && a < po + n) {
                                const float sd = clampf(expf(prow[a + n]), kStdMin, kStdMax);
                                const float sdo = clampf(expf(orow[a + n]), kStdMin, kStdMax);
                                const float q = sd / sdo, rr = q * q;
                                const float dq = (l[k] - lo[k]) / sdo;
                                klg += 0.5f * (rr + dq * dq - 1.f - logf(rr));
                            }
                        }
                    }
                }
                kltot += warp_sum(klg);
                t.s_kl = kltot;
                t.m_kl = kltot;
            }
            const float g_lp = ppo_policy_terms(lp, lp_old[i], adv[i], adv_mean, adv_std, clip_lo, clip_hi, w, t);
            t.s_ent = Htot;
            const float we = w * c_ent, wk = (orow ? w * c_kl : 0.f);
            for (int s = 0; s < ml.K; ++s) {
                const int po = ml.pofs[s], n = ml.size[s];
                if (ml.kind[s] == kMixedCategorical) {
#pragma unroll
                    for (int k = 0; k < LPL; ++k) {
                        const int a = k * 32 + lane;
                        if (a >= po && a < po + n) {
                            float g = g_lp * ((a == act_idx[s] ? 1.f : 0.f) - p[k]);
                            g += we * p[k] * (logp[k] + segH[s]);
                            if (orow) g += wk * p[k] * ((logp[k] - lq[k]) - segKL[s]);
                            dl[k] = g;
                        }
                    }
                } else {
#pragma unroll
                    for (int k = 0; k < LPL; ++k) {
                        const int a = k * 32 + lane;
                        if (a < po || a >= po + 2 * n) continue;
                        const bool is_mean = a < po + n;
                        const int j = is_mean ? a - po : a - po - n;
                        const float m = is_mean ? l[k] : prow[po + j];
                        const float ls = is_mean ? prow[po + n + j] : l[k];
                        const float ex = expf(ls);
                        const float sd = clampf(ex, kStdMin, kStdMax);
                        const float inv_var = 1.f / (sd * sd);
                        const float dlt = arow[ml.aofs[s] + j] - m;
                        float g;
                        if (is_mean) {
                            g = g_lp * dlt * inv_var;
                            if (orow) {
                                const float sdo = clampf(expf(orow[po + n + j]), kStdMin, kStdMax);
                                g += wk * ((m - orow[po + j]) / sdo) / sdo;
                            }
                        } else {
                            g = g_lp * (dlt * dlt * inv_var - 1.f) - we;
                            if (orow) {
                                const float q = sd / clampf(expf(orow[po + n + j]), kStdMin, kStdMax);
                                g += wk * (q * q - 1.f);
                            }
                            g *= (ex >= kStdMin && ex <= kStdMax) ? 1.f : 0.f;   // the clamp passes gradient inside only
                        }
                        dl[k] = g;
                    }
                }
            }
            dv = ppo_value_terms(v, v_old[i], targets[i], clip_value, w, c_val, t);
        }
        wide_store<LPL>(dlogits + i * A, A, lane, dl);
        if (lane == 0) dvalues[i] = dv;
        if (lane == r) acc = t;
    }
    ppo_store_partials(acc, part, sm);
}

template <int LPL>
__global__ void __launch_bounds__(256) action_ratio_mixed_kernel(const float* __restrict__ params, const MixedLayout ml,
                                                                 const float* __restrict__ actions,
                                                                 const float* __restrict__ lp_old, int64_t batch,
                                                                 float* __restrict__ ratio) {
    const int lane = threadIdx.x & 31;
    const int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    if (i >= batch) return;   // warp-uniform
    float l[LPL], p[LPL], logp[LPL], segH[kMixedMaxHeads], Htot;
    int act_idx[kMixedMaxHeads];
    wide_load<LPL>(params + i * ml.A, ml.A, lane, l);
    const float lp = mixed_log_prob<LPL>(params + i * ml.A, actions + i * ml.W, ml, lane, l, p, logp, segH, act_idx, Htot);
    if (lane == 0) ratio[i] = clampf(expf(lp - lp_old[i]), 0.05f, 20.0f);
}

// ---- host side: width -> kernel instantiation, and the tail every loss entry point shares -----------------------------
template <int N>
using Int = std::integral_constant<int, N>;

// f(Int<LPL>) for a one-warp-per-sample row of n > 32 elements (LPL = elements per lane)
template <class F>
static void with_lpl(int n, F&& f) {
    if (n <= 64) f(Int<2>{});
    else if (n <= 128) f(Int<4>{});
    else if (n <= 256) f(Int<8>{});
    else if (n <= 512) f(Int<16>{});
    else f(Int<32>{});
}

// narrow(Int<AMAX>) for rows of up to 32 elements (one thread per sample), else wide(Int<LPL>)
template <class Narrow, class Wide>
static void with_width(int n, Narrow&& narrow, Wide&& wide) {
    if (n <= 8) narrow(Int<8>{});
    else if (n <= 16) narrow(Int<16>{});
    else if (n <= 32) narrow(Int<32>{});
    else with_lpl(n, wide);
}

// a mixed Tuple takes one warp per sample at every width
template <class F>
static void with_mixed_lpl(int A, F&& f) {
    if (A <= 32) f(Int<1>{});
    else with_lpl(A, f);
}

// the launch of a loss kernel: clip window, grid, and the workspace split (loss partials first, ppo_loss_finalize_kernel
// reduces them)
struct LossLaunch {
    float clip_lo, clip_hi;
    unsigned grid;
    double* part;
    cudaStream_t st;
};

static LossLaunch loss_launch(int64_t batch, float clip_ratio, void* workspace, void* stream) {
    LossLaunch L;
    L.clip_hi = 1.0f + clip_ratio;      // learner.py:544
    L.clip_lo = 1.0f / L.clip_hi;       // :546
    L.grid = (unsigned)ceil_div(batch, 256);
    L.part = (double*)workspace;
    L.st = (cudaStream_t)stream;
    return L;
}

// checks the loss kernel's launch and runs the finalize
static int loss_finalize(const LossLaunch& L, int64_t batch, float c_ent, int expl_mode, float c_val, float c_kl,
                         double* stats) {
    SFB_LAUNCH_OK();
    ppo_loss_finalize_kernel<<<1, 256, 0, L.st>>>(L.part, (int)L.grid, batch, c_ent, expl_mode, c_val, c_kl, stats);
    SFB_LAUNCH_OK();
    return 0;
}

// grid of a ratio kernel: 256 samples per block (one per thread) or 8 (one per warp)
static unsigned ratio_grid(int64_t batch, bool wide) { return (unsigned)ceil_div(batch, wide ? 8 : 256); }

static int make_segs(Segs& sg, int A, int num_heads, const int32_t* head_sizes) {
    SFB_CHECK_ARG(num_heads >= 1 && num_heads <= 8 && head_sizes, "tuple action space: 1 <= number of heads <= 8");
    int tot = 0;
    sg.n = num_heads;
    for (int k = 0; k < 8; ++k) sg.len[k] = k < num_heads ? head_sizes[k] : 0;
    for (int k = 0; k < num_heads; ++k) tot += head_sizes[k];
    SFB_CHECK_ARG(tot == A && A <= kWideMax, "tuple action space: head sizes must sum to A = %d (<= %d), got %d", A, kWideMax,
                  tot);
    return 0;
}

}  // namespace sfb

using namespace sfb;

extern "C" {

int64_t sfb200_loss_workspace_bytes(int64_t batch) {
    int64_t blocks = ceil_div(batch > 0 ? batch : 1, 256);
    return (blocks * kNumPart + (int64_t)kLossMaxBlocks * 3) * (int64_t)sizeof(double);
}

int sfb200_action_ratio(const float* logits, int A, const float* actions_f32, const float* log_prob_old, int64_t batch,
                        float* ratio, void* stream) {
    SFB_CHECK_ARG(logits && actions_f32 && log_prob_old && ratio && batch >= 0, "action_ratio: bad arguments");
    SFB_CHECK_ARG(A >= 1 && A <= kWideMax, "action_ratio: supports 1 <= A <= %d, got %d", kWideMax, A);
    if (batch == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    const Segs one{1, {A}};
    with_width(
        A,
        [&](auto am) {
            action_ratio_kernel<decltype(am)::value><<<ratio_grid(batch, false), 256, 0, st>>>(logits, A, actions_f32,
                                                                                              log_prob_old, batch, ratio);
        },
        [&](auto lpl) {
            action_ratio_wide_kernel<decltype(lpl)::value><<<ratio_grid(batch, true), 256, 0, st>>>(
                logits, A, one, actions_f32, log_prob_old, batch, ratio);
        });
    SFB_LAUNCH_OK();
    return 0;
}

int sfb200_adv_stats(const float* adv, const uint8_t* valids, int64_t batch, double* stats, double* dp_partials,
                     void* workspace, void* stream) {
    SFB_CHECK_ARG(adv && valids && stats && workspace && batch > 0, "adv_stats: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    int64_t blocks = ceil_div(batch, 256 * 4);
    if (blocks > kLossMaxBlocks) blocks = kLossMaxBlocks;
    // the adv-stat partials live after the loss partials in the workspace
    double* part = (double*)workspace + ceil_div(batch, 256) * kNumPart;
    adv_stats_partial_kernel<<<(unsigned)blocks, 256, 0, st>>>(adv, valids, batch, part);
    SFB_LAUNCH_OK();
    adv_stats_finalize_kernel<<<1, 32, 0, st>>>(part, (int)blocks, stats, dp_partials);
    SFB_LAUNCH_OK();
    return 0;
}

int sfb200_adv_stats_finalize(const double* dp_partials, double* stats, void* stream) {
    SFB_CHECK_ARG(dp_partials && stats, "adv_stats_finalize: bad arguments");
    adv_stats_from_partials_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(dp_partials, stats);
    SFB_LAUNCH_OK();
    return 0;
}

int sfb200_ppo_loss_fwd_bwd(const float* logits, const float* values, int A, const float* actions_f32,
                            const float* log_prob_old, const float* values_old, const float* adv, const float* targets,
                            const uint8_t* valids, const float* logits_old, int64_t batch, float clip_ratio,
                            float clip_value, float exploration_coeff, int exploration_loss, float value_coeff,
                            float kl_coeff, float grad_scale, float* dlogits, float* dvalues, double* stats,
                            void* workspace, void* stream) {
    SFB_CHECK_ARG(exploration_loss == 0 || exploration_loss == 1, "ppo_loss_fwd_bwd: exploration_loss must be 0 (entropy) or 1 (symmetric_kl)");
    SFB_CHECK_ARG(logits && values && actions_f32 && log_prob_old && values_old && adv && targets && valids && dlogits &&
                      dvalues && stats && workspace && batch > 0, "ppo_loss_fwd_bwd: bad arguments");
    SFB_CHECK_ARG(A >= 1 && A <= kWideMax, "ppo_loss_fwd_bwd: supports 1 <= A <= %d, got %d", kWideMax, A);
    const LossLaunch L = loss_launch(batch, clip_ratio, workspace, stream);
    auto launch = [&](auto kernel) {
        kernel<<<L.grid, 256, 0, L.st>>>(logits, values, A, actions_f32, log_prob_old, values_old, adv, targets, valids,
                                         logits_old, batch, L.clip_lo, L.clip_hi, clip_value, exploration_coeff,
                                         exploration_loss, value_coeff, kl_coeff, grad_scale, dlogits, dvalues, stats, L.part);
    };
    with_width(A, [&](auto am) { launch(ppo_loss_kernel<decltype(am)::value>); },
               [&](auto lpl) { launch(ppo_loss_wide_kernel<decltype(lpl)::value>); });
    return loss_finalize(L, batch, exploration_coeff, exploration_loss, value_coeff, kl_coeff, stats);
}

int sfb200_action_ratio_tuple(const float* logits, int A, int num_heads, const int32_t* head_sizes_host,
                              const float* actions_f32, const float* log_prob_old, int64_t batch, float* ratio,
                              void* stream) {
    SFB_CHECK_ARG(logits && actions_f32 && log_prob_old && ratio && batch >= 0, "action_ratio_tuple: bad arguments");
    Segs sg;
    if (int rc = make_segs(sg, A, num_heads, head_sizes_host)) return rc;
    if (batch == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    auto launch = [&](auto kernel, bool wide) {
        kernel<<<ratio_grid(batch, wide), 256, 0, st>>>(logits, A, sg, actions_f32, log_prob_old, batch, ratio);
    };
    with_width(A, [&](auto am) { launch(action_ratio_tuple_kernel<decltype(am)::value>, false); },
               [&](auto lpl) { launch(action_ratio_wide_kernel<decltype(lpl)::value>, true); });
    SFB_LAUNCH_OK();
    return 0;
}

int sfb200_ppo_loss_fwd_bwd_tuple(const float* logits, const float* values, int A, int num_heads,
                                  const int32_t* head_sizes_host, const float* actions_f32, const float* log_prob_old,
                                  const float* values_old, const float* adv, const float* targets, const uint8_t* valids,
                                  const float* logits_old, int64_t batch, float clip_ratio, float clip_value,
                                  float exploration_coeff, int exploration_loss, float value_coeff, float kl_coeff,
                                  float grad_scale, float* dlogits, float* dvalues, double* stats, void* workspace,
                                  void* stream) {
    SFB_CHECK_ARG(logits && values && actions_f32 && log_prob_old && values_old && adv && targets && valids && dlogits &&
                      dvalues && stats && workspace && batch > 0, "ppo_loss_fwd_bwd_tuple: bad arguments");
    SFB_CHECK_ARG(exploration_loss == 0 || exploration_loss == 1, "ppo_loss_fwd_bwd_tuple: exploration_loss must be 0 or 1");
    Segs sg;
    if (int rc = make_segs(sg, A, num_heads, head_sizes_host)) return rc;
    const LossLaunch L = loss_launch(batch, clip_ratio, workspace, stream);
    auto launch = [&](auto kernel) {
        kernel<<<L.grid, 256, 0, L.st>>>(logits, values, A, sg, actions_f32, log_prob_old, values_old, adv, targets, valids,
                                         logits_old, batch, L.clip_lo, L.clip_hi, clip_value, exploration_coeff,
                                         exploration_loss, value_coeff, kl_coeff, grad_scale, dlogits, dvalues, stats, L.part);
    };
    with_width(A, [&](auto am) { launch(ppo_loss_tuple_kernel<decltype(am)::value>); },
               [&](auto lpl) { launch(ppo_loss_tuple_wide_kernel<decltype(lpl)::value>); });
    return loss_finalize(L, batch, exploration_coeff, exploration_loss, value_coeff, kl_coeff, stats);
}

int sfb200_action_ratio_continuous(const float* params, int act_dim, const float* actions_f32, const float* log_prob_old,
                                   int64_t batch, float* ratio, void* stream) {
    SFB_CHECK_ARG(params && actions_f32 && log_prob_old && ratio && batch >= 0, "action_ratio_continuous: bad arguments");
    SFB_CHECK_ARG(act_dim >= 1 && act_dim <= kWideMax, "action_ratio_continuous: supports 1 <= act_dim <= %d, got %d",
                  kWideMax, act_dim);
    if (batch == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    auto launch = [&](auto kernel, bool wide) {
        kernel<<<ratio_grid(batch, wide), 256, 0, st>>>(params, act_dim, actions_f32, log_prob_old, batch, ratio);
    };
    with_width(act_dim, [&](auto ah) { launch(action_ratio_gauss_kernel<decltype(ah)::value>, false); },
               [&](auto lpl) { launch(action_ratio_gauss_wide_kernel<decltype(lpl)::value>, true); });
    SFB_LAUNCH_OK();
    return 0;
}

int sfb200_ppo_loss_fwd_bwd_continuous(const float* params, const float* values, int act_dim, int adaptive_stddev,
                                       float tanh_scale, const float* actions_f32, const float* log_prob_old,
                                       const float* values_old, const float* adv, const float* targets,
                                       const uint8_t* valids, const float* params_old, int64_t batch, float clip_ratio,
                                       float clip_value, float exploration_coeff, float value_coeff, float kl_coeff,
                                       float grad_scale, float* dlogits, float* dlogstd, float* dvalues, double* stats,
                                       void* workspace, void* stream) {
    SFB_CHECK_ARG(params && values && actions_f32 && log_prob_old && values_old && adv && targets && valids && dlogits &&
                      dvalues && stats && workspace && batch > 0, "ppo_loss_fwd_bwd_continuous: bad arguments");
    SFB_CHECK_ARG(act_dim >= 1 && act_dim <= kWideMax, "ppo_loss_fwd_bwd_continuous: supports 1 <= act_dim <= %d, got %d",
                  kWideMax, act_dim);
    SFB_CHECK_ARG(adaptive_stddev || dlogstd, "ppo_loss_fwd_bwd_continuous: dlogstd is required when adaptive_stddev=0");
    const LossLaunch L = loss_launch(batch, clip_ratio, workspace, stream);
    auto launch = [&](auto kernel) {
        kernel<<<L.grid, 256, 0, L.st>>>(params, values, act_dim, adaptive_stddev, tanh_scale, actions_f32, log_prob_old,
                                         values_old, adv, targets, valids, params_old, batch, L.clip_lo, L.clip_hi,
                                         clip_value, exploration_coeff, value_coeff, kl_coeff, grad_scale, dlogits, dlogstd,
                                         dvalues, stats, L.part);
    };
    with_width(act_dim, [&](auto ah) { launch(ppo_loss_gauss_kernel<decltype(ah)::value>); },
               [&](auto lpl) { launch(ppo_loss_gauss_wide_kernel<decltype(lpl)::value>); });
    return loss_finalize(L, batch, exploration_coeff, 0, value_coeff, kl_coeff, stats);
}

int sfb200_action_ratio_mixed(const float* params, int A, int num_heads, const int32_t* head_kinds_host,
                              const int32_t* head_sizes_host, const float* actions_f32, const float* log_prob_old,
                              int64_t batch, float* ratio, void* stream) {
    SFB_CHECK_ARG(params && actions_f32 && log_prob_old && ratio && batch >= 0, "action_ratio_mixed: bad arguments");
    MixedLayout ml;
    if (int rc = make_mixed_layout(ml, A, num_heads, head_kinds_host, head_sizes_host, "action_ratio_mixed")) return rc;
    if (batch == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    with_mixed_lpl(A, [&](auto lpl) {
        action_ratio_mixed_kernel<decltype(lpl)::value><<<ratio_grid(batch, true), 256, 0, st>>>(params, ml, actions_f32,
                                                                                                 log_prob_old, batch, ratio);
    });
    SFB_LAUNCH_OK();
    return 0;
}

int sfb200_ppo_loss_fwd_bwd_mixed(const float* params, const float* values, int A, int num_heads,
                                  const int32_t* head_kinds_host, const int32_t* head_sizes_host,
                                  const float* actions_f32, const float* log_prob_old, const float* values_old,
                                  const float* adv, const float* targets, const uint8_t* valids, const float* params_old,
                                  int64_t batch, float clip_ratio, float clip_value, float exploration_coeff,
                                  float value_coeff, float kl_coeff, float grad_scale, float* dlogits, float* dvalues,
                                  double* stats, void* workspace, void* stream) {
    SFB_CHECK_ARG(params && values && actions_f32 && log_prob_old && values_old && adv && targets && valids && dlogits &&
                      dvalues && stats && workspace && batch > 0, "ppo_loss_fwd_bwd_mixed: bad arguments");
    MixedLayout ml;
    if (int rc = make_mixed_layout(ml, A, num_heads, head_kinds_host, head_sizes_host, "ppo_loss_fwd_bwd_mixed")) return rc;
    const LossLaunch L = loss_launch(batch, clip_ratio, workspace, stream);
    with_mixed_lpl(A, [&](auto lpl) {
        ppo_loss_mixed_kernel<decltype(lpl)::value><<<L.grid, 256, 0, L.st>>>(
            params, values, ml, actions_f32, log_prob_old, values_old, adv, targets, valids, params_old, batch, L.clip_lo,
            L.clip_hi, clip_value, exploration_coeff, value_coeff, kl_coeff, grad_scale, dlogits, dvalues, stats, L.part);
    });
    return loss_finalize(L, batch, exploration_coeff, 0, value_coeff, kl_coeff, stats);
}

}  // extern "C"
