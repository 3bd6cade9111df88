// Heads of models whose distribution_linear has more than 31 rows (ModelSpec.wide_heads): the logits are a GEMM on the
// regular engine (sfb200_linear_act_forward, bias included) written straight into their final place, so what is left
// here is the value head, the distribution tail over the stored logits, and the parts of the backward the two
// linear_backward GEMMs do not cover.  Same semantics as heads_row_tail / tuple_row_tail / gaussian_row_tail
// (heads_tail.cuh), for up to kWideMaxRows logits per row.
#include "heads_tail.cuh"

namespace sfb {

constexpr int kWideMaxRows = 1024;

// One warp per row, LPL slots per lane.  Slot q = k*32 + lane holds element (q - 1) mod 32*LPL: up to 31 elements sit
// on the lanes the narrow tail puts them on (lane a+1 = element a), so every warp reduction below adds the same terms
// in the same order as heads_row_tail (the empty slots contribute exact zeros / -inf); a row of exactly 32*LPL
// elements puts the last one in slot 0.
template <int LPL>
__device__ __forceinline__ int wide_elem(int k, int lane) {
    const int q = k * 32 + lane;
    return q == 0 ? 32 * LPL - 1 : q - 1;
}
// the lane / slot holding element a
template <int LPL>
__device__ __forceinline__ float wide_pick(const float (&v)[LPL], int a, int lane) {
    const int q = (a + 1) & (32 * LPL - 1);
    float mine = 0.f;
#pragma unroll
    for (int k = 0; k < LPL; ++k)
        if (k == (q >> 5)) mine = v[k];
    return __shfl_sync(0xffffffffu, mine, q & 31);
}

struct WideTail {
    const float* h; int64_t ldh; int H; const float* Wv; const float* bv;   // value head input
    float* lg; int64_t ldl;      // logits / [means | log_std] rows, read (and, for a learned stddev, completed) in place
    int A;                       // rows of distribution_linear
    const float* noise; uint64_t seed, offset_host; const int64_t* offset_dev; const float* pv_scalar;
};

// CategoricalActionDistribution with the optional mask (heads_row_tail)
template <int LPL>
__device__ __forceinline__ void wide_categorical(int lane, int64_t row, const WideTail& w, const HeadsOut& out,
                                                 uint64_t offset, float pv) {
    const int A = w.A;
    const float* lr = w.lg + row * w.ldl;
    const bool masked = out.action_mask != nullptr;
    float x[LPL], e[LPL];
    bool ok[LPL];
    float mloc = -INFINITY;
#pragma unroll
    for (int k = 0; k < LPL; ++k) {
        const int a = wide_elem<LPL>(k, lane);
        const bool is_logit = a < A;
        const bool allowed = is_logit && (!masked || out.action_mask[row * out.mask_stride + a] != 0);
        float v = is_logit ? lr[a] : -INFINITY;
        if (masked && is_logit && !allowed) v = __fadd_rn(v, -1.0e9f);   // masked_softmax :84-95
        x[k] = v;
        ok[k] = allowed;
        mloc = fmaxf(mloc, v);
    }
    const float m = warp_max(mloc);
    float sl = 0.f;
#pragma unroll
    for (int k = 0; k < LPL; ++k) {
        e[k] = (wide_elem<LPL>(k, lane) < A) ? expf(x[k] - m) : 0.f;
        sl += e[k];
    }
    const float s = warp_sum(sl);
    const float logs = logf(s);
    float p[LPL];
#pragma unroll
    for (int k = 0; k < LPL; ++k) p[k] = __fdiv_rn(e[k], s);                 // softmax :116
    if (masked) {
        float ps = 0.f;
#pragma unroll
        for (int k = 0; k < LPL; ++k) {
            p[k] = __fmul_rn(p[k], ok[k] ? 1.f : 0.f);                         // :88
            ps += p[k];
        }
        const float den = __fadd_rn(warp_sum(ps), 1.0e-13f);                   // :89
        bool any = false;
#pragma unroll
        for (int k = 0; k < LPL; ++k) {
            p[k] = __fdiv_rn(p[k], den);
            any |= p[k] > 0.f;
        }
        if (__ballot_sync(0xffffffffu, any) == 0u)                             // :137-140 nothing allowed: uniform
#pragma unroll
            for (int k = 0; k < LPL; ++k) p[k] = 1.0e-6f;
    }
    float best = -INFINITY;
    int idx = 0x7fffffff;
#pragma unroll
    for (int k = 0; k < LPL; ++k) {
        const int a = wide_elem<LPL>(k, lane);
        if (a >= A) continue;
        float q = 1.f;
        if (!out.deterministic) {
            if (w.noise) q = w.noise[row * A + a];
            else {
                curandStatePhilox4_32_10_t st;
                curand_init(w.seed, (unsigned long long)(row * A + a), offset, &st);
                q = fmaxf(-logf(curand_uniform(&st)), 1.0e-30f);              // Exp(1); uniform is in (0, 1]
            }
        }
        const float r = __fdiv_rn(p[k], q);
        if (r > best || (r == best && a < idx)) { best = r; idx = a; }
    }
    argmax_first(best, idx);
    float logp[LPL];
#pragma unroll
    for (int k = 0; k < LPL; ++k) logp[k] = (x[k] - m) - logs;                 // log_softmax :125
    const float lp = wide_pick<LPL>(logp, idx, lane);                           // log_prob :145-148
    if (lane == 0) {
        out.actions_f32[row * out.actions_stride] = (float)idx;
        if (out.env_actions) out.env_actions[row] = idx;
        if (out.log_prob) out.log_prob[row * out.log_prob_stride] = lp;
        if (out.pv_out) out.pv_out[row * out.pv_stride] = pv;
    }
}

// TupleActionDistribution (tuple_row_tail): the categorical recipe per head over its own logit segment
template <int LPL>
__device__ __forceinline__ void wide_tuple(int lane, int64_t row, const WideTail& w, const HeadsOut& out, uint64_t offset,
                                           float pv) {
    const int A = w.A;
    const float* lr = w.lg + row * w.ldl;
    float x[LPL], q[LPL];
#pragma unroll
    for (int k = 0; k < LPL; ++k) {
        const int a = wide_elem<LPL>(k, lane);
        x[k] = a < A ? lr[a] : 0.f;
        q[k] = 1.f;
        if (a < A && !out.deterministic) {
            if (w.noise) q[k] = w.noise[row * A + a];
            else {
                curandStatePhilox4_32_10_t st;
                curand_init(w.seed, (unsigned long long)(row * A + a), offset, &st);
                q[k] = fmaxf(-logf(curand_uniform(&st)), 1.0e-30f);
            }
        }
    }
    float lp_total = 0.f;
    int start = 0;
    const int K = out.num_seg;
    for (int s = 0; s < K; ++s) {
        const int n = out.seg_len[s];
        float mloc = -INFINITY;
#pragma unroll
        for (int k = 0; k < LPL; ++k) {
            const int a = wide_elem<LPL>(k, lane);
            if (a >= start && a < start + n) mloc = fmaxf(mloc, x[k]);
        }
        const float m = warp_max(mloc);
        float e[LPL], sl = 0.f;
#pragma unroll
        for (int k = 0; k < LPL; ++k) {
            const int a = wide_elem<LPL>(k, lane);
            e[k] = (a >= start && a < start + n) ? expf(x[k] - m) : 0.f;
            sl += e[k];
        }
        const float sum = warp_sum(sl);
        const float logs = logf(sum);
        float best = -INFINITY, logp[LPL];
        int idx = 0x7fffffff;
#pragma unroll
        for (int k = 0; k < LPL; ++k) {
            const int a = wide_elem<LPL>(k, lane);
            logp[k] = (x[k] - m) - logs;
            if (a >= start && a < start + n) {
                const float r = __fdiv_rn(__fdiv_rn(e[k], sum), q[k]);
                if (r > best || (r == best && a - start < idx)) { best = r; idx = a - start; }
            }
        }
        argmax_first(best, idx);
        lp_total += wide_pick<LPL>(logp, start + idx, lane);
        if (lane == 0) {
            out.actions_f32[row * out.actions_stride + s] = (float)idx;
            if (out.env_actions) out.env_actions[row * K + s] = idx;
        }
        start += n;
    }
    if (lane == 0) {
        if (out.log_prob) out.log_prob[row * out.log_prob_stride] = lp_total;
        if (out.pv_out) out.pv_out[row * out.pv_stride] = pv;
    }
}

// ContinuousActionDistribution (gaussian_row_tail).  The params row is completed in place: tanh-scaled means and the
// learned log-stddev vector (adaptive_stddev=False, action_parameterization.py:64-78); an adaptive row is left as the
// GEMM wrote it.
template <int LPL>
__device__ __forceinline__ void wide_gaussian(int lane, int64_t row, const WideTail& w, const HeadsOut& out,
                                              uint64_t offset, float pv) {
    const int Ad = out.act_dim;
    float* lr = w.lg + row * w.ldl;
    float mean[LPL], lstd[LPL];
#pragma unroll
    for (int k = 0; k < LPL; ++k) {
        const int d = wide_elem<LPL>(k, lane);
        mean[k] = 0.f;
        lstd[k] = 0.f;
        if (d < Ad) {
            mean[k] = lr[d];
            if (out.dist == 1) lstd[k] = lr[Ad + d];
            else {
                lstd[k] = out.learned_log_std[d];
                if (out.tanh_scale > 0.f) mean[k] = tanhf(__fdiv_rn(mean[k], out.tanh_scale)) * out.tanh_scale;
                lr[d] = mean[k];
                lr[Ad + d] = lstd[k];
            }
        }
    }
    if (out.actions_f32 == nullptr) return;   // distribution parameters only (warp-uniform)
    float lps = 0.f;
#pragma unroll
    for (int k = 0; k < LPL; ++k) {
        const int d = wide_elem<LPL>(k, lane);
        if (d >= Ad) continue;
        const float sd = clampf(expf(lstd[k]), kStddevMin, kStddevMax);
        float eps = 0.f;
        if (!out.deterministic) {
            if (w.noise) eps = w.noise[row * Ad + d];
            else {
                curandStatePhilox4_32_10_t st;
                curand_init(w.seed, (unsigned long long)(row * Ad + d), offset, &st);
                eps = curand_normal(&st);
            }
        }
        const float a = __fadd_rn(__fmul_rn(eps, sd), mean[k]);   // Normal.sample(): product and sum rounded separately
        const float dd = a - mean[k];
        lps += -(dd * dd) / (2.f * (sd * sd)) - logf(sd) - kHalfLog2Pi;
        out.actions_f32[row * out.actions_stride + d] = a;
        if (out.env_actions_f32) out.env_actions_f32[row * Ad + d] = a;
    }
    const float lp = warp_sum(lps);
    if (lane == 0) {
        if (out.log_prob) out.log_prob[row * out.log_prob_stride] = lp;
        if (out.pv_out) out.pv_out[row * out.pv_stride] = pv;
    }
}

template <int LPL>
__global__ void __launch_bounds__(256) heads_tail_wide_kernel(int64_t rows, const WideTail w, const HeadsOut out) {
    pdl_wait();
    pdl_trigger();
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const float pv = w.pv_scalar ? *w.pv_scalar : 0.f;
    const uint64_t offset = w.offset_host + (w.offset_dev ? (uint64_t)*w.offset_dev : 0ull);
    for (int64_t row = warp; row < rows; row += nwarps) {
        // critic_linear: fixed-order lane partials + butterfly (deterministic)
        const float* hr = w.h + row * w.ldh;
        float acc = 0.f;
        for (int j = lane; j < w.H; j += 32) acc = fmaf(hr[j], w.Wv[j], acc);
        const float v = warp_sum(acc) + w.bv[0];
        if (lane == 0) out.values[row * out.values_stride] = v;
        if (w.lg == nullptr) continue;             // values only (the learner's bootstrap value)
        if (out.dist != 0) wide_gaussian<LPL>(lane, row, w, out, offset, pv);
        else if (out.actions_f32 == nullptr) continue;
        else if (out.num_seg > 1) wide_tuple<LPL>(lane, row, w, out, offset, pv);
        else wide_categorical<LPL>(lane, row, w, out, offset, pv);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Backward pieces around the two linear_backward GEMMs (dWa = dlogits^T . h and dz = (dlogits . Wa) * act'(h)):
//   dz[:, value_col + j] (+)= act'(h[:, j]) * dvalues * Wv[j]      (the rank-1 value term)
//   db_prev[c] = sum_i dz[i, c] (c < width),  dWv[j] = sum_i dvalues[i] h[i, j],  dba = sum_i dlogits[i, :],  dbv = sum dvalues
// grid (column blocks, row groups): a thread owns one column of [dz (width) | dlogits (A) | dvalues] and walks the rows of
// its group in order; part[group] = [db (width) | dba (A) | dbv | dWv (H)], reduced over the groups in a fixed order.
constexpr int kWideBwdMaxGroups = 128;

static int64_t wide_bwd_groups(int64_t rows) {
    int64_t g = ceil_div(rows > 0 ? rows : 1, 64);
    return g < kWideBwdMaxGroups ? g : kWideBwdMaxGroups;
}

__global__ void __launch_bounds__(256) heads_wide_backward_kernel(
    const float* __restrict__ h, int64_t ldh, int64_t rows, int H, const float* __restrict__ Wv,
    const float* __restrict__ dlogits, int A, const float* __restrict__ dvalues, int act, float* __restrict__ dz,
    int64_t lddz, int width, int value_col, int accumulate, int64_t rows_per_group, float* __restrict__ part) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    const int ncols = width + A + 1;
    if (c >= ncols) return;
    const int64_t r0 = blockIdx.y * rows_per_group;
    const int64_t r1 = (r0 + rows_per_group < rows) ? r0 + rows_per_group : rows;
    float* my = part + (int64_t)blockIdx.y * (ncols + H);
    if (c < width) {
        const int j = c - value_col;
        const bool vcol = j >= 0 && j < H;
        const float wv = vcol ? Wv[j] : 0.f;
        float sdb = 0.f, sdw = 0.f;
        for (int64_t i = r0; i < r1; ++i) {
            float d;
            if (vcol) {
                const float hv = h[i * ldh + j], dv = dvalues[i];
                const float t = (dv * wv) * act_bwd_from_out(hv, act);
                d = accumulate ? dz[i * lddz + c] + t : t;
                dz[i * lddz + c] = d;
                sdw = fmaf(dv, hv, sdw);
            } else {
                d = dz[i * lddz + c];
            }
            sdb += d;
        }
        my[c] = sdb;
        if (vcol) my[ncols + j] = sdw;
    } else if (c < width + A) {
        const int a = c - width;
        float s = 0.f;
        for (int64_t i = r0; i < r1; ++i) s += dlogits[i * A + a];
        my[c] = s;
    } else {
        float s = 0.f;
        for (int64_t i = r0; i < r1; ++i) s += dvalues[i];
        my[c] = s;
    }
}

__global__ void __launch_bounds__(256) heads_wide_backward_reduce_kernel(const float* __restrict__ part, int groups,
                                                                         int width, int A, int H, float* __restrict__ db_prev,
                                                                         float* __restrict__ dba, float* __restrict__ dbv,
                                                                         float* __restrict__ dWv) {
    const int ncols = width + A + 1;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ncols + H) return;
    float s = 0.f;
    for (int g = 0; g < groups; ++g) s += part[(int64_t)g * (ncols + H) + i];
    if (i < width) { if (db_prev) db_prev[i] = s; }
    else if (i < width + A) dba[i - width] = s;
    else if (i == width + A) dbv[0] = s;
    else dWv[i - ncols] = s;
}

}  // namespace sfb

using namespace sfb;

extern "C" {

int sfb200_heads_tail_wide(const float* h, int64_t ldh, int64_t rows, int H, const float* Wv, const float* bv,
                           float* logits, int64_t logits_stride, int A, int dist_kind, int act_dim, int adaptive_stddev,
                           const float* learned_log_std, float tanh_scale, int num_heads, const int32_t* head_sizes_host,
                           float* values, int64_t values_stride, const float* noise, uint64_t philox_seed,
                           uint64_t philox_offset, const int64_t* philox_offset_dev, float* actions_f32,
                           int64_t actions_stride, void* env_actions, float* log_prob, int64_t log_prob_stride,
                           const float* policy_version_scalar, float* policy_version_out, int64_t pv_stride,
                           void* stream) {
    SFB_CHECK_ARG(h && Wv && bv && values && rows >= 0 && H > 0, "heads_tail_wide: bad arguments");
    SFB_CHECK_ARG(A >= 1 && A <= kWideMaxRows, "heads_tail_wide: supports 1 <= distribution_linear rows <= %d, got %d",
                  kWideMaxRows, A);
    SFB_CHECK_ARG(dist_kind >= 0 && dist_kind <= 2, "heads_tail_wide: dist_kind 0 categorical, 1 tuple, 2 Gaussian");
    SFB_CHECK_ARG(logits || !actions_f32, "heads_tail_wide: sampling needs the logits rows");
    HeadsOut out{values, values_stride, logits, logits_stride, actions_f32, actions_stride, nullptr, log_prob,
                 log_prob_stride, policy_version_out, pv_stride, 0, 0, nullptr, 0.f, nullptr};
    int slots = A;
    if (dist_kind == 2) {
        SFB_CHECK_ARG(act_dim >= 1 && A == (adaptive_stddev ? 2 * act_dim : act_dim),
                      "heads_tail_wide: A = %d does not match act_dim %d", A, act_dim);
        SFB_CHECK_ARG(adaptive_stddev || learned_log_std, "heads_tail_wide: learned_log_std is required when adaptive_stddev=0");
        out.dist = adaptive_stddev ? 1 : 2;
        out.act_dim = act_dim;
        out.learned_log_std = learned_log_std;
        out.tanh_scale = tanh_scale;
        out.env_actions_f32 = (float*)env_actions;
        slots = act_dim;
    } else {
        out.env_actions = (int32_t*)env_actions;
        if (dist_kind == 1) {
            SFB_CHECK_ARG(num_heads >= 1 && num_heads <= 8 && head_sizes_host, "heads_tail_wide (tuple): 1 <= number of heads <= 8");
            int tot = 0;
            for (int k = 0; k < num_heads; ++k) {
                SFB_CHECK_ARG(head_sizes_host[k] >= 1, "heads_tail_wide (tuple): empty head");
                out.seg_len[k] = head_sizes_host[k];
                tot += head_sizes_host[k];
            }
            SFB_CHECK_ARG(tot == A, "heads_tail_wide (tuple): the heads' sizes sum to %d but distribution_linear has %d rows",
                          tot, A);
            out.num_seg = num_heads;
        }
    }
    if (int rc = apply_sampling_mode(out, A)) return rc;
    if (rows == 0) return 0;
    const WideTail w{h, ldh, H, Wv, bv, logits, logits_stride, A, noise, philox_seed, philox_offset, philox_offset_dev,
                     policy_version_scalar};
    int64_t blocks = ceil_div(rows, 8);
    const int64_t cap = (int64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    cudaStream_t st = (cudaStream_t)stream;
#define SFB_HTW(LPL) SFB_CUDA_OK(launch_pdl(heads_tail_wide_kernel<LPL>, dim3((unsigned)blocks), dim3(256), 0, st, rows, w, out))
    if (slots <= 64) SFB_HTW(2);
    else if (slots <= 128) SFB_HTW(4);
    else if (slots <= 256) SFB_HTW(8);
    else if (slots <= 512) SFB_HTW(16);
    else SFB_HTW(32);
#undef SFB_HTW
    SFB_LAUNCH_OK();
    return 0;
}

int64_t sfb200_heads_wide_backward_workspace_bytes(int64_t rows, int width, int H, int A) {
    return wide_bwd_groups(rows) * ((int64_t)width + A + 1 + H) * (int64_t)sizeof(float);
}

int sfb200_heads_wide_backward(const float* h, int64_t ldh, int64_t rows, int H, const float* Wv, const float* dlogits,
                               int A, const float* dvalues, int act, float* dz, int64_t lddz, int width, int value_col,
                               int accumulate, float* dWv, float* dbv, float* dba, float* db_prev, void* workspace,
                               void* stream) {
    SFB_CHECK_ARG(h && Wv && dlogits && dvalues && dz && dWv && dbv && dba && workspace && rows > 0 && H > 0 && A >= 1,
                  "heads_wide_backward: bad arguments");
    SFB_CHECK_ARG(value_col >= 0 && value_col + H <= width, "heads_wide_backward: value columns [%d, %d) outside dz width %d",
                  value_col, value_col + H, width);
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t groups = wide_bwd_groups(rows);
    const int64_t rpg = ceil_div(rows, groups);
    const int ncols = width + A + 1;
    float* part = (float*)workspace;
    heads_wide_backward_kernel<<<dim3((unsigned)ceil_div(ncols, 256), (unsigned)ceil_div(rows, rpg)), 256, 0, st>>>(
        h, ldh, rows, H, Wv, dlogits, A, dvalues, act, dz, lddz, width, value_col, accumulate, rpg, part);
    SFB_LAUNCH_OK();
    heads_wide_backward_reduce_kernel<<<(unsigned)ceil_div(ncols + H, 256), 256, 0, st>>>(
        part, (int)ceil_div(rows, rpg), width, A, H, db_prev, dba, dbv, dWv);
    SFB_LAUNCH_OK();
    return 0;
}

}  // extern "C"
