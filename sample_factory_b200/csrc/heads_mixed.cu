// Heads of a Tuple action space with Box members (mixed_layout.cuh): the distribution tail runs over the STORED params
// row (the trajectory's action_logits slot, the learner's minibatch logits, or the plan's scratch), one warp per row with
// a loop over the members.  A categorical member runs the recipe of tuple_row_tail, a Gaussian member that of
// gaussian_row_tail (heads_tail.cuh).  The params rows come from the regular heads kernels run in values / logits-only
// mode (up to 31 rows: fused partials or heads_forward) or from the distribution_linear GEMM (wider rows), so one kernel
// serves all three entry points.
#include "heads_tail.cuh"
#include "mixed_layout.cuh"

namespace sfb {

struct MixedTail {
    const float* h; int64_t ldh; int H; const float* Wv; const float* bv;   // value head; h == nullptr: values are stored
    const float* lg; int64_t ldl;                                          // params rows
    float* values; int64_t values_stride;
    float* actions; int64_t actions_stride;
    float* log_prob; int64_t log_prob_stride;
    float* pv_out; int64_t pv_stride;
    const float* noise; uint64_t seed, offset_host; const int64_t* offset_dev; const float* pv_scalar;
    int deterministic;
    void* env[kMixedMaxHeads];     // per member: int32 [rows] (Discrete) or float32 [rows, d] (Box); may be null
};

// Slot k of lane l holds params column k*32 + l.
template <int LPL>
__global__ void __launch_bounds__(256) heads_tail_mixed_kernel(int64_t rows, const MixedTail t, const MixedLayout ml) {
    pdl_wait();
    pdl_trigger();
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const float pv = t.pv_scalar ? *t.pv_scalar : 0.f;
    const uint64_t offset = t.offset_host + (t.offset_dev ? (uint64_t)*t.offset_dev : 0ull);
    for (int64_t row = warp; row < rows; row += nwarps) {
        if (t.h) {   // critic_linear: fixed-order lane partials + butterfly (deterministic)
            const float* hr = t.h + row * t.ldh;
            float acc = 0.f;
            for (int j = lane; j < t.H; j += 32) acc = fmaf(hr[j], t.Wv[j], acc);
            const float v = warp_sum(acc) + t.bv[0];
            if (lane == 0) t.values[row * t.values_stride] = v;
        }
        const float* lr = t.lg + row * t.ldl;
        const int64_t nrow = row * ml.Wn;      // Philox subsequence / explicit noise row: row * W' + column
        float x[LPL];
#pragma unroll
        for (int k = 0; k < LPL; ++k) x[k] = (k * 32 + lane < ml.A) ? lr[k * 32 + lane] : 0.f;
        float lp_total = 0.f;
        for (int s = 0; s < ml.K; ++s) {
            const int po = ml.pofs[s], n = ml.size[s], ao = ml.aofs[s], no = ml.nofs[s];
            if (ml.kind[s] == kMixedCategorical) {
                float mloc = -INFINITY;
#pragma unroll
                for (int k = 0; k < LPL; ++k) {
                    const int a = k * 32 + lane;
                    if (a >= po && a < po + n) mloc = fmaxf(mloc, x[k]);
                }
                const float m = warp_max(mloc);
                float e[LPL], sl = 0.f;
#pragma unroll
                for (int k = 0; k < LPL; ++k) {
                    const int a = k * 32 + lane;
                    e[k] = (a >= po && a < po + n) ? expf(x[k] - m) : 0.f;
                    sl += e[k];
                }
                const float sum = warp_sum(sl);
                const float logs = logf(sum);
                float best = -INFINITY;
                int idx = 0x7fffffff;
#pragma unroll
                for (int k = 0; k < LPL; ++k) {
                    const int a = k * 32 + lane;
                    if (a < po || a >= po + n) continue;
                    const int j = a - po;
                    float q = 1.f;
                    if (!t.deterministic) {
                        if (t.noise) q = t.noise[nrow + no + j];
                        else {
                            curandStatePhilox4_32_10_t st;
                            curand_init(t.seed, (unsigned long long)(nrow + no + j), offset, &st);
                            q = fmaxf(-logf(curand_uniform(&st)), 1.0e-30f);   // Exp(1); uniform is in (0, 1]
                        }
                    }
                    const float r = __fdiv_rn(__fdiv_rn(e[k], sum), q);          // torch.multinomial == argmax(p / q)
                    if (r > best || (r == best && j < idx)) { best = r; idx = j; }
                }
                argmax_first(best, idx);
                const int ai = po + idx;
                float mine = 0.f;
#pragma unroll
                for (int k = 0; k < LPL; ++k)
                    if (k == (ai >> 5)) mine = (x[k] - m) - logs;                 // log_softmax :125
                lp_total += __shfl_sync(0xffffffffu, mine, ai & 31);
                if (lane == 0) {
                    t.actions[row * t.actions_stride + ao] = (float)idx;
                    if (t.env[s]) static_cast<int32_t*>(t.env[s])[row] = idx;
                }
            } else {
                float lps = 0.f;
#pragma unroll
                for (int k = 0; k < LPL; ++k) {
                    const int a = k * 32 + lane;
                    if (a < po || a >= po + n) continue;
                    const int j = a - po;
                    const float mean = x[k];
                    const float sd = clampf(expf(lr[a + n]), kStddevMin, kStddevMax);
                    float eps = 0.f;
                    if (!t.deterministic) {
                        if (t.noise) eps = t.noise[nrow + no + j];
                        else {
                            curandStatePhilox4_32_10_t st;
                            curand_init(t.seed, (unsigned long long)(nrow + no + j), offset, &st);
                            eps = curand_normal(&st);
                        }
                    }
                    const float act = __fadd_rn(__fmul_rn(eps, sd), mean);   // Normal.sample(): rounded separately
                    const float d = act - mean;
                    lps += -(d * d) / (2.f * (sd * sd)) - logf(sd) - kHalfLog2Pi;   // normal.py:84-94
                    t.actions[row * t.actions_stride + ao + j] = act;
                    if (t.env[s]) static_cast<float*>(t.env[s])[row * n + j] = act;
                }
                lp_total += warp_sum(lps);                                        // Independent(.., 1)
            }
        }
        if (lane == 0) {
            if (t.log_prob) t.log_prob[row * t.log_prob_stride] = lp_total;   // sum over the members (:231-241)
            if (t.pv_out) t.pv_out[row * t.pv_stride] = pv;
        }
    }
}

static int launch_tail_mixed(int64_t rows, const MixedTail& t, const MixedLayout& ml, cudaStream_t st) {
    if (rows == 0) return 0;
    int64_t blocks = ceil_div(rows, 8);
    const int64_t cap = (int64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
#define SFB_HTM(LPL) SFB_CUDA_OK(launch_pdl(heads_tail_mixed_kernel<LPL>, dim3((unsigned)blocks), dim3(256), 0, st, rows, t, ml))
    if (ml.A <= 32) SFB_HTM(1);
    else if (ml.A <= 64) SFB_HTM(2);
    else if (ml.A <= 128) SFB_HTM(4);
    else if (ml.A <= 256) SFB_HTM(8);
    else if (ml.A <= 512) SFB_HTM(16);
    else SFB_HTM(32);
#undef SFB_HTM
    SFB_LAUNCH_OK();
    return 0;
}

// validates the arguments, applies the calling thread's sampling mode and fills everything but the value-head fields
static int make_mixed_tail(MixedTail& t, MixedLayout& ml, int A, int num_heads, const int32_t* kinds, const int32_t* sizes,
                           float* values, int64_t values_stride, float* params, int64_t params_stride, const float* noise,
                           uint64_t seed, uint64_t offset, const int64_t* offset_dev, float* actions_f32,
                           int64_t actions_stride, void** env_actions_host, float* log_prob, int64_t log_prob_stride,
                           const float* pv_scalar, float* pv_out, int64_t pv_stride, const char* who) {
    if (int rc = make_mixed_layout(ml, A, num_heads, kinds, sizes, who)) return rc;
    SFB_CHECK_ARG(values && params && actions_f32, "%s: values, params and actions are required", who);
    // masks: the reference indexes a Tuple's mask per head along the batch axis, so they are rejected here (dist != 0)
    HeadsOut mode{};
    mode.actions_f32 = actions_f32;
    mode.dist = 1;
    if (int rc = apply_sampling_mode(mode, A)) return rc;
    t = MixedTail{};
    t.lg = params; t.ldl = params_stride;
    t.values = values; t.values_stride = values_stride;
    t.actions = actions_f32; t.actions_stride = actions_stride;
    t.log_prob = log_prob; t.log_prob_stride = log_prob_stride;
    t.pv_out = pv_out; t.pv_stride = pv_stride;
    t.noise = noise; t.seed = seed; t.offset_host = offset; t.offset_dev = offset_dev; t.pv_scalar = pv_scalar;
    t.deterministic = mode.deterministic;
    for (int k = 0; k < num_heads; ++k) t.env[k] = env_actions_host ? env_actions_host[k] : nullptr;
    return 0;
}

}  // namespace sfb

using namespace sfb;

extern "C" {

int sfb200_heads_tail_wide_mixed(const float* h, int64_t ldh, int64_t rows, int H, const float* Wv, const float* bv,
                                 float* params, int64_t params_stride, int A, int num_heads, const int32_t* head_kinds_host,
                                 const int32_t* head_sizes_host, float* values, int64_t values_stride, const float* noise,
                                 uint64_t philox_seed, uint64_t philox_offset, const int64_t* philox_offset_dev,
                                 float* actions_f32, int64_t actions_stride, void** env_actions_host, float* log_prob,
                                 int64_t log_prob_stride, const float* policy_version_scalar, float* policy_version_out,
                                 int64_t pv_stride, void* stream) {
    SFB_CHECK_ARG(h && Wv && bv && rows >= 0 && H > 0, "heads_tail_wide_mixed: bad arguments");
    MixedTail t;
    MixedLayout ml;
    if (int rc = make_mixed_tail(t, ml, A, num_heads, head_kinds_host, head_sizes_host, values, values_stride, params,
                                 params_stride, noise, philox_seed, philox_offset, philox_offset_dev, actions_f32,
                                 actions_stride, env_actions_host, log_prob, log_prob_stride, policy_version_scalar,
                                 policy_version_out, pv_stride, "heads_tail_wide_mixed"))
        return rc;
    t.h = h; t.ldh = ldh; t.H = H; t.Wv = Wv; t.bv = bv;
    return launch_tail_mixed(rows, t, ml, (cudaStream_t)stream);
}

int sfb200_heads_forward_mixed(const float* h, int64_t ldh, int64_t rows, int H, int A, int num_heads,
                               const int32_t* head_kinds_host, const int32_t* head_sizes_host, const float* Wv,
                               const float* bv, const float* Wa, const float* ba, float* values, int64_t values_stride,
                               float* params, int64_t params_stride, const float* noise, uint64_t philox_seed,
                               uint64_t philox_offset, const int64_t* philox_offset_dev, float* actions_f32,
                               int64_t actions_stride, void** env_actions_host, float* log_prob, int64_t log_prob_stride,
                               const float* policy_version_scalar, float* policy_version_out, int64_t pv_stride,
                               void* stream) {
    MixedTail t;
    MixedLayout ml;
    if (int rc = make_mixed_tail(t, ml, A, num_heads, head_kinds_host, head_sizes_host, values, values_stride, params,
                                 params_stride, noise, philox_seed, philox_offset, philox_offset_dev, actions_f32,
                                 actions_stride, env_actions_host, log_prob, log_prob_stride, policy_version_scalar,
                                 policy_version_out, pv_stride, "heads_forward_mixed"))
        return rc;
    // values and the params rows (nothing is sampled without actions), then the tail over the stored rows
    if (int rc = sfb200_heads_forward(h, ldh, rows, H, A, Wv, bv, Wa, ba, values, values_stride, params, params_stride,
                                      nullptr, 0, 0, nullptr, nullptr, 0, nullptr, nullptr, 0, nullptr, nullptr, 0, stream))
        return rc;
    return launch_tail_mixed(rows, t, ml, (cudaStream_t)stream);
}

int sfb200_heads_from_partials_mixed(const float* head_partials, int P, int64_t rows, int A, int num_heads,
                                     const int32_t* head_kinds_host, const int32_t* head_sizes_host, const float* bv,
                                     const float* ba, float* values, int64_t values_stride, float* params,
                                     int64_t params_stride, const float* noise, uint64_t philox_seed,
                                     uint64_t philox_offset, const int64_t* philox_offset_dev, float* actions_f32,
                                     int64_t actions_stride, void** env_actions_host, float* log_prob,
                                     int64_t log_prob_stride, const float* policy_version_scalar,
                                     float* policy_version_out, int64_t pv_stride, void* stream) {
    MixedTail t;
    MixedLayout ml;
    if (int rc = make_mixed_tail(t, ml, A, num_heads, head_kinds_host, head_sizes_host, values, values_stride, params,
                                 params_stride, noise, philox_seed, philox_offset, philox_offset_dev, actions_f32,
                                 actions_stride, env_actions_host, log_prob, log_prob_stride, policy_version_scalar,
                                 policy_version_out, pv_stride, "heads_from_partials_mixed"))
        return rc;
    if (int rc = sfb200_heads_from_partials(head_partials, P, rows, A, bv, ba, values, values_stride, params, params_stride,
                                            nullptr, 0, 0, nullptr, nullptr, 0, nullptr, nullptr, 0, nullptr, nullptr, 0,
                                            stream))
        return rc;
    return launch_tail_mixed(rows, t, ml, (cudaStream_t)stream);
}

}  // extern "C"
