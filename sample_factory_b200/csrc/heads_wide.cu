// Heads over stored params rows.  Models whose distribution_linear has more than 31 rows (ModelSpec.wide_heads): the
// logits are a GEMM on the regular engine (sfb200_linear_act_forward, bias included) written straight into their final
// place, so what is left here is the value head, the distribution tail over the stored logits, and the parts of the
// backward the two linear_backward GEMMs do not cover.  A Tuple space with Box members (mixed_layout.cuh): its params
// rows come from the regular heads kernels run in values / logits-only mode (up to 31 rows: fused partials or
// heads_forward) or from the distribution_linear GEMM (wider rows), and the tail runs over the stored rows at every width.
#include <type_traits>

#include "heads_tail.cuh"

namespace sfb {

constexpr int kWideMaxRows = 1024;

// One warp per stored params row (the logits a distribution_linear GEMM wrote in place, the trajectory's action_logits
// slot, the learner's minibatch logits or a plan's scratch): the value head when h is given, then row_tail over the row
// held LPL elements per lane under slot map S.  Without actions, only a learned-stddev row has anything left to do.
template <int LPL, int S>
__global__ void __launch_bounds__(256) heads_tail_rows_kernel(int64_t rows, const float* __restrict__ h, int64_t ldh, int H,
                                                              const float* __restrict__ Wv, const HeadsFinish f) {
    pdl_wait();
    pdl_trigger();
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const HeadsOut& out = f.out;
    const float pv = f.pv_scalar ? *f.pv_scalar : 0.f;
    const uint64_t offset = f.offset_host + (f.offset_dev ? (uint64_t)*f.offset_dev : 0ull);
    const bool tail = out.logits && (out.actions_f32 || out.lay.m.kind[0] == kMixedGaussianLearned);
    for (int64_t row = warp; row < rows; row += nwarps) {
        if (h) {   // critic_linear: fixed-order lane partials + butterfly (deterministic)
            const float* hr = h + row * ldh;
            float acc = 0.f;
            for (int j = lane; j < H; j += 32) acc = fmaf(hr[j], Wv[j], acc);
            const float v = warp_sum(acc) + f.bv[0];
            if (lane == 0) out.values[row * out.values_stride] = v;
        }
        if (!tail) continue;
        const float* lr = out.logits + row * out.logits_stride;
        float x[LPL];
#pragma unroll
        for (int k = 0; k < LPL; ++k) {
            const int a = slot_elem<LPL, S>(k, lane);
            x[k] = a < out.lay.m.A ? lr[a] : 0.f;
        }
        row_tail<LPL, S>(x, lane, row, out, f.noise, f.seed, offset, pv);
    }
}

template <int N>
using Int = std::integral_constant<int, N>;

// A wide Discrete / Tuple / Box row (S = 1, LPL >= 2 by the widest member) bit-matches the narrow heads up to 31
// elements.  A mixed Tuple takes S = 0 at every width (LPL >= 1 by the row width).
static int launch_tail_rows(int64_t rows, const float* h, int64_t ldh, int H, const float* Wv, const HeadsFinish& f,
                            bool mixed, cudaStream_t st) {
    if (rows == 0) return 0;
    const MixedLayout& m = f.out.lay.m;
    const int width = (!mixed && m.kind[0] != kMixedCategorical) ? m.size[0] : m.A;
    int64_t blocks = ceil_div(rows, 8);
    const int64_t cap = (int64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    auto go = [&](auto lpl, auto s) {
        return launch_pdl(heads_tail_rows_kernel<decltype(lpl)::value, decltype(s)::value>, dim3((unsigned)blocks), dim3(256),
                          0, st, rows, h, ldh, H, Wv, f);
    };
    auto with_s = [&](auto s) {
        if constexpr (decltype(s)::value == 0)
            if (width <= 32) return go(Int<1>{}, s);
        if (width <= 64) return go(Int<2>{}, s);
        if (width <= 128) return go(Int<4>{}, s);
        if (width <= 256) return go(Int<8>{}, s);
        if (width <= 512) return go(Int<16>{}, s);
        return go(Int<32>{}, s);
    };
    SFB_CUDA_OK(mixed ? with_s(Int<0>{}) : with_s(Int<1>{}));
    SFB_LAUNCH_OK();
    return 0;
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
    if (dist_kind == 2)
        SFB_CHECK_ARG(act_dim >= 1 && A == (adaptive_stddev ? 2 * act_dim : act_dim),
                      "heads_tail_wide: A = %d does not match act_dim %d", A, act_dim);
    HeadsFinish f{{values, values_stride, logits, logits_stride, actions_f32, actions_stride, log_prob, log_prob_stride,
                   policy_version_out, pv_stride},
                  bv, nullptr, noise, philox_seed, philox_offset, philox_offset_dev, policy_version_scalar};
    if (int rc = make_heads_layout(f.out, dist_kind, A, num_heads, nullptr, head_sizes_host, act_dim, adaptive_stddev,
                                   learned_log_std, tanh_scale, env_actions, nullptr, "heads_tail_wide"))
        return rc;
    return launch_tail_rows(rows, h, ldh, H, Wv, f, false, (cudaStream_t)stream);
}

// The three entry points of a Tuple space with Box members: the tail always runs over the stored params rows
int sfb200_heads_tail_wide_mixed(const float* h, int64_t ldh, int64_t rows, int H, const float* Wv, const float* bv,
                                 float* params, int64_t params_stride, int A, int num_heads, const int32_t* head_kinds_host,
                                 const int32_t* head_sizes_host, float* values, int64_t values_stride, const float* noise,
                                 uint64_t philox_seed, uint64_t philox_offset, const int64_t* philox_offset_dev,
                                 float* actions_f32, int64_t actions_stride, void** env_actions_host, float* log_prob,
                                 int64_t log_prob_stride, const float* policy_version_scalar, float* policy_version_out,
                                 int64_t pv_stride, void* stream) {
    SFB_CHECK_ARG(h && Wv && bv && rows >= 0 && H > 0, "heads_tail_wide_mixed: bad arguments");
    HeadsFinish f{{values, values_stride, params, params_stride, actions_f32, actions_stride, log_prob, log_prob_stride,
                   policy_version_out, pv_stride},
                  bv, nullptr, noise, philox_seed, philox_offset, philox_offset_dev, policy_version_scalar};
    if (int rc = make_heads_layout(f.out, 3, A, num_heads, head_kinds_host, head_sizes_host, 0, 0, nullptr, 0.f, nullptr,
                                   env_actions_host, "heads_tail_wide_mixed"))
        return rc;
    return launch_tail_rows(rows, h, ldh, H, Wv, f, true, (cudaStream_t)stream);
}

int sfb200_heads_forward_mixed(const float* h, int64_t ldh, int64_t rows, int H, int A, int num_heads,
                               const int32_t* head_kinds_host, const int32_t* head_sizes_host, const float* Wv,
                               const float* bv, const float* Wa, const float* ba, float* values, int64_t values_stride,
                               float* params, int64_t params_stride, const float* noise, uint64_t philox_seed,
                               uint64_t philox_offset, const int64_t* philox_offset_dev, float* actions_f32,
                               int64_t actions_stride, void** env_actions_host, float* log_prob, int64_t log_prob_stride,
                               const float* policy_version_scalar, float* policy_version_out, int64_t pv_stride,
                               void* stream) {
    HeadsFinish f{{values, values_stride, params, params_stride, actions_f32, actions_stride, log_prob, log_prob_stride,
                   policy_version_out, pv_stride},
                  bv, ba, noise, philox_seed, philox_offset, philox_offset_dev, policy_version_scalar};
    if (int rc = make_heads_layout(f.out, 3, A, num_heads, head_kinds_host, head_sizes_host, 0, 0, nullptr, 0.f, nullptr,
                                   env_actions_host, "heads_forward_mixed"))
        return rc;
    // values and the params rows (nothing is sampled without actions), then the tail over the stored rows
    if (int rc = sfb200_heads_forward(h, ldh, rows, H, A, Wv, bv, Wa, ba, values, values_stride, params, params_stride,
                                      nullptr, 0, 0, nullptr, nullptr, 0, nullptr, nullptr, 0, nullptr, nullptr, 0, stream))
        return rc;
    return launch_tail_rows(rows, nullptr, 0, 0, nullptr, f, true, (cudaStream_t)stream);
}

int sfb200_heads_from_partials_mixed(const float* head_partials, int P, int64_t rows, int A, int num_heads,
                                     const int32_t* head_kinds_host, const int32_t* head_sizes_host, const float* bv,
                                     const float* ba, float* values, int64_t values_stride, float* params,
                                     int64_t params_stride, const float* noise, uint64_t philox_seed,
                                     uint64_t philox_offset, const int64_t* philox_offset_dev, float* actions_f32,
                                     int64_t actions_stride, void** env_actions_host, float* log_prob,
                                     int64_t log_prob_stride, const float* policy_version_scalar,
                                     float* policy_version_out, int64_t pv_stride, void* stream) {
    HeadsFinish f{{values, values_stride, params, params_stride, actions_f32, actions_stride, log_prob, log_prob_stride,
                   policy_version_out, pv_stride},
                  bv, ba, noise, philox_seed, philox_offset, philox_offset_dev, policy_version_scalar};
    if (int rc = make_heads_layout(f.out, 3, A, num_heads, head_kinds_host, head_sizes_host, 0, 0, nullptr, 0.f, nullptr,
                                   env_actions_host, "heads_from_partials_mixed"))
        return rc;
    if (int rc = sfb200_heads_from_partials(head_partials, P, rows, A, bv, ba, values, values_stride, params, params_stride,
                                            nullptr, 0, 0, nullptr, nullptr, 0, nullptr, nullptr, 0, nullptr, nullptr, 0,
                                            stream))
        return rc;
    return launch_tail_rows(rows, nullptr, 0, 0, nullptr, f, true, (cudaStream_t)stream);
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
