// HBM-bound elementwise kernels of the sampler / batch-prep path (see include/sfb200.h for the reference sites).
// All are streaming kernels: coalesced 128-bit accesses where alignment allows, grid sized in multiples of the SM
// count, no shared-memory staging (no reuse).
#include "common.cuh"
#include "step_tail.cuh"

namespace sfb {

// One body serves sfb200_normalize_obs, sfb200_sampler_pre_step and the fused post+pre step: optional second output
// (raw copy into the trajectory at [.., t]) so obs is read from HBM once.
struct NormArgs {
    const void* x; int64_t ldx;          // float32, or uint8 when the kernel is instantiated with U8 (image observations:
    float* y; int64_t ldy;               // the reference converts with .float() first, normalize.py:40-46)
    void* raw_copy; int64_t ld_copy;     // same element type as x
    int64_t rows; int dim;
    ObsNorm n;
    const float* rnn_src; int rnn_dim; float* rnn_dst; int64_t rnn_dst_stride; int64_t rnn_rows;
};

template <bool VEC4, bool U8>
__device__ __forceinline__ void normalize_body(const NormArgs& a) {
    const bool do_rms = a.n.mean != nullptr;
    const int64_t tid0 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t nthr = (int64_t)gridDim.x * blockDim.x;
    if (a.rnn_src) {   // sampler pre-step: traj.rnn_states[:, t] <- rnn (tiny; folded in to save a launch)
        const int64_t tot = a.rnn_rows * a.rnn_dim;
        for (int64_t i = tid0; i < tot; i += nthr) {
            const int64_t r = i / a.rnn_dim;
            a.rnn_dst[r * a.rnn_dst_stride + (i - r * a.rnn_dim)] = a.rnn_src[i];
        }
    }
    const float* xf = reinterpret_cast<const float*>(a.x);
    const uint8_t* xb = reinterpret_cast<const uint8_t*>(a.x);
    float* cf = reinterpret_cast<float*>(a.raw_copy);
    uint8_t* cb = reinterpret_cast<uint8_t*>(a.raw_copy);
    if (VEC4) {
        const int dim4 = a.dim >> 2;
        const int64_t total = a.rows * (int64_t)dim4;
        for (int64_t i = tid0; i < total; i += nthr) {
            const int64_t r = i / dim4;
            const int c = (int)(i - r * dim4) << 2;
            float in[4];
            if (U8) {
                const uchar4 v = *reinterpret_cast<const uchar4*>(xb + r * a.ldx + c);
                if (a.raw_copy) *reinterpret_cast<uchar4*>(cb + r * a.ld_copy + c) = v;
                in[0] = (float)v.x; in[1] = (float)v.y; in[2] = (float)v.z; in[3] = (float)v.w;
            } else {
                const float4 v = *reinterpret_cast<const float4*>(xf + r * a.ldx + c);
                if (a.raw_copy) *reinterpret_cast<float4*>(cf + r * a.ld_copy + c) = v;
                in[0] = v.x; in[1] = v.y; in[2] = v.z; in[3] = v.w;
            }
            if (a.y) {
                float out[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    float mu = 0.f, is = 1.f;
                    if (do_rms) col_stats(a.n.mean, a.n.var, c + k, a.n.eps, mu, is);
                    out[k] = norm_one(in[k], a.n.sub, a.n.inv_scale, a.n.do_sub, a.n.do_scale, do_rms, mu, is, a.n.clip);
                }
                *reinterpret_cast<float4*>(a.y + r * a.ldy + c) = make_float4(out[0], out[1], out[2], out[3]);
            }
        }
    } else {
        const int64_t total = a.rows * (int64_t)a.dim;
        for (int64_t i = tid0; i < total; i += nthr) {
            const int64_t r = i / a.dim;
            const int c = (int)(i - r * a.dim);
            float v;
            if (U8) {
                const uint8_t b = xb[r * a.ldx + c];
                if (a.raw_copy) cb[r * a.ld_copy + c] = b;
                v = (float)b;
            } else {
                v = xf[r * a.ldx + c];
                if (a.raw_copy) cf[r * a.ld_copy + c] = v;
            }
            if (a.y) {
                float mu = 0.f, is = 1.f;
                if (do_rms) col_stats(a.n.mean, a.n.var, c, a.n.eps, mu, is);
                a.y[r * a.ldy + c] = norm_one(v, a.n.sub, a.n.inv_scale, a.n.do_sub, a.n.do_scale, do_rms, mu, is, a.n.clip);
            }
        }
    }
}

template <bool VEC4, bool U8>
__global__ void __launch_bounds__(256) normalize_kernel(const NormArgs a) {
    pdl_wait();
    pdl_trigger();
    normalize_body<VEC4, U8>(a);
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

static bool make_norm_args(NormArgs& a, const void* x, int64_t ldx, float* y, int64_t ldy, void* raw_copy,
                           int64_t ld_copy, int64_t rows, int dim, const double* mean, const double* var, float sub_mean,
                           float inv_scale, float eps, float clip, const float* rnn_src, int rnn_dim, float* rnn_dst,
                           int64_t rnn_dst_stride, bool u8 = false) {
    a = NormArgs{x, ldx, y, ldy, raw_copy, ld_copy, rows, dim, make_obs_norm(mean, var, sub_mean, inv_scale, eps, clip),
                 rnn_src, rnn_dim, rnn_dst, rnn_dst_stride, rows};
    const uintptr_t in_mask = u8 ? 3u : 15u;   // uchar4 vs float4 accesses on the input / raw-copy side
    return (dim % 4 == 0) && (ldx % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) & in_mask) == 0) &&
           (!y || ((ldy % 4 == 0) && aligned16(y))) &&
           (!raw_copy || ((ld_copy % 4 == 0) && ((reinterpret_cast<uintptr_t>(raw_copy) & in_mask) == 0)));
}

static int launch_normalize(const void* x, int64_t ldx, float* y, int64_t ldy, void* raw_copy, int64_t ld_copy,
                            int64_t rows, int dim, const double* mean, const double* var, float sub_mean,
                            float inv_scale, float eps, float clip, cudaStream_t st, const float* rnn_src = nullptr,
                            int rnn_dim = 0, float* rnn_dst = nullptr, int64_t rnn_dst_stride = 0, bool u8 = false) {
    if (rows == 0 || dim == 0) return 0;
    NormArgs a;
    const bool vec = make_norm_args(a, x, ldx, y, ldy, raw_copy, ld_copy, rows, dim, mean, var, sub_mean, inv_scale, eps,
                                    clip, rnn_src, rnn_dim, rnn_dst, rnn_dst_stride, u8);
    const int64_t work = vec ? rows * (int64_t)(dim / 4) : rows * (int64_t)dim;
    int64_t blocks = ceil_div(work, 256);
    const int64_t cap = (int64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    const dim3 g((unsigned)blocks), b(256);
    if (u8) {
        if (vec) SFB_CUDA_OK(launch_pdl(normalize_kernel<true, true>, g, b, 0, st, a));
        else SFB_CUDA_OK(launch_pdl(normalize_kernel<false, true>, g, b, 0, st, a));
    } else {
        if (vec) SFB_CUDA_OK(launch_pdl(normalize_kernel<true, false>, g, b, 0, st, a));
        else SFB_CUDA_OK(launch_pdl(normalize_kernel<false, false>, g, b, 0, st, a));
    }
    SFB_LAUNCH_OK();
    return 0;
}

// ---- small strided helpers ----------------------------------------------------------------------------------------
__global__ void copy_rows_kernel(const float* __restrict__ src, int64_t ss, float* __restrict__ dst, int64_t ds,
                                 int64_t rows, int dim) {
    const int64_t total = rows * (int64_t)dim;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / dim;
        const int c = (int)(i - r * dim);
        dst[r * ds + c] = src[r * ss + c];
    }
}

// ---- row gather (shuffled minibatches: learner.py:498-526 `buffer[indices]`) --------------------------------------------
// dst[r, :] = src[idx[r], :] for rows of row_bytes bytes; WB = bytes moved per thread access (16 / 4 / 1)
template <int WB>
__global__ void __launch_bounds__(256) gather_rows_kernel(const uint8_t* __restrict__ src, int64_t row_bytes,
                                                          const int32_t* __restrict__ idx, int64_t rows,
                                                          uint8_t* __restrict__ dst) {
    const int64_t per_row = row_bytes / WB;
    const int64_t total = rows * per_row;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / per_row, c = (i - r * per_row) * WB;
        const uint8_t* s = src + (int64_t)idx[r] * row_bytes + c;
        uint8_t* d = dst + r * row_bytes + c;
        if (WB == 16) *reinterpret_cast<uint4*>(d) = *reinterpret_cast<const uint4*>(s);
        else if (WB == 4) *reinterpret_cast<uint32_t*>(d) = *reinterpret_cast<const uint32_t*>(s);
        else *d = *s;
    }
}

template <int WB>
__global__ void __launch_bounds__(256) copy_rows_bytes_kernel(const uint8_t* __restrict__ src, int64_t ss,
                                                              uint8_t* __restrict__ dst, int64_t ds, int64_t rows,
                                                              int64_t row_bytes) {
    const int64_t per_row = row_bytes / WB;
    const int64_t total = rows * per_row;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / per_row, c = (i - r * per_row) * WB;
        if (WB == 16) *reinterpret_cast<uint4*>(dst + r * ds + c) = *reinterpret_cast<const uint4*>(src + r * ss + c);
        else if (WB == 4) *reinterpret_cast<uint32_t*>(dst + r * ds + c) = *reinterpret_cast<const uint32_t*>(src + r * ss + c);
        else dst[r * ds + c] = src[r * ss + c];
    }
}

// ---- post env step -------------------------------------------------------------------------------------------------
struct PostArgs {
    const float* rew; const uint8_t* term; const uint8_t* trunc; int64_t n;
    EpisodeArgs e; int64_t* step_counter;
};

// All threads of the grid must call this (warp reductions inside); thread i < n handles env i.
__device__ __forceinline__ void post_step_body(const PostArgs& a) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (a.step_counter && i == 0) *a.step_counter += 1;
    double c = 0.0, s_ret = 0.0, s_len = 0.0, s_min = 0.0, s_max = 0.0;
    if (i < a.n) {
        const Episode ep = load_episode(a.e, i, true);
        Episode fin;
        if (post_step_env(a.e, i, i * a.e.stride, a.rew[i], a.term[i] != 0, a.trunc[i] != 0, ep, fin)) {
            c = 1.0; s_ret = fin.ret; s_len = fin.len; s_min = fin.mn; s_max = fin.mx;
        }
    }
    if (a.e.stats) {
        c = warp_sum(c);
        if (c > 0.0) {   // warp-uniform after the reduction
            s_ret = warp_sum(s_ret); s_len = warp_sum(s_len); s_min = warp_sum(s_min); s_max = warp_sum(s_max);
            if ((threadIdx.x & 31) == 0) {
                atomicAdd(a.e.stats + 0, c); atomicAdd(a.e.stats + 1, s_ret); atomicAdd(a.e.stats + 2, s_len);
                atomicAdd(a.e.stats + 3, s_min); atomicAdd(a.e.stats + 4, s_max);
            }
        }
    }
}

__global__ void __launch_bounds__(256) post_step_kernel(const PostArgs a) { post_step_body(a); }

// advance_rollouts part 2 of step t fused with generate_policy_request + normalisation of step t+1 (both consume the
// env's outputs; nothing sits between them on the stream): one launch instead of two per env step.
template <bool VEC4, bool U8>
__global__ void __launch_bounds__(256) post_pre_step_kernel(const PostArgs pa, const NormArgs na) {
    pdl_wait();
    pdl_trigger();
    post_step_body(pa);
    normalize_body<VEC4, U8>(na);
}

// ---- synthetic tape env ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) tape_env_kernel(const int32_t* __restrict__ actions,
                                                       const float* __restrict__ actions_f32, int act_dim, int64_t n,
                                                       int num_actions,
                                                       int64_t env_off, int term_period, int trunc_period,
                                                       int64_t* step_counter, int64_t step_host,
                                                       const float* __restrict__ tape, int64_t tape_len, int dim,
                                                       float* __restrict__ obs_out, float* __restrict__ rew,
                                                       uint8_t* __restrict__ term, uint8_t* __restrict__ trunc) {
    pdl_wait();
    pdl_trigger();
    const int64_t step = step_counter ? *step_counter : step_host;
    const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t nthreads = (int64_t)gridDim.x * blockDim.x;
    if (tid < n) {
        const int64_t env = env_off + tid;
        // Discrete: action / n ; Box: first action component clipped to [-1, 1] (same rules as the oracle's env)
        rew[tid] = actions_f32 ? clampf(actions_f32[tid * act_dim], -1.f, 1.f) : (float)actions[tid] / (float)num_actions;
        bool tm, tr;
        tape_done(step, env, term_period, trunc_period, tm, tr);
        term[tid] = tm; trunc[tid] = tr;
    }
    if (obs_out) {
        const float* src = tape + ((step + 1) % tape_len) * n * dim;
        const int64_t total = n * (int64_t)dim;
        if ((dim & 3) == 0) {
            const float4* s4 = reinterpret_cast<const float4*>(src);
            float4* d4 = reinterpret_cast<float4*>(obs_out);
            for (int64_t i = tid; i < (total >> 2); i += nthreads) d4[i] = s4[i];
        } else {
            for (int64_t i = tid; i < total; i += nthreads) obs_out[i] = src[i];
        }
    }
    if (step_counter) {
        __syncthreads();
        if (threadIdx.x == 0) advance_step_counters(step_counter, step + 1, nullptr, 0, gridDim.x);
    }
}

// ---- valids ----------------------------------------------------------------------------------------------------------
__global__ void valids_kernel(const int32_t* __restrict__ pid, const float* __restrict__ pver, int64_t n_traj, int T,
                              int32_t this_policy, float train_step_host, const int64_t* __restrict__ train_step_dev,
                              float max_lag, uint8_t* __restrict__ valids) {
    const float train_step = train_step_dev ? (float)train_step_dev[0] : train_step_host;
    const int64_t total = n_traj * (int64_t)(T + 1);
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / (T + 1);
        int t = (int)(i - r * (T + 1));
        if (t == T) t = T - 1;                                         // learner.py:955
        const int64_t j = r * T + t;
        const bool v = (pid[j] == this_policy) && (__fsub_rn(train_step, pver[j]) < max_lag);   // :950-953
        valids[i] = v ? 1 : 0;
    }
}

// ---- scalar running-mean-std apply (returns normaliser) ---------------------------------------------------------------
__global__ void rms_scalar_kernel(float* __restrict__ x, int64_t n, const double* __restrict__ mean,
                                  const double* __restrict__ var, float eps, float clip, int denorm) {
    const float mu = (float)mean[0];
    const float sigma = __fsqrt_rn(__fadd_rn((float)var[0], eps));
    const float inv = __fdiv_rn(1.0f, sigma);
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        float v = x[i];
        if (denorm) v = __fadd_rn(__fmul_rn(clampf(v, -clip, clip), sigma), mu);    // running_mean_std.py:107-108
        else v = clampf(__fmul_rn(__fsub_rn(v, mu), inv), -clip, clip);             // :109-110
        x[i] = v;
    }
}

static unsigned grid_for(int64_t work, int threads = 256, int waves = 8) {
    int64_t blocks = ceil_div(work, threads);
    const int64_t cap = (int64_t)sm_count() * waves;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    return (unsigned)blocks;
}

}  // namespace sfb

using namespace sfb;

extern "C" {

static int normalize_obs_impl(const void* x, bool u8, int64_t ldx, float* y, int64_t ldy, int64_t rows, int dim,
                              const double* mean, const double* var, float sub_mean, float inv_scale, float eps,
                              float clip, void* stream) {
    SFB_CHECK_ARG(x && y && rows >= 0 && dim > 0, "normalize_obs: bad arguments");
    SFB_CHECK_ARG((mean == nullptr) == (var == nullptr), "normalize_obs: mean/var must both be set or both NULL");
    return launch_normalize(x, ldx, y, ldy, nullptr, 0, rows, dim, mean, var, sub_mean, inv_scale, eps, clip,
                            (cudaStream_t)stream, nullptr, 0, nullptr, 0, u8);
}

int sfb200_normalize_obs(const float* x, int64_t ldx, float* y, int64_t ldy, int64_t rows, int dim, const double* mean,
                         const double* var, float sub_mean, float inv_scale, float eps, float clip, void* stream) {
    return normalize_obs_impl(x, false, ldx, y, ldy, rows, dim, mean, var, sub_mean, inv_scale, eps, clip, stream);
}

int sfb200_normalize_obs_u8(const uint8_t* x, int64_t ldx, float* y, int64_t ldy, int64_t rows, int dim,
                            const double* mean, const double* var, float sub_mean, float inv_scale, float eps,
                            float clip, void* stream) {
    return normalize_obs_impl(x, true, ldx, y, ldy, rows, dim, mean, var, sub_mean, inv_scale, eps, clip, stream);
}

static int sampler_pre_step_impl(const void* obs, bool u8, int64_t n_envs, int dim, void* traj_obs_t,
                                 int64_t traj_obs_stride, const float* rnn, int rnn_dim, float* traj_rnn_t,
                                 int64_t traj_rnn_stride, float* x_norm, const double* mean, const double* var,
                                 float sub_mean, float inv_scale, float eps, float clip, void* stream) {
    SFB_CHECK_ARG(obs && traj_obs_t && n_envs >= 0 && dim > 0, "sampler_pre_step: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    const bool with_rnn = rnn && traj_rnn_t && rnn_dim > 0;
    return launch_normalize(obs, dim, x_norm, dim, traj_obs_t, traj_obs_stride, n_envs, dim, mean, var, sub_mean,
                            inv_scale, eps, clip, st, with_rnn ? rnn : nullptr, rnn_dim, traj_rnn_t, traj_rnn_stride, u8);
}

int sfb200_sampler_pre_step(const float* obs, int64_t n_envs, int dim, float* traj_obs_t, int64_t traj_obs_stride,
                            const float* rnn, int rnn_dim, float* traj_rnn_t, int64_t traj_rnn_stride, float* x_norm,
                            const double* mean, const double* var, float sub_mean, float inv_scale, float eps,
                            float clip, void* stream) {
    return sampler_pre_step_impl(obs, false, n_envs, dim, traj_obs_t, traj_obs_stride, rnn, rnn_dim, traj_rnn_t,
                                 traj_rnn_stride, x_norm, mean, var, sub_mean, inv_scale, eps, clip, stream);
}

int sfb200_sampler_pre_step_u8(const uint8_t* obs, int64_t n_envs, int dim, uint8_t* traj_obs_t, int64_t traj_obs_stride,
                               const float* rnn, int rnn_dim, float* traj_rnn_t, int64_t traj_rnn_stride, float* x_norm,
                               const double* mean, const double* var, float sub_mean, float inv_scale, float eps,
                               float clip, void* stream) {
    return sampler_pre_step_impl(obs, true, n_envs, dim, traj_obs_t, traj_obs_stride, rnn, rnn_dim, traj_rnn_t,
                                 traj_rnn_stride, x_norm, mean, var, sub_mean, inv_scale, eps, clip, stream);
}

int sfb200_copy_rows_bytes(const void* src, int64_t src_stride_bytes, void* dst, int64_t dst_stride_bytes, int64_t rows,
                           int64_t row_bytes, void* stream) {
    SFB_CHECK_ARG(src && dst && rows >= 0 && row_bytes > 0, "copy_rows_bytes: bad arguments");
    if (rows == 0) return 0;
    const uintptr_t al = reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst) | (uintptr_t)row_bytes |
                         (uintptr_t)src_stride_bytes | (uintptr_t)dst_stride_bytes;
    const int wb = (al % 16 == 0) ? 16 : ((al % 4 == 0) ? 4 : 1);
    int64_t blocks = ceil_div(rows * (row_bytes / wb), 256);
    const int64_t cap = (int64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    const dim3 g((unsigned)blocks), b(256);
    cudaStream_t st = (cudaStream_t)stream;
    const uint8_t* s8 = (const uint8_t*)src;
    uint8_t* d8 = (uint8_t*)dst;
    if (wb == 16) copy_rows_bytes_kernel<16><<<g, b, 0, st>>>(s8, src_stride_bytes, d8, dst_stride_bytes, rows, row_bytes);
    else if (wb == 4) copy_rows_bytes_kernel<4><<<g, b, 0, st>>>(s8, src_stride_bytes, d8, dst_stride_bytes, rows, row_bytes);
    else copy_rows_bytes_kernel<1><<<g, b, 0, st>>>(s8, src_stride_bytes, d8, dst_stride_bytes, rows, row_bytes);
    SFB_LAUNCH_OK();
    return 0;
}

int sfb200_gather_rows(const void* src, int64_t row_bytes, const int32_t* idx, int64_t rows, void* dst, void* stream) {
    SFB_CHECK_ARG(src && idx && dst && row_bytes > 0 && rows >= 0, "gather_rows: bad arguments");
    if (rows == 0) return 0;
    const uintptr_t al = reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst) | (uintptr_t)row_bytes;
    const int wb = (al % 16 == 0) ? 16 : ((al % 4 == 0) ? 4 : 1);
    int64_t blocks = ceil_div(rows * (row_bytes / wb), 256);
    const int64_t cap = (int64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    const dim3 g((unsigned)blocks), b(256);
    cudaStream_t st = (cudaStream_t)stream;
    const uint8_t* s8 = (const uint8_t*)src;
    uint8_t* d8 = (uint8_t*)dst;
    if (wb == 16) gather_rows_kernel<16><<<g, b, 0, st>>>(s8, row_bytes, idx, rows, d8);
    else if (wb == 4) gather_rows_kernel<4><<<g, b, 0, st>>>(s8, row_bytes, idx, rows, d8);
    else gather_rows_kernel<1><<<g, b, 0, st>>>(s8, row_bytes, idx, rows, d8);
    SFB_LAUNCH_OK();
    return 0;
}

int sfb200_copy_rows(const float* src, int64_t src_stride, float* dst, int64_t dst_stride, int64_t rows, int dim,
                     void* stream) {
    SFB_CHECK_ARG(src && dst && rows >= 0 && dim > 0, "copy_rows: bad arguments");
    if (rows == 0) return 0;
    copy_rows_kernel<<<grid_for(rows * dim), 256, 0, (cudaStream_t)stream>>>(src, src_stride, dst, dst_stride, rows, dim);
    SFB_LAUNCH_OK();
    return 0;
}

static int make_post_args(PostArgs& a, const float* rew, const uint8_t* terminated, const uint8_t* truncated,
                          int64_t n_envs, float reward_scale, float reward_clip, int32_t policy_id, float* traj_rewards_t,
                          uint8_t* traj_dones_t, uint8_t* traj_time_outs_t, int32_t* traj_policy_id_t,
                          int64_t traj_stride, float* ep_return, int32_t* ep_len, float* ep_min_raw, float* ep_max_raw,
                          int32_t len_increment, double* stats, int64_t* step_counter, float* fin_return_t,
                          int32_t* fin_len_t) {
    SFB_CHECK_ARG(!fin_return_t == !fin_len_t, "sampler_post_step: fin_return_t and fin_len_t come together");
    SFB_CHECK_ARG(rew && terminated && truncated && traj_rewards_t && traj_dones_t && traj_time_outs_t &&
                      traj_policy_id_t, "sampler_post_step: NULL argument");
    SFB_CHECK_ARG(!ep_return || (ep_len && ep_min_raw && ep_max_raw), "sampler_post_step: episode arrays incomplete");
    a = PostArgs{rew, terminated, truncated, n_envs,
                 EpisodeArgs{reward_scale, reward_clip, policy_id, traj_rewards_t, traj_dones_t, traj_time_outs_t,
                             traj_policy_id_t, traj_stride, ep_return, ep_len, ep_min_raw, ep_max_raw, len_increment,
                             ep_return ? stats : nullptr, ep_return ? fin_return_t : nullptr, fin_len_t},
                 step_counter};
    return 0;
}

int sfb200_sampler_post_step(const float* rew, const uint8_t* terminated, const uint8_t* truncated, int64_t n_envs,
                             float reward_scale, float reward_clip, int32_t policy_id, float* traj_rewards_t,
                             uint8_t* traj_dones_t, uint8_t* traj_time_outs_t, int32_t* traj_policy_id_t,
                             int64_t traj_stride, float* ep_return, int32_t* ep_len, float* ep_min_raw,
                             float* ep_max_raw, int32_t len_increment, double* stats, int64_t* step_counter,
                             float* fin_return_t, int32_t* fin_len_t, void* stream) {
    PostArgs a;
    if (int rc = make_post_args(a, rew, terminated, truncated, n_envs, reward_scale, reward_clip, policy_id,
                                traj_rewards_t, traj_dones_t, traj_time_outs_t, traj_policy_id_t, traj_stride, ep_return,
                                ep_len, ep_min_raw, ep_max_raw, len_increment, stats, step_counter, fin_return_t,
                                fin_len_t))
        return rc;
    if (n_envs == 0) return 0;
    post_step_kernel<<<(unsigned)ceil_div(n_envs, 256), 256, 0, (cudaStream_t)stream>>>(a);
    SFB_LAUNCH_OK();
    return 0;
}

static int sampler_post_pre_step_impl(bool u8, const float* rew, const uint8_t* terminated, const uint8_t* truncated, int64_t n_envs,
                                 float reward_scale, float reward_clip, int32_t policy_id, float* traj_rewards_t,
                                 uint8_t* traj_dones_t, uint8_t* traj_time_outs_t, int32_t* traj_policy_id_t,
                                 int64_t traj_stride, float* ep_return, int32_t* ep_len, float* ep_min_raw,
                                 float* ep_max_raw, int32_t len_increment, double* stats, int64_t* step_counter,
                                 float* fin_return_t, int32_t* fin_len_t,
                                 const void* obs, int dim, void* traj_obs_next, int64_t traj_obs_stride,
                                 const float* rnn, int rnn_dim, float* traj_rnn_next, int64_t traj_rnn_stride,
                                 float* x_norm, const double* mean, const double* var, float sub_mean, float inv_scale,
                                 float eps, float clip, void* stream) {
    PostArgs pa;
    if (int rc = make_post_args(pa, rew, terminated, truncated, n_envs, reward_scale, reward_clip, policy_id,
                                traj_rewards_t, traj_dones_t, traj_time_outs_t, traj_policy_id_t, traj_stride, ep_return,
                                ep_len, ep_min_raw, ep_max_raw, len_increment, stats, step_counter, fin_return_t,
                                fin_len_t))
        return rc;
    SFB_CHECK_ARG(obs && traj_obs_next && dim > 0, "sampler_post_pre_step: bad arguments");
    SFB_CHECK_ARG((mean == nullptr) == (var == nullptr), "sampler_post_pre_step: mean/var must both be set or both NULL");
    if (n_envs == 0) return 0;
    const bool with_rnn = rnn && traj_rnn_next && rnn_dim > 0;
    NormArgs na;
    const bool vec = make_norm_args(na, obs, dim, x_norm, dim, traj_obs_next, traj_obs_stride, n_envs, dim, mean, var,
                                    sub_mean, inv_scale, eps, clip, with_rnn ? rnn : nullptr, rnn_dim, traj_rnn_next,
                                    traj_rnn_stride, u8);
    const int64_t work = vec ? n_envs * (int64_t)(dim / 4) : n_envs * (int64_t)dim;
    int64_t blocks = ceil_div(work, 256);
    const int64_t cap = (int64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < ceil_div(n_envs, 256)) blocks = ceil_div(n_envs, 256);   // every env needs its post-step thread
    cudaStream_t st = (cudaStream_t)stream;
    const dim3 g((unsigned)blocks), b(256);
    if (u8) {
        if (vec) SFB_CUDA_OK(launch_pdl(post_pre_step_kernel<true, true>, g, b, 0, st, pa, na));
        else SFB_CUDA_OK(launch_pdl(post_pre_step_kernel<false, true>, g, b, 0, st, pa, na));
    } else {
        if (vec) SFB_CUDA_OK(launch_pdl(post_pre_step_kernel<true, false>, g, b, 0, st, pa, na));
        else SFB_CUDA_OK(launch_pdl(post_pre_step_kernel<false, false>, g, b, 0, st, pa, na));
    }
    SFB_LAUNCH_OK();
    return 0;
}

#define SFB_POST_PRE_ARGS                                                                                                  \
    rew, terminated, truncated, n_envs, reward_scale, reward_clip, policy_id, traj_rewards_t, traj_dones_t,              \
        traj_time_outs_t, traj_policy_id_t, traj_stride, ep_return, ep_len, ep_min_raw, ep_max_raw, len_increment, stats, \
        step_counter, fin_return_t, fin_len_t, obs, dim, traj_obs_next, traj_obs_stride, rnn, rnn_dim, traj_rnn_next,     \
        traj_rnn_stride, x_norm, mean, var, sub_mean, inv_scale, eps, clip, stream

int sfb200_sampler_post_pre_step(const float* rew, const uint8_t* terminated, const uint8_t* truncated, int64_t n_envs,
                                 float reward_scale, float reward_clip, int32_t policy_id, float* traj_rewards_t,
                                 uint8_t* traj_dones_t, uint8_t* traj_time_outs_t, int32_t* traj_policy_id_t,
                                 int64_t traj_stride, float* ep_return, int32_t* ep_len, float* ep_min_raw,
                                 float* ep_max_raw, int32_t len_increment, double* stats, int64_t* step_counter,
                                 float* fin_return_t, int32_t* fin_len_t,
                                 const float* obs, int dim, float* traj_obs_next, int64_t traj_obs_stride,
                                 const float* rnn, int rnn_dim, float* traj_rnn_next, int64_t traj_rnn_stride,
                                 float* x_norm, const double* mean, const double* var, float sub_mean, float inv_scale,
                                 float eps, float clip, void* stream) {
    return sampler_post_pre_step_impl(false, SFB_POST_PRE_ARGS);
}

int sfb200_sampler_post_pre_step_u8(const float* rew, const uint8_t* terminated, const uint8_t* truncated, int64_t n_envs,
                                    float reward_scale, float reward_clip, int32_t policy_id, float* traj_rewards_t,
                                    uint8_t* traj_dones_t, uint8_t* traj_time_outs_t, int32_t* traj_policy_id_t,
                                    int64_t traj_stride, float* ep_return, int32_t* ep_len, float* ep_min_raw,
                                    float* ep_max_raw, int32_t len_increment, double* stats, int64_t* step_counter,
                                    float* fin_return_t, int32_t* fin_len_t,
                                    const uint8_t* obs, int dim, uint8_t* traj_obs_next, int64_t traj_obs_stride,
                                    const float* rnn, int rnn_dim, float* traj_rnn_next, int64_t traj_rnn_stride,
                                    float* x_norm, const double* mean, const double* var, float sub_mean,
                                    float inv_scale, float eps, float clip, void* stream) {
    return sampler_post_pre_step_impl(true, SFB_POST_PRE_ARGS);
}
#undef SFB_POST_PRE_ARGS

static int tape_env_step_impl(const int32_t* actions, const float* actions_f32, int act_dim, int64_t n_envs,
                              int num_actions, int64_t env_index_offset, int term_period, int trunc_period,
                              int64_t* step_counter, int64_t step_host, const float* tape, int64_t tape_len, int dim,
                              float* obs_out, float* rew, uint8_t* terminated, uint8_t* truncated, void* stream) {
    SFB_CHECK_ARG((actions || (actions_f32 && act_dim > 0)) && rew && terminated && truncated && n_envs > 0 && num_actions > 0 && term_period > 0 &&
                      trunc_period > 0, "tape_env_step: bad arguments");
    SFB_CHECK_ARG(!obs_out || (tape && tape_len > 0 && dim > 0), "tape_env_step: obs_out needs a tape");
    cudaStream_t st = (cudaStream_t)stream;
    int64_t work = n_envs;
    if (obs_out) work = n_envs * (int64_t)dim / 4 > work ? n_envs * (int64_t)dim / 4 : work;
    unsigned g = grid_for(work);
    if ((int64_t)g * 256 < n_envs) g = (unsigned)ceil_div(n_envs, 256);
    SFB_CUDA_OK(launch_pdl(tape_env_kernel, dim3(g), dim3(256), 0, st, actions, actions_f32, act_dim, n_envs, num_actions, env_index_offset,
                           term_period, trunc_period, step_counter, step_host, tape, tape_len, dim, obs_out,
                           rew, terminated, truncated));
    SFB_LAUNCH_OK();
    return 0;
}

int sfb200_tape_env_step(const int32_t* actions, int64_t n_envs, int num_actions, int64_t env_index_offset,
                         int term_period, int trunc_period, int64_t* step_counter, int64_t step_host, const float* tape,
                         int64_t tape_len, int dim, float* obs_out, float* rew, uint8_t* terminated,
                         uint8_t* truncated, void* stream) {
    return tape_env_step_impl(actions, nullptr, 0, n_envs, num_actions, env_index_offset, term_period, trunc_period,
                              step_counter, step_host, tape, tape_len, dim, obs_out, rew, terminated, truncated, stream);
}

int sfb200_tape_env_step_continuous(const float* actions_f32, int act_dim, int64_t n_envs, int64_t env_index_offset,
                                    int term_period, int trunc_period, int64_t* step_counter, int64_t step_host,
                                    const float* tape, int64_t tape_len, int dim, float* obs_out, float* rew,
                                    uint8_t* terminated, uint8_t* truncated, void* stream) {
    return tape_env_step_impl(nullptr, actions_f32, act_dim, n_envs, 1, env_index_offset, term_period, trunc_period,
                              step_counter, step_host, tape, tape_len, dim, obs_out, rew, terminated, truncated, stream);
}

static int compute_valids_impl(const int32_t* policy_id, const float* policy_version, int64_t n_traj, int T,
                               int32_t this_policy, float train_step, const int64_t* train_step_dev,
                               float max_policy_lag, uint8_t* valids, void* stream) {
    SFB_CHECK_ARG(policy_id && policy_version && valids && n_traj >= 0 && T > 0, "compute_valids: bad arguments");
    if (n_traj == 0) return 0;
    valids_kernel<<<grid_for(n_traj * (T + 1)), 256, 0, (cudaStream_t)stream>>>(policy_id, policy_version, n_traj, T,
                                                                                  this_policy, train_step, train_step_dev,
                                                                                  max_policy_lag, valids);
    SFB_LAUNCH_OK();
    return 0;
}

int sfb200_compute_valids(const int32_t* policy_id, const float* policy_version, int64_t n_traj, int T,
                          int32_t this_policy, float train_step, float max_policy_lag, uint8_t* valids, void* stream) {
    return compute_valids_impl(policy_id, policy_version, n_traj, T, this_policy, train_step, nullptr, max_policy_lag,
                               valids, stream);
}

int sfb200_compute_valids_dev(const int32_t* policy_id, const float* policy_version, int64_t n_traj, int T,
                              int32_t this_policy, const int64_t* train_step_dev, float max_policy_lag, uint8_t* valids,
                              void* stream) {
    SFB_CHECK_ARG(train_step_dev, "compute_valids_dev: the device train-step counter is required");
    return compute_valids_impl(policy_id, policy_version, n_traj, T, this_policy, 0.f, train_step_dev, max_policy_lag,
                               valids, stream);
}

int sfb200_rms_apply_scalar(float* x, int64_t n, const double* mean, const double* var, float eps, float clip,
                            int denormalize, void* stream) {
    SFB_CHECK_ARG(x && mean && var && n >= 0, "rms_apply_scalar: bad arguments");
    if (n == 0) return 0;
    rms_scalar_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(x, n, mean, var, eps, clip, denormalize);
    SFB_LAUNCH_OK();
    return 0;
}

}  // extern "C"
