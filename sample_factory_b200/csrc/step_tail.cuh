// The rules of a sampler step after the policy heads, written once for the per-stage kernels (elementwise.cu), the fused
// step tail (heads.cu, sampler_tail_tape_kernel) and the persistent rollout (rollout_fused.cu): the observation
// normaliser, the synthetic tape env's done rule, the post step of one env and the ticket that advances the step
// counters.  Lane layouts, and how each kernel adds up the episode statistics, stay with the kernels.
#pragma once
#include "common.cuh"

namespace sfb {

// ---- observation normaliser (normalize.py:40-67, running_mean_std.py:96-110) ----------------------------------------
// y = clamp(((x - sub) * inv_scale - mu) * (1/sqrt(var+eps)), +-clip), each op rounded separately (IEEE, no FMA
// contraction) exactly like the reference's chain of in-place ATen ops.
__device__ __forceinline__ float norm_one(float x, float sub, float inv_scale, bool do_sub, bool do_scale, bool do_rms,
                                          float mu, float inv_sigma, float clip) {
    if (do_sub) x = __fsub_rn(x, sub);
    if (do_scale) x = __fmul_rn(x, inv_scale);
    if (do_rms) {
        x = __fmul_rn(__fsub_rn(x, mu), inv_sigma);
        x = clampf(x, -clip, clip);
    }
    return x;
}

__device__ __forceinline__ void col_stats(const double* mean, const double* var, int c, float eps, float& mu,
                                          float& inv_sigma) {
    mu = (float)mean[c];
    float sigma = __fsqrt_rn(__fadd_rn((float)var[c], eps));
    inv_sigma = __fdiv_rn(1.0f, sigma);
}

struct ObsNorm {
    const double* mean; const double* var;   // running statistics per column, or NULL
    float sub, inv_scale; int do_sub, do_scale; float eps, clip;

    // column c of an observation, mu / 1 / sigma from the block's cached statistics (fill_col_stats) when do_rms
    __device__ __forceinline__ float apply(float x, bool do_rms, const float* cstat, int dim, int c) const {
        return norm_one(x, sub, inv_scale, do_sub, do_scale, do_rms, do_rms ? cstat[c] : 0.f, do_rms ? cstat[dim + c] : 1.f,
                        clip);
    }
};

// subtract / scale only where they change a value (the reference skips them at their defaults)
static inline ObsNorm make_obs_norm(const double* mean, const double* var, float sub_mean, float inv_scale, float eps,
                                    float clip) {
    return ObsNorm{mean, var, sub_mean, inv_scale, fabsf(sub_mean) > 1e-8f, fabsf(inv_scale - 1.0f) > 1e-8f, eps, clip};
}

// cstat[2][dim] <- mu, 1 / sigma of every column, by the whole block (the caller synchronises before reading them)
__device__ __forceinline__ void fill_col_stats(const ObsNorm& n, int dim, float* cstat) {
    for (int c = threadIdx.x; c < dim; c += blockDim.x) col_stats(n.mean, n.var, c, n.eps, cstat[c], cstat[dim + c]);
}

// ---- synthetic tape env (envs.TapeVecEnv; the oracle's env has the same rules) --------------------------------------
__device__ __forceinline__ void tape_done(int64_t step, int64_t env, int term_period, int trunc_period, bool& tm,
                                          bool& tr) {
    tm = ((step * 7 + env * 13) % term_period) == 0;
    tr = (((step + env) % trunc_period) == 0) && !tm;
}

// ---- post step: advance_rollouts part 2 (batched_sampling.py:319-357) ------------------------------------------------
struct EpisodeArgs {
    float reward_scale, reward_clip; int32_t policy_id;
    float* t_rew; uint8_t* t_done; uint8_t* t_to; int32_t* t_pid; int64_t stride;   // trajectory slot, row stride
    float* ep_ret; int32_t* ep_len; float* ep_min; float* ep_max; int32_t len_inc;   // episode accumulators, or NULL
    double* stats;                                   // [5]: finished episodes, sums of return, length, min, max
    float* fin_ret; int32_t* fin_len;                // per slot: return / length of an episode that ended there, or NULL
};

// an env's episode accumulators: running (loaded), or those of an episode that just ended
struct Episode { float ret; int32_t len; float mn, mx; };

__device__ __forceinline__ Episode load_episode(const EpisodeArgs& e, int64_t env, bool active) {
    Episode ep{0.f, 0, 0.f, 0.f};
    if (active && e.ep_ret) ep = Episode{e.ep_ret[env], e.ep_len[env], e.ep_min[env], e.ep_max[env]};
    return ep;
}

// The post step of env `env` whose trajectory slot is `slot`: reward scale and clip, done / time-out flags, policy id,
// and the episode accounting (_process_env_step :215-287, on the RAW reward: :336 passes rewards_cpu) from the
// accumulators `ep` the caller loaded.  Returns true when an episode ended; `fin` then holds its summary.
__device__ __forceinline__ bool post_step_env(const EpisodeArgs& e, int64_t env, int64_t slot, float r_raw, bool tm,
                                              bool tr, Episode ep, Episode& fin) {
    const bool done = tm || tr;                                   // batched_sampling.py:317
    float r = __fmul_rn(r_raw, e.reward_scale);                     // :209
    r = clampf(r, -e.reward_clip, e.reward_clip);                   // :210
    e.t_rew[slot] = r;
    e.t_done[slot] = done ? 1 : 0;
    e.t_to[slot] = tr ? 1 : 0;                                      // :328
    e.t_pid[slot] = e.policy_id;
    if (!e.ep_ret) return false;
    fin = Episode{ep.ret + r_raw, ep.len + e.len_inc, fminf(ep.mn, r_raw), fmaxf(ep.mx, r_raw)};
    if (e.fin_ret) {
        e.fin_ret[slot] = done ? fin.ret : __int_as_float(0x7fc00000);
        e.fin_len[slot] = done ? fin.len : -1;
    }
    const Episode next = done ? Episode{0.f, 0, INFINITY, -INFINITY} : fin;
    e.ep_ret[env] = next.ret; e.ep_len[env] = next.len; e.ep_min[env] = next.mn; e.ep_max[env] = next.mx;
    return done;
}

// ---- step counters ---------------------------------------------------------------------------------------------------
// Run by one thread of every block after a block barrier that follows the block's reads of the counters: the last of the
// `blocks` blocks to take a ticket (env_step[1]) sets env_step[0] = env_next and, if sampler_step is set,
// *sampler_step = sampler_next.
__device__ __forceinline__ void advance_step_counters(int64_t* env_step, int64_t env_next, int64_t* sampler_step,
                                                      int64_t sampler_next, unsigned blocks) {
    __threadfence();
    unsigned long long* ticket = reinterpret_cast<unsigned long long*>(env_step + 1);
    if (atomicAdd(ticket, 1ull) == (unsigned long long)blocks - 1ull) {
        *ticket = 0ull;
        env_step[0] = env_next;
        if (sampler_step) *sampler_step = sampler_next;
    }
}

}  // namespace sfb
