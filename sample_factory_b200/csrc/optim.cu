// Global grad-norm clip + Adam on flat parameter / gradient / moment buffers (learner.py:782-797; torch
// clip_grad_norm_ and torch.optim.Adam semantics, SURVEY App.A-12).  HBM-bound: 28 B/param (+4 B for the norm pass).
#include <math.h>

#include "common.cuh"
#include "adam_core.cuh"

namespace sfb {

constexpr int kNormBlocks = 480;   // partial slots in the 4 KiB workspace (doubles)

__global__ void __launch_bounds__(256) sumsq_kernel(const float* __restrict__ g, int64_t n, double* __restrict__ part) {
    __shared__ double sm[8];
    double s = 0.0;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const double v = (double)g[i];
        s += v * v;
    }
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 32) {
        double t = threadIdx.x < 8 ? sm[threadIdx.x] : 0.0;
        t = warp_sum(t);
        if (threadIdx.x == 0) part[blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(256) clip_adam_kernel(const AdamArgs a, const double* __restrict__ part, int nparts) {
    clip_adam_body(a, part, nparts);
}


// ---- LAMB (algo/utils/optimizers.py:13-175, list-params path: bias correction on, weight decay, per-tensor trust ratio,
// no look-ahead).  The flat buffer is walked per tensor (grid.y = tensor index) because the trust ratio needs the norms
// of each parameter tensor and of its update:
//   stage 1: m, v <- moments(g * clip_coef);  u = m_hat / (sqrt(v_hat) + eps) + wd * p  (written over g);
//            per-(tensor, chunk) partial sums of p^2 and u^2
//   stage 2: one warp per tensor: trust = clamp(min(|p|, 10) / |u|, min_trust, 1/min_trust)  (1 if either norm is 0)
//   stage 3: p -= lr * trust * u
constexpr int kLambChunk = 4096;   // elements per block

__global__ void __launch_bounds__(256) lamb_stage1_kernel(const float* __restrict__ p, float* __restrict__ g,
                                                          float* __restrict__ m, float* __restrict__ v,
                                                          const int64_t* __restrict__ seg_off,
                                                          const int64_t* __restrict__ seg_n, float b1, float omb1, float b2,
                                                          float omb2, float inv_bc1, float inv_bc2_sqrt,
                                                          const int64_t* __restrict__ steps_done_dev, double beta1,
                                                          double beta2, float eps, float wd,
                                                          float max_norm, const double* __restrict__ gpart, int n_gpart,
                                                          float* __restrict__ grad_norm_out, double* __restrict__ part,
                                                          int chunks_max) {
    __shared__ double sm[2][8];
    __shared__ float s_coef, s_inv_bc1, s_inv_bc2_sqrt;
    if (threadIdx.x < 32) {
        double t = 0.0;
        for (int k = threadIdx.x; k < n_gpart; k += 32) t += gpart[k];
        t = warp_sum(t);
        if (threadIdx.x == 0) {
            const float total = (float)sqrt(t);
            s_coef = max_norm > 0.f ? fminf(__fdiv_rn(max_norm, total + 1e-6f), 1.0f) : 1.f;
            if (grad_norm_out && blockIdx.x == 0 && blockIdx.y == 0) grad_norm_out[0] = total;
            if (steps_done_dev) {
                // the step count lives on the device (a CUDA-graph-replayed learner): the host expression of
                // sfb200_clip_lamb_step, in double and in the same order
                const double step = (double)(steps_done_dev[0] + 1);
                const double bc1 = __dsub_rn(1.0, pow(beta1, step)), bc2 = __dsub_rn(1.0, pow(beta2, step));
                inv_bc1 = (float)__ddiv_rn(1.0, bc1);
                inv_bc2_sqrt = (float)__ddiv_rn(1.0, __dsqrt_rn(bc2));
            }
            s_inv_bc1 = inv_bc1;
            s_inv_bc2_sqrt = inv_bc2_sqrt;
        }
    }
    __syncthreads();
    const float coef = s_coef;
    inv_bc1 = s_inv_bc1;
    inv_bc2_sqrt = s_inv_bc2_sqrt;
    const int t_idx = blockIdx.y;
    const int64_t off = seg_off[t_idx], n = seg_n[t_idx];
    const int64_t c0 = (int64_t)blockIdx.x * kLambChunk;
    double sp = 0.0, su = 0.0;
    for (int64_t i = c0 + threadIdx.x; i < n && i < c0 + kLambChunk; i += 256) {
        const int64_t j = off + i;
        const float gi = g[j] * coef;
        const float mi = m[j] * b1 + omb1 * gi;               // exp_avg.mul_(beta1).add_(grad, alpha=1-beta1)
        const float vi = v[j] * b2 + (omb2 * gi) * gi;        // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1-beta2)
        m[j] = mi;
        v[j] = vi;
        const float pj = p[j];
        float u = __fdiv_rn(mi * inv_bc1, __fsqrt_rn(vi) * inv_bc2_sqrt + eps);
        u = u + wd * pj;                                       // adam_step.add_(p, alpha=weight_decay)
        g[j] = u;
        sp += (double)pj * pj;
        su += (double)u * u;
    }
    sp = warp_sum(sp);
    su = warp_sum(su);
    if ((threadIdx.x & 31) == 0) { sm[0][threadIdx.x >> 5] = sp; sm[1][threadIdx.x >> 5] = su; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0.0, b = 0.0;
        for (int w = 0; w < 8; ++w) { a += sm[0][w]; b += sm[1][w]; }
        part[((int64_t)t_idx * chunks_max + blockIdx.x) * 2 + 0] = a;
        part[((int64_t)t_idx * chunks_max + blockIdx.x) * 2 + 1] = b;
    }
}

__global__ void lamb_stage2_kernel(const double* __restrict__ part, const int64_t* __restrict__ seg_n, int chunks_max,
                                   float min_trust, float* __restrict__ trust) {
    const int t_idx = blockIdx.x;
    const int64_t chunks = (seg_n[t_idx] + kLambChunk - 1) / kLambChunk;
    double a = 0.0, b = 0.0;
    for (int64_t c = threadIdx.x; c < chunks; c += 32) {
        a += part[((int64_t)t_idx * chunks_max + c) * 2 + 0];
        b += part[((int64_t)t_idx * chunks_max + c) * 2 + 1];
    }
    a = warp_sum(a);
    b = warp_sum(b);
    if (threadIdx.x == 0) {
        const float wn = (float)sqrt(a), sn = (float)sqrt(b);   // torch.norm(...).item()
        float tr = 1.f;
        if (wn != 0.f && sn != 0.f && min_trust != 1.0f) {
            tr = fminf(wn, 10.0f) / sn;
            tr = fminf(fmaxf(tr, min_trust), 1.0f / min_trust);
        }
        trust[t_idx] = tr;
    }
}

__global__ void __launch_bounds__(256) lamb_stage3_kernel(float* __restrict__ p, const float* __restrict__ u,
                                                          const int64_t* __restrict__ seg_off,
                                                          const int64_t* __restrict__ seg_n,
                                                          const float* __restrict__ trust, double lr,
                                                          const double* __restrict__ lr_dev,
                                                          const double* __restrict__ lr_num,
                                                          const double* __restrict__ lr_den) {
    const int t_idx = blockIdx.y;
    const int64_t off = seg_off[t_idx], n = seg_n[t_idx];
    double lr_eff = lr_dev ? lr_dev[0] : lr;
    if (lr_num && lr_den) lr_eff = lr_eff * lr_num[0] / lr_den[0];      // learner.py:788-794
    const float step = (float)lr_eff * trust[t_idx];
    const int64_t c0 = (int64_t)blockIdx.x * kLambChunk;
    for (int64_t i = c0 + threadIdx.x; i < n && i < c0 + kLambChunk; i += 256) {
        const int64_t j = off + i;
        p[j] = p[j] - step * u[j];                                      // p.add_(adam_step, alpha=-lr * trust_ratio)
    }
}

// Learning-rate rules between minibatches (learner.py KlAdaptiveScheduler / LinearDecayScheduler) for a learner replayed
// as CUDA graphs.  One thread; every operation is an explicitly rounded double operation so nothing is contracted and
// the result is bit-identical to the host's Python float arithmetic.  Python's max(a, b) / min(a, b) return `a` unless
// `b` is strictly larger / smaller: the selects below keep that order.
__global__ void lr_schedule_kernel(int rule, double* __restrict__ lr_dev, const double* __restrict__ kl_dev,
                                   double thr, double min_lr, double max_lr, int64_t* __restrict__ step_dev,
                                   int64_t num_updates, double lr0) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    double lr = lr_dev[0];
    if (rule == 0) {
        const double kl = kl_dev[0];
        if (kl > __dmul_rn(2.0, thr)) {
            const double t = __ddiv_rn(lr, 1.5);
            lr = min_lr > t ? min_lr : t;
        }
        if (kl < __dmul_rn(0.5, thr)) {
            const double t = __dmul_rn(lr, 1.5);
            lr = max_lr < t ? max_lr : t;
        }
    } else {
        const int64_t step = step_dev[0] + 1;
        step_dev[0] = step;
        lr = step >= num_updates ? 0.0
                                 : __dadd_rn(lr0, __dmul_rn(__dsub_rn(0.0, lr0), __ddiv_rn((double)step, (double)num_updates)));
    }
    lr_dev[0] = lr;
}

}  // namespace sfb

using namespace sfb;

extern "C" {

static int clip_adam_impl(float* p, float* g, float* m, float* v, int64_t n, int64_t step, const int64_t* step_dev,
                          double lr, const double* lr_dev, double beta1, double beta2, double eps, double max_grad_norm,
                          const double* lr_scale_num, const double* lr_scale_den, float* grad_norm_out, void* workspace,
                          void* stream) {
    SFB_CHECK_ARG(p && g && m && v && workspace && n > 0 && (step >= 1 || step_dev), "clip_adam_step: bad arguments");
    SFB_CHECK_ARG((lr_scale_num == nullptr) == (lr_scale_den == nullptr), "clip_adam_step: lr_scale num/den mismatch");
    cudaStream_t st = (cudaStream_t)stream;
    double* part = (double*)workspace;
    int64_t nb = ceil_div(n, 256 * 4);
    if (nb > kNormBlocks) nb = kNormBlocks;
    sumsq_kernel<<<(unsigned)nb, 256, 0, st>>>(g, n, part);
    SFB_LAUNCH_OK();
    int64_t blocks = ceil_div(n, 256 * 2);
    const int64_t cap = (int64_t)sm_count() * 4;
    if (blocks > cap) blocks = cap;
    const AdamArgs aa = make_adam_args(p, g, m, v, n, lr, lr_dev, beta1, beta2, step, step_dev, eps, max_grad_norm,
                                       lr_scale_num, lr_scale_den, grad_norm_out);
    clip_adam_kernel<<<(unsigned)blocks, 256, 0, st>>>(aa, part, (int)nb);
    SFB_LAUNCH_OK();
    return 0;
}

int sfb200_clip_adam_step(float* p, float* g, float* m, float* v, int64_t n, int64_t step, double lr, double beta1,
                          double beta2, double eps, double max_grad_norm, const double* lr_scale_num,
                          const double* lr_scale_den, float* grad_norm_out, void* workspace, void* stream) {
    return clip_adam_impl(p, g, m, v, n, step, nullptr, lr, nullptr, beta1, beta2, eps, max_grad_norm, lr_scale_num,
                          lr_scale_den, grad_norm_out, workspace, stream);
}

int sfb200_clip_adam_step_dev(float* p, float* g, float* m, float* v, int64_t n, const int64_t* steps_done_dev,
                              const double* lr_dev, double beta1, double beta2, double eps, double max_grad_norm,
                              const double* lr_scale_num, const double* lr_scale_den, float* grad_norm_out,
                              void* workspace, void* stream) {
    SFB_CHECK_ARG(steps_done_dev && lr_dev, "clip_adam_step_dev: the device step counter and learning rate are required");
    return clip_adam_impl(p, g, m, v, n, 0, steps_done_dev, 0.0, lr_dev, beta1, beta2, eps, max_grad_norm, lr_scale_num,
                          lr_scale_den, grad_norm_out, workspace, stream);
}

__global__ void advance_counters_kernel(int64_t* a, int64_t* b) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        if (a) a[0] += 1;
        if (b) b[0] += 1;
    }
}

int sfb200_advance_counters(int64_t* a, int64_t* b, void* stream) {
    advance_counters_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(a, b);
    SFB_LAUNCH_OK();
    return 0;
}

int64_t sfb200_lamb_workspace_bytes(int num_tensors, int64_t max_numel) {
    const int64_t chunks = ceil_div(max_numel > 0 ? max_numel : 1, kLambChunk);
    return (int64_t)kNormBlocks * 8 + (int64_t)num_tensors * chunks * 2 * 8 + (int64_t)num_tensors * 4 + 64;
}

static int clip_lamb_impl(float* p, float* g, float* m, float* v, int64_t n, const int64_t* seg_offsets,
                          const int64_t* seg_numel, int num_tensors, int64_t max_numel, int64_t step,
                          const int64_t* step_dev, double lr, const double* lr_dev, double beta1, double beta2, double eps,
                          double weight_decay, double min_trust, double max_grad_norm, const double* lr_scale_num,
                          const double* lr_scale_den, float* grad_norm_out, void* workspace, void* stream) {
    SFB_CHECK_ARG(p && g && m && v && seg_offsets && seg_numel && workspace && n > 0 && num_tensors > 0 && max_numel > 0 &&
                      (step >= 1 || step_dev), "clip_lamb_step: bad arguments");
    SFB_CHECK_ARG((lr_scale_num == nullptr) == (lr_scale_den == nullptr), "clip_lamb_step: lr_scale num/den mismatch");
    SFB_CHECK_ARG(min_trust >= 0.0 && min_trust <= 1.0, "clip_lamb_step: min_trust must be in [0, 1]");
    cudaStream_t st = (cudaStream_t)stream;
    double* gpart = (double*)workspace;
    const int chunks = (int)ceil_div(max_numel, kLambChunk);
    double* part = gpart + kNormBlocks;
    float* trust = (float*)(part + (int64_t)num_tensors * chunks * 2);
    int64_t nb = ceil_div(n, 256 * 4);
    if (nb > kNormBlocks) nb = kNormBlocks;
    sumsq_kernel<<<(unsigned)nb, 256, 0, st>>>(g, n, gpart);     // global grad norm over the whole flat buffer (padding is 0)
    SFB_LAUNCH_OK();
    float inv_bc1 = 0.f, inv_bc2_sqrt = 0.f;     // (formed in the kernel from *step_dev when the step lives on the device)
    if (!step_dev) {
        const double bc1 = 1.0 - pow(beta1, (double)step);
        const double bc2 = 1.0 - pow(beta2, (double)step);
        inv_bc1 = (float)(1.0 / bc1);
        inv_bc2_sqrt = (float)(1.0 / sqrt(bc2));
    }
    dim3 grid((unsigned)chunks, (unsigned)num_tensors);
    lamb_stage1_kernel<<<grid, 256, 0, st>>>(p, g, m, v, seg_offsets, seg_numel, (float)beta1, (float)(1.0 - beta1), (float)beta2,
                                             (float)(1.0 - beta2), inv_bc1, inv_bc2_sqrt, step_dev, beta1, beta2, (float)eps,
                                             (float)weight_decay, (float)max_grad_norm, gpart, (int)nb, grad_norm_out, part,
                                             chunks);
    SFB_LAUNCH_OK();
    lamb_stage2_kernel<<<(unsigned)num_tensors, 32, 0, st>>>(part, seg_numel, chunks, (float)min_trust, trust);
    SFB_LAUNCH_OK();
    lamb_stage3_kernel<<<grid, 256, 0, st>>>(p, g, seg_offsets, seg_numel, trust, lr, lr_dev, lr_scale_num, lr_scale_den);
    SFB_LAUNCH_OK();
    return 0;
}

int sfb200_clip_lamb_step(float* p, float* g, float* m, float* v, int64_t n, const int64_t* seg_offsets,
                          const int64_t* seg_numel, int num_tensors, int64_t max_numel, int64_t step, double lr,
                          double beta1, double beta2, double eps, double weight_decay, double min_trust,
                          double max_grad_norm, const double* lr_scale_num, const double* lr_scale_den,
                          float* grad_norm_out, void* workspace, void* stream) {
    return clip_lamb_impl(p, g, m, v, n, seg_offsets, seg_numel, num_tensors, max_numel, step, nullptr, lr, nullptr, beta1,
                          beta2, eps, weight_decay, min_trust, max_grad_norm, lr_scale_num, lr_scale_den, grad_norm_out,
                          workspace, stream);
}

int sfb200_clip_lamb_step_dev(float* p, float* g, float* m, float* v, int64_t n, const int64_t* seg_offsets,
                              const int64_t* seg_numel, int num_tensors, int64_t max_numel, const int64_t* steps_done_dev,
                              const double* lr_dev, double beta1, double beta2, double eps, double weight_decay,
                              double min_trust, double max_grad_norm, const double* lr_scale_num,
                              const double* lr_scale_den, float* grad_norm_out, void* workspace, void* stream) {
    SFB_CHECK_ARG(steps_done_dev && lr_dev, "clip_lamb_step_dev: the device step counter and learning rate are required");
    return clip_lamb_impl(p, g, m, v, n, seg_offsets, seg_numel, num_tensors, max_numel, 0, steps_done_dev, 0.0, lr_dev,
                          beta1, beta2, eps, weight_decay, min_trust, max_grad_norm, lr_scale_num, lr_scale_den,
                          grad_norm_out, workspace, stream);
}

int sfb200_lr_schedule_step(int rule, double* lr_dev, const double* kl_dev, double kl_threshold, double min_lr,
                            double max_lr, int64_t* step_dev, int64_t num_updates, double lr0, void* stream) {
    SFB_CHECK_ARG(lr_dev && (rule == 0 || rule == 1) && (rule != 0 || kl_dev) && (rule != 1 || step_dev),
                  "lr_schedule_step: bad arguments");
    lr_schedule_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(rule, lr_dev, kl_dev, kl_threshold, min_lr, max_lr, step_dev,
                                                          num_updates, lr0);
    SFB_LAUNCH_OK();
    return 0;
}

}  // extern "C"
