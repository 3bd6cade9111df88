// clip_grad_norm_ + torch.optim.Adam on flat buffers (learner.py:782-797; SURVEY App.A-12), shared by the single-GPU
// launch (optim.cu) and the data-parallel kernel that fuses the NVLink gradient all-reduce in front of it (comm.cu).
#pragma once
#include <math.h>

#include "common.cuh"

namespace sfb {

struct AdamArgs {
    float* p; const float* g; float* m; float* v; int64_t n;
    double lr; const double* lr_dev; double beta1, beta2; int64_t step_host; const int64_t* step_dev;
    float omb1, beta2f, omb2, eps, max_norm;
    const double* lr_num; const double* lr_den;
    float* grad_norm_out;
    uint16_t* p_hi16; int64_t lo16_offset;      // registered fp16 twins of the parameters (api.cu), or NULL
};

static inline AdamArgs make_adam_args(float* p, const float* g, float* m, float* v, int64_t n, double lr, const double* lr_dev,
                                      double beta1, double beta2, int64_t step, const int64_t* step_dev, double eps,
                                      double max_grad_norm, const double* lr_scale_num, const double* lr_scale_den,
                                      float* grad_norm_out) {
    AdamArgs a{p, g, m, v, n, lr, lr_dev, beta1, beta2, step, step_dev,
               (float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2), (float)eps, (float)max_grad_norm,
               lr_scale_num, lr_scale_den, grad_norm_out, nullptr, 0};
    a.p_hi16 = f16_twin_lookup_mut(p, n, &a.lo16_offset);
    return a;
}

// Called by every thread of a 256-thread block (grid-stride over the parameters).  `part[0..nparts)` are the partial
// sums of squares of the gradient; every block reduces them itself, in the same order -> identical clip coefficient.
__device__ __forceinline__ void clip_adam_body(const AdamArgs& a, const double* __restrict__ part, int nparts) {
    __shared__ float s_coef;
    __shared__ float s_step;
    __shared__ float s_bc2;
    if (threadIdx.x < 32) {
        double t = 0.0;
        for (int k = threadIdx.x; k < nparts; k += 32) t += part[k];
        t = warp_sum(t);
        if (threadIdx.x == 0) {
            const float total = (float)sqrt(t);
            float coef = 1.f;
            if (a.max_norm > 0.f) coef = fminf(__fdiv_rn(a.max_norm, total + 1e-6f), 1.0f);   // clip_grad.py
            s_coef = coef;
            // step count and learning rate may live on the device (a CUDA-graph-captured learner replays this launch)
            const double step = (double)(a.step_dev ? a.step_dev[0] + 1 : a.step_host);
            const double bc1 = 1.0 - pow(a.beta1, step), bc2 = 1.0 - pow(a.beta2, step);
            double lr_eff = a.lr_dev ? a.lr_dev[0] : a.lr;
            if (a.lr_num && a.lr_den) lr_eff = lr_eff * a.lr_num[0] / a.lr_den[0];          // learner.py:788-794
            s_step = (float)(lr_eff / bc1);                                                 // adam.py step_size
            s_bc2 = (float)sqrt(bc2);
            if (a.grad_norm_out && blockIdx.x == 0) a.grad_norm_out[0] = total;
        }
    }
    __syncthreads();
    const float coef = s_coef, step_size = s_step, bc2_sqrt = s_bc2;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * blockDim.x) {
        const float gi = a.g[i] * coef;
        float mi = a.m[i], vi = a.v[i];
        mi = mi + a.omb1 * (gi - mi);                      // exp_avg.lerp_(grad, 1-beta1)
        vi = vi * a.beta2f + (a.omb2 * gi) * gi;           // exp_avg_sq.mul_(b2).addcmul_(g, g, value=1-b2)
        const float denom = __fdiv_rn(__fsqrt_rn(vi), bc2_sqrt) + a.eps;
        const float pn = a.p[i] - step_size * __fdiv_rn(mi, denom);   // param.addcdiv_(exp_avg, denom, value=-step_size)
        a.p[i] = pn;
        if (a.p_hi16) f16_split1(pn * (float)(1 << kF16WShift), a.p_hi16[i], a.p_hi16[i + a.lo16_offset]);   // fp16 twins stay current
        a.m[i] = mi;
        a.v[i] = vi;
    }
}

}  // namespace sfb
