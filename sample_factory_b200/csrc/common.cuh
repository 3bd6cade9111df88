// Shared helpers for libsfb200 kernels (sm_100a).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/sfb200.h"

namespace sfb {

void set_error(const char* fmt, ...);
void count_launch();   // every kernel launch of this library is counted (sfb200_launch_count)

#define SFB_CHECK_ARG(cond, ...)            \
    do {                                    \
        if (!(cond)) {                      \
            sfb::set_error(__VA_ARGS__);    \
            return 1;                       \
        }                                   \
    } while (0)

#define SFB_CUDA_OK(expr)                                                                   \
    do {                                                                                    \
        cudaError_t _e = (expr);                                                            \
        if (_e != cudaSuccess) {                                                            \
            sfb::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return 2;                                                                       \
        }                                                                                   \
    } while (0)

#define SFB_LAUNCH_OK()                                                                     \
    do {                                                                                    \
        sfb::count_launch();                                                                \
        cudaError_t _e = cudaGetLastError();                                                \
        if (_e != cudaSuccess) {                                                            \
            sfb::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, __LINE__); \
            return 3;                                                                       \
        }                                                                                   \
    } while (0)

int sm_count();
// Registered fp16 twins of weight buffers (api.cu): [hi16[n] | lo16[n]] with hi = fp16(w * 2^kF16WShift),
// lo = fp16((w * 2^kF16WShift - hi) * 2^kF16LoShift) -- the weight operand of the fp16-split GEMM (gemm_tc.cu, "F16" kernel).
struct F16Twin { const uint16_t* hi; const uint16_t* lo; };
F16Twin f16_twin_lookup(const float* p, int64_t count);
uint16_t* f16_twin_lookup_mut(float* p, int64_t count, int64_t* lo_offset);
// the same twins stored TRANSPOSED ([K][N] for a weight matrix W[N][K]): the weight operand of dX = dz . W, K-major
F16Twin f16_twinT_lookup(const float* W, int N, int K);
int f16_twins_check(const float* W, F16Twin tw, int N, int K, bool transposed, cudaStream_t st);
bool f16_check_enabled();   // SFB200_CHECK_F16=1 (gemm_tc.cu)
// device float holding an upper bound of |x| over an activation buffer that contains [p, p + bytes), else NULL
const float* operand_bound_lookup(const void* p, int64_t bytes);
bool pdl_enabled();   // SFB200_PDL=0 turns programmatic dependent launch off (api.cu)

// Programmatic dependent launch: kernels launched through launch_pdl() may be made resident while their predecessor on
// the stream is still running; every such kernel calls pdl_wait() before it touches global memory (the wait returns
// once the predecessor grid has completed and its writes are visible) and pdl_trigger() to let ITS successor start
// launching.  Inside the sampler's per-step kernel chain this hides the launch latency of each dependent kernel.
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                     Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// ---------------------------------------------------------------- device helpers
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// activation applied to a pre-activation value
__device__ __forceinline__ float act_fwd(float z, int act) {
    switch (act) {
        case SFB200_ACT_ELU: return z > 0.f ? z : expm1f(z);   // nn.ELU(alpha=1)
        case SFB200_ACT_RELU: return fmaxf(z, 0.f);
        case SFB200_ACT_TANH: return tanhf(z);
        default: return z;
    }
}
// derivative of the activation expressed through its OUTPUT h = act(z)
__device__ __forceinline__ float act_bwd_from_out(float h, int act) {
    switch (act) {
        case SFB200_ACT_ELU: return h > 0.f ? 1.f : h + 1.f;   // z<=0: d/dz (e^z-1) = e^z = h+1
        case SFB200_ACT_RELU: return h > 0.f ? 1.f : 0.f;
        case SFB200_ACT_TANH: return 1.f - h * h;
        default: return 1.f;
    }
}

// the 3xTF32 operand split: hi = w with the 13 low mantissa bits cleared (what the tensor core reads of w), lo = the
// tf32-representable part of the remainder
__device__ __forceinline__ uint32_t tf32_lo_bits(uint32_t w) {
    const uint32_t h = w & 0xffffe000u;
    return __float_as_uint(__uint_as_float(w) - __uint_as_float(h)) & 0xffffe000u;
}

// ---- fp16 operand split (the "3xFP16" engine) ---------------------------------------------------------------------
// v = x * 2^e is represented as hi + lo * 2^-11 with hi = fp16(v) (round to nearest) and lo = fp16((v - hi) * 2^11): 22
// significand bits like the tf32 pair, but on the fp16 tensor-core path (twice the MMA rate, half the operand bytes).
// fp16 has 5 exponent bits, so e is chosen from a known bound of |x|: bound * 2^e lands in [2^14, 2^15) -- one binade of
// headroom below the largest fp16 -- and elements down to 2^-29 of the bound keep full relative precision (smaller ones
// keep an ABSOLUTE error of 2^-36 * 2^-e, i.e. 2^-50 of the bound).  Weights use the fixed shift kF16WShift (|w| < 255).
constexpr int kF16WShift = 8;
constexpr int kF16LoShift = 11;
__device__ __forceinline__ int f16_shift_for_bound(float bound) {
    const int eb = (int)((__float_as_uint(bound) >> 23) & 0xffu) - 127;      // floor(log2(bound)) for normal floats
    int e = 14 - eb;
    return e < -100 ? -100 : (e > 100 ? 100 : e);                            // (bound 0 / denormal -> huge e: clamp)
}
__device__ __forceinline__ float pow2f_int(int e) { return __uint_as_float((uint32_t)(e + 127) << 23); }
// two scaled values -> packed (hi, lo) half2 words, element 0 in the low 16 bits
__device__ __forceinline__ void f16_split2(float v0, float v1, uint32_t& hi, uint32_t& lo) {
    const __half2 h = __floats2half2_rn(v0, v1);
    const float2 hf = __half22float2(h);
    const __half2 l = __floats2half2_rn((v0 - hf.x) * 2048.f, (v1 - hf.y) * 2048.f);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = *reinterpret_cast<const uint32_t*>(&l);
}
__device__ __forceinline__ void f16_split1(float v, uint16_t& hi, uint16_t& lo) {
    const __half h = __float2half_rn(v);
    const __half l = __float2half_rn((v - __half2float(h)) * 2048.f);
    hi = *reinterpret_cast<const uint16_t*>(&h);
    lo = *reinterpret_cast<const uint16_t*>(&l);
}

__device__ __forceinline__ float clampf(float x, float lo, float hi) { return fminf(fmaxf(x, lo), hi); }

}  // namespace sfb
