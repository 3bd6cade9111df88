// Library-level entry points of libsfb200 (see include/sfb200.h).
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace sfb {
static thread_local char g_err[512] = "";
static thread_local int g_sm_count = 0;

static unsigned long long g_launches = 0;
void count_launch() { __atomic_fetch_add(&g_launches, 1ull, __ATOMIC_RELAXED); }

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

// ---- fp16 twins of weight buffers, their transposed per-matrix copies, activation bounds (the fp16-split GEMM engine)
struct F16Range { const float* base; uint16_t* twins; int64_t n; };            // twins = [hi16[n] | lo16[n]]
struct F16TRange { const float* W; int N, K; uint16_t* twins; };               // twins = [hiT[K][N] | loT[K][N]]
struct BoundRange { const char* base; int64_t bytes; const float* bound; };
static F16Range g_f16[32];
static int g_f16_n = 0;
static F16TRange g_f16t[64];
static int g_f16t_n = 0;
static BoundRange g_bound[64];
static int g_bound_n = 0;

uint16_t* f16_twin_lookup_mut(float* p, int64_t count, int64_t* lo_offset) {
    for (int i = 0; i < g_f16_n; ++i) {
        const F16Range& r = g_f16[i];
        if (p >= r.base && p + count <= r.base + r.n) {
            if (lo_offset) *lo_offset = r.n;
            return r.twins + (p - r.base);
        }
    }
    return nullptr;
}
F16Twin f16_twin_lookup(const float* p, int64_t count) {
    int64_t off = 0;
    const uint16_t* hi = f16_twin_lookup_mut(const_cast<float*>(p), count, &off);
    return F16Twin{hi, hi ? hi + off : nullptr};
}
F16Twin f16_twinT_lookup(const float* W, int N, int K) {
    for (int i = 0; i < g_f16t_n; ++i)
        if (g_f16t[i].W == W && g_f16t[i].N == N && g_f16t[i].K == K)
            return F16Twin{g_f16t[i].twins, g_f16t[i].twins + (int64_t)N * K};
    return F16Twin{nullptr, nullptr};
}
const float* operand_bound_lookup(const void* p, int64_t bytes) {
    const char* c = static_cast<const char*>(p);
    for (int i = 0; i < g_bound_n; ++i)
        if (c >= g_bound[i].base && c + bytes <= g_bound[i].base + g_bound[i].bytes) return g_bound[i].bound;
    return nullptr;
}

__global__ void f16_split_kernel(const float* __restrict__ w, uint16_t* __restrict__ hi, uint16_t* __restrict__ lo, int64_t n) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        f16_split1(w[i] * (float)(1 << kF16WShift), hi[i], lo[i]);
}

// W[N][K] fp32 -> hiT / loT [K][N] fp16 (32 x 32 tiles through shared memory: coalesced on both sides)
__global__ void __launch_bounds__(256) f16_split_transposed_kernel(const float* __restrict__ W, int N, int K,
                                                                   uint16_t* __restrict__ hiT, uint16_t* __restrict__ loT) {
    __shared__ float tile[32][33];
    const int n0 = blockIdx.y * 32, k0 = blockIdx.x * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int r = ty; r < 32; r += 8)
        tile[r][tx] = (n0 + r < N && k0 + tx < K) ? W[(int64_t)(n0 + r) * K + k0 + tx] : 0.f;
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {
        const int k = k0 + r, n = n0 + tx;
        if (k < K && n < N) f16_split1(tile[tx][r] * (float)(1 << kF16WShift), hiT[(int64_t)k * N + n], loT[(int64_t)k * N + n]);
    }
}

// Upper bound of |act(x W^T + b)| over all inputs with |x| <= in_bound: max_n (in_bound * sum_k |W[n][k]| + |b[n]|)
// (ELU / ReLU / tanh are 1-Lipschitz with act(0) = 0; tanh additionally <= 1).  One warp per output row, eight rows per
// block; block maxima meet in an atomicMax on the bit pattern (non-negative floats order like unsigned ints), the block that
// arrives last publishes the bound.  out = [bound, scratch bits, arrival counter, -]; scratch and counter are left at zero.
__global__ void __launch_bounds__(256) linear_out_bound_kernel(const float* __restrict__ W, const float* __restrict__ b, int N,
                                                              int K, const float* __restrict__ in_bound,
                                                              float* __restrict__ out, int act) {
    __shared__ float s_v[8];
    unsigned int* scratch = reinterpret_cast<unsigned int*>(out) + 1;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n = blockIdx.x * 8 + warp;
    float v = 0.f;
    if (n < N) {
        float t = 0.f;
        for (int k = lane; k < K; k += 32) t += fabsf(W[(int64_t)n * K + k]);
        t = warp_sum(t);
        v = in_bound[0] * t * 1.0001f + (b ? fabsf(b[n]) : 0.f);      // (the row sum is rounded: a hair of slack)
    }
    if (lane == 0) s_v[warp] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int i = 1; i < 8; ++i) v = fmaxf(v, s_v[i]);
        atomicMax(scratch, __float_as_uint(v));
        __threadfence();
        if (atomicAdd(scratch + 1, 1u) == gridDim.x - 1) {
            __threadfence();
            float r = __uint_as_float(*reinterpret_cast<volatile unsigned int*>(scratch));
            if (act == SFB200_ACT_TANH) r = fminf(r, 1.f);
            out[0] = r;
            scratch[0] = 0u;
            scratch[1] = 0u;
        }
    }
}

// Gradient factor of a layer: max_k sum_n |W[n][k]|, so that |dz_in[m][k]| = |sum_n dz_out[m][n] W[n][k]| * |act'| <=
// bound(dz_out) * factor (act' <= 1).  32 columns per block, each summed over the rows in a fixed order by 8 row phases;
// block maxima meet as in linear_out_bound_kernel.  out = [factor, scratch bits, arrival counter, -].
__global__ void __launch_bounds__(256) linear_in_grad_bound_kernel(const float* __restrict__ W, int N, int K,
                                                                  float* __restrict__ out) {
    __shared__ float s_p[8][33];
    unsigned int* scratch = reinterpret_cast<unsigned int*>(out) + 1;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int k = blockIdx.x * 32 + tx;
    float t = 0.f;
    if (k < K)
        for (int n = ty; n < N; n += 8) t += fabsf(W[(int64_t)n * K + k]);
    s_p[ty][tx] = t;
    __syncthreads();
    if (ty == 0) {
        for (int i = 1; i < 8; ++i) t += s_p[i][tx];
        const float v = warp_max(t * 1.0001f);   // (the column sum is rounded: a hair of slack)
        if (tx == 0) {
            atomicMax(scratch, __float_as_uint(v));
            __threadfence();
            if (atomicAdd(scratch + 1, 1u) == gridDim.x - 1) {
                __threadfence();
                out[0] = __uint_as_float(*reinterpret_cast<volatile unsigned int*>(scratch));
                scratch[0] = 0u;
                scratch[1] = 0u;
            }
        }
    }
}

// Upper bound of the gradient that heads_backward writes for the last hidden layer:
// |dz[m][j]| = |dv[m] Wv[j] + sum_a dl[m][a] Wa[a][j]| * |act'| <= (|dv[m]| + sum_a |dl[m][a]|) * max(|Wv|_inf, |Wa|_inf),
// act' <= 1 for ELU / ReLU / tanh.  1.2 MB of per-sample gradients at the cfg-2 minibatch: 64 blocks take the row maxima
// (atomicMax on the bit pattern of a non-negative float), the block that arrives last folds in the weight maximum.
// out = [bound, scratch bits, arrival counter]; scratch and counter are left at zero.
// The last block also runs the chain down the hidden layers below: bound(dz[i]) = bound(dz[i+1]) * factor(W[i+1])
// (linear_in_grad_bound_kernel) into chain[4 i], i = n_chain-1 .. 0, with factor(W[j]) at factors[4 j].
__global__ void __launch_bounds__(256) heads_dz_bound_kernel(const float* __restrict__ dlogits, const float* __restrict__ dvalues,
                                                            int64_t rows, int A, const float* __restrict__ Wv,
                                                            const float* __restrict__ Wa, int H, float* __restrict__ out,
                                                            const float* __restrict__ factors, float* __restrict__ chain,
                                                            int n_chain) {
    __shared__ float s_r[8], s_w[8];
    unsigned int* scratch = reinterpret_cast<unsigned int*>(out) + 1;
    float r = 0.f, w = 0.f;
    // (every block takes the weight maximum itself -- 4.6 K elements from L2 -- instead of leaving it to a serial last phase)
    for (int i = threadIdx.x; i < H; i += blockDim.x) w = fmaxf(w, fabsf(Wv[i]));
    for (int i = threadIdx.x; i < A * H; i += blockDim.x) w = fmaxf(w, fabsf(Wa[i]));
    for (int64_t m = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; m < rows; m += (int64_t)gridDim.x * blockDim.x) {
        float t = fabsf(dvalues[m]);
        for (int a = 0; a < A; ++a) t += fabsf(dlogits[m * A + a]);
        r = fmaxf(r, t);
    }
    for (int o = 16; o > 0; o >>= 1) {
        r = fmaxf(r, __shfl_xor_sync(0xffffffffu, r, o));
        w = fmaxf(w, __shfl_xor_sync(0xffffffffu, w, o));
    }
    if ((threadIdx.x & 31) == 0) { s_r[threadIdx.x >> 5] = r; s_w[threadIdx.x >> 5] = w; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int i = 1; i < 8; ++i) { r = fmaxf(r, s_r[i]); w = fmaxf(w, s_w[i]); }
        atomicMax(scratch, __float_as_uint(r * w * 1.0001f));
        __threadfence();
        if (atomicAdd(scratch + 1, 1u) == gridDim.x - 1) {
            __threadfence();
            float b = __uint_as_float(*reinterpret_cast<volatile unsigned int*>(scratch));
            out[0] = b;
            scratch[0] = 0u;
            scratch[1] = 0u;
            for (int i = n_chain - 1; i >= 0; --i) {
                b = b * factors[4 * (i + 1)] * 1.0001f;   // (the product is rounded: a hair of slack)
                chain[4 * i] = b;
            }
        }
    }
}

// SFB200_CHECK_F16=1 verifies fp16 twins (row-major: ld = K; transposed: element (n, k) at k * N + n) before every use
__global__ void f16_check_twins_kernel(const float* __restrict__ W, const uint16_t* __restrict__ hi, const uint16_t* __restrict__ lo,
                                       int N, int K, int transposed) {
    const int64_t n_el = (int64_t)N * K;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n_el; i += (int64_t)gridDim.x * blockDim.x) {
        uint16_t h, l;
        f16_split1(W[i] * (float)(1 << kF16WShift), h, l);
        const int64_t j = transposed ? (i % K) * N + i / K : i;
        if (hi[j] != h || lo[j] != l) {
            printf("libsfb200: STALE fp16 twins at element %lld (call sfb200_refresh_f16_twins / _transposed after writing weights)\n",
                   (long long)i);
            __trap();
        }
    }
}

int f16_twins_check(const float* W, F16Twin tw, int N, int K, bool transposed, cudaStream_t st) {
    int64_t blocks = ceil_div((int64_t)N * K, 256);
    if (blocks > 1024) blocks = 1024;
    f16_check_twins_kernel<<<(unsigned)blocks, 256, 0, st>>>(W, tw.hi, tw.lo, N, K, transposed ? 1 : 0);
    SFB_LAUNCH_OK();
    return 0;
}

bool pdl_enabled() {
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("SFB200_PDL");
        v = (e && e[0] == '0') ? 0 : 1;
    }
    return v == 1;
}

int sm_count() {
    if (g_sm_count == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) == cudaSuccess) {
            int n = 0;
            if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess) g_sm_count = n;
        }
        if (g_sm_count <= 0) g_sm_count = 132;   // no device to ask (host-only callers sizing workspaces): the H100's
    }
    return g_sm_count;
}
}  // namespace sfb

extern "C" {

int sfb200_abi_version(void) { return SFB200_ABI_VERSION; }

const char* sfb200_last_error(void) { return sfb::g_err; }

int sfb200_set_device(int device) {
    SFB_CUDA_OK(cudaSetDevice(device));
    sfb::g_sm_count = 0;
    return 0;
}

int sfb200_sm_count(void) { return sfb::sm_count(); }

int sfb200_register_f16_twins(const float* base, void* twins, int64_t n) {
    SFB_CHECK_ARG(base && twins && n > 0, "register_f16_twins: bad arguments");
    for (int i = 0; i < sfb::g_f16_n; ++i)
        if (sfb::g_f16[i].base == base) {
            sfb::g_f16[i] = sfb::F16Range{base, static_cast<uint16_t*>(twins), n};
            return 0;
        }
    SFB_CHECK_ARG(sfb::g_f16_n < 32, "register_f16_twins: table full");
    sfb::g_f16[sfb::g_f16_n++] = sfb::F16Range{base, static_cast<uint16_t*>(twins), n};
    return 0;
}

int sfb200_unregister_f16_twins(const float* base) {
    for (int i = 0; i < sfb::g_f16_n; ++i)
        if (sfb::g_f16[i].base == base) {
            sfb::g_f16[i] = sfb::g_f16[--sfb::g_f16_n];
            break;
        }
    // transposed per-matrix twins of matrices inside this buffer go with it
    return 0;
}

int sfb200_refresh_f16_twins(const float* base, void* stream) {
    for (int i = 0; i < sfb::g_f16_n; ++i)
        if (sfb::g_f16[i].base == base) {
            const sfb::F16Range& r = sfb::g_f16[i];
            int64_t blocks = sfb::ceil_div(r.n, 256);
            if (blocks > 1184) blocks = 1184;
            sfb::f16_split_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(r.base, r.twins, r.twins + r.n, r.n);
            SFB_LAUNCH_OK();
            return 0;
        }
    sfb::set_error("refresh_f16_twins: buffer is not registered");
    return 1;
}

int sfb200_register_f16_transposed(const float* W, int N, int K, void* twinsT) {
    SFB_CHECK_ARG(W && twinsT && N > 0 && K > 0, "register_f16_transposed: bad arguments");
    for (int i = 0; i < sfb::g_f16t_n; ++i)
        if (sfb::g_f16t[i].W == W) {
            sfb::g_f16t[i] = sfb::F16TRange{W, N, K, static_cast<uint16_t*>(twinsT)};
            return 0;
        }
    SFB_CHECK_ARG(sfb::g_f16t_n < 64, "register_f16_transposed: table full");
    sfb::g_f16t[sfb::g_f16t_n++] = sfb::F16TRange{W, N, K, static_cast<uint16_t*>(twinsT)};
    return 0;
}

int sfb200_unregister_f16_transposed(const float* W) {
    for (int i = 0; i < sfb::g_f16t_n; ++i)
        if (sfb::g_f16t[i].W == W) {
            sfb::g_f16t[i] = sfb::g_f16t[--sfb::g_f16t_n];
            return 0;
        }
    return 0;
}

int sfb200_refresh_f16_transposed(const float* W, void* stream) {
    for (int i = 0; i < sfb::g_f16t_n; ++i)
        if (sfb::g_f16t[i].W == W) {
            const sfb::F16TRange& r = sfb::g_f16t[i];
            dim3 grid((unsigned)sfb::ceil_div(r.K, 32), (unsigned)sfb::ceil_div(r.N, 32));
            sfb::f16_split_transposed_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(r.W, r.N, r.K, r.twins,
                                                                                      r.twins + (int64_t)r.N * r.K);
            SFB_LAUNCH_OK();
            return 0;
        }
    sfb::set_error("refresh_f16_transposed: matrix is not registered");
    return 1;
}

int sfb200_register_operand_bound(const void* base, int64_t bytes, const float* bound_dev) {
    SFB_CHECK_ARG(base && bytes > 0 && bound_dev, "register_operand_bound: bad arguments");
    for (int i = 0; i < sfb::g_bound_n; ++i)
        if (sfb::g_bound[i].base == base) {
            sfb::g_bound[i] = sfb::BoundRange{static_cast<const char*>(base), bytes, bound_dev};
            return 0;
        }
    SFB_CHECK_ARG(sfb::g_bound_n < 64, "register_operand_bound: table full");
    sfb::g_bound[sfb::g_bound_n++] = sfb::BoundRange{static_cast<const char*>(base), bytes, bound_dev};
    return 0;
}

int sfb200_unregister_operand_bound(const void* base) {
    for (int i = 0; i < sfb::g_bound_n; ++i)
        if (sfb::g_bound[i].base == base) {
            sfb::g_bound[i] = sfb::g_bound[--sfb::g_bound_n];
            return 0;
        }
    return 0;
}

int sfb200_linear_out_bound(const float* W, const float* b, int N, int K, const float* in_bound_dev, float* out_bound_dev,
                            int act, void* stream) {
    SFB_CHECK_ARG(W && in_bound_dev && out_bound_dev && N > 0 && K > 0, "linear_out_bound: bad arguments");
    sfb::linear_out_bound_kernel<<<(unsigned)sfb::ceil_div(N, 8), 256, 0, (cudaStream_t)stream>>>(W, b, N, K, in_bound_dev, out_bound_dev, act);
    SFB_LAUNCH_OK();
    return 0;
}

int sfb200_linear_in_grad_bound(const float* W, int N, int K, float* out_dev, void* stream) {
    SFB_CHECK_ARG(W && out_dev && N > 0 && K > 0, "linear_in_grad_bound: bad arguments");
    sfb::linear_in_grad_bound_kernel<<<(unsigned)sfb::ceil_div(K, 32), 256, 0, (cudaStream_t)stream>>>(W, N, K, out_dev);
    SFB_LAUNCH_OK();
    return 0;
}

int sfb200_heads_dz_bound(const float* dlogits, const float* dvalues, int64_t rows, int A, const float* Wv, const float* Wa,
                          int H, float* out_bound_dev, const float* factors_dev, float* chain_dev, int n_chain, void* stream) {
    SFB_CHECK_ARG(dlogits && dvalues && Wv && Wa && out_bound_dev && rows > 0 && A > 0 && H > 0 && n_chain >= 0 &&
                      (n_chain == 0 || (factors_dev && chain_dev)),
                  "heads_dz_bound: bad arguments");
    sfb::heads_dz_bound_kernel<<<128, 256, 0, (cudaStream_t)stream>>>(dlogits, dvalues, rows, A, Wv, Wa, H, out_bound_dev,
                                                                      factors_dev, chain_dev, n_chain);
    SFB_LAUNCH_OK();
    return 0;
}

uint64_t sfb200_launch_count(void) { return __atomic_load_n(&sfb::g_launches, __ATOMIC_RELAXED); }

}  // extern "C"
