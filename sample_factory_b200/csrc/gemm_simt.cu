// CUDA-core fp32 GEMM engine (SFB200_GEMM_SIMT_FP32): exact-fp32 FFMA tiles, the parity-grade baseline engine and
// the fallback for shapes the wgmma engine does not take.  C[m,n] = sum_k A(m,k) * B(n,k) with either operand stored
// K-contiguous ([rows, K]) or row-contiguous ([K, rows]); 128x128x16 CTA tile, 256 threads, 8x8 register micro-tile,
// double-buffered shared memory, optional split-K (deterministic two-pass reduce).
#include <cstdlib>

#include "common.cuh"
#include "gemm.h"

namespace sfb {

constexpr int BM = 128, BN = 128, BK = 16, LDS = BM + 4;

struct Epilogue {
    int mode;            // 0: plain store, 1: act(acc + bias[n]), 2: acc * act'(aux[m,n]), 3: acc + bias[n] + aux[m,n]
    int act;
    const float* bias;   // [N]
    const float* aux;    // [M, ld_aux]
    int64_t ld_aux;
};

__device__ __forceinline__ float apply_epilogue(float acc, int64_t m, int n, const Epilogue& e) {
    if (e.mode == 1) return act_fwd(acc + (e.bias ? e.bias[n] : 0.f), e.act);
    if (e.mode == 2) return acc * act_bwd_from_out(e.aux[m * e.ld_aux + n], e.act);
    if (e.mode == 3) return (acc + e.bias[n]) + e.aux[m * e.ld_aux + n];
    return acc;
}

// Loads one BKxB{M,N} operand tile into registers (2 float4 per thread), zero-filled out of bounds.
template <bool KCONT>
__device__ __forceinline__ void load_tile(const float* __restrict__ P, int64_t ld, int64_t row0, int64_t rows, int k0,
                                          int k_end, bool vec_ok, float4 (&r)[2]) {
    const int t = threadIdx.x;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (KCONT) {
            const int64_t row = row0 + (t >> 2) + 64 * i;
            const int k = k0 + ((t & 3) << 2);
            if (row < rows) {
                const float* src = P + row * ld + k;
                if (vec_ok && k + 3 < k_end) v = *reinterpret_cast<const float4*>(src);
                else {
                    if (k < k_end) v.x = src[0];
                    if (k + 1 < k_end) v.y = src[1];
                    if (k + 2 < k_end) v.z = src[2];
                    if (k + 3 < k_end) v.w = src[3];
                }
            }
        } else {
            const int k = k0 + (t >> 5) + 8 * i;
            const int64_t row = row0 + ((t & 31) << 2);
            if (k < k_end) {
                const float* src = P + (int64_t)k * ld + row;
                if (vec_ok && row + 3 < rows) v = *reinterpret_cast<const float4*>(src);
                else {
                    if (row < rows) v.x = src[0];
                    if (row + 1 < rows) v.y = src[1];
                    if (row + 2 < rows) v.z = src[2];
                    if (row + 3 < rows) v.w = src[3];
                }
            }
        }
        r[i] = v;
    }
}

template <bool KCONT>
__device__ __forceinline__ void store_tile(float (*S)[LDS], const float4 (&r)[2]) {
    const int t = threadIdx.x;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        if (KCONT) {
            const int row = (t >> 2) + 64 * i;
            const int k = (t & 3) << 2;
            S[k + 0][row] = r[i].x;
            S[k + 1][row] = r[i].y;
            S[k + 2][row] = r[i].z;
            S[k + 3][row] = r[i].w;
        } else {
            const int k = (t >> 5) + 8 * i;
            const int row = (t & 31) << 2;
            *reinterpret_cast<float4*>(&S[k][row]) = r[i];
        }
    }
}

template <bool A_KCONT, bool B_KCONT>
__global__ void __launch_bounds__(256, 2) gemm_simt_kernel(const float* __restrict__ A, int64_t lda,
                                                        const float* __restrict__ B, int64_t ldb, float* __restrict__ C,
                                                        int64_t ldc, int64_t M, int N, int K, int k_chunk, bool a_vec,
                                                        bool b_vec, Epilogue epi) {
    __shared__ __align__(16) float As[2][BK][LDS];
    __shared__ __align__(16) float Bs[2][BK][LDS];
    const int t = threadIdx.x;
    const int tx = t & 15, ty = t >> 4;
    const int64_t m0 = (int64_t)blockIdx.y * BM;
    const int n0 = blockIdx.x * BN;
    const int k_begin = blockIdx.z * k_chunk;
    const int k_end = (k_begin + k_chunk < K) ? k_begin + k_chunk : K;
    if (gridDim.z > 1) C += (int64_t)blockIdx.z * M * ldc;   // split-K partial slab

    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

    float4 ra[2], rb[2];
    load_tile<A_KCONT>(A, lda, m0, M, k_begin, k_end, a_vec, ra);
    load_tile<B_KCONT>(B, ldb, n0, N, k_begin, k_end, b_vec, rb);
    store_tile<A_KCONT>(As[0], ra);
    store_tile<B_KCONT>(Bs[0], rb);
    __syncthreads();

    int buf = 0;
    for (int k0 = k_begin; k0 < k_end; k0 += BK) {
        const bool has_next = k0 + BK < k_end;
        if (has_next) {
            load_tile<A_KCONT>(A, lda, m0, M, k0 + BK, k_end, a_vec, ra);
            load_tile<B_KCONT>(B, ldb, n0, N, k0 + BK, k_end, b_vec, rb);
        }
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][kk][64 + ty * 4]);
            const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
            const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][kk][64 + tx * 4]);
            const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        if (has_next) {
            store_tile<A_KCONT>(As[buf ^ 1], ra);
            store_tile<B_KCONT>(Bs[buf ^ 1], rb);
            __syncthreads();
            buf ^= 1;
        }
    }

    const bool c_vec = (ldc % 4 == 0) && ((reinterpret_cast<uintptr_t>(C) & 15u) == 0);
    const bool do_epi = gridDim.z == 1;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int64_t m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
        if (m >= M) continue;
#pragma unroll
        for (int jh = 0; jh < 2; ++jh) {
            const int n = n0 + jh * 64 + tx * 4;
            float o[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float v = acc[i][jh * 4 + j];
                o[j] = (do_epi && n + j < N) ? apply_epilogue(v, m, n + j, epi) : v;
            }
            float* dst = C + m * ldc + n;
            if (c_vec && n + 3 < N) *reinterpret_cast<float4*>(dst) = make_float4(o[0], o[1], o[2], o[3]);
            else {
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (n + j < N) dst[j] = o[j];
            }
        }
    }
}

__global__ void __launch_bounds__(256) splitk_reduce_kernel(const float* __restrict__ part, int splits, int64_t M, int N,
                                                            float* __restrict__ C, int64_t ldc, Epilogue epi) {
    const int64_t total = M * (int64_t)N;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        float s = 0.f;
        for (int z = 0; z < splits; ++z) s += part[(int64_t)z * total + i];   // fixed order: deterministic
        const int64_t m = i / N;
        const int n = (int)(i - m * N);
        C[m * ldc + n] = apply_epilogue(s, m, n, epi);
    }
}

// column sums of X[M, N] (bias gradients): partial over row groups, then a fixed-order reduce.
__global__ void __launch_bounds__(256) colsum_partial_kernel(const float* __restrict__ X, int64_t ldx, int64_t M, int N,
                                                             int64_t rows_per_group, float* __restrict__ part) {
    const int64_t r0 = blockIdx.x * rows_per_group;
    const int64_t r1 = (r0 + rows_per_group < M) ? r0 + rows_per_group : M;
    for (int n = blockIdx.y * 256 + threadIdx.x; n < N; n += gridDim.y * 256) {
        float s = 0.f;
        for (int64_t r = r0; r < r1; ++r) s += X[r * ldx + n];
        part[(int64_t)blockIdx.x * N + n] = s;
    }
}
// one warp per output column, lanes stride over the row groups
__global__ void colsum_reduce_kernel(const float* __restrict__ part, int groups, int N, float* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (n >= N) return;
    float s = 0.f;
    for (int g = lane; g < groups; g += 32) s += part[(int64_t)g * N + n];
    s = warp_sum(s);
    if (lane == 0) out[n] = s;
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// SFB200_SPLITK_LEGACY=1: the split-K rule this engine had before it was sized to the device (A/B comparison: dW sums
// then group as they did, so results are bit-identical to that build's)
static bool splitk_legacy() {
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("SFB200_SPLITK_LEGACY");
        v = (e && e[0] == '1') ? 1 : 0;
    }
    return v == 1;
}

// Split-K slices of a GEMM with an M x N output reduced over K, on a device of `sms` SMs: fewer tiles than SMs -> as many
// slices as still give every CTA an SM in one wave (tiles * s <= sms); otherwise none.  At least 128 k per slice, at
// most 64 slices.
int choose_splits(int64_t M, int N, int K, int sms) {
    const int64_t tiles = ceil_div(M, BM) * ceil_div(N, BN);
    int64_t s = tiles < sms ? sms / tiles : 1;
    if (splitk_legacy()) s = tiles >= 148 ? 1 : ceil_div(2 * (int64_t)148, tiles);
    const int64_t max_by_k = K / (BK * 8) > 0 ? K / (BK * 8) : 1;
    if (s > max_by_k) s = max_by_k;
    if (s > 64) s = 64;
    if (s < 1) s = 1;
    return (int)s;
}
// on the current device (sm_count(): 132, the H100's, when there is no device to ask, so that workspace sizes can be
// computed without one)
int choose_splits(int64_t M, int N, int K) { return choose_splits(M, N, K, sm_count()); }

// C[M,N] = epilogue( sum_k A(m,k) B(n,k) ); ws needed only when splits > 1.
int gemm_simt(bool a_kcont, const float* A, int64_t lda, bool b_kcont, const float* B, int64_t ldb, float* C, int64_t ldc,
              int64_t M, int N, int K, int splits, const Epilogue& epi, float* ws, cudaStream_t st) {
    if (M == 0 || N == 0) return 0;
    // grid.y holds the 128-row blocks (<= 65535): taller outputs (im2col rows of a conv over many frames) run in row slabs
    constexpr int64_t kMaxRows = 65535LL * BM;
    if (M > kMaxRows && splits == 1) {
        for (int64_t m0 = 0; m0 < M; m0 += kMaxRows) {
            Epilogue e = epi;
            if (e.aux) e.aux += m0 * e.ld_aux;
            const float* Am = a_kcont ? A + m0 * lda : A + m0;
            const int rc = gemm_simt(a_kcont, Am, lda, b_kcont, B, ldb, C + m0 * ldc, ldc,
                                     (M - m0 < kMaxRows) ? M - m0 : kMaxRows, N, K, 1, e, ws, st);
            if (rc) return rc;
        }
        return 0;
    }
    SFB_CHECK_ARG(ceil_div(M, BM) <= 65535, "gemm_simt: M too large (%lld)", (long long)M);
    const bool a_vec = (lda % 4 == 0) && aligned16(A) && (a_kcont || true);
    const bool b_vec = (ldb % 4 == 0) && aligned16(B);
    int k_chunk = K;
    if (splits > 1) {
        k_chunk = (int)(ceil_div(ceil_div(K, splits), BK) * BK);
        splits = (int)ceil_div(K, k_chunk);
    }
    dim3 grid((unsigned)ceil_div(N, BN), (unsigned)ceil_div(M, BM), (unsigned)splits);
    float* out = splits > 1 ? ws : C;
    const int64_t ld_out = splits > 1 ? N : ldc;
    SFB_CHECK_ARG(splits == 1 || ws != nullptr, "gemm_simt: split-K needs a workspace");
#define SFB_GEMM(AK, BKC) \
    gemm_simt_kernel<AK, BKC><<<grid, 256, 0, st>>>(A, lda, B, ldb, out, ld_out, M, N, K, k_chunk, a_vec, b_vec, epi)
    if (a_kcont && b_kcont) SFB_GEMM(true, true);
    else if (a_kcont && !b_kcont) SFB_GEMM(true, false);
    else if (!a_kcont && b_kcont) SFB_GEMM(false, true);
    else SFB_GEMM(false, false);
#undef SFB_GEMM
    SFB_LAUNCH_OK();
    if (splits > 1) {
        int64_t blocks = ceil_div(M * N, 256);
        const int64_t cap = (int64_t)sm_count() * 8;
        if (blocks > cap) blocks = cap;
        splitk_reduce_kernel<<<(unsigned)blocks, 256, 0, st>>>(ws, splits, M, N, C, ldc, epi);
        SFB_LAUNCH_OK();
    }
    return 0;
}

int splitk_reduce(const float* part, int splits, int64_t M, int N, float* C, int64_t ldc, cudaStream_t st) {
    Epilogue none{0, 0, nullptr, nullptr, 0};
    int64_t blocks = ceil_div(M * N, 256);
    const int64_t cap = (int64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    splitk_reduce_kernel<<<(unsigned)blocks, 256, 0, st>>>(part, splits, M, N, C, ldc, none);
    SFB_LAUNCH_OK();
    return 0;
}

constexpr int kColsumMaxGroups = 256;

int colsum(const float* X, int64_t ldx, int64_t M, int N, float* out, float* ws, cudaStream_t st) {
    int64_t groups = sm_count() * 2;
    if (groups > kColsumMaxGroups) groups = kColsumMaxGroups;
    int64_t rpg = ceil_div(M, groups);
    if (rpg < 16) rpg = 16;
    groups = ceil_div(M, rpg);
    dim3 grid((unsigned)groups, (unsigned)ceil_div(N, 256));
    colsum_partial_kernel<<<grid, 256, 0, st>>>(X, ldx, M, N, rpg, ws);
    SFB_LAUNCH_OK();
    colsum_reduce_kernel<<<(unsigned)ceil_div((int64_t)N * 32, 256), 256, 0, st>>>(ws, (int)groups, N, out);
    SFB_LAUNCH_OK();
    return 0;
}

int colsum_reduce(const float* part, int64_t groups, int N, float* out, cudaStream_t st) {
    colsum_reduce_kernel<<<(unsigned)ceil_div((int64_t)N * 32, 256), 256, 0, st>>>(part, (int)groups, N, out);
    SFB_LAUNCH_OK();
    return 0;
}

int64_t colsum_workspace_floats(int N) { return (int64_t)kColsumMaxGroups * N; }

}  // namespace sfb

using namespace sfb;

extern "C" {

int sfb200_linear_act_forward(const float* x, int64_t ldx, const float* W, const float* b, float* y, int64_t ldy,
                              int64_t M, int N, int K, int act, int engine, void* stream) {
    SFB_CHECK_ARG(x && W && y && M >= 0 && N > 0 && K > 0, "linear_act_forward: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    if (engine != SFB200_GEMM_SIMT_FP32) {
        int rc = tc_linear_act_forward(x, ldx, W, b, y, ldy, M, N, K, act, engine, st);
        if (rc != SFB_TC_UNSUPPORTED) return rc;
        // shape not covered by the tensor-core engine: exact-fp32 CUDA-core tiles (still on device)
    }
    Epilogue epi{1, act, b, nullptr, 0};
    return gemm_simt(true, x, ldx, true, W, K, y, ldy, M, N, K, 1, epi, nullptr, st);
}

int sfb200_linear_residual_forward(const float* x, int64_t ldx, const float* W, const float* b, const float* r,
                                   int64_t ldr, float* y, int64_t ldy, int64_t M, int N, int K, int engine, void* stream) {
    SFB_CHECK_ARG(x && W && b && r && y && M >= 0 && N > 0 && K > 0, "linear_residual_forward: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    if (engine != SFB200_GEMM_SIMT_FP32) {
        int rc = tc_linear_residual_forward(x, ldx, W, b, r, ldr, y, ldy, M, N, K, engine, st);
        if (rc != SFB_TC_UNSUPPORTED) return rc;
    }
    Epilogue epi{3, SFB200_ACT_NONE, b, r, ldr};
    return gemm_simt(true, x, ldx, true, W, K, y, ldy, M, N, K, 1, epi, nullptr, st);
}

int sfb200_linear_heads_partials(int N, int A, int engine) { return tc_linear_heads_partials(N, A, engine); }

int sfb200_linear_act_heads_forward(const float* x, int64_t ldx, const float* W, const float* b, float* y, int64_t ldy,
                                    int64_t M, int N, int K, int act, int engine, const float* Wv, const float* Wa,
                                    int A, float* head_partials, void* stream) {
    SFB_CHECK_ARG(x && W && b && Wv && Wa && head_partials && M >= 0 && N > 0 && K > 0,
                  "linear_act_heads_forward: bad arguments");
    if (M == 0) return 0;
    int rc = tc_linear_act_heads_forward(x, ldx, W, b, y, ldy, M, N, K, act, engine, Wv, Wa, A, head_partials,
                                         (cudaStream_t)stream);
    SFB_CHECK_ARG(rc != SFB_TC_UNSUPPORTED,
                  "linear_act_heads_forward: shape/engine not covered (N=%d K=%d A=%d engine=%d); "
                  "sfb200_linear_heads_partials() tells when to use the separate calls", N, K, A, engine);
    return rc;
}

int sfb200_linear_backward_splits(int64_t M, int N, int K, int sm_count) {
    const int m = (int)(M > 0x7fffffff ? 0x7fffffff : M);
    return sm_count > 0 ? choose_splits(N, K, m, sm_count) : choose_splits(N, K, m);
}

int64_t sfb200_linear_backward_workspace_bytes(int64_t M, int N, int K) {
    // split-K slabs for dW [N,K] reduced over M, plus colsum partials for db_prev [K]
    const int splits = choose_splits(N, K, (int)(M > 0x7fffffff ? 0x7fffffff : M));
    // colsum partials: kColsumMaxGroups rows for the standalone kernel, M/32 rows when the dX GEMM's epilogue writes them
    int64_t cs_rows = M / 32 + 1;
    if (cs_rows < kColsumMaxGroups) cs_rows = kColsumMaxGroups;
    return ((int64_t)splits * N * K + cs_rows * K) * (int64_t)sizeof(float);
}

int sfb200_linear_backward(const float* dz, int64_t lddz, const float* x, int64_t ldx, const float* W, int64_t M, int N,
                           int K, int act_prev, float* dW, float* dx, int64_t lddx, float* db_prev, int engine,
                           void* workspace, void* stream) {
    SFB_CHECK_ARG(dz && x && W && (dW || dx) && workspace && M > 0 && N > 0 && K > 0 && M <= 0x7fffffff,
                  "linear_backward: bad arguments");
    SFB_CHECK_ARG(!db_prev || dx, "linear_backward: db_prev needs dx");
    cudaStream_t st = (cudaStream_t)stream;
    float* ws = (float*)workspace;
    const int splits = choose_splits(N, K, (int)M);
    float* ws_colsum = ws + (int64_t)splits * N * K;
    int rc;
    if (engine != SFB200_GEMM_SIMT_FP32) {
        int fused = 0;
        rc = tc_linear_backward(dz, lddz, x, ldx, W, M, N, K, act_prev, dW, dx, lddx, engine, ws, st,
                                db_prev ? ws_colsum : nullptr, &fused);
        if (rc == 0 || rc != SFB_TC_UNSUPPORTED) {
            if (rc) return rc;
            if (db_prev && fused) return colsum_reduce(ws_colsum, M / 32, K, db_prev, st);
            if (db_prev) return colsum(dx, lddx, M, K, db_prev, ws_colsum, st);
            return 0;
        }
    }
    // dW[n,k] = sum_m dz[m,n] * x[m,k]   (both operands row-contiguous in the reduced dimension's rows)
    Epilogue none{0, 0, nullptr, nullptr, 0};
    rc = dW ? gemm_simt(false, dz, lddz, false, x, ldx, dW, K, N, K, (int)M, splits, none, ws, st) : 0;
    if (rc) return rc;
    if (dx) {
        // dx[m,k] = (sum_n dz[m,n] * W[n,k]) * act_prev'(x[m,k])
        Epilogue e{act_prev == SFB200_ACT_NONE ? 0 : 2, act_prev, nullptr, x, ldx};
        rc = gemm_simt(true, dz, lddz, false, W, K, dx, lddx, M, K, N, 1, e, nullptr, st);
        if (rc) return rc;
        if (db_prev) return colsum(dx, lddx, M, K, db_prev, ws_colsum, st);
    }
    return 0;
}

int64_t sfb200_colsum_workspace_bytes(int N) { return colsum_workspace_floats(N) * (int64_t)sizeof(float); }

int sfb200_colsum(const float* x, int64_t ldx, int64_t M, int N, float* out, void* workspace, void* stream) {
    SFB_CHECK_ARG(x && out && workspace && M > 0 && N > 0, "colsum: bad arguments");
    return colsum(x, ldx, M, N, out, (float*)workspace, (cudaStream_t)stream);
}

}  // extern "C"
