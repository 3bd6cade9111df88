// The sampler's policy step for MLP policies as ONE wgmma kernel (model/actor_critic.py:160-195, model/encoder.py:72-91):
//
//     h1 = act(x W1^T + b1)          [M, H1]   x = normalised observations [M, K1], K1 = 32 or 64
//     h2 = act(h1 W2^T + b2)         [M, H2]
//     partial head dot products      h2 . [Wv ; Wa]^T over 32-column segments  (finished by heads_from_partials)
//
// A CTA owns a 128-row x 128-column tile of h2 and walks the K dimension of layer 2 in chunks of 32: for every chunk it
// first computes the matching 32 columns of h1 ITSELF (layer 1 is short-K, so recomputing it in each of the H2/128 column
// CTAs costs less than exchanging it), turns that accumulator into the next A operand in shared memory (bias +
// activation + tf32 hi/lo split into the swizzled K-major layout) and the layer-2 wgmmas consume it from there.  h1 never
// exists in global memory.  All flops are 3xTF32 (two accumulators, see gemm_tc.cu).
//
// 256 threads = two warpgroups of 64 rows each (wgmma M = 64); thread 0 issues the TMA loads: the x tile once, then per
// chunk W1[c*32.., :] and W2[n0.., c*32..] into a double-buffered raw stage (chunk c+1 is in flight while c is computed).
// Registers: layer-2 accumulators 2 x 64, layer-1 accumulators 2 x 16 per thread.
#include <cuda.h>

#include "common.cuh"
#include "gemm.h"
#include "heads_tail.cuh"
#include "tc_ptx.cuh"
#include "wgmma_tile.cuh"

namespace sfb {

constexpr int PS_THREADS = 256;
constexpr int PS_MAX_H1 = 1024;

struct PsSmem {
    static constexpr int XC = 0;                        // x hi/lo: per 32-k block [hi 16 KB | lo 16 KB], two blocks
    static constexpr int W1C = XC + 2 * 32768;          // W1 chunk hi/lo: per k block [hi 4 KB | lo 4 KB], two blocks
    static constexpr int H1C = W1C + 2 * 8192;          // h1 chunk [128 rows][32] hi | lo
    static constexpr int W2C = H1C + 32768;             // W2 tile [128 n][32 k] hi | lo
    static constexpr int XRAW = H1C;                    // x raw (two [128][32] boxes) before the chunk loop uses H1C / W2C
    static constexpr int RAW = W2C + 32768;             // 2 stages x [W1 raw 2 x 4 KB | W2 raw 16 KB]
    static constexpr int RAW_STAGE = 2 * 4096 + 16384;
    static constexpr int BARS = RAW + 2 * RAW_STAGE;
    static constexpr int TOTAL = 1024 + BARS + 64;
};

struct PsArgs {
    int64_t M;
    int K1, H1, H2, act;
    const float* b1;
    const float* b2;
    TcEpilogue epi;     // head weights / head_part; bias = b2
};

template <int ACT>
__device__ __forceinline__ void split_rows32(const uint8_t* raw, uint8_t* hi, uint8_t* lo, int t) {
    // [32 rows][32 k] K-major raw -> tf32 hi / lo, swizzled: 256 float4, one per thread
    const int r = t >> 3, c = t & 7;
    const uint4 v = reinterpret_cast<const uint4*>(raw)[t];
    const uint32_t off = (uint32_t)(r * 128 + (((c ^ r) & 7) << 4));
    *reinterpret_cast<uint4*>(hi + off) = make_uint4(v.x & 0xffffe000u, v.y & 0xffffe000u, v.z & 0xffffe000u, v.w & 0xffffe000u);
    *reinterpret_cast<uint4*>(lo + off) = make_uint4(tf32_lo_bits(v.x), tf32_lo_bits(v.y), tf32_lo_bits(v.z), tf32_lo_bits(v.w));
}

template <int KA, int ACT>
__global__ void __launch_bounds__(PS_THREADS, 1)
policy_mlp2_heads_kernel(const __grid_constant__ CUtensorMap tx, const __grid_constant__ CUtensorMap tw1,
                         const __grid_constant__ CUtensorMap tw2, const PsArgs a) {
    using S = PsSmem;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_align_1024(smem_raw);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S::BARS);
    uint64_t* x_bar = bars;
    uint64_t* full = bars + 1;              // [2] chunk stages
    const int t = threadIdx.x, wg = t >> 7, lane = t & 31;
    const int n0 = blockIdx.x * TBN;
    const int64_t m0 = (int64_t)blockIdx.y * TBM;
    const int NC = a.H1 / 32;

    if (t == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tx) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tw1) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tw2) : "memory");
        mbar_init(x_bar, 1);
        mbar_init(&full[0], 1);
        mbar_init(&full[1], 1);
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();
    pdl_trigger();

    auto issue_chunk = [&](int c) {
        uint8_t* st = smem + S::RAW + (c & 1) * S::RAW_STAGE;
        mbar_expect_tx(&full[c & 1], KA * 4096 + 16384);
        for (int kb = 0; kb < KA; ++kb) tma_load_2d(st + kb * 4096, &tw1, &full[c & 1], 32 * kb, 32 * c);
        tma_load_2d(st + 2 * 4096, &tw2, &full[c & 1], 32 * c, n0);
    };
    if (t == 0) {
        mbar_expect_tx(x_bar, KA * 16384);
        for (int kb = 0; kb < KA; ++kb) tma_load_2d(smem + S::XRAW + kb * 16384, &tx, x_bar, 32 * kb, (int)m0);
        issue_chunk(0);
    }
    mbar_wait(x_bar, 0);
    for (int kb = 0; kb < KA; ++kb)
        split_tile<false, true>(smem + S::XRAW + kb * 16384, smem + S::XC + kb * 32768, smem + S::XC + kb * 32768 + 16384, t);
    __syncthreads();

    float acc[64], cross[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = cross[i] = 0.f;
    const int r_in = wg * 64 + ((t >> 5) & 3) * 16 + (lane >> 2);   // first of the thread's two rows in the tile
    uint8_t* h1_hi = smem + S::H1C;
    uint8_t* h1_lo = h1_hi + 16384;
    uint8_t* w2_hi = smem + S::W2C;
    uint8_t* w2_lo = w2_hi + 16384;
    for (int c = 0; c < NC; ++c) {
        if (t == 0 && c + 1 < NC) issue_chunk(c + 1);   // its stage was read by everyone before the last barrier
        mbar_wait(&full[c & 1], (c >> 1) & 1);
        const uint8_t* st = smem + S::RAW + (c & 1) * S::RAW_STAGE;
        for (int kb = 0; kb < KA; ++kb)
            split_rows32<ACT>(st + kb * 4096, smem + S::W1C + kb * 8192, smem + S::W1C + kb * 8192 + 4096, t);
        split_tile<false, true>(st + 2 * 4096, w2_hi, w2_lo, t);
        fence_proxy_async_smem();
        __syncthreads();
        // ---- layer 1, columns [32c, 32c+32) of h1 for this warpgroup's 64 rows
        float d1[16], x1[16];
        wgmma_fence();
#pragma unroll
        for (int kb = 0; kb < KA; ++kb) {
            const uint64_t dxh = make_smem_desc(smem_u32(smem + S::XC + kb * 32768 + wg * 8192));
            const uint64_t dxl = make_smem_desc(smem_u32(smem + S::XC + kb * 32768 + 16384 + wg * 8192));
            const uint64_t dwh = make_smem_desc(smem_u32(smem + S::W1C + kb * 8192));
            const uint64_t dwl = make_smem_desc(smem_u32(smem + S::W1C + kb * 8192 + 4096));
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint64_t o = (uint64_t)(2 * k);
                wgmma_m64n32k8_tf32(d1, dxh + o, dwh + o, (kb | k) != 0);
                wgmma_m64n32k8_tf32(x1, dxh + o, dwl + o, (kb | k) != 0);
                wgmma_m64n32k8_tf32(x1, dxl + o, dwh + o, 1);
            }
        }
        wgmma_commit();
        wgmma_wait_all();
        // bias + activation + tf32 split -> the layer-2 A operand
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const int col = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
            const int row = r_in + 8 * ((i >> 1) & 1);
            const float h = act_fwd_ct<ACT>(d1[i] + x1[i] + a.b1[32 * c + col]);
            const uint32_t w = __float_as_uint(h);
            const uint32_t off = sw128_offset(row, col);
            *reinterpret_cast<uint32_t*>(h1_hi + off) = w & 0xffffe000u;
            *reinterpret_cast<uint32_t*>(h1_lo + off) = tf32_lo_bits(w);
        }
        fence_proxy_async_smem();
        __syncthreads();
        // ---- layer 2: acc (+)= h1[:, 32c..] . W2[n0.., 32c..]^T
        const uint64_t dah = make_smem_desc(smem_u32(h1_hi + wg * 8192));
        const uint64_t dal = make_smem_desc(smem_u32(h1_lo + wg * 8192));
        const uint64_t dbh = make_smem_desc(smem_u32(w2_hi));
        const uint64_t dbl = make_smem_desc(smem_u32(w2_lo));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint64_t o = (uint64_t)(2 * k);
            wgmma_m64n128k8_tf32(acc, dah + o, dbh + o, 1);
            wgmma_m64n128k8_tf32(cross, dah + o, dbl + o, 1);
            wgmma_m64n128k8_tf32(cross, dal + o, dbh + o, 1);
        }
        wgmma_commit();
        wgmma_wait_all();
        __syncthreads();   // every operand buffer of this chunk is free again
    }
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] += cross[i];
    TileCoord tc;
    tc.m0 = m0;
    tc.n0 = n0;
    tc.k_begin = 0;
    tc.num_kb = 0;
    tc.z = 0;
    heads_tile<ACT, 4>(acc, tc, m0 + r_in, lane, nullptr, 0, a.M, a.H2, a.epi);
}

template <int KA, int ACT>
static int launch_ps(const CUtensorMap& tx, const CUtensorMap& tw1, const CUtensorMap& tw2, const PsArgs& a, cudaStream_t st) {
    auto kern = policy_mlp2_heads_kernel<KA, ACT>;
    static bool attr_set = false;
    if (!attr_set) {
        SFB_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, PsSmem::TOTAL));
        attr_set = true;
    }
    const dim3 grid((unsigned)(a.H2 / 128), (unsigned)ceil_div(a.M, 128));
    SFB_CUDA_OK(launch_pdl(kern, grid, dim3(PS_THREADS), (size_t)PsSmem::TOTAL, st, tx, tw1, tw2, a));
    SFB_LAUNCH_OK();
    return 0;
}

// Does the fused two-layer policy step cover this model?  (3xTF32 engine, registered tf32-lo twins for both weight
// matrices -- i.e. the model's own weights --, K1 in {32, 64}, H1 a multiple of 32, H2 a multiple of 128 up to 512,
// <= 8 head rows.)
int tc_policy_mlp2_supported(const float* W1, const float* W2, int K1, int H1, int H2, int A, int engine) {
    if (engine != SFB200_GEMM_TC_3XTF32 || !tc_init()) return 0;
    if (!(K1 == 32 || K1 == 64) || H1 % 32 != 0 || H1 < 32 || H1 > PS_MAX_H1 || H2 % 128 != 0 || H2 < 128 || H2 > 512) return 0;
    if (A < 1 || A + 1 > kHeadAP) return 0;
    if (!tf32_lo_lookup(W1, (int64_t)H1 * K1) || !tf32_lo_lookup(W2, (int64_t)H2 * H1)) return 0;
    return 4 * (H2 / 128);
}

int tc_policy_mlp2_heads_forward(const float* x, int64_t ldx, int64_t M, int K1, const float* W1, const float* b1, int H1,
                                 const float* W2, const float* b2, int H2, int act, int engine, const float* Wv,
                                 const float* Wa, int A, float* head_part, cudaStream_t st) {
    if (!tc_policy_mlp2_supported(W1, W2, K1, H1, H2, A, engine)) return SFB_TC_UNSUPPORTED;
    if ((reinterpret_cast<uintptr_t>(x) & 15u) || ldx % 4 != 0 || (reinterpret_cast<uintptr_t>(head_part) & 15u) || !b1 || !b2 ||
        (reinterpret_cast<uintptr_t>(Wv) & 7u) || (reinterpret_cast<uintptr_t>(Wa) & 7u) || M < 1 || M > 0x7fffffff)
        return SFB_TC_UNSUPPORTED;
    if (tf32_lo_check_enabled()) {
        int rc = tf32_lo_check(W1, tf32_lo_lookup(W1, (int64_t)H1 * K1), (int64_t)H1 * K1, st);
        if (!rc) rc = tf32_lo_check(W2, tf32_lo_lookup(W2, (int64_t)H2 * H1), (int64_t)H2 * H1, st);
        if (rc) return rc;
    }
    CUtensorMap tx, tw1, tw2;
    bool ok = make_tmap(&tx, x, (uint64_t)K1, (uint64_t)M, (uint64_t)ldx, 32, 128);
    ok = ok && make_tmap(&tw1, W1, (uint64_t)K1, (uint64_t)H1, (uint64_t)K1, 32, 32);
    ok = ok && make_tmap(&tw2, W2, (uint64_t)H1, (uint64_t)H2, (uint64_t)H1, 32, 128);
    if (!ok) return SFB_TC_UNSUPPORTED;
    PsArgs a{M, K1, H1, H2, act, b1, b2, TcEpilogue{1, act, b2, nullptr, 0, Wv, Wa, A, head_part}};
#define SFB_PS(KAv)                                                                            \
    switch (act) {                                                                             \
        case SFB200_ACT_ELU: return launch_ps<KAv, SFB200_ACT_ELU>(tx, tw1, tw2, a, st);        \
        case SFB200_ACT_RELU: return launch_ps<KAv, SFB200_ACT_RELU>(tx, tw1, tw2, a, st);      \
        case SFB200_ACT_TANH: return launch_ps<KAv, SFB200_ACT_TANH>(tx, tw1, tw2, a, st);      \
        default: return launch_ps<KAv, SFB200_ACT_NONE>(tx, tw1, tw2, a, st);                   \
    }
    if (K1 == 64) { SFB_PS(2) }
    SFB_PS(1)
#undef SFB_PS
}

}  // namespace sfb

using namespace sfb;

extern "C" {

int sfb200_policy_mlp2_partials(const float* W1, const float* W2, int K1, int H1, int H2, int A, int engine) {
    return tc_policy_mlp2_supported(W1, W2, K1, H1, H2, A, engine);
}

int sfb200_policy_mlp2_heads_forward(const float* x, int64_t ldx, int64_t M, int K1, const float* W1, const float* b1, int H1,
                                     const float* W2, const float* b2, int H2, int act, int engine, const float* Wv,
                                     const float* Wa, int A, float* head_partials, void* stream) {
    SFB_CHECK_ARG(x && W1 && b1 && W2 && b2 && Wv && Wa && head_partials && M >= 0, "policy_mlp2_heads_forward: bad arguments");
    if (M == 0) return 0;
    const int rc = tc_policy_mlp2_heads_forward(x, ldx, M, K1, W1, b1, H1, W2, b2, H2, act, engine, Wv, Wa, A, head_partials,
                                                (cudaStream_t)stream);
    SFB_CHECK_ARG(rc != SFB_TC_UNSUPPORTED,
                  "policy_mlp2_heads_forward: model not covered (K1=%d H1=%d H2=%d A=%d engine=%d); "
                  "sfb200_policy_mlp2_partials() tells when to use the per-layer calls", K1, H1, H2, A, engine);
    return rc;
}

}  // extern "C"
