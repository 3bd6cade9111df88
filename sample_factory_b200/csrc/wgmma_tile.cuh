// Device-side building blocks of the wgmma GEMM tiles shared by the GEMM engine (gemm_tc.cu) and the persistent rollout
// (rollout_fused.cu): operand split passes into the swizzled
// K-major layout, tile coordinates and the register epilogues (bias + activation, activation derivative, head partials).
// sm_90a only.
#pragma once
#include "common.cuh"
#include "heads_tail.cuh"
#include "tc_ptx.cuh"

namespace sfb {

struct TcEpilogue {
    int mode;            // 0 plain, 1 act(acc + bias[n]), 2 acc * act'(aux[m,n]), 3 residual (store_tile_residual)
    int act;
    const float* bias;
    const float* aux;
    int64_t ld_aux;
    // fused policy/value heads (mode 1 only): partial dot products of the activated output row with [Wv ; Wa] over each
    // 64-column half of the tile -> head_part[(n_tile*2 + half)][m][kHeadPad]; C may be NULL (output row not stored)
    const float* head_wv;
    const float* head_wa;
    int head_A;
    float* head_part;
    // finish the heads inside this kernel: the n-tile CTAs of a 128-row block count themselves in fin_counters[m_block];
    // the one that arrives last sums the partials of its rows and runs the distribution tail (sampling, log-prob, ...) --
    // the separate finishing launch disappears.  fin_counters: M/128 zero-initialised ints, left at zero again.
    int* fin_counters;
    HeadsFinish fin;
};

constexpr int kHeadAP = 9;     // value + up to 8 action outputs
constexpr int kHeadPad = 12;   // floats per (partial, row): three 16 B stores
constexpr int TC_THREADS = 384;

// Shared memory of gemm_wgmma_kernel: a ring of A_STAGES TMA slots for the raw A tile, a ring of B_STAGES slots for the B
// tile, two conversion buffers (the split of stage kb+1 is written into one while the wgmmas of stage kb read the other),
// the mbarriers.
//   tf32 form: raw A / raw B fp32 tiles of 32 k (16 KB each, both released once split); conversion buffer =
//              [A hi | A lo | B hi | B lo] (64 KB)
//   fp16 form: raw A fp32 tile of 64 k (32 KB, released once split); B = the weight tile's fp16 [hi | lo] twins, TMA-loaded
//              in the swizzled layout wgmma reads (32 KB, released once its wgmmas completed); conversion buffer =
//              [A hi | A lo] (32 KB)
template <bool F16>
struct TcSmem {
    static constexpr int KBK = F16 ? 64 : TBK;                    // k per stage
    static constexpr int A_STAGES = F16 ? 2 : 3;
    static constexpr int B_STAGES = 3;
    static constexpr int A_RAW = TBM * KBK * 4;
    static constexpr int B_SLOT = F16 ? 2 * TBN * 64 * 2 : TBN * TBK * 4;
    static constexpr int A_HALF = TBM * 128;                      // one split half of A: [128 rows][128 B], swizzled K-major
    static constexpr int B_HALF = TBN * 128;
    static constexpr int CONV = F16 ? 2 * A_HALF : 2 * A_HALF + 2 * B_HALF;
    static constexpr int B_RING = A_STAGES * A_RAW;               // offsets from the 1024-aligned base
    static constexpr int CONV_OFF = B_RING + B_STAGES * B_SLOT;
    static constexpr int BARS_OFF = CONV_OFF + 2 * CONV;
    static constexpr int BARS = 2 * (A_STAGES + B_STAGES) * 8 + 16;
    static constexpr int TOTAL = 1024 /*align slack*/ + BARS_OFF + BARS;
    static_assert(TOTAL <= 227 * 1024, "shared memory");
};

// ELU via the fast exponential: |error| <= ~2.4e-7 absolute (2 ulp of exp on [0,1]) -- inside the 1e-5 parity budget
__device__ __forceinline__ float act_fwd_fast(float z, int act) {
    if (act == SFB200_ACT_ELU) return z > 0.f ? z : (__expf(z) - 1.f);
    return act_fwd(z, act);
}

__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// raw tile (TMA, no swizzle) -> tf32 hi / lo halves in the swizzled K-major layout.  K-major raw: [rows][32 k];
// MN-major raw: [32 k][rows] (transposed on the way).  ct = thread 0 .. THREADS-1 (ROWS = 64: one warpgroup's rows of a
// K-major tile, the pointers already offset to them).
template <bool MN, bool SPLIT3, int ROWS = TBM, int THREADS = 2 * ROWS>
__device__ __forceinline__ void split_tile(const uint8_t* raw, uint8_t* hi, uint8_t* lo, int ct) {
    static_assert(!MN || (ROWS == TBM && THREADS == 2 * TBM), "MN-major tiles: whole tiles only");
#pragma unroll
    for (int q = 0; q < (ROWS * TBK / 4) / THREADS; ++q) {
        const int i = ct + THREADS * q;
        const float4 v = reinterpret_cast<const float4*>(raw)[i];
        const float e[4] = {v.x, v.y, v.z, v.w};
        if (!MN) {
            const int r = i >> 3, c = i & 7;                           // row r, k = 4c .. 4c+3
            const uint32_t off = (uint32_t)(r * 128 + (((c ^ r) & 7) << 4));
            uint4 h, l;
            uint32_t* hp = &h.x;
            uint32_t* lp = &l.x;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint32_t w = __float_as_uint(e[j]);
                hp[j] = SPLIT3 ? (w & 0xffffe000u) : w;
                lp[j] = tf32_lo_bits(w);
            }
            *reinterpret_cast<uint4*>(hi + off) = h;
            if (SPLIT3) *reinterpret_cast<uint4*>(lo + off) = l;
        } else {
            // item i = (row r, 4-k chunk c): four scalar loads down column r of the [32 k][128 rows] raw tile (a warp
            // reads 32 consecutive rows of one k: 32 banks), one 16 B store per half (the 8 rows of a quarter-warp land
            // in 8 distinct swizzled chunks: no bank conflict)
            const int r = i & 127, c = i >> 7;
            const float* col = reinterpret_cast<const float*>(raw) + c * 4 * TBM + r;
            const uint32_t off = (uint32_t)(r * 128 + (((c ^ r) & 7) << 4));
            uint4 h, l;
            uint32_t* hp = &h.x;
            uint32_t* lp = &l.x;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint32_t w = __float_as_uint(col[j * TBM]);
                hp[j] = SPLIT3 ? (w & 0xffffe000u) : w;
                lp[j] = tf32_lo_bits(w);
            }
            *reinterpret_cast<uint4*>(hi + off) = h;
            if (SPLIT3) *reinterpret_cast<uint4*>(lo + off) = l;
        }
    }
}

// fp16-split engine: raw fp32 K-major tile [rows][64 k] -> scaled fp16 hi / lo halves (lo carries a 2^11 factor,
// common.cuh) in the swizzled K-major [rows][64 fp16] layout.  (MN-major operands never take the fp16 form: the weight
// operand of dX comes from its transposed twins instead, gemm_tc.cu.)
// ct, ROWS and THREADS as for split_tile.
template <bool MN, int ROWS = TBM, int THREADS = 2 * ROWS>
__device__ __forceinline__ void split_tile_f16(const uint8_t* raw, uint8_t* hi, uint8_t* lo, int ct, float scale) {
    static_assert(!MN, "fp16 split: K-major tiles only");
#pragma unroll 4
    for (int q = 0; q < (ROWS * 64 / 4) / THREADS; ++q) {
        const int i = ct + THREADS * q;
        const float4 v = reinterpret_cast<const float4*>(raw)[i];
        const int r = i >> 4, c4 = i & 15;                         // row r, k = 4*c4 .. 4*c4+3
        const uint32_t off = (uint32_t)(r * 128 + ((((c4 >> 1) ^ r) & 7) << 4) + (c4 & 1) * 8);
        uint2 h, l;
        f16_split2(v.x * scale, v.y * scale, h.x, l.x);
        f16_split2(v.z * scale, v.w * scale, h.y, l.y);
        *reinterpret_cast<uint2*>(hi + off) = h;
        *reinterpret_cast<uint2*>(lo + off) = l;
    }
}

struct TileCoord {
    int64_t m0;
    int n0, k_begin, num_kb, z;
};

// work item -> tile and split-K slice: n fastest, then m, then the slice, so the CTAs that run at the same time (consecutive
// items) share their A rows and the whole of B in L2
__host__ __device__ __forceinline__ TileCoord tile_coord(int tile, int tiles_n, int tiles_per_z, int K, int k_chunk, int kbk = TBK) {
    TileCoord t;
    t.z = tile / tiles_per_z;
    const int r = tile - t.z * tiles_per_z;
    const int mb = r / tiles_n;
    t.m0 = (int64_t)mb * TBM;
    t.n0 = (r - mb * tiles_n) * TBN;
    t.k_begin = t.z * k_chunk;
    const int k_end = (t.k_begin + k_chunk < K) ? t.k_begin + k_chunk : K;
    t.num_kb = (k_end - t.k_begin + kbk - 1) / kbk;
    return t;
}

// Epilogue of one warpgroup's 64 x 128 accumulator: pair j (j = 0..31) of a thread is d[2j], d[2j+1] = columns
// n0 + 8*(j/2) + 2*(lane%4) + {0, 1} of row  row_base + 8*(j%2).
__device__ __forceinline__ void store_tile(const float (&acc)[64], const TileCoord& tc, int64_t row_base, int lane, float* C,
                                           int64_t ldc, int64_t M, int N, int mode, const TcEpilogue& epi) {
    const bool v2 = (ldc % 2 == 0) && ((reinterpret_cast<uintptr_t>(C) & 7u) == 0);
#pragma unroll
    for (int j = 0; j < 32; ++j) {
        const int64_t m = row_base + 8 * (j & 1);
        const int n = tc.n0 + 8 * (j >> 1) + 2 * (lane & 3);
        if (m >= M || n >= N) continue;
        float v0 = acc[2 * j], v1 = acc[2 * j + 1];
        const bool two = n + 1 < N;
        if (mode == 1) {
            v0 = act_fwd_fast(v0 + (epi.bias ? epi.bias[n] : 0.f), epi.act);
            if (two) v1 = act_fwd_fast(v1 + (epi.bias ? epi.bias[n + 1] : 0.f), epi.act);
        } else if (mode == 2) {
            const float* h = epi.aux + m * epi.ld_aux + n;
            v0 *= act_bwd_from_out(h[0], epi.act);
            if (two) v1 *= act_bwd_from_out(h[1], epi.act);
        }
        float* dst = C + m * ldc + n;
        if (two && v2) {
            *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
        } else {
            dst[0] = v0;
            if (two) dst[1] = v1;
        }
    }
}

// Residual epilogue (a ResBlock's second conv plus its identity path, model/encoder.py:166-169): C = (acc + bias[n]) +
// aux[m, n].  A separate instantiation (gemm_wgmma_kernel<..., RES = true>), so the other epilogues keep their code.
__device__ __forceinline__ void store_tile_residual(const float (&acc)[64], const TileCoord& tc, int64_t row_base, int lane,
                                                    float* C, int64_t ldc, int64_t M, int N, const TcEpilogue& epi) {
#pragma unroll
    for (int j = 0; j < 32; ++j) {
        const int64_t m = row_base + 8 * (j & 1);
        const int n = tc.n0 + 8 * (j >> 1) + 2 * (lane & 3);
        if (m >= M || n >= N) continue;
        const float* r = epi.aux + m * epi.ld_aux + n;
        float* dst = C + m * ldc + n;
        dst[0] = (acc[2 * j] + epi.bias[n]) + r[0];
        if (n + 1 < N) dst[1] = (acc[2 * j + 1] + epi.bias[n + 1]) + r[1];
    }
}

// Epilogue with the policy/value heads folded in (forward layers feeding critic_linear / distribution_linear,
// actor_critic.py:171-186): y = act(acc + bias) is formed in registers, optionally stored, and contracted with the (A+1)
// head weight rows -- the separate heads kernel's re-read of y disappears.  Per 64-column half of the tile the four
// threads of a quad hold a row's 64 values; a fixed-order quad reduction gives the partial.  Two partials per tile.
template <int ACT>
__device__ __forceinline__ void heads_tile(float (&acc)[64], const TileCoord& tc, int64_t row_base, int lane, float* C,
                                           int64_t ldc, int64_t M, int N, const TcEpilogue& epi) {
    constexpr int JP = 16;   // accumulator pairs of a thread per partial (per 64 columns)
#pragma unroll
    for (int j = 0; j < 32; ++j) {
        const int n = tc.n0 + 8 * (j >> 1) + 2 * (lane & 3);
        acc[2 * j] = act_fwd_ct<ACT>(acc[2 * j] + epi.bias[n]);
        acc[2 * j + 1] = act_fwd_ct<ACT>(acc[2 * j + 1] + epi.bias[n + 1]);
        const int64_t m = row_base + 8 * (j & 1);
        if (C && m < M) *reinterpret_cast<float2*>(C + m * ldc + n) = make_float2(acc[2 * j], acc[2 * j + 1]);
    }
    const int p0 = (tc.n0 / TBN) * 2;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
#pragma unroll
        for (int rs = 0; rs < 2; ++rs) {
            float hp[kHeadAP];
#pragma unroll
            for (int a = 0; a < kHeadAP; ++a) {
                float s = 0.f;
                if (a <= epi.head_A) {
                    const float* w = a == 0 ? epi.head_wv : epi.head_wa + (int64_t)(a - 1) * N;
#pragma unroll
                    for (int jj = 0; jj < JP / 2; ++jj) {
                        const int j = JP * half + 2 * jj + rs;
                        const int n = tc.n0 + 8 * (j >> 1) + 2 * (lane & 3);
                        const float2 wv = __ldg(reinterpret_cast<const float2*>(w + n));
                        s = fmaf(acc[2 * j], wv.x, s);
                        s = fmaf(acc[2 * j + 1], wv.y, s);
                    }
                }
                s += __shfl_xor_sync(0xffffffffu, s, 1);
                s += __shfl_xor_sync(0xffffffffu, s, 2);
                hp[a] = s;
            }
            const int64_t m = row_base + 8 * rs;
            if ((lane & 3) == 0 && m < M) {
                float4* dst = reinterpret_cast<float4*>(epi.head_part + ((int64_t)(p0 + half) * M + m) * kHeadPad);
                dst[0] = make_float4(hp[0], hp[1], hp[2], hp[3]);
                dst[1] = make_float4(hp[4], hp[5], hp[6], hp[7]);
                dst[2] = make_float4(hp[8], 0.f, 0.f, 0.f);
            }
        }
    }
}

}  // namespace sfb
