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
// fp16 form of the head partials: the B operand for 128 columns of [Wv; Wa] (fill_head_weights_f16)
constexpr int kHeadTileBytes = 8192;

// Shared memory of gemm_wgmma_kernel: a ring of A_STAGES TMA slots for the raw A tile, a ring of B_STAGES slots for the B
// tile, CONV_BUFS conversion buffers (the split of stage kb+1 is written into one while the wgmmas of earlier stages read
// the others), the mbarriers.
//   tf32 form: raw A / raw B fp32 tiles of 32 k (16 KB each, both released once split); two conversion buffers =
//              [A hi | A lo | B hi | B lo] (64 KB)
//   fp16 form: raw A fp32 tile of 64 k as two 128B-swizzled [128 rows][32 k] boxes (32 KB, released once the consumers
//              hold their fragments in registers); B = the weight tile's fp16 [hi | lo] twins, TMA-loaded in the swizzled
//              layout wgmma reads (32 KB, released once its wgmmas completed); no conversion buffer: 3 A + 4 B slots,
//              224 KB.  Four B slots: a warpgroup holds two (the stages in flight) while the producer fills the others.
//              With the heads folded in (HEADS): 2 A slots (an A slot is free once both halves are in registers) and
//              the [Wv; Wa] operand of the head partials (fill_head_weights_f16, N <= 512 columns: 32 KB), written once
//              per CTA: 224 KB.  (3 A + 3 B slots gave outputs that changed from launch to launch in rows of later items
//              even without the partials' wgmmas; the cause was not found, so the B ring keeps its four slots.)
//   fp16 dW form (DW16, gemm_dw_f16_kernel): raw MN-major A fp32 tile of 32 k as four 128B-swizzled [32 k][32 rows]
//              boxes (16 KB, released once in registers), raw MN-major B tile as in the tf32 form (16 KB, released once
//              split); three conversion buffers [B hi | B lo], each [32 k][128 rows] fp16 MN-major (8 KB): with two
//              stages of wgmmas in flight per warpgroup and the warpgroups up to a stage apart, three are read or
//              written at once.  4 A + 4 B slots: 176 KB.
template <bool F16, bool DW16 = false, bool HEADS = false>
struct TcSmem {
    static constexpr int KBK = F16 ? 64 : TBK;                    // k per stage
    static constexpr int A_STAGES = (F16 && HEADS) ? 2 : F16 ? 3 : DW16 ? 4 : 3;
    static constexpr int B_STAGES = (F16 || DW16) ? 4 : 3;
    static constexpr int A_RAW = TBM * KBK * 4;
    static constexpr int B_SLOT = F16 ? 2 * TBN * 64 * 2 : TBN * TBK * 4;
    // one split half of A (tf32 form): [128 rows][128 B] swizzled K-major
    static constexpr int A_HALF = TBM * 128;
    // one split half of B: tf32 form [128 rows][128 B] swizzled K-major; DW16 [32 k][128 rows] fp16 (split_tile_f16_mn)
    static constexpr int B_HALF = DW16 ? TBN * TBK * 2 : TBN * 128;
    static constexpr int CONV = F16 ? 0 : DW16 ? 2 * B_HALF : 2 * A_HALF + 2 * B_HALF;
    static constexpr int CONV_BUFS = F16 ? 0 : DW16 ? 3 : 2;
    static constexpr int B_RING = A_STAGES * A_RAW;               // offsets from the 1024-aligned base
    static constexpr int CONV_OFF = B_RING + B_STAGES * B_SLOT;
    static constexpr int HW_OFF = CONV_OFF + CONV_BUFS * CONV;   // fp16 form with heads: fill_head_weights_f16's layout
    static constexpr int BARS_OFF = HW_OFF + ((F16 && HEADS) ? (512 / TBN) * kHeadTileBytes : 0);
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
// common.cuh) in the swizzled K-major [rows][64 fp16] layout.  (The weight operand of dX comes from its transposed twins,
// gemm_tc.cu; dW's MN-major activations are split by split_tile_f16_mn below.)
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

// fp16 dW form: raw fp32 MN-major tile [32 k][128 rows] -> scaled fp16 hi / lo halves in the MN-major 128B-swizzled
// layout fp16 wgmma reads with its transpose bit set (make_smem_desc_mn): per half, atom (k / 8, rows / 64) is 1024 B at
// (rows / 64) * 4096 + (k / 8) * 1024, row k % 8 of it holds the 64 rows as eight 16 B chunks, chunk c at c ^ (k % 8).
// No transpose: a thread turns four consecutive rows at one k into 8 B of hi and 8 B of lo (a half-warp writes one whole
// 128 B row: no bank conflict).  ct = 0 .. 255.
__device__ __forceinline__ void split_tile_f16_mn(const uint8_t* raw, uint8_t* hi, uint8_t* lo, int ct, float scale) {
#pragma unroll
    for (int q = 0; q < (TBK * TBM / 4) / 256; ++q) {
        const int i = ct + 256 * q;
        const float4 v = reinterpret_cast<const float4*>(raw)[i];
        const int k = i >> 5, r = (i & 31) * 4;                    // k, rows r .. r+3
        const int c = (r >> 3) & 7;
        const uint32_t off = (uint32_t)((r >> 6) * 4096 + (k >> 3) * 1024 + (k & 7) * 128 + ((c ^ (k & 7)) << 4) + (r & 4) * 2);
        uint2 h, l;
        f16_split2(v.x * scale, v.y * scale, h.x, l.x);
        f16_split2(v.z * scale, v.w * scale, h.y, l.y);
        *reinterpret_cast<uint2*>(hi + off) = h;
        *reinterpret_cast<uint2*>(lo + off) = l;
    }
}

// A thread's fp16 A operand of half a stage in registers (the register-A form of fp16 wgmma): per k16 step the four
// .f16x2 words of its m64k16 fragment, hi and lo halves.  Word j holds rows row + 8 * (j & 1), k = k16 + 2 * (lane % 4) +
// 8 * (j / 2) + {0, 1} (element 0 in the low 16 bits), row = the warpgroup's first row + 16 * warp + lane / 4 -- the
// mma.m16n8k16 A layout, one warp per 16 rows.
template <int KS>
struct F16Frags {
    uint32_t hi[KS][4], lo[KS][4];
};

// fp16 form: fragments (32 k) of the rows from row0 (0 or 64) of a raw fp32 K-major [128 rows][32 k] box that TMA stored
// with the 128B swizzle, times scale, split by f16_split2: the bits split_tile_f16 writes.  lt = thread of the warpgroup.
// A warp's float2 loads cover eight rows of 32 B; the swizzle puts them in distinct 16 B columns pairwise, so each load
// is the two wavefronts its 256 B need.
__device__ __forceinline__ void load_a_frags_f16(const uint8_t* box, int row0, int lt, float scale, F16Frags<2>& f) {
    const int r = row0 + 16 * (lt >> 5) + ((lt & 31) >> 2), q = lt & 3;
#pragma unroll
    for (int s = 0; s < 2; ++s) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 x = *reinterpret_cast<const float2*>(box + sw128_offset(r + 8 * (j & 1), 16 * s + 2 * q + 8 * (j >> 1)));
            f16_split2(x.x * scale, x.y * scale, f.hi[s][j], f.lo[s][j]);
        }
    }
}

// fp16 dW form: the fragments of k = k16 .. k16+15 from a raw fp32 MN-major tile [32 k][128 rows] that TMA stored as four
// 128B-swizzled [32 k][32 rows] boxes (box b: rows 32b .. 32b+31; element (k, row) at b * 4096 + sw128_offset(k, row % 32)),
// the bits split_tile_f16_mn writes.  Scalar loads: a warp reads eight rows at four k, which the swizzle spreads over 32
// banks.
__device__ __forceinline__ void load_a_frags_f16_mn(const uint8_t* raw, int k16, int row0, int lt, float scale, F16Frags<1>& f) {
    const int r = row0 + 16 * (lt >> 5) + ((lt & 31) >> 2), q = lt & 3;
    const float* p = reinterpret_cast<const float*>(raw);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int m = r + 8 * (j & 1), k = k16 + 2 * q + 8 * (j >> 1);
        const float x0 = p[((m >> 5) * 4096 + sw128_offset(k, m & 31)) / 4];
        const float x1 = p[((m >> 5) * 4096 + sw128_offset(k + 1, m & 31)) / 4];
        f16_split2(x0 * scale, x1 * scale, f.hi[0][j], f.lo[0][j]);
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
// store_tile guards every element and takes the mode at run time: the epilogue of ragged tiles (and of every tile of the
// rollout's tf32 form).  Whole tiles of the GEMM engine take store_tile_whole below.
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

// The tile lies wholly inside C (and inside aux, when the epilogue reads it) and every pair of a thread is one aligned
// float2: the whole-tile epilogues below need no per-element guard.  rows = rows of the CTA's tile from tc.m0.
__device__ __forceinline__ bool tile_is_whole(const TileCoord& tc, int rows, const float* C, int64_t ldc, int64_t M, int N,
                                              const float* aux = nullptr, int64_t ld_aux = 0) {
    return tc.m0 + rows <= M && tc.n0 + TBN <= N && ldc % 2 == 0 && ld_aux % 2 == 0 &&
           ((reinterpret_cast<uintptr_t>(C) | reinterpret_cast<uintptr_t>(aux)) & 7u) == 0;
}

// A thread's 32 bias values (columns n0 + 8*c + 2*(lane%4) + {0, 1}, c = 0..15) in one batch of loads
__device__ __forceinline__ void load_bias_pairs(const float* bias, int n0, int lane, float (&b)[32]) {
    const float* p = bias + n0 + 2 * (lane & 3);
#pragma unroll
    for (int c = 0; c < 16; ++c) {
        b[2 * c] = __ldg(p + 8 * c);
        b[2 * c + 1] = __ldg(p + 8 * c + 1);
    }
}

// store_tile for a whole tile (tile_is_whole) with the mode (TcEpilogue::mode, 3 = residual) and the activation fixed at
// compile time: straight-line code, every global load of the thread (bias, the 32 float2 of aux) issued before the first
// multiply, then 32 float2 stores.  Per element the expressions are store_tile's / store_tile_residual's, so the bits are
// theirs.  tr: the traced thread's stamps (word 11: the loads have landed), else NULL.
template <int MODE, int ACT>
__device__ __forceinline__ void store_tile_whole(const float (&acc)[64], const TileCoord& tc, int64_t row_base, int lane,
                                                 float* C, int64_t ldc, const TcEpilogue& epi, unsigned long long* tr) {
    const int nq = tc.n0 + 2 * (lane & 3);
    float b[32];
    float2 h[32];
    if (MODE == 1 || MODE == 3) {
        if (epi.bias) {
            load_bias_pairs(epi.bias, tc.n0, lane, b);
        } else {
#pragma unroll
            for (int i = 0; i < 32; ++i) b[i] = 0.f;
        }
    }
    if (MODE == 2 || MODE == 3) {
        const float* ap = epi.aux + row_base * epi.ld_aux + nq;
#pragma unroll
        for (int j = 0; j < 32; ++j) h[j] = *reinterpret_cast<const float2*>(ap + (j & 1) * 8 * epi.ld_aux + 8 * (j >> 1));
    }
    if (tr) tr[11] = tc_now_after(MODE == 0 ? 0.f : MODE == 1 ? b[31] : h[31].y);
    float* cp = C + row_base * ldc + nq;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
        float v0 = acc[2 * j], v1 = acc[2 * j + 1];
        if (MODE == 1) {
            v0 = act_fwd_fast(__fadd_rn(v0, b[j & ~1]), ACT);
            v1 = act_fwd_fast(__fadd_rn(v1, b[j | 1]), ACT);
        } else if (MODE == 2) {
            v0 *= act_bwd_from_out(h[j].x, ACT);
            v1 *= act_bwd_from_out(h[j].y, ACT);
        } else if (MODE == 3) {
            v0 = __fadd_rn(__fadd_rn(v0, b[j & ~1]), h[j].x);
            v1 = __fadd_rn(__fadd_rn(v1, b[j | 1]), h[j].y);
        }
        *reinterpret_cast<float2*>(cp + (j & 1) * 8 * ldc + 8 * (j >> 1)) = make_float2(v0, v1);
    }
}

// store_tile_whole with the activation chosen once per tile
template <int MODE>
__device__ __forceinline__ void store_tile_whole_act(const float (&acc)[64], const TileCoord& tc, int64_t row_base, int lane,
                                                     float* C, int64_t ldc, const TcEpilogue& epi, unsigned long long* tr) {
    switch (epi.act) {
        case SFB200_ACT_ELU: store_tile_whole<MODE, SFB200_ACT_ELU>(acc, tc, row_base, lane, C, ldc, epi, tr); break;
        case SFB200_ACT_RELU: store_tile_whole<MODE, SFB200_ACT_RELU>(acc, tc, row_base, lane, C, ldc, epi, tr); break;
        case SFB200_ACT_TANH: store_tile_whole<MODE, SFB200_ACT_TANH>(acc, tc, row_base, lane, C, ldc, epi, tr); break;
        default: store_tile_whole<MODE, SFB200_ACT_NONE>(acc, tc, row_base, lane, C, ldc, epi, tr); break;
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
// Loads come in batches ahead of the math that uses them: the thread's 32 bias values once, then per (half, head row) the
// eight float2 of the weight row that both of the thread's rows (rs = 0, 1) multiply.  Each partial keeps its order of
// operations: FMAs over jj = 0..7, then the quad sum over lanes ^ 1, ^ 2.
// tr: the traced thread's stamps (11: bias landed, 12: y stored, 13: partials stored), else NULL.
// y = act(acc + bias) in place, stored into C (when not NULL) -- the first half of both heads epilogues
template <int ACT>
__device__ __forceinline__ void heads_act_tile(float (&acc)[64], const TileCoord& tc, int64_t row_base, int lane, float* C,
                                               int64_t ldc, int64_t M, const TcEpilogue& epi, unsigned long long* tr) {
    const int nq = tc.n0 + 2 * (lane & 3);
    float b[32];
    load_bias_pairs(epi.bias, tc.n0, lane, b);
    if (tr) tr[11] = tc_now_after(b[31]);
#pragma unroll
    for (int j = 0; j < 32; ++j) {
        acc[2 * j] = act_fwd_ct<ACT>(acc[2 * j] + b[j & ~1]);
        acc[2 * j + 1] = act_fwd_ct<ACT>(acc[2 * j + 1] + b[j | 1]);
        const int64_t m = row_base + 8 * (j & 1);
        if (C && m < M) *reinterpret_cast<float2*>(C + m * ldc + nq + 8 * (j >> 1)) = make_float2(acc[2 * j], acc[2 * j + 1]);
    }
    if (tr) tr[12] = tc_now_after(acc[63]);
}

template <int ACT>
__device__ __forceinline__ void heads_tile(float (&acc)[64], const TileCoord& tc, int64_t row_base, int lane, float* C,
                                           int64_t ldc, int64_t M, int N, const TcEpilogue& epi,
                                           unsigned long long* tr = nullptr) {
    constexpr int JP = 16;   // accumulator pairs of a thread per partial (per 64 columns)
    const int nq = tc.n0 + 2 * (lane & 3);
    heads_act_tile<ACT>(acc, tc, row_base, lane, C, ldc, M, epi, tr);
    const int p0 = (tc.n0 / TBN) * 2;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        float hp[2][kHeadAP];
#pragma unroll
        for (int a = 0; a < kHeadAP; ++a) {
            float s[2] = {0.f, 0.f};
            if (a <= epi.head_A) {
                const float* w = (a == 0 ? epi.head_wv : epi.head_wa + (int64_t)(a - 1) * N) + nq + 64 * half;
                float2 wv[JP / 2];
#pragma unroll
                for (int jj = 0; jj < JP / 2; ++jj) wv[jj] = __ldg(reinterpret_cast<const float2*>(w + 8 * jj));
#pragma unroll
                for (int jj = 0; jj < JP / 2; ++jj) {
#pragma unroll
                    for (int rs = 0; rs < 2; ++rs) {
                        const int j = JP * half + 2 * jj + rs;
                        s[rs] = fmaf(acc[2 * j], wv[jj].x, s[rs]);
                        s[rs] = fmaf(acc[2 * j + 1], wv[jj].y, s[rs]);
                    }
                }
            }
#pragma unroll
            for (int rs = 0; rs < 2; ++rs) {
                s[rs] += __shfl_xor_sync(0xffffffffu, s[rs], 1);
                s[rs] += __shfl_xor_sync(0xffffffffu, s[rs], 2);
                hp[rs][a] = s[rs];
            }
        }
#pragma unroll
        for (int rs = 0; rs < 2; ++rs) {
            const int64_t m = row_base + 8 * rs;
            if ((lane & 3) == 0 && m < M) {
                float4* dst = reinterpret_cast<float4*>(epi.head_part + ((int64_t)(p0 + half) * M + m) * kHeadPad);
                dst[0] = make_float4(hp[rs][0], hp[rs][1], hp[rs][2], hp[rs][3]);
                dst[1] = make_float4(hp[rs][4], hp[rs][5], hp[rs][6], hp[rs][7]);
                dst[2] = make_float4(hp[rs][8], 0.f, 0.f, 0.f);
            }
        }
    }
    if (tr) tr[13] = tc_now();
}

// ---- the head partials on the tensor cores (fp16 form) -------------------------------------------------------------
// The B operand of head_partials_f16 for columns [n_begin, n_begin + cols) of [Wv; Wa] (Wa's rows ld_wa floats apart),
// split as the weights' fp16 twins hold them (f16_split1 of w * 2^kF16WShift: the same bits).  Per 128-column tile
// (kHeadTileBytes at dst + (column / 128) * kHeadTileBytes) and k16 step kk (the tile's columns 64 h + 16 kk .. + 15 of
// both halves h): two MN-major 128B-swizzled atoms [8 k][64 n] (k = 0..7, then 8..15; the layout of split_tile_f16_mn)
// whose 64 n are, for half h, 32 h + a = hi and 32 h + 16 + a = lo of output row a (a = 0 .. 15, rows A+1 .. 15 zero).
// Threads t = 0 .. nthreads-1 of the caller share the work, a column each, its (up to kHeadAP) loads issued together; it
// is followed by fence_proxy_async_smem and a barrier before the first wgmma reads it.  cols: a multiple of 128.
__device__ __forceinline__ void fill_head_weights_f16(uint8_t* dst, const float* wv, const float* wa, int A, int64_t ld_wa,
                                                      int n_begin, int cols, int t, int nthreads) {
    for (int n = t; n < cols; n += nthreads) {
        float w[16];
#pragma unroll
        for (int a = 0; a < 16; ++a)
            w[a] = a == 0 ? wv[n_begin + n] : (a < kHeadAP && a <= A) ? wa[(int64_t)(a - 1) * ld_wa + n_begin + n] : 0.f;
        const int h = (n >> 6) & 1, kr = n & 7;   // half; k row inside the atom
        uint8_t* row = dst + (n >> 7) * kHeadTileBytes + ((n >> 4) & 3) * 2048 + ((n >> 3) & 1) * 1024 + kr * 128;
#pragma unroll
        for (int a = 0; a < 16; ++a) {
            uint16_t hi, lo;
            f16_split1(w[a] * (float)(1 << kF16WShift), hi, lo);
            const int nh = 32 * h + a, nl = nh + 16;
            *reinterpret_cast<uint16_t*>(row + ((((nh >> 3) ^ kr) & 7) << 4) + (nh & 7) * 2) = hi;
            *reinterpret_cast<uint16_t*>(row + ((((nl >> 3) ^ kr) & 7) << 4) + (nl & 7) * 2) = lo;
        }
    }
}

// The two head partials of a warpgroup's 64 x 128 tile of activated values y (a thread's 64 accumulator values, in the
// wgmma layout) in the 3-pass fp16 form: y * 2^s split into hi + lo * 2^-11 in registers -- the accumulator pairs of two
// adjacent n8 blocks are the register-A fragment of one k16 step -- times the [Wv; Wa] hi / lo operand at hw
// (fill_head_weights_f16, the tile's 8 KB), ((main + c1 * 2^-11) + c2 * 2^-11) * 2^-(s + kF16WShift) with main = y_hi . w_hi,
// c1 = y_hi . w_lo, c2 = y_lo . w_hi.  s is chosen per row and half from the row's own max |y| over the 64 columns
// (f16_shift_for_bound), so no bound has to be known and the bits of a row's partial depend on its 64 values and the
// weights only, whatever the tile shape around them.  Columns A+1 .. 15 come out 0.
// The MMAs are register-A wgmmas with B MN-major over the 64 rows of the operand: N = 128 is the GEMM engine's m64n128k16
// (LBO 0: columns 64 .. 127 repeat 0 .. 63 and are not read), N = 64 the m64n64k16 of the persistent rollout, whose
// larger live state across the step loop leaves no room for a 64-register accumulator; columns 0 .. 63 come out the
// same either way.  Per half, four k16 steps of y_hi give main in columns 32 h + 0..15 and y_hi . w_lo in 32 h + 16..31, then
// four of y_lo, from a fresh accumulator, give y_lo . w_hi in 32 h + 0..15.  Every pass writes junk into the other
// columns (the other half's weights), so the four passes run one after the other through one accumulator.
// hp[half][i]: row + 8 * ((i / 2) % 2), column 8 * (i / 4) + 2 * (lane % 4) + i % 2.  Every thread of the warpgroup calls it (wgmma is warpgroup-wide).
template <int N>
__device__ __forceinline__ void head_partials_f16(const float (&y)[64], uint32_t hw, float (&hp)[2][8]) {
    static_assert(N == 64 || N == 128, "m64n64k16 or m64n128k16");
    int shift[2][2];   // per half and row (rs: row + 8 rs)
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int rs = 0; rs < 2; ++rs) {
            float mx = 0.f;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                const int i = 32 * h + 4 * jj + 2 * rs;
                mx = fmaxf(mx, fmaxf(fabsf(y[i]), fabsf(y[i + 1])));
            }
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));   // the quad holds the row's 64 columns
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            shift[h][rs] = f16_shift_for_bound(mx);
        }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        F16Frags<4> f;   // the half's k16 steps (split here: the other half stays 32 values of y meanwhile)
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int i = 32 * h + 8 * kk + 2 * j;
                const float sc = pow2f_int(shift[h][j & 1]);
                f16_split2(y[i] * sc, y[i + 1] * sc, f.hi[kk][j], f.lo[kk][j]);
            }
        // Nothing may write a register the asynchronous wgmmas below read or accumulate into while they run: the
        // fragments are pinned complete before the fence (register arithmetic is not ordered by its memory clobber), and
        // the accumulator is not zero-filled but overwritten by the first wgmma of each pass (scale-d 0) -- a zero-fill the
        // compiler placed among the wgmmas corrupted whole rows of partials.
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int j = 0; j < 4; ++j) asm volatile("" : "+r"(f.hi[k][j]), "+r"(f.lo[k][j]));
        float d[N / 2];
        float (&part)[8] = hp[h];   // main + (y_hi . w_lo) * 2^-11, then + (y_lo . w_hi) * 2^-11, then scaled
#pragma unroll
        for (int pass = 0; pass < 2; ++pass) {
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const uint64_t db = make_smem_desc_mn(hw + kk * 2048, 0);
                if constexpr (N == 128) wgmma_m64n128k16_f16_rs<1>(d, pass ? f.lo[kk] : f.hi[kk], db, kk != 0);
                else wgmma_m64n64k16_f16_rs_mn(d, pass ? f.lo[kk] : f.hi[kk], db, kk != 0);
            }
            wgmma_commit();
            wgmma_wait_all();
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                if (pass == 0) part[i] = fmaf(d[16 * h + 8 + i], 1.f / 2048.f, d[16 * h + i]);
                else part[i] = __fmul_rn(fmaf(d[16 * h + i], 1.f / 2048.f, part[i]),
                                         pow2f_int(-(shift[h][(i >> 1) & 1] + kF16WShift)));
            }
        }
    }
}

// heads_tile of the fp16 form: y as there, the partials from head_partials_f16 (hw: the [Wv; Wa] operand of the whole
// layer, fill_head_weights_f16 from column 0).  A thread writes its columns of the kHeadPad row: 2q, 2q+1 and, for q < 2,
// 8 + 2q, 9 + 2q (q = lane % 4).
template <int ACT>
__device__ __forceinline__ void heads_tile_f16(float (&acc)[64], const TileCoord& tc, int64_t row_base, int lane, float* C,
                                               int64_t ldc, int64_t M, const TcEpilogue& epi, uint32_t hw,
                                               unsigned long long* tr) {
    heads_act_tile<ACT>(acc, tc, row_base, lane, C, ldc, M, epi, tr);
    const int p0 = (tc.n0 / TBN) * 2, q = lane & 3;
    float hp[2][8];
    head_partials_f16<128>(acc, hw + (uint32_t)(tc.n0 / TBN) * kHeadTileBytes, hp);
#pragma unroll
    for (int half = 0; half < 2; ++half)
#pragma unroll
        for (int rs = 0; rs < 2; ++rs) {
            const int64_t m = row_base + 8 * rs;
            if (m >= M) continue;
            float* dst = epi.head_part + ((int64_t)(p0 + half) * M + m) * kHeadPad + 2 * q;
            *reinterpret_cast<float2*>(dst) = make_float2(hp[half][2 * rs], hp[half][2 * rs + 1]);
            if (q < 2) *reinterpret_cast<float2*>(dst + 8) = make_float2(hp[half][4 + 2 * rs], hp[half][5 + 2 * rs]);
        }
    if (tr) tr[13] = tc_now();
}

}  // namespace sfb
