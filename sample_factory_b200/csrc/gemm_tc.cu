// wgmma / TMA GEMM engine for sm_90a (SFB200_GEMM_TC_3XTF32, SFB200_GEMM_TC_TF32).
//
//   C[m,n] = epilogue( sum_k A(m,k) * B(n,k) ),   fp32 in HBM, fp32 accumulate in registers.
//
// Precision: the tensor core has no fp32 MMA. tf32 keeps 10 mantissa bits, so a single pass is ~1e-3 relative -- not
// parity grade.  The 3xTF32 mode splits every operand element into  hi = a & ~0x1fff  (exactly representable in tf32)
// and  lo = (a - hi) & ~0x1fff  and issues  hi*hi'  into one accumulator and  hi*lo' + lo*hi'  into a second one (summed
// in the epilogue): each product is exact in fp32, the dropped lo*lo' term is 2^-22 relative, i.e. fp32-grade results.
// (Two accumulators keep the 2^-11 smaller cross terms apart from the large partial sums, which removes most of the
// roundings applied to them.)
//
// Work item = one 128 x 128 output tile (x split-K slice).  The kernel is persistent: the grid is the CTAs the device holds
// at once (one per SM), CTA b runs items b, b + grid, b + 2 grid, ... (a fixed schedule; no result depends on it).  Barriers
// are set up once per CTA, ring slots and mbarrier phases run on across items, and the producer does not wait for the
// consumers' epilogue: it loads the first stages of item i+1 while the epilogue of item i runs.
// 384 threads = three warpgroups:
//   warpgroup 0   : TMA producer (one thread): raw fp32 A and B tiles -> 3-slot shared-memory rings, mbarrier complete_tx
//   warpgroups 1-2: consumers.  Per k-block of 32 they split the raw tiles into tf32 hi / lo halves written K-major with the
//                   128B swizzle wgmma reads, release the raw stage to the producer, then each issues the wgmmas of its
//                   64 output rows (m64n128k8) -- while those run, the next k-block is split into the other conversion
//                   buffer -- and finally runs the epilogue from its accumulator registers.
// Operands may be K-major ([rows, K], K contiguous) or MN-major ([K, rows], rows contiguous): the backward GEMMs
// (dX = dZ.W, dW = dZ^T.X) read the activations in the layout the forward pass wrote them -- the split pass transposes
// MN-major tiles on the fly (tf32 wgmma reads K-major operands only).
// Split-K tiles write raw partial sums to a workspace that the SIMT engine's fixed-order reduce kernel sums.
#include <cuda.h>

#include <cstdlib>
#include <cudaTypedefs.h>

#include "common.cuh"
#include "gemm.h"
#include "heads_tail.cuh"
#include "tc_ptx.cuh"
#include "wgmma_tile.cuh"

namespace sfb {

// ------------------------------------------------------------------------------------------------ the kernel
// register budgets after the producer warpgroup hands its share to the consumers (the item loop's state does not fit
// beside two 64-register accumulators in 168): 128 x 40 + 256 x 232 = the 384 x 168 the launch gets
constexpr int kProducerRegs = 40;
constexpr int kConsumerRegs = 232;

// F16: the fp16-split engine (A K-major with a registered bound |A| <= a_bound[0], B a weight matrix with |w| < 255):
// A * 2^a_shift is split into fp16 hi + lo * 2^-11 pairs (22 significand bits like the tf32 pair, on the fp16 MMA path at
// twice the tf32 rate); B = W * 2^kF16WShift in the same form is the weight's registered fp16 twins, which tmap_b (a 3-D
// fp16 map, planes hi / lo) loads with the 128B swizzle straight into the layout wgmma reads.  A stage covers 64 k.
// B_MN only names the twin the host chose (the transposed one for dX = dz . W), so dX stays its own instantiation.
// RES: the residual epilogue (store_tile_residual), forward layout only.
//
// Mainloop: tf32 form: the split of stage kb+1 runs while the wgmmas of stage kb are in flight (two conversion buffers).
// fp16 forms: each warpgroup reads the raw fp32 A of its own 64 rows (128B-swizzled by TMA) straight into the register
// fragments of the register-A form of fp16 wgmma, splitting them on the way, and keeps two groups of wgmmas (half a stage
// each) in flight.  A and B have their own TMA rings: a raw slot goes back to the producer as soon as it is split or in
// registers, an fp16 B slot (the twin tiles the wgmmas read in place) once its wgmmas have completed.  Every accumulator
// receives the same wgmmas in the same k order as a serial loop would issue.
//
// DW16: the fp16 form of dW = dz^T . x (gemm_dw_f16_kernel): both operands are MN-major activations with registered
// bounds (a_bound, b_bound), in 32-k stages.  A goes into register fragments as in the fp16 form; the consumers split raw
// B into scaled fp16 hi / lo halves in the MN-major layout (split_tile_f16_mn, no transpose, three conversion buffers),
// which fp16 wgmma reads with its transpose bit set; the three MMAs and the output scaling are the fp16 form's, the
// epilogue the plain one.
template <bool A_MN, bool B_MN, bool SPLIT3, bool HEADS, bool F16, bool RES, bool DW16>
__device__ __forceinline__ void gemm_tc_body(const CUtensorMap& tmap_a, const CUtensorMap& tmap_b, float* __restrict__ C,
                                             int64_t ldc, int64_t M, int N, int K, int k_chunk, int splits,
                                             const TcEpilogue& epi, const float* __restrict__ a_bound,
                                             const float* __restrict__ b_bound, unsigned long long* __restrict__ trace) {
    static_assert(!F16 || (!A_MN && SPLIT3), "fp16-split engine: K-major activations, 3-pass");
    static_assert(!DW16 || (A_MN && B_MN && SPLIT3 && !HEADS && !F16 && !RES), "fp16 dW form: MN-major operands, plain epilogue");
    if (trace && threadIdx.x == 0) trace[blockIdx.x * kTraceWords + 8] = tc_now();
    using S = TcSmem<F16, DW16, HEADS>;
    constexpr int KBK = S::KBK;
    constexpr int SA = S::A_STAGES, SB = S::B_STAGES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_align_1024(smem_raw);
    uint8_t* conv = smem + S::CONV_OFF;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S::BARS_OFF);
    uint64_t* full_a = bars;                // A slot landed (count 1 + tx)
    uint64_t* empty_a = bars + SA;          // A slot split / in registers in every consumer thread (count 256)
    uint64_t* full_b = bars + 2 * SA;
    uint64_t* empty_b = bars + 2 * SA + SB; // B slot split (tf32) / read by the completed wgmmas (fp16), count 256
    int* s_last = reinterpret_cast<int*>(bars + 2 * (SA + SB));

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tiles_n = (N + TBN - 1) / TBN;
    const int tiles_per_z = tiles_n * (int)((M + TBM - 1) / TBM);
    const int items = tiles_per_z * splits;

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_a) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_b) : "memory");
        for (int s = 0; s < SA; ++s) {
            mbar_init(&full_a[s], 1);
            mbar_init(&empty_a[s], 256);
        }
        for (int s = 0; s < SB; ++s) {
            mbar_init(&full_b[s], 1);
            mbar_init(&empty_b[s], 256);
        }
        fence_barrier_init();
    }
    __syncthreads();
    // everything above is CTA-local setup: under programmatic dependent launch it overlaps the tail of the previous
    // kernel; global memory is only touched after the wait
    pdl_wait();
    pdl_trigger();
    if (trace && threadIdx.x == 0) trace[blockIdx.x * kTraceWords + 9] = tc_now();

    // g0: stages of the CTA's earlier items -- stage g = g0 + kb uses ring slots g % SA, g % SB (and conversion buffer g & 1
    // in the tf32 form, g % 3 in DW16)
    if (warp < 4) {
        // ===================================================== TMA producer
        setmaxnreg_dec<kProducerRegs>();
        if (threadIdx.x != 0) return;
        int g0 = 0;
        for (int item = blockIdx.x; item < items; item += gridDim.x) {
            const TileCoord tc = tile_coord(item, tiles_n, tiles_per_z, K, k_chunk, KBK);
            for (int kb = 0; kb < tc.num_kb; ++kb) {
                const int k0 = tc.k_begin + kb * KBK;
                const int g = g0 + kb;
                const int sa = g % SA, sb = g % SB;
                mbar_wait(&empty_a[sa], ((g / SA) & 1) ^ 1);
                if (trace && kb == 0) trace[item * kTraceWords + 6] = tc_now();
                mbar_expect_tx(&full_a[sa], S::A_RAW);
                uint8_t* pa = smem + sa * S::A_RAW;
                if (F16) {   // two swizzled [128 rows][32 k] boxes
                    tma_load_2d(pa, &tmap_a, &full_a[sa], k0, (int)tc.m0);
                    tma_load_2d(pa + TBM * 128, &tmap_a, &full_a[sa], k0 + 32, (int)tc.m0);
                } else if (DW16) {   // four swizzled [32 k][32 rows] boxes
                    for (int b = 0; b < TBM / 32; ++b) tma_load_2d(pa + b * 4096, &tmap_a, &full_a[sa], (int)tc.m0 + 32 * b, k0);
                } else if (A_MN) {
                    tma_load_2d(pa, &tmap_a, &full_a[sa], (int)tc.m0, k0);
                } else {
                    tma_load_2d(pa, &tmap_a, &full_a[sa], k0, (int)tc.m0);
                }
                mbar_wait(&empty_b[sb], ((g / SB) & 1) ^ 1);
                mbar_expect_tx(&full_b[sb], S::B_SLOT);
                uint8_t* pb = smem + S::B_RING + sb * S::B_SLOT;
                if (F16) tma_load_3d(pb, &tmap_b, &full_b[sb], k0, tc.n0, 0);   // [hi | lo] twin tiles
                else if (B_MN) tma_load_2d(pb, &tmap_b, &full_b[sb], tc.n0, k0);
                else tma_load_2d(pb, &tmap_b, &full_b[sb], k0, tc.n0);
            }
            if (trace) trace[item * kTraceWords + 7] = tc_now();
            g0 += tc.num_kb;
        }
        return;
    }

    // ===================================================== consumers
    setmaxnreg_inc<kConsumerRegs>();
    const int ct = threadIdx.x - 128;          // 0..255
    const int wg = ct >> 7;                    // 64-row half of the tile
    if constexpr (HEADS && F16) {
        // the [Wv; Wa] operand of the head partials, all N columns: written once, read by every item's epilogue
        fill_head_weights_f16(smem + S::HW_OFF, epi.head_wv, epi.head_wa, epi.head_A, N, 0, N, ct, 256);
        fence_proxy_async_smem();
        consumer_sync();
    }

    // fp16-split engine: binary shift of the A operand from its bound (written by an earlier kernel of the stream)
    const int a_shift = (F16 || DW16) ? f16_shift_for_bound(a_bound[0]) : 0;
    const float a_scale = pow2f_int(a_shift);
    const int b_shift = DW16 ? f16_shift_for_bound(b_bound[0]) : kF16WShift;
    const float b_scale = pow2f_int(b_shift);
    // tf32 form: split stage g into conversion buffer g & 1
    auto split_stage = [&](int g) {
        const int sa = g % SA, sb = g % SB;
        const uint8_t* pa = smem + sa * S::A_RAW;
        uint8_t* cv = conv + (g & 1) * S::CONV;
        mbar_wait(&full_a[sa], (g / SA) & 1);
        split_tile<A_MN, SPLIT3>(pa, cv, cv + S::A_HALF, ct);
        mbar_wait(&full_b[sb], (g / SB) & 1);
        split_tile<B_MN, SPLIT3>(smem + S::B_RING + sb * S::B_SLOT, cv + 2 * S::A_HALF, cv + 2 * S::A_HALF + S::B_HALF, ct);
        mbar_arrive(&empty_b[sb]);
        mbar_arrive(&empty_a[sa]);
        fence_proxy_async_smem();              // generic-proxy writes -> visible to the tensor core (async proxy)
    };
    // fp16 forms: the A fragments of half h of stage g in registers (F16: 32 k, the h-th swizzled box; DW16: 16 k).  The
    // A slot goes back to the producer once both halves are in registers.
    constexpr int KS = KBK / 32;   // k16 steps per half stage
    using Frags = F16Frags<KS>;
    auto load_frags = [&](int g, int h, Frags& f) {
        const int sa = g % SA;
        const uint8_t* pa = smem + sa * S::A_RAW;
        if (h == 0) mbar_wait(&full_a[sa], (g / SA) & 1);
        if constexpr (F16) load_a_frags_f16(pa + h * (TBM * 128), wg * 64, ct & 127, a_scale, f);
        else if constexpr (DW16) load_a_frags_f16_mn(pa, 16 * h, wg * 64, ct & 127, a_scale, f);
        if (h == 1) mbar_arrive(&empty_a[sa]);
    };
    // DW16: split raw B stage g into conversion buffer g % 3 (its hi / lo halves, MN-major), release the raw slot
    auto split_b = [&](int g) {
        const int sb = g % SB;
        uint8_t* cv = conv + (g % 3) * S::CONV;
        mbar_wait(&full_b[sb], (g / SB) & 1);
        split_tile_f16_mn(smem + S::B_RING + sb * S::B_SLOT, cv, cv + S::B_HALF, ct, b_scale);
        mbar_arrive(&empty_b[sb]);
        fence_proxy_async_smem();
    };
    // fp16 forms: the wgmmas of half h of stage g, A from the fragments f, as one committed group
    auto issue_f16 = [&](int g, int h, const Frags& f, float (&acc)[64], float (&cross)[64]) {
        if constexpr (F16) {
            const int sb = g % SB;
            const uint8_t* bt = smem + S::B_RING + sb * S::B_SLOT;
            const uint64_t db_hi = make_smem_desc(smem_u32(bt)) + (uint64_t)(64 >> 4) * h;   // 64 B: 32 k of fp16
            const uint64_t db_lo = make_smem_desc(smem_u32(bt + S::B_HALF)) + (uint64_t)(64 >> 4) * h;
            if (h == 0) mbar_wait(&full_b[sb], (g / SB) & 1);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < KS; ++k) {
                const uint64_t o = (uint64_t)(32 >> 4) * k;   // 32 B per k16 inside the swizzle row
                wgmma_m64n128k16_f16_rs<0>(acc, f.hi[k], db_hi + o);
                wgmma_m64n128k16_f16_rs<0>(cross, f.hi[k], db_lo + o);
                wgmma_m64n128k16_f16_rs<0>(cross, f.lo[k], db_hi + o);
            }
        } else {
            const uint8_t* cv = conv + (g % 3) * S::CONV;
            const uint64_t o = (uint64_t)(2048 >> 4) * h;   // a k-step of 16 is two 1024 B atoms
            wgmma_fence();
            wgmma_m64n128k16_f16_rs<1>(acc, f.hi[0], make_smem_desc_mn(smem_u32(cv)) + o);
            wgmma_m64n128k16_f16_rs<1>(cross, f.hi[0], make_smem_desc_mn(smem_u32(cv + S::B_HALF)) + o);
            wgmma_m64n128k16_f16_rs<1>(cross, f.lo[0], make_smem_desc_mn(smem_u32(cv)) + o);
        }
        wgmma_commit();
    };
    int g0 = 0;
    for (int item = blockIdx.x; item < items; item += gridDim.x) {
        const TileCoord tc = tile_coord(item, tiles_n, tiles_per_z, K, k_chunk, KBK);
        unsigned long long* tr = (trace && ct == 0) ? trace + item * kTraceWords : nullptr;
        if (tr) {
            tr[0] = tc_smid();
            tr[1] = blockIdx.x;
            tr[2] = tc_now();
            mbar_wait(&full_a[g0 % SA], (g0 / SA) & 1);   // (split_stage waits again: it passes at once)
            tr[3] = tc_now();
        }
        float acc[64], cross[64];
        if constexpr (F16 || DW16) {
            // Two groups of wgmmas in flight, a group being half a stage: half 0 of each stage is issued from the
            // fragment set fa, half 1 from fb; after each issue wait_group 1 retires the group before, whose fragment
            // set then takes the next half's A, and, when that group ended stage g-1, whose B slot (F16) goes back to
            // the producer.  F16: the warpgroups share nothing but the mbarriers.  DW16: both warpgroups read the whole
            // split B of a stage, so a consumer barrier follows each split (the wgmmas issued before keep running).
            Frags fa, fb;
            load_frags(g0, 0, fa);
            if constexpr (DW16) {
                split_b(g0);
                consumer_sync();
            }
#pragma unroll
            for (int i = 0; i < 64; ++i) acc[i] = cross[i] = 0.f;
            for (int kb = 0; kb < tc.num_kb; ++kb) {
                const int g = g0 + kb;
                issue_f16(g, 0, fa, acc, cross);
                wgmma_wait_1();
                if (F16 && kb > 0) mbar_arrive(&empty_b[(g - 1) % SB]);   // stage g-1's wgmmas are done with its B twins
                load_frags(g, 1, fb);
                issue_f16(g, 1, fb, acc, cross);
                wgmma_wait_1();
                if (kb + 1 < tc.num_kb) {
                    load_frags(g + 1, 0, fa);
                    if constexpr (DW16) {
                        split_b(g + 1);
                        consumer_sync();
                    }
                }
            }
            wgmma_wait_all();
            if (F16) mbar_arrive(&empty_b[(g0 + tc.num_kb - 1) % SB]);
        } else {
#pragma unroll
            for (int i = 0; i < 64; ++i) acc[i] = cross[i] = 0.f;
            split_stage(g0);
            consumer_sync();
            for (int kb = 0; kb < tc.num_kb; ++kb) {
                const int g = g0 + kb;
                const uint8_t* cv = conv + (g & 1) * S::CONV;
                const uint64_t da_hi = make_smem_desc(smem_u32(cv + wg * 64 * 128));
                const uint64_t da_lo = make_smem_desc(smem_u32(cv + S::A_HALF + wg * 64 * 128));
                const uint64_t db_hi = make_smem_desc(smem_u32(cv + 2 * S::A_HALF));
                const uint64_t db_lo = make_smem_desc(smem_u32(cv + 2 * S::A_HALF + S::B_HALF));
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < TBK / WG_K; ++k) {
                    const uint64_t o = (uint64_t)(32 >> 4) * k;   // 32 B per k-step of 8 tf32 inside the swizzle row
                    wgmma_m64n128k8_tf32(acc, da_hi + o, db_hi + o, 1);
                    if (SPLIT3) {
                        wgmma_m64n128k8_tf32(cross, da_hi + o, db_lo + o, 1);
                        wgmma_m64n128k8_tf32(cross, da_lo + o, db_hi + o, 1);
                    }
                }
                wgmma_commit();
                if (kb + 1 < tc.num_kb) split_stage(g + 1);    // overlaps the wgmmas just issued
                wgmma_wait_all();
                consumer_sync();                       // split g+1 complete, buffer g & 1 free for g+2, in both warpgroups
            }
        }
        g0 += tc.num_kb;
        if (tr) tr[4] = tc_now();
        if (F16 || DW16) {
            // (main + cross * 2^-11) * 2^-(operand shifts): exact power-of-two scalings
            const float out_scale = pow2f_int(-(a_shift + b_shift));
#pragma unroll
            // (a rounded product of its own: the straight-line epilogues must not contract it with their bias add)
            for (int i = 0; i < 64; ++i) acc[i] = __fmul_rn(fmaf(cross[i], 1.f / 2048.f, acc[i]), out_scale);
        } else if (SPLIT3) {
#pragma unroll
            for (int i = 0; i < 64; ++i) acc[i] += cross[i];
        }
        if (tr) tr[10] = tc_now_after(acc[63]);

        // the epilogue's mode and activation are chosen once per item; whole tiles (all of them at the learner's shapes)
        // then run straight-line code
        const int64_t row_base = tc.m0 + wg * 64 + ((ct >> 5) & 3) * 16 + (lane >> 2);
        if constexpr (HEADS && F16) {
            const uint32_t hw = smem_u32(smem + S::HW_OFF);
            switch (epi.act) {
                case SFB200_ACT_ELU: heads_tile_f16<SFB200_ACT_ELU>(acc, tc, row_base, lane, C, ldc, M, epi, hw, tr); break;
                case SFB200_ACT_RELU: heads_tile_f16<SFB200_ACT_RELU>(acc, tc, row_base, lane, C, ldc, M, epi, hw, tr); break;
                case SFB200_ACT_TANH: heads_tile_f16<SFB200_ACT_TANH>(acc, tc, row_base, lane, C, ldc, M, epi, hw, tr); break;
                default: heads_tile_f16<SFB200_ACT_NONE>(acc, tc, row_base, lane, C, ldc, M, epi, hw, tr); break;
            }
        } else if constexpr (HEADS) {
            switch (epi.act) {
                case SFB200_ACT_ELU: heads_tile<SFB200_ACT_ELU>(acc, tc, row_base, lane, C, ldc, M, N, epi, tr); break;
                case SFB200_ACT_RELU: heads_tile<SFB200_ACT_RELU>(acc, tc, row_base, lane, C, ldc, M, N, epi, tr); break;
                case SFB200_ACT_TANH: heads_tile<SFB200_ACT_TANH>(acc, tc, row_base, lane, C, ldc, M, N, epi, tr); break;
                default: heads_tile<SFB200_ACT_NONE>(acc, tc, row_base, lane, C, ldc, M, N, epi, tr); break;
            }
        }
        if constexpr (HEADS) {
            if (epi.fin_counters) {
                // last-arriving n-tile CTA of this 128-row block finishes the heads (threadFenceReduction pattern)
                const int mb = (int)(tc.m0 / TBM);
                __threadfence();
                consumer_sync();
                if (ct == 0) *s_last = (atomicAdd(&epi.fin_counters[mb], 1) == tiles_n - 1) ? 1 : 0;
                consumer_sync();
                if (*s_last) {
                    __threadfence();
                    const float pv = epi.fin.pv_scalar ? *epi.fin.pv_scalar : 0.f;
                    const uint64_t offset = epi.fin.offset_host + (epi.fin.offset_dev ? (uint64_t)*epi.fin.offset_dev : 0ull);
                    for (int r = ct >> 5; r < TBM; r += 8) {
                        const int64_t row = tc.m0 + r;
                        if (row < M) heads_finish_row(epi.head_part, 2 * tiles_n, M, row, lane, epi.fin, pv, offset);
                    }
                    if (ct == 0) epi.fin_counters[mb] = 0;
                }
            }
        } else if constexpr (RES) {
            if (tile_is_whole(tc, TBM, C, ldc, M, N, epi.aux, epi.ld_aux))
                store_tile_whole<3, SFB200_ACT_NONE>(acc, tc, row_base, lane, C, ldc, epi, tr);
            else
                store_tile_residual(acc, tc, row_base, lane, C, ldc, M, N, epi);
        } else {
            float* Cz = C + (splits > 1 ? (int64_t)tc.z * M * ldc : 0);
            const int mode = splits == 1 ? epi.mode : 0;
            if (!tile_is_whole(tc, TBM, Cz, ldc, M, N, mode == 2 ? epi.aux : nullptr, mode == 2 ? epi.ld_aux : 0))
                store_tile(acc, tc, row_base, lane, Cz, ldc, M, N, mode, epi);
            else if (mode == 1)
                store_tile_whole_act<1>(acc, tc, row_base, lane, Cz, ldc, epi, tr);
            else if (mode == 2)
                store_tile_whole_act<2>(acc, tc, row_base, lane, Cz, ldc, epi, tr);
            else
                store_tile_whole<0, SFB200_ACT_NONE>(acc, tc, row_base, lane, Cz, ldc, epi, tr);
        }
        if (tr) tr[5] = tc_now();
    }
}

template <bool A_MN, bool B_MN, bool SPLIT3, bool HEADS, bool F16 = false, bool RES = false>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                  float* __restrict__ C, int64_t ldc, int64_t M, int N, int K, int k_chunk, int splits, TcEpilogue epi,
                  const float* __restrict__ a_bound, unsigned long long* __restrict__ trace) {
    gemm_tc_body<A_MN, B_MN, SPLIT3, HEADS, F16, RES, false>(tmap_a, tmap_b, C, ldc, M, N, K, k_chunk, splits, epi, a_bound,
                                                             nullptr, trace);
}

// dW = dz^T . x in the fp16 form (DW16 above); b_bound: the registered bound of x
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_dw_f16_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                   float* __restrict__ C, int64_t ldc, int64_t M, int N, int K, int k_chunk, int splits, TcEpilogue epi,
                   const float* __restrict__ a_bound, unsigned long long* __restrict__ trace, const float* __restrict__ b_bound) {
    gemm_tc_body<true, true, true, false, false, false, true>(tmap_a, tmap_b, C, ldc, M, N, K, k_chunk, splits, epi, a_bound,
                                                              b_bound, trace);
}

// ------------------------------------------------------------------------------------------------ host side
static PFN_cuTensorMapEncodeTiled_v12000 g_encode = nullptr;
static int g_tc_state = 0;   // 0 unknown, 1 ok, -1 unavailable

bool tc_init() {
    if (g_tc_state != 0) return g_tc_state > 0;
    g_tc_state = -1;
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn ||
        qres != cudaDriverEntryPointSuccess) {
        cudaGetLastError();
        return false;
    }
    int dev = 0, major = 0, minor = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev) != cudaSuccess || major != 9 || minor != 0) {
        cudaGetLastError();
        return false;
    }
    g_encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
    g_tc_state = 1;
    return true;
}

// 2-D fp32 tensor map, without swizzle or with the 128B swizzle (box0 * 4 = 128 B then). dim0 = contiguous dim.
bool make_tmap(CUtensorMap* out, const float* base, uint64_t dim0, uint64_t dim1, uint64_t stride1_elems, uint32_t box0,
               uint32_t box1, bool swizzle128) {
    cuuint64_t gdim[2] = {dim0, dim1};
    cuuint64_t gstride[1] = {stride1_elems * sizeof(float)};
    cuuint32_t box[2] = {box0, box1};
    cuuint32_t estride[2] = {1, 1};
    CUresult r = g_encode(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), gdim, gstride, box, estride,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                          CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

// 3-D fp16 map over a weight's [hi | lo] twins, planes lo_offset elements apart, each plane [rows][K] row-major: box
// 64 k x box_rows rows x both planes with the 128B swizzle, i.e. two [box_rows][64 fp16] tiles in the K-major layout
// wgmma reads (what split_tile_f16 writes).  False when TMA cannot describe the twins (alignment).
bool make_tmap_f16_twins(CUtensorMap* out, const uint16_t* hi, int64_t lo_offset, uint64_t K, uint64_t rows,
                         uint32_t box_rows) {
    if ((reinterpret_cast<uintptr_t>(hi) & 15u) || (K * 2) % 16 != 0 || (lo_offset * 2) % 16 != 0 || lo_offset <= 0)
        return false;
    cuuint64_t gdim[3] = {K, rows, 2};
    cuuint64_t gstride[2] = {K * 2, (cuuint64_t)lo_offset * 2};
    cuuint32_t box[3] = {64, box_rows, 2};
    cuuint32_t estride[3] = {1, 1, 1};
    CUresult r = g_encode(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<uint16_t*>(hi), gdim, gstride, box, estride,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

// SFB200_TC_F16=0 turns the fp16-split engine off (every 3-pass GEMM then runs the tf32 split; A/B comparison)
static bool f16_enabled() {
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("SFB200_TC_F16");
        v = (e && e[0] == '0') ? 0 : 1;
    }
    return v == 1;
}

// SFB200_CHECK_F16=1: verify registered fp16 twins against the weights on the device before every use (debugging aid):
// the twins are what selects the fp16-split form, so a stale registration shows here
bool f16_check_enabled() {
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("SFB200_CHECK_F16");
        v = (e && e[0] == '1') ? 1 : 0;
    }
    return v == 1;
}

// debug trace of the calling host thread (sfb200_gemm_set_trace): the wgmma launches that follow stamp into it
static thread_local unsigned long long* g_gemm_trace = nullptr;
static thread_local int64_t g_gemm_trace_words = 0;

static bool operand_ok(const float* p, int64_t ld) {
    return ((reinterpret_cast<uintptr_t>(p) & 15u) == 0) && (ld % 4 == 0) && ld > 0;
}

template <bool A_MN, bool B_MN, bool SPLIT3, bool HEADS, bool F16, bool RES, bool DW16>
static auto tc_kernel() {
    if constexpr (DW16) return gemm_dw_f16_kernel;
    else return gemm_wgmma_kernel<A_MN, B_MN, SPLIT3, HEADS, F16, RES>;
}

template <bool A_MN, bool B_MN, bool SPLIT3, bool HEADS = false, bool F16 = false, bool RES = false, bool DW16 = false>
static int launch_tc(const CUtensorMap& ta, const CUtensorMap& tb, float* C, int64_t ldc, int64_t M, int N, int K,
                     int k_chunk, int splits, const TcEpilogue& epi, cudaStream_t st, const float* a_bound = nullptr,
                     const float* b_bound = nullptr) {
    auto kern = tc_kernel<A_MN, B_MN, SPLIT3, HEADS, F16, RES, DW16>();
    constexpr int smem = TcSmem<F16, DW16, HEADS>::TOTAL;
    static int ctas_per_sm = 0;   // of this instantiation: 1 (shared memory), asked rather than assumed
    if (!ctas_per_sm) {
        SFB_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        SFB_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas_per_sm, kern, TC_THREADS, (size_t)smem));
        SFB_CHECK_ARG(ctas_per_sm > 0, "gemm_wgmma_kernel does not fit on this device");
    }
    const int64_t items = ceil_div(N, TBN) * ceil_div(M, TBM) * splits;
    const int64_t resident = (int64_t)ctas_per_sm * sm_count();
    SFB_CHECK_ARG(!g_gemm_trace || items * kTraceWords <= g_gemm_trace_words,
                  "gemm trace buffer too small: %lld work items need %lld words", (long long)items,
                  (long long)(items * kTraceWords));
    const dim3 grid((unsigned)(items < resident ? items : resident));
    if constexpr (DW16)
        SFB_CUDA_OK(launch_pdl(kern, grid, dim3(TC_THREADS), (size_t)smem, st, ta, tb, C, ldc, M, N, K, k_chunk, splits, epi,
                               a_bound, g_gemm_trace, b_bound));
    else
        SFB_CUDA_OK(launch_pdl(kern, grid, dim3(TC_THREADS), (size_t)smem, st, ta, tb, C, ldc, M, N, K, k_chunk, splits, epi,
                               a_bound, g_gemm_trace));
    SFB_LAUNCH_OK();
    return 0;
}

// k of one split-K slice: whole stages; *splits becomes the slices that leaves (none of them empty)
static int split_k_chunk(int K, int* splits) {
    if (*splits <= 1) return K;
    const int k_chunk = (int)(ceil_div(ceil_div(K, *splits), TBK) * TBK);
    *splits = (int)ceil_div(K, k_chunk);
    return k_chunk;
}

// C[M,N] = epi( sum_k A(m,k) B(n,k) ). Returns SFB_TC_UNSUPPORTED when the shape/alignment is not covered.
static int gemm_tc(bool a_mn, const float* A, int64_t lda, bool b_mn, const float* B, int64_t ldb, float* C, int64_t ldc,
                   int64_t M, int N, int K, int splits, const TcEpilogue& epi, float* ws, bool split3, cudaStream_t st) {
    if (!tc_init()) return SFB_TC_UNSUPPORTED;
    if (!operand_ok(A, lda) || !operand_ok(B, ldb) || M < 1 || N < 8 || K < 8) return SFB_TC_UNSUPPORTED;
    if (M > 0x7fffffff || ceil_div(M, TBM) * ceil_div(N, TBN) * 64 > 0x7fffffff) return SFB_TC_UNSUPPORTED;
    // fp16-split engine: A is a K-major activation buffer with a registered bound, B a weight matrix with registered fp16
    // twins (the transposed twins when B is read MN-major, i.e. dX = dz . W: both registrations say that |w| < 255),
    // K a multiple of the 64-k stage.  The kernel reads B from the twins, so a twin TMA cannot describe keeps the tf32 form.
    if (!a_mn && split3 && splits == 1 && K % 64 == 0 && f16_enabled() && epi.mode != 3) {
        const float* a_bound = operand_bound_lookup(A, ((int64_t)(M - 1) * lda + K) * (int64_t)sizeof(float));
        F16Twin tw{nullptr, nullptr};
        if (a_bound) {
            if (!b_mn && ldb == K) tw = f16_twin_lookup(B, (int64_t)N * K);
            else if (b_mn && ldb == N) tw = f16_twinT_lookup(B, K, N);
        }
        // (B(n, k) is twin[n][k] in both cases: W[n][k] forward, the transposed twin [K_w][N_w] for dX)
        CUtensorMap ta16, tb16;
        if (tw.hi && make_tmap_f16_twins(&tb16, tw.hi, tw.lo - tw.hi, (uint64_t)K, (uint64_t)N, TBN) &&
            (!epi.head_part || !b_mn)) {
            if (f16_check_enabled()) {
                // B = W[N][K] row-major (forward) or W[K][N] row-major read along its other axis (dX: twins transposed)
                const int rc_chk = b_mn ? f16_twins_check(B, tw, K, N, true, st) : f16_twins_check(B, tw, N, K, false, st);
                if (rc_chk) return rc_chk;
            }
            if (!make_tmap(&ta16, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda, 32, TBM, true)) return SFB_TC_UNSUPPORTED;
            if (epi.head_part) return launch_tc<false, false, true, true, true>(ta16, tb16, C, ldc, M, N, K, K, 1, epi, st, a_bound);
            return b_mn ? launch_tc<false, true, true, false, true>(ta16, tb16, C, ldc, M, N, K, K, 1, epi, st, a_bound)
                        : launch_tc<false, false, true, false, true>(ta16, tb16, C, ldc, M, N, K, K, 1, epi, st, a_bound);
        }
    }
    CUtensorMap ta, tb;
    bool ok;
    if (a_mn) ok = make_tmap(&ta, A, (uint64_t)M, (uint64_t)K, (uint64_t)lda, TBM, TBK);
    else ok = make_tmap(&ta, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda, TBK, TBM);
    if (b_mn) ok = ok && make_tmap(&tb, B, (uint64_t)N, (uint64_t)K, (uint64_t)ldb, TBN, TBK);
    else ok = ok && make_tmap(&tb, B, (uint64_t)K, (uint64_t)N, (uint64_t)ldb, TBK, TBN);
    if (!ok) return SFB_TC_UNSUPPORTED;

    const int k_chunk = split_k_chunk(K, &splits);
    if (splits > 1 && !ws) return SFB_TC_UNSUPPORTED;
    float* out = splits > 1 ? ws : C;
    const int64_t ld_out = splits > 1 ? N : ldc;

    int rc;
    if (epi.mode == 3) {
        if (a_mn || b_mn || splits != 1) return SFB_TC_UNSUPPORTED;
        return split3 ? launch_tc<false, false, true, false, false, true>(ta, tb, C, ldc, M, N, K, K, 1, epi, st)
                      : launch_tc<false, false, false, false, false, true>(ta, tb, C, ldc, M, N, K, K, 1, epi, st);
    }
    if (epi.head_part) {
        if (a_mn || b_mn || splits != 1) return SFB_TC_UNSUPPORTED;
        rc = split3 ? launch_tc<false, false, true, true>(ta, tb, out, ld_out, M, N, K, k_chunk, splits, epi, st)
                    : launch_tc<false, false, false, true>(ta, tb, out, ld_out, M, N, K, k_chunk, splits, epi, st);
        return rc;
    }
    // fp16 form of dW = dz^T . x: both operands MN-major activations with registered bounds, split in the kernel
    const float* a_bound = nullptr;
    const float* b_bound = nullptr;
    if (a_mn && b_mn && split3 && epi.mode == 0 && f16_enabled()) {
        a_bound = operand_bound_lookup(A, ((int64_t)(K - 1) * lda + M) * (int64_t)sizeof(float));
        if (a_bound) b_bound = operand_bound_lookup(B, ((int64_t)(K - 1) * ldb + N) * (int64_t)sizeof(float));
    }
#define SFB_TC(AM, BM_)                                                                                          \
    (split3 ? launch_tc<AM, BM_, true>(ta, tb, out, ld_out, M, N, K, k_chunk, splits, epi, st)                 \
            : launch_tc<AM, BM_, false>(ta, tb, out, ld_out, M, N, K, k_chunk, splits, epi, st))
    CUtensorMap ta_sw;   // DW16: A in four swizzled [32 k][32 rows] boxes per stage
    if (b_bound && !make_tmap(&ta_sw, A, (uint64_t)M, (uint64_t)K, (uint64_t)lda, 32, TBK, true)) return SFB_TC_UNSUPPORTED;
    if (b_bound)
        rc = launch_tc<true, true, true, false, false, false, true>(ta_sw, tb, out, ld_out, M, N, K, k_chunk, splits, epi,
                                                                   st, a_bound, b_bound);
    else if (!a_mn && !b_mn) rc = SFB_TC(false, false);
    else if (!a_mn && b_mn) rc = SFB_TC(false, true);
    else if (a_mn && b_mn) rc = SFB_TC(true, true);
    else rc = SFB_TC(true, false);
#undef SFB_TC
    if (rc) return rc;
    if (splits > 1) return splitk_reduce(ws, splits, M, N, C, ldc, st);
    return 0;
}

int tc_linear_act_forward(const float* x, int64_t ldx, const float* W, const float* b, float* y, int64_t ldy, int64_t M,
                          int N, int K, int act, int engine, cudaStream_t st) {
    TcEpilogue epi{1, act, b, nullptr, 0};
    return gemm_tc(false, x, ldx, false, W, K, y, ldy, M, N, K, 1, epi, nullptr, engine == SFB200_GEMM_TC_3XTF32, st);
}

int tc_linear_residual_forward(const float* x, int64_t ldx, const float* W, const float* b, const float* r, int64_t ldr,
                               float* y, int64_t ldy, int64_t M, int N, int K, int engine, cudaStream_t st) {
    TcEpilogue epi{3, SFB200_ACT_NONE, b, r, ldr};
    return gemm_tc(false, x, ldx, false, W, K, y, ldy, M, N, K, 1, epi, nullptr, engine == SFB200_GEMM_TC_3XTF32, st);
}

// Number of head partials the fused forward produces per row for an N-wide layer, or 0 when the fused path does not
// cover the shape (callers then run the layer and the heads kernel separately).
int tc_linear_heads_partials(int N, int A, int engine) {
    if (engine == SFB200_GEMM_SIMT_FP32 || !tc_init()) return 0;
    if (N % TBN != 0 || N > 512 || A < 1 || A + 1 > kHeadAP) return 0;
    return 2 * (N / TBN);
}

int tc_linear_act_heads_forward(const float* x, int64_t ldx, const float* W, const float* b, float* y, int64_t ldy,
                                int64_t M, int N, int K, int act, int engine, const float* Wv, const float* Wa, int A,
                                float* head_part, cudaStream_t st, const HeadsFinish* fin, int* fin_counters) {
    if (tc_linear_heads_partials(N, A, engine) == 0 || !b) return SFB_TC_UNSUPPORTED;
    if (y && (ldy % 2 != 0 || (reinterpret_cast<uintptr_t>(y) & 7u))) return SFB_TC_UNSUPPORTED;
    if ((reinterpret_cast<uintptr_t>(head_part) & 15u) || (reinterpret_cast<uintptr_t>(Wv) & 7u) ||
        (reinterpret_cast<uintptr_t>(Wa) & 7u))
        return SFB_TC_UNSUPPORTED;
    TcEpilogue epi{1, act, b, nullptr, 0, Wv, Wa, A, head_part};
    if (fin && fin_counters) {
        epi.fin = *fin;
        epi.fin_counters = fin_counters;
    }
    return gemm_tc(false, x, ldx, false, W, K, y, y ? ldy : N, M, N, K, 1, epi, nullptr, engine == SFB200_GEMM_TC_3XTF32, st);
}

int tc_linear_backward(const float* dz, int64_t lddz, const float* x, int64_t ldx, const float* W, int64_t M, int N, int K,
                       int act_prev, float* dW, float* dx, int64_t lddx, int engine, float* ws, cudaStream_t st,
                       float* colsum_part, int* colsum_fused) {
    const bool split3 = engine == SFB200_GEMM_TC_3XTF32;
    // dW[n,k] = sum_m dz[m,n] x[m,k]: both operands are stored with the reduced index m as the row -> MN-major
    TcEpilogue none{0, 0, nullptr, nullptr, 0};
    const int splits = choose_splits(N, K, (int)M);
    int rc = dW ? gemm_tc(true, dz, lddz, true, x, ldx, dW, K, N, K, (int)M, splits, none, ws, split3, st) : 0;
    if (rc) return rc;
    (void)colsum_part;
    if (colsum_fused) *colsum_fused = 0;   // the caller reduces the columns of dx itself
    if (dx) {
        // dx[m,k] = (sum_n dz[m,n] W[n,k]) * act_prev'(x[m,k]): A = dz K-major, B(k, n) = W[n,k] MN-major
        TcEpilogue e{act_prev == SFB200_ACT_NONE ? 0 : 2, act_prev, nullptr, x, ldx};
        rc = gemm_tc(false, dz, lddz, true, W, K, dx, lddx, M, K, N, 1, e, nullptr, split3, st);
        if (rc) return rc;
    }
    return 0;
}

}  // namespace sfb

extern "C" int sfb200_tc_available(void) { return sfb::tc_init() ? 1 : 0; }

extern "C" int sfb200_gemm_work_item(int64_t item, int64_t M, int N, int K, int splits, int64_t* out) {
    SFB_CHECK_ARG(out && M > 0 && N > 0 && K > 0 && splits > 0, "gemm_work_item: bad arguments");
    const int k_chunk = sfb::split_k_chunk(K, &splits);
    const int tiles_n = (int)sfb::ceil_div(N, sfb::TBN);
    const int tiles_per_z = tiles_n * (int)sfb::ceil_div(M, sfb::TBM);
    SFB_CHECK_ARG(item >= 0 && item < (int64_t)tiles_per_z * splits, "gemm_work_item: item out of range");
    const sfb::TileCoord t = sfb::tile_coord((int)item, tiles_n, tiles_per_z, K, k_chunk, sfb::TBK);
    out[0] = t.m0, out[1] = t.n0, out[2] = t.k_begin, out[3] = t.num_kb * sfb::TBK, out[4] = t.z;
    out[5] = (int64_t)tiles_per_z * splits;
    return 0;
}

extern "C" int sfb200_gemm_set_trace(void* trace_dev, int64_t n_words) {
    sfb::g_gemm_trace = (unsigned long long*)trace_dev;
    sfb::g_gemm_trace_words = trace_dev ? n_words : 0;
    return 0;
}
