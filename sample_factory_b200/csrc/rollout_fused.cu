// A whole rollout of the cfg-2 class of policies (two-layer MLP, Discrete actions, synthetic tape env) as ONE persistent
// kernel: `T` env steps x { layer-1 GEMM, layer-2 GEMM + head partials, heads finish + sampling + env step + post-step +
// pre-step of the next step } without leaving the SMs (batched_sampling.py:298-388 + inference_worker.py:313-341 +
// actor_critic.py:160-195 for every step of the rollout).
//
// Decomposition: all data dependencies of a step stay inside a block of BM env rows -- layer 2 needs all H1 columns of the
// block's h1, the heads need all H2 columns of its h2, the next step's layer 1 needs the block's new observations -- so a
// thread-block CLUSTER of CX = H2/BN CTAs owns a row block for the whole rollout and the only synchronisation is the
// cluster barrier (three per step); there is no grid-wide barrier and no kernel boundary.  CTA c of the cluster computes
// columns [BN c, BN c + BN) of h1, then of h2 (partial head products), then finishes rows [c BM/CX.., ) of the block.
// Hand-offs between the phases of a step, by layout:
//   h1, x_norm          every layout: global memory (L2-resident), read back by TMA.  fp16 form: h1 is written by TMA
//                       tile stores from shared-memory staging (store_h1_tma).  Each CTA loads its A tiles itself:
//                       multicasting them to both CTAs of a cluster measured slower (DESIGN §7).
//   head partials       fp16 form (both layouts): written by the layer-2 epilogue straight into the shared memory of the
//                       CTA that finishes the row (st.shared::cluster), summed from there by the tail; barrier 2 orders
//                       writer and reader, and barriers 3 and 1 of the next step come between the tail's reads and the
//                       next writes.  tf32 form: global memory.
//   b1, b2, [Wv; Wa] rows, bv, ba   fp16 form: copied into shared memory once per launch (this CTA's BN columns; [Wv; Wa]
//                       as the fp16 B operand of the tensor-core head partials), read from there by both epilogues and
//                       the tail.  tf32 form (no room beside its 104 KB slots): global.
// The CTA tile (rf_wide): BM x BN = 64 x 256 for H2 >= 256 (the two consumer warpgroups side by side on N over one 64-row
// A tile), 128 x 128 for H2 = 128 (the warpgroups stacked on M).  At H2 = 512 that makes clusters of two: a TPC is two SMs,
// so every GPC holds a whole number of them and the whole grid (64 clusters at 4096 envs) is resident at once.  Clusters
// of four strand two SMs in every GPC of 14 or 18 SMs: on the H100 measured (DESIGN §7) 30 of the 32 clusters of the
// old 128 x 128 decomposition were resident, and the last two ran as a second wave after the first.
//
// Each GEMM tile is the wgmma tile of gemm_tc.cu (3-pass split operands, main | cross accumulators in registers); the step
// tail samples with categorical_draw (heads_tail.cuh) and steps the env on the rules of step_tail.cuh, as
// sampler_tail_tape_kernel (heads.cu) does.
//
//   warps 0-3   TMA producer (one elected thread; the warpgroup gives its registers to the consumers).  It walks the
//               same sequence of ring uses as the consumers and puts the weight tiles, which do not depend on the step,
//               in flight across the cluster barriers: the first W2 tiles between its arrive at and its wait on barrier 1,
//               the next step's W1 tiles between its arrive at and its wait on barrier 2.  h1 and x_norm tiles are issued
//               only after the barrier that publishes them.
//   warps 4-11  two wgmma warpgroups (64 x 128 each): multiply, run the epilogues and the step tail (an 8-lane group per
//               row: four rows per warp).  One wgmma group stays in flight; a ring slot goes back to the producer when
//               its wgmmas have completed.
//
// fp16-split form (weights with registered fp16 twins, bounded activations): a stage covers 64 k.  The weight tiles are
// the twins, TMA-loaded in the swizzled layout wgmma reads.  The layer-1 epilogue stores h1 * 2^shift_h already split into
// fp16 [hi | lo] planes (the h1 scratch holds the hi plane, then the lo plane N*H1 halves later), so layer 2 -- 8 of the 9
// stages of a step at H1 = 512 -- is pure TMA -> wgmma.  Only x_norm (layer 1's A, written as fp32 by the step tail) is
// split in shared memory.  Every wgmma receives the operands the fp32 buffers would give after split_tile_f16.
// tf32 form: raw fp32 tiles of 32 k; the consumers split both operands (A into the conversion buffer, B into the back of
// its ring slot), as gemm_tc.cu's tf32 form does.
#include <cuda.h>

#include <cstdlib>

#include "common.cuh"
#include "gemm.h"
#include "heads_tail.cuh"
#include "step_tail.cuh"
#include "tc_ptx.cuh"
#include "wgmma_tile.cuh"

namespace sfb {

constexpr int RF_THREADS = 384;
constexpr int RF_HEAD_AP = 9;
constexpr int RF_MAX_DIM = 128;
constexpr int RF_TRACE_WORDS = 32;   // phase stamps per step (sfb200_rollout_set_trace)
// register budgets after the hand-over: 128 x 24 + 256 x 240 = the 384 x 168 the launch gets (the consumers hold the
// tensor-core head partials beside the step loop's state; the producer issues TMA loads only)
constexpr int RF_PRODUCER_REGS = 24;
constexpr int RF_CONSUMER_REGS = 240;

// CTA tile of a layer: BM x BN = 64 x 256 (warpgroup w: columns n0 + 128 w of the same 64 rows) for H2 >= 256, else
// 128 x 128 (warpgroup w: rows m0 + 64 w).  Same rule on the host (launch shape, TMA boxes) and in the kernel.
__host__ __device__ __forceinline__ bool rf_wide(int H2) { return H2 >= 256; }
__host__ __device__ __forceinline__ int rf_bm(int H2) { return rf_wide(H2) ? 64 : 128; }
__host__ __device__ __forceinline__ int rf_bn(int H2) { return rf_wide(H2) ? 256 : 128; }

// Ring slot of a stage (KBK k) for a BM x BN tile; all offsets multiples of 1024 B (the 128B swizzle atoms):
//   fp16 form: [A BM x 256 B | B hi BN x 128 B | B lo]: A = raw fp32 x_norm tile (layer 1) or the [hi | lo] h1 planes
//              (layer 2), B = the weight's [hi | lo] twin planes.  80 KB for 64 x 256, 64 KB for 128 x 128.
//   tf32 form: [A raw BM x 128 B | B raw BN x 128 B | B hi | B lo].  104 KB for 64 x 256, 64 KB for 128 x 128.
// Two slots: three 80 KB stages do not fit.  The conversion buffer [A hi | A lo] (BM x 256 B: the operands split in shared
// memory) follows the slots.  fp16 form: then a 16 KB staging buffer of the h1 store (store_h1_tma), the head partials of
// the rows this CTA finishes ([P][rows][kHeadPartPad] floats, P * rows = H2 / 64 * BM / CX = 256 in every layout: 12 KB)
// and the step-invariant operands of the CTA's BN <= 256 columns: b1, b2, the [Wv; Wa] operand of the head partials
// (fill_head_weights_f16: 16 rows x 256 columns, hi and lo planes, 16 KB), then bv, ba (16 floats).  The tf32 form has
// no room for them (two 104 KB slots).  The mbarriers and the normaliser statistics follow the largest layout.
template <bool F16>
struct RfSmem {
    static constexpr int STAGES = 2;
    static constexpr int KBK = F16 ? 64 : TBK;
    __host__ __device__ static constexpr int slot(int bm, int bn) { return F16 ? (bm + bn) * 256 : (bm + 3 * bn) * 128; }
    __host__ __device__ static constexpr int a_bytes(int bm) { return bm * KBK * 4; }   // A of a stage; B starts here
    __host__ __device__ static constexpr int b_hi(int bm, int bn) { return F16 ? bm * 256 : (bm + bn) * 128; }
    __host__ __device__ static constexpr int stage_tx(int bm, int bn) { return (bm + bn) * KBK * 4; }
    static constexpr int OFF_CONV_END = STAGES * slot(64, 256) + 64 * 256;   // the 64 x 256 layout's conversion buffer ends here
    static constexpr int OFF_PART = OFF_CONV_END + (F16 ? 64 * 256 : 0);
    static constexpr int OFF_B1 = OFF_PART + (F16 ? 256 * kHeadPartPad * 4 : 0);
    static constexpr int OFF_B2 = OFF_B1 + (F16 ? 256 * 4 : 0);
    static constexpr int OFF_HW = OFF_B2 + (F16 ? 256 * 4 : 0);
    static constexpr int OFF_HB = OFF_HW + (F16 ? (256 / TBN) * kHeadTileBytes : 0);
    static constexpr int OFF_BARS = OFF_HB + (F16 ? 16 * 4 : 0);   // full[STAGES], empty[STAGES]
    static constexpr int OFF_CSTAT = OFF_BARS + 64;
    static constexpr int TOTAL = OFF_CSTAT + 2 * RF_MAX_DIM * 4 + 1024 /*align slack*/;
    static_assert(2 * STAGES * 8 <= 64 && TOTAL + 64 <= 227 * 1024, "shared memory");
    static_assert(STAGES * slot(128, 128) + 128 * 256 <= OFF_PART, "the 128 x 128 layout fits below the partials");
    static_assert(a_bytes(64) % 1024 == 0 && slot(64, 256) % 1024 == 0 && OFF_CONV_END % 1024 == 0,
                  "h1 staging boxes (slot A regions, conversion buffer, the buffer after it) on 1024 B swizzle atoms");
    static_assert(OFF_HW % 1024 == 0, "the head operand on 1024 B swizzle atoms");
};


struct RolloutArgs {
    int64_t N; int T, K1, H1, H2;
    const float* b1; const float* b2; const float* wv; const float* wa; int A; const float* bv; const float* ba;
    float* h1; float* part; float* x_norm;
    // trajectory slots of step 0 (slot t = + t * per-step element count), row strides in elements
    float* values; int64_t values_rs; float* logits; int64_t logits_rs; float* actions; int64_t actions_rs;
    int32_t* env_actions; float* log_prob; int64_t lp_rs; float* pv_out; int64_t pv_rs; const float* pv_scalar;
    const float* noise; uint64_t seed; int64_t* sampler_step;
    // tape env
    const float* tape; int64_t tape_len; int64_t env_off; int term_period, trunc_period; int64_t* env_step;
    float* env_obs; float* env_rew; uint8_t* env_term; uint8_t* env_trunc;
    EpisodeArgs e;   // post step; the trajectory pointers at step 0 (slot t = + t)
    // pre step
    float* traj_obs; int64_t traj_obs_rs; const float* rnn; int rnn_dim; float* traj_rnn; int64_t traj_rnn_rs;
    ObsNorm n;
    // debug, or NULL: [T][RF_TRACE_WORDS] globaltimer stamps of CTA (0,0)'s first epilogue thread, then per CTA
    // (blockIdx.y * gridDim.x + blockIdx.x) four words: %smid, globaltimer at entry, after the programmatic-dependency
    // wait, at exit
    unsigned long long* trace;
    const float* bound_x; const float* bound_h1;   // fp16-split form: bounds of |x_norm| and |h1| (device floats), else NULL
};

__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_sync_all() {
    cluster_arrive();
    cluster_wait();
}
// generic-proxy global stores -> async-proxy (TMA) loads: the .global form is a single FENCE.VIEW.ASYNC.G; the unqualified
// form adds a MEMBAR.ALL.GPU (the cluster barrier's release already carries one)
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async.global;" ::: "memory"); }
__device__ __forceinline__ unsigned long long rf_now() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ uint32_t smid() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(r));
    return r;
}
// shared::cluster address of the same offset in the shared memory of CTA `rank` of the cluster
__device__ __forceinline__ uint32_t mapa_shared(uint32_t addr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
    return r;
}
__device__ __forceinline__ void st_cluster_f2(uint32_t addr, float2 v) {
    asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(v.x), "f"(v.y) : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}

// The ring: use u (counted from 0 over the whole rollout, identically by the producer and the consumers) lives in slot
// u % STAGES; its full / empty mbarriers are in phase (u / STAGES) & 1.  A step uses the ring K1/KBK + H1/KBK times
// (layer 1, then layer 2).
// TMA producer, run by all of warpgroup 0 (every warp takes part in the cluster barriers); `leader` issues the loads.
template <bool F16>
__device__ __forceinline__ void rf_produce(const CUtensorMap* tmap_x, const CUtensorMap* tmap_w1, const CUtensorMap* tmap_h1,
                                           const CUtensorMap* tmap_w2, int T, int K1, int H1, int bm, int bn, int m0, int n0,
                                           uint8_t* smem, uint64_t* full, uint64_t* empty, bool leader) {
    using S = RfSmem<F16>;
    constexpr int KBK = S::KBK;
    const int slot_bytes = S::slot(bm, bn), b_off = S::a_bytes(bm);
    const uint32_t stage_tx = (uint32_t)S::stage_tx(bm, bn);
    const int n1 = K1 / KBK, n2 = H1 / KBK;
    uint32_t pu = 0;   // next use to claim
    // claim the next use: wait until its slot is free, expect the whole stage, load the weight tile (B)
    auto weight = [&](const CUtensorMap* tb, int kb) {
        const uint32_t s = pu % S::STAGES;
        mbar_wait(&empty[s], ((pu / S::STAGES) & 1) ^ 1);
        mbar_expect_tx(&full[s], stage_tx);
        uint8_t* dst = smem + s * slot_bytes + b_off;
        if (F16) tma_load_3d(dst, tb, &full[s], 64 * kb, n0, 0);   // [hi | lo] twin tiles
        else tma_load_2d(dst, tb, &full[s], TBK * kb, n0);
        ++pu;
    };
    // the activation tile (A) of a claimed use
    auto activation = [&](uint32_t u, const CUtensorMap* ta, bool planes, int kb) {
        const uint32_t s = u % S::STAGES;
        if (planes) tma_load_3d(smem + s * slot_bytes, ta, &full[s], 64 * kb, m0, 0);   // [hi | lo] h1 tiles
        else tma_load_2d(smem + s * slot_bytes, ta, &full[s], KBK * kb, m0);
    };
    // Claims made before a cluster barrier only wait for slots the consumers free before they arrive there (uses of the
    // previous phase), so no claim can wait on the barrier it precedes: at most STAGES uses ahead.
    const int pre2 = n2 < S::STAGES ? n2 : S::STAGES;
    int pre1 = 0;   // W1 tiles of this step already in flight
    for (int t = 0; t < T; ++t) {
        // x_norm(t) is published (pre-step(0) before the launch, the tail of step t-1 before barrier 3)
        if (leader) {
            fence_proxy_async_all();
            const uint32_t u1 = pu - pre1;
            for (int j = 0; j < n1; ++j) {
                if (j >= pre1) weight(tmap_w1, j);
                activation(u1 + j, tmap_x, false, j);
            }
        }
        __syncwarp();
        cluster_arrive();                   // barrier 1: h1 of the row block complete
        const uint32_t u2 = pu;
        if (leader)
            for (int j = 0; j < pre2; ++j) weight(tmap_w2, j);
        __syncwarp();
        cluster_wait();
        if (leader) {
            fence_proxy_async_all();
            for (int j = 0; j < n2; ++j) {
                if (j >= pre2) weight(tmap_w2, j);
                activation(u2 + j, tmap_h1, F16, j);
            }
        }
        __syncwarp();
        cluster_arrive();                   // barrier 2: all head partials of the row block written
        pre1 = t + 1 < T ? (n1 < S::STAGES ? n1 : S::STAGES) : 0;
        if (leader)
            for (int j = 0; j < pre1; ++j) weight(tmap_w1, j);
        __syncwarp();
        cluster_wait();
        cluster_sync_all();                 // barrier 3: the next policy input complete
    }
}

// One BM x BN tile acc = A[m0.., :K] . B[n0.., :K]^T (nkb stages) by the 256 consumer threads (ct = 0..255), each
// warpgroup its 64 x 128 piece; `cu` the consumers' use counter.  SPLIT_A: the A tile is raw fp32, split here into the
// conversion buffer (each warpgroup its own 64 rows of a 128-row tile; both together the one 64-row tile of the wide
// layout, which both read); the tf32 form splits both operands.  3xTF32, or with F16 the fp16-split form of gemm_tc.cu
// (A * 2^a_shift, weights * 2^kF16WShift, 64 k per stage).  Every accumulator receives its wgmmas in k order.
// tr: the traced thread's stamps of this step, else NULL: slot s_land when the last stage has landed, s_split when its
// split is done (tiles that split), s_done when the last wgmmas have completed; s_each >= 0: slot s_each + kb when stage
// kb < 16 has landed (A and B complete one full barrier, so they land together here).
template <bool F16, bool SPLIT_A>
__device__ __forceinline__ void rf_tile(int nkb, bool wide, uint8_t* smem, uint64_t* full, uint64_t* empty, uint32_t& cu,
                                        float (&acc)[64], float (&cross)[64], int ct, int a_shift, unsigned long long* tr,
                                        int s_land, int s_split, int s_done, int s_each) {
    using S = RfSmem<F16>;
    const int wg = ct >> 7, lt = ct & 127;
    const int bm = wide ? 64 : 128, bn = wide ? 256 : 128;
    const int slot_bytes = S::slot(bm, bn), b_hi = S::b_hi(bm, bn);
    const int a_row = wide ? 0 : 64 * wg, b_row = wide ? 128 * wg : 0;   // this warpgroup's rows of the A / B tiles
    uint8_t* conv = smem + S::STAGES * slot_bytes;
    // (the first wgmmas overwrite them; defined values keep the accumulators from being live across the whole rollout)
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = cross[i] = 0.f;
    int held = -1;   // slot of the wgmma group still in flight
    for (int kb = 0; kb < nkb; ++kb, ++cu) {
        const int s = (int)(cu % S::STAGES);
        uint8_t* slot = smem + s * slot_bytes;
        mbar_wait(&full[s], (cu / S::STAGES) & 1);
        if (tr) {
            const unsigned long long now = rf_now();
            if (kb == nkb - 1) tr[s_land] = now;
            if (s_each >= 0 && kb < 16) tr[s_each + kb] = now;
        }
        const uint8_t* at = slot;
        if (SPLIT_A || !F16) {
            // the conversion buffer is read by the wgmmas in flight: this warpgroup's, and in the wide layout the other's
            if (held >= 0) {
                wgmma_wait_all();
                mbar_arrive(&empty[held]);
                held = -1;
                if (wide) consumer_sync();
            }
            if constexpr (F16) {
                if (wide) split_tile_f16<false, 64, 256>(slot, conv, conv + 8192, ct, pow2f_int(a_shift));
                else split_tile_f16<false, 64>(slot + wg * 64 * 256, conv + wg * 8192, conv + 16384 + wg * 8192, lt,
                                               pow2f_int(a_shift));
            } else if (wide) {
                split_tile<false, true, 64, 256>(slot, conv, conv + 8192, ct);
                split_tile<false, true, 256, 256>(slot + 8192, slot + b_hi, slot + b_hi + 32768, ct);
            } else {
                split_tile<false, true, 64>(slot + wg * 64 * 128, conv + wg * 8192, conv + 16384 + wg * 8192, lt);
                split_tile<false, true>(slot + 16384, slot + b_hi, slot + b_hi + 16384, ct);
            }
            fence_proxy_async_smem();
            consumer_sync();
            if (tr && kb == nkb - 1) tr[s_split] = rf_now();
            at = conv;
        }
        const uint64_t da_hi = make_smem_desc(smem_u32(at + a_row * 128));
        const uint64_t da_lo = make_smem_desc(smem_u32(at + bm * 128 + a_row * 128));
        const uint64_t db_hi = make_smem_desc(smem_u32(slot + b_hi + b_row * 128));
        const uint64_t db_lo = make_smem_desc(smem_u32(slot + b_hi + bn * 128 + b_row * 128));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < TBK / WG_K; ++k) {
            const uint64_t o = (uint64_t)(2 * k);
            if constexpr (F16) {
                wgmma_m64n128k16_f16(acc, da_hi + o, db_hi + o, (kb | k) != 0);
                wgmma_m64n128k16_f16(cross, da_hi + o, db_lo + o, (kb | k) != 0);
                wgmma_m64n128k16_f16(cross, da_lo + o, db_hi + o, 1);
            } else {
                wgmma_m64n128k8_tf32(acc, da_hi + o, db_hi + o, (kb | k) != 0);
                wgmma_m64n128k8_tf32(cross, da_hi + o, db_lo + o, (kb | k) != 0);
                wgmma_m64n128k8_tf32(cross, da_lo + o, db_hi + o, 1);
            }
        }
        wgmma_commit();
        if (held >= 0) {
            wgmma_wait_1();                  // the previous stage's wgmmas are done with its slot
            mbar_arrive(&empty[held]);
        }
        held = s;
    }
    wgmma_wait_all();
    if (tr) tr[s_done] = rf_now();
    mbar_arrive(&empty[held]);
    if (F16) {
        const float out_scale = pow2f_int(-(a_shift + kF16WShift));
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = fmaf(cross[i], 1.f / 2048.f, acc[i]) * out_scale;
    } else {
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] += cross[i];
    }
}

// Layer-1 epilogue of the fp16 form: h1 = act(acc + b1) exactly as store_tile forms it, times 2^shift_h, split by
// f16_split2 into the hi and lo planes of the h1 scratch -- the bits split_tile_f16 would make of the fp32 h1 tile.  bias:
// b1 of the warpgroup's first column n0 (the CTA's copy in shared memory).
// The values go through shared memory: each 64-column box of tmap_h1 (the [hi | lo] x BM rows x 64 k box layer 2 loads,
// 128B swizzle: the 16-byte chunk c of row r at chunk c ^ (r % 8), conflict-free for a warp's eight rows) is written in
// the layer-2 A layout and stored by one thread with a TMA tile store, which writes whole 128-byte lines (a warp's direct
// stores wrote eight 16-byte pieces) and clips the rows past N.  box[h]: the staging buffer of the warpgroup's box h
// (columns n0 + 64 h); rt: the thread's first row inside the tile; `issuer` stores the boxes of its warpgroup (64 x 256:
// each warpgroup its own two; 128 x 128: thread 0 the two boxes both warpgroups wrote).  Before box h is written, the
// consumer barrier of box h - 1 has passed; before box 0, rf_tile's last barrier (after layer 1's split): see the caller.
__device__ __forceinline__ void store_h1_tma(const float (&acc)[64], const CUtensorMap* tmap_h1, int n0, int m0, int rt,
                                             int lane, uint8_t* const (&box)[2], int plane_bytes, bool issuer,
                                             const float* bias, int act, float scale) {
    float b[32];
    const float* bp = bias + 2 * (lane & 3);
#pragma unroll
    for (int c = 0; c < 16; ++c) {
        b[2 * c] = bp[8 * c];
        b[2 * c + 1] = bp[8 * c + 1];
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
            const int j = 16 * h + jj;
            const int r = rt + 8 * (j & 1), c = (j >> 1) & 7;
            const float v0 = act_fwd_fast(acc[2 * j] + b[j & ~1], act);
            const float v1 = act_fwd_fast(acc[2 * j + 1] + b[j | 1], act);
            uint32_t hv, lv;
            f16_split2(v0 * scale, v1 * scale, hv, lv);
            uint8_t* dst = box[h] + r * 128 + (((c ^ r) & 7) << 4) + 4 * (lane & 3);
            *reinterpret_cast<uint32_t*>(dst) = hv;
            *reinterpret_cast<uint32_t*>(dst + plane_bytes) = lv;
        }
        fence_proxy_async_smem();   // these generic writes -> the TMA store's reads
        consumer_sync();
        if (issuer) {
            tma_store_3d(tmap_h1, box[h], n0 + 64 * h, m0, 0);
            bulk_commit();
        }
    }
}

// Layer-2 epilogue of the fp16 form: heads_tile_f16's arithmetic (same y, same head_partials_f16, so the same bits) with
// b2 and the [Wv; Wa] operand read from the CTA's copies in shared memory (`b2`: BN columns; `hw`: fill_head_weights_f16
// from the CTA's first column), and each row's two partials written into the shared memory of the cluster CTA that
// finishes the row: rows [c rpc, c rpc + rpc) of the block belong to CTA c, partial p of its row r at
// part + ((p * rpc + r) * kHeadPartPad) floats.  nl: the warpgroup's first column inside the CTA's tile; p0: its first
// partial (global column / 64); rb: the thread's first row inside the block.
template <int ACT>
__device__ __forceinline__ void rf_heads_tile(float (&acc)[64], int nl, int p0, int rb, int lane, const float* b2,
                                              uint32_t hw, uint32_t part, int rpc) {
    const int q = lane & 3, nq = nl + 2 * q;
    float b[32];
#pragma unroll
    for (int c = 0; c < 16; ++c) {
        b[2 * c] = b2[nq + 8 * c];
        b[2 * c + 1] = b2[nq + 8 * c + 1];
    }
#pragma unroll
    for (int j = 0; j < 32; ++j) {
        acc[2 * j] = act_fwd_ct<ACT>(acc[2 * j] + b[j & ~1]);
        acc[2 * j + 1] = act_fwd_ct<ACT>(acc[2 * j + 1] + b[j | 1]);
    }
    float hp[2][8];
    head_partials_f16<64>(acc, hw + (uint32_t)(nl / TBN) * kHeadTileBytes, hp);
#pragma unroll
    for (int half = 0; half < 2; ++half)
#pragma unroll
        for (int rs = 0; rs < 2; ++rs) {
            const int r = rb + 8 * rs;
            const uint32_t dst = mapa_shared(part + (uint32_t)((((p0 + half) * rpc + r % rpc) * kHeadPartPad + 2 * q) * 4),
                                             (uint32_t)(r / rpc));
            st_cluster_f2(dst, make_float2(hp[half][2 * rs], hp[half][2 * rs + 1]));
            if (q < 2) st_cluster_f2(dst + 32, make_float2(hp[half][4 + 2 * rs], hp[half][5 + 2 * rs]));
        }
}

template <int ACT, bool F16>
__global__ void __launch_bounds__(RF_THREADS, 1)
rollout_mlp2_tape_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w1,
                         const __grid_constant__ CUtensorMap tmap_h1, const __grid_constant__ CUtensorMap tmap_w2,
                         const RolloutArgs a) {
    using S = RfSmem<F16>;
    constexpr int KBK = S::KBK;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_align_1024(smem_raw);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + S::OFF_BARS);   // [STAGES] slot landed (TMA)
    uint64_t* empty = full + S::STAGES;                                  // [STAGES] slot read by every consumer's wgmmas
    float* cstat = reinterpret_cast<float*>(smem + S::OFF_CSTAT);       // [2][K1]: mu, 1 / sigma of the observation normaliser
    // fp16 form: the head partials of this CTA's rows, and its copies of the step-invariant operands (RfSmem)
    float* s_part = reinterpret_cast<float*>(smem + S::OFF_PART);
    float* s_b1 = reinterpret_cast<float*>(smem + S::OFF_B1);
    float* s_b2 = reinterpret_cast<float*>(smem + S::OFF_B2);
    uint8_t* s_hw = smem + S::OFF_HW;                                   // [Wv; Wa] operand of the head partials
    float* s_hb = reinterpret_cast<float*>(smem + S::OFF_HB);           // bv, then ba

    // episode statistics of finished episodes: accumulated per CTA over the WHOLE rollout in shared memory, five global
    // atomics per CTA at the end (inside this kernel every cluster barrier's release would otherwise have to wait for
    // hundreds of same-address atomics per step to drain)
    __shared__ double s_stats[5];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x < 5) s_stats[threadIdx.x] = 0.0;
    const int cx = (int)cluster_ctarank();           // == blockIdx.x (cluster spans the x dimension)
    const int CX = gridDim.x;
    const bool wide = rf_wide(a.H2);
    const int BM = rf_bm(a.H2), BN = rf_bn(a.H2);
    const int n0 = cx * BN;
    const int64_t m0 = (int64_t)blockIdx.y * BM;
    const int P = a.H2 / 64;                         // head partials per row: one per 64 columns
    const bool do_rms = a.n.mean != nullptr;
    unsigned long long* cta_trace =
        a.trace ? a.trace + (int64_t)a.T * RF_TRACE_WORDS + 4 * ((int64_t)blockIdx.y * gridDim.x + blockIdx.x) : nullptr;
    if (cta_trace && threadIdx.x == 0) {
        cta_trace[0] = smid();
        cta_trace[1] = rf_now();
    }

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_x) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_w1) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_h1) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_w2) : "memory");
        for (int s = 0; s < S::STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 256);
        }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();
    pdl_trigger();
    if (cta_trace && threadIdx.x == 0) cta_trace[2] = rf_now();
    if (do_rms) fill_col_stats(a.n, a.K1, cstat);
    if (F16) {   // the weights do not change inside a rollout: one copy per launch
        for (int i = threadIdx.x; i < BN; i += RF_THREADS) {
            s_b1[i] = a.b1[n0 + i];
            s_b2[i] = a.b2[n0 + i];
        }
        fill_head_weights_f16(s_hw, a.wv, a.wa, a.A, a.H2, n0, BN, threadIdx.x, RF_THREADS);
        fence_proxy_async_smem();   // -> the head partials' wgmmas
        if (threadIdx.x <= a.A) s_hb[threadIdx.x] = threadIdx.x == 0 ? a.bv[0] : a.ba[threadIdx.x - 1];
    }
    __syncthreads();
    const int64_t env_step0 = a.env_step[0];
    const uint64_t philox0 = a.sampler_step ? (uint64_t)*a.sampler_step : 0ull;

    if (warp < 4) {
        setmaxnreg_dec<RF_PRODUCER_REGS>();
        rf_produce<F16>(&tmap_x, &tmap_w1, &tmap_h1, &tmap_w2, a.T, a.K1, a.H1, BM, BN, (int)m0, n0, smem, full, empty,
                        threadIdx.x == 0);
    } else {
        setmaxnreg_inc<RF_CONSUMER_REGS>();
        const float pv = a.pv_scalar ? *a.pv_scalar : 0.f;
        // fp16-split form: binary shifts of the two activation operands from their bounds (constant over the rollout: the
        // weights, hence the bounds, do not change inside a rollout)
        const int shift_x = F16 ? f16_shift_for_bound(a.bound_x[0]) : 0;
        const int shift_h = F16 ? f16_shift_for_bound(a.bound_h1[0]) : 0;
        const bool tracer = a.trace != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 128;
#define RF_TRACE(slot) do { if (tracer) a.trace[(int64_t)t * RF_TRACE_WORDS + (slot)] = rf_now(); } while (0)
        uint32_t cu = 0;
        const TcEpilogue epi_heads{1, ACT, a.b2, nullptr, 0, a.wv, a.wa, a.A, a.part};
        const TcEpilogue epi_h1{1, ACT, a.b1, nullptr, 0};
        const int ct = threadIdx.x - 128;
        // this warpgroup's 64 x 128 piece of the CTA tile: rows m0 + 64 wg (128 x 128) or columns n0 + 128 wg (64 x 256)
        const int64_t row_base = m0 + (wide ? 0 : (ct >> 7) * 64) + ((ct >> 5) & 3) * 16 + (lane >> 2);
        TileCoord tc;
        tc.m0 = m0; tc.n0 = n0 + (wide ? (ct >> 7) * 128 : 0); tc.k_begin = 0; tc.num_kb = 0; tc.z = 0;

        // fp16 form: the staging buffers of the warpgroup's two h1 boxes (store_h1_tma), BM x 256 B each.  Free from the end
        // of layer 1's split to barrier 1: the A regions of the two ring slots (the x_norm tile was split out of its slot,
        // and h1 tiles land only after barrier 1), and in the 64 x 256 layout, for warpgroup 0, the buffer after the
        // conversion buffer and then the conversion buffer itself, which both warpgroups' layer-1 wgmmas read: the
        // barrier after its first box comes after both warpgroups have waited for those wgmmas.
        uint8_t* const conv = smem + S::STAGES * S::slot(BM, BN);
        uint8_t* const h1_box[2] = {wide && ct < 128 ? conv + BM * 256 : smem,
                                    wide && ct < 128 ? conv : smem + S::slot(BM, BN)};
        const bool h1_issuer = wide ? (ct & 127) == 0 : ct == 0;

        for (int t = 0; t < a.T; ++t) {
            RF_TRACE(0);
            unsigned long long* const tr = tracer ? a.trace + (int64_t)t * RF_TRACE_WORDS : nullptr;
            {
                float acc[64], cross[64];
                rf_tile<F16, true>(a.K1 / KBK, wide, smem, full, empty, cu, acc, cross, ct, shift_x, tr, 1, 2, 5, -1);
                if (F16) {
                    store_h1_tma(acc, &tmap_h1, tc.n0, (int)m0, (int)(row_base - m0), lane, h1_box, BM * 128, h1_issuer,
                                 s_b1 + (tc.n0 - n0), ACT, pow2f_int(shift_h));
                    RF_TRACE(6);           // staging written, last box store issued
                    // The h1 tiles were written by the async proxy (TMA stores), and the peers read them with TMA loads:
                    // once an issuer's bulk groups have completed, its writes are performed and visible to it, and its
                    // arrive (release) at barrier 1 below publishes them to the cluster (the loads follow the producers'
                    // acquire).  Nothing generic is left to order, so no proxy fence here; the issuers must not arrive
                    // before the wait.  The wait also frees the staging buffers (the next writes into the slot A regions
                    // are the TMA loads after barrier 1).
                    if (h1_issuer) bulk_wait_all();
                } else {
                    store_tile(acc, tc, row_base, lane, a.h1, a.H1, a.N, a.H1, 1, epi_h1);
                    RF_TRACE(6);               // epilogue stores issued
                    fence_proxy_async_all();   // h1 stores -> the peers' TMA loads
                }
                RF_TRACE(3);
            }
            cluster_sync_all();   // h1 of the row block complete
            RF_TRACE(4);
            {
                float acc[64], cross[64];
                rf_tile<F16, !F16>(a.H1 / KBK, wide, smem, full, empty, cu, acc, cross, ct, shift_h, tr, 11, 14, 12, 16);
                if (F16)
                    rf_heads_tile<ACT>(acc, tc.n0 - n0, tc.n0 / 64, (int)(row_base - m0), lane, s_b2, smem_u32(s_hw),
                                       smem_u32(s_part), BM / CX);
                else
                    heads_tile<ACT>(acc, tc, row_base, lane, nullptr, 0, a.N, a.H2, epi_heads);
                RF_TRACE(7);
            }
            cluster_sync_all();   // all head partials of the row block written
            RF_TRACE(8);

            // ===================================================== step tail: this CTA's share of the block's rows.
            // FOUR rows per warp at a time: an 8-lane group owns a row (one lane per action logit, the group leader also the value
            // and the env's scalars), so the 32 rows of a CTA are ONE pass of eight warps -- the per-row dependency chain (partial
            // sums from L2 -> softmax -> Philox -> argmax -> env rule -> stores, ~4.7 us measured) is paid once per step, not once
            // per row a warp owns.
            {
                const int g = lane & 7;                       // position inside the 8-lane group
                const int grp = lane >> 3;                    // which of the warp's four rows
                const int act_idx = (g + 7) & 7;              // action index held by this lane (position (a + 1) % 8)
                const bool has_logit = act_idx < a.A;
                const bool leader = g == 0;
                const bool last = (t + 1 == a.T);
                const int64_t step = env_step0 + t;
                const uint64_t offset = philox0 + (uint64_t)t;
                const float* src_step = a.tape + ((step + 1) % a.tape_len) * a.N * a.K1;
                const float* noise_t = a.noise ? a.noise + (int64_t)t * a.N * a.A : nullptr;
                const int rpc = BM / CX;                      // rows of the block this CTA finishes
                for (int base = 0; base < rpc; base += 32) {
                    const int rr = base + (warp - 4) * 4 + grp;
                    const int64_t row = m0 + cx * rpc + rr;
                    const bool ok = rr < rpc && row < a.N;
                    // ---- loads first: head partials, next observation (K1 / 8 floats per lane), episode accumulators
                    float x = 0.f, val = 0.f;
                    float ob[RF_MAX_DIM / 8];
                    const int cpl = a.K1 >> 3;                // observation columns per lane (K1 is a multiple of 32)
                    if (ok) {
                        // the fp16 form's partials are in this CTA's shared memory ([P][rpc] rows), the tf32 form's in L2
                        if (F16) {
                            if (has_logit)
                                for (int p = 0; p < P; ++p) x += s_part[(p * rpc + rr) * kHeadPartPad + 1 + act_idx];
                            if (leader)
                                for (int p = 0; p < P; ++p) val += s_part[(p * rpc + rr) * kHeadPartPad];
                        } else {
                            if (has_logit)
                                for (int p = 0; p < P; ++p) x += a.part[((int64_t)p * a.N + row) * kHeadPartPad + 1 + act_idx];
                            if (leader)
                                for (int p = 0; p < P; ++p) val += a.part[((int64_t)p * a.N + row) * kHeadPartPad];
                        }
                        const float4* src4 = reinterpret_cast<const float4*>(src_step + row * a.K1 + g * cpl);
#pragma unroll
                        for (int q = 0; q < RF_MAX_DIM / 32; ++q)
                            if (4 * q < cpl) {
                                const float4 f4 = src4[q];
                                ob[4 * q] = f4.x; ob[4 * q + 1] = f4.y; ob[4 * q + 2] = f4.z; ob[4 * q + 3] = f4.w;
                            }
                    }
                    const Episode ep = load_episode(a.e, row, ok && leader);
                    if (tr && base == 0) tr[13] = tc_now_after(val);   // partials landed
                    x += has_logit ? (F16 ? s_hb[1 + act_idx] : a.ba[act_idx]) : 0.f;
                    val += F16 ? s_hb[0] : a.bv[0];
                    float lp;
                    const int idx = categorical_draw<8>(x, act_idx, a.A, ok, noise_t, row * a.A, a.seed, offset, lp);
                    if (tr && base == 0) tr[15] = tc_now_after(lp);    // action sampled
                    if (!ok) continue;
                    // ---- trajectory slot t, env step, post step, pre step of t + 1
                    if (has_logit) a.logits[row * a.logits_rs + (int64_t)t * a.A + act_idx] = x;
                    float* obs_next = a.traj_obs + row * a.traj_obs_rs + (int64_t)(t + 1) * a.K1 + g * cpl;
                    float* env_o = a.env_obs + row * a.K1 + g * cpl;
                    float* xn = a.x_norm + row * a.K1 + g * cpl;
#pragma unroll
                    for (int q4 = 0; q4 < RF_MAX_DIM / 32; ++q4)
                        if (4 * q4 < cpl) {
                            const float4 f4 = make_float4(ob[4 * q4], ob[4 * q4 + 1], ob[4 * q4 + 2], ob[4 * q4 + 3]);
                            reinterpret_cast<float4*>(env_o)[q4] = f4;
                            reinterpret_cast<float4*>(obs_next)[q4] = f4;
                            if (!last) {
                                const int c = g * cpl + 4 * q4;
                                reinterpret_cast<float4*>(xn)[q4] =
                                    make_float4(a.n.apply(f4.x, do_rms, cstat, a.K1, c), a.n.apply(f4.y, do_rms, cstat, a.K1, c + 1),
                                                a.n.apply(f4.z, do_rms, cstat, a.K1, c + 2), a.n.apply(f4.w, do_rms, cstat, a.K1, c + 3));
                            }
                        }
                    if (a.rnn)
                        for (int j = g; j < a.rnn_dim; j += 8)
                            a.traj_rnn[row * a.traj_rnn_rs + (int64_t)(t + 1) * a.rnn_dim + j] = a.rnn[row * a.rnn_dim + j];
                    if (leader) {
                        const float r_raw = (float)idx / (float)a.A;
                        bool tm, to;
                        tape_done(step, a.env_off + row, a.term_period, a.trunc_period, tm, to);
                        a.values[row * a.values_rs + t] = val;
                        a.actions[row * a.actions_rs + t] = (float)idx;
                        a.env_actions[row] = idx;
                        a.log_prob[row * a.lp_rs + t] = lp;
                        a.pv_out[row * a.pv_rs + t] = pv;
                        a.env_rew[row] = r_raw;
                        a.env_term[row] = tm;
                        a.env_trunc[row] = to;
                        Episode fin;
                        if (post_step_env(a.e, row, row * a.e.stride + t, r_raw, tm, to, ep, fin) && a.e.stats) {
                            atomicAdd(&s_stats[0], 1.0); atomicAdd(&s_stats[1], (double)fin.ret);
                            atomicAdd(&s_stats[2], (double)fin.len); atomicAdd(&s_stats[3], (double)fin.mn);
                            atomicAdd(&s_stats[4], (double)fin.mx);
                        }
                    }
                }
                fence_proxy_async_all();   // x_norm stores -> the peers' TMA loads of the next step
                RF_TRACE(9);                          // tail done
            }

            cluster_sync_all();   // the row block's next policy input is complete; nobody still reads this step's partials
            RF_TRACE(10);
        }
#undef RF_TRACE
    }

    // every block has read the two step counters at its start; the last one to finish advances them by T
    __syncthreads();
    if (threadIdx.x < 5 && a.e.stats && s_stats[0] > 0.0) atomicAdd(a.e.stats + threadIdx.x, s_stats[threadIdx.x]);
    if (threadIdx.x == 0) {
        if (cta_trace) cta_trace[3] = rf_now();
        advance_step_counters(a.env_step, env_step0 + a.T, a.sampler_step, (int64_t)philox0 + a.T, gridDim.x * gridDim.y);
    }
}

// The launch configuration of rollout_mlp2_tape_kernel<ACT, F16> for N envs and hidden width H2 -- what the launch and the
// occupancy query (sfb200_rollout_occupancy) both use.  `attr` must outlive cfg.
template <int ACT, bool F16>
static int rollout_launch_config(int64_t N, int H2, cudaStream_t st, cudaLaunchConfig_t& cfg, cudaLaunchAttribute (&attr)[2]) {
    auto kern = rollout_mlp2_tape_kernel<ACT, F16>;
    static bool attr_set = false;
    if (!attr_set) {
        SFB_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, RfSmem<F16>::TOTAL));
        attr_set = true;
    }
    const int CX = H2 / rf_bn(H2);
    cfg = {};
    cfg.gridDim = dim3((unsigned)CX, (unsigned)ceil_div(N, rf_bm(H2)));
    cfg.blockDim = dim3(RF_THREADS);
    cfg.dynamicSmemBytes = RfSmem<F16>::TOTAL;
    cfg.stream = st;
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)CX;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_enabled() ? 2 : 1;
    return 0;
}

template <int ACT, bool F16>
static int launch_rollout(const CUtensorMap* tm, const RolloutArgs& a, cudaStream_t st) {
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute attr[2];
    const int rc = rollout_launch_config<ACT, F16>(a.N, a.H2, st, cfg, attr);
    if (rc) return rc;
    SFB_CUDA_OK(cudaLaunchKernelEx(&cfg, rollout_mlp2_tape_kernel<ACT, F16>, tm[0], tm[1], tm[2], tm[3], a));
    SFB_LAUNCH_OK();
    return 0;
}

// clusters the launch for N envs needs, and how many of them the device holds at once (cudaOccupancyMaxActiveClusters)
template <int ACT, bool F16>
static int rollout_occupancy(int64_t N, int H2, int* needed, int* resident) {
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute attr[2];
    const int rc = rollout_launch_config<ACT, F16>(N, H2, 0, cfg, attr);
    if (rc) return rc;
    SFB_CUDA_OK(cudaOccupancyMaxActiveClusters(resident, rollout_mlp2_tape_kernel<ACT, F16>, &cfg));
    *needed = (int)(cfg.gridDim.x * cfg.gridDim.y / attr[0].val.clusterDim.x);
    return 0;
}

// Covered: 3xTF32 engine, both weight matrices 16-byte aligned (TMA sources), K1 a multiple of 32 up to 128,
// H1 == H2 in {128, 256, 512}, <= 8 action outputs.
int tc_rollout_mlp2_supported(const float* W1, const float* W2, int K1, int H1, int H2, int A, int engine) {
    if (engine != SFB200_GEMM_TC_3XTF32 || !tc_init()) return 0;
    if (!(K1 == 32 || K1 == 64 || K1 == 96 || K1 == 128) || H1 != H2 || !(H2 == 128 || H2 == 256 || H2 == 512)) return 0;
    if (A < 1 || A + 1 > RF_HEAD_AP) return 0;
    if ((reinterpret_cast<uintptr_t>(W1) & 15u) || (reinterpret_cast<uintptr_t>(W2) & 15u)) return 0;
    return 2 * (H2 / 128);
}

// fp16-split form (common.cuh): taken when the weights have registered fp16 twins and both activation buffers (x_norm, the
// h1 scratch) have registered bounds -- the same rule as the per-layer GEMMs; SFB200_TC_F16=0 keeps the tf32 split
static bool rollout_f16_enabled() {
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("SFB200_TC_F16");
        v = (e && e[0] == '0') ? 0 : 1;
    }
    return v == 1;
}

#define SFB_RF_LAUNCH(F16v)                                                                  \
    switch (act) {                                                                           \
        case SFB200_ACT_ELU: return launch_rollout<SFB200_ACT_ELU, F16v>(tm, a, st);     \
        case SFB200_ACT_RELU: return launch_rollout<SFB200_ACT_RELU, F16v>(tm, a, st);   \
        case SFB200_ACT_TANH: return launch_rollout<SFB200_ACT_TANH, F16v>(tm, a, st);   \
        default: return launch_rollout<SFB200_ACT_NONE, F16v>(tm, a, st);                \
    }

static int g_rollout_form = -1;   // form of the last launch: 1 fp16 split, 0 tf32 split

int tc_rollout_mlp2_tape(const float* W1, const float* W2, int act, int engine, const RolloutArgs& a_in, cudaStream_t st) {
    if (!tc_rollout_mlp2_supported(W1, W2, a_in.K1, a_in.H1, a_in.H2, a_in.A, engine)) return SFB_TC_UNSUPPORTED;
    if ((reinterpret_cast<uintptr_t>(a_in.wv) & 7u) || (reinterpret_cast<uintptr_t>(a_in.wa) & 7u)) return SFB_TC_UNSUPPORTED;
    RolloutArgs a = a_in;
    const uint32_t BM = (uint32_t)rf_bm(a.H2), BN = (uint32_t)rf_bn(a.H2);   // TMA boxes: A tiles BM rows, weight tiles BN
    if (rollout_f16_enabled() && a.K1 % 64 == 0 && a.H1 % 64 == 0) {
        const F16Twin t1 = f16_twin_lookup(W1, (int64_t)a.H1 * a.K1), t2 = f16_twin_lookup(W2, (int64_t)a.H2 * a.H1);
        const float* bx = operand_bound_lookup(a.x_norm, a.N * a.K1 * (int64_t)sizeof(float));
        const float* bh = operand_bound_lookup(a.h1, a.N * a.H1 * (int64_t)sizeof(float));
        if (t1.hi && t2.hi && bx && bh) {
            if (f16_check_enabled()) {
                int rc = f16_twins_check(W1, t1, a.H1, a.K1, false, st);
                if (!rc) rc = f16_twins_check(W2, t2, a.H2, a.H1, false, st);
                if (rc) return rc;
            }
            a.bound_x = bx;
            a.bound_h1 = bh;
            // the h1 scratch (N x H1 floats) holds the split h1: hi plane [N][H1] halves, then the lo plane
            CUtensorMap tm[4];
            bool ok = make_tmap(&tm[0], a.x_norm, (uint64_t)a.K1, (uint64_t)a.N, (uint64_t)a.K1, 64, BM);
            ok = ok && make_tmap_f16_twins(&tm[1], t1.hi, t1.lo - t1.hi, (uint64_t)a.K1, (uint64_t)a.H1, BN);
            ok = ok && make_tmap_f16_twins(&tm[2], reinterpret_cast<const uint16_t*>(a.h1), a.N * a.H1, (uint64_t)a.H1,
                                           (uint64_t)a.N, BM);
            ok = ok && make_tmap_f16_twins(&tm[3], t2.hi, t2.lo - t2.hi, (uint64_t)a.H1, (uint64_t)a.H2, BN);
            if (ok) {   // (twins TMA cannot describe keep the tf32 form, as in gemm_tc)
                g_rollout_form = 1;
                SFB_RF_LAUNCH(true)
            }
        }
    }
    a.bound_x = a.bound_h1 = nullptr;
    CUtensorMap tm[4];
    bool ok = make_tmap(&tm[0], a.x_norm, (uint64_t)a.K1, (uint64_t)a.N, (uint64_t)a.K1, TBK, BM);
    ok = ok && make_tmap(&tm[1], W1, (uint64_t)a.K1, (uint64_t)a.H1, (uint64_t)a.K1, TBK, BN);
    ok = ok && make_tmap(&tm[2], a.h1, (uint64_t)a.H1, (uint64_t)a.N, (uint64_t)a.H1, TBK, BM);
    ok = ok && make_tmap(&tm[3], W2, (uint64_t)a.H1, (uint64_t)a.H2, (uint64_t)a.H1, TBK, BN);
    if (!ok) return SFB_TC_UNSUPPORTED;
    g_rollout_form = 0;
    SFB_RF_LAUNCH(false)
}
#undef SFB_RF_LAUNCH

}  // namespace sfb

using namespace sfb;

extern "C" {

static unsigned long long* g_rollout_trace = nullptr;
/* debug: device buffer of T x 16 uint64 that the next rollouts fill with phase time stamps (NULL switches it off) */
int sfb200_rollout_set_trace(void* trace_dev) {
    g_rollout_trace = (unsigned long long*)trace_dev;
    return 0;
}

int sfb200_rollout_last_form(void) { return g_rollout_form; }

int sfb200_rollout_occupancy(int64_t n_envs, int K1, int H1, int H2, int A, int engine, int act, int* clusters_needed,
                             int* clusters_resident) {
    SFB_CHECK_ARG(n_envs > 0 && clusters_needed && clusters_resident, "rollout_occupancy: bad arguments");
    SFB_CHECK_ARG(tc_rollout_mlp2_supported(nullptr, nullptr, K1, H1, H2, A, engine),
                  "rollout_occupancy: model not covered (K1=%d H1=%d H2=%d A=%d engine=%d)", K1, H1, H2, A, engine);
    // the instance a launch with registered fp16 twins and bounds takes
    if (rollout_f16_enabled() && K1 % 64 == 0 && H1 % 64 == 0) {
        switch (act) {
            case SFB200_ACT_ELU: return rollout_occupancy<SFB200_ACT_ELU, true>(n_envs, H2, clusters_needed, clusters_resident);
            case SFB200_ACT_RELU: return rollout_occupancy<SFB200_ACT_RELU, true>(n_envs, H2, clusters_needed, clusters_resident);
            case SFB200_ACT_TANH: return rollout_occupancy<SFB200_ACT_TANH, true>(n_envs, H2, clusters_needed, clusters_resident);
            default: return rollout_occupancy<SFB200_ACT_NONE, true>(n_envs, H2, clusters_needed, clusters_resident);
        }
    }
    switch (act) {
        case SFB200_ACT_ELU: return rollout_occupancy<SFB200_ACT_ELU, false>(n_envs, H2, clusters_needed, clusters_resident);
        case SFB200_ACT_RELU: return rollout_occupancy<SFB200_ACT_RELU, false>(n_envs, H2, clusters_needed, clusters_resident);
        case SFB200_ACT_TANH: return rollout_occupancy<SFB200_ACT_TANH, false>(n_envs, H2, clusters_needed, clusters_resident);
        default: return rollout_occupancy<SFB200_ACT_NONE, false>(n_envs, H2, clusters_needed, clusters_resident);
    }
}

int sfb200_rollout_mlp2_partials(const float* W1, const float* W2, int K1, int H1, int H2, int A, int engine) {
    return tc_rollout_mlp2_supported(W1, W2, K1, H1, H2, A, engine);
}

int sfb200_rollout_mlp2_tape(int64_t n_envs, int T, int K1, const float* W1, const float* b1, int H1, const float* W2,
                             const float* b2, int H2, int act, int engine, const float* Wv, const float* bv, const float* Wa,
                             const float* ba, int A, float* h1_scratch, float* head_partials, float* x_norm,
                             float* values_0, int64_t values_stride, float* logits_0, int64_t logits_stride,
                             const float* noise, uint64_t philox_seed, int64_t* sampler_step, float* actions_0,
                             int64_t actions_stride, int32_t* env_actions, float* log_prob_0, int64_t log_prob_stride,
                             const float* policy_version_scalar, float* policy_version_0, int64_t pv_stride,
                             const float* tape, int64_t tape_len, int64_t env_index_offset, int term_period, int trunc_period,
                             int64_t* env_step_counter, float* env_obs, float* env_rew, uint8_t* env_terminated,
                             uint8_t* env_truncated, float reward_scale, float reward_clip, int32_t policy_id,
                             float* traj_rewards_0, uint8_t* traj_dones_0, uint8_t* traj_time_outs_0, int32_t* traj_policy_id_0,
                             int64_t traj_stride, float* ep_return, int32_t* ep_len, float* ep_min_raw, float* ep_max_raw,
                             int32_t len_increment, double* stats, float* fin_return_0, int32_t* fin_len_0, float* traj_obs_0,
                             int64_t traj_obs_stride, const float* rnn, int rnn_dim, float* traj_rnn_0, int64_t traj_rnn_stride,
                             const double* mean, const double* var, float sub_mean, float inv_scale, float eps, float clip,
                             void* stream) {
    SFB_CHECK_ARG(n_envs > 0 && T > 0 && W1 && b1 && W2 && b2 && Wv && bv && Wa && ba && h1_scratch && head_partials && x_norm,
                  "rollout_mlp2_tape: bad model arguments");
    SFB_CHECK_ARG(values_0 && logits_0 && actions_0 && env_actions && log_prob_0 && policy_version_0 && policy_version_scalar,
                  "rollout_mlp2_tape: bad heads arguments");
    SFB_CHECK_ARG(tape && tape_len > 0 && term_period > 0 && trunc_period > 0 && env_step_counter && env_obs && env_rew &&
                      env_terminated && env_truncated, "rollout_mlp2_tape: bad env arguments");
    SFB_CHECK_ARG(traj_rewards_0 && traj_dones_0 && traj_time_outs_0 && traj_policy_id_0 && traj_obs_0,
                  "rollout_mlp2_tape: bad trajectory arguments");
    SFB_CHECK_ARG((mean == nullptr) == (var == nullptr), "rollout_mlp2_tape: mean/var must both be set or both NULL");
    SFB_CHECK_ARG(K1 <= RF_MAX_DIM, "rollout_mlp2_tape: observation rows of up to %d floats", RF_MAX_DIM);
    SFB_CHECK_ARG((reinterpret_cast<uintptr_t>(h1_scratch) & 15u) == 0 && (reinterpret_cast<uintptr_t>(x_norm) & 15u) == 0 &&
                      (reinterpret_cast<uintptr_t>(head_partials) & 15u) == 0, "rollout_mlp2_tape: scratch buffers must be 16-byte aligned");
    const bool with_rnn = rnn && traj_rnn_0 && rnn_dim > 0;
    const RolloutArgs a{n_envs, T, K1, H1, H2, b1, b2, Wv, Wa, A, bv, ba, h1_scratch, head_partials, x_norm,
                        values_0, values_stride, logits_0, logits_stride, actions_0, actions_stride, env_actions, log_prob_0,
                        log_prob_stride, policy_version_0, pv_stride, policy_version_scalar, noise, philox_seed, sampler_step,
                        tape, tape_len, env_index_offset, term_period, trunc_period, env_step_counter, env_obs, env_rew,
                        env_terminated, env_truncated,
                        EpisodeArgs{reward_scale, reward_clip, policy_id, traj_rewards_0, traj_dones_0, traj_time_outs_0,
                                    traj_policy_id_0, traj_stride, ep_return, ep_len, ep_min_raw, ep_max_raw, len_increment, stats,
                                    fin_return_0, fin_len_0},
                        traj_obs_0, traj_obs_stride, with_rnn ? rnn : nullptr, rnn_dim, traj_rnn_0, traj_rnn_stride,
                        make_obs_norm(mean, var, sub_mean, inv_scale, eps, clip), g_rollout_trace, nullptr, nullptr};
    const int rc = tc_rollout_mlp2_tape(W1, W2, act, engine, a, (cudaStream_t)stream);
    SFB_CHECK_ARG(rc != SFB_TC_UNSUPPORTED, "rollout_mlp2_tape: model not covered (K1=%d H1=%d H2=%d A=%d engine=%d); "
                  "sfb200_rollout_mlp2_partials() tells when to use the per-step calls", K1, H1, H2, A, engine);
    return rc;
}

}  // extern "C"
