// TMA / mbarrier / wgmma PTX wrappers, wgmma shared-memory descriptors and compile-time activations of the GEMM engine
// (gemm_tc.cu).  sm_90a only (wgmma.mma_async is an sm_90a instruction).
#pragma once
#include <cuda.h>
#include <cudaTypedefs.h>

#include "common.cuh"

namespace sfb {

constexpr int TBM = 128;        // tile rows: two consumer warpgroups of 64 rows (wgmma M = 64)
constexpr int TBN = 128;        // tile columns (wgmma N)
constexpr int TBK = 32;         // k per stage: 32 fp32 = 128 B = one swizzle row
constexpr int WG_K = 8;         // k per tf32 wgmma

// ------------------------------------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
// 1024-byte aligned start inside the dynamic shared-memory window (the 128B swizzle atoms need it).  Plain pointer
// arithmetic on the __shared__ array -- NOT a round trip through uintptr_t, which makes the compiler forget the address
// space and emit generic loads / stores for every shared-memory access derived from it.
__device__ __forceinline__ uint8_t* smem_align_1024(uint8_t* raw) {
    return raw + ((1024u - (smem_u32(raw) & 1023u)) & 1023u);
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
        "@P1 bra.uni WAIT_DONE;\n"
        "bra.uni WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
            smem_u32(smem_dst)),
        "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}

__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
            smem_u32(smem_dst)),
        "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}

// shared -> global tile store into the issuing thread's bulk group; elements outside the tensor are not written
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* tmap, const void* smem_src, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(tmap),
                 "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// every bulk group of the thread has completed: its writes are performed and visible to the thread
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// all but the most recently committed wgmma group of this warpgroup have completed
__device__ __forceinline__ void wgmma_wait_1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }

// gemm_wgmma_kernel's debug trace (sfb200_gemm_set_trace): %globaltimer in ns, %smid, 16 words per work item
constexpr int kTraceWords = 16;
__device__ __forceinline__ unsigned long long tc_now() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// the time at which `dep` is in its register: the timer read is predicated on a test of dep, so the stamp waits for the
// load (or the math) that produces it.  (0 for a NaN.)
__device__ __forceinline__ unsigned long long tc_now_after(float dep) {
    unsigned long long t;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.num.f32 p, %1, %1;\n"
        "mov.u64 %0, 0;\n"
        "@p mov.u64 %0, %%globaltimer;\n"
        "}\n"
        : "=l"(t)
        : "f"(dep));
    return t;
}
__device__ __forceinline__ uint32_t tc_smid() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(r));
    return r;
}

// warpgroup-wide register budget hand-over (every warp of the warpgroup executes it)
template <int REGS>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(REGS)); }
template <int REGS>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(REGS)); }

// D[64 x 128] (+)= A[64 x 8] * B[128 x 8]^T, tf32 operands from shared memory (K-major, 128B swizzle), fp32
// accumulators in the registers of the issuing warpgroup (PTX wgmma.mma_async m64n128k8 .tf32).  scale_d = 0 overwrites D.
// Accumulator fragment: thread t of the warpgroup holds d[i] at row 16*(t/32) + (t%32)/4 + 8*((i/2)%2),
// column 8*(i/4) + 2*(t%4) + i%2.
__device__ __forceinline__ void wgmma_m64n128k8_tf32(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, "
        "%64, %65, p, 1, 1;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
          "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
          "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),
          "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]),
          "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),
          "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(desc_a), "l"(desc_b), "r"(scale_d));
}

// The same shape with fp16 operands (k16 per instruction), both K-major (imm-trans 0), fp32 accumulate.
__device__ __forceinline__ void wgmma_m64n128k16_f16(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, "
        "%64, %65, p, 1, 1, 0, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]),
          "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]),
          "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
          "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]),
          "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]),
          "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]),
          "+f"(d[63])
        : "l"(desc_a), "l"(desc_b), "r"(scale_d));
}

// The same shape with the fp16 A operand in registers: a[4] is the thread's m64k16 fragment (warp w of the warpgroup
// holds rows 16w .. 16w+15 in the mma.m16n8k16 A layout, F16Frags in wgmma_tile.cuh), B from shared memory, K-major
// (TRANS_B = 0) or MN-major (TRANS_B = 1).  scale_d = 0 overwrites D.
template <int TRANS_B>
__device__ __forceinline__ void wgmma_m64n128k16_f16_rs(float (&d)[64], const uint32_t (&a)[4], uint64_t desc_b,
                                                        uint32_t scale_d = 1) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %70, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, "
        "{%64, %65, %66, %67}, %68, p, 1, 1, %69;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]),
          "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]),
          "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
          "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]),
          "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]),
          "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]),
          "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "n"(TRANS_B), "r"(scale_d));
}

// m64n64k16 with the fp16 A operand in registers (as above) and B MN-major (transpose bit set); scale_d = 0 overwrites D.
// Accumulator fragment: d[i] at row 16*(t/32) + (t%32)/4 + 8*((i/2)%2), column 8*(i/4) + 2*(t%4) + i%2.
__device__ __forceinline__ void wgmma_m64n64k16_f16_rs_mn(float (&d)[32], const uint32_t (&a)[4], uint64_t desc_b,
                                                          uint32_t scale_d) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %37, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
        "{%32, %33, %34, %35}, %36, p, 1, 1, 1;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(scale_d));
}

// ------------------------------------------------------------------------------------------------ descriptors
// wgmma shared-memory matrix descriptor: start>>4 [0,14) | LBO>>4 [16,30) | SBO>>4 [32,46) | layout [62,64) (1 = 128B swizzle).
// K-major tile [rows][32 fp32] with the 128B swizzle (16 B chunk index XOR row % 8, 8-row atoms of 1024 B): SBO = 1024
// (next 8 rows), LBO unused (1).  A k-step of 8 tf32 = 32 B advances the start address inside the swizzle row.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3fff);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024u >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
// MN-major 16-bit tile with the 128B swizzle (split_tile_f16_mn): 1024 B atoms of [8 k][64 rows]; LBO = 4096 (next 64
// rows), SBO = 1024 (next 8 k).  A k-step of 16 advances the start address by two atoms.  (lbo = 0: rows 64 .. 127 read
// the atoms of rows 0 .. 63 again -- head_partials_f16, whose B has 64 rows.)
__device__ __forceinline__ uint64_t make_smem_desc_mn(uint32_t smem_addr, uint32_t lbo = 4096) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3fff);
    d |= (uint64_t)(lbo >> 4) << 16;
    d |= (uint64_t)(1024u >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
// byte offset of element (row, k) of a K-major [rows][32 fp32] tile in the 128B-swizzled layout
__device__ __forceinline__ uint32_t sw128_offset(int row, int k) {
    return (uint32_t)(row * 128 + ((((k >> 2) ^ row) & 7) << 4) + (k & 3) * 4);
}

template <int ACT>
__device__ __forceinline__ float act_fwd_ct(float z) {
    if (ACT == SFB200_ACT_ELU) {
        // __expf(z) - 1 for z <= 0, computed unconditionally: __expf is ex2.approx(z * log2(e)) plus a rescaling branch for
        // results below 2^-126, which (e - 1) rounds to -1 either way -- same bits, half the instructions, no predication
        float e;
        asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(z * 1.4426950216293334961f));
        return z > 0.f ? z : e - 1.f;
    }
    if (ACT == SFB200_ACT_RELU) return fmaxf(z, 0.f);
    if (ACT == SFB200_ACT_TANH) return tanhf(z);
    return z;
}
template <int ACT>
__device__ __forceinline__ float act_bwd_ct(float h) {
    if (ACT == SFB200_ACT_ELU) return h > 0.f ? 1.f : h + 1.f;
    if (ACT == SFB200_ACT_RELU) return h > 0.f ? 1.f : 0.f;
    if (ACT == SFB200_ACT_TANH) return 1.f - h * h;
    return 1.f;
}

// host side (gemm_tc.cu): driver entry point for cuTensorMapEncodeTiled resolved at run time; 2-D fp32 tensor maps
// without swizzle (the engine re-lays the tiles out itself), or with the 128B swizzle for tiles read straight into
// wgmma register fragments (box0 = 32). dim0 = contiguous dimension.
bool tc_init();
bool make_tmap(CUtensorMap* out, const float* base, uint64_t dim0, uint64_t dim1, uint64_t stride1_elems, uint32_t box0,
               uint32_t box1, bool swizzle128 = false);
// 3-D fp16 map over a [hi | lo] pair of row-major [rows][K] planes, lo_offset elements apart: box 64 k x box_rows rows x
// both planes with the 128B swizzle (the weights' registered twins; the rollout's split h1 scratch)
bool make_tmap_f16_twins(CUtensorMap* out, const uint16_t* hi, int64_t lo_offset, uint64_t K, uint64_t rows,
                         uint32_t box_rows);

}  // namespace sfb
