// sfb200_env_ingest: the tensors a batched tensor env returns every step, in their own dtypes and row strides, converted
// into the sampler's static buffers in one launch (see include/sfb200.h).  A streaming kernel: each thread converts one
// 16-byte chunk of a source row (one 128-bit load where the source allows it) and writes it with the widest store its
// destination alignment allows.
#include <cuda_bf16.h>

#include "common.cuh"

namespace sfb {

struct IngestEntry {
    const uint8_t* src;
    uint8_t* dst;
    int64_t src_stride, dst_stride;   // elements of the source / destination type
    int64_t rows, cols, chunks;       // chunks: 16-byte source chunks per row
    int32_t dtype, kind, vec;         // vec: every chunk start is 16-byte aligned (128-bit loads)
};

struct IngestArgs {
    IngestEntry e[SFB200_INGEST_MAX];
};

// per source dtype: the raw element type, its exact conversion to float32 (torch's .to(torch.float32): round to nearest
// even for float64 and 32/64-bit integers) and x != 0 evaluated in the source type
template <int DT> struct Src;
template <> struct Src<SFB200_DT_F32> {
    using T = float;
    static __device__ __forceinline__ float f(T v) { return v; }
    static __device__ __forceinline__ bool nz(T v) { return v != 0.f; }
};
template <> struct Src<SFB200_DT_F16> {
    using T = uint16_t;
    static __device__ __forceinline__ float f(T v) { return __half2float(__ushort_as_half(v)); }
    static __device__ __forceinline__ bool nz(T v) { return f(v) != 0.f; }
};
template <> struct Src<SFB200_DT_BF16> {
    using T = uint16_t;
    static __device__ __forceinline__ float f(T v) { return __uint_as_float((uint32_t)v << 16); }
    static __device__ __forceinline__ bool nz(T v) { return f(v) != 0.f; }
};
template <> struct Src<SFB200_DT_F64> {
    using T = double;
    static __device__ __forceinline__ float f(T v) { return __double2float_rn(v); }
    static __device__ __forceinline__ bool nz(T v) { return v != 0.0; }
};
template <> struct Src<SFB200_DT_I8> {
    using T = int8_t;
    static __device__ __forceinline__ float f(T v) { return (float)v; }
    static __device__ __forceinline__ bool nz(T v) { return v != 0; }
};
template <> struct Src<SFB200_DT_I16> {
    using T = int16_t;
    static __device__ __forceinline__ float f(T v) { return (float)v; }
    static __device__ __forceinline__ bool nz(T v) { return v != 0; }
};
template <> struct Src<SFB200_DT_I32> {
    using T = int32_t;
    static __device__ __forceinline__ float f(T v) { return __int2float_rn(v); }
    static __device__ __forceinline__ bool nz(T v) { return v != 0; }
};
template <> struct Src<SFB200_DT_I64> {
    using T = long long;
    static __device__ __forceinline__ float f(T v) { return __ll2float_rn(v); }
    static __device__ __forceinline__ bool nz(T v) { return v != 0; }
};
template <> struct Src<SFB200_DT_U8> {
    using T = uint8_t;
    static __device__ __forceinline__ float f(T v) { return (float)v; }
    static __device__ __forceinline__ bool nz(T v) { return v != 0; }
};
template <> struct Src<SFB200_DT_BOOL> {
    using T = uint8_t;
    static __device__ __forceinline__ float f(T v) { return v ? 1.f : 0.f; }
    static __device__ __forceinline__ bool nz(T v) { return v != 0; }
};

static int dtype_size(int dt) {
    switch (dt) {
        case SFB200_DT_F64: case SFB200_DT_I64: return 8;
        case SFB200_DT_F32: case SFB200_DT_I32: return 4;
        case SFB200_DT_F16: case SFB200_DT_BF16: case SFB200_DT_I16: return 2;
        case SFB200_DT_I8: case SFB200_DT_U8: case SFB200_DT_BOOL: return 1;
        default: return 0;
    }
}

// elements [c0, c0 + V) of row r (fewer at the end of the row)
template <int DT>
__device__ __forceinline__ void ingest_chunk(const IngestEntry& e, int64_t r, int64_t c0) {
    using S = Src<DT>;
    using T = typename S::T;
    constexpr int V = 16 / sizeof(T);
    const T* s = reinterpret_cast<const T*>(e.src) + r * e.src_stride + c0;
    const int64_t left = e.cols - c0;
    const int n = left < V ? (int)left : V;
    union {
        uint4 u;
        T v[V];
    } buf;
    if (e.vec && n == V) {
        buf.u = __ldg(reinterpret_cast<const uint4*>(s));
    } else {
#pragma unroll
        for (int i = 0; i < V; ++i) buf.v[i] = i < n ? s[i] : T(0);
    }
    const int64_t d0 = r * e.dst_stride + c0;
    if (e.kind == SFB200_INGEST_F32) {
        float* d = reinterpret_cast<float*>(e.dst) + d0;
        if (V % 4 == 0 && n == V && (reinterpret_cast<uintptr_t>(d) & 15) == 0) {
#pragma unroll
            for (int i = 0; i < V; i += 4)
                *reinterpret_cast<float4*>(d + i) =
                    make_float4(S::f(buf.v[i]), S::f(buf.v[i + 1]), S::f(buf.v[i + 2]), S::f(buf.v[i + 3]));
        } else {
#pragma unroll
            for (int i = 0; i < V; ++i)
                if (i < n) d[i] = S::f(buf.v[i]);
        }
        return;
    }
    uint8_t* d = e.dst + d0;
    if (V % 4 == 0 && n == V && (reinterpret_cast<uintptr_t>(d) & 3) == 0) {
        // one byte per element, four per 32-bit store (uint8 copy or the bool x != 0)
#pragma unroll
        for (int i = 0; i < V; i += 4) {
            uint32_t w = 0;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint32_t b = e.kind == SFB200_INGEST_U8 ? (uint32_t)(uint8_t)buf.v[i + j] : (uint32_t)S::nz(buf.v[i + j]);
                w |= b << (8 * j);
            }
            *reinterpret_cast<uint32_t*>(d + i) = w;
        }
    } else {
#pragma unroll
        for (int i = 0; i < V; ++i)
            if (i < n) d[i] = e.kind == SFB200_INGEST_U8 ? (uint8_t)buf.v[i] : (uint8_t)S::nz(buf.v[i]);
    }
}

template <int DT>
__device__ __forceinline__ void ingest_entry(const IngestEntry& e) {
    constexpr int V = 16 / sizeof(typename Src<DT>::T);
    const int64_t total = e.rows * e.chunks;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += stride) {
        const int64_t r = i / e.chunks;
        ingest_chunk<DT>(e, r, (i - r * e.chunks) * V);
    }
}

// blockIdx.y selects the entry (all threads of a block take the same dtype branch)
__global__ void __launch_bounds__(256) env_ingest_kernel(const __grid_constant__ IngestArgs a) {
    const IngestEntry& e = a.e[blockIdx.y];
    switch (e.dtype) {
        case SFB200_DT_F32: ingest_entry<SFB200_DT_F32>(e); break;
        case SFB200_DT_F16: ingest_entry<SFB200_DT_F16>(e); break;
        case SFB200_DT_BF16: ingest_entry<SFB200_DT_BF16>(e); break;
        case SFB200_DT_F64: ingest_entry<SFB200_DT_F64>(e); break;
        case SFB200_DT_I8: ingest_entry<SFB200_DT_I8>(e); break;
        case SFB200_DT_I16: ingest_entry<SFB200_DT_I16>(e); break;
        case SFB200_DT_I32: ingest_entry<SFB200_DT_I32>(e); break;
        case SFB200_DT_I64: ingest_entry<SFB200_DT_I64>(e); break;
        case SFB200_DT_U8: ingest_entry<SFB200_DT_U8>(e); break;
        default: ingest_entry<SFB200_DT_BOOL>(e); break;
    }
}

}  // namespace sfb

using namespace sfb;

int sfb200_env_ingest(const int64_t* desc_host, int n_desc, int64_t rows, void* stream) {
    SFB_CHECK_ARG(desc_host && n_desc > 0 && n_desc <= SFB200_INGEST_MAX && rows >= 0,
                  "env_ingest: bad arguments (n_desc=%d, at most %d entries)", n_desc, SFB200_INGEST_MAX);
    if (rows == 0) return 0;
    IngestArgs a = {};
    int64_t max_items = 0;
    for (int k = 0; k < n_desc; ++k) {
        const int64_t* d = desc_host + (int64_t)k * SFB200_INGEST_FIELDS;
        IngestEntry& e = a.e[k];
        e.src = reinterpret_cast<const uint8_t*>(d[0]);
        e.dtype = (int32_t)d[1];
        e.src_stride = d[2];
        e.cols = d[3];
        e.dst = reinterpret_cast<uint8_t*>(d[4]);
        e.dst_stride = d[5];
        e.kind = (int32_t)d[6];
        const int es = dtype_size(e.dtype);
        SFB_CHECK_ARG(e.src && e.dst && es > 0 && e.cols > 0 && e.src_stride >= 0 && e.dst_stride >= 0,
                      "env_ingest: entry %d: bad source / destination (dtype %d, cols %lld)", k, e.dtype, (long long)e.cols);
        SFB_CHECK_ARG(e.kind == SFB200_INGEST_F32 || e.kind == SFB200_INGEST_BOOL ||
                      (e.kind == SFB200_INGEST_U8 && e.dtype == SFB200_DT_U8),
                      "env_ingest: entry %d: destination kind %d does not take dtype %d", k, e.kind, e.dtype);
        e.rows = rows;
        if (e.src_stride == e.cols && e.dst_stride == e.cols) {   // dense source and destination: one long row
            e.cols *= rows;
            e.rows = 1;
        }
        const int V = 16 / es;
        e.vec = (reinterpret_cast<uintptr_t>(e.src) % 16 == 0) && (e.rows == 1 || (e.src_stride * es) % 16 == 0);
        e.chunks = ceil_div(e.cols, V);
        if (e.rows * e.chunks > max_items) max_items = e.rows * e.chunks;
    }
    int64_t blocks = ceil_div(max_items, 256);
    const int64_t cap = (int64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    env_ingest_kernel<<<dim3((unsigned)blocks, (unsigned)n_desc), 256, 0, (cudaStream_t)stream>>>(a);
    SFB_LAUNCH_OK();
    return 0;
}
