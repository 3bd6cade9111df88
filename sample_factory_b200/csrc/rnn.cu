// Recurrent core (reference model/core.py:19-64: nn.GRU / nn.LSTM) as elementwise cell kernels around the GEMM engine,
// one layer per call:  gi = x.W_ih^T + b_ih  and  gh = h.W_hh^T + b_hh  are sfb200_linear_act_forward calls, the kernels
// here do the gate math forward and backward.  Stacked layers pass their slice of the layer-major state rows as a
// pointer offset with the full row stride (rnn_core.py).  All HBM-bound streaming kernels (one pass over the gate tensors).
// Episode-boundary handling (batched_sampling.py:332-335, rnn_utils.py:143-149): a row whose `reset` flag is set starts
// the NEXT step from a zero state, and no gradient flows back across that boundary.
#include "common.cuh"

namespace sfb {

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// ---------------------------------------------------------------------------------------------------------------- GRU
// r = s(gi_r+gh_r) ; z = s(gi_z+gh_z) ; n = tanh(gi_n + r*gh_n) ; h' = (1-z)*n + z*h         (torch.nn.GRU, gates r,z,n)
__global__ void __launch_bounds__(256) gru_fwd_kernel(const float* __restrict__ gi, int64_t ldgi,
                                                      const float* __restrict__ gh, int64_t ldgh,
                                                      const float* __restrict__ h_in, int64_t ldh, float* __restrict__ h_out,
                                                      int64_t ldo, float* __restrict__ h_next, int64_t ldn,
                                                      const uint8_t* __restrict__ reset_next, int64_t reset_stride,
                                                      float* __restrict__ gates, int64_t ldg, int64_t M, int H) {
    const int64_t total = M * (int64_t)H;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t m = i / H;
        const int j = (int)(i - m * H);
        const float* a = gi + m * ldgi;
        const float* b = gh + m * ldgh;
        const float r = sigmoidf_(a[j] + b[j]);
        const float z = sigmoidf_(a[H + j] + b[H + j]);
        const float n = tanhf(a[2 * H + j] + r * b[2 * H + j]);
        const float h = h_in[m * ldh + j];
        const float hn = (1.f - z) * n + z * h;
        h_out[m * ldo + j] = hn;
        if (h_next) h_next[m * ldn + j] = (reset_next && reset_next[m * reset_stride]) ? 0.f : hn;
        if (gates) {
            float* g = gates + m * ldg;
            g[j] = r; g[H + j] = z; g[2 * H + j] = n;
        }
    }
}

// dh = dh_out + (1-reset)*(carry_a + carry_b);  dn = dh*(1-z); dz = dh*(h-n); dh_in_direct = dh*z
// dn_pre = dn*(1-n^2); dgi_n = dn_pre; dgh_n = dn_pre*r; dr = dn_pre*gh_n; dr_pre = dr*r*(1-r); dz_pre = dz*z*(1-z)
__global__ void __launch_bounds__(256) gru_bwd_kernel(const float* __restrict__ dh_out, int64_t lddo,
                                                      const float* __restrict__ carry_a, const float* __restrict__ carry_b,
                                                      int64_t ldc, const uint8_t* __restrict__ reset, int64_t reset_stride,
                                                      const float* __restrict__ gates, int64_t ldg,
                                                      const float* __restrict__ gh, int64_t ldgh,
                                                      const float* __restrict__ h_in, int64_t ldh, float* __restrict__ dgi,
                                                      int64_t lddgi, float* __restrict__ dgh, int64_t lddgh,
                                                      float* __restrict__ dh_direct, int64_t lddd, int64_t M, int H) {
    const int64_t total = M * (int64_t)H;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t m = i / H;
        const int j = (int)(i - m * H);
        float dh = dh_out ? dh_out[m * lddo + j] : 0.f;
        if (carry_a && !(reset && reset[m * reset_stride])) {
            dh += carry_a[m * ldc + j];
            if (carry_b) dh += carry_b[m * ldc + j];
        }
        const float* g = gates + m * ldg;
        const float r = g[j], z = g[H + j], n = g[2 * H + j];
        const float h = h_in[m * ldh + j];
        const float ghn = gh[m * ldgh + 2 * H + j];
        const float dn_pre = dh * (1.f - z) * (1.f - n * n);
        const float dz_pre = dh * (h - n) * z * (1.f - z);
        const float dr_pre = dn_pre * ghn * r * (1.f - r);
        float* a = dgi + m * lddgi;
        float* b = dgh + m * lddgh;
        a[j] = dr_pre; a[H + j] = dz_pre; a[2 * H + j] = dn_pre;
        b[j] = dr_pre; b[H + j] = dz_pre; b[2 * H + j] = dn_pre * r;
        dh_direct[m * lddd + j] = dh * z;
    }
}

// --------------------------------------------------------------------------------------------------------------- LSTM
// g = gi + gh ; i,f,o = s(.), gg = tanh(.) ; c' = f*c + i*gg ; h' = o*tanh(c')        (torch.nn.LSTM, gates i,f,g,o)
// state layout [h || c] (reference core.py:51-53)
__global__ void __launch_bounds__(256) lstm_fwd_kernel(const float* __restrict__ gi, int64_t ldgi,
                                                       const float* __restrict__ gh, int64_t ldgh,
                                                       const float* __restrict__ state_in, int64_t lds,
                                                       float* __restrict__ state_out, int64_t ldo,
                                                       float* __restrict__ state_next, int64_t ldn,
                                                       const uint8_t* __restrict__ reset_next, int64_t reset_stride,
                                                       float* __restrict__ gates, int64_t ldg, int64_t M, int H) {
    const int64_t total = M * (int64_t)H;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t m = i / H;
        const int j = (int)(i - m * H);
        const float* a = gi + m * ldgi;
        const float* b = gh + m * ldgh;
        const float ig = sigmoidf_(a[j] + b[j]);
        const float fg = sigmoidf_(a[H + j] + b[H + j]);
        const float gg = tanhf(a[2 * H + j] + b[2 * H + j]);
        const float og = sigmoidf_(a[3 * H + j] + b[3 * H + j]);
        const float c = state_in[m * lds + H + j];
        const float cn = fg * c + ig * gg;
        const float hn = og * tanhf(cn);
        state_out[m * ldo + j] = hn;
        state_out[m * ldo + H + j] = cn;
        if (state_next) {
            const bool rs = reset_next && reset_next[m * reset_stride];
            state_next[m * ldn + j] = rs ? 0.f : hn;
            state_next[m * ldn + H + j] = rs ? 0.f : cn;
        }
        if (gates) {
            float* g = gates + m * ldg;
            g[j] = ig; g[H + j] = fg; g[2 * H + j] = gg; g[3 * H + j] = og;
        }
    }
}

// dh = dh_out + (1-reset)*dh_carry ; dc' = (1-reset)*dc_carry + dh*o*(1-tanh(c')^2)
// do = dh*tanh(c') ; di = dc'*gg ; df = dc'*c ; dgg = dc'*i ; dc_in = dc'*f ; pre-activation grads -> dgates (= dgi = dgh)
__global__ void __launch_bounds__(256) lstm_bwd_kernel(const float* __restrict__ dh_out, int64_t lddo,
                                                       const float* __restrict__ dh_carry, const float* __restrict__ dc_carry,
                                                       int64_t ldc, const uint8_t* __restrict__ reset, int64_t reset_stride,
                                                       const float* __restrict__ gates, int64_t ldg,
                                                       const float* __restrict__ state_in, int64_t lds,
                                                       const float* __restrict__ state_out, int64_t ldo,
                                                       float* __restrict__ dgates, int64_t lddg, float* __restrict__ dc_in,
                                                       int64_t lddc, int64_t M, int H) {
    const int64_t total = M * (int64_t)H;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t m = i / H;
        const int j = (int)(i - m * H);
        const bool cut = reset && reset[m * reset_stride];
        float dh = dh_out ? dh_out[m * lddo + j] : 0.f;
        float dc = 0.f;
        if (!cut) {
            if (dh_carry) dh += dh_carry[m * ldc + j];
            if (dc_carry) dc = dc_carry[m * ldc + j];
        }
        const float* g = gates + m * ldg;
        const float ig = g[j], fg = g[H + j], gg = g[2 * H + j], og = g[3 * H + j];
        const float c = state_in[m * lds + H + j];
        const float tc = tanhf(state_out[m * ldo + H + j]);
        dc += dh * og * (1.f - tc * tc);
        float* d = dgates + m * lddg;
        d[j] = dc * gg * ig * (1.f - ig);
        d[H + j] = dc * c * fg * (1.f - fg);
        d[2 * H + j] = dc * ig * (1.f - gg * gg);
        d[3 * H + j] = dh * tc * og * (1.f - og);
        dc_in[m * lddc + j] = dc * fg;
    }
}

__global__ void mask_rows_kernel(const float* __restrict__ src, int64_t lds, float* __restrict__ dst, int64_t ldd,
                                 const uint8_t* __restrict__ reset, int64_t reset_stride, int64_t M, int dim) {
    const int64_t total = M * (int64_t)dim;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t m = i / dim;
        const int j = (int)(i - m * dim);
        dst[m * ldd + j] = reset[m * reset_stride] ? 0.f : src[m * lds + j];
    }
}

static unsigned grid_rnn(int64_t work) {
    int64_t blocks = ceil_div(work, 256);
    const int64_t cap = (int64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    return (unsigned)blocks;
}

}  // namespace sfb

using namespace sfb;

extern "C" {

int sfb200_gru_cell_forward(const float* gi, int64_t ldgi, const float* gh, int64_t ldgh, const float* h_in, int64_t ldh,
                            float* h_out, int64_t ldo, float* h_next, int64_t ldn, const uint8_t* reset_next,
                            int64_t reset_stride, float* gates, int64_t ldg, int64_t M, int H, void* stream) {
    SFB_CHECK_ARG(gi && gh && h_in && h_out && M >= 0 && H > 0, "gru_cell_forward: bad arguments");
    if (M == 0) return 0;
    gru_fwd_kernel<<<grid_rnn(M * H), 256, 0, (cudaStream_t)stream>>>(gi, ldgi, gh, ldgh, h_in, ldh, h_out, ldo, h_next, ldn,
                                                                     reset_next, reset_stride, gates, ldg, M, H);
    SFB_LAUNCH_OK();
    return 0;
}

int sfb200_gru_cell_backward(const float* dh_out, int64_t lddo, const float* carry_a, const float* carry_b, int64_t ldc,
                             const uint8_t* reset, int64_t reset_stride, const float* gates, int64_t ldg, const float* gh,
                             int64_t ldgh, const float* h_in, int64_t ldh, float* dgi, int64_t lddgi, float* dgh,
                             int64_t lddgh, float* dh_direct, int64_t lddd, int64_t M, int H, void* stream) {
    SFB_CHECK_ARG(gates && gh && h_in && dgi && dgh && dh_direct && M >= 0 && H > 0, "gru_cell_backward: bad arguments");
    if (M == 0) return 0;
    gru_bwd_kernel<<<grid_rnn(M * H), 256, 0, (cudaStream_t)stream>>>(dh_out, lddo, carry_a, carry_b, ldc, reset, reset_stride,
                                                                     gates, ldg, gh, ldgh, h_in, ldh, dgi, lddgi, dgh, lddgh,
                                                                     dh_direct, lddd, M, H);
    SFB_LAUNCH_OK();
    return 0;
}

int sfb200_lstm_cell_forward(const float* gi, int64_t ldgi, const float* gh, int64_t ldgh, const float* state_in,
                             int64_t lds, float* state_out, int64_t ldo, float* state_next, int64_t ldn,
                             const uint8_t* reset_next, int64_t reset_stride, float* gates, int64_t ldg, int64_t M, int H,
                             void* stream) {
    SFB_CHECK_ARG(gi && gh && state_in && state_out && M >= 0 && H > 0, "lstm_cell_forward: bad arguments");
    if (M == 0) return 0;
    lstm_fwd_kernel<<<grid_rnn(M * H), 256, 0, (cudaStream_t)stream>>>(gi, ldgi, gh, ldgh, state_in, lds, state_out, ldo,
                                                                      state_next, ldn, reset_next, reset_stride, gates, ldg,
                                                                      M, H);
    SFB_LAUNCH_OK();
    return 0;
}

int sfb200_lstm_cell_backward(const float* dh_out, int64_t lddo, const float* dh_carry, const float* dc_carry, int64_t ldc,
                              const uint8_t* reset, int64_t reset_stride, const float* gates, int64_t ldg,
                              const float* state_in, int64_t lds, const float* state_out, int64_t ldo, float* dgates,
                              int64_t lddg, float* dc_in, int64_t lddc, int64_t M, int H, void* stream) {
    SFB_CHECK_ARG(gates && state_in && state_out && dgates && dc_in && M >= 0 && H > 0, "lstm_cell_backward: bad arguments");
    if (M == 0) return 0;
    lstm_bwd_kernel<<<grid_rnn(M * H), 256, 0, (cudaStream_t)stream>>>(dh_out, lddo, dh_carry, dc_carry, ldc, reset,
                                                                      reset_stride, gates, ldg, state_in, lds, state_out, ldo,
                                                                      dgates, lddg, dc_in, lddc, M, H);
    SFB_LAUNCH_OK();
    return 0;
}

int sfb200_mask_rows(const float* src, int64_t src_stride, float* dst, int64_t dst_stride, const uint8_t* reset,
                     int64_t reset_stride, int64_t rows, int dim, void* stream) {
    SFB_CHECK_ARG(src && dst && reset && rows >= 0 && dim > 0, "mask_rows: bad arguments");
    if (rows == 0) return 0;
    mask_rows_kernel<<<grid_rnn(rows * dim), 256, 0, (cudaStream_t)stream>>>(src, src_stride, dst, dst_stride, reset,
                                                                            reset_stride, rows, dim);
    SFB_LAUNCH_OK();
    return 0;
}

}  // extern "C"
