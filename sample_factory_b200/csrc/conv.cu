// Convolutional encoder support (reference: model/encoder.py:88-145, ConvEncoderImpl = Conv2d stacks without padding).
// A Conv2d is run as  im2col -> GEMM engine (wgmma / SIMT, bias + activation in the GEMM epilogue)  so the tensor-core
// path, its fp32-parity split and the backward GEMMs are shared with the MLP layers:
//   forward :  col[m, k] = x[b, ci, oh*s+kh, ow*s+kw]        m = (b, oh, ow), k = (ci, kh, kw)  == Conv2d weight flatten
//              y[m, co]  = act(col[m, :] . W[co, :] + b[co])  -> activations are kept NHWC ([B*OH*OW, C] row-major)
//   backward:  dW = dy^T col (GEMM), dcol = dy W (GEMM), dx = col2im(dcol) * act'(x)  (gather form: deterministic)
// The first layer reads the (normalised) observation in the reference's NCHW order, later layers read NHWC; the last
// layer's output is permuted back to the (C, H, W) flatten order the reference's fully connected layer expects
// (encoder.py:115).  All kernels are HBM-bound gathers / scatters with coalesced accesses on the side that allows it.
#include "common.cuh"

namespace sfb {

// x: NCHW [B, C, H, W] (in_nchw) or NHWC [B, H, W, C];  col: [B*OH*OW, C*KH*KW]
template <bool IN_NCHW>
__global__ void __launch_bounds__(256) im2col_kernel(const float* __restrict__ x, float* __restrict__ col, int64_t B, int C,
                                                     int H, int W, int KS, int stride, int OH, int OW) {
    const int K = C * KS * KS;
    const int64_t total = B * OH * OW * (int64_t)K;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t m = i / K;
        const int k = (int)(i - m * K);
        const int ci = k / (KS * KS);
        const int r = k - ci * KS * KS;
        const int kh = r / KS, kw = r - kh * KS;
        const int64_t b = m / (OH * OW);
        const int p = (int)(m - b * OH * OW);
        const int oh = p / OW, ow = p - oh * OW;
        const int ih = oh * stride + kh, iw = ow * stride + kw;
        const int64_t src = IN_NCHW ? ((b * C + ci) * H + ih) * W + iw : ((b * H + ih) * W + iw) * C + ci;
        col[i] = x[src];
    }
}

// dx[b, ih, iw, ci] (NHWC) = act'(x[b, ih, iw, ci]) * sum over the windows (oh, ow, kh, kw) that cover (ih, iw) of
// dcol[(b, oh, ow), (ci, kh, kw)].  Gather form: every output element is written by exactly one thread, in a fixed order.
__global__ void __launch_bounds__(256) col2im_kernel(const float* __restrict__ dcol, const float* __restrict__ x_act,
                                                     float* __restrict__ dx, int64_t B, int C, int H, int W, int KS,
                                                     int stride, int OH, int OW, int act) {
    const int K = C * KS * KS;
    const int64_t total = B * H * W * (int64_t)C;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int ci = (int)(i % C);
        const int64_t pix = i / C;
        const int iw = (int)(pix % W);
        const int64_t t = pix / W;
        const int ih = (int)(t % H);
        const int64_t b = t / H;
        float s = 0.f;
        // kh ranges over ih - oh*stride with 0 <= kh < KS and 0 <= oh < OH
        for (int kh = ih % stride; kh < KS; kh += stride) {
            const int oh = (ih - kh) / stride;
            if (ih < kh || oh >= OH) continue;
            for (int kw = iw % stride; kw < KS; kw += stride) {
                const int ow = (iw - kw) / stride;
                if (iw < kw || ow >= OW) continue;
                s += dcol[((b * OH + oh) * OW + ow) * K + (ci * KS + kh) * KS + kw];
            }
        }
        dx[i] = s * act_bwd_from_out(x_act[i], act);
    }
}

// [B, P, C] (NHWC rows) <-> [B, C, P] (the reference's (C, H, W) flatten); tiny (conv head output)
__global__ void __launch_bounds__(256) permute_bpc_kernel(const float* __restrict__ src, float* __restrict__ dst, int64_t B,
                                                          int P, int C, int to_cp) {
    const int64_t total = B * P * (int64_t)C;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        // i indexes dst
        const int64_t b = i / ((int64_t)P * C);
        const int r = (int)(i - b * P * C);
        int p, c;
        if (to_cp) { c = r / P; p = r - c * P; }   // dst [B, C, P]
        else { p = r / C; c = r - p * C; }          // dst [B, P, C]
        const int64_t s = to_cp ? (b * P + p) * C + c : (b * C + c) * P + p;
        dst[i] = src[s];
    }
}

static unsigned conv_grid(int64_t work) {
    int64_t blocks = ceil_div(work, 256);
    const int64_t cap = (int64_t)sm_count() * 16;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    return (unsigned)blocks;
}

}  // namespace sfb

using namespace sfb;

extern "C" {

int sfb200_im2col(const float* x, int in_nchw, int64_t B, int C, int H, int W, int kernel, int stride, float* col,
                  void* stream) {
    SFB_CHECK_ARG(x && col && B >= 0 && C > 0 && H >= kernel && W >= kernel && kernel > 0 && stride > 0, "im2col: bad arguments");
    if (B == 0) return 0;
    const int OH = (H - kernel) / stride + 1, OW = (W - kernel) / stride + 1;
    const int64_t total = B * OH * OW * (int64_t)C * kernel * kernel;
    cudaStream_t st = (cudaStream_t)stream;
    if (in_nchw) im2col_kernel<true><<<conv_grid(total), 256, 0, st>>>(x, col, B, C, H, W, kernel, stride, OH, OW);
    else im2col_kernel<false><<<conv_grid(total), 256, 0, st>>>(x, col, B, C, H, W, kernel, stride, OH, OW);
    SFB_LAUNCH_OK();
    return 0;
}

int sfb200_col2im_act_backward(const float* dcol, const float* x_act, int64_t B, int C, int H, int W, int kernel,
                               int stride, int act, float* dx, void* stream) {
    SFB_CHECK_ARG(dcol && x_act && dx && B >= 0 && C > 0 && H >= kernel && W >= kernel && kernel > 0 && stride > 0,
                  "col2im_act_backward: bad arguments");
    if (B == 0) return 0;
    const int OH = (H - kernel) / stride + 1, OW = (W - kernel) / stride + 1;
    col2im_kernel<<<conv_grid(B * H * W * (int64_t)C), 256, 0, (cudaStream_t)stream>>>(dcol, x_act, dx, B, C, H, W, kernel,
                                                                                       stride, OH, OW, act);
    SFB_LAUNCH_OK();
    return 0;
}

int sfb200_permute_bpc(const float* src, float* dst, int64_t B, int P, int C, int to_channel_major, void* stream) {
    SFB_CHECK_ARG(src && dst && B >= 0 && P > 0 && C > 0, "permute_bpc: bad arguments");
    if (B == 0) return 0;
    permute_bpc_kernel<<<conv_grid(B * P * (int64_t)C), 256, 0, (cudaStream_t)stream>>>(src, dst, B, P, C, to_channel_major);
    SFB_LAUNCH_OK();
    return 0;
}

}  // extern "C"
