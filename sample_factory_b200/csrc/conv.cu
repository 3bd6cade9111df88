// Convolutional encoder support (reference: model/encoder.py:88-145, ConvEncoderImpl = Conv2d stacks without padding;
// model/encoder.py:153-221, ResnetEncoder = padded 3x3 convs, 3x3 / stride 2 max-pools and pre-activation residual blocks).
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
// col = im2col(act(x)) with `pad` zeros around the ACTIVATED input (Conv2d(act(x), padding=pad)); pad = 0 with act = none
// is the plain gather of the convnet_* stacks
template <bool IN_NCHW>
__global__ void __launch_bounds__(256) im2col_kernel(const float* __restrict__ x, float* __restrict__ col, int64_t B, int C,
                                                     int H, int W, int KS, int stride, int pad, int act, int OH, int OW) {
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
        const int ih = oh * stride + kh - pad, iw = ow * stride + kw - pad;
        float v = 0.f;
        if (ih >= 0 && ih < H && iw >= 0 && iw < W) {
            const int64_t src = IN_NCHW ? ((b * C + ci) * H + ih) * W + iw : ((b * H + ih) * W + iw) * C + ci;
            v = act_fwd(x[src], act);
        }
        col[i] = v;
    }
}

// derivative of the activation from its INPUT z (autograd's elu_backward(is_result=false), threshold_backward, and
// tanh_backward of tanh(z))
__device__ __forceinline__ float act_bwd_from_in(float z, int act) {
    switch (act) {
        case SFB200_ACT_ELU: return z > 0.f ? 1.f : expf(z);
        case SFB200_ACT_RELU: return z > 0.f ? 1.f : 0.f;
        case SFB200_ACT_TANH: { const float h = tanhf(z); return 1.f - h * h; }
        default: return 1.f;
    }
}

// dx[b, ih, iw, ci] (NHWC) = act'(x[b, ih, iw, ci]) * sum over the windows (oh, ow, kh, kw) that cover (ih, iw) of
// dcol[(b, oh, ow), (ci, kh, kw)]  (+ dres[b, ih, iw, ci]).  act' comes from the stored activation OUTPUT (from_input = 0)
// or from the stored INPUT of the activation (from_input = 1: a residual block's act(x), whose identity path adds dres).
// Gather form: every output element is written by exactly one thread, in a fixed order.
__global__ void __launch_bounds__(256) col2im_kernel(const float* __restrict__ dcol, const float* __restrict__ x_act,
                                                     const float* __restrict__ dres, float* __restrict__ dx, int64_t B,
                                                     int C, int H, int W, int KS, int stride, int pad, int OH, int OW,
                                                     int act, int from_input) {
    const int K = C * KS * KS;
    const int64_t total = B * H * W * (int64_t)C;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int ci = (int)(i % C);
        const int64_t pix = i / C;
        const int iw = (int)(pix % W);
        const int64_t t = pix / W;
        const int ih = (int)(t % H);
        const int64_t b = t / H;
        const int ihp = ih + pad, iwp = iw + pad;   // position in the padded input
        float s = 0.f;
        // kh ranges over ihp - oh*stride with 0 <= kh < KS and 0 <= oh < OH
        for (int kh = ihp % stride; kh < KS; kh += stride) {
            const int oh = (ihp - kh) / stride;
            if (ihp < kh || oh >= OH) continue;
            for (int kw = iwp % stride; kw < KS; kw += stride) {
                const int ow = (iwp - kw) / stride;
                if (iwp < kw || ow >= OW) continue;
                s += dcol[((b * OH + oh) * OW + ow) * K + (ci * KS + kh) * KS + kw];
            }
        }
        float d = s * (from_input ? act_bwd_from_in(x_act[i], act) : act_bwd_from_out(x_act[i], act));
        if (dres) d += dres[i];
        dx[i] = d;
    }
}

// MaxPool2d(3, stride 2, padding 1) on NHWC rows (encoder.py:191): y = the window maximum, idx = its position kh*3+kw.
// torch's rule: the first maximum in row-major window order wins, a NaN wins over numbers (and a later NaN over an
// earlier one); padding never wins (the scan starts at the first in-bounds element).
__global__ void __launch_bounds__(256) maxpool3s2_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                         uint8_t* __restrict__ idx, int64_t B, int C, int H, int W,
                                                         int OH, int OW) {
    const int64_t total = B * OH * OW * (int64_t)C;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const int64_t pix = i / C;
        const int ow = (int)(pix % OW);
        const int64_t t = pix / OW;
        const int oh = (int)(t % OH);
        const int64_t b = t / OH;
        float m = -INFINITY;
        int best = -1;
        for (int kh = 0; kh < 3; ++kh) {
            const int ih = oh * 2 - 1 + kh;
            if (ih < 0 || ih >= H) continue;
            for (int kw = 0; kw < 3; ++kw) {
                const int iw = ow * 2 - 1 + kw;
                if (iw < 0 || iw >= W) continue;
                const float v = x[((b * H + ih) * W + iw) * C + c];
                if (best < 0 || v > m || isnan(v)) { m = v; best = kh * 3 + kw; }
            }
        }
        y[i] = m;
        idx[i] = (uint8_t)best;
    }
}

// backward of the pool (gather): dx[b, ih, iw, c] = sum, over the <= 2x2 windows covering (ih, iw) in (oh, ow) order,
// of dy where the window's stored index points at (ih, iw) -- the order autograd's scatter-add visits them
__global__ void __launch_bounds__(256) maxpool3s2_bwd_kernel(const float* __restrict__ dy, const uint8_t* __restrict__ idx,
                                                             float* __restrict__ dx, int64_t B, int C, int H, int W,
                                                             int OH, int OW) {
    const int64_t total = B * H * W * (int64_t)C;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const int64_t pix = i / C;
        const int iw = (int)(pix % W);
        const int64_t t = pix / W;
        const int ih = (int)(t % H);
        const int64_t b = t / H;
        float s = 0.f;
        // window oh covers rows 2*oh-1 .. 2*oh+1
        for (int oh = ih / 2; oh <= (ih + 1) / 2; ++oh) {
            if (oh >= OH) continue;
            const int kh = ih - (oh * 2 - 1);
            for (int ow = iw / 2; ow <= (iw + 1) / 2; ++ow) {
                if (ow >= OW) continue;
                const int kw = iw - (ow * 2 - 1);
                const int64_t o = ((b * OH + oh) * OW + ow) * C + c;
                if (idx[o] == kh * 3 + kw) s += dy[o];
            }
        }
        dx[i] = s;
    }
}

// [B, P, C] (NHWC rows) <-> [B, C, P] (the reference's (C, H, W) flatten); tiny (conv head output)
// act: applied on the way (the ResnetEncoder's final activation, encoder.py:202, fused into the flatten permute)
__global__ void __launch_bounds__(256) permute_bpc_kernel(const float* __restrict__ src, float* __restrict__ dst, int64_t B,
                                                          int P, int C, int to_cp, int act) {
    const int64_t total = B * P * (int64_t)C;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        // i indexes dst
        const int64_t b = i / ((int64_t)P * C);
        const int r = (int)(i - b * P * C);
        int p, c;
        if (to_cp) { c = r / P; p = r - c * P; }   // dst [B, C, P]
        else { p = r / C; c = r - p * C; }          // dst [B, P, C]
        const int64_t s = to_cp ? (b * P + p) * C + c : (b * C + c) * P + p;
        dst[i] = act_fwd(src[s], act);
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
    return sfb200_im2col_pad_act(x, in_nchw, B, C, H, W, kernel, stride, 0, SFB200_ACT_NONE, col, stream);
}

int sfb200_im2col_pad_act(const float* x, int in_nchw, int64_t B, int C, int H, int W, int kernel, int stride, int pad,
                          int act, float* col, void* stream) {
    SFB_CHECK_ARG(x && col && B >= 0 && C > 0 && kernel > 0 && stride > 0 && pad >= 0 && pad < kernel &&
                      H + 2 * pad >= kernel && W + 2 * pad >= kernel,
                  "im2col: bad arguments");
    if (B == 0) return 0;
    const int OH = (H + 2 * pad - kernel) / stride + 1, OW = (W + 2 * pad - kernel) / stride + 1;
    const int64_t total = B * OH * OW * (int64_t)C * kernel * kernel;
    cudaStream_t st = (cudaStream_t)stream;
    if (in_nchw)
        im2col_kernel<true><<<conv_grid(total), 256, 0, st>>>(x, col, B, C, H, W, kernel, stride, pad, act, OH, OW);
    else im2col_kernel<false><<<conv_grid(total), 256, 0, st>>>(x, col, B, C, H, W, kernel, stride, pad, act, OH, OW);
    SFB_LAUNCH_OK();
    return 0;
}

int sfb200_col2im_act_backward(const float* dcol, const float* x_act, int64_t B, int C, int H, int W, int kernel,
                               int stride, int act, float* dx, void* stream) {
    return sfb200_col2im_pad_act_backward(dcol, x_act, 0, nullptr, B, C, H, W, kernel, stride, 0, act, dx, stream);
}

int sfb200_col2im_pad_act_backward(const float* dcol, const float* x_act, int from_input, const float* dres, int64_t B,
                                   int C, int H, int W, int kernel, int stride, int pad, int act, float* dx, void* stream) {
    SFB_CHECK_ARG(dcol && x_act && dx && B >= 0 && C > 0 && kernel > 0 && stride > 0 && pad >= 0 && pad < kernel &&
                      H + 2 * pad >= kernel && W + 2 * pad >= kernel,
                  "col2im_act_backward: bad arguments");
    if (B == 0) return 0;
    const int OH = (H + 2 * pad - kernel) / stride + 1, OW = (W + 2 * pad - kernel) / stride + 1;
    col2im_kernel<<<conv_grid(B * H * W * (int64_t)C), 256, 0, (cudaStream_t)stream>>>(
        dcol, x_act, dres, dx, B, C, H, W, kernel, stride, pad, OH, OW, act, from_input);
    SFB_LAUNCH_OK();
    return 0;
}

int sfb200_maxpool3s2_forward(const float* x, int64_t B, int C, int H, int W, float* y, uint8_t* idx, void* stream) {
    SFB_CHECK_ARG(x && y && idx && B >= 0 && C > 0 && H > 0 && W > 0, "maxpool3s2_forward: bad arguments");
    if (B == 0) return 0;
    const int OH = (H + 1) / 2, OW = (W + 1) / 2;
    maxpool3s2_kernel<<<conv_grid(B * OH * OW * (int64_t)C), 256, 0, (cudaStream_t)stream>>>(x, y, idx, B, C, H, W, OH, OW);
    SFB_LAUNCH_OK();
    return 0;
}

int sfb200_maxpool3s2_backward(const float* dy, const uint8_t* idx, int64_t B, int C, int H, int W, float* dx,
                               void* stream) {
    SFB_CHECK_ARG(dy && idx && dx && B >= 0 && C > 0 && H > 0 && W > 0, "maxpool3s2_backward: bad arguments");
    if (B == 0) return 0;
    const int OH = (H + 1) / 2, OW = (W + 1) / 2;
    maxpool3s2_bwd_kernel<<<conv_grid(B * H * W * (int64_t)C), 256, 0, (cudaStream_t)stream>>>(dy, idx, dx, B, C, H, W, OH,
                                                                                             OW);
    SFB_LAUNCH_OK();
    return 0;
}

int sfb200_permute_bpc(const float* src, float* dst, int64_t B, int P, int C, int to_channel_major, void* stream) {
    SFB_CHECK_ARG(src && dst && B >= 0 && P > 0 && C > 0, "permute_bpc: bad arguments");
    if (B == 0) return 0;
    permute_bpc_kernel<<<conv_grid(B * P * (int64_t)C), 256, 0, (cudaStream_t)stream>>>(src, dst, B, P, C, to_channel_major,
                                                                                       SFB200_ACT_NONE);
    SFB_LAUNCH_OK();
    return 0;
}

int sfb200_act_permute_bpc(const float* src, float* dst, int64_t B, int P, int C, int act, void* stream) {
    SFB_CHECK_ARG(src && dst && B >= 0 && P > 0 && C > 0, "act_permute_bpc: bad arguments");
    if (B == 0) return 0;
    permute_bpc_kernel<<<conv_grid(B * P * (int64_t)C), 256, 0, (cudaStream_t)stream>>>(src, dst, B, P, C, 1, act);
    SFB_LAUNCH_OK();
    return 0;
}

}  // extern "C"
