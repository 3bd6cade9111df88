"""Conv head of the reference's ConvEncoder (model/encoder.py:88-145) on the device.

Every Conv2d (no padding) runs as  im2col -> GEMM engine  with bias + activation in the GEMM epilogue, so the wgmma
3xTF32 path and its backward GEMMs are shared with the MLP layers (csrc/conv.cu explains the layouts).  Activations are
kept NHWC ([B*OH*OW, C] rows = GEMM output); the last layer is permuted to the (C, H, W) flatten order the reference's
fully connected layers expect (encoder.py:115), so the weights keep the reference layout and checkpoints round-trip.
"""
from __future__ import annotations

from typing import List, Optional

import torch
from torch import Tensor

from . import ops
from .model import PolicyModel


class ConvHead:
    """Buffers + launch sequence for the conv head of one model at up to `max_rows` observations per call."""

    def __init__(self, model: PolicyModel, engine: int, max_rows: int, need_backward: bool):
        self.model, self.engine, self.max_rows = model, engine, max_rows
        spec = model.spec
        self.layers = spec.conv_layers
        assert self.layers, "ConvHead needs image observations (spec.obs_shape)"
        self.act = ops.ACT[spec.nonlinearity]
        dev = model.device
        f32 = dict(dtype=torch.float32, device=dev)
        self.col: List[Tensor] = []     # im2col matrices [rows*OH*OW, C_in*k*k]  (reused as d(col) in the backward)
        self.y: List[Tensor] = []       # activated outputs, NHWC [rows*OH*OW, C_out]
        self.dz: List[Tensor] = []      # gradients w.r.t. the pre-activations, same shape as y
        lin_ws = 4
        max_c = 1
        for (ci, h, w, co, k, s, ho, wo) in self.layers:
            self.col.append(torch.empty((max_rows * ho * wo, ci * k * k), **f32))
            self.y.append(torch.empty((max_rows * ho * wo, co), **f32))
            if need_backward:
                self.dz.append(torch.empty((max_rows * ho * wo, co), **f32))
                lin_ws = max(lin_ws, ops.linear_backward_workspace_bytes(max_rows * ho * wo, co, ci * k * k) // 4 + 4)
            max_c = max(max_c, co)
        self.feat = torch.empty((max_rows, spec.conv_out_size), **f32)   # (C,H,W)-flattened output of the head
        if need_backward:
            self.lin_ws = torch.empty(lin_ws, **f32)
            self.colsum_ws = torch.empty(ops.colsum_workspace_bytes(max_c) // 4 + 4, **f32)

    # ------------------------------------------------------------------------------------------------------------
    def forward(self, x: Tensor) -> Tensor:
        """x: [M, C*H*W] normalised observations, rows in (C,H,W) order (may be a strided row view) -> [M, conv_out]"""
        M = x.shape[0]
        assert M <= self.max_rows
        if not x.is_contiguous():
            x = x.contiguous()
        src, nchw = x, True
        for li, ((ci, h, w, co, k, s, ho, wo), (W, b)) in enumerate(zip(self.layers, self.model.conv_params())):
            col = self.col[li][: M * ho * wo]
            y = self.y[li][: M * ho * wo]
            ops.im2col(src, nchw, M, ci, h, w, k, s, col)
            ops.linear_act_forward(col, W.view(co, ci * k * k), b, y, self.act, self.engine)   # Conv2d + activation
            src, nchw = y, False
        ci, h, w, co, k, s, ho, wo = self.layers[-1]
        ops.permute_bpc(src, self.feat[:M], M, ho * wo, co, True)     # NHWC rows -> (C,H,W) flatten (encoder.py:115)
        return self.feat[:M]

    def backward(self, dfeat: Tensor) -> None:
        """dfeat: [M, conv_out] gradient w.r.t. the PRE-activation of the last conv layer in (C,H,W) flatten order (the
        first fully connected layer's backward applies act' of `feat`).  Accumulates nothing: writes the conv weight /
        bias gradients of this minibatch into model.grads."""
        M = dfeat.shape[0]
        L = len(self.layers)
        ci, h, w, co, k, s, ho, wo = self.layers[-1]
        ops.permute_bpc(dfeat, self.dz[L - 1][: M * ho * wo], M, ho * wo, co, False)
        params, grads = self.model.conv_params(), self.model.conv_params(grads=True)
        none = ops.ACT["none"]
        for li in range(L - 1, -1, -1):
            ci, h, w, co, k, s, ho, wo = self.layers[li]
            rows = M * ho * wo
            dz = self.dz[li][:rows]
            col = self.col[li][:rows]
            W, _ = params[li]
            gW, gb = grads[li]
            ops.colsum(dz, gb, self.colsum_ws)                                       # bias gradient
            if li > 0:
                # dW = dz^T col ; d(col) = dz W  (overwrites col: it is not needed after dW)
                ops.linear_backward(dz, col, W.view(co, ci * k * k), none, gW.view(co, ci * k * k), col, None,
                                    self.engine, self.lin_ws)
                pci, ph, pw, pco, pk, ps, pho, pwo = self.layers[li - 1]
                # col2im + activation derivative of the previous layer's (activated, NHWC) output
                ops.col2im_act_backward(col, self.y[li - 1][: M * pho * pwo], M, ci, h, w, k, s, self.act,
                                        self.dz[li - 1][: M * pho * pwo])
            else:
                ops.linear_backward(dz, col, W.view(co, ci * k * k), none, gW.view(co, ci * k * k), None, None,
                                    self.engine, self.lin_ws)


class ResnetHead:
    """Buffers + launch sequence for the reference's ResnetEncoder conv head (model/encoder.py:153-221, resnet_impala) at
    up to `max_rows` observations per call; the interface of ConvHead (forward -> feat, backward(dfeat), .feat).

    Per stage:  z = conv(x, pad 1)  ->  x0 = maxpool3s2(z) (+ uint8 argmax indices)  ->  per block
    a = conv_a(act(x_j))  and  x_{j+1} = conv_b(act(a)) + x_j  (residual GEMM epilogue).  Both activations are applied
    by the im2col that feeds the conv (expm1f for ELU, as torch computes it, rather than the wgmma epilogue's fast-exp
    ELU), and the backward takes act' from the stored activation inputs x_j and a, as autograd's elu_backward does.
    After the last stage  feat = act(x)  in (C,H,W) order.
    Memory: ONE im2col scratch sized by the largest conv (the backward recomputes each conv's im2col instead of keeping
    one per layer), the block inputs / inner activations (NHWC) and pool indices, one pre-pool scratch shared with the
    pool's input gradient, and three gradient buffers (ping-pong + the inner d(pre-activation))."""

    def __init__(self, model: PolicyModel, engine: int, max_rows: int, need_backward: bool):
        self.model, self.engine, self.max_rows = model, engine, max_rows
        spec = model.spec
        assert spec.is_resnet
        self.stages = spec.resnet_stages
        self.act = ops.ACT[spec.nonlinearity]
        f32 = dict(dtype=torch.float32, device=model.device)
        col_k = max(max(h * w * ci * 9, hp * wp * co * 9) for (ci, h, w, co, hp, wp, _b) in self.stages)
        self.col = torch.empty(max_rows * col_k, **f32)
        self.z = torch.empty(max_rows * max(h * w * co for (_ci, h, w, co, _hp, _wp, _b) in self.stages), **f32)
        # x[s] = [x_0, x_1, ..., x_blocks] (block inputs; x_blocks is the stage output), a[s] = conv_a outputs
        self.x: List[List[Tensor]] = []
        self.a: List[List[Tensor]] = []
        self.idx: List[Tensor] = []
        for (_ci, _h, _w, co, hp, wp, blocks) in self.stages:
            rows = max_rows * hp * wp
            self.x.append([torch.empty((rows, co), **f32) for _ in range(blocks + 1)])
            self.a.append([torch.empty((rows, co), **f32) for _ in range(blocks)])
            self.idx.append(torch.empty((rows, co), dtype=torch.uint8, device=model.device))
        self.feat = torch.empty((max_rows, spec.conv_out_size), **f32)
        self.x_in: Optional[Tensor] = None
        if need_backward:
            g = max(hp * wp * co for (_ci, _h, _w, co, hp, wp, _b) in self.stages)
            self.g = [torch.empty(max_rows * g, **f32) for _ in range(3)]
            lin_ws, max_c = 4, 1
            for (ci, h, w, co, hp, wp, _b) in self.stages:
                lin_ws = max(lin_ws, ops.linear_backward_workspace_bytes(max_rows * h * w, co, ci * 9) // 4 + 4,
                             ops.linear_backward_workspace_bytes(max_rows * hp * wp, co, co * 9) // 4 + 4)
                max_c = max(max_c, co)
            self.lin_ws = torch.empty(lin_ws, **f32)
            self.colsum_ws = torch.empty(ops.colsum_workspace_bytes(max_c) // 4 + 4, **f32)

    @staticmethod
    def _view(buf: Tensor, rows: int, cols: int) -> Tensor:
        return buf[: rows * cols].view(rows, cols)

    # ------------------------------------------------------------------------------------------------------------
    def forward(self, x: Tensor) -> Tensor:
        """x: [M, C*H*W] normalised observations, rows in (C,H,W) order -> [M, conv_out] = act(conv head output)"""
        M = x.shape[0]
        assert M <= self.max_rows
        if not x.is_contiguous():
            x = x.contiguous()
        self.x_in = x                     # the first conv's im2col is recomputed from it in the backward
        params = iter(self.model.conv_params())
        none = ops.ACT["none"]
        src, nchw = x, True
        for s, (ci, h, w, co, hp, wp, blocks) in enumerate(self.stages):
            W, b = next(params)
            col = self._view(self.col, M * h * w, ci * 9)
            z = self._view(self.z, M * h * w, co)
            ops.im2col_pad_act(src, nchw, M, ci, h, w, 3, 1, 1, none, col)
            ops.linear_act_forward(col, W.view(co, ci * 9), b, z, none, self.engine)       # Conv2d(3, padding 1)
            ops.maxpool3s2_forward(z, M, co, h, w, self.x[s][0][: M * hp * wp], self.idx[s][: M * hp * wp])
            col = self._view(self.col, M * hp * wp, co * 9)
            for j in range(blocks):
                (Wa, ba), (Wb, bb) = next(params), next(params)
                xj, aj, xn = (t[: M * hp * wp] for t in (self.x[s][j], self.a[s][j], self.x[s][j + 1]))
                ops.im2col_pad_act(xj, False, M, co, hp, wp, 3, 1, 1, self.act, col)                # act(x), padded
                ops.linear_act_forward(col, Wa.view(co, co * 9), ba, aj, none, self.engine)       # conv_a(.)
                ops.im2col_pad_act(aj, False, M, co, hp, wp, 3, 1, 1, self.act, col)                # act(a), padded
                ops.linear_residual_forward(col, Wb.view(co, co * 9), bb, xj, xn, self.engine)   # conv_b(.) + x
            src, nchw = self.x[s][blocks][: M * hp * wp], False
        _ci, _h, _w, co, hp, wp, _b = self.stages[-1]
        ops.act_permute_bpc(src, self.feat[:M], M, hp * wp, co, self.act)    # act, (C,H,W) flatten (encoder.py:202, 217)
        return self.feat[:M]

    def backward(self, dfeat: Tensor) -> None:
        """dfeat: [M, conv_out] gradient w.r.t. the conv head's output BEFORE its final activation, (C,H,W) order (the
        first fully connected layer's backward applies act' of `feat`).  Writes the conv weight / bias gradients of this
        minibatch into model.grads.  Needs the activations of the last forward() on the same rows."""
        M = dfeat.shape[0]
        none = ops.ACT["none"]
        params, grads = self.model.conv_params(), self.model.conv_params(grads=True)
        li = len(params)
        _ci, _h, _w, co, hp, wp, _b = self.stages[-1]
        gi = 0                                                        # ping-pong index of the current gradient
        g = self._view(self.g[gi], M * hp * wp, co)
        ops.permute_bpc(dfeat, g, M, hp * wp, co, False)
        for s in range(len(self.stages) - 1, -1, -1):
            ci, h, w, co, hp, wp, blocks = self.stages[s]
            rows = M * hp * wp
            col = self._view(self.col, rows, co * 9)
            for j in range(blocks - 1, -1, -1):
                li -= 2
                (Wa, _), (Wb, _) = params[li], params[li + 1]
                (gWa, gba), (gWb, gbb) = grads[li], grads[li + 1]
                xj, aj = self.x[s][j][:rows], self.a[s][j][:rows]
                dza = self._view(self.g[2], rows, co)
                # conv_b: dW = g^T im2col(act(a)), db = colsum(g), d(col) = g W (in place of col), then act'(a)
                ops.colsum(g, gbb, self.colsum_ws)
                ops.im2col_pad_act(aj, False, M, co, hp, wp, 3, 1, 1, self.act, col)
                ops.linear_backward(g, col, Wb.view(co, co * 9), none, gWb.view(co, co * 9), col, None, self.engine,
                                    self.lin_ws)
                ops.col2im_pad_act_backward(col, aj, True, None, M, co, hp, wp, 3, 1, 1, self.act, dza)
                # conv_a on act(x_j): dx_j = col2im(dcol) * act'(x_j) + g (identity path)
                ops.colsum(dza, gba, self.colsum_ws)
                ops.im2col_pad_act(xj, False, M, co, hp, wp, 3, 1, 1, self.act, col)
                ops.linear_backward(dza, col, Wa.view(co, co * 9), none, gWa.view(co, co * 9), col, None, self.engine,
                                    self.lin_ws)
                gn = self._view(self.g[1 - gi], rows, co)
                ops.col2im_pad_act_backward(col, xj, True, g, M, co, hp, wp, 3, 1, 1, self.act, gn)
                g, gi = gn, 1 - gi
            # max-pool, then the stage-entry conv
            li -= 1
            W, _ = params[li]
            gW, gb = grads[li]
            dz = self._view(self.z, M * h * w, co)
            ops.maxpool3s2_backward(g, self.idx[s][:rows], M, co, h, w, dz)
            ops.colsum(dz, gb, self.colsum_ws)
            col = self._view(self.col, M * h * w, ci * 9)
            if s > 0:
                prev = self.x[s - 1][-1][: M * h * w]
                ops.im2col_pad_act(prev, False, M, ci, h, w, 3, 1, 1, none, col)
                ops.linear_backward(dz, col, W.view(co, ci * 9), none, gW.view(co, ci * 9), col, None, self.engine,
                                    self.lin_ws)
                gn = self._view(self.g[1 - gi], M * h * w, ci)
                ops.col2im_pad_act_backward(col, prev, False, None, M, ci, h, w, 3, 1, 1, none, gn)
                g, gi = gn, 1 - gi
            else:
                ops.im2col_pad_act(self.x_in, True, M, ci, h, w, 3, 1, 1, none, col)
                ops.linear_backward(dz, col, W.view(co, ci * 9), none, gW.view(co, ci * 9), None, None, self.engine,
                                    self.lin_ws)
