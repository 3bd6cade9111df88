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
