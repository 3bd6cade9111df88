"""Recurrent core on the device: the reference's ModelCoreRNN (model/core.py:19-64, one-layer nn.GRU / nn.LSTM) and the
learner's done-aware BPTT (algo/learning/learner.py:556-577, algo/learning/rnn_utils.py:11-158).

The reference packs every run of steps between done-or-invalid boundaries into a PackedSequence so cuDNN never carries
state across an episode boundary.  On the device the same computation is a masked time loop over the `recurrence`
steps of all chunks at once: a row whose previous step was done-or-invalid starts from a ZERO state (rnn_utils.py:143-149)
and the backward pass cuts the gradient at the same places; a chunk's first step starts from the stored rnn_state
(constant).  Every step is: two GEMMs on the wgmma engine (x.W_ih^T batched over ALL steps up front, h.W_hh^T per
step) + one fused cell kernel (csrc/rnn.cu).  The weight gradients are two large GEMMs over the stacked time-major
buffers, not R small ones.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
from torch import Tensor

from . import ops
from .model import PolicyModel


class RnnCore:
    def __init__(self, model: PolicyModel, engine: int):
        self.model = model
        self.spec = model.spec
        self.engine = engine
        self.H = self.spec.rnn_size
        self.G = self.spec.rnn_gates
        self.S = self.spec.rnn_state_size
        self.is_lstm = self.spec.rnn_type == "lstm"
        self.none = ops.ACT["none"]

    # ------------------------------------------------------------------------------------------------ single step
    def alloc_step(self, M: int):
        dev, H, G = self.model.device, self.H, self.G
        f32 = dict(dtype=torch.float32, device=dev)
        return dict(gi=torch.empty((M, G * H), **f32), gh=torch.empty((M, G * H), **f32))

    def step(self, x: Tensor, state_in: Tensor, state_out: Tensor, bufs) -> Tensor:
        """One recurrent step for M rows (sampler step / bootstrap value). Returns the core output view [M, H]."""
        W_ih, W_hh, b_ih, b_hh = self.model.rnn_params()
        H = self.H
        ops.linear_act_forward(x, W_ih, b_ih, bufs["gi"], self.none, self.engine)
        ops.linear_act_forward(state_in[:, :H], W_hh, b_hh, bufs["gh"], self.none, self.engine)
        if self.is_lstm:
            ops.lstm_cell_forward(bufs["gi"], bufs["gh"], state_in, state_out)
        else:
            ops.gru_cell_forward(bufs["gi"], bufs["gh"], state_in, state_out)
        return state_out[:, :H]

    # ------------------------------------------------------------------------------------------------ BPTT
    def alloc_bptt(self, B: int, R: int):
        dev, H, G, S = self.model.device, self.H, self.G, self.S
        n = B // R
        f32 = dict(dtype=torch.float32, device=dev)
        b = dict(
            n=n, R=R,
            gi_all=torch.empty((B, G * H), **f32),            # env-major: row c*R + t
            dgi_all=torch.empty((B, G * H), **f32),
            gh=torch.empty((R, n, G * H), **f32),             # time-major
            dgh=torch.empty((R, n, G * H), **f32),
            gates=torch.empty((R, n, G * H), **f32),
            state_in=torch.empty((R + 1, n, S), **f32),       # input state of step t (after the reset mask)
            state_out=torch.empty((R, n, S), **f32),          # unmasked output state of step t
            core_out=torch.empty((B, H), **f32),              # env-major
            carry_gemm=torch.empty((n, H), **f32),
            carry_direct=[torch.empty((n, H), **f32) for _ in range(2)],
            doi=torch.empty((n, R), dtype=torch.bool, device=dev),
            colsum_ws=torch.empty(ops.colsum_workspace_bytes(G * H) // 4 + 4, **f32),
        )
        return b

    def forward_bptt(self, head: Tensor, rnn_states: Tensor, dones: Tensor, valids: Tensor, b) -> Tensor:
        """head [B, in] env-major (row c*R+t); rnn_states [B, S] stored states (only rows c*R are used);
        dones / valids [B] bool.  Returns core_out [B, H] env-major."""
        W_ih, W_hh, b_ih, b_hh = self.model.rnn_params()
        n, R, H, G = b["n"], b["R"], self.H, self.G
        torch.logical_or(dones.view(n, R), ~valids.view(n, R), out=b["doi"])      # done_or_invalid, learner.py:560
        ops.linear_act_forward(head, W_ih, b_ih, b["gi_all"], self.none, self.engine)
        ops.copy_rows(rnn_states.view(n, R * self.S)[:, : self.S], b["state_in"][0])   # chunk-start states
        gi3 = b["gi_all"].view(n, R, G * H)
        core3 = b["core_out"].view(n, R, H)
        for t in range(R):
            s_in, s_out = b["state_in"][t], b["state_out"][t]
            ops.linear_act_forward(s_in[:, :H], W_hh, b_hh, b["gh"][t], self.none, self.engine)
            reset_next = b["doi"][:, t]
            if self.is_lstm:
                ops.lstm_cell_forward(gi3[:, t], b["gh"][t], s_in, s_out, b["state_in"][t + 1], reset_next, b["gates"][t])
                ops.copy_rows(s_out[:, :H], core3[:, t])
            else:
                ops.gru_cell_forward(gi3[:, t], b["gh"][t], s_in, core3[:, t], b["state_in"][t + 1], reset_next,
                                     b["gates"][t])
        return b["core_out"]

    def backward_bptt(self, d_core: Tensor, b, lin_ws: Tensor) -> Tensor:
        """d_core [B, H] env-major = dL/d core_out.  Fills the gradients of W_hh, b_ih, b_hh and returns dgi_all
        [B, G*H] env-major (the caller turns it into dW_ih and the encoder gradient with one linear_backward)."""
        W_ih, W_hh, b_ih, b_hh = self.model.rnn_params()
        dW_ih, dW_hh, db_ih, db_hh = self.model.rnn_params(grads=True)
        n, R, H, G = b["n"], b["R"], self.H, self.G
        dcore3 = d_core.view(n, R, H)
        dgi3 = b["dgi_all"].view(n, R, G * H)
        carry_gemm: Optional[Tensor] = None
        carry_direct: Optional[Tensor] = None
        for t in range(R - 1, -1, -1):
            reset = b["doi"][:, t] if t < R - 1 else None      # boundary between step t and t+1
            direct = b["carry_direct"][t & 1]
            if self.is_lstm:
                ops.lstm_cell_backward(dcore3[:, t], carry_gemm, carry_direct, reset, b["gates"][t], b["state_in"][t],
                                       b["state_out"][t], b["dgh"][t], direct)
                ops.copy_rows(b["dgh"][t], dgi3[:, t])          # dgi == dgh for the LSTM
            else:
                ops.gru_cell_backward(dcore3[:, t], carry_gemm, carry_direct, reset, b["gates"][t], b["gh"][t],
                                      b["state_in"][t][:, :H], dgi3[:, t], b["dgh"][t], direct)
            carry_direct = direct
            if t > 0:
                # gradient through h_in(t) = masked h_out(t-1):  dgh(t) . W_hh
                ops.linear_backward(b["dgh"][t], b["state_in"][t][:, :H], W_hh, self.none, None, b["carry_gemm"], None,
                                    self.engine, lin_ws)
                carry_gemm = b["carry_gemm"]
        # weight gradients over the stacked time-major buffers
        dgh_all = b["dgh"].view(R * n, G * H)
        h_in_all = b["state_in"][:R].view(R * n, self.S)[:, :H]
        ops.linear_backward(dgh_all, h_in_all, W_hh, self.none, dW_hh, None, None, self.engine, lin_ws)
        ops.colsum(dgh_all, db_hh, b["colsum_ws"])
        ops.colsum(b["dgi_all"], db_ih, b["colsum_ws"])
        return b["dgi_all"]

    def lin_ws_bytes(self, B: int, R: int, in_size: int) -> int:
        n = B // R
        G, H = self.G, self.H
        return max(ops.linear_backward_workspace_bytes(R * n, G * H, H), ops.linear_backward_workspace_bytes(n, G * H, H),
                   ops.linear_backward_workspace_bytes(B, G * H, in_size))
