"""Recurrent core on the device: the reference's ModelCoreRNN (model/core.py:19-64, nn.GRU / nn.LSTM with
rnn_num_layers stacked layers) and the learner's done-aware BPTT (algo/learning/learner.py:556-577,
algo/learning/rnn_utils.py:11-158).

The reference packs every run of steps between done-or-invalid boundaries into a PackedSequence so cuDNN never carries
state across an episode boundary.  On the device the same computation is a masked time loop over the `recurrence`
steps of all chunks at once: a row whose previous step was done-or-invalid starts from a ZERO state (rnn_utils.py:143-149)
and the backward pass cuts the gradient at the same places; a chunk's first step starts from the stored rnn_state
(constant).  Every step is: two GEMMs on the wgmma engine (x.W_ih^T batched over ALL steps up front, h.W_hh^T per
step) + one fused cell kernel (csrc/rnn.cu).  The weight gradients are two large GEMMs over the stacked time-major
buffers, not R small ones.

Stacked layers run one after the other over the whole chunk: layer k's input for every step is layer k-1's output
h, so its x.W_ih^T is again one GEMM over all steps.  A state row is layer-major (core.py:42-60): layer k owns the
columns [k*Sl, (k+1)*Sl) with Sl = H (GRU, h) or 2H (LSTM, [h | c]); every kernel addresses its slice through a pointer
offset and the full row stride.  A slice that starts off a 16-byte boundary (H % 4 != 0) is an operand TMA cannot
describe, and the GEMM engine takes its SIMT path for it.

Separate actor / critic weights (ActorCriticSeparateWeights._core_rnn, model/actor_critic.py:228-273) run one RnnCore
per tower: it is bound to its parameters (prefix "actor_core." / "critic_core.") and to its half of the state row
[actor state | critic state] by a column offset, so neither tower's state is split off or concatenated back.  The two
towers' BPTT buffers keep what each backward reads back; the scratch one backward uses at a time and the reset mask are
shared (alloc_bptt(shared=...)), since the towers run one after the other.
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import Tensor

from . import ops
from .model import PolicyModel


class RnnCore:
    def __init__(self, model: PolicyModel, engine: int, tower: str = ""):
        """tower: "" (the shared model's core), "actor_" or "critic_" (one tower of a separate-weights model)"""
        self.model = model
        self.spec = model.spec
        self.engine = engine
        self.tower = tower
        self.H = self.spec.rnn_size
        self.G = self.spec.rnn_gates
        self.S = self.spec.rnn_state_size            # the full state row
        self.L = self.spec.rnn_num_layers
        self.Sl = self.spec.rnn_layer_state_size     # one layer's columns of a state row
        self.col = self.spec.rnn_tower_state_size if tower == "critic_" else 0     # first column of this core's half
        self.is_lstm = self.spec.rnn_type == "lstm"
        self.none = ops.ACT["none"]

    def _params(self, grads: bool = False, layer: int = 0):
        return self.model.rnn_params(grads=grads, layer=layer, tower=self.tower)

    def _slice(self, state: Tensor, k: int) -> Tensor:
        """layer k's columns of this core in [rows, S] state rows"""
        c = self.col + k * self.Sl
        return state[:, c: c + self.Sl]

    # ------------------------------------------------------------------------------------------------ single step
    def alloc_step(self, M: int):
        dev, H, G = self.model.device, self.H, self.G
        f32 = dict(dtype=torch.float32, device=dev)
        return dict(gi=torch.empty((M, G * H), **f32), gh=torch.empty((M, G * H), **f32))

    def step(self, x: Tensor, state_in: Tensor, state_out: Tensor, bufs) -> Tensor:
        """One recurrent step for M rows (sampler step / bootstrap value). Returns the core output view [M, H]
        (the top layer's new h)."""
        H = self.H
        for k in range(self.L):
            W_ih, W_hh, b_ih, b_hh = self._params(layer=k)
            s_in, s_out = self._slice(state_in, k), self._slice(state_out, k)
            ops.linear_act_forward(x, W_ih, b_ih, bufs["gi"], self.none, self.engine)
            ops.linear_act_forward(s_in[:, :H], W_hh, b_hh, bufs["gh"], self.none, self.engine)
            if self.is_lstm:
                ops.lstm_cell_forward(bufs["gi"], bufs["gh"], s_in, s_out)
            else:
                ops.gru_cell_forward(bufs["gi"], bufs["gh"], s_in, s_out)
            x = s_out[:, :H]
        return x

    # ------------------------------------------------------------------------------------------------ BPTT
    def alloc_bptt(self, B: int, R: int, shared: Optional[dict] = None):
        """Per layer only what the backward reads back (gates, gh for the GRU, input / output states, core_out); the
        GEMM outputs and gradient scratch that one layer uses at a time are shared by all layers.  shared: the buffers of
        the other tower's core -- its scratch and reset mask serve this core too."""
        dev, H, G, Sl = self.model.device, self.H, self.G, self.Sl
        n = B // R
        f32 = dict(dtype=torch.float32, device=dev)
        gh_shared = None    # the LSTM backward never reads gh: one buffer serves every layer (and both towers)
        if self.is_lstm:
            gh_shared = shared["layers"][0]["gh"] if shared is not None else torch.empty((R, n, G * H), **f32)
        layers = []
        for _ in range(self.L):
            layers.append(dict(
                gh=gh_shared if gh_shared is not None else torch.empty((R, n, G * H), **f32),   # time-major
                gates=torch.empty((R, n, G * H), **f32),
                state_in=torch.empty((R + 1, n, Sl), **f32),      # input state of step t (after the reset mask)
                state_out=torch.empty((R, n, Sl), **f32) if self.is_lstm else None,   # unmasked output state of step t
                core_out=torch.empty((B, H), **f32),              # env-major: row c*R + t
            ))
        b = dict(n=n, R=R, layers=layers, core_out=layers[-1]["core_out"])      # the core's output: the top layer's h
        if shared is not None:
            b.update({k: v for k, v in shared.items() if k not in b})
            return b
        b.update(
            gi_all=torch.empty((B, G * H), **f32),            # env-major: row c*R + t
            dgi_all=torch.empty((B, G * H), **f32),
            dgh=torch.empty((R, n, G * H), **f32),
            carry_gemm=torch.empty((n, H), **f32),
            carry_direct=[torch.empty((n, H), **f32) for _ in range(2)],
            # dL/d core_out of the layer below the one running its backward (written by that layer's dX GEMM)
            d_core_below=torch.empty((B, H), **f32) if self.L > 1 else None,
            doi=torch.empty((n, R), dtype=torch.bool, device=dev),
            colsum_ws=torch.empty(ops.colsum_workspace_bytes(G * H) // 4 + 4, **f32),
        )
        return b

    def forward_bptt(self, head: Tensor, rnn_states: Tensor, dones: Optional[Tensor], valids: Tensor, b) -> Tensor:
        """head [B, in] env-major (row c*R+t); rnn_states [B, S] stored states (only rows c*R are used);
        dones / valids [B] bool (dones None: the reset mask in b is already this minibatch's, computed by the other
        tower's core).  Returns core_out [B, H] env-major."""
        n, R, H, G, S = b["n"], b["R"], self.H, self.G, self.S
        if dones is not None:
            torch.logical_or(dones.view(n, R), ~valids.view(n, R), out=b["doi"])      # done_or_invalid, learner.py:560
        gi3 = b["gi_all"].view(n, R, G * H)
        x = head
        for k, lb in enumerate(b["layers"]):
            W_ih, W_hh, b_ih, b_hh = self._params(layer=k)
            ops.linear_act_forward(x, W_ih, b_ih, b["gi_all"], self.none, self.engine)
            ops.copy_rows(self._slice(rnn_states.view(n, R * S), k), lb["state_in"][0])   # chunk-start states
            core3 = lb["core_out"].view(n, R, H)
            for t in range(R):
                s_in = lb["state_in"][t]
                ops.linear_act_forward(s_in[:, :H], W_hh, b_hh, lb["gh"][t], self.none, self.engine)
                reset_next = b["doi"][:, t]
                if self.is_lstm:
                    s_out = lb["state_out"][t]
                    ops.lstm_cell_forward(gi3[:, t], lb["gh"][t], s_in, s_out, lb["state_in"][t + 1], reset_next,
                                          lb["gates"][t])
                    ops.copy_rows(s_out[:, :H], core3[:, t])
                else:
                    ops.gru_cell_forward(gi3[:, t], lb["gh"][t], s_in, core3[:, t], lb["state_in"][t + 1], reset_next,
                                         lb["gates"][t])
            x = lb["core_out"]
        return b["core_out"]

    def backward_bptt(self, d_core: Tensor, b, lin_ws: Tensor) -> Tensor:
        """d_core [B, H] env-major = dL/d core_out.  Fills the gradients of every layer's W_hh, b_ih, b_hh and of W_ih
        above layer 0, and returns layer 0's dgi_all [B, G*H] env-major (the caller turns it into dW_ih of layer 0 and
        the encoder gradient with one linear_backward)."""
        n, R, H, G = b["n"], b["R"], self.H, self.G
        dgi3 = b["dgi_all"].view(n, R, G * H)
        for k in range(self.L - 1, -1, -1):
            lb = b["layers"][k]
            W_ih, W_hh, b_ih, b_hh = self._params(layer=k)
            dW_ih, dW_hh, db_ih, db_hh = self._params(grads=True, layer=k)
            dcore3 = (d_core if k == self.L - 1 else b["d_core_below"]).view(n, R, H)
            carry_gemm: Optional[Tensor] = None
            carry_direct: Optional[Tensor] = None
            for t in range(R - 1, -1, -1):
                reset = b["doi"][:, t] if t < R - 1 else None      # boundary between step t and t+1
                direct = b["carry_direct"][t & 1]
                if self.is_lstm:
                    ops.lstm_cell_backward(dcore3[:, t], carry_gemm, carry_direct, reset, lb["gates"][t],
                                           lb["state_in"][t], lb["state_out"][t], b["dgh"][t], direct)
                    ops.copy_rows(b["dgh"][t], dgi3[:, t])          # dgi == dgh for the LSTM
                else:
                    ops.gru_cell_backward(dcore3[:, t], carry_gemm, carry_direct, reset, lb["gates"][t], lb["gh"][t],
                                          lb["state_in"][t][:, :H], dgi3[:, t], b["dgh"][t], direct)
                carry_direct = direct
                if t > 0:
                    # gradient through h_in(t) = masked h_out(t-1):  dgh(t) . W_hh
                    ops.linear_backward(b["dgh"][t], lb["state_in"][t][:, :H], W_hh, self.none, None, b["carry_gemm"],
                                        None, self.engine, lin_ws)
                    carry_gemm = b["carry_gemm"]
            # weight gradients over the stacked time-major buffers
            dgh_all = b["dgh"].view(R * n, G * H)
            h_in_all = lb["state_in"][:R].view(R * n, self.Sl)[:, :H]
            ops.linear_backward(dgh_all, h_in_all, W_hh, self.none, dW_hh, None, None, self.engine, lin_ws)
            ops.colsum(dgh_all, db_hh, b["colsum_ws"])
            ops.colsum(b["dgi_all"], db_ih, b["colsum_ws"])
            if k > 0:
                # layer k's input is layer k-1's output: dW_ih of layer k and dL/d core_out of layer k-1 in one call
                ops.linear_backward(b["dgi_all"], b["layers"][k - 1]["core_out"], W_ih, self.none, dW_ih,
                                    b["d_core_below"], None, self.engine, lin_ws)
        return b["dgi_all"]

    def lin_ws_bytes(self, B: int, R: int, in_size: int) -> int:
        n = B // R
        G, H = self.G, self.H
        ws = max(ops.linear_backward_workspace_bytes(R * n, G * H, H), ops.linear_backward_workspace_bytes(n, G * H, H),
                 ops.linear_backward_workspace_bytes(B, G * H, in_size))
        if self.L > 1:      # dW_ih / dX of the layers above the first: [B, G*H] x H
            ws = max(ws, ops.linear_backward_workspace_bytes(B, G * H, H))
        return ws
