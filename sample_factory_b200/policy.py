"""Forward pass of the actor-critic on the device: encoder MLP -> (recurrent core) -> decoder MLP -> heads
(reference: ActorCriticSharedWeights.forward_head / forward_core / forward_tail, model/actor_critic.py:160-195).

One function serves the three call sites of the hot path (sampler policy step, learner bootstrap value, learner
minibatch forward).  When the tensor feeding critic_linear / distribution_linear is the output of an MLP layer and the
wgmma engine covers the shape, that layer and the heads run as ONE GEMM whose epilogue leaves partial head dot
products (sfb200_linear_act_heads_forward) followed by a tiny finishing kernel (sfb200_heads_from_partials); the
activated layer output is stored only if the caller needs it (the learner's backward does, the sampler does not).

Dict observations with several keys (MultiInputEncoder) start with a key encoder stage: each key's MLP runs on its column
slice of the normalised rows and its last layer writes its block of one concatenated buffer, which then feeds the
recurrent core, the decoder MLP or (unfused) the heads like the output of a single encoder would.

Encoders without fully connected layers hand their input on unchanged: the heads (or the decoder / core) read the
normalised rows of a linear policy, or the conv head's features, through the unfused heads kernels.

Models whose distribution_linear has more than 31 rows, or whose rows do not fit the narrow heads forward's shared memory
(ModelSpec.wide_heads), store the last hidden layer, run
distribution_linear as a GEMM on the same engine straight into the logits' final place, and finish with
sfb200_heads_tail_wide (value head + distribution tail, one warp per row).
"""
from __future__ import annotations

import os
from typing import Callable, Dict, List, Optional

import torch
from torch import Tensor

from . import ops
from .model import TOWERS, PolicyModel


class HeadsPlan:
    """Per call-site forward plan: decides once per (model, engine) whether the fused last-layer + heads path applies,
    owns its scratch, and owns the conv head's buffers for image observations."""

    def __init__(self, model: PolicyModel, engine: int, max_rows: int, need_backward: bool = False):
        spec = model.spec
        self.conv = None
        if spec.obs_shape is not None:
            from .conv_encoder import ConvHead, ResnetHead

            self.conv = (ResnetHead if spec.is_resnet else ConvHead)(model, engine, max_rows, need_backward)
        self.tail_is_mlp = bool(spec.decoder_mlp_layers) or (not spec.use_rnn and bool(spec.fc_encoder_layers))
        self.engine = engine
        # Dict observations: per key the hidden activations of its MLP but the last, and the [rows, sum of the key output
        # widths] concatenation the last layers write (identity encoders: the normalised row itself is the concatenation)
        self.keys = spec.dict_obs and bool(spec.encoder_mlp_layers)
        if self.keys:
            f32 = dict(dtype=torch.float32, device=model.device)
            widths = spec.encoder_mlp_layers
            self.key_h = [[torch.empty((max_rows, w), **f32) for w in widths[:-1]] for _ in spec.obs_keys]
            self.enc_cat = torch.empty((max_rows, spec.fc_encoder_input), **f32)
            if need_backward:
                self.key_dz = [[torch.empty((max_rows, w), **f32) for w in widths[:-1]] for _ in spec.obs_keys]
                self.denc_cat = torch.empty((max_rows, spec.fc_encoder_input), **f32)
                self.db_enc_cat = torch.empty(spec.fc_encoder_input, **f32)
        # heads wider than 31 rows: no fused-partials path (P stays 0); call sites that sample without keeping the logits
        # get them in this scratch (so do Tuples with Box members, whose tail reads the stored params rows)
        self.wide = spec.wide_heads
        self.wide_logits: Optional[Tensor] = None
        if (self.wide or spec.action_heads) and not need_backward:
            self.wide_logits = torch.empty((max_rows, spec.num_action_params), dtype=torch.float32, device=model.device)
        # separate actor / critic weights: per-tower activations and ONE concatenated tail [rows, 2H] = [actor | critic].
        # tower_h[tw][i] / tower_dz[tw][i]: output of the tower's MLP layer i (encoder then decoder) and its gradient; the
        # layer that feeds the heads writes its half of tail_cat instead (None here).  With a recurrent core and no decoder
        # the core's output feeds the heads: every MLP layer keeps its buffer and the core output is copied into tail_cat.
        self.separate = spec.separate_towers
        if self.separate:
            f32 = dict(dtype=torch.float32, device=model.device)
            widths, H = spec.hidden, spec.tail_input_size
            self.tower_tail_is_mlp = bool(spec.decoder_mlp_layers) or not spec.use_rnn
            n_tail = 1 if self.tower_tail_is_mlp else 0

            def per_layer():
                return [torch.empty((max_rows, w), **f32) for w in widths[:len(widths) - n_tail]] + [None] * n_tail

            self.tower_h = {tw: per_layer() for tw in TOWERS}
            self.tail_cat = torch.empty((max_rows, 2 * H), **f32)
            if need_backward:
                A = spec.num_linear_action_outputs
                self.tower_dz = {tw: per_layer() for tw in TOWERS}
                self.dz_cat = torch.empty((max_rows, 2 * H), **f32)
                self.db_cat = torch.empty(2 * H, **f32)
                if not self.wide:     # (the wide backward writes the heads' gradients directly)
                    self.gWv_cat = torch.empty((1, 2 * H), **f32)
                    self.gWa_cat = torch.empty((A, 2 * H), **f32)
        self.P = 0
        if self.separate:
            return
        self.part: Optional[Tensor] = None
        if self.tail_is_mlp and not self.wide:
            self.P = ops.linear_heads_partials(spec.tail_input_size, spec.num_linear_action_outputs, engine)
        if self.P > 0:
            self.part = torch.empty(self.P * max_rows * ops.HEAD_PART_PAD, dtype=torch.float32, device=model.device)
            # optional: the GEMM finishes the heads itself (last-arriving CTA per 128-row block; these are its arrival
            # counters).  One launch less per policy step, but the finishing CTA walks its 128 rows 16 deep per warp while
            # heads_from_partials is fully parallel, so the separate launch stays the default.
            self.counters = torch.zeros((max_rows + 127) // 128, dtype=torch.int32, device=model.device)
            self.finish_in_gemm = os.environ.get("SFB200_HEADS_FINISH_IN_GEMM", "0") == "1" and not spec.action_heads


def forward_policy(model: PolicyModel, x: Tensor, outs: List[Tensor], act: int, engine: int, plan: HeadsPlan,
                   heads_kwargs: Dict, rnn_fn: Optional[Callable[[Tensor], Tensor]] = None,
                   store_tail: bool = True, finish_fn: Optional[Callable] = None,
                   tower_rnn_fns: Optional[Dict[str, Callable[[Tensor], Tensor]]] = None) -> Tensor:
    """x [M, D] (rows may be strided) -> heads outputs described by `heads_kwargs` (the keyword arguments of
    ops.heads_forward after the weights).  outs: one [>=M, h] buffer per MLP layer.  Returns the tensor that fed the
    heads (None if it was not stored).  Separate actor / critic weights with recurrent cores take one core function
    per tower in tower_rnn_fns ({"actor_": fn, "critic_": fn}) instead of rnn_fn."""
    M = x.shape[0]
    if plan.separate:
        return _forward_separate(model, x, act, engine, plan, heads_kwargs, tower_rnn_fns)
    if plan.conv is not None:        # ConvEncoder: conv head first, its fully connected layers are `enc` below
        x = plan.conv.forward(x)
    if plan.keys:                    # MultiInputEncoder: the key encoders write the concatenation, `enc` below is empty
        x = _forward_keys(model, x, act, engine, plan)
    enc, dec = model.encoder_layers(), model.decoder_layers()
    Wv, bv = model.critic
    Wa, ba = model.actor
    n_mlp = len(enc) + len(dec)
    fused = plan.P > 0
    k = 0
    tail: Optional[Tensor] = x
    for group, layers in (("enc", enc), ("dec", dec)):
        if group == "dec" and rnn_fn is not None:
            tail = rnn_fn(tail)
        for (W, b) in layers:
            last = fused and k == n_mlp - 1
            if last and plan.finish_in_gemm:
                out = outs[k][:M] if store_tail else None
                sp = model.spec
                dk = model.dist_kwargs() if sp.continuous else {}
                ops.linear_act_heads_forward_fused(tail, W, b, out, act, engine, Wv, bv, Wa, ba, plan.part, plan.counters,
                                                   **heads_kwargs, head_sizes=sp.action_segments, continuous=sp.continuous,
                                                   **dk)
                return out
            if last:
                out = outs[k][:M] if store_tail else None
                ops.linear_act_heads_forward(tail, W, b, out, act, engine, Wv, Wa, plan.part)
                tail = out
            else:
                ops.linear_act_forward(tail, W, b, outs[k][:M], act, engine)
                tail = outs[k][:M]
            k += 1
    if plan.wide:
        _heads_wide(model, tail, tail, Wv, bv, Wa, ba, plan, M, heads_kwargs)
    elif finish_fn is not None and fused:
        finish_fn(plan.part, plan.P, M, bv, ba)
    else:
        _heads(model, tail, Wv, bv, Wa, ba, fused, plan, M, heads_kwargs)
    return tail


def _forward_keys(model: PolicyModel, x: Tensor, act: int, engine: int, plan: HeadsPlan) -> Tensor:
    """MultiInputEncoder.forward (encoder.py:50-60): key k's MlpEncoder on the column slice x[:, c_k : c_k + d_k] (a
    pointer offset at the full row stride); its last layer writes columns [k*N, (k+1)*N) of the concatenation"""
    M = x.shape[0]
    sp = model.spec
    col = 0
    for k, (layers, c, (_, d)) in enumerate(zip(model.key_encoder_layers(), sp.key_offsets, sp.obs_keys)):
        t = x[:, c: c + d]
        n = sp.key_out_sizes[k]
        for i, (W, b) in enumerate(layers):
            out = plan.enc_cat[:M, col: col + n] if i == len(layers) - 1 else plan.key_h[k][i][:M]
            ops.linear_act_forward(t, W, b, out, act, engine)
            t = out
        col += n
    return plan.enc_cat[:M]


def _forward_separate(model: PolicyModel, x: Tensor, act: int, engine: int, plan: HeadsPlan, heads_kwargs: Dict,
                      tower_rnn_fns: Optional[Dict[str, Callable[[Tensor], Tensor]]] = None) -> Tensor:
    """ActorCriticSeparateWeights (model/actor_critic.py:283-318): two towers (encoder MLP -> core -> decoder MLP) on the
    same normalised observation; each tower's last stage writes its half of one [M, 2H] tail, and the heads read it
    through zero-padded weights (PolicyModel.refresh_cat_heads), so value = critic half . Wv and logits = actor half .
    Wa^T.  The last stage is the last MLP layer, or -- a recurrent core without a decoder -- the core, whose output (the
    top layer's h, a slice of the state row or of the BPTT buffers) is copied into its half with one copy_rows."""
    M = x.shape[0]
    H = model.spec.tail_input_size
    for tw, col in zip(TOWERS, (0, H)):
        t = x
        enc, dec = model.tower_encoder_layers(tw), model.tower_decoder_layers(tw)
        for k, (W, b) in enumerate(enc + dec):
            if tower_rnn_fns is not None and k == len(enc):
                t = tower_rnn_fns[tw](t)
            out = plan.tail_cat[:M, col: col + H] if plan.tower_h[tw][k] is None else plan.tower_h[tw][k][:M]
            ops.linear_act_forward(t, W, b, out, act, engine)
            t = out
        if not plan.tower_tail_is_mlp:      # a core without a decoder feeds the heads
            ops.copy_rows(tower_rnn_fns[tw](t), plan.tail_cat[:M, col: col + H])
    Wv, bv = model.critic
    Wa, ba = model.actor
    tail = plan.tail_cat[:M]
    if plan.wide:     # logits from the actor half, the value from the critic half, with the heads' own weights
        _heads_wide(model, tail[:, :H], tail[:, H:], Wv, bv, Wa, ba, plan, M, heads_kwargs)
    else:
        _heads(model, tail, model.Wv_cat, bv, model.Wa_cat, ba, False, plan, M, heads_kwargs)
    return tail


def _heads(model: PolicyModel, tail: Tensor, Wv: Tensor, bv: Tensor, Wa: Tensor, ba: Tensor, fused: bool, plan: HeadsPlan,
           M: int, heads_kwargs: Dict) -> None:
    P = plan.P
    sp = model.spec
    if sp.action_heads and heads_kwargs.get("actions_f32") is not None:
        # Tuple with Box members: the params rows are stored (the plan's scratch if the caller keeps none), then the tail
        kw = _mixed_kwargs(plan, heads_kwargs)
        if fused:
            ops.heads_from_partials_mixed(plan.part, P, M, bv, ba, sp.head_kinds, sp.head_sizes, **kw)
        else:
            ops.heads_forward_mixed(tail, Wv, bv, Wa, ba, sp.head_kinds, sp.head_sizes, **kw)
        return
    if model.spec.continuous:   # Box action space: Gaussian heads (action_distributions.py:290-323)
        dk = model.dist_kwargs()
        if fused:
            ops.heads_from_partials_continuous(plan.part, P, M, bv, ba, **dk, **heads_kwargs)
        else:
            ops.heads_forward_continuous(tail, Wv, bv, Wa, ba, **dk, **heads_kwargs)
    elif model.spec.action_segments:   # Tuple of Discretes: independent categorical heads (action_distributions.py:197-286)
        if fused:
            ops.heads_from_partials_tuple(plan.part, P, M, bv, ba, model.spec.action_segments, **heads_kwargs)
        else:
            ops.heads_forward_tuple(tail, Wv, bv, Wa, ba, model.spec.action_segments, **heads_kwargs)
    elif fused:
        ops.heads_from_partials(plan.part, P, M, bv, ba, **heads_kwargs)
    else:
        ops.heads_forward(tail, Wv, bv, Wa, ba, **heads_kwargs)


def _heads_wide(model: PolicyModel, tail_a: Tensor, tail_v: Tensor, Wv: Tensor, bv: Tensor, Wa: Tensor, ba: Tensor,
                plan: HeadsPlan, M: int, heads_kwargs: Dict) -> None:
    """Wide heads: distribution_linear as a GEMM on the regular engine into the logits' final place (the trajectory slot,
    the learner's minibatch logits, or the plan's scratch; for a learned stddev the means half of each params row), then
    sfb200_heads_tail_wide.  A values-only call (the bootstrap value) skips the GEMM."""
    sp = model.spec
    kw = dict(heads_kwargs)
    logits, stride = kw.pop("logits", None), kw.pop("logits_stride", 0)
    if logits is None and kw.get("actions_f32") is not None:
        logits, stride = plan.wide_logits, plan.wide_logits.stride(0)
    A = sp.num_linear_action_outputs
    if logits is not None:
        dst = logits.as_strided((M, A), (stride, 1))
        ops.linear_act_forward(tail_a, Wa, ba, dst, ops.ACT["none"], plan.engine)
    if sp.action_heads and kw.get("actions_f32") is not None:
        ops.heads_tail_wide_mixed(tail_v, Wv, bv, logits, stride, A, sp.head_kinds, sp.head_sizes, **kw)
        return
    dk = model.dist_kwargs() if sp.continuous else {}
    ops.heads_tail_wide(tail_v, Wv, bv, logits, stride, A, head_sizes=sp.action_segments, continuous=sp.continuous,
                        **dk, **kw)


def _mixed_kwargs(plan: HeadsPlan, heads_kwargs: Dict) -> Dict:
    """heads_kwargs with a params destination: the caller's logits rows, else the plan's scratch"""
    kw = dict(heads_kwargs)
    if kw.get("logits") is None:
        kw["logits"], kw["logits_stride"] = plan.wide_logits, plan.wide_logits.stride(0)
    return kw
