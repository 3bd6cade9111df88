"""Device-resident actor-critic parameters for the hot path.

Mirrors the reference's ActorCriticSharedWeights with MlpEncoder -> ModelCoreIdentity -> MlpDecoder -> critic_linear /
distribution_linear (model/actor_critic.py:136-195, encoder.py:72-91, core.py:67-77, decoder.py:15-35) as DATA: one
flat fp32 parameter buffer in HBM (plus flat grad / Adam-moment buffers of the same shape) so that grad-norm, Adam and
the NCCL all-reduce are single launches over contiguous memory.  Tensor names and order are the reference's
state_dict keys, so checkpoints round-trip (learner.py:323-332).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import torch
from torch import Tensor

OBS_NORM_PREFIX_BASE = "obs_normalizer.running_mean_std.running_mean_std."
OBS_NORM_PREFIX = OBS_NORM_PREFIX_BASE + "obs."
RET_NORM_PREFIX = "returns_normalizer."


@dataclass
class ModelSpec:
    obs_dim: int
    num_actions: int  # Discrete(n)
    encoder_mlp_layers: List[int] = field(default_factory=lambda: [512, 512])
    decoder_mlp_layers: List[int] = field(default_factory=list)
    nonlinearity: str = "elu"
    normalize_input: bool = True
    normalize_returns: bool = True
    obs_subtract_mean: float = 0.0
    obs_scale: float = 1.0
    use_rnn: bool = False        # model/core.py: ModelCoreRNN between encoder and decoder (rnn_num_layers layers)
    rnn_type: str = "gru"
    rnn_size: int = 512
    # Box action space (action_distributions.py:290-323): num_actions is then the action DIMENSION
    continuous: bool = False
    adaptive_stddev: bool = True        # cfg.py:577; False -> one learned log-stddev vector (action_parameterization.py:42)
    continuous_tanh_scale: float = 0.0  # cfg.py:583
    initial_stddev: float = 1.0         # cfg.py:591
    # Tuple(Discrete(n_0), ..., Discrete(n_{K-1})) action space (action_distributions.py:197-286): the heads' sizes;
    # num_actions is then sum(n_k) (the number of logits)
    action_segments: Optional[List[int]] = None
    # Tuple action space with at least one Box member: [("discrete", n) | ("box", d), ...] in member order.  The Tuple
    # always uses ActionParameterizationDefault (actor_critic.py:43-53): distribution_linear has sum(n or 2d) rows, a Box
    # member's rows are [means | log_std], and adaptive_stddev / continuous_tanh_scale / initial_stddev are not read.
    # num_actions is then the number of rows.  An all-Discrete list is stored as action_segments instead.
    action_heads: Optional[List[Tuple[str, int]]] = None
    # image observations: obs_shape = (C, H, W) selects the ConvEncoder (model/encoder.py:88-145); obs_dim = C*H*W and the
    # fully connected layers after the conv head (encoder_conv_mlp_layers) take the place of encoder_mlp_layers
    obs_shape: Optional[Tuple[int, int, int]] = None
    encoder_conv_architecture: str = "convnet_atari"
    encoder_conv_mlp_layers: List[int] = field(default_factory=lambda: [512])
    obs_uint8: bool = False              # dtype of the observation rows in the trajectory buffers
    # False -> ActorCriticSeparateWeights (model/actor_critic.py:198-322): an actor tower (encoder MLP -> recurrent core
    # if use_rnn -> decoder MLP) feeding distribution_linear and a critic tower feeding critic_linear.  Each tower's core
    # owns one half of a state row, [actor state | critic state], each half laid out like a shared model's row.  Vector
    # observations of one key only (conv / ResNet encoders and Dict observations raise ValueError).  Towers with no layer
    # and no core run as the shared identity model (separate_towers)
    share_weights: bool = True
    # Dict observations of 1-D keys (MultiInputEncoder, model/encoder.py:33-70): [(key, d), ...] in sorted key order.  The
    # keys lie side by side in one packed row, key k in columns [c_k, c_k + d_k); every key has its own MlpEncoder with
    # encoder_mlp_layers ([] = identity) and the encoders' outputs are concatenated.  One key takes the single-key path,
    # with the parameter and normaliser names of that key.  Keyword-only: positional construction keeps its meaning.
    obs_keys: Optional[List[Tuple[str, int]]] = field(default=None, kw_only=True)
    # stacked recurrent core: nn.GRU / nn.LSTM(in, rnn_size, rnn_num_layers) (model/core.py:27-31); layer k > 0 reads
    # layer k-1's new h, the state rows are layer-major [h_0 | h_1 | ...] (GRU) / [h_0 | c_0 | h_1 | c_1 | ...] (LSTM)
    rnn_num_layers: int = 1

    CONV_ARCH = {  # model/encoder.py:127-134: (out_channels, kernel, stride); no padding
        "convnet_simple": [(32, 8, 4), (64, 4, 2), (128, 3, 2)],
        "convnet_impala": [(16, 8, 4), (32, 4, 2)],
        "convnet_atari": [(32, 8, 4), (64, 4, 2), (64, 3, 1)],
    }

    @property
    def conv_layers(self) -> List[Tuple[int, int, int, int, int, int, int, int]]:
        """[(C_in, H_in, W_in, C_out, kernel, stride, H_out, W_out)] of the conv head ([] for vector observations)"""
        if self.obs_shape is None:
            return []
        c, h, w = self.obs_shape
        out = []
        if self.is_resnet:
            return out      # described by resnet_stages
        for (co, k, s) in self.CONV_ARCH[self.encoder_conv_architecture]:
            ho, wo = (h - k) // s + 1, (w - k) // s + 1
            out.append((c, h, w, co, k, s, ho, wo))
            c, h, w = co, ho, wo
        return out

    RESNET_STAGES = [(16, 2), (32, 2), (32, 2)]   # model/encoder.py:182 (resnet_impala): (channels, res blocks)

    @property
    def is_resnet(self) -> bool:
        return self.obs_shape is not None and self.encoder_conv_architecture == "resnet_impala"

    @property
    def resnet_stages(self) -> List[Tuple[int, int, int, int, int, int, int]]:
        """[(C_in, H, W, C_out, H_pool, W_pool, blocks)] of the ResnetEncoder (encoder.py:173-221): per stage a 3x3 conv
        with padding 1 (H x W kept), a 3x3 / stride 2 / padding 1 max-pool (-> ceil(H/2) x ceil(W/2)) and `blocks`
        residual blocks of two 3x3 convs at C_out channels"""
        c, h, w = self.obs_shape
        out = []
        for (co, blocks) in self.RESNET_STAGES:
            hp, wp = (h + 1) // 2, (w + 1) // 2
            out.append((c, h, w, co, hp, wp, blocks))
            c, h, w = co, hp, wp
        return out

    @property
    def conv_out_size(self) -> int:
        if self.is_resnet:
            _c, _h, _w, co, hp, wp, _b = self.resnet_stages[-1]
            return co * hp * wp
        c, _, _, co, _, _, ho, wo = self.conv_layers[-1]
        return co * ho * wo

    def conv_param_layout(self) -> List[Tuple[str, Tuple[int, int, int, int]]]:
        """[(reference state_dict prefix, weight shape)] of the conv head's Conv2d layers in parameters() order.
        ResnetEncoder: conv_head.{j} is a stage's entry conv, conv_head.{j}.res_block_core.{1,3} the two convs of a block
        (Sequential indices of encoder.py:157-162 / 188-202)."""
        if not self.is_resnet:
            return [(f"encoder.encoders.obs.enc.conv_head.{2 * i}", (co, ci, k, k))
                    for i, (ci, _h, _w, co, k, _s, _ho, _wo) in enumerate(self.conv_layers)]
        out, j = [], 0
        for (ci, _h, _w, co, _hp, _wp, blocks) in self.resnet_stages:
            out.append((f"encoder.encoders.obs.conv_head.{j}", (co, ci, 3, 3)))
            j += 2
            for _ in range(blocks):
                out += [(f"encoder.encoders.obs.conv_head.{j}.res_block_core.{r}", (co, co, 3, 3)) for r in (1, 3)]
                j += 1
        return out

    @property
    def dict_obs(self) -> bool:
        """several observation keys: per-key encoders whose outputs are concatenated (the key encoder stage)"""
        return self.obs_keys is not None and len(self.obs_keys) > 1

    @property
    def obs_key(self) -> str:
        """the observation key of a single-key model"""
        return self.obs_keys[0][0] if self.obs_keys else "obs"

    @property
    def key_offsets(self) -> List[int]:
        """first column of each key in the packed observation row"""
        out, c = [], 0
        for _, d in self.obs_keys:
            out.append(c)
            c += d
        return out

    @property
    def key_out_sizes(self) -> List[int]:
        """width of each key encoder's output: encoder_mlp_layers[-1], or d_k for the identity encoder"""
        return [self.encoder_mlp_layers[-1] if self.encoder_mlp_layers else d for _, d in self.obs_keys]

    def key_encoder_name(self, key: str, i: int, what: str) -> str:
        return f"encoder.encoders.{key}.mlp_head.{2 * i}.{what}"

    @property
    def fc_encoder_layers(self) -> List[int]:
        """widths of the fully connected encoder layers (after the conv head for image observations; none after the
        key encoders of a Dict model)"""
        if self.dict_obs:
            return []
        return list(self.encoder_conv_mlp_layers) if self.obs_shape is not None else list(self.encoder_mlp_layers)

    @property
    def fc_encoder_input(self) -> int:
        if self.dict_obs:       # the concatenated key encoder outputs
            return sum(self.key_out_sizes)
        return self.conv_out_size if self.obs_shape is not None else self.obs_dim

    def fc_encoder_name(self, i: int, what: str) -> str:
        if self.is_resnet:      # ResnetEncoder keeps its mlp_layers directly (no `.enc.` wrapper, encoder.py:208)
            return f"encoder.encoders.obs.mlp_layers.{2 * i}.{what}"
        if self.obs_shape is not None:
            return f"encoder.encoders.obs.enc.mlp_layers.{2 * i}.{what}"
        return self.key_encoder_name(self.obs_key, i, what)

    @property
    def obs_norm_prefixes(self) -> List[Tuple[str, int, int]]:
        """[(state_dict prefix, first column, width)] of the per-key RunningMeanStdInPlace (running_mean_std.py:113-136)"""
        if self.obs_keys is None:
            return [(OBS_NORM_PREFIX, 0, self.obs_dim)]
        return [(f"{OBS_NORM_PREFIX_BASE}{k}.", c, d) for (k, d), c in zip(self.obs_keys, self.key_offsets)]

    @classmethod
    def from_cfg(cls, cfg, env) -> "ModelSpec":
        """The model the reference would build for this cfg / env (model/actor_critic.py:136-158, create_actor_critic):
        Discrete(n) envs expose `num_actions = n`; Box(A) envs expose `continuous = True` and `num_actions = A`."""
        obs_shape = getattr(env, "obs_shape", None)   # (C, H, W) image observations -> ConvEncoder (encoder.py:218-227)
        obs_keys = getattr(env, "obs_keys", None)
        keys_to_normalize = getattr(cfg, "normalize_input_keys", None)
        if obs_keys and len(obs_keys) > 1 and keys_to_normalize is not None and (
                set(keys_to_normalize) != {k for k, _ in obs_keys}):
            raise ValueError(f"normalize_input_keys={list(keys_to_normalize)} selects a subset of the Dict observation keys "
                             f"{[k for k, _ in obs_keys]}: the device path normalises every key of a multi-key Dict")
        return cls(env.obs_dim, env.num_actions, list(cfg.encoder_mlp_layers), list(cfg.decoder_mlp_layers),
                   cfg.nonlinearity, cfg.normalize_input, cfg.normalize_returns, cfg.obs_subtract_mean, cfg.obs_scale,
                   bool(cfg.use_rnn), cfg.rnn_type, cfg.rnn_size,
                   obs_shape=None if obs_shape is None else tuple(obs_shape),
                   encoder_conv_architecture=getattr(cfg, "encoder_conv_architecture", "convnet_atari"),
                   encoder_conv_mlp_layers=list(getattr(cfg, "encoder_conv_mlp_layers", [512])),
                   obs_uint8=bool(getattr(env, "obs_uint8", False)),
                   share_weights=bool(getattr(cfg, "actor_critic_share_weights", True)),
                   action_segments=(list(env.action_segments) if getattr(env, "action_segments", None) else None),
                   action_heads=([tuple(h) for h in env.action_heads] if getattr(env, "action_heads", None) else None),
                   continuous=bool(getattr(env, "continuous", False)),
                   adaptive_stddev=bool(getattr(cfg, "adaptive_stddev", True)),
                   continuous_tanh_scale=float(getattr(cfg, "continuous_tanh_scale", 0.0)),
                   initial_stddev=float(getattr(cfg, "initial_stddev", 1.0)),
                   rnn_num_layers=int(getattr(cfg, "rnn_num_layers", 1)),
                   obs_keys=([tuple(k) for k in obs_keys] if obs_keys else None))

    @property
    def num_linear_action_outputs(self) -> int:
        """rows of distribution_linear"""
        if not self.continuous:
            return self.num_actions
        return 2 * self.num_actions if self.adaptive_stddev else self.num_actions

    NARROW_HEADS_MAX = 31      # rows the warp-per-row heads kernels hold (lane 0 = value, lanes 1..A = logits)
    NARROW_HEADS_SMEM = 200 * 1024     # bytes of [critic_linear | distribution_linear] the narrow heads forward stages
    MAX_LINEAR_ACTION_OUTPUTS = 1024
    MAX_TUPLE_HEADS = 8

    @property
    def wide_heads(self) -> bool:
        """distribution_linear has more than 31 rows, or its rows and critic_linear's do not fit the narrow heads forward's
        shared memory (heads reading conv features thousands wide): the heads run as a GEMM on the regular engine plus
        sfb200_heads_tail_wide instead of the fused warp-per-row heads kernels"""
        A = self.num_linear_action_outputs
        width = self.tail_input_size * (2 if self.separate_towers else 1)     # what the narrow kernels read per row
        return A > self.NARROW_HEADS_MAX or (A + 1) * width * 4 > self.NARROW_HEADS_SMEM

    @property
    def separate_towers(self) -> bool:
        """separate actor / critic weights whose towers hold an MLP layer or a core.  Towers that are identities own no
        parameters (ActorCriticSeparateWeights then has only the heads, actor_critic.py:198-322): such a model runs as
        the shared-weights identity model and differs from it only in the width of its state rows"""
        return not self.share_weights and (bool(self.hidden) or self.use_rnn)

    @property
    def heads_read_input(self) -> bool:
        """a linear policy: no MLP layer and no core, the heads read the normalised observation rows (the concatenated
        key rows of a Dict model with identity key encoders)"""
        return not self.hidden and not self.use_rnn and self.obs_shape is None and not (
            self.dict_obs and self.encoder_mlp_layers)

    def __post_init__(self) -> None:
        if self.use_rnn and self.rnn_num_layers < 1:
            raise ValueError(f"rnn_num_layers must be >= 1, got {self.rnn_num_layers}")
        if self.action_heads:
            heads = [(str(k), int(n)) for k, n in self.action_heads]
            if any(k not in ("discrete", "box") or n < 1 for k, n in heads):
                raise ValueError(f"action_heads members are ('discrete', n) or ('box', d) with n, d >= 1, got {heads}")
            if self.continuous or self.action_segments:
                raise ValueError("action_heads describes the whole action space: continuous / action_segments must be unset")
            if all(k == "discrete" for k, _ in heads):        # a Tuple of Discretes keeps its own path
                self.action_segments, self.action_heads = [n for _, n in heads], None
            else:
                self.action_heads = heads
                rows = sum(n if k == "discrete" else 2 * n for k, n in heads)
                if self.num_actions != rows:
                    raise ValueError(f"a Tuple with members {heads} has {rows} distribution_linear rows, num_actions is "
                                     f"{self.num_actions}")
        if self.obs_keys is not None:
            self._check_obs_keys()
        if not self.share_weights and self.obs_shape is not None:
            raise ValueError(f"separate actor / critic weights (actor_critic_share_weights=False) with an image encoder "
                             f"({self.encoder_conv_architecture}) are not supported on the device path")
        tup = self.action_segments or self.action_heads
        if tup and len(tup) > self.MAX_TUPLE_HEADS:
            raise ValueError(f"Tuple action spaces are supported with at most {self.MAX_TUPLE_HEADS} heads, got "
                             f"{len(tup)}")
        n = self.num_linear_action_outputs
        if n > self.MAX_LINEAR_ACTION_OUTPUTS:
            what = (f"Box({self.num_actions}) with adaptive_stddev={self.adaptive_stddev}" if self.continuous else
                    f"{'Tuple' if tup else 'Discrete'} with {self.num_actions} logits")
            raise ValueError(f"{what} needs {n} distribution_linear rows; the device path supports at most "
                             f"{self.MAX_LINEAR_ACTION_OUTPUTS}")

    def _check_obs_keys(self) -> None:
        keys = [(str(k), int(d)) for k, d in self.obs_keys]
        names = [k for k, _ in keys]
        if not keys or names != sorted(set(names)):
            raise ValueError(f"obs_keys must be unique keys in sorted order (MultiInputEncoder's order), got {names}")
        if any(d < 1 for _, d in keys):
            raise ValueError(f"obs_keys widths must be >= 1, got {keys}")
        if sum(d for _, d in keys) != self.obs_dim:
            raise ValueError(f"obs_keys {keys} span {sum(d for _, d in keys)} columns, obs_dim is {self.obs_dim}")
        self.obs_keys = keys
        if len(keys) == 1:
            return
        if self.obs_shape is not None:
            raise ValueError("Dict observations with several keys: 1-D keys only (image keys are not supported)")
        if not self.share_weights:
            raise ValueError("Dict observations with several keys are not supported with actor_critic_share_weights=False")
        if abs(self.obs_subtract_mean) > 1e-8 or abs(self.obs_scale - 1.0) > 1e-8:
            raise ValueError("Dict observations with several keys: obs_subtract_mean / obs_scale apply to the key 'obs' only "
                             "(normalize.py:59-65) and are not supported; leave them at 0 / 1")

    @property
    def num_action_params(self) -> int:
        """calc_num_action_parameters (action_distributions.py:33-44): width of `action_logits`"""
        return 2 * self.num_actions if self.continuous else self.num_actions

    @property
    def action_width(self) -> int:
        """calc_num_actions (:16-30): width of `actions`"""
        if self.action_segments:
            return len(self.action_segments)
        if self.action_heads:
            return sum(1 if k == "discrete" else n for k, n in self.action_heads)
        return self.num_actions if self.continuous else 1

    @property
    def head_kinds(self) -> List[int]:
        """action_heads as the kernels' head_kinds (0 = categorical, 1 = Gaussian with state-dependent log-std)"""
        return [0 if k == "discrete" else 1 for k, _ in self.action_heads]

    @property
    def head_sizes(self) -> List[int]:
        return [n for _, n in self.action_heads]

    @property
    def hidden(self) -> List[int]:
        # ModelCoreIdentity (use_rnn=False) passes the encoder output straight to the decoder MLP
        return self.fc_encoder_layers + list(self.decoder_mlp_layers)

    @property
    def rnn_state_size(self) -> int:
        """model/model_utils.py:11-24"""
        if not self.use_rnn:
            return 1 if self.share_weights else 2       # "actor and critic need separate states" (model_utils.py:20-22)
        return self.rnn_tower_state_size * (1 if self.share_weights else 2)

    @property
    def rnn_tower_state_size(self) -> int:
        """width of one core's columns of a state row (separate weights: [actor state | critic state], each this wide)"""
        return self.rnn_layer_state_size * self.rnn_num_layers

    @property
    def rnn_layer_state_size(self) -> int:
        """width of one layer's slice of a state row: h (GRU) or [h | c] (LSTM)"""
        return self.rnn_size * (2 if self.rnn_type == "lstm" else 1)

    @property
    def rnn_gates(self) -> int:
        return 4 if self.rnn_type == "lstm" else 3

    @property
    def tail_input_size(self) -> int:
        """width of the tensor that feeds critic_linear / distribution_linear"""
        if self.decoder_mlp_layers:
            return self.decoder_mlp_layers[-1]     # (separate weights: the width of ONE tower's tail)
        if self.use_rnn:
            return self.rnn_size
        return self.fc_encoder_layers[-1] if self.fc_encoder_layers else self.fc_encoder_input

    def param_shapes(self) -> List[Tuple[str, Tuple[int, ...]]]:
        """(reference state_dict key, shape) in nn.Module.parameters() order."""
        out = []
        if not self.share_weights:
            # registration order of ActorCriticSeparateWeights.__init__ (actor_critic.py:208-225): per tower its encoder
            # then its core, then both decoders
            for tw in TOWERS:
                d = self.obs_dim
                for i, h in enumerate(self.encoder_mlp_layers):
                    out.append((f"{tw}encoder.encoders.obs.mlp_head.{2 * i}.weight", (h, d)))
                    out.append((f"{tw}encoder.encoders.obs.mlp_head.{2 * i}.bias", (h,)))
                    d = h
                if self.use_rnn:
                    out += self._rnn_shapes(f"{tw}core.", d)
                    d = self.rnn_size
            d_enc = d
            for tw in TOWERS:
                d = d_enc
                for i, h in enumerate(self.decoder_mlp_layers):
                    out.append((f"{tw}decoder.mlp.{2 * i}.weight", (h, d)))
                    out.append((f"{tw}decoder.mlp.{2 * i}.bias", (h,)))
                    d = h
            out.append(("critic_linear.weight", (1, d)))
            out.append(("critic_linear.bias", (1,)))
            if self.continuous and not self.adaptive_stddev:
                out.append(("action_parameterization.learned_stddev", (self.num_actions,)))
            out.append(("action_parameterization.distribution_linear.weight", (self.num_linear_action_outputs, d)))
            out.append(("action_parameterization.distribution_linear.bias", (self.num_linear_action_outputs,)))
            return out
        if self.dict_obs:       # MultiInputEncoder: encoders.{key}, keys in sorted order (encoder.py:36-48)
            for key, d in self.obs_keys:
                for i, h in enumerate(self.encoder_mlp_layers):
                    out.append((self.key_encoder_name(key, i, "weight"), (h, d)))
                    out.append((self.key_encoder_name(key, i, "bias"), (h,)))
                    d = h
        for prefix, wshape in self.conv_param_layout():
            out.append((f"{prefix}.weight", wshape))
            out.append((f"{prefix}.bias", (wshape[0],)))
        d = self.fc_encoder_input
        for i, h in enumerate(self.fc_encoder_layers):
            out.append((self.fc_encoder_name(i, "weight"), (h, d)))
            out.append((self.fc_encoder_name(i, "bias"), (h,)))
            d = h
        if self.use_rnn:
            out += self._rnn_shapes("core.", d)
            d = self.rnn_size
        for i, h in enumerate(self.decoder_mlp_layers):
            out.append((f"decoder.mlp.{2 * i}.weight", (h, d)))
            out.append((f"decoder.mlp.{2 * i}.bias", (h,)))
            d = h
        out.append(("critic_linear.weight", (1, d)))
        out.append(("critic_linear.bias", (1,)))
        if self.continuous and not self.adaptive_stddev:
            # a module's own parameters precede its children's in nn.Module.parameters()
            out.append(("action_parameterization.learned_stddev", (self.num_actions,)))
        out.append(("action_parameterization.distribution_linear.weight", (self.num_linear_action_outputs, d)))
        out.append(("action_parameterization.distribution_linear.bias", (self.num_linear_action_outputs,)))
        return out

    def _rnn_shapes(self, prefix: str, d: int) -> List[Tuple[str, Tuple[int, ...]]]:
        """one core's parameters (prefix "core." / "actor_core." / "critic_core.", input width d), in nn.GRU / nn.LSTM
        registration order: per layer ih, hh, biases"""
        G, H = self.rnn_gates, self.rnn_size
        out = []
        for k in range(self.rnn_num_layers):
            out += [(f"{prefix}core.weight_ih_l{k}", (G * H, d)), (f"{prefix}core.weight_hh_l{k}", (G * H, H)),
                    (f"{prefix}core.bias_ih_l{k}", (G * H,)), (f"{prefix}core.bias_hh_l{k}", (G * H,))]
            d = H
        return out


TOWERS = ("actor_", "critic_")      # separate actor / critic weights: the towers' state_dict prefixes, in state-row order


def _align(n: int, a: int = 64) -> int:
    return (n + a - 1) // a * a


class PolicyModel:
    """Flat parameter storage + normalizer buffers on one device."""

    def __init__(self, spec: ModelSpec, device: torch.device, seed: int = 0, policy_init_gain: float = 1.0,
                 policy_initialization: str = "orthogonal"):
        assert policy_initialization in ("orthogonal", "xavier_uniform", "torch_default"), policy_initialization
        spec.__post_init__()      # (the limits of the heads, also for a spec changed after its construction)
        self.policy_initialization = policy_initialization
        self.spec = spec
        self.device = device
        shapes = spec.param_shapes()
        # every tensor starts on a 256-byte boundary inside the flat buffer (vector loads / TMA alignment)
        offsets, off = [], 0
        for _, shp in shapes:
            offsets.append(off)
            off += _align(math.prod(shp))
        self.numel_padded = off
        self.num_params = sum(math.prod(s) for _, s in shapes)
        self.flat = torch.zeros(off, dtype=torch.float32, device=device)
        self.grad = torch.zeros_like(self.flat)
        self.exp_avg = torch.zeros_like(self.flat)
        self.exp_avg_sq = torch.zeros_like(self.flat)
        self.params: Dict[str, Tensor] = {}
        self.grads: Dict[str, Tensor] = {}
        self._slices: Dict[str, Tuple[int, Tuple[int, ...]]] = {}
        for (name, shp), o in zip(shapes, offsets):
            n = math.prod(shp)
            self.params[name] = self.flat[o : o + n].view(shp)
            self.grads[name] = self.grad[o : o + n].view(shp)
            self._slices[name] = (o, shp)
        self.names = [n for n, _ in shapes]

        # running_mean_std.py:45-47
        self.obs_mean = torch.zeros(spec.obs_dim, dtype=torch.float64, device=device)
        self.obs_var = torch.ones(spec.obs_dim, dtype=torch.float64, device=device)
        self.obs_count = torch.ones(1, dtype=torch.float64, device=device)
        self.ret_mean = torch.zeros(1, dtype=torch.float64, device=device)
        self.ret_var = torch.ones(1, dtype=torch.float64, device=device)
        self.ret_count = torch.ones(1, dtype=torch.float64, device=device)

        self._init_weights(seed, policy_init_gain)
        self._register_f16()
        self.refresh_cat_heads()

    # ---- fp16-split form of the 3-pass GEMM engine (include/sfb200.h): fp16 twins of the weights + activation bounds ----
    def _register_f16(self) -> None:
        """Plain MLP policies with normalised inputs: every hidden activation has a bound that follows from the weights
        (normalised observations are clipped to +-5, running_mean_std.py:96-110; |act(x W^T + b)| <= |x|_inf * max_n
        |W[n,:]|_1 + |b|_inf), so the forward GEMMs -- and dX, through transposed twins -- can take the fp16 operand path."""
        sp = self.spec
        self.f16_twins = None
        self.f16_T: Dict[str, Tensor] = {}
        self.bound_x = self.bound_h = self.grad_fac = None
        ok = (self.flat.is_cuda and sp.normalize_input and sp.obs_shape is None and not sp.use_rnn and sp.share_weights
              and not sp.decoder_mlp_layers and not sp.dict_obs and len(sp.hidden) >= 1)
        if not ok:
            return
        from . import ops

        self.f16_twins = torch.empty(2 * self.flat.numel(), dtype=torch.float16, device=self.device)
        ops.register_f16_twins(self.flat, self.f16_twins)
        self.bound_x = torch.full((1,), 5.0, dtype=torch.float32, device=self.device)
        self.bound_h = torch.zeros(4 * len(sp.hidden), dtype=torch.float32, device=self.device)   # [bound, scratch, counter, -] per layer
        # per hidden layer i >= 1: max_k sum_n |W_i[n][k]|, the factor from the bound of dz[i] to that of dz[i-1] (same layout)
        self.grad_fac = torch.zeros(4 * len(sp.hidden), dtype=torch.float32, device=self.device)
        self.refresh_bounds()

    def refresh_bounds(self) -> None:
        """bounds of the hidden activations and gradient factors from the current weights (one tiny kernel per layer) + the
        transposed twins"""
        if self.f16_twins is None:
            return
        from . import ops

        act = ops.ACT[self.spec.nonlinearity]
        inb = self.bound_x
        layers = self.hidden_layers()
        for i, (W, b) in enumerate(layers[:-1]):       # (the last hidden layer feeds the heads, not a GEMM)
            ops.linear_out_bound(W, b, inb, self.bound_h[4 * i: 4 * i + 4], act)
            inb = self.bound_h[4 * i: 4 * i + 1]
        for i in range(1, len(layers)):                # layers whose input gradient the learner takes
            ops.linear_in_grad_bound(layers[i][0], self.grad_fac[4 * i: 4 * i + 4])
        for name in self.f16_T:
            ops.refresh_f16_transposed(self.params[name])

    def enable_f16_transposed(self, name: str) -> None:
        """transposed fp16 twins of one weight matrix (the learner's dX = dz . W reads W along its other axis)"""
        if self.f16_twins is None or name in self.f16_T:
            return
        from . import ops

        W = self.params[name]
        self.f16_T[name] = torch.empty(2 * W.numel(), dtype=torch.float16, device=self.device)
        ops.register_f16_transposed(W, self.f16_T[name])

    def weights_changed(self) -> None:
        """Call after writing `flat` / `params[...]` by anything other than the Adam kernel (which keeps the fp16 twins
        current)."""
        if self.f16_twins is not None:
            from . import ops

            ops.refresh_f16_twins(self.flat)
            self.refresh_bounds()
        self.refresh_cat_heads()

    def rebind_grad(self, grad: Tensor) -> None:
        """Move the flat gradient buffer (data parallel: into the NVLink comm buffer the peers read, dist_utils.PeerComm)"""
        assert grad.shape == self.flat.shape and grad.dtype == torch.float32 and grad.is_contiguous()
        grad.zero_()
        self.grad = grad
        self.grads = {n: grad[o: o + math.prod(shp)].view(shp) for n, (o, shp) in self._slices.items()}

    def __del__(self):
        try:
            # the twin registries are keyed by device address: a stale entry would pick the fp16 form for whatever
            # buffer the allocator places there next
            if getattr(self, "f16_twins", None) is not None:
                from . import ops

                for name in self.f16_T:
                    ops.unregister_f16_transposed(self.params[name])
                ops.unregister_f16_twins(self.flat)
        except Exception:
            pass

    def _init_weights(self, seed: int, gain: float) -> None:
        """ActorCritic.initialize_weights (actor_critic.py:73-96): biases 0 in every mode; Linear / Conv2d weights orthogonal
        (gain), xavier_uniform (gain), or left at the PyTorch default U(-1/sqrt(fan_in), 1/sqrt(fan_in)) (torch_default)."""
        mode = self.policy_initialization
        g = torch.Generator(device="cpu").manual_seed(seed)
        for name in self.names:
            p = self.params[name]
            if name == "action_parameterization.learned_stddev":
                p.fill_(math.log(self.spec.initial_stddev))   # action_parameterization.py:59-61
            elif ".core.weight_" in name or ".core.bias_" in name:
                # RNNs keep the PyTorch default init U(-1/sqrt(H), 1/sqrt(H)) (actor_critic.py:83-88)
                k = 1.0 / math.sqrt(self.spec.rnn_size)
                p.copy_((torch.rand(p.shape, generator=g) * 2 - 1) * k)
            elif name.endswith(".bias"):
                p.zero_()
            else:
                w = torch.empty(p.shape, dtype=torch.float32)
                if mode == "orthogonal":
                    torch.nn.init.orthogonal_(w, gain=gain, generator=g)
                elif mode == "xavier_uniform":
                    torch.nn.init.xavier_uniform_(w, gain=gain, generator=g)
                else:   # nn.Linear / nn.Conv2d reset_parameters: kaiming_uniform_(a=sqrt(5)) == U(-1/sqrt(fan_in), 1/sqrt(fan_in))
                    bound = 1.0 / math.sqrt(math.prod(p.shape[1:]))
                    w.uniform_(-bound, bound, generator=g)
                p.copy_(w)

    # ---- inference-side weight snapshot (async_rl: the reference's inference workers hold their own copy of the
    # weights and refresh it when the learner publishes a new version, model_sharing.py:17-94, inference_worker.py:207-233)
    def inference_copy(self) -> "PolicyModel":
        twin = object.__new__(PolicyModel)
        twin.spec, twin.device = self.spec, self.device
        twin.numel_padded, twin.num_params, twin.names, twin._slices = self.numel_padded, self.num_params, self.names, self._slices
        twin.flat = self.flat.clone()
        twin.grad = twin.exp_avg = twin.exp_avg_sq = None
        twin.params = {n: twin.flat[o : o + math.prod(shp)].view(shp) for n, (o, shp) in self._slices.items()}
        twin.grads = {}
        for k in ("obs_mean", "obs_var", "obs_count", "ret_mean", "ret_var", "ret_count"):
            setattr(twin, k, getattr(self, k).clone())
        twin._register_f16()
        twin.refresh_cat_heads()
        return twin

    def copy_weights_from(self, other: "PolicyModel") -> None:
        """Refresh this snapshot from the learner's model (D2D copies on the current stream)."""
        self.flat.copy_(other.flat)
        if self.f16_twins is not None and other.f16_twins is not None:
            self.f16_twins.copy_(other.f16_twins)
            self.bound_h.copy_(other.bound_h)      # (scratch words are zero between launches)
            self.grad_fac.copy_(other.grad_fac)
            self.refresh_cat_heads()
        else:
            self.weights_changed()
        self.obs_mean.copy_(other.obs_mean)
        self.obs_var.copy_(other.obs_var)

    # ---- layer access ---------------------------------------------------------------------------------------
    def hidden_layers(self) -> List[Tuple[Tensor, Tensor]]:
        """[(W [out,in], b [out]), ...] for encoder then decoder MLP layers."""
        return self.encoder_layers() + self.decoder_layers()

    def encoder_layers(self, grads: bool = False) -> List[Tuple[Tensor, Tensor]]:
        """the fully connected encoder layers (MlpEncoder, or the layers after the conv head of a ConvEncoder)"""
        src = self.grads if grads else self.params
        sp = self.spec
        return [(src[sp.fc_encoder_name(i, "weight")], src[sp.fc_encoder_name(i, "bias")])
                for i in range(len(sp.fc_encoder_layers))]

    def key_encoder_layers(self, grads: bool = False) -> List[List[Tuple[Tensor, Tensor]]]:
        """Dict models: per key (sorted order) the [(W, b)] of its MlpEncoder ([] for identity encoders)"""
        src = self.grads if grads else self.params
        sp = self.spec
        return [[(src[sp.key_encoder_name(k, i, "weight")], src[sp.key_encoder_name(k, i, "bias")])
                 for i in range(len(sp.encoder_mlp_layers))] for k, _ in sp.obs_keys]

    def tower_layers(self, tower: str, grads: bool = False) -> List[Tuple[Tensor, Tensor]]:
        """separate actor / critic weights: [(W, b)] of one tower ("actor_" / "critic_"), encoder then decoder MLP"""
        return self.tower_encoder_layers(tower, grads) + self.tower_decoder_layers(tower, grads)

    def tower_encoder_layers(self, tower: str, grads: bool = False) -> List[Tuple[Tensor, Tensor]]:
        """[(W, b)] of one tower's encoder MLP (the layers before its core)"""
        src = self.grads if grads else self.params
        return [(src[f"{tower}encoder.encoders.obs.mlp_head.{2 * i}.weight"], src[f"{tower}encoder.encoders.obs.mlp_head.{2 * i}.bias"])
                for i in range(len(self.spec.encoder_mlp_layers))]

    def tower_decoder_layers(self, tower: str, grads: bool = False) -> List[Tuple[Tensor, Tensor]]:
        """[(W, b)] of one tower's decoder MLP (the layers after its core)"""
        src = self.grads if grads else self.params
        return [(src[f"{tower}decoder.mlp.{2 * i}.weight"], src[f"{tower}decoder.mlp.{2 * i}.bias"])
                for i in range(len(self.spec.decoder_mlp_layers))]

    def refresh_cat_heads(self) -> None:
        """separate weights: the heads kernels read ONE tail [M, 2H] = [actor tail | critic tail]; critic_linear and
        distribution_linear are embedded in zero-padded [., 2H] matrices (value <- critic half, logits <- actor half)."""
        if not self.spec.separate_towers:
            return
        H = self.spec.tail_input_size
        if not hasattr(self, "Wv_cat"):
            A = self.spec.num_linear_action_outputs
            self.Wv_cat = torch.zeros((1, 2 * H), dtype=torch.float32, device=self.device)
            self.Wa_cat = torch.zeros((A, 2 * H), dtype=torch.float32, device=self.device)
        self.Wv_cat[:, H:].copy_(self.params["critic_linear.weight"])
        self.Wa_cat[:, :H].copy_(self.params["action_parameterization.distribution_linear.weight"])

    def conv_params(self, grads: bool = False) -> List[Tuple[Tensor, Tensor]]:
        """[(W [C_out, C_in, k, k], b [C_out])] of the conv head, in ModelSpec.conv_param_layout() order"""
        src = self.grads if grads else self.params
        return [(src[f"{p}.weight"], src[f"{p}.bias"]) for p, _ in self.spec.conv_param_layout()]

    def decoder_layers(self, grads: bool = False) -> List[Tuple[Tensor, Tensor]]:
        src = self.grads if grads else self.params
        return [(src[f"decoder.mlp.{2 * i}.weight"], src[f"decoder.mlp.{2 * i}.bias"])
                for i in range(len(self.spec.decoder_mlp_layers))]

    def rnn_params(self, grads: bool = False, layer: int = 0, tower: str = "") -> Tuple[Tensor, Tensor, Tensor, Tensor]:
        """(W_ih [G*H, in], W_hh [G*H, H], b_ih, b_hh) of one layer of the GRU/LSTM core (in = H above layer 0); tower
        "actor_" / "critic_" selects that tower's core of a separate-weights model"""
        src = self.grads if grads else self.params
        p, k = f"{tower}core.core.", layer
        return (src[f"{p}weight_ih_l{k}"], src[f"{p}weight_hh_l{k}"], src[f"{p}bias_ih_l{k}"], src[f"{p}bias_hh_l{k}"])

    def hidden_layer_grads(self) -> List[Tuple[Tensor, Tensor]]:
        return self.encoder_layers(grads=True) + self.decoder_layers(grads=True)

    @property
    def learned_log_std(self):
        """the learned log-stddev vector (None unless continuous with adaptive_stddev=False)"""
        return self.params.get("action_parameterization.learned_stddev")

    def dist_kwargs(self) -> Dict:
        """distribution description for the continuous heads / loss ops"""
        sp = self.spec
        return dict(act_dim=sp.num_actions, adaptive_stddev=sp.adaptive_stddev, learned_log_std=self.learned_log_std,
                    tanh_scale=sp.continuous_tanh_scale)

    @property
    def critic(self) -> Tuple[Tensor, Tensor]:
        return self.params["critic_linear.weight"], self.params["critic_linear.bias"]

    @property
    def actor(self) -> Tuple[Tensor, Tensor]:
        return (self.params["action_parameterization.distribution_linear.weight"],
                self.params["action_parameterization.distribution_linear.bias"])

    # ---- checkpoint compatibility (learner.py:323-332: 'model' entry) -------------------------------------------
    def state_dict(self) -> Dict[str, Tensor]:
        sd: Dict[str, Tensor] = {}
        if self.spec.normalize_input:
            # one RunningMeanStdInPlace per key (running_mean_std.py:113-136), statistics of the key's own shape; the keys of
            # a packed row share one count
            for prefix, c, d in self.spec.obs_norm_prefixes:
                shp = self.spec.obs_shape if self.spec.obs_shape is not None else (d,)
                sd[prefix + "running_mean"] = self.obs_mean[c: c + d].clone().view(shp)
                sd[prefix + "running_var"] = self.obs_var[c: c + d].clone().view(shp)
                sd[prefix + "count"] = self.obs_count.clone()
        if self.spec.normalize_returns:
            sd[RET_NORM_PREFIX + "running_mean"] = self.ret_mean.clone()
            sd[RET_NORM_PREFIX + "running_var"] = self.ret_var.clone()
            sd[RET_NORM_PREFIX + "count"] = self.ret_count.clone()
        for n in self.names:
            sd[n] = self.params[n].clone()
        return sd

    def load_state_dict(self, sd: Dict[str, Tensor], strict: bool = True) -> None:
        known = set(self.names)
        obs_norm = {}       # state_dict key -> (buffer, first column, width) of the per-key normaliser statistics
        for prefix, c, d in self.spec.obs_norm_prefixes:
            obs_norm[prefix + "running_mean"] = (self.obs_mean, c, d)
            obs_norm[prefix + "running_var"] = (self.obs_var, c, d)
            obs_norm[prefix + "count"] = (self.obs_count, 0, 1)
        for k, v in sd.items():
            v = torch.as_tensor(v)
            if k in known:
                self.params[k].copy_(v.to(self.device, torch.float32).view(self.params[k].shape))
            elif k in obs_norm:
                buf, c, d = obs_norm[k]
                buf[c: c + d].copy_(v.to(self.device).reshape(-1))     # image observations: [C,H,W] statistics, flat here
            elif k == RET_NORM_PREFIX + "running_mean":
                self.ret_mean.copy_(v.to(self.device).view(1))
            elif k == RET_NORM_PREFIX + "running_var":
                self.ret_var.copy_(v.to(self.device).view(1))
            elif k == RET_NORM_PREFIX + "count":
                self.ret_count.copy_(v.to(self.device).view(1))
            elif strict:
                raise KeyError(f"unexpected key in state_dict: {k}")
        self.weights_changed()
        if strict:
            missing = known - set(sd.keys())
            if missing:
                raise KeyError(f"missing keys in state_dict: {sorted(missing)}")

    def optimizer_state_dict(self, step: int, lr: float, betas, eps: float) -> dict:
        """torch.optim.Adam.state_dict() layout so reference tooling can load it (learner.py:329)."""
        state = {}
        for i, n in enumerate(self.names):
            o, shp = self._slices[n]
            k = math.prod(shp)
            state[i] = dict(step=torch.tensor(float(step)), exp_avg=self.exp_avg[o : o + k].view(shp).clone(),
                            exp_avg_sq=self.exp_avg_sq[o : o + k].view(shp).clone())
        group = dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=0, amsgrad=False, maximize=False, foreach=None,
                     capturable=False, differentiable=False, fused=None, decoupled_weight_decay=False,
                     params=list(range(len(self.names))))
        return dict(state=state, param_groups=[group])

    def load_optimizer_state_dict(self, osd: dict) -> int:
        step = 0
        for i, n in enumerate(self.names):
            if i not in osd["state"]:
                continue
            st = osd["state"][i]
            o, shp = self._slices[n]
            k = math.prod(shp)
            self.exp_avg[o : o + k].copy_(st["exp_avg"].to(self.device).reshape(-1))
            self.exp_avg_sq[o : o + k].copy_(st["exp_avg_sq"].to(self.device).reshape(-1))
            step = int(float(st["step"]))
        return step
