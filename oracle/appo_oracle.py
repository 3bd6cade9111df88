"""CPU ORACLE -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A plain PyTorch-fp32 (CPU) restatement of the reference's APPO hot path
(rollout sampler -> PPO/V-trace learner), written from the reference's
behaviour and citing the reference file:line each function follows
(paths relative to the reference's sample_factory/ package).

Who may import this: tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference leg -- only as the checker / the timed CPU
baseline.  The product (sample_factory_b200/) must never import it.

Parity pinning: this oracle is PINNED against outputs of the reference itself,
executed in the build container from a reference checkout (oracle/install_ref.py: reference_dir()) under oracle/ref_shims.py
by tests/golden/make_golden.py; the resulting vectors are committed under
tests/golden/*.npz and checked by tests/test_oracle_golden.py (no GPU needed).
The reference's only known-answer vector for this path (logits [0,1,2] ->
probs [0.09003057, 0.24472847, 0.66524096], tests/algo/test_action_distributions.py:142-173)
is checked there too.

All tensors are torch CPU tensors; layouts are the reference's trajectory
layout (algo/utils/shared_buffers.py:79-117): [num_traj, T(+1), ...].
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import torch
from torch import Tensor

NORM_EPS = 1e-5  # algo/utils/running_mean_std.py:17
NORM_CLIP = 5.0  # algo/utils/running_mean_std.py:18


@dataclass
class OracleCfg:
    """The subset of reference flags (cfg/cfg.py) that the hot path reads. Defaults = reference defaults."""

    obs_dim: int = 64
    num_actions: int = 8  # Discrete(n), or the dimension of a Box action space when `continuous`
    # gym.spaces.Tuple(Discrete(n_0), Discrete(n_1), ...) -> TupleActionDistribution (action_distributions.py:197-286):
    # independent categorical heads over consecutive logit segments; num_actions is then sum(n_k)
    action_segments: Optional[List[int]] = None
    action_mask: bool = False   # the env's obs dict carries an "action_mask" entry (inference_worker.py:324-331)
    continuous: bool = False           # gym.spaces.Box action space -> ContinuousActionDistribution
    adaptive_stddev: bool = True       # cfg.py:577: False -> one learned log-stddev vector (mujoco examples)
    continuous_tanh_scale: float = 0.0  # cfg.py:583 (only read by the non-adaptive parameterization)
    initial_stddev: float = 1.0        # cfg.py:591
    encoder_mlp_layers: List[int] = field(default_factory=lambda: [512, 512])
    decoder_mlp_layers: List[int] = field(default_factory=list)
    nonlinearity: str = "elu"
    rollout: int = 32
    recurrence: int = 32
    batch_size: int = 1024
    num_batches_per_epoch: int = 1
    num_epochs: int = 1
    gamma: float = 0.99
    gae_lambda: float = 0.95
    ppo_clip_ratio: float = 0.1
    ppo_clip_value: float = 1.0
    exploration_loss_coeff: float = 0.003
    exploration_loss: str = "entropy"   # or "symmetric_kl" (learner.py:181-186, categorical distributions only)
    optimizer: str = "adam"             # or "lamb" (learner.py:228-243, algo/utils/optimizers.py)
    # False -> ActorCriticSeparateWeights (model/actor_critic.py:198-322): an actor tower feeding distribution_linear and a
    # critic tower feeding critic_linear (MLP encoders / decoders only in this restatement; rnn placeholder state size 2)
    actor_critic_share_weights: bool = True
    value_loss_coeff: float = 0.5
    kl_loss_coeff: float = 0.0
    max_grad_norm: float = 4.0
    learning_rate: float = 1e-4
    adam_eps: float = 1e-6
    adam_beta1: float = 0.9
    adam_beta2: float = 0.999
    normalize_input: bool = True
    normalize_returns: bool = True
    obs_subtract_mean: float = 0.0
    obs_scale: float = 1.0
    value_bootstrap: bool = False
    with_vtrace: bool = False
    vtrace_rho: float = 1.0
    vtrace_c: float = 1.0
    reward_scale: float = 1.0
    reward_clip: float = 1000.0
    max_policy_lag: int = 1000
    policy_id: int = 0
    # image observations: obs_shape = (C, H, W) selects the ConvEncoder (model/encoder.py:88-145), obs_dim = C*H*W
    obs_shape: Optional[Tuple[int, int, int]] = None
    encoder_conv_architecture: str = "convnet_atari"                       # cfg.py:506-517
    encoder_conv_mlp_layers: List[int] = field(default_factory=lambda: [512])   # cfg.py:520-526
    use_rnn: bool = False      # model/core.py:19-64 (ModelCoreRNN) between encoder and decoder
    rnn_type: str = "gru"
    rnn_size: int = 512


# --------------------------------------------------------------------------------------
# Parameter naming = reference state_dict keys (model/actor_critic.py:136-158, encoder.py:72-84)
# --------------------------------------------------------------------------------------
CONV_ARCH = {  # model/encoder.py:127-134: (out_channels, kernel, stride) per Conv2d, input channels chain from obs
    "convnet_simple": [(32, 8, 4), (64, 4, 2), (128, 3, 2)],
    "convnet_impala": [(16, 8, 4), (32, 4, 2)],
    "convnet_atari": [(32, 8, 4), (64, 4, 2), (64, 3, 1)],
}


def conv_w(i: int) -> str:
    return f"encoder.encoders.obs.enc.conv_head.{2 * i}.weight"   # Sequential(Conv2d, act, Conv2d, act, ...)


def conv_b(i: int) -> str:
    return f"encoder.encoders.obs.enc.conv_head.{2 * i}.bias"


def conv_fc_w(i: int) -> str:
    return f"encoder.encoders.obs.enc.mlp_layers.{2 * i}.weight"


def conv_fc_b(i: int) -> str:
    return f"encoder.encoders.obs.enc.mlp_layers.{2 * i}.bias"


def conv_out_shapes(cfg: "OracleCfg") -> List[Tuple[int, int, int]]:
    """(C, H, W) after every conv layer (no padding: out = (in - k) // s + 1)"""
    c, h, w = cfg.obs_shape
    out = []
    for (co, k, s_) in CONV_ARCH[cfg.encoder_conv_architecture]:
        h, w = (h - k) // s_ + 1, (w - k) // s_ + 1
        out.append((co, h, w))
    return out


def enc_w(i: int, tower: str = "") -> str:
    return f"{tower}encoder.encoders.obs.mlp_head.{2 * i}.weight"


def enc_b(i: int, tower: str = "") -> str:
    return f"{tower}encoder.encoders.obs.mlp_head.{2 * i}.bias"


def dec_w(i: int, tower: str = "") -> str:
    return f"{tower}decoder.mlp.{2 * i}.weight"


def dec_b(i: int, tower: str = "") -> str:
    return f"{tower}decoder.mlp.{2 * i}.bias"


RNN_W_IH, RNN_W_HH, RNN_B_IH, RNN_B_HH = (
    "core.core.weight_ih_l0", "core.core.weight_hh_l0", "core.core.bias_ih_l0", "core.core.bias_hh_l0",
)
CRITIC_W, CRITIC_B = "critic_linear.weight", "critic_linear.bias"
ACTION_W, ACTION_B = (
    "action_parameterization.distribution_linear.weight",
    "action_parameterization.distribution_linear.bias",
)
LEARNED_STD = "action_parameterization.learned_stddev"
OBS_MEAN = "obs_normalizer.running_mean_std.running_mean_std.obs.running_mean"
OBS_VAR = "obs_normalizer.running_mean_std.running_mean_std.obs.running_var"
OBS_COUNT = "obs_normalizer.running_mean_std.running_mean_std.obs.count"
RET_MEAN, RET_VAR, RET_COUNT = (
    "returns_normalizer.running_mean",
    "returns_normalizer.running_var",
    "returns_normalizer.count",
)


def param_names(cfg: OracleCfg) -> List[str]:
    """Trainable parameter order == nn.Module.parameters() order of the reference model."""
    names = []
    if not cfg.actor_critic_share_weights:
        # module registration order of ActorCriticSeparateWeights.__init__ (actor_critic.py:208-225)
        assert cfg.obs_shape is None and not cfg.use_rnn
        for tw in ("actor_", "critic_"):
            for i in range(len(cfg.encoder_mlp_layers)):
                names += [enc_w(i, tw), enc_b(i, tw)]
        for tw in ("actor_", "critic_"):
            for i in range(len(cfg.decoder_mlp_layers)):
                names += [dec_w(i, tw), dec_b(i, tw)]
        names += [CRITIC_W, CRITIC_B]
        if cfg.continuous and not cfg.adaptive_stddev:
            names += [LEARNED_STD]
        names += [ACTION_W, ACTION_B]
        return names
    if cfg.obs_shape is not None:
        for i in range(len(CONV_ARCH[cfg.encoder_conv_architecture])):
            names += [conv_w(i), conv_b(i)]
        for i in range(len(cfg.encoder_conv_mlp_layers)):
            names += [conv_fc_w(i), conv_fc_b(i)]
    else:
        for i in range(len(cfg.encoder_mlp_layers)):
            names += [enc_w(i), enc_b(i)]
    if cfg.use_rnn:
        names += [RNN_W_IH, RNN_W_HH, RNN_B_IH, RNN_B_HH]
    for i in range(len(cfg.decoder_mlp_layers)):
        names += [dec_w(i), dec_b(i)]
    names += [CRITIC_W, CRITIC_B]
    if cfg.continuous and not cfg.adaptive_stddev:
        # ActionParameterizationContinuousNonAdaptiveStddev (action_parameterization.py:42-62): nn.Module.parameters()
        # yields a module's own parameters before its children's, so learned_stddev precedes distribution_linear.*
        names += [LEARNED_STD]
    names += [ACTION_W, ACTION_B]
    return names


def num_linear_action_outputs(cfg: OracleCfg) -> int:
    """rows of distribution_linear: n (Discrete), 2A (Box, adaptive stddev), A (Box, learned stddev)"""
    if not cfg.continuous:
        return cfg.num_actions
    return 2 * cfg.num_actions if cfg.adaptive_stddev else cfg.num_actions


def num_action_params(cfg: OracleCfg) -> int:
    """calc_num_action_parameters (action_distributions.py:33-44): width of `action_logits`"""
    return 2 * cfg.num_actions if cfg.continuous else cfg.num_actions


def action_width(cfg: OracleCfg) -> int:
    """calc_num_actions (action_distributions.py:16-30): width of `actions`"""
    if cfg.action_segments:
        return len(cfg.action_segments)
    return cfg.num_actions if cfg.continuous else 1


def rnn_state_size(cfg: OracleCfg) -> int:
    """model/model_utils.py:11-24 (single layer): 1 placeholder without RNN, H for GRU, 2H for LSTM; doubled when actor and
    critic have separate weights."""
    if not cfg.use_rnn:
        return 1 if cfg.actor_critic_share_weights else 2
    return cfg.rnn_size * (2 if cfg.rnn_type == "lstm" else 1)


def init_state(cfg: OracleCfg, seed: int = 0) -> Dict[str, Tensor]:
    """Random weights (NOT the reference's orthogonal init -- parity tests load weights, SURVEY App.A-15)
    plus normalizer buffers initialised as running_mean_std.py:45-47 (mean 0, var 1, count 1, float64)."""
    g = torch.Generator().manual_seed(seed)
    st: Dict[str, Tensor] = {}
    d = cfg.obs_dim
    if not cfg.actor_critic_share_weights:
        for tw in ("actor_", "critic_"):
            d = cfg.obs_dim
            for i, h in enumerate(cfg.encoder_mlp_layers):
                st[enc_w(i, tw)] = torch.randn(h, d, generator=g) / math.sqrt(d)
                st[enc_b(i, tw)] = torch.randn(h, generator=g) * 0.01
                d = h
            for i, h in enumerate(cfg.decoder_mlp_layers):
                st[dec_w(i, tw)] = torch.randn(h, d, generator=g) / math.sqrt(d)
                st[dec_b(i, tw)] = torch.randn(h, generator=g) * 0.01
                d = h
    elif cfg.obs_shape is not None:
        ci = cfg.obs_shape[0]
        for i, (co, k, _s) in enumerate(CONV_ARCH[cfg.encoder_conv_architecture]):
            st[conv_w(i)] = torch.randn(co, ci, k, k, generator=g) / math.sqrt(ci * k * k)
            st[conv_b(i)] = torch.randn(co, generator=g) * 0.01
            ci = co
        c_, h_, w_ = conv_out_shapes(cfg)[-1]
        d = c_ * h_ * w_
        for i, h in enumerate(cfg.encoder_conv_mlp_layers):
            st[conv_fc_w(i)] = torch.randn(h, d, generator=g) / math.sqrt(d)
            st[conv_fc_b(i)] = torch.randn(h, generator=g) * 0.01
            d = h
    else:
        for i, h in enumerate(cfg.encoder_mlp_layers):
            st[enc_w(i)] = torch.randn(h, d, generator=g) / math.sqrt(d)
            st[enc_b(i)] = torch.randn(h, generator=g) * 0.01
            d = h
    if cfg.use_rnn:
        H, G = cfg.rnn_size, (4 if cfg.rnn_type == "lstm" else 3)
        k = 1.0 / math.sqrt(H)
        st[RNN_W_IH] = (torch.rand(G * H, d, generator=g) * 2 - 1) * k
        st[RNN_W_HH] = (torch.rand(G * H, H, generator=g) * 2 - 1) * k
        st[RNN_B_IH] = (torch.rand(G * H, generator=g) * 2 - 1) * k
        st[RNN_B_HH] = (torch.rand(G * H, generator=g) * 2 - 1) * k
        d = H
    if cfg.actor_critic_share_weights:
        for i, h in enumerate(cfg.decoder_mlp_layers):
            st[dec_w(i)] = torch.randn(h, d, generator=g) / math.sqrt(d)
            st[dec_b(i)] = torch.randn(h, generator=g) * 0.01
            d = h
    st[CRITIC_W] = torch.randn(1, d, generator=g) / math.sqrt(d)
    st[CRITIC_B] = torch.zeros(1)
    st[ACTION_W] = torch.randn(num_linear_action_outputs(cfg), d, generator=g) / math.sqrt(d)
    st[ACTION_B] = torch.zeros(num_linear_action_outputs(cfg))
    if cfg.continuous and not cfg.adaptive_stddev:
        st[LEARNED_STD] = torch.full((cfg.num_actions,), math.log(cfg.initial_stddev))
    st[OBS_MEAN] = torch.zeros(cfg.obs_dim, dtype=torch.float64)
    st[OBS_VAR] = torch.ones(cfg.obs_dim, dtype=torch.float64)
    st[OBS_COUNT] = torch.ones(1, dtype=torch.float64)
    st[RET_MEAN] = torch.zeros(1, dtype=torch.float64)
    st[RET_VAR] = torch.ones(1, dtype=torch.float64)
    st[RET_COUNT] = torch.ones(1, dtype=torch.float64)
    return st


# --------------------------------------------------------------------------------------
# Normalizers
# --------------------------------------------------------------------------------------
def rms_update(mean: Tensor, var: Tensor, count: Tensor, x: Tensor) -> None:
    """In-place running-moment update. running_mean_std.py:49-62 (merge) and :72-77 (batch moments:
    fp32 `x.mean(0)`, unbiased fp32 `x.var(0)`, merged into the float64 buffers)."""
    batch_count = x.shape[0]
    batch_mean = x.mean(0)
    batch_var = x.var(0)  # unbiased
    delta = batch_mean - mean  # fp32 - fp64 -> fp64
    tot_count = count + batch_count
    new_mean = mean + delta * batch_count / tot_count
    m_a = var * count
    m_b = batch_var * batch_count
    m2 = m_a + m_b + (delta**2) * count * batch_count / tot_count
    new_var = m2 / tot_count
    mean[:], var[:], count[:] = new_mean, new_var, tot_count


def rms_normalize_(x: Tensor, mean: Tensor, var: Tensor) -> None:
    """running_mean_std.py:96-110, normalize branch (in place): (x-mu) * (1/sqrt(var+eps)), clamp +-5."""
    mu = mean.float()
    sigma = torch.sqrt(var.float() + NORM_EPS)
    x.sub_(mu).mul_(1 / sigma).clamp_(-NORM_CLIP, NORM_CLIP)


def rms_denormalize_(x: Tensor, mean: Tensor, var: Tensor) -> None:
    """running_mean_std.py:107-108, denormalize branch (in place): clamp +-5, * sigma, + mu."""
    mu = mean.float()
    sigma = torch.sqrt(var.float() + NORM_EPS)
    x.clamp_(-NORM_CLIP, NORM_CLIP).mul_(sigma).add_(mu)


def normalize_obs(cfg: OracleCfg, st: Dict[str, Tensor], obs: Tensor, update_stats: bool) -> Tensor:
    """utils/normalize.py:51-70: clone -> (sub mean) -> (scale) -> running-mean-std (stats updated only in
    training mode, running_mean_std.py:66)."""
    x = obs.float().clone()
    if abs(cfg.obs_subtract_mean) > 1e-8:
        x.sub_(cfg.obs_subtract_mean)
    if abs(cfg.obs_scale - 1.0) > 1e-8:
        x.mul_(1.0 / cfg.obs_scale)
    if cfg.normalize_input:
        if update_stats:
            rms_update(st[OBS_MEAN], st[OBS_VAR], st[OBS_COUNT], x)
        rms_normalize_(x, st[OBS_MEAN], st[OBS_VAR])
    return x


# --------------------------------------------------------------------------------------
# Model forward (model/actor_critic.py:160-195, encoder.py:82-84, decoder.py:28, action_parameterization.py:33-39)
# --------------------------------------------------------------------------------------
def _act(cfg: OracleCfg, x: Tensor) -> Tensor:
    if cfg.nonlinearity == "elu":
        return torch.nn.functional.elu(x)
    if cfg.nonlinearity == "relu":
        return torch.relu(x)
    if cfg.nonlinearity == "tanh":
        return torch.tanh(x)
    raise ValueError(cfg.nonlinearity)


def encoder_forward(cfg: OracleCfg, st: Dict[str, Tensor], x: Tensor) -> Tensor:
    """forward_head (actor_critic.py:160-162): MlpEncoder, or ConvEncoder (encoder.py:88-118) for image observations
    (x arrives as flat [B, C*H*W] rows in CHW order, the layout of the trajectory buffers)."""
    if cfg.obs_shape is not None:
        h = x.view(x.shape[0], *cfg.obs_shape)
        for i, (_co, _k, s_) in enumerate(CONV_ARCH[cfg.encoder_conv_architecture]):
            h = _act(cfg, torch.nn.functional.conv2d(h, st[conv_w(i)], st[conv_b(i)], stride=s_))
        h = h.contiguous().view(h.shape[0], -1)   # :115 (C, H, W) flatten order
        for i in range(len(cfg.encoder_conv_mlp_layers)):
            h = _act(cfg, torch.nn.functional.linear(h, st[conv_fc_w(i)], st[conv_fc_b(i)]))
        return h
    h = x
    for i in range(len(cfg.encoder_mlp_layers)):
        h = _act(cfg, torch.nn.functional.linear(h, st[enc_w(i)], st[enc_b(i)]))
    return h


def tail_forward(cfg: OracleCfg, st: Dict[str, Tensor], h: Tensor) -> Tuple[Tensor, Tensor]:
    """forward_tail (actor_critic.py:168-186): decoder MLP -> critic_linear / distribution_linear."""
    for i in range(len(cfg.decoder_mlp_layers)):
        h = _act(cfg, torch.nn.functional.linear(h, st[dec_w(i)], st[dec_b(i)]))
    values = torch.nn.functional.linear(h, st[CRITIC_W], st[CRITIC_B]).squeeze(-1)
    logits = torch.nn.functional.linear(h, st[ACTION_W], st[ACTION_B])
    if cfg.continuous and not cfg.adaptive_stddev:
        # ActionParameterizationContinuousNonAdaptiveStddev.forward (action_parameterization.py:64-78)
        means = logits
        if cfg.continuous_tanh_scale > 0:
            means = torch.tanh(means / cfg.continuous_tanh_scale) * cfg.continuous_tanh_scale
        logits = torch.cat((means, st[LEARNED_STD].repeat(means.shape[0], 1)), dim=1)
    return values, logits


def rnn_cell(cfg: OracleCfg, st: Dict[str, Tensor], x: Tensor, state: Tensor) -> Tuple[Tensor, Tensor]:
    """One step of ModelCoreRNN (model/core.py:37-64) written out: torch.nn.GRU / LSTM cell equations, gate order as in
    the PyTorch weight layout (GRU: r,z,n ; LSTM: i,f,g,o); LSTM state = [h || c] (core.py:51-53).
    Returns (core_output [B,H], new_state [B, H or 2H])."""
    H = cfg.rnn_size
    gi = torch.nn.functional.linear(x, st[RNN_W_IH], st[RNN_B_IH])
    if cfg.rnn_type == "gru":
        h = state
        gh = torch.nn.functional.linear(h, st[RNN_W_HH], st[RNN_B_HH])
        r = torch.sigmoid(gi[:, :H] + gh[:, :H])
        z = torch.sigmoid(gi[:, H:2 * H] + gh[:, H:2 * H])
        n = torch.tanh(gi[:, 2 * H:] + r * gh[:, 2 * H:])
        h_new = (1 - z) * n + z * h
        return h_new, h_new
    h, c = state[:, :H], state[:, H:]
    g = gi + torch.nn.functional.linear(h, st[RNN_W_HH], st[RNN_B_HH])
    i_, f_, g_, o_ = torch.sigmoid(g[:, :H]), torch.sigmoid(g[:, H:2 * H]), torch.tanh(g[:, 2 * H:3 * H]), torch.sigmoid(g[:, 3 * H:])
    c_new = f_ * c + i_ * g_
    h_new = o_ * torch.tanh(c_new)
    return h_new, torch.cat([h_new, c_new], dim=1)


def _tower(cfg: OracleCfg, st: Dict[str, Tensor], x: Tensor, tw: str) -> Tensor:
    h = x
    for i in range(len(cfg.encoder_mlp_layers)):
        h = _act(cfg, torch.nn.functional.linear(h, st[enc_w(i, tw)], st[enc_b(i, tw)]))
    for i in range(len(cfg.decoder_mlp_layers)):
        h = _act(cfg, torch.nn.functional.linear(h, st[dec_w(i, tw)], st[dec_b(i, tw)]))
    return h


def separate_forward(cfg: OracleCfg, st: Dict[str, Tensor], x: Tensor) -> Tuple[Tensor, Tensor]:
    """ActorCriticSeparateWeights.forward (actor_critic.py:283-318) without recurrent cores: the critic tower feeds
    critic_linear, the actor tower feeds the action parameterization."""
    values = torch.nn.functional.linear(_tower(cfg, st, x, "critic_"), st[CRITIC_W], st[CRITIC_B]).squeeze(-1)
    logits = torch.nn.functional.linear(_tower(cfg, st, x, "actor_"), st[ACTION_W], st[ACTION_B])
    if cfg.continuous and not cfg.adaptive_stddev:
        means = logits
        if cfg.continuous_tanh_scale > 0:
            means = torch.tanh(means / cfg.continuous_tanh_scale) * cfg.continuous_tanh_scale
        logits = torch.cat((means, st[LEARNED_STD].repeat(means.shape[0], 1)), dim=1)
    return values, logits


def model_forward(cfg: OracleCfg, st: Dict[str, Tensor], x: Tensor, rnn_state: Optional[Tensor] = None):
    """ActorCriticSharedWeights.forward (actor_critic.py:188-195): (values, logits, new_rnn_state)."""
    if not cfg.actor_critic_share_weights:
        values, logits = separate_forward(cfg, st, x)
        return values, logits, rnn_state
    h = encoder_forward(cfg, st, x)
    new_state = rnn_state
    if cfg.use_rnn:
        h, new_state = rnn_cell(cfg, st, h, rnn_state)
    values, logits = tail_forward(cfg, st, h)
    return values, logits, new_state


def mlp_forward(cfg: OracleCfg, st: Dict[str, Tensor], x: Tensor) -> Tuple[Tensor, Tensor]:
    """normalized obs [B, D] -> (values [B], action_logits [B, A]) for the non-recurrent model."""
    assert not cfg.use_rnn
    return tail_forward(cfg, st, encoder_forward(cfg, st, x))


# --------------------------------------------------------------------------------------
# Categorical distribution (algo/utils/action_distributions.py:99-194)
# --------------------------------------------------------------------------------------
def cat_probs(logits: Tensor) -> Tensor:
    return torch.softmax(logits, dim=-1)  # :116


def cat_log_probs(logits: Tensor) -> Tensor:
    return torch.log_softmax(logits, dim=-1)  # :125


def cat_sample(logits: Tensor, noise_q: Tensor) -> Tensor:
    """:135-143. torch.multinomial(p, 1, True) == argmax(p / q), q ~ Exp(1) (SURVEY App.E, re-verified by
    make_golden.py against the reference run). The noise is an explicit input."""
    return torch.argmax(cat_probs(logits) / noise_q, dim=-1, keepdim=True)


def cat_log_prob(logits: Tensor, actions: Tensor) -> Tensor:
    """:145-148"""
    return torch.gather(cat_log_probs(logits), -1, actions.long().view(-1, 1)).view(-1)


def masked_cat_probs(logits: Tensor, mask: Tensor) -> Tensor:
    """masked_softmax :84-90: invalid logits pushed down by 1e9, softmax, times mask, renormalised with +1e-13"""
    p = torch.softmax(logits + (mask == 0) * -1e9, dim=-1)
    p = p * mask
    return p / (p.sum(dim=-1, keepdim=True) + 1e-13)


def masked_cat_log_probs(logits: Tensor, mask: Tensor) -> Tensor:
    """masked_log_softmax :93-95"""
    return torch.log_softmax(logits + (mask == 0) * -1e9, dim=-1)


def masked_cat_sample(logits: Tensor, mask: Tensor, noise_q: Tensor) -> Tensor:
    """sample() with an action mask :135-143: rows whose probabilities are all zero fall back to 1e-6 everywhere"""
    p = masked_cat_probs(logits, mask)
    all_zero = (p.sum(dim=-1) == 0).unsqueeze(-1)
    p = torch.where(all_zero, torch.full_like(p, 1e-6), p)
    return torch.argmax(p / noise_q, dim=-1, keepdim=True)


def masked_cat_log_prob(logits: Tensor, mask: Tensor, actions: Tensor) -> Tensor:
    return torch.gather(masked_cat_log_probs(logits, mask), -1, actions.long().view(-1, 1)).view(-1)


def cat_entropy(logits: Tensor) -> Tensor:
    """:150-152"""
    return -(cat_log_probs(logits) * cat_probs(logits)).sum(-1)


def cat_symmetric_kl_with_uniform_prior(logits: Tensor) -> Tensor:
    """:168-177"""
    probs, log_probs = cat_probs(logits), cat_log_probs(logits)
    u = 1 / logits.shape[-1]
    log_u = math.log(u)
    return 0.5 * ((probs * (log_probs - log_u)).sum(-1) + (u * (log_u - log_probs)).sum(-1))


def cat_kl(logits_p: Tensor, logits_q: Tensor) -> Tensor:
    """KL(p || q), :154-158,179-180"""
    return (cat_probs(logits_p) * (cat_log_probs(logits_p) - cat_log_probs(logits_q))).sum(-1)


# --------------------------------------------------------------------------------------
# Diagonal Gaussian distribution (algo/utils/action_distributions.py:290-323 = Independent(Normal(means, std), 1);
# torch/distributions/normal.py for the arithmetic; SURVEY App.C)
# --------------------------------------------------------------------------------------
STDDEV_MIN, STDDEV_MAX = 1e-4, 1e4  # action_distributions.py:291-292


def gauss_split(params: Tensor) -> Tuple[Tensor, Tensor, Tensor]:
    """_init_impl :299-306 -> (means, log_std, clamped stddevs)"""
    means, log_std = torch.chunk(params, 2, dim=1)
    return means, log_std, torch.clamp(log_std.exp(), STDDEV_MIN, STDDEV_MAX)


def gauss_sample(params: Tensor, eps: Tensor) -> Tensor:
    """Normal.sample() == torch.normal(mean, std) == eps * std + mean with the product and the sum rounded separately
    (eps = the N(0,1) draw; an explicit input here, recovered from the reference's generator by make_golden.py)."""
    means, _, std = gauss_split(params)
    return eps * std + means


def gauss_log_prob(params: Tensor, actions: Tensor) -> Tensor:
    """Independent(Normal).log_prob: sum over the action dimension of normal.py:84-94"""
    means, _, std = gauss_split(params)
    var = std**2
    lp = -((actions - means) ** 2) / (2 * var) - std.log() - math.log(math.sqrt(2 * math.pi))
    return lp.sum(-1)


def gauss_entropy(params: Tensor) -> Tensor:
    """normal.py:107-108 summed over the action dimension"""
    _, _, std = gauss_split(params)
    return (0.5 + 0.5 * math.log(2 * math.pi) + torch.log(std)).sum(-1)


def gauss_kl(params_p: Tensor, params_q: Tensor) -> Tensor:
    """KL(p || q) of Independent Normals (torch/distributions/kl.py _kl_normal_normal, summed)"""
    mp, _, sp = gauss_split(params_p)
    mq, _, sq = gauss_split(params_q)
    var_ratio = (sp / sq).pow(2)
    t1 = ((mp - mq) / sq).pow(2)
    return (0.5 * (var_ratio + t1 - 1 - var_ratio.log())).sum(-1)


# Tuple of independent categorical heads (action_distributions.py:197-286): everything is a sum over the heads
def tuple_split(cfg: OracleCfg, logits: Tensor):
    return torch.split(logits, list(cfg.action_segments), dim=1)


def tuple_sample(cfg: OracleCfg, logits: Tensor, noise_q: Tensor) -> Tensor:
    """:243-252: each head samples on its own; noise_q [N, sum n_k] holds the heads' Exp(1) draws side by side"""
    return torch.cat([cat_sample(l, q) for l, q in zip(tuple_split(cfg, logits), tuple_split(cfg, noise_q))], dim=1)


def tuple_log_prob(cfg: OracleCfg, logits: Tensor, actions: Tensor) -> Tensor:
    acts = actions.view(logits.shape[0], -1)
    return sum(cat_log_prob(l, acts[:, k]) for k, l in enumerate(tuple_split(cfg, logits)))


def dist_log_prob(cfg: OracleCfg, logits: Tensor, actions: Tensor) -> Tensor:
    if cfg.action_segments:
        return tuple_log_prob(cfg, logits, actions)
    return gauss_log_prob(logits, actions.view(logits.shape[0], -1)) if cfg.continuous else cat_log_prob(logits, actions)


def dist_entropy(cfg: OracleCfg, logits: Tensor) -> Tensor:
    if cfg.action_segments:
        return sum(cat_entropy(l) for l in tuple_split(cfg, logits))
    return gauss_entropy(logits) if cfg.continuous else cat_entropy(logits)


def dist_kl(cfg: OracleCfg, logits_p: Tensor, logits_q: Tensor) -> Tensor:
    if cfg.action_segments:
        return sum(cat_kl(lp, lq) for lp, lq in zip(tuple_split(cfg, logits_p), tuple_split(cfg, logits_q)))
    return gauss_kl(logits_p, logits_q) if cfg.continuous else cat_kl(logits_p, logits_q)


def dist_symmetric_kl(cfg: OracleCfg, logits: Tensor) -> Tensor:
    if cfg.action_segments:
        return sum(cat_symmetric_kl_with_uniform_prior(l) for l in tuple_split(cfg, logits))
    return cat_symmetric_kl_with_uniform_prior(logits)


# --------------------------------------------------------------------------------------
# Sampler: one policy step + one env step  (inference_worker.py:313-341, batched_sampling.py:298-388)
# --------------------------------------------------------------------------------------
def alloc_trajectories(cfg: OracleCfg, num_traj: int) -> Dict[str, Tensor]:
    """shared_buffers.py:79-117 layout (single 'obs' key, rnn placeholder size 1 -- model_utils.py:11-24)."""
    T, B = cfg.rollout, num_traj
    t: Dict[str, Tensor] = {}
    if cfg.obs_shape is not None:   # image observations keep the env's dtype (uint8), shared_buffers.py:88-96
        t["obs"] = torch.zeros((B, T + 1, cfg.obs_dim), dtype=torch.uint8)
    else:
        t["obs"] = torch.full((B, T + 1, cfg.obs_dim), -4242.42)
    t["rnn_states"] = torch.full((B, T + 1, rnn_state_size(cfg)), -4242.42)
    t["actions"] = torch.full((B, T, action_width(cfg)), -4242.42)
    t["action_logits"] = torch.full((B, T, num_action_params(cfg)), -4242.42)
    t["log_prob_actions"] = torch.full((B, T), -4242.42)
    t["values"] = torch.full((B, T + 1), -4242.42)
    t["policy_version"] = torch.full((B, T), -4242.42)
    t["rewards"] = torch.full((B, T), -42.42)
    t["dones"] = torch.ones((B, T), dtype=torch.bool)
    t["time_outs"] = torch.zeros((B, T), dtype=torch.bool)
    t["policy_id"] = torch.full((B, T), -1, dtype=torch.int32)
    t["valids"] = torch.zeros((B, T + 1), dtype=torch.bool)
    return t


def policy_step(cfg: OracleCfg, st: Dict[str, Tensor], obs: Tensor, noise_q: Tensor, rnn_state: Optional[Tensor] = None,
                action_mask: Optional[Tensor] = None):
    """inference_worker.py:313-341 body for the categorical model:
    normalize (eval mode: no stat update) -> forward -> sample -> log-prob.
    `action_mask` [N, A] (0 = action not allowed) is the obs dict's "action_mask" entry (:324-331); the stored logits
    stay the raw ones.  Returns (actions int64 [N,1], logits [N,A], log_prob [N], values [N], new_rnn_state)."""
    x = normalize_obs(cfg, st, obs, update_stats=False)
    values, logits, new_state = model_forward(cfg, st, x, rnn_state)
    if action_mask is not None:
        assert not cfg.action_segments and not cfg.continuous, "action masks: plain Discrete action spaces only"
        actions = masked_cat_sample(logits, action_mask, noise_q)
        log_prob = masked_cat_log_prob(logits, action_mask, actions)
        return actions, logits, log_prob, values, new_state
    if cfg.action_segments:
        actions = tuple_sample(cfg, logits, noise_q)
        log_prob = tuple_log_prob(cfg, logits, actions)
    elif cfg.continuous:   # noise_q: [N, A] standard-normal draws
        actions = gauss_sample(logits, noise_q)
        log_prob = gauss_log_prob(logits, actions)
    else:
        actions = cat_sample(logits, noise_q)
        log_prob = cat_log_prob(logits, actions)
    return actions, logits, log_prob, values, new_state


class TapeVecEnv:
    """Synthetic batched env used by goldens, tests and bench (NOT part of the reference; the reference's
    batched-env contract is make_env.py:147-237: step(actions) -> obs, rew, terminated, truncated, infos).

    obs_t is read from a pre-generated tape (independent of actions, so oracle and GPU rollouts stay aligned),
    reward = action / num_actions, terminated / truncated follow fixed integer rules of (global step, env)."""

    def __init__(self, tape: Tensor, num_actions: int, term_period: int = 37, trunc_period: int = 11,
                 with_action_mask: bool = False):
        self.tape = tape  # [L, N, D]
        self.L, self.num_agents, self.obs_dim = tape.shape
        self.num_actions = num_actions
        self.term_period, self.trunc_period = term_period, trunc_period
        self.with_action_mask = with_action_mask
        self.t = 0

    def action_mask(self) -> Tensor:
        """int64 [N, A] mask that goes with the CURRENT observation (obs dict key "action_mask"): a fixed integer rule of
        (step, env, action); every 29th (step + env) row allows nothing (the reference's all-zero fallback)."""
        return tape_action_mask(self.t, torch.arange(self.num_agents), self.num_actions)

    def reset(self) -> Tensor:
        self.t = 0
        return self.tape[0]

    def step(self, actions: Tensor) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
        env = torch.arange(self.num_agents)
        t = self.t
        if actions.is_floating_point():   # Box action space [N, A]: reward = first action component, clipped
            rew = actions.view(self.num_agents, -1)[:, 0].clamp(-1.0, 1.0)
        else:                             # Discrete, or Tuple of Discretes [N, K]: first component / num_actions
            rew = actions.view(self.num_agents, -1)[:, 0].float() / float(self.num_actions)
        terminated = ((t * 7 + env * 13) % self.term_period) == 0
        truncated = (((t + env) % self.trunc_period) == 0) & ~terminated
        self.t += 1
        return self.tape[self.t % self.L], rew, terminated, truncated


def tape_action_mask(t: int, env: Tensor, num_actions: int) -> Tensor:
    a = torch.arange(num_actions).view(1, -1)
    e = env.view(-1, 1)
    allowed = (((t * 3 + e * 5 + a * 7) % 3) == 0) | (a == (t + e) % num_actions)
    allowed = allowed & (((t + e) % 29) != 0)
    return allowed.to(torch.int64)


def rollout(
    cfg: OracleCfg,
    st: Dict[str, Tensor],
    env: TapeVecEnv,
    last_obs: Tensor,
    traj: Dict[str, Tensor],
    noise: Tensor,
    policy_version: int,
    rnn_state: Optional[Tensor] = None,
) -> Tensor:
    """T steps of batched_sampling.py:298-388 + inference_worker.py:313-341 into `traj` (in place).
    noise: [T, N, A] Exp(1) draws. rnn_state [N, S] (S = rnn_state_size) is the runner's last_rnn_state, updated IN
    PLACE (zeros initially, batched_sampling.py:190). Returns the obs after the last step."""
    if rnn_state is None:
        rnn_state = torch.zeros(last_obs.shape[0], rnn_state_size(cfg))
    for t in range(cfg.rollout):
        # generate_policy_request :374-388
        traj["obs"][:, t] = last_obs
        traj["rnn_states"][:, t] = rnn_state
        mask = env.action_mask() if getattr(env, "with_action_mask", False) else None
        actions, logits, log_prob, values, new_state = policy_step(cfg, st, last_obs, noise[t], rnn_state, mask)
        # advance_rollouts part 1 :308-311 (actions stored as float32, SURVEY App.A-1)
        traj["actions"][:, t] = actions.float()
        traj["action_logits"][:, t] = logits
        traj["log_prob_actions"][:, t] = log_prob
        traj["values"][:, t] = values
        traj["policy_version"][:, t] = float(policy_version)  # inference_worker.py:332
        # preprocess_actions :30-82 (discrete: int32, squeezed; Box: float, as is)
        if cfg.continuous:
            env_actions = actions
        elif cfg.action_segments:
            env_actions = actions.to(torch.int32)          # [N, K]: one index per head
        else:
            env_actions = actions.to(torch.int32).squeeze(-1)
        last_obs, rew, terminated, truncated = env.step(env_actions)
        dones = terminated | truncated  # :317
        # _process_rewards :208-213
        r = (rew * cfg.reward_scale).clamp(-cfg.reward_clip, cfg.reward_clip)
        traj["rewards"][:, t] = r
        traj["dones"][:, t] = dones
        traj["time_outs"][:, t] = truncated
        traj["policy_id"][:, t] = cfg.policy_id
        # reset next-step hidden states on episode boundaries :332-335
        rnn_state[:] = new_state * (1.0 - dones.float()).unsqueeze(-1)
    # _finalize_trajectories :289-296
    traj["obs"][:, cfg.rollout] = last_obs
    traj["rnn_states"][:, cfg.rollout] = rnn_state
    return last_obs


# --------------------------------------------------------------------------------------
# Learner: batch preparation (algo/learning/learner.py:943-1034)
# --------------------------------------------------------------------------------------
def gae_advantages(rewards: Tensor, dones: Tensor, values: Tensor, valids: Tensor, gamma: float, lam: float) -> Tensor:
    """algo/utils/rl_utils.py:78-94 + :51-73. rewards/dones [N,T], values/valids [N,T+1] -> adv [N,T]."""
    d = dones.float()
    vl = valids.float()
    deltas = (rewards - values[:, :-1]) * vl[:, :-1] + (1 - d) * (gamma * values[:, 1:] * vl[:, 1:])
    T = rewards.shape[1]
    adv = torch.zeros_like(rewards)
    cumulative = torch.zeros_like(rewards[:, 0])
    discount = gamma * lam
    for i in range(T - 1, -1, -1):
        discount_valid = discount * vl[:, i] + (1 - vl[:, i])
        cumulative = deltas[:, i] + discount_valid * cumulative * (1.0 - d[:, i])
        adv[:, i] = cumulative
    return adv


def prepare_batch(cfg: OracleCfg, st: Dict[str, Tensor], batch: Dict[str, Tensor], train_step: int):
    """learner.py:943-1034. Mutates normalizer statistics in `st` exactly where the reference does.
    Returns (buff dict of flat [N*T,...] tensors, dataset_size, num_invalids)."""
    buff = {k: v.clone() for k, v in batch.items()}
    valids = buff["policy_id"] == cfg.policy_id  # :950
    buff["valids"][:, :-1] = valids & (train_step - buff["policy_version"] < cfg.max_policy_lag)  # :953
    buff["valids"][:, -1] = buff["valids"][:, -2]  # :955

    B, T1, D = buff["obs"].shape
    # :961 -> :925-941: stats updated ONCE over all N*(T+1) rows, before the bootstrap forward
    nobs = normalize_obs(cfg, st, buff["obs"].reshape(B * T1, D), update_stats=True).view(B, T1, D)
    buff["normalized_obs"] = nobs
    del buff["obs"]

    next_values, _, _ = model_forward(cfg, st, nobs[:, -1], buff["rnn_states"][:, -1])  # :965-966 (values_only)
    buff["values"][:, -1] = next_values  # :967

    if cfg.normalize_returns:  # :969-975
        denorm_values = buff["values"].clone()
        rms_denormalize_(denorm_values, st[RET_MEAN], st[RET_VAR])
    else:
        denorm_values = buff["values"]

    if cfg.value_bootstrap:  # :980-990
        buff["rewards"].add_(cfg.gamma * denorm_values[:, :-1] * buff["time_outs"] * buff["dones"])

    if not cfg.with_vtrace:  # :992-1003
        buff["advantages"] = gae_advantages(
            buff["rewards"], buff["dones"], denorm_values, buff["valids"], cfg.gamma, cfg.gae_lambda
        )
        buff["returns"] = buff["advantages"] + buff["valids"][:, :-1] * denorm_values[:, :-1]

    for key in ["normalized_obs", "rnn_states", "values", "valids"]:  # :1006-1007
        buff[key] = buff[key][:, :-1]

    dataset_size = buff["actions"].shape[0] * buff["actions"].shape[1]
    for k in list(buff.keys()):  # :1009-1012
        v = buff[k]
        buff[k] = v.reshape((dataset_size,) + tuple(v.shape[2:]))

    if cfg.normalize_returns and not cfg.with_vtrace:  # :1018-1019 (in place, training mode -> stat update)
        r = buff["returns"]
        rms_update(st[RET_MEAN], st[RET_VAR], st[RET_COUNT], r.view(-1, 1))
        rms_normalize_(r, st[RET_MEAN], st[RET_VAR])

    num_invalids = dataset_size - int(buff["valids"].sum().item())  # :1021
    if num_invalids > 0:  # :1029-1032
        inv = buff["valids"] == 0
        buff["actions"][inv] = 0
        buff["log_prob_actions"][inv] = -1
    return buff, dataset_size, num_invalids


# --------------------------------------------------------------------------------------
# Learner: losses (learner.py:537-669, :431-477) and V-trace (:602-640)
# --------------------------------------------------------------------------------------
def _masked_select(x: Tensor, mask: Tensor, num_invalids: int) -> Tensor:
    """algo/utils/torch_utils.py:50-55"""
    if num_invalids == 0:
        return x
    return torch.masked_select(x, mask)


def vtrace(
    cfg: OracleCfg, ratio: Tensor, values: Tensor, rewards: Tensor, dones: Tensor, recurrence: int
) -> Tuple[Tensor, Tensor]:
    """learner.py:602-640 (SURVEY App.D). All flat [n*R] env-major. Returns (vs, adv)."""
    R = recurrence
    rho = torch.clamp(ratio, max=cfg.vtrace_rho)
    c = torch.clamp(ratio, max=cfg.vtrace_c)
    n = ratio.numel() // R
    vs = torch.zeros(n * R)
    adv = torch.zeros(n * R)
    next_values = (values[R - 1 :: R] - rewards[R - 1 :: R]) / cfg.gamma
    next_vs = next_values
    for i in reversed(range(R)):
        r_i = rewards[i::R]
        nd_gamma = (1.0 - dones[i::R]) * cfg.gamma
        v_i = values[i::R]
        delta_s = rho[i::R] * (r_i + nd_gamma * next_values - v_i)
        adv[i::R] = rho[i::R] * (r_i + nd_gamma * next_vs - v_i)
        next_vs = v_i + delta_s + nd_gamma * c[i::R] * (next_vs - next_values)
        vs[i::R] = next_vs
        next_values = v_i
    return vs, adv


def calculate_losses(cfg: OracleCfg, params: Dict[str, Tensor], mb: Dict[str, Tensor], num_invalids: int):
    """learner.py:537-669 for the non-recurrent categorical model. `params` may require grad.
    Returns dict with policy_loss, exploration_loss, kl_loss, value_loss, loss, and the intermediates the
    parity tests name (ratio, adv (normalised), adv_mean, adv_std, values, targets, kl_old)."""
    clip_hi = 1.0 + cfg.ppo_clip_ratio  # :544
    clip_lo = 1.0 / clip_hi  # :546
    valids = mb["valids"]

    if not cfg.actor_critic_share_weights:
        head = None
    else:
        head = encoder_forward(cfg, params, mb["normalized_obs"])  # forward_head :553
    if head is None:
        core = None
    elif cfg.use_rnn:
        # :558-577 + rnn_utils.py:11-158.  The reference packs every run of steps between done-or-invalid boundaries
        # into a PackedSequence; a segment that starts inside a chunk starts from a ZERO state (rnn_utils.py:143-149,
        # is_new_episode), a segment at a chunk start from the stored rnn_state.  The same computation as a masked loop:
        R = cfg.recurrence
        n = head.shape[0] // R
        x = head.view(n, R, -1)
        doi = torch.logical_or(mb["dones"], ~valids).view(n, R).float()  # done_or_invalid :560
        state = mb["rnn_states"].view(n, R, -1)[:, 0]
        outs = []
        for t in range(R):
            if t > 0:
                state = state * (1.0 - doi[:, t - 1]).unsqueeze(-1)
            out, state = rnn_cell(cfg, params, x[:, t], state)
            outs.append(out)
        core = torch.stack(outs, 1).reshape(n * R, -1)
    else:
        core = head  # ModelCoreIdentity :579
    if core is None:
        values, logits = separate_forward(cfg, params, mb["normalized_obs"])
    else:
        values, logits = tail_forward(cfg, params, core)  # :586
    log_prob = dist_log_prob(cfg, logits, mb["actions"])  # :588
    ratio = torch.exp(log_prob - mb["log_prob_actions"])  # :589
    ratio = torch.clamp(ratio, 0.05, 20.0)  # :592

    with torch.no_grad():
        if cfg.with_vtrace:
            targets, adv = vtrace(
                cfg, ratio.detach(), values.detach(), mb["rewards"], mb["dones"].float(), cfg.recurrence
            )
        else:
            adv, targets = mb["advantages"], mb["returns"]  # :643-644
        adv_std, adv_mean = torch.std_mean(_masked_select(adv, valids, num_invalids))  # :646
        adv = (adv - adv_mean) / torch.clamp_min(adv_std, 1e-7)  # :647

    # _policy_loss :431-439
    pl = torch.min(ratio * adv, torch.clamp(ratio, clip_lo, clip_hi) * adv)
    policy_loss = -_masked_select(pl, valids, num_invalids).mean()
    # _entropy_exploration_loss :473-477
    if cfg.exploration_loss_coeff == 0.0:
        exploration_loss = torch.zeros(())
    elif cfg.exploration_loss == "symmetric_kl":   # _symmetric_kl_exploration_loss :479-486
        assert not cfg.continuous
        kl_prior = _masked_select(dist_symmetric_kl(cfg, logits), valids, num_invalids).mean()
        if not torch.isfinite(kl_prior):
            kl_prior = torch.zeros(kl_prior.shape)
        exploration_loss = cfg.exploration_loss_coeff * torch.clamp(kl_prior, max=30)
    else:
        ent = _masked_select(dist_entropy(cfg, logits), valids, num_invalids)
        exploration_loss = -cfg.exploration_loss_coeff * ent.mean()
    # _kl_loss :461-471 (only part of the loss if coeff != 0; kl_old is always computed for stats :758-768)
    kl_old = _masked_select(dist_kl(cfg, logits, mb["action_logits"]), valids, num_invalids)
    kl_loss = cfg.kl_loss_coeff * kl_old.mean() if cfg.kl_loss_coeff != 0.0 else torch.zeros(())
    # _value_loss :441-459
    old_values = mb["values"]
    v_clipped = old_values + torch.clamp(values - old_values, -cfg.ppo_clip_value, cfg.ppo_clip_value)
    vl = torch.max((values - targets).pow(2), (v_clipped - targets).pow(2))
    value_loss = _masked_select(vl, valids, num_invalids).mean() * cfg.value_loss_coeff

    loss = policy_loss + exploration_loss + kl_loss + value_loss  # :734-736
    return dict(
        loss=loss,
        policy_loss=policy_loss,
        exploration_loss=exploration_loss,
        kl_loss=kl_loss,
        value_loss=value_loss,
        ratio=ratio,
        adv=adv,
        adv_mean=adv_mean,
        adv_std=adv_std,
        values=values,
        targets=targets,
        kl_old=kl_old.detach(),
        logits=logits,
    )


# --------------------------------------------------------------------------------------
# Optimizer: clip_grad_norm_ + Adam exactly as torch 2.11 executes them (SURVEY App.A-12)
# --------------------------------------------------------------------------------------
def clip_grad_norm_(grads: List[Tensor], max_norm: float) -> Tensor:
    """torch/nn/utils/clip_grad.py: total = ||(||g_i||_2)_i||_2 ; coef = min(max_norm/(total+1e-6), 1)."""
    total = torch.linalg.vector_norm(torch.stack([torch.linalg.vector_norm(g, 2.0) for g in grads]), 2.0)
    coef = torch.clamp(max_norm / (total + 1e-6), max=1.0)
    for g in grads:
        g.mul_(coef)
    return total


def adam_step(p: Tensor, g: Tensor, m: Tensor, v: Tensor, step: int, lr: float, b1: float, b2: float, eps: float):
    """torch/optim/adam.py single-tensor path (no weight decay, no amsgrad)."""
    m.lerp_(g, 1 - b1)
    v.mul_(b2).addcmul_(g, g, value=1 - b2)
    bc1 = 1 - b1**step
    bc2 = 1 - b2**step
    step_size = lr / bc1
    denom = (v.sqrt() / math.sqrt(bc2)).add_(eps)
    p.addcdiv_(m, denom, value=-step_size)


LAMB_WEIGHT_DECAY, LAMB_MIN_TRUST = 1e-4, 0.01   # optimizers.py:22-23 defaults (the learner passes lr, betas, eps only)


def lamb_step(p: Tensor, g: Tensor, m: Tensor, v: Tensor, step: int, lr: float, b1: float, b2: float, eps: float):
    """algo/utils/optimizers.py:58-134 (list-params path, bias correction on, no look-ahead); `step` starts at 1."""
    m.mul_(b1).add_(g, alpha=(1 - b1))
    v.mul_(b2).addcmul_(g, g, value=(1 - b2))
    mh = m.clone().mul_(1 / (1 - b1**step))
    vh = v.sqrt().mul_(1 / math.sqrt(1 - b2**step))
    adam_step = mh.div_(vh.add_(eps))
    adam_step.add_(p, alpha=LAMB_WEIGHT_DECAY)
    weight_norm = torch.norm(p).item()
    step_norm = torch.norm(adam_step).item()
    if weight_norm == 0 or step_norm == 0:
        trust_ratio = 1
    else:
        trust_ratio = min(weight_norm, 10.0) / step_norm
        trust_ratio = min(max(trust_ratio, LAMB_MIN_TRUST), 1.0 / LAMB_MIN_TRUST)
    p.add_(adam_step, alpha=-lr * trust_ratio)


class OracleLearner:
    """State holder mirroring algo/learning/learner.py:125-255 for the path's numerics."""

    def __init__(self, cfg: OracleCfg, state: Dict[str, Tensor]):
        self.cfg = cfg
        self.st = {k: v.clone() for k, v in state.items()}
        self.names = param_names(cfg)
        self.m = {k: torch.zeros_like(self.st[k]) for k in self.names}
        self.v = {k: torch.zeros_like(self.st[k]) for k in self.names}
        self.opt_step = 0
        self.train_step = 0
        self.curr_lr = cfg.learning_rate
        self.env_steps = 0
        self.log: List[Dict[str, float]] = []

    def train(self, batch: Dict[str, Tensor], mb_indices=None) -> Dict[str, Tensor]:
        """learner.py:1036-1067 -> _prepare_batch -> _train (:671-841). Returns the prepared flat buffer.
        mb_indices (shuffle_minibatches, learner.py:498-526): a permutation of the flat sample indices built from
        recurrence-length chunks; minibatch b is buffer[mb_indices[b*B:(b+1)*B]] (`_get_minibatch` :528-535).  The reference
        draws a NEW permutation at the start of every epoch (`_get_minibatches` is called inside the epoch loop, :707-713):
        pass a sequence with one permutation per epoch (a single tensor is used for every epoch)."""
        cfg = self.cfg
        buff, experience_size, num_invalids = prepare_batch(cfg, self.st, batch, self.train_step)
        if num_invalids >= experience_size:
            return buff
        prev_epoch_actor_loss = 1e9
        for _epoch in range(cfg.num_epochs):
            nmb = cfg.num_batches_per_epoch
            epoch_actor_losses = []
            epoch_indices = mb_indices[_epoch] if isinstance(mb_indices, (list, tuple)) else mb_indices
            for b in range(nmb):
                if nmb == 1:
                    mb = buff
                elif epoch_indices is not None:
                    ind = epoch_indices[b * cfg.batch_size: (b + 1) * cfg.batch_size].long()   # :509-517
                    mb = {k: v[ind] for k, v in buff.items()}
                else:
                    sl = slice(b * cfg.batch_size, (b + 1) * cfg.batch_size)  # :521
                    mb = {k: v[sl] for k, v in buff.items()}
                params = {k: self.st[k].clone().requires_grad_(True) for k in self.names}
                out = calculate_losses(cfg, params, mb, num_invalids)
                out["loss"].backward()  # :779
                grads = [params[k].grad for k in self.names]
                gnorm = None
                if cfg.max_grad_norm > 0.0:  # :781-784
                    gnorm = clip_grad_norm_(grads, cfg.max_grad_norm)
                lr = self.curr_lr
                if num_invalids > 0:  # :788-794
                    lr = self.curr_lr * (experience_size - num_invalids) / experience_size
                self.opt_step += 1
                with torch.no_grad():
                    for k, g in zip(self.names, grads):
                        (lamb_step if cfg.optimizer == "lamb" else adam_step)(
                            self.st[k], g, self.m[k], self.v[k], self.opt_step, lr,
                            cfg.adam_beta1, cfg.adam_beta2, cfg.adam_eps,
                        )
                self.train_step += 1  # _after_optimizer_step :388-392
                actor_loss = out["policy_loss"] + out["exploration_loss"] + out["kl_loss"]
                epoch_actor_losses.append(float(actor_loss.detach()))
                self.log.append(
                    dict(
                        policy_loss=float(out["policy_loss"].detach()),
                        value_loss=float(out["value_loss"].detach()),
                        exploration_loss=float(out["exploration_loss"].detach()),
                        kl_loss=float(out["kl_loss"].detach()),
                        loss=float(out["loss"].detach()),
                        adv_mean=float(out["adv_mean"]),
                        adv_std=float(out["adv_std"]),
                        kl_old_mean=float(out["kl_old"].mean()),
                        grad_norm=float(gnorm) if gnorm is not None else float("nan"),
                        lr=lr,
                    )
                )
            new_loss = sum(epoch_actor_losses) / len(epoch_actor_losses)  # :827-839
            if abs(prev_epoch_actor_loss - new_loss) < 1e-6:
                break
            prev_epoch_actor_loss = new_loss
        self.env_steps += experience_size  # :1056-1059 (frameskip 1)
        return buff
