"""Environment boundary: registry (reference envs/env_utils.py:12-31, envs/create_env.py:13-46) and the two env contracts
the engine accepts.

1. The engine's batched GPU-env contract, which the device sampler drives directly (what the reference's BatchedVecEnv
   guarantees, make_env.py:147-237):

    env.num_agents : int
    env.obs_dim / env.num_actions
    env.reset() -> obs                       float32 [num_agents, obs_dim]
    env.step(actions) -> (obs, rew, terminated, truncated)
        actions    int32  [num_agents]   (device tensor when env_gpu_actions, else numpy; batched_sampling.py:62-82)
        obs        float32 [num_agents, obs_dim]
        rew        float32 [num_agents]; terminated / truncated bool [num_agents]
    auto-reset is the env's job (make_env.py:89-94).
    env.obs_keys (optional): a Dict observation of 1-D keys, [(key, d), ...] in sorted key order.  Each obs row is then the
        keys laid side by side as float32 (key k in columns [c_k, c_k + d_k), obs_dim = sum(d)), and the model builds one
        encoder per key (MultiInputEncoder).  An "action_mask" key is not part of the row.

2. The reference's gymnasium-API contracts, adapted by host_env.create_batched_env: a plain (single- or multi-agent) env
   is wrapped into host_env.BatchedHostEnv; a batched tensor env (IsaacGym / Brax style: one env with num_agents = N,
   reset() -> (obs, info), step(actions) -> (obs, rew, terminated, truncated, infos), torch tensors batched along dim 0 on
   the GPU or the CPU, obs a tensor or a dict of tensors described by observation_space) into
   host_env.BatchedTensorEnvAdapter, which converts each step's tensors into static buffers with one kernel.

`TapeVecEnv` is the synthetic env of BASELINE.json config 2 (Box(64) obs, Discrete(8)): GPU-resident, one CUDA kernel
per step, buffers reused across steps so a whole rollout can be captured in a CUDA graph.  `HostTapeVecEnv` is the
same env living in host memory (numpy + pinned buffers) -- the shape of a CPU-simulated env -- used for the
end-to-end (H2D/D2H inside the timed region) measurement.
"""
from __future__ import annotations

from typing import Callable, Dict, Optional, Tuple

import numpy as np
import torch
from torch import Tensor

from . import ops

_ENV_REGISTRY: Dict[str, Callable] = {}


def register_env(env_name: str, make_env_func: Callable) -> None:
    """Same contract as the reference: make_env_func(full_env_name, cfg, env_config, render_mode=None) -> env."""
    assert callable(make_env_func), f"{make_env_func=} must be callable"
    _ENV_REGISTRY[env_name] = make_env_func


def create_env(full_env_name: str, cfg=None, env_config=None, render_mode: Optional[str] = None):
    if full_env_name not in _ENV_REGISTRY:
        raise ValueError(f"Env name {full_env_name} is not registered. See register_env()!")
    return _ENV_REGISTRY[full_env_name](full_env_name, cfg, env_config, render_mode)


def global_env_registry() -> Dict[str, Callable]:
    return _ENV_REGISTRY


class TrainingInfoInterface:
    """envs/env_utils.py:117-129: envs that implement curricula receive the training progress at the end of every rollout
    (batched_sampling.py:351-354); `training_info` is guaranteed to contain 'approx_total_training_steps'."""

    def __init__(self):
        self.training_info: Dict[str, object] = dict()

    def set_training_info(self, training_info):
        self.training_info = training_info


class RewardShapingInterface:
    """envs/env_utils.py:74-90 (used by the reference's PBT to mutate reward shaping; the device runner only forwards a
    scheme the caller put into Runner.training_info['reward_shaping'])."""

    def get_default_reward_shaping(self):
        raise NotImplementedError

    def set_reward_shaping(self, reward_shaping, agent_idx) -> None:
        raise NotImplementedError


def set_training_info(env, training_info) -> None:
    """forward the training info (and an optional reward-shaping scheme) to an env that implements the interfaces"""
    if training_info is None:
        return
    shaping = training_info.get("reward_shaping") if isinstance(training_info, dict) else None
    if shaping is not None and hasattr(env, "set_reward_shaping"):
        env.set_reward_shaping(shaping, slice(0, env.num_agents))
    if hasattr(env, "set_training_info"):
        env.set_training_info(training_info)


class TapeVecEnv:
    """GPU-resident synthetic vector env.  obs_t = tape[t % L] (pre-generated N(0,1)-like tape in HBM),
    reward = action / num_actions, terminated / truncated = fixed integer rules of (step, env).
    Identical rules to oracle.appo_oracle.TapeVecEnv so CPU and GPU rollouts are comparable step by step."""

    is_gpu_env = True

    def __init__(self, tape: Tensor, num_actions: int, term_period: int = 37, trunc_period: int = 11,
                 env_index_offset: int = 0, continuous: bool = False, obs_shape=None, action_segments=None,
                 with_action_mask: bool = False, action_heads=None, obs_keys=None):
        assert tape.is_cuda and tape.dim() == 3 and tape.is_contiguous()
        # Dict observation layout over the tape row ([(key, d), ...], see the module docstring); the env rules are unchanged
        self.obs_keys = None if obs_keys is None else [(str(k), int(d)) for k, d in obs_keys]
        assert self.obs_keys is None or sum(d for _, d in self.obs_keys) == tape.shape[2]
        assert tape.dtype in (torch.float32, torch.uint8)
        self.tape = tape
        # image observations: uint8 tape rows of C*H*W bytes with obs_shape = (C, H, W) -> the model builds a ConvEncoder
        self.obs_uint8 = tape.dtype == torch.uint8
        self.obs_shape = None if obs_shape is None else tuple(obs_shape)
        assert self.obs_shape is None or int(np.prod(self.obs_shape)) == tape.shape[2]
        assert not self.obs_uint8 or tape.shape[2] % 16 == 0, "uint8 observation rows must be a multiple of 16 bytes"
        # continuous: Box(num_actions) action space, actions arrive as float32 [num_agents, num_actions] and
        # reward = clamp(actions[:, 0], -1, 1); otherwise Discrete(num_actions), int32 [num_agents]
        self.continuous = continuous
        # Tuple(Discrete(n_0), ...) action space: actions arrive as int32 [num_agents, K]; reward = actions[:, 0] / num_actions
        # with num_actions = sum(n_k) (same rule as the oracle's env)
        self.action_segments = None if action_segments is None else list(action_segments)
        # Tuple with Box members ([("discrete", n) | ("box", d), ...], num_actions = distribution_linear rows): actions
        # arrive as one tensor per member; the reward comes from member 0 by the rule of its kind
        self.action_heads = None if action_heads is None else [tuple(h) for h in action_heads]
        self.tape_len, self.num_agents, self.obs_dim = tape.shape
        self.num_actions = num_actions
        self.term_period, self.trunc_period = term_period, trunc_period
        self.env_index_offset = env_index_offset
        dev = tape.device
        # device-side so CUDA graphs can replay: [0] = env step, [1] = block ticket used to advance it in-kernel
        self.step_counter = torch.zeros(2, dtype=torch.int64, device=dev)
        self.obs = torch.empty((self.num_agents, self.obs_dim), dtype=tape.dtype, device=dev)
        self.rew = torch.empty(self.num_agents, dtype=torch.float32, device=dev)
        self.terminated = torch.empty(self.num_agents, dtype=torch.bool, device=dev)
        self.truncated = torch.empty(self.num_agents, dtype=torch.bool, device=dev)
        # the env kernel copies observation rows as 32-bit words: uint8 rows are handed over as float32 views
        self._tape_w = tape.view(torch.float32) if self.obs_uint8 else tape
        self._obs_w = self.obs.view(torch.float32) if self.obs_uint8 else self.obs
        self._a0 = torch.empty(self.num_agents, dtype=torch.int32, device=dev) if self.action_segments else None
        # with_action_mask: observations come as the reference's dict {"obs", "action_mask"}; the mask is the oracle env's
        # integer rule of (step, env, action), computed from the device-side step counter (graph-replay safe)
        self.with_action_mask = with_action_mask
        if with_action_mask:
            e = (torch.arange(self.num_agents, device=dev, dtype=torch.int64) + env_index_offset).view(-1, 1)
            a = torch.arange(num_actions, device=dev, dtype=torch.int64).view(1, -1)
            self._mask_e, self._mask_a, self._mask_ea = e, a, e * 5 + a * 7
            self.action_mask = torch.empty((self.num_agents, num_actions), dtype=torch.bool, device=dev)

    def _obs_out(self):
        if not self.with_action_mask:
            return self.obs
        t = self.step_counter[0]
        allowed = (((t * 3 + self._mask_ea) % 3) == 0) | (self._mask_a == (t + self._mask_e) % self.num_actions)
        torch.logical_and(allowed, ((t + self._mask_e) % 29) != 0, out=self.action_mask)
        return {"obs": self.obs, "action_mask": self.action_mask}

    def reset(self) -> Tensor:
        self.step_counter.zero_()
        self.obs.copy_(self.tape[0])
        return self._obs_out()

    def step(self, actions: Tensor) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
        if self.action_heads:
            a0 = actions[0]
            if self.action_heads[0][0] == "box":
                ops.tape_env_step_continuous(a0, self.env_index_offset, self.term_period, self.trunc_period,
                                             self.step_counter, 0, self._tape_w, self._obs_w, self.rew, self.terminated,
                                             self.truncated)
            else:
                ops.tape_env_step(a0, self.num_actions, self.env_index_offset, self.term_period, self.trunc_period,
                                  self.step_counter, 0, self._tape_w, self._obs_w, self.rew, self.terminated, self.truncated)
        elif self.continuous:
            ops.tape_env_step_continuous(actions, self.env_index_offset, self.term_period, self.trunc_period,
                                         self.step_counter, 0, self._tape_w, self._obs_w, self.rew, self.terminated,
                                         self.truncated)
        else:
            if self.action_segments:
                self._a0.copy_(actions[:, 0])      # first head's index (a strided gather; this env is test scaffolding)
                actions = self._a0
            ops.tape_env_step(actions, self.num_actions, self.env_index_offset, self.term_period, self.trunc_period,
                              self.step_counter, 0, self._tape_w, self._obs_w, self.rew, self.terminated, self.truncated)
        return self._obs_out(), self.rew, self.terminated, self.truncated


class HostTapeVecEnv:
    """The same env simulated on the HOST (numpy, pinned staging buffers): every step the sampler copies the
    observation batch host->device and the actions device->host, as it must for any CPU-simulated env."""

    is_gpu_env = False
    static_outputs = True   # step() always returns the same device tensors -> the sampler can graph-capture around it

    def __init__(self, tape: np.ndarray, num_actions: int, device: torch.device, term_period: int = 37,
                 trunc_period: int = 11, env_index_offset: int = 0):
        self.tape = torch.from_numpy(np.ascontiguousarray(tape, dtype=np.float32)).pin_memory()
        self.tape_len, self.num_agents, self.obs_dim = self.tape.shape
        self.num_actions = num_actions
        self.term_period, self.trunc_period = term_period, trunc_period
        self.device = device
        self.t = 0
        self.env_idx = np.arange(self.num_agents, dtype=np.int64) + env_index_offset
        self._res_term = ((self.env_idx * 13) % term_period).astype(np.int32)
        self._res_trunc = (self.env_idx % trunc_period).astype(np.int32)
        n = self.num_agents
        self.actions_host = torch.empty(n, dtype=torch.int32).pin_memory()
        # reward / terminated / truncated travel in ONE packed staging buffer (one H2D copy instead of three)
        self.pack_host = torch.empty(6 * n, dtype=torch.uint8).pin_memory()
        self.rew_host = self.pack_host[: 4 * n].view(torch.float32)
        self.term_host = self.pack_host[4 * n: 5 * n].view(torch.bool)
        self.trunc_host = self.pack_host[5 * n:].view(torch.bool)
        self.obs = torch.empty((n, self.obs_dim), dtype=torch.float32, device=device)
        self.pack = torch.empty(6 * n, dtype=torch.uint8, device=device)
        self.rew = self.pack[: 4 * n].view(torch.float32)
        self.terminated = self.pack[4 * n: 5 * n].view(torch.bool)
        self.truncated = self.pack[5 * n:].view(torch.bool)
        self.h2d_bytes = 0
        self.d2h_bytes = 0

    def reset(self) -> Tensor:
        self.t = 0
        self.obs.copy_(self.tape[0], non_blocking=True)
        self.h2d_bytes += self.obs.numel() * 4
        return self.obs

    def step(self, actions: Tensor) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
        self.step_async(actions)
        return self.step_wait()

    def enqueue_actions_d2h(self, actions: Tensor) -> None:
        """the D2H copy of the actions into the pinned staging buffer (static pointers: may be captured into a CUDA graph)"""
        self.actions_host.copy_(actions, non_blocking=True)

    def mark_actions_enqueued(self) -> None:
        if not hasattr(self, "_actions_ready"):
            self._actions_ready = torch.cuda.Event()
        self._actions_ready.record(torch.cuda.current_stream())

    def step_async(self, actions: Tensor) -> None:
        """first half of step(): enqueue the D2H copy of the actions (the sampler's double-buffered mode lets the GPU work
        on another env group while the host waits for this copy and simulates, rollout_worker.py:97-143)"""
        self.enqueue_actions_d2h(actions)
        self.mark_actions_enqueued()

    def step_wait(self) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
        # D2H: the actions the host simulator needs (synchronises -- a host env cannot start before it has them)
        self._actions_ready.synchronize()
        self.d2h_bytes += self.actions_host.numel() * 4
        a = self.actions_host.numpy()
        t = self.t
        np.divide(a, float(self.num_actions), out=self.rew_host.numpy(), casting="unsafe")
        # terminated / truncated rules of the tape env: (7 t + 13 i) % P == 0  <=>  (13 i) % P == (-7 t) % P, so one comparison of
        # a precomputed residue array against a scalar per rule (no integer divisions, no temporaries per step)
        term, trunc = self.term_host.numpy(), self.trunc_host.numpy()
        np.equal(self._res_term, (-7 * t) % self.term_period, out=term)
        np.equal(self._res_trunc, (-t) % self.trunc_period, out=trunc)
        np.greater(trunc, term, out=trunc)               # trunc & ~term
        self.t += 1
        # H2D: next observation batch + step results
        self.obs.copy_(self.tape[self.t % self.tape_len], non_blocking=True)
        self.pack.copy_(self.pack_host, non_blocking=True)
        self.h2d_bytes += self.obs.numel() * 4 + self.rew.numel() * 4 + 2 * self.num_agents
        return self.obs, self.rew, self.terminated, self.truncated
