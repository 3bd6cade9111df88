"""Adapter from ordinary (CPU, single-agent, gymnasium-API) environments to the batched contract the device sampler
drives -- the role of the reference's make_env_func_batched stack (algo/utils/make_env.py:89-237:
BatchedMultiAgentWrapper auto-reset, SequentialVectorizeWrapper :240-335, BatchedVecEnv tensor conversion) and of
preprocess_actions (batched_sampling.py:30-82).  This is what lets an sf_examples-style `make_env_func` that returns a
plain `gym.Env` (BASELINE.json config 1: CartPole-v1, 64 envs) run on the device engine unmodified:

    register_env("CartPole-v1", lambda name, cfg, env_config, render_mode=None:
                 BatchedHostEnv(lambda i: gym.make(name), num_envs=64, device=...))

Per step: actions D2H (one sync: a host simulator cannot start without them), a Python loop over the envs with
auto-reset, results staged in pinned buffers, one H2D copy of the observation batch and one of the packed
reward / terminated / truncated record.  The output tensors are static (the sampler captures its per-step kernels in
CUDA graphs around env.step).  Duck-typed on the gymnasium API (reset(seed=...) -> (obs, info);
step(a) -> (obs, reward, terminated, truncated, info)); gymnasium itself is not imported.

BatchedTensorEnvAdapter is the same role for batched tensor envs (IsaacGym / Brax style: ONE env with num_agents = N that
returns torch tensors batched along dim 0): no copies of the env, no per-agent loop, one ingest kernel per step.
create_batched_env picks the adapter from what the registered factory returns.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Tuple

import numpy as np
import torch
from torch import Tensor


def _space_info(space) -> Tuple[bool, int]:
    """(continuous, n) from a gymnasium-like action space: Discrete(n) -> (False, n); Box(shape=(A,)) -> (True, A)"""
    if hasattr(space, "n"):
        return False, int(space.n)
    shape = tuple(getattr(space, "shape", ()))
    if len(shape) != 1:
        raise NotImplementedError("Non-trivial shape Box action spaces not currently supported. Try to flatten the space.")
    return True, int(shape[0])


def _tuple_members(space) -> Optional[List[Tuple[str, int]]]:
    """[("discrete", n) | ("box", d), ...] of a gymnasium-like Tuple action space, None for any other space"""
    members = getattr(space, "spaces", None)
    if not isinstance(members, (tuple, list)):
        return None
    out = []
    for m in members:
        continuous, n = _space_info(m)
        out.append(("box" if continuous else "discrete", n))
    return out


def _main_obs_space(obs_space):
    """(space of the policy input, key or None, obs_keys or None).  Dict observation spaces (make_env.py:147-176 wraps
    everything into Dict(obs=...)): an "action_mask" entry is consumed by the sampler (actor_critic.py:345-351).  The key
    "obs" alone keeps its space (any shape); other keys must be 1-D and are packed side by side in sorted key order
    (MultiInputEncoder's order, encoder.py:36), one encoder per key: obs_keys = [(key, d), ...]."""
    spaces = getattr(obs_space, "spaces", None)
    if not isinstance(spaces, dict):
        return obs_space, None, None
    keys = sorted(k for k in spaces if k != "action_mask")
    if not keys:
        raise NotImplementedError("Dict observation space without a policy input (only 'action_mask')")
    if keys == ["obs"]:
        return spaces["obs"], "obs", None
    obs_keys = []
    for k in keys:
        shape = tuple(getattr(spaces[k], "shape", None) or ())
        if len(shape) == 0:
            raise NotImplementedError(f"Dict observation key {k!r} is a scalar space {spaces[k]}: MultiInputEncoder "
                                      "supports 1-D (vector) keys here (the reference raises for scalar keys too)")
        if len(shape) > 1:
            raise NotImplementedError(f"Dict observation key {k!r} has shape {shape}: the device path supports Dict "
                                      "observations of 1-D keys only (image keys in a Dict are not supported yet)")
        obs_keys.append((k, int(shape[0])))
    return None, None, obs_keys


def _parse_spaces(env, observation_space, action_space) -> None:
    """The attributes of the engine's env contract that follow from the spaces (obs_dim, obs_keys, obs_shape / obs_uint8,
    continuous, num_actions, action_segments, action_heads) and the adapter's _obs_key / _mask_key / _key_cols, set on
    `env` -- one rule for BatchedHostEnv and BatchedTensorEnvAdapter."""
    obs_space, env._obs_key, env.obs_keys = _main_obs_space(observation_space)
    is_dict = isinstance(getattr(observation_space, "spaces", None), dict)
    env._mask_key = "action_mask" if (is_dict and "action_mask" in observation_space.spaces) else None
    if env.obs_keys is not None:
        # Dict of 1-D keys: every key's array is cast to float32 (normalize.py:43-45) into its columns of the packed row
        env.obs_uint8, env.obs_shape = False, None
        env.obs_dim = sum(d for _, d in env.obs_keys)
        env._key_cols = []
        c = 0
        for _, d in env.obs_keys:
            env._key_cols.append(slice(c, c + d))
            c += d
    else:
        shape = tuple(obs_space.shape)
        env.obs_uint8 = np.dtype(getattr(obs_space, "dtype", np.float32)) == np.uint8
        env.obs_shape = shape if len(shape) == 3 else None       # (C, H, W) image observations -> ConvEncoder
        env.obs_dim = int(np.prod(shape))
    # Tuple action spaces (preprocess_actions, batched_sampling.py:46-57): all-Discrete -> action_segments (the sampler
    # hands over int32 [n, K]); with Box members -> action_heads (one device tensor per member) and num_actions = the
    # rows of distribution_linear.  An env receives a Python tuple per step (Tuple.sample()'s layout), a multi-agent env
    # the list of per-member batches of its agents.
    members = _tuple_members(action_space)
    env.action_segments = env.action_heads = None
    if members is None:
        env.continuous, env.num_actions = _space_info(action_space)
    else:
        env.continuous = False
        if all(k == "discrete" for k, _ in members):
            env.action_segments = [n for _, n in members]
            env.num_actions = sum(env.action_segments)
        else:
            env.action_heads = members
            env.num_actions = sum(n if k == "discrete" else 2 * n for k, n in members)


def _pinned_actions(env, n: int):
    """pinned host staging for the sampler's env_actions (preprocess_actions, batched_sampling.py:30-82): int32 [n]
    (Discrete), float32 [n, A] (Box), int32 [n, K] (all-Discrete Tuple), or one buffer per member (Tuple with Box members)"""
    if env.action_heads:
        return [torch.empty(n, dtype=torch.int32).pin_memory() if k == "discrete" else
                torch.empty((n, d), dtype=torch.float32).pin_memory() for k, d in env.action_heads]
    if env.continuous:
        adt, ashape = torch.float32, (n, env.num_actions)
    else:
        adt, ashape = torch.int32, ((n, len(env.action_segments)) if env.action_segments else (n,))
    return torch.empty(ashape, dtype=adt).pin_memory()


class BatchedHostEnv:
    is_gpu_env = False
    static_outputs = True

    def __init__(self, make_env: Callable[[int], object], num_envs: int, device: torch.device, seed: Optional[int] = None,
                 first_reset=None):
        self.envs: List = [make_env(i) for i in range(num_envs)]
        # (obs, info) of env 0's first (seeded) reset when create_batched_env already made it to inspect the observation
        self._first_reset = first_reset
        e0 = self.envs[0]
        # Multi-agent envs (envs/env_utils.py "is_multiagent": lists of per-agent observations / rewards / dones in and out,
        # the env resets itself -- sf_examples/train_custom_multi_env.py): agent j of env i is row i * A + j.  An agent can
        # report info["is_active"] = False: its next step is recorded with policy id -1 and masked by the learner
        # (non_batched_sampling.py:82-84,197-203).
        self.agents_per_env = int(getattr(e0, "num_agents", 1))
        self.multi_agent = bool(getattr(e0, "is_multiagent", False)) or self.agents_per_env > 1
        self.num_agents = num_envs * self.agents_per_env
        self.device = device
        _parse_spaces(self, e0.observation_space, e0.action_space)
        self._seed = seed
        self._seeded = False
        n = self.num_agents
        self.inactive = None        # device bool [num_agents]: rows whose agent was inactive when the last step was taken
        if self.multi_agent:
            self.inactive_next = torch.zeros(n, dtype=torch.bool).pin_memory()
            self.inactive_host = torch.zeros(n, dtype=torch.bool).pin_memory()
            self.inactive = torch.zeros(n, dtype=torch.bool, device=device)
        odt = torch.uint8 if self.obs_uint8 else torch.float32
        self.obs_host = torch.empty((n, self.obs_dim), dtype=odt).pin_memory()
        self.obs = torch.empty((n, self.obs_dim), dtype=odt, device=device)
        self.actions_host = _pinned_actions(self, n)
        # reward / terminated / truncated travel in ONE packed staging buffer (one H2D copy instead of three)
        self.pack_host = torch.empty(6 * n, dtype=torch.uint8).pin_memory()
        self.rew_host = self.pack_host[: 4 * n].view(torch.float32)
        self.term_host = self.pack_host[4 * n: 5 * n].view(torch.bool)
        self.trunc_host = self.pack_host[5 * n:].view(torch.bool)
        self.pack = torch.empty(6 * n, dtype=torch.uint8, device=device)
        self.rew = self.pack[: 4 * n].view(torch.float32)
        self.terminated = self.pack[4 * n: 5 * n].view(torch.bool)
        self.truncated = self.pack[5 * n:].view(torch.bool)
        self.h2d_bytes = 0
        self.d2h_bytes = 0
        self.episode_infos: List[dict] = []   # infos of finished episodes since the last pop (batched_sampling.py:228-270)
        if self._mask_key:
            self.mask_host = torch.ones((n, self.num_actions), dtype=torch.bool).pin_memory()
            self.action_mask = torch.ones((n, self.num_actions), dtype=torch.bool, device=device)

    def _put_obs(self, i: int, obs) -> None:
        if self._mask_key:
            self.mask_host[i].copy_(torch.as_tensor(np.asarray(obs[self._mask_key])).reshape(-1) != 0)
        if self.obs_keys is not None:
            row = self.obs_host[i].numpy()
            for (k, _), cols in zip(self.obs_keys, self._key_cols):
                row[cols] = np.asarray(obs[k]).reshape(-1)
            return
        if self._obs_key is not None:
            obs = obs[self._obs_key]
        self.obs_host[i].copy_(torch.as_tensor(np.asarray(obs)).reshape(-1))

    def _obs_out(self):
        if not self._mask_key:
            return self.obs
        self.action_mask.copy_(self.mask_host, non_blocking=True)
        return {"obs": self.obs, "action_mask": self.action_mask}

    def reset(self) -> Tensor:
        for i, e in enumerate(self.envs):
            kw = {}
            if self._seed is not None and not self._seeded:
                kw["seed"] = self._seed + i        # per-env seed = global env id (batched_sampling.py:177)
            if i == 0 and self._first_reset is not None:
                obs, _info = self._first_reset
                self._first_reset = None
            else:
                obs, _info = e.reset(**kw)
            if self.multi_agent:
                for j in range(self.agents_per_env):
                    self._put_obs(i * self.agents_per_env + j, obs[j])
            else:
                self._put_obs(i, obs)
        self._seeded = True
        self.obs.copy_(self.obs_host, non_blocking=True)
        self.h2d_bytes += self.obs_host.numel() * self.obs_host.element_size()
        return self._obs_out()

    def step(self, actions: Tensor) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
        self.step_async(actions)
        return self.step_wait()

    def enqueue_actions_d2h(self, actions: Tensor) -> None:
        """the D2H copy of the actions into the pinned staging buffer (static pointers: may be captured into a CUDA graph);
        a Tuple with Box members copies each member's tensor into its own staging buffer"""
        if self.action_heads:
            for h, d in zip(self.actions_host, actions):
                h.copy_(d, non_blocking=True)
        else:
            self.actions_host.copy_(actions, non_blocking=True)

    def mark_actions_enqueued(self) -> None:
        if not hasattr(self, "_actions_ready"):
            self._actions_ready = torch.cuda.Event()
        self._actions_ready.record(torch.cuda.current_stream())

    def step_async(self, actions: Tensor) -> None:
        """first half of step(): enqueue the D2H copy of the actions (double-buffered sampling: the GPU serves another env
        group while the host waits for this copy and steps these envs, rollout_worker.py:97-143)"""
        self.enqueue_actions_d2h(actions)
        self.mark_actions_enqueued()

    def step_wait(self) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
        self._actions_ready.synchronize()
        staged = self.actions_host if self.action_heads else [self.actions_host]
        self.d2h_bytes += sum(h.numel() * h.element_size() for h in staged)
        a = [h.numpy() for h in staged] if self.action_heads else self.actions_host.numpy()
        rew, term, trunc = self.rew_host.numpy(), self.term_host.numpy(), self.trunc_host.numpy()
        if self.multi_agent:
            return self._step_multi_agent(a, rew, term, trunc)
        for i, e in enumerate(self.envs):
            obs, r, tm, tr, info = e.step(self._env_action(a, i))
            rew[i], term[i], trunc[i] = r, bool(tm), bool(tr)
            if tm or tr:                             # BatchedMultiAgentWrapper auto-reset (make_env.py:89-94)
                if info:
                    self.episode_infos.append(info)
                obs, _ = e.reset()
            self._put_obs(i, obs)
        self.obs.copy_(self.obs_host, non_blocking=True)
        self.pack.copy_(self.pack_host, non_blocking=True)
        self.h2d_bytes += self.obs_host.numel() * self.obs_host.element_size() + self.pack_host.numel()
        return self._obs_out(), self.rew, self.terminated, self.truncated

    def _env_action(self, a, row: int):
        """the action of one single-agent env: an int (Discrete), a float32 row (Box), or a tuple with a numpy integer per
        Discrete member and a float32 ndarray[d] per Box member (Tuple)"""
        if self.action_heads:
            return tuple(m[row] if k == "discrete" else m[row].copy() for m, (k, _) in zip(a, self.action_heads))
        if self.action_segments:
            return tuple(a[row])
        return a[row] if self.continuous else int(a[row])

    def _step_multi_agent(self, a, rew, term, trunc):
        A = self.agents_per_env
        self.inactive_host.copy_(self.inactive_next)          # the status the agents had when these actions were computed
        nxt = self.inactive_next.numpy()
        for i, e in enumerate(self.envs):
            rows = slice(i * A, (i + 1) * A)
            if self.action_heads:           # per member: int32 [A] / float32 [A, d] (preprocess_actions)
                acts = [m[rows].copy() for m in a]
            elif self.action_segments:
                acts = [a[rows, k].copy() for k in range(len(self.action_segments))]
            else:
                acts = [a[i * A + j] if self.continuous else int(a[i * A + j]) for j in range(A)]
            obs, r, tm, tr, infos = e.step(acts)               # (multi-agent envs auto-reset themselves)
            for j in range(A):
                row = i * A + j
                rew[row], term[row], trunc[row] = r[j], bool(tm[j]), bool(tr[j])
                info = infos[j] if infos else {}
                nxt[row] = not info.get("is_active", True)
                if (tm[j] or tr[j]) and info:
                    self.episode_infos.append(info)
                self._put_obs(row, obs[j])
        self.obs.copy_(self.obs_host, non_blocking=True)
        self.pack.copy_(self.pack_host, non_blocking=True)
        self.inactive.copy_(self.inactive_host, non_blocking=True)
        self.h2d_bytes += self.obs_host.numel() * self.obs_host.element_size() + self.pack_host.numel() + self.num_agents
        return self._obs_out(), self.rew, self.terminated, self.truncated

    def set_reward_shaping(self, reward_shaping, agent_idx=None) -> None:
        """RewardShapingInterface pass-through (PBT mutates the scheme, envs/env_utils.py:74-90)"""
        for e in self.envs:
            if hasattr(e, "set_reward_shaping"):
                e.set_reward_shaping(reward_shaping, slice(0, self.agents_per_env))

    def get_default_reward_shaping(self):
        e0 = self.envs[0]
        return e0.get_default_reward_shaping() if hasattr(e0, "get_default_reward_shaping") else None

    def set_training_info(self, training_info) -> None:
        for e in self.envs:
            if hasattr(e, "set_training_info"):
                e.set_training_info(training_info)

    def close(self) -> None:
        for e in self.envs:
            if hasattr(e, "close"):
                e.close()


class BatchedTensorEnvAdapter:
    """A batched tensor env (IsaacGym / Brax style: sf_examples/isaacgym_examples/train_isaacgym.py,
    sf_examples/brax/train_brax.py) behind the engine's env contract (envs.py).  The env is ONE object with num_agents = N
    (make_env.py:36-45); reset() -> (obs, info) and step(actions) -> (obs, rew, terminated, truncated, infos) return torch
    tensors batched along dim 0 -- obs a tensor or a dict of tensors -- on the GPU or the CPU, in the env's own dtypes
    (BatchedVecEnv hands them through unchanged, make_env.py:147-237).

    - Outputs: every reset() / step() result is converted by ONE sfb200_env_ingest launch into static device buffers: obs
      (float32 [N, obs_dim], the keys of a Dict side by side; uint8 for one uint8 image key), rew (float32),
      terminated / truncated (x != 0) and the action mask.  Each key's per-agent elements must be dense, any row stride
      is allowed.  CPU tensors travel by one pinned H2D copy each first.  A bare tensor counts as {"obs": tensor}; keys
      that are not in observation_space (IsaacGym's "states") are ignored.
    - Actions: the sampler's env_actions (preprocess_actions, batched_sampling.py:30-82).  With env_gpu_actions they are
      handed over as device tensors (no host synchronisation); otherwise they come by one pinned D2H copy as numpy.
    - Streams: reset() / step() run on the current CUDA stream (the sampler's: an env group of SplitSampler keeps its own).
    - infos are ignored: episode statistics come from the sampler's device-side accounting, as for device envs.

    static_outputs: the sampler captures its launches on either side of step() into CUDA graphs.  The env's step() is user
    code that may synchronise or allocate, so it is never captured (is_gpu_env = False)."""

    is_gpu_env = False
    static_outputs = True

    def __init__(self, env, device: torch.device, env_gpu_actions: bool = False, seed: Optional[int] = None,
                 first_reset=None):
        from . import ops

        self.env = env
        self.device = device
        self.env_gpu_actions = bool(env_gpu_actions)
        self.num_agents = n = int(env.num_agents)
        _parse_spaces(self, env.observation_space, env.action_space)
        keys = [k for k, _ in self.obs_keys] if self.obs_keys is not None else [self._obs_key or "obs"]
        if len(keys) + 4 > ops.INGEST_MAX:
            raise NotImplementedError(f"{len(keys)} observation keys: the ingest launch takes at most "
                                      f"{ops.INGEST_MAX - 4} keys beside reward, terminated, truncated and the mask")
        self.obs = torch.empty((n, self.obs_dim), dtype=torch.uint8 if self.obs_uint8 else torch.float32, device=device)
        self.rew = torch.zeros(n, dtype=torch.float32, device=device)
        self.terminated = torch.zeros(n, dtype=torch.bool, device=device)
        self.truncated = torch.zeros(n, dtype=torch.bool, device=device)
        self.action_mask = torch.ones((n, self.num_actions), dtype=torch.bool, device=device) if self._mask_key else None
        # obs destinations: (key, columns, first column, kind)
        if self.obs_keys is not None:
            self._obs_dst = [(k, d, cols.start, ops.INGEST_F32) for (k, d), cols in zip(self.obs_keys, self._key_cols)]
        else:
            self._obs_dst = [(keys[0], self.obs_dim, 0, ops.INGEST_U8 if self.obs_uint8 else ops.INGEST_F32)]
        self.actions_host = None if self.env_gpu_actions else _pinned_actions(self, n)
        self._actions_ready = None
        self._seed = seed
        self._first_reset = first_reset      # (obs, info) of the seeded reset create_batched_env made to detect the env
        self._seeded = first_reset is not None

    def _src(self, t, name: str, cols: int):
        """(device tensor, row stride, cols) of one returned tensor; refuses what the ingest kernel cannot read"""
        from . import ops

        if not isinstance(t, torch.Tensor):
            raise TypeError(f"batched tensor env: {name!r} is a {type(t).__name__}, expected a torch tensor")
        if t.dim() == 0 or t.shape[0] != self.num_agents or t.numel() != self.num_agents * cols:
            raise ValueError(f"batched tensor env: {name!r} has shape {tuple(t.shape)}, expected {self.num_agents} rows "
                             f"of {cols} elements")
        if t.dtype not in ops.INGEST_DTYPES:
            raise TypeError(f"batched tensor env: {name!r} has dtype {t.dtype}")
        expected = 1
        for size, stride in zip(reversed(t.shape[1:]), reversed(t.stride()[1:])):
            if size != 1 and stride != expected:
                raise ValueError(f"batched tensor env: the per-agent elements of {name!r} are not dense (shape "
                                 f"{tuple(t.shape)}, strides {t.stride()}); any row stride is allowed")
            expected *= size
        if not t.is_cuda:
            t = (t if t.is_pinned() else t.pin_memory()).to(self.device, non_blocking=True)
        return t, t.stride(0), cols

    def _ingest(self, obs, rew=None, terminated=None, truncated=None) -> None:
        from . import ops

        if not isinstance(obs, dict):
            obs = {"obs": obs}
        entries = []
        for k, cols, c0, kind in self._obs_dst:
            if k not in obs:
                raise KeyError(f"batched tensor env: observation key {k!r} of observation_space was not returned")
            src = self._src(obs[k], k, cols)
            if kind == ops.INGEST_U8 and src[0].dtype != torch.uint8:
                raise TypeError(f"batched tensor env: {k!r} is a uint8 image space but the env returned {src[0].dtype}")
            entries.append((*src, self.obs, c0, kind))
        if self._mask_key:
            entries.append((*self._src(obs[self._mask_key], self._mask_key, self.num_actions), self.action_mask, 0,
                            ops.INGEST_BOOL))
        if rew is not None:
            entries += [(*self._src(rew, "reward", 1), self.rew.view(-1, 1), 0, ops.INGEST_F32),
                        (*self._src(terminated, "terminated", 1), self.terminated.view(-1, 1), 0, ops.INGEST_BOOL),
                        (*self._src(truncated, "truncated", 1), self.truncated.view(-1, 1), 0, ops.INGEST_BOOL)]
        ops.env_ingest(entries, self.num_agents)

    def _obs_out(self):
        if self.action_mask is None:
            return self.obs
        return {"obs": self.obs, "action_mask": self.action_mask}

    def reset(self):
        if self._first_reset is not None:
            obs, _info = self._first_reset
            self._first_reset = None
        else:
            kw = {} if (self._seed is None or self._seeded) else {"seed": self._seed}
            obs, _info = self.env.reset(**kw)
            self._seeded = True
        self._ingest(obs)
        return self._obs_out()

    def _env_actions(self, actions):
        if self.env_gpu_actions:
            return list(actions) if self.action_heads else actions
        if self.action_heads:
            for h, d in zip(self.actions_host, actions):
                h.copy_(d, non_blocking=True)
        else:
            self.actions_host.copy_(actions, non_blocking=True)
        if self._actions_ready is None:
            self._actions_ready = torch.cuda.Event()
        self._actions_ready.record(torch.cuda.current_stream())
        self._actions_ready.synchronize()
        return [h.numpy() for h in self.actions_host] if self.action_heads else self.actions_host.numpy()

    def step(self, actions):
        obs, rew, terminated, truncated, _infos = self.env.step(self._env_actions(actions))
        self._ingest(obs, rew, terminated, truncated)
        return self._obs_out(), self.rew, self.terminated, self.truncated

    def set_reward_shaping(self, reward_shaping, agent_idx=None) -> None:
        if hasattr(self.env, "set_reward_shaping"):
            self.env.set_reward_shaping(reward_shaping, agent_idx)

    def get_default_reward_shaping(self):
        return self.env.get_default_reward_shaping() if hasattr(self.env, "get_default_reward_shaping") else None

    def set_training_info(self, training_info) -> None:
        if hasattr(self.env, "set_training_info"):
            self.env.set_training_info(training_info)

    def close(self) -> None:
        if hasattr(self.env, "close"):
            self.env.close()


def is_batched_env(env) -> bool:
    """Does `env` already speak the batched device contract of sample_factory_b200.envs (TapeVecEnv, BatchedHostEnv, user
    GPU envs)?  Anything else is treated as an ordinary gymnasium-API env."""
    return hasattr(env, "is_gpu_env") and hasattr(env, "num_agents") and hasattr(env, "obs_dim")


def _is_tensor_batch(obs, n: int) -> bool:
    """a torch tensor, or a non-empty dict of torch tensors, with leading dim n"""
    values = list(obs.values()) if isinstance(obs, dict) else [obs]
    return bool(values) and all(isinstance(v, torch.Tensor) and v.dim() > 0 and v.shape[0] == n for v in values)


def create_batched_env(cfg, env_config: dict, device: torch.device, num_envs: Optional[int] = None):
    """The reference's make_env_func_batched (algo/utils/make_env.py:338-351) for this engine: create the registered env and
    - return it as is if it speaks the engine's batched contract (envs.py);
    - if it is a multi-agent env (make_env.py:36-45) whose first reset() observation is a torch tensor or a dict of torch
      tensors with leading dim num_agents (a batched tensor env, IsaacGym / Brax style), wrap that ONE env into a
      BatchedTensorEnvAdapter;
    - otherwise (a plain gymnasium-API env: what every sf_examples `make_env_func` returns, or a multi-agent env returning
      lists / numpy) wrap num_workers * num_envs_per_worker instances of it -- each created through the SAME registered
      factory with the reference's env_config (worker_index, vector_index, env_id; batched_sampling.py:166-174) -- into a
      BatchedHostEnv: BatchedMultiAgentWrapper auto-reset, dict-observation unwrapping and tensor conversion happen there.
    The reset that tells a batched tensor env apart is the first (seeded) reset BatchedHostEnv would make of env 0; its
    result is handed over, so no env is reset more often than before."""
    from .envs import create_env

    first = create_env(cfg.env, cfg, env_config)
    if is_batched_env(first):
        return first
    if not (hasattr(first, "observation_space") and hasattr(first, "action_space")):
        raise TypeError(f"{type(first).__name__} is neither a batched device env nor a gymnasium-API env")
    epw = int(cfg.num_envs_per_worker)
    if num_envs is not None and num_envs < 1:
        raise ValueError(f"total_envs={int(cfg.num_workers) * epw} must be divisible by the number of policies")
    n = int(num_envs) if num_envs is not None else int(cfg.num_workers) * epw
    w0 = int(env_config.get("worker_index", 0)) if env_config else 0
    seed = None if getattr(cfg, "seed", None) is None else int(cfg.seed) + w0 * n
    agents = int(getattr(first, "num_agents", 1))
    first_reset = None
    if bool(getattr(first, "is_multiagent", False)) or agents > 1:
        first_reset = first.reset(**({} if seed is None else {"seed": seed}))
        if _is_tensor_batch(first_reset[0], agents):
            policies = int((env_config or {}).get("num_policies", getattr(cfg, "num_policies", 1)))
            if policies > 1:
                raise ValueError(f"num_policies={policies} with the batched tensor env {type(first).__name__}: a batched "
                                 "env belongs to one policy (batched_sampling.py:130); splitting its rows across policies "
                                 "is not supported")
            return BatchedTensorEnvAdapter(first, device, env_gpu_actions=bool(getattr(cfg, "env_gpu_actions", False)),
                                           seed=seed, first_reset=first_reset)
    made = {0: first}

    def make(i: int):
        if i in made:
            return made.pop(i)
        ec = dict(worker_index=w0 * int(cfg.num_workers) + i // epw, vector_index=i % epw, env_id=w0 * n + i)
        return create_env(cfg.env, cfg, ec)

    return BatchedHostEnv(make, n, device, seed=seed, first_reset=first_reset)
