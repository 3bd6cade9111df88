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


class BatchedHostEnv:
    is_gpu_env = False
    static_outputs = True

    def __init__(self, make_env: Callable[[int], object], num_envs: int, device: torch.device, seed: Optional[int] = None):
        self.envs: List = [make_env(i) for i in range(num_envs)]
        e0 = self.envs[0]
        # Multi-agent envs (envs/env_utils.py "is_multiagent": lists of per-agent observations / rewards / dones in and out,
        # the env resets itself -- sf_examples/train_custom_multi_env.py): agent j of env i is row i * A + j.  An agent can
        # report info["is_active"] = False: its next step is recorded with policy id -1 and masked by the learner
        # (non_batched_sampling.py:82-84,197-203).
        self.agents_per_env = int(getattr(e0, "num_agents", 1))
        self.multi_agent = bool(getattr(e0, "is_multiagent", False)) or self.agents_per_env > 1
        self.num_agents = num_envs * self.agents_per_env
        self.device = device
        obs_space, self._obs_key, self.obs_keys = _main_obs_space(e0.observation_space)
        is_dict = isinstance(getattr(e0.observation_space, "spaces", None), dict)
        self._mask_key = "action_mask" if (is_dict and "action_mask" in e0.observation_space.spaces) else None
        if self.obs_keys is not None:
            # Dict of 1-D keys: every key's array is cast to float32 (normalize.py:43-45) into its columns of the packed row
            self.obs_uint8, self.obs_shape = False, None
            self.obs_dim = sum(d for _, d in self.obs_keys)
            self._key_cols = []
            c = 0
            for _, d in self.obs_keys:
                self._key_cols.append(slice(c, c + d))
                c += d
        else:
            shape = tuple(obs_space.shape)
            self.obs_uint8 = np.dtype(getattr(obs_space, "dtype", np.float32)) == np.uint8
            self.obs_shape = shape if len(shape) == 3 else None       # (C, H, W) image observations -> ConvEncoder
            self.obs_dim = int(np.prod(shape))
        # Tuple action spaces (preprocess_actions, batched_sampling.py:46-57): all-Discrete -> action_segments (the sampler
        # hands over int32 [n, K]); with Box members -> action_heads (one device tensor per member) and num_actions = the
        # rows of distribution_linear.  An env receives a Python tuple per step (Tuple.sample()'s layout), a multi-agent env
        # the list of per-member batches of its agents.
        members = _tuple_members(e0.action_space)
        self.action_segments = self.action_heads = None
        if members is None:
            self.continuous, self.num_actions = _space_info(e0.action_space)
        else:
            self.continuous = False
            if all(k == "discrete" for k, _ in members):
                self.action_segments = [n for _, n in members]
                self.num_actions = sum(self.action_segments)
            else:
                self.action_heads = members
                self.num_actions = sum(n if k == "discrete" else 2 * n for k, n in members)
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
        if self.action_heads:
            self.actions_host = [torch.empty(n, dtype=torch.int32).pin_memory() if k == "discrete" else
                                 torch.empty((n, d), dtype=torch.float32).pin_memory() for k, d in self.action_heads]
        else:
            if self.continuous:
                adt, ashape = torch.float32, (n, self.num_actions)
            else:
                adt, ashape = torch.int32, ((n, len(self.action_segments)) if self.action_segments else (n,))
            self.actions_host = torch.empty(ashape, dtype=adt).pin_memory()
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


def is_batched_env(env) -> bool:
    """Does `env` already speak the batched device contract of sample_factory_b200.envs (TapeVecEnv, BatchedHostEnv, user
    GPU envs)?  Anything else is treated as an ordinary gymnasium-API env."""
    return hasattr(env, "is_gpu_env") and hasattr(env, "num_agents") and hasattr(env, "obs_dim")


def create_batched_env(cfg, env_config: dict, device: torch.device, num_envs: Optional[int] = None):
    """The reference's make_env_func_batched (algo/utils/make_env.py:338-351) for this engine: create the registered env and,
    if the factory returned a plain single-agent gymnasium-API env (what every sf_examples `make_env_func` returns), wrap
    num_workers * num_envs_per_worker instances of it -- each created through the SAME registered factory with the
    reference's env_config (worker_index, vector_index, env_id; batched_sampling.py:166-174) -- into a BatchedHostEnv:
    BatchedMultiAgentWrapper auto-reset, dict-observation unwrapping and tensor conversion happen there."""
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
    made = {0: first}

    def make(i: int):
        if i in made:
            return made.pop(i)
        ec = dict(worker_index=w0 * int(cfg.num_workers) + i // epw, vector_index=i % epw, env_id=w0 * n + i)
        return create_env(cfg.env, cfg, ec)

    seed = None if getattr(cfg, "seed", None) is None else int(cfg.seed) + w0 * n
    return BatchedHostEnv(make, n, device, seed=seed)
