"""Sampler-only APIs over the device trajectory store (SURVEY 8f row 1): the reference's `SyncSamplingAPI`
(algo/sampling/sync_sampling_api.py:16-65), `EvalSamplingAPI` (algo/sampling/evaluation_sampling_api.py:234-315) and the
`eval.py` driver (eval.py:83-124), same method names and meaning.

The reference runs a `SamplingLoop` event loop on a thread that owns rollout / inference workers and hands trajectory
slices to a callback.  Here the sampler is one object on one CUDA stream, so the loop is a plain call: every
`get_trajectories_sync()` runs one rollout on the device and returns a *clone* of the trajectory record (the reference
also clones before releasing the buffers, sync_sampling_api.py:37); `EvalSamplingAPI` pumps rollouts while its
statistics are being polled, which is what the reference's background thread does between polls.
"""
from __future__ import annotations

import json
import os
import time
from dataclasses import dataclass
from typing import Dict, List, Optional

import torch
from torch import Tensor

from . import ops
from .checkpoint import load_checkpoint
from .cfg import preprocess_cfg
from .host_env import create_batched_env
from .model import ModelSpec, PolicyModel
from .sampler import DeviceSampler
from .trajectory import alloc_for_spec


class StatusCode:
    SUCCESS, FAILURE, INTERRUPTED = 0, 1, 2


@dataclass
class EnvInfo:
    """algo/utils/env_info.py:18-41 (the fields this path reads)."""
    obs_dim: int
    num_actions: int
    num_agents: int


def obtain_env_info(cfg) -> EnvInfo:
    """env_info.py:79-103 (in-process: creating a device env is cheap, no subprocess needed)."""
    env = create_batched_env(cfg, dict(worker_index=0, vector_index=0, env_id=0), torch.device("cuda", torch.cuda.current_device()))
    info = EnvInfo(env.obs_dim, env.num_actions, env.num_agents)
    if hasattr(env, "close"):
        env.close()
    return info


def samples_per_trajectory(traj: Dict[str, Tensor]) -> int:
    """algo/utils/rl_utils.py:115-117"""
    shape = traj["rewards"].shape
    return int(shape[0] * shape[1])


def _model_spec(cfg, env) -> ModelSpec:
    return ModelSpec.from_cfg(cfg, env)


class _DeviceSamplingLoop:
    """What SamplingLoop (evaluation_sampling_api.py:31-231) owns: env, trajectory buffers, the policy, the sampler."""

    def __init__(self, cfg, env_info: Optional[EnvInfo], model: Optional[PolicyModel], record_episodes: bool,
                 deterministic: bool = False):
        if not torch.cuda.is_available():
            raise RuntimeError("sample_factory_b200 needs a CUDA device (H100, sm_90a); there is no CPU execution path")
        self.cfg = cfg
        self.device = torch.device("cuda", torch.cuda.current_device())
        ops.bind_device(self.device)
        if not preprocess_cfg(cfg):
            raise ValueError("invalid configuration (see cfg.verify_cfg)")
        self.env = create_batched_env(cfg, dict(worker_index=0, vector_index=0, env_id=0), self.device)
        if env_info is not None:
            assert (env_info.obs_dim, env_info.num_actions, env_info.num_agents) == (
                self.env.obs_dim, self.env.num_actions, self.env.num_agents), "env_info does not match the env"
        spec = _model_spec(cfg, self.env)
        self.model = model if model is not None else PolicyModel(spec, self.device, seed=cfg.seed or 0,
                                                                 policy_init_gain=cfg.policy_init_gain,
                                 policy_initialization=getattr(cfg, "policy_initialization", "orthogonal"))
        engine = ops.ENGINES[getattr(cfg, "gemm_engine", "auto")] if getattr(cfg, "gemm_engine", "auto") != "auto" else (
            ops.GEMM_TC_3XTF32 if ops.tc_available() else ops.GEMM_SIMT)
        self.traj = alloc_for_spec(spec, self.env.num_agents, cfg.rollout, self.device)
        self.sampler = DeviceSampler(cfg, self.env, self.model, self.traj, engine=engine,
                                     use_cuda_graph=bool(getattr(cfg, "cuda_graph", True)),
                                     philox_seed=(cfg.seed or 0) * 1000003, record_episodes=record_episodes,
                                     deterministic=deterministic)
        self.stopped = False
        self.started = False
        self.status = StatusCode.SUCCESS

    def start(self, policy_version: int = 0):
        self.sampler.reset()
        self.sampler.set_policy_version(policy_version)
        self.started = True

    def rollout(self) -> Dict[str, Tensor]:
        assert self.started and not self.stopped
        self.sampler.rollout()
        return self.traj


class SyncSamplingAPI:
    """sync_sampling_api.py:16-65.  `param_servers` of the reference (shared policy weights) = `model` here."""

    def __init__(self, cfg, env_info: Optional[EnvInfo] = None, buffer_mgr=None, model: Optional[PolicyModel] = None):
        assert buffer_mgr is None, "trajectory buffers are owned by the device sampler"
        self.sampling_loop = _DeviceSamplingLoop(cfg, env_info, model, record_episodes=False)

    @property
    def model(self) -> PolicyModel:
        return self.sampling_loop.model

    def start(self, init_model_data=None):
        """init_model_data: optional (policy_id, state_dict, device, policy_version) as produced by Learner.init()."""
        version = 0
        if init_model_data is not None:
            _, state_dict, _, version = init_model_data
            self.sampling_loop.model.load_state_dict(state_dict, strict=False)
        self.sampling_loop.start(int(version))

    def set_policy_version(self, version: int) -> None:
        self.sampling_loop.sampler.set_policy_version(version)

    def get_trajectories_sync(self) -> Optional[Dict[str, Tensor]]:
        if self.sampling_loop.stopped:
            return None
        traj = self.sampling_loop.rollout()
        return {k: v.clone() for k, v in traj.items()}

    def stop(self) -> int:
        self.sampling_loop.stopped = True
        torch.cuda.synchronize()
        return self.sampling_loop.status


class EvalSamplingAPI:
    """evaluation_sampling_api.py:234-315: sample with the latest checkpoint of the experiment, collect per-episode stats.
    eval_stats has the reference's layout {stat_name: [per-policy list of per-episode values]}."""

    def __init__(self, cfg, env_info: Optional[EnvInfo] = None):
        self.cfg = cfg
        self.env_info = env_info
        self.sampling_loop: Optional[_DeviceSamplingLoop] = None
        self.total_samples = 0
        self._stats: Dict[str, List[List[float]]] = {}
        self.auto_pump = True

    def init(self):
        self.sampling_loop = _DeviceSamplingLoop(self.cfg, self.env_info, None, record_episodes=True)
        ck = load_checkpoint(self.cfg, self.sampling_loop.model, self.sampling_loop.device)   # Learner.init -> load
        self._policy_version = 0 if ck is None else ck["train_step"]
        self._stats = {k: [[] for _ in range(self.cfg.num_policies)] for k in ("reward", "len", "episode_number")}

    def start(self, init_model_data=None):
        if init_model_data is not None:
            _, state_dict, _, self._policy_version = init_model_data
            self.sampling_loop.model.load_state_dict(state_dict, strict=False)
        self.sampling_loop.start(int(self._policy_version))

    def pump(self, rollouts: int = 1) -> None:
        """Run `rollouts` rollouts and fold the finished episodes into eval_stats (the reference's background thread)."""
        for _ in range(rollouts):
            traj = self.sampling_loop.rollout()
            self.total_samples += samples_per_trajectory(traj)
            ret, ln = self.sampling_loop.sampler.finished_episodes()
            s = self._stats
            n0 = len(s["episode_number"][0])
            s["reward"][0].extend(float(x) for x in ret)
            s["len"][0].extend(int(x) for x in ln)
            s["episode_number"][0].extend(range(n0, n0 + len(ret)))

    def _polled(self):
        if self.auto_pump and self.sampling_loop is not None and self.sampling_loop.started and not self.sampling_loop.stopped:
            self.pump()

    @property
    def eval_stats(self):
        return self._stats

    @property
    def eval_episodes(self):
        self._polled()
        return self._stats.get("episode_number", [[] for _ in range(self.cfg.num_policies)])

    @property
    def eval_env_steps(self):
        lens = self._stats.get("len", [[] for _ in range(self.cfg.num_policies)])
        return [sum(lens[p]) for p in range(self.cfg.num_policies)]

    def stop(self) -> int:
        self.sampling_loop.stopped = True
        torch.cuda.synchronize()
        return self.sampling_loop.status


def generate_trajectories(cfg, env_info: Optional[EnvInfo], sample_env_episodes: int = 1024) -> int:
    """eval.py:83-114"""
    sampler = EvalSamplingAPI(cfg, env_info)
    sampler.init()
    sampler.start()
    t0 = time.time()
    episodes = 0
    while episodes < sample_env_episodes:
        episodes = len(sampler.eval_episodes[0])
    status = sampler.stop()
    dt = max(time.time() - t0, 1e-9)
    results = {}
    for key, stat in sampler.eval_stats.items():
        vals = stat[0]
        if not vals or key == "episode_number":
            continue
        results[f"{key}/{key}"] = float(sum(vals) / len(vals))
        results[f"{key}/{key}_min"], results[f"{key}/{key}_max"] = float(min(vals)), float(max(vals))
    print(f"[sf_b200] eval: {episodes} episodes, {sampler.total_samples} samples, {sampler.total_samples / dt:.0f} FPS")
    print(json.dumps(results, indent=4))
    out_dir = os.path.join(cfg.train_dir, cfg.experiment, getattr(cfg, "csv_folder_name", None) or "")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "eval_p0.csv"), "w") as f:     # eval.py:66-80 (pandas DataFrame.to_csv layout)
        keys = list(sampler.eval_stats.keys())
        f.write("," + ",".join(keys) + "\n")
        for i in range(len(sampler.eval_stats[keys[0]][0])):
            f.write(f"{i}," + ",".join(str(sampler.eval_stats[k][0][i]) for k in keys) + "\n")
    return status


def do_eval(cfg) -> int:
    """eval.py:117-124"""
    cfg.episode_counter = True
    cfg.decorrelate_envs_on_one_worker = False
    return generate_trajectories(cfg, obtain_env_info(cfg), cfg.sample_env_episodes)
