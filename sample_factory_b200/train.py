"""Training entry point with the reference's public surface (sample_factory/train.py:12-41, algo/runners/runner.py):

    cfg = parse_full_cfg(parser)          # sample_factory_b200.cfg
    register_env("my_env", make_env_func)  # sample_factory_b200.envs
    status = run_rl(cfg)                   # 0 success / 1 failure / 2 interrupted (algo/utils/misc.py:32-33)

The reference's Runner wires rollout workers, inference workers, a batcher and a learner through signal/slot event
loops across processes (runner.py:626-678).  Here the same components are three objects on ONE GPU stream pair and the
control loop is ~30 lines: rollout -> train -> (stats, checkpoint), repeated until the env-step / time budget is used.
Sync mode (async_rl=False) samples and learns back to back on one stream.  Async mode (async_rl=True, the reference's
default: "collect the next batch while the learner trains on the current one", cfg.py:53-61) is a fork-join per
iteration on two CUDA streams: the sampler (high-priority stream) collects rollout i+1 into its own trajectory set with
a SNAPSHOT of the weights while the learner trains on rollout i; at the join the learner's stream copies the fresh
trajectories across (the reference Batcher's copy, batcher.py:170-218; 45 MB D2D) and refreshes the snapshot.  Samples
are therefore one iteration (num_epochs x num_batches_per_epoch SGD steps) old when they are trained on -- recorded per
sample in traj["policy_version"] and masked by max_policy_lag exactly as in the reference (learner.py:950-953).
"""
from __future__ import annotations

import json
import os
import time
from collections import deque
from typing import Callable, Dict, List, Optional

import torch

from . import ops
from .cfg import preprocess_cfg
from .checkpoint import load_checkpoint, save_best, save_checkpoint
from .dist_utils import init_from_env
from .envs import set_training_info
from .host_env import create_batched_env
from .learner import Learner
from .model import ModelSpec, PolicyModel
from .sampler import DeviceSampler, SplitSampler
from .trajectory import alloc_for_spec


class StatusCode:
    SUCCESS, FAILURE, INTERRUPTED = 0, 1, 2


def experiment_dir(cfg) -> str:
    """utils/utils.py:409: <train_dir>/<experiment>"""
    d = os.path.join(cfg.train_dir, cfg.experiment)
    os.makedirs(d, exist_ok=True)
    return d


def select_engine(cfg) -> int:
    name = getattr(cfg, "gemm_engine", "auto")
    if name == "auto":
        return ops.GEMM_TC_3XTF32 if ops.tc_available() else ops.GEMM_SIMT
    return ops.ENGINES[name]


class Runner:
    """Single-policy runner (runner.py:81-184 attributes that examples/tests read are kept: env_steps, policy_avg_stats,
    register_observer / register_msg_handler hooks)."""

    def __init__(self, cfg, population=(0, 1)):
        self.cfg = cfg
        # (index, size) of this policy in a population (multi_policy.MultiPolicyRunner): it owns 1/size of the envs, the
        # reference's sync-mode agent -> policy mapping (agent_policy_mapping.py:39-45: global env index % num_policies)
        self.population = population
        self.policy_id = int(getattr(cfg, "policy_id", 0))
        self.env_steps = 0
        self.total_train_seconds = 0.0
        self.policy_avg_stats: Dict[str, List[deque]] = {}
        self.policy_lag: List[Dict[str, float]] = [dict()]     # runner.py:132,289: version_diff_{min,avg,max} per policy
        self.writers: Dict[int, object] = {}                   # runner.py:199-205: one tensorboard SummaryWriter per policy
        self.observers: List = []
        self.msg_handlers: Dict[str, List[Callable]] = {}
        self.fps_history: deque = deque(maxlen=64)
        self.initialized = False
        self.rollout_hook: Optional[Callable[[int], None]] = None   # called with the rollout index before each rollout
        # what the reference's runner publishes to the rollout workers (runner.py training_info / batched_sampling.py:351-354)
        self.training_info: Dict[str, object] = dict(approx_total_training_steps=0)
        self.rollouts_started = 0

    # ---- reference-compatible hooks --------------------------------------------------------------------------
    def register_observer(self, observer) -> None:
        self.observers.append(observer)

    def _notify(self, hook: str, *args) -> None:
        """AlgoObserver hooks (runner.py:52-73): on_init / on_start / on_training_step / extra_summaries / on_stop"""
        for o in self.observers:
            fn = getattr(o, hook, None)
            if fn is not None:
                fn(self, *args)

    def register_msg_handler(self, key: str, func: Callable) -> None:
        self.msg_handlers.setdefault(key, []).append(func)

    def register_episodic_stats_handler(self, func: Callable) -> None:
        self.register_msg_handler("episodic", func)

    # ----------------------------------------------------------------------------------------------------------
    def init(self) -> int:
        cfg = self.cfg
        self.rank, self.local_rank, self.world_size = init_from_env()
        if not torch.cuda.is_available():
            raise RuntimeError("sample_factory_b200 needs a CUDA device (H100, sm_90a); there is no CPU execution path")
        self.device = torch.device("cuda", self.local_rank)
        torch.cuda.set_device(self.device)
        ops.bind_device(self.device)
        if cfg.seed is not None:
            torch.manual_seed(cfg.seed + self.rank)
        if not preprocess_cfg(cfg):
            raise ValueError("invalid configuration (see cfg.verify_cfg)")
        # env instances: one batched env, or -- the reference's double-buffered sampling, rollout_worker.py:97-143 --
        # worker_num_splits groups of num_envs_per_worker / worker_num_splits env instances each (one instance per group
        # on this path), created with the reference's env_config (batched_sampling.py:166-174)
        n_splits = int(cfg.worker_num_splits) if (cfg.batched_sampling and cfg.worker_num_splits > 1 and
                                                   cfg.num_envs_per_worker == cfg.worker_num_splits) else 1
        self.envs = []
        p_idx, p_cnt = self.population
        n_host = None
        if p_cnt > 1:
            # plain CPU envs: this member wraps 1/P of the env instances (agent_policy_mapping.py:35-37 demands divisibility; a
            # factory that returns a batched device env sizes the member's share itself and ignores this)
            total = int(cfg.num_workers) * int(cfg.num_envs_per_worker)
            n_host = total // p_cnt if total % p_cnt == 0 else -1
        for s_ in range(n_splits):
            slot = (self.rank * p_cnt + p_idx) * n_splits + s_
            env_config = dict(worker_index=self.rank * p_cnt + p_idx, vector_index=s_, env_id=slot)
            if p_cnt > 1:       # a factory that returns a batched device env sizes it for one policy's share itself
                env_config.update(policy_index=p_idx, num_policies=p_cnt)
            self.envs.append(create_batched_env(cfg, env_config, self.device, num_envs=n_host))
        self.env = self.envs[0]
        from .model_factory import global_model_factory

        global_model_factory().check_supported()      # custom torch modules: explicit error through the registry API
        spec = ModelSpec.from_cfg(cfg, self.env)
        # (population members start from different weights: seed + index)
        self.model = PolicyModel(spec, self.device, seed=(cfg.seed or 0) + p_idx, policy_init_gain=cfg.policy_init_gain,
                                 policy_initialization=getattr(cfg, "policy_initialization", "orthogonal"))
        N = sum(e.num_agents for e in self.envs)
        self.engine = select_engine(cfg)
        self.traj = alloc_for_spec(spec, N, cfg.rollout, self.device)
        if self.world_size > 1:
            # identical replicas: broadcast rank 0's initial weights
            torch.distributed.broadcast(self.model.flat, src=0)
            self.model.weights_changed()
        self.async_rl = bool(cfg.async_rl)
        if self.async_rl:
            # the sampler owns a second trajectory set and a weight snapshot; it runs on its own high-priority stream
            self.sampler_model = self.model.inference_copy()
            self.sampler_traj = alloc_for_spec(spec, N, cfg.rollout, self.device)
            self.sampler_stream = torch.cuda.Stream(device=self.device, priority=-1)
            self.ev_rollout, self.ev_join = torch.cuda.Event(), torch.cuda.Event()
            self.snapshot_version = 0
            self.rollouts_in_flight = 0
        else:
            self.sampler_model, self.sampler_traj = self.model, self.traj
        sampler_kw = dict(engine=self.engine, use_cuda_graph=bool(getattr(cfg, "cuda_graph", True)),
                          philox_seed=(cfg.seed or 0) * 1000003 + self.rank * p_cnt + p_idx)
        if n_splits > 1:
            self.sampler = SplitSampler(cfg, self.envs, self.sampler_model, self.sampler_traj, **sampler_kw)
        else:
            self.sampler = DeviceSampler(cfg, self.env, self.sampler_model, self.sampler_traj, **sampler_kw)
        # The learner's dataset (batch_size x num_batches_per_epoch samples) may be a FRACTION of one rollout of all envs
        # (the reference's batcher then emits several training batches per rollout, batcher.py:170-218 -- e.g. the
        # sf_examples defaults: 160 envs x 32 steps, batch_size 512) or a MULTIPLE of it (rollouts are accumulated);
        # cfg/arguments.py:147-178.  Fractions train on row ranges of the rollout buffers in place, multiples are copied
        # into an accumulation set (the batcher's copy).
        T = cfg.rollout
        dataset = cfg.batch_size * cfg.num_batches_per_epoch
        if dataset % T != 0 or not ((N * T) % dataset == 0 or dataset % (N * T) == 0):
            raise ValueError(f"batch_size * num_batches_per_epoch = {dataset} must be a multiple of rollout = {T} and divide "
                             f"(or be a multiple of) the {N * T} samples one rollout of the {N} envs produces")
        self.k_split = max(1, (N * T) // dataset)
        self.k_acc = max(1, dataset // (N * T))
        n_learn = dataset // T
        self.learner = Learner(cfg, self.model, n_learn, engine=self.engine)
        self._train_views = None
        if self.k_split > 1:
            self._train_views = [{k: v[j * n_learn: (j + 1) * n_learn] for k, v in self.traj.items()} for j in range(self.k_split)]
        if self.k_acc > 1:
            self.accum = alloc_for_spec(spec, n_learn, T, self.device)
            self._acc_fill = 0
        if cfg.restart_behavior == "resume":
            ck = load_checkpoint(cfg, self.model, self.device, policy_id=self.policy_id)
            if ck is not None:
                self.learner.train_step, self.learner.env_steps = ck["train_step"], ck["env_steps"]
                self.learner.opt_step = ck["opt_step"]
                self.learner.curr_lr = ck.get("curr_lr", cfg.learning_rate)
                self.env_steps = ck["env_steps"]
                if self.async_rl:
                    self.sampler_model.copy_weights_from(self.model)
                    self.snapshot_version = self.learner.train_step
        if self.rank == 0:
            if p_idx == 0:
                with open(os.path.join(experiment_dir(cfg), "config.json"), "w") as f:
                    json.dump({k: v for k, v in vars(cfg).items() if _jsonable(v)}, f, indent=2)
            from .tb_writer import SummaryWriter

            # runner.py:199-205: <experiment_dir>/.summary/<policy_id>/events.out.tfevents.*
            self.writers[self.policy_id] = SummaryWriter(os.path.join(experiment_dir(cfg), ".summary", str(self.policy_id)))
        self.sampler.reset()
        self.initialized = True
        self._notify("on_init")
        return StatusCode.SUCCESS

    def load_state_dict(self, state_dict, strict: bool = False) -> None:
        """Replace the policy weights / normaliser state (warm start); the sampler's snapshot follows."""
        self.model.load_state_dict(state_dict, strict=strict)
        if self.async_rl:
            self.sampler_model.copy_weights_from(self.model)

    def _before_rollout(self) -> None:
        if self.rollout_hook is not None:
            self.rollout_hook(self.rollouts_started)
        self.rollouts_started += 1
        self.training_info["approx_total_training_steps"] = self.env_steps
        for e in self.envs:                                    # TrainingInfoInterface / RewardShapingInterface envs
            set_training_info(e, self.training_info)

    def iteration(self) -> None:
        """One sampler rollout + one learner update (the unit the FPS counter advances by N*T env steps)."""
        if self.async_rl:
            return self._iteration_async()
        self._before_rollout()
        self.sampler.set_policy_version(self.learner.train_step)
        self.sampler.rollout()
        self._train()
        self.env_steps = self.learner.env_steps

    def _train(self) -> None:
        """Learner.train on the freshly collected rollout in self.traj (see the dataset / rollout note in init)"""
        if self.k_split > 1:
            for view in self._train_views:
                self.learner.train(view)
        elif self.k_acc > 1:
            n = self.traj["rewards"].shape[0]
            j = self._acc_fill
            for k, v in self.traj.items():
                self.accum[k][j * n: (j + 1) * n].copy_(v, non_blocking=True)
            self._acc_fill += 1
            if self._acc_fill == self.k_acc:
                self._acc_fill = 0
                self.learner.train(self.accum)
        else:
            self.learner.train(self.traj)

    def _sample_on_side_stream(self) -> None:
        with torch.cuda.stream(self.sampler_stream):
            self.sampler_stream.wait_event(self.ev_join)        # snapshot + trajectory hand-off of the last join done
            self._before_rollout()
            self.sampler.set_policy_version(self.snapshot_version)
            self.sampler.rollout()
            self.ev_rollout.record(self.sampler_stream)

    def _join(self) -> None:
        """Learner stream: wait for the rollout, take its trajectories (Batcher copy) and publish the new weights."""
        main = torch.cuda.current_stream()
        main.wait_event(self.ev_rollout)
        for k, v in self.sampler_traj.items():
            self.traj[k].copy_(v, non_blocking=True)
        self.sampler_model.copy_weights_from(self.model)
        self.snapshot_version = self.learner.train_step
        self.ev_join.record(main)

    def _iteration_async(self) -> None:
        if self.rollouts_in_flight == 0:       # prime the pipeline: the first rollout has nothing to overlap with
            self.ev_join.record(torch.cuda.current_stream())
            self._sample_on_side_stream()
            self._join()
            self.rollouts_in_flight = 1
        # fork: the learner trains on rollout i while the sampler collects rollout i+1 with the snapshot taken at the
        # last join.  A device env's rollout is one graph launch -> enqueue it first; a host env keeps the host busy for
        # the whole rollout -> enqueue the learner's launches first.
        if getattr(self.env, "is_gpu_env", False):
            self._sample_on_side_stream()
            self._train()
        else:
            self._train()
            self._sample_on_side_stream()
        self._join()
        self.env_steps = self.learner.env_steps

    def _report_experiment_summaries(self, fps: float, train_stats: Dict[str, float]) -> None:
        """runner.py:368-423 (+ the learner's train summaries, learner.py:843-923) as tensorboard scalars"""
        w = self.writers.get(self.policy_id)
        if w is None:
            return
        steps = self.env_steps
        if fps == fps:
            w.add_scalar("perf/_fps", fps, steps)
        for key, stat in self.policy_avg_stats.items():
            vals = [v for v in stat[0] if isinstance(v, (int, float)) and v == v]
            if not vals:
                continue
            if key in ("reward", "len"):
                tag = f"{key}/{key}"
                w.add_scalar(tag + "_min", float(min(vals)), steps)
                w.add_scalar(tag + "_max", float(max(vals)), steps)
            else:
                tag = key if "/" in key else f"policy_stats/avg_{key}"
            w.add_scalar(tag, float(sum(vals) / len(vals)), steps)
        for key, val in train_stats.items():
            if isinstance(val, (int, float)) and val == val:
                w.add_scalar(f"train/{key}", float(val), steps)
        for key, val in self.policy_lag[0].items():
            w.add_scalar(f"train/{key}", float(val), steps)
        w.flush()

    def _time_is_up(self, t_start: float) -> bool:
        """train_for_seconds.  Data parallel: a per-rank wall clock would let one rank leave the loop while the others
        enter the next collective, so the ranks decide together (max elapsed time, every 8th iteration)."""
        elapsed = time.time() - t_start
        if self.world_size == 1:
            return elapsed >= self.cfg.train_for_seconds
        self._stop_checks = getattr(self, "_stop_checks", 0) + 1
        if self._stop_checks % 8 != 1:
            return False
        t = torch.tensor([elapsed], dtype=torch.float64, device=self.device)
        torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MAX)
        return float(t.item()) >= self.cfg.train_for_seconds

    def run(self) -> int:
        cfg = self.cfg
        assert self.initialized
        t_start = last_report = last_save = last_best = time.time()
        steps_at_report = self.env_steps
        status = StatusCode.SUCCESS
        self._notify("on_start")
        iterations = 0
        try:
            while self.env_steps < cfg.train_for_env_steps and not self._time_is_up(t_start):
                self.iteration()
                iterations += 1
                if self.observers:
                    self._notify("on_training_step", iterations)
                now = time.time()
                if now - last_report >= cfg.experiment_summaries_interval:
                    torch.cuda.synchronize()
                    now = time.time()
                    fps = (self.env_steps - steps_at_report) / (now - last_report)
                    self.fps_history.append(fps)
                    ep = self.sampler.pop_episode_stats()
                    st = self.learner.fetch_stats()
                    for key in ("version_diff_min", "version_diff_avg", "version_diff_max"):
                        if key in st:
                            self.policy_lag[0][key] = st[key]
                    for key, val in ep.items():                    # runner.py:296-308 running episodic statistics
                        self.policy_avg_stats.setdefault(key, [deque(maxlen=cfg.stats_avg)])[0].append(val)
                    for h in self.msg_handlers.get("episodic", []):
                        h(self, ep, 0)
                    if self.rank == 0:
                        self._report_experiment_summaries(fps, st)
                        if self.observers and self.writers.get(self.policy_id) is not None:
                            self._notify("extra_summaries", self.policy_id, self.env_steps, self.writers[self.policy_id])
                        print(f"[sf_b200] env_steps {self.env_steps} fps {fps:.0f} loss {st.get('loss', float('nan')):.4f} "
                              f"reward {ep.get('reward', float('nan')):.3f} episodes {ep.get('episodes', 0)}", flush=True)
                    last_report, steps_at_report = now, self.env_steps
                if now - last_save >= cfg.save_every_sec and self.rank == 0:
                    save_checkpoint(cfg, self.model, self.learner)
                    last_save = now
                if now - last_best >= cfg.save_best_every_sec and self.rank == 0:          # runner.py:459-476
                    last_best = now
                    hist = self.policy_avg_stats.get(cfg.save_best_metric)
                    if hist and len(hist[0]) > 0 and self.env_steps >= cfg.save_best_after:
                        vals = [v for v in hist[0] if v == v]
                        if vals:
                            save_best(cfg, self.model, self.learner, cfg.save_best_metric, float(sum(vals) / len(vals)))
        except KeyboardInterrupt:
            status = StatusCode.INTERRUPTED
        torch.cuda.synchronize()
        self.total_train_seconds = time.time() - t_start
        self._notify("on_stop")
        if self.rank == 0:
            save_checkpoint(cfg, self.model, self.learner)
            fps = self.env_steps / max(self.total_train_seconds, 1e-9)
            print(f"[sf_b200] Collected {{0: {self.env_steps}}}, FPS: {fps:.1f}", flush=True)   # runner.py:763-764
            for w in self.writers.values():
                w.close()
        return status


def _jsonable(v) -> bool:
    try:
        json.dumps(v)
        return True
    except TypeError:
        return False


def make_runner(cfg):
    """train.py:12-28 (+ the population runner for num_policies > 1, multi_policy.py)"""
    if getattr(cfg, "num_policies", 1) > 1:
        from .multi_policy import MultiPolicyRunner

        return cfg, MultiPolicyRunner(cfg)
    return cfg, Runner(cfg)


def run_rl(cfg) -> int:
    """train.py:31-41"""
    cfg, runner = make_runner(cfg)
    status = runner.init()
    if status == StatusCode.SUCCESS:
        status = runner.run()
    return status
