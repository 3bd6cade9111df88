"""bench.py --config {3,4,5}: the other BASELINE.json configs through the same engine and the same JSON contract as the
headline (config 2) line.  Synthetic tape envs of the named shapes, random-init weights of the named architectures.

  3  mujoco Ant-like   Box(27) obs -> Box(8) actions, tanh MLP 64-64, learned stddev, fixed-KL, value bootstrap, 2 epochs x 4
                       minibatches (sf_examples/mujoco/mujoco_params.py:1-38), 2048 envs per GPU, rollout 64, async_rl=True
  4  atari-like        uint8 [4,84,84] frames, convnet_atari + FC 512, ReLU, obs_scale 255, 4 epochs x 4 minibatches
                       (sf_examples/atari/atari_params.py:1-45), 1024 envs in total (1024 envs), rollout 32
                       (the reference's 128 would make one minibatch 32 768 frames; 8 192 keeps the im2col buffers at 3.4 GB)
  5  isaacgym-like     Box(256) obs, MLP 512-256-128 -> LSTM-512, rollout = recurrence = 16, batch 32768, value bootstrap,
                       KL-adaptive lr (sf_examples/isaacgym_examples/train_isaacgym.py:169-208, 310-350), 4096 envs per GPU
                       (32768 envs sharded over 8 GPUs in BASELINE.json)

`value`: env-steps/s with the env resident in HBM.  `e2e`: the same Runner with a HOST env (numpy tape, pinned staging): the
observation batch H2D and the actions D2H every env step.  `roofline`: the contraction op with the largest accumulated
device time inside three eagerly launched iterations (CUDA events around every GEMM-class op), as algorithmic
2*M*N*K / time against the measured bf16 peak.  `cpu_baseline`: the oracle port on a bounded sample (fewer envs, same
model / rollout / minibatch structure), env-steps/s."""
from __future__ import annotations

import json
import os
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
METRIC = "env-steps/sec (sampler+learner)"
UNIT = "env-steps/s"

CONFIGS = {
    3: dict(name="mujoco Ant-like continuous, 2048 envs per GPU, async double-buffered (BASELINE.json configs[2])",
            envs=2048, envs_total=False, T=64, obs_dim=27, A=8, continuous=True, obs_shape=None, uint8=False, async_rl=True,
            flags=["--use_rnn=False", "--recurrence=1", "--num_batches_per_epoch=4", "--num_epochs=2", "--encoder_mlp_layers",
                   "64", "64", "--nonlinearity=tanh", "--adaptive_stddev=False", "--kl_loss_coeff=0.1", "--value_loss_coeff=1.3",
                   "--max_grad_norm=3.5", "--exploration_loss_coeff=0.0", "--ppo_clip_ratio=0.2", "--learning_rate=0.00295",
                   "--value_bootstrap=True", "--policy_initialization=torch_default"],
            oracle=dict(continuous=True, adaptive_stddev=False, encoder_mlp_layers=[64, 64], nonlinearity="tanh", recurrence=1,
                        num_batches_per_epoch=4, num_epochs=2, kl_loss_coeff=0.1, value_loss_coeff=1.3, max_grad_norm=3.5,
                        exploration_loss_coeff=0.0, ppo_clip_ratio=0.2, learning_rate=0.00295, value_bootstrap=True),
            cpu_envs=2048),
    4: dict(name="atari-like uint8 [4,84,84] frames, convnet_atari + FC512, 1024 envs in total (BASELINE.json configs[3])",
            envs=1024, envs_total=True, T=32, obs_dim=4 * 84 * 84, A=6, continuous=False, obs_shape=(4, 84, 84), uint8=True,
            async_rl=False,
            flags=["--use_rnn=False", "--recurrence=1", "--num_batches_per_epoch=4", "--num_epochs=4",
                   "--encoder_conv_architecture=convnet_atari", "--encoder_conv_mlp_layers", "512", "--nonlinearity=relu",
                   "--obs_scale=255.0", "--exploration_loss_coeff=0.01", "--max_grad_norm=0.5", "--adam_eps=1e-5",
                   "--learning_rate=0.00025"],
            oracle=dict(obs_shape=(4, 84, 84), encoder_conv_architecture="convnet_atari", encoder_conv_mlp_layers=[512],
                        encoder_mlp_layers=[], nonlinearity="relu", obs_scale=255.0, recurrence=1, num_batches_per_epoch=4,
                        num_epochs=4, exploration_loss_coeff=0.01, max_grad_norm=0.5, adam_eps=1e-5, learning_rate=0.00025),
            cpu_envs=64),
    5: dict(name="isaacgym-like Box(256), MLP 512-256-128 -> LSTM-512, 4096 envs per GPU (BASELINE.json configs[4])",
            envs=4096, envs_total=False, T=16, obs_dim=256, A=8, continuous=False, obs_shape=None, uint8=False, async_rl=False,
            flags=["--use_rnn=True", "--rnn_type=lstm", "--rnn_size=512", "--recurrence=16", "--num_batches_per_epoch=2",
                   "--num_epochs=2", "--encoder_mlp_layers", "512", "256", "128", "--value_bootstrap=True", "--reward_scale=0.01",
                   "--lr_schedule=kl_adaptive_epoch", "--lr_schedule_kl_threshold=0.016", "--max_grad_norm=1.0"],
            oracle=dict(encoder_mlp_layers=[512, 256, 128], use_rnn=True, rnn_type="lstm", rnn_size=512, recurrence=16,
                        num_batches_per_epoch=2, num_epochs=2, value_bootstrap=True, reward_scale=0.01, max_grad_norm=1.0),
            cpu_envs=512),
}


class HostTapeEnv:
    """The synthetic env simulated on the HOST for any of the configs (numpy tape in pinned memory, float32 or uint8 frames,
    Discrete or Box actions): actions D2H and the observation batch H2D every step -- same rules as envs.TapeVecEnv."""

    is_gpu_env = False
    static_outputs = True

    def __init__(self, tape: torch.Tensor, num_actions: int, device, continuous=False, obs_shape=None, env_index_offset=0,
                 term_period=37, trunc_period=11):
        self.tape = tape.pin_memory()
        self.tape_len, self.num_agents, self.obs_dim = tape.shape
        self.num_actions, self.continuous = num_actions, continuous
        self.obs_shape = None if obs_shape is None else tuple(obs_shape)
        self.obs_uint8 = tape.dtype == torch.uint8
        self.term_period, self.trunc_period = term_period, trunc_period
        n = self.num_agents
        self.env_idx = np.arange(n, dtype=np.int64) + env_index_offset
        self.t = 0
        ashape, adt = ((n, num_actions), torch.float32) if continuous else ((n,), torch.int32)
        self.actions_host = torch.empty(ashape, dtype=adt).pin_memory()
        self.pack_host = torch.empty(6 * n, dtype=torch.uint8).pin_memory()
        self.rew_host = self.pack_host[: 4 * n].view(torch.float32)
        self.term_host = self.pack_host[4 * n: 5 * n].view(torch.bool)
        self.trunc_host = self.pack_host[5 * n:].view(torch.bool)
        self.obs = torch.empty((n, self.obs_dim), dtype=tape.dtype, device=device)
        self.pack = torch.empty(6 * n, dtype=torch.uint8, device=device)
        self.rew = self.pack[: 4 * n].view(torch.float32)
        self.terminated = self.pack[4 * n: 5 * n].view(torch.bool)
        self.truncated = self.pack[5 * n:].view(torch.bool)
        self.h2d_bytes = self.d2h_bytes = 0

    def reset(self):
        self.t = 0
        self.obs.copy_(self.tape[0], non_blocking=True)
        self.h2d_bytes += self.obs.numel() * self.obs.element_size()
        return self.obs

    def step(self, actions):
        self.actions_host.copy_(actions, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        self.d2h_bytes += self.actions_host.numel() * self.actions_host.element_size()
        a = self.actions_host.numpy()
        if self.continuous:
            np.clip(a[:, 0], -1.0, 1.0, out=self.rew_host.numpy())
        else:
            np.divide(a, float(self.num_actions), out=self.rew_host.numpy(), casting="unsafe")
        t = self.t
        term = ((t * 7 + self.env_idx * 13) % self.term_period) == 0
        self.term_host.numpy()[:] = term
        self.trunc_host.numpy()[:] = (((t + self.env_idx) % self.trunc_period) == 0) & ~term
        self.t += 1
        self.obs.copy_(self.tape[self.t % self.tape_len], non_blocking=True)
        self.pack.copy_(self.pack_host, non_blocking=True)
        self.h2d_bytes += self.obs.numel() * self.obs.element_size() + self.pack_host.numel()
        return self.obs, self.rew, self.terminated, self.truncated


def _cfg(c, env_name, n_envs, engine, async_rl, graphs=True):
    from sample_factory_b200.cfg import parse_full_cfg, parse_sf_args

    nmb = next(int(x.split("=")[1]) for x in c["flags"] if x.startswith("--num_batches_per_epoch"))
    batch = n_envs * c["T"] // nmb
    argv = [f"--env={env_name}", "--experiment=bench_cfg", "--train_dir=/tmp/sfb200_bench", "--restart_behavior=overwrite",
            f"--async_rl={async_rl}", "--serial_mode=True", "--batched_sampling=True", "--num_workers=1",
            "--num_envs_per_worker=1", "--worker_num_splits=1", f"--rollout={c['T']}", f"--batch_size={batch}",
            "--env_gpu_actions=True", "--env_gpu_observations=True", "--seed=0", f"--gemm_engine={engine}",
            f"--cuda_graph={graphs}", f"--learner_cuda_graph={graphs}", "--save_every_sec=1000000000"] + c["flags"]
    parser, _ = parse_sf_args(argv)
    return parse_full_cfg(parser, argv)


def oracle_cpu(c, steps=2, warmup=1):
    """the oracle port on a bounded sample of the config (fewer envs), best of a small thread-count sweep"""
    from oracle import appo_oracle as O

    n, T = c["cpu_envs"], c["T"]
    nmb = c["oracle"]["num_batches_per_epoch"]
    ocfg = O.OracleCfg(obs_dim=c["obs_dim"], num_actions=c["A"], rollout=T, batch_size=n * T // nmb, **c["oracle"])
    gen = torch.Generator().manual_seed(0)
    if c["uint8"]:
        tape = torch.randint(0, 256, (T + 1, n, c["obs_dim"]), dtype=torch.uint8, generator=gen)
    else:
        tape = torch.randn(2 * T + 1, n, c["obs_dim"], generator=gen)
    best = None
    total = os.cpu_count() or 1
    for threads in sorted({t for t in (8, 16, 32, total) if t <= total}):
        torch.set_num_threads(threads)
        learner = O.OracleLearner(ocfg, O.init_state(ocfg, seed=0))
        env = O.TapeVecEnv(tape, c["A"])
        last = env.reset()
        times = []
        for it in range(warmup + steps):
            t0 = time.perf_counter()
            with torch.no_grad():
                noise = (torch.randn(T, n, c["A"], generator=gen) if c["continuous"] else
                         torch.empty(T, n, c["A"]).exponential_(generator=gen))
                traj = O.alloc_trajectories(ocfg, n)
                last = O.rollout(ocfg, learner.st, env, last, traj, noise, learner.train_step)
            learner.train(traj)
            if it >= warmup:
                times.append(time.perf_counter() - t0)
        v = n * T * len(times) / sum(times)
        if best is None or v > best["value"]:
            best = dict(value=v, cores=threads, ms_per_step=1e3 * sum(times) / len(times))
    best.update(unit=UNIT, kind="port",
                sample=f"{steps} iterations of {n} envs x {T} steps + learner after {warmup} warm-up (bounded sample: the config's "
                       f"model / rollout / epoch structure at {n} instead of {c['envs']} envs), oracle port, torch CPU, "
                       f"{best['cores']} of {total} host threads (best of a sweep)")
    return best


def run_config(args, load_peaks, ClockSampler):
    from sample_factory_b200 import ops
    from sample_factory_b200.dist_utils import init_from_env
    from sample_factory_b200.envs import TapeVecEnv, register_env
    from sample_factory_b200.train import Runner

    c = CONFIGS[args.config]
    rank, local_rank, world = init_from_env()
    assert world == args.gpus, f"--gpus {args.gpus} but WORLD_SIZE={world}"
    dev = torch.device("cuda", local_rank)
    torch.cuda.set_device(dev)
    ops.bind_device(dev)
    dist = torch.distributed
    peaks = load_peaks()
    n_envs = c["envs"] // world if c["envs_total"] else c["envs"]
    T = c["T"]
    gen = torch.Generator().manual_seed(77 + rank)
    tape_len = 2 * T + 1 if not c["uint8"] else T + 1
    if c["uint8"]:
        tape_cpu = torch.randint(0, 256, (tape_len, n_envs, c["obs_dim"]), dtype=torch.uint8, generator=gen)
    else:
        tape_cpu = torch.randn(tape_len, n_envs, c["obs_dim"], generator=gen)
    tape_dev = tape_cpu.to(dev)
    register_env("bench_cfg_dev", lambda name, cfg, env_config, render_mode=None: TapeVecEnv(
        tape_dev, c["A"], continuous=c["continuous"], obs_shape=c["obs_shape"], env_index_offset=rank * n_envs))
    register_env("bench_cfg_host", lambda name, cfg, env_config, render_mode=None: HostTapeEnv(
        tape_cpu, c["A"], dev, continuous=c["continuous"], obs_shape=c["obs_shape"], env_index_offset=rank * n_envs))

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(x):
        if world == 1:
            return x
        t = torch.tensor([x], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    runner = Runner(_cfg(c, "bench_cfg_dev", n_envs, args.engine, c["async_rl"]))
    runner.init()
    clocks = ClockSampler(local_rank)
    clocks.start()
    for _ in range(args.warmup):
        runner.iteration()
    barrier()
    clocks.lines.clear()
    n0 = ops.launch_count()
    replay = 0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    barrier()
    e0.record()
    for _ in range(args.steps):
        runner.iteration()
        replay += runner.sampler.graph_replay_launches + runner.learner.graph_replay_launches
    e1.record()
    barrier()
    ms_total = max_over_ranks(e0.elapsed_time(e1))
    clock_info = clocks.stop()
    launches = ops.launch_count() - n0 + replay
    value = world * n_envs * T * args.steps / (ms_total / 1e3)
    learner_graph = bool(runner.learner.use_graph)

    # ---- dominant contraction: CUDA events around every GEMM-class op during three eagerly launched iterations
    timed = {}

    def wrap(name, key_work):
        fn = getattr(ops, name)

        def wrapped(*a, **k):
            key, work = key_work(*a, **k)
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            r = fn(*a, **k)
            e.record()
            timed.setdefault(key, dict(work=work, ev=[]))["ev"].append((s, e))
            return r

        setattr(ops, name, wrapped)
        return fn

    orig = dict(
        linear_act_forward=wrap("linear_act_forward", lambda x, W, *a, **k: (
            f"forward GEMM [{x.shape[0]}x{W.shape[0]}x{W.shape[1]}]", 2.0 * x.shape[0] * W.shape[0] * W.shape[1])),
        linear_act_heads_forward=wrap("linear_act_heads_forward", lambda x, W, *a, **k: (
            f"forward GEMM + heads [{x.shape[0]}x{W.shape[0]}x{W.shape[1]}]", 2.0 * x.shape[0] * W.shape[0] * W.shape[1])),
        linear_backward=wrap("linear_backward", lambda dz, x, W, act_prev, dW, dx, *a, **k: (
            f"backward GEMMs dW{'+dX' if dx is not None else ''} [{dz.shape[0]}x{W.shape[0]}x{W.shape[1]}]",
            2.0 * dz.shape[0] * W.shape[0] * W.shape[1] * ((dW is not None) + (dx is not None)))))
    runner.learner.use_graph = False
    sampler_graph = runner.sampler.use_cuda_graph
    runner.sampler.use_cuda_graph = False
    for _ in range(3):
        runner.iteration()
    torch.cuda.synchronize()
    for k, fn in orig.items():
        setattr(ops, k, fn)
    runner.sampler.use_cuda_graph = sampler_graph
    roofline = None
    if timed:
        tot = {k: sum(s.elapsed_time(e) for s, e in d["ev"]) for k, d in timed.items()}
        key = max(tot, key=tot.get)
        d = timed[key]
        avg_ms = tot[key] / len(d["ev"])
        ach = d["work"] / (avg_ms * 1e-3) / 1e12
        roofline = dict(kernel=key + " (wgmma 3xTF32 engine: ceiling = peak / 6)", bound="tensor", achieved=ach,
                        peak=peaks["tflops_burst"], unit="TFLOP/s", frac=ach / peaks["tflops_burst"], traffic=None,
                        avg_kernel_ms=avg_ms, launches_timed=len(d["ev"]), share_of_gemm_time=tot[key] / sum(tot.values()),
                        peak_source=peaks["source"] + ", bf16 burst")
    del runner
    torch.cuda.empty_cache()

    # ---- end to end: host env, copies inside the timed region
    e2e = None
    if not args.no_e2e:
        r2 = Runner(_cfg(c, "bench_cfg_host", n_envs, args.engine, False))
        r2.init()
        for _ in range(max(3, args.warmup)):
            r2.iteration()
            r2.learner.fetch_stats()
        barrier()
        env = r2.env
        h0, d0 = env.h2d_bytes, env.d2h_bytes
        stats_bytes = 0
        t0 = time.perf_counter()
        for _ in range(args.steps):
            r2.iteration()
            st = r2.learner.fetch_stats()
            stats_bytes += 8 * sum(1 for v in st.values() if isinstance(v, float))
        barrier()
        dt = max_over_ranks(time.perf_counter() - t0)
        e2e = dict(value=world * n_envs * T * args.steps / dt, unit=UNIT, h2d_bytes_per_step=(env.h2d_bytes - h0) // args.steps,
                   d2h_bytes_per_step=(env.d2h_bytes - d0 + stats_bytes) // args.steps, ms_per_step=1e3 * dt / args.steps,
                   api="sample_factory_b200.train.Runner.iteration() with a HOST env (numpy tape, pinned staging): observation "
                       "batch H2D + actions D2H every env step, loss statistics D2H every iteration")
        del r2
        torch.cuda.empty_cache()

    cpu_baseline = None
    if world == 1 and rank == 0 and not args.no_cpu_baseline:
        cpu_baseline = oracle_cpu(c)
    if rank == 0:
        out = dict(metric=METRIC + f" -- {c['name']}", value=value, unit=UNIT, n_gpus=world, steps=args.steps, warmup=args.warmup,
                   ms_per_step=ms_total / args.steps, higher_is_better=True, scaling="strong" if c["envs_total"] else "weak",
                   vs_baseline=None, dtype="f32 (3-pass operand split on wgmma -- scaled fp16 hi/lo pairs where the operand ranges are known, tf32 hi/lo pairs elsewhere -- fp32 accumulate)", data="synthetic",
                   config=dict(workload=c["name"], envs_per_gpu=n_envs, rollout=T, global_batch=world * n_envs * T,
                               parallelism=f"dp{world}", async_rl=c["async_rl"], cuda_graph_learner=learner_graph,
                               l2_policy="trajectory set + learner activations exceed the 126 MB L2; no explicit flush"),
                   clocks=clock_info, e2e=e2e, gpu_launches=int(launches), roofline=roofline, cpu_baseline=cpu_baseline)
        print(json.dumps(out), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def run_config_reference(args):
    """--impl reference --config N: the CPU path for that config (oracle port, bounded sample), same JSON contract"""
    if int(os.environ.get("RANK", "0")) != 0:
        return
    c = CONFIGS[args.config]
    r = oracle_cpu(c, steps=max(1, min(args.steps, 3)), warmup=max(1, min(args.warmup, 1)))
    out = dict(impl="reference", metric=METRIC + f" -- {c['name']}", value=r["value"], unit=UNIT, n_gpus=args.gpus, steps=args.steps,
               warmup=args.warmup, ms_per_step=r["ms_per_step"], higher_is_better=True, scaling="weak", vs_baseline=None,
               dtype="f32", data="synthetic", config=dict(workload=c["name"]), cpu_baseline=r,
               e2e=dict(value=r["value"], unit=UNIT, h2d_bytes_per_step=0, d2h_bytes_per_step=0))
    print(json.dumps(out), flush=True)
