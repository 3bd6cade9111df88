"""Cost of a batched tensor env (IsaacGym / Brax style) behind BatchedTensorEnvAdapter against the native device env, through
the public Runner API, with config 2's model and sizes:

  4096 tape envs, Box(64) observations, Discrete(8), MLP [512, 512], rollout 32, 4 x 32768 minibatches, one epoch
    native  TapeVecEnv: the engine's own env contract, the whole rollout one CUDA graph
    cuda    the same rules as a batched tensor env on the GPU: fresh tensors every step (obs float32, reward float64,
            terminated int64, truncated uint8), device actions (env_gpu_actions=True); one ingest launch per step
    cpu     the same env returning CPU tensors, numpy actions (env_gpu_actions=False): a pinned D2H copy of the actions,
            a pinned H2D copy per output, then the ingest launch

    python tools/batched_tensor_env_bench.py [--iters 5] [--warmup 2]

One iteration = Runner.iteration() (one rollout + one train()).  env-steps/s = N*T per iteration over a host clock around
the timed iterations, which end in a device synchronise.  A separate instrumented iteration records CUDA events around
every sfb200_env_ingest call (that span includes host enqueue latency whenever the device waits for the host), then times
the last step's launch 200 times back to back in one CUDA graph: the kernel's time, and the bytes it reads and writes per step (computed from
the tensors' shapes and dtypes) over that time.  The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N, T, A, OBS = 4096, 32, 8, 64


class BatchedTapeEnv:
    """TapeVecEnv's rules as a batched tensor env: one env, num_agents = N, fresh tensors from every reset() / step()"""

    def __init__(self, inner, on_cpu):
        from gymnasium import spaces
        import numpy as np

        self.e, self.on_cpu = inner, on_cpu
        self.num_agents, self.is_multiagent = inner.num_agents, True
        self.observation_space = spaces.Box(-np.inf, np.inf, (inner.obs_dim,), np.float32)
        self.action_space = spaces.Discrete(inner.num_actions)

    def _out(self, t):
        return t.cpu() if self.on_cpu else t

    def reset(self, **kw):
        return self._out(self.e.reset().clone()), {}

    def step(self, actions):
        obs, rew, term, trunc = self.e.step(torch.as_tensor(actions).to(self.e.tape.device))
        return (self._out(obs.clone()), self._out(rew.double()), self._out(term.to(torch.int64)),
                self._out(trunc.to(torch.uint8)), {})


def make_runner(variant, train_dir):
    from sample_factory_b200.cfg import parse_full_cfg, parse_sf_args
    from sample_factory_b200.envs import TapeVecEnv, register_env
    from sample_factory_b200.train import Runner

    dev = torch.device("cuda", 0)
    tape = torch.randn(2 * T + 1, N, OBS, generator=torch.Generator().manual_seed(2)).to(dev)
    if variant == "native":
        make = lambda name, cfg, env_config, render_mode=None: TapeVecEnv(tape, A)
    else:
        make = lambda name, cfg, env_config, render_mode=None: BatchedTapeEnv(TapeVecEnv(tape, A), variant == "cpu")
    register_env(f"bt_bench_{variant}", make)
    argv = [f"--env=bt_bench_{variant}", f"--experiment=bt_{variant}", f"--train_dir={train_dir}",
            "--restart_behavior=overwrite", "--batched_sampling=True", "--num_workers=1", "--num_envs_per_worker=1",
            "--worker_num_splits=1", "--seed=0", "--save_every_sec=100000", "--experiment_summaries_interval=100000",
            "--use_rnn=False", "--async_rl=False", f"--rollout={T}", "--recurrence=1", "--batch_size=32768",
            "--num_batches_per_epoch=4", "--encoder_mlp_layers", "512", "512", f"--env_gpu_actions={variant != 'cpu'}"]
    parser, _ = parse_sf_args(argv)
    r = Runner(parse_full_cfg(parser, argv))
    r.init()
    return r


def ingest_cost(r):
    """(ms between CUDA events around each sfb200_env_ingest call, ms per launch back to back, bytes it moves per env
    step) over one instrumented iteration"""
    from sample_factory_b200 import ops

    real, pairs, moved, last = ops.env_ingest, [], [], []

    def timed(entries, rows):
        last[:] = [entries, rows]
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        real(entries, rows)
        b.record()
        pairs.append((a, b))
        moved.append(sum(rows * cols * (src.element_size() + dst.element_size()) for src, _, cols, dst, _, _ in entries))

    ops.env_ingest = timed
    try:
        r.iteration()
        torch.cuda.synchronize()
    finally:
        ops.env_ingest = real
    span = sum(a.elapsed_time(b) for a, b in pairs) / len(pairs)
    # the same launch 200 times back to back in one CUDA graph (the last step's tensors): the kernel's own time, without
    # the host's enqueue latency that the in-loop span includes whenever the device waits for the host
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(200):
            real(*last)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    g.replay()
    b.record()
    torch.cuda.synchronize()
    return span, a.elapsed_time(b) / 200, sum(moved) / len(moved)


def run(variant, iters, warmup):
    with tempfile.TemporaryDirectory() as train_dir:
        r = make_runner(variant, train_dir)
        for _ in range(warmup):
            r.iteration()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(iters):
            r.iteration()
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3 / iters
        out = dict(variant=variant, env_steps_per_s=N * T / (ms / 1e3), ms_per_iter=ms)
        if variant != "native":
            span_ms, kernel_ms, nbytes = ingest_cost(r)
            out.update(ingest_span_us_per_step=span_ms * 1e3, ingest_kernel_us=kernel_ms * 1e3,
                       ingest_bytes_per_step=nbytes, ingest_kernel_gb_per_s=nbytes / (kernel_ms * 1e-3) / 1e9)
        del r
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("batched_tensor_env_bench needs a GPU")
    from sample_factory_b200 import ops

    ops.bind_device(torch.device("cuda", 0))
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    for variant in ("native", "cuda", "cpu", "native", "cuda", "cpu"):        # alternated: two samples of each
        print(json.dumps(dict(run(variant, a.iters, a.warmup), device=card)), flush=True)


if __name__ == "__main__":
    main()
