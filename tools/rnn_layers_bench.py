"""Throughput of stacked recurrent cores (--rnn_num_layers) on config 5's stack, through the public Runner API:

  4096 tape envs, Box(256) observations, MLP 512-256-128 -> LSTM-512 x L, rollout = recurrence = 16,
  2 x 32768 minibatches, 2 epochs, value bootstrap, KL-adaptive lr (train_isaacgym.py:169-208, 310-350)

    python tools/rnn_layers_bench.py [--layers 1 2 3] [--iters 5] [--warmup 2] [--dump-outputs DIR]

One iteration = Runner.iteration() (one rollout + one train()).  The per-iteration time is a host clock around the timed
iterations, which end in a device synchronise; env-steps/s = N*T per iteration over it.  A separate profiled iteration
splits the GPU time into GEMMs (gemm_*), recurrent cell kernels (gru_* / lstm_* / mask_rows) and everything else.  The
card's name and power limit are read in the same run and printed with the numbers.

--dump-outputs DIR writes what the last timed iteration computed, for each L, to DIR/L<L>/<name>.npy: the trajectories
(with the recurrent states, without the observation inputs), the learner's returns / advantages / minibatch log and
the updated parameters.  At L = 1 the script passes no --rnn_num_layers flag, so it runs unchanged on a checkout
without stacked cores and the two dumps can be compared bit for bit.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N, T, OBS = 4096, 16, 256
GEMM_KERNELS = ("gemm_",)
CELL_KERNELS = ("gru_", "lstm_", "mask_rows")
DUMP_MAX_BYTES = 64 << 20


def make_runner(layers, train_dir):
    from sample_factory_b200.cfg import parse_full_cfg, parse_sf_args
    from sample_factory_b200.envs import TapeVecEnv, register_env
    from sample_factory_b200.train import Runner

    dev = torch.device("cuda", 0)
    tape = torch.randn(2 * T + 1, N, OBS, generator=torch.Generator().manual_seed(2)).to(dev)
    register_env("rnn_layers_bench", lambda name, cfg, env_config, render_mode=None: TapeVecEnv(tape, 8))
    argv = ["--env=rnn_layers_bench", f"--experiment=rnn_l{layers}", f"--train_dir={train_dir}",
            "--restart_behavior=overwrite", "--batched_sampling=True", "--num_workers=1", "--num_envs_per_worker=1",
            "--worker_num_splits=1", "--seed=0", "--save_every_sec=100000", "--experiment_summaries_interval=100000",
            "--use_rnn=True", "--rnn_type=lstm", "--rnn_size=512", "--async_rl=False", f"--rollout={T}",
            f"--recurrence={T}", "--batch_size=32768", "--num_batches_per_epoch=2", "--num_epochs=2",
            "--encoder_mlp_layers", "512", "256", "128", "--value_bootstrap=True", "--reward_scale=0.01",
            "--lr_schedule=kl_adaptive_epoch", "--lr_schedule_kl_threshold=0.016", "--max_grad_norm=1.0"]
    if layers != 1:
        argv.append(f"--rnn_num_layers={layers}")
    parser, _ = parse_sf_args(argv)
    r = Runner(parse_full_cfg(parser, argv))
    r.init()
    return r


def dump_outputs(out_dir, runner):
    """one DIR/<name>.npy per output; arrays beyond a quarter of the remaining 64 MB are cut to a fixed, seeded sample of
    rows (the same rows on every run)"""
    os.makedirs(out_dir, exist_ok=True)
    torch.cuda.synchronize()
    arrays = {f"traj_{k}": v for k, v in runner.traj.items() if k != "obs"}
    arrays["learner_returns"] = runner.learner.returns
    arrays["learner_advantages"] = runner.learner.advantages
    arrays["learner_minibatch_log"] = runner.learner.minibatch_log()
    arrays["model_params"] = runner.model.flat
    budget = DUMP_MAX_BYTES
    gen = torch.Generator().manual_seed(0)
    for name, t in arrays.items():
        t = t.detach().cpu()
        t = t.double() if t.dtype == torch.float64 else t.float()
        if t.numel() * t.element_size() > budget // 4 and t.dim() > 0:
            keep = max(1, (budget // 4) // max(1, t[0].numel() * t.element_size()))
            t = t[torch.randperm(t.shape[0], generator=gen)[:keep].sort().values]
        budget -= t.numel() * t.element_size()
        np.save(os.path.join(out_dir, f"{name}.npy"), t.numpy())


def run(layers, iters, warmup, dump_dir):
    from torch.profiler import ProfilerActivity, profile

    with tempfile.TemporaryDirectory() as train_dir:
        r = make_runner(layers, train_dir)
        assert r.traj["rnn_states"].shape[2] == 2 * 512 * layers
        for _ in range(warmup):
            r.iteration()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(iters):
            r.iteration()
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3 / iters
        if dump_dir:
            dump_outputs(os.path.join(dump_dir, f"L{layers}"), r)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            r.iteration()
            torch.cuda.synchronize()
        split = dict(gemm=0.0, cell=0.0, other=0.0)
        for e in prof.key_averages():
            t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            if any(k in e.key for k in GEMM_KERNELS):
                split["gemm"] += t
            elif any(k in e.key for k in CELL_KERNELS):
                split["cell"] += t
            else:
                split["other"] += t
        peak = torch.cuda.max_memory_allocated() / 2**30
        del r
    return dict(rnn_num_layers=layers, env_steps_per_s=N * T / (ms / 1e3), ms_per_iter=ms,
                profiled_ms=dict(gemm=split["gemm"] / 1e3, cell=split["cell"] / 1e3, other=split["other"] / 1e3),
                peak_mem_gib=peak)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, nargs="+", default=[1, 2, 3])
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--dump-outputs", dest="dump_outputs", default=None, metavar="DIR")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rnn_layers_bench needs a GPU")
    from sample_factory_b200 import ops

    ops.bind_device(torch.device("cuda", 0))
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    for layers in a.layers:
        torch.cuda.reset_peak_memory_stats()
        print(json.dumps(dict(run(layers, a.iters, a.warmup, a.dump_outputs), device=card)), flush=True)


if __name__ == "__main__":
    main()
