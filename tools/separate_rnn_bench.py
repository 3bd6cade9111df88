"""Throughput of separate actor / critic weights with recurrent cores against the shared-weights model, through the public
Runner API, on config 5's stack:

  4096 tape envs, Box(256) rows, Discrete(8), MLP [512, 256, 128] -> LSTM-512, rollout = recurrence = 16,
  2 x 32768 minibatches, 2 epochs
    shared    one encoder, one core (ActorCriticSharedWeights)
    separate  per tower its own encoder and core, state rows [actor | critic] (ActorCriticSeparateWeights)

    python tools/separate_rnn_bench.py [--iters 5] [--warmup 2]

The separate model runs every encoder GEMM, every core GEMM and every cell kernel twice, so about twice the shared
model's GEMM and cell time is expected.  The variants alternate (two samples of each).  One iteration =
Runner.iteration() (one rollout + one train()); the per-iteration time is a host clock around the timed iterations,
which end in a device synchronise; env-steps/s = N*T per iteration over it.  A separate profiled iteration splits the
GPU time into GEMM kernels (gemm_*), recurrent cell kernels (gru_* / lstm_*) and the rest.  The card's name and power
limit are read in the same run.
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

N, T, A, OBS = 4096, 16, 8, 256


def make_runner(variant, train_dir):
    from sample_factory_b200.cfg import parse_full_cfg, parse_sf_args
    from sample_factory_b200.envs import TapeVecEnv, register_env
    from sample_factory_b200.train import Runner

    dev = torch.device("cuda", 0)
    tape = torch.randn(2 * T + 1, N, OBS, generator=torch.Generator().manual_seed(2)).to(dev)
    register_env(f"sep_bench_{variant}", lambda name, cfg, env_config, render_mode=None: TapeVecEnv(tape, A))
    argv = [f"--env=sep_bench_{variant}", f"--experiment=sep_{variant}", f"--train_dir={train_dir}",
            "--restart_behavior=overwrite", "--batched_sampling=True", "--num_workers=1", "--num_envs_per_worker=1",
            "--worker_num_splits=1", "--seed=0", "--save_every_sec=100000", "--experiment_summaries_interval=100000",
            "--use_rnn=True", "--rnn_type=lstm", "--rnn_size=512", f"--actor_critic_share_weights={variant == 'shared'}",
            "--async_rl=False", f"--rollout={T}", f"--recurrence={T}", "--batch_size=32768", "--num_batches_per_epoch=2",
            "--num_epochs=2", "--encoder_mlp_layers", "512", "256", "128", "--value_bootstrap=True", "--reward_scale=0.01",
            "--max_grad_norm=1.0"]
    parser, _ = parse_sf_args(argv)
    r = Runner(parse_full_cfg(parser, argv))
    r.init()
    return r


def run(variant, iters, warmup):
    from torch.profiler import ProfilerActivity, profile

    with tempfile.TemporaryDirectory() as train_dir:
        r = make_runner(variant, train_dir)
        assert r.model.spec.share_weights == (variant == "shared")
        for _ in range(warmup):
            r.iteration()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(iters):
            r.iteration()
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3 / iters
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            r.iteration()
            torch.cuda.synchronize()
        split = dict(gemm=0.0, cell=0.0, rest=0.0)
        for e in prof.key_averages():
            t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            k = "gemm" if "gemm_" in e.key else ("cell" if ("gru_" in e.key or "lstm_" in e.key) else "rest")
            split[k] += t
        peak = torch.cuda.max_memory_allocated() / 2**30
        del r
    return dict(variant=variant, env_steps_per_s=N * T / (ms / 1e3), ms_per_iter=ms,
                **{f"{k}_gpu_ms": v / 1e3 for k, v in split.items()}, peak_mem_gib=peak)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("separate_rnn_bench needs a GPU")
    from sample_factory_b200 import ops

    ops.bind_device(torch.device("cuda", 0))
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    for variant in ("shared", "separate", "shared", "separate"):
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        print(json.dumps(dict(run(variant, a.iters, a.warmup), device=card)), flush=True)


if __name__ == "__main__":
    main()
