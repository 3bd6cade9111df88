"""Throughput of a Dict observation model (MultiInputEncoder) against the same tape row as a single key, through the
public Runner API:

  4096 tape envs, rows of 31 floats, Discrete(8), MLP [512, 512], rollout 32, 4 x 32768 minibatches, one epoch
    dict    keys achieved_goal(3), desired_goal(3), observation(25): one MLP [512, 512] per key, outputs concatenated
    single  the whole row as the key "obs": one MLP [512, 512]

    python tools/dict_obs_bench.py [--iters 5] [--warmup 2]

By construction the Dict model runs three encoder MLPs where the single-key model runs one: per sample its encoder
FLOPs are 2 * (31 * 512 + 3 * 512 * 512) against 2 * (31 * 512 + 512 * 512), and its heads read a 1536-wide
concatenation instead of 512 columns.  The script prints that ratio next to the rates.

One iteration = Runner.iteration() (one rollout + one train()).  The per-iteration time is a host clock around the timed
iterations, which end in a device synchronise; env-steps/s = N*T per iteration over it.  A separate profiled iteration
gives the share of GPU time in GEMM kernels (gemm_*); with this model (no decoder, no core, narrow heads) every GEMM
is an encoder layer's forward or backward.  The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import os
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N, T, A = 4096, 32, 8
KEYS = [("achieved_goal", 3), ("desired_goal", 3), ("observation", 25)]
OBS = sum(d for _, d in KEYS)
HIDDEN = 512


def encoder_flops_per_sample(n_keys_mlp: int) -> int:
    """forward FLOPs of the encoder MLPs for one sample (first layers read the whole row in total)"""
    return 2 * (OBS * HIDDEN + n_keys_mlp * HIDDEN * HIDDEN)


def make_runner(variant, train_dir):
    from sample_factory_b200.cfg import parse_full_cfg, parse_sf_args
    from sample_factory_b200.envs import TapeVecEnv, register_env
    from sample_factory_b200.train import Runner

    dev = torch.device("cuda", 0)
    tape = torch.randn(2 * T + 1, N, OBS, generator=torch.Generator().manual_seed(2)).to(dev)
    keys = KEYS if variant == "dict" else None
    register_env(f"dict_bench_{variant}", lambda name, cfg, env_config, render_mode=None: TapeVecEnv(tape, A, obs_keys=keys))
    argv = [f"--env=dict_bench_{variant}", f"--experiment=dict_{variant}", f"--train_dir={train_dir}",
            "--restart_behavior=overwrite", "--batched_sampling=True", "--num_workers=1", "--num_envs_per_worker=1",
            "--worker_num_splits=1", "--seed=0", "--save_every_sec=100000", "--experiment_summaries_interval=100000",
            "--use_rnn=False", "--async_rl=False", f"--rollout={T}", "--recurrence=1", "--batch_size=32768", "--num_batches_per_epoch=4",
            "--encoder_mlp_layers", str(HIDDEN), str(HIDDEN)]
    parser, _ = parse_sf_args(argv)
    r = Runner(parse_full_cfg(parser, argv))
    r.init()
    return r


def run(variant, iters, warmup):
    from torch.profiler import ProfilerActivity, profile

    with tempfile.TemporaryDirectory() as train_dir:
        r = make_runner(variant, train_dir)
        assert r.model.spec.dict_obs == (variant == "dict")
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
        gemm = total = 0.0
        for e in prof.key_averages():
            t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            total += t
            if "gemm_" in e.key:
                gemm += t
        peak = torch.cuda.max_memory_allocated() / 2**30
        del r
    return dict(variant=variant, env_steps_per_s=N * T / (ms / 1e3), ms_per_iter=ms, gemm_share_of_gpu_time=gemm / total,
                profiled_gpu_ms=total / 1e3, peak_mem_gib=peak)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dict_obs_bench needs a GPU")
    from sample_factory_b200 import ops

    ops.bind_device(torch.device("cuda", 0))
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    ratio = encoder_flops_per_sample(len(KEYS)) / encoder_flops_per_sample(1)
    for variant in ("single", "dict", "single", "dict"):        # alternated: two samples of each
        torch.cuda.reset_peak_memory_stats()
        print(json.dumps(dict(run(variant, a.iters, a.warmup), encoder_flop_ratio_dict_over_single=ratio, device=card)),
              flush=True)


if __name__ == "__main__":
    main()
