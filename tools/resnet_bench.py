#!/usr/bin/env python
"""Throughput and kernel-time shares of the resnet_impala image encoder (the reference's ResnetEncoder,
model/encoder.py:153-221) through the public Runner: 1024 device tape envs, uint8 [4, 84, 84] frames, resnet_impala +
FC 512, ReLU, obs_scale 255, rollout 16, batch 4096 x 4 minibatches x 1 epoch.

  python tools/resnet_bench.py [--iters K] [--warmup W] [--profile-iters P]

Prints one JSON line:
  env_steps_per_s    env steps / s over K timed iterations (rollout + learner), CUDA events around the window
  kernel_share       GPU time of each kernel class over the GPU time of the profiled iterations (torch.profiler, a
                     separate run after the timed window): the encoder's gathers (im2col, col2im), the max-pool forward /
                     backward, the final act + permute, and the GEMM engines (conv GEMMs and the FC / heads GEMMs
                     together; the convs dominate)
  gpu, power_limit_w read in the same run
Needs a CUDA device; writes nothing into the repository tree (the Runner's train_dir is a temporary directory)."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

N_ENVS, ROLLOUT, SHAPE, N_ACTIONS = 1024, 16, (4, 84, 84), 6

KERNEL_CLASSES = [  # (class, substring of the kernel's name), first match wins
    ("im2col", "im2col_kernel"),
    ("col2im", "col2im_kernel"),
    ("maxpool_backward", "maxpool3s2_bwd_kernel"),
    ("maxpool_forward", "maxpool3s2_kernel"),
    ("act_permute", "permute_bpc_kernel"),
    ("gemm_wgmma", "gemm_wgmma_kernel"),
    ("gemm_simt", "gemm_simt_kernel"),
    ("gemm_splitk_reduce", "splitk_reduce_kernel"),
    ("colsum", "colsum_"),
]


def power_limit_w() -> float | None:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return float(out.strip().splitlines()[0])
    except Exception:
        return None


def make_runner(train_dir: str):
    from sample_factory_b200.cfg import parse_full_cfg, parse_sf_args
    from sample_factory_b200.envs import TapeVecEnv, register_env
    from sample_factory_b200.train import Runner

    dev = torch.device("cuda", 0)
    gen = torch.Generator().manual_seed(0)
    tape = torch.randint(0, 256, (2 * ROLLOUT + 1, N_ENVS, SHAPE[0] * SHAPE[1] * SHAPE[2]), dtype=torch.uint8,
                         generator=gen).to(dev)
    register_env("resnet_bench_atari", lambda name, cfg, env_config, render_mode=None: TapeVecEnv(tape, N_ACTIONS, obs_shape=SHAPE))
    argv = ["--env=resnet_bench_atari", "--experiment=resnet_bench", f"--train_dir={train_dir}",
            "--restart_behavior=overwrite", "--batched_sampling=True", "--num_workers=1", "--num_envs_per_worker=1",
            "--worker_num_splits=1", "--seed=0", "--save_every_sec=1000000", "--experiment_summaries_interval=1000000",
            "--use_rnn=False", "--async_rl=False", f"--rollout={ROLLOUT}", "--recurrence=1", "--batch_size=4096",
            "--num_batches_per_epoch=4", "--num_epochs=1", "--encoder_conv_architecture=resnet_impala",
            "--encoder_conv_mlp_layers", "512", "--nonlinearity=relu", "--obs_scale=255.0",
            "--exploration_loss_coeff=0.01", "--max_grad_norm=0.5", "--adam_eps=1e-5"]
    parser, _ = parse_sf_args(argv)
    cfg = parse_full_cfg(parser, argv)
    r = Runner(cfg)
    r.init()
    return r


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile-iters", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("resnet_bench needs a CUDA device")

    with tempfile.TemporaryDirectory() as train_dir:
        r = make_runner(train_dir)
        for _ in range(args.warmup):
            r.iteration()
        torch.cuda.synchronize()
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        steps0 = r.env_steps
        start.record()
        for _ in range(args.iters):
            r.iteration()
        end.record()
        torch.cuda.synchronize()
        seconds = start.elapsed_time(end) / 1e3
        steps = r.env_steps - steps0
        iter_ms = 1e3 * seconds / args.iters

        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.profile_iters):
                r.iteration()
            torch.cuda.synchronize()
        per_class = defaultdict(float)
        total_us = 0.0
        for ev in prof.events():
            if ev.device_type != torch.autograd.DeviceType.CUDA:
                continue
            us = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
            total_us += us
            cls = next((c for c, key in KERNEL_CLASSES if key in ev.name), "other")
            per_class[cls] += us
        spec = r.model.spec

    out = dict(
        metric="env-steps/s (sampler + learner), resnet_impala + FC 512, 1024 envs x [4,84,84] uint8",
        env_steps_per_s=steps / seconds,
        iteration_ms=iter_ms,
        timed_iterations=args.iters,
        env_steps_per_iteration=N_ENVS * ROLLOUT,
        conv_out_size=spec.conv_out_size,
        profiled_gpu_ms_per_iteration=total_us / 1e3 / max(1, args.profile_iters),
        kernel_share={k: round(v / total_us, 4) for k, v in sorted(per_class.items(), key=lambda kv: -kv[1])} if total_us else {},
        gpu=torch.cuda.get_device_name(0),
        power_limit_w=power_limit_w(),
    )
    print(json.dumps(out))


if __name__ == "__main__":
    main()
