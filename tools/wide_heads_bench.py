"""Throughput of models with heads wider than 31 rows (ModelSpec.wide_heads) on the device path, and the profiled share of
the wide-heads kernels (sfb200_heads_tail_wide, the wide loss / ratio kernels, sfb200_heads_wide_backward):

  (i)  4096 tape envs, Discrete(362) with action masks, MLP 512-512, cfg-2's rollout (32) and batch (4 x 32768)
  (ii) Box(21) with the default adaptive stddev (42 distribution_linear rows), MLP 256-128-64

    python tools/wide_heads_bench.py [--iters 5] [--warmup 2] [--engine 3xtf32]

One iteration = one rollout + one train(); env-steps/s = N*T per iteration over the mean CUDA-event time."""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import appo_oracle as O  # noqa: E402
from tests.test_gpu_engine import build  # noqa: E402

CASES = {
    "discrete362_masked_mlp512": dict(N=4096, T=32, ocfg=dict(num_actions=362, action_mask=True, encoder_mlp_layers=[512, 512],
                                                              batch_size=32768, num_batches_per_epoch=4)),
    "box21_adaptive_mlp256_128_64": dict(N=4096, T=32, ocfg=dict(num_actions=21, continuous=True,
                                                                 encoder_mlp_layers=[256, 128, 64], batch_size=32768,
                                                                 num_batches_per_epoch=4)),
}
WIDE_KERNELS = ("wide", "heads_tail_rows")   # ppo_loss_*wide*, action_ratio_*wide*, heads_wide_backward_*, the stored-row tail


def run(name, spec, iters, warmup, engine):
    dev = torch.device("cuda", 0)
    N, T = spec["N"], spec["T"]
    ocfg = O.OracleCfg(rollout=T, recurrence=1, num_epochs=1, **spec["ocfg"])
    st0 = O.init_state(ocfg, seed=0)
    tape = torch.randn(T + 1, N, ocfg.obs_dim, generator=torch.Generator().manual_seed(0))
    cfg, model, traj, env, sampler, learner = build(ocfg, N, st0, tape, dev, engine=engine, graph=True)
    sampler.reset()

    def step():
        sampler.set_policy_version(learner.train_step)
        sampler.rollout()
        learner.train(traj)

    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        step()
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / iters
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    total = wide = 0.0
    for e in prof.key_averages():
        t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        total += t
        if any(k in e.key for k in WIDE_KERNELS):
            wide += t
    return dict(case=name, env_steps_per_s=N * T / (ms / 1e3), ms_per_iter=ms, wide_kernel_share=wide / max(total, 1e-9),
                device=torch.cuda.get_device_name(0), wide_heads=model.spec.wide_heads)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--engine", default="3xtf32", choices=["simt", "3xtf32"])
    a = ap.parse_args()
    from sample_factory_b200 import ops

    ops.bind_device(torch.device("cuda", 0))
    for name, spec in CASES.items():
        print(json.dumps(run(name, spec, a.iters, a.warmup, a.engine)), flush=True)


if __name__ == "__main__":
    main()
