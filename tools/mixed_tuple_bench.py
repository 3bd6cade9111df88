"""Throughput of Tuple action spaces with Box members (ModelSpec.action_heads) on the device path, and the profiled share
of the mixed kernels (heads_tail_rows_kernel, ppo_loss_mixed_kernel, action_ratio_mixed_kernel):

  (i)  4096 tape envs, Tuple(Discrete(5), Box(3), Discrete(3)) (14 distribution_linear rows), MLP 512-512, rollout 32,
       4 x 32768 minibatches
  (ii) the same with Tuple(Discrete(24), Box(8), Discrete(5)) (45 rows: the wide heads path)

    python tools/mixed_tuple_bench.py [--iters 5] [--warmup 2] [--engine 3xtf32]

One iteration = one rollout + one train(); env-steps/s = N*T per iteration over the mean CUDA-event time.  The card's
name and power limit are printed with the numbers."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import appo_oracle as O  # noqa: E402
from tests.test_gpu_engine import make_cfg  # noqa: E402

CASES = {
    "d5_b3_d3_mlp512": [("discrete", 5), ("box", 3), ("discrete", 3)],
    "d24_b8_d5_mlp512_wide": [("discrete", 24), ("box", 8), ("discrete", 5)],
}
MIXED_KERNELS = ("mixed", "heads_tail_rows")


def run(name, heads, iters, warmup, engine):
    from sample_factory_b200 import ops
    from sample_factory_b200.envs import TapeVecEnv
    from sample_factory_b200.learner import Learner
    from sample_factory_b200.model import ModelSpec, PolicyModel
    from sample_factory_b200.sampler import DeviceSampler
    from sample_factory_b200.trajectory import alloc_for_spec

    dev = torch.device("cuda", 0)
    N, T = 4096, 32
    rows = sum(n if k == "discrete" else 2 * n for k, n in heads)
    ocfg = O.OracleCfg(rollout=T, recurrence=1, num_epochs=1, num_actions=rows, encoder_mlp_layers=[512, 512],
                       batch_size=32768, num_batches_per_epoch=4)
    cfg = make_cfg(ocfg)
    spec = ModelSpec(ocfg.obs_dim, rows, [512, 512], action_heads=heads)
    model = PolicyModel(spec, dev)
    traj = alloc_for_spec(spec, N, T, dev)
    tape = torch.randn(T + 1, N, ocfg.obs_dim, generator=torch.Generator().manual_seed(0)).to(dev)
    env = TapeVecEnv(tape, rows, action_heads=heads)
    sampler = DeviceSampler(cfg, env, model, traj, engine=ops.ENGINES[engine], use_cuda_graph=True)
    learner = Learner(cfg, model, N, engine=ops.ENGINES[engine])
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
    total = mixed = 0.0
    for e in prof.key_averages():
        t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        total += t
        if any(k in e.key for k in MIXED_KERNELS):
            mixed += t
    return dict(case=name, env_steps_per_s=N * T / (ms / 1e3), ms_per_iter=ms, mixed_kernel_share=mixed / max(total, 1e-9),
                wide_heads=spec.wide_heads, heads_partials=sampler.heads_plan.P)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--engine", default="3xtf32", choices=["simt", "3xtf32"])
    a = ap.parse_args()
    from sample_factory_b200 import ops

    ops.bind_device(torch.device("cuda", 0))
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    for name, heads in CASES.items():
        print(json.dumps(dict(run(name, heads, a.iters, a.warmup, a.engine), device=card)), flush=True)


if __name__ == "__main__":
    main()
