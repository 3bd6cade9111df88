"""Where the GPU time of the bench.py workload goes, per kernel (GPU box only).

Runs the headline workload (bench.make_cfg, the same synthetic tape env and sizes) through Runner, records a few
iterations under torch.profiler with CUDA activities, and writes the GPU time per iteration of every kernel name to
<out>/learner_profile.json.  Kernel names keep their template arguments, so the forward, dX and dW instantiations of
gemm_wgmma_kernel<A_MN, B_MN, SPLIT3, HEADS, F16, RES> show up as separate rows.  Profile-only: take throughput numbers
from bench.py with the profiler off.

  python tools/learner_profile.py --out DIR [--iters 5] [--warmup 3] [--engine auto]
"""
from __future__ import annotations

import argparse
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.feature_bench import card  # noqa: E402

import torch  # noqa: E402


def kernel_key(name: str) -> str:
    """'void sfb::gemm_wgmma_kernel<true, true, true, false, false, false>(CUtensorMap, ...)' ->
    'gemm_wgmma_kernel<1,1,1,0,0,0>': namespace, return type and parameter list dropped, bool template args as 0/1."""
    depth, cut = 0, len(name)
    for i, ch in enumerate(name):          # the parameter list is the first '(' outside template brackets
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            cut = i
            break
    s = name[:cut].strip()
    if s.startswith("void "):
        s = s[5:]
    s = re.sub(r"\b\w+::", "", s)
    s = s.replace("true", "1").replace("false", "0").replace(" ", "")
    return s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--engine", default="auto", choices=["auto", "simt", "3xtf32", "tf32"])
    args = ap.parse_args()
    assert torch.cuda.is_available(), "learner_profile.py needs a GPU"

    import bench
    from sample_factory_b200 import ops
    from sample_factory_b200.envs import TapeVecEnv, register_env
    from sample_factory_b200.train import Runner

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    ops.bind_device(dev)
    gen = torch.Generator().manual_seed(1234)
    tape = torch.randn(bench.TAPE_LEN, bench.N_ENVS, bench.OBS_DIM, generator=gen).to(dev)
    register_env("synthetic_tape", lambda name, cfg, env_config, render_mode=None: TapeVecEnv(tape, bench.N_ACTIONS))
    runner = Runner(bench.make_cfg("synthetic_tape", args.engine, True, learner_graph=True))
    runner.init()
    for _ in range(args.warmup):
        runner.iteration()
    torch.cuda.synchronize()

    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.iters):
            runner.iteration()
        torch.cuda.synchronize()

    per = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        k = kernel_key(ev.name)
        d = per.setdefault(k, {"us_per_iter": 0.0, "launches_per_iter": 0.0})
        d["us_per_iter"] += ev.device_time_total / args.iters
        d["launches_per_iter"] += 1.0 / args.iters
    total = sum(d["us_per_iter"] for d in per.values())
    rows = sorted(per.items(), key=lambda kv: -kv[1]["us_per_iter"])
    hw = card()
    result = {
        **hw,
        "workload": bench.WORKLOAD,
        "iters": args.iters,
        "gpu_us_per_iter": total,
        "kernels": {k: {"us_per_iter": round(d["us_per_iter"], 2), "launches_per_iter": round(d["launches_per_iter"], 2),
                        "share": round(d["us_per_iter"] / total, 4)} for k, d in rows},
    }
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "learner_profile.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(f"{hw['gpu']} ({hw['power_limit_w']} W, {hw['max_sm_clock_mhz']} MHz): {total / 1e3:.3f} ms of kernel time per "
          "iteration")
    for k, d in rows[:20]:
        print(f"  {d['us_per_iter']:9.1f} us  {d['launches_per_iter']:6.1f} x  {k}")


if __name__ == "__main__":
    main()
