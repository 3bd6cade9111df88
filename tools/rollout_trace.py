"""Per-phase time of the persistent rollout kernel (csrc/rollout_fused.cu) on the bench.py workload (GPU box only).

Runs the headline workload (bench.make_cfg, the same synthetic tape env and sizes) through Runner with the kernel's
phase trace switched on (sfb200_rollout_set_trace): CTA (0, 0)'s first consumer thread stamps %globaltimer at the phase
boundaries of every step into a [T][16] buffer.  Prints, per step, the mean time of each phase over the steps of the
last --iters rollouts (step 0 left out: it includes the launch ramp), with the GPU's name and power limit, and writes
<out>/rollout_trace.json.  The stamps are one CTA's view; barrier phases include waiting for the cluster's slowest CTA.

  python tools/rollout_trace.py --out DIR [--iters 5] [--warmup 3] [--engine auto]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

# (name, first stamp slot, last stamp slot) -- the RF_TRACE slots of the kernel
PHASES = [("layer 1", 0, 3), ("barrier 1", 3, 4), ("layer 2 + heads", 4, 7), ("barrier 2", 7, 8), ("tail", 8, 9),
          ("barrier 3", 9, 10)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--engine", default="auto", choices=["auto", "3xtf32"])
    args = ap.parse_args()
    assert torch.cuda.is_available(), "rollout_trace.py needs a GPU"

    import bench
    from sample_factory_b200 import ops
    from sample_factory_b200._lib import lib
    from sample_factory_b200.envs import TapeVecEnv, register_env
    from sample_factory_b200.train import Runner

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    ops.bind_device(dev)
    gen = torch.Generator().manual_seed(1234)
    tape = torch.randn(bench.TAPE_LEN, bench.N_ENVS, bench.OBS_DIM, generator=gen).to(dev)
    register_env("synthetic_tape", lambda name, cfg, env_config, render_mode=None: TapeVecEnv(tape, bench.N_ACTIONS))
    T = bench.ROLLOUT
    trace = torch.zeros((T, 16), dtype=torch.int64, device=dev)
    # set before the first rollout: the sampler's CUDA graph captures the kernel arguments, the trace pointer included
    lib().call("sfb200_rollout_set_trace", trace.data_ptr())
    try:
        runner = Runner(bench.make_cfg("synthetic_tape", args.engine, True, learner_graph=True))
        runner.init()
        assert getattr(runner.sampler, "fused_rollout", False), "the bench workload did not take the persistent kernel"
        for _ in range(args.warmup):
            runner.iteration()
        torch.cuda.synchronize()
        sums = [0.0] * len(PHASES)
        count = 0
        for _ in range(args.iters):
            trace.zero_()
            runner.iteration()
            torch.cuda.synchronize()
            st = trace.cpu()
            for t in range(1, T):
                for i, (_, a, b) in enumerate(PHASES):
                    sums[i] += (int(st[t, b]) - int(st[t, a])) / 1e3
                count += 1
    finally:
        lib().call("sfb200_rollout_set_trace", None)
    form = {1: "fp16 split", 0: "tf32 split"}.get(ops.rollout_last_form(), "?")
    per = {name: round(s / count, 2) for (name, _, _), s in zip(PHASES, sums)}
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    total = sum(per.values())
    result = {"gpu": gpu, "workload": bench.WORKLOAD, "form": form, "rollouts": args.iters, "steps_per_rollout": T,
              "us_per_step": per, "us_per_step_total": round(total, 2)}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "rollout_trace.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(f"{gpu}: persistent rollout kernel, {form} form, us per step (mean of steps 1..{T - 1}, {args.iters} rollouts)")
    for name, v in per.items():
        print(f"  {name:16s} {v:8.2f}")
    print(f"  {'step':16s} {total:8.2f}")


if __name__ == "__main__":
    main()
