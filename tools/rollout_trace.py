"""Per-phase time of the persistent rollout kernel (csrc/rollout_fused.cu) on the bench.py workload (GPU box only).

Runs the headline workload (bench.make_cfg, the same synthetic tape env and sizes) through Runner with the kernel's
phase trace switched on (sfb200_rollout_set_trace): CTA (0, 0)'s first consumer thread stamps %globaltimer at the phase
boundaries of every step into a [T][32] buffer.  Prints, per step, the mean time of each phase over the steps of the
last --iters rollouts (step 0 left out: it includes the launch ramp), then of the sub-phases inside them (stages
landed, split, wgmmas, epilogues, the tail's partial sums and sampling), with the GPU's name and power limit, and writes
<out>/rollout_trace.json.  The stamps are one CTA's view; barrier phases include waiting for the cluster's slowest CTA.

In the fp16 form the layer-1 epilogue writes h1 into shared-memory staging boxes and stores them by TMA: "L1 epilogue"
ends when the staging is written (and the last box store issued), "L1 store drained" when the traced thread's bulk
stores have completed, just before it arrives at barrier 1.  (tf32 form: stores issued, then the proxy fence.)  Layer 2's
stages are stamped one by one when the consumer's wait for the stage returns: A and B complete one barrier, so they
are seen landing together; "L2 stage j landed" is the time since barrier 1 ended.

Every CTA also stamps its SM id and its entry / start (after the programmatic-dependency wait) / exit times: the tool
prints the spread of the start times, how many CTAs started more than one step after the first (a second wave: the
grid needs more clusters than the device holds at once, sfb200_rollout_occupancy), and the kernel's span against one
CTA's span.

  python tools/rollout_trace.py --out DIR [--iters 5] [--warmup 3] [--engine auto]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.feature_bench import card  # noqa: E402

import torch  # noqa: E402

# (name, first stamp slot, last stamp slot) -- the RF_TRACE slots of the kernel
PHASES = [("layer 1", 0, 3), ("barrier 1", 3, 4), ("layer 2 + heads", 4, 7), ("barrier 2", 7, 8), ("tail", 8, 9),
          ("barrier 3", 9, 10)]
# sub-phases inside them (slot 2: layer 1's split, 14: layer 2's split, stamped only by tiles that split in shared memory);
# a sub-phase is averaged over the steps that stamped both ends
SUBPHASES = [("L1 A landed", 0, 1), ("L1 split", 1, 2), ("L1 wgmmas", 2, 5), ("L1 wgmmas (no split)", 1, 5),
             ("L1 epilogue", 5, 6), ("L1 store drained", 6, 3), ("L2 stages", 4, 11), ("L2 last split", 11, 14),
             ("L2 last wgmmas", 14, 12), ("L2 last wgmmas (no split)", 11, 12), ("L2 heads epilogue", 12, 7),
             ("tail partials landed", 8, 13), ("tail sampling", 13, 15), ("tail stores", 15, 9)]
# slots 16 + j: layer-2 stage j landed (j < 16), reported relative to the end of barrier 1 (slot 4)
WORDS = 32
SUBPHASES += [(f"L2 stage {j} landed", 4, 16 + j) for j in range(16)]


def cta_summary(ctas, step_us):
    """per-CTA stamps of several rollouts -> start spread, late starters (more than a step after the first CTA), the
    kernel's span and a CTA's median span (means over the rollouts), the last rollout's stamps relative to its first
    start"""
    spread = late = span = cta_span = 0.0
    for rows in ctas:
        t0 = min(r[2] for r in rows)
        starts = [(r[2] - t0) / 1e3 for r in rows]
        spans = sorted((r[3] - r[2]) / 1e3 for r in rows)
        spread += max(starts)
        late += sum(s > step_us for s in starts)
        span += (max(r[3] for r in rows) - t0) / 1e3
        cta_span += spans[len(spans) // 2]
    n = len(ctas)
    last = ctas[-1]
    t0 = min(r[2] for r in last)
    late_last = sorted(((r[0], (r[2] - t0) / 1e3, (r[3] - r[2]) / 1e3) for r in last if (r[2] - t0) / 1e3 > step_us),
                       key=lambda x: x[1])
    return {"count": len(last), "start_spread_us": round(spread / n, 2), "late_starts": round(late / n, 2),
            "kernel_span_us": round(span / n, 1), "cta_span_us": round(cta_span / n, 1),
            "late": [(sm, round(st, 1), round(sp, 1)) for sm, st, sp in late_last],
            "last_rollout": [{"smid": r[0], "entry_us": round((r[1] - t0) / 1e3, 2), "start_us": round((r[2] - t0) / 1e3, 2),
                              "exit_us": round((r[3] - t0) / 1e3, 2)} for r in last]}


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
    T, N, H = bench.ROLLOUT, bench.N_ENVS, bench.HIDDEN[-1]
    n_words = T * WORDS + 4 * (N // 32 + 4)   # phase stamps, then four words per CTA (include/sfb200.h)
    trace = torch.zeros(n_words, dtype=torch.int64, device=dev)
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
        sub_sums = [0.0] * len(SUBPHASES)
        sub_counts = [0] * len(SUBPHASES)
        ctas = []   # per rollout: [(smid, entry, start, exit)] of every CTA that ran
        for _ in range(args.iters):
            trace.zero_()
            runner.iteration()
            torch.cuda.synchronize()
            flat = trace.cpu()
            st = flat[:T * WORDS].view(T, WORDS)
            for t in range(1, T):
                for i, (_, a, b) in enumerate(PHASES):
                    sums[i] += (int(st[t, b]) - int(st[t, a])) / 1e3
                count += 1
                for i, (_, a, b) in enumerate(SUBPHASES):
                    if int(st[t, a]) and int(st[t, b]):
                        sub_sums[i] += (int(st[t, b]) - int(st[t, a])) / 1e3
                        sub_counts[i] += 1
            c = flat[T * WORDS:].view(-1, 4).tolist()
            ctas.append([tuple(r) for r in c if r[2] != 0])
        act = ops.ACT[runner.sampler.model.spec.nonlinearity]
        needed, resident = ops.rollout_occupancy(N, bench.OBS_DIM, bench.HIDDEN[0], H, bench.N_ACTIONS,
                                                 runner.sampler.engine, act)
    finally:
        lib().call("sfb200_rollout_set_trace", None)
    form = {1: "fp16 split", 0: "tf32 split"}.get(ops.rollout_last_form(), "?")
    per = {name: round(s / count, 2) for (name, _, _), s in zip(PHASES, sums)}
    hw = card()
    sub = {name: round(v / n, 2) for (name, _, _), v, n in zip(SUBPHASES, sub_sums, sub_counts) if n}
    total = sum(per.values())
    waves = cta_summary(ctas, total)
    result = {**hw, "workload": bench.WORKLOAD, "form": form, "rollouts": args.iters, "steps_per_rollout": T,
              "us_per_step": per, "us_per_step_total": round(total, 2), "us_per_step_sub": sub,
              "occupancy": {"clusters_needed": needed, "clusters_resident": resident}, "ctas": waves}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "rollout_trace.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(f"{hw['gpu']} ({hw['power_limit_w']} W, {hw['max_sm_clock_mhz']} MHz): persistent rollout kernel, {form} form, "
          f"us per step (mean of steps 1..{T - 1}, {args.iters} rollouts)")
    for name, v in per.items():
        print(f"  {name:16s} {v:8.2f}")
    print(f"  {'step':16s} {total:8.2f}")
    print("sub-phases, us per step:")
    for name, v in sub.items():
        print(f"  {name:26s} {v:8.2f}")
    print(f"occupancy: {needed} clusters needed, {resident} resident at once")
    print(f"CTAs per rollout: {waves['count']}; start spread {waves['start_spread_us']:.2f} us; "
          f"{waves['late_starts']} started more than a step ({total:.1f} us) after the first; "
          f"kernel span {waves['kernel_span_us']:.1f} us vs one CTA's span {waves['cta_span_us']:.1f} us (means over "
          f"{args.iters} rollouts)")
    for sm, st, sp in waves["late"][:16]:
        print(f"  late CTA on SM {sm}: started {st:.1f} us after the first, ran {sp:.1f} us")


if __name__ == "__main__":
    main()
