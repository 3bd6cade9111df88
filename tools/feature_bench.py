#!/usr/bin/env python
"""Throughput, kernel-time split and peak memory of each feature workload through the public Runner, all measured the
same way as bench.py.

  python tools/feature_bench.py --list
  python tools/feature_bench.py WORKLOAD [WORKLOAD ...] [--iters K] [--warmup W] [--profile-iters P]
                                [--engine auto|3xtf32|simt] [--dump-outputs DIR]
  python tools/feature_bench.py --all

One iteration = Runner.iteration() (one rollout + one train()).  Per variant: W warm-up iterations, a synchronise, CUDA
events around K timed iterations, a synchronise; then a separate torch.profiler pass of P iterations sorts the kernels into
the workload's classes (the first matching substring decides, the rest is "other").  One JSON line per variant:
  env_steps_per_s, ms_per_iter  N * T env steps per iteration over the event time
  kernel_ms, kernel_share       GPU time per iteration of each class, and its share of the profiled GPU time
  peak_allocated_gib            torch.cuda.max_memory_allocated() from the Runner's construction to the end of the variant
  gpu, power_limit_w, max_sm_clock_mhz   read by nvidia-smi in the same process
plus the workload's own facts.  The nofc workload adds its heads-routes lines, batched_tensor_env one ingest line per
adapter variant.  --dump-outputs DIR (rnn_layers) writes what the last timed iteration of each L computed to DIR/L<L>/.
Needs a CUDA device; writes nothing into the repository tree (each Runner's train_dir is a temporary directory)."""
from __future__ import annotations

import argparse
import functools
import json
import os
import shutil
import subprocess
import sys
import tempfile
from collections import defaultdict
from dataclasses import dataclass
from typing import Callable, Optional

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

BASE_ARGV = ["--restart_behavior=overwrite", "--batched_sampling=True", "--num_workers=1", "--num_envs_per_worker=1",
             "--worker_num_splits=1", "--seed=0", "--save_every_sec=1000000", "--experiment_summaries_interval=1000000",
             "--async_rl=False"]


def card() -> dict:
    """name, power limit and max SM clock of the current CUDA device (an nvidia-smi query; it changes no setting)"""
    uuid = torch.cuda.get_device_properties(torch.cuda.current_device()).uuid
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                          f"--id=GPU-{uuid}"], capture_output=True, text=True, check=True, timeout=60).stdout
    name, power, clock = (s.strip() for s in out.strip().splitlines()[0].split(","))
    return dict(gpu=name, power_limit_w=float(power), max_sm_clock_mhz=int(clock))


def full_argv(name: str, argv: list, train_dir: str, engine: str = "auto") -> list:
    return [f"--env={name}", f"--experiment={name}", f"--train_dir={train_dir}", f"--gemm_engine={engine}"] + BASE_ARGV + argv


def make_runner(name: str, env_factory: Callable, argv: list, engine: str = "auto"):
    """registers env_factory() as `name` and returns an initialised Runner on the base argv + argv"""
    from sample_factory_b200.cfg import parse_full_cfg, parse_sf_args
    from sample_factory_b200.envs import register_env
    from sample_factory_b200.train import Runner

    register_env(name, lambda full_env_name, cfg, env_config, render_mode=None: env_factory())
    argv = full_argv(name, argv, tempfile.mkdtemp(prefix="feature_bench_"), engine)
    parser, _ = parse_sf_args(argv)
    r = Runner(parse_full_cfg(parser, argv))
    r.init()
    return r


def timed(runner, iters: int, warmup: int):
    """bench.py's method: (ms per iteration, env-steps/s) over CUDA events around `iters` iterations after `warmup`"""
    for _ in range(warmup):
        runner.iteration()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        runner.iteration()
    end.record()
    torch.cuda.synchronize()
    ms = start.elapsed_time(end) / iters
    steps = sum(e.num_agents for e in runner.envs) * runner.cfg.rollout
    return ms, steps / (ms / 1e3)


def kernel_split(runner, classes: list, iters: int):
    """({class: GPU ms per iteration}, {class: share of the profiled GPU time}) over `iters` profiled iterations;
    classes = [(class, substring of the kernel's name), ...], the first match wins, unmatched kernels are "other"."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            runner.iteration()
        torch.cuda.synchronize()
    us = defaultdict(float)
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            us[next((c for c, key in classes if key in ev.name), "other")] += ev.device_time_total
    total = sum(us.values())
    order = sorted(us, key=lambda c: -us[c])
    return ({c: round(us[c] / 1e3 / iters, 3) for c in order}, {c: round(us[c] / total, 4) for c in order})


@functools.lru_cache(maxsize=None)
def tape(rows: int, n: int, width: int, seed: int, uint8: bool = False):
    """the observation tape of a TapeVecEnv on cuda:0 (cached within a workload: the image tapes take seconds to draw)"""
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(0, 256, (rows, n, width), dtype=torch.uint8, generator=g) if uint8 else \
        torch.randn(rows, n, width, generator=g)
    return t.to("cuda")


def tape_env(rows, n, width, seed, num_actions, uint8=False, **kw):
    from sample_factory_b200.envs import TapeVecEnv

    return TapeVecEnv(tape(rows, n, width, seed, uint8), num_actions, **kw)


@dataclass
class Variant:
    label: str
    env: Callable          # () -> env
    argv: list             # beyond BASE_ARGV


@dataclass
class Workload:
    variants: list
    classes: list                       # kernel classes, see kernel_split
    order: Optional[list] = None        # labels in the order they run (alternated samples); default: each once
    facts: Optional[Callable] = None    # (runner, label) -> extra fields of the line; asserts the feature path was taken
    after_timing: Optional[Callable] = None     # (runner, label, args) -> extra lines, between timing and profiling
    extra_lines: Optional[Callable] = None      # (args) -> lines measured once, before the variants


GEMM = [("gemm", "gemm_")]
RNN_CLASSES = GEMM + [("cell", "gru_"), ("cell", "lstm_"), ("cell", "mask_rows")]
FLAT_ARGV = ["--use_rnn=False", "--recurrence=1", "--rollout=32", "--batch_size=32768", "--num_batches_per_epoch=4"]
CFG5_ARGV = ["--use_rnn=True", "--rnn_type=lstm", "--rnn_size=512", "--rollout=16", "--recurrence=16",
             "--batch_size=32768", "--num_batches_per_epoch=2", "--num_epochs=2", "--encoder_mlp_layers", "512", "256",
             "128", "--value_bootstrap=True", "--reward_scale=0.01", "--max_grad_norm=1.0"]
IMAGE_ARGV = ["--num_epochs=1", "--nonlinearity=relu", "--obs_scale=255.0", "--exploration_loss_coeff=0.01",
              "--max_grad_norm=0.5", "--adam_eps=1e-5"]
IMAGE = (4, 84, 84)
IMAGE_CLASSES = [("im2col", "im2col"), ("col2im", "col2im"), ("maxpool_backward", "maxpool3s2_bwd"),
                 ("maxpool_forward", "maxpool3s2"), ("act_permute", "permute_bpc"), ("heads", "heads_"), ("rnn", "rnn_"),
                 ("gemm_wgmma", "gemm_wgmma"), ("gemm_simt", "gemm_simt"), ("gemm_splitk_reduce", "splitk_reduce"),
                 ("colsum", "colsum_"), ("adam", "adam"), ("loss", "loss")]


# ---------------------------------------------------------------------------------------------- batched_tensor_env
class BatchedTapeEnv:
    """TapeVecEnv's rules as a batched tensor env (IsaacGym / Brax style): one env, num_agents = N, fresh tensors from every
    reset() / step() (obs float32, reward float64, terminated int64, truncated uint8), on the GPU or on the CPU"""

    def __init__(self, inner, on_cpu):
        import numpy as np
        from gymnasium import spaces

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


def ingest_cost(r, label, args):
    """events around each sfb200_env_ingest call of one instrumented iteration (the span includes the host's enqueue
    latency whenever the device waits for the host), then the last step's launch 200 times back to back in one CUDA
    graph: the kernel's own time, and the bytes it reads and writes per step (from the tensors' shapes and dtypes)"""
    if label == "native":
        return []
    from sample_factory_b200 import ops

    real, pairs, moved, last = ops.env_ingest, [], [], []

    def traced(entries, rows):
        last[:] = [entries, rows]
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        real(entries, rows)
        b.record()
        pairs.append((a, b))
        moved.append(sum(rows * cols * (src.element_size() + dst.element_size()) for src, _, cols, dst, _, _ in entries))

    ops.env_ingest = traced
    try:
        r.iteration()
        torch.cuda.synchronize()
    finally:
        ops.env_ingest = real
    span = sum(a.elapsed_time(b) for a, b in pairs) / len(pairs)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(200):
            real(*last)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    g.replay()
    b.record()
    torch.cuda.synchronize()
    kernel_ms, nbytes = a.elapsed_time(b) / 200, sum(moved) / len(moved)
    return [dict(ingest_span_us_per_step=span * 1e3, ingest_kernel_us=kernel_ms * 1e3, ingest_bytes_per_step=nbytes,
                 ingest_kernel_gb_per_s=nbytes / (kernel_ms * 1e-3) / 1e9)]


def batched_env(label):
    inner = tape_env(65, 4096, 64, 2, 8)
    return inner if label == "native" else BatchedTapeEnv(inner, label == "cpu")


# -------------------------------------------------------------------------------------------------------- dict_obs
DICT_KEYS = [("achieved_goal", 3), ("desired_goal", 3), ("observation", 25)]


def encoder_flops_per_sample(n_key_mlps, obs=31, hidden=512):
    """forward FLOPs of the encoder MLPs [512, 512] for one sample (the first layers read the whole row in total)"""
    return 2 * (obs * hidden + n_key_mlps * hidden * hidden)


def dict_facts(r, label):
    assert r.model.spec.dict_obs == (label == "dict")
    return dict(encoder_flop_ratio_dict_over_single=encoder_flops_per_sample(len(DICT_KEYS)) / encoder_flops_per_sample(1))


# ------------------------------------------------------------------------------------------ mixed_tuple, wide_heads
def heads_facts(r, wide):
    spec, plan = r.model.spec, r.sampler.heads_plan
    assert spec.action_heads == r.env.action_heads and spec.continuous == r.env.continuous
    assert spec.wide_heads == wide and not (wide and plan.P), "wide heads take no fused head partials"
    return dict(wide_heads=spec.wide_heads, heads_partials=plan.P)


def mixed_variant(label, heads):
    rows = sum(n if kind == "discrete" else 2 * n for kind, n in heads)
    return Variant(label, lambda: tape_env(33, 4096, 64, 0, rows, action_heads=heads),
                   FLAT_ARGV + ["--encoder_mlp_layers", "512", "512"])


# ------------------------------------------------------------------------------------------------------------ nofc
def nofc_variant(arch, gru, fc):
    core = ["--use_rnn=True", "--rnn_type=gru", "--rnn_size=512", "--recurrence=32"] if gru else \
        ["--use_rnn=False", "--recurrence=1"]
    return Variant(f"{arch}_{'fc512' if fc else 'nofc'}_{'gru512' if gru else 'nocore'}",
                   lambda: tape_env(65, 1024, 28224, 0, 6, uint8=True, obs_shape=IMAGE),
                   ["--rollout=32", "--batch_size=8192", "--num_batches_per_epoch=4",
                    f"--encoder_conv_architecture={arch}", "--encoder_conv_mlp_layers"] + (["512"] if fc else []) +
                   IMAGE_ARGV + core)


def _events_ms(fn, reps=50, warm=5) -> float:
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def bench_heads_routes(args) -> list:
    """the two routes the learner can take for distribution_linear / critic_linear on conv features, H = 3136
    (convnet_atari) and 3872 (resnet_impala), 6 actions: the narrow warp-per-row kernels (heads_forward, heads_backward)
    against the wide route (the logits as a GEMM + heads_tail_wide, linear_backward + heads_wide_backward), forward of a
    learner minibatch and a sampler step, backward of a learner minibatch"""
    from sample_factory_b200 import ops

    dev = torch.device("cuda", 0)
    eng = ops.GEMM_TC_3XTF32 if ops.tc_available() else ops.GEMM_SIMT
    relu = ops.ACT["relu"]
    A, batch, n_envs = 6, 8192, 1024
    g = torch.Generator(device="cpu").manual_seed(0)
    out = []
    for H in (3136, 3872):
        Wv = (torch.randn(1, H, generator=g) / H ** 0.5).to(dev)
        Wa = (torch.randn(A, H, generator=g) / H ** 0.5).to(dev)
        bv, ba = torch.zeros(1, device=dev), torch.zeros(A, device=dev)
        gWv, gbv, gWa, gba = torch.empty_like(Wv), torch.empty_like(bv), torch.empty_like(Wa), torch.empty_like(ba)
        for rows in (batch, n_envs):
            h = torch.relu(torch.randn(rows, H, generator=g)).to(dev)
            values, logits = torch.empty(rows, device=dev), torch.empty((rows, A), device=dev)
            dlogits = (torch.randn(rows, A, generator=g) * 1e-3).to(dev)
            dvalues = (torch.randn(rows, generator=g) * 1e-3).to(dev)
            dz = torch.empty((rows, H), device=dev)
            ws_n = torch.empty(ops.heads_backward_workspace_bytes(H, A) // 4 + 4, device=dev)
            ws_w = torch.empty(ops.heads_wide_backward_workspace_bytes(rows, H, H, A) // 4 + 4, device=dev)
            lin_ws = torch.empty(ops.linear_backward_workspace_bytes(rows, A, H) // 4 + 4, device=dev)

            def narrow_fwd():
                ops.heads_forward(h, Wv, bv, Wa, ba, values, 1, logits, A)

            def wide_fwd():
                ops.linear_act_forward(h, Wa, ba, logits, ops.ACT["none"], eng)
                ops.heads_tail_wide(h, Wv, bv, logits, A, A, values=values, values_stride=1)

            def narrow_bwd():
                ops.heads_backward(h, Wv, Wa, dlogits, dvalues, relu, dz, gWv.view(-1), gbv, gWa, gba, None, ws_n)

            def wide_bwd():
                ops.linear_backward(dlogits, h, Wa, relu, gWa, dz, None, eng, lin_ws)
                ops.heads_wide_backward(h, Wv, dlogits, dvalues, relu, dz, 0, True, gWv.view(-1), gbv, gba, None, ws_w)

            row = dict(variant="heads_route", heads_route=f"H={H}, rows={rows}, {A} actions",
                       narrow_forward_ms=round(_events_ms(narrow_fwd), 4), wide_forward_ms=round(_events_ms(wide_fwd), 4))
            if rows == batch:
                row.update(narrow_backward_ms=round(_events_ms(narrow_bwd), 4),
                           wide_backward_ms=round(_events_ms(wide_bwd), 4),
                           narrow_backward_workspace_mib=round(ws_n.numel() * 4 / 2 ** 20, 1))
            out.append(row)
    return out


# ------------------------------------------------------------------------------------------------------ rnn_layers
DUMP_MAX_BYTES = 64 << 20


def dump_outputs(r, label, args):
    """DIR/<label>/<name>.npy per output of the last timed iteration: the trajectories (with the recurrent states, without
    the observation inputs), the learner's returns / advantages / minibatch log and the updated parameters; arrays beyond
    a quarter of the remaining 64 MB are cut to a fixed, seeded sample of rows (the same rows on every run)"""
    import numpy as np

    if not args.dump_outputs:
        return []
    out_dir = os.path.join(args.dump_outputs, label)
    os.makedirs(out_dir, exist_ok=True)
    torch.cuda.synchronize()
    arrays = {f"traj_{k}": v for k, v in r.traj.items() if k != "obs"}
    arrays["learner_returns"] = r.learner.returns
    arrays["learner_advantages"] = r.learner.advantages
    arrays["learner_minibatch_log"] = r.learner.minibatch_log()
    arrays["model_params"] = r.model.flat
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
    return []


def rnn_facts(r, label):
    layers = int(label[1:])
    assert r.traj["rnn_states"].shape[2] == 2 * 512 * layers
    return dict(rnn_num_layers=layers)


# ---------------------------------------------------------------------------------------------------- separate_rnn
def separate_facts(r, label):
    assert r.model.spec.share_weights == (label == "shared")
    return {}


# ------------------------------------------------------------------------------------------------------- the table
def _cfg5_env():
    return tape_env(33, 4096, 256, 2, 8)


WORKLOADS = {
    # config 2's model and sizes: the native device env against the same rules as a batched tensor env on the GPU
    # (device actions, one ingest launch per step) and on CPU tensors (numpy actions, pinned copies each way)
    "batched_tensor_env": Workload(
        [Variant(v, functools.partial(batched_env, v), FLAT_ARGV + ["--encoder_mlp_layers", "512", "512",
                                                                     f"--env_gpu_actions={v != 'cpu'}"])
         for v in ("native", "cuda", "cpu")],
        GEMM + [("ingest", "env_ingest")], after_timing=ingest_cost),
    # a Dict of keys (3, 3, 25) with one MLP [512, 512] per key against the same 31-float row as one key
    "dict_obs": Workload(
        [Variant(v, lambda keys=keys: tape_env(65, 4096, 31, 2, 8, obs_keys=keys),
                 FLAT_ARGV + ["--encoder_mlp_layers", "512", "512"])
         for v, keys in (("dict", DICT_KEYS), ("single", None))],
        GEMM, facts=dict_facts),
    # Tuple action spaces with Box members: 14 distribution_linear rows, and 45 (the wide heads path)
    "mixed_tuple": Workload(
        [mixed_variant("d5_b3_d3_mlp512", [("discrete", 5), ("box", 3), ("discrete", 3)]),
         mixed_variant("d24_b8_d5_mlp512_wide", [("discrete", 24), ("box", 8), ("discrete", 5)])],
        [("mixed", "mixed"), ("mixed", "heads_tail_rows")], facts=lambda r, v: heads_facts(r, v.endswith("_wide"))),
    # image encoders with and without their FC layer, each with no core and with a GRU-512
    "nofc": Workload(
        [nofc_variant(arch, gru, fc) for arch in ("convnet_atari", "resnet_impala") for gru in (False, True)
         for fc in (True, False)],
        IMAGE_CLASSES, facts=lambda r, v: dict(heads_input=r.model.spec.tail_input_size,
                                               wide_heads=r.model.spec.wide_heads),
        extra_lines=bench_heads_routes),
    "resnet": Workload(
        [Variant("resnet_impala_fc512", lambda: tape_env(33, 1024, 28224, 0, 6, uint8=True, obs_shape=IMAGE),
                 ["--use_rnn=False", "--rollout=16", "--recurrence=1", "--batch_size=4096", "--num_batches_per_epoch=4",
                  "--encoder_conv_architecture=resnet_impala", "--encoder_conv_mlp_layers", "512"] + IMAGE_ARGV)],
        IMAGE_CLASSES, facts=lambda r, v: dict(conv_out_size=r.model.spec.conv_out_size)),
    # config 5's stack with L stacked LSTM layers; L = 1 passes no --rnn_num_layers flag
    "rnn_layers": Workload(
        [Variant(f"L{n}", _cfg5_env, CFG5_ARGV + ["--lr_schedule=kl_adaptive_epoch", "--lr_schedule_kl_threshold=0.016"] +
                 ([f"--rnn_num_layers={n}"] if n > 1 else [])) for n in (1, 2, 3)],
        RNN_CLASSES, facts=rnn_facts, after_timing=dump_outputs),
    # config 5's stack with one encoder and core, and with one per tower
    "separate_rnn": Workload(
        [Variant(v, _cfg5_env, CFG5_ARGV + [f"--actor_critic_share_weights={v == 'shared'}"])
         for v in ("shared", "separate")],
        GEMM + [("cell", "gru_"), ("cell", "lstm_")], order=["shared", "separate", "shared", "separate"],
        facts=separate_facts),
    # heads wider than 31 rows: Discrete(362) with action masks; Box(21) with adaptive stddev (42 rows)
    "wide_heads": Workload(
        [Variant("discrete362_masked_mlp512", lambda: tape_env(33, 4096, 64, 0, 362, with_action_mask=True),
                 FLAT_ARGV + ["--encoder_mlp_layers", "512", "512"]),
         Variant("box21_adaptive_mlp256_128_64", lambda: tape_env(33, 4096, 64, 0, 21, continuous=True),
                 FLAT_ARGV + ["--encoder_mlp_layers", "256", "128", "64"])],
        [("wide", "wide"), ("wide", "heads_tail_rows")], facts=lambda r, v: heads_facts(r, True)),
}


def run_workload(name: str, w: Workload, args, hw: dict) -> None:
    def emit(line):
        print(json.dumps(dict(workload=name, **line, **hw)), flush=True)

    for line in w.extra_lines(args) if w.extra_lines else []:
        emit(line)
    variants = {v.label: v for v in w.variants}
    for label in w.order or list(variants):
        v = variants[label]
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        r = make_runner(f"{name}_{label}", v.env, v.argv, args.engine)
        try:
            facts = w.facts(r, label) if w.facts else {}
            ms, rate = timed(r, args.iters, args.warmup)
            extra = w.after_timing(r, label, args) if w.after_timing else []
            kernel_ms, kernel_share = kernel_split(r, w.classes, args.profile_iters)
            emit(dict(variant=label, env_steps_per_s=rate, ms_per_iter=ms, kernel_ms=kernel_ms, kernel_share=kernel_share,
                      peak_allocated_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 3), **facts))
            for line in extra:
                emit(dict(variant=label, **line))
        finally:
            shutil.rmtree(r.cfg.train_dir, ignore_errors=True)
            del r
    tape.cache_clear()


def main(argv=None) -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("workloads", nargs="*", metavar="WORKLOAD")
    ap.add_argument("--list", action="store_true", help="print the workloads and their variants")
    ap.add_argument("--all", action="store_true", help="run every workload")
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile-iters", type=int, default=1)
    ap.add_argument("--engine", default="auto", choices=["auto", "3xtf32", "simt"])
    ap.add_argument("--dump-outputs", default=None, metavar="DIR", help="rnn_layers: write each L's outputs to DIR/L<L>/")
    args = ap.parse_args(argv)
    if args.list:
        for name, w in WORKLOADS.items():
            print(f"{name}: {', '.join(v.label for v in w.variants)}")
        return
    names = list(WORKLOADS) if args.all else args.workloads
    if not names or set(names) - set(WORKLOADS):
        ap.error(f"name workloads among {', '.join(WORKLOADS)}, or pass --all or --list")
    if not torch.cuda.is_available():
        raise SystemExit("feature_bench.py needs a CUDA device; there is no CPU fallback")
    hw = card()
    for name in names:
        run_workload(name, WORKLOADS[name], args, hw)


if __name__ == "__main__":
    main()
