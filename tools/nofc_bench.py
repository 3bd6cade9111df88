#!/usr/bin/env python
"""Image encoders with and without their fully connected layer (--encoder_conv_mlp_layers 512 vs empty) through the
public Runner: 1024 device tape envs, uint8 [4, 84, 84] frames, ReLU, obs_scale 255, rollout 32, batch 8192 x 4
minibatches x 1 epoch; convnet_atari and resnet_impala, each with no core and with a GRU-512 (recurrence 32).

  python tools/nofc_bench.py [--iters K] [--warmup W] [--profile-iters P]

Prints one JSON line per model and one for the heads routes:
  env_steps_per_s     env steps / s over K timed iterations (rollout + learner), CUDA events around the window
  kernel_ms           GPU time per iteration of each kernel class (torch.profiler, a separate run after the timed window)
  peak_allocated_gib  torch.cuda.max_memory_allocated() from the Runner's construction to the end of the run
  heads routes        forward + backward of critic_linear / distribution_linear on [rows, H] features, H = 3136 (convnet_atari)
                      and 3872 (resnet_impala), 6 actions: the narrow warp-per-row kernels (heads_forward, heads_backward)
                      against the wide route (the logits as a GEMM on the wgmma engine + heads_tail_wide, linear_backward +
                      heads_wide_backward); CUDA events over 50 repetitions after 5 warm-up ones
  gpu, power_limit_w  read in the same run
Needs a CUDA device; writes nothing into the repository tree (the Runner's train_dir is a temporary directory)."""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

from tools.resnet_bench import power_limit_w  # noqa: E402

N_ENVS, ROLLOUT, SHAPE, N_ACTIONS, BATCH = 1024, 32, (4, 84, 84), 6, 8192

KERNEL_CLASSES = [  # (class, substring of the kernel's name), first match wins
    ("im2col", "im2col"),
    ("col2im", "col2im"),
    ("maxpool", "maxpool3s2"),
    ("act_permute", "permute_bpc"),
    ("heads", "heads_"),
    ("rnn", "rnn_"),
    ("gemm_wgmma", "gemm_wgmma"),
    ("gemm_simt", "gemm_simt"),
    ("gemm_splitk_reduce", "splitk_reduce"),
    ("colsum", "colsum_"),
    ("adam", "adam"),
    ("loss", "loss"),
]


def make_runner(train_dir: str, tape, arch: str, fc: bool, gru: bool):
    from sample_factory_b200.cfg import parse_full_cfg, parse_sf_args
    from sample_factory_b200.envs import TapeVecEnv, register_env
    from sample_factory_b200.train import Runner

    name = f"nofc_bench_{arch}_{int(fc)}_{int(gru)}"
    register_env(name, lambda full_env_name, cfg, env_config, render_mode=None: TapeVecEnv(tape, N_ACTIONS, obs_shape=SHAPE))
    core = ["--use_rnn=True", "--rnn_type=gru", "--rnn_size=512", f"--recurrence={ROLLOUT}"] if gru else \
        ["--use_rnn=False", "--recurrence=1"]
    argv = [f"--env={name}", f"--experiment={name}", f"--train_dir={train_dir}", "--restart_behavior=overwrite",
            "--batched_sampling=True", "--num_workers=1", "--num_envs_per_worker=1", "--worker_num_splits=1", "--seed=0",
            "--save_every_sec=1000000", "--experiment_summaries_interval=1000000", "--async_rl=False",
            f"--rollout={ROLLOUT}", f"--batch_size={BATCH}", "--num_batches_per_epoch=4", "--num_epochs=1",
            f"--encoder_conv_architecture={arch}", "--encoder_conv_mlp_layers"] + (["512"] if fc else []) + [
            "--nonlinearity=relu", "--obs_scale=255.0", "--exploration_loss_coeff=0.01", "--max_grad_norm=0.5",
            "--adam_eps=1e-5"] + core
    parser, _ = parse_sf_args(argv)
    cfg = parse_full_cfg(parser, argv)
    r = Runner(cfg)
    r.init()
    return r


def bench_model(args, tape, arch: str, fc: bool, gru: bool) -> dict:
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    with tempfile.TemporaryDirectory() as train_dir:
        r = make_runner(train_dir, tape, arch, fc, gru)
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

        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.profile_iters):
                r.iteration()
            torch.cuda.synchronize()
        per_class = defaultdict(float)
        for ev in prof.events():
            if ev.device_type != torch.autograd.DeviceType.CUDA:
                continue
            us = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
            per_class[next((c for c, key in KERNEL_CLASSES if key in ev.name), "other")] += us
        spec = r.model.spec
        out = dict(model=f"{arch} {'+ FC 512' if fc else 'without FC'}, {'GRU-512' if gru else 'no core'}",
                   env_steps_per_s=steps / seconds, iteration_ms=1e3 * seconds / args.iters,
                   heads_input=spec.tail_input_size, wide_heads=spec.wide_heads,
                   kernel_ms={k: round(v / 1e3 / args.profile_iters, 3)
                              for k, v in sorted(per_class.items(), key=lambda kv: -kv[1])},
                   peak_allocated_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 3))
        del r
    return out


def _time(fn, reps=50, warm=5) -> float:
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


def bench_heads_routes() -> list:
    """the two routes the learner can take for distribution_linear / critic_linear on conv features (forward of a
    learner minibatch and a sampler step, backward of a learner minibatch)"""
    from sample_factory_b200 import ops

    dev = torch.device("cuda", 0)
    eng = ops.GEMM_TC_3XTF32 if ops.tc_available() else ops.GEMM_SIMT
    relu = ops.ACT["relu"]
    A = N_ACTIONS
    g = torch.Generator(device="cpu").manual_seed(0)
    out = []
    for H in (3136, 3872):
        Wv = (torch.randn(1, H, generator=g) / H ** 0.5).to(dev)
        Wa = (torch.randn(A, H, generator=g) / H ** 0.5).to(dev)
        bv, ba = torch.zeros(1, device=dev), torch.zeros(A, device=dev)
        gWv, gbv, gWa, gba = torch.empty_like(Wv), torch.empty_like(bv), torch.empty_like(Wa), torch.empty_like(ba)
        for rows in (BATCH, N_ENVS):
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

            row = dict(heads_route=f"H={H}, rows={rows}, {A} actions",
                       narrow_forward_ms=round(_time(narrow_fwd), 4), wide_forward_ms=round(_time(wide_fwd), 4))
            if rows == BATCH:
                row.update(narrow_backward_ms=round(_time(narrow_bwd), 4), wide_backward_ms=round(_time(wide_bwd), 4),
                           narrow_backward_workspace_mib=round(ws_n.numel() * 4 / 2 ** 20, 1))
            out.append(row)
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile-iters", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("nofc_bench needs a CUDA device")
    from sample_factory_b200 import ops

    ops.bind_device(torch.device("cuda", 0))
    hw = dict(gpu=torch.cuda.get_device_name(0), power_limit_w=power_limit_w())
    for row in bench_heads_routes():
        print(json.dumps(dict(row, **hw)), flush=True)
    gen = torch.Generator().manual_seed(0)
    tape = torch.randint(0, 256, (2 * ROLLOUT + 1, N_ENVS, SHAPE[0] * SHAPE[1] * SHAPE[2]), dtype=torch.uint8,
                         generator=gen).to("cuda")
    for arch in ("convnet_atari", "resnet_impala"):
        for gru in (False, True):
            for fc in (True, False):
                print(json.dumps(dict(bench_model(args, tape, arch, fc, gru), **hw)), flush=True)


if __name__ == "__main__":
    main()
