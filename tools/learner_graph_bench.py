#!/usr/bin/env python
"""The learner launched kernel by kernel against the learner replayed as CUDA graphs (--learner_cuda_graph, one graph per
epoch), on the stacks of bench_configs.py configs 3, 4 and 5 (several epochs; kl_adaptive_epoch in 5).

  python tools/learner_graph_bench.py [--iters K] [--warmup W] [--profile-iters P] [--engine auto|3xtf32|simt]

Measured through tools/feature_bench.py's machinery (Runner, CUDA events around K iterations, kernel split, card read in
the same process), eager and graphed variants alternated, each twice.  Per variant two JSON lines: feature_bench's line
(ms_per_iter, env_steps_per_s, kernel_ms, ...) and a learner line:
  learner_ms_per_train     CUDA events around every train() of K more iterations (the span includes the device's waits
                           for the host's launches)
  kernel_launches          libsfb200 launches of the last train()
  graph_replay_launches    those of them replayed from graphs (0 eager)
  epochs_run               epochs of the last train() (early stopping)
Needs a CUDA device; writes nothing into the repository tree."""
from __future__ import annotations

import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

from tools import feature_bench as fb  # noqa: E402

CONFIGS = (3, 4, 5)


def variant(config: int, graph: bool) -> fb.Variant:
    """bench_configs.py config `config`'s envs, model and learner flags, the learner eager or replayed as CUDA graphs
    (the rollout is graphed in both; synchronous, so each iteration's train() runs alone on the GPU)"""
    import bench_configs

    c = bench_configs.CONFIGS[config]
    nmb = next(int(x.split("=")[1]) for x in c["flags"] if x.startswith("--num_batches_per_epoch"))
    rows = c["T"] + 1 if c["uint8"] else 2 * c["T"] + 1
    return fb.Variant(f"config{config}_{'graph' if graph else 'eager'}",
                      lambda: fb.tape_env(rows, c["envs"], c["obs_dim"], 77, c["A"], c["uint8"],
                                          continuous=c["continuous"], obs_shape=c["obs_shape"]),
                      [f"--rollout={c['T']}", f"--batch_size={c['envs'] * c['T'] // nmb}",
                       f"--learner_cuda_graph={graph}"] + c["flags"])


def facts(r, label):
    assert r.learner.use_graph == label.endswith("_graph")
    cfg = r.cfg
    return dict(num_epochs=cfg.num_epochs, num_batches_per_epoch=cfg.num_batches_per_epoch, lr_schedule=cfg.lr_schedule)


def learner_cost(r, label, args):
    """CUDA events around every Learner.train() of --iters more iterations, and the launches of the last train()"""
    learner, spans = r.learner, []
    real = learner.train

    def traced(batch):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = real(batch)
        b.record()
        spans.append((a, b))
        return out

    learner.train = traced
    try:
        for _ in range(args.iters):
            r.iteration()
        torch.cuda.synchronize()
    finally:
        del learner.train
    return [dict(learner_ms_per_train=sum(a.elapsed_time(b) for a, b in spans) / len(spans),
                 train_calls_timed=len(spans), kernel_launches=learner.kernel_launches,
                 graph_replay_launches=learner.graph_replay_launches,
                 epochs_run=learner.num_minibatches_done // r.cfg.num_batches_per_epoch)]


WORKLOAD = fb.Workload(
    [variant(c, g) for c in CONFIGS for g in (False, True)],
    fb.IMAGE_CLASSES + [("cell", "lstm_")],
    order=[f"config{c}_{m}" for c in CONFIGS for m in ("eager", "graph", "eager", "graph")],
    facts=facts, after_timing=learner_cost)


def main(argv=None) -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile-iters", type=int, default=1)
    ap.add_argument("--engine", default="auto", choices=["auto", "3xtf32", "simt"])
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("learner_graph_bench.py needs a CUDA device; there is no CPU fallback")
    fb.run_workload("learner_graph", WORKLOAD, args, fb.card())


if __name__ == "__main__":
    main()
