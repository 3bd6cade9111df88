"""Worker for tests/test_gpu_multi.py (launched under torch.distributed.run, one process per GPU).

Checks the data-parallel contract of DESIGN.md section 6:  G ranks x N/G envs  ==  1 process x N envs, for
  A. the default multi-rank learner (NVLink peer-memory exchanges, csrc/comm.cu), kernels launched one by one,
  B. the same learner replayed as ONE CUDA graph (cfg.learner_cuda_graph=True, the default of bench.py),
  C. two epochs with the KL-adaptive learning-rate schedule (host decisions taken on all-reduced loss statistics: the
     replicas must agree on every learning rate and on the early-stopping decision),
  D. (SFB200_DP_TEST_NCCL=1) the torch.distributed / NCCL fallback path (SFB200_DP_COMM=nccl).
Rank 0 additionally trains a non-parallel learner on the concatenated batch and compares parameters, normalizer statistics,
loss terms and learning rates."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import appo_oracle as O  # noqa: E402  (only to build inputs: init weights + an oracle rollout)
from sample_factory_b200 import ops  # noqa: E402
from sample_factory_b200.dist_utils import init_from_env  # noqa: E402
from sample_factory_b200.learner import Learner  # noqa: E402
from sample_factory_b200.model import ModelSpec, PolicyModel  # noqa: E402
from sample_factory_b200.trajectory import alloc_trajectory_tensors  # noqa: E402
from tests.device_harness import make_cfg  # noqa: E402

N, T, NMB = 512, 16, 4
SUMMED = ["policy_loss", "value_loss", "exploration_loss", "kl_loss", "kl_old_mean", "entropy_mean", "value_mean",
          "total_loss", "fraction_clipped", "ratio_mean_abs_dev"]
EXACT = ["num_valid", "adv_mean", "adv_std", "kl_old_max", "ratio_min", "ratio_max"]


def main():
    rank, local_rank, world = init_from_env("nccl")
    dev = torch.device("cuda", local_rank)
    torch.cuda.set_device(dev)
    ops.bind_device(dev)
    engine = ops.GEMM_TC_3XTF32 if ops.tc_available() else ops.GEMM_SIMT
    base = dict(obs_dim=64, num_actions=8, encoder_mlp_layers=[256, 256], rollout=T, recurrence=1,
                num_batches_per_epoch=NMB, kl_loss_coeff=0.1)
    st0 = O.init_state(O.OracleCfg(batch_size=N * T // NMB, **base), seed=7)
    gen = torch.Generator().manual_seed(5)
    # three iterations of data from an oracle rollout (identical on every rank: same seeds)
    tape = torch.randn(3 * T + 1, N, 64, generator=gen)
    env = O.TapeVecEnv(tape, 8)
    last = env.reset()
    batches = []
    for it in range(3):
        traj = O.alloc_trajectories(O.OracleCfg(batch_size=N * T // NMB, **base), N)
        noise = torch.empty(T, N, 8).exponential_(generator=gen)
        last = O.rollout(O.OracleCfg(batch_size=N * T // NMB, **base), st0, env, last, traj, noise, 0)
        traj["policy_id"][torch.rand(N, T, generator=gen) < 0.1] = -1     # some invalid samples
        batches.append(traj)

    # env shard of this rank: the single-process minibatch b is envs [b*N/NMB, (b+1)*N/NMB); each rank takes its slice
    per_mb = N // NMB
    per_rank = per_mb // world
    idx = torch.cat([torch.arange(b * per_mb + rank * per_rank, b * per_mb + (rank + 1) * per_rank) for b in range(NMB)])
    spec = ModelSpec(64, 8, [256, 256])

    def run(parallel, graph=False, **over):
        n_envs = N // world if parallel else N
        ocfg = O.OracleCfg(batch_size=n_envs * T // NMB, **base)
        model = PolicyModel(spec, dev)
        model.load_state_dict(st0)
        traj_dev = alloc_trajectory_tensors(64, 8, n_envs, T, dev)
        learner = Learner(make_cfg(ocfg, learner_cuda_graph=graph, **over), model, n_envs, engine=engine,
                          data_parallel=parallel)
        assert learner.use_graph == graph, (learner.use_graph, graph)
        logs, lrs = [], []
        for b in batches:
            for k, v in b.items():
                traj_dev[k].copy_((v[idx] if parallel else v).view(traj_dev[k].shape))
            learner.train(traj_dev)
            logs.append(learner.minibatch_log().numpy().copy())
            lrs.append(learner.curr_lr)
        torch.cuda.synchronize()
        return model, learner, logs, lrs

    def norm_stats(m):
        return torch.cat([m.obs_mean, m.obs_var, m.ret_mean, m.ret_var])

    def replicas_identical(model, what):
        for t in (model.flat, norm_stats(model)):
            ref = t.clone()
            dist.broadcast(ref, src=0)
            assert torch.equal(t, ref), f"{what}: replicas diverged"

    def same_lrs(lrs):
        t = torch.tensor(lrs, dtype=torch.float64, device=dev)
        ref = t.clone()
        dist.broadcast(ref, src=0)
        assert torch.equal(t, ref), f"replicas use different learning rates: {lrs}"

    def check_vs_single(model_dp, logs_dp, lrs_dp, learner_dp, model_1, logs_1, lrs_1, learner_1, what, atol=2e-6):
        np.testing.assert_allclose(model_dp.flat.cpu().numpy(), model_1.flat.cpu().numpy(), atol=atol, err_msg=what)
        np.testing.assert_allclose(norm_stats(model_dp).cpu().numpy(), norm_stats(model_1).cpu().numpy(), rtol=1e-6, atol=1e-7)
        assert len(logs_dp) == len(logs_1)
        for l_dp, l_1 in zip(logs_dp, logs_1):
            assert l_dp.shape == l_1.shape, (what, l_dp.shape, l_1.shape)     # same early-stopping decision
            for key in EXACT:
                np.testing.assert_allclose(l_dp[:, ops.LS[key]], l_1[:, ops.LS[key]], rtol=1e-5, atol=1e-6, err_msg=f"{what} {key}")
            for key in SUMMED:    # global means = sum of the ranks' partial means (all-reduced loss statistics)
                np.testing.assert_allclose(l_dp[:, ops.LS[key]], l_1[:, ops.LS[key]], rtol=1e-4, atol=2e-6, err_msg=f"{what} {key}")
        np.testing.assert_allclose(lrs_dp, lrs_1, rtol=0, atol=0, err_msg=f"{what}: learning rates")
        assert learner_dp.env_steps == learner_1.env_steps and learner_dp.train_step == learner_1.train_step

    # ---- A: eager data parallel
    model_dp, learner_dp, logs_dp, lrs_dp = run(True)
    assert learner_dp.world_size == world
    use_peer = os.environ.get("SFB200_DP_COMM", "peer") != "nccl"
    assert (learner_dp.comm is not None) == use_peer
    replicas_identical(model_dp, "eager")

    # ---- B: the whole train() as one CUDA graph (call 1 eager, call 2 captures + replays, call 3 replays)
    if use_peer:
        model_g, learner_g, logs_g, _ = run(True, graph=True)
        assert learner_g._graph is not None and learner_g.graph_replay_launches > 0
        replicas_identical(model_g, "graph")
        np.testing.assert_allclose(model_g.flat.cpu().numpy(), model_dp.flat.cpu().numpy(), atol=1e-7, rtol=0)
        assert torch.equal(norm_stats(model_g), norm_stats(model_dp))
        for lg, ld in zip(logs_g, logs_dp):
            np.testing.assert_allclose(lg, ld, rtol=1e-6, atol=1e-7)
        assert learner_g.train_step == learner_dp.train_step and learner_g.env_steps == learner_dp.env_steps
        if rank == 0:
            print("DP_GRAPH_OK")

    # ---- C: two epochs, KL-adaptive learning rate per minibatch and per epoch (host decisions on global statistics)
    sched = {}
    for name in ("kl_adaptive_minibatch", "kl_adaptive_epoch"):
        over = dict(num_epochs=2, lr_schedule=name, lr_schedule_kl_threshold=1e-4, learning_rate=3e-4)
        sched[name] = run(True, **over) + (over,)
        replicas_identical(sched[name][0], name)
        same_lrs(sched[name][3])

    if rank == 0:
        model_1, learner_1, logs_1, lrs_1 = run(False)
        assert learner_1.world_size == 1
        check_vs_single(model_dp, logs_dp, lrs_dp, learner_dp, model_1, logs_1, lrs_1, learner_1, "eager")
        for name, (m, l, lg, lr, over) in sched.items():
            m1, l1, lg1, lr1 = run(False, **over)
            assert len(set(lr1)) > 1 or lr1[0] != over["learning_rate"], f"{name}: the schedule never moved ({lr1})"
            check_vs_single(m, lg, lr, l, m1, lg1, lr1, l1, name, atol=5e-6)
        print("DP_EQUIVALENCE_OK world", world, "engine", engine, "comm", "peer" if use_peer else "nccl")
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
