"""The persistent rollout kernel (csrc/rollout_fused.cu: producer warpgroup, TMA ring, fp16 weight twins and h1 handed
over already split) against the per-step launches with the fused step tail, at the shapes the kernel's ring and
decomposition distinguish: the bench shape in both operand forms, clusters of 1 / 2 / 4 CTAs, one to four layer-1
stages, partial row blocks, odd step counts (ring phases), one action, weights that move between rollouts, and a
CUDA-graph replay.  Comparison rule of test_gpu_engine._compare_rollout_runs: everything bit-identical except logits /
values / log-probs (2e-6)."""
import os
import subprocess
import sys

import pytest
import torch

from oracle import appo_oracle as O
from tests.test_gpu_engine import _compare_rollout_runs, build

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _pair(ocfg, N, seed, graph=False):
    """one model, two samplers over identical envs: per-step launches (fused tail) and the persistent kernel"""
    from sample_factory_b200 import ops
    from sample_factory_b200.envs import TapeVecEnv
    from sample_factory_b200.sampler import DeviceSampler
    from sample_factory_b200.trajectory import alloc_for_spec

    dev = torch.device("cuda", 0)
    ops.bind_device(dev)
    if not ops.tc_available():
        pytest.skip("wgmma engine not available")
    st0 = O.init_state(ocfg, seed=seed)
    tape = torch.randn(2 * ocfg.rollout + 3, N, ocfg.obs_dim, generator=torch.Generator().manual_seed(seed + 1))
    old = {k: os.environ.get(k) for k in ("SFB200_TAIL_FUSED", "SFB200_ROLLOUT_FUSED")}
    try:
        os.environ["SFB200_TAIL_FUSED"] = "1"
        os.environ["SFB200_ROLLOUT_FUSED"] = "0"
        cfg, model, traj_s, env_s, sampler_s, learner = build(ocfg, N, st0, tape, dev, engine="3xtf32")
        os.environ["SFB200_ROLLOUT_FUSED"] = "1"
        traj_p = alloc_for_spec(model.spec, N, ocfg.rollout, dev)
        env_p = TapeVecEnv(tape.to(dev).contiguous(), ocfg.num_actions)
        sampler_p = DeviceSampler(cfg, env_p, model, traj_p, engine=ops.GEMM_TC_3XTF32, use_cuda_graph=graph)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    assert sampler_s.fused_tail and not sampler_s.fused_rollout
    assert sampler_p.fused_rollout
    return model, learner, (sampler_s, traj_s, env_s), (sampler_p, traj_p, env_p)


def _state(sampler, traj, env):
    return dict(traj=[{k: v.clone() for k, v in traj.items()}], obs=env.obs.clone(), rew=env.rew.clone(),
                term=env.terminated.clone(), step=env.step_counter.clone(), pstep=sampler.step_counter.clone(),
                stats=sampler.episode_stats.clone(), ep=(sampler.ep_return.clone(), sampler.ep_len.clone()))


def _check(obs_dim=64, hidden=512, num_actions=8, N=512, T=4, rollouts=2, train=False, graph=False, form=None,
           normalize=True, nonlinearity="elu"):
    """rollouts of both samplers compared after each one (train: learner.train on the persistent trajectories in between,
    so the weights, their fp16 twins and the h1 bound change); form: the operand form the kernel must have taken;
    normalize=False: a model without fp16 twins (every GEMM of both paths in the tf32 form)"""
    from sample_factory_b200 import ops

    ocfg = O.OracleCfg(obs_dim=obs_dim, num_actions=num_actions, encoder_mlp_layers=[hidden, hidden], rollout=T,
                       recurrence=1, batch_size=N * T // 2, num_batches_per_epoch=2, normalize_input=normalize,
                       nonlinearity=nonlinearity)
    model, learner, (ss, ts, es), (sp, tp, ep) = _pair(ocfg, N, seed=3 + hidden + obs_dim + N + T, graph=graph)
    ss.reset()
    sp.reset()
    if graph:
        ss.rollout()   # the graphed sampler's first rollout() also runs its eager warm-up rollout
    for it in range(rollouts):
        for k in tp:          # what a rollout does not write (the bootstrap value column, learner outputs) alike
            ts[k].copy_(tp[k])
        ss.set_policy_version(it)
        sp.set_policy_version(it)
        ss.rollout()
        sp.rollout()
        if form is not None:
            assert ops.rollout_last_form() == form
        torch.cuda.synchronize()
        _compare_rollout_runs(_state(ss, ts, es), _state(sp, tp, ep), f"rollout {it}")
        if train:
            learner.train(tp)
    if graph:
        assert sp.graph_replay_launches == 2


def test_bench_shape_fp16_form():
    _check(N=4096, T=32, form=1)


def test_bench_shape_tf32_form():
    """SFB200_TC_F16=0 is read once per process: the same check in a fresh one"""
    code = ("import sys; sys.path.insert(0, sys.argv[1]); from tests.test_gpu_rollout_pipeline import _check; "
            "_check(N=4096, T=32, form=0); print('ok')")
    env = dict(os.environ, SFB200_TC_F16="0")
    res = subprocess.run([sys.executable, "-c", code, ROOT], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0 and "ok" in res.stdout, res.stdout[-3000:] + res.stderr[-3000:]


@pytest.mark.parametrize("form", ["fp16", "tf32"])
@pytest.mark.parametrize("act", ["relu", "tanh"])
def test_activations(act, form):
    """rollout_mlp2_tape_kernel<ACT, F16> for ReLU (unbounded: the fp16 form splits h1 by a bound that grows with the
    weights) and tanh (h1 bound capped at 1 by linear_out_bound); the tf32 form in a fresh process, as above"""
    if form == "fp16":
        _check(N=1000, T=5, form=1, nonlinearity=act)
        return
    code = ("import sys; sys.path.insert(0, sys.argv[1]); from tests.test_gpu_rollout_pipeline import _check; "
            f"_check(N=1000, T=5, form=0, nonlinearity={act!r}); print('ok')")
    env = dict(os.environ, SFB200_TC_F16="0")
    res = subprocess.run([sys.executable, "-c", code, ROOT], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0 and "ok" in res.stdout, res.stdout[-3000:] + res.stderr[-3000:]


@pytest.mark.parametrize("hidden", [128, 256])
def test_cluster_sizes(hidden):
    _check(hidden=hidden, N=1000, T=5, form=1)


@pytest.mark.parametrize("obs_dim,form", [(32, 0), (96, 0), (128, 1)])
def test_obs_dims(obs_dim, form):
    """K1 = 32 / 96 take the tf32 form (stages of 32 k); the per-step layer 2 would take the fp16 form from the twins, so
    those run a model without twins, where both paths split in tf32.  K1 = 128: two fp16 layer-1 stages."""
    _check(obs_dim=obs_dim, N=1000, T=5, form=form, normalize=form == 1)


@pytest.mark.parametrize("N", [1000, 100])
def test_partial_row_blocks(N):
    _check(N=N, T=6, form=1)


@pytest.mark.parametrize("T", [1, 3])
def test_odd_step_counts(T):
    _check(N=1000, T=T, rollouts=3, form=1)


def test_one_action():
    _check(num_actions=1, N=1000, T=5, form=1)


def test_weights_move_between_rollouts():
    _check(N=1000, T=8, rollouts=3, train=True, form=1)


def test_cuda_graph_replay():
    _check(N=1000, T=6, rollouts=3, graph=True, form=1)
