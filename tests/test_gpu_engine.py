"""End-to-end parity of the device engine (DeviceSampler + Learner, through the C ABI) against
  (a) the committed golden vectors produced by the reference itself (tests/golden/*.npz), and
  (b) the CPU oracle on larger seeded inputs,
plus size-independent properties at BASELINE.json's full size (N=4096, T=32)."""
import numpy as np
import pytest
import torch

from oracle import appo_oracle as O
from tests.device_harness import (DEV, ENGINES, TOL, build, build_case, compare_rollout_runs, graphed_sampler_matches_eager,
                                  make_cfg, need, ops_for, replay_learner, replay_sampler)
from tests.golden_utils import load_case

pytestmark = pytest.mark.gpu


GOLDEN_CASES = ["tiny_gae", "tiny_vtrace", "tiny_gru", "tiny_lstm", "cfg2_small", "tiny_gauss", "tiny_gauss_adaptive", "tiny_conv", "tiny_symkl", "tiny_lamb", "tiny_tuple", "tiny_separate", "tiny_mask"]


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_rollout_matches_reference_golden(name, engine):
    """Sampler vs the REFERENCE's own trajectories (same weights, same obs tape, same Exp(1) noise)."""
    case = load_case(name)
    replay_sampler(case, build_case(case, engine))


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_learner_matches_reference_golden(name, engine):
    """Learner.train on the REFERENCE's trajectories: returns / advantages / loss terms / post-Adam weights /
    normalizer statistics against what the reference itself computed."""
    case = load_case(name)
    replay_learner(case, build_case(case, engine), rewards=True)


@pytest.mark.parametrize("engine", ENGINES)
def test_closed_loop_vs_oracle_cfg2_shape(engine):
    """Sampler + learner for 2 iterations at N=256, T=32, cfg-2 model/hyper-parameters vs the oracle run on the same
    tape / noise / initial weights (the tape env keeps both rollouts aligned)."""
    from sample_factory_b200 import ops

    N, T = 256, 32
    ocfg = O.OracleCfg(rollout=T, recurrence=1, batch_size=N * T // 4, num_batches_per_epoch=4, num_epochs=1)
    st0 = O.init_state(ocfg, seed=3)
    gen = torch.Generator().manual_seed(11)
    tape = torch.randn(2 * T + 1, N, ocfg.obs_dim, generator=gen) * 1.2 - 0.2
    need(engine)
    cfg, model, traj, env, sampler, learner = build(ocfg, N, st0, tape, engine=engine)
    olearner = O.OracleLearner(ocfg, st0)
    oenv = O.TapeVecEnv(tape, ocfg.num_actions)
    olast = oenv.reset()
    sampler.reset()
    for it in range(2):
        noise = torch.empty(T, N, ocfg.num_actions).exponential_(generator=gen)
        otraj = O.alloc_trajectories(ocfg, N)
        olast = O.rollout(ocfg, olearner.st, oenv, olast, otraj, noise, olearner.train_step)
        sampler.noise = noise.to(DEV)
        sampler.set_policy_version(learner.train_step)
        sampler.rollout()
        got = {k: v.cpu() for k, v in traj.items()}
        mism = (got["actions"] != otraj["actions"]).float().mean().item()
        assert mism == 0.0, f"action mismatch fraction {mism}"
        for k in ["obs", "rewards", "dones", "time_outs", "policy_id", "policy_version"]:
            assert torch.equal(got[k], otraj[k]), k
        np.testing.assert_allclose(got["action_logits"].numpy(), otraj["action_logits"].numpy(), atol=TOL)
        np.testing.assert_allclose(got["values"][:, :-1].numpy(), otraj["values"][:, :-1].numpy(), atol=TOL)
        n0 = len(olearner.log)
        buff = olearner.train(otraj)
        learner.train(traj)
        np.testing.assert_allclose(learner.returns.view(-1).cpu().numpy(), buff["returns"].numpy(), atol=TOL)
        np.testing.assert_allclose(learner.advantages.view(-1).cpu().numpy(), buff["advantages"].numpy(), atol=TOL)
        log = learner.minibatch_log().numpy()
        for j, d in enumerate(olearner.log[n0:]):
            for key in ["policy_loss", "value_loss", "exploration_loss", "kl_loss"]:
                assert abs(log[j, ops.LS[key]] - d[key]) < TOL, (it, j, key, log[j, ops.LS[key]], d[key])
            assert abs(learner.grad_norm_log[j].item() - d["grad_norm"]) < 1e-4
        sd = model.state_dict()
        for k in O.param_names(ocfg):
            np.testing.assert_allclose(sd[k].cpu().numpy(), olearner.st[k].numpy(), atol=TOL, err_msg=k)


def test_full_size_properties_and_graph_replay():
    """N=4096, T=32 (BASELINE.json config 2): size-independent properties.
    * CUDA-graph replay and eager execution of the same rollout produce identical trajectories (Philox noise is a
      pure function of (seed, env, step) and both counters live on the device)
    * GAE linearity in the rewards; value targets = adv + values; returns-normaliser round trip
    * a training iteration changes the weights, keeps everything finite, and leaves padding untouched."""
    from sample_factory_b200 import ops

    N, T = 4096, 32
    ocfg = O.OracleCfg(rollout=T, recurrence=1, batch_size=N * T // 4, num_batches_per_epoch=4)
    st0 = O.init_state(ocfg, seed=5)
    tape = torch.randn(3 * T + 1, N, ocfg.obs_dim, generator=torch.Generator().manual_seed(12))
    A = build(ocfg, N, st0, tape)
    graphed_sampler_matches_eager(A, build(ocfg, N, st0, tape, graph=True))
    modelA, trajA, learnerA = A.model, A.traj, A.learner
    a = trajA["actions"]
    assert a.min().item() >= 0 and a.max().item() <= ocfg.num_actions - 1
    assert torch.all(trajA["policy_id"] == 0) and torch.isfinite(trajA["action_logits"]).all()
    freq = torch.bincount(a.view(-1).long(), minlength=ocfg.num_actions).float() / a.numel()
    assert freq.min().item() > 0.01, "every action should be sampled under near-uniform initial logits"

    # GAE linearity at full size
    r1 = torch.randn(N, T, device=DEV)
    r2 = torch.randn(N, T, device=DEV)
    dones = trajA["dones"]
    zeros_v = torch.zeros(N, T + 1, device=DEV)
    ones_valid = torch.ones(N, T + 1, dtype=torch.bool, device=DEV)
    outs = []
    for r in (r1, r2, r1 + r2):
        adv = torch.empty(N, T, device=DEV)
        ret = torch.empty(N, T, device=DEV)
        ops.gae_returns(r.clone(), dones, trajA["time_outs"], zeros_v, ones_valid, 0.99, 0.95, False, None, None, adv, ret)
        outs.append(adv)
        assert torch.equal(adv, ret)   # values == 0 -> returns == advantages
    assert (outs[0] + outs[1] - outs[2]).abs().max().item() < 1e-4

    before = modelA.flat.clone()
    learnerA.train(trajA)
    torch.cuda.synchronize()
    assert torch.isfinite(modelA.flat).all() and not torch.equal(before, modelA.flat)
    stats = learnerA.fetch_stats()
    assert all(np.isfinite(v) for v in stats.values()), stats
    assert stats["num_valid"] == N * T // 4
    assert torch.isfinite(learnerA.advantages).all() and torch.isfinite(learnerA.returns).all()
    # padding between tensors in the flat buffer must stay zero (zero grad -> zero Adam update)
    mask = torch.ones_like(modelA.flat, dtype=torch.bool)
    for n in modelA.names:
        o, shp = modelA._slices[n]
        mask[o:o + int(np.prod(shp))] = False
    assert torch.all(modelA.flat[mask] == 0)


def test_action_mask_graph_replay_and_mask_respected():
    """Action-mask env (obs dict) under the production path: in-kernel Philox noise, CUDA-graph replay == eager, every
    sampled action is allowed by the mask of its step (rows that allow nothing excepted), and the fused GEMM + heads path
    (hidden 128) honours the mask too."""
    N, T = 512, 16
    ocfg = O.OracleCfg(obs_dim=32, num_actions=8, encoder_mlp_layers=[128, 128], rollout=T, recurrence=1,
                       batch_size=N * T // 2, num_batches_per_epoch=2, action_mask=True)
    st0 = O.init_state(ocfg, seed=6)
    tape = torch.randn(3 * T + 1, N, ocfg.obs_dim, generator=torch.Generator().manual_seed(13))
    engine = "3xtf32" if ops_for().tc_available() else "simt"
    B = build(ocfg, N, st0, tape, engine, graph=True)
    graphed_sampler_matches_eager(build(ocfg, N, st0, tape, engine), B)
    trajB = B.traj
    a = trajB["actions"][:, :, 0].cpu().long()
    env_idx = torch.arange(N)
    some_allowed = torch.zeros(N, T, dtype=torch.bool)
    for t in range(T):
        m = O.tape_action_mask(t, env_idx, ocfg.num_actions)
        some_allowed[:, t] = m.sum(1) > 0
        ok = m.gather(1, a[:, t:t + 1]).view(-1).bool() | ~some_allowed[:, t]
        assert bool(ok.all()), f"forbidden action sampled at step {t}"
    assert int(some_allowed.sum()) > 0.9 * N * T and not bool(some_allowed.all())
    # log-probs are the masked ones: exp(lp) sums over allowed actions only -> lp >= unmasked log-softmax of the action
    lg = trajB["action_logits"].cpu()
    lp_unmasked = torch.log_softmax(lg, -1).gather(2, a.unsqueeze(-1)).squeeze(-1)
    assert bool((trajB["log_prob_actions"].cpu() >= lp_unmasked - 1e-5)[some_allowed].all())
    np.testing.assert_allclose(trajB["log_prob_actions"].cpu()[~some_allowed].numpy(), -np.log(ocfg.num_actions), atol=1e-6)


def test_async_double_buffered_runner_matches_lagged_oracle(tmp_path):
    """async_rl=True (train.py): the sampler collects rollout i+1 on its own stream with a weight snapshot while the
    learner trains on rollout i.  The schedule is deterministic, so the oracle can replay it: rollout r is sampled
    with the weights published at the join before it (r0, r1 <- W0; r2 <- W after train(0); ...), stamped with that
    version, and trained on one iteration later (policy lag = 4 SGD steps, inside max_policy_lag)."""
    import copy

    from sample_factory_b200 import ops
    from sample_factory_b200.envs import TapeVecEnv, register_env
    from sample_factory_b200.train import Runner

    N, T, ITERS = 128, 16, 3
    ocfg = O.OracleCfg(obs_dim=32, num_actions=8, encoder_mlp_layers=[128, 128], rollout=T, recurrence=1,
                       batch_size=N * T // 4, num_batches_per_epoch=4, num_epochs=1)
    st0 = O.init_state(ocfg, seed=13)
    gen = torch.Generator().manual_seed(17)
    tape = torch.randn((ITERS + 1) * T + 1, N, ocfg.obs_dim, generator=gen)
    noises = [torch.empty(T, N, ocfg.num_actions).exponential_(generator=gen) for _ in range(ITERS + 1)]
    register_env("async_tape", lambda n, c, e, render_mode=None: TapeVecEnv(tape.to(DEV).contiguous(), ocfg.num_actions))
    cfg = make_cfg(ocfg, env="async_tape", train_dir=str(tmp_path), experiment="async", cuda_graph=False, seed=0,
                   gemm_engine="simt", async_rl=True, restart_behavior="overwrite")
    runner = Runner(cfg)
    assert runner.init() == 0
    runner.load_state_dict(st0)
    runner.rollout_hook = lambda r: setattr(runner.sampler, "noise", noises[r].to(DEV))

    olearner = O.OracleLearner(ocfg, copy.deepcopy(st0))
    oenv = O.TapeVecEnv(tape, ocfg.num_actions)
    olast = oenv.reset()
    snap, snap_version = copy.deepcopy(olearner.st), 0
    pending = O.alloc_trajectories(ocfg, N)
    olast = O.rollout(ocfg, snap, oenv, olast, pending, noises[0], snap_version)      # priming rollout
    for it in range(ITERS):
        runner.iteration()
        torch.cuda.synchronize()
        nxt = O.alloc_trajectories(ocfg, N)
        olast = O.rollout(ocfg, snap, oenv, olast, nxt, noises[it + 1], snap_version)   # overlaps train(it) on the device
        olearner.train(pending)
        snap, snap_version = copy.deepcopy(olearner.st), olearner.train_step              # the join
        # the learner's buffer now holds rollout it+1, sampled with the PREVIOUS snapshot
        got = {k: v.cpu() for k, v in runner.traj.items()}
        for k in ["obs", "actions", "rewards", "dones", "policy_version"]:
            assert torch.equal(got[k], nxt[k]), (it, k)
        np.testing.assert_allclose(got["action_logits"].numpy(), nxt["action_logits"].numpy(), atol=TOL)
        sd = runner.model.state_dict()
        for k in O.param_names(ocfg):
            np.testing.assert_allclose(sd[k].cpu().numpy(), olearner.st[k].numpy(), atol=TOL, err_msg=f"{it} {k}")
        assert runner.learner.train_step == olearner.train_step == 4 * (it + 1)
        pending = nxt
    assert runner.rollouts_started == ITERS + 1 and runner.env_steps == ITERS * N * T
    lag = runner.learner.train_step - got["policy_version"].max().item()
    assert lag == 4.0      # samples in the buffer are one iteration (4 SGD steps) behind the learner


def test_split_sampler_matches_single_sampler():
    """worker_num_splits = 2 (two env groups on two streams, one graph) fills the trajectory buffers exactly like one
    sampler over all envs: same weights, same tape, same explicit noise -> identical trajectories (eager), and the
    graph-captured fork/join rollout reproduces the eager one with Philox noise."""
    from sample_factory_b200 import ops
    from sample_factory_b200.envs import TapeVecEnv
    from sample_factory_b200.sampler import DeviceSampler, SplitSampler

    N, T = 256, 8
    ocfg = O.OracleCfg(rollout=T, recurrence=1, batch_size=N * T, num_batches_per_epoch=1, encoder_mlp_layers=[128, 128])
    st0 = O.init_state(ocfg, seed=8)
    tape = (torch.randn(2 * T + 1, N, ocfg.obs_dim, generator=torch.Generator().manual_seed(5)) * 1.1).to(DEV)
    cfg, model, traj, env, sampler, _ = build(ocfg, N, st0, tape.cpu(), engine="3xtf32" if ops.tc_available() else "simt")
    eng = sampler.engine
    noise = torch.empty(T, N, ocfg.num_actions).exponential_(generator=torch.Generator().manual_seed(9)).to(DEV)
    sampler.reset()
    sampler.noise = noise
    sampler.rollout()
    ref = {k: v.clone() for k, v in traj.items()}
    for v in traj.values():
        v.zero_()
    h = N // 2
    envs = [TapeVecEnv(tape[:, :h].contiguous(), ocfg.num_actions, env_index_offset=0),
            TapeVecEnv(tape[:, h:].contiguous(), ocfg.num_actions, env_index_offset=h)]
    split = SplitSampler(cfg, envs, model, traj, engine=eng, use_cuda_graph=False)
    split.reset()
    split.noise = noise
    split.rollout()
    torch.cuda.synchronize()
    for k in ref:
        if k == "valids":
            continue
        if k == "values":      # column T (bootstrap value) belongs to the learner
            assert torch.equal(traj[k][:, :T], ref[k][:, :T]), k
            continue
        assert torch.equal(traj[k], ref[k]), k
    # graph-captured fork / join: replays are deterministic functions of (weights, tape, Philox counters)
    def run(use_graph, n):
        es = [TapeVecEnv(tape[:, :h].contiguous(), ocfg.num_actions, env_index_offset=0),
              TapeVecEnv(tape[:, h:].contiguous(), ocfg.num_actions, env_index_offset=h)]
        sp = SplitSampler(cfg, es, model, traj, engine=eng, use_cuda_graph=use_graph, philox_seed=3)
        sp.reset()
        outs = []
        for _ in range(n):
            sp.rollout()
            torch.cuda.synchronize()
            outs.append({k: traj[k].clone() for k in ("actions", "values", "rewards", "dones", "obs")})
        return outs, sp
    eager, _ = run(False, 4)
    graphed, sp = run(True, 3)
    assert sp.graph_replay_launches > 0
    # the graph path runs one un-captured warm-up rollout first (its trajectories are overwritten by the first replay), so
    # replay i continues from env step / Philox offset (i+1)*T
    for a, b in zip(eager[1:], graphed):
        for k in a:
            assert torch.equal(a[k], b[k]), k


@pytest.mark.parametrize("use_graph", [False, True])
def test_double_buffered_host_sampling_matches_one_group_after_the_other(use_graph):
    """worker_num_splits = 2 over HOST envs (rollout_worker.py:97-143): stepping the two env groups interleaved -- the GPU serves
    one group on its own stream while the host simulates the other -- fills the trajectory buffers exactly like running the
    groups' rollouts one after the other (same weights, tapes, Philox streams), with per-step launches and with per-step graphs"""
    from sample_factory_b200 import ops
    from sample_factory_b200.envs import HostTapeVecEnv
    from sample_factory_b200.sampler import SplitSampler

    N, T = 256, 8
    ocfg = O.OracleCfg(rollout=T, recurrence=1, batch_size=N * T, num_batches_per_epoch=1, encoder_mlp_layers=[128, 128])
    st0 = O.init_state(ocfg, seed=8)
    tape = torch.randn(5 * T + 1, N, ocfg.obs_dim, generator=torch.Generator().manual_seed(5)) * 1.1
    cfg, model, traj, env, sampler, _ = build(ocfg, N, st0, tape, engine="3xtf32" if ops.tc_available() else "simt")
    h = N // 2

    def run(interleaved, n):
        es = [HostTapeVecEnv(tape[:, :h].contiguous().numpy(), ocfg.num_actions, DEV, env_index_offset=0),
              HostTapeVecEnv(tape[:, h:].contiguous().numpy(), ocfg.num_actions, DEV, env_index_offset=h)]
        sp = SplitSampler(cfg, es, model, traj, engine=sampler.engine, use_cuda_graph=use_graph, philox_seed=3)
        assert sp.host_interleaved
        if not interleaved:
            sp.host_interleaved = False      # the groups' whole rollouts one after the other (sub-samplers on their streams)
        sp.reset()
        outs = []
        for _ in range(n):
            sp.rollout()
            torch.cuda.synchronize()
            outs.append({k: traj[k].clone() for k in ("actions", "values", "rewards", "dones", "obs", "policy_version")})
        return outs, sp

    seq, _ = run(False, 4)
    inter, sp = run(True, 4)
    if use_graph:
        assert all(s._step_graphs is not None for s in sp.subs) and sp.graph_replay_launches > 0
    for a, b in zip(seq, inter):
        for k in a:
            if k == "values":
                assert torch.equal(a[k][:, :T], b[k][:, :T]), k
            else:
                assert torch.equal(a[k], b[k]), k


def test_graphed_learner_matches_eager():
    """cfg.learner_cuda_graph: Learner.train() replayed as ONE CUDA graph (device-resident step counters / lr) produces the
    same parameters, Adam moments and loss statistics as the launch-by-launch learner, iteration after iteration."""
    from sample_factory_b200 import ops

    N, T = 128, 8
    ocfg = O.OracleCfg(rollout=T, recurrence=1, batch_size=N * T // 2, num_batches_per_epoch=2, encoder_mlp_layers=[128, 128])
    st0 = O.init_state(ocfg, seed=2)
    tape = torch.randn(6 * T + 1, N, ocfg.obs_dim, generator=torch.Generator().manual_seed(3))
    eng = "3xtf32" if ops.tc_available() else "simt"
    cfgA, modelA, trajA, envA, samplerA, learnerA = build(ocfg, N, st0, tape, engine=eng)
    cfgB, modelB, trajB, envB, samplerB, learnerB = build(ocfg, N, st0, tape, engine=eng, learner_cuda_graph=True)
    assert learnerB.use_graph and not learnerA.use_graph
    samplerA.reset()
    for it in range(5):
        noise = torch.empty(T, N, ocfg.num_actions).exponential_(generator=torch.Generator().manual_seed(20 + it)).to(DEV)
        samplerA.noise = noise
        samplerA.set_policy_version(learnerA.train_step)
        samplerA.rollout()
        for k in trajA:
            trajB[k].copy_(trajA[k])
        learnerA.train(trajA)
        learnerB.train(trajB)
        torch.cuda.synchronize()
        assert learnerA.train_step == learnerB.train_step == 2 * (it + 1)
        assert torch.equal(modelA.flat, modelB.flat), it
        assert torch.equal(modelA.exp_avg_sq, modelB.exp_avg_sq) and torch.equal(modelA.obs_mean, modelB.obs_mean)
        assert torch.equal(learnerA.minibatch_log(), learnerB.minibatch_log())
        sa, sb = learnerA.fetch_stats(), learnerB.fetch_stats()
        assert sa["grad_norm"] == sb["grad_norm"] and sa["loss"] == sb["loss"]
    assert learnerB.graph_replay_launches > 0 and learnerB.kernel_launches == learnerA.kernel_launches + 2  # + advance_counters


@pytest.mark.parametrize("explicit_noise", [True, False])
def test_fused_tail_and_rollout_match_separate_launches(explicit_noise, monkeypatch):
    """The per-layer GEMMs followed by ONE step-tail launch (csrc/heads.cu sampler_tail_tape_kernel: heads finish +
    sampling + tape-env step + post-step(t) + pre-step(t+1)), and the whole rollout as one persistent kernel
    (csrc/rollout_fused.cu), produce the same trajectories, episode statistics, env state and next policy input as the
    per-layer / per-stage launches: bit-identical for everything downstream of the logits (same device functions),
    logits / values at rounding level."""
    need("3xtf32")
    N, T = 1000, 12
    ocfg = O.OracleCfg(rollout=T, recurrence=1, batch_size=N * T // 4, num_batches_per_epoch=4)
    st0 = O.init_state(ocfg, seed=9)
    gen = torch.Generator().manual_seed(3)
    tape = torch.randn(2 * T + 1, N, ocfg.obs_dim, generator=gen)
    noise = torch.empty(T, N, ocfg.num_actions).exponential_(generator=gen).to(DEV)
    runs = {}
    for mode in ("separate", "tail", "persistent"):
        monkeypatch.setenv("SFB200_TAIL_FUSED", "0" if mode == "separate" else "1")
        monkeypatch.setenv("SFB200_ROLLOUT_FUSED", "1" if mode == "persistent" else "0")
        cfg, model, traj, env, sampler, learner = build(ocfg, N, st0, tape, engine="3xtf32")
        assert sampler.fused_tail == (mode != "separate")
        assert sampler.fused_rollout == (mode == "persistent")
        sampler.reset()
        out = []
        for it in range(2):
            if explicit_noise:
                sampler.noise = noise
            sampler.set_policy_version(5 + it)
            sampler.rollout()
            out.append({k: v.clone() for k, v in traj.items()})
        torch.cuda.synchronize()
        runs[mode] = dict(traj=out, x_norm=sampler.x_norm.clone(), obs=env.obs.clone(), rew=env.rew.clone(),
                          term=env.terminated.clone(), step=env.step_counter.clone(), pstep=sampler.step_counter.clone(),
                          stats=sampler.episode_stats.clone(), ep=(sampler.ep_return.clone(), sampler.ep_len.clone()),
                          launches=sampler.kernel_launches_per_rollout)
    launches = {mode: r["launches"] for mode, r in runs.items()}
    assert launches["separate"] > launches["tail"] > launches["persistent"], launches
    assert launches["persistent"] == 2, launches     # pre-step(0) + ONE kernel for T steps
    for other in ("tail", "persistent"):
        compare_rollout_runs(runs["separate"], runs[other], other)


@pytest.mark.parametrize("rnn", [False, True])
@pytest.mark.parametrize("engine", ENGINES)
def test_shuffle_minibatches_matches_oracle(engine, rnn):
    """cfg.shuffle_minibatches (learner.py:498-526, a new permutation every epoch :707-713): the same permutations of
    recurrence-length chunks on both sides -> same minibatches -> same losses and post-Adam weights; with a recurrent core the
    chunks keep their BPTT structure."""
    from sample_factory_b200 import ops

    need(engine)
    N, T = 64, 16
    R = 8 if rnn else 1
    kw = dict(use_rnn=True, rnn_type="gru", rnn_size=64, recurrence=R) if rnn else dict(recurrence=1)
    ocfg = O.OracleCfg(obs_dim=24, num_actions=5, encoder_mlp_layers=[128, 128], rollout=T, batch_size=N * T // 4,
                       num_batches_per_epoch=4, num_epochs=2, **kw)
    st0 = O.init_state(ocfg, seed=2)
    gen = torch.Generator().manual_seed(8)
    tape = torch.randn(T + 1, N, ocfg.obs_dim, generator=gen)
    cfg, model, traj, env, sampler, learner = build(ocfg, N, st0, tape, engine=engine, shuffle_minibatches=True)
    assert learner.shuffle
    olearner = O.OracleLearner(ocfg, st0)
    oenv = O.TapeVecEnv(tape, ocfg.num_actions)
    otraj = O.alloc_trajectories(ocfg, N)
    noise = torch.empty(T, N, ocfg.num_actions).exponential_(generator=gen)
    O.rollout(ocfg, olearner.st, oenv, oenv.reset(), otraj, noise, 0)
    otraj["policy_id"][torch.rand(N, T, generator=gen) < 0.1] = -1
    for k, v in otraj.items():
        if k in traj:
            traj[k].copy_(v.view(traj[k].shape))
    E = N * T
    rng = np.random.RandomState(4)
    perms = []
    for _ in range(ocfg.num_epochs):
        starts = rng.permutation(np.arange(0, E, R))
        perms.append((starts[:, None] + np.arange(R)[None, :]).reshape(-1))
    assert not np.array_equal(perms[0], perms[1])
    learner.set_minibatch_permutation(np.stack(perms))
    buff = olearner.train(otraj, mb_indices=[torch.from_numpy(p) for p in perms])
    learner.train(traj)
    log = learner.minibatch_log().numpy()
    assert log.shape[0] == len(olearner.log) == 8
    for j, d in enumerate(olearner.log):
        for key in ["policy_loss", "value_loss", "exploration_loss", "kl_loss"]:
            assert abs(log[j, ops.LS[key]] - d[key]) < TOL, (j, key, log[j, ops.LS[key]], d[key])
        assert abs(log[j, ops.LS["adv_mean"]] - d["adv_mean"]) < TOL
    sd = model.state_dict()
    for k in O.param_names(ocfg):
        np.testing.assert_allclose(sd[k].cpu().numpy(), olearner.st[k].numpy(), atol=2e-5, err_msg=k)
    # without an explicit permutation every train() draws its own (np.random, like the reference)
    np.random.seed(0)
    learner.train(traj)
    p1 = learner.perm_host.clone()
    learner.train(traj)
    assert not torch.equal(p1, learner.perm_host) and torch.equal(torch.sort(p1.long())[0], torch.arange(E))
    assert torch.isfinite(model.flat).all()
