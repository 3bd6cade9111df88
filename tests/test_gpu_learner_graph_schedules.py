"""The learner replayed as CUDA graphs (cfg.learner_cuda_graph) for every learning-rate schedule, several epochs and LAMB:
one graph per epoch, the per-minibatch learning-rate rules on the device (sfb200_lr_schedule_step), LAMB's step counter
and learning rate in device memory (sfb200_clip_lamb_step_dev).  Each case runs an eager and a graphed learner from the
same state on the same trajectories, and they must agree bit for bit: parameters, both Adam moments, the minibatch loss
rows, the learning-rate sequence and the counters."""
import math

import numpy as np
import pytest
import torch

from oracle import appo_oracle as O
from tests.device_harness import DEV, ENGINES, build, ops_for, sampled_feed

pytestmark = pytest.mark.gpu

N, T, NMB = 128, 8, 2
B = N * T // NMB
SCHEDULES = ["constant", "kl_adaptive_minibatch", "kl_adaptive_epoch", "linear_decay"]


def _ocfg(**kw):
    base = dict(obs_dim=24, num_actions=5, encoder_mlp_layers=[64, 64], rollout=T, recurrence=1, batch_size=B,
                num_batches_per_epoch=NMB, kl_loss_coeff=0.1)
    base.update(kw)
    return O.OracleCfg(**base)


def _pair(ocfg, engine, seed=0, **over):
    """an eager and a graphed rig from the same initial weights over the same tape"""
    st0 = O.init_state(ocfg, seed=seed)
    tape = torch.randn(4 * T + 1, N, ocfg.obs_dim, generator=torch.Generator().manual_seed(seed + 1))
    a = build(ocfg, N, st0, tape, engine, **over)
    b = build(ocfg, N, st0, tape, engine, learner_cuda_graph=True, **over)
    assert b.learner.use_graph and not a.learner.use_graph
    return a, b


def _same_state(a, b, what):
    for name in ("flat", "exp_avg", "exp_avg_sq", "obs_mean", "obs_var"):
        assert torch.equal(getattr(a.model, name), getattr(b.model, name)), (what, name)
    assert torch.equal(a.learner.minibatch_log(), b.learner.minibatch_log()), what
    la, lb = a.learner, b.learner
    assert (la.train_step, la.opt_step, la.num_minibatches_done, la.env_steps) == \
           (lb.train_step, lb.opt_step, lb.num_minibatches_done, lb.env_steps), what


def _run(a, b, iters=4, perms=None):
    """train both learners `iters` times on the same rollouts of a's sampler -> the eager learner's lr sequence"""
    feed = sampled_feed(a, b)
    lrs = []
    for it in range(iters):
        feed(it)
        if perms is not None:
            for r in (a, b):
                r.learner.set_minibatch_permutation(perms[it])
        a.learner.train(a.traj)
        b.learner.train(b.traj)
        torch.cuda.synchronize()
        _same_state(a, b, it)
        assert a.learner.curr_lr == b.learner.curr_lr, (it, a.learner.curr_lr, b.learner.curr_lr)
        if hasattr(a.learner.lr_scheduler, "step"):
            assert a.learner.lr_scheduler.step == b.learner.lr_scheduler.step
        lrs.append(a.learner.curr_lr)
    assert b.learner.graph_replay_launches > 0
    return lrs


def _schedule_over(schedule, epochs):
    over = dict(lr_schedule=schedule, num_epochs=epochs, learning_rate=3e-4)
    if schedule.startswith("kl_adaptive"):
        over["lr_schedule_kl_threshold"] = 1e-5        # the KL of these updates is well above 2x: the rate moves
    if schedule == "linear_decay":
        # num_updates = 6 * epochs of the 8 * epochs minibatch steps of four train() calls: reaches 0 within the run
        over["train_for_env_steps"] = 6 * B
    return over


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("epochs", [1, 3])
@pytest.mark.parametrize("schedule", SCHEDULES)
def test_graphed_schedules_match_eager(schedule, epochs, engine):
    ops_for(engine)
    a, b = _pair(_ocfg(num_epochs=epochs), engine, **_schedule_over(schedule, epochs))
    lrs = _run(a, b)
    if schedule.startswith("kl_adaptive"):
        assert len(set(lrs)) > 1 or lrs[0] != 3e-4, lrs
    if schedule == "linear_decay":
        assert lrs[-1] == 0.0 and 0.0 < lrs[0] < 3e-4, lrs
    if schedule == "constant":
        assert lrs == [3e-4] * 4


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("epochs", [1, 2])
def test_graphed_lamb_matches_eager(epochs, engine):
    ops_for(engine)
    a, b = _pair(_ocfg(num_epochs=epochs, optimizer="lamb"), engine, optimizer="lamb", num_epochs=epochs)
    _run(a, b)


def test_graphed_shuffled_epochs_match_eager():
    """shuffle_minibatches with 3 epochs: each later epoch's graph holds the re-gather and the advantage partials"""
    ops = ops_for("simt")
    eng = "3xtf32" if ops.tc_available() else "simt"
    a, b = _pair(_ocfg(num_epochs=3), eng, num_epochs=3, shuffle_minibatches=True)
    rng = np.random.default_rng(4)
    perms = [np.stack([rng.permutation(N * T) for _ in range(3)]) for _ in range(4)]
    _run(a, b, perms=perms)


def test_graphed_recurrent_kl_adaptive_epoch_matches_eager():
    """config 5's shape at a small size: a GRU core, recurrence = rollout, kl_adaptive_epoch over 2 epochs"""
    ops = ops_for("simt")
    eng = "3xtf32" if ops.tc_available() else "simt"
    ocfg = _ocfg(use_rnn=True, rnn_type="gru", rnn_size=32, recurrence=T, num_epochs=2)
    a, b = _pair(ocfg, eng, **_schedule_over("kl_adaptive_epoch", 2))
    lrs = _run(a, b)
    assert len(set(lrs)) > 1 or lrs[0] != 3e-4, lrs


def test_graphed_early_stopping_matches_eager():
    """learning_rate = 0 and no shuffle: epoch 2 repeats epoch 1's losses exactly, so both learners stop after it"""
    ops = ops_for("simt")
    eng = "3xtf32" if ops.tc_available() else "simt"
    a, b = _pair(_ocfg(num_epochs=3, learning_rate=0.0), eng, num_epochs=3, learning_rate=0.0)
    _run(a, b)
    assert a.learner.num_minibatches_done == b.learner.num_minibatches_done == 2 * NMB
    assert b.learner.train_step == 4 * 2 * NMB


def test_graphed_checkpoint_round_trip(tmp_path):
    """in graph mode the checkpoint stores the device's learning rate, and a learner resumed from it continues the eager
    learner's learning-rate sequence (and weights)"""
    from sample_factory_b200.checkpoint import load_checkpoint, save_checkpoint

    ops = ops_for("simt")
    eng = "3xtf32" if ops.tc_available() else "simt"
    ocfg = _ocfg(num_epochs=2)
    over = dict(_schedule_over("kl_adaptive_minibatch", 2), train_dir=str(tmp_path), experiment="resume")
    over["lr_schedule_kl_threshold"] = 1e-3       # (the rate goes down and up again)
    a, b = _pair(ocfg, eng, **over)
    feed = sampled_feed(a, b)
    lrs = []
    for it in range(2):
        feed(it)
        a.learner.train(a.traj)
        b.learner.train(b.traj)
        lrs.append(a.learner.curr_lr)
    save_checkpoint(b.cfg, b.model, b.learner)
    ck = torch.load(sorted((tmp_path / "resume" / "checkpoint_p0").glob("checkpoint_*"))[-1], weights_only=False)
    assert ck["curr_lr"] == b.learner.lr_dev.item() == lrs[-1]

    st0 = O.init_state(ocfg, seed=9)        # other weights: everything must come from the checkpoint
    c = build(ocfg, N, st0, torch.zeros(T + 1, N, ocfg.obs_dim), eng, learner_cuda_graph=True, **over)
    info = load_checkpoint(c.cfg, c.model, DEV)
    c.learner.train_step, c.learner.env_steps, c.learner.opt_step = info["train_step"], info["env_steps"], info["opt_step"]
    c.learner.curr_lr = info["curr_lr"]
    assert c.learner.lr_dev.item() == lrs[-1]
    for it in range(2, 5):
        a.sampler.set_policy_version(a.learner.train_step)
        a.sampler.rollout()
        for k in a.traj:
            c.traj[k].copy_(a.traj[k])
        a.learner.train(a.traj)
        c.learner.train(c.traj)
        torch.cuda.synchronize()
        _same_state(a, c, it)
        lrs.append(a.learner.curr_lr)
        assert c.learner.curr_lr == lrs[-1], (it, lrs, c.learner.curr_lr)
    assert len(set(lrs)) > 1, lrs
    assert c.learner.graph_replay_launches > 0


# ------------------------------------------------------------------------------------------------ kernel level
def _ulps(x):
    """x and the doubles one ulp below and above it"""
    return [np.nextafter(x, -math.inf), x, np.nextafter(x, math.inf)]


def test_lr_schedule_kernel_matches_host_rules():
    """sfb200_lr_schedule_step against KlAdaptiveScheduler.update / LinearDecayScheduler.update, bit for bit: KL values at
    2 thr and 0.5 thr and one ulp either side, learning rates at and one ulp around the min / max clamps"""
    from sample_factory_b200.cfg import default_cfg
    from sample_factory_b200.learner import KlAdaptiveScheduler, LinearDecayScheduler

    ops = ops_for("simt")
    cfg = default_cfg()
    cfg.num_batches_per_epoch = NMB
    lr_dev = torch.zeros(1, dtype=torch.float64, device=DEV)
    kl_dev = torch.zeros(1, dtype=torch.float64, device=DEV)
    for thr, lo, hi in [(0.008, 1e-6, 1e-2), (0.016, 7.3e-7, 3e-3), (1e-5, 1e-6, 1e-2)]:
        cfg.lr_schedule_kl_threshold, cfg.lr_adaptive_min, cfg.lr_adaptive_max = thr, lo, hi
        sched = KlAdaptiveScheduler(cfg, per_epoch=False)
        kls = _ulps(2.0 * thr) + _ulps(0.5 * thr) + [0.0, thr, 1e3 * thr]
        lrs = [3e-4, lo, hi] + _ulps(lo * 1.5) + _ulps(hi / 1.5)      # lr / 1.5 and lr * 1.5 at and around the clamps
        for kl in kls:
            for lr in lrs:
                want = sched.update(float(lr), [float(kl)])
                lr_dev.fill_(float(lr))
                kl_dev.fill_(float(kl))
                ops.lr_schedule_kl_adaptive(lr_dev, kl_dev[0], thr, lo, hi)
                got = lr_dev.item()
                assert got == want, (thr, kl, lr, got, want)

    step_dev = torch.zeros(1, dtype=torch.int64, device=DEV)
    for lr0, steps, batch, epochs in [(3e-4, 7 * 32, 32, 1), (0.00295, 1000 * 64, 64, 3), (1.0, 10240, 1024, 1),
                                      (2.5e-4, 3, 1, 2)]:
        cfg.learning_rate, cfg.train_for_env_steps, cfg.batch_size, cfg.num_epochs = lr0, steps, batch, epochs
        sched = LinearDecayScheduler(cfg)
        step_dev.zero_()
        lr_dev.fill_(lr0)
        lr = lr0
        for _ in range(sched.num_updates + 2):
            lr = sched.update(lr, [])
            ops.lr_schedule_linear_decay(lr_dev, step_dev, sched.num_updates, sched.lr0)
            assert lr_dev.item() == lr and step_dev.item() == sched.step, (lr0, sched.step, lr_dev.item(), lr)
        assert lr == 0.0


def test_lamb_dev_matches_host_step():
    """sfb200_clip_lamb_step_dev (step and lr in device memory) writes the same bits as sfb200_clip_lamb_step over many
    step counts: the bias corrections formed in the kernel equal the host's"""
    ops = ops_for("simt")
    gen = torch.Generator().manual_seed(3)
    sizes = [1000, 37, 9000]
    offs = np.cumsum([0] + sizes[:-1]).tolist()
    n = sum(sizes)
    seg_off = torch.tensor(offs, dtype=torch.int64, device=DEV)
    seg_n = torch.tensor(sizes, dtype=torch.int64, device=DEV)
    ws = torch.empty(ops.lamb_workspace_bytes(3, max(sizes)) // 4 + 4, dtype=torch.float32, device=DEV)
    p0 = torch.randn(n, generator=gen).to(DEV)
    g0 = torch.randn(n, generator=gen).to(DEV)
    m0 = (torch.randn(n, generator=gen) * 0.1).to(DEV)
    v0 = (torch.rand(n, generator=gen) * 0.01).to(DEV)
    num = torch.tensor([900.0], dtype=torch.float64, device=DEV)
    den = torch.tensor([1024.0], dtype=torch.float64, device=DEV)
    steps_dev = torch.zeros(1, dtype=torch.int64, device=DEV)
    lr_dev = torch.zeros(1, dtype=torch.float64, device=DEV)
    steps = list(range(1, 401)) + [1000, 4321, 16000, 20000, 100000, 10 ** 7]
    for beta1, beta2 in [(0.9, 0.999), (0.5, 0.9999)]:
        for step in steps:
            lr = 3e-4 * (1 + step % 7)
            host = [t.clone() for t in (p0, g0, m0, v0)]
            dev = [t.clone() for t in (p0, g0, m0, v0)]
            gn_h = torch.zeros(1, device=DEV)
            gn_d = torch.zeros(1, device=DEV)
            ops.clip_lamb_step(*host, seg_off, seg_n, max(sizes), step, lr, beta1, beta2, 1e-6, 1e-4, 0.01, 4.0, num, den,
                               gn_h, ws)
            steps_dev.fill_(step - 1)
            lr_dev.fill_(lr)
            ops.clip_lamb_step_dev(*dev, seg_off, seg_n, max(sizes), steps_dev, lr_dev, beta1, beta2, 1e-6, 1e-4, 0.01, 4.0,
                                   num, den, gn_d, ws)
            for name, x, y in zip("pgmv", host, dev):
                assert torch.equal(x, y), (beta1, beta2, step, name)
            assert torch.equal(gn_h, gn_d)
            assert steps_dev.item() == step - 1       # (the launch reads the counter; sfb200_advance_counters moves it)
