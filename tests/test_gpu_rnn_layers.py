"""Stacked recurrent cores (--rnn_num_layers > 1) on the device: RnnCore against torch's own multi-layer nn.GRU / nn.LSTM
with autograd, the sampler and the learner against the reference-executed fixtures tiny_gru2 / tiny_lstm3 /
tiny_shuffle_gru2, enjoy() on a two-layer checkpoint, and config 5's stack with two LSTM layers at full size."""
import os

import numpy as np
import pytest
import torch

from oracle import appo_oracle as O
from tests import rnn_layers_oracle as RO
from tests.device_harness import (DEV, ENGINES, TOL, build, build_case, check_finite, graphed_learner_matches_eager,
                                  make_cfg, model_spec, ops_for, replay_learner, replay_sampler, runner)

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ RnnCore vs torch
def _torch_state(rnn_type, state, L, H):
    """[M, S] layer-major state rows -> nn.GRU h_0 / nn.LSTM (h_0, c_0), each [L, M, H] (core.py:42-53)"""
    s = state.view(state.shape[0], L, -1).permute(1, 0, 2)
    if rnn_type == "gru":
        return s.contiguous()
    return s[:, :, :H].contiguous(), s[:, :, H:].contiguous()


def _core(rnn, rnn_type, L, H, D, engine):
    from sample_factory_b200.model import ModelSpec, PolicyModel
    from sample_factory_b200.rnn_core import RnnCore

    ops = ops_for(engine)
    spec = ModelSpec(D, 3, [D], [], "elu", False, False, use_rnn=True, rnn_type=rnn_type, rnn_size=H, rnn_num_layers=L)
    model = PolicyModel(spec, torch.device("cuda", 0))
    model.load_state_dict({f"core.core.{k}": v.detach().clone() for k, v in rnn.state_dict().items()}, strict=False)
    return model, RnnCore(model, ops.ENGINES[engine])


SHAPES = [(2, 32, 24), (3, 64, 40), (2, 30, 20)]      # (L, H, D); H = 30: layer slices off a 16-byte boundary


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("rnn_type", ["gru", "lstm"])
@pytest.mark.parametrize("L,H,D", SHAPES)
def test_step_matches_torch_stacked_rnn(L, H, D, rnn_type, engine):
    """One sampler step of RnnCore: the core output and the whole new state row (every layer's slice) against
    nn.GRU / nn.LSTM(num_layers=L) on one time step"""
    M = 77
    gen = torch.Generator().manual_seed(100 + L * 10 + H)
    rnn = (torch.nn.GRU if rnn_type == "gru" else torch.nn.LSTM)(D, H, L)
    Sl = H if rnn_type == "gru" else 2 * H
    x = torch.randn(M, D, generator=gen)
    state = torch.rand(M, L * Sl, generator=gen) - 0.5
    with torch.no_grad():
        out, new = rnn(x.view(1, M, D), _torch_state(rnn_type, state, L, H))
        if rnn_type == "gru":
            want = new.permute(1, 0, 2).reshape(M, -1)
        else:
            want = torch.cat(new, dim=2).permute(1, 0, 2).reshape(M, -1)
    model, core = _core(rnn, rnn_type, L, H, D, engine)
    dev = model.device
    bufs = core.alloc_step(M)
    s_out = torch.full((M, L * Sl), float("nan"), device=dev)
    got = core.step(x.to(dev), state.to(dev), s_out, bufs)
    np.testing.assert_allclose(got.cpu().numpy(), out.view(M, H).numpy(), atol=TOL)
    np.testing.assert_allclose(s_out.cpu().numpy(), want.numpy(), atol=TOL)


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("rnn_type", ["gru", "lstm"])
@pytest.mark.parametrize("L,H,D", SHAPES)
def test_bptt_matches_torch_stacked_rnn(L, H, D, rnn_type, engine):
    """forward_bptt / backward_bptt over chunks with mid-chunk resets against a step-by-step nn.GRU / nn.LSTM(num_layers=L)
    loop that zeroes every layer's state after a done (the ground truth of tests/algo/test_rnn.py, stacked): the core
    output, the input gradient, and the gradient of every parameter of every layer"""
    N, R = 24, 9
    B = N * R
    gen = torch.Generator().manual_seed(200 + L * 10 + H)
    rnn = (torch.nn.GRU if rnn_type == "gru" else torch.nn.LSTM)(D, H, L)
    Sl = H if rnn_type == "gru" else 2 * H
    dones = torch.rand(B, generator=gen) < 0.2
    valids = torch.rand(B, generator=gen) > 0.05
    doi = (dones | ~valids).view(N, R)
    states = torch.rand(B, L * Sl, generator=gen) - 0.5
    x = torch.randn(B, D, generator=gen, requires_grad=True)
    d_core = torch.randn(B, H, generator=gen)

    hx = _torch_state(rnn_type, states.view(N, R, -1)[:, 0], L, H)
    xs = x.view(N, R, D)
    outs = []
    for t in range(R):
        if t > 0:
            keep = (1 - doi[:, t - 1].float()).view(1, N, 1)
            hx = hx * keep if rnn_type == "gru" else (hx[0] * keep, hx[1] * keep)
        out, hx = rnn(xs[:, t].reshape(1, N, D), hx)
        outs.append(out.view(N, H))
    loopy = torch.stack(outs, dim=1).reshape(B, H)
    (loopy * d_core).sum().backward()

    model, core = _core(rnn, rnn_type, L, H, D, engine)
    dev = model.device
    b = core.alloc_bptt(B, R)
    got = core.forward_bptt(x.detach().to(dev), states.to(dev), dones.to(dev), valids.to(dev), b)
    np.testing.assert_allclose(got.cpu().numpy(), loopy.detach().numpy(), atol=TOL)
    model.grad.zero_()
    lin_ws = torch.empty(core.lin_ws_bytes(B, R, D) // 4 + 4, device=dev)
    dgi = core.backward_bptt(d_core.to(dev), b, lin_ws).cpu().double()
    tol = dict(atol=1e-4, rtol=1e-4)
    np.testing.assert_allclose((dgi @ rnn.weight_ih_l0.detach().double()).float().numpy(), x.grad.numpy(), **tol)
    np.testing.assert_allclose((dgi.t() @ x.detach().double()).float().numpy(), rnn.weight_ih_l0.grad.numpy(), **tol)
    for name, p in rnn.named_parameters():
        if name == "weight_ih_l0":       # (the learner's linear_backward over dgi_all, checked above)
            continue
        np.testing.assert_allclose(model.grads[f"core.core.{name}"].cpu().numpy(), p.grad.numpy(), err_msg=name, **tol)


def test_misaligned_layer_slices_take_the_simt_gemm():
    """H % 4 != 0 puts layer k > 0's slice of a state row off a 16-byte boundary, which TMA cannot describe: on the
    wgmma engine those GEMMs run as gemm_simt_kernel (the step test above checks their results), an aligned H runs none"""
    from torch.profiler import ProfilerActivity, profile

    ops_for("3xtf32")
    counts = {}
    for H in (30, 32):
        rnn = torch.nn.GRU(24, H, 2)
        model, core = _core(rnn, "gru", 2, H, 24, "3xtf32")
        dev = model.device
        M = 256
        x = torch.randn(M, 24, device=dev)
        s_in, s_out = torch.zeros(M, 2 * H, device=dev), torch.empty(M, 2 * H, device=dev)
        bufs = core.alloc_step(M)
        core.step(x, s_in, s_out, bufs)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            core.step(x, s_in, s_out, bufs)
            torch.cuda.synchronize()
        names = [e.key for e in prof.key_averages()]
        counts[H] = (sum(1 for n in names if "gemm_simt_kernel" in n), sum(1 for n in names if "gemm_wgmma_kernel" in n))
    assert counts[30][0] >= 1, counts
    assert counts[32][0] == 0 and counts[32][1] >= 1, counts


# ------------------------------------------------------------------------------------------------ vs the reference
GOLDEN = ["tiny_gru2", "tiny_lstm3"]


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", GOLDEN)
def test_sampler_matches_reference_golden(name, engine):
    """the sampler on the reference's weights, obs tape and Exp(1) noise: actions bit-exact, the recorded states and the
    policy outputs at 1e-5, and the state recorded after a done step zero in every layer"""
    case = RO.load_stacked_case(name)
    rig = build_case(case, engine)
    ocfg, T = case[2], case[2].rollout
    assert rig.model.spec.rnn_state_size == O.rnn_state_size(ocfg) == rig.traj["rnn_states"].shape[2]

    def state_zero_after_done(got, it):
        after_done = got["rnn_states"][:, 1:T + 1][got["dones"].view(-1, T).bool()]
        assert after_done.shape[0] > 0 and torch.all(after_done == 0)
    replay_sampler(case, rig, exact=("obs", "rewards", "dones", "actions"), check_iteration=state_zero_after_done)


def _learner_vs_golden(name, engine, graph):
    case = RO.load_stacked_case(name)
    rig = build_case(case, engine, learner_cuda_graph=graph)
    assert rig.learner.use_graph == graph
    replay_learner(case, rig)


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", GOLDEN + ["tiny_shuffle_gru2"])
def test_learner_matches_reference_golden(name, engine):
    """Learner.train on the reference's trajectories (bootstrap value through the stacked step, BPTT with every layer
    reset at done-or-invalid boundaries): returns, advantages, losses at 1e-5, post-Adam weights at 2e-5"""
    _learner_vs_golden(name, engine, graph=False)


@pytest.mark.parametrize("engine", ENGINES)
def test_graphed_learner_matches_reference_golden(engine):
    """the same through one CUDA graph per train() (cfg.learner_cuda_graph; one epoch, so tiny_lstm3)"""
    _learner_vs_golden("tiny_lstm3", engine, graph=True)


def test_graphed_sampler_and_learner_match_eager():
    """two-layer GRU: the CUDA-graph sampler and learner produce exactly the eager trajectories and weights"""
    eng = "3xtf32" if ops_for().tc_available() else "simt"
    N, T = 64, 8
    ocfg = RO.StackedCfg(obs_dim=20, num_actions=5, encoder_mlp_layers=[64], rollout=T, recurrence=T, batch_size=N * T // 2,
                       num_batches_per_epoch=2, use_rnn=True, rnn_type="gru", rnn_size=64, rnn_num_layers=2)
    st0 = O.init_state(ocfg, seed=4)
    tape = torch.randn(3 * T + 1, N, ocfg.obs_dim, generator=torch.Generator().manual_seed(5))
    a = build(ocfg, N, st0, tape, eng)
    b = build(ocfg, N, st0, tape, eng, graph=True, learner_cuda_graph=True)
    for smp in (a.sampler, b.sampler):
        smp.reset()
        smp.rollout()
    for smp in (a.sampler, b.sampler):     # (graph capture ran the first rollout eagerly: re-align both)
        smp.reset()
        smp.step_counter.zero_()

    def feed(it):
        for r in (a, b):
            r.sampler.set_policy_version(r.learner.train_step)
            r.sampler.rollout()
        torch.cuda.synchronize()
        for k in a.traj:
            assert torch.equal(a.traj[k], b.traj[k]), (it, k)
    graphed_learner_matches_eager(a, b, feed, iters=3)


# ------------------------------------------------------------------------------------------------ enjoy / full size
def test_enjoy_two_layer_checkpoint_matches_oracle(tmp_path):
    """enjoy(cfg) on a saved two-layer GRU checkpoint, deterministic actions: the mean episode reward equals an oracle
    rollout of the same weights with unit noise (argmax), the recurrent state carried across rollouts"""
    import json
    from types import SimpleNamespace

    from sample_factory_b200.checkpoint import save_checkpoint
    from sample_factory_b200.enjoy import enjoy
    from sample_factory_b200.envs import TapeVecEnv, register_env
    from sample_factory_b200.model import PolicyModel

    ops = ops_for()
    dev = torch.device("cuda", 0)
    N, T = 48, 8
    ocfg = RO.StackedCfg(obs_dim=12, num_actions=5, encoder_mlp_layers=[32], rollout=T, recurrence=T, use_rnn=True,
                       rnn_type="gru", rnn_size=32, rnn_num_layers=2)
    st = O.init_state(ocfg, seed=11)
    tape = torch.randn(40, N, ocfg.obs_dim, generator=torch.Generator().manual_seed(4)) * 2
    register_env("rnn2_enjoy", lambda full_env_name, cfg, env_config, render_mode=None: TapeVecEnv(tape.to(dev).contiguous(), 5))
    cfg = make_cfg(ocfg, env="rnn2_enjoy", train_dir=str(tmp_path), experiment="api", cuda_graph=False, seed=0,
                   gemm_engine="simt")
    cfg.cli_args = {}
    os.makedirs(os.path.join(str(tmp_path), "api"), exist_ok=True)
    saved = {k: v for k, v in vars(cfg).items() if isinstance(v, (int, float, str, bool, list, type(None)))}
    with open(os.path.join(str(tmp_path), "api", "config.json"), "w") as f:
        json.dump(saved, f)
    model = PolicyModel(model_spec(ocfg), DEV)
    model.load_state_dict(st, strict=False)
    save_checkpoint(cfg, model, SimpleNamespace(policy_id=0, train_step=5, env_steps=100, opt_step=5, curr_lr=1e-4))
    max_ep = 60
    cfg.cli_args = dict(eval_deterministic=True, max_num_episodes=max_ep)
    cfg.eval_deterministic, cfg.max_num_episodes = True, max_ep
    status, avg = enjoy(cfg)
    assert status == 0

    oenv = O.TapeVecEnv(tape, ocfg.num_actions)
    olast = oenv.reset()
    rnn_state = torch.zeros(N, O.rnn_state_size(ocfg))
    ep_ret, ep_len, want_ret = np.zeros(N, dtype=np.float32), np.zeros(N, dtype=np.int64), []
    ones = torch.ones(T, N, ocfg.num_actions)
    while len(want_ret) < max_ep:
        otraj = O.alloc_trajectories(ocfg, N)
        olast = O.rollout(ocfg, st, oenv, olast, otraj, ones, 5, rnn_state)
        raw = (otraj["actions"][:, :, 0] / ocfg.num_actions).numpy()
        dones = otraj["dones"].numpy()
        for t in range(T):
            ep_ret += raw[:, t]
            ep_len += 1
            for n in np.nonzero(dones[:, t])[0]:
                want_ret.append(float(ep_ret[n]))
                ep_ret[n], ep_len[n] = 0.0, 0
    np.testing.assert_allclose(avg, float(np.mean(want_ret[:max_ep])), rtol=1e-5, atol=1e-6)


def test_run_rl_trains_three_gru_layers(tmp_path):
    """--rnn_num_layers=3 through run_rl: no refusal, a checkpoint with every layer's tensors"""
    from sample_factory_b200.cfg import parse_full_cfg, parse_sf_args
    from sample_factory_b200.checkpoint import checkpoint_dir, get_checkpoints
    from sample_factory_b200.envs import TapeVecEnv, register_env
    from sample_factory_b200.train import run_rl

    ops_for()
    dev = torch.device("cuda", 0)
    tape = torch.randn(33, 256, 16, generator=torch.Generator().manual_seed(6)).to(dev)
    register_env("rnn3_run_rl", lambda name, cfg, env_config, render_mode=None: TapeVecEnv(tape, 4))
    argv = ["--env=rnn3_run_rl", "--experiment=rnn3", f"--train_dir={tmp_path}", "--restart_behavior=overwrite",
            "--use_rnn=True", "--rnn_type=gru", "--rnn_size=64", "--rnn_num_layers=3", "--rollout=16", "--recurrence=8",
            "--batch_size=1024", "--num_batches_per_epoch=4", "--encoder_mlp_layers", "64", "--async_rl=False",
            "--batched_sampling=True", "--num_workers=1", "--num_envs_per_worker=1", "--worker_num_splits=1", "--seed=0",
            "--train_for_env_steps=16384", "--save_every_sec=100000", "--experiment_summaries_interval=100000"]
    parser, _ = parse_sf_args(argv)
    cfg = parse_full_cfg(parser, argv)
    assert run_rl(cfg) == 0
    files = get_checkpoints(checkpoint_dir(cfg, 0))
    assert files
    sd = torch.load(files[-1], map_location="cpu", weights_only=False)["model"]
    assert sd["core.core.weight_ih_l2"].shape == (192, 64) and torch.isfinite(sd["core.core.weight_hh_l2"]).all()


PEAK_GIB = 7.0


def test_cfg5_two_lstm_layers_4096_envs_per_gpu():
    """config 5's stack with --rnn_num_layers=2 through Runner: Box(256) obs, MLP [512,256,128] -> 2 x LSTM-512, 4096 envs,
    rollout = recurrence = 16, 2 x 32768 minibatches, 2 epochs.  Peak allocated memory stays under 7 GiB (5.15 GiB
    measured by this test on an H100 80GB HBM3); the large items: the trajectories with 2048-wide states (0.6 GB), the
    flat [E, 2048] state copy (0.5 GB), per layer the BPTT buffers the backward reads (gates / state_in / state_out /
    core_out, 0.6 GB), the gate and gradient buffers all layers share (1.1 GB)."""
    from sample_factory_b200.envs import TapeVecEnv

    dev = torch.device("cuda", 0)
    N, T = 4096, 16
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    tape = torch.randn(2 * T + 1, N, 256, generator=torch.Generator().manual_seed(2)).to(dev)
    r = runner("synthetic_isaac_l2", lambda name, cfg, env_config, render_mode=None: TapeVecEnv(tape, 8),
                ["--use_rnn=True", "--rnn_type=lstm", "--rnn_size=512", "--rnn_num_layers=2", "--async_rl=False",
                 f"--rollout={T}", f"--recurrence={T}", "--batch_size=32768", "--num_batches_per_epoch=2",
                 "--num_epochs=2", "--encoder_mlp_layers", "512", "256", "128", "--value_bootstrap=True",
                 "--reward_scale=0.01", "--lr_schedule=kl_adaptive_epoch", "--lr_schedule_kl_threshold=0.016",
                 "--max_grad_norm=1.0"])
    assert r.model.spec.rnn_num_layers == 2 and r.model.spec.rnn_state_size == 2048
    assert r.traj["rnn_states"].shape == (N, T + 1, 2048)
    assert "core.core.weight_ih_l1" in r.model.params and r.model.params["core.core.weight_ih_l1"].shape == (2048, 512)
    lr0 = r.learner.curr_lr
    w1 = r.model.params["core.core.weight_hh_l1"].clone()
    st = check_finite(r, 3, 3 * N * T)
    assert st["num_valid"] == 32768
    assert r.learner.curr_lr != lr0
    assert not torch.equal(w1, r.model.params["core.core.weight_hh_l1"])      # the upper layer trains
    hs = r.traj["rnn_states"]
    assert torch.isfinite(hs).all() and hs[..., 1024:].abs().max().item() > 0
    nxt = hs[:, 1:T + 1][r.traj["dones"]]
    assert nxt.numel() > 0 and torch.all(nxt == 0)
    peak = (torch.cuda.max_memory_allocated() - base) / 2**30
    print(f"peak allocated: {peak:.2f} GiB")
    assert peak < PEAK_GIB, peak
