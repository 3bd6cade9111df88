"""Separate actor / critic weights with recurrent cores on the device: the sampler and the learner against the
reference-executed fixtures tiny_separate_gru / tiny_separate_lstm2 / tiny_shuffle_separate_gru, the two towers' forward
and backward (per tower: heads -> decoder -> BPTT -> encoder) against torch nn.GRU / nn.LSTM towers with autograd, config
5's stack with separate weights at full size, and a host env through run_rl and enjoy with the default GRU core."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import appo_oracle as O
from tests import separate_rnn_oracle as SO
from tests.device_harness import (ENGINES, MiniCartPole, build, build_case, check_finite, ops_for, replay_learner,
                                  replay_sampler, runner)

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ vs the reference
GOLDEN = ["tiny_separate_gru", "tiny_separate_lstm2"]


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", GOLDEN + ["tiny_shuffle_separate_gru"])
def test_sampler_matches_reference_golden(name, engine):
    """the sampler on the reference's weights, obs tape and noise: Discrete actions bit-exact (Box actions, floats of the
    means, and their rewards at 1e-5), the [actor | critic] state rows, logits, values and log-probs at 1e-5, and both
    halves of the state recorded after a done step zero"""
    case = SO.load_separate_rnn_case(name)
    rig = build_case(case, engine)
    ocfg, T = case[2], case[2].rollout
    assert rig.model.spec.rnn_state_size == O.rnn_state_size(ocfg) == rig.traj["rnn_states"].shape[2]
    S = rig.model.spec.rnn_tower_state_size

    def check_states(got, it):
        after_done = got["rnn_states"][:, 1:T + 1][got["dones"].view(-1, T).bool()]
        assert after_done.shape[0] > 0 and torch.all(after_done == 0)
        assert got["rnn_states"][..., :S].abs().max() > 0 and got["rnn_states"][..., S:].abs().max() > 0
    replay_sampler(case, rig, exact=("obs", "dones", "rewards", "actions"), check_iteration=check_states)


def _learner_vs_golden(name, engine, graph):
    case = SO.load_separate_rnn_case(name)
    rig = build_case(case, engine, learner_cuda_graph=graph)
    assert rig.learner.use_graph == graph
    replay_learner(case, rig)


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", GOLDEN + ["tiny_shuffle_separate_gru"])
def test_learner_matches_reference_golden(name, engine):
    """Learner.train on the reference's trajectories (bootstrap value through both towers' steps, per-tower BPTT with
    resets at done-or-invalid boundaries): returns, advantages, losses at 1e-5, post-Adam weights at 2e-5"""
    _learner_vs_golden(name, engine, graph=False)


@pytest.mark.parametrize("engine", ENGINES)
def test_graphed_learner_matches_reference_golden(engine):
    """the same through one CUDA graph per train() (cfg.learner_cuda_graph; one epoch, so tiny_separate_lstm2)"""
    _learner_vs_golden("tiny_separate_lstm2", engine, graph=True)


# ------------------------------------------------------------------------------------------------ vs torch autograd
class _TorchTower(torch.nn.Module):
    def __init__(self, D, enc, rnn_type, H, L, dec):
        super().__init__()
        self.enc = torch.nn.ModuleList()
        d = D
        for h in enc:
            self.enc.append(torch.nn.Linear(d, h))
            d = h
        self.core = (torch.nn.GRU if rnn_type == "gru" else torch.nn.LSTM)(d, H, L)
        self.dec = torch.nn.ModuleList()
        d = H
        for h in dec:
            self.dec.append(torch.nn.Linear(d, h))
            d = h
        self.rnn_type, self.H, self.L = rnn_type, H, L

    def forward(self, x, state, doi, n, R):
        """x [n*R, D] env-major, state [n, L*Sl] chunk-start states, doi [n, R]: the masked step loop"""
        for lin in self.enc:
            x = torch.nn.functional.elu(lin(x))
        s = state.view(n, self.L, -1).permute(1, 0, 2)
        hx = s.contiguous() if self.rnn_type == "gru" else (s[..., :self.H].contiguous(), s[..., self.H:].contiguous())
        xs = x.view(n, R, -1)
        outs = []
        for t in range(R):
            if t > 0:
                keep = (1 - doi[:, t - 1].float()).view(1, n, 1)
                hx = hx * keep if self.rnn_type == "gru" else (hx[0] * keep, hx[1] * keep)
            out, hx = self.core(xs[:, t].unsqueeze(0), hx)
            outs.append(out[0])
        y = torch.stack(outs, 1).reshape(n * R, -1)
        for lin in self.dec:
            y = torch.nn.functional.elu(lin(y))
        return y


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("dec", [[], [96]])
@pytest.mark.parametrize("rnn_type", ["gru", "lstm"])
def test_two_tower_bptt_matches_torch_autograd(rnn_type, dec, engine):
    """512 rows, R = 16, H = 128, two layers: the learner's minibatch forward (values, logits) and its explicit backward
    (heads over the concatenated tail -> per tower decoder -> BPTT -> W_ih / encoder) against nn.GRU / nn.LSTM towers
    with autograd, for given d(logits) / d(values) -- every parameter gradient of both towers and of the heads"""
    ops = ops_for(engine)
    dev = torch.device("cuda", 0)
    n, R, H, L, D, A = 32, 16, 128, 2, 40, 6
    B = n * R
    gen = torch.Generator().manual_seed(31 + len(dec))
    ocfg = SO.SeparateRnnCfg(obs_dim=D, num_actions=A, encoder_mlp_layers=[64], decoder_mlp_layers=list(dec), rollout=R,
                             recurrence=R, batch_size=B, num_batches_per_epoch=2, use_rnn=True, rnn_type=rnn_type,
                             rnn_size=H, rnn_num_layers=L, actor_critic_share_weights=False, normalize_input=False)
    torch.manual_seed(5)
    towers = {tw: _TorchTower(D, [64], rnn_type, H, L, dec) for tw in SO.TOWERS}
    Ht = dec[-1] if dec else H
    critic, action = torch.nn.Linear(Ht, 1), torch.nn.Linear(Ht, A)
    sd = {}
    for tw, m in towers.items():
        sd[f"{tw}encoder.encoders.obs.mlp_head.0.weight"], sd[f"{tw}encoder.encoders.obs.mlp_head.0.bias"] = m.enc[0].weight, m.enc[0].bias
        for k, p in m.core.named_parameters():
            sd[f"{tw}core.core.{k}"] = p
        for i, lin in enumerate(m.dec):
            sd[f"{tw}decoder.mlp.{2 * i}.weight"], sd[f"{tw}decoder.mlp.{2 * i}.bias"] = lin.weight, lin.bias
    sd[O.CRITIC_W], sd[O.CRITIC_B], sd[O.ACTION_W], sd[O.ACTION_B] = critic.weight, critic.bias, action.weight, action.bias
    cfg, model, traj, _, sampler, learner = build(ocfg, 2 * n, {k: v.detach().clone() for k, v in sd.items()},
                                                  torch.zeros(2, 2 * n, D), engine)     # (minibatches of n chunks)
    Sw = model.spec.rnn_tower_state_size
    x = torch.randn(B, D, generator=gen)
    states = torch.rand(B, 2 * Sw, generator=gen) - 0.5
    dones = torch.rand(B, generator=gen) < 0.15
    valids = torch.rand(B, generator=gen) > 0.05
    dlogits = torch.randn(B, A, generator=gen) * 0.1
    dvalues = torch.randn(B, generator=gen) * 0.1
    doi = (dones | ~valids).view(n, R)

    chunk0 = states.view(n, R, -1)[:, 0]
    ya = towers["actor_"](x, chunk0[:, :Sw], doi, n, R)
    yc = towers["critic_"](x, chunk0[:, Sw:], doi, n, R)
    logits, values = action(ya), critic(yc).squeeze(-1)
    ((logits * dlogits).sum() + (values * dvalues).sum()).backward()

    from sample_factory_b200.policy import forward_policy

    xd, sd_, dd, vd = x.to(dev), states.to(dev), dones.to(dev), valids.to(dev)
    fns = {tw: (lambda head, tw=tw: learner.tower_rnn[tw].forward_bptt(head, sd_, dd if tw == "actor_" else None, vd,
                                                                      learner.tower_rnn_bufs[tw])) for tw in SO.TOWERS}
    forward_policy(model, xd, learner.h, learner.act, learner.engine, learner.heads_plan,
                   dict(values=learner.mb_values, values_stride=1, logits=learner.mb_logits, logits_stride=A),
                   store_tail=True, tower_rnn_fns=fns)
    np.testing.assert_allclose(learner.mb_logits.cpu().numpy(), logits.detach().numpy(), atol=1e-4)
    np.testing.assert_allclose(learner.mb_values.cpu().numpy(), values.detach().numpy(), atol=1e-4)
    model.grad.zero_()
    learner.dlogits.copy_(dlogits)
    learner.dvalues.copy_(dvalues)
    learner._backward_separate(xd)
    torch.cuda.synchronize()
    for name, p in sd.items():
        g = model.grads[name].cpu()
        assert torch.isfinite(g).all(), name
        np.testing.assert_allclose(g.numpy().reshape(p.grad.shape), p.grad.numpy(), atol=2e-4, rtol=2e-3, err_msg=name)


# ------------------------------------------------------------------------------------------------ full size / host env
PEAK_GIB = 7.0


def test_cfg5_separate_weights_4096_envs_per_gpu():
    """config 5's stack with --actor_critic_share_weights=False through Runner: Box(256) obs, per tower MLP [512,256,128]
    -> LSTM-512, 4096 envs, rollout = recurrence = 16, 2 x 32768 minibatches, 2 epochs, three iterations: finite losses,
    both towers train, the state rows [actor | critic] reset at dones, and the peak allocated memory bounded"""
    from sample_factory_b200.envs import TapeVecEnv

    dev = torch.device("cuda", 0)
    N, T = 4096, 16
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    tape = torch.randn(2 * T + 1, N, 256, generator=torch.Generator().manual_seed(2)).to(dev)
    r = runner("synthetic_isaac_sep", lambda name, cfg, env_config, render_mode=None: TapeVecEnv(tape, 8),
                ["--use_rnn=True", "--rnn_type=lstm", "--rnn_size=512", "--actor_critic_share_weights=False",
                 "--async_rl=False", f"--rollout={T}", f"--recurrence={T}", "--batch_size=32768",
                 "--num_batches_per_epoch=2", "--num_epochs=2", "--encoder_mlp_layers", "512", "256", "128",
                 "--value_bootstrap=True", "--reward_scale=0.01", "--lr_schedule=kl_adaptive_epoch",
                 "--lr_schedule_kl_threshold=0.016", "--max_grad_norm=1.0"])
    assert not r.model.spec.share_weights and r.model.spec.rnn_state_size == 2048
    assert r.traj["rnn_states"].shape == (N, T + 1, 2048)
    w = {tw: r.model.params[f"{tw}core.core.weight_hh_l0"].clone() for tw in SO.TOWERS}
    st = check_finite(r, 3, 3 * N * T)
    assert st["num_valid"] == 32768
    for tw in SO.TOWERS:
        assert not torch.equal(w[tw], r.model.params[f"{tw}core.core.weight_hh_l0"]), tw
    hs = r.traj["rnn_states"]
    assert torch.isfinite(hs).all() and hs[..., :1024].abs().max().item() > 0 and hs[..., 1024:].abs().max().item() > 0
    nxt = hs[:, 1:T + 1][r.traj["dones"]]
    assert nxt.numel() > 0 and torch.all(nxt == 0)
    peak = (torch.cuda.max_memory_allocated() - base) / 2**30
    print(f"peak allocated: {peak:.2f} GiB")
    assert peak < PEAK_GIB, peak


def test_host_env_run_rl_and_enjoy_with_default_gru(tmp_path):
    """a gymnasium-API CPU env (the CartPole re-implementation) through run_rl with --actor_critic_share_weights=False and
    otherwise default model flags (GRU-512 core per tower); enjoy() then loads the checkpoint it wrote"""
    from sample_factory_b200.cfg import parse_full_cfg, parse_sf_args
    from sample_factory_b200.checkpoint import checkpoint_dir, get_checkpoints
    from sample_factory_b200.enjoy import enjoy
    from sample_factory_b200.envs import register_env
    from sample_factory_b200.host_env import BatchedHostEnv
    from sample_factory_b200.train import run_rl

    ops_for()
    dev = torch.device("cuda", 0)
    register_env("MiniCartPoleSep-v0", lambda name, cfg, env_config, render_mode=None: BatchedHostEnv(
        lambda i: MiniCartPole(max_steps=50), 32, dev, seed=cfg.seed))
    argv = ["--env=MiniCartPoleSep-v0", "--experiment=sep", f"--train_dir={tmp_path}", "--restart_behavior=overwrite",
            "--actor_critic_share_weights=False", "--rollout=16", "--batch_size=256", "--num_batches_per_epoch=2",
            "--async_rl=False", "--seed=0", "--train_for_env_steps=2048", "--save_every_sec=100000",
            "--experiment_summaries_interval=100000"]
    parser, _ = parse_sf_args(argv)
    cfg = parse_full_cfg(parser, argv)
    assert cfg.use_rnn and cfg.rnn_type == "gru" and cfg.rnn_size == 512 and not cfg.actor_critic_share_weights
    assert run_rl(cfg) == 0
    files = get_checkpoints(checkpoint_dir(cfg, 0))
    assert files
    sd = torch.load(files[-1], map_location="cpu", weights_only=False)["model"]
    assert sd["actor_core.core.weight_ih_l0"].shape == (3 * 512, 512) and sd["critic_core.core.weight_hh_l0"].shape == (1536, 512)
    assert all(torch.isfinite(v).all() for v in sd.values())
    cfg.cli_args = dict(max_num_episodes=20)
    cfg.max_num_episodes = 20
    status, avg = enjoy(cfg)
    assert status == 0 and np.isfinite(avg) and avg > 0
