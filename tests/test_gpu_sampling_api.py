"""Sampler-only APIs (SURVEY 8f row 1): SyncSamplingAPI / EvalSamplingAPI / do_eval against the oracle rollout on the same
tape, noise and weights, in the style of the reference's sf_examples/sampler + eval.py usage."""
import os

import numpy as np
import pytest
import torch

from oracle import appo_oracle as O
from tests.device_harness import TOL, make_cfg

pytestmark = pytest.mark.gpu


def _cfg(ocfg, env_name, tmp_path, **over):
    cfg = make_cfg(ocfg, env=env_name, train_dir=str(tmp_path), experiment="api", cuda_graph=False, seed=0,
                   gemm_engine="simt", **over)
    return cfg


def _register(name, tape, A, dev):
    from sample_factory_b200.envs import TapeVecEnv, register_env

    register_env(name, lambda full_env_name, cfg, env_config, render_mode=None: TapeVecEnv(tape.to(dev).contiguous(), A))


def test_sync_sampling_api_matches_oracle(tmp_path):
    from sample_factory_b200.sampling_api import SyncSamplingAPI, obtain_env_info, samples_per_trajectory

    dev = torch.device("cuda", 0)
    N, T = 128, 16
    ocfg = O.OracleCfg(obs_dim=24, num_actions=6, encoder_mlp_layers=[64, 64], rollout=T)
    st = O.init_state(ocfg, seed=5)
    gen = torch.Generator().manual_seed(21)
    tape = torch.randn(3 * T + 1, N, ocfg.obs_dim, generator=gen)
    _register("api_tape", tape, ocfg.num_actions, dev)
    cfg = _cfg(ocfg, "api_tape", tmp_path)
    env_info = obtain_env_info(cfg)
    assert (env_info.obs_dim, env_info.num_actions, env_info.num_agents) == (24, 6, N)
    api = SyncSamplingAPI(cfg, env_info)
    api.start(init_model_data=(0, st, dev, 7))       # InitModelData = (policy_id, state_dict, device, policy_version)
    oenv = O.TapeVecEnv(tape, ocfg.num_actions)
    olast = oenv.reset()
    prev = None
    for it in range(3):
        noise = torch.empty(T, N, ocfg.num_actions).exponential_(generator=gen)
        otraj = O.alloc_trajectories(ocfg, N)
        olast = O.rollout(ocfg, st, oenv, olast, otraj, noise, 7)
        api.sampling_loop.sampler.noise = noise.to(dev)
        traj = api.get_trajectories_sync()
        assert samples_per_trajectory(traj) == N * T
        got = {k: v.cpu() for k, v in traj.items()}
        for k in ["obs", "actions", "rewards", "dones", "time_outs", "policy_id", "policy_version"]:
            assert torch.equal(got[k], otraj[k]), k
        np.testing.assert_allclose(got["action_logits"].numpy(), otraj["action_logits"].numpy(), atol=TOL)
        np.testing.assert_allclose(got["log_prob_actions"].numpy(), otraj["log_prob_actions"].numpy(), atol=TOL)
        np.testing.assert_allclose(got["values"][:, :-1].numpy(), otraj["values"][:, :-1].numpy(), atol=TOL)
        # a clone is handed out (sync_sampling_api.py:37): the next rollout must not change the previous result
        if prev is not None:
            assert torch.equal(prev[0]["actions"], prev[1])
        prev = (traj, traj["actions"].clone())
    assert api.stop() == 0
    assert api.get_trajectories_sync() is None


def _episodes_from_traj(rewards_raw, dones, ep_ret, ep_len, out_ret, out_len):
    """host restatement of _process_env_step's episode accounting (batched_sampling.py:215-287), (step, env) order"""
    N, T = dones.shape
    for t in range(T):
        ep_ret += rewards_raw[:, t]
        ep_len += 1
        for n in np.nonzero(dones[:, t])[0]:
            out_ret.append(float(ep_ret[n]))
            out_len.append(int(ep_len[n]))
            ep_ret[n] = 0.0
            ep_len[n] = 0


def test_eval_sampling_api_episode_stats_and_checkpoint(tmp_path):
    from types import SimpleNamespace

    from sample_factory_b200.checkpoint import save_checkpoint
    from sample_factory_b200.model import ModelSpec, PolicyModel
    from sample_factory_b200.sampling_api import EvalSamplingAPI, do_eval

    dev = torch.device("cuda", 0)
    N, T = 64, 16
    ocfg = O.OracleCfg(obs_dim=12, num_actions=4, encoder_mlp_layers=[32], rollout=T)
    st = O.init_state(ocfg, seed=9)
    tape = torch.randn(64, N, ocfg.obs_dim, generator=torch.Generator().manual_seed(3))
    _register("api_tape_eval", tape, ocfg.num_actions, dev)
    cfg = _cfg(ocfg, "api_tape_eval", tmp_path, reward_scale=0.5)     # episode stats use the RAW reward (:336)
    # a trained-policy checkpoint in the experiment dir: EvalSamplingAPI.init() must pick it up (Learner.init -> load)
    from sample_factory_b200 import ops

    ops.bind_device(dev)
    model = PolicyModel(ModelSpec(ocfg.obs_dim, ocfg.num_actions, [32], [], ocfg.nonlinearity, True, True), dev)
    model.load_state_dict(st, strict=False)
    save_checkpoint(cfg, model, SimpleNamespace(policy_id=0, train_step=41, env_steps=1000, opt_step=41, curr_lr=1e-4))

    api = EvalSamplingAPI(cfg)
    api.init()
    api.auto_pump = False
    got_sd = api.sampling_loop.model.state_dict()
    for k in O.param_names(ocfg):
        assert torch.equal(got_sd[k].cpu(), st[k]), k
    api.start()
    ep_ret, ep_len = np.zeros(N, dtype=np.float32), np.zeros(N, dtype=np.int64)
    want_ret, want_len = [], []
    for _ in range(4):
        api.pump()
        tr = api.sampling_loop.traj
        assert torch.all(tr["policy_version"] == 41.0)
        raw = tr["actions"][:, :, 0].cpu().numpy() / ocfg.num_actions          # the tape env's reward rule
        np.testing.assert_allclose(tr["rewards"].cpu().numpy(), np.clip(raw * 0.5, -cfg.reward_clip, cfg.reward_clip), atol=1e-7)
        _episodes_from_traj(raw.astype(np.float32), tr["dones"].cpu().numpy(), ep_ret, ep_len, want_ret, want_len)
    assert api.total_samples == 4 * N * T
    stats = api.eval_stats
    assert len(want_ret) > 50 and stats["len"][0] == want_len
    np.testing.assert_allclose(stats["reward"][0], want_ret, rtol=1e-6, atol=1e-6)
    assert stats["episode_number"][0] == list(range(len(want_ret)))
    assert api.eval_env_steps == [sum(want_len)]
    assert len(api.eval_episodes[0]) == len(want_ret)
    assert api.stop() == 0

    # eval.py driver: runs until sample_env_episodes episodes, writes eval_p0.csv
    cfg.sample_env_episodes = 100
    cfg.csv_folder_name = None
    assert do_eval(cfg) == 0
    lines = open(os.path.join(str(tmp_path), "api", "eval_p0.csv")).read().strip().split("\n")
    assert lines[0] == ",reward,len,episode_number" and len(lines) - 1 >= 100


def test_enjoy_deterministic_matches_oracle(tmp_path):
    """enjoy(cfg) (reference enjoy.py:103-295): saved config + latest checkpoint, eval_deterministic argmax actions, mean
    reward over the first max_num_episodes finished episodes -- against an oracle rollout with unit noise
    (argmax(p / 1) = argmax(p))."""
    import json
    from types import SimpleNamespace

    from sample_factory_b200 import ops
    from sample_factory_b200.checkpoint import save_checkpoint
    from sample_factory_b200.enjoy import enjoy
    from sample_factory_b200.model import ModelSpec, PolicyModel

    dev = torch.device("cuda", 0)
    N, T = 48, 8
    ocfg = O.OracleCfg(obs_dim=12, num_actions=5, encoder_mlp_layers=[32, 32], rollout=T)
    st = O.init_state(ocfg, seed=11)
    tape = torch.randn(40, N, ocfg.obs_dim, generator=torch.Generator().manual_seed(4)) * 2
    _register("api_tape_enjoy", tape, ocfg.num_actions, dev)
    cfg = _cfg(ocfg, "api_tape_enjoy", tmp_path)
    cfg.cli_args = {}          # (default_cfg records algo / env / experiment as "passed on the command line")
    os.makedirs(os.path.join(str(tmp_path), "api"), exist_ok=True)
    with pytest.raises(Exception, match="Could not load saved parameters"):
        enjoy(cfg)
    saved = {k: v for k, v in vars(cfg).items() if isinstance(v, (int, float, str, bool, list, type(None)))}
    with open(os.path.join(str(tmp_path), "api", "config.json"), "w") as f:
        json.dump(saved, f)
    with pytest.raises(RuntimeError, match="Could not load checkpoint"):
        enjoy(cfg)
    ops.bind_device(dev)
    model = PolicyModel(ModelSpec(ocfg.obs_dim, ocfg.num_actions, [32, 32], [], ocfg.nonlinearity, True, True), dev)
    model.load_state_dict(st, strict=False)
    save_checkpoint(cfg, model, SimpleNamespace(policy_id=0, train_step=5, env_steps=100, opt_step=5, curr_lr=1e-4))

    max_ep = 70
    cfg.cli_args = dict(eval_deterministic=True, max_num_episodes=max_ep)     # explicitly passed flags override the file
    cfg.eval_deterministic, cfg.max_num_episodes = True, max_ep
    status, avg = enjoy(cfg)
    assert status == 0

    oenv = O.TapeVecEnv(tape, ocfg.num_actions)
    olast = oenv.reset()
    ep_ret, ep_len = np.zeros(N, dtype=np.float32), np.zeros(N, dtype=np.int64)
    want_ret, want_len = [], []
    ones = torch.ones(T, N, ocfg.num_actions)
    while len(want_ret) < max_ep:
        otraj = O.alloc_trajectories(ocfg, N)
        olast = O.rollout(ocfg, st, oenv, olast, otraj, ones, 5)
        raw = (otraj["actions"][:, :, 0] / ocfg.num_actions).numpy()
        _episodes_from_traj(raw, otraj["dones"].numpy(), ep_ret, ep_len, want_ret, want_len)
    np.testing.assert_allclose(avg, float(np.mean(want_ret[:max_ep])), rtol=1e-5, atol=1e-6)
    # sampling (non-deterministic) mode gives a different answer on the same checkpoint
    cfg.cli_args = dict(eval_deterministic=False, max_num_episodes=max_ep)
    cfg.eval_deterministic = False
    status2, avg2 = enjoy(cfg)
    assert status2 == 0 and np.isfinite(avg2) and abs(avg2 - avg) > 1e-4
