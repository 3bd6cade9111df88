"""Dict observations with several 1-D keys (MultiInputEncoder) on the device: the key encoders' forward and backward
against torch autograd of the oracle's MultiInputEncoder restatement (aligned and unaligned key layouts, with and without a
layer after the concatenation), the sampler and the learner against the reference-executed fixtures tiny_dict /
tiny_dict_lstm / tiny_dict_mask, a gymnasium-API env with a three-key Dict through BatchedHostEnv, run_rl and enjoy, and a
full-size run through Runner."""

import numpy as np
import pytest
import torch

from oracle import appo_oracle as O
from tests import dict_obs_oracle as DO
from tests.device_harness import (DEV, ENGINES, TOL, build, build_case, check_finite, ops_for, replay_learner,
                                  replay_sampler, runner)

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ vs torch autograd
LAYOUTS = {"aligned": [("a", 8), ("b", 16)], "unaligned": [("achieved_goal", 3), ("desired_goal", 3), ("observation", 13)]}


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("decoder", [[], [48]])
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_key_encoders_match_torch_autograd(layout, decoder, engine):
    """one rollout and one learner step of a Dict model on random weights: the policy outputs (forward through the key
    encoders into the concatenation) and the post-Adam weights of every key encoder layer (their gradients come from
    the per-key backward chains) against the oracle, whose gradients are torch autograd through MultiInputEncoder"""
    keys = LAYOUTS[layout]
    N, T = 64, 8
    ocfg = DO.DictCfg(obs_dim=sum(d for _, d in keys), num_actions=5, encoder_mlp_layers=[32, 24],
                      decoder_mlp_layers=decoder, rollout=T, recurrence=1, batch_size=N * T, num_batches_per_epoch=1,
                      obs_keys=keys)
    st = O.init_state(ocfg, seed=3)
    tape = torch.randn(T + 1, N, ocfg.obs_dim, generator=torch.Generator().manual_seed(8)) * 1.5 + 0.3
    noise = torch.empty(T, N, 5).exponential_(generator=torch.Generator().manual_seed(9))
    dev = DEV
    cfg, model, traj, _, sampler, learner = build(ocfg, N, st, tape, engine)
    assert model.spec.dict_obs and learner.heads_plan.keys and not sampler.fused_rollout
    if not decoder:     # the concatenation feeds the heads directly: unfused heads
        assert learner.heads_plan.P == 0 and sampler.heads_plan.P == 0
    sampler.reset()
    sampler.noise = noise.to(dev).contiguous()
    sampler.rollout()
    otraj = O.alloc_trajectories(ocfg, N)
    oenv = O.TapeVecEnv(tape, 5)
    O.rollout(ocfg, {k: v.clone() for k, v in st.items()}, oenv, oenv.reset(), otraj, noise, 0)
    got = {k: v.cpu() for k, v in traj.items()}
    assert torch.equal(got["obs"], otraj["obs"])
    assert torch.equal(got["actions"].view(-1), otraj["actions"].view(-1))
    np.testing.assert_allclose(got["action_logits"].numpy(), otraj["action_logits"].numpy(), atol=TOL)
    np.testing.assert_allclose(got["values"][:, :-1].numpy(), otraj["values"][:, :-1].numpy(), atol=TOL)
    olearner = O.OracleLearner(ocfg, st)
    olearner.train({k: v.clone() for k, v in otraj.items()})
    learner.train(traj)
    torch.cuda.synchronize()
    got_state = model.state_dict()
    for k in O.param_names(ocfg):
        np.testing.assert_allclose(got_state[k].cpu().numpy(), olearner.st[k].numpy(), atol=2 * TOL, rtol=1e-5, err_msg=k)
    for k, _ in keys:
        mean = f"{DO.NORM_BASE}{k}.running_mean"
        np.testing.assert_allclose(got_state[mean].cpu().numpy(), olearner.st[mean].numpy(), atol=1e-8, rtol=1e-6)


# ------------------------------------------------------------------------------------------------ vs the reference
GOLDEN = ["tiny_dict", "tiny_dict_lstm", "tiny_dict_mask"]


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", GOLDEN)
def test_sampler_matches_reference_golden(name, engine):
    """the sampler on the reference's weights, packed obs tape and noise: Discrete actions bit-exact, policy outputs 1e-5"""
    case = DO.load_dict_case(name)
    replay_sampler(case, build_case(case, engine), exact=("obs", "dones", "rewards", "actions"))


def _learner_vs_golden(name, engine, graph):
    case = DO.load_dict_case(name)
    rig = build_case(case, engine, learner_cuda_graph=graph)
    assert rig.learner.use_graph == graph
    replay_learner(case, rig, traj_of=DO.traj_from)


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", GOLDEN)
def test_learner_matches_reference_golden(name, engine):
    """Learner.train on the reference's trajectories: returns, advantages, losses at 1e-5, post-Adam weights and the
    per-key normaliser statistics against the reference's"""
    _learner_vs_golden(name, engine, graph=False)


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", ["tiny_dict_lstm", "tiny_dict_mask"])
def test_graphed_learner_matches_reference_golden(name, engine):
    """the same through one CUDA graph per train() (one epoch: tiny_dict_lstm, tiny_dict_mask)"""
    _learner_vs_golden(name, engine, graph=True)


# ------------------------------------------------------------------------------------------------ gymnasium-API envs
class _Box:
    def __init__(self, shape, dtype=np.float32):
        self.shape, self.dtype = shape, dtype


class _Discrete:
    def __init__(self, n):
        self.n, self.shape = n, ()


class _Dict:
    def __init__(self, spaces):
        self.spaces = spaces


def _goal_obs(t, i, mask):
    b = 0.1 * t + 0.01 * i
    o = {"observation": np.sin(np.arange(6, dtype=np.float32) + b).astype(np.float32),
         "desired_goal": np.array([t % 3, i % 5, 1]), "achieved_goal": np.cos(np.arange(3) * b)}    # int64 / float64 keys
    if mask:
        o["action_mask"] = np.array([1, 1, 0, (t + i) % 2], dtype=np.int8)
    return o


class GoalEnv:
    """single-agent gymnasium-API env: Dict(achieved_goal [3] float64, desired_goal [3] int64, observation [6] float32,
    action_mask [4]), Discrete(4); episodes of 9 steps"""

    def __init__(self, i):
        self.i, self.t = i, 0
        self.observation_space = _Dict({"observation": _Box((6,)), "desired_goal": _Box((3,), np.int64),
                                        "achieved_goal": _Box((3,), np.float64), "action_mask": _Box((4,), np.int8)})
        self.action_space = _Discrete(4)

    def reset(self, seed=None):
        self.t = 0
        return _goal_obs(self.t, self.i, True), {}

    def step(self, a):
        assert 0 <= int(a) < 4
        self.t += 1
        return _goal_obs(self.t, self.i, True), float(a == 1), self.t >= 9, False, {}


class GoalMultiAgentEnv:
    """multi-agent version: two agents, one observation dict per agent, the env resets itself"""

    is_multiagent = True
    num_agents = 2

    def __init__(self, i):
        self.i, self.t = i, 0
        self.observation_space = _Dict({"observation": _Box((6,)), "desired_goal": _Box((3,), np.int64),
                                        "achieved_goal": _Box((3,), np.float64)})
        self.action_space = _Discrete(4)

    def _obs(self):
        return [_goal_obs(self.t, 2 * self.i + j, False) for j in range(2)]

    def reset(self, seed=None):
        self.t = 0
        return self._obs(), {}

    def step(self, actions):
        self.t += 1
        done = self.t >= 7
        if done:
            self.t = 0
        return self._obs(), [1.0, 0.0], [done, done], [False, False], [{}, {}]


def _packed(t, i, mask):
    o = _goal_obs(t, i, mask)
    return np.concatenate([o["achieved_goal"], o["desired_goal"], o["observation"]]).astype(np.float32)


@pytest.mark.parametrize("multi_agent", [False, True])
def test_host_env_dict_rows_run_rl_and_enjoy(tmp_path, multi_agent):
    """a three-key Dict through BatchedHostEnv: packed rows in sorted key order (float / int keys cast to float32), the
    action mask kept apart; run_rl trains on it (default model: per-key MLPs -> GRU core) and enjoy() runs its checkpoint"""
    from sample_factory_b200.cfg import parse_full_cfg, parse_sf_args
    from sample_factory_b200.checkpoint import checkpoint_dir, get_checkpoints
    from sample_factory_b200.enjoy import enjoy
    from sample_factory_b200.envs import register_env
    from sample_factory_b200.host_env import BatchedHostEnv
    from sample_factory_b200.train import run_rl

    ops_for()
    dev = torch.device("cuda", 0)
    cls = GoalMultiAgentEnv if multi_agent else GoalEnv
    env = BatchedHostEnv(cls, 4, dev)
    assert env.obs_keys == [("achieved_goal", 3), ("desired_goal", 3), ("observation", 6)] and env.obs_dim == 12
    obs = env.reset()
    rows = (obs if multi_agent else obs["obs"]).cpu().numpy()
    for r in range(env.num_agents):
        np.testing.assert_array_equal(rows[r], _packed(0, r, not multi_agent))
    if not multi_agent:
        assert obs["action_mask"].cpu().tolist()[3] == [True, True, False, True]
    name = f"goal_dict_{int(multi_agent)}"
    register_env(name, lambda full_env_name, cfg, env_config, render_mode=None: cls(
        (env_config or {}).get("env_id", 0)))
    argv = [f"--env={name}", f"--experiment={name}", f"--train_dir={tmp_path}", "--restart_behavior=overwrite",
            "--rollout=16", "--batch_size=256", "--num_batches_per_epoch=1", "--encoder_mlp_layers", "32", "32",
            "--async_rl=False", "--batched_sampling=True", "--num_workers=1", "--num_envs_per_worker=16" if not multi_agent
            else "--num_envs_per_worker=8", "--worker_num_splits=1", "--seed=0", "--train_for_env_steps=1024",
            "--save_every_sec=100000", "--experiment_summaries_interval=100000"]
    parser, _ = parse_sf_args(argv)
    cfg = parse_full_cfg(parser, argv)
    assert run_rl(cfg) == 0
    files = get_checkpoints(checkpoint_dir(cfg, 0))
    sd = torch.load(files[-1], map_location="cpu", weights_only=False)["model"]
    for k, d in env.obs_keys:
        assert sd[f"encoder.encoders.{k}.mlp_head.0.weight"].shape == (32, d)
        assert sd[f"obs_normalizer.running_mean_std.running_mean_std.{k}.running_mean"].shape == (d,)
    assert sd["core.core.weight_ih_l0"].shape == (3 * 512, 96)      # (the reference's default GRU core reads the concatenation)
    cfg.cli_args = dict(max_num_episodes=8)
    cfg.max_num_episodes = 8
    status, avg = enjoy(cfg)
    assert status == 0 and np.isfinite(avg)


# ------------------------------------------------------------------------------------------------ full size
PEAK_GIB = 1.5


def test_dict_goal_env_4096_envs_full_size():
    """keys (25, 3, 3) with MLP [512, 512] per key through Runner: 4096 envs, T = 32, 4 x 32768 minibatches.  Peak
    allocated memory stays under 1.5 GiB (0.99 GiB measured by this test on an H100 80GB HBM3); the large items: per key
    one [32768, 512] hidden activation and its gradient, the [32768, 1536] concatenation and its gradient, the trajectories."""
    from sample_factory_b200.envs import TapeVecEnv

    dev = torch.device("cuda", 0)
    N, T = 4096, 32
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    keys = [("achieved_goal", 3), ("desired_goal", 3), ("observation", 25)]
    tape = torch.randn(2 * T + 1, N, 31, generator=torch.Generator().manual_seed(2)).to(dev)
    r = runner("synthetic_goal_dict", lambda name, cfg, env_config, render_mode=None: TapeVecEnv(tape, 8, obs_keys=keys),
                ["--use_rnn=False", "--async_rl=False", f"--rollout={T}", "--recurrence=1", "--batch_size=32768", "--num_batches_per_epoch=4",
                 "--encoder_mlp_layers", "512", "512"])
    assert r.model.spec.obs_keys == keys and r.model.spec.fc_encoder_input == 1536
    assert not getattr(r.sampler, "fused_rollout", False)
    w = r.model.params["encoder.encoders.desired_goal.mlp_head.0.weight"].clone()
    st = check_finite(r, 2, 2 * N * T)
    assert st["num_valid"] == 32768
    assert not torch.equal(w, r.model.params["encoder.encoders.desired_goal.mlp_head.0.weight"])
    peak = (torch.cuda.max_memory_allocated() - base) / 2**30
    print(f"peak allocated: {peak:.2f} GiB")
    assert peak < PEAK_GIB, peak
