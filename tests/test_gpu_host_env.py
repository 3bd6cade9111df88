"""BatchedHostEnv (sample_factory_b200/host_env.py): ordinary single-agent CPU envs with the gymnasium API behind the
device sampler -- the plumbing of BASELINE.json config 1 (CartPole-v1, 64 envs).  The env here is a small CartPole
re-implementation (gymnasium is not installed in this image); the check is semantic equivalence with the oracle's
rollout over a CPU batched wrapper with the reference's auto-reset rule (make_env.py:89-94)."""
import numpy as np
import pytest
import torch

from oracle import appo_oracle as O
from tests.device_harness import MiniCartPole, make_cfg

pytestmark = pytest.mark.gpu


class CpuBatched:
    """what the reference's BatchedMultiAgentWrapper / SequentialVectorizeWrapper give the oracle's rollout()"""

    def __init__(self, envs, seed):
        self.envs, self.seed = envs, seed
        self.num_agents = len(envs)

    def reset(self):
        return torch.from_numpy(np.stack([e.reset(seed=self.seed + i)[0] for i, e in enumerate(self.envs)]))

    def step(self, actions):
        obs, rew, term, trunc = [], [], [], []
        for e, a in zip(self.envs, actions.tolist()):
            o, r, tm, tr, _ = e.step(int(a))
            if tm or tr:
                o, _ = e.reset()
            obs.append(o); rew.append(r); term.append(tm); trunc.append(tr)
        return (torch.from_numpy(np.stack(obs)), torch.tensor(rew, dtype=torch.float32), torch.tensor(term),
                torch.tensor(trunc))


def test_host_env_rollout_matches_oracle():
    from sample_factory_b200 import ops
    from sample_factory_b200.host_env import BatchedHostEnv
    from sample_factory_b200.model import ModelSpec, PolicyModel
    from sample_factory_b200.sampler import DeviceSampler
    from sample_factory_b200.trajectory import alloc_for_spec

    dev = torch.device("cuda", 0)
    ops.bind_device(dev)
    N, T = 16, 24
    ocfg = O.OracleCfg(obs_dim=4, num_actions=2, encoder_mlp_layers=[64, 64], nonlinearity="tanh", rollout=T, recurrence=1,
                       batch_size=N * T, num_batches_per_epoch=1, reward_scale=0.1)
    st = O.init_state(ocfg, seed=4)
    env = BatchedHostEnv(lambda i: MiniCartPole(), N, dev, seed=100)
    assert (env.obs_dim, env.num_actions, env.continuous, env.obs_shape) == (4, 2, False, None)
    cfg = make_cfg(ocfg)
    spec = ModelSpec.from_cfg(cfg, env)
    model = PolicyModel(spec, dev)
    model.load_state_dict(st, strict=False)
    traj = alloc_for_spec(spec, N, T, dev)
    # eager sampler with explicit noise: step-by-step equivalence with the oracle over the CPU batched wrapper
    env = BatchedHostEnv(lambda i: MiniCartPole(), N, dev, seed=100)
    sampler = DeviceSampler(cfg, env, model, traj, engine=ops.GEMM_SIMT, use_cuda_graph=False)
    sampler.reset()
    cpu_env = CpuBatched([MiniCartPole() for _ in range(N)], seed=100)
    last = cpu_env.reset()
    rnn_state = torch.zeros(N, 1)
    for it in range(2):
        noise = torch.empty(T, N, 2).exponential_(generator=torch.Generator().manual_seed(7 + it))
        ref = O.alloc_trajectories(ocfg, N)
        last = O.rollout(ocfg, st, cpu_env, last, ref, noise, 0, rnn_state)
        sampler.noise = noise.to(dev)
        sampler.set_policy_version(0)
        sampler.rollout()
        got = {k: v.cpu() for k, v in traj.items()}
        for k in ["obs", "rewards", "dones", "time_outs"]:
            assert torch.equal(got[k].view(ref[k].shape), ref[k]), (k, it)
        assert torch.equal(got["actions"].view(ref["actions"].shape), ref["actions"])
        np.testing.assert_allclose(got["values"][:, :-1].numpy(), ref["values"][:, :-1].numpy(), atol=1e-5)
    assert traj["dones"].any() and len(env.episode_infos) > 0
    # CUDA graphs around the host env.step (Philox noise): runs, finishes episodes, accounts its transfers
    env2 = BatchedHostEnv(lambda i: MiniCartPole(), N, dev, seed=100)
    sampler2 = DeviceSampler(cfg, env2, model, traj, engine=ops.GEMM_SIMT, use_cuda_graph=True)
    sampler2.reset()
    for _ in range(3):
        sampler2.rollout()
    torch.cuda.synchronize()
    assert sampler2.graph_replay_launches > 0
    assert torch.isfinite(traj["values"][:, :-1]).all() and traj["dones"].any()
    assert len(env2.episode_infos) > 0 and env2.h2d_bytes > 0 and env2.d2h_bytes > 0


def test_cartpole_learns_through_run_rl():
    """End to end through the reference-style public API (register_env + parse_full_cfg + Runner): PPO on the CartPole
    re-implementation behind BatchedHostEnv must actually learn -- the mean episode length has to grow well beyond the
    random-policy level (~22 steps).  Catches sign / scaling errors no parity test of a single kernel would."""
    from sample_factory_b200.cfg import parse_full_cfg, parse_sf_args
    from sample_factory_b200.envs import register_env
    from sample_factory_b200.host_env import BatchedHostEnv
    from sample_factory_b200.train import Runner

    dev = torch.device("cuda", 0)
    register_env("MiniCartPole-v0", lambda name, cfg, env_config, render_mode=None: BatchedHostEnv(
        lambda i: MiniCartPole(max_steps=200), 64, dev, seed=cfg.seed))
    argv = ["--env=MiniCartPole-v0", "--experiment=cartpole_test", "--train_dir=/tmp/sfb200_tests", "--restart_behavior=overwrite",
            "--use_rnn=False", "--recurrence=1", "--rollout=32", "--batch_size=512", "--num_batches_per_epoch=4",
            "--num_epochs=4", "--encoder_mlp_layers", "64", "64", "--nonlinearity=tanh", "--learning_rate=0.001",
            "--reward_scale=0.1", "--gamma=0.99", "--exploration_loss_coeff=0.001", "--async_rl=False", "--seed=0",
            "--save_every_sec=100000", "--experiment_summaries_interval=100000"]
    parser, _ = parse_sf_args(argv)
    cfg = parse_full_cfg(parser, argv)
    runner = Runner(cfg)
    runner.init()
    lens = []
    for it in range(300):
        runner.iteration()
        if it == 3 or (it + 1) % 25 == 0:       # first report after 4 iterations (~random policy), then every 25
            ep = runner.sampler.pop_episode_stats()
            if ep.get("episodes", 0) > 0:
                lens.append(ep["len"])
    torch.cuda.synchronize()
    st = runner.learner.fetch_stats()
    assert np.isfinite(st["loss"]) and runner.env_steps == 300 * 64 * 32
    assert lens[0] < 60, lens                  # early: close to the random policy
    assert max(lens[-4:]) > 2.5 * lens[0] and max(lens[-4:]) > 90, lens
