"""Batched tensor envs (IsaacGym / Brax style: one env, num_agents = N, torch tensors batched along dim 0) on the host side:
the attributes BatchedTensorEnvAdapter derives from the spaces, and which adapter create_batched_env picks -- with the
call sequence of every other kind of env unchanged."""
import numpy as np
import pytest
import torch

from gymnasium import spaces

CPU = torch.device("cpu")


class SpacesEnv:
    def __init__(self, observation_space, action_space, n=6):
        self.observation_space, self.action_space, self.num_agents = observation_space, action_space, n


def _adapter(obs_space, act_space, n=6):
    from sample_factory_b200.host_env import BatchedTensorEnvAdapter

    return BatchedTensorEnvAdapter(SpacesEnv(obs_space, act_space, n), CPU, env_gpu_actions=True)


BOX4 = spaces.Box(-1.0, 1.0, (4,), np.float32)
SPACE_CASES = {
    "discrete": (BOX4, spaces.Discrete(5),
                 dict(obs_dim=4, num_actions=5, continuous=False, action_segments=None, action_heads=None, obs_keys=None)),
    "box": (BOX4, spaces.Box(-1.0, 1.0, (3,), np.float32),
            dict(obs_dim=4, num_actions=3, continuous=True, action_segments=None, action_heads=None)),
    "tuple_discrete": (BOX4, spaces.Tuple([spaces.Discrete(3), spaces.Discrete(2)]),
                       dict(num_actions=5, continuous=False, action_segments=[3, 2], action_heads=None)),
    "tuple_box": (BOX4, spaces.Tuple([spaces.Discrete(3), spaces.Box(-1.0, 1.0, (2,), np.float32)]),
                  dict(num_actions=7, continuous=False, action_segments=None, action_heads=[("discrete", 3), ("box", 2)])),
    "dict_keys": (spaces.Dict({"b": spaces.Box(-1.0, 1.0, (3,), np.float32), "a": spaces.Box(0, 9, (2,), np.int64)}),
                  spaces.Discrete(4), dict(obs_dim=5, obs_keys=[("a", 2), ("b", 3)], obs_shape=None, obs_uint8=False)),
    "uint8_image": (spaces.Dict({"obs": spaces.Box(0, 255, (3, 8, 8), np.uint8)}), spaces.Discrete(4),
                    dict(obs_dim=192, obs_shape=(3, 8, 8), obs_uint8=True, obs_keys=None)),
    "mask": (spaces.Dict({"obs": BOX4, "action_mask": spaces.Box(0, 1, (6,), np.int8)}), spaces.Discrete(6),
             dict(obs_dim=4, num_actions=6, obs_keys=None, _mask_key="action_mask")),
}


@pytest.mark.parametrize("case", sorted(SPACE_CASES))
def test_spaces_give_the_engine_attributes(case):
    obs_space, act_space, want = SPACE_CASES[case]
    a = _adapter(obs_space, act_space)
    for k, v in want.items():
        assert getattr(a, k) == v, (case, k, getattr(a, k))
    assert a.num_agents == 6 and a.static_outputs and not a.is_gpu_env
    assert a.obs.shape == (6, a.obs_dim) and a.obs.dtype == (torch.uint8 if a.obs_uint8 else torch.float32)
    assert (a.action_mask is not None) == (case == "mask")


def test_extra_returned_keys_are_ignored_and_bare_tensors_are_the_obs_key():
    a = _adapter(BOX4, spaces.Discrete(2))
    assert a._obs_dst == [("obs", 4, 0, 0)]
    a = _adapter(spaces.Dict({"obs": BOX4}), spaces.Discrete(2))
    assert [k for k, *_ in a._obs_dst] == ["obs"]      # IsaacGym's "states" beside "obs" is never read


def test_non_dense_keys_are_refused_with_their_name():
    a = _adapter(spaces.Dict({"obs": spaces.Box(-1.0, 1.0, (2, 3), np.float32)}), spaces.Discrete(2), n=4)
    bad = torch.zeros(4, 2, 6)[:, :, ::2]
    with pytest.raises(ValueError, match="'obs'.*not dense"):
        a._ingest({"obs": bad})
    with pytest.raises(ValueError, match="'reward'"):
        a._src(torch.zeros(4, 2)[:, 0:1].expand(4, 3), "reward", 1)


# ------------------------------------------------------------------------------------------------ detection
class _NoEvent:
    def record(self, *a):
        pass

    def synchronize(self):
        pass


class RecordingEnv:
    """kind: "single" (gymnasium single-agent, numpy), "ma_list" (multi-agent, lists), "ma_numpy" (multi-agent, numpy
    arrays), "tensor" (batched torch tensors: the adapter's kind)"""

    def __init__(self, kind, idx, log):
        self.kind, self.idx, self.log = kind, idx, log
        self.observation_space = spaces.Box(-1.0, 1.0, (3,), np.float32)
        self.action_space = spaces.Discrete(2)
        if kind != "single":
            self.num_agents = 4
            self.is_multiagent = True

    def _obs(self):
        if self.kind == "single":
            return np.full(3, self.idx, np.float32)
        if self.kind == "ma_list":
            return [np.full(3, self.idx, np.float32) for _ in range(4)]
        if self.kind == "ma_numpy":
            return np.full((4, 3), self.idx, np.float32)
        return {"obs": torch.full((4, 3), float(self.idx)), "states": torch.zeros(4, 9)}

    def reset(self, **kw):
        self.log.append((self.idx, "reset", tuple(sorted(kw.items()))))
        return self._obs(), {}

    def step(self, actions):
        self.log.append((self.idx, "step", str(np.asarray(actions).tolist())))
        if self.kind == "single":
            return self._obs(), 1.0, False, False, {}
        return self._obs(), [1.0] * 4, [False] * 4, [False] * 4, [{}] * 4


def _cfg(name, **over):
    from sample_factory_b200.cfg import default_cfg

    cfg = default_cfg()
    cfg.env, cfg.num_workers, cfg.num_envs_per_worker, cfg.seed = name, 1, 3, 11
    for k, v in over.items():
        setattr(cfg, k, v)
    return cfg


def _register(kind, log):
    from sample_factory_b200.envs import register_env

    counter = iter(range(1000))
    name = f"recording_{kind}"
    register_env(name, lambda full_name, cfg, env_config, render_mode=None: RecordingEnv(kind, next(counter), log))
    return name


@pytest.mark.parametrize("kind", ["single", "ma_list", "ma_numpy"])
def test_host_envs_keep_their_path_and_call_sequence(kind, monkeypatch):
    """gymnasium single-agent envs and multi-agent envs returning lists / numpy still get BatchedHostEnv, and every env
    instance sees exactly the reset / step calls it saw when BatchedHostEnv was built directly"""
    from sample_factory_b200.envs import create_env
    from sample_factory_b200.host_env import BatchedHostEnv, create_batched_env

    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)     # (no CUDA driver here)
    monkeypatch.setattr(torch.cuda, "Event", _NoEvent)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: None)

    def drive(env):
        env.reset()
        for _ in range(2):
            env.step(torch.zeros(env.num_agents, dtype=torch.int32))

    log_new, log_old = [], []
    cfg = _cfg(_register(kind, log_new))
    env = create_batched_env(cfg, dict(worker_index=0, vector_index=0, env_id=0), CPU)
    assert type(env) is BatchedHostEnv
    drive(env)
    cfg_old = _cfg(_register(kind, log_old))
    env = BatchedHostEnv(lambda i: create_env(cfg_old.env, cfg_old, {}), 3, CPU, seed=11)
    drive(env)
    per_env = lambda log: sorted(log, key=lambda e: e[0])     # (stable: each instance's calls in their order)
    assert per_env(log_new) == per_env(log_old)
    assert (0, "reset", (("seed", 11),)) in log_new and sum(e[1] == "reset" for e in log_new) == 3


def test_tensor_batched_env_gets_the_adapter_with_one_reset():
    from sample_factory_b200.host_env import BatchedTensorEnvAdapter, create_batched_env

    log = []
    cfg = _cfg(_register("tensor", log), env_gpu_actions=True)
    env = create_batched_env(cfg, dict(worker_index=0, vector_index=0, env_id=0), CPU)
    assert type(env) is BatchedTensorEnvAdapter
    assert env.num_agents == 4 and env.obs_dim == 3 and env.env_gpu_actions
    assert log == [(0, "reset", (("seed", 11),))]      # one env (no num_workers x num_envs_per_worker copies), one reset
    assert env._first_reset is not None                # handed to the adapter's first reset()


def test_num_policies_above_one_is_refused():
    from sample_factory_b200.host_env import create_batched_env

    cfg = _cfg(_register("tensor", []), num_policies=2)
    with pytest.raises(ValueError, match="num_policies=2 with the batched tensor env RecordingEnv"):
        create_batched_env(cfg, dict(worker_index=0, vector_index=0, env_id=0), CPU)
    cfg = _cfg(_register("tensor", []))
    with pytest.raises(ValueError, match="num_policies=2"):
        create_batched_env(cfg, dict(worker_index=0, vector_index=0, env_id=0, policy_index=0, num_policies=2), CPU)
