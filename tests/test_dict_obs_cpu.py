"""Dict observations with several 1-D keys (MultiInputEncoder) off the GPU: the CPU oracle with its Dict extension
(tests/dict_obs_oracle.py) against the reference-executed fixtures tiny_dict / tiny_dict_lstm / tiny_dict_mask (made by
tests/golden/make_golden_dict_obs.py), the parameter list against the reference's state_dict, the host env's packing and
refusals, and the reference's checkpoint of a Dict model loading through checkpoint.py."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import appo_oracle as O
from tests import dict_obs_oracle as DO
from tests.golden_utils import state_from

CASES = ["tiny_dict", "tiny_dict_lstm", "tiny_dict_mask"]


def _spec(cfg, **kw):
    from sample_factory_b200.model import ModelSpec

    return ModelSpec(cfg.obs_dim, cfg.num_actions, list(cfg.encoder_mlp_layers), list(cfg.decoder_mlp_layers),
                     cfg.nonlinearity, use_rnn=cfg.use_rnn, rnn_type=cfg.rnn_type, rnn_size=cfg.rnn_size,
                     continuous=cfg.continuous, obs_keys=cfg.obs_keys, **kw)


@pytest.mark.parametrize("name", CASES)
def test_fixture_packs_the_reference_key_buffers(name):
    z, meta, cfg = DO.load_dict_case(name)
    for it in range(meta["iters"]):
        packed = np.concatenate([z[f"it{it}/traj/obs/{k}"] for k, _ in cfg.obs_keys], axis=2)
        np.testing.assert_array_equal(packed, z[f"it{it}/traj/obs"])


@pytest.mark.parametrize("name", CASES)
def test_oracle_rollout_matches_reference(name):
    z, meta, cfg = DO.load_dict_case(name)
    env = O.TapeVecEnv(torch.from_numpy(z["tape"]), cfg.num_actions, with_action_mask=cfg.action_mask)
    last_obs = env.reset()
    rnn_state = torch.zeros(meta["N"], O.rnn_state_size(cfg))
    for it in range(meta["iters"]):
        st = state_from(z, "init/") if it == 0 else state_from(z, f"it{it - 1}/state/")
        traj = O.alloc_trajectories(cfg, meta["N"])
        noise = torch.from_numpy(z[f"it{it}/noise"])
        last_obs = O.rollout(cfg, st, env, last_obs, traj, noise, int(z[f"it{it}/train_step_before"]), rnn_state)
        skip = {"policy_id", "policy_version"} if (meta["poison"] and it == meta["iters"] - 1) else set()
        float_actions = ["actions", "rewards"] if cfg.continuous else []   # Box: eps * std + mean of the restated forward
        for k in ["obs", "actions", "rewards", "dones", "time_outs", "policy_id", "policy_version"]:
            if k in float_actions:
                np.testing.assert_allclose(traj[k].numpy(), z[f"it{it}/traj/{k}"], atol=1e-5, rtol=0, err_msg=k)
            elif k not in skip:
                np.testing.assert_array_equal(traj[k].numpy(), z[f"it{it}/traj/{k}"], err_msg=k)
        np.testing.assert_allclose(traj["rnn_states"].numpy(), z[f"it{it}/traj/rnn_states"], atol=1e-6, rtol=0)
        for k in ["action_logits", "log_prob_actions"]:
            np.testing.assert_allclose(traj[k].numpy(), z[f"it{it}/traj/{k}"], atol=1e-6, rtol=0, err_msg=k)
        np.testing.assert_allclose(traj["values"][:, :-1].numpy(), z[f"it{it}/traj/values"][:, :-1], atol=1e-6, rtol=0)


@pytest.mark.parametrize("name", CASES)
def test_oracle_learner_matches_reference(name):
    z, meta, cfg = DO.load_dict_case(name)
    learner = O.OracleLearner(cfg, state_from(z, "init/"))
    for it in range(meta["iters"]):
        assert learner.train_step == int(z[f"it{it}/train_step_before"])
        n_log = len(learner.log)
        mb_key = f"it{it}/mb_indices"
        mb_indices = [torch.from_numpy(r.copy()) for r in z[mb_key]] if mb_key in z.files else None
        buff = learner.train(DO.traj_from(z, it, cfg), mb_indices=mb_indices)
        assert learner.train_step == int(z[f"it{it}/train_step_after"])
        p = f"it{it}/prep/"
        np.testing.assert_array_equal(buff["valids"].numpy(), z[p + "valids"])
        for k in ["advantages", "returns"]:
            np.testing.assert_allclose(buff[k].numpy(), z[p + k], atol=1e-5, rtol=0, err_msg=k)
        logs = learner.log[n_log:]
        for key in ["policy_loss", "value_loss", "exploration_loss", "kl_loss", "adv_mean", "adv_std"]:
            got = np.array([d[key] for d in logs])
            np.testing.assert_allclose(got, z[f"it{it}/loss/{key}"], atol=1e-5, rtol=1e-5, err_msg=key)
        for k, v in state_from(z, f"it{it}/state/").items():
            tol = 1e-9 if v.dtype == torch.float64 else 1e-5
            np.testing.assert_allclose(learner.st[k].numpy(), v.numpy(), atol=tol, rtol=1e-6, err_msg=k)


def test_oracle_extension_keeps_single_key_models():
    a = O.OracleCfg(obs_dim=10, num_actions=4, encoder_mlp_layers=[16])
    b = DO.DictCfg(obs_dim=10, num_actions=4, encoder_mlp_layers=[16], obs_keys=[("obs", 10)])
    assert O.param_names(a) == O.param_names(b)
    sa, sb = O.init_state(a, seed=1), O.init_state(b, seed=1)
    assert sa.keys() == sb.keys() and all(torch.equal(sa[k], sb[k]) for k in sa)


@pytest.mark.parametrize("name", CASES)
def test_param_shapes_match_reference_state_dict(name):
    """names, order and shapes of param_shapes() are the reference's trainable state_dict entries"""
    z, _meta, cfg = DO.load_dict_case(name)
    ref = [(k[len("init/"):], tuple(z[k].shape)) for k in z.files if k.startswith("init/")]
    ref = [(k, s) for k, s in ref if not k.startswith(("obs_normalizer.", "returns_normalizer."))]
    assert _spec(cfg).param_shapes() == ref
    assert O.param_names(cfg) == [k for k, _ in ref]


def test_model_spec_obs_keys_checks_and_from_cfg():
    from sample_factory_b200.cfg import default_cfg
    from sample_factory_b200.model import ModelSpec

    assert "obs_keys" in ModelSpec.__dataclass_fields__ and ModelSpec.__dataclass_fields__["obs_keys"].kw_only
    spec = ModelSpec(19, 5, [64, 64], obs_keys=[("achieved_goal", 3), ("desired_goal", 3), ("observation", 13)])
    assert spec.dict_obs and spec.key_offsets == [0, 3, 6] and spec.fc_encoder_input == 192 and spec.hidden == []
    assert spec.tail_input_size == 192
    one = ModelSpec(13, 5, [64], obs_keys=[("observation", 13)])
    assert not one.dict_obs and one.param_shapes()[0][0] == "encoder.encoders.observation.mlp_head.0.weight"
    with pytest.raises(ValueError, match="sorted"):
        ModelSpec(6, 5, [8], obs_keys=[("b", 3), ("a", 3)])
    with pytest.raises(ValueError, match="obs_dim"):
        ModelSpec(7, 5, [8], obs_keys=[("a", 3), ("b", 3)])
    with pytest.raises(ValueError, match=">= 1"):
        ModelSpec(3, 5, [8], obs_keys=[("a", 3), ("b", 0)])
    with pytest.raises(ValueError, match="actor_critic_share_weights"):
        ModelSpec(6, 5, [8], share_weights=False, obs_keys=[("a", 3), ("b", 3)])
    with pytest.raises(ValueError, match="obs_scale"):
        ModelSpec(6, 5, [8], obs_scale=255.0, obs_keys=[("a", 3), ("b", 3)])
    with pytest.raises(ValueError, match="obs_subtract_mean"):
        ModelSpec(6, 5, [8], obs_subtract_mean=1.0, obs_keys=[("a", 3), ("b", 3)])
    cfg = default_cfg()
    env = SimpleNamespace(obs_dim=6, num_actions=4, obs_keys=[("a", 2), ("b", 4)])
    assert ModelSpec.from_cfg(cfg, env).obs_keys == [("a", 2), ("b", 4)]
    cfg.normalize_input_keys = ["a", "b"]
    assert ModelSpec.from_cfg(cfg, env).dict_obs
    cfg.normalize_input_keys = ["a"]
    with pytest.raises(ValueError, match="normalize_input_keys"):
        ModelSpec.from_cfg(cfg, env)


class _Space:
    def __init__(self, shape=None, n=None, dtype=np.float32):
        self.shape, self.dtype = shape, dtype
        if n is not None:
            self.n = n


class _Dict:
    def __init__(self, spaces):
        self.spaces = spaces


class _GoalEnv:
    """gymnasium-API env with a Dict observation: achieved_goal float64 [3], desired_goal int [3], observation float32 [5]"""

    def __init__(self, i, mask=False):
        self.i, self.t, self.mask = i, 0, mask
        spaces = {"observation": _Space((5,)), "desired_goal": _Space((3,), dtype=np.int64),
                  "achieved_goal": _Space((3,), dtype=np.float64)}
        if mask:
            spaces["action_mask"] = _Space((4,), dtype=np.int8)
        self.observation_space = _Dict(spaces)
        self.action_space = _Space(n=4)

    def _obs(self):
        b = 100 * self.i + 10 * self.t
        o = {"observation": np.arange(5, dtype=np.float32) + b, "desired_goal": np.array([1, 2, 3]) + b,
             "achieved_goal": np.array([0.5, 1.5, 2.5]) + b}
        if self.mask:
            o["action_mask"] = np.array([1, 0, 1, self.t % 2], dtype=np.int8)
        return o

    def reset(self, seed=None):
        self.t = 0
        return self._obs(), {}

    def step(self, a):
        self.t += 1
        return self._obs(), 1.0, False, False, {}


def test_host_env_packs_dict_keys_in_sorted_order(monkeypatch):
    from sample_factory_b200.host_env import BatchedHostEnv

    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)      # (no CUDA driver here: pageable buffers)

    env = BatchedHostEnv(lambda i: _GoalEnv(i, mask=True), 2, torch.device("cpu"))
    assert env.obs_keys == [("achieved_goal", 3), ("desired_goal", 3), ("observation", 5)] and env.obs_dim == 11
    assert not env.obs_uint8 and env.obs_shape is None
    for i, e in enumerate(env.envs):
        env._put_obs(i, e.reset()[0])
    row = env.obs_host[1].numpy()
    np.testing.assert_array_equal(row, np.concatenate([[100.5, 101.5, 102.5], [101, 102, 103], np.arange(5) + 100.0]))
    assert env.obs_host.dtype == torch.float32
    assert env.mask_host[0].tolist() == [True, False, True, False]


def test_host_env_refuses_unsupported_dict_keys():
    from sample_factory_b200.host_env import _main_obs_space

    with pytest.raises(NotImplementedError, match="image keys"):
        _main_obs_space(_Dict({"pixels": _Space((3, 8, 8)), "state": _Space((4,))}))
    with pytest.raises(NotImplementedError, match="scalar"):
        _main_obs_space(_Dict({"speed": _Space(()), "state": _Space((4,))}))
    space, key, keys = _main_obs_space(_Dict({"obs": _Space((4,)), "action_mask": _Space((2,))}))
    assert key == "obs" and keys is None and space.shape == (4,)
    assert _main_obs_space(_Dict({"observation": _Space((4,))}))[2] == [("observation", 4)]


def test_loads_dict_checkpoint_written_by_the_reference(tmp_path):
    """the checkpoint the reference's Learner.save() wrote after the last tiny_dict_lstm iteration: checkpoint.py restores
    every tensor, including the per-key normaliser statistics, and state_dict() writes it back in the reference's layout"""
    from sample_factory_b200.cfg import default_cfg
    from sample_factory_b200.checkpoint import checkpoint_dir, load_checkpoint
    from sample_factory_b200.model import PolicyModel
    from tests.rnn_layers_oracle import checkpoint_from

    z, meta, ocfg = DO.load_dict_case("tiny_dict_lstm")
    model = PolicyModel(_spec(ocfg), torch.device("cpu"))
    cfg = default_cfg()
    cfg.train_dir, cfg.experiment = str(tmp_path), "ck"
    ref = checkpoint_from(z)
    torch.save(ref, os.path.join(checkpoint_dir(cfg, 0), f"checkpoint_{ref['train_step']:09d}_{ref['env_steps']}.pth"))
    info = load_checkpoint(cfg, model, torch.device("cpu"))
    assert info["train_step"] == ref["train_step"]
    got = model.state_dict()
    assert list(got.keys()) == list(ref["model"].keys())
    assert "obs_normalizer.running_mean_std.running_mean_std.b.running_var" in got
    for k, v in ref["model"].items():
        assert got[k].dtype == v.dtype and got[k].shape == v.shape and torch.equal(got[k], v), k
    osd = model.optimizer_state_dict(info["opt_step"], ref["curr_lr"], (0.9, 0.999), 1e-6)
    for i, st in ref["optimizer"]["state"].items():
        assert torch.equal(osd["state"][i]["exp_avg"], st["exp_avg"]), i
        assert torch.equal(osd["state"][i]["exp_avg_sq"], st["exp_avg_sq"]), i
