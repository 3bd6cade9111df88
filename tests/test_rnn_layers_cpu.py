"""Stacked recurrent cores (--rnn_num_layers > 1) off the GPU: the CPU oracle with its stacked-core extension
(tests/rnn_layers_oracle.py) against the reference-executed fixtures tiny_gru2 / tiny_lstm3 / tiny_shuffle_gru2 (made by
tests/golden/make_golden_rnn_layers.py), the parameter list and state size against torch / the reference's helper, the
cfg checks, and the reference's checkpoint of a two-layer model loading through checkpoint.py."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import appo_oracle as O
from tests import rnn_layers_oracle as RO
from tests.golden_utils import state_from, traj_from

CASES = ["tiny_gru2", "tiny_lstm3", "tiny_shuffle_gru2"]


@pytest.mark.parametrize("name", CASES)
def test_oracle_rollout_matches_reference(name):
    """the checks and tolerances of test_oracle_golden.py on the stacked-core fixtures"""
    z, meta, cfg = RO.load_stacked_case(name)
    assert cfg.rnn_num_layers >= 2 and O.rnn_state_size(cfg) == z["it0/traj/rnn_states"].shape[2]
    env = O.TapeVecEnv(torch.from_numpy(z["tape"]), cfg.num_actions)
    last_obs = env.reset()
    rnn_state = torch.zeros(meta["N"], O.rnn_state_size(cfg))
    for it in range(meta["iters"]):
        st = state_from(z, "init/") if it == 0 else state_from(z, f"it{it - 1}/state/")
        traj = O.alloc_trajectories(cfg, meta["N"])
        noise = torch.from_numpy(z[f"it{it}/noise"])
        last_obs = O.rollout(cfg, st, env, last_obs, traj, noise, int(z[f"it{it}/train_step_before"]), rnn_state)
        skip = {"policy_id", "policy_version"} if (meta["poison"] and it == meta["iters"] - 1) else set()
        for k in ["obs", "actions", "rewards", "dones", "time_outs", "policy_id", "policy_version"]:
            if k not in skip:
                np.testing.assert_array_equal(traj[k].numpy(), z[f"it{it}/traj/{k}"], err_msg=k)
        np.testing.assert_allclose(traj["rnn_states"].numpy(), z[f"it{it}/traj/rnn_states"], atol=1e-6, rtol=0)
        for k in ["action_logits", "log_prob_actions"]:
            np.testing.assert_allclose(traj[k].numpy(), z[f"it{it}/traj/{k}"], atol=1e-6, rtol=0, err_msg=k)
        np.testing.assert_allclose(traj["values"][:, :-1].numpy(), z[f"it{it}/traj/values"][:, :-1], atol=1e-6, rtol=0)


@pytest.mark.parametrize("name", CASES)
def test_oracle_learner_matches_reference(name):
    z, meta, cfg = RO.load_stacked_case(name)
    learner = O.OracleLearner(cfg, state_from(z, "init/"))
    assert "core.core.weight_hh_l1" in learner.names
    for it in range(meta["iters"]):
        assert learner.train_step == int(z[f"it{it}/train_step_before"])
        n_log = len(learner.log)
        mb_key = f"it{it}/mb_indices"
        mb_indices = [torch.from_numpy(r.copy()) for r in z[mb_key]] if mb_key in z.files else None
        buff = learner.train(traj_from(z, it, cfg), mb_indices=mb_indices)
        assert learner.train_step == int(z[f"it{it}/train_step_after"])
        p = f"it{it}/prep/"
        np.testing.assert_array_equal(buff["valids"].numpy(), z[p + "valids"])
        for k in ["advantages", "returns"]:
            np.testing.assert_allclose(buff[k].numpy(), z[p + k], atol=1e-5, rtol=0, err_msg=k)
        np.testing.assert_allclose(buff["rewards"].numpy(), z[p + "rewards"], atol=1e-6, rtol=0)
        logs = learner.log[n_log:]
        for key in ["policy_loss", "value_loss", "exploration_loss", "kl_loss", "adv_mean", "adv_std"]:
            got = np.array([d[key] for d in logs])
            np.testing.assert_allclose(got, z[f"it{it}/loss/{key}"], atol=1e-5, rtol=1e-5, err_msg=key)
        for k, v in state_from(z, f"it{it}/state/").items():
            tol = 1e-9 if v.dtype == torch.float64 else 1e-5
            np.testing.assert_allclose(learner.st[k].numpy(), v.numpy(), atol=tol, rtol=1e-6, err_msg=k)


def test_oracle_extension_keeps_one_layer_models():
    """a one-layer StackedCfg and a plain OracleCfg describe the same model"""
    a = O.OracleCfg(obs_dim=10, num_actions=4, encoder_mlp_layers=[16], use_rnn=True, rnn_type="lstm", rnn_size=8)
    b = RO.StackedCfg(obs_dim=10, num_actions=4, encoder_mlp_layers=[16], use_rnn=True, rnn_type="lstm", rnn_size=8)
    assert O.param_names(a) == O.param_names(b) and O.rnn_state_size(a) == O.rnn_state_size(b) == 16
    sa, sb = O.init_state(a, seed=1), O.init_state(b, seed=1)
    assert sa.keys() == sb.keys() and all(torch.equal(sa[k], sb[k]) for k in sa)


@pytest.mark.parametrize("rnn_type", ["gru", "lstm"])
@pytest.mark.parametrize("L", [1, 2, 3])
def test_param_shapes_match_torch_rnn(rnn_type, L):
    """the core's entries of param_shapes(): names, order and shapes of nn.GRU / nn.LSTM(num_layers=L) under the
    reference's `core.core.` prefix, between the encoder and the heads"""
    from sample_factory_b200.model import ModelSpec

    spec = ModelSpec(16, 4, [24], [20], use_rnn=True, rnn_type=rnn_type, rnn_size=12, rnn_num_layers=L)
    shapes = spec.param_shapes()
    names = [n for n, _ in shapes]
    core = [(n, s) for n, s in shapes if n.startswith("core.core.")]
    rnn = (torch.nn.GRU if rnn_type == "gru" else torch.nn.LSTM)(24, 12, L)
    assert core == [(f"core.core.{n}", tuple(p.shape)) for n, p in rnn.named_parameters()]
    first = names.index(core[0][0])
    assert names[first: first + len(core)] == [n for n, _ in core]      # contiguous, in parameters() order
    assert names[first - 1].startswith("encoder.") and names[first + len(core)] == "decoder.mlp.0.weight"
    assert dict(shapes)["decoder.mlp.0.weight"] == (20, 12)


@pytest.mark.parametrize("rnn_type", ["gru", "lstm"])
@pytest.mark.parametrize("L", [1, 2, 3])
def test_rnn_state_size_matches_reference_helper(rnn_type, L):
    from sample_factory.model.model_utils import get_rnn_size
    from sample_factory_b200.model import ModelSpec

    cfg = SimpleNamespace(use_rnn=True, rnn_size=40, rnn_num_layers=L, rnn_type=rnn_type, actor_critic_share_weights=True)
    spec = ModelSpec(8, 3, [16], use_rnn=True, rnn_type=rnn_type, rnn_size=40, rnn_num_layers=L)
    assert spec.rnn_state_size == get_rnn_size(cfg) == 40 * L * (2 if rnn_type == "lstm" else 1)
    assert O.rnn_state_size(RO.StackedCfg(use_rnn=True, rnn_type=rnn_type, rnn_size=40, rnn_num_layers=L)) == get_rnn_size(cfg)


def test_model_spec_reads_rnn_num_layers_from_cfg():
    from sample_factory_b200.cfg import default_cfg
    from sample_factory_b200.model import ModelSpec

    cfg = default_cfg()
    cfg.rnn_num_layers, cfg.rnn_type, cfg.rnn_size = 3, "lstm", 16
    spec = ModelSpec.from_cfg(cfg, SimpleNamespace(obs_dim=10, num_actions=4))
    assert spec.rnn_num_layers == 3 and spec.rnn_state_size == 3 * 2 * 16
    assert ModelSpec.__dataclass_fields__["rnn_num_layers"].default == 1
    assert list(ModelSpec.__dataclass_fields__)[-1] == "rnn_num_layers"     # positional construction keeps its meaning
    with pytest.raises(ValueError, match="rnn_num_layers"):
        ModelSpec(10, 4, [16], use_rnn=True, rnn_num_layers=0)


def test_verify_cfg_accepts_stacked_cores_and_rejects_zero(capsys):
    from sample_factory_b200.cfg import default_cfg, preprocess_cfg

    cfg = default_cfg()
    cfg.rnn_num_layers = 2
    assert preprocess_cfg(cfg)
    cfg = default_cfg()
    cfg.rnn_num_layers = 0
    assert not preprocess_cfg(cfg)
    assert "rnn_num_layers" in capsys.readouterr().err


def test_loads_two_layer_checkpoint_written_by_the_reference(tmp_path):
    """the checkpoint the reference's Learner.save() wrote after the last tiny_gru2 iteration (stored in the fixture,
    written back out with torch.save in the reference's file layout): checkpoint.py restores every tensor of the model
    and of the Adam state unchanged, and the weights are the reference's post-training state"""
    from sample_factory_b200.cfg import default_cfg
    from sample_factory_b200.checkpoint import checkpoint_dir, load_checkpoint
    from sample_factory_b200.model import ModelSpec, PolicyModel

    z, meta, ocfg = RO.load_stacked_case("tiny_gru2")
    spec = ModelSpec(ocfg.obs_dim, ocfg.num_actions, list(ocfg.encoder_mlp_layers), list(ocfg.decoder_mlp_layers),
                     use_rnn=True, rnn_type=ocfg.rnn_type, rnn_size=ocfg.rnn_size, rnn_num_layers=ocfg.rnn_num_layers)
    model = PolicyModel(spec, torch.device("cpu"))
    cfg = default_cfg()
    cfg.train_dir, cfg.experiment = str(tmp_path), "ck"
    ref = RO.checkpoint_from(z)
    torch.save(ref, os.path.join(checkpoint_dir(cfg, 0), f"checkpoint_{ref['train_step']:09d}_{ref['env_steps']}.pth"))
    info = load_checkpoint(cfg, model, torch.device("cpu"))
    assert info["train_step"] == ref["train_step"] and info["env_steps"] == ref["env_steps"]
    assert info["curr_lr"] == ref["curr_lr"]
    got = model.state_dict()
    assert list(got.keys()) == list(ref["model"].keys())
    assert any(k.endswith("_l1") for k in got)
    for k, v in ref["model"].items():
        assert got[k].dtype == v.dtype and torch.equal(got[k].view(v.shape), v), k
    for k, v in state_from(z, f"it{meta['iters'] - 1}/state/").items():
        assert torch.equal(got[k].view(v.shape), v), k
    osd = model.optimizer_state_dict(info["opt_step"], ref["curr_lr"], (0.9, 0.999), 1e-6)
    assert len(osd["state"]) == len(ref["optimizer"]["state"])
    for i, st in ref["optimizer"]["state"].items():
        assert torch.equal(osd["state"][i]["exp_avg"], st["exp_avg"]), i
        assert torch.equal(osd["state"][i]["exp_avg_sq"], st["exp_avg_sq"]), i
        assert float(osd["state"][i]["step"]) == float(st["step"])
    assert osd["param_groups"][0]["params"] == ref["optimizer"]["param_groups"][0]["params"]
