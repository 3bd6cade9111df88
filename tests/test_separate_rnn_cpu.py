"""Separate actor / critic weights with recurrent cores off the GPU: the CPU oracle with its extension
(tests/separate_rnn_oracle.py) against the reference-executed fixtures tiny_separate_gru / tiny_separate_lstm2 /
tiny_shuffle_separate_gru (made by tests/golden/make_golden_separate_rnn.py), the parameter layout and state width
against the reference, the reference's checkpoint through checkpoint.py, and the models the spec refuses."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import appo_oracle as O
from tests import separate_rnn_oracle as SO
from tests.golden_utils import state_from, traj_from

CASES = ["tiny_separate_gru", "tiny_separate_lstm2", "tiny_shuffle_separate_gru"]


def spec_of(ocfg):
    from sample_factory_b200.model import ModelSpec

    return ModelSpec(ocfg.obs_dim, ocfg.num_actions, list(ocfg.encoder_mlp_layers), list(ocfg.decoder_mlp_layers),
                     use_rnn=True, rnn_type=ocfg.rnn_type, rnn_size=ocfg.rnn_size, rnn_num_layers=ocfg.rnn_num_layers,
                     continuous=ocfg.continuous, share_weights=False)


@pytest.mark.parametrize("name", CASES)
def test_oracle_rollout_matches_reference(name):
    """trajectories bit for bit (actions, rewards, dones, ...), states / logits / values / log-probs at 1e-6.  Box
    actions are floats (eps * std + mean) and the reward is the first action component: they inherit the last-bit
    differences between torch's CPU LSTM and the oracle's written-out cell, so they are compared at 1e-6 too."""
    z, meta, cfg = SO.load_separate_rnn_case(name)
    assert not cfg.actor_critic_share_weights and O.rnn_state_size(cfg) == z["it0/traj/rnn_states"].shape[2]
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
            if k in skip:
                continue
            if cfg.continuous and k in ("actions", "rewards"):
                np.testing.assert_allclose(traj[k].numpy(), z[f"it{it}/traj/{k}"], atol=1e-6, rtol=0, err_msg=k)
            else:
                np.testing.assert_array_equal(traj[k].numpy(), z[f"it{it}/traj/{k}"], err_msg=k)
        np.testing.assert_allclose(traj["rnn_states"].numpy(), z[f"it{it}/traj/rnn_states"], atol=1e-6, rtol=0)
        for k in ["action_logits", "log_prob_actions"]:
            np.testing.assert_allclose(traj[k].numpy(), z[f"it{it}/traj/{k}"], atol=1e-6, rtol=0, err_msg=k)
        np.testing.assert_allclose(traj["values"][:, :-1].numpy(), z[f"it{it}/traj/values"][:, :-1], atol=1e-6, rtol=0)


@pytest.mark.parametrize("name", CASES)
def test_oracle_learner_matches_reference(name):
    z, meta, cfg = SO.load_separate_rnn_case(name)
    learner = O.OracleLearner(cfg, state_from(z, "init/"))
    assert "critic_core.core.weight_hh_l0" in learner.names
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
            if p + k in z.files:
                np.testing.assert_allclose(buff[k].numpy(), z[p + k], atol=1e-5, rtol=0, err_msg=k)
        np.testing.assert_allclose(buff["rewards"].numpy(), z[p + "rewards"], atol=1e-6, rtol=0)
        logs = learner.log[n_log:]
        for key in ["policy_loss", "value_loss", "exploration_loss", "kl_loss", "adv_mean", "adv_std"]:
            got = np.array([d[key] for d in logs])
            np.testing.assert_allclose(got, z[f"it{it}/loss/{key}"], atol=1e-5, rtol=1e-5, err_msg=key)
        for k, v in state_from(z, f"it{it}/state/").items():
            tol = 1e-9 if v.dtype == torch.float64 else 1e-5
            np.testing.assert_allclose(learner.st[k].numpy(), v.numpy(), atol=tol, rtol=1e-6, err_msg=k)


@pytest.mark.parametrize("name", CASES)
def test_param_shapes_match_reference(name):
    """param_shapes(): the reference's parameters() order and shapes (the fixture's init/ keys are its state_dict)"""
    z, _meta, ocfg = SO.load_separate_rnn_case(name)
    shapes = spec_of(ocfg).param_shapes()
    ref = [(k[len("init/"):], tuple(z[k].shape)) for k in z.files if k.startswith("init/")
           and not k.startswith(("init/obs_normalizer.", "init/returns_normalizer."))]
    assert shapes == ref
    assert [n for n, _ in shapes] == O.param_names(ocfg)


def test_oracle_extension_keeps_other_models():
    a = O.OracleCfg(obs_dim=10, num_actions=4, encoder_mlp_layers=[16], actor_critic_share_weights=False)
    b = SO.SeparateRnnCfg(obs_dim=10, num_actions=4, encoder_mlp_layers=[16], actor_critic_share_weights=False)
    assert O.param_names(a) == O.param_names(b) and O.rnn_state_size(a) == O.rnn_state_size(b) == 2
    st = O.init_state(a, seed=3)
    x = torch.randn(5, 10)
    va, la, _ = O.model_forward(a, st, x, torch.zeros(5, 2))
    vb, lb, _ = O.model_forward(b, st, x, torch.zeros(5, 2))
    assert torch.equal(va, vb) and torch.equal(la, lb)


@pytest.mark.parametrize("share", [True, False])
@pytest.mark.parametrize("L", [1, 2])
@pytest.mark.parametrize("rnn_type", ["gru", "lstm"])
def test_rnn_state_size_matches_reference_helper(rnn_type, L, share):
    from sample_factory.model.model_utils import get_rnn_size
    from sample_factory_b200.model import ModelSpec

    cfg = SimpleNamespace(use_rnn=True, rnn_size=24, rnn_num_layers=L, rnn_type=rnn_type,
                          actor_critic_share_weights=share)
    spec = ModelSpec(8, 3, [16], use_rnn=True, rnn_type=rnn_type, rnn_size=24, rnn_num_layers=L, share_weights=share)
    assert spec.rnn_state_size == get_rnn_size(cfg)
    assert spec.rnn_tower_state_size * (1 if share else 2) == get_rnn_size(cfg)


def test_checkpoint_written_by_the_reference_round_trips(tmp_path):
    """the checkpoint the reference's Learner.save() wrote after training tiny_separate_gru: checkpoint.py restores every
    tensor of the model and the Adam state, and state_dict() writes it back with the reference's keys in its order"""
    from sample_factory_b200.cfg import default_cfg
    from sample_factory_b200.checkpoint import checkpoint_dir, load_checkpoint
    from sample_factory_b200.model import PolicyModel

    z, meta, ocfg = SO.load_separate_rnn_case("tiny_separate_gru")
    model = PolicyModel(spec_of(ocfg), torch.device("cpu"))
    cfg = default_cfg()
    cfg.train_dir, cfg.experiment = str(tmp_path), "ck"
    ref = SO.checkpoint_from(z)
    torch.save(ref, os.path.join(checkpoint_dir(cfg, 0), f"checkpoint_{ref['train_step']:09d}_{ref['env_steps']}.pth"))
    info = load_checkpoint(cfg, model, torch.device("cpu"))
    assert info["train_step"] == ref["train_step"] and info["env_steps"] == ref["env_steps"]
    got = model.state_dict()
    assert list(got.keys()) == list(ref["model"].keys())
    assert any(k.startswith("critic_core.core.") for k in got)
    for k, v in ref["model"].items():
        assert got[k].dtype == v.dtype and torch.equal(got[k].view(v.shape), v), k
    osd = model.optimizer_state_dict(info["opt_step"], ref["curr_lr"], (0.9, 0.999), 1e-6)
    assert len(osd["state"]) == len(ref["optimizer"]["state"])
    for i, st in ref["optimizer"]["state"].items():
        assert torch.equal(osd["state"][i]["exp_avg"], st["exp_avg"]), i
        assert torch.equal(osd["state"][i]["exp_avg_sq"], st["exp_avg_sq"]), i


def test_rnn_params_and_tower_layers_per_tower():
    from sample_factory_b200.model import ModelSpec, PolicyModel

    spec = ModelSpec(10, 4, [16, 12], [8], use_rnn=True, rnn_type="lstm", rnn_size=6, rnn_num_layers=2,
                     share_weights=False)
    m = PolicyModel(spec, torch.device("cpu"), seed=5)
    for tw in ("actor_", "critic_"):
        W_ih, W_hh, b_ih, b_hh = m.rnn_params(layer=1, tower=tw)
        assert W_ih.data_ptr() == m.params[f"{tw}core.core.weight_ih_l1"].data_ptr() and W_ih.shape == (24, 6)
        assert m.rnn_params(layer=0, tower=tw)[0].shape == (24, 12)
        # torch-default init U(-1/sqrt(H), 1/sqrt(H)) for every core tensor, biases included
        for p in (W_ih, W_hh, b_ih, b_hh):
            assert float(p.abs().max()) <= 1 / 6 ** 0.5 and float(p.abs().max()) > 0
        enc, dec = m.tower_encoder_layers(tw), m.tower_decoder_layers(tw)
        assert [W.shape for W, _ in enc] == [(16, 10), (12, 16)] and [W.shape for W, _ in dec] == [(8, 6)]
        assert m.tower_layers(tw) == enc + dec
    assert not torch.equal(m.params["actor_core.core.weight_hh_l0"], m.params["critic_core.core.weight_hh_l0"])


def test_refusals():
    from sample_factory_b200.model import ModelSpec

    for arch in ("convnet_simple", "resnet_impala"):
        with pytest.raises(ValueError, match="actor_critic_share_weights=False.*image encoder"):
            ModelSpec(3 * 64 * 64, 4, share_weights=False, use_rnn=True, obs_shape=(3, 64, 64),
                      encoder_conv_architecture=arch)
    with pytest.raises(ValueError, match="actor_critic_share_weights"):
        ModelSpec(6, 5, [8], share_weights=False, use_rnn=True, obs_keys=[("a", 3), ("b", 3)])


def test_from_cfg_builds_the_default_recurrent_model():
    """the reference's defaults plus --actor_critic_share_weights=False: two GRU-512 cores"""
    from sample_factory_b200.cfg import default_cfg
    from sample_factory_b200.model import ModelSpec

    cfg = default_cfg()
    cfg.actor_critic_share_weights = False
    spec = ModelSpec.from_cfg(cfg, SimpleNamespace(obs_dim=10, num_actions=4))
    assert not spec.share_weights and spec.use_rnn and spec.rnn_type == "gru" and spec.rnn_size == 512
    assert spec.rnn_state_size == 2 * 512
    names = [n for n, _ in spec.param_shapes()]
    assert "actor_core.core.weight_ih_l0" in names and "critic_core.core.weight_hh_l0" in names
