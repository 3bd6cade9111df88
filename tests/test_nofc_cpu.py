"""Encoders without fully connected layers (--encoder_mlp_layers / --encoder_conv_mlp_layers empty) off the GPU: the CPU
oracle against the reference-executed fixtures of tests/golden/make_golden_nofc.py, the device model's parameter layout,
the reference's checkpoint, ModelSpec.from_cfg, and the combinations that stay refused."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import tests.resnet_oracle as R
import tests.test_oracle_golden as G
from oracle import appo_oracle as O
from tests import dict_obs_oracle as DO
from tests.golden_utils import load_case, state_from, traj_from

R.install()

CASES = ["tiny_linear", "tiny_linear_box", "tiny_conv_nofc", "tiny_conv_nofc_gru", "tiny_resnet_nofc"]
IMAGE_CASES = ["tiny_conv_nofc", "tiny_conv_nofc_gru", "tiny_resnet_nofc"]     # weights stored as float16 deltas


def spec_of(cfg, meta, **kw):
    from sample_factory_b200.model import ModelSpec

    return ModelSpec(cfg.obs_dim, cfg.num_actions, list(cfg.encoder_mlp_layers), list(cfg.decoder_mlp_layers),
                     cfg.nonlinearity, use_rnn=cfg.use_rnn, rnn_type=cfg.rnn_type, rnn_size=cfg.rnn_size,
                     continuous=cfg.continuous, adaptive_stddev=cfg.adaptive_stddev,
                     obs_shape=tuple(meta["obs_shape"]) if meta.get("obs_shape") else None,
                     encoder_conv_architecture=cfg.encoder_conv_architecture,
                     encoder_conv_mlp_layers=list(cfg.encoder_conv_mlp_layers), **kw)


@pytest.mark.parametrize("name", CASES)
def test_oracle_rollout_matches_reference(name):
    """trajectories bit for bit, policy outputs at 1e-6"""
    G.test_rollout_matches_reference(name)


@pytest.mark.parametrize("name", CASES)
def test_oracle_learner_matches_reference(name):
    """returns, advantages, loss terms, normaliser statistics (and for the vector cases the weights); the image cases'
    post-Adam weights are rebuilt from their float16 differences"""
    G.test_learner_matches_reference(name)
    if name not in IMAGE_CASES:
        return
    z, meta, cfg = load_case(name)
    learner = O.OracleLearner(cfg, state_from(z, "init/"))
    mb_indices = [torch.from_numpy(r.copy()) for r in z["it0/mb_indices"]] if "it0/mb_indices" in z.files else None
    learner.train(traj_from(z, 0, cfg), mb_indices=mb_indices)
    ref = R.post_state(z, 0)
    for k in O.param_names(cfg):
        np.testing.assert_allclose(learner.st[k].numpy(), ref[k].numpy(), atol=1e-5, rtol=1e-6, err_msg=k)


def test_oracle_dict_identity_matches_reference():
    import tests.test_dict_obs_cpu as D

    D.test_oracle_rollout_matches_reference("tiny_dict_identity")
    D.test_oracle_learner_matches_reference("tiny_dict_identity")


def _reference_layout(z):
    normalizers = (O.OBS_MEAN, O.OBS_VAR, O.OBS_COUNT, O.RET_MEAN, O.RET_VAR, O.RET_COUNT)
    return [(k[len("init/"):], tuple(z[k].shape)) for k in z.files
            if k.startswith("init/") and k[len("init/"):] not in normalizers]


@pytest.mark.parametrize("name", CASES)
def test_param_shapes_match_reference(name):
    """param_shapes() == the reference model's trainable parameters (keys, shapes, parameters() order)"""
    z, meta, cfg = load_case(name)
    spec = spec_of(cfg, meta)
    assert spec.param_shapes() == _reference_layout(z)
    assert spec.fc_encoder_layers == [] and spec.hidden == list(cfg.decoder_mlp_layers) and not spec.separate_towers
    assert spec.heads_read_input == (name in ("tiny_linear", "tiny_linear_box"))
    assert spec.tail_input_size == (cfg.decoder_mlp_layers[-1] if cfg.decoder_mlp_layers else spec.fc_encoder_input)


def test_dict_identity_layout_and_separate_identity_towers():
    from sample_factory_b200.model import ModelSpec

    z, meta, cfg = DO.load_dict_case("tiny_dict_identity")
    spec = ModelSpec(cfg.obs_dim, cfg.num_actions, [], obs_keys=list(cfg.obs_keys))
    assert spec.dict_obs and spec.heads_read_input and spec.param_shapes() == [
        (k, s) for k, s in _reference_layout(z) if not k.startswith("obs_normalizer.")]
    # ActorCriticSeparateWeights with identity towers: the parameters of the shared identity model, a state row of 2
    z, meta, cfg = load_case("tiny_linear")
    shared, separate = spec_of(cfg, meta), spec_of(cfg, meta, share_weights=False)
    assert separate.param_shapes() == shared.param_shapes() == _reference_layout(z)
    assert not separate.separate_towers and separate.heads_read_input
    assert (shared.rnn_state_size, separate.rnn_state_size) == (1, 2)


def test_wide_route_is_chosen_from_the_shape():
    """the narrow heads forward stages [critic_linear | distribution_linear] in 200 KB of shared memory; wider rows take
    the GEMM + heads_tail_wide route"""
    from sample_factory_b200.model import ModelSpec

    atari = ModelSpec(4 * 84 * 84, 6, [], obs_shape=(4, 84, 84), encoder_conv_mlp_layers=[])
    assert atari.conv_out_size == 3136 and not atari.wide_heads            # 7 * 3136 * 4 = 86 KB
    resnet = ModelSpec(4 * 84 * 84, 6, [], obs_shape=(4, 84, 84), encoder_conv_architecture="resnet_impala",
                       encoder_conv_mlp_layers=[])
    assert resnet.conv_out_size == 3872 and not resnet.wide_heads
    assert ModelSpec(4 * 84 * 84, 18, [], obs_shape=(4, 84, 84), encoder_conv_mlp_layers=[]).wide_heads    # 19 rows
    assert not ModelSpec(64, 8, [512, 512]).wide_heads and ModelSpec(64, 40, [512]).wide_heads


def test_loads_linear_checkpoint_written_by_the_reference():
    """the reference's checkpoint of tiny_linear (model + Adam state) into the device model's flat buffers, and back"""
    from sample_factory_b200.model import PolicyModel

    z, meta, cfg = load_case("tiny_linear")
    sd = {k: torch.from_numpy(z[f"ckpt/model/{k}"].copy()) for k in z["ckpt/model_keys"].tolist()}
    model = PolicyModel(spec_of(cfg, meta), torch.device("cpu"))
    model.load_state_dict(sd)
    out = model.state_dict()
    assert set(out) == set(sd)
    for k, v in sd.items():
        assert torch.equal(out[k].to(v.dtype).view(v.shape), v), k
    osd = dict(state={i: dict(step=torch.tensor(float(z[f"ckpt/optimizer/{i}/step"])),
                              exp_avg=torch.from_numpy(z[f"ckpt/optimizer/{i}/exp_avg"].copy()),
                              exp_avg_sq=torch.from_numpy(z[f"ckpt/optimizer/{i}/exp_avg_sq"].copy()))
                      for i in range(int(z["ckpt/num_opt_states"]))})
    assert len(osd["state"]) == len(model.names) == 4      # critic_linear, distribution_linear
    assert model.load_optimizer_state_dict(osd) == int(z["ckpt/train_step"])
    back = model.optimizer_state_dict(int(z["ckpt/train_step"]), 1e-4, (0.9, 0.999), 1e-6)
    for i, st in osd["state"].items():
        assert torch.equal(back["state"][i]["exp_avg"], st["exp_avg"].view(back["state"][i]["exp_avg"].shape))
        assert torch.equal(back["state"][i]["exp_avg_sq"], st["exp_avg_sq"].view(back["state"][i]["exp_avg_sq"].shape))


@pytest.mark.parametrize("flags,expect", [
    (dict(encoder_mlp_layers=[]), dict(hidden=[], heads_read_input=True)),
    (dict(encoder_mlp_layers=[], actor_critic_share_weights=False), dict(hidden=[], separate_towers=False)),
    (dict(obs_shape=(4, 84, 84), encoder_conv_mlp_layers=[], encoder_conv_architecture="convnet_atari"),
     dict(tail_input_size=3136, wide_heads=False)),
    (dict(obs_shape=(4, 84, 84), encoder_conv_mlp_layers=[], encoder_conv_architecture="resnet_impala"),
     dict(tail_input_size=3872)),
    (dict(obs_shape=(4, 84, 84), encoder_conv_mlp_layers=[], use_rnn=True, rnn_num_layers=2),
     dict(tail_input_size=512, fc_encoder_input=128 * 4 * 4)),
    (dict(obs_shape=(1, 36, 36), encoder_conv_mlp_layers=[], encoder_conv_architecture="convnet_simple",
          decoder_mlp_layers=[32]), dict(tail_input_size=32, hidden=[32])),
])
def test_from_cfg_builds_models_without_fc_layers(flags, expect):
    from sample_factory_b200.cfg import default_cfg
    from sample_factory_b200.model import ModelSpec

    cfg = default_cfg()
    cfg.use_rnn = False
    obs_shape = flags.pop("obs_shape", None)
    for k, v in flags.items():
        setattr(cfg, k, v)
    dim = int(np.prod(obs_shape)) if obs_shape else 24
    env = SimpleNamespace(obs_dim=dim, num_actions=6, obs_shape=obs_shape, obs_uint8=obs_shape is not None)
    spec = ModelSpec.from_cfg(cfg, env)
    for k, v in expect.items():
        assert getattr(spec, k) == v, k


def test_remaining_combinations_are_refused():
    from sample_factory_b200.model import ModelSpec

    with pytest.raises(ValueError, match="image encoder"):
        ModelSpec(4 * 84 * 84, 6, [], obs_shape=(4, 84, 84), encoder_conv_mlp_layers=[], share_weights=False)
    with pytest.raises(ValueError, match="actor_critic_share_weights=False"):
        ModelSpec(12, 5, [], obs_keys=[("a", 5), ("b", 7)], share_weights=False)
    with pytest.raises(ValueError, match="image keys"):
        ModelSpec(4 * 10 * 10 + 3, 5, [], obs_shape=(4, 10, 10), obs_keys=[("a", 3), ("obs", 400)])
