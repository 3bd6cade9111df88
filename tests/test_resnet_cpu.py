"""resnet_impala image encoder (the reference's ResnetEncoder, model/encoder.py:153-221) without a GPU: the CPU oracle
against the reference-generated `tiny_resnet` fixture, the device model's parameter layout, and the cfg surface."""
import numpy as np

import tests.resnet_oracle as R
import tests.test_oracle_golden as G
from tests.golden_utils import load_case, state_from, traj_from

R.install()


def test_oracle_rollout_matches_reference_resnet():
    G.test_rollout_matches_reference("tiny_resnet")


def test_oracle_learner_matches_reference_resnet():
    """returns, advantages, loss terms and normaliser statistics (the shared check), then the post-Adam weights, which
    the fixture stores as float16 differences from the initial weights"""
    from oracle import appo_oracle as O

    G.test_learner_matches_reference("tiny_resnet")
    z, meta, cfg = load_case("tiny_resnet")
    learner = O.OracleLearner(cfg, state_from(z, "init/"))
    learner.train(traj_from(z, 0, cfg))
    ref = R.post_state(z, 0)
    for k in O.param_names(cfg):
        np.testing.assert_allclose(learner.st[k].numpy(), ref[k].numpy(), atol=1e-5, rtol=1e-6, err_msg=k)


def test_model_spec_layout_matches_reference_resnet():
    """ModelSpec.param_shapes() == the reference model's trainable parameters (keys, shapes, parameters() order)"""
    from oracle import appo_oracle as O
    from sample_factory_b200.model import ModelSpec

    z, meta, cfg = load_case("tiny_resnet")
    spec = ModelSpec(cfg.obs_dim, cfg.num_actions, nonlinearity=cfg.nonlinearity, obs_shape=tuple(meta["obs_shape"]),
                     encoder_conv_architecture="resnet_impala", encoder_conv_mlp_layers=list(cfg.encoder_conv_mlp_layers))
    normalizers = (O.OBS_MEAN, O.OBS_VAR, O.OBS_COUNT, O.RET_MEAN, O.RET_VAR, O.RET_COUNT)
    ref = [(k[len("init/"):], tuple(z[k].shape)) for k in z.files
           if k.startswith("init/") and k[len("init/"):] not in normalizers]
    assert spec.param_shapes() == ref
    assert [k for k, _ in ref] == O.param_names(cfg)
    # 10 -> 5 -> 3 -> 2 through the padded pools; the reference's conv_head_out_size for the frame sizes users run
    assert spec.conv_out_size == 32 * 2 * 2 == z["init/encoder.encoders.obs.mlp_layers.0.weight"].shape[1]
    assert ModelSpec(4 * 84 * 84, 6, obs_shape=(4, 84, 84), encoder_conv_architecture="resnet_impala").conv_out_size == 3872
    assert ModelSpec(3 * 64 * 64, 6, obs_shape=(3, 64, 64), encoder_conv_architecture="resnet_impala").conv_out_size == 2048
    # the plain conv stacks keep their layout
    atari = ModelSpec(4 * 84 * 84, 6, obs_shape=(4, 84, 84), encoder_conv_architecture="convnet_atari")
    assert [k for k, _ in atari.param_shapes()][:2] == ["encoder.encoders.obs.enc.conv_head.0.weight",
                                                        "encoder.encoders.obs.enc.conv_head.0.bias"]


def test_cfg_accepts_resnet_impala():
    from sample_factory_b200.cfg import parse_full_cfg, parse_sf_args, verify_cfg

    argv = ["--env=atari_breakout", "--use_rnn=False", "--encoder_conv_architecture=resnet_impala", "--encoder_conv_mlp_layers", "512"]
    parser, _ = parse_sf_args(argv)
    cfg = parse_full_cfg(parser, argv)
    assert cfg.encoder_conv_architecture == "resnet_impala"
    assert verify_cfg(cfg)


def test_oracle_resnet_forward_shapes():
    """the oracle's encoder on the frame size of the full-size run: [4, 84, 84] -> 32 x 11 x 11 -> FC"""
    import torch
    from oracle import appo_oracle as O

    cfg = O.OracleCfg(obs_dim=4 * 84 * 84, num_actions=6, obs_shape=(4, 84, 84), encoder_conv_architecture="resnet_impala",
                      encoder_conv_mlp_layers=[16])
    st = O.init_state(cfg, seed=1)
    assert R.conv_out_shape(cfg) == (32, 11, 11)
    h = O.encoder_forward(cfg, st, torch.rand(2, cfg.obs_dim))
    assert h.shape == (2, 16) and np.isfinite(h.numpy()).all()
