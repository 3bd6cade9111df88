"""BASELINE.json configs 3, 4 and 5 at (or near) their named sizes through the public Runner API with synthetic envs:
size-independent properties only (the numerics of each ingredient are pinned by the reference goldens at small sizes:
tiny_gauss, tiny_conv, tiny_gru / tiny_lstm).  These runs catch what small cases cannot: workspace sizing, 32-bit
index overflow, kernel shape limits, memory footprint."""
import pytest
import torch

from tests.device_harness import check_finite, runner

pytestmark = pytest.mark.gpu


def test_cfg3_continuous_async_2048_envs():
    """config 3: Ant-like Box(27) obs -> Box(8) actions, 2048 envs, mujoco flags (sf_examples/mujoco/mujoco_params.py:1-38:
    tanh MLP [64,64], learned stddev, fixed-KL, value bootstrap, 2 epochs), async double-buffered rollout / learn."""
    from sample_factory_b200.envs import TapeVecEnv

    dev = torch.device("cuda", 0)
    N, T = 2048, 64
    tape = torch.randn(2 * T + 1, N, 27, generator=torch.Generator().manual_seed(0)).to(dev)
    r = runner("synthetic_ant", lambda name, cfg, env_config, render_mode=None: TapeVecEnv(tape, 8, continuous=True),
                ["--use_rnn=False", "--async_rl=True", f"--rollout={T}", "--recurrence=1", "--batch_size=32768",
                 "--num_batches_per_epoch=4", "--num_epochs=2", "--encoder_mlp_layers", "64", "64", "--nonlinearity=tanh",
                 "--adaptive_stddev=False", "--kl_loss_coeff=0.1", "--value_loss_coeff=1.3", "--max_grad_norm=3.5",
                 "--exploration_loss_coeff=0.0", "--ppo_clip_ratio=0.2", "--learning_rate=0.00295", "--value_bootstrap=True",
                 "--policy_initialization=torch_default"])
    assert r.async_rl and r.model.spec.continuous and not r.model.spec.adaptive_stddev
    st = check_finite(r, 4, 4 * N * T)
    # async: the samples are one iteration (8 SGD steps) old when trained on (policy lag recorded per sample)
    assert st["version_diff_min"] >= 8 and st["version_diff_max"] <= 16, st
    a = r.traj["actions"]
    assert a.shape == (N, T, 8) and torch.isfinite(a).all() and a.std().item() > 0.3
    assert r.traj["action_logits"].shape == (N, T, 16)
    ls = r.model.learned_log_std
    assert ls is not None and torch.isfinite(ls).all() and not torch.all(ls == 0)     # the learned stddev trains


def test_cfg4_atari_conv_1024_envs():
    """config 4: uint8 [4,84,84] frames, convnet_atari + FC 512, ReLU, obs_scale 255, 1024 envs (atari flags,
    sf_examples/atari/atari_params.py:1-45; rollout shortened to 16 to bound the test's memory and time)."""
    from sample_factory_b200.envs import TapeVecEnv

    dev = torch.device("cuda", 0)
    N, T = 1024, 16
    tape = torch.randint(0, 256, (T + 1, N, 4 * 84 * 84), dtype=torch.uint8, generator=torch.Generator().manual_seed(1)).to(dev)
    r = runner("synthetic_atari", lambda name, cfg, env_config, render_mode=None: TapeVecEnv(tape, 6, obs_shape=(4, 84, 84)),
                ["--use_rnn=False", "--async_rl=False", f"--rollout={T}", "--recurrence=1", "--batch_size=4096",
                 "--num_batches_per_epoch=4", "--num_epochs=1", "--encoder_conv_architecture=convnet_atari",
                 "--encoder_conv_mlp_layers", "512", "--nonlinearity=relu", "--obs_scale=255.0",
                 "--exploration_loss_coeff=0.01", "--max_grad_norm=0.5", "--adam_eps=1e-5"])
    sp = r.model.spec
    assert sp.obs_uint8 and sp.conv_out_size == 64 * 7 * 7 and r.traj["obs"].dtype == torch.uint8
    before = r.model.params["encoder.encoders.obs.enc.conv_head.0.weight"].clone()
    check_finite(r, 2, 2 * N * T)
    assert not torch.equal(before, r.model.params["encoder.encoders.obs.enc.conv_head.0.weight"])
    # per-pixel input statistics after two updates: mean of uniform 0..255 frames / 255 is ~0.5
    assert abs(r.model.obs_mean.mean().item() - 0.5) < 0.02 and r.model.obs_count.item() == 1 + 2 * N * (T + 1)


def test_cfg5_lstm_4096_envs_per_gpu():
    """config 5 (one GPU's shard): Box(256) obs, MLP [512,256,128] -> LSTM-512, 4096 envs, rollout = recurrence = 16,
    batch 32768, value bootstrap, KL-adaptive lr per epoch (train_isaacgym.py:169-208, 310-350)."""
    from sample_factory_b200.envs import TapeVecEnv

    dev = torch.device("cuda", 0)
    N, T = 4096, 16
    tape = torch.randn(2 * T + 1, N, 256, generator=torch.Generator().manual_seed(2)).to(dev)
    r = runner("synthetic_isaac", lambda name, cfg, env_config, render_mode=None: TapeVecEnv(tape, 8),
                ["--use_rnn=True", "--rnn_type=lstm", "--rnn_size=512", "--async_rl=False", f"--rollout={T}",
                 f"--recurrence={T}", "--batch_size=32768", "--num_batches_per_epoch=2", "--num_epochs=2",
                 "--encoder_mlp_layers", "512", "256", "128", "--value_bootstrap=True", "--reward_scale=0.01",
                 "--lr_schedule=kl_adaptive_epoch", "--lr_schedule_kl_threshold=0.016", "--max_grad_norm=1.0"])
    assert r.model.spec.rnn_state_size == 1024 and r.traj["rnn_states"].shape == (N, T + 1, 1024)
    lr0 = r.learner.curr_lr
    st = check_finite(r, 3, 3 * N * T)
    assert st["num_valid"] == 32768
    assert r.learner.curr_lr != lr0         # the KL-adaptive scheduler moved the learning rate
    hs = r.traj["rnn_states"]
    assert torch.isfinite(hs).all() and hs.abs().max().item() > 0
    # done-aware state reset (batched_sampling.py:332-335): the state recorded after a done step is zero
    d = r.traj["dones"]
    nxt = hs[:, 1:T + 1][d]
    assert nxt.numel() > 0 and torch.all(nxt == 0)
