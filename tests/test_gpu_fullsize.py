"""Numeric parity at BASELINE.json's sizes (not just `isfinite`): for every config the device sampler + learner are run
closed-loop next to the CPU oracle (oracle/appo_oracle.py -- pinned to the reference by tests/golden/*) on the same tape,
the same initial weights and the same sampling noise, and compared value by value:

  rollout   actions (indices bit-exact -- a flip needs p_i/q_i == p_j/q_j to within the 1e-6 logit difference; at 131 072
            samples a handful of such near-ties can exist, so at most 4 per rollout are tolerated and reported), observations /
            rewards / dones / policy stamps exact, logits / values / log-probs / recurrent states at 1e-5
  learner   trained on the ORACLE's trajectories (identical inputs on both sides): returns, advantages, every loss term at
            1e-5, grad-norm at 5e-4 relative (it sums 3e5..1.7e6 squared gradients of weights that already differ by
            rounding after the previous SGD steps), post-Adam weights and normaliser statistics at 2e-5 (Adam amplifies a 1e-6
            gradient difference where |g| ~ adam_eps, DESIGN.md section 7).

cfg-2 runs at its exact size (4096 envs x 32 steps, 512-512 MLP).  cfg-3 / cfg-4 / cfg-5 run their real layer stacks and
hyper-parameters (sf_examples/mujoco/mujoco_params.py, atari/atari_params.py, isaacgym_examples/train_isaacgym.py:310-350)
at env counts the CPU oracle finishes in seconds."""
import numpy as np
import pytest
import torch

from oracle import appo_oracle as O
from tests.device_harness import DEV, TOL, build, need

pytestmark = pytest.mark.gpu

CASES = {
    # BASELINE.json configs[1]: exact size
    "cfg2_4096x32": dict(N=4096, T=32, iters=2, ocfg=dict(rollout=32, recurrence=1, batch_size=32768, num_batches_per_epoch=4)),
    # configs[2]: Ant-like Box(27) -> Box(8), tanh 64-64, learned stddev, fixed KL, value bootstrap, 2 epochs x 4 minibatches
    "cfg3_ant_2048x64": dict(N=2048, T=64, iters=1, ocfg=dict(
        obs_dim=27, num_actions=8, continuous=True, adaptive_stddev=False, encoder_mlp_layers=[64, 64], nonlinearity="tanh",
        rollout=64, recurrence=1, batch_size=32768, num_batches_per_epoch=4, num_epochs=2, kl_loss_coeff=0.1,
        value_loss_coeff=1.3, max_grad_norm=3.5, exploration_loss_coeff=0.0, ppo_clip_ratio=0.2, learning_rate=0.00295,
        value_bootstrap=True)),
    # configs[3]: uint8 [4,84,84] frames, convnet_atari + FC 512, ReLU, obs_scale 255 (256 envs x 8 steps)
    "cfg4_atari_256x8": dict(N=256, T=8, iters=1, uint8=True, ocfg=dict(
        obs_dim=4 * 84 * 84, obs_shape=(4, 84, 84), num_actions=6, encoder_conv_architecture="convnet_atari",
        encoder_conv_mlp_layers=[512], encoder_mlp_layers=[], nonlinearity="relu", obs_scale=255.0, rollout=8, recurrence=1,
        batch_size=512, num_batches_per_epoch=4, exploration_loss_coeff=0.01, max_grad_norm=0.5, adam_eps=1e-5),
        # four SGD steps with adam_eps = 1e-5 on 1.7 M conv / FC weights: the few whose |g| ~ eps move by up to lr = 1e-4 per
        # step in a direction a 1e-7 gradient difference decides (measured: 104 of 1 605 632 FC weights off by > 6e-5, max 1.5e-4)
        w_atol=6e-5, w_frac=3e-4,
        # (after ONE step the first moments agree to 1.4e-7 / 7.7e-4 relative, the amplified weight
        # differences feed back into the gradients of steps 2-4)
        m_atol=5e-5),
    # configs[4]: Box(256), MLP 512-256-128 -> LSTM-512, rollout = recurrence = 16, value bootstrap (one GPU's shard, 1024 envs)
    "cfg5_lstm_1024x16": dict(N=1024, T=16, iters=1, ocfg=dict(
        obs_dim=256, encoder_mlp_layers=[512, 256, 128], use_rnn=True, rnn_type="lstm", rnn_size=512, rollout=16, recurrence=16,
        batch_size=8192, num_batches_per_epoch=2, value_bootstrap=True, reward_scale=0.01, max_grad_norm=1.0)),
}


@pytest.mark.parametrize("name", list(CASES))
def test_full_size_parity_vs_oracle(name):
    from sample_factory_b200 import ops

    need("3xtf32")
    case = CASES[name]
    N, T = case["N"], case["T"]
    ocfg = O.OracleCfg(**case["ocfg"])
    st0 = O.init_state(ocfg, seed=5)
    gen = torch.Generator().manual_seed(23)
    if case.get("uint8"):
        tape = torch.randint(0, 256, (case["iters"] * T + 1, N, ocfg.obs_dim), dtype=torch.uint8, generator=gen)
    else:
        tape = torch.randn(case["iters"] * T + 1, N, ocfg.obs_dim, generator=gen) * 1.2 - 0.2
    cfg, model, traj, env, sampler, learner = build(ocfg, N, st0, tape, "3xtf32")
    olearner = O.OracleLearner(ocfg, st0)
    oenv = O.TapeVecEnv(tape, ocfg.num_actions)
    olast = oenv.reset()
    sampler.reset()
    A = ocfg.num_actions
    for it in range(case["iters"]):
        if ocfg.continuous:
            noise = torch.randn(T, N, A, generator=gen)
        else:
            noise = torch.empty(T, N, A).exponential_(generator=gen)
        otraj = O.alloc_trajectories(ocfg, N)
        olast = O.rollout(ocfg, olearner.st, oenv, olast, otraj, noise, olearner.train_step)
        sampler.noise = noise.to(DEV)
        sampler.set_policy_version(learner.train_step)
        sampler.rollout()
        got = {k: v.cpu() for k, v in traj.items()}
        # ---- rollout parity
        assert torch.equal(got["obs"].view(otraj["obs"].shape), otraj["obs"])
        for k in ["dones", "time_outs", "policy_id", "policy_version"]:
            assert torch.equal(got[k], otraj[k]), k
        np.testing.assert_allclose(got["action_logits"].numpy(), otraj["action_logits"].numpy(), atol=TOL)
        np.testing.assert_allclose(got["values"][:, :-1].numpy(), otraj["values"][:, :-1].numpy(), atol=TOL)
        np.testing.assert_allclose(got["rnn_states"].numpy(), otraj["rnn_states"].numpy(), atol=TOL)
        if ocfg.continuous:
            np.testing.assert_allclose(got["actions"].numpy(), otraj["actions"].numpy(), atol=TOL)
            np.testing.assert_allclose(got["rewards"].numpy(), otraj["rewards"].numpy(), atol=TOL)
            np.testing.assert_allclose(got["log_prob_actions"].numpy(), otraj["log_prob_actions"].numpy(), atol=2e-5)
        else:
            flips = got["actions"].view(otraj["actions"].shape) != otraj["actions"]
            n_flip = int(flips.sum())
            assert n_flip <= 4, f"{n_flip} of {flips.numel()} action indices differ from the oracle"
            same = ~flips.view(N, T)
            assert torch.equal(got["rewards"][same], otraj["rewards"][same])
            np.testing.assert_allclose(got["log_prob_actions"][same].numpy(), otraj["log_prob_actions"][same].numpy(), atol=TOL)
            if n_flip:
                print(f"[{name}] iteration {it}: {n_flip} near-tie action flips of {flips.numel()}")
        # ---- learner parity on identical inputs (the oracle's trajectories)
        for k, v in otraj.items():
            if k in traj:
                traj[k].copy_(v.view(traj[k].shape))
        n0 = len(olearner.log)
        buff = olearner.train(otraj)
        learner.train(traj)
        np.testing.assert_allclose(learner.returns.view(-1).cpu().numpy(), buff["returns"].numpy(), atol=TOL)
        np.testing.assert_allclose(learner.advantages.view(-1).cpu().numpy(), buff["advantages"].numpy(), atol=TOL)
        log = learner.minibatch_log().numpy()
        assert log.shape[0] == len(olearner.log) - n0
        for j, d in enumerate(olearner.log[n0:]):
            for key in ["policy_loss", "value_loss", "exploration_loss", "kl_loss"]:
                assert abs(log[j, ops.LS[key]] - d[key]) < TOL, (name, it, j, key, log[j, ops.LS[key]], d[key])
            gn = learner.grad_norm_log[j].item()
            assert abs(gn - d["grad_norm"]) <= 5e-4 * max(1.0, abs(d["grad_norm"])), (j, gn, d["grad_norm"])
        sd = model.state_dict()
        n_sgd = len(olearner.log) - n0
        for k in O.param_names(ocfg):
            # Adam's first moment is linear in the gradients of the SGD steps: the well-conditioned check of the backward pass
            off, shp = model._slices[k]
            m_dev = model.exp_avg[off: off + int(np.prod(shp))].view(shp).cpu().numpy()
            np.testing.assert_allclose(m_dev, olearner.m[k].numpy(), atol=case.get("m_atol", 2e-6), err_msg=f"{name} exp_avg {k}")
            # the weights themselves: lr * m / (sqrt(v) + eps) amplifies a 1e-7 gradient difference where |g| ~ adam_eps (dead
            # ReLU units, saturated inputs) up to a full lr-sized step, so: all but a vanishing fraction within w_atol, and
            # nobody further away than the n_sgd * lr such elements can move
            d = np.abs(sd[k].cpu().numpy() - olearner.st[k].numpy())
            frac = float((d > case.get("w_atol", 2e-5)).mean())
            assert frac < case.get("w_frac", 0.0) + 1e-12, (name, k, frac, float(d.max()))
            assert float(d.max()) < n_sgd * ocfg.learning_rate * 1.05 + 2e-5, (name, k, float(d.max()))
        for k in (O.OBS_MEAN, O.OBS_VAR):
            np.testing.assert_allclose(sd[k].cpu().numpy().reshape(-1), olearner.st[k].numpy().reshape(-1), rtol=1e-6, atol=1e-6)
        # keep the two closed loops on identical weights for the next iteration (differences stay at rounding level anyway)
        model.load_state_dict({k: v.clone() for k, v in olearner.st.items()}, strict=False)
