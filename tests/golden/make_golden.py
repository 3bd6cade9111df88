"""Generate golden vectors by EXECUTING THE REFERENCE (from a reference checkout (oracle/install_ref.py: reference_dir()), under oracle/ref_shims.py).

Run in the build container only:   python tests/golden/make_golden.py
Writes tests/golden/<case>.npz.  The reference is a Python package and cannot travel to the GPU box, so the
vectors it produced are committed as fixtures, together with this script.

What is driven (unmodified reference code):
  * BatchedVectorEnvRunner.{init,update_trajectory_buffers,generate_policy_request,advance_rollouts}
    (algo/sampling/batched_sampling.py:154-388)
  * the body of InferenceWorker._handle_policy_steps (algo/sampling/inference_worker.py:313-341), inlined because
    the worker class itself needs a live signal_slot event loop
  * BufferMgr / alloc_trajectory_tensors (algo/utils/shared_buffers.py)
  * Learner.init / Learner.train (algo/learning/learner.py:178-255, 1036-1067), with _calculate_losses wrapped
    only to RECORD its return values.
The env is oracle.appo_oracle.TapeVecEnv (ours; registered through the reference's own register_env).
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_shims  # noqa: E402

ref_shims.install()

import gymnasium as gym  # noqa: E402  (shim)

from oracle.appo_oracle import TapeVecEnv  # noqa: E402
from sample_factory.algo.learning.learner import Learner  # noqa: E402
from sample_factory.algo.sampling.batched_sampling import BatchedVectorEnvRunner  # noqa: E402
from sample_factory.algo.utils.env_info import extract_env_info  # noqa: E402
from sample_factory.algo.utils.make_env import make_env_func_batched  # noqa: E402
from sample_factory.algo.utils.model_sharing import ParameterServer  # noqa: E402
from sample_factory.algo.utils.rl_utils import prepare_and_normalize_obs  # noqa: E402
from sample_factory.algo.utils.shared_buffers import BufferMgr  # noqa: E402
from sample_factory.algo.utils.tensor_dict import TensorDict  # noqa: E402
from sample_factory.cfg.arguments import default_cfg, preprocess_cfg  # noqa: E402
from sample_factory.envs.env_utils import register_env  # noqa: E402
from sample_factory.utils.timing import Timing  # noqa: E402

OUT_DIR = os.path.dirname(os.path.abspath(__file__))


class RefTapeEnv(gym.Env):
    """Adapter: TapeVecEnv behind the reference's batched-env contract (make_env.py:147-237)."""

    def __init__(self, tape_env: TapeVecEnv, continuous: bool = False, obs_shape=None, action_segments=None):
        self.e = tape_env
        self.obs_shape = obs_shape
        self.action_segments = action_segments
        self.num_agents = tape_env.num_agents
        self.is_multiagent = True
        self.observation_space = gym.spaces.Dict(
            {"obs": gym.spaces.Box(-np.inf, np.inf, (tape_env.obs_dim,), np.float32)}
        )
        self.action_space = gym.spaces.Discrete(tape_env.num_actions)
        if obs_shape is not None:   # uint8 image observations (C, H, W) -> ConvEncoder (model/encoder.py:88-145)
            self.observation_space = gym.spaces.Dict({"obs": gym.spaces.Box(0, 255, tuple(obs_shape), np.uint8)})
        if action_segments:   # Tuple of Discretes -> TupleActionDistribution (action_distributions.py:197-286)
            self.action_space = gym.spaces.Tuple([gym.spaces.Discrete(n) for n in action_segments])
        if continuous:   # Box(A) action space -> ContinuousActionDistribution (action_distributions.py:290-323)
            self.action_space = gym.spaces.Box(-1.0, 1.0, (tape_env.num_actions,), np.float32)
        if tape_env.with_action_mask:   # obs dict entry the inference worker pops (inference_worker.py:324-331)
            self.observation_space = gym.spaces.Dict({
                "obs": self.observation_space["obs"],
                "action_mask": gym.spaces.Box(0, 1, (tape_env.num_actions,), np.int8)})

    def _obs(self, o):
        o = o.clone() if self.obs_shape is None else o.view(self.num_agents, *self.obs_shape).clone()
        if self.e.with_action_mask:
            return {"obs": o, "action_mask": self.e.action_mask().to(torch.int8)}
        return {"obs": o}

    def reset(self, **kw):
        return self._obs(self.e.reset()), {}

    def step(self, actions):
        if self.action_segments and isinstance(actions, (list, tuple)):
            # (a Tuple space with non-discrete members gets a LIST of per-head arrays, batched_sampling.py:44-56; an
            # all-discrete Tuple -- the case here -- gets one int32 [N, K] array, :40-41)
            actions = np.stack([np.asarray(a) for a in actions], axis=1)
        obs, rew, term, trunc = self.e.step(torch.as_tensor(actions))  # numpy int32 / float32 (batched_sampling.py:62-82)
        return self._obs(obs), rew, term, trunc, {}

    def close(self):
        pass


def run_case(name: str, N: int, T: int, obs_dim: int, A: int, hidden, iters: int, overrides: dict, poison: bool,
             save_checkpoint: bool = False, continuous: bool = False, obs_shape=None, action_segments=None,
             action_mask: bool = False):
    torch.manual_seed(1234)
    np.random.seed(1234)
    tape_len = T * iters + 1
    if obs_shape is not None:
        assert obs_dim == int(np.prod(obs_shape))
        tape = torch.randint(0, 256, (tape_len, N, obs_dim), dtype=torch.uint8)
    else:
        tape = torch.randn(tape_len, N, obs_dim) * 1.5 + 0.3
    tape_env = TapeVecEnv(tape, A, with_action_mask=action_mask)

    env_name = f"tape_{name}"
    register_env(env_name, lambda full_env_name, cfg, env_config, render_mode=None: RefTapeEnv(tape_env, continuous, obs_shape, action_segments))

    cfg = default_cfg(env=env_name, experiment=f"golden_{name}")
    cfg.device = "cpu"
    cfg.serial_mode = True
    cfg.async_rl = False
    cfg.batched_sampling = True
    cfg.num_workers = 1
    cfg.num_envs_per_worker = 1
    cfg.worker_num_splits = 1
    cfg.use_rnn = False
    cfg.encoder_mlp_layers = list(hidden)
    cfg.rollout = T
    cfg.seed = 0
    cfg.train_dir = "/tmp/sfb200_golden"
    cfg.env_gpu_actions = False
    cfg.env_gpu_observations = False
    cfg.use_env_info_cache = False
    for k, v in overrides.items():
        assert hasattr(cfg, k), k
        setattr(cfg, k, v)

    tmp_env = make_env_func_batched(cfg, env_config=None)
    env_info = extract_env_info(tmp_env, cfg)
    assert preprocess_cfg(cfg, env_info)

    buffer_mgr = BufferMgr(cfg, env_info)
    policy_versions = buffer_mgr.policy_versions
    param_server = ParameterServer(0, policy_versions, cfg.serial_mode)
    learner = Learner(cfg, env_info, policy_versions, 0, param_server)
    learner.init()
    ac = learner.actor_critic
    init_state = {k: v.detach().clone().numpy() for k, v in ac.state_dict().items()}

    timing = Timing()
    runner = BatchedVectorEnvRunner(cfg, env_info, 1, 0, 0, buffer_mgr, "cpu", [None])
    runner.init(timing)

    rec_losses = []
    orig_calc = learner._calculate_losses

    def calc_wrapper(mb, num_invalids):
        out = orig_calc(mb, num_invalids)
        action_distribution, policy_loss, exploration_loss, kl_old, kl_loss, value_loss, summ = out
        rec_losses.append(
            dict(
                policy_loss=float(policy_loss),
                exploration_loss=float(exploration_loss),
                kl_loss=float(kl_loss),
                value_loss=float(value_loss),
                adv_mean=float(summ["adv_mean"]),
                adv_std=float(summ["adv_std"]),
            )
        )
        return out

    learner._calculate_losses = calc_wrapper

    out = {}
    out["tape"] = tape.numpy()
    for k, v in init_state.items():
        out[f"init/{k}"] = v

    for it in range(iters):
        noise_steps = []
        for t in range(T):
            assert runner.update_trajectory_buffers(timing)
            req = runner.generate_policy_request()
            assert req is not None
            (traj_slice, step) = req[0]
            # ---- InferenceWorker._handle_policy_steps body (inference_worker.py:313-341) ----
            with torch.no_grad():
                obs = TensorDict({k: v[traj_slice, step] for k, v in runner.traj_tensors["obs"].items()})
                rnn_states = runner.traj_tensors["rnn_states"][traj_slice, step]
                if ac.training:
                    ac.eval()
                mask = obs.pop("action_mask") if "action_mask" in obs else None          # inference_worker.py:324-326
                normalized_obs = prepare_and_normalize_obs(ac, obs)
                rng_before = torch.get_rng_state()
                policy_outputs = ac(normalized_obs, rnn_states, action_mask=mask)
                rng_after = torch.get_rng_state()
                torch.set_rng_state(rng_before)
                if action_segments:
                    # every head draws its own multinomial, in order (action_distributions.py:243-252)
                    qs = []
                    for k, lk in enumerate(torch.split(policy_outputs["action_logits"], list(action_segments), dim=1)):
                        pk = torch.softmax(lk, -1)
                        qk = torch.empty_like(pk).exponential_()
                        assert torch.equal(torch.argmax(pk / qk, -1), policy_outputs["actions"][:, k]), "multinomial identity"
                        qs.append(qk)
                    q = torch.cat(qs, dim=1)
                elif continuous:
                    # recover the N(0,1) draws Normal.sample() consumed (SURVEY App.C) and prove  a == eps*std + mean
                    params = policy_outputs["action_logits"]
                    mu, log_std = torch.chunk(params, 2, dim=1)
                    std = torch.clamp(log_std.exp(), 1e-4, 1e4)
                    q = torch.empty_like(mu).normal_()
                    assert torch.equal(q * std + mu, policy_outputs["actions"]), "normal sample identity"
                elif mask is not None:
                    # masked categorical (action_distributions.py:84-95,135-143): same identity on the masked probabilities
                    from sample_factory.algo.utils.action_distributions import masked_softmax

                    probs = masked_softmax(policy_outputs["action_logits"], mask)
                    probs = torch.where((probs.sum(-1) == 0).unsqueeze(-1), torch.full_like(probs, 1e-6), probs)
                    q = torch.empty_like(probs).exponential_()
                    assert torch.equal(torch.argmax(probs / q, -1), policy_outputs["actions"]), "multinomial identity"
                    assert bool((mask.gather(1, policy_outputs["actions"].view(-1, 1)).view(-1) | (mask.sum(-1) == 0)).all())
                else:
                    # recover the Exp(1) noise torch.multinomial consumed (SURVEY App.E) and prove the identity
                    probs = torch.softmax(policy_outputs["action_logits"], -1)
                    q = torch.empty_like(probs).exponential_()
                    assert torch.equal(torch.argmax(probs / q, -1), policy_outputs["actions"]), "multinomial identity"
                torch.set_rng_state(rng_after)
                noise_steps.append(q.clone())
                policy_outputs["policy_version"] = torch.empty([N]).fill_(int(policy_versions[0].item()))
                # _prepare_policy_outputs_batched :235-269
                if policy_outputs["actions"].ndim < 2:
                    policy_outputs["actions"] = policy_outputs["actions"].unsqueeze(-1)
                for key in runner.policy_output_tensors.keys():
                    runner.policy_output_tensors[key][:] = policy_outputs[key].reshape(
                        runner.policy_output_tensors[key].shape
                    )
            complete, _stats = runner.advance_rollouts(0, timing)
        assert len(complete) == 1
        sl = complete[0]["traj_buffer_idx"]
        batch = runner.traj_tensors[sl]

        if poison and it == iters - 1:
            # invalid-data splice in the spirit of tests/algo/test_learner.py:109-168: foreign policy id + stale version
            g = torch.Generator().manual_seed(77)
            mask = torch.rand(N, T, generator=g) < 0.15
            batch["policy_id"][mask] = -1
            stale = torch.rand(N, T, generator=g) < 0.05
            batch["policy_version"][stale] = -5000.0

        pre = {}
        for k in ["actions", "action_logits", "log_prob_actions", "values", "policy_version", "rewards", "dones",
                  "time_outs", "policy_id", "rnn_states"]:
            pre[k] = batch[k].clone().numpy()
        pre["obs"] = batch["obs"]["obs"].clone().numpy().reshape(N, T + 1, -1)
        for k, v in pre.items():
            out[f"it{it}/traj/{k}"] = v
        out[f"it{it}/noise"] = torch.stack(noise_steps).numpy()
        out[f"it{it}/train_step_before"] = np.int64(learner.train_step)

        # capture _prepare_batch outputs by wrapping
        captured = {}
        orig_prepare = learner._prepare_batch

        def prep_wrapper(b):
            buff, n, ninv = orig_prepare(b)
            for k in ["advantages", "returns", "valids", "values", "rewards", "log_prob_actions", "actions"]:
                if k in buff:
                    captured[k] = buff[k].clone().numpy()
            captured["num_invalids"] = np.int64(ninv)
            captured["bootstrap_values"] = b["values"][:, -1].clone().numpy()
            return buff, n, ninv

        learner._prepare_batch = prep_wrapper
        # shuffle_minibatches: record the permutations the reference drew (learner.py:507-519; a new one every epoch, :713)
        drawn = []
        orig_get_mbs = learner._get_minibatches

        def get_mbs_wrapper(batch_size, experience_size):
            mbs = orig_get_mbs(batch_size, experience_size)
            if cfg.shuffle_minibatches and mbs[0] is not None:
                drawn.append(np.concatenate(mbs).astype(np.int64))
            return mbs

        learner._get_minibatches = get_mbs_wrapper
        n_before = len(rec_losses)
        learner.train(batch)
        learner._prepare_batch = orig_prepare
        learner._get_minibatches = orig_get_mbs
        if drawn:      # one permutation per epoch that ran (learner.py:707-713)
            out[f"it{it}/mb_indices"] = np.stack(drawn)
        for k, v in captured.items():
            out[f"it{it}/prep/{k}"] = v
        ls = rec_losses[n_before:]
        for key in ls[0].keys():
            out[f"it{it}/loss/{key}"] = np.array([d[key] for d in ls], dtype=np.float64)
        for k, v in ac.state_dict().items():
            out[f"it{it}/state/{k}"] = v.detach().clone().numpy()
        out[f"it{it}/train_step_after"] = np.int64(learner.train_step)
        # hand the buffers back (sync mode: Batcher releases after training, batcher.py:220-267)
        runner.traj_buffer_queue.put(sl)

    if save_checkpoint:
        # the reference's own checkpoint file after the last iteration (Learner.save, learner.py:323-360): the fixture for
        # the checkpoint-compatibility tests (SURVEY 8f row 2)
        import shutil

        assert learner.save()
        files = Learner.get_checkpoints(Learner.checkpoint_dir(cfg, 0))
        shutil.copy(files[-1], os.path.join(OUT_DIR, f"{name}_checkpoint.pth"))
        print("checkpoint fixture:", os.path.basename(files[-1]))

    meta = dict(N=N, T=T, obs_dim=obs_dim, A=A, hidden=list(hidden), iters=iters, poison=poison, continuous=continuous,
                decoder=list(cfg.decoder_mlp_layers),
                obs_shape=None if obs_shape is None else tuple(obs_shape),
                action_segments=None if action_segments is None else list(action_segments), action_mask=action_mask,
                **overrides)
    out["meta"] = np.array(repr(meta))
    # a few flags the oracle needs, straight from the reference cfg object
    for k in ["gamma", "gae_lambda", "ppo_clip_ratio", "ppo_clip_value", "exploration_loss_coeff", "value_loss_coeff",
              "kl_loss_coeff", "max_grad_norm", "learning_rate", "adam_eps", "adam_beta1", "adam_beta2",
              "reward_scale", "reward_clip", "max_policy_lag", "batch_size", "num_batches_per_epoch", "num_epochs",
              "recurrence", "vtrace_rho", "vtrace_c"]:
        out[f"cfg/{k}"] = np.float64(getattr(cfg, k))
    for k in ["continuous_tanh_scale", "initial_stddev", "obs_scale", "obs_subtract_mean"]:
        out[f"cfg/{k}"] = np.float64(getattr(cfg, k))
    out["cfg/nonlinearity"] = np.array(cfg.nonlinearity)
    out["cfg/exploration_loss"] = np.array(cfg.exploration_loss)
    out["cfg/optimizer"] = np.array(cfg.optimizer)
    out["cfg/encoder_conv_architecture"] = np.array(cfg.encoder_conv_architecture)
    out["cfg/encoder_conv_mlp_layers"] = np.array(list(cfg.encoder_conv_mlp_layers), dtype=np.int64)
    out["cfg/continuous"] = np.bool_(continuous)
    for k in ["normalize_input", "normalize_returns", "value_bootstrap", "with_vtrace", "use_rnn", "adaptive_stddev",
              "actor_critic_share_weights"]:
        out[f"cfg/{k}"] = np.bool_(getattr(cfg, k))
    out["cfg/rnn_size"] = np.float64(cfg.rnn_size)
    out["cfg/rnn_type"] = np.array(cfg.rnn_type)
    path = os.path.join(OUT_DIR, f"{name}.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {os.path.getsize(path) / 1e6:.2f} MB, losses: {rec_losses[-1]}")


def kat_action_distribution():
    """The reference's own known-answer vector (tests/algo/test_action_distributions.py:142-173), re-evaluated with
    the reference's CategoricalActionDistribution so the fixture carries reference outputs, not just literals."""
    from sample_factory.algo.utils.action_distributions import CategoricalActionDistribution

    logits = torch.tensor([[0.0, 1.0, 2.0]])
    d = CategoricalActionDistribution(logits)
    np.savez(
        os.path.join(OUT_DIR, "kat_categorical.npz"),
        logits=logits.numpy(),
        probs=d.probs.numpy(),
        log_probs=d.log_probs.numpy(),
        entropy=d.entropy().numpy(),
        log_prob_a2=d.log_prob(torch.tensor([[2]])).numpy(),
        literal_probs=np.array([0.09003057, 0.24472847, 0.66524096], dtype=np.float32),
    )


def kat_masked_categorical():
    """Masked categorical in the style of the reference's tests/algo/test_action_distributions.py:22-43 (Discrete sizes,
    batch sizes, integer masks incl. rows that allow nothing), evaluated with the reference's own class."""
    from sample_factory.algo.utils.action_distributions import CategoricalActionDistribution

    gen = torch.Generator().manual_seed(99)
    out = {}
    for i, (n, b) in enumerate([(3, 1), (5, 128), (16, 512), (31, 64)]):
        logits = torch.randn(b, n, generator=gen) * 3
        mask = (torch.rand(b, n, generator=gen) < 0.5).to(torch.int64)
        if b > 4:
            mask[::9] = 0
            mask[1::9] = 1
        d = CategoricalActionDistribution(logits, mask)
        out[f"c{i}/logits"], out[f"c{i}/mask"] = logits.numpy(), mask.numpy()
        out[f"c{i}/probs"], out[f"c{i}/log_probs"] = d.probs.numpy(), d.log_probs.numpy()
        out[f"c{i}/entropy"] = d.entropy().numpy()
        a = torch.argmax(d.probs, -1, keepdim=True)
        out[f"c{i}/argmax"], out[f"c{i}/log_prob_argmax"] = a.numpy(), d.log_prob(a).numpy()
    np.savez_compressed(os.path.join(OUT_DIR, "kat_masked_categorical.npz"), **out)


_ONLY = set(sys.argv[1:])   # optional: regenerate only the named cases


def _selected(fn):
    def wrapper(name, *a, **k):
        if _ONLY and name not in _ONLY:
            return
        return fn(name, *a, **k)
    return wrapper


run_case = _selected(run_case)

if __name__ == "__main__":
    if not _ONLY:
        kat_action_distribution()
    if not _ONLY or "kat_masked_categorical" in _ONLY:
        kat_masked_categorical()
    # tiny dims, 2 iterations, invalids + value bootstrap + fixed-KL, 2 epochs x 2 minibatches
    run_case(
        "tiny_gae", N=32, T=8, obs_dim=16, A=8, hidden=[64, 64], iters=2,
        overrides=dict(batch_size=128, num_batches_per_epoch=2, num_epochs=2, value_bootstrap=True,
                       kl_loss_coeff=0.1, reward_scale=0.7, reward_clip=0.5),
        poison=True, save_checkpoint=True,
    )
    # V-trace variant (requires recurrence == rollout, no returns normalisation: arguments.py:129-134,193-194)
    run_case(
        "tiny_vtrace", N=32, T=8, obs_dim=16, A=8, hidden=[64, 64], iters=2,
        overrides=dict(batch_size=128, num_batches_per_epoch=2, num_epochs=1, with_vtrace=True, recurrence=8,
                       normalize_returns=False),
        poison=False,
    )
    # recurrent cores (model/core.py): GRU (the reference default) and LSTM, BPTT over the whole rollout with
    # done-or-invalid resets (rnn_utils.py); poisoned data exercises the "invalid" boundaries
    run_case(
        "tiny_gru", N=32, T=8, obs_dim=16, A=8, hidden=[64], iters=2,
        overrides=dict(batch_size=128, num_batches_per_epoch=2, num_epochs=2, use_rnn=True, rnn_type="gru", rnn_size=32,
                       recurrence=8, value_bootstrap=True),
        poison=True,
    )
    run_case(
        "tiny_lstm", N=32, T=8, obs_dim=16, A=8, hidden=[64], iters=2,
        overrides=dict(batch_size=128, num_batches_per_epoch=2, num_epochs=1, use_rnn=True, rnn_type="lstm", rnn_size=32,
                       recurrence=4),
        poison=False,
    )
    # BASELINE cfg-5's real layer stack (sf_examples/isaacgym_examples/train_isaacgym.py:310-324 AllegroHandLSTM: MLP
    # 512-256-128 -> LSTM-512, rollout = recurrence = 16, reward_scale 0.01, max_grad_norm 1.0, value bootstrap), few envs
    run_case(
        "cfg5_stack", N=16, T=16, obs_dim=64, A=8, hidden=[512, 256, 128], iters=1,
        overrides=dict(batch_size=128, num_batches_per_epoch=2, num_epochs=2, use_rnn=True, rnn_type="lstm", rnn_size=512,
                       recurrence=16, value_bootstrap=True, reward_scale=0.01, max_grad_norm=1.0),
        poison=True,
    )
    # shuffle_minibatches (learner.py:498-526): the permutation of recurrence-length chunks the reference drew is recorded, so the
    # oracle (and through it the device learner) can be fed the same minibatches; MLP (chunks of 1) and GRU (chunks of 4)
    run_case(
        "tiny_shuffle", N=32, T=8, obs_dim=16, A=8, hidden=[64, 64], iters=2,
        overrides=dict(batch_size=64, num_batches_per_epoch=4, num_epochs=2, shuffle_minibatches=True),
        poison=True,
    )
    run_case(
        "tiny_shuffle_gru", N=32, T=8, obs_dim=16, A=8, hidden=[64], iters=2,
        overrides=dict(batch_size=64, num_batches_per_epoch=4, num_epochs=1, use_rnn=True, rnn_type="gru", rnn_size=32,
                       recurrence=4, shuffle_minibatches=True),
        poison=True,
    )
    # continuous actions (BASELINE cfg-3, mujoco-style flags sf_examples/mujoco/mujoco_params.py:1-38): Box(6) actions,
    # tanh MLP [64,64], one learned log-stddev vector (adaptive_stddev=False) with tanh-squashed means, fixed-KL loss,
    # value bootstrap, no entropy bonus; and the default adaptive-stddev parameterization (2A linear outputs)
    run_case(
        "tiny_gauss", N=32, T=8, obs_dim=16, A=6, hidden=[64, 64], iters=2,
        overrides=dict(batch_size=128, num_batches_per_epoch=2, num_epochs=2, nonlinearity="tanh", adaptive_stddev=False,
                       continuous_tanh_scale=1.5, initial_stddev=0.7, kl_loss_coeff=0.1, value_bootstrap=True,
                       exploration_loss_coeff=0.0, ppo_clip_ratio=0.2, value_loss_coeff=1.3, max_grad_norm=3.5,
                       learning_rate=0.00295),
        poison=True, continuous=True,
    )
    run_case(
        "tiny_gauss_adaptive", N=32, T=8, obs_dim=16, A=6, hidden=[64, 64], iters=2,
        overrides=dict(batch_size=128, num_batches_per_epoch=2, num_epochs=1, kl_loss_coeff=0.05),
        poison=False, continuous=True,
    )
    # image observations (BASELINE cfg-4, atari-style flags sf_examples/atari/atari_params.py:1-45): uint8 [4, 44, 44]
    # frames, convnet_atari (32@8s4, 64@4s2, 64@3s1) + FC 128, ReLU, obs_scale=255, per-pixel input normalisation,
    # 2 epochs x 2 minibatches, small grad-norm clip
    run_case(
        "tiny_conv", N=8, T=8, obs_dim=4 * 44 * 44, A=6, hidden=[], iters=2,
        overrides=dict(batch_size=32, num_batches_per_epoch=2, num_epochs=2, nonlinearity="relu", obs_scale=255.0,
                       encoder_conv_architecture="convnet_atari", encoder_conv_mlp_layers=[128],
                       exploration_loss_coeff=0.01, max_grad_norm=0.5, adam_eps=1e-5, ppo_clip_ratio=0.1),
        poison=True, obs_shape=(4, 44, 44),
    )
    # symmetric-KL-to-uniform exploration loss (learner.py:479-486) instead of the entropy bonus
    run_case(
        "tiny_symkl", N=32, T=8, obs_dim=16, A=5, hidden=[64, 64], iters=2,
        overrides=dict(batch_size=128, num_batches_per_epoch=2, num_epochs=1, exploration_loss="symmetric_kl",
                       exploration_loss_coeff=0.01),
        poison=True,
    )
    # Tuple(Discrete(3), Discrete(2), Discrete(4)) action space: three independent categorical heads over 9 logits
    run_case(
        "tiny_tuple", N=32, T=8, obs_dim=16, A=9, hidden=[64, 64], iters=2,
        overrides=dict(batch_size=128, num_batches_per_epoch=2, num_epochs=1, kl_loss_coeff=0.05),
        poison=True, action_segments=[3, 2, 4],
    )
    # separate actor / critic towers (ActorCriticSeparateWeights, model/actor_critic.py:198-322), with decoder MLPs
    run_case(
        "tiny_separate", N=32, T=8, obs_dim=16, A=8, hidden=[64, 48], iters=2,
        overrides=dict(batch_size=128, num_batches_per_epoch=2, num_epochs=2, actor_critic_share_weights=False,
                       decoder_mlp_layers=[32], value_bootstrap=True),
        poison=True,
    )
    # LAMB optimizer (algo/utils/optimizers.py) instead of Adam: per-tensor trust ratios, weight decay 1e-4
    run_case(
        "tiny_lamb", N=32, T=8, obs_dim=16, A=8, hidden=[64, 64], iters=2,
        overrides=dict(batch_size=128, num_batches_per_epoch=2, num_epochs=2, optimizer="lamb", learning_rate=3e-3),
        poison=True,
    )
    # action masks (obs dict key "action_mask", inference_worker.py:324-331 -> masked_softmax / masked_log_softmax,
    # action_distributions.py:84-95): masked sampling in the rollout; the learner ignores the mask, like the reference
    run_case(
        "tiny_mask", N=64, T=8, obs_dim=16, A=7, hidden=[64, 64], iters=2,
        overrides=dict(batch_size=256, num_batches_per_epoch=2, num_epochs=2),
        poison=True, action_mask=True,
    )
    # cfg-2 hyper-parameters and model (300 553 params) at a reduced env count
    run_case(
        "cfg2_small", N=64, T=32, obs_dim=64, A=8, hidden=[512, 512], iters=1,
        overrides=dict(batch_size=512, num_batches_per_epoch=4, num_epochs=1),
        poison=False,
    )
