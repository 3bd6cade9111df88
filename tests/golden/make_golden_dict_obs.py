"""Generate the fixtures of Dict observations with several 1-D keys (MultiInputEncoder, model/encoder.py:33-70) by
executing the reference (the driver of make_golden.py):  python tests/golden/make_golden_dict_obs.py [case ...]

  tiny_dict       keys achieved_goal(3), desired_goal(3), observation(13): MLP [64, 64] per key, Discrete(5), entropy bonus,
                  poisoned data.  Key offsets 0 / 3 / 6 are not 16-byte aligned.
  tiny_dict_lstm  keys a(8), b(16): MLP [32] per key, LSTM 32, decoder [32], Box(3), value bootstrap; also carries the
                  checkpoint the reference's Learner.save() wrote after the last iteration (under ckpt/)
  tiny_dict_mask  keys extra(4), obs(12) + action_mask: identity encoders (encoder_mlp_layers=[]), decoder [64],
                  Discrete(40), shuffled minibatches

The adapter env splits each row of the tape into the keys (sorted key order, key k in columns [c_k, c_k + d_k)).  Each
fixture stores the per-key observations the reference's trajectory buffers held (it{i}/traj/obs/{key}), the packed rows
(it{i}/traj/obs) and cfg/obs_keys.
"""
from __future__ import annotations

import os
import shutil
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import make_golden as MG  # noqa: E402  (installs the reference shims)
from make_golden import (OUT_DIR, BatchedVectorEnvRunner, Learner, ParameterServer, BufferMgr, TensorDict,  # noqa: E402
                         Timing, TapeVecEnv, default_cfg, extract_env_info, gym, make_env_func_batched,
                         prepare_and_normalize_obs, preprocess_cfg, register_env)
from make_golden_rnn_layers import _checkpoint_arrays  # noqa: E402


class DictTapeEnv(MG.RefTapeEnv):
    """RefTapeEnv whose observation is a Dict of 1-D keys cut from the tape row (sorted key order, like gymnasium's Dict)"""

    def __init__(self, tape_env, keys, continuous: bool):
        super().__init__(tape_env, continuous)
        self.keys = keys
        spaces = {k: gym.spaces.Box(-np.inf, np.inf, (d,), np.float32) for k, d in keys}
        if tape_env.with_action_mask:
            spaces["action_mask"] = gym.spaces.Box(0, 1, (tape_env.num_actions,), np.int8)
        self.observation_space = gym.spaces.Dict(dict(sorted(spaces.items())))

    def _obs(self, o):
        out, c = {}, 0
        for k, d in self.keys:
            out[k] = o[:, c: c + d].clone()
            c += d
        if self.e.with_action_mask:
            out["action_mask"] = self.e.action_mask().to(torch.int8)
        return out


def run_case(name: str, N: int, T: int, keys, A: int, hidden, iters: int, overrides: dict, poison: bool,
             continuous: bool = False, action_mask: bool = False, save_checkpoint: bool = False):
    if MG._ONLY and name not in MG._ONLY:
        return
    assert [k for k, _ in keys] == sorted(k for k, _ in keys)
    obs_dim = sum(d for _, d in keys)
    shutil.rmtree(os.path.join("/tmp/sfb200_golden", f"golden_{name}"), ignore_errors=True)
    torch.manual_seed(1234)
    np.random.seed(1234)
    tape = torch.randn(T * iters + 1, N, obs_dim) * 1.5 + 0.3
    tape_env = TapeVecEnv(tape, A, with_action_mask=action_mask)

    env_name = f"tape_{name}"
    register_env(env_name, lambda full_env_name, cfg, env_config, render_mode=None: DictTapeEnv(tape_env, keys, continuous))

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
        _dist, policy_loss, exploration_loss, _kl_old, kl_loss, value_loss, summ = out
        rec_losses.append(dict(policy_loss=float(policy_loss), exploration_loss=float(exploration_loss),
                               kl_loss=float(kl_loss), value_loss=float(value_loss), adv_mean=float(summ["adv_mean"]),
                               adv_std=float(summ["adv_std"])))
        return out

    learner._calculate_losses = calc_wrapper

    out = {"tape": tape.numpy()}
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
                if continuous:
                    mu, log_std = torch.chunk(policy_outputs["action_logits"], 2, dim=1)
                    std = torch.clamp(log_std.exp(), 1e-4, 1e4)
                    q = torch.empty_like(mu).normal_()
                    assert torch.equal(q * std + mu, policy_outputs["actions"]), "normal sample identity"
                elif mask is not None:
                    from sample_factory.algo.utils.action_distributions import masked_softmax

                    probs = masked_softmax(policy_outputs["action_logits"], mask)
                    probs = torch.where((probs.sum(-1) == 0).unsqueeze(-1), torch.full_like(probs, 1e-6), probs)
                    q = torch.empty_like(probs).exponential_()
                    assert torch.equal(torch.argmax(probs / q, -1), policy_outputs["actions"]), "multinomial identity"
                else:
                    probs = torch.softmax(policy_outputs["action_logits"], -1)
                    q = torch.empty_like(probs).exponential_()
                    assert torch.equal(torch.argmax(probs / q, -1), policy_outputs["actions"]), "multinomial identity"
                torch.set_rng_state(rng_after)
                noise_steps.append(q.clone())
                policy_outputs["policy_version"] = torch.empty([N]).fill_(int(policy_versions[0].item()))
                if policy_outputs["actions"].ndim < 2:
                    policy_outputs["actions"] = policy_outputs["actions"].unsqueeze(-1)
                for key in runner.policy_output_tensors.keys():
                    runner.policy_output_tensors[key][:] = policy_outputs[key].reshape(
                        runner.policy_output_tensors[key].shape)
            complete, _stats = runner.advance_rollouts(0, timing)
        assert len(complete) == 1
        sl = complete[0]["traj_buffer_idx"]
        batch = runner.traj_tensors[sl]

        if poison and it == iters - 1:
            g = torch.Generator().manual_seed(77)
            pmask = torch.rand(N, T, generator=g) < 0.15
            batch["policy_id"][pmask] = -1
            stale = torch.rand(N, T, generator=g) < 0.05
            batch["policy_version"][stale] = -5000.0

        for k in ["actions", "action_logits", "log_prob_actions", "values", "policy_version", "rewards", "dones",
                  "time_outs", "policy_id", "rnn_states"]:
            out[f"it{it}/traj/{k}"] = batch[k].clone().numpy()
        # one buffer per key in the reference (shared_buffers.py:85-91); the device layout is the packed row
        per_key = [batch["obs"][k].clone().numpy() for k, _ in keys]
        for (k, _), v in zip(keys, per_key):
            out[f"it{it}/traj/obs/{k}"] = v
        out[f"it{it}/traj/obs"] = np.concatenate(per_key, axis=2)
        out[f"it{it}/noise"] = torch.stack(noise_steps).numpy()
        out[f"it{it}/train_step_before"] = np.int64(learner.train_step)

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
        if drawn:
            out[f"it{it}/mb_indices"] = np.stack(drawn)
        for k, v in captured.items():
            out[f"it{it}/prep/{k}"] = v
        ls = rec_losses[n_before:]
        for key in ls[0].keys():
            out[f"it{it}/loss/{key}"] = np.array([d[key] for d in ls], dtype=np.float64)
        for k, v in ac.state_dict().items():
            out[f"it{it}/state/{k}"] = v.detach().clone().numpy()
        out[f"it{it}/train_step_after"] = np.int64(learner.train_step)
        runner.traj_buffer_queue.put(sl)

    if save_checkpoint:
        assert learner.save()
        files = Learner.get_checkpoints(Learner.checkpoint_dir(cfg, 0))
        out.update(_checkpoint_arrays(files[-1]))

    meta = dict(N=N, T=T, obs_dim=obs_dim, A=A, hidden=list(hidden), iters=iters, poison=poison, continuous=continuous,
                decoder=list(cfg.decoder_mlp_layers), obs_shape=None, action_segments=None, action_mask=action_mask,
                obs_keys=[tuple(k) for k in keys], **overrides)
    out["meta"] = np.array(repr(meta))
    out["cfg/obs_keys"] = np.array(repr([tuple(k) for k in keys]))
    for k in ["gamma", "gae_lambda", "ppo_clip_ratio", "ppo_clip_value", "exploration_loss_coeff", "value_loss_coeff",
              "kl_loss_coeff", "max_grad_norm", "learning_rate", "adam_eps", "adam_beta1", "adam_beta2",
              "reward_scale", "reward_clip", "max_policy_lag", "batch_size", "num_batches_per_epoch", "num_epochs",
              "recurrence", "vtrace_rho", "vtrace_c", "continuous_tanh_scale", "initial_stddev", "obs_scale",
              "obs_subtract_mean"]:
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


if __name__ == "__main__":
    run_case("tiny_dict", N=32, T=8, keys=[("achieved_goal", 3), ("desired_goal", 3), ("observation", 13)], A=5,
             hidden=[64, 64], iters=2, poison=True,
             overrides=dict(batch_size=128, num_batches_per_epoch=2, num_epochs=2, exploration_loss_coeff=0.01))
    run_case("tiny_dict_lstm", N=32, T=8, keys=[("a", 8), ("b", 16)], A=3, hidden=[32], iters=2, poison=False,
             continuous=True, save_checkpoint=True,
             overrides=dict(batch_size=128, num_batches_per_epoch=2, num_epochs=1, use_rnn=True, rnn_type="lstm",
                            rnn_size=32, decoder_mlp_layers=[32], recurrence=8, value_bootstrap=True))
    run_case("tiny_dict_mask", N=64, T=8, keys=[("extra", 4), ("obs", 12)], A=40, hidden=[], iters=2, poison=True,
             action_mask=True,
             overrides=dict(batch_size=128, num_batches_per_epoch=4, num_epochs=1, decoder_mlp_layers=[64],
                            shuffle_minibatches=True))
