"""Generate the fixtures of Tuple action spaces with Discrete and 1-D Box members by executing the reference (the driver of
make_golden.py, with the member-by-member noise recovery such a Tuple needs):  python tests/golden/make_golden_mixed.py

  tiny_mixed       Tuple(Discrete(3), Box(2), Discrete(4)): 11 distribution_linear rows, entropy bonus, poisoned data
  tiny_mixed_kl    Tuple(Box(3), Discrete(5)): fixed-KL loss, value bootstrap, tanh; adaptive_stddev=False and
                   continuous_tanh_scale=1.5 are set and must be ignored (a Tuple always uses ActionParameterizationDefault)
  tiny_wide_mixed  Tuple(Discrete(24), Box(8), Discrete(5)): 45 rows (not a multiple of 4: unaligned logits stride), V-trace

For every policy step the script re-draws, from the generator state the reference used, the Exp(1) noise of each Discrete
member (proving the multinomial identity argmax(p / q)) and the N(0,1) noise of each Box member (proving a == eps*std + mean
bit for bit), concatenated in member order.  The adapter env receives the reference's per-member action list
(batched_sampling.py:46-57) and takes its reward from member 0 (oracle.appo_oracle.TapeVecEnv's rules).
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import make_golden as MG  # noqa: E402  (installs the reference shims)
from make_golden import (OUT_DIR, BatchedVectorEnvRunner, Learner, ParameterServer, BufferMgr, TensorDict,  # noqa: E402
                         Timing, TapeVecEnv, default_cfg, extract_env_info, gym, make_env_func_batched,
                         prepare_and_normalize_obs, preprocess_cfg, register_env)


class MixedTapeEnv(MG.RefTapeEnv):
    """RefTapeEnv with a Tuple action space of Discrete / Box members; step() gets one array per member"""

    seen = []

    def __init__(self, tape_env, heads):
        super().__init__(tape_env)
        self.action_space = gym.spaces.Tuple([gym.spaces.Discrete(n) if k == "discrete" else
                                              gym.spaces.Box(-1.0, 1.0, (n,), np.float32) for k, n in heads])

    def step(self, actions):
        assert isinstance(actions, list)
        MixedTapeEnv.seen = [("discrete" if a.dtype == np.int32 else "box", a.dtype.type, a.shape) for a in actions]
        obs, rew, term, trunc = self.e.step(torch.as_tensor(actions[0]))
        return self._obs(obs), rew, term, trunc, {}


def run_case(name: str, N: int, T: int, obs_dim: int, heads, hidden, iters: int, overrides: dict, poison: bool):
    A = sum(n if k == "discrete" else 2 * n for k, n in heads)      # distribution_linear rows
    torch.manual_seed(1234)
    np.random.seed(1234)
    tape_len = T * iters + 1
    tape = torch.randn(tape_len, N, obs_dim) * 1.5 + 0.3
    tape_env = TapeVecEnv(tape, A)

    env_name = f"tape_{name}"
    register_env(env_name, lambda full_env_name, cfg, env_config, render_mode=None: MixedTapeEnv(tape_env, heads))

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
                # TupleActionDistribution.sample draws member by member (action_distributions.py:243-252): a Discrete
                # member's multinomial consumes Exp(1) draws, a Box member's Normal.sample N(0,1) draws (SURVEY App.C/E)
                params_all, acts_all = policy_outputs["action_logits"], policy_outputs["actions"]
                ps = torch.split(params_all, [n if k == "discrete" else 2 * n for k, n in heads], dim=1)
                acs = torch.split(acts_all, [1 if k == "discrete" else n for k, n in heads], dim=1)
                qs = []
                for (kind, n), pk, ak in zip(heads, ps, acs):
                    if kind == "discrete":
                        probs = torch.softmax(pk, -1)
                        qk = torch.empty_like(probs).exponential_()
                        assert torch.equal(torch.argmax(probs / qk, -1).to(ak.dtype), ak[:, 0]), "multinomial identity"
                    else:
                        mu, log_std = torch.chunk(pk, 2, dim=1)
                        std = torch.clamp(log_std.exp(), 1e-4, 1e4)
                        qk = torch.empty_like(mu).normal_()
                        assert torch.equal((qk * std + mu).to(ak.dtype), ak), "normal sample identity"
                    qs.append(qk)
                q = torch.cat(qs, dim=1)
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

    assert MixedTapeEnv.seen == [("discrete", np.int32, (N,)) if k == "discrete" else ("box", np.float32, (N, n))
                                 for k, n in heads], MixedTapeEnv.seen      # preprocess_actions' per-member list
    meta = dict(N=N, T=T, obs_dim=obs_dim, A=A, hidden=list(hidden), iters=iters, poison=poison, continuous=False,
                decoder=list(cfg.decoder_mlp_layers), obs_shape=None, action_segments=None, action_mask=False,
                action_heads=[tuple(h) for h in heads], **overrides)
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
    out["cfg/continuous"] = np.bool_(False)
    for k in ["normalize_input", "normalize_returns", "value_bootstrap", "with_vtrace", "use_rnn", "adaptive_stddev",
              "actor_critic_share_weights"]:
        out[f"cfg/{k}"] = np.bool_(getattr(cfg, k))
    out["cfg/rnn_size"] = np.float64(cfg.rnn_size)
    out["cfg/rnn_type"] = np.array(cfg.rnn_type)
    path = os.path.join(OUT_DIR, f"{name}.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {os.path.getsize(path) / 1e6:.2f} MB, losses: {rec_losses[-1]}")


if __name__ == "__main__":
    only = set(sys.argv[1:])
    cases = [
        dict(name="tiny_mixed", N=32, T=8, obs_dim=16, heads=[("discrete", 3), ("box", 2), ("discrete", 4)],
             hidden=[64, 64], iters=2, poison=True,
             overrides=dict(batch_size=128, num_batches_per_epoch=2, num_epochs=2, exploration_loss_coeff=0.01)),
        dict(name="tiny_mixed_kl", N=32, T=8, obs_dim=16, heads=[("box", 3), ("discrete", 5)], hidden=[64, 64], iters=2,
             poison=False,
             overrides=dict(batch_size=128, num_batches_per_epoch=2, num_epochs=1, kl_loss_coeff=0.1, value_bootstrap=True,
                            nonlinearity="tanh", adaptive_stddev=False, continuous_tanh_scale=1.5)),
        dict(name="tiny_wide_mixed", N=32, T=8, obs_dim=16, heads=[("discrete", 24), ("box", 8), ("discrete", 5)],
             hidden=[64, 64], iters=2, poison=False,
             overrides=dict(batch_size=128, num_batches_per_epoch=2, num_epochs=1, with_vtrace=True, recurrence=8,
                            normalize_returns=False)),
    ]
    for c in cases:
        if not only or c["name"] in only:
            run_case(**c)
