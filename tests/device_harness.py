"""Scaffolding the GPU tests share: the device and engine helpers, one builder of model + tape env + sampler + learner
from an oracle config, the replays of the reference-executed fixtures (tests/golden/*.npz) through the sampler and the
learner, the graph-vs-eager comparisons, and the helpers more than one GPU test file uses.

A fixture test loads its case with its feature's loader -- (z, meta, ocfg) from load_case, load_mixed_case,
RO.load_stacked_case, SO.load_separate_rnn_case or DO.load_dict_case -- and then:

    rig = build_case(case, engine)
    replay_sampler(case, rig)         # or replay_learner(case, rig)

The keyword options of the replays name where a feature's check differs from the default one."""
import math
import os
import re
import subprocess
import time
import warnings
from collections import namedtuple

import numpy as np
import pytest
import torch

from oracle import appo_oracle as O
from tests.golden_utils import state_from, traj_from

DEV = torch.device("cuda", 0)
TOL = 1e-5
ENGINES = ["simt", "3xtf32"]


def need(engine):
    """skip unless `engine` ("simt" / "3xtf32") can run here"""
    from sample_factory_b200 import ops

    if engine != "simt" and not ops.tc_available():
        pytest.skip("wgmma engine not available")


def ops_for(engine="simt"):
    """bind cuda:0 and return the ops module; skips when `engine` needs the wgmma engine and it is unavailable"""
    from sample_factory_b200 import ops

    ops.bind_device(DEV)
    need(engine)
    return ops


def g(seed):
    return torch.Generator().manual_seed(seed)


TEMPLATED = r"\w+_kernel<[^<>]*>"           # the templated sfb kernels
ANY_KERNEL = r"\w+_kernel(?:<[^<>]*>)?"      # every sfb kernel, templated or not


def launched(fn, names=TEMPLATED, expected=None):
    """the sfb kernels fn launches whose name (without the namespace) matches `names`.  The profiler keeps only device
    records whose time stamps fall inside its capture window, so the window is padded on both sides.  Even so a record
    can go missing (seen after a module had run many profiles with heavy device work between them).  fn is idempotent
    and launches at least one kernel, so the profile is taken again when it holds no sfb kernel at all or, given the
    `expected` set, only a strict subset of it.  A lost record only ever removes a name: a call that launches a kernel
    outside `expected` shows it in every profile, and one that really launches fewer kernels shows the same strict
    subset every time, so neither can pass check_launched."""
    from torch.profiler import ProfilerActivity, profile

    for attempt in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            time.sleep(0.02)
            fn()
            torch.cuda.synchronize()
            time.sleep(0.02)
        evs = [e.name for e in prof.events()]
        mangled = [n for n in evs if n.startswith("_Z")]
        if mangled:
            evs += subprocess.run(["c++filt"], input="\n".join(mangled), capture_output=True, text=True,
                                  check=True).stdout.splitlines()
        got = {m.group(1) for n in evs for m in [re.search(rf"sfb::({names})", n)] if m}
        if not any("sfb::" in n for n in evs):
            warnings.warn(f"profile {attempt} recorded no sfb kernel ({len(evs)} events): taken again")
        elif expected is not None and got < set(expected):
            warnings.warn(f"profile {attempt} recorded only {sorted(got)} of {sorted(expected)}: taken again")
        else:
            break
    return got


def check_launched(fn, kernels, names=TEMPLATED):
    got = launched(fn, names, expected=kernels)
    assert got == set(kernels), f"launched {sorted(got)}, expected {sorted(kernels)}"


@pytest.fixture(scope="module")
def dev():
    """cuda:0, bound for the module's tests (import it into a test module to use it)"""
    ops_for()
    return DEV


@pytest.fixture(scope="module", name="dev")
def tc_dev():
    """the `dev` fixture of modules that test the wgmma engine only: skips their tests where it is unavailable"""
    ops_for("3xtf32")
    return DEV


# ----------------------------------------------------------------------------------------------- builders
def make_cfg(ocfg: O.OracleCfg, **over):
    """the device cfg of an oracle config (the extended configs' rnn_num_layers included), then `over`"""
    from sample_factory_b200.cfg import default_cfg

    cfg = default_cfg()
    for k in ["rollout", "recurrence", "batch_size", "num_batches_per_epoch", "num_epochs", "gamma", "gae_lambda",
              "ppo_clip_ratio", "ppo_clip_value", "exploration_loss_coeff", "value_loss_coeff", "kl_loss_coeff",
              "max_grad_norm", "learning_rate", "adam_eps", "adam_beta1", "adam_beta2", "normalize_input",
              "normalize_returns", "value_bootstrap", "with_vtrace", "vtrace_rho", "vtrace_c", "reward_scale",
              "reward_clip", "max_policy_lag", "nonlinearity", "obs_subtract_mean", "obs_scale", "use_rnn", "rnn_type",
              "rnn_size", "adaptive_stddev", "continuous_tanh_scale", "initial_stddev", "exploration_loss", "optimizer", "actor_critic_share_weights"]:
        setattr(cfg, k, getattr(ocfg, k))
    cfg.encoder_mlp_layers = list(ocfg.encoder_mlp_layers)
    cfg.decoder_mlp_layers = list(ocfg.decoder_mlp_layers)
    cfg.encoder_conv_architecture = ocfg.encoder_conv_architecture
    cfg.encoder_conv_mlp_layers = list(ocfg.encoder_conv_mlp_layers)
    cfg.rnn_num_layers = getattr(ocfg, "rnn_num_layers", 1)
    cfg.async_rl = False
    for k, v in over.items():
        setattr(cfg, k, v)
    return cfg


def model_spec(ocfg, obs_uint8=False):
    """the ModelSpec of an oracle config, the extended configs' obs_keys / action_heads / rnn_num_layers included"""
    from sample_factory_b200.model import ModelSpec

    return ModelSpec(ocfg.obs_dim, ocfg.num_actions, list(ocfg.encoder_mlp_layers), list(ocfg.decoder_mlp_layers),
                     ocfg.nonlinearity, ocfg.normalize_input, ocfg.normalize_returns, ocfg.obs_subtract_mean,
                     ocfg.obs_scale, ocfg.use_rnn, ocfg.rnn_type, ocfg.rnn_size, continuous=ocfg.continuous,
                     adaptive_stddev=ocfg.adaptive_stddev, continuous_tanh_scale=ocfg.continuous_tanh_scale,
                     initial_stddev=ocfg.initial_stddev, obs_shape=ocfg.obs_shape,
                     encoder_conv_architecture=ocfg.encoder_conv_architecture,
                     encoder_conv_mlp_layers=list(ocfg.encoder_conv_mlp_layers), obs_uint8=obs_uint8,
                     action_segments=ocfg.action_segments, share_weights=ocfg.actor_critic_share_weights,
                     action_heads=getattr(ocfg, "action_heads", None), obs_keys=getattr(ocfg, "obs_keys", None),
                     rnn_num_layers=getattr(ocfg, "rnn_num_layers", 1))


Rig = namedtuple("Rig", "cfg model traj env sampler learner")


def build(ocfg, N, state, tape, engine="simt", graph=False, **cfg_over):
    """model (loaded from `state`) + TapeVecEnv over `tape` + DeviceSampler (CUDA graph if `graph`) + Learner for N envs;
    skips when `engine` is unavailable"""
    from sample_factory_b200.envs import TapeVecEnv
    from sample_factory_b200.learner import Learner
    from sample_factory_b200.model import PolicyModel
    from sample_factory_b200.sampler import DeviceSampler
    from sample_factory_b200.trajectory import alloc_for_spec

    ops = ops_for(engine)
    cfg = make_cfg(ocfg, **cfg_over)
    model = PolicyModel(model_spec(ocfg, obs_uint8=tape.dtype == torch.uint8), DEV)
    model.load_state_dict(state, strict=False)
    traj = alloc_for_spec(model.spec, N, ocfg.rollout, DEV)
    env = TapeVecEnv(tape.to(DEV).contiguous(), ocfg.num_actions, continuous=ocfg.continuous, obs_shape=ocfg.obs_shape,
                     action_segments=ocfg.action_segments, with_action_mask=ocfg.action_mask,
                     action_heads=getattr(ocfg, "action_heads", None), obs_keys=getattr(ocfg, "obs_keys", None))
    sampler = DeviceSampler(cfg, env, model, traj, engine=ops.ENGINES[engine], use_cuda_graph=graph)
    learner = Learner(cfg, model, N, engine=ops.ENGINES[engine])
    return Rig(cfg, model, traj, env, sampler, learner)


def shuffled(z):
    """the fixture was trained on shuffled minibatches (it stores the permutations the reference drew)"""
    return "it0/mb_indices" in z.files


def build_case(case, engine, **cfg_over):
    """build() on a fixture's initial weights and tape, shuffling its minibatches if the reference did"""
    z, meta, ocfg = case
    return build(ocfg, meta["N"], state_from(z, "init/"), torch.from_numpy(z["tape"]), engine,
                 shuffle_minibatches=shuffled(z), **cfg_over)


# ----------------------------------------------------------------------------------------------- fixture replays
def _equal(got, ref, k):
    assert torch.equal(got[k].view(ref[k].shape), ref[k]), k


def _close(got, ref, k, rtol=1e-7):
    np.testing.assert_allclose(got[k].view(ref[k].shape).numpy(), ref[k].numpy(), atol=TOL, rtol=rtol, err_msg=k)


SAMPLER_EXACT = ("obs", "dones", "time_outs", "rewards", "actions", "policy_id", "policy_version")


def replay_sampler(case, rig, exact=SAMPLER_EXACT, states=True, discrete_cols=None, check_iteration=None):
    """the sampler on the reference's weights, obs tape and noise of every iteration against the reference's
    trajectories: the `exact` keys bit-exact, logits / values / log-probs (and with `states` the recurrent states) at
    1e-5.  Float actions -- Box actions, or the Tuple with Box members whose Discrete columns are `discrete_cols` -- and
    their rewards are compared at 1e-5 (relative 2e-5 more for the Tuple's actions), the Discrete columns bit-exact.  The
    policy stamps are not compared where the reference trained on deliberately stale samples (the last iteration of a
    poisoned fixture).  check_iteration(got, it) adds a feature's own checks."""
    z, meta, ocfg = case
    floats = ocfg.continuous or discrete_cols is not None
    rig.sampler.reset()
    for it in range(meta["iters"]):
        rig.model.load_state_dict(state_from(z, "init/") if it == 0 else state_from(z, f"it{it - 1}/state/"), strict=False)
        rig.sampler.set_policy_version(int(z[f"it{it}/train_step_before"]))
        rig.sampler.noise = torch.from_numpy(z[f"it{it}/noise"]).to(DEV).contiguous()
        rig.sampler.rollout()
        got = {k: v.cpu() for k, v in rig.traj.items()}
        ref = {k[len(f"it{it}/traj/"):]: torch.from_numpy(z[k]) for k in z.files if k.startswith(f"it{it}/traj/")}
        poisoned = meta.get("poison") and it == meta["iters"] - 1
        for k in exact:
            if floats and k in ("rewards", "actions"):
                _close(got, ref, k, rtol=2e-5 if discrete_cols is not None and k == "actions" else 1e-7)
            elif not (poisoned and k in ("policy_id", "policy_version")):
                _equal(got, ref, k)
        if discrete_cols is not None:
            assert torch.equal(got["actions"][:, :, discrete_cols], ref["actions"][:, :, discrete_cols])
        for k in ("action_logits", "log_prob_actions") + (("rnn_states",) if states else ()):
            _close(got, ref, k)
        np.testing.assert_allclose(got["values"][:, :-1].numpy(), ref["values"][:, :-1].numpy(), atol=TOL)
        if check_iteration is not None:
            check_iteration(got, it)


def upload_traj(traj_dev, traj_cpu):
    for k, v in traj_cpu.items():
        traj_dev[k].copy_(v.view(traj_dev[k].shape))


def post_state(z, it):
    return state_from(z, f"it{it}/state/")


def check_state(got, want):
    """post-Adam weights at 2e-5 and float64 normaliser statistics: the obs statistics are functions of exact inputs
    (1e-8); the returns statistics are moments of fp32 returns that themselves carry the 1e-5 tolerance (1e-6 on the
    moments).  An element whose gradient is comparable to adam_eps moves by lr * g / (|g| + eps), which amplifies a 1e-6
    gradient difference to ~1e-5 on the weight (seen on 2 of 8192 conv weights): hence 2e-5 on the weights."""
    for k, v in want.items():
        tol = (1e-6 if k.startswith("returns_normalizer") else 1e-8) if v.dtype == torch.float64 else 2 * TOL
        np.testing.assert_allclose(got[k].cpu().numpy().reshape(v.shape), v.numpy(), atol=tol, rtol=1e-6, err_msg=k)


def replay_learner(case, rig, prep=True, rewards=False, losses=True, upload=upload_traj, traj_of=traj_from,
                   state_of=post_state):
    """Learner.train on the reference's trajectories of every iteration (traj_of(z, it, ocfg), copied in by upload), on
    the reference's minibatch permutations if it shuffled, against what the reference computed: the train steps; with
    `prep` the valids, bootstrap values, advantages and returns (not under V-trace, whose targets the fixtures do not
    store) at 1e-5 and with `rewards` the prepared rewards at 1e-6; with `losses` the six loss columns of every minibatch
    at 1e-5; and the state after the iteration, state_of(z, it), by check_state."""
    from sample_factory_b200 import ops

    z, meta, ocfg = case
    learner, traj = rig.learner, rig.traj
    assert learner.shuffle == shuffled(z)
    for it in range(meta["iters"]):
        assert learner.train_step == int(z[f"it{it}/train_step_before"])
        upload(traj, traj_of(z, it, ocfg))
        if learner.shuffle:
            learner.set_minibatch_permutation(z[f"it{it}/mb_indices"])
        learner.train(traj)
        torch.cuda.synchronize()
        assert learner.train_step == int(z[f"it{it}/train_step_after"])
        p = f"it{it}/prep/"
        if prep:
            assert torch.equal(learner.valids_flat.view(-1).cpu(), torch.from_numpy(z[p + "valids"]))
            np.testing.assert_allclose(traj["values"][:, -1].cpu().numpy(), z[p + "bootstrap_values"], atol=TOL)
            if not ocfg.with_vtrace:
                np.testing.assert_allclose(learner.advantages.view(-1).cpu().numpy(), z[p + "advantages"], atol=TOL)
                np.testing.assert_allclose(learner.returns.view(-1).cpu().numpy(), z[p + "returns"], atol=TOL)
        if rewards:
            np.testing.assert_allclose(traj["rewards"].view(-1).cpu().numpy(), z[p + "rewards"], atol=1e-6)
        if losses:
            log = learner.minibatch_log().numpy()
            assert log.shape[0] == len(z[f"it{it}/loss/policy_loss"])
            for key in ["policy_loss", "value_loss", "exploration_loss", "kl_loss", "adv_mean", "adv_std"]:
                np.testing.assert_allclose(log[:, ops.LS[key]], z[f"it{it}/loss/{key}"], atol=TOL, rtol=1e-5, err_msg=key)
        check_state(rig.model.state_dict(), state_of(z, it))


# ----------------------------------------------------------------------------------------------- graph vs eager
def graphed_sampler_matches_eager(a, b):
    """rig b's sampler is CUDA-graphed, a's eager: after re-aligning both (the graphed sampler's first rollout runs an
    eager warm-up and the capture) a second rollout from the same state writes the same bits"""
    for smp in (a.sampler, b.sampler):
        smp.reset()
        smp.rollout()
    for smp in (a.sampler, b.sampler):
        smp.reset()
        smp.step_counter.zero_()
        smp.rollout()
    torch.cuda.synchronize()
    for k in a.traj:
        assert torch.equal(a.traj[k], b.traj[k]), f"graphed sampler differs from eager for {k}"


def graphed_learner_matches_eager(a, b, feed, iters=4, exp_avg_sq=False):
    """rig b's learner replays train() as one CUDA graph, a's launches kernel by kernel: after feed(it) has filled both
    trajectory buffers, each of `iters` train() calls (the first captures, later ones replay) leaves the same weights,
    (with exp_avg_sq) second Adam moments and minibatch losses"""
    assert b.learner.use_graph and not a.learner.use_graph
    for it in range(iters):
        feed(it)
        a.learner.train(a.traj)
        b.learner.train(b.traj)
        torch.cuda.synchronize()
        assert torch.equal(a.model.flat, b.model.flat), it
        if exp_avg_sq:
            assert torch.equal(a.model.exp_avg_sq, b.model.exp_avg_sq), it
        assert torch.equal(a.learner.minibatch_log(), b.learner.minibatch_log()), it
    assert b.learner.graph_replay_launches > 0


def sampled_feed(a, b):
    """feed for graphed_learner_matches_eager: a rollout of a's sampler, copied into b's buffers"""
    def feed(it):
        a.sampler.set_policy_version(a.learner.train_step)
        a.sampler.rollout()
        for k in a.traj:
            b.traj[k].copy_(a.traj[k])
    return feed


# ----------------------------------------------------------------------------------------------- persistent rollout
def compare_rollout_runs(a, b, what):
    """logits, values and log-probs agree to ~2 ulp of their size; everything else is bit-identical"""
    for ta, tb in zip(a["traj"], b["traj"]):
        for k in ta:
            if k in ("action_logits", "values", "log_prob_actions"):
                np.testing.assert_allclose(ta[k].cpu().numpy(), tb[k].cpu().numpy(), rtol=0, atol=2e-6, err_msg=f"{what} {k}")
            elif k != "valids":
                assert torch.equal(ta[k], tb[k]), (what, k)
    for k in ("obs", "rew", "term", "step", "pstep"):
        assert torch.equal(a[k], b[k]), (what, k)
    np.testing.assert_allclose(a["stats"].cpu().numpy(), b["stats"].cpu().numpy(), rtol=1e-12)
    assert torch.equal(a["ep"][0], b["ep"][0]) and torch.equal(a["ep"][1], b["ep"][1])


def rollout_pair(ocfg, N, seed, graph=False):
    """one model, two samplers over identical envs: per-step launches (fused tail) and the persistent kernel"""
    from sample_factory_b200.envs import TapeVecEnv
    from sample_factory_b200.sampler import DeviceSampler
    from sample_factory_b200.trajectory import alloc_for_spec

    ops = ops_for("3xtf32")
    st0 = O.init_state(ocfg, seed=seed)
    tape = torch.randn(2 * ocfg.rollout + 3, N, ocfg.obs_dim, generator=torch.Generator().manual_seed(seed + 1))
    old = {k: os.environ.get(k) for k in ("SFB200_TAIL_FUSED", "SFB200_ROLLOUT_FUSED")}
    try:
        os.environ["SFB200_TAIL_FUSED"] = "1"
        os.environ["SFB200_ROLLOUT_FUSED"] = "0"
        cfg, model, traj_s, env_s, sampler_s, learner = build(ocfg, N, st0, tape, "3xtf32")
        os.environ["SFB200_ROLLOUT_FUSED"] = "1"
        traj_p = alloc_for_spec(model.spec, N, ocfg.rollout, DEV)
        env_p = TapeVecEnv(tape.to(DEV).contiguous(), ocfg.num_actions)
        sampler_p = DeviceSampler(cfg, env_p, model, traj_p, engine=ops.GEMM_TC_3XTF32, use_cuda_graph=graph)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    assert sampler_s.fused_tail and not sampler_s.fused_rollout
    assert sampler_p.fused_rollout
    return model, learner, (sampler_s, traj_s, env_s), (sampler_p, traj_p, env_p)


def rollout_state(sampler, traj, env):
    return dict(traj=[{k: v.clone() for k, v in traj.items()}], obs=env.obs.clone(), rew=env.rew.clone(),
                term=env.terminated.clone(), step=env.step_counter.clone(), pstep=sampler.step_counter.clone(),
                stats=sampler.episode_stats.clone(), ep=(sampler.ep_return.clone(), sampler.ep_len.clone()))


def check_persistent_rollout(obs_dim=64, hidden=512, num_actions=8, N=512, T=4, rollouts=2, train=False, graph=False, form=None,
                             normalize=True, nonlinearity="elu"):
    """the per-step launches (fused tail) and the persistent rollout kernel on one model: rollouts of both samplers
    compared after each one (train: learner.train on the persistent trajectories in between,
    so the weights, their fp16 twins and the h1 bound change); form: the operand form the kernel must have taken;
    normalize=False: a model without fp16 twins (every GEMM of both paths in the tf32 form)"""
    from sample_factory_b200 import ops

    ocfg = O.OracleCfg(obs_dim=obs_dim, num_actions=num_actions, encoder_mlp_layers=[hidden, hidden], rollout=T,
                       recurrence=1, batch_size=N * T // 2, num_batches_per_epoch=2, normalize_input=normalize,
                       nonlinearity=nonlinearity)
    model, learner, (ss, ts, es), (sp, tp, ep) = rollout_pair(ocfg, N, seed=3 + hidden + obs_dim + N + T, graph=graph)
    ss.reset()
    sp.reset()
    if graph:
        ss.rollout()   # the graphed sampler's first rollout() also runs its eager warm-up rollout
    for it in range(rollouts):
        for k in tp:          # what a rollout does not write (the bootstrap value column, learner outputs) alike
            ts[k].copy_(tp[k])
        ss.set_policy_version(it)
        sp.set_policy_version(it)
        ss.rollout()
        sp.rollout()
        if form is not None:
            assert ops.rollout_last_form() == form
        torch.cuda.synchronize()
        compare_rollout_runs(rollout_state(ss, ts, es), rollout_state(sp, tp, ep), f"rollout {it}")
        if train:
            learner.train(tp)
    if graph:
        assert sp.graph_replay_launches == 2


# ----------------------------------------------------------------------------------------------- host envs and runners
class _Space:
    def __init__(self, shape=None, n=None, dtype=np.float32):
        self.shape, self.dtype = shape, dtype
        if n is not None:
            self.n = n


class MiniCartPole:
    """classic cart-pole dynamics (Barto, Sutton & Anderson), float64 state, float32 observations"""

    def __init__(self, max_steps=40):
        self.observation_space = _Space(shape=(4,))
        self.action_space = _Space(shape=(), n=2)
        self.max_steps = max_steps
        self.rng = np.random.RandomState(0)
        self.s, self.t = None, 0

    def reset(self, seed=None):
        if seed is not None:
            self.rng = np.random.RandomState(seed)
        self.s = self.rng.uniform(-0.05, 0.05, size=4)
        self.t = 0
        return self.s.astype(np.float32), {}

    def step(self, a):
        x, xd, th, thd = self.s
        f = 10.0 if a == 1 else -10.0
        ct, st = math.cos(th), math.sin(th)
        tmp = (f + 0.05 * thd * thd * st) / 1.1
        tha = (9.8 * st - ct * tmp) / (0.5 * (4.0 / 3.0 - 0.1 * ct * ct / 1.1))
        xa = tmp - 0.05 * tha * ct / 1.1
        self.s = np.array([x + 0.02 * xd, xd + 0.02 * xa, th + 0.02 * thd, thd + 0.02 * tha])
        self.t += 1
        terminated = bool(abs(self.s[0]) > 2.4 or abs(self.s[2]) > 12 * math.pi / 180)
        truncated = bool(self.t >= self.max_steps and not terminated)
        return self.s.astype(np.float32), 1.0, terminated, truncated, {"t": self.t}


def runner(env_name, make_env, argv_extra):
    """a Runner over the env `make_env` registers as `env_name`, one process, the flags of argv_extra"""
    from sample_factory_b200.cfg import parse_full_cfg, parse_sf_args
    from sample_factory_b200.envs import register_env
    from sample_factory_b200.train import Runner

    register_env(env_name, make_env)
    argv = [f"--env={env_name}", "--experiment=cfg_test", "--train_dir=/tmp/sfb200_tests", "--restart_behavior=overwrite",
            "--batched_sampling=True", "--num_workers=1", "--num_envs_per_worker=1", "--worker_num_splits=1", "--seed=0",
            "--save_every_sec=100000", "--experiment_summaries_interval=100000"] + argv_extra
    parser, _ = parse_sf_args(argv)
    cfg = parse_full_cfg(parser, argv)
    r = Runner(cfg)
    r.init()
    return r


def check_finite(r, n_iter, expect_steps):
    """n_iter iterations of the Runner r: finite statistics and weights, expect_steps env steps; returns the statistics"""
    for _ in range(n_iter):
        r.iteration()
    torch.cuda.synchronize()
    st = r.learner.fetch_stats()
    bad = {k: v for k, v in st.items() if isinstance(v, float) and not np.isfinite(v)}
    assert not bad, bad
    assert torch.isfinite(r.model.flat).all()
    assert r.env_steps == expect_steps
    return st


# --------------------------------------------------------------------------------------------------------------- heads
def masked_rows(M, A, seed):
    mask = torch.rand(M, A, generator=g(seed)) > 0.6
    mask[0] = False                  # a row that allows nothing: uniform fallback
    mask[1] = False
    mask[1, A - 1] = True            # only the last action
    return mask


def wide_tail(ops, h, Wv, bv, logits, A, noise=None, mask=None, deterministic=False, **kw):
    """run sfb200_heads_tail_wide on rows already holding the logits; returns (values, actions, log_prob, pv)"""
    M = h.shape[0]
    values = torch.full((M,), float("nan"), device=DEV)
    width = kw.get("act_dim", 0) if kw.get("continuous") else (len(kw["head_sizes"]) if kw.get("head_sizes") else 1)
    actions = torch.full((M, width), float("nan"), device=DEV)
    lp = torch.full((M,), float("nan"), device=DEV)
    pv_out = torch.full((M,), float("nan"), device=DEV)
    pv = torch.full((1,), 7.0, device=DEV)
    env = torch.empty((M, width), dtype=torch.float32 if kw.get("continuous") else torch.int32, device=DEV)
    if mask is not None or deterministic:
        ops.set_sampling_mode(mask, deterministic)
    try:
        ops.heads_tail_wide(h, Wv, bv, logits, logits.stride(0), A, values, 1, noise=noise, actions_f32=actions,
                            actions_stride=width, env_actions=env, log_prob=lp, log_prob_stride=1,
                            policy_version_scalar=pv, policy_version_out=pv_out, pv_stride=1, philox_seed=5, **kw)
    finally:
        ops.set_sampling_mode(None, False)
    torch.cuda.synchronize()
    assert torch.all(pv_out == 7.0)
    return values.cpu(), actions.cpu(), lp.cpu(), env.cpu()


# ---------------------------------------------------------------------------------------------------------- wgmma GEMM
class Registered:
    """fp16 twins + transposed twins of W, bounds of x and dz, registered for the duration of a block"""

    def __init__(self, W, x=None, dz=None):
        from sample_factory_b200 import ops

        self.W, self.x, self.dz = W, x, dz
        self.twins = torch.empty(2 * W.numel(), dtype=torch.float16, device=W.device)
        self.twinsT = torch.empty(2 * W.numel(), dtype=torch.float16, device=W.device)
        ops.register_f16_twins(W.view(-1), self.twins)
        ops.register_f16_transposed(W, self.twinsT)
        self.bounds = []                                 # (the library keeps the bound's address: keep it alive)
        for t in (x, dz):
            if t is not None:
                self.bounds.append(torch.full((1,), float(t.abs().max().item()), device=W.device))
                ops.register_operand_bound(t, self.bounds[-1])

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        from sample_factory_b200 import ops

        for t in (self.x, self.dz):
            if t is not None:
                ops.unregister_operand_bound(t)
        ops.unregister_f16_transposed(self.W)
        ops.unregister_f16_twins(self.W.view(-1))


def tc_dw(dev, dz, x, bounds=None):
    """dW = dz^T x on the wgmma engine; bounds = (bound of dz, bound of x) registered for the call, or None (the tf32
    form)"""
    from sample_factory_b200 import ops

    M, N = dz.shape
    K = x.shape[1]
    W = torch.zeros(N, K, device=dev)
    ws = torch.empty(ops.linear_backward_workspace_bytes(M, N, K) // 4 + 4, device=dev)
    dW = torch.full((N, K), float("nan"), device=dev)
    keep = []
    if bounds is not None:
        for t, b in zip((dz, x), bounds):
            keep.append(torch.full((1,), float(b), device=dev))
            ops.register_operand_bound(t, keep[-1])
    try:
        ops.linear_backward(dz, x, W, ops.ACT["none"], dW, None, None, ops.GEMM_TC_3XTF32, ws)
        torch.cuda.synchronize()
    finally:
        if bounds is not None:
            ops.unregister_operand_bound(dz)
            ops.unregister_operand_bound(x)
    return dW


def mlp_learner(dev, hidden, N=512, T=16):
    """a 64 -> hidden -> 8 MLP model with its sampler (reset) and learner on the wgmma engine, N tape envs x T steps"""
    from sample_factory_b200.cfg import default_cfg
    from sample_factory_b200.envs import TapeVecEnv
    from sample_factory_b200.learner import Learner
    from sample_factory_b200.model import ModelSpec, PolicyModel
    from sample_factory_b200.sampler import DeviceSampler
    from sample_factory_b200 import ops
    from sample_factory_b200.trajectory import alloc_trajectory_tensors

    cfg = default_cfg()
    cfg.use_rnn, cfg.async_rl = False, False
    cfg.encoder_mlp_layers = list(hidden)
    cfg.rollout, cfg.recurrence, cfg.batch_size, cfg.num_batches_per_epoch = T, 1, N * T // 2, 2
    model = PolicyModel(ModelSpec(64, 8, list(hidden)), dev)
    traj = alloc_trajectory_tensors(64, 8, N, T, dev)
    tape = torch.randn(T + 1, N, 64, generator=g(74)).to(dev)
    sampler = DeviceSampler(cfg, TapeVecEnv(tape, 8), model, traj, engine=ops.GEMM_TC_3XTF32)
    learner = Learner(cfg, model, N, engine=ops.GEMM_TC_3XTF32)
    sampler.reset()
    return model, sampler, learner, traj


# ----------------------------------------------------------------------------------------------- Tuples with Box members
def discrete_cols(heads):
    """the action columns of a Tuple's Discrete members"""
    cols, c = [], 0
    for k, n in heads:
        if k == "discrete":
            cols.append(c)
        c += 1 if k == "discrete" else n
    return cols


def mixed_noise(heads, T, N, gen):
    return torch.cat([torch.empty(T, N, n).exponential_(generator=gen) if k == "discrete" else
                      torch.randn(T, N, n, generator=gen) for k, n in heads], 2)


def mixed_rig(heads, kw, N, T, st_seed, engine, graph=False, **cfg_over):
    """(ocfg, initial weights, tape, rig) of a Tuple(heads) policy, MLP [64, 128] unless kw says otherwise"""
    from tests import mixed_oracle as MO

    base = dict(rollout=T, recurrence=T if kw.get("with_vtrace") else 1, batch_size=N * T // 2, num_batches_per_epoch=2,
                encoder_mlp_layers=[64, 128], obs_dim=24)
    base.update(kw)
    ocfg = MO.MixedCfg(num_actions=MO.rows_of(heads), action_heads=heads, **base)
    MO.install()
    st0 = O.init_state(ocfg, seed=st_seed)
    tape = torch.randn(4 * T + 1, N, ocfg.obs_dim, generator=g(st_seed + 10)) * 1.3 - 0.1
    return ocfg, st0, tape, build(ocfg, N, st0, tape, engine, graph, **cfg_over)


def mixed_closed_loop_vs_oracle(heads, kw, engine, partials):
    """sampler + learner for 3 iterations against the torch restatement (tests/mixed_oracle.py) on the same tape, noise
    and initial weights; `partials`: the sampler's heads take the fused partials"""
    from sample_factory_b200 import ops
    from tests import mixed_oracle as MO

    N, T = 64, 8
    ocfg, st0, tape, (cfg, model, traj, env, sampler, learner) = mixed_rig(heads, kw, N, T, 3, engine)
    assert (sampler.heads_plan.P > 0) == partials
    olearner = O.OracleLearner(ocfg, st0)
    oenv = O.TapeVecEnv(tape, ocfg.num_actions)
    olast = oenv.reset()
    sampler.reset()
    gen = g(21)
    dcols = discrete_cols(heads)
    for it in range(3):
        noise = mixed_noise(heads, T, N, gen)
        otraj = O.alloc_trajectories(ocfg, N)
        olast = MO.rollout(ocfg, olearner.st, oenv, olast, otraj, noise, olearner.train_step)
        sampler.noise = noise.to(DEV)
        sampler.set_policy_version(learner.train_step)
        sampler.rollout()
        got = {k: v.cpu() for k, v in traj.items()}
        assert torch.equal(got["actions"][:, :, dcols], otraj["actions"][:, :, dcols]), it
        # Box actions eps * std + mean inherit the 1e-7-relative differences of the params
        np.testing.assert_allclose(got["actions"].numpy(), otraj["actions"].numpy(), rtol=2e-5, atol=TOL)
        for k in ["obs", "dones", "time_outs", "policy_id", "policy_version"]:
            assert torch.equal(got[k], otraj[k]), k
        np.testing.assert_allclose(got["rewards"].numpy(), otraj["rewards"].numpy(), atol=TOL)
        np.testing.assert_allclose(got["action_logits"].numpy(), otraj["action_logits"].numpy(), atol=TOL)
        np.testing.assert_allclose(got["values"][:, :-1].numpy(), otraj["values"][:, :-1].numpy(), atol=TOL)
        np.testing.assert_allclose(got["log_prob_actions"].numpy(), otraj["log_prob_actions"].numpy(), atol=TOL)
        n0 = len(olearner.log)
        olearner.train(otraj)
        learner.train(traj)
        log = learner.minibatch_log().numpy()
        for j, d in enumerate(olearner.log[n0:]):
            for key in ["policy_loss", "value_loss", "exploration_loss", "kl_loss"]:
                assert abs(log[j, ops.LS[key]] - d[key]) < TOL, (it, j, key, log[j, ops.LS[key]], d[key])
        sd = model.state_dict()
        for k in O.param_names(ocfg):
            np.testing.assert_allclose(sd[k].cpu().numpy(), olearner.st[k].numpy(), atol=2e-5, err_msg=k)
