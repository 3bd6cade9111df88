"""Tuple action spaces with Box members (ModelSpec.action_heads): the three heads entry points against torch through the
policy forward (fused partials, unfused, wide), Philox statistics, the loss / ratio kernels against autograd, closed
loops of sampler + learner against the torch restatement (tests/mixed_oracle.py) on both engines, CUDA-graph replay,
and gymnasium-API CPU envs with Tuple spaces behind BatchedHostEnv."""
import math

import numpy as np
import pytest
import torch

from oracle import appo_oracle as O
from tests import mixed_oracle as MO
from tests.device_harness import (DEV, ENGINES, build_case, discrete_cols, g, graphed_learner_matches_eager,
                                  graphed_sampler_matches_eager, mixed_closed_loop_vs_oracle, mixed_rig, ops_for,
                                  replay_learner, replay_sampler, sampled_feed)
from tests.golden_utils import load_mixed_case

pytestmark = pytest.mark.gpu


def _model(heads, hidden=(64, 128), seed=0, obs_dim=16):
    from sample_factory_b200.model import ModelSpec, PolicyModel

    spec = ModelSpec(obs_dim, MO.rows_of(heads), list(hidden), action_heads=heads)
    model = PolicyModel(spec, DEV, seed=seed)
    gen = g(seed + 1)
    for k in model.names:          # non-trivial biases and larger weights: spread-out logits and stddevs
        p = model.params[k]
        scale = 0.2 if k.endswith("bias") else 1.5 / math.sqrt(p.shape[-1])
        p.copy_((torch.randn(p.shape, generator=gen) * scale).to(DEV))
    model.weights_changed()
    return model


def _policy(model, engine, x, noise=None, deterministic=False):
    """forward_policy with sampling outputs; returns (plan, values, params, actions, log_prob, env actions, pv_out)"""
    from sample_factory_b200.policy import HeadsPlan, forward_policy

    ops = ops_for()
    sp = model.spec
    M = x.shape[0]
    plan = HeadsPlan(model, engine, M)
    outs = [torch.empty((M, h), device=DEV) for h in sp.hidden]
    values = torch.full((M,), float("nan"), device=DEV)
    params = torch.full((M, sp.num_action_params), float("nan"), device=DEV)
    actions = torch.full((M, sp.action_width), float("nan"), device=DEV)
    lp = torch.full((M,), float("nan"), device=DEV)
    pv_out = torch.full((M,), float("nan"), device=DEV)
    env = [torch.full((M,), -7, dtype=torch.int32, device=DEV) if k == "discrete" else
           torch.full((M, n), float("nan"), device=DEV) for k, n in sp.action_heads]
    kw = dict(values=values, values_stride=1, logits=params, logits_stride=params.stride(0), noise=noise, philox_seed=9,
              philox_offset=3, actions_f32=actions, actions_stride=actions.stride(0), env_actions=env, log_prob=lp,
              log_prob_stride=1, policy_version_scalar=torch.full((1,), 4.0, device=DEV), policy_version_out=pv_out,
              pv_stride=1)
    if deterministic:
        ops.set_sampling_mode(None, True)
    try:
        forward_policy(model, x, outs, ops.ACT[sp.nonlinearity], engine, plan, kw, store_tail=False)
    finally:
        ops.set_sampling_mode(None, False)
    torch.cuda.synchronize()
    return plan, values.cpu(), params.cpu(), actions.cpu(), lp.cpu(), [e.cpu() for e in env], pv_out.cpu()


def _torch_forward(model, x):
    h = x
    for W, b in model.hidden_layers():
        h = torch.nn.functional.elu(h @ W.T + b)
    Wv, bv = model.critic
    Wa, ba = model.actor
    return (h @ Wv.T + bv).view(-1).cpu(), (h @ Wa.T + ba).cpu()


NARROW = [[("discrete", 3), ("box", 2), ("discrete", 4)], [("box", 3), ("discrete", 5)], [("box", 1)]]
FUSED = [[("discrete", 3), ("box", 2)], [("box", 3), ("discrete", 2)], [("box", 1)]]    # <= 8 rows: fused partials
WIDE = [[("discrete", 24), ("box", 8), ("discrete", 5)], [("box", 300), ("discrete", 62), ("box", 100)],
        [("discrete", 7), ("box", 2), ("discrete", 31), ("box", 5), ("discrete", 1)], [("box", 512)]]


@pytest.mark.parametrize("heads,path", [(h, "partials") for h in FUSED] + [(h, "forward") for h in NARROW] +
                         [(h, "wide") for h in WIDE])
@pytest.mark.parametrize("deterministic", [False, True])
def test_mixed_tail_matches_torch(heads, path, deterministic):
    ops = ops_for()
    if path == "partials" and not ops.tc_available():
        pytest.skip("wgmma engine not available")
    engine = ops.GEMM_TC_3XTF32 if path == "partials" else ops.GEMM_SIMT
    model = _model(heads, seed=len(heads))
    M = 777
    x = torch.randn(M, model.spec.obs_dim, generator=g(5)).to(DEV)
    Wn = MO.noise_width_of(heads)
    noise = torch.cat([torch.empty(M, n).exponential_(generator=g(6 + i)) if k == "discrete" else
                       torch.randn(M, n, generator=g(6 + i)) for i, (k, n) in enumerate(heads)], 1)
    assert noise.shape == (M, Wn)
    plan, values, params, actions, lp, env, pv = _policy(model, engine, x, noise.to(DEV), deterministic)
    assert (plan.P > 0) == (path == "partials") and plan.wide == (path == "wide")
    want_v, want_p = _torch_forward(model, x)
    np.testing.assert_allclose(values.numpy(), want_v.numpy(), atol=1e-5)
    np.testing.assert_allclose(params.numpy(), want_p.numpy(), atol=1e-5)
    # actions from the kernel's own params: Discrete indices bit-exact, Box values eps * std + mean up to the last bits
    # of expf (the stddev), means exactly in deterministic mode
    want_a = MO.mixed_sample(heads, params, noise, deterministic=deterministic)
    dcols = discrete_cols(heads)
    assert torch.equal(actions[:, dcols], want_a[:, dcols])
    if deterministic:
        assert torch.equal(actions, want_a)
    np.testing.assert_allclose(actions.numpy(), want_a.numpy(), rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(lp.numpy(), MO.mixed_log_prob(heads, params, actions).numpy(), rtol=1e-5, atol=1e-4)
    for e, w in zip(env, MO.env_actions(heads, actions)):
        assert e.dtype == w.dtype and torch.equal(e, w)
    assert torch.all(pv == 4.0)


def test_mixed_philox_statistics():
    """Philox draws: categorical frequencies follow the softmax, (a - mean) / std of a Box member is N(0, 1) per dim"""
    ops = ops_for()
    heads = [("discrete", 5), ("box", 3), ("discrete", 3)]
    model = _model(heads, seed=3)
    M = 1 << 16
    x = torch.randn(1, model.spec.obs_dim, generator=g(2)).expand(M, -1).contiguous().to(DEV)   # one state, many draws
    _, _, params, actions, lp, _, _ = _policy(model, ops.GEMM_SIMT, x)
    p0, box, p1 = torch.split(params[0], [5, 6, 3])
    for col, logits in ((0, p0), (4, p1)):
        freq = torch.bincount(actions[:, col].long(), minlength=logits.numel()).double() / M
        want = torch.softmax(logits.double(), 0)
        assert torch.all((freq - want).abs() < 5 * torch.sqrt(want * (1 - want) / M) + 1e-4), (freq, want)
    m, ls = box[:3], box[3:]
    z = (actions[:, 1:4].double() - m.double()) / ls.double().exp().clamp(1e-4, 1e4)
    assert torch.all(z.mean(0).abs() < 0.03) and torch.all((z.var(0) - 1).abs() < 0.03), (z.mean(0), z.var(0))
    assert len(torch.unique(actions[:, 1])) > M // 2            # distinct draws per row (subsequence row * W' + column)
    np.testing.assert_allclose(lp.numpy(), MO.mixed_log_prob(heads, params, actions).numpy(), atol=1e-5)


# ----------------------------------------------------------------------------------------------- loss kernels
def _torch_ppo(lp, lp_old, ent, kl, values, v_old, targets, adv, valids, c_ent, c_kl, clip=0.1, clip_v=0.2, c_val=0.5):
    vf = valids.double()
    n = vf.sum()
    am, asd = adv[valids].double().mean(), adv[valids].double().std().clamp_min(1e-7)
    advn = (adv.double() - am) / asd
    ratio = torch.exp(lp - lp_old).clamp(0.05, 20.0)
    pl = -(torch.min(ratio * advn, ratio.clamp(1 / (1 + clip), 1 + clip) * advn) * vf).sum() / n
    vc = v_old + (values - v_old).clamp(-clip_v, clip_v)
    vl = c_val * (torch.max((values - targets) ** 2, (vc - targets) ** 2) * vf).sum() / n
    return pl + vl - c_ent * (ent * vf).sum() / n + c_kl * (kl * vf).sum() / n


@pytest.mark.parametrize("heads", NARROW + WIDE)
@pytest.mark.parametrize("c_kl", [0.0, 0.05])
def test_mixed_loss_and_ratio_match_autograd(heads, c_kl):
    ops = ops_for()
    B = 600
    A = MO.rows_of(heads)
    gen = g(A)
    adv = torch.randn(B, generator=gen)
    valids = torch.rand(B, generator=gen) > 0.1
    v_old, targets = torch.randn(B, generator=gen), torch.randn(B, generator=gen)
    values = v_old + 0.3 * torch.randn(B, generator=gen)
    params = torch.randn(B, A, generator=gen) * 1.5
    lo = 0
    for k, n in heads:                  # some stddevs outside [1e-4, 1e4]: no gradient through the clamp
        if k == "box":
            params[:7, lo + n: lo + 2 * n] = -12.0
            params[7:11, lo + n: lo + 2 * n] = 11.0
        lo += n if k == "discrete" else 2 * n
    params_old = params + 0.2 * torch.randn(B, A, generator=gen)
    params_old[:11] = params[:11]       # (a finite KL for the clamped rows)
    noise = torch.cat([torch.empty(B, n).exponential_(generator=gen) if k == "discrete" else torch.randn(B, n, generator=gen)
                       for k, n in heads], 1)
    actions = MO.mixed_sample(heads, params_old, noise)
    lp_old = MO.mixed_log_prob(heads, params_old, actions) + 0.05 * torch.randn(B, generator=gen)
    c_ent = 0.01
    P = params.double().requires_grad_()
    V = values.double().requires_grad_()
    lp = MO.mixed_log_prob(heads, P, actions.double())
    ent = MO.mixed_entropy(heads, P)
    kl = MO.mixed_kl(heads, P, params_old.double())
    loss = _torch_ppo(lp, lp_old.double(), ent, kl, V, v_old.double(), targets.double(), adv, valids, c_ent, c_kl)
    loss.backward()
    stats = torch.zeros(ops.LS_SIZE, dtype=torch.float64, device=DEV)
    ws = torch.empty(ops.loss_workspace_bytes(B) // 8 + 8, dtype=torch.float64, device=DEV)
    vd = valids.to(DEV)
    ops.adv_stats(adv.to(DEV), vd, stats, None, ws)
    dl, dv = torch.empty(B, A, device=DEV), torch.empty(B, device=DEV)
    kinds, sizes = [0 if k == "discrete" else 1 for k, _ in heads], [n for _, n in heads]
    ops.ppo_loss_fwd_bwd_mixed(params.to(DEV), values.to(DEV), kinds, sizes, actions.to(DEV), lp_old.to(DEV),
                               v_old.to(DEV), adv.to(DEV), targets.to(DEV), vd, params_old.to(DEV), 0.1, 0.2, c_ent, 0.5,
                               c_kl, 1.0, dl, dv, stats, ws)
    s = stats.cpu()
    tot = s[ops.LS["total_loss"]].item()
    assert abs(tot - loss.item()) < 1e-5 * max(1.0, abs(loss.item())), (tot, loss.item())
    n = valids.sum().item()
    for key, want in (("entropy_mean", ent), ("kl_old_mean", kl)):
        w = (want.detach() * valids).sum().item() / n
        assert abs(s[ops.LS[key]].item() - w) < 1e-5 * max(1.0, abs(w)), (key, s[ops.LS[key]].item(), w)
    # rows 0..6 have stddevs at the 1e-4 clamp: their mean gradients carry a 1e8 factor on (a - mean), whose float32
    # rounding leaves ~1e-4 relative differences to the float64 reference
    np.testing.assert_allclose(dl.cpu().numpy()[11:], P.grad.numpy()[11:], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(dl.cpu().numpy()[:11], P.grad.numpy()[:11], rtol=1e-3, atol=1e-5)
    np.testing.assert_allclose(dv.cpu().numpy(), V.grad.numpy(), atol=1e-5)
    ratio = torch.empty(B, device=DEV)
    ops.action_ratio_mixed(params.to(DEV), kinds, sizes, actions.to(DEV), lp_old.to(DEV), ratio)
    want = torch.exp(lp.detach() - lp_old.double()).clamp(0.05, 20).numpy()
    np.testing.assert_allclose(ratio.cpu().numpy()[11:], want[11:], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(ratio.cpu().numpy()[:11], want[:11], rtol=1e-3, atol=1e-6)     # (the clamped rows)


# ----------------------------------------------------------------------------------------------- closed loops
CASES = {
    # Tuple(Discrete(3), Box(2)): 7 rows, fused partials on the wgmma engine
    "mixed_fused": dict(heads=[("discrete", 3), ("box", 2)], kw=dict()),
    # Tuple(Discrete(3), Box(2), Discrete(4)): 11 rows (narrow, unfused heads), entropy
    "mixed": dict(heads=[("discrete", 3), ("box", 2), ("discrete", 4)], kw=dict(exploration_loss_coeff=0.01)),
    # Tuple(Box(3), Discrete(5)): fixed KL, value bootstrap, tanh; the stddev options are set but not read
    "mixed_kl": dict(heads=[("box", 3), ("discrete", 5)],
                     kw=dict(kl_loss_coeff=0.3, value_bootstrap=True, nonlinearity="tanh", adaptive_stddev=False,
                             continuous_tanh_scale=1.5)),
    # Tuple(Discrete(24), Box(8), Discrete(5)): 45 rows (wide), V-trace
    "wide_mixed": dict(heads=[("discrete", 24), ("box", 8), ("discrete", 5)],
                       kw=dict(with_vtrace=True, normalize_returns=False)),
}


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("case", list(CASES))
def test_mixed_closed_loop_vs_oracle(case, engine):
    """sampler + learner for 3 iterations against the torch restatement on the same tape, noise and initial weights"""
    mixed_closed_loop_vs_oracle(CASES[case]["heads"], CASES[case]["kw"], engine,
                                partials=case == "mixed_fused" and engine != "simt")


@pytest.mark.parametrize("case", ["mixed", "wide_mixed"])
def test_mixed_graphed_learner_and_sampler_match_eager(case):
    eng = "3xtf32" if ops_for().tc_available() else "simt"
    heads, kw = CASES[case]["heads"], CASES[case]["kw"]
    a = mixed_rig(heads, kw, 64, 8, 5, eng)[3]
    b = mixed_rig(heads, kw, 64, 8, 5, eng, graph=True, learner_cuda_graph=True)[3]
    assert b.sampler.use_cuda_graph
    graphed_sampler_matches_eager(a, b)
    graphed_learner_matches_eager(a, b, sampled_feed(a, b), iters=3)


# ----------------------------------------------------------------------------------------------- reference fixtures
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", ["tiny_mixed", "tiny_mixed_kl", "tiny_wide_mixed"])
def test_mixed_rollout_matches_reference_golden(name, engine):
    """the sampler against the reference's own trajectories (same weights, tape and recovered per-member noise)"""
    case = load_mixed_case(name)
    replay_sampler(case, build_case(case, engine), exact=("obs", "dones", "time_outs", "rewards", "actions"), states=False,
                   discrete_cols=discrete_cols(case[2].action_heads))


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", ["tiny_mixed", "tiny_mixed_kl", "tiny_wide_mixed"])
def test_mixed_learner_matches_reference_golden(name, engine):
    """Learner.train on the reference's trajectories: loss terms (1e-5) and post-Adam weights (2e-5)"""
    case = load_mixed_case(name)
    replay_learner(case, build_case(case, engine), prep=False)


# ----------------------------------------------------------------------------------------------- host envs
class _Space:
    def __init__(self, shape=None, n=None, spaces=None):
        self.shape = shape
        if n is not None:
            self.n = n
        if spaces is not None:
            self.spaces = tuple(spaces)


class MixedIdentityEnv:
    """Tuple(Discrete(4), Box(-1, 1, (4,))) in the spirit of the reference's identity envs: the observation is a one-hot
    target t and a point c; reward = [a0 == t] - 0.25 * ||a1 - c||^2 (clipped per coordinate to [-1, 1])"""

    received = []

    def __init__(self, discrete_only=False, max_steps=16):
        self.discrete_only = discrete_only
        members = [_Space(shape=(), n=4), _Space(shape=(), n=3)] if discrete_only else [_Space(shape=(), n=4),
                                                                                         _Space(shape=(4,))]
        self.action_space = _Space(spaces=members)
        self.observation_space = _Space(shape=(8,))
        self.rng = np.random.RandomState(0)
        self.max_steps = max_steps

    def _obs(self):
        self.target = self.rng.randint(4)
        self.point = self.rng.uniform(-0.5, 0.5, size=4).astype(np.float32)
        o = np.zeros(8, dtype=np.float32)
        o[self.target] = 1.0
        o[4:] = self.point
        return o

    def reset(self, seed=None):
        if seed is not None:
            self.rng = np.random.RandomState(seed)
        self.t = 0
        return self._obs(), {}

    def step(self, action):
        assert isinstance(action, tuple) and len(action) == 2
        a0, a1 = action
        MixedIdentityEnv.received.append((type(a0), getattr(a1, "dtype", type(a1)), getattr(a1, "shape", None)))
        r = 1.0 if int(a0) == self.target else 0.0
        if not self.discrete_only:
            r -= 0.25 * float(np.sum((np.clip(a1, -1, 1) - self.point) ** 2))
        self.t += 1
        return self._obs(), r, False, self.t >= self.max_steps, {}


class MultiAgentMixedEnv(MixedIdentityEnv):
    """two agents: step() receives the reference's per-member batches (int32 [2], float32 [2, 4])"""

    num_agents = 2
    is_multiagent = True

    def reset(self, seed=None):
        o, _ = super().reset(seed)
        return [o, o.copy()], {}

    def step(self, actions):
        assert isinstance(actions, list) and len(actions) == 2
        a0, a1 = actions
        assert a0.dtype == np.int32 and a0.shape == (2,) and a1.dtype == np.float32 and a1.shape == (2, 4)
        MultiAgentMixedEnv.received.append(("multi", a0.dtype, a1.shape))
        o, r, tm, tr, info = super().step((a0[0], a1[0]))
        return [o, o.copy()], [r, r], [tm, tm], [tr, tr], [info, info]


def _train(env_name, make, tmp_path, env_steps):
    """run_rl on 32 envs behind BatchedHostEnv; returns the cfg (checkpoint and config are in tmp_path)"""
    from sample_factory_b200.cfg import parse_full_cfg, parse_sf_args
    from sample_factory_b200.envs import register_env
    from sample_factory_b200.host_env import BatchedHostEnv
    from sample_factory_b200.train import run_rl

    register_env(env_name, lambda name, cfg, env_config, render_mode=None: BatchedHostEnv(make, 32, DEV, seed=cfg.seed))
    argv = [f"--env={env_name}", "--experiment=mixed", f"--train_dir={tmp_path}", "--restart_behavior=overwrite",
            "--use_rnn=False", "--recurrence=1", "--rollout=16", "--batch_size=256", "--num_batches_per_epoch=2",
            "--num_epochs=2", "--encoder_mlp_layers", "64", "64", "--learning_rate=0.003", "--gamma=0.5",
            "--exploration_loss_coeff=0.001", "--async_rl=False", "--seed=0", f"--train_for_env_steps={env_steps}",
            "--save_every_sec=100000", "--experiment_summaries_interval=100000"]
    parser, _ = parse_sf_args(argv)
    cfg = parse_full_cfg(parser, argv)
    assert run_rl(cfg) == 0
    torch.cuda.synchronize()
    return cfg


def _enjoy(cfg):
    from sample_factory_b200.enjoy import enjoy

    cfg.cli_args = dict(max_num_episodes=16, eval_deterministic=True)
    cfg.max_num_episodes, cfg.eval_deterministic = 16, True
    status, avg = enjoy(cfg)
    assert status == 0 and math.isfinite(avg)
    return avg


def test_tuple_with_box_host_env_trains_and_enjoys(tmp_path):
    """Tuple(Discrete(4), Box(4)) CPU env through run_rl: the env receives (numpy integer, float32 ndarray[4]) per step,
    and the deterministic policy enjoy() loads from the checkpoint has learned both members (a random policy scores
    about -5 per 16-step episode, a perfect one 16)"""
    ops_for()
    MixedIdentityEnv.received.clear()
    cfg = _train("MixedIdentity-v0", lambda i: MixedIdentityEnv(), tmp_path, 60000)
    assert set(MixedIdentityEnv.received) == {(np.int32, np.dtype(np.float32), (4,))}
    assert _enjoy(cfg) > 8.0


def test_tuple_multi_agent_host_env_receives_member_batches(tmp_path):
    ops_for()
    MultiAgentMixedEnv.received.clear()
    _train("MixedIdentityMA-v0", lambda i: MultiAgentMixedEnv(), tmp_path, 2000)
    assert ("multi", np.dtype(np.int32), (2, 4)) in MultiAgentMixedEnv.received      # (step() checks the layout)


def test_tuple_of_discrete_host_env_trains(tmp_path):
    """Tuple(Discrete(4), Discrete(3)) CPU env (rejected by the host adapter before): trains, and member 0 is learned"""
    ops_for()
    MixedIdentityEnv.received.clear()
    cfg = _train("TupleDiscrete-v0", lambda i: MixedIdentityEnv(discrete_only=True), tmp_path, 40000)
    assert MixedIdentityEnv.received and all(np.issubdtype(r[0], np.integer) for r in MixedIdentityEnv.received)
    assert _enjoy(cfg) > 0.6 * 16
