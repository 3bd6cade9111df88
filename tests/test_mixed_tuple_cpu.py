"""Tuple action spaces with Box members, CPU side: the ModelSpec predicates and limits, construction-time checks, the
torch restatement (tests/mixed_oracle.py) against torch.distributions, and the oracle with that restatement against the
fixtures the reference produced (tests/golden/make_golden_mixed.py)."""
import math
import types

import numpy as np
import pytest
import torch

from sample_factory_b200.cfg import default_cfg
from sample_factory_b200.learner import Learner
from sample_factory_b200.model import ModelSpec
from tests import mixed_oracle as MO
from tests.golden_utils import load_mixed_case


def _spec(heads, **kw):
    return ModelSpec(obs_dim=8, num_actions=MO.rows_of(heads), action_heads=heads, **kw)


# rows / width by calc_num_action_parameters and calc_num_actions (action_distributions.py:16-44): Discrete(n) -> n / 1,
# Box(d) -> 2d / d, a Tuple sums its members
@pytest.mark.parametrize("heads,rows,width,wide", [
    ([("discrete", 4), ("box", 4)], 12, 5, False),
    ([("discrete", 3), ("box", 2), ("discrete", 4)], 11, 4, False),
    ([("box", 3), ("discrete", 5)], 11, 4, False),
    ([("box", 15), ("discrete", 1)], 31, 16, False),
    ([("box", 16)], 32, 16, True),
    ([("discrete", 24), ("box", 8), ("discrete", 5)], 45, 10, True),
    ([("box", 512)], 1024, 512, True),
])
def test_mixed_spec_rows_width_and_wide(heads, rows, width, wide):
    spec = _spec(heads)
    assert spec.num_linear_action_outputs == rows
    assert spec.num_action_params == rows          # ActionParameterizationDefault: params == distribution_linear rows
    assert spec.action_width == width
    assert spec.wide_heads is wide
    assert spec.head_kinds == [0 if k == "discrete" else 1 for k, _ in heads]
    assert spec.head_sizes == [n for _, n in heads]
    names = dict(spec.param_shapes())
    assert "action_parameterization.learned_stddev" not in names
    assert names["action_parameterization.distribution_linear.weight"] == (rows, 512)


def test_mixed_spec_ignores_stddev_options():
    base = _spec([("box", 3), ("discrete", 5)])
    other = _spec([("box", 3), ("discrete", 5)], adaptive_stddev=False, continuous_tanh_scale=1.5, initial_stddev=0.3)
    assert base.param_shapes() == other.param_shapes()


def test_all_discrete_heads_keep_the_tuple_path():
    spec = ModelSpec(obs_dim=8, num_actions=7, action_heads=[("discrete", 3), ("discrete", 4)])
    assert spec.action_heads is None and spec.action_segments == [3, 4]


def test_mixed_spec_limits():
    with pytest.raises(ValueError, match="at most 8 heads, got 9"):
        _spec([("discrete", 2)] * 8 + [("box", 1)])
    with pytest.raises(ValueError, match="1025 distribution_linear rows; the device path supports at most 1024"):
        _spec([("box", 512), ("discrete", 1)])
    with pytest.raises(ValueError, match="num_actions"):
        ModelSpec(obs_dim=8, num_actions=5, action_heads=[("box", 2)])
    with pytest.raises(ValueError, match="action_heads members"):
        ModelSpec(obs_dim=8, num_actions=2, action_heads=[("multibinary", 2)])


def test_from_cfg_reads_action_heads():
    cfg = default_cfg()
    env = types.SimpleNamespace(obs_dim=6, num_actions=11, action_heads=[("discrete", 3), ("box", 2), ("discrete", 4)])
    spec = ModelSpec.from_cfg(cfg, env)
    assert spec.action_heads == [("discrete", 3), ("box", 2), ("discrete", 4)]
    assert not spec.continuous and spec.action_segments is None and spec.action_width == 4


def test_symmetric_kl_with_box_member_raises_at_construction():
    cfg = default_cfg()
    cfg.exploration_loss = "symmetric_kl"
    cfg.rollout, cfg.recurrence, cfg.batch_size, cfg.num_batches_per_epoch = 4, 1, 8, 1
    model = types.SimpleNamespace(spec=_spec([("discrete", 4), ("box", 4)]), device=torch.device("cpu"))
    with pytest.raises(ValueError, match="symmetric_kl"):
        Learner(cfg, model, 2)


def test_restatement_matches_torch_distributions():
    """the oracle's mixed distribution against torch.distributions member by member"""
    heads = [("discrete", 3), ("box", 2), ("discrete", 4)]
    g = torch.Generator().manual_seed(0)
    N = 64
    params = torch.randn(N, MO.rows_of(heads), generator=g)
    params_old = params + 0.1 * torch.randn(params.shape, generator=g)
    noise = torch.cat([torch.empty(N, 3).exponential_(generator=g), torch.randn(N, 2, generator=g),
                       torch.empty(N, 4).exponential_(generator=g)], 1)
    acts = MO.mixed_sample(heads, params, noise)
    assert acts.shape == (N, 4)

    def dists(p):
        lg0, box, lg1 = torch.split(p, [3, 4, 4], dim=1)
        m, ls = torch.chunk(box, 2, dim=1)
        std = torch.clamp(ls.exp(), 1e-4, 1e4)
        return [torch.distributions.Categorical(logits=lg0),
                torch.distributions.Independent(torch.distributions.Normal(m, std), 1),
                torch.distributions.Categorical(logits=lg1)]

    d, do = dists(params), dists(params_old)
    lp = d[0].log_prob(acts[:, 0]) + d[1].log_prob(acts[:, 1:3]) + d[2].log_prob(acts[:, 3])
    torch.testing.assert_close(MO.mixed_log_prob(heads, params, acts), lp, atol=1e-5, rtol=0)
    torch.testing.assert_close(MO.mixed_entropy(heads, params), sum(x.entropy() for x in d), atol=1e-5, rtol=0)
    kl = sum(torch.distributions.kl_divergence(a, b) for a, b in zip(d, do))
    torch.testing.assert_close(MO.mixed_kl(heads, params, params_old), kl, atol=1e-5, rtol=0)
    # the Box member's draw is eps * std + mean with the product and the sum rounded separately
    m, ls = torch.chunk(params[:, 3:7], 2, dim=1)
    assert torch.equal(acts[:, 1:3], noise[:, 3:5] * torch.clamp(ls.exp(), 1e-4, 1e4) + m)
    det = MO.mixed_sample(heads, params, noise, deterministic=True)
    assert torch.equal(det[:, 1:3], m) and torch.equal(det[:, 0], params[:, :3].argmax(1).float())
    assert math.isfinite(float(lp.sum()))


# ----------------------------------------------------------------------------------------------- reference fixtures
MIXED_CASES = ["tiny_mixed", "tiny_mixed_kl", "tiny_wide_mixed"]


@pytest.mark.parametrize("name", MIXED_CASES)
def test_mixed_rollout_matches_reference(name):
    from oracle import appo_oracle as O
    from tests.golden_utils import state_from

    z, meta, cfg = load_mixed_case(name)
    assert cfg.num_actions == MO.rows_of(cfg.action_heads)
    env = O.TapeVecEnv(torch.from_numpy(z["tape"]), cfg.num_actions)
    last_obs = env.reset()
    for it in range(meta["iters"]):
        st = state_from(z, "init/") if it == 0 else state_from(z, f"it{it - 1}/state/")
        traj = O.alloc_trajectories(cfg, meta["N"])
        noise = torch.from_numpy(z[f"it{it}/noise"])
        assert noise.shape[-1] == MO.noise_width_of(cfg.action_heads)
        last_obs = MO.rollout(cfg, st, env, last_obs, traj, noise, int(z[f"it{it}/train_step_before"]))
        skip = {"policy_id", "policy_version"} if (meta["poison"] and it == meta["iters"] - 1) else set()
        for k in ["obs", "actions", "rewards", "dones", "time_outs", "policy_id", "policy_version"]:
            if k not in skip:
                np.testing.assert_array_equal(traj[k].numpy(), z[f"it{it}/traj/{k}"], err_msg=k)   # bit-exact
        for k in ["action_logits", "log_prob_actions"]:
            np.testing.assert_allclose(traj[k].numpy(), z[f"it{it}/traj/{k}"], atol=1e-6, rtol=0, err_msg=k)
        np.testing.assert_allclose(traj["values"][:, :-1].numpy(), z[f"it{it}/traj/values"][:, :-1], atol=1e-6, rtol=0)


@pytest.mark.parametrize("name", MIXED_CASES)
def test_mixed_learner_matches_reference(name):
    from oracle import appo_oracle as O
    from tests.golden_utils import state_from, traj_from

    z, meta, cfg = load_mixed_case(name)
    learner = O.OracleLearner(cfg, state_from(z, "init/"))
    assert "action_parameterization.learned_stddev" not in learner.st      # the stddev options are not read
    for it in range(meta["iters"]):
        n_log = len(learner.log)
        buff = learner.train(traj_from(z, it, cfg))
        assert learner.train_step == int(z[f"it{it}/train_step_after"])
        p = f"it{it}/prep/"
        np.testing.assert_array_equal(buff["valids"].numpy(), z[p + "valids"])
        for k in ["advantages", "returns"]:
            if p + k in z.files:
                np.testing.assert_allclose(buff[k].numpy(), z[p + k], atol=1e-5, rtol=0, err_msg=k)
        for key in ["policy_loss", "value_loss", "exploration_loss", "kl_loss", "adv_mean", "adv_std"]:
            got = np.array([d[key] for d in learner.log[n_log:]])
            np.testing.assert_allclose(got, z[f"it{it}/loss/{key}"], atol=1e-5, rtol=1e-5, err_msg=key)
        for k, v in state_from(z, f"it{it}/state/").items():
            tol = 1e-9 if v.dtype == torch.float64 else 1e-5
            np.testing.assert_allclose(learner.st[k].numpy(), v.numpy(), atol=tol, rtol=1e-6, err_msg=k)
