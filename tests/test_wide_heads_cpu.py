"""Heads wider than 31 distribution_linear rows, CPU side: the oracle against the reference-generated wide fixtures
(tests/golden/make_golden_wide.py), the ModelSpec.wide_heads predicate, and the construction-time limits."""
import pytest

import tests.test_oracle_golden as G
from sample_factory_b200.model import ModelSpec

WIDE_CASES = ["tiny_wide_mask", "tiny_wide_tuple", "tiny_wide_gauss", "tiny_wide_gauss_learned"]


@pytest.mark.parametrize("name", WIDE_CASES)
def test_wide_rollout_matches_reference(name):
    G.test_rollout_matches_reference(name)


@pytest.mark.parametrize("name", WIDE_CASES)
def test_wide_learner_matches_reference(name):
    G.test_learner_matches_reference(name)


@pytest.mark.parametrize("kw,rows,wide", [
    (dict(num_actions=31), 31, False),
    (dict(num_actions=32), 32, True),
    (dict(num_actions=362), 362, True),
    (dict(num_actions=15, continuous=True), 30, False),
    (dict(num_actions=16, continuous=True), 32, True),                             # adaptive stddev: 2 rows per dim
    (dict(num_actions=31, continuous=True, adaptive_stddev=False), 31, False),
    (dict(num_actions=32, continuous=True, adaptive_stddev=False), 32, True),
    (dict(num_actions=45, action_segments=[24, 5, 16]), 45, True),
    (dict(num_actions=9, action_segments=[3, 2, 4]), 9, False),
])
def test_wide_heads_predicate(kw, rows, wide):
    spec = ModelSpec(obs_dim=8, **kw)
    assert spec.num_linear_action_outputs == rows
    assert spec.wide_heads is wide


@pytest.mark.parametrize("kw", [
    dict(num_actions=1024),
    dict(num_actions=512, continuous=True),
    dict(num_actions=1024, continuous=True, adaptive_stddev=False),
    dict(num_actions=1024, action_segments=[1000, 24]),
    dict(num_actions=16, action_segments=[2] * 8),
])
def test_limits_accepted(kw):
    ModelSpec(obs_dim=8, **kw)


@pytest.mark.parametrize("kw,match", [
    (dict(num_actions=1025), "at most 1024"),
    (dict(num_actions=513, continuous=True), "at most 1024"),
    (dict(num_actions=1025, continuous=True, adaptive_stddev=False), "at most 1024"),
    (dict(num_actions=1025, action_segments=[1000, 25]), "at most 1024"),
    (dict(num_actions=18, action_segments=[2] * 9), "at most 8 heads"),
])
def test_limits_rejected_at_construction(kw, match):
    with pytest.raises(ValueError, match=match):
        ModelSpec(obs_dim=8, **kw)


def test_policy_model_rechecks_a_changed_spec():
    import torch

    from sample_factory_b200.model import PolicyModel

    spec = ModelSpec(obs_dim=8, num_actions=64, encoder_mlp_layers=[16])
    spec.num_actions = 2048
    with pytest.raises(ValueError, match="at most 1024"):
        PolicyModel(spec, torch.device("cpu"))
