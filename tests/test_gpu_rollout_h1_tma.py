"""The fp16 form of the persistent rollout kernel stores h1 by TMA from shared-memory staging boxes.  Whole rollouts are
compared against the per-step launches with the rule of device_harness.compare_rollout_runs (bit-identical but for
logits / values / log-probs, 2e-6) at the bench shape (4096 envs, 512-512, T = 32: clusters of two) and at 4000 envs
(the last 64-row block has 32 rows, so the TMA stores clip), for every activation.

After the rollouts the h1 scratch holds the last step's h1 * 2^shift as fp16 [hi | lo] planes, [N][H1] halves each.
Rebuilt as hi + lo / 2048 they must match the per-step path's fp32 h1 of that step in every row: a box stored to the
wrong place, a stale staging buffer, or rows past N written into the next plane would all show here."""
import math

import pytest
import torch

from oracle import appo_oracle as O
from tests.device_harness import compare_rollout_runs, rollout_pair, rollout_state

pytestmark = pytest.mark.gpu


def _check(N, nonlinearity, T=32, hidden=512, rollouts=2):
    from sample_factory_b200 import ops

    ocfg = O.OracleCfg(obs_dim=64, num_actions=8, encoder_mlp_layers=[hidden, hidden], rollout=T, recurrence=1,
                       batch_size=N * T // 2, num_batches_per_epoch=2, nonlinearity=nonlinearity)
    model, _, (ss, ts, es), (sp, tp, ep) = rollout_pair(ocfg, N, seed=11 + N + T)
    ss.reset()
    sp.reset()
    for it in range(rollouts):
        for k in tp:
            ts[k].copy_(tp[k])
        ss.set_policy_version(it)
        sp.set_policy_version(it)
        ss.rollout()
        sp.rollout()
        assert ops.rollout_last_form() == 1
        torch.cuda.synchronize()
        compare_rollout_runs(rollout_state(ss, ts, es), rollout_state(sp, tp, ep), f"{nonlinearity} N={N} rollout {it}")

    bound = float(model.bound_h[0])
    shift = max(-100, min(100, 15 - math.frexp(bound)[1]))    # f16_shift_for_bound: bound * 2^shift in [2^14, 2^15)
    planes = sp.h[0].view(torch.float16).view(2, N, hidden).float()
    h1 = (planes[0] + planes[1] / 2048.0) * 2.0 ** -shift
    ref = ss.h[0]
    assert torch.isfinite(h1).all()
    torch.testing.assert_close(h1, ref, rtol=2e-6, atol=2e-6 * bound)


@pytest.mark.parametrize("nonlinearity", ["elu", "relu", "tanh"])
def test_bench_shape(nonlinearity):
    _check(4096, nonlinearity)


@pytest.mark.parametrize("nonlinearity", ["elu", "relu", "tanh"])
def test_clipped_row_block(nonlinearity):
    _check(4000, nonlinearity, T=7)
