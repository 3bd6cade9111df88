"""Generate the wide-heads fixtures (distribution_linear with more than 31 rows) by executing the reference (same driver as
make_golden.py, whose run_case this script calls):  python tests/golden/make_golden_wide.py [case ...]

  tiny_wide_mask           Discrete(96) with action masks, MLP [64, 64], symmetric-KL exploration loss, poisoned data
  tiny_wide_tuple          Tuple(Discrete(24), Discrete(5), Discrete(16)): 45 logits, not a multiple of 4, so the logits
                           GEMM writes trajectory slots at an unaligned row stride; V-trace (recurrence = rollout)
  tiny_wide_gauss          Box(20) with the default adaptive stddev (40 distribution_linear rows), fixed-KL loss,
                           value bootstrap
  tiny_wide_gauss_learned  Box(36), one learned log-stddev vector (36 rows) and tanh-squashed means
"""
from __future__ import annotations

import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import make_golden as MG  # noqa: E402

if __name__ == "__main__":
    MG.run_case(
        "tiny_wide_mask", N=32, T=8, obs_dim=16, A=96, hidden=[64, 64], iters=2,
        overrides=dict(batch_size=128, num_batches_per_epoch=2, num_epochs=1, exploration_loss="symmetric_kl",
                       exploration_loss_coeff=0.01),
        poison=True, action_mask=True,
    )
    MG.run_case(
        "tiny_wide_tuple", N=32, T=8, obs_dim=16, A=45, hidden=[64, 64], iters=2,
        overrides=dict(batch_size=128, num_batches_per_epoch=2, num_epochs=1, with_vtrace=True, recurrence=8,
                       normalize_returns=False),
        poison=False, action_segments=[24, 5, 16],
    )
    MG.run_case(
        "tiny_wide_gauss", N=32, T=8, obs_dim=16, A=20, hidden=[64, 64], iters=2,
        overrides=dict(batch_size=128, num_batches_per_epoch=2, num_epochs=1, kl_loss_coeff=0.05, value_bootstrap=True),
        poison=True, continuous=True,
    )
    MG.run_case(
        "tiny_wide_gauss_learned", N=32, T=8, obs_dim=16, A=36, hidden=[64, 64], iters=2,
        overrides=dict(batch_size=128, num_batches_per_epoch=2, num_epochs=1, nonlinearity="tanh", adaptive_stddev=False,
                       continuous_tanh_scale=1.5, initial_stddev=0.7, kl_loss_coeff=0.1, exploration_loss_coeff=0.0),
        poison=True, continuous=True,
    )
