"""Generate the fixtures of separate actor / critic weights with recurrent cores (--actor_critic_share_weights=False
--use_rnn=True) by executing the reference (the driver of make_golden.py, through make_golden_rnn_layers.run_case):
python tests/golden/make_golden_separate_rnn.py [case ...]

  tiny_separate_gru          GRU, H = 32, MLP [64], decoder MLP [32], Discrete(8): recurrence 8, value bootstrap,
                             poisoned data, 2 epochs x 2 minibatches; also carries the reference's checkpoint (ckpt/).
                             One iteration of 16 envs keeps it under 0.5 MB: the checkpoint's model tensors are the
                             post-training state bit for bit, so they are stored once, under it0/state/
                             (ckpt/model_in = that prefix).
  tiny_separate_lstm2        LSTM, 2 layers, H = 16, no encoder / decoder MLP (each core reads the observation, its
                             output feeds the heads), Box(3): V-trace (recurrence = rollout, normalize_returns=False)
  tiny_shuffle_separate_gru  GRU, H = 32, MLP [32]: recurrence 4 < rollout 8, shuffled minibatches

Each fixture records cfg/rnn_num_layers; the state rows are [actor state | critic state] (model_utils.py:11-24).
"""
from __future__ import annotations

import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402

import make_golden_rnn_layers as MR  # noqa: E402  (installs the reference shims)


def store_checkpoint_model_once(name: str, state_prefix: str) -> None:
    """drop the checkpoint's model tensors that equal the fixture's post-training state bit for bit (all of them: the
    reference saves the model it just trained) and record where they are"""
    path = os.path.join(MR.MG.OUT_DIR, f"{name}.npz")
    with np.load(path, allow_pickle=False) as z:
        out = {k: z[k] for k in z.files}
    for k in out["ckpt/model_keys"].tolist():
        a, b = out[f"ckpt/model/{k}"], out[f"{state_prefix}{k}"]
        assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b), k
        del out[f"ckpt/model/{k}"]
    out["ckpt/model_in"] = np.array(state_prefix)
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {os.path.getsize(path) / 1e6:.2f} MB")


if __name__ == "__main__":
    MR.run_case("tiny_separate_gru", 1, N=16, T=8, obs_dim=8, A=8, hidden=[64], iters=1,
                overrides=dict(batch_size=64, num_batches_per_epoch=2, num_epochs=2, use_rnn=True, rnn_type="gru",
                               rnn_size=32, decoder_mlp_layers=[32], recurrence=8, value_bootstrap=True,
                               actor_critic_share_weights=False),
                poison=True, save_checkpoint=True)
    if not MR.MG._ONLY or "tiny_separate_gru" in MR.MG._ONLY:
        store_checkpoint_model_once("tiny_separate_gru", "it0/state/")
    MR.run_case("tiny_separate_lstm2", 2, N=32, T=8, obs_dim=16, A=3, hidden=[], iters=2,
                overrides=dict(batch_size=128, num_batches_per_epoch=2, num_epochs=1, use_rnn=True, rnn_type="lstm",
                               rnn_size=16, recurrence=8, with_vtrace=True, normalize_returns=False,
                               actor_critic_share_weights=False),
                poison=False, continuous=True)
    MR.run_case("tiny_shuffle_separate_gru", 1, N=32, T=8, obs_dim=16, A=8, hidden=[32], iters=2,
                overrides=dict(batch_size=64, num_batches_per_epoch=4, num_epochs=1, use_rnn=True, rnn_type="gru",
                               rnn_size=32, recurrence=4, shuffle_minibatches=True, actor_critic_share_weights=False),
                poison=True)
