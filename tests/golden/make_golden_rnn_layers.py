"""Generate the fixtures of stacked recurrent cores (--rnn_num_layers > 1) by executing the reference (the driver of
make_golden.py):  python tests/golden/make_golden_rnn_layers.py [case ...]

  tiny_gru2          GRU, 2 layers, H = 32, MLP [64]: recurrence 8, value bootstrap, poisoned data; also carries the
                     checkpoint the reference's Learner.save() wrote after the last iteration (under ckpt/)
  tiny_lstm3         LSTM, 3 layers, H = 32, MLP [64], decoder MLP [32]: recurrence 4, poisoned data
  tiny_shuffle_gru2  GRU, 2 layers: shuffled minibatches (the permutations the reference drew are recorded)

Each fixture also records cfg/rnn_num_layers.  The checkpoint is stored as arrays (its model state_dict in key order,
the Adam state per parameter index, the counters and the param_groups as a literal) so the tests can write it back out
with torch.save and load it through the product's checkpoint code.
"""
from __future__ import annotations

import os
import shutil
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import make_golden as MG  # noqa: E402  (installs the reference shims)


def _checkpoint_arrays(path: str) -> dict:
    ck = torch.load(path, map_location="cpu", weights_only=False)
    out = {"ckpt/model_keys": np.array(list(ck["model"].keys()))}
    for k, v in ck["model"].items():
        out[f"ckpt/model/{k}"] = v.numpy()
    state = ck["optimizer"]["state"]
    out["ckpt/num_opt_states"] = np.int64(len(state))
    for i, st in state.items():
        out[f"ckpt/optimizer/{i}/step"] = np.float64(float(st["step"]))
        out[f"ckpt/optimizer/{i}/exp_avg"] = st["exp_avg"].numpy()
        out[f"ckpt/optimizer/{i}/exp_avg_sq"] = st["exp_avg_sq"].numpy()
    out["ckpt/param_groups"] = np.array(repr(ck["optimizer"]["param_groups"]))
    for k in ("train_step", "env_steps"):
        out[f"ckpt/{k}"] = np.int64(ck[k])
    for k in ("best_performance", "curr_lr"):
        out[f"ckpt/{k}"] = np.float64(ck[k])
    return out


def run_case(name: str, rnn_num_layers: int, save_checkpoint: bool = False, **kw):
    if MG._ONLY and name not in MG._ONLY:
        return
    kw["overrides"] = dict(kw["overrides"], rnn_num_layers=rnn_num_layers)
    # the reference's Learner.init() resumes from a checkpoint of an earlier run in the same experiment directory
    shutil.rmtree(os.path.join("/tmp/sfb200_golden", f"golden_{name}"), ignore_errors=True)
    MG.run_case(name, save_checkpoint=save_checkpoint, **kw)
    path = os.path.join(MG.OUT_DIR, f"{name}.npz")
    with np.load(path, allow_pickle=False) as z:
        out = {k: z[k] for k in z.files}
    out["cfg/rnn_num_layers"] = np.float64(rnn_num_layers)
    if save_checkpoint:
        ck_path = os.path.join(MG.OUT_DIR, f"{name}_checkpoint.pth")
        out.update(_checkpoint_arrays(ck_path))
        os.remove(ck_path)
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {os.path.getsize(path) / 1e6:.2f} MB")


if __name__ == "__main__":
    run_case("tiny_gru2", 2, N=32, T=8, obs_dim=16, A=8, hidden=[64], iters=2,
             overrides=dict(batch_size=128, num_batches_per_epoch=2, num_epochs=2, use_rnn=True, rnn_type="gru",
                            rnn_size=32, recurrence=8, value_bootstrap=True),
             poison=True, save_checkpoint=True)
    run_case("tiny_lstm3", 3, N=32, T=8, obs_dim=16, A=8, hidden=[64], iters=2,
             overrides=dict(batch_size=128, num_batches_per_epoch=2, num_epochs=1, use_rnn=True, rnn_type="lstm",
                            rnn_size=32, decoder_mlp_layers=[32], recurrence=4),
             poison=True)
    run_case("tiny_shuffle_gru2", 2, N=32, T=8, obs_dim=16, A=8, hidden=[64], iters=2,
             overrides=dict(batch_size=64, num_batches_per_epoch=4, num_epochs=1, use_rnn=True, rnn_type="gru",
                            rnn_size=32, recurrence=4, shuffle_minibatches=True),
             poison=True)
