"""Generate the fixtures of encoders without fully connected layers (--encoder_mlp_layers empty, --encoder_conv_mlp_layers
empty) by executing the reference (the driver of make_golden.py):  python tests/golden/make_golden_nofc.py [case ...]

  tiny_linear          identity MlpEncoder, no core, no decoder: the heads read the normalised observation (a linear
                       policy); Discrete(6) with an action mask, value bootstrap, poisoned data; also carries the
                       reference's checkpoint (tiny_linear_checkpoint.pth is folded in under ckpt/)
  tiny_linear_box      identity MlpEncoder, Box(3) with one learned log-stddev vector, fixed-KL loss
  tiny_dict_identity   keys a(5), b(7), identity key encoders, no core / decoder: the heads read the packed row; one
                       epoch, so the learner's CUDA graph covers a train() call
  tiny_conv_nofc       convnet_atari on uint8 [4, 44, 44], obs_scale 255, ReLU, the heads read the conv features (256)
  tiny_conv_nofc_gru   convnet_simple on uint8 [1, 36, 36] (128 features) -> GRU 32 -> decoder [32], recurrence 4 <
                       rollout 8, shuffled minibatches
  tiny_resnet_nofc     resnet_impala on uint8 [4, 10, 10], the heads read the features (128)

The image cases keep their files small with make_golden_resnet.py's rounding: the reference's initial weights are
rounded to multiples of 2^-8 right after Learner.init(), and the post-Adam weights are stored as float16 differences from
the initial ones (it0/state_delta_f16/<name>; tests/resnet_oracle.py: post_state() rebuilds them).
"""
from __future__ import annotations

import os
import shutil
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import make_golden as MG  # noqa: E402  (installs the reference shims)
import make_golden_dict_obs as MD  # noqa: E402
from make_golden_rnn_layers import _checkpoint_arrays  # noqa: E402

_orig_init = MG.Learner.init


def _init_on_grid(self, *a, **k):
    out = _orig_init(self, *a, **k)
    with torch.no_grad():
        for p in self.actor_critic.parameters():
            p.copy_(torch.round(p * 256.0) / 256.0)
    return out


def _rewrite(name: str, fn) -> None:
    path = os.path.join(MG.OUT_DIR, f"{name}.npz")
    with np.load(path, allow_pickle=False) as z:
        out = {k: z[k] for k in z.files}
    fn(out)
    np.savez_compressed(path, **out)
    print(f"rewrote {path}: {os.path.getsize(path) / 1e6:.2f} MB")


def _weights_as_deltas(out: dict) -> None:
    for k in [k for k in out if k.startswith("it0/state/") and out[k].dtype == np.float32]:
        name = k[len("it0/state/"):]
        out[f"it0/state_delta_f16/{name}"] = (out.pop(k).astype(np.float64) - out[f"init/{name}"]).astype(np.float16)


def fresh(name: str) -> None:
    """the reference's Learner.init() resumes from a checkpoint of an earlier run in the same experiment directory"""
    shutil.rmtree(os.path.join("/tmp/sfb200_golden", f"golden_{name}"), ignore_errors=True)


def image_case(name: str, **kw) -> None:
    if MG._ONLY and name not in MG._ONLY:
        return
    fresh(name)
    MG.Learner.init = _init_on_grid
    try:
        MG.run_case(name, **kw)
    finally:
        MG.Learner.init = _orig_init
    _rewrite(name, _weights_as_deltas)


def fold_checkpoint(name: str) -> None:
    """the checkpoint file the reference wrote goes into the fixture (ckpt/...) and is deleted"""
    if MG._ONLY and name not in MG._ONLY:
        return
    ck_path = os.path.join(MG.OUT_DIR, f"{name}_checkpoint.pth")
    _rewrite(name, lambda out: out.update(_checkpoint_arrays(ck_path)))
    os.remove(ck_path)


if __name__ == "__main__":
    for case in ("tiny_linear", "tiny_linear_box"):
        fresh(case)
    MG.run_case("tiny_linear", N=32, T=8, obs_dim=16, A=6, hidden=[], iters=2,
                overrides=dict(batch_size=128, num_batches_per_epoch=2, num_epochs=2, value_bootstrap=True),
                poison=True, save_checkpoint=True, action_mask=True)
    fold_checkpoint("tiny_linear")
    MG.run_case("tiny_linear_box", N=32, T=8, obs_dim=16, A=3, hidden=[], iters=2,
                overrides=dict(batch_size=128, num_batches_per_epoch=2, num_epochs=1, adaptive_stddev=False,
                               initial_stddev=0.7, kl_loss_coeff=0.1, exploration_loss_coeff=0.0),
                poison=True, continuous=True)
    MD.run_case("tiny_dict_identity", N=32, T=8, keys=[("a", 5), ("b", 7)], A=5, hidden=[], iters=2, poison=True,
                overrides=dict(batch_size=128, num_batches_per_epoch=2, num_epochs=1))
    image_case("tiny_conv_nofc", N=2, T=4, obs_dim=4 * 44 * 44, A=6, hidden=[], iters=1,
               overrides=dict(batch_size=4, num_batches_per_epoch=2, num_epochs=2, nonlinearity="relu", obs_scale=255.0,
                              encoder_conv_architecture="convnet_atari", encoder_conv_mlp_layers=[],
                              exploration_loss_coeff=0.01, max_grad_norm=0.5, adam_eps=1e-5, ppo_clip_ratio=0.1),
               poison=True, obs_shape=(4, 44, 44))
    image_case("tiny_conv_nofc_gru", N=4, T=8, obs_dim=36 * 36, A=5, hidden=[], iters=1,
               overrides=dict(batch_size=8, num_batches_per_epoch=4, num_epochs=1, obs_scale=255.0,
                              encoder_conv_architecture="convnet_simple", encoder_conv_mlp_layers=[], use_rnn=True,
                              rnn_type="gru", rnn_size=32, decoder_mlp_layers=[32], recurrence=4,
                              shuffle_minibatches=True),
               poison=True, obs_shape=(1, 36, 36))
    image_case("tiny_resnet_nofc", N=8, T=8, obs_dim=4 * 10 * 10, A=5, hidden=[], iters=1,
               overrides=dict(batch_size=32, num_batches_per_epoch=2, num_epochs=2, obs_scale=255.0,
                              encoder_conv_architecture="resnet_impala", encoder_conv_mlp_layers=[]),
               poison=True, obs_shape=(4, 10, 10))
