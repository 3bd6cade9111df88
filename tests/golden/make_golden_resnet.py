"""Generate tests/golden/tiny_resnet.npz by executing the reference (same driver as make_golden.py, whose run_case this
script calls):  python tests/golden/make_golden_resnet.py

The case: the IMPALA ResNet encoder (ResnetEncoder, model/encoder.py:153-221) on uint8 [4, 10, 10] frames (rows of 400
bytes, a multiple of the 16 the device tape env reads at a time), 10 -> 5 -> 3 -> 2 through the padded pools (odd sizes
included), FC 64, ELU, obs_scale 255, one iteration of 2 epochs x 2 minibatches on poisoned data.

The fixture's size is dominated by the ~105 k conv weights, stored twice (initial and post-Adam).  To keep it small:
  * the reference's initial weights are rounded to multiples of 2^-8 right after Learner.init() (a coarse grid
    compresses well; the model, its optimizer and everything after are the reference's own);
  * the post-Adam weights are stored as float16 differences from the initial ones, `it0/state_delta_f16/<name>`
    (|difference| <= 4 Adam steps of lr 1e-4, so float16 keeps it to <= 2.5e-7, far inside the 1e-5 / 2e-5 checks);
    `it0/state/` keeps the float64 normaliser statistics.  tests/resnet_oracle.py: post_state() rebuilds the weights."""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import make_golden as MG  # noqa: E402

_orig_init = MG.Learner.init


def _init_on_grid(self, *a, **k):
    out = _orig_init(self, *a, **k)
    with torch.no_grad():
        for p in self.actor_critic.parameters():
            p.copy_(torch.round(p * 256.0) / 256.0)
    return out


if __name__ == "__main__":
    MG.Learner.init = _init_on_grid
    MG.run_case(
        "tiny_resnet", N=8, T=8, obs_dim=4 * 10 * 10, A=5, hidden=[], iters=1,
        overrides=dict(batch_size=32, num_batches_per_epoch=2, num_epochs=2, obs_scale=255.0,
                       encoder_conv_architecture="resnet_impala", encoder_conv_mlp_layers=[64]),
        poison=True, obs_shape=(4, 10, 10),
    )
    path = os.path.join(MG.OUT_DIR, "tiny_resnet.npz")
    z = dict(np.load(path))
    for k in [k for k in z if k.startswith("it0/state/") and z[k].dtype == np.float32]:
        name = k[len("it0/state/"):]
        z[f"it0/state_delta_f16/{name}"] = (z.pop(k).astype(np.float64) - z[f"init/{name}"]).astype(np.float16)
    np.savez_compressed(path, **z)
    print(f"rewrote {path}: {os.path.getsize(path) / 1e6:.2f} MB")
