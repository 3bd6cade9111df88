"""Helpers to load the committed reference-generated fixtures (tests/golden/*.npz, made by make_golden.py)."""
import ast
import os

import numpy as np
import torch

from oracle import appo_oracle as O

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load_case(name):
    z = np.load(os.path.join(GOLDEN_DIR, f"{name}.npz"), allow_pickle=False)
    meta = ast.literal_eval(str(z["meta"]))
    _arrays = ("cfg/rnn_type", "cfg/nonlinearity", "cfg/encoder_conv_architecture", "cfg/encoder_conv_mlp_layers",
               "cfg/exploration_loss", "cfg/optimizer")
    c = {k[4:]: z[k].item() for k in z.files if k.startswith("cfg/") and k not in _arrays}
    cfg = O.OracleCfg(
        obs_dim=meta["obs_dim"], num_actions=meta["A"], encoder_mlp_layers=list(meta["hidden"]),
        decoder_mlp_layers=list(meta.get("decoder", [])),
        actor_critic_share_weights=bool(c.get("actor_critic_share_weights", True)),
        rollout=meta["T"], recurrence=int(c["recurrence"]), batch_size=int(c["batch_size"]),
        num_batches_per_epoch=int(c["num_batches_per_epoch"]), num_epochs=int(c["num_epochs"]),
        gamma=c["gamma"], gae_lambda=c["gae_lambda"], ppo_clip_ratio=c["ppo_clip_ratio"],
        ppo_clip_value=c["ppo_clip_value"], exploration_loss_coeff=c["exploration_loss_coeff"],
        value_loss_coeff=c["value_loss_coeff"], kl_loss_coeff=c["kl_loss_coeff"], max_grad_norm=c["max_grad_norm"],
        learning_rate=c["learning_rate"], adam_eps=c["adam_eps"], adam_beta1=c["adam_beta1"],
        adam_beta2=c["adam_beta2"], normalize_input=bool(c["normalize_input"]),
        normalize_returns=bool(c["normalize_returns"]), value_bootstrap=bool(c["value_bootstrap"]),
        with_vtrace=bool(c["with_vtrace"]), vtrace_rho=c["vtrace_rho"], vtrace_c=c["vtrace_c"],
        reward_scale=c["reward_scale"], reward_clip=c["reward_clip"], max_policy_lag=int(c["max_policy_lag"]),
        use_rnn=bool(c.get("use_rnn", False)), rnn_size=int(c.get("rnn_size", 512)),
        rnn_type=str(z["cfg/rnn_type"]) if "cfg/rnn_type" in z.files else "gru",
        nonlinearity=str(z["cfg/nonlinearity"]) if "cfg/nonlinearity" in z.files else "elu",
        continuous=bool(c.get("continuous", False)), adaptive_stddev=bool(c.get("adaptive_stddev", True)),
        continuous_tanh_scale=float(c.get("continuous_tanh_scale", 0.0)), initial_stddev=float(c.get("initial_stddev", 1.0)),
        exploration_loss=str(z["cfg/exploration_loss"]) if "cfg/exploration_loss" in z.files else "entropy",
        optimizer=str(z["cfg/optimizer"]) if "cfg/optimizer" in z.files else "adam",
        obs_scale=float(c.get("obs_scale", 1.0)), obs_subtract_mean=float(c.get("obs_subtract_mean", 0.0)),
        obs_shape=tuple(meta["obs_shape"]) if meta.get("obs_shape") else None,
        action_segments=list(meta["action_segments"]) if meta.get("action_segments") else None,
        action_mask=bool(meta.get("action_mask", False)),
        encoder_conv_architecture=(str(z["cfg/encoder_conv_architecture"]) if "cfg/encoder_conv_architecture" in z.files
                                   else "convnet_atari"),
        encoder_conv_mlp_layers=([int(v) for v in z["cfg/encoder_conv_mlp_layers"]] if "cfg/encoder_conv_mlp_layers" in z.files
                                 else [512]),
    )
    return z, meta, cfg


def load_mixed_case(name):
    """a fixture of tests/golden/make_golden_mixed.py -> (npz, meta, MixedCfg)"""
    import dataclasses

    from tests import mixed_oracle as MO

    z, meta, cfg = load_case(name)
    MO.install()
    return z, meta, MO.MixedCfg(**dataclasses.asdict(cfg), action_heads=[tuple(h) for h in meta["action_heads"]])


def state_from(z, prefix):
    """prefix 'init/' or 'it0/state/' -> dict of torch tensors keyed by reference state_dict names."""
    st = {k[len(prefix):]: torch.from_numpy(z[k].copy()) for k in z.files if k.startswith(prefix)}
    for k in (O.OBS_MEAN, O.OBS_VAR):   # image observations: per-pixel statistics [C,H,W] -> flat, like the obs rows
        if k in st and st[k].dim() > 1:
            st[k] = st[k].reshape(-1)
    return st


def traj_from(z, it, cfg):
    """Rebuild the trajectory batch (reference layout) the reference learner consumed in iteration `it`."""
    p = f"it{it}/traj/"
    t = {k[len(p):]: torch.from_numpy(z[k].copy()) for k in z.files if k.startswith(p)}
    N = t["actions"].shape[0]
    t["valids"] = torch.zeros((N, cfg.rollout + 1), dtype=torch.bool)
    return t
