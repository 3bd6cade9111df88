"""The CPU oracle's Tuple action space with Discrete and Box members (the reference's TupleActionDistribution with
ActionParameterizationDefault, action_distributions.py:197-286 / actor_critic.py:43-53), written in torch fp32:
torch.split of the distribution_linear outputs per member ([means | log_std] for a Box member), one distribution per
member, log-prob / entropy / KL summed over the members.

`install()` extends oracle.appo_oracle with it: action_width, policy_step and the dist_* functions handle a MixedCfg with
`action_heads` and hand every other configuration to the original functions unchanged, so the oracle's learner (which
looks these names up at call time) trains the mixed model too.  `rollout` is the oracle's rollout with the reference's
preprocess_actions for such a Tuple (batched_sampling.py:46-57): one entry per member, int32 [N] or float32 [N, d]."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch
from torch import Tensor

from oracle import appo_oracle as O

_ORIG = {}


@dataclass
class MixedCfg(O.OracleCfg):
    # [("discrete", n) | ("box", d), ...]; num_actions = distribution_linear rows = sum(n or 2d)
    action_heads: Optional[List[Tuple[str, int]]] = None

    def __post_init__(self):
        # the oracle's functions only know this space once they are extended: a MixedCfg never meets the originals
        install()


def rows_of(heads) -> int:
    return sum(n if k == "discrete" else 2 * n for k, n in heads)


def width_of(heads) -> int:
    return sum(1 if k == "discrete" else n for k, n in heads)


def noise_width_of(heads) -> int:
    return sum(n for _, n in heads)


def _split(heads, params: Tensor, actions: Optional[Tensor] = None):
    ps = torch.split(params, [n if k == "discrete" else 2 * n for k, n in heads], dim=1)
    if actions is None:
        return ps
    acts = torch.split(actions.view(params.shape[0], -1), [1 if k == "discrete" else n for k, n in heads], dim=1)
    return ps, acts


def mixed_sample(heads, params: Tensor, noise: Tensor, deterministic: bool = False) -> Tensor:
    """[N, W] float actions; noise [N, W'] = per member Exp(1) per logit / N(0,1) per Box dimension"""
    qs = torch.split(noise, [n for _, n in heads], dim=1)
    out = []
    for (k, _), p, q in zip(heads, _split(heads, params), qs):
        if k == "discrete":
            a = torch.argmax(O.cat_probs(p), -1, keepdim=True) if deterministic else O.cat_sample(p, q)
            out.append(a.float())
        else:
            out.append(O.gauss_split(p)[0].clone() if deterministic else O.gauss_sample(p, q))
    return torch.cat(out, dim=1)


def mixed_log_prob(heads, params: Tensor, actions: Tensor) -> Tensor:
    ps, acts = _split(heads, params, actions)
    return sum(O.cat_log_prob(p, a) if k == "discrete" else O.gauss_log_prob(p, a) for (k, _), p, a in zip(heads, ps, acts))


def mixed_entropy(heads, params: Tensor) -> Tensor:
    return sum(O.cat_entropy(p) if k == "discrete" else O.gauss_entropy(p) for (k, _), p in zip(heads, _split(heads, params)))


def mixed_kl(heads, params_p: Tensor, params_q: Tensor) -> Tensor:
    return sum(O.cat_kl(p, q) if k == "discrete" else O.gauss_kl(p, q)
               for (k, _), p, q in zip(heads, _split(heads, params_p), _split(heads, params_q)))


def env_actions(heads, actions: Tensor) -> List[Tensor]:
    """preprocess_actions: int32 [N] per Discrete member (squeezed), float32 [N, d] per Box member"""
    acts = torch.split(actions, [1 if k == "discrete" else n for k, n in heads], dim=1)
    return [a.to(torch.int32).squeeze(-1) if k == "discrete" else a for (k, _), a in zip(heads, acts)]


def _heads(cfg):
    return getattr(cfg, "action_heads", None)


def _action_width(cfg):
    return width_of(cfg.action_heads) if _heads(cfg) else _ORIG["action_width"](cfg)


def _policy_step(cfg, st, obs, noise_q, rnn_state=None, action_mask=None):
    if not _heads(cfg):
        return _ORIG["policy_step"](cfg, st, obs, noise_q, rnn_state, action_mask)
    assert action_mask is None
    x = O.normalize_obs(cfg, st, obs, update_stats=False)
    values, logits, new_state = O.model_forward(cfg, st, x, rnn_state)
    actions = mixed_sample(cfg.action_heads, logits, noise_q)
    return actions, logits, mixed_log_prob(cfg.action_heads, logits, actions), values, new_state


def _dist_log_prob(cfg, logits, actions):
    return mixed_log_prob(cfg.action_heads, logits, actions) if _heads(cfg) else _ORIG["dist_log_prob"](cfg, logits, actions)


def _dist_entropy(cfg, logits):
    return mixed_entropy(cfg.action_heads, logits) if _heads(cfg) else _ORIG["dist_entropy"](cfg, logits)


def _dist_kl(cfg, logits_p, logits_q):
    return mixed_kl(cfg.action_heads, logits_p, logits_q) if _heads(cfg) else _ORIG["dist_kl"](cfg, logits_p, logits_q)


def install() -> None:
    if _ORIG:
        return
    for name, fn in (("action_width", _action_width), ("policy_step", _policy_step), ("dist_log_prob", _dist_log_prob),
                     ("dist_entropy", _dist_entropy), ("dist_kl", _dist_kl)):
        _ORIG[name] = getattr(O, name)
        setattr(O, name, fn)


def rollout(cfg: MixedCfg, st: Dict[str, Tensor], env: O.TapeVecEnv, last_obs: Tensor, traj: Dict[str, Tensor],
            noise: Tensor, policy_version: int) -> Tensor:
    """O.rollout for a mixed Tuple (non-recurrent): noise [T, N, W']"""
    install()
    for t in range(cfg.rollout):
        traj["obs"][:, t] = last_obs
        traj["rnn_states"][:, t] = 0.0
        actions, logits, log_prob, values, _ = O.policy_step(cfg, st, last_obs, noise[t])
        traj["actions"][:, t] = actions
        traj["action_logits"][:, t] = logits
        traj["log_prob_actions"][:, t] = log_prob
        traj["values"][:, t] = values
        traj["policy_version"][:, t] = float(policy_version)
        # the tape env's rules on member 0: index / num_actions (Discrete) or clamp(a[:, 0], -1, 1) (Box)
        last_obs, rew, terminated, truncated = env.step(env_actions(cfg.action_heads, actions)[0])
        dones = terminated | truncated
        traj["rewards"][:, t] = (rew * cfg.reward_scale).clamp(-cfg.reward_clip, cfg.reward_clip)
        traj["dones"][:, t] = dones
        traj["time_outs"][:, t] = truncated
        traj["policy_id"][:, t] = cfg.policy_id
    traj["obs"][:, cfg.rollout] = last_obs
    traj["rnn_states"][:, cfg.rollout] = 0.0
    return last_obs
