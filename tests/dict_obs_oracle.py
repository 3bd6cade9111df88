"""The CPU oracle's Dict observations of several 1-D keys (the reference's MultiInputEncoder, model/encoder.py:33-70, and
RunningMeanStdDictInPlace, algo/utils/running_mean_std.py:113-136), written in torch fp32 on top of oracle.appo_oracle.

`install()` extends oracle.appo_oracle: param_names, init_state, encoder_forward and normalize_obs handle a DictCfg with
two or more obs_keys and hand every other configuration to the original functions unchanged, so the oracle's rollout and
learner (which look these names up at call time) run the Dict model on packed rows.

  * rows are packed: key k in columns [c_k, c_k + d_k), keys in sorted order
  * each key is normalised as its own tensor with its own statistics obs_normalizer.running_mean_std.running_mean_std.{key}.*
  * each key has an MlpEncoder encoder.encoders.{key}.mlp_head.{2i}.* (encoder_mlp_layers = [] is the identity) and the
    outputs are concatenated along dim 1, in key order"""
from __future__ import annotations

import dataclasses
import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch
from torch import Tensor

from oracle import appo_oracle as O

_ORIG = {}
NORM_BASE = "obs_normalizer.running_mean_std.running_mean_std."


@dataclass
class DictCfg(O.OracleCfg):
    obs_keys: Optional[List[Tuple[str, int]]] = None     # [(key, d), ...] sorted; sum(d) == obs_dim

    def __post_init__(self):
        install()


def _multi(cfg) -> bool:
    keys = getattr(cfg, "obs_keys", None)
    return keys is not None and len(keys) > 1


def _slices(cfg):
    c = 0
    for k, d in cfg.obs_keys:
        yield k, c, d
        c += d


def key_w(key: str, i: int) -> str:
    return f"encoder.encoders.{key}.mlp_head.{2 * i}.weight"


def key_b(key: str, i: int) -> str:
    return f"encoder.encoders.{key}.mlp_head.{2 * i}.bias"


def norm_names(key: str) -> Tuple[str, str, str]:
    return tuple(f"{NORM_BASE}{key}.{f}" for f in ("running_mean", "running_var", "count"))


def encoder_out_size(cfg) -> int:
    return sum(cfg.encoder_mlp_layers[-1] if cfg.encoder_mlp_layers else d for _, d in cfg.obs_keys)


def _after_encoder_cfg(cfg):
    """the same model with the concatenation as its 'observation' and no encoder layers (core / decoder / heads shapes)"""
    return dataclasses.replace(cfg, obs_dim=encoder_out_size(cfg), encoder_mlp_layers=[], obs_keys=None)


def param_names(cfg) -> List[str]:
    if not _multi(cfg):
        return _ORIG["param_names"](cfg)
    names = [n for k, _ in cfg.obs_keys for i in range(len(cfg.encoder_mlp_layers)) for n in (key_w(k, i), key_b(k, i))]
    return names + _ORIG["param_names"](_after_encoder_cfg(cfg))


def init_state(cfg, seed: int = 0) -> Dict[str, Tensor]:
    if not _multi(cfg):
        return _ORIG["init_state"](cfg, seed)
    st = _ORIG["init_state"](_after_encoder_cfg(cfg), seed)
    for n in (O.OBS_MEAN, O.OBS_VAR, O.OBS_COUNT):
        del st[n]
    g = torch.Generator().manual_seed(seed + 104729)
    for k, d in cfg.obs_keys:
        for i, h in enumerate(cfg.encoder_mlp_layers):
            st[key_w(k, i)] = torch.randn(h, d, generator=g) / math.sqrt(d)
            st[key_b(k, i)] = torch.randn(h, generator=g) * 0.01
            d = h
    for k, d in cfg.obs_keys:
        mean, var, count = norm_names(k)
        st[mean], st[var], st[count] = (torch.zeros(d, dtype=torch.float64), torch.ones(d, dtype=torch.float64),
                                        torch.ones(1, dtype=torch.float64))
    return st


def normalize_obs(cfg, st: Dict[str, Tensor], obs: Tensor, update_stats: bool) -> Tensor:
    """normalize.py:51-70 on a Dict: each key's slice is normalised as its own tensor with its own statistics"""
    if not _multi(cfg):
        return _ORIG["normalize_obs"](cfg, st, obs, update_stats)
    assert abs(cfg.obs_subtract_mean) < 1e-8 and abs(cfg.obs_scale - 1.0) < 1e-8
    x = obs.float().clone()
    if cfg.normalize_input:
        for k, c, d in _slices(cfg):
            xk = x[:, c: c + d].clone()
            mean, var, count = norm_names(k)
            if update_stats:
                O.rms_update(st[mean], st[var], st[count], xk)
            O.rms_normalize_(xk, st[mean], st[var])
            x[:, c: c + d] = xk
    return x


def encoder_forward(cfg, st: Dict[str, Tensor], x: Tensor) -> Tensor:
    """MultiInputEncoder.forward (encoder.py:50-60)"""
    if not _multi(cfg):
        return _ORIG["encoder_forward"](cfg, st, x)
    outs = []
    for k, c, d in _slices(cfg):
        h = x[:, c: c + d]
        for i in range(len(cfg.encoder_mlp_layers)):
            h = O._act(cfg, torch.nn.functional.linear(h, st[key_w(k, i)], st[key_b(k, i)]))
        outs.append(h)
    return torch.cat(outs, 1)


def install() -> None:
    """route appo_oracle's observation / encoder description through this module (idempotent)"""
    for name, fn in (("param_names", param_names), ("init_state", init_state), ("normalize_obs", normalize_obs),
                     ("encoder_forward", encoder_forward)):
        if name not in _ORIG:
            _ORIG[name] = getattr(O, name)
            setattr(O, name, fn)


def load_dict_case(name: str):
    """a fixture of tests/golden/make_golden_dict_obs.py -> (npz, meta, DictCfg)"""
    import ast

    from tests.golden_utils import load_case

    z, meta, cfg = load_case(name)
    keys = [tuple(k) for k in ast.literal_eval(str(z["cfg/obs_keys"]))]
    return z, meta, DictCfg(**dataclasses.asdict(cfg), obs_keys=keys)


def traj_from(z, it, cfg):
    """the trajectory batch the reference learner consumed in iteration `it`, observations as packed rows"""
    from tests import golden_utils

    t = golden_utils.traj_from(z, it, cfg)
    return {k: v for k, v in t.items() if not k.startswith("obs/")}
