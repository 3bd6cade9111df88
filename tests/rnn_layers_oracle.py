"""The CPU oracle's stacked recurrent core (the reference's nn.GRU / nn.LSTM(input, rnn_size, rnn_num_layers),
model/core.py:19-64), written in torch fp32 on top of oracle.appo_oracle's one-layer cell.

`install()` extends oracle.appo_oracle with it: param_names, init_state, rnn_state_size and rnn_cell handle a StackedCfg
with rnn_num_layers > 1 and hand every other configuration to the original functions unchanged, so the oracle's rollout
and learner (which look these names up at call time) run the stacked model too.

  * parameters per layer k, in parameters() order: core.core.{weight_ih,weight_hh,bias_ih,bias_hh}_l{k}; layer k > 0
    reads H inputs
  * state rows are layer-major (core.py:42-60): [h_0 | h_1 | ...] (GRU), [h_0 | c_0 | h_1 | c_1 | ...] (LSTM);
    get_rnn_size (model_utils.py:11-24) = H * L, doubled for the LSTM
  * one step: layer k runs the one-layer cell on its slice of the state, its input is layer k-1's new h; the core
    output is the top layer's h.  A done / invalid boundary zeroes the whole row, so every layer restarts from zero."""
from __future__ import annotations

import dataclasses
import math
from dataclasses import dataclass
from typing import Dict, List, Tuple

import torch
from torch import Tensor

from oracle import appo_oracle as O

_ORIG = {}


@dataclass
class StackedCfg(O.OracleCfg):
    rnn_num_layers: int = 1     # cfg.py:543

    def __post_init__(self):
        install()


def layers_of(cfg) -> int:
    return getattr(cfg, "rnn_num_layers", 1) if cfg.use_rnn else 1


def rnn_names(k: int) -> Tuple[str, str, str, str]:
    return (f"core.core.weight_ih_l{k}", f"core.core.weight_hh_l{k}", f"core.core.bias_ih_l{k}",
            f"core.core.bias_hh_l{k}")


def layer_state_size(cfg) -> int:
    return cfg.rnn_size * (2 if cfg.rnn_type == "lstm" else 1)


def param_names(cfg) -> List[str]:
    names = _ORIG["param_names"](cfg)
    L = layers_of(cfg)
    if L == 1:
        return names
    i = names.index(O.RNN_B_HH) + 1
    upper = [n for k in range(1, L) for n in rnn_names(k)]
    return names[:i] + upper + names[i:]


def init_state(cfg, seed: int = 0) -> Dict[str, Tensor]:
    """the original initial state plus layers 1..L-1 at the PyTorch RNN default U(-1/sqrt(H), 1/sqrt(H))"""
    st = _ORIG["init_state"](cfg, seed)
    L = layers_of(cfg)
    if L == 1:
        return st
    H, G = cfg.rnn_size, (4 if cfg.rnn_type == "lstm" else 3)
    g = torch.Generator().manual_seed(seed + 7919)
    b = 1.0 / math.sqrt(H)
    for k in range(1, L):
        w_ih, w_hh, b_ih, b_hh = rnn_names(k)
        st[w_ih] = (torch.rand(G * H, H, generator=g) * 2 - 1) * b
        st[w_hh] = (torch.rand(G * H, H, generator=g) * 2 - 1) * b
        st[b_ih] = (torch.rand(G * H, generator=g) * 2 - 1) * b
        st[b_hh] = (torch.rand(G * H, generator=g) * 2 - 1) * b
    return st


def rnn_state_size(cfg) -> int:
    if layers_of(cfg) == 1:
        return _ORIG["rnn_state_size"](cfg)
    return layer_state_size(cfg) * layers_of(cfg)


def rnn_cell(cfg, st: Dict[str, Tensor], x: Tensor, state: Tensor) -> Tuple[Tensor, Tensor]:
    L = layers_of(cfg)
    if L == 1:
        return _ORIG["rnn_cell"](cfg, st, x, state)
    Sl = layer_state_size(cfg)
    new_states = []
    for k in range(L):
        layer = dict(zip((O.RNN_W_IH, O.RNN_W_HH, O.RNN_B_IH, O.RNN_B_HH), (st[n] for n in rnn_names(k))))
        x, s = _ORIG["rnn_cell"](cfg, layer, x, state[:, k * Sl:(k + 1) * Sl])
        new_states.append(s)
    return x, torch.cat(new_states, dim=1)


def install() -> None:
    """route appo_oracle's recurrent-core description through this module (idempotent)"""
    for name, fn in (("param_names", param_names), ("init_state", init_state), ("rnn_state_size", rnn_state_size),
                     ("rnn_cell", rnn_cell)):
        if name not in _ORIG:
            _ORIG[name] = getattr(O, name)
            setattr(O, name, fn)


def load_stacked_case(name: str):
    """a fixture of tests/golden/make_golden_rnn_layers.py -> (npz, meta, StackedCfg)"""
    from tests.golden_utils import load_case

    z, meta, cfg = load_case(name)
    return z, meta, StackedCfg(**dataclasses.asdict(cfg), rnn_num_layers=int(z["cfg/rnn_num_layers"]))


def checkpoint_from(z) -> dict:
    """the reference's checkpoint dict (Learner._get_checkpoint_dict, learner.py:323-332) as the fixture stores it:
    train_step, env_steps, best_performance, model (state_dict in its key order), optimizer (Adam.state_dict), curr_lr"""
    p = "ckpt/"
    model = {k: torch.from_numpy(z[f"{p}model/{k}"].copy()) for k in z[f"{p}model_keys"].tolist()}
    state = {}
    for i in range(int(z[f"{p}num_opt_states"])):
        state[i] = dict(step=torch.tensor(float(z[f"{p}optimizer/{i}/step"])),
                        exp_avg=torch.from_numpy(z[f"{p}optimizer/{i}/exp_avg"].copy()),
                        exp_avg_sq=torch.from_numpy(z[f"{p}optimizer/{i}/exp_avg_sq"].copy()))
    import ast

    groups = ast.literal_eval(str(z[f"{p}param_groups"]))
    return dict(train_step=int(z[f"{p}train_step"]), env_steps=int(z[f"{p}env_steps"]),
                best_performance=float(z[f"{p}best_performance"]), model=model,
                optimizer=dict(state=state, param_groups=groups), curr_lr=float(z[f"{p}curr_lr"]))
