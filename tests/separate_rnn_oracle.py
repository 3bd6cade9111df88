"""The CPU oracle's separate actor / critic weights with recurrent cores (ActorCriticSeparateWeights with use_rnn,
model/actor_critic.py:198-322), written in torch fp32 on top of oracle.appo_oracle and the stacked-core extension of
tests/rnn_layers_oracle.py.

`install()` extends oracle.appo_oracle with it: param_names, rnn_state_size, model_forward, separate_forward and
calculate_losses handle a SeparateRnnCfg with actor_critic_share_weights=False and use_rnn=True, and hand every other
configuration to the functions they replace unchanged, so the oracle's rollout and learner (which look these names up at
call time) run the model too.

  * parameters in registration order (actor_critic.py:208-224): actor encoder, actor core, critic encoder, critic core,
    actor decoder, critic decoder, critic_linear, action_parameterization; a core is {tower}core.core.{weight_ih,
    weight_hh,bias_ih,bias_hh}_l{k} per layer k
  * state rows are [actor state | critic state], each half laid out like a shared model's layer-major row
    (model_utils.py:11-24: get_rnn_size doubles)
  * each tower: encoder MLP -> its core on its half of the state -> decoder MLP; the critic tower feeds critic_linear,
    the actor tower the action parameterization
  * learner: each tower's core runs the done-aware BPTT of the shared model (the same masked loop as
    appo_oracle.calculate_losses: zero state after a done-or-invalid step, the chunk's stored state at its start)"""
from __future__ import annotations

import dataclasses
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch
from torch import Tensor

from oracle import appo_oracle as O
from tests import rnn_layers_oracle as RO

TOWERS = ("actor_", "critic_")
_ORIG = {}
_MB: Dict[str, Tensor] = {}     # the minibatch calculate_losses is working on (read by separate_forward)


@dataclass
class SeparateRnnCfg(RO.StackedCfg):
    def __post_init__(self):
        RO.install()
        install()


def is_separate_rnn(cfg) -> bool:
    return not cfg.actor_critic_share_weights and cfg.use_rnn


def core_names(tw: str, L: int) -> List[str]:
    return [f"{tw}core.core.{w}_l{k}" for k in range(L) for w in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]


def param_names(cfg) -> List[str]:
    if not is_separate_rnn(cfg):
        return _ORIG["param_names"](cfg)
    names = []
    for tw in TOWERS:
        for i in range(len(cfg.encoder_mlp_layers)):
            names += [O.enc_w(i, tw), O.enc_b(i, tw)]
        names += core_names(tw, RO.layers_of(cfg))
    for tw in TOWERS:
        for i in range(len(cfg.decoder_mlp_layers)):
            names += [O.dec_w(i, tw), O.dec_b(i, tw)]
    names += [O.CRITIC_W, O.CRITIC_B]
    if cfg.continuous and not cfg.adaptive_stddev:
        names += [O.LEARNED_STD]
    return names + [O.ACTION_W, O.ACTION_B]


def tower_state_size(cfg) -> int:
    return RO.layer_state_size(cfg) * RO.layers_of(cfg)


def rnn_state_size(cfg) -> int:
    if not is_separate_rnn(cfg):
        return _ORIG["rnn_state_size"](cfg)
    return 2 * tower_state_size(cfg)


def _mlp(cfg, st, h: Tensor, names) -> Tensor:
    for w, b in names:
        h = O._act(cfg, torch.nn.functional.linear(h, st[w], st[b]))
    return h


def _encoder(cfg, st, x: Tensor, tw: str) -> Tensor:
    return _mlp(cfg, st, x, [(O.enc_w(i, tw), O.enc_b(i, tw)) for i in range(len(cfg.encoder_mlp_layers))])


def _decoder(cfg, st, h: Tensor, tw: str) -> Tensor:
    return _mlp(cfg, st, h, [(O.dec_w(i, tw), O.dec_b(i, tw)) for i in range(len(cfg.decoder_mlp_layers))])


def _cell(cfg, st, tw: str, x: Tensor, state: Tensor) -> Tuple[Tensor, Tensor]:
    """one step of a tower's core: the (stacked) cell of the shared model on the tower's parameters"""
    core = {n[len(tw):]: v for n, v in st.items() if n.startswith(f"{tw}core.")}
    return O.rnn_cell(cfg, core, x, state)


def _heads(cfg, st, h_actor: Tensor, h_critic: Tensor) -> Tuple[Tensor, Tensor]:
    values = torch.nn.functional.linear(h_critic, st[O.CRITIC_W], st[O.CRITIC_B]).squeeze(-1)
    logits = torch.nn.functional.linear(h_actor, st[O.ACTION_W], st[O.ACTION_B])
    if cfg.continuous and not cfg.adaptive_stddev:
        means = logits
        if cfg.continuous_tanh_scale > 0:
            means = torch.tanh(means / cfg.continuous_tanh_scale) * cfg.continuous_tanh_scale
        logits = torch.cat((means, st[O.LEARNED_STD].repeat(means.shape[0], 1)), dim=1)
    return values, logits


def model_forward(cfg, st, x: Tensor, rnn_state: Optional[Tensor] = None):
    """ActorCriticSeparateWeights.forward (actor_critic.py:315-322), one step: (values, logits, new_rnn_state)"""
    if not is_separate_rnn(cfg):
        return _ORIG["model_forward"](cfg, st, x, rnn_state)
    S = tower_state_size(cfg)
    outs, states = {}, []
    for j, tw in enumerate(TOWERS):
        h, s = _cell(cfg, st, tw, _encoder(cfg, st, x, tw), rnn_state[:, j * S:(j + 1) * S])
        outs[tw] = _decoder(cfg, st, h, tw)
        states.append(s)
    values, logits = _heads(cfg, st, outs["actor_"], outs["critic_"])
    return values, logits, torch.cat(states, dim=1)


def separate_forward(cfg, st, x: Tensor) -> Tuple[Tensor, Tensor]:
    """the minibatch forward of calculate_losses (learner.py:553-586): per tower the masked BPTT loop over the
    recurrence-length chunks, starting from the tower's half of each chunk's stored state"""
    if not is_separate_rnn(cfg):
        return _ORIG["separate_forward"](cfg, st, x)
    mb = _MB
    R = cfg.recurrence
    n = x.shape[0] // R
    S = tower_state_size(cfg)
    doi = torch.logical_or(mb["dones"], ~mb["valids"]).view(n, R).float()      # done_or_invalid :560
    outs = {}
    for j, tw in enumerate(TOWERS):
        head = _encoder(cfg, st, x, tw).view(n, R, -1)
        state = mb["rnn_states"].view(n, R, -1)[:, 0, j * S:(j + 1) * S]
        core = []
        for t in range(R):
            if t > 0:
                state = state * (1.0 - doi[:, t - 1]).unsqueeze(-1)
            out, state = _cell(cfg, st, tw, head[:, t], state)
            core.append(out)
        outs[tw] = _decoder(cfg, st, torch.stack(core, 1).reshape(n * R, -1), tw)
    return _heads(cfg, st, outs["actor_"], outs["critic_"])


def calculate_losses(cfg, params, mb, num_invalids):
    if not is_separate_rnn(cfg):
        return _ORIG["calculate_losses"](cfg, params, mb, num_invalids)
    _MB.update(mb)
    try:
        return _ORIG["calculate_losses"](cfg, params, mb, num_invalids)
    finally:
        _MB.clear()


def install() -> None:
    """route appo_oracle's model description through this module (idempotent)"""
    for name, fn in (("param_names", param_names), ("rnn_state_size", rnn_state_size), ("model_forward", model_forward),
                     ("separate_forward", separate_forward), ("calculate_losses", calculate_losses)):
        if name not in _ORIG:
            _ORIG[name] = getattr(O, name)
            setattr(O, name, fn)


def load_separate_rnn_case(name: str):
    """a fixture of tests/golden/make_golden_separate_rnn.py -> (npz, meta, SeparateRnnCfg)"""
    from tests.golden_utils import load_case

    z, meta, cfg = load_case(name)
    return z, meta, SeparateRnnCfg(**dataclasses.asdict(cfg), rnn_num_layers=int(z["cfg/rnn_num_layers"]))


def checkpoint_from(z) -> dict:
    """the reference's checkpoint dict as the fixture stores it (rnn_layers_oracle.checkpoint_from); its model tensors,
    equal to the post-training state, are stored once under the prefix ckpt/model_in"""
    prefix = str(z["ckpt/model_in"])
    zz = {k: z[k] for k in z.files}
    for k in z["ckpt/model_keys"].tolist():
        zz[f"ckpt/model/{k}"] = z[f"{prefix}{k}"]
    return RO.checkpoint_from(zz)
