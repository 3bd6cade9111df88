"""The CPU oracle's ResnetEncoder branch (the reference's model/encoder.py:153-221, resnet_impala), written in torch fp32
from the architecture: per stage Conv2d(3, padding 1) -> MaxPool2d(3, stride 2, padding 1) -> residual blocks
x + conv(act(conv(act(x)))), act(x) after the last stage, (C, H, W) flatten, fully connected layers.

`install()` extends oracle.appo_oracle with it: param_names, init_state and encoder_forward handle
`encoder_conv_architecture == "resnet_impala"` and hand every other configuration to the original functions unchanged,
so the oracle's rollout and learner (which look these names up at call time) run the ResNet model too."""
from __future__ import annotations

import dataclasses
import math
from typing import Dict, List, Tuple

import torch
import torch.nn.functional as F
from torch import Tensor

from oracle import appo_oracle as O

RESNET_STAGES = [(16, 2), (32, 2), (32, 2)]   # model/encoder.py:182 (resnet_impala): (channels, res blocks)

_ORIG = {}


def is_resnet(cfg) -> bool:
    return cfg.obs_shape is not None and cfg.encoder_conv_architecture == "resnet_impala"


def resnet_conv_names() -> List[str]:
    """state_dict prefixes of the convs in parameters() order: per stage the entry conv conv_head.{j} (the MaxPool2d is
    conv_head.{j+1}) and the two convs of every block, conv_head.{j}.res_block_core.{1,3} (encoder.py:157-162, 188-202)"""
    names, j = [], 0
    for _c, blocks in RESNET_STAGES:
        names.append(f"encoder.encoders.obs.conv_head.{j}")
        j += 2
        for _ in range(blocks):
            names += [f"encoder.encoders.obs.conv_head.{j}.res_block_core.{r}" for r in (1, 3)]
            j += 1
    return names


def fc_w(i: int) -> str:
    return f"encoder.encoders.obs.mlp_layers.{2 * i}.weight"   # no `.enc.` segment (encoder.py:208)


def fc_b(i: int) -> str:
    return f"encoder.encoders.obs.mlp_layers.{2 * i}.bias"


def conv_out_shape(cfg) -> Tuple[int, int, int]:
    """(C, H, W) of the conv head's output: 3x3 convs with padding 1 keep the size, every pool gives ceil(in / 2)"""
    _c, h, w = cfg.obs_shape
    for _co, _blocks in RESNET_STAGES:
        h, w = (h + 1) // 2, (w + 1) // 2
    return RESNET_STAGES[-1][0], h, w


def _tail_cfg(cfg, d: int):
    """the same model without an encoder: its parameters are the core / decoder / heads that follow the encoder"""
    return dataclasses.replace(cfg, obs_shape=None, obs_dim=d, encoder_mlp_layers=[])


def param_names(cfg) -> List[str]:
    if not is_resnet(cfg):
        return _ORIG["param_names"](cfg)
    names = []
    for p in resnet_conv_names():
        names += [p + ".weight", p + ".bias"]
    for i in range(len(cfg.encoder_conv_mlp_layers)):
        names += [fc_w(i), fc_b(i)]
    return names + _ORIG["param_names"](_tail_cfg(cfg, cfg.obs_dim))


def init_state(cfg, seed: int = 0) -> Dict[str, Tensor]:
    """random weights (like appo_oracle.init_state, not the reference's orthogonal init) + normalizer buffers"""
    if not is_resnet(cfg):
        return _ORIG["init_state"](cfg, seed)
    g = torch.Generator().manual_seed(seed)
    st: Dict[str, Tensor] = {}
    ci = cfg.obs_shape[0]
    names = iter(resnet_conv_names())
    for co, blocks in RESNET_STAGES:
        for _ in range(1 + 2 * blocks):
            p = next(names)
            st[p + ".weight"] = torch.randn(co, ci, 3, 3, generator=g) / math.sqrt(ci * 9)
            st[p + ".bias"] = torch.randn(co, generator=g) * 0.01
            ci = co
    d = math.prod(conv_out_shape(cfg))
    for i, h in enumerate(cfg.encoder_conv_mlp_layers):
        st[fc_w(i)] = torch.randn(h, d, generator=g) / math.sqrt(d)
        st[fc_b(i)] = torch.randn(h, generator=g) * 0.01
        d = h
    tail = _ORIG["init_state"](_tail_cfg(cfg, d), seed + 1)
    for k in (O.OBS_MEAN, O.OBS_VAR):
        tail.pop(k)
    st.update(tail)
    st[O.OBS_MEAN] = torch.zeros(cfg.obs_dim, dtype=torch.float64)
    st[O.OBS_VAR] = torch.ones(cfg.obs_dim, dtype=torch.float64)
    return st


def encoder_forward(cfg, st: Dict[str, Tensor], x: Tensor) -> Tensor:
    if not is_resnet(cfg):
        return _ORIG["encoder_forward"](cfg, st, x)
    h = x.view(x.shape[0], *cfg.obs_shape)
    names = iter(resnet_conv_names())
    for _co, blocks in RESNET_STAGES:
        p = next(names)
        h = F.max_pool2d(F.conv2d(h, st[p + ".weight"], st[p + ".bias"], padding=1), 3, stride=2, padding=1)
        for _ in range(blocks):
            pa, pb = next(names), next(names)
            r = F.conv2d(O._act(cfg, h), st[pa + ".weight"], st[pa + ".bias"], padding=1)
            h = h + F.conv2d(O._act(cfg, r), st[pb + ".weight"], st[pb + ".bias"], padding=1)
    h = O._act(cfg, h).reshape(h.shape[0], -1)
    for i in range(len(cfg.encoder_conv_mlp_layers)):
        h = O._act(cfg, F.linear(h, st[fc_w(i)], st[fc_b(i)]))
    return h


def install() -> None:
    """route appo_oracle's model description through this module (idempotent)"""
    for name, fn in (("param_names", param_names), ("init_state", init_state), ("encoder_forward", encoder_forward)):
        if name not in _ORIG:
            _ORIG[name] = getattr(O, name)
            setattr(O, name, fn)


def post_state(z, it: int = 0) -> Dict[str, Tensor]:
    """the reference's state after iteration `it` of a fixture written by tests/golden/make_golden_resnet.py: weights =
    initial weights + the stored float16 differences, normaliser statistics as stored"""
    from tests.golden_utils import state_from

    st = state_from(z, f"it{it}/state/")
    init = state_from(z, "init/")
    p = f"it{it}/state_delta_f16/"
    for k in z.files:
        if k.startswith(p):
            name = k[len(p):]
            st[name] = (init[name].double() + torch.from_numpy(z[k]).double()).float()
    return st
