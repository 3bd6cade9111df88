"""Every width instantiation of the loss, action-ratio and heads kernels against a float64 reference.

The host picks a kernel instantiation from the row width or the activation (with_width / with_lpl / with_mixed_lpl in
csrc/loss.cu, launch_tail_rows in csrc/heads_wide.cu, heads_forward_impl / sfb200_heads_backward in csrc/heads.cu).  Each
instantiation is compiled on its own (registers, unrolling, spills, slot map), so one of them can be wrong while its
neighbours are right.  Every case below names an entry point, a width or member layout, and the instantiations the call
must launch: the case runs under torch.profiler and asserts that exactly those templated kernels ran, then compares
the outputs with a float64 reference built from the oracle (oracle/appo_oracle.py, tests/mixed_oracle.py; autograd for
the loss gradients).  Widths sit on both sides of every bucket edge and of the slot wrap at a full row.

Every loss case carries edge rows: invalid rows, raw ratios below 0.05 and above 20 (no gradient through the clamp),
ratios inside and outside the clip window with advantages of both signs, values exactly at and beyond the value clip,
logits spread by 100 (probabilities that are exactly 0 in float32) and Gaussian log-stddevs beyond the stddev clamp.
Whole-batch cases pin the minibatch with no valid row and with exactly one.

test_every_instantiation_has_a_case (CPU) reads the ptxas reports of an sm_90a build and fails when a templated kernel
has no case here (or in ROLLOUT_CASES, run by tests/test_gpu_rollout_pipeline.py) and is not on ALLOWLIST."""
import math
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from oracle import appo_oracle as O
from tests import mixed_oracle as MO
from tests.device_harness import DEV, check_launched, g, masked_rows, ops_for, wide_tail

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "sample_factory_b200", "csrc", "build")


# ----------------------------------------------------------------------------------------------- the table
def _cat(w):
    return f"ppo_loss_kernel<{w}>", f"action_ratio_kernel<{w}>"


def _cat_wide(lpl):
    return f"ppo_loss_wide_kernel<{lpl}>", f"action_ratio_wide_kernel<{lpl}>"


def _tup(w):
    return f"ppo_loss_tuple_kernel<{w}>", f"action_ratio_tuple_kernel<{w}>"


def _tup_wide(lpl):     # a Tuple's ratio shares the plain Discrete's wide kernel
    return f"ppo_loss_tuple_wide_kernel<{lpl}>", f"action_ratio_wide_kernel<{lpl}>"


def _gauss(w):
    return f"ppo_loss_gauss_kernel<{w}>", f"action_ratio_gauss_kernel<{w}>"


def _gauss_wide(lpl):
    return f"ppo_loss_gauss_wide_kernel<{lpl}>", f"action_ratio_gauss_wide_kernel<{lpl}>"


def _mixed(lpl):
    return f"ppo_loss_mixed_kernel<{lpl}>", f"action_ratio_mixed_kernel<{lpl}>"


# loss + ratio: (space, layout, instantiations).  discrete: A; tuple: head sizes; gauss: (act_dim, adaptive);
# mixed: members.  Tuples of 33+ logits have a head that crosses a 32-element slot boundary; mixed Tuples of 33+ rows
# have a Box member whose means and log-stddevs sit in different slots.
LOSS_CASES = [
    ("discrete", 1, _cat(8)), ("discrete", 8, _cat(8)), ("discrete", 9, _cat(16)), ("discrete", 16, _cat(16)),
    ("discrete", 17, _cat(32)), ("discrete", 31, _cat(32)), ("discrete", 32, _cat(32)),
    ("discrete", 33, _cat_wide(2)), ("discrete", 64, _cat_wide(2)), ("discrete", 65, _cat_wide(4)),
    ("discrete", 128, _cat_wide(4)), ("discrete", 129, _cat_wide(8)), ("discrete", 200, _cat_wide(8)),
    ("discrete", 256, _cat_wide(8)), ("discrete", 257, _cat_wide(16)), ("discrete", 512, _cat_wide(16)),
    ("discrete", 513, _cat_wide(32)), ("discrete", 1024, _cat_wide(32)),
    ("tuple", [1], _tup(8)), ("tuple", [3, 5], _tup(8)), ("tuple", [4, 5], _tup(16)), ("tuple", [7, 9], _tup(16)),
    ("tuple", [10, 7], _tup(32)), ("tuple", [20, 12], _tup(32)),
    ("tuple", [20, 13], _tup_wide(2)), ("tuple", [5, 5, 5, 5, 5, 5, 5, 29], _tup_wide(2)),
    ("tuple", [30, 34], _tup_wide(2)), ("tuple", [40, 25], _tup_wide(4)), ("tuple", [100, 28], _tup_wide(4)),
    ("tuple", [60, 69], _tup_wide(8)), ("tuple", [200, 56], _tup_wide(8)), ("tuple", [31, 226], _tup_wide(16)),
    ("tuple", [300, 212], _tup_wide(16)), ("tuple", [500, 13], _tup_wide(32)), ("tuple", [8, 16, 8, 992], _tup_wide(32)),
] + [
    ("gauss", (ad, adaptive), kern) for adaptive in (True, False) for ad, kern in [
        (1, _gauss(8)), (8, _gauss(8)), (9, _gauss(16)), (16, _gauss(16)), (17, _gauss(32)), (32, _gauss(32)),
        (33, _gauss_wide(2)), (64, _gauss_wide(2)), (65, _gauss_wide(4)), (100, _gauss_wide(4)),
        (128, _gauss_wide(4)), (129, _gauss_wide(8)), (256, _gauss_wide(8)), (257, _gauss_wide(16)),
        (512, _gauss_wide(16)), (513, _gauss_wide(32)), (1024, _gauss_wide(32))]
] + [
    ("mixed", [("box", 1)], _mixed(1)), ("mixed", [("discrete", 3), ("box", 2), ("discrete", 4)], _mixed(1)),
    ("mixed", [("box", 16)], _mixed(1)), ("mixed", [("discrete", 1), ("box", 16)], _mixed(2)),
    ("mixed", [("box", 32)], _mixed(2)), ("mixed", [("discrete", 5), ("box", 30)], _mixed(4)),
    ("mixed", [("box", 20), ("discrete", 40), ("box", 22)], _mixed(4)),
    ("mixed", [("box", 50), ("discrete", 29)], _mixed(8)), ("mixed", [("box", 100), ("discrete", 56)], _mixed(8)),
    ("mixed", [("discrete", 1), ("box", 128)], _mixed(16)),
    ("mixed", [("discrete", 200), ("box", 100), ("discrete", 112)], _mixed(16)),
    ("mixed", [("box", 256), ("discrete", 1)], _mixed(32)),
    ("mixed", [("box", 500), ("discrete", 24)], _mixed(32)),
]

# heads_tail_wide (slot map S = 1): (space, layout, mode, instantiation); the bucket is the widest member's width
TAIL_CASES = [
    ("discrete", 1, "plain", 2), ("discrete", 8, "mask", 2), ("discrete", 32, "deterministic", 2),
    ("discrete", 33, "plain", 2), ("discrete", 64, "mask", 2), ("discrete", 65, "plain", 4),
    ("discrete", 128, "deterministic", 4), ("discrete", 129, "mask", 8), ("discrete", 256, "plain", 8),
    ("discrete", 257, "plain", 16), ("discrete", 512, "mask", 16), ("discrete", 513, "deterministic", 32),
    ("discrete", 1024, "mask", 32),
    ("tuple", [20, 13], "plain", 2), ("tuple", [40, 25], "plain", 4), ("tuple", [60, 69], "deterministic", 8),
    ("tuple", [31, 226], "plain", 16), ("tuple", [500, 13], "plain", 32),
    ("gauss", (1, True), "plain", 2), ("gauss", (33, True), "deterministic", 2), ("gauss", (65, True), "plain", 4),
    ("gauss", (129, True), "plain", 8), ("gauss", (257, True), "deterministic", 16), ("gauss", (512, True), "plain", 16),
    ("gauss", (32, False), "plain", 2), ("gauss", (64, False), "deterministic", 2), ("gauss", (128, False), "plain", 4),
    ("gauss", (256, False), "plain", 8), ("gauss", (512, False), "plain", 16), ("gauss", (513, False), "plain", 32),
    ("gauss", (1024, False), "deterministic", 32),
]
TAIL_CASES = [(s, lay, mode, (f"heads_tail_rows_kernel<{lpl}, 1>",)) for s, lay, mode, lpl in TAIL_CASES]

# heads_tail_wide_mixed (slot map S = 0, bucket by row width): the mixed loss layouts
MIXED_TAIL_CASES = [(lay, (f"heads_tail_rows_kernel<{k[0][len('ppo_loss_mixed_kernel<'):-1]}, 0>",))
                    for s, lay, k in LOSS_CASES if s == "mixed"]

# narrow heads_forward: (rows, H, ldh, A, mode, instantiation); VEC needs H % 4 == 0 and 16-byte aligned rows
FORWARD_CASES = [
    (300, 64, 64, 1, "plain", "<9, 2, true>"), (300, 64, 64, 8, "mask", "<9, 2, true>"),
    (8192, 64, 64, 5, "deterministic", "<9, 2, true>"), (8193, 64, 64, 8, "plain", "<9, 4, true>"),
    (300, 50, 50, 8, "plain", "<9, 4, false>"), (9000, 64, 65, 7, "mask", "<9, 4, false>"),
    (300, 64, 64, 9, "plain", "<17, 2, true>"), (301, 128, 128, 16, "deterministic", "<17, 2, true>"),
    (300, 50, 50, 12, "mask", "<17, 2, false>"), (300, 96, 97, 16, "plain", "<17, 2, false>"),
    (300, 64, 64, 17, "plain", "<32, 1, true>"), (300, 64, 64, 31, "mask", "<32, 1, true>"),
    (300, 50, 50, 24, "plain", "<32, 1, false>"), (300, 64, 65, 31, "deterministic", "<32, 1, false>"),
]
FORWARD_CASES = [c[:5] + ((f"heads_forward_kernel{c[5]}",),) for c in FORWARD_CASES]

# heads_backward: (rows, H, A, activation, instantiation).  16384+ rows with H / 2 dividing 256 take two columns per
# thread (the pipelined kernel when a 32-row tile is a multiple of its 8-deep queue, H >= 128), fewer rows four.
BACKWARD_CASES = [
    (300, 64, 8, "elu", "heads_backward_vec_kernel<9, 4, 4, 2>"),
    (16383, 64, 1, "tanh", "heads_backward_vec_kernel<9, 4, 4, 2>"),
    (16411, 64, 8, "relu", "heads_backward_vec_kernel<9, 2, 8, 4>"),
    (16411, 128, 8, "none", "heads_backward_pipe_kernel<8, 3, 0>"),
    (16411, 128, 5, "elu", "heads_backward_pipe_kernel<8, 3, 1>"),
    (16411, 256, 8, "relu", "heads_backward_pipe_kernel<8, 3, 2>"),
    (16411, 128, 2, "tanh", "heads_backward_pipe_kernel<8, 3, 3>"),
    (300, 96, 8, "relu", "heads_backward_kernel<9>"), (300, 50, 3, "none", "heads_backward_kernel<9>"),
    (300, 64, 9, "tanh", "heads_backward_kernel<17>"), (300, 50, 16, "elu", "heads_backward_kernel<17>"),
    (16411, 64, 12, "relu", "heads_backward_kernel<17>"),
    (300, 64, 17, "elu", "heads_backward_kernel<32>"), (300, 50, 31, "tanh", "heads_backward_kernel<32>"),
]
BACKWARD_CASES = [c[:4] + ((c[4],),) for c in BACKWARD_CASES]

# the persistent rollout kernel <ACT, F16> (ACT 1 ELU, 2 ReLU, 3 tanh; F16 the fp16-split operand form): the tests of
# tests/test_gpu_rollout_pipeline.py that launch it, and assert the form it took
ROLLOUT_CASES = {
    "rollout_mlp2_tape_kernel<1, true>": "test_gpu_rollout_pipeline.py::test_bench_shape_fp16_form",
    "rollout_mlp2_tape_kernel<1, false>": "test_gpu_rollout_pipeline.py::test_bench_shape_tf32_form",
    "rollout_mlp2_tape_kernel<2, true>": "test_gpu_rollout_pipeline.py::test_activations[relu-fp16]",
    "rollout_mlp2_tape_kernel<2, false>": "test_gpu_rollout_pipeline.py::test_activations[relu-tf32]",
    "rollout_mlp2_tape_kernel<3, true>": "test_gpu_rollout_pipeline.py::test_activations[tanh-fp16]",
    "rollout_mlp2_tape_kernel<3, false>": "test_gpu_rollout_pipeline.py::test_activations[tanh-tf32]",
}

# compiled but reached by no model
ALLOWLIST = {
    "rollout_mlp2_tape_kernel<0, true>": "ACT none: a model always has an activation; only the C ABI can ask for it",
    "rollout_mlp2_tape_kernel<0, false>": "ACT none: a model always has an activation; only the C ABI can ask for it",
}


def _expected():
    out = set()
    for cases in (LOSS_CASES, TAIL_CASES, MIXED_TAIL_CASES, FORWARD_CASES, BACKWARD_CASES):
        for c in cases:
            out.update(c[-1])
    return out


def _lid(layout):
    if isinstance(layout, int):
        return str(layout)
    if isinstance(layout, tuple):
        return f"{layout[0]}{'' if layout[1] else '-learned'}"
    return "+".join(str(x) if isinstance(x, int) else f"{x[0][0]}{x[1]}" for x in layout)


# ----------------------------------------------------------------------------------------------- the table is complete
def _compiled_kernels():
    names = []
    for log in ("loss", "heads", "heads_wide", "rollout_fused"):
        path = os.path.join(BUILD, f"{log}.ptxas.log")
        assert os.path.isfile(path), f"{path} missing: build the library first (__graft_entry__.build())"
        names += re.findall(r"Function properties for (\S+)", open(path).read())
    demangled = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True,
                               check=True).stdout.splitlines()
    return {m.group(1) for n in demangled for m in [re.match(r"void sfb::(\w+_kernel<[^<>]*>)\(", n)] if m}


def test_every_instantiation_has_a_case():
    compiled = _compiled_kernels()
    covered = _expected() | set(ROLLOUT_CASES) | set(ALLOWLIST)
    assert not compiled - covered, f"instantiations with no case in this table: {sorted(compiled - covered)}"
    assert not covered - compiled, f"cases name instantiations the build does not have: {sorted(covered - compiled)}"


# ----------------------------------------------------------------------------------------------- helpers
def _heads_of(space, layout):
    if space == "discrete":
        return [("discrete", layout)]
    if space == "tuple":
        return [("discrete", n) for n in layout]
    if space == "gauss":
        return [("box", layout[0])]
    return list(layout)


def _noise(heads, M, gen):
    return torch.cat([torch.empty(M, n).exponential_(generator=gen) if k == "discrete" else torch.randn(M, n, generator=gen)
                      for k, n in heads], 1)


# ----------------------------------------------------------------------------------------------- loss and ratio
B = 300                                  # not a multiple of 256 (thread per sample) nor of 32 (warp per sample)
CLIP, CLIP_V, C_ENT, C_KL, C_VAL = 0.1, 0.25, 0.01, 0.05, 0.5
TS = 1.5                                 # tanh_scale of a learned-stddev Box
R_LOW, R_HIGH = slice(0, 4), slice(4, 8)            # raw ratio e^-5 < 0.05 and e^5 > 20
V_EDGE = slice(8, 12)                    # v_old = 0, values = +-CLIP_V (at the clip) and +-2 CLIP_V (beyond)
SPREAD = slice(12, 16)                   # categorical logits x 100
SD_LOW, SD_HIGH = slice(16, 19), slice(19, 22)      # log-stddev -12 / +11: beyond the [1e-4, 1e4] clamp
ONE_VALID = 40


def _loss_inputs(space, layout, seed, valid):
    heads = _heads_of(space, layout)
    A = MO.rows_of(heads)
    learned = space == "gauss" and not layout[1]
    gen = g(seed)
    params = torch.randn(B, A, generator=gen) * 1.5
    z = None
    lo = 0
    for k, n in heads:
        if k == "discrete":
            params[SPREAD, lo:lo + n] *= 100.0
        else:
            params[:, lo + n:lo + 2 * n] *= 0.2
            params[SD_LOW, lo + n:lo + 2 * n] = -12.0
            params[SD_HIGH, lo + n:lo + 2 * n] = 11.0
        lo += n if k == "discrete" else 2 * n
    if learned:                          # [tanh-scaled means | one log-stddev vector], one dimension beyond the clamp
        Ad = layout[0]
        z = params[:, :Ad].clone()
        log_std = torch.randn(Ad, generator=gen) * 0.3
        log_std[0] = 11.0
        params = torch.cat([torch.tanh(z / TS) * TS, log_std.expand(B, Ad)], 1).contiguous()
    params_old = params + 0.1 * torch.randn(B, A, generator=gen)
    params_old[SD_LOW.start:SD_HIGH.stop] = params[SD_LOW.start:SD_HIGH.stop]   # actions near the means of those rows
    actions = MO.mixed_sample(heads, params_old, _noise(heads, B, gen))
    lp = MO.mixed_log_prob(heads, params.double(), actions.double())
    delta = 0.3 * torch.randn(B, generator=gen).double()
    # min(r A, clip(r) A) has a kink at the bounds of the clip window: keep every ratio exp(-delta) 1e-3 away from them,
    # so that the float32 log-prob cannot put a row on the other side than float64 does
    for bound in (1.0 + CLIP, 1.0 / (1.0 + CLIP)):
        delta[(torch.exp(-delta) / bound - 1.0).abs() < 1e-3] += 0.01
    delta[R_LOW], delta[R_HIGH] = 5.0, -5.0
    lp_old = (lp + delta).float()
    adv = torch.randn(B, generator=gen) * 2
    adv[R_LOW] = adv[R_HIGH] = torch.tensor([3.0, -3.0, 3.0, -3.0])   # both sides of min(r A, clip(r) A) at each bound
    v_old, targets = torch.randn(B, generator=gen), torch.randn(B, generator=gen)
    values = v_old + 0.3 * torch.randn(B, generator=gen)
    v_old[V_EDGE] = 0.0
    values[V_EDGE] = torch.tensor([CLIP_V, -CLIP_V, 2 * CLIP_V, -2 * CLIP_V])
    if valid == "mixed":
        valids = torch.rand(B, generator=gen) > 0.1
        valids[:SD_HIGH.stop] = True
        valids[SD_HIGH.stop:SD_HIGH.stop + 3] = False
    else:
        valids = torch.zeros(B, dtype=torch.bool)
        if valid == "one":
            valids[ONE_VALID] = True
    return dict(heads=heads, params=params, z=z, params_old=params_old, actions=actions, lp_old=lp_old, adv=adv,
                v_old=v_old, targets=targets, values=values, valids=valids)


def _loss_reference(space, layout, expl, d):
    """float64 autograd of the PPO loss (learner.py:431-486, 586-657) -> (stats, d params, d log_std or None, d values)"""
    heads, valids = d["heads"], d["valids"]
    learned = space == "gauss" and not layout[1]
    V = d["values"].double().requires_grad_()
    if learned:
        Ad = layout[0]
        Z = d["z"].double().requires_grad_()
        S = d["params"][:, Ad:].double().clone().requires_grad_()
        P = torch.cat([torch.tanh(Z / TS) * TS, S], 1)
        leaves = [Z, S]
    else:
        P = d["params"].double().requires_grad_()
        leaves = [P]
    lp = MO.mixed_log_prob(heads, P, d["actions"].double())
    kl = MO.mixed_kl(heads, P, d["params_old"].double())
    vf = valids.double()
    n = vf.sum()
    adv = d["adv"].double()
    if n >= 2:
        advn = (adv - adv[valids].mean()) / adv[valids].std().clamp_min(1e-7)
    else:   # one valid row: adv - mean = 0 over the 1e-7 floor of the stddev (torch.std of one sample is NaN)
        advn = torch.zeros_like(adv)
    ratio = torch.exp(lp - d["lp_old"].double()).clamp(0.05, 20.0)
    hi = 1.0 + CLIP
    pl = -(torch.min(ratio * advn, ratio.clamp(1.0 / hi, hi) * advn) * vf).sum() / n
    v_old, targets = d["v_old"].double(), d["targets"].double()
    vc = v_old + (V - v_old).clamp(-CLIP_V, CLIP_V)
    vl = C_VAL * (torch.max((V - targets) ** 2, (vc - targets) ** 2) * vf).sum() / n
    if expl == "entropy":
        el = -C_ENT * (MO.mixed_entropy(heads, P) * vf).sum() / n
    else:
        segs = torch.split(P, [nk for _, nk in heads], dim=1)
        skl = sum(O.cat_symmetric_kl_with_uniform_prior(s) for s in segs)
        el = C_ENT * torch.clamp((skl * vf).sum() / n, max=30.0)
    kll = C_KL * (kl * vf).sum() / n
    total = pl + vl + el + kll
    total.backward()
    r = ratio.detach()[valids]
    stats = dict(num_valid=n.item(), policy_loss=pl.item(), value_loss=vl.item(), exploration_loss=el.item(),
                 kl_loss=kll.item(), total_loss=total.item(), ratio_min=r.min().item(), ratio_max=r.max().item(),
                 kl_old_max=kl.detach()[valids].max().item())
    return stats, leaves[0].grad, (leaves[1].grad if learned else None), V.grad, ratio.detach(), lp.detach()


def _run_loss(space, layout, expl, valid, kernels):
    ops = ops_for()
    d = _loss_inputs(space, layout, seed=7 * len(_lid(layout)) + MO.rows_of(_heads_of(space, layout)), valid=valid)
    heads = d["heads"]
    A = MO.rows_of(heads)
    dd = {k: v.to(DEV) for k, v in d.items() if isinstance(v, torch.Tensor)}
    stats = torch.zeros(ops.LS_SIZE, dtype=torch.float64, device=DEV)
    ws = torch.empty(ops.loss_workspace_bytes(B) // 8 + 8, dtype=torch.float64, device=DEV)
    learned = space == "gauss" and not layout[1]
    dl = torch.full((B, A // 2 if learned else A), float("nan"), device=DEV)
    dls = torch.full((B, A // 2), float("nan"), device=DEV) if learned else None
    dv = torch.full((B,), float("nan"), device=DEV)
    ratio = torch.full((B,), float("nan"), device=DEV)
    common = (dd["lp_old"], dd["v_old"], dd["adv"], dd["targets"], dd["valids"], dd["params_old"], CLIP, CLIP_V, C_ENT)
    kinds, sizes = [0 if k == "discrete" else 1 for k, _ in heads], [n for _, n in heads]

    def run():
        ops.adv_stats(dd["adv"], dd["valids"], stats, None, ws)
        if space == "discrete":
            ops.ppo_loss_fwd_bwd(dd["params"], dd["values"], dd["actions"].view(-1), *common, C_VAL, C_KL, 1.0, dl, dv,
                                 stats, ws, exploration_loss=expl)
            ops.action_ratio(dd["params"], dd["actions"].view(-1), dd["lp_old"], ratio)
        elif space == "tuple":
            ops.ppo_loss_fwd_bwd_tuple(dd["params"], dd["values"], sizes, dd["actions"], *common, C_VAL, C_KL, 1.0, dl,
                                       dv, stats, ws, exploration_loss=expl)
            ops.action_ratio_tuple(dd["params"], sizes, dd["actions"], dd["lp_old"], ratio)
        elif space == "gauss":
            ops.ppo_loss_fwd_bwd_continuous(dd["params"], dd["values"], layout[1], 0.0 if layout[1] else TS,
                                            dd["actions"], *common, C_VAL, C_KL, 1.0, dl, dls, dv, stats, ws)
            ops.action_ratio_continuous(dd["params"], dd["actions"], dd["lp_old"], ratio)
        else:
            ops.ppo_loss_fwd_bwd_mixed(dd["params"], dd["values"], kinds, sizes, dd["actions"], *common, C_VAL, C_KL,
                                       1.0, dl, dv, stats, ws)
            ops.action_ratio_mixed(dd["params"], kinds, sizes, dd["actions"], dd["lp_old"], ratio)

    check_launched(run, kernels)
    s = {k: stats[i].item() for k, i in ops.LS.items() if i < ops.LS_SIZE}
    out = dict(dl=dl.cpu(), dls=None if dls is None else dls.cpu(), dv=dv.cpu(), ratio=ratio.cpu())
    return d, s, out


def _rtol(lp):
    """per row, of the ratio and of the gradients, whose policy terms carry the ratio's relative error: exp(lp - lp_old)
    turns the absolute rounding of the float32 log-prob into relative error, and that grows with |lp| (a sum over up to
    1024 elements): five float32 roundings of |lp|, at least 1e-5"""
    return np.maximum(1e-5, 5 * 2.0 ** -24 * lp.abs().numpy())


def _assert_close(got, want, rtol, atol):
    """assert_allclose, loosened to rtol 1e-3 on the rows with stddevs at the clamp: a log-stddev of -12 puts a 1e8 factor
    on (a - mean), and either clamp makes the log-prob a sum of |terms| ~ 10 per dimension, whose float32 rounding leaves
    ~1e-4 relative (test_gpu_mixed_tuple.test_mixed_loss_and_ratio_match_autograd)"""
    got, want = got.numpy(), want.numpy()
    rt = rtol.copy()
    rt[SD_LOW.start:SD_HIGH.stop] = np.maximum(rt[SD_LOW.start:SD_HIGH.stop], 1e-3)
    rt = rt.reshape((-1,) + (1,) * (got.ndim - 1))
    bad = np.abs(got - want) > atol + rt * np.abs(want)
    if bad.ndim > 1:
        bad = bad.any(axis=tuple(range(1, bad.ndim)))
    idx = np.flatnonzero(bad)
    assert idx.size == 0, (f"rows {idx[:10].tolist()} differ beyond rtol {rt.ravel()[idx[:3]]}: "
                           f"{got[idx[:3]]} vs {want[idx[:3]]}")


LOSS_PARAMS = [pytest.param(s, lay, k, e, id=f"{s}-{_lid(lay)}-{e}") for s, lay, k in LOSS_CASES
               for e in (("entropy", "symmetric_kl") if s in ("discrete", "tuple") else ("entropy",))]


@pytest.mark.gpu
@pytest.mark.parametrize("space,layout,kernels,expl", LOSS_PARAMS)
def test_loss_and_ratio(space, layout, kernels, expl):
    d, s, out = _run_loss(space, layout, expl, "mixed", kernels)
    want, g_p, g_s, g_v, ratio, lp = _loss_reference(space, layout, expl, d)
    valids = d["valids"]
    assert s["num_valid"] == want["num_valid"]
    for key in ("policy_loss", "value_loss", "exploration_loss", "kl_loss", "total_loss"):
        assert abs(s[key] - want[key]) < 1e-5 * max(1.0, abs(want[key])), (key, s[key], want[key])
    # the clamped rows are valid: the summaries hold the clamp bounds exactly
    assert s["ratio_min"] == float(np.float32(0.05)) and s["ratio_max"] == 20.0, (s["ratio_min"], s["ratio_max"])
    assert abs(s["kl_old_max"] - want["kl_old_max"]) < 1e-4 * max(1.0, abs(want["kl_old_max"]))
    rtol = _rtol(lp)
    _assert_close(out["dl"], g_p, rtol, 1e-5)
    if g_s is not None:
        _assert_close(out["dls"], g_s, rtol, 1e-5)
    np.testing.assert_allclose(out["dv"].numpy(), g_v.numpy(), rtol=1e-5, atol=1e-5)
    for t in (out["dl"], out["dv"]) + ((out["dls"],) if g_s is not None else ()):
        assert torch.all(t[~valids] == 0), "an invalid row got a gradient"
    # no gradient through the outer ratio clamp: rows with a raw ratio outside [0.05, 20] keep only the exploration and
    # KL terms, which the reference holds
    assert torch.all(out["ratio"][R_LOW] == float(np.float32(0.05))) and torch.all(out["ratio"][R_HIGH] == 20.0)
    _assert_close(out["ratio"], ratio, rtol, 1e-6)


# one instantiation per kernel family, narrow and wide
WHOLE_BATCH = [c for c in LOSS_CASES if (c[0], _lid(c[1])) in {
    ("discrete", "8"), ("discrete", "200"), ("tuple", "4+5"), ("tuple", "40+25"), ("gauss", "9"), ("gauss", "65-learned"),
    ("mixed", "d3+b2+d4"), ("mixed", "d5+b30")}]


@pytest.mark.gpu
@pytest.mark.parametrize("space,layout,kernels", [pytest.param(*c, id=f"{c[0]}-{_lid(c[1])}") for c in WHOLE_BATCH])
def test_loss_no_valid_row(space, layout, kernels):
    """An all-invalid minibatch: every loss 0, every gradient exactly 0; the extrema keep the identities of an empty
    min / max (+inf, -inf), which the data-parallel reduction of the summaries (dist_utils) combines correctly"""
    d, s, out = _run_loss(space, layout, "entropy", "none", kernels)
    assert s["num_valid"] == 0 and s["adv_mean"] == 0 and s["adv_std"] == 0
    for key in ("policy_loss", "value_loss", "exploration_loss", "kl_loss", "total_loss", "kl_old_mean",
                "entropy_mean", "ratio_mean_abs_dev", "fraction_clipped"):
        assert s[key] == 0, (key, s[key])
    assert s["ratio_min"] == math.inf and s["ratio_max"] == -math.inf and s["kl_old_max"] == -math.inf
    for t in (out["dl"], out["dv"]) + ((out["dls"],) if out["dls"] is not None else ()):
        assert torch.all(t == 0)


@pytest.mark.gpu
@pytest.mark.parametrize("space,layout,kernels", [pytest.param(*c, id=f"{c[0]}-{_lid(c[1])}") for c in WHOLE_BATCH])
def test_loss_single_valid_row(space, layout, kernels):
    """One valid row: torch.std of one advantage is NaN, which would poison the weights.  The kernels keep a finite
    result: adv_std 0 (clamped to 1e-7), normalised advantage 0, so the policy gradient is 0 while the value, exploration
    and KL terms match torch"""
    d, s, out = _run_loss(space, layout, "entropy", "one", kernels)
    want, g_p, g_s, g_v, _, _ = _loss_reference(space, layout, "entropy", d)
    assert s["num_valid"] == 1 and s["adv_mean"] == d["adv"][ONE_VALID].item() and s["adv_std"] == 0
    assert all(math.isfinite(s[k]) for k in ("policy_loss", "value_loss", "exploration_loss", "kl_loss", "total_loss"))
    assert s["policy_loss"] == 0
    for key in ("value_loss", "exploration_loss", "kl_loss", "total_loss"):
        assert abs(s[key] - want[key]) < 1e-5 * max(1.0, abs(want[key])), (key, s[key], want[key])
    r = out["ratio"][ONE_VALID].item()
    assert s["ratio_min"] == r and s["ratio_max"] == r
    others = torch.ones(B, dtype=torch.bool)
    others[ONE_VALID] = False
    for got, ref in ((out["dl"], g_p), (out["dv"], g_v)) + (((out["dls"], g_s),) if g_s is not None else ()):
        assert torch.all(torch.isfinite(got)) and torch.all(got[others] == 0)
        np.testing.assert_allclose(got.numpy(), ref.numpy(), rtol=1e-5, atol=1e-6)


# ----------------------------------------------------------------------------------------------- heads tails
@pytest.mark.gpu
@pytest.mark.parametrize("space,layout,mode,kernels", [pytest.param(*c, id=f"{c[0]}-{_lid(c[1])}-{c[2]}")
                                                       for c in TAIL_CASES])
def test_heads_tail_wide(space, layout, mode, kernels):
    """sfb200_heads_tail_wide over stored rows: values against float64, actions bit-exact against the oracle's sampling
    of the same rows (Box actions up to the rounding of expf), log-probs against the oracle"""
    ops = ops_for()
    M, H = 300, 96
    gen = g(11 + len(_lid(layout)))
    h = torch.randn(M, H, generator=gen)
    Wv, bv = torch.randn(1, H, generator=gen) * 0.1, torch.randn(1, generator=gen)
    det = mode == "deterministic"
    if space == "gauss":
        ad, adaptive = layout
        A = 2 * ad if adaptive else ad
        raw = torch.randn(M, 2 * ad, generator=gen)
        raw[:, ad:] *= 0.3
        learned = torch.randn(ad, generator=gen) * 0.3
        eps = torch.randn(M, ad, generator=gen)
        params = raw.clone().to(DEV)
        kw = dict(noise=eps.to(DEV), deterministic=det, continuous=True, act_dim=ad, adaptive_stddev=adaptive,
                  learned_log_std=None if adaptive else learned.to(DEV), tanh_scale=0.0 if adaptive else TS)
        res = []
        check_launched(lambda: res.append(wide_tail(ops, h.to(DEV), Wv.to(DEV), bv.to(DEV), params, A, **kw)), kernels)
        v, act, lp, env = res[0]
        means = raw[:, :ad] if adaptive else torch.tanh(raw[:, :ad] / TS) * TS
        log_std = raw[:, ad:] if adaptive else learned.expand(M, ad)
        np.testing.assert_allclose(params.cpu()[:, :ad].numpy(), means.numpy(), atol=1e-6)
        np.testing.assert_allclose(params.cpu()[:, ad:].numpy(), log_std.numpy(), atol=0)
        sd = log_std.exp().clamp(1e-4, 1e4)
        want_a = (torch.zeros_like(eps) if det else eps) * sd + means
        if det:
            assert torch.equal(act, params.cpu()[:, :ad]), "deterministic Gaussian actions are the means"
        np.testing.assert_allclose(act.numpy(), want_a.numpy(), atol=1e-5)
        assert torch.equal(env, act)
        want_lp = O.gauss_log_prob(params.cpu().double(), act.double())
        np.testing.assert_allclose(lp.numpy(), want_lp.numpy(), atol=1e-4, rtol=1e-5)
    else:
        segs = [layout] if space == "discrete" else layout
        A = sum(segs)
        logits = torch.randn(M, A, generator=gen) * 2
        logits[::17] *= 100.0                               # probabilities exactly 0
        q = torch.empty(M, A).exponential_(generator=gen)
        mask = masked_rows(M, A, 5) if mode == "mask" else None
        ld = logits.clone().to(DEV)
        kw = dict(noise=q.to(DEV), mask=None if mask is None else mask.to(DEV), deterministic=det)
        if space == "tuple":
            kw["head_sizes"] = segs
        res = []
        check_launched(lambda: res.append(wide_tail(ops, h.to(DEV), Wv.to(DEV), bv.to(DEV), ld, A, **kw)), kernels)
        v, act, lp, env = res[0]
        assert torch.equal(ld.cpu(), logits)
        qq = torch.ones_like(q) if det else q
        want_lp, start = torch.zeros(M, dtype=torch.float64), 0
        for k, n in enumerate(segs):
            seg = logits[:, start:start + n]
            if mask is None:
                a = O.cat_sample(seg, qq[:, start:start + n]).view(-1)
                want_lp += O.cat_log_prob(seg.double(), a)
            else:   # (in float32: a row that allows nothing keeps the rounding of its -1e9 shift)
                a = O.masked_cat_sample(seg, mask, qq).view(-1)
                want_lp += O.masked_cat_log_prob(seg, mask, a).double()
            assert torch.equal(act[:, k].long(), a) and torch.equal(env[:, k].long(), a), f"head {k}: actions differ"
            start += n
        np.testing.assert_allclose(lp.numpy(), want_lp.numpy(), rtol=1e-6, atol=1e-5)
    np.testing.assert_allclose(v.numpy(), (h.double() @ Wv.double().view(-1) + bv.double()).numpy(), atol=1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("layout,kernels", [pytest.param(*c, id=_lid(c[0])) for c in MIXED_TAIL_CASES])
@pytest.mark.parametrize("deterministic", [False, True])
def test_heads_tail_wide_mixed(layout, kernels, deterministic):
    ops = ops_for()
    heads = list(layout)
    A, W = MO.rows_of(heads), MO.width_of(heads)
    M, H = 300, 64
    gen = g(23 + A)
    h = torch.randn(M, H, generator=gen)
    Wv, bv = torch.randn(1, H, generator=gen) * 0.1, torch.randn(1, generator=gen)
    params = torch.randn(M, A, generator=gen) * 1.5
    lo = 0
    for k, n in heads:
        if k == "box":
            params[:, lo + n:lo + 2 * n] *= 0.3
        else:
            params[::17, lo:lo + n] *= 100.0
        lo += n if k == "discrete" else 2 * n
    noise = _noise(heads, M, gen)
    pd = params.clone().to(DEV)
    values = torch.full((M,), float("nan"), device=DEV)
    actions = torch.full((M, W), float("nan"), device=DEV)
    lp = torch.full((M,), float("nan"), device=DEV)
    pv_out = torch.full((M,), float("nan"), device=DEV)
    env = [torch.full((M,), -7, dtype=torch.int32, device=DEV) if k == "discrete" else
           torch.full((M, n), float("nan"), device=DEV) for k, n in heads]
    kinds, sizes = [0 if k == "discrete" else 1 for k, _ in heads], [n for _, n in heads]

    def run():
        ops.heads_tail_wide_mixed(h.to(DEV), Wv.to(DEV), bv.to(DEV), pd, A, A, kinds, sizes, values, 1,
                                  noise=noise.to(DEV), actions_f32=actions, actions_stride=W, env_actions=env,
                                  log_prob=lp, log_prob_stride=1, policy_version_scalar=torch.full((1,), 4.0, device=DEV),
                                  policy_version_out=pv_out, pv_stride=1)

    if deterministic:
        ops.set_sampling_mode(None, True)
    try:
        check_launched(run, kernels)
    finally:
        ops.set_sampling_mode(None, False)
    assert torch.equal(pd.cpu(), params)
    np.testing.assert_allclose(values.cpu().numpy(), (h.double() @ Wv.double().view(-1) + bv.double()).numpy(), atol=1e-5)
    got = actions.cpu()
    want = MO.mixed_sample(heads, params, noise, deterministic=deterministic)
    dcols, c = [], 0
    for k, n in heads:
        if k == "discrete":
            dcols.append(c)
        c += 1 if k == "discrete" else n
    assert torch.equal(got[:, dcols], want[:, dcols]), "categorical member actions must be bit-exact"
    if deterministic:
        assert torch.equal(got, want)
    np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(lp.cpu().numpy(), MO.mixed_log_prob(heads, params.double(), got.double()).numpy(),
                               rtol=1e-5, atol=1e-4)
    for e, w in zip(env, MO.env_actions(heads, got)):
        assert torch.equal(e.cpu(), w)
    assert torch.all(pv_out == 4.0)


# ----------------------------------------------------------------------------------------------- narrow heads
@pytest.mark.gpu
@pytest.mark.parametrize("rows,H,ldh,A,mode,kernels", [pytest.param(*c, id=f"{c[0]}x{c[1]}-ld{c[2]}-A{c[3]}-{c[4]}")
                                                       for c in FORWARD_CASES])
def test_heads_forward(rows, H, ldh, A, mode, kernels):
    """sfb200_heads_forward: values and logits against float64, actions bit-exact against the oracle's sampling of the
    kernel's logits (ldh > H: rows that are not 16-byte aligned)"""
    ops = ops_for()
    gen = g(rows + H + A)
    base = torch.randn(rows, ldh, generator=gen)
    h = base[:, ldh - H:]
    Wv, bv = torch.randn(1, H, generator=gen) / math.sqrt(H), torch.randn(1, generator=gen)
    Wa, ba = torch.randn(A, H, generator=gen) / math.sqrt(H) * 2, torch.randn(A, generator=gen) * 0.1
    noise = torch.empty(rows, A).exponential_(generator=gen)
    mask = torch.rand(rows, A, generator=gen) < 0.5
    mask[::13] = False
    mask[1::13] = True
    hd = base.to(DEV)[:, ldh - H:]
    values, logits = torch.empty(rows, device=DEV), torch.empty(rows, A, device=DEV)
    actions, lp = torch.empty(rows, device=DEV), torch.empty(rows, device=DEV)
    env = torch.empty(rows, dtype=torch.int32, device=DEV)

    def run():
        ops.heads_forward(hd, Wv.to(DEV), bv.to(DEV), Wa.to(DEV), ba.to(DEV), values, 1, logits, A,
                          None if mode == "deterministic" else noise.to(DEV), actions_f32=actions, actions_stride=1,
                          env_actions=env, log_prob=lp, log_prob_stride=1)

    mask_dev = mask.to(DEV)              # (the sampling mode keeps a pointer to it)
    ops.set_sampling_mode(mask_dev if mode == "mask" else None, mode == "deterministic")
    try:
        check_launched(run, kernels)
    finally:
        ops.set_sampling_mode(None, False)
    hh = h.double()
    np.testing.assert_allclose(values.cpu().numpy(), (hh @ Wv.double().view(-1) + bv.double()).numpy(), atol=1e-5)
    np.testing.assert_allclose(logits.cpu().numpy(), (hh @ Wa.double().t() + ba.double()).numpy(), atol=1e-5)
    dl = logits.cpu()
    if mode == "plain":
        a = O.cat_sample(dl, noise)
        want_lp = O.cat_log_prob(dl.double(), a)
    elif mode == "mask":
        m64 = mask.to(torch.int64)
        a = O.masked_cat_sample(dl, m64, noise)
        want_lp = O.masked_cat_log_prob(dl, m64, a)     # (float32: see test_heads_tail_wide)
    else:
        a = torch.argmax(O.cat_probs(dl), -1)
        want_lp = O.cat_log_probs(dl.double()).max(-1).values
    assert torch.equal(env.cpu().long(), a.view(-1)), "action indices must be bit-exact"
    assert torch.equal(actions.cpu(), a.view(-1).float())
    np.testing.assert_allclose(lp.cpu().numpy(), want_lp.numpy(), atol=2e-6, rtol=1e-6)


@pytest.mark.gpu
@pytest.mark.parametrize("rows,H,A,act,kernels", [pytest.param(*c, id=f"{c[0]}x{c[1]}-A{c[2]}-{c[3]}")
                                                  for c in BACKWARD_CASES])
def test_heads_backward(rows, H, A, act, kernels):
    ops = ops_for()
    gen = g(rows + H + A)
    pre = torch.randn(rows, H, generator=gen)
    fn = {"elu": torch.nn.functional.elu, "relu": torch.relu, "tanh": torch.tanh, "none": lambda t: t}[act]
    h = fn(pre)
    Wv = torch.randn(1, H, generator=gen) / math.sqrt(H)
    Wa = torch.randn(A, H, generator=gen) / math.sqrt(H)
    dlogits = torch.randn(rows, A, generator=gen) / rows
    dvalues = torch.randn(rows, generator=gen) / rows
    P = pre.double().requires_grad_()
    out = (fn(P) @ Wa.double().t() * dlogits.double()).sum() + (fn(P) @ Wv.double().view(-1) * dvalues.double()).sum()
    out.backward()
    dz_ref = P.grad
    dz, dWv, dbv = torch.empty(rows, H, device=DEV), torch.empty(H, device=DEV), torch.empty(1, device=DEV)
    dWa, dba, dbp = torch.empty(A, H, device=DEV), torch.empty(A, device=DEV), torch.empty(H, device=DEV)
    ws = torch.empty(ops.heads_backward_workspace_bytes(H, A) // 4 + 4, device=DEV)
    args = (h.to(DEV), Wv.to(DEV).view(-1), Wa.to(DEV), dlogits.to(DEV), dvalues.to(DEV), ops.ACT[act], dz, dWv, dbv,
            dWa, dba, dbp, ws)
    check_launched(lambda: ops.heads_backward(*args), kernels)
    tol = dict(atol=1e-5, rtol=1e-4)          # test_gpu_kernels.test_heads_backward
    np.testing.assert_allclose(dz.cpu().numpy(), dz_ref.numpy(), **tol)
    np.testing.assert_allclose(dWa.cpu().numpy(), (dlogits.double().t() @ h.double()).numpy(), **tol)
    np.testing.assert_allclose(dWv.cpu().numpy(), (dvalues.double() @ h.double()).numpy(), **tol)
    np.testing.assert_allclose(dba.cpu().numpy(), dlogits.double().sum(0).numpy(), **tol)
    np.testing.assert_allclose(dbv.cpu().numpy(), dvalues.double().sum().view(1).numpy(), **tol)
    np.testing.assert_allclose(dbp.cpu().numpy(), dz_ref.sum(0).numpy(), **tol)
