"""The fused policy / value heads on Box and Tuple action spaces against float64.

The last MLP layer's wgmma GEMM (linear_act_heads_forward) leaves per-row partial dot products of the heads; a finishing
step adds the biases and runs the distribution tail -- the separate heads_from_partials* launch, or the GEMM itself
(linear_act_heads_forward_fused, dist_kind 0 / 1 / 2).  HeadsPlan takes this path whenever the tail is 128 / 256 / 384 /
512 wide and value + A <= 9: every Box(<= 4) with adaptive stddev, every Box(<= 8) with a learned stddev and every Tuple of
Discretes with <= 8 logits, in the sampler and in the learner.

Kernel level: on the kernel's own last-layer activations y (the GEMM has its own tests), values and params rows within
1e-5 of sum_k |y_k w_k| + |b| of the float64 products (the rule of test_gpu_heads_f16.py), and the sampled actions and
log-probs against a float64 restatement of the distributions -- pinned once against oracle/appo_oracle.py below -- within
bounds derived from that params error.  Categorical indices must match wherever the float64 margin between the top two
p/q exceeds what the logit error can move; near-ties are counted and printed.  The separate and the in-GEMM finish agree
bit for bit, storing y or not changes nothing, the Philox draws are a function of (seed, offset), and the shapes just
outside the fused path get no partials (so a routing change cannot silently test the unfused kernels instead).

Model level: Box(4) adaptive, Box(8) learned with tanh scaling and Tuple(Discrete(3), Discrete(5)) sampled and trained
closed-loop next to the CPU oracle on the fused path, and again with the heads finished inside the GEMM."""
import math
from dataclasses import dataclass
from typing import Optional, Tuple

import numpy as np
import pytest
import torch

from oracle import appo_oracle as O
from tests.device_harness import DEV, TOL, Registered, build, g, masked_rows, model_spec, need, ops_for

pytestmark = pytest.mark.gpu

EPS32 = 2.0 ** -23                      # one ulp of 1.0f
LOG_SQRT_2PI = 0.5 * math.log(2 * math.pi)
K_IN = 192                              # the last layer's input width (the partials only depend on the output width)


# ------------------------------------------------------------------------------------------------------ action spaces
@dataclass(frozen=True)
class Space:
    kind: str                           # "box", "tuple" or "discrete"
    n: int = 0                          # Box: act_dim; Discrete: number of actions
    adaptive: bool = True
    tanh_scale: float = 0.0
    segs: Tuple[int, ...] = ()
    mask: bool = False                  # Discrete: an action mask (set_sampling_mode)
    det: bool = False                   # deterministic sampling (set_sampling_mode)

    @property
    def A(self):                        # rows of distribution_linear
        if self.kind == "box":
            return 2 * self.n if self.adaptive else self.n
        return sum(self.segs) if self.kind == "tuple" else self.n

    @property
    def width(self):                    # floats per action row
        return self.n if self.kind == "box" else (len(self.segs) if self.kind == "tuple" else 1)

    @property
    def params(self):                   # floats per params row
        return 2 * self.n if self.kind == "box" else self.A

    @property
    def segments(self):
        return list(self.segs) if self.kind == "tuple" else [self.n]

    def __str__(self):
        if self.kind == "box":
            s = f"box{self.n}_" + ("adaptive" if self.adaptive else f"learned_ts{self.tanh_scale:g}")
        elif self.kind == "tuple":
            s = "tuple" + "_".join(map(str, self.segs))
        else:
            s = f"discrete{self.n}" + ("_masked" if self.mask else "")
        return s + ("_det" if self.det else "")


SPACES = [Space("box", 1), Space("box", 3), Space("box", 4),
          Space("box", 1, adaptive=False), Space("box", 8, adaptive=False),
          Space("box", 1, adaptive=False, tanh_scale=1.5), Space("box", 8, adaptive=False, tanh_scale=1.5),
          Space("tuple", segs=(1,)), Space("tuple", segs=(2, 3)), Space("tuple", segs=(3, 5)), Space("tuple", segs=(8,)),
          Space("tuple", segs=(1,) * 8),
          Space("discrete", 6, mask=True), Space("discrete", 8, det=True), Space("box", 3, det=True),
          Space("tuple", segs=(3, 5), det=True)]
WIDTHS = [128, 256, 384, 512]
ROWS = [1, 127, 129, 4133]
ACTS = ["elu", "relu", "tanh"]
SCALES = [1.0, 1e-6, 300.0]


@dataclass(frozen=True)
class Case:
    sp: Space
    N: int
    M: int
    act: str
    scale: float
    edge: bool = False                  # logits x100 / log-stddevs of +-12 / extreme explicit noise
    philox: bool = False                # noise=None: the Philox draws
    strided: bool = True                # outputs through trajectory slices traj[:, t]

    def __str__(self):
        return (f"{self.sp}-N{self.N}-M{self.M}-{self.act}-x{self.scale:g}" + ("-edge" if self.edge else "") +
                ("-philox" if self.philox else "") + ("" if self.strided else "-dense"))


def _cases():
    """every space at three (width, rows, activation, input scale) points that rotate through all four tables, then the
    edge rows, the Philox draws and M = 32768"""
    out = []
    for i, sp in enumerate(SPACES):
        for j in range(3):
            M = ROWS[(i + 2 * j) % 4]
            if sp.mask and M < 2:
                M = 2
            out.append(Case(sp, WIDTHS[(i + j) % 4], M, ACTS[(i + j) % 3], SCALES[(i + 2 * j) % 3], strided=(i + j) % 2 == 0))
    for sp, N in [(Space("box", 4), 512), (Space("box", 3), 128), (Space("box", 8, adaptive=False, tanh_scale=1.5), 256),
                  (Space("box", 1, adaptive=False), 384), (Space("tuple", segs=(3, 5)), 256), (Space("tuple", segs=(8,)), 128),
                  (Space("tuple", segs=(1,) * 8), 512), (Space("discrete", 6, mask=True), 384)]:
        out.append(Case(sp, N, 4133, "relu", 1.0, edge=True))
    for sp, N in [(Space("box", 4), 256), (Space("box", 8, adaptive=False, tanh_scale=1.5), 512),
                  (Space("tuple", segs=(2, 3)), 384), (Space("discrete", 6, mask=True), 128)]:
        out.append(Case(sp, N, 129, "elu", 1.0, philox=True))
    for sp, N, act in [(Space("box", 4), 512, "elu"), (Space("box", 8, adaptive=False, tanh_scale=1.5), 256, "tanh"),
                       (Space("tuple", segs=(3, 5)), 512, "relu")]:
        out.append(Case(sp, N, 32768, act, 1.0))
    return out


CASES = _cases()


# ------------------------------------------------------------------------------ the distributions, restated in float64
def cat_ref(z: torch.Tensor, q: Optional[torch.Tensor], mask: Optional[torch.Tensor] = None):
    """CategoricalActionDistribution of float64 logits z [M, n]: (log_softmax [M, n], sampled index [M], log of the
    margin between the two largest p/q [M]).  q: Exp(1) draws (torch.multinomial(p, 1) == argmax(p / q), first index on
    ties), or ones for the deterministic argmax of p.  mask (bool [M, n]): masked_softmax / masked_log_softmax -- a
    forbidden logit gets -1e9 added in fp32 (so a row that allows nothing keeps only the fp32 rounding of z - 1e9), p is
    renormalised over the allowed actions (+1e-13), and a row left with all p == 0 falls back to 1e-6 everywhere"""
    x = z
    if mask is not None:
        x = torch.where(mask, z, (z.float() + torch.tensor(-1e9, dtype=torch.float32)).double())
    logp = torch.log_softmax(x, dim=1)
    if q is None:
        return logp, None, None
    p = torch.softmax(x, dim=1)
    if mask is not None:
        p = p * mask
        p = p / (p.sum(1, keepdim=True) + 1e-13)
        p = torch.where((p == 0).all(1, keepdim=True), torch.full_like(p, 1e-6), p)
    lr = torch.log(p) - torch.log(q)
    idx = torch.argmax(lr, dim=1)
    if z.shape[1] == 1:
        return logp, idx, torch.full_like(lr[:, 0], math.inf)
    top = torch.topk(lr, 2, dim=1).values
    return logp, idx, top[:, 0] - top[:, 1]


def gauss_ref(mean: torch.Tensor, log_std: torch.Tensor, eps: torch.Tensor):
    """ContinuousActionDistribution: sd = clamp(exp(log_std), 1e-4, 1e4), the draw eps * sd + mean"""
    sd = torch.clamp(torch.exp(log_std), O.STDDEV_MIN, O.STDDEV_MAX)
    return sd, eps * sd + mean


def gauss_log_prob_ref(a: torch.Tensor, mean: torch.Tensor, sd: torch.Tensor):
    """Independent(Normal(mean, sd), 1).log_prob(a)"""
    return (-(a - mean) ** 2 / (2 * sd ** 2) - torch.log(sd) - LOG_SQRT_2PI).sum(1)


def learned_means_ref(z: torch.Tensor, tanh_scale: float):
    """ActionParameterizationContinuousNonAdaptiveStddev: tanh(z / ts) * ts when ts > 0"""
    return torch.tanh(z / tanh_scale) * tanh_scale if tanh_scale > 0 else z


def test_float64_restatement_matches_oracle():
    """the float64 restatement above against the oracle's distribution functions (pinned to the reference by the goldens)
    on fp32 inputs: the same indices, log-probs within 1e-5, Gaussian draws within a few ulp"""
    gen = g(5)
    M, n = 4096, 7
    z = torch.randn(M, n, generator=gen) * 3
    q = torch.empty(M, n).exponential_(generator=gen)
    logp, idx, margin = cat_ref(z.double(), q.double())
    assert torch.equal(O.cat_sample(z, q).view(-1)[margin > 1e-5], idx[margin > 1e-5])
    np.testing.assert_allclose(O.cat_log_prob(z, idx).numpy(), logp.gather(1, idx.view(-1, 1)).view(-1).numpy(), atol=1e-5)
    _, idx1, _ = cat_ref(z.double(), torch.ones(M, n, dtype=torch.float64))
    assert torch.equal(O.cat_sample(z, torch.ones(M, n)).view(-1), idx1)
    mask = masked_rows(M, n, 6)
    logp, idx, margin = cat_ref(z.double(), q.double(), mask)
    assert torch.equal(O.masked_cat_sample(z, mask, q).view(-1)[margin > 1e-5], idx[margin > 1e-5])
    assert idx[0] == torch.argmin(q[0]) and idx[1] == n - 1            # allows nothing; allows only the last action
    np.testing.assert_allclose(O.masked_cat_log_prob(z, mask, idx).numpy(),
                               logp.gather(1, idx.view(-1, 1)).view(-1).numpy(), atol=1e-5)
    cfg = O.OracleCfg(num_actions=8, action_segments=[3, 5])
    zt = torch.randn(M, 8, generator=gen)
    qt = torch.empty(M, 8).exponential_(generator=gen)
    acts = O.tuple_sample(cfg, zt, qt)
    lp_ref = torch.zeros(M, dtype=torch.float64)
    for k, (o, m) in enumerate([(0, 3), (3, 5)]):
        lpk, ik, mk = cat_ref(zt[:, o:o + m].double(), qt[:, o:o + m].double())
        assert torch.equal(acts[:, k][mk > 1e-5], ik[mk > 1e-5])
        lp_ref += lpk.gather(1, acts[:, k].view(-1, 1)).view(-1)
    np.testing.assert_allclose(O.tuple_log_prob(cfg, zt, acts).numpy(), lp_ref.numpy(), atol=1e-5)
    params = torch.cat([torch.randn(M, 4, generator=gen), torch.randn(M, 4, generator=gen) * 6], 1)   # some clamped
    eps = torch.randn(M, 4, generator=gen)
    a32 = O.gauss_sample(params, eps)
    sd, a = gauss_ref(params[:, :4].double(), params[:, 4:].double(), eps.double())
    assert torch.all((a32.double() - a).abs() <= 4 * EPS32 * ((eps.double() * sd).abs() + a.abs()))
    np.testing.assert_allclose(O.gauss_log_prob(params, a32).numpy(),
                               gauss_log_prob_ref(a32.double(), params[:, :4].double(), sd).numpy(), rtol=1e-6, atol=1e-5)
    for ts in (0.0, 1.5):
        ocfg = O.OracleCfg(obs_dim=8, num_actions=3, continuous=True, adaptive_stddev=False, continuous_tanh_scale=ts,
                           encoder_mlp_layers=[16], initial_stddev=0.3)
        st = O.init_state(ocfg, seed=2)
        h = torch.randn(9, 16, generator=gen) * 3
        _, prm = O.tail_forward(ocfg, st, h)
        zz = h.double() @ st[O.ACTION_W].double().T + st[O.ACTION_B].double()
        np.testing.assert_allclose(prm[:, :3].numpy(), learned_means_ref(zz, ts).numpy(), atol=1e-6)
        assert torch.equal(prm[:, 3:], st[O.LEARNED_STD].view(1, 3).expand(9, 3))


# ---------------------------------------------------------------------------------------------------- kernel level
def _inputs(c: Case, seed: int):
    sp, N, M = c.sp, c.N, c.M
    gen = g(seed)
    x = torch.randn(M, K_IN, generator=gen) * c.scale
    W = torch.randn(N, K_IN, generator=gen) / math.sqrt(K_IN)
    b = torch.randn(N, generator=gen) * 0.1 * c.scale
    Wv = torch.randn(1, N, generator=gen) / math.sqrt(N)
    bv = torch.randn(1, generator=gen)
    Wa = torch.randn(sp.A, N, generator=gen) / math.sqrt(N)
    ba = torch.randn(sp.A, generator=gen) * 0.1
    lls = torch.randn(sp.n, generator=gen) * 0.5 if sp.kind == "box" and not sp.adaptive else None
    if c.edge:
        if sp.kind != "box":                         # logits spread x100: probabilities exactly 0 in fp32
            Wa, ba = Wa * 100, ba * 100
        elif sp.adaptive:                            # log-stddevs around +-12, beyond the clamp on both sides
            Wa[sp.n:] *= 0.01
            ba[sp.n:] = torch.tensor([12.0, -12.0]).repeat(sp.n)[:sp.n]
        else:
            lls = torch.tensor([12.0, -12.0, 0.5]).repeat(sp.n)[:sp.n]
    noise = None
    if not c.philox and not sp.det:
        if sp.kind == "box":
            noise = torch.randn(M, sp.n, generator=gen) * (4.0 if c.edge else 1.0)
        else:
            noise = torch.empty(M, sp.A).exponential_(generator=gen)
            if c.edge:                               # Exp(1) tails: draws of 1e-20 and of 60
                noise[::7] *= 1e-20
                noise[3::11] += 60.0
    mask = masked_rows(M, sp.n, seed) if sp.mask else None
    dev = lambda t: None if t is None else t.to(DEV).contiguous()
    return tuple(map(dev, (x, W, b, Wv, bv, Wa, ba, lls, noise, mask)))


def _outputs(sp: Space, M: int, strided: bool):
    """the output slots, as slices traj[:, t] of trajectory-shaped buffers (strides != row width) or dense"""
    T, t = (3, 1) if strided else (0, 0)

    def slot(*tail, extra=0):
        if not strided:
            return torch.full((M,) + tail, float("nan"), device=DEV)
        return torch.full((M, T + extra) + tail, float("nan"), device=DEV)[:, t]

    env = (torch.full((M, sp.n), float("nan"), device=DEV) if sp.kind == "box" else
           torch.full((M, sp.width) if sp.kind == "tuple" else (M,), -1, dtype=torch.int32, device=DEV))
    return dict(values=slot(extra=1), params=slot(sp.params), actions=slot(sp.width), log_prob=slot(), pv=slot(), env=env)


def _kw(o, noise, seed, pv):
    return dict(values=o["values"], values_stride=o["values"].stride(0), logits=o["params"],
                logits_stride=o["params"].stride(0), noise=noise, philox_seed=seed, philox_offset=3,
                actions_f32=o["actions"], actions_stride=o["actions"].stride(0), env_actions=o["env"], log_prob=o["log_prob"],
                log_prob_stride=o["log_prob"].stride(0), policy_version_scalar=pv, policy_version_out=o["pv"],
                pv_stride=o["pv"].stride(0))


def _finish(ops, sp, part, P, M, bv, ba, lls, kw):
    """the separate finishing launch of the space"""
    if sp.kind == "box":
        ops.heads_from_partials_continuous(part, P, M, bv, ba, sp.n, sp.adaptive, lls, sp.tanh_scale, **kw)
    elif sp.kind == "tuple":
        ops.heads_from_partials_tuple(part, P, M, bv, ba, list(sp.segs), **kw)
    else:
        ops.heads_from_partials(part, P, M, bv, ba, **kw)


def _fused(ops, sp, x, W, b, y, act, Wv, bv, Wa, ba, part, counters, lls, kw):
    """the heads finished inside the GEMM (last-arriving CTA of every 128-row block)"""
    ops.linear_act_heads_forward_fused(x, W, b, y, act, ops.GEMM_TC_3XTF32, Wv, bv, Wa, ba, part, counters, **kw,
                                       head_sizes=list(sp.segs) if sp.kind == "tuple" else None,
                                       act_dim=sp.n if sp.kind == "box" else 0, adaptive_stddev=sp.adaptive,
                                       learned_log_std=lls, tanh_scale=sp.tanh_scale, continuous=sp.kind == "box")


def _sampling(ops, sp, mask, fn):
    if sp.mask or sp.det:
        ops.set_sampling_mode(mask, sp.det)
    try:
        fn()
    finally:
        ops.set_sampling_mode(None, False)


def _cpu(o):
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in o.items()}


def _assert_same(a, b, what):
    for k in a:
        assert torch.equal(a[k], b[k]), f"{what}: {k}"


@pytest.mark.parametrize("c", CASES, ids=str)
def test_fused_heads_vs_float64(c: Case):
    ops = ops_for("3xtf32")
    sp, N, M = c.sp, c.N, c.M
    P = ops.linear_heads_partials(N, sp.A, ops.GEMM_TC_3XTF32)
    assert P == 2 * (N // 128), f"{c}: the fused heads path must cover this shape"
    seed = 1000 + 37 * CASES.index(c)
    x, W, b, Wv, bv, Wa, ba, lls, noise, mask = _inputs(c, seed)
    pv = torch.full((1,), 7.0, device=DEV)
    act = ops.ACT[c.act]
    with Registered(W, x=x):
        y = torch.full((M, N), float("nan"), device=DEV)
        part = torch.full((P * M * ops.HEAD_PART_PAD,), float("nan"), device=DEV)
        ops.linear_act_heads_forward(x, W, b, y, act, ops.GEMM_TC_3XTF32, Wv, Wa, part)
        part_ns = torch.full_like(part, float("nan"))
        ops.linear_act_heads_forward(x, W, b, None, act, ops.GEMM_TC_3XTF32, Wv, Wa, part_ns)
        runs = []
        for pt in (part, part_ns, part):             # storing y or not; the same launch twice (Philox: same draws)
            o = _outputs(sp, M, c.strided)
            _sampling(ops, sp, mask, lambda: _finish(ops, sp, pt, P, M, bv, ba, lls, _kw(o, noise, seed, pv)))
            runs.append(_cpu(o))
        counters = torch.zeros((M + 127) // 128, dtype=torch.int32, device=DEV)
        for rep in range(2):                         # twice: the arrival counters are left at zero
            o = _outputs(sp, M, c.strided)
            y4 = torch.full((M, N), float("nan"), device=DEV) if rep == 0 else None
            p4 = torch.full_like(part, float("nan"))
            _sampling(ops, sp, mask, lambda: _fused(ops, sp, x, W, b, y4, act, Wv, bv, Wa, ba, p4, counters, lls,
                                                    _kw(o, noise, seed, pv)))
            runs.append(_cpu(o))
            assert torch.all(counters == 0), rep
            if rep == 0:
                assert torch.equal(y4, y)
        torch.cuda.synchronize()
    assert torch.equal(part, part_ns)
    for i, what in [(1, "y not stored"), (2, "second launch"), (3, "in-GEMM finish"), (4, "in-GEMM finish, y not stored")]:
        _assert_same(runs[0], runs[i], what)
    _check_float64(c, y, Wv, bv, Wa, ba, lls, noise, mask, runs[0])


def _check_float64(c: Case, y, Wv, bv, Wa, ba, lls, noise, mask, o):
    """the outputs `o` of one finishing launch against the float64 heads on the kernel's y"""
    sp, M = c.sp, c.M
    Wh = torch.cat([Wv.view(1, -1), Wa]).double()
    bh = torch.cat([bv.view(1), ba]).double()
    yd = y.double()
    z = (yd @ Wh.T + bh).cpu()
    err = (1e-5 * (yd.abs() @ Wh.abs().T + bh.abs())).cpu()      # the partials' error rule, with the bias
    assert torch.all(o["pv"] == 7.0)
    dv = (o["values"].double() - z[:, 0]).abs()
    assert torch.all(dv <= err[:, 0]), f"values: max excess {(dv - err[:, 0]).max().item():.3g}"
    params = o["params"].double()
    acts = o["actions"].double()
    lp = o["log_prob"].double()
    q = None if noise is None else noise.double().cpu()
    if sp.kind == "box":
        Ad = sp.n
        zm, em = z[:, 1:1 + Ad], err[:, 1:1 + Ad]
        if sp.adaptive:
            mean, e_mean = zm, em
            log_std, e_ls = z[:, 1 + Ad:], err[:, 1 + Ad:]
        else:
            mean = learned_means_ref(zm, sp.tanh_scale)
            # tanh is 1-Lipschitz: the z error passes through, plus the rounding of tanhf, the division and the product
            e_mean = em + (4 * EPS32 * (mean.abs() + sp.tanh_scale) if sp.tanh_scale > 0 else 0.0)
            log_std, e_ls = lls.double().cpu().view(1, Ad).expand(M, Ad), torch.zeros(M, Ad, dtype=torch.float64)
        d_mean = (params[:, :Ad] - mean).abs()
        assert torch.all(d_mean <= e_mean), f"means: max excess {(d_mean - e_mean).max().item():.3g}"
        d_ls = (params[:, Ad:] - log_std).abs()
        assert torch.all(d_ls <= e_ls), f"log-stddevs: max excess {(d_ls - e_ls).max().item():.3g}"
        assert torch.equal(o["env"], o["actions"])
        # sd = clamp(exp(log_std)) moves by at most a relative expm1(e_ls) (the clamp only contracts), plus expf's and
        # the clamp's rounding (4 ulp)
        e_sd_rel = torch.expm1(e_ls) + 4 * EPS32
        sd, _ = gauss_ref(mean, log_std, torch.zeros_like(mean))
        if sp.det or q is not None:
            eps = torch.zeros_like(mean) if sp.det else q
            _, a_ref = gauss_ref(mean, log_std, eps)
            # a = eps * sd + mean: the mean's error, |eps| sd times sd's relative error, and the rounding of the product
            # and of the sum (an ulp of |eps sd| and of |a| each, doubled)
            e_a = e_mean + (eps.abs() * sd) * e_sd_rel + 2 * EPS32 * (eps.abs() * sd + a_ref.abs())
            d_a = (acts - a_ref).abs()
            assert torch.all(d_a <= e_a), f"actions: max excess {(d_a - e_a).max().item():.3g}"
        # log N(a; mean, sd) at the kernel's own action a, d = a - mean, r = |d| / sd:
        #   d^2 / (2 sd^2) moves by r / sd * (the mean's error + the rounding of a - mean) and by r^2 * sd's relative
        #   error; log sd by the log-stddev's error; the terms round to 4 ulp each, the sum over dimensions to Ad ulp of
        #   the sum of their magnitudes.  (1.01: the second-order terms.)
        d = acts - mean
        r = d.abs() / sd
        terms = r ** 2 / 2 + torch.log(sd).abs() + LOG_SQRT_2PI
        e_lp = (1.01 * (r / sd * (e_mean + EPS32 * d.abs()) + r ** 2 * e_sd_rel + e_ls) + 4 * EPS32 * terms).sum(1) \
            + Ad * EPS32 * terms.sum(1)
        lp_ref = gauss_log_prob_ref(acts, mean, sd)
        d_lp = (lp - lp_ref).abs()
        assert torch.all(d_lp <= e_lp), f"log-probs: max excess {(d_lp - e_lp).max().item():.3g}"
        print(f"{c}: max |err| / bound: means {(d_mean / e_mean.clamp_min(1e-300)).max().item():.3g}, "
              f"log-probs {(d_lp / e_lp).max().item():.3g}")
        return
    # Discrete / Tuple of Discretes: the logits, then per segment the index and its log-prob
    d_z = (params - z[:, 1:]).abs()
    assert torch.all(d_z <= err[:, 1:]), f"logits: max excess {(d_z - err[:, 1:]).max().item():.3g}"
    env = o["env"].view(M, -1)
    assert torch.equal(env.double(), acts.view(M, -1))
    lp_ref = torch.zeros(M, dtype=torch.float64)
    e_lp = torch.zeros(M, dtype=torch.float64)
    near = flips = 0
    off = 0
    for k, n in enumerate(sp.segments):
        zs, es = z[:, 1 + off:1 + off + n], err[:, 1 + off:1 + off + n]
        qs = torch.ones(M, n, dtype=torch.float64) if sp.det else (None if q is None else q[:, off:off + n])
        logp, idx_ref, margin = cat_ref(zs, qs, mask.cpu() if mask is not None else None)
        idx = acts.view(M, -1)[:, k].long()
        assert torch.all((idx >= 0) & (idx < n)), k
        if mask is not None:                         # (whatever the draws) an allowed action wherever there is one
            mk = mask.cpu()
            assert torch.all(mk.gather(1, idx.view(-1, 1)).view(-1) | ~mk.any(1))
        emax = es.max(1).values
        if idx_ref is not None:
            # the logits' errors move log(p_i / q_i) - log(p_j / q_j) by at most e_i + e_j (the softmax denominator is
            # shared); expf, the sum and the two divisions round by n + 6 ulp more
            tie = margin <= 2 * emax + (n + 6) * EPS32
            wrong = idx != idx_ref
            assert not torch.any(wrong & ~tie), \
                f"segment {k}: rows {torch.nonzero(wrong & ~tie).view(-1)[:8].tolist()} sample a different index"
            near += int(tie.sum())
            flips += int(wrong.sum())
        # log_softmax at the chosen index: its logit's error, twice the largest (max and log-sum-exp), rounding
        lpk = logp.gather(1, idx.view(-1, 1)).view(-1)
        lp_ref += lpk
        e_lp += es.gather(1, idx.view(-1, 1)).view(-1) + 2 * emax + 8 * EPS32 * (lpk.abs() + 1) + n * EPS32
        off += n
    d_lp = (lp - lp_ref).abs()
    assert torch.all(d_lp <= e_lp), f"log-probs: max excess {(d_lp - e_lp).max().item():.3g}"
    print(f"{c}: {near} near-tie rows, {flips} indices differ from float64; max |err| / bound: logits "
          f"{(d_z / err[:, 1:]).max().item():.3g}, log-probs {(d_lp / e_lp).max().item():.3g}")
    assert flips <= 4, f"{flips} near-tie flips"


OUTSIDE = {"box5_adaptive": (Space("box", 5), 256), "box9_learned": (Space("box", 9, adaptive=False), 256),
           "tuple3_2_4": (Space("tuple", segs=(3, 2, 4)), 256), "discrete8_N64": (Space("discrete", 8), 64),
           "discrete8_N640": (Space("discrete", 8), 640)}


@pytest.mark.parametrize("name", list(OUTSIDE))
def test_just_outside_the_fused_path(name):
    """the shapes next to the covered ones get no partials, in the library and in the model's HeadsPlan"""
    from sample_factory_b200.model import PolicyModel
    from sample_factory_b200.policy import HeadsPlan

    ops = ops_for("3xtf32")
    sp, N = OUTSIDE[name]
    assert ops.linear_heads_partials(N, sp.A, ops.GEMM_TC_3XTF32) == 0
    ocfg = _ocfg(sp, [N, N], obs_dim=16)
    plan = HeadsPlan(PolicyModel(model_spec(ocfg), DEV), ops.GEMM_TC_3XTF32, 64)
    assert plan.P == 0
    inside = dict(box5_adaptive=Space("box", 4), box9_learned=Space("box", 8, adaptive=False),
                  tuple3_2_4=Space("tuple", segs=(3, 5)), discrete8_N64=None, discrete8_N640=None)[name]
    if inside is not None:                           # and their neighbours inside do
        assert HeadsPlan(PolicyModel(model_spec(_ocfg(inside, [N, N], obs_dim=16)), DEV), ops.GEMM_TC_3XTF32, 64).P > 0


def _ocfg(sp: Space, layers, **kw):
    over = dict(num_actions=sp.A if sp.kind != "box" else sp.n, encoder_mlp_layers=list(layers))
    if sp.kind == "box":
        over.update(continuous=True, adaptive_stddev=sp.adaptive, continuous_tanh_scale=sp.tanh_scale)
    elif sp.kind == "tuple":
        over.update(action_segments=list(sp.segs))
    over.update(kw)
    return O.OracleCfg(**over)


# ----------------------------------------------------------------------------------------------------- model level
MODELS = {
    "box4_adaptive": (Space("box", 4), [256, 256], {}),
    "box8_learned_ts1.5_bootstrap": (Space("box", 8, adaptive=False, tanh_scale=1.5), [512, 512],
                                     dict(value_bootstrap=True, initial_stddev=0.7)),
    "tuple3_5": (Space("tuple", segs=(3, 5)), [256, 256], {}),
}


@pytest.mark.parametrize("name,in_gemm", [("box4_adaptive", False), ("box8_learned_ts1.5_bootstrap", False),
                                          ("tuple3_5", False), ("box4_adaptive", True), ("tuple3_5", True)])
def test_fused_heads_closed_loop_vs_oracle(name, in_gemm, monkeypatch):
    """sampler + learner on the fused heads path next to the oracle: N = 1000 envs (not a multiple of 128), T = 8, two
    iterations on the same tape, noise and initial weights.  in_gemm: a second rig whose plans finish the heads inside
    the GEMM writes the same trajectories and trains to the same weights"""
    from sample_factory_b200 import ops

    need("3xtf32")
    sp, layers, kw = MODELS[name]
    N, T, iters = 1000, 8, 2
    ocfg = _ocfg(sp, layers, obs_dim=24, rollout=T, recurrence=1, batch_size=N * T // 2, num_batches_per_epoch=2, **kw)
    st0 = O.init_state(ocfg, seed=11)
    gen = g(29)
    tape = torch.randn(iters * T + 1, N, ocfg.obs_dim, generator=gen) * 1.2 - 0.2
    monkeypatch.delenv("SFB200_HEADS_FINISH_IN_GEMM", raising=False)
    cfg, model, traj, env, sampler, learner = build(ocfg, N, st0, tape, "3xtf32")
    assert sampler.heads_plan.P > 0 and learner.heads_plan.P > 0
    assert not sampler.heads_plan.finish_in_gemm and not learner.heads_plan.finish_in_gemm
    twin = None
    if in_gemm:
        with monkeypatch.context() as mp:
            mp.setenv("SFB200_HEADS_FINISH_IN_GEMM", "1")
            twin = build(ocfg, N, st0, tape, "3xtf32")
        assert twin.sampler.heads_plan.finish_in_gemm and twin.learner.heads_plan.finish_in_gemm
        twin.sampler.reset()
    olearner = O.OracleLearner(ocfg, st0)
    oenv = O.TapeVecEnv(tape, ocfg.num_actions)
    olast = oenv.reset()
    sampler.reset()
    A = ocfg.num_actions
    for it in range(iters):
        noise = torch.randn(T, N, A, generator=gen) if ocfg.continuous else torch.empty(T, N, A).exponential_(generator=gen)
        otraj = O.alloc_trajectories(ocfg, N)
        olast = O.rollout(ocfg, olearner.st, oenv, olast, otraj, noise, olearner.train_step)
        for rig in [(sampler, learner)] + ([(twin.sampler, twin.learner)] if twin else []):
            rig[0].noise = noise.to(DEV)
            rig[0].set_policy_version(rig[1].train_step)
            rig[0].rollout()
        got = {k: v.cpu() for k, v in traj.items()}
        if twin:
            for k in traj:
                assert torch.equal(traj[k], twin.traj[k]), f"iteration {it}: the in-GEMM finish wrote different {k}"
        # ---- rollout
        assert torch.equal(got["obs"].view(otraj["obs"].shape), otraj["obs"])
        for k in ["dones", "time_outs", "policy_id", "policy_version"]:
            assert torch.equal(got[k], otraj[k]), k
        np.testing.assert_allclose(got["action_logits"].numpy(), otraj["action_logits"].numpy(), atol=TOL)
        np.testing.assert_allclose(got["values"][:, :-1].numpy(), otraj["values"][:, :-1].numpy(), atol=TOL)
        if ocfg.continuous:
            # a = eps * sd + mean: the means at 1e-5, and sd = exp(log_std) off by the relative 1e-5 of the log-stddevs
            # the params carry, times |eps sd| (measured: 7.2e-5 at |eps sd| ~ 20, 3.6e-6 relative, with adaptive stddev)
            eps_sd = (otraj["actions"] - otraj["action_logits"][..., :A]).abs()
            d_a = (got["actions"] - otraj["actions"]).abs()
            assert torch.all(d_a <= TOL * (1 + eps_sd)), f"actions: max |diff| {d_a.max().item():.3g}"
            np.testing.assert_allclose(got["rewards"].numpy(), otraj["rewards"].numpy(), atol=TOL)
            np.testing.assert_allclose(got["log_prob_actions"].numpy(), otraj["log_prob_actions"].numpy(), atol=TOL)
        else:
            flips = (got["actions"].view(otraj["actions"].shape) != otraj["actions"]).any(-1)
            n_flip = int(flips.sum())
            print(f"[{name}] iteration {it}: {n_flip} near-tie action flips of {flips.numel()} steps")
            assert n_flip <= 4, f"{n_flip} of {flips.numel()} action rows differ from the oracle"
            same = ~flips
            assert torch.equal(got["rewards"][same], otraj["rewards"][same])
            np.testing.assert_allclose(got["log_prob_actions"][same].numpy(), otraj["log_prob_actions"][same].numpy(),
                                       atol=TOL)
        # ---- learner on the oracle's trajectories
        for k, v in otraj.items():
            if k in traj:
                traj[k].copy_(v.view(traj[k].shape))
                if twin:
                    twin.traj[k].copy_(v.view(traj[k].shape))
        n0 = len(olearner.log)
        buff = olearner.train(otraj)
        learner.train(traj)
        if twin:
            twin.learner.train(twin.traj)
        torch.cuda.synchronize()
        np.testing.assert_allclose(learner.returns.view(-1).cpu().numpy(), buff["returns"].numpy(), atol=TOL)
        np.testing.assert_allclose(learner.advantages.view(-1).cpu().numpy(), buff["advantages"].numpy(), atol=TOL)
        log = learner.minibatch_log().numpy()
        assert log.shape[0] == len(olearner.log) - n0
        for j, d in enumerate(olearner.log[n0:]):
            for key in ["policy_loss", "value_loss", "exploration_loss", "kl_loss"]:
                assert abs(log[j, ops.LS[key]] - d[key]) < TOL, (name, it, j, key, log[j, ops.LS[key]], d[key])
        for k in O.param_names(ocfg):
            off, shp = model._slices[k]
            m_dev = model.exp_avg[off: off + int(np.prod(shp))].view(shp).cpu().numpy()
            np.testing.assert_allclose(m_dev, olearner.m[k].numpy(), atol=2e-6, err_msg=f"{name} exp_avg {k}")
        if twin:
            assert torch.equal(learner.minibatch_log(), twin.learner.minibatch_log()), it
            assert torch.equal(model.flat, twin.model.flat), it
            assert torch.equal(model.exp_avg, twin.model.exp_avg), it
        # both loops continue from the oracle's weights (the differences stay at rounding level anyway)
        model.load_state_dict({k: v.clone() for k, v in olearner.st.items()}, strict=False)
        if twin:
            twin.model.load_state_dict({k: v.clone() for k, v in olearner.st.items()}, strict=False)
