"""Heads wider than 31 distribution_linear rows (ModelSpec.wide_heads): sfb200_heads_tail_wide against torch and against
the narrow heads kernel, the wide loss / ratio kernels and the wide heads backward against autograd, the reference-generated
wide fixtures on both engines, CUDA-graph replay, and a 1024-env closed loop on Discrete(362) with action masks."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import appo_oracle as O
from tests.device_harness import (DEV, ENGINES, TOL, build, build_case, g, graphed_learner_matches_eager,
                                  graphed_sampler_matches_eager, masked_rows, need, ops_for, replay_learner, replay_sampler,
                                  sampled_feed, wide_tail)
from tests.golden_utils import load_case

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("A", [32, 33, 45, 96, 362, 1024])
@pytest.mark.parametrize("mode", ["plain", "mask", "deterministic"])
def test_categorical_tail_matches_torch(A, mode):
    ops = ops_for()
    M, H = 300, 96
    h = torch.randn(M, H, generator=g(A))
    Wv, bv = torch.randn(1, H, generator=g(1)) * 0.1, torch.randn(1, generator=g(2))
    logits = torch.randn(M, A, generator=g(3)) * 2
    q = torch.empty(M, A).exponential_(generator=g(4))
    mask = masked_rows(M, A, 5) if mode == "mask" else None
    ld = logits.clone().to(DEV)
    v, act, lp, env = wide_tail(ops, h.to(DEV), Wv.to(DEV), bv.to(DEV), ld, A, noise=q.to(DEV),
                            mask=None if mask is None else mask.to(DEV), deterministic=mode == "deterministic")
    assert torch.equal(ld.cpu(), logits)      # the stored logits stay the raw logits
    np.testing.assert_allclose(v.numpy(), (h.double() @ Wv.double().view(-1) + bv.double()).numpy(), atol=1e-5)
    qq = torch.ones_like(q) if mode == "deterministic" else q
    if mask is None:
        ref_a = O.cat_sample(logits, qq)
        ref_lp = O.cat_log_prob(logits, ref_a)
    else:
        ref_a = O.masked_cat_sample(logits, mask, qq)
        ref_lp = O.masked_cat_log_prob(logits, mask, ref_a)
        allowed = mask.any(1)
        assert torch.all(mask[allowed].gather(1, act[allowed].long()).view(-1)), "a masked action was drawn"
    assert torch.equal(act.view(-1).long(), ref_a.view(-1).long()), "actions must be bit-exact"
    assert torch.equal(env.view(-1).long(), ref_a.view(-1).long())
    np.testing.assert_allclose(lp.numpy(), ref_lp.view(-1).numpy(), atol=1e-5)


@pytest.mark.parametrize("segs", [[24, 5, 16], [300, 62], [8, 16, 8, 992]])
def test_tuple_tail_matches_torch(segs):
    ops = ops_for()
    A = sum(segs)
    M, H = 200, 64
    h = torch.randn(M, H, generator=g(1))
    Wv, bv = torch.randn(1, H, generator=g(2)) * 0.1, torch.randn(1, generator=g(3))
    logits = torch.randn(M, A, generator=g(4)) * 2
    q = torch.empty(M, A).exponential_(generator=g(5))
    v, act, lp, env = wide_tail(ops, h.to(DEV), Wv.to(DEV), bv.to(DEV), logits.clone().to(DEV), A, noise=q.to(DEV),
                            head_sizes=segs)
    start, ref_lp = 0, torch.zeros(M)
    for k, n in enumerate(segs):
        a = O.cat_sample(logits[:, start:start + n], q[:, start:start + n]).view(-1)
        assert torch.equal(act[:, k].long(), a.long()) and torch.equal(env[:, k].long(), a.long()), k
        ref_lp += O.cat_log_prob(logits[:, start:start + n], a).view(-1)
        start += n
    np.testing.assert_allclose(lp.numpy(), ref_lp.numpy(), atol=1e-5)


@pytest.mark.parametrize("act_dim,adaptive", [(16, True), (17, True), (40, True), (512, True), (32, False), (36, False),
                                              (1024, False)])
@pytest.mark.parametrize("deterministic", [False, True])
def test_gaussian_tail_matches_torch(act_dim, adaptive, deterministic):
    ops = ops_for()
    M, H = 128, 64
    h = torch.randn(M, H, generator=g(1))
    Wv, bv = torch.randn(1, H, generator=g(2)) * 0.1, torch.randn(1, generator=g(3))
    raw = torch.randn(M, 2 * act_dim, generator=g(4))
    learned = torch.randn(act_dim, generator=g(5)) * 0.3
    ts = 0.0 if adaptive else 1.5
    eps = torch.randn(M, act_dim, generator=g(6))
    params = raw.clone().to(DEV)
    A = 2 * act_dim if adaptive else act_dim
    v, act, lp, env = wide_tail(ops, h.to(DEV), Wv.to(DEV), bv.to(DEV), params, A, noise=eps.to(DEV),
                            deterministic=deterministic, continuous=True, act_dim=act_dim, adaptive_stddev=adaptive,
                            learned_log_std=None if adaptive else learned.to(DEV), tanh_scale=ts)
    means = raw[:, :act_dim] if adaptive else torch.tanh(raw[:, :act_dim] / ts) * ts
    log_std = raw[:, act_dim:] if adaptive else learned.expand(M, act_dim)
    np.testing.assert_allclose(params.cpu()[:, :act_dim].numpy(), means.numpy(), atol=1e-6)
    np.testing.assert_allclose(params.cpu()[:, act_dim:].numpy(), log_std.numpy(), atol=0)
    sd = log_std.exp().clamp(1e-4, 1e4)
    e = torch.zeros_like(eps) if deterministic else eps
    ref_a = e * sd + means
    np.testing.assert_allclose(act.numpy(), ref_a.numpy(), atol=1e-5)
    np.testing.assert_allclose(env.numpy(), act.numpy(), atol=0)
    ref_lp = torch.distributions.Normal(means, sd).log_prob(act).sum(-1)
    np.testing.assert_allclose(lp.numpy(), ref_lp.numpy(), atol=1e-4, rtol=1e-5)
    np.testing.assert_allclose(v.numpy(), (h @ Wv.view(-1) + bv).numpy(), atol=1e-5)


@pytest.mark.parametrize("A", [8, 17, 31])
@pytest.mark.parametrize("masked", [False, True])
def test_wide_tail_matches_narrow_heads(A, masked):
    """Up to 31 logits the wide tail puts every logit on the lane the narrow tail uses: same action indices bit for bit"""
    ops = ops_for()
    M, H = 512, 64
    h = torch.randn(M, H, generator=g(A)).to(DEV)
    Wv, bv = (torch.randn(1, H, generator=g(1)) * 0.2).to(DEV), torch.randn(1, generator=g(2)).to(DEV)
    Wa, ba = (torch.randn(A, H, generator=g(3)) * 0.3).to(DEV), torch.randn(A, generator=g(4)).to(DEV)
    q = torch.empty(M, A).exponential_(generator=g(5)).to(DEV)
    mask = masked_rows(M, A, 6).to(DEV) if masked else None
    vals, logits = torch.empty(M, device=DEV), torch.empty(M, A, device=DEV)
    acts, lp = torch.empty(M, device=DEV), torch.empty(M, device=DEV)
    if mask is not None:
        ops.set_sampling_mode(mask, False)
    ops.heads_forward(h, Wv, bv, Wa, ba, vals, 1, logits, A, noise=q, actions_f32=acts, actions_stride=1, log_prob=lp,
                      log_prob_stride=1)
    ops.set_sampling_mode(None, False)
    v2, a2, lp2, _ = wide_tail(ops, h, Wv, bv, logits.clone(), A, noise=q, mask=mask)
    assert torch.equal(a2.view(-1), acts.cpu())
    np.testing.assert_allclose(v2.numpy(), vals.cpu().numpy(), atol=1e-6)
    np.testing.assert_allclose(lp2.numpy(), lp.cpu().numpy(), atol=1e-6)


def test_philox_sampling_distribution_a362():
    """Philox draws: action frequencies follow the (masked) softmax, and no masked action is ever drawn"""
    ops = ops_for()
    A, M, H = 362, 20000, 32
    row = torch.randn(A, generator=g(1)) * 1.5
    mask_row = torch.rand(A, generator=g(2)) > 0.3
    logits = row.expand(M, A).contiguous().to(DEV)
    mask = mask_row.expand(M, A).contiguous().to(DEV)
    h = torch.zeros(M, H, device=DEV)
    counts = torch.zeros(A)
    p = O.masked_cat_probs(row.view(1, -1), mask_row.view(1, -1)).view(-1)
    for rep in range(5):
        values = torch.empty(M, device=DEV)
        acts = torch.empty(M, device=DEV)
        ops.set_sampling_mode(mask, False)
        ops.heads_tail_wide(h, torch.zeros(1, H, device=DEV), torch.zeros(1, device=DEV), logits, A, A, values, 1,
                            philox_seed=123, philox_offset=rep, actions_f32=acts, actions_stride=1)
        ops.set_sampling_mode(None, False)
        a = acts.long().cpu()
        assert torch.all(mask_row[a]), "a masked action was drawn"
        counts += torch.bincount(a, minlength=A).float()
    n = counts.sum()
    expect = p * n
    big = expect > 50
    z = (counts[big] - expect[big]) / torch.sqrt(expect[big] * (1 - p[big]))
    assert z.abs().max() < 5.0, z.abs().max()
    tv = 0.5 * (counts / n - p).abs().sum()
    assert tv < 0.03, tv


# ----------------------------------------------------------------------------------------------- loss kernels
def _loss_inputs(B, seed):
    gen = g(seed)
    adv = torch.randn(B, generator=gen)
    valids = torch.rand(B, generator=gen) > 0.1
    v_old, targets = torch.randn(B, generator=gen), torch.randn(B, generator=gen)
    values = v_old + 0.3 * torch.randn(B, generator=gen)
    return adv, valids, v_old, targets, values


def _torch_ppo(lp, lp_old, ent, kl, values, v_old, targets, adv, valids, c_ent, c_kl, clip=0.1, clip_v=0.2, c_val=0.5):
    vf = valids.double()
    n = vf.sum()
    am, asd = adv[valids].double().mean(), adv[valids].double().std().clamp_min(1e-7)
    advn = (adv.double() - am) / asd
    ratio = torch.exp(lp - lp_old).clamp(0.05, 20.0)
    pl = -(torch.min(ratio * advn, ratio.clamp(1 / (1 + clip), 1 + clip) * advn) * vf).sum() / n
    vc = v_old + (values - v_old).clamp(-clip_v, clip_v)
    vl = c_val * (torch.max((values - targets) ** 2, (vc - targets) ** 2) * vf).sum() / n
    return pl + vl + c_ent * (ent * vf).sum() / n + c_kl * (kl * vf).sum() / n


@pytest.mark.parametrize("A", [33, 96, 362, 1024])
@pytest.mark.parametrize("expl", ["entropy", "symmetric_kl"])
def test_categorical_loss_and_ratio_match_autograd(A, expl):
    ops = ops_for()
    B = 600
    adv, valids, v_old, targets, values = _loss_inputs(B, A)
    logits = torch.randn(B, A, generator=g(1)) * 1.5
    logits_old = logits + 0.2 * torch.randn(B, A, generator=g(2))
    actions = torch.randint(0, A, (B,), generator=g(3)).float()
    lp_old = O.cat_log_prob(logits_old, actions.long()).view(-1) + 0.05 * torch.randn(B, generator=g(4))
    c_ent, c_kl = 0.01, 0.05
    L = logits.double().requires_grad_()
    V = values.double().requires_grad_()
    logp = torch.log_softmax(L, -1)
    p = logp.exp()
    lp = logp.gather(1, actions.long().view(-1, 1)).view(-1)
    if expl == "entropy":
        ent = (logp * p).sum(-1)                          # -entropy: the loss adds -c * entropy
    else:
        u = 1.0 / A
        ent = 0.5 * ((p * (logp - np.log(u))).sum(-1) + (u * (np.log(u) - logp)).sum(-1))
    kl = (p * (logp - torch.log_softmax(logits_old.double(), -1))).sum(-1)
    loss = _torch_ppo(lp, lp_old.double(), ent, kl, V, v_old.double(), targets.double(), adv, valids, c_ent, c_kl)
    loss.backward()
    stats = torch.zeros(ops.LS_SIZE, dtype=torch.float64, device=DEV)
    ws = torch.empty(ops.loss_workspace_bytes(B) // 8 + 8, dtype=torch.float64, device=DEV)
    vd = valids.to(DEV)
    ops.adv_stats(adv.to(DEV), vd, stats, None, ws)
    dl, dv = torch.empty(B, A, device=DEV), torch.empty(B, device=DEV)
    ops.ppo_loss_fwd_bwd(logits.to(DEV), values.to(DEV), actions.to(DEV), lp_old.to(DEV), v_old.to(DEV), adv.to(DEV),
                         targets.to(DEV), vd, logits_old.to(DEV), 0.1, 0.2, c_ent, 0.5, c_kl, 1.0, dl, dv, stats, ws,
                         exploration_loss=expl)
    s = stats.cpu()
    tot = s[ops.LS["total_loss"]].item()
    assert abs(tot - loss.item()) < 1e-5 * max(1.0, abs(loss.item())), (tot, loss.item())
    np.testing.assert_allclose(dl.cpu().numpy(), L.grad.numpy(), atol=1e-5)
    np.testing.assert_allclose(dv.cpu().numpy(), V.grad.numpy(), atol=1e-5)
    ratio = torch.empty(B, device=DEV)
    ops.action_ratio(logits.to(DEV), actions.to(DEV), lp_old.to(DEV), ratio)
    np.testing.assert_allclose(ratio.cpu().numpy(), torch.exp(lp.detach() - lp_old.double()).clamp(0.05, 20).numpy(),
                               rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("segs", [[24, 5, 16], [300, 62], [8, 16, 8, 992]])
@pytest.mark.parametrize("expl", ["entropy", "symmetric_kl"])
def test_tuple_loss_and_ratio_match_autograd(segs, expl):
    ops = ops_for()
    A, B = sum(segs), 400
    adv, valids, v_old, targets, values = _loss_inputs(B, A)
    logits = torch.randn(B, A, generator=g(1)) * 1.5
    logits_old = logits + 0.2 * torch.randn(B, A, generator=g(2))
    actions = torch.stack([torch.randint(0, n, (B,), generator=g(3 + k)) for k, n in enumerate(segs)], 1).float()
    lp_old = 0.05 * torch.randn(B, generator=g(9))
    L = logits.double().requires_grad_()
    V = values.double().requires_grad_()
    lp = ent = kl = 0
    start = 0
    for k, n in enumerate(segs):
        logp = torch.log_softmax(L[:, start:start + n], -1)
        p = logp.exp()
        lp = lp + logp.gather(1, actions[:, k].long().view(-1, 1)).view(-1)
        if expl == "entropy":
            ent = ent + (logp * p).sum(-1)
        else:
            u = 1.0 / n
            ent = ent + 0.5 * ((p * (logp - np.log(u))).sum(-1) + (u * (np.log(u) - logp)).sum(-1))
        kl = kl + (p * (logp - torch.log_softmax(logits_old[:, start:start + n].double(), -1))).sum(-1)
        start += n
    lp_old = lp.detach().float() + lp_old
    loss = _torch_ppo(lp, lp_old.double(), ent, kl, V, v_old.double(), targets.double(), adv, valids, 0.01, 0.05)
    loss.backward()
    stats = torch.zeros(ops.LS_SIZE, dtype=torch.float64, device=DEV)
    ws = torch.empty(ops.loss_workspace_bytes(B) // 8 + 8, dtype=torch.float64, device=DEV)
    vd = valids.to(DEV)
    ops.adv_stats(adv.to(DEV), vd, stats, None, ws)
    dl, dv = torch.empty(B, A, device=DEV), torch.empty(B, device=DEV)
    ops.ppo_loss_fwd_bwd_tuple(logits.to(DEV), values.to(DEV), segs, actions.to(DEV), lp_old.to(DEV), v_old.to(DEV),
                               adv.to(DEV), targets.to(DEV), vd, logits_old.to(DEV), 0.1, 0.2, 0.01, 0.5, 0.05, 1.0, dl,
                               dv, stats, ws, exploration_loss=expl)
    assert abs(stats[ops.LS["total_loss"]].item() - loss.item()) < 1e-5 * max(1.0, abs(loss.item()))
    np.testing.assert_allclose(dl.cpu().numpy(), L.grad.numpy(), atol=1e-5)
    np.testing.assert_allclose(dv.cpu().numpy(), V.grad.numpy(), atol=1e-5)
    ratio = torch.empty(B, device=DEV)
    ops.action_ratio_tuple(logits.to(DEV), segs, actions.to(DEV), lp_old.to(DEV), ratio)
    np.testing.assert_allclose(ratio.cpu().numpy(), torch.exp(lp.detach() - lp_old.double()).clamp(0.05, 20).numpy(),
                               rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("act_dim", [17, 40, 512])
@pytest.mark.parametrize("adaptive", [True, False])
def test_gaussian_loss_and_ratio_match_autograd(act_dim, adaptive):
    ops = ops_for()
    B = 300
    adv, valids, v_old, targets, values = _loss_inputs(B, act_dim)
    ts = 0.0 if adaptive else 1.5
    z = torch.randn(B, act_dim, generator=g(1))
    means = z if adaptive else torch.tanh(z / ts) * ts
    log_std = (torch.randn(B, act_dim, generator=g(2)) * 0.3) if adaptive else (torch.randn(act_dim, generator=g(2)) * 0.3).expand(B, act_dim)
    params = torch.cat([means, log_std], 1).contiguous()
    params_old = params + 0.05 * torch.randn(B, 2 * act_dim, generator=g(3))
    actions = means + torch.randn(B, act_dim, generator=g(4)) * log_std.exp()
    c_ent, c_kl = 0.003, 0.05

    Z = z.double().requires_grad_()
    S = log_std.double().clone().requires_grad_()
    V = values.double().requires_grad_()
    M = Z if adaptive else torch.tanh(Z / ts) * ts
    sd = S.exp().clamp(1e-4, 1e4)
    dist = torch.distributions.Normal(M, sd)
    lp = dist.log_prob(actions.double()).sum(-1)
    lp_old = (lp.detach() + 0.05 * torch.randn(B, generator=g(5)).double()).float()
    ent = -dist.entropy().sum(-1)
    sdo = params_old[:, act_dim:].double().exp().clamp(1e-4, 1e4)
    kl = torch.distributions.kl_divergence(dist, torch.distributions.Normal(params_old[:, :act_dim].double(), sdo)).sum(-1)
    loss = _torch_ppo(lp, lp_old.double(), ent, kl, V, v_old.double(), targets.double(), adv, valids, c_ent, c_kl)
    loss.backward()

    stats = torch.zeros(ops.LS_SIZE, dtype=torch.float64, device=DEV)
    ws = torch.empty(ops.loss_workspace_bytes(B) // 8 + 8, dtype=torch.float64, device=DEV)
    vd = valids.to(DEV)
    ops.adv_stats(adv.to(DEV), vd, stats, None, ws)
    dl = torch.empty(B, 2 * act_dim if adaptive else act_dim, device=DEV)
    dls = None if adaptive else torch.empty(B, act_dim, device=DEV)
    dv = torch.empty(B, device=DEV)
    ops.ppo_loss_fwd_bwd_continuous(params.to(DEV), values.to(DEV), adaptive, ts, actions.to(DEV), lp_old.to(DEV),
                                    v_old.to(DEV), adv.to(DEV), targets.to(DEV), vd, params_old.to(DEV), 0.1, 0.2, c_ent,
                                    0.5, c_kl, 1.0, dl, dls, dv, stats, ws)
    assert abs(stats[ops.LS["total_loss"]].item() - loss.item()) < 1e-5 * max(1.0, abs(loss.item()))
    got_dm = dl[:, :act_dim].cpu()
    got_ds = dl[:, act_dim:].cpu() if adaptive else dls.cpu()
    np.testing.assert_allclose(got_dm.numpy(), Z.grad.numpy(), atol=1e-5)
    np.testing.assert_allclose(got_ds.numpy(), S.grad.numpy(), atol=1e-5)
    np.testing.assert_allclose(dv.cpu().numpy(), V.grad.numpy(), atol=1e-5)
    ratio = torch.empty(B, device=DEV)
    ops.action_ratio_continuous(params.to(DEV), actions.to(DEV), lp_old.to(DEV), ratio)
    np.testing.assert_allclose(ratio.cpu().numpy(), torch.exp(lp.detach() - lp_old.double()).clamp(0.05, 20).numpy(),
                               rtol=1e-4, atol=1e-6)


# ----------------------------------------------------------------------------------------------- heads backward
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("tail", ["elu", "tanh", "gru", "separate"])
@pytest.mark.parametrize("A", [45, 362])
def test_wide_heads_backward_matches_autograd(engine, tail, A):
    """linear_backward (dWa, dz) + sfb200_heads_wide_backward vs autograd through critic_linear / distribution_linear and
    the tail's activation (a GRU tail feeds the heads its raw output: act' = 1, no bias gradient)"""
    need(engine)
    ops = ops_for()
    B, H = 700, 128
    sep = tail == "separate"
    act = {"elu": "elu", "tanh": "tanh", "gru": "none", "separate": "elu"}[tail]
    width = 2 * H if sep else H
    pre = torch.randn(B, width, generator=g(1))
    hcat = {"elu": F.elu, "tanh": torch.tanh, "none": lambda t: t}[act](pre)
    Wv, Wa = torch.randn(1, H, generator=g(2)) * 0.2, torch.randn(A, H, generator=g(3)) * 0.1
    dlog, dval = torch.randn(B, A, generator=g(4)) * 0.01, torch.randn(B, generator=g(5)) * 0.01

    P = pre.double().requires_grad_()
    Hx = {"elu": F.elu, "tanh": torch.tanh, "none": lambda t: t}[act](P)
    WV, WA = Wv.double().requires_grad_(), Wa.double().requires_grad_()
    BV, BA = torch.zeros(1, dtype=torch.float64, requires_grad=True), torch.zeros(A, dtype=torch.float64, requires_grad=True)
    ha, hv = (Hx[:, :H], Hx[:, H:]) if sep else (Hx, Hx)
    out = ((ha @ WA.t() + BA) * dlog.double()).sum() + ((hv @ WV.view(-1) + BV) * dval.double()).sum()
    out.backward()

    d = {k: v.to(DEV) for k, v in dict(h=hcat, Wv=Wv, Wa=Wa, dlog=dlog, dval=dval).items()}
    dz = torch.full((B, width), float("nan"), device=DEV)
    dWa, dWv = torch.empty(A, H, device=DEV), torch.empty(H, device=DEV)
    dba, dbv, db = torch.empty(A, device=DEV), torch.empty(1, device=DEV), torch.empty(width, device=DEV)
    eng = ops.ENGINES[engine]
    lin_ws = torch.empty(ops.linear_backward_workspace_bytes(B, A, H) // 4 + 4, device=DEV)
    hws = torch.empty(ops.heads_wide_backward_workspace_bytes(B, width, H, A) // 4 + 4, device=DEV)
    a = ops.ACT[act]
    if sep:
        ops.linear_backward(d["dlog"], d["h"][:, :H], d["Wa"], a, dWa, dz[:, :H], None, eng, lin_ws)
        ops.heads_wide_backward(d["h"][:, H:], d["Wv"], d["dlog"], d["dval"], a, dz, H, False, dWv, dbv, dba, db, hws)
    else:
        ops.linear_backward(d["dlog"], d["h"], d["Wa"], a, dWa, dz, None, eng, lin_ws)
        ops.heads_wide_backward(d["h"], d["Wv"], d["dlog"], d["dval"], a, dz, 0, True, dWv, dbv, dba,
                                None if act == "none" else db, hws)
    torch.cuda.synchronize()
    tol = 1e-5
    np.testing.assert_allclose(dz.cpu().numpy(), P.grad.numpy(), atol=tol)
    np.testing.assert_allclose(dWa.cpu().numpy(), WA.grad.numpy(), atol=tol)
    np.testing.assert_allclose(dWv.cpu().numpy(), WV.grad.view(-1).numpy(), atol=tol)
    np.testing.assert_allclose(dba.cpu().numpy(), BA.grad.numpy(), atol=tol)
    np.testing.assert_allclose(dbv.cpu().numpy(), BV.grad.numpy(), atol=tol)
    if act != "none":
        np.testing.assert_allclose(db.cpu().numpy(), P.grad.sum(0).numpy(), atol=1e-4)


# ----------------------------------------------------------------------------------------------- end to end
WIDE_CASES = ["tiny_wide_mask", "tiny_wide_tuple", "tiny_wide_gauss", "tiny_wide_gauss_learned"]


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", WIDE_CASES)
def test_wide_rollout_matches_reference_golden(name, engine):
    case = load_case(name)
    replay_sampler(case, build_case(case, engine))


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", WIDE_CASES)
def test_wide_learner_matches_reference_golden(name, engine):
    case = load_case(name)
    replay_learner(case, build_case(case, engine), rewards=True)


def _wide_ocfg(N, T, **kw):
    base = dict(rollout=T, recurrence=1, batch_size=N * T // 2, num_batches_per_epoch=2, num_actions=362,
                action_mask=True, encoder_mlp_layers=[128, 128])
    base.update(kw)
    return O.OracleCfg(**base)


def test_wide_graphed_learner_and_sampler_match_eager():
    """Discrete(362) with masks: the learner replayed as one CUDA graph and the graphed sampler give the same bits as the
    launch-by-launch versions"""
    N, T = 128, 8
    ocfg = _wide_ocfg(N, T)
    st0 = O.init_state(ocfg, seed=2)
    tape = torch.randn(6 * T + 1, N, ocfg.obs_dim, generator=g(3))
    eng = "3xtf32" if ops_for().tc_available() else "simt"
    a = build(ocfg, N, st0, tape, eng)
    b = build(ocfg, N, st0, tape, eng, graph=True, learner_cuda_graph=True)
    assert a.model.spec.wide_heads and b.sampler.use_cuda_graph and a.sampler.heads_plan.P == 0
    # graphed sampler: its first rollout runs eagerly and captures, so compare a second rollout from the same state
    graphed_sampler_matches_eager(a, b)
    graphed_learner_matches_eager(a, b, sampled_feed(a, b), exp_avg_sq=True)


@pytest.mark.parametrize("engine", ENGINES)
def test_closed_loop_vs_oracle_discrete362_masked(engine):
    """1024 tape envs, Discrete(362) with action masks, MLP 512-512: sampler + learner for 2 iterations against the oracle
    on the same tape, noise and initial weights"""
    from sample_factory_b200 import ops

    need(engine)
    N, T = 1024, 8
    ocfg = _wide_ocfg(N, T, batch_size=N * T // 4, num_batches_per_epoch=4, encoder_mlp_layers=[512, 512])
    st0 = O.init_state(ocfg, seed=3)
    gen = g(11)
    tape = torch.randn(2 * T + 1, N, ocfg.obs_dim, generator=gen) * 1.2 - 0.2
    cfg, model, traj, env, sampler, learner = build(ocfg, N, st0, tape, engine)
    olearner = O.OracleLearner(ocfg, st0)
    oenv = O.TapeVecEnv(tape, ocfg.num_actions, with_action_mask=True)
    olast = oenv.reset()
    sampler.reset()
    for it in range(2):
        noise = torch.empty(T, N, ocfg.num_actions).exponential_(generator=gen)
        otraj = O.alloc_trajectories(ocfg, N)
        olast = O.rollout(ocfg, olearner.st, oenv, olast, otraj, noise, olearner.train_step)
        sampler.noise = noise.to(DEV)
        sampler.set_policy_version(learner.train_step)
        sampler.rollout()
        got = {k: v.cpu() for k, v in traj.items()}
        mism = (got["actions"] != otraj["actions"]).float().mean().item()
        assert mism == 0.0, f"action mismatch fraction {mism}"
        for k in ["obs", "rewards", "dones", "time_outs", "policy_id", "policy_version"]:
            assert torch.equal(got[k], otraj[k]), k
        np.testing.assert_allclose(got["action_logits"].numpy(), otraj["action_logits"].numpy(), atol=TOL)
        np.testing.assert_allclose(got["values"][:, :-1].numpy(), otraj["values"][:, :-1].numpy(), atol=TOL)
        np.testing.assert_allclose(got["log_prob_actions"].numpy(), otraj["log_prob_actions"].numpy(), atol=TOL)
        n0 = len(olearner.log)
        olearner.train(otraj)
        learner.train(traj)
        log = learner.minibatch_log().numpy()
        for j, d in enumerate(olearner.log[n0:]):
            for key in ["policy_loss", "value_loss", "exploration_loss", "kl_loss"]:
                assert abs(log[j, ops.LS[key]] - d[key]) < TOL, (it, j, key, log[j, ops.LS[key]], d[key])
        sd = model.state_dict()
        for k in O.param_names(ocfg):
            np.testing.assert_allclose(sd[k].cpu().numpy(), olearner.st[k].numpy(), atol=2 * TOL, err_msg=k)
