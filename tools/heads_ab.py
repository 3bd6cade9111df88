"""Bit-for-bit A/B of the heads entry points between two builds of libsfb200.so.

    python tools/heads_ab.py --lib path/to/libsfb200.so --out a.npz
    python tools/heads_ab.py --compare a.npz b.npz

Runs heads_forward (every instantiation the dispatch picks), heads_from_partials, heads_tail_wide and the three mixed
Tuple entry points on seeded inputs: Discrete (masked, with an all-masked row), Tuple, Box adaptive and learned
(tanh_scale 0 and 1.5), each with explicit noise, Philox and deterministic sampling, plus the values-only and
params-only modes.  Every output (values, params rows, actions, env actions, log-prob, policy-version stamp) is stored
as int32 bit patterns, so -0.0 and NaN payloads count.

The step-tail section runs the entry points after the heads -- sampler_tail_tape_step, sampler_post_step,
sampler_post_pre_step, tape_env_step(_continuous) and the persistent rollout_mlp2_tape (tf32 form: no fp16 twins are
registered here) -- over N = 4000 envs (a partial last row block), K1 in {32, 64, 96, 128} and H in {128, 256, 512},
with explicit noise and Philox, with and without the normaliser's running statistics and with and without the episode,
fin_* and stats buffers.  Every env, trajectory, episode and counter buffer is compared bit for bit, except the episode
statistics (keys ending in /stats): sums of double atomics in a run-dependent order, compared with rtol 1e-12."""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

MIXED_NARROW = [[("discrete", 3), ("box", 2), ("discrete", 4)], [("box", 3), ("discrete", 5)], [("box", 1)]]
MIXED_PARTIALS = [[("discrete", 3), ("box", 2)], [("box", 3), ("discrete", 2)], [("box", 1)]]
MIXED_WIDE = [[("discrete", 24), ("box", 8), ("discrete", 5)], [("box", 300), ("discrete", 62), ("box", 100)],
              [("discrete", 7), ("box", 2), ("discrete", 31), ("box", 5), ("discrete", 1)], [("box", 512)]]
WIDE_A = [32, 33, 64, 65, 128, 129, 256, 257, 512, 513, 1024]
MODES = ("noise", "philox", "det")


def run(out_path):
    import torch

    from sample_factory_b200 import ops

    dev = torch.device("cuda", 0)
    ops.bind_device(dev)
    res = {}
    g = torch.Generator(device="cpu").manual_seed(0)

    def rnd(*shape, scale=1.0):
        return (torch.randn(*shape, generator=g) * scale).to(dev)

    def keep(name, **arrays):
        torch.cuda.synchronize()
        for k, v in arrays.items():
            if v is not None:
                res[f"{name}/{k}"] = v.detach().contiguous().view(torch.int32).cpu().numpy()

    def sample_args(rows, n_noise, n_act, mode, env_dtype, env_w, tag):
        o = dict(actions_f32=torch.full((rows, n_act), -7.0, device=dev),
                 log_prob=torch.full((rows,), -7.0, device=dev),
                 policy_version_scalar=torch.tensor([3.0], device=dev), policy_version_out=torch.zeros(rows, device=dev))
        o["env_actions"] = torch.full((rows, env_w), -7, dtype=env_dtype, device=dev)
        o.update(actions_stride=n_act, log_prob_stride=1, pv_stride=1)
        if mode == "noise":
            o["noise"] = torch.rand(rows, n_noise, generator=g).clamp_min(1e-6).to(dev) if tag == "cat" else rnd(rows, n_noise)
        else:
            o.update(philox_seed=1234, philox_offset=56)
        ops.set_sampling_mode(None, mode == "det")
        return o

    def outs(o):
        return {k: o[k] for k in ("actions_f32", "log_prob", "policy_version_out", "env_actions")}

    # ---- narrow heads: spaces x sampling modes x the heads_forward instantiations (A+1 <= 9 / 17 / 32, rows <= / >
    #      8192, vectorised / H % 4 != 0) and heads_from_partials
    spaces = [("discrete", dict(A=5)), ("discrete", dict(A=16)), ("discrete", dict(A=31)), ("tuple", dict(sizes=[3, 4, 2])),
              ("tuple", dict(sizes=[9, 11, 6])), ("box_adaptive", dict(d=4)), ("box_adaptive", dict(d=15)),
              ("box_learned0", dict(d=6)), ("box_learned1.5", dict(d=6))]
    for sname, sp in spaces:
        if sname == "discrete":
            A, n_act, n_noise, kind = sp["A"], 1, sp["A"], "cat"
        elif sname == "tuple":
            A, n_act, n_noise, kind = sum(sp["sizes"]), len(sp["sizes"]), sum(sp["sizes"]), "cat"
        else:
            d = sp["d"]
            A = 2 * d if sname == "box_adaptive" else d
            n_act, n_noise, kind = d, d, "box"
        for rows, H in [(1000, 64), (9000, 64), (1000, 37)]:
            h = rnd(rows, H, scale=0.5)
            Wv, bv, Wa, ba = rnd(H, scale=0.1), rnd(1), rnd(A, H, scale=0.2), rnd(A)
            for mode in MODES + ("values", "params"):
                sm = mode if mode in MODES else "philox"
                o = sample_args(rows, n_noise, n_act, sm, torch.float32 if kind == "box" else torch.int32,
                                n_act if kind == "box" else n_act, kind)
                if mode == "values":
                    o = {}
                values = torch.full((rows,), -7.0, device=dev)
                params = torch.full((rows, 2 * n_act if kind == "box" else A), -7.0, device=dev) if mode != "values" else None
                if mode == "params":
                    o = {}
                common = dict(logits=params, logits_stride=0 if params is None else params.shape[1], **o)
                name = f"fwd/{sname}{A}/{rows}x{H}/{mode}"
                if sname == "discrete":
                    ops.heads_forward(h, Wv, bv, Wa, ba, values, 1, **common)
                elif sname == "tuple":
                    ops.heads_forward_tuple(h, Wv, bv, Wa, ba, sp["sizes"], values, 1, **common)
                else:
                    ls = rnd(d, scale=0.3) if sname != "box_adaptive" else None
                    ts = 1.5 if sname == "box_learned1.5" else 0.0
                    ops.heads_forward_continuous(h, Wv, bv, Wa, ba, d, sname == "box_adaptive", ls, ts, values, 1, **common)
                keep(name, values=values, params=params, **(outs(o) if o else {}))
                if A + 1 <= 11 and rows == 1000 and H == 64:
                    P = 3
                    part = rnd(P, rows, 12)
                    values = torch.full((rows,), -7.0, device=dev)
                    params = torch.full_like(params, -7.0) if params is not None else None
                    o2 = {k: (torch.full_like(v, -7) if torch.is_tensor(v) and k != "noise" and k != "policy_version_scalar" else v)
                          for k, v in o.items()}
                    ops.set_sampling_mode(None, mode == "det")
                    common = dict(logits=params, logits_stride=0 if params is None else params.shape[1], **o2)
                    if sname == "discrete":
                        ops.heads_from_partials(part, P, rows, bv, ba, values, 1, **common)
                    elif sname == "tuple":
                        ops.heads_from_partials_tuple(part, P, rows, bv, ba, sp["sizes"], values, 1, **common)
                    else:
                        ops.heads_from_partials_continuous(part, P, rows, bv, ba, d, sname == "box_adaptive", ls, ts,
                                                           values, 1, **common)
                    keep(f"partials/{sname}{A}/{mode}", values=values, params=params, **(outs(o2) if o2 else {}))
    # masked Discrete, one row with nothing allowed
    for A in (5, 20, 300):
        rows, H = 2000, 64
        h = rnd(rows, H, scale=0.5)
        Wv, bv, Wa, ba = rnd(H, scale=0.1), rnd(1), rnd(A, H, scale=0.2), rnd(A)
        mask = (torch.rand(rows, A, generator=g) > 0.4).to(torch.uint8).to(dev)
        mask[7] = 0
        for mode in MODES:
            o = sample_args(rows, A, 1, mode, torch.int32, 1, "cat")
            ops.set_sampling_mode(mask, mode == "det")
            values = torch.full((rows,), -7.0, device=dev)
            params = torch.full((rows, A), -7.0, device=dev)
            if A <= 31:
                ops.heads_forward(h, Wv, bv, Wa, ba, values, 1, logits=params, logits_stride=A, **o)
            else:
                params.copy_(rnd(rows, A))
                ops.heads_tail_wide(h, Wv, bv, params, A, A, values, 1, **o)
            keep(f"masked/{A}/{mode}", values=values, params=params, **outs(o))
    ops.set_sampling_mode(None, False)
    # ---- wide heads over stored rows
    for A in WIDE_A:
        rows, H = 3000, 64
        h = rnd(rows, H, scale=0.5)
        Wv, bv = rnd(H, scale=0.1), rnd(1)
        for kind in ("discrete", "tuple", "box_adaptive", "box_learned0", "box_learned1.5"):
            if kind == "tuple":
                sizes = [A // 3, A // 3, A - 2 * (A // 3)]
            if kind == "box_adaptive" and A % 2:
                continue
            d = A // 2 if kind == "box_adaptive" else A
            box = kind.startswith("box")
            n_act = d if box else (3 if kind == "tuple" else 1)
            for mode in MODES + ("values", "params"):
                sm = mode if mode in MODES else "philox"
                o = sample_args(rows, d if box else A, n_act, sm, torch.float32 if box else torch.int32, n_act,
                                "box" if box else "cat")
                if mode in ("values", "params"):
                    o = {}
                values = torch.full((rows,), -7.0, device=dev)
                params = None
                if mode != "values":
                    params = torch.full((rows, 2 * d if box else A), -7.0, device=dev)
                    params[:, :A] = rnd(rows, A)
                kw = {}
                if kind == "tuple":
                    kw["head_sizes"] = sizes
                if box:
                    kw.update(continuous=True, act_dim=d, adaptive_stddev=kind == "box_adaptive",
                              learned_log_std=rnd(d, scale=0.3) if kind != "box_adaptive" else None,
                              tanh_scale=1.5 if kind == "box_learned1.5" else 0.0)
                ops.heads_tail_wide(h, Wv, bv, params, 0 if params is None else params.shape[1], A, values, 1, **o, **kw)
                keep(f"wide/{kind}/{A}/{mode}", values=values, params=params, **(outs(o) if o else {}))
    # ---- mixed Tuple spaces, all three entry points
    for path, lists in (("forward", MIXED_NARROW), ("partials", MIXED_PARTIALS), ("wide", MIXED_WIDE)):
        for li, members in enumerate(lists):
            kinds = [0 if k == "discrete" else 1 for k, _ in members]
            sizes = [n for _, n in members]
            A = sum(n if k == 0 else 2 * n for k, n in zip(kinds, sizes))
            W = sum(1 if k == 0 else n for k, n in zip(kinds, sizes))
            Wn = sum(sizes)
            rows, H = 3000, 64
            h = rnd(rows, H, scale=0.5)
            Wv, bv, Wa, ba = rnd(H, scale=0.1), rnd(1), rnd(A, H, scale=0.2), rnd(A)
            for mode in MODES:
                ops.set_sampling_mode(None, mode == "det")
                o = dict(actions_f32=torch.full((rows, W), -7.0, device=dev), actions_stride=W,
                         log_prob=torch.full((rows,), -7.0, device=dev), log_prob_stride=1,
                         policy_version_scalar=torch.tensor([3.0], device=dev),
                         policy_version_out=torch.zeros(rows, device=dev), pv_stride=1)
                env = [torch.full((rows,), -7, dtype=torch.int32, device=dev) if k == 0 else
                       torch.full((rows, n), -7.0, device=dev) for k, n in zip(kinds, sizes)]
                if mode == "noise":
                    nz = torch.empty(rows, Wn)
                    c = 0
                    for k, n in zip(kinds, sizes):
                        nz[:, c:c + n] = torch.rand(rows, n, generator=g).clamp_min(1e-6) if k == 0 else \
                            torch.randn(rows, n, generator=g)
                        c += n
                    o["noise"] = nz.to(dev)
                else:
                    o.update(philox_seed=99, philox_offset=7)
                values = torch.full((rows,), -7.0, device=dev)
                params = torch.full((rows, A), -7.0, device=dev)
                if path == "forward":
                    ops.heads_forward_mixed(h, Wv, bv, Wa, ba, kinds, sizes, values, 1, params, A, env_actions=env, **o)
                elif path == "partials":
                    P = 2
                    part = rnd(P, rows, 12)
                    ops.heads_from_partials_mixed(part, P, rows, bv, ba, kinds, sizes, values, 1, params, A,
                                                  env_actions=env, **o)
                else:
                    params.copy_(rnd(rows, A))
                    ops.heads_tail_wide_mixed(h, Wv, bv, params, A, A, kinds, sizes, values, 1, env_actions=env, **o)
                keep(f"mixed/{path}/{li}/{mode}", values=values, params=params, actions=o["actions_f32"],
                     log_prob=o["log_prob"], pv=o["policy_version_out"],
                     **{f"env{i}": e for i, e in enumerate(env)})
    ops.set_sampling_mode(None, False)
    step_tail(ops, dev, g, rnd, keep)
    res.update(res_stats)
    np.savez_compressed(out_path, **res)
    print(f"{len(res)} arrays -> {out_path}")


def step_tail(ops, dev, g, rnd, keep):
    import torch

    from sample_factory_b200.envs import TapeVecEnv
    from sample_factory_b200.trajectory import alloc_trajectory_tensors

    N, A, T, R = 4000, 6, 5, 16

    def episode(full):
        """episode accumulators, stats and fin_* buffers (all None when not full)"""
        if not full:
            return dict(ep_return=None, ep_len=None, ep_min_raw=None, ep_max_raw=None, stats=None)
        return dict(ep_return=rnd(N), ep_len=torch.randint(0, 50, (N,), generator=g, dtype=torch.int32).to(dev),
                    ep_min_raw=rnd(N), ep_max_raw=rnd(N), stats=torch.zeros(8, dtype=torch.float64, device=dev))

    def fin(full, t_=T):
        if not full:
            return None, None
        return torch.full((N, t_), -7.0, device=dev), torch.full((N, t_), -7, dtype=torch.int32, device=dev)

    def keep_tail(name, env, ep, traj, **more):
        """the env, episode and trajectory buffers a step-tail entry point writes; the episode statistics aside"""
        out = dict(env_obs=env.obs, env_rew=env.rew, env_term=env.terminated, env_trunc=env.truncated,
                   env_step=env.step_counter, **{k: v for k, v in ep.items() if k != "stats"}, **traj, **more)
        keep(name, **{k: v.int() if v is not None and v.dtype == torch.bool else v for k, v in out.items()})
        if ep["stats"] is not None:
            res_stats[f"{name}/stats"] = ep["stats"].cpu().numpy()

    def norm(rms, dim):
        if not rms:
            return dict(mean=None, var=None, sub_mean=0.0, inv_scale=1.0)
        return dict(mean=rnd(dim, scale=0.3).double(), var=(rnd(dim).abs() + 0.5).double(), sub_mean=0.25, inv_scale=0.5)

    for K1 in (32, 64, 96, 128):
        tape = rnd(2 * T + 1, N, K1)
        for full in (True, False):
            for rms in (True, False):
                tag = f"{K1}/{'ep' if full else 'noep'}/{'rms' if rms else 'norms'}"
                # ---- per-stage kernels: env step (Discrete and Box), post step, post + pre step
                env = TapeVecEnv(tape, A)
                env.step_counter[0] = 3
                acts = torch.randint(0, A, (N,), generator=g, dtype=torch.int32).to(dev)
                ops.tape_env_step(acts, A, 5, env.term_period, env.trunc_period, env.step_counter, 0, tape, env.obs, env.rew,
                                  env.terminated, env.truncated)
                keep(f"tail/env/{tag}", obs=env.obs, rew=env.rew, term=env.terminated.int(), trunc=env.truncated.int(),
                     step=env.step_counter)
                acts_f = rnd(N, 3)
                ops.tape_env_step_continuous(acts_f, 5, env.term_period, env.trunc_period, None, 7, None, None, env.rew,
                                             env.terminated, env.truncated)
                keep(f"tail/env_box/{tag}", rew=env.rew, term=env.terminated.int(), trunc=env.truncated.int())
                traj = alloc_trajectory_tensors(K1, A, N, T, dev, rnn_size=R)
                ep = episode(full)
                fr, fl = fin(full)
                pstep = torch.zeros(1, dtype=torch.int64, device=dev)
                ops.sampler_post_step(env.rew, env.terminated, env.truncated, 0.5, 0.3, 2, traj["rewards"][:, 0],
                                      traj["dones"][:, 0], traj["time_outs"][:, 0], traj["policy_id"][:, 0], ep["ep_return"],
                                      ep["ep_len"], ep["ep_min_raw"], ep["ep_max_raw"], 2, ep["stats"], pstep,
                                      None if fr is None else fr[:, 0], None if fl is None else fl[:, 0])
                rnn = rnd(N, R)
                x_norm = torch.full((N, K1), -7.0, device=dev)
                ops.sampler_post_pre_step(env.rew, env.terminated, env.truncated, 1.0, 10.0, 1, traj["rewards"][:, 1],
                                          traj["dones"][:, 1], traj["time_outs"][:, 1], traj["policy_id"][:, 1],
                                          ep["ep_return"], ep["ep_len"], ep["ep_min_raw"], ep["ep_max_raw"], 1, ep["stats"],
                                          pstep, None if fr is None else fr[:, 1], None if fl is None else fl[:, 1],
                                          obs=env.obs, traj_obs_next=traj["obs"][:, 2], rnn=rnn,
                                          traj_rnn_next=traj["rnn_states"][:, 2], x_norm=x_norm, **norm(rms, K1))
                keep_tail(f"tail/post/{tag}", env, ep, traj, pstep=pstep, x_norm=x_norm, fin_ret=fr, fin_len=fl)
                for mode in ("noise", "philox"):
                    noise = torch.rand(T, N, A, generator=g).clamp_min(1e-6).to(dev) if mode == "noise" else None
                    # ---- fused step tail (heads.cu): T steps on random partials
                    env = TapeVecEnv(tape, A, env_index_offset=11)
                    traj = alloc_trajectory_tensors(K1, A, N, T, dev, rnn_size=R)
                    ep = episode(full)
                    fr, fl = fin(full)
                    sstep = torch.full((1,), 4, dtype=torch.int64, device=dev)
                    env_actions = torch.full((N,), -7, dtype=torch.int32, device=dev)
                    x_norm = torch.full((N, K1), -7.0, device=dev)
                    bv, ba, P = rnd(1), rnd(A), 3
                    pv = torch.tensor([2.0], device=dev)
                    tr = traj
                    for t in range(T):
                        part = rnd(P, N, 12)
                        ops.sampler_tail_tape_step(
                            part, P, N, bv, ba, values=tr["values"][:, t], values_stride=tr["values"].stride(0),
                            logits=tr["action_logits"][:, t], logits_stride=tr["action_logits"].stride(0),
                            noise=None if noise is None else noise[t], philox_seed=77, sampler_step=sstep,
                            actions_f32=tr["actions"][:, t], actions_stride=tr["actions"].stride(0),
                            env_actions=env_actions,
                            log_prob=tr["log_prob_actions"][:, t], log_prob_stride=tr["log_prob_actions"].stride(0),
                            policy_version_scalar=pv, policy_version_out=tr["policy_version"][:, t],
                            pv_stride=tr["policy_version"].stride(0), env=env, reward_scale=0.5, reward_clip=0.3,
                            policy_id=1, traj_rewards=tr["rewards"][:, t], traj_dones=tr["dones"][:, t],
                            traj_time_outs=tr["time_outs"][:, t], traj_policy_id=tr["policy_id"][:, t], len_increment=2,
                            fin_return=None if fr is None else fr[:, t], fin_len=None if fl is None else fl[:, t],
                            traj_obs_next=tr["obs"][:, t + 1], rnn=rnn, traj_rnn_next=tr["rnn_states"][:, t + 1],
                            x_norm=None if t == T - 1 else x_norm, **ep, **norm(rms, K1))
                    keep_tail(f"tail/fused/{tag}/{mode}", env, ep, traj, x_norm=x_norm, fin_ret=fr, fin_len=fl,
                              env_actions=env_actions, sstep=sstep)
                    # ---- persistent rollout (rollout_fused.cu)
                    for H in (128, 256, 512):
                        W1, b1, W2, b2 = rnd(H, K1, scale=0.1), rnd(H, scale=0.1), rnd(H, H, scale=0.05), rnd(H, scale=0.1)
                        Wv, bv, Wa, ba = rnd(H, scale=0.1), rnd(1), rnd(A, H, scale=0.1), rnd(A)
                        assert ops.rollout_mlp2_partials(W1, W2, A, ops.GEMM_TC_3XTF32)
                        env = TapeVecEnv(tape, A, env_index_offset=11)
                        env.step_counter[0] = 2
                        traj = alloc_trajectory_tensors(K1, A, N, T, dev, rnn_size=R)
                        ep = episode(full)
                        fr, fl = fin(full)
                        sstep = torch.full((1,), 9, dtype=torch.int64, device=dev)
                        env_actions = torch.full((N,), -7, dtype=torch.int32, device=dev)
                        x_norm = rnd(N, K1)
                        h1 = torch.zeros(N, H, device=dev)
                        part = torch.zeros(H // 64, N, 12, device=dev)
                        ops.rollout_mlp2_tape(T, W1, b1, W2, b2, ops.ACT["elu"], ops.GEMM_TC_3XTF32, Wv, bv, Wa, ba, h1,
                                              part, x_norm, traj, env, noise, 55, sstep, env_actions, pv, 0.5, 0.3, 1,
                                              ep["ep_return"], ep["ep_len"], ep["ep_min_raw"], ep["ep_max_raw"], 2,
                                              ep["stats"], fr, fl, rnn, **norm(rms, K1))
                        keep_tail(f"tail/rollout/{H}/{tag}/{mode}", env, ep, traj, x_norm=x_norm, fin_ret=fr, fin_len=fl,
                                  env_actions=env_actions, sstep=sstep)


res_stats = {}   # episode statistics of the step-tail section: float64, compared with rtol 1e-12


def compare(a_path, b_path):
    a, b = np.load(a_path), np.load(b_path)
    assert sorted(a.files) == sorted(b.files), set(a.files) ^ set(b.files)
    stats = [k for k in a.files if k.endswith("/stats")]
    for k in stats:
        np.testing.assert_allclose(a[k], b[k], rtol=1e-12, err_msg=k)
    bad = [k for k in a.files if k not in stats and (a[k].shape != b[k].shape or not np.array_equal(a[k], b[k]))]
    for k in bad[:20]:
        print("DIFFERS", k, int((a[k] != b[k]).sum()) if a[k].shape == b[k].shape else "shape")
    print(f"{len(a.files) - len(stats) - len(bad)} / {len(a.files) - len(stats)} arrays bit-identical, "
          f"{len(stats)} episode statistics within rtol 1e-12")
    return 1 if bad else 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", help="libsfb200.so to load (default: the in-tree build)")
    ap.add_argument("--out")
    ap.add_argument("--compare", nargs=2)
    args = ap.parse_args()
    if args.compare:
        sys.exit(compare(*args.compare))
    if args.lib:
        from sample_factory_b200 import _lib

        _lib.LIB_PATH = os.path.abspath(args.lib)
    run(args.out)


if __name__ == "__main__":
    main()
