"""Bit-for-bit A/B of the heads entry points between two builds of libsfb200.so.

    python tools/heads_ab.py --lib path/to/libsfb200.so --out a.npz
    python tools/heads_ab.py --compare a.npz b.npz

Runs heads_forward (every instantiation the dispatch picks), heads_from_partials, heads_tail_wide and the three mixed
Tuple entry points on seeded inputs: Discrete (masked, with an all-masked row), Tuple, Box adaptive and learned
(tanh_scale 0 and 1.5), each with explicit noise, Philox and deterministic sampling, plus the values-only and
params-only modes.  Every output (values, params rows, actions, env actions, log-prob, policy-version stamp) is stored
as int32 bit patterns, so -0.0 and NaN payloads count."""
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
    np.savez_compressed(out_path, **res)
    print(f"{len(res)} arrays -> {out_path}")


def compare(a_path, b_path):
    a, b = np.load(a_path), np.load(b_path)
    assert sorted(a.files) == sorted(b.files), set(a.files) ^ set(b.files)
    bad = [k for k in a.files if a[k].shape != b[k].shape or not np.array_equal(a[k], b[k])]
    for k in bad[:20]:
        print("DIFFERS", k, int((a[k] != b[k]).sum()) if a[k].shape == b[k].shape else "shape")
    print(f"{len(a.files) - len(bad)} / {len(a.files)} arrays bit-identical")
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
