"""Bit-for-bit A/B of the wgmma GEMM entry points between two builds of libsfb200.so (GPU box only).

    python tools/gemm_ab.py --lib path/to/libsfb200.so [--header path/to/sfb200.h] --out a.npz
    python tools/gemm_ab.py --compare a.npz b.npz

Runs, on seeded inputs, the forward (plain, with the heads folded in, residual) and dX in the fp16 and the tf32 form,
and dW (tf32 form, split-K), at the learner's size (M = 32768, 512 wide) and at ragged sizes: fewer work items than SMs,
more, M < 128, N and K that are no multiples of the tile, a split-K whose last slice is short.  Outputs are stored as
int32 bit patterns.  Forward and dX take no part in split-K, so they must not differ between builds that issue the same
wgmmas in the same order; dW depends on the split-K rule (SFB200_SPLITK_LEGACY=1 pins the earlier one), so --compare
lists it apart, and each run prints dW's largest error against an fp64 product.  dW is run twice: without bounds (the
tf32 form) and with both operands' bounds registered (the fp16 form, not bit-identical to the tf32 one)."""
from __future__ import annotations

import argparse
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = [(32768, 512, 512), (32768, 512, 64), (1000, 72, 200), (100, 128, 64), (17000, 512, 128), (4096, 256, 192),
          (5000, 130, 320)]


def run(out_path):
    import torch

    from sample_factory_b200 import ops

    dev = torch.device("cuda", 0)
    ops.bind_device(dev)
    eng = ops.GEMM_TC_3XTF32
    res = {}

    def keep(name, t):
        torch.cuda.synchronize()
        res[name] = t.detach().contiguous().view(torch.int32).cpu().numpy()

    for M, N, K in SHAPES:
        g = torch.Generator().manual_seed(M + N + K)
        rnd = lambda *s: torch.randn(*s, generator=g).to(dev)
        flat = rnd(N * K) / math.sqrt(K)
        W = flat.view(N, K)
        x, b, r = rnd(M, K), rnd(N) * 0.1, rnd(M, N)
        xa = torch.nn.functional.elu(x)
        dz = rnd(M, N) / M
        ws = torch.empty(ops.linear_backward_workspace_bytes(M, N, K) // 4 + 4, device=dev)
        A = 6
        Wv, Wa = rnd(N) * 0.1, (rnd(A, N) * 0.1).contiguous()
        P = ops.linear_heads_partials(N, A, eng)

        def all_forms(tag):
            y = torch.zeros(M, N, device=dev)
            ops.linear_act_forward(x, W, b, y, ops.ACT["elu"], eng)
            keep(f"{tag}/forward/{M}x{N}x{K}", y)
            y = torch.zeros(M, N, device=dev)
            ops.linear_residual_forward(x, W, b, r, y, eng)
            keep(f"{tag}/residual/{M}x{N}x{K}", y)
            if P:
                y = torch.zeros(M, N, device=dev)
                part = torch.zeros(P * M * ops.HEAD_PART_PAD, device=dev)
                ops.linear_act_heads_forward(x, W, b, y, ops.ACT["elu"], eng, Wv, Wa, part)
                keep(f"{tag}/heads_y/{M}x{N}x{K}", y)
                keep(f"{tag}/heads_partials/{M}x{N}x{K}", part)
            dx = torch.zeros(M, K, device=dev)
            ops.linear_backward(dz, xa, W, ops.ACT["elu"], None, dx, None, eng, ws)
            keep(f"{tag}/dx/{M}x{N}x{K}", dx)

        all_forms("tf32")
        if K % 64 == 0:
            twins = torch.empty(2 * N * K, dtype=torch.float16, device=dev)
            twinsT = torch.empty(2 * N * K, dtype=torch.float16, device=dev)
            ops.register_f16_twins(flat, twins)
            ops.register_f16_transposed(W, twinsT)
            bx, bz = (torch.full((1,), float(t.abs().max()), device=dev) for t in (x, dz))
            ops.register_operand_bound(x, bx)
            ops.register_operand_bound(dz, bz)
            try:
                all_forms("fp16")
            finally:
                ops.unregister_operand_bound(x)
                ops.unregister_operand_bound(dz)
                ops.unregister_f16_transposed(W)
                ops.unregister_f16_twins(flat)
        ref = dz.double().t() @ x.double()
        dW = torch.zeros(N, K, device=dev)
        ops.linear_backward(dz, x, W, ops.ACT["none"], dW, None, None, eng, ws)
        keep(f"dW/{M}x{N}x{K}", dW)
        print(f"dW {M}x{N}x{K}: max |err| vs fp64 {float((dW.double() - ref).abs().max()):.3e} of max "
              f"{float(ref.abs().max()):.3e}")
        # dW with both operands' bounds registered: the fp16 form (a build without it runs the tf32 form again)
        bx, bz = (torch.full((1,), float(t.abs().max()), device=dev) for t in (x, dz))
        ops.register_operand_bound(x, bx)
        ops.register_operand_bound(dz, bz)
        try:
            dW = torch.zeros(N, K, device=dev)
            ops.linear_backward(dz, x, W, ops.ACT["none"], dW, None, None, eng, ws)
        finally:
            ops.unregister_operand_bound(x)
            ops.unregister_operand_bound(dz)
        keep(f"dW16/{M}x{N}x{K}", dW)
        print(f"dW with bounds {M}x{N}x{K}: max |err| vs fp64 {float((dW.double() - ref).abs().max()):.3e} of max "
              f"{float(ref.abs().max()):.3e}")
    np.savez_compressed(out_path, **res)
    print(f"{len(res)} arrays -> {out_path}")


def compare(a_path, b_path):
    a, b = np.load(a_path), np.load(b_path)
    assert sorted(a.files) == sorted(b.files), set(a.files) ^ set(b.files)
    bad = [k for k in a.files if a[k].shape != b[k].shape or not np.array_equal(a[k], b[k])]
    for k in bad:
        print("DIFFERS", k, int((a[k] != b[k]).sum()), "of", a[k].size)
    n_dw = sum(k.startswith("dW") for k in a.files)
    bad_dw = [k for k in bad if k.startswith("dW")]
    n_dw16 = sum(k.startswith("dW16/") for k in a.files)
    bad_dw16 = sum(k.startswith("dW16/") for k in bad)
    print(f"forward / dX: {len(a.files) - n_dw - (len(bad) - len(bad_dw))} / {len(a.files) - n_dw} arrays bit-identical; "
          f"dW: {n_dw - n_dw16 - (len(bad_dw) - bad_dw16)} / {n_dw - n_dw16}; dW with bounds: {n_dw16 - bad_dw16} / {n_dw16}")
    return 1 if len(bad) > len(bad_dw) else 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", help="libsfb200.so to load (default: the in-tree build)")
    ap.add_argument("--header", help="include/sfb200.h of that build, when it lacks entry points this tree declares")
    ap.add_argument("--out")
    ap.add_argument("--compare", nargs=2)
    args = ap.parse_args()
    if args.compare:
        sys.exit(compare(*args.compare))
    if args.lib:
        from sample_factory_b200 import _lib

        _lib.LIB_PATH = os.path.abspath(args.lib)
        if args.header:
            parse = _lib.parse_header
            _lib.parse_header = lambda: parse(os.path.abspath(args.header))
    run(args.out)


if __name__ == "__main__":
    main()
