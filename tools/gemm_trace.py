"""Where a work item's time goes in the wgmma GEMM (csrc/gemm_tc.cu) at the learner's shapes of the headline workload
(GPU box only).

Switches the kernel's trace on (sfb200_gemm_set_trace: one consumer thread and the producer thread of every CTA stamp
%globaltimer and %smid per work item) and runs, at M = 32768: the layer-2 forward with the heads folded in and dX
(fp16 form, 512 x 512), the layer-1 forward (fp16 form, 512 x 64: one stage per item, so nearly all epilogue), dW2
(512 x 512) and dW1 (512 x 64) (split-K; both operands have registered bounds, so a library with the fp16 dW form runs
that, gemm_dw_f16_kernel, and one without it the tf32 form).  Prints per GEMM: CTAs, work items and
items per CTA, the mean microseconds of an item split into fill (item begun -> its first stage landed), mainloop and
epilogue, the epilogue split at the stamps inside it (a library without them leaves the words zero and the parts
unprinted): accumulators combined, the epilogue's batch of global loads landed, and then either the stores issued, or for
the fused heads: activated row stored, head partials stored, heads finished; the once-per-CTA setup (kernel entry -> barriers initialised and the programmatic-dependency wait passed), how
far ahead of the consumers the producer issued an item's first load, and the kernel's span against the busiest CTA's sum
of phases.  The stamps cost a few stores per item; the times are a profile, not a benchmark.

  python tools/gemm_trace.py --out DIR [--lib path/to/libsfb200.so] [--reps 5]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.feature_bench import card  # noqa: E402

M, H, OBS, A = 32768, 512, 64, 8


def epilogue_parts(t, us):
    """the epilogue between its stamps (words 10-13; 4 and 5 are its ends), whole-tile items only"""
    t = t[(t[:, 10] != 0) & (t[:, 11] != 0)]
    if t.shape[0] == 0:
        return None
    parts = {"combine": us(t[:, 10] - t[:, 4]), "loads": us(t[:, 11] - t[:, 10])}
    if bool((t[:, 13] != 0).all()):
        parts.update({"act_store": us(t[:, 12] - t[:, 11]), "head_partials": us(t[:, 13] - t[:, 12]),
                      "heads_finish": us(t[:, 5] - t[:, 13])})
    else:
        parts["math_store"] = us(t[:, 5] - t[:, 11])
    return parts


def summarize(t):
    """t: [items, 16] int64 stamps of one launch -> dict of means in us"""
    import torch

    t = t[t[:, 2] != 0]
    cta = t[:, 1]
    first = t[:, 8] != 0                         # the CTA's first item carries the entry / setup stamps
    us = lambda a: float(a.double().mean()) / 1e3
    fill, main, epi = t[:, 3] - t[:, 2], t[:, 4] - t[:, 3], t[:, 5] - t[:, 4]
    # an item's fill as the CTA sees it starts at the setup stamp for its first item
    fill = torch.where(first, t[:, 3] - t[:, 9], fill)
    later = ~first
    per_cta = torch.zeros(int(cta.max()) + 1, dtype=torch.int64)
    per_cta.index_add_(0, cta, fill + main + epi)
    per_cta.index_add_(0, cta[first], (t[:, 9] - t[:, 8])[first])
    counts = torch.bincount(cta)
    return {
        "ctas": int((counts > 0).sum()), "items": int(t.shape[0]), "sms": int(t[:, 0].unique().numel()),
        "items_per_cta_max": int(counts.max()),
        "setup_us": us((t[:, 9] - t[:, 8])[first]),
        "fill_first_item_us": us(fill[first]),
        "fill_later_items_us": us(fill[later]) if bool(later.any()) else None,
        "mainloop_us": us(main), "epilogue_us": us(epi),
        "epilogue_parts_us": epilogue_parts(t, us),
        "item_us": us(fill + main + epi),
        "producer_lead_us": us((t[:, 2] - t[:, 6])[later]) if bool(later.any()) else None,
        "kernel_span_us": float(t[:, 5].max() - t[:, 8][first].min()) / 1e3,
        "busiest_cta_sum_us": float(per_cta.max()) / 1e3,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--lib", help="libsfb200.so to load (default: the in-tree build)")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if args.lib:
        from sample_factory_b200 import _lib

        _lib.LIB_PATH = os.path.abspath(args.lib)
    import torch

    from sample_factory_b200 import ops

    assert torch.cuda.is_available(), "gemm_trace.py needs a GPU"
    dev = torch.device("cuda", 0)
    ops.bind_device(dev)
    eng = ops.GEMM_TC_3XTF32
    gen = torch.Generator().manual_seed(0)
    rnd = lambda *s: torch.randn(*s, generator=gen).to(dev)

    flat = rnd(H * H) / math.sqrt(H)
    W2 = flat.view(H, H)
    W1 = (rnd(H, OBS) / math.sqrt(OBS)).contiguous()
    flat1 = W1.view(-1)
    b1 = rnd(H) * 0.1
    b2, Wv, Wa = rnd(H) * 0.1, rnd(H) * 0.1, (rnd(A, H) * 0.1).contiguous()
    h1, x0 = torch.nn.functional.elu(rnd(M, H)), rnd(M, OBS)
    dz = rnd(M, H) / M
    y, dx, dW2, dW1 = (torch.empty(M, H, device=dev), torch.empty(M, H, device=dev), torch.empty(H, H, device=dev),
                       torch.empty(H, OBS, device=dev))
    part = torch.empty(ops.linear_heads_partials(H, A, eng) * M * ops.HEAD_PART_PAD, device=dev)
    ws = torch.empty(ops.linear_backward_workspace_bytes(M, H, H) // 4 + 4, device=dev)
    twins = torch.empty(2 * H * H, dtype=torch.float16, device=dev)
    twinsT = torch.empty(2 * H * H, dtype=torch.float16, device=dev)
    ops.register_f16_twins(flat, twins)
    ops.register_f16_transposed(W2, twinsT)
    twins1 = torch.empty(2 * H * OBS, dtype=torch.float16, device=dev)
    ops.register_f16_twins(flat1, twins1)
    bounds = [torch.full((1,), float(t.abs().max()), device=dev) for t in (h1, dz, x0)]
    ops.register_operand_bound(h1, bounds[0])
    ops.register_operand_bound(dz, bounds[1])
    ops.register_operand_bound(x0, bounds[2])

    gemms = [
        ("forward + heads, fp16 form <0,0,1,1,1,0> [32768 x 512 x 512]",
         lambda: ops.linear_act_heads_forward(h1, W2, b2, y, ops.ACT["elu"], eng, Wv, Wa, part)),
        ("dX, fp16 form <0,1,1,0,1,0> [32768 x 512 x 512]",
         lambda: ops.linear_backward(dz, h1, W2, ops.ACT["elu"], None, dx, None, eng, ws)),
        ("layer-1 forward, fp16 form <0,0,1,0,1,0> [32768 x 512 x 64]",
         lambda: ops.linear_act_forward(x0, W1, b1, y, ops.ACT["elu"], eng)),
        ("dW2, split-K [512 x 512, k = 32768]",
         lambda: ops.linear_backward(dz, h1, W2, ops.ACT["elu"], dW2, None, None, eng, ws)),
        ("dW1, split-K [512 x 64, k = 32768]",
         lambda: ops.linear_backward(dz, x0, W1, ops.ACT["none"], dW1, None, None, eng, ws)),
    ]
    trace = torch.zeros(4096 * ops.GEMM_TRACE_WORDS, dtype=torch.int64, device=dev)
    hw = card()
    result = {**hw, "lib": args.lib or "in-tree", "reps": args.reps, "gemms": {}}
    print(f"{hw['gpu']} ({hw['power_limit_w']} W, {hw['max_sm_clock_mhz']} MHz); library: {result['lib']}; means over "
          f"{args.reps} launches, us")
    try:
        for name, fn in gemms:
            fn()
            torch.cuda.synchronize()
            ops.set_gemm_trace(trace)
            rows = []
            for _ in range(args.reps):
                trace.zero_()
                fn()
                torch.cuda.synchronize()
                rows.append(summarize(trace.cpu().view(-1, ops.GEMM_TRACE_WORDS)))
            ops.set_gemm_trace(None)
            avg = lambda vs: None if vs[0] is None else round(sum(vs) / len(vs), 2)
            mean = {k: avg([r[k] for r in rows]) for k in rows[0] if k != "epilogue_parts_us"}
            parts = rows[0]["epilogue_parts_us"]
            mean["epilogue_parts_us"] = parts and {k: avg([r["epilogue_parts_us"][k] for r in rows]) for k in parts}
            result["gemms"][name] = mean
            print(name)
            print(f"  {mean['items']:.0f} items on {mean['ctas']:.0f} CTAs ({mean['sms']:.0f} SMs), at most "
                  f"{mean['items_per_cta_max']:.0f} per CTA")
            print(f"  per CTA: setup {mean['setup_us']};  per item: fill {mean['fill_first_item_us']} (first) / "
                  f"{mean['fill_later_items_us']} (later), mainloop {mean['mainloop_us']}, epilogue {mean['epilogue_us']}, "
                  f"total {mean['item_us']}")
            if mean["epilogue_parts_us"]:
                print("  epilogue: " + ", ".join(f"{k} {v}" for k, v in mean["epilogue_parts_us"].items()))
            print(f"  producer issued a later item's first load {mean['producer_lead_us']} before the consumers began it")
            print(f"  kernel span {mean['kernel_span_us']} vs busiest CTA's sum {mean['busiest_cta_sum_us']}")
    finally:
        ops.set_gemm_trace(None)
        ops.unregister_operand_bound(h1)
        ops.unregister_operand_bound(dz)
        ops.unregister_operand_bound(x0)
        ops.unregister_f16_twins(flat1)
        ops.unregister_f16_transposed(W2)
        ops.unregister_f16_twins(flat)
    os.makedirs(args.out, exist_ok=True)
    tag = "" if not args.lib else "_" + os.path.basename(os.path.dirname(os.path.abspath(args.lib)))
    with open(os.path.join(args.out, f"gemm_trace{tag}.json"), "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
