"""dW / dX micro-benchmark at the cfg-2 learner shapes (CUDA events, L2 flushed between launches). GPU box only."""
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from sample_factory_b200 import ops

dev = torch.device("cuda", 0)
ops.bind_device(dev)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
eng = ops.ENGINES["3xtf32"]


def timeit(fn, reps=12):
    fn(); torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2] * 1e3


for (M, N, K) in [(32768, 512, 512), (32768, 512, 64)]:
    flat = torch.randn(N * K, device=dev) / math.sqrt(K)
    W = flat.view(N, K)
    x = torch.randn(M, K, device=dev)
    dz = torch.randn(M, N, device=dev)
    dW, dx = torch.empty(N, K, device=dev), torch.empty(M, K, device=dev)
    ws = torch.empty(ops.linear_backward_workspace_bytes(M, N, K) // 4 + 4, device=dev)
    y = torch.empty(M, N, device=dev)
    b = torch.zeros(N, device=dev)
    t_fw = timeit(lambda: ops.linear_act_forward(x, W, b, y, ops.ACT["elu"], eng))
    print(f"M={M} N={N} K={K}: fwd {t_fw:.1f} us ({2*M*N*K/t_fw/1e6:.0f} TFLOP/s)")
    t_dw = timeit(lambda: ops.linear_backward(dz, x, W, ops.ACT["elu"], dW, None, None, eng, ws))
    t_dx = timeit(lambda: ops.linear_backward(dz, x, W, ops.ACT["elu"], None, dx, None, eng, ws))
    print(f"M={M} N={N} K={K}: dW {t_dw:.1f} us ({2*M*N*K/t_dw/1e6:.0f} TFLOP/s)  dX {t_dx:.1f} us ({2*M*N*K/t_dx/1e6:.0f} TFLOP/s)")
    if K % 64 == 0:
        twins = torch.empty(2 * N * K, dtype=torch.float16, device=dev)
        twinsT = torch.empty(2 * N * K, dtype=torch.float16, device=dev)
        ops.register_f16_twins(flat, twins); ops.register_f16_transposed(W, twinsT)
        bx = torch.full((1,), float(x.abs().max()), device=dev); bz = torch.full((1,), float(dz.abs().max()), device=dev)
        ops.register_operand_bound(x, bx); ops.register_operand_bound(dz, bz)
        t_fw16 = timeit(lambda: ops.linear_act_forward(x, W, b, y, ops.ACT["elu"], eng))
        t_dx16 = timeit(lambda: ops.linear_backward(dz, x, W, ops.ACT["elu"], None, dx, None, eng, ws))
        print(f"M={M} N={N} K={K}: fp16-split fwd {t_fw16:.1f} us ({2*M*N*K/t_fw16/1e6:.0f} TFLOP/s)  dX {t_dx16:.1f} us ({2*M*N*K/t_dx16/1e6:.0f} TFLOP/s)")
        ops.unregister_operand_bound(x); ops.unregister_operand_bound(dz)
        ops.unregister_f16_transposed(W); ops.unregister_f16_twins(flat)
    ref = dz.double().t() @ x.double()
    print("   dW max abs err vs fp64:", float((dW.double() - ref).abs().max()), "of max", float(ref.abs().max()))
    # dW with both operands' bounds registered: the fp16 form (dz^T and x split in the kernel)
    bx = torch.full((1,), float(x.abs().max()), device=dev); bz = torch.full((1,), float(dz.abs().max()), device=dev)
    ops.register_operand_bound(x, bx); ops.register_operand_bound(dz, bz)
    t_dw16 = timeit(lambda: ops.linear_backward(dz, x, W, ops.ACT["elu"], dW, None, None, eng, ws))
    ops.unregister_operand_bound(x); ops.unregister_operand_bound(dz)
    print(f"M={M} N={N} K={K}: fp16-split dW {t_dw16:.1f} us ({2*M*N*K/t_dw16/1e6:.0f} TFLOP/s)")
    print("   fp16-split dW max abs err vs fp64:", float((dW.double() - ref).abs().max()), "of max", float(ref.abs().max()))
