"""The fp16-form mainloops of the wgmma GEMM (csrc/gemm_tc.cu) take the A operand from registers and keep two groups of
wgmmas in flight: gemm_wgmma_kernel's fp16 forward and dX, and gemm_dw_f16_kernel.  Checked against float64 products
at the fp32-grade bound of test_fp16_split_engine_is_fp32_grade (3e-6 of the largest output): one 64-k stage, two,
an odd number, eight; ragged M and N; enough work items per CTA (M = 32768) that every A / B ring slot and mbarrier
phase wraps many times; activations of magnitude 1e-6 and 300.  The same call run twice gives the same bits."""
import math

import pytest
import torch

from tests.device_harness import g, ops_for, tc_dev, tc_dw  # noqa: F401  (tc_dev: the `dev` fixture)

pytestmark = pytest.mark.gpu


# (M, N, K, amplitude of the activations): K / 64 stages of the forward, N / 64 of dX
FWD_CASES = [(300, 512, 64, 1.0), (2048, 512, 128, 1.0), (1000, 200, 192, 1.0), (32768, 512, 512, 1.0),
             (4096, 256, 320, 1e-6), (1000, 384, 128, 300.0)]


@pytest.mark.parametrize("M,N,K,amp", FWD_CASES)
def test_fp16_forward_and_dx_against_fp64(dev, M, N, K, amp):
    ops = ops_for()
    x = (torch.randn(M, K, generator=g(270)) * amp).to(dev)
    W = (torch.randn(N, K, generator=g(271)) / math.sqrt(K)).to(dev).contiguous()
    b = (torch.randn(N, generator=g(272)) * 0.1 * amp).to(dev)
    dz = (torch.randn(M, N, generator=g(273)) * amp).to(dev)
    xa = torch.nn.functional.elu(torch.randn(M, K, generator=g(274))).to(dev)
    twins = torch.empty(2 * W.numel(), dtype=torch.float16, device=dev)
    twinsT = torch.empty(2 * W.numel(), dtype=torch.float16, device=dev)
    bound = torch.full((1,), float(x.abs().max()), device=dev)
    dbound = torch.full((1,), float(dz.abs().max()), device=dev)
    ops.register_f16_twins(W.view(-1), twins)
    ops.register_f16_transposed(W, twinsT)
    ops.register_operand_bound(x, bound)
    ops.register_operand_bound(dz, dbound)
    try:
        outs, dxs = [], []
        ws = torch.empty(ops.linear_backward_workspace_bytes(M, N, K) // 4 + 4, device=dev)
        for _ in range(2):
            out = torch.full((M, N), float("nan"), device=dev)
            ops.linear_act_forward(x, W, b, out, ops.ACT["none"], ops.GEMM_TC_3XTF32)
            dx = torch.full((M, K), float("nan"), device=dev)
            ops.linear_backward(dz, xa, W, ops.ACT["elu"], None, dx, None, ops.GEMM_TC_3XTF32, ws)
            torch.cuda.synchronize()
            outs.append(out)
            dxs.append(dx)
    finally:
        ops.unregister_operand_bound(dz)
        ops.unregister_operand_bound(x)
        ops.unregister_f16_transposed(W)
        ops.unregister_f16_twins(W.view(-1))
    ref = torch.nn.functional.linear(x.double(), W.double(), b.double())
    err, scale = float((outs[0].double() - ref).abs().max()), float(ref.abs().max())
    assert err < 3e-6 * scale, (err, scale)
    dref = (dz.double() @ W.double()) * torch.where(xa > 0, torch.ones_like(xa), xa + 1).double()
    derr, dscale = float((dxs[0].double() - dref).abs().max()), float(dref.abs().max())
    assert derr < 3e-6 * dscale, (derr, dscale)
    assert torch.equal(outs[0], outs[1]) and torch.equal(dxs[0], dxs[1])


# (batch M, N, K, scale of dz, scale of x): batch / 32 stages in all, cut into split-K slices by choose_splits -- 96 is
# three stages, 1000 a short last stage, 17000 a short last slice
DW_CASES = [(96, 512, 512, 1.0, 1.0), (1000, 200, 72, 1.0, 1.0), (17000, 512, 128, 1.0, 1.0),
            (32768, 512, 512, 1.0, 1.0), (4096, 256, 192, 1e-6, 300.0)]


@pytest.mark.parametrize("M,N,K,sz,sx", DW_CASES)
def test_fp16_dw_against_fp64(dev, M, N, K, sz, sx):
    dz = (torch.randn(M, N, generator=g(275)) * sz).to(dev)
    x = (torch.nn.functional.elu(torch.randn(M, K, generator=g(276))) * sx).to(dev)
    bounds = (float(dz.abs().max()), float(x.abs().max()))
    dw = tc_dw(dev, dz, x, bounds)
    ref = dz.double().t() @ x.double()
    top = float((dz.double().abs().t() @ x.double().abs()).max())
    err = float((dw.double() - ref).abs().max())
    assert err < 3e-6 * top, (err, top)
    assert torch.equal(dw, tc_dw(dev, dz, x, bounds))
