"""The persistent wgmma GEMM (csrc/gemm_tc.cu): one CTA per SM walks the work items, ring slots and mbarrier phases run
on from one item to the next.  Checked here: results stay fp32-grade in every epilogue and both forms when a CTA runs
many items (M = 32768), exactly one, or the grid is smaller than the device; dW with a split-K sized to the SMs, the
last slice short; and, through the kernel's trace, that every work item ran exactly once on the CTA the fixed schedule
gives it, with tracing changing no bit of the output."""
import math

import numpy as np
import pytest
import torch

from tests.device_harness import Registered, g, ops_for, tc_dev  # noqa: F401  (tc_dev: the `dev` fixture)

pytestmark = pytest.mark.gpu


# many items per CTA; ragged N and K; M < 128 (one item); fewer items than SMs; a few more items than SMs
SHAPES = [(32768, 512, 512), (1000, 72, 200), (100, 128, 64), (4096, 256, 192), (17000, 128, 128)]


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("form", ["fp16", "tf32"])
def test_forward_epilogues_and_dx(dev, M, N, K, form):
    ops = ops_for()
    eng = ops.GEMM_TC_3XTF32
    if form == "fp16" and K % 64 != 0:
        pytest.skip("the fp16 form takes K in multiples of 64")
    x = torch.randn(M, K, generator=g(40)).to(dev)
    W = (torch.randn(N, K, generator=g(41)) / math.sqrt(K)).to(dev).contiguous()
    b = (torch.randn(N, generator=g(42)) * 0.1).to(dev)
    r = torch.randn(M, N, generator=g(43)).to(dev)
    dz = (torch.randn(M, N, generator=g(44)) / M).to(dev)
    xa = torch.nn.functional.elu(x)
    A = 6
    Wv = (torch.randn(N, generator=g(45)) * 0.1).to(dev)
    Wa = (torch.randn(A, N, generator=g(46)) * 0.1).to(dev).contiguous()
    P = ops.linear_heads_partials(N, A, eng)
    ws = torch.empty(ops.linear_backward_workspace_bytes(M, N, K) // 4 + 4, device=dev)

    def run():
        y, yr, yh = (torch.zeros(M, N, device=dev) for _ in range(3))
        ops.linear_act_forward(x, W, b, y, ops.ACT["elu"], eng)
        ops.linear_residual_forward(x, W, b, r, yr, eng)
        part = None
        if P:
            part = torch.zeros(P, M, ops.HEAD_PART_PAD, device=dev)
            ops.linear_act_heads_forward(x, W, b, yh, ops.ACT["elu"], eng, Wv, Wa, part)
        dx = torch.zeros(M, K, device=dev)
        ops.linear_backward(dz, xa, W, ops.ACT["elu"], None, dx, None, eng, ws)
        torch.cuda.synchronize()
        return y, yr, yh, part, dx

    if form == "fp16":
        with Registered(W, x, dz):
            y, yr, yh, part, dx = run()
    else:
        y, yr, yh, part, dx = run()
    z = torch.nn.functional.linear(x.double(), W.double(), b.double())
    ref = torch.nn.functional.elu(z)
    np.testing.assert_allclose(y.cpu().numpy(), ref.cpu().numpy(), atol=1e-5, rtol=1e-5)
    np.testing.assert_allclose(yr.cpu().numpy(), (z + r.double()).cpu().numpy(), atol=1e-5, rtol=1e-5)
    if P:
        assert torch.equal(yh, y)
        heads = ref @ torch.cat([Wv.view(1, N), Wa]).double().t()
        np.testing.assert_allclose(part.sum(0)[:, :A + 1].cpu().numpy(), heads.cpu().numpy(), atol=1e-5, rtol=1e-5)
    dref = (dz.double() @ W.double()) * torch.where(xa > 0, torch.ones_like(xa), xa + 1).double()
    np.testing.assert_allclose(dx.cpu().numpy(), dref.cpu().numpy(), atol=1e-5, rtol=1e-4)


# dW [N, K] over M: 8 slices of 16 tiles, 32 of 4, a short last slice (17000 = 31 x 544 + 136), more tiles than SMs (no
# split, 144 items on the H100's 132 SMs), one tile with ragged edges
@pytest.mark.parametrize("M,N,K", [(32768, 512, 512), (32768, 512, 64), (17000, 512, 128), (2048, 1536, 1536), (1000, 72, 200)])
def test_dw_with_device_sized_split_k(dev, M, N, K):
    ops = ops_for()
    dz = (torch.randn(M, N, generator=g(50)) / M).to(dev)
    x = torch.randn(M, K, generator=g(51)).to(dev)
    W = (torch.randn(N, K, generator=g(52)) / math.sqrt(K)).to(dev)
    tiles = -(-N // 128) * -(-K // 128)
    splits = ops.linear_backward_splits(M, N, K)
    assert tiles * splits <= max(ops.sm_count(), tiles)
    ws = torch.empty(ops.linear_backward_workspace_bytes(M, N, K) // 4 + 4, device=dev)
    dW = torch.zeros(N, K, device=dev)
    ops.linear_backward(dz, x, W, ops.ACT["none"], dW, None, None, ops.GEMM_TC_3XTF32, ws)
    ref = dz.double().t() @ x.double()
    np.testing.assert_allclose(dW.cpu().numpy(), ref.cpu().numpy(), atol=1e-5, rtol=1e-4)


@pytest.mark.parametrize("M,N,K", [(32768, 512, 512), (1000, 72, 200), (100, 128, 64)])
def test_trace_shows_every_item_once_on_its_cta(dev, M, N, K):
    ops = ops_for()
    x = torch.randn(M, K, generator=g(60)).to(dev)
    W = (torch.randn(N, K, generator=g(61)) / math.sqrt(K)).to(dev).contiguous()
    b = (torch.randn(N, generator=g(62)) * 0.1).to(dev)
    y0, y1 = torch.zeros(M, N, device=dev), torch.zeros(M, N, device=dev)
    ops.linear_act_forward(x, W, b, y0, ops.ACT["elu"], ops.GEMM_TC_3XTF32)
    items = -(-M // 128) * -(-N // 128)
    trace = torch.zeros((items + 3) * ops.GEMM_TRACE_WORDS, dtype=torch.int64, device=dev)
    ops.set_gemm_trace(trace)
    try:
        ops.linear_act_forward(x, W, b, y1, ops.ACT["elu"], ops.GEMM_TC_3XTF32)
        torch.cuda.synchronize()
        small = torch.zeros(ops.GEMM_TRACE_WORDS, dtype=torch.int64, device=dev)
        if items > 1:
            ops.set_gemm_trace(small)
            with pytest.raises(Exception, match="trace buffer too small"):
                ops.linear_act_forward(x, W, b, y1, ops.ACT["elu"], ops.GEMM_TC_3XTF32)
    finally:
        ops.set_gemm_trace(None)
    assert torch.equal(y0, y1)
    t = trace.cpu().view(-1, ops.GEMM_TRACE_WORDS)
    assert bool((t[items:] == 0).all())
    t = t[:items]
    grid = min(items, ops.sm_count())          # one CTA per SM: 225 KB of shared memory each
    assert t[:, 1].tolist() == [i % grid for i in range(items)]
    # consumer: begun <= first stage landed <= mainloop done <= epilogue done; producer: first load <= last load
    assert bool((t[:, 2] > 0).all()) and bool((t[:, 2:5] <= t[:, 3:6]).all()) and bool((t[:, 6] <= t[:, 7]).all())
    # a CTA's items follow each other, and all of them ran on the CTA's SM
    for cta in range(min(grid, 4)):
        mine = t[cta::grid]
        assert bool((mine[:-1, 5] <= mine[1:, 2]).all()) and mine[:, 0].unique().numel() == 1
    assert bool((t[:grid, 8] > 0).all()) and bool((t[:grid, 8] <= t[:grid, 9]).all()) and bool((t[grid:, 8] == 0).all())
