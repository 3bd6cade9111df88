"""The head partials of the fp16-form heads GEMM (gemm_wgmma_kernel<0,0,1,1,1,0>, head_partials_f16 in
csrc/wgmma_tile.cuh: a 3-pass fp16 GEMM per 64-column half on register-A wgmmas, the operand shift chosen per row)
against float64, on the kernel's own activations y: per row the error stays within 1e-5 of the row's sum of |y_k w_k|
(the scale any reordering of the dot product errs by) for activations of magnitude 1, 1e-6 and 300 under every
activation, at M = 32768 and at a ragged M, with one and with eight action outputs.  Three launches on the same inputs
(storing y twice, then not) give the same y and the same partials: outputs that changed from launch to launch were how
an earlier ring layout's race showed.  The same function runs in the persistent rollout;
tests/test_gpu_rollout_pipeline.py holds that it and the per-step launches give the same actions."""
import math

import numpy as np
import pytest
import torch

from tests.device_harness import ops_for

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("scale", [1.0, 1e-6, 300.0])
@pytest.mark.parametrize("act", ["elu", "relu", "tanh", "none"])
@pytest.mark.parametrize("M,A", [(32768, 8), (1000, 1), (4133, 8)])
def test_partials_against_float64(M, A, act, scale):
    ops = ops_for("3xtf32")
    dev = torch.device("cuda", 0)
    K = N = 512
    g = torch.Generator().manual_seed(M + 31 * A + 7 * len(act) + int(math.log10(scale) + 10))
    x = (torch.randn(M, K, generator=g) * scale).to(dev)
    W = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(dev).contiguous()
    b = (torch.randn(N, generator=g) * 0.1 * scale).to(dev)
    Wv = (torch.randn(N, generator=g) / math.sqrt(N)).to(dev)
    Wa = (torch.randn(A, N, generator=g) / math.sqrt(N)).to(dev).contiguous()
    P = ops.linear_heads_partials(N, A, ops.GEMM_TC_3XTF32)
    assert P == 8
    twins = torch.empty(2 * W.numel(), dtype=torch.float16, device=dev)
    bound = torch.full((1,), float(x.abs().max()), device=dev)
    ops.register_f16_twins(W.view(-1), twins)
    ops.register_operand_bound(x, bound)
    try:
        y = torch.full((M, N), float("nan"), device=dev)
        part = torch.full((P, M, ops.HEAD_PART_PAD), float("nan"), device=dev)
        ops.linear_act_heads_forward(x, W, b, y, ops.ACT[act], ops.GEMM_TC_3XTF32, Wv, Wa, part)
        y2 = torch.full_like(y, float("nan"))
        part2 = torch.full_like(part, float("nan"))
        ops.linear_act_heads_forward(x, W, b, y2, ops.ACT[act], ops.GEMM_TC_3XTF32, Wv, Wa, part2)
        part_ns = torch.full_like(part, float("nan"))
        ops.linear_act_heads_forward(x, W, b, None, ops.ACT[act], ops.GEMM_TC_3XTF32, Wv, Wa, part_ns)
        torch.cuda.synchronize()
    finally:
        ops.unregister_operand_bound(x)
        ops.unregister_f16_twins(W.view(-1))
    assert torch.equal(y, y2) and torch.equal(part, part2)
    assert torch.equal(part, part_ns)                      # storing y or not: the same partials
    assert torch.all(part[:, :, A + 1:] == 0)              # padding columns
    Wh = torch.cat([Wv.view(1, N), Wa]).double()
    yd = y.double().view(M, P, 64)
    ref = torch.einsum("mpk,apk->pma", yd, Wh.view(A + 1, P, 64))
    mag = torch.einsum("mpk,apk->pma", yd.abs(), Wh.abs().view(A + 1, P, 64))
    err = (part[:, :, :A + 1].double() - ref).abs()
    # the fp32 FMA form of the same partials, for the record
    f32 = torch.einsum("mpk,apk->pma", y.view(M, P, 64), Wh.float().view(A + 1, P, 64))
    err32 = (f32.double() - ref).abs()
    rel = (err / mag.clamp_min(1e-300)).max().item()
    print(f"M={M} A={A} {act} x{scale}: max |err| / sum|y w| = {rel:.3g} (fp32 einsum: "
          f"{(err32 / mag.clamp_min(1e-300)).max().item():.3g})")
    assert rel <= 1e-5, rel
    np.testing.assert_array_less(err.cpu().numpy(), (1e-5 * mag + 1e-30).cpu().numpy())
