"""dW = dz^T . x in the fp16 form (gemm_dw_f16_kernel, csrc/gemm_tc.cu): when both MN-major operands lie in buffers with
registered bounds, the kernel splits both into scaled fp16 hi / lo halves itself and runs the fp16 MMAs with the
transpose bits set.  Checked here: the error against an fp64 product stays fp32-grade (below 3e-6 of the largest entry of
|dz|^T |x|, the scale a sum of 32768 products rounds at, and within 2x of the tf32 form's error on the same inputs) at the learner's shapes, at ragged and one-stage sizes, with operands
scaled far from 1 and with a bound much looser than the data; the kernel really runs (its result differs from the tf32
form's); a learner step of the headline model runs it for both dW GEMMs; and the bounds the learner derives for the
gradients of the lower hidden layers hold."""
import os
import subprocess
import sys

import pytest
import torch

from tests.device_harness import g, mlp_learner, ops_for, tc_dev, tc_dw  # noqa: F401  (tc_dev: the `dev` fixture)

pytestmark = pytest.mark.gpu


# dW2 and dW1 at the learner's shapes, a short last split-K slice (17000), one 32-k stage, ragged tiles; operands scaled
# by 1e-6 and by 300; a bound 64x looser than the data.  (M, N, K, scale of dz, scale of x, bound / max|operand|)
CASES = [(32768, 512, 512, 1.0, 1.0, 1.0), (32768, 512, 64, 1.0, 1.0, 1.0), (17000, 512, 128, 1.0, 1.0, 1.0),
         (32, 64, 64, 1.0, 1.0, 1.0), (1000, 72, 200, 1.0, 1.0, 1.0), (4096, 256, 192, 1e-6, 1.0, 1.0),
         (4096, 256, 192, 1.0, 300.0, 1.0), (8192, 512, 512, 1e-6, 300.0, 1.0), (32768, 512, 512, 1.0, 1.0, 64.0)]


@pytest.mark.parametrize("M,N,K,sz,sx,looser", CASES)
def test_dw_f16_error_against_fp64(dev, M, N, K, sz, sx, looser):
    dz = (torch.randn(M, N, generator=g(70)) * sz).to(dev)
    x = (torch.nn.functional.elu(torch.randn(M, K, generator=g(71))) * sx).to(dev)
    dw16 = tc_dw(dev, dz, x, (float(dz.abs().max()) * looser, float(x.abs().max()) * looser))
    dw32 = tc_dw(dev, dz, x)
    ref = dz.double().t() @ x.double()
    top = float((dz.double().abs().t() @ x.double().abs()).max())
    err16 = float((dw16.double() - ref).abs().max())
    err32 = float((dw32.double() - ref).abs().max())
    assert not torch.equal(dw16, dw32), "the fp16 dW form did not run"
    assert err16 < 3e-6 * top, (err16, top)
    assert err16 <= 2.0 * err32, (err16, err32)


def test_dw_f16_needs_both_bounds(dev):
    """one operand without a bound keeps the tf32 form (bit for bit)"""
    ops = ops_for()
    M, N, K = 4096, 256, 128
    dz = torch.randn(M, N, generator=g(72)).to(dev)
    x = torch.randn(M, K, generator=g(73)).to(dev)
    dw32 = tc_dw(dev, dz, x)
    bound = torch.full((1,), float(dz.abs().max()), device=dev)
    ops.register_operand_bound(dz, bound)
    try:
        only_dz = tc_dw(dev, dz, x)
    finally:
        ops.unregister_operand_bound(dz)
    assert torch.equal(only_dz, dw32)


_PROFILE_STEP = """
import torch
from torch.profiler import ProfilerActivity, profile
from tests.device_harness import mlp_learner
dev = torch.device("cuda", 0)
from sample_factory_b200 import ops
ops.bind_device(dev)
model, sampler, learner, traj = mlp_learner(dev, (512, 512))
sampler.rollout()
learner.train(traj)
sampler.rollout()
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    learner.train(traj)
    torch.cuda.synchronize()
print(learner.cfg.num_epochs * learner.cfg.num_batches_per_epoch)
for ev in prof.events():
    if ev.device_type == torch.autograd.DeviceType.CUDA:
        print(ev.name)
"""


def test_learner_runs_dw_f16_for_both_layers(dev):
    """the headline model (two hidden layers of 512): every dW of a learner step takes the fp16 form.  (The profiled step
    runs in a process of its own: a profiler session leaves state behind that other tests' profiles would meet.)"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-c", _PROFILE_STEP], cwd=root, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-3000:]
    lines = out.stdout.splitlines()
    minibatches, names = int(lines[0]), lines[1:]
    n_dw16 = sum("gemm_dw_f16_kernel" in n for n in names)
    n_dw32 = sum("gemm_wgmma_kernel<true, true, true, false, false, false>" in n for n in names)
    assert n_dw16 == 2 * minibatches, names       # dW2 and dW1 per minibatch
    assert n_dw32 == 0


def test_hidden_gradient_bounds_hold(dev):
    """after several learner steps, |dz[i]| <= its bound, and the bound is bound(dz[i+1]) * max_k sum_n |W_{i+1}[n][k]|
    within 1.001 (three hidden layers: a chain of two products)"""
    model, sampler, learner, traj = mlp_learner(dev, (256, 256, 256))
    L = 3
    for _ in range(3):
        sampler.rollout()
        learner.train(traj)
    torch.cuda.synchronize()
    bounds = learner.dz_bound.view(L, 4)[:, 0].double().cpu()
    Ws = [w.double().cpu() for w, _ in model.hidden_layers()]
    for i in range(L - 1):
        dz = learner.dz[i]
        assert float(dz.abs().max()) <= float(bounds[i]), (i, float(dz.abs().max()), float(bounds[i]))
        expect = float(bounds[i + 1]) * float(Ws[i + 1].abs().sum(0).max())
        assert expect <= float(bounds[i]) <= 1.001 * expect, (i, float(bounds[i]), expect)
    assert float(learner.dz[L - 1].abs().max()) <= float(bounds[L - 1])
    assert bool((learner.dz_bound.view(L, 4)[:, 1:3] == 0).all()), "scratch words left non-zero"
    assert bool((model.grad_fac.view(L, 4)[:, 1:3] == 0).all()), "scratch words left non-zero"
