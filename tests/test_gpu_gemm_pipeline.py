"""The wgmma GEMM mainloop (csrc/gemm_tc.cu): the fp16 form takes its weight operand from the registered fp16 twins,
the tf32 form splits both operands itself (MN-major tiles transposed on the way), and the split of one stage overlaps
the wgmmas of the previous one.  Checked here: the twins really are the operand, they follow every weight write, and
the pipeline's edge cases (one stage, an odd stage count, an uneven split-K chunk, partial tiles) stay fp32-grade."""
import math

import numpy as np
import pytest
import torch

from tests.device_harness import Registered, g, ops_for, tc_dev  # noqa: F401  (tc_dev: the `dev` fixture)

pytestmark = pytest.mark.gpu


def torch_twins(w):
    """[hi | lo] as the kernels define them: hi = fp16(w * 2^8), lo = fp16((w * 2^8 - hi) * 2^11)"""
    v = w.float() * 256.0
    hi = v.half()
    lo = ((v - hi.float()) * 2048.0).half()
    return hi, lo


def test_fp16_form_reads_the_weight_twins(dev, monkeypatch):
    """Perturbing one element W[n][k] of the hi twin changes the forward output in column n only, and the same element
    of the transposed hi twin changes dX in column k only: the kernel's B operand is the twin, not a re-split of W."""
    monkeypatch.delenv("SFB200_CHECK_F16", raising=False)
    ops = ops_for()
    M, N, K = 512, 256, 192
    x = torch.randn(M, K, generator=g(1)).to(dev)
    W = (torch.randn(N, K, generator=g(2)) / math.sqrt(K)).to(dev).contiguous()
    b = torch.zeros(N, device=dev)
    dz = torch.randn(M, N, generator=g(3)).to(dev)
    ws = torch.empty(ops.linear_backward_workspace_bytes(M, N, K) // 4 + 4, device=dev)
    n, k = 77, 131
    W0 = W.clone()
    with Registered(W, x, dz) as r:
        y0 = torch.empty(M, N, device=dev)
        ops.linear_act_forward(x, W, b, y0, ops.ACT["none"], ops.GEMM_TC_3XTF32)
        dx0 = torch.empty(M, K, device=dev)
        ops.linear_backward(dz, x, W, ops.ACT["none"], None, dx0, None, ops.GEMM_TC_3XTF32, ws)

        r.twins[n * K + k] += 64.0                      # hi twin of W[n][k] (forward operand)
        y1 = torch.empty(M, N, device=dev)
        ops.linear_act_forward(x, W, b, y1, ops.ACT["none"], ops.GEMM_TC_3XTF32)
        changed = (y1 != y0).any(0).nonzero().view(-1).tolist()
        assert changed == [n], changed

        r.twinsT[k * N + n] += 64.0                     # the same element in the transposed twin (dX operand)
        dx1 = torch.empty(M, K, device=dev)
        ops.linear_backward(dz, x, W, ops.ACT["none"], None, dx1, None, ops.GEMM_TC_3XTF32, ws)
        changed = (dx1 != dx0).any(0).nonzero().view(-1).tolist()
        assert changed == [k], changed
    assert torch.equal(W, W0)


def _check_model_twins(model):
    for name, p in model.params.items():
        off = model._slices[name][0]
        n = p.numel()
        hi, lo = torch_twins(p.reshape(-1))
        assert torch.equal(model.f16_twins[off: off + n], hi), name
        assert torch.equal(model.f16_twins[model.flat.numel() + off: model.flat.numel() + off + n], lo), name
    for name, tT in model.f16_T.items():
        W = model.params[name]
        hi, lo = torch_twins(W.t().contiguous().view(-1))
        assert torch.equal(tT[: W.numel()], hi) and torch.equal(tT[W.numel():], lo), name


def test_twins_follow_every_weight_write(dev):
    """The twins carry the weights into the fp16-form GEMMs, so they must equal torch's split of the current weights
    after every API that writes weights: Adam and LAMB learner steps, weights_changed, load_state_dict,
    copy_weights_from."""
    from sample_factory_b200.cfg import default_cfg
    from sample_factory_b200.envs import TapeVecEnv
    from sample_factory_b200.learner import Learner
    from sample_factory_b200.model import ModelSpec, PolicyModel
    from sample_factory_b200.sampler import DeviceSampler
    from sample_factory_b200.trajectory import alloc_trajectory_tensors

    ops = ops_for()
    N, T = 256, 8
    spec = ModelSpec(64, 8, [128, 128])
    for optimizer in ("adam", "lamb"):
        cfg = default_cfg()
        cfg.use_rnn, cfg.async_rl = False, False
        cfg.encoder_mlp_layers = [128, 128]
        cfg.rollout, cfg.recurrence, cfg.batch_size, cfg.num_batches_per_epoch = T, 1, N * T // 2, 2
        cfg.optimizer = optimizer
        model = PolicyModel(spec, dev)
        assert model.f16_twins is not None
        traj = alloc_trajectory_tensors(64, 8, N, T, dev)
        tape = torch.randn(T + 1, N, 64, generator=g(10)).to(dev)
        sampler = DeviceSampler(cfg, TapeVecEnv(tape, 8), model, traj, engine=ops.GEMM_TC_3XTF32)
        learner = Learner(cfg, model, N, engine=ops.GEMM_TC_3XTF32)
        sampler.reset()
        sampler.rollout()
        learner.train(traj)
        torch.cuda.synchronize()
        assert model.f16_T, "the learner registers transposed twins"
        _check_model_twins(model)

    model.flat.mul_(0.5)
    model.weights_changed()
    _check_model_twins(model)

    other = PolicyModel(spec, dev)
    with torch.no_grad():
        other.flat.copy_(torch.randn(other.flat.shape, generator=g(11)).to(dev) * 0.1)
    other.weights_changed()
    model.load_state_dict({k: v.detach().clone() for k, v in other.params.items()}, strict=False)
    assert all(torch.equal(model.params[k], other.params[k]) for k in model.names)
    _check_model_twins(model)

    snap = model.inference_copy()
    model.flat.mul_(-1.0)
    model.weights_changed()
    snap.copy_weights_from(model)
    _check_model_twins(snap)


def _fp64_forward(x, W, b, act):
    z = torch.nn.functional.linear(x.double(), W.double(), b.double())
    return torch.nn.functional.elu(z) if act == "elu" else z


# one 64-k stage, an odd stage count (3 and 5), M not a multiple of 128, N < 128, N not a multiple of 128
@pytest.mark.parametrize("M,N,K", [(300, 64, 64), (1000, 96, 192), (129, 200, 320), (4096, 512, 64)])
@pytest.mark.parametrize("form", ["fp16", "tf32"])
def test_forward_and_dx_pipeline_edges(dev, M, N, K, form):
    ops = ops_for()
    x = torch.randn(M, K, generator=g(20)).to(dev)
    W = (torch.randn(N, K, generator=g(21)) / math.sqrt(K)).to(dev).contiguous()
    b = (torch.randn(N, generator=g(22)) * 0.1).to(dev)
    dz = (torch.randn(M, N, generator=g(23)) / M).to(dev)
    xa = torch.nn.functional.elu(x)
    ws = torch.empty(ops.linear_backward_workspace_bytes(M, N, K) // 4 + 4, device=dev)

    def run():
        y = torch.empty(M, N, device=dev)
        ops.linear_act_forward(x, W, b, y, ops.ACT["elu"], ops.GEMM_TC_3XTF32)
        dx = torch.empty(M, K, device=dev)
        ops.linear_backward(dz, xa, W, ops.ACT["elu"], None, dx, None, ops.GEMM_TC_3XTF32, ws)
        return y, dx

    if form == "fp16":
        with Registered(W, x, dz):
            y, dx = run()
        y_tf32, dx_tf32 = run()
        assert not torch.equal(y, y_tf32), "the fp16 form did not run"
        # (dX reduces over N: the fp16 form needs N % 64 == 0, other widths keep the tf32 form)
        assert torch.equal(dx, dx_tf32) == (N % 64 != 0)
    else:
        y, dx = run()
    ref = _fp64_forward(x, W, b, "elu")
    np.testing.assert_allclose(y.cpu().numpy(), ref.cpu().numpy(), atol=1e-5, rtol=1e-5)
    dref = (dz.double() @ W.double()) * torch.where(xa > 0, torch.ones_like(xa), xa + 1).double()
    np.testing.assert_allclose(dx.cpu().numpy(), dref.cpu().numpy(), atol=1e-5, rtol=1e-4)


# dW = dz^T x on the tf32 form (both operands MN-major, split-K): one 32-k stage, odd stage counts, uneven last chunk
@pytest.mark.parametrize("M,N,K", [(32, 64, 64), (96, 130, 40), (1000, 70, 200), (4000, 512, 64), (32768, 512, 512)])
def test_dw_pipeline_edges(dev, M, N, K):
    ops = ops_for()
    dz = (torch.randn(M, N, generator=g(30)) / M).to(dev)
    x = torch.randn(M, K, generator=g(31)).to(dev)
    W = (torch.randn(N, K, generator=g(32)) / math.sqrt(K)).to(dev)
    ws = torch.empty(ops.linear_backward_workspace_bytes(M, N, K) // 4 + 4, device=dev)
    dW = torch.empty(N, K, device=dev)
    ops.linear_backward(dz, x, W, ops.ACT["none"], dW, None, None, ops.GEMM_TC_3XTF32, ws)
    ref = dz.double().t() @ x.double()
    np.testing.assert_allclose(dW.cpu().numpy(), ref.cpu().numpy(), atol=1e-5, rtol=1e-4)
