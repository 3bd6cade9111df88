"""The persistent rollout kernel (csrc/rollout_fused.cu) holds one row block per cluster for the whole rollout, so a grid
that needs more clusters than the device holds at once runs its last clusters as a second wave, after the first ones
have finished: the kernel then takes two rollouts' time.  At the bench shape the launch must fit in one wave."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_bench_shape_runs_in_one_wave():
    from sample_factory_b200 import ops

    dev = torch.device("cuda", 0)
    ops.bind_device(dev)
    if not ops.tc_available():
        pytest.skip("wgmma engine not available")
    # 4096 envs, MLP 64 -> 512 -> 512 ELU, 8 actions: clusters of two CTAs over 64-row blocks
    needed, resident = ops.rollout_occupancy(4096, 64, 512, 512, 8, ops.GEMM_TC_3XTF32, ops.ACT["elu"])
    assert needed == 64
    assert needed <= resident, f"{needed} clusters needed, {resident} resident at once: a second wave"
