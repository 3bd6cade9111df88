"""The persistent rollout kernel (csrc/rollout_fused.cu: producer warpgroup, TMA ring, fp16 weight twins and h1 handed
over already split) against the per-step launches with the fused step tail, at the shapes the kernel's ring and
decomposition distinguish: the bench shape in both operand forms, clusters of 1 / 2 / 4 CTAs, one to four layer-1
stages, partial row blocks, odd step counts (ring phases), one action, weights that move between rollouts, and a
CUDA-graph replay.  Comparison rule of device_harness.compare_rollout_runs: everything bit-identical except logits /
values / log-probs (2e-6)."""
import os
import subprocess
import sys

import pytest

from tests.device_harness import check_persistent_rollout

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_bench_shape_fp16_form():
    check_persistent_rollout(N=4096, T=32, form=1)


def test_bench_shape_tf32_form():
    """SFB200_TC_F16=0 is read once per process: the same check in a fresh one"""
    code = ("import sys; sys.path.insert(0, sys.argv[1]); from tests.device_harness import check_persistent_rollout; "
            "check_persistent_rollout(N=4096, T=32, form=0); print('ok')")
    env = dict(os.environ, SFB200_TC_F16="0")
    res = subprocess.run([sys.executable, "-c", code, ROOT], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0 and "ok" in res.stdout, res.stdout[-3000:] + res.stderr[-3000:]


@pytest.mark.parametrize("form", ["fp16", "tf32"])
@pytest.mark.parametrize("act", ["relu", "tanh"])
def test_activations(act, form):
    """rollout_mlp2_tape_kernel<ACT, F16> for ReLU (unbounded: the fp16 form splits h1 by a bound that grows with the
    weights) and tanh (h1 bound capped at 1 by linear_out_bound); the tf32 form in a fresh process, as above"""
    if form == "fp16":
        check_persistent_rollout(N=1000, T=5, form=1, nonlinearity=act)
        return
    code = ("import sys; sys.path.insert(0, sys.argv[1]); from tests.device_harness import check_persistent_rollout; "
            f"check_persistent_rollout(N=1000, T=5, form=0, nonlinearity={act!r}); print('ok')")
    env = dict(os.environ, SFB200_TC_F16="0")
    res = subprocess.run([sys.executable, "-c", code, ROOT], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0 and "ok" in res.stdout, res.stdout[-3000:] + res.stderr[-3000:]


@pytest.mark.parametrize("hidden", [128, 256])
def test_cluster_sizes(hidden):
    check_persistent_rollout(hidden=hidden, N=1000, T=5, form=1)


@pytest.mark.parametrize("obs_dim,form", [(32, 0), (96, 0), (128, 1)])
def test_obs_dims(obs_dim, form):
    """K1 = 32 / 96 take the tf32 form (stages of 32 k); the per-step layer 2 would take the fp16 form from the twins, so
    those run a model without twins, where both paths split in tf32.  K1 = 128: two fp16 layer-1 stages."""
    check_persistent_rollout(obs_dim=obs_dim, N=1000, T=5, form=form, normalize=form == 1)


@pytest.mark.parametrize("N", [1000, 100])
def test_partial_row_blocks(N):
    check_persistent_rollout(N=N, T=6, form=1)


@pytest.mark.parametrize("T", [1, 3])
def test_odd_step_counts(T):
    check_persistent_rollout(N=1000, T=T, rollouts=3, form=1)


def test_one_action():
    check_persistent_rollout(num_actions=1, N=1000, T=5, form=1)


def test_weights_move_between_rollouts():
    check_persistent_rollout(N=1000, T=8, rollouts=3, train=True, form=1)


def test_cuda_graph_replay():
    check_persistent_rollout(N=1000, T=6, rollouts=3, graph=True, form=1)
