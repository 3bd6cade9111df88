"""tools/feature_bench.py without a GPU: the workload table, the feature every variant's argv and env select, and the
refusal to run without a CUDA device."""
import ast
import glob
import os
import subprocess
import sys
from types import SimpleNamespace

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

from tools import feature_bench as fb  # noqa: E402

WORKLOADS = ["batched_tensor_env", "dict_obs", "mixed_tuple", "nofc", "resnet", "rnn_layers", "separate_rnn", "wide_heads"]
VARIANTS = [(w, v) for w in WORKLOADS for v in fb.WORKLOADS[w].variants]


def test_list_names_the_eight_workloads(capsys):
    fb.main(["--list"])
    listed = [line.split(":")[0] for line in capsys.readouterr().out.splitlines()]
    assert listed == WORKLOADS
    assert sum(len(w.order or w.variants) for w in fb.WORKLOADS.values()) == 25


def cfg_of(workload, variant, tmp_path):
    from sample_factory_b200.cfg import parse_full_cfg, parse_sf_args

    argv = fb.full_argv(f"{workload}_{variant.label}", variant.argv, str(tmp_path))
    parser, _ = parse_sf_args(argv)
    return parse_full_cfg(parser, argv)


def env_of(variant, monkeypatch):
    """the variant's env factory with TapeVecEnv replaced by a record of its arguments (a TapeVecEnv needs a device tape)"""
    monkeypatch.setattr(fb, "tape_env", lambda rows, n, width, seed, num_actions, uint8=False, **kw: SimpleNamespace(
        num_agents=n, obs_dim=width, num_actions=num_actions, uint8=uint8, **kw))
    return variant.env()


@pytest.mark.parametrize("workload,variant", VARIANTS, ids=[f"{w}-{v.label}" for w, v in VARIANTS])
def test_variant_selects_its_feature(workload, variant, tmp_path, monkeypatch):
    cfg, env, label = cfg_of(workload, variant, tmp_path), env_of(variant, monkeypatch), variant.label
    assert cfg.gemm_engine == "auto" and cfg.train_dir == str(tmp_path) and not cfg.async_rl
    if workload == "batched_tensor_env":
        assert cfg.env_gpu_actions == (label != "cpu")
        assert isinstance(env, fb.BatchedTapeEnv) == (label != "native")
        assert label == "native" or env.on_cpu == (label == "cpu")
    elif workload == "dict_obs":
        assert env.obs_keys == (fb.DICT_KEYS if label == "dict" else None)
        assert cfg.encoder_mlp_layers == [512, 512]
    elif workload == "mixed_tuple":
        heads = {"d5_b3_d3_mlp512": [("discrete", 5), ("box", 3), ("discrete", 3)],
                 "d24_b8_d5_mlp512_wide": [("discrete", 24), ("box", 8), ("discrete", 5)]}[label]
        assert env.action_heads == heads and env.num_actions == {"d5_b3_d3_mlp512": 14, "d24_b8_d5_mlp512_wide": 45}[label]
    elif workload in ("nofc", "resnet"):
        arch = label.split("_fc512")[0].split("_nofc")[0]
        assert cfg.encoder_conv_architecture == arch and env.uint8 and env.obs_shape == (4, 84, 84)
        assert cfg.encoder_conv_mlp_layers == ([512] if "_fc512" in label else [])
        assert cfg.use_rnn == label.endswith("gru512") and (not cfg.use_rnn or cfg.rnn_type == "gru")
    elif workload == "rnn_layers":
        layers = int(label[1:])
        assert cfg.rnn_num_layers == layers and cfg.use_rnn and cfg.rnn_type == "lstm"
        assert (layers == 1) == (not any(a.startswith("--rnn_num_layers") for a in variant.argv))
    elif workload == "separate_rnn":
        assert cfg.actor_critic_share_weights == (label == "shared") and cfg.use_rnn and cfg.rnn_type == "lstm"
    else:
        assert env.with_action_mask if label.startswith("discrete362") else env.continuous
        assert env.num_actions == (362 if label.startswith("discrete362") else 21)


def test_no_measurement_tool_imports_tests():
    """the workload and trace tools stand apart from the test harness (conv_grad_check.py, a kernel accuracy check
    against the CPU oracle, still builds its rig from it)"""
    for path in glob.glob(os.path.join(ROOT, "tools", "*.py")):
        if path.endswith("conv_grad_check.py"):
            continue
        for node in ast.walk(ast.parse(open(path).read())):
            names = [a.name for a in node.names] if isinstance(node, ast.Import) else \
                [node.module or ""] if isinstance(node, ast.ImportFrom) else []
            assert not any(n == "tests" or n.startswith("tests.") for n in names), path


def test_refuses_to_run_without_a_cuda_device():
    res = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "feature_bench.py"), "resnet"], capture_output=True,
                         text=True, env=dict(os.environ, CUDA_VISIBLE_DEVICES=""), timeout=300)
    assert res.returncode != 0 and "needs a CUDA device" in res.stderr
    assert '"env_steps_per_s"' not in res.stdout
