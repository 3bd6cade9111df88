"""tools/learner_graph_bench.py without a GPU: the config each variant runs, the alternation of eager and graphed
learners, and the refusal to run without a CUDA device."""
import os
import subprocess
import sys
from types import SimpleNamespace

import pytest

from tools import feature_bench as fb
from tools import learner_graph_bench as lgb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def cfg_of(variant, tmp_path):
    from sample_factory_b200.cfg import parse_full_cfg, parse_sf_args

    argv = fb.full_argv(f"learner_graph_{variant.label}", variant.argv, str(tmp_path))
    parser, _ = parse_sf_args(argv)
    return parse_full_cfg(parser, argv)


def env_of(variant, monkeypatch):
    """the variant's env factory with TapeVecEnv replaced by a record of its arguments (a TapeVecEnv needs a device tape)"""
    monkeypatch.setattr(fb, "tape_env", lambda rows, n, width, seed, num_actions, uint8=False, **kw: SimpleNamespace(
        num_agents=n, obs_dim=width, num_actions=num_actions, uint8=uint8, **kw))
    return variant.env()


def test_variants_alternate_eager_and_graphed():
    labels = [v.label for v in lgb.WORKLOAD.variants]
    assert labels == [f"config{c}_{m}" for c in (3, 4, 5) for m in ("eager", "graph")]
    assert lgb.WORKLOAD.order == [f"config{c}_{m}" for c in (3, 4, 5) for m in ("eager", "graph", "eager", "graph")]
    assert set(lgb.WORKLOAD.order) == set(labels)


@pytest.mark.parametrize("variant", lgb.WORKLOAD.variants, ids=lambda v: v.label)
def test_variant_runs_its_config(variant, tmp_path, monkeypatch):
    import bench_configs

    config, mode = int(variant.label[len("config")]), variant.label.split("_")[1]
    c = bench_configs.CONFIGS[config]
    cfg, env = cfg_of(variant, tmp_path), env_of(variant, monkeypatch)
    assert cfg.learner_cuda_graph == (mode == "graph") and cfg.cuda_graph and not cfg.async_rl
    assert (cfg.num_epochs, cfg.rollout, cfg.batch_size * cfg.num_batches_per_epoch) == \
           ({3: 2, 4: 4, 5: 2}[config], c["T"], c["envs"] * c["T"])
    assert cfg.lr_schedule == ("kl_adaptive_epoch" if config == 5 else "constant")
    assert (env.num_agents, env.obs_dim, env.num_actions, env.uint8) == (c["envs"], c["obs_dim"], c["A"], c["uint8"])
    assert env.continuous == c["continuous"] and env.obs_shape == c["obs_shape"]


def test_refuses_to_run_without_a_cuda_device():
    res = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "learner_graph_bench.py")], capture_output=True,
                         text=True, env=dict(os.environ, CUDA_VISIBLE_DEVICES=""), timeout=300)
    assert res.returncode != 0 and "needs a CUDA device" in res.stderr
    assert '"env_steps_per_s"' not in res.stdout
