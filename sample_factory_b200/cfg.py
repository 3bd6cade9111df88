"""Configuration boundary: the reference's flag surface (cfg/cfg.py, ~120 flags) and its two-pass parse
(cfg/arguments.py:24-94): `parse_sf_args` builds the parser and does a permissive first pass so example scripts can add
env-specific flags / override defaults, `parse_full_cfg` does the strict parse and records cli_args.

Flags that configure the reference's process tree (num_workers splits, heartbeat, cpu affinity, ...) are accepted and
kept in cfg for compatibility; on the device engine they are no-ops (there is no process tree).  Two extra flags exist
only here: --policy_id is fixed 0 (single-policy data-parallel path) and --gemm_engine selects the GEMM engine.
"""
from __future__ import annotations

import argparse
import copy
import os
import sys
from typing import List, Optional, Tuple


class AttrDict(dict):
    """utils/attr_dict.py equivalent: dict with attribute access (what cfg becomes after a JSON reload)."""

    __setattr__ = dict.__setitem__

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e


def str2bool(v):
    if isinstance(v, bool):
        return v
    if isinstance(v, str) and v.lower() in ("true", "1", "yes", "y", "t"):
        return True
    if isinstance(v, str) and v.lower() in ("false", "0", "no", "n", "f"):
        return False
    raise argparse.ArgumentTypeError("Boolean value expected")


# (name, type, default, nargs, choices) -- names, types and defaults as in the reference parser
_F = [
    ("algo", str, "APPO", None, None), ("env", str, None, None, None),
    ("experiment", str, "default_experiment", None, None),
    ("train_dir", str, os.path.join(os.getcwd(), "train_dir"), None, None),
    ("restart_behavior", str, "resume", None, ["resume", "restart", "overwrite"]),
    ("device", str, "gpu", None, ["gpu", "cpu"]), ("seed", int, None, None, None),
    ("num_policies", int, 1, None, None), ("async_rl", str2bool, True, None, None),
    ("serial_mode", str2bool, False, None, None), ("batched_sampling", str2bool, False, None, None),
    ("num_batches_to_accumulate", int, 2, None, None), ("worker_num_splits", int, 2, None, None),
    ("policy_workers_per_policy", int, 1, None, None), ("max_policy_lag", int, 1000, None, None),
    ("num_workers", int, 8, None, None), ("num_envs_per_worker", int, 2, None, None),
    ("batch_size", int, 1024, None, None), ("num_batches_per_epoch", int, 1, None, None),
    ("num_epochs", int, 1, None, None), ("rollout", int, 32, None, None), ("recurrence", int, -1, None, None),
    ("shuffle_minibatches", str2bool, False, None, None), ("gamma", float, 0.99, None, None),
    ("reward_scale", float, 1.0, None, None), ("reward_clip", float, 1000.0, None, None),
    ("value_bootstrap", str2bool, False, None, None), ("normalize_returns", str2bool, True, None, None),
    ("exploration_loss_coeff", float, 0.003, None, None), ("value_loss_coeff", float, 0.5, None, None),
    ("kl_loss_coeff", float, 0.0, None, None),
    ("exploration_loss", str, "entropy", None, ["entropy", "symmetric_kl"]),
    ("gae_lambda", float, 0.95, None, None), ("ppo_clip_ratio", float, 0.1, None, None),
    ("ppo_clip_value", float, 1.0, None, None), ("with_vtrace", str2bool, False, None, None),
    ("vtrace_rho", float, 1.0, None, None), ("vtrace_c", float, 1.0, None, None),
    ("optimizer", str, "adam", None, ["adam", "lamb"]), ("adam_eps", float, 1e-6, None, None),
    ("adam_beta1", float, 0.9, None, None), ("adam_beta2", float, 0.999, None, None),
    ("max_grad_norm", float, 4.0, None, None), ("learning_rate", float, 1e-4, None, None),
    ("lr_schedule", str, "constant", None, ["constant", "kl_adaptive_minibatch", "kl_adaptive_epoch"]),
    ("lr_schedule_kl_threshold", float, 0.008, None, None), ("lr_adaptive_min", float, 1e-6, None, None),
    ("lr_adaptive_max", float, 1e-2, None, None), ("obs_subtract_mean", float, 0.0, None, None),
    ("obs_scale", float, 1.0, None, None), ("normalize_input", str2bool, True, None, None),
    ("normalize_input_keys", str, None, "*", None), ("decorrelate_experience_max_seconds", int, 0, None, None),
    ("decorrelate_envs_on_one_worker", str2bool, True, None, None), ("actor_worker_gpus", int, [], "*", None),
    ("set_workers_cpu_affinity", str2bool, True, None, None), ("force_envs_single_thread", str2bool, False, None, None),
    ("default_niceness", int, 0, None, None), ("log_to_file", str2bool, True, None, None),
    ("experiment_summaries_interval", int, 10, None, None), ("flush_summaries_interval", int, 30, None, None),
    ("stats_avg", int, 100, None, None), ("summaries_use_frameskip", str2bool, True, None, None),
    ("heartbeat_interval", int, 20, None, None), ("heartbeat_reporting_interval", int, 180, None, None),
    ("train_for_env_steps", int, int(1e10), None, None), ("train_for_seconds", int, int(1e10), None, None),
    ("save_every_sec", int, 120, None, None), ("keep_checkpoints", int, 2, None, None),
    ("load_checkpoint_kind", str, "latest", None, ["latest", "best"]), ("save_milestones_sec", int, -1, None, None),
    ("save_best_every_sec", int, 5, None, None), ("save_best_metric", str, "reward", None, None),
    ("save_best_after", int, 100000, None, None), ("benchmark", str2bool, False, None, None),
    ("encoder_mlp_layers", int, [512, 512], "*", None),
    ("encoder_conv_architecture", str, "convnet_simple", None,
     ["convnet_simple", "convnet_impala", "convnet_atari", "resnet_impala"]),
    ("encoder_conv_mlp_layers", int, [512], "*", None), ("use_rnn", str2bool, True, None, None),
    ("rnn_size", int, 512, None, None), ("rnn_type", str, "gru", None, ["gru", "lstm"]),
    ("rnn_num_layers", int, 1, None, None), ("decoder_mlp_layers", int, [], "*", None),
    ("nonlinearity", str, "elu", None, ["elu", "relu", "tanh"]),
    ("policy_initialization", str, "orthogonal", None, ["orthogonal", "xavier_uniform", "torch_default"]),
    ("policy_init_gain", float, 1.0, None, None), ("actor_critic_share_weights", str2bool, True, None, None),
    ("adaptive_stddev", str2bool, True, None, None), ("continuous_tanh_scale", float, 0.0, None, None),
    ("initial_stddev", float, 1.0, None, None), ("use_env_info_cache", str2bool, False, None, None),
    ("env_gpu_actions", str2bool, False, None, None), ("env_gpu_observations", str2bool, True, None, None),
    ("env_frameskip", int, 1, None, None), ("env_framestack", int, 1, None, None),
    ("pixel_format", str, "CHW", None, None), ("use_record_episode_statistics", str2bool, False, None, None),
    ("episode_counter", str2bool, False, None, None), ("with_wandb", str2bool, False, None, None),
    ("wandb_user", str, None, None, None), ("wandb_project", str, "sample_factory", None, None),
    ("wandb_group", str, None, None, None), ("wandb_job_type", str, "SF", None, None),
    ("wandb_tags", str, [], "*", None), ("wandb_dir", str, os.path.join(os.getcwd(), "wandb"), None, None),
    ("with_pbt", str2bool, False, None, None), ("pbt_mix_policies_in_one_env", str2bool, True, None, None),
    ("pbt_period_env_steps", int, int(5e6), None, None), ("pbt_start_mutation", int, int(2e7), None, None),
    ("pbt_replace_fraction", float, 0.3, None, None), ("pbt_mutation_rate", float, 0.15, None, None),
    ("pbt_replace_reward_gap", float, 0.1, None, None), ("pbt_replace_reward_gap_absolute", float, 1e-6, None, None),
    ("pbt_optimize_gamma", str2bool, False, None, None), ("pbt_target_objective", str, "true_objective", None, None),
    ("pbt_perturb_min", float, 1.1, None, None), ("pbt_perturb_max", float, 1.5, None, None),
    # engine-specific additions
    ("gemm_engine", str, "auto", None, ["auto", "simt", "3xtf32", "tf32"]),
    ("cuda_graph", str2bool, True, None, None),
    # replay Learner.train() as one CUDA graph (constant lr schedule, one epoch, Adam, single process); removes the host's
    # ~90 kernel launches per iteration -- matters when the host is busy stepping CPU envs
    ("learner_cuda_graph", str2bool, False, None, None),
]


def _build_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(formatter_class=argparse.ArgumentDefaultsHelpFormatter, add_help=False)
    p.add_argument("-h", "--help", action="store_true", help="Print the help message")
    for name, typ, default, nargs, choices in _F:
        kw = dict(type=typ, default=default)
        if nargs is not None:
            kw["nargs"] = nargs
        if choices is not None:
            kw["choices"] = choices
        p.add_argument(f"--{name}", **kw)
    return p


def parse_sf_args(argv: Optional[List[str]] = None, evaluation: bool = False) -> Tuple[argparse.ArgumentParser, argparse.Namespace]:
    """cfg/arguments.py:24-47: first (permissive) pass; returns the parser so callers can add flags / set_defaults."""
    if argv is None:
        argv = sys.argv[1:]
    parser = _build_parser()
    if evaluation:
        # cfg/cfg.py:640-720 add_eval_args: the full evaluation surface (rendering / video / hub flags are accepted; they
        # configure host-side tooling outside the hot path)
        for name in ("no_render", "save_video", "push_to_hub"):
            parser.add_argument(f"--{name}", action="store_true")
        for name, typ, default in [("fps", int, 0), ("eval_env_frameskip", int, None), ("video_frames", int, int(1e9)),
                                   ("video_name", str, None), ("max_num_frames", int, int(1e9)),
                                   ("max_num_episodes", int, int(1e9)), ("hf_repository", str, None), ("policy_index", int, 0),
                                   ("eval_deterministic", str2bool, False), ("train_script", str, None),
                                   ("enjoy_script", str, None), ("sample_env_episodes", int, 256),
                                   ("csv_folder_name", str, None)]:
            parser.add_argument(f"--{name}", type=typ, default=default)
    partial_cfg, _ = parser.parse_known_args(argv)
    return parser, partial_cfg


def parse_full_cfg(parser: argparse.ArgumentParser, argv: Optional[List[str]] = None) -> argparse.Namespace:
    """cfg/arguments.py:50-94: strict parse + cli_args (only explicitly passed flags) + command_line."""
    if argv is None:
        argv = sys.argv[1:]
    args = parser.parse_args(argv)
    if args.help:
        parser.print_help()
        sys.exit(0)
    args.command_line = " ".join(argv)
    # a flag cannot be given the value None on the command line, so None-defaults isolate the explicitly passed ones
    no_defaults = copy.deepcopy(parser)
    no_defaults.set_defaults(**{name: None for name in vars(args)})
    args.cli_args = {k: v for k, v in vars(no_defaults.parse_args(argv)).items() if v is not None}
    args.git_hash, args.git_repo_name = "unknown", "sample_factory_b200"
    args.policy_id = 0
    return args


def default_cfg(algo: str = "APPO", env: str = "env", experiment: str = "test") -> argparse.Namespace:
    """cfg/arguments.py:219-224"""
    argv = [f"--algo={algo}", f"--env={env}", f"--experiment={experiment}"]
    parser, _ = parse_sf_args(argv)
    return parse_full_cfg(parser, argv)


def preprocess_cfg(cfg) -> bool:
    """cfg/arguments.py:97-102"""
    if cfg.recurrence == -1:
        cfg.recurrence = cfg.rollout if cfg.use_rnn else 1
    return verify_cfg(cfg)


def verify_cfg(cfg, num_agents_total: Optional[int] = None) -> bool:
    """cfg/arguments.py:105-201: same checks, same outcome (False + one logged line per problem; warnings do not fail)."""
    import sys

    ok = True

    def cfg_error(msg: str) -> None:
        nonlocal ok
        ok = False
        print(f"[sf_b200] cfg error: {msg}", file=sys.stderr)

    if cfg.num_envs_per_worker % cfg.worker_num_splits != 0:                                                # :123-127
        cfg_error(f"{cfg.num_envs_per_worker=} must be a multiple of {cfg.worker_num_splits=} (for double-buffered "
                  "sampling you need to use even number of envs per worker)")
    if cfg.normalize_returns and cfg.with_vtrace:                                                           # :129-134
        cfg_error("Normalized returns are not supported with vtrace!")
    if num_agents_total is not None and not cfg.async_rl:                                                   # :147-178
        samples = num_agents_total * cfg.rollout
        per_iteration = cfg.batch_size * cfg.num_batches_per_epoch
        if per_iteration % samples != 0 and samples % per_iteration != 0:
            cfg_error(f"sync mode: samples per training iteration ({cfg.num_batches_per_epoch=} * {cfg.batch_size=} = "
                      f"{per_iteration}) and samples per rollout ({samples}) must divide one another")
    # values the argument parser accepts (reference surface) that the kernel path does not implement: refuse with a reason
    if getattr(cfg, "rnn_num_layers", 1) < 1:
        cfg_error(f"{cfg.rnn_num_layers=} must be >= 1 (the number of stacked GRU / LSTM layers, model/core.py:27-31)")
    if getattr(cfg, "num_policies", 1) < 1:
        cfg_error(f"{cfg.num_policies=} must be >= 1")
    if cfg.use_rnn:                                                                                         # :187-194
        if cfg.recurrence <= 1:
            cfg_error(f"{cfg.recurrence=} must be > 1 to train an RNN. Recommeded value is recurrence == {cfg.rollout=}.")
        elif cfg.rollout % cfg.recurrence != 0:
            cfg_error(f"{cfg.rollout=} must be a multiple of {cfg.recurrence=}")
        if cfg.with_vtrace and cfg.recurrence != cfg.rollout:
            cfg_error(f"{cfg.recurrence=} must be equal to {cfg.rollout=} when using vtrace.")
    elif cfg.with_vtrace and (cfg.recurrence != cfg.rollout or cfg.recurrence <= 1):
        # (learner.py:684-687: the V-trace scan runs over `recurrence` steps)
        cfg_error(f"vtrace needs {cfg.recurrence=} == {cfg.rollout=} > 1")
    return ok
