"""Device PPO / V-trace learner mirroring algo/learning/learner.py (Learner.train :1036, _prepare_batch :943-1034,
_calculate_losses :537-669, _train :671-841) with every tensor op replaced by a libsfb200 kernel.

Differences from the reference that are deliberate (GPU-first) and do not change results:
  * no autograd: the backward pass is explicit (sfb200_ppo_loss_fwd_bwd -> heads_backward -> linear_backward)
  * no per-minibatch host syncs: loss scalars stay in a device stats block and are read once per epoch
  * V-trace runs on the device (the reference moves the minibatch to the CPU, :602-640)
  * data parallel (new functionality, SURVEY 2a): gradients, normalizer moments and advantage statistics are
    all-reduced over NCCL so that G GPUs x N envs equals one GPU with G*N envs.
"""
from __future__ import annotations

import math
import os
from typing import Dict, List, Optional

import numpy as np
import torch
import torch.distributed as dist
from torch import Tensor

from . import ops
from .dist_utils import PeerComm, _ls_masks, peer_comm_wanted, pooled_moments_
from .model import TOWERS, PolicyModel
from .policy import HeadsPlan, forward_policy
from .rnn_core import RnnCore


class KlAdaptiveScheduler:
    """learner.py:46-86 (per-minibatch and per-epoch variants)."""

    def __init__(self, cfg, per_epoch: bool):
        self.thr = cfg.lr_schedule_kl_threshold
        self.min_lr, self.max_lr = cfg.lr_adaptive_min, cfg.lr_adaptive_max
        self.per_epoch = per_epoch
        self.n = cfg.num_batches_per_epoch if per_epoch else 1

    def invoke_after_each_minibatch(self):
        return not self.per_epoch

    def invoke_after_each_epoch(self):
        return self.per_epoch

    def update(self, lr, recent_kls):
        mean_kl = float(np.mean(recent_kls[-self.n:]))
        if mean_kl > 2.0 * self.thr:
            lr = max(lr / 1.5, self.min_lr)
        if mean_kl < 0.5 * self.thr:
            lr = min(lr * 1.5, self.max_lr)
        return lr


class LinearDecayScheduler:
    """learner.py:88-100 + utils/decay.py:4-47 restricted to the two-point schedule it is used with."""

    def __init__(self, cfg):
        self.num_updates = cfg.train_for_env_steps // cfg.batch_size * cfg.num_epochs
        self.lr0 = cfg.learning_rate
        self.step = 0

    def invoke_after_each_minibatch(self):
        return True

    def invoke_after_each_epoch(self):
        return False

    def update(self, lr, recent_kls):
        self.step += 1
        if self.step >= self.num_updates:
            return 0.0
        return self.lr0 + (0.0 - self.lr0) * (self.step / self.num_updates)


class ConstantScheduler:
    def invoke_after_each_minibatch(self):
        return False

    def invoke_after_each_epoch(self):
        return False

    def update(self, lr, recent_kls):
        return lr


def get_lr_scheduler(cfg):
    """learner.py:103-113"""
    if cfg.lr_schedule == "constant":
        return ConstantScheduler()
    if cfg.lr_schedule == "kl_adaptive_minibatch":
        return KlAdaptiveScheduler(cfg, per_epoch=False)
    if cfg.lr_schedule == "kl_adaptive_epoch":
        return KlAdaptiveScheduler(cfg, per_epoch=True)
    if cfg.lr_schedule == "linear_decay":
        return LinearDecayScheduler(cfg)
    raise RuntimeError(f"Unknown scheduler {cfg.lr_schedule}")


class Learner:
    def __init__(self, cfg, model: PolicyModel, num_traj: int, engine: int = ops.GEMM_SIMT,
                 process_group: Optional["dist.ProcessGroup"] = None, data_parallel: bool = True):
        self.cfg = cfg
        self.model = model
        self.device = model.device
        self.engine = engine
        self.pg = process_group
        self.world_size = dist.get_world_size(process_group) if (data_parallel and (process_group is not None or (
            dist.is_available() and dist.is_initialized()))) else 1
        if self.world_size > 1 and self.pg is None:
            self.pg = dist.group.WORLD
        spec = model.spec
        self.act = ops.ACT[spec.nonlinearity]
        self.N, self.T = num_traj, cfg.rollout
        self.policy_id = cfg.policy_id
        self.train_step = 0  # number of SGD steps == policy version (learner.py:142, :388-392)
        self.env_steps = 0
        self._curr_lr = cfg.learning_rate        # (see the curr_lr property: lr_dev holds it while train() replays graphs)
        self._lr_on_device = False
        self.lr_scheduler = get_lr_scheduler(cfg)
        self.last_stats: Dict[str, float] = {}

        # verify_cfg-style invariants of the path (cfg/arguments.py:105-201)
        E = self.N * self.T
        assert cfg.batch_size * cfg.num_batches_per_epoch == E, (
            f"sync mode: batch_size*num_batches_per_epoch ({cfg.batch_size}*{cfg.num_batches_per_epoch}) must equal "
            f"num_traj*rollout ({E})")
        if cfg.with_vtrace:
            assert cfg.recurrence == cfg.rollout and cfg.recurrence > 1, "V-trace requires recurrence == rollout > 1"
            assert not cfg.normalize_returns, "normalize_returns is incompatible with V-trace (arguments.py:129-134)"
        assert cfg.exploration_loss in ("entropy", "symmetric_kl"), f"{cfg.exploration_loss} not supported!"   # learner.py:186
        assert cfg.exploration_loss == "entropy" or not spec.continuous, (
            "symmetric_kl is defined for categorical distributions only (ContinuousActionDistribution has no "
            "symmetric_kl_with_uniform_prior in the reference either)")
        if cfg.exploration_loss == "symmetric_kl" and spec.action_heads:
            raise ValueError("exploration_loss='symmetric_kl' is not defined for Tuple action spaces with Box members: the "
                             "reference's ContinuousActionDistribution has no symmetric_kl_with_uniform_prior")
        assert not (spec.continuous and spec.adaptive_stddev and spec.continuous_tanh_scale > 0), (
            "continuous_tanh_scale is only read by the non-adaptive parameterization (action_parameterization.py:33-78)")
        # learner.py:498-526, :707-713: minibatches = a random permutation of recurrence-length chunks of the dataset, drawn
        # at the start of every epoch.  Device path: the permutation is drawn on the host (np.random, like the reference), copied to the
        # device, and ONE gather pass per train() rearranges every per-sample array the minibatch steps read; the steps then
        # run on contiguous slices exactly as in the unshuffled case.
        self.shuffle = bool(cfg.shuffle_minibatches) and cfg.num_batches_per_epoch > 1
        if spec.use_rnn:
            assert cfg.rollout % cfg.recurrence == 0, "rollout must be a multiple of recurrence (learner.py:500)"
            assert cfg.batch_size % cfg.recurrence == 0

        dev = self.device
        f32 = dict(dtype=torch.float32, device=dev)
        D = spec.obs_dim
        A = spec.num_action_params           # width of action_logits: n logits, or [means | log_std] for a Box space
        A_lin = spec.num_linear_action_outputs   # rows of distribution_linear
        B = cfg.batch_size
        self.E = E
        # batch-prep buffers
        self.normalized_obs = torch.empty((self.N, self.T + 1, D), **f32)
        self.h_boot = [torch.empty((self.N, h), **f32) for h in spec.hidden]
        self.advantages = torch.empty((self.N, self.T), **f32)
        self.returns = torch.empty((self.N, self.T), **f32)
        self.obs_flat_compact = torch.empty((E, D), **f32)  # normalized obs without the T+1 column, flat [N*T, D]
        self.values_old = torch.empty((self.N, self.T), **f32)
        self.valids_flat = torch.empty((self.N, self.T), dtype=torch.bool, device=dev)
        self.bmean = torch.empty(max(D, 1), **f32)
        self.bvar = torch.empty(max(D, 1), **f32)
        self.rmean = torch.empty(1, **f32)
        self.rvar = torch.empty(1, **f32)
        self.moments_ws = torch.empty(max(ops.moments_workspace_bytes(D), ops.moments_workspace_bytes(1)) // 4, **f32)
        self.num_invalids_dev = torch.zeros(1, dtype=torch.float64, device=dev)
        self.num_valid_dev = torch.zeros(1, dtype=torch.float64, device=dev)
        self.batch_stats = torch.zeros(ops.LS_SIZE, dtype=torch.float64, device=dev)
        # minibatch activations
        self.h = [torch.empty((B, h), **f32) for h in spec.hidden]
        self.dz = [torch.empty((B, h), **f32) for h in spec.hidden]
        # fp16-split form of the GEMM engine (model._register_f16): tell the library the bounds of the activation buffers the
        # forward GEMMs (normalised observations, hidden activations), dX and dW (gradients of the hidden layers) read
        self.dz_bound = None
        if getattr(self.model, "f16_twins", None) is not None and self.engine == ops.GEMM_TC_3XTF32:
            L = len(spec.hidden)
            # [bound, scratch, counter, -] per hidden layer's dz (sfb200_heads_dz_bound: the last one, then the chain below)
            self.dz_bound = torch.zeros(4 * L, **f32)
            ops.register_operand_bounds(self, [(self.obs_flat_compact, self.model.bound_x)] +
                                        [(self.dz[i], self.dz_bound[4 * i: 4 * i + 1]) for i in range(L)] +
                                        [(self.h[i], self.model.bound_h[4 * i: 4 * i + 1]) for i in range(L - 1)])
            for i in range(1, len(spec.hidden)):            # layers whose input gradient is needed: dX reads W transposed
                self.model.enable_f16_transposed(spec.fc_encoder_name(i, "weight"))
        self.mb_values = torch.empty(B, **f32)
        self.mb_logits = torch.empty((B, A), **f32)
        self.dlogits = torch.empty((B, A_lin), **f32)
        # learned log-stddev vector (continuous, adaptive_stddev=False): per-sample gradient, column-summed per minibatch
        self.dlogstd = self.colsum_ws = None
        if spec.continuous and not spec.adaptive_stddev:
            self.dlogstd = torch.empty((B, spec.num_actions), **f32)
            self.colsum_ws = torch.empty(ops.colsum_workspace_bytes(spec.num_actions) // 4 + 4, **f32)
        self.dvalues = torch.empty(B, **f32)
        self.ratio = torch.empty(B, **f32)
        self.vs = torch.empty(B, **f32)
        self.vt_adv = torch.empty(B, **f32)
        self.loss_stats = torch.zeros(ops.LS_SIZE, dtype=torch.float64, device=dev)
        n_mb_total = cfg.num_epochs * cfg.num_batches_per_epoch
        self.loss_stats_log = torch.zeros((n_mb_total, ops.LS_SIZE), dtype=torch.float64, device=dev)
        self.grad_norm_log = torch.zeros(n_mb_total, **f32)
        self.dp_partials = torch.zeros(3, dtype=torch.float64, device=dev)
        # GAE mode: the advantages are final after _prepare_batch, so the per-minibatch (count, sum, sumsq) of ALL minibatches
        # are taken there and made global with ONE all-reduce (instead of one per SGD step); row b serves minibatch b of
        # every epoch.  (V-trace advantages depend on the current policy: they keep the per-step path.)
        self.mb_partials = torch.zeros((cfg.num_batches_per_epoch, 3), dtype=torch.float64, device=dev)
        self.loss_ws = torch.empty(ops.loss_workspace_bytes(max(B, E)) // 8 + 8, dtype=torch.float64, device=dev)
        tail_w = spec.tail_input_size * (2 if spec.separate_towers else 1)     # separate weights: [actor tail | critic tail]
        lin_ws = 4
        if spec.wide_heads:
            # heads wider than 31 rows: linear_backward for dWa / dz, sfb200_heads_wide_backward for the rest
            self.heads_ws = torch.empty(ops.heads_wide_backward_workspace_bytes(B, tail_w, spec.tail_input_size, A_lin) // 4 + 4,
                                        **f32)
            lin_ws = ops.linear_backward_workspace_bytes(B, A_lin, spec.tail_input_size) // 4 + 4
        else:
            self.heads_ws = torch.empty(ops.heads_backward_workspace_bytes(tail_w, A_lin) // 4 + 4, **f32)
        if spec.dict_obs:
            for _, d in spec.obs_keys:       # the key encoders' chains
                for h in spec.encoder_mlp_layers:
                    lin_ws = max(lin_ws, ops.linear_backward_workspace_bytes(B, h, d) // 4 + 4)
                    d = h
        d = spec.fc_encoder_input
        for h in spec.fc_encoder_layers:
            lin_ws = max(lin_ws, ops.linear_backward_workspace_bytes(B, h, d) // 4 + 4)
            d = h
        self.rnn: Optional[RnnCore] = None
        # separate actor / critic weights: one core per tower on its half of the state rows; the second tower's BPTT
        # buffers share the first one's scratch and reset mask (the towers' backwards run one after the other)
        self.tower_rnn: Optional[Dict[str, RnnCore]] = None
        if spec.use_rnn:
            # recurrent core (model/core.py): BPTT buffers for one minibatch + single-step buffers for the bootstrap value
            if spec.share_weights:
                self.rnn = RnnCore(model, engine)
                self.rnn_bufs = self.rnn.alloc_bptt(B, cfg.recurrence)
                self.rnn_boot = self.rnn.alloc_step(self.N)
                core = self.rnn
            else:
                self.tower_rnn = {tw: RnnCore(model, engine, tw) for tw in TOWERS}
                self.tower_rnn_bufs = {}
                for tw in TOWERS:
                    self.tower_rnn_bufs[tw] = self.tower_rnn[tw].alloc_bptt(B, cfg.recurrence,
                                                                            self.tower_rnn_bufs.get(TOWERS[0]))
                self.rnn_boot = self.tower_rnn[TOWERS[0]].alloc_step(self.N)     # (the towers step one after the other)
                core = self.tower_rnn[TOWERS[0]]
            self.boot_state_out = torch.empty((self.N, spec.rnn_state_size), **f32)
            self.d_core = torch.empty((B, spec.rnn_size), **f32)
            self.rnn_states_flat = torch.empty((E, spec.rnn_state_size), **f32)
            lin_ws = max(lin_ws, core.lin_ws_bytes(B, cfg.recurrence, d) // 4 + 4)
            d = spec.rnn_size
        for h in spec.decoder_mlp_layers:
            lin_ws = max(lin_ws, ops.linear_backward_workspace_bytes(B, h, d) // 4 + 4)
            d = h
        self.lin_ws = torch.empty(lin_ws, **f32)
        self.heads_plan = HeadsPlan(model, engine, max(B, self.N), need_backward=True)
        # image observations: gradient w.r.t. the conv head's output (pre-activation of its last layer, (C,H,W) order)
        self.dfeat = torch.empty((B, spec.conv_out_size), **f32) if spec.obs_shape is not None else None
        # linear policy: the heads backward writes the gradient w.r.t. the normalised observation rows here; nothing reads it
        # (the [B, obs_dim] store is as wide as the rows the kernel reads anyway)
        self.dobs = torch.empty((B, D), **f32) if spec.heads_read_input else None
        self.adam_ws = torch.empty(1024, **f32)
        assert cfg.optimizer in ("adam", "lamb"), f"Unknown optimizer {cfg.optimizer}"    # learner.py:228-230
        if cfg.optimizer == "lamb":
            # per-tensor view of the flat buffers for the trust ratios (algo/utils/optimizers.py:101-134)
            segs = [model._slices[n] for n in model.names]
            numels = [math.prod(shp) for _, shp in segs]
            self.lamb_off = torch.tensor([o for o, _ in segs], dtype=torch.int64, device=dev)
            self.lamb_numel = torch.tensor(numels, dtype=torch.int64, device=dev)
            self.lamb_max = max(numels)
            self.lamb_ws = torch.empty(ops.lamb_workspace_bytes(len(segs), self.lamb_max) // 4 + 4, **f32)
        self.opt_step = 0
        self.kernel_launches = 0
        self._mb: Dict[str, Tensor] = {}
        if self.shuffle:
            chunk = cfg.recurrence if spec.use_rnn or cfg.with_vtrace else max(1, cfg.recurrence)
            assert E % chunk == 0
            self._perm_chunk = chunk
            self.perm_host = torch.empty(E, dtype=torch.int32).pin_memory()
            self.perm_dev = torch.arange(E, dtype=torch.int32, device=dev)
            self._perm_queue: List[np.ndarray] = []      # explicit permutations for the next epochs (tests); else np.random
            self._sh: Dict[str, Tensor] = {}
        # CUDA-graph replay of train() (cfg.learner_cuda_graph): one graph per epoch and trajectory set.  The step
        # counters, the learning rate and the per-minibatch learning-rate rules live in device memory (the *_dev entry
        # points, sfb200_lr_schedule_step); what stays on the host is the one sync per epoch the eager path also takes
        # (early stopping, kl_adaptive_epoch), between two replays.
        # Data parallel: every exchange is a libsfb200 kernel over NVLink peer memory (csrc/comm.cu) -- the gradient lives in
        # the comm buffer the peers read, so train() is kernels only and is captured like the single-GPU learner.
        # SFB200_DP_COMM=nccl keeps the exchanges on torch.distributed: its graph is opt-in with SFB200_DP_GRAPH=1 (the
        # NCCL all-reduces are then captured with the kernels) and limited to constant lr, one epoch and Adam, the case
        # the multi-rank equivalence test covers (tests/dp_worker.py, see DESIGN section 7).
        self.comm: Optional[PeerComm] = None
        if self.world_size > 1 and model.flat.is_cuda and peer_comm_wanted():
            self.comm = PeerComm(dev, model.flat.numel(), self.pg)
            model.rebind_grad(self.comm.grad)
            self.grad_reduced = torch.zeros_like(model.flat)
            self._ls_keep, self._ls_max, self._ls_min, self._ls_avg = _ls_masks()
        nccl_graph = (os.environ.get("SFB200_DP_GRAPH", "0") == "1" and cfg.lr_schedule == "constant" and
                      cfg.num_epochs == 1 and cfg.optimizer == "adam")
        self.use_graph = (bool(getattr(cfg, "learner_cuda_graph", False)) and
                          (self.world_size == 1 or self.comm is not None or nccl_graph))
        # [optimizer steps taken, train_step, linear-decay schedule step]
        self.counters_dev = torch.zeros(3, dtype=torch.int64, device=dev)
        self.lr_dev = torch.full((1,), float(cfg.learning_rate), dtype=torch.float64, device=dev)
        self._graph: Optional[torch.cuda.CUDAGraph] = None            # the last graph replayed
        self._graphs: Dict[tuple, torch.cuda.CUDAGraph] = {}          # (trajectory set, epoch) -> its graph
        self._epoch_launches: Dict[int, int] = {}                     # epoch -> launches of its body (eager warm-up)
        self._replayed_launches = 0

    # ------------------------------------------------------------------------------------------------------------
    def _allreduce(self, t: Tensor) -> None:
        """sum of a small float64 buffer over the ranks, in place"""
        if self.world_size == 1:
            return
        if self.comm is not None:
            ops.dp_allreduce_f64(self.comm.comm, t)
        else:
            dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.pg)

    def _allreduce_loss_rows(self, rows: Tensor) -> None:
        """per-minibatch loss statistics rows [k, LS_SIZE] -> global values (means add up, extrema take max / min)"""
        if self.world_size == 1:
            return
        if self.comm is not None:
            ops.dp_allreduce_f64(self.comm.comm, rows, ops.LS_SIZE, self._ls_max, self._ls_min, self._ls_keep, self._ls_avg)
            return
        from .dist_utils import _ls_masks
        keep, mx, mn, avg = _ls_masks()
        summed = rows.clone()
        dist.all_reduce(summed, op=dist.ReduceOp.SUM, group=self.pg)
        big, small = rows.clone(), rows.clone()
        dist.all_reduce(big, op=dist.ReduceOp.MAX, group=self.pg)
        dist.all_reduce(small, op=dist.ReduceOp.MIN, group=self.pg)
        for c in range(ops.LS_SIZE):
            bit = 1 << c
            if bit & keep:
                continue
            rows[..., c] = big[..., c] if bit & mx else (small[..., c] if bit & mn else summed[..., c])
            if bit & avg:
                rows[..., c] /= self.world_size

    def _update_rms(self, x2d: Tensor, mean: Tensor, var: Tensor, count: Tensor, bmean: Tensor, bvar: Tensor) -> None:
        """running_mean_std.py:66-77 on device. Under data parallelism the batch moments are made global first."""
        rows, dim = x2d.shape
        ops.batch_moments(x2d, bmean[:dim], bvar[:dim], self.moments_ws)
        total = rows
        if self.comm is not None:
            ops.dp_pooled_moments(self.comm.comm, bmean[:dim], bvar[:dim], rows)
            total = rows * self.world_size
        elif self.world_size > 1:
            total = pooled_moments_(bmean[:dim], bvar[:dim], rows, self.pg)
        ops.rms_merge(mean, var, count, bmean[:dim], bvar[:dim], float(total))

    # ------------------------------------------------------------------------------------------------------------
    def _prepare_batch(self, batch: Dict[str, Tensor]) -> None:
        """learner.py:943-1034 (sync mode: operates on the trajectory buffers in place like the reference)."""
        cfg, m, spec = self.cfg, self.model, self.model.spec
        N, T, D = self.N, self.T, spec.obs_dim
        if self.use_graph:
            ops.compute_valids_dev(batch["policy_id"], batch["policy_version"], self.policy_id, self.counters_dev[1:2],
                                   cfg.max_policy_lag, batch["valids"])
        else:
            ops.compute_valids(batch["policy_id"], batch["policy_version"], self.policy_id, self.train_step,
                               cfg.max_policy_lag, batch["valids"])                                 # :950-955
        obs2d = batch["obs"].view(N * (T + 1), D)
        nobs2d = self.normalized_obs.view(N * (T + 1), D)
        inv_scale = 1.0 / spec.obs_scale
        if spec.normalize_input:                                                                     # :961, :925-941
            src = obs2d
            if abs(spec.obs_subtract_mean) > 1e-8 or abs(spec.obs_scale - 1.0) > 1e-8 or obs2d.dtype != torch.float32:
                # stats are taken AFTER sub-mean / scaling (normalize.py:62-67): stage the scaled obs first
                ops.normalize_obs(obs2d, nobs2d, None, None, spec.obs_subtract_mean, inv_scale)
                src = nobs2d
                self._update_rms(src, m.obs_mean, m.obs_var, m.obs_count, self.bmean, self.bvar)
                ops.normalize_obs(src, nobs2d, m.obs_mean, m.obs_var, 0.0, 1.0)
            else:
                self._update_rms(src, m.obs_mean, m.obs_var, m.obs_count, self.bmean, self.bvar)
                ops.normalize_obs(src, nobs2d, m.obs_mean, m.obs_var, 0.0, 1.0)
        else:
            ops.normalize_obs(obs2d, nobs2d, None, None, spec.obs_subtract_mean, inv_scale)
        # bootstrap value for step T (:965-967): forward on normalized_obs[:, T] in place (strided rows)
        boot_rnn = tower_boot = None
        if self.rnn is not None:
            boot_rnn = lambda head: self.rnn.step(head, batch["rnn_states"][:, T], self.boot_state_out, self.rnn_boot)
        elif self.tower_rnn is not None:     # (both towers run; only the critic's half of the tail reaches the value)
            tower_boot = {tw: (lambda head, c=c: c.step(head, batch["rnn_states"][:, T], self.boot_state_out, self.rnn_boot))
                          for tw, c in self.tower_rnn.items()}
        forward_policy(m, self.normalized_obs[:, T], self.h_boot, self.act, self.engine, self.heads_plan,
                       dict(values=batch["values"][:, T], values_stride=batch["values"].stride(0)), boot_rnn,
                       store_tail=False, tower_rnn_fns=tower_boot)
        # :969-1003 fused
        ops.gae_returns(batch["rewards"], batch["dones"], batch["time_outs"], batch["values"], batch["valids"],
                        cfg.gamma, cfg.gae_lambda, cfg.value_bootstrap,
                        m.ret_mean if spec.normalize_returns else None,
                        m.ret_var if spec.normalize_returns else None, self.advantages, self.returns)
        # :1006-1012 drop the T+1 column and flatten: strided copies into dense [N*T, ...] buffers
        ops.copy_rows(self.normalized_obs.view(N, (T + 1) * D)[:, : T * D], self.obs_flat_compact.view(N, T * D))
        ops.copy_rows(batch["values"][:, :T], self.values_old)
        ops.copy_rows_bytes(batch["valids"][:, :T], self.valids_flat)
        if spec.use_rnn:
            S = spec.rnn_state_size
            ops.copy_rows(batch["rnn_states"].view(N, (T + 1) * S)[:, : T * S], self.rnn_states_flat.view(N, T * S))
        if spec.normalize_returns and not cfg.with_vtrace:                                          # :1018-1019
            r = self.returns.view(-1, 1)
            self._update_rms(r, m.ret_mean, m.ret_var, m.ret_count, self.rmean, self.rvar)
            ops.rms_apply_scalar(self.returns.view(-1), m.ret_mean, m.ret_var, denormalize=False)
        self._bind_minibatch_arrays(batch)
        # :1021 num_invalids, kept on the device (lr scaling :788-794 happens inside the Adam kernel)
        if cfg.with_vtrace:
            ops.adv_stats(self.advantages.view(-1), self.valids_flat.view(-1), self.batch_stats, None, self.loss_ws)
            nv = self.batch_stats[ops.LS["num_valid"] : ops.LS["num_valid"] + 1]
            if self.world_size > 1:
                self._allreduce(nv)
            ops.copy_rows_bytes(nv.view(1, 1), self.num_valid_dev.view(1, 1))
        else:
            self._minibatch_adv_partials()

    def _minibatch_adv_partials(self) -> None:
        """GAE mode: (count, sum, sum of squares) of the advantages of every minibatch of the CURRENT sample order (the
        normalisation statistics of learner.py:646-647), made global with one all-reduce; + the global valid count"""
        cfg = self.cfg
        B = cfg.batch_size
        adv_flat, val_flat = self._mb["adv"], self._mb["valids"]
        for b in range(cfg.num_batches_per_epoch):
            ops.adv_stats(adv_flat[b * B : (b + 1) * B], val_flat[b * B : (b + 1) * B], self.batch_stats,
                          self.mb_partials[b], self.loss_ws)
        if self.world_size > 1:
            self._allreduce(self.mb_partials)
        ops.colsum_f64(self.mb_partials, 0, self.num_valid_dev)                            # global valid count

    def set_minibatch_permutation(self, indices) -> None:
        """The sample order of the epochs of the NEXT train() call (shuffle_minibatches): one array [E] as learner.py:498-526
        builds them, or a sequence of them, one per epoch.  Epochs without an explicit permutation draw np.random.permutation
        over the recurrence-length chunks like the reference."""
        assert self.shuffle
        arr = np.asarray(indices, dtype=np.int64)
        rows = arr.reshape(1, -1) if arr.ndim == 1 else arr.reshape(arr.shape[0], -1)
        for idx in rows:
            assert idx.shape[0] == self.E and np.array_equal(np.sort(idx), np.arange(self.E))
        self._perm_queue = [idx.copy() for idx in rows]

    def _upload_permutation(self) -> None:
        """host side of the shuffle (outside any graph capture): draw / take the permutation, enqueue its H2D copy"""
        if self._perm_queue:
            idx = self._perm_queue.pop(0)
        else:
            c = self._perm_chunk
            starts = np.random.permutation(np.arange(0, self.E, c))                   # :505-506
            idx = (starts[:, None] + np.arange(c)[None, :]).reshape(-1)              # :509-510
        self.perm_host.copy_(torch.from_numpy(idx.astype(np.int32)))
        self.perm_dev.copy_(self.perm_host, non_blocking=True)

    def _bind_minibatch_arrays(self, batch: Dict[str, Tensor]) -> None:
        """flat [E, ...] views of everything a minibatch step reads; with shuffle_minibatches: gathered copies in the
        permuted order (minibatch b is then rows [b*B, (b+1)*B) as usual)"""
        spec, E = self.model.spec, self.E
        src = dict(obs=self.obs_flat_compact, actions=batch["actions"].view(E, spec.action_width),
                   lp_old=batch["log_prob_actions"].view(E, 1), logits_old=batch["action_logits"].view(E, spec.num_action_params),
                   valids=self.valids_flat.view(E, 1), v_old=self.values_old.view(E, 1), adv=self.advantages.view(E, 1),
                   ret=self.returns.view(E, 1), dones=batch["dones"].view(E, 1), rewards=batch["rewards"].view(E, 1))
        if spec.use_rnn:
            src["rnn"] = self.rnn_states_flat
        if self.shuffle:
            for k, v in src.items():
                if k not in self._sh:
                    self._sh[k] = torch.empty_like(v)
                ops.gather_rows(v, self.perm_dev, self._sh[k])
            src = self._sh
        self._mb = {k: (v if k in ("obs", "actions", "logits_old", "rnn") else v.view(E)) for k, v in src.items()}

    # ------------------------------------------------------------------------------------------------------------
    def _minibatch_step(self, batch: Dict[str, Tensor], b: int, log_idx: int) -> None:
        cfg, m, spec = self.cfg, self.model, self.model.spec
        B = cfg.batch_size
        sl = slice(b * B, (b + 1) * B)                                                               # :521
        loss_stats = self.loss_stats_log[log_idx]      # the kernels write this minibatch's statistics row in place
        A = spec.num_action_params
        mbv = self._mb
        x0 = mbv["obs"][sl]
        actions = mbv["actions"][sl]
        if not spec.continuous and not spec.action_segments and not spec.action_heads:
            actions = actions.view(-1)
        lp_old = mbv["lp_old"][sl]
        logits_old = mbv["logits_old"][sl]
        valids = mbv["valids"][sl]
        v_old = mbv["v_old"][sl]
        # forward (:553-579)
        mb_rnn = mb_tower = None
        if self.rnn is not None:
            mb_rnn = lambda head: self.rnn.forward_bptt(head, mbv["rnn"][sl], mbv["dones"][sl], valids, self.rnn_bufs)
        elif self.tower_rnn is not None:     # the first tower's core computes the minibatch's reset mask for both
            mb_tower = {tw: (lambda head, tw=tw: self.tower_rnn[tw].forward_bptt(
                head, mbv["rnn"][sl], mbv["dones"][sl] if tw == TOWERS[0] else None, valids, self.tower_rnn_bufs[tw]))
                for tw in TOWERS}
        x = forward_policy(m, x0, self.h, self.act, self.engine, self.heads_plan,
                           dict(values=self.mb_values, values_stride=1, logits=self.mb_logits, logits_stride=A), mb_rnn,
                           store_tail=True, tower_rnn_fns=mb_tower)
        Wv, bv = m.critic
        Wa, ba = m.actor
        if cfg.with_vtrace:                                                                          # :602-640
            if spec.action_heads:
                ops.action_ratio_mixed(self.mb_logits, spec.head_kinds, spec.head_sizes, actions, lp_old, self.ratio)
            elif spec.action_segments:
                ops.action_ratio_tuple(self.mb_logits, spec.action_segments, actions, lp_old, self.ratio)
            elif spec.continuous:
                ops.action_ratio_continuous(self.mb_logits, actions, lp_old, self.ratio)
            else:
                ops.action_ratio(self.mb_logits, actions, lp_old, self.ratio)
            ops.vtrace(self.ratio, self.mb_values, mbv["rewards"][sl], mbv["dones"][sl],
                       cfg.recurrence, cfg.gamma, cfg.vtrace_rho, cfg.vtrace_c, self.vs, self.vt_adv)
            adv, targets = self.vt_adv, self.vs
        else:
            adv, targets = mbv["adv"][sl], mbv["ret"][sl]                                              # :643-644
        # :646-647 advantage statistics (global under data parallelism)
        if not cfg.with_vtrace:
            ops.adv_stats_finalize(self.mb_partials[b], loss_stats)       # partials taken in _prepare_batch
        elif self.world_size > 1:
            ops.adv_stats(adv, valids, loss_stats, self.dp_partials, self.loss_ws)
            self._allreduce(self.dp_partials)
            ops.adv_stats_finalize(self.dp_partials, loss_stats)
        else:
            ops.adv_stats(adv, valids, loss_stats, None, self.loss_ws)
        # losses forward + backward (:651-657, :779)
        if spec.action_heads:
            ops.ppo_loss_fwd_bwd_mixed(self.mb_logits, self.mb_values, spec.head_kinds, spec.head_sizes, actions, lp_old,
                                       v_old, adv, targets, valids, logits_old, cfg.ppo_clip_ratio, cfg.ppo_clip_value,
                                       cfg.exploration_loss_coeff, cfg.value_loss_coeff, cfg.kl_loss_coeff, 1.0,
                                       self.dlogits, self.dvalues, loss_stats, self.loss_ws)
        elif spec.action_segments:
            ops.ppo_loss_fwd_bwd_tuple(self.mb_logits, self.mb_values, spec.action_segments, actions, lp_old, v_old, adv,
                                       targets, valids, logits_old, cfg.ppo_clip_ratio, cfg.ppo_clip_value,
                                       cfg.exploration_loss_coeff, cfg.value_loss_coeff, cfg.kl_loss_coeff, 1.0,
                                       self.dlogits, self.dvalues, loss_stats, self.loss_ws,
                                       exploration_loss=cfg.exploration_loss)
        elif spec.continuous:
            ops.ppo_loss_fwd_bwd_continuous(self.mb_logits, self.mb_values, spec.adaptive_stddev, spec.continuous_tanh_scale,
                                            actions, lp_old, v_old, adv, targets, valids, logits_old, cfg.ppo_clip_ratio,
                                            cfg.ppo_clip_value, cfg.exploration_loss_coeff, cfg.value_loss_coeff,
                                            cfg.kl_loss_coeff, 1.0, self.dlogits, self.dlogstd, self.dvalues,
                                            loss_stats, self.loss_ws)
            if self.dlogstd is not None:   # gradient of the learned log-stddev vector = column sum over the minibatch
                ops.colsum(self.dlogstd, m.grads["action_parameterization.learned_stddev"], self.colsum_ws)
        else:
            ops.ppo_loss_fwd_bwd(self.mb_logits, self.mb_values, actions, lp_old, v_old, adv, targets, valids, logits_old,
                                 cfg.ppo_clip_ratio, cfg.ppo_clip_value, cfg.exploration_loss_coeff, cfg.value_loss_coeff,
                                 cfg.kl_loss_coeff, 1.0, self.dlogits, self.dvalues, loss_stats, self.loss_ws,
                                 exploration_loss=cfg.exploration_loss)
        self.loss_stats_log[log_idx].copy_(loss_stats)
        if self.heads_plan.separate:
            self._backward_separate(x0)
        else:
            self._backward_shared(batch, x, x0, sl, valids)
        # gradient all-reduce: ONE NCCL call on the flat buffer (SURVEY 8e); mean over ranks is folded into the sums:
        # each rank's loss already divides by the GLOBAL valid count, so the rank gradients simply add up.
        # :781-797 clip + Adam (+ lr scaling by the valid fraction, on device)
        self.opt_step += 1
        grad = m.grad
        if self.comm is not None:
            grad = self.grad_reduced
            if cfg.optimizer == "adam":
                # peer pull + sum + grad-norm + clip + Adam in ONE kernel (csrc/comm.cu)
                dev_ctr = self.use_graph
                ops.dp_grad_allreduce_clip_adam(
                    self.comm.comm, grad, m.flat, m.exp_avg, m.exp_avg_sq, self.opt_step,
                    self.counters_dev[0:1] if dev_ctr else None, 0.0 if dev_ctr else self.curr_lr,
                    self.lr_dev if dev_ctr else None,
                    cfg.adam_beta1, cfg.adam_beta2, cfg.adam_eps, cfg.max_grad_norm, self.num_valid_dev,
                    self.exp_size_total_dev(), self.grad_norm_log[log_idx: log_idx + 1], self.comm.workspace)
                if dev_ctr:
                    ops.advance_counters(self.counters_dev[0:1], self.counters_dev[1:2])
                m.refresh_cat_heads()
                m.refresh_bounds()
                self.train_step += 1
                return
            ops.dp_grad_allreduce(self.comm.comm, grad, self.comm.workspace)
        elif self.world_size > 1:
            dist.all_reduce(m.grad, op=dist.ReduceOp.SUM, group=self.pg)
        if cfg.optimizer == "lamb" and self.use_graph:
            ops.clip_lamb_step_dev(m.flat, grad, m.exp_avg, m.exp_avg_sq, self.lamb_off, self.lamb_numel, self.lamb_max,
                                   self.counters_dev[0:1], self.lr_dev, cfg.adam_beta1, cfg.adam_beta2, cfg.adam_eps, 1e-4,
                                   0.01, cfg.max_grad_norm, self.num_valid_dev, self.exp_size_total_dev(),
                                   self.grad_norm_log[log_idx : log_idx + 1], self.lamb_ws)
            ops.advance_counters(self.counters_dev[0:1], self.counters_dev[1:2])
        elif cfg.optimizer == "lamb":
            ops.clip_lamb_step(m.flat, grad, m.exp_avg, m.exp_avg_sq, self.lamb_off, self.lamb_numel, self.lamb_max,
                               self.opt_step, self.curr_lr, cfg.adam_beta1, cfg.adam_beta2, cfg.adam_eps, 1e-4, 0.01,
                               cfg.max_grad_norm, self.num_valid_dev, self.exp_size_total_dev(),
                               self.grad_norm_log[log_idx : log_idx + 1], self.lamb_ws)
        elif self.use_graph:
            ops.clip_adam_step_dev(m.flat, grad, m.exp_avg, m.exp_avg_sq, self.counters_dev[0:1], self.lr_dev,
                                   cfg.adam_beta1, cfg.adam_beta2, cfg.adam_eps, cfg.max_grad_norm, self.num_valid_dev,
                                   self.exp_size_total_dev(), self.grad_norm_log[log_idx : log_idx + 1], self.adam_ws)
            ops.advance_counters(self.counters_dev[0:1], self.counters_dev[1:2])
        else:
            ops.clip_adam_step(m.flat, grad, m.exp_avg, m.exp_avg_sq, self.opt_step, self.curr_lr, cfg.adam_beta1,
                               cfg.adam_beta2, cfg.adam_eps, cfg.max_grad_norm, self.num_valid_dev,
                               self.exp_size_total_dev(), self.grad_norm_log[log_idx : log_idx + 1], self.adam_ws)
        m.refresh_cat_heads()        # separate actor / critic weights: re-embed the updated head weights (no-op otherwise)
        if m.f16_twins is not None:
            if cfg.optimizer == "lamb":
                ops.refresh_f16_twins(m.flat)      # (the Adam kernels keep the fp16 twins current themselves)
            m.refresh_bounds()         # activation bounds + transposed twins follow the new weights (fp16-split GEMM engine)
        self.train_step += 1                                                                         # :388-392

    def _backward_shared(self, batch: Dict[str, Tensor], x: Tensor, x0: Tensor, sl: slice, valids: Tensor) -> None:
        """explicit backward pass of the shared-weights model (the reference's loss.backward(), learner.py:779)"""
        cfg, m, spec = self.cfg, self.model, self.model.spec
        Wv, bv = m.critic
        Wa, ba = m.actor
        # backward: heads -> decoder MLP -> (recurrent core, BPTT) -> encoder MLP
        g = m.grads
        none = ops.ACT["none"]
        enc, dec = m.encoder_layers(), m.decoder_layers()
        genc, gdec = m.encoder_layers(grads=True), m.decoder_layers(grads=True)
        Le, Ld = len(enc), len(dec)
        rnn = self.rnn is not None
        plan = self.heads_plan
        B = x0.shape[0]
        # the encoder's output as the next stage reads it: (activations, activation, their gradient, gradient of the bias that
        # made them); Dict models: the key encoders' concatenation (identity encoders: the normalised rows, no gradient)
        if plan.keys:
            x_enc, act_enc, d_enc, db_enc = plan.enc_cat[:B], self.act, plan.denc_cat[:B], plan.db_enc_cat
        elif Le > 0:
            x_enc, act_enc, d_enc, db_enc = self.h[Le - 1], self.act, self.dz[Le - 1], genc[-1][1]
        elif plan.conv is not None:      # conv head without fully connected layers: its activated features, bias in the head
            x_enc, act_enc, d_enc, db_enc = plan.conv.feat[:B], self.act, self.dfeat, None
        else:
            x_enc, act_enc, d_enc, db_enc = x0, none, None, None
        tail_is_mlp = Ld > 0 or not rnn            # is the tensor feeding the heads the decoder's or the encoder's output?
        tail_dz = (self.dz[Le + Ld - 1] if Ld > 0 else d_enc) if tail_is_mlp else self.d_core
        if tail_dz is None:                        # linear policy: the input gradient goes to a scratch nobody reads
            tail_dz = self.dobs
        tail_db = gdec[-1][1] if Ld > 0 else (None if rnn else db_enc)
        if self.dz_bound is not None and tail_is_mlp:
            L = len(spec.hidden)
            ops.heads_dz_bound(self.dlogits, self.dvalues, Wv, Wa, self.dz_bound[4 * (L - 1):], m.grad_fac, self.dz_bound,
                               L - 1)
        tail_act = (self.act if Ld > 0 else act_enc) if tail_is_mlp else none
        if spec.wide_heads:
            # dWa = dlogits^T . x and tail_dz = (dlogits . Wa) * act'(x) on the GEMM engine, then the value term, the bias /
            # value gradients and db_prev (the bound above covers the sum: the formula holds for any number of rows)
            ops.linear_backward(self.dlogits, x, Wa, tail_act, g["action_parameterization.distribution_linear.weight"],
                                tail_dz, None, self.engine, self.lin_ws)
            ops.heads_wide_backward(x, Wv, self.dlogits, self.dvalues, tail_act, tail_dz, 0, True,
                                    g["critic_linear.weight"].view(-1), g["critic_linear.bias"],
                                    g["action_parameterization.distribution_linear.bias"], tail_db, self.heads_ws)
        else:
            ops.heads_backward(x, Wv, Wa, self.dlogits, self.dvalues, tail_act, tail_dz,
                               g["critic_linear.weight"].view(-1), g["critic_linear.bias"],
                               g["action_parameterization.distribution_linear.weight"],
                               g["action_parameterization.distribution_linear.bias"], tail_db, self.heads_ws)
        for j in range(Ld - 1, -1, -1):
            W, dW = dec[j][0], gdec[j][0]
            if j > 0:
                x_in, act_prev, dx, dbp = self.h[Le + j - 1], self.act, self.dz[Le + j - 1], gdec[j - 1][1]
            elif rnn:
                x_in, act_prev, dx, dbp = self.rnn_bufs["core_out"], none, self.d_core, None
            else:
                x_in, act_prev, dx, dbp = x_enc, act_enc, d_enc, db_enc
            ops.linear_backward(self.dz[Le + j], x_in, W, act_prev, dW, dx, dbp, self.engine, self.lin_ws)
        if rnn:
            dgi_all = self.rnn.backward_bptt(self.d_core, self.rnn_bufs, self.lin_ws)
            W_ih = m.rnn_params()[0]
            dW_ih = m.rnn_params(grads=True)[0]
            ops.linear_backward(dgi_all, x_enc, W_ih, act_enc, dW_ih, d_enc, db_enc, self.engine, self.lin_ws)
        if plan.keys:
            self._backward_keys(x0)
        if Le == 0 and plan.conv is not None:
            plan.conv.backward(self.dfeat)
        for li in range(Le - 1, -1, -1):
            W, dW = enc[li][0], genc[li][0]
            if li > 0:
                ops.linear_backward(self.dz[li], self.h[li - 1], W, self.act, dW, self.dz[li - 1], genc[li - 1][1],
                                    self.engine, self.lin_ws)
            elif self.heads_plan.conv is not None:
                # first fully connected layer of a ConvEncoder: its input is the conv head's activated output
                conv = self.heads_plan.conv
                ops.linear_backward(self.dz[li], conv.feat[: x0.shape[0]], W, self.act, dW, self.dfeat, None, self.engine,
                                    self.lin_ws)
                conv.backward(self.dfeat)
            else:
                ops.linear_backward(self.dz[li], x0, W, none, dW, None, None, self.engine, self.lin_ws)

    def _backward_keys(self, x0: Tensor) -> None:
        """backward of the key encoders (MultiInputEncoder): key k's chain starts from its column block of d(concatenation),
        and the bias gradient of its last layer is its block of the concatenation's column sums"""
        m, spec, plan = self.model, self.model.spec, self.heads_plan
        B = x0.shape[0]
        none = ops.ACT["none"]
        col = 0
        for k, (layers, glayers, c, (_, d)) in enumerate(zip(m.key_encoder_layers(), m.key_encoder_layers(grads=True),
                                                            spec.key_offsets, spec.obs_keys)):
            n = spec.key_out_sizes[k]
            L = len(layers)
            glayers[L - 1][1].copy_(plan.db_enc_cat[col: col + n])
            dz = plan.denc_cat[:B, col: col + n]
            for i in range(L - 1, -1, -1):
                W, dW = layers[i][0], glayers[i][0]
                if i > 0:
                    dx = plan.key_dz[k][i - 1][:B]
                    ops.linear_backward(dz, plan.key_h[k][i - 1][:B], W, self.act, dW, dx, glayers[i - 1][1], self.engine,
                                        self.lin_ws)
                    dz = dx
                else:
                    ops.linear_backward(dz, x0[:, c: c + d], W, none, dW, None, None, self.engine, self.lin_ws)
            col += n

    def _backward_separate(self, x0: Tensor) -> None:
        """backward of ActorCriticSeparateWeights: one heads-backward over the concatenated tail [B, 2H] (zero-padded head
        weights route d(logits) into the actor half and d(value) into the critic half), then per tower its decoder MLP
        chain, its core's BPTT and its encoder MLP chain.  A tail that is a core's output has no activation and no bias."""
        m, spec, plan = self.model, self.model.spec, self.heads_plan
        B = x0.shape[0]
        H = spec.tail_input_size
        g = m.grads
        none = ops.ACT["none"]
        tail_act = self.act if plan.tower_tail_is_mlp else none
        db_cat = plan.db_cat if plan.tower_tail_is_mlp else None
        if spec.wide_heads:
            # logits GEMM backward on the actor half (Wa itself, not the zero-padded Wa_cat), then the critic half's value
            # term and the column sums of both halves
            Wv, Wa = m.critic[0], m.actor[0]
            ops.linear_backward(self.dlogits, plan.tail_cat[:B, :H], Wa, tail_act,
                                g["action_parameterization.distribution_linear.weight"], plan.dz_cat[:B, :H], None,
                                self.engine, self.lin_ws)
            ops.heads_wide_backward(plan.tail_cat[:B, H:], Wv, self.dlogits, self.dvalues, tail_act, plan.dz_cat[:B], H,
                                    False, g["critic_linear.weight"].view(-1), g["critic_linear.bias"],
                                    g["action_parameterization.distribution_linear.bias"], db_cat, self.heads_ws)
        else:
            ops.heads_backward(plan.tail_cat[:B], m.Wv_cat, m.Wa_cat, self.dlogits, self.dvalues, tail_act, plan.dz_cat[:B],
                               plan.gWv_cat.view(-1), g["critic_linear.bias"], plan.gWa_cat,
                               g["action_parameterization.distribution_linear.bias"], db_cat, self.heads_ws)
            g["critic_linear.weight"].copy_(plan.gWv_cat[:, H:])                                   # (the padded halves are
            g["action_parameterization.distribution_linear.weight"].copy_(plan.gWa_cat[:, :H])     #  not parameters: dropped)
        for tw, col in zip(TOWERS, (0, H)):
            enc, genc = m.tower_encoder_layers(tw), m.tower_encoder_layers(tw, grads=True)
            dec, gdec = m.tower_decoder_layers(tw), m.tower_decoder_layers(tw, grads=True)
            Le = len(enc)
            layers, glayers = enc + dec, genc + gdec
            acts = [plan.tail_cat[:B, col: col + H] if h is None else h[:B] for h in plan.tower_h[tw]]
            dzs = [plan.dz_cat[:B, col: col + H] if dz is None else dz[:B] for dz in plan.tower_dz[tw]]
            if plan.tower_tail_is_mlp:
                glayers[-1][1].copy_(plan.db_cat[col: col + H])      # bias gradient of the tower's last layer
            if self.tower_rnn is None:
                self._mlp_chain_backward(layers, glayers, acts, dzs, 0, x0)
                continue
            # the encoder's output as the core reads it: (activations, activation, their gradient, its bias gradient)
            if Le > 0:
                x_enc, act_enc, d_enc, db_enc = acts[Le - 1], self.act, dzs[Le - 1], genc[-1][1]
            else:
                x_enc, act_enc, d_enc, db_enc = x0, none, None, None
            core, bufs = self.tower_rnn[tw], self.tower_rnn_bufs[tw]
            d_core = self.d_core if dec else plan.dz_cat[:B, col: col + H]
            if dec:
                self._mlp_chain_backward(layers, glayers, acts, dzs, Le, bufs["core_out"], none, d_core)
            dgi_all = core.backward_bptt(d_core, bufs, self.lin_ws)
            ops.linear_backward(dgi_all, x_enc, core._params()[0], act_enc, core._params(grads=True)[0], d_enc, db_enc,
                                self.engine, self.lin_ws)
            if Le > 0:
                self._mlp_chain_backward(enc, genc, acts, dzs, 0, x0)

    def _mlp_chain_backward(self, layers, glayers, acts, dzs, first: int, x_in: Tensor, act_in: Optional[int] = None,
                            dx_in: Optional[Tensor] = None) -> None:
        """backward of the MLP layers [first, len(layers)) whose output gradients dzs[i] of acts[i] are known from the top
        one down: dW of every layer, and the gradient of every layer's input -- for layer `first` the input is x_in
        (activation act_in, gradient dx_in, or none)"""
        none = ops.ACT["none"]
        for k in range(len(layers) - 1, first - 1, -1):
            W, dW = layers[k][0], glayers[k][0]
            if k > first:
                ops.linear_backward(dzs[k], acts[k - 1], W, self.act, dW, dzs[k - 1], glayers[k - 1][1], self.engine,
                                    self.lin_ws)
            else:
                ops.linear_backward(dzs[k], x_in, W, none if act_in is None else act_in, dW, dx_in, None, self.engine,
                                    self.lin_ws)

    def exp_size_total_dev(self) -> Tensor:
        if not hasattr(self, "_exp_total"):
            self._exp_total = torch.full((1,), float(self.E * self.world_size), dtype=torch.float64, device=self.device)
        return self._exp_total

    # ------------------------------------------------------------------------------------------------------------
    def train(self, batch: Dict[str, Tensor]) -> Dict[str, float]:
        """learner.py:1036-1067. `batch` is the trajectory dict (reference layout) on this learner's device."""
        cfg = self.cfg
        if self.use_graph:
            return self._train_graphed(batch)
        if self._lr_on_device:      # graphs ran before (use_graph was switched off since): continue from the device's lr
            self._curr_lr, self._lr_on_device = float(self.lr_dev.item()), False
        launches0 = ops.launch_count()
        if self.shuffle:
            self._upload_permutation()
        self._prepare_batch(batch)
        recent_kls: List[float] = []
        prev_epoch_actor_loss = 1e9
        log_idx = reduced_upto = 0
        nmb = cfg.num_batches_per_epoch
        for epoch in range(cfg.num_epochs):
            first = log_idx
            if self.shuffle and epoch > 0:
                # the reference reshuffles at the start of every epoch (learner.py:707-713): new permutation, new gather pass
                # (the previous epoch ended with a host sync, so the pinned index buffer is free)
                self._upload_permutation()
                self._bind_minibatch_arrays(batch)
                if not cfg.with_vtrace:
                    self._minibatch_adv_partials()     # the minibatches' advantage statistics follow the new composition
            for b in range(nmb):
                self._minibatch_step(batch, b, log_idx)
                log_idx += 1
                if isinstance(self.lr_scheduler, KlAdaptiveScheduler) and self.lr_scheduler.invoke_after_each_minibatch():
                    # data parallel: the decision must be taken on the GLOBAL KL or the replicas' learning rates diverge
                    self._allreduce_loss_rows(self.loss_stats_log[log_idx - 1: log_idx])
                    reduced_upto = log_idx
                    kl = float(self.loss_stats_log[log_idx - 1, ops.LS["kl_old_mean"]].item())   # host sync by request
                    recent_kls.append(kl)
                    self.curr_lr = self.lr_scheduler.update(self.curr_lr, recent_kls)
                elif self.lr_scheduler.invoke_after_each_minibatch():
                    self.curr_lr = self.lr_scheduler.update(self.curr_lr, recent_kls)       # (linear decay: no KL needed)
            if reduced_upto < log_idx:     # data parallel: global loss statistics before any host decision / report
                self._allreduce_loss_rows(self.loss_stats_log[reduced_upto: log_idx])
                reduced_upto = log_idx
            if self._needs_epoch_sync():
                prev_epoch_actor_loss = self._end_of_epoch(first, log_idx, recent_kls, prev_epoch_actor_loss)
                if prev_epoch_actor_loss is None:
                    break
        if self.shuffle:
            self._perm_queue = []          # (permutations set for epochs an early stop skipped do not leak into the next call)
        self.num_minibatches_done = log_idx
        self.kernel_launches = ops.launch_count() - launches0   # counted by the library itself
        self._snapshot_policy_lag(batch, log_idx)
        self.env_steps += self.E * self.world_size * (cfg.env_frameskip if cfg.summaries_use_frameskip else 1)
        return dict(env_steps=self.env_steps, train_step=self.train_step)

    # ---- population-based training hooks (learner.py:388-428) ---------------------------------------------------
    def set_new_cfg(self, new_cfg: Dict) -> None:
        """Replace hyper-parameters (PBT, learner.py:394-408).  The kernels take them as launch arguments, so captured graphs
        are dropped and re-captured on the next train(); a changed learning rate applies only with lr_schedule=constant."""
        changed = False
        for key, value in new_cfg.items():
            if getattr(self.cfg, key) != value:
                setattr(self.cfg, key, value)
                changed = True
        if self.cfg.lr_schedule == "constant" and self.curr_lr != self.cfg.learning_rate:
            self.curr_lr = self.cfg.learning_rate
            changed = True
        if changed:
            self._graphs.clear()
            self._graph = None

    def load_policy_from(self, other: "Learner") -> None:
        """Take weights, normaliser and optimiser state of another policy's learner (PBT replacement: the reference loads the
        donor's checkpoint with load_progress=False, learner.py:300-310, then advances the policy version by max_policy_lag + 1
        so that experience collected with the old weights is dropped, :415-428).  Same device: device-to-device copies."""
        m, o = self.model, other.model
        m.flat.copy_(o.flat)
        m.exp_avg.copy_(o.exp_avg)
        m.exp_avg_sq.copy_(o.exp_avg_sq)
        for k in ("obs_mean", "obs_var", "obs_count", "ret_mean", "ret_var", "ret_count"):
            getattr(m, k).copy_(getattr(o, k))
        m.weights_changed()
        self.opt_step = other.opt_step
        self.curr_lr = other.curr_lr
        self.train_step += self.cfg.max_policy_lag + 1

    @property
    def curr_lr(self) -> float:
        """The learning rate.  While train() replays CUDA graphs it lives in lr_dev, where the device-side rules advance
        it: reading it then is a host sync, and setting it writes lr_dev (checkpoint resume, PBT)."""
        return float(self.lr_dev.item()) if self._lr_on_device else self._curr_lr

    @curr_lr.setter
    def curr_lr(self, lr: float) -> None:
        if self.use_graph:
            self.lr_dev.fill_(float(lr))
            self._lr_on_device = True
        else:
            self._curr_lr, self._lr_on_device = lr, False

    def _needs_epoch_sync(self) -> bool:
        """the host reads an epoch's loss rows (early stopping, kl_adaptive_epoch) unless nothing could use them"""
        return self.cfg.num_epochs > 1 or self.lr_scheduler.invoke_after_each_epoch()

    def _end_of_epoch(self, first: int, last: int, recent_kls: List[float], prev_loss: float) -> Optional[float]:
        """The host decisions after the epoch whose loss rows are [first, last), with one sync (the reference syncs per
        minibatch): the per-epoch learning-rate rule, then early stopping (:827-837).  -> the epoch's actor loss, or
        None to stop."""
        rows = self.loss_stats_log[first:last].cpu()
        if self.lr_scheduler.invoke_after_each_epoch():
            recent_kls.extend(rows[:, ops.LS["kl_old_mean"]].tolist())
            self.curr_lr = self.lr_scheduler.update(self.curr_lr, recent_kls)
        actor = rows[:, ops.LS["policy_loss"]] + rows[:, ops.LS["exploration_loss"]] + rows[:, ops.LS["kl_loss"]]
        new_loss = float(actor.mean())
        return None if abs(prev_loss - new_loss) < 1e-6 else new_loss

    def _epoch_body(self, batch: Dict[str, Tensor], epoch: int) -> None:
        """Epoch `epoch` of train() with no host dependence (the graph-capturable form).  Epoch 0 prepares the batch; a
        later epoch over shuffled minibatches gathers them in its new order first.  The per-minibatch learning-rate rules
        run on the device after every optimizer step, on the all-reduced loss row like the eager path."""
        cfg, sched = self.cfg, self.lr_scheduler
        nmb = cfg.num_batches_per_epoch
        if epoch == 0:
            self._prepare_batch(batch)
        elif self.shuffle:
            self._bind_minibatch_arrays(batch)
            if not cfg.with_vtrace:
                self._minibatch_adv_partials()
        kl_per_minibatch = isinstance(sched, KlAdaptiveScheduler) and sched.invoke_after_each_minibatch()
        first = epoch * nmb
        for b in range(nmb):
            i = first + b
            self._minibatch_step(batch, b, i)
            if kl_per_minibatch:
                self._allreduce_loss_rows(self.loss_stats_log[i: i + 1])
                ops.lr_schedule_kl_adaptive(self.lr_dev, self.loss_stats_log[i, ops.LS["kl_old_mean"]], sched.thr,
                                            sched.min_lr, sched.max_lr)
            elif isinstance(sched, LinearDecayScheduler):
                ops.lr_schedule_linear_decay(self.lr_dev, self.counters_dev[2:3], sched.num_updates, sched.lr0)
        if not kl_per_minibatch:
            self._allreduce_loss_rows(self.loss_stats_log[first: first + nmb])

    def _run_epoch(self, batch: Dict[str, Tensor], ptrs: tuple, epoch: int) -> int:
        """Epoch `epoch` of a graphed train(): eagerly the first time any trajectory set reaches it (kernel attributes,
        allocator warm-up), then captured once per trajectory set and replayed.  -> the launches replayed."""
        if epoch not in self._epoch_launches:
            n0 = ops.launch_count()
            self._epoch_body(batch, epoch)
            self._epoch_launches[epoch] = ops.launch_count() - n0
            return 0
        graph = self._graphs.get((ptrs, epoch))
        captured = graph is None
        if captured:
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            # (multi-rank with NCCL exchanges: the watchdog thread polls events while this thread captures)
            mode = "thread_local" if (self.world_size > 1 and self.comm is None) else "global"
            with torch.cuda.graph(graph, capture_error_mode=mode):
                self._epoch_body(batch, epoch)
            self._graphs[(ptrs, epoch)] = graph
        self._graph = graph
        graph.replay()
        return 0 if captured else self._epoch_launches[epoch]     # (a capture pass counted its launches itself)

    def _train_graphed(self, batch: Dict[str, Tensor]) -> Dict[str, float]:
        """train() as one graph launch per epoch, with the eager path's host sync between two epochs only where it has a
        decision to take.  Host mirrors of the counters advance by the minibatches that ran."""
        cfg, sched = self.cfg, self.lr_scheduler
        nmb = cfg.num_batches_per_epoch
        # one captured graph per trajectory set (the runner may train on several row ranges of the rollout buffers, or on an
        # accumulation buffer: cfg/arguments.py:147-178 allows datasets that are a fraction / a multiple of one rollout)
        ptrs = tuple(v.data_ptr() for v in batch.values())
        # the device counters follow the host values whenever these were changed from outside (checkpoint resume)
        decay_step = sched.step if isinstance(sched, LinearDecayScheduler) else 0
        self.counters_dev.copy_(torch.tensor([self.opt_step, self.train_step, decay_step], dtype=torch.int64),
                                non_blocking=True)
        if not self._lr_on_device:
            self.lr_dev.fill_(float(self._curr_lr))
            self._lr_on_device = True
        opt0, train0 = self.opt_step, self.train_step
        recent_kls: List[float] = []
        prev_epoch_actor_loss = 1e9
        done = replayed = launches = 0
        for epoch in range(cfg.num_epochs):
            if self.shuffle:
                self._upload_permutation()       # (H2D copy enqueued in front of the graph; the gathers are captured)
            replayed += self._run_epoch(batch, ptrs, epoch)
            launches += self._epoch_launches[epoch]
            done += nmb
            if self._needs_epoch_sync():
                prev_epoch_actor_loss = self._end_of_epoch(done - nmb, done, recent_kls, prev_epoch_actor_loss)
                if prev_epoch_actor_loss is None:
                    break
        if self.shuffle:
            self._perm_queue = []
        # _minibatch_step advanced the host mirrors during eager / capture passes only: set them explicitly
        self.opt_step, self.train_step = opt0 + done, train0 + done
        if isinstance(sched, LinearDecayScheduler):
            sched.step += done
        self.num_minibatches_done = done
        self._snapshot_policy_lag(batch, done)
        self.kernel_launches = launches
        self._replayed_launches = replayed
        self.env_steps += self.E * self.world_size * (cfg.env_frameskip if cfg.summaries_use_frameskip else 1)
        return dict(env_steps=self.env_steps, train_step=self.train_step)

    @property
    def graph_replay_launches(self) -> int:
        """kernel launches of the last train() that happened through graph replay (not seen by the launch counter)"""
        return self._replayed_launches if self.use_graph else 0

    def _snapshot_policy_lag(self, batch: Dict[str, Tensor], n: int) -> None:
        """Keep the last minibatch's policy versions: the caller may overwrite the trajectory set (async join) before
        fetch_stats() is asked for the policy lag."""
        bi = (n - 1) % self.cfg.num_batches_per_epoch          # position of the last minibatch inside its epoch
        sl = slice(bi * self.cfg.batch_size, (bi + 1) * self.cfg.batch_size)
        if not hasattr(self, "_lag_pv"):
            self._lag_pv = torch.empty(self.cfg.batch_size, dtype=torch.float32, device=self.device)
            self._lag_pid = torch.empty(self.cfg.batch_size, dtype=torch.int32, device=self.device)
        ops.copy_rows_bytes(batch["policy_version"].view(self.E)[sl].view(1, -1), self._lag_pv.view(1, -1))
        ops.copy_rows_bytes(batch["policy_id"].view(self.E)[sl].view(1, -1), self._lag_pid.view(1, -1))
        self._lag = (self._lag_pv, self._lag_pid, self.train_step - 1)

    def fetch_stats(self) -> Dict[str, float]:
        """Loss summaries of the LAST minibatch of the last train() (learner.py:843-923 keys). Host sync."""
        n = getattr(self, "num_minibatches_done", 0)
        if n == 0:
            return {}
        row = self.loss_stats_log[n - 1].cpu().tolist()
        out = {k: row[i] for k, i in ops.LS.items()}
        out["grad_norm"] = float(self.grad_norm_log[n - 1].item())
        out["lr"] = self.curr_lr
        out["loss"] = out["total_loss"]
        out["adam_max_second_moment"] = float(self.model.exp_avg_sq.max().item())            # learner.py:908-913
        lag = getattr(self, "_lag", None)
        if lag is not None:   # policy lag of the last minibatch (learner.py:915-918)
            pv, pid, version = lag
            vd = (float(version) - pv)[pid == self.policy_id]
            if vd.numel() > 0:
                out["version_diff_avg"], out["version_diff_min"], out["version_diff_max"] = (
                    float(vd.mean().item()), float(vd.min().item()), float(vd.max().item()))
        return out

    def minibatch_log(self) -> Tensor:
        """[num_minibatches_done, LS_SIZE] float64 (host) -- per-minibatch loss terms of the last train()."""
        return self.loss_stats_log[: self.num_minibatches_done].cpu()
