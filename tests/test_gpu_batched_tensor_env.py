"""Batched tensor envs (IsaacGym / Brax style) on the device path: sfb200_env_ingest against torch's conversions, the
reference-executed fixtures through BatchedTensorEnvAdapter (env on the CPU with numpy actions -- how the reference made
them -- and on CUDA with device actions), bit-identity with the native TapeVecEnv path (worker_num_splits = 2, step
graphs, the async runner), no host synchronisation per step, and a torch CartPole trained through run_rl and enjoyed."""
import math

import numpy as np
import pytest
import torch

from gymnasium import spaces
from oracle import appo_oracle as O
from tests import dict_obs_oracle as DO
from tests.device_harness import DEV, TOL, build, build_case, make_cfg, ops_for
from tests.golden_utils import load_case, load_mixed_case, state_from

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ kernel
def _values(dtype, shape, gen):
    """seeded values of `dtype` that include the conversions' edge cases: ties and values that round (float64, 32/64-bit
    integers), float32 denormals / overflow / underflow from float64, zeros and negative zeros"""
    if dtype == torch.bool:
        return torch.randint(0, 2, shape, generator=gen).bool()
    if dtype.is_floating_point:
        x = torch.randn(shape, generator=gen, dtype=torch.float64) * 300.0
        flat = x.view(-1)
        special = [0.0, -0.0, 1.0 + 2.0 ** -24, 1.0 + 3 * 2.0 ** -24, 2.0 ** -140, 1e-300, -1e-300, 3.5e38, -1e39, 0.1]
        k = min(len(special), flat.numel())
        flat[:k] = torch.tensor(special[:k], dtype=torch.float64)
        return x.to(dtype)
    info = torch.iinfo(dtype)
    x = torch.randint(max(info.min, -2 ** 62), min(info.max, 2 ** 62), shape, generator=gen, dtype=torch.int64)
    flat = x.view(-1)
    special = [0, 2 ** 40 + 1, 2 ** 25 + 1, 2 ** 25 + 3, -(2 ** 53 + 1), 2 ** 63 - 1, 2 ** 24 + 1, -(2 ** 31), 127, -128]
    special = [v for v in special if info.min <= v <= info.max]
    flat[:len(special[:flat.numel()])] = torch.tensor(special[:flat.numel()], dtype=torch.int64)
    return x.to(dtype)


def _bits(t):
    return t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t


DTYPES = [torch.float32, torch.float16, torch.bfloat16, torch.float64, torch.int8, torch.int16, torch.int32, torch.int64,
          torch.uint8, torch.bool]


@pytest.mark.parametrize("n", [1, 37, 1029, 4099])
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_ingest_matches_torch_conversions(dtype, n):
    """keys of 3 / 5 / 1 / 9 / 16 columns at odd column offsets, with dense, strided (padded or misaligned) and 3-D rows;
    a dense reward-like vector; a bool x != 0 mask -- bit-equal to .to(torch.float32) and != 0"""
    ops = ops_for()
    gen = torch.Generator().manual_seed(n * 31 + DTYPES.index(dtype))
    keys = []
    for i, cols in enumerate([3, 5, 1, 9, 16]):
        if i % 3 == 0:
            src = _values(dtype, (n, cols), gen)                             # dense rows
        elif i % 3 == 1:
            src = _values(dtype, (n, cols + 3), gen)[:, 1:1 + cols]          # padded rows, misaligned start
        else:
            src = _values(dtype, (n, 2, 2 * cols), gen)[:, 1, :cols]         # every other row of a 3-D tensor
        keys.append(src.to(DEV))
    width = 1 + sum(k.shape[1] for k in keys) + 2
    obs = torch.full((n, width), float("nan"), device=DEV)
    rew = torch.full((n, 1), float("nan"), device=DEV)
    mask_src = _values(dtype, (n, 7), gen).to(DEV)
    mask = torch.zeros((n, 7), dtype=torch.bool, device=DEV)
    vec = _values(dtype, (n,), gen).to(DEV)
    entries, c = [], 1
    for k in keys:
        entries.append((k, k.stride(0), k.shape[1], obs, c, ops.INGEST_F32))
        c += k.shape[1]
    entries += [(vec, 1, 1, rew, 0, ops.INGEST_F32), (mask_src, 7, 7, mask, 0, ops.INGEST_BOOL)]
    ops.env_ingest(entries, n)
    torch.cuda.synchronize()
    c = 1
    for k in keys:
        want = k.cpu().to(torch.float32)
        assert torch.equal(_bits(obs[:, c:c + k.shape[1]].cpu()), _bits(want)), (dtype, c)
        c += k.shape[1]
    assert torch.isnan(obs[:, 0]).all() and torch.isnan(obs[:, c:]).all()        # nothing outside the keys' columns
    assert torch.equal(_bits(rew.view(-1).cpu()), _bits(vec.cpu().to(torch.float32)))
    assert torch.equal(mask.cpu(), mask_src.cpu() != 0)
    if dtype == torch.uint8:        # image rows: uint8 copy, padded rows and an odd row length
        img = _values(torch.uint8, (n, 3 * 8 * 8 + 5), gen).to(DEV)[:, 2:2 + 3 * 8 * 8]
        out = torch.zeros((n, 3 * 8 * 8), dtype=torch.uint8, device=DEV)
        ops.env_ingest([(img, img.stride(0), img.shape[1], out, 0, ops.INGEST_U8)], n)
        assert torch.equal(out, img)


# ------------------------------------------------------------------------------------------------ test env
class TensorTapeEnv:
    """The tape env behind the reference's batched-env contract (what tests/golden/make_golden.py's RefTapeEnv drives the
    reference through): one env with num_agents = N whose reset() / step() return FRESH tensors every call, on the CPU or
    on CUDA.  Dtypes vary: float64 rewards, int64 terminated, uint8 truncated and action mask, optionally float64
    observations; Dict observations come as column slices of one tensor (strided rows); an extra key "states" is returned
    that the observation space does not declare."""

    def __init__(self, inner, on_cpu=False, obs_dtype=torch.float32):
        self.e, self.on_cpu, self.obs_dtype = inner, on_cpu, obs_dtype
        self.num_agents = inner.num_agents
        self.is_multiagent = True
        A = inner.num_actions
        box = lambda d: spaces.Box(-np.inf, np.inf, (d,), np.float32)
        if inner.obs_keys:
            obs = {k: box(d) for k, d in inner.obs_keys}
        elif inner.obs_shape is not None:
            obs = {"obs": spaces.Box(0, 255, inner.obs_shape, np.uint8)}
        else:
            obs = {"obs": box(inner.obs_dim)}
        if inner.with_action_mask:
            obs["action_mask"] = spaces.Box(0, 1, (A,), np.uint8)
        self.observation_space = spaces.Dict(obs)
        if inner.action_heads:
            self.action_space = spaces.Tuple([spaces.Discrete(n) if k == "discrete" else spaces.Box(-1.0, 1.0, (n,), np.float32)
                                              for k, n in inner.action_heads])
        elif inner.action_segments:
            self.action_space = spaces.Tuple([spaces.Discrete(n) for n in inner.action_segments])
        elif inner.continuous:
            self.action_space = spaces.Box(-1.0, 1.0, (A,), np.float32)
        else:
            self.action_space = spaces.Discrete(A)
        self.resets = self.steps = 0

    def _move(self, t):
        return t.cpu() if self.on_cpu else t

    def _obs(self, o):
        mask = None
        if isinstance(o, dict):
            o, mask = o["obs"], o["action_mask"]
        e = self.e
        if e.obs_shape is not None:
            out = {"obs": self._move(o.view(self.num_agents, *e.obs_shape).clone())}
        else:
            full = self._move(o.to(self.obs_dtype, copy=True))
            if e.obs_keys:
                out, c = {}, 0
                for k, d in e.obs_keys:
                    out[k] = full[:, c:c + d]
                    c += d
            else:
                out = {"obs": full}
        out["states"] = self._move(torch.zeros(self.num_agents, 5, device=o.device))
        if mask is not None:
            out["action_mask"] = self._move(mask.to(torch.uint8))
        return out

    def reset(self, **kw):
        self.resets += 1
        return self._obs(self.e.reset()), {}

    def step(self, actions):
        self.steps += 1
        dev = self.e.tape.device
        if isinstance(actions, list):
            actions = [torch.as_tensor(a).to(dev) for a in actions]
        else:
            actions = torch.as_tensor(actions).to(dev)
        obs, rew, term, trunc = self.e.step(actions)
        return (self._obs(obs), self._move(rew.double()), self._move(term.to(torch.int64)),
                self._move(trunc.to(torch.uint8)), {})


def _adapter(inner, on_cpu, **kw):
    from sample_factory_b200.host_env import BatchedTensorEnvAdapter

    return BatchedTensorEnvAdapter(TensorTapeEnv(inner, on_cpu, **kw), DEV, env_gpu_actions=not on_cpu)


# ------------------------------------------------------------------------------------------------ vs the reference
GOLDEN = ["tiny_gae", "tiny_gauss", "tiny_tuple", "tiny_conv", "tiny_mask", "tiny_mixed", "tiny_dict"]


def _golden_setup(name):
    """(z, meta, ocfg, cfg, model, traj, native tape env, learner) of a reference-executed fixture"""
    load = {"tiny_mixed": load_mixed_case, "tiny_dict": DO.load_dict_case}.get(name, load_case)
    z, meta, ocfg = case = load(name)
    cfg, model, traj, env, sampler, learner = build_case(case, "simt")
    return z, meta, ocfg, cfg, model, traj, env, learner


@pytest.mark.parametrize("where", ["cpu", "cuda"])
@pytest.mark.parametrize("name", GOLDEN)
def test_adapter_matches_reference_golden(name, where):
    """the sampler over the adapter, then the learner on what it sampled, against the reference's own trajectories and
    post-Adam weights: Discrete actions bit-exact, policy outputs 1e-5, weights 2e-5"""
    from sample_factory_b200.sampler import DeviceSampler

    ops = ops_for()
    z, meta, ocfg, cfg, model, traj, native, learner = _golden_setup(name)
    env = _adapter(native, where == "cpu", obs_dtype=torch.float64 if name == "tiny_gae" else torch.float32)
    assert (env.obs_dim, env.num_actions, env.obs_uint8) == (model.spec.obs_dim, model.spec.num_actions, model.spec.obs_uint8)
    sampler = DeviceSampler(cfg, env, model, traj, engine=ops.GEMM_SIMT)
    float_actions = bool(getattr(ocfg, "continuous", False) or getattr(ocfg, "action_heads", None))
    sampler.reset()
    for it in range(meta["iters"]):
        model.load_state_dict(state_from(z, "init/") if it == 0 else state_from(z, f"it{it - 1}/state/"), strict=False)
        sampler.set_policy_version(int(z[f"it{it}/train_step_before"]))
        sampler.noise = torch.from_numpy(z[f"it{it}/noise"]).to(DEV).contiguous()
        sampler.rollout()
        got = {k: v.cpu() for k, v in traj.items()}
        ref = {k: torch.from_numpy(z[f"it{it}/traj/{k}"]) for k in
               ["obs", "actions", "action_logits", "log_prob_actions", "values", "rewards", "dones", "time_outs"]
               if f"it{it}/traj/{k}" in z.files}
        for k in ["obs", "dones", "time_outs"] + ([] if float_actions else ["rewards", "actions"]):
            if k in ref:
                assert torch.equal(got[k].view(ref[k].shape), ref[k]), (name, it, k)
        if float_actions:
            np.testing.assert_allclose(got["actions"].view(ref["actions"].shape).numpy(), ref["actions"].numpy(),
                                       rtol=2e-5, atol=TOL)
            np.testing.assert_allclose(got["rewards"].view(ref["rewards"].shape).numpy(), ref["rewards"].numpy(), atol=TOL)
        for k in ["action_logits", "log_prob_actions"]:
            np.testing.assert_allclose(got[k].view(ref[k].shape).numpy(), ref[k].numpy(), atol=TOL, err_msg=k)
        np.testing.assert_allclose(got["values"][:, :-1].numpy(), ref["values"][:, :-1].numpy(), atol=TOL)
        if meta.get("poison") and it == meta["iters"] - 1:
            continue            # the reference trained on deliberately stale samples there
        assert learner.train_step == int(z[f"it{it}/train_step_before"])
        learner.train(traj)
        torch.cuda.synchronize()
        got_state = model.state_dict()
        for k, v in state_from(z, f"it{it}/state/").items():
            tol = (1e-6 if k.startswith("returns_normalizer") else 1e-8) if v.dtype == torch.float64 else 2 * TOL
            np.testing.assert_allclose(got_state[k].cpu().numpy().reshape(v.shape), v.numpy(), atol=tol, rtol=1e-6,
                                       err_msg=f"{name} it{it} {k}")
    assert env.env.resets == 1 and env.env.steps == meta["iters"] * ocfg.rollout


# ------------------------------------------------------------------------------------------------ vs the native env
def _cfg2_small(N, T):
    ocfg = O.OracleCfg(rollout=T, recurrence=1, batch_size=N * T // 2, num_batches_per_epoch=2, num_epochs=1,
                       encoder_mlp_layers=[128, 128])
    tape = (torch.randn(4 * T + 1, N, ocfg.obs_dim, generator=torch.Generator().manual_seed(5)) * 1.1).to(DEV)
    return ocfg, tape


def _collect(sampler, traj, n):
    outs = []
    sampler.reset()
    for _ in range(n):
        sampler.rollout()
        torch.cuda.synchronize()
        outs.append({k: v.clone() for k, v in traj.items() if k != "valids"})
    return outs


def _assert_same(a, b):
    for x, y in zip(a, b):
        for k in x:
            assert torch.equal(x[k], y[k]), k


@pytest.mark.parametrize("where", ["cpu", "cuda"])
def test_adapter_rollouts_are_bit_identical_to_the_native_env(where, monkeypatch):
    """one sampler (eager, then the per-step graphs of host envs) and worker_num_splits = 2 (two adapters, each on its own
    stream) reproduce the native TapeVecEnv rollouts bit for bit (Philox noise, the native path's per-step launches)"""
    from sample_factory_b200.envs import TapeVecEnv
    from sample_factory_b200.sampler import DeviceSampler, SplitSampler

    monkeypatch.setenv("SFB200_TAIL_FUSED", "0")
    ops = ops_for()
    N, T = 256, 16
    ocfg, tape = _cfg2_small(N, T)
    cfg, model, traj, _, _, _ = build(ocfg, N, O.init_state(ocfg, seed=8), tape.cpu())
    kw = dict(engine=ops.GEMM_SIMT, philox_seed=3)
    native = _collect(DeviceSampler(cfg, TapeVecEnv(tape, ocfg.num_actions), model, traj, **kw), traj, 3)
    for graph in (False, True):
        s = DeviceSampler(cfg, _adapter(TapeVecEnv(tape, ocfg.num_actions), where == "cpu"), model, traj, use_cuda_graph=graph, **kw)
        _assert_same(native, _collect(s, traj, 3))
        assert s.graph_replay_launches > 0 if graph else True
    h = N // 2
    halves = lambda: [TapeVecEnv(tape[:, :h].contiguous(), ocfg.num_actions, env_index_offset=0),
                      TapeVecEnv(tape[:, h:].contiguous(), ocfg.num_actions, env_index_offset=h)]
    native = _collect(SplitSampler(cfg, halves(), model, traj, **kw), traj, 3)
    split = SplitSampler(cfg, [_adapter(e, where == "cpu") for e in halves()], model, traj, **kw)
    _assert_same(native, _collect(split, traj, 3))


def test_async_runner_over_the_adapter_matches_the_native_env(tmp_path, monkeypatch):
    """async_rl (the sampler on its own stream, one rollout ahead of the learner): trajectories and weights after every
    iteration are bit-identical to the same runner over the native env"""
    from sample_factory_b200.envs import TapeVecEnv, register_env
    from sample_factory_b200.host_env import BatchedTensorEnvAdapter
    from sample_factory_b200.train import Runner

    monkeypatch.setenv("SFB200_TAIL_FUSED", "0")
    N, T = 128, 16
    ocfg, tape = _cfg2_small(N, T)
    register_env("bt_native", lambda n, c, e, render_mode=None: TapeVecEnv(tape, ocfg.num_actions))
    register_env("bt_tensor", lambda n, c, e, render_mode=None: TensorTapeEnv(TapeVecEnv(tape, ocfg.num_actions)))
    runs = []
    for name in ("bt_native", "bt_tensor"):
        cfg = make_cfg(ocfg, env=name, train_dir=str(tmp_path), experiment=name, cuda_graph=False, seed=0,
                         gemm_engine="simt", async_rl=True, restart_behavior="overwrite", env_gpu_actions=True)
        r = Runner(cfg)
        assert r.init() == 0
        assert isinstance(r.env, BatchedTensorEnvAdapter) == (name == "bt_tensor")
        out = []
        for _ in range(3):
            r.iteration()
            torch.cuda.synchronize()
            out.append({"flat": r.model.flat.clone(), **{k: v.clone() for k, v in r.traj.items() if k != "valids"}})
        runs.append(out)
    _assert_same(*runs)


def test_cuda_env_with_gpu_actions_never_synchronises_the_host():
    """a CUDA batched env with env_gpu_actions: after the first (eager) rollout and the graph capture, rollouts run under
    torch.cuda.set_sync_debug_mode("error")"""
    from sample_factory_b200.envs import TapeVecEnv
    from sample_factory_b200.sampler import DeviceSampler

    ops = ops_for()
    N, T = 256, 16
    ocfg, tape = _cfg2_small(N, T)
    cfg, model, traj, _, _, _ = build(ocfg, N, O.init_state(ocfg, seed=8), tape.cpu())
    for graph in (False, True):
        s = DeviceSampler(cfg, _adapter(TapeVecEnv(tape, ocfg.num_actions), False), model, traj, engine=ops.GEMM_SIMT,
                          use_cuda_graph=graph)
        s.reset()
        s.rollout()
        s.rollout()
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            for _ in range(2):
                s.rollout()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        torch.cuda.synchronize()
        assert torch.isfinite(traj["values"]).all()


# ------------------------------------------------------------------------------------------------ end to end
class TorchCartPole:
    """N cart-poles simulated with torch on the device -- the shape of a BraxEnv / IsaacGymVecEnv: one env, num_agents = N,
    reset(seed) -> (obs, info), step(actions) -> (obs, reward, terminated, truncated, infos), auto-reset inside"""

    def __init__(self, n=1024, max_steps=200, device=DEV):
        self.num_agents, self.is_multiagent, self.max_steps, self.device = n, True, max_steps, device
        self.observation_space = spaces.Box(-np.inf, np.inf, (4,), np.float32)
        self.action_space = spaces.Discrete(2)
        self.gen = torch.Generator(device=device).manual_seed(0)
        self.s = torch.zeros(n, 4, device=device)
        self.t = torch.zeros(n, dtype=torch.int32, device=device)

    def _reset_rows(self, rows):
        fresh = (torch.rand(self.num_agents, 4, generator=self.gen, device=self.device) - 0.5) * 0.1
        self.s = torch.where(rows.view(-1, 1), fresh, self.s)
        self.t = torch.where(rows, torch.zeros_like(self.t), self.t)

    def reset(self, seed=None):
        if seed is not None:
            self.gen.manual_seed(seed)
        self._reset_rows(torch.ones(self.num_agents, dtype=torch.bool, device=self.device))
        return self.s.clone(), {}

    def step(self, actions):
        x, xd, th, thd = self.s.unbind(1)
        f = torch.where(actions.view(-1) == 1, 10.0, -10.0)
        ct, st = torch.cos(th), torch.sin(th)
        tmp = (f + 0.05 * thd * thd * st) / 1.1
        tha = (9.8 * st - ct * tmp) / (0.5 * (4.0 / 3.0 - 0.1 * ct * ct / 1.1))
        xa = tmp - 0.05 * tha * ct / 1.1
        self.s = torch.stack([x + 0.02 * xd, xd + 0.02 * xa, th + 0.02 * thd, thd + 0.02 * tha], 1)
        self.t += 1
        terminated = (self.s[:, 0].abs() > 2.4) | (self.s[:, 2].abs() > 12 * math.pi / 180)
        truncated = (self.t >= self.max_steps) & ~terminated
        self._reset_rows(terminated | truncated)
        return self.s.clone(), torch.ones(self.num_agents, device=self.device), terminated, truncated, {}


def test_torch_cartpole_trains_through_run_rl_and_enjoys(tmp_path):
    """run_rl's sequence (make_runner, init, run) on 1024 torch cart-poles on the GPU with device actions: a report of the
    last 10 reaches a mean episode length of 100 steps and three times the first report's (a random policy lasts ~22),
    and enjoy() loads the checkpoint run() saved and runs the 1024 agents of the one env"""
    from sample_factory_b200.cfg import parse_full_cfg, parse_sf_args
    from sample_factory_b200.enjoy import enjoy
    from sample_factory_b200.envs import register_env
    from sample_factory_b200.host_env import BatchedTensorEnvAdapter
    from sample_factory_b200.train import make_runner

    ops_for()
    register_env("TorchCartPole-v0", lambda name, cfg, env_config, render_mode=None: TorchCartPole())
    iters = 150
    argv = ["--env=TorchCartPole-v0", "--experiment=torch_cartpole", f"--train_dir={tmp_path}", "--restart_behavior=overwrite",
            "--use_rnn=False", "--recurrence=1", "--rollout=32", "--batch_size=8192", "--num_batches_per_epoch=4",
            "--num_epochs=4", "--encoder_mlp_layers", "64", "64", "--nonlinearity=tanh", "--learning_rate=0.001",
            "--reward_scale=0.1", "--gamma=0.99", "--exploration_loss_coeff=0.001", "--async_rl=False", "--seed=0",
            "--env_gpu_actions=True", "--batched_sampling=True", "--num_workers=1", "--num_envs_per_worker=1",
            "--worker_num_splits=1", f"--train_for_env_steps={iters * 1024 * 32}", "--save_every_sec=100000",
            "--experiment_summaries_interval=0"]
    parser, _ = parse_sf_args(argv)
    cfg = parse_full_cfg(parser, argv)
    cfg, runner = make_runner(cfg)
    assert runner.init() == 0
    assert isinstance(runner.env, BatchedTensorEnvAdapter) and runner.env.num_agents == 1024
    lens = []
    runner.register_episodic_stats_handler(lambda r, ep, policy: lens.append(ep.get("len", 0.0)))
    assert runner.run() == 0
    assert len(lens) == iters and runner.env_steps == iters * 1024 * 32
    print("mean episode length per iteration:", [round(v, 1) for v in lens[::10]], lens[-10:])
    assert max(lens[-10:]) > 100 and max(lens[-10:]) > 3 * lens[0], lens
    cfg.cli_args = dict(max_num_episodes=64)
    cfg.max_num_episodes = 64
    status, avg = enjoy(cfg)
    assert status == 0 and avg > 15.0, avg          # reward 1 per step
