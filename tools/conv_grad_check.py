"""Gradient accuracy of the conv encoder's backward at the cfg-4 parity shape: Adam's first moment after ONE SGD step
(= 0.1 x clipped gradient) for the wgmma 3xTF32 engine and the exact-fp32 CUDA-core engine against the CPU oracle."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from oracle import appo_oracle as O
from tests.test_gpu_engine import build

dev = torch.device("cuda", 0)
N, T = 256, 8
ocfg = O.OracleCfg(obs_dim=4 * 84 * 84, obs_shape=(4, 84, 84), num_actions=6, encoder_conv_architecture="convnet_atari",
                   encoder_conv_mlp_layers=[512], encoder_mlp_layers=[], nonlinearity="relu", obs_scale=255.0, rollout=T,
                   recurrence=1, batch_size=N * T, num_batches_per_epoch=1, exploration_loss_coeff=0.01, max_grad_norm=0.5,
                   adam_eps=1e-5)
st0 = O.init_state(ocfg, seed=5)
gen = torch.Generator().manual_seed(23)
tape = torch.randint(0, 256, (T + 1, N, ocfg.obs_dim), dtype=torch.uint8, generator=gen)
olearner = O.OracleLearner(ocfg, st0)
oenv = O.TapeVecEnv(tape, ocfg.num_actions)
otraj = O.alloc_trajectories(ocfg, N)
noise = torch.empty(T, N, 6).exponential_(generator=gen)
O.rollout(ocfg, olearner.st, oenv, oenv.reset(), otraj, noise, 0)
olearner.train(otraj)
for engine in ("simt", "3xtf32"):
    cfg, model, traj, env, sampler, learner = build(ocfg, N, st0, tape, dev, engine=engine)
    for k, v in otraj.items():
        if k in traj:
            traj[k].copy_(v.view(traj[k].shape))
    learner.train(traj)
    torch.cuda.synchronize()
    print(f"engine {engine}: grad_norm {learner.grad_norm_log[0].item():.6f} (oracle {olearner.log[0]['grad_norm']:.6f})")
    for k in O.param_names(ocfg):
        off, shp = model._slices[k]
        m_dev = model.exp_avg[off: off + int(np.prod(shp))].view(shp).cpu().double()
        m_ref = olearner.m[k].double()
        rel = float((m_dev - m_ref).norm() / (m_ref.norm() + 1e-30))
        print(f"   {k:60s} |m| {float(m_ref.abs().max()):.3e}  max abs diff {float((m_dev - m_ref).abs().max()):.3e}  rel L2 {rel:.3e}")
