"""Data-parallel exchange micro-benchmark + correctness check (run under torch.distributed.run, one process per GPU):

  * sfb200_dp_allreduce_f64 / sfb200_dp_pooled_moments against torch.distributed (NCCL) results,
  * sfb200_dp_grad_allreduce_clip_adam (ONE kernel: NVLink peer pull + grad-norm + clip + Adam) against
    NCCL all-reduce + sfb200_clip_adam_step on the same inputs (bit-identical replicas, 1e-7 vs the NCCL sum order),
  * device time per SGD-step exchange, eager and replayed from a CUDA graph, next to ncclAllReduce + the two-kernel Adam.

    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 tools/dp_comm_bench.py
Prints one JSON line on rank 0."""
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sample_factory_b200 import ops  # noqa: E402
from sample_factory_b200.dist_utils import PeerComm, init_from_env, pooled_moments_  # noqa: E402


def timed(fn, iters=200, warm=20):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    t = torch.tensor([e0.elapsed_time(e1) / iters * 1e3], dtype=torch.float64, device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())     # us per call, max over ranks


def main():
    rank, local_rank, world = init_from_env("nccl")
    dev = torch.device("cuda", local_rank)
    torch.cuda.set_device(dev)
    ops.bind_device(dev)
    n = int(os.environ.get("DP_BENCH_PARAMS", 300553 + 87))       # cfg-2 model (padded flat buffer)
    n = (n + 63) // 64 * 64
    comm = PeerComm(dev, n)
    g = torch.Generator(device=dev).manual_seed(100 + rank)
    out = dict(world=world, params=n)

    # ---- small fp64 all-reduce
    buf = torch.randn(4, 16, dtype=torch.float64, device=dev, generator=g)
    ref = buf.clone()
    dist.all_reduce(ref)
    mine = buf.clone()
    ops.dp_allreduce_f64(comm.comm, mine)
    torch.cuda.synchronize()
    out["f64_sum_max_abs_diff"] = float((mine - ref).abs().max())
    a = buf.clone()
    dist.all_reduce(mx := buf.clone(), op=dist.ReduceOp.MAX)
    dist.all_reduce(mn := buf.clone(), op=dist.ReduceOp.MIN)
    ops.dp_allreduce_f64(comm.comm, a, 16, max_mask=1 << 3, min_mask=1 << 5, keep_mask=1 << 0)
    torch.cuda.synchronize()
    assert torch.equal(a[:, 3], mx[:, 3]) and torch.equal(a[:, 5], mn[:, 5]) and torch.equal(a[:, 0], buf[:, 0])
    assert torch.allclose(a[:, 1], ref[:, 1], rtol=1e-14)
    # ---- pooled moments
    x = torch.randn(1000, 64, device=dev, generator=g) * (1 + rank) + rank
    bm, bv = x.mean(0), x.var(0)
    bm2, bv2 = bm.clone(), bv.clone()
    pooled_moments_(bm, bv, 1000)
    ops.dp_pooled_moments(comm.comm, bm2, bv2, 1000)
    torch.cuda.synchronize()
    out["pooled_moments_max_abs_diff"] = float(max((bm - bm2).abs().max(), (bv - bv2).abs().max()))

    # ---- fused gradient all-reduce + clip + Adam vs NCCL + clip_adam_step
    p0 = torch.randn(n, device=dev, generator=torch.Generator(device=dev).manual_seed(7)) * 0.05   # same on all ranks
    grad = torch.randn(n, device=dev, generator=g)
    comm.grad.copy_(grad)
    nv = torch.full((1,), 1000.0, dtype=torch.float64, device=dev)
    tot = torch.full((1,), 1024.0, dtype=torch.float64, device=dev)
    gn_a, gn_b = torch.zeros(1, device=dev), torch.zeros(1, device=dev)
    ws = torch.zeros(1024, device=dev)
    pa, ma, va = p0.clone(), torch.zeros(n, device=dev), torch.zeros(n, device=dev)
    pb, mb, vb = p0.clone(), torch.zeros(n, device=dev), torch.zeros(n, device=dev)
    gred = torch.zeros(n, device=dev)
    for step in (1, 2, 3):
        gsum = grad.clone()
        dist.all_reduce(gsum)
        ops.clip_adam_step(pa, gsum, ma, va, step, 1e-3, 0.9, 0.999, 1e-6, 4.0, nv, tot, gn_a, ws)
        ops.dp_grad_allreduce_clip_adam(comm.comm, gred, pb, mb, vb, step, None, 1e-3, None, 0.9, 0.999, 1e-6, 4.0, nv, tot,
                                        gn_b, comm.workspace)
    torch.cuda.synchronize()
    out["adam_params_max_abs_diff_vs_nccl"] = float((pa - pb).abs().max())
    out["grad_norm_rel_diff"] = float(((gn_a - gn_b).abs() / gn_a).item())
    ref_p = pb.clone()
    dist.broadcast(ref_p, src=0)
    out["replicas_bit_identical"] = bool(torch.equal(ref_p, pb))

    # ---- timings (us per SGD-step exchange, max over ranks)
    gtmp = grad.clone()

    def nccl_path():
        dist.all_reduce(gtmp)
        ops.clip_adam_step(pa, gtmp, ma, va, 4, 1e-3, 0.9, 0.999, 1e-6, 4.0, nv, tot, gn_a, ws)

    def peer_path():
        ops.dp_grad_allreduce_clip_adam(comm.comm, gred, pb, mb, vb, 4, None, 1e-3, None, 0.9, 0.999, 1e-6, 4.0, nv, tot, gn_b,
                                        comm.workspace)

    def peer_small():
        ops.dp_allreduce_f64(comm.comm, mine)

    def nccl_small():
        dist.all_reduce(ref)

    out["us_nccl_allreduce_plus_clip_adam"] = timed(nccl_path)
    out["us_nccl_allreduce_only"] = timed(lambda: dist.all_reduce(gtmp))
    out["us_peer_fused_allreduce_clip_adam"] = timed(peer_path)
    out["us_single_gpu_clip_adam_only"] = timed(lambda: ops.clip_adam_step(pa, gtmp, ma, va, 4, 1e-3, 0.9, 0.999, 1e-6, 4.0, nv, tot, gn_a, ws))
    out["us_peer_f64_allreduce_64"] = timed(peer_small)
    out["us_nccl_f64_allreduce_64"] = timed(nccl_small)
    # replayed from a CUDA graph (what the learner does): 4 SGD-step exchanges per graph
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=side):
            for _ in range(4):
                peer_path()
    torch.cuda.synchronize()
    out["us_peer_fused_in_graph"] = timed(gr.replay, iters=100) / 4
    ref_p = pb.clone()
    dist.broadcast(ref_p, src=0)
    out["replicas_bit_identical_after_graph"] = bool(torch.equal(ref_p, pb))
    if rank == 0:
        print("DP_COMM_BENCH " + json.dumps(out), flush=True)
    dist.barrier()
    comm.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
