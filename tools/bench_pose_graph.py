#!/usr/bin/env python
"""Global step of BASELINE configs[4] on N GPUs: the block-sparse pose adjustment (dl_pose_graph_solve_sparse) with the
constraints sharded by submap owner and the normal-equation blocks reduced with ncclAllReduce(fp64) issued from the C-ABI. Launch
with torchrun like bench.py:
  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 tools/bench_pose_graph.py
Prints one JSON line on rank 0: solve time, all-reduce count / bytes / device time, achieved bus bandwidth, and whether every rank
ended with bit-identical poses. --shape trajectory builds a drive (each node seen by its two active submaps, every --loop-every-th
node also by an older submap) instead of random constraints."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "d-liom_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def _power_limit_w(device):
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(device), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        return float(out)
    except (OSError, ValueError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--submaps", type=int, default=8)
    ap.add_argument("--nodes", type=int, default=400)
    ap.add_argument("--per-node", type=int, default=3, help="constraints per node (to random submaps)")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--shape", choices=("random", "trajectory"), default="random")
    ap.add_argument("--loop-every", type=int, default=1, help="trajectory shape: one loop closure every this many nodes")
    args = ap.parse_args()
    import torch
    import dliom
    from test_posegraph_oracle import aa_to_q, compose, inverse
    rank, local, world = int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    torch.cuda.set_device(local)
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    ctx = dliom.Context(local)
    idt = torch.zeros(128, dtype=torch.uint8, device=f"cuda:{local}")
    if rank == 0:
        idt.copy_(torch.tensor(list(dliom.comm_unique_id()), dtype=torch.uint8))
    if dist is not None:
        dist.broadcast(idt, 0)
    comm = dliom.Comm(ctx, bytes(idt.cpu().numpy().tolist()), rank, world)
    # the same graph on every rank (same seed); each rank keeps the constraints of the submaps it owns
    S, N = args.submaps, args.nodes
    if args.shape == "trajectory":
        from test_posegraph_schur_oracle import trajectory_graph
        start_submaps, start_nodes, cons = trajectory_graph(S, N, loops_every=args.loop_every)
        truth = None
    else:
        rng = np.random.default_rng(7)
        submaps = [np.array([0, 0, 0, 1.0, 0, 0, 0])] + [np.array([*rng.uniform(-30, 30, 2), rng.uniform(-1, 1), *aa_to_q([0, 0, rng.uniform(-3, 3)])])
                                                          for _ in range(S - 1)]
        truth = [np.array([*rng.uniform(-40, 40, 2), rng.uniform(-2, 2), *aa_to_q(rng.uniform(-0.5, 0.5, 3))]) for _ in range(N)]
        cons = []
        for n in range(N):
            for s in rng.choice(S, size=min(args.per_node, S), replace=False):
                noise = np.array([*rng.normal(0, 0.03, 3), *aa_to_q(rng.normal(0, 0.01, 3))])
                cons.append((int(s), n, compose(compose(inverse(submaps[s]), truth[n]), noise), 1.1e4 ** 0.5, 1e5 ** 0.5))
        start_nodes = [compose(t, np.array([*rng.uniform(-0.5, 0.5, 3), *aa_to_q(rng.uniform(-0.1, 0.1, 3))])) for t in truth]
        start_submaps = [submaps[0]] + [compose(s, np.array([*rng.uniform(-0.3, 0.3, 3), *aa_to_q(rng.uniform(-0.05, 0.05, 3))])) for s in submaps[1:]]
    mine = [c for c in cons if c[0] % world == rank]
    times = []
    for _ in range(args.repeats):
        torch.cuda.synchronize()
        if dist is not None:
            dist.barrier()
        t0 = time.perf_counter()
        s_out, n_out, summary, info = ctx.pose_graph_solve_sparse(start_submaps, start_nodes, mine, comm=comm)
        times.append(time.perf_counter() - t0)
    digest = torch.tensor([float(np.sum(np.abs(n_out))), float(np.sum(np.abs(s_out)))], dtype=torch.float64, device=f"cuda:{local}")
    lo, hi = digest.clone(), digest.clone()
    tmax = torch.tensor([min(times)], dtype=torch.float64, device=f"cuda:{local}")
    if dist is not None:
        dist.all_reduce(lo, op=dist.ReduceOp.MIN)
        dist.all_reduce(hi, op=dist.ReduceOp.MAX)
        dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
    if rank == 0:
        props = torch.cuda.get_device_properties(local)
        err = (max(np.linalg.norm(compose(inverse(t), compose(inverse(s_out[0]), p))[:3]) for t, p in zip(truth, n_out))
               if truth is not None else None)
        ar_ms = info.all_reduce_min_ms if info.all_reduce_min_ms > 0 else info.all_reduce_ms / max(info.all_reduce_count, 1)
        print(json.dumps({"what": "dl_pose_graph_solve_sparse: SPA, Schur complement of the node blocks, ncclAllReduce(fp64) of the blocks",
                          "ranks": world, "shape": args.shape,
                          "submaps": S, "nodes": N, "constraints": len(cons), "constraints_this_rank": len(mine),
                          "local_parameters": info.num_local_parameters, "iterations": summary["num_iterations"],
                          "evaluations": summary["num_evaluations"], "initial_cost": summary["initial_cost"],
                          "final_cost": summary["final_cost"], "solve_s": float(tmax[0]),
                          "all_reduce": {"count": info.all_reduce_count, "bytes_each": int(info.all_reduce_bytes), "ms_each": ar_ms,
                                         "ms_mean": info.all_reduce_ms / max(info.all_reduce_count, 1),
                                         "algbw_gbs": info.all_reduce_bytes / (ar_ms * 1e-3) / 1e9 if ar_ms > 0 else None,
                                         "busbw_gbs": (info.all_reduce_bytes / (ar_ms * 1e-3) / 1e9 * 2 * (world - 1) / world)
                                         if ar_ms > 0 and world > 1 else None},
                          "replicas_bit_identical": bool(torch.equal(lo, hi)), "max_node_error_m": err,
                          "gpu": {"name": props.name, "power_limit_w": _power_limit_w(local)},
                          "reduced_parameters": info.num_reduced_parameters, "pairs": info.num_pairs,
                          "setup_exchange_bytes": int(info.setup_exchange_bytes)}))
    comm.close()
    if dist is not None:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
