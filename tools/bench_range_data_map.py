"""The range-data map (dl_range_data_map, dl_range_data_map_dev) on synthetic graphs; prints one JSON line.

Workload: --nodes nodes (default 200 and 2 000) added with add_node into one shared pair of small grids, no matches (so no search
and no solve), each at a random local pose, with --returns returns (default 30 000, a 16-beam scan after the front end's
filters is of that order) attached by set_node_range_data. The map is then taken --runs times per variant, alternating the
host variant (numpy output) and the _dev variant (torch CUDA tensor).

Reported per size: the kernel time (CUDA events around the one pg3d_range_data_map launch, recorded by the library's stage
bracket in runs of their own with profiling on), the whole-call time of both variants (host clock up to the call's return,
which waits for the device; the Python sizing query is included), the achieved bytes/s of the kernel against the 3.35 TB/s HBM3 data-sheet
bound, with bytes counted from shapes (12 B read + 12 B written per point, plus the node table), the attach cost per node
(host clock around set_node_range_data, which ends in a device synchronise), the node store's HBM, and the numpy float32
reference's time on the same map (context only: it is a CPU restatement, not a competitor). Medians of --runs. The card's name
and power limit are read in the same call.

    python tools/bench_range_data_map.py [--nodes 200 2000] [--returns 30000] [--runs 7]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "d-liom_b200"), os.path.join(ROOT, "tools"),
          os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet, HBM3
TABLE_BYTES = 80            # one node of the kernel's table (RangeDataMapNode)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001  (reported, not hidden)
        return {"error": str(e)}


def make_graph(ctx, num_nodes, num_returns, rng):
    import dliom
    g = dliom.PoseGraph3D(ctx, dliom.PoseGraph3DOptions.defaults(optimize_every_n_nodes=0))
    hg, lg = dliom.Grid(ctx, 0.1), dliom.Grid(ctx, 0.45)
    for grid in (hg, lg):
        grid.set_cells([0], [0], [0], [1])
    cloud = rng.uniform(-1, 1, (200, 3)).astype(np.float32)
    identity = np.array([0, 0, 0, 1, 0, 0, 0], np.float64)
    returns = rng.uniform(-80, 80, (num_returns, 3)).astype(np.float32)
    locals_, attach_ms = [], []
    for j in range(num_nodes):
        q = rng.normal(size=4)
        local = np.concatenate([rng.uniform(-500, 500, 3), q / np.linalg.norm(q)])
        g.add_node(0, float(j), local, cloud, cloud, [(0, False, hg, lg, identity)])
        t0 = time.perf_counter()
        g.set_node_range_data(0, j, returns)
        attach_ms.append(1e3 * (time.perf_counter() - t0))
        locals_.append(local)
    return g, (hg, lg), returns, locals_, attach_ms


def measure(ctx, num_nodes, num_returns, runs, rng):
    import range_data_map_reference as ref
    g, grids, returns, locals_, attach_ms = make_graph(ctx, num_nodes, num_returns, rng)
    total = num_nodes * num_returns
    g.range_data_map()                       # warm-up of both variants (module load, scratch growth)
    g.range_data_map(device=True)
    host_ms, dev_ms, kernel_ms = [], [], []
    for _ in range(runs):                    # whole calls, profiling off
        t0 = time.perf_counter()
        pts, _ = g.range_data_map()
        host_ms.append(1e3 * (time.perf_counter() - t0))
        t0 = time.perf_counter()
        dev, _ = g.range_data_map(device=True)
        dev_ms.append(1e3 * (time.perf_counter() - t0))
        del dev
    ctx.set_profiling(True)                  # kernel alone: CUDA events around the one launch (the library's stage bracket)
    ctx.read_profile()
    for _ in range(runs):
        dev, _ = g.range_data_map(device=True)
        ms, calls = ctx.read_profile()["pg3d_range_data_map"]
        assert calls == 1
        kernel_ms.append(ms)
        del dev
    ctx.set_profiling(False)
    same = g.range_data_map(device=True)[0].cpu().numpy().tobytes() == pts.tobytes()
    poses = g.node_poses(0)
    t0 = time.perf_counter()
    want, _ = ref.range_data_map([(0, j, locals_[j], poses[j], returns) for j in range(num_nodes)])
    ref_ms = 1e3 * (time.perf_counter() - t0)
    live, used, cap = g.store_usage()
    bytes_moved = 24 * total + TABLE_BYTES * num_nodes
    k = float(np.median(kernel_ms))
    out = {
        "nodes": num_nodes, "returns_per_node": num_returns, "points": total,
        "kernel_ms": k, "host_call_ms": float(np.median(host_ms)), "dev_call_ms": float(np.median(dev_ms)),
        "kernel_bytes": bytes_moved, "kernel_bytes_per_s": bytes_moved / (k * 1e-3),
        "kernel_share_of_hbm_bound": bytes_moved / (k * 1e-3) / HBM_BYTES_PER_S,
        "attach_ms_per_node": float(np.median(attach_ms)), "attach_bytes_per_node": 12 * num_returns,
        "store_live_bytes": live, "store_used_bytes": used, "store_capacity_bytes": cap,
        "reference_numpy_ms": ref_ms, "host_equals_dev": bool(same), "host_equals_reference": want.tobytes() == pts.tobytes(),
        "runs": runs,
    }
    g.close()
    del grids
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, nargs="+", default=[200, 2000])
    ap.add_argument("--returns", type=int, default=30000)
    ap.add_argument("--runs", type=int, default=7)
    args = ap.parse_args()
    import dliom
    ctx = dliom.Context(0)
    rng = np.random.default_rng(5)
    results = [measure(ctx, n, args.returns, args.runs, rng) for n in args.nodes]
    print(json.dumps({"bench": "range_data_map", "card": card(), "sizes": results}))


if __name__ == "__main__":
    main()
