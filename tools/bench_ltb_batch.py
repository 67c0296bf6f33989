"""LocalTrajectoryBuilder3D for many trajectories: T builders stepped one after another through dl_ltb_add_range_data versus the
same T builders' twins stepped by one dl_ltb_add_range_data_batch call, alternated step by step in the same run. Trajectories
start at different times of the synthetic drive (tools/synth.py, tools/imu_synth.py: 200 Hz IMU, 10 Hz scans, 16 and 64
beams); num_range_data is small so that submap hand-overs happen inside the timed window. After every step the two arms'
matching results, states, clouds and histograms must be byte-identical, otherwise the script exits with status 1.

Prints one JSON line: per (beams, T) the scans/s of both arms, the median and spread (min, max) of the step time (wall clock
around work that ends in a device synchronise), kernel launches per step, and the GPU's name and power limit.

    python tools/bench_ltb_batch.py --trajectories 1 8 32 --beams 16 64 --steps 8 --warmup 3
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "d-liom_b200"), os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_map_writer import gpu_info  # noqa: E402

NOISE = [3.99e-2, 1.56e-2, 6.4e-5, 3.6e-5]


def options(num_range_data):
    import dliom
    import orc
    fo = dliom.FrontendOptions.from_oracle(orc.FrontEndOptions.defaults())
    return dliom.LtbOptions.defaults(fo, NOISE, imu_weight=0.7, num_range_data=num_range_data, max_time_seconds=0.05)


def make_steps(scene, T, beams, count):
    """[step][trajectory] -> (time, imu samples, x y z t rows); trajectory j starts 0.7 s after trajectory j - 1."""
    import imu_synth
    import synth
    out = []
    for k in range(count):
        row = []
        for j in range(T):
            t1 = 2.0 + 0.7 * j + 0.1 * k
            dt, acc, gyr = imu_synth.samples(t1 - 0.1, t1)
            imu = [(t1 - 0.1 + i / 200.0, acc[i], gyr[i]) for i in range(0 if k == 0 else 1, len(dt))]
            r = synth.make_scan(scene, beams, t1)
            row.append((t1, imu, np.ascontiguousarray(np.stack([r["x"], r["y"], r["z"], r["t"]], 1), np.float32)))
        out.append(row)
    return out


def same(a, b, ra, rb):
    if bytes(ra) != bytes(rb):
        return False
    if not np.array_equal(a.state()[0].view(np.uint64), b.state()[0].view(np.uint64)):
        return False
    if not np.array_equal(a.histogram().view(np.uint32), b.histogram().view(np.uint32)):
        return False
    return all(np.array_equal(a.cloud(w).view(np.uint32), b.cloud(w).view(np.uint32)) for w in range(4))


def run_shape(scene, T, beams, steps, warmup, num_range_data):
    import dliom
    import imu_synth
    data = make_steps(scene, T, beams, warmup + steps)
    ctx_single, ctx_batch = dliom.Context(0), dliom.Context(0)
    single = [dliom.LocalTrajectoryBuilder(ctx_single, options(num_range_data)) for _ in range(T)]
    batch = [dliom.LocalTrajectoryBuilder(ctx_batch, options(num_range_data)) for _ in range(T)]
    for j in range(T):
        s0 = imu_synth.state(data[0][j][0] - 0.1)
        single[j].set_initial_state(s0)
        batch[j].set_initial_state(s0)
    times = {"single": [], "batch": []}
    launches = {"single": [], "batch": []}
    for k, row in enumerate(data):
        for j, (_, imu, _) in enumerate(row):
            for b in (single[j], batch[j]):
                for t, a, g in imu:
                    b.add_imu_data(t, a, g)
        order = ("single", "batch") if k % 2 == 0 else ("batch", "single")
        res = {}
        for arm in order:
            ctx = ctx_single if arm == "single" else ctx_batch
            n0 = ctx.launches
            t0 = time.perf_counter()
            if arm == "single":   # every dl_ltb_add_range_data ends in a device synchronise
                res[arm] = [single[j].add_range_data(t1, xyzt) for j, (t1, _, xyzt) in enumerate(row)]
            else:
                res[arm] = dliom.add_range_data_batch(batch, [r[0] for r in row], [r[2] for r in row])
            dt = time.perf_counter() - t0
            if k >= warmup:
                times[arm].append(dt)
                launches[arm].append(ctx.launches - n0)
        for j in range(T):
            if not same(single[j], batch[j], res["single"][j], res["batch"][j]):
                print(json.dumps({"error": f"beams {beams} T {T} step {k} trajectory {j}: the batch differs from the single calls"}))
                sys.exit(1)
    submaps = sum(b.num_submaps() for b in batch)
    for b in single + batch:
        b.close()
    out = {"beams": beams, "trajectories": T, "steps": steps, "submaps_at_end": submaps}
    for arm in ("single", "batch"):
        t = np.array(times[arm])
        out[arm] = {"scans_per_s": T * len(t) / t.sum(), "step_ms_median": 1e3 * float(np.median(t)),
                    "step_ms_min": 1e3 * float(t.min()), "step_ms_max": 1e3 * float(t.max()),
                    "launches_per_step": float(np.median(launches[arm]))}
    out["speedup"] = out["batch"]["scans_per_s"] / out["single"]["scans_per_s"]
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--trajectories", type=int, nargs="+", default=[1, 8, 32])
    ap.add_argument("--beams", type=int, nargs="+", default=[16, 64])
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--num-range-data", type=int, default=4)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this benchmark measures the GPU and has no CPU fall-back")
    import synth
    scene = synth.Scene(42)
    name, power = gpu_info()
    shapes = [run_shape(scene, T, beams, args.steps, args.warmup, args.num_range_data) for beams in args.beams for T in args.trajectories]
    print(json.dumps({"metric": "LocalTrajectoryBuilder3D scans/s: T single calls vs one batch call per step", "gpu": name,
                      "power_limit": power, "num_range_data": args.num_range_data, "identical": True, "shapes": shapes}))


if __name__ == "__main__":
    main()
