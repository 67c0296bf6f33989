"""LocalTrajectoryBuilder3D for many trajectories: T builders stepped one after another through dl_ltb_add_range_data versus the
same T builders' twins stepped by one dl_ltb_add_range_data_batch call, alternated step by step in the same run. Trajectories
start at different times of the synthetic drive (tools/synth.py, tools/imu_synth.py: 200 Hz IMU, 10 Hz scans, 16 and 64
beams); num_range_data is small so that submap hand-overs happen inside the timed window. After every step the two arms'
matching results, states, clouds and histograms must be byte-identical, otherwise the script exits with status 1.

Prints one JSON line: per (beams, T) the scans/s of both arms, the median and spread (min, max) of the step time (wall clock
around work that ends in a device synchronise), kernel launches per step, and the GPU's name and power limit.

--rtcsm turns on the online correlative pre-match (use_online_correlative_scan_matching) with D-LIOM's window
(basic_config_3d.lua: 0.1 m, 3 degrees, translation / rotation delta cost weights 0.1 / 0.3). Two more arms then step twins
of the same builders with the pre-match off, alternated with the others, and each shape reports the pre-match's share of the
step, 1 - (step time without) / (step time with), for the single calls and for the batch.

    python tools/bench_ltb_batch.py --trajectories 1 8 32 --beams 16 64 --steps 8 --warmup 3 [--rtcsm]
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


DLIOM_RTCSM = (0.1, float(np.deg2rad(3.0)), 0.1, 0.3)   # D-LIOM's basic_config_3d.lua real_time_correlative_scan_matcher


def options(num_range_data, rtcsm=False):
    import dliom
    import orc
    fo = dliom.FrontendOptions.from_oracle(orc.FrontEndOptions.defaults())
    return dliom.LtbOptions.defaults(fo, NOISE, imu_weight=0.7, num_range_data=num_range_data, max_time_seconds=0.05,
                                     use_rtcsm=int(rtcsm), rtcsm=DLIOM_RTCSM)


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


def run_shape(scene, T, beams, steps, warmup, num_range_data, rtcsm=False):
    import dliom
    import imu_synth
    data = make_steps(scene, T, beams, warmup + steps)
    # arm -> (batched, pre-match on); the "_off" arms exist only to measure the pre-match's share of the step
    arms = {"single": (False, rtcsm), "batch": (True, rtcsm)}
    if rtcsm:
        arms.update({"single_off": (False, False), "batch_off": (True, False)})
    ctxs = {arm: dliom.Context(0) for arm in arms}
    builders = {arm: [dliom.LocalTrajectoryBuilder(ctxs[arm], options(num_range_data, on)) for _ in range(T)]
                for arm, (_, on) in arms.items()}
    for j in range(T):
        s0 = imu_synth.state(data[0][j][0] - 0.1)
        for arm in arms:
            builders[arm][j].set_initial_state(s0)
    times = {arm: [] for arm in arms}
    launches = {arm: [] for arm in arms}
    names = list(arms)
    for k, row in enumerate(data):
        for j, (_, imu, _) in enumerate(row):
            for arm in arms:
                for t, a, g in imu:
                    builders[arm][j].add_imu_data(t, a, g)
        order = names[k % len(names):] + names[:k % len(names)]   # every arm takes every position in turn
        res = {}
        for arm in order:
            ctx, bs = ctxs[arm], builders[arm]
            n0 = ctx.launches
            t0 = time.perf_counter()
            if not arms[arm][0]:   # every dl_ltb_add_range_data ends in a device synchronise
                res[arm] = [bs[j].add_range_data(t1, xyzt) for j, (t1, _, xyzt) in enumerate(row)]
            else:
                res[arm] = dliom.add_range_data_batch(bs, [r[0] for r in row], [r[2] for r in row])
            dt = time.perf_counter() - t0
            if k >= warmup:
                times[arm].append(dt)
                launches[arm].append(ctx.launches - n0)
        for pair in (("single", "batch"), ("single_off", "batch_off")):
            if pair[0] not in arms:
                continue
            for j in range(T):
                a, b = (builders[arm][j] for arm in pair)
                if not same(a, b, res[pair[0]][j], res[pair[1]][j]):
                    print(json.dumps({"error": f"beams {beams} T {T} step {k} trajectory {j}: the batch differs from the single calls"}))
                    sys.exit(1)
    submaps = sum(b.num_submaps() for b in builders["batch"])
    for bs in builders.values():
        for b in bs:
            b.close()
    out = {"beams": beams, "trajectories": T, "steps": steps, "submaps_at_end": submaps}
    for arm in arms:
        t = np.array(times[arm])
        out[arm] = {"scans_per_s": T * len(t) / t.sum(), "step_ms_median": 1e3 * float(np.median(t)),
                    "step_ms_min": 1e3 * float(t.min()), "step_ms_max": 1e3 * float(t.max()),
                    "launches_per_step": float(np.median(launches[arm]))}
    out["speedup"] = out["batch"]["scans_per_s"] / out["single"]["scans_per_s"]
    if rtcsm:
        out["prematch_share_of_step"] = {arm: 1.0 - out[arm + "_off"]["step_ms_median"] / out[arm]["step_ms_median"]
                                         for arm in ("single", "batch")}
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--trajectories", type=int, nargs="+", default=[1, 8, 32])
    ap.add_argument("--beams", type=int, nargs="+", default=[16, 64])
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--num-range-data", type=int, default=4)
    ap.add_argument("--rtcsm", action="store_true", help="with the online correlative pre-match (D-LIOM's window)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this benchmark measures the GPU and has no CPU fall-back")
    import synth
    scene = synth.Scene(42)
    name, power = gpu_info()
    shapes = [run_shape(scene, T, beams, args.steps, args.warmup, args.num_range_data, args.rtcsm)
              for beams in args.beams for T in args.trajectories]
    print(json.dumps({"metric": "LocalTrajectoryBuilder3D scans/s: T single calls vs one batch call per step", "gpu": name,
                      "power_limit": power, "num_range_data": args.num_range_data,
                      "prematch": {"linear_search_window": DLIOM_RTCSM[0], "angular_search_window": DLIOM_RTCSM[1],
                                   "translation_delta_cost_weight": DLIOM_RTCSM[2], "rotation_delta_cost_weight": DLIOM_RTCSM[3]}
                      if args.rtcsm else None, "identical": True, "shapes": shapes}))


if __name__ == "__main__":
    main()
