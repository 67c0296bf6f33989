"""Map writer benchmark: synthetic 64-beam scans along the street trajectory (tools/synth.py) written into a map with
min_max_range_filter and voxel_filter_and_remove_moving_objects at 5 cm, all messages in one call per pass. Prints one JSON
line: milliseconds per pass (device work + copies, each call ends in a device synchronise), points/s, pass-2 samples/s, a CPU
oracle arm on a subset of the scans, and the GPU's name and power limit. The oracle arm is the numpy test oracle
(tests/map_writer_oracle.py): it checks the output bit for bit; its time is that of a correctness reference, not of a CPU
implementation.

With --xray the same invocation also times the final pass with the six X-ray stages of the reference's backpack pipeline
(assets_writer_backpack_3d.lua: gray YZ / XY / XZ at 5 cm, color_points for two LiDAR frames, the three again in colour; messages
alternate between the two frame ids) against the final pass without them, alternating the two, and reports the X-ray share of
the final pass, point-stages per second, the device bytes the stages hold (cudaMemGetInfo difference) and the image sizes.

With --ros-map it times the final pass with one write_ros_map grid stage (assets_writer_ros_map.lua: 0.05 m, hit 0.55, miss
0.49, insert_free_space) against the final pass without it, alternating the two, and reports the stage's milliseconds, walk cells
per second, the grid's size and the device bytes the stage holds. Walk cells are counted from the shapes in an untimed run with
one message per call: per walk |dx| + |dy| + 1 pixels of CastRay's ends at the grid's final limits (a walk through an exact pixel
corner visits one cell fewer, which this count ignores).

    python tools/bench_map_writer.py --scans 300 --voxel 0.05 --repeat 3
    python tools/bench_map_writer.py --scans 300 --voxel 0.05 --repeat 3 --xray
    python tools/bench_map_writer.py --scans 300 --voxel 0.05 --repeat 3 --ros-map
"""
import math
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "d-liom_b200"), os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        name, power = [s.strip() for s in out[0].split(",")]
        return name, power
    except Exception as e:   # reported, not hidden: the line says what could not be read
        return f"unknown ({e})", "unknown"


def make_run(num_scans, beams, period=0.1):
    import synth
    scene = synth.Scene()
    node_t = np.arange(0.0, period * (num_scans + 1) + 1e-9, 0.02)
    times = np.round(node_t * 1e7).astype(np.int64)
    poses = np.array([synth.pose7(t) for t in node_t])
    rows, msgs, first = [], [], 0
    for k in range(num_scans):
        end = period * (k + 1)
        r = synth.make_scan(scene, beams, end)
        rows.append(np.stack([r["x"], r["y"], r["z"], r["t"]], 1).astype(np.float32))
        msgs.append((int(round(end * 1e7)), first, len(r), 0, (0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0)))
        first += len(r)
    return times, poses, msgs, np.concatenate(rows)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=300)
    ap.add_argument("--beams", type=int, default=64)
    ap.add_argument("--voxel", type=float, default=0.05)
    ap.add_argument("--min-range", type=float, default=1.0)
    ap.add_argument("--max-range", type=float, default=60.0)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--cpu-scans", type=int, default=2)
    ap.add_argument("--xray", action="store_true", help="also time the final pass with the backpack pipeline's X-ray stages")
    ap.add_argument("--ros-map", action="store_true", help="also time the final pass with one 0.05 m write_ros_map grid stage")
    args = ap.parse_args()

    import torch
    import dliom
    import map_writer_oracle as mo

    if not torch.cuda.is_available():
        raise SystemExit("bench_map_writer: no CUDA device")
    times, poses, msgs, rows = make_run(args.scans, args.beams)
    ctx = dliom.Context(0)
    rows_dev = torch.from_numpy(rows).cuda()
    out_dev = torch.empty((len(rows), 3), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()

    def run():
        w = dliom.MapWriter(ctx, range_filter=(args.min_range, args.max_range), outlier_voxel_size=args.voxel)
        w.add_trajectory(0, times, poses)
        ms, infos = [], []
        while True:
            t0 = time.perf_counter()
            n, _, info = w.process_dev(msgs, rows_dev.data_ptr(), len(rows), out_dev.data_ptr())
            ms.append((time.perf_counter() - t0) * 1e3)
            infos.append(info)
            if not w.flush():
                break
        cells = len(w.voxels()[0])
        w.close()
        return ms, infos, n, cells

    run()   # warm-up: module load, allocations of the scratch and the table
    runs = [run() for _ in range(args.repeat)]
    best = min(runs, key=lambda r: sum(r[0]))
    ms, infos, n_out, cells = best
    assert all(r[2] == n_out for r in runs)
    samples = infos[1]["num_samples"]
    # CPU arm: the numpy oracle on the first scans (one thread)
    sub = msgs[:args.cpu_scans]
    sub_rows = rows[:sub[-1][1] + sub[-1][2]]
    t0 = time.perf_counter()
    want = mo.write_map({0: mo.Trajectory(times, poses)}, sub, sub_rows, range_filter=(args.min_range, args.max_range),
                        voxel_size=args.voxel)
    cpu_s = time.perf_counter() - t0
    w = dliom.MapWriter(ctx, range_filter=(args.min_range, args.max_range), outlier_voxel_size=args.voxel)
    w.add_trajectory(0, times, poses)
    got = w.write_map(sub, sub_rows)[0]
    name, power = gpu_info()
    line = {
        "workload": {"scans": args.scans, "beams": args.beams, "rows": int(len(rows)), "voxel_size": args.voxel,
                     "range": [args.min_range, args.max_range]},
        "gpu": name, "power_limit": power,
        "ms_per_pass": [round(m, 3) for m in ms], "ms_total": round(sum(ms), 3),
        "points_per_s": round(len(rows) * len(ms) / (sum(ms) / 1e3)),
        "pass2_samples": int(samples), "pass2_samples_per_s": round(samples / (ms[1] / 1e3)),
        "points_out": int(n_out), "cells": int(cells), "dropped_moving": int(infos[2]["dropped_moving"]),
        "all_runs_ms_total": [round(sum(r[0]), 3) for r in runs],
        "cpu_oracle": {"scans": len(sub), "rows": int(len(sub_rows)), "s": round(cpu_s, 3),
                       "points_per_s": round(len(sub_rows) * 3 / cpu_s), "samples_per_s": round(want["num_samples"] / cpu_s),
                       "bit_identical": bool(got.tobytes() == want["points"].tobytes())},
    }
    if args.xray:
        line["xray"] = bench_xray(ctx, args, times, poses, msgs, rows, rows_dev, out_dev)
    if args.ros_map:
        line["ros_map"] = bench_ros_map(ctx, args, times, poses, msgs, rows, rows_dev, out_dev)
    print(json.dumps(line))


XRAY_VOXEL = 5e-2


def backpack_stages():
    """assets_writer_backpack_3d.lua after its range filter (transform.lua's rotations), frame ids 0 and 1."""
    import dliom
    xy, xz, yz = [(0.0, 0.0, 0.0) + tuple(dliom.roll_pitch_yaw(*a))
                  for a in ((0.0, -math.pi / 2.0, 0.0), (0.0, 0.0, -math.pi / 2), (0.0, 0.0, math.pi))]
    gray = [("xray", yz), ("xray", xy), ("xray", xz)]
    return gray + [("color", 0, (255, 0, 0)), ("color", 1, (0, 255, 0))] + gray


def bench_xray(ctx, args, times, poses, msgs, rows, rows_dev, out_dev):
    import torch
    import dliom
    msgs = [m + (k % 2,) for k, m in enumerate(msgs)]

    def final_pass(with_stages):
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        w = dliom.MapWriter(ctx, range_filter=(args.min_range, args.max_range), outlier_voxel_size=args.voxel)
        w.add_trajectory(0, times, poses)
        ids = []
        if with_stages:
            for s in backpack_stages():
                if s[0] == "xray":
                    ids.append(w.add_xray(XRAY_VOXEL, s[1]))
                else:
                    w.add_color(s[1], s[2])
        while True:
            t0 = time.perf_counter()
            n, _, info = w.process_dev(msgs, rows_dev.data_ptr(), len(rows), out_dev.data_ptr())
            ms = (time.perf_counter() - t0) * 1e3    # the call ends in a device synchronise
            if not w.flush():
                break
        held = free0 - torch.cuda.mem_get_info()[0]
        t0 = time.perf_counter()
        shapes = [list(w.xray_image(i).shape) for i in ids]
        image_ms = (time.perf_counter() - t0) * 1e3
        w.close()
        return ms, n, held, shapes, image_ms

    final_pass(True)    # warm-up: the X-ray table, the sort's scratch
    with_ms, without_ms = [], []
    for _ in range(args.repeat):
        a = final_pass(False)
        b = final_pass(True)
        without_ms.append(a[0])
        with_ms.append(b[0])
    n, held_with, shapes, image_ms = b[1], b[2], b[3], b[4]
    held_without = a[2]
    best_with, best_without = min(with_ms), min(without_ms)
    stages = sum(1 for s in backpack_stages() if s[0] == "xray")
    return {"stages": stages, "voxel_size": XRAY_VOXEL, "points": int(n),
            "final_pass_ms_without": [round(v, 3) for v in without_ms], "final_pass_ms_with": [round(v, 3) for v in with_ms],
            "xray_share_of_final_pass": round((best_with - best_without) / best_with, 4),
            "point_stages_per_s": round(n * stages / ((best_with - best_without) / 1e3)),
            "device_bytes_held_by_stages": int(held_with - held_without), "image_ms_all_stages": round(image_ms, 3),
            "image_sizes_hw": shapes}


ROS_MAP = (0.05, 0.55, 0.49)   # assets_writer_ros_map.lua's write_ros_map


def walk_cells(ctx, args, times, poses, msgs, rows, info):
    """Sum over walks of |dx| + |dy| + 1 pixels between CastRay's superscaled ends, at the grid's final limits; the batches
    come from an untimed writer fed one message per call."""
    import dliom
    import probability_grid_reference as pg
    w = dliom.MapWriter(ctx, range_filter=(args.min_range, args.max_range), outlier_voxel_size=args.voxel)
    w.add_trajectory(0, times, poses)
    while True:
        out = [w.process([m], rows) for m in msgs]
        if not w.flush():
            break
    w.close()
    ss = pg.Limits(info["resolution"], info["max_x"], info["max_y"], info["num_x_cells"], info["num_y_cells"]).superscaled()
    total = 0
    for pts, origin, _ in out:
        if np.isnan(origin[0][0]) or len(pts) == 0:
            continue
        bx, by = ss.cell_index(origin[0][0], origin[0][1])
        ex, ey = ss.cell_indices(pts[:, 0], pts[:, 1])
        total += int((np.abs(ex // 1000 - bx // 1000) + np.abs(ey // 1000 - by // 1000) + 1).sum())
    return total


def bench_ros_map(ctx, args, times, poses, msgs, rows, rows_dev, out_dev):
    import torch
    import dliom

    def final_pass(with_stage):
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        w = dliom.MapWriter(ctx, range_filter=(args.min_range, args.max_range), outlier_voxel_size=args.voxel)
        w.add_trajectory(0, times, poses)
        stage = w.add_probability_grid(*ROS_MAP) if with_stage else None
        while True:
            t0 = time.perf_counter()
            n, _, _ = w.process_dev(msgs, rows_dev.data_ptr(), len(rows), out_dev.data_ptr())
            ms = (time.perf_counter() - t0) * 1e3    # the call ends in a device synchronise
            if not w.flush():
                break
        held = free0 - torch.cuda.mem_get_info()[0]
        info = None
        if with_stage:
            t0 = time.perf_counter()
            info, _, _ = w.probability_grid(stage)
            read_ms = (time.perf_counter() - t0) * 1e3
        w.close()
        return ms, n, held, info, (read_ms if with_stage else None)

    final_pass(True)    # warm-up
    with_ms, without_ms = [], []
    for _ in range(args.repeat):
        a = final_pass(False)
        b = final_pass(True)
        without_ms.append(a[0])
        with_ms.append(b[0])
    n, held_with, info, read_ms = b[1], b[2], b[3], b[4]
    stage_ms = min(with_ms) - min(without_ms)
    cells = walk_cells(ctx, args, times, poses, msgs, rows, info)
    return {"resolution": ROS_MAP[0], "hit": ROS_MAP[1], "miss": ROS_MAP[2], "points": int(n),
            "final_pass_ms_without": [round(v, 3) for v in without_ms], "final_pass_ms_with": [round(v, 3) for v in with_ms],
            "stage_ms": round(stage_ms, 3), "walk_cells": cells, "walk_cells_per_s": round(cells / (stage_ms / 1e3)),
            "grid_cells_xy": [info["num_x_cells"], info["num_y_cells"]], "cropped_wh": [info["width"], info["height"]],
            "device_bytes_held_by_stage": int(held_with - a[2]), "read_back_ms": round(read_ms, 3)}


if __name__ == "__main__":
    main()
