"""Mapping against pure localization on the same long drive, through dliom.PoseGraph3D; prints one JSON line.

Both arms first map trajectory 0 of the synthetic street (tools/synth.py, 120 scans) through a LocalTrajectoryBuilder (dl_ltb)
and freeze it. Then the street is driven again --passes times, each pass a new trajectory (1, 2, ...) with its own builder and
its local frame offset by a planar transform, fed live into the graph (add_node_from_builder); its finished submaps are matched
to the map's submap of the same index, the match derived from the synthetic truth, as the host SURF stage would. The mapping arm
keeps everything. The localization arm gives every pass add_pure_localization_trimmer(t, 3) and set_initial_trajectory_pose, and
ends it with finish_trajectory, so the pass's submaps and nodes are trimmed and their clouds die in the node store; over enough
passes the dead clouds pass 4 MiB and pg3d_store_compact runs.

Reported per arm: the median add_node time (host wall clock around the call, which ends in a device synchronise), builder-grid
plus node-store bytes over time. For the localization arm also the cost of trimming: the trims happen inside the optimization
that add_node times, so a twin graph without trimmers receives the same nodes, runs the same optimizations, and then trims by
hand what the arm's trimmer reported (dl_pg3d_trim_submap, host clock around the C call, which ends in a device synchronise when
it compacts); the trims that compacted the store are listed with the bytes they moved. The card's name and power limit are read
in the same call.

    python tools/bench_localization.py [--scans 120] [--passes 10] [--optimize-every 5] [--num-range-data 3]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "d-liom_b200"), os.path.join(ROOT, "tools"),
          os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

NOISE = [3.99e-2, 1.56e-2, 6.4e-5, 3.6e-5]
OFFSET = np.concatenate([[4.0, -3.0, 0.0], [np.cos(np.deg2rad(2.5)), 0.0, 0.0, np.sin(np.deg2rad(2.5))]])  # world <- trajectory 1


def make_builder(ctx, offset, first_time, num_range_data):
    import dliom
    import imu_synth
    import orc
    import pose_graph3d_oracle as pg
    fo = dliom.FrontendOptions.from_oracle(orc.FrontEndOptions.defaults())
    b = dliom.LocalTrajectoryBuilder(ctx, dliom.LtbOptions.defaults(fo, NOISE, imu_weight=0.7, num_range_data=num_range_data,
                                                                     max_time_seconds=0.05))
    s = imu_synth.state(first_time - 0.1)
    inv = pg.inverse(offset)
    b.set_initial_state(np.concatenate([pg.compose(inv, s[:7]), pg.rotate(inv[3:], s[7:10]), s[10:]]))
    return b


def scans_of(num_scans):
    """[(time, [(imu time, acc, gyr)], RangeMeasurement rows)] of the drive: one 16-beam scan every 0.1 s from t = 2 s."""
    import imu_synth
    import synth
    scene = synth.Scene(42)
    out = []
    for k in range(num_scans):
        t1 = 2.0 + 0.1 * k
        dt, acc, gyr = imu_synth.samples(t1 - 0.1, t1)
        ts = t1 - 0.1 + np.arange(len(dt)) / 200.0
        out.append((t1, [(ts[j], acc[j], gyr[j]) for j in range(0 if k == 0 else 1, len(dt))], synth.make_scan(scene, 16, t1)))
    return out


def feed(graph, trajectory_id, builder, scans, matches_for=None, after_node=None):
    """Scans into the builder, every inserted node into the graph (add_node_from_builder). matches_for(index, local pose)
    gives the matches of a finished submap; after_node(result, info, add_node ms) sees every node."""
    for t1, imu, rows in scans:
        for ts, acc, gyr in imu:
            builder.add_imu_data(ts, acc, gyr)
        r = builder.add_synchronized_range_data(t1, rows, np.zeros((1, 3), np.float32))
        if not (r.has_result and r.inserted):
            continue
        matches = []
        if matches_for is not None:
            idx = r.insertion_submap_index[0]
            _, _, pose, _, fin = builder.submap(idx)
            if fin:
                matches = matches_for(idx, pose)
        t0 = time.perf_counter()
        info = graph.add_node_from_builder(trajectory_id, builder, r, matches)
        ms = 1e3 * (time.perf_counter() - t0)
        if after_node is not None:
            after_node(r, info, ms)


def map_graph(ctx, options, scans, num_range_data):
    """Trajectory 0 mapped into a fresh graph, finally optimized and frozen -> (graph, its builder, {finished submap index: local
    pose})."""
    import dliom
    g = dliom.PoseGraph3D(ctx, options)
    b0 = make_builder(ctx, np.array([0.0, 0, 0, 1, 0, 0, 0]), scans[0][0], num_range_data)
    feed(g, 0, b0, scans)
    g.run_final_optimization()
    g.freeze_trajectory(0)
    return g, b0, {i: b0.submap(i)[2] for i in range(b0.num_submaps()) if b0.submap(i)[4]}


def truth_matches(local0, offset):
    """matches_for of feed(): the map's finished submap of the same index, from the synthetic truth."""
    import pose_graph3d_oracle as pg

    def matches_for(idx, pose):
        if idx not in local0:
            return []
        x, y, th = pg.match_from_truth(pose, local0[idx], offset, pg.IDENTITY)
        return [(0, idx, x, y, th)]
    return matches_for


def builder_grid_bytes(builder):
    """Voxel bytes of the grids the builder still holds: dl_grid_num_bricks bricks of 1 KiB each (the index levels are small)."""
    total = 0
    for i in range(builder.num_submaps()):
        for g in builder.submap(i)[:2]:
            if g.h:
                total += 1024 * g.num_bricks
    return total


def run_arm(ctx, options, scans, num_range_data, passes, localize):
    import dliom
    import pose_graph3d_oracle as pg
    g, b0, local0 = map_graph(ctx, options, scans, num_range_data)
    twin, twin_b0 = None, None
    if localize:
        twin, twin_b0, _ = map_graph(ctx, dliom.PoseGraph3DOptions(0, options.every_nodes_to_find_constraint,
                                                              options.matcher_translation_weight, options.matcher_rotation_weight,
                                                              options.constraint_builder, options.optimization_problem),
                               scans, num_range_data)
    times, trims, compactions, series, builders = [], [], [], [], []

    def timed_twin_trims(trimmed):
        for t, i in trimmed:
            _, used_before, _ = twin.store_usage()
            t0 = time.perf_counter()
            st = ctx.L.dl_pg3d_trim_submap(twin.h, t, i)
            ms = 1e3 * (time.perf_counter() - t0)
            ctx.check(st)
            live, used, _ = twin.store_usage()
            if used < used_before:      # the store was compacted: `live` bytes were copied
                compactions.append(dict(ms=ms, moved_bytes=live, freed_bytes=used_before - used))
            else:
                trims.append(ms)

    for k in range(1, passes + 1):
        b = make_builder(ctx, OFFSET, scans[0][0], num_range_data)
        builders.append(b)
        if localize:
            rel = pg.compose(pg.inverse(g.node_poses(0)[0]), OFFSET)   # before the map's first node: relative to its pose
            for graph in (g, twin):
                graph.set_initial_trajectory_pose(k, 0, rel, -1.0)
            g.add_pure_localization_trimmer(k, 3)

        def after_node(r, info, ms, b=b, k=k):
            times.append(ms)
            if localize:
                subs = [(r.insertion_submap_index[i],) + tuple(b.submap(r.insertion_submap_index[i])[j] for j in (4, 0, 1, 2))
                        for i in range(r.num_insertion_submaps)]
                twin.add_node(k, r.time, np.array(r.local_pose[:]), b.cloud(2), b.cloud(3), subs, pending_matches[0])
                if info.optimized:
                    twin.run_final_optimization()
                    timed_twin_trims(g.last_trimmed())
            live, used, cap = g.store_usage()
            series.append(dict(node=len(times), builder_grid_bytes=sum(builder_grid_bytes(x) for x in builders),
                               store_used_bytes=used, store_live_bytes=live, store_capacity_bytes=cap))

        matches_for = truth_matches(local0, OFFSET)
        pending_matches = [[]]

        def recording_matches(idx, pose):
            pending_matches[0] = matches_for(idx, pose)
            return pending_matches[0]

        def reset_then(r, info, ms, f=after_node):
            f(r, info, ms)
            pending_matches[0] = []
        feed(g, k, b, scans, recording_matches, reset_then)
        if localize:
            g.finish_trajectory(k)
            twin.finish_trajectory(k)
            timed_twin_trims(g.last_trimmed())
            live, used, cap = g.store_usage()
            series.append(dict(node=len(times), builder_grid_bytes=sum(builder_grid_bytes(x) for x in builders),
                               store_used_bytes=used, store_live_bytes=live, store_capacity_bytes=cap, finished=k))
    out = dict(median_add_node_ms=float(np.median(times)), nodes=len(times), final=series[-1],
               peak_builder_grid_bytes=max(s["builder_grid_bytes"] for s in series),
               peak_store_used_bytes=max(s["store_used_bytes"] for s in series),
               series=series[::max(1, len(series) // 16)])
    if localize:
        out.update(trims_without_compaction=len(trims), median_trim_ms=float(np.median(trims)) if trims else None,
                   compactions=compactions)
        twin.close()
        twin_b0.close()
    g.close()
    for b in builders:
        b.close()
    b0.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=120)
    ap.add_argument("--passes", type=int, default=10)
    ap.add_argument("--optimize-every", type=int, default=5)
    ap.add_argument("--num-range-data", type=int, default=3)
    args = ap.parse_args()
    import dliom
    from bench_global_slam import gpu_name_and_power
    name, power = gpu_name_and_power()
    ctx = dliom.Context(0)
    options = dliom.PoseGraph3DOptions.defaults(optimize_every_n_nodes=args.optimize_every, every_nodes_to_find_constraint=2,
                                                min_score=0.3, min_low_resolution_score=0.3)
    scans = scans_of(args.scans)
    result = dict(gpu=name, power_limit=power, scans=args.scans, passes=args.passes, optimize_every_n_nodes=args.optimize_every,
                  num_range_data=args.num_range_data,
                  mapping=run_arm(ctx, options, scans, args.num_range_data, args.passes, False),
                  localization=run_arm(ctx, options, scans, args.num_range_data, args.passes, True))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
