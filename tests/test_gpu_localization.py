"""Pure localization on the device (dl_pg3d_*, dl_ltb_release_submap): the periodic graph with a PureLocalizationTrimmer and an
initial trajectory pose against the trimming oracle (tests/pose_graph3d_trimming_oracle.py) fed the device's searches and
solves; the node store's compaction through the searches; rejections; and the end-to-end localization of a second drive in a
frozen map with its grids released and its store bounded."""
import numpy as np
import pytest

import pose_graph3d_oracle as pg
import pose_graph3d_trimming_oracle as tg
from helpers import pose_error
from test_gpu_pose_graph3d import _ids, options, recorded  # noqa: F401  (the recorded two-trajectory drive)

pytestmark = pytest.mark.gpu


def state(g, trajectories=(0, 1)):
    """Everything a rejected call must leave as it was."""
    return ([g.node_poses(t).tobytes() for t in trajectories], [g.submap_poses(t).tobytes() for t in trajectories],
            [(g.ids(t), g.ids(t, 1)) for t in trajectories], [(c[0], c[1], c[2].tobytes(), c[5]) for c in g.constraints()],
            g.store_usage(), g.store_bytes())


def test_trimmer_and_initial_pose_match_the_oracle(recorded):  # noqa: F811
    """Trajectory 0 then trajectory 1 with a PureLocalizationTrimmer(1, 3) and an initial pose, optimizing every 4 nodes: after
    every add_node the device's ids, trimmed submaps, constraint ids, tags and weights equal the oracle's exactly, and its poses
    and INTRA_SUBMAP measurements to 1e-9 / 1e-12: the oracle's numpy Rigid3 arithmetic (np.cross, np.linalg.norm) does not
    evaluate in the device's operation order, so the last bits differ, and the oracle's solves are the sparse call on the
    oracle's own inputs. The device's solves over holes are pinned bit for bit to dl_pose_graph_solve_sparse on the device's
    exported inputs by the next test; INTER_SUBMAP measurements are the device search's and compared exactly there too."""
    import dliom
    ctx, nodes = recorded
    g = dliom.PoseGraph3D(ctx, options(optimize_every_n_nodes=4))
    o = tg.PoseGraph3D(4, 2)
    rel = np.concatenate([[0.5, -0.25, 0.0], pg.yaw_quaternion(0.05)])
    t_init = nodes[5][1]["time"] + 0.037      # between two of trajectory 0's nodes
    g.set_initial_trajectory_pose(1, 0, rel, t_init)
    o.set_initial_trajectory_pose(1, 0, rel, t_init)
    g.add_pure_localization_trimmer(1, 3)
    o.add_pure_localization_trimmer(1, 3)
    trimmed = []
    for t, i, n in _ids(nodes):
        info = g.add_node(t, n["time"], n["local"], n["hi"], n["lo"], n["ins"], n["matches"])
        dev = g.last_searches() if info.num_searched else []

        def search(pairs):
            assert [(s, nid) for s, nid, _ in pairs] == [(s, nid) for s, nid, _, _ in dev]
            return [(c.found, np.array(c.pose[:]), c.translation_weight, c.rotation_weight) for _, _, _, c in dev]

        def solve(sp, npo, cons, frozen):
            ws, wn, _, _ = ctx.pose_graph_solve_sparse(sp, npo, cons, max_iter=50, frozen=frozen)
            return ws, wn

        assert o.add_node(t, n["local"], [(k, f, p) for k, f, _, _, p in n["ins"]], n["matches"], search, solve,
                          time=n["time"]) == bool(info.optimized)
        assert g.last_trimmed() == o.last_trimmed
        trimmed += o.last_trimmed
        if info.optimized and t == 1:
            assert len(g.ids(1, 1)) <= 3
        for tt in (0, 1):
            assert g.ids(tt) == o.ids(tt) and g.ids(tt, 1) == o.ids(tt, False)
            assert np.abs(g.node_poses(tt) - o.node_poses(tt)).max(initial=0) < 1e-9
            assert np.abs(g.submap_poses(tt) - o.submap_poses(tt)).max(initial=0) < 1e-9
        table = g.constraints()
        assert [(c[0], c[1], c[5], c[3], c[4]) for c in table] == [(c[0], c[1], c[5], c[3], c[4]) for c in o.constraints]
        assert all(np.abs(c[2] - w[2]).max() < 1e-12 if c[5] == pg.INTRA else np.array_equal(c[2], w[2])
                   for c, w in zip(table, o.constraints))
    assert trimmed and all(s[0] == 1 for s in trimmed)
    print(f"{len(o.solves)} solves, trimmed {trimmed}")


def test_periodic_solves_over_holes_are_the_sparse_call_bit_for_bit(recorded):  # noqa: F811
    """A twin graph without trigger or trimmer receives the same nodes; at every node where the periodic graph (trimmer kept 3)
    optimized, the twin's run_final_optimization equals dl_pose_graph_solve_sparse on the twin's exported optimization poses
    and constraint table, rows skipping the holes, bit for bit; the twin then trims by hand what the trimmer trimmed, and both
    graphs hold the same ids and poses, bit for bit."""
    import dliom
    ctx, nodes = recorded
    a = dliom.PoseGraph3D(ctx, options(optimize_every_n_nodes=4))
    b = dliom.PoseGraph3D(ctx, options())
    a.add_pure_localization_trimmer(1, 3)
    checked = 0
    for t, n in nodes:
        info = a.add_node(t, n["time"], n["local"], n["hi"], n["lo"], n["ins"], n["matches"])
        b.add_node(t, n["time"], n["local"], n["hi"], n["lo"], n["ins"], n["matches"])
        if not info.optimized:
            continue
        ts = [tt for tt in (0, 1) if b.ids(tt, 1)]
        sp = np.concatenate([b.optimization_poses(tt)[0] for tt in ts])
        npo = np.concatenate([b.optimization_poses(tt)[1] for tt in ts])
        srow = {(tt, i): k for k, (tt, i) in enumerate((tt, i) for tt in ts for i in b.ids(tt, 1))}
        nrow = {(tt, i): k for k, (tt, i) in enumerate((tt, i) for tt in ts for i in b.ids(tt))}
        summary = b.run_final_optimization()
        cons = [(srow[s], nrow[nd], z, tw, rw) for s, nd, z, tw, rw, _ in b.constraints()]
        ws, wn, wsum, _ = ctx.pose_graph_solve_sparse(sp, npo, cons, max_iter=50)
        assert summary == wsum == info.summary.as_dict()
        assert np.array_equal(np.concatenate([b.optimization_poses(tt)[0] for tt in ts]), ws)
        assert np.array_equal(np.concatenate([b.node_poses(tt) for tt in ts]), wn)
        for s in a.last_trimmed():
            b.trim_submap(*s)
        for tt in (0, 1):
            assert a.ids(tt) == b.ids(tt) and a.ids(tt, 1) == b.ids(tt, 1)
            assert np.array_equal(a.node_poses(tt), b.node_poses(tt))
            assert np.array_equal(a.submap_poses(tt), b.submap_poses(tt))
        assert [(c[0], c[1], c[2].tobytes()) for c in a.constraints()] == [(c[0], c[1], c[2].tobytes()) for c in b.constraints()]
        checked += 1
    assert checked >= 8 and a.ids(1, 1)[0] > 0


def test_compaction_keeps_every_live_cloud(recorded):  # noqa: F811
    """Trajectory 2's huge clouds go into the store first; finishing trajectory 2 with a trimmer trims it whole, its clouds die,
    and the store is compacted (every live node moves). Trajectory 1's later searches, which read nodes uploaded before the
    compaction, give the same dl_constraint records, bit for bit, as in a graph that never held trajectory 2."""
    import dliom
    ctx, nodes = recorded
    n0 = [(t, n) for t, n in nodes if t == 0]
    n1 = [(t, n) for t, n in nodes if t == 1]
    k = next(i for i, (_, n) in enumerate(n1) if n["ins"][0][1])      # trajectory 1's first node finishing a submap
    big = np.tile(n0[0][1]["hi"], (1 + 700_000 // len(n0[0][1]["hi"]), 1))
    _, _, hg, lg, pose = n0[0][1]["ins"][0]
    g, h = dliom.PoseGraph3D(ctx, options()), dliom.PoseGraph3D(ctx, options())
    for j in range(2):
        g.add_node(2, 1.0 + j, n0[0][1]["local"], big, n0[0][1]["lo"], [(0, False, hg, lg, pose)])
    for graph in (g, h):
        for t, n in n0 + n1[:k]:
            graph.add_node(t, n["time"], n["local"], n["hi"], n["lo"], n["ins"], n["matches"])
    live, used, cap = g.store_usage()
    assert used - live == 0 and live > 2 * 12 * len(big)
    g.add_pure_localization_trimmer(2, 3)
    g.finish_trajectory(2)
    assert g.last_trimmed() == [(2, 0)] and g.ids(2) == [] and g.is_trajectory_finished(2)
    live2, used2, cap2 = g.store_usage()
    assert used2 == live2 == live - 2 * 12 * (len(big) + len(n0[0][1]["lo"]))      # compacted
    assert live2 == h.store_usage()[0]
    compared = 0
    for t, n in n1[k:]:
        ig = g.add_node(t, n["time"], n["local"], n["hi"], n["lo"], n["ins"], n["matches"])
        ih = h.add_node(t, n["time"], n["local"], n["hi"], n["lo"], n["ins"], n["matches"])
        assert ig.num_searched == ih.num_searched
        if ig.num_searched:
            sg, sh = g.last_searches(), h.last_searches()
            assert [(s[0], s[1]) for s in sg] == [(s[0], s[1]) for s in sh]
            assert all(bytes(x[3]) == bytes(y[3]) for x, y in zip(sg, sh))
            compared += len(sg)
    assert compared > 0


def test_rejections_leave_the_graph_unchanged(recorded):  # noqa: F811
    import dliom
    ctx, nodes = recorded
    n0 = [(t, n) for t, n in nodes if t == 0]
    n1 = [(t, n) for t, n in nodes if t == 1]
    g = dliom.PoseGraph3D(ctx, options())
    for t, n in n0:
        g.add_node(t, n["time"], n["local"], n["hi"], n["lo"], n["ins"], n["matches"])
    last = g.ids(0, 1)[-1]

    def refused(call, *args):
        s0 = state(g)
        with pytest.raises(dliom.DlError) as e:
            call(*args)
        assert e.value.status == -2 and state(g) == s0, call

    refused(g.trim_submap, 0, last)          # unfinished
    refused(g.trim_submap, 0, 99)            # unknown
    refused(g.trim_submap, 3, 0)
    refused(g.add_pure_localization_trimmer, 1, 2)
    g.run_final_optimization()
    g.trim_submap(0, 0)
    assert g.last_trimmed() == [(0, 0)] and g.ids(0, 1)[0] == 1
    refused(g.trim_submap, 0, 0)             # already trimmed
    # a match naming a trimmed submap
    k = next(i for i, (_, n) in enumerate(n1) if n["ins"][0][1])
    for t, n in n1[:k]:
        g.add_node(t, n["time"], n["local"], n["hi"], n["lo"], n["ins"], n["matches"])
    t, n = n1[k]
    assert n["matches"][0][:2] == (0, 0)
    refused(g.add_node, t, n["time"], n["local"], n["hi"], n["lo"], n["ins"], n["matches"])
    g.add_node(t, n["time"], n["local"], n["hi"], n["lo"], n["ins"])
    found = 0
    for k in range(k + 1, len(n1)):          # on to trajectory 1's next finished submap, matched to the map's submap 1
        t, n = n1[k]
        found += g.add_node(t, n["time"], n["local"], n["hi"], n["lo"], n["ins"], n["matches"]).num_found
        if n["matches"]:
            break
    assert found > 0
    refused(g.trim_submap, 0, 2)             # constraints pending
    g.run_final_optimization()
    # finished: every submap of trajectory 1 trimmed, finishing twice or adding a node refused
    g.add_pure_localization_trimmer(1, 3)
    g.finish_trajectory(1)
    assert g.ids(1) == [] and g.ids(1, 1) == []
    refused(g.finish_trajectory, 1)
    t, n = n1[-1]
    refused(g.add_node, t, n["time"], n["local"], n["hi"], n["lo"], n["ins"], n["matches"])
    # an initial pose relative to a trajectory without nodes
    g.set_initial_trajectory_pose(5, 9, pg.IDENTITY, 0.0)
    refused(g.local_to_global, 5)
    t, n = n0[0]
    refused(g.add_node, 5, n["time"], n["local"], n["hi"], n["lo"], n["ins"][:1])


def errors_to_truth(poses, times):
    import synth
    return np.array([pose_error(p, synth.pose7(t)) for p, t in zip(poses, times)]).reshape(-1, 2)


@pytest.mark.parametrize("with_matches", [True, False])
def test_localization_end_to_end(with_matches):
    """Trajectory 0 mapped and frozen; trajectory 1 (60 scans, num_range_data 2: over 20 submaps) localized live with
    add_pure_localization_trimmer(1, 3), optimizing every 4 nodes, from an initial pose off by 1 m and 5 degrees at its first
    node. With the map's matches every remaining node of trajectory 1 is within 10 % of that error after each optimization that
    has INTER_SUBMAP constraints; without them (the control) every node keeps at least 90 % of it. Right after each
    optimization the builder holds grids for at most 3 of the submaps the graph has seen (plus the submap it opened in the
    same call, which the graph sees with the next node), and the store keeps used <= 2 * live or fewer than 4 MiB dead. After
    finish_trajectory nothing of trajectory 1 is left in the graph and the builder holds its two active submaps' grids only."""
    import dliom
    import bench_localization as bl
    ctx = dliom.Context(0)
    opts = options(optimize_every_n_nodes=4)
    scans = bl.scans_of(60)
    g, b0, local0 = bl.map_graph(ctx, opts, scans, 2)
    offset = bl.OFFSET
    b1 = bl.make_builder(ctx, offset, scans[0][0], 2)
    # the injected error D (1 m forward, 5 deg yaw) in the frame of the first node's true local pose
    import synth
    first_local = pg.compose(pg.inverse(offset), synth.pose7(scans[0][0]))
    d = np.concatenate([[1.0, 0.0, 0.0], pg.yaw_quaternion(np.deg2rad(5.0))])
    x = pg.compose(pg.compose(first_local, d), pg.inverse(first_local))
    rel = pg.compose(pg.compose(pg.inverse(g.node_poses(0)[0]), offset), x)
    g.set_initial_trajectory_pose(1, 0, rel, -1.0)
    g.add_pure_localization_trimmer(1, 3)
    times1 = {}
    checks = dict(optimized=0, with_inter=0, worst=np.zeros(2), best=np.full(2, np.inf))
    node_bytes = []

    def after_node(r, info, ms):
        times1[info.node_index] = r.time
        node_bytes.append(12 * (r.num_high_resolution + r.num_low_resolution))
        if not info.optimized:
            return
        checks["optimized"] += 1
        seen = set(g.ids(1, 1)) | {s[1] for s in g.last_trimmed()}
        held = [i for i in range(b1.num_submaps()) if b1.submap(i)[0].h]
        newest_unseen = b1.num_submaps() - 1 not in seen and b1.num_submaps() - 1 > max(g.ids(1, 1))
        assert len(held) <= 3 + int(newest_unseen), (held, g.ids(1, 1))
        live, used, _ = g.store_usage()
        assert used <= 2 * live + max(node_bytes) or used - live < 4 << 20
        inter = [c for c in g.constraints() if c[5] == dliom.PG3D_INTER_SUBMAP and c[1][0] == 1]
        err = errors_to_truth(g.node_poses(1), [times1[i] for i in g.ids(1)])
        if with_matches and inter:
            checks["with_inter"] += 1
            checks["worst"] = np.maximum(checks["worst"], err.max(0))
            assert err[:, 0].max() < 0.1 and err[:, 1].max() < np.deg2rad(0.5), err
        if not with_matches:
            checks["best"] = np.minimum(checks["best"], err.min(0))
            assert err[:, 0].min() >= 0.9 and err[:, 1].min() >= np.deg2rad(4.5), err

    bl.feed(g, 1, b1, scans, bl.truth_matches(local0, offset) if with_matches else None, after_node)
    assert b1.num_submaps() >= 20 and checks["optimized"] >= 10
    assert checks["with_inter"] >= 5 if with_matches else True
    g.finish_trajectory(1)
    assert g.ids(1) == [] and g.ids(1, 1) == [] and not [c for c in g.constraints() if c[1][0] == 1 or c[0][0] == 1]
    held = [i for i in range(b1.num_submaps()) if b1.submap(i)[0].h]
    assert held == [b1.num_submaps() - 2, b1.num_submaps() - 1]
    w = checks["worst"] if with_matches else checks["best"]
    print(f"localization with_matches={with_matches}: {checks['optimized']} optimizations, {b1.num_submaps()} submaps; "
          f"{'worst' if with_matches else 'smallest'} node error vs truth {w[0]:.4f} m / {np.rad2deg(w[1]):.4f} deg "
          f"(injected 1 m / 5 deg); store usage after finish {g.store_usage()}")
    g.close()
    b1.close()
    b0.close()


def write_localization_drive(path, builders, nodes, optimize_every_n_nodes, keep, rel, time):
    """The input of host/example_localization.cc: options, the initial pose, then both trajectories' recorded events."""
    import struct
    import dliom
    matches = {(t, i): n["matches"] for t, i, n in _ids(nodes)}
    with open(path, "wb") as f:
        f.write(struct.pack("<ii", optimize_every_n_nodes, keep) + np.asarray(rel, np.float64).tobytes() + struct.pack("<d", time))
        for t, b in enumerate(builders):
            f.write(bytes(dliom.NavState.from16(b.init)))
            f.write(struct.pack("<i", len(b.events)))
            for e in b.events:
                if e[0] == "imu":
                    f.write(struct.pack("<id", 0, e[1]) + np.asarray(e[2], np.float64).tobytes() + np.asarray(e[3], np.float64).tobytes())
                    continue
                m = matches[(t, e[3])]
                f.write(struct.pack("<idi", 1, e[1], len(e[2])) + e[2].tobytes() + struct.pack("<i", len(m)))
                for mt, mi, x, y, th in m:
                    f.write(struct.pack("<ii3d", mt, mi, x, y, th))


def test_cpp_localization_example_equals_the_python_replay(recorded, tmp_path):  # noqa: F811
    """build/example_localization (host/example_localization.cc, built by build()): the recorded drive replayed through the C++
    LocalTrajectoryBuilder3D and PoseGraph3D with SetInitialTrajectoryPose, a PureLocalizationTrimmer and FinishTrajectory
    prints, to the last bit, what the same replay through dliom prints: trajectory 1's remaining node ids and poses after every
    optimization, the submaps left, the builder's submaps still holding grids, and the state after FinishTrajectory."""
    import os
    import subprocess
    import dliom
    import orc
    from test_gpu_pose_graph3d import NOISE
    ctx, nodes = recorded
    exe = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "build", "example_localization")
    rel = np.concatenate([[0.4, -0.3, 0.0], pg.yaw_quaternion(0.04)])
    t_init = nodes[3][1]["time"] + 0.05
    path = str(tmp_path / "drive.bin")
    write_localization_drive(path, ctx.pose_graph_builders, nodes, 4, 3, rel, t_init)
    out = subprocess.run([exe, path], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    # the Python replay: fresh builders fed the recorded events, nodes through add_node_from_builder
    g = dliom.PoseGraph3D(ctx, options(optimize_every_n_nodes=4))
    fo = dliom.FrontendOptions.from_oracle(orc.FrontEndOptions.defaults())
    matches = {(t, i): n["matches"] for t, i, n in _ids(nodes)}
    want, builders, k = [], [], 0
    for t, rec in enumerate(ctx.pose_graph_builders):
        if t == 1:
            g.run_final_optimization()
            g.freeze_trajectory(0)
            g.set_initial_trajectory_pose(1, 0, rel, t_init)
            g.add_pure_localization_trimmer(1, 3)
        b = dliom.LocalTrajectoryBuilder(ctx, dliom.LtbOptions.defaults(fo, NOISE, imu_weight=0.7, num_range_data=3,
                                                                         max_time_seconds=0.05))
        builders.append(b)
        b.set_initial_state(rec.init)
        for e in rec.events:
            if e[0] == "imu":
                b.add_imu_data(e[1], e[2], e[3])
                continue
            rows = np.zeros(len(e[2]), dtype=[("x", np.float32), ("y", np.float32), ("z", np.float32), ("t", np.float32),
                                              ("origin_index", np.uint64), ("_pad", np.uint64)])
            rows["x"], rows["y"], rows["z"], rows["t"] = e[2].T
            r = b.add_synchronized_range_data(e[1], rows, np.zeros((1, 3), np.float32))
            if not (r.has_result and r.inserted):
                continue
            info = g.add_node_from_builder(t, b, r, matches[(t, e[3])])
            if t != 1 or not info.optimized:
                continue
            held = sum(1 for i in range(b.num_submaps()) if b.submap(i)[0].h)
            want.append(("opt", k, len(g.ids(1, 1)), held))
            k += 1
            for i, p in zip(g.ids(1), g.node_poses(1)):
                want.append(("node", i, *p))
    g.finish_trajectory(1)
    held = sum(1 for i in range(builders[1].num_submaps()) if builders[1].submap(i)[0].h)
    want.append(("finished", len(g.ids(1)), len(g.ids(1, 1)), held))
    got = []
    for line in out.stdout.strip().splitlines():
        kind, *v = line.split()
        got.append((kind, int(v[0]), *[float(x) for x in v[1:]]) if kind == "node" else (kind, *[int(x) for x in v]))
    assert got == want        # %.17g round-trips every double
    assert k > 0 and held == 2 and want[-1][1:3] == (0, 0)
    g.close()
    for b in builders:
        b.close()
