"""mapping::PoseGraph3D on the device (dl_pose_graph_3d_*): two trajectories of the synthetic street driven through dl_ltb, the
second one's local frame offset from the first's by a known planar transform; submap matches derived from the synthetic truth
and perturbed inside the coarse window. Checked against the numpy oracle's bookkeeping (tests/pose_graph3d_oracle.py), against
dl_constraint_search_batch and dl_pose_graph_solve_sparse bit for bit, and for the loop actually closing."""
import numpy as np
import pytest

import imu_synth
import pose_graph3d_oracle as pg
from helpers import pose_error

pytestmark = pytest.mark.gpu
NOISE = [3.99e-2, 1.56e-2, 6.4e-5, 3.6e-5]
OFFSET = np.concatenate([[4.0, -3.0, 0.0], pg.yaw_quaternion(np.deg2rad(5.0))])   # world <- trajectory 1's local frame
MATCH_PERTURBATION = (0.3, -0.2, 0.01)    # m, m, rad added to every true match: inside the 5 m coarse window
NUM_SCANS = 24


def state_in(local_to_world, s16):
    inv = pg.inverse(local_to_world)
    p = pg.compose(inv, s16[:7])
    v = pg.rotate(inv[3:], s16[7:10])
    return np.concatenate([p, v, s16[10:]])


def drive(ctx, offset):
    """One trajectory through a LocalTrajectoryBuilder -> (builder, [node records]). A record: time, local pose, clouds,
    insertion submaps (index, finished after the insert, hi grid, lo grid, local pose)."""
    import dliom
    import orc
    import synth
    scene = synth.Scene(42)
    fo = dliom.FrontendOptions.from_oracle(orc.FrontEndOptions.defaults())
    b = dliom.LocalTrajectoryBuilder(ctx, dliom.LtbOptions.defaults(fo, NOISE, imu_weight=0.7, num_range_data=3,
                                                                     max_time_seconds=0.05))
    times = [2.0 + 0.1 * k for k in range(NUM_SCANS)]
    init = state_in(offset, imu_synth.state(times[0] - 0.1))
    b.set_initial_state(init)
    nodes, events = [], []
    for k, t1 in enumerate(times):
        dt, acc, gyr = imu_synth.samples(t1 - 0.1, t1)
        ts = t1 - 0.1 + np.arange(len(dt)) / 200.0
        for j in range(0 if k == 0 else 1, len(dt)):
            b.add_imu_data(ts[j], acc[j], gyr[j])
            events.append(("imu", ts[j], acc[j], gyr[j]))
        rows = synth.make_scan(scene, 16, t1)     # RangeMeasurement rows, origin index 0: what the C++ builder's synchroniser
        r = b.add_synchronized_range_data(t1, rows, np.zeros((1, 3), np.float32))   # makes of a single LiDAR's cloud
        events.append(("range", t1, np.stack([rows["x"], rows["y"], rows["z"], rows["t"]], 1).astype(np.float32), len(nodes)))
        assert r.has_result == 1 and r.inserted == 1
        ins = []
        for i in range(r.num_insertion_submaps):
            hg, lg, pose, _, fin = b.submap(r.insertion_submap_index[i])
            ins.append((r.insertion_submap_index[i], fin, hg, lg, pose))
        nodes.append(dict(time=t1, local=np.array(r.local_pose[:]), hi=b.cloud(2), lo=b.cloud(3), ins=ins))
    b.init, b.events = init, events
    return b, nodes


@pytest.fixture(scope="module")
def recorded():
    import dliom
    ctx = dliom.Context(0)
    b0, n0 = drive(ctx, pg.IDENTITY)
    b1, n1 = drive(ctx, OFFSET)
    local0 = {i: p for n in n0 for i, _, _, _, p in n["ins"]}
    # matches of trajectory 1's finished submaps: the same-index submap of trajectory 0, from the truth, perturbed
    for n in n1:
        idx, fin, _, _, pose = n["ins"][0]
        n["matches"] = []
        if fin:
            x, y, th = pg.match_from_truth(pose, local0[idx], OFFSET, pg.IDENTITY)
            n["matches"] = [(0, idx, x + MATCH_PERTURBATION[0], y + MATCH_PERTURBATION[1], th + MATCH_PERTURBATION[2])]
    for n in n0:
        n["matches"] = []
    ctx.pose_graph_builders = (b0, b1)    # their events and initial states, for the replays
    yield ctx, [(0, n) for n in n0] + [(1, n) for n in n1]
    b0.close()
    b1.close()


def options(optimize_every_n_nodes=0):
    import dliom
    return dliom.PoseGraph3DOptions.defaults(optimize_every_n_nodes=optimize_every_n_nodes, every_nodes_to_find_constraint=2,
                                             min_score=0.3, min_low_resolution_score=0.3)


def replay(ctx, nodes, opts, freeze=(), final=True):
    import dliom
    g = dliom.PoseGraph3D(ctx, opts)
    for t in freeze:
        g.freeze_trajectory(t)
    infos = [g.add_node(t, n["time"], n["local"], n["hi"], n["lo"], n["ins"], n["matches"]) for t, n in nodes]
    if final:
        g.run_final_optimization()
    return g, infos


def test_drive_matches_oracle_search_batch_and_sparse_solve(recorded):
    """(a) ids, INTRA constraints, pairs and guesses equal the oracle's; (b) every search equals dl_constraint_search_batch on the
    same pairs and guesses bit for bit; (c) the final optimization equals dl_pose_graph_solve_sparse on the exported graph."""
    import dliom
    ctx, nodes = recorded
    opts = options()
    g = dliom.PoseGraph3D(ctx, opts)
    o = pg.PoseGraph3D(0, 2)
    grids = {}
    searched = 0
    for t, n in nodes:
        for idx, _, hg, lg, _ in n["ins"]:
            grids[(t, idx)] = (hg, lg)
        info = g.add_node(t, n["time"], n["local"], n["hi"], n["lo"], n["ins"], n["matches"])
        dev = g.last_searches() if info.num_searched else []
        assert info.num_searched == len(dev) and info.optimized == 0

        def search(pairs):
            assert [(s, nid) for s, nid, _ in pairs] == [(s, nid) for s, nid, _, _ in dev]
            for (_, _, guess), (_, _, dguess, _) in zip(pairs, dev):
                assert np.abs(guess - dguess).max() < 1e-12
            clouds = {nid: (nodes_by_id[nid]["hi"], nodes_by_id[nid]["lo"]) for _, nid, _, _ in dev}
            want = ctx.constraint_search_batch(opts.constraint_builder, [d[2] for d in dev], [clouds[d[1]][0] for d in dev],
                                               [clouds[d[1]][1] for d in dev], [grids[d[0]][0] for d in dev],
                                               [grids[d[0]][1] for d in dev])
            for w, (_, _, _, got) in zip(want, dev):
                assert bytes(w) == bytes(got)     # bit-identical records
            return [(c.found, np.array(c.pose[:]), c.translation_weight, c.rotation_weight) for c in want]

        nodes_by_id = {(tt, i): nn for tt, i, nn in _ids(nodes)}
        o.add_node(t, n["local"], [(i, f, p) for i, f, _, _, p in n["ins"]], n["matches"], search)
        searched += len(dev)
    assert searched == len(o.searched) > 0     # no pair searched on one side only
    assert sum(1 for c in g.constraints() if c[5] == dliom.PG3D_INTER_SUBMAP) == 0   # pending until optimized
    # (c) export the graph, solve it with the sparse call, compare with the object's own final optimization
    sp = np.concatenate([g.optimization_poses(t)[0] for t in (0, 1)])
    npo = np.concatenate([g.optimization_poses(t)[1] for t in (0, 1)])
    summary = g.run_final_optimization()
    table = g.constraints()
    ns = [len(g.optimization_poses(t)[0]) for t in (0, 1)]
    nn = [len(g.optimization_poses(t)[1]) for t in (0, 1)]
    sbase, nbase = {0: 0, 1: ns[0]}, {0: 0, 1: nn[0]}
    cons = [(sbase[s[0]] + s[1], nbase[n[0]] + n[1], z, tw, rw) for s, n, z, tw, rw, _ in table]
    ws, wn, wsum, _ = ctx.pose_graph_solve_sparse(sp, npo, cons, max_iter=opts.optimization_problem.max_num_iterations)
    assert np.array_equal(np.concatenate([g.optimization_poses(t)[0] for t in (0, 1)]), ws)
    assert np.array_equal(np.concatenate([g.node_poses(t) for t in (0, 1)]), wn)
    assert summary == wsum
    # (a) the oracle's final optimization on the same solve; the tables agree
    o.optimize(lambda a, b, c, f: ctx.pose_graph_solve_sparse(a, b, c, max_iter=50, frozen=f)[:2])
    assert [(c[0], c[1], c[5]) for c in table] == [(c[0], c[1], c[5]) for c in o.constraints]
    for c, w in zip(table, o.constraints):
        tol = 1e-12 if c[5] == dliom.PG3D_INTRA_SUBMAP else 0.0
        assert np.abs(c[2] - w[2]).max() <= tol and (c[3], c[4]) == (w[3], w[4])
    inter = [c for c in table if c[5] == dliom.PG3D_INTER_SUBMAP]
    assert len(inter) > 0
    for t in (0, 1):
        assert len(g.node_poses(t)) == NUM_SCANS
        assert np.abs(g.node_poses(t) - o.node_poses(t)).max() < 1e-9
        assert np.abs(g.submap_poses(t) - o.submap_poses(t)).max() < 1e-9
    print(f"searched {searched} pairs, {len(inter)} INTER_SUBMAP constraints, final solve {summary}")


def _ids(nodes):
    count = {}
    for t, n in nodes:
        i = count.get(t, 0)
        count[t] = i + 1
        yield t, i, n


def errors_to_truth(poses, nodes):
    import synth
    return np.array([pose_error(p, synth.pose7(n["time"])) for p, n in zip(poses, nodes)])


def test_loop_closes_and_clouds_are_uploaded_once(recorded):
    ctx, nodes = recorded
    g, infos = replay(ctx, nodes, options(), final=False)
    n1 = [n for t, n in nodes if t == 1]
    before = errors_to_truth(g.node_poses(1), n1)
    off_t = np.linalg.norm(OFFSET[:3])
    assert before[:, 0].min() > 0.5 * off_t and before[:, 1].min() > np.deg2rad(4.0)   # off by the injected offset
    g.run_final_optimization()
    after = errors_to_truth(g.node_poses(1), n1)
    after0 = errors_to_truth(g.node_poses(0), [n for t, n in nodes if t == 0])
    print(f"trajectory 1 vs truth: before {before[:, 0].max():.3f} m / {np.rad2deg(before[:, 1].max()):.3f} deg, after "
          f"{after[:, 0].max():.4f} m / {np.rad2deg(after[:, 1].max()):.4f} deg (trajectory 0: {after0[:, 0].max():.4f} m / "
          f"{np.rad2deg(after0[:, 1].max()):.4f} deg)")
    assert after[:, 0].max() < 0.2 and after[:, 1].max() < np.deg2rad(1.0)
    # every cloud byte crossed the bus once, at its node's add_node
    want = sum(12 * (len(n["hi"]) + len(n["lo"])) for _, n in nodes)
    assert sum(i.cloud_bytes_uploaded for i in infos) == want == g.store_bytes()[0]
    assert all(i.cloud_bytes_uploaded == 12 * (len(n["hi"]) + len(n["lo"])) for i, (_, n) in zip(infos, nodes))
    assert sum(i.num_searched for i in infos) > 0


def test_periodic_optimization_is_deterministic_and_frozen_trajectory_stays(recorded):
    ctx, nodes = recorded
    a, ia = replay(ctx, nodes, options(optimize_every_n_nodes=10))
    b, _ = replay(ctx, nodes, options(optimize_every_n_nodes=10))
    assert [i.optimized for i in ia].count(1) == 4      # after nodes 11, 22, 33 and 44 (the count must exceed 10)
    assert [k for k, i in enumerate(ia) if i.optimized] == [10, 21, 32, 43]
    for t in (0, 1):
        assert np.array_equal(a.node_poses(t), b.node_poses(t))
        assert np.array_equal(a.submap_poses(t), b.submap_poses(t))
    f, _ = replay(ctx, nodes, options(optimize_every_n_nodes=10), freeze=(0,))
    unopt, _ = replay(ctx, [(t, n) for t, n in nodes if t == 0], options(), final=False)
    for freeze, graph in (((), a), ((0,), f)):
        checked = checked_periodic_run(ctx, nodes, freeze)
        checked.run_final_optimization()     # replay() ends with the final optimization too
        for t in (0, 1):
            assert np.array_equal(graph.node_poses(t), checked.node_poses(t))
    for want, got in zip(unopt.optimization_poses(0), f.optimization_poses(0)):   # submaps, nodes
        assert np.array_equal(want, got)


def exported_poses(g):
    """The graph's optimization poses per trajectory that has submaps: {trajectory: (submaps, nodes)}."""
    return {t: g.optimization_poses(t) for t in (0, 1) if len(g.optimization_poses(t)[0])}


def solve_exported(ctx, g, poses, frozen_trajectories, max_iter):
    """dl_pose_graph_solve_sparse on exported optimization poses, the graph's constraint table (pending constraints appended by
    the optimization) and the frozen mask."""
    ts = sorted(poses)
    sbase = dict(zip(ts, np.cumsum([0] + [len(poses[t][0]) for t in ts])[:-1]))
    nbase = dict(zip(ts, np.cumsum([0] + [len(poses[t][1]) for t in ts])[:-1]))
    cons = [(sbase[s[0]] + s[1], nbase[n[0]] + n[1], z, tw, rw) for s, n, z, tw, rw, _ in g.constraints()]
    frozen = [t in frozen_trajectories for t in ts for _ in poses[t][0]] + [t in frozen_trajectories for t in ts for _ in poses[t][1]]
    ws, wn, wsum, _ = ctx.pose_graph_solve_sparse(np.concatenate([poses[t][0] for t in ts]), np.concatenate([poses[t][1] for t in ts]),
                                                  cons, max_iter=max_iter, frozen=frozen)
    return ts, ws, wn, wsum


def checked_periodic_run(ctx, nodes, freeze):
    """The optimize_every_n_nodes = 10 drive, with every periodic optimization compared bit for bit against the sparse call on
    the graph exported just before it: a twin graph without the trigger receives the same nodes and runs the same step through
    run_final_optimization at the nodes where the periodic graph optimized."""
    import dliom
    a = dliom.PoseGraph3D(ctx, options(optimize_every_n_nodes=10))
    b = dliom.PoseGraph3D(ctx, options())
    for t in freeze:
        a.freeze_trajectory(t)
        b.freeze_trajectory(t)
    checked = 0
    for t, n in nodes:
        info = a.add_node(t, n["time"], n["local"], n["hi"], n["lo"], n["ins"], n["matches"])
        b.add_node(t, n["time"], n["local"], n["hi"], n["lo"], n["ins"], n["matches"])
        if not info.optimized:
            continue
        before = exported_poses(b)
        summary = b.run_final_optimization()
        assert [c[:2] for c in a.constraints()] == [c[:2] for c in b.constraints()]
        ts, ws, wn, wsum = solve_exported(ctx, b, before, freeze, 50)
        assert summary == wsum == info.summary.as_dict()
        for graph in (a, b):
            assert np.array_equal(np.concatenate([graph.optimization_poses(t)[0] for t in ts]), ws)
            assert np.array_equal(np.concatenate([graph.node_poses(t) for t in ts]), wn)
        checked += 1
    assert checked == 4
    return a


def test_invalid_matches_are_rejected_and_leave_the_graph_unchanged(recorded):
    import dliom
    ctx, nodes = recorded
    n0 = [(t, n) for t, n in nodes if t == 0]
    n1 = [(t, n) for t, n in nodes if t == 1]
    k = next(i for i, (_, n) in enumerate(n1) if n["ins"][0][1])          # trajectory 1's first node finishing a submap
    g, _ = replay(ctx, n0 + n1[:k], options(), final=False)
    t, n = n1[k]
    fin_idx = n["ins"][0][0]
    unfinished0 = max(i for _, nn in n0 for i, _, _, _, _ in nn["ins"])

    def state():
        return ([g.node_poses(tt).tobytes() for tt in (0, 1)], [g.submap_poses(tt).tobytes() for tt in (0, 1)],
                [(c[0], c[1], c[2].tobytes(), c[5]) for c in g.constraints()], g.store_bytes())

    s0 = state()
    bad = [[(0, 99, 0.0, 0.0, 0.0)],                      # unknown submap
           [(0, unfinished0, 0.0, 0.0, 0.0)],             # unfinished submap
           [(1, fin_idx, 0.0, 0.0, 0.0)],                 # the finished submap itself
           [(0, 0, 0.0, 0.0, 0.0), (0, 0, 1.0, 0.0, 0.0)]]  # a submap twice
    for m in bad:
        with pytest.raises(dliom.DlError) as e:
            g.add_node(t, n["time"], n["local"], n["hi"], n["lo"], n["ins"], m)
        assert e.value.status == -2, m
        assert state() == s0
    # matches with no finished submap
    t2, n2 = n1[k + 1]
    assert not n2["ins"][0][1]
    with pytest.raises(dliom.DlError) as e:
        g.add_node(t2, n2["time"], n2["local"], n2["hi"], n2["lo"], n2["ins"], [(0, 0, 0.0, 0.0, 0.0)])
    assert e.value.status == -2 and state() == s0
    # a same-trajectory submap within two indices: trajectory 0 replayed past its submap 3's finish, matched to submap 2
    g0, _ = replay(ctx, [], options(), final=False)

    def state0():
        return ([g0.node_poses(tt).tobytes() for tt in (0, 2)], [g0.submap_poses(tt).tobytes() for tt in (0, 2)],
                [(c[0], c[1], c[2].tobytes(), c[5]) for c in g0.constraints()], g0.store_bytes())

    for tt, nn in n0:
        if nn["ins"][0][1] and nn["ins"][0][0] == 3:
            before = state0()
            with pytest.raises(dliom.DlError) as e:
                g0.add_node(tt, nn["time"], nn["local"], nn["hi"], nn["lo"], nn["ins"], [(0, 2, 0.0, 0.0, 0.0)])
            assert e.value.status == -2 and state0() == before
            break
        g0.add_node(tt, nn["time"], nn["local"], nn["hi"], nn["lo"], nn["ins"], nn["matches"])
    else:
        pytest.fail("trajectory 0 never finished its submap 3")
    # a new submap whose index is not the trajectory's next one
    tt, nn = n0[0]
    skip = [(5, False, nn["ins"][0][2], nn["ins"][0][3], nn["ins"][0][4])]
    before = state0()
    with pytest.raises(dliom.DlError) as e:
        g0.add_node(2, nn["time"], nn["local"], nn["hi"], nn["lo"], skip)
    assert e.value.status == -2 and state0() == before
    # the graph goes on after the rejections
    g.add_node(t, n["time"], n["local"], n["hi"], n["lo"], n["ins"], n["matches"])


def test_add_node_from_builder_equals_the_recorded_nodes(recorded):
    """PoseGraph3D.add_node_from_builder (the GlobalTrajectoryBuilder wiring): trajectory 0 driven live into a graph gives the same
    poses and constraints, bit for bit, as its recorded nodes passed to add_node."""
    import dliom
    ctx, nodes = recorded
    b = ctx.pose_graph_builders[0]
    live = dliom.PoseGraph3D(ctx, options(optimize_every_n_nodes=10))
    # the recorded events of trajectory 0 into a fresh builder that feeds the graph as it goes
    import orc
    fo = dliom.FrontendOptions.from_oracle(orc.FrontEndOptions.defaults())
    b2 = dliom.LocalTrajectoryBuilder(ctx, dliom.LtbOptions.defaults(fo, NOISE, imu_weight=0.7, num_range_data=3,
                                                                      max_time_seconds=0.05))
    b2.set_initial_state(b.init)
    for e in b.events:
        if e[0] == "imu":
            b2.add_imu_data(e[1], e[2], e[3])
            continue
        rows = np.zeros(len(e[2]), dtype=[("x", np.float32), ("y", np.float32), ("z", np.float32), ("t", np.float32),
                                          ("origin_index", np.uint64), ("_pad", np.uint64)])
        rows["x"], rows["y"], rows["z"], rows["t"] = e[2].T
        r = b2.add_synchronized_range_data(e[1], rows, np.zeros((1, 3), np.float32))
        live.add_node_from_builder(0, b2, r)
    live.run_final_optimization()
    want, _ = replay(ctx, [(t, n) for t, n in nodes if t == 0], options(optimize_every_n_nodes=10))
    assert np.array_equal(live.node_poses(0), want.node_poses(0))
    assert np.array_equal(live.submap_poses(0), want.submap_poses(0))
    assert [(c[0], c[1], c[2].tobytes()) for c in live.constraints()] == [(c[0], c[1], c[2].tobytes()) for c in want.constraints()]
    assert len(live._grids) == 2 * len(live.submap_poses(0))      # one handle per borrowed grid
    live.close()
    b2.close()


def write_drive(path, builders, nodes, optimize_every_n_nodes, frozen):
    import struct
    import dliom
    matches = {(t, i): n["matches"] for t, i, n in _ids(nodes)}
    with open(path, "wb") as f:
        f.write(struct.pack("<i", optimize_every_n_nodes))
        f.write(struct.pack("<i", len(frozen)) + b"".join(struct.pack("<i", t) for t in frozen))
        f.write(struct.pack("<i", len(builders)))
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


def test_cpp_example_replays_the_drive_bit_for_bit(recorded, tmp_path):
    """host/example_global_slam.cc: the two trajectories replayed through the C++ LocalTrajectoryBuilder3D and PoseGraph3D print
    the same node and submap poses, to the last bit, as the Python run of the same drive."""
    import subprocess
    from test_pose_graph3d_oracle import build_global_slam_example
    ctx, nodes = recorded
    exe = build_global_slam_example(tmp_path)
    path = str(tmp_path / "drive.bin")
    write_drive(path, ctx.pose_graph_builders, nodes, 10, [])
    out = subprocess.run([exe, path], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    want, _ = replay(ctx, nodes, options(optimize_every_n_nodes=10))
    lines = out.stdout.strip().splitlines()
    got = {}
    for line in lines[:-1]:
        k, t, i, *p = line.split()
        got.setdefault((k, int(t)), []).append([float(v) for v in p])     # %.17g: exact round trip
    for t in (0, 1):
        assert np.array_equal(np.array(got[("node", t)]), want.node_poses(t))
        assert np.array_equal(np.array(got[("submap", t)]), want.submap_poses(t))
    intra = sum(1 for c in want.constraints() if c[5] == 0)
    assert lines[-1].split()[-2:] == [str(intra), str(len(want.constraints()) - intra)]
