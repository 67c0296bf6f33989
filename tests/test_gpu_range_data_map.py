"""The range-data map on the device (dl_range_data_map_*): the recorded two-trajectory drive of tests/test_gpu_pose_graph3d.py
replayed through fresh LocalTrajectoryBuilders with every node's range_data_in_local returns attached
(add_node_from_builder(range_data=True)). The map is checked bit for bit against the float32 reference
(tests/range_data_map_reference.py), a twin graph without range data is checked to be unchanged by the attaching, and pure
localization's trims and compaction, the edges, every rejection and a map of more than 2^31 output bytes are covered."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import pose_graph3d_oracle as pg
import range_data_map_reference as ref
from test_gpu_pose_graph3d import NOISE, _ids, options, recorded, write_drive  # noqa: F401  (the recorded drive)

pytestmark = pytest.mark.gpu
OPTIMIZE_EVERY = 10
ERR_ARG = -2


def replay_events(ctx, rec):
    """Fresh builders fed the recorded events: yields (trajectory, builder, MatchingResult, node ordinal) per inserted node."""
    import dliom
    import orc
    fo = dliom.FrontendOptions.from_oracle(orc.FrontEndOptions.defaults())
    for t, r in enumerate(rec):
        b = dliom.LocalTrajectoryBuilder(ctx, dliom.LtbOptions.defaults(fo, NOISE, imu_weight=0.7, num_range_data=3,
                                                                         max_time_seconds=0.05))
        b.set_initial_state(r.init)
        for e in r.events:
            if e[0] == "imu":
                b.add_imu_data(e[1], e[2], e[3])
                continue
            rows = np.zeros(len(e[2]), dtype=[("x", np.float32), ("y", np.float32), ("z", np.float32), ("t", np.float32),
                                              ("origin_index", np.uint64), ("_pad", np.uint64)])
            rows["x"], rows["y"], rows["z"], rows["t"] = e[2].T
            res = b.add_synchronized_range_data(e[1], rows, np.zeros((1, 3), np.float32))
            if res.has_result and res.inserted:
                yield t, b, res, e[3]


@pytest.fixture(scope="module")
def mapped(recorded):  # noqa: F811
    """Graph `a` (range data attached) and its twin `b` (none) fed the same nodes in lockstep, both finally optimized.
    Per node: its id, local pose and returns; per add_node the infos and last searches of both graphs."""
    import dliom
    ctx, nodes = recorded
    matches = {(t, i): n["matches"] for t, i, n in _ids(nodes)}
    a = dliom.PoseGraph3D(ctx, options(optimize_every_n_nodes=OPTIMIZE_EVERY))
    b = dliom.PoseGraph3D(ctx, options(optimize_every_n_nodes=OPTIMIZE_EVERY))
    builders, records, steps = [], {}, []
    for t, builder, res, k in replay_events(ctx, ctx.pose_graph_builders):
        if not builders or builders[-1] is not builder:
            builders.append(builder)
        ia = a.add_node_from_builder(t, builder, res, matches[(t, k)], range_data=True)
        subs = []
        for j in range(res.num_insertion_submaps):
            hg, lg, pose, _, fin = builder.submap(res.insertion_submap_index[j])
            subs.append((res.insertion_submap_index[j], fin, hg, lg, pose))
        ib = b.add_node(t, res.time, np.array(res.local_pose[:]), builder.cloud(2), builder.cloud(3), subs, matches[(t, k)])
        records[(t, ia.node_index)] = dict(local=np.array(res.local_pose[:]), returns=builder.cloud(0))
        steps.append((ia, ib, a.last_searches() if ia.num_searched else [], b.last_searches() if ib.num_searched else []))
    a.run_final_optimization()
    b.run_final_optimization()
    yield ctx, a, b, records, steps
    a.close()
    b.close()
    for builder in builders:
        builder.close()


def reference_map(g, records, trajectory_ids=None):
    """The float32 reference on the graph's live nodes with range data, at their DL_PG3D_NODE_POSES."""
    nodes = []
    for t in sorted({t for t, _ in records}):
        if trajectory_ids is not None and t not in trajectory_ids:
            continue
        for i, pose in zip(g.ids(t), g.node_poses(t)):
            if (t, i) in records:
                nodes.append((t, i, records[(t, i)]["local"], pose, records[(t, i)]["returns"]))
    return ref.range_data_map(nodes)


def check_map(g, records, trajectory_ids=None):
    points, nodes = g.range_data_map(trajectory_ids)
    want, table = reference_map(g, records, trajectory_ids)
    assert points.dtype == np.float32 and points.shape == want.shape
    assert points.tobytes() == want.tobytes()
    assert [(t, i, f, n) for t, i, f, n, _ in nodes] == table
    dev, dev_nodes = g.range_data_map(trajectory_ids, device=True)
    assert dev.is_cuda and dev.cpu().numpy().tobytes() == points.tobytes()
    assert [(t, i, f, n, p.tobytes()) for t, i, f, n, p in dev_nodes] == [(t, i, f, n, p.tobytes()) for t, i, f, n, p in nodes]
    return points, nodes


def test_map_equals_the_reference_bit_for_bit(mapped):
    """Every point equals the float32 reference bit for bit; the node list is node_poses() and ids() of every node in
    (trajectory, index) order; the host and _dev outputs are byte-identical."""
    ctx, a, _, records, _ = mapped
    points, nodes = check_map(a, records)
    assert len(nodes) == len(records) and len(points) == sum(len(r["returns"]) for r in records.values()) > 0
    for t in (0, 1):
        rows = [n for n in nodes if n[0] == t]
        assert [n[1] for n in rows] == a.ids(t)
        assert np.array_equal(np.array([n[4] for n in rows]), a.node_poses(t))
    launches = ctx.launches
    a.range_data_map()
    assert ctx.launches == launches + 1      # one launch whatever the node count
    print(f"map of {len(nodes)} nodes, {len(points)} points: bit-identical to the reference")


def test_attaching_changes_nothing_else(mapped):
    """The twin without range data has byte-identical poses, constraints, searches and cloud_bytes_uploaded; only the store
    counts differ, by the returns' bytes."""
    _, a, b, records, steps = mapped
    for ia, ib, sa, sb in steps:
        assert (ia.node_index, ia.num_searched, ia.num_found, ia.optimized, ia.cloud_bytes_uploaded) == \
               (ib.node_index, ib.num_searched, ib.num_found, ib.optimized, ib.cloud_bytes_uploaded)
        assert bytes(ia.summary) == bytes(ib.summary)
        assert [(s[0], s[1], s[2].tobytes(), bytes(s[3])) for s in sa] == [(s[0], s[1], s[2].tobytes(), bytes(s[3])) for s in sb]
    assert sum(ia.optimized for ia, _, _, _ in steps) > 0 and sum(ia.num_found for ia, _, _, _ in steps) > 0
    for t in (0, 1):
        assert a.node_poses(t).tobytes() == b.node_poses(t).tobytes()
        assert a.submap_poses(t).tobytes() == b.submap_poses(t).tobytes()
        assert [x.tobytes() for x in a.optimization_poses(t)] == [x.tobytes() for x in b.optimization_poses(t)]
    assert [(c[0], c[1], c[2].tobytes(), c[3], c[4], c[5]) for c in a.constraints()] == \
           [(c[0], c[1], c[2].tobytes(), c[3], c[4], c[5]) for c in b.constraints()]
    extra = 12 * sum(len(r["returns"]) for r in records.values())
    assert a.store_bytes()[0] == b.store_bytes()[0] + extra
    assert a.store_usage()[0] == b.store_usage()[0] + extra
    assert b.range_data_map()[0].shape == (0, 3) and b.range_data_map()[1] == []


def store_rule(g):
    live, used, _ = g.store_usage()
    return used <= 2 * live or used - live < 4 << 20


def test_pure_localization_trims_and_compacts(mapped, recorded):  # noqa: F811
    """Trajectory 2 (two nodes carrying 700 k returns each) is finished under a trimmer: its nodes leave the map and the store
    is compacted. Then trajectory 0, and trajectory 1 under PureLocalizationTrimmer(1, 3), optimizing every 4 nodes: after
    every call the store rule holds and the map equals the reference on the live nodes, bit for bit."""
    import dliom
    ctx, nodes = recorded
    _, _, _, records, _ = mapped
    g = dliom.PoseGraph3D(ctx, options(optimize_every_n_nodes=4))
    n0 = [(t, i, n) for t, i, n in _ids(nodes) if t == 0]
    _, _, hg, lg, pose = n0[0][2]["ins"][0]
    big = np.tile(records[(0, 0)]["returns"], (1 + 700_000 // len(records[(0, 0)]["returns"]), 1))
    recs = dict(records)
    for j in range(2):
        g.add_node(2, 1.0 + j, n0[0][2]["local"], n0[0][2]["hi"], n0[0][2]["lo"], [(0, False, hg, lg, pose)])
        g.set_node_range_data(2, j, big)
        recs[(2, j)] = dict(local=n0[0][2]["local"], returns=big)
    live, used, _ = g.store_usage()
    assert live == used >= 2 * 12 * len(big)
    check_map(g, recs)
    g.add_pure_localization_trimmer(2, 3)
    g.finish_trajectory(2)
    assert g.ids(2) == [] and g.range_data_map([2])[1] == []
    live2, used2, _ = g.store_usage()
    assert live2 == used2 == 0      # compacted: nothing live was left
    g.add_pure_localization_trimmer(1, 3)
    checked = 0
    for t, i, n in _ids(nodes):
        info = g.add_node(t, n["time"], n["local"], n["hi"], n["lo"], n["ins"], n["matches"])
        g.set_node_range_data(t, info.node_index, records[(t, i)]["returns"])
        assert store_rule(g), g.store_usage()
        if g.last_trimmed():
            points, got = check_map(g, recs)
            assert {(x[0], x[1]) for x in got} == {(tt, ii) for tt in (0, 1) for ii in g.ids(tt)}
            checked += 1
    assert checked > 0
    g.finish_trajectory(1)
    assert store_rule(g) and g.ids(1) == []
    points, got = check_map(g, recs)
    assert [x[0] for x in got] == [0] * len(g.ids(0)) and len(got) == len(g.ids(0)) > 0
    live, used, _ = g.store_usage()
    print(f"pure localization: {checked} maps checked after trims; store after finish live {live} used {used}")
    g.close()


def state(g, trajectories=(0, 1)):
    """Everything a rejected call must leave as it was."""
    return ([g.node_poses(t).tobytes() for t in trajectories], [(g.ids(t), g.ids(t, 1)) for t in trajectories],
            [(c[0], c[1], c[2].tobytes(), c[5]) for c in g.constraints()], g.store_usage(), g.store_bytes(),
            [(x[0], x[1], x[2], x[3]) for x in g.range_data_map()[1]], g.range_data_map()[0].tobytes())


def test_edges_and_rejections(mapped, recorded):  # noqa: F811
    """An empty graph; a trajectory without attached nodes; a node with 0 returns; a subset of trajectories; a size query
    followed by a fill; every DL_ERR_ARG case, the graph unchanged afterwards."""
    import dliom
    ctx, nodes = recorded
    _, a, _, records, _ = mapped
    L = ctx.L
    g = dliom.PoseGraph3D(ctx, options())
    pts, got = g.range_data_map()
    assert pts.shape == (0, 3) and got == []
    dev, got = g.range_data_map(device=True)
    assert tuple(dev.shape) == (0, 3) and got == []
    recs = {}
    for t, i, n in _ids(nodes):
        g.add_node(t, n["time"], n["local"], n["hi"], n["lo"], n["ins"], n["matches"])
        if t == 0 and i < 6:      # trajectory 1 gets none; node (0, 2) has 0 returns
            r = records[(t, i)]["returns"][:0] if i == 2 else records[(t, i)]["returns"]
            g.set_node_range_data(t, i, r)
            recs[(t, i)] = dict(local=records[(t, i)]["local"], returns=r)
    g.run_final_optimization()
    points, got = check_map(g, recs)
    assert [(x[0], x[1]) for x in got] == [(0, i) for i in range(6)] and got[2][3] == 0 and got[3][2] == got[2][2]
    assert g.range_data_map([1])[1] == [] and g.range_data_map([])[1] == []
    # a subset of the mapped graph: trajectory 1's rows, rebased
    full, full_nodes = a.range_data_map()
    sub, sub_nodes = check_map(a, records, [1])
    first = next(x[2] for x in full_nodes if x[0] == 1)
    assert sub.tobytes() == full[first:].tobytes()
    assert [(x[1], x[2] + first, x[3]) for x in sub_nodes] == [(x[1], x[2], x[3]) for x in full_nodes if x[0] == 1]
    # a size query, then a fill; a capacity one short writes only the counts
    nn, npts = C.c_int32(-1), C.c_int64(-1)
    assert L.dl_range_data_map(g.h, 0, None, 0, None, C.byref(nn), 0, None, C.byref(npts)) == 0
    assert (nn.value, npts.value) == (6, len(points))
    out = np.full((npts.value, 3), np.nan, np.float32)
    table = (dliom.RangeDataMapNode * nn.value)()
    assert L.dl_range_data_map(g.h, 0, None, nn.value - 1, C.cast(table, C.c_void_p), C.byref(nn), npts.value,
                               out.ctypes.data, C.byref(npts)) == ERR_ARG
    assert (nn.value, npts.value) == (6, len(points)) and np.isnan(out).all() and table[0].num_points == 0
    assert L.dl_range_data_map(g.h, 0, None, nn.value, C.cast(table, C.c_void_p), C.byref(nn), npts.value - 1,
                               out.ctypes.data, C.byref(npts)) == ERR_ARG
    assert np.isnan(out).all()
    assert L.dl_range_data_map(g.h, 0, None, nn.value, C.cast(table, C.c_void_p), C.byref(nn), npts.value,
                               out.ctypes.data, C.byref(npts)) == 0
    assert out.tobytes() == points.tobytes() and [table[k].first_point for k in range(6)] == [x[2] for x in got]
    # rejections, the graph unchanged
    s0 = state(g)

    def refused(status):
        assert status == ERR_ARG and state(g) == s0

    r = records[(0, 7)]["returns"]
    refused(L.dl_range_data_map_set_node(g.h, 0, 99, r.ctypes.data, len(r)))        # unknown node
    refused(L.dl_range_data_map_set_node(g.h, 7, 0, r.ctypes.data, len(r)))         # unknown trajectory
    refused(L.dl_range_data_map_set_node(g.h, 0, 1, r.ctypes.data, len(r)))         # already has range data
    refused(L.dl_range_data_map_set_node(g.h, 0, 2, r.ctypes.data, len(r)))         # ... even with 0 returns
    refused(L.dl_range_data_map_set_node(g.h, 0, 7, r.ctypes.data, -1))             # num_returns < 0
    refused(L.dl_range_data_map_set_node(g.h, 0, 7, None, 5))                       # NULL returns
    ids = np.array([0, 0], np.int32)
    for entry in (L.dl_range_data_map, L.dl_range_data_map_dev):
        refused(entry(g.h, 2, ids.ctypes.data, 6, C.cast(table, C.c_void_p), C.byref(nn), npts.value, out.ctypes.data,
                      C.byref(npts)))                                               # repeated id
        refused(entry(g.h, 1, np.array([5], np.int32).ctypes.data, 0, None, C.byref(nn), 0, None, C.byref(npts)))  # unknown
        refused(entry(g.h, -1, ids.ctypes.data, 0, None, C.byref(nn), 0, None, C.byref(npts)))   # num_trajectories < 0
    with pytest.raises(dliom.DlError):
        g.range_data_map([0, 5])
    # a trimmed node
    g.trim_submap(0, 0)
    gone = [i for i in range(6) if i not in g.ids(0)]
    assert gone
    s0 = state(g)
    refused(L.dl_range_data_map_set_node(g.h, 0, gone[0], r.ctypes.data, len(r)))
    assert {x[1] for x in g.range_data_map()[1]} == set(range(6)) - set(gone)
    check_map(g, recs)
    g.close()


def test_map_over_two_gigabytes():
    """More than 2^31 output bytes (180 M points from six nodes of 30 M returns at random poses) through the _dev variant:
    every node boundary and a seeded sample of 200 000 points equal the reference bit for bit."""
    import dliom
    import torch
    ctx = dliom.Context(0)
    rng = np.random.default_rng(11)
    g = dliom.PoseGraph3D(ctx, options())
    hg, lg = dliom.Grid(ctx, 0.1), dliom.Grid(ctx, 0.45)
    for grid in (hg, lg):
        grid.set_cells([0], [0], [0], [1])
    cloud = rng.uniform(-1, 1, (100, 3)).astype(np.float32)
    per_node, num_nodes = 30_000_000, 6
    returns = rng.uniform(-100, 100, (per_node, 3)).astype(np.float32)
    locals_ = []
    for j in range(num_nodes):
        q = rng.normal(size=4)
        local = np.concatenate([rng.uniform(-200, 200, 3), q / np.linalg.norm(q)])
        g.add_node(0, float(j), local, cloud, cloud, [(0, False, hg, lg, pg.IDENTITY)])
        g.set_node_range_data(0, j, returns)
        locals_.append(local)
    assert g.store_usage()[0] >= 12 * per_node * num_nodes
    points, nodes = g.range_data_map(device=True)
    total = per_node * num_nodes
    assert tuple(points.shape) == (total, 3) and 12 * total > 2 ** 31
    poses = g.node_poses(0)
    assert [(x[1], x[2], x[3]) for x in nodes] == [(j, j * per_node, per_node) for j in range(num_nodes)]
    rows = np.sort(rng.integers(0, total, 200_000))
    for j in range(num_nodes):
        rows = np.concatenate([rows, [j * per_node, j * per_node + 1, (j + 1) * per_node - 2, (j + 1) * per_node - 1]])
    got = points[torch.from_numpy(rows).to(points.device)].cpu().numpy()
    node = rows // per_node
    want = np.empty((len(rows), 3), np.float32)
    for j in range(num_nodes):
        sel = node == j
        want[sel] = ref.node_points(locals_[j], poses[j], returns[rows[sel] - j * per_node])
    assert got.tobytes() == want.tobytes()
    del points
    g.close()
    ctx.close()


def test_cpp_example_writes_the_python_map(mapped, recorded, tmp_path):  # noqa: F811
    """host/example_range_data_map.cc replays the recorded drive with EnableRangeDataCache and writes a PCD byte-identical to
    write_pcd of the Python map of the same drive."""
    import dliom
    from test_range_data_map_reference import build_range_data_map_example
    ctx, nodes = recorded
    _, a, _, _, _ = mapped
    exe = build_range_data_map_example(tmp_path)
    drive = str(tmp_path / "drive.bin")
    write_drive(drive, ctx.pose_graph_builders, nodes, OPTIMIZE_EVERY, [])
    out = subprocess.run([exe, drive, str(tmp_path / "cpp.pcd")], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    points, got = a.range_data_map()
    dliom.write_pcd(str(tmp_path / "py.pcd"), points)
    assert out.stdout.split() == ["nodes", str(len(got)), "points", str(len(points))]
    assert open(tmp_path / "cpp.pcd", "rb").read() == open(tmp_path / "py.pcd", "rb").read()
    assert os.path.getsize(tmp_path / "cpp.pcd") > 12 * len(points) > 0
