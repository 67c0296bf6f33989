"""The map writer on the device (dl_map_writer_*) against the CPU oracle (tests/map_writer_oracle.py): trajectory lookup and
transform, range filter, moving-object removal on the synthetic street with a transient box, argument errors, determinism and
the device-buffer entry point. Points, origins, drop counts and the cell table must be bit-identical."""
import numpy as np
import pytest

import map_writer_oracle as mo

pytestmark = pytest.mark.gpu

IDENTITY = (0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0)


def random_pose(rng, scale=20.0):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    return tuple(rng.uniform(-scale, scale, 3)) + tuple(q)


def random_case(seed, n_msgs=24, n_rows=3000):
    """Random trajectories (repeated node times included) and messages with all-zero or per-point times, some of them partly or
    wholly outside their trajectory's span, some stamped exactly on a node."""
    rng = np.random.default_rng(seed)
    trajs = {}
    for tid in (0, 7):
        times = np.cumsum(rng.integers(0, 3_000_000, 30))
        times[5] = times[4]                                   # a repeated node time
        poses = [random_pose(rng) for _ in times]
        poses[10] = poses[9][:3] + tuple(-v for v in poses[9][3:])   # the same rotation with the opposite sign
        trajs[tid] = (times.astype(np.int64), np.array(poses))
    rows, msgs, first = [], [], 0
    for m in range(n_msgs):
        tid = (0, 7)[m % 2]
        times = trajs[tid][0]
        n = int(rng.integers(1, n_rows))
        pts = rng.uniform(-30, 30, (n, 3))
        if m % 3 == 0:
            t = np.zeros(n)
        else:
            t = np.sort(np.repeat(rng.uniform(-0.1, 0.0, n // 16 + 1), 16)[:n])
        stamp = int(rng.integers(times[0] - 500_000, times[-1] + 500_000))
        if m % 5 == 0:
            stamp = int(times[int(rng.integers(0, len(times)))])   # exact node tick for t = 0 rows
        if m == 7:
            stamp = int(times[-1]) + 2_000_000                      # wholly after the span: no batch
        msgs.append((stamp, first, n, tid, random_pose(rng, 1.0)))
        rows.append(np.concatenate([pts, t[:, None]], 1).astype(np.float32))
        first += n
    msgs.append((int(trajs[0][0][3]), first, 0, 0, IDENTITY))       # an empty message
    return trajs, msgs, np.concatenate(rows)


def oracle_trajs(trajs):
    return {k: mo.Trajectory(t, p) for k, (t, p) in trajs.items()}


def make_writer(ctx, trajs, **kw):
    import dliom
    w = dliom.MapWriter(ctx, **kw)
    for k, (t, p) in trajs.items():
        w.add_trajectory(k, t, p)
    return w


def assert_same(got_pts, got_origins, info, want):
    assert got_pts.tobytes() == np.ascontiguousarray(want["points"], np.float32).tobytes()
    assert got_origins.tobytes() == want["origins"].tobytes()      # NaN rows for messages without a batch, bit for bit
    for k in ("dropped_no_pose", "dropped_range", "dropped_moving", "messages_without_batch"):
        assert info[k] == want[k], k


@pytest.fixture(scope="module")
def ctx():
    import dliom
    return dliom.Context(0)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_lookup_and_transform_match_the_oracle(ctx, seed):
    trajs, msgs, rows = random_case(seed)
    want = mo.write_map(oracle_trajs(trajs), msgs, rows)
    assert want["dropped_no_pose"] > 0 and want["messages_without_batch"] >= 2 and len(want["points"]) > 0
    pts, origins, info = make_writer(ctx, trajs).write_map(msgs, rows)
    assert info["final_pass"] == 1 and info["num_rows"] == len(rows)
    assert_same(pts, origins, info, want)


def test_range_filter_matches_the_oracle_on_its_bounds(ctx):
    trajs, msgs, rows = random_case(4)
    ot = oracle_trajs(trajs)
    ranges = []
    for msg in msgs:
        p, o, _ = mo.handle_message(ot, msg, rows)
        if o is not None:
            ranges.append(mo.norm_f(*(p - o).T))
    r = np.sort(np.concatenate(ranges).astype(np.float64))
    bounds = (float(r[len(r) // 4]), float(r[3 * len(r) // 4]))     # exactly some points' ranges: kept (inclusive)
    want = mo.write_map(ot, msgs, rows, range_filter=bounds)
    assert want["dropped_range"] > 0
    pts, origins, info = make_writer(ctx, trajs, range_filter=bounds).write_map(msgs, rows)
    assert_same(pts, origins, info, want)
    assert np.isin(bounds, r).all()


# ---- the synthetic street with a box standing in the corridor during the first scans only
BOX_LO, BOX_HI = np.array([14.0, -1.0, -1.8]), np.array([16.0, 1.0, 0.2])


def street(num_scans=16, transient_scans=5, beams=16):
    import synth
    scene, with_box = synth.Scene(), synth.Scene()
    with_box.box_lo = np.vstack([with_box.box_lo, BOX_LO])
    with_box.box_hi = np.vstack([with_box.box_hi, BOX_HI])
    node_t = np.arange(0.0, 0.1 * (num_scans + 1) + 1e-9, 0.02)
    trajs = {0: (np.round(node_t * 1e7).astype(np.int64), np.array([synth.pose7(t) for t in node_t]))}
    rows, msgs, first = [], [], 0
    for k in range(num_scans):
        end = 0.1 * (k + 1)
        r = synth.make_scan(with_box if k < transient_scans else scene, beams, end)
        xyzt = np.stack([r["x"], r["y"], r["z"], r["t"]], 1).astype(np.float32)
        if k % 4 == 3:
            xyzt[:, 3] = 0.0          # the fork's RsLiDAR conversion: one time per message
        msgs.append((int(round(end * 1e7)), first, len(xyzt), 0, IDENTITY))
        rows.append(xyzt)
        first += len(xyzt)
    return trajs, msgs, np.concatenate(rows)


def test_moving_object_removal_matches_the_oracle_on_the_street(ctx):
    trajs, msgs, rows = street()
    voxel, bounds = 0.2, (1.0, 40.0)
    want = mo.write_map(oracle_trajs(trajs), msgs, rows, range_filter=bounds, voxel_size=voxel)
    w = make_writer(ctx, trajs, range_filter=bounds, outlier_voxel_size=voxel)
    infos, restarts = [], []
    while True:
        pts, origins, info = w.process(msgs, rows)
        infos.append(info)
        if info["pass_"] == 1:
            cells, hits, rays = w.voxels()
            assert cells.tolist() == want["cells"].tolist() and hits.tolist() == want["hits"].tolist()
            assert rays.tolist() == want["rays"].tolist()
            assert info["num_samples"] == want["num_samples"]
        restarts.append(w.flush())
        if not restarts[-1]:
            break
    assert restarts == [True, True, False] and [i["pass_"] for i in infos] == [0, 1, 2]
    assert infos[0]["num_points_out"] == 0 and infos[1]["num_points_out"] == 0
    assert_same(pts, origins, infos[2], want)
    # the box's points of the first scans: most of them removed, while most of the map stays
    inside = lambda p: ((p > BOX_LO - 0.05) & (p < BOX_HI + 0.05)).all(1)
    before = mo.write_map(oracle_trajs(trajs), msgs, rows, range_filter=bounds)["points"]
    n_box_in, n_box_out = int(inside(before).sum()), int(inside(pts).sum())
    print(f"transient box: {n_box_in} points before, {n_box_out} after; map {len(before)} -> {len(pts)}")
    assert n_box_in > 200 and n_box_out < 0.5 * n_box_in
    assert len(pts) > 0.7 * len(before)
    with pytest.raises(Exception):
        w.process(msgs, rows)                       # after the final flush


def test_errors_leave_the_writer_unchanged(ctx):
    import dliom
    trajs, msgs, rows = street(num_scans=4, transient_scans=0)
    w = make_writer(ctx, trajs, outlier_voxel_size=0.05)
    with pytest.raises(dliom.DlError) as e:
        w.add_trajectory(0, trajs[0][0], trajs[0][1])                                  # added twice
    assert e.value.status == -2
    with pytest.raises(dliom.DlError):
        w.add_trajectory(1, [5, 4], [IDENTITY, IDENTITY])                              # times decrease
    far = rows.copy()
    far[msgs[1][1] + 3, :3] = (500.0, 0.0, 0.0)                                        # 10 000 cells of 5 cm: beyond +-8192
    bad = [
        [(msgs[0][0], 0, 10, 9, IDENTITY)],                                            # unknown trajectory
        [(msgs[0][0], len(rows) - 5, 10, 0, IDENTITY)],                                # rows out of range
        [(msgs[0][0], -1, 10, 0, IDENTITY)],
    ]
    for b in bad:
        with pytest.raises(dliom.DlError) as e:
            w.process(b, rows)
        assert e.value.status == -2
    shifted = (1000.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0)    # points near the map origin seen from a sensor 1 km away
    near = np.array([[-999.9, 0.0, 0.0, 0.0]], np.float32)
    with pytest.raises(dliom.DlError) as e:
        w.process([(msgs[0][0], 0, 1, 0, shifted)], near)
    assert e.value.status == -2 and "origin" in str(e.value)
    with pytest.raises(ValueError):
        mo.write_map(oracle_trajs(trajs), [(msgs[0][0], 0, 1, 0, shifted)], near, voxel_size=0.05)
    with pytest.raises(dliom.DlError) as e:
        w.process(msgs, far)
    assert e.value.status == -2 and "extent" in str(e.value)
    assert len(w.voxels()[0]) == 0
    ref = make_writer(ctx, trajs, outlier_voxel_size=0.05)
    out_w, out_ref = [], []
    for writer, out in ((w, out_w), (ref, out_ref)):
        while True:
            out.append(writer.process(msgs, rows))
            if writer.flush() is False:
                break
    assert out_w[-1][0].tobytes() == out_ref[-1][0].tobytes()
    with pytest.raises(dliom.DlError):
        w.flush()
    fresh = make_writer(ctx, trajs)
    fresh.process(msgs[:1], rows)
    with pytest.raises(dliom.DlError):
        fresh.add_trajectory(3, [0], [IDENTITY])                                       # after processing began


def test_repeat_runs_and_device_buffers_agree_bit_for_bit(ctx):
    import torch
    trajs, msgs, rows = street(num_scans=8, transient_scans=3)
    kw = dict(range_filter=(1.0, 60.0), outlier_voxel_size=0.1)
    a = make_writer(ctx, trajs, **kw).write_map(msgs, rows)
    b = make_writer(ctx, trajs, **kw).write_map(msgs, rows)
    assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()
    w = make_writer(ctx, trajs, **kw)
    rows_dev = torch.from_numpy(rows).cuda()
    out_dev = torch.zeros((len(rows), 3), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    while True:
        n, origins, info = w.process_dev(msgs, rows_dev.data_ptr(), len(rows), out_dev.data_ptr())
        if not w.flush():
            break
    ctx.synchronize()
    assert n == len(a[0])
    assert out_dev[:n].cpu().numpy().tobytes() == a[0].tobytes() and origins.tobytes() == a[1].tobytes()
    assert info == a[2]


def test_cpp_example_writes_the_same_pcd_bytes(ctx, tmp_path):
    """host/example_write_map.cc (io::MapWriter + io::PcdWritingPointsProcessor) writes the same points.pcd, byte for byte, as
    the Python writer over dliom.MapWriter on the same input."""
    import subprocess
    import dliom
    from test_map_writer_oracle import build_write_map_example, write_map_input
    trajs, msgs, rows = street(num_scans=8, transient_scans=3)
    kw = dict(range_filter=(1.0, 40.0), outlier_voxel_size=0.2)
    pts = make_writer(ctx, trajs, **kw).write_map(msgs, rows)[0]
    want = tmp_path / "want.pcd"
    dliom.write_pcd(str(want), pts)
    exe = build_write_map_example(tmp_path)
    path = str(tmp_path / "input.bin")
    write_map_input(path, trajs, msgs, rows, range_filter=kw["range_filter"], voxel_size=kw["outlier_voxel_size"])
    got = tmp_path / "points.pcd"
    r = subprocess.run([exe, path, str(got)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.strip() == f"points {len(pts)}" and len(pts) > 0
    assert got.read_bytes() == want.read_bytes()


# ---- end to end: two trajectories through dl_ltb and PoseGraph3D, then their maps (a copy of test_gpu_pose_graph3d.py's drive)
NOISE = [3.99e-2, 1.56e-2, 6.4e-5, 3.6e-5]
MATCH_PERTURBATION = (0.3, -0.2, 0.01)
NUM_SCANS = 24


def drive(ctx, offset):
    """One trajectory through a LocalTrajectoryBuilder -> (builder, [node records with the node's scan rows])."""
    import dliom
    import imu_synth
    import orc
    import pose_graph3d_oracle as pg
    import synth
    scene = synth.Scene(42)
    fo = dliom.FrontendOptions.from_oracle(orc.FrontEndOptions.defaults())
    b = dliom.LocalTrajectoryBuilder(ctx, dliom.LtbOptions.defaults(fo, NOISE, imu_weight=0.7, num_range_data=3,
                                                                     max_time_seconds=0.05))
    times = [2.0 + 0.1 * k for k in range(NUM_SCANS)]
    s16 = imu_synth.state(times[0] - 0.1)
    inv = pg.inverse(offset)
    b.set_initial_state(np.concatenate([pg.compose(inv, s16[:7]), pg.rotate(inv[3:], s16[7:10]), s16[10:]]))
    nodes = []
    for k, t1 in enumerate(times):
        dt, acc, gyr = imu_synth.samples(t1 - 0.1, t1)
        ts = t1 - 0.1 + np.arange(len(dt)) / 200.0
        for j in range(0 if k == 0 else 1, len(dt)):
            b.add_imu_data(ts[j], acc[j], gyr[j])
        rows = synth.make_scan(scene, 16, t1)
        r = b.add_synchronized_range_data(t1, rows, np.zeros((1, 3), np.float32))
        assert r.has_result == 1 and r.inserted == 1
        ins = []
        for i in range(r.num_insertion_submaps):
            hg, lg, pose, _, fin = b.submap(r.insertion_submap_index[i])
            ins.append((r.insertion_submap_index[i], fin, hg, lg, pose))
        nodes.append(dict(time=t1, local=np.array(r.local_pose[:]), hi=b.cloud(2), lo=b.cloud(3), ins=ins,
                          rows=np.stack([rows["x"], rows["y"], rows["z"], rows["t"]], 1).astype(np.float32)))
    return b, nodes


def voxel_set(points, size=0.2):
    return set(map(tuple, np.floor(np.asarray(points, np.float64) / size + 0.5).astype(np.int64).tolist()))


def test_end_to_end_optimized_poses_align_the_maps(ctx):
    """Trajectory 1's local frame is 4 m / -3 m / 5 degrees off trajectory 0's. Written with the pose graph's optimized node poses,
    its map overlaps trajectory 0's map far more, at 0.2 m voxels, than written with its uncorrected local poses."""
    import dliom
    import pose_graph3d_oracle as pg
    offset = np.concatenate([[4.0, -3.0, 0.0], pg.yaw_quaternion(np.deg2rad(5.0))])
    b0, n0 = drive(ctx, pg.IDENTITY)
    b1, n1 = drive(ctx, offset)
    local0 = {i: p for n in n0 for i, _, _, _, p in n["ins"]}
    g = dliom.PoseGraph3D(ctx, dliom.PoseGraph3DOptions.defaults(optimize_every_n_nodes=0, every_nodes_to_find_constraint=2,
                                                                min_score=0.3, min_low_resolution_score=0.3))
    for tid, nodes in ((0, n0), (1, n1)):
        for n in nodes:
            idx, fin, _, _, pose = n["ins"][0]
            matches = []
            if tid == 1 and fin:
                x, y, th = pg.match_from_truth(pose, local0[idx], offset, pg.IDENTITY)
                matches = [(0, idx, x + MATCH_PERTURBATION[0], y + MATCH_PERTURBATION[1], th + MATCH_PERTURBATION[2])]
            g.add_node(tid, n["time"], n["local"], n["hi"], n["lo"], n["ins"], matches)
    g.run_final_optimization()

    def messages(tid, nodes):
        msgs, rows, first = [], [], 0
        for n in nodes:
            msgs.append((int(dliom.seconds_to_ticks(n["time"])), first, len(n["rows"]), tid, IDENTITY))
            rows.append(n["rows"])
            first += len(n["rows"])
        return msgs, np.concatenate(rows)

    def write(tid, nodes, poses=None):
        w = dliom.MapWriter(ctx, range_filter=(1.0, 40.0))
        times = [n["time"] for n in nodes]
        if poses is None:
            w.add_pose_graph_trajectory(g, tid, times)
        else:
            w.add_trajectory(tid, dliom.seconds_to_ticks(times), poses)
        msgs, rows = messages(tid, nodes)
        pts, _, info = w.write_map(msgs, rows)
        want = mo.write_map({tid: mo.Trajectory(dliom.seconds_to_ticks(times), g.node_poses(tid) if poses is None else poses)},
                            msgs, rows, range_filter=(1.0, 40.0))
        assert pts.tobytes() == want["points"].tobytes()
        return pts

    map0 = voxel_set(write(0, n0))
    optimized = voxel_set(write(1, n1))
    uncorrected = voxel_set(write(1, n1, np.array([n["local"] for n in n1])))
    overlap_opt = len(optimized & map0) / len(optimized)
    overlap_unc = len(uncorrected & map0) / len(uncorrected)
    print(f"0.2 m voxel overlap with trajectory 0's map: optimized {overlap_opt:.3f}, uncorrected {overlap_unc:.3f}")
    assert overlap_opt > 0.8 and overlap_unc < 0.4    # measured on an H100: 0.916 and 0.191
    b0.close()
    b1.close()

