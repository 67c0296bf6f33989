"""CPU checks of the map writer: the oracle pinned to the reference's TransformInterpolationBuffer tests and to an independent
scalar reading of the three moving-object-removal passes, the C-ABI's layouts and argument checks, the PCD writer."""
import ctypes
import math
import struct

import numpy as np
import pytest

import map_writer_oracle as mo

IDENTITY = (0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0)


def yaw_pose(t, angle):
    return tuple(t) + (math.cos(angle / 2), 0.0, 0.0, math.sin(angle / 2))


def test_reference_has():   # transform_interpolation_buffer_test.cc:29-44
    one = mo.Trajectory([50], [IDENTITY])
    assert not one.has(25) and one.has(50) and not one.has(75)
    two = mo.Trajectory([50, 100], [IDENTITY, IDENTITY])
    assert [two.has(t) for t in (25, 50, 75, 100, 125)] == [False, True, True, True, False]
    assert not mo.Trajectory([], []).has(50)


def test_reference_lookup():   # transform_interpolation_buffer_test.cc:46-63, IsNearly(..., 1e-6)
    end = mo.compose_d((10.0, 10.0, 10.0, 1.0, 0.0, 0.0, 0.0), yaw_pose((0, 0, 0), 2.0))
    got = mo.Trajectory([50, 100], [IDENTITY, end]).lookup(75)
    want = yaw_pose((5.0, 5.0, 5.0), 1.0)
    assert np.allclose(got, want, atol=1e-6)


def test_reference_lookup_single_transform():   # transform_interpolation_buffer_test.cc:65-71
    assert mo.Trajectory([75], [IDENTITY]).lookup(75) == IDENTITY


def test_lookup_exact_tick_and_repeated_times():
    a, b, c = yaw_pose((1, 2, 3), 0.1), yaw_pose((4, 5, 6), 0.2), yaw_pose((7, 8, 9), 0.3)
    tr = mo.Trajectory([10, 20, 20, 30], [a, b, c, a])
    assert tr.lookup(20) == b                       # lower_bound: the first of the equal times
    assert tr.lookup(10) == a and tr.lookup(30) == a
    mid = tr.lookup(25)                             # between the second 20 and 30
    assert np.allclose(mid[:3], (np.array(c[:3]) + a[:3]) / 2)
    with pytest.raises(ValueError):
        mo.Trajectory([20, 10], [a, b])


def test_lookup_takes_the_short_arc():
    q = yaw_pose((0, 0, 0), 0.4)
    neg = q[:3] + tuple(-v for v in q[3:])          # the same rotation with the opposite sign: d < 0 flips scale1
    got = mo.Trajectory([0, 10], [IDENTITY, neg]).lookup(5)
    assert np.allclose(np.abs(got[3:]), np.abs(yaw_pose((0, 0, 0), 0.2)[3:]), atol=1e-12)


def test_from_seconds_truncates():
    rows = np.array([[1, 0, 0, 1.5e-7], [1, 0, 0, -1.5e-7]], np.float32)
    tr = {0: mo.Trajectory([999, 1000, 1001], [yaw_pose((0, 0, 0), 0), yaw_pose((5, 0, 0), 0), yaw_pose((9, 0, 0), 0)])}
    pts, origin, dropped = mo.handle_message(tr, (1000, 0, 1, 0, IDENTITY), rows)
    assert dropped == 0 and pts[0, 0] == np.float32(10.0)       # 1.5 ticks -> 1: the node at 1001
    pts, origin, dropped = mo.handle_message(tr, (1000, 1, 1, 0, IDENTITY), rows)
    assert pts[0, 0] == np.float32(1.0)                          # -1.5 ticks -> -1: the node at 999


# ---- an independent scalar reading (one Python float32 value at a time) of HandleMessage's transform and the three passes
def r32(v):
    return struct.unpack("f", struct.pack("f", v))[0]


def scalar_apply(pose_f, p):
    tx, ty, tz, qw, qx, qy, qz = [float(v) for v in pose_f]
    x, y, z = [float(v) for v in p]
    uv = [r32(r32(qy * z) - r32(qz * y)), r32(r32(qz * x) - r32(qx * z)), r32(r32(qx * y) - r32(qy * x))]
    uv = [r32(u + u) for u in uv]
    c = [r32(r32(qy * uv[2]) - r32(qz * uv[1])), r32(r32(qz * uv[0]) - r32(qx * uv[2])), r32(r32(qx * uv[1]) - r32(qy * uv[0]))]
    v = [x, y, z]
    return [r32(r32(r32(v[k] + r32(qw * uv[k])) + c[k]) + t) for k, t in enumerate((tx, ty, tz))]


def scalar_round(v):   # lround: |v| + 0.5 is exact in double for a float32 v
    return int(math.copysign(math.floor(abs(v) + 0.5), v))


def scalar_cell(p, res):
    return tuple(scalar_round(r32(c / res)) for c in p)


def scalar_norm(d):
    return r32(math.sqrt(r32(r32(d[0] * d[0]) + r32(r32(d[1] * d[1]) + r32(d[2] * d[2])))))


def scalar_passes(batches, voxel_size):
    res = r32(voxel_size)
    hits, rays = {}, {}
    for pts, o in batches:
        for p in pts:
            c = scalar_cell(p, res)
            hits[c] = hits.get(c, 0) + 1
    for pts, o in batches:
        for p in pts:
            d = [r32(p[k] - o[k]) for k in range(3)]
            length = scalar_norm(d)
            x = 0.0
            while x < length:
                s = r32(x / length)
                c = scalar_cell([r32(o[k] + r32(s * d[k])) for k in range(3)], res)
                if hits.get(c, 0) > 0:
                    rays[c] = rays.get(c, 0) + 1
                x = r32(x + voxel_size)
    kept = [p for pts, o in batches for p in pts
            if rays.get(scalar_cell(p, res), 0) < 3.0 * hits.get(scalar_cell(p, res), 0)]
    return hits, rays, kept


def small_scene(seed, n_msgs=4, n_pts=40):
    rng = np.random.default_rng(seed)
    times = [0, 2_000_000, 4_000_000, 6_000_000]
    poses = [yaw_pose((0.5 * k, 0.1 * k, 0.0), 0.05 * k) for k in range(4)]
    trajs = {3: mo.Trajectory(times, poses)}
    rows, msgs, first = [], [], 0
    for m in range(n_msgs):
        # a wall at x = 4 seen from the sensor plus a few loose points, some repeated so that cells collect hits
        wall = np.stack([np.full(n_pts, 4.0), rng.uniform(-1, 1, n_pts), rng.uniform(0, 1, n_pts)], axis=1)
        wall[n_pts // 2:] = wall[:n_pts - n_pts // 2]
        t = np.zeros(n_pts) if m % 2 == 0 else np.repeat(rng.uniform(-0.05, 0.0, n_pts // 8), 8)[:n_pts]
        msgs.append((1_000_000 + 1_500_000 * m, first, n_pts, 3, (0.1, 0.0, 0.2, 1, 0, 0, 0)))
        first += n_pts
        rows.append(np.concatenate([wall, t[:, None]], axis=1).astype(np.float32))
    return trajs, msgs, np.concatenate(rows)


def test_oracle_matches_an_independent_scalar_reading():
    trajs, msgs, rows = small_scene(1)
    for voxel in (0.05, 0.2):
        got = mo.write_map(trajs, msgs, rows, voxel_size=voxel)
        batches = []
        for msg in msgs:
            stamp, first, n, traj, s2t = msg
            pts = []
            for row in rows[first:first + n]:
                tick = stamp + int(float(row[3]) * 1e7)
                if not trajs[traj].has(tick):
                    continue
                pose = np.array(mo.compose_d(trajs[traj].lookup(tick), s2t)).astype(np.float32)
                pts.append(scalar_apply(pose, row[:3]))
                origin = scalar_apply(pose, (0.0, 0.0, 0.0))
            if pts:
                batches.append((pts, origin))
        hits, rays, kept = scalar_passes(batches, voxel)
        cells = sorted(hits)
        assert [tuple(c) for c in got["cells"].tolist()] == cells
        assert got["hits"].tolist() == [hits[c] for c in cells]
        assert got["rays"].tolist() == [rays.get(c, 0) for c in cells]
        assert np.array_equal(got["points"], np.array(kept, np.float32).reshape(-1, 3))
        assert sum(got["rays"]) > 0 and got["dropped_moving"] >= 0


def test_oracle_drops_points_without_a_pose_and_gates_the_range():
    trajs, msgs, rows = small_scene(2)
    late = (99_000_000, 0, 8, 3, IDENTITY)           # after the trajectory: no batch
    got = mo.write_map(trajs, msgs + [late], rows, range_filter=(0.0, 4.2))
    assert got["dropped_no_pose"] == 8 and got["messages_without_batch"] == 1
    assert np.isnan(got["origins"][-1]).all()
    assert got["dropped_range"] > 0
    ranges = []
    for m, msg in enumerate(msgs):
        pts, origin, _ = mo.handle_message(trajs, msg, rows)
        ranges.append(mo.norm_f(*(pts - origin).T))
    r = np.concatenate(ranges).astype(np.float64)
    assert got["dropped_range"] == int((r > 4.2).sum())


def test_oracle_rejects_a_cell_beyond_the_grid_extent():
    trajs = {0: mo.Trajectory([0], [IDENTITY])}
    rows = np.array([[8192.6 * 0.05, 0, 0, 0]], np.float32)
    with pytest.raises(ValueError):
        mo.write_map(trajs, [(0, 0, 1, 0, IDENTITY)], rows, voxel_size=0.05)
    assert len(mo.write_map(trajs, [(0, 0, 1, 0, IDENTITY)], rows)["points"]) == 1


# ---- C-ABI surface without a device
def test_map_writer_layouts_match_header():
    import dliom
    assert ctypes.sizeof(dliom.MapWriterOptions) == 32
    assert ctypes.sizeof(dliom.MapMessage) == 3 * 8 + 8 + 7 * 8
    assert ctypes.sizeof(dliom.MapWriterInfo) == 8 + 7 * 8


def test_map_writer_argument_checks_without_a_writer():
    import dliom
    L = dliom.lib()
    out = ctypes.c_void_p()
    o = dliom.MapWriterOptions()
    assert L.dl_map_writer_create(None, ctypes.byref(o), ctypes.byref(out)) == -2
    assert L.dl_map_writer_add_trajectory(None, 0, 0, None, None) == -2
    n = ctypes.c_int64(0)
    assert L.dl_map_writer_process(None, 0, None, None, 0, None, ctypes.byref(n), None, None) == -2
    assert L.dl_map_writer_process_dev(None, 0, None, None, 0, None, ctypes.byref(n), None, None) == -2
    r = ctypes.c_int32(0)
    assert L.dl_map_writer_flush(None, ctypes.byref(r)) == -2
    assert L.dl_map_writer_voxels(None, 0, None, None, None, ctypes.byref(n)) == -2
    L.dl_map_writer_destroy(None)


def test_seconds_to_ticks_is_llround():
    import dliom
    t = np.array([0.0, 1.5e-7, -1.5e-7, 2.49e-7, 12.3456789, -0.25e-7])
    assert dliom.seconds_to_ticks(t).tolist() == [0, 2, -2, 2, 123456789, 0]


def test_pcd_writer_layout(tmp_path):
    import dliom
    pts = np.array([[1, 2, 3], [-4.5, 0.25, 1e-3]], np.float32)
    path = tmp_path / "points.pcd"
    dliom.write_pcd(str(path), pts)
    data = path.read_bytes()
    header = (b"# generated by Cartographer\nVERSION .7\nFIELDS x y z\nSIZE 4 4 4\nTYPE F F F\nCOUNT 1 1 1\n"
              b"WIDTH 000000000000002\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS 000000000000002\nDATA binary\n")
    assert data == header + pts.tobytes()


# ---- the C++ example (io::MapWriter + io::PcdWritingPointsProcessor)
def build_write_map_example(out_dir):
    """host/example_write_map.cc built with -Wall -Werror."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    host = os.path.join(root, "d-liom_b200", "host")
    exe = os.path.join(str(out_dir), "example_write_map")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", os.path.join(host, "example_write_map.cc"), "-o", exe,
                           "-L" + os.path.join(root, "d-liom_b200"), "-ldliom_b200", "-Wl,-rpath," + os.path.join(root, "d-liom_b200")])
    return exe


def write_map_input(path, trajectories, msgs, rows, range_filter=None, voxel_size=0.0):
    """The input file of example_write_map: trajectories {id: (ticks, poses7)}, msgs [(stamp, first_row, n, id, s2t7)]."""
    with open(path, "wb") as f:
        lo, hi = range_filter if range_filter is not None else (0.0, 0.0)
        f.write(struct.pack("<iddd", int(range_filter is not None), lo, hi, voxel_size))
        f.write(struct.pack("<i", len(trajectories)))
        for tid, (times, poses) in trajectories.items():
            f.write(struct.pack("<ii", tid, len(times)))
            f.write(np.asarray(times, "<i8").tobytes() + np.asarray(poses, "<f8").reshape(-1, 7).tobytes())
        f.write(struct.pack("<i", len(msgs)))
        for stamp, first, n, tid, s2t in msgs:
            f.write(struct.pack("<qi", stamp, tid) + np.asarray(s2t, "<f8").tobytes() + struct.pack("<i", n))
            f.write(np.ascontiguousarray(rows[first:first + n], "<f4").tobytes())


def test_cpp_write_map_example_compiles_and_fails_loudly_without_a_gpu(tmp_path):
    import subprocess
    import torch
    exe = build_write_map_example(tmp_path)
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    path = str(tmp_path / "input.bin")
    write_map_input(path, {0: ([0, 10], [IDENTITY, IDENTITY])}, [(5, 0, 1, 0, IDENTITY)], np.zeros((1, 4), np.float32))
    r = subprocess.run([exe, path, str(tmp_path / "points.pcd")], capture_output=True, text=True)
    assert r.returncode == 2 and "dliom error -1" in r.stderr
