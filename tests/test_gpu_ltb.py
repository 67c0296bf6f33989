"""mapping::LocalTrajectoryBuilder3D over the device path (dl_ltb_*; reference interface local_trajectory_builder_3d.h:81-113):
a synthetic drive fed sample by sample (200 Hz IMU, 10 Hz 16-beam scans). Every scan is checked against the oracle chain run on
the builder's OWN state and maps at that scan (its submap grids are exported and loaded into oracle grids), so the comparison
is per call and does not fork: pose / velocity / biases of the fused solve, the node's point clouds bit for bit, the device
histogram, the submap bookkeeping of ActiveSubmaps3D and the inserted grids cell for cell."""
import numpy as np
import pytest

import imu_synth
from helpers import apply_pose, pose_error

pytestmark = pytest.mark.gpu
NOISE = [3.99e-2, 1.56e-2, 6.4e-5, 3.6e-5]


def drive(n):
    import synth
    scene = synth.Scene(42)
    times = [2.0 + 0.1 * k for k in range(n)]
    return times, [synth.make_scan(scene, 16, t) for t in times]


def make_builder(ctx, orc, **kw):
    import dliom
    fo = dliom.FrontendOptions.from_oracle(orc.FrontEndOptions.defaults())
    return dliom.LocalTrajectoryBuilder(ctx, dliom.LtbOptions.defaults(fo, NOISE, imu_weight=0.7, **kw))


def oracle_grids(orc, hi, lo):
    ohi, olo = orc.Grid(0.1), orc.Grid(0.45)
    ohi.set_cells(*hi.export())
    olo.set_cells(*lo.export())
    return ohi, olo


def cells(export):
    return {(int(x), int(y), int(z)): int(v) for x, y, z, v in zip(*export)}


def test_builder_follows_the_oracle_chain_scan_by_scan(orc):
    import dliom
    ctx = dliom.Context(0)
    opts = orc.FrontEndOptions.defaults()
    times, scans = drive(12)
    b = make_builder(ctx, orc, num_range_data=5, max_time_seconds=0.05)   # 0.1 s between scans: the motion filter never drops
    b.set_initial_state(imu_synth.state(times[0] - 0.1))
    origin = np.zeros((1, 3), np.float32)
    last_t = None
    latch = None
    submap0_returns = []
    inserted = 0
    matching_index = 0
    for k, (t1, rows) in enumerate(zip(times, scans)):
        dt, acc, gyr = imu_synth.samples(t1 - 0.1, t1)
        ts = t1 - 0.1 + np.arange(len(dt)) / 200.0
        first = 0 if k == 0 else 1          # sample 0 of an interval is the last sample of the previous one
        iv_dt, iv_acc, iv_gyr = ([latch[0]] if latch else []), ([latch[1]] if latch else []), ([latch[2]] if latch else [])
        for j in range(first, len(dt)):
            b.add_imu_data(ts[j], acc[j], gyr[j])
            d = 1.0 / 500.0 if last_t is None else ts[j] - last_t
            last_t = ts[j]
            iv_dt.append(d); iv_acc.append(acc[j]); iv_gyr.append(gyr[j])
        latch = (iv_dt[-1], iv_acc[-1], iv_gyr[-1])
        state_i, init = b.state()
        assert init
        hi, lo, sp, nrd, fin = b.submap(matching_index)
        ohi, olo = oracle_grids(orc, hi, lo)
        xyzt = np.stack([rows["x"], rows["y"], rows["z"], rows["t"]], 1)
        r = b.add_range_data(t1, xyzt)
        assert r.has_result == 1 and r.inserted == 1 and r.scan.ok == 1
        secs, want, pred, ok, iters = orc.frontend_batch_imu(opts, [rows], origin, NOISE, [state_i], [(np.array(iv_dt), np.array(iv_acc), np.array(iv_gyr))],
                                                             sp, ohi, olo, 1, imu_weight=0.7)
        assert ok[0] == 1
        got = NavStateVec(r.state)
        dtn, drn = pose_error(got[:7], want[0][:7])
        assert dtn < 1e-6 and drn < 1e-7, (k, dtn, drn)
        assert np.allclose(got[7:], want[0][7:], atol=1e-6)
        assert np.allclose(np.array(r.local_pose[:]), got[:7], atol=0)
        assert r.scan.summary.num_iterations == iters[0]
        # the node's clouds: adaptive filter outputs of the returns in the tracking frame, bit for bit
        ing = orc.ingest_scan(opts, rows, origin, state_i[:7], pred[0][:7])
        pts = ing["returns_tracking"]
        hk, _ = orc.adaptive_voxel_filter(pts, opts.hi_max_length, opts.hi_min_num_points, opts.hi_max_range)
        lk, _ = orc.adaptive_voxel_filter(pts, opts.lo_max_length, opts.lo_min_num_points, opts.lo_max_range)
        assert np.array_equal(b.cloud(2).view(np.uint32), pts[hk].view(np.uint32))
        assert np.array_equal(b.cloud(3).view(np.uint32), pts[lk].view(np.uint32))
        assert (r.num_returns, r.num_high_resolution, r.num_low_resolution) == (len(pts), len(hk), len(lk))
        # range_data_in_local = opt_pose.cast<float>() * returns (float transform; compared to the double one to float accuracy)
        local = b.cloud(0)
        assert len(local) == len(pts) and np.abs(local - apply_pose(got[:7], pts.astype(np.float64))).max() < 2e-4
        assert len(b.cloud(1)) == r.num_misses
        # rotational histogram of the gravity-aligned returns (device atan2f: tolerance, not bits)
        aligned = apply_pose(np.concatenate([[0, 0, 0], got[3:7]]), pts.astype(np.float64)).astype(np.float32)
        wh = orc.compute_histogram(aligned, 120)
        gh = b.histogram()
        assert abs(gh.sum() - wh.sum()) <= 2e-3 * wh.sum() + 1e-3
        assert np.abs(gh - wh).sum() <= 0.02 * wh.sum() + 1e-3
        # ActiveSubmaps3D bookkeeping (submap_3d.cc:300-326)
        inserted += 1
        expect_insertion = [0] if inserted <= 5 else ([0, 1] if inserted <= 10 else [1, 2])
        assert [r.insertion_submap_index[i] for i in range(r.num_insertion_submaps)] == expect_insertion
        if inserted <= 10:
            submap0_returns.append((np.array(r.origin_in_local[:], np.float32), local.copy()))
        if inserted == 10:
            matching_index = 1          # submap 0 finished when submap 2 was added; submap 1 is the matching submap now
    assert b.num_submaps() == 3
    _, _, p0, n0, f0 = b.submap(0)
    _, _, p1, n1, f1 = b.submap(1)
    _, _, p2, n2, f2 = b.submap(2)
    assert (n0, f0, n1, f1, n2, f2) == (10, True, 7, False, 2, False)
    assert np.array_equal(p0, orc.IDENTITY_POSE) and np.linalg.norm(p1[:3]) > 0.3
    # submap 0 lives at the identity: its grids must equal the oracle inserter fed with the same ten range data
    ohi, olo = orc.Grid(0.1), orc.Grid(0.45)
    for o, local in submap0_returns:
        d = local - o
        r2 = (d[:, 0] * d[:, 0] + (d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])).astype(np.float32)
        ohi.insert_range_data(o, local[np.sqrt(r2).astype(np.float32) <= np.float32(20.0)])
        olo.insert_range_data(o, local)
    hi0, lo0, *_ = b.submap(0)
    assert cells(hi0.export()) == cells(ohi.export()) and cells(lo0.export()) == cells(olo.export())
    b.close()
    ctx.close()


def NavStateVec(s):
    return np.array(list(s.p) + list(s.q) + list(s.v) + list(s.ba) + list(s.bg))


def test_builder_initialisation_motion_filter_and_drops(orc):
    """InitializeStatic from the buffered IMU (LTB:203-229), the motion filter (motion_filter.cc:37-57), no-IMU and empty scans."""
    import dliom
    ctx = dliom.Context(0)
    times, scans = drive(4)
    xyzt = [np.stack([r["x"], r["y"], r["z"], r["t"]], 1) for r in scans]
    b = make_builder(ctx, orc, frames_for_static_initialization=1, max_time_seconds=5.0, max_distance_meters=50.0, max_angle_radians=3.0)
    # a tilted, resting IMU: specific force = R^T (0, 0, 9.8) + bias_a; rate = bias_g
    tilt = imu_synth.state(0.0)
    roll = 0.05
    Rt_g = np.array([0.0, 9.8 * np.sin(roll), 9.8 * np.cos(roll)])
    for j in range(200):
        b.add_imu_data(j / 200.0, Rt_g, [1e-3, -2e-3, 5e-4])
    for k in range(3):     # LTB:376: `accumulated_frame_num++ > frames` -> the third scan initialises, none of them is matched
        r = b.add_range_data(1.0 + 0.1 * k, xyzt[0])
        assert r.has_result == 0
    st, init = b.state()
    assert init
    # gravity alignment: R takes the measured up direction (0, sin, cos) to +z -> +0.05 about x; biases: gyro mean, accelerometer ~ 0
    assert np.allclose(st[3:7], [np.cos(roll / 2), np.sin(roll / 2), 0, 0], atol=1e-9)
    assert np.allclose(st[13:16], [1e-3, -2e-3, 5e-4], atol=1e-12) and np.abs(st[10:13]).max() < 1e-9
    assert np.allclose(st[:3], 0) and np.allclose(st[7:10], 0)
    # no IMU since the last scan -> nullptr (predicted_states_.empty(), LTB:426); an empty scan -> nullptr
    assert b.add_range_data(1.3, xyzt[0]).has_result == 0
    assert b.add_range_data(1.4, np.zeros((0, 4), np.float32)).has_result == 0
    # motion filter: with generous thresholds only the first matched scan is inserted
    b2 = make_builder(ctx, orc, max_time_seconds=5.0, max_distance_meters=50.0, max_angle_radians=3.0)
    b2.set_initial_state(imu_synth.state(times[0] - 0.1))
    flags = []
    last = None
    for k, t1 in enumerate(times):
        dt, acc, gyr = imu_synth.samples(t1 - 0.1, t1)
        for j in range(0 if k == 0 else 1, len(dt)):
            b2.add_imu_data(t1 - 0.1 + j / 200.0, acc[j], gyr[j])
        r = b2.add_range_data(t1, xyzt[k])
        assert r.has_result == 1
        flags.append(r.inserted)
    assert flags == [1, 0, 0, 0]
    _, _, _, n0, _ = b2.submap(0)
    assert n0 == 1 and b2.num_submaps() == 1
    b.close(); b2.close(); ctx.close()


def _synchronize(prior, secondary_queue):
    """Python twin of RangeDataSynchronizer::AddRangeData for the prior sensor (range_data_synchronizer.cc:43-109):
    prior = (time, xyzt float32 [n,4]); secondary_queue = list of (time, xyzt). Returns RangeMeasurement rows + number merged."""
    from synth import RANGE_DTYPE
    t_end, a = prior
    start = t_end + float(a[0, 3])
    while secondary_queue and secondary_queue[0][0] < start:
        secondary_queue.pop(0)
    rows = np.zeros(len(a), RANGE_DTYPE)
    rows["x"], rows["y"], rows["z"], rows["t"] = a[:, 0], a[:, 1], a[:, 2], a[:, 3]
    if not secondary_queue:
        return rows, 0
    tb, bpts = secondary_queue[0]
    if tb + float(bpts[0, 3]) > t_end:
        return rows, 0
    tt = tb + bpts[:, 3].astype(np.float64)
    inside = np.nonzero((tt >= start) & (tt <= t_end))[0]
    i_start = int(inside[0])
    after = np.nonzero((np.arange(len(tt)) > i_start) & (tt > t_end))[0]
    i_end = int(after[0]) - 1 if len(after) else len(tt) - 1
    sel = bpts[i_start:i_end + 1]
    extra = np.zeros(len(sel), RANGE_DTYPE)
    extra["x"], extra["y"], extra["z"] = sel[:, 0], sel[:, 1], sel[:, 2]
    extra["t"] = (sel[:, 3].astype(np.float64) + tb - t_end).astype(np.float32)
    extra["origin_index"] = 1
    merged = np.concatenate([rows, extra])
    return merged[np.argsort(merged["t"], kind="stable")], len(sel)


def test_cpp_shim_replays_a_two_lidar_drive(orc, tmp_path):
    """host/dliom_b200.hpp: mapping::LocalTrajectoryBuilder3D + RangeDataSynchronizer (two LiDARs, the kaist / viral set-up) driven
    by a C++ program from a recorded event file; the same events through the Python binding with a Python restatement of the
    synchroniser must give the same poses to the last bit (same C-ABI object underneath)."""
    import os
    import struct
    import subprocess
    import dliom
    import synth
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    host = os.path.join(root, "d-liom_b200", "host")
    exe = str(tmp_path / "example_trajectory")
    subprocess.check_call(["g++", "-std=c++17", "-O1", os.path.join(host, "example_trajectory.cc"), "-o", exe,
                           "-L" + os.path.join(root, "d-liom_b200"), "-ldliom_b200", "-Wl,-rpath," + os.path.join(root, "d-liom_b200")])
    scene = synth.Scene(42)
    n = 8
    times = [2.0 + 0.1 * k for k in range(n)]
    init = imu_synth.state(times[0] - 0.1)
    events = []
    for k, t1 in enumerate(times):
        dt, acc, gyr = imu_synth.samples(t1 - 0.1, t1)
        for j in range(0 if k == 0 else 1, len(dt)):
            events.append(("imu", t1 - 0.1 + j / 200.0, acc[j], gyr[j]))
        for kind, t in ((2, t1 - 0.03), (1, t1)):      # the secondary sweep ends 30 ms before the prior one
            r = synth.make_scan(scene, 16, t)
            events.append(("range", kind, t, np.stack([r["x"], r["y"], r["z"], r["t"]], 1).astype(np.float32)))
    path = str(tmp_path / "drive.bin")
    with open(path, "wb") as f:
        f.write(dliom.NavState.from16(init))
        f.write(struct.pack("<i", len(events)))
        for e in events:
            if e[0] == "imu":
                f.write(struct.pack("<id", 0, e[1]) + np.asarray(e[2], np.float64).tobytes() + np.asarray(e[3], np.float64).tobytes())
            else:
                f.write(struct.pack("<id", e[1], e[2]) + np.zeros(3, np.float32).tobytes() + struct.pack("<i", len(e[3])) + e[3].tobytes())
    out = subprocess.run([exe, path], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = out.stdout.strip().splitlines()
    results = [l.split() for l in lines if l.startswith("result")]
    assert len([l for l in lines if l.startswith("none")]) == n      # the secondary clouds are only queued
    assert len(results) == n
    # the Python twin
    ctx = dliom.Context(0)
    fo = dliom.FrontendOptions.from_oracle(orc.FrontEndOptions.defaults())
    b = dliom.LocalTrajectoryBuilder(ctx, dliom.LtbOptions.defaults(fo, NOISE, imu_weight=0.7, num_range_data=5, max_time_seconds=0.05))
    b.set_initial_state(init)
    queue, k = [], 0
    for e in events:
        if e[0] == "imu":
            b.add_imu_data(e[1], e[2], e[3])
        elif e[1] == 2:
            queue.append((e[2], e[3]))
        else:
            rows, merged = _synchronize((e[2], e[3]), queue)
            assert merged > 0 and rows["t"].min() >= -0.1 and rows["t"].max() == 0.0
            r = b.add_synchronized_range_data(e[2], rows, np.zeros((2, 3), np.float32))
            got = results[k]
            assert r.has_result == 1 and float(got[1]) == pytest.approx(e[2])
            assert [float(v) for v in got[2:9]] == list(r.local_pose)          # printed with %.17g: exact round trip
            assert int(got[9]) == r.inserted == 1 and int(got[10]) == r.num_returns and int(got[11]) == b.num_submaps()
            assert (int(got[12]), int(got[13]), int(got[14])) == (r.num_high_resolution, r.num_low_resolution, r.num_insertion_submaps)
            k += 1
    assert b.num_submaps() == 2
    b.close()
    ctx.close()


def test_two_stage_mode_follows_the_reference_chain(orc):
    """dl_ltb_options.two_stage = 1: predict -> plain CeresScanMatcher3D::Match from the prediction (LTB:535-542) -> window update
    with the matched pose as a prior (LTB:555, :693-863, here dl_window_optimize_batch). The oracle runs the same chain with its
    own smoother state (estimate + carried information); the maps it matches against are the builder's own, exported per scan."""
    import dliom
    ctx = dliom.Context(0)
    opts = orc.FrontEndOptions.defaults()
    times, scans = drive(7)
    b = make_builder(ctx, orc, num_range_data=50, max_time_seconds=0.05, two_stage=1, ceres_pose_noise_t=0.02, ceres_pose_noise_r=0.01,
                     prior_pose_noise=0.01, prior_velocity_noise=0.2, prior_bias_noise=0.01)
    state = imu_synth.state(times[0] - 0.1)
    b.set_initial_state(state)
    info = np.diag([1 / 0.01 ** 2] * 6 + [1 / 0.2 ** 2] * 3 + [1 / 0.01 ** 2] * 6)
    origin = np.zeros((1, 3), np.float32)
    last_t, latch = None, None
    for k, (t1, rows) in enumerate(zip(times, scans)):
        dt, acc, gyr = imu_synth.samples(t1 - 0.1, t1)
        ts = t1 - 0.1 + np.arange(len(dt)) / 200.0
        iv_dt, iv_acc, iv_gyr = ([latch[0]] if latch else []), ([latch[1]] if latch else []), ([latch[2]] if latch else [])
        for j in range(0 if k == 0 else 1, len(dt)):
            b.add_imu_data(ts[j], acc[j], gyr[j])
            d = 1.0 / 500.0 if last_t is None else ts[j] - last_t
            last_t = ts[j]
            iv_dt.append(d); iv_acc.append(acc[j]); iv_gyr.append(gyr[j])
        latch = (iv_dt[-1], iv_acc[-1], iv_gyr[-1])
        hi, lo, sp, _, _ = b.submap(0)
        ohi, olo = oracle_grids(orc, hi, lo)
        xyzt = np.stack([rows["x"], rows["y"], rows["z"], rows["t"]], 1)
        r = b.add_range_data(t1, xyzt)
        assert r.has_result == 1 and r.scan.ok == 1
        # the oracle's chain from ITS state
        m = orc.imu_preintegrate(NOISE, state[10:13], state[13:16], np.array(iv_dt), np.array(iv_acc), np.array(iv_gyr))
        pred = orc.imu_predict(state, m)
        _, poses, ok = orc.frontend_batch(opts, [rows], origin, [state[:7]], [pred[:7]], sp, ohi, olo, 1)
        assert ok[0] == 1
        dtm, drm = pose_error(np.array(r.scan.pose_estimate_local[:]), poses[0])
        assert dtm < 1e-6 and drm < 1e-7                                   # stage one: the plain match
        _, state, info, ws = orc.window_optimize(state, info, m, poses[0], sigma_t=0.02, sigma_r=0.01, imu_weight=0.7, initial_j=pred)
        got = NavStateVec(r.state)
        dtn, drn = pose_error(got[:7], state[:7])
        assert dtn < 2e-6 and drn < 1e-6, (k, dtn, drn)                      # stage two: the window
        assert np.abs(got[7:] - state[7:]).max() < 1e-5
        # the window moves the pose only a little away from the matcher (sigma 2 cm / 0.01 rad against a good prediction)
        assert pose_error(got[:7], poses[0])[0] < 0.05
    b.close()
    ctx.close()
