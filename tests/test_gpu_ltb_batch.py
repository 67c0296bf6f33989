"""dl_ltb_add_range_data_batch: several LocalTrajectoryBuilder3D objects advanced in one call. Every check runs the same inputs
through a second set of builders, on a context of their own, one dl_ltb_add_synchronized_range_data call at a time, and asks
for byte equality: the matching results, the node clouds, the histograms, the states, the submap bookkeeping and, at the
end, every grid cell."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import imu_synth

NOISE = [3.99e-2, 1.56e-2, 6.4e-5, 3.6e-5]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DL_OK, DL_ERR_ARG = 0, -2   # dl_status


def make_options(orc, **kw):
    import dliom
    fo = dliom.FrontendOptions.from_oracle(orc.FrontEndOptions.defaults())
    kw.setdefault("max_time_seconds", 0.05)   # 0.1 s between scans: the motion filter never holds a scan back
    return dliom.LtbOptions.defaults(fo, NOISE, imu_weight=0.7, **kw)


class Trajectory:
    """One synthetic drive, started at its own time: 200 Hz IMU and 10 Hz 16-beam scans of the shared scene."""

    def __init__(self, scene, t0, beams=16):
        self.scene, self.t0, self.beams = scene, t0, beams
        self.k = 0

    def next(self):
        import synth
        t1 = self.t0 + 0.1 * self.k
        dt, acc, gyr = imu_synth.samples(t1 - 0.1, t1)
        imu = [(t1 - 0.1 + j / 200.0, acc[j], gyr[j]) for j in range(0 if self.k == 0 else 1, len(dt))]
        rows = synth.make_scan(self.scene, self.beams, t1)
        self.k += 1
        return t1, imu, np.stack([rows["x"], rows["y"], rows["z"], rows["t"]], 1).astype(np.float32)


def feed_imu(builder, imu):
    for t, a, g in imu:
        builder.add_imu_data(t, a, g)


def builder_pair(ctxs, orc, t0, **kw):
    """The same builder twice, one per context (0: batched, 1: single calls), initialised at the drive's state."""
    import dliom
    out = []
    for ctx in ctxs:
        b = dliom.LocalTrajectoryBuilder(ctx, make_options(orc, **kw))
        b.set_initial_state(imu_synth.state(t0 - 0.1))
        out.append(b)
    return out


def single(builder, time, scan, origins=None):
    import dliom
    rows, row_floats, o = dliom._ltb_rows(scan, origins)
    r = dliom.MatchingResult()
    builder.ctx.check(builder.ctx.L.dl_ltb_add_synchronized_range_data(builder.h, float(time), rows.ctypes.data, len(rows), row_floats,
                                                                       o, len(o), ctypes.byref(r)))
    return r


def assert_same_builder(a, b, ra=None, rb=None):
    if ra is not None:
        assert bytes(ra) == bytes(rb)
    sa, ia = a.state()
    sb, ib = b.state()
    assert ia == ib and np.array_equal(sa.view(np.uint64), sb.view(np.uint64))
    for which in range(4):
        assert np.array_equal(a.cloud(which).view(np.uint32), b.cloud(which).view(np.uint32)), which
    assert np.array_equal(a.histogram().view(np.uint32), b.histogram().view(np.uint32))
    assert a.num_submaps() == b.num_submaps()
    for i in range(a.num_submaps()):
        _, _, pa, na, fa = a.submap(i)
        _, _, pb, nb, fb = b.submap(i)
        assert np.array_equal(pa.view(np.uint64), pb.view(np.uint64)) and (na, fa) == (nb, fb)


def assert_same_grids(a, b):
    for i in range(a.num_submaps()):
        ga, gb = a.submap(i)[:2], b.submap(i)[:2]
        for x, y in zip(ga, gb):
            ex, ey = x.export(), y.export()
            assert all(np.array_equal(u, v) for u, v in zip(ex, ey)), i


@pytest.mark.gpu
def test_batch_equals_single_calls_over_a_drive(orc):
    """Four trajectories with staggered starts, 15 scans each, num_range_data 3: the hand-overs fall on different steps."""
    import dliom
    import synth
    ctxs = [dliom.Context(0), dliom.Context(0)]
    scene = synth.Scene(42)
    trajs = [Trajectory(scene, 2.0 + 0.53 * j) for j in range(4)]
    pairs = [builder_pair(ctxs, orc, tr.t0, num_range_data=3) for tr in trajs]
    for step in range(15 + 3):
        members = [j for j in range(4) if j <= step < j + 15]
        inputs = []
        for j in members:
            t1, imu, xyzt = trajs[j].next()
            feed_imu(pairs[j][0], imu)
            feed_imu(pairs[j][1], imu)
            inputs.append((t1, xyzt))
        got = dliom.add_range_data_batch([pairs[j][0] for j in members], [t for t, _ in inputs], [x for _, x in inputs])
        for j, (t1, xyzt), r in zip(members, inputs, got):
            want = single(pairs[j][1], t1, xyzt)
            assert r.has_result == 1 and r.inserted == 1
            assert_same_builder(pairs[j][0], pairs[j][1], r, want)
    assert {pairs[j][0].num_submaps() for j in range(4)} == {6}
    for a, b in pairs:
        assert_same_grids(a, b)
    for p in pairs:
        for b in p:
            b.close()


@pytest.mark.gpu
def test_mixed_members_in_one_call(orc):
    """Initialising, no IMU since the last scan, an empty scan, a dropped scan, a motion-filtered scan and a normal one."""
    import dliom
    import synth
    ctxs = [dliom.Context(0), dliom.Context(0)]
    scene = synth.Scene(42)
    trajs = [Trajectory(scene, 2.0 + 0.41 * j) for j in range(6)]
    kw = dict(max_time_seconds=5.0, max_distance_meters=50.0, max_angle_radians=3.0)   # only a builder's first scan is inserted
    pairs = [builder_pair(ctxs, orc, tr.t0, **kw) for tr in trajs]
    # member 0 is still initialising: a builder without an initial state
    pairs[0] = [dliom.LocalTrajectoryBuilder(ctx, make_options(orc, **kw)) for ctx in ctxs]
    # member 4 has inserted one scan already: its second is held back by the motion filter
    t1, imu, xyzt = trajs[4].next()
    for b in pairs[4]:
        feed_imu(b, imu)
        assert b.add_range_data(t1, xyzt).inserted == 1
    times, scans = [], []
    for j in range(6):
        t1, imu, xyzt = trajs[j].next()
        if j == 2:
            xyzt = np.zeros((0, 4), np.float32)
        if j == 3:
            xyzt = xyzt.copy()
            xyzt[:, :3] *= 1000.0                      # every point beyond max_range: no returns, the scan is dropped
        for b in pairs[j]:
            if j != 1:                                 # member 1: no IMU since its last scan (none at all)
                feed_imu(b, imu)
        times.append(t1)
        scans.append(xyzt)
    got = dliom.add_range_data_batch([p[0] for p in pairs], times, scans)
    for j in range(6):
        want = single(pairs[j][1], times[j], scans[j])
        assert_same_builder(pairs[j][0], pairs[j][1], got[j], want)
    assert [r.has_result for r in got] == [0, 0, 0, 0, 1, 1]
    assert got[3].scan.ok == 0 and got[4].inserted == 0 and got[5].inserted == 1
    for p in pairs:
        for b in p:
            b.close()


@pytest.mark.gpu
def test_two_stage_members(orc):
    import dliom
    import synth
    ctxs = [dliom.Context(0), dliom.Context(0)]
    scene = synth.Scene(7)
    trajs = [Trajectory(scene, 2.0 + 0.3 * j) for j in range(3)]
    pairs = [builder_pair(ctxs, orc, tr.t0, num_range_data=4, two_stage=1, ceres_pose_noise_t=0.02, ceres_pose_noise_r=0.01)
             for tr in trajs]
    for _ in range(6):
        inputs = []
        for j, tr in enumerate(trajs):
            t1, imu, xyzt = tr.next()
            feed_imu(pairs[j][0], imu)
            feed_imu(pairs[j][1], imu)
            inputs.append((t1, xyzt))
        got = dliom.add_range_data_batch([p[0] for p in pairs], [t for t, _ in inputs], [x for _, x in inputs])
        for j, r in enumerate(got):
            assert r.has_result == 1
            assert_same_builder(pairs[j][0], pairs[j][1], r, single(pairs[j][1], *inputs[j]))
    for a, b in pairs:
        assert_same_grids(a, b)
    for p in pairs:
        for b in p:
            b.close()


@pytest.mark.gpu
def test_range_measurement_rows_next_to_xyzt_rows(orc):
    """A member with 32-byte RangeMeasurement rows and two origins in the same call as members with x y z t rows."""
    import dliom
    import synth
    from synth import RANGE_DTYPE
    ctxs = [dliom.Context(0), dliom.Context(0)]
    scene = synth.Scene(42)
    trajs = [Trajectory(scene, 2.0 + 0.5 * j) for j in range(3)]
    pairs = [builder_pair(ctxs, orc, tr.t0) for tr in trajs]
    two = np.array([[0.0, 0.0, 0.0], [0.1, -0.2, 0.05]], np.float32)
    for _ in range(3):
        times, scans, origins = [], [], []
        for j, tr in enumerate(trajs):
            t1, imu, xyzt = tr.next()
            for b in pairs[j]:
                feed_imu(b, imu)
            if j == 1:
                rows = np.zeros(len(xyzt), RANGE_DTYPE)
                rows["x"], rows["y"], rows["z"], rows["t"] = xyzt[:, 0], xyzt[:, 1], xyzt[:, 2], xyzt[:, 3]
                rows["origin_index"] = np.arange(len(xyzt)) % 2
                scans.append(rows)
                origins.append(two)
            else:
                scans.append(xyzt)
                origins.append(np.zeros((1, 3), np.float32))
            times.append(t1)
        got = dliom.add_range_data_batch([p[0] for p in pairs], times, scans, origins)
        for j in range(3):
            assert_same_builder(pairs[j][0], pairs[j][1], got[j], single(pairs[j][1], times[j], scans[j], origins[j]))
    for a, b in pairs:
        assert_same_grids(a, b)
    for p in pairs:
        for b in p:
            b.close()


def _rotate_f32(q, p):
    """dl_math.cuh's rotate() in float32, one rounding per operation (no contraction), in its order."""
    w, x, y, z = (np.float32(v) for v in q)

    def cross(ax, ay, az, bx, by, bz):
        return ay * bz - az * by, az * bx - ax * bz, ax * by - ay * bx
    px, py, pz = p[:, 0], p[:, 1], p[:, 2]
    ux, uy, uz = cross(x, y, z, px, py, pz)
    ux, uy, uz = ux + ux, uy + uy, uz + uz
    cx, cy, cz = cross(x, y, z, ux, uy, uz)
    return np.stack([(px + w * ux) + cx, (py + w * uy) + cy, (pz + w * uz) + cz], 1).astype(np.float32)


@pytest.mark.gpu
def test_local_frame_and_histogram_input_keep_the_host_bits(orc):
    """range_data_in_local = opt_pose.cast<float>() * returns and the histogram of the gravity-aligned returns, as the host loops
    they replace computed them: a float32 restatement of dl_math.cuh's rotate / apply (one rounding per operation) applied to the
    oracle chain's tracking-frame returns gives cloud 0 bit for bit, and the device histogram of that restated aligned cloud is
    the builder's histogram bit for bit."""
    import dliom
    import synth
    ctx = dliom.Context(0)
    opts = orc.FrontEndOptions.defaults()
    scene = synth.Scene(42)
    t1 = 2.0
    b = dliom.LocalTrajectoryBuilder(ctx, make_options(orc))
    state_i = imu_synth.state(t1 - 0.1)
    b.set_initial_state(state_i)
    dt, acc, gyr = imu_synth.samples(t1 - 0.1, t1)
    ts = t1 - 0.1 + np.arange(len(dt)) / 200.0
    for j in range(len(dt)):
        b.add_imu_data(ts[j], acc[j], gyr[j])
    iv_dt = np.array([1.0 / 500.0] + [ts[j] - ts[j - 1] for j in range(1, len(dt))])   # LTB:183-185
    rows = synth.make_scan(scene, 16, t1)
    origin = np.zeros((1, 3), np.float32)
    hi, lo, sp, _, _ = b.submap(0)
    ohi, olo = orc.Grid(0.1), orc.Grid(0.45)
    ohi.set_cells(*hi.export())
    olo.set_cells(*lo.export())
    _, _, pred, ok, _ = orc.frontend_batch_imu(opts, [rows], origin, NOISE, [state_i], [(iv_dt, np.asarray(acc), np.asarray(gyr))],
                                                sp, ohi, olo, 1, imu_weight=0.7)
    assert ok[0] == 1
    r = dliom.add_range_data_batch([b], [t1], [np.stack([rows["x"], rows["y"], rows["z"], rows["t"]], 1).astype(np.float32)])[0]
    assert r.inserted == 1
    pts = orc.ingest_scan(opts, rows, origin, state_i[:7], pred[0][:7])["returns_tracking"].astype(np.float32)
    hk, _ = orc.adaptive_voxel_filter(pts, opts.hi_max_length, opts.hi_min_num_points, opts.hi_max_range)
    assert np.array_equal(b.cloud(2).view(np.uint32), pts[hk].view(np.uint32))         # the same tracking-frame returns
    pose = np.array(r.local_pose[:], np.float64)
    local = _rotate_f32(pose[3:7].astype(np.float32), pts) + pose[:3].astype(np.float32)
    assert np.array_equal(b.cloud(0).view(np.uint32), local.astype(np.float32).view(np.uint32))
    aligned = _rotate_f32(pose[3:7].astype(np.float32), pts)
    want = ctx.rotational_histogram(aligned, 120)
    assert np.array_equal(b.histogram().view(np.uint32), np.asarray(want, np.float32).view(np.uint32))
    b.close()


def _item(b, t, xyzt, origin):
    import dliom
    return dliom.LtbBatchItem(b.h, t, xyzt.ctypes.data, len(xyzt), 4, 1, origin.ctypes.data)


@pytest.mark.gpu
def test_rejected_calls_leave_the_builders_untouched(orc):
    import dliom
    import synth
    ctx, other = dliom.Context(0), dliom.Context(0)
    scene = synth.Scene(42)
    trajs = [Trajectory(scene, 2.0 + 0.5 * j) for j in range(3)]
    b0 = dliom.LocalTrajectoryBuilder(ctx, make_options(orc))
    b1 = dliom.LocalTrajectoryBuilder(ctx, make_options(orc))
    b_other = dliom.LocalTrajectoryBuilder(other, make_options(orc))
    b_diff = dliom.LocalTrajectoryBuilder(ctx, make_options(orc, num_range_data=7))
    builders = [b0, b1, b_other, b_diff]
    inputs = []
    for b, tr in zip(builders, trajs + [trajs[0]]):
        b.set_initial_state(imu_synth.state(tr.t0 - 0.1))
        t1, imu, xyzt = tr.next()
        feed_imu(b, imu)
        inputs.append((t1, xyzt))
    origin = np.zeros(3, np.float32)
    before = [(b.state()[0].copy(), b.num_submaps()) for b in builders]
    results = (dliom.MatchingResult * 4)()

    def call(items):
        arr = (dliom.LtbBatchItem * len(items))(*items)
        return ctx.L.dl_ltb_add_range_data_batch(len(items), arr, results)

    good = [_item(b0, inputs[0][0], inputs[0][1], origin), _item(b1, inputs[1][0], inputs[1][1], origin)]
    assert call(good + [_item(b0, inputs[0][0], inputs[0][1], origin)]) == DL_ERR_ARG          # a builder twice
    assert call(good + [_item(b_other, inputs[2][0], inputs[2][1], origin)]) == DL_ERR_ARG     # two contexts
    assert call(good + [_item(b_diff, inputs[3][0], inputs[3][1], origin)]) == DL_ERR_ARG      # options differ
    null_rows = dliom.LtbBatchItem(b1.h, inputs[1][0], None, 5, 4, 1, origin.ctypes.data)
    assert call([good[0], null_rows]) == DL_ERR_ARG                                             # rows missing
    for b, (s, n) in zip(builders, before):
        assert np.array_equal(b.state()[0], s) and b.num_submaps() == n and b.cloud(2).shape == (0, 3)
    assert ctx.L.dl_ltb_add_range_data_batch(0, None, None) == DL_OK
    assert call(good) == DL_OK and results[0].inserted == 1 and results[1].inserted == 1


@pytest.mark.gpu
def test_kernel_launches_do_not_grow_with_the_members(orc):
    """The batch does not loop over its members on the host: an 8-member call makes at most twice the launches of a 1-member
    call at the same point of the drive, where eight single calls make about eight times as many."""
    import dliom
    import synth
    scene = synth.Scene(42)

    def launches(count, batched):
        ctx = dliom.Context(0)
        trajs = [Trajectory(scene, 2.0 + 0.37 * j) for j in range(count)]
        bs = [dliom.LocalTrajectoryBuilder(ctx, make_options(orc)) for _ in trajs]
        for b, tr in zip(bs, trajs):
            b.set_initial_state(imu_synth.state(tr.t0 - 0.1))
        per_step = []
        for _ in range(3):   # the first steps grow the fresh grids; the last one is measured
            inputs = []
            for b, tr in zip(bs, trajs):
                t1, imu, xyzt = tr.next()
                feed_imu(b, imu)
                inputs.append((t1, xyzt))
            before = ctx.launches
            if batched:
                dliom.add_range_data_batch(bs, [t for t, _ in inputs], [x for _, x in inputs])
            else:
                for b, (t1, xyzt) in zip(bs, inputs):
                    b.add_range_data(t1, xyzt)
            per_step.append(ctx.launches - before)
        for b in bs:
            b.close()
        return per_step[-1]

    one, eight, eight_single = launches(1, True), launches(8, True), launches(8, False)
    assert eight <= 2 * one, (one, eight)
    assert eight_single >= 6 * one, (one, eight_single)


def test_batch_item_layout_matches_the_header(tmp_path):
    """ctypes' LtbBatchItem against the C compiler's dl_ltb_batch_item: size and every field's offset."""
    import dliom
    src = tmp_path / "layout.c"
    fields = [f for f, _ in dliom.LtbBatchItem._fields_]
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "dliom_b200.h"\nint main(void) {\n'
                   '  printf("%zu", sizeof(dl_ltb_batch_item));\n' +
                   "".join(f'  printf(" %zu", offsetof(dl_ltb_batch_item, {f}));\n' for f in fields) + '  return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert got == [ctypes.sizeof(dliom.LtbBatchItem)] + [getattr(dliom.LtbBatchItem, f).offset for f in fields]


@pytest.mark.gpu
def test_cpp_shim_batch_equals_per_builder_calls(tmp_path):
    """host/dliom_b200.hpp: the static LocalTrajectoryBuilder3D::AddRangeData over (builder, sensor id, cloud) items, driven by a
    C++ program for two trajectories, prints the same node poses, bit for bit (%.17g), as the per-builder AddRangeData."""
    import struct
    import dliom
    import synth
    host = os.path.join(ROOT, "d-liom_b200", "host")
    exe = str(tmp_path / "example_trajectories_batch")
    subprocess.check_call(["g++", "-std=c++17", "-O1", os.path.join(host, "example_trajectories_batch.cc"), "-o", exe,
                           "-L" + os.path.join(ROOT, "d-liom_b200"), "-ldliom_b200", "-Wl,-rpath," + os.path.join(ROOT, "d-liom_b200")])
    scene = synth.Scene(42)
    trajs = [Trajectory(scene, 2.0 + 0.6 * j) for j in range(2)]
    steps = 8
    path = str(tmp_path / "drives.bin")
    with open(path, "wb") as f:
        f.write(struct.pack("<i", len(trajs)))
        for tr in trajs:
            f.write(dliom.NavState.from16(imu_synth.state(tr.t0 - 0.1)))
        f.write(struct.pack("<i", steps))
        for _ in range(steps):
            for tr in trajs:
                t1, imu, xyzt = tr.next()
                f.write(struct.pack("<i", len(imu)))
                for t, a, g in imu:
                    f.write(struct.pack("<d", t) + np.asarray(a, np.float64).tobytes() + np.asarray(g, np.float64).tobytes())
                f.write(struct.pack("<di", t1, len(xyzt)) + xyzt.tobytes())
    out = {}
    for mode in ("single", "batch"):
        r = subprocess.run([exe, path, mode], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        out[mode] = r.stdout.strip().splitlines()
    results = [l for l in out["single"] if l.startswith("result")]
    assert len(results) == 2 * steps and all(l.split()[10] == "1" for l in results)   # every scan matched and inserted
    assert max(int(l.split()[12]) for l in results) >= 3                                # submaps were handed over
    assert out["batch"] == out["single"]
