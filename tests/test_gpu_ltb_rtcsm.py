"""LocalTrajectoryBuilder3D with the online correlative pre-match (use_online_correlative_scan_matching, LTB:514-521) in both
solve modes and in many-trajectory batches. Every scan is checked against the oracle chain run on the builder's OWN state and
its own exported grids at that scan: the pre-match (orc.rtcsm_match / match_scan), then the plain match and the window update
(two-stage) or the fused solve seeded with the pre-match's pose (fused)."""
import ctypes

import numpy as np
import pytest

import imu_synth
from helpers import pose_error, workload

pytestmark = pytest.mark.gpu
NOISE = [3.99e-2, 1.56e-2, 6.4e-5, 3.6e-5]
ORIGIN = np.zeros((1, 3), np.float32)
DL_ERR_ARG, DL_ERR_SCORE = -2, -5   # dl_status


class Drive:
    """One synthetic drive (200 Hz IMU, 10 Hz 16-beam scans) and the IMU interval its builder is integrating: sample 0 of an
    interval is the last sample of the interval its previous committed scan used."""

    def __init__(self, scene, t0, beams=16):
        self.scene, self.t0, self.beams = scene, t0, beams
        self.k, self.last_t, self.iv = 0, None, []

    def next(self, acc_offset=None):
        import synth
        t1 = self.t0 + 0.1 * self.k
        dt, acc, gyr = imu_synth.samples(t1 - 0.1, t1)
        if acc_offset is not None:
            acc = acc + np.asarray(acc_offset, np.float64)
        ts = t1 - 0.1 + np.arange(len(dt)) / 200.0
        imu = []
        for j in range(0 if self.k == 0 else 1, len(dt)):
            d = 1.0 / 500.0 if self.last_t is None else ts[j] - self.last_t   # LTB:183-185
            self.last_t = ts[j]
            self.iv.append((d, acc[j], gyr[j]))
            imu.append((ts[j], acc[j], gyr[j]))
        self.k += 1
        return t1, imu, synth.make_scan(self.scene, self.beams, t1)

    def interval(self):
        return (np.array([v[0] for v in self.iv]), np.array([v[1] for v in self.iv]), np.array([v[2] for v in self.iv]))

    def committed(self):
        self.iv = self.iv[-1:]


def xyzt(rows):
    return np.stack([rows["x"], rows["y"], rows["z"], rows["t"]], 1).astype(np.float32)


def feed(builder, imu):
    for t, a, g in imu:
        builder.add_imu_data(t, a, g)


def make_builder(ctx, opts, **kw):
    import dliom
    fo = dliom.FrontendOptions.from_oracle(opts)
    kw.setdefault("max_time_seconds", 0.05)   # 0.1 s between scans: the motion filter never holds a scan back
    return dliom.LocalTrajectoryBuilder(ctx, dliom.LtbOptions.defaults(fo, NOISE, imu_weight=0.7, **kw))


def oracle_grids(orc, hi, lo):
    ohi, olo = orc.Grid(0.1), orc.Grid(0.45)
    ohi.set_cells(*hi.export())
    olo.set_cells(*lo.export())
    return ohi, olo


def cells(export):
    return {(int(x), int(y), int(z)): int(v) for x, y, z, v in zip(*export)}


def nav(s):
    return np.array(list(s.p) + list(s.q) + list(s.v) + list(s.ba) + list(s.bg))


def bits(x):
    return int(np.float32(x).view(np.uint32))


def matching_submap(b):
    """The active submaps' front (LTB:502-505): the oldest submap not finished."""
    return min(i for i in range(b.num_submaps()) if not b.submap(i)[4])


def oracle_scan(orc, opts, state_i, iv, rows, sp, ohi, olo):
    """Pre-integrate, predict, ingest, then the oracle's match_scan (filters -> pre-match -> plain match) on the given grids."""
    m = orc.imu_preintegrate(NOISE, state_i[10:13], state_i[13:16], *iv)
    pred = orc.imu_predict(state_i, m)
    ing = orc.ingest_scan(opts, rows, ORIGIN, state_i[:7], pred[:7])
    pts = ing["returns_tracking"]
    cur = ing["current_pose"].astype(np.float64)
    ms = orc.match_scan(opts, pts, cur, sp, ohi, olo)
    return {"m": m, "pred": pred, "pts": pts, "cur": cur, "ms": ms}


def oracle_fused(orc, opts, state_i, c, ohi, olo):
    """The fused chain of a submap at the identity: the pre-match from the prediction, then the fused solve whose state j starts
    at the pre-match's pose with the prediction's velocity and biases, pulled to the prediction's translation (LTB:536)."""
    pts, ms = c["pts"], c["ms"]
    hc, lc = pts[ms["hi_keep"]], pts[ms["lo_keep"]]
    pre = orc.rtcsm_match(ohi, hc, c["cur"], opts.rtcsm_linear_window, opts.rtcsm_angular_window, opts.rtcsm_w_t, opts.rtcsm_w_r)
    init = c["pred"].copy()
    init[:7] = pre["pose"]
    want, ws = orc.fused_match([hc, lc], [ohi, olo], [opts.occ_w0, opts.occ_w1], opts.trans_w, opts.rot_w, c["cur"][:3], state_i,
                               init, c["m"], imu_weight=0.7, max_iter=opts.max_iter)
    return pre, want, ws


def assert_clouds(b, c):
    pts, ms = c["pts"], c["ms"]
    assert np.array_equal(b.cloud(2).view(np.uint32), pts[ms["hi_keep"]].view(np.uint32))
    assert np.array_equal(b.cloud(3).view(np.uint32), pts[ms["lo_keep"]].view(np.uint32))


def assert_submap0_cells(orc, b, inserted):
    """Submap 0 lives at the identity: its grids equal the oracle inserter fed with the builder's own range data."""
    ohi, olo = orc.Grid(0.1), orc.Grid(0.45)
    for o, local in inserted:
        d = local - o
        r2 = (d[:, 0] * d[:, 0] + (d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])).astype(np.float32)
        ohi.insert_range_data(o, local[np.sqrt(r2).astype(np.float32) <= np.float32(20.0)])
        olo.insert_range_data(o, local)
    hi0, lo0, *_ = b.submap(0)
    assert cells(hi0.export()) == cells(ohi.export()) and cells(lo0.export()) == cells(olo.export())


def test_two_stage_prematch_follows_the_reference_chain(orc):
    """Pre-match -> plain match from its pose (target: the prediction's translation) -> window update (LTB:514-555)."""
    import dliom
    import synth
    ctx = dliom.Context(0)
    opts = orc.FrontEndOptions.defaults(use_rtcsm=1)
    drv = Drive(synth.Scene(42), 2.0)
    b = make_builder(ctx, opts, num_range_data=50, two_stage=1, ceres_pose_noise_t=0.02, ceres_pose_noise_r=0.01,
                     prior_pose_noise=0.01, prior_velocity_noise=0.2, prior_bias_noise=0.01)
    state = imu_synth.state(drv.t0 - 0.1)
    b.set_initial_state(state)
    info = np.diag([1 / 0.01 ** 2] * 6 + [1 / 0.2 ** 2] * 3 + [1 / 0.01 ** 2] * 6)
    inserted = []
    for k in range(7):
        t1, imu, rows = drv.next()
        feed(b, imu)
        sb, _ = b.state()
        hi, lo, sp, _, _ = b.submap(0)
        ohi, olo = oracle_grids(orc, hi, lo)
        iv = drv.interval()
        r = b.add_range_data(t1, xyzt(rows))
        assert r.has_result == 1 and r.scan.ok == 1 and r.inserted == 1
        drv.committed()
        # stage one on the builder's own state and grids: the pre-match's score bit for bit, the plain match from its pose
        c = oracle_scan(orc, opts, sb, iv, rows, sp, ohi, olo)
        assert c["ms"]["ok"]
        assert bits(r.rtcsm_score) == bits(c["ms"]["rtcsm_score"]) and r.rtcsm_score > 0
        dtm, drm = pose_error(np.array(r.scan.pose_estimate_local[:]), c["ms"]["pose_estimate_local"])
        assert dtm < 1e-6 and drm < 1e-7, (k, dtm, drm)
        assert_clouds(b, c)
        # stage two: the oracle's own chain (its state and carried information), as test_gpu_ltb's two-stage check
        m = orc.imu_preintegrate(NOISE, state[10:13], state[13:16], *iv)
        pred = orc.imu_predict(state, m)
        _, poses, ok = orc.frontend_batch(opts, [rows], ORIGIN, [state[:7]], [pred[:7]], sp, ohi, olo, 1)
        assert ok[0] == 1
        _, state, info, _ = orc.window_optimize(state, info, m, poses[0], sigma_t=0.02, sigma_r=0.01, imu_weight=0.7, initial_j=pred)
        got = nav(r.state)
        dtn, drn = pose_error(got[:7], state[:7])
        assert dtn < 2e-6 and drn < 1e-6, (k, dtn, drn)
        assert np.abs(got[7:] - state[7:]).max() < 1e-5
        inserted.append((np.array(r.origin_in_local[:], np.float32), b.cloud(0).copy()))
    assert b.num_submaps() == 1
    assert_submap0_cells(orc, b, inserted)
    b.close()
    ctx.close()


def test_fused_prematch_seeds_the_fused_solve(orc):
    """Fused mode: the pre-match's pose replaces the pose part of state j's initial value; velocity and biases stay the
    prediction's."""
    import dliom
    import synth
    ctx = dliom.Context(0)
    opts = orc.FrontEndOptions.defaults(use_rtcsm=1)
    drv = Drive(synth.Scene(42), 2.0)
    b = make_builder(ctx, opts, num_range_data=50)
    b.set_initial_state(imu_synth.state(drv.t0 - 0.1))
    inserted = []
    for k in range(8):
        t1, imu, rows = drv.next()
        feed(b, imu)
        sb, _ = b.state()
        hi, lo, sp, _, _ = b.submap(0)
        assert np.array_equal(sp, orc.IDENTITY_POSE)
        ohi, olo = oracle_grids(orc, hi, lo)
        iv = drv.interval()
        r = b.add_range_data(t1, xyzt(rows))
        assert r.has_result == 1 and r.scan.ok == 1 and r.inserted == 1
        drv.committed()
        c = oracle_scan(orc, opts, sb, iv, rows, sp, ohi, olo)
        pre, want, ws = oracle_fused(orc, opts, sb, c, ohi, olo)
        assert bits(r.rtcsm_score) == bits(pre["score"]) == bits(c["ms"]["rtcsm_score"])
        got = nav(r.state)
        dtn, drn = pose_error(got[:7], want[:7])
        assert dtn < 1e-6 and drn < 1e-7, (k, dtn, drn)
        assert np.allclose(got[7:], want[7:], atol=1e-6)
        assert r.scan.summary.num_iterations == ws["num_iterations"]
        assert_clouds(b, c)
        inserted.append((np.array(r.origin_in_local[:], np.float32), b.cloud(0).copy()))
    assert_submap0_cells(orc, b, inserted)
    b.close()
    ctx.close()


def test_fused_frontend_batch_with_prematch(orc):
    """One multi-scan dl_frontend_match_batch_imu_samples call with the pre-match against a fixed submap."""
    import dliom
    ctx = dliom.Context(0)
    w = workload()
    o = orc.FrontEndOptions.defaults(use_rtcsm=1)
    hi, lo = dliom.Grid.from_oracle(ctx, w["hi"]), dliom.Grid.from_oracle(ctx, w["lo"])
    fo = dliom.FrontendOptions.from_oracle(o)
    intervals, states_i = [], []
    for s in range(len(w["scans"])):
        t1 = w["times"][s]
        intervals.append(imu_synth.samples(t1 - 0.1, t1, noise=(3.99e-2, 1.56e-2), seed=30 + s))
        states_i.append(imu_synth.state(t1 - 0.1, ba=(0.01, -0.02, 0.005), bg=(1e-3, -2e-3, 5e-4)))
    imu = dliom.ImuSamples(NOISE, intervals, states_i, imu_weight=0.7)
    res, states, _ = ctx.frontend_match_batch_imu_samples(fo, w["scans"], w["origin"], imu, w["submap_pose"], hi, lo)
    for s in range(len(w["scans"])):
        c = oracle_scan(orc, o, states_i[s], intervals[s], w["scans"][s], w["submap_pose"], w["hi"], w["lo"])
        pre, want, ws = oracle_fused(orc, o, states_i[s], c, w["hi"], w["lo"])
        assert res[s].ok == 1
        assert bits(res[s].rtcsm_score) == bits(pre["score"])
        dtn, drn = pose_error(states[s][:7], want[:7])
        assert dtn < 1e-6 and drn < 1e-7, (s, dtn, drn)
        assert np.allclose(states[s][7:], want[7:], atol=1e-6)
        assert res[s].summary.num_iterations == ws["num_iterations"]
    ctx.close()


@pytest.mark.parametrize("two_stage", [0, 1])
def test_displaced_prediction_is_pulled_back(orc, two_stage):
    """An accelerometer offset over one interval displaces the prediction inside the search window: the pre-match moves
    the pose off the initial one, to the oracle's candidate, and the solve continues from there."""
    import dliom
    import synth
    ctx = dliom.Context(0)
    opts = orc.FrontEndOptions.defaults(use_rtcsm=1)
    drv = Drive(synth.Scene(42), 2.0)
    b = make_builder(ctx, opts, num_range_data=50, two_stage=two_stage)
    b.set_initial_state(imu_synth.state(drv.t0 - 0.1))
    for k in range(5):
        t1, imu, rows = drv.next(acc_offset=(20.0, -10.0, 0.0) if k == 4 else None)   # about 0.11 m off after 0.1 s
        feed(b, imu)
        sb, _ = b.state()
        hi, lo, sp, _, _ = b.submap(0)
        ohi, olo = oracle_grids(orc, hi, lo)
        iv = drv.interval()
        r = b.add_range_data(t1, xyzt(rows))
        assert r.has_result == 1 and r.scan.ok == 1
        drv.committed()
        c = oracle_scan(orc, opts, sb, iv, rows, sp, ohi, olo)
        pre, want, _ = oracle_fused(orc, opts, sb, c, ohi, olo)
        assert bits(r.rtcsm_score) == bits(pre["score"])
        if k == 4:   # the pre-match moved off the prediction: a translation step (0.1 m) or a rotation step (~7 mrad)
            dtp, drp = pose_error(pre["pose"], c["cur"])
            assert dtp > 0.05 or drp > 3e-3, (dtp, drp)
        if two_stage:
            dtm, drm = pose_error(np.array(r.scan.pose_estimate_local[:]), c["ms"]["pose_estimate_local"])
        else:
            dtm, drm = pose_error(nav(r.state)[:7], want[:7])
        assert dtm < 1e-6 and drm < 1e-7, (k, dtm, drm)
    b.close()
    ctx.close()


def _single(builder, time, scan):
    import dliom
    rows, row_floats, o = dliom._ltb_rows(scan, None)
    r = dliom.MatchingResult()
    st = builder.ctx.L.dl_ltb_add_synchronized_range_data(builder.h, float(time), rows.ctypes.data, len(rows), row_floats, o, len(o),
                                                          ctypes.byref(r))
    return st, r


def _snapshot(b):
    s, init = b.state()
    subs = []
    for i in range(b.num_submaps()):
        hi, lo, pose, n, fin = b.submap(i)
        subs.append((pose.tobytes(), n, fin, [a.tobytes() for a in hi.export()], [a.tobytes() for a in lo.export()]))
    return (s.tobytes(), init, [b.cloud(w).tobytes() for w in range(4)], b.histogram().tobytes(), subs)


def test_batch_of_trajectories_on_different_grids(orc):
    """Five builders whose matching submaps differ, stepped by one dl_ltb_add_range_data_batch call per step against twins
    stepped by single calls: byte-identical results and builder state, hand-overs inside the run, one member still
    initialising and one scan dropped; every member's score is the oracle's on its own grid."""
    import dliom
    import synth
    opts = orc.FrontEndOptions.defaults(use_rtcsm=1)
    ctxs = [dliom.Context(0), dliom.Context(0)]
    scene = synth.Scene(42)
    drives = [Drive(scene, 2.0 + 0.53 * j) for j in range(5)]
    pairs = []
    for j, d in enumerate(drives):
        pair = [make_builder(ctx, opts, num_range_data=3) for ctx in ctxs]
        if j != 4:                                     # member 4 stays initialising (InitializeStatic needs 7 frames)
            for bb in pair:
                bb.set_initial_state(imu_synth.state(d.t0 - 0.1))
        pairs.append(pair)
    scored = 0
    for step in range(7):
        inputs, before = [], []
        for j, d in enumerate(drives):
            t1, imu, rows = d.next()
            scan = xyzt(rows)
            if j == 2 and step == 3:
                scan = scan.copy()
                scan[:, :3] *= 1000.0                  # every point beyond max_range: the scan is dropped
            for bb in pairs[j]:
                feed(bb, imu)
            b = pairs[j][0]
            sb, init = b.state()
            grids = None
            if init:
                i = matching_submap(b)
                hi, lo, sp, _, _ = b.submap(i)
                grids = (sp, *oracle_grids(orc, hi, lo), hi.export())
            inputs.append((t1, scan, rows))
            before.append((sb, d.interval(), grids))
        if step == 4:   # the members' matching grids differ
            hs = [before[j][2][3] for j in range(4)]
            assert any(len(hs[0][0]) != len(h[0]) or not all(np.array_equal(u, v) for u, v in zip(hs[0], h)) for h in hs[1:])
        got = dliom.add_range_data_batch([p[0] for p in pairs], [t for t, _, _ in inputs], [s for _, s, _ in inputs])
        for j in range(5):
            st, want = _single(pairs[j][1], inputs[j][0], inputs[j][1])
            assert st == 0
            assert bytes(got[j]) == bytes(want)
            assert _snapshot(pairs[j][0]) == _snapshot(pairs[j][1])
            r = got[j]
            if r.scan.ok == 1:
                drives[j].committed()
            if not r.has_result:
                continue
            sb, iv, (sp, ohi, olo, _) = before[j]
            c = oracle_scan(orc, opts, sb, iv, inputs[j][2], sp, ohi, olo)
            assert bits(r.rtcsm_score) == bits(c["ms"]["rtcsm_score"]) and r.rtcsm_score > 0, (step, j)
            scored += 1
        assert got[4].has_result == 0
        if step == 3:
            assert got[2].scan.ok == 0 and got[2].has_result == 0
    assert scored == 4 * 7 - 1
    assert all(pairs[j][0].num_submaps() >= 3 for j in range(4))   # hand-overs happened inside the run
    for p in pairs:
        for bb in p:
            bb.close()


@pytest.mark.parametrize("two_stage", [0, 1])
def test_nonpositive_candidate_score_fails_the_call(orc, two_stage):
    """A translation cost weight of 1e3 drives exp(-(|t| w)^2) of the window-edge candidates to 0 in float: the reference
    CHECK-fails (real_time_correlative_scan_matcher_3d.cc:111). The batch fails with DL_ERR_SCORE and no builder changes."""
    import dliom
    import synth
    ctx = dliom.Context(0)
    opts = orc.FrontEndOptions.defaults(use_rtcsm=1, rtcsm_w_t=1e3)
    drives = [Drive(synth.Scene(42), 2.0 + 0.4 * j) for j in range(3)]
    bs = [make_builder(ctx, opts, num_range_data=50, two_stage=two_stage) for _ in drives]
    times, scans = [], []
    for b, d in zip(bs, drives):
        b.set_initial_state(imu_synth.state(d.t0 - 0.1))
        t1, imu, rows = d.next()
        feed(b, imu)
        times.append(t1)
        scans.append(xyzt(rows))
    before = [_snapshot(b) for b in bs]
    with pytest.raises(dliom.DlError) as e:
        dliom.add_range_data_batch(bs, times, scans)
    assert e.value.status == DL_ERR_SCORE
    assert [_snapshot(b) for b in bs] == before
    st, _ = _single(bs[0], times[0], scans[0])
    assert st == DL_ERR_SCORE and _snapshot(bs[0]) == before[0]
    for b in bs:
        b.close()
    ctx.close()


def test_only_optimize_yaw(orc):
    """Two-stage builders take only_optimize_yaw: the plain match after the pre-match is the oracle's yaw-only ceres_match.
    The fused solve still refuses it."""
    import dliom
    import synth
    ctx = dliom.Context(0)
    opts = orc.FrontEndOptions.defaults(use_rtcsm=1, only_yaw=1)
    drv = Drive(synth.Scene(42), 2.0)
    b = make_builder(ctx, opts, num_range_data=50, two_stage=1)
    b.set_initial_state(imu_synth.state(drv.t0 - 0.1))
    for k in range(5):
        t1, imu, rows = drv.next()
        feed(b, imu)
        sb, _ = b.state()
        hi, lo, sp, _, _ = b.submap(0)
        ohi, olo = oracle_grids(orc, hi, lo)
        iv = drv.interval()
        r = b.add_range_data(t1, xyzt(rows))
        assert r.has_result == 1 and r.scan.ok == 1
        drv.committed()
        c = oracle_scan(orc, opts, sb, iv, rows, sp, ohi, olo)
        pts, ms = c["pts"], c["ms"]
        hc, lc = pts[ms["hi_keep"]], pts[ms["lo_keep"]]
        pre = orc.rtcsm_match(ohi, hc, c["cur"], opts.rtcsm_linear_window, opts.rtcsm_angular_window, opts.rtcsm_w_t, opts.rtcsm_w_r)
        want, _ = orc.ceres_match([hc, lc], [ohi, olo], [opts.occ_w0, opts.occ_w1], opts.trans_w, opts.rot_w, c["cur"][:3],
                                  pre["pose"], only_yaw=True, max_iter=opts.max_iter)
        got = np.array(r.scan.pose_estimate_local[:])
        dtm, drm = pose_error(got, want)
        assert dtm < 1e-6 and drm < 1e-7, (k, dtm, drm)
        assert bits(r.rtcsm_score) == bits(pre["score"])
        # yaw only: roll and pitch of the matched pose are the pre-match's
        def tilt(q):
            w, x, y, z = q
            return np.array([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)])
        assert np.abs(tilt(got[3:]) - tilt(pre["pose"][3:])).max() < 1e-8
    b.close()
    fo = dliom.FrontendOptions.from_oracle(opts)
    with pytest.raises(dliom.DlError) as e:
        dliom.LocalTrajectoryBuilder(ctx, dliom.LtbOptions.defaults(fo, NOISE, imu_weight=0.7))
    assert e.value.status == DL_ERR_ARG
    ctx.close()
