"""The device correlative scan matcher (dl_rtcsm_match and the front end's pre-match) against the numpy reference of
tests/rtcsm_reference.py, bit for bit: every candidate score (but the exp-ambiguous ones, which are counted), the best index,
score and pose, and the window."""
import ctypes as C

import numpy as np
import pytest

import rtcsm_cases as cases
import rtcsm_reference as ref
from helpers import pose_error, workload

pytestmark = pytest.mark.gpu

f32 = np.float32


@pytest.fixture(scope="module")
def ctx():
    import dliom
    c = dliom.Context(0)
    yield c
    c.close()


def device_grid(ctx, g):
    import dliom
    d = dliom.Grid(ctx, g.resolution)
    if len(g.cells):
        d.set_cells(*g.export())
    else:
        d.sync()
    return d


def assert_equals_reference(got, c):
    m = c.result
    assert (got["linear"], got["angular"]) == (m.window.linear, m.window.angular)
    assert got["angular_step"].view(np.uint32) == f32(m.window.step).view(np.uint32)
    assert got["max_scan_range"].view(np.uint32) == f32(m.window.max_scan_range).view(np.uint32)
    assert got["num_candidates"] == m.num_candidates
    differ = got["scores"].view(np.uint32) != m.scores.view(np.uint32)
    ambiguous = m.ambiguous()
    bad = np.flatnonzero(differ & ~ambiguous)
    assert len(bad) == 0, f"{len(bad)} scores differ, first at index {bad[0]}"
    if differ.any():
        print(f"{c.name}: {int(differ.sum())} of {int(ambiguous.sum())} exp-ambiguous scores differ")
    assert got["best_index"] == m.best_index
    assert got["score"].view(np.uint32) == m.score.view(np.uint32)
    assert np.array_equal(got["pose"], m.pose)


@pytest.mark.parametrize("name", cases.NAMES)
def test_case_equals_reference(ctx, name):
    c = cases.get(name)
    got = ctx.rtcsm_match(device_grid(ctx, c.grid), *c.args, want_scores=True)
    assert_equals_reference(got, c)


@pytest.mark.parametrize("history", ["fresh", "after_large_call"])
def test_far_point_does_not_depend_on_history(history):
    """A farthest point between 200 m and the acosf cliff widens the angular window beyond what a 200 m bound assumes; the call
    must succeed on a fresh context and on one whose scratch a larger call has grown."""
    import dliom
    c = cases.get("far_250m")
    ctx = dliom.Context(0)
    try:
        if history == "after_large_call":
            big = cases.get("shape_L3_A2")
            ctx.rtcsm_match(device_grid(ctx, big.grid), *big.args, want_scores=True)
        got = ctx.rtcsm_match(device_grid(ctx, c.grid), *c.args, want_scores=True)
        assert_equals_reference(got, c)
        again = ctx.rtcsm_match(device_grid(ctx, c.grid), *c.args)
        assert again["best_index"] == c.result.best_index
    finally:
        ctx.close()


# ----------------------------------------------------------------------------------------------- the front end's pre-match
def _crop(rows, radius):
    xyz = rows.view(np.float32).reshape(-1, 8)[:, :3]
    return rows[np.linalg.norm(xyz, axis=1) <= radius].copy()


def _cluster_rows(orc, points, t=0.0):
    xyzt = np.column_stack([np.asarray(points, np.float32), np.full(len(points), t, np.float32)])
    return orc.make_ranges(xyzt)


def _frontend_case(orc, opts):
    """Six scans on the 16-beam drive's high-resolution grid: four drive scans cropped at different radii (several R in one
    launch), one whose returns all lie beyond the high-resolution filter's range (empty cloud), and a small cluster near the
    sensor in unknown space, where every candidate reads 0.1 and (zero weights) all tie."""
    w = workload()
    s = w["scans"]
    far = _crop(s[1], 60.0)
    far = far[np.linalg.norm(far.view(np.float32).reshape(-1, 8)[:, :3], axis=1) >= 18.0]
    cluster = _cluster_rows(orc, [[0.22, 0.0, 0.01], [0.0, 0.21, 0.02], [-0.2, 0.03, 0.0], [0.02, -0.22, 0.05],
                                  [0.1, 0.1, 0.21]], -0.05)
    scans = [_crop(s[0], 6.0), far, _crop(s[2], 11.0), s[3], _crop(s[1], 8.5), cluster]
    prev = np.array([w["prev"][0], w["prev"][1], w["prev"][2], w["prev"][3], w["prev"][1], w["prev"][0]])
    cur = np.array([w["cur"][0], w["cur"][1], w["cur"][2], w["cur"][3], w["cur"][1], w["cur"][0]])
    want = []
    for b, rows in enumerate(scans):
        ing = orc.ingest_scan(opts, rows, w["origin"], prev[b], cur[b])
        pred = ing["current_pose"].astype(np.float64)
        m = orc.match_scan(opts, ing["returns_tracking"], pred, w["submap_pose"], w["hi"], w["lo"])
        hi_cloud = ing["returns_tracking"][m["hi_keep"]]
        r = None
        if len(hi_cloud):
            q = pred[3:] / np.sqrt((pred[4] * pred[4] + pred[5] * pred[5]) + (pred[6] * pred[6] + pred[3] * pred[3]))
            init = np.concatenate([pred[:3], q])            # submap pose identity: compose() renormalises in double
            grid = ref.SparseGrid.from_export(w["hi"].resolution, w["hi"].export())
            r = ref.match(grid, hi_cloud, init, opts.rtcsm_linear_window, opts.rtcsm_angular_window, opts.rtcsm_w_t,
                          opts.rtcsm_w_r)
        want.append((m, r))
    return w, scans, prev, cur, want


@pytest.mark.parametrize("parity", ["odd", "even"])
def test_frontend_prematch_equals_reference(ctx, orc, parity):
    """dl_frontend_match_batch_dev with an odd cap_rows (every other cloud 8 bytes off a 16-byte boundary) and an even one:
    every scan's rtcsm_score equals the reference on its high-resolution cloud, and the solved pose the oracle's."""
    import dliom
    opts = orc.FrontEndOptions.defaults(use_rtcsm=1, min_range=0.0, rtcsm_w_t=0.0, rtcsm_w_r=0.0)
    w, scans, prev, cur, want = _frontend_case(orc, opts)
    rs = [r for _, r in want if r is not None]
    assert len({r.window.angular for r in rs}) >= 3                         # several R in one launch
    assert want[1][1] is None and want[1][0]["hi_keep"].size == 0             # the empty high-resolution cloud
    tie = want[5][1]
    assert len(tie.tied()) == tie.num_candidates and tie.best_index == 0     # the tie scan
    fo = dliom.FrontendOptions.from_oracle(opts)
    hi, lo = device_grid(ctx, ref.SparseGrid.from_export(w["hi"].resolution, w["hi"].export())), dliom.Grid.from_oracle(ctx, w["lo"])
    sizes = np.array([len(s) for s in scans], np.int64)
    cap = int(sizes.max())
    cap += (cap % 2 == 0) if parity == "odd" else (cap % 2 == 1)
    rows = np.zeros((len(scans), cap, 8), np.float32)
    for b, sc in enumerate(scans):
        rows[b, :len(sc)] = sc.view(np.float32).reshape(-1, 8)
    d_rows = ctx.device_alloc(rows.nbytes)
    d_res = ctx.device_alloc(len(scans) * C.sizeof(dliom.ScanResult))
    try:
        ctx.copy_to_device(d_rows, rows)
        ctx.frontend_match_batch_dev(fo, d_rows, cap, sizes, w["origin"], prev, cur, w["submap_pose"], hi, lo, d_res)
        res = ctx.fetch_results(d_res, len(scans))
    finally:
        for p in (d_rows, d_res):
            ctx.device_free(p)
    for b, (r, (m, mine)) in enumerate(zip(res, want)):
        assert r.num_high_resolution == len(m["hi_keep"]), b
        if mine is None:
            assert r.rtcsm_score == 0, b
            continue
        assert f32(r.rtcsm_score).view(np.uint32) == mine.score.view(np.uint32) == f32(m["rtcsm_score"]).view(np.uint32), b
        assert m["ok"] and r.ok == 1, b
        dt, dr = pose_error(np.array(r.pose_estimate_local), m["pose_estimate_local"])
        assert dt < 1e-7 and dr < 1e-8, (b, dt, dr)


def test_frontend_prematch_range_floor(ctx, orc):
    """A cloud entirely within 3 resolutions of the sensor: max_scan_range is the 3 * resolution floor. The angular window is
    chosen so that the floor decides A (2 at the floor, 1 at the cloud's own extent); with every score tied, index 0 (the
    corner candidate) is the solve's start, so the pose shows which window ran."""
    import dliom
    opts = orc.FrontEndOptions.defaults(use_rtcsm=1, min_range=0.0, rtcsm_w_t=0.0, rtcsm_w_r=0.0)
    w = workload()
    res = w["hi"].resolution
    rows = _cluster_rows(orc, [[0.22, 0.0, 0.01], [0.0, 0.21, 0.02], [-0.2, 0.03, 0.0], [0.02, -0.22, 0.05],
                               [0.1, 0.1, 0.21]], -0.05)
    ing = orc.ingest_scan(opts, rows, w["origin"], w["prev"][0], w["cur"][0])
    hi_keep = orc.match_scan(opts, ing["returns_tracking"], ing["current_pose"].astype(np.float64), w["submap_pose"], w["hi"],
                             w["lo"])["hi_keep"]
    hi_cloud = ing["returns_tracking"][hi_keep]
    s_floor = np.float64(ref.angular_step(res, f32(3.0) * f32(res)))
    s_own = np.float64(ref.angular_step(res, ref.norm(hi_cloud).max()))
    opts.rtcsm_angular_window = 0.75 * (s_floor + s_own)
    floor = ref.window(hi_cloud, res, 0.15, opts.rtcsm_angular_window)
    own = ref.round_to_int_double(opts.rtcsm_angular_window / s_own)
    assert floor.max_scan_range == f32(3.0) * f32(res) and floor.angular == 2 and own == 1
    m = orc.match_scan(opts, ing["returns_tracking"], ing["current_pose"].astype(np.float64), w["submap_pose"], w["hi"], w["lo"])
    fo = dliom.FrontendOptions.from_oracle(opts)
    hi, lo = dliom.Grid.from_oracle(ctx, w["hi"]), dliom.Grid.from_oracle(ctx, w["lo"])
    r = ctx.frontend_match_batch(fo, [rows], w["origin"], w["prev"][:1], w["cur"][:1], w["submap_pose"], hi, lo)[0]
    assert f32(r.rtcsm_score) == f32(m["rtcsm_score"]) and m["ok"] and r.ok == 1
    dt, dr = pose_error(np.array(r.pose_estimate_local), m["pose_estimate_local"])
    assert dt < 1e-7 and dr < 1e-8, (dt, dr)
