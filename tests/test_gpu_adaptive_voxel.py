"""The device adaptive voxel filter (dl_voxel.cu) against the oracle, bit for bit (survivor indices and pass edges), on clouds built
to sit on its edges (adaptive_voxel_cases.py: each generator checks with the numpy reference that it lands on its edge), and the
batched front end with pairs of every kind in one launch. Every case runs once on a fresh dliom.Context, and the standalone call
makes exactly one kernel launch (none for an empty cloud)."""
import functools

import numpy as np
import pytest

import adaptive_voxel_cases as K
import adaptive_voxel_reference as R
from helpers import workload

pytestmark = pytest.mark.gpu

f32 = np.float32
CASES = K.all_cases()


@functools.lru_cache(maxsize=None)
def oracle(name):
    case = next(c for c in CASES if c.name == name)
    return tuple(np.asarray(x) for x in __import__("orc").adaptive_voxel_filter(case.rows, *case.opts))


def run(case):
    """-> (survivors, pass edges, kernel launches of the call) on a fresh context."""
    import dliom
    ctx = dliom.Context(0)
    try:
        before = ctx.launches
        keep, passes = ctx.adaptive_voxel_filter(case.rows, *case.opts)
        return keep, passes, ctx.launches - before
    finally:
        ctx.close()


def check(case, want_keep, want_passes):
    keep, passes, launches = run(case)
    assert launches == (1 if len(case.rows) else 0)
    assert np.array_equal(passes.view(np.uint32), np.asarray(want_passes, f32).view(np.uint32)), (passes, want_passes)
    assert np.array_equal(keep, want_keep)


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_device_matches_the_oracle(orc, case):
    want_keep, want_passes = oracle(case.name)
    check(case, want_keep, want_passes)


@pytest.mark.parametrize("which", [0, 1], ids=["shuffled_street_scan_high_resolution", "shuffled_street_scan_low_resolution"])
def test_device_matches_the_oracle_on_a_shuffled_street_scan(orc, which):
    case = K.street_cases(orc)[which]
    want_keep, want_passes = orc.adaptive_voxel_filter(case.rows, *case.opts)
    check(case, want_keep, want_passes)


# ------------------------------------------------------------------------------------------- batched front end
# A 5 cm first voxel filter leaves ~18 000 returns per 16-beam sweep. High-resolution filter 2 m / 300 / 15 m, low-resolution
# filter 10 cm / 200 / 60 m. Per scan, in a period of five: a sweep (high: bisection, 120 to 210 voxels at 2 m; low: ~11 000 voxels at
# 10 cm, far beyond the search's result table), the same sweep scaled by 0.3 toward the sensor (high: bisection; low: first edge
# sufficient), twice, and the first 150 rows of a sweep (sparse enough for both).
def batch_scans(w, count):
    scans, prev, cur = [], [], []
    for i in range(count):
        rows = w["scans"][i].copy()
        kind = i % 5
        if kind in (1, 3):
            for c in "xyz":
                rows[c] *= np.float32(0.3)
        elif kind == 4:
            rows = rows[:150].copy()
        scans.append(rows)
        prev.append(w["prev"][i])
        cur.append(w["cur"][i])
    return scans, np.array(prev), np.array(cur)


def pair_kind(pts, max_length, min_num_points, max_range):
    c = R.xyz(pts)[R.crop(pts, max_range)]
    if f32(len(c)) <= f32(min_num_points):
        return "sparse"
    v = R.num_voxels(c, max_length)
    if v > 8192:
        return "first_edge_over_8192_voxels"
    return "first_edge" if f32(v) >= f32(min_num_points) else "bisection"


@functools.lru_cache(maxsize=None)
def batch_case():
    import orc
    w = workload(num_scans=42)
    opts = orc.FrontEndOptions.defaults(voxel_filter_size=0.05, hi_max_length=2.0, hi_min_num_points=300, hi_max_range=15.0,
                                        lo_max_length=0.1, lo_min_num_points=200, lo_max_range=60.0)
    scans, prev, cur = batch_scans(w, 40)
    filters = ((opts.hi_max_length, opts.hi_min_num_points, opts.hi_max_range),
               (opts.lo_max_length, opts.lo_min_num_points, opts.lo_max_range))
    want, kinds = [], []
    for s in range(len(scans)):
        ing = orc.ingest_scan(opts, scans[s], w["origin"], prev[s], cur[s])
        pts = ing["returns_tracking"]
        m = orc.match_scan(opts, pts, ing["current_pose"].astype(np.float64), w["submap_pose"], w["hi"], w["lo"])
        row = {"pose": m["pose_estimate_local"], "iterations": m["summary"]["num_iterations"], "ok": m["ok"]}
        for tag, f in zip(("high", "low"), filters):
            keep, passes = orc.adaptive_voxel_filter(pts, *f)
            row[tag] = (len(R.crop(pts, f[2])), len(passes), len(keep))
        want.append(row)
        kinds.append(tuple(pair_kind(pts, *f) for f in filters))
    # every five consecutive scans (any launch of at least five) hold pairs of all four kinds
    for s in range(len(scans) - 4):
        assert {k for ks in kinds[s:s + 5] for k in ks} == {"sparse", "first_edge", "bisection", "first_edge_over_8192_voxels"}, \
            kinds
    return w, opts, scans, prev, cur, want


def counts(r):
    return (r.ok, r.num_cropped_high, r.num_passes_high, r.num_high_resolution, r.num_cropped_low, r.num_passes_low,
            r.num_low_resolution, r.summary.num_iterations)


def rotation_error(qa, qb):
    """Angle [rad] between two unit quaternions, to first order 2 |qa - qb| (signs aligned). helpers.pose_error takes
    2 arccos(|qa . qb|), which cannot resolve less than 2 arccos(1 - 2^-53) = 2.1e-8 rad."""
    qa, qb = qa / np.linalg.norm(qa), qb / np.linalg.norm(qb)
    return 2 * np.linalg.norm(qa - np.sign(np.dot(qa, qb)) * qb)


def check_against_oracle(results, want):
    for s, (r, wnt) in enumerate(zip(results, want)):
        assert r.ok == 1 and wnt["ok"], s
        assert (r.num_cropped_high, r.num_passes_high, r.num_high_resolution) == wnt["high"], s
        assert (r.num_cropped_low, r.num_passes_low, r.num_low_resolution) == wnt["low"], s
        assert r.summary.num_iterations == wnt["iterations"], s
        got = np.array(r.pose_estimate_local)
        dt = np.linalg.norm(got[:3] - wnt["pose"][:3])
        assert dt < 1e-7 and rotation_error(got[3:], wnt["pose"][3:]) < 1e-8, (s, dt, rotation_error(got[3:], wnt["pose"][3:]))


def repeat_identical(ctx, call, first, calls):
    """`calls` more batch calls on `ctx`: identical results. Returns the set of kernel launch counts per call."""
    launches = set()
    for _ in range(calls):
        before = ctx.launches
        again = call()
        launches.add(ctx.launches - before)
        for a, b in zip(again, first):
            assert list(a.pose_estimate_local) == list(b.pose_estimate_local) and counts(a) == counts(b)
    return launches


def test_frontend_batch_pairs_of_every_kind_against_the_oracle_with_steady_launches(orc):
    """Host scans (5 sub-batches per call) and device-resident scans (2 per call), 40 scans: every pair's cropped size, pass
    count and survivor count against the oracle, the pose within 1e-7 m / 1e-8 rad of orc.match_scan with the same iteration
    count; then 4 (host) and 8 (device) more calls on the same context, i.e. 20 and 16 more sub-batch launches, which must
    repeat every pose and count bit for bit with the same number of kernel launches."""
    import ctypes as C
    import dliom
    w, opts, scans, prev, cur, want = batch_case()
    fo = dliom.FrontendOptions.from_oracle(opts)

    ctx = dliom.Context(0)
    hi, lo = dliom.Grid.from_oracle(ctx, w["hi"]), dliom.Grid.from_oracle(ctx, w["lo"])
    args = (w["origin"], prev, cur, w["submap_pose"], hi, lo)
    before = ctx.launches
    first = ctx.frontend_match_batch(fo, scans, *args)
    launches = {ctx.launches - before}
    check_against_oracle(first, want)
    launches |= repeat_identical(ctx, lambda: ctx.frontend_match_batch(fo, scans, *args), first, 4)
    assert len(launches) == 1, launches
    ctx.close()

    ctx = dliom.Context(0)
    hi, lo = dliom.Grid.from_oracle(ctx, w["hi"]), dliom.Grid.from_oracle(ctx, w["lo"])
    sizes = np.array([len(s) for s in scans], np.int64)
    cap = int(sizes.max())
    rows = np.zeros((len(scans), cap, 8), np.float32)
    for b, sc in enumerate(scans):
        rows[b, :len(sc)] = sc.view(np.float32).reshape(-1, 8)
    d_rows = ctx.device_alloc(rows.nbytes)
    d_res = ctx.device_alloc(len(scans) * C.sizeof(dliom.ScanResult))
    ctx.copy_to_device(d_rows, rows)

    def dev():
        ctx.frontend_match_batch_dev(fo, d_rows, cap, sizes, w["origin"], prev, cur, w["submap_pose"], hi, lo, d_res)
        return ctx.fetch_results(d_res, len(scans))

    first_dev = dev()
    check_against_oracle(first_dev, want)
    for a, b in zip(first_dev, first):
        assert list(a.pose_estimate_local) == list(b.pose_estimate_local) and counts(a) == counts(b)
    assert len(repeat_identical(ctx, dev, first_dev, 8)) == 1
    for p in (d_rows, d_res):
        ctx.device_free(p)
    ctx.close()
