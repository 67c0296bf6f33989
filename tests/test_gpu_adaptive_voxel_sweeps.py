"""The single-CTA search of the device adaptive voxel filter (adaptive_voxel_kernel in dl_voxel.cu) on the limits of its counting
sweeps, bit for bit against the oracle (survivors and pass edges). Each sweep streams the cloud and counts the voxels of a few edges
on byte maps over the cloud's cell box; the search replays on the stored counts, and an edge it asks for that was not counted costs
one more sweep. Every generator checks with the numpy reference (adaptive_voxel_reference.py) that its cloud lands where its name
says. Every standalone call is one launch of the search.

The limits:
  MAP_BYTES     32 768  cells of byte map per sweep; an edge whose box alone is larger sends the pair to generic mode
  RESULT_SLOTS   2 048  voxels of the result table at the result edge; more send the pair to generic mode
A sweep that counts an edge still halving also counts the next halving e/2 and the midpoint (e/2 + e)/2, as far as they fit."""
import functools

import numpy as np
import pytest

import adaptive_voxel_cases as K
import adaptive_voxel_reference as R

f32 = np.float32
MAP_BYTES = 32768
RESULT_SLOTS = 2048


def line_case(name, cells, voxels, opts=(1.0, 150.0, 1e5)):
    """`voxels` points on the x axis at the integers 0, ..., cells - 1 (both ends included): at the first edge 1 m the cell box is
    cells x 1 x 1 and every point is its own voxel, which suffices."""
    ks = np.unique(np.concatenate([[0, cells - 1], np.linspace(0, cells - 1, voxels).round()])).astype(np.int64)
    pts = np.zeros((len(ks), 3), f32)
    pts[:, 0] = ks
    pts = pts[np.random.RandomState(cells).permutation(len(pts))]
    case = K.Case(name, pts, opts)
    keep, passes, edge = R.search(pts, *opts)
    assert R.cell_box(pts, opts[0]) == (cells, 1, 1) and passes.tolist() == [opts[0]] and len(keep) == len(pts)
    return case


def budget_cases():
    return [line_case("map_budget_exactly_full", MAP_BYTES, 1000), line_case("map_budget_one_cell_over", MAP_BYTES + 1, 1000)]


def result_table_case(voxels):
    """`voxels` occupied cells of a 64 x 64 plane at 1 m, three points each in shuffled order: the first edge suffices."""
    rng = np.random.RandomState(voxels)
    grid = np.stack(np.meshgrid(np.arange(64), np.arange(64), indexing="ij"), -1).reshape(-1, 2)
    cells = grid[rng.choice(len(grid), voxels, replace=False)]
    pts = np.zeros((3 * voxels, 3), f32)
    pts[:, :2] = np.repeat(cells, 3, axis=0) + rng.uniform(-0.4, 0.4, (3 * voxels, 2))
    pts = pts[rng.permutation(len(pts))]
    opts = (1.0, 150.0, 1e3)
    keep, passes, _ = R.search(pts, *opts)
    assert passes.tolist() == [1.0] and len(keep) == voxels and np.prod(R.cell_box(pts, 1.0)) <= MAP_BYTES
    return K.Case(f"result_table_{voxels}_voxels", pts, opts)


def plane_case(name, side, target_passes, min_from):
    """8 000 uniform points on a side x side plane; min_num_points = the voxel count at edge `min_from`, so that the search walks
    exactly `target_passes` (edges as multiples of max_length 1)."""
    rng = np.random.RandomState(int(side * 7))
    pts = np.zeros((8000, 3), f32)
    pts[:, :2] = rng.uniform(0, side, (len(pts), 2))
    opts = (1.0, float(R.num_voxels(pts, f32(min_from))), 1e3)
    keep, passes, _ = R.search(pts, *opts)
    assert passes.tolist() == [f32(e) for e in target_passes], passes
    assert len(keep) <= RESULT_SLOTS and np.prod(R.cell_box(pts, passes.min())) <= MAP_BYTES
    return K.Case(name, pts, opts)


def bisection_cases():
    # [L/2, L]: always too few -> towards L/2, four midpoints; always enough -> towards L, three. The first midpoint 3L/4 is
    # counted with L and L/2, every later one costs a sweep of its own.
    low_path = [1.0, 0.5, 0.75, 0.625, 0.5625, 0.53125]
    high_path = [1.0, 0.5, 0.75, 0.875, 0.9375]
    return [plane_case("deepest_low_path", 20.0, low_path, 0.5), plane_case("deepest_high_path", 30.0, high_path, 0.9375)]


def exhausted_case():
    """Three voxels, min_num_points 150: every halving falls short and the search runs out at L/128 (sweeps of {e, e/2, 3e/4})."""
    pts = np.repeat(np.array([[1.0, -2.0, 0.5], [3.0, 1.0, 0.0], [-2.0, 2.0, 1.0]], f32), 700, axis=0)
    pts = pts[np.random.RandomState(5).permutation(len(pts))]
    opts = (2.0, 150.0, 15.0)
    keep, passes, edge = R.search(pts, *opts)
    assert len(passes) == 8 and edge == passes[-1] == f32(2.0) / 128 and len(keep) == 3
    return K.Case("three_voxels_exhaust_the_search", pts, opts)


def cases():
    return budget_cases() + [result_table_case(RESULT_SLOTS), result_table_case(RESULT_SLOTS + 1)] + bisection_cases() + \
        [exhausted_case()]


CASES = cases()


def test_the_reference_and_the_oracle_agree_on_the_sweep_clouds(orc):
    for case in CASES:
        keep, passes = R.adaptive_voxel_filter(case.rows, *case.opts)
        want_keep, want_passes = orc.adaptive_voxel_filter(case.rows, *case.opts)
        assert np.array_equal(keep, want_keep) and np.array_equal(np.asarray(want_passes, f32).view(np.uint32),
                                                                   passes.view(np.uint32)), case.name


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_device_matches_the_oracle_on_the_sweep_limits(orc, case):
    import dliom
    want_keep, want_passes = orc.adaptive_voxel_filter(case.rows, *case.opts)
    ctx = dliom.Context(0)
    try:
        before = ctx.launches
        keep, passes = ctx.adaptive_voxel_filter(case.rows, *case.opts)
        assert ctx.launches - before == 1
    finally:
        ctx.close()
    assert np.array_equal(passes.view(np.uint32), np.asarray(want_passes, f32).view(np.uint32)), (passes, want_passes)
    assert np.array_equal(keep, want_keep)


# ------------------------------------------------------------------------------------------- the benchmark's shape
@functools.lru_cache(maxsize=None)
def bench_shape_batch():
    """74 64-beam sweeps over the first 1.3 s of the stretch that bench.py registers, under the front end's default filters
    (2 m / 150 / 15 m and 4 m / 200 / 60 m): every pair of both filters needs the bisection, as in one sub-batch of bench.py
    (further along the stretch, some high-resolution pairs stop at the first edge)."""
    import orc
    import synth
    from helpers import workload
    w = workload()  # the submap grids; the sweeps are made here
    scene = synth.Scene(42)
    opts = orc.FrontEndOptions.defaults()
    filters = ((opts.hi_max_length, opts.hi_min_num_points, opts.hi_max_range),
               (opts.lo_max_length, opts.lo_min_num_points, opts.lo_max_range))
    times = [2.05 + 1.3 * j / 74 for j in range(74)]
    scans = [synth.make_scan(scene, 64, t) for t in times]
    prev = np.array([synth.pose7(t - 0.1) for t in times])
    cur = np.array([synth.pose7(t) for t in times])
    want = []
    for s in range(74):
        pts = orc.ingest_scan(opts, scans[s], w["origin"], prev[s], cur[s])["returns_tracking"]
        row = []
        for f in filters:
            keep, passes = orc.adaptive_voxel_filter(pts, *f)
            c = R.xyz(pts)[R.crop(pts, f[2])]
            assert f32(len(c)) > f32(f[1]) and f32(R.num_voxels(c, f[0])) < f32(f[1]) and len(passes) > 2, (s, f)
            row.append((len(c), len(passes), len(keep)))
        want.append(row)
    return w, opts, scans, prev, cur, want


@pytest.mark.gpu
def test_bench_shape_batch_every_pair_bisects(orc):
    """Cropped size, pass count and survivor count of all 148 pairs of the batch against the oracle."""
    import dliom
    w, opts, scans, prev, cur, want = bench_shape_batch()
    ctx = dliom.Context(0)
    try:
        hi, lo = dliom.Grid.from_oracle(ctx, w["hi"]), dliom.Grid.from_oracle(ctx, w["lo"])
        res = ctx.frontend_match_batch(dliom.FrontendOptions.from_oracle(opts), scans, w["origin"], prev, cur, w["submap_pose"],
                                       hi, lo)
    finally:
        ctx.close()
    for s, (r, wnt) in enumerate(zip(res, want)):
        assert (r.num_cropped_high, r.num_passes_high, r.num_high_resolution) == wnt[0], s
        assert (r.num_cropped_low, r.num_passes_low, r.num_low_resolution) == wnt[1], s
