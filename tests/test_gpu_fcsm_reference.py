"""The device loop-closure coarse matcher (dl_fcsm_match_3dof, dl_constraint_search_batch) against the numpy reference of
tests/fcsm_reference.py, bit for bit: every leaf score, and found, score, offset (lowest index among equal scores),
pose_estimate, low-resolution score and num_candidates, on the pruned search and on the exhaustive one."""
import os
import threading

import numpy as np
import pytest

import fcsm_cases as cases
import fcsm_reference as ref

pytestmark = pytest.mark.gpu

f32 = np.float32
PRUNED_LAUNCHES, EXHAUSTIVE_LAUNCHES = 5, 3     # prepare, bounds, 2 block rounds, finish / prepare, search, finish


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


def search(ctx, hi, lo, case, exhaustive=False, want_scores=False):
    """-> (result, kernel launches of the call)."""
    if exhaustive:
        os.environ["DLIOM_FCSM_EXHAUSTIVE"] = "1"
    try:
        before = ctx.launches
        r = ctx.fcsm_match_3dof(hi, lo, case.hi_points, case.lo_points, case.pose, case.min_score, xy_window=case.xy_window,
                                z_window=case.z_window, min_low_resolution_score=case.min_low, want_scores=want_scores)
        return r, ctx.launches - before
    finally:
        os.environ.pop("DLIOM_FCSM_EXHAUSTIVE", None)


def assert_same(got, want):
    assert bool(got.found) == want.found
    assert got.num_candidates == want.num_candidates
    if not want.found:
        return
    assert f32(got.score).view(np.uint32) == f32(want.score).view(np.uint32)
    assert tuple(got.offset) == want.offset
    assert np.array_equal(np.array(got.pose_estimate[:]).view(np.uint64), want.pose.view(np.uint64))
    assert f32(got.low_resolution_score).view(np.uint32) == f32(want.low_resolution_score).view(np.uint32)


@pytest.mark.parametrize("name", cases.NAMES)
def test_case_equals_reference(ctx, name):
    """Every leaf score from the exhaustive kernel; the answer from the default search (the path the case names, confirmed by
    its launch count) and from the forced exhaustive search."""
    case = cases.get(name)
    want = case.run(all_ties=False)
    hi, lo = device_grid(ctx, case.hi), device_grid(ctx, case.lo)
    (got, scores), _ = search(ctx, hi, lo, case, want_scores=True)
    assert scores.shape == want.scores.shape
    bad = np.flatnonzero(scores.view(np.uint32).reshape(-1) != want.scores.view(np.uint32).reshape(-1))
    assert len(bad) == 0, f"{len(bad)} leaves differ, first at offset {want.offset_of(int(bad[0]))}"
    assert_same(got, want)
    search(ctx, hi, lo, case)                                   # builds the search index once (all_scores does not)
    got, launches = search(ctx, hi, lo, case)
    assert launches == (PRUNED_LAUNCHES if case.path == "pruned" else EXHAUSTIVE_LAUNCHES)
    assert_same(got, want)
    got, launches = search(ctx, hi, lo, case, exhaustive=True)
    assert launches == EXHAUSTIVE_LAUNCHES
    assert_same(got, want)


def test_constraint_search_batch_across_the_chunk(ctx):
    """1 100 pairs of small clouds in two chunks of up to 1 024 pairs: grids of three resolutions (so three windows), cloud
    sizes from 1 to 40, guesses that miss (pruned by min_score). Pair 500 searches an empty grid, so the first chunk runs the
    exhaustive search and the second the pruned one. Every pair equals the reference: found, score, low-resolution score and
    coarse pose; a pair not found reports its own guess as the coarse pose, which pins the guess each pair read."""
    import dliom
    rng = np.random.default_rng(77)
    refs, devs = [], []
    for res in (0.1, 0.15, 0.2):
        hi, lo, _, _ = cases._scatter(int(res * 100), 1, 1, box=(12, 12, 5), density=0.2)
        hi = ref.SparseGrid(res, hi.cells, hi.values)
        refs.append((hi, lo))
        devs.append((device_grid(ctx, hi), device_grid(ctx, lo)))
    empty = (ref.SparseGrid(0.1), refs[0][1])
    empty_dev = (device_grid(ctx, empty[0]), devs[0][1])
    pairs = []
    for k in range(1100):
        s = k % 3
        n_hi, n_lo = int(rng.integers(1, 41)), int(rng.integers(1, 41))
        hp = (rng.uniform(-1, 1, (n_hi, 3)) * [1.0, 1.0, 0.4]).astype(f32)
        lp = (rng.uniform(-1, 1, (n_lo, 3)) * [1.0, 1.0, 0.4]).astype(f32)
        far = k % 7 == 3
        yaw = rng.uniform(-0.1, 0.1)
        guess = np.array([*(rng.uniform(-0.2, 0.2, 3) + (30.0 if far else 0.0)), np.cos(yaw / 2), 0, 0, np.sin(yaw / 2)])
        grids, dev = (empty, empty_dev) if k == 500 else (refs[s], devs[s])
        pairs.append((hp, lp, guess, grids, dev))
    opt = dliom.ConstraintOptions.defaults(min_score=0.2, min_low_resolution_score=0.15, xy_window=0.6, z_window=0.3)
    got = ctx.constraint_search_batch(opt, [p[2] for p in pairs], [p[0] for p in pairs], [p[1] for p in pairs],
                                      [p[4][0] for p in pairs], [p[4][1] for p in pairs])
    found = np.zeros(len(pairs), bool)
    for k, (c, (hp, lp, guess, (hi, lo), _)) in enumerate(zip(got, pairs)):
        want = ref.match_3dof(hi, lo, hp, lp, guess, 0.2, 0.6, 0.3, 0.15)
        assert bool(c.found) == want.found, k
        if want.found:
            found[k] = True
            assert f32(c.score) == want.score and f32(c.low_resolution_score) == want.low_resolution_score, k
            assert np.array_equal(np.array(c.coarse_pose[:]), want.pose), k
        else:
            assert np.array_equal(np.array(c.coarse_pose[:]), ref.pose7_of(*ref.float_pose(guess))), k
    # both chunks hold found pairs and pairs pruned by min_score (every 7th guess is 30 m off)
    assert not found[500] and 500 < found[:1024].sum() < 1024 and 50 < found[1024:].sum() < 76


def test_one_submap_two_contexts_and_changes(ctx):
    """One submap searched from two contexts on two threads; then after set_cells and after a device insert (the search index
    is rebuilt from the grid's version). The reference reads the grid back from the device after the insert."""
    import dliom
    hi_ref, lo_ref, hp, lp = cases._scatter(800, 300, 200)
    hi, lo = device_grid(ctx, hi_ref), device_grid(ctx, lo_ref)
    guesses = [np.array([*np.random.default_rng(k).uniform(-0.3, 0.3, 3), 1, 0, 0, 0]) for k in range(6)]

    def check(hi_ref):
        wants = [ref.match_3dof(hi_ref, lo_ref, hp, lp, g, 0.1, 0.8, 0.4, 0.2) for g in guesses]
        assert any(w.found for w in wants)
        other = dliom.Context(0)
        out = {}
        try:
            def run(name, c):
                out[name] = [c.fcsm_match_3dof(hi, lo, hp, lp, g, 0.1, xy_window=0.8, z_window=0.4, min_low_resolution_score=0.2)
                             for g in guesses]
            threads = [threading.Thread(target=run, args=(n, c)) for n, c in (("a", ctx), ("b", other))]
            for t in threads:
                t.start()
            for t in threads:
                t.join()
        finally:
            other.close()
        for name in ("a", "b"):
            for got, want in zip(out[name], wants):
                assert_same(got, want)

    check(hi_ref)
    cells = np.array([[x, 2, 1] for x in range(-10, 10)], np.int32)
    hi.set_cells(cells[:, 0], cells[:, 1], cells[:, 2], np.full(len(cells), 32767, np.uint16))
    hi_ref = ref.SparseGrid(hi_ref.resolution, np.concatenate([hi_ref.cells, cells]),
                            np.concatenate([hi_ref.values, np.full(len(cells), 32767, np.uint16)]))
    check(hi_ref)
    hi.insert_range_data(np.zeros(3, f32), np.array([[0.5, -0.4, 0.2], [0.9, 0.3, -0.1], [-0.7, 0.2, 0.3]], f32), 0.9, 0.1, 3)
    check(ref.SparseGrid.from_export(hi_ref.resolution, hi.export()))


def test_all_scores_capacity_is_checked(ctx):
    """A score buffer with room for one leaf too few is refused with DL_ERR_ARG before any work; one of the exact size is
    filled."""
    import ctypes as C
    import dliom
    case = cases.get("window_7_3")
    hi, lo = device_grid(ctx, case.hi), device_grid(ctx, case.lo)
    want = case.run(all_ties=False)
    opt = dliom.FcsmOptions(8, 3, 0.77, case.min_low, case.xy_window, case.z_window, 0.26)
    scores = np.zeros(want.num_candidates, f32)
    for capacity, status in ((want.num_candidates - 1, -2), (want.num_candidates, 0)):
        r = dliom.FcsmResult()
        before = ctx.launches
        st = ctx.L.dl_fcsm_match_3dof(ctx.h, C.byref(opt), np.ascontiguousarray(case.pose), case.hi_points, len(case.hi_points),
                                      case.lo_points, len(case.lo_points), hi.h, lo.h, np.float32(case.min_score), C.byref(r),
                                      scores.ctypes.data_as(C.c_void_p), capacity)
        assert st == status and (ctx.launches > before) == (status == 0)
    assert np.array_equal(scores.view(np.uint32), want.scores.reshape(-1).view(np.uint32))
