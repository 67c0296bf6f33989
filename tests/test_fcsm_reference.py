"""The numpy reference of the loop-closure coarse matcher (fcsm_reference) against hand-worked answers, the C++ oracle's branch
and bound against it on every case of fcsm_cases, and the literal restatement of the reference's branch and bound against the
exhaustive maximum (the admissibility of its bounds)."""
import numpy as np
import pytest

import fcsm_cases as cases
import fcsm_reference as ref

f32 = np.float32
SMALL = [n for n in cases.NAMES if n not in cases.NOT_SMALL]
# The reference's PrecomputeGrid writes cells up to 3 below the data at full resolution: data within 3 cells of -8 192 grows
# its grid past the +-8 192 limit, a CHECK failure (the oracle stops there too). The device has no such grid; those cases are
# pinned to the numpy reference only.
ORACLE = [n for n in cases.NAMES if n not in cases.NOT_IN_ORACLE]


def _grid(res, cells, values):
    return ref.SparseGrid(res, np.asarray(cells).reshape(-1, 3), np.asarray(values, np.uint16))


# ----------------------------------------------------------------------------------------------- hand-worked answers
def test_precomputation_values_hand_worked():
    assert ref.LUT[0] == 0 and ref.LUT[1] == 0 and ref.LUT[32767] == 255
    assert ref.LUT[5462] == 43                  # (p - 0.1) * 255 / 0.8 is exactly 42.5 here: rounds away from zero
    assert (np.diff(ref.LUT[1:]) >= 0).all() and set(ref.LUT[1:].tolist()) == set(range(256))


def test_window_rounding_hand_worked():
    r = float(f32(0.1))
    assert ref.window(5.0, 1.0, 0.1) == (50, 10)
    assert ref.window(np.nextafter(0.5 * r, 0.0), 0.5 * r, 0.1) == (0, 1)
    assert ref.lround_double(0.49999999999999994) == 0 and ref.lround_double(0.5) == 1 and ref.lround_double(2.5) == 3


def test_one_point_hand_worked():
    """One point at the origin, one cell of value 32 767 at (2, 0, 0): the leaf (2, 0, 0) scores 0.1 + 255 * 0.8 / 255."""
    hi = _grid(0.1, [[2, 0, 0]], [32767])
    lo = _grid(0.5, [[0, 0, 0]], [32767])
    m = ref.match_3dof(hi, lo, np.zeros((1, 3), f32), np.zeros((1, 3), f32), cases.IDENTITY, 0.5, 0.3, 0.1, 0.5, all_ties=True)
    assert m.found and m.offset == (2, 0, 0) and m.tied == [m.index_of((2, 0, 0))]
    assert m.score == f32(0.1) + f32(255.0) * ((f32(0.9) - f32(0.1)) / f32(255.0))
    assert np.array_equal(m.pose, np.array([f32(0.1) * f32(2.0), 0, 0, 1, 0, 0, 0], np.float64))
    assert m.low_resolution_score == ref.value_to_probability(32767)       # lo cell round(0.2 / 0.5) = 0
    assert m.num_candidates == 7 * 7 * 3 and (m.wxy, m.wz) == (3, 1)
    assert (np.sort(m.scores.reshape(-1))[:-1] == f32(0.1)).all()


def test_three_points_hand_worked():
    """Points at cells (0, 0, 0), (0, 1, 0), (0, 5, 0); cell (1, 0, 0) = 255, cell (1, 1, 0) = 128: the leaf (1, 0, 0) sums
    383 over 3 points, the leaf (1, -1, 0) 255."""
    v128 = int(np.flatnonzero(ref.LUT == 128)[0])
    hi = _grid(0.1, [[1, 0, 0], [1, 1, 0]], [32767, v128])
    pts = np.array([[0, 0, 0], [0, 0.1, 0], [0, 0.5, 0]], f32)
    lo = _grid(0.5, [[0, 0, 0]], [32767])
    m = ref.match_3dof(hi, lo, pts, pts, cases.IDENTITY, 0.1, 0.3, 0.0, 0.0)
    step = (f32(0.9) - f32(0.1)) / f32(255.0)
    assert m.offset == (1, 0, 0) and m.score == f32(0.1) + (f32(383.0) / f32(3.0)) * step
    assert m.scores[0, 2, 4] == f32(0.1) + (f32(255.0) / f32(3.0)) * step            # leaf (1, -1, 0)
    hit, empty = ref.value_to_probability(32767), ref.value_to_probability(0)     # lo cells (0, 0, 0), (0, 0, 0), (0, 1, 0)
    assert m.low_resolution_score == f32(f32(f32(hit + hit) + empty) / f32(3.0))


def test_tie_and_gate_hand_worked():
    m = cases.symmetric_ties().run()
    assert m.offset == (0, -3, 0) and sorted(m.offset_of(i) for i in m.tied) == [(-3, 0, 0), (0, -3, 0), (0, 3, 0), (3, 0, 0)]
    m = cases.tie_gate().run()
    assert m.offset == (4, 0, 0) and [m.offset_of(i) for i in m.rejected] == [(-4, 0, 0)]
    assert m.low_resolution_score == ref.value_to_probability(32767)
    lo_fail = _grid(0.5, [[3, 0, 0]], [32767])
    c = cases.tie_gate()
    assert not ref.match_3dof(c.hi, lo_fail, c.hi_points, c.lo_points, c.pose, 0.85, 0.6, 0.2, 0.5).found


def test_low_resolution_sum_is_sequential_float():
    """The gate adds in float, in point order: 3 000 probabilities whose float sum differs from the float64 sum."""
    c = cases.get("cloud_hi64_lo3000")
    m = c.run(all_ties=False)
    t, q = ref.candidate_pose(c.pose, c.hi.resolution, m.offset)
    probs = ref.value_to_probability(c.lo.lookup(ref.cell_index(ref.transform(c.lo_points, t, q), c.lo.resolution)))
    acc = f32(0)
    for p in probs:
        acc = f32(acc + p)
    assert m.low_resolution_score == f32(acc / f32(3000))


# ----------------------------------------------------------------------------------------------- the oracle
def test_case_classes():
    """The cases the oracle skips are exactly those with data within 3 cells of -8 192, and the small ones are small."""
    for name in cases.NAMES:
        c = cases.get(name)
        assert (name in cases.NOT_IN_ORACLE) == (len(c.hi.cells) > 0 and c.hi.cells.min() < -8192 + 3), name
        assert (name in cases.NOT_SMALL) == (not c.small), name


@pytest.mark.parametrize("name", ORACLE)
def test_oracle_equals_reference(orc, name):
    """The oracle's precomputation stack and branch and bound (stock depth 8 / full depth 3): found, score, low-resolution
    score and pose bits; the offset exactly where the best score is unique, else one of the tied leaves that pass the gate."""
    case = cases.get(name)
    want = case.run()
    hi, lo = orc.Grid(case.hi.resolution), orc.Grid(case.lo.resolution)
    hi.set_cells(*case.hi.export())
    lo.set_cells(*case.lo.export())
    got = orc.fcsm_match_3dof(hi, lo, case.hi_points, case.lo_points, case.pose, case.min_score, xy_window=case.xy_window,
                              z_window=case.z_window, min_low_resolution_score=case.min_low)
    assert bool(got.found) == want.found
    if not want.found:
        return
    assert f32(got.score) == want.score
    assert want.index_of(tuple(got.offset)) in want.tied
    if len(want.tied) == 1:
        assert tuple(got.offset) == want.offset
    t, q = ref.candidate_pose(case.pose, case.hi.resolution, tuple(got.offset))
    assert np.array_equal(np.array(got.pose[:]), ref.pose7_of(t, q))
    assert f32(got.low_resolution_score) == ref.low_resolution_score(case.lo, case.lo_points, t, q)
    assert got.leaves_scored <= want.num_candidates


# ----------------------------------------------------------------------------------------------- the literal branch and bound
SHAPES = [(8, 3), (6, 6), (5, 2), (4, 1), (3, 3), (1, 1)]


@pytest.mark.parametrize("name", SMALL)
def test_branch_and_bound_is_exact_at_stock_depth(name):
    """The reference's search as written (depth 8, full-resolution depth 3: five half-resolution levels) returns the best
    leaf that passes the gate, i.e. the exhaustive answer up to ties."""
    case = cases.get(name)
    want = case.run()
    got, leaves = ref.branch_and_bound(case.hi, case.lo, case.hi_points, case.lo_points, case.pose, case.min_score,
                                       case.xy_window, case.z_window, case.min_low, depth=8, full_depth=3)
    assert got.found == want.found
    if want.found:
        assert got.score == want.score and want.index_of(got.offset) in want.tied
        assert leaves <= want.num_candidates


@pytest.mark.parametrize("shape", SHAPES[1:], ids=[f"d{d}_f{f}" for d, f in SHAPES[1:]])
def test_branch_and_bound_is_exact_at_other_depths(shape):
    depth, full = shape
    for case in [cases.get(n) for n in SMALL if n.startswith(("brick_rows", "cloud_hi", "window_", "round_one", "gate_", "margin"))][::3]:
        want = case.run()
        got, _ = ref.branch_and_bound(case.hi, case.lo, case.hi_points, case.lo_points, case.pose, case.min_score,
                                      case.xy_window, case.z_window, case.min_low, depth=depth, full_depth=full)
        assert got.found == want.found, case.name
        if want.found:
            assert got.score == want.score and want.index_of(got.offset) in want.tied, case.name
