"""The numpy reference of the real-time correlative scan matcher (rtcsm_reference) against hand-worked answers and the
reference's own test fixture, its cell indices against exact rational arithmetic, and the C++ oracle against it on every case
of rtcsm_cases, bit for bit."""
from fractions import Fraction

import numpy as np
import pytest

import rtcsm_cases as cases
import rtcsm_reference as ref
from helpers import SEVEN

f32 = np.float32
IDENTITY = cases.IDENTITY


def _grid(cells, values, res=0.1):
    return ref.SparseGrid(res, np.asarray(cells).reshape(-1, 3), np.asarray(values, np.uint16))


# ----------------------------------------------------------------------------------------------- hand-worked answers
def test_one_point_one_cell_hand_worked():
    """One point at the origin, one cell of value 32 767 at (1, 0, 0), linear window 1 cell, no rotations, zero weights: the
    candidate x = +1 (index 14 in z, y, x order) scores 0.9, every other 0.1."""
    g = _grid([[1, 0, 0]], [32767])
    m = ref.match(g, np.zeros((1, 3), f32), IDENTITY, 0.1, 0.0, 0.0, 0.0)
    assert (m.window.linear, m.window.angular) == (1, 0) and m.num_candidates == 27
    assert m.window.max_scan_range == f32(3.0) * f32(0.1)
    assert m.best_index == 14 and m.score == ref.value_to_probability(32767)
    assert (np.delete(m.scores, 14) == f32(0.1)).all()
    assert np.array_equal(m.pose, np.array([f32(0.1), 0, 0, 1, 0, 0, 0], np.float64))


def test_sum_order_matters_hand_worked():
    """Three points whose probabilities p0 + p1 + p2 differ in float32 between (p0 + p1) + p2 and p0 + (p1 + p2): the score
    is the sum strictly in point order, divided by float(3)."""
    vals = np.arange(1, 32768)
    p = ref.value_to_probability(vals)
    a, b, c = None, None, None
    for i in range(0, 32767, 97):
        for j in range(5, 32767, 389):
            for k in range(3, 32767, 1013):
                if (p[i] + p[j]) + p[k] != p[i] + (p[j] + p[k]):
                    a, b, c = vals[i], vals[j], vals[k]
                    break
            if a is not None:
                break
        if a is not None:
            break
    assert a is not None
    g = _grid([[0, 0, 0], [3, 0, 0], [6, 0, 0]], [a, b, c])
    pts = np.array([[0, 0, 0], [0.3, 0, 0], [0.6, 0, 0]], f32)
    m = ref.match(g, pts, IDENTITY, 0.0, 0.0, 0.0, 0.0)
    pa, pb, pc = ref.value_to_probability([a, b, c])
    assert m.scores[0] == ((pa + pb) + pc) / f32(3.0)
    assert m.scores[0] != (pa + (pb + pc)) / f32(3.0)


def test_penalty_hand_worked():
    """One translation cell off the centre with w_t = 2: the score is float(double(p) * exp(-(0.1f * 2)^2)), the norm promoted
    to double before the weight."""
    g = _grid([[0, 0, 0]], [20000])
    m = ref.match(g, np.zeros((1, 3), f32), IDENTITY, 0.1, 0.0, 2.0, 0.0)
    p = np.float64(ref.value_to_probability(20000))
    a = np.float64(f32(0.1)) * 2.0
    assert m.scores[13] == f32(p) and m.scores[14] == f32(np.float64(f32(0.1)) * np.exp(-(a * a)))
    assert m.best_index == 13


def test_window_edges_hand_worked():
    r = f32(0.1)
    assert ref.window(np.zeros((1, 3), f32), 0.1, 0.15, 0.0).linear == 1          # 0.15 / 0.1f = 1.4999999776482582
    assert ref.round_to_int_double(2.5) == 3 and ref.round_to_int_double(-2.5) == -3
    assert ref.round_to_int_double(np.inf) == 0 and ref.round_to_int_double(np.nan) == 0     # glibc: LONG_MIN, low 32 bits
    assert ref.angular_step(0.1, cases.CLIFF) == 0 and ref.angular_step(0.1, np.nextafter(cases.CLIFF, f32(0))) > 0
    assert ref.max_scan_range(np.array([[0.1, 0.1, 0.1]], f32), r) == f32(3.0) * r


def test_angle_axis_cutoff_in_double():
    """Below the squared-norm cutoff 1e-8 (compared in double) the quaternion is (1, v / 2); above it sin / cos in double."""
    small = ref.angle_axis_to_quat(np.array([9.9e-5, 0, 0], f32))
    assert small[0] == 1 and small[1] == f32(0.5) * f32(9.9e-5)
    big = ref.angle_axis_to_quat(np.array([0.02, 0, 0], f32))
    assert big[0] == f32(np.cos(np.float64(f32(0.02)) / 2))


@pytest.mark.parametrize("t,angle,axis", [((-1, 0, 0), 0.0, (1, 0, 0)), ((-0.8, 0, 0), 0.0, (1, 0, 0)),
                                          ((-1, 0, -0.2), 0.0, (1, 0, 0)), ((-0.9, -0.2, 0.2), 0.0, (1, 0, 0)),
                                          ((-1, 0, 0), 0.8 / 180 * np.pi, (1, 0, 0)), ((-1, 0, 0), 0.8 / 180 * np.pi, (0, 1, 0)),
                                          ((-1, 0, 0), 0.8 / 180 * np.pi, (0, 1, 1))])
def test_reference_fixture_seven_starts(orc, t, angle, axis):
    """real_time_correlative_scan_matcher_3d_test.cc: from each of the seven starts the match lands on (-1, 0, 0) within
    1e-3; the whole score cube equals the oracle's."""
    from helpers import seven_point_grid
    og = seven_point_grid(orc, 0.1)
    g = ref.SparseGrid.from_export(og.resolution, og.export())
    init = orc.angle_axis_pose(t, angle, axis)
    m = ref.match(g, SEVEN, init, 0.3, np.deg2rad(1.0), 1e-1, 1.0)
    assert (m.window.linear, m.window.angular) == (3, 1) and m.num_candidates == 9261
    assert np.allclose(m.pose[:3], [-1, 0, 0], atol=1e-3) and abs(abs(m.pose[3]) - 1) < 1e-6
    want = orc.rtcsm_match(og, SEVEN, init, 0.3, np.deg2rad(1.0), 1e-1, 1.0, want_scores=True)
    assert np.array_equal(want["scores"].view(np.uint32), m.scores.view(np.uint32))


# ----------------------------------------------------------------------------------------------- exact cell indices
def _nearest_f32(x):
    """The float32 nearest to the rational x (ties to even)."""
    f = f32(float(x))
    best = None
    for c in (np.nextafter(f, f32(-np.inf)), f, np.nextafter(f, f32(np.inf))):
        d = abs(Fraction(float(c)) - x)
        key = (d, int(np.array(c, f32).view(np.uint32)) & 1)
        if best is None or key < best[0]:
            best = (key, c)
    return best[1]


def _lround(x):
    fl = x.numerator // x.denominator
    frac = x - fl
    if x >= 0:
        return fl + (1 if frac >= Fraction(1, 2) else 0)
    return -_lround(-x)


@pytest.mark.parametrize("name", cases.BOUNDARY)
def test_boundary_cells_are_correctly_rounded_quotients(name):
    """The centre candidate's cell of every point: the IEEE quotient (the correctly rounded x / resolution), then lround half
    away from zero — computed here with exact rationals."""
    c = cases.get(name)
    m = c.result
    R, L = len(m.cands.cand_q), len(m.cands.cand_t)
    w = ref.rotate(m.cands.cand_q[R // 2], c.points) + m.cands.cand_t[L // 2]
    got = ref.cell_index(w, c.grid.resolution)
    res = Fraction(float(f32(c.grid.resolution)))
    on_half = 0
    for p, cell in zip(w, got):
        for x, k in zip(p, cell):
            q = _nearest_f32(Fraction(float(x)) / res)
            on_half += Fraction(float(q)) - Fraction(float(q)).numerator // Fraction(float(q)).denominator == Fraction(1, 2)
            assert _lround(Fraction(float(q))) == k
    assert on_half > 0


# ----------------------------------------------------------------------------------------------- the oracle on every case
@pytest.mark.parametrize("name", cases.NAMES)
def test_oracle_equals_reference(orc, name):
    c = cases.get(name)
    m = c.result
    og = orc.Grid(c.grid.resolution)
    if len(c.grid.cells):
        og.set_cells(*c.grid.export())
    got = orc.rtcsm_match(og, *c.args, want_scores=True)
    assert (got["linear"], got["angular"]) == (m.window.linear, m.window.angular)
    assert f32(got["angular_step"]).view(np.uint32) == f32(m.window.step).view(np.uint32)
    assert f32(got["max_scan_range"]).view(np.uint32) == f32(m.window.max_scan_range).view(np.uint32)
    assert np.array_equal(got["scores"].view(np.uint32), m.scores.view(np.uint32))
    assert got["best_index"] == m.best_index and f32(got["score"]) == m.score
    assert np.array_equal(got["pose"], m.pose)
