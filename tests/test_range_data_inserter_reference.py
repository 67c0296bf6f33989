"""CPU tests of the numpy reference of the range-data inserter (tests/range_data_inserter_reference.py): hand-worked answers
first, then the C++ oracle pinned to the reference, bit for bit, on every case of tests/range_data_inserter_cases.py."""
import numpy as np
import pytest

import range_data_inserter_cases as cases
import range_data_inserter_reference as ref

f32 = np.float32
ODDS_PAIRS = [(0.55, 0.49), (0.7, 0.4), (0.9, 0.1), (0.99, 0.01), (0.5000001, 0.4999999), (0.50000001, 0.0)]
ALL = cases.all_cases()


def cells_of(grid):
    x, y, z, v = grid.export()
    return {(int(a), int(b), int(c)): int(d) for a, b, c, d in zip(x, y, z, v)}


# ----------------------------------------------------------------------------------------------- hand-worked answers
def test_probability_values_round_trips():
    """probability_values_test: Odds / ProbabilityFromOdds round trips; values 1 and 32767 are 0.1f and 0.9f."""
    for p in (ref.K_MIN, ref.K_MAX, f32(0.5)):
        assert abs(float(ref.probability_from_odds(ref.odds(p))) - float(p)) < 1e-6
    assert ref.value_to_probability(0) == f32(0.1) and ref.value_to_probability(1) == f32(0.1)
    # 32767 * kScale + (0.1f - kScale) rounds to 0.8999999f, one ulp below kMaxProbability
    assert ref.value_to_probability(32767) == np.nextafter(ref.K_MAX, f32(0))
    assert ref.value_to_probability(32768 + 5) == ref.value_to_probability(5)     # the marker bit is ignored
    assert ref.probability_to_value(f32(0.1)) == 1 and ref.probability_to_value(f32(0.9)) == 32767
    assert ref.probability_to_value(f32(0.0)) == 1 and ref.probability_to_value(f32(1.0)) == 32767   # clamped
    # (0.5 - 0.1) * (32766 / 0.8) = 16383 (float32: 16383.0), + 1
    assert ref.probability_to_value(f32(0.5)) == 16384
    v = np.arange(1, 32768)
    assert (ref.probability_to_value(ref.value_to_probability(v)) == v).all()


def test_round_to_int_and_cell_index_by_hand():
    assert ref.round_to_int([0.5, 1.5, -0.5, -1.5, 0.49999997, 2.4999998]).tolist() == [1, 2, -1, -2, 0, 2]
    # 0.65f / 0.1f in float32 is 6.4999995 -> 6, not 7; 0.25f / 0.1f is 2.5 -> 3 (half away from zero), -0.25 -> -3
    assert ref.cell_index(_p(0.65, 0.25, -0.25), 0.1)[0].tolist() == [6, 3, -3]


def test_odds_tables_by_hand():
    hit, miss = ref.tables(0.55, 0.49)
    assert hit[0] - 32768 == ref.probability_to_value(f32(0.55)) and miss[0] - 32768 == ref.probability_to_value(f32(0.49))
    # odds 1: every value maps to itself (0 maps to 0.5)
    same, _ = ref.tables(0.50000001, 0.4)
    assert same[0] == 16384 + 32768 and (same[1:] - 32768 == np.arange(1, 32768)).all()
    _, zero = ref.tables(0.6, 0.0)
    assert (zero == 1 + 32768).all()                                 # a miss of 0 sends every cell to value 1
    assert (hit >= 32768).all() and (miss >= 32768).all()


def test_truncation_differs_from_floor_by_hand():
    """Origin cell 0, hit cell (-2, 3, 1): num_samples 3, two free-space voxels, samples 1 and 2:
    position 1: (-2 / 3, 3 / 3, 1 / 3) = (0, 1, 0) truncated, (-1, 1, 0) floored;
    position 2: (-4 / 3, 6 / 3, 2 / 3) = (-1, 2, 0) truncated, (-2, 2, 0) floored.
    A second ray to (1, 1, 0) has one sample, the origin cell."""
    hits, misses, ray, ns = ref.rays(_p(0, 0, 0), _p([-2, 3, 1], [1, 1, 0]), 1.0, 2)
    assert ns.tolist() == [3, 1]
    assert misses.tolist() == [[0, 1, 0], [-1, 2, 0], [0, 0, 0]]
    assert ray.tolist() == [0, 0, 1]


def test_hit_beats_miss_by_hand():
    """Hits at 3 and 4 on the x axis from the origin, two free-space voxels: ray 4 samples 2 and 3; cell 3 is a hit."""
    g = ref.Grid(1.0)
    ref.insert(g, _p(0, 0, 0)[0], _p([3, 0, 0], [4, 0, 0]), 0.55, 0.49, 2)
    hit, miss = ref.tables(0.55, 0.49)
    h, m = int(hit[0]) - 32768, int(miss[0]) - 32768
    assert cells_of(g) == {(1, 0, 0): m, (2, 0, 0): m, (3, 0, 0): h, (4, 0, 0): h}
    assert g.num_bricks == 1


def test_origin_cell_miss_by_hand():
    """num_free >= num_samples: sample 0 is the origin cell itself."""
    g = ref.Grid(1.0)
    ref.insert(g, _p(0.2, 0, 0)[0], _p([-2, 0, 0]), 0.55, 0.49, 5)
    m, h = int(ref.tables(0.55, 0.49)[1][0]) - 32768, int(ref.tables(0.55, 0.49)[0][0]) - 32768
    assert cells_of(g) == {(-2, 0, 0): h, (-1, 0, 0): m, (0, 0, 0): m}
    g2 = ref.Grid(1.0)
    ref.insert(g2, _p(0.2, 0, 0)[0], _p([-2, 0, 0]), 0.55, 0.49, 1)
    assert cells_of(g2) == {(-2, 0, 0): h, (-1, 0, 0): m}


def test_reference_fixture_by_hand():
    """range_data_inserter_3d_test.cc: after one Insert hits are 0.7, ray cells 0.4 (1e-4); after many, 0.9 and 0.1 (1e-3)."""
    c = cases.reference_fixture()
    g = ref.Grid(1.0)
    s = c.steps[0]
    ref.insert(g, s.origin, s.returns, s.hit, s.miss, s.num_free)
    prob = lambda p: float(ref.value_to_probability(g.lookup(ref.order_key(ref.cell_index(_p(*p), 1.0)))[0]))
    assert abs(prob((0, 0, -4)) - 0.4) < 1e-4 and abs(prob((0, 0, -3)) - 0.4) < 1e-4 and abs(prob((-2, 0, 4)) - 0.7) < 1e-4
    for x in range(-4, 5):
        for y in range(-4, 5):
            known = g.lookup(ref.order_key(np.array([[x, y, 4]])))[0] != 0
            assert known == (-3 <= x <= 0 and y == x + 2)
    for _ in range(1000):
        ref.insert(g, s.origin, s.returns, s.hit, s.miss, s.num_free)
    assert abs(prob((-2, 0, 4)) - 0.9) < 1e-3 and abs(prob((-2, 0, 3)) - 0.1) < 1e-3 and abs(prob((0, 0, -3)) - 0.1) < 1e-3


def test_order_and_bricks_by_hand():
    """Iterator order: top cell, then brick, then cell, each flat z-major; independent of bits."""
    g = ref.Grid(1.0)
    g.set_cells([0, 1, 8, 0, 64, -1], [0, 0, 0, 1, 0, 0], [0, 0, 0, 0, 0, 0], [1, 2, 3, 4, 5, 6])
    x, y, z, v = g.export()
    # (-1, 0, 0) lies in the top cell below the origin's; (8, 0, 0) is the origin's top cell, next brick; (64, 0, 0) the next
    # top cell along x
    assert list(zip(x.tolist(), y.tolist())) == [(-1, 0), (0, 0), (1, 0), (0, 1), (8, 0), (64, 0)]
    assert v.tolist() == [6, 1, 2, 4, 3, 5]
    assert g.num_bricks == 4 and g.bits == 2
    assert ref.bits_for([[-64, 0, 0]]) == 1 and ref.bits_for([[-65, 0, 0]]) == 2 and ref.bits_for([[63, 0, 0]]) == 1
    assert ref.bits_for([[8191, 0, 0]]) == 8 and not ref.in_range([[8192, 0, 0]]) and ref.in_range([[-8192, 0, 0]])


def test_num_samples_and_range_errors_by_hand():
    g = ref.Grid(1.0)
    with pytest.raises(ref.InsertError) as e:
        ref.insert(g, _p(-32768, 0, 0)[0], _p([0, 0, 0]), num_free=0)      # CHECK_LT whatever num_free is
    assert e.value.status == ref.ERR_ARG and g.export()[0].size == 0
    with pytest.raises(ref.InsertError) as e:
        ref.insert(g, _p(0, 0, 0)[0], _p([8192, 0, 0]), num_free=0)
    assert e.value.status == ref.ERR_GRID_RANGE and g.export()[0].size == 0
    ref.insert(g, _p(-32767, 0, 0)[0], _p([0, 0, 0]), num_free=2)
    assert cells_of(g).keys() == {(-2, 0, 0), (-1, 0, 0), (0, 0, 0)}


def test_submap_transform_by_hand():
    """Submap at (10, 0, 0) rotated 90 degrees about z: local (10, 5, 0) is (5, 0, 0) in the submap; range 5 is near at
    max range 5 (<=) and far at 4."""
    c = np.cos(np.pi / 4)
    pose = np.array([10, 0, 0, c, 0, 0, c])
    t, q = ref.to_submap_transform(pose)
    p = ref.transform(_p(10, 5, 0), t, q)[0]
    assert np.allclose(p, [5, 0, 0], atol=1e-5)
    o = ref.transform(_p(10, 0, 0), t, q)[0]
    assert np.allclose(o, [0, 0, 0], atol=1e-5)
    pts = np.array([[5, 0, 0]], f32)
    assert ref.near_mask(pts, [0, 0, 0], 5)[0] and not ref.near_mask(pts, [0, 0, 0], 4)[0]


def _p(*rows):
    return np.array(rows, f32).reshape(-1, 3)


# ----------------------------------------------------------------------------------------------- the oracle against the reference
def test_oracle_value_to_probability_table_equals_reference(orc):
    want = np.zeros(65536, f32)
    orc.lib().orc_value_to_probability_table(want)
    assert np.array_equal(ref.value_to_probability(np.arange(65536)), want)


@pytest.mark.parametrize("hit,miss", ODDS_PAIRS)
def test_oracle_odds_tables_equal_reference(orc, hit, miss):
    want_hit, want_miss = ref.tables(hit, miss)
    assert (orc.lookup_table_to_apply_odds(orc.lib().orc_odds(f32(hit))) == want_hit).all()
    assert (orc.lookup_table_to_apply_odds(orc.lib().orc_odds(f32(miss))) == want_miss).all()


@pytest.mark.parametrize("case", ALL, ids=[c.name for c in ALL])
def test_oracle_equals_reference(orc, case):
    """Every Insert of the case into the oracle's HybridGrid: same cells, order and values as the reference, same success or
    failure. After a failed Insert the oracle's grid is left half written (the reference aborts there), so the comparison
    stops at the first failure."""
    g = ref.Grid(case.resolution)
    og = orc.Grid(case.resolution)
    for step, status in zip(case.steps, case.status):
        if status == ref.ERR_ARG:
            # the oracle has no CHECK_LT(num_samples, 1 << 15): it walks the ray. The reference refuses it; nothing to compare.
            return
        try:
            og.insert_range_data(step.origin, step.returns, step.hit, step.miss, step.num_free)
            got = 0
        except RuntimeError:
            got = ref.ERR_GRID_RANGE
        assert got == status
        if status:
            return
        ref.insert(g, step.origin, step.returns, step.hit, step.miss, step.num_free)
        for a, b in zip(og.export(), g.export()):
            assert np.array_equal(a, b)
        assert og.bits() == g.bits


SUBMAP_POSES = [np.array([0, 0, 0, 1, 0, 0, 0.0]),
                np.array([312.5, -187.25, 4.0, *(np.array([0.9, 0.1, -0.2, 0.37]) / np.linalg.norm([0.9, 0.1, -0.2, 0.37]))])]


@pytest.mark.parametrize("pose", range(len(SUBMAP_POSES)))
@pytest.mark.parametrize("max_range", [0, 1, 20])
def test_oracle_submap_insert_equals_reference(orc, pose, max_range):
    import synth
    rows = synth.make_scan(synth.Scene(42), 16, 2.0)
    local = (np.stack([rows["x"], rows["y"], rows["z"]], 1) + SUBMAP_POSES[pose][:3]).astype(f32)
    origin = SUBMAP_POSES[pose][:3].astype(f32) + f32(0.3)
    hi, lo = ref.Grid(0.1), ref.Grid(0.45)
    ohi, olo = orc.Grid(0.1), orc.Grid(0.45)
    for k in range(2):
        ref.submap_insert(hi, lo, SUBMAP_POSES[pose], origin, local[k::2], max_range)
        orc.submap_insert_range_data(ohi, olo, SUBMAP_POSES[pose], origin, local[k::2], max_range)
    for o, r in ((ohi, hi), (olo, lo)):
        for a, b in zip(o.export(), r.export()):
            assert np.array_equal(a, b)
    # one grid as both: Insert(near) then Insert(all) into it
    same, osame = ref.Grid(0.2), orc.Grid(0.2)
    ref.submap_insert(same, same, SUBMAP_POSES[pose], origin, local, max_range)
    orc.submap_insert_range_data(osame, osame, SUBMAP_POSES[pose], origin, local, max_range)
    for a, b in zip(osame.export(), same.export()):
        assert np.array_equal(a, b)
