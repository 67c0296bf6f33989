"""The probability-grid reference (tests/probability_grid_reference.py) pinned to the reference's own fixtures
(range_data_inserter_2d_test.cc, probability_grid_test.cc, map_limits_test.cc, xy_index_test.cc), to an exact-rational reading
of CastRay, to a direct float evaluation of every table entry, and to hand-written PGM / YAML files. The device's two
shortcuts are checked here too: a per-cell atomicMax stamp in any order gives the marker rule's grid, and the known-cells box
is the box of the cells != 0."""
from fractions import Fraction

import numpy as np
import pytest

import probability_grid_reference as pg

f32 = np.float32


def fixture_grid():
    """RangeDataInserterTest2D: MapLimits(1., (1., 5.), 5 x 5), hit 0.7, miss 0.4, insert_free_space."""
    return pg.Grid.from_limits(pg.Limits(1.0, 1.0, 5.0, 5, 5)), pg.correspondence_cost_table(0.7), pg.correspondence_cost_table(0.4)


def insert_point_cloud(g, hit, miss):
    points = np.array([[-3.5, 0.5, 0], [-2.5, 1.5, 0], [-1.5, 2.5, 0], [-0.5, 3.5, 0]], np.float32)
    g.insert(np.array([-0.5, 0.5, 0], np.float32), points, hit, miss)
    g.finish_update()


def test_insert_point_cloud():
    g, hit, miss = fixture_grid()
    insert_point_cloud(g, hit, miss)
    l = g.limits
    assert (l.max_x, l.max_y, l.num_x, l.num_y) == (1.0, 5.0, 5, 5)
    U, M, H = 0, 1, 2
    expected = [[U, U, U, U, U], [U, H, M, M, M], [U, U, H, M, M], [U, U, U, H, M], [U, U, U, U, H]]
    for row in range(5):
        for column in range(5):
            state = expected[column][row]
            if state == U:
                assert not g.is_known(row, column)
            else:
                want = 0.4 if state == M else 0.7
                assert abs(float(g.get_probability(row, column)) - want) <= 1e-4


def test_probability_progression():
    g, hit, miss = fixture_grid()
    insert_point_cloud(g, hit, miss)
    hit_cell, miss_cell = g.limits.cell_index(-3.5, 0.5), g.limits.cell_index(-2.5, 0.5)
    assert abs(float(g.get_probability(*hit_cell)) - 0.7) <= 1e-4
    assert abs(float(g.get_probability(*miss_cell)) - 0.4) <= 1e-4
    for _ in range(1000):
        insert_point_cloud(g, hit, miss)
    assert abs(float(g.get_probability(*hit_cell)) - float(pg.MAX_PROBABILITY)) <= 1e-3
    assert abs(float(g.get_probability(*miss_cell)) - float(pg.MIN_PROBABILITY)) <= 1e-3


def test_apply_odds():
    g = pg.Grid.from_limits(pg.Limits(1.0, 1.0, 1.0, 2, 2))
    assert all(g.limits.contains(x, y) for x in (0, 1) for y in (0, 1))
    assert not any(g.is_known(x, y) for x in (0, 1) for y in (0, 1))
    g.set_probability(1, 0, 0.5)
    g.apply_lookup_table(1, 0, pg.correspondence_cost_table(0.9))
    g.finish_update()
    assert g.get_probability(1, 0) > 0.5
    g.set_probability(0, 1, 0.5)
    g.apply_lookup_table(0, 1, pg.correspondence_cost_table(0.1))
    g.finish_update()
    assert g.get_probability(0, 1) < 0.5
    g.apply_lookup_table(1, 1, pg.correspondence_cost_table(0.42))     # an unknown cell
    assert abs(float(g.get_probability(1, 1)) - 0.42) <= 1e-4
    g.apply_lookup_table(1, 1, pg.correspondence_cost_table(0.9))      # ignored until FinishUpdate
    assert abs(float(g.get_probability(1, 1)) - 0.42) <= 1e-4
    g.finish_update()
    g.apply_lookup_table(1, 1, pg.correspondence_cost_table(0.9))
    assert g.get_probability(1, 1) > 0.42


def test_get_probability():
    g = pg.Grid.from_limits(pg.Limits(1.0, 1.0, 2.0, 2, 2))
    c = g.limits.cell_index(-0.5, 0.5)
    g.set_probability(*c, pg.MAX_PROBABILITY)
    assert abs(float(g.get_probability(*c)) - float(pg.MAX_PROBABILITY)) <= 1e-6
    for p in ((-0.5, 1.5), (0.5, 0.5), (0.5, 1.5)):
        i = g.limits.cell_index(*p)
        assert g.limits.contains(*i) and not g.is_known(*i)


def test_get_cell_index():
    l = pg.Limits(2.0, 8.0, 14.0, 14, 8)
    cases = {(7, 13): (0, 0), (7, -13): (13, 0), (-7, 13): (0, 7), (-7, -13): (13, 7), (0.5, 0.5): (6, 3), (1.5, 1.5): (6, 3),
             (0.5, -0.5): (7, 3), (-0.5, 0.5): (6, 4), (-0.5, -0.5): (7, 4)}
    for p, want in cases.items():
        assert l.cell_index(*p) == want


def test_correct_cropping():
    g = pg.Grid.from_limits(pg.Limits(0.05, 10.0, 10.0, 400, 400))
    rng = np.random.default_rng(42)
    for x, y in pg.xy_index_range((100, 100), (299, 299)):
        g.set_probability(x, y, rng.uniform(0.1, 0.9))
    assert g.cropped() == (100, 100, 200, 200)


def test_map_limits_construct_and_get():
    l = pg.Limits(42.0, 3.0, 0.0, 2, 3)
    assert (l.num_x, l.num_y, l.max_x, l.max_y, l.resolution) == (2, 3, 3.0, 0.0, 42.0)


def test_xy_index_range_iterator():
    got = list(pg.xy_index_range((1, 2), (3, 4)))
    assert got[0] == (1, 2) and len(got) == 9
    assert all(1 <= x <= 3 and 2 <= y <= 4 for x, y in got)


# ---- CastRay
def exact_pixels(begin, end):
    """The full pixels whose open interior the segment between the two subpixel centres meets, plus both end pixels, in exact
    rationals (an independent reading: no stepping)."""
    S = pg.SUBPIXEL
    p = [Fraction(2 * begin[k] + 1, 2 * S) for k in (0, 1)]
    q = [Fraction(2 * end[k] + 1, 2 * S) for k in (0, 1)]
    out = {(begin[0] // S, begin[1] // S), (end[0] // S, end[1] // S)}
    for X in range(min(begin[0], end[0]) // S, max(begin[0], end[0]) // S + 1):
        for Y in range(min(begin[1], end[1]) // S, max(begin[1], end[1]) // S + 1):
            lo, hi = Fraction(0), Fraction(1)
            ok = True
            for k, (a, b) in enumerate(((X, X + 1), (Y, Y + 1))):
                d = q[k] - p[k]
                if d == 0:
                    ok &= a < p[k] < b
                else:
                    t0, t1 = (a - p[k]) / d, (b - p[k]) / d
                    lo, hi = max(lo, min(t0, t1)), min(hi, max(t0, t1))
            if ok and (lo < hi):
                out.add((X, Y))
    return out


def literal_walk(begin, end):
    visits = []
    pg.cast_ray(begin, end, lambda x, y: visits.append((x, y)))
    return visits


def segments(rng, n, span):
    """Random segments plus every edge: 45-degree corner crossings both ways, axis-aligned, one pixel, one subpixel."""
    S = pg.SUBPIXEL
    out = [tuple(map(int, rng.integers(0, span, 4))) for _ in range(n)]
    for k in range(1, 6):
        out += [(S * 2 + 499, S * 2 + 499, S * (2 + k) + 499, S * (2 + k) + 499),          # through pixel corners, rising
                (S * 2 + 499, S * 8 + 499, S * (2 + k) + 499, S * (8 - k) + 499),          # and falling
                (S * (2 + k) + 499, S * 2 + 499, S * 2 + 499, S * (2 + k) + 499),          # swapped ends
                (S * 3 + 10, S * 1 + 7, S * 3 + 900, S * (1 + k) + 5),                     # one column
                (S * 1 + 7, S * 4 + 3, S * (1 + k) + 5, S * 4 + 996),                      # dy = 0 in pixels
                (S + 1, S + 2, S + 1, S + 2 + k * 0),                                      # one subpixel
                (S + 1, S + 2, S + 998, S + 997)]                                          # one pixel
    return out


def test_cast_ray_matches_the_exact_reading():
    rng = np.random.default_rng(7)
    for bx, by, ex, ey in segments(rng, 20000, 9 * pg.SUBPIXEL):
        visits = literal_walk((bx, by), (ex, ey))
        assert len(visits) == len(set(visits)), (bx, by, ex, ey)          # no pixel twice within one walk
        assert set(visits) == exact_pixels((bx, by), (ex, ey)), (bx, by, ex, ey)


def test_walk_cells_equals_the_literal_walk():
    rng = np.random.default_rng(11)
    for span in (3 * pg.SUBPIXEL, 40 * pg.SUBPIXEL, 400 * pg.SUBPIXEL):
        segs = segments(rng, 400, span)
        for bx, by in {(s[0], s[1]) for s in segs[::37]} | {(2499, 2499)}:
            ends = np.array([(s[2], s[3]) for s in segs], np.int64)
            x, y = pg.walk_cells(bx, by, ends[:, 0], ends[:, 1])
            want = []
            for e in ends:
                want += literal_walk((bx, by), (int(e[0]), int(e[1])))
            assert sorted(zip(x.tolist(), y.tolist())) == sorted(want)


# ---- Insert: the fast form, the stamp claim and the known-cells box
def random_batches(rng, n, spread, res, far=False):
    out = []
    for k in range(n):
        o = rng.normal(0, spread / 4, 3).astype(np.float32)
        m = int(rng.integers(0, 300))
        pts = (o + rng.normal(0, spread, (m, 3))).astype(np.float32)
        if far and k == n // 2:
            pts[:5, :2] += np.float32(40 * spread)           # several doublings inside one batch
        if m and k % 3 == 0:                                 # points on superscaled rounding boundaries, and repeated cells
            pts[:, :2] = (np.round(pts[:, :2] / (res / 2)) * (res / 2)).astype(np.float32)
        out.append((o, pts))
    return out


@pytest.mark.parametrize("res,free", [(0.05, True), (0.1, False), (0.5, True), (1.0, True)])
def test_insert_fast_equals_the_literal_insert(res, free):
    rng = np.random.default_rng(int(res * 100) + free)
    batches = random_batches(rng, 10, 2.0, res, far=True)
    a = pg.run_batches(res, 0.55, 0.49, batches, free, fast=False)
    b = pg.run_batches(res, 0.55, 0.49, batches, free, fast=True)
    assert a.info() == b.info() and np.array_equal(a.cells, b.cells)
    assert a.limits.num_x > 100                                  # it grew


def test_stamp_claims_in_any_order_give_the_marker_rule_and_the_box_is_the_known_cells():
    """The device's rule: batch k claims with atomicMax(stamp, 2k + 1) for a hit and 2k for a walk, every hit before every walk,
    and the claim that lifts the stamp past 2k - 1 applies the table. Visits in shuffled order must give the literal grid; the
    box of the cells != 0 must equal the tracked known-cells box."""
    rng = np.random.default_rng(3)
    res = 0.25
    batches = random_batches(rng, 8, 2.0, res)
    ht, mt = pg.correspondence_cost_table(0.55), pg.correspondence_cost_table(0.49)
    ref = pg.run_batches(res, 0.55, 0.49, batches, fast=False)
    g = pg.Grid(res)
    stamps = np.zeros_like(g.cells, np.uint32)
    for k, (origin, pts) in enumerate(batches, start=1):
        before = g.limits
        g.grow_as_needed(origin, pts)
        if g.cells.shape != stamps.shape:
            stamps = np.zeros_like(g.cells, np.uint32)                     # a fresh stamp is 0, below every claim
        del before
        ss = g.limits.superscaled()
        begin = ss.cell_index(origin[0], origin[1])
        ends = [ss.cell_index(p[0], p[1]) for p in pts]
        hits = [(e[0] // pg.SUBPIXEL, e[1] // pg.SUBPIXEL) for e in ends]
        walks = []
        for e in ends:
            walks += literal_walk(begin, e)
        for cells, claim, table in ((hits, 2 * k + 1, ht), (walks, 2 * k, mt)):
            for i in rng.permutation(len(cells)):
                x, y = cells[i]
                old = stamps[y, x]
                stamps[y, x] = max(old, claim)
                if old < 2 * k:
                    g.cells[y, x] = table[g.cells[y, x]] - pg.UPDATE_MARKER
    assert np.array_equal(g.cells, ref.cells)
    ys, xs = np.nonzero(g.cells)
    assert [xs.min(), ys.min(), xs.max(), ys.max()] == ref.box


def test_growth_refused_beyond_the_int_limit():
    g = pg.Grid(1.0)
    g.insert_fast(np.zeros(3, np.float32), np.array([[1000.0, 0, 0]], np.float32), pg.correspondence_cost_table(0.55),
                  pg.correspondence_cost_table(0.49))
    before = (g.limits.num_x, g.limits.max_x, g.cells.copy())
    with pytest.raises(pg.GrowthRefused):
        g.grow_as_needed(np.zeros(3, np.float32), np.array([[2e6, 0, 0]], np.float32))   # 2e6 cells: beyond 100 * 2^14
    assert g.limits.num_x == before[0] and g.limits.max_x == before[1] and np.array_equal(g.cells, before[2])   # unchanged
    l = pg.grown_limits(pg.Limits(1.0, 50.0, 50.0, 100, 100), f32(50.0 * 2 ** 14 - 1), f32(0.0))
    assert l.num_x == pg.MAX_CELLS                   # the largest grid the int arithmetic allows


def test_empty_grid_is_one_unknown_pixel():
    g = pg.Grid(0.05)
    g.insert_fast(np.array([3.0, -2.0, 0.0], np.float32), np.zeros((0, 3), np.float32), pg.correspondence_cost_table(0.55),
                  pg.correspondence_cost_table(0.49))
    assert g.cropped() == (0, 0, 1, 1) and g.image().tolist() == [[128]]


# ---- tables and colours, entry by entry with float32 scalars
def direct_table(probability):
    one = f32(1.0)
    lo, hi = one - (one - f32(0.1)), one - f32(0.1)
    scale = (hi - lo) / f32(32766.0)

    def to_value(c):
        c = min(max(f32(c), lo), hi)
        return pg.lround(float((c - lo) * (f32(32766.0) / (hi - lo)))) + 1

    p = f32(probability)
    odds = p / (one - p)
    out = [to_value(one - odds / (odds + one)) + 32768]
    for v in range(1, 32768):
        q = one - (f32(v) * scale + (lo - scale))
        o = odds * (q / (one - q))
        out.append(to_value(one - o / (o + one)) + 32768)
    return out


@pytest.mark.parametrize("hit,miss", [(0.55, 0.49), (0.7, 0.4), (0.9, 0.12)])
def test_every_table_entry_against_a_direct_float_evaluation(hit, miss):
    for p in (hit, miss):
        assert pg.correspondence_cost_table(p).tolist() == direct_table(p)


def test_colour_table():
    colors = pg.color_table()
    one = f32(1.0)
    values = pg.value_to_correspondence_cost()
    for v in range(1, 32768, 7):
        p = one - values[v]
        want = pg.lround(float(f32(255.0) * (((one - p) - f32(0.1)) / ((one - f32(0.1)) - f32(0.1)))))
        assert colors[v] == want
    assert colors[0] == 128 and colors.max() == 255 and colors[1:].min() == 0


# ---- the ROS map files
def test_ros_map_files_match_hand_written_bytes():
    image = np.array([[1, 2, 3], [4, 5, 6]], np.uint8)            # 3 wide, 2 high, unrotated
    info = {"resolution": 0.05, "max_x": 12.3456785, "max_y": -0.0000004, "offset_x": 7, "offset_y": 11}
    pgm, yaml = pg.ros_map(info, image, "out/map.pgm")
    assert pg.rotate90_clockwise(image).tolist() == [[4, 1], [5, 2], [6, 3]]
    assert pgm == b"P5\n# Cartographer map; 0.050000 m/pixel\n2 3\n255\n\x04\x01\x05\x02\x06\x03"
    # origin x = 12.3456785 - (11 + 2) * 0.05 = 11.6956785 -> %f rounds to 11.695679 (11.69567849999... in binary: 11.695678)
    ox, oy = 12.3456785 - 13 * 0.05, -0.0000004 - 10 * 0.05
    assert "%f" % ox in ("11.695678", "11.695679") and "%f" % oy == "-0.500000"
    assert yaml == ("image: out/map.pgm\nresolution: 0.050000\norigin: [" + "%f" % ox + ", -0.500000, 0.0]\nnegate: 0\n"
                    "occupied_thresh: 0.65\nfree_thresh: 0.196\n").encode()
    # origin x = 0.25 + 2^-21 - 1 = -0.749999523162841796875 exactly: %f rounds it to -0.750000
    info2 = {"resolution": 1.0, "max_x": 0.25 + 2.0 ** -21, "max_y": 2.0, "offset_x": 0, "offset_y": 0}
    pgm2, yaml2 = pg.ros_map(info2, np.array([[128]], np.uint8), "m.pgm")
    assert pgm2 == b"P5\n# Cartographer map; 1.000000 m/pixel\n1 1\n255\n\x80"
    assert yaml2 == b"image: m.pgm\nresolution: 1.000000\norigin: [-0.750000, 1.000000, 0.0]\nnegate: 0\n" \
                    b"occupied_thresh: 0.65\nfree_thresh: 0.196\n"


def test_python_writers_equal_the_reference_bytes(tmp_path):
    import dliom
    rng = np.random.default_rng(5)
    g = pg.run_batches(0.1, 0.55, 0.49, random_batches(rng, 4, 2.0, 0.1))
    info, image = g.info(), g.image()
    stem = str(tmp_path / "map")
    dliom.write_ros_map(stem, info, image)
    pgm, yaml = pg.ros_map(info, image, stem + ".pgm")
    assert open(stem + ".pgm", "rb").read() == pgm and open(stem + ".yaml", "rb").read() == yaml
    dliom.write_probability_grid_png(str(tmp_path / "grid.png"), image)
    import zlib
    data = open(tmp_path / "grid.png", "rb").read()
    idat = data[data.index(b"IDAT") + 4:data.index(b"IEND") - 8]
    raw = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(image.shape[0], 1 + 3 * image.shape[1])
    assert (raw[:, 0] == 0).all() and np.array_equal(raw[:, 1::3], image) and np.array_equal(raw[:, 3::3], image)
