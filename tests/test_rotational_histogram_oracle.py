"""RotationalScanMatcher::ComputeHistogram: the numpy reference model (rotational_histogram_reference.py) against values computed by
hand on small slices, and the C++ oracle (orc.compute_histogram) against the model bit for bit on clouds cleared of the points an
atan2 implementation could decide either way."""
import numpy as np
import pytest

import rotational_histogram_reference as R

f32 = np.float32
SIZES = [1, 7, 120, 1024]


def bits(h):
    return np.asarray(h, f32).view(np.uint32)


def ring(radius, degrees, z=0.0):
    a = np.radians(np.asarray(degrees, np.float64))
    return np.stack([radius * np.cos(a), radius * np.sin(a), np.full(len(a), z)], 1).astype(f32)


def pile_slice():
    """A 24-point ring of radius 1 (5 deg + 15 deg k) and 40 points piled 0.15 m off its centre, piled points first."""
    pile = np.tile(np.array([[0.15, 0.0, 0.0]], f32), (40, 1))
    return np.concatenate([pile, ring(1.0, 5.0 + 15.0 * np.arange(24))])


def expected_pile_histogram(size):
    """By hand: the pile lies 0.056 m from the first centroid (0.094, 0) and is dropped; the ring sorts from its 185 deg point.
    `last` moves every 4th point (chord 2 sin 30 deg = 1.0 > 0.9), so each anchor adds the chords to its next 3 points: direction
    anchor + 90 + 7.5 m deg, weight 1 - sin(7.5 m deg) against the ring's own centre, the sorted slice's centroid."""
    h = np.zeros(size)
    for j in range(6):
        anchor = 185.0 + 60.0 * j
        for m in (1, 2, 3):
            direction = (anchor + 90.0 + 7.5 * m) % 180.0
            h[int(direction / (180.0 / size))] += 1.0 - np.sin(np.radians(7.5 * m))
    return h


def test_pile_uses_the_centroid_of_the_sorted_slice():
    pts = pile_slice()
    for size in (8, 7, 120):
        got = R.compute_histogram(pts, size)
        assert np.abs(got - expected_pile_histogram(size)).max() < 2e-6, size
    # the centroid of the whole slice would weigh the same chords differently: the case tells the two readings apart
    order, (cx, cy), _, _ = R.sort_slice(pts[:, 0], pts[:, 1])
    assert sorted(order) == list(range(40, 64)) and abs(cx - 0.09375) < 1e-6
    ring_only = R.compute_histogram(pts[40:], 8)
    assert np.array_equal(bits(ring_only), bits(R.compute_histogram(pts, 8)))


def test_reset_of_last_and_the_minus_x_delta_with_signed_zero():
    """B sorts first; P lies 3.08 m from it (> 0.9: `last` = P, nothing added); Q - P = (-0.6, dy). dy = +0 gives atan2 = +pi,
    which stays pi and maps to bucket size (clamped to the last); dy = -0 gives -pi, wrapped to 0 -> bucket 0."""
    for qy, bucket in ((0.0, 7), (-0.0, 0)):
        pts = np.array([[-0.2, -3.0, 0.0], [0.5, 0.0, 0.0], [-0.1, qy, 0.0]], f32)
        order, _, _, _ = R.sort_slice(pts[:, 0], pts[:, 1])
        assert order.tolist() == [0, 1, 2]
        pos, dx, dy, value = R.walk(pts[order, 0], pts[order, 1])
        assert pos.tolist() == [2] and dx[0] == f32(-0.6) and dy[0] == 0 and np.signbit(dy[0]) == np.signbit(qy)
        cx = 0.2 / 3.0
        want = 1.0 - (0.1 + cx) / np.hypot(0.1 + cx, 1.0)
        h = R.compute_histogram(pts, 8)
        assert np.flatnonzero(h).tolist() == [bucket] and abs(h[bucket] - want) < 1e-6


def test_first_point_is_skipped_at_distance_zero():
    # two points 0.5 m apart on the same slice: the first is `last` itself (distance 0, skipped), the second adds its delta
    pts = np.array([[1.0, 0.25, 0.05], [1.0, -0.25, -0.05]], f32)     # slice 0 both; centroid (1, 0); sorted: the -y point first
    pos, dx, dy, value = R.walk(*(pts[[1, 0], c] for c in (0, 1)))
    assert pos.tolist() == [1] and (dx[0], dy[0]) == (0.0, f32(0.5))
    # delta +y against direction +y: weight 0 -> the histogram stays zero although a bucket was chosen
    assert value.tolist() == [0.0] and not R.compute_histogram(pts, 8).any()
    # a single point on its slice: no delta at all
    assert not R.compute_histogram(np.array([[3.0, 1.0, 0.0]], f32), 8).any()


def test_point_exactly_0_2_m_from_the_centroid_is_kept():
    for r, kept in ((f32(0.2), True), (np.nextafter(f32(0.2), f32(0)), False)):
        # input order keeps the centroid exactly (0, 0): r - r = 0, then four corners summing to 0
        pts = np.array([[r, 0, 0], [-r, 0, 0], [1, 1, 0], [-1, 1, 0], [-1, -1, 0], [1, -1, 0]], f32)
        order, (cx, cy), dx, dy = R.sort_slice(pts[:, 0], pts[:, 1])
        assert (cx, cy) == (0.0, 0.0) and (np.sqrt(dx[0] * dx[0] + dy[0] * dy[0]) == f32(0.2)) == kept
        assert order.tolist() == ([4, 5, 0, 2, 3, 1] if kept else [4, 5, 2, 3])


def test_slices_round_half_away_from_zero():
    z = np.array([0.1, -0.1, 0.29, 0.3, -0.3], f32)
    assert [k for k, _ in R.slices(np.stack([z * 0, z * 0, z], 1))] == [-2, -1, 1, 2]
    assert R.round_to_int(np.array([0.5, -0.5, 1.5, -2.5, 0.49999997], f32)).tolist() == [1, -1, 2, -3, 0]


def test_bucket_formula_edges():
    assert R.bucket_of([R.PI, -R.PI, 0.0, -0.0], 8).tolist() == [7, 0, 0, 0]
    assert R.bucket_of([R.PI / f32(2)], 8).tolist() == [4]            # 4 - 0.5 = 3.5 rounds away from zero
    assert R.bucket_of([R.PI, 1.0, -2.0], 1).tolist() == [0, 0, 0]


def random_clouds(rng):
    yield rng.uniform(-4, 4, (4000, 3)).astype(f32) * np.array([1, 1, 0.25], f32)
    yield (rng.normal(0, 2, (3000, 3)) * np.array([1, 1, 0.5])).astype(f32)
    pts = rng.uniform(-1.5, 1.5, (1500, 3)).astype(f32)               # coarse grid: many exact angle ties and axis deltas
    yield (np.round(pts * 4) / 4).astype(f32)


@pytest.mark.parametrize("size", SIZES)
def test_oracle_matches_the_model_on_cleaned_random_clouds(orc, size):
    rng = np.random.RandomState(size)
    for pts in random_clouds(rng):
        c = R.clean(pts, size)
        assert len(c) > 0.5 * len(pts)       # the grid cloud loses its 45 deg deltas to the boundaries of the even sizes
        want = R.compute_histogram(c, size)
        assert want.sum() > 1.0
        assert np.array_equal(bits(orc.compute_histogram(c, size)), bits(want))


def street_scans():
    """Returns of the synthetic street (helpers.workload, 16 beams) after ingest, gravity-aligned."""
    from helpers import apply_pose, workload
    import orc
    w = workload()
    for rows, prev, cur in zip(w["scans"], w["prev"], w["truth"]):
        pts = orc.ingest_scan(w["opts"], rows, w["origin"], prev, cur)["returns_tracking"]
        yield apply_pose(np.concatenate([[0, 0, 0], cur[3:7]]), pts.astype(np.float64)).astype(f32)


@pytest.mark.parametrize("size", SIZES)
def test_oracle_matches_the_model_on_the_cleaned_street(orc, size):
    for pts in list(street_scans())[:2]:
        c = R.clean(pts, size)
        want = R.compute_histogram(c, size)
        assert len(c) > 0.95 * len(pts) and want.sum() > 10.0
        assert np.array_equal(bits(orc.compute_histogram(c, size)), bits(want))


def test_uncleaned_street_differs_only_where_the_classifier_allows(orc):
    for pts in list(street_scans())[:2]:
        amb = R.ambiguous_points(pts, 120)
        want, got = R.compute_histogram(pts, 120), orc.compute_histogram(pts, 120)
        print(f"{len(pts)} points, {len(amb)} ambiguous, L1 oracle - model {np.abs(got - want).sum():.3g}")
        if len(amb) == 0:
            assert np.array_equal(bits(got), bits(want))


def test_classifier_flags_near_ties_and_boundaries_not_exact_ties():
    # two points whose angles around the centroid differ by ~1 ulp: both ambiguous; the same delta twice: an exact tie, not
    eps = np.spacing(f32(1.0))
    base = np.array([[1, 1, 0], [-1, 1, 0], [-1, -1, 0], [1, -1, 0]], f32)
    near = np.concatenate([base, np.array([[2, 0.5, 0], [2, 0.5 + eps, 0]], f32)])
    amb = R.ambiguous_points(near, 1)
    assert {4, 5} <= set(amb.tolist())
    same = np.concatenate([base, np.array([[2, 0.5, 0], [2, 0.5, 0]], f32)])
    assert not ({4, 5} & set(R.ambiguous_points(same, 1).tolist()))
    # B sorts first, then Q (2.7 m away: `last` = Q), then P: the walk delta P - Q = (-0.5, -0.5) lies at 45 deg (mod 180), on a
    # bucket boundary of 4 buckets and of none of 3
    pts = np.array([[-0.2, -3.0, 0], [0.5, 0.0, 0], [1.0, 0.5, 0]], f32)
    assert R.ambiguous_points(pts, 4).tolist() == [1] and R.ambiguous_points(pts, 3).tolist() == []
