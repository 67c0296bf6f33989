"""dl_rotational_histogram (RotationalScanMatcher::ComputeHistogram on the device) against the C++ oracle and the numpy reference
model, bit for bit, on clouds cleared of the points an atan2 implementation could decide either way
(rotational_histogram_reference.clean). The cases follow the kernel's edges: the walk's centroid of the sorted slice, points lost
to the 0.2 m rule, short and long slices, exact and near angle ties, signed zeros, slice keys, the sort's sizes and the limits."""
import numpy as np
import pytest

import rotational_histogram_reference as R
from test_rotational_histogram_oracle import SIZES, bits, pile_slice, ring, street_scans

pytestmark = pytest.mark.gpu
f32 = np.float32
DL_ERR_ARG = -2


@pytest.fixture(scope="module")
def ctx():
    import dliom
    c = dliom.Context(0)
    yield c
    c.close()


def check(ctx, orc, pts, size):
    """Device == oracle == model, bit for bit, on a cloud with no ambiguous point (asserted)."""
    pts = np.ascontiguousarray(pts, f32).reshape(-1, 3)
    assert len(R.ambiguous_points(pts, size)) == 0
    want = R.compute_histogram(pts, size)
    assert np.array_equal(bits(orc.compute_histogram(pts, size)), bits(want))
    got = ctx.rotational_histogram(pts, size)
    assert np.array_equal(bits(got), bits(want)), (np.flatnonzero(got != want)[:8], np.abs(got - want).sum())
    return want


def clean_all(pts):
    """The cloud without the points that are ambiguous for any of SIZES."""
    while True:
        c = pts
        for size in SIZES:
            c = R.clean(c, size)
        if len(c) == len(pts):
            return c
        pts = c


def cleaned_cloud(rng, n, make):
    """Exactly n points, none ambiguous for any of SIZES: ambiguous points are replaced by fresh ones until the cloud is clean."""
    pts = make(rng, n)
    while True:
        c = clean_all(pts)
        if len(c) == n:
            return c
        pts = np.concatenate([c, make(rng, n - len(c))])


def uniform(zmin, zmax, xy=3.0):
    return lambda rng, n: np.stack([rng.uniform(-xy, xy, n), rng.uniform(-xy, xy, n), rng.uniform(zmin, zmax, n)], 1).astype(f32)


def test_pile_uses_the_centroid_of_the_sorted_slice(ctx, orc):
    for size in (8, 120):
        assert len(R.clean(pile_slice(), size)) == 64
        check(ctx, orc, pile_slice(), size)


def test_slices_losing_none_one_or_all_points(ctx, orc):
    rng = np.random.RandomState(1)
    none = ring(1.5, 7.0 + 20.0 * np.arange(18), z=0.0)
    one = np.concatenate([ring(1.2, 3.0 + 24.0 * np.arange(15), z=0.4), [[0.05, -0.03, 0.4]]]).astype(f32)
    blob = np.concatenate([rng.uniform(-0.05, 0.05, (10, 2)), np.full((10, 1), 0.8)], 1).astype(f32)
    pts = np.concatenate([none, one, blob, pile_slice() + np.array([0, 0, 1.2], f32)])
    for size in SIZES:
        order, _, _, _ = R.sort_slice(one[:, 0], one[:, 1])
        assert len(order) == len(one) - 1 and len(R.sort_slice(blob[:, 0], blob[:, 1])[0]) == 0
        check(ctx, orc, R.clean(pts, size), size)
    # the lost blob contributes nothing: the cloud without it gives the same bits
    assert np.array_equal(bits(ctx.rotational_histogram(np.concatenate([none, one]), 120)),
                          bits(ctx.rotational_histogram(np.concatenate([none, one, blob]), 120)))


@pytest.mark.parametrize("count", [1, 2, 16, 17])
def test_slice_sizes(ctx, orc, count):
    rng = np.random.RandomState(count)
    make = lambda rng, n: np.concatenate([rng.uniform(-1.5, 1.5, (n, 2)), rng.uniform(-0.09, 0.09, (n, 1))], 1).astype(f32)
    slices = [cleaned_cloud(rng, count, make) + np.array([0, 0, 0.2 * k], f32) for k in range(6)]
    for size in SIZES:
        check(ctx, orc, R.clean(np.concatenate(slices), size), size)


def test_exact_ties_and_signed_zero_keep_input_order(ctx, orc):
    """Centroid exactly (0, +0). P1 = (1, +0) and P2 = (1.5, -0) tie at angle +-0 and keep input order: P1 is `last` when the walk
    reaches C, so C's delta is C - P1. A key that put -0 before +0 would make it C - P2."""
    pts = np.array([[1.0, 0.0, 0], [1.5, -0.0, 0], [1.25, 0.5, 0], [-2.0, -1.5, 0], [-1.75, 1.0, 0]], f32)
    order, (cx, cy), _, _ = R.sort_slice(pts[:, 0], pts[:, 1])
    assert order.tolist() == [3, 0, 1, 2, 4] and (cx, cy) == (0.0, 0.0) and not np.signbit(cy)
    pos, dx, dy, _ = R.walk(pts[order, 0], pts[order, 1])
    assert pos.tolist() == [2, 3] and (dx[1], dy[1]) == (f32(0.25), f32(0.5))
    for size in SIZES:
        want = check(ctx, orc, pts, size)
        assert want.sum() > 0.2
    # more ties on the axes (+-0, +-pi/2, +pi) in one slice of 16, in the other input order as well
    axes = np.array([[1, 0, 0], [2, -0.0, 0], [0.75, 0, 0], [0, 1, 0], [-0.0, 2, 0], [0, 0.5, 0], [-1, 0, 0], [-2.5, 0, 0],
                     [0, -1.25, 0], [0, -2, 0], [0.5, 0.5, 0], [-0.5, 0.75, 0], [0.75, -1.0, 0], [-1.5, -1.0, 0],
                     [1.25, 1.5, 0], [-0.25, -0.75, 0]], f32)
    for p in (axes, axes[::-1]):
        for size in SIZES:
            check(ctx, orc, R.clean(p, size), size)


def test_angles_sharing_the_sort_key_prefix(ctx, orc):
    """Angles 40 ulps apart inside one 256-ulp run of the key's 24 angle bits, in reverse input order: the exact-angle fix-up
    orders them. Each point has its mirror image next to it in input order, so the first centroid is exactly (0, 0)."""
    theta0 = np.float64(np.nextafter(f32(1.0), f32(2.0))) + 10 * np.spacing(f32(1.0))
    pts = []
    for k in reversed(range(6)):
        a = theta0 + 40 * k * np.spacing(f32(1.0))
        p = np.array([(1.0 + 0.5 * k) * np.cos(a), (1.0 + 0.5 * k) * np.sin(a), 0.0], f32)
        pts += [p, -p]
    pts = np.array(pts, f32)
    d = np.arctan2(pts[:, 1].astype(np.float64), pts[:, 0].astype(np.float64))
    prefix = (np.float32(d[0::2]).view(np.uint32) | np.uint32(0x80000000)) >> np.uint32(8)
    assert len(set(prefix.tolist())) == 1
    pts = np.concatenate([pts, ring(2.0, 11.0 + 30.0 * np.arange(12))])
    for size in SIZES:
        assert len(R.clean(pts, size)) == len(pts)
        check(ctx, orc, pts, size)


def test_slice_keys_round_half_away_and_the_slice_limit(ctx, orc):
    rng = np.random.RandomState(7)
    base = ring(1.0, 2.0 + 25.0 * np.arange(14))
    pts = np.concatenate([base + np.array([0, 0, z], f32) for z in (0.1, -0.1, 0.3, -0.3, 104857.4, -104857.6)])
    pts[:, :2] += rng.uniform(-0.02, 0.02, (len(pts), 2)).astype(f32)
    keys = [k for k, _ in R.slices(pts)]
    assert keys[0] == -(1 << 19) and keys[-1] == (1 << 19) - 1 and {-1, 1} <= set(keys)
    assert R.round_to_int(np.array([0.1, -0.1], f32) / f32(0.2)).tolist() == [1, -1]       # 0.1f / 0.2f is exactly 0.5
    for size in SIZES:
        check(ctx, orc, R.clean(pts, size), size)
    import dliom
    for z in (104857.6, -104857.8):
        beyond = np.concatenate([pts, [[0.5, 0.5, z]]]).astype(f32)
        assert R.round_to_int(f32(z) / f32(0.2)) in ((1 << 19), -(1 << 19) - 1)
        with pytest.raises(dliom.DlError) as e:
            ctx.rotational_histogram(beyond, 120)
        assert e.value.status == DL_ERR_ARG


@pytest.mark.parametrize("n", [1, 63, 64, 65, 1023, 1024, 1025])
def test_cloud_sizes_around_the_sort_padding(ctx, orc, n):
    pts = cleaned_cloud(np.random.RandomState(n), n, uniform(-0.5, 0.5))
    assert len(pts) == n
    for size in SIZES:
        check(ctx, orc, pts, size)


def test_more_than_1024_slices(ctx, orc):
    pts = cleaned_cloud(np.random.RandomState(3), 6000, uniform(-300.0, 300.0))
    assert len(R.slices(pts)) > 1024
    for size in SIZES:
        check(ctx, orc, pts, size)


def test_one_slice_of_more_than_1024_points(ctx, orc):
    pts = cleaned_cloud(np.random.RandomState(4), 3000, uniform(-0.09, 0.09, xy=4.0))
    assert len(R.slices(pts)) == 1
    for size in SIZES:
        check(ctx, orc, pts, size)


def test_2_pow_20_points_and_one_more(ctx, orc):
    """2^20 points on 4 slices, nearly all in a 0.1 m blob around each slice's centre (dropped by SortSlice), 2 000 on rings."""
    import dliom
    rng = np.random.RandomState(5)
    n = 1 << 20
    blob = np.concatenate([rng.uniform(-0.1, 0.1, (n, 2)), rng.randint(0, 4, (n, 1)) * 0.2], 1).astype(f32)
    for k in range(4):
        blob[n - 2000 + 500 * k: n - 1500 + 500 * k] = ring(2.0 + 0.1 * k, 360.0 * rng.uniform(0, 1, 500), z=0.2 * k)
    for size in (120, 1024):
        pts = blob
        while True:                            # refill with blob points at the centre: dropped, they decide no angle
            c = R.clean(pts, size)
            if len(c) == n:
                break
            pts = np.concatenate([c, np.zeros((n - len(c), 3), f32)])
        check(ctx, orc, pts, size)
    with pytest.raises(dliom.DlError) as e:
        ctx.rotational_histogram(np.zeros((n + 1, 3), f32), 120)
    assert e.value.status == DL_ERR_ARG


def test_histogram_sizes_and_empty_cloud(ctx, orc):
    import dliom
    pts = pile_slice()
    for size in (0, 1025, -1):
        with pytest.raises(dliom.DlError) as e:
            ctx.rotational_histogram(pts, size)
        assert e.value.status == DL_ERR_ARG
    for size in SIZES:
        assert not ctx.rotational_histogram(np.zeros((0, 3), f32), size).any()


def drive_scans():
    """The 16-beam drive of test_gpu_ltb.py, ingested and gravity-aligned; and one full-size 64-beam scan."""
    import orc
    import synth
    from helpers import apply_pose
    scene = synth.Scene(42)
    opts = orc.FrontEndOptions.defaults()
    out = []
    for beams, t in ((16, 2.0), (16, 2.1), (64, 2.0)):
        rows = synth.make_scan(scene, beams, t)
        pts = orc.ingest_scan(opts, rows, np.zeros((1, 3), np.float32), synth.pose7(t - 0.1), synth.pose7(t))["returns_tracking"]
        q = synth.pose7(t)[3:7]
        out.append(apply_pose(np.concatenate([[0, 0, 0], q]), pts.astype(np.float64)).astype(f32))
    return out


@pytest.fixture(scope="module")
def scenes():
    return drive_scans() + list(street_scans())[:1]


@pytest.mark.parametrize("size", [7, 120, 1024])
def test_scene_clouds_cleaned(ctx, orc, scenes, size):
    for pts in scenes:
        c = R.clean(pts, size)
        # every removal moves its slice's centroid and with it every angle of the slice: on the 64-beam scan's ground slice
        # (9 000 points) new near ties keep appearing, and a third of the scan goes before none is left
        assert len(c) > 0.6 * len(pts)
        want = check(ctx, orc, c, size)
        assert want.sum() > 10.0


def test_scene_clouds_uncleaned_differ_only_at_ambiguous_points(ctx, orc, scenes):
    for pts in scenes:
        amb = R.ambiguous_points(pts, 120)
        want = orc.compute_histogram(pts, 120)
        got = ctx.rotational_histogram(pts, 120)
        diff = np.abs(got - want)
        print(f"{len(pts)} points, {len(amb)} ambiguous, {np.count_nonzero(diff)} buckets differ, L1 {diff.sum():.3g} "
              f"of {want.sum():.4g}")
        if len(amb) == 0:
            assert np.array_equal(bits(got), bits(want))
