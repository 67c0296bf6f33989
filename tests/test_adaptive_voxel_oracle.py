"""The adaptive voxel filter: the numpy reference model (adaptive_voxel_reference.py) against results worked out by hand, and the
C++ oracle (orc.adaptive_voxel_filter) against the model bit for bit, survivors and pass edges, on every cloud of
adaptive_voxel_cases.py (the clouds the GPU test runs on the device's edges)."""
import numpy as np
import pytest

import adaptive_voxel_cases as K
import adaptive_voxel_reference as R

f32 = np.float32
CASES = K.all_cases()


def bits(passes):
    return np.asarray(passes, f32).view(np.uint32)


def test_lround_ties_away_from_zero_in_float64():
    q = np.array([0.5, -0.5, 1.5, -2.5, 2.5, np.nextafter(f32(0.5), f32(0)), -np.nextafter(f32(0.5), f32(0)), 0.0, -0.0], f32)
    assert R.round_to_int(q).tolist() == [1, -1, 2, -3, 3, 0, 0, 0, 0]
    # the float32 reading would move the largest float below a half up to the next cell
    assert np.floor(q[5] + f32(0.5)) == 1.0
    # the quotient is rounded to float32 first: 0.3f / 0.2f is the tie 1.5 (-> 2, -2 away from zero), 0.45f / 0.3f is 1.4999999
    assert np.float32(0.3) / np.float32(0.2) == 1.5 and np.float32(0.45) / np.float32(0.3) < 1.5
    assert R.cells(np.array([[0.3, 0.45, -0.3]], f32), 0.2).tolist() == [[2, 2, -2]]
    assert R.cells(np.array([[0.45, 0.0, 0.0]], f32), 0.3).tolist() == [[1, 0, 0]]


def test_crop_uses_eigen_order_and_drops_nan():
    pts = np.array([[5, 12, 0], [5, np.nextafter(f32(12), f32(13)), 0], [np.nan, 0, 0], [0, np.inf, 0], [0, 0, -13]], f32)
    assert R.crop(pts, 13.0).tolist() == [0, 4]
    stride8 = np.full((5, 8), np.nan, f32)
    stride8[:, :3] = pts
    assert R.crop(stride8, 13.0).tolist() == [0, 4]


def test_first_point_per_voxel_in_input_order():
    pc = np.array([[0, 0, 0], [0.1, -0.1, 0.1], [0.3, -0.1, 0], [0, 0, 0.1]], f32)
    assert R.voxel_filter(pc, 0.3).tolist() == [0, 2]
    pc = np.array([[1, 1, 1], [5, 5, 5], [1.1, 1, 1], [5.1, 5, 5], [-1, 0, 0]], f32)[::-1]
    assert R.voxel_filter(pc, 1.0).tolist() == [0, 1, 2]


def test_bisection_by_hand():
    """Three points on the x axis at 0, 0.3 and 0.6 m, max_length 1, min_num_points 2.5: 1 m -> cells 0 0 1 (2 voxels), 0.5 m ->
    0 1 1 (2), 0.25 m -> 0 1 2 (3, enough); refine between 0.25 and 0.5: 0.375 -> 0 1 2 (3, low = 0.375), 0.4375 -> 0 1 1 (2, high),
    0.40625 -> 0 1 1 (2, high); (0.40625 - 0.375) / 0.375 < 0.1 stops. The result is the 0.375 pass: all three points."""
    pts = np.array([[0, 0, 0], [0.3, 0, 0], [0.6, 0, 0]], f32)
    keep, passes, edge = R.search(pts, 1.0, 2.5, 10.0)
    assert passes.tolist() == [1.0, 0.5, 0.25, 0.375, 0.4375, 0.40625] and edge == f32(0.375) and keep.tolist() == [0, 1, 2]
    # min_num_points is a float: 3 points are sparse enough for 3, not for 2.9999
    assert R.search(pts, 1.0, 3.0, 10.0)[1].tolist() == []
    assert len(R.search(pts, 1.0, f32(2.9999), 10.0)[1]) == 6
    # the first edge suffices at 2 voxels for min_num_points 2
    assert R.search(pts, 1.0, 2.0, 10.0)[1].tolist() == [1.0]


def test_exhausted_search_returns_the_last_halving():
    pts = np.tile(np.array([[0.2, 0.1, 0.0]], f32), (5, 1))
    keep, passes, edge = R.search(pts, 2.0, 2.0, 10.0)
    assert passes.tolist() == [2.0 / 2 ** j for j in range(8)] and edge == f32(2.0 / 128) and keep.tolist() == [0]


def test_crop_keeps_input_indices():
    pts = np.array([[100, 0, 0], [0, 0, 0], [100, 0, 0], [0.1, 0, 0], [3, 0, 0]], f32)
    keep, passes = R.adaptive_voxel_filter(pts, 1.0, 1.0, 10.0)
    assert keep.tolist() == [1, 4] and passes.tolist() == [1.0]


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_oracle_matches_the_model(orc, case):
    want_keep, want_passes = R.adaptive_voxel_filter(case.rows, *case.opts)
    if len(case.rows) == 0:
        assert len(want_keep) == 0 and len(want_passes) == 0
    keep, passes = orc.adaptive_voxel_filter(case.rows, *case.opts)
    assert np.array_equal(keep, want_keep)
    assert np.array_equal(bits(passes), bits(want_passes))


@pytest.mark.parametrize("which", [0, 1], ids=["high_resolution", "low_resolution"])
def test_oracle_matches_the_model_on_a_shuffled_street_scan(orc, which):
    case = K.street_cases(orc)[which]
    want_keep, want_passes = R.adaptive_voxel_filter(case.rows, *case.opts)
    keep, passes = orc.adaptive_voxel_filter(case.rows, *case.opts)
    assert len(want_keep) > 100 and np.array_equal(keep, want_keep)
    assert np.array_equal(bits(passes), bits(want_passes))
