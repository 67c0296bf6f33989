"""CPU checks of tests/submap_image_reference.py (AddToTextureProto / ProjectToCvMat restated in float32 numpy) on hand-worked
cases; the device is compared with it in tests/test_gpu_submap_images.py."""
import math

import numpy as np

import submap_image_reference as ref

F = np.float32
IDENTITY = np.array([0, 0, 0, 1, 0, 0, 0], np.float64)


def value_of(p):
    """The grid value whose probability is the float just at or above p."""
    v = np.arange(1, 32768)
    return int(v[np.searchsorted(ref.value_to_probability(v), F(p))])


def test_sum_follows_iterator_order_and_the_order_matters():
    # one column, 5 cells at z = -70, -3, 0, 5, 64 (three top cells); input order scrambled
    zs = np.array([64, 0, -70, 5, -3])
    vals = np.array([29799, 30130, 30581, 25254, 28758])  # iterator order: 30581 28758 30130 25254 29799
    xs = ys = np.zeros(5, np.int64)
    order = ref.iterator_order(xs, ys, zs)
    assert zs[order].tolist() == [-70, -3, 0, 5, 64]
    p = ref.value_to_probability(vals[order])
    forward = F(0)
    for v in p:
        forward = F(forward + v)
    backward = F(0)
    for v in p[::-1]:
        backward = F(backward + v)
    assert forward != backward  # the order check has teeth
    got = ref.projection(xs, ys, zs, vals, 1.0, IDENTITY)
    assert got["pixels"].tolist() == [[int(ref.lround(F(forward - F(0.1)) * F(F(255) / F(ref.K_MAX - ref.K_MIN)))[()]) & 255]]


# One column (x = y = 0) across 64- and 8-cell boundaries: iterator order is z ascending. The values were searched so that the
# pixel's output byte under the reverse summation order differs from the byte under iterator order.
ORDER_Z = [-70, -66, -9, -3, 0, 5, 7, 63, 64, 71, 130]
ORDER_PROJECTION_VALUES = [22248, 26698, 26950, 24269, 29076, 21373, 18697, 17727, 32513, 29663, 31653]
ORDER_TEXTURE_VALUES = [23515, 26482, 21870, 16570, 26246, 20683, 23069, 20206, 19445, 29639, 31459]


_ITERATOR_ORDER = ref.iterator_order


def reversed_iterator_order(xs, ys, zs):
    return _ITERATOR_ORDER(xs, ys, zs)[::-1]


def order_case(values):
    """The column's cells listed in descending z (neither iterator order nor its image in a fresh grid's brick pool)."""
    n = len(ORDER_Z)
    return np.zeros(n, np.int64), np.zeros(n, np.int64), np.array(ORDER_Z[::-1]), np.array(values[::-1])


def test_output_bytes_depend_on_the_summation_order(monkeypatch):
    for resolution in (1.0, 0.2):
        proj = ref.projection(*order_case(ORDER_PROJECTION_VALUES), resolution, IDENTITY)
        tex = ref.texture(*order_case(ORDER_TEXTURE_VALUES), resolution, IDENTITY)
        with monkeypatch.context() as m:
            m.setattr(ref, "iterator_order", reversed_iterator_order)
            proj_reversed = ref.projection(*order_case(ORDER_PROJECTION_VALUES), resolution, IDENTITY)
            tex_reversed = ref.texture(*order_case(ORDER_TEXTURE_VALUES), resolution, IDENTITY)
        assert proj["pixels"].tolist() == [[201]] and proj_reversed["pixels"].tolist() == [[200]]
        assert tex["cells"].tolist() == [[[53, 0]]] and tex_reversed["cells"].tolist() == [[[54, 0]]]


def test_iterator_order_with_negative_indices():
    xs = np.array([0, -1, 7, 8, -64, 63])
    order = ref.iterator_order(xs, np.zeros(6, np.int64), np.zeros(6, np.int64))
    assert xs[order].tolist() == [-64, -1, 0, 7, 8, 63]
    # z % 8 before y % 8 before x % 8 inside a brick; the brick's slot in its node before that
    xs, ys, zs = np.array([1, 0, 0, 0]), np.array([0, 1, 0, 0]), np.array([0, 0, 1, 8])
    assert ref.iterator_order(xs, ys, zs).tolist() == [0, 1, 2, 3]


def test_obstructed_limit_either_side_of_0_501():
    below, at = value_of(0.501) - 1, value_of(0.501)
    assert ref.value_to_probability([below])[0] < F(0.501) <= ref.value_to_probability([at])[0]
    for v, width in ((below, 0), (at, 1)):
        assert ref.projection([3], [4], [0], [v], 0.5, IDENTITY)["width"] == width
        assert ref.texture([3], [4], [0], [v], 0.5, IDENTITY)["width"] == width


def test_texture_z_difference_and_free_space():
    # z_difference 2: (0, 0); 3 with 4 cells: free_space 0, average = sum / 4 of probability 0.9 -> 255 -> delta -127
    assert ref.pixel_value(3, 0, 2, F(2.7), F(0.9)) == (0, 0)
    assert ref.pixel_value(4, 0, 3, F(4 * 0.9), F(0.9)) == (0, 127)
    # free_space > 0: 2 cells over z_difference 6 -> free_space 4, weight 0.6 toward 1 - max_probability
    count, s, mp = 2, F(F(0.9) + F(0.7)), F(0.9)
    fsw = F(F(0.15) * F(4))
    avg = F(F(s + F(F(F(1) - mp) * fsw)) / F(F(count) + fsw))
    assert ref.pixel_value(count, 0, 6, s, mp) == (0, ref.log_odds_integer(avg) - 128)
    assert avg < F(s / F(2))


def test_texture_clamps_at_both_ends_and_delta_0_gives_alpha_1():
    assert ref.pixel_value(4, 0, 3, F(4.0), F(0.9)) == ref.pixel_value(4, 0, 3, F(3.6), F(0.9)) == (0, 127)   # average 1 -> 0.9
    assert ref.pixel_value(4, 0, 3, F(0.0), F(0.9)) == ref.pixel_value(4, 0, 3, F(0.4), F(0.9)) == (127, 0)   # 0 -> 0.1
    assert ref.log_odds_integer(F(0.5)) == 128
    assert ref.pixel_value(4, 0, 3, F(2.0), F(0.5)) == (0, 1)


def test_projection_wraps_above_255_and_below_0():
    xs, ys = np.array([0, 0, 0, 0, 2]), np.array([0, 0, 0, 0, 0])
    zs, vals = np.array([0, 1, 2, 3, 0]), np.array([32767] * 5)
    got = ref.projection(xs, ys, zs, vals, 1.0, IDENTITY)
    s = F(0)
    for _ in range(4):
        s = F(s + F(0.9))
    dense = int(ref.lround(F(s - F(0.1)) * F(F(255) / F(ref.K_MAX - ref.K_MIN)))[()])
    assert dense > 255 and got["pixels"].tolist() == [[dense & 255, 224, 255]]
    assert int(ref.lround(F(F(0) - F(0.1)) * F(318.75))[()]) == -32  # the empty pixel: -32 -> 224
    assert (got["width"], got["height"], got["ox"], got["oy"]) == (3, 1, 0.0, 0.0)


def test_texture_layout_and_slice_pose():
    # cells at (x, y) = (1, 2) and (3, -1): height = 3, width = 4, (max_x - x) * width + (max_y - y)
    xs, ys = np.repeat([1, 3], 4), np.repeat([2, -1], 4)
    zs, vals = np.tile([0, 1, 2, 3], 2), np.full(8, 32767)
    t = ref.texture(xs, ys, zs, vals, 0.5, IDENTITY)
    assert (t["width"], t["height"]) == (4, 3)
    lit = np.argwhere(t["cells"][..., 1] > 0).tolist()
    assert lit == [[0, 3], [2, 0]]
    assert t["slice_pose"].tolist() == [1.5, 1.0, 0.0, 1.0, 0.0, 0.0, 0.0]


def test_projection_removes_yaw_and_keeps_roll_and_pitch():
    def pose(yaw, roll, pitch):
        cy, sy, cp, sp, cr, sr = (f(a / 2) for a in (yaw, pitch, roll) for f in (math.cos, math.sin))
        return np.array([5, 6, 7, cy * cp * cr + sy * sp * sr, cy * cp * sr - sy * sp * cr, cy * sp * cr + sy * cp * sr,
                         sy * cp * cr - cy * sp * sr])
    q = ref.projection_rotation(pose(1.1, 0.0, 0.0))
    assert abs(float(q[0]) - 1) < 1e-6 and max(abs(float(c)) for c in q[1:]) < 1e-6
    q = ref.projection_rotation(pose(-2.5, 0.2, -0.1))
    d = ref.rotate(tuple(float(c) for c in q), (1.0, 0.0, 0.0), dtype=np.float64)
    assert abs(math.atan2(float(d[1]), float(d[0]))) < 1e-6      # no yaw left
    assert abs(float(d[2]) - math.sin(0.1)) < 1e-6                 # the pitch stays
    cells = ref.projection([10, -4], [0, 3], [0, 0], [32767, 32767], 0.25, pose(0.8, 0.0, 0.0))
    assert (cells["width"], cells["height"], cells["ox"], cells["oy"]) == (15, 4, -1.0, 0.0)


def test_cpp_submap_images_example_compiles_and_fails_loudly_without_a_gpu(tmp_path):
    """host/example_submap_images.cc builds with -Wall -Werror; without a device it reports the error and exits 2."""
    import struct
    import subprocess
    import pytest
    import dliom
    from test_gpu_submap_images import build_example
    exe = build_example(tmp_path)
    try:
        dliom.Context(0).close()
        pytest.skip("a GPU is present: tests/test_gpu_submap_images.py runs the example")
    except dliom.DlError:
        pass
    path = str(tmp_path / "drive.bin")
    with open(path, "wb") as f:
        f.write(struct.pack("<ii", 0, 0))
    r = subprocess.run([exe, path, str(tmp_path)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 2 and "dliom error" in r.stderr and r.stdout == ""
