"""The float32 reference of the range-data map (tests/range_data_map_reference.py), pinned without a GPU: against an fp64
evaluation of the same float poses, on the identities the arithmetic must keep, and on its output order and offsets. Also
builds host/example_range_data_map.cc and checks that it fails loudly without a device."""
import os

import numpy as np
import pytest

import range_data_map_reference as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def random_pose(rng, scale=50.0):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    return np.concatenate([rng.uniform(-scale, scale, 3), q])


def fp64_points(local7, global7, returns):
    """Matrix form in float64 of the float-cast poses: R_G (R_L^T (p - t_L)) + t_G, with R from the (non-renormalised)
    float quaternion through its unit rotation matrix, which it equals to float rounding."""
    def matrix(q):
        w, x, y, z = np.asarray(q, np.float64) / np.linalg.norm(np.asarray(q, np.float64))
        return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                         [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                         [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
    lt, lq = ref.cast_float(local7)
    gt, gq = ref.cast_float(global7)
    p = np.asarray(returns, np.float64)
    tp = (p - lt.astype(np.float64)) @ matrix(lq)
    return tp @ matrix(gq).T + gt.astype(np.float64)


def test_reference_against_fp64():
    rng = np.random.default_rng(7)
    worst = 0.0
    for _ in range(20):
        local7, global7 = random_pose(rng), random_pose(rng)
        returns = rng.uniform(-80, 80, (2000, 3)).astype(np.float32)
        got = ref.node_points(local7, global7, returns).astype(np.float64)
        want = fp64_points(local7, global7, returns)
        scale = np.abs(returns).max() + np.abs(local7[:3]).max() + np.abs(global7[:3]).max()
        err = np.abs(got - want).max() / scale
        worst = max(worst, err)
    assert worst < 8 * np.finfo(np.float32).eps, worst
    print(f"largest error against fp64, relative to the coordinate scale: {worst:.3g}")


def test_identity_poses_return_the_points_bit_for_bit():
    rng = np.random.default_rng(1)
    returns = rng.uniform(-100, 100, (1000, 3)).astype(np.float32)
    identity = np.array([0, 0, 0, 1, 0, 0, 0], np.float64)
    assert np.array_equal(ref.node_points(identity, identity, returns), returns)


def test_equal_local_and_global_pose_return_the_points_to_rounding():
    rng = np.random.default_rng(2)
    for _ in range(10):
        pose = random_pose(rng)
        returns = rng.uniform(-60, 60, (1000, 3)).astype(np.float32)
        got = ref.node_points(pose, pose, returns)
        scale = np.abs(returns).max() + np.abs(pose[:3]).max()
        assert np.abs(got - returns).max() <= 8 * np.finfo(np.float32).eps * scale


def test_negated_quaternions_give_the_same_points():
    """-q rotates like q. In this operation order every product and cross product meets two negated factors, and IEEE negation
    is exact, so the result is not only equal to rounding but bit for bit."""
    rng = np.random.default_rng(3)
    for _ in range(10):
        local7, global7 = random_pose(rng), random_pose(rng)
        returns = rng.uniform(-60, 60, (500, 3)).astype(np.float32)
        want = ref.node_points(local7, global7, returns)
        for neg_local, neg_global in ((True, False), (False, True), (True, True)):
            l7, g7 = local7.copy(), global7.copy()
            if neg_local:
                l7[3:] = -l7[3:]
            if neg_global:
                g7[3:] = -g7[3:]
            got = ref.node_points(l7, g7, returns)
            scale = np.abs(returns).max() + np.abs(local7[:3]).max() + np.abs(global7[:3]).max()
            assert np.abs(got - want).max() <= 4 * np.finfo(np.float32).eps * scale
            assert np.array_equal(got, want)


def test_order_and_offsets():
    rng = np.random.default_rng(4)
    nodes = []
    for t, i, n in [(3, 5, 10), (0, 2, 7), (3, 1, 0), (0, 0, 4), (1, 9, 1)]:
        nodes.append((t, i, random_pose(rng), random_pose(rng), rng.uniform(-5, 5, (n, 3)).astype(np.float32)))
    points, table = ref.range_data_map(nodes)
    assert [(t, i) for t, i, _, _ in table] == [(0, 0), (0, 2), (1, 9), (3, 1), (3, 5)]
    assert [(f, n) for _, _, f, n in table] == [(0, 4), (4, 7), (11, 1), (12, 0), (12, 10)]
    assert points.shape == (22, 3) and points.dtype == np.float32
    by_id = {(t, i): (l7, g7, r) for t, i, l7, g7, r in nodes}
    for t, i, f, n in table:
        assert np.array_equal(points[f:f + n], ref.node_points(*by_id[(t, i)]))
    empty, none = ref.range_data_map([])
    assert empty.shape == (0, 3) and none == []


def test_cpp_range_data_map_example_compiles_and_fails_loudly_without_a_gpu(tmp_path):
    """host/example_range_data_map.cc (mapping::PoseGraph3D::EnableRangeDataCache / RangeDataMap) builds with -Wall -Werror;
    without a device it exits with status 2 and a dliom error, writing no map."""
    import subprocess
    import dliom
    exe = build_range_data_map_example(tmp_path)
    try:
        dliom.Context(0).close()
        pytest.skip("a GPU is present: tests/test_gpu_range_data_map.py runs the example")
    except dliom.DlError:
        pass
    drive = tmp_path / "drive.bin"
    drive.write_bytes(b"")
    r = subprocess.run([exe, str(drive), str(tmp_path / "map.pcd")], capture_output=True, text=True, timeout=120)
    assert r.returncode == 2 and "dliom error" in r.stderr and r.stdout == ""
    assert not (tmp_path / "map.pcd").exists()


def test_c_abi_argument_checks_without_a_graph():
    import ctypes as C
    import dliom
    L = dliom.lib()
    assert C.sizeof(dliom.RangeDataMapNode) == 80
    n, m = C.c_int32(0), C.c_int64(0)
    assert L.dl_range_data_map_set_node(None, 0, 0, None, 0) == -2
    assert L.dl_range_data_map(None, 0, None, 0, None, C.byref(n), 0, None, C.byref(m)) == -2
    assert L.dl_range_data_map_dev(None, 0, None, 0, None, C.byref(n), 0, None, C.byref(m)) == -2


def build_range_data_map_example(out_dir):
    import subprocess
    host = os.path.join(ROOT, "d-liom_b200", "host")
    exe = os.path.join(str(out_dir), "example_range_data_map")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", os.path.join(host, "example_range_data_map.cc"), "-o",
                           exe, "-L" + os.path.join(ROOT, "d-liom_b200"), "-ldliom_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "d-liom_b200")])
    return exe
