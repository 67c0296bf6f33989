"""The block-sparse (Schur) pose-graph oracle (tests/schur_oracle.py) pinned to the dense oracle (oracle/orc_posegraph.h) on
small graphs: the same LM trajectory (iterations, termination) and the same poses to 1e-10, so that it can stand in for the dense
oracle at sizes the dense one cannot hold. Then the frozen poses of OptimizationProblem3D::Solve's frozen_trajectories, and the
C-ABI surface of the device's sparse solve (no GPU needed)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import schur_oracle
from test_posegraph_oracle import aa_to_q, angle, compose, inverse, qmul

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IDENT = np.array([0, 0, 0, 1.0, 0, 0, 0])


def same_poses(a, b, tol):
    for p, q in zip(a, b):
        rel = compose(inverse(np.asarray(q)), np.asarray(p))
        assert np.linalg.norm(rel[:3]) < tol and angle(rel) < tol, (p, q)


def same_as_dense(orc, submaps, nodes, cons, fix_z=False, max_iter=50):
    ws, wn, wsum = orc.pose_graph_solve(submaps, nodes, cons, fix_z=fix_z, max_iter=max_iter)
    ss, sn, ssum = schur_oracle.solve(orc, submaps, nodes, cons, fix_z=fix_z, max_iter=max_iter)
    assert ssum["num_iterations"] == wsum["num_iterations"]
    assert ssum["termination"] == wsum["termination"]
    assert ssum["num_successful_steps"] == wsum["num_successful_steps"]
    assert abs(ssum["initial_cost"] - wsum["initial_cost"]) <= 1e-12 * max(wsum["initial_cost"], 1.0)
    assert abs(ssum["final_cost"] - wsum["final_cost"]) <= 1e-9 * max(wsum["final_cost"], 1e-12)
    same_poses(ss, ws, 1e-10)
    same_poses(sn, wn, 1e-10)
    return ss, sn, ssum


def reduces_noise_graph(n=100):
    """optimization_problem_3d_test.cc:106-196 with the oracle's construction (tests/test_posegraph_oracle.py)."""
    rng = np.random.default_rng(0)

    def random_transform(ts, rs):
        return np.array([*rng.uniform(-ts, ts, 3), *aa_to_q(rng.uniform(-rs, rs, 3))])

    def random_yaw_only(ts, rs):
        return np.array([*rng.uniform(-ts, ts, 3), *aa_to_q([0, 0, rng.uniform(-rs, rs)])])

    def add_noise(t, noise):
        return np.array([*(t[:3] + noise[:3]), *qmul(noise[3:], t[3:])])
    truth = [random_transform(10.0, 3.0) for _ in range(n)]
    noise = [random_yaw_only(0.2, 0.3) for _ in range(n)]
    nodes = [add_noise(t, z) for t, z in zip(truth, noise)]
    submap2 = np.array([0, 0, 0, *aa_to_q([0, 0, np.pi])])
    cons = []
    for j in range(n):
        cons.append((0, j, add_noise(truth[j], noise[j]), 1.0, 1.0))
        cons.append((1, j, add_noise(truth[j], random_yaw_only(0.2, 0.3)), 1.0, 1.0))
        cons.append((2, j, compose(compose(inverse(submap2), truth[j]), random_transform(1e3, 3.0)), 1e-9, 1e-9))
    return [IDENT, IDENT, submap2], nodes, cons, truth


def exact_recovery_graph():
    rng = np.random.default_rng(2)
    submaps = [IDENT, np.array([4.0, 1.0, 0.2, *aa_to_q([0, 0, 0.5])])]
    truth = [np.array([*rng.uniform(-8, 8, 3), *aa_to_q(rng.uniform(-0.6, 0.6, 3))]) for _ in range(12)]
    cons = [(s, n, compose(inverse(submaps[s]), truth[n]), 1.0, 1.0) for s in range(2) for n in range(12)]
    start_nodes = [compose(t, np.array([*rng.uniform(-0.5, 0.5, 3), *aa_to_q(rng.uniform(-0.2, 0.2, 3))])) for t in truth]
    start_submaps = [submaps[0], compose(submaps[1], np.array([0.3, -0.2, 0.1, *aa_to_q([0.02, -0.03, 0.1])]))]
    return start_submaps, start_nodes, cons


def trajectory_graph(num_submaps, num_nodes, loops_every=5, seed=3):
    """A drive: node k is seen by its two active submaps (consecutive) and, every few nodes, by one older submap (loop closure)."""
    rng = np.random.default_rng(seed)
    per = max(num_nodes // num_submaps, 1)
    truth_s = [IDENT] + [np.array([3.0 * s, np.sin(s), 0.1 * s, *aa_to_q([0, 0, 0.05 * s])]) for s in range(1, num_submaps)]
    truth_n = [np.array([3.0 * k / per, np.sin(k / per) + 0.3, 0.1 * k / per, *aa_to_q([0.01, -0.02, 0.05 * k / per])])
               for k in range(num_nodes)]
    cons = []
    for k in range(num_nodes):
        first = min(k // per, num_submaps - 1)
        seen = {first, min(first + 1, num_submaps - 1)}
        if k % loops_every == 0 and first > 1:
            seen.add(int(rng.integers(0, first - 1)))
        for s in sorted(seen):
            noise = np.array([*rng.normal(0, 0.02, 3), *aa_to_q(rng.normal(0, 0.005, 3))])
            cons.append((s, k, compose(compose(inverse(truth_s[s]), truth_n[k]), noise), 1.1e4 ** 0.5, 1e5 ** 0.5))
    start_s = [truth_s[0]] + [compose(t, np.array([*rng.uniform(-0.2, 0.2, 3), *aa_to_q(rng.uniform(-0.03, 0.03, 3))]))
                              for t in truth_s[1:]]
    start_n = [compose(t, np.array([*rng.uniform(-0.3, 0.3, 3), *aa_to_q(rng.uniform(-0.05, 0.05, 3))])) for t in truth_n]
    return start_s, start_n, cons


def test_schur_matches_dense_reduces_noise(orc):
    submaps, nodes, cons, truth = reduces_noise_graph()
    _, sn, _ = same_as_dense(orc, submaps, nodes, cons)
    before = sum(np.linalg.norm(t[:3] - p[:3]) for t, p in zip(truth, nodes))
    after = sum(np.linalg.norm(t[:3] - p[:3]) for t, p in zip(truth, sn))
    assert 0.8 * before > after


def test_schur_matches_dense_exact_recovery(orc):
    submaps, nodes, cons = exact_recovery_graph()
    _, _, s = same_as_dense(orc, submaps, nodes, cons)
    assert s["termination"] == 0 and s["final_cost"] < 1e-12 * max(s["initial_cost"], 1.0)


def test_schur_matches_dense_fix_z(orc):
    rng = np.random.default_rng(4)
    truth = [np.array([*rng.uniform(-5, 5, 3), *aa_to_q(rng.uniform(-0.3, 0.3, 3))]) for _ in range(6)]
    lifted = [t + np.array([0.2, -0.1, 0.4, 0, 0, 0, 0]) for t in truth]
    cons = [(0, k, truth[k], 1.0, 1.0) for k in range(6)]
    _, sn, _ = same_as_dense(orc, [IDENT], lifted, cons, fix_z=True)
    assert all(a[2] == b[2] for a, b in zip(sn, lifted))
    s3, n3, c3 = trajectory_graph(4, 24)
    same_as_dense(orc, s3, n3, c3, fix_z=True)


def test_schur_matches_dense_single_view_and_unconstrained_nodes(orc):
    submaps, nodes, cons = trajectory_graph(4, 24)
    cons = [c for c in cons if not (c[1] == 7 and c[0] != min(c[0] for c in cons if c[1] == 7))]   # node 7: one submap only
    cons = [c for c in cons if c[1] != 11]                                                          # node 11: no constraint
    assert sum(c[1] == 7 for c in cons) == 1
    _, sn, _ = same_as_dense(orc, submaps, nodes, cons)
    assert np.array_equal(sn[11], nodes[11])


def test_schur_trajectory_shape_with_loop_closures(orc):
    submaps, nodes, cons = trajectory_graph(6, 60, loops_every=3)
    same_as_dense(orc, submaps, nodes, cons)


def test_frozen_poses_stay_bit_unchanged(orc):
    submaps, nodes, cons = trajectory_graph(5, 40)
    frozen = np.zeros(45, bool)
    frozen[[2, 3]] = True            # two submaps
    frozen[5 + np.arange(10, 20)] = True
    ss, sn, s = schur_oracle.solve(orc, submaps, nodes, cons, frozen=frozen)
    out = np.concatenate([ss, sn])
    start = np.concatenate([submaps, nodes])
    assert np.array_equal(out[frozen], start[frozen])
    assert not np.array_equal(out[~frozen][1:], start[~frozen][1:])
    assert s["final_cost"] < 0.5 * s["initial_cost"] and s["num_reduced_parameters"] == 2 + 6 * 2


def test_frozen_first_submap_keeps_its_rotation(orc):
    submaps, nodes, cons = trajectory_graph(3, 18)
    frozen = np.zeros(21, bool)
    frozen[0] = True
    ss, sn, s = schur_oracle.solve(orc, submaps, nodes, cons, frozen=frozen)
    assert np.array_equal(ss[0], submaps[0]) and s["num_reduced_parameters"] == 6 * 2
    free, _, _ = schur_oracle.solve(orc, submaps, nodes, cons)
    assert not np.array_equal(free[0], submaps[0])    # unfrozen, its roll and pitch move


def test_constraints_between_frozen_poses_add_a_fixed_cost(orc):
    submaps, nodes, cons = trajectory_graph(4, 24)
    frozen = np.zeros(28, bool)
    frozen[[1, 4 + 3, 4 + 4]] = True
    extra = [(1, 3, compose(compose(inverse(submaps[1]), nodes[3]), np.array([0.1, 0, 0, 1.0, 0, 0, 0])), 2.0, 1.0),
             (1, 4, compose(inverse(submaps[1]), nodes[4]), 1.0, 1.0)]
    a = schur_oracle.solve(orc, submaps, nodes, cons, frozen=frozen)
    b = schur_oracle.solve(orc, submaps, nodes, cons + extra, frozen=frozen)
    fixed = 0.5 * (0.1 * 2.0) ** 2      # the first extra constraint is off by 0.1 m along x, weight 2; the second is exact
    assert a[2]["num_iterations"] == b[2]["num_iterations"] and a[2]["num_pairs"] == b[2]["num_pairs"]
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert abs(b[2]["initial_cost"] - a[2]["initial_cost"] - fixed) < 1e-14 * a[2]["initial_cost"]
    assert abs(b[2]["final_cost"] - a[2]["final_cost"] - fixed) < 1e-12


def test_all_frozen_returns_at_once(orc):
    submaps, nodes, cons = trajectory_graph(2, 6)
    ss, sn, s = schur_oracle.solve(orc, submaps, nodes, cons, frozen=np.ones(8, bool))
    assert np.array_equal(ss, np.asarray(submaps)) and np.array_equal(sn, np.asarray(nodes))
    assert s["termination"] == 0 and s["num_iterations"] == 0 and s["initial_cost"] == s["final_cost"] > 0


# ---- the C-ABI and C++ surface (no GPU)
def header():
    with open(os.path.join(ROOT, "include", "dliom_b200.h")) as f:
        return f.read()


def test_sparse_symbol_is_exported_and_structs_match_the_header():
    import dliom
    assert "dl_pose_graph_solve_sparse" in dliom.EXPORTS
    assert hasattr(dliom.lib(), "dl_pose_graph_solve_sparse")
    body = re.search(r"typedef struct dl_pose_graph_sparse_info \{(.*?)\} dl_pose_graph_sparse_info;", header(), re.S).group(1)
    fields = re.findall(r"^\s*(int32_t|int64_t|float|double)\s+(\w+);", body, re.M)
    assert [n for _, n in fields] == [n for n, _ in dliom.PoseGraphSparseInfo._fields_]
    size = {"int32_t": 4, "int64_t": 8, "float": 4, "double": 8}
    assert C.sizeof(dliom.PoseGraphSparseInfo) == sum(size[t] for t, _ in fields) == 40
    assert C.sizeof(dliom.SpaConstraint) == 4 + 4 + 8 * 9


def have_gpu():
    import dliom
    try:
        dliom.Context(0).close()
        return True
    except dliom.DlError:
        return False


def test_sparse_call_without_a_gpu_fails_loudly():
    """The entry point rejects a missing context before touching a device; without a device the context cannot be made."""
    import dliom
    poses = np.ascontiguousarray(np.stack([IDENT, IDENT]))
    cs = dliom.spa_constraints([(0, 0, IDENT, 1.0, 1.0)])
    opt = dliom.PoseGraphOptions(50, 0)
    assert dliom.lib().dl_pose_graph_solve_sparse(None, None, C.byref(opt), 1, 1, poses, None, C.cast(cs, C.c_void_p), 1,
                                                  None, None) == -2      # DL_ERR_ARG
    if have_gpu():
        pytest.skip("a GPU is present")
    with pytest.raises(dliom.DlError):
        dliom.Context(0)


# ---- the C++ mirror: optimization::OptimizationProblem3D (host/dliom_b200.hpp) and its example program
def build_pose_graph_example(out_dir):
    import subprocess
    host = os.path.join(ROOT, "d-liom_b200", "host")
    exe = os.path.join(str(out_dir), "example_pose_graph")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", os.path.join(host, "example_pose_graph.cc"), "-o", exe,
                           "-L" + os.path.join(ROOT, "d-liom_b200"), "-ldliom_b200", "-Wl,-rpath," + os.path.join(ROOT, "d-liom_b200")])
    return exe


def write_pose_graph(path, submaps, nodes, constraints, frozen_trajectories):
    """submaps / nodes: (trajectory_id, pose7) in id order per trajectory; constraints: ((traj, submap index), (traj, node index),
    zbar7, translation_weight, rotation_weight)."""
    import struct
    with open(path, "wb") as f:
        for items in (submaps, nodes):
            f.write(struct.pack("<i", len(items)))
            for t, p in items:
                f.write(struct.pack("<i7d", t, *p))
        f.write(struct.pack("<i", len(constraints)))
        for (st, si), (nt, ni), z, tw, rw in constraints:
            f.write(struct.pack("<4i9d", st, si, nt, ni, *z, tw, rw))
        f.write(struct.pack("<i", len(frozen_trajectories)))
        for t in frozen_trajectories:
            f.write(struct.pack("<i", t))


def two_trajectory_graph():
    """Trajectory 0 (a loaded map) and trajectory 1 driving along it; trajectory 1's nodes are also seen from trajectory 0's
    submaps. -> (submaps, nodes, constraints) in the layout of write_pose_graph."""
    s0, n0, c0 = trajectory_graph(3, 18, seed=3)
    s1, n1, c1 = trajectory_graph(3, 18, seed=5)
    shift = np.array([0.5, 0.2, 0.0, 1.0, 0, 0, 0])
    s1, n1 = [compose(shift, p) for p in s1], [compose(shift, p) for p in n1]
    submaps = [(0, p) for p in s0] + [(1, p) for p in s1]
    nodes = [(0, p) for p in n0] + [(1, p) for p in n1]
    cons = [((0, s), (0, n), z, tw, rw) for s, n, z, tw, rw in c0]
    cons += [((1, s), (1, n), z, tw, rw) for s, n, z, tw, rw in c1]   # relative poses: unchanged by the common shift
    for n in range(0, 18, 3):   # cross-trajectory constraints from the map's submaps
        s = min(n // 6, 2)
        cons.append(((0, s), (1, n), compose(inverse(submaps[s][1]), nodes[18 + n][1]), 100.0, 300.0))
    return submaps, nodes, cons


def test_cpp_pose_graph_shim_compiles_and_fails_loudly_without_a_gpu(tmp_path):
    import subprocess
    exe = build_pose_graph_example(tmp_path)
    if have_gpu():
        pytest.skip("a GPU is present: tests/test_gpu_posegraph_sparse.py runs the example")
    path = str(tmp_path / "graph.bin")
    write_pose_graph(path, *two_trajectory_graph(), [0])
    r = subprocess.run([exe, path], capture_output=True, text=True, timeout=120)
    assert r.returncode == 2 and "dliom error" in r.stderr and r.stdout == ""
