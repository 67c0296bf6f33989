"""Device block-sparse pose adjustment (csrc/dl_posegraph_sparse.cu, dl_pose_graph_solve_sparse; reference
OptimizationProblem3D::Solve, optimization_problem_3d.cc:259-589) against the dense oracle (oracle/orc_posegraph.h, pinned to the
reference's ReducesNoise test) and the block-sparse CPU oracle (tests/schur_oracle.py): same LM trajectory (iterations,
termination), poses to 1e-8 on small graphs and 1e-6 at trajectory scale; frozen poses; run-to-run bit identity, also with
blocking host waits; the all-reduce bookkeeping; argument errors."""
import os
import subprocess
import sys

import numpy as np
import pytest

import schur_oracle
from test_posegraph_oracle import aa_to_q, angle, compose, inverse
from test_posegraph_schur_oracle import (IDENT, build_pose_graph_example, exact_recovery_graph, reduces_noise_graph, same_poses,
                                        trajectory_graph, two_trajectory_graph, write_pose_graph)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ctx():
    import dliom
    c = dliom.Context(0)
    yield c
    c.close()


def same_trajectory(a, b):
    assert a["num_iterations"] == b["num_iterations"] and a["termination"] == b["termination"]
    assert a["num_successful_steps"] == b["num_successful_steps"]


def lifted_graph():
    """One submap, six nodes whose start poses are lifted off the constraints: with fix_z the z must stay where it starts."""
    rng = np.random.default_rng(4)
    truth = [np.array([*rng.uniform(-5, 5, 3), *aa_to_q(rng.uniform(-0.3, 0.3, 3))]) for _ in range(6)]
    lifted = [t + np.array([0.2, -0.1, 0.4, 0, 0, 0, 0]) for t in truth]
    return [IDENT], lifted, [(0, k, truth[k], 1.0, 1.0) for k in range(6)]


def weighted_two_submap_graph():
    """Two submaps see all 20 nodes, weighted like loop closures (pose_graph.lua: sqrt(1.1e4) translation, sqrt(1e5) rotation)."""
    rng = np.random.default_rng(8)
    submaps = [IDENT, np.array([3.0, -1.0, 0.1, *aa_to_q([0, 0, -0.4])])]
    truth = [np.array([*rng.uniform(-6, 6, 3), *aa_to_q(rng.uniform(-0.5, 0.5, 3))]) for _ in range(20)]
    cons = [(s, n, compose(compose(inverse(submaps[s]), truth[n]), np.array([*rng.normal(0, 0.02, 3), *aa_to_q(rng.normal(0, 0.01, 3))])),
             1.1e4 ** 0.5, 1e5 ** 0.5) for s in range(2) for n in range(20)]
    start = [compose(t, np.array([*rng.uniform(-0.3, 0.3, 3), *aa_to_q(rng.uniform(-0.1, 0.1, 3))])) for t in truth]
    return submaps, start, cons


def test_matches_oracle_on_small_graphs(ctx, orc):
    *reduces_noise, truth = reduces_noise_graph()
    graphs = {"reduces_noise": (*reduces_noise, False), "exact_recovery": (*exact_recovery_graph(), False),
              "lifted": (*lifted_graph(), True), "weighted": (*weighted_two_submap_graph(), False),
              "trajectory": (*trajectory_graph(4, 24), True), "loops": (*trajectory_graph(6, 60, loops_every=3), False)}
    for name, (submaps, nodes, cons, fix_z) in graphs.items():
        ws, wn, wsum = orc.pose_graph_solve(submaps, nodes, cons, fix_z=fix_z)
        gs, gn, gsum, info = ctx.pose_graph_solve_sparse(submaps, nodes, cons, fix_z=fix_z)
        same_trajectory(gsum, wsum)
        assert abs(gsum["initial_cost"] - wsum["initial_cost"]) <= 1e-12 * max(wsum["initial_cost"], 1.0)
        same_poses(gs, ws, 1e-8)
        same_poses(gn, wn, 1e-8)
        assert np.array_equal(gs[0][:3], np.asarray(submaps[0])[:3])
        assert info.num_local_parameters == 2 + (3 + (2 if fix_z else 3)) * (len(submaps) + len(nodes) - 1)
        assert info.num_reduced_parameters == 2 + (3 + (2 if fix_z else 3)) * (len(submaps) - 1)
        assert info.num_pairs == len({(c[0], c[1]) for c in cons}) and info.all_reduce_count == 0
        if fix_z:
            assert all(a[2] == b[2] for a, b in zip(gn, nodes))
        if name == "exact_recovery":
            assert gsum["termination"] == 0 and gsum["final_cost"] < 1e-12 * max(gsum["initial_cost"], 1.0)
        if name == "reduces_noise":
            def errors(ps):
                return (sum(np.linalg.norm(t[:3] - p[:3]) for t, p in zip(truth, ps)),
                        sum(angle(compose(inverse(t), p)) for t, p in zip(truth, ps)))
            (t_before, r_before), (t_after, r_after) = errors(nodes), errors(gn)
            assert 0.8 * t_before > t_after and 0.8 * r_before > r_after          # the reference's assertion
            assert abs(gsum["final_cost"] - wsum["final_cost"]) <= 1e-9 * wsum["final_cost"]


def test_frozen_masks_match_the_oracle(ctx, orc):
    submaps, nodes, cons = trajectory_graph(5, 40)
    extra = [(2, 12, compose(compose(inverse(submaps[2]), nodes[12]), np.array([0.1, 0, 0, 1.0, 0, 0, 0])), 2.0, 1.0)]
    for frozen_idx in ([2, 3, *(5 + np.arange(10, 20))], [0], [0, 1, 2, 3, 4]):
        frozen = np.zeros(45, bool)
        frozen[frozen_idx] = True
        ws, wn, wsum = schur_oracle.solve(orc, submaps, nodes, cons + extra, frozen=frozen)
        gs, gn, gsum, info = ctx.pose_graph_solve_sparse(submaps, nodes, cons + extra, frozen=frozen)
        same_trajectory(gsum, wsum)
        assert abs(gsum["initial_cost"] - wsum["initial_cost"]) <= 1e-12 * wsum["initial_cost"]
        assert abs(gsum["final_cost"] - wsum["final_cost"]) <= 1e-8 * wsum["final_cost"]
        same_poses(gs, ws, 1e-8)
        same_poses(gn, wn, 1e-8)
        out, start = np.concatenate([gs, gn]), np.concatenate([submaps, nodes])
        assert np.array_equal(out[frozen], start[frozen])
        assert info.num_reduced_parameters == wsum["num_reduced_parameters"] and info.num_pairs == wsum["num_pairs"]
    gs, gn, gsum, info = ctx.pose_graph_solve_sparse(submaps, nodes, cons + extra, frozen=np.ones(45, bool))
    ws, wn, wsum = schur_oracle.solve(orc, submaps, nodes, cons + extra, frozen=np.ones(45, bool))
    assert np.array_equal(gs, np.asarray(submaps)) and np.array_equal(gn, np.asarray(nodes))
    assert gsum["termination"] == 0 and gsum["num_iterations"] == 0
    assert abs(gsum["initial_cost"] - wsum["initial_cost"]) <= 1e-12 * wsum["initial_cost"] and info.num_local_parameters == 0


def test_trajectory_scale_against_the_schur_oracle(ctx, orc):
    """10 000 nodes, 50 submaps, ~30 000 constraints: two active submaps per node and one loop closure to an older submap."""
    submaps, nodes, cons = trajectory_graph(50, 10000, loops_every=1)
    assert 29000 < len(cons) < 31000
    gs, gn, gsum, info = ctx.pose_graph_solve_sparse(submaps, nodes, cons)
    ws, wn, wsum = schur_oracle.solve(orc, submaps, nodes, cons)
    assert info.num_reduced_parameters == 2 + 6 * 49
    same_trajectory(gsum, wsum)
    same_poses(gs, ws, 1e-6)
    same_poses(gn, wn, 1e-6)
    assert gsum["final_cost"] < 1e-2 * gsum["initial_cost"]


def test_bit_identical_runs_and_world_of_one(ctx):
    import dliom
    submaps, nodes, cons = trajectory_graph(8, 400, loops_every=2)
    a = ctx.pose_graph_solve_sparse(submaps, nodes, cons)
    b = ctx.pose_graph_solve_sparse(submaps, nodes, cons)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2] == b[2]
    comm = dliom.Comm(ctx, dliom.comm_unique_id(), 0, 1)
    c = ctx.pose_graph_solve_sparse(submaps, nodes, cons, comm=comm)
    comm.close()
    assert np.array_equal(a[0], c[0]) and np.array_equal(a[1], c[1]) and a[2] == c[2]
    info = c[3]
    assert info.all_reduce_count == c[2]["num_evaluations"] and info.all_reduce_ms > 0
    P, K = len(submaps) + len(nodes), info.num_pairs
    assert info.all_reduce_bytes == 8 * (2 + 42 * P + 36 * K)
    assert info.setup_exchange_bytes == 32 + 4 + 4 + 8 * K    # meta, two agreed reservations, the pair list
    blocking = dliom.Context(0)
    blocking.set_blocking_sync(True)    # every host wait of the solve sleeps on an event instead of spinning
    comm = dliom.Comm(blocking, dliom.comm_unique_id(), 0, 1)
    d = blocking.pose_graph_solve_sparse(submaps, nodes, cons)
    e = blocking.pose_graph_solve_sparse(submaps, nodes, cons, comm=comm)
    comm.close()
    blocking.close()
    for r in (d, e):
        assert np.array_equal(a[0], r[0]) and np.array_equal(a[1], r[1]) and a[2] == r[2]


def test_argument_errors_before_any_collective(ctx):
    import dliom
    with pytest.raises(dliom.DlError) as e:
        ctx.pose_graph_solve_sparse([IDENT], [IDENT], [(0, 3, IDENT, 1.0, 1.0)])                # node outside the graph
    assert e.value.status == -2 and "outside" in str(e.value)
    comm = dliom.Comm(ctx, dliom.comm_unique_id(), 0, 1)
    with pytest.raises(dliom.DlError) as e:
        ctx.pose_graph_solve_sparse([IDENT], [IDENT], [(0, 3, IDENT, 1.0, 1.0)], comm=comm)
    assert e.value.status == -2 and "outside" in str(e.value)
    with pytest.raises(dliom.DlError) as e:
        ctx.pose_graph_solve_sparse([IDENT] * 600, [IDENT], [], comm=comm)                     # 2 + 6 * 599 > 3072
    assert e.value.status == -2 and "3072" in str(e.value)
    assert ctx.pose_graph_solve_sparse([IDENT] * 600, [IDENT], [], comm=comm,                  # frozen submaps do not count
                                       frozen=[False] * 100 + [True] * 501)[3].num_reduced_parameters == 2 + 6 * 99
    comm.close()


_TWO_RANKS = r"""
import sys, numpy as np
sys.path[:0] = [{root!r} + "/d-liom_b200", {root!r} + "/tests"]
import dliom
from test_posegraph_schur_oracle import trajectory_graph
rank, uid = int(sys.argv[1]), bytes.fromhex(sys.argv[2])
ctx = dliom.Context(rank)
comm = dliom.Comm(ctx, uid, rank, 2)
submaps, nodes, cons = trajectory_graph(8, 400, loops_every=2)
mine = [c for i, c in enumerate(cons) if (c[0] + i) % 2 == rank]
s, n, summ, info = ctx.pose_graph_solve_sparse(submaps, nodes, mine, comm=comm)
np.save(sys.argv[3], np.concatenate([s, n]))
comm.close(); ctx.close()
"""


def test_two_ranks_give_bit_identical_replicas(ctx, tmp_path):
    count = subprocess.run([sys.executable, "-c", "import torch; print(torch.cuda.device_count())"], capture_output=True, text=True)
    if int(count.stdout.strip() or 0) < 2:    # in a fresh process: torch cannot load next to the library's NCCL
        pytest.skip("needs two GPUs")
    import dliom
    uid = dliom.comm_unique_id().hex()
    script = tmp_path / "rank.py"
    script.write_text(_TWO_RANKS.format(root=ROOT))
    outs = [tmp_path / f"r{r}.npy" for r in range(2)]
    procs = [subprocess.Popen([sys.executable, str(script), str(r), uid, str(outs[r])]) for r in range(2)]
    assert [p.wait(timeout=300) for p in procs] == [0, 0]
    a, b = np.load(outs[0]), np.load(outs[1])
    assert np.array_equal(a, b)
    submaps, nodes, cons = trajectory_graph(8, 400, loops_every=2)
    s, n, _, _ = ctx.pose_graph_solve_sparse(submaps, nodes, cons)
    same_poses(a, np.concatenate([s, n]), 1e-8)


def test_cpp_optimization_problem_with_a_frozen_trajectory_matches_python(ctx, orc, tmp_path):
    """host/dliom_b200.hpp: optimization::OptimizationProblem3D::Solve(constraints, frozen_trajectories = {0}) through the example
    program, against the Python call on the same graph laid out in id order: the same poses to the last bit (same C-ABI call)."""
    submaps, nodes, cons = two_trajectory_graph()
    exe = build_pose_graph_example(tmp_path)
    path = str(tmp_path / "graph.bin")
    write_pose_graph(path, submaps, nodes, cons, [0])
    out = subprocess.run([exe, path], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    lines = out.stdout.split("\n")
    got_s = np.array([[float(v) for v in l.split()[3:]] for l in lines if l.startswith("submap ")])
    got_n = np.array([[float(v) for v in l.split()[3:]] for l in lines if l.startswith("node ")])
    summary = next(l.split()[1:] for l in lines if l.startswith("summary "))
    S = len(submaps)
    index_s = {(t, i): k for k, (t, i) in enumerate([(t, sum(1 for u, _ in submaps[:k] if u == t)) for k, (t, _) in enumerate(submaps)])}
    index_n = {(t, i): k for k, (t, i) in enumerate([(t, sum(1 for u, _ in nodes[:k] if u == t)) for k, (t, _) in enumerate(nodes)])}
    flat = [(index_s[s], index_n[n], z, tw, rw) for s, n, z, tw, rw in cons]
    frozen = [t == 0 for t, _ in submaps] + [t == 0 for t, _ in nodes]
    ws, wn, wsum, _ = ctx.pose_graph_solve_sparse([p for _, p in submaps], [p for _, p in nodes], flat, frozen=frozen)
    assert np.array_equal(got_s, ws) and np.array_equal(got_n, wn)
    assert int(summary[0]) == wsum["num_iterations"] and int(summary[1]) == wsum["termination"] == 0
    assert np.array_equal(ws[:3], np.array([p for _, p in submaps[:3]]))       # trajectory 0 is frozen
    assert not np.array_equal(wn[18:], np.array([p for _, p in nodes[18:]]))
    os_, on, osum = schur_oracle.solve(orc, [p for _, p in submaps], [p for _, p in nodes], flat, frozen=frozen)
    assert osum["num_iterations"] == wsum["num_iterations"]
    same_poses(ws, os_, 1e-8)
    same_poses(wn, on, 1e-8)
    assert S == 6
