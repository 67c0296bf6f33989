"""Pure localization's bookkeeping (tests/pose_graph3d_trimming_oracle.py) on the CPU: equal to the mapping oracle on untrimmed
sequences; the reference's trimmer tests restated on add_node-built graphs; the edge cases of MarkSubmapAsTrimmed, the
append ban, FinishTrajectory and the initial trajectory pose; and the C-ABI surface of dl_pg3d_* / dl_ltb_release_submap that
needs no GPU."""
import ctypes as C

import numpy as np
import pytest

import pose_graph3d_oracle as pg
import pose_graph3d_trimming_oracle as tg
from test_pose_graph3d_oracle import drive, pose


def line(i):
    return pose(0.5 * i, 0.1 * np.sin(i), 0.01 * i, 0.01, -0.02, 0.05 * i)


def keep_poses(sp, npo, cons, frozen):
    return sp, npo


def test_untrimmed_sequences_equal_the_mapping_oracle():
    """Two trajectories, matches, periodic optimizations with a recording solve: every pair, guess, solve input, constraint and
    pose equals pose_graph3d_oracle.py's."""
    def search(pairs):
        return [(n[1] % 3 == 0, pg.compose(guess, pose(0.01, 0.0, 0.0)), 1.0, 2.0) for _, n, guess in pairs]

    def solve(sp, npo, cons, frozen):    # deterministic stand-in: a small move of every free pose
        move = np.array([0.001, -0.002, 0.0005, 1, 0, 0, 0])
        return ([pg.compose(p, move) if not f else p for p, f in zip(sp, frozen[:len(sp)])],
                [pg.compose(p, move) if not f else p for p, f in zip(npo, frozen[len(sp):])])

    graphs = [pg.PoseGraph3D(4, 2), tg.PoseGraph3D(4, 2)]
    for g in graphs:
        g.frozen.add(0)
        drive(g, 0, 12, 2, line, solve=solve)
        drive(g, 1, 10, 2, lambda i: line(i + 0.3), search=search, solve=solve,
              matches_for=lambda k: [(0, 1, 0.1, 0.0, 0.02), (0, 3, 0.0, 0.1, 0.0)] if k < 2 else [(0, 0, 0.0, 0.0, 0.0)])
    a, b = graphs
    b.run_final_optimization(solve)
    a.optimize(solve)
    assert [(s, n) for s, n, _ in a.searched] == [(s, n) for s, n, _ in b.searched] and a.searched
    assert all(np.array_equal(x[2], y[2]) for x, y in zip(a.searched, b.searched))
    assert len(a.solves) == len(b.solves) > 2
    for x, y in zip(a.solves, b.solves):
        assert x[0] == y[0] and x[1] == y[1] and x[5] == y[5]
        assert np.array_equal(x[2], y[2]) and np.array_equal(x[3], y[3])
        assert [(c[0], c[1]) for c in x[4]] == [(c[0], c[1]) for c in y[4]]
    assert [(c[0], c[1], c[5]) for c in a.constraints] == [(c[0], c[1], c[5]) for c in b.constraints]
    for t in (0, 1):
        assert np.array_equal(a.node_poses(t), b.node_poses(t))
        assert np.array_equal(a.submap_poses(t), b.submap_poses(t))
        assert b.ids(t) == list(range(len(a.nodes[t]))) and b.ids(t, False) == list(range(len(a.submaps[t])))


def test_pure_localization_trimmer_keeps_15_of_17():
    """pose_graph_trimmer_test.cc:29-39: keep 15 of 17 submaps -> submaps 0 and 1 are trimmed. Here 17 submaps of an
    add_node-built trajectory, the newest two active, so the retain rule also removes the nodes only they held."""
    g = tg.PoseGraph3D(0, 1)
    drive(g, 42, 34, 2, line)           # submaps 0..16, 0..15 finished
    assert list(g.submaps[42]) == list(range(17))
    g.add_pure_localization_trimmer(42, 15)
    g.run_final_optimization(keep_poses)
    assert g.last_trimmed == [(42, 0), (42, 1)]
    assert g.ids(42, False) == list(range(2, 17))
    assert g.ids(42)[0] == 4                 # nodes 0..3 were only in submaps 0 and 1; node 4 is held by submap 2


def test_pure_localization_trimmer_counts():
    """pose_graph_3d_test.cc:138-195 restated: 12 nodes, num_range_data 2 -> submaps 0..5 (5 unfinished), each node after the
    first two in two submaps. Keep 3: submaps 0, 1, 2 go; node k is held by submaps k//2 - 1 and k//2, so nodes 0..5 go
    (a node of submap 2 also in submap 1 goes with submap 1's trim); left: nodes 6..11 with INTRA constraints 6, 7 -> 3;
    8, 9 -> 3, 4; 10, 11 -> 4, 5: ten. A second final optimization changes nothing."""
    g = tg.PoseGraph3D(0, 1)
    drive(g, 2, 12, 2, line)
    assert len(g.constraints) == 22
    g.add_pure_localization_trimmer(2, 3)
    for _ in range(2):
        g.run_final_optimization(keep_poses)
        assert g.ids(2, False) == [3, 4, 5] and g.ids(2) == [6, 7, 8, 9, 10, 11]
        assert len(g.constraints) == 10 and len(g.node_poses(2)) == 6 and len(g.submap_poses(2)) == 3
    assert g.trimmers == [[2, 3]]          # not finished until the trajectory is


def test_even_submap_trimmer_counts():
    """pose_graph_3d_test.cc:217-272 restated (a host trimmer: the even submap ids): submaps 0, 2, 4 go; node k is held by
    submaps k//2 - 1 and k//2, so only nodes 0 and 1 (submap 0 alone) go; left: submaps 1, 3, 5, nodes 2..11, one INTRA each."""
    g = tg.PoseGraph3D(0, 1)
    drive(g, 2, 12, 2, line)
    for _ in range(2):
        g.run_final_optimization(keep_poses)
        for i in [i for i in g.ids(2, False) if i % 2 == 0]:
            g.trim_submap(2, i)
        assert g.ids(2, False) == [1, 3, 5] and g.ids(2) == list(range(2, 12)) and len(g.constraints) == 10


def test_trimming_the_anchor_moves_it_to_the_next_submap():
    g = tg.PoseGraph3D(0, 1)
    drive(g, 0, 8, 2, line)
    g.run_final_optimization(keep_poses)
    g.trim_submap(0, 0)
    seen = []
    g.run_final_optimization(lambda sp, npo, cons, frozen: (seen.append(sp[0].copy()), (sp, npo))[1])
    assert g.solves[-1][0][0] == (0, 1)      # the solve's first submap, the one it holds
    assert np.array_equal(seen[0], g.submaps[0][1]["global"])


def test_trimming_the_highest_index_forbids_appends():
    g = tg.PoseGraph3D(0, 1)
    drive(g, 0, 8, 2, line)                  # submaps 0..3, 0..2 finished
    g.run_final_optimization(keep_poses)
    g.finish_trajectory(0, keep_poses)      # every submap finished; no trimmer
    g2 = tg.PoseGraph3D(0, 1)
    drive(g2, 0, 8, 2, line)
    for s in g2.submaps[0].values():
        s["finished"] = True                 # as after FinishTrajectory, without the finished-trajectory rule
    g2.trim_submap(0, 3)
    assert g2.can_append[0] == [False, True]   # node 7 is still held by submap 2
    with pytest.raises(tg.Rejected):       # a node opening submap 4 would append a submap
        g2.add_node(0, line(8), [(3, False, line(6)), (4, False, line(8))])
    with pytest.raises(tg.Rejected):       # and a finished trajectory takes no node at all
        g.add_node(0, line(8), [(3, False, line(6))])
    # the highest node index trimmed: submap 2 and 3 hold nodes 4..7; trimming both removes 6, 7
    g2.trim_submap(0, 2)
    assert g2.ids(0)[-1] == 5 and g2.can_append[0] == [False, False]


def test_node_retained_through_its_second_submap():
    g = tg.PoseGraph3D(0, 1)
    drive(g, 0, 8, 2, line)                  # node 2, 3 in submaps 0 and 1
    g.run_final_optimization(keep_poses)
    g.trim_submap(0, 0)
    assert g.ids(0) == list(range(2, 8))
    assert [c[0] for c in g.constraints if c[1] == (0, 2)] == [(0, 1)]


def test_trimming_is_refused_with_constraints_pending_or_unfinished_or_unknown():
    g = tg.PoseGraph3D(0, 1)
    drive(g, 0, 8, 2, line)
    g.pending = [((0, 0), (0, 5), pg.IDENTITY, 1.0, 1.0, pg.INTER)]
    before = (list(g.submaps[0]), list(g.nodes[0]), len(g.constraints))
    for t, i in ((0, 0), (0, 3), (0, 9), (5, 0)):
        with pytest.raises(tg.Rejected):
            g.trim_submap(t, i)
        assert (list(g.submaps[0]), list(g.nodes[0]), len(g.constraints)) == before
    with pytest.raises(tg.Rejected):
        g.add_pure_localization_trimmer(0, 2)
    g.run_final_optimization(keep_poses)
    g.trim_submap(0, 0)
    with pytest.raises(tg.Rejected):          # already trimmed
        g.trim_submap(0, 0)
    with pytest.raises(tg.Rejected):          # a match naming a trimmed submap
        drive(g, 1, 4, 2, line, matches_for=lambda k: [(0, 0, 0.0, 0.0, 0.0)])


def test_finish_trajectory_trims_everything_and_finishes_the_trimmer():
    g = tg.PoseGraph3D(0, 1)
    drive(g, 0, 12, 2, line)
    g.add_pure_localization_trimmer(0, 3)
    g.finish_trajectory(0, keep_poses)
    assert g.ids(0, False) == [] and g.ids(0) == [] and g.constraints == [] and g.trimmers == []
    assert g.last_trimmed == [(0, i) for i in range(6)]
    with pytest.raises(tg.Rejected):
        g.finish_trajectory(0, keep_poses)


def test_interpolation_clamps_and_exact_node_time():
    times = [1.0, 2.0, 3.5]
    poses = [pose(0, 0, 0), pose(1.0, 2.0, 0.5, 0.1, 0.0, 0.4), pose(3.0, 1.0, 0.0, 0.0, 0.2, -0.3)]
    assert np.array_equal(tg.interpolate(times, poses, 0.5), poses[0])
    assert np.array_equal(tg.interpolate(times, poses, 9.0), poses[2])
    assert np.array_equal(tg.interpolate(times, poses, 1.0), poses[0])   # lower_bound at the first node: the clamp
    exact = tg.interpolate(times, poses, 2.0)                               # an inner node: Interpolate with factor 1
    assert np.abs(exact - poses[1]).max() < 1e-15
    mid = tg.interpolate(times, poses, 2.75)
    assert np.allclose(mid[:3], (np.array(poses[1][:3]) + poses[2][:3]) / 2, atol=1e-15)
    half = pg.qmul(poses[1][3:], np.array([1.0, 0, 0, 0]))
    angle = 2 * np.arccos(abs(np.dot(half, poses[2][3:])))                # slerp halves the angle
    assert abs(2 * np.arccos(abs(np.dot(mid[3:], poses[1][3:]))) - angle / 2) < 1e-12


def test_initial_trajectory_pose_places_the_first_node():
    g = tg.PoseGraph3D(0, 1)
    drive(g, 0, 6, 2, line)
    for k, n in g.nodes[0].items():
        n["time"] = float(k)
    rel = pose(1.0, 0.0, 0.0, yaw=np.deg2rad(5))
    g.set_initial_trajectory_pose(1, 0, rel, 2.5)
    g.add_node(1, pose(0, 0, 0), [(0, False, pose(0, 0, 0))], time=10.0)
    want = pg.compose(tg.interpolate([0.0, 1, 2, 3, 4, 5], [n["global"] for n in g.nodes[0].values()], 2.5), rel)
    assert np.abs(g.node_poses(1)[0] - want).max() < 1e-15
    g3 = tg.PoseGraph3D(0, 1)
    g3.set_initial_trajectory_pose(1, 7, rel, 0.0)
    with pytest.raises(tg.Rejected):
        g3.add_node(1, pose(0, 0, 0), [(0, False, pose(0, 0, 0))])


# ---- the C-ABI surface without a GPU
def test_structs_symbols_and_argument_checks():
    import dliom
    from test_pose_graph3d_oracle import fields_of
    assert [n for _, n, _ in fields_of("dl_pg3d_submap_id")] == [n for n, _ in dliom.Pg3dSubmapId._fields_]
    assert C.sizeof(dliom.Pg3dSubmapId) == 8
    L = dliom.lib()
    names = [e for e in dliom.EXPORTS if e.startswith("dl_pg3d_")] + ["dl_ltb_release_submap"]
    assert len(names) == 9
    for s in names:
        assert hasattr(L, s), s
    ERR_ARG = -2
    n = C.c_int32(0)
    assert L.dl_pg3d_trim_submap(None, 0, 0) == ERR_ARG
    assert L.dl_pg3d_add_pure_localization_trimmer(None, 0, 3) == ERR_ARG
    assert L.dl_pg3d_finish_trajectory(None, 0) == ERR_ARG
    assert L.dl_pg3d_is_trajectory_finished(None, 0, C.byref(n)) == ERR_ARG
    assert L.dl_pg3d_set_initial_trajectory_pose(None, 1, 0, None, 0.0) == ERR_ARG
    assert L.dl_pg3d_ids(None, 0, 0, 0, None, C.byref(n)) == ERR_ARG
    assert L.dl_pg3d_last_trimmed(None, 0, None, C.byref(n)) == ERR_ARG
    assert L.dl_pg3d_store_usage(None, None, None, None) == ERR_ARG
    assert L.dl_ltb_release_submap(None, 0) == ERR_ARG


def test_cpp_localization_example_is_built_and_fails_loudly_without_a_gpu(tmp_path):
    """build() builds host/example_localization.cc; without a device it exits with status 2 and a dliom error."""
    import os
    import subprocess
    import dliom
    exe = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "build", "example_localization")
    assert os.access(exe, os.X_OK)
    try:
        dliom.Context(0).close()
        pytest.skip("a GPU is present: tests/test_gpu_localization.py runs the example")
    except dliom.DlError:
        pass
    path = tmp_path / "drive.bin"
    path.write_bytes(b"")
    r = subprocess.run([exe, str(path)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 2 and "dliom error" in r.stderr and r.stdout == ""
