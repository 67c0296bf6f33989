"""PoseGraph3D's bookkeeping (tests/pose_graph3d_oracle.py) on the CPU, and the C-ABI surface of dl_pose_graph_3d_* that needs no
GPU: struct layouts against the header, the exported symbols and the entry points' argument checks."""
import ctypes as C
import os
import re

import numpy as np

import pose_graph3d_oracle as pg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def pose(x, y, z, roll=0.0, pitch=0.0, yaw=0.0):
    def axis(a, i):
        q = np.zeros(4)
        q[0], q[1 + i] = np.cos(a / 2), np.sin(a / 2)
        return q
    q = pg.qmul(pg.qmul(axis(yaw, 2), axis(pitch, 1)), axis(roll, 0))
    return np.concatenate([[x, y, z], q])


def drive(graph, t, n, per_submap, local_of, search=None, solve=None, matches_for=None):
    """ActiveSubmaps3D's hand-over for `n` nodes (num_range_data = per_submap): insertion submaps [k] then [k, k+1]; the front
    finishes at its 2 * per_submap-th insert. local_of(i) gives node i's local pose; submap k sits at its first node's pose."""
    inserts = {}
    first_pose = {}
    active = [0]
    first_pose[0] = local_of(0)
    log = []
    for i in range(n):
        ins = []
        for k in active:
            inserts[k] = inserts.get(k, 0) + 1
        for k in active:
            ins.append((k, inserts[k] == 2 * per_submap, first_pose[k]))
        matches = matches_for(ins[0][0]) if (matches_for and ins[0][1]) else ()
        log.append(([k for k, _, _ in ins], graph.add_node(t, local_of(i), ins, matches, search, solve)))
        if inserts[active[-1]] == per_submap:
            new = active[-1] + 1
            first_pose[new] = local_of(i + 1)
            active.append(new)
        if inserts[active[0]] == 2 * per_submap:
            active.pop(0)
    return log


def test_initialize_global_submap_poses_and_hand_over():
    g = pg.PoseGraph3D(0, 1)
    local = lambda i: pose(0.5 * i, 0.1 * np.sin(i), 0.01 * i, 0.01, -0.02, 0.05 * i)
    log = drive(g, 0, 12, 3, local)
    assert [ids for ids, _ in log] == [[0]] * 3 + [[0, 1]] * 3 + [[1, 2]] * 3 + [[2, 3]] * 3
    subs = g.submaps[0]
    assert len(subs) == 4 and [s["finished"] for s in subs] == [True, True, True, False]
    # one-submap branch: local_to_global (identity before any optimization) * local pose
    assert np.allclose(subs[0]["global"], subs[0]["local"], atol=1e-15)
    # two-submap branch: front's global * front local^-1 * back local
    for k in range(1, 4):
        want = pg.compose(pg.compose(subs[k - 1]["global"], pg.inverse(subs[k - 1]["local"])), subs[k]["local"])
        assert np.allclose(subs[k]["global"], want, atol=1e-15)
    assert subs[1]["node_ids"] == [3, 4, 5, 6, 7, 8]


def test_intra_constraints_and_node_global_pose():
    g = pg.PoseGraph3D(0, 1)
    local = lambda i: pose(1.0 * i, 0.2, 0.0, 0.03, 0.01, 0.1 * i)
    drive(g, 0, 5, 2, local)
    intra = [c for c in g.constraints if c[5] == pg.INTRA]
    assert [(c[0], c[1]) for c in intra] == [((0, 0), (0, 0)), ((0, 0), (0, 1)), ((0, 0), (0, 2)), ((0, 1), (0, 2)),
                                             ((0, 0), (0, 3)), ((0, 1), (0, 3)), ((0, 1), (0, 4)), ((0, 2), (0, 4))]
    for (t, s), (_, n), zbar, tw, rw, _ in intra:
        want = pg.compose(pg.inverse(g.submaps[t][s]["local"]), g.nodes[t][n]["local"])
        assert np.abs(zbar - want).max() < 1e-12 and (tw, rw) == (5e2, 1.6e3)
        # the node's problem pose seen from the submap's problem pose is the INTRA measurement
        rel = pg.compose(pg.inverse(g.submaps[t][s]["global"]), g.nodes[t][n]["problem_global"])
        assert np.abs(rel[:3] - want[:3]).max() < 1e-12


def test_guess_composition_removes_yaw_and_recovers_the_true_relative_pose():
    """Two submaps whose local poses carry roll and pitch, their local frames placed in one world by two planar transforms: with
    M2D the yaw-and-xy relation of the two yaw-free gravity-aligned frames, the guess is the node's true pose in the target."""
    w_from, w_to = pose(3.0, -2.0, 0.0, yaw=0.3), pose(-1.0, 4.0, 0.0, yaw=-0.7)
    s_from, s_to = pose(10.0, 1.0, 0.2, 0.04, -0.03, 0.9), pose(2.0, -3.0, 0.2, -0.02, 0.05, -1.2)   # same height: M2D has no z
    node = pose(11.0, 1.5, 0.25, 0.05, -0.01, 1.0)
    m = pg.match_from_truth(s_from, s_to, w_from, w_to)
    guess = pg.pose_guess(s_from, s_to, m, node)
    truth = pg.compose(pg.inverse(pg.compose(w_to, s_to)), pg.compose(w_from, node))
    assert np.abs(guess[:3] - truth[:3]).max() < 1e-12
    assert min(np.abs(guess[3:] - truth[3:]).max(), np.abs(guess[3:] + truth[3:]).max()) < 1e-12
    # the relation is planar only because the gravity alignments have no yaw left
    assert abs(pg.get_yaw(pg.yaw_free_alignment(s_from)[3:])) < 1e-12
    # without the yaw removal the same M2D misses
    t_g1_s1 = pg.inverse(np.concatenate([[0, 0, 0], s_to[3:]]))
    t_s2_g2 = np.concatenate([[0, 0, 0], s_from[3:]])
    naive = pg.compose(pg.compose(pg.compose(t_g1_s1, pg.embed_2d(*m)), t_s2_g2), pg.compose(pg.inverse(s_from), node))
    assert np.abs(naive[:3] - truth[:3]).max() > 0.1


def test_fan_out_sampling_and_computed_constraints_dedup():
    """The counter restarts per matched submap and runs over the finished submap's nodes in id order; a pair already FOUND for
    the target is skipped, a pair searched and not found is searched again."""
    g = pg.PoseGraph3D(0, 2)
    local = lambda i: pose(0.5 * i, 0.0, 0.0)
    drive(g, 0, 12, 2, local)                       # trajectory 0: submaps 0..4 (0..3 finished once driven further)
    calls = []

    def search(pairs):
        calls.append([(s, n) for s, n, _ in pairs])
        return [(n[1] % 4 == 0, pg.IDENTITY, 1.0, 2.0) for _, n, _ in pairs]   # nodes 0, 4, 8, ... are found

    matches = lambda k: [(0, 1, 0.0, 0.0, 0.0), (0, 0, 0.0, 0.0, 0.0)] if k == 0 else [(0, 0, 0.0, 0.0, 0.0)] if k == 1 else []
    drive(g, 1, 6, 2, local, search=search, matches_for=matches)
    # trajectory 1's submap 0 finishes at its 4th insert (nodes 0..3): j = 0, 2 of each target, targets in id order
    assert calls[0] == [((0, 0), (1, 0)), ((0, 0), (1, 2)), ((0, 1), (1, 0)), ((0, 1), (1, 2))]
    # submap 1 (nodes 2..5) finishes at node 5, matched to (0, 0): node 2 was searched there and pruned, so it is searched again
    assert calls[1] == [((0, 0), (1, 2)), ((0, 0), (1, 4))]
    assert len(calls) == 2 and g.computed == {(0, 0): {(1, 0), (1, 4)}, (0, 1): {(1, 0)}}
    # a second finished submap matched to the same targets: found pairs are not searched again, pruned ones are
    g2 = pg.PoseGraph3D(0, 1)
    drive(g2, 0, 12, 2, local)
    calls.clear()
    g2.computed[(0, 0)] = {(1, 1)}
    drive(g2, 1, 4, 2, local, search=search, matches_for=lambda k: [(0, 0, 0.0, 0.0, 0.0)] if k == 0 else [])
    assert calls == [[((0, 0), (1, 0)), ((0, 0), (1, 2)), ((0, 0), (1, 3))]]


def test_handle_work_queue_dedup_across_tags_and_trigger_is_strictly_greater():
    solves = []

    def solve(sp, npo, cons, frozen):
        solves.append(len(cons))
        return sp, npo

    g = pg.PoseGraph3D(3, 1)
    local = lambda i: pose(0.5 * i, 0.0, 0.0)
    log = drive(g, 0, 8, 2, local, solve=solve)
    assert [opt for _, opt in log] == [False, False, False, True, False, False, False, True]   # count > 3, then reset
    assert g.since_last == 0
    # a found INTER pair equal to an INTRA pair is dropped; a duplicate INTER pair enters once
    g.pending = [((0, 0), (0, 1), pg.IDENTITY, 1.0, 1.0, pg.INTER), ((0, 0), (0, 7), pg.IDENTITY, 1.0, 1.0, pg.INTER),
                 ((0, 0), (0, 7), pg.IDENTITY, 1.0, 1.0, pg.INTER)]
    n0 = len(g.constraints)
    g.optimize(solve)
    assert len(g.constraints) == n0 + 1 and g.constraints[-1][1] == (0, 7) and g.pending == []


# ---- the C-ABI surface without a GPU
def header():
    with open(os.path.join(ROOT, "include", "dliom_b200.h")) as f:
        return f.read()


SIZES = {"int32_t": 4, "int64_t": 8, "double": 8, "float": 4}


def fields_of(name):
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), header(), re.S).group(1)
    out = []
    for line in body.split(";"):
        line = re.sub(r"/\*.*?\*/", "", line, flags=re.S).strip()
        if not line:
            continue
        m = re.match(r"(?:const\s+)?([\w]+)\s*(\*?)\s*(.+)$", line)
        typ, ptr, names = m.groups()
        for nm in names.split(","):
            nm = nm.strip().lstrip("*")
            arr = re.match(r"(\w+)\[(\d+)\]", nm)
            out.append((typ + ptr, arr.group(1) if arr else nm, int(arr.group(2)) if arr else 1))
    return out


def test_structs_match_the_header():
    import dliom
    for cname, py in [("dl_pose_graph_3d_options", dliom.PoseGraph3DOptions), ("dl_pg3d_insertion_submap", dliom.Pg3dInsertionSubmap),
                      ("dl_pg3d_node", dliom.Pg3dNode), ("dl_pg3d_submap_match", dliom.Pg3dSubmapMatch),
                      ("dl_pg3d_add_node_info", dliom.Pg3dAddNodeInfo), ("dl_pg3d_constraint", dliom.Pg3dConstraint),
                      ("dl_pg3d_search", dliom.Pg3dSearch)]:
        hdr = fields_of(cname)
        assert [n for _, n, _ in hdr] == [n for n, _ in py._fields_], cname
        for (typ, name, count), (_, ctype) in zip(hdr, py._fields_):
            if typ in SIZES:
                assert C.sizeof(ctype) == SIZES[typ] * count, (cname, name)
            elif typ.endswith("*"):
                assert C.sizeof(ctype) == 8 * count, (cname, name)
    assert C.sizeof(dliom.Pg3dInsertionSubmap) == 4 + 4 + 8 + 8 + 56
    assert C.sizeof(dliom.Pg3dNode) == 4 + 4 + 8 + 56 + 4 * 8 + 2 * 80
    assert C.sizeof(dliom.Pg3dSubmapMatch) == 32
    assert C.sizeof(dliom.Pg3dConstraint) == 16 + 56 + 16 + 8
    assert C.sizeof(dliom.Pg3dAddNodeInfo) == 16 + 8 + 24 + C.sizeof(dliom.SolveSummary)
    assert C.sizeof(dliom.PoseGraph3DOptions) == 8 + 16 + C.sizeof(dliom.ConstraintOptions) + 8
    for name in ("DL_PG3D_INTRA_SUBMAP 0", "DL_PG3D_INTER_SUBMAP 1", "DL_PG3D_NODE_POSES 0", "DL_PG3D_SUBMAP_POSES 1",
                 "DL_PG3D_OPTIMIZATION_NODES 2", "DL_PG3D_OPTIMIZATION_SUBMAPS 3"):
        assert "#define " + name in header()


def test_symbols_are_exported_and_arguments_are_checked():
    import dliom
    L = dliom.lib()
    for s in [e for e in dliom.EXPORTS if e.startswith("dl_pose_graph_3d_")]:
        assert hasattr(L, s), s
    assert len([e for e in dliom.EXPORTS if e.startswith("dl_pose_graph_3d_")]) == 10
    opt = dliom.PoseGraph3DOptions.defaults()
    out = C.c_void_p()
    ERR_ARG = -2
    assert L.dl_pose_graph_3d_create(None, C.byref(opt), C.byref(out)) == ERR_ARG
    node = dliom.Pg3dNode()
    assert L.dl_pose_graph_3d_add_node(None, C.byref(node), 0, None, None) == ERR_ARG
    assert L.dl_pose_graph_3d_freeze_trajectory(None, 0) == ERR_ARG
    assert L.dl_pose_graph_3d_run_final_optimization(None, None) == ERR_ARG
    n = C.c_int32(0)
    assert L.dl_pose_graph_3d_poses(None, 0, 0, 0, None, C.byref(n)) == ERR_ARG
    assert L.dl_pose_graph_3d_local_to_global(None, 0, None) == ERR_ARG
    assert L.dl_pose_graph_3d_constraints(None, 0, None, C.byref(n)) == ERR_ARG
    assert L.dl_pose_graph_3d_last_searches(None, 0, None, C.byref(n)) == ERR_ARG
    assert L.dl_pose_graph_3d_store_bytes(None, None, None) == ERR_ARG
    L.dl_pose_graph_3d_destroy(None)   # no-op


def build_global_slam_example(out_dir):
    """host/example_global_slam.cc (mapping::LocalTrajectoryBuilder3D + mapping::PoseGraph3D) built with -Wall -Werror."""
    import subprocess
    host = os.path.join(ROOT, "d-liom_b200", "host")
    exe = os.path.join(str(out_dir), "example_global_slam")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", os.path.join(host, "example_global_slam.cc"), "-o", exe,
                           "-L" + os.path.join(ROOT, "d-liom_b200"), "-ldliom_b200", "-Wl,-rpath," + os.path.join(ROOT, "d-liom_b200")])
    return exe


def test_cpp_global_slam_example_compiles_and_fails_loudly_without_a_gpu(tmp_path):
    import subprocess
    import struct
    import dliom
    exe = build_global_slam_example(tmp_path)
    try:
        dliom.Context(0).close()
        import pytest
        pytest.skip("a GPU is present: tests/test_gpu_pose_graph3d.py runs the example")
    except dliom.DlError:
        pass
    path = str(tmp_path / "drive.bin")
    with open(path, "wb") as f:
        f.write(struct.pack("<iii", 0, 0, 0))
    r = subprocess.run([exe, path], capture_output=True, text=True, timeout=120)
    assert r.returncode == 2 and "dliom error" in r.stderr and r.stdout == ""
