"""Edge cases of the block-sparse pose-graph solve (dl_pose_graph_solve_sparse), one small graph per edge (at most 4 submaps and
16 nodes, so that a 50-digit solve takes seconds). Shared by the CPU reference tests and the device tests. A case is a
posegraph_reference.problem.

Every decision quantity of every case's 50-digit trace keeps at least half a decade from its threshold (tested). ALLOWANCES
names the cases that cannot, with the reason and the one thing they are allowed; nothing else is relaxed for them."""
import numpy as np

import posegraph_reference as pr
from test_posegraph_oracle import aa_to_q, compose, inverse

IDENT = np.array([0, 0, 0, 1.0, 0, 0, 0])

# name -> (reason, allowance). Empty: every case keeps its margins.
ALLOWANCES = {}


def _pose(t, aa):
    return np.array([*t, *aa_to_q(aa)])


def graph(num_submaps=2, num_nodes=5, seed=0, views=2, noise=(0.02, 0.005), start=(0.3, 0.05), tw=1.0, rw=1.0, offset=(0, 0, 0),
          first_tilt=(0.0, 0.0)):
    """Submaps 3 m apart along x, nodes between them; node k is seen by submap k % S and, with views = 2, the next one. Constraints
    carry noise (translation sigma, rotation sigma); start poses are the truth moved by up to `start`. offset moves the whole
    graph; first_tilt tilts the first submap's start (roll, pitch) so that ConstantYawQuaternionPlus has work."""
    rng = np.random.default_rng(seed)
    off = np.asarray(offset, float)
    truth_s = [_pose(off + [3.0 * s, 0.4 * np.sin(s), 0.1 * s], [0, 0, 0.1 * s]) for s in range(num_submaps)]
    truth_s[0] = np.array([*off, 1.0, 0, 0, 0])
    truth_n = [_pose(off + [3.0 * num_submaps * (k + 0.5) / num_nodes, 0.5 * np.cos(k), 0.05 * k], rng.uniform(-0.3, 0.3, 3))
               for k in range(num_nodes)]
    cons = []
    for k in range(num_nodes):
        for v in range(views):
            s = (k + v) % num_submaps
            z = compose(compose(inverse(truth_s[s]), truth_n[k]), _pose(rng.normal(0, noise[0], 3), rng.normal(0, noise[1], 3)))
            cons.append((s, k, z, tw, rw))
    sub = [truth_s[0] if first_tilt == (0.0, 0.0) else compose(truth_s[0], _pose([0, 0, 0], [*first_tilt, 0]))]
    sub += [compose(t, _pose(rng.uniform(-start[0], start[0], 3), rng.uniform(-start[1], start[1], 3))) for t in truth_s[1:]]
    nod = [compose(t, _pose(rng.uniform(-start[0], start[0], 3), rng.uniform(-start[1], start[1], 3))) for t in truth_n]
    return sub, nod, cons


def _rot_error_case(angle, seed):
    """A noisy base graph plus one node at the first submap's (identity) rotation whose constraint has a rotation error of
    exactly `angle` about a tilted axis at the start (q_j^-1 q_i zbar = zbar)."""
    sub, nod, cons = graph(seed=seed)
    axis = np.array([0.3, -0.5, 0.8])
    axis /= np.linalg.norm(axis)
    nod = nod + [np.array([1.2, -0.4, 0.1, 1.0, 0, 0, 0])]
    return sub, nod, cons + [(0, len(nod) - 1, np.array([1.0, -0.3, 0.05, *aa_to_q(angle * axis)]), 1.0, 1.0)]


def _negated(g, which):
    sub, nod, cons = [np.array(p) for p in g[0]], [np.array(p) for p in g[1]], list(g[2])
    if which == "submap":
        sub[1][3:] *= -1
    elif which == "node":
        nod[2][3:] *= -1
    else:
        s, n, z, tw, rw = cons[3]
        cons[3] = (s, n, np.array([*z[:3], *(-z[3:])]), tw, rw)
    return sub, nod, cons


def _lifted(g):
    """Every start z but the first submap's moved off the constraints."""
    return ([g[0][0]] + [p + np.array([0, 0, 0.4, 0, 0, 0, 0]) for p in g[0][1:]],
            [p + np.array([0, 0, -0.3, 0, 0, 0, 0]) for p in g[1]], g[2])


def cases():
    """name -> (what the case is the edge of, posegraph_reference.problem). The seeds are the first from 100 on whose fp64 trace
    keeps every decision 0.6 decades from its threshold and takes the path the case is named for."""
    out = {}

    def add(name, why, g, **kw):
        out[name] = (why, pr.problem(*g, **kw))

    base = graph(seed=105)
    add("base", "two submaps, five nodes seen twice, noisy constraints: terminates by the function tolerance", base)
    # rotation residual
    add("rot_zero", "rotation error exactly 0 at the start: the angle-axis derivative at |v| = 0", _rot_error_case(0.0, 105))
    add("rot_below_cutoff", "rotation error 0.9e-7: the linearised branch of the angle-axis map", _rot_error_case(0.9e-7, 105))
    add("rot_above_cutoff", "rotation error 1.1e-7: the exact branch just above the cutoff", _rot_error_case(1.1e-7, 105))
    add("rot_pi_below", "rotation error pi - 1e-3: w > 0 just before the flip", _rot_error_case(np.pi - 1e-3, 105))
    add("rot_pi_above", "rotation error pi + 1e-3: w < 0, the flip to the shorter rotation", _rot_error_case(np.pi + 1e-3, 105))
    for which in ("submap", "node", "zbar"):
        add(f"neg_q_{which}", f"base with one {which} quaternion negated: the same rotation", _negated(base, which))
    # parameterisations
    add("first_submap_tilted", "the first submap starts tilted: ConstantYawQuaternionPlus moves roll and pitch only, its translation "
        "is constant", graph(seed=102, first_tilt=(0.04, -0.03)))
    add("fix_z", "fix_z with every start z off the constraints: SubsetParameterization keeps each z bit-unchanged; two rejected "
        "steps", _lifted(graph(seed=137)), fix_z=True)
    add("frozen_first_submap", "a frozen first submap: its rotation loses its two parameters too",
        graph(num_submaps=3, num_nodes=6, seed=100), frozen=[True] + [False] * 8)
    # frozen poses
    add("frozen_trajectory", "submap 1 and nodes 1, 2 frozen (a frozen trajectory's poses)", graph(num_submaps=3, num_nodes=6, seed=100),
        frozen=[False, True, False] + [False, True, True, False, False, False])
    g = graph(num_submaps=3, num_nodes=6, seed=101)
    z = compose(compose(inverse(g[0][1]), g[1][1]), _pose([0.1, 0, 0], [0, 0, 0.02]))
    add("frozen_pair_fixed_cost", "a constraint between two frozen poses: it only adds a fixed cost", (g[0], g[1], g[2] + [(1, 1, z, 2.0, 1.0)]),
        frozen=[False, True, False] + [False, True, False, False, False, False])
    add("all_frozen", "everything frozen: no parameters, CONVERGENCE at once with the fixed cost", graph(seed=6), frozen=[True] * 7)
    # unconstrained poses
    g = graph(seed=105)
    add("unconstrained_far_node", "a node no constraint refers to, at 1e6 m: it must not enter ||x|| and the parameter tolerance",
        (g[0], g[1] + [_pose([1e6, -2e5, 3e3], [0.1, 0.2, 0.3])], g[2]))
    add("unconstrained_submap", "a submap no constraint refers to", (g[0] + [_pose([40.0, -3.0, 1.0], [0.0, 0.1, 0.5])], g[1], g[2]))
    g = graph(num_submaps=3, num_nodes=6, seed=104)
    add("unconstrained_first_submap", "the first submap has no constraint: neither of its blocks is in the program",
        (g[0], g[1], [c for c in g[2] if c[0] != 0]))
    # weights and structure
    add("translation_weight_zero", "translation_weight = 0: H is singular, only the LM diagonal keeps it positive definite",
        graph(seed=100, tw=0.0))
    add("rotation_weight_zero", "rotation_weight = 0: H is singular, only the LM diagonal keeps it positive definite",
        graph(seed=104, rw=0.0))
    add("weight_ratio_1e5", "translation / rotation weight 1e5 (pose_graph.lua's loop-closure weights are 1.1e4 / 1e5)",
        graph(seed=104, tw=100.0, rw=1e-3))
    g = graph(num_submaps=2, num_nodes=4, seed=103)
    add("repeated_constraints", "the same (submap, node) pair constrained three times with different measurements",
        (g[0], g[1], g[2] + [(0, 1, compose(g[2][2][2], _pose([0.03, 0, 0], [0, 0.01, 0])), 1.0, 2.0),
                             (0, 1, compose(g[2][2][2], _pose([0, -0.02, 0], [0.01, 0, 0])), 0.5, 1.0)]))
    add("single_view", "every node seen by a single submap", graph(num_submaps=2, num_nodes=6, seed=104, views=1))
    # LM paths
    add("exact_recovery", "consistent constraints: the residual goes to rounding and the gradient tolerance ends the solve",
        graph(num_submaps=2, num_nodes=5, seed=100, noise=(0.0, 0.0), tw=0.1, rw=0.1))
    add("parameter_tolerance", "the graph 1e4 m from the origin: ||x|| makes the parameter threshold larger than the last step",
        graph(num_submaps=2, num_nodes=5, seed=100, offset=(1e4, -4e3, 50.0)))
    add("function_tolerance", "noisy constraints: the function tolerance ends the solve",
        graph(num_submaps=3, num_nodes=8, seed=100, noise=(0.05, 0.01)))
    add("max_iter_1", "NO_CONVERGENCE after max_num_iterations = 1", graph(seed=100), max_iter=1)
    add("max_iter_2", "NO_CONVERGENCE after max_num_iterations = 2", graph(seed=100), max_iter=2)
    add("max_iter_50", "NO_CONVERGENCE after max_num_iterations = 50; fix_z with every start z off the constraints: the first four "
        "steps are rejected, each followed by a radius cut", _lifted(graph(seed=101)), fix_z=True, max_iter=50)
    add("trajectory_4x12", "4 submaps, 12 nodes, loop-closure weights", graph(num_submaps=4, num_nodes=12, seed=102, tw=1.1e4 ** 0.5,
                                                                             rw=1e5 ** 0.5))
    return out
