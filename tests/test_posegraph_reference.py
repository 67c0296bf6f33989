"""The pose-graph solve's independent reference (tests/posegraph_reference.py) on the edges of tests/posegraph_cases.py, without a
GPU: the 50-digit run against an fp64 run of the same reference, against the block-sparse CPU oracle (tests/schur_oracle.py) and
the dense C++ oracle (oracle/orc_posegraph.h), the properties any correct solve has, the margins that make exact iteration counts
a fair requirement, and the rule that poses no constraint refers to stay out of the program. The device is compared to the same
reference in tests/test_gpu_posegraph_reference.py."""
import math

import numpy as np
import pytest

import imu_reference as ir
import posegraph_cases as pc
import posegraph_reference as pr
import schur_oracle

EXACT = ir.Exact()
CASES = pc.cases()
SUMMARY_COUNTS = ("termination", "num_iterations", "num_successful_steps", "num_unsuccessful_steps", "num_evaluations")


@pytest.fixture(scope="module")
def exact():
    return {name: pr.solve(p, EXACT) for name, (_, p) in CASES.items()}


def pose_error(a, b):
    """Largest translation difference and rotation angle between two pose lists (q and -q the same rotation). The angle is
    2 atan2(|vec(q_a^-1 q_b)|, |w|), which resolves small angles (an arccos of the dot product stops at 3e-8)."""
    a, b = np.asarray(a, float).reshape(-1, 7), np.asarray(b, float).reshape(-1, 7)
    if not len(a):
        return 0.0
    dt = np.abs(a[:, :3] - b[:, :3]).max()
    qa, qb = a[:, 3:] / np.linalg.norm(a[:, 3:], axis=1)[:, None], b[:, 3:] / np.linalg.norm(b[:, 3:], axis=1)[:, None]
    rel = np.array([pr._qmul(tuple(u * [1, -1, -1, -1]), tuple(v)) for u, v in zip(qa, qb)])
    return max(dt, float(np.max(2 * np.arctan2(np.linalg.norm(rel[:, 1:], axis=1), np.abs(rel[:, 0])))))


def cost_floor(p):
    """The fp64 rounding floor of a cost: each residual entry carries up to 64 eps w (1 + |t_i| + |t_j| + |z_t|) of rounding
    (tests/test_gpu_posegraph_reference.py derives the bound), so costs below 1/2 6m (that)^2 are rounding."""
    S, x, eps = p["S"], p["x"], np.finfo(np.float64).eps
    e = [64 * eps * max(tw, rw) * (1 + np.abs(x[s, :3]).max() + np.abs(x[S + n, :3]).max() + np.abs(z[:3]).max())
         for s, n, z, tw, rw in p["constraints"]]
    return 0.5 * 6 * sum(v * v for v in e)


def cost_tolerance(rel, summary, p):
    """rel of the cost, plus the rounding floor, plus 1e-12 of the initial cost: where the residuals go towards zero (consistent
    constraints) the final cost is the square of what the last steps left, so its relative difference is not bounded, while
    the path's sums carry rounding of the size of the initial cost."""
    return lambda k: rel * summary[k] + cost_floor(p) + 1e-12 * summary["initial_cost"]


def _poses(o):
    return np.concatenate([o["submaps"], o["nodes"]])


def test_every_decision_keeps_half_a_decade(exact):
    """Exact iteration counts and terminations can only be required where no decision is near its threshold. The table lists
    every case with its smallest margin (in decades) and the decision it belongs to."""
    rows, bad = [], []
    for name in sorted(CASES):
        d = exact[name]["decisions"]
        worst = min(d, key=lambda v: pr.margin(*v)) if d else ("none", 0.0, 0.0)
        m = pr.margin(*worst) if d else math.inf
        rows.append(f"{name:28s} {m:6.2f}  {worst[0]} {worst[1]:.3e} vs {worst[2]:.3e}")
        if m < 0.5 and name not in pc.ALLOWANCES:
            bad.append(name)
    print("\n" + "\n".join(rows))
    assert not bad, bad


def test_each_lm_path_is_taken(exact):
    trace = {name: [t[0] for t in exact[name]["trace"]] for name in CASES}
    e = exact["exact_recovery"]
    assert e["decisions"][-1][0] == "gradient" and e["decisions"][-1][1] <= pr.GRADIENT_TOL
    assert trace["parameter_tolerance"][-1] == "parameter" and trace["function_tolerance"][-1] == "function"
    rejected = trace["max_iter_50"]
    assert rejected[0] == "rejected" and exact["max_iter_50"]["summary"]["num_unsuccessful_steps"] > 0
    for k in (1, 2, 50):
        s = exact[f"max_iter_{k}"]["summary"]
        assert s["termination"] == pr.NO_CONVERGENCE and s["num_iterations"] == k + 1
    assert all("invalid" not in t for t in trace.values())
    s = exact["all_frozen"]["summary"]
    assert s["termination"] == pr.CONVERGENCE and s["num_iterations"] == 0 and s["initial_cost"] == s["final_cost"] > 0


@pytest.mark.parametrize("name", sorted(CASES))
def test_exact_matches_fp64(exact, name):
    """fp64 with h = 6e-6 differences: Jacobians to ~1e-10 relative, so the same decisions (every margin is >= half a decade),
    costs to 1e-8 (see cost_tolerance) and poses to 1e-6 (the differences' Jacobian error, carried through the damped
    system's conditioning to where the function tolerance stops an unconverged point)."""
    e, f = exact[name], pr.solve(CASES[name][1], ir.FP64)
    assert {k: f["summary"][k] for k in SUMMARY_COUNTS} == {k: e["summary"][k] for k in SUMMARY_COUNTS}
    for k in ("initial_cost", "final_cost"):
        assert abs(f["summary"][k] - e["summary"][k]) <= cost_tolerance(1e-8, e["summary"], CASES[name][1])(k)
    assert pose_error(_poses(f), _poses(e)) <= 1e-6


@pytest.mark.parametrize("name", sorted(CASES))
def test_reference_matches_the_oracles(orc, exact, name):
    """The block-sparse oracle (JetN derivatives, Schur step) on every case; the dense oracle (no frozen poses) where nothing is
    frozen. Same decisions, costs to 1e-9 (see cost_tolerance), poses to 1e-8."""
    e, p = exact[name], CASES[name][1]
    S, x = p["S"], p["x"]
    runs = [schur_oracle.solve(orc, x[:S], x[S:], p["constraints"], fix_z=p["fix_z"], max_iter=p["max_iter"], frozen=p["frozen"])]
    if not p["frozen"].any():
        runs.append(orc.pose_graph_solve(x[:S], x[S:], p["constraints"], fix_z=p["fix_z"], max_iter=p["max_iter"]))
    for ss, sn, s in runs:
        for k in ("termination", "num_iterations", "num_successful_steps"):
            assert s[k] == e["summary"][k], (k, s[k], e["summary"][k])
        for k in ("initial_cost", "final_cost"):
            assert abs(s[k] - e["summary"][k]) <= cost_tolerance(1e-9, e["summary"], p)(k)
        assert pose_error(np.concatenate([ss, sn]), _poses(e)) <= 1e-8


def test_unconstrained_poses_come_back_unchanged(exact):
    for name, poses in (("unconstrained_far_node", [len(CASES["unconstrained_far_node"][1]["x"]) - 1]),
                        ("unconstrained_submap", [2]), ("unconstrained_first_submap", [0])):
        p = CASES[name][1]
        assert np.array_equal(_poses(exact[name])[poses], p["x"][poses])
    assert exact["unconstrained_far_node"]["num_local_parameters"] == exact["base"]["num_local_parameters"]


def test_keeping_unused_blocks_would_change_the_solve(exact):
    """With the node at 1e6 m kept in x, ||x|| ~ 1e6 makes the parameter threshold ~1e-2, and the solve stops early."""
    p = CASES["unconstrained_far_node"][1]
    real, kept = exact["unconstrained_far_node"], pr.solve(p, EXACT, keep_unused=True)
    a, b = real["summary"], kept["summary"]
    print(f"\nunused blocks removed: {a['num_iterations']} iterations, {real['trace'][-1][0]}; "
          f"kept: {b['num_iterations']} iterations, {kept['trace'][-1][0]}")
    assert (a["termination"], a["num_iterations"]) != (b["termination"], b["num_iterations"])
    assert kept["trace"][-1][0] == "parameter" and real["trace"][-1][0] == "function"


def test_zero_step_at_the_optimum(exact):
    """At the end of the exact-recovery solve the residuals are rounding of the measurements: the next LM step is below 1e-9."""
    e = exact["exact_recovery"]
    prog = e["program"]
    r, J = pr.evaluate(prog, e["x"], EXACT)
    scale = e["final"]["scale"]
    diag = pr._arr([min(max(v, pr.MIN_LM_DIAGONAL), pr.MAX_LM_DIAGONAL) for v in (J * scale[None, :] * J * scale[None, :]).sum(0)], EXACT)
    (st, _), _ = pr.step(prog, J, r, scale, diag, 1e4, EXACT)
    assert float(EXACT.sqrt(sum(v * v for v in st))) < 1e-9


@pytest.mark.parametrize("name", ["neg_q_submap", "neg_q_node", "neg_q_zbar"])
def test_quaternion_sign_does_not_matter(exact, name):
    a, b = exact[name], exact["base"]
    assert {k: a["summary"][k] for k in SUMMARY_COUNTS} == {k: b["summary"][k] for k in SUMMARY_COUNTS}
    assert abs(a["summary"]["final_cost"] - b["summary"]["final_cost"]) <= 1e-14 * b["summary"]["final_cost"]
    assert pose_error(_poses(a), _poses(b)) <= 1e-14


def _first_step(p, A, shift=(0, 0, 0)):
    """The first LM step at p's start, with every pose moved by `shift` in arithmetic A (not in the floats of p)."""
    prog = pr.Program(p)
    x = pr.to_A(p["x"], A)
    for q in range(len(x)):
        for k in range(3):
            x[q, k] = x[q, k] + A.num(shift[k])
    r, J = pr.evaluate(prog, x, A)
    scale = pr._arr([1 / (1 + A.sqrt(sum((J[i, a] * J[i, a] for i in range(J.shape[0])), A.num(0)))) for a in range(prog.n)], A)
    Js = J * scale[None, :]
    diag = pr._arr([min(max(Js[:, a].dot(Js[:, a]), pr.MIN_LM_DIAGONAL), pr.MAX_LM_DIAGONAL) for a in range(prog.n)], A)
    (st, mcc), _ = pr.step(prog, J, r, scale, diag, pr.INITIAL_RADIUS, A)
    return prog, J, r, scale, diag, st, mcc


@pytest.mark.parametrize("name", ["base", "weight_ratio_1e5", "unconstrained_first_submap"])
def test_translating_the_graph_leaves_the_step_unchanged(name):
    p = CASES[name][1]
    a, b = _first_step(p, EXACT)[5], _first_step(p, EXACT, shift=(12.5, -7.25, 3.0))[5]
    assert max(abs(float(u - v)) for u, v in zip(a, b)) <= 1e-25


@pytest.mark.parametrize("name", ["base", "frozen_trajectory", "fix_z", "unconstrained_submap", "repeated_constraints",
                                  "trajectory_4x12"])
def test_schur_step_equals_the_dense_step(name):
    """The reference's fp64 Jacobian, assembled into the per-pose and per-pair blocks the Schur elimination takes: the same step
    and model cost change as the dense normal equations, to rounding."""
    p = CASES[name][1]
    prog, J, r, scale, diag, st, mcc = _first_step(p, ir.FP64)
    S = p["S"]
    sg = schur_oracle.SchurPoseGraph(None, S, p["x"], p["constraints"], p["fix_z"], p["frozen"])
    assert list(sg.dim) == list(prog.rdim + prog.tdim)
    P = len(p["x"])
    g6, H6, Hk = np.zeros((P, 6)), np.zeros((P, 6, 6)), np.zeros((len(sg.pairs), 6, 6))
    sc6, dg6 = np.zeros((P, 6)), np.zeros((P, 6))
    for q in range(P):
        o, d = prog.off[q], prog.off[q + 1] - prog.off[q]
        sc6[q, :d], dg6[q, :d] = scale[o:o + d], diag[o:o + d]
    for i, (s, n, *_) in enumerate(prog.cons):
        rows = J[6 * i:6 * i + 6]
        blk = {}
        for q in (s, S + n):
            o, d = prog.off[q], prog.off[q + 1] - prog.off[q]
            blk[q] = np.zeros((6, 6))
            blk[q][:, :d] = rows[:, o:o + d]
            g6[q] += blk[q].T @ r[6 * i:6 * i + 6]
            H6[q] += blk[q].T @ blk[q]
        Hk[sg.pair_of[(s, n)]] += blk[s].T @ blk[S + n]
    out = sg.step(g6, H6, Hk, sc6, dg6, pr.INITIAL_RADIUS)
    assert out is not None
    dense = np.zeros((P, 6))
    for q in range(P):
        o, d = prog.off[q], prog.off[q + 1] - prog.off[q]
        dense[q, :d] = st[o:o + d]
    assert np.abs(out[0] - dense).max() <= 1e-10 * np.abs(dense).max()
    assert abs(out[1] - mcc) <= 1e-10 * abs(mcc)
