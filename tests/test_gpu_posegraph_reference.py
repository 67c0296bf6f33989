"""The device pose-graph solve (dl_pose_graph_solve_sparse, dl_pose_graph_evaluate) against the independent 50-digit reference
(tests/posegraph_reference.py) on the edges of tests/posegraph_cases.py.

Tolerances, fixed before the first device run:
- factors: a residual is w (z_t - R_i^T (t_j - t_i)) or w AngleAxis(q_j^-1 q_i z_q); in fp64 each is a short chain of products
  and sums of unit quaternion entries and translations, so its error is a few ulp of w (1 + |t_i| + |t_j| + |z_t|). The same holds
  for the forward-mode derivatives: near the 1e-7 cutoff d(angle / sin(angle / 2)) cancels to about 2 eps / angle, but it is
  multiplied by the vector part (about angle / 2), so the product stays at a few ulp. Bound: 64 eps w (1 + |t_i| + |t_j| + |z_t|)
  per entry, w the larger weight.
- solves: every decision of every case keeps half a decade from its threshold in the 50-digit trace (tests/test_posegraph_reference.py),
  far more than fp64 rounding moves a decision, so termination, num_iterations, num_evaluations and the step counts must match
  exactly. Costs to 1e-9 relative (the reference's own fp64 run agrees to 1e-8 with h = 6e-6 differences; the device's
  derivatives are exact up to rounding), plus the rounding floor of a cost (1/2 6m of the residual bound above, squared), which
  only matters where the residuals go to rounding (exact recovery). Poses to 1e-7 (translation, rotation angle) and in the metric of the reference's H at
  its final point: 1/2 d^T H d <= 1e-9 final_cost + the rounding floor + 1e-24 tr(H), d the local difference (the cost excess a pose difference
  causes must stay below what the cost comparison allows, plus a floor of rounding in the residuals themselves).
- frozen poses, unconstrained poses, every z under fix_z and the first submap's translation: bit-unchanged."""
import os
import subprocess
import sys

import numpy as np
import pytest

import imu_reference as ir
import posegraph_cases as pc
import posegraph_reference as pr
from test_posegraph_reference import SUMMARY_COUNTS, cost_floor, pose_error
from test_posegraph_schur_oracle import trajectory_graph

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXACT = ir.Exact()
CASES = pc.cases()
EPS = np.finfo(np.float64).eps


@pytest.fixture(scope="module")
def ctx():
    import dliom
    c = dliom.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def exact():
    return {name: pr.solve(p, EXACT) for name, (_, p) in CASES.items()}


def _run(ctx, p, **kw):
    S, x = p["S"], p["x"]
    return ctx.pose_graph_solve_sparse(x[:S], x[S:], p["constraints"], fix_z=p["fix_z"], max_iter=p["max_iter"],
                                       frozen=p["frozen"] if p["frozen"].any() else None, **kw)


def _local_difference(prog, a, b):
    """a (-) b in the program's local parameters, to first order: rotation slots the vector part of the relative rotation in the
    chart's convention (left product, right product for the first submap), translation slots the difference."""
    d = np.zeros(prog.n)
    for q in range(prog.P):
        o, r, t = prog.off[q], prog.rdim[q], prog.tdim[q]
        if not r + t:
            continue
        qa, qb = np.asarray(a[q, 3:], float), np.asarray(b[q, 3:], float)
        rel = np.array(pr._qmul(tuple(qb * [1, -1, -1, -1]), tuple(qa))) if r == 2 else \
            np.array(pr._qmul(tuple(qa), tuple(qb * [1, -1, -1, -1])))
        rel = rel if rel[0] >= 0 else -rel
        d[o:o + r] = rel[1:1 + r]
        d[o + r:o + r + t] = a[q, :t] - b[q, :t]
    return d


@pytest.mark.parametrize("name", sorted(CASES))
def test_factors_match_the_reference(ctx, name):
    """dl_pose_graph_evaluate at the case's start point against the 50-digit residuals and central-difference Jacobians."""
    p = CASES[name][1]
    S, x = p["S"], p["x"]
    if not p["constraints"]:
        return
    r, J = ctx.pose_graph_evaluate(x[:S], x[S:], p["constraints"], fix_z=p["fix_z"], frozen=p["frozen"])
    prog = pr.Program(p)
    rr, JJ = pr.evaluate(prog, pr.to_A(x, EXACT), EXACT, cons=p["constraints"])
    rr, JJ = pr._f(rr), pr._f(JJ)
    for i, (s, n, z, tw, rw) in enumerate(p["constraints"]):
        bound = 64 * EPS * max(tw, rw, 1e-300) * (1 + np.abs(x[s, :3]).max() + np.abs(x[S + n, :3]).max() + np.abs(z[:3]).max())
        assert np.abs(r[i] - rr[6 * i:6 * i + 6]).max() <= bound, (i, r[i], rr[6 * i:6 * i + 6])
        want = np.zeros((6, 12))
        for q, c0 in ((s, 0), (S + n, 6)):
            o, d = prog.off[q], prog.off[q + 1] - prog.off[q]
            want[:, c0:c0 + d] = JJ[6 * i:6 * i + 6, o:o + d]
        assert np.abs(J[i] - want).max() <= bound, (i, np.abs(J[i] - want).max(), bound)


def test_factors_at_the_angle_axis_edges(ctx):
    """One constraint with rotation errors of 0, either side of the 1e-7 cutoff, either side of pi, and 90 degrees, with each
    quaternion negated: the residual and the Jacobian against the 50-digit reference."""
    axis = np.array([0.3, -0.5, 0.8]) / np.linalg.norm([0.3, -0.5, 0.8])
    xi = np.array([0.4, -0.2, 0.1, *pc.aa_to_q([0.1, -0.2, 0.3])])
    for angle in (0.0, 0.9e-7, 1.1e-7, np.pi / 2, np.pi - 1e-3, np.pi + 1e-3):
        qz = pc.aa_to_q(angle * axis)
        for flip in range(3):
            sub = [pc.IDENT.copy(), xi.copy()]
            node = np.array([1.0, 0.5, -0.3, *pc.aa_to_q([0.1, -0.2, 0.3])])
            z = np.array([0.5, 0.8, -0.3, *qz])
            if flip == 1:
                sub[1][3:] *= -1
            elif flip == 2:
                z[3:] *= -1
            p = pr.problem(sub, [node], [(1, 0, z, 3.0, 7.0), (0, 0, z, 1.0, 1.0)])
            r, J = ctx.pose_graph_evaluate(sub, [node], p["constraints"])
            prog = pr.Program(p)
            rr, JJ = pr.evaluate(prog, pr.to_A(p["x"], EXACT), EXACT)
            rr, JJ = pr._f(rr), pr._f(JJ)
            for i, (s, n, zz, tw, rw) in enumerate(p["constraints"]):
                bound = 64 * EPS * max(tw, rw) * (1 + np.abs(p["x"][s, :3]).max() + np.abs(p["x"][2 + n, :3]).max() + np.abs(zz[:3]).max())
                assert np.abs(r[i] - rr[6 * i:6 * i + 6]).max() <= bound, (angle, flip, i)
                want = np.zeros((6, 12))
                for q, c0 in ((s, 0), (2 + n, 6)):
                    o, d = prog.off[q], prog.off[q + 1] - prog.off[q]
                    want[:, c0:c0 + d] = JJ[6 * i:6 * i + 6, o:o + d]
                assert np.abs(J[i] - want).max() <= bound, (angle, flip, i, np.abs(J[i] - want).max())


@pytest.mark.parametrize("name", sorted(CASES))
def test_solve_matches_the_reference(ctx, exact, name):
    p, e = CASES[name][1], exact[name]
    gs, gn, s, info = _run(ctx, p)
    for k in SUMMARY_COUNTS:
        assert s[k] == e["summary"][k], (k, s[k], e["summary"][k])
    for k in ("initial_cost", "final_cost"):
        assert abs(s[k] - e["summary"][k]) <= 1e-9 * e["summary"][k] + cost_floor(p), (k, s[k], e["summary"][k])
    got = np.concatenate([gs, gn])
    assert pose_error(got, np.concatenate([e["submaps"], e["nodes"]])) <= 1e-7
    assert info.num_local_parameters == e["num_local_parameters"]
    if e["num_local_parameters"]:
        prog = e["program"]
        d = _local_difference(prog, got, e["x"])
        H = pr.hessian(prog, e["final"]["J"], EXACT)
        assert 0.5 * d @ H @ d <= 1e-9 * e["summary"]["final_cost"] + cost_floor(p) + 1e-24 * np.trace(H)
    # what must not move, bit for bit
    x = p["x"]
    keep = p["frozen"].copy()
    used = np.zeros(len(x), bool)
    for c in p["constraints"]:
        used[c[0]] = used[p["S"] + c[1]] = True
    keep |= ~used
    assert np.array_equal(got[keep], x[keep])
    assert np.array_equal(got[0, :3], x[0, :3])
    if p["fix_z"]:
        assert np.array_equal(got[:, 2], x[:, 2])


def test_trajectory_scale_against_the_fp64_reference(ctx):
    """trajectory_graph(6, 60, loops_every=3) against the reference's fp64 run: exact counts where every decision of the fp64
    trace keeps half a decade, costs to 1e-8 (h = 6e-6 differences), poses to 1e-6."""
    submaps, nodes, cons = trajectory_graph(6, 60, loops_every=3)
    p = pr.problem(submaps, nodes, cons)
    f = pr.solve(p, ir.FP64)
    gs, gn, s, _ = ctx.pose_graph_solve_sparse(submaps, nodes, cons)
    assert min(pr.margin(*d) for d in f["decisions"]) >= 0.5
    for k in SUMMARY_COUNTS:
        assert s[k] == f["summary"][k], (k, s[k], f["summary"][k])
    for k in ("initial_cost", "final_cost"):
        assert abs(s[k] - f["summary"][k]) <= 1e-8 * f["summary"][k]
    assert pose_error(np.concatenate([gs, gn]), np.concatenate([f["submaps"], f["nodes"]])) <= 1e-6


def test_world_of_one_finds_the_referenced_poses(ctx):
    """With a communicator the referenced poses are read off the exchanged pair lists: the same result as without one, and the
    set-up exchange carries only the meta, two agreed reservations and the pair list."""
    import dliom
    p = CASES["unconstrained_far_node"][1]
    a = _run(ctx, p)
    comm = dliom.Comm(ctx, dliom.comm_unique_id(), 0, 1)
    b = _run(ctx, p, comm=comm)
    comm.close()
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2] == b[2]
    K = b[3].num_pairs
    assert b[3].setup_exchange_bytes == 32 + 4 + 4 + 8 * K and b[3].num_local_parameters == a[3].num_local_parameters


_TWO_RANKS = r"""
import sys, numpy as np
sys.path[:0] = [{root!r} + "/d-liom_b200", {root!r} + "/tests"]
import dliom
import posegraph_cases as pc
rank, uid = int(sys.argv[1]), bytes.fromhex(sys.argv[2])
ctx = dliom.Context(rank)
comm = dliom.Comm(ctx, uid, rank, 2)
p = pc.cases()["trajectory_4x12"][1]
S = p["S"]
# node 11 and submap 3 are referenced on rank 1 only; rank 0 holds every other constraint
mine = [c for c in p["constraints"] if (c[1] == 11 or c[0] == 3) == (rank == 1)]
s, n, summ, info = ctx.pose_graph_solve_sparse(p["x"][:S], p["x"][S:], mine, comm=comm)
np.save(sys.argv[3], np.concatenate([s, n]))
comm.close(); ctx.close()
"""


def test_two_ranks_with_a_pose_referenced_on_one_rank(ctx, tmp_path):
    count = subprocess.run([sys.executable, "-c", "import torch; print(torch.cuda.device_count())"], capture_output=True, text=True)
    if int(count.stdout.strip() or 0) < 2:    # in a fresh process: torch cannot load next to the library's NCCL
        pytest.skip("needs two GPUs")
    import dliom
    uid = dliom.comm_unique_id().hex()
    script = tmp_path / "rank.py"
    script.write_text(_TWO_RANKS.format(root=ROOT))
    outs = [tmp_path / f"r{r}.npy" for r in range(2)]
    procs = [subprocess.Popen([sys.executable, str(script), str(r), uid, str(outs[r])]) for r in range(2)]
    assert [q.wait(timeout=300) for q in procs] == [0, 0]
    a, b = np.load(outs[0]), np.load(outs[1])
    assert np.array_equal(a, b)
    p = CASES["trajectory_4x12"][1]
    s, n, _, _ = _run(ctx, p)
    assert pose_error(a, np.concatenate([s, n])) <= 1e-8
