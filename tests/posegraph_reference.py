"""Independent reference of the block-sparse pose-graph solve (dl_pose_graph_solve_sparse), written from
OptimizationProblem3D::Solve (optimization_problem_3d.cc:283-343, SPA constraints only, TrivialLoss), SpaCostFunction3D
(spa_cost_function_3d.h:47-60 with cost_helpers_impl.h's ComputeUnscaledError), RotationQuaternionToAngleAxisVector
(transform.h:60-80) and the documented behaviour of Ceres 1.13's Problem, Program and TrustRegionMinimizer.

  blocks     one rotation (4) and one translation (3) block per submap and node. The first submap's rotation uses
             ConstantYawQuaternionPlus (rotation_parameterization.h:29-40: x * (cos|d|, s d0, s d1, 0), s = sin|d| / |d|, the
             identity chart (1, d0, d1, 0) below |d| = 1e-6) and its translation is constant; every other rotation uses
             ceres::QuaternionParameterization ((cos|d|, sin|d| / |d| d) * x); with fix_z every translation uses
             SubsetParameterization(3, {2}). A frozen pose has both blocks constant.
  program    Program::RemoveFixedBlocks: constant blocks and blocks no residual uses leave the minimised program; a residual
             block whose blocks are all constant leaves it and adds only to the fixed cost. With no parameters left the solve
             returns at once with CONVERGENCE: costs = the fixed cost, no iterations.
  Jacobian   central differences in each block's local chart (h = 1e-20 at 50 digits, h = 6e-6 in fp64), so no derivative is
             shared with the device's forward-mode duals or the oracle's JetN.
  solve      the dense normal equations over all live local parameters (no Schur complement), in the working precision, and
             Ceres 1.13's LM loop: Jacobi scaling from the column norms at iteration zero only, LM diagonal = the scaled column
             norms squared clamped to [1e-6, 1e32] and divided by the radius, model_cost_change = -(g.d + 1/2 d^T H d), a step
             valid when finite and that change is positive; five consecutive invalid steps give FAILURE, and an invalid step
             is treated as a rejected one (LevenbergMarquardtStrategy::StepIsInvalid: radius / decrease_factor, decrease_factor
             doubled); the parameter tolerance before the function tolerance; the gradient check
             ||x - Plus(x, -g)||_inf after a successful iteration; monotonic steps; the best point is returned.
  summary    dl_solve_summary's fields: initial_cost / final_cost with the fixed cost added (the tolerances see the rest),
             num_iterations (recorded iterations, iteration zero included), num_successful_steps, num_unsuccessful_steps,
             num_evaluations (the start plus one per candidate), termination 0 / 1 / 2.

Every decision the loop takes is returned with its quantity and threshold ("decisions"), with the condition number of the
damped system of each step, so that tests can require the decisions to keep a margin from their thresholds.

A problem is a dict of floats (see `problem`); every function takes the arithmetic A of imu_reference (FP64 or Exact)."""
import math

import numpy as np

from imu_reference import FP64, Exact

CONVERGENCE, NO_CONVERGENCE, FAILURE = 0, 1, 2
MIN_LM_DIAGONAL, MAX_LM_DIAGONAL = 1e-6, 1e32
INITIAL_RADIUS, MAX_RADIUS, MIN_RADIUS = 1e4, 1e16, 1e-32
MIN_RELATIVE_DECREASE, FUNCTION_TOL, GRADIENT_TOL, PARAMETER_TOL = 1e-3, 1e-6, 1e-10, 1e-8
MAX_CONSECUTIVE_INVALID = 5


def problem(submaps, nodes, constraints, fix_z=False, max_iter=50, frozen=None):
    """submaps / nodes: 7-vectors (t xyz, q wxyz); constraints: (submap, node, zbar7, translation_weight, rotation_weight)."""
    S = len(submaps)
    x = np.concatenate([np.asarray(submaps, float).reshape(S, 7), np.asarray(nodes, float).reshape(-1, 7)])
    return dict(S=S, x=x, constraints=[(int(s), int(n), np.asarray(z, float), float(tw), float(rw)) for s, n, z, tw, rw in constraints],
                fix_z=bool(fix_z), max_iter=int(max_iter),
                frozen=np.zeros(len(x), bool) if frozen is None else np.asarray(frozen, bool).copy())


def _m(A):
    return A.ctx if isinstance(A, Exact) else math


def _arr(v, A):
    return np.array(v, dtype=object if isinstance(A, Exact) else float)


def _f(v):
    return np.array([float(a) for a in np.ravel(v)]).reshape(np.shape(v))


# ------------------------------------------------------------------ the residual
def _qmul(a, b):   # ceres::QuaternionProduct / Eigen's product, (w, x, y, z)
    return (a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3],
            a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
            a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1],
            a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0])


def _rotate(q, v):   # Eigen's Quaternion * Vector3: v + w uv + q.vec x uv, uv = 2 q.vec x v
    uv = (2 * (q[2] * v[2] - q[3] * v[1]), 2 * (q[3] * v[0] - q[1] * v[2]), 2 * (q[1] * v[1] - q[2] * v[0]))
    return (v[0] + q[0] * uv[0] + (q[2] * uv[2] - q[3] * uv[1]),
            v[1] + q[0] * uv[1] + (q[3] * uv[0] - q[1] * uv[2]),
            v[2] + q[0] * uv[2] + (q[1] * uv[1] - q[2] * uv[0]))


def angle_axis(q, A):
    """RotationQuaternionToAngleAxisVector: normalise, flip to w >= 0, angle = 2 atan2(|vec|, w), scale = 2 below 1e-7."""
    n = A.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3])
    w, x, y, z = q[0] / n, q[1] / n, q[2] / n, q[3] / n
    if w < 0:
        w, x, y, z = -w, -x, -y, -z
    angle = 2 * _m(A).atan2(A.sqrt(x * x + y * y + z * z), w)
    scale = A.num(2) if angle < 1e-7 else angle / _m(A).sin(angle / 2)
    return (scale * x, scale * y, scale * z)


def residual(c, xi, xj, A):
    """SpaCostFunction3D (c_i = the submap's pose, c_j = the node's; 7-vectors t, q in A): [tw (zbar_t - R_i^-1 (t_j - t_i)),
    rw AngleAxis((q_j^-1 q_i) zbar_q)]."""
    _, _, z, tw, rw = c
    qi, qj = tuple(xi[3:7]), tuple(xj[3:7])
    h_t = _rotate((qi[0], -qi[1], -qi[2], -qi[3]), tuple(xj[k] - xi[k] for k in range(3)))
    hr_inv = _qmul((qj[0], -qj[1], -qj[2], -qj[3]), qi)
    aa = angle_axis(_qmul(hr_inv, tuple(A.num(v) for v in z[3:7])), A)
    return [A.num(tw) * (A.num(z[k]) - h_t[k]) for k in range(3)] + [A.num(rw) * aa[k] for k in range(3)]


# ------------------------------------------------------------------ blocks and the program
class Program:
    """The minimised program of one problem: per pose its live local parameters (rotation then translation)."""

    def __init__(self, p):
        self.S, self.P = p["S"], len(p["x"])
        used = np.zeros(self.P, bool)
        for s, n, *_ in p["constraints"]:
            used[s] = used[self.S + n] = True
        live = used & ~p["frozen"]
        self.tdof = 2 if p["fix_z"] else 3
        self.rdim = np.array([0 if not live[q] else (2 if q == 0 else 3) for q in range(self.P)])
        self.tdim = np.array([0 if not live[q] or q == 0 else self.tdof for q in range(self.P)])
        self.off = np.concatenate([[0], np.cumsum(self.rdim + self.tdim)])
        self.n = int(self.off[-1])
        self.live = self.rdim + self.tdim > 0
        # residual blocks: live unless both poses are constant
        self.cons = [c for c in p["constraints"] if self.live[c[0]] or self.live[self.S + c[1]]]
        self.fixed = [c for c in p["constraints"] if not (self.live[c[0]] or self.live[self.S + c[1]])]

    def plus_pose(self, q, xq, d, A):
        """x (+) d for pose q (d: its rdim + tdim local parameters)."""
        out = list(xq)
        r = self.rdim[q]
        rot = tuple(xq[3:7])
        if r == 2:
            nn = A.sqrt(d[0] * d[0] + d[1] * d[1])
            s = A.num(1) if nn < 1e-6 else _m(A).sin(nn) / nn
            out[3:7] = _qmul(rot, (A.num(1) if nn < 1e-6 else _m(A).cos(nn), s * d[0], s * d[1], A.num(0)))
        elif r == 3:
            nn = A.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2])
            if nn > 0:
                s = _m(A).sin(nn) / nn
                out[3:7] = _qmul((_m(A).cos(nn), s * d[0], s * d[1], s * d[2]), rot)
        for k in range(self.tdim[q]):
            out[k] = xq[k] + d[r + k]
        return out

    def plus(self, x, delta, A):
        out = x.copy()
        for q in range(self.P):
            if self.live[q]:
                out[q] = _arr(self.plus_pose(q, x[q], delta[self.off[q]:self.off[q + 1]], A), A)
        return out

    def ambient(self, x):
        """The state vector Ceres's norms see: every live block's ambient values."""
        v = []
        for q in range(self.P):
            if self.rdim[q]:
                v += list(x[q, 3:7])
            if self.tdim[q]:
                v += list(x[q, :3])
        return v


def to_A(x, A):
    return np.array([[A.num(v) for v in row] for row in x], dtype=object if isinstance(A, Exact) else float)


def evaluate(prog, x, A, cons=None, jacobian=True):
    """-> residuals [m] and the local Jacobian [m, n] (central differences), both in A."""
    cons = prog.cons if cons is None else cons
    h = A.num("1e-20") if isinstance(A, Exact) else 6e-6
    r, J = [], (A.zeros(6 * len(cons), prog.n) if jacobian else None)
    for i, c in enumerate(cons):
        s, pn = c[0], prog.S + c[1]
        r += residual(c, x[s], x[pn], A)
        if not jacobian:
            continue
        for q in (s, pn):
            o, d = prog.off[q], prog.off[q + 1] - prog.off[q]
            for a in range(d):
                cols = []
                for sign in (1, -1):
                    dl = [A.num(0)] * d
                    dl[a] = sign * h
                    xq = prog.plus_pose(q, x[q], dl, A)
                    cols.append(residual(c, xq, x[pn], A) if q == s else residual(c, x[s], xq, A))
                for k in range(6):
                    J[6 * i + k, o + a] = (cols[0][k] - cols[1][k]) / (2 * h)
    return _arr(r, A), J


def cholesky_solve(H, b, A):
    """H^-1 b, or None when H is not positive definite."""
    if isinstance(A, Exact):
        try:
            y = A.ctx.cholesky_solve(A.ctx.matrix(H.tolist()), A.ctx.matrix(list(b)))
        except ValueError:
            return None
        return _arr([y[k] for k in range(len(b))], A)
    try:
        L = np.linalg.cholesky(H)
    except np.linalg.LinAlgError:
        return None
    return np.linalg.solve(L.T, np.linalg.solve(L, b))


def _norm(v, A):
    return A.sqrt(sum((a * a for a in v), A.num(0)))


def step(prog, J, r, scale, diag, radius, A):
    """The LM step at one point: (Js^T Js + D / radius) y = Js^T r, step = -y. -> (step, model_cost_change, kappa) or None."""
    Js = J * scale[None, :]
    H, g = Js.T.dot(Js), Js.T.dot(r)
    Hd = H.copy()
    for a in range(prog.n):
        Hd[a, a] = Hd[a, a] + diag[a] / A.num(radius)
    kappa = float(np.linalg.cond(_f(Hd)))
    y = cholesky_solve(Hd, g, A)
    if y is None or not all(math.isfinite(float(v)) for v in y):
        return None, kappa
    st = -y
    return (st, -(st.dot(g) + st.dot(H.dot(st)) / 2)), kappa


def solve(p, A=FP64, keep_unused=False):
    """Ceres 1.13's LM on the program of p. keep_unused: keep the poses no constraint refers to in x (a counterfactual the tests
    use to show that the removal matters). -> dict(submaps, nodes (floats), summary, decisions, kappas, num_local_parameters)."""
    prog = Program(p)
    if keep_unused:
        prog.rdim = np.array([0 if p["frozen"][k] else (2 if k == 0 else 3) for k in range(prog.P)])
        prog.tdim = np.array([0 if p["frozen"][k] or k == 0 else prog.tdof for k in range(prog.P)])
        prog.off = np.concatenate([[0], np.cumsum(prog.rdim + prog.tdim)])
        prog.n, prog.live = int(prog.off[-1]), prog.rdim + prog.tdim > 0
    x = to_A(p["x"], A)
    fixed_cost = A.num(0)
    if prog.fixed:
        rf, _ = evaluate(prog, x, A, prog.fixed, jacobian=False)
        fixed_cost = rf.dot(rf) / 2
    out = dict(num_local_parameters=prog.n, decisions=[], kappas=[], trace=[])
    dec = out["decisions"]
    summary = dict(num_successful_steps=0, num_unsuccessful_steps=0, num_iterations=0, num_evaluations=1)
    if prog.n == 0:
        summary.update(initial_cost=float(fixed_cost), final_cost=float(fixed_cost), termination=CONVERGENCE)
        out.update(submaps=_f(x[:prog.S]), nodes=_f(x[prog.S:]), summary=summary, x=x)
        return out

    def linearise(at):
        r, J = evaluate(prog, at, A)
        return r.dot(r) / 2, r, J

    def gradient_max_norm(at, J, r):
        g = J.T.dot(r)
        a, b = prog.ambient(at), prog.ambient(prog.plus(at, -g, A))
        return max(abs(u - v) for u, v in zip(a, b))

    x_cost, r, J = linearise(x)
    scale = _arr([1 / (1 + A.sqrt(sum((J[i, a] * J[i, a] for i in range(J.shape[0])), A.num(0)))) for a in range(prog.n)], A)
    gmax, x_norm = gradient_max_norm(x, J, r), _norm(prog.ambient(x), A)
    initial_cost, minimum_cost, best = x_cost, None, x.copy()
    radius, decrease_factor, reuse_diagonal, num_invalid = INITIAL_RADIUS, 2.0, False, 0
    it_cost, it_successful, iteration, costs, diag = x_cost, True, 0, [], None
    while True:
        if it_successful:
            summary["num_successful_steps"] += 1
            if minimum_cost is None or x_cost < minimum_cost:
                minimum_cost, best = x_cost, x.copy()
        else:
            summary["num_unsuccessful_steps"] += 1
        costs.append(it_cost)
        if iteration >= p["max_iter"]:
            termination = NO_CONVERGENCE
            break
        if it_successful:
            dec.append(("gradient", float(gmax), GRADIENT_TOL))
            if gmax <= GRADIENT_TOL:
                termination = CONVERGENCE
                break
        if radius <= MIN_RADIUS:
            termination = CONVERGENCE
            break
        iteration += 1
        if not reuse_diagonal:
            Js = J * scale[None, :]
            diag = _arr([min(max(Js[:, a].dot(Js[:, a]), MIN_LM_DIAGONAL), MAX_LM_DIAGONAL) for a in range(prog.n)], A)
        reuse_diagonal = True
        st, kappa = step(prog, J, r, scale, diag, radius, A)
        out["kappas"].append(kappa)
        if st is not None:
            dec.append(("model_cost_change", float(st[1]), 0.0))
        if st is None or not st[1] > 0:
            num_invalid += 1
            out["trace"].append(("invalid", radius))
            if num_invalid >= MAX_CONSECUTIVE_INVALID:
                termination = FAILURE
                break
            radius /= decrease_factor
            decrease_factor *= 2.0
            it_cost, it_successful = x_cost, False
            continue
        num_invalid = 0
        d, mcc = st
        cand = prog.plus(x, d * scale, A)
        rc, _ = evaluate(prog, cand, A, jacobian=False)
        cand_cost = rc.dot(rc) / 2
        summary["num_evaluations"] += 1
        if not math.isfinite(float(cand_cost)):
            cand_cost = A.num(np.finfo(np.float64).max)
        step_norm = _norm([u - v for u, v in zip(prog.ambient(x), prog.ambient(cand))], A)
        ptol = PARAMETER_TOL * (x_norm + PARAMETER_TOL)
        dec.append(("parameter", float(step_norm), float(ptol)))
        if step_norm <= ptol:
            out["trace"].append(("parameter", radius))
            termination = CONVERGENCE
            break
        dec.append(("function", float(abs(x_cost - cand_cost)), float(FUNCTION_TOL * x_cost)))
        if abs(x_cost - cand_cost) <= FUNCTION_TOL * x_cost:
            out["trace"].append(("function", radius))
            termination = CONVERGENCE
            break
        relative_decrease = (x_cost - cand_cost) / mcc
        dec.append(("relative_decrease", float(relative_decrease), MIN_RELATIVE_DECREASE))
        if relative_decrease > MIN_RELATIVE_DECREASE:
            out["trace"].append(("accepted", radius))
            x = cand
            x_cost, r, J = linearise(x)
            gmax, x_norm = gradient_max_norm(x, J, r), _norm(prog.ambient(x), A)
            it_cost, it_successful = x_cost, True
            radius = min(MAX_RADIUS, radius / max(1.0 / 3.0, 1.0 - float(2 * relative_decrease - 1) ** 3))
            decrease_factor, reuse_diagonal = 2.0, False
        else:
            out["trace"].append(("rejected", radius))
            it_cost, it_successful = cand_cost, False
            radius /= decrease_factor
            decrease_factor *= 2.0
            reuse_diagonal = True
    summary.update(initial_cost=float(initial_cost + fixed_cost), final_cost=float(min([initial_cost] + costs) + fixed_cost),
                   termination=termination, num_iterations=len(costs))
    out.update(submaps=_f(best[:prog.S]), nodes=_f(best[prog.S:]), summary=summary, x=best, program=prog,
               final=dict(J=J, r=r, scale=scale))
    return out


def margin(name, q, t):
    """Decades between a decision quantity and its threshold; inf where the decision cannot be close (a zero quantity, a cost
    that rose against the relative-decrease threshold, a positive model change against 0)."""
    if name == "model_cost_change":
        return math.inf if q > 0 else 0.0
    if q <= 0 or t <= 0:
        return math.inf
    return abs(math.log10(q / t))


def hessian(prog, J, A):
    """H = J^T J in the local parameters (unscaled), as floats: the metric poses are compared in."""
    return _f(J.T.dot(J))
