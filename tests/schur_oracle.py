"""CPU oracle of the block-sparse pose-graph solve (test infrastructure).

The same problem as the oracle's dense solve (oracle/orc_posegraph.h: OptimizationProblem3D::Solve with SPA constraints only) and
the same trust-region state machine and constants as oracle/orc_nls.h's solve_trust_region with monotonic steps, but the Jacobian
is kept per residual block (6 x 12 per constraint) and the normal equations are solved by eliminating the node blocks (Schur
complement) and factoring the submaps' reduced system densely. Memory grows with the number of constraints, not with the square
of the number of poses, so it checks the device's sparse solve at sizes the dense oracle cannot hold.

Also the frozen poses of OptimizationProblem3D::Solve's frozen_trajectories (optimization_problem_3d.cc:283-329), restating
Ceres 1.13 from memory, as orc_nls.h does: constant parameter blocks are removed from the minimised program (a frozen first submap
loses its rotation parameters too); residual blocks whose parameters are all constant leave it and only add a fixed cost;
Summary::initial_cost / final_cost are reported as x_cost + fixed_cost, while the function tolerance sees x_cost; with no
parameters left the solve returns at once with CONVERGENCE.

The SPA residual and its ambient Jacobian come from the oracle library itself (orc.spa_residual: its JetN autodiff)."""
import numpy as np
import scipy.linalg

MIN_LM_DIAGONAL, MAX_LM_DIAGONAL = 1e-6, 1e32
INITIAL_RADIUS, MAX_RADIUS, MIN_RADIUS = 1e4, 1e16, 1e-32
MIN_RELATIVE_DECREASE, FUNCTION_TOL, GRADIENT_TOL, PARAMETER_TOL = 1e-3, 1e-6, 1e-10, 1e-8
MAX_CONSECUTIVE_INVALID = 5
CONVERGENCE, NO_CONVERGENCE, FAILURE = 0, 1, 2


def _qmul(a, b):   # (..., 4) quaternion products, (w, x, y, z)
    return np.stack([a[..., 0] * b[..., 0] - a[..., 1] * b[..., 1] - a[..., 2] * b[..., 2] - a[..., 3] * b[..., 3],
                     a[..., 0] * b[..., 1] + a[..., 1] * b[..., 0] + a[..., 2] * b[..., 3] - a[..., 3] * b[..., 2],
                     a[..., 0] * b[..., 2] + a[..., 2] * b[..., 0] + a[..., 3] * b[..., 1] - a[..., 1] * b[..., 3],
                     a[..., 0] * b[..., 3] + a[..., 3] * b[..., 0] + a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1]], -1)


class SchurPoseGraph:
    def __init__(self, orc, num_submaps, poses7, constraints, fix_z, frozen):
        self.orc, self.S = orc, num_submaps
        self.P = len(poses7)
        tdof = 2 if fix_z else 3
        fr = np.zeros(self.P, bool) if frozen is None else np.asarray(frozen, bool)
        self.dim = np.array([0 if fr[p] else (2 if p == 0 else 3 + tdof) for p in range(self.P)])
        self.roff = np.concatenate([[0], np.cumsum(self.dim[:self.S])])
        self.n_red = int(self.roff[-1])
        live = [c for c in constraints if self.dim[c[0]] + self.dim[self.S + c[1]] > 0]
        self.fixed = [c for c in constraints if self.dim[c[0]] + self.dim[self.S + c[1]] == 0]
        self.cons = live
        self.pairs = sorted({(int(c[0]), int(c[1])) for c in live})
        self.pair_of = {p: k for k, p in enumerate(self.pairs)}
        self.node_pairs = [[] for _ in range(self.P - self.S)]
        for k, (s, n) in enumerate(self.pairs):
            self.node_pairs[n].append(k)
        # ambient parameters the norms see: rotation of every live pose, translation of every live pose but the first submap
        mask = np.zeros((self.P, 7), bool)
        for p in range(self.P):
            if self.dim[p]:
                mask[p, 3:] = True
                mask[p, :3] = self.dim[p] != 2
        self.mask = mask

    # ---- residuals, local Jacobians (6 x 12: submap slots 0..5, node slots 6..11)
    def _project(self, q, de, d):
        out = np.zeros(6)
        w, x, y, z = q
        if d == 2:
            c0, c1 = np.array([-x, w, z, -y]), np.array([-y, -z, w, x])
            out[0], out[1] = de[:4] @ c0, de[:4] @ c1
        elif d > 0:
            jj = np.array([[-x, -y, -z], [w, z, -y], [-z, w, x], [y, -x, w]])
            out[:3] = de[:4] @ jj
            out[3:d] = de[4:4 + d - 3]
        return out

    def residuals(self, x, cons, jacobian):
        m = len(cons)
        res, J = np.zeros((m, 6)), (np.zeros((m, 6, 12)) if jacobian else None)
        for i, (s, n, z, tw, rw) in enumerate(cons):
            e, jac = self.orc.spa_residual(x[s], x[self.S + n], z, tw, rw)
            res[i] = e
            if jacobian:
                for r in range(6):
                    J[i, r, :6] = self._project(x[s, 3:], jac[r, :7], self.dim[s])
                    J[i, r, 6:] = self._project(x[self.S + n, 3:], jac[r, 7:], self.dim[self.S + n])
        return res, J

    def evaluate(self, x):
        res, J = self.residuals(x, self.cons, True)
        g, H, Hk = np.zeros((self.P, 6)), np.zeros((self.P, 6, 6)), np.zeros((len(self.pairs), 6, 6))
        for i, (s, n, *_) in enumerate(self.cons):
            Js, Jn = J[i, :, :6], J[i, :, 6:]
            g[s] += Js.T @ res[i]
            g[self.S + n] += Jn.T @ res[i]
            H[s] += Js.T @ Js
            H[self.S + n] += Jn.T @ Jn
            Hk[self.pair_of[(int(s), int(n))]] += Js.T @ Jn
        return 0.5 * float(np.sum(res * res)), g, H, Hk

    def plus(self, x, delta):
        out = x.copy()
        for p in range(self.P):
            d = self.dim[p]
            if d == 0:
                continue
            q, dl = x[p, 3:], delta[p]
            if d == 2:   # ConstantYawQuaternionPlus
                nn = np.sqrt(dl[0] * dl[0] + dl[1] * dl[1])
                s = 1.0 if nn < 1e-6 else np.sin(nn) / nn
                out[p, 3:] = _qmul(q, np.array([1.0 if nn < 1e-6 else np.cos(nn), s * dl[0], s * dl[1], 0.0]))
                continue
            nn = np.sqrt(dl[0] * dl[0] + dl[1] * dl[1] + dl[2] * dl[2])
            if nn > 0:
                s = np.sin(nn) / nn
                out[p, 3:] = _qmul(np.array([np.cos(nn), s * dl[0], s * dl[1], s * dl[2]]), q)
            out[p, :d - 3] = x[p, :d - 3] + dl[3:d]
        return out

    # ---- (S H S + D / radius) y = S g by Schur elimination of the node blocks. -> (step = -y per pose, model cost change) or None
    def step(self, g, H, Hk, scale, diag, radius):
        S, dim = self.S, self.dim
        gs = scale * g
        Hs = scale[:, :, None] * H * scale[:, None, :]
        node_L, z = {}, {}
        for p in range(S, self.P):
            d = dim[p]
            if d == 0:
                continue
            A = Hs[p, :d, :d] + np.diag(diag[p, :d] / radius)
            try:
                node_L[p] = np.linalg.cholesky(A)
            except np.linalg.LinAlgError:
                return None
            z[p] = scipy.linalg.cho_solve((node_L[p], True), gs[p, :d])
        W, Y = {}, {}
        for k, (s, n) in enumerate(self.pairs):
            p, ds, dn = S + n, dim[s], dim[S + n]
            if ds == 0 or dn == 0:
                continue
            W[k] = scale[s, :ds, None] * Hk[k, :ds, :dn] * scale[p, None, :dn]
            Y[k] = scipy.linalg.cho_solve((node_L[p], True), W[k].T)
        A = np.zeros((self.n_red, self.n_red))
        b = np.zeros(self.n_red)
        for s in range(S):
            d = dim[s]
            if d:
                o = self.roff[s]
                A[o:o + d, o:o + d] = Hs[s, :d, :d] + np.diag(diag[s, :d] / radius)
                b[o:o + d] = gs[s, :d]
        for k, (s, n) in enumerate(self.pairs):
            if k in W:
                o = self.roff[s]
                b[o:o + dim[s]] -= W[k] @ z[S + n]
        for n, ks in enumerate(self.node_pairs):
            for k1 in ks:
                for k2 in ks:
                    if k1 in W and k2 in W:
                        s1, s2 = self.pairs[k1][0], self.pairs[k2][0]
                        o1, o2 = self.roff[s1], self.roff[s2]
                        A[o1:o1 + dim[s1], o2:o2 + dim[s2]] -= W[k1] @ Y[k2]
        step = np.zeros((self.P, 6))
        if self.n_red:
            try:
                L = np.linalg.cholesky(A)
            except np.linalg.LinAlgError:
                return None
            y_red = scipy.linalg.cho_solve((L, True), b)
            for s in range(S):
                step[s, :dim[s]] = -y_red[self.roff[s]:self.roff[s] + dim[s]]
        for p in range(S, self.P):
            d = dim[p]
            if d == 0:
                continue
            y = z[p].copy()
            for k in self.node_pairs[p - S]:
                if k in Y:
                    s = self.pairs[k][0]
                    y -= Y[k] @ (-step[s, :dim[s]])
            step[p, :d] = -y
        if not np.all(np.isfinite(step)):
            return None
        quad = 0.0
        for p in range(self.P):
            quad += step[p] @ Hs[p] @ step[p]
        for k, (s, n) in enumerate(self.pairs):
            if k in W:
                quad += 2.0 * step[s, :dim[s]] @ W[k] @ step[S + n, :dim[S + n]]
        return step, -(float(np.sum(step * gs)) + 0.5 * quad)

    def norms(self, x, y):
        d = (x - y)[self.mask]
        return (float(np.max(np.abs(d))) if d.size else 0.0), float(np.sqrt(np.sum(x[self.mask] ** 2))), float(np.sqrt(np.sum(d * d)))


def solve(orc, submap_poses, node_poses, constraints, fix_z=False, max_iter=50, frozen=None):
    """-> (submap poses, node poses, summary dict with the keys of orc.pose_graph_solve's, num_reduced_parameters, num_pairs)."""
    S = len(submap_poses)
    x = np.concatenate([np.asarray(submap_poses, np.float64).reshape(S, 7),
                        np.asarray(node_poses, np.float64).reshape(-1, 7)])
    pg = SchurPoseGraph(orc, S, x, list(constraints), fix_z, frozen)
    fixed_cost = 0.0
    if pg.fixed:
        res, _ = pg.residuals(x, pg.fixed, False)
        fixed_cost = 0.5 * float(np.sum(res * res))
    summary = {"num_reduced_parameters": pg.n_red, "num_pairs": len(pg.pairs), "num_successful_steps": 0,
               "num_unsuccessful_steps": 0, "num_iterations": 0, "num_evaluations": 1}
    if not pg.dim.any():
        cost = 0.5 * float(np.sum(pg.residuals(x, pg.cons, False)[0] ** 2)) if pg.cons else 0.0
        summary.update(initial_cost=cost + fixed_cost, final_cost=cost + fixed_cost, termination=CONVERGENCE)
        return x[:S].copy(), x[S:].copy(), summary

    def gradient_max_norm(at, g):
        return pg.norms(at, pg.plus(at, -g))[0]

    x_cost, g, H, Hk = pg.evaluate(x)
    live = np.arange(6)[None, :] < pg.dim[:, None]
    scale = np.where(live, 1.0 / (1.0 + np.sqrt(np.where(live, np.einsum("pii->pi", H), 0.0))), 0.0)
    gmax, x_norm = gradient_max_norm(x, g), pg.norms(x, x)[1]
    best, minimum_cost = x.copy(), np.finfo(np.float64).max
    radius, decrease_factor, reuse_diagonal, num_invalid = INITIAL_RADIUS, 2.0, False, 0
    initial_cost, costs = x_cost, []
    it_cost, it_successful, iteration = x_cost, True, 0
    diag = None
    termination = None
    while True:
        if it_successful:
            summary["num_successful_steps"] += 1
            if x_cost < minimum_cost:
                minimum_cost, best = x_cost, x.copy()
        else:
            summary["num_unsuccessful_steps"] += 1
        costs.append(it_cost)
        if iteration >= max_iter:
            termination = NO_CONVERGENCE
            break
        if it_successful and gmax <= GRADIENT_TOL:
            termination = CONVERGENCE
            break
        if radius <= MIN_RADIUS:
            termination = CONVERGENCE
            break
        iteration += 1
        if not reuse_diagonal:
            hd = np.einsum("pii->pi", H) * scale * scale
            diag = np.where(live, np.clip(hd, MIN_LM_DIAGONAL, MAX_LM_DIAGONAL), 0.0)
        reuse_diagonal = True
        out = pg.step(g, H, Hk, scale, diag, radius)
        if out is None or not out[1] > 0.0:
            num_invalid += 1
            if num_invalid >= MAX_CONSECUTIVE_INVALID:
                termination = FAILURE
                break
            radius *= 0.5
            it_cost, it_successful = x_cost, False
            continue
        num_invalid = 0
        step, model_cost_change = out
        cand = pg.plus(x, step * scale)
        cand_cost = 0.5 * float(np.sum(pg.residuals(cand, pg.cons, False)[0] ** 2))
        summary["num_evaluations"] += 1
        if not np.isfinite(cand_cost):
            cand_cost = np.finfo(np.float64).max
        if pg.norms(x, cand)[2] <= PARAMETER_TOL * (x_norm + PARAMETER_TOL):
            termination = CONVERGENCE
            break
        if abs(x_cost - cand_cost) <= FUNCTION_TOL * x_cost:
            termination = CONVERGENCE
            break
        relative_decrease = (x_cost - cand_cost) / model_cost_change
        if relative_decrease > MIN_RELATIVE_DECREASE:
            x = cand
            x_cost, g, H, Hk = pg.evaluate(x)
            gmax, x_norm = gradient_max_norm(x, g), pg.norms(x, x)[1]
            it_cost, it_successful = x_cost, True
            radius = min(MAX_RADIUS, radius / max(1.0 / 3.0, 1.0 - (2.0 * relative_decrease - 1.0) ** 3))
            decrease_factor, reuse_diagonal = 2.0, False
        else:
            it_cost, it_successful = cand_cost, False
            radius /= decrease_factor
            decrease_factor *= 2.0
            reuse_diagonal = True
    summary.update(initial_cost=initial_cost + fixed_cost, final_cost=min([initial_cost] + costs) + fixed_cost,
                   termination=termination, num_iterations=len(costs))
    return best[:S].copy(), best[S:].copy(), summary
