"""Independent reference of the window update (dl_window_optimize_batch): the lag-one fixed-lag smoother that stands in for
LocalTrajectoryBuilder3D::WindowOptimize (LTB:693-863), written from the model the header states and from the IMU residual
of integration_base.h:267-301.

  variables  x_i, x_j: 15 tangent parameters each, order p, theta, v, b_a, b_g; x (+) d = (p + d_p, exp(d_theta) q, ...)
             with exp(d) = (cos|d|, sin|d|/|d| d), |d| the half angle (imu_reference.plus)
  residuals  15 prior:   x_i (-) mean, the rotation part d with exp(d) = q_i mean^-1 (sign chosen so that w >= 0),
                         d = atan2(|v|, w) / |v| v, the limit v / w only at |v| = 0
             15 IMU:     integration_base.h:292-299 with the first-order bias correction of :283-290 at x_i's biases
             6 pose:     p_j - z_p, 2 vec(z_q^-1 q_j) (sign chosen so that w >= 0)
             2 gravity:  Unit3 semantics: both directions normalised, R_j b_ref projected onto an orthonormal basis of the
                         tangent plane of g_dir (Unit3::basis' rule: the axis of g_dir's smallest component, which is NOT the
                         device's rule, so the basis itself is an independent check: cost and steps do not depend on it)
  weight     block diagonal: prior information, imu_weight^2 Sigma^-1 (imu_reference.information), 1 / sigma^2
  solve      Gauss-Newton on 1/2 r^T W r with H = J^T W J; stop after the step whose norm is < 1e-10 (one more
             evaluation gives the final cost and linearisation) or after max_num_iterations steps (10 when 0); the
             information of x_j is the Schur complement H_jj - H_ji H_ii^-1 H_ij

Jacobians are central differences in the tangent chart: h = 1e-20 at 50 digits (Exact), h = 6e-6 in fp64. The device uses
forward-mode duals and the C++ oracle fp64 differences with h = 1e-6, so none of the three shares its derivatives.
Problems are plain floats (see `problem`); every function takes the arithmetic `A` of imu_reference (FP64 or Exact)."""
import math

import numpy as np

import imu_reference as ir
from imu_reference import FP64, Exact, conj, qmul, rotate, vadd, vsub, vmul

CONVERGED = 1e-10
NRES, NVAR = 38, 30


def problem(mean_i, prior, pre, matched, sigma_t=0.05, sigma_r=0.01, imu_weight=1.0, G=(0.0, 0.0, 9.8), max_iter=10,
            gravity_factor=None, initial_j=None, basis=None):
    """One window problem in floats. pre: an fp64 imu_reference.Preintegration (what the device gets as dl_preintegration).
    gravity_factor: None or (sigma, g_dir, b_ref). basis: None (Unit3's rule) or a function g_hat -> (b1, b2)."""
    return dict(mean_i=np.asarray(mean_i, float), prior=np.asarray(prior, float), pre=pre, matched=np.asarray(matched, float),
                sigma_t=sigma_t, sigma_r=sigma_r, imu_weight=imu_weight, G=tuple(G), max_iter=max_iter,
                gravity_factor=gravity_factor, initial_j=None if initial_j is None else np.asarray(initial_j, float), basis=basis)


class _Interval:
    """The fields of dl_preintegration in arithmetic A (the attribute names imu_reference.predict reads)."""

    def __init__(self, pre, A):
        self.A = A
        self.sum_dt = A.num(pre.sum_dt)
        self.dp, self.dv = tuple(A.num(x) for x in pre.dp), tuple(A.num(x) for x in pre.dv)
        self.dq = tuple(A.num(x) for x in pre.dq)
        self.ba, self.bg = tuple(A.num(x) for x in pre.ba), tuple(A.num(x) for x in pre.bg)
        self.J = [[A.num(pre.J[i, j]) for j in range(15)] for i in range(15)]
        self.P = pre.P


def _ctx(A):
    return A.ctx if isinstance(A, Exact) else math


def _unit3_basis(g, A):
    """Unit3::basis: the axis of g's smallest |component|, b1 = normalised g x axis, b2 = g x b1."""
    m = min(range(3), key=lambda k: abs(g[k]))
    axis = tuple(A.num(1.0 if k == m else 0.0) for k in range(3))
    b1 = ir.cross(g, axis)
    n = A.sqrt(b1[0] * b1[0] + b1[1] * b1[1] + b1[2] * b1[2])
    b1 = vmul(1 / n, b1)
    return b1, ir.cross(g, b1)


def _unit(v, A):
    v = tuple(A.num(x) for x in v)
    n = A.sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2])
    return vmul(1 / n, v)


def _log(e, A):
    """d with exp(d) = e / |e|: atan2(|v|, w) / |v| v after choosing the sign with w >= 0; v / w at |v| = 0."""
    if e[0] < 0:
        e = tuple(-c for c in e)
    vn = A.sqrt(e[1] * e[1] + e[2] * e[2] + e[3] * e[3])
    f = 1 / e[0] if vn == 0 else _ctx(A).atan2(vn, e[0]) / vn
    return [f * e[1], f * e[2], f * e[3]]


def residuals(p, m, xi, xj, A):
    """The 38 residuals at (x_i, x_j) (16-vectors in A); m = _Interval(p['pre'], A)."""
    mean = [A.num(v) for v in p["mean_i"]]
    r = [xi[k] - mean[k] for k in range(3)]
    r += _log(qmul(tuple(xi[3:7]), conj(tuple(mean[3:7]))), A)
    r += [xi[7 + k] - mean[7 + k] for k in range(9)]
    # IMU (integration_base.h:283-299)
    pi, qi, vi, bai, bgi = tuple(xi[0:3]), tuple(xi[3:7]), tuple(xi[7:10]), tuple(xi[10:13]), tuple(xi[13:16])
    pj, qj, vj, baj, bgj = tuple(xj[0:3]), tuple(xj[3:7]), tuple(xj[7:10]), tuple(xj[10:13]), tuple(xj[13:16])
    dba, dbg = vsub(bai, m.ba), vsub(bgi, m.bg)

    def blk(r0, c0, d):
        return tuple(m.J[r0 + i][c0] * d[0] + m.J[r0 + i][c0 + 1] * d[1] + m.J[r0 + i][c0 + 2] * d[2] for i in range(3))
    th = blk(3, 12, dbg)
    cq = qmul(m.dq, (A.num(1), th[0] / 2, th[1] / 2, th[2] / 2))          # delta_q * Utility::deltaQ(dq_dbg * dbg)
    cp = vadd(vadd(m.dp, blk(0, 9, dba)), blk(0, 12, dbg))
    cv = vadd(vadd(m.dv, blk(6, 9, dba)), blk(6, 12, dbg))
    T = m.sum_dt
    G = tuple(A.num(g) for g in p["G"])
    n2 = cq[0] * cq[0] + cq[1] * cq[1] + cq[2] * cq[2] + cq[3] * cq[3]
    cq_inv = (cq[0] / n2, -cq[1] / n2, -cq[2] / n2, -cq[3] / n2)         # Eigen's inverse(): conjugate / squared norm
    qi_inv = conj(qi)
    rp = vsub(rotate(qi_inv, vsub(vsub(vadd(vmul(T * T / 2, G), pj), pi), vmul(T, vi))), cp)
    rv = vsub(rotate(qi_inv, vsub(vadd(vmul(T, G), vj), vi)), cv)
    e = qmul(cq_inv, qmul(qi_inv, qj))
    r += list(rp) + [2 * e[1], 2 * e[2], 2 * e[3]] + list(rv) + list(vsub(baj, bai)) + list(vsub(bgj, bgi))
    # pose prior
    z = [A.num(v) for v in p["matched"]]
    r += [pj[k] - z[k] for k in range(3)]
    ez = qmul(conj(tuple(z[3:7])), qj)
    if ez[0] < 0:
        ez = tuple(-c for c in ez)
    r += [2 * ez[1], 2 * ez[2], 2 * ez[3]]
    # gravity direction (Unit3::error: the tangent-basis coordinates of R_j b_ref)
    gf = p["gravity_factor"]
    if gf:
        g, b = _unit(gf[1], A), _unit(gf[2], A)
        b1, b2 = (p["basis"] or _unit3_basis)(g, A)
        n = rotate(qj, b)
        r += [b1[0] * n[0] + b1[1] * n[1] + b1[2] * n[2], b2[0] * n[0] + b2[1] * n[1] + b2[2] * n[2]]
    else:
        r += [A.num(0), A.num(0)]
    return r


def row_scales(p, xi, xj):
    """Magnitude of the operands that enter each residual row (floats): the scale of that row's rounding error, for r and J."""
    T = p["pre"].sum_dt
    n = lambda v: float(np.linalg.norm(np.asarray(v, float)))
    G = n(p["G"])
    Jm = np.abs(p["pre"].J).max()
    bias = n(np.asarray(xi[10:16], float) - np.concatenate([p["pre"].ba, p["pre"].bg]))
    s = np.ones(NRES)
    s[0:3] = max(n(xi[0:3]), n(p["mean_i"][0:3]), 1.0)
    s[6:15] = [max(abs(float(xi[7 + k])), abs(p["mean_i"][7 + k]), 1.0) for k in range(9)]
    s[15:18] = 0.5 * G * T * T + n(xj[0:3]) + n(xi[0:3]) + T * n(xi[7:10]) + n(p["pre"].dp) + Jm * bias + 1.0
    s[18:21] = 2.0 * (1.0 + Jm * bias)
    s[21:24] = G * T + n(xj[7:10]) + n(xi[7:10]) + n(p["pre"].dv) + Jm * bias + 1.0
    s[24:30] = [max(abs(float(xi[10 + k])), abs(float(xj[10 + k])), 1.0) for k in range(6)]
    s[30:33] = max(n(xj[0:3]), n(p["matched"][0:3]), 1.0)
    s[33:36] = 2.0
    return s


def weights(p, m, A):
    """W (38 x 38) or None when Sigma is not positive definite."""
    Wi = ir.information(m.P, p["imu_weight"], A)
    if Wi is None:
        return None
    W = A.zeros(NRES, NRES)
    for a in range(15):
        for b in range(15):
            W[a, b] = A.num(p["prior"][a, b])
            W[15 + a, 15 + b] = Wi[a, b]
    st, sr = A.num(p["sigma_t"]), A.num(p["sigma_r"])
    for k in range(3):
        W[30 + k, 30 + k] = 1 / (st * st)
        W[33 + k, 33 + k] = 1 / (sr * sr)
    if p["gravity_factor"]:
        sg = A.num(p["gravity_factor"][0])
        W[36, 36] = W[37, 37] = 1 / (sg * sg)
    return W


def jacobian(p, m, xi, xj, A):
    h = A.num("1e-20") if isinstance(A, Exact) else 6e-6
    J = A.zeros(NRES, NVAR)
    for k in range(NVAR):
        cols = []
        for s in (1, -1):
            d = [A.num(0)] * 15
            d[k % 15] = s * h
            cols.append(residuals(p, m, ir.plus(xi, d, A), xj, A) if k < 15 else residuals(p, m, xi, ir.plus(xj, d, A), A))
        for a in range(NRES):
            J[a, k] = (cols[0][a] - cols[1][a]) / (2 * h)
    return J


def _arr(v, A):
    return np.array(v, dtype=object if isinstance(A, Exact) else float)


def normal_equations(W, J, r, A):
    """H = J^T W J, g = J^T W r, cost = 1/2 r^T W r, with W's three blocks and diagonal tail multiplied separately."""
    WJ, Wr = A.zeros(NRES, NVAR), _arr([A.num(0)] * NRES, A)
    for b0, b1 in ((0, 15), (15, 30)):
        WJ[b0:b1] = W[b0:b1, b0:b1].dot(J[b0:b1])
        Wr[b0:b1] = W[b0:b1, b0:b1].dot(r[b0:b1])
    for a in range(30, NRES):
        WJ[a] = W[a, a] * J[a]
        Wr[a] = W[a, a] * r[a]
    return J.T.dot(WJ), J.T.dot(Wr), r.dot(Wr) / 2


def cholesky_solve(H, rhs, A):
    """H^-1 rhs (rhs a vector or a matrix), or None when H is not positive definite."""
    if isinstance(A, Exact):
        M = A.ctx.matrix(H.tolist())
        R = rhs if rhs.ndim == 2 else rhs.reshape(-1, 1)
        out = A.zeros(R.shape[0], R.shape[1])
        for c in range(R.shape[1]):
            try:
                x = A.ctx.cholesky_solve(M, A.ctx.matrix(R[:, c].tolist()))
            except ValueError:   # mpmath's Cholesky: a pivot is not > 0
                return None
            for a in range(R.shape[0]):
                out[a, c] = x[a]
        return out if rhs.ndim == 2 else out[:, 0]
    try:
        L = np.linalg.cholesky(H)
    except np.linalg.LinAlgError:
        return None
    return np.linalg.solve(L.T, np.linalg.solve(L, rhs))


def evaluate(p, xi, xj, A=FP64):
    """r (38), J (38 x 30), W (38 x 38) at the given float states, or None for W when Sigma is not positive definite."""
    m = _Interval(p["pre"], A)
    xi, xj = [A.num(v) for v in xi], [A.num(v) for v in xj]
    return _arr(residuals(p, m, xi, xj, A), A), jacobian(p, m, xi, xj, A), weights(p, m, A)


def solve(p, A=FP64):
    """The whole window update. -> dict: xi, xj, information (floats), initial_cost, final_cost, iterations, termination,
    num_evaluations, steps (the step norms), H (the final normal matrix, floats), kappa_H, kappa_Hii, kappa_sigma."""
    m = _Interval(p["pre"], A)
    W = weights(p, m, A)
    out = dict(termination=2, iterations=0, num_evaluations=1, steps=[], kappa_sigma=_cond(p["pre"].P))
    if W is None:
        return out
    xi = [A.num(v) for v in p["mean_i"]]
    xj = [A.num(v) for v in p["initial_j"]] if p["initial_j"] is not None else ir.predict(p["mean_i"], m, p["G"])
    max_iter = p["max_iter"] if p["max_iter"] > 0 else 10
    it, converged = 0, False
    while True:
        r = _arr(residuals(p, m, xi, xj, A), A)
        H, g, cost = normal_equations(W, jacobian(p, m, xi, xj, A), r, A)
        if it == 0:
            out["initial_cost"] = float(cost)
        if converged or it >= max_iter:
            break
        d = cholesky_solve(H, -g, A)
        if d is None:
            out.update(iterations=it, num_evaluations=it + 1)
            return out
        xi, xj = ir.plus(xi, d[:15], A), ir.plus(xj, d[15:], A)
        it += 1
        step = A.sqrt(sum(v * v for v in d))
        out["steps"].append(float(step))
        converged = step < CONVERGED
    X = cholesky_solve(H[:15, :15], H[:15, 15:], A)
    if X is None:
        out.update(iterations=it, num_evaluations=it + 1)
        return out
    info = H[15:, 15:] - H[15:, :15].dot(X)
    Hf = ir.to_float(H)
    out.update(xi=ir.to_float(xi), xj=ir.to_float(xj), information=ir.to_float(info), final_cost=float(cost), iterations=it,
               termination=0 if converged else 1, num_evaluations=it + 1, H=Hf, kappa_H=_cond(Hf), kappa_Hii=_cond(Hf[:15, :15]),
               exact=dict(H=H, info=info) if isinstance(A, Exact) else None)
    return out


def _cond(M):
    M = np.asarray(M, float)
    w = np.linalg.eigvalsh(0.5 * (M + M.T))
    return float(np.abs(w).max() / np.abs(w).min()) if np.abs(w).min() > 0 else math.inf


def minus(x, y):
    """x (-) y for 16-vectors (floats): 15 tangent components, the rotation by _log."""
    x, y = np.asarray(x, float), np.asarray(y, float)
    d = np.zeros(15)
    d[0:3] = x[0:3] - y[0:3]
    d[3:6] = _log(qmul(tuple(x[3:7]), conj(tuple(y[3:7] / np.linalg.norm(y[3:7])))), FP64)
    d[6:15] = x[7:16] - y[7:16]
    return d
