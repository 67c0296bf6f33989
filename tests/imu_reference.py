"""Independent reference of the IMU row: the mid-point pre-integrator of integration_base.h (push_back :109-123,
midPointIntegration :156-236, propagate :238-265, noise layout :28-51), the prediction of LTB:188-199, the factor of the
fused solve in the submap frame with its information matrix, and the 15-dim residual of :267-301 with the first-order
bias correction of :283-290.

Two precisions:
- fp64 in the evaluation order the device states (DESIGN §2: Eigen's `q * v = (v + w uv) + q.vec x uv`, uv = 2 q.vec x v,
  4-term sums as (x² + y²) + (z² + w²); 3x3 products, the F / V entries and the 15x15 sums left to right). Scalars are
  Python floats and the 15x15 products are numpy elementwise operations one term at a time, so no FMA and no BLAS
  reordering can enter: every value is the correctly rounded result of the stated sequence of operations.
- mpmath at 50 digits (`Exact`): the same formulas without rounding, to bound the fp64 reference's error and to
  differentiate numerically.

Row / column order of the 15x15 matrices follows the F matrix code: p, theta, v, b_a, b_g. Quaternions are (w, x, y, z);
nav states are 16-vectors p(3) q(4) v(3) ba(3) bg(3)."""
import math

import mpmath
import numpy as np

G_DEFAULT = (0.0, 0.0, 9.8)
KAIST_NOISE = (3.99e-2, 1.56e-2, 6.4e-5, 3.6e-5)   # acc_n, gyr_n, acc_w, gyr_w: D/config/kaist.lua:38-43


class Arith:
    """Scalar arithmetic of one precision: fp64 (Python floats) or mpmath."""
    def num(self, x):
        return float(x)

    def sqrt(self, x):
        return math.sqrt(x)

    def zeros(self, r, c):
        return np.zeros((r, c))

    def eye(self, n):
        return np.eye(n)


class Exact(Arith):
    """mpmath at `dps` digits. Matrices are numpy object arrays of mpf."""
    def __init__(self, dps=50):
        self.ctx = mpmath.mp.clone()
        self.ctx.dps = dps

    def num(self, x):
        return self.ctx.mpf(x)

    def sqrt(self, x):
        return self.ctx.sqrt(x)

    def zeros(self, r, c):
        z = np.empty((r, c), dtype=object)
        z[...] = self.ctx.mpf(0)
        return z

    def eye(self, n):
        z = self.zeros(n, n)
        for i in range(n):
            z[i, i] = self.ctx.mpf(1)
        return z


FP64 = Arith()


# ------------------------------------------------------------------ 3-vectors and quaternions (tuples)
def vadd(a, b):
    return (a[0] + b[0], a[1] + b[1], a[2] + b[2])


def vsub(a, b):
    return (a[0] - b[0], a[1] - b[1], a[2] - b[2])


def vmul(s, a):
    return (s * a[0], s * a[1], s * a[2])


def cross(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def rotate(q, v):
    """Eigen's q * v: uv = 2 (q.vec x v); (v + w uv) + q.vec x uv."""
    qv = (q[1], q[2], q[3])
    uv = cross(qv, v)
    uv = (uv[0] + uv[0], uv[1] + uv[1], uv[2] + uv[2])
    c = cross(qv, uv)
    return ((v[0] + q[0] * uv[0]) + c[0], (v[1] + q[0] * uv[1]) + c[1], (v[2] + q[0] * uv[2]) + c[2])


def qmul(a, b):
    """Eigen's generic quaternion product, terms left to right."""
    return (a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3],
            a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
            a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3],
            a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1])


def conj(q):
    return (q[0], -q[1], -q[2], -q[3])


def squared_norm(q):
    """Eigen's 4-term redux over the coefficients (x, y, z, w): (x² + y²) + (z² + w²)."""
    return (q[1] * q[1] + q[2] * q[2]) + (q[3] * q[3] + q[0] * q[0])


def normalized(q, A=FP64):
    n = A.sqrt(squared_norm(q))
    return (q[0] / n, q[1] / n, q[2] / n, q[3] / n)


def rotation_matrix(q):
    """Eigen's Quaternion::toRotationMatrix (no normalisation)."""
    tx, ty, tz = 2 * q[1], 2 * q[2], 2 * q[3]
    twx, twy, twz = tx * q[0], ty * q[0], tz * q[0]
    txx, txy, txz = tx * q[1], ty * q[1], tz * q[1]
    tyy, tyz, tzz = ty * q[2], tz * q[2], tz * q[3]
    return [[1 - (tyy + tzz), txy - twz, txz + twy],
            [txy + twz, 1 - (txx + tzz), tyz - twx],
            [txz - twy, tyz + twx, 1 - (txx + tyy)]]


def skew(v):
    return [[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]]


def mul33(A, B):
    return [[A[i][0] * B[0][j] + A[i][1] * B[1][j] + A[i][2] * B[2][j] for j in range(3)] for i in range(3)]


# ------------------------------------------------------------------ pre-integration
class Preintegration:
    """IntegrationBase: linearisation biases, the deltas, the 15x15 Jacobian and covariance."""

    def __init__(self, noise4, ba, bg, A=FP64):
        self.A = A
        n = [A.num(x) for x in noise4]
        an, gn, aw, gw = n[0] * n[0], n[1] * n[1], n[2] * n[2], n[3] * n[3]
        self.nd = [an] * 3 + [gn] * 3 + [an] * 3 + [gn] * 3 + [aw] * 3 + [gw] * 3   # diagonal of `noise` (:36-51)
        self.ba = tuple(A.num(x) for x in ba)
        self.bg = tuple(A.num(x) for x in bg)
        self.sum_dt = A.num(0)
        zero, one = A.num(0), A.num(1)
        self.dp = (zero, zero, zero)
        self.dv = (zero, zero, zero)
        self.dq = (one, zero, zero, zero)
        self.J = A.eye(15)
        self.P = A.zeros(15, 15)
        self.latched = False
        self.acc_0 = self.gyr_0 = None

    def push_back(self, dt, acc, gyr):
        """The first sample only latches acc_0 / gyr_0 (:111-118); every later one is one propagate step."""
        A = self.A
        acc = tuple(A.num(x) for x in acc)
        gyr = tuple(A.num(x) for x in gyr)
        if not self.latched:
            self.latched = True
            self.acc_0, self.gyr_0 = acc, gyr
            return
        self.propagate(A.num(dt), acc, gyr)

    def propagate(self, dt, acc_1, gyr_1):
        A = self.A
        ba, bg, dq = self.ba, self.bg, self.dq
        a0 = vsub(self.acc_0, ba)
        a1 = vsub(acc_1, ba)
        # midPointIntegration, state (:162-171)
        un_acc_0 = rotate(dq, a0)
        un_gyr = vsub(vmul(0.5, vadd(self.gyr_0, gyr_1)), bg)
        rq = qmul(dq, (A.num(1), un_gyr[0] * dt / 2, un_gyr[1] * dt / 2, un_gyr[2] * dt / 2))
        un_acc_1 = rotate(rq, a1)
        un_acc = vmul(0.5, vadd(un_acc_0, un_acc_1))
        rp = vadd(vadd(self.dp, vmul(dt, self.dv)), vmul(0.5 * dt * dt, un_acc))
        rv = vadd(self.dv, vmul(dt, un_acc))
        # F (15x15) and V (15x18), entry by entry (:176-232)
        Rw, Ra0, Ra1 = skew(un_gyr), skew(a0), skew(a1)
        R0, R1 = rotation_matrix(dq), rotation_matrix(rq)
        IRw = [[(1.0 if i == j else 0.0) - Rw[i][j] * dt for j in range(3)] for i in range(3)]
        R0a0, R1a1 = mul33(R0, Ra0), mul33(R1, Ra1)
        R1a1I = mul33(R1a1, IRw)
        F, V = A.zeros(15, 15), A.zeros(15, 18)
        for i in range(3):
            for j in range(3):
                idn = A.num(1.0 if i == j else 0.0)
                F[i, j] = idn
                F[i, 3 + j] = -0.25 * R0a0[i][j] * dt * dt + -0.25 * R1a1I[i][j] * dt * dt
                F[i, 6 + j] = idn * dt
                F[i, 9 + j] = -0.25 * (R0[i][j] + R1[i][j]) * dt * dt
                F[i, 12 + j] = -0.25 * R1a1[i][j] * dt * dt * -dt
                F[3 + i, 3 + j] = IRw[i][j]
                F[3 + i, 12 + j] = -1.0 * idn * dt
                F[6 + i, 3 + j] = -0.5 * R0a0[i][j] * dt - 0.5 * R1a1I[i][j] * dt
                F[6 + i, 6 + j] = idn
                F[6 + i, 9 + j] = -0.5 * (R0[i][j] + R1[i][j]) * dt
                F[6 + i, 12 + j] = -0.5 * R1a1[i][j] * dt * -dt
                F[9 + i, 9 + j] = idn
                F[12 + i, 12 + j] = idn
                v03 = 0.25 * -R1a1[i][j] * dt * dt * 0.5 * dt
                v63 = 0.5 * -R1a1[i][j] * dt * 0.5 * dt
                V[i, j] = 0.25 * R0[i][j] * dt * dt
                V[i, 3 + j] = v03
                V[i, 6 + j] = 0.25 * R1[i][j] * dt * dt
                V[i, 9 + j] = v03
                V[3 + i, 3 + j] = 0.5 * idn * dt
                V[3 + i, 9 + j] = 0.5 * idn * dt
                V[6 + i, j] = 0.5 * R0[i][j] * dt
                V[6 + i, 3 + j] = v63
                V[6 + i, 6 + j] = 0.5 * R1[i][j] * dt
                V[6 + i, 9 + j] = v63
                V[9 + i, 12 + j] = idn * dt
                V[12 + i, 15 + j] = idn * dt
        # propagate: J <- F J, P <- (F P) F^T + (V N) V^T, every sum over c in increasing order from 0
        self.J = _mm(F, self.J, A)
        T = _mm(F, self.P, A)
        a = A.zeros(15, 15)
        for c in range(15):
            a = a + T[:, c:c + 1] * F[:, c][None, :]
        b = A.zeros(15, 15)
        for c in range(18):
            b = b + (V[:, c:c + 1] * self.nd[c]) * V[:, c][None, :]
        self.P = a + b
        self.dp, self.dv = rp, rv
        self.dq = normalized(rq, A)
        self.sum_dt = self.sum_dt + dt
        self.acc_0, self.gyr_0 = acc_1, gyr_1


def _mm(X, Y, A):
    s = A.zeros(X.shape[0], Y.shape[1])
    for c in range(X.shape[1]):
        s = s + X[:, c:c + 1] * Y[c:c + 1, :]
    return s


def preintegrate(noise4, ba, bg, dt, acc, gyr, A=FP64):
    m = Preintegration(noise4, ba, bg, A)
    for k in range(len(dt)):
        m.push_back(dt[k], acc[k], gyr[k])
    return m


# ------------------------------------------------------------------ prediction, frames, factor
def unpack(x, A=FP64):
    x = [A.num(v) for v in x]
    return tuple(x[0:3]), tuple(x[3:7]), tuple(x[7:10]), tuple(x[10:13]), tuple(x[13:16])


def predict(state_i, m, G=G_DEFAULT):
    """dl_imu_predict (LTB:188-199): p + T v - 1/2 T² G + q dp, v - T G + q dv, normalised q dq; biases copied."""
    A = m.A
    p, q, v, ba, bg = unpack(state_i, A)
    G = tuple(A.num(g) for g in G)
    T = m.sum_dt
    pj = vadd(vsub(vadd(p, vmul(T, v)), vmul(0.5 * T * T, G)), rotate(q, m.dp))
    vj = vadd(vsub(v, vmul(T, G)), rotate(q, m.dv))
    qj = normalized(qmul(q, m.dq), A)
    return list(pj) + list(qj) + list(vj) + list(ba) + list(bg)


def compose(l, r, A=FP64):
    """Rigid3 * Rigid3 (rigid_transform.h:206-212): (l.q r.t + l.t, normalised l.q r.q)."""
    return vadd(rotate(l[1], r[0]), l[0]), normalized(qmul(l[1], r[1]), A)


def inverse(r):
    qi = conj(r[1])
    t = rotate(qi, r[0])
    return (-t[0], -t[1], -t[2]), qi


def information(cov, weight, A=FP64):
    """W = weight² Sigma^-1: Cholesky row by row (Sigma = L L^T), L^-1 column by column, then
    W_ab = weight² sum_{k >= max(a, b)} Li_ka Li_kb. None if Sigma is not positive definite (a pivot is not > 0)."""
    S = [[A.num(cov[i][j]) for j in range(15)] for i in range(15)]
    L = [[A.num(0)] * 15 for _ in range(15)]
    for i in range(15):
        for j in range(i + 1):
            s = S[i][j]
            for k in range(j):
                s = s - L[i][k] * L[j][k]
            if i == j:
                if not s > 0:
                    return None
                L[i][i] = A.sqrt(s)
            else:
                L[i][j] = s / L[j][j]
    Li = [[A.num(0)] * 15 for _ in range(15)]
    for c in range(15):
        for i in range(c, 15):
            s = A.num(1.0 if i == c else 0.0)
            for k in range(c, i):
                s = s - L[i][k] * Li[k][c]
            Li[i][c] = s / L[i][i]
    w = A.num(weight)
    W = A.zeros(15, 15)
    for a in range(15):
        for b in range(15):
            s = A.num(0)
            for k in range(max(a, b), 15):
                s = s + Li[k][a] * Li[k][b]
            W[a, b] = w * w * s
    return W


def corrected_deltas(m, ba_i, bg_i):
    """First-order bias correction (:283-290), sums left to right: dp + J_p,ba dba + J_p,bg dbg (likewise dv), and the
    inverse of corrected_delta_q = delta_q (1, 1/2 J_q,bg dbg) as Eigen's inverse(): conjugate / squared norm. At the
    linearisation biases the raw deltas and conj(delta_q)."""
    A = m.A
    dba = vsub(tuple(A.num(x) for x in ba_i), m.ba)
    dbg = vsub(tuple(A.num(x) for x in bg_i), m.bg)
    if all(x == 0 for x in dba + dbg):
        return m.dp, m.dv, conj(m.dq)
    J = m.J

    def blk(r, c, d):
        return tuple(J[r + i, c] * d[0] + J[r + i, c + 1] * d[1] + J[r + i, c + 2] * d[2] for i in range(3))
    dp = vadd(vadd(m.dp, blk(0, 9, dba)), blk(0, 12, dbg))
    dv = vadd(vadd(m.dv, blk(6, 9, dba)), blk(6, 12, dbg))
    th = blk(3, 12, dbg)
    c = qmul(m.dq, (A.num(1), 0.5 * th[0], 0.5 * th[1], 0.5 * th[2]))
    n2 = squared_norm(c)
    return dp, dv, (c[0] / n2, -c[1] / n2, -c[2] / n2, -c[3] / n2)


class Factor:
    """The IMU factor of the fused solve in the submap frame, as the device prepares it once per scan: state i composed
    with to_submap = submap_local_pose^-1, v and G rotated into the submap frame, the corrected deltas, and W."""

    def __init__(self, state_i, m, submap_local_pose, G=G_DEFAULT, imu_weight=1.0):
        A = m.A
        self.m, self.A = m, A
        p, q, v, ba, bg = unpack(state_i, A)
        sp = [A.num(x) for x in submap_local_pose]
        to_submap = inverse((tuple(sp[0:3]), tuple(sp[3:7])))
        self.predicted = predict(state_i, m, G)
        pj, qj, vj, _, _ = unpack(self.predicted, A)
        self.pi, self.qi = compose(to_submap, (p, q), A)
        pose_j = compose(to_submap, (pj, qj), A)
        self.vi = rotate(to_submap[1], v)
        self.G = rotate(to_submap[1], tuple(A.num(g) for g in G))
        self.bai, self.bgi = ba, bg
        self.dp, self.dv, self.dq_inv = corrected_deltas(m, ba, bg)
        self.x16 = list(pose_j[0]) + list(pose_j[1]) + list(rotate(to_submap[1], vj)) + list(ba) + list(bg)
        self.W = information(m.P, imu_weight, A)

    def residual(self, x16):
        """r (15) of :292-299 at x16 = state j in the submap frame."""
        A = self.A
        pj, qj, vj, baj, bgj = unpack(x16, A)
        T = self.m.sum_dt
        qi_inv = conj(self.qi)
        rp = vsub(rotate(qi_inv, vsub(vsub(vadd(vmul(0.5 * T * T, self.G), pj), self.pi), vmul(T, self.vi))), self.dp)
        rv = vsub(rotate(qi_inv, vsub(vadd(vmul(T, self.G), vj), self.vi)), self.dv)
        e = qmul(qmul(self.dq_inv, qi_inv), qj)
        return (list(rp) + [2 * e[1], 2 * e[2], 2 * e[3]] + list(rv) + list(vsub(baj, self.bai)) + list(vsub(bgj, self.bgi)))

    def jacobian(self, x16):
        """d r / d delta in the chart of dl_fused_match_batch: p += d[0:3]; q <- (cos|d|, sin|d|/|d| d) (x) q with
        d = delta[3:6]; v, ba, bg += delta[6:15]. Only the three 3x3 blocks are not constant."""
        A = self.A
        _, qj, _, _, _ = unpack(x16, A)
        qi_inv = conj(self.qi)
        Aq = qmul(self.dq_inv, qi_inv)
        J = A.zeros(15, 15)
        zero, one = A.num(0), A.num(1)
        for b in range(3):
            e = tuple(one if k == b else zero for k in range(3))
            col = rotate(qi_inv, e)
            c = qmul(qmul(Aq, (zero,) + e), qj)
            for a in range(3):
                J[a, b] = col[a]
                J[6 + a, 6 + b] = col[a]
                J[3 + a, 3 + b] = 2 * c[1 + a]
        for a in range(9, 15):
            J[a, a] = one
        return J

    def normal_equations(self, x16):
        """H = J^T W J, g = J^T W r, cost2 = r^T W r (sums in index order)."""
        A = self.A
        r = np.array(self.residual(x16), dtype=object if isinstance(A, Exact) else float)
        J = self.jacobian(x16)
        WJ = _mm(self.W, J, A)
        H = _mm(J.T.copy(), WJ, A)
        Wr = _mm(self.W, r.reshape(15, 1), A)[:, 0]
        g = _mm(J.T.copy(), Wr.reshape(15, 1), A)[:, 0]
        cost2 = A.num(0)
        for c in range(15):
            cost2 = cost2 + r[c] * Wr[c]
        return r, H, g, cost2


def plus(x16, delta, A):
    """The solve's chart: q <- (cos|d|, sin|d|/|d| d) (x) q, everything else additive."""
    x = [A.num(v) for v in x16]
    d = [A.num(v) for v in delta]
    y = list(x)
    for k in range(3):
        y[k] = x[k] + d[k]
    n = A.sqrt(d[3] * d[3] + d[4] * d[4] + d[5] * d[5])
    if n == 0:
        dq = (A.num(1), d[3], d[4], d[5])
    else:
        ctx = A.ctx if isinstance(A, Exact) else math
        s = ctx.sin(n) / n
        dq = (ctx.cos(n), s * d[3], s * d[4], s * d[5])
    y[3:7] = list(qmul(dq, tuple(x[3:7])))
    for k in range(9):
        y[7 + k] = x[7 + k] + d[6 + k]
    return y


def to_float(M):
    return np.array(M, dtype=float)
