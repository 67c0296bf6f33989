"""Reference model of the real-time correlative scan matcher (test infrastructure), restated in numpy from the reference's
semantics (SM = C/mapping/internal/3d/scan_matching/, C/ = cartographer/cartographer/):
  Match                       SM/real_time_correlative_scan_matcher_3d.cc:34-53  every candidate scored; the best is kept with a
                                                                                 strict '>' from -1 in emplace order
  GenerateExhaustiveSearchTransforms  :55-95  linear window RoundToInt(double window / float resolution); max_scan_range the
                              farthest point (Eigen's norm sqrt(x*x + (y*y + z*z))), floored at 3 * resolution; angular step
                              kSafetyMargin * acosf(1.f - res * res / (2.f * (max_scan_range * max_scan_range))) in float,
                              kSafetyMargin = 1.f - 1e-3f; angular window RoundToInt(double window / float step); candidates
                              emplaced in the order z, y, x, rz, ry, rx
  AngleAxisVectorToRotationQuaternion<float>  C/transform/transform.h:85-99  squared norm compared with the double cutoff 1e-8;
                              above it sin(n / 2.) / n and cos(n / 2.) in double, narrowed to float; below, scale 0.5, w = 1
  ScoreCandidate              :97-113  initial.cast<float>() * transform (Rigid3f product, rotation renormalised); every point
                              transformed (Eigen's q * v), GetCellIndex by float division and lround, the probabilities added
                              in float strictly in point order; / float(n); then
                              score *= exp(-Pow2(norm(t) * w_t + GetAngle(transform) * w_r)): the float terms promote to
                              double, exp in double, the product narrowed to float on assignment
  GetAngle                    C/transform/transform.h:33-37  2.f * atan2f(norm(q.vec()), |q.w|)
The probability table, RoundToInt of float values, GetCellIndex and q * v are those of range_data_inserter_reference; the
quaternion product and normalisation those of fcsm_reference.

Every transcendental the reference takes from libm (acosf, atan2f, sin, cos, exp) and the lround of the two windows are called
through ctypes on glibc's libm, so this module computes what the reference binary computes on glibc x86-64, not what numpy's
own SIMD routines give (they can differ by an ulp). In particular a farthest point at or beyond about 4096 resolutions makes
the float argument of acosf exactly 1 (the "cliff"): the step is 0, the quotient +inf, and glibc's lround(+inf) is LONG_MIN,
whose low 32 bits (RoundToInt's cast to int) are 0: one rotation, A = 0.

The reference CHECK-fails when the best score is not positive (:111). Here, as on the device, a score of 0 (the penalty
underflowed) never wins: best_index is the first index of the largest positive score, and -1 when there is none.

The device's exp is not glibc's. ambiguous() flags the candidates whose float score would change if exp moved by one double
ulp either way; those are the only scores that cannot be demanded bit for bit.
"""
import ctypes
from dataclasses import dataclass, field

import numpy as np

from fcsm_reference import SparseGrid, normalized, qmul
from range_data_inserter_reference import cell_index, rotate, round_to_int, value_to_probability

f32 = np.float32
RES_FLOOR = f32(3.0)
K_SAFETY = f32(1.0) - f32(1e-3)
PROBABILITY = value_to_probability(np.arange(32768))     # every uint16 value (marker ignored) -> its probability

_libm = ctypes.CDLL("libm.so.6")
for _name, _res, _args in (("acosf", ctypes.c_float, [ctypes.c_float]), ("atan2f", ctypes.c_float, [ctypes.c_float] * 2),
                           ("sin", ctypes.c_double, [ctypes.c_double]), ("cos", ctypes.c_double, [ctypes.c_double]),
                           ("exp", ctypes.c_double, [ctypes.c_double]), ("lround", ctypes.c_long, [ctypes.c_double]),
                           ("nextafter", ctypes.c_double, [ctypes.c_double] * 2)):
    getattr(_libm, _name).restype = _res
    getattr(_libm, _name).argtypes = _args


def acosf(x):
    return f32(_libm.acosf(float(x)))


def atan2f(y, x):
    return f32(_libm.atan2f(float(y), float(x)))


def libm_exp(x):
    return _libm.exp(float(x))


def round_to_int_double(q):
    """RoundToInt(double): glibc's lround, then the cast to int (low 32 bits)."""
    return ctypes.c_int32(_libm.lround(float(q))).value


def norm(v):
    """Eigen's norm of float32 3-vectors (rows): sqrt(x*x + (y*y + z*z))."""
    v = np.asarray(v, f32).reshape(-1, 3)
    x, y, z = v[:, 0], v[:, 1], v[:, 2]
    return np.sqrt(x * x + (y * y + z * z))


# ----------------------------------------------------------------------------------------------- window
@dataclass
class Window:
    linear: int              # L of the reference: translations -L..L per axis
    angular: int             # A: rotations -A..A per axis
    step: np.float32         # angular step (radians)
    max_scan_range: np.float32

    @property
    def num_translations(self):
        return (2 * self.linear + 1) ** 3

    @property
    def num_rotations(self):
        return (2 * self.angular + 1) ** 3


def max_scan_range(points, resolution):
    m = RES_FLOOR * f32(resolution)
    if len(points):
        m = max(m, norm(points).max())
    return f32(m)


def angular_step(resolution, max_range):
    r, m = f32(resolution), f32(max_range)
    return K_SAFETY * acosf(f32(1.0) - (r * r) / (f32(2.0) * (m * m)))


def window(points, resolution, linear_window, angular_window):
    r = f32(resolution)
    m = max_scan_range(points, r)
    step = angular_step(r, m)
    with np.errstate(divide="ignore", invalid="ignore"):
        a = np.float64(angular_window) / np.float64(step)
    return Window(round_to_int_double(np.float64(linear_window) / np.float64(r)), round_to_int_double(a), step, m)


# ----------------------------------------------------------------------------------------------- candidates
def angle_axis_to_quat(aa):
    x, y, z = (f32(c) for c in aa)
    sq = x * x + (y * y + z * z)
    s, w = f32(0.5), f32(1.0)
    if np.float64(sq) > 1e-8:
        n = np.float64(np.sqrt(sq))
        s = f32(_libm.sin(n / 2.0) / n)
        w = f32(_libm.cos(n / 2.0))
    return np.array([w, s * x, s * y, s * z], f32)


def rotation_angle(q):
    return f32(2.0) * atan2f(norm(q[1:])[0], abs(q[0]))


def float_pose(pose7):
    p = np.asarray(pose7, np.float64).reshape(7)
    return p[:3].astype(f32), p[3:].astype(f32)


@dataclass
class Candidates:
    """The outer product the reference emplaces: candidate l * R + r = translation l (z, y, x order) with rotation r (rz, ry,
    rx order). cand_* are initial * transform; pen_* the double penalty terms of the transform alone."""
    cand_q: np.ndarray       # [R, 4] float32
    cand_t: np.ndarray       # [L, 3] float32
    pen_r: np.ndarray        # [R] float64: GetAngle * w_r
    pen_t: np.ndarray        # [L] float64: norm * w_t


def candidates(win, resolution, initial_pose, w_t, w_r):
    t0, q0 = float_pose(initial_pose)
    r = f32(resolution)
    A, L = win.angular, win.linear
    qs, pr = [], []
    for rz in range(-A, A + 1):
        for ry in range(-A, A + 1):
            for rx in range(-A, A + 1):
                q = angle_axis_to_quat((f32(rx) * win.step, f32(ry) * win.step, f32(rz) * win.step))
                qs.append(normalized(qmul(q0, q)))
                pr.append(np.float64(rotation_angle(q)) * w_r)
    ax = np.arange(-L, L + 1)
    zyx = np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3)
    off = (zyx[:, ::-1].astype(f32) * r).astype(f32)            # (x, y, z) * resolution
    ts = rotate(q0, off) + t0
    pt = norm(off).astype(np.float64) * w_t
    return Candidates(np.array(qs, f32).reshape(-1, 4), ts.astype(f32), np.array(pr, np.float64), pt)


def rotate_many(q, v):
    """rotate() of every row of v by every quaternion of q: [R, n, 3], the same float32 operations."""
    w = q[:, None, 0:1]
    qv = np.broadcast_to(q[:, None, 1:], (len(q), len(v), 3))
    vv = np.broadcast_to(v[None], qv.shape)

    def cross(a, b):
        return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1],
                         a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                         a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], axis=-1)

    uv = cross(qv, vv)
    uv = uv + uv
    return (vv + w * uv) + cross(qv, uv)


# ----------------------------------------------------------------------------------------------- grid lookup
class DenseLookup:
    """uint16 value of any cell of a SparseGrid, through a dense box over its cells (0 outside, as the grid reads)."""

    MAX_CELLS = 1 << 27

    def __init__(self, grid):
        cells = grid.cells
        if len(cells) == 0:
            self.lo, self.dim, self.values = np.zeros(3, np.int64), np.zeros(3, np.int64), np.zeros(1, np.uint16)
            return
        self.lo = cells.min(axis=0)
        self.dim = cells.max(axis=0) - self.lo + 1
        assert int(np.prod(self.dim)) <= self.MAX_CELLS, "grid box too large for the dense lookup"
        self.values = np.zeros(int(np.prod(self.dim)) + 1, np.uint16)      # the last entry stands for every absent cell
        self.values[self._flat(cells)] = grid.values

    def _flat(self, c):
        c = c - self.lo
        return (c[..., 0] * self.dim[1] + c[..., 1]) * self.dim[2] + c[..., 2]

    def __call__(self, cells):
        c = np.asarray(cells, np.int64)
        inside = ((c >= self.lo) & (c < self.lo + self.dim)).all(axis=-1)
        flat = np.where(inside, self._flat(np.where(inside[..., None], c, self.lo)), len(self.values) - 1)
        return self.values[flat]


# ----------------------------------------------------------------------------------------------- the match
@dataclass
class Result:
    window: Window
    scores: np.ndarray               # [K] float32, candidate order
    best_index: int                  # -1: no positive score
    score: np.float32
    pose: np.ndarray                 # float64 [7]: the best candidate's float pose, cast
    raw: np.ndarray = field(repr=False)     # [K] float64: the sum / n, promoted (before the penalty)
    exponent: np.ndarray = field(repr=False)  # [K] float64: -(a * a)
    cands: Candidates = field(repr=False, default=None)

    @property
    def num_candidates(self):
        return len(self.scores)

    def ambiguous(self):
        """Candidates whose score changes if exp moves by one double ulp."""
        uniq, inv = np.unique(self.exponent, return_inverse=True)
        e = np.array([libm_exp(x) for x in uniq])[inv]
        up = np.array([_libm.nextafter(x, np.inf) for x in e])
        down = np.array([_libm.nextafter(x, -np.inf) for x in e])
        now = (self.raw * e).astype(f32)
        return ((self.raw * up).astype(f32) != now) | ((self.raw * down).astype(f32) != now)

    def tied(self):
        """Every index with the best score."""
        if self.best_index < 0:
            return np.zeros(0, np.int64)
        return np.flatnonzero(self.scores == self.score)


def point_sums(grid, points, cands, resolution, lookup=None):
    """The float32 sum of every candidate's probabilities, added in point order: [L * R] in candidate order."""
    pts = np.asarray(points, f32).reshape(-1, 3)
    lookup = lookup or DenseLookup(grid)
    r = f32(resolution)
    R, L = len(cands.cand_q), len(cands.cand_t)
    total = np.zeros(L * R, f32)
    chunk = max(1, (1 << 22) // max(1, L * R))
    for i0 in range(0, len(pts), chunk):
        rp = rotate_many(cands.cand_q, pts[i0:i0 + chunk])                  # [R, m, 3]
        w = rp[None] + cands.cand_t[:, None, None, :]                          # [L, R, m, 3]
        prob = PROBABILITY[lookup(cell_index(w.reshape(-1, 3), r).reshape(w.shape)) & 0x7FFF]    # [L, R, m]
        prob = prob.reshape(L * R, -1)
        for j in range(prob.shape[1]):
            total += prob[:, j]
    return total


def match(grid, points, initial_pose, linear_window, angular_window, w_t, w_r, lookup=None):
    """RealTimeCorrelativeScanMatcher3D::Match on a SparseGrid -> Result."""
    pts = np.asarray(points, f32).reshape(-1, 3)
    assert len(pts) > 0
    r = grid.resolution
    win = window(pts, r, linear_window, angular_window)
    cands = candidates(win, r, initial_pose, w_t, w_r)
    raw = (point_sums(grid, pts, cands, r, lookup) / f32(len(pts))).astype(np.float64)
    a = (cands.pen_t[:, None] + cands.pen_r[None, :]).reshape(-1)
    exponent = -(a * a)
    uniq, inv = np.unique(exponent, return_inverse=True)
    scores = (raw * np.array([libm_exp(x) for x in uniq])[inv]).astype(f32)
    best = int(np.argmax(scores)) if scores.max() > 0 else -1        # first index of the maximum: strict '>' in order
    pose = np.zeros(7)
    if best >= 0:
        l, rr = divmod(best, len(cands.cand_q))
        pose = np.concatenate([cands.cand_t[l], cands.cand_q[rr]]).astype(np.float64)
    return Result(win, scores, best, scores[best] if best >= 0 else f32(0), pose, raw, exponent, cands)
