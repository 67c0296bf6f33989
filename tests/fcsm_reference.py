"""Reference model of the loop-closure coarse matcher (test infrastructure), restated in numpy from the reference's semantics
(SM = C/mapping/internal/3d/scan_matching/, C/ = cartographer/cartographer/):
  ConvertToPrecomputationGrid  SM/precomputation_grid_3d.cc:49-61  RoundToInt((ValueToProbability(v) - 0.1f) * (255.f / (0.9f - 0.1f)))
  PrecomputeGrid               SM/precomputation_grid_3d.cc:63-81  max over the 8 cells c - shift * octant, halved (>> 1) at
                                                                    half resolution
  PrecomputationGridStack3D    SM/fast_correlative_scan_matcher_3d.cc:57-77
  MatchWith3DofInitial         :165-196  window half-widths RoundToInt(double window / float resolution); one discrete scan
  DiscretizeScan               :252-295  GetCellIndex(pose * p) with the float pose as given (not normalised)
  ScoreCandidates              :384-407  ToProbability(sum / float(n)) = 0.1f + (float(sum) / float(n)) * ((0.9f - 0.1f) / 255.f)
  GetPoseFromCandidate         :421-427  Translation(resolution * offset) * pose; Rigid3f composition normalises the rotation
  BranchAndBound               :429-492
  low-resolution matcher       SM/low_resolution_matcher.cc:23-35  float sum of GetProbability(GetCellIndex(pose * p)) in point
                                                                    order, / float(size), compared >= with the double option
The probability table, RoundToInt and GetCellIndex are those of range_data_inserter_reference.

match_3dof scores the whole window at once: every point is paired with every occupied cell within the window's reach and the
pairs are added into a dense integer window volume, so windows of tens of millions of leaves stay cheap. The answer is the leaf
with the highest score strictly above min_score that passes the low-resolution gate; among equal scores the lowest linear
index (z, y, x) wins. That is the device's documented tie rule: the reference's order among equal scores comes from an
unstable std::sort. The gate is evaluated lazily, in that order, until a leaf passes, as the reference's leaf level does.

PrecomputationStack and branch_and_bound are a literal restatement of the reference's search (dict grids, recursion), for CPU
tests of its admissibility on small inputs only.
"""
from dataclasses import dataclass, field

import numpy as np

import range_data_inserter_reference as rdi
from range_data_inserter_reference import cell_index, round_to_int, value_to_probability

f32 = np.float32
K_MIN, K_MAX = rdi.K_MIN, rdi.K_MAX
STEP = (K_MAX - K_MIN) / f32(255.0)       # PrecomputationGrid3D::ToProbability's scale
IDENTITY = np.array([1.0, 0.0, 0.0, 0.0], f32)


def precomputation_value(values):
    """ConvertToPrecomputationGrid's 8-bit value of uint16 cell values (the update marker ignored). int64."""
    return round_to_int((value_to_probability(values) - K_MIN) * (f32(255.0) / (K_MAX - K_MIN)))


LUT = precomputation_value(np.arange(32768))    # every cell value -> its 8-bit value


def to_probability(sums, n):
    """ToProbability(sum / float(n)) of integer sums: float32."""
    return K_MIN + (np.asarray(sums).astype(f32) / f32(n)) * STEP


def lround_double(q):
    """std::lround of one double (exact: q - floor(q) is exact for |q| < 2^52)."""
    fl = np.floor(q)
    r = int(fl) + int(q - fl >= 0.5)
    return r if q >= 0 else -lround_double(-q)


def window(xy_window, z_window, resolution):
    """(wxy, wz): RoundToInt(double window / float resolution)."""
    r = float(f32(resolution))
    return lround_double(xy_window / r), lround_double(z_window / r)


class SparseGrid:
    """A HybridGrid's content: occupied cells (int [n, 3], inside +-8192) and their uint16 values."""

    def __init__(self, resolution, cells=None, values=None):
        self.resolution = f32(resolution)
        cells = np.zeros((0, 3), np.int64) if cells is None else np.asarray(cells, np.int64).reshape(-1, 3)
        values = np.zeros(0, np.uint16) if values is None else np.asarray(values, np.uint16).reshape(-1)
        assert rdi.in_range(cells) and len(cells) == len(values)
        keys = self._key(cells)
        keys, last = np.unique(keys[::-1], return_index=True)       # the last write of a cell wins
        self.keys, self.values = keys, values[::-1][last]
        self.cells = cells[::-1][last]

    @staticmethod
    def _key(cells):
        c = np.asarray(cells, np.int64) + rdi.LIMIT
        return (c[:, 0] << 28) | (c[:, 1] << 14) | c[:, 2]

    @classmethod
    def from_export(cls, resolution, exported):
        xs, ys, zs, vs = exported
        return cls(resolution, np.stack([xs, ys, zs], axis=1), vs)

    def export(self):
        """(x, y, z, value) arrays for dl_grid_set_cells / the oracle's set_cells."""
        c = self.cells.astype(np.int32)
        return c[:, 0].copy(), c[:, 1].copy(), c[:, 2].copy(), self.values.copy()

    def lookup(self, cells):
        """uint16 value of every cell (0 where never written or outside +-8192)."""
        cells = np.asarray(cells, np.int64).reshape(-1, 3)
        inside = ((cells >= -rdi.LIMIT) & (cells < rdi.LIMIT)).all(axis=1)
        keys = self._key(np.where(inside[:, None], cells, 0))
        if len(self.keys) == 0:
            return np.zeros(len(cells), np.uint16)
        pos = np.minimum(np.searchsorted(self.keys, keys), len(self.keys) - 1)
        return np.where(inside & (self.keys[pos] == keys), self.values[pos], 0).astype(np.uint16)

    def v8(self):
        """(cells, 8-bit values) of the cells whose 8-bit value is non-zero."""
        v = LUT[self.values & 0x7FFF]
        keep = v > 0
        return self.cells[keep], v[keep]


# ----------------------------------------------------------------------------------------------- poses
def float_pose(pose7):
    p = np.asarray(pose7, np.float64).reshape(7)
    return p[:3].astype(f32), p[3:].astype(f32)


def transform(points, t, q):
    return rdi.rotate(q, np.asarray(points, f32).reshape(-1, 3)) + t


def discretize(points, pose7, resolution):
    """DiscretizeScan's full-resolution cells: int64 [n, 3]."""
    t, q = float_pose(pose7)
    return cell_index(transform(points, t, q), resolution)


def qmul(a, b):
    return np.array([((a[0] * b[0] - a[1] * b[1]) - a[2] * b[2]) - a[3] * b[3],
                     ((a[0] * b[1] + a[1] * b[0]) + a[2] * b[3]) - a[3] * b[2],
                     ((a[0] * b[2] + a[2] * b[0]) + a[3] * b[1]) - a[1] * b[3],
                     ((a[0] * b[3] + a[3] * b[0]) + a[1] * b[2]) - a[2] * b[1]], f32)


def normalized(q):
    n = np.sqrt((q[1] * q[1] + q[2] * q[2]) + (q[3] * q[3] + q[0] * q[0]))
    return (q / n).astype(f32)


def candidate_pose(pose7, resolution, offset):
    """GetPoseFromCandidate -> (t float32[3], q float32[4])."""
    t, q = float_pose(pose7)
    shift = f32(resolution) * np.asarray(offset, np.int64).astype(f32)
    return rdi.rotate(IDENTITY, t[None])[0] + shift, normalized(qmul(IDENTITY, q))


def pose7_of(t, q):
    """The float pose widened to double, as the result reports it."""
    return np.concatenate([t, q]).astype(np.float64)


def low_resolution_score(lo, lo_points, t, q):
    """The low-resolution matcher at pose (t, q): float32."""
    cells = cell_index(transform(lo_points, t, q), lo.resolution)
    probs = value_to_probability(lo.lookup(cells))
    return f32(np.add.accumulate(probs, dtype=f32)[-1] / f32(len(probs)))


# ----------------------------------------------------------------------------------------------- the whole window
def window_sums(hi, cells, wxy, wz):
    """Integer correlation sum of every leaf: int32 [2 wz + 1, 2 wxy + 1, 2 wxy + 1] (z, y, x), offsets from -w."""
    side, depth = 2 * wxy + 1, 2 * wz + 1
    sums = np.zeros(depth * side * side, np.int32)
    occ, val = hi.v8()
    order = np.argsort(occ[:, 0], kind="stable")
    occ, val = occ[order], val[order]
    points, count = np.unique(np.asarray(cells, np.int64).reshape(-1, 3), axis=0, return_counts=True)
    idx, add = [], []
    for c, k in zip(points, count):
        a, b = np.searchsorted(occ[:, 0], c[0] - wxy, "left"), np.searchsorted(occ[:, 0], c[0] + wxy, "right")
        o = occ[a:b] - c
        keep = (np.abs(o[:, 1]) <= wxy) & (np.abs(o[:, 2]) <= wz)
        o = o[keep]
        idx.append(((o[:, 2] + wz) * side + (o[:, 1] + wxy)) * side + (o[:, 0] + wxy))
        add.append(val[a:b][keep] * k)
    if idx:
        np.add.at(sums, np.concatenate(idx), np.concatenate(add).astype(np.int32))
    return sums.reshape(depth, side, side)


@dataclass
class Match:
    found: bool
    score: float = 0.0
    offset: tuple = (0, 0, 0)
    pose: np.ndarray = None
    low_resolution_score: float = 0.0
    num_candidates: int = 0
    wxy: int = 0
    wz: int = 0
    scores: np.ndarray = None                     # every leaf, (z, y, x)
    rejected: list = field(default_factory=list)  # linear indices the gate turned down before the answer, in order
    tied: list = field(default_factory=list)      # linear indices of every leaf that shares the answer's score and passes

    def offset_of(self, index):
        side = 2 * self.wxy + 1
        return (index % side - self.wxy, (index // side) % side - self.wxy, index // (side * side) - self.wz)

    def index_of(self, offset):
        side = 2 * self.wxy + 1
        return ((offset[2] + self.wz) * side + (offset[1] + self.wxy)) * side + (offset[0] + self.wxy)


def match_3dof(hi, lo, hi_points, lo_points, pose7, min_score, xy_window=5.0, z_window=1.0, min_low_resolution_score=0.55,
               all_ties=False):
    """MatchWith3DofInitial, scored exhaustively. all_ties: also list every passing leaf tied with the answer."""
    wxy, wz = window(xy_window, z_window, hi.resolution)
    cells = discretize(hi_points, pose7, hi.resolution)
    scores = to_probability(window_sums(hi, cells, wxy, wz), len(cells))
    m = Match(False, num_candidates=scores.size, wxy=wxy, wz=wz, scores=scores)
    flat = scores.reshape(-1)
    above = flat > f32(min_score)
    lo_points = np.asarray(lo_points, f32).reshape(-1, 3)

    def gate(index):
        t, q = candidate_pose(pose7, hi.resolution, m.offset_of(index))
        low = low_resolution_score(lo, lo_points, t, q)
        return float(low) >= float(min_low_resolution_score), low, t, q

    for level in np.unique(flat[above])[::-1]:
        for index in np.flatnonzero(flat == level):
            ok, low, t, q = gate(int(index))
            if not ok:
                m.rejected.append(int(index))
                continue
            m.found, m.score, m.offset = True, f32(level), m.offset_of(int(index))
            m.pose, m.low_resolution_score = pose7_of(t, q), low
            if all_ties:
                m.tied = [int(i) for i in np.flatnonzero(flat == level) if i >= index and gate(int(i))[0]]
            return m
    return m


# ----------------------------------------------------------------------------------------------- the reference's own search
def _half(v):
    return v >> 1        # DivideByTwoRoundingTowardsNegativeInfinity (arithmetic shift; Python's >> floors too)


def precompute_grid(grid, half_resolution, shift):
    out = {}
    for (x, y, z), v in grid.items():
        for i in range(8):
            c = (x - shift * (i & 1), y - shift * ((i >> 1) & 1), z - shift * ((i >> 2) & 1))
            if half_resolution:
                c = tuple(_half(a) for a in c)
            out[c] = max(v, out.get(c, 0))
    return out


class PrecomputationStack:
    """PrecomputationGridStack3D as dicts cell -> 8-bit value."""

    def __init__(self, hi, depth, full_depth):
        assert depth >= 1 and full_depth >= 1
        occ, val = hi.v8()
        self.grids = [{tuple(int(a) for a in c): int(v) for c, v in zip(occ, val)}]
        last_width = 1
        for d in range(1, depth):
            half_resolution = d >= full_depth
            next_width = 1 << d
            full_voxels = 1 << max(0, d - full_depth)
            shift = (next_width - last_width + (full_voxels - 1)) // full_voxels     # positive: C division
            self.grids.append(precompute_grid(self.grids[-1], half_resolution, shift))
            last_width = next_width

    @property
    def max_depth(self):
        return len(self.grids) - 1


@dataclass
class _Candidate:
    offset: tuple
    score: float = -np.inf
    low_resolution_score: float = 0.0


def branch_and_bound(hi, lo, hi_points, lo_points, pose7, min_score, xy_window=5.0, z_window=1.0, min_low_resolution_score=0.55,
                     depth=8, full_depth=3, stack=None):
    """The reference's MatchWith3DofInitial as written: -> (Match without scores, leaves scored)."""
    stack = stack or PrecomputationStack(hi, depth, full_depth)
    wxy, wz = window(xy_window, z_window, hi.resolution)
    full = [tuple(int(a) for a in c) for c in discretize(hi_points, pose7, hi.resolution)]
    full_d = min(full_depth, depth)
    per_depth = [full] * full_d
    start = (-wxy, -wxy, -wz)
    for i in range(depth - full_d):
        e = i + 1
        low_start = tuple(s >> e for s in start)
        per_depth.append([tuple(((c[a] + start[a]) >> e) - low_start[a] for a in range(3)) for c in full])
    lo_points = np.asarray(lo_points, f32).reshape(-1, 3)
    leaves = [0]

    def score(d, candidates):
        e = max(0, d - full_depth + 1)
        grid = stack.grids[d]
        for c in candidates:
            off = tuple(o >> e for o in c.offset)
            s = sum(grid.get((p[0] + off[0], p[1] + off[1], p[2] + off[2]), 0) for p in per_depth[d])
            c.score = f32(to_probability(s, len(per_depth[d])))
            leaves[0] += d == 0
        candidates.sort(key=lambda c: -c.score)

    def search(candidates, d, floor):
        if d == 0:
            for c in candidates:
                if c.score <= floor:
                    return _Candidate((0, 0, 0))
                t, q = candidate_pose(pose7, hi.resolution, c.offset)
                low = low_resolution_score(lo, lo_points, t, q)
                if float(low) >= float(min_low_resolution_score):
                    return _Candidate(c.offset, c.score, low)
            return _Candidate((0, 0, 0))
        best = _Candidate((0, 0, 0), floor)
        for c in candidates:
            if c.score <= floor:
                break
            higher = []
            half_width = 1 << (d - 1)
            for z in (0, half_width):
                if c.offset[2] + z > wz:
                    break
                for y in (0, half_width):
                    if c.offset[1] + y > wxy:
                        break
                    for x in (0, half_width):
                        if c.offset[0] + x > wxy:
                            break
                        higher.append(_Candidate((c.offset[0] + x, c.offset[1] + y, c.offset[2] + z)))
            score(d - 1, higher)
            sub = search(higher, d - 1, best.score)
            if best.score < sub.score:           # std::max keeps the first unless it is less
                best = sub
        return best

    step = 1 << stack.max_depth
    lowest = [_Candidate((x, y, z)) for z in range(-wz, wz + 1, step) for y in range(-wxy, wxy + 1, step)
              for x in range(-wxy, wxy + 1, step)]
    score(stack.max_depth, lowest)
    best = search(lowest, stack.max_depth, f32(min_score))
    side = 2 * wxy + 1
    m = Match(False, num_candidates=side * side * (2 * wz + 1), wxy=wxy, wz=wz)
    if best.score > f32(min_score):
        t, q = candidate_pose(pose7, hi.resolution, best.offset)
        m.found, m.score, m.offset, m.pose, m.low_resolution_score = True, f32(best.score), best.offset, pose7_of(t, q), \
            best.low_resolution_score
    return m, leaves[0]
