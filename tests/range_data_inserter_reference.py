"""Reference model of the range-data inserter (test infrastructure), restated in numpy from the reference's semantics
(C/ = cartographer/cartographer/, PV = C/mapping/probability_values.{h,cc}, RDI = C/mapping/3d/range_data_inserter_3d.cc,
HG = C/mapping/3d/hybrid_grid.h):
  ValueToProbability             PV.cc:27-37  value * kScale + (0.1f - kScale), kScale = (0.9f - 0.1f) / 32766.f; 0 -> 0.1f
  BoundedFloatToValue            PV.h:30-41   lround((clamp(p, 0.1f, 0.9f) - 0.1f) * (32766.f / (0.9f - 0.1f))) + 1
  Odds / ProbabilityFromOdds     PV.h:43-49   p / (1.f - p), o / (o + 1.f)
  ComputeLookupTableToApplyOdds  PV.cc:70-80  entry 0 from the odds alone, entry v from odds * Odds(ValueToProbability(v));
                                              every entry carries the update marker 32768. The options are doubles, Odds
                                              takes a float: the probability is rounded to float first.
  GetCellIndex                   HG:430-435   lround(float(x / resolution)) per axis
  RangeDataInserter3D::Insert    RDI:27-51, 76-92  every hit with the hit table, then for every ray the samples
                                              max(0, num_samples - num_free) .. num_samples - 1 at
                                              origin_cell + delta * position / num_samples (C++ truncating division) with the
                                              miss table; a cell is updated at most once per Insert (the update marker), so a
                                              hit wins over a miss. CHECK_LT(num_samples, 1 << 15) (RDI:37) and the grid's
                                              CHECK_LE(new_bits, 8) (HG:391) abort the reference; here they raise InsertError
                                              before the grid changes.
  Submap3D::InsertRangeData      C/mapping/3d/submap_3d.cc:42-51, 264-279  local_pose().inverse() in double, cast to float;
                                              the high-resolution grid takes the returns with |p - origin| <= max_range, the
                                              low-resolution grid all of them.
Every float32 expression is one IEEE operation per numpy operation (no fusion). lround of a float32 value is
sign(q) * floor(|q| + 0.5) in float64, where it is exact. Eigen's norm of a 3-vector is sqrt(x*x + (y*y + z*z)); a quaternion
rotates v as (v + w * uv) + q.vec x uv with uv = 2 (q.vec x v).

The grid is the HybridGrid's content as ordered arrays: its cells in iterator order (top cell, 8^3 brick, cell, each flat in
z-major order) and the set of bricks the reference has allocated. That order does not depend on the grid's `bits`: the top
level is shifted by half its size, 32 << bits cells, a multiple of 64, so every top cell of a smaller grid is a top cell of
the largest one.
"""
import numpy as np

f32 = np.float32
K_MIN = f32(0.1)
K_MAX = f32(1.0) - K_MIN
UPDATE_MARKER = 32768
MAX_SAMPLES = 1 << 15
LIMIT = 8192                 # cells of a grid at bits 8 lie in [-8192, 8192)
ERR_ARG, ERR_GRID_RANGE = -2, -3   # the statuses the library reports for the two CHECK failures (DL_ERR_ARG, DL_ERR_GRID_RANGE)


class InsertError(Exception):
    def __init__(self, status, message):
        super().__init__(message)
        self.status = status


# ----------------------------------------------------------------------------------------------- probability values
def round_to_int(q):
    """std::lround of float32 (or float64) values: half away from zero, exact in float64. int64."""
    q = np.asarray(q, np.float64)
    return (np.sign(q) * np.floor(np.abs(q) + 0.5)).astype(np.int64)


def value_to_probability(values):
    """ValueToProbability of uint16 values (the update marker is ignored, as the reference's doubled table does)."""
    v = np.asarray(values, np.int64) & 0x7FFF
    k_scale = (K_MAX - K_MIN) / f32(32766.0)
    p = v.astype(f32) * k_scale + (K_MIN - k_scale)
    return np.where(v == 0, K_MIN, p).astype(f32)


def bounded_float_to_value(x, lower, upper):
    x = np.asarray(x, f32)
    lower, upper = f32(lower), f32(upper)
    clamped = np.where(x > upper, upper, np.where(x < lower, lower, x)).astype(f32)
    return (round_to_int((clamped - lower) * (f32(32766.0) / (upper - lower))) + 1).astype(np.uint16)


def probability_to_value(p):
    return bounded_float_to_value(p, K_MIN, K_MAX)


def odds(p):
    p = np.asarray(p, f32)
    return (p / (f32(1.0) - p)).astype(f32)


def probability_from_odds(o):
    o = np.asarray(o, f32)
    return (o / (o + f32(1.0))).astype(f32)


def lookup_table_to_apply_odds(o):
    """ComputeLookupTableToApplyOdds(o): uint16[32768], every entry with the update marker."""
    o = f32(o)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        table = probability_to_value(probability_from_odds(o * odds(value_to_probability(np.arange(32768))))).astype(np.int64)
        table[0] = int(probability_to_value(probability_from_odds(o)))
    return (table + UPDATE_MARKER).astype(np.uint16)


def tables(hit_probability, miss_probability):
    """(hit table, miss table) of RangeDataInserter3D: Odds(options.hit_probability()) with the double narrowed to float."""
    return lookup_table_to_apply_odds(odds(f32(hit_probability))), lookup_table_to_apply_odds(odds(f32(miss_probability)))


# ----------------------------------------------------------------------------------------------- cells and order
def cell_index(points, resolution):
    """HybridGrid::GetCellIndex of float32 rows: int64 [n, 3]."""
    p = np.asarray(points, f32).reshape(-1, 3)
    return round_to_int(p / f32(resolution))


def trunc_div(a, b):
    """C++ integer division (truncation toward zero) of int64 arrays, b > 0."""
    return np.sign(a) * (np.abs(a) // b)


def order_key(cells):
    """Iterator position of every cell (int [n, 3], inside +-8192): top cell, brick, cell, each flat z-major."""
    s = np.asarray(cells, np.int64) + LIMIT
    x, y, z = s[:, 0], s[:, 1], s[:, 2]
    top = ((z >> 6) << 16) | ((y >> 6) << 8) | (x >> 6)
    brick = (((z >> 3) & 7) << 6) | (((y >> 3) & 7) << 3) | ((x >> 3) & 7)
    cell = ((z & 7) << 6) | ((y & 7) << 3) | (x & 7)
    return (top << 18) | (brick << 9) | cell


def key_to_cells(keys):
    keys = np.asarray(keys, np.int64)
    top, brick, cell = keys >> 18, (keys >> 9) & 511, keys & 511
    out = np.empty((len(keys), 3), np.int64)
    for axis, shift in ((0, 0), (1, 8), (2, 16)):
        t = (top >> shift) & 255
        b = (brick >> (3 * axis)) & 7
        c = (cell >> (3 * axis)) & 7
        out[:, axis] = t * 64 + b * 8 + c - LIMIT
    return out


def brick_key(keys):
    return np.asarray(keys, np.int64) >> 9


def bits_for(cells):
    """The smallest top-level `bits` (>= 1) whose grid holds every cell: cell c fits iff -32 << bits <= c < 32 << bits."""
    if len(cells) == 0:
        return 1
    need = np.maximum(-np.asarray(cells, np.int64).min(), np.asarray(cells, np.int64).max() + 1)
    bits = 1
    while (32 << bits) < need:
        bits += 1
    return bits


def in_range(cells):
    c = np.asarray(cells, np.int64)
    return len(c) == 0 or bool((c >= -LIMIT).all() and (c < LIMIT).all())


# ----------------------------------------------------------------------------------------------- the grid
class Grid:
    """HybridGrid content: `keys` (iterator order, ascending) with their uint16 `values`, the allocated bricks, `bits`."""

    def __init__(self, resolution):
        self.resolution = f32(resolution)
        self.keys = np.zeros(0, np.int64)
        self.values = np.zeros(0, np.uint16)
        self.bricks = np.zeros(0, np.int64)
        self.bits = 1

    def copy(self):
        g = Grid(self.resolution)
        g.keys, g.values, g.bricks, g.bits = self.keys.copy(), self.values.copy(), self.bricks.copy(), self.bits
        return g

    def lookup(self, keys):
        """Current values of `keys` (0 where the cell was never written)."""
        pos = np.searchsorted(self.keys, keys)
        pos = np.minimum(pos, max(len(self.keys) - 1, 0))
        hit = len(self.keys) > 0
        found = (self.keys[pos] == keys) if hit else np.zeros(len(keys), bool)
        return np.where(found, self.values[pos] if hit else 0, 0).astype(np.uint16)

    def write(self, keys, values):
        """Sets cells (unique keys) and allocates their bricks."""
        keys = np.asarray(keys, np.int64)
        old = np.isin(keys, self.keys, assume_unique=True)
        if old.any():
            pos = np.searchsorted(self.keys, keys[old])
            self.values[pos] = values[old]
        if (~old).any():
            all_keys = np.concatenate([self.keys, keys[~old]])
            all_values = np.concatenate([self.values, np.asarray(values, np.uint16)[~old]])
            order = np.argsort(all_keys, kind="stable")
            self.keys, self.values = all_keys[order], all_values[order]
        self.bricks = np.union1d(self.bricks, brick_key(keys))

    def set_cells(self, xs, ys, zs, values):
        """dl_grid_set_cells / HybridGrid::mutable_value in order: the last write of a cell wins."""
        cells = np.stack([np.asarray(a, np.int64) for a in (xs, ys, zs)], axis=1).reshape(-1, 3)
        if not in_range(cells):
            raise InsertError(ERR_GRID_RANGE, "cell index outside +-8192 cells")
        keys = order_key(cells)
        last = len(keys) - 1 - np.unique(keys[::-1], return_index=True)[1]
        self.write(keys[last], np.asarray(values, np.uint16)[last])
        self.bits = max(self.bits, bits_for(cells))

    def export(self):
        """(x, y, z, value) of every non-zero cell in iterator order, as int32 / uint16 arrays."""
        keep = self.values != 0
        c = key_to_cells(self.keys[keep])
        return (c[:, 0].astype(np.int32), c[:, 1].astype(np.int32), c[:, 2].astype(np.int32), self.values[keep].copy())

    @property
    def num_bricks(self):
        return len(self.bricks)


# ----------------------------------------------------------------------------------------------- Insert
def rays(origin, returns, resolution, num_free):
    """(hit cells [n, 3], miss cells [m, 3], miss ray index [m], num_samples [n]) of one Insert, samples in ray order."""
    hits = cell_index(returns, resolution)
    o = cell_index(np.asarray(origin, f32).reshape(1, 3), resolution)[0]
    delta = hits - o
    num_samples = np.abs(delta).max(axis=1) if len(hits) else np.zeros(0, np.int64)
    count = np.minimum(num_samples, max(int(num_free), 0))
    ray = np.repeat(np.arange(len(hits)), count)
    first = np.repeat(np.cumsum(count) - count, count)
    position = (num_samples - count)[ray] + (np.arange(len(ray)) - first)
    misses = o + trunc_div(delta[ray] * position[:, None], np.maximum(num_samples[ray], 1)[:, None])
    return hits, misses.reshape(-1, 3), ray, num_samples


class Plan:
    """One checked Insert: what it will write, computed before anything is written."""

    def __init__(self, grid, origin, returns, num_free):
        returns = np.asarray(returns, f32).reshape(-1, 3)
        self.grid = grid
        self.hits, self.misses, self.ray, self.num_samples = rays(origin, returns, grid.resolution, num_free)
        # a CHECK failure aborts the reference; this reading reports num_samples before the range
        if len(self.num_samples) and self.num_samples.max() >= MAX_SAMPLES:
            raise InsertError(ERR_ARG, "CHECK_LT(num_samples, 1 << 15)")
        self.touched = np.concatenate([self.hits, self.misses])
        if not in_range(self.touched):
            raise InsertError(ERR_GRID_RANGE, "cell index outside +-8192 cells")

    def apply(self, hit_table, miss_table):
        g = self.grid
        hit_keys = np.unique(order_key(self.hits))
        miss_keys = np.setdiff1d(np.unique(order_key(self.misses)), hit_keys, assume_unique=True)
        new_hits = hit_table[g.lookup(hit_keys)].astype(np.int64) - UPDATE_MARKER
        new_misses = miss_table[g.lookup(miss_keys)].astype(np.int64) - UPDATE_MARKER
        keys = np.concatenate([hit_keys, miss_keys])
        values = np.concatenate([new_hits, new_misses]).astype(np.uint16)
        g.write(keys, values)
        g.bits = max(g.bits, bits_for(self.touched))


def insert(grid, origin, returns, hit=0.55, miss=0.49, num_free=2):
    """RangeDataInserter3D::Insert into `grid`; raises InsertError (grid unchanged) where the reference CHECK-fails."""
    plan = Plan(grid, origin, returns, num_free)
    plan.apply(*tables(hit, miss))


# ----------------------------------------------------------------------------------------------- Submap3D
def _cross(a, b):
    return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1],
                     a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                     a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], axis=1)


def rotate(q, v):
    """Eigen's q * v (w x y z quaternion, rows v) in the dtype of the inputs."""
    v = np.asarray(v).reshape(-1, 3)
    w, qv = q[0], np.broadcast_to(np.asarray(q[1:], v.dtype), v.shape)
    uv = _cross(qv, v)
    uv = uv + uv
    return (v + w * uv) + _cross(qv, uv)


def to_submap_transform(submap_local_pose):
    """local_pose().inverse().cast<float>(): (t float32[3], q float32[4] w x y z). Pose: t.x t.y t.z q.w q.x q.y q.z."""
    p = np.asarray(submap_local_pose, np.float64)
    qi = np.array([p[3], -p[4], -p[5], -p[6]])
    ti = -rotate(qi, p[None, :3])[0]
    return ti.astype(f32), qi.astype(f32)


def transform(points, t, q):
    return rotate(q, np.asarray(points, f32).reshape(-1, 3)) + t


def near_mask(points, origin, max_range):
    """FilterRangeDataByMaxRange: (p - origin).norm() <= max_range, the int option compared as a float."""
    d = np.asarray(points, f32).reshape(-1, 3) - np.asarray(origin, f32).reshape(1, 3)
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    return np.sqrt(x * x + (y * y + z * z)) <= f32(int(max_range))


def submap_insert(hi, lo, submap_local_pose, origin, returns, high_resolution_max_range=20, hit=0.55, miss=0.49, num_free=2):
    """Submap3D::InsertRangeData; hi and lo may be one grid (then two Inserts into it, near points first). Both Inserts are
    checked before either writes."""
    t, q = to_submap_transform(submap_local_pose)
    all_points = transform(returns, t, q)
    o = transform(np.asarray(origin, f32).reshape(1, 3), t, q)[0]
    near = all_points[near_mask(all_points, o, high_resolution_max_range)]
    plans = [Plan(hi, o, near, num_free), Plan(lo, o, all_points, num_free)]
    hit_table, miss_table = tables(hit, miss)
    for p in plans:
        p.apply(hit_table, miss_table)
    return all_points, near, o
