"""Reference model of the adaptive voxel filter (test infrastructure), restated in numpy from the reference's semantics
(C/ = cartographer/cartographer/, VF = C/sensor/internal/voxel_filter.cc):
  FilterByMaxRange         VF:28-38   keep a point iff point.norm() <= max_range, in input order
  AdaptivelyVoxelFiltered  VF:40-77   `min_num_points` is a float (adaptive_voxel_filter_options.proto:25): size() is compared
                                      as float; the bisection runs on float scalars, statement for statement
  VoxelFilter::Filter      VF:107-131 the first point of every voxel survives, in input order
  GetCellIndex             VF:126-131 common::RoundToInt(point / resolution) = lround of the float quotient, per axis
Every float32 expression is one IEEE operation per numpy operation. Eigen's norm of a 3-vector is sqrt(x*x + (y*y + z*z)).
lround of a float32 quotient q is sign(q) * floor(|q| + 0.5) evaluated in float64, where it is exact; in float32 `q + 0.5`
rounds up to the next integer for some q just below a half (0.49999997 + 0.5 = 1.0) and would move those points.
"""
import numpy as np

f32 = np.float32
BISECTION_STOP = f32(1e-2)   # high_length > 1e-2f * max_length
REFINE_STOP = f32(1e-1)      # (high_length - low_length) / low_length > 1e-1f
TWO = f32(2.0)


def xyz(points):
    """The first three columns of float32 rows of any stride."""
    p = np.asarray(points, f32)
    return (p if p.ndim == 2 else p.reshape(-1, 3))[:, :3]


def norms(points):
    p = xyz(points)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    return np.sqrt(x * x + (y * y + z * z))


def crop(points, max_range):
    """FilterByMaxRange: input indices of the points with norm <= max_range (NaN rows fail the comparison)."""
    return np.flatnonzero(norms(points) <= f32(max_range))


def round_to_int(q):
    """std::lround of float32 values: half away from zero, exact in float64."""
    q = np.asarray(q, np.float64)
    return (np.sign(q) * np.floor(np.abs(q) + 0.5)).astype(np.int64)


def cells(points, edge):
    """GetCellIndex of every row: lround(float32(coordinate / edge)) per axis, int64 [n, 3]."""
    return round_to_int(xyz(points) / f32(edge))


def first_per_voxel(c):
    """Positions (ascending) of the first row of every distinct cell of the int [n, 3] array `c`."""
    if len(c) == 0:
        return np.zeros(0, np.int64)
    order = np.lexsort((c[:, 2], c[:, 1], c[:, 0]))        # stable: equal cells keep input order
    s = c[order]
    start = np.ones(len(s), bool)
    start[1:] = (s[1:] != s[:-1]).any(axis=1)
    return np.sort(order[start])


def voxel_filter(points, edge):
    """VoxelFilter(edge).Filter: positions of the survivors."""
    return first_per_voxel(cells(points, edge))


def num_voxels(points, edge):
    return len(voxel_filter(points, edge))


def cell_box(points, edge):
    """(nx, ny, nz): the cells from the cell of the componentwise minimum corner to that of the maximum corner, per axis."""
    p = xyz(points)
    lo, hi = cells(p.min(axis=0, keepdims=True), edge)[0], cells(p.max(axis=0, keepdims=True), edge)[0]
    return tuple(int(v) for v in hi - lo + 1)


def adaptive_voxel_filter(points, max_length, min_num_points, max_range):
    """AdaptivelyVoxelFiltered(options, FilterByMaxRange(points, max_range)) -> (input indices of the survivors, the edges of
    every voxel filter pass in order as float32)."""
    keep, passes, _ = search(points, max_length, min_num_points, max_range)
    return keep, passes


def search(points, max_length, min_num_points, max_range):
    """adaptive_voxel_filter, plus the edge whose pass produced the survivors (None when the cloud was sparse enough)."""
    max_length, min_num_points = f32(max_length), f32(min_num_points)
    rows = crop(points, max_range)
    cropped = xyz(points)[rows]
    passes = []

    def run(edge):
        passes.append(edge)
        return voxel_filter(cropped, edge)

    def enough(keep):
        return f32(len(keep)) >= min_num_points

    if f32(len(rows)) <= min_num_points:             # 'point_cloud' is already sparse enough
        return rows, np.array(passes, f32), None
    result, edge = run(max_length), max_length
    if enough(result):                               # the first edge suffices
        return rows[result], np.array(passes, f32), edge
    high_length = max_length
    while high_length > BISECTION_STOP * max_length:
        low_length = high_length / TWO
        result, edge = run(low_length), low_length
        if enough(result):
            while (high_length - low_length) / low_length > REFINE_STOP:
                mid_length = (low_length + high_length) / TWO
                candidate = run(mid_length)
                if enough(candidate):
                    low_length = mid_length
                    result, edge = candidate, mid_length
                else:
                    high_length = mid_length
            return rows[result], np.array(passes, f32), edge
        high_length = high_length / TWO
    return rows[result], np.array(passes, f32), edge  # no edge reached min_num_points: the last low_length's survivors
