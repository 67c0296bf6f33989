"""CPU oracle of the map writer (dl_map_writer_*), test infrastructure: the assets writer's point pipeline restated in numpy, one
documented evaluation order per expression (the orders of oracle/orc_math.h), fp64 in Python floats (glibc's acos / sin through
`math`), float32 in numpy float32 arrays (every operation IEEE round-to-nearest, no contraction).

Restated (C/ = cartographer/, R/ = cartographer_ros/cartographer_ros/):
  TransformInterpolationBuffer::Has / Lookup   C/transform/transform_interpolation_buffer.cc:45-66
  Interpolate                                   C/transform/timestamped_transform.cc:22-37 (lerp + Eigen slerp in double)
  HandleMessage                                 R/assets_writer.cc:120-160
  MinMaxRangeFiteringPointsProcessor            C/io/min_max_range_filtering_points_processor.cc:39-50
  OutlierRemovingPointsProcessor                C/io/outlier_removing_points_processor.cc:81-119
  HybridGridBase::GetCellIndex                  C/mapping/3d/hybrid_grid.h:430-434 (float division, lround)
The oracle lives with the tests, as tests/schur_oracle.py does, so that the C++ oracle's sources stay as they are.
"""
import bisect
import math

import numpy as np

f32 = np.float32
EPS = 2.220446049250313e-16
GRID_HALF = 8192


class Trajectory:
    """TransformInterpolationBuffer over (universal ticks, pose7) nodes; times must be non-decreasing."""

    def __init__(self, times, poses):
        self.times = [int(t) for t in times]
        self.poses = [tuple(float(v) for v in p) for p in np.asarray(poses, np.float64).reshape(-1, 7)]
        if any(b < a for a, b in zip(self.times, self.times[1:])):
            raise ValueError("node times decrease")

    def has(self, tick):
        return bool(self.times) and self.times[0] <= tick <= self.times[-1]

    def lookup(self, tick):
        i = bisect.bisect_left(self.times, tick)
        if self.times[i] == tick:
            return self.poses[i]
        s, e = self.poses[i - 1], self.poses[i]
        duration = (self.times[i] - self.times[i - 1]) / 1e7
        factor = ((tick - self.times[i - 1]) / 1e7) / duration
        t = tuple(s[k] + (e[k] - s[k]) * factor for k in range(3))
        sw, sx, sy, sz = s[3:]
        ew, ex, ey, ez = e[3:]
        d = (sx * ex + sy * ey) + (sz * ez + sw * ew)
        abs_d = abs(d)
        if abs_d >= 1.0 - EPS:
            scale0, scale1 = 1.0 - factor, factor
        else:
            theta = math.acos(abs_d)
            sin_theta = math.sin(theta)
            scale0 = math.sin((1.0 - factor) * theta) / sin_theta
            scale1 = math.sin(factor * theta) / sin_theta
        if d < 0:
            scale1 = -scale1
        q = (scale0 * sw + scale1 * ew, scale0 * sx + scale1 * ex, scale0 * sy + scale1 * ey, scale0 * sz + scale1 * ez)
        return t + q


# ---- double pose algebra (orc_math.h orders)
def _cross(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def rotate_d(q, v):
    qv = q[1:]
    uv = _cross(qv, v)
    uv = (uv[0] + uv[0], uv[1] + uv[1], uv[2] + uv[2])
    c = _cross(qv, uv)
    return tuple((v[k] + q[0] * uv[k]) + c[k] for k in range(3))


def compose_d(l, r):
    t = rotate_d(l[3:], r[:3])
    t = tuple(t[k] + l[k] for k in range(3))
    aw, ax, ay, az = l[3:]
    bw, bx, by, bz = r[3:]
    q = (aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
         aw * by + ay * bw + az * bx - ax * bz, aw * bz + az * bw + ax * by - ay * bx)
    n = math.sqrt((q[1] * q[1] + q[2] * q[2]) + (q[3] * q[3] + q[0] * q[0]))
    return t + tuple(c / n for c in q)


# ---- float32 point algebra on (n,) arrays
def apply_f(pose_f, x, y, z):
    """Rigid3f * p, pose_f = 7 float32 (t, q wxyz), x / y / z float32 arrays."""
    tx, ty, tz, qw, qx, qy, qz = pose_f
    uvx = qy * z - qz * y
    uvy = qz * x - qx * z
    uvz = qx * y - qy * x
    uvx, uvy, uvz = uvx + uvx, uvy + uvy, uvz + uvz
    cx = qy * uvz - qz * uvy
    cy = qz * uvx - qx * uvz
    cz = qx * uvy - qy * uvx
    return ((x + qw * uvx) + cx) + tx, ((y + qw * uvy) + cy) + ty, ((z + qw * uvz) + cz) + tz


def norm_f(x, y, z):
    return np.sqrt(x * x + (y * y + z * z))


def lround(q):
    """std::lround of float32 values (ties away from zero), exact through float64."""
    a = np.abs(q.astype(np.float64))
    r = np.floor(a)
    r = r + (a - r >= 0.5)
    return (np.sign(q) * r).astype(np.int64)


def cell_index(x, y, z, res):
    return lround(x / res), lround(y / res), lround(z / res)


def cell_key(cx, cy, cz):
    return ((cx + GRID_HALF) << 28) | ((cy + GRID_HALF) << 14) | (cz + GRID_HALF)


def in_extent(cx, cy, cz):
    return ((cx >= -GRID_HALF) & (cx < GRID_HALF) & (cy >= -GRID_HALF) & (cy < GRID_HALF) & (cz >= -GRID_HALF)
            & (cz < GRID_HALF))


def handle_message(trajectories, msg, rows):
    """HandleMessage -> (points (k, 3) float32, origin (3,) float32 or None, dropped by Has)."""
    stamp, first, n, traj, s2t = msg
    r = np.asarray(rows[first:first + n], np.float32)
    tr = trajectories[traj]
    s2t = tuple(float(v) for v in s2t)
    out = np.zeros((n, 3), np.float32)
    kept = np.zeros(n, bool)
    last_pose = None
    bits = r[:, 3].view(np.uint32) if n else np.zeros(0, np.uint32)
    pose_of = {}
    for b in np.unique(bits):
        t = float(np.uint32(b).view(np.float32))
        tick = int(stamp) + int(t * 1e7)   # FromSeconds truncates toward zero
        pose_of[int(b)] = (np.array(compose_d(tr.lookup(tick), s2t), np.float64).astype(np.float32)
                           if tr.has(tick) else None)
    for b, pose in pose_of.items():
        if pose is None:
            continue
        sel = bits == b
        x, y, z = apply_f(pose, r[sel, 0], r[sel, 1], r[sel, 2])
        out[sel, 0], out[sel, 1], out[sel, 2] = x, y, z
        kept |= sel
    if kept.any():
        last = int(np.nonzero(kept)[0][-1])
        zero = np.zeros(1, np.float32)
        last_pose = pose_of[int(bits[last])]
        origin = np.array([c[0] for c in apply_f(last_pose, zero, zero, zero)], np.float32)
    else:
        origin = None
    return out[kept], origin, int(n - kept.sum())


def range_gate(points, origin, min_range, max_range):
    d = norm_f(points[:, 0] - origin[0], points[:, 1] - origin[1], points[:, 2] - origin[2]).astype(np.float64)
    return (min_range <= d) & (d <= max_range)


def ray_samples(points, origin, voxel_size, res):
    """ProcessInPhaseTwo's samples of every point of one batch -> (cell keys of the samples inside the extent, sample count)."""
    o = origin
    dx, dy, dz = points[:, 0] - o[0], points[:, 1] - o[1], points[:, 2] - o[2]
    length = norm_f(dx, dy, dz)
    x = np.zeros(len(points), np.float32)
    keys, count = [], 0
    active = np.nonzero(x < length)[0]
    while len(active):
        count += len(active)
        s = x[active] / length[active]
        cx, cy, cz = cell_index(o[0] + s * dx[active], o[1] + s * dy[active], o[2] + s * dz[active], res)
        inside = in_extent(cx, cy, cz)
        keys.append(cell_key(cx[inside], cy[inside], cz[inside]))
        x[active] = (x[active].astype(np.float64) + voxel_size).astype(np.float32)
        active = active[x[active] < length[active]]
    return (np.concatenate(keys) if keys else np.zeros(0, np.int64)), count


def write_map(trajectories, msgs, rows, range_filter=None, voxel_size=0.0):
    """The whole pipeline over all passes. trajectories: {id: Trajectory}; msgs: [(stamp, first_row, num_rows, trajectory_id,
    sensor_to_tracking7)]; rows: (n, 4) float32. Returns a dict: points, origins (NaN rows for messages without a batch),
    dropped_no_pose, dropped_range, dropped_moving, messages_without_batch, num_samples, and with voxel_size > 0 the cell table
    (cells (k, 3), hits, rays) sorted by cell index."""
    batches, origins = [], np.full((len(msgs), 3), np.nan, np.float32)
    no_pose = dropped_range = 0
    for m, msg in enumerate(msgs):
        pts, origin, dropped = handle_message(trajectories, msg, rows)
        no_pose += dropped
        if origin is None:
            continue
        origins[m] = origin
        if range_filter is not None:
            keep = range_gate(pts, origin, *range_filter)
            dropped_range += int((~keep).sum())
            pts = pts[keep]
        batches.append((pts, origin))
    res = {"origins": origins, "dropped_no_pose": no_pose, "dropped_range": dropped_range, "dropped_moving": 0,
           "messages_without_batch": sum(1 for o in origins if np.isnan(o[0])), "num_samples": 0}
    allpts = np.concatenate([b[0] for b in batches]) if batches else np.zeros((0, 3), np.float32)
    if voxel_size <= 0:
        res["points"] = allpts
        return res
    r = f32(voxel_size)
    cx, cy, cz = cell_index(allpts[:, 0], allpts[:, 1], allpts[:, 2], r)
    if not in_extent(cx, cy, cz).all():
        raise ValueError("a cell lies beyond the hybrid grid's largest extent")
    for pts, origin in batches:   # the device also bounds every ray by checking its origin's cell
        ox, oy, oz = cell_index(origin[:1], origin[1:2], origin[2:3], r)
        if len(pts) and not in_extent(ox, oy, oz).all():
            raise ValueError("a batch origin lies beyond the hybrid grid's largest extent")
    hit_keys, hits = np.unique(cell_key(cx, cy, cz), return_counts=True)
    sample_keys, samples = [], 0
    for pts, origin in batches:
        k, c = ray_samples(pts, origin, float(voxel_size), r)
        sample_keys.append(k)
        samples += c
    sk = np.concatenate(sample_keys) if sample_keys else np.zeros(0, np.int64)
    sk = sk[np.isin(sk, hit_keys)]
    ray_keys, ray_counts = np.unique(sk, return_counts=True)
    rays = np.zeros(len(hit_keys), np.int64)
    rays[np.searchsorted(hit_keys, ray_keys)] = ray_counts
    pos = np.searchsorted(hit_keys, cell_key(cx, cy, cz))
    keep = rays[pos].astype(np.float64) < 3.0 * hits[pos].astype(np.float64)
    res["points"] = allpts[keep]
    res["dropped_moving"] = int((~keep).sum())
    res["num_samples"] = samples
    res["cells"] = np.stack([((hit_keys >> 28) & 0x3fff) - GRID_HALF, ((hit_keys >> 14) & 0x3fff) - GRID_HALF,
                             (hit_keys & 0x3fff) - GRID_HALF], axis=1).astype(np.int32)
    res["hits"], res["rays"] = hits.astype(np.int32), rays.astype(np.int32)
    return res
