"""Reference model of RotationalScanMatcher::ComputeHistogram (test infrastructure), restated in numpy float32 from the reference's
semantics, statement by statement (C/ = cartographer/cartographer/, RSM = C/mapping/internal/3d/scan_matching/rotational_scan_matcher.cc):
  ComputeHistogram               RSM:156-167  std::map of slices RoundToInt(z / 0.2f) -> ascending keys, points in input order
  SortSlice                      RSM:93-118   centroid of the slice; points closer than 0.2 m dropped; std::sort by atan2 angle
  AddPointCloudSliceToHistogram  RSM:61-88    centroid of the SORTED slice; `last` walk; weight 1 - |dot| of the unit vectors
  ComputeCentroid                RSM:52-59    sequential float sum / static_cast<float>(size)
  AddValueToHistogram            RSM:35-50    (float)M_PI wrapping, bucket clamp
  common::RoundToInt = lround    C/common/port.h:41 (half away from zero); common::atan2(v) = atan2(v.y, v.x)  C/common/math.h:70-72
Every float32 expression is one IEEE operation per numpy operation (no contraction). The model's atan2 is fp64 atan2 of the exact
float deltas rounded to float32, i.e. a correctly rounded atan2f; equal angles keep input order (a stable sort), which is what
libstdc++'s std::sort does for at most 16 elements (a plain insertion sort). Beyond 16 the order of equal angles is unspecified.

`ambiguous_points` finds the points whose result could change with the atan2 implementation: the reference's glibc atan2f, the
device's atan2f and this model's are each within a few ulps of the true angle (CUDA 12 documents atan2f to 3 ulp; glibc's
x86_64 atan2f is listed at <= 2), so a point is ambiguous when, within `margin_ulps`, its sort angle reaches the angle of a
neighbour with a different delta, or its walk angle reaches a bucket boundary. `clean` removes them until none are left; on the
cleaned cloud every correct implementation must produce the same histogram bit for bit.
"""
import numpy as np

f32 = np.float32
SLICE_HEIGHT = f32(0.2)
MIN_DISTANCE = f32(0.2)
MAX_DISTANCE = f32(0.9)
PI = f32(np.pi)            # static_cast<float>(M_PI) = 3.14159274
INSERTION_SORT_MAX = 16    # libstdc++ _S_threshold: std::sort of at most 16 elements is a stable insertion sort


def round_to_int(x):
    """std::lround of float32 values (half away from zero); exact in fp64."""
    x = np.asarray(x, np.float64)
    return (np.sign(x) * np.floor(np.abs(x) + 0.5)).astype(np.int64)


def atan2_f32(dy, dx):
    """Correctly rounded atan2f (fp64 atan2 of the float inputs, rounded once); IEEE special cases for zero inputs."""
    return np.arctan2(np.asarray(dy, np.float64), np.asarray(dx, np.float64)).astype(f32)


def exact_atan2(dy, dx):
    """True where the float atan2 result is fixed by the C / CUDA special cases (a zero input): +-0, +-pi/2 or +-pi rounded."""
    return (np.asarray(dy) == 0) | (np.asarray(dx) == 0)


def centroid(x, y):
    """ComputeCentroid (RSM:52-59) of the x and y columns: sequential float sums divided by the float count."""
    n = f32(len(x))
    return np.add.accumulate(x, dtype=f32)[-1] / n, np.add.accumulate(y, dtype=f32)[-1] / n


def bucket_of(angle, size):
    """AddValueToHistogram's bucket (RSM:35-50) for float32 angles."""
    a = np.array(angle, f32, ndmin=1)
    while (a > PI).any():
        a = np.where(a > PI, a - PI, a).astype(f32)
    while (a < 0).any():
        a = np.where(a < 0, a + PI, a).astype(f32)
    zero_to_one = a / PI
    return np.clip(round_to_int(f32(size) * zero_to_one - f32(0.5)), 0, size - 1)


def slices(points):
    """ComputeHistogram's std::map (RSM:159-162): [(key, input indices in input order)] in ascending key order."""
    p = np.asarray(points, f32).reshape(-1, 3)
    keys = round_to_int(p[:, 2] / SLICE_HEIGHT)
    order = np.argsort(keys, kind="stable")
    starts = np.flatnonzero(np.diff(keys[order], prepend=keys[order][:1] - 1))
    return [(int(keys[order[b]]), order[b:e]) for b, e in zip(starts, list(starts[1:]) + [len(order)])]


def sort_slice(x, y, angles=None):
    """SortSlice (RSM:93-118) of one slice's x, y columns -> (kept indices in sorted order, first centroid, deltas dx, dy).
    `angles` replaces the model's atan2 of the deltas (one value per point) to play a different atan2 implementation."""
    cx, cy = centroid(x, y)
    dx, dy = x - cx, y - cy
    kept = np.nonzero(~(np.sqrt(dx * dx + dy * dy) < MIN_DISTANCE))[0]
    a = (atan2_f32(dy, dx) if angles is None else np.asarray(angles, f32))[kept]
    return kept[np.argsort(a, kind="stable")], (cx, cy), dx, dy


def walk(x, y):
    """AddPointCloudSliceToHistogram (RSM:61-88) of a sorted slice -> (positions, deltas dx, dy, values) of the points it adds,
    in walk order. The direction term uses the centroid of this (sorted) slice."""
    if len(x) == 0:
        return np.zeros(0, np.int64), np.zeros(0, f32), np.zeros(0, f32), np.zeros(0, f32)
    cx, cy = centroid(x, y)
    ccx, ccy = x - cx, y - cy
    direction_norm = np.sqrt(ccx * ccx + ccy * ccy)
    lx, ly = x[0], y[0]
    pos, ex, ey = [], [], []
    for k in range(len(x)):
        dx, dy = x[k] - lx, y[k] - ly
        distance = np.sqrt(dx * dx + dy * dy)
        if distance < MIN_DISTANCE or direction_norm[k] < MIN_DISTANCE:
            continue
        if distance > MAX_DISTANCE:
            lx, ly = x[k], y[k]
            continue
        pos.append(k); ex.append(dx); ey.append(dy)
    pos = np.array(pos, np.int64)
    dx, dy = np.array(ex, f32), np.array(ey, f32)
    distance = np.sqrt(dx * dx + dy * dy)
    dot = (dx / distance) * (ccx[pos] / direction_norm[pos]) + (dy / distance) * (ccy[pos] / direction_norm[pos])
    value = np.maximum(f32(0), f32(1) - np.abs(dot))
    return pos, dx, dy, value


def events(points):
    """The reference's (point index, walk dx, walk dy, value) additions in the order of its += chain."""
    p = np.asarray(points, f32).reshape(-1, 3)
    out = []
    for _, idx in slices(p):
        order, _, _, _ = sort_slice(p[idx, 0], p[idx, 1])
        s = idx[order]
        pos, dx, dy, value = walk(p[s, 0], p[s, 1])
        out.append((s[pos], dx, dy, value))
    if not out:
        return np.zeros(0, np.int64), np.zeros(0, f32), np.zeros(0, f32), np.zeros(0, f32)
    return tuple(np.concatenate(c) for c in zip(*out))


def compute_histogram(points, size):
    """RotationalScanMatcher::ComputeHistogram(points, size) in float32."""
    _, dx, dy, value = events(points)
    buckets = bucket_of(atan2_f32(dy, dx), size) if len(value) else np.zeros(0, np.int64)
    h = np.zeros(size, f32)
    for b in np.unique(buckets):
        h[b] = np.add.accumulate(value[buckets == b], dtype=f32)[-1]    # 0 + v0 + v1 + ... in order (0 + v0 is exact)
    return h


def _ulps(angle64, margin_ulps):
    return margin_ulps * np.spacing(np.abs(angle64).astype(f32)).astype(np.float64)


def _sort_ambiguous(dx, dy, kept, margin_ulps):
    """Kept positions whose sort angle could be ordered differently against a neighbour with a different delta."""
    theta = np.arctan2(dy[kept].astype(np.float64), dx[kept].astype(np.float64))
    exact = exact_atan2(dy[kept], dx[kept])
    w = np.where(exact, 0.0, _ulps(theta, margin_ulps))
    order = np.argsort(theta, kind="stable")
    t, w, ex = theta[order], w[order], exact[order]
    ident = dx[kept][order].view(np.uint32).astype(np.uint64) << np.uint64(32) | dy[kept][order].view(np.uint32)
    bad = np.zeros(len(t), bool)
    wmax = w.max() if len(w) else 0.0
    for k in range(1, len(t)):
        i, j = np.arange(len(t) - k), np.arange(k, len(t))
        near = t[j] - t[i] <= w[i] + wmax
        if not near.any():
            break
        i, j = i[near], j[near]
        overlap = (t[j] - w[j] <= t[i] + w[i]) & (ident[i] != ident[j])
        # both angles fixed by the special cases and equal (e.g. +0 and -0): an exact tie, ordered by input position, which only
        # the insertion sort of a short slice keeps
        tie = ex[i] & ex[j] & (t[i] == t[j])
        if len(t) <= INSERTION_SORT_MAX:
            overlap &= ~tie
        bad[i[overlap]] = True
        bad[j[overlap]] = True
    return kept[order[bad]]


def ambiguous_points(points, size, margin_ulps=8):
    """Input indices of the points whose contribution could depend on the atan2 implementation (see the module docstring)."""
    p = np.asarray(points, f32).reshape(-1, 3)
    out = []
    for _, idx in slices(p):
        x, y = p[idx, 0], p[idx, 1]
        order, _, dx, dy = sort_slice(x, y)
        kept = np.sort(order)
        out.append(idx[_sort_ambiguous(dx, dy, kept, margin_ulps)])
        s = idx[order]
        pos, wdx, wdy, _ = walk(p[s, 0], p[s, 1])
        theta = np.arctan2(wdy.astype(np.float64), wdx.astype(np.float64))
        w = np.where(exact_atan2(wdy, wdx), 0.0, _ulps(theta, margin_ulps))
        lo, hi = bucket_of((theta - w).astype(f32), size), bucket_of((theta + w).astype(f32), size)
        mid = bucket_of(theta.astype(f32), size)
        out.append(s[pos[(lo != mid) | (hi != mid)]])
    return np.unique(np.concatenate(out)) if out else np.zeros(0, np.int64)


def clean(points, size, margin_ulps=8):
    """The cloud without ambiguous points, removed until none are left (removing points moves the centroids)."""
    p = np.asarray(points, f32).reshape(-1, 3)
    while True:
        bad = ambiguous_points(p, size, margin_ulps)
        if len(bad) == 0:
            return p
        p = np.delete(p, bad, axis=0)
