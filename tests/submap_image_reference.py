"""Independent numpy reading of Submap3D's X-ray texture (AddToTextureProto, C/mapping/3d/submap_3d.cc:53-178) and the fork's
ProjectToCvMat (:381-464), from a grid's cells (x, y, z, value arrays in any order).

Everything is float32 step by step in the reference's expression order (numpy float32 ufuncs round every operation, nothing is
contracted); logf, atan2, sin and cos are glibc's (ctypes / math); lround rounds half away from zero. The cells are put in
HybridGrid::Iterator order here, from the cell index alone, and every per-pixel float sum is taken in that order.
"""
import ctypes
import math

import numpy as np

F = np.float32
K_MIN = F(0.1)
K_MAX = F(F(1.0) - K_MIN)
_LIBM = ctypes.CDLL("libm.so.6")
_LIBM.logf.restype = ctypes.c_float
_LIBM.logf.argtypes = [ctypes.c_float]


def iterator_order(xs, ys, zs):
    """Indices putting the cells in HybridGrid::Iterator order: lexicographic in (z/64, y/64, x/64, z/8 % 8, y/8 % 8, x/8 % 8,
    z % 8, y % 8, x % 8) (floor division)."""
    xs, ys, zs = (np.asarray(a, np.int64) for a in (xs, ys, zs))
    keys = [xs & 7, ys & 7, zs & 7, (xs >> 3) & 7, (ys >> 3) & 7, (zs >> 3) & 7, xs >> 6, ys >> 6, zs >> 6]
    return np.lexsort(keys)


def value_to_probability(values):
    """kValueToProbability (probability_values.cc:27-34): value * kScale + (lower - kScale), 0 -> kMinProbability."""
    v = np.asarray(values).astype(np.int64) & 32767
    k_scale = F((K_MAX - K_MIN) / F(32766.0))
    p = v.astype(F) * k_scale + F(K_MIN - k_scale)
    return np.where(v == 0, K_MIN, p).astype(F)


def lround(x):
    x = np.asarray(x, F).astype(np.float64)
    return np.where(x < 0, -np.floor(-x + 0.5), np.floor(x + 0.5)).astype(np.int64)


def _cross(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def rotate(q, v, dtype=F):
    """Eigen's q * v: uv = 2 (q.vec x v); (v + w uv) + q.vec x uv. q = (w, x, y, z); v = (3, n) or (3,) in dtype."""
    w, qv = dtype(q[0]), tuple(dtype(c) for c in q[1:])
    v = tuple(np.asarray(c, dtype) for c in v)
    uv = _cross(qv, v)
    uv = tuple(c + c for c in uv)
    c = _cross(qv, uv)
    return tuple((v[i] + w * uv[i]) + c[i] for i in range(3))


def qmul(a, b):
    return ((a[0] * b[0] - a[1] * b[1]) - a[2] * b[2] - a[3] * b[3],
            ((a[0] * b[1] + a[1] * b[0]) + a[2] * b[3]) - a[3] * b[2],
            ((a[0] * b[2] + a[2] * b[0]) + a[3] * b[1]) - a[1] * b[3],
            ((a[0] * b[3] + a[3] * b[0]) + a[1] * b[2]) - a[2] * b[1])


def qnormalized(q):
    n = np.sqrt((q[1] * q[1] + q[2] * q[2]) + (q[3] * q[3] + q[0] * q[0]))
    return tuple(c / n for c in q)


def projection_rotation(pose):
    """ProjectToCvMat :385-390 -> float32 quaternion (w, x, y, z); the translation is zero."""
    qd = tuple(float(c) for c in pose[3:])
    rotation = tuple(F(c) for c in qd)
    d = rotate(qd, (1.0, 0.0, 0.0), dtype=np.float64)  # GetYaw
    yaw = math.atan2(float(d[1]), float(d[0]))
    half = 0.5 * -yaw
    s = math.sin(half)
    inverse_yaw = (F(math.cos(half)), F(s * 0.0), F(s * 0.0), F(s * 1.0))
    return qnormalized(qmul(inverse_yaw, rotation))


def log_odds_integer(p):
    """ProbabilityToLogOddsInteger (submaps.h:37-53) with glibc logf."""
    def logit(x):
        return F(_LIBM.logf(float(F(x / F(F(1.0) - x)))))
    lo, hi = logit(K_MIN), logit(K_MAX)
    return int(lround(F(F(F(logit(F(p)) - lo) * F(254.0)) / F(hi - lo)))) + 1


def _voxels(xs, ys, zs, values, resolution, q, t):
    """ExtractVoxelData: the kept cells in iterator order -> (ix, iy, iz, probability)."""
    order = iterator_order(xs, ys, zs)
    xs, ys, zs = (np.asarray(a, np.int64)[order] for a in (xs, ys, zs))
    values = np.asarray(values, np.int64)[order]
    p = value_to_probability(values)
    keep = (values != 0) & ~(p < F(0.501))
    xs, ys, zs, p = xs[keep], ys[keep], zs[keep], p[keep]
    r = F(resolution)
    centre = (xs.astype(F) * r, ys.astype(F) * r, zs.astype(F) * r)
    moved = rotate(q, centre)
    moved = tuple(moved[i] + F(t[i]) for i in range(3))
    inverse = F(F(1.0) / r)
    return lround(moved[0] * inverse), lround(moved[1] * inverse), lround(moved[2] * inverse), p


def _accumulate(pixel, iz, p, num_pixels):
    """PixelData per pixel; probability_sum in the given (iterator) order."""
    count = np.bincount(pixel, minlength=num_pixels).astype(np.int64)
    min_z = np.full(num_pixels, np.iinfo(np.int64).max)
    max_z = np.full(num_pixels, np.iinfo(np.int64).min)
    np.minimum.at(min_z, pixel, iz)
    np.maximum.at(max_z, pixel, iz)
    max_p = np.full(num_pixels, F(0.5), F)
    np.maximum.at(max_p, pixel, p)
    s = np.zeros(num_pixels, F)
    order = np.argsort(pixel, kind="stable")
    sp, pp = pixel[order], p[order]
    start = np.searchsorted(sp, sp, side="left")
    rank = np.arange(len(sp)) - start
    for r in range(int(rank.max()) + 1 if len(rank) else 0):  # one addition per cell, in order, per pixel
        m = rank == r
        s[sp[m]] = s[sp[m]] + pp[m]
    return count, min_z, max_z, s, max_p


def pixel_value(count, min_z, max_z, s, max_p):
    """ComputePixelValues for one pixel -> (value, alpha)."""
    z_difference = F(max_z - min_z) if count > 0 else F(0)
    if z_difference < F(3.0):
        return 0, 0
    free_space = max(F(z_difference - F(count)), F(0.0))
    free_space_weight = F(F(0.15) * free_space)
    total_weight = F(F(count) + free_space_weight)
    free_space_probability = F(F(1.0) - max_p)
    average = F(F(s + F(free_space_probability * free_space_weight)) / total_weight)
    average = K_MAX if average > K_MAX else (K_MIN if average < K_MIN else average)
    delta = 128 - log_odds_integer(average)
    alpha = 0 if delta > 0 else -delta
    value = delta if delta > 0 else 0
    return value, (alpha if (value or alpha) else 1)


def texture(xs, ys, zs, values, resolution, pose):
    """AddToTextureProto -> dict(resolution, width, height, slice_pose, cells (height, width, 2) uint8). No obstructed cell:
    0 x 0 and an all-zero slice pose (the reference is undefined there)."""
    pose = np.asarray(pose, np.float64)
    q = tuple(F(c) for c in pose[3:])
    ix, iy, iz, p = _voxels(xs, ys, zs, values, resolution, q, tuple(F(c) for c in pose[:3]))
    r = F(resolution)
    if len(ix) == 0:
        return {"resolution": r, "width": 0, "height": 0, "slice_pose": np.zeros(7), "cells": np.zeros((0, 0, 2), np.uint8)}
    min_x, max_x, min_y, max_y = ix.min(), ix.max(), iy.min(), iy.max()
    width, height = int(max_y - min_y + 1), int(max_x - min_x + 1)
    pixel = (max_x - ix) * width + (max_y - iy)
    acc = _accumulate(pixel, iz, p, width * height)
    cells = np.zeros((width * height, 2), np.uint8)
    for k in np.unique(pixel):
        cells[k] = pixel_value(*(a[k] for a in acc))
    # slice_pose = global.inverse() * Translation(max_x * res, max_y * res, global z), the products in float
    qi = (pose[3], -pose[4], -pose[5], -pose[6])
    ti = tuple(-c for c in rotate(qi, pose[:3], dtype=np.float64))
    v = (float(F(F(max_x) * r)), float(F(F(max_y) * r)), float(pose[2]))
    rv = rotate(qi, v, dtype=np.float64)
    qn = qnormalized(qmul(tuple(np.float64(c) for c in qi), (1.0, 0.0, 0.0, 0.0)))
    slice_pose = np.array([rv[0] + ti[0], rv[1] + ti[1], rv[2] + ti[2], *qn], np.float64)
    return {"resolution": r, "width": width, "height": height, "slice_pose": slice_pose,
            "cells": cells.reshape(height, width, 2)}


def projection(xs, ys, zs, values, resolution, pose):
    """ProjectToCvMat -> dict(resolution, width, height, ox, oy, pixels (height, width) uint8). No obstructed cell: 0 x 0."""
    pose = np.asarray(pose, np.float64)
    q = projection_rotation(pose)
    ix, iy, iz, p = _voxels(xs, ys, zs, values, resolution, q, (F(0), F(0), F(0)))
    r = F(resolution)
    if len(ix) == 0:
        return {"resolution": r, "width": 0, "height": 0, "ox": 0.0, "oy": 0.0, "pixels": np.zeros((0, 0), np.uint8)}
    min_x, max_x, min_y, max_y = ix.min(), ix.max(), iy.min(), iy.max()
    width, height = int(max_x - min_x + 1), int(max_y - min_y + 1)
    pixel = (iy - min_y) * width + (ix - min_x)
    s = _accumulate(pixel, iz, p, width * height)[3]
    scale = F(F(255.0) / F(K_MAX - K_MIN))
    pixels = (lround(F(s - K_MIN) * scale) & 0xFF).astype(np.uint8)
    return {"resolution": r, "width": width, "height": height, "ox": int(min_x) * float(r), "oy": int(min_y) * float(r),
            "pixels": pixels.reshape(height, width)}
