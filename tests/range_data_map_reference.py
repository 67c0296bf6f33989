"""Independent float32 restatement of pb_range_data_to_ros_cloud's map (pb_range_data_to_ros_cloud_main.cc:155-176).

Per node: L = local_pose.cast<float>() and G = global_pose.cast<float>() (transform::Rigid3::cast, rigid_transform.h:167-175:
the translation and the quaternion coefficients each cast, no renormalisation); per point tp = L.inverse() * p, then
gp = G * tp. Rigid3::inverse (rigid_transform.h:189-193) is (-(conj(q) * t), conj(q)); Rigid3 * Vector3 (:214-219) is
q * p + t, and Quaternion * Vector3 is Eigen 3.3's QuaternionBase::_transformVector:
    uv = q.vec().cross(v); uv += uv; return v + q.w() * uv + q.vec().cross(uv);
evaluated left to right, with Eigen's cross product (a.y b.z - a.z b.y, a.z b.x - a.x b.z, a.x b.y - a.y b.x). Every line
below is one IEEE float32 operation per coordinate (numpy float32 arrays: no contraction into FMA, no wider intermediate).
"""
import numpy as np

F = np.float32


def cast_float(pose7):
    """Rigid3d::cast<float>(): (t xyz, q wxyz) doubles -> float32 coefficients."""
    p = np.asarray(pose7, np.float64)
    return p[:3].astype(F), p[3:].astype(F)


def _cross(ax, ay, az, bx, by, bz):
    return ay * bz - az * by, az * bx - ax * bz, ax * by - ay * bx


def quaternion_times_vector(q, vx, vy, vz):
    w, qx, qy, qz = (F(c) for c in q)
    ux, uy, uz = _cross(qx, qy, qz, vx, vy, vz)
    ux, uy, uz = ux + ux, uy + uy, uz + uz
    cx, cy, cz = _cross(qx, qy, qz, ux, uy, uz)
    return (vx + w * ux) + cx, (vy + w * uy) + cy, (vz + w * uz) + cz


def rigid_times_vector(t, q, vx, vy, vz):
    rx, ry, rz = quaternion_times_vector(q, vx, vy, vz)
    return rx + F(t[0]), ry + F(t[1]), rz + F(t[2])


def rigid_inverse(t, q):
    qc = np.array([q[0], -q[1], -q[2], -q[3]], F)
    x, y, z = quaternion_times_vector(qc, F(t[0]), F(t[1]), F(t[2]))
    return np.array([-x, -y, -z], F), qc


def node_points(local7, global7, returns):
    """One node's returns (n x 3, the builder's local frame) at its global pose, as the tool computes them."""
    p = np.ascontiguousarray(returns, F).reshape(-1, 3)
    lt, lq = cast_float(local7)
    gt, gq = cast_float(global7)
    it, iq = rigid_inverse(lt, lq)
    tx, ty, tz = rigid_times_vector(it, iq, p[:, 0], p[:, 1], p[:, 2])
    gx, gy, gz = rigid_times_vector(gt, gq, tx, ty, tz)
    return np.stack([gx, gy, gz], 1).astype(F)


def range_data_map(nodes):
    """nodes: [(trajectory_id, node_index, local7, global7, returns)] -> (points, [(trajectory_id, node_index, first_point,
    num_points)]) with the nodes in ascending (trajectory, node index) order and each node's points in attach order."""
    order = sorted(nodes, key=lambda n: (n[0], n[1]))
    parts, table, first = [], [], 0
    for t, i, local7, global7, returns in order:
        pts = node_points(local7, global7, returns)
        parts.append(pts)
        table.append((t, i, first, len(pts)))
        first += len(pts)
    points = np.concatenate(parts) if parts else np.zeros((0, 3), F)
    return points, table
