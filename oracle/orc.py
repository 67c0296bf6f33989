"""TEST INFRASTRUCTURE — ctypes view of the CPU oracle (oracle/build/liborc.so).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this.
Poses are numpy float64[7]: t.x t.y t.z q.w q.x q.y q.z.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
f64p = np.ctypeslib.ndpointer(np.float64, flags="C_CONTIGUOUS")
i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
i64p = np.ctypeslib.ndpointer(np.int64, flags="C_CONTIGUOUS")
u16p = np.ctypeslib.ndpointer(np.uint16, flags="C_CONTIGUOUS")


class SolveSummary(C.Structure):
    _fields_ = [("initial_cost", C.c_double), ("final_cost", C.c_double), ("num_iterations", C.c_int),
                ("num_successful_steps", C.c_int), ("num_unsuccessful_steps", C.c_int), ("termination", C.c_int),
                ("num_residual_evaluations", C.c_int), ("num_jacobian_evaluations", C.c_int)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class Preintegration(C.Structure):
    """Pre-integrated IMU measurement (layout shared with dl_preintegration in include/dliom_b200.h)."""
    _fields_ = [("sum_dt", C.c_double), ("delta_p", C.c_double * 3), ("delta_q", C.c_double * 4),
                ("delta_v", C.c_double * 3), ("ba", C.c_double * 3), ("bg", C.c_double * 3),
                ("jacobian", C.c_double * 225), ("covariance", C.c_double * 225)]


class FcsmResult(C.Structure):
    _fields_ = [("found", C.c_int), ("score", C.c_float), ("pose", C.c_double * 7), ("rotational_score", C.c_float),
                ("low_resolution_score", C.c_float), ("offset", C.c_int * 3), ("reserved", C.c_int),
                ("leaves_scored", C.c_int64)]


class FrontEndOptions(C.Structure):
    """Field-for-field the parameters LocalTrajectoryBuilder3D reads on the hot path; defaults =
    configuration_files/trajectory_builder_3d.lua."""
    _fields_ = [("min_range", C.c_float), ("max_range", C.c_float), ("voxel_filter_size", C.c_float),
                ("hi_max_length", C.c_float), ("hi_min_num_points", C.c_float), ("hi_max_range", C.c_float),
                ("lo_max_length", C.c_float), ("lo_min_num_points", C.c_float), ("lo_max_range", C.c_float),
                ("use_rtcsm", C.c_int), ("scan_period", C.c_double),
                ("rtcsm_linear_window", C.c_double), ("rtcsm_angular_window", C.c_double),
                ("rtcsm_w_t", C.c_double), ("rtcsm_w_r", C.c_double),
                ("occ_w0", C.c_double), ("occ_w1", C.c_double), ("trans_w", C.c_double), ("rot_w", C.c_double),
                ("only_yaw", C.c_int), ("nonmono", C.c_int), ("max_iter", C.c_int)]

    @staticmethod
    def defaults(**kw):
        o = FrontEndOptions(min_range=1.0, max_range=60.0, voxel_filter_size=0.15,
                            hi_max_length=2.0, hi_min_num_points=150, hi_max_range=15.0,
                            lo_max_length=4.0, lo_min_num_points=200, lo_max_range=60.0,
                            use_rtcsm=0, scan_period=0.1,
                            rtcsm_linear_window=0.15, rtcsm_angular_window=np.deg2rad(1.0),
                            rtcsm_w_t=1e-1, rtcsm_w_r=1e-1,
                            occ_w0=1.0, occ_w1=6.0, trans_w=5.0, rot_w=4e2, only_yaw=0, nonmono=0, max_iter=12)
        for k, v in kw.items():
            setattr(o, k, v)
        return o


def build():
    subprocess.check_call(["make", "-s", "-C", _HERE])


def lib():
    global _LIB
    if _LIB is not None:
        return _LIB
    path = os.path.join(_HERE, "build", "liborc.so")
    if not os.path.exists(path):
        build()
    L = C.CDLL(path)
    L.orc_value_to_probability.restype = C.c_float
    L.orc_value_to_probability.argtypes = [C.c_uint16]
    L.orc_probability_to_value.restype = C.c_uint16
    L.orc_probability_to_value.argtypes = [C.c_float]
    L.orc_odds.restype = C.c_float
    L.orc_odds.argtypes = [C.c_float]
    L.orc_lookup_table_to_apply_odds.argtypes = [C.c_float, u16p]
    L.orc_value_to_probability_table.argtypes = [f32p]
    L.orc_grid_create.restype = C.c_void_p
    L.orc_grid_create.argtypes = [C.c_float]
    L.orc_grid_destroy.argtypes = [C.c_void_p]
    L.orc_grid_resolution.restype = C.c_float
    L.orc_grid_resolution.argtypes = [C.c_void_p]
    L.orc_grid_bits.argtypes = [C.c_void_p]
    L.orc_grid_set_probability.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float]
    L.orc_grid_set_value.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_uint16]
    L.orc_grid_value.restype = C.c_uint16
    L.orc_grid_value.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
    L.orc_grid_probability.restype = C.c_float
    L.orc_grid_probability.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
    L.orc_grid_cell_index.argtypes = [C.c_void_p, f32p, i32p]
    L.orc_grid_center_of_cell.argtypes = [C.c_void_p, i32p, f32p]
    L.orc_grid_apply_lookup_table.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, u16p]
    L.orc_grid_finish_update.argtypes = [C.c_void_p]
    L.orc_grid_num_cells.restype = C.c_int64
    L.orc_grid_num_cells.argtypes = [C.c_void_p]
    L.orc_grid_export.argtypes = [C.c_void_p, i32p, i32p, i32p, u16p]
    L.orc_grid_insert_range_data.argtypes = [C.c_void_p, f32p, f32p, C.c_int64, C.c_double, C.c_double, C.c_int]
    L.orc_submap_insert_range_data.argtypes = [C.c_void_p, C.c_void_p, f64p, f32p, f32p, C.c_int64, C.c_double, C.c_double,
                                               C.c_int, C.c_int]
    L.orc_interpolate.restype = C.c_double
    L.orc_interpolate.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_double]
    L.orc_interpolate_grad.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_double, f64p]
    L.orc_voxel_filter.restype = C.c_int64
    L.orc_voxel_filter.argtypes = [f32p, C.c_int64, C.c_int, C.c_float, i64p]
    L.orc_voxel_indices.argtypes = [f32p, C.c_int64, C.c_int, C.c_float, i32p]
    L.orc_adaptive_voxel_filter.restype = C.c_int64
    L.orc_adaptive_voxel_filter.argtypes = [f32p, C.c_int64, C.c_int, C.c_float, C.c_float, C.c_float, i64p, f32p,
                                            C.POINTER(C.c_int)]
    L.orc_rtcsm_match.restype = C.c_float
    L.orc_rtcsm_match.argtypes = [C.c_void_p, f32p, C.c_int64, f64p, C.c_double, C.c_double, C.c_double, C.c_double,
                                  f64p, C.POINTER(C.c_int64), i32p, f32p, C.c_void_p]
    L.orc_ceres_match.argtypes = [C.c_int, C.POINTER(C.c_void_p), i64p, C.POINTER(C.c_void_p), f64p, C.c_double,
                                  C.c_double, C.c_int, C.c_int, C.c_int, f64p, f64p, f64p, C.POINTER(SolveSummary),
                                  C.c_void_p]
    L.orc_ceres_normal_equations.argtypes = [C.c_int, C.POINTER(C.c_void_p), i64p, C.POINTER(C.c_void_p), f64p,
                                             C.c_double, C.c_double, f64p, f64p, f64p, f64p, f64p, f64p]
    L.orc_ingest_scan.argtypes = [C.POINTER(FrontEndOptions), C.c_void_p, C.c_int64, f32p, f64p, f64p, i64p, f32p,
                                  f32p, f32p, f32p, i64p]
    L.orc_match_scan.argtypes = [C.POINTER(FrontEndOptions), f32p, C.c_int64, f64p, f64p, C.c_void_p, C.c_void_p,
                                 f64p, f64p, C.POINTER(SolveSummary), i64p, i64p, i64p, C.POINTER(C.c_float)]
    L.orc_frontend_batch.restype = C.c_double
    L.orc_frontend_batch.argtypes = [C.POINTER(FrontEndOptions), C.c_int, C.POINTER(C.c_void_p), i64p, f32p, f64p,
                                     f64p, f64p, C.c_void_p, C.c_void_p, C.c_int, f64p, i32p]
    L.orc_fcsm_match_3dof.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double,
                                      f64p, f32p, C.c_int64, f32p, C.c_int64, C.c_float, C.POINTER(FcsmResult)]
    L.orc_decode_point_cloud2.restype = C.c_int64
    L.orc_decode_point_cloud2.argtypes = [C.c_int] * 6 + [C.c_void_p, C.c_int64, f64p, f32p, C.POINTER(C.c_double)]
    L.orc_angle_of_angle_axis_f.restype = C.c_float
    L.orc_angle_of_angle_axis_f.argtypes = [f32p]
    L.orc_rotation_delta_cost.restype = C.c_double
    L.orc_rotation_delta_cost.argtypes = [C.c_double, f64p, f64p]
    L.orc_precomputation_values.argtypes = [C.c_void_p, C.c_int, C.c_int64, np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS"),
                                            np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")]
    L.orc_pose_graph_solve.argtypes = [C.c_int, C.c_int, f64p, C.c_int, np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS"), f64p, f64p,
                                       C.c_int, C.c_int, C.POINTER(SolveSummary), C.c_int]
    L.orc_spa_residual.argtypes = [f64p, f64p, f64p, C.c_double, C.c_double, f64p, f64p]
    L.orc_fcsm_match_full.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double,
                                      C.c_double, f64p, f64p, f32p, C.c_int64, f32p, C.c_int64, C.c_void_p, C.c_int, C.c_float,
                                      C.POINTER(FcsmResult), C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_void_p]
    L.orc_rotational_match.argtypes = [f32p, C.c_int, C.c_float, f32p, C.c_float, f32p, C.c_int, f32p]
    L.orc_compute_histogram.argtypes = [f32p, C.c_int64, C.c_int, f32p]
    L.orc_fcsm_create.restype = C.c_void_p
    L.orc_fcsm_create.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double]
    L.orc_fcsm_destroy.argtypes = [C.c_void_p]
    L.orc_fcsm_match.argtypes = [C.c_void_p, f64p, f32p, C.c_int64, f32p, C.c_int64, C.c_float, C.POINTER(FcsmResult)]
    L.orc_imu_preintegrate.argtypes = [f64p, f64p, f64p, C.c_int, f64p, f64p, f64p, C.POINTER(Preintegration)]
    L.orc_imu_predict.argtypes = [f64p, C.POINTER(Preintegration), f64p, f64p]
    L.orc_imu_residual.argtypes = [f64p, f64p, C.POINTER(Preintegration), f64p, f64p, C.c_void_p]
    L.orc_fused_match.argtypes = [C.c_int, C.POINTER(C.c_void_p), i64p, C.POINTER(C.c_void_p), f64p, C.c_double,
                                  C.c_double, C.c_int, C.c_int, f64p, f64p, f64p, C.POINTER(Preintegration), f64p,
                                  C.c_double, f64p, C.POINTER(SolveSummary)]
    _LIB = L
    return L


IDENTITY_POSE = np.array([0, 0, 0, 1, 0, 0, 0], np.float64)


def pose(t=(0, 0, 0), q=(1, 0, 0, 0)):
    return np.array(list(t) + list(q), np.float64)


def angle_axis_pose(t, angle, axis):
    """Rigid3d(t, AngleAxisd(angle, axis)) — Eigen: w = cos(a/2), xyz = sin(a/2) * axis (axis used as given)."""
    axis = np.asarray(axis, np.float64)
    return pose(t, [np.cos(angle / 2)] + list(np.sin(angle / 2) * axis))


class Grid:
    """The oracle's HybridGrid (uint16 probability values in a sparse 3-level voxel tree)."""

    def __init__(self, resolution):
        self.L = lib()
        self.h = C.c_void_p(self.L.orc_grid_create(np.float32(resolution)))
        self.resolution = np.float32(resolution)

    def __del__(self):
        if getattr(self, "h", None):
            self.L.orc_grid_destroy(self.h)
            self.h = None

    def cell_index(self, p):
        out = np.zeros(3, np.int32)
        self.L.orc_grid_cell_index(self.h, np.ascontiguousarray(p, np.float32), out)
        return out

    def center_of_cell(self, idx):
        out = np.zeros(3, np.float32)
        self.L.orc_grid_center_of_cell(self.h, np.ascontiguousarray(idx, np.int32), out)
        return out

    def set_probability(self, idx, p):
        if self.L.orc_grid_set_probability(self.h, int(idx[0]), int(idx[1]), int(idx[2]), np.float32(p)):
            raise RuntimeError("grid growth limit (CHECK_LE(new_bits, 8))")

    def set_value(self, idx, v):
        if self.L.orc_grid_set_value(self.h, int(idx[0]), int(idx[1]), int(idx[2]), int(v)):
            raise RuntimeError("grid growth limit")

    def set_cells(self, xs, ys, zs, values):
        """Bulk set_value from the ToProto layout (what Grid.export() of either implementation returns)."""
        xs, ys, zs = (np.ascontiguousarray(a, np.int32) for a in (xs, ys, zs))
        values = np.ascontiguousarray(values, np.uint16)
        f = self.L.orc_grid_set_cells
        if f(self.h, C.c_int64(len(xs)), xs.ctypes.data_as(C.c_void_p), ys.ctypes.data_as(C.c_void_p),
             zs.ctypes.data_as(C.c_void_p), values.ctypes.data_as(C.c_void_p)):
            raise RuntimeError("grid growth limit")

    def value(self, idx):
        return self.L.orc_grid_value(self.h, int(idx[0]), int(idx[1]), int(idx[2]))

    def probability(self, idx):
        return self.L.orc_grid_probability(self.h, int(idx[0]), int(idx[1]), int(idx[2]))

    def apply_lookup_table(self, idx, table):
        return bool(self.L.orc_grid_apply_lookup_table(self.h, int(idx[0]), int(idx[1]), int(idx[2]), table))

    def finish_update(self):
        self.L.orc_grid_finish_update(self.h)

    def bits(self):
        return self.L.orc_grid_bits(self.h)

    def export(self):
        """(x, y, z, value) parallel arrays in the reference's iteration order (HybridGrid proto layout)."""
        n = self.L.orc_grid_num_cells(self.h)
        xs, ys, zs = (np.zeros(n, np.int32) for _ in range(3))
        vs = np.zeros(n, np.uint16)
        if n:
            self.L.orc_grid_export(self.h, xs, ys, zs, vs)
        return xs, ys, zs, vs

    def insert_range_data(self, origin, returns, hit=0.55, miss=0.49, num_free=2):
        returns = np.ascontiguousarray(returns, np.float32).reshape(-1, 3)
        if self.L.orc_grid_insert_range_data(self.h, np.ascontiguousarray(origin, np.float32), returns, len(returns),
                                             hit, miss, num_free):
            raise RuntimeError("grid growth limit (CHECK_LE(new_bits, 8))")

    def interpolate(self, x, y, z):
        return self.L.orc_interpolate(self.h, x, y, z)

    def interpolate_grad(self, x, y, z):
        out = np.zeros(4)
        self.L.orc_interpolate_grad(self.h, x, y, z, out)
        return out


def submap_insert_range_data(hi, lo, local_pose, origin, returns, high_resolution_max_range=20, hit=0.55, miss=0.49,
                             num_free=2):
    """Submap3D::InsertRangeData of local-frame range data into the grids (hi may be lo) of the submap at local_pose."""
    returns = np.ascontiguousarray(returns, np.float32).reshape(-1, 3)
    if lib().orc_submap_insert_range_data(hi.h, lo.h, np.ascontiguousarray(local_pose, np.float64),
                                          np.ascontiguousarray(origin, np.float32), returns, len(returns), hit, miss, num_free,
                                          int(high_resolution_max_range)):
        raise RuntimeError("grid growth limit (CHECK_LE(new_bits, 8))")


def lookup_table_to_apply_odds(odds):
    """ComputeLookupTableToApplyOdds(odds) (float odds): uint16[32768], update marker included."""
    out = np.zeros(32768, np.uint16)
    lib().orc_lookup_table_to_apply_odds(np.float32(odds), out)
    return out


def voxel_filter(points, resolution):
    """Indices (input order) of the first point in each voxel. points: (n, stride) float32, stride >= 3."""
    points = np.ascontiguousarray(points, np.float32)
    n, stride = points.shape
    keep = np.zeros(max(n, 1), np.int64)
    m = lib().orc_voxel_filter(points, n, stride, np.float32(resolution), keep)
    return keep[:m].copy()


def voxel_indices(points, resolution):
    points = np.ascontiguousarray(points, np.float32)
    n, stride = points.shape
    out = np.zeros((n, 3), np.int32)
    lib().orc_voxel_indices(points, n, stride, np.float32(resolution), out)
    return out


def adaptive_voxel_filter(points, max_length, min_num_points, max_range):
    points = np.ascontiguousarray(points, np.float32)
    n, stride = points.shape
    keep = np.zeros(max(n, 1), np.int64)
    passes = np.zeros(32, np.float32)
    npass = C.c_int(0)
    m = lib().orc_adaptive_voxel_filter(points, n, stride, max_length, min_num_points, max_range, keep, passes,
                                        C.byref(npass))
    return keep[:m].copy(), passes[:npass.value].copy()


def rtcsm_match(grid, points, initial_pose, linear_window, angular_window, w_t, w_r, want_scores=False):
    points = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
    out_pose = np.zeros(7)
    best = C.c_int64(-1)
    window = np.zeros(2, np.int32)
    step = np.zeros(2, np.float32)
    scores = None
    sp = None
    if want_scores:
        # upper bound on the candidate count is not known before the call: run once for the window
        lib().orc_rtcsm_match(grid.h, points, len(points), np.ascontiguousarray(initial_pose, np.float64),
                              linear_window, angular_window, w_t, w_r, out_pose, C.byref(best), window, step, None)
        k = (2 * window[0] + 1) ** 3 * (2 * window[1] + 1) ** 3
        scores = np.zeros(int(k), np.float32)
        sp = scores.ctypes.data_as(C.c_void_p)
    score = lib().orc_rtcsm_match(grid.h, points, len(points), np.ascontiguousarray(initial_pose, np.float64),
                                  linear_window, angular_window, w_t, w_r, out_pose, C.byref(best), window, step, sp)
    return {"score": np.float32(score), "pose": out_pose, "best_index": best.value, "linear": int(window[0]),
            "angular": int(window[1]), "angular_step": step[0], "max_scan_range": step[1], "scores": scores}


def _pairs(clouds, grids):
    clouds = [np.ascontiguousarray(c, np.float32).reshape(-1, 3) for c in clouds]
    n = len(clouds)
    cp = (C.c_void_p * n)(*[c.ctypes.data for c in clouds])
    gp = (C.c_void_p * n)(*[g.h.value for g in grids])
    sizes = np.array([len(c) for c in clouds], np.int64)
    return clouds, cp, gp, sizes


def ceres_match(clouds, grids, occ_weights, trans_w, rot_w, target_translation, initial_pose, only_yaw=False,
                nonmono=False, max_iter=12):
    clouds, cp, gp, sizes = _pairs(clouds, grids)
    out_pose = np.zeros(7)
    s = SolveSummary()
    costs = np.full(max_iter + 2, np.nan)
    lib().orc_ceres_match(len(clouds), cp, sizes, gp, np.asarray(occ_weights, np.float64), trans_w, rot_w,
                          int(only_yaw), int(nonmono), max_iter, np.ascontiguousarray(target_translation, np.float64),
                          np.ascontiguousarray(initial_pose, np.float64), out_pose, C.byref(s),
                          costs.ctypes.data_as(C.c_void_p))
    d = s.as_dict()
    d["iteration_costs"] = costs[:s.num_iterations].copy()
    return out_pose, d


def ceres_normal_equations(clouds, grids, occ_weights, trans_w, rot_w, target_translation, reference_pose, at_pose):
    clouds, cp, gp, sizes = _pairs(clouds, grids)
    cost = np.zeros(1)
    g = np.zeros(6)
    h = np.zeros(36)
    lib().orc_ceres_normal_equations(len(clouds), cp, sizes, gp, np.asarray(occ_weights, np.float64), trans_w, rot_w,
                                     np.ascontiguousarray(target_translation, np.float64),
                                     np.ascontiguousarray(reference_pose, np.float64),
                                     np.ascontiguousarray(at_pose, np.float64), cost, g, h)
    return cost[0], g, h.reshape(6, 6)


RANGE_DTYPE = np.dtype([("x", np.float32), ("y", np.float32), ("z", np.float32), ("t", np.float32),
                        ("origin_index", np.uint64), ("_pad", np.uint64)])
assert RANGE_DTYPE.itemsize == 32


def make_ranges(xyzt, origin_index=0):
    r = np.zeros(len(xyzt), RANGE_DTYPE)
    r["x"], r["y"], r["z"], r["t"] = xyzt[:, 0], xyzt[:, 1], xyzt[:, 2], xyzt[:, 3]
    r["origin_index"] = origin_index
    return r


def ingest_scan(opts, ranges, origins, prev_pose, cur_pose):
    n = len(ranges)
    origins = np.ascontiguousarray(origins, np.float32).reshape(-1, 3)
    first_keep = np.zeros(n, np.int64)
    rl, rt, mt = (np.zeros((n, 3), np.float32) for _ in range(3))
    cp = np.zeros(7, np.float32)
    counts = np.zeros(4, np.int64)
    lib().orc_ingest_scan(C.byref(opts), ranges.ctypes.data_as(C.c_void_p), n, origins,
                          np.ascontiguousarray(prev_pose, np.float64), np.ascontiguousarray(cur_pose, np.float64),
                          first_keep, rl, rt, mt, cp, counts)
    return {"first_keep": first_keep[:counts[0]].copy(), "returns_local": rl[:counts[1]].copy(),
            "returns_tracking": rt[:counts[2]].copy(), "misses_tracking": mt[:counts[3]].copy(), "current_pose": cp}


def match_scan(opts, returns_tracking, pose_prediction, submap_local_pose, hi_grid, lo_grid):
    pts = np.ascontiguousarray(returns_tracking, np.float32).reshape(-1, 3)
    n = len(pts)
    obs, est = np.zeros(7), np.zeros(7)
    s = SolveSummary()
    hi_keep, lo_keep = np.zeros(max(n, 1), np.int64), np.zeros(max(n, 1), np.int64)
    counts = np.zeros(2, np.int64)
    score = C.c_float(0)
    ok = lib().orc_match_scan(C.byref(opts), pts, n, np.ascontiguousarray(pose_prediction, np.float64),
                              np.ascontiguousarray(submap_local_pose, np.float64), hi_grid.h, lo_grid.h, obs, est,
                              C.byref(s), hi_keep, lo_keep, counts, C.byref(score))
    return {"ok": bool(ok), "pose_observation_in_submap": obs, "pose_estimate_local": est, "summary": s.as_dict(),
            "hi_keep": hi_keep[:counts[0]].copy(), "lo_keep": lo_keep[:counts[1]].copy(), "rtcsm_score": score.value}


def frontend_batch(opts, ranges_list, origin, prev_poses, cur_poses, submap_local_pose, hi_grid, lo_grid, threads):
    """CPU baseline: the whole per-scan hot path for independent scans over `threads` host threads."""
    n = len(ranges_list)
    rp = (C.c_void_p * n)(*[r.ctypes.data for r in ranges_list])
    sizes = np.array([len(r) for r in ranges_list], np.int64)
    poses = np.zeros((n, 7))
    ok = np.zeros(n, np.int32)
    secs = lib().orc_frontend_batch(C.byref(opts), n, rp, sizes, np.ascontiguousarray(origin, np.float32),
                                    np.ascontiguousarray(prev_poses, np.float64),
                                    np.ascontiguousarray(cur_poses, np.float64),
                                    np.ascontiguousarray(submap_local_pose, np.float64), hi_grid.h, lo_grid.h,
                                    threads, poses, ok)
    return secs, poses, ok


def frontend_batch_imu(opts, ranges_list, origin, noise4, states_i, intervals, submap_local_pose, hi_grid, lo_grid, threads,
                       imu_weight=1.0, gravity=(0.0, 0.0, 9.8)):
    """CPU restatement of dl_frontend_match_batch_imu_samples (pre-integrate -> predict -> ingest -> filters -> fused solve) for
    independent scans on `threads` pooled host threads. intervals: per scan (dt[n], acc[n,3], gyr[n,3]).
    -> (seconds, states [n,16], predicted [n,16], ok [n], iterations [n])."""
    n = len(ranges_list)
    rp = (C.c_void_p * n)(*[r.ctypes.data for r in ranges_list])
    sizes = np.array([len(r) for r in ranges_list], np.int64)
    offsets = np.zeros(n + 1, np.int32)
    for k, iv in enumerate(intervals):
        offsets[k + 1] = offsets[k] + len(iv[0])
    cat = lambda i, w: (np.ascontiguousarray(np.concatenate([np.asarray(iv[i], np.float64).reshape(-1, w) for iv in intervals]))
                        if offsets[-1] else np.zeros((0, w)))
    dt, acc, gyr = cat(0, 1).reshape(-1), cat(1, 3), cat(2, 3)
    states, pred = np.zeros((n, 16)), np.zeros((n, 16))
    ok, iters = np.zeros(n, np.int32), np.zeros(n, np.int32)
    f = lib().orc_frontend_batch_imu
    f.restype = C.c_double
    secs = f(C.byref(opts), C.c_int(n), rp, sizes.ctypes.data_as(C.c_void_p),
             np.ascontiguousarray(origin, np.float32).ctypes.data_as(C.c_void_p),
             np.ascontiguousarray(noise4, np.float64).ctypes.data_as(C.c_void_p),
             np.ascontiguousarray(gravity, np.float64).ctypes.data_as(C.c_void_p), C.c_double(imu_weight),
             np.ascontiguousarray(np.asarray(states_i, np.float64).reshape(n, 16)).ctypes.data_as(C.c_void_p),
             offsets.ctypes.data_as(C.c_void_p), dt.ctypes.data_as(C.c_void_p), acc.ctypes.data_as(C.c_void_p),
             gyr.ctypes.data_as(C.c_void_p), np.ascontiguousarray(submap_local_pose, np.float64).ctypes.data_as(C.c_void_p),
             hi_grid.h, lo_grid.h, C.c_int(threads), states.ctypes.data_as(C.c_void_p), pred.ctypes.data_as(C.c_void_p),
             ok.ctypes.data_as(C.c_void_p), iters.ctypes.data_as(C.c_void_p))
    return secs, states, pred, ok, iters


# ---------------------------------------------------------------- IMU (orc_imu.h)
GRAVITY = np.array([0.0, 0.0, 9.8])


def nav_state(p=(0, 0, 0), q=(1, 0, 0, 0), v=(0, 0, 0), ba=(0, 0, 0), bg=(0, 0, 0)):
    """16 doubles: p(3) q(4 wxyz) v(3) ba(3) bg(3)."""
    return np.array(list(p) + list(q) + list(v) + list(ba) + list(bg), np.float64)


def imu_preintegrate(noise4, ba, bg, dt, acc, gyr):
    m = Preintegration()
    dt = np.ascontiguousarray(dt, np.float64)
    lib().orc_imu_preintegrate(np.ascontiguousarray(noise4, np.float64), np.ascontiguousarray(ba, np.float64),
                               np.ascontiguousarray(bg, np.float64), len(dt), dt,
                               np.ascontiguousarray(acc, np.float64).reshape(-1, 3),
                               np.ascontiguousarray(gyr, np.float64).reshape(-1, 3), C.byref(m))
    return m


def imu_predict(state_i, m, G=GRAVITY):
    out = np.zeros(16)
    lib().orc_imu_predict(np.ascontiguousarray(state_i, np.float64), C.byref(m), np.ascontiguousarray(G, np.float64), out)
    return out


def imu_residual(state_i, state_j, m, G=GRAVITY, jacobian=True):
    r = np.zeros(15)
    J = np.zeros((15, 15))
    lib().orc_imu_residual(np.ascontiguousarray(state_i, np.float64), np.ascontiguousarray(state_j, np.float64),
                           C.byref(m), np.ascontiguousarray(G, np.float64), r,
                           J.ctypes.data_as(C.c_void_p) if jacobian else None)
    return r, J


def window_optimize(mean_i, prior_info, m, matched_pose, sigma_t=0.05, sigma_r=0.01, imu_weight=1.0, G=GRAVITY, max_iter=10,
                    gravity_factor=None, initial_j=None):
    """The fixed-lag smoother standing in for WindowOptimize (orc_window.h). gravity_factor: None or (sigma, direction, body_ref).
    -> (state_i smoothed, state_j, information 15x15, summary dict)."""
    opts = np.array([sigma_t, sigma_r, imu_weight, *G, max_iter, 1.0 if gravity_factor else 0.0,
                     gravity_factor[0] if gravity_factor else 1.0], np.float64)
    dirs = np.array([*(gravity_factor[1] if gravity_factor else (0, 0, 1)), *(gravity_factor[2] if gravity_factor else (0, 0, 1))], np.float64)
    xi, xj, info = np.zeros(16), np.zeros(16), np.zeros(225)
    it, term = C.c_int(0), C.c_int(0)
    costs = np.zeros(2)
    init = np.ascontiguousarray(initial_j, np.float64) if initial_j is not None else None
    f = lib().orc_window_optimize
    ok = f(opts.ctypes.data_as(C.c_void_p), dirs.ctypes.data_as(C.c_void_p),
           np.ascontiguousarray(mean_i, np.float64).ctypes.data_as(C.c_void_p),
           np.ascontiguousarray(prior_info, np.float64).reshape(-1).ctypes.data_as(C.c_void_p), C.byref(m),
           np.ascontiguousarray(matched_pose, np.float64).ctypes.data_as(C.c_void_p),
           init.ctypes.data_as(C.c_void_p) if init is not None else None, xi.ctypes.data_as(C.c_void_p), xj.ctypes.data_as(C.c_void_p),
           info.ctypes.data_as(C.c_void_p), C.byref(it), costs.ctypes.data_as(C.c_void_p), C.byref(term))
    if not ok:
        raise RuntimeError("a covariance or the normal equations are not positive definite")
    return xi, xj, info.reshape(15, 15), {"num_iterations": it.value, "initial_cost": costs[0], "final_cost": costs[1],
                                          "termination": term.value}


def fused_match(clouds, grids, occ_weights, trans_w, rot_w, target_translation, state_i, initial_j, m, G=GRAVITY,
                imu_weight=1.0, nonmono=False, max_iter=12):
    clouds, cp, gp, sizes = _pairs(clouds, grids)
    out = np.zeros(16)
    s = SolveSummary()
    ok = lib().orc_fused_match(len(clouds), cp, sizes, gp, np.asarray(occ_weights, np.float64), trans_w, rot_w,
                               int(nonmono), max_iter, np.ascontiguousarray(target_translation, np.float64),
                               np.ascontiguousarray(state_i, np.float64), np.ascontiguousarray(initial_j, np.float64),
                               C.byref(m), np.ascontiguousarray(G, np.float64), imu_weight, out, C.byref(s))
    if not ok:
        raise RuntimeError("pre-integration covariance is not positive definite")
    return out, s.as_dict()


def fcsm_match_3dof(hi_grid, lo_grid, hi_points, lo_points, pose_guess, min_score, xy_window=5.0, z_window=1.0,
                    min_low_resolution_score=0.55, min_rotational_score=0.77, depth=8, full_depth=3):
    """FastCorrelativeScanMatcher3D::MatchWith3DofInitial with the reference's precomputation stack + branch and bound."""
    hi_points = np.ascontiguousarray(hi_points, np.float32).reshape(-1, 3)
    lo_points = np.ascontiguousarray(lo_points, np.float32).reshape(-1, 3)
    r = FcsmResult()
    lib().orc_fcsm_match_3dof(hi_grid.h, lo_grid.h, depth, full_depth, min_rotational_score, min_low_resolution_score,
                              xy_window, z_window, np.ascontiguousarray(pose_guess, np.float64), hi_points, len(hi_points),
                              lo_points, len(lo_points), np.float32(min_score), C.byref(r))
    return r


class FastCorrelativeScanMatcher:
    """Per-submap matcher object: the precomputation stack is built once (what the reference caches per finished submap);
    match() may be called from several threads."""

    def __init__(self, hi_grid, lo_grid, xy_window=5.0, z_window=1.0, min_low_resolution_score=0.55, min_rotational_score=0.77,
                 depth=8, full_depth=3):
        self.grids = (hi_grid, lo_grid)
        self.h = lib().orc_fcsm_create(hi_grid.h, lo_grid.h, depth, full_depth, min_rotational_score, min_low_resolution_score,
                                       xy_window, z_window)

    def __del__(self):
        if getattr(self, "h", None):
            lib().orc_fcsm_destroy(self.h)
            self.h = None

    def match(self, hi_points, lo_points, pose_guess, min_score):
        hi_points = np.ascontiguousarray(hi_points, np.float32).reshape(-1, 3)
        lo_points = np.ascontiguousarray(lo_points, np.float32).reshape(-1, 3)
        r = FcsmResult()
        lib().orc_fcsm_match(self.h, np.ascontiguousarray(pose_guess, np.float64), hi_points, len(hi_points), lo_points,
                             len(lo_points), np.float32(min_score), C.byref(r))
        return r


TIME_NONE, TIME_FLOAT32_SECONDS, TIME_UINT32_NANOSECONDS, TIME_FLOAT64_SECONDS = 0, 1, 2, 3


def decode_point_cloud2(data, point_step, offsets, time_type, sensor_to_tracking):
    """SensorBridge::HandlePointCloud2Message + HandleRangefinder on raw message bytes -> (rows [k, 4], stamp offset s).
    offsets = (x, y, z, time) byte offsets inside a point."""
    data = np.ascontiguousarray(data, np.uint8).reshape(-1)
    n = len(data) // point_step
    rows = np.zeros((max(n, 1), 4), np.float32)
    off = C.c_double(0)
    k = lib().orc_decode_point_cloud2(point_step, *[int(v) for v in offsets], int(time_type), data.ctypes.data_as(C.c_void_p), n,
                                      np.ascontiguousarray(sensor_to_tracking, np.float64), rows, C.byref(off))
    return rows[:k].copy(), off.value


def fcsm_match_full(hi_grid, lo_grid, hi_points, lo_points, node_pose, submap_pose, min_score, xy_window=5.0, z_window=1.0,
                    angular_window=0.2617993877991494, min_low_resolution_score=0.55, min_rotational_score=0.77, depth=8,
                    full_depth=3, histogram=None, histogram_size=10, submap_histogram=None):
    """FastCorrelativeScanMatcher3D::Match: yaw steps inside the angular window x the translation window."""
    hi_points = np.ascontiguousarray(hi_points, np.float32).reshape(-1, 3)
    lo_points = np.ascontiguousarray(lo_points, np.float32).reshape(-1, 3)
    r = FcsmResult()
    si, ns = C.c_int(0), C.c_int(0)
    hist = None if histogram is None else np.ascontiguousarray(histogram, np.float32)
    sub = None if submap_histogram is None else np.ascontiguousarray(submap_histogram, np.float32)
    lib().orc_fcsm_match_full(hi_grid.h, lo_grid.h, depth, full_depth, min_rotational_score, min_low_resolution_score, xy_window,
                              z_window, angular_window, np.ascontiguousarray(node_pose, np.float64),
                              np.ascontiguousarray(submap_pose, np.float64), hi_points, len(hi_points), lo_points, len(lo_points),
                              None if hist is None else hist.ctypes.data_as(C.c_void_p), histogram_size if hist is None else len(hist),
                              np.float32(min_score), C.byref(r), C.byref(si), C.byref(ns),
                              None if sub is None else sub.ctypes.data_as(C.c_void_p))
    return r, si.value, ns.value


def rotational_match(submap_histogram, histogram, initial_angle, angles, submap_angle=0.0):
    sh = np.ascontiguousarray(submap_histogram, np.float32)
    h = np.ascontiguousarray(histogram, np.float32)
    a = np.ascontiguousarray(angles, np.float32)
    out = np.zeros(len(a), np.float32)
    lib().orc_rotational_match(sh, len(sh), np.float32(submap_angle), h, np.float32(initial_angle), a, len(a), out)
    return out


def compute_histogram(points, size):
    p = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
    out = np.zeros(size, np.float32)
    lib().orc_compute_histogram(p, len(p), size, out)
    return out


def pose_graph_solve(submap_poses, node_poses, constraints, fix_z=False, max_iter=50, linear_solver="normal_cholesky"):
    """OptimizationProblem3D::Solve reduced to what this fork keeps active: SPA constraints only.
    constraints: iterable of (submap_index, node_index, zbar_ij pose7, translation_weight, rotation_weight).
    Returns (submap poses, node poses, summary dict)."""
    S, N = len(submap_poses), len(node_poses)
    poses = np.ascontiguousarray(np.concatenate([np.asarray(submap_poses, np.float64).reshape(S, 7),
                                                 np.asarray(node_poses, np.float64).reshape(N, 7)]))
    cs = list(constraints)
    idx = np.ascontiguousarray([[c[0], c[1]] for c in cs], np.int32).reshape(-1, 2)
    zbar = np.ascontiguousarray([c[2] for c in cs], np.float64).reshape(-1, 7)
    w = np.ascontiguousarray([[c[3], c[4]] for c in cs], np.float64).reshape(-1, 2)
    s = SolveSummary()
    lib().orc_pose_graph_solve(S, N, poses, len(cs), idx, zbar, w, int(fix_z), max_iter, C.byref(s),
                               {"dense_qr": 0, "normal_cholesky": 1}[linear_solver])
    return poses[:S].copy(), poses[S:].copy(), s.as_dict()


def spa_residual(pose_i, pose_j, zbar, translation_weight, rotation_weight):
    e, jac = np.zeros(6), np.zeros(84)
    lib().orc_spa_residual(np.ascontiguousarray(pose_i, np.float64), np.ascontiguousarray(pose_j, np.float64),
                           np.ascontiguousarray(zbar, np.float64), translation_weight, rotation_weight, e, jac)
    return e, jac.reshape(6, 14)


def rotation_delta_cost(scale, target_q, q):
    return lib().orc_rotation_delta_cost(float(scale), np.ascontiguousarray(target_q, np.float64), np.ascontiguousarray(q, np.float64))


def precomputation_values(grid, depth, cells):
    xyz = np.ascontiguousarray(cells, np.int32).reshape(-1, 3)
    out = np.zeros(len(xyz), np.int32)
    lib().orc_precomputation_values(grid.h, depth, len(xyz), xyz, out)
    return out


def angle_of_angle_axis_f(aa):
    return float(lib().orc_angle_of_angle_axis_f(np.ascontiguousarray(aa, np.float32)))
