"""ctypes binding of libdliom_b200.so (the C-ABI in include/dliom_b200.h) for tests and bench.py.

The product is the shared library; this module only marshals numpy arrays into its plain-pointer signatures.
There is no fallback: if the library is missing, or no CUDA device is present, calls raise.
"""
import ctypes as C
import math
import os
import struct

import numpy as np

_PKG = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(_PKG, "libdliom_b200.so")
_LIB = None

f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
f64p = np.ctypeslib.ndpointer(np.float64, flags="C_CONTIGUOUS")
i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
i64p = np.ctypeslib.ndpointer(np.int64, flags="C_CONTIGUOUS")
u16p = np.ctypeslib.ndpointer(np.uint16, flags="C_CONTIGUOUS")

DL_MAX_PAIRS = 4
EXPORTS = [
    "dl_context_create", "dl_context_destroy", "dl_last_error", "dl_status_string", "dl_context_kernel_launches",
    "dl_context_stream", "dl_context_synchronize", "dl_context_set_profiling", "dl_context_set_blocking_sync", "dl_context_read_profile", "dl_grid_create", "dl_grid_destroy", "dl_grid_set_cells",
    "dl_grid_sync", "dl_grid_resolution", "dl_grid_num_bricks", "dl_grid_lookup", "dl_grid_interpolate",
    "dl_grid_insert_range_data", "dl_submap_insert_range_data", "dl_grid_export_cells",
    "dl_voxel_filter", "dl_voxel_indices", "dl_adaptive_voxel_filter", "dl_rtcsm_match", "dl_fcsm_match_3dof", "dl_fcsm_match", "dl_constraint_search_batch", "dl_ceres_match",
    "dl_ceres_match_batch", "dl_ceres_normal_equations", "dl_imu_preintegrate", "dl_imu_predict", "dl_imu_factor_evaluate", "dl_fused_match_batch", "dl_ingest_scan", "dl_decode_point_cloud2", "dl_decode_point_cloud2_dev", "dl_frontend_match_batch", "dl_frontend_match_batch_imu", "dl_frontend_submit", "dl_frontend_collect",
    "dl_frontend_match_batch_dev", "dl_frontend_fetch_results", "dl_device_alloc", "dl_device_free",
    "dl_copy_to_device", "dl_copy_to_host",
    "dl_frontend_match_batch_imu_samples", "dl_frontend_match_batch_imu_samples_dev", "dl_frontend_submit_imu_samples",
    "dl_frontend_collect_imu",
    "dl_comm_unique_id", "dl_comm_create", "dl_comm_destroy", "dl_comm_rank", "dl_comm_world_size", "dl_comm_last_error",
    "dl_comm_all_gather_dev", "dl_comm_all_reduce_f64_dev", "dl_comm_broadcast_dev", "dl_constraint_search_exchange",
    "dl_pose_graph_solve_sparse", "dl_pose_graph_evaluate", "dl_window_optimize_batch", "dl_window_evaluate", "dl_rotational_histogram", "dl_ltb_create", "dl_ltb_destroy", "dl_ltb_set_initial_state", "dl_ltb_add_imu_data",
    "dl_ltb_add_range_data", "dl_ltb_add_synchronized_range_data", "dl_ltb_get_cloud", "dl_ltb_get_histogram", "dl_ltb_num_submaps", "dl_ltb_get_submap", "dl_ltb_get_state",
    "dl_ltb_add_range_data_batch", "dl_ltb_release_submap",
    "dl_pose_graph_3d_create", "dl_pose_graph_3d_destroy", "dl_pose_graph_3d_add_node", "dl_pose_graph_3d_freeze_trajectory",
    "dl_pose_graph_3d_run_final_optimization", "dl_pose_graph_3d_poses", "dl_pose_graph_3d_local_to_global",
    "dl_pose_graph_3d_constraints", "dl_pose_graph_3d_last_searches", "dl_pose_graph_3d_store_bytes",
    "dl_pg3d_trim_submap", "dl_pg3d_add_pure_localization_trimmer", "dl_pg3d_finish_trajectory", "dl_pg3d_is_trajectory_finished",
    "dl_pg3d_set_initial_trajectory_pose", "dl_pg3d_ids", "dl_pg3d_last_trimmed", "dl_pg3d_store_usage",
    "dl_range_data_map_set_node", "dl_range_data_map", "dl_range_data_map_dev",
    "dl_map_writer_create", "dl_map_writer_destroy", "dl_map_writer_add_trajectory", "dl_map_writer_process",
    "dl_map_writer_process_dev", "dl_map_writer_flush", "dl_map_writer_voxels", "dl_map_writer_add_color",
    "dl_map_writer_add_xray", "dl_map_writer_xray_image", "dl_map_writer_add_probability_grid", "dl_map_writer_probability_grid",
    "dl_submap_textures", "dl_submap_projections",
]


class DlError(RuntimeError):
    def __init__(self, status, message):
        super().__init__(f"dliom_b200 status {status}: {message}")
        self.status = status


class StageTime(C.Structure):
    _fields_ = [("name", C.c_char * 32), ("ms", C.c_double), ("calls", C.c_int64)]


class AdaptiveVoxelFilterOptions(C.Structure):
    _fields_ = [("max_length", C.c_float), ("min_num_points", C.c_float), ("max_range", C.c_float)]


class RtcsmOptions(C.Structure):
    _fields_ = [("linear_search_window", C.c_double), ("angular_search_window", C.c_double),
                ("translation_delta_cost_weight", C.c_double), ("rotation_delta_cost_weight", C.c_double)]


class RtcsmInfo(C.Structure):
    _fields_ = [("best_index", C.c_int64), ("num_candidates", C.c_int64), ("linear_window", C.c_int32),
                ("angular_window", C.c_int32), ("angular_step", C.c_float), ("max_scan_range", C.c_float)]


class RangeDataInserterOptions(C.Structure):
    _fields_ = [("hit_probability", C.c_double), ("miss_probability", C.c_double), ("num_free_space_voxels", C.c_int32),
                ("reserved", C.c_int32)]


class ImuNoise(C.Structure):
    _fields_ = [("acc_n", C.c_double), ("gyr_n", C.c_double), ("acc_w", C.c_double), ("gyr_w", C.c_double)]


class Preintegration(C.Structure):
    _fields_ = [("sum_dt", C.c_double), ("delta_p", C.c_double * 3), ("delta_q", C.c_double * 4),
                ("delta_v", C.c_double * 3), ("linearized_ba", C.c_double * 3), ("linearized_bg", C.c_double * 3),
                ("jacobian", C.c_double * 225), ("covariance", C.c_double * 225)]


class NavState(C.Structure):
    _fields_ = [("p", C.c_double * 3), ("q", C.c_double * 4), ("v", C.c_double * 3), ("ba", C.c_double * 3),
                ("bg", C.c_double * 3)]

    @staticmethod
    def from16(x):
        s = NavState()
        s.p[:], s.q[:], s.v[:], s.ba[:], s.bg[:] = x[0:3], x[3:7], x[7:10], x[10:13], x[13:16]
        return s

    def to16(self):
        return np.array(list(self.p) + list(self.q) + list(self.v) + list(self.ba) + list(self.bg))


class FcsmOptions(C.Structure):
    _fields_ = [("branch_and_bound_depth", C.c_int32), ("full_resolution_depth", C.c_int32),
                ("min_rotational_score", C.c_double), ("min_low_resolution_score", C.c_double),
                ("linear_xy_search_window", C.c_double), ("linear_z_search_window", C.c_double),
                ("angular_search_window", C.c_double)]


class FcsmResult(C.Structure):
    _fields_ = [("found", C.c_int32), ("score", C.c_float), ("pose_estimate", C.c_double * 7),
                ("rotational_score", C.c_float), ("low_resolution_score", C.c_float), ("offset", C.c_int32 * 3),
                ("scan_index", C.c_int32), ("num_candidates", C.c_int64)]


class CeresOptions(C.Structure):
    _fields_ = [("num_occupied_space_weights", C.c_int32), ("occupied_space_weight", C.c_double * DL_MAX_PAIRS),
                ("translation_weight", C.c_double), ("rotation_weight", C.c_double), ("only_optimize_yaw", C.c_int32),
                ("use_nonmonotonic_steps", C.c_int32), ("max_num_iterations", C.c_int32), ("num_threads", C.c_int32)]

    @staticmethod
    def make(occ, trans_w, rot_w, only_yaw=False, nonmono=False, max_iter=12):
        o = CeresOptions()
        o.num_occupied_space_weights = len(occ)
        for i, w in enumerate(occ):
            o.occupied_space_weight[i] = w
        o.translation_weight, o.rotation_weight = trans_w, rot_w
        o.only_optimize_yaw, o.use_nonmonotonic_steps = int(only_yaw), int(nonmono)
        o.max_num_iterations, o.num_threads = max_iter, 1
        return o


class SolveSummary(C.Structure):
    _fields_ = [("initial_cost", C.c_double), ("final_cost", C.c_double), ("num_iterations", C.c_int32),
                ("num_successful_steps", C.c_int32), ("num_unsuccessful_steps", C.c_int32),
                ("termination", C.c_int32), ("num_evaluations", C.c_int32), ("reserved", C.c_int32)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_ if k != "reserved"}


class PointCloud2Layout(C.Structure):
    _fields_ = [("point_step", C.c_int32), ("offset_x", C.c_int32), ("offset_y", C.c_int32), ("offset_z", C.c_int32),
                ("offset_time", C.c_int32), ("time_type", C.c_int32)]


TIME_NONE, TIME_FLOAT32_SECONDS, TIME_UINT32_NANOSECONDS, TIME_FLOAT64_SECONDS = 0, 1, 2, 3


class FrontendImu(C.Structure):
    _fields_ = [("imu_weight", C.c_double), ("gravity", C.c_double * 3), ("states_i", C.c_void_p),
                ("predicted_states", C.c_void_p), ("preintegrations", C.c_void_p), ("states_out", C.c_void_p)]


class ConstraintOptions(C.Structure):
    _fields_ = [("min_score", C.c_double), ("loop_closure_translation_weight", C.c_double),
                ("loop_closure_rotation_weight", C.c_double), ("fast_correlative_scan_matcher_3d", FcsmOptions),
                ("ceres_scan_matcher_3d", CeresOptions)]

    @staticmethod
    def defaults(**kw):
        """constraint_builder block of configuration_files/pose_graph.lua:17-73."""
        o = ConstraintOptions()
        o.min_score = kw.pop("min_score", 0.55)
        o.loop_closure_translation_weight, o.loop_closure_rotation_weight = 1.1e4, 1e5
        o.fast_correlative_scan_matcher_3d = FcsmOptions(8, 3, 0.77, kw.pop("min_low_resolution_score", 0.55),
                                                         kw.pop("xy_window", 5.0), kw.pop("z_window", 1.0), 0.2617993877991494)
        o.ceres_scan_matcher_3d = CeresOptions.make([5.0, 30.0], 10.0, 1.0, False, False, 10)
        assert not kw, kw
        return o


class Constraint(C.Structure):
    _fields_ = [("found", C.c_int32), ("score", C.c_float), ("rotational_score", C.c_float),
                ("low_resolution_score", C.c_float), ("coarse_pose", C.c_double * 7), ("pose", C.c_double * 7),
                ("translation_weight", C.c_double), ("rotation_weight", C.c_double), ("summary", SolveSummary)]


class ConstraintRow(C.Structure):   # dl_constraint_row, 96 bytes
    _fields_ = [("submap_id", C.c_int32), ("node_id", C.c_int32), ("found", C.c_int32), ("rank", C.c_int32),
                ("score", C.c_float), ("low_resolution_score", C.c_float), ("pose", C.c_double * 7),
                ("translation_weight", C.c_double), ("rotation_weight", C.c_double)]


class ExchangeInfo(C.Structure):
    _fields_ = [("bytes_sent", C.c_int64), ("bytes_received", C.c_int64), ("collective_ms", C.c_float),
                ("found_total", C.c_int32)]


class FrontendOptions(C.Structure):
    _fields_ = [("min_range", C.c_float), ("max_range", C.c_float), ("voxel_filter_size", C.c_float),
                ("high_resolution_adaptive_voxel_filter", AdaptiveVoxelFilterOptions),
                ("low_resolution_adaptive_voxel_filter", AdaptiveVoxelFilterOptions),
                ("use_online_correlative_scan_matching", C.c_int32), ("range_row_floats", C.c_int32),
                ("scan_period", C.c_double),
                ("real_time_correlative_scan_matcher", RtcsmOptions), ("ceres_scan_matcher", CeresOptions),
                ("host_scan_stride_rows", C.c_int64), ("time_run_offsets", C.c_void_p), ("time_run_first_row", C.c_void_p),
                ("time_run_value", C.c_void_p)]

    @staticmethod
    def from_oracle(o):
        """Same parameters as an oracle FrontEndOptions block (oracle/orc.py), field for field."""
        f = FrontendOptions()
        f.min_range, f.max_range, f.voxel_filter_size = o.min_range, o.max_range, o.voxel_filter_size
        f.high_resolution_adaptive_voxel_filter = AdaptiveVoxelFilterOptions(o.hi_max_length, o.hi_min_num_points,
                                                                             o.hi_max_range)
        f.low_resolution_adaptive_voxel_filter = AdaptiveVoxelFilterOptions(o.lo_max_length, o.lo_min_num_points,
                                                                            o.lo_max_range)
        f.use_online_correlative_scan_matching = o.use_rtcsm
        f.range_row_floats = 8
        f.scan_period = o.scan_period
        f.real_time_correlative_scan_matcher = RtcsmOptions(o.rtcsm_linear_window, o.rtcsm_angular_window, o.rtcsm_w_t,
                                                            o.rtcsm_w_r)
        f.ceres_scan_matcher = CeresOptions.make([o.occ_w0, o.occ_w1], o.trans_w, o.rot_w, o.only_yaw, o.nonmono,
                                                 o.max_iter)
        return f


class ScanResult(C.Structure):
    _fields_ = [("pose_estimate_local", C.c_double * 7), ("pose_observation_in_submap", C.c_double * 7),
                ("summary", SolveSummary), ("rtcsm_score", C.c_float), ("ok", C.c_int32),
                ("num_first_filter", C.c_int32), ("num_returns", C.c_int32), ("num_misses", C.c_int32),
                ("num_high_resolution", C.c_int32), ("num_low_resolution", C.c_int32),
                ("num_cropped_high", C.c_int32), ("num_cropped_low", C.c_int32), ("num_passes_high", C.c_int32),
                ("num_passes_low", C.c_int32), ("reserved", C.c_int32)]


class ImuSamples:
    """dl_frontend_imu_samples + the arrays it points to (kept alive with the object). intervals: per scan (dt[n], acc[n,3],
    gyr[n,3]); states_i: per scan 16-vectors (p q v ba bg) at the previous scan."""

    class Struct(C.Structure):
        _fields_ = [("noise", ImuNoise), ("imu_weight", C.c_double), ("gravity", C.c_double * 3), ("states_i", C.c_void_p),
                    ("offsets", C.c_void_p), ("dt", C.c_void_p), ("acc", C.c_void_p), ("gyr", C.c_void_p)]

    def __init__(self, noise4, intervals, states_i, imu_weight=1.0, gravity=(0.0, 0.0, 9.8), pin=False):
        n = len(intervals)
        self.n = n
        self.offsets = np.zeros(n + 1, np.int32)
        for k, (dt, _, _) in enumerate(intervals):
            self.offsets[k + 1] = self.offsets[k] + len(dt)
        cat = lambda i, w: (np.ascontiguousarray(np.concatenate([np.asarray(iv[i], np.float64).reshape(-1, w) for iv in intervals]))
                            if n and self.offsets[-1] else np.zeros((0, w)))
        self.dt, self.acc, self.gyr = cat(0, 1).reshape(-1), cat(1, 3), cat(2, 3)
        self.states = np.ascontiguousarray(np.asarray(states_i, np.float64).reshape(n, 16))
        if pin:   # page-lock the arrays so the streaming submit's uploads are truly asynchronous
            import torch
            self._pinned = [torch.from_numpy(a).pin_memory() for a in (self.dt, self.acc, self.gyr, self.states)]
            self.dt, self.acc, self.gyr, self.states = [t.numpy() for t in self._pinned]
        self.struct = ImuSamples.Struct(ImuNoise(*[float(v) for v in noise4]), float(imu_weight), (C.c_double * 3)(*gravity),
                                        self.states.ctypes.data, self.offsets.ctypes.data, self.dt.ctypes.data,
                                        self.acc.ctypes.data, self.gyr.ctypes.data)


class WindowOptions(C.Structure):   # dl_window_options
    _fields_ = [("pose_sigma_translation", C.c_double), ("pose_sigma_rotation", C.c_double), ("imu_weight", C.c_double),
                ("gravity", C.c_double * 3), ("max_num_iterations", C.c_int32), ("use_gravity_factor", C.c_int32),
                ("gravity_sigma", C.c_double), ("gravity_direction", C.c_double * 3), ("body_reference_direction", C.c_double * 3)]


class SpaConstraint(C.Structure):   # dl_spa_constraint
    _fields_ = [("submap", C.c_int32), ("node", C.c_int32), ("zbar", C.c_double * 7), ("translation_weight", C.c_double),
                ("rotation_weight", C.c_double)]


class PoseGraphOptions(C.Structure):
    _fields_ = [("max_num_iterations", C.c_int32), ("fix_z", C.c_int32)]


class PoseGraphSparseInfo(C.Structure):   # dl_pose_graph_sparse_info
    _fields_ = [("num_local_parameters", C.c_int32), ("all_reduce_count", C.c_int32), ("all_reduce_bytes", C.c_int64),
                ("all_reduce_ms", C.c_float), ("all_reduce_min_ms", C.c_float), ("num_reduced_parameters", C.c_int32),
                ("num_pairs", C.c_int32), ("setup_exchange_bytes", C.c_int64)]


class LtbOptions(C.Structure):   # dl_ltb_options
    _fields_ = [("frontend", FrontendOptions), ("imu_noise", ImuNoise), ("imu_weight", C.c_double), ("gravity", C.c_double),
                ("high_resolution", C.c_float), ("low_resolution", C.c_float), ("num_range_data", C.c_int32),
                ("high_resolution_max_range", C.c_int32), ("range_data_inserter", RangeDataInserterOptions),
                ("motion_filter_max_time_seconds", C.c_double), ("motion_filter_max_distance_meters", C.c_double),
                ("motion_filter_max_angle_radians", C.c_double), ("rotational_histogram_size", C.c_int32),
                ("frames_for_static_initialization", C.c_int32), ("two_stage", C.c_int32), ("reserved", C.c_int32),
                ("ceres_pose_noise_t", C.c_double), ("ceres_pose_noise_r", C.c_double), ("prior_pose_noise", C.c_double),
                ("prior_velocity_noise", C.c_double), ("prior_bias_noise", C.c_double)]

    @staticmethod
    def defaults(frontend, noise4, **kw):
        """trajectory_builder_3d.lua defaults: submaps 0.1 / 0.45 m, 20 m, 160 range data; motion filter 0.5 s / 0.1 m / 0.004 rad."""
        o = LtbOptions()
        o.frontend = frontend
        o.imu_noise = ImuNoise(*[float(v) for v in noise4])
        o.imu_weight, o.gravity = kw.pop("imu_weight", 1.0), kw.pop("gravity", 9.8)
        o.high_resolution, o.low_resolution = kw.pop("high_resolution", 0.1), kw.pop("low_resolution", 0.45)
        o.num_range_data, o.high_resolution_max_range = kw.pop("num_range_data", 160), kw.pop("high_resolution_max_range", 20)
        o.range_data_inserter = RangeDataInserterOptions(kw.pop("hit", 0.55), kw.pop("miss", 0.49), kw.pop("num_free", 2), 0)
        o.motion_filter_max_time_seconds = kw.pop("max_time_seconds", 0.5)
        o.motion_filter_max_distance_meters = kw.pop("max_distance_meters", 0.1)
        o.motion_filter_max_angle_radians = kw.pop("max_angle_radians", 0.004)
        o.rotational_histogram_size = kw.pop("rotational_histogram_size", 120)
        o.frames_for_static_initialization = kw.pop("frames_for_static_initialization", 7)
        o.two_stage = int(kw.pop("two_stage", 0))
        # the correlative pre-match (LTB:514-521) and the yaw-only solve, over what `frontend` carries
        if "use_rtcsm" in kw:
            o.frontend.use_online_correlative_scan_matching = int(kw.pop("use_rtcsm"))
        if "rtcsm" in kw:   # (linear_search_window, angular_search_window, translation / rotation_delta_cost_weight)
            o.frontend.real_time_correlative_scan_matcher = RtcsmOptions(*[float(v) for v in kw.pop("rtcsm")])
        if "only_optimize_yaw" in kw:
            o.frontend.ceres_scan_matcher.only_optimize_yaw = int(kw.pop("only_optimize_yaw"))
        o.ceres_pose_noise_t, o.ceres_pose_noise_r = kw.pop("ceres_pose_noise_t", 1e-2), kw.pop("ceres_pose_noise_r", 1e-2)
        o.prior_pose_noise = kw.pop("prior_pose_noise", 1e-2)
        o.prior_velocity_noise, o.prior_bias_noise = kw.pop("prior_velocity_noise", 1e4), kw.pop("prior_bias_noise", 1e-2)
        assert not kw, kw
        return o


class MatchingResult(C.Structure):   # dl_matching_result
    _fields_ = [("has_result", C.c_int32), ("inserted", C.c_int32), ("time", C.c_double), ("local_pose", C.c_double * 7),
                ("state", NavState), ("scan", ScanResult), ("origin_in_local", C.c_float * 3), ("num_returns", C.c_int32),
                ("num_misses", C.c_int32), ("num_high_resolution", C.c_int32), ("num_low_resolution", C.c_int32),
                ("num_insertion_submaps", C.c_int32), ("insertion_submap_index", C.c_int32 * 2), ("reserved", C.c_int32)]

    @property
    def rtcsm_score(self):
        """The correlative pre-match's best score (0 when use_online_correlative_scan_matching is off)."""
        return self.scan.rtcsm_score


class LtbBatchItem(C.Structure):   # dl_ltb_batch_item
    _fields_ = [("builder", C.c_void_p), ("time", C.c_double), ("rows", C.c_void_p), ("n", C.c_int64), ("row_floats", C.c_int32),
                ("num_origins", C.c_int32), ("origins", C.c_void_p)]


class PoseGraph3DOptions(C.Structure):   # dl_pose_graph_3d_options
    _fields_ = [("optimize_every_n_nodes", C.c_int32), ("every_nodes_to_find_constraint", C.c_int32),
                ("matcher_translation_weight", C.c_double), ("matcher_rotation_weight", C.c_double),
                ("constraint_builder", ConstraintOptions), ("optimization_problem", PoseGraphOptions)]

    @staticmethod
    def defaults(optimize_every_n_nodes=90, every_nodes_to_find_constraint=5, max_num_iterations=50, fix_z=False, **kw):
        """pose_graph.lua: matcher weights 5e2 / 1.6e3, optimize_every_n_nodes 90, every_nodes_to_find_constraint 5, 50 iterations; kw go to
        ConstraintOptions.defaults."""
        return PoseGraph3DOptions(int(optimize_every_n_nodes), int(every_nodes_to_find_constraint), 5e2, 1.6e3,
                                  ConstraintOptions.defaults(**kw), PoseGraphOptions(int(max_num_iterations), int(bool(fix_z))))


class Pg3dInsertionSubmap(C.Structure):   # dl_pg3d_insertion_submap
    _fields_ = [("submap_index", C.c_int32), ("finished", C.c_int32), ("high_resolution_grid", C.c_void_p),
                ("low_resolution_grid", C.c_void_p), ("local_pose", C.c_double * 7)]


class Pg3dNode(C.Structure):   # dl_pg3d_node
    _fields_ = [("trajectory_id", C.c_int32), ("num_insertion_submaps", C.c_int32), ("time", C.c_double),
                ("local_pose", C.c_double * 7), ("high_resolution_points", C.c_void_p), ("num_high_resolution", C.c_int64),
                ("low_resolution_points", C.c_void_p), ("num_low_resolution", C.c_int64),
                ("insertion_submaps", Pg3dInsertionSubmap * 2)]


class Pg3dSubmapMatch(C.Structure):   # dl_pg3d_submap_match
    _fields_ = [("trajectory_id", C.c_int32), ("submap_index", C.c_int32), ("x", C.c_double), ("y", C.c_double),
                ("theta", C.c_double)]


class Pg3dAddNodeInfo(C.Structure):   # dl_pg3d_add_node_info
    _fields_ = [("node_index", C.c_int32), ("num_searched", C.c_int32), ("num_found", C.c_int32), ("optimized", C.c_int32),
                ("cloud_bytes_uploaded", C.c_int64), ("bookkeeping_ms", C.c_double), ("search_ms", C.c_double),
                ("solve_ms", C.c_double), ("summary", SolveSummary)]


class Pg3dConstraint(C.Structure):   # dl_pg3d_constraint
    _fields_ = [("submap_trajectory_id", C.c_int32), ("submap_index", C.c_int32), ("node_trajectory_id", C.c_int32),
                ("node_index", C.c_int32), ("zbar", C.c_double * 7), ("translation_weight", C.c_double),
                ("rotation_weight", C.c_double), ("tag", C.c_int32), ("reserved", C.c_int32)]


class Pg3dSearch(C.Structure):   # dl_pg3d_search
    _fields_ = [("submap_trajectory_id", C.c_int32), ("submap_index", C.c_int32), ("node_trajectory_id", C.c_int32),
                ("node_index", C.c_int32), ("pose_guess", C.c_double * 7), ("result", Constraint)]


class Pg3dSubmapId(C.Structure):   # dl_pg3d_submap_id
    _fields_ = [("trajectory_id", C.c_int32), ("submap_index", C.c_int32)]


class RangeDataMapNode(C.Structure):   # dl_range_data_map_node
    _fields_ = [("trajectory_id", C.c_int32), ("node_index", C.c_int32), ("first_point", C.c_int64), ("num_points", C.c_int64),
                ("global_pose", C.c_double * 7)]


class MapWriterOptions(C.Structure):   # dl_map_writer_options
    _fields_ = [("range_filter", C.c_int32), ("reserved", C.c_int32), ("min_range", C.c_double), ("max_range", C.c_double),
                ("outlier_voxel_size", C.c_double)]


class MapMessage(C.Structure):   # dl_map_message
    _fields_ = [("stamp", C.c_int64), ("first_row", C.c_int64), ("num_rows", C.c_int64), ("trajectory_id", C.c_int32),
                ("frame_id", C.c_int32), ("sensor_to_tracking", C.c_double * 7)]


class MapWriterColor(C.Structure):   # dl_map_writer_color
    _fields_ = [("frame_id", C.c_int32), ("rgb", C.c_uint8 * 3), ("pad", C.c_uint8)]


class MapWriterXray(C.Structure):   # dl_map_writer_xray
    _fields_ = [("voxel_size", C.c_double), ("transform", C.c_double * 7)]


class MapWriterGridOptions(C.Structure):   # dl_map_writer_grid_options
    _fields_ = [("resolution", C.c_double), ("hit_probability", C.c_double), ("miss_probability", C.c_double),
                ("insert_free_space", C.c_int32), ("reserved", C.c_int32)]


class MapWriterGridInfo(C.Structure):   # dl_map_writer_grid_info
    _fields_ = [("resolution", C.c_double), ("max_x", C.c_double), ("max_y", C.c_double), ("num_x_cells", C.c_int32),
                ("num_y_cells", C.c_int32), ("offset_x", C.c_int32), ("offset_y", C.c_int32), ("width", C.c_int32),
                ("height", C.c_int32)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class MapWriterInfo(C.Structure):   # dl_map_writer_info
    _fields_ = [("pass_", C.c_int32), ("final_pass", C.c_int32), ("num_rows", C.c_int64), ("dropped_no_pose", C.c_int64),
                ("dropped_range", C.c_int64), ("dropped_moving", C.c_int64), ("messages_without_batch", C.c_int64),
                ("num_samples", C.c_int64), ("num_points_out", C.c_int64)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


PG3D_INTRA_SUBMAP, PG3D_INTER_SUBMAP = 0, 1
PG3D_NODE_POSES, PG3D_SUBMAP_POSES, PG3D_OPTIMIZATION_NODES, PG3D_OPTIMIZATION_SUBMAPS = 0, 1, 2, 3


class SubmapImageQuery(C.Structure):   # dl_submap_image_query
    _fields_ = [("grid", C.c_void_p), ("pose", C.c_double * 7)]


class SubmapTexture(C.Structure):   # dl_submap_texture
    _fields_ = [("resolution", C.c_float), ("width", C.c_int32), ("height", C.c_int32), ("reserved", C.c_int32),
                ("slice_pose", C.c_double * 7), ("offset", C.c_int64)]


class SubmapProjection(C.Structure):   # dl_submap_projection
    _fields_ = [("resolution", C.c_float), ("width", C.c_int32), ("height", C.c_int32), ("reserved", C.c_int32),
                ("ox", C.c_double), ("oy", C.c_double), ("offset", C.c_int64)]


def spa_constraints(constraints):
    """(submap, node, zbar7, translation_weight, rotation_weight) tuples -> a dl_spa_constraint array (numpy-packed: graphs of
    tens of thousands of constraints)."""
    n = len(constraints)
    arr = np.zeros(max(n, 1), dtype=np.dtype([("submap", np.int32), ("node", np.int32), ("zbar", np.float64, 7),
                                               ("tw", np.float64), ("rw", np.float64)], align=True))
    if n:
        arr["submap"][:n] = [c[0] for c in constraints]
        arr["node"][:n] = [c[1] for c in constraints]
        arr["zbar"][:n] = np.asarray([c[2] for c in constraints], np.float64).reshape(n, 7)
        arr["tw"][:n] = [c[3] for c in constraints]
        arr["rw"][:n] = [c[4] for c in constraints]
    assert arr.dtype.itemsize == C.sizeof(SpaConstraint)
    return (SpaConstraint * len(arr)).from_buffer(arr)


def lib():
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` first")
    L = C.CDLL(LIB_PATH)
    vp, ip = C.c_void_p, C.POINTER
    L.dl_context_create.argtypes = [C.c_int, ip(vp)]
    L.dl_context_destroy.argtypes = [vp]
    L.dl_context_destroy.restype = None
    L.dl_last_error.argtypes = [vp]
    L.dl_last_error.restype = C.c_char_p
    L.dl_status_string.argtypes = [C.c_int]
    L.dl_status_string.restype = C.c_char_p
    L.dl_context_kernel_launches.argtypes = [vp]
    L.dl_context_kernel_launches.restype = C.c_int64
    L.dl_context_stream.argtypes = [vp]
    L.dl_context_stream.restype = C.c_uint64
    L.dl_context_synchronize.argtypes = [vp]
    L.dl_context_set_profiling.argtypes = [vp, C.c_int]
    L.dl_context_set_blocking_sync.argtypes = [vp, C.c_int]
    L.dl_context_read_profile.argtypes = [vp, ip(StageTime), C.c_int32, ip(C.c_int32)]
    L.dl_grid_create.argtypes = [vp, C.c_float, ip(vp)]
    L.dl_grid_destroy.argtypes = [vp]
    L.dl_grid_destroy.restype = None
    L.dl_grid_set_cells.argtypes = [vp, C.c_int64, i32p, i32p, i32p, u16p]
    L.dl_grid_sync.argtypes = [vp]
    L.dl_grid_resolution.argtypes = [vp]
    L.dl_grid_resolution.restype = C.c_float
    L.dl_grid_num_bricks.argtypes = [vp]
    L.dl_grid_num_bricks.restype = C.c_int64
    L.dl_grid_lookup.argtypes = [vp, vp, C.c_int64, i32p, u16p]
    L.dl_grid_interpolate.argtypes = [vp, vp, C.c_int64, f64p, f64p]
    L.dl_grid_insert_range_data.argtypes = [vp, vp, ip(RangeDataInserterOptions), f32p, f32p, C.c_int64]
    L.dl_submap_insert_range_data.argtypes = [vp, vp, vp, ip(RangeDataInserterOptions), f64p, C.c_int32, f32p, f32p, C.c_int64]
    L.dl_grid_export_cells.argtypes = [vp, C.c_int64, vp, vp, vp, vp, ip(C.c_int64)]
    L.dl_voxel_filter.argtypes = [vp, f32p, C.c_int64, C.c_int, C.c_float, i64p, ip(C.c_int64)]
    L.dl_voxel_indices.argtypes = [vp, f32p, C.c_int64, C.c_int, C.c_float, i32p]
    L.dl_adaptive_voxel_filter.argtypes = [vp, ip(AdaptiveVoxelFilterOptions), f32p, C.c_int64, C.c_int, i64p,
                                           ip(C.c_int64), f32p, ip(C.c_int)]
    L.dl_rtcsm_match.argtypes = [vp, ip(RtcsmOptions), f64p, f32p, C.c_int64, vp, f64p, ip(C.c_float), ip(RtcsmInfo), vp]
    L.dl_fcsm_match_3dof.argtypes = [vp, ip(FcsmOptions), f64p, f32p, C.c_int64, f32p, C.c_int64, vp, vp, C.c_float,
                                     ip(FcsmResult), vp, C.c_int64]
    L.dl_fcsm_match.argtypes = [vp, ip(FcsmOptions), f32p, f32p, C.c_int32, f64p, f64p, f64p, f32p, C.c_int64, f32p, C.c_int64, vp, vp,
                                C.c_float, ip(FcsmResult)]
    L.dl_constraint_search_batch.argtypes = [vp, ip(ConstraintOptions), C.c_int32, f64p, f32p, i64p, f32p, i64p, C.c_void_p,
                                             C.c_void_p, ip(Constraint)]
    L.dl_ceres_match.argtypes = [vp, ip(CeresOptions), f64p, f64p, C.c_int32, ip(vp), i64p, ip(vp), f64p,
                                 ip(SolveSummary)]
    L.dl_ceres_match_batch.argtypes = [vp, ip(CeresOptions), C.c_int32, C.c_int32, f64p, f64p, ip(vp), i64p, ip(vp),
                                       f64p, ip(SolveSummary)]
    L.dl_ceres_normal_equations.argtypes = [vp, ip(CeresOptions), f64p, f64p, f64p, C.c_int32, ip(vp), i64p, ip(vp),
                                            f64p, f64p, f64p]
    L.dl_imu_preintegrate.argtypes = [vp, ip(ImuNoise), C.c_int32, i32p, f64p, f64p, f64p, f64p, ip(Preintegration)]
    L.dl_imu_predict.argtypes = [ip(NavState), ip(Preintegration), f64p, ip(NavState)]
    L.dl_imu_factor_evaluate.argtypes = [vp, C.c_int32, ip(NavState), ip(Preintegration), f64p, f64p, C.c_double, vp, i32p,
                                         ip(NavState), f64p, f64p, f64p, f64p, f64p]
    L.dl_fused_match_batch.argtypes = [vp, ip(CeresOptions), C.c_double, f64p, C.c_int32, C.c_int32, f64p, ip(NavState),
                                       ip(NavState), ip(Preintegration), ip(vp), i64p, ip(vp), ip(NavState),
                                       ip(SolveSummary)]
    L.dl_ingest_scan.argtypes = [vp, ip(FrontendOptions), vp, C.c_int64, f32p, C.c_int32, f64p, f64p, i64p, f32p, f32p,
                                 f32p, f32p, i64p]
    L.dl_frontend_match_batch.argtypes = [vp, ip(FrontendOptions), C.c_int32, ip(vp), i64p, f32p, C.c_int32, f64p,
                                          f64p, f64p, vp, vp, ip(ScanResult)]
    L.dl_decode_point_cloud2.argtypes = [vp, ip(PointCloud2Layout), vp, C.c_int64, f64p, f32p, ip(C.c_int64), ip(C.c_double)]
    L.dl_decode_point_cloud2_dev.argtypes = [vp, ip(PointCloud2Layout), vp, C.c_int64, f64p, vp, ip(C.c_int64), ip(C.c_double)]
    L.dl_frontend_match_batch_imu.argtypes = [vp, ip(FrontendOptions), ip(FrontendImu), C.c_int32, ip(vp), i64p, f32p, C.c_int32,
                                              f64p, vp, vp, ip(ScanResult)]
    L.dl_frontend_match_batch_imu_samples.argtypes = [vp, ip(FrontendOptions), vp, C.c_int32, ip(vp), i64p, f32p, C.c_int32, f64p,
                                                      vp, vp, ip(ScanResult), vp, vp]
    L.dl_frontend_match_batch_imu_samples_dev.argtypes = [vp, ip(FrontendOptions), vp, C.c_int32, vp, C.c_int64, i64p, f32p,
                                                          C.c_int32, f64p, vp, vp, vp, vp]
    L.dl_frontend_submit_imu_samples.argtypes = [vp, ip(FrontendOptions), vp, C.c_int32, ip(vp), i64p, f32p, C.c_int32, f64p, vp, vp]
    L.dl_frontend_collect_imu.argtypes = [vp, C.c_int32, ip(ScanResult), vp]
    L.dl_comm_unique_id.argtypes = [vp]
    L.dl_comm_create.argtypes = [vp, vp, C.c_int32, C.c_int32, ip(vp)]
    L.dl_comm_destroy.argtypes = [vp]
    L.dl_comm_destroy.restype = None
    L.dl_comm_rank.argtypes = [vp]
    L.dl_comm_world_size.argtypes = [vp]
    L.dl_comm_last_error.restype = C.c_char_p
    L.dl_comm_all_gather_dev.argtypes = [vp, vp, vp, C.c_int64]
    L.dl_comm_all_reduce_f64_dev.argtypes = [vp, vp, C.c_int64]
    L.dl_comm_broadcast_dev.argtypes = [vp, vp, C.c_int64, C.c_int32]
    L.dl_constraint_search_exchange.argtypes = [vp, vp, ip(ConstraintOptions), C.c_int32, C.c_int32, i32p, i32p, f64p, f32p, i64p,
                                                f32p, i64p, C.c_void_p, C.c_void_p, ip(ConstraintRow), ip(ExchangeInfo)]
    L.dl_window_optimize_batch.argtypes = [vp, ip(WindowOptions), C.c_int32, vp, f64p, vp, f64p, vp, vp, vp, f64p, vp]
    L.dl_window_evaluate.argtypes = [vp, ip(WindowOptions), C.c_int32, vp, f64p, vp, f64p, vp, vp, i32p, f64p, f64p, f64p]
    L.dl_pose_graph_evaluate.argtypes = [vp, ip(PoseGraphOptions), C.c_int32, C.c_int32, f64p, vp, vp, C.c_int32, f64p, f64p]
    L.dl_pose_graph_solve_sparse.argtypes = [vp, vp, ip(PoseGraphOptions), C.c_int32, C.c_int32, f64p, vp, vp, C.c_int32,
                                             ip(SolveSummary), ip(PoseGraphSparseInfo)]
    L.dl_pose_graph_3d_create.argtypes = [vp, ip(PoseGraph3DOptions), ip(vp)]
    L.dl_pose_graph_3d_destroy.argtypes = [vp]
    L.dl_pose_graph_3d_destroy.restype = None
    L.dl_pose_graph_3d_add_node.argtypes = [vp, ip(Pg3dNode), C.c_int32, vp, vp]
    L.dl_pose_graph_3d_freeze_trajectory.argtypes = [vp, C.c_int32]
    L.dl_pose_graph_3d_run_final_optimization.argtypes = [vp, vp]
    L.dl_pose_graph_3d_poses.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, vp, ip(C.c_int32)]
    L.dl_pose_graph_3d_local_to_global.argtypes = [vp, C.c_int32, vp]
    L.dl_pose_graph_3d_constraints.argtypes = [vp, C.c_int32, vp, ip(C.c_int32)]
    L.dl_pose_graph_3d_last_searches.argtypes = [vp, C.c_int32, vp, ip(C.c_int32)]
    L.dl_pose_graph_3d_store_bytes.argtypes = [vp, ip(C.c_int64), ip(C.c_int64)]
    L.dl_pg3d_trim_submap.argtypes = [vp, C.c_int32, C.c_int32]
    L.dl_pg3d_add_pure_localization_trimmer.argtypes = [vp, C.c_int32, C.c_int32]
    L.dl_pg3d_finish_trajectory.argtypes = [vp, C.c_int32]
    L.dl_pg3d_is_trajectory_finished.argtypes = [vp, C.c_int32, ip(C.c_int32)]
    L.dl_pg3d_set_initial_trajectory_pose.argtypes = [vp, C.c_int32, C.c_int32, vp, C.c_double]
    L.dl_pg3d_ids.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, vp, ip(C.c_int32)]
    L.dl_pg3d_last_trimmed.argtypes = [vp, C.c_int32, vp, ip(C.c_int32)]
    L.dl_pg3d_store_usage.argtypes = [vp, ip(C.c_int64), ip(C.c_int64), ip(C.c_int64)]
    L.dl_range_data_map_set_node.argtypes = [vp, C.c_int32, C.c_int32, vp, C.c_int64]
    for name in ("dl_range_data_map", "dl_range_data_map_dev"):
        getattr(L, name).argtypes = [vp, C.c_int32, vp, C.c_int32, vp, ip(C.c_int32), C.c_int64, vp, ip(C.c_int64)]
    L.dl_map_writer_create.argtypes = [vp, ip(MapWriterOptions), ip(vp)]
    L.dl_map_writer_destroy.argtypes = [vp]
    L.dl_map_writer_destroy.restype = None
    L.dl_map_writer_add_trajectory.argtypes = [vp, C.c_int32, C.c_int32, vp, vp]
    L.dl_map_writer_process.argtypes = [vp, C.c_int32, vp, vp, C.c_int64, vp, ip(C.c_int64), vp, ip(MapWriterInfo)]
    L.dl_map_writer_process_dev.argtypes = [vp, C.c_int32, vp, vp, C.c_int64, vp, ip(C.c_int64), vp, ip(MapWriterInfo)]
    L.dl_map_writer_flush.argtypes = [vp, ip(C.c_int32)]
    L.dl_map_writer_voxels.argtypes = [vp, C.c_int64, vp, vp, vp, ip(C.c_int64)]
    L.dl_map_writer_add_color.argtypes = [vp, ip(MapWriterColor)]
    L.dl_map_writer_add_xray.argtypes = [vp, ip(MapWriterXray), ip(C.c_int32)]
    L.dl_map_writer_xray_image.argtypes = [vp, C.c_int32, C.c_int64, vp, ip(C.c_int32), ip(C.c_int32)]
    L.dl_map_writer_add_probability_grid.argtypes = [vp, ip(MapWriterGridOptions), ip(C.c_int32)]
    L.dl_map_writer_probability_grid.argtypes = [vp, C.c_int32, ip(MapWriterGridInfo), C.c_int64, vp, vp]
    L.dl_rotational_histogram.argtypes = [vp, f32p, C.c_int64, C.c_int32, f32p]
    L.dl_submap_textures.argtypes = [vp, C.c_int32, ip(SubmapImageQuery), ip(SubmapTexture), C.c_int64, vp, ip(C.c_int64)]
    L.dl_submap_projections.argtypes = [vp, C.c_int32, ip(SubmapImageQuery), ip(SubmapProjection), C.c_int64, vp,
                                        ip(C.c_int64)]
    L.dl_ltb_create.argtypes = [vp, ip(LtbOptions), ip(vp)]
    L.dl_ltb_destroy.argtypes = [vp]
    L.dl_ltb_destroy.restype = None
    L.dl_ltb_set_initial_state.argtypes = [vp, ip(NavState)]
    L.dl_ltb_add_imu_data.argtypes = [vp, C.c_double, f64p, f64p]
    L.dl_ltb_add_range_data.argtypes = [vp, C.c_double, f32p, C.c_int64, f32p, ip(MatchingResult)]
    L.dl_ltb_add_synchronized_range_data.argtypes = [vp, C.c_double, vp, C.c_int64, C.c_int32, f32p, C.c_int32, ip(MatchingResult)]
    L.dl_ltb_get_cloud.argtypes = [vp, C.c_int32, vp, C.c_int64, ip(C.c_int64)]
    L.dl_ltb_get_histogram.argtypes = [vp, f32p, C.c_int32]
    L.dl_ltb_num_submaps.argtypes = [vp]
    L.dl_ltb_get_submap.argtypes = [vp, C.c_int32, ip(vp), ip(vp), f64p, ip(C.c_int32), ip(C.c_int32)]
    L.dl_ltb_get_state.argtypes = [vp, ip(NavState), ip(C.c_int32)]
    L.dl_ltb_add_range_data_batch.argtypes = [C.c_int32, ip(LtbBatchItem), ip(MatchingResult)]
    L.dl_ltb_release_submap.argtypes = [vp, C.c_int32]
    L.dl_frontend_submit.argtypes = [vp, ip(FrontendOptions), C.c_int32, ip(vp), i64p, f32p, C.c_int32, f64p, f64p, f64p, vp, vp]
    L.dl_frontend_collect.argtypes = [vp, C.c_int32, ip(ScanResult)]
    L.dl_frontend_match_batch_dev.argtypes = [vp, ip(FrontendOptions), C.c_int32, vp, C.c_int64, i64p, f32p, C.c_int32,
                                              f64p, f64p, f64p, vp, vp, vp]
    L.dl_frontend_fetch_results.argtypes = [vp, vp, C.c_int32, ip(ScanResult)]
    L.dl_device_alloc.argtypes = [vp, C.c_int64, ip(vp)]
    L.dl_device_free.argtypes = [vp, vp]
    L.dl_copy_to_device.argtypes = [vp, vp, vp, C.c_int64]
    L.dl_copy_to_host.argtypes = [vp, vp, vp, C.c_int64]
    _LIB = L
    return L


class TimeRuns:
    """Per-point times of a batch of scans as runs (dl_frontend_options::time_run_*), for 12-byte x y z rows. Built from the per-scan
    time arrays; attach() points an options block at the arrays (which stay alive with this object)."""

    def __init__(self, times_per_scan, pin=False):
        offs, firsts, values = [0], [], []
        for t in times_per_scan:
            t = np.ascontiguousarray(t, np.float32)
            if len(t):
                start = np.concatenate([[0], np.nonzero(t[1:].view(np.uint32) != t[:-1].view(np.uint32))[0] + 1])
                firsts.append(start.astype(np.int32))
                values.append(t[start])
                offs.append(offs[-1] + len(start))
            else:
                offs.append(offs[-1])
        self.offsets = np.ascontiguousarray(offs, np.int32)
        self.first_row = np.ascontiguousarray(np.concatenate(firsts) if firsts else np.zeros(0, np.int32), np.int32)
        self.value = np.ascontiguousarray(np.concatenate(values) if values else np.zeros(0, np.float32), np.float32)
        if pin:   # page-locked: the per-batch upload of the table is then asynchronous
            import torch
            self._pinned = [torch.from_numpy(a).pin_memory() for a in (self.offsets, self.first_row, self.value)]
            self.offsets, self.first_row, self.value = [t.numpy() for t in self._pinned]

    @property
    def nbytes(self):
        return self.offsets.nbytes + self.first_row.nbytes + self.value.nbytes

    def attach(self, options):
        options.range_row_floats = 3
        options.time_run_offsets = self.offsets.ctypes.data
        options.time_run_first_row = self.first_row.ctypes.data
        options.time_run_value = self.value.ctypes.data
        options._time_runs = self
        return options


class HostScanBatch:
    """Per-scan host row arrays + the pointer/size tables the C-ABI takes (built once, reusable across calls)."""

    def __init__(self, ranges_list):
        self.rows = list(ranges_list)
        self.n = len(self.rows)
        self.pointers = (C.c_void_p * max(self.n, 1))(*[r.ctypes.data for r in self.rows])
        self.sizes = np.array([len(r) for r in self.rows], np.int64)


class Context:
    def __init__(self, device=0):
        self.L = lib()
        h = C.c_void_p()
        st = self.L.dl_context_create(device, C.byref(h))
        if st != 0:
            raise DlError(st, self.L.dl_last_error(None).decode())
        self.h = h
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            self.L.dl_context_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def check(self, st):
        if st != 0:
            raise DlError(st, self.L.dl_last_error(self.h).decode() or self.L.dl_status_string(st).decode())

    @property
    def launches(self):
        return self.L.dl_context_kernel_launches(self.h)

    @property
    def stream(self):
        return self.L.dl_context_stream(self.h)

    def synchronize(self):
        self.check(self.L.dl_context_synchronize(self.h))

    def set_profiling(self, on):
        self.check(self.L.dl_context_set_profiling(self.h, int(on)))

    def set_blocking_sync(self, on=True):
        """Host waits of this context sleep instead of spinning (background threads on hosts with few CPUs)."""
        self.check(self.L.dl_context_set_blocking_sync(self.h, int(on)))

    def read_profile(self):
        """{stage: (total ms, calls)} since the last read (device time between CUDA events on the context stream)."""
        buf = (StageTime * 16)()
        n = C.c_int32(0)
        self.check(self.L.dl_context_read_profile(self.h, buf, 16, C.byref(n)))
        return {buf[i].name.decode(): (buf[i].ms, buf[i].calls) for i in range(n.value)}

    # ---- grid
    def grid(self, resolution):
        return Grid(self, resolution)

    # ---- filters
    def voxel_filter(self, points, resolution):
        points = np.ascontiguousarray(points, np.float32)
        n, stride = points.shape
        keep = np.zeros(max(n, 1), np.int64)
        m = C.c_int64(0)
        self.check(self.L.dl_voxel_filter(self.h, points, n, stride, resolution, keep, C.byref(m)))
        return keep[:m.value].copy()

    def voxel_indices(self, points, resolution):
        points = np.ascontiguousarray(points, np.float32)
        n, stride = points.shape
        out = np.zeros((max(n, 1), 3), np.int32)
        self.check(self.L.dl_voxel_indices(self.h, points, n, stride, resolution, out))
        return out[:n]

    def adaptive_voxel_filter(self, points, max_length, min_num_points, max_range):
        points = np.ascontiguousarray(points, np.float32)
        n, stride = points.shape
        keep = np.zeros(max(n, 1), np.int64)
        passes = np.zeros(32, np.float32)
        m, npass = C.c_int64(0), C.c_int(0)
        opt = AdaptiveVoxelFilterOptions(max_length, min_num_points, max_range)
        self.check(self.L.dl_adaptive_voxel_filter(self.h, C.byref(opt), points, n, stride, keep, C.byref(m), passes,
                                                   C.byref(npass)))
        return keep[:m.value].copy(), passes[:npass.value].copy()

    # ---- RotationalScanMatcher::ComputeHistogram
    def rotational_histogram(self, points, size):
        """Histogram of `size` buckets of the n x 3 cloud (gravity-aligned frame); size in [1, 1024], n <= 2^20."""
        points = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
        out = np.zeros(max(int(size), 0), np.float32)
        self.check(self.L.dl_rotational_histogram(self.h, points, len(points), int(size), out))
        return out

    # ---- submap images
    def _submap_images(self, fn, record, queries):
        n = len(queries)
        qs = (SubmapImageQuery * max(n, 1))()
        for k, (grid, pose) in enumerate(queries):
            qs[k].grid = grid.h if isinstance(grid, Grid) else grid
            qs[k].pose[:] = [float(v) for v in np.asarray(pose, np.float64).reshape(7)]
        recs = (record * max(n, 1))()
        size = C.c_int64(0)
        self.check(fn(self.h, n, qs, recs, 0, None, C.byref(size)))
        out = np.zeros(max(size.value, 1), np.uint8)
        self.check(fn(self.h, n, qs, recs, size.value, out.ctypes.data_as(C.c_void_p), C.byref(size)))
        return [recs[k] for k in range(n)], out

    def submap_textures(self, queries):
        """Submap3D::ToResponseProto's textures of (grid, global pose 7-vector) queries, one call: a dict per query with
        resolution, width, height, slice_pose and cells, a (height, width, 2) uint8 array of (value, alpha) (not gzipped)."""
        recs, out = self._submap_images(self.L.dl_submap_textures, SubmapTexture, queries)
        return [{"resolution": r.resolution, "width": r.width, "height": r.height, "slice_pose": np.array(r.slice_pose[:]),
                 "cells": out[r.offset:r.offset + 2 * r.width * r.height].reshape(r.height, r.width, 2).copy()} for r in recs]

    def project_submaps(self, queries):
        """ProjectToCvMat of (grid, pose 7-vector) queries, one call: a dict per query with resolution, width, height, ox, oy and
        pixels, a (height, width) uint8 array (row y - min_y, column x - min_x)."""
        recs, out = self._submap_images(self.L.dl_submap_projections, SubmapProjection, queries)
        return [{"resolution": r.resolution, "width": r.width, "height": r.height, "ox": r.ox, "oy": r.oy,
                 "pixels": out[r.offset:r.offset + r.width * r.height].reshape(r.height, r.width).copy()} for r in recs]

    # ---- matchers
    def rtcsm_match(self, grid, points, initial_pose, linear_window, angular_window, w_t, w_r, want_scores=False):
        points = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
        opt = RtcsmOptions(linear_window, angular_window, w_t, w_r)
        pose = np.zeros(7)
        score = C.c_float(0)
        info = RtcsmInfo()
        init = np.ascontiguousarray(initial_pose, np.float64)
        scores = None
        sp = None
        if want_scores:
            self.check(self.L.dl_rtcsm_match(self.h, C.byref(opt), init, points, len(points), grid.h, pose,
                                             C.byref(score), C.byref(info), None))
            scores = np.zeros(info.num_candidates, np.float32)
            sp = scores.ctypes.data_as(C.c_void_p)
        self.check(self.L.dl_rtcsm_match(self.h, C.byref(opt), init, points, len(points), grid.h, pose, C.byref(score),
                                         C.byref(info), sp))
        return {"score": np.float32(score.value), "pose": pose, "best_index": info.best_index,
                "linear": info.linear_window, "angular": info.angular_window, "angular_step": np.float32(info.angular_step),
                "max_scan_range": np.float32(info.max_scan_range), "num_candidates": info.num_candidates,
                "scores": scores}

    def fcsm_match_3dof(self, hi_grid, lo_grid, hi_points, lo_points, pose_guess, min_score, xy_window=5.0, z_window=1.0,
                        min_low_resolution_score=0.55, min_rotational_score=0.77, depth=8, full_depth=3, want_scores=False):
        """MatchWith3DofInitial -> FcsmResult; with want_scores, (FcsmResult, float32 score of every leaf as a
        [2 wz + 1, 2 wxy + 1, 2 wxy + 1] (z, y, x) array), from the exhaustive search. The array is sized by the header's
        formula; the library checks its capacity against its own count and refuses a call it would overrun."""
        hi_points = np.ascontiguousarray(hi_points, np.float32).reshape(-1, 3)
        lo_points = np.ascontiguousarray(lo_points, np.float32).reshape(-1, 3)
        opt = FcsmOptions(depth, full_depth, min_rotational_score, min_low_resolution_score, xy_window, z_window, 0.26)
        r = FcsmResult()
        scores = None
        if want_scores:
            res = float(self.L.dl_grid_resolution(hi_grid.h))    # window / float resolution in double, then lround
            wxy, wz = (int(np.floor(q)) + int(q - np.floor(q) >= 0.5) for q in (xy_window / res, z_window / res))
            scores = np.zeros((2 * wz + 1, 2 * wxy + 1, 2 * wxy + 1), np.float32) if min(wxy, wz) >= 0 else np.zeros(1, np.float32)
        self.check(self.L.dl_fcsm_match_3dof(self.h, C.byref(opt), np.ascontiguousarray(pose_guess, np.float64), hi_points,
                                             len(hi_points), lo_points, len(lo_points), hi_grid.h, lo_grid.h,
                                             np.float32(min_score), C.byref(r),
                                             None if scores is None else scores.ctypes.data_as(C.c_void_p),
                                             0 if scores is None else scores.size))
        return r if scores is None else (r, scores)

    def fcsm_match(self, hi_grid, lo_grid, hi_points, lo_points, node_pose, submap_pose, min_score, submap_histogram=None,
                   scan_histogram=None, histogram_size=10, gravity_alignment=(1.0, 0.0, 0.0, 0.0), xy_window=5.0, z_window=1.0,
                   angular_window=0.2617993877991494, min_low_resolution_score=0.55, min_rotational_score=0.77, depth=8,
                   full_depth=3):
        """FastCorrelativeScanMatcher3D::Match (yaw search x translation window)."""
        hi_points = np.ascontiguousarray(hi_points, np.float32).reshape(-1, 3)
        lo_points = np.ascontiguousarray(lo_points, np.float32).reshape(-1, 3)
        sh = np.zeros(histogram_size, np.float32) if submap_histogram is None else np.ascontiguousarray(submap_histogram, np.float32)
        nh = np.zeros(len(sh), np.float32) if scan_histogram is None else np.ascontiguousarray(scan_histogram, np.float32)
        opt = FcsmOptions(depth, full_depth, min_rotational_score, min_low_resolution_score, xy_window, z_window, angular_window)
        r = FcsmResult()
        self.check(self.L.dl_fcsm_match(self.h, C.byref(opt), sh, nh, len(sh), np.ascontiguousarray(node_pose, np.float64),
                                        np.ascontiguousarray(submap_pose, np.float64), np.ascontiguousarray(gravity_alignment, np.float64),
                                        hi_points, len(hi_points), lo_points, len(lo_points), hi_grid.h, lo_grid.h,
                                        np.float32(min_score), C.byref(r)))
        return r

    def constraint_search_batch(self, options, pose_guesses, hi_clouds, lo_clouds, hi_grids, lo_grids):
        """ConstraintBuilder3D::ComputeConstraint for len(pose_guesses) (node, submap) pairs -> list of Constraint."""
        count = len(pose_guesses)
        his = [np.ascontiguousarray(c, np.float32).reshape(-1, 3) for c in hi_clouds]
        los = [np.ascontiguousarray(c, np.float32).reshape(-1, 3) for c in lo_clouds]
        hi_off = np.concatenate([[0], np.cumsum([len(c) for c in his])]).astype(np.int64)
        lo_off = np.concatenate([[0], np.cumsum([len(c) for c in los])]).astype(np.int64)
        hi_all = np.ascontiguousarray(np.concatenate(his) if count else np.zeros((1, 3), np.float32))
        lo_all = np.ascontiguousarray(np.concatenate(los) if count else np.zeros((1, 3), np.float32))
        hg = (C.c_void_p * max(count, 1))(*[g.h for g in hi_grids])
        lg = (C.c_void_p * max(count, 1))(*[g.h for g in lo_grids])
        out = (Constraint * max(count, 1))()
        self.check(self.L.dl_constraint_search_batch(self.h, C.byref(options), count,
                                                     np.ascontiguousarray(pose_guesses, np.float64).reshape(-1, 7), hi_all,
                                                     hi_off, lo_all, lo_off, hg, lg, out))
        return list(out)[:count]

    def constraint_search_exchange(self, comm, options, capacity, submap_ids, node_ids, pose_guesses, hi_clouds, lo_clouds,
                                   hi_grids, lo_grids):
        """This rank's (node, submap) searches + the ncclAllGather of the constraint rows -> (table of world * capacity
        ConstraintRow, ExchangeInfo). Pruned pairs have found == 0, unused slots found == -1."""
        return self.constraint_exchange_plan(comm, options, capacity, submap_ids, node_ids, pose_guesses, hi_clouds, lo_clouds,
                                             hi_grids, lo_grids)()

    def constraint_exchange_plan(self, comm, options, capacity, submap_ids, node_ids, pose_guesses, hi_clouds, lo_clouds,
                                 hi_grids, lo_grids):
        """The marshalled arguments of constraint_search_exchange as a callable: a caller that repeats the same exchange (or
        runs it from a worker thread, like the reference's constraint-builder pool) pays the numpy packing once."""
        count = len(pose_guesses)
        his = [np.ascontiguousarray(c, np.float32).reshape(-1, 3) for c in hi_clouds]
        los = [np.ascontiguousarray(c, np.float32).reshape(-1, 3) for c in lo_clouds]
        hi_off = np.concatenate([[0], np.cumsum([len(c) for c in his])]).astype(np.int64)
        lo_off = np.concatenate([[0], np.cumsum([len(c) for c in los])]).astype(np.int64)
        hi_all = np.ascontiguousarray(np.concatenate(his) if count else np.zeros((1, 3), np.float32))
        lo_all = np.ascontiguousarray(np.concatenate(los) if count else np.zeros((1, 3), np.float32))
        hg = (C.c_void_p * max(count, 1))(*[g.h for g in hi_grids])
        lg = (C.c_void_p * max(count, 1))(*[g.h for g in lo_grids])
        sub = np.ascontiguousarray(submap_ids, np.int32)
        nod = np.ascontiguousarray(node_ids, np.int32)
        guesses = np.ascontiguousarray(pose_guesses, np.float64).reshape(-1, 7)
        keep = (hi_grids, lo_grids)   # the grids must outlive the plan

        def run():
            table = (ConstraintRow * (comm.world * capacity))()
            info = ExchangeInfo()
            self.check(self.L.dl_constraint_search_exchange(self.h, comm.h, C.byref(options), count, capacity, sub, nod, guesses,
                                                            hi_all, hi_off, lo_all, lo_off, hg, lg, table, C.byref(info)))
            return table, info
        run.keep = keep
        return run

    def window_optimize_batch(self, means_i, prior_infos, preints, matched_poses, sigma_t=0.05, sigma_r=0.01, imu_weight=1.0,
                              gravity=(0.0, 0.0, 9.8), max_iter=10, gravity_factor=None, initial_j=None, states_i_out=True):
        """WindowOptimize's stand-in (dl_window_optimize_batch) for len(means_i) trajectories. means_i / initial_j: 16-vectors;
        prior_infos: (n, 15, 15); preints: ctypes Preintegration objects. -> (states_i smoothed, states_j, informations, summaries);
        states_i_out=False passes NULL for the smoothed previous keys and returns None in their place."""
        n = len(means_i)
        opt = self._window_options(sigma_t, sigma_r, imu_weight, gravity, max_iter, gravity_factor)
        si = (NavState * n)(*[NavState.from16(x) for x in means_i])
        pm = (Preintegration * n)(*preints)
        init = (NavState * n)(*[NavState.from16(x) for x in initial_j]) if initial_j is not None else None
        out_i, out_j = (NavState * n)(), (NavState * n)()
        info = np.zeros((n, 15, 15))
        sums = (SolveSummary * n)()
        self.check(self.L.dl_window_optimize_batch(self.h, C.byref(opt), n, C.cast(si, C.c_void_p),
                                                   np.ascontiguousarray(prior_infos, np.float64).reshape(-1), C.cast(pm, C.c_void_p),
                                                   np.ascontiguousarray(matched_poses, np.float64).reshape(-1),
                                                   C.cast(init, C.c_void_p) if init is not None else None,
                                                   C.cast(out_i, C.c_void_p) if states_i_out else None,
                                                   C.cast(out_j, C.c_void_p), info.reshape(-1), C.cast(sums, C.c_void_p)))
        return (np.array([o.to16() for o in out_i]) if states_i_out else None, np.array([o.to16() for o in out_j]), info,
                [s.as_dict() for s in sums])

    @staticmethod
    def _window_options(sigma_t, sigma_r, imu_weight, gravity, max_iter, gravity_factor):
        return WindowOptions(sigma_t, sigma_r, imu_weight, (C.c_double * 3)(*gravity), int(max_iter), 1 if gravity_factor else 0,
                             float(gravity_factor[0]) if gravity_factor else 1.0,
                             (C.c_double * 3)(*(gravity_factor[1] if gravity_factor else (0, 0, 1))),
                             (C.c_double * 3)(*(gravity_factor[2] if gravity_factor else (0, 0, 1))))

    def window_evaluate(self, means_i, prior_infos, preints, matched_poses, x_i, x_j, sigma_t=0.05, sigma_r=0.01, imu_weight=1.0,
                        gravity=(0.0, 0.0, 9.8), gravity_factor=None):
        """The window's factors at given (x_i, x_j) (dl_window_evaluate); arguments as window_optimize_batch, x_i / x_j: 16-vectors.
        -> dict of ok [n], residual [n,38], jacobian [n,38,30], weight [n,38,38]."""
        n = len(means_i)
        opt = self._window_options(sigma_t, sigma_r, imu_weight, gravity, 10, gravity_factor)
        si = (NavState * n)(*[NavState.from16(x) for x in means_i])
        pm = (Preintegration * n)(*preints)
        xi = (NavState * n)(*[NavState.from16(x) for x in x_i])
        xj = (NavState * n)(*[NavState.from16(x) for x in x_j])
        ok = np.zeros(n, np.int32)
        r, J, W = np.zeros((n, 38)), np.zeros((n, 38, 30)), np.zeros((n, 38, 38))
        self.check(self.L.dl_window_evaluate(self.h, C.byref(opt), n, C.cast(si, C.c_void_p),
                                             np.ascontiguousarray(prior_infos, np.float64).reshape(-1), C.cast(pm, C.c_void_p),
                                             np.ascontiguousarray(matched_poses, np.float64).reshape(-1), C.cast(xi, C.c_void_p),
                                             C.cast(xj, C.c_void_p), ok, r.reshape(-1), J.reshape(-1), W.reshape(-1)))
        return {"ok": ok, "residual": r, "jacobian": J, "weight": W}

    def pose_graph_solve_sparse(self, submap_poses, node_poses, constraints, fix_z=False, max_iter=50, comm=None, frozen=None):
        """OptimizationProblem3D::Solve (SPA only) on the device, block-sparse (Schur complement of the node blocks), for whole
        trajectories. constraints: this rank's (submap, node, zbar7, translation_weight, rotation_weight) tuples; with `comm` the
        normal-equation blocks are all-reduced over the ranks. frozen: None or len(submaps) + len(nodes) flags (submaps first).
        -> (submaps, nodes, summary, PoseGraphSparseInfo)."""
        S, N = len(submap_poses), len(node_poses)
        poses = np.ascontiguousarray(np.concatenate([np.asarray(submap_poses, np.float64).reshape(S, 7),
                                                     np.asarray(node_poses, np.float64).reshape(N, 7)]))
        cs = spa_constraints(constraints)
        fz = None
        if frozen is not None:
            fz = np.ascontiguousarray(np.asarray(frozen, bool).astype(np.uint8).reshape(-1))
            if len(fz) != S + N:
                raise ValueError(f"frozen has {len(fz)} flags, the graph {S + N} poses")
        opt = PoseGraphOptions(int(max_iter), int(bool(fix_z)))
        s, info = SolveSummary(), PoseGraphSparseInfo()
        self.check(self.L.dl_pose_graph_solve_sparse(self.h, comm.h if comm else None, C.byref(opt), S, N, poses,
                                                     fz.ctypes.data if fz is not None else None, C.cast(cs, C.c_void_p),
                                                     len(constraints), C.byref(s), C.byref(info)))
        return poses[:S].copy(), poses[S:].copy(), s.as_dict(), info

    def pose_graph_evaluate(self, submap_poses, node_poses, constraints, fix_z=False, frozen=None):
        """The solve's factors at given poses (dl_pose_graph_evaluate); arguments as pose_graph_solve_sparse.
        -> (residuals [m, 6], local Jacobians [m, 6, 12]: submap slots 0..5, node slots 6..11)."""
        S, N, m = len(submap_poses), len(node_poses), len(constraints)
        poses = np.ascontiguousarray(np.concatenate([np.asarray(submap_poses, np.float64).reshape(S, 7),
                                                     np.asarray(node_poses, np.float64).reshape(N, 7)]))
        cs = spa_constraints(constraints)
        fz = None if frozen is None else np.ascontiguousarray(np.asarray(frozen, bool).astype(np.uint8).reshape(-1))
        if fz is not None and len(fz) != S + N:
            raise ValueError(f"frozen has {len(fz)} flags, the graph {S + N} poses")
        r, J = np.zeros((m, 6)), np.zeros((m, 6, 12))
        self.check(self.L.dl_pose_graph_evaluate(self.h, C.byref(PoseGraphOptions(50, int(bool(fix_z)))), S, N, poses,
                                                 fz.ctypes.data if fz is not None else None, C.cast(cs, C.c_void_p), m,
                                                 r.reshape(-1), J.reshape(-1)))
        return r, J

    @staticmethod
    def _pairs(clouds, grids):
        clouds = [np.ascontiguousarray(c, np.float32).reshape(-1, 3) for c in clouds]
        n = len(clouds)
        cp = (C.c_void_p * n)(*[c.ctypes.data for c in clouds])
        gp = (C.c_void_p * n)(*[g.h.value for g in grids])
        sizes = np.array([len(c) for c in clouds], np.int64)
        return clouds, cp, gp, sizes

    def ceres_match(self, clouds, grids, occ_weights, trans_w, rot_w, target_translation, initial_pose, only_yaw=False,
                    nonmono=False, max_iter=12):
        clouds, cp, gp, sizes = self._pairs(clouds, grids)
        opt = CeresOptions.make(occ_weights, trans_w, rot_w, only_yaw, nonmono, max_iter)
        pose = np.zeros(7)
        s = SolveSummary()
        self.check(self.L.dl_ceres_match(self.h, C.byref(opt), np.ascontiguousarray(target_translation, np.float64),
                                         np.ascontiguousarray(initial_pose, np.float64), len(clouds), cp, sizes, gp,
                                         pose, C.byref(s)))
        return pose, s.as_dict()

    def ceres_match_batch(self, problems, grids_per_problem, occ_weights, trans_w, rot_w, targets, initial_poses,
                          nonmono=False, max_iter=12):
        """problems: list (per problem) of list (per pair) of clouds."""
        count, num_pairs = len(problems), len(problems[0])
        flat_c = [c for p in problems for c in p]
        flat_g = [g for p in grids_per_problem for g in p]
        clouds, cp, gp, sizes = self._pairs(flat_c, flat_g)
        opt = CeresOptions.make(occ_weights, trans_w, rot_w, False, nonmono, max_iter)
        poses = np.zeros((count, 7))
        sums = (SolveSummary * count)()
        self.check(self.L.dl_ceres_match_batch(self.h, C.byref(opt), count, num_pairs,
                                               np.ascontiguousarray(targets, np.float64),
                                               np.ascontiguousarray(initial_poses, np.float64), cp, sizes, gp, poses,
                                               sums))
        return poses, [s.as_dict() for s in sums]

    def ceres_normal_equations(self, clouds, grids, occ_weights, trans_w, rot_w, target_translation, reference_pose,
                               at_pose):
        clouds, cp, gp, sizes = self._pairs(clouds, grids)
        opt = CeresOptions.make(occ_weights, trans_w, rot_w)
        cost, g, h = np.zeros(1), np.zeros(6), np.zeros(36)
        self.check(self.L.dl_ceres_normal_equations(self.h, C.byref(opt),
                                                    np.ascontiguousarray(target_translation, np.float64),
                                                    np.ascontiguousarray(reference_pose, np.float64),
                                                    np.ascontiguousarray(at_pose, np.float64), len(clouds), cp, sizes,
                                                    gp, cost, g, h))
        return cost[0], g, h.reshape(6, 6)

    # ---- IMU
    def imu_preintegrate(self, noise4, intervals, biases):
        """intervals: list of (dt[n], acc[n,3], gyr[n,3]); biases: (count, 6). Returns a ctypes array of Preintegration."""
        count = len(intervals)
        offsets = np.zeros(count + 1, np.int32)
        for k, (dt, _, _) in enumerate(intervals):
            offsets[k + 1] = offsets[k] + len(dt)
        dt = np.ascontiguousarray(np.concatenate([i[0] for i in intervals]), np.float64)
        acc = np.ascontiguousarray(np.concatenate([np.asarray(i[1]).reshape(-1, 3) for i in intervals]), np.float64)
        gyr = np.ascontiguousarray(np.concatenate([np.asarray(i[2]).reshape(-1, 3) for i in intervals]), np.float64)
        out = (Preintegration * count)()
        noise = ImuNoise(*noise4)
        self.check(self.L.dl_imu_preintegrate(self.h, C.byref(noise), count, offsets, dt, acc, gyr,
                                              np.ascontiguousarray(biases, np.float64).reshape(count, 6), out))
        return out

    def imu_predict(self, state_i16, m, gravity=(0.0, 0.0, 9.8)):
        si, sj = NavState.from16(state_i16), NavState()
        self.check(self.L.dl_imu_predict(C.byref(si), C.byref(m), np.ascontiguousarray(gravity, np.float64), C.byref(sj)))
        return sj.to16()

    def imu_factor_evaluate(self, states_i, preints, submap_poses, imu_weight=1.0, gravity=(0.0, 0.0, 9.8), x16=None):
        """The fused solve's IMU factor alone (dl_imu_factor_evaluate). states_i: [n,16] local frame; preints: Preintegration
        structs; submap_poses: [n,7]; x16: [n,16] in the submap frame or None (the prepared start). -> dict of ok [n],
        predicted [n,16], information [n,15,15], residual [n,15], hessian [n,15,15], gradient [n,15], cost2 [n]."""
        n = len(preints)
        si = (NavState * n)(*[NavState.from16(x) for x in states_i])
        pm = (Preintegration * n)(*preints)
        pred = (NavState * n)()
        ok = np.zeros(n, np.int32)
        info, hess = np.zeros((n, 15, 15)), np.zeros((n, 15, 15))
        res, grad, cost2 = np.zeros((n, 15)), np.zeros((n, 15)), np.zeros(n)
        x = None if x16 is None else np.ascontiguousarray(x16, np.float64).reshape(n, 16)
        self.check(self.L.dl_imu_factor_evaluate(self.h, n, si, pm, np.ascontiguousarray(submap_poses, np.float64).reshape(n, 7),
                                                 np.ascontiguousarray(gravity, np.float64), float(imu_weight),
                                                 None if x is None else x.ctypes.data, ok, pred, info, res, hess, grad, cost2))
        return {"ok": ok, "predicted": np.array([p.to16() for p in pred]), "information": info, "residual": res,
                "hessian": hess, "gradient": grad, "cost2": cost2}

    def fused_match_batch(self, problems, grids_per_problem, occ_weights, trans_w, rot_w, submap_poses, states_i,
                          initial_states_j, preints, imu_weight=1.0, gravity=(0.0, 0.0, 9.8), nonmono=False, max_iter=12):
        count, num_pairs = len(problems), len(problems[0])
        clouds, cp, gp, sizes = self._pairs([c for p in problems for c in p], [g for p in grids_per_problem for g in p])
        opt = CeresOptions.make(occ_weights, trans_w, rot_w, False, nonmono, max_iter)
        si = (NavState * count)(*[NavState.from16(x) for x in states_i])
        sj = (NavState * count)(*[NavState.from16(x) for x in initial_states_j])
        pm = (Preintegration * count)(*preints)
        out = (NavState * count)()
        sums = (SolveSummary * count)()
        self.check(self.L.dl_fused_match_batch(self.h, C.byref(opt), imu_weight, np.ascontiguousarray(gravity, np.float64),
                                               count, num_pairs, np.ascontiguousarray(submap_poses, np.float64), si, sj,
                                               pm, cp, sizes, gp, out, sums))
        return np.array([o.to16() for o in out]), [s.as_dict() for s in sums]

    # ---- front end
    def ingest_scan(self, options, ranges, origins, prev_pose, cur_pose):
        n = len(ranges)
        origins = np.ascontiguousarray(origins, np.float32).reshape(-1, 3)
        first_keep = np.zeros(n, np.int64)
        rl, rt, mt = (np.zeros((n, 3), np.float32) for _ in range(3))
        cp = np.zeros(7, np.float32)
        counts = np.zeros(4, np.int64)
        self.check(self.L.dl_ingest_scan(self.h, C.byref(options), ranges.ctypes.data_as(C.c_void_p), n, origins,
                                         len(origins), np.ascontiguousarray(prev_pose, np.float64),
                                         np.ascontiguousarray(cur_pose, np.float64), first_keep, rl, rt, mt, cp, counts))
        return {"first_keep": first_keep[:counts[0]].copy(), "returns_local": rl[:counts[1]].copy(),
                "returns_tracking": rt[:counts[2]].copy(), "misses_tracking": mt[:counts[3]].copy(), "current_pose": cp}

    def frontend_match_batch(self, options, ranges_list, origins, prev_poses, cur_poses, submap_local_pose, hi, lo):
        """ranges_list: list of per-scan row arrays, or a HostScanBatch (the pointer table a C++ caller would hold)."""
        hb = ranges_list if isinstance(ranges_list, HostScanBatch) else HostScanBatch(ranges_list)
        origins = np.ascontiguousarray(origins, np.float32).reshape(-1, 3)
        results = (ScanResult * hb.n)()
        self.check(self.L.dl_frontend_match_batch(self.h, C.byref(options), hb.n, hb.pointers, hb.sizes, origins, len(origins),
                                                  np.ascontiguousarray(prev_poses, np.float64),
                                                  np.ascontiguousarray(cur_poses, np.float64),
                                                  np.ascontiguousarray(submap_local_pose, np.float64), hi.h, lo.h,
                                                  results))
        return results

    def decode_point_cloud2(self, data, point_step, offsets, time_type, sensor_to_tracking):
        """Raw sensor_msgs/PointCloud2 bytes -> (TimedPointCloud rows [k, 4] in the tracking frame, stamp offset seconds)."""
        data = np.ascontiguousarray(data, np.uint8).reshape(-1)
        n = len(data) // point_step
        lay = PointCloud2Layout(point_step, *[int(v) for v in offsets], int(time_type))
        rows = np.zeros((max(n, 1), 4), np.float32)
        k, off = C.c_int64(0), C.c_double(0)
        self.check(self.L.dl_decode_point_cloud2(self.h, C.byref(lay), data.ctypes.data_as(C.c_void_p), n,
                                                 np.ascontiguousarray(sensor_to_tracking, np.float64), rows, C.byref(k), C.byref(off)))
        return rows[:k.value].copy(), off.value

    def decode_point_cloud2_dev(self, data_dev_ptr, num_points, point_step, offsets, time_type, sensor_to_tracking, rows_dev_ptr):
        lay = PointCloud2Layout(point_step, *[int(v) for v in offsets], int(time_type))
        k, off = C.c_int64(0), C.c_double(0)
        self.check(self.L.dl_decode_point_cloud2_dev(self.h, C.byref(lay), data_dev_ptr, num_points,
                                                     np.ascontiguousarray(sensor_to_tracking, np.float64), rows_dev_ptr,
                                                     C.byref(k), C.byref(off)))
        return k.value, off.value

    def frontend_match_batch_imu(self, options, ranges_list, origins, states_i, predicted_states, preints, submap_local_pose,
                                 hi, lo, imu_weight=1.0, gravity=(0.0, 0.0, 9.8)):
        """Front end with the IMU residual fused into each scan's solve -> (results, estimated states as 16-vectors)."""
        hb = ranges_list if isinstance(ranges_list, HostScanBatch) else HostScanBatch(ranges_list)
        n = hb.n
        origins = np.ascontiguousarray(origins, np.float32).reshape(-1, 3)
        si = (NavState * n)(*[NavState.from16(x) for x in states_i])
        sj = (NavState * n)(*[NavState.from16(x) for x in predicted_states])
        pm = (Preintegration * n)(*preints)
        out = (NavState * n)()
        imu = FrontendImu(imu_weight, (C.c_double * 3)(*gravity), C.cast(si, C.c_void_p), C.cast(sj, C.c_void_p),
                          C.cast(pm, C.c_void_p), C.cast(out, C.c_void_p))
        results = (ScanResult * n)()
        self.check(self.L.dl_frontend_match_batch_imu(self.h, C.byref(options), C.byref(imu), n, hb.pointers, hb.sizes, origins,
                                                      len(origins), np.ascontiguousarray(submap_local_pose, np.float64), hi.h,
                                                      lo.h, results))
        return results, np.array([o.to16() for o in out])

    def frontend_match_batch_imu_samples(self, options, ranges_list, origins, imu, submap_local_pose, hi, lo):
        """Front end fed with raw IMU samples (ImuSamples): pre-integration, prediction and fused solve on the device.
        -> (results, estimated states [n,16], predicted states [n,16])."""
        hb = ranges_list if isinstance(ranges_list, HostScanBatch) else HostScanBatch(ranges_list)
        n = hb.n
        origins = np.ascontiguousarray(origins, np.float32).reshape(-1, 3)
        out, pred = np.zeros((n, 16)), np.zeros((n, 16))
        results = (ScanResult * n)()
        self.check(self.L.dl_frontend_match_batch_imu_samples(self.h, C.byref(options), C.addressof(imu.struct), n, hb.pointers,
                                                              hb.sizes, origins, len(origins),
                                                              np.ascontiguousarray(submap_local_pose, np.float64), hi.h, lo.h,
                                                              results, out.ctypes.data, pred.ctypes.data))
        return results, out, pred

    def frontend_match_batch_imu_samples_dev(self, options, imu, ranges_dev_ptr, cap_rows, sizes, origins, submap_local_pose, hi,
                                             lo, results_dev_ptr, states_dev_ptr):
        sizes = np.ascontiguousarray(sizes, np.int64)
        origins = np.ascontiguousarray(origins, np.float32).reshape(-1, 3)
        self.check(self.L.dl_frontend_match_batch_imu_samples_dev(self.h, C.byref(options), C.addressof(imu.struct), len(sizes),
                                                                  ranges_dev_ptr, cap_rows, sizes, origins, len(origins),
                                                                  np.ascontiguousarray(submap_local_pose, np.float64), hi.h,
                                                                  lo.h, results_dev_ptr, states_dev_ptr))

    def frontend_submit_imu_samples(self, options, host_batch, origins, imu, submap_local_pose, hi, lo):
        hb = host_batch if isinstance(host_batch, HostScanBatch) else HostScanBatch(host_batch)
        origins = np.ascontiguousarray(origins, np.float32).reshape(-1, 3)
        self.check(self.L.dl_frontend_submit_imu_samples(self.h, C.byref(options), C.addressof(imu.struct), hb.n, hb.pointers,
                                                         hb.sizes, origins, len(origins),
                                                         np.ascontiguousarray(submap_local_pose, np.float64), hi.h, lo.h))
        self._submitted = (hb, hb.n, imu)   # keeps the host buffers alive until collect

    def frontend_collect_imu(self):
        n = self._submitted[1]
        results = (ScanResult * n)()
        states = np.zeros((n, 16))
        self.check(self.L.dl_frontend_collect_imu(self.h, n, results, states.ctypes.data))
        self._submitted = None
        return results, states

    def frontend_submit(self, options, host_batch, origins, prev_poses, cur_poses, submap_local_pose, hi, lo):
        """Streaming form: returns as soon as the batch is enqueued; frontend_collect() returns its results."""
        hb = host_batch if isinstance(host_batch, HostScanBatch) else HostScanBatch(host_batch)
        origins = np.ascontiguousarray(origins, np.float32).reshape(-1, 3)
        self.check(self.L.dl_frontend_submit(self.h, C.byref(options), hb.n, hb.pointers, hb.sizes, origins, len(origins),
                                             np.ascontiguousarray(prev_poses, np.float64),
                                             np.ascontiguousarray(cur_poses, np.float64),
                                             np.ascontiguousarray(submap_local_pose, np.float64), hi.h, lo.h))
        self._submitted = (hb, hb.n)   # keeps the host buffers alive until collect

    def frontend_collect(self):
        n = self._submitted[1]
        results = (ScanResult * n)()
        self.check(self.L.dl_frontend_collect(self.h, n, results))
        self._submitted = None
        return results

    def frontend_match_batch_dev(self, options, ranges_dev_ptr, cap_rows, sizes, origins, prev_poses, cur_poses,
                                 submap_local_pose, hi, lo, results_dev_ptr):
        sizes = np.ascontiguousarray(sizes, np.int64)
        origins = np.ascontiguousarray(origins, np.float32).reshape(-1, 3)
        self.check(self.L.dl_frontend_match_batch_dev(self.h, C.byref(options), len(sizes), ranges_dev_ptr, cap_rows,
                                                      sizes, origins, len(origins),
                                                      np.ascontiguousarray(prev_poses, np.float64),
                                                      np.ascontiguousarray(cur_poses, np.float64),
                                                      np.ascontiguousarray(submap_local_pose, np.float64), hi.h, lo.h,
                                                      results_dev_ptr))

    def fetch_results(self, results_dev_ptr, n):
        results = (ScanResult * n)()
        self.check(self.L.dl_frontend_fetch_results(self.h, results_dev_ptr, n, results))
        return results

    def submap_insert_range_data(self, hi, lo, submap_local_pose, origin, returns, high_resolution_max_range=20, hit=0.55,
                                 miss=0.49, num_free=2):
        returns = np.ascontiguousarray(returns, np.float32).reshape(-1, 3)
        opt = RangeDataInserterOptions(hit, miss, num_free, 0)
        self.check(self.L.dl_submap_insert_range_data(self.h, hi.h, lo.h, C.byref(opt),
                                                      np.ascontiguousarray(submap_local_pose, np.float64),
                                                      int(high_resolution_max_range), np.ascontiguousarray(origin, np.float32),
                                                      returns, len(returns)))

    def device_alloc(self, nbytes):
        p = C.c_void_p()
        self.check(self.L.dl_device_alloc(self.h, nbytes, C.byref(p)))
        return p

    def device_free(self, p):
        self.check(self.L.dl_device_free(self.h, p))

    def copy_to_device(self, dst, src_array):
        src_array = np.ascontiguousarray(src_array)
        self.check(self.L.dl_copy_to_device(self.h, dst, src_array.ctypes.data_as(C.c_void_p), src_array.nbytes))


class LocalTrajectoryBuilder:
    """mapping::LocalTrajectoryBuilder3D over the device path (dl_ltb_*): add_imu_data / add_range_data -> MatchingResult."""

    def __init__(self, ctx, options):
        self.ctx, self.options = ctx, options
        self.h = C.c_void_p()
        ctx.check(ctx.L.dl_ltb_create(ctx.h, C.byref(options), C.byref(self.h)))

    def close(self):
        if self.h:
            self.ctx.L.dl_ltb_destroy(self.h)
            self.h = None

    def set_initial_state(self, state16):
        s = NavState.from16(state16)
        self.ctx.check(self.ctx.L.dl_ltb_set_initial_state(self.h, C.byref(s)))

    def add_imu_data(self, time, acc, gyr):
        self.ctx.check(self.ctx.L.dl_ltb_add_imu_data(self.h, float(time), np.ascontiguousarray(acc, np.float64),
                                                      np.ascontiguousarray(gyr, np.float64)))

    def add_range_data(self, time, xyzt, origin=(0.0, 0.0, 0.0)):
        rows = np.ascontiguousarray(xyzt, np.float32).reshape(-1, 4)
        out = MatchingResult()
        self.ctx.check(self.ctx.L.dl_ltb_add_range_data(self.h, float(time), rows, len(rows), np.ascontiguousarray(origin, np.float32),
                                                        C.byref(out)))
        return out

    def add_synchronized_range_data(self, time, rows, origins):
        """rows: RANGE_DTYPE-like 32-byte RangeMeasurement records (x y z t + u64 origin index), time-sorted; origins: (k, 3)."""
        rows = np.ascontiguousarray(rows)
        origins = np.ascontiguousarray(origins, np.float32).reshape(-1, 3)
        out = MatchingResult()
        self.ctx.check(self.ctx.L.dl_ltb_add_synchronized_range_data(self.h, float(time), rows.ctypes.data, len(rows), 8, origins,
                                                                     len(origins), C.byref(out)))
        return out

    def cloud(self, which):
        n = C.c_int64(0)
        self.ctx.check(self.ctx.L.dl_ltb_get_cloud(self.h, which, None, 0, C.byref(n)))
        out = np.zeros((max(n.value, 1), 3), np.float32)
        self.ctx.check(self.ctx.L.dl_ltb_get_cloud(self.h, which, out.ctypes.data, n.value, C.byref(n)))
        return out[:n.value]

    def histogram(self):
        out = np.zeros(self.options.rotational_histogram_size, np.float32)
        self.ctx.check(self.ctx.L.dl_ltb_get_histogram(self.h, out, len(out)))
        return out

    def num_submaps(self):
        return self.ctx.L.dl_ltb_num_submaps(self.h)

    def submap(self, index):
        """-> (hi Grid view, lo Grid view, local pose, num_range_data, finished); the grids stay owned by the builder."""
        hi, lo = C.c_void_p(), C.c_void_p()
        pose = np.zeros(7)
        n, fin = C.c_int32(0), C.c_int32(0)
        self.ctx.check(self.ctx.L.dl_ltb_get_submap(self.h, index, C.byref(hi), C.byref(lo), pose, C.byref(n), C.byref(fin)))
        return Grid.borrowed(self.ctx, hi), Grid.borrowed(self.ctx, lo), pose, n.value, bool(fin.value)

    def release_submap(self, index):
        """Frees the device grids of a finished submap (dl_ltb_release_submap); submap(index) then returns NULL grid handles."""
        self.ctx.check(self.ctx.L.dl_ltb_release_submap(self.h, int(index)))

    def state(self):
        s = NavState()
        init = C.c_int32(0)
        self.ctx.check(self.ctx.L.dl_ltb_get_state(self.h, C.byref(s), C.byref(init)))
        return s.to16(), bool(init.value)


def _ltb_rows(scan, origins):
    """-> (contiguous rows, row_floats, contiguous (k, 3) float32 origins) of one scan for the dl_ltb_* calls: an (n, 4) float
    array of x y z t rows with one origin, or 32-byte RangeMeasurement records (x y z t + u64 origin index) with k origins."""
    rows = np.ascontiguousarray(scan)
    if rows.dtype.itemsize == 32 and rows.dtype.names:
        row_floats = 8
    else:
        rows = np.ascontiguousarray(rows, np.float32).reshape(-1, 4)
        row_floats = 4
    origins = np.ascontiguousarray(np.zeros((1, 3)) if origins is None else origins, np.float32).reshape(-1, 3)
    return rows, row_floats, origins


def add_range_data_batch(builders, times, scans, origins=None):
    """dl_ltb_add_range_data_batch: one add_range_data (x y z t rows) or add_synchronized_range_data (RangeMeasurement records)
    per builder, all in one call; -> one MatchingResult per builder, byte for byte the single calls' results. origins: None (one
    origin at zero each) or one origin array per builder. The builders must share a context and have equal options."""
    builders = list(builders)
    if not (len(times) == len(scans) == len(builders)) or (origins is not None and len(origins) != len(builders)):
        raise ValueError("one time, scan (and origin array) per builder")
    keep = []   # the arrays must outlive the call
    items = (LtbBatchItem * max(len(builders), 1))()
    for k, b in enumerate(builders):
        rows, row_floats, o = _ltb_rows(scans[k], None if origins is None else origins[k])
        keep += [rows, o]
        items[k] = LtbBatchItem(b.h, float(times[k]), rows.ctypes.data, len(rows), row_floats, len(o), o.ctypes.data)
    results = (MatchingResult * max(len(builders), 1))()
    if builders:
        ctx = builders[0].ctx
        ctx.check(ctx.L.dl_ltb_add_range_data_batch(len(builders), items, results))
    return [results[k] for k in range(len(builders))]


class PoseGraph3D:
    """mapping::PoseGraph3D on the fork's live loop-closure path (dl_pose_graph_3d_*): nodes from the local trajectory builders,
    submap matches from the host SURF stage -> INTRA / INTER_SUBMAP constraints and optimized poses. Node clouds are uploaded
    once into the object's device node store."""

    def __init__(self, ctx, options=None):
        self.ctx, self.options = ctx, options if options is not None else PoseGraph3DOptions.defaults()
        self.h = C.c_void_p()
        self._grids = {}   # the borrowed grids' Python handles stay alive with the graph, one entry per grid
        self._submap_grids = {}   # (trajectory, submap index) -> its two keys in _grids
        self._feeders = {}        # (trajectory, submap index) -> the LocalTrajectoryBuilder whose grids add_node_from_builder passed
        ctx.check(ctx.L.dl_pose_graph_3d_create(ctx.h, C.byref(self.options), C.byref(self.h)))

    def close(self):
        if self.h:
            self.ctx.L.dl_pose_graph_3d_destroy(self.h)
            self.h = None

    def __del__(self):
        if getattr(self, "h", None) and getattr(self.ctx, "h", None):
            self.close()

    def add_node(self, trajectory_id, time, local_pose, hi_points, lo_points, insertion_submaps, matches=()):
        """insertion_submaps: 1 or 2 (submap_index, finished, hi Grid, lo Grid, local_pose7); matches: (trajectory_id,
        submap_index, x, y, theta) of earlier finished submaps, only when insertion_submaps[0] finished -> Pg3dAddNodeInfo."""
        hi = np.ascontiguousarray(hi_points, np.float32).reshape(-1, 3)
        lo = np.ascontiguousarray(lo_points, np.float32).reshape(-1, 3)
        n = Pg3dNode()
        n.trajectory_id, n.num_insertion_submaps, n.time = int(trajectory_id), len(insertion_submaps), float(time)
        n.local_pose[:] = [float(v) for v in local_pose]
        n.high_resolution_points, n.num_high_resolution = hi.ctypes.data, len(hi)
        n.low_resolution_points, n.num_low_resolution = lo.ctypes.data, len(lo)
        for i, (index, finished, hg, lg, pose) in enumerate(insertion_submaps[:2]):
            s = n.insertion_submaps[i]
            s.submap_index, s.finished = int(index), int(bool(finished))
            s.high_resolution_grid, s.low_resolution_grid = hg.h, lg.h
            s.local_pose[:] = [float(v) for v in pose]
            keys = [g.h.value if isinstance(g.h, C.c_void_p) else g.h for g in (hg, lg)]
            self._grids[keys[0]], self._grids[keys[1]] = hg, lg
            self._submap_grids[(int(trajectory_id), int(index))] = keys
        m = (Pg3dSubmapMatch * max(len(matches), 1))(*[Pg3dSubmapMatch(int(t), int(i), float(x), float(y), float(th))
                                                        for t, i, x, y, th in matches])
        info = Pg3dAddNodeInfo()
        self._checked_forgetting_trimmed(self.ctx.L.dl_pose_graph_3d_add_node(self.h, C.byref(n), len(matches),
                                                                              C.cast(m, C.c_void_p), C.byref(info)))
        return info

    def add_node_from_builder(self, trajectory_id, builder, result, matches=(), range_data=False):
        """GlobalTrajectoryBuilder's AddNode call site: the node of a dl_ltb MatchingResult with insertion submaps, its clouds
        and the submaps' grids, local poses and finished flags from the builder. range_data=True also attaches the builder's
        range_data_in_local returns (cloud 0) to the new node (set_node_range_data), for range_data_map."""
        subs = []
        for i in range(result.num_insertion_submaps):
            index = result.insertion_submap_index[i]
            hg, lg, pose, _, finished = builder.submap(index)
            subs.append((index, finished, hg, lg, pose))
            self._feeders[(int(trajectory_id), int(index))] = builder
        info = self.add_node(trajectory_id, result.time, np.array(result.local_pose[:]), builder.cloud(2), builder.cloud(3),
                             subs, matches)
        if range_data:
            self.set_node_range_data(trajectory_id, info.node_index, builder.cloud(0))
        return info

    def set_node_range_data(self, trajectory_id, node_index, returns):
        """Attach a node's range_data_in_local returns (n x 3, the builder's local frame) to the node store
        (dl_range_data_map_set_node): once per node."""
        r = np.ascontiguousarray(returns, np.float32).reshape(-1, 3)
        self.ctx.check(self.ctx.L.dl_range_data_map_set_node(self.h, int(trajectory_id), int(node_index), r.ctypes.data, len(r)))

    def range_data_map(self, trajectory_ids=None, device=False):
        """The range-data map (dl_range_data_map): every live node with range data of the listed trajectories (None: all)
        in (trajectory, node index) order, its returns at the node's optimized pose -> (points n x 3 float32, nodes: [(trajectory
        id, node index, first point, num points, global pose7)]). device=True: points is a torch CUDA tensor on the context's
        device, filled by dl_range_data_map_dev."""
        ids = None if trajectory_ids is None else np.ascontiguousarray(trajectory_ids, np.int32).reshape(-1)
        args = (0 if ids is None else len(ids), None if ids is None else ids.ctypes.data)
        nn, npts = C.c_int32(0), C.c_int64(0)
        self.ctx.check(self.ctx.L.dl_range_data_map(self.h, *args, 0, None, C.byref(nn), 0, None, C.byref(npts)))
        nodes = (RangeDataMapNode * max(nn.value, 1))()
        if device:
            import torch
            dev = torch.device("cuda", self.ctx.device)
            points = torch.empty((max(npts.value, 1), 3), dtype=torch.float32, device=dev)
            torch.cuda.current_stream(dev).synchronize()   # the allocation is ordered on torch's stream, the fill on the context's
            self.ctx.check(self.ctx.L.dl_range_data_map_dev(self.h, *args, nn.value, C.cast(nodes, C.c_void_p), C.byref(nn),
                                                                 npts.value, points.data_ptr(), C.byref(npts)))
        else:
            points = np.zeros((max(npts.value, 1), 3), np.float32)
            self.ctx.check(self.ctx.L.dl_range_data_map(self.h, *args, nn.value, C.cast(nodes, C.c_void_p), C.byref(nn),
                                                             npts.value, points.ctypes.data, C.byref(npts)))
        return points[:npts.value], [(n.trajectory_id, n.node_index, n.first_point, n.num_points, np.array(n.global_pose[:]))
                                     for n in list(nodes)[:nn.value]]

    def _checked_forgetting_trimmed(self, status):
        """After a call that may have trimmed, whatever its status (the call empties the trimmed list when it starts, so a
        failure after some trims reports those): the graph no longer reads the trimmed submaps' grids. Their handles are
        dropped unless another submap in the graph passed the same grid, and a submap fed by add_node_from_builder has its
        grids released on that builder if the builder has finished it (its active submaps, trimmed by finish_trajectory, stay
        until the builder is closed). Then the status is checked."""
        for t, i in self.last_trimmed():
            keys = self._submap_grids.pop((t, i), ())
            still_used = {k for ks in self._submap_grids.values() for k in ks}
            for key in keys:
                if key not in still_used:
                    self._grids.pop(key, None)
            builder = self._feeders.pop((t, i), None)
            if builder is not None and builder.submap(i)[4]:
                builder.release_submap(i)
        self.ctx.check(status)

    def freeze_trajectory(self, trajectory_id):
        self.ctx.check(self.ctx.L.dl_pose_graph_3d_freeze_trajectory(self.h, int(trajectory_id)))

    def run_final_optimization(self):
        s = SolveSummary()
        self._checked_forgetting_trimmed(self.ctx.L.dl_pose_graph_3d_run_final_optimization(self.h, C.byref(s)))
        return s.as_dict()

    def trim_submap(self, trajectory_id, submap_index):
        """TrimmingHandle::MarkSubmapAsTrimmed (dl_pg3d_trim_submap)."""
        self._checked_forgetting_trimmed(self.ctx.L.dl_pg3d_trim_submap(self.h, int(trajectory_id), int(submap_index)))

    def add_pure_localization_trimmer(self, trajectory_id, num_submaps_to_keep=3):
        """PureLocalizationTrimmer (dl_pg3d_add_pure_localization_trimmer): runs after every optimization."""
        self.ctx.check(self.ctx.L.dl_pg3d_add_pure_localization_trimmer(self.h, int(trajectory_id), int(num_submaps_to_keep)))

    def finish_trajectory(self, trajectory_id):
        """FinishTrajectory (dl_pg3d_finish_trajectory): every submap finished, then the final optimization and the trimmers."""
        self._checked_forgetting_trimmed(self.ctx.L.dl_pg3d_finish_trajectory(self.h, int(trajectory_id)))

    def is_trajectory_finished(self, trajectory_id):
        f = C.c_int32(0)
        self.ctx.check(self.ctx.L.dl_pg3d_is_trajectory_finished(self.h, int(trajectory_id), C.byref(f)))
        return bool(f.value)

    def set_initial_trajectory_pose(self, from_trajectory_id, to_trajectory_id, relative_pose, time):
        """SetInitialTrajectoryPose (dl_pg3d_set_initial_trajectory_pose): relative_pose 7 (t xyz, q wxyz), time in seconds."""
        p = np.ascontiguousarray(relative_pose, np.float64).reshape(7)
        self.ctx.check(self.ctx.L.dl_pg3d_set_initial_trajectory_pose(self.h, int(from_trajectory_id), int(to_trajectory_id),
                                                                      p.ctypes.data, float(time)))

    def ids(self, trajectory_id, which=None):
        """Indices of the rows of node_poses (which = PG3D_NODE_POSES, the default) or submap_poses (PG3D_SUBMAP_POSES)."""
        which = PG3D_NODE_POSES if which is None else which
        n = C.c_int32(0)
        self.ctx.check(self.ctx.L.dl_pg3d_ids(self.h, int(trajectory_id), which, 0, None, C.byref(n)))
        out = np.zeros(max(n.value, 1), np.int32)
        self.ctx.check(self.ctx.L.dl_pg3d_ids(self.h, int(trajectory_id), which, n.value, out.ctypes.data, C.byref(n)))
        return out[:n.value].tolist()

    def last_trimmed(self):
        """[(trajectory, submap index)] trimmed by the last call that could trim."""
        n = C.c_int32(0)
        self.ctx.check(self.ctx.L.dl_pg3d_last_trimmed(self.h, 0, None, C.byref(n)))
        out = (Pg3dSubmapId * max(n.value, 1))()
        self.ctx.check(self.ctx.L.dl_pg3d_last_trimmed(self.h, n.value, C.cast(out, C.c_void_p), C.byref(n)))
        return [(s.trajectory_id, s.submap_index) for s in list(out)[:n.value]]

    def store_usage(self):
        """Node store bytes: (live, used, capacity)."""
        v = [C.c_int64(0) for _ in range(3)]
        self.ctx.check(self.ctx.L.dl_pg3d_store_usage(self.h, *[C.byref(x) for x in v]))
        return tuple(x.value for x in v)

    def _poses(self, trajectory_id, which):
        n = C.c_int32(0)
        self.ctx.check(self.ctx.L.dl_pose_graph_3d_poses(self.h, int(trajectory_id), which, 0, None, C.byref(n)))
        out = np.zeros((max(n.value, 1), 7))
        self.ctx.check(self.ctx.L.dl_pose_graph_3d_poses(self.h, int(trajectory_id), which, n.value, out.ctypes.data, C.byref(n)))
        return out[:n.value]

    def node_poses(self, trajectory_id):
        return self._poses(trajectory_id, PG3D_NODE_POSES)

    def submap_poses(self, trajectory_id):
        return self._poses(trajectory_id, PG3D_SUBMAP_POSES)

    def optimization_poses(self, trajectory_id):
        """(submap_data, node_data) poses of the optimization problem: what the next solve starts from."""
        return self._poses(trajectory_id, PG3D_OPTIMIZATION_SUBMAPS), self._poses(trajectory_id, PG3D_OPTIMIZATION_NODES)

    def local_to_global(self, trajectory_id):
        out = np.zeros(7)
        self.ctx.check(self.ctx.L.dl_pose_graph_3d_local_to_global(self.h, int(trajectory_id), out.ctypes.data))
        return out

    def constraints(self):
        """[(submap (trajectory, index), node (trajectory, index), zbar7, translation_weight, rotation_weight, tag)]"""
        n = C.c_int32(0)
        self.ctx.check(self.ctx.L.dl_pose_graph_3d_constraints(self.h, 0, None, C.byref(n)))
        out = (Pg3dConstraint * max(n.value, 1))()
        self.ctx.check(self.ctx.L.dl_pose_graph_3d_constraints(self.h, n.value, C.cast(out, C.c_void_p), C.byref(n)))
        return [((c.submap_trajectory_id, c.submap_index), (c.node_trajectory_id, c.node_index), np.array(c.zbar[:]),
                 c.translation_weight, c.rotation_weight, c.tag) for c in list(out)[:n.value]]

    def last_searches(self):
        """The (node, submap) searches of the last add_node call: [(submap id, node id, guess7, Constraint)]"""
        n = C.c_int32(0)
        self.ctx.check(self.ctx.L.dl_pose_graph_3d_last_searches(self.h, 0, None, C.byref(n)))
        out = (Pg3dSearch * max(n.value, 1))()
        self.ctx.check(self.ctx.L.dl_pose_graph_3d_last_searches(self.h, n.value, C.cast(out, C.c_void_p), C.byref(n)))
        return [((s.submap_trajectory_id, s.submap_index), (s.node_trajectory_id, s.node_index), np.array(s.pose_guess[:]), s.result)
                for s in list(out)[:n.value]]

    def store_bytes(self):
        """(cloud bytes uploaded since creation, node store capacity in bytes)"""
        up, cap = C.c_int64(0), C.c_int64(0)
        self.ctx.check(self.ctx.L.dl_pose_graph_3d_store_bytes(self.h, C.byref(up), C.byref(cap)))
        return up.value, cap.value


def seconds_to_ticks(seconds):
    """Seconds -> universal ticks of 100 ns, llround(t * 1e7) (rounded half away from zero), for node times given in seconds
    (dl_pg3d_node::time) where the map writer takes ticks (proto::Trajectory::Node::timestamp)."""
    t = np.asarray(seconds, np.float64) * 1e7
    whole = np.trunc(t)
    return (whole + np.sign(t) * (np.abs(t - whole) >= 0.5)).astype(np.int64)


class MapWriter:
    """The assets writer's point pipeline (dl_map_writer_*): trajectory lookup and transform to the map, optional
    min_max_range_filter and voxel_filter_and_remove_moving_objects, with the restart protocol: stream every message through
    process(), then flush(); repeat while flush() returns True. Output points come from the final pass only."""

    def __init__(self, ctx, range_filter=None, outlier_voxel_size=0.0):
        """range_filter: None or (min_range, max_range)."""
        self.ctx = ctx
        o = MapWriterOptions()
        if range_filter is not None:
            o.range_filter, o.min_range, o.max_range = 1, float(range_filter[0]), float(range_filter[1])
        o.outlier_voxel_size = float(outlier_voxel_size)
        self.h = C.c_void_p()
        ctx.check(ctx.L.dl_map_writer_create(ctx.h, C.byref(o), C.byref(self.h)))

    def close(self):
        if self.h:
            self.ctx.L.dl_map_writer_destroy(self.h)
            self.h = None

    def __del__(self):
        if getattr(self, "h", None) and getattr(self.ctx, "h", None):
            self.close()

    def add_trajectory(self, trajectory_id, times_ticks, poses):
        t = np.ascontiguousarray(times_ticks, np.int64)
        p = np.ascontiguousarray(poses, np.float64).reshape(-1, 7)
        self.ctx.check(self.ctx.L.dl_map_writer_add_trajectory(self.h, int(trajectory_id), len(t), t.ctypes.data, p.ctypes.data))

    def add_pose_graph_trajectory(self, graph, trajectory_id, node_times_seconds):
        """A PoseGraph3D trajectory: its node poses (GetTrajectoryNodePoses) at the nodes' times, converted with seconds_to_ticks."""
        self.add_trajectory(trajectory_id, seconds_to_ticks(node_times_seconds), graph.node_poses(trajectory_id))

    def add_color(self, frame_id, rgb):
        """color_points: messages whose frame_id (an integer) equals this one get every point coloured rgb / 255.f; rgb are
        the Lua values, converted with static_cast<uint8>. Added before processing begins, in pipeline order."""
        c = MapWriterColor()
        c.frame_id = int(frame_id)
        c.rgb[:] = [int(v) & 0xFF for v in rgb]
        self.ctx.check(self.ctx.L.dl_map_writer_add_color(self.h, C.byref(c)))

    def add_xray(self, voxel_size, transform7):
        """write_xray_image of the final pass's points (transform: Rigid3d t, q wxyz) -> the stage number for xray_image()."""
        x = MapWriterXray()
        x.voxel_size = float(voxel_size)
        x.transform[:] = [float(v) for v in transform7]
        stage = C.c_int32(0)
        self.ctx.check(self.ctx.L.dl_map_writer_add_xray(self.h, C.byref(x), C.byref(stage)))
        return stage.value

    def xray_image(self, stage):
        """After the final flush: (height, width) uint32 Cairo ARGB32 words, (0, 0) for an empty bounding box."""
        w, h = C.c_int32(0), C.c_int32(0)
        self.ctx.check(self.ctx.L.dl_map_writer_xray_image(self.h, int(stage), 0, None, C.byref(w), C.byref(h)))
        img = np.zeros((h.value, w.value), np.uint32)
        if img.size:
            self.ctx.check(self.ctx.L.dl_map_writer_xray_image(self.h, int(stage), img.size, img.ctypes.data, C.byref(w),
                                                               C.byref(h)))
        return img

    def add_probability_grid(self, resolution, hit, miss, insert_free_space=True):
        """write_probability_grid / write_ros_map of the final pass's batches (range_data_inserter: hit_probability,
        miss_probability, insert_free_space) -> the stage number for probability_grid()."""
        o = MapWriterGridOptions()
        o.resolution, o.hit_probability, o.miss_probability = float(resolution), float(hit), float(miss)
        o.insert_free_space = int(bool(insert_free_space))
        stage = C.c_int32(0)
        self.ctx.check(self.ctx.L.dl_map_writer_add_probability_grid(self.h, C.byref(o), C.byref(stage)))
        return stage.value

    def probability_grid(self, stage):
        """After the final flush: (info dict, cells (height, width) uint16, pixels (height, width) uint8) of the cropped box
        (ComputeCroppedLimits; DrawProbabilityGrid's grey values, unrotated)."""
        info = MapWriterGridInfo()
        self.ctx.check(self.ctx.L.dl_map_writer_probability_grid(self.h, int(stage), C.byref(info), 0, None, None))
        cells = np.zeros((info.height, info.width), np.uint16)
        pixels = np.zeros((info.height, info.width), np.uint8)
        self.ctx.check(self.ctx.L.dl_map_writer_probability_grid(self.h, int(stage), C.byref(info), cells.size,
                                                                 cells.ctypes.data, pixels.ctypes.data))
        return info.as_dict(), cells, pixels

    @staticmethod
    def messages(msgs):
        """[(stamp ticks, first_row, num_rows, trajectory_id, sensor_to_tracking7[, frame_id])] -> a dl_map_message array"""
        arr = (MapMessage * max(len(msgs), 1))()
        for k, msg in enumerate(msgs):
            stamp, first, n, traj, s2t = msg[:5]
            arr[k].stamp, arr[k].first_row, arr[k].num_rows, arr[k].trajectory_id = int(stamp), int(first), int(n), int(traj)
            arr[k].frame_id = int(msg[5]) if len(msg) > 5 else 0
            arr[k].sensor_to_tracking[:] = [float(v) for v in s2t]
        return arr

    def process(self, msgs, rows):
        """rows: (n, 4) float32 x y z t -> (points (k, 3) float32, origins (len(msgs), 3), info dict)"""
        rows = np.ascontiguousarray(rows, np.float32).reshape(-1, 4)
        m = self.messages(msgs)
        total = sum(int(x[2]) for x in msgs)
        out = np.zeros((max(total, 1), 3), np.float32)
        origins = np.zeros((max(len(msgs), 1), 3), np.float32)
        n, info = C.c_int64(0), MapWriterInfo()
        self.ctx.check(self.ctx.L.dl_map_writer_process(self.h, len(msgs), C.cast(m, C.c_void_p), rows.ctypes.data, len(rows),
                                                        out.ctypes.data, C.byref(n), origins.ctypes.data, C.byref(info)))
        return out[:n.value], origins[:len(msgs)], info.as_dict()

    def process_dev(self, msgs, rows_dev_ptr, num_rows, points_dev_ptr):
        """Device rows in, device points out -> (number of points, origins, info dict)"""
        m = self.messages(msgs)
        origins = np.zeros((max(len(msgs), 1), 3), np.float32)
        n, info = C.c_int64(0), MapWriterInfo()
        self.ctx.check(self.ctx.L.dl_map_writer_process_dev(self.h, len(msgs), C.cast(m, C.c_void_p), rows_dev_ptr, int(num_rows),
                                                            points_dev_ptr, C.byref(n), origins.ctypes.data, C.byref(info)))
        return n.value, origins[:len(msgs)], info.as_dict()

    def flush(self):
        """True if every message must be streamed again."""
        r = C.c_int32(0)
        self.ctx.check(self.ctx.L.dl_map_writer_flush(self.h, C.byref(r)))
        return bool(r.value)

    def voxels(self):
        """(cells (k, 3) int32, hits, rays), sorted by cell index"""
        n = C.c_int64(0)
        self.ctx.check(self.ctx.L.dl_map_writer_voxels(self.h, 0, None, None, None, C.byref(n)))
        cells = np.zeros((max(n.value, 1), 3), np.int32)
        hits, rays = np.zeros(max(n.value, 1), np.int32), np.zeros(max(n.value, 1), np.int32)
        self.ctx.check(self.ctx.L.dl_map_writer_voxels(self.h, n.value, cells.ctypes.data, hits.ctypes.data, rays.ctypes.data,
                                                       C.byref(n)))
        return cells[:n.value], hits[:n.value], rays[:n.value]

    def write_map(self, msgs, rows):
        """Every pass over the same messages; the final pass's points."""
        while True:
            pts, origins, info = self.process(msgs, rows)
            if not self.flush():
                return pts, origins, info


def write_pcd(path, points):
    """io::PcdWritingPointsProcessor (io/pcd_writing_points_processor.cc:35-66): binary PCD v0.7, x y z floats, no colour,
    WIDTH and POINTS zero-padded to 15 digits, 12 bytes per point in order."""
    pts = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
    n = len(pts)
    header = ("# generated by Cartographer\nVERSION .7\nFIELDS x y z\nSIZE 4 4 4\nTYPE F F F\nCOUNT 1 1 1\n"
              f"WIDTH {n:015d}\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS {n:015d}\nDATA binary\n")
    with open(path, "wb") as f:
        f.write(header.encode())
        f.write(pts.tobytes())


def roll_pitch_yaw(roll, pitch, yaw):
    """transform::RollPitchYaw (transform/rigid_transform.cc:40-46): AngleAxisd(yaw, Z) * AngleAxisd(pitch, Y) *
    AngleAxisd(roll, X), each AngleAxis (cos(a/2), sin(a/2) * axis), the products in Eigen's order -> (w, x, y, z)."""
    def product(a, b):
        aw, ax, ay, az = a
        bw, bx, by, bz = b
        return (aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                aw * by + ay * bw + az * bx - ax * bz, aw * bz + az * bw + ax * by - ay * bx)
    r = (math.cos(0.5 * roll), math.sin(0.5 * roll), 0.0, 0.0)
    p = (math.cos(0.5 * pitch), 0.0, math.sin(0.5 * pitch), 0.0)
    y = (math.cos(0.5 * yaw), 0.0, 0.0, math.sin(0.5 * yaw))
    return product(product(y, p), r)


def png_bytes(argb):
    """An 8-bit RGB PNG (colour type 2, every X-ray pixel is opaque) of (height, width) Cairo ARGB32 words: filter 0 on every
    row, a zlib stream of stored deflate blocks (at most 65535 bytes each), one IDAT chunk. The same bytes as
    io::WritePng (dliom_b200.hpp)."""
    img = np.ascontiguousarray(argb, np.uint32)
    h, w = img.shape
    if h == 0 or w == 0:
        raise ValueError("png_bytes: an empty image has no PNG")
    rgb = np.stack([(img >> 16) & 0xFF, (img >> 8) & 0xFF, img & 0xFF], axis=-1).astype(np.uint8)
    raw = np.concatenate([np.zeros((h, 1), np.uint8), rgb.reshape(h, 3 * w)], axis=1).tobytes()
    blocks = [raw[k:k + 65535] for k in range(0, len(raw), 65535)]
    z = bytearray(b"\x78\x01")
    for k, b in enumerate(blocks):
        z += struct.pack("<BHH", int(k == len(blocks) - 1), len(b), len(b) ^ 0xFFFF) + b
    z += struct.pack(">I", _adler32(raw))

    def chunk(kind, data):
        return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", _crc32(kind + data))
    return (b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0)) + chunk(b"IDAT", bytes(z))
            + chunk(b"IEND", b""))


def write_png(path, argb):
    """png_bytes(argb) into path."""
    data = png_bytes(argb)
    with open(path, "wb") as f:
        f.write(data)


def grey_argb(pixels):
    """(height, width) uint8 grey values -> Cairo ARGB32 words (r = g = b), what png_bytes takes."""
    v = np.asarray(pixels, np.uint32)
    return 0xFF000000 | (v << 16) | (v << 8) | v


def write_probability_grid_png(path, pixels):
    """write_probability_grid (draw_trajectories = false): the grey image of MapWriter.probability_grid as an RGB PNG."""
    write_png(path, grey_argb(pixels))


def ros_map_bytes(info, pixels, pgm_filename):
    """write_ros_map (ros_map_writing_points_processor.cc:59-80, ros_map.cc): the image rotated 90 degrees clockwise
    (Image::Rotate90DegreesClockwise), WritePgm's bytes and WriteYaml's bytes (std::to_string is %f) -> (pgm, yaml)."""
    rotated = np.rot90(np.asarray(pixels, np.uint8), -1)
    height, width = rotated.shape
    res = info["resolution"]
    pgm = (f"P5\n# Cartographer map; {res:f} m/pixel\n{width} {height}\n255\n").encode() + rotated.tobytes()
    origin_x = info["max_x"] - (info["offset_y"] + width) * res
    origin_y = info["max_y"] - (info["offset_x"] + height) * res
    yaml = (f"image: {pgm_filename}\nresolution: {res:f}\norigin: [{origin_x:f}, {origin_y:f}, 0.0]\nnegate: 0\n"
            "occupied_thresh: 0.65\nfree_thresh: 0.196\n").encode()
    return pgm, yaml


def write_ros_map(filestem, info, pixels):
    """<filestem>.pgm and <filestem>.yaml as the reference writes them (the YAML names the PGM as opened)."""
    pgm, yaml = ros_map_bytes(info, pixels, filestem + ".pgm")
    with open(filestem + ".pgm", "wb") as f:
        f.write(pgm)
    with open(filestem + ".yaml", "wb") as f:
        f.write(yaml)


_CRC_TABLE = None


def _crc32(data):
    """CRC-32 of PNG (ISO 3309, reflected polynomial 0xEDB88320), table-driven."""
    global _CRC_TABLE
    if _CRC_TABLE is None:
        t = np.arange(256, dtype=np.uint32)
        for _ in range(8):
            t = np.where(t & 1, np.uint32(0xEDB88320) ^ (t >> 1), t >> 1).astype(np.uint32)
        _CRC_TABLE = [int(v) for v in t]
    c = 0xFFFFFFFF
    for b in data:
        c = _CRC_TABLE[(c ^ b) & 0xFF] ^ (c >> 8)
    return c ^ 0xFFFFFFFF


def _adler32(data):
    """Adler-32 of zlib (RFC 1950): sums modulo 65521, over blocks of 5552 bytes so that int64 sums cannot overflow."""
    a, b = 1, 0
    arr = np.frombuffer(data, np.uint8).astype(np.int64)
    for k in range(0, len(arr), 5552):
        blk = arr[k:k + 5552]
        n = len(blk)
        b = (b + n * a + int(np.dot(np.arange(n, 0, -1, dtype=np.int64), blk))) % 65521
        a = (a + int(blk.sum())) % 65521
    return (b << 16) | a


def comm_unique_id():
    """128 bytes from ncclGetUniqueId (rank 0 calls this and distributes the bytes)."""
    buf = (C.c_uint8 * 128)()
    st = lib().dl_comm_unique_id(C.cast(buf, C.c_void_p))
    if st != 0:
        raise DlError(st, (lib().dl_comm_last_error() or b"").decode())
    return bytes(buf)


class Comm:
    """NCCL communicator owned by the C-ABI library (dl_comm), bound to one Context (its stream carries the collectives)."""

    def __init__(self, ctx, unique_id, rank, world):
        self.ctx, self.rank, self.world = ctx, rank, world
        self.h = C.c_void_p()
        idbuf = (C.c_uint8 * 128)(*unique_id)
        ctx.check(ctx.L.dl_comm_create(ctx.h, C.cast(idbuf, C.c_void_p), rank, world, C.byref(self.h)))

    def close(self):
        if self.h:
            self.ctx.L.dl_comm_destroy(self.h)
            self.h = None

    def all_gather_dev(self, send_ptr, recv_ptr, bytes_per_rank):
        self.ctx.check(self.ctx.L.dl_comm_all_gather_dev(self.h, send_ptr, recv_ptr, bytes_per_rank))

    def all_reduce_f64_dev(self, ptr, count):
        self.ctx.check(self.ctx.L.dl_comm_all_reduce_f64_dev(self.h, ptr, count))

    def broadcast_dev(self, ptr, nbytes, root):
        self.ctx.check(self.ctx.L.dl_comm_broadcast_dev(self.h, ptr, nbytes, root))


class Grid:
    """Device mirror of a HybridGrid. Fill with the proto layout (x, y, z, value arrays), then sync()."""

    def __init__(self, ctx, resolution):
        self.ctx = ctx
        h = C.c_void_p()
        ctx.check(ctx.L.dl_grid_create(ctx.h, np.float32(resolution), C.byref(h)))
        self.h = h

    @classmethod
    def borrowed(cls, ctx, handle):
        """A view of a grid owned by someone else (a LocalTrajectoryBuilder's submap): never destroyed from here."""
        g = cls.__new__(cls)
        g.ctx, g.h, g._borrowed = ctx, handle, True
        return g

    def close(self):
        if getattr(self, "h", None) and getattr(self.ctx, "h", None) and not getattr(self, "_borrowed", False):
            self.ctx.L.dl_grid_destroy(self.h)
        self.h = None

    def __del__(self):
        self.close()

    def set_cells(self, xs, ys, zs, values, sync=True):
        xs, ys, zs = (np.ascontiguousarray(a, np.int32) for a in (xs, ys, zs))
        values = np.ascontiguousarray(values, np.uint16)
        self.ctx.check(self.ctx.L.dl_grid_set_cells(self.h, len(xs), xs, ys, zs, values))
        if sync:
            self.sync()

    def sync(self):
        self.ctx.check(self.ctx.L.dl_grid_sync(self.h))

    @property
    def num_bricks(self):
        return self.ctx.L.dl_grid_num_bricks(self.h)

    def lookup(self, xyz):
        xyz = np.ascontiguousarray(xyz, np.int32).reshape(-1, 3)
        out = np.zeros(max(len(xyz), 1), np.uint16)
        self.ctx.check(self.ctx.L.dl_grid_lookup(self.ctx.h, self.h, len(xyz), xyz, out))
        return out[:len(xyz)]

    def interpolate(self, xyz):
        xyz = np.ascontiguousarray(xyz, np.float64).reshape(-1, 3)
        out = np.zeros((max(len(xyz), 1), 4))
        self.ctx.check(self.ctx.L.dl_grid_interpolate(self.ctx.h, self.h, len(xyz), xyz, out))
        return out[:len(xyz)]

    def insert_range_data(self, origin, returns, hit=0.55, miss=0.49, num_free=2):
        """RangeDataInserter3D::Insert on the device grid (points already in the grid frame)."""
        returns = np.ascontiguousarray(returns, np.float32).reshape(-1, 3)
        opt = RangeDataInserterOptions(hit, miss, num_free, 0)
        self.ctx.check(self.ctx.L.dl_grid_insert_range_data(self.ctx.h, self.h, C.byref(opt),
                                                            np.ascontiguousarray(origin, np.float32), returns, len(returns)))

    def export(self):
        """(x, y, z, value) of every non-zero cell, in the reference's HybridGrid iteration order."""
        n = C.c_int64(0)
        self.ctx.check(self.ctx.L.dl_grid_export_cells(self.h, 0, None, None, None, None, C.byref(n)))
        xs, ys, zs = (np.zeros(max(n.value, 1), np.int32) for _ in range(3))
        vs = np.zeros(max(n.value, 1), np.uint16)
        vp = lambda arr: arr.ctypes.data_as(C.c_void_p)
        self.ctx.check(self.ctx.L.dl_grid_export_cells(self.h, n.value, vp(xs), vp(ys), vp(zs), vp(vs), C.byref(n)))
        return xs[:n.value], ys[:n.value], zs[:n.value], vs[:n.value]

    @staticmethod
    def from_oracle(ctx, oracle_grid):
        g = Grid(ctx, oracle_grid.resolution)
        g.set_cells(*oracle_grid.export())
        return g
