// Argument blocks of the batched front-end kernels (dl_frontend.cu, dl_imu.cu) and their launchers.
#pragma once
#include <functional>

#include "dl_internal.cuh"

namespace dl {

// Eigen's QuaternionBase::slerp(t, b) from a, in two halves: the part that depends on the two quaternions only (theta =
// acos|d|, sin(theta), the |d| >= 1 - eps and d < 0 switches) and the per-t blend. Host and device, double arithmetic.
struct SlerpConstants {
  double theta, sin_theta;
  int linear, negative_dot;
};
DL_HD SlerpConstants slerp_constants(const Quatd& a, const Quatd& b) {
  SlerpConstants c;
  const double d = (a.x * b.x + a.y * b.y) + (a.z * b.z + a.w * b.w);  // a.dot(b)
  const double abs_d = fabs(d);
  const double one = 1.0 - 2.220446049250313e-16;
  c.linear = abs_d >= one;
  c.negative_dot = d < 0;
  c.theta = c.linear ? 0.0 : acos(abs_d);
  c.sin_theta = c.linear ? 1.0 : sin(c.theta);
  return c;
}
DL_HD Quatd slerp(const Quatd& a, const Quatd& b, double t, const SlerpConstants& c) {
  double scale0, scale1;
  if (c.linear) {
    scale0 = 1.0 - t;
    scale1 = t;
  } else {
    scale0 = sin((1.0 - t) * c.theta) / c.sin_theta;
    scale1 = sin(t * c.theta) / c.sin_theta;
  }
  if (c.negative_dot) scale1 = -scale1;
  return {scale0 * a.w + scale1 * b.w, scale0 * a.x + scale1 * b.x, scale0 * a.y + scale1 * b.y, scale0 * a.z + scale1 * b.z};
}

// Per-scan constants of the deskew, prepared on the host with the reference's double arithmetic (LTB:426-428,
// LTB:871-879): prev = previous optimised pose, cur = IMU-predicted pose at scan end, rel = prev^-1 * cur, and the
// scan-constant half of Eigen's slerp from the identity to rel.q.
struct ScanConstants {
  Rigidd prev, cur, rel;
  SlerpConstants slerp;
};

// LTB:426-428 and the scan-constant half of Eigen's slerp, in the reference's double arithmetic. Host and device.
DL_HD ScanConstants make_scan_constants(const Rigidd& prev, const Rigidd& cur) {
  ScanConstants c;
  c.prev = prev;
  c.cur = cur;
  c.rel = compose(inverse(c.prev), c.cur);
  c.slerp = slerp_constants(Quatd{1.0, 0.0, 0.0, 0.0}, c.rel.q);
  return c;
}

// Device-side preparation of the IMU-coupled front end (dl_imu.cu), one warp per scan: from the pre-integration of the
// samples since the previous scan and the state there -> the predicted state (LTB:188-199), the deskew constants, the
// factor of the fused solve in the submap frame (incl. the 15x15 information matrix) and the solve's initial state.
struct ImuPrepareArgs {
  int count;
  const dl_preintegration* preint;
  const dl_nav_state* states_i;  // local frame
  const Rigidd* to_submap;       // per scan: inverse of its matching submap's local pose
  double gravity[3];
  double imu_weight;
  ScanConstants* scans;
  ImuTerm* terms;
  double* init16;                // 16 doubles per scan: p q v ba bg of the prediction, submap frame
  dl_nav_state* predicted;       // local frame
  int32_t* ok;                   // 0: the pre-integration covariance is not positive definite (or no samples)
};
int launch_imu_prepare(dl_context* ctx, const ImuPrepareArgs& a);

// Fused front half (dl_frontend.cu): rows per tile, and the most hash partitions a scan's tile winners are split into.
constexpr int kFrontendTile = 2048;
constexpr int kFrontendParts = 256;
struct FrontendArgs {
  const float* ranges;   // scan b starts at row b * in_cap; rows of row_floats floats (3: x y z, 4: x y z t, 8: + u64 origin index)
  const int32_t* run_offsets;    // row_floats == 3: per-point times as runs (dl_frontend_options::time_run_*), device copies
  const int32_t* run_first_row;
  const float* run_value;
  float* run_pose;               // optional: deskew pose of every run, 8 floats (t xyz, q wxyz, pad), fe_run_poses
  int max_runs;                  // most runs any scan of the batch has
  int64_t in_cap;
  int row_floats;
  int first_scan;        // kernels handle scans [first_scan, first_scan + gridDim.y): lets sub-batches pipeline
  const int32_t* counts;
  const ScanConstants* scans;
  const float* origins;
  const int32_t* origin_base;    // per scan: its first origin in `origins` (a row's origin index counts from there)
  int64_t cap;           // per-scan capacity of every per-point array below
  float first_resolution, second_resolution, min_range, max_range;
  double scan_period;
  uint32_t* first_bits;          // per scan one bitmap of bit_words words: bit i = point i survives the first filter
  int4* stage;                   // per scan one 2048-entry segment per row tile: the tile winners grouped by hash partition
  int32_t* part_ends;            // per scan and row tile, kFrontendParts ints: end of each partition's entries in its segment
  uint32_t* spill;               // per scan 2 slots per stage entry: tables of the partitions too large for shared memory
  int32_t* spill_used;           // per scan 2 (first, second filter): slots of `spill` taken so far
  int idx_bits, axis_bits;       // widths of the index field and of one axis of the key
  uint32_t* bits;                // per scan two bitmaps (returns, misses) of bit_words words: bit i = point i survives
  int64_t bit_words;             // ceil(cap / 32)
  float* local;                  // float4 per input row: local-frame point of a first-filter survivor + class in .w
  float* returns_tracking;
  float* misses_tracking;
  int32_t *n_first, *n_returns_local, *n_returns, *n_misses, *last_index;
  float* current_pose;
  int32_t* error_flag;            // one per scan
};
int launch_fe_prepare(dl_context* ctx, const FrontendArgs& a, int batch);
int launch_fe_first_filter(dl_context* ctx, FrontendArgs a, int first_scan, int num_scans);
int launch_fe_rest(dl_context* ctx, FrontendArgs a, int first_scan, int batch);

struct ResultArgs {
  int batch;
  const int32_t* first_counts;
  const int32_t* return_counts;
  const int32_t* miss_counts;
  const int32_t* adaptive_counts;  // 2 per scan: high, low resolution
  const int32_t* adaptive_cropped;
  const int32_t* adaptive_passes;
  const float* rtcsm_scores;       // optional
  const NlsOutput* nls;
  const FusedOutput* fused;        // optional: the fused (IMU) solve's output replaces `nls`
  const Rigidd* submap;            // per scan: the local pose of its matching submap
  const int32_t* error_flag;       // per scan: set by the fused front half when a voxel key could not be packed
  const int32_t* imu_ok;           // optional: 0 = the scan's IMU factor could not be formed (result ok = -2)
  dl_nav_state* states_out;        // optional (fused solve): the estimated state in the LOCAL frame
  dl_scan_result* results;
};

int launch_gather_rows(dl_context* ctx, const float* in, int64_t cap_in, int pairs_per_cloud, const int32_t* keep,
                       const int32_t* keep_counts, int64_t cap_out, float* out, int pairs);
int launch_initial_pose(dl_context* ctx, int batch, const float* current_pose, const Rigidd* submap_inverse,
                        double* initial_pose, double* target_translation);
int launch_finalize_results(dl_context* ctx, const ResultArgs& a);

// ---- the batched front end's host side (dl_frontend.cu), shared with the trajectory builders' batch (dl_ltb.cu)
// The submaps a front-end batch matches against: one for every scan (the public front-end entry points) or one per scan
// (dl_ltb_add_range_data_batch, whose scans come from different trajectories).
struct DL_SHARED SubmapSet {
  const double* poses = nullptr;             // 7 doubles: the local pose, once or per scan
  const dl_grid* const* hi = nullptr;        // one grid, or one per scan
  const dl_grid* const* lo = nullptr;
  bool per_scan = false;
  const double* pose(int b) const { return poses + (per_scan ? 7 * b : 0); }
  const dl_grid* high(int b) const { return hi[per_scan ? b : 0]; }
  const dl_grid* low(int b) const { return lo[per_scan ? b : 0]; }
};
// The single-submap form; the grid pointers must outlive the call.
struct DL_SHARED OneSubmap : SubmapSet {
  const dl_grid* h;
  const dl_grid* l;
  OneSubmap(const double* pose7, const dl_grid* hi_grid, const dl_grid* lo_grid) : h(hi_grid), l(lo_grid) {
    poses = pose7;
    hi = &h;
    lo = &l;
  }
  OneSubmap(const OneSubmap&) = delete;
};

struct DL_SHARED FrontendBuffers {
  int batch = 0;
  int64_t cap = 0, tcap = 0;
  int32_t *counts0, *n1, *n_ret, *n2, *n3, *countsA, *npassesA, *croppedA;
  uint32_t *tableA, *scratchA;
  int32_t* keepA;
  float *returns_tracking, *misses_tracking, *clouds, *current_pose, *origins, *passesA, *rtcsm_scores;
  int32_t* rtcsm_nonpositive = nullptr;  // pre-match only (carve_prematch): per scan, a candidate scored <= 0 (CHECK_GT)
  // fused front half
  int64_t bit_words = 0;
  uint32_t* bits;              // two survivor bitmaps per scan
  uint32_t* first_bits;        // the first filter's survivor bitmap per scan
  int4* stage;                 // tile winners by hash partition, and their ends per tile (dl_frontend.cu)
  int32_t *part_ends, *spill_used;
  uint32_t* spill;
  int32_t *last_index, *error_flag;
  float* local4;
  ScanConstants* scans;
  AdaptiveParams* filters;
  Rigidd *submap, *submap_inverse;  // per scan: its matching submap's local pose and the inverse (host arithmetic)
  int32_t* origin_base;             // per scan: its first origin in `origins`
  double *initial_pose, *target;
  NlsProblem* problems;
  NlsOutput* nls_out;
  // 12-byte rows only (carve_time_runs)
  int32_t *run_offsets = nullptr, *run_first_row = nullptr;
  float *run_value = nullptr, *run_pose = nullptr;
};

// IMU coupling of one front-end run: either finished pre-integrations (`host`, factors built on the host) or raw samples
// (`samples`, everything on the device), and its device buffers (carve_imu).
struct DL_SHARED ImuRun {
  const dl_frontend_imu* host = nullptr;
  const dl_frontend_imu_samples* samples = nullptr;
  dl_nav_state* d_states_out = nullptr;  // in: optional caller-provided device buffer for the estimated states
  ImuTerm* d_terms = nullptr;
  double* d_init16 = nullptr;
  FusedOutput* d_fused = nullptr;
  dl_nav_state* d_states = nullptr;      // estimated states, local frame
  // raw samples only
  int32_t* d_off = nullptr;
  double *d_dt = nullptr, *d_acc = nullptr, *d_gyr = nullptr;
  dl_nav_state* d_si = nullptr;
  dl_preintegration* d_pre = nullptr;
  dl_nav_state* d_predicted = nullptr;   // predicted states, local frame
  int32_t* d_ok = nullptr;               // per scan: its IMU factor could be formed
};

// Where the scans of a batch are: host rows, one pointer per scan, which the batch uploads into its scratch; or device rows
// (scan b at row b * cap_rows) with a caller-provided device buffer for the results (and, with raw IMU samples, one for the
// estimated states in ImuRun::d_states_out).
struct DL_SHARED FrontendScans {
  const void* const* host = nullptr;
  bool on_device = false;
  const void* dev = nullptr;
  int64_t cap_rows = 0;
  dl_scan_result* results_dev = nullptr;
};

// Validates, reserves, carves and enqueues one front-end batch: the one place that sizes a batch's scratch. On return
// *d_results_out holds the device results (not yet synchronised).
// `more` (optional) carves the caller's own buffers into the same reservation, after the batch's: they stay valid as long as the
// batch's (the trajectory builders' batch keeps the tracking-frame clouds on the device until insertion has read them).
// origin_base (optional): per scan, where its origins start in `origins`.
DL_SHARED int frontend_enqueue(dl_context* ctx, const dl_frontend_options* options, int num_scans, const FrontendScans& in,
                               const int64_t* sizes, const float* origins, int num_origins, const double* prev_poses,
                               const double* predicted_poses, const SubmapSet& submaps, dl_scan_result** d_results_out,
                               ImuRun* imu = nullptr, FrontendBuffers* buffers_out = nullptr, const int32_t* origin_base = nullptr,
                               const std::function<void(Arena&)>* more = nullptr);
// The fused solve refuses only_optimize_yaw; the raw IMU samples of `num_scans` scans.
DL_SHARED int check_imu_options(dl_context* ctx, const dl_frontend_options* options);
DL_SHARED int check_imu_samples(dl_context* ctx, const dl_frontend_options* options, const dl_frontend_imu_samples* imu,
                                int num_scans);

}  // namespace dl
