// Argument blocks of the batched front-end kernels (dl_frontend.cu, dl_imu.cu) and their launchers.
#pragma once
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

}  // namespace dl
