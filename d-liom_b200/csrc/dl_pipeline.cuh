// Argument blocks of the batched front-end kernels (dl_ingest.cu) and their launchers.
#pragma once
#include "dl_internal.cuh"

namespace dl {

// Per-scan constants of the deskew, prepared on the host with the reference's double arithmetic (LTB:426-428,
// LTB:871-879): prev = previous optimised pose, cur = IMU-predicted pose at scan end, rel = prev^-1 * cur, and the
// scan-constant part of Eigen's slerp (theta = acos|d|, sin(theta), the |d| >= 1 - eps and d < 0 switches).
struct ScanConstants {
  Rigidd prev, cur, rel;
  double theta, sin_theta;
  int linear_slerp, negative_dot;
};

// LTB:426-428 and the scan-constant half of Eigen's slerp, in the reference's double arithmetic. Host and device.
DL_HD ScanConstants make_scan_constants(const Rigidd& prev, const Rigidd& cur) {
  ScanConstants c;
  c.prev = prev;
  c.cur = cur;
  c.rel = compose(inverse(c.prev), c.cur);
  const double d = (0.0 * c.rel.q.x + 0.0 * c.rel.q.y) + (0.0 * c.rel.q.z + 1.0 * c.rel.q.w);  // Identity.dot(rel.q)
  const double abs_d = fabs(d);
  const double one = 1.0 - 2.220446049250313e-16;
  c.linear_slerp = abs_d >= one;
  c.negative_dot = d < 0;
  c.theta = c.linear_slerp ? 0.0 : acos(abs_d);
  c.sin_theta = c.linear_slerp ? 1.0 : sin(c.theta);
  return c;
}

// Device-side preparation of the IMU-coupled front end (dl_imu.cu), one warp per scan: from the pre-integration of the
// samples since the previous scan and the state there -> the predicted state (LTB:188-199), the deskew constants, the
// factor of the fused solve in the submap frame (incl. the 15x15 information matrix) and the solve's initial state.
struct ImuPrepareArgs {
  int count;
  const dl_preintegration* preint;
  const dl_nav_state* states_i;  // local frame
  Rigidd to_submap;              // inverse of the submap's local pose
  double gravity[3];
  double imu_weight;
  ScanConstants* scans;
  ImuTerm* terms;
  double* init16;                // 16 doubles per scan: p q v ba bg of the prediction, submap frame
  dl_nav_state* predicted;       // local frame
  int32_t* ok;                   // 0: the pre-integration covariance is not positive definite (or no samples)
};
int launch_imu_prepare(dl_context* ctx, const ImuPrepareArgs& a);

struct IngestArgs {
  const float* ranges;        // all scans, RangeMeasurement rows (8 floats); scan b starts at row b * in_cap
  int64_t in_cap;
  const ScanConstants* scans;
  const float* origins;       // 3 floats per sensor
  const int32_t* keep;        // first voxel filter survivors, b * cap + k -> row within the scan
  const int32_t* keep_counts;
  int64_t cap;
  int tiles;
  float min_range, max_range;
  double scan_period;
  float* tmp_points;          // b * cap * 3
  uint8_t* cls;               // b * cap
  int32_t* tile_counts;       // b * tiles * 2
  float* returns_local;       // b * cap * 3
  float* misses_local;
  int32_t* num_returns;
  int32_t* num_misses;
  float* current_pose;        // b * 7 floats (t, q wxyz)
};

// Fused front half (dl_frontend.cu).
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
  int64_t cap;           // per-scan capacity of every per-point array below
  int tiles;             // ceil(cap / 256)
  int64_t tcap1, tcap2;  // table capacities (powers of two)
  float first_resolution, second_resolution, min_range, max_range;
  double scan_period;
  uint32_t* table1;              // first filter: slot -> min point index
  uint32_t* first_bits;          // per scan one bitmap of bit_words words: bit i = point i survives the first filter
  unsigned long long* slots2;    // second filter: slot -> [miss | relative voxel key | point index] (dl_frontend.cu)
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
  Rigidd submap;
  const int32_t* error_flag;       // per scan: set by the fused front half when a voxel key could not be packed
  const int32_t* imu_ok;           // optional: 0 = the scan's IMU factor could not be formed (result ok = -2)
  dl_nav_state* states_out;        // optional (fused solve): the estimated state in the LOCAL frame
  dl_scan_result* results;
};

int launch_ingest(dl_context* ctx, const IngestArgs& a, int batch);
int launch_gather_to_tracking(dl_context* ctx, const float* in, int64_t cap, const int32_t* keep,
                              const int32_t* keep_counts, const float* current_pose, float* out, int batch);
int launch_gather_rows(dl_context* ctx, const float* in, int64_t cap_in, int pairs_per_cloud, const int32_t* keep,
                       const int32_t* keep_counts, int64_t cap_out, float* out, int pairs);
int launch_initial_pose(dl_context* ctx, int batch, const float* current_pose, const Rigidd& submap_inverse,
                        double* initial_pose, double* target_translation);
int launch_finalize_results(dl_context* ctx, const ResultArgs& a);

}  // namespace dl
