// Header-only C++ mirror of the reference's matcher / filter classes over the dliom_b200 C-ABI.
//
// Same class names, argument meaning and call shapes as the reference interfaces they replace
// (C/ = src/cartographer/cartographer/, SM/ = C/mapping/internal/3d/scan_matching/):
//   sensor::VoxelFilter, sensor::AdaptiveVoxelFilter        C/sensor/internal/voxel_filter.h:34-79
//   scan_matching::RealTimeCorrelativeScanMatcher3D          SM/real_time_correlative_scan_matcher_3d.h:33-60
//   scan_matching::CeresScanMatcher3D                        SM/ceres_scan_matcher_3d.h:34-61
//   mapping::RangeDataSynchronizer                           C/mapping/internal/3d/range_data_synchronizer.h:30-68
//   mapping::LocalTrajectoryBuilder3D                        C/mapping/internal/3d/local_trajectory_builder_3d.h:81-113
//   io::MapWriter, io::PcdWritingPointsProcessor             cartographer_ros/assets_writer.cc:120-160, C/io/*_points_processor.cc
//   io::ColoringPointsProcessor, io::XRayPointsProcessor     C/io/coloring_points_processor.cc, C/io/xray_points_processor.cc
//   io::ProbabilityGridPointsProcessor, io::DrawProbabilityGrid  C/io/probability_grid_points_processor.cc
//   cartographer_ros::RosMapWritingPointsProcessor           cartographer_ros/ros_map_writing_points_processor.cc, ros_map.cc
//   transform::RollPitchYaw                                  C/transform/rigid_transform.cc:40-46
// Eigen / protobuf types are replaced by the plain structs below (this image has neither); INTEGRATION.md shows
// the three-line adapters for Eigen::Vector3f / transform::Rigid3d / proto options in a real Cartographer tree.
// Errors: the reference CHECK-aborts; this shim throws dliom::Error carrying the C-ABI status and message.
#pragma once
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <deque>
#include <map>
#include <set>
#include <stdexcept>
#include <string>
#include <utility>
#include <memory>
#include <vector>

#include "../../include/dliom_b200.h"

namespace dliom {

struct Error : std::runtime_error {
  int status;
  Error(int s, const std::string& m) : std::runtime_error(m), status(s) {}
};

struct Rigid3d {  // transform::Rigid3d: translation + rotation quaternion (w, x, y, z)
  double t[3] = {0, 0, 0};
  double q[4] = {1, 0, 0, 0};
  void to7(double* p) const { for (int i = 0; i < 3; ++i) p[i] = t[i]; for (int i = 0; i < 4; ++i) p[3 + i] = q[i]; }
  static Rigid3d from7(const double* p) { Rigid3d r; for (int i = 0; i < 3; ++i) r.t[i] = p[i]; for (int i = 0; i < 4; ++i) r.q[i] = p[3 + i]; return r; }
};
using PointCloud = std::vector<std::array<float, 3>>;       // sensor::PointCloud
using TimedPointCloud = std::vector<std::array<float, 4>>;  // sensor::TimedPointCloud

class Context {  // one per host thread (re-entrancy contract of CeresScanMatcher3D::Match)
 public:
  explicit Context(int device = 0) {
    const int st = dl_context_create(device, &ctx_);
    if (st != DL_OK) throw Error(st, dl_last_error(nullptr));
  }
  ~Context() { dl_context_destroy(ctx_); }
  Context(const Context&) = delete;
  Context& operator=(const Context&) = delete;
  dl_context* get() const { return ctx_; }
  void check(int st) const { if (st != DL_OK) throw Error(st, dl_last_error(ctx_)); }
 private:
  dl_context* ctx_ = nullptr;
};

// Device mirror of a mapping::HybridGrid. Fill from `for (auto it : hybrid_grid)` (x, y, z, value), or from
// HybridGrid::ToProto()'s parallel arrays; call Update() with the touched cells after each InsertRangeData.
class DeviceHybridGrid {
 public:
  DeviceHybridGrid(Context* ctx, float resolution) : ctx_(ctx) { ctx->check(dl_grid_create(ctx->get(), resolution, &grid_)); }
  ~DeviceHybridGrid() { dl_grid_destroy(grid_); }
  DeviceHybridGrid(const DeviceHybridGrid&) = delete;
  DeviceHybridGrid& operator=(const DeviceHybridGrid&) = delete;
  void Update(const std::vector<int32_t>& x, const std::vector<int32_t>& y, const std::vector<int32_t>& z,
              const std::vector<uint16_t>& value) {
    ctx_->check(dl_grid_set_cells(grid_, (int64_t)x.size(), x.data(), y.data(), z.data(), value.data()));
    ctx_->check(dl_grid_sync(grid_));
  }
  float resolution() const { return dl_grid_resolution(grid_); }
  const dl_grid* get() const { return grid_; }
 private:
  Context* ctx_;
  dl_grid* grid_ = nullptr;
};

namespace sensor {

class VoxelFilter {  // voxel_filter.h:34-62 (hot-path use: a temporary per call, LTB:393-395, :479-484)
 public:
  VoxelFilter(Context* ctx, float size) : ctx_(ctx), resolution_(size) {}
  PointCloud Filter(const PointCloud& point_cloud) { return FilterRows(point_cloud); }
  TimedPointCloud Filter(const TimedPointCloud& timed_point_cloud) { return FilterRows(timed_point_cloud); }
 private:
  template <typename Cloud>
  Cloud FilterRows(const Cloud& in) {
    std::vector<int64_t> keep(in.size() ? in.size() : 1);
    int64_t n_keep = 0;
    ctx_->check(dl_voxel_filter(ctx_->get(), in.empty() ? nullptr : in[0].data(), (int64_t)in.size(),
                                (int)(sizeof(in[0]) / sizeof(float)), resolution_, keep.data(), &n_keep));
    Cloud out;
    out.reserve(n_keep);
    for (int64_t i = 0; i < n_keep; ++i) out.push_back(in[keep[i]]);
    return out;
  }
  Context* ctx_;
  float resolution_;
};

struct AdaptiveVoxelFilterOptions {  // proto::AdaptiveVoxelFilterOptions
  float max_length, min_num_points, max_range;
};
class AdaptiveVoxelFilter {  // voxel_filter.h:66-79
 public:
  AdaptiveVoxelFilter(Context* ctx, const AdaptiveVoxelFilterOptions& options) : ctx_(ctx), options_(options) {}
  PointCloud Filter(const PointCloud& point_cloud) const {
    std::vector<int64_t> keep(point_cloud.size() ? point_cloud.size() : 1);
    int64_t n_keep = 0;
    const dl_adaptive_voxel_filter_options o{options_.max_length, options_.min_num_points, options_.max_range};
    ctx_->check(dl_adaptive_voxel_filter(ctx_->get(), &o, point_cloud.empty() ? nullptr : point_cloud[0].data(),
                                         (int64_t)point_cloud.size(), 3, keep.data(), &n_keep, nullptr, nullptr));
    PointCloud out;
    out.reserve(n_keep);
    for (int64_t i = 0; i < n_keep; ++i) out.push_back(point_cloud[keep[i]]);
    return out;
  }
 private:
  Context* ctx_;
  AdaptiveVoxelFilterOptions options_;
};

}  // namespace sensor

namespace scan_matching {

struct RealTimeCorrelativeScanMatcherOptions {  // proto::RealTimeCorrelativeScanMatcherOptions
  double linear_search_window, angular_search_window, translation_delta_cost_weight, rotation_delta_cost_weight;
};
class RealTimeCorrelativeScanMatcher3D {  // real_time_correlative_scan_matcher_3d.h:33-60
 public:
  RealTimeCorrelativeScanMatcher3D(Context* ctx, const RealTimeCorrelativeScanMatcherOptions& options)
      : ctx_(ctx), options_(options) {}
  // Returns the best score; *pose_estimate receives the best candidate (CHECK_NOTNULL in the reference).
  float Match(const Rigid3d& initial_pose_estimate, const PointCloud& point_cloud, const DeviceHybridGrid& hybrid_grid,
              Rigid3d* pose_estimate) const {
    if (!pose_estimate) throw Error(DL_ERR_ARG, "pose_estimate is null");
    const dl_rtcsm_options o{options_.linear_search_window, options_.angular_search_window,
                             options_.translation_delta_cost_weight, options_.rotation_delta_cost_weight};
    double init[7], out[7];
    initial_pose_estimate.to7(init);
    float score = 0.f;
    ctx_->check(dl_rtcsm_match(ctx_->get(), &o, init, point_cloud.empty() ? nullptr : point_cloud[0].data(),
                               (int64_t)point_cloud.size(), hybrid_grid.get(), out, &score, nullptr, nullptr));
    *pose_estimate = Rigid3d::from7(out);
    return score;
  }
 private:
  Context* ctx_;
  RealTimeCorrelativeScanMatcherOptions options_;
};

struct CeresScanMatcherOptions3D {  // proto::CeresScanMatcherOptions3D + common::proto::CeresSolverOptions
  std::vector<double> occupied_space_weight;
  double translation_weight = 5., rotation_weight = 4e2;
  bool only_optimize_yaw = false;
  bool use_nonmonotonic_steps = false;
  int max_num_iterations = 12;
  int num_threads = 1;
};
struct SolverSummary {  // the fields of ceres::Solver::Summary the reference reads (LTB:543) + counters
  double initial_cost = 0, final_cost = 0;
  int num_iterations = 0, num_successful_steps = 0, num_unsuccessful_steps = 0, termination = 1;
};
using PointCloudAndHybridGridPointers = std::pair<const PointCloud*, const DeviceHybridGrid*>;

class CeresScanMatcher3D {  // ceres_scan_matcher_3d.h:41-61
 public:
  CeresScanMatcher3D(Context* ctx, const CeresScanMatcherOptions3D& options) : ctx_(ctx), options_(options) {}
  void Match(const std::array<double, 3>& target_translation, const Rigid3d& initial_pose_estimate,
             const std::vector<PointCloudAndHybridGridPointers>& point_clouds_and_hybrid_grids,
             Rigid3d* pose_estimate, SolverSummary* summary) const {
    dl_ceres_options o{};
    o.num_occupied_space_weights = (int32_t)options_.occupied_space_weight.size();
    for (size_t i = 0; i < options_.occupied_space_weight.size() && i < DL_MAX_PAIRS; ++i)
      o.occupied_space_weight[i] = options_.occupied_space_weight[i];
    o.translation_weight = options_.translation_weight;
    o.rotation_weight = options_.rotation_weight;
    o.only_optimize_yaw = options_.only_optimize_yaw;
    o.use_nonmonotonic_steps = options_.use_nonmonotonic_steps;
    o.max_num_iterations = options_.max_num_iterations;
    o.num_threads = options_.num_threads;
    std::vector<const float*> clouds;
    std::vector<int64_t> sizes;
    std::vector<const dl_grid*> grids;
    for (const auto& pg : point_clouds_and_hybrid_grids) {
      clouds.push_back(pg.first->empty() ? nullptr : (*pg.first)[0].data());
      sizes.push_back((int64_t)pg.first->size());
      grids.push_back(pg.second->get());
    }
    double init[7], out[7];
    initial_pose_estimate.to7(init);
    dl_solve_summary s{};
    ctx_->check(dl_ceres_match(ctx_->get(), &o, target_translation.data(), init, (int32_t)clouds.size(), clouds.data(),
                               sizes.data(), grids.data(), out, &s));
    *pose_estimate = Rigid3d::from7(out);
    if (summary)
      *summary = {s.initial_cost, s.final_cost, s.num_iterations, s.num_successful_steps, s.num_unsuccessful_steps,
                  s.termination};
  }
 private:
  Context* ctx_;
  CeresScanMatcherOptions3D options_;
};

struct FastCorrelativeScanMatcherOptions3D {  // proto::FastCorrelativeScanMatcherOptions3D (pose_graph.lua:49-57)
  int branch_and_bound_depth = 8, full_resolution_depth = 3;
  double min_rotational_score = 0.77, min_low_resolution_score = 0.55;
  double linear_xy_search_window = 5., linear_z_search_window = 1., angular_search_window = 0.2617993877991494;
  dl_fcsm_options c() const {
    return {branch_and_bound_depth, full_resolution_depth, min_rotational_score, min_low_resolution_score,
            linear_xy_search_window, linear_z_search_window, angular_search_window};
  }
};

// fast_correlative_scan_matcher_3d.h:59-160, the entry point this fork calls (MatchWith3DofInitial). The constructor takes
// the two grids like the reference's; no precomputation stack is built — the device scores the whole window.
class FastCorrelativeScanMatcher3D {
 public:
  struct Result {
    float score;
    Rigid3d pose_estimate;
    float rotational_score;
    float low_resolution_score;
  };
  FastCorrelativeScanMatcher3D(Context* ctx, const DeviceHybridGrid& hybrid_grid, const DeviceHybridGrid* low_resolution_hybrid_grid,
                               const FastCorrelativeScanMatcherOptions3D& options)
      : ctx_(ctx), hi_(&hybrid_grid), lo_(low_resolution_hybrid_grid), options_(options) {}
  // nullptr when no leaf above min_score passes the low-resolution gate, like the reference.
  std::unique_ptr<Result> MatchWith3DofInitial(const Rigid3d& pose_in_submap_guess, const PointCloud& high_resolution_point_cloud,
                                               const PointCloud& low_resolution_point_cloud, float min_score) const {
    const dl_fcsm_options o = options_.c();
    double guess[7];
    pose_in_submap_guess.to7(guess);
    dl_fcsm_result r{};
    ctx_->check(dl_fcsm_match_3dof(ctx_->get(), &o, guess,
                                   high_resolution_point_cloud.empty() ? nullptr : high_resolution_point_cloud[0].data(),
                                   (int64_t)high_resolution_point_cloud.size(),
                                   low_resolution_point_cloud.empty() ? nullptr : low_resolution_point_cloud[0].data(),
                                   (int64_t)low_resolution_point_cloud.size(), hi_->get(), lo_->get(), min_score, &r, nullptr, 0));
    if (!r.found) return nullptr;
    return std::unique_ptr<Result>(new Result{r.score, Rigid3d::from7(r.pose_estimate), r.rotational_score, r.low_resolution_score});
  }
  // fast_correlative_scan_matcher_3d.h:85-95: the full search (yaw steps x translation window). `submap_histogram` is what the
  // reference's RotationalScanMatcher accumulates from the submap's nodes; `scan_histogram` / `gravity_alignment` (w x y z) come
  // from the node's TrajectoryNode::Data.
  std::unique_ptr<Result> Match(const Rigid3d& global_node_pose, const Rigid3d& global_submap_pose,
                                const std::vector<float>& submap_histogram, const std::vector<float>& scan_histogram,
                                const std::array<double, 4>& gravity_alignment, const PointCloud& high_resolution_point_cloud,
                                const PointCloud& low_resolution_point_cloud, float min_score) const {
    if (submap_histogram.size() != scan_histogram.size() || submap_histogram.empty()) throw Error(DL_ERR_ARG, "histogram sizes differ");
    const dl_fcsm_options o = options_.c();
    double node[7], submap[7];
    global_node_pose.to7(node);
    global_submap_pose.to7(submap);
    dl_fcsm_result r{};
    ctx_->check(dl_fcsm_match(ctx_->get(), &o, submap_histogram.data(), scan_histogram.data(), (int32_t)scan_histogram.size(), node,
                              submap, gravity_alignment.data(),
                              high_resolution_point_cloud.empty() ? nullptr : high_resolution_point_cloud[0].data(),
                              (int64_t)high_resolution_point_cloud.size(),
                              low_resolution_point_cloud.empty() ? nullptr : low_resolution_point_cloud[0].data(),
                              (int64_t)low_resolution_point_cloud.size(), hi_->get(), lo_->get(), min_score, &r));
    if (!r.found) return nullptr;
    return std::unique_ptr<Result>(new Result{r.score, Rigid3d::from7(r.pose_estimate), r.rotational_score, r.low_resolution_score});
  }
 private:
  Context* ctx_;
  const DeviceHybridGrid* hi_;
  const DeviceHybridGrid* lo_;
  FastCorrelativeScanMatcherOptions3D options_;
};

}  // namespace scan_matching

namespace constraints {

struct ConstraintBuilderOptions {  // proto::ConstraintBuilderOptions, the fields ComputeConstraint reads (pose_graph.lua:17-73)
  double min_score = 0.55;
  double loop_closure_translation_weight = 1.1e4, loop_closure_rotation_weight = 1e5;
  scan_matching::FastCorrelativeScanMatcherOptions3D fast_correlative_scan_matcher_options_3d;
  scan_matching::CeresScanMatcherOptions3D ceres_scan_matcher_options_3d;
  ConstraintBuilderOptions() {
    ceres_scan_matcher_options_3d.occupied_space_weight = {5., 30.};
    ceres_scan_matcher_options_3d.translation_weight = 10.;
    ceres_scan_matcher_options_3d.rotation_weight = 1.;
    ceres_scan_matcher_options_3d.max_num_iterations = 10;
  }
  dl_constraint_options c() const {
    dl_constraint_options o{};
    o.min_score = min_score;
    o.loop_closure_translation_weight = loop_closure_translation_weight;
    o.loop_closure_rotation_weight = loop_closure_rotation_weight;
    o.fast_correlative_scan_matcher_3d = fast_correlative_scan_matcher_options_3d.c();
    const auto& m = ceres_scan_matcher_options_3d;
    o.ceres_scan_matcher_3d.num_occupied_space_weights = (int32_t)m.occupied_space_weight.size();
    for (size_t i = 0; i < m.occupied_space_weight.size() && i < DL_MAX_PAIRS; ++i)
      o.ceres_scan_matcher_3d.occupied_space_weight[i] = m.occupied_space_weight[i];
    o.ceres_scan_matcher_3d.translation_weight = m.translation_weight;
    o.ceres_scan_matcher_3d.rotation_weight = m.rotation_weight;
    o.ceres_scan_matcher_3d.only_optimize_yaw = m.only_optimize_yaw;
    o.ceres_scan_matcher_3d.use_nonmonotonic_steps = m.use_nonmonotonic_steps;
    o.ceres_scan_matcher_3d.max_num_iterations = m.max_num_iterations;
    o.ceres_scan_matcher_3d.num_threads = m.num_threads;
    return o;
  }
};

struct Constraint {  // PoseGraphInterface::Constraint (INTER_SUBMAP)
  int submap_index, node_index;
  Rigid3d zbar_ij;
  double translation_weight, rotation_weight;
  float score, low_resolution_score;
};

// The compute half of ConstraintBuilder3D (constraint_builder_3d.cc:202-333): queue (node, submap) searches with
// MaybeAddConstraint, then Compute() runs all of them in one device batch and returns the constraints found
// (the reference schedules one thread-pool task per pair and collects them in RunWhenDoneCallback, :335-358).
class ConstraintBuilder3D {
 public:
  ConstraintBuilder3D(Context* ctx, const ConstraintBuilderOptions& options) : ctx_(ctx), options_(options) {}
  void MaybeAddConstraint(int submap_index, const DeviceHybridGrid* high_resolution_grid, const DeviceHybridGrid* low_resolution_grid,
                          int node_index, const PointCloud& high_resolution_point_cloud,
                          const PointCloud& low_resolution_point_cloud, const Rigid3d& node_pose_in_submap_guess) {
    ids_.push_back({submap_index, node_index});
    hi_grids_.push_back(high_resolution_grid->get());
    lo_grids_.push_back(low_resolution_grid->get());
    for (const auto& p : high_resolution_point_cloud) hi_.insert(hi_.end(), p.begin(), p.end());
    for (const auto& p : low_resolution_point_cloud) lo_.insert(lo_.end(), p.begin(), p.end());
    hi_off_.push_back((int64_t)hi_.size() / 3);
    lo_off_.push_back((int64_t)lo_.size() / 3);
    double g[7];
    node_pose_in_submap_guess.to7(g);
    guesses_.insert(guesses_.end(), g, g + 7);
  }
  int GetNumQueuedSearches() const { return (int)ids_.size(); }
  std::vector<Constraint> Compute() {
    const dl_constraint_options o = options_.c();
    std::vector<dl_constraint> raw(ids_.size());
    ctx_->check(dl_constraint_search_batch(ctx_->get(), &o, (int32_t)ids_.size(), guesses_.data(), hi_.data(), hi_off_.data(),
                                           lo_.data(), lo_off_.data(), hi_grids_.data(), lo_grids_.data(), raw.data()));
    std::vector<Constraint> out;
    for (size_t k = 0; k < raw.size(); ++k)
      if (raw[k].found)
        out.push_back({ids_[k][0], ids_[k][1], Rigid3d::from7(raw[k].pose), raw[k].translation_weight, raw[k].rotation_weight,
                       raw[k].score, raw[k].low_resolution_score});
    ids_.clear(); hi_grids_.clear(); lo_grids_.clear(); hi_.clear(); lo_.clear(); guesses_.clear();
    hi_off_.assign(1, 0); lo_off_.assign(1, 0);
    return out;
  }
 private:
  Context* ctx_;
  ConstraintBuilderOptions options_;
  std::vector<std::array<int, 2>> ids_;
  std::vector<const dl_grid*> hi_grids_, lo_grids_;
  std::vector<float> hi_, lo_;
  std::vector<int64_t> hi_off_{0}, lo_off_{0};
  std::vector<double> guesses_;
};

}  // namespace constraints

namespace sensor {
struct ImuData {  // sensor::ImuData (C/sensor/imu_data.h)
  double time;
  std::array<double, 3> linear_acceleration, angular_velocity;
};
struct TimedPointCloudData {  // sensor::TimedPointCloudData (C/sensor/timed_point_cloud_data.h:27-31)
  double time;  // acquisition time of the LAST point; ranges[i][3] <= 0 is relative to it
  std::array<float, 3> origin;
  TimedPointCloud ranges;
};
struct RangeMeasurement {  // TimedPointCloudOriginData::RangeMeasurement (timed_point_cloud_data.h:33-42), 32 bytes
  std::array<float, 4> point_time;
  uint64_t origin_index;
  uint64_t pad_ = 0;
};
static_assert(sizeof(RangeMeasurement) == 32, "RangeMeasurement layout");
struct TimedPointCloudOriginData {
  double time = 0;
  std::vector<std::array<float, 3>> origins;
  std::vector<RangeMeasurement> ranges;
};
struct RangeData {  // sensor::RangeData
  std::array<float, 3> origin;
  PointCloud returns, misses;
};
}  // namespace sensor

namespace mapping {

// range_data_synchronizer.{h,cc}: the FIRST expected sensor is the prior LiDAR; clouds of the others are queued and the part of
// the oldest queued cloud that overlaps the prior cloud's sweep [start, end] is merged into it, re-stamped relative to the prior
// cloud's end and sorted by time. Host bookkeeping before the path, kept on the host here too.
class RangeDataSynchronizer {
 public:
  explicit RangeDataSynchronizer(const std::vector<std::string>& expected_range_sensor_ids)
      : expected_sensor_ids_(expected_range_sensor_ids.begin(), expected_range_sensor_ids.end()),
        prior_sensor_id_(expected_range_sensor_ids.empty() ? std::string() : expected_range_sensor_ids.front()) {}

  sensor::TimedPointCloudOriginData AddRangeData(const std::string& sensor_id, const sensor::TimedPointCloudData& data, bool deskew) {
    if (!expected_sensor_ids_.count(sensor_id)) throw Error(DL_ERR_ARG, "unexpected range sensor id (CHECK_NE)");
    sensor::TimedPointCloudOriginData result;
    sensor::TimedPointCloudData cloud = data;
    if (deskew) StampRangeData(&cloud, 0.1);
    if (sensor_id != prior_sensor_id_) {
      secondary_.push_back(cloud);
      return result;
    }
    if (secondary_.empty() || cloud.ranges.empty()) return Single(cloud);
    const double end = cloud.time, start = end + cloud.ranges.front()[3];
    while (!secondary_.empty() && secondary_.front().time < start) secondary_.pop_front();  // pop old clouds
    if (secondary_.empty()) return Single(cloud);
    const sensor::TimedPointCloudData& sec = secondary_.front();
    if (sec.ranges.empty() || sec.time + sec.ranges.front()[3] > end) return Single(cloud);  // "secondary lidar may be too fast"
    int i_start = -1, i_end = -1;
    for (int i = 0; i < (int)sec.ranges.size(); ++i) {
      const double t = sec.time + sec.ranges[i][3];
      if (t >= start && t <= end && i_start == -1) i_start = i;
      if (i_start != -1 && t > end) {
        i_end = i - 1;
        break;
      }
    }
    if (i_start == -1) throw Error(DL_ERR_ARG, "no overlap between the two sweeps (CHECK)");
    if (i_end == -1) i_end = (int)sec.ranges.size() - 1;
    result.time = cloud.time;
    result.origins = {cloud.origin, sec.origin};
    result.ranges.reserve(cloud.ranges.size() + (size_t)(i_end - i_start + 1));
    for (size_t i = 0; i < cloud.ranges.size(); ++i) result.ranges.push_back({data.ranges[i], 0});  // the prior cloud keeps its own times
    for (int i = i_start; i <= i_end; ++i) {
      sensor::RangeMeasurement m{sec.ranges[i], 1};
      const double relative_t = sec.ranges[i][3];
      m.point_time[3] = (float)(relative_t + sec.time - end);
      result.ranges.push_back(m);
    }
    std::stable_sort(result.ranges.begin(), result.ranges.end(),
                     [](const sensor::RangeMeasurement& a, const sensor::RangeMeasurement& b) { return a.point_time[3] < b.point_time[3]; });
    return result;
  }

 private:
  static sensor::TimedPointCloudOriginData Single(const sensor::TimedPointCloudData& cloud) {  // ToTimedPointCloudOriginData
    sensor::TimedPointCloudOriginData r;
    r.time = cloud.time;
    r.origins = {cloud.origin};
    r.ranges.reserve(cloud.ranges.size());
    for (const auto& p : cloud.ranges) r.ranges.push_back({p, 0});
    return r;
  }
  static void StampRangeData(sensor::TimedPointCloudData* cloud, double scan_period) {  // :117-131, the "very naive" stamping
    const int n = (int)cloud->ranges.size();
    if (n < 2) return;
    const double duration = scan_period / (n - 1);
    for (int i = 0; i < n; ++i) cloud->ranges[i][3] = (float)(-scan_period + i * duration);
    cloud->ranges.back()[3] = 0.f;
  }
  const std::set<std::string> expected_sensor_ids_;
  const std::string prior_sensor_id_;
  std::deque<sensor::TimedPointCloudData> secondary_;
};

struct LocalTrajectoryBuilderOptions3D {  // proto::LocalTrajectoryBuilderOptions3D, the fields the path reads
  dl_ltb_options c{};
  bool enable_manual_deskew = false;      // eable_mannually_discrew: re-stamp the points uniformly over the scan period
  LocalTrajectoryBuilderOptions3D() {     // trajectory_builder_3d.lua defaults
    dl_frontend_options& f = c.frontend;
    f.min_range = 1.f; f.max_range = 60.f; f.voxel_filter_size = 0.15f;
    f.high_resolution_adaptive_voxel_filter = {2.f, 150.f, 15.f};
    f.low_resolution_adaptive_voxel_filter = {4.f, 200.f, 60.f};
    f.scan_period = 0.1;
    f.use_online_correlative_scan_matching = 0;  // 1: the correlative pre-match seeds the solve (LTB:514-521)
    f.real_time_correlative_scan_matcher = {0.15, 3.14159265358979323846 / 180., 1e-1, 1e-1};
    f.ceres_scan_matcher.num_occupied_space_weights = 2;
    f.ceres_scan_matcher.occupied_space_weight[0] = 1.; f.ceres_scan_matcher.occupied_space_weight[1] = 6.;
    f.ceres_scan_matcher.translation_weight = 5.; f.ceres_scan_matcher.rotation_weight = 4e2;
    f.ceres_scan_matcher.max_num_iterations = 12; f.ceres_scan_matcher.num_threads = 1;
    c.imu_noise = {3.99e-2, 1.56e-2, 6.4e-5, 3.6e-5};
    c.imu_weight = 1.; c.gravity = 9.8;
    c.high_resolution = 0.1f; c.low_resolution = 0.45f; c.num_range_data = 160; c.high_resolution_max_range = 20;
    c.range_data_inserter = {0.55, 0.49, 2, 0};
    c.motion_filter_max_time_seconds = 0.5; c.motion_filter_max_distance_meters = 0.1; c.motion_filter_max_angle_radians = 0.004;
    c.rotational_histogram_size = 120; c.frames_for_static_initialization = 7;
    c.two_stage = 0;  // 1 = the reference's chain: plain match, then the window update (dl_window_optimize_batch)
    c.ceres_pose_noise_t = 1e-2; c.ceres_pose_noise_r = 1e-2; c.prior_pose_noise = 1e-2; c.prior_velocity_noise = 1e4; c.prior_bias_noise = 1e-2;
  }
};

struct TrajectoryNodeData {  // mapping::TrajectoryNode::Data (C/mapping/trajectory_node.h)
  double time;
  std::array<double, 4> gravity_alignment;  // w x y z
  PointCloud high_resolution_point_cloud, low_resolution_point_cloud;
  std::vector<float> rotational_scan_matcher_histogram;
  Rigid3d local_pose;
};

class LocalTrajectoryBuilder3D {  // local_trajectory_builder_3d.h:81-113
 public:
  struct InsertionResult {
    std::shared_ptr<const TrajectoryNodeData> constant_data;
    std::vector<int> insertion_submaps;  // indices; the grids are reachable through submap()
  };
  struct MatchingResult {
    double time;
    Rigid3d local_pose;
    sensor::RangeData range_data_in_local;
    std::unique_ptr<const InsertionResult> insertion_result;  // nullptr if dropped by the motion filter
    float rtcsm_score = 0.f;  // the correlative pre-match's score (kRealTimeCorrelativeScanMatcherScoreMetric); 0 when it is off
  };
  LocalTrajectoryBuilder3D(Context* ctx, const LocalTrajectoryBuilderOptions3D& options,
                           const std::vector<std::string>& expected_range_sensor_ids)
      : ctx_(ctx), options_(options), synchronizer_(expected_range_sensor_ids) {
    ctx->check(dl_ltb_create(ctx->get(), &options.c, &builder_));
  }
  ~LocalTrajectoryBuilder3D() { dl_ltb_destroy(builder_); }
  LocalTrajectoryBuilder3D(const LocalTrajectoryBuilder3D&) = delete;
  LocalTrajectoryBuilder3D& operator=(const LocalTrajectoryBuilder3D&) = delete;

  void AddImuData(const sensor::ImuData& imu_data) {
    ctx_->check(dl_ltb_add_imu_data(builder_, imu_data.time, imu_data.linear_acceleration.data(), imu_data.angular_velocity.data()));
  }
  // Returns nullptr while initialising, when no IMU arrived since the last scan, when the secondary LiDAR's cloud was only
  // queued, or when the scan was dropped (empty filtered clouds), like the reference.
  std::unique_ptr<MatchingResult> AddRangeData(const std::string& sensor_id, const sensor::TimedPointCloudData& unsynchronized_data) {
    const sensor::TimedPointCloudOriginData data = synchronizer_.AddRangeData(sensor_id, unsynchronized_data, options_.enable_manual_deskew);
    if (data.ranges.empty()) return nullptr;
    dl_matching_result r{};
    ctx_->check(dl_ltb_add_synchronized_range_data(builder_, data.time, data.ranges.data(), (int64_t)data.ranges.size(), 8,
                                                   data.origins[0].data(), (int32_t)data.origins.size(), &r));
    return Result(r);
  }
  // One AddRangeData of the batch form below.
  struct RangeDataItem {
    LocalTrajectoryBuilder3D* builder;
    std::string sensor_id;
    const sensor::TimedPointCloudData* data;
  };
  // AddRangeData of several trajectories in one dl_ltb_add_range_data_batch call: result k is what items[k].builder->AddRangeData(
  // items[k].sensor_id, *items[k].data) would have returned, and every builder ends in the same state. Each builder's own
  // RangeDataSynchronizer runs first; builders whose data is only queued return nullptr and take no part. The builders must share
  // one Context and appear once each (Error(DL_ERR_ARG) before any synchroniser runs), and have equal options (Error(DL_ERR_ARG)
  // from dl_ltb_add_range_data_batch, after the synchronisers have run but before any builder is touched).
  static std::vector<std::unique_ptr<MatchingResult>> AddRangeData(const std::vector<RangeDataItem>& items) {
    std::vector<std::unique_ptr<MatchingResult>> out(items.size());
    if (items.empty()) return out;
    Context* ctx = items[0].builder->ctx_;
    for (size_t k = 0; k < items.size(); ++k) {
      if (items[k].builder->ctx_ != ctx) throw Error(DL_ERR_ARG, "the builders of a batch must share one Context");
      for (size_t j = 0; j < k; ++j)
        if (items[j].builder == items[k].builder) throw Error(DL_ERR_ARG, "a builder appears twice in one batch");
    }
    std::vector<sensor::TimedPointCloudOriginData> data;
    std::vector<size_t> which;
    data.reserve(items.size());
    for (size_t k = 0; k < items.size(); ++k) {
      LocalTrajectoryBuilder3D* b = items[k].builder;
      data.push_back(b->synchronizer_.AddRangeData(items[k].sensor_id, *items[k].data, b->options_.enable_manual_deskew));
      if (!data.back().ranges.empty()) which.push_back(k);
    }
    std::vector<dl_ltb_batch_item> batch;
    for (size_t k : which) {
      const sensor::TimedPointCloudOriginData& d = data[k];
      batch.push_back(dl_ltb_batch_item{items[k].builder->builder_, d.time, d.ranges.data(), (int64_t)d.ranges.size(), 8,
                                        (int32_t)d.origins.size(), d.origins[0].data()});
    }
    std::vector<dl_matching_result> r(batch.size());
    ctx->check(dl_ltb_add_range_data_batch((int32_t)batch.size(), batch.data(), r.data()));
    for (size_t j = 0; j < which.size(); ++j) out[which[j]] = items[which[j]].builder->Result(r[j]);
    return out;
  }
  void AddOdometryData(double /*time*/, const Rigid3d& /*pose*/) {}  // the fork never constructs its extrapolator (LTB:574-582)
  // Replaces the NDT initialisation when the caller knows the state (tests, re-localisation).
  void SetInitialState(const dl_nav_state& state) { ctx_->check(dl_ltb_set_initial_state(builder_, &state)); }
  int num_submaps() const { return dl_ltb_num_submaps(builder_); }
  dl_local_trajectory_builder* get() const { return builder_; }

 private:
  // MatchingResult / InsertionResult of a dl_matching_result this builder has just produced (LTB:559-622).
  std::unique_ptr<MatchingResult> Result(const dl_matching_result& r) const {
    if (!r.has_result) return nullptr;
    std::unique_ptr<MatchingResult> out(new MatchingResult);
    out->time = r.time;
    out->local_pose = Rigid3d::from7(r.local_pose);
    out->rtcsm_score = r.scan.rtcsm_score;
    out->range_data_in_local.origin = {r.origin_in_local[0], r.origin_in_local[1], r.origin_in_local[2]};
    out->range_data_in_local.returns = Cloud(0);
    out->range_data_in_local.misses = Cloud(1);
    if (r.inserted) {
      auto node = std::make_shared<TrajectoryNodeData>();
      node->time = r.time;
      node->gravity_alignment = {r.local_pose[3], r.local_pose[4], r.local_pose[5], r.local_pose[6]};
      node->high_resolution_point_cloud = Cloud(2);
      node->low_resolution_point_cloud = Cloud(3);
      node->rotational_scan_matcher_histogram.resize(options_.c.rotational_histogram_size);
      ctx_->check(dl_ltb_get_histogram(builder_, node->rotational_scan_matcher_histogram.data(), options_.c.rotational_histogram_size));
      node->local_pose = out->local_pose;
      std::unique_ptr<InsertionResult> ins(new InsertionResult);
      ins->constant_data = node;
      for (int k = 0; k < r.num_insertion_submaps; ++k) ins->insertion_submaps.push_back(r.insertion_submap_index[k]);
      out->insertion_result = std::move(ins);
    }
    return out;
  }
  PointCloud Cloud(int which) const {
    int64_t n = 0;
    ctx_->check(dl_ltb_get_cloud(builder_, which, nullptr, 0, &n));
    PointCloud c((size_t)n);
    if (n) ctx_->check(dl_ltb_get_cloud(builder_, which, c[0].data(), n, &n));
    return c;
  }
  Context* ctx_;
  LocalTrajectoryBuilderOptions3D options_;
  RangeDataSynchronizer synchronizer_;
  dl_local_trajectory_builder* builder_ = nullptr;
};

// A builder's submap (dl_ltb_get_submap): its device grids stay owned by the builder.
struct Submap3D {
  const dl_grid* high_resolution_grid = nullptr;
  const dl_grid* low_resolution_grid = nullptr;
  Rigid3d local_pose;
  int num_range_data = 0;
  bool finished = false;
};
inline Submap3D GetSubmap(Context* ctx, const LocalTrajectoryBuilder3D& builder, int index) {
  dl_grid *hi = nullptr, *lo = nullptr;
  double pose[7];
  int32_t n = 0, finished = 0;
  ctx->check(dl_ltb_get_submap(builder.get(), index, &hi, &lo, pose, &n, &finished));
  return {hi, lo, Rigid3d::from7(pose), n, finished != 0};
}

// proto::SubmapQuery::Response (Submap3D::ToResponseProto, submap_3d.cc:253-262): textures[0] high, [1] low resolution. The
// cells are raw interleaved (value, alpha) bytes; common::FastGzipString them when filling the proto.
struct SubmapTexture {
  std::vector<uint8_t> cells;
  int width = 0, height = 0;
  double resolution = 0;
  Rigid3d slice_pose;
};
struct SubmapQueryResponse {
  int submap_version = 0;
  std::vector<SubmapTexture> textures;
};
// Every (submap, global submap pose) in one device call (dl_submap_textures).
inline std::vector<SubmapQueryResponse> ToResponseProto(Context* ctx, const std::vector<std::pair<Submap3D, Rigid3d>>& submaps) {
  std::vector<dl_submap_image_query> queries;
  for (const auto& s : submaps)
    for (const dl_grid* g : {s.first.high_resolution_grid, s.first.low_resolution_grid}) {
      dl_submap_image_query q{g, {}};
      s.second.to7(q.pose);
      queries.push_back(q);
    }
  std::vector<dl_submap_texture> textures(queries.size());
  int64_t bytes = 0;
  ctx->check(dl_submap_textures(ctx->get(), (int32_t)queries.size(), queries.data(), textures.data(), 0, nullptr, &bytes));
  std::vector<uint8_t> cells((size_t)bytes);
  ctx->check(dl_submap_textures(ctx->get(), (int32_t)queries.size(), queries.data(), textures.data(), bytes, cells.data(), &bytes));
  std::vector<SubmapQueryResponse> out(submaps.size());
  for (size_t k = 0; k < submaps.size(); ++k) {
    out[k].submap_version = submaps[k].first.num_range_data;
    for (size_t j = 2 * k; j < 2 * k + 2; ++j) {
      const dl_submap_texture& t = textures[j];
      const uint8_t* first = cells.data() + t.offset;
      out[k].textures.push_back({std::vector<uint8_t>(first, first + 2 * (size_t)t.width * t.height), t.width, t.height,
                                 t.resolution, Rigid3d::from7(t.slice_pose)});
    }
  }
  return out;
}
inline SubmapQueryResponse ToResponseProto(Context* ctx, const Submap3D& submap, const Rigid3d& global_submap_pose) {
  return ToResponseProto(ctx, {{submap, global_submap_pose}})[0];
}

// The fork's ProjectToCvMat (submap_3d.cc:381-464): the 8-bit image of cv::Mat(height, width, CV_8UC1), row-major, before its
// cv::threshold / cv::erode. Pass the submap's local pose, as ConstraintBuilder3D::ExtractFeaturesForSubmap does.
struct SubmapProjection {
  int width = 0, height = 0;
  std::vector<uint8_t> pixels;
  double ox = 0, oy = 0, resolution = 0;
};
// Every (grid, pose) in one device call (dl_submap_projections).
inline std::vector<SubmapProjection> ProjectToCvMat(Context* ctx, const std::vector<std::pair<const dl_grid*, Rigid3d>>& grids) {
  std::vector<dl_submap_image_query> queries;
  for (const auto& g : grids) {
    dl_submap_image_query q{g.first, {}};
    g.second.to7(q.pose);
    queries.push_back(q);
  }
  std::vector<dl_submap_projection> records(queries.size());
  int64_t bytes = 0;
  ctx->check(dl_submap_projections(ctx->get(), (int32_t)queries.size(), queries.data(), records.data(), 0, nullptr, &bytes));
  std::vector<uint8_t> pixels((size_t)bytes);
  ctx->check(dl_submap_projections(ctx->get(), (int32_t)queries.size(), queries.data(), records.data(), bytes, pixels.data(), &bytes));
  std::vector<SubmapProjection> out;
  for (const dl_submap_projection& r : records) {
    const uint8_t* first = pixels.data() + r.offset;
    out.push_back({r.width, r.height, std::vector<uint8_t>(first, first + (size_t)r.width * r.height), r.ox, r.oy, r.resolution});
  }
  return out;
}
inline SubmapProjection ProjectToCvMat(Context* ctx, const dl_grid* hybrid_grid, const Rigid3d& transform) {
  return ProjectToCvMat(ctx, {{hybrid_grid, transform}})[0];
}

}  // namespace mapping

namespace optimization {

struct SubmapId {  // mapping::SubmapId
  int trajectory_id, submap_index;
  bool operator<(const SubmapId& o) const { return trajectory_id != o.trajectory_id ? trajectory_id < o.trajectory_id : submap_index < o.submap_index; }
};
struct NodeId {  // mapping::NodeId
  int trajectory_id, node_index;
  bool operator<(const NodeId& o) const { return trajectory_id != o.trajectory_id ? trajectory_id < o.trajectory_id : node_index < o.node_index; }
};
struct SubmapSpec3D { Rigid3d global_pose; };  // optimization_problem_3d.h: SubmapSpec3D
struct NodeSpec3D { Rigid3d global_pose; };    // the part of NodeSpec3D that Solve reads (time, local pose and gravity feed the
                                               // IMU / odometry terms this fork comments out)
struct Constraint {  // PoseGraphInterface::Constraint: node observed from submap
  SubmapId submap_id;
  NodeId node_id;
  Rigid3d zbar_ij;
  double translation_weight, rotation_weight;
};
struct OptimizationProblemOptions {  // proto::OptimizationProblemOptions, the fields Solve reads (pose_graph.lua)
  int max_num_iterations = 50;
  bool fix_z_in_3d = false;
};

// optimization::OptimizationProblem3D (optimization_problem_3d.h) as this fork's Solve runs it, on the device's block-sparse pose
// adjustment (dl_pose_graph_solve_sparse). Submaps and nodes are kept per trajectory in id order; the first submap in that order
// keeps its translation and yaw; every submap and node of a trajectory in frozen_trajectories is constant. With a communicator,
// `constraints` are this rank's share and every rank ends with the same poses.
class OptimizationProblem3D {
 public:
  explicit OptimizationProblem3D(Context* ctx, const OptimizationProblemOptions& options = {}, dl_comm* comm = nullptr)
      : ctx_(ctx), options_(options), comm_(comm) {}
  void AddSubmap(int trajectory_id, const Rigid3d& global_submap_pose) {
    submap_data_[{trajectory_id, next_submap_[trajectory_id]++}] = {global_submap_pose};
  }
  void AddTrajectoryNode(int trajectory_id, const NodeSpec3D& node_data) { node_data_[{trajectory_id, next_node_[trajectory_id]++}] = node_data; }
  void SetMaxNumIterations(int32_t max_num_iterations) { options_.max_num_iterations = max_num_iterations; }

  void Solve(const std::vector<Constraint>& constraints, const std::set<int>& frozen_trajectories = {}) {
    if (node_data_.empty() || submap_data_.empty()) return;  // the reference: nothing to optimize
    std::map<SubmapId, int> submap_index;
    std::map<NodeId, int> node_index;
    std::vector<double> poses;
    std::vector<uint8_t> frozen;
    for (const auto& kv : submap_data_) {
      submap_index[kv.first] = (int)submap_index.size();
      poses.resize(poses.size() + 7);
      kv.second.global_pose.to7(poses.data() + poses.size() - 7);
      frozen.push_back(frozen_trajectories.count(kv.first.trajectory_id) ? 1 : 0);
    }
    for (const auto& kv : node_data_) {
      node_index[kv.first] = (int)node_index.size();
      poses.resize(poses.size() + 7);
      kv.second.global_pose.to7(poses.data() + poses.size() - 7);
      frozen.push_back(frozen_trajectories.count(kv.first.trajectory_id) ? 1 : 0);
    }
    std::vector<dl_spa_constraint> cs;
    cs.reserve(constraints.size());
    for (const Constraint& c : constraints) {
      const auto si = submap_index.find(c.submap_id);
      const auto ni = node_index.find(c.node_id);
      if (si == submap_index.end() || ni == node_index.end()) throw Error(DL_ERR_ARG, "constraint refers to an unknown submap or node");
      dl_spa_constraint d{};
      d.submap = si->second;
      d.node = ni->second;
      c.zbar_ij.to7(d.zbar);
      d.translation_weight = c.translation_weight;
      d.rotation_weight = c.rotation_weight;
      cs.push_back(d);
    }
    const dl_pose_graph_options o{options_.max_num_iterations, options_.fix_z_in_3d ? 1 : 0};
    ctx_->check(dl_pose_graph_solve_sparse(ctx_->get(), comm_, &o, (int32_t)submap_data_.size(), (int32_t)node_data_.size(), poses.data(),
                                           frozen.data(), cs.data(), (int32_t)cs.size(), &summary_, &info_));
    const double* p = poses.data();
    for (auto& kv : submap_data_) { kv.second.global_pose = Rigid3d::from7(p); p += 7; }
    for (auto& kv : node_data_) { kv.second.global_pose = Rigid3d::from7(p); p += 7; }
  }

  const std::map<SubmapId, SubmapSpec3D>& submap_data() const { return submap_data_; }
  const std::map<NodeId, NodeSpec3D>& node_data() const { return node_data_; }
  const dl_solve_summary& summary() const { return summary_; }
  const dl_pose_graph_sparse_info& info() const { return info_; }

 private:
  Context* ctx_;
  OptimizationProblemOptions options_;
  dl_comm* comm_;
  std::map<SubmapId, SubmapSpec3D> submap_data_;
  std::map<NodeId, NodeSpec3D> node_data_;
  std::map<int, int> next_submap_, next_node_;
  dl_solve_summary summary_{};
  dl_pose_graph_sparse_info info_{};
};

}  // namespace optimization

namespace mapping {

struct PoseGraphOptions {  // proto::PoseGraphOptions, the fields the live loop-closure path reads (pose_graph.lua)
  int optimize_every_n_nodes = 90;
  int every_nodes_to_find_constraint = 5;   // constraint_builder.every_nodes_to_find_constraint
  double matcher_translation_weight = 5e2, matcher_rotation_weight = 1.6e3;
  constraints::ConstraintBuilderOptions constraint_builder_options;
  optimization::OptimizationProblemOptions optimization_problem_options;
};
struct SubmapMatch {  // one entry of ConstraintBuilder3D's matched_submaps: an earlier finished submap and Embed3D(Rigid2d)
  optimization::SubmapId submap_id;
  double x, y, theta;
};
struct PoseGraphConstraint {  // PoseGraphInterface::Constraint with its tag
  enum Tag { INTRA_SUBMAP = DL_PG3D_INTRA_SUBMAP, INTER_SUBMAP = DL_PG3D_INTER_SUBMAP };
  optimization::SubmapId submap_id;
  optimization::NodeId node_id;
  Rigid3d zbar_ij;
  double translation_weight, rotation_weight;
  Tag tag;
};

class PoseGraph3D;

// PoseGraphInterface's trimming side (pose_graph_trimmer.h): what a trimmer sees of the graph, and the trimmer itself.
class Trimmable {
 public:
  virtual ~Trimmable() = default;
  virtual std::vector<optimization::SubmapId> GetSubmapIds(int trajectory_id) const = 0;
  virtual std::vector<PoseGraphConstraint> GetConstraints() const = 0;
  virtual bool IsFinished(int trajectory_id) const = 0;
  virtual void MarkSubmapAsTrimmed(const optimization::SubmapId& submap_id) = 0;  // dl_pg3d_trim_submap
};
class PoseGraphTrimmer {
 public:
  virtual ~PoseGraphTrimmer() = default;
  virtual void Trim(Trimmable* pose_graph) = 0;
  virtual bool IsFinished() = 0;
};
// PureLocalizationTrimmer (pose_graph_trimmer.cc:24-45). Its policy lives in the C object (dl_pg3d_add_pure_localization_trimmer):
// PoseGraph3D::AddTrimmer registers it there, and the graph runs it after each optimization, so Trim is never called on it.
class PureLocalizationTrimmer : public PoseGraphTrimmer {
 public:
  PureLocalizationTrimmer(int trajectory_id, int num_submaps_to_keep)
      : trajectory_id_(trajectory_id), num_submaps_to_keep_(num_submaps_to_keep) {}
  void Trim(Trimmable*) override {}
  bool IsFinished() override { return false; }
  int trajectory_id() const { return trajectory_id_; }
  int num_submaps_to_keep() const { return num_submaps_to_keep_; }

 private:
  int trajectory_id_, num_submaps_to_keep_;
};

// mapping::PoseGraph3D (pose_graph_3d.cc) on the live loop-closure path: a thin owner of the C object dl_pose_graph_3d, which
// holds the graph, the device node store and the constraint table, runs the searches and the solve (include/dliom_b200.h).
// AddNode is the call GlobalTrajectoryBuilder makes (global_trajectory_builder.cc:80-82) with the builder whose submaps the
// node was inserted into; `matches` is the host SURF stage's output for a newly finished submap (empty otherwise).
class PoseGraph3D {
 public:
  PoseGraph3D(Context* ctx, const PoseGraphOptions& options) : ctx_(ctx) {
    dl_pose_graph_3d_options o{};
    o.optimize_every_n_nodes = options.optimize_every_n_nodes;
    o.every_nodes_to_find_constraint = options.every_nodes_to_find_constraint;
    o.matcher_translation_weight = options.matcher_translation_weight;
    o.matcher_rotation_weight = options.matcher_rotation_weight;
    o.constraint_builder = options.constraint_builder_options.c();
    o.optimization_problem = {options.optimization_problem_options.max_num_iterations,
                              options.optimization_problem_options.fix_z_in_3d ? 1 : 0};
    ctx->check(dl_pose_graph_3d_create(ctx->get(), &o, &graph_));
  }
  ~PoseGraph3D() { dl_pose_graph_3d_destroy(graph_); }
  PoseGraph3D(const PoseGraph3D&) = delete;
  PoseGraph3D& operator=(const PoseGraph3D&) = delete;

  // Pure localization. After every call that may trim (AddNode, RunFinalOptimization, FinishTrajectory), the grids of the
  // submaps the graph trimmed are released on the LocalTrajectoryBuilder3D that AddNode got them from, if that builder has
  // finished them (dl_ltb_release_submap); then, if the call optimized, the host trimmers run in the order added, after the
  // ones the C object runs itself, and finished host trimmers are dropped (HandleWorkQueue, :492-501).
  void AddTrimmer(std::unique_ptr<PoseGraphTrimmer> trimmer) {
    if (const auto* p = dynamic_cast<const PureLocalizationTrimmer*>(trimmer.get())) {
      ctx_->check(dl_pg3d_add_pure_localization_trimmer(graph_, p->trajectory_id(), p->num_submaps_to_keep()));
      return;
    }
    trimmers_.push_back(std::move(trimmer));
  }
  void FinishTrajectory(int trajectory_id) {  // every submap finished, then the final optimization and the trimmers
    const int st = dl_pg3d_finish_trajectory(graph_, trajectory_id);
    AfterCall(st, st == DL_OK);
  }
  bool IsTrajectoryFinished(int trajectory_id) const {
    int32_t finished = 0;
    ctx_->check(dl_pg3d_is_trajectory_finished(graph_, trajectory_id, &finished));
    return finished != 0;
  }
  void SetInitialTrajectoryPose(int from_trajectory_id, int to_trajectory_id, const Rigid3d& pose, double time) {
    double p[7];
    pose.to7(p);
    ctx_->check(dl_pg3d_set_initial_trajectory_pose(graph_, from_trajectory_id, to_trajectory_id, p, time));
  }
  // The node and submap poses of one trajectory keyed by their ids (MapById's view: trimmed ids are absent).
  std::map<optimization::NodeId, Rigid3d> GetTrajectoryNodePosesById(int trajectory_id) const {
    std::map<optimization::NodeId, Rigid3d> out;
    const std::vector<Rigid3d> poses = Poses(trajectory_id, DL_PG3D_NODE_POSES);
    const std::vector<int32_t> ids = Ids(trajectory_id, DL_PG3D_NODE_POSES);
    for (size_t i = 0; i < ids.size() && i < poses.size(); ++i) out[{trajectory_id, ids[i]}] = poses[i];
    return out;
  }
  std::map<optimization::SubmapId, Rigid3d> GetAllSubmapPosesById(int trajectory_id) const {
    std::map<optimization::SubmapId, Rigid3d> out;
    const std::vector<Rigid3d> poses = Poses(trajectory_id, DL_PG3D_SUBMAP_POSES);
    const std::vector<int32_t> ids = Ids(trajectory_id, DL_PG3D_SUBMAP_POSES);
    for (size_t i = 0; i < ids.size() && i < poses.size(); ++i) out[{trajectory_id, ids[i]}] = poses[i];
    return out;
  }

  // -> the node's id; the submaps' grids, local poses and finished flags come from the builder (dl_ltb_get_submap).
  optimization::NodeId AddNode(int trajectory_id, const LocalTrajectoryBuilder3D& builder,
                               const LocalTrajectoryBuilder3D::InsertionResult& insertion_result,
                               const std::vector<SubmapMatch>& matches = {}, dl_pg3d_add_node_info* info = nullptr) {
    const TrajectoryNodeData& data = *insertion_result.constant_data;
    dl_pg3d_node node{};
    node.trajectory_id = trajectory_id;
    node.num_insertion_submaps = (int32_t)insertion_result.insertion_submaps.size();
    if (node.num_insertion_submaps < 1 || node.num_insertion_submaps > 2) throw Error(DL_ERR_ARG, "one or two insertion submaps");
    node.time = data.time;
    data.local_pose.to7(node.local_pose);
    node.high_resolution_points = data.high_resolution_point_cloud.empty() ? nullptr : data.high_resolution_point_cloud[0].data();
    node.num_high_resolution = (int64_t)data.high_resolution_point_cloud.size();
    node.low_resolution_points = data.low_resolution_point_cloud.empty() ? nullptr : data.low_resolution_point_cloud[0].data();
    node.num_low_resolution = (int64_t)data.low_resolution_point_cloud.size();
    for (int i = 0; i < node.num_insertion_submaps; ++i) {
      dl_pg3d_insertion_submap& s = node.insertion_submaps[i];
      dl_grid *hi = nullptr, *lo = nullptr;
      int32_t num_range_data = 0;
      s.submap_index = insertion_result.insertion_submaps[i];
      ctx_->check(dl_ltb_get_submap(builder.get(), s.submap_index, &hi, &lo, s.local_pose, &num_range_data, &s.finished));
      s.high_resolution_grid = hi;
      s.low_resolution_grid = lo;
    }
    std::vector<dl_pg3d_submap_match> m;
    for (const SubmapMatch& sm : matches) m.push_back({sm.submap_id.trajectory_id, sm.submap_id.submap_index, sm.x, sm.y, sm.theta});
    dl_pg3d_add_node_info local{};
    const int st = dl_pose_graph_3d_add_node(graph_, &node, (int32_t)m.size(), m.data(), &local);
    if (st == DL_OK)
      for (int i = 0; i < node.num_insertion_submaps; ++i) feeders_[{trajectory_id, node.insertion_submaps[i].submap_index}] = &builder;
    if (st == DL_OK && range_data_cache_) {  // the builder's range_data_in_local.returns of this node
      int64_t n = 0;
      ctx_->check(dl_ltb_get_cloud(builder.get(), 0, nullptr, 0, &n));
      PointCloud returns((size_t)n);
      if (n) ctx_->check(dl_ltb_get_cloud(builder.get(), 0, returns[0].data(), n, &n));
      ctx_->check(dl_range_data_map_set_node(graph_, trajectory_id, local.node_index, n ? returns[0].data() : nullptr, n));
    }
    AfterCall(st, st == DL_OK && local.optimized);
    if (info) *info = local;
    return {trajectory_id, local.node_index};
  }
  void FreezeTrajectory(int trajectory_id) { ctx_->check(dl_pose_graph_3d_freeze_trajectory(graph_, trajectory_id)); }
  // MapBuilderBridge::EnableFullCloudCache (map_builder_bridge.cc:591-607), the cache behind --save_range_data: after it, AddNode
  // also keeps the node's range_data_in_local.returns in the graph's node store (dl_range_data_map_set_node).
  void EnableRangeDataCache() { range_data_cache_ = true; }
  // pb_range_data_to_ros_cloud's map (dl_range_data_map): every node with cached range data, in (trajectory, node index)
  // order, its returns at the node's optimized pose; `nodes` gives each node's rows of `points` and the pose used.
  struct RangeDataMapResult {
    std::vector<dl_range_data_map_node> nodes;
    PointCloud points;
  };
  RangeDataMapResult RangeDataMap() const { return RangeDataMap(nullptr); }
  RangeDataMapResult RangeDataMap(const std::vector<int32_t>& trajectory_ids) const { return RangeDataMap(&trajectory_ids); }
  dl_solve_summary RunFinalOptimization() {
    dl_solve_summary s{};
    const int st = dl_pose_graph_3d_run_final_optimization(graph_, &s);
    AfterCall(st, st == DL_OK);
    return s;
  }
  std::vector<Rigid3d> GetTrajectoryNodePoses(int trajectory_id) const { return Poses(trajectory_id, DL_PG3D_NODE_POSES); }
  // GetAllSubmapPoses for one trajectory: the optimized pose, or extrapolated with the local-to-global transform.
  std::vector<Rigid3d> GetAllSubmapPoses(int trajectory_id) const { return Poses(trajectory_id, DL_PG3D_SUBMAP_POSES); }
  Rigid3d GetLocalToGlobalTransform(int trajectory_id) const {
    double p[7];
    ctx_->check(dl_pose_graph_3d_local_to_global(graph_, trajectory_id, p));
    return Rigid3d::from7(p);
  }
  std::vector<PoseGraphConstraint> constraints() const {
    int32_t n = 0;
    ctx_->check(dl_pose_graph_3d_constraints(graph_, 0, nullptr, &n));
    std::vector<dl_pg3d_constraint> raw((size_t)n);
    if (n) ctx_->check(dl_pose_graph_3d_constraints(graph_, n, raw.data(), &n));
    std::vector<PoseGraphConstraint> out;
    for (const dl_pg3d_constraint& c : raw)
      out.push_back({{c.submap_trajectory_id, c.submap_index}, {c.node_trajectory_id, c.node_index}, Rigid3d::from7(c.zbar),
                     c.translation_weight, c.rotation_weight, (PoseGraphConstraint::Tag)c.tag});
    return out;
  }
  dl_pose_graph_3d* get() const { return graph_; }

 private:
  // TrimmingHandle (pose_graph_3d.cc:955-1058) over the C calls.
  class TrimmingHandle : public Trimmable {
   public:
    explicit TrimmingHandle(PoseGraph3D* parent) : parent_(parent) {}
    std::vector<optimization::SubmapId> GetSubmapIds(int trajectory_id) const override {
      std::vector<optimization::SubmapId> out;
      for (const int32_t i : parent_->Ids(trajectory_id, DL_PG3D_SUBMAP_POSES)) out.push_back({trajectory_id, i});
      return out;
    }
    std::vector<PoseGraphConstraint> GetConstraints() const override { return parent_->constraints(); }
    bool IsFinished(int trajectory_id) const override { return parent_->IsTrajectoryFinished(trajectory_id); }
    void MarkSubmapAsTrimmed(const optimization::SubmapId& submap_id) override {
      const int st = dl_pg3d_trim_submap(parent_->graph_, submap_id.trajectory_id, submap_id.submap_index);
      parent_->AfterCall(st, false);
    }

   private:
    PoseGraph3D* parent_;
  };
  // The trimmed submaps' grids back to their builders (also after a failed call: it reports what it trimmed before failing),
  // then the call's status, then the host trimmers if it optimized.
  void AfterCall(int status, bool optimized) {
    int32_t n = 0;
    ctx_->check(dl_pg3d_last_trimmed(graph_, 0, nullptr, &n));
    std::vector<dl_pg3d_submap_id> trimmed((size_t)n);
    if (n) ctx_->check(dl_pg3d_last_trimmed(graph_, n, trimmed.data(), &n));
    for (const dl_pg3d_submap_id& id : trimmed) {
      const auto it = feeders_.find({id.trajectory_id, id.submap_index});
      if (it == feeders_.end()) continue;
      const LocalTrajectoryBuilder3D* builder = it->second;
      feeders_.erase(it);
      int32_t finished = 0;
      ctx_->check(dl_ltb_get_submap(builder->get(), id.submap_index, nullptr, nullptr, nullptr, nullptr, &finished));
      if (finished) ctx_->check(dl_ltb_release_submap(builder->get(), id.submap_index));
    }
    ctx_->check(status);
    if (!optimized || trimmers_.empty()) return;
    TrimmingHandle handle(this);
    for (auto& trimmer : trimmers_) trimmer->Trim(&handle);
    trimmers_.erase(std::remove_if(trimmers_.begin(), trimmers_.end(),
                                   [](std::unique_ptr<PoseGraphTrimmer>& t) { return t->IsFinished(); }),
                    trimmers_.end());
  }
  std::vector<int32_t> Ids(int trajectory_id, int which) const {
    int32_t n = 0;
    ctx_->check(dl_pg3d_ids(graph_, trajectory_id, which, 0, nullptr, &n));
    std::vector<int32_t> ids((size_t)n);
    if (n) ctx_->check(dl_pg3d_ids(graph_, trajectory_id, which, n, ids.data(), &n));
    return ids;
  }
  RangeDataMapResult RangeDataMap(const std::vector<int32_t>* ids) const {
    const int32_t num_ids = ids ? (int32_t)ids->size() : 0;
    const int32_t* id_ptr = ids ? ids->data() : nullptr;
    int32_t num_nodes = 0;
    int64_t num_points = 0;
    ctx_->check(dl_range_data_map(graph_, num_ids, id_ptr, 0, nullptr, &num_nodes, 0, nullptr, &num_points));
    RangeDataMapResult out;
    out.nodes.resize((size_t)num_nodes + 1);  // never empty: data() is then non-null and the call fills, not sizes
    out.points.resize((size_t)num_points + 1);
    ctx_->check(dl_range_data_map(graph_, num_ids, id_ptr, num_nodes, out.nodes.data(), &num_nodes, num_points,
                                  out.points[0].data(), &num_points));
    out.nodes.resize((size_t)num_nodes);
    out.points.resize((size_t)num_points);
    return out;
  }
  std::vector<Rigid3d> Poses(int trajectory_id, int which) const {
    int32_t n = 0;
    ctx_->check(dl_pose_graph_3d_poses(graph_, trajectory_id, which, 0, nullptr, &n));
    std::vector<double> p(7 * (size_t)n);
    if (n) ctx_->check(dl_pose_graph_3d_poses(graph_, trajectory_id, which, n, p.data(), &n));
    std::vector<Rigid3d> out;
    for (int32_t i = 0; i < n; ++i) out.push_back(Rigid3d::from7(&p[7 * (size_t)i]));
    return out;
  }
  Context* ctx_;
  dl_pose_graph_3d* graph_ = nullptr;
  std::map<optimization::SubmapId, const LocalTrajectoryBuilder3D*> feeders_;  // where AddNode got each submap's grids
  std::vector<std::unique_ptr<PoseGraphTrimmer>> trimmers_;                     // host trimmers, in the order added
  bool range_data_cache_ = false;                                               // EnableRangeDataCache
};

}  // namespace mapping

namespace transform {

// RollPitchYaw (transform/rigid_transform.cc:40-46): AngleAxisd(yaw, Z) * AngleAxisd(pitch, Y) * AngleAxisd(roll, X), each angle
// axis as (cos(a / 2), sin(a / 2) * axis), multiplied in Eigen's quaternion-product order. Returns (w, x, y, z).
inline std::array<double, 4> RollPitchYaw(double roll, double pitch, double yaw) {
  auto product = [](const std::array<double, 4>& a, const std::array<double, 4>& b) -> std::array<double, 4> {
    return {a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3], a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
            a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3], a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1]};
  };
  const std::array<double, 4> r = {std::cos(0.5 * roll), std::sin(0.5 * roll), 0.0, 0.0};
  const std::array<double, 4> p = {std::cos(0.5 * pitch), 0.0, std::sin(0.5 * pitch), 0.0};
  const std::array<double, 4> y = {std::cos(0.5 * yaw), 0.0, 0.0, std::sin(0.5 * yaw)};
  return product(product(y, p), r);
}

}  // namespace transform

namespace io {

// The assets writer's processors (cartographer_ros/assets_writer.cc with the fork's assets_writer_tongji.lua), on the device in
// the fixed order HandleMessage -> MinMaxRangeFiteringPointsProcessor -> OutlierRemovingPointsProcessor (dl_map_writer_*).
struct MinMaxRangeFilteringOptions {  // min_max_range_filter (io/min_max_range_filtering_points_processor.cc:26-33)
  double min_range = 0.0, max_range = 0.0;
};
struct OutlierRemovingOptions {  // voxel_filter_and_remove_moving_objects (io/outlier_removing_points_processor.cc:26-32)
  double voxel_size = 0.0;
};
struct MapWriterOptions {
  bool min_max_range_filter = false;
  MinMaxRangeFilteringOptions range;
  bool remove_moving_objects = false;
  OutlierRemovingOptions outlier;
};
struct Message {  // one sensor message = one PointsBatch: x y z t rows (t in seconds, relative to stamp), sensor frame
  int64_t stamp = 0;  // universal ticks (common::ToUniversal)
  int trajectory_id = 0;
  std::string frame_id;  // PointsBatch::frame_id: what color_points stages match, exactly
  Rigid3d sensor_to_tracking;
  TimedPointCloud rows;
};
enum class FlushResult { kRestartStream, kFinished };  // PointsProcessor::FlushResult

class MapWriter {
 public:
  MapWriter(Context* ctx, const MapWriterOptions& options) : ctx_(ctx) {
    dl_map_writer_options o{};
    o.range_filter = options.min_max_range_filter ? 1 : 0;
    o.min_range = options.range.min_range;
    o.max_range = options.range.max_range;
    o.outlier_voxel_size = options.remove_moving_objects ? options.outlier.voxel_size : 0.0;
    ctx->check(dl_map_writer_create(ctx->get(), &o, &writer_));
  }
  ~MapWriter() { dl_map_writer_destroy(writer_); }
  MapWriter(const MapWriter&) = delete;
  MapWriter& operator=(const MapWriter&) = delete;
  // TransformInterpolationBuffer(proto::Trajectory): node timestamps (universal ticks, non-decreasing) and global poses
  void AddTrajectory(int trajectory_id, const std::vector<int64_t>& times, const std::vector<Rigid3d>& poses) {
    if (times.size() != poses.size()) throw Error(DL_ERR_ARG, "AddTrajectory: times and poses differ in length");
    std::vector<double> p(7 * poses.size());
    for (size_t i = 0; i < poses.size(); ++i) poses[i].to7(&p[7 * i]);
    ctx_->check(dl_map_writer_add_trajectory(writer_, trajectory_id, (int32_t)times.size(), times.data(), p.data()));
  }
  // Streams messages (one call for many); returns the points of the final pass, in order, and nothing in earlier passes.
  PointCloud Process(const std::vector<Message>& messages) {
    std::vector<dl_map_message> m(messages.size());
    TimedPointCloud rows;
    for (size_t k = 0; k < messages.size(); ++k) {
      m[k].stamp = messages[k].stamp;
      m[k].first_row = (int64_t)rows.size();
      m[k].num_rows = (int64_t)messages[k].rows.size();
      m[k].trajectory_id = messages[k].trajectory_id;
      m[k].frame_id = FrameId(messages[k].frame_id);
      messages[k].sensor_to_tracking.to7(m[k].sensor_to_tracking);
      rows.insert(rows.end(), messages[k].rows.begin(), messages[k].rows.end());
    }
    PointCloud out(rows.size());
    int64_t n = 0;
    ctx_->check(dl_map_writer_process(writer_, (int32_t)m.size(), m.data(), rows.empty() ? nullptr : rows[0].data(),
                                      (int64_t)rows.size(), out.empty() ? nullptr : out[0].data(), &n, nullptr, &last_info_));
    out.resize((size_t)n);
    return out;
  }
  FlushResult Flush() {
    int32_t restart = 0;
    ctx_->check(dl_map_writer_flush(writer_, &restart));
    return restart ? FlushResult::kRestartStream : FlushResult::kFinished;
  }
  const dl_map_writer_info& last_info() const { return last_info_; }
  // Stages after the final multi-pass stage, added before the first Process in pipeline order (what ColoringPointsProcessor
  // and XRayPointsProcessor call).
  void AddColor(const std::string& frame_id, const std::array<uint8_t, 3>& rgb) {
    dl_map_writer_color c{};
    c.frame_id = FrameId(frame_id);
    for (int i = 0; i < 3; ++i) c.rgb[i] = rgb[i];
    ctx_->check(dl_map_writer_add_color(writer_, &c));
  }
  int AddXRay(double voxel_size, const Rigid3d& transform) {
    dl_map_writer_xray x{};
    x.voxel_size = voxel_size;
    transform.to7(x.transform);
    int32_t stage = 0;
    ctx_->check(dl_map_writer_add_xray(writer_, &x, &stage));
    return stage;
  }
  // A probability-grid stage (what ProbabilityGridPointsProcessor and RosMapWritingPointsProcessor call).
  int AddProbabilityGrid(double resolution, double hit_probability, double miss_probability, bool insert_free_space = true) {
    dl_map_writer_grid_options o{};
    o.resolution = resolution;
    o.hit_probability = hit_probability;
    o.miss_probability = miss_probability;
    o.insert_free_space = insert_free_space ? 1 : 0;
    int32_t stage = 0;
    ctx_->check(dl_map_writer_add_probability_grid(writer_, &o, &stage));
    return stage;
  }
  // After the final Flush: the grid's limits and cropped box; the cropped cells and grey pixels, row-major.
  dl_map_writer_grid_info ProbabilityGrid(int stage, std::vector<uint16_t>* cells, std::vector<uint8_t>* pixels) const {
    dl_map_writer_grid_info info{};
    ctx_->check(dl_map_writer_probability_grid(writer_, stage, &info, 0, nullptr, nullptr));
    const size_t n = (size_t)info.width * (size_t)info.height;
    if (cells) cells->assign(n, 0);
    if (pixels) pixels->assign(n, 0);
    ctx_->check(dl_map_writer_probability_grid(writer_, stage, &info, (int64_t)n, cells ? cells->data() : nullptr,
                                               pixels ? pixels->data() : nullptr));
    return info;
  }
  // After the final Flush: Cairo ARGB32 words, row-major; 0 x 0 for an empty bounding box.
  std::vector<uint32_t> XRayImage(int stage, int* width, int* height) const {
    int32_t w = 0, h = 0;
    ctx_->check(dl_map_writer_xray_image(writer_, stage, 0, nullptr, &w, &h));
    std::vector<uint32_t> argb((size_t)w * (size_t)h);
    if (!argb.empty()) ctx_->check(dl_map_writer_xray_image(writer_, stage, (int64_t)argb.size(), argb.data(), &w, &h));
    *width = w;
    *height = h;
    return argb;
  }

 private:
  // PointsBatch::frame_id strings as the C-ABI's integers: equal strings, equal integers
  int32_t FrameId(const std::string& frame_id) {
    const auto it = frame_ids_.emplace(frame_id, (int32_t)frame_ids_.size()).first;
    return it->second;
  }
  Context* ctx_;
  dl_map_writer* writer_ = nullptr;
  dl_map_writer_info last_info_{};
  std::map<std::string, int32_t> frame_ids_;
};

// io::ColoringPointsProcessor (io/coloring_points_processor.cc): batches of `frame_id` get `color` (the Lua values after
// static_cast<uint8>) for the X-ray stages added after it.
class ColoringPointsProcessor {
 public:
  ColoringPointsProcessor(MapWriter* writer, const std::array<uint8_t, 3>& color, const std::string& frame_id) {
    writer->AddColor(frame_id, color);
  }
};

// PNG bytes of an X-ray image: 8-bit RGB (colour type 2: every pixel is opaque), filter 0 on every row, one IDAT chunk holding a
// zlib stream of stored deflate blocks, CRC-32 and Adler-32 computed here. The same bytes as dliom.png_bytes.
inline std::vector<uint8_t> PngBytes(const std::vector<uint32_t>& argb, int width, int height) {
  auto be32 = [](std::vector<uint8_t>* out, uint32_t v) {
    for (int s = 24; s >= 0; s -= 8) out->push_back((uint8_t)(v >> s));
  };
  std::vector<uint8_t> raw;
  raw.reserve((size_t)height * (1 + 3 * (size_t)width));
  for (int y = 0; y < height; ++y) {
    raw.push_back(0);
    for (int x = 0; x < width; ++x) {
      const uint32_t c = argb[(size_t)y * width + x];
      raw.push_back((uint8_t)(c >> 16));
      raw.push_back((uint8_t)(c >> 8));
      raw.push_back((uint8_t)c);
    }
  }
  std::vector<uint8_t> z = {0x78, 0x01};
  for (size_t k = 0; k < raw.size(); k += 65535) {
    const size_t n = std::min<size_t>(65535, raw.size() - k);
    z.push_back(k + n >= raw.size() ? 1 : 0);
    z.push_back((uint8_t)n);
    z.push_back((uint8_t)(n >> 8));
    z.push_back((uint8_t)~n);
    z.push_back((uint8_t)(~n >> 8));
    z.insert(z.end(), raw.begin() + k, raw.begin() + k + n);
  }
  uint32_t a = 1, b = 0;  // Adler-32
  for (uint8_t v : raw) {
    a = (a + v) % 65521;
    b = (b + a) % 65521;
  }
  be32(&z, b << 16 | a);
  uint32_t table[256];  // CRC-32, reflected polynomial 0xEDB88320
  for (uint32_t n = 0; n < 256; ++n) {
    uint32_t c = n;
    for (int k = 0; k < 8; ++k) c = (c & 1) ? 0xEDB88320u ^ (c >> 1) : c >> 1;
    table[n] = c;
  }
  std::vector<uint8_t> png = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};
  auto chunk = [&](const char* kind, const std::vector<uint8_t>& data) {
    be32(&png, (uint32_t)data.size());
    const size_t start = png.size();
    png.insert(png.end(), kind, kind + 4);
    png.insert(png.end(), data.begin(), data.end());
    uint32_t c = 0xFFFFFFFFu;
    for (size_t i = start; i < png.size(); ++i) c = table[(c ^ png[i]) & 0xFF] ^ (c >> 8);
    be32(&png, c ^ 0xFFFFFFFFu);
  };
  std::vector<uint8_t> ihdr;
  be32(&ihdr, (uint32_t)width);
  be32(&ihdr, (uint32_t)height);
  ihdr.insert(ihdr.end(), {8, 2, 0, 0, 0});
  chunk("IHDR", ihdr);
  chunk("IDAT", z);
  chunk("IEND", {});
  return png;
}

// io::XRayPointsProcessor (io/xray_points_processor.cc) with draw_trajectories = false and without separate_floors: the final
// pass's points seen through `transform` at `voxel_size`; Flush, after the writer's final Flush, writes <output_filename>.png
// (nothing for an empty bounding box, where the reference only warns).
class XRayPointsProcessor {
 public:
  XRayPointsProcessor(MapWriter* writer, double voxel_size, const Rigid3d& transform, const std::string& output_filename)
      : writer_(writer), stage_(writer->AddXRay(voxel_size, transform)), output_filename_(output_filename) {}
  void Flush() const {
    int width = 0, height = 0;
    const std::vector<uint32_t> argb = writer_->XRayImage(stage_, &width, &height);
    if (argb.empty()) return;
    const std::vector<uint8_t> png = PngBytes(argb, width, height);
    const std::string path = output_filename_ + ".png";
    std::FILE* f = std::fopen(path.c_str(), "wb");
    if (!f) throw Error(DL_ERR_ARG, "cannot open " + path);
    const bool ok = std::fwrite(png.data(), 1, png.size(), f) == png.size();
    if (std::fclose(f) != 0 || !ok) throw Error(DL_ERR_ARG, "PNG write failed: " + path);
  }
  int stage() const { return stage_; }

 private:
  MapWriter* writer_;
  int stage_;
  std::string output_filename_;
};

inline void WriteFile(const std::string& path, const std::string& bytes) {
  std::FILE* f = std::fopen(path.c_str(), "wb");
  if (!f) throw Error(DL_ERR_ARG, "cannot open " + path);
  const bool ok = std::fwrite(bytes.data(), 1, bytes.size(), f) == bytes.size();
  if (std::fclose(f) != 0 || !ok) throw Error(DL_ERR_ARG, "write failed: " + path);
}

// io::Image of DrawProbabilityGrid: grey values (r = g = b), row-major.
struct GreyImage {
  int width = 0, height = 0;
  std::vector<uint8_t> pixels;
  // Image::Rotate90DegreesClockwise (io/image.cc:67-76)
  void Rotate90DegreesClockwise() {
    std::vector<uint8_t> out;
    out.reserve(pixels.size());
    for (int x = 0; x < width; ++x)
      for (int y = height - 1; y >= 0; --y) out.push_back(pixels[(size_t)y * width + x]);
    pixels.swap(out);
    std::swap(width, height);
  }
};

// io::DrawProbabilityGrid (io/probability_grid_points_processor.cc:127-148) of a grid stage after the writer's final Flush:
// the cropped box (1 x 1 at offset 0 for an empty grid), 128 for unknown cells; *info receives the limits and the offset.
inline GreyImage DrawProbabilityGrid(const MapWriter& writer, int stage, dl_map_writer_grid_info* info) {
  GreyImage image;
  *info = writer.ProbabilityGrid(stage, nullptr, &image.pixels);
  image.width = info->width;
  image.height = info->height;
  return image;
}

// io::ProbabilityGridPointsProcessor with draw_trajectories = false: Flush, after the writer's final Flush, writes
// <filename>.png (grey in 8-bit RGB, PngBytes).
class ProbabilityGridPointsProcessor {
 public:
  ProbabilityGridPointsProcessor(MapWriter* writer, double resolution, double hit_probability, double miss_probability,
                                 bool insert_free_space, const std::string& filename)
      : writer_(writer), stage_(writer->AddProbabilityGrid(resolution, hit_probability, miss_probability, insert_free_space)),
        filename_(filename) {}
  void Flush() const {
    dl_map_writer_grid_info info;
    const GreyImage image = DrawProbabilityGrid(*writer_, stage_, &info);
    std::vector<uint32_t> argb(image.pixels.size());
    for (size_t i = 0; i < argb.size(); ++i) argb[i] = 0xFF000000u | image.pixels[i] * 0x010101u;
    const std::vector<uint8_t> png = PngBytes(argb, image.width, image.height);
    WriteFile(filename_ + ".png", std::string(png.begin(), png.end()));
  }
  int stage() const { return stage_; }

 private:
  MapWriter* writer_;
  int stage_;
  std::string filename_;
};

// io::PcdWritingPointsProcessor (io/pcd_writing_points_processor.cc:35-130): binary PCD v0.7, x y z floats, no colour. The header
// (WIDTH and POINTS zero-padded to 15 digits) is written before the first points and rewritten with the count at Flush.
class PcdWritingPointsProcessor {
 public:
  explicit PcdWritingPointsProcessor(const std::string& filename) : file_(std::fopen(filename.c_str(), "wb")) {
    if (!file_) throw Error(DL_ERR_ARG, "cannot open " + filename);
  }
  ~PcdWritingPointsProcessor() { if (file_) std::fclose(file_); }
  PcdWritingPointsProcessor(const PcdWritingPointsProcessor&) = delete;
  PcdWritingPointsProcessor& operator=(const PcdWritingPointsProcessor&) = delete;
  void Process(const PointCloud& points) {
    if (points.empty()) return;
    if (num_points_ == 0) WriteHeader(0);
    for (const auto& p : points)
      if (std::fwrite(p.data(), 4, 3, file_) != 3) throw Error(DL_ERR_ARG, "PCD write failed");
    num_points_ += (int64_t)points.size();
  }
  void Flush() {
    WriteHeader(num_points_);
    const bool ok = std::fclose(file_) == 0;
    file_ = nullptr;
    if (!ok) throw Error(DL_ERR_ARG, "PCD close failed");
  }

 private:
  void WriteHeader(int64_t num_points) {
    char header[320];
    const int len = std::snprintf(header, sizeof(header),
                                  "# generated by Cartographer\nVERSION .7\nFIELDS x y z\nSIZE 4 4 4\nTYPE F F F\nCOUNT 1 1 1\n"
                                  "WIDTH %015lld\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS %015lld\nDATA binary\n",
                                  (long long)num_points, (long long)num_points);
    if (std::fseek(file_, 0, SEEK_SET) != 0 || std::fwrite(header, 1, (size_t)len, file_) != (size_t)len)
      throw Error(DL_ERR_ARG, "PCD header write failed");
    if (std::fseek(file_, 0, SEEK_END) != 0) throw Error(DL_ERR_ARG, "PCD seek failed");
  }
  std::FILE* file_;
  int64_t num_points_ = 0;
};

}  // namespace io

namespace cartographer_ros {

// std::to_string(double): "%f"
inline std::string ToString(double v) {
  char buf[512];
  std::snprintf(buf, sizeof(buf), "%f", v);
  return buf;
}

// WritePgm (ros_map.cc): the header, then the red channel row by row
inline std::string PgmBytes(const io::GreyImage& image, double resolution) {
  std::string out = "P5\n# Cartographer map; " + ToString(resolution) + " m/pixel\n" + std::to_string(image.width) + " " +
                    std::to_string(image.height) + "\n255\n";
  out.append(image.pixels.begin(), image.pixels.end());
  return out;
}

// WriteYaml (ros_map.cc): map_saver's constants
inline std::string YamlBytes(double resolution, double origin_x, double origin_y, const std::string& pgm_filename) {
  return "image: " + pgm_filename + "\n" + "resolution: " + ToString(resolution) + "\n" + "origin: [" + ToString(origin_x) +
         ", " + ToString(origin_y) + ", 0.0]\nnegate: 0\noccupied_thresh: 0.65\nfree_thresh: 0.196\n";
}

// cartographer_ros::RosMapWritingPointsProcessor (ros_map_writing_points_processor.cc): Flush, after the writer's final Flush,
// writes <filestem>.pgm (the image rotated 90 degrees clockwise) and <filestem>.yaml.
class RosMapWritingPointsProcessor {
 public:
  RosMapWritingPointsProcessor(io::MapWriter* writer, double resolution, double hit_probability, double miss_probability,
                               bool insert_free_space, const std::string& filestem)
      : writer_(writer), stage_(writer->AddProbabilityGrid(resolution, hit_probability, miss_probability, insert_free_space)),
        filestem_(filestem) {}
  void Flush() const {
    dl_map_writer_grid_info info;
    io::GreyImage image = io::DrawProbabilityGrid(*writer_, stage_, &info);
    const std::string pgm_filename = filestem_ + ".pgm";
    image.Rotate90DegreesClockwise();
    io::WriteFile(pgm_filename, PgmBytes(image, info.resolution));
    const double origin_x = info.max_x - (info.offset_y + image.width) * info.resolution;
    const double origin_y = info.max_y - (info.offset_x + image.height) * info.resolution;
    io::WriteFile(filestem_ + ".yaml", YamlBytes(info.resolution, origin_x, origin_y, pgm_filename));
  }
  int stage() const { return stage_; }

 private:
  io::MapWriter* writer_;
  int stage_;
  std::string filestem_;
};

}  // namespace cartographer_ros
}  // namespace dliom
