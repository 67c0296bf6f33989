// TEST INFRASTRUCTURE — CPU oracle (see orc_math.h header).
//
// (1) Range-data insertion used to BUILD test submaps the way the reference does:
//       C/mapping/3d/range_data_inserter_3d.cc:27-51 (misses), :76-92 (Insert)
//       C/mapping/3d/submap_3d.cc:42-51 (FilterRangeDataByMaxRange), :264-279 (Submap3D::InsertRangeData)
// (2) The per-scan front half of LocalTrajectoryBuilder3D::AddRangeData /
//     AddAccumulatedRangeData up to and including the scan match:
//       LTB:393-395 (first voxel filter), :426-445 + :871-879 (deskew by interpolated relative pose),
//       :454-472 (transform + range gate), :476-487 (second voxel filters, back to tracking frame),
//       :502-542 (adaptive filters, optional RT-CSM, Ceres match), :553-554 (pose back to local frame)
//     (LTB = C/mapping/internal/3d/local_trajectory_builder_3d.cc). The GTSAM window that follows is
//     restated separately (orc_imu.h).
#pragma once
#include <cstdint>
#include <vector>

#include "orc_filters.h"
#include "orc_grid.h"
#include "orc_math.h"
#include "orc_nls.h"
#include "orc_rtcsm.h"

namespace orc {

struct RangeDataInserterOptions {
  double hit_probability = 0.55;
  double miss_probability = 0.49;
  int num_free_space_voxels = 2;
};

class RangeDataInserter {
 public:
  explicit RangeDataInserter(const RangeDataInserterOptions& o)
      : opt_(o),
        hit_table_(lookup_table_to_apply_odds(odds((float)o.hit_probability))),
        miss_table_(lookup_table_to_apply_odds(odds((float)o.miss_probability))) {}

  void Insert(const V3f& origin, const float* returns, int64_t n, HybridGrid* grid) const {
    for (int64_t i = 0; i < n; ++i) {
      grid->ApplyLookupTable(grid->GetCellIndex(V3f{returns[3 * i], returns[3 * i + 1], returns[3 * i + 2]}), hit_table_);
    }
    const I3 origin_cell = grid->GetCellIndex(origin);
    for (int64_t i = 0; i < n; ++i) {
      const I3 hit_cell = grid->GetCellIndex(V3f{returns[3 * i], returns[3 * i + 1], returns[3 * i + 2]});
      const I3 delta{hit_cell.x - origin_cell.x, hit_cell.y - origin_cell.y, hit_cell.z - origin_cell.z};
      const int num_samples = std::max(std::abs(delta.x), std::max(std::abs(delta.y), std::abs(delta.z)));
      for (int position = std::max(0, num_samples - opt_.num_free_space_voxels); position < num_samples; ++position) {
        // integer arithmetic: origin + delta * position / num_samples (C++ truncating division)
        const I3 miss_cell{origin_cell.x + delta.x * position / num_samples,
                           origin_cell.y + delta.y * position / num_samples,
                           origin_cell.z + delta.z * position / num_samples};
        grid->ApplyLookupTable(miss_cell, miss_table_);
      }
    }
    grid->FinishUpdate();
  }

 private:
  RangeDataInserterOptions opt_;
  std::vector<uint16_t> hit_table_, miss_table_;
};

// Submap3D::InsertRangeData of range data in the local frame (origin + returns; misses are not inserted by the reference)
// into the grids of the submap at local_pose.
inline void submap_insert_range_data(const Rigid3d& local_pose, const V3f& origin, const float* returns, int64_t n,
                                     const RangeDataInserter& ins, int high_resolution_max_range, HybridGrid* hi, HybridGrid* lo) {
  const Rigid3f to_submap = cast_f(inverse(local_pose));
  const V3f o = apply(to_submap, origin);
  std::vector<float> all, near;
  all.reserve(3 * n);
  for (int64_t i = 0; i < n; ++i) {
    const V3f p = apply(to_submap, V3f{returns[3 * i], returns[3 * i + 1], returns[3 * i + 2]});
    all.insert(all.end(), {p.x, p.y, p.z});
    if (norm(p - o) <= (float)high_resolution_max_range) near.insert(near.end(), {p.x, p.y, p.z});
  }
  ins.Insert(o, near.data(), (int64_t)near.size() / 3, hi);
  ins.Insert(o, all.data(), n, lo);
}

struct Submap {
  Rigid3d local_pose;
  HybridGrid hi, lo;
  int num_range_data = 0;
  Submap(float hi_res, float lo_res, const Rigid3d& pose) : local_pose(pose), hi(hi_res), lo(lo_res) {}

  void InsertRangeData(const V3f& origin, const float* returns, int64_t n, const RangeDataInserter& ins,
                       int high_resolution_max_range) {
    submap_insert_range_data(local_pose, origin, returns, n, ins, high_resolution_max_range, &hi, &lo);
    ++num_range_data;
  }
};

// ----------------------------------------------------------------------------- per-scan front end
struct alignas(16) RangeMeasurement {  // timed_point_cloud_data.h:33-36 (16-byte aligned Vector4f + size_t = 32 bytes)
  float x, y, z, t;
  uint64_t origin_index;
};

struct FrontEndOptions {
  float min_range = 0.5f, max_range = 100.f;
  float voxel_filter_size = 0.15f;
  double scan_period = 0.1;
  AdaptiveVoxelFilterOptions hi_filter{2.f, 150.f, 15.f};
  AdaptiveVoxelFilterOptions lo_filter{4.f, 200.f, 60.f};
  bool use_online_correlative_scan_matching = false;
  RtcsmOptions rtcsm{0.15, 0.017453292519943295, 1e-1, 1e-1};
  CeresMatcherOptions ceres;
};

// Identity.slerp(s, q) in double (Eigen QuaternionBase::slerp) and s * t: LTB:871-879.
inline Rigid3d interpolate_pose(double s, const Rigid3d& rel) {
  const double one = 1.0 - 2.220446049250313e-16;
  const Quatd id{1, 0, 0, 0};
  const double d = qdot(id, rel.q);
  const double abs_d = std::fabs(d);
  double scale0, scale1;
  if (abs_d >= one) {
    scale0 = 1.0 - s;
    scale1 = s;
  } else {
    const double theta = std::acos(abs_d);
    const double sin_theta = std::sin(theta);
    scale0 = std::sin((1.0 - s) * theta) / sin_theta;
    scale1 = std::sin(s * theta) / sin_theta;
  }
  if (d < 0) scale1 = -scale1;
  Rigid3d out;
  out.q = {scale0 * id.w + scale1 * rel.q.w, scale0 * id.x + scale1 * rel.q.x, scale0 * id.y + scale1 * rel.q.y,
           scale0 * id.z + scale1 * rel.q.z};
  out.t = scale(s, rel.t);
  return out;
}

struct ScanIngest {
  std::vector<int64_t> first_filter_keep;  // indices into the input ranges
  std::vector<float> returns_local, misses_local;          // after deskew + gate (LTB:454-472)
  std::vector<float> returns_tracking, misses_tracking;    // after second filter, back in tracking frame
  Rigid3f current_pose;                                     // hits_poses.back()
  V3f origin_tracking;
};

// prev = pose of the previous optimised state, cur = IMU-predicted pose at scan end (both local frame).
inline ScanIngest ingest_scan(const FrontEndOptions& opt, const RangeMeasurement* ranges, int64_t n,
                              const V3f* origins, const Rigid3d& prev, const Rigid3d& cur) {
  ScanIngest out;
  static_assert(sizeof(RangeMeasurement) == 32, "RangeMeasurement layout");
  VoxelFilter(0.5f * opt.voxel_filter_size).Filter(&ranges[0].x, n, 8, &out.first_filter_keep);
  const int64_t m = (int64_t)out.first_filter_keep.size();
  const Rigid3d rel = compose(inverse(prev), cur);
  const bool no_deskew = m > 0 && std::fabs(ranges[out.first_filter_keep[0]].t) < 1e-3;  // float |t| vs double 1e-3
  const Rigid3f cur_f = cast_f(cur);
  Rigid3f pose = cur_f;
  for (int64_t k = 0; k < m; ++k) {
    const RangeMeasurement& h = ranges[out.first_filter_keep[k]];
    if (!no_deskew) {
      const double s = (opt.scan_period + h.t) / opt.scan_period;
      pose = cast_f(compose(prev, interpolate_pose(s, rel)));
    }
    const V3f hit = apply(pose, V3f{h.x, h.y, h.z});
    const V3f org = apply(pose, origins[h.origin_index]);
    const V3f delta = hit - org;
    const float range = norm(delta);
    if (range >= opt.min_range) {
      if (range <= opt.max_range) {
        out.returns_local.insert(out.returns_local.end(), {hit.x, hit.y, hit.z});
      } else {
        const V3f miss = org + scale(opt.max_range / range, delta);
        out.misses_local.insert(out.misses_local.end(), {miss.x, miss.y, miss.z});
      }
    }
  }
  out.current_pose = pose;
  const Rigid3f back = inverse(out.current_pose);
  auto filter_and_transform = [&](const std::vector<float>& in, std::vector<float>* dst) {
    std::vector<int64_t> keep;
    VoxelFilter(opt.voxel_filter_size).Filter(in.data(), (int64_t)in.size() / 3, 3, &keep);
    for (int64_t i : keep) {
      const V3f p = apply(back, V3f{in[3 * i], in[3 * i + 1], in[3 * i + 2]});
      dst->insert(dst->end(), {p.x, p.y, p.z});
    }
  };
  filter_and_transform(out.returns_local, &out.returns_tracking);
  filter_and_transform(out.misses_local, &out.misses_tracking);
  out.origin_tracking = apply(back, out.current_pose.t);
  return out;
}

struct ScanMatchOutput {
  bool ok = false;
  std::vector<int64_t> hi_keep, lo_keep;  // indices into returns_tracking
  Rigid3d initial_ceres_pose, pose_observation_in_submap, pose_estimate_local;
  float rtcsm_score = 0.f;
  int64_t rtcsm_best_index = -1;
  SolveSummary summary;
};

// AddAccumulatedRangeData up to the scan match (LTB:492-554).
inline ScanMatchOutput match_scan(const FrontEndOptions& opt, const float* returns_tracking, int64_t n,
                                  const Rigid3d& pose_prediction, const Rigid3d& submap_local_pose,
                                  const HybridGrid& hi_grid, const HybridGrid& lo_grid) {
  ScanMatchOutput out;
  if (n == 0) return out;
  const Rigid3d to_submap = inverse(submap_local_pose);
  out.initial_ceres_pose = compose(to_submap, pose_prediction);
  const V3d target_translation = out.initial_ceres_pose.t;
  out.hi_keep = AdaptiveVoxelFilter(opt.hi_filter, returns_tracking, n, 3);
  if (out.hi_keep.empty()) return out;
  std::vector<float> hi_cloud, lo_cloud;
  for (int64_t i : out.hi_keep) hi_cloud.insert(hi_cloud.end(), returns_tracking + 3 * i, returns_tracking + 3 * i + 3);
  if (opt.use_online_correlative_scan_matching) {
    const RtcsmResult r =
        rtcsm_match(opt.rtcsm, out.initial_ceres_pose, hi_cloud.data(), (int64_t)hi_cloud.size() / 3, hi_grid);
    out.initial_ceres_pose = r.pose;
    out.rtcsm_score = r.score;
    out.rtcsm_best_index = r.best_index;
  }
  out.lo_keep = AdaptiveVoxelFilter(opt.lo_filter, returns_tracking, n, 3);
  if (out.lo_keep.empty()) return out;
  for (int64_t i : out.lo_keep) lo_cloud.insert(lo_cloud.end(), returns_tracking + 3 * i, returns_tracking + 3 * i + 3);
  ceres_scan_match(opt.ceres, target_translation, out.initial_ceres_pose,
                   {{hi_cloud.data(), (int64_t)hi_cloud.size() / 3, &hi_grid},
                    {lo_cloud.data(), (int64_t)lo_cloud.size() / 3, &lo_grid}},
                   &out.pose_observation_in_submap, &out.summary);
  out.pose_estimate_local = compose(submap_local_pose, out.pose_observation_in_submap);
  out.ok = true;
  return out;
}

}  // namespace orc
