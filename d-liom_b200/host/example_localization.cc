// Pure localization through the C++ mirrors of mapping::LocalTrajectoryBuilder3D and mapping::PoseGraph3D (dliom_b200.hpp), wired
// as MapBuilder does with pure_localization (map_builder.cc:147-151): trajectory 0 is mapped, finally optimized and frozen; then
// trajectory 1 starts from SetInitialTrajectoryPose relative to trajectory 0, a PureLocalizationTrimmer keeps its newest
// submaps, every MatchingResult with an InsertionResult becomes PoseGraph3D::AddNode (with the host SURF stage's matches when
// the node finished a submap), and FinishTrajectory ends it. The graph releases trimmed grids on trajectory 1's builder.
// Input file (little endian), written by tests/test_gpu_localization.py:
//   int32 optimize_every_n_nodes, int32 num_submaps_to_keep, 7 doubles relative pose (t xyz, q wxyz), double time; then for
//   trajectory 0 and trajectory 1: dl_nav_state initial state, int32 num_events, then per event: int32 kind, double time,
//     kind 0 (imu): 3 doubles acc, 3 doubles gyr;
//     kind 1 (range data): int32 n, n x 4 floats (x y z t), int32 num_matches, then per match: int32 trajectory id,
//       int32 submap index, 3 doubles x y theta.
// Output: after every AddNode of trajectory 1 that optimized, "opt <k> <submaps left> <builder submaps holding grids>" and one
// line per remaining node of trajectory 1: "node <index> <pose, 7 x %.17g>"; after FinishTrajectory, "finished <nodes left>
// <submaps left> <builder submaps holding grids>".
#include <cstdio>
#include <memory>
#include <vector>

#include "dliom_b200.hpp"

namespace {

int held_grids(dliom::Context* ctx, const dliom::mapping::LocalTrajectoryBuilder3D& builder) {
  int held = 0;
  for (int i = 0; i < builder.num_submaps(); ++i)
    if (dliom::mapping::GetSubmap(ctx, builder, i).high_resolution_grid) ++held;
  return held;
}

}  // namespace

int main(int argc, char** argv) {
  using namespace dliom;
  if (argc < 2) return 3;
  std::FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 3;
  try {
    Context ctx(0);
    mapping::PoseGraphOptions options;
    int32_t keep = 0;
    double rel[7], time = 0.0;
    if (std::fread(&options.optimize_every_n_nodes, 4, 1, f) != 1 || std::fread(&keep, 4, 1, f) != 1 ||
        std::fread(rel, 8, 7, f) != 7 || std::fread(&time, 8, 1, f) != 1)
      return 3;
    options.every_nodes_to_find_constraint = 2;
    options.constraint_builder_options.min_score = 0.3;
    options.constraint_builder_options.fast_correlative_scan_matcher_options_3d.min_low_resolution_score = 0.3;
    mapping::PoseGraph3D pose_graph(&ctx, options);
    mapping::LocalTrajectoryBuilderOptions3D ltb_options;
    ltb_options.c.num_range_data = 3;
    ltb_options.c.motion_filter_max_time_seconds = 0.05;
    ltb_options.c.imu_weight = 0.7;
    std::vector<std::unique_ptr<mapping::LocalTrajectoryBuilder3D>> builders;  // own the submap grids the graph borrows
    int optimizations = 0;
    for (int trajectory_id = 0; trajectory_id < 2; ++trajectory_id) {
      if (trajectory_id == 1) {  // the map is done: freeze it, then localize
        pose_graph.RunFinalOptimization();
        pose_graph.FreezeTrajectory(0);
        pose_graph.SetInitialTrajectoryPose(1, 0, Rigid3d::from7(rel), time);
        pose_graph.AddTrimmer(std::unique_ptr<mapping::PoseGraphTrimmer>(new mapping::PureLocalizationTrimmer(1, keep)));
      }
      builders.emplace_back(new mapping::LocalTrajectoryBuilder3D(&ctx, ltb_options, {"lidar"}));
      mapping::LocalTrajectoryBuilder3D& builder = *builders.back();
      dl_nav_state init{};
      int32_t num_events = 0, n = 0;
      if (std::fread(&init, sizeof(init), 1, f) != 1 || std::fread(&num_events, 4, 1, f) != 1) return 3;
      builder.SetInitialState(init);
      for (int e = 0; e < num_events; ++e) {
        int32_t kind;
        double t;
        if (std::fread(&kind, 4, 1, f) != 1 || std::fread(&t, 8, 1, f) != 1) return 3;
        if (kind == 0) {
          sensor::ImuData imu{t, {}, {}};
          if (std::fread(imu.linear_acceleration.data(), 8, 3, f) != 3 || std::fread(imu.angular_velocity.data(), 8, 3, f) != 3) return 3;
          builder.AddImuData(imu);
          continue;
        }
        sensor::TimedPointCloudData cloud{t, {0.f, 0.f, 0.f}, {}};
        if (std::fread(&n, 4, 1, f) != 1) return 3;
        cloud.ranges.resize(n);
        if (n && std::fread(cloud.ranges[0].data(), 16, n, f) != (size_t)n) return 3;
        std::vector<mapping::SubmapMatch> matches;
        if (std::fread(&n, 4, 1, f) != 1) return 3;
        for (int k = 0; k < n; ++k) {
          int32_t ids[2];
          double xyt[3];
          if (std::fread(ids, 4, 2, f) != 2 || std::fread(xyt, 8, 3, f) != 3) return 3;
          matches.push_back({{ids[0], ids[1]}, xyt[0], xyt[1], xyt[2]});
        }
        const auto result = builder.AddRangeData("lidar", cloud);
        if (!result || !result->insertion_result) continue;
        dl_pg3d_add_node_info info{};
        pose_graph.AddNode(trajectory_id, builder, *result->insertion_result, matches, &info);
        if (trajectory_id != 1 || !info.optimized) continue;
        std::printf("opt %d %zu %d\n", optimizations++, pose_graph.GetAllSubmapPosesById(1).size(), held_grids(&ctx, builder));
        for (const auto& kv : pose_graph.GetTrajectoryNodePosesById(1)) {
          std::printf("node %d", kv.first.node_index);
          for (double v : kv.second.t) std::printf(" %.17g", v);
          for (double v : kv.second.q) std::printf(" %.17g", v);
          std::printf("\n");
        }
      }
    }
    std::fclose(f);
    pose_graph.FinishTrajectory(1);
    std::printf("finished %zu %zu %d\n", pose_graph.GetTrajectoryNodePosesById(1).size(), pose_graph.GetAllSubmapPosesById(1).size(),
                held_grids(&ctx, *builders[1]));
    return 0;
  } catch (const Error& e) {
    std::fprintf(stderr, "dliom error %d: %s\n", e.status, e.what());
    return 2;
  }
}
