// The range-data map of a SLAM run: the counterpart of the fork's `--save_range_data` followed by pb_range_data_to_ros_cloud.
// A recorded multi-trajectory drive is replayed as host/example_global_slam.cc replays it (same input file), with
// PoseGraph3D::EnableRangeDataCache (MapBuilderBridge::EnableFullCloudCache) on, so every node keeps its range_data_in_local
// returns in the graph's device node store. After RunFinalOptimization the map (every node's returns at its optimized pose) is
// written as a binary PCD through io::PcdWritingPointsProcessor.
// Usage: example_range_data_map <drive file> <output.pcd>. Prints one line: nodes and points of the map.
#include <cstdio>
#include <memory>
#include <vector>

#include "dliom_b200.hpp"

int main(int argc, char** argv) {
  using namespace dliom;
  if (argc < 3) return 3;
  std::FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 3;
  try {
    Context ctx(0);
    mapping::PoseGraphOptions options;
    int32_t n = 0;
    if (std::fread(&options.optimize_every_n_nodes, 4, 1, f) != 1) return 3;
    options.every_nodes_to_find_constraint = 2;
    options.constraint_builder_options.min_score = 0.3;
    options.constraint_builder_options.fast_correlative_scan_matcher_options_3d.min_low_resolution_score = 0.3;
    mapping::PoseGraph3D pose_graph(&ctx, options);
    pose_graph.EnableRangeDataCache();
    if (std::fread(&n, 4, 1, f) != 1) return 3;
    for (int k = 0; k < n; ++k) {
      int32_t t = 0;
      if (std::fread(&t, 4, 1, f) != 1) return 3;
      pose_graph.FreezeTrajectory(t);
    }
    mapping::LocalTrajectoryBuilderOptions3D ltb_options;
    ltb_options.c.num_range_data = 3;
    ltb_options.c.motion_filter_max_time_seconds = 0.05;
    ltb_options.c.imu_weight = 0.7;
    int32_t num_trajectories = 0;
    if (std::fread(&num_trajectories, 4, 1, f) != 1) return 3;
    std::vector<std::unique_ptr<mapping::LocalTrajectoryBuilder3D>> builders;  // own the submap grids the graph borrows
    for (int trajectory_id = 0; trajectory_id < num_trajectories; ++trajectory_id) {
      builders.emplace_back(new mapping::LocalTrajectoryBuilder3D(&ctx, ltb_options, {"lidar"}));
      mapping::LocalTrajectoryBuilder3D& builder = *builders.back();
      dl_nav_state init{};
      int32_t num_events = 0;
      if (std::fread(&init, sizeof(init), 1, f) != 1 || std::fread(&num_events, 4, 1, f) != 1) return 3;
      builder.SetInitialState(init);
      for (int e = 0; e < num_events; ++e) {
        int32_t kind;
        double time;
        if (std::fread(&kind, 4, 1, f) != 1 || std::fread(&time, 8, 1, f) != 1) return 3;
        if (kind == 0) {
          sensor::ImuData imu{time, {}, {}};
          if (std::fread(imu.linear_acceleration.data(), 8, 3, f) != 3 || std::fread(imu.angular_velocity.data(), 8, 3, f) != 3) return 3;
          builder.AddImuData(imu);
          continue;
        }
        sensor::TimedPointCloudData cloud{time, {0.f, 0.f, 0.f}, {}};
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
        if (result && result->insertion_result) pose_graph.AddNode(trajectory_id, builder, *result->insertion_result, matches);
      }
    }
    std::fclose(f);
    pose_graph.RunFinalOptimization();
    const mapping::PoseGraph3D::RangeDataMapResult map = pose_graph.RangeDataMap();
    io::PcdWritingPointsProcessor pcd(argv[2]);
    pcd.Process(map.points);
    pcd.Flush();
    std::printf("nodes %zu points %zu\n", map.nodes.size(), map.points.size());
    return 0;
  } catch (const Error& e) {
    std::fprintf(stderr, "dliom error %d: %s\n", e.status, e.what());
    return 2;
  }
}
