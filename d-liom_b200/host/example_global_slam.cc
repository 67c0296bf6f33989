// Replays a recorded multi-trajectory drive through the C++ mirrors of mapping::LocalTrajectoryBuilder3D and mapping::PoseGraph3D
// (dliom_b200.hpp), wired the way GlobalTrajectoryBuilder::AddSensorData feeds the reference's (global_trajectory_builder.cc:56-104):
// every MatchingResult with an InsertionResult becomes PoseGraph3D::AddNode, with the host SURF stage's submap matches when the
// node finished a submap. The trajectories are driven one after another; each has its own builder (one LiDAR, "lidar").
// Input file (little endian), written by tests/test_gpu_pose_graph3d.py:
//   int32 optimize_every_n_nodes; int32 num_frozen, that many int32 frozen trajectory ids; int32 num_trajectories, then per
//   trajectory: dl_nav_state initial state, int32 num_events, then per event: int32 kind, double time,
//     kind 0 (imu): 3 doubles acc, 3 doubles gyr;
//     kind 1 (range data): int32 n, n x 4 floats (x y z t), int32 num_matches, then per match: int32 trajectory id,
//       int32 submap index, 3 doubles x y theta.
// Output: per trajectory in id order, one line per node then per submap: kind, trajectory id, index, pose (7, %.17g); then the
// final optimization's summary.
#include <cstdio>
#include <memory>
#include <vector>

#include "dliom_b200.hpp"

int main(int argc, char** argv) {
  using namespace dliom;
  if (argc < 2) return 3;
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
    const dl_solve_summary s = pose_graph.RunFinalOptimization();
    for (int trajectory_id = 0; trajectory_id < num_trajectories; ++trajectory_id) {
      const char* kinds[2] = {"node", "submap"};
      const std::vector<Rigid3d> poses[2] = {pose_graph.GetTrajectoryNodePoses(trajectory_id),
                                             pose_graph.GetAllSubmapPoses(trajectory_id)};
      for (int k = 0; k < 2; ++k)
        for (size_t i = 0; i < poses[k].size(); ++i) {
          std::printf("%s %d %zu", kinds[k], trajectory_id, i);
          for (double v : poses[k][i].t) std::printf(" %.17g", v);
          for (double v : poses[k][i].q) std::printf(" %.17g", v);
          std::printf("\n");
        }
    }
    int intra = 0, inter = 0;
    for (const auto& c : pose_graph.constraints()) (c.tag == mapping::PoseGraphConstraint::INTRA_SUBMAP ? intra : inter)++;
    std::printf("summary %d %d %.17g %.17g %d %d\n", s.num_iterations, s.termination, s.initial_cost, s.final_cost, intra, inter);
    return 0;
  } catch (const Error& e) {
    std::fprintf(stderr, "dliom error %d: %s\n", e.status, e.what());
    return 2;
  }
}
