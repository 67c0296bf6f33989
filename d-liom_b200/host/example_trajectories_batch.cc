// Several trajectories stepped together, the way a MapBuilder holding one mapping::LocalTrajectoryBuilder3D per trajectory would:
// `batch` hands every trajectory's scan of a step to the static LocalTrajectoryBuilder3D::AddRangeData in one call, `single` calls
// each builder's own AddRangeData. Both must print the same lines.
// Input file (little endian), written by tests/test_gpu_ltb_batch.py:
//   int32 T, T x dl_nav_state (initial states), int32 num_steps, then per step and trajectory: int32 m, m x (double time,
//   3 doubles acc, 3 doubles gyr), double scan time, int32 n, n x 4 floats (x y z t).
// Output: one line per MatchingResult: trajectory, time, pose (7), inserted, number of returns, number of submaps.
#include <cstdio>
#include <cstring>
#include <memory>
#include <vector>

#include "dliom_b200.hpp"

int main(int argc, char** argv) {
  using namespace dliom;
  if (argc < 3) return 3;
  const bool batch = std::strcmp(argv[2], "batch") == 0;
  std::FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 3;
  try {
    Context ctx(0);
    mapping::LocalTrajectoryBuilderOptions3D options;
    options.c.num_range_data = 3;
    options.c.motion_filter_max_time_seconds = 0.05;
    options.c.imu_weight = 0.7;
    int32_t T = 0, steps = 0;
    if (std::fread(&T, 4, 1, f) != 1 || T < 1) return 3;
    std::vector<std::unique_ptr<mapping::LocalTrajectoryBuilder3D>> builders;
    for (int j = 0; j < T; ++j) {
      dl_nav_state init{};
      if (std::fread(&init, sizeof(init), 1, f) != 1) return 3;
      builders.emplace_back(new mapping::LocalTrajectoryBuilder3D(&ctx, options, {"lidar"}));
      builders.back()->SetInitialState(init);
    }
    if (std::fread(&steps, 4, 1, f) != 1) return 3;
    for (int s = 0; s < steps; ++s) {
      std::vector<sensor::TimedPointCloudData> clouds(T);
      for (int j = 0; j < T; ++j) {
        int32_t m;
        if (std::fread(&m, 4, 1, f) != 1) return 3;
        for (int i = 0; i < m; ++i) {
          sensor::ImuData imu{0, {}, {}};
          if (std::fread(&imu.time, 8, 1, f) != 1 || std::fread(imu.linear_acceleration.data(), 8, 3, f) != 3 ||
              std::fread(imu.angular_velocity.data(), 8, 3, f) != 3)
            return 3;
          builders[j]->AddImuData(imu);
        }
        int32_t n;
        clouds[j].origin = {0.f, 0.f, 0.f};
        if (std::fread(&clouds[j].time, 8, 1, f) != 1 || std::fread(&n, 4, 1, f) != 1) return 3;
        clouds[j].ranges.resize(n);
        if (n && std::fread(clouds[j].ranges[0].data(), 16, n, f) != (size_t)n) return 3;
      }
      std::vector<std::unique_ptr<mapping::LocalTrajectoryBuilder3D::MatchingResult>> results;
      if (batch) {
        std::vector<mapping::LocalTrajectoryBuilder3D::RangeDataItem> items;
        for (int j = 0; j < T; ++j) items.push_back({builders[j].get(), "lidar", &clouds[j]});
        results = mapping::LocalTrajectoryBuilder3D::AddRangeData(items);
      } else {
        for (int j = 0; j < T; ++j) results.push_back(builders[j]->AddRangeData("lidar", clouds[j]));
      }
      for (int j = 0; j < T; ++j) {
        const auto& result = results[j];
        if (!result) {
          std::printf("none %d\n", j);
          continue;
        }
        std::printf("result %d %.17g", j, result->time);
        for (int k = 0; k < 3; ++k) std::printf(" %.17g", result->local_pose.t[k]);
        for (int k = 0; k < 4; ++k) std::printf(" %.17g", result->local_pose.q[k]);
        std::printf(" %d %zu %d\n", result->insertion_result ? 1 : 0, result->range_data_in_local.returns.size(),
                    builders[j]->num_submaps());
      }
    }
    std::fclose(f);
    return 0;
  } catch (const Error& e) {
    std::fprintf(stderr, "dliom error %d: %s\n", e.status, e.what());
    return 2;
  }
}
