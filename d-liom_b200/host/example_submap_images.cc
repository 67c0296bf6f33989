// Replays a drive through mapping::LocalTrajectoryBuilder3D and mapping::PoseGraph3D (every inserted node goes to AddNode, no
// loop-closure matches) and writes every submap's images as binary PGM files: the two ToResponseProto textures (value and alpha
// bytes as two images each) at the pose graph's global submap pose, as MapBuilder::SubmapToProto serves them, and the
// ProjectToCvMat image the loop detector reads, at the submap's local pose; all submaps of all trajectories in one device call
// per kind. Input file: the format of example_trajectories_batch.cc. Usage: example_submap_images <input> <output directory>
// Output: <dir>/t<trajectory>_s<submap>_tex<0|1>_value.pgm, ..._alpha.pgm, <dir>/t<trajectory>_s<submap>_projection.pgm, and
// one line per submap: trajectory, submap, num_range_data, global pose (7), local pose (7), texture sizes, projection size,
// ox, oy (%.17g).
#include <cstdio>
#include <memory>
#include <string>
#include <vector>

#include "dliom_b200.hpp"

static bool write_pgm(const std::string& path, int width, int height, const uint8_t* bytes, int stride) {
  std::FILE* f = std::fopen(path.c_str(), "wb");
  if (!f) return false;
  std::fprintf(f, "P5\n%d %d\n255\n", width, height);
  for (long i = 0; i < (long)width * height; ++i) std::fputc(bytes[i * stride], f);
  return std::fclose(f) == 0;
}

int main(int argc, char** argv) {
  using namespace dliom;
  if (argc < 3) return 3;
  std::FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 3;
  const std::string dir = argv[2];
  try {
    Context ctx(0);
    mapping::LocalTrajectoryBuilderOptions3D options;
    options.c.num_range_data = 3;
    options.c.motion_filter_max_time_seconds = 0.05;
    options.c.imu_weight = 0.7;
    int32_t T = 0, steps = 0;
    if (std::fread(&T, 4, 1, f) != 1 || T < 1) return 3;
    mapping::PoseGraphOptions graph_options;
    graph_options.optimize_every_n_nodes = 6;
    mapping::PoseGraph3D pose_graph(&ctx, graph_options);
    std::vector<std::unique_ptr<mapping::LocalTrajectoryBuilder3D>> builders;
    for (int j = 0; j < T; ++j) {
      dl_nav_state init{};
      if (std::fread(&init, sizeof(init), 1, f) != 1) return 3;
      builders.emplace_back(new mapping::LocalTrajectoryBuilder3D(&ctx, options, {"lidar"}));
      builders.back()->SetInitialState(init);
    }
    if (std::fread(&steps, 4, 1, f) != 1) return 3;
    for (int s = 0; s < steps; ++s) {
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
        sensor::TimedPointCloudData cloud;
        int32_t n;
        cloud.origin = {0.f, 0.f, 0.f};
        if (std::fread(&cloud.time, 8, 1, f) != 1 || std::fread(&n, 4, 1, f) != 1) return 3;
        cloud.ranges.resize(n);
        if (n && std::fread(cloud.ranges[0].data(), 16, n, f) != (size_t)n) return 3;
        const auto result = builders[j]->AddRangeData("lidar", cloud);
        if (result && result->insertion_result) pose_graph.AddNode(j, *builders[j], *result->insertion_result, {});
      }
    }
    std::fclose(f);
    pose_graph.RunFinalOptimization();
    std::vector<std::pair<mapping::Submap3D, Rigid3d>> submaps;
    std::vector<std::pair<const dl_grid*, Rigid3d>> high_grids;
    std::vector<std::pair<int, int>> ids;
    for (int j = 0; j < T; ++j) {
      const std::vector<Rigid3d> global_poses = pose_graph.GetAllSubmapPoses(j);
      for (int i = 0; i < builders[j]->num_submaps() && i < (int)global_poses.size(); ++i) {
        const mapping::Submap3D submap = mapping::GetSubmap(&ctx, *builders[j], i);
        submaps.push_back({submap, global_poses.at(i)});
        high_grids.push_back({submap.high_resolution_grid, submap.local_pose});
        ids.push_back({j, i});
      }
    }
    const std::vector<mapping::SubmapQueryResponse> responses = mapping::ToResponseProto(&ctx, submaps);
    const std::vector<mapping::SubmapProjection> projections = mapping::ProjectToCvMat(&ctx, high_grids);
    for (size_t k = 0; k < ids.size(); ++k) {
      const std::string stem = dir + "/t" + std::to_string(ids[k].first) + "_s" + std::to_string(ids[k].second);
      std::printf("submap %d %d %d", ids[k].first, ids[k].second, responses[k].submap_version);
      for (const Rigid3d& pose : {submaps[k].second, submaps[k].first.local_pose}) {
        for (double v : pose.t) std::printf(" %.17g", v);
        for (double v : pose.q) std::printf(" %.17g", v);
      }
      for (int t = 0; t < 2; ++t) {
        const mapping::SubmapTexture& tex = responses[k].textures[t];
        const std::string name = stem + "_tex" + std::to_string(t);
        if (!write_pgm(name + "_value.pgm", tex.width, tex.height, tex.cells.data(), 2) ||
            !write_pgm(name + "_alpha.pgm", tex.width, tex.height, tex.cells.data() + (tex.cells.empty() ? 0 : 1), 2))
          return 4;
        std::printf(" %dx%d", tex.width, tex.height);
      }
      const mapping::SubmapProjection& p = projections[k];
      if (!write_pgm(stem + "_projection.pgm", p.width, p.height, p.pixels.data(), 1)) return 4;
      std::printf(" %dx%d %.17g %.17g\n", p.width, p.height, p.ox, p.oy);
    }
    return 0;
  } catch (const Error& e) {
    std::fprintf(stderr, "dliom error %d: %s\n", e.status, e.what());
    return 2;
  }
}
