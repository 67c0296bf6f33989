// Reads like SM/ceres_scan_matcher_3d_test.cc:34-116 and SM/real_time_correlative_scan_matcher_3d_test.cc:36-117,
// but runs the GPU path through the C++ shim. Build: g++ -std=c++17 example_match.cc -L.. -ldliom_b200
#include <cmath>
#include <cstdio>

#include "dliom_b200.hpp"

int main() {
  using namespace dliom;
  try {
    Context ctx(0);
    const PointCloud cloud = {{-3.f, 2.f, 0.f}, {-4.f, 2.f, 0.f}, {-5.f, 2.f, 0.f}, {-6.f, 2.f, 0.f},
                              {-6.f, 3.f, 1.f}, {-6.f, 4.f, 2.f}, {-7.f, 3.f, 1.f}};
    // hybrid_grid_.SetProbability(GetCellIndex(expected_pose * point), 1.) with expected_pose = Translation(-1,0,0);
    // ProbabilityToValue(1.) clamps to 0.9 -> 32767.
    DeviceHybridGrid grid(&ctx, 1.f);
    std::vector<int32_t> x, y, z;
    std::vector<uint16_t> v;
    for (const auto& p : cloud) {
      x.push_back((int32_t)std::lround(p[0] - 1.f)); y.push_back((int32_t)std::lround(p[1])); z.push_back((int32_t)std::lround(p[2]));
      v.push_back(32767);
    }
    grid.Update(x, y, z, v);
    scan_matching::CeresScanMatcherOptions3D options;
    options.occupied_space_weight = {1.};
    options.translation_weight = 0.01;
    options.rotation_weight = 0.1;
    options.use_nonmonotonic_steps = true;
    options.max_num_iterations = 10;
    scan_matching::CeresScanMatcher3D matcher(&ctx, options);
    Rigid3d initial, pose;
    initial.t[0] = -0.9; initial.t[1] = -0.2; initial.t[2] = 0.2;
    scan_matching::SolverSummary summary;
    matcher.Match({initial.t[0], initial.t[1], initial.t[2]}, initial, {{&cloud, &grid}}, &pose, &summary);
    std::printf("pose %.6f %.6f %.6f  final_cost %.6g  iterations %d\n", pose.t[0], pose.t[1], pose.t[2], summary.final_cost,
                summary.num_iterations);
    const bool ok = summary.final_cost <= 1e-2 && std::fabs(pose.t[0] + 1.) < 3e-2 && std::fabs(pose.t[1]) < 3e-2;
    const PointCloud filtered = sensor::VoxelFilter(&ctx, 2.5f).Filter(cloud);
    std::printf("voxel filter kept %zu of %zu\n", filtered.size(), cloud.size());
    // loop closure: the same cloud against the same grid from a guess 2 cells off; window 3 m, min_score 0.5
    constraints::ConstraintBuilderOptions cb;
    cb.min_score = 0.5;
    cb.fast_correlative_scan_matcher_options_3d.linear_xy_search_window = 3.;
    cb.fast_correlative_scan_matcher_options_3d.linear_z_search_window = 3.;
    cb.fast_correlative_scan_matcher_options_3d.min_low_resolution_score = 0.5;
    constraints::ConstraintBuilder3D builder(&ctx, cb);
    Rigid3d guess;
    guess.t[0] = 1.; guess.t[1] = -1.;
    builder.MaybeAddConstraint(/*submap*/ 3, &grid, &grid, /*node*/ 17, cloud, cloud, guess);
    Rigid3d far;
    far.t[0] = 40.;
    builder.MaybeAddConstraint(3, &grid, &grid, 18, cloud, cloud, far);
    const auto found = builder.Compute();
    std::printf("constraints found %zu", found.size());
    bool loop_ok = found.size() == 1 && found[0].node_index == 17 && std::fabs(found[0].zbar_ij.t[0] + 1.) < 0.1 &&
                   std::fabs(found[0].zbar_ij.t[1]) < 0.1 && found[0].translation_weight == 1.1e4;
    if (!found.empty()) std::printf("  node %d -> %.3f %.3f %.3f score %.3f", found[0].node_index, found[0].zbar_ij.t[0],
                                    found[0].zbar_ij.t[1], found[0].zbar_ij.t[2], found[0].score);
    std::printf("\n");
    return ok && loop_ok ? 0 : 1;
  } catch (const Error& e) {
    std::fprintf(stderr, "dliom error %d: %s\n", e.status, e.what());
    return 2;
  }
}
