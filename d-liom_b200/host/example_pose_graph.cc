// Runs OptimizationProblem3D::Solve through the C++ mirror (dliom_b200.hpp, optimization::OptimizationProblem3D) on a pose graph
// read from a file, the way PoseGraph3D::RunOptimization feeds the reference's (pose_graph_3d.cc), with some trajectories frozen
// as after loading a map.
// Input file (little endian), written by tests/test_gpu_posegraph_sparse.py:
//   int32 num_submaps, then per submap: int32 trajectory_id, 7 doubles global pose (t xyz, q wxyz), in id order per trajectory;
//   int32 num_nodes, then per node: the same;
//   int32 num_constraints, then per constraint: int32 submap trajectory, submap index, node trajectory, node index,
//     7 doubles zbar_ij, double translation_weight, double rotation_weight;
//   int32 num_frozen, then that many int32 frozen trajectory ids.
// Output: one line per submap, then per node, in id order: trajectory id, index, pose (7); then the summary.
#include <cstdio>
#include <set>
#include <vector>

#include "dliom_b200.hpp"

namespace {
bool read_pose(std::FILE* f, int32_t* trajectory, dliom::Rigid3d* pose) {
  double p[7];
  if (std::fread(trajectory, 4, 1, f) != 1 || std::fread(p, 8, 7, f) != 7) return false;
  *pose = dliom::Rigid3d::from7(p);
  return true;
}
}  // namespace

int main(int argc, char** argv) {
  using namespace dliom;
  if (argc < 2) return 3;
  std::FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 3;
  try {
    Context ctx(0);
    optimization::OptimizationProblem3D problem(&ctx);
    int32_t n = 0, trajectory = 0;
    Rigid3d pose;
    if (std::fread(&n, 4, 1, f) != 1) return 3;
    for (int k = 0; k < n; ++k) {
      if (!read_pose(f, &trajectory, &pose)) return 3;
      problem.AddSubmap(trajectory, pose);
    }
    if (std::fread(&n, 4, 1, f) != 1) return 3;
    for (int k = 0; k < n; ++k) {
      if (!read_pose(f, &trajectory, &pose)) return 3;
      problem.AddTrajectoryNode(trajectory, {pose});
    }
    std::vector<optimization::Constraint> constraints;
    if (std::fread(&n, 4, 1, f) != 1) return 3;
    for (int k = 0; k < n; ++k) {
      int32_t ids[4];
      double z[9];
      if (std::fread(ids, 4, 4, f) != 4 || std::fread(z, 8, 9, f) != 9) return 3;
      constraints.push_back({{ids[0], ids[1]}, {ids[2], ids[3]}, Rigid3d::from7(z), z[7], z[8]});
    }
    std::set<int> frozen_trajectories;
    if (std::fread(&n, 4, 1, f) != 1) return 3;
    for (int k = 0; k < n; ++k) {
      if (std::fread(&trajectory, 4, 1, f) != 1) return 3;
      frozen_trajectories.insert(trajectory);
    }
    std::fclose(f);
    problem.SetMaxNumIterations(50);
    problem.Solve(constraints, frozen_trajectories);
    for (const auto& kv : problem.submap_data()) {
      std::printf("submap %d %d", kv.first.trajectory_id, kv.first.submap_index);
      for (double v : kv.second.global_pose.t) std::printf(" %.17g", v);
      for (double v : kv.second.global_pose.q) std::printf(" %.17g", v);
      std::printf("\n");
    }
    for (const auto& kv : problem.node_data()) {
      std::printf("node %d %d", kv.first.trajectory_id, kv.first.node_index);
      for (double v : kv.second.global_pose.t) std::printf(" %.17g", v);
      for (double v : kv.second.global_pose.q) std::printf(" %.17g", v);
      std::printf("\n");
    }
    const dl_solve_summary& s = problem.summary();
    std::printf("summary %d %d %.17g %.17g\n", s.num_iterations, s.termination, s.initial_cost, s.final_cost);
    return 0;
  } catch (const Error& e) {
    std::fprintf(stderr, "dliom error %d: %s\n", e.status, e.what());
    return 2;
  }
}
