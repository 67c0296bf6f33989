// Writes the map of a finished run the way cartographer_ros's assets writer does (assets_writer.cc with the fork's
// assets_writer_tongji.lua, plus the moving-object removal): trajectories and sensor messages in, points.pcd out, through the
// C++ mirrors io::MapWriter and io::PcdWritingPointsProcessor (dliom_b200.hpp). Every message is streamed in one call per pass,
// and the stream is restarted while Flush asks for it; the PCD writer receives the final pass's points.
// Usage: example_write_map <input file> <output .pcd>
// Input file (little endian), written by tests/test_gpu_map_writer.py:
//   int32 range_filter, double min_range, double max_range, double outlier_voxel_size (0: no moving-object removal);
//   int32 num_trajectories, then per trajectory: int32 id, int32 n, n int64 node times (universal ticks), n x 7 doubles poses;
//   int32 num_messages, then per message: int64 stamp (ticks), int32 trajectory id, 7 doubles sensor_to_tracking, int32 n,
//     n x 4 floats (x y z t).
// Output: "points <count>" on stdout.
#include <cstdio>
#include <vector>

#include "dliom_b200.hpp"

namespace {

template <typename T>
bool read(std::FILE* f, T* out, size_t n = 1) {
  return std::fread(out, sizeof(T), n, f) == n;
}

}  // namespace

int main(int argc, char** argv) {
  using namespace dliom;
  if (argc < 3) return 3;
  std::FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 3;
  io::MapWriterOptions options;
  int32_t range_filter = 0, num_trajectories = 0, num_messages = 0;
  if (!read(f, &range_filter) || !read(f, &options.range.min_range) || !read(f, &options.range.max_range) ||
      !read(f, &options.outlier.voxel_size))
    return 3;
  options.min_max_range_filter = range_filter != 0;
  options.remove_moving_objects = options.outlier.voxel_size > 0.0;
  struct Trajectory {
    int32_t id;
    std::vector<int64_t> times;
    std::vector<Rigid3d> poses;
  };
  std::vector<Trajectory> trajectories;
  if (!read(f, &num_trajectories)) return 3;
  for (int k = 0; k < num_trajectories; ++k) {
    Trajectory t;
    int32_t n = 0;
    if (!read(f, &t.id) || !read(f, &n) || n < 0) return 3;
    t.times.resize(n);
    if (n && !read(f, t.times.data(), (size_t)n)) return 3;
    for (int i = 0; i < n; ++i) {
      double p[7];
      if (!read(f, p, 7)) return 3;
      t.poses.push_back(Rigid3d::from7(p));
    }
    trajectories.push_back(std::move(t));
  }
  std::vector<io::Message> messages;
  if (!read(f, &num_messages)) return 3;
  for (int k = 0; k < num_messages; ++k) {
    io::Message m;
    double s2t[7];
    int32_t id = 0, n = 0;
    if (!read(f, &m.stamp) || !read(f, &id) || !read(f, s2t, 7) || !read(f, &n) || n < 0) return 3;
    m.trajectory_id = id;
    m.sensor_to_tracking = Rigid3d::from7(s2t);
    m.rows.resize(n);
    if (n && !read(f, m.rows[0].data(), 4 * (size_t)n)) return 3;
    messages.push_back(std::move(m));
  }
  std::fclose(f);
  try {
    Context ctx(0);
    io::MapWriter writer(&ctx, options);
    for (const Trajectory& t : trajectories) writer.AddTrajectory(t.id, t.times, t.poses);
    io::PcdWritingPointsProcessor pcd(argv[2]);
    int64_t num_points = 0;
    for (;;) {
      const PointCloud points = writer.Process(messages);
      pcd.Process(points);
      num_points += (int64_t)points.size();
      if (writer.Flush() == io::FlushResult::kFinished) break;
    }
    pcd.Flush();
    std::printf("points %lld\n", (long long)num_points);
    return 0;
  } catch (const Error& e) {
    std::fprintf(stderr, "dliom error %d: %s\n", e.status, e.what());
    return 2;
  }
}
