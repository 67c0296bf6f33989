// Writes the 2D occupancy map of a finished run the way the reference's ROS map pipeline does
// (cartographer_ros/configuration_files/assets_writer_ros_map.lua: write_ros_map at 0.05 m with hit_probability 0.55,
// miss_probability 0.49 and insert_free_space), plus the same grid as write_probability_grid's PNG, through io::MapWriter,
// cartographer_ros::RosMapWritingPointsProcessor and io::ProbabilityGridPointsProcessor (dliom_b200.hpp). Trajectories are not
// drawn on the PNG (draw_trajectories = false).
// Usage: example_ros_map <input file> <output directory>
// Input file: the format of example_write_map.cc (range filter and moving-object removal come from it).
// Output: <directory>/map.pgm, map.yaml, probability_grid.png; "points <count>" and "grid <width> <height>" (the cropped grid).
#include <cstdio>
#include <string>
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
    const std::string dir = std::string(argv[2]) + "/";
    cartographer_ros::RosMapWritingPointsProcessor ros_map(&writer, 0.05, 0.55, 0.49, true, dir + "map");
    io::ProbabilityGridPointsProcessor grid(&writer, 0.05, 0.55, 0.49, true, dir + "probability_grid");
    int64_t num_points = 0;
    for (;;) {
      num_points += (int64_t)writer.Process(messages).size();
      if (writer.Flush() == io::FlushResult::kFinished) break;
    }
    ros_map.Flush();
    grid.Flush();
    dl_map_writer_grid_info info;
    io::DrawProbabilityGrid(writer, grid.stage(), &info);
    std::printf("points %lld\ngrid %d %d\n", (long long)num_points, info.width, info.height);
    return 0;
  } catch (const Error& e) {
    std::fprintf(stderr, "dliom error %d: %s\n", e.status, e.what());
    return 2;
  }
}
