// Writes the X-ray images of a finished run the way the reference's stock 3D pipeline does
// (cartographer_ros/configuration_files/assets_writer_backpack_3d.lua with transform.lua, VOXEL_SIZE = 5e-2): three gray
// write_xray_image stages (YZ, XY, XZ), color_points for the horizontal (red) and the vertical (green) LiDAR, and the three
// X-rays again in colour, through io::MapWriter, io::ColoringPointsProcessor and io::XRayPointsProcessor (dliom_b200.hpp).
// Trajectories are not drawn (draw_trajectories = false).
// Usage: example_xray <input file> <output directory>
// Input file: the format of example_write_map.cc (range filter and moving-object removal come from it). Messages alternate
// between the two LiDARs: even messages are frame "horizontal_vlp16_link", odd ones "vertical_vlp16_link".
// Output: <directory>/xray_{yz,xy,xz}_all{,_color}.png, "points <count>" and one "<name> <width> <height>" line per image.
#include <cmath>
#include <cstdio>
#include <memory>
#include <string>
#include <vector>

#include "dliom_b200.hpp"

namespace {

template <typename T>
bool read(std::FILE* f, T* out, size_t n = 1) {
  return std::fread(out, sizeof(T), n, f) == n;
}

// transform.lua: rotation = {roll, pitch, yaw}, translation zero
dliom::Rigid3d Rotation(double roll, double pitch, double yaw) {
  dliom::Rigid3d r;
  const std::array<double, 4> q = dliom::transform::RollPitchYaw(roll, pitch, yaw);
  for (int i = 0; i < 4; ++i) r.q[i] = q[i];
  return r;
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
    m.frame_id = k % 2 == 0 ? "horizontal_vlp16_link" : "vertical_vlp16_link";
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
    const double kVoxelSize = 5e-2;
    const Rigid3d xy = Rotation(0., -M_PI / 2., 0.), xz = Rotation(0., 0., -M_PI / 2), yz = Rotation(0., 0., M_PI);
    const std::string dir = std::string(argv[2]) + "/";
    std::vector<std::pair<std::string, std::unique_ptr<io::XRayPointsProcessor>>> xrays;
    auto add_xray = [&](const std::string& name, const Rigid3d& transform) {
      xrays.emplace_back(name, std::make_unique<io::XRayPointsProcessor>(&writer, kVoxelSize, transform, dir + name));
    };
    add_xray("xray_yz_all", yz);
    add_xray("xray_xy_all", xy);
    add_xray("xray_xz_all", xz);
    io::ColoringPointsProcessor horizontal(&writer, {255, 0, 0}, "horizontal_vlp16_link");
    io::ColoringPointsProcessor vertical(&writer, {0, 255, 0}, "vertical_vlp16_link");
    add_xray("xray_yz_all_color", yz);
    add_xray("xray_xy_all_color", xy);
    add_xray("xray_xz_all_color", xz);
    int64_t num_points = 0;
    for (;;) {
      num_points += (int64_t)writer.Process(messages).size();
      if (writer.Flush() == io::FlushResult::kFinished) break;
    }
    std::printf("points %lld\n", (long long)num_points);
    for (const auto& x : xrays) {
      x.second->Flush();
      int width = 0, height = 0;
      writer.XRayImage(x.second->stage(), &width, &height);
      std::printf("%s %d %d\n", x.first.c_str(), width, height);
    }
    return 0;
  } catch (const Error& e) {
    std::fprintf(stderr, "dliom error %d: %s\n", e.status, e.what());
    return 2;
  }
}
