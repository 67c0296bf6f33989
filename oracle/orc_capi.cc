// TEST INFRASTRUCTURE — CPU oracle (see orc_math.h header). Flat C interface for ctypes
// (tests/, __graft_entry__.smoke(), bench.py's cpu_baseline / --impl reference only).
// Poses cross this interface as 7 doubles: t.x t.y t.z q.w q.x q.y q.z.
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <cstring>
#include <thread>

#include "orc_decode.h"
#include "orc_fcsm.h"
#include "orc_filters.h"
#include "orc_frontend.h"
#include "orc_grid.h"
#include "orc_imu.h"
#include "orc_nls.h"
#include "orc_posegraph.h"
#include "orc_rtcsm.h"
#include "orc_window.h"

using namespace orc;

namespace {
Rigid3d pose_in(const double* p) { return {{p[0], p[1], p[2]}, {p[3], p[4], p[5], p[6]}}; }
void pose_out(const Rigid3d& r, double* p) {
  p[0] = r.t.x; p[1] = r.t.y; p[2] = r.t.z; p[3] = r.q.w; p[4] = r.q.x; p[5] = r.q.y; p[6] = r.q.z;
}
}  // namespace

extern "C" {

// ---- probability tables
float orc_value_to_probability(uint16_t v) { return value_to_probability(v); }
uint16_t orc_probability_to_value(float p) { return probability_to_value(p); }
float orc_odds(float p) { return odds(p); }
void orc_lookup_table_to_apply_odds(float o, uint16_t* out) {
  const auto t = lookup_table_to_apply_odds(o);
  std::memcpy(out, t.data(), 32768 * sizeof(uint16_t));
}
void orc_value_to_probability_table(float* out65536) {
  std::memcpy(out65536, value_to_probability_table().data(), 65536 * sizeof(float));
}

// ---- grid
void* orc_grid_create(float resolution) { return new HybridGrid(resolution); }
void orc_grid_destroy(void* g) { delete (HybridGrid*)g; }
float orc_grid_resolution(void* g) { return ((HybridGrid*)g)->resolution(); }
int orc_grid_bits(void* g) { return ((HybridGrid*)g)->bits(); }
int orc_grid_set_probability(void* g, int x, int y, int z, float p) {
  try { ((HybridGrid*)g)->SetProbability({x, y, z}, p); } catch (...) { return 1; }
  return 0;
}
int orc_grid_set_value(void* g, int x, int y, int z, uint16_t v) {
  try { *((HybridGrid*)g)->mutable_value({x, y, z}) = v; } catch (...) { return 1; }
  return 0;
}
// Bulk form of orc_grid_set_value (the HybridGrid::ToProto layout: parallel x / y / z / value arrays). Returns 1 past the growth limit.
int orc_grid_set_cells(void* g, int64_t n, const int32_t* x, const int32_t* y, const int32_t* z, const uint16_t* v) {
  try {
    for (int64_t i = 0; i < n; ++i) *((HybridGrid*)g)->mutable_value({x[i], y[i], z[i]}) = v[i];
  } catch (...) { return 1; }
  return 0;
}
uint16_t orc_grid_value(void* g, int x, int y, int z) { return ((HybridGrid*)g)->value({x, y, z}); }
float orc_grid_probability(void* g, int x, int y, int z) { return ((HybridGrid*)g)->GetProbability({x, y, z}); }
void orc_grid_cell_index(void* g, const float* p, int* out) {
  const I3 i = ((HybridGrid*)g)->GetCellIndex({p[0], p[1], p[2]});
  out[0] = i.x; out[1] = i.y; out[2] = i.z;
}
void orc_grid_center_of_cell(void* g, const int* i, float* out) {
  const V3f c = ((HybridGrid*)g)->GetCenterOfCell({i[0], i[1], i[2]});
  out[0] = c.x; out[1] = c.y; out[2] = c.z;
}
int orc_grid_apply_lookup_table(void* g, int x, int y, int z, const uint16_t* table) {
  std::vector<uint16_t> t(table, table + 32768);
  return ((HybridGrid*)g)->ApplyLookupTable({x, y, z}, t) ? 1 : 0;
}
void orc_grid_finish_update(void* g) { ((HybridGrid*)g)->FinishUpdate(); }
int64_t orc_grid_num_cells(void* g) {
  int64_t n = 0;
  ((HybridGrid*)g)->ForEachCell([&](const I3&, uint16_t) { ++n; });
  return n;
}
// Parallel arrays in the reference's iteration order (the HybridGrid proto layout, hybrid_grid.h:530-542).
void orc_grid_export(void* g, int* xs, int* ys, int* zs, uint16_t* vs) {
  int64_t n = 0;
  ((HybridGrid*)g)->ForEachCell([&](const I3& i, uint16_t v) { xs[n] = i.x; ys[n] = i.y; zs[n] = i.z; vs[n] = v; ++n; });
}
// Returns 1 past the growth limit (the grid then holds whatever the Insert wrote before it stopped).
int orc_grid_insert_range_data(void* g, const float* origin, const float* returns, int64_t n, double hit_p,
                               double miss_p, int num_free) {
  RangeDataInserter ins(RangeDataInserterOptions{hit_p, miss_p, num_free});
  try { ins.Insert({origin[0], origin[1], origin[2]}, returns, n, (HybridGrid*)g); } catch (...) { return 1; }
  return 0;
}
// Submap::InsertRangeData into two caller-owned grids (which may be one grid): the transform and range filter of
// Submap3D::InsertRangeData, then Insert(near) into hi and Insert(all) into lo. Returns 1 past the growth limit.
int orc_submap_insert_range_data(void* hi, void* lo, const double* local_pose, const float* origin, const float* returns,
                                 int64_t n, double hit_p, double miss_p, int num_free, int high_resolution_max_range) {
  RangeDataInserter ins(RangeDataInserterOptions{hit_p, miss_p, num_free});
  try {
    submap_insert_range_data(pose_in(local_pose), {origin[0], origin[1], origin[2]}, returns, n, ins,
                             high_resolution_max_range, (HybridGrid*)hi, (HybridGrid*)lo);
  } catch (...) { return 1; }
  return 0;
}

// ---- interpolation
double orc_interpolate(void* g, double x, double y, double z) {
  return InterpolatedGrid(*(HybridGrid*)g).GetProbability(x, y, z);
}
// out[0] = value, out[1..3] = d/dx, d/dy, d/dz (forward-mode Jets)
void orc_interpolate_grad(void* g, double x, double y, double z, double* out) {
  const Jet r = InterpolatedGrid(*(HybridGrid*)g).GetProbability(Jet(x, 0), Jet(y, 1), Jet(z, 2));
  out[0] = r.a; out[1] = r.v[0]; out[2] = r.v[1]; out[3] = r.v[2];
}

// ---- filters
int64_t orc_voxel_filter(const float* pts, int64_t n, int stride, float resolution, int64_t* keep) {
  std::vector<int64_t> k;
  VoxelFilter(resolution).Filter(pts, n, stride, &k);
  std::memcpy(keep, k.data(), k.size() * sizeof(int64_t));
  return (int64_t)k.size();
}
void orc_voxel_indices(const float* pts, int64_t n, int stride, float resolution, int* out) {
  for (int64_t i = 0; i < n; ++i) {
    const I3 c = cell_index({pts[i * stride], pts[i * stride + 1], pts[i * stride + 2]}, resolution);
    out[3 * i] = c.x; out[3 * i + 1] = c.y; out[3 * i + 2] = c.z;
  }
}
int64_t orc_adaptive_voxel_filter(const float* pts, int64_t n, int stride, float max_length, float min_num_points,
                                  float max_range, int64_t* keep, float* passes, int* num_passes) {
  std::vector<float> p;
  const auto k = AdaptiveVoxelFilter({max_length, min_num_points, max_range}, pts, n, stride, &p);
  std::memcpy(keep, k.data(), k.size() * sizeof(int64_t));
  if (passes) std::memcpy(passes, p.data(), std::min<size_t>(p.size(), 32) * sizeof(float));
  if (num_passes) *num_passes = (int)p.size();
  return (int64_t)k.size();
}

// ---- correlative matcher
// window_out: [linear, angular]; step_out: [angular_step, max_scan_range]
float orc_rtcsm_match(void* grid, const float* pts, int64_t n, const double* initial_pose, double linear_window,
                      double angular_window, double w_t, double w_r, double* pose, int64_t* best_index,
                      int* window_out, float* step_out, float* all_scores) {
  std::vector<float> scores;
  const RtcsmResult r = rtcsm_match({linear_window, angular_window, w_t, w_r}, pose_in(initial_pose), pts, n,
                                    *(HybridGrid*)grid, all_scores ? &scores : nullptr);
  pose_out(r.pose, pose);
  if (best_index) *best_index = r.best_index;
  if (window_out) { window_out[0] = r.window.linear; window_out[1] = r.window.angular; }
  if (step_out) { step_out[0] = r.window.angular_step; step_out[1] = r.window.max_scan_range; }
  if (all_scores) std::memcpy(all_scores, scores.data(), scores.size() * sizeof(float));
  return r.score;
}

// ---- wire format -> TimedPointCloud
int64_t orc_decode_point_cloud2(int point_step, int off_x, int off_y, int off_z, int off_t, int time_type, const uint8_t* data,
                                int64_t n, const double* sensor_to_tracking, float* rows_out, double* stamp_offset) {
  return decode_point_cloud2(PointCloud2Layout{point_step, off_x, off_y, off_z, off_t, time_type}, data, n,
                             pose_in(sensor_to_tracking), rows_out, stamp_offset);
}

// ---- loop-closure coarse matcher (branch and bound)
struct OrcFcsmResult {
  int found;
  float score;
  double pose[7];
  float rotational_score, low_resolution_score;
  int offset[3];
  int reserved;
  int64_t leaves_scored;
};
static FcsmOptions fcsm_options(int depth, int full_depth, double min_rot, double min_low, double wxy, double wz) {
  FcsmOptions o;
  o.branch_and_bound_depth = depth; o.full_resolution_depth = full_depth; o.min_rotational_score = min_rot;
  o.min_low_resolution_score = min_low; o.linear_xy_search_window = wxy; o.linear_z_search_window = wz;
  return o;
}
static void fcsm_out(const FcsmResult& r, OrcFcsmResult* out) {
  std::memset(out, 0, sizeof(*out));
  out->found = r.found ? 1 : 0;
  out->score = r.score;
  pose_out(r.pose, out->pose);
  out->rotational_score = r.rotational_score;
  out->low_resolution_score = r.low_resolution_score;
  out->offset[0] = r.offset.x; out->offset[1] = r.offset.y; out->offset[2] = r.offset.z;
  out->leaves_scored = r.leaves_scored;
}
// Matcher object = what ConstraintBuilder3D keeps per finished submap (precomputation stack built once).
void* orc_fcsm_create(void* hi, void* lo, int depth, int full_depth, double min_rot, double min_low, double wxy, double wz) {
  return new FastCorrelativeScanMatcher(*(HybridGrid*)hi, (const HybridGrid*)lo, fcsm_options(depth, full_depth, min_rot, min_low, wxy, wz));
}
void orc_fcsm_destroy(void* m) { delete (FastCorrelativeScanMatcher*)m; }
void orc_fcsm_match(void* m, const double* pose_guess, const float* hi_pts, int64_t n_hi, const float* lo_pts, int64_t n_lo,
                    float min_score, OrcFcsmResult* out) {
  fcsm_out(((const FastCorrelativeScanMatcher*)m)->MatchWith3DofInitial(pose_in(pose_guess), hi_pts, n_hi, lo_pts, n_lo, min_score), out);
}
// Full Match (with the yaw search); histogram may be null (= the zero histogram of the reference's own test fixture).
void orc_fcsm_match_full(void* hi, void* lo, int depth, int full_depth, double min_rot, double min_low, double wxy, double wz,
                         double angular_window, const double* node_pose, const double* submap_pose, const float* hi_pts,
                         int64_t n_hi, const float* lo_pts, int64_t n_lo, const float* histogram, int histogram_size,
                         float min_score, OrcFcsmResult* out, int* scan_index, int* num_scans, const float* submap_histogram) {
  FcsmOptions o = fcsm_options(depth, full_depth, min_rot, min_low, wxy, wz);
  o.angular_search_window = angular_window;
  Histogram sh(histogram_size, 0.f);
  if (submap_histogram)
    for (int i = 0; i < histogram_size; ++i) sh[i] = submap_histogram[i];
  std::vector<std::pair<Histogram, float>> at_angles;
  at_angles.emplace_back(sh, 0.f);
  FastCorrelativeScanMatcher m(*(HybridGrid*)hi, (const HybridGrid*)lo, o, at_angles);
  Histogram h(histogram_size, 0.f);
  if (histogram)
    for (int i = 0; i < histogram_size; ++i) h[i] = histogram[i];
  const FcsmResult r = m.Match(pose_in(node_pose), pose_in(submap_pose), hi_pts, n_hi, lo_pts, n_lo, h, Quatd{1., 0., 0., 0.}, min_score);
  fcsm_out(r, out);
  *scan_index = r.scan_index;
  *num_scans = r.num_scans;
}
// RotationalScanMatcher: one submap histogram at angle 0, scores of `histogram` at the given angles
void orc_rotational_match(const float* submap_histogram, int size, float submap_angle, const float* histogram, float initial_angle,
                          const float* angles, int num_angles, float* scores_out) {
  std::vector<std::pair<Histogram, float>> at_angles;
  at_angles.emplace_back(Histogram(submap_histogram, submap_histogram + size), submap_angle);
  RotationalScanMatcher m(at_angles);
  const std::vector<float> s = m.Match(Histogram(histogram, histogram + size), initial_angle, std::vector<float>(angles, angles + num_angles));
  for (int i = 0; i < num_angles; ++i) scores_out[i] = s[i];
}
void orc_compute_histogram(const float* pts, int64_t n, int size, float* out) {
  const Histogram h = compute_histogram(pts, n, size);
  for (int i = 0; i < size; ++i) out[i] = h[i];
}
void orc_fcsm_match_3dof(void* hi, void* lo, int depth, int full_depth, double min_rot, double min_low, double wxy, double wz,
                         const double* pose_guess, const float* hi_pts, int64_t n_hi, const float* lo_pts, int64_t n_lo,
                         float min_score, OrcFcsmResult* out) {
  FastCorrelativeScanMatcher m(*(HybridGrid*)hi, (const HybridGrid*)lo, fcsm_options(depth, full_depth, min_rot, min_low, wxy, wz));
  fcsm_out(m.MatchWith3DofInitial(pose_in(pose_guess), hi_pts, n_hi, lo_pts, n_lo, min_score), out);
}

// ---- Ceres-equivalent matcher
struct OrcSolveSummary {
  double initial_cost, final_cost;
  int num_iterations;  // recorded iterations, including iteration 0
  int num_successful_steps, num_unsuccessful_steps, termination;
  int num_residual_evaluations, num_jacobian_evaluations;
};

static CeresMatcherOptions make_ceres_options(int n_pairs, const double* occ_w, double trans_w, double rot_w,
                                              int only_yaw, int nonmono, int max_iter) {
  CeresMatcherOptions o;
  o.occupied_space_weight.assign(occ_w, occ_w + n_pairs);
  o.translation_weight = trans_w;
  o.rotation_weight = rot_w;
  o.only_optimize_yaw = only_yaw != 0;
  o.use_nonmonotonic_steps = nonmono != 0;
  o.max_num_iterations = max_iter;
  return o;
}

void orc_ceres_match(int n_pairs, const float* const* clouds, const int64_t* sizes, void* const* grids,
                     const double* occ_w, double trans_w, double rot_w, int only_yaw, int nonmono, int max_iter,
                     const double* target_translation, const double* initial_pose, double* pose,
                     OrcSolveSummary* summary, double* iteration_costs /* >= max_iter + 1, optional */) {
  std::vector<CloudAndGrid> pairs;
  for (int i = 0; i < n_pairs; ++i) pairs.push_back({clouds[i], sizes[i], (const HybridGrid*)grids[i]});
  SolveSummary s;
  Rigid3d out;
  ceres_scan_match(make_ceres_options(n_pairs, occ_w, trans_w, rot_w, only_yaw, nonmono, max_iter),
                   {target_translation[0], target_translation[1], target_translation[2]}, pose_in(initial_pose), pairs,
                   &out, &s);
  pose_out(out, pose);
  if (summary) {
    *summary = {s.initial_cost, s.final_cost, (int)s.iterations.size(), s.num_successful_steps,
                s.num_unsuccessful_steps, s.termination, s.num_residual_evaluations, s.num_jacobian_evaluations};
  }
  if (iteration_costs)
    for (size_t i = 0; i < s.iterations.size(); ++i) iteration_costs[i] = s.iterations[i].cost;
}

// transform::GetAngle(Rigid3f::Rotation(AngleAxisVectorToRotationQuaternion(aa))) in float (transform.h:33-37, :85-99)
float orc_angle_of_angle_axis_f(const float* aa) { return rotation_angle(angle_axis_to_quat(V3f{aa[0], aa[1], aa[2]})); }

// RotationDeltaCostFunctor3D alone (rotation_delta_cost_functor_3d.h:42-53): sum of squared residuals at rotation q for a
// functor built with `scale` and `target` — the quantity the reference's own unit test checks.
double orc_rotation_delta_cost(double scale, const double* target_q, const double* q) {
  CeresMatcherOptions o;
  o.translation_weight = 0.;
  o.rotation_weight = scale;
  const Rigid3d initial{{0., 0., 0.}, {target_q[0], target_q[1], target_q[2], target_q[3]}};
  ScanMatchProblem p(o, {0., 0., 0.}, initial, {});
  const double x[7] = {0., 0., 0., q[0], q[1], q[2], q[3]};
  double r[3] = {0., 0., 0.};
  p.Evaluate(x, r, nullptr);
  return r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
}
// PrecomputeGrid chain of precomputation_grid_3d_test.cc: depth 0 = ConvertToPrecomputationGrid, depth d = PrecomputeGrid(
// previous, false, (1 << (d - 1)) * Ones): value (0..255) at the queried cells of the depth-`depth` grid.
void orc_precomputation_values(void* grid, int depth, int64_t n, const int32_t* xyz, int32_t* out) {
  std::unique_ptr<HybridGrid> g = convert_to_precomputation_grid(*(HybridGrid*)grid);
  for (int d = 1; d <= depth; ++d) {
    const int s = 1 << (d - 1);
    g = precompute_grid(*g, false, I3{s, s, s});
  }
  for (int64_t i = 0; i < n; ++i) out[i] = g->value(I3{xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]});
}

// ---- sparse pose adjustment (the fork's OptimizationProblem3D::Solve without landmarks / fixed frames)
// poses7: num_submaps + num_nodes rows (t xyz, q wxyz), in-out. constraints: per row submap index, node index; zbar 7 doubles;
// weights 2 doubles. Returns residuals at the solution when residuals_out != null (6 per constraint).
void orc_pose_graph_solve(int num_submaps, int num_nodes, double* poses7, int num_constraints, const int32_t* submap_node,
                          const double* zbar7, const double* weights2, int fix_z, int max_iter, OrcSolveSummary* summary,
                          int linear_solver) {
  std::vector<SpaConstraint> cs(num_constraints);
  for (int i = 0; i < num_constraints; ++i)
    cs[i] = {submap_node[2 * i], submap_node[2 * i + 1], pose_in(zbar7 + 7 * i), weights2[2 * i], weights2[2 * i + 1]};
  SolveSummary s;
  solve_pose_graph(num_submaps, num_nodes, poses7, cs, fix_z != 0, max_iter, &s, linear_solver ? kNormalCholesky : kDenseQr);
  if (summary)
    *summary = {s.initial_cost, s.final_cost, (int)s.iterations.size(), s.num_successful_steps, s.num_unsuccessful_steps,
                s.termination, s.num_residual_evaluations, s.num_jacobian_evaluations};
}
// One SPA residual (6) and its 6 x 14 ambient Jacobian (d / d [q_i(4) t_i(3) q_j(4) t_j(3)], row-major) for finite-difference checks
void orc_spa_residual(const double* pose_i7, const double* pose_j7, const double* zbar7, double tw, double rw, double* e6,
                      double* jac84) {
  const SpaConstraint c{0, 0, pose_in(zbar7), tw, rw};
  using J = JetN<14>;
  J qi[4], ti[3], qj[4], tj[3], e[6];
  for (int k = 0; k < 4; ++k) { qi[k] = J::variable(pose_i7[3 + k], k); qj[k] = J::variable(pose_j7[3 + k], 7 + k); }
  for (int k = 0; k < 3; ++k) { ti[k] = J::variable(pose_i7[k], 4 + k); tj[k] = J::variable(pose_j7[k], 11 + k); }
  spa_residual(c, qi, ti, qj, tj, e);
  for (int r = 0; r < 6; ++r) {
    e6[r] = e[r].a;
    for (int k = 0; k < 14; ++k) jac84[14 * r + k] = e[r].v[k];
  }
}

// Cost, local gradient (6) and local Gauss-Newton matrix J^T J (6x6 row-major) at a pose: the quantities
// the device reduction produces, for a direct kernel-level comparison.
void orc_ceres_normal_equations(int n_pairs, const float* const* clouds, const int64_t* sizes, void* const* grids,
                                const double* occ_w, double trans_w, double rot_w, const double* target_translation,
                                const double* reference_pose, const double* at_pose, double* cost, double* g6,
                                double* h36) {
  std::vector<CloudAndGrid> pairs;
  for (int i = 0; i < n_pairs; ++i) pairs.push_back({clouds[i], sizes[i], (const HybridGrid*)grids[i]});
  ScanMatchProblem problem(make_ceres_options(n_pairs, occ_w, trans_w, rot_w, 0, 0, 1),
                           {target_translation[0], target_translation[1], target_translation[2]},
                           pose_in(reference_pose), pairs);
  const int m = problem.num_residuals();
  std::vector<double> r(m), J((size_t)m * 6);
  problem.Evaluate(at_pose, r.data(), J.data());
  double c = 0;
  for (int i = 0; i < 6; ++i) g6[i] = 0;
  for (int i = 0; i < 36; ++i) h36[i] = 0;
  for (int i = 0; i < m; ++i) {
    c += r[i] * r[i];
    for (int a = 0; a < 6; ++a) {
      g6[a] += J[(size_t)i * 6 + a] * r[i];
      for (int b = 0; b < 6; ++b) h36[a * 6 + b] += J[(size_t)i * 6 + a] * J[(size_t)i * 6 + b];
    }
  }
  *cost = 0.5 * c;
}

// ---- IMU pre-integration and the fused solve (orc_imu.h). States cross as 16 doubles: p(3) q(4 wxyz) v(3) ba(3) bg(3).
struct OrcPreintegration {
  double sum_dt;
  double delta_p[3], delta_q[4], delta_v[3], ba[3], bg[3];
  double jacobian[225], covariance[225];  // row-major 15x15, order p, theta, v, ba, bg
};
static void preint_out(const Preintegration& p, OrcPreintegration* o) {
  o->sum_dt = p.sum_dt;
  o->delta_p[0] = p.delta_p.x; o->delta_p[1] = p.delta_p.y; o->delta_p[2] = p.delta_p.z;
  o->delta_q[0] = p.delta_q.w; o->delta_q[1] = p.delta_q.x; o->delta_q[2] = p.delta_q.y; o->delta_q[3] = p.delta_q.z;
  o->delta_v[0] = p.delta_v.x; o->delta_v[1] = p.delta_v.y; o->delta_v[2] = p.delta_v.z;
  o->ba[0] = p.ba.x; o->ba[1] = p.ba.y; o->ba[2] = p.ba.z;
  o->bg[0] = p.bg.x; o->bg[1] = p.bg.y; o->bg[2] = p.bg.z;
  for (int i = 0; i < 15; ++i)
    for (int j = 0; j < 15; ++j) {
      o->jacobian[i * 15 + j] = p.jacobian[i][j];
      o->covariance[i * 15 + j] = p.covariance[i][j];
    }
}
static Preintegration preint_in(const OrcPreintegration& o) {
  Preintegration p;
  p.sum_dt = o.sum_dt;
  p.delta_p = {o.delta_p[0], o.delta_p[1], o.delta_p[2]};
  p.delta_q = {o.delta_q[0], o.delta_q[1], o.delta_q[2], o.delta_q[3]};
  p.delta_v = {o.delta_v[0], o.delta_v[1], o.delta_v[2]};
  p.ba = {o.ba[0], o.ba[1], o.ba[2]};
  p.bg = {o.bg[0], o.bg[1], o.bg[2]};
  for (int i = 0; i < 15; ++i)
    for (int j = 0; j < 15; ++j) {
      p.jacobian[i][j] = o.jacobian[i * 15 + j];
      p.covariance[i][j] = o.covariance[i * 15 + j];
    }
  return p;
}

// n samples (dt, acc xyz, gyr xyz); the first only latches acc_0 / gyr_0 (integration_base.h:111-118).
void orc_imu_preintegrate(const double* noise4, const double* ba, const double* bg, int n, const double* dt,
                          const double* acc, const double* gyr, OrcPreintegration* out) {
  Preintegration p;
  preint_reset(&p, {ba[0], ba[1], ba[2]}, {bg[0], bg[1], bg[2]});
  const ImuNoise noise{noise4[0], noise4[1], noise4[2], noise4[3]};
  for (int i = 0; i < n; ++i)
    preint_push(&p, dt[i], {acc[3 * i], acc[3 * i + 1], acc[3 * i + 2]}, {gyr[3 * i], gyr[3 * i + 1], gyr[3 * i + 2]}, noise);
  preint_out(p, out);
}
void orc_imu_predict(const double* state_i, const OrcPreintegration* m, const double* G, double* state_j) {
  const NavState j = imu_predict(FusedProblem::unpack(state_i), preint_in(*m), {G[0], G[1], G[2]});
  FusedProblem::pack(j, state_j);
}
void orc_imu_residual(const double* state_i, const double* state_j, const OrcPreintegration* m, const double* G,
                      double* r15, double* J225) {
  double J[15][15];
  imu_residual(FusedProblem::unpack(state_i), FusedProblem::unpack(state_j), preint_in(*m), {G[0], G[1], G[2]}, r15,
               J225 ? J : nullptr);
  if (J225)
    for (int i = 0; i < 15; ++i)
      for (int j = 0; j < 15; ++j) J225[i * 15 + j] = J[i][j];
}
int orc_fused_match(int n_pairs, const float* const* clouds, const int64_t* sizes, void* const* grids,
                    const double* occ_w, double trans_w, double rot_w, int nonmono, int max_iter,
                    const double* target_translation, const double* state_i, const double* initial_j,
                    const OrcPreintegration* m, const double* G, double imu_weight, double* state_j,
                    OrcSolveSummary* summary) {
  std::vector<CloudAndGrid> pairs;
  for (int i = 0; i < n_pairs; ++i) pairs.push_back({clouds[i], sizes[i], (const HybridGrid*)grids[i]});
  SolveSummary s;
  NavState out;
  const bool ok = fused_scan_match(make_ceres_options(n_pairs, occ_w, trans_w, rot_w, 0, nonmono, max_iter),
                                   {target_translation[0], target_translation[1], target_translation[2]},
                                   FusedProblem::unpack(state_i), FusedProblem::unpack(initial_j), preint_in(*m),
                                   {G[0], G[1], G[2]}, imu_weight, pairs, &out, &s);
  if (!ok) return 0;
  FusedProblem::pack(out, state_j);
  if (summary)
    *summary = {s.initial_cost, s.final_cost, (int)s.iterations.size(), s.num_successful_steps,
                s.num_unsuccessful_steps, s.termination, s.num_residual_evaluations, s.num_jacobian_evaluations};
  return 1;
}

// ---- two-stage window (orc_window.h). options10: sigma_t, sigma_r, imu_weight, gravity xyz, max_iter, use_gravity, gravity_sigma;
//      directions6: gravity direction xyz, body reference direction xyz. States as 16 doubles. Returns 1 on success.
int orc_window_optimize(const double* options9, const double* directions6, const double* mean_i, const double* prior_info225,
                        const OrcPreintegration* m, const double* matched7, const double* initial_j_or_null, double* xi_out,
                        double* xj_out, double* info_out225, int* iterations, double* costs2, int* termination) {
  WindowOptions o;
  o.pose_sigma_t = options9[0]; o.pose_sigma_r = options9[1]; o.imu_weight = options9[2];
  o.gravity = {options9[3], options9[4], options9[5]};
  o.max_num_iterations = (int)options9[6]; o.use_gravity_factor = options9[7] != 0.; o.gravity_sigma = options9[8];
  o.gravity_direction = {directions6[0], directions6[1], directions6[2]};
  o.body_reference_direction = {directions6[3], directions6[4], directions6[5]};
  return window_optimize(o, mean_i, prior_info225, preint_in(*m), pose_in(matched7), initial_j_or_null, xi_out, xj_out, info_out225,
                         iterations, costs2, costs2 + 1, termination) ? 1 : 0;
}

// ---- per-scan front end
struct OrcFrontEndOptions {
  float min_range, max_range, voxel_filter_size;
  float hi_max_length, hi_min_num_points, hi_max_range;
  float lo_max_length, lo_min_num_points, lo_max_range;
  int use_rtcsm;
  double scan_period;
  double rtcsm_linear_window, rtcsm_angular_window, rtcsm_w_t, rtcsm_w_r;
  double occ_w0, occ_w1, trans_w, rot_w;
  int only_yaw, nonmono, max_iter;
};

static FrontEndOptions make_frontend(const OrcFrontEndOptions& o) {
  FrontEndOptions f;
  f.min_range = o.min_range; f.max_range = o.max_range; f.voxel_filter_size = o.voxel_filter_size;
  f.scan_period = o.scan_period;
  f.hi_filter = {o.hi_max_length, o.hi_min_num_points, o.hi_max_range};
  f.lo_filter = {o.lo_max_length, o.lo_min_num_points, o.lo_max_range};
  f.use_online_correlative_scan_matching = o.use_rtcsm != 0;
  f.rtcsm = {o.rtcsm_linear_window, o.rtcsm_angular_window, o.rtcsm_w_t, o.rtcsm_w_r};
  const double w[2] = {o.occ_w0, o.occ_w1};
  f.ceres = make_ceres_options(2, w, o.trans_w, o.rot_w, o.only_yaw, o.nonmono, o.max_iter);
  return f;
}

// Scan ingest. ranges: n rows of 8 floats (x y z t + 8 bytes origin index). Outputs sized by the caller
// (n rows each); counts returned through n_out[4] = {first_keep, returns_local, returns_tracking, misses_tracking}.
void orc_ingest_scan(const OrcFrontEndOptions* o, const void* ranges, int64_t n, const float* origins,
                     const double* prev_pose, const double* cur_pose, int64_t* first_keep, float* returns_local,
                     float* returns_tracking, float* misses_tracking, float* current_pose7f, int64_t* n_out) {
  const ScanIngest s = ingest_scan(make_frontend(*o), (const RangeMeasurement*)ranges, n, (const V3f*)origins,
                                   pose_in(prev_pose), pose_in(cur_pose));
  std::memcpy(first_keep, s.first_filter_keep.data(), s.first_filter_keep.size() * sizeof(int64_t));
  std::memcpy(returns_local, s.returns_local.data(), s.returns_local.size() * sizeof(float));
  std::memcpy(returns_tracking, s.returns_tracking.data(), s.returns_tracking.size() * sizeof(float));
  std::memcpy(misses_tracking, s.misses_tracking.data(), s.misses_tracking.size() * sizeof(float));
  const Rigid3f& c = s.current_pose;
  const float cp[7] = {c.t.x, c.t.y, c.t.z, c.q.w, c.q.x, c.q.y, c.q.z};
  std::memcpy(current_pose7f, cp, sizeof(cp));
  n_out[0] = (int64_t)s.first_filter_keep.size();
  n_out[1] = (int64_t)s.returns_local.size() / 3;
  n_out[2] = (int64_t)s.returns_tracking.size() / 3;
  n_out[3] = (int64_t)s.misses_tracking.size() / 3;
}

// Adaptive filters + (RT-CSM) + Ceres match for one scan already in the tracking frame.
// Returns 1 on success. counts[2] = {n_hi, n_lo}.
int orc_match_scan(const OrcFrontEndOptions* o, const float* returns_tracking, int64_t n, const double* pose_prediction,
                   const double* submap_local_pose, void* hi_grid, void* lo_grid, double* pose_observation_in_submap,
                   double* pose_estimate_local, OrcSolveSummary* summary, int64_t* hi_keep, int64_t* lo_keep,
                   int64_t* counts, float* rtcsm_score) {
  const ScanMatchOutput r = match_scan(make_frontend(*o), returns_tracking, n, pose_in(pose_prediction),
                                       pose_in(submap_local_pose), *(HybridGrid*)hi_grid, *(HybridGrid*)lo_grid);
  if (!r.ok) return 0;
  pose_out(r.pose_observation_in_submap, pose_observation_in_submap);
  pose_out(r.pose_estimate_local, pose_estimate_local);
  if (summary)
    *summary = {r.summary.initial_cost, r.summary.final_cost, (int)r.summary.iterations.size(),
                r.summary.num_successful_steps, r.summary.num_unsuccessful_steps, r.summary.termination,
                r.summary.num_residual_evaluations, r.summary.num_jacobian_evaluations};
  if (hi_keep) std::memcpy(hi_keep, r.hi_keep.data(), r.hi_keep.size() * sizeof(int64_t));
  if (lo_keep) std::memcpy(lo_keep, r.lo_keep.data(), r.lo_keep.size() * sizeof(int64_t));
  if (counts) { counts[0] = (int64_t)r.hi_keep.size(); counts[1] = (int64_t)r.lo_keep.size(); }
  if (rtcsm_score) *rtcsm_score = r.rtcsm_score;
  return 1;
}

}  // extern "C"

// Persistent worker pool for the CPU baseline: threads are created once and reused by every call; the scans of a batch
// are handed out one at a time from an atomic counter (a work queue), so a batch that is not a multiple of the thread
// count does not leave a strided tail. This is the loop-closure thread-pool pattern of the reference
// (C/common/thread_pool.cc:37-107) applied to independent scans.
namespace {
class WorkerPool {
 public:
  static WorkerPool& get() {
    static WorkerPool* pool = new WorkerPool;  // never destroyed: the workers sleep on its condition variable until exit
    return *pool;
  }
  // Runs f(item) for item in [0, n) on `threads` threads (the caller is one of them); returns when all are done.
  void run(int threads, int n, const std::function<void(int)>& f) {
    threads = std::max(1, std::min(threads, n));
    std::unique_lock<std::mutex> lock(mu_);
    while ((int)workers_.size() < threads - 1) workers_.emplace_back([this, id = (int)workers_.size()] { loop(id); });
    f_ = &f;
    n_ = n;
    next_.store(0);
    active_ = threads - 1;
    pending_ = threads - 1;
    ++generation_;
    lock.unlock();
    cv_.notify_all();
    drain();
    lock.lock();
    done_.wait(lock, [this] { return pending_ == 0; });
    f_ = nullptr;
  }

 private:
  void drain() {
    for (;;) {
      const int i = next_.fetch_add(1);
      if (i >= n_) break;
      (*f_)(i);
    }
  }
  void loop(int id) {
    uint64_t seen = 0;
    for (;;) {
      std::unique_lock<std::mutex> lock(mu_);
      cv_.wait(lock, [&] { return generation_ != seen; });
      seen = generation_;
      const bool mine = id < active_;
      lock.unlock();
      if (!mine) continue;
      drain();
      lock.lock();
      if (--pending_ == 0) done_.notify_all();
    }
  }
  std::mutex mu_;
  std::condition_variable cv_, done_;
  std::vector<std::thread> workers_;
  const std::function<void(int)>* f_ = nullptr;
  int n_ = 0, active_ = 0, pending_ = 0;
  uint64_t generation_ = 0;
  std::atomic<int> next_{0};
};
}  // namespace

extern "C" {

// Whole per-scan hot path (ingest + match) for a batch of independent scans on `threads` host threads:
// the CPU baseline. scans share the option block and the submap. Returns wall seconds.
double orc_frontend_batch(const OrcFrontEndOptions* o, int num_scans, const void* const* ranges, const int64_t* sizes,
                          const float* origin, const double* prev_poses, const double* cur_poses,
                          const double* submap_local_pose, void* hi_grid, void* lo_grid, int threads,
                          double* poses_out /* 7 per scan */, int* ok_out) {
  const FrontEndOptions fe = make_frontend(*o);
  const auto t0 = std::chrono::steady_clock::now();
  WorkerPool::get().run(threads, num_scans, [&](int s) {
    const ScanIngest ing = ingest_scan(fe, (const RangeMeasurement*)ranges[s], sizes[s], (const V3f*)origin,
                                       pose_in(prev_poses + 7 * s), pose_in(cur_poses + 7 * s));
    const ScanMatchOutput r =
        match_scan(fe, ing.returns_tracking.data(), (int64_t)ing.returns_tracking.size() / 3,
                   cast_d(ing.current_pose), pose_in(submap_local_pose), *(HybridGrid*)hi_grid, *(HybridGrid*)lo_grid);
    ok_out[s] = r.ok ? 1 : 0;
    if (r.ok) pose_out(r.pose_estimate_local, poses_out + 7 * s);
  });
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

// The same with the IMU in the loop (BASELINE configs[1]: 64-beam + 200 Hz IMU), restating what dl_frontend_match_batch_imu_samples
// computes: per scan, pre-integrate the samples since the previous scan (integration_base.h:109-265), predict the state
// (LTB:188-199), ingest with that prediction (LTB:393-487), adaptive filters (LTB:506-530), then the scan match with the
// pre-integration residual in the same solve (the north-star's fused form; the reference chains a GTSAM update instead).
// states: 16 doubles each, LOCAL frame. ok_out: 1, 0 (scan dropped) or -2 (no IMU factor).
double orc_frontend_batch_imu(const OrcFrontEndOptions* o, int num_scans, const void* const* ranges, const int64_t* sizes,
                              const float* origin, const double* noise4, const double* gravity, double imu_weight,
                              const double* states_i, const int32_t* offsets, const double* dt, const double* acc,
                              const double* gyr, const double* submap_local_pose, void* hi_grid, void* lo_grid, int threads,
                              double* states_out, double* predicted_out, int* ok_out, int* iterations_out) {
  const FrontEndOptions fe = make_frontend(*o);
  const ImuNoise noise{noise4[0], noise4[1], noise4[2], noise4[3]};
  const V3d G{gravity[0], gravity[1], gravity[2]};
  const Rigid3d submap = pose_in(submap_local_pose), to_submap = inverse(submap);
  const HybridGrid& hi = *(HybridGrid*)hi_grid;
  const HybridGrid& lo = *(HybridGrid*)lo_grid;
  const auto t0 = std::chrono::steady_clock::now();
  WorkerPool::get().run(threads, num_scans, [&](int s) {
    const NavState si = FusedProblem::unpack(states_i + 16 * s);
    Preintegration m;
    preint_reset(&m, si.ba, si.bg);
    for (int k = offsets[s]; k < offsets[s + 1]; ++k)
      preint_push(&m, dt[k], {acc[3 * k], acc[3 * k + 1], acc[3 * k + 2]}, {gyr[3 * k], gyr[3 * k + 1], gyr[3 * k + 2]}, noise);
    const NavState pred = imu_predict(si, m, G);
    if (predicted_out) FusedProblem::pack(pred, predicted_out + 16 * s);
    ok_out[s] = 0;
    if (iterations_out) iterations_out[s] = 0;
    const ScanIngest ing = ingest_scan(fe, (const RangeMeasurement*)ranges[s], sizes[s], (const V3f*)origin, Rigid3d{si.p, si.q},
                                       Rigid3d{pred.p, pred.q});
    const float* pts = ing.returns_tracking.data();
    const int64_t n = (int64_t)ing.returns_tracking.size() / 3;
    if (n == 0) return;
    const std::vector<int64_t> hk = AdaptiveVoxelFilter(fe.hi_filter, pts, n, 3);
    if (hk.empty()) return;
    const std::vector<int64_t> lk = AdaptiveVoxelFilter(fe.lo_filter, pts, n, 3);
    if (lk.empty()) return;
    std::vector<float> hc, lc;
    for (int64_t i : hk) hc.insert(hc.end(), pts + 3 * i, pts + 3 * i + 3);
    for (int64_t i : lk) lc.insert(lc.end(), pts + 3 * i, pts + 3 * i + 3);
    // everything the solve sees lives in the submap frame
    const Rigid3d pose_i = compose(to_submap, Rigid3d{si.p, si.q});
    const Rigid3d init_pose = compose(to_submap, cast_d(ing.current_pose));
    NavState a = si, b = pred;
    a.p = pose_i.t; a.q = pose_i.q; a.v = rotate(to_submap.q, si.v);
    b.p = init_pose.t; b.q = init_pose.q; b.v = rotate(to_submap.q, pred.v);
    NavState out;
    SolveSummary sum;
    if (!fused_scan_match(fe.ceres, init_pose.t, a, b, m, rotate(to_submap.q, G), imu_weight,
                          {{hc.data(), (int64_t)hk.size(), &hi}, {lc.data(), (int64_t)lk.size(), &lo}}, &out, &sum)) {
      ok_out[s] = -2;
      return;
    }
    const Rigid3d est = compose(submap, Rigid3d{out.p, out.q});
    out.p = est.t; out.q = est.q; out.v = rotate(submap.q, out.v);
    FusedProblem::pack(out, states_out + 16 * s);
    ok_out[s] = 1;
    if (iterations_out) iterations_out[s] = (int)sum.iterations.size();
  });
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

}  // extern "C"
