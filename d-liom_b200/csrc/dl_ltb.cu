// LocalTrajectoryBuilder3D, host only: its device work runs in the batched front end (dl_frontend.cu), the window update
// (dl_window.cu), the inserter (dl_inserter.cu) and the rotational histogram (dl_histogram.cu).
//
// The per-trajectory object of the reference front end (local_trajectory_builder_3d.h:81-113) over the device path:
// AddImuData buffers the samples of the running interval, AddRangeData runs a scan through the IMU-coupled front end
// against the matching submap (active_submaps_.submaps().front(), LTB:502-505) — the scans of many builders in one batch
// (dl_ltb_add_range_data_batch; the single calls are its batch of one) — then does what AddAccumulatedRangeData /
// InsertIntoSubmap do after the match: motion filter (motion_filter.cc:37-57), insertion into both active submaps on the
// device (submap_3d.cc:264-279, :300-326 incl. the submap hand-over), rotational histogram of the inserted scan (LTB:605-610).
// Differences, all stated in the header: the fused solve replaces the match + GTSAM window (so `local_pose` is the solve's
// pose), num_accumulated_range_data = 1, a single range sensor (the synchroniser for several is the host-side
// dliom::sensor::RangeDataSynchronizer of the C++ shim), initialisation = InitializeStatic or a state given by the caller.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <functional>
#include <vector>

#include "dl_internal.cuh"
#include "dl_pipeline.cuh"

using namespace dl;

struct LtbSubmap {
  dl_grid* hi = nullptr;
  dl_grid* lo = nullptr;
  Rigidd local_pose{{0, 0, 0}, {1, 0, 0, 0}};
  int num_range_data = 0;
  int finished = 0;
  int index = 0;
};
struct dl_local_trajectory_builder {
  dl_context* ctx = nullptr;
  dl_ltb_options opt{};
  bool initialized = false;
  int accumulated_frames = 0;
  std::vector<double> init_acc, init_gyr;  // xyz per sample
  dl_nav_state prev_state{};
  double last_imu_time = -1.0;
  std::vector<double> dt, acc, gyr;        // the running interval; sample 0 is the latch
  std::vector<LtbSubmap> active, finished;
  int next_index = 0;
  int64_t motion_total = 0;
  double motion_last_time = 0;
  Rigidd motion_last_pose{{0, 0, 0}, {1, 0, 0, 0}};
  std::vector<float> clouds[4];            // returns / misses in the local frame, high / low resolution cloud in the tracking frame
  std::vector<float> histogram;
  double window_information[225];          // two-stage mode: the marginal of the previous key (prior of the next window update)
  void reset_window_information() {        // prior_pose_noise_, prior_vel_noise_, prior_bias_noise_ (LTB:84-90)
    for (double& v : window_information) v = 0.;
    const double sp = opt.prior_pose_noise > 0 ? opt.prior_pose_noise : 1e-2, sv = opt.prior_velocity_noise > 0 ? opt.prior_velocity_noise : 1e4,
                 sb = opt.prior_bias_noise > 0 ? opt.prior_bias_noise : 1e-2;
    for (int k = 0; k < 15; ++k) {
      const double s = k < 6 ? sp : (k < 9 ? sv : sb);
      window_information[k * 15 + k] = 1.0 / (s * s);
    }
  }
};

namespace {
// The empty grids of a new submap; on failure nothing is left allocated.
int ltb_make_grids(const dl_local_trajectory_builder* b, LtbSubmap* s) {
  int st = dl_grid_create(b->ctx, b->opt.high_resolution, &s->hi);
  if (st == DL_OK) st = dl_grid_create(b->ctx, b->opt.low_resolution, &s->lo);
  if (st == DL_OK) st = dl_grid_sync(s->hi);
  if (st == DL_OK) st = dl_grid_sync(s->lo);
  if (st != DL_OK) {
    dl_grid_destroy(s->hi);
    dl_grid_destroy(s->lo);
    s->hi = s->lo = nullptr;
  }
  return st;
}
// ActiveSubmaps3D::AddSubmap (submap_3d.cc:315-326) with the grids of `s` (ltb_make_grids).
void ltb_add_submap(dl_local_trajectory_builder* b, const Rigidd& pose, LtbSubmap s) {
  if (b->active.size() > 1) {
    b->active.front().finished = 1;
    b->finished.push_back(b->active.front());
    b->active.erase(b->active.begin());
  }
  s.local_pose = pose;
  s.index = b->next_index++;
  b->active.push_back(s);
}
double rotation_angle_d(const Quatd& q) {  // transform::GetAngle (transform.h:33-37)
  return 2.0 * std::atan2(std::sqrt(q.x * q.x + q.y * q.y + q.z * q.z), std::fabs(q.w));
}
// InitializeStatic after frames_for_static_initialization scans (LTB:372-381, :203-229): the mean specific force fixes roll /
// pitch, the residual of the two the accelerometer bias, the mean rate the gyroscope bias.
void ltb_initialize_static(dl_local_trajectory_builder* b) {
  if (!(b->accumulated_frames++ > b->opt.frames_for_static_initialization && !b->init_acc.empty())) return;
  const size_t m = b->init_acc.size() / 3;
  double am[3] = {0, 0, 0}, gm[3] = {0, 0, 0};
  for (size_t k = 0; k < m; ++k)
    for (int c = 0; c < 3; ++c) { am[c] += b->init_acc[3 * k + c]; gm[c] += b->init_gyr[3 * k + c]; }
  for (int c = 0; c < 3; ++c) { am[c] /= (double)m; gm[c] /= (double)m; }
  // R = FromTwoVectors(accel_mean, (0, 0, g)): the rotation taking the measured up direction to +z
  const double an = std::sqrt(am[0] * am[0] + am[1] * am[1] + am[2] * am[2]);
  Quatd q{1, 0, 0, 0};
  if (an > 0) {
    const Vec3d u{am[0] / an, am[1] / an, am[2] / an}, v{0, 0, 1};
    const double c = dot3(u, v);
    if (c > -1.0 + 1e-12) {
      const Vec3d ax = cross3(u, v);
      const double s2 = std::sqrt((1.0 + c) * 2.0);
      q = qnormalized(Quatd{s2 * 0.5, ax.x / s2, ax.y / s2, ax.z / s2});
    } else {
      q = Quatd{0, 1, 0, 0};
    }
  }
  dl_nav_state st{};
  st.q[0] = q.w; st.q[1] = q.x; st.q[2] = q.y; st.q[3] = q.z;
  const Vec3d g_body = rotate(qconj(q), Vec3d{0, 0, -b->opt.gravity});  // R^T g_vec
  st.ba[0] = g_body.x + am[0]; st.ba[1] = g_body.y + am[1]; st.ba[2] = g_body.z + am[2];
  for (int c = 0; c < 3; ++c) st.bg[c] = gm[c];
  b->prev_state = st;
  b->initialized = true;
  b->reset_window_information();
  b->init_acc.clear(); b->init_gyr.clear();
}

// The batched front end takes one options block and one IMU noise, so the members of a batch must agree on every field the
// builder reads (bit for bit; the frontend's row layout and host stride are the builder's own and always equal).
bool same_ltb_options(const dl_ltb_options& a, const dl_ltb_options& b) {
#define DL_SAME(field) (std::memcmp(&a.field, &b.field, sizeof(a.field)) == 0)
  const bool frontend = DL_SAME(frontend.min_range) && DL_SAME(frontend.max_range) && DL_SAME(frontend.voxel_filter_size) &&
      DL_SAME(frontend.high_resolution_adaptive_voxel_filter) && DL_SAME(frontend.low_resolution_adaptive_voxel_filter) &&
      DL_SAME(frontend.use_online_correlative_scan_matching) && DL_SAME(frontend.range_row_floats) &&
      DL_SAME(frontend.scan_period) && DL_SAME(frontend.real_time_correlative_scan_matcher) &&
      DL_SAME(frontend.ceres_scan_matcher.num_occupied_space_weights) && DL_SAME(frontend.ceres_scan_matcher.occupied_space_weight) &&
      DL_SAME(frontend.ceres_scan_matcher.translation_weight) && DL_SAME(frontend.ceres_scan_matcher.rotation_weight) &&
      DL_SAME(frontend.ceres_scan_matcher.only_optimize_yaw) && DL_SAME(frontend.ceres_scan_matcher.use_nonmonotonic_steps) &&
      DL_SAME(frontend.ceres_scan_matcher.max_num_iterations) && DL_SAME(frontend.host_scan_stride_rows);
  return frontend && DL_SAME(imu_noise) && DL_SAME(imu_weight) && DL_SAME(gravity) && DL_SAME(high_resolution) &&
         DL_SAME(low_resolution) && DL_SAME(num_range_data) && DL_SAME(high_resolution_max_range) &&
         DL_SAME(range_data_inserter.hit_probability) && DL_SAME(range_data_inserter.miss_probability) &&
         DL_SAME(range_data_inserter.num_free_space_voxels) && DL_SAME(motion_filter_max_time_seconds) &&
         DL_SAME(motion_filter_max_distance_meters) && DL_SAME(motion_filter_max_angle_radians) &&
         DL_SAME(rotational_histogram_size) && DL_SAME(frames_for_static_initialization) && DL_SAME(two_stage) &&
         DL_SAME(ceres_pose_noise_t) && DL_SAME(ceres_pose_noise_r) && DL_SAME(prior_pose_noise) &&
         DL_SAME(prior_velocity_noise) && DL_SAME(prior_bias_noise);
#undef DL_SAME
}

// One member of dl_ltb_add_range_data_batch: what the device work found for it and what its builder takes over at the commit.
struct LtbMember {
  dl_local_trajectory_builder* b = nullptr;
  const dl_ltb_batch_item* item = nullptr;
  int slot = -1;                       // its scan in the front-end batch; -1: an early return applies
  dl_matching_result out{};
  dl_preintegration m{};               // two-stage mode: the interval's pre-integration and the predicted state
  dl_nav_state pred{};
  dl_nav_state state{};                // the node's state (has_result)
  bool window_reset = false;           // two-stage: FailureDetection fell back and re-seeds the carried information
  std::vector<double> window_information;
  bool motion_filtered = false;
  Rigidd opt_pose{{0, 0, 0}, {1, 0, 0, 0}};
  std::vector<float> clouds[4];
  std::vector<float> histogram;
  bool hands_over = false;             // this insert completes the newest submap: `next` holds the grids of the one it adds
  LtbSubmap next;
};

// The builder takes over what the device work found for its member (the single call's tail, LTB:553-622). Cannot fail: the
// grids of a hand-over were made beforehand.
void ltb_commit(dl_local_trajectory_builder* b, LtbMember& m, double time) {
  if (m.out.scan.ok != 1) return;  // dropped like the reference's nullptr (LTB:497-534); the interval keeps integrating
  if (b->opt.two_stage) {
    if (m.window_reset) b->reset_window_information();
    else std::memcpy(b->window_information, m.window_information.data(), sizeof(b->window_information));
  }
  // the estimate becomes the previous state; the last sample of the interval latches the next one
  b->prev_state = m.state;
  {
    const size_t last = b->dt.size() - 1;
    const double ldt = b->dt[last];
    const double la[3] = {b->acc[3 * last], b->acc[3 * last + 1], b->acc[3 * last + 2]};
    const double lg[3] = {b->gyr[3 * last], b->gyr[3 * last + 1], b->gyr[3 * last + 2]};
    b->dt.assign(1, ldt);
    b->acc.assign(la, la + 3);
    b->gyr.assign(lg, lg + 3);
  }
  for (int c = 0; c < 4; ++c) b->clouds[c].swap(m.clouds[c]);
  ++b->motion_total;
  if (m.motion_filtered) return;  // insertion_result == nullptr
  b->motion_last_time = time;
  b->motion_last_pose = m.opt_pose;
  for (LtbSubmap& sm : b->active) sm.num_range_data++;
  if (m.hands_over)  // ActiveSubmaps3D::InsertRangeData (submap_3d.cc:300-313)
    ltb_add_submap(b, Rigidd{{(double)m.out.origin_in_local[0], (double)m.out.origin_in_local[1], (double)m.out.origin_in_local[2]},
                             m.opt_pose.q}, m.next);
  b->histogram.swap(m.histogram);
}

// The device work of a batch: the front end over every participating member's scan, each against its own matching submap, then
// (two-stage) the window update of all of them, the local frame and the histogram input, insertion into every inserted member's
// active submaps and their histograms. The host waits a fixed number of times, whatever the number of members, except once for
// each grid pool or top level that has to grow.
int ltb_batch_device(dl_context* ctx, const dl_ltb_options& opt, bool two_stage, const double* gravity, std::vector<LtbMember>& ms,
                     const std::vector<int>& part) {
  const int P = (int)part.size();
  // ---- the scans' rows: one layout for the batch (4-float rows become RangeMeasurement rows of origin index 0 when mixed)
  bool mixed = false;
  for (int i : part) mixed = mixed || ms[i].item->row_floats != ms[part[0]].item->row_floats;
  const int rf = mixed ? 8 : ms[part[0]].item->row_floats;
  std::vector<std::vector<float>> widened(P);
  std::vector<const void*> ranges(P);
  std::vector<int64_t> sizes(P);
  std::vector<int32_t> origin_base(P);
  std::vector<float> origins;
  for (int s = 0; s < P; ++s) {
    const dl_ltb_batch_item& it = *ms[part[s]].item;
    ranges[s] = it.rows;
    sizes[s] = it.n;
    origin_base[s] = (int32_t)(origins.size() / 3);
    origins.insert(origins.end(), it.origins, it.origins + 3 * (size_t)it.num_origins);
    if (it.row_floats != rf) {
      std::vector<float>& w = widened[s];
      w.assign((size_t)it.n * 8, 0.f);
      for (int64_t r = 0; r < it.n; ++r) std::memcpy(&w[8 * r], (const float*)it.rows + 4 * r, 4 * sizeof(float));
      ranges[s] = w.data();
    }
  }
  // ---- matching submaps (active_submaps_.submaps().front(), LTB:502-505)
  std::vector<double> submap_poses(7 * (size_t)P);
  std::vector<const dl_grid*> his(P), los(P);
  for (int s = 0; s < P; ++s) {
    const LtbSubmap& matching = ms[part[s]].b->active.front();
    pose_to7(matching.local_pose, submap_poses.data() + 7 * s);
    his[s] = matching.hi;
    los[s] = matching.lo;
  }
  SubmapSet submaps;
  submaps.poses = submap_poses.data();
  submaps.hi = his.data();
  submaps.lo = los.data();
  submaps.per_scan = true;
  // ---- the IMU intervals, concatenated
  std::vector<int32_t> offsets(P + 1, 0);
  std::vector<double> dt, acc, gyr;
  std::vector<dl_nav_state> states_i(P);
  for (int s = 0; s < P; ++s) {
    const dl_local_trajectory_builder* b = ms[part[s]].b;
    dt.insert(dt.end(), b->dt.begin(), b->dt.end());
    acc.insert(acc.end(), b->acc.begin(), b->acc.end());
    gyr.insert(gyr.end(), b->gyr.begin(), b->gyr.end());
    offsets[s + 1] = (int32_t)dt.size();
    states_i[s] = b->prev_state;
  }
  dl_frontend_options fo = opt.frontend;
  fo.range_row_floats = rf;
  dl_frontend_imu_samples imu{};
  imu.noise = opt.imu_noise;
  imu.imu_weight = opt.imu_weight;
  imu.gravity[0] = gravity[0]; imu.gravity[1] = gravity[1]; imu.gravity[2] = gravity[2];
  imu.states_i = states_i.data();
  imu.offsets = offsets.data();
  imu.dt = dt.data(); imu.acc = acc.data(); imu.gyr = gyr.data();
  std::vector<double> prev7, pred7;
  if (two_stage) {
    // the reference's chain: predict (AddImuData, LTB:188-199) -> plain match from the prediction (LTB:535-542) -> window (LTB:555)
    std::vector<double> bias(6 * (size_t)P);
    for (int s = 0; s < P; ++s)
      for (int c = 0; c < 3; ++c) { bias[6 * s + c] = states_i[s].ba[c]; bias[6 * s + 3 + c] = states_i[s].bg[c]; }
    std::vector<dl_preintegration> pre(P);
    DL_TRY(dl_imu_preintegrate(ctx, &opt.imu_noise, P, offsets.data(), dt.data(), acc.data(), gyr.data(), bias.data(), pre.data()));
    prev7.resize(7 * (size_t)P);
    pred7.resize(7 * (size_t)P);
    for (int s = 0; s < P; ++s) {
      LtbMember& m = ms[part[s]];
      m.m = pre[s];
      DL_TRY(dl_imu_predict(&states_i[s], &m.m, imu.gravity, &m.pred));
      for (int k = 0; k < 3; ++k) { prev7[7 * s + k] = states_i[s].p[k]; pred7[7 * s + k] = m.pred.p[k]; }
      for (int k = 0; k < 4; ++k) { prev7[7 * s + 3 + k] = states_i[s].q[k]; pred7[7 * s + 3 + k] = m.pred.q[k]; }
    }
  } else {
    DL_TRY(check_imu_samples(ctx, &fo, &imu, P));
  }
  // ---- scratch of everything after the front end, carved into the front end's reservation: its tracking-frame clouds stay
  //      valid until insertion and the histograms have read them. Sizes are the scans' row counts (bounds of every cloud).
  const dl_range_data_inserter_options& io = opt.range_data_inserter;
  const int H = opt.rotational_histogram_size;
  struct Slot {
    float *returns_local, *misses_local, *aligned, *histogram;
    HistogramScratch hs;
    SubmapInsertScratch ins[2];
  };
  std::vector<Slot> slots(P);
  InsertScratch is;
  void *d_local_jobs, *d_transform_jobs, *d_hist_args;
  int32_t* d_hist_err;
  float* d_gather;
  size_t gather_floats = 0;
  for (int s = 0; s < P; ++s) gather_floats += 12 * (size_t)sizes[s] + (size_t)H;
  WindowBuffers w{};
  const std::function<void(Arena&)> more = [&](Arena& a) {
    for (int s = 0; s < P; ++s) {
      const int64_t n = sizes[s];
      Slot& sl = slots[s];
      sl.returns_local = a.take<float>(3 * (size_t)n);
      sl.misses_local = a.take<float>(3 * (size_t)n);
      sl.aligned = a.take<float>(3 * (size_t)n);
      sl.histogram = a.take<float>((size_t)H);
      carve_rotational_histogram(a, n, &sl.hs);
      for (int k = 0; k < (int)ms[part[s]].b->active.size() && k < 2; ++k) carve_submap_insert(a, io, n, &sl.ins[k]);
    }
    carve_insert(a, 4 * P, &is);
    d_local_jobs = a.take<char>(local_frame_jobs_bytes(P));
    d_transform_jobs = a.take<char>(transform_jobs_bytes(2 * P));
    d_hist_args = a.take<char>(rotational_histograms_args_bytes(P));
    d_hist_err = a.take<int32_t>((size_t)P);
    d_gather = a.take<float>(gather_floats);
    if (two_stage) carve_window(a, P, &w);
  };
  // ---- the front end: every scan against its own matching submap
  dl_scan_result* d_results = nullptr;
  FrontendBuffers f;
  ImuRun run;
  run.samples = &imu;
  DL_TRY(frontend_enqueue(ctx, &fo, P, FrontendScans{ranges.data()}, sizes.data(), origins.data(), (int)(origins.size() / 3),
                          two_stage ? prev7.data() : nullptr, two_stage ? pred7.data() : nullptr, submaps, &d_results,
                          two_stage ? nullptr : &run, &f, origin_base.data(), &more));
  std::vector<dl_scan_result> r(P);
  std::vector<dl_nav_state> fused_states(P);
  std::vector<float> cur7(7 * (size_t)P);
  std::vector<int32_t> nonpositive(fo.use_online_correlative_scan_matching ? P : 0, 0);
  DL_TRY(d2h(ctx, r.data(), d_results, P));
  if (!two_stage) DL_TRY(d2h(ctx, fused_states.data(), run.d_states, P));
  DL_TRY(d2h(ctx, cur7.data(), f.current_pose, 7 * (size_t)P));
  DL_TRY(d2h(ctx, nonpositive.data(), f.rtcsm_nonpositive, nonpositive.size()));
  DL_TRY(sync(ctx));
  // The reference CHECK-fails on a pre-match candidate whose score is not > 0 (real_time_correlative_scan_matcher_3d.cc:111).
  // The pre-match runs before the insertion, so no grid has changed yet: the call fails and no builder is committed.
  for (int32_t flag : nonpositive)
    if (flag) return ctx->fail(DL_ERR_SCORE, "a correlative pre-match candidate scored <= 0 (CHECK_GT(score, 0))");
  std::vector<int> ok;  // slots whose scan was matched (scan.ok == 1)
  for (int s = 0; s < P; ++s) {
    LtbMember& m = ms[part[s]];
    m.out.scan = r[s];
    if (r[s].ok == 1) ok.push_back(s);
    if (!two_stage) m.state = fused_states[s];
  }
  if (ok.empty()) return DL_OK;
  if (two_stage) {
    // WindowOptimize(pose_estimate) (LTB:555): the matched pose is a prior on the new key next to the IMU factor and the carried
    // marginal of the previous key; one solve per member, all in one launch (dl_window_optimize_batch's kernel).
    dl_window_options wo{};
    wo.pose_sigma_translation = opt.ceres_pose_noise_t > 0 ? opt.ceres_pose_noise_t : 1e-2;
    wo.pose_sigma_rotation = opt.ceres_pose_noise_r > 0 ? opt.ceres_pose_noise_r : 1e-2;
    wo.imu_weight = opt.imu_weight > 0 ? opt.imu_weight : 1.0;
    wo.gravity[2] = opt.gravity;
    wo.max_num_iterations = 10;
    const size_t n = ok.size();
    std::vector<dl_nav_state> si(n), init(n), sj(n);
    std::vector<double> prior(n * 225), z(n * 7), info(n * 225);
    std::vector<dl_preintegration> pre(n);
    std::vector<dl_solve_summary> sums(n);
    for (size_t j = 0; j < n; ++j) {
      const LtbMember& m = ms[part[ok[j]]];
      si[j] = m.b->prev_state;
      init[j] = m.pred;
      pre[j] = m.m;
      std::memcpy(prior.data() + 225 * j, m.b->window_information, 225 * sizeof(double));
      std::memcpy(z.data() + 7 * j, m.out.scan.pose_estimate_local, 7 * sizeof(double));
    }
    DL_TRY(window_optimize(ctx, wo, (int)n, w, si.data(), prior.data(), pre.data(), z.data(), init.data(), nullptr, sj.data(),
                           info.data(), sums.data()));
    for (size_t j = 0; j < n; ++j) {
      LtbMember& m = ms[part[ok[j]]];
      if (sums[j].termination == 2) {  // the reference's FailureDetection path (LTB:856-859): matched pose + predicted rest, re-seed
        m.state = m.pred;
        for (int k = 0; k < 3; ++k) m.state.p[k] = m.out.scan.pose_estimate_local[k];
        for (int k = 0; k < 4; ++k) m.state.q[k] = m.out.scan.pose_estimate_local[3 + k];
        m.window_reset = true;
      } else {
        m.state = sj[j];
        m.window_information.assign(info.data() + 225 * j, info.data() + 225 * (j + 1));
      }
    }
  }
  // ---- per matched member: the node, the motion filter, the local frame and the histogram input
  std::vector<LocalFrameJob> local_jobs;
  std::vector<int> inserted;  // slots
  for (int s : ok) {
    LtbMember& m = ms[part[s]];
    const dl_local_trajectory_builder* b = m.b;
    const dl_scan_result& rs = r[s];
    dl_matching_result& out = m.out;
    out.has_result = 1;
    out.state = m.state;
    const Rigidd opt_pose{{m.state.p[0], m.state.p[1], m.state.p[2]}, {m.state.q[0], m.state.q[1], m.state.q[2], m.state.q[3]}};
    m.opt_pose = opt_pose;
    pose_to7(opt_pose, out.local_pose);
    // filtered_range_data_in_local = TransformRangeData(filtered_range_data_in_tracking, opt_pose.cast<float>()) (LTB:559-560)
    const Rigidf opt_f = to_float(opt_pose);
    const float* c7 = cur7.data() + 7 * s;
    const Rigidf cur{{c7[0], c7[1], c7[2]}, {c7[3], c7[4], c7[5], c7[6]}};
    const Vec3f origin_tracking = apply(inverse(cur), cur.t);  // LTB:485-487: the origin back in the tracking frame
    const Vec3f origin_local = apply(opt_f, origin_tracking);
    out.origin_in_local[0] = origin_local.x; out.origin_in_local[1] = origin_local.y; out.origin_in_local[2] = origin_local.z;
    out.num_returns = rs.num_returns; out.num_misses = rs.num_misses;
    out.num_high_resolution = rs.num_high_resolution; out.num_low_resolution = rs.num_low_resolution;
    // MotionFilter::IsSimilar (motion_filter.cc:37-57), against the builder's memory before this scan
    m.motion_filtered = b->motion_total + 1 > 1 && m.item->time - b->motion_last_time <= opt.motion_filter_max_time_seconds &&
        norm3(sub(opt_pose.t, b->motion_last_pose.t)) <= opt.motion_filter_max_distance_meters &&
        rotation_angle_d(compose(inverse(opt_pose), b->motion_last_pose).q) <= opt.motion_filter_max_angle_radians;
    const Slot& sl = slots[s];
    const Quatf gq{(float)opt_pose.q.w, (float)opt_pose.q.x, (float)opt_pose.q.y, (float)opt_pose.q.z};
    local_jobs.push_back(LocalFrameJob{f.returns_tracking + (size_t)s * f.cap * 3, f.misses_tracking + (size_t)s * f.cap * 3,
                                       rs.num_returns, rs.num_misses, opt_f, Rigidf{{0.f, 0.f, 0.f}, gq}, sl.returns_local,
                                       sl.misses_local, sl.aligned});
    if (m.motion_filtered) continue;
    // InsertIntoSubmap (LTB:584-622): the insertion submaps are queried BEFORE the insert
    out.num_insertion_submaps = (int32_t)b->active.size();
    for (size_t k = 0; k < b->active.size() && k < 2; ++k) out.insertion_submap_index[k] = b->active[k].index;
    out.inserted = 1;
    inserted.push_back(s);
  }
  DL_TRY(launch_local_frame(ctx, local_jobs.data(), (int)local_jobs.size(), d_local_jobs));
  // ---- ComputeHistogram(TransformPointCloud(returns in tracking, Rotation(gravity_alignment.cast<float>())), size): one launch,
  //      before the insertion, so that a cloud the histogram refuses fails the call while every grid is still untouched
  std::vector<HistogramScratch> hs;
  std::vector<const float*> hpts;
  std::vector<int64_t> hn;
  std::vector<float*> hout;
  for (int s : inserted) {
    if (r[s].num_returns > (1 << 20)) return ctx->fail(DL_ERR_ARG, "more than 2^20 points in a rotational histogram");
    hs.push_back(slots[s].hs);
    hpts.push_back(slots[s].aligned);
    hn.push_back(r[s].num_returns);
    hout.push_back(slots[s].histogram);
  }
  DL_TRY(launch_rotational_histograms(ctx, hs.data(), hpts.data(), hn.data(), (int)hs.size(), H, hout.data(), d_hist_args));
  if (!inserted.empty()) {  // the error flags, gathered on the device: one read-back
    for (size_t j = 0; j < inserted.size(); ++j)
      DL_CUDA(ctx, cudaMemcpyAsync(d_hist_err + j, hs[j].counters + 1, sizeof(int32_t), cudaMemcpyDeviceToDevice, ctx->stream));
    std::vector<int32_t> hist_err(inserted.size(), 0);
    DL_TRY(d2h(ctx, hist_err.data(), d_hist_err, hist_err.size()));
    DL_TRY(sync(ctx));
    for (int32_t e : hist_err)
      if (e) return ctx->fail(DL_ERR_ARG, "a point lies outside +-2^19 slices of 0.2 m");
  }
  // ---- insertion into both active submaps of every inserted member at both resolutions (Submap3D::InsertRangeData): no grid
  //      appears twice (distinct builders, distinct submaps), so all jobs run side by side
  std::vector<TransformJob> transforms;
  std::vector<InsertJob> inserts;
  for (int s : inserted) {
    const LtbMember& m = ms[part[s]];
    int k = 0;
    for (const LtbSubmap& sm : m.b->active) {
      double sp[7];
      pose_to7(sm.local_pose, sp);
      TransformJob t;
      InsertJob ij[2];
      submap_insert_jobs(sm.hi, sm.lo, sp, opt.high_resolution_max_range, m.out.origin_in_local, slots[s].returns_local,
                         m.out.num_returns, slots[s].ins[k++], &t, ij);
      transforms.push_back(t);
      inserts.insert(inserts.end(), ij, ij + 2);
    }
  }
  if (!inserts.empty()) {
    DL_TRY(launch_transform_filter(ctx, transforms.data(), (int)transforms.size(), d_transform_jobs));
    DL_TRY(upload_odds_tables(ctx, io, is));
    DL_TRY(insert_range_data_device(ctx, inserts.data(), (int)inserts.size(), io.num_free_space_voxels, is.hit_table, is.miss_table,
                                    is.bbox, is.args));
  }
  // ---- the nodes' clouds and the histograms, gathered on the device and read back in one copy
  struct Piece {
    std::vector<float>* dst;
    const float* src;
  };
  std::vector<Piece> pieces;
  for (int s : ok) {
    LtbMember& m = ms[part[s]];
    const Slot& sl = slots[s];
    const int32_t counts[4] = {r[s].num_returns, r[s].num_misses, r[s].num_high_resolution, r[s].num_low_resolution};
    const float* src[4] = {sl.returns_local, sl.misses_local, f.clouds + (size_t)(2 * s) * f.cap * 3,
                           f.clouds + (size_t)(2 * s + 1) * f.cap * 3};
    for (int c = 0; c < 4; ++c) {
      m.clouds[c].resize((size_t)counts[c] * 3);
      pieces.push_back(Piece{&m.clouds[c], src[c]});
    }
  }
  for (int s : inserted) {
    LtbMember& m = ms[part[s]];
    m.histogram.assign(H, 0.f);
    pieces.push_back(Piece{&m.histogram, slots[s].histogram});
  }
  size_t at = 0;
  for (const Piece& p : pieces) {
    if (!p.dst->empty())
      DL_CUDA(ctx, cudaMemcpyAsync(d_gather + at, p.src, p.dst->size() * sizeof(float), cudaMemcpyDeviceToDevice, ctx->stream));
    at += p.dst->size();
  }
  std::vector<float> gathered(at);
  DL_TRY(d2h(ctx, gathered.data(), d_gather, at));
  DL_TRY(sync(ctx));
  at = 0;
  for (const Piece& p : pieces) {
    if (!p.dst->empty()) std::memcpy(p.dst->data(), gathered.data() + at, p.dst->size() * sizeof(float));
    at += p.dst->size();
  }
  return DL_OK;
}
}  // namespace

extern "C" {

int dl_ltb_create(dl_context* ctx, const dl_ltb_options* options, dl_local_trajectory_builder** out) {
  if (!ctx || !options || !out) return DL_ERR_ARG;
  if (!(options->high_resolution > 0.f) || !(options->low_resolution > 0.f) || options->num_range_data < 1 ||
      options->rotational_histogram_size < 1 || options->rotational_histogram_size > 1024)
    return ctx->fail(DL_ERR_ARG, "dl_ltb_options: resolutions, num_range_data or rotational_histogram_size out of range");
  DL_TRY(check_ceres_options(ctx, &options->frontend.ceres_scan_matcher, 2));
  DL_TRY(check_inserter(ctx, &options->range_data_inserter));
  if (!options->two_stage) DL_TRY(check_imu_options(ctx, &options->frontend));  // the two-stage chain's plain solve takes only_optimize_yaw
  dl_local_trajectory_builder* b = new dl_local_trajectory_builder;
  b->ctx = ctx;
  b->opt = *options;
  b->opt.frontend.range_row_floats = 4;
  b->opt.frontend.host_scan_stride_rows = 0;
  // "We always want to have at least one submap ... create it at the origin" (submap_3d.cc:286-295)
  LtbSubmap first;
  const int st = ltb_make_grids(b, &first);
  if (st != DL_OK) {
    delete b;
    return st;
  }
  ltb_add_submap(b, Rigidd{{0, 0, 0}, {1, 0, 0, 0}}, first);
  *out = b;
  return DL_OK;
}

void dl_ltb_destroy(dl_local_trajectory_builder* b) {
  if (!b) return;
  for (auto* list : {&b->active, &b->finished})
    for (LtbSubmap& s : *list) {
      dl_grid_destroy(s.hi);
      dl_grid_destroy(s.lo);
    }
  delete b;
}

int dl_ltb_set_initial_state(dl_local_trajectory_builder* b, const dl_nav_state* state) {
  if (!b || !state) return DL_ERR_ARG;
  b->prev_state = *state;
  b->initialized = true;
  b->dt.clear(); b->acc.clear(); b->gyr.clear();
  b->reset_window_information();
  return DL_OK;
}

int dl_ltb_add_imu_data(dl_local_trajectory_builder* b, double time, const double* linear_acceleration, const double* angular_velocity) {
  if (!b || !linear_acceleration || !angular_velocity) return DL_ERR_ARG;
  if (!b->initialized) {  // init_imu_buffer_opt_ (LTB:165-176)
    b->init_acc.insert(b->init_acc.end(), linear_acceleration, linear_acceleration + 3);
    b->init_gyr.insert(b->init_gyr.end(), angular_velocity, angular_velocity + 3);
    return DL_OK;
  }
  const double dt = b->last_imu_time < 0 ? 1.0 / 500.0 : time - b->last_imu_time;  // LTB:183-185
  b->last_imu_time = time;
  b->dt.push_back(dt);
  b->acc.insert(b->acc.end(), linear_acceleration, linear_acceleration + 3);
  b->gyr.insert(b->gyr.end(), angular_velocity, angular_velocity + 3);
  return DL_OK;
}

int dl_ltb_add_range_data(dl_local_trajectory_builder* b, double time, const float* xyzt, int64_t n, const float* origin,
                          dl_matching_result* out) {
  return dl_ltb_add_synchronized_range_data(b, time, xyzt, n, 4, origin, 1, out);
}

int dl_ltb_add_synchronized_range_data(dl_local_trajectory_builder* b, double time, const void* rows, int64_t n, int32_t row_floats,
                                       const float* origin, int32_t num_origins, dl_matching_result* out) {
  if (!b) return DL_ERR_ARG;
  const dl_ltb_batch_item item{b, time, rows, n, row_floats, num_origins, origin};
  return dl_ltb_add_range_data_batch(1, &item, out);
}

int dl_ltb_add_range_data_batch(int32_t count, const dl_ltb_batch_item* items, dl_matching_result* results) {
  if (count < 0) return DL_ERR_ARG;
  if (count == 0) return DL_OK;
  if (!items || !results) return DL_ERR_ARG;
  // ---- validation: nothing is touched before every member has passed
  dl_context* ctx = items[0].builder ? items[0].builder->ctx : nullptr;
  for (int k = 0; k < count; ++k) {
    const dl_ltb_batch_item& it = items[k];
    dl_local_trajectory_builder* b = it.builder;
    if (!b || it.n < 0 || it.n > 0x3fffffff || (it.n > 0 && !it.rows) || !it.origins || it.num_origins < 1 ||
        (it.row_floats != 4 && it.row_floats != 8))
      return DL_ERR_ARG;
    if (it.row_floats == 4 && it.num_origins != 1) return b->ctx->fail(DL_ERR_ARG, "x y z t rows carry no origin index: one origin only");
    if (b->ctx != ctx) return b->ctx->fail(DL_ERR_ARG, "the builders of a batch must share one dl_context");
    for (int j = 0; j < k; ++j)
      if (items[j].builder == b) return ctx->fail(DL_ERR_ARG, "a builder appears twice in one batch");
    if (!same_ltb_options(b->opt, items[0].builder->opt))
      return ctx->fail(DL_ERR_ARG, "the builders of a batch must have equal dl_ltb_options");
  }
  const dl_ltb_options& opt = items[0].builder->opt;
  const bool two_stage = opt.two_stage != 0;
  const double gravity[3] = {0, 0, opt.gravity};
  // ---- who takes part in the device work: the members none of the single call's early returns applies to
  std::vector<LtbMember> ms(count);
  std::vector<int> part;  // members with a front-end scan, in batch order
  for (int k = 0; k < count; ++k) {
    LtbMember& m = ms[k];
    m.b = items[k].builder;
    m.item = &items[k];
    std::memset(&m.out, 0, sizeof(m.out));
    m.out.time = items[k].time;
    // "Range data collator filling buffer" (LTB:366-369); initialising (LTB:372-381); predicted_states_.empty(): no IMU since
    // the last scan (LTB:426)
    if (items[k].n == 0 || !m.b->initialized || m.b->dt.size() < 2) continue;
    m.slot = (int)part.size();
    part.push_back(k);
  }
  const int P = (int)part.size();
  if (P > 0) DL_TRY(ltb_batch_device(ctx, opt, two_stage, gravity, ms, part));
  // ---- the grids of the submaps this call hands over to, made before any builder changes: the commit below cannot fail
  for (LtbMember& m : ms) {
    if (m.slot < 0 || !m.out.inserted || m.b->active.back().num_range_data + 1 != opt.num_range_data) continue;
    const int st = ltb_make_grids(m.b, &m.next);
    if (st != DL_OK) {
      for (LtbMember& o : ms)
        if (o.hands_over) {
          dl_grid_destroy(o.next.hi);
          dl_grid_destroy(o.next.lo);
        }
      return st;
    }
    m.hands_over = true;
  }
  // ---- commit: every builder's host state, now that the device work has succeeded
  for (int k = 0; k < count; ++k) {
    LtbMember& m = ms[k];
    dl_local_trajectory_builder* b = m.b;
    if (items[k].n > 0 && !b->initialized) ltb_initialize_static(b);
    if (m.slot >= 0) ltb_commit(b, m, items[k].time);
    results[k] = m.out;
  }
  return DL_OK;
}

int dl_ltb_get_cloud(const dl_local_trajectory_builder* b, int32_t which, float* out, int64_t capacity_points, int64_t* num_points) {
  if (!b || which < 0 || which > 3 || !num_points) return DL_ERR_ARG;
  const std::vector<float>& c = b->clouds[which];
  *num_points = (int64_t)c.size() / 3;
  if (out && capacity_points >= *num_points) std::memcpy(out, c.data(), c.size() * sizeof(float));
  return DL_OK;
}

int dl_ltb_get_histogram(const dl_local_trajectory_builder* b, float* out, int32_t capacity) {
  if (!b || !out || capacity < (int32_t)b->histogram.size()) return DL_ERR_ARG;
  std::memcpy(out, b->histogram.data(), b->histogram.size() * sizeof(float));
  return DL_OK;
}

int32_t dl_ltb_num_submaps(const dl_local_trajectory_builder* b) { return b ? (int32_t)(b->finished.size() + b->active.size()) : 0; }

int dl_ltb_get_submap(dl_local_trajectory_builder* b, int32_t index, dl_grid** high_resolution_grid, dl_grid** low_resolution_grid,
                      double* local_pose, int32_t* num_range_data, int32_t* finished) {
  if (!b) return DL_ERR_ARG;
  for (auto* list : {&b->finished, &b->active})
    for (LtbSubmap& s : *list)
      if (s.index == index) {
        if (high_resolution_grid) *high_resolution_grid = s.hi;
        if (low_resolution_grid) *low_resolution_grid = s.lo;
        if (local_pose) pose_to7(s.local_pose, local_pose);
        if (num_range_data) *num_range_data = s.num_range_data;
        if (finished) *finished = s.finished;
        return DL_OK;
      }
  return b->ctx->fail(DL_ERR_ARG, "no submap with this index");
}

int dl_ltb_release_submap(dl_local_trajectory_builder* b, int32_t index) {
  if (!b) return DL_ERR_ARG;
  for (LtbSubmap& s : b->finished)
    if (s.index == index) {
      if (!s.hi) return b->ctx->fail(DL_ERR_ARG, "the submap's grids were already released");
      dl_grid_destroy(s.hi);
      dl_grid_destroy(s.lo);
      s.hi = s.lo = nullptr;
      return DL_OK;
    }
  for (const LtbSubmap& s : b->active)
    if (s.index == index) return b->ctx->fail(DL_ERR_ARG, "an active submap cannot be released");
  return b->ctx->fail(DL_ERR_ARG, "no submap with this index");
}

int dl_ltb_get_state(const dl_local_trajectory_builder* b, dl_nav_state* state, int32_t* initialized) {
  if (!b) return DL_ERR_ARG;
  if (state) *state = b->prev_state;
  if (initialized) *initialized = b->initialized ? 1 : 0;
  return DL_OK;
}

}  // extern "C"
