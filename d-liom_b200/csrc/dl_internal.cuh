// Internal declarations shared by the translation units of libdliom_b200.so.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <memory>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/dliom_b200.h"
#include "dl_math.cuh"

namespace dl {

constexpr int kNumSMs = 132;  // H100 SXM

// ------------------------------------------------------------------------------------------------ device grid
// Index-array form of HybridGrid's three levels (hybrid_grid.h:411-412): top cell = 64^3 voxels
// (DynamicGrid meta cell), node = 8^3 bricks (NestedGrid), brick = 8^3 uint16 voxels, z-major (FlatGrid).
// A brick is 1 KiB and 1 KiB-aligned in HBM, so a whole brick is one bulk-copy unit.
struct GridView {
  const int32_t* __restrict__ top;    // (1 << bits)^3 entries -> node index, -1 = absent
  const int32_t* __restrict__ nodes;  // num_nodes * 512 entries -> brick index, -1 = absent
  const uint16_t* __restrict__ bricks;  // num_bricks * 512 voxels
  float resolution;
  int bits;
};

// HybridGrid::value(): origin shift by grid_size/2, unsigned bounds test, three dependent reads.
__device__ __forceinline__ uint16_t grid_value(const GridView& g, int x, int y, int z) {
  const int gs = 64 << g.bits;
  const int half = gs >> 1;
  const unsigned sx = (unsigned)(x + half), sy = (unsigned)(y + half), sz = (unsigned)(z + half);
  if (sx >= (unsigned)gs || sy >= (unsigned)gs || sz >= (unsigned)gs) return 0;
  const int node = __ldg(g.top + ((((sz >> 6) << g.bits) + (sy >> 6)) << g.bits) + (sx >> 6));
  if (node < 0) return 0;
  const int brick = __ldg(g.nodes + (size_t)node * 512 + ((((sz >> 3) & 7) << 6) | (((sy >> 3) & 7) << 3) | ((sx >> 3) & 7)));
  if (brick < 0) return 0;
  return __ldg(g.bricks + (size_t)brick * 512 + (((sz & 7) << 6) | ((sy & 7) << 3) | (sx & 7)));
}

// ------------------------------------------------------------------------------------------------ owned memory
// A handle's device allocation (Pinned: page-locked host memory) and its capacity in elements, freed by the destructor.
// Structs that kernels take by value keep raw pointers, filled from these owners on the host side.
// Invariant: a buffer that work queued on the context's stream may still read or write is released or replaced only after a
// ctx->wait_stream() that covers that work. grow() waits before it frees or swaps, the destroy functions wait before they
// delete their handle, and a buffer a kernel re-lays into is move-assigned only after a wait.
template <typename T, bool Pinned = false>
struct Buffer {
  struct Free {
    void operator()(T* p) const { Pinned ? cudaFreeHost(p) : cudaFree(p); }
  };
  std::unique_ptr<T, Free> ptr;
  size_t cap = 0;
  T* get() const { return ptr.get(); }
  void reset() {
    ptr.reset();
    cap = 0;
  }
};
template <typename T>
using DeviceBuffer = Buffer<T>;
using PinnedBuffer = Buffer<uint8_t, true>;

}  // namespace dl

// ------------------------------------------------------------------------------------------------ handles
struct dl_context {
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaStream_t copy_stream = nullptr;   // uploads of host scans, overlapped with the kernels of the previous sub-batch
  cudaStream_t aux_stream = nullptr;    // odd sub-batches of the front end (see frontend_run)
  cudaStream_t tail_stream = nullptr;   // high priority: the front end's raw-IMU chain (pre-integration, prediction), next to the first filter
  cudaEvent_t staging_done = nullptr;   // the pinned staging block of the previous call has been consumed
  cudaEvent_t batch_done = nullptr;     // dl_frontend_submit: everything of the batch in flight, incl. the result download
  dl::DeviceBuffer<uint8_t> d_fcsm_lut; // loop-closure search: cell value -> 8-bit precomputation value (dl_fcsm.cu), built on first use
  int in_flight = 0;                    // scans of the submitted, not yet collected batch
  bool in_flight_states = false;        // ... and whether it also stages the estimated IMU states
  dl_scan_result* staged_results = nullptr;  // where in h_pinned the in-flight batch's results land
  dl_nav_state* staged_states = nullptr;     // ... and its estimated IMU states
  std::string error;
  int64_t launches = 0;
  // growable scratch arenas (device + pinned host), reused across calls
  dl::DeviceBuffer<uint8_t> d_scratch;
  dl::PinnedBuffer h_pinned;
  // optional per-stage timing (events recorded on `stream`)
  bool profiling = false;
  struct Mark {
    int stage;
    cudaEvent_t begin, end;
  };
  std::vector<Mark> marks;
  std::vector<cudaEvent_t> event_pool;
  std::vector<std::string> stage_names;
  std::vector<double> stage_ms;
  std::vector<int64_t> stage_calls;
  int stage_id(const char* name);
  cudaEvent_t take_event();

  int fail(int status, const std::string& msg) {
    error = msg;
    return status;
  }
  int cuda_fail(cudaError_t e, const char* what) {
    error = std::string(what) + ": " + cudaGetErrorString(e);
    return DL_ERR_CUDA;
  }
  int reserve_device(size_t bytes);
  int reserve_pinned(size_t bytes);
  // Host wait for everything on `stream`. blocking_sync: the thread sleeps on a cudaEventBlockingSync event instead of
  // spinning in cudaStreamSynchronize — for background threads (loop closure, pose graph) on hosts with fewer CPUs than threads.
  bool blocking_sync = false;
  cudaEvent_t sync_event = nullptr;
  cudaError_t wait_stream() {
    if (!blocking_sync) return cudaStreamSynchronize(stream);
    if (!sync_event) {
      const cudaError_t e = cudaEventCreateWithFlags(&sync_event, cudaEventBlockingSync | cudaEventDisableTiming);
      if (e != cudaSuccess) return e;
    }
    const cudaError_t e = cudaEventRecord(sync_event, stream);
    return e != cudaSuccess ? e : cudaEventSynchronize(sync_event);
  }
};

struct dl_grid {
  dl_context* ctx = nullptr;
  float resolution = 0.f;
  int bits = 1;
  // host mirror of the three levels
  std::vector<int32_t> top;                 // (1<<bits)^3
  std::vector<int32_t> nodes;               // num_nodes * 512
  std::vector<uint16_t> bricks;             // num_bricks * 512
  std::vector<uint8_t> brick_dirty;         // per brick
  bool structure_dirty = true;
  // device copies
  dl::DeviceBuffer<int32_t> d_top;
  dl::DeviceBuffer<int32_t> d_nodes;
  dl::DeviceBuffer<uint16_t> d_bricks;
  dl::DeviceBuffer<int32_t> d_counters;  // [0] nodes in use, [1] bricks in use, [2] scratch (update-list length)
  bool mirror_stale = false;      // the device copy was modified by dl_grid_insert_range_data: the host mirror is behind
  uint64_t version = 1;           // bumped by every modification (cells set, sync, device insert)
  // loop-closure search index (dl_fcsm.cu), built on first use and rebuilt when `version` moved on
  dl::DeviceBuffer<uint8_t> d_m8;
  uint64_t m8_version = 0;        // 0 = none
  int m8_org[3] = {0, 0, 0}, m8_dim[3] = {0, 0, 0};
  std::mutex index_mutex;
  dl::GridView view() const { return {d_top.get(), d_nodes.get(), d_bricks.get(), resolution, bits}; }
};

#define DL_CUDA(ctx, call)                                  \
  do {                                                      \
    cudaError_t e__ = (call);                               \
    if (e__ != cudaSuccess) return (ctx)->cuda_fail(e__, #call); \
  } while (0)

#define DL_TRY(expr)                \
  do {                              \
    const int st__ = (expr);        \
    if (st__ != DL_OK) return st__; \
  } while (0)

// Host helpers and types that several units of the library share. Hidden, so that like file-local code they bind inside the
// library and stay out of its exported symbols.
#define DL_SHARED __attribute__((visibility("hidden")))

#define DL_LAUNCH_CHECK(ctx, name)                          \
  do {                                                      \
    (ctx)->launches++;                                      \
    cudaError_t e__ = cudaGetLastError();                   \
    if (e__ != cudaSuccess) return (ctx)->cuda_fail(e__, name); \
  } while (0)

namespace dl {

// Allocates `count` elements into `b`, replacing what it held (see the invariant at Buffer), and sets their bytes to `fill` on
// the context's stream unless fill < 0. On failure `b` is unchanged.
template <typename T, bool Pinned>
int alloc(dl_context* ctx, Buffer<T, Pinned>& b, size_t count, int fill = -1) {
  void* p = nullptr;
  const cudaError_t e = Pinned ? cudaMallocHost(&p, count * sizeof(T)) : cudaMalloc(&p, count * sizeof(T));
  if (e != cudaSuccess) return ctx->cuda_fail(e, Pinned ? "cudaMallocHost" : "cudaMalloc");
  Buffer<T, Pinned> fresh;
  fresh.ptr.reset(static_cast<T*>(p));
  fresh.cap = count;
  if (fill >= 0) DL_CUDA(ctx, cudaMemsetAsync(p, fill, count * sizeof(T), ctx->stream));
  b = std::move(fresh);
  return DL_OK;
}
// Replaces `b` by `want` elements (the caller decides when and by how much to grow), keeping its first `keep` elements and
// setting the others' bytes to `fill` unless fill < 0.
//   keep == 0: wait, free, allocate, so that the old and the new buffer never coexist. A failed allocation leaves `b` empty.
//   keep > 0:  allocate and fill, copy the prefix on the context's stream, wait, swap. On failure `b` is unchanged.
template <typename T, bool Pinned>
int grow(dl_context* ctx, Buffer<T, Pinned>& b, size_t want, size_t keep = 0, int fill = -1) {
  if (keep == 0) {
    if (b.get()) {
      DL_CUDA(ctx, ctx->wait_stream());
      b.reset();
    }
    return alloc(ctx, b, want, fill);
  }
  Buffer<T, Pinned> fresh;
  DL_TRY(alloc(ctx, fresh, want, fill));
  DL_CUDA(ctx, cudaMemcpyAsync(fresh.get(), b.get(), keep * sizeof(T), cudaMemcpyDeviceToDevice, ctx->stream));
  DL_CUDA(ctx, ctx->wait_stream());
  b = std::move(fresh);
  return DL_OK;
}

// Copies of `count` elements on the context's stream; the host waits for them (and everything before) with sync().
template <typename T>
int h2d(dl_context* ctx, T* dst, const T* src, size_t count) {
  if (count == 0) return DL_OK;
  DL_CUDA(ctx, cudaMemcpyAsync(dst, src, count * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
  return DL_OK;
}
template <typename T>
int d2h(dl_context* ctx, T* dst, const T* src, size_t count) {
  if (count == 0) return DL_OK;
  DL_CUDA(ctx, cudaMemcpyAsync(dst, src, count * sizeof(T), cudaMemcpyDeviceToHost, ctx->stream));
  return DL_OK;
}
inline int sync(dl_context* ctx) {
  DL_CUDA(ctx, ctx->wait_stream());
  return DL_OK;
}

// RAII stage bracket: records begin/end events on the context stream when profiling is on.
struct StageScope {
  dl_context* ctx;
  int mark = -1;
  StageScope(dl_context* c, const char* name) : ctx(c) {
    if (!c->profiling) return;
    dl_context::Mark m{c->stage_id(name), c->take_event(), c->take_event()};
    cudaEventRecord(m.begin, c->stream);
    mark = (int)c->marks.size();
    c->marks.push_back(m);
  }
  ~StageScope() {
    if (mark >= 0) cudaEventRecord(ctx->marks[mark].end, ctx->stream);
  }
};

struct Arena {  // bump allocator over the context's device scratch; with a null base it only counts (`off` = bytes taken)
  char* base;
  size_t off = 0;
  explicit Arena(void* p) : base((char*)p) {}
  template <typename T>
  T* take(size_t count) {
    off = (off + 255) & ~size_t(255);
    T* p = base ? (T*)(base + off) : nullptr;
    off += count * sizeof(T);
    return p;
  }
};
// Reserves the device scratch of one call and carves it. `carve(Arena&)` makes only takes (no copies, launches or other side
// effects): it runs once on a counting arena, the reservation is what that took plus `extra` bytes for takes whose sizes are
// not known before the call's device work, and it runs again on the scratch. `rest`, if given, continues after the carve.
template <typename Carve>
int carve_scratch(dl_context* ctx, Carve&& carve, size_t extra = 0, Arena* rest = nullptr) {
  Arena count(nullptr);
  carve(count);
  const int st = ctx->reserve_device(count.off + extra);
  if (st != DL_OK) return st;
  Arena a(ctx->d_scratch.get());
  carve(a);
  if (rest) *rest = a;
  return DL_OK;
}

// ---- kernel launchers (each defined in its own .cu), all asynchronous on `stream`, device pointers only.

// dl_voxel.cu: the smallest power of two >= v, at least 64 (the capacity of a voxel filter's hash table)
DL_SHARED int64_t next_pow2(int64_t v);

struct AdaptiveParams {
  float max_length, min_num_points, max_range;
};
// One CTA per (cloud, filter) pair: adaptive bisection entirely on the device.
// filters: num_filters parameter blocks; outputs indexed [(b * num_filters + f) * cap ...].
int launch_adaptive_voxel_filter(dl_context* ctx, const float* points, int stride, int64_t cap, const int32_t* counts,
                                 int batch, const AdaptiveParams* filters_dev, int num_filters, uint32_t* table,
                                 int64_t table_cap, uint32_t* scratch /* pairs * 2 * cap */, int32_t* keep, int32_t* keep_counts,
                                 float* passes /* (batch*num_filters) * 32 */, int32_t* num_passes,
                                 int32_t* cropped_counts /* optional, batch*num_filters */);

struct RtcsmScan {  // one scan of a batched correlative search (dl_rtcsm.cu), device pointers
  GridView grid;        // the grid this scan is scored against
  const float* points;  // n x 3
  int32_t n;
  const Quatf* cand_q;  // R rotations (composed with the initial pose, normalised)
  const Vec3f* cand_t;  // L translations (composed with the initial pose)
  const double* pen_r;  // R: angle * rotation_delta_cost_weight
  const double* pen_t;  // L: |t| * translation_delta_cost_weight
  int32_t R, L;
  float* scores;                     // optional, R * L
  unsigned long long* best;          // (score bits << 32) | ~index, zeroed before the launch
  int32_t* nonpositive;              // optional, zeroed before the launch: set to 1 when a candidate's score is not > 0
};
// dl_rtcsm.cu: the host part of the batched correlative search, shared by dl_rtcsm_match and the front end's pre-match
DL_SHARED Quatf angle_axis_to_quat(const Vec3f& aa);
struct DL_SHARED RtcsmTables {
  int linear = 0, angular = 0;
  float step = 0.f;
  std::vector<Quatf> cand_q;
  std::vector<Vec3f> cand_t;
  std::vector<double> pen_r, pen_t;
};
// One batched correlative search. Clouds are on the device: cloud k = points[k] with counts[k] rows (host-known). The tables
// of every scan (R rotations, L translations, their penalties) are built on the host with the reference's float operations
// — the angular window depends on each cloud's farthest point through acosf, which must be the host's to stay bit-exact —
// and go up in ONE copy; one launch scores all (scan, rotation, translation) candidates.
struct DL_SHARED RtcsmBatchItem {
  const dl_grid* grid;  // the grid this scan is scored against; every grid of a batch has the plan's resolution
  const float* d_points;
  int64_t n;
  Rigidd initial;
  float max_scan_range;
  float* d_scores;          // optional
  int32_t* d_nonpositive;   // optional: set to 1 when a candidate's score is not > 0
};
// plan_rtcsm_batch builds the tables and lays out the one upload (every scan's tables, the descriptors, the CTA prefix); take()
// carves that upload and the argmax words, so a caller can count the scratch before it reserves it; run_rtcsm_batch uploads
// and launches.
struct DL_SHARED RtcsmBatchPlan {
  std::vector<RtcsmTables> tables;
  std::vector<size_t> off_q, off_t, off_pr, off_pt;
  std::vector<int32_t> prefix;
  size_t off_scans = 0, off_prefix = 0, blob = 0;
  unsigned char* d_blob = nullptr;
  RtcsmScan* d_scans = nullptr;
  unsigned long long* d_best = nullptr;
  void take(Arena& a) {
    d_blob = a.take<unsigned char>(blob);
    d_best = a.take<unsigned long long>(tables.size());
    d_scans = (RtcsmScan*)(d_blob + off_scans);
  }
};
DL_SHARED int plan_rtcsm_batch(dl_context* ctx, const dl_rtcsm_options& opt, float resolution,
                               const std::vector<RtcsmBatchItem>& items, RtcsmBatchPlan* plan);
DL_SHARED int run_rtcsm_batch(dl_context* ctx, const std::vector<RtcsmBatchItem>& items, const RtcsmBatchPlan& plan);
DL_SHARED size_t rtcsm_scratch_bound(const dl_rtcsm_options& opt, float resolution, float max_range);
int launch_rtcsm_pick(dl_context* ctx, const RtcsmScan* scans_dev, int num_scans, double* pose_out, const int32_t* pose_slot,
                      float* score_out, const int32_t* score_slot);
int launch_max_range_batch(dl_context* ctx, const float* points, int64_t stride_floats, const int32_t* counts, int count_stride,
                           int batch, float init, float* out);

// ---- NLS
struct NlsProblem {  // one scan-to-submap registration problem, device pointers
  const float* cloud[DL_MAX_PAIRS];
  int32_t count[DL_MAX_PAIRS];
  const int32_t* count_dev[DL_MAX_PAIRS];  // optional: read the count from device memory instead
  GridView grid[DL_MAX_PAIRS];
  double target_t[3];
  double initial[7];
  const double* initial_dev;  // optional: 7 doubles on the device override `initial` (and target_t = its translation
                              // unless target_dev is set)
  const double* target_dev;
  const int32_t* enabled_dev;  // optional: the problem is skipped (output untouched) when *enabled_dev == 0
};
struct NlsOptions {
  int num_pairs;
  double occ_weight[DL_MAX_PAIRS];
  double trans_weight, rot_weight;
  int only_yaw, nonmono, max_iter;
  int cluster;  // CTAs per problem (thread-block cluster; 0 / 1 = one CTA): > 1 for clouds of tens of thousands of points, see dl_nls.cu
};
struct NlsOutput {
  double pose[7];
  dl_solve_summary summary;
};
int launch_nls(dl_context* ctx, const NlsOptions& opt, const NlsProblem* problems_dev, int count, NlsOutput* out_dev);
// dl_nls.cu: the checks of a dl_ceres_options block for `num_pairs` (cloud, grid) pairs, and the kernels' form of it
DL_SHARED int check_ceres_options(dl_context* ctx, const dl_ceres_options* o, int num_pairs);
DL_SHARED NlsOptions to_nls_options(const dl_ceres_options& o, int num_pairs);
struct FusedOutput {
  double state[16];  // p(3) q(4 wxyz) v(3) ba(3) bg(3)
  dl_solve_summary summary;
};
// IMU term of the fused solve in the SUBMAP frame (built on the host by build_imu_term or on the device by imu_prepare_kernel):
// state i (fixed), the pre-integrated deltas, gravity, and W = weight^2 * Sigma^-1 (row-major 15x15, order p, theta, v, ba, bg).
// dp, dq, dv carry the bias correction of imu_term_deltas: the residual reads conj(dq) as the inverse of the corrected delta_q.
struct ImuTerm {
  double pi[3], qi[4], vi[3], bai[3], bgi[3];
  double dp[3], dq[4], dv[3];
  double G[3];
  double sum_dt;
  double W[225];
};
constexpr int kImuTermDoubles = 16 + 10 + 3 + 1 + 225;
static_assert(sizeof(ImuTerm) == kImuTermDoubles * sizeof(double), "ImuTerm layout");

// State i's biases and the pre-integrated deltas of its factor, with the first-order bias correction of
// integration_base.h:283-290 folded in once per scan (dba = ba_i - linearized_ba, dbg = bg_i - linearized_bg):
//   dp + J_p,ba dba + J_p,bg dbg,   dv + J_v,ba dba + J_v,bg dbg,   c = delta_q (x) (1, 1/2 J_q,bg dbg).
// dq holds c / |c|^2, so that its conjugate is Eigen's c.inverse() (the corrected quaternion is not unit). Sums run left to
// right, like the window smoother's copy of this residual (dl_window.cu). Biases equal to the linearisation point leave the
// raw deltas, bit for bit. Host (build_imu_term) and device (imu_prepare_kernel).
DL_HD void imu_term_deltas(const dl_preintegration& m, const double* ba_i, const double* bg_i, ImuTerm* t) {
  double dba[3], dbg[3];
  bool at_linearisation = true;
  for (int k = 0; k < 3; ++k) {
    t->bai[k] = ba_i[k]; t->bgi[k] = bg_i[k];
    t->dp[k] = m.delta_p[k]; t->dv[k] = m.delta_v[k];
    dba[k] = ba_i[k] - m.linearized_ba[k];
    dbg[k] = bg_i[k] - m.linearized_bg[k];
    at_linearisation = at_linearisation && dba[k] == 0.0 && dbg[k] == 0.0;
  }
  for (int k = 0; k < 4; ++k) t->dq[k] = m.delta_q[k];
  if (at_linearisation) return;
  const double* J = m.jacobian;
  auto blk = [&](int r, int c, const double* d) {  // row r of the 3x3 block at (r, c) times d
    return J[r * 15 + c] * d[0] + J[r * 15 + c + 1] * d[1] + J[r * 15 + c + 2] * d[2];
  };
  double th[3];
  for (int k = 0; k < 3; ++k) {
    t->dp[k] = m.delta_p[k] + blk(k, 9, dba) + blk(k, 12, dbg);
    t->dv[k] = m.delta_v[k] + blk(6 + k, 9, dba) + blk(6 + k, 12, dbg);
    th[k] = blk(3 + k, 12, dbg);
  }
  const Quatd c = qmul(Quatd{m.delta_q[0], m.delta_q[1], m.delta_q[2], m.delta_q[3]}, Quatd{1.0, 0.5 * th[0], 0.5 * th[1], 0.5 * th[2]});
  const double n2 = (c.x * c.x + c.y * c.y) + (c.z * c.z + c.w * c.w);
  t->dq[0] = c.w / n2; t->dq[1] = c.x / n2; t->dq[2] = c.y / n2; t->dq[3] = c.z / n2;
}
// dl_imu.cu: one pre-integration factor in the submap frame and the initial 16-vector of state j. False if the covariance is
// not positive definite.
DL_SHARED bool build_imu_term(const Rigidd& to_submap, const dl_nav_state& si, const dl_nav_state& sj, const dl_preintegration& m,
                              const double* gravity, double imu_weight, ImuTerm* t, double* x16);
int launch_nls_fused(dl_context* ctx, const NlsOptions& opt, const NlsProblem* problems_dev, const ImuTerm* imu_terms_dev,
                     const double* initial16_dev, int count, FusedOutput* out_dev);
// The fused solve's IMU normal equations of each prepared factor at x16_dev (16 doubles per factor, submap frame), into
// kImuFactorOutDoubles doubles per factor: residual (15), H (225, row-major), g (15), r^T W r. Factors with ok == 0 are skipped.
constexpr int kImuFactorOutDoubles = 15 + 225 + 15 + 1;
int launch_imu_factor_evaluate(dl_context* ctx, int count, const ImuTerm* terms_dev, const int32_t* ok_dev, const double* x16_dev,
                               double* out_dev);
int launch_imu_preintegrate(dl_context* ctx, int count, const int32_t* offsets, const double* dts, const double* accs,
                            const double* gyrs, const double* biases, int bias_stride, const dl_imu_noise& noise,
                            dl_preintegration* out);
struct DecodeArgs {  // one sensor_msgs/PointCloud2 message (dl_decode.cu)
  const uint8_t* data;
  int64_t n;
  int point_step, offset_x, offset_y, offset_z, offset_time, time_type;
  bool xyz_aligned, time_aligned;  // fields readable with aligned loads
  Rigidf sensor_to_tracking;
  int32_t* tile_counts;  // ceil(n / 256)
  float* rows_out;
  int32_t* num_out;
  double* stamp_offset;
};
struct FcsmPair {  // one (node, submap) loop-closure search, device pointers
  GridView hi, lo;
  const float* hi_pts;
  const float* lo_pts;
  int* cells;      // 3 * n_hi: full-resolution cell of every high-resolution point at the guess
  float* lo_rot;   // 3 * n_lo: rotated low-resolution points
  int n_hi, n_lo;
  Rigidf pose;     // float cast of the pose guess (cc:171-173)
  int wxy, wz;     // window half-widths in cells
  float min_score;
  double min_low;
  // search index of the high-resolution grid (dense sliding 8^3 maximum of the 8-bit values); null = exhaustive search
  const uint8_t* m8;
  int m8_org[3], m8_dim[3];
};
struct FcsmPick {
  int found;
  float score, low_resolution_score;
  int offset[3];
  long long num_candidates;
  double pose[7];  // coarse pose (the guess itself when nothing was found)
};
constexpr int kFcsmRun = 8;  // x offsets per search thread (dl_fcsm.cu)
// One RangeDataInserter3D::Insert per job (dl_inserter.cu). Device pointers; the grid's frame.
struct InsertJob {
  dl_grid* grid;
  Vec3f origin;
  const float* returns;     // n x 3
  int n;                    // the point count, or an upper bound of it when n_dev is given
  const int32_t* n_dev;     // optional: the point count on the device (a transform filter's near count)
  uint32_t* update_list;    // n * (1 + num_free) entries
};
// Runs the jobs' Inserts with one set of host steps for all of them (one bounding-box read-back, then one counter read-back
// per pool level); jobs of one grid run in list order, one after another. d_bbox: 8 ints per job; d_args:
// insert_args_bytes(count) bytes.
size_t insert_args_bytes(int jobs);
int insert_range_data_device(dl_context* ctx, const InsertJob* jobs, int count, int num_free, const uint16_t* d_hit_table,
                             const uint16_t* d_miss_table, int32_t* d_bbox, void* d_args);
struct DL_SHARED InsertScratch {
  uint16_t *hit_table, *miss_table;
  int32_t* bbox;
  void* args;
};
DL_SHARED void carve_insert(Arena& a, int jobs, InsertScratch* s);
DL_SHARED int upload_odds_tables(dl_context* ctx, const dl_range_data_inserter_options& o, const InsertScratch& s);
DL_SHARED int check_inserter(dl_context* ctx, const dl_range_data_inserter_options* o);
// TransformRangeData into the submap frame + FilterRangeDataByMaxRange (submap_3d.cc:42-51, :264-279) of one cloud per job:
// `all` receives every point, `near` (count in *near_count) those within max_range of the origin, in input order.
struct TransformJob {
  const float* in;
  int n;
  Rigidf to_submap;
  Vec3f origin_submap;
  float max_range;
  float *all, *near;
  int32_t* near_count;
  int32_t* tile_counts;     // ceil(n / 256)
};
size_t transform_jobs_bytes(int jobs);
int launch_transform_filter(dl_context* ctx, const TransformJob* jobs, int count, void* d_jobs);
// The submap-frame transform and range filter of Submap3D::InsertRangeData for one cloud (carve_transform) and its two Inserts.
struct DL_SHARED SubmapInsertScratch {
  float *all, *near;
  int32_t *near_count, *tiles;
  uint32_t *update_hi, *update_lo;
};
DL_SHARED void carve_submap_insert(Arena& a, const dl_range_data_inserter_options& o, int64_t n, SubmapInsertScratch* s);
DL_SHARED void submap_insert_jobs(dl_grid* hi, dl_grid* lo, const double* submap_local_pose, int32_t high_resolution_max_range,
                                  const float* origin, const float* d_returns, int n, const SubmapInsertScratch& s,
                                  TransformJob* transform, InsertJob* inserts);
// range_data_in_local and the histogram's gravity-aligned returns of one scan per job.
struct LocalFrameJob {
  const float *returns, *misses;   // tracking frame
  int num_returns, num_misses;
  Rigidf pose;                     // opt_pose.cast<float>()
  Rigidf gravity_alignment;        // its rotation only
  float *returns_local, *misses_local, *returns_aligned;
};
size_t local_frame_jobs_bytes(int jobs);
int launch_local_frame(dl_context* ctx, const LocalFrameJob* jobs, int count, void* d_jobs);
// dl_window.cu
constexpr int kWindowEvalDoubles = 38 + 38 * 30 + 38 * 38;  // per problem: residual, Jacobian, weight
// Device buffers of `count` window updates (carve_window) and the upload / launch / read-back of dl_window_optimize_batch on them,
// shared with the trajectory builders' batch, which carves them next to its front end's buffers.
struct DL_SHARED WindowBuffers {
  dl_nav_state *si, *init, *si_out, *sj_out;
  double *prior, *z, *info;
  dl_preintegration* pre;
  dl_solve_summary* sum;
};
DL_SHARED void carve_window(Arena& a, int count, WindowBuffers* w);
DL_SHARED int window_optimize(dl_context* ctx, const dl_window_options& options, int count, const WindowBuffers& w,
                              const dl_nav_state* states_i, const double* prior_information, const dl_preintegration* preintegrations,
                              const double* matched_poses, const dl_nav_state* initial_states_j, dl_nav_state* states_i_out,
                              dl_nav_state* states_j_out, double* information_out, dl_solve_summary* summaries);
// dl_histogram.cu
struct HistogramScratch {  // device scratch of one rotational histogram of n points
  unsigned long long* keys;
  int* slice_first;
  float* centroid;
  int* ev_bucket;
  float* ev_value;
  int* counters;
};
void carve_rotational_histogram(Arena& a, int64_t n, HistogramScratch* s);
// `count` clouds in one launch, one CTA each: cloud k = n[k] (>= 1) points at d_points[k], scratch s[k] carved for at least n[k],
// histogram k (`size` floats) at d_histograms[k]. d_args: rotational_histograms_args_bytes(count) bytes of device memory. The error
// flag of cloud k is s[k].counters[1].
size_t rotational_histograms_args_bytes(int count);
int launch_rotational_histograms(dl_context* ctx, const HistogramScratch* s, const float* const* d_points, const int64_t* n,
                                 int count, int size, float* const* d_histograms, void* d_args);
// dl_comm.cu: staging buffers of the constraint exchange and the timed all-gather
int comm_reserve(dl_comm* c, size_t bytes_per_rank);
void* comm_send_buffer(dl_comm* c);
void* comm_recv_buffer(dl_comm* c);
int comm_all_gather(dl_comm* c, const void* send_dev, void* recv_dev, size_t bytes, float* ms);
// The clouds of a batch of (node, submap) loop-closure searches. Pair k has hi_off[k+1] - hi_off[k] high-resolution points
// (likewise low). Host batch (hi_store == nullptr): they are rows [off[k], off[k+1]) of the host arrays hi_pts / lo_pts and the
// search uploads them. Device-resident (hi_store / lo_store set, dl_posegraph3d.cu's node store): they already sit on the
// device at hi_store + 3 * hi_begin[k] (lo likewise); nothing is uploaded and the host arrays are not read.
struct PairClouds {
  const float* hi_pts = nullptr;
  const float* lo_pts = nullptr;
  const int64_t* hi_off = nullptr;
  const int64_t* lo_off = nullptr;
  const float* hi_store = nullptr;
  const float* lo_store = nullptr;
  const int64_t* hi_begin = nullptr;
  const int64_t* lo_begin = nullptr;
};
// dl_fcsm.cu: the option checks of dl_constraint_search_batch (fast correlative matcher, and the refine's two-weight Ceres
// options), shared by every entry point that searches.
int check_constraint_options(dl_context* ctx, const dl_constraint_options& options);
// dl_fcsm.cu: dl_constraint_search_batch's body (coarse search, min_score prune, refine) for `count` pairs in chunks of 1024.
int constraint_search(dl_context* ctx, const dl_constraint_options& options, int count, const double* guesses,
                      const PairClouds& clouds, const dl_grid* const* hi_grids, const dl_grid* const* lo_grids,
                      dl_constraint* constraints);
// dl_api.cu: the flat index of top cell (x, y, z) in a grid's top level of 2^bits cells per axis; downloads a grid's host mirror
// where the device copy is ahead; uploads it where the device copy is behind; grows its node pool (level 0) or brick pool
// (level 1) from `used` entries in use by `add` more, keeping those in use
DL_SHARED inline size_t top_flat(int x, int y, int z, int bits) { return ((((size_t)z << bits) + y) << bits) + x; }
DL_SHARED int grid_download(dl_grid* g);
int grid_ensure_device_state(dl_grid* g);
int grid_grow_pool(dl_grid* g, int level, size_t used, size_t add);
int launch_interpolate(dl_context* ctx, const GridView& grid, int64_t n, const double* xyz, double* out);
int launch_grid_lookup(dl_context* ctx, const GridView& grid, int64_t n, const int32_t* xyz, uint16_t* out);

}  // namespace dl
