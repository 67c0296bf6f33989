// Exhaustive correlative scan matcher: the correlation-score cube, for a BATCH of scans in one launch.
//
// Replaces RealTimeCorrelativeScanMatcher3D::Match / ScoreCandidate
// (SM/real_time_correlative_scan_matcher_3d.cc:34-53, :97-113). The reference transforms the whole cloud once per
// candidate and sums nearest-voxel probabilities in float, sequentially in point order; to reproduce every score BIT FOR
// BIT each candidate is owned by one thread that walks the cloud in that order with the same float operations
// (compiled -fmad=false). Candidate = (rotation r, translation l), index l * R + r = the reference's emplace order
// (loops z,y,x,rz,ry,rx; :74-92); its pose is Rigid3f(cand_t[l], cand_q[r]), both precomputed on the host with the
// reference's float ops, so candidate * p = rotate(cand_q[r], p) + cand_t[l].
//
// Work decomposition (round 2; round 1 gave every candidate thread the full quaternion rotation of every point, K * N
// rotations, and the host synchronised three times per scan):
//   * ROTATION OUTER: rotate(cand_q[r], p) depends on r only. A warp owns (scan, r, 32 consecutive translations): its lanes
//     rotate 32 points at a time (one each) into a per-warp shared-memory strip, then every lane adds ITS translation, takes
//     the cell index and the voxel — R * N rotations instead of K * N, the same float ops in the same order.
//   * The cloud is staged into shared memory by the TMA unit: cp.async.bulk global -> shared, completion on an mbarrier,
//     two tiles in flight (the next tile streams in while the current one is scored). All warps of a CTA belong to one scan
//     and share the staged tiles.
//   * All scans of a front-end batch are scored by ONE launch: CTA -> scan through a prefix table, each scan against the grid
//     its descriptor names (the trajectory builders' batch matches every scan against its own submap); the argmax of each scan is
//     a packed 64-bit atomicMax (score bits << 32 | ~index: among equal scores the lowest index wins, the reference's strict
//     '>' in emplace order), and rtcsm_pick_kernel turns it into the matcher's initial pose on the device.
//
// Algorithmic traffic (SURVEY 8d): per rotation the cloud is read once and every (point, translation) reads one 2-byte
// voxel: R * (12 N + 2 N L) bytes per scan. The voxel reads are L1/L2 hits (a translation window touches <= 8 bricks).
#include <cstdint>
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "dl_internal.cuh"

namespace dl {
namespace {

constexpr int kWarps = 8;             // warps per CTA, each an independent (r, translation chunk) task of the CTA's scan
constexpr int kBlock = kWarps * 32;
constexpr int kTile = 512;            // points per staged tile
constexpr int kTileBytes = kTile * 12;

// ---- mbarrier + bulk-copy (TMA) primitives, sm_90+ PTX
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity)
      : "memory");
}
// global -> shared bulk copy executed by the TMA unit; `bytes` a multiple of 16, both addresses 16-byte aligned
__device__ __forceinline__ void tma_load_bulk(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

__global__ void __launch_bounds__(kBlock) rtcsm_score_kernel(const RtcsmScan* __restrict__ scans, const int32_t* __restrict__ cta_prefix,
                                                             int num_scans) {
  // two staged tiles (+16 B: the copy starts at the 16-byte boundary below the scan's first point)
  __shared__ __align__(128) unsigned char stage[2][kTileBytes + 32];
  __shared__ __align__(8) uint64_t full[2];
  __shared__ float strip[kWarps][32 * 3];

  // which scan does this CTA belong to: last s with cta_prefix[s] <= blockIdx.x
  int s = 0;
  {
    int lo = 0, hi = num_scans - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (cta_prefix[mid] <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
    }
    s = lo;
  }
  const RtcsmScan sc = scans[s];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int task = ((int)blockIdx.x - cta_prefix[s]) * kWarps + warp;   // (r, chunk) = (task / chunks, task % chunks)
  const int chunks = (sc.L + 31) >> 5;
  const bool warp_active = task < sc.R * chunks;
  const int r = warp_active ? task / chunks : 0;
  const int l = (warp_active ? task - r * chunks : 0) * 32 + lane;
  const bool active = warp_active && l < sc.L;
  const Quatf q = sc.cand_q[r];
  const Vec3f t = active ? sc.cand_t[l] : Vec3f{0.f, 0.f, 0.f};
  const CellDivider res = make_divider(sc.grid.resolution);

  // tile k of the cloud = bytes [k * kTileBytes, ...) of the scan's points, fetched from the 16-byte boundary below
  const unsigned char* src = reinterpret_cast<const unsigned char*>(sc.points);
  const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(src) & 15u);
  const long long total_bytes = (long long)sc.n * 12;
  const int tiles = (sc.n + kTile - 1) / kTile;
  auto issue = [&](int k) {
    const long long begin = (long long)k * kTileBytes;
    const uint32_t want = (uint32_t)min((long long)kTileBytes, total_bytes - begin) + mis;
    const uint32_t bytes = (want + 15u) & ~15u;
    mbar_expect_tx(&full[k & 1], bytes);
    tma_load_bulk(stage[k & 1], src + begin - mis, bytes, &full[k & 1]);
  };
  if (threadIdx.x == 0) {
    mbar_init(&full[0], 1);
    mbar_init(&full[1], 1);
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    issue(0);
    if (tiles > 1) issue(1);
  }

  float score = 0.f;
  float* my = strip[warp];
  for (int k = 0; k < tiles; ++k) {
    mbar_wait(&full[k & 1], (uint32_t)((k >> 1) & 1));
    const float* pts = reinterpret_cast<const float*>(stage[k & 1] + mis);
    const int count = min(kTile, sc.n - k * kTile);
    if (warp_active) {
      for (int base = 0; base < count; base += 32) {
        const int j = base + lane;
        if (j < count) {
          const Vec3f rp = rotate(q, Vec3f{pts[3 * j], pts[3 * j + 1], pts[3 * j + 2]});
          my[3 * lane] = rp.x; my[3 * lane + 1] = rp.y; my[3 * lane + 2] = rp.z;
        }
        __syncwarp();
        const int m = min(32, count - base);
        if (active) {
#pragma unroll 4
          for (int jj = 0; jj < m; ++jj) {
            const Vec3f w = add(Vec3f{my[3 * jj], my[3 * jj + 1], my[3 * jj + 2]}, t);
            const Int3 c = cell_index(w, res);
            score += value_to_probability(grid_value(sc.grid, c.x, c.y, c.z));
          }
        }
        __syncwarp();
      }
    }
    __syncthreads();  // every warp is done with stage[k & 1]: it can be refilled
    if (threadIdx.x == 0 && k + 2 < tiles) issue(k + 2);
  }

  unsigned long long packed = 0ull;
  if (active) {
    const long long idx = (long long)l * sc.R + r;
    score /= (float)sc.n;
    // float * double -> double; exp in double; narrowed on assignment (cc:103-110)
    const double a = sc.pen_t[l] + sc.pen_r[r];
    score = (float)((double)score * exp(-(a * a)));
    if (sc.scores) sc.scores[idx] = score;
    if (sc.nonpositive && !(score > 0.f)) *sc.nonpositive = 1;  // where the reference's CHECK_GT(score, 0.f) aborts (cc:111)
    if (score > 0.f) packed = ((unsigned long long)__float_as_uint(score) << 32) | (0xFFFFFFFFull - (unsigned long long)idx);
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    const unsigned long long o = __shfl_xor_sync(0xffffffffu, packed, d);
    packed = o > packed ? o : packed;
  }
  if (lane == 0 && packed) atomicMax(sc.best, packed);
}

// Best candidate of every scan -> pose (double, for the matcher that follows) and score. A scan without a positive score
// (the reference CHECK-fails there) keeps its initial pose and reports score 0.
__global__ void rtcsm_pick_kernel(const RtcsmScan* __restrict__ scans, int num_scans, double* __restrict__ pose_out /* 7 per scan, optional */,
                                  const int32_t* __restrict__ pose_slot, float* __restrict__ score_out, const int32_t* __restrict__ score_slot) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= num_scans) return;
  const RtcsmScan sc = scans[s];
  const unsigned long long best = *sc.best;
  float score = 0.f;
  if (best) {
    score = __uint_as_float((unsigned)(best >> 32));
    const long long idx = (long long)(0xFFFFFFFFull - (best & 0xFFFFFFFFull));
    const long long l = idx / sc.R, r = idx - l * sc.R;
    if (pose_out) pose_to7(to_double(Rigidf{sc.cand_t[l], sc.cand_q[r]}), pose_out + 7 * (size_t)pose_slot[s]);
  }
  if (score_out) score_out[score_slot[s]] = score;
}

// Farthest point of every cloud (max_scan_range of cc:63-71), clouds at a constant stride with per-cloud counts on the device.
__global__ void max_range_batch_kernel(const float* __restrict__ points, int64_t stride_floats, const int32_t* __restrict__ counts,
                                       int count_stride, float init, float* __restrict__ out) {
  const int b = blockIdx.y;
  const int n = counts[(size_t)b * count_stride];
  const float* p = points + (size_t)b * stride_floats;
  float m = 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    m = fmaxf(m, norm3(Vec3f{p[3 * i], p[3 * i + 1], p[3 * i + 2]}));
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, d));
  // non-negative floats order like their bit patterns; out[b] was preset to `init` (3 * resolution, cc:63-66)
  if ((threadIdx.x & 31) == 0) atomicMax((unsigned*)out + b, __float_as_uint(fmaxf(m, init)));
}

}  // namespace

int rtcsm_ctas_for(int64_t R, int64_t L) {
  const int64_t chunks = (L + 31) / 32;
  return (int)((R * chunks + kWarps - 1) / kWarps);
}

int launch_rtcsm_batch(dl_context* ctx, const RtcsmScan* scans_dev, const int32_t* cta_prefix_dev, int num_scans, int total_ctas) {
  if (num_scans <= 0 || total_ctas <= 0) return DL_OK;
  rtcsm_score_kernel<<<total_ctas, kBlock, 0, ctx->stream>>>(scans_dev, cta_prefix_dev, num_scans);
  DL_LAUNCH_CHECK(ctx, "rtcsm_score_kernel");
  return DL_OK;
}

int launch_rtcsm_pick(dl_context* ctx, const RtcsmScan* scans_dev, int num_scans, double* pose_out, const int32_t* pose_slot,
                      float* score_out, const int32_t* score_slot) {
  if (num_scans <= 0) return DL_OK;
  rtcsm_pick_kernel<<<(num_scans + 127) / 128, 128, 0, ctx->stream>>>(scans_dev, num_scans, pose_out, pose_slot, score_out, score_slot);
  DL_LAUNCH_CHECK(ctx, "rtcsm_pick_kernel");
  return DL_OK;
}

// out: `batch` floats. Cloud b = points + b * stride_floats with counts[b * count_stride] rows.
int launch_max_range_batch(dl_context* ctx, const float* points, int64_t stride_floats, const int32_t* counts, int count_stride,
                           int batch, float init, float* out) {
  if (batch <= 0) return DL_OK;
  DL_CUDA(ctx, cudaMemsetAsync(out, 0, sizeof(float) * batch, ctx->stream));
  max_range_batch_kernel<<<dim3(8, batch), 256, 0, ctx->stream>>>(points, stride_floats, counts, count_stride, init, out);
  DL_LAUNCH_CHECK(ctx, "max_range_batch_kernel");
  return DL_OK;
}

}  // namespace dl

// ------------------------------------------------------------------------------------------------ RT-CSM (host part)
using namespace dl;

namespace {

float rotation_angle(const Quatf& q) {  // transform.h:33-37
  return 2.f * std::atan2(norm3(Vec3f{q.x, q.y, q.z}), std::fabs(q.w));
}

// GenerateExhaustiveSearchTransforms (SM/real_time_correlative_scan_matcher_3d.cc:55-95), factored into the
// R rotations and L translations it is the outer product of, each composed with the initial pose.
void build_rtcsm_tables(const dl_rtcsm_options& opt, float resolution, float max_scan_range, const Rigidf& initial,
                        RtcsmTables* t) {
  t->linear = (int)std::lround(opt.linear_search_window / resolution);  // double / float -> double
  const float kSafetyMargin = 1.f - 1e-3f;
  t->step = kSafetyMargin * std::acos(1.f - (resolution * resolution) / (2.f * (max_scan_range * max_scan_range)));
  t->angular = (int)std::lround(opt.angular_search_window / t->step);
  const int L = t->linear, A = t->angular;
  for (int rz = -A; rz <= A; ++rz)
    for (int ry = -A; ry <= A; ++ry)
      for (int rx = -A; rx <= A; ++rx) {
        const Quatf q = angle_axis_to_quat(Vec3f{rx * t->step, ry * t->step, rz * t->step});
        t->cand_q.push_back(qnormalized(qmul(initial.q, q)));
        t->pen_r.push_back(rotation_angle(q) * opt.rotation_delta_cost_weight);
      }
  for (int z = -L; z <= L; ++z)
    for (int y = -L; y <= L; ++y)
      for (int x = -L; x <= L; ++x) {
        const Vec3f off{x * resolution, y * resolution, z * resolution};
        t->cand_t.push_back(add(rotate(initial.q, off), initial.t));
        t->pen_t.push_back(norm3(off) * opt.translation_delta_cost_weight);
      }
}

// The farthest point of a host cloud, floored at 3 * resolution (cc:63-71), with the norm the device reduction uses.
float max_scan_range_host(const float* points, int64_t n, float resolution) {
  float m = 3.f * resolution;
  for (int64_t i = 0; i < n; ++i) m = std::max(m, norm3(Vec3f{points[3 * i], points[3 * i + 1], points[3 * i + 2]}));
  return m;
}

}  // namespace

namespace dl {

// AngleAxisVectorToRotationQuaternion<float> (C/transform/transform.h:85-99): the cutoff compare and sin/cos run
// in double, results narrow to float.
Quatf angle_axis_to_quat(const Vec3f& aa) {
  float s = 0.5f, w = 1.f;
  if ((double)dot3(aa, aa) > 1e-8) {
    const float n = norm3(aa);
    s = (float)(std::sin((double)n / 2.) / (double)n);
    w = (float)std::cos((double)n / 2.);
  }
  return {w, s * aa.x, s * aa.y, s * aa.z};
}
int plan_rtcsm_batch(dl_context* ctx, const dl_rtcsm_options& opt, float resolution, const std::vector<RtcsmBatchItem>& items,
                     RtcsmBatchPlan* plan) {
  const int B = (int)items.size();
  plan->tables.assign(B, RtcsmTables{});
  plan->off_q.resize(B); plan->off_t.resize(B); plan->off_pr.resize(B); plan->off_pt.resize(B);
  plan->prefix.assign(B + 1, 0);
  auto align16 = [](size_t v) { return (v + 15) & ~size_t(15); };
  size_t blob = 0;
  for (int k = 0; k < B; ++k) {
    build_rtcsm_tables(opt, resolution, items[k].max_scan_range, to_float(items[k].initial), &plan->tables[k]);
    const RtcsmTables& t = plan->tables[k];
    const int64_t R = (int64_t)t.cand_q.size(), L = (int64_t)t.cand_t.size();
    if (R * L >= 0xFFFFFFFFll) return ctx->fail(DL_ERR_ARG, "more than 2^32-1 correlative candidates");
    plan->off_q[k] = blob; blob = align16(blob + R * sizeof(Quatf));
    plan->off_t[k] = blob; blob = align16(blob + L * sizeof(Vec3f));
    plan->off_pr[k] = blob; blob = align16(blob + R * sizeof(double));
    plan->off_pt[k] = blob; blob = align16(blob + L * sizeof(double));
    plan->prefix[k + 1] = plan->prefix[k] + rtcsm_ctas_for(R, L);
  }
  plan->off_scans = blob; blob = align16(blob + (size_t)B * sizeof(RtcsmScan));
  plan->off_prefix = blob; blob = align16(blob + (size_t)(B + 1) * sizeof(int32_t));
  plan->blob = blob;
  return DL_OK;
}
// `plan` has taken its scratch; items[k].d_points / d_scores / d_nonpositive are read here.
int run_rtcsm_batch(dl_context* ctx, const std::vector<RtcsmBatchItem>& items, const RtcsmBatchPlan& plan) {
  const int B = (int)items.size();
  if (B == 0) return DL_OK;
  std::vector<unsigned char> host(plan.blob);
  for (int k = 0; k < B; ++k) {
    const RtcsmTables& t = plan.tables[k];
    std::memcpy(host.data() + plan.off_q[k], t.cand_q.data(), t.cand_q.size() * sizeof(Quatf));
    std::memcpy(host.data() + plan.off_t[k], t.cand_t.data(), t.cand_t.size() * sizeof(Vec3f));
    std::memcpy(host.data() + plan.off_pr[k], t.pen_r.data(), t.pen_r.size() * sizeof(double));
    std::memcpy(host.data() + plan.off_pt[k], t.pen_t.data(), t.pen_t.size() * sizeof(double));
    RtcsmScan sc{};
    sc.grid = items[k].grid->view();
    sc.points = items[k].d_points;
    sc.n = (int32_t)items[k].n;
    sc.cand_q = (const Quatf*)(plan.d_blob + plan.off_q[k]);
    sc.cand_t = (const Vec3f*)(plan.d_blob + plan.off_t[k]);
    sc.pen_r = (const double*)(plan.d_blob + plan.off_pr[k]);
    sc.pen_t = (const double*)(plan.d_blob + plan.off_pt[k]);
    sc.R = (int32_t)t.cand_q.size();
    sc.L = (int32_t)t.cand_t.size();
    sc.scores = items[k].d_scores;
    sc.best = plan.d_best + k;
    sc.nonpositive = items[k].d_nonpositive;
    std::memcpy(host.data() + plan.off_scans + (size_t)k * sizeof(RtcsmScan), &sc, sizeof(sc));
  }
  std::memcpy(host.data() + plan.off_prefix, plan.prefix.data(), (size_t)(B + 1) * sizeof(int32_t));
  DL_TRY(h2d(ctx, plan.d_blob, host.data(), plan.blob));
  DL_CUDA(ctx, cudaMemsetAsync(plan.d_best, 0, sizeof(unsigned long long) * B, ctx->stream));
  DL_TRY(sync(ctx));  // `host` is pageable and local
  return launch_rtcsm_batch(ctx, plan.d_scans, (const int32_t*)(plan.d_blob + plan.off_prefix), B, plan.prefix[B]);
}

// Upper bound of the scratch one scan of the front end's correlative pre-match takes (tables, descriptor, prefix, argmax word).
// The tables' size follows from the cloud's farthest point, which a device reduction finds after the front end has carved its
// scratch, so it is bounded from the options. Every point the pre-match sees has passed the high-resolution filter's
// norm3(p) <= max_range, so max_scan_range <= max(3 * resolution, max_range). The float step does not grow with the range, so
// A is largest at that range, until the argument of acosf rounds to 1 (about 4096 resolutions): there the step is 0 and A is 0,
// and below it the step is never smaller than 0.999f * acosf(1 - 2^-24). So A is bounded by its value at max_range, or by the
// smallest positive step when max_range is past that cliff.
size_t rtcsm_scratch_bound(const dl_rtcsm_options& opt, float resolution, float max_range) {
  const int L1 = 2 * (int)std::lround(opt.linear_search_window / resolution) + 1;
  const float r = max_range > 3.f * resolution ? max_range : 3.f * resolution;
  const float kSafetyMargin = 1.f - 1e-3f;
  float step = kSafetyMargin * std::acos(1.f - (resolution * resolution) / (2.f * (r * r)));
  if (!(step > 0.f)) step = kSafetyMargin * std::acos(std::nextafter(1.f, 0.f));
  const int A1 = 2 * (int)std::lround(opt.angular_search_window / step) + 1;
  const size_t R = (size_t)A1 * A1 * A1, L = (size_t)L1 * L1 * L1;
  Arena bound(nullptr);  // the plan's takes at the largest tables, with room for the blob's 16-byte alignment
  bound.take<unsigned char>(R * 16 + L * 12 + R * 8 + L * 8 + 256 + sizeof(RtcsmScan) + 64);
  bound.take<unsigned long long>(1);
  return bound.off + 4096;
}

}  // namespace dl

extern "C" {

int dl_rtcsm_match(dl_context* ctx, const dl_rtcsm_options* options, const double* initial_pose, const float* points,
                   int64_t n, const dl_grid* grid, double* pose_out, float* score_out, dl_rtcsm_info* info,
                   float* all_scores) {
  if (!ctx || !options || !initial_pose || !grid || !pose_out || n < 0 || (n > 0 && !points)) return DL_ERR_ARG;  // CHECK_NOTNULL(pose_estimate)
  if (n == 0) return ctx->fail(DL_ERR_EMPTY, "empty point cloud");
  if (grid->structure_dirty) return ctx->fail(DL_ERR_ARG, "dl_grid_sync not called after dl_grid_set_cells");
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  // The cloud is on the host: its farthest point, hence the tables and the exact scratch, are known before the carve.
  const float max_scan_range = max_scan_range_host(points, n, grid->resolution);
  std::vector<RtcsmBatchItem> items{RtcsmBatchItem{grid, nullptr, n, pose_from7(initial_pose), max_scan_range, nullptr, nullptr}};
  RtcsmBatchPlan plan;
  DL_TRY(plan_rtcsm_batch(ctx, *options, grid->resolution, items, &plan));
  const RtcsmTables& t = plan.tables[0];
  const int64_t R = (int64_t)t.cand_q.size(), K = R * (int64_t)t.cand_t.size();
  float* d_pts;
  float* d_scores = nullptr;
  DL_TRY(carve_scratch(ctx, [&](Arena& c) {
    d_pts = c.take<float>(3 * n);
    if (all_scores) d_scores = c.take<float>(K);
    plan.take(c);
  }));
  DL_TRY(h2d(ctx, d_pts, points, 3 * n));
  items[0].d_points = d_pts;
  items[0].d_scores = d_scores;
  DL_TRY(run_rtcsm_batch(ctx, items, plan));
  unsigned long long best = 0;
  DL_TRY(d2h(ctx, &best, plan.d_best, 1));
  if (all_scores) DL_TRY(d2h(ctx, all_scores, d_scores, K));
  DL_TRY(sync(ctx));
  if (best == 0) return ctx->fail(DL_ERR_SCORE, "no candidate with a positive score (CHECK_GT(score, 0))");
  const uint32_t score_bits = (uint32_t)(best >> 32);
  const int64_t index = (int64_t)(0xFFFFFFFFull - (best & 0xFFFFFFFFull));
  float score;
  std::memcpy(&score, &score_bits, 4);
  const int64_t l = index / R, r = index - l * R;
  pose_to7(to_double(Rigidf{t.cand_t[l], t.cand_q[r]}), pose_out);
  if (score_out) *score_out = score;
  if (info) {
    info->best_index = index;
    info->num_candidates = K;
    info->linear_window = t.linear;
    info->angular_window = t.angular;
    info->angular_step = t.step;
    info->max_scan_range = max_scan_range;
  }
  return DL_OK;
}

}  // extern "C"
