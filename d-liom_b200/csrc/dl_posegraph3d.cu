// mapping::PoseGraph3D on the fork's live loop-closure path (C/mapping/internal/3d/pose_graph_3d.cc,
// C/mapping/internal/constraints/constraint_builder_3d.cc:162-333): id bookkeeping, InitializeGlobalSubmapPoses, INTRA_SUBMAP
// constraints, the fan-out of the host's submap matches into (node, submap) searches, the optimization trigger and
// RunOptimization's update. The graph bookkeeping is host code (a few hundred bytes per node); the node clouds live in a device
// node store, uploaded once per node, and every search reads them there through dl::constraint_search — the kernels of
// dl_constraint_search_batch. The optimization calls dl_pose_graph_solve_sparse on the graph's poses: that call is the block-sparse
// solve's one host entry (it takes host poses, sets up the CSR lists and runs the LM state machine on the host), and the poses
// it moves are 56 bytes per submap or node, so there is no second copy of its set-up here. Pure localization adds trimming
// (TrimmingHandle::MarkSubmapAsTrimmed, :1002-1058, and PureLocalizationTrimmer, C/mapping/pose_graph_trimmer.cc:24-45),
// FinishTrajectory (:535-547) and SetInitialTrajectoryPose (:849-876); a trimmed node's clouds become dead ranges of the
// node store, and pg3d_store_compact copies the live ones into a fresh store once the dead outweigh them. The range-data map
// (dl_range_data_map_set_node, dl_range_data_map) keeps a node's range_data_in_local returns in the same store and
// emits them at the optimized node poses with one launch of pg3d_range_data_map. See include/dliom_b200.h.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <map>
#include <set>
#include <utility>
#include <vector>

#include "dl_internal.cuh"
#include "dl_pipeline.cuh"

using namespace dl;

namespace {

struct Submap {
  const dl_grid* hi = nullptr;
  const dl_grid* lo = nullptr;
  Rigidd local;
  bool finished = false;
  std::vector<int32_t> node_ids;  // InternalSubmapData::node_ids: nodes of this trajectory inserted into it, in id order
  Rigidd global;                  // optimization_problem_->submap_data()
  bool optimized = false;         // present in global_submap_poses_ (the result of the last RunOptimization) ...
  Rigidd optimized_global;        // ... with this pose
};
struct Node {
  double time = 0.0;
  Rigidd local;
  Rigidd global;          // trajectory_nodes_' global_pose
  Rigidd problem_global;  // optimization_problem_->node_data()
  int64_t hi_begin = 0, n_hi = 0, lo_begin = 0, n_lo = 0;  // points in the node store
  bool has_range_data = false;    // dl_range_data_map_set_node was called: n_rd returns at rd_begin in the node store
  int64_t rd_begin = 0, n_rd = 0;
};
struct Trajectory {
  // MapById (C/mapping/id.h): indices in order; a trimmed index is a hole
  std::map<int32_t, Submap> submaps;
  std::map<int32_t, Node> nodes;
  int32_t num_submaps = 0, num_nodes = 0;  // indices handed out so far: the index of the next append
  // Trim of the highest index forbids later appends (id.h:289-300). The ban outlives the last element: a trajectory whose
  // every submap was trimmed takes no new nodes.
  bool submaps_can_append = true, nodes_can_append = true;
};
using Id = std::pair<int32_t, int32_t>;  // (trajectory_id, index)
struct InitialTrajectoryPose {  // PoseGraph3D::InitialTrajectoryPose
  int32_t to_trajectory_id;
  Rigidd relative_pose;
  double time;
};
struct StoreSegment {  // one live node's clouds (high- then low-resolution xyz floats), or its returns, in the old and the fresh store
  int64_t src, dst, floats;
};
// One node of a range-data map: its returns in the store, its rows of the output and the two transforms of
// pb_range_data_to_ros_cloud_main.cc:155-176, local_pose.cast<float>().inverse() and global_pose.cast<float>().
struct RangeDataMapNode {
  int64_t src, dst, count;  // store point, first output point, points (> 0)
  Rigidf local_inverse, global;
};
constexpr int64_t kMinDeadFloats = (int64_t)1 << 20;  // compaction waits for at least this many dead floats (4 MiB)
constexpr int kCompactBlock = 256;

// One block per live node: its contiguous segment is copied with consecutive threads on consecutive floats (coalesced).
__global__ void __launch_bounds__(kCompactBlock) pg3d_store_compact(const float* __restrict__ src, float* __restrict__ dst,
                                                                    const StoreSegment* __restrict__ segments) {
  const StoreSegment s = segments[blockIdx.x];
  for (int64_t i = threadIdx.x; i < s.floats; i += kCompactBlock) dst[s.dst + i] = src[s.src + i];
}

constexpr int kMapBlock = 256;
constexpr int kMapTile = 1024;  // output points per CTA: 12 KiB of xyz, staged in shared memory

// The last node in [lo, hi] whose first output point is <= p (every node of the table has points, so `dst` increases).
__device__ __forceinline__ int map_node_of(const RangeDataMapNode* __restrict__ nodes, int lo, int hi, int64_t p) {
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (nodes[mid].dst <= p) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// One CTA per kMapTile output points. Each point is read from the store (consecutive threads, consecutive points) and moved
// by two separate Rigid3f * Vector3f products, tp = L^-1 * p and then G * tp, as the tool does; folding them into one composed
// transform would change the bits. The tile's xyz rows are staged in shared memory and written out as float4 when the output
// is 16-byte aligned.
__global__ void __launch_bounds__(kMapBlock) pg3d_range_data_map(const float* __restrict__ store,
                                                                 const RangeDataMapNode* __restrict__ nodes, int num_nodes,
                                                                 int64_t total, float* __restrict__ out) {
  __shared__ __align__(16) float tile[3 * kMapTile];
  __shared__ int range[2];
  const int64_t first = (int64_t)blockIdx.x * kMapTile;
  const int n = (int)min((int64_t)kMapTile, total - first);
  if (threadIdx.x < 2) range[threadIdx.x] = map_node_of(nodes, 0, num_nodes - 1, first + (threadIdx.x ? n - 1 : 0));
  __syncthreads();
  for (int k = threadIdx.x; k < n; k += kMapBlock) {
    const int64_t p = first + k;
    const RangeDataMapNode& node = nodes[map_node_of(nodes, range[0], range[1], p)];
    const float* s = store + 3 * (node.src + (p - node.dst));
    const Vec3f tp = apply(node.local_inverse, Vec3f{s[0], s[1], s[2]});
    const Vec3f gp = apply(node.global, tp);
    tile[3 * k] = gp.x;
    tile[3 * k + 1] = gp.y;
    tile[3 * k + 2] = gp.z;
  }
  __syncthreads();
  float* o = out + 3 * first;
  if (n == kMapTile && ((uintptr_t)out & 15) == 0) {  // 3 * kMapTile floats from a multiple of 4 floats: whole float4s
    const float4* t4 = reinterpret_cast<const float4*>(tile);
    float4* o4 = reinterpret_cast<float4*>(o);
    for (int j = threadIdx.x; j < 3 * kMapTile / 4; j += kMapBlock) o4[j] = t4[j];
  } else {
    for (int j = threadIdx.x; j < 3 * n; j += kMapBlock) o[j] = tile[j];
  }
}

double ms_since(std::chrono::steady_clock::time_point t0) {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}
Rigidd identity() { return {{0.0, 0.0, 0.0}, {1.0, 0.0, 0.0, 0.0}}; }
Rigidd rotation_only(const Quatd& q) { return {{0.0, 0.0, 0.0}, q}; }
// Eigen::AngleAxis(angle, UnitZ) as a quaternion
Quatd yaw_quaternion(double angle) { return {std::cos(0.5 * angle), 0.0, 0.0, std::sin(0.5 * angle)}; }
// transform::GetYaw: atan2 of the rotated x axis
double get_yaw(const Quatd& q) {
  const Vec3d d = rotate(q, Vec3d{1.0, 0.0, 0.0});
  return std::atan2(d.y, d.x);
}
// The rotation-only gravity alignment of a submap pose with its yaw removed (constraint_builder_3d.cc:241-251):
// Embed3D(Rigid2d::Rotation(-yaw)) * Rigid3d::Rotation(rotation).
Rigidd yaw_free_alignment(const Rigidd& submap_pose) {
  const Rigidd aligned = rotation_only(submap_pose.q);
  return compose(rotation_only(yaw_quaternion(-get_yaw(aligned.q))), aligned);
}

}  // namespace

struct dl_pose_graph_3d {
  dl_context* ctx = nullptr;
  dl_pose_graph_3d_options options{};
  std::map<int32_t, Trajectory> trajectories;
  std::set<int32_t> frozen;
  std::vector<dl_pg3d_constraint> constraints;           // constraints_
  std::vector<dl_pg3d_constraint> pending;               // found by the searches, not yet handed to the optimization
  std::map<Id, std::set<Id>> computed;                   // ConstraintBuilder3D::computed_constraints_: submap -> nodes
  int32_t num_nodes_since_last_loop_closure = 0;
  std::vector<dl_pg3d_search> last_searches;             // of the last add_node call
  DeviceBuffer<float> d_store;                           // node store: xyz floats, each node's high- then low-resolution cloud
  int64_t store_used = 0;                                // in floats
  int64_t store_live = 0;                                // floats of the nodes still in the graph; the rest of store_used is dead
  int64_t bytes_uploaded = 0;
  std::set<int32_t> finished_trajectories;               // finished_trajectories_
  std::map<int32_t, InitialTrajectoryPose> initial_poses;  // initial_trajectory_poses_
  struct PureLocalizationTrimmer {
    int32_t trajectory_id, num_submaps_to_keep;
  };
  std::vector<PureLocalizationTrimmer> trimmers;         // trimmers_, in the order they were added
  std::vector<dl_pg3d_submap_id> last_trimmed;

  // GetInterpolatedGlobalTrajectoryPose (:858-876): lower_bound by node time, clamped to the first and last node, else
  // transform::Interpolate of the two nodes around `time`. false: the trajectory has no nodes (the reference CHECKs).
  bool interpolated_global_pose(int32_t trajectory_id, double time, Rigidd* out) const {
    const auto it = trajectories.find(trajectory_id);
    if (it == trajectories.end() || it->second.nodes.empty()) return false;
    const std::map<int32_t, Node>& nodes = it->second.nodes;
    const auto end = std::find_if(nodes.begin(), nodes.end(), [time](const std::pair<const int32_t, Node>& n) {
      return !(n.second.time < time);
    });
    if (end == nodes.begin()) {
      *out = end->second.global;
      return true;
    }
    if (end == nodes.end()) {
      *out = std::prev(end)->second.global;
      return true;
    }
    const Node& a = std::prev(end)->second;
    const Node& b = end->second;
    const double factor = (time - a.time) / (b.time - a.time);  // timestamped_transform.cc:22-37, on the double node times
    out->t = {a.global.t.x + (b.global.t.x - a.global.t.x) * factor, a.global.t.y + (b.global.t.y - a.global.t.y) * factor,
              a.global.t.z + (b.global.t.z - a.global.t.z) * factor};
    out->q = slerp(a.global.q, b.global.q, factor, slerp_constants(a.global.q, b.global.q));
    return true;
  }
  // ComputeLocalToGlobalTransform (:914-935) over global_submap_poses_ (optimized) or submap_data (the problem's poses): the
  // last optimized submap that is still in the graph; before any, the initial trajectory pose if one was set. false: that
  // pose needs a trajectory without nodes.
  bool local_to_global(int32_t trajectory_id, bool optimized, Rigidd* out) const {
    const auto it = trajectories.find(trajectory_id);
    if (it != trajectories.end())
      for (auto s = it->second.submaps.rbegin(); s != it->second.submaps.rend(); ++s)
        if (!optimized || s->second.optimized) {
          *out = compose(optimized ? s->second.optimized_global : s->second.global, inverse(s->second.local));
          return true;
        }
    const auto ip = initial_poses.find(trajectory_id);
    if (ip == initial_poses.end()) {
      *out = identity();
      return true;
    }
    Rigidd at;
    if (!interpolated_global_pose(ip->second.to_trajectory_id, ip->second.time, &at)) return false;
    *out = compose(at, ip->second.relative_pose);
    return true;
  }
  int reserve_store(int64_t floats) {
    const int64_t capacity = (int64_t)d_store.cap;
    if (store_used + floats <= capacity) return DL_OK;
    const int64_t cap = std::max<int64_t>({store_used + floats, 2 * capacity, (int64_t)1 << 20});
    DL_CUDA(ctx, cudaSetDevice(ctx->device));
    return grow(ctx, d_store, (size_t)cap, (size_t)store_used);
  }
  int optimize(dl_solve_summary* summary);
  int run_trimmers();
  int check_trimmable(int32_t trajectory_id, int32_t submap_index) const;
  int mark_submap_as_trimmed(const Id& submap_id);
  int compact_store();
  int range_data_map(int32_t num_trajectories, const int32_t* trajectory_ids, int32_t node_capacity, dl_range_data_map_node* nodes,
                     int32_t* num_nodes, int64_t capacity_points, float* points, int64_t* num_points, bool device_points);
};

namespace {

struct Pair {  // one (node, submap) search of the fan-out
  Id submap, node;
  double guess[7];
  int64_t hi_begin, n_hi, lo_begin, n_lo;
};

int check_options(dl_context* ctx, const dl_pose_graph_3d_options& o) {
  if (o.optimize_every_n_nodes < 0) return ctx->fail(DL_ERR_ARG, "optimize_every_n_nodes must be >= 0");
  if (o.every_nodes_to_find_constraint < 1) return ctx->fail(DL_ERR_ARG, "every_nodes_to_find_constraint must be >= 1");
  if (o.optimization_problem.max_num_iterations < 0) return ctx->fail(DL_ERR_ARG, "max_num_iterations must be >= 0");
  return check_constraint_options(ctx, o.constraint_builder);  // the checks of dl_constraint_search_batch
}

}  // namespace

// HandleWorkQueue (:444-470) + RunOptimization (:718-770)
int dl_pose_graph_3d::optimize(dl_solve_summary* summary) {
  const size_t table_size = constraints.size();  // a failed solve puts the pending constraints back
  for (const dl_pg3d_constraint& c : pending) {
    bool has_added = false;
    for (const dl_pg3d_constraint& t : constraints)
      if (t.submap_trajectory_id == c.submap_trajectory_id && t.submap_index == c.submap_index &&
          t.node_trajectory_id == c.node_trajectory_id && t.node_index == c.node_index) {
        has_added = true;
        break;
      }
    if (!has_added) constraints.push_back(c);
  }
  if (summary) std::memset(summary, 0, sizeof(*summary));
  // poses: submaps then nodes, each in (trajectory, index) order over the ids still in the graph. The solve holds its first
  // submap, so after a trim of the first one the next remaining submap is the anchor (optimization_problem_3d.cc:286-316).
  std::map<Id, int32_t> submap_row, node_row;
  int32_t S = 0, N = 0;
  for (const auto& [id, t] : trajectories) {
    for (const auto& kv : t.submaps) submap_row[Id{id, kv.first}] = S++;
    for (const auto& kv : t.nodes) node_row[Id{id, kv.first}] = N++;
  }
  if (S == 0) {  // RunOptimization: nothing to optimize
    pending.clear();
    return run_trimmers();
  }
  std::vector<double> poses(7 * (size_t)(S + N));
  std::vector<uint8_t> frozen_mask(S + N, 0);
  for (const auto& [id, t] : trajectories) {
    const uint8_t f = frozen.count(id) ? 1 : 0;
    for (const auto& [i, s] : t.submaps) {
      const int32_t r = submap_row[Id{id, i}];
      pose_to7(s.global, &poses[7 * (size_t)r]);
      frozen_mask[r] = f;
    }
    for (const auto& [i, n] : t.nodes) {
      const int32_t r = S + node_row[Id{id, i}];
      pose_to7(n.problem_global, &poses[7 * (size_t)r]);
      frozen_mask[r] = f;
    }
  }
  std::vector<dl_spa_constraint> spa(constraints.size());
  for (size_t k = 0; k < constraints.size(); ++k) {
    const dl_pg3d_constraint& c = constraints[k];
    dl_spa_constraint& s = spa[k];
    s.submap = submap_row.at(Id{c.submap_trajectory_id, c.submap_index});
    s.node = node_row.at(Id{c.node_trajectory_id, c.node_index});
    std::memcpy(s.zbar, c.zbar, sizeof(s.zbar));
    s.translation_weight = c.translation_weight;
    s.rotation_weight = c.rotation_weight;
  }
  dl_solve_summary local{};
  const int st = dl_pose_graph_solve_sparse(ctx, nullptr, &options.optimization_problem, S, N, poses.data(), frozen_mask.data(),
                                            spa.data(), (int32_t)spa.size(), &local, nullptr);
  if (st != DL_OK) {
    constraints.resize(table_size);
    return st;
  }
  pending.clear();
  if (summary) *summary = local;
  for (auto& [id, t] : trajectories) {
    for (auto& [i, s] : t.submaps) s.global = pose_from7(&poses[7 * (size_t)submap_row[Id{id, i}]]);
    for (auto& [i, n] : t.nodes) {
      n.problem_global = pose_from7(&poses[7 * (size_t)(S + node_row[Id{id, i}])]);
      // every node is in node_data here (the calls are synchronous), so RunOptimization's extrapolation of the nodes added
      // after the solve started (:748-762) has nothing to move
      n.global = n.problem_global;
    }
  }
  for (auto& [id, t] : trajectories)  // global_submap_poses_ = submap_data
    for (auto& [i, s] : t.submaps) {
      s.optimized = true;
      s.optimized_global = s.global;
    }
  num_nodes_since_last_loop_closure = 0;
  return run_trimmers();
}

// HandleWorkQueue (:492-501): every trimmer in the order added, then the finished ones are dropped.
// PureLocalizationTrimmer::Trim (pose_graph_trimmer.cc:30-43): all but the newest num_submaps_to_keep submaps, all of them
// once the trajectory is finished, which also finishes the trimmer.
int dl_pose_graph_3d::run_trimmers() {
  for (PureLocalizationTrimmer& tr : trimmers) {
    if (finished_trajectories.count(tr.trajectory_id)) tr.num_submaps_to_keep = 0;
    std::vector<int32_t> ids;
    const auto it = trajectories.find(tr.trajectory_id);
    if (it != trajectories.end())
      for (const auto& kv : it->second.submaps) ids.push_back(kv.first);
    for (size_t i = 0; i + (size_t)tr.num_submaps_to_keep < ids.size(); ++i) {
      DL_TRY(check_trimmable(tr.trajectory_id, ids[i]));
      DL_TRY(mark_submap_as_trimmed(Id{tr.trajectory_id, ids[i]}));
    }
  }
  trimmers.erase(std::remove_if(trimmers.begin(), trimmers.end(),
                                [](const PureLocalizationTrimmer& tr) { return tr.num_submaps_to_keep == 0; }),
                 trimmers.end());
  return DL_OK;
}

int dl_pose_graph_3d::check_trimmable(int32_t trajectory_id, int32_t submap_index) const {
  const auto it = trajectories.find(trajectory_id);
  if (it == trajectories.end() || !it->second.submaps.count(submap_index))
    return ctx->fail(DL_ERR_ARG, "trim: no such submap in the graph (unknown or already trimmed)");
  if (!it->second.submaps.at(submap_index).finished) return ctx->fail(DL_ERR_ARG, "trim: the submap is not finished");
  if (!pending.empty()) return ctx->fail(DL_ERR_ARG, "trim: constraints are pending; trim right after an optimization");
  return DL_OK;
}

// TrimmingHandle::MarkSubmapAsTrimmed (:1002-1058) and OptimizationProblem3D::TrimSubmap / TrimTrajectoryNode
// (optimization_problem_3d.cc:229-251): the submap, its constraints, and the nodes left without an INTRA_SUBMAP constraint
// together with all of theirs leave the graph. Their clouds become dead ranges of the node store.
int dl_pose_graph_3d::mark_submap_as_trimmed(const Id& submap_id) {
  const auto submap_of = [](const dl_pg3d_constraint& c) { return Id{c.submap_trajectory_id, c.submap_index}; };
  const auto node_of = [](const dl_pg3d_constraint& c) { return Id{c.node_trajectory_id, c.node_index}; };
  std::set<Id> nodes_to_retain;
  for (const dl_pg3d_constraint& c : constraints)
    if (c.tag == DL_PG3D_INTRA_SUBMAP && submap_of(c) != submap_id) nodes_to_retain.insert(node_of(c));
  std::set<Id> nodes_to_remove;
  std::vector<dl_pg3d_constraint> kept;
  for (const dl_pg3d_constraint& c : constraints) {
    if (submap_of(c) == submap_id) {
      if (c.tag == DL_PG3D_INTRA_SUBMAP && !nodes_to_retain.count(node_of(c))) nodes_to_remove.insert(node_of(c));
    } else {
      kept.push_back(c);
    }
  }
  constraints.clear();
  for (const dl_pg3d_constraint& c : kept)
    if (!nodes_to_remove.count(node_of(c))) constraints.push_back(c);
  Trajectory& t = trajectories.at(submap_id.first);
  const auto s = t.submaps.find(submap_id.second);
  if (std::next(s) == t.submaps.end()) t.submaps_can_append = false;
  t.submaps.erase(s);
  computed.erase(submap_id);  // ConstraintBuilder3D::DeleteScanMatcher: the submap is never a search target again
  for (const Id& node_id : nodes_to_remove) {
    Trajectory& nt = trajectories.at(node_id.first);
    const auto n = nt.nodes.find(node_id.second);
    if (std::next(n) == nt.nodes.end()) nt.nodes_can_append = false;
    store_live -= 3 * (n->second.n_hi + n->second.n_lo + n->second.n_rd);
    nt.nodes.erase(n);
    for (auto& kv : computed) kv.second.erase(node_id);
  }
  last_trimmed.push_back(dl_pg3d_submap_id{submap_id.first, submap_id.second});
  if (store_used - store_live > store_live && store_used - store_live >= kMinDeadFloats) return compact_store();
  return DL_OK;
}

// Every live node's clouds into a fresh store, in (trajectory, index) order, by one launch of pg3d_store_compact; then the old
// buffer is freed and the offsets are rewritten. Each compaction copies at most as many floats as died since the last one,
// so the copying costs O(1) per uploaded float. A failure leaves the old store and every offset as they were.
int dl_pose_graph_3d::compact_store() {
  std::vector<StoreSegment> segments;
  int64_t live = 0;
  for (const auto& [id, t] : trajectories)
    for (const auto& [i, n] : t.nodes) {
      segments.push_back(StoreSegment{3 * n.hi_begin, live, 3 * (n.n_hi + n.n_lo)});
      live += 3 * (n.n_hi + n.n_lo);
      if (n.n_rd > 0) {  // returns attached later: one more segment
        segments.push_back(StoreSegment{3 * n.rd_begin, live, 3 * n.n_rd});
        live += 3 * n.n_rd;
      }
    }
  if (live == 0) {  // nothing left to copy: the store is freed, and the next add_node grows a new one
    DL_CUDA(ctx, cudaSetDevice(ctx->device));
    DL_CUDA(ctx, ctx->wait_stream());
    d_store.reset();
    store_used = store_live = 0;
    return DL_OK;
  }
  const int64_t cap = std::max<int64_t>(2 * live, (int64_t)1 << 20);
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  DL_TRY(ctx->reserve_device(std::max<size_t>(segments.size(), 1) * sizeof(StoreSegment)));
  DeviceBuffer<float> fresh;
  const int st = alloc(ctx, fresh, (size_t)cap);
  if (st != DL_OK) {
    cudaGetLastError();  // an allocation failure is not sticky: clear it for the next launch check
    return st;
  }
  StoreSegment* d_segments = reinterpret_cast<StoreSegment*>(ctx->d_scratch.get());  // live > 0: segments is not empty
  DL_TRY(h2d(ctx, d_segments, segments.data(), segments.size()));
  pg3d_store_compact<<<(unsigned)segments.size(), kCompactBlock, 0, ctx->stream>>>(d_store.get(), fresh.get(), d_segments);
  DL_LAUNCH_CHECK(ctx, "pg3d_store_compact");
  DL_CUDA(ctx, ctx->wait_stream());
  d_store = std::move(fresh);
  store_used = store_live = live;
  size_t k = 0;
  for (auto& [id, t] : trajectories)
    for (auto& [i, n] : t.nodes) {
      n.hi_begin = segments[k++].dst / 3;
      n.lo_begin = n.hi_begin + n.n_hi;
      if (n.n_rd > 0) n.rd_begin = segments[k++].dst / 3;
    }
  return DL_OK;
}

// The body of dl_range_data_map and its _dev variant: the selection and the counts on the host, then, when there are
// points to write, one upload of the table of nodes with points, one launch and one host wait (after the download into
// `points` for the host variant).
int dl_pose_graph_3d::range_data_map(int32_t num_trajectories, const int32_t* trajectory_ids, int32_t node_capacity,
                                     dl_range_data_map_node* nodes, int32_t* num_nodes, int64_t capacity_points, float* points,
                                     int64_t* num_points, bool device_points) {
  if (!num_nodes || !num_points || node_capacity < 0 || capacity_points < 0) return DL_ERR_ARG;
  if (num_trajectories < 0) return ctx->fail(DL_ERR_ARG, "num_trajectories must be >= 0");
  std::vector<const std::pair<const int32_t, Trajectory>*> selected;
  if (!trajectory_ids) {
    for (const auto& kv : trajectories) selected.push_back(&kv);
  } else {
    std::set<int32_t> ids;
    for (int32_t k = 0; k < num_trajectories; ++k)
      if (!ids.insert(trajectory_ids[k]).second) return ctx->fail(DL_ERR_ARG, "a trajectory id is listed twice");
    for (const int32_t id : ids) {
      const auto it = trajectories.find(id);
      if (it == trajectories.end()) return ctx->fail(DL_ERR_ARG, "unknown trajectory id");
      selected.push_back(&*it);
    }
  }
  int64_t count = 0, total = 0;
  for (const auto* t : selected)
    for (const auto& [i, n] : t->second.nodes)
      if (n.has_range_data) {
        ++count;
        total += n.n_rd;
      }
  if (count > INT32_MAX) return ctx->fail(DL_ERR_ARG, "more than INT32_MAX nodes with range data");
  *num_nodes = (int32_t)count;
  *num_points = total;
  if (!nodes || !points) return DL_OK;
  if (node_capacity < count) return ctx->fail(DL_ERR_ARG, "node_capacity smaller than the map's nodes");
  if (capacity_points < total) return ctx->fail(DL_ERR_ARG, "capacity_points smaller than the map's points");
  std::vector<RangeDataMapNode> table;  // the nodes with points: the kernel's binary search needs increasing first points
  int32_t k = 0;
  int64_t offset = 0;
  for (const auto* t : selected)
    for (const auto& [i, n] : t->second.nodes) {
      if (!n.has_range_data) continue;
      dl_range_data_map_node& out = nodes[k++];
      out.trajectory_id = t->first;
      out.node_index = i;
      out.first_point = offset;
      out.num_points = n.n_rd;
      pose_to7(n.global, out.global_pose);
      if (n.n_rd > 0) table.push_back(RangeDataMapNode{n.rd_begin, offset, n.n_rd, inverse(to_float(n.local)), to_float(n.global)});
      offset += n.n_rd;
    }
  if (total == 0) return DL_OK;
  RangeDataMapNode* d_table = nullptr;
  float* d_points = points;
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  DL_TRY(carve_scratch(ctx, [&](Arena& a) {
    d_table = a.take<RangeDataMapNode>(table.size());
    if (!device_points) d_points = a.take<float>(3 * (size_t)total);
  }));
  DL_TRY(h2d(ctx, d_table, table.data(), table.size()));
  const int64_t blocks = (total + kMapTile - 1) / kMapTile;
  if (blocks > INT32_MAX) return ctx->fail(DL_ERR_ARG, "map too large for one launch");
  {
    StageScope stage(ctx, "pg3d_range_data_map");
    pg3d_range_data_map<<<(unsigned)blocks, kMapBlock, 0, ctx->stream>>>(d_store.get(), d_table, (int)table.size(), total, d_points);
    DL_LAUNCH_CHECK(ctx, "pg3d_range_data_map");
  }
  if (!device_points) DL_TRY(d2h(ctx, points, d_points, 3 * (size_t)total));
  return sync(ctx);
}

extern "C" {

int dl_pose_graph_3d_create(dl_context* ctx, const dl_pose_graph_3d_options* options, dl_pose_graph_3d** out) {
  if (!ctx || !options || !out) return DL_ERR_ARG;
  *out = nullptr;
  DL_TRY(check_options(ctx, *options));
  dl_pose_graph_3d* g = new dl_pose_graph_3d;
  g->ctx = ctx;
  g->options = *options;
  *out = g;
  return DL_OK;
}

void dl_pose_graph_3d_destroy(dl_pose_graph_3d* g) {
  if (!g) return;
  if (g->d_store.get()) {
    cudaSetDevice(g->ctx->device);
    g->ctx->wait_stream();
  }
  delete g;
}

int dl_pose_graph_3d_add_node(dl_pose_graph_3d* g, const dl_pg3d_node* node, int32_t num_matches,
                              const dl_pg3d_submap_match* matches, dl_pg3d_add_node_info* info) {
  if (!g || !node || num_matches < 0 || (num_matches > 0 && !matches)) return DL_ERR_ARG;
  g->last_trimmed.clear();
  dl_context* ctx = g->ctx;
  const auto t0 = std::chrono::steady_clock::now();
  const int m = node->num_insertion_submaps;
  if (m != 1 && m != 2) return ctx->fail(DL_ERR_ARG, "a node has one or two insertion submaps");
  if (node->num_high_resolution < 1 || node->num_low_resolution < 1 || !node->high_resolution_points || !node->low_resolution_points)
    return ctx->fail(DL_ERR_EMPTY, "a node needs non-empty high- and low-resolution clouds");
  if (node->num_high_resolution > INT32_MAX || node->num_low_resolution > INT32_MAX) return ctx->fail(DL_ERR_ARG, "cloud too large");
  const dl_pg3d_insertion_submap* ins = node->insertion_submaps;
  for (int i = 0; i < m; ++i)
    if (!ins[i].high_resolution_grid || !ins[i].low_resolution_grid) return ctx->fail(DL_ERR_ARG, "insertion submap without grids");
  const int32_t tid = node->trajectory_id;
  if (tid < 0) return ctx->fail(DL_ERR_ARG, "negative trajectory id");
  if (g->finished_trajectories.count(tid)) return ctx->fail(DL_ERR_ARG, "the trajectory is finished");
  const auto tit = g->trajectories.find(tid);
  if (tit != g->trajectories.end() && !tit->second.nodes_can_append)
    return ctx->fail(DL_ERR_ARG, "the trajectory's highest node index was trimmed: no more nodes can be appended");
  const int32_t S = tit == g->trajectories.end() ? 0 : tit->second.num_submaps;  // submap indices handed out, holes included
  // AddNode's "is insertion_submaps.back() new" and InitializeGlobalSubmapPoses' CHECKs, as index rules
  bool back_is_new;
  if (m == 1) {
    if (ins[0].submap_index != 0 || S > 1) return ctx->fail(DL_ERR_ARG, "one insertion submap: it must be the trajectory's submap 0");
    back_is_new = S == 0;
  } else {
    const int32_t a = ins[0].submap_index, b = ins[1].submap_index;
    if (S >= 1 && a == S - 1 && b == S) back_is_new = true;
    else if (S >= 2 && a == S - 2 && b == S - 1) back_is_new = false;
    else return ctx->fail(DL_ERR_ARG, "insertion submaps do not continue the trajectory's submap sequence");
  }
  if (back_is_new && tit != g->trajectories.end() && !tit->second.submaps_can_append)
    return ctx->fail(DL_ERR_ARG, "the trajectory's highest submap index was trimmed: no more submaps can be appended");
  if (tit != g->trajectories.end())
    for (int i = 0; i < m; ++i) {
      if (ins[i].submap_index >= S) continue;
      const auto it = tit->second.submaps.find(ins[i].submap_index);
      if (it == tit->second.submaps.end()) return ctx->fail(DL_ERR_ARG, "insertion submap was trimmed");
      if (it->second.finished) return ctx->fail(DL_ERR_ARG, "insertion submap is already finished");
    }
  Rigidd local_to_global;  // GetLocalToGlobalTransform, for the node's pose (:115-116) and a first submap (:67-110)
  if (!g->local_to_global(tid, true, &local_to_global))
    return ctx->fail(DL_ERR_ARG, "the initial trajectory pose refers to a trajectory without nodes");
  const bool newly_finished = ins[0].finished != 0;
  if (!newly_finished && num_matches > 0) return ctx->fail(DL_ERR_ARG, "submap matches passed but no insertion submap finished");
  const Id front_id{tid, ins[0].submap_index};
  std::vector<dl_pg3d_submap_match> sorted(matches, matches + num_matches);
  std::sort(sorted.begin(), sorted.end(), [](const dl_pg3d_submap_match& x, const dl_pg3d_submap_match& y) {
    return Id{x.trajectory_id, x.submap_index} < Id{y.trajectory_id, y.submap_index};
  });
  for (size_t k = 0; k < sorted.size(); ++k) {
    const Id to{sorted[k].trajectory_id, sorted[k].submap_index};
    if (to == front_id) return ctx->fail(DL_ERR_ARG, "a match names the finished submap itself");
    if (to.first == tid && std::abs(to.second - front_id.second) <= 2)
      return ctx->fail(DL_ERR_ARG, "a match names a same-trajectory submap within two indices");
    const auto it = g->trajectories.find(to.first);
    if (it == g->trajectories.end() || !it->second.submaps.count(to.second))
      return ctx->fail(DL_ERR_ARG, "a match names an unknown or trimmed submap");
    if (!it->second.submaps.at(to.second).finished) return ctx->fail(DL_ERR_ARG, "a match names an unfinished submap");
    if (k > 0 && to == Id{sorted[k - 1].trajectory_id, sorted[k - 1].submap_index})
      return ctx->fail(DL_ERR_ARG, "a submap is matched twice");
  }

  // ---- 2. the node's clouds into the node store (store_used moves on only at the commit below)
  const int64_t n_hi = node->num_high_resolution, n_lo = node->num_low_resolution;
  DL_TRY(g->reserve_store(3 * (n_hi + n_lo)));
  const int64_t hi_begin = g->store_used / 3, lo_begin = hi_begin + n_hi;
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  DL_TRY(h2d(ctx, g->d_store.get() + 3 * hi_begin, node->high_resolution_points, 3 * (size_t)n_hi));
  DL_TRY(h2d(ctx, g->d_store.get() + 3 * lo_begin, node->low_resolution_points, 3 * (size_t)n_lo));
  DL_TRY(sync(ctx));  // pageable host memory
  const int64_t uploaded = 12 * (n_hi + n_lo);

  // ---- 4. fan-out and searches of a newly finished submap, before anything is committed
  const Rigidd local_pose = pose_from7(node->local_pose);
  const int32_t node_index = tit == g->trajectories.end() ? 0 : tit->second.num_nodes;
  std::vector<Pair> pairs;
  std::vector<dl_constraint> results;
  double search_ms = 0.0;
  if (newly_finished && !sorted.empty()) {
    const Trajectory* tr = tit == g->trajectories.end() ? nullptr : &tit->second;
    const Rigidd local_from = pose_from7(ins[0].local_pose);  // a finished submap was seen before: the same pose
    const Submap* from = tr && front_id.second < S ? &tr->submaps.at(front_id.second) : nullptr;
    const Rigidd from_local = from ? from->local : local_from;
    std::vector<int32_t> nodes_in_submap;
    if (from)
      for (const int32_t n : from->node_ids)
        if (tr->nodes.count(n)) nodes_in_submap.push_back(n);  // trimmed nodes are holes
    nodes_in_submap.push_back(node_index);  // this node was just inserted into it
    const Rigidd T_S2_G2 = yaw_free_alignment(from_local);
    const Rigidd from_local_inv = inverse(from_local);
    for (const dl_pg3d_submap_match& mt : sorted) {
      const Id to{mt.trajectory_id, mt.submap_index};
      const Submap& target = g->trajectories.at(to.first).submaps.at(to.second);
      const Rigidd T_G1_S1 = inverse(yaw_free_alignment(target.local));
      const Rigidd submap_to_submap_2d{{mt.x, mt.y, 0.0}, yaw_quaternion(mt.theta)};  // Embed3D(Rigid2d)
      const Rigidd left = compose(compose(T_G1_S1, submap_to_submap_2d), T_S2_G2);
      const auto done = g->computed.find(to);
      int j = 0;
      for (const int32_t n : nodes_in_submap) {
        if (j++ % g->options.every_nodes_to_find_constraint != 0) continue;
        if (done != g->computed.end() && done->second.count(Id{tid, n})) continue;
        const bool is_new = n == node_index;
        const Node* nd = is_new ? nullptr : &tr->nodes.at(n);
        Pair p;
        p.submap = to;
        p.node = Id{tid, n};
        pose_to7(compose(left, compose(from_local_inv, is_new ? local_pose : nd->local)), p.guess);
        p.hi_begin = is_new ? hi_begin : nd->hi_begin;
        p.n_hi = is_new ? n_hi : nd->n_hi;
        p.lo_begin = is_new ? lo_begin : nd->lo_begin;
        p.n_lo = is_new ? n_lo : nd->n_lo;
        pairs.push_back(p);
      }
    }
    if (!pairs.empty()) {
      const auto ts = std::chrono::steady_clock::now();
      const int n = (int)pairs.size();
      std::vector<double> guesses(7 * (size_t)n);
      std::vector<int64_t> hi_off(n + 1, 0), lo_off(n + 1, 0), hib(n), lob(n);
      std::vector<const dl_grid*> hg(n), lg(n);
      for (int k = 0; k < n; ++k) {
        const Pair& p = pairs[k];
        std::memcpy(&guesses[7 * (size_t)k], p.guess, sizeof(p.guess));
        hi_off[k + 1] = hi_off[k] + p.n_hi;
        lo_off[k + 1] = lo_off[k] + p.n_lo;
        hib[k] = p.hi_begin;
        lob[k] = p.lo_begin;
        const Submap& target = g->trajectories.at(p.submap.first).submaps.at(p.submap.second);
        if (target.hi->structure_dirty || target.lo->structure_dirty)
          return ctx->fail(DL_ERR_ARG, "dl_grid_sync not called after dl_grid_set_cells");
        hg[k] = target.hi;
        lg[k] = target.lo;
      }
      PairClouds pc;
      pc.hi_off = hi_off.data();
      pc.lo_off = lo_off.data();
      pc.hi_store = g->d_store.get();
      pc.lo_store = g->d_store.get();
      pc.hi_begin = hib.data();
      pc.lo_begin = lob.data();
      results.resize(n);
      DL_TRY(constraint_search(ctx, g->options.constraint_builder, n, guesses.data(), pc, hg.data(), lg.data(), results.data()));
      search_ms = ms_since(ts);
    }
  }

  // ---- commit: 1. AddNode, 3. ComputeConstraintsForNode, 4. the searches' results
  Trajectory& t = g->trajectories[tid];
  g->store_used += 3 * (n_hi + n_lo);
  g->store_live += 3 * (n_hi + n_lo);
  g->bytes_uploaded += uploaded;
  Node nd;
  nd.time = node->time;
  nd.local = local_pose;
  nd.global = compose(local_to_global, local_pose);  // GetLocalToGlobalTransform * local_pose (:115-116)
  nd.hi_begin = hi_begin;
  nd.n_hi = n_hi;
  nd.lo_begin = lo_begin;
  nd.n_lo = n_lo;
  if (back_is_new) {
    Submap s;
    s.hi = ins[m - 1].high_resolution_grid;
    s.lo = ins[m - 1].low_resolution_grid;
    s.local = pose_from7(ins[m - 1].local_pose);
    // InitializeGlobalSubmapPoses (:67-110)
    if (m == 1) s.global = compose(local_to_global, s.local);
    else {
      const Submap& front = t.submaps.at(ins[0].submap_index);
      s.global = compose(compose(front.global, inverse(front.local)), s.local);
    }
    t.submaps[t.num_submaps++] = s;
  }
  const Submap& matching = t.submaps.at(ins[0].submap_index);
  nd.problem_global = compose(compose(matching.global, inverse(matching.local)), local_pose);  // :345-347
  t.nodes[t.num_nodes++] = nd;
  for (int i = 0; i < m; ++i) {
    Submap& s = t.submaps.at(ins[i].submap_index);
    s.node_ids.push_back(node_index);
    dl_pg3d_constraint c{};
    c.submap_trajectory_id = tid;
    c.submap_index = ins[i].submap_index;
    c.node_trajectory_id = tid;
    c.node_index = node_index;
    pose_to7(compose(inverse(s.local), local_pose), c.zbar);  // :358-359
    c.translation_weight = g->options.matcher_translation_weight;
    c.rotation_weight = g->options.matcher_rotation_weight;
    c.tag = DL_PG3D_INTRA_SUBMAP;
    g->constraints.push_back(c);
  }
  int32_t found = 0;
  g->last_searches.assign(pairs.size(), dl_pg3d_search{});
  for (size_t k = 0; k < pairs.size(); ++k) {
    dl_pg3d_search& s = g->last_searches[k];
    s.submap_trajectory_id = pairs[k].submap.first;
    s.submap_index = pairs[k].submap.second;
    s.node_trajectory_id = pairs[k].node.first;
    s.node_index = pairs[k].node.second;
    std::memcpy(s.pose_guess, pairs[k].guess, sizeof(s.pose_guess));
    s.result = results[k];
  }
  if (newly_finished) {
    t.submaps.at(ins[0].submap_index).finished = true;
    for (size_t k = 0; k < pairs.size(); ++k) {
      if (!results[k].found) continue;
      ++found;
      g->computed[pairs[k].submap].insert(pairs[k].node);  // constraint_builder_3d.cc:334
      dl_pg3d_constraint c{};
      c.submap_trajectory_id = pairs[k].submap.first;
      c.submap_index = pairs[k].submap.second;
      c.node_trajectory_id = pairs[k].node.first;
      c.node_index = pairs[k].node.second;
      std::memcpy(c.zbar, results[k].pose, sizeof(c.zbar));
      c.translation_weight = results[k].translation_weight;
      c.rotation_weight = results[k].rotation_weight;
      c.tag = DL_PG3D_INTER_SUBMAP;
      g->pending.push_back(c);
    }
  }
  const double bookkeeping_ms = ms_since(t0) - search_ms;

  // ---- 5. the optimization trigger (:393-398)
  ++g->num_nodes_since_last_loop_closure;
  dl_solve_summary summary{};
  int32_t optimized = 0;
  double solve_ms = 0.0;
  if (g->options.optimize_every_n_nodes > 0 && g->num_nodes_since_last_loop_closure > g->options.optimize_every_n_nodes) {
    const auto ts = std::chrono::steady_clock::now();
    DL_TRY(g->optimize(&summary));
    solve_ms = ms_since(ts);
    optimized = 1;
  }
  if (info) {
    std::memset(info, 0, sizeof(*info));
    info->node_index = node_index;
    info->num_searched = (int32_t)pairs.size();
    info->num_found = found;
    info->optimized = optimized;
    info->cloud_bytes_uploaded = uploaded;
    info->bookkeeping_ms = bookkeeping_ms;
    info->search_ms = search_ms;
    info->solve_ms = solve_ms;
    info->summary = summary;
  }
  return DL_OK;
}

int dl_pose_graph_3d_freeze_trajectory(dl_pose_graph_3d* g, int32_t trajectory_id) {
  if (!g || trajectory_id < 0) return DL_ERR_ARG;
  g->frozen.insert(trajectory_id);
  return DL_OK;
}

int dl_pose_graph_3d_run_final_optimization(dl_pose_graph_3d* g, dl_solve_summary* summary) {
  if (!g) return DL_ERR_ARG;
  g->last_trimmed.clear();
  // max_num_final_iterations is set and then overwritten with the regular cap (pose_graph_3d.cc:677-682): the same solve
  return g->optimize(summary);
}

int dl_pose_graph_3d_poses(const dl_pose_graph_3d* g, int32_t trajectory_id, int32_t which, int32_t capacity, double* poses,
                           int32_t* count) {
  if (!g || !count || which < DL_PG3D_NODE_POSES || which > DL_PG3D_OPTIMIZATION_SUBMAPS || capacity < 0) return DL_ERR_ARG;
  const auto it = g->trajectories.find(trajectory_id);
  const bool nodes = which == DL_PG3D_NODE_POSES || which == DL_PG3D_OPTIMIZATION_NODES;
  const int32_t n = it == g->trajectories.end() ? 0 : (int32_t)(nodes ? it->second.nodes.size() : it->second.submaps.size());
  *count = n;
  if (!poses) return DL_OK;
  if (capacity < n) return g->ctx->fail(DL_ERR_ARG, "capacity smaller than the trajectory");
  if (n == 0) return DL_OK;
  Rigidd extrapolate = identity();
  if (which == DL_PG3D_SUBMAP_POSES && !g->local_to_global(trajectory_id, true, &extrapolate))
    return g->ctx->fail(DL_ERR_ARG, "the initial trajectory pose refers to a trajectory without nodes");
  size_t i = 0;
  if (nodes)
    for (const auto& kv : it->second.nodes)
      pose_to7(which == DL_PG3D_NODE_POSES ? kv.second.global : kv.second.problem_global, poses + 7 * i++);
  else
    for (const auto& kv : it->second.submaps) {
      const Submap& s = kv.second;
      const Rigidd p = which == DL_PG3D_OPTIMIZATION_SUBMAPS ? s.global : s.optimized ? s.optimized_global : compose(extrapolate, s.local);
      pose_to7(p, poses + 7 * i++);
    }
  return DL_OK;
}

int dl_pose_graph_3d_local_to_global(const dl_pose_graph_3d* g, int32_t trajectory_id, double* pose) {
  if (!g || !pose) return DL_ERR_ARG;
  Rigidd p;
  if (!g->local_to_global(trajectory_id, true, &p))
    return g->ctx->fail(DL_ERR_ARG, "the initial trajectory pose refers to a trajectory without nodes");
  pose_to7(p, pose);
  return DL_OK;
}

int dl_pose_graph_3d_constraints(const dl_pose_graph_3d* g, int32_t capacity, dl_pg3d_constraint* out, int32_t* count) {
  if (!g || !count || capacity < 0) return DL_ERR_ARG;
  const int32_t n = (int32_t)g->constraints.size();
  *count = n;
  if (!out) return DL_OK;
  if (capacity < n) return g->ctx->fail(DL_ERR_ARG, "capacity smaller than the constraint table");
  std::copy(g->constraints.begin(), g->constraints.end(), out);
  return DL_OK;
}

int dl_pose_graph_3d_last_searches(const dl_pose_graph_3d* g, int32_t capacity, dl_pg3d_search* out, int32_t* count) {
  if (!g || !count || capacity < 0) return DL_ERR_ARG;
  const int32_t n = (int32_t)g->last_searches.size();
  *count = n;
  if (!out) return DL_OK;
  if (capacity < n) return g->ctx->fail(DL_ERR_ARG, "capacity smaller than the search list");
  std::copy(g->last_searches.begin(), g->last_searches.end(), out);
  return DL_OK;
}

int dl_pose_graph_3d_store_bytes(const dl_pose_graph_3d* g, int64_t* uploaded, int64_t* capacity) {
  if (!g) return DL_ERR_ARG;
  if (uploaded) *uploaded = g->bytes_uploaded;
  if (capacity) *capacity = (int64_t)g->d_store.cap * (int64_t)sizeof(float);
  return DL_OK;
}

int dl_pg3d_trim_submap(dl_pose_graph_3d* g, int32_t trajectory_id, int32_t submap_index) {
  if (!g) return DL_ERR_ARG;
  g->last_trimmed.clear();
  DL_TRY(g->check_trimmable(trajectory_id, submap_index));
  return g->mark_submap_as_trimmed(Id{trajectory_id, submap_index});
}

int dl_pg3d_add_pure_localization_trimmer(dl_pose_graph_3d* g, int32_t trajectory_id, int32_t num_submaps_to_keep) {
  if (!g || trajectory_id < 0) return DL_ERR_ARG;
  if (num_submaps_to_keep < 3) return g->ctx->fail(DL_ERR_ARG, "a pure-localization trimmer keeps at least 3 submaps");
  g->trimmers.push_back(dl_pose_graph_3d::PureLocalizationTrimmer{trajectory_id, num_submaps_to_keep});
  return DL_OK;
}

int dl_pg3d_finish_trajectory(dl_pose_graph_3d* g, int32_t trajectory_id) {
  if (!g || trajectory_id < 0) return DL_ERR_ARG;
  g->last_trimmed.clear();
  if (!g->finished_trajectories.insert(trajectory_id).second) return g->ctx->fail(DL_ERR_ARG, "the trajectory is already finished");
  const auto it = g->trajectories.find(trajectory_id);
  if (it != g->trajectories.end())
    for (auto& kv : it->second.submaps) kv.second.finished = true;
  return g->optimize(nullptr);  // DispatchOptimization: the step of dl_pose_graph_3d_run_final_optimization
}

int dl_pg3d_is_trajectory_finished(const dl_pose_graph_3d* g, int32_t trajectory_id, int32_t* finished) {
  if (!g || !finished) return DL_ERR_ARG;
  *finished = g->finished_trajectories.count(trajectory_id) ? 1 : 0;
  return DL_OK;
}

int dl_pg3d_set_initial_trajectory_pose(dl_pose_graph_3d* g, int32_t from_trajectory_id, int32_t to_trajectory_id,
                                        const double* relative_pose, double time) {
  if (!g || !relative_pose || from_trajectory_id < 0 || to_trajectory_id < 0) return DL_ERR_ARG;
  for (int k = 0; k < 7; ++k)
    if (!std::isfinite(relative_pose[k])) return g->ctx->fail(DL_ERR_ARG, "the relative pose is not finite");
  if (!std::isfinite(time)) return g->ctx->fail(DL_ERR_ARG, "the time is not finite");
  g->initial_poses[from_trajectory_id] = InitialTrajectoryPose{to_trajectory_id, pose_from7(relative_pose), time};
  return DL_OK;
}

int dl_pg3d_ids(const dl_pose_graph_3d* g, int32_t trajectory_id, int32_t which, int32_t capacity, int32_t* indices,
                int32_t* count) {
  if (!g || !count || which < DL_PG3D_NODE_POSES || which > DL_PG3D_OPTIMIZATION_SUBMAPS || capacity < 0) return DL_ERR_ARG;
  const auto it = g->trajectories.find(trajectory_id);
  const bool nodes = which == DL_PG3D_NODE_POSES || which == DL_PG3D_OPTIMIZATION_NODES;
  const int32_t n = it == g->trajectories.end() ? 0 : (int32_t)(nodes ? it->second.nodes.size() : it->second.submaps.size());
  *count = n;
  if (!indices) return DL_OK;
  if (capacity < n) return g->ctx->fail(DL_ERR_ARG, "capacity smaller than the trajectory");
  if (n == 0) return DL_OK;
  int32_t i = 0;
  if (nodes)
    for (const auto& kv : it->second.nodes) indices[i++] = kv.first;
  else
    for (const auto& kv : it->second.submaps) indices[i++] = kv.first;
  return DL_OK;
}

int dl_pg3d_last_trimmed(const dl_pose_graph_3d* g, int32_t capacity, dl_pg3d_submap_id* out, int32_t* count) {
  if (!g || !count || capacity < 0) return DL_ERR_ARG;
  const int32_t n = (int32_t)g->last_trimmed.size();
  *count = n;
  if (!out) return DL_OK;
  if (capacity < n) return g->ctx->fail(DL_ERR_ARG, "capacity smaller than the trimmed list");
  std::copy(g->last_trimmed.begin(), g->last_trimmed.end(), out);
  return DL_OK;
}

int dl_pg3d_store_usage(const dl_pose_graph_3d* g, int64_t* live_bytes, int64_t* used_bytes, int64_t* capacity_bytes) {
  if (!g) return DL_ERR_ARG;
  if (live_bytes) *live_bytes = g->store_live * (int64_t)sizeof(float);
  if (used_bytes) *used_bytes = g->store_used * (int64_t)sizeof(float);
  if (capacity_bytes) *capacity_bytes = (int64_t)g->d_store.cap * (int64_t)sizeof(float);
  return DL_OK;
}

int dl_range_data_map_set_node(dl_pose_graph_3d* g, int32_t trajectory_id, int32_t node_index, const float* returns,
                               int64_t num_returns) {
  if (!g) return DL_ERR_ARG;
  dl_context* ctx = g->ctx;
  if (num_returns < 0) return ctx->fail(DL_ERR_ARG, "num_returns must be >= 0");
  if (!returns && num_returns > 0) return ctx->fail(DL_ERR_ARG, "returns is NULL");
  const auto t = g->trajectories.find(trajectory_id);
  if (t == g->trajectories.end() || !t->second.nodes.count(node_index))
    return ctx->fail(DL_ERR_ARG, "range data for an unknown or trimmed node");
  Node& n = t->second.nodes.at(node_index);
  if (n.has_range_data) return ctx->fail(DL_ERR_ARG, "the node already has range data");
  // the returns into the node store (store_used moves on only at the commit below)
  DL_TRY(g->reserve_store(3 * num_returns));
  const int64_t begin = g->store_used / 3;
  if (num_returns > 0) {
    DL_CUDA(ctx, cudaSetDevice(ctx->device));
    DL_TRY(h2d(ctx, g->d_store.get() + 3 * begin, returns, 3 * (size_t)num_returns));
    DL_TRY(sync(ctx));  // pageable host memory
  }
  g->store_used += 3 * num_returns;
  g->store_live += 3 * num_returns;
  g->bytes_uploaded += 12 * num_returns;
  n.has_range_data = true;
  n.rd_begin = begin;
  n.n_rd = num_returns;
  return DL_OK;
}

int dl_range_data_map(dl_pose_graph_3d* g, int32_t num_trajectories, const int32_t* trajectory_ids, int32_t node_capacity,
                      dl_range_data_map_node* nodes, int32_t* num_nodes, int64_t capacity_points, float* points, int64_t* num_points) {
  if (!g) return DL_ERR_ARG;
  return g->range_data_map(num_trajectories, trajectory_ids, node_capacity, nodes, num_nodes, capacity_points, points, num_points,
                           false);
}

int dl_range_data_map_dev(dl_pose_graph_3d* g, int32_t num_trajectories, const int32_t* trajectory_ids, int32_t node_capacity,
                          dl_range_data_map_node* nodes, int32_t* num_nodes, int64_t capacity_points, float* points_dev,
                          int64_t* num_points) {
  if (!g) return DL_ERR_ARG;
  return g->range_data_map(num_trajectories, trajectory_ids, node_capacity, nodes, num_nodes, capacity_points, points_dev,
                           num_points, true);
}

}  // extern "C"
