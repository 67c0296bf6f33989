// The assets writer's point pipeline on the device (cartographer_ros/assets_writer.cc:120-160 HandleMessage with the processors
// of the fork's dlio/config/assets_writer_tongji.lua plus the moving-object removal): trajectory lookup, transform to the map,
// min_max_range_filter and voxel_filter_and_remove_moving_objects with the reference's restart protocol. See include/dliom_b200.h.
//
// One call takes many messages; its rows are numbered in message order ("virtual rows"). Per call:
//   mw_heads_count / tile prefix   a run is a maximal stretch of a message's rows with the same time bits; count run heads
//   mw_run_poses                   one pose per run (fp64 lookup + slerp + composition, cast to float), the run of every row,
//                                  and per message the last run with a pose (integer atomicMax: the batch origin)
//   mw_select (count / scatter)    transform, Has, range gate, ordered compaction by tile counts (the decode's scheme)
//   pass 1  mw_insert_hits          cell -> hits in an open-addressing table (64-bit key CAS, 32-bit atomicAdd)
//   pass 2  mw_rays                 one thread per point walks its ray; consecutive samples in one cell share a lookup and an atomic
//   pass 3  mw_gate (count/scatter) remove iff !(rays < 3 * hits), ordered compaction into the output
// The acos / sin of a node interval's slerp are computed on the host (glibc), once per interval; the per-run sin of the
// interpolation factor is the device's (DESIGN §4).
//
// X-ray stages (final pass only, every stage in one read of the output points, in chunks of kXrayChunk points):
//   mw_xray_check     every stage's cell inside +-8192, before anything changes
//   mw_xray_insert    per stage: claim the voxel key (64-bit CAS), count the point in its column and, if the voxel is new, the
//                     column's occupied voxels (integer atomics), extend the bounding box (warp min / max, then integer atomics);
//                     for a stage with colours, one (stage, column slot) sort key per point
//   stable radix sort of the keys (values: point indices), then mw_xray_fold: one thread per column adds its points' colours
//                     in stream order onto the column's float sums, which is the reference's order of float additions
//   mw_xray_pixels    IntoImage after the final flush, with log(n) from a host-built glibc table
#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstring>
#include <map>
#include <mutex>
#include <vector>

#include <cub/cub.cuh>

#include "dl_internal.cuh"
#include "dl_pipeline.cuh"

using namespace dl;

namespace {

constexpr int kBlock = 256;
constexpr int kGridHalf = 8192;  // 64 << 8 cells per axis at the largest extent the reference's grid grows to (bits = 8)
constexpr unsigned long long kEmpty = ~0ull;

struct NodeRec {          // node i of a trajectory, and the slerp constants of the interval (i - 1, i), computed on the host
  Rigidd pose;
  SlerpConstants slerp;
};
struct TrajRec {
  int64_t first, count;   // nodes [first, first + count) of the writer's node arrays
};
struct MsgRec {
  int64_t stamp, first_row, voff;  // voff: first virtual row of the message
  int32_t slot, frame;
  Rigidd sensor_to_tracking;
};
struct RunPose {
  Rigidf sensor_to_map;
  int32_t valid;
};
enum Counter { kNoPose = 0, kRange = 1, kSamples = 2, kOutside = 3, kNumCounters = 4 };

struct SelectArgs {
  const float4* rows;
  int64_t num_rows;          // bound of the call's row buffer
  const MsgRec* msgs;
  int num_msgs;
  int64_t n;                 // virtual rows
  const int64_t* times;      // the writer's node tables
  const NodeRec* nodes;
  const TrajRec* trajs;
  int32_t* head_tiles;       // per tile: run heads, then their exclusive prefix
  int32_t* num_runs;
  int32_t* run_of_row;
  RunPose* runs;
  int32_t* msg_last_run;     // -1: no kept point
  float* origins;            // 3 per message
  int range_filter;
  double min_range, max_range;
  int32_t* keep_tiles;
  int32_t* num_keep;
  float4* compact;           // x y z + message index (bits) of every kept point, in order
  float* out_xyz;            // or x y z only, straight into the output
  int32_t* out_msg;          // with out_xyz, optional: the message of every output point (the X-ray stages' colours)
  int check_extent;
  float resolution;
  unsigned long long* counters;
};

struct Table {
  unsigned long long* keys;
  int32_t* hits;
  int32_t* rays;
  float4* sums;              // optional per-slot payload (the X-ray table's column colour sums), moved by the rehash
  int64_t mask;
  int shift;
  int32_t* num_cells;
};
// The owners behind a Table, which kernels take by value.
struct TableBuffers {
  DeviceBuffer<unsigned long long> keys;
  DeviceBuffer<int32_t> hits, rays, num_cells;
  DeviceBuffer<float4> sums;
  Table view() const {
    int shift = 64;
    for (size_t c = keys.cap; c > 1; c >>= 1) --shift;
    return Table{keys.get(), hits.get(), rays.get(), sums.get(), (int64_t)keys.cap - 1, shift, num_cells.get()};
  }
};

__device__ __forceinline__ int message_of(const MsgRec* msgs, int num_msgs, int64_t v) {
  int lo = 0, hi = num_msgs;  // last message with voff <= v (empty messages share the next one's voff)
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (msgs[mid].voff <= v) lo = mid; else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ int block_inclusive_scan(int value, int* total) {
  __shared__ int warp_sums[kBlock / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int inc = value;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int o = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc += o;
  }
  __syncthreads();
  if (lane == 31) warp_sums[warp] = inc;
  __syncthreads();
  int base = 0, sum = 0;
#pragma unroll
  for (int w = 0; w < kBlock / 32; ++w) {
    if (w < warp) base += warp_sums[w];
    sum += warp_sums[w];
  }
  *total = sum;
  return base + inc;
}

// exclusive prefix of per-tile counts in place (one CTA), total -> *total
__global__ void __launch_bounds__(kBlock) mw_tile_prefix(int32_t* counts, int tiles, int32_t* total) {
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < tiles; base += kBlock) {
    const int t = base + threadIdx.x;
    const int v = t < tiles ? counts[t] : 0;
    int sum;
    const int inc = block_inclusive_scan(v, &sum);
    if (t < tiles) counts[t] = carry + inc - v;
    __syncthreads();
    if (threadIdx.x == 0) carry += sum;
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = carry;
}

struct RowRef {
  int m;
  float4 p;
  bool head;
};
__device__ __forceinline__ RowRef row_ref(const SelectArgs& a, int64_t v) {
  RowRef r;
  r.m = message_of(a.msgs, a.num_msgs, v);
  const MsgRec& msg = a.msgs[r.m];
  const int64_t row = msg.first_row + (v - msg.voff);
  r.p = a.rows[row];
  r.head = v == msg.voff || __float_as_uint(a.rows[row - 1].w) != __float_as_uint(r.p.w);
  return r;
}

__global__ void __launch_bounds__(kBlock) mw_heads_count(SelectArgs a) {
  const int64_t v = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  const bool head = v < a.n && row_ref(a, v).head;
  const int c = __syncthreads_count(head);
  if (threadIdx.x == 0) a.head_tiles[blockIdx.x] = c;
}

// TransformInterpolationBuffer::Has + Lookup (transform_interpolation_buffer.cc:45-66) and Interpolate
// (timestamped_transform.cc:22-37): lower_bound over the node times, an exact tick returns the node's pose unchanged.
__device__ bool lookup(const int64_t* times, const NodeRec* nodes, int64_t count, int64_t tick, Rigidd* out) {
  if (count == 0 || tick < times[0] || tick > times[count - 1]) return false;
  int64_t lo = 0, hi = count;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (times[mid] < tick) lo = mid + 1; else hi = mid;
  }
  const NodeRec& e = nodes[lo];
  if (times[lo] == tick) {
    *out = e.pose;
    return true;
  }
  const NodeRec& s = nodes[lo - 1];
  const double duration = (double)(times[lo] - times[lo - 1]) / 1e7;  // common::ToSeconds
  const double factor = ((double)(tick - times[lo - 1]) / 1e7) / duration;
  out->t = {s.pose.t.x + (e.pose.t.x - s.pose.t.x) * factor, s.pose.t.y + (e.pose.t.y - s.pose.t.y) * factor,
            s.pose.t.z + (e.pose.t.z - s.pose.t.z) * factor};
  out->q = slerp(s.pose.q, e.pose.q, factor, e.slerp);  // theta and sin(theta) of the interval come from the host
  return true;
}

__global__ void __launch_bounds__(kBlock) mw_run_poses(SelectArgs a) {
  const int64_t v = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  RowRef r{};
  if (v < a.n) r = row_ref(a, v);
  int total;
  const int inc = block_inclusive_scan(r.head ? 1 : 0, &total);
  if (v >= a.n) return;
  const int run = a.head_tiles[blockIdx.x] + inc - 1;
  a.run_of_row[v] = run;
  if (!r.head) return;
  const MsgRec& msg = a.msgs[r.m];
  // FromSeconds: duration_cast of double seconds to int64 ticks, truncation toward zero
  const int64_t tick = msg.stamp + (int64_t)((double)r.p.w * 1e7);
  const TrajRec tr = a.trajs[msg.slot];
  Rigidd tracking_to_map;
  RunPose out{};
  if (lookup(a.times + tr.first, a.nodes + tr.first, tr.count, tick, &tracking_to_map)) {
    out.sensor_to_map = to_float(compose(tracking_to_map, msg.sensor_to_tracking));
    out.valid = 1;
    atomicMax(a.msg_last_run + r.m, run);
  }
  a.runs[run] = out;
}

// origin = sensor_to_map * Vector3f::Zero() of the message's last kept point
__global__ void mw_origins(SelectArgs a) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= a.num_msgs) return;
  const int run = a.msg_last_run[m];
  Vec3f o{__int_as_float(0x7fc00000), __int_as_float(0x7fc00000), __int_as_float(0x7fc00000)};
  if (run >= 0) o = apply(a.runs[run].sensor_to_map, Vec3f{0.f, 0.f, 0.f});
  a.origins[3 * m] = o.x;
  a.origins[3 * m + 1] = o.y;
  a.origins[3 * m + 2] = o.z;
}

__device__ __forceinline__ bool in_extent(const Int3& c) {
  return c.x >= -kGridHalf && c.x < kGridHalf && c.y >= -kGridHalf && c.y < kGridHalf && c.z >= -kGridHalf && c.z < kGridHalf;
}
__device__ __forceinline__ unsigned long long cell_key(const Int3& c) {
  return ((unsigned long long)(c.x + kGridHalf) << 28) | ((unsigned long long)(c.y + kGridHalf) << 14) |
         (unsigned long long)(c.z + kGridHalf);
}
__device__ __forceinline__ int64_t slot_of(const Table& t, unsigned long long key) {
  return (int64_t)((key * 0x9E3779B97F4A7C15ull) >> t.shift);
}

// kind 0: count kept rows per tile; kind 1: scatter them in order (compact list and / or x y z output)
template <int kind>
__global__ void __launch_bounds__(kBlock) mw_select(SelectArgs a) {
  const int64_t v = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  bool keep = false, no_pose = false, out_of_range = false, outside = false;
  Vec3f q{};
  int m = 0;
  if (v < a.n) {
    m = message_of(a.msgs, a.num_msgs, v);
    const MsgRec& msg = a.msgs[m];
    const float4 p = a.rows[msg.first_row + (v - msg.voff)];
    const RunPose pose = a.runs[a.run_of_row[v]];
    if (!pose.valid) {
      no_pose = true;
    } else {
      q = apply(pose.sensor_to_map, Vec3f{p.x, p.y, p.z});
      keep = true;
      if (a.range_filter) {
        const Vec3f o{a.origins[3 * m], a.origins[3 * m + 1], a.origins[3 * m + 2]};
        const double range = (double)norm3(sub(q, o));
        if (!(a.min_range <= range && range <= a.max_range)) {
          keep = false;
          out_of_range = true;
        }
      }
      // Pass 1 also checks the batch origin: with both ends of every ray inside the extent a ray is at most ~28 400 voxels
      // long, so pass 2's float step x += voxel_size always advances (a far origin would stall it and loop forever).
      if (keep && kind == 0 && a.check_extent)
        outside = !in_extent(cell_index(q, a.resolution)) ||
                  !in_extent(cell_index(Vec3f{a.origins[3 * m], a.origins[3 * m + 1], a.origins[3 * m + 2]}, a.resolution));
    }
  }
  if (kind == 0) {
    const int c = __syncthreads_count(keep);
    const int c_no_pose = __syncthreads_count(no_pose);
    const int c_range = __syncthreads_count(out_of_range);
    const int c_outside = __syncthreads_count(outside);
    if (threadIdx.x == 0) {
      a.keep_tiles[blockIdx.x] = c;
      if (c_no_pose) atomicAdd(a.counters + kNoPose, (unsigned long long)c_no_pose);
      if (c_range) atomicAdd(a.counters + kRange, (unsigned long long)c_range);
      if (c_outside) atomicAdd(a.counters + kOutside, (unsigned long long)c_outside);
    }
    return;
  }
  int total;
  const int inc = block_inclusive_scan(keep ? 1 : 0, &total);
  if (!keep) return;
  const int64_t pos = (int64_t)a.keep_tiles[blockIdx.x] + inc - 1;
  if (a.compact) a.compact[pos] = make_float4(q.x, q.y, q.z, __int_as_float(m));
  if (a.out_xyz) {
    a.out_xyz[3 * pos] = q.x;
    a.out_xyz[3 * pos + 1] = q.y;
    a.out_xyz[3 * pos + 2] = q.z;
    if (a.out_msg) a.out_msg[pos] = m;
  }
}

// the slot of `key`, inserting it if absent (*fresh: this thread's CAS inserted it)
__device__ __forceinline__ int64_t claim(const Table& t, unsigned long long key, bool* fresh) {
  *fresh = false;
  for (int64_t s = slot_of(t, key);; s = (s + 1) & t.mask) {
    unsigned long long k = t.keys[s];
    if (k == kEmpty) {
      k = atomicCAS(t.keys + s, kEmpty, key);
      if (k == kEmpty) {
        atomicAdd(t.num_cells, 1);
        *fresh = true;
        return s;
      }
    }
    if (k == key) return s;
  }
}

// pass 1: ++hits of every kept point's cell (ProcessInPhaseOne)
__global__ void __launch_bounds__(kBlock) mw_insert_hits(Table t, const float4* pts, int64_t n, float resolution) {
  const int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  const float4 p = pts[i];
  bool fresh;
  atomicAdd(t.hits + claim(t, cell_key(cell_index(Vec3f{p.x, p.y, p.z}, resolution)), &fresh), 1);
}

__device__ __forceinline__ int64_t find(const Table& t, unsigned long long key) {
  for (int64_t s = slot_of(t, key);; s = (s + 1) & t.mask) {
    const unsigned long long k = t.keys[s];
    if (k == key) return s;
    if (k == kEmpty) return -1;
  }
}

// table growth: every cell moves to the larger table with its counts
__global__ void __launch_bounds__(kBlock) mw_rehash(Table to, Table from, int64_t from_cap) {
  const int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  if (i >= from_cap) return;
  const unsigned long long key = from.keys[i];
  if (key == kEmpty) return;
  int64_t s = slot_of(to, key);
  while (atomicCAS(to.keys + s, kEmpty, key) != kEmpty) s = (s + 1) & to.mask;
  to.hits[s] = from.hits[i];
  to.rays[s] = from.rays[i];
  if (to.sums) to.sums[s] = from.sums[i];
}

// pass 2 (ProcessInPhaseTwo): samples at x = 0, voxel_size, ... (< length, x a float advanced in double) along the ray from the
// batch origin; a sample's cell gains a ray if it has hits. Consecutive samples in one cell are counted with one lookup.
__global__ void __launch_bounds__(kBlock) mw_rays(Table t, const float4* pts, int64_t n, const float* origins, float resolution,
                                                  double voxel_size, unsigned long long* counters) {
  const int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  long long samples = 0;
  if (i < n) {
    const float4 p = pts[i];
    const int m = __float_as_int(p.w);
    const Vec3f o{origins[3 * m], origins[3 * m + 1], origins[3 * m + 2]};
    const Vec3f delta = sub(Vec3f{p.x, p.y, p.z}, o);
    const float length = norm3(delta);
    const CellDivider div = make_divider(resolution);
    unsigned long long run_key = kEmpty;
    int run_count = 0;
    for (float x = 0.f; x < length; x = (float)((double)x + voxel_size)) {
      ++samples;
      const float s = x / length;
      const Int3 c = cell_index(add(o, mul(s, delta)), div);
      const unsigned long long key = in_extent(c) ? cell_key(c) : kEmpty;  // beyond the extent: reads 0 hits
      if (key != run_key) {
        if (run_count > 0 && run_key != kEmpty) {
          const int64_t slot = find(t, run_key);
          if (slot >= 0) atomicAdd(t.rays + slot, run_count);
        }
        run_key = key;
        run_count = 0;
      }
      ++run_count;
    }
    if (run_count > 0 && run_key != kEmpty) {
      const int64_t slot = find(t, run_key);
      if (slot >= 0) atomicAdd(t.rays + slot, run_count);
    }
  }
  // block sum of the sample counts, one 64-bit integer atomic per block
  __shared__ long long warp_sums[kBlock / 32];
  for (int d = 16; d > 0; d >>= 1) samples += __shfl_down_sync(0xffffffffu, samples, d);
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = samples;
  __syncthreads();
  if (threadIdx.x == 0) {
    long long s = 0;
    for (int w = 0; w < kBlock / 32; ++w) s += warp_sums[w];
    if (s) atomicAdd(counters + kSamples, (unsigned long long)s);
  }
}

// pass 3 (ProcessInPhaseThree): keep iff rays < 3 * hits (kMissPerHitLimit, compared in double); kind 0 counts, 1 scatters
template <int kind>
__global__ void __launch_bounds__(kBlock) mw_gate(Table t, const float4* pts, int64_t n, float resolution, int32_t* tiles,
                                                  float* out_xyz, int32_t* out_msg) {
  const int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  bool keep = false;
  float4 p{};
  if (i < n) {
    p = pts[i];
    const Int3 c = cell_index(Vec3f{p.x, p.y, p.z}, resolution);
    int hits = 0, rays = 0;
    const int64_t slot = in_extent(c) ? find(t, cell_key(c)) : -1;
    if (slot >= 0) {
      hits = t.hits[slot];
      rays = t.rays[slot];
    }
    keep = (double)rays < 3.0 * (double)hits;
  }
  if (kind == 0) {
    const int c = __syncthreads_count(keep);
    if (threadIdx.x == 0) tiles[blockIdx.x] = c;
    return;
  }
  int total;
  const int inc = block_inclusive_scan(keep ? 1 : 0, &total);
  if (!keep) return;
  const int64_t pos = (int64_t)tiles[blockIdx.x] + inc - 1;
  out_xyz[3 * pos] = p.x;
  out_xyz[3 * pos + 1] = p.y;
  out_xyz[3 * pos + 2] = p.z;
  if (out_msg) out_msg[pos] = __float_as_int(p.w);
}

// ---- X-ray stages. Keys of the X-ray table: bit 46 voxel (1) or column (0), bits 42..45 the stage, bits 0..41 cell_key(x, y, z)
// (x = -kGridHalf for a column). Per column slot: hits = points, rays = occupied voxels, sums = colour sums (r, g, b).
constexpr int kMaxStages = DL_MAP_WRITER_MAX_STAGES;
constexpr unsigned long long kVoxelBit = 1ull << 46;
constexpr int kLogTable = 2 * kGridHalf;     // a column holds at most 16384 distinct voxels
constexpr int64_t kXrayChunk = 1 << 21;      // points per insert: bounds the table's growth per reservation

struct XrayStage {
  Rigidf transform;
  float resolution;
  int32_t num_colors;        // colour stages added before this stage: colors[0, num_colors)
  int32_t sum_index;         // index among the stages with colours, -1 for a stage without (its sums stay 0)
};
struct ColorStage {
  int32_t frame;
  float r, g, b;             // Uint8ComponentToFloat
};
struct XrayArgs {
  const float* points;       // x y z of the final pass's output, in order
  const int32_t* point_msg;  // message of every point
  const MsgRec* msgs;
  int64_t first, n;          // points [first, first + n) of the call
  int num_stages;
  XrayStage stages[kMaxStages];
  ColorStage colors[kMaxStages];
  int32_t sum_stage[kMaxStages];  // stage of every sum_index
  int32_t* bbox;             // 6 per stage: min x y z, max x y z
  unsigned long long* sort_keys;  // [sum_index * n + i]: sum_index << slot_bits | column slot
  int32_t* sort_vals;        // point index
  int slot_bits;
  unsigned long long* outside;
};

__device__ __forceinline__ Int3 xray_cell(const XrayStage& s, float x, float y, float z) {
  return cell_index(apply(s.transform, Vec3f{x, y, z}), s.resolution);
}

__global__ void __launch_bounds__(kBlock) mw_xray_check(XrayArgs a) {
  const int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  bool outside = false;
  if (i < a.n) {
    const float* p = a.points + 3 * (a.first + i);
    for (int s = 0; s < a.num_stages; ++s) outside |= !in_extent(xray_cell(a.stages[s], p[0], p[1], p[2]));
  }
  const int c = __syncthreads_count(outside);
  if (threadIdx.x == 0 && c) atomicAdd(a.outside, (unsigned long long)c);
}

__global__ void __launch_bounds__(kBlock) mw_xray_insert(Table t, XrayArgs a) {
  const int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  const bool active = i < a.n;
  float x = 0.f, y = 0.f, z = 0.f;
  if (active) {
    const float* p = a.points + 3 * (a.first + i);
    x = p[0]; y = p[1]; z = p[2];
  }
  for (int s = 0; s < a.num_stages; ++s) {
    Int3 c{INT_MAX, INT_MAX, INT_MAX}, d{INT_MIN, INT_MIN, INT_MIN};
    if (active) {
      c = xray_cell(a.stages[s], x, y, z);
      d = c;
      const unsigned long long stage = (unsigned long long)s << 42;
      bool fresh_voxel, fresh_column;
      claim(t, kVoxelBit | stage | cell_key(c), &fresh_voxel);
      const int64_t col = claim(t, stage | cell_key(Int3{-kGridHalf, c.y, c.z}), &fresh_column);
      atomicAdd(t.hits + col, 1);
      if (fresh_voxel) atomicAdd(t.rays + col, 1);
      const int k = a.stages[s].sum_index;
      if (k >= 0) {
        a.sort_keys[k * a.n + i] = ((unsigned long long)k << a.slot_bits) | (unsigned long long)col;
        a.sort_vals[k * a.n + i] = (int32_t)i;
      }
    }
    // Eigen::AlignedBox3i::extend: integer min / max, one atomic per warp and bound
    const int lo[3] = {__reduce_min_sync(0xffffffffu, c.x), __reduce_min_sync(0xffffffffu, c.y), __reduce_min_sync(0xffffffffu, c.z)};
    const int hi[3] = {__reduce_max_sync(0xffffffffu, d.x), __reduce_max_sync(0xffffffffu, d.y), __reduce_max_sync(0xffffffffu, d.z)};
    if ((threadIdx.x & 31) == 0 && lo[0] != INT_MAX) {
      int32_t* box = a.bbox + 6 * s;
      for (int k = 0; k < 3; ++k) {
        atomicMin(box + k, lo[k]);
        atomicMax(box + 3 + k, hi[k]);
      }
    }
  }
}

// the colour stage `s` gives a point of frame `frame`: the last matching colour stage before it, else kDefaultColor
__device__ __forceinline__ float4 point_color(const XrayArgs& a, int s, int32_t frame) {
  for (int c = a.stages[s].num_colors - 1; c >= 0; --c)
    if (a.colors[c].frame == frame) return make_float4(a.colors[c].r, a.colors[c].g, a.colors[c].b, 0.f);
  return make_float4(0.f, 0.f, 0.f, 0.f);
}

// one thread per run of equal sorted keys (one column of one stage): the run's points in stream order onto the float sums
__global__ void __launch_bounds__(kBlock) mw_xray_fold(Table t, XrayArgs a, const unsigned long long* keys, const int32_t* vals,
                                                       int64_t count) {
  const int64_t j = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  if (j >= count || (j > 0 && keys[j - 1] == keys[j])) return;
  const unsigned long long key = keys[j];
  const int64_t slot = (int64_t)(key & ((1ull << a.slot_bits) - 1));
  const int s = a.sum_stage[key >> a.slot_bits];
  float4 sum = t.sums[slot];
  for (int64_t k = j; k < count && keys[k] == key; ++k) {
    const float4 c = point_color(a, s, a.msgs[a.point_msg[a.first + vals[k]]].frame);
    sum.x += c.x;
    sum.y += c.y;
    sum.z += c.z;
  }
  t.sums[slot] = sum;
}

__global__ void __launch_bounds__(kBlock) mw_xray_max_voxels(Table t, int64_t cap, int stage, int32_t* max_voxels) {
  const int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  int v = 0;
  if (i < cap) {
    const unsigned long long key = t.keys[i];
    if (key != kEmpty && !(key & kVoxelBit) && (int)((key >> 42) & 15) == stage) v = t.rays[i];
  }
  v = __reduce_max_sync(0xffffffffu, v);
  if ((threadIdx.x & 31) == 0 && v) atomicMax(max_voxels, v);
}

// Mix (xray_points_processor.cc): a * (1. - t) in double, t * b in float, the sum in double, returned as float
__device__ __forceinline__ float mix(float a, float b, float t) { return (float)((double)a * (1.0 - (double)t) + (double)(t * b)); }
// FloatComponentToUint8: lround(Clamp(c, 0.f, 1.f) * 255), the product in float
__device__ __forceinline__ uint32_t to_uint8(float c) {
  const float v = c > 1.f ? 1.f : (c < 0.f ? 0.f : c);
  return (uint32_t)(uint8_t)lroundf(v * 255.f);
}

// IntoImage: one thread per slot; the column pixels of the stage (the image starts white: empty columns)
__global__ void __launch_bounds__(kBlock) mw_xray_pixels(Table t, int64_t cap, int stage, const double* log_n, float max_log,
                                                         int max_y, int max_z, int width, uint32_t* argb) {
  const int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  if (i >= cap) return;
  const unsigned long long key = t.keys[i];
  if (key == kEmpty || (key & kVoxelBit) || (int)((key >> 42) & 15) != stage) return;
  const int y = (int)((key >> 14) & 0x3fff) - kGridHalf, z = (int)(key & 0x3fff) - kGridHalf;
  const float count = (float)(uint32_t)t.hits[i];
  const float4 sum = t.sums[i];
  const float saturation = (float)(log_n[t.rays[i]] / (double)max_log);
  const uint32_t r = to_uint8(mix(1.f, sum.x / count, saturation));
  const uint32_t g = to_uint8(mix(1.f, sum.y / count, saturation));
  const uint32_t b = to_uint8(mix(1.f, sum.z / count, saturation));
  argb[(int64_t)(max_z - z) * width + (max_y - y)] = 0xFF000000u | r << 16 | g << 8 | b;  // Uint8ColorToCairo
}

// ---- Probability-grid stages (write_probability_grid, write_ros_map). Cells are uint16 correspondence-cost values without the
// update marker; a per-cell 32-bit stamp replaces it: batch k (counted from 1 over the writer's life) claims a cell with
// atomicMax(stamp, 2k + 1) for a hit and 2k for a walk, and the claimer that lifts the stamp past 2k - 1 applies the table once.
// Hits run in one launch before the walks, so a hit wins over every miss of its batch and no FinishUpdate pass is needed.
constexpr int kSubpixel = 1000;              // ray_casting.cc kSubpixelScale
constexpr int kGridBoxChunk = 32;            // points per lane of mw_grid_boxes

// Per message of a call: the float box of its output points' x y as order-preserving keys, and its first / last output point.
struct GridBoxes {
  uint32_t* keys;            // 4 per message: ~key of min x, min y, key of max x, max y (0: no point)
  int32_t* first;            // per message: first and last output point (first = INT_MAX: no point)
  int32_t* last;
  unsigned long long* nonfinite;
};

__device__ __forceinline__ uint32_t float_key(float f) {
  const uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// one warp per 32 * kGridBoxChunk consecutive points, lane l takes every 32nd; runs of one message are reduced per lane, then
// per warp when every lane holds the same message
__global__ void __launch_bounds__(kBlock) mw_grid_boxes(const float* pts, const int32_t* msg, int64_t n, GridBoxes b) {
  const int lane = threadIdx.x & 31;
  const int64_t base = ((int64_t)blockIdx.x * kBlock + (threadIdx.x & ~31)) * kGridBoxChunk;
  int cur = -1, first = INT_MAX, last = -1;
  uint32_t lo_x = ~0u, lo_y = ~0u, hi_x = 0, hi_y = 0;
  bool bad = false;
  auto flush = [&](bool warp_wide) {
    if (warp_wide) {
      lo_x = __reduce_min_sync(0xffffffffu, lo_x);
      lo_y = __reduce_min_sync(0xffffffffu, lo_y);
      hi_x = __reduce_max_sync(0xffffffffu, hi_x);
      hi_y = __reduce_max_sync(0xffffffffu, hi_y);
      first = __reduce_min_sync(0xffffffffu, first);
      last = __reduce_max_sync(0xffffffffu, last);
      if (lane != 0) return;
    }
    if (cur < 0) return;
    atomicMax(b.keys + 4 * cur, ~lo_x);
    atomicMax(b.keys + 4 * cur + 1, ~lo_y);
    atomicMax(b.keys + 4 * cur + 2, hi_x);
    atomicMax(b.keys + 4 * cur + 3, hi_y);
    atomicMin(b.first + cur, first);
    atomicMax(b.last + cur, last);
  };
  for (int k = 0; k < kGridBoxChunk; ++k) {
    const int64_t i = base + (int64_t)k * 32 + lane;
    if (i >= n) break;
    const int m = msg[i];
    if (m != cur) {
      flush(false);
      cur = m;
      first = INT_MAX; last = -1;
      lo_x = ~0u; lo_y = ~0u; hi_x = 0; hi_y = 0;
    }
    const float x = pts[3 * i], y = pts[3 * i + 1];
    if (!isfinite(x) || !isfinite(y)) {
      bad = true;
      continue;
    }
    first = min(first, (int)i);
    last = (int)i;
    lo_x = min(lo_x, float_key(x)); lo_y = min(lo_y, float_key(y));
    hi_x = max(hi_x, float_key(x)); hi_y = max(hi_y, float_key(y));
  }
  flush(__all_sync(0xffffffffu, cur == __shfl_sync(0xffffffffu, cur, 0)));
  const unsigned bad_lanes = __ballot_sync(0xffffffffu, bad);
  if (lane == 0 && bad_lanes) atomicAdd(b.nonfinite, (unsigned long long)__popc(bad_lanes));
}

// One batch of one grid stage, at the batch's own limits; cells land at (x + off_x, y + off_y) of the allocated grid.
struct GridBatch {
  const float* pts;          // the batch's x y z points
  int32_t n;
  int32_t begin_x, begin_y;  // the origin's superscaled cell
  int32_t off_x, off_y;
  int32_t stride;            // num_x_cells of the allocated grid
  double max_x, max_y, resolution;  // the superscaled limits' max and resolution / 1000
  uint16_t* cells;
  uint32_t* stamps;
  const uint16_t* table;     // the hit or the miss table, without the update marker
  uint32_t claim;            // 2k + 1 (hits) or 2k (walks)
};

// ApplyLookupTable with the stamp in place of kUpdateMarker (a plain load first: most revisits near the origin stop there)
__device__ __forceinline__ void grid_visit(const GridBatch& g, int x, int y) {
  const int64_t idx = (int64_t)(y + g.off_y) * g.stride + (x + g.off_x);
  const uint32_t lowest = g.claim & ~1u;  // 2k: any claim of this batch
  if (*(volatile uint32_t*)(g.stamps + idx) >= lowest) return;
  if (atomicMax(g.stamps + idx, g.claim) < lowest) g.cells[idx] = __ldg(g.table + g.cells[idx]);
}

// MapLimits::GetCellIndex at the superscaled limits: the float promoted to double, IEEE division, lround
__device__ __forceinline__ int2 grid_end(const GridBatch& g, int i) {
  const double px = (double)g.pts[3 * i], py = (double)g.pts[3 * i + 1];
  return make_int2((int)llround((g.max_y - py) / g.resolution - 0.5), (int)llround((g.max_x - px) / g.resolution - 0.5));
}

__global__ void __launch_bounds__(kBlock) mw_grid_hits(GridBatch g) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= g.n) return;
  const int2 e = grid_end(g, i);
  grid_visit(g, e.x / kSubpixel, e.y / kSubpixel);
}

// CastRay (ray_casting.cc:29-146): x ascending, the vertical special case, int64 sub_y with the sub_y == denominator corner rule
__global__ void __launch_bounds__(kBlock) mw_grid_walks(GridBatch g) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= g.n) return;
  const int2 e = grid_end(g, i);
  int2 b = make_int2(g.begin_x, g.begin_y), end = e;
  if (b.x > end.x) {
    b = e;
    end = make_int2(g.begin_x, g.begin_y);
  }
  if (b.x / kSubpixel == end.x / kSubpixel) {
    const int x = b.x / kSubpixel, last = max(b.y, end.y) / kSubpixel;
    for (int y = min(b.y, end.y) / kSubpixel; y <= last; ++y) grid_visit(g, x, y);
    return;
  }
  const int64_t dx = end.x - b.x, dy = end.y - b.y, denominator = 2 * kSubpixel * dx;
  int cx = b.x / kSubpixel, cy = b.y / kSubpixel;
  int64_t sub_y = (2 * (b.y % kSubpixel) + 1) * dx;
  const int first_pixel = 2 * kSubpixel - 2 * (b.x % kSubpixel) - 1;
  const int last_pixel = 2 * (end.x % kSubpixel) + 1;
  const int end_x = end.x / kSubpixel;
  sub_y += dy * first_pixel;
  if (dy > 0) {
    while (true) {
      grid_visit(g, cx, cy);
      while (sub_y > denominator) {
        sub_y -= denominator;
        ++cy;
        grid_visit(g, cx, cy);
      }
      ++cx;
      if (sub_y == denominator) {
        sub_y -= denominator;
        ++cy;
      }
      if (cx == end_x) break;
      sub_y += dy * 2 * kSubpixel;
    }
    sub_y += dy * last_pixel;
    grid_visit(g, cx, cy);
    while (sub_y > denominator) {
      sub_y -= denominator;
      ++cy;
      grid_visit(g, cx, cy);
    }
    return;
  }
  while (true) {
    grid_visit(g, cx, cy);
    while (sub_y < 0) {
      sub_y += denominator;
      --cy;
      grid_visit(g, cx, cy);
    }
    ++cx;
    if (sub_y == 0) {
      sub_y += denominator;
      --cy;
    }
    if (cx == end_x) break;
    sub_y += dy * 2 * kSubpixel;
  }
  sub_y += dy * last_pixel;
  grid_visit(g, cx, cy);
  while (sub_y < 0) {
    sub_y += denominator;
    --cy;
    grid_visit(g, cx, cy);
  }
}

// The known-cells box: no table entry returns a cell to 0 (unknown), so it is the box of the cells != 0
__global__ void __launch_bounds__(kBlock) mw_grid_known_box(const uint16_t* cells, int nx, int64_t count, int32_t* box) {
  const int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  int x0 = INT_MAX, y0 = INT_MAX, x1 = INT_MIN, y1 = INT_MIN;
  if (i < count && cells[i] != 0) {
    x0 = x1 = (int)(i % nx);
    y0 = y1 = (int)(i / nx);
  }
  x0 = __reduce_min_sync(0xffffffffu, x0);
  y0 = __reduce_min_sync(0xffffffffu, y0);
  x1 = __reduce_max_sync(0xffffffffu, x1);
  y1 = __reduce_max_sync(0xffffffffu, y1);
  if ((threadIdx.x & 31) == 0 && x0 != INT_MAX) {
    atomicMin(box, x0);
    atomicMin(box + 1, y0);
    atomicMax(box + 2, x1);
    atomicMax(box + 3, y1);
  }
}

// the cropped box's cells and DrawProbabilityGrid's grey values (colour table indexed by the cell value)
__global__ void __launch_bounds__(kBlock) mw_grid_crop(const uint16_t* cells, int nx, int ox, int oy, int width, int64_t count,
                                                       const uint8_t* colors, uint16_t* out_cells, uint8_t* out_pixels) {
  const int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  if (i >= count) return;
  const int64_t x = i % width, y = i / width;
  const uint16_t v = cells[(oy + y) * (int64_t)nx + ox + x];
  out_cells[i] = v;
  out_pixels[i] = colors[v];
}

// std::log(double n) for n = 0 .. kLogTable, glibc's (through a volatile pointer, never the compiler's folding)
const std::vector<double>& log_table() {
  static std::vector<double> table;
  static std::once_flag once;
  std::call_once(once, [] {
    double (*volatile glibc_log)(double) = ::log;
    table.resize(kLogTable + 1);
    for (int n = 0; n <= kLogTable; ++n) table[n] = glibc_log((double)n);
  });
  return table;
}

// kValueToCorrespondenceCost (probability_values.cc:27-36, 59-63): SlowValueToBoundedFloat in float, host arithmetic
// (-ffp-contract=off)
float value_to_correspondence_cost(int value) {
  const float lo = 1.f - (1.f - 0.1f), hi = 1.f - 0.1f;  // kMinCorrespondenceCost, kMaxCorrespondenceCost
  if (value == 0) return hi;
  const float scale = (hi - lo) / 32766.f;
  return (float)value * scale + (lo - scale);
}
// CorrespondenceCostToValue (probability_values.h:32-44, 85-88)
uint16_t correspondence_cost_to_value(float c) {
  const float lo = 1.f - (1.f - 0.1f), hi = 1.f - 0.1f;
  const float clamped = c > hi ? hi : (c < lo ? lo : c);
  return (uint16_t)((int)lroundf((clamped - lo) * (32766.f / (hi - lo))) + 1);
}
// ComputeLookupTableToApplyCorrespondenceCostOdds(Odds((float)probability)) (probability_values.cc:85-100), without the update
// marker
void compute_correspondence_cost_table(double probability, uint16_t* table) {
  const float p = (float)probability;
  const float odds = p / (1.f - p);
  auto from_odds = [](float o) { return o / (o + 1.f); };
  table[0] = correspondence_cost_to_value(1.f - from_odds(odds));
  for (int cell = 1; cell != 32768; ++cell) {
    const float q = 1.f - value_to_correspondence_cost(cell);  // CorrespondenceCostToProbability
    table[cell] = correspondence_cost_to_value(1.f - from_odds(odds * (q / (1.f - q))));
  }
}
// DrawProbabilityGrid's grey value of every cell value: 128 if unknown, else ProbabilityToColor(GetProbability)
// (probability_grid_points_processor.cc:49-54, 137-146)
std::vector<uint8_t> grid_color_table() {
  std::vector<uint8_t> colors(32768);
  colors[0] = 128;
  for (int v = 1; v < 32768; ++v) {
    const float p = 1.f - value_to_correspondence_cost(v);
    const float probability = 1.f - p;
    colors[v] = (uint8_t)(int)lroundf(255 * ((probability - 0.1f) / ((1.f - 0.1f) - 0.1f)));
  }
  return colors;
}

struct GridLimits {          // MapLimits: max (double), cell counts
  double max_x, max_y;
  int32_t nx, ny;
};
struct GridStage {
  double resolution;
  int32_t insert_free_space;
  GridLimits limits;         // after the last call
  DeviceBuffer<uint16_t> cells;   // allocated at `limits` once a batch arrived (before that every cell is unknown)
  DeviceBuffer<uint32_t> stamps;
  DeviceBuffer<uint16_t> tables;  // hit [0, 32768), miss [32768, 65536)
  int64_t batches = 0;       // k of the last batch
};
// One call's growth of one stage, decided before anything changes: every batch's limits and cell offset in the grid of the
// call's final limits, and the new buffers when the grid grows (or is first allocated).
struct GridPlan {
  GridLimits final_limits;
  std::vector<GridLimits> at;
  std::vector<int2> offset;
  int32_t grow_x = 0, grow_y = 0;  // where the previous content lands
  DeviceBuffer<uint16_t> cells;
  DeviceBuffer<uint32_t> stamps;
};

// MapLimits::GetCellIndex (map_limits.h:69-76)
void grid_cell_index(const GridLimits& l, double resolution, float px, float py, long* x, long* y) {
  *x = std::lround((l.max_y - (double)py) / resolution - 0.5);
  *y = std::lround((l.max_x - (double)px) / resolution - 0.5);
}
// Grid2D::GrowLimits (grid_2d.cc:116-145) on the limits alone; false where a doubling would pass DL_MAP_WRITER_MAX_GRID_CELLS.
// (*add_x, *add_y) accumulate the translation of the cells.
bool grid_grow_limits(GridLimits* l, double resolution, float px, float py, int32_t* add_x, int32_t* add_y) {
  for (;;) {
    long x, y;
    grid_cell_index(*l, resolution, px, py, &x, &y);
    if (x >= 0 && y >= 0 && x < l->nx && y < l->ny) return true;
    if (2 * (int64_t)l->nx > DL_MAP_WRITER_MAX_GRID_CELLS || 2 * (int64_t)l->ny > DL_MAP_WRITER_MAX_GRID_CELLS) return false;
    const int32_t xo = l->nx / 2, yo = l->ny / 2;
    l->max_x = l->max_x + resolution * (double)yo;
    l->max_y = l->max_y + resolution * (double)xo;
    l->nx *= 2;
    l->ny *= 2;
    *add_x += xo;
    *add_y += yo;
  }
}
float key_float(uint32_t k) {
  const uint32_t b = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  float f;
  std::memcpy(&f, &b, sizeof(f));
  return f;
}

unsigned tiles_of(int64_t n) { return (unsigned)((n + kBlock - 1) / kBlock); }

}  // namespace

struct dl_map_writer {
  dl_context* ctx = nullptr;
  dl_map_writer_options options{};
  float resolution = 0.f;          // (float)outlier_voxel_size: HybridGridBase's float resolution
  std::map<int32_t, int32_t> slot_of;  // trajectory id -> slot
  std::vector<TrajRec> trajs;
  std::vector<int64_t> times;
  std::vector<NodeRec> nodes;
  bool tables_dirty = false;
  DeviceBuffer<int64_t> d_times;
  DeviceBuffer<NodeRec> d_nodes;
  DeviceBuffer<TrajRec> d_trajs;
  int pass = 0;                    // 0 .. num_passes - 1
  bool started = false, finished = false;
  DeviceBuffer<RunPose> d_runs;
  TableBuffers table;              // cell -> (hits, rays)
  int64_t num_cells = 0;
  // X-ray and colour stages, in pipeline order
  std::vector<XrayStage> xrays;
  std::vector<ColorStage> colors;
  std::vector<int32_t> sum_stage;  // stage of every sum_index
  TableBuffers xray;               // voxel and column keys of every X-ray stage (see the key layout above), with colour sums
  int64_t xray_entries = 0;
  DeviceBuffer<int32_t> d_bbox;    // 6 per stage
  DeviceBuffer<double> d_log;      // log_table()
  // probability-grid stages, in the order they were added
  std::vector<GridStage> grids;
  DeviceBuffer<uint8_t> d_grid_colors;  // grid_color_table()
  struct GridCall {                // the batches of one final-pass call and every stage's plan
    std::vector<int32_t> first, count;
    std::vector<float> origins;    // x y per batch
    std::vector<GridPlan> plans;
  };

  int num_passes() const { return options.outlier_voxel_size > 0 ? 3 : 1; }
  int num_stages() const { return (int)(xrays.size() + colors.size() + grids.size()); }
  bool final_pass() const { return pass == num_passes() - 1; }

  int upload_tables() {
    if (!tables_dirty) return DL_OK;
    const size_t nn = std::max<size_t>(nodes.size(), 1), nt = std::max<size_t>(trajs.size(), 1);
    DL_TRY(grow(ctx, d_times, nn));
    DL_TRY(grow(ctx, d_nodes, nn));
    DL_TRY(grow(ctx, d_trajs, nt));
    DL_TRY(h2d(ctx, d_times.get(), times.data(), times.size()));
    DL_TRY(h2d(ctx, d_nodes.get(), nodes.data(), nodes.size()));
    DL_TRY(h2d(ctx, d_trajs.get(), trajs.data(), trajs.size()));
    tables_dirty = false;
    return DL_OK;
  }
  int reserve_runs(int64_t n) {
    if (n <= (int64_t)d_runs.cap) return DL_OK;
    return grow(ctx, d_runs, (size_t)std::max<int64_t>({n, 2 * (int64_t)d_runs.cap, 4096}));
  }
  // Load factor <= 1/2 after `adding` more entries: sized from a count of the points about to be inserted.
  int reserve_table(TableBuffers* t, int64_t used, int64_t adding, bool sums) {
    int64_t cap = 1024;
    while (cap < 2 * (used + adding)) cap <<= 1;
    const int64_t capacity = (int64_t)t->keys.cap;
    if (cap <= capacity) return DL_OK;
    TableBuffers fresh;
    DL_TRY(alloc(ctx, fresh.keys, (size_t)cap, 0xff));
    DL_TRY(alloc(ctx, fresh.hits, (size_t)cap, 0));
    DL_TRY(alloc(ctx, fresh.rays, (size_t)cap, 0));
    if (sums) DL_TRY(alloc(ctx, fresh.sums, (size_t)cap, 0));
    if (capacity > 0) {
      mw_rehash<<<tiles_of(capacity), kBlock, 0, ctx->stream>>>(fresh.view(), t->view(), capacity);
      DL_LAUNCH_CHECK(ctx, "mw_rehash");
    }
    DL_CUDA(ctx, ctx->wait_stream());
    fresh.num_cells = std::move(t->num_cells);
    *t = std::move(fresh);
    return DL_OK;
  }
  int insert_xray(const float* points, const int32_t* point_msg, const MsgRec* msgs, int64_t n, void* sort_scratch,
                  size_t sort_bytes, unsigned long long* keys, int32_t* vals, unsigned long long* outside);
  XrayArgs xray_args() const {
    XrayArgs a{};
    a.num_stages = (int)xrays.size();
    std::copy(xrays.begin(), xrays.end(), a.stages);
    std::copy(colors.begin(), colors.end(), a.colors);
    std::copy(sum_stage.begin(), sum_stage.end(), a.sum_stage);
    a.bbox = d_bbox.get();
    return a;
  }
  // the X-ray table, the bounding boxes and the log table, at the first X-ray stage
  int init_xray() {
    if (xray.num_cells.get()) return DL_OK;
    DL_CUDA(ctx, cudaSetDevice(ctx->device));
    std::vector<int32_t> box(6 * kMaxStages);
    for (int s = 0; s < kMaxStages; ++s)
      for (int k = 0; k < 3; ++k) {
        box[6 * s + k] = INT_MAX;
        box[6 * s + 3 + k] = INT_MIN;
      }
    const std::vector<double>& logs = log_table();
    DL_TRY(alloc(ctx, d_bbox, box.size()));
    DL_TRY(alloc(ctx, d_log, logs.size()));
    DL_TRY(h2d(ctx, d_bbox.get(), box.data(), box.size()));
    DL_TRY(h2d(ctx, d_log.get(), logs.data(), logs.size()));
    DL_TRY(sync(ctx));                         // `box` is pageable and local
    return alloc(ctx, xray.num_cells, 1, 0);  // last: the counter marks the X-ray state as made
  }
  int process(int32_t num_messages, const dl_map_message* messages, const float* rows_host, const float* rows_dev,
              int64_t num_rows, float* points_host, float* points_dev, int64_t* num_points_out, float* origins_out,
              dl_map_writer_info* info);
  int plan_grids(const float* points, const int32_t* point_msg, int64_t n, const float* origins, int num_messages,
                 const std::vector<int32_t>& last_run, const GridBoxes& boxes, GridCall* call);
  int apply_grids(const float* points, GridCall* call);
};

namespace {

bool valid_pose7(const double* p) {
  for (int k = 0; k < 7; ++k)
    if (!std::isfinite(p[k])) return false;
  return true;
}

}  // namespace

int dl_map_writer::process(int32_t num_messages, const dl_map_message* messages, const float* rows_host, const float* rows_dev,
                           int64_t num_rows, float* points_host, float* points_dev, int64_t* num_points_out, float* origins_out,
                           dl_map_writer_info* info) {
  if (!num_points_out || num_messages < 0 || (num_messages > 0 && !messages) || num_rows < 0)
    return ctx->fail(DL_ERR_ARG, "dl_map_writer_process: bad arguments");
  if (finished) return ctx->fail(DL_ERR_ARG, "dl_map_writer_process: the final pass was flushed");
  // validate every message before any work
  std::vector<MsgRec> msgs((size_t)std::max(num_messages, 1));
  int64_t n = 0;
  for (int32_t m = 0; m < num_messages; ++m) {
    const dl_map_message& g = messages[m];
    const auto it = slot_of.find(g.trajectory_id);
    if (it == slot_of.end()) return ctx->fail(DL_ERR_ARG, "dl_map_writer_process: unknown trajectory " + std::to_string(g.trajectory_id));
    if (g.first_row < 0 || g.num_rows < 0 || g.first_row > num_rows || g.num_rows > num_rows - g.first_row)
      return ctx->fail(DL_ERR_ARG, "dl_map_writer_process: message rows outside the row buffer");
    if (!valid_pose7(g.sensor_to_tracking)) return ctx->fail(DL_ERR_ARG, "dl_map_writer_process: sensor_to_tracking is not finite");
    msgs[m] = MsgRec{g.stamp, g.first_row, n, it->second, g.frame_id, pose_from7(g.sensor_to_tracking)};
    n += g.num_rows;
  }
  if (n >= (1ll << 31)) return ctx->fail(DL_ERR_ARG, "dl_map_writer_process: more than 2^31 - 1 rows in one call");
  if (n > 0 && !rows_host && !rows_dev) return ctx->fail(DL_ERR_ARG, "dl_map_writer_process: no rows");
  if (n > 0 && final_pass() && !points_host && !points_dev) return ctx->fail(DL_ERR_ARG, "dl_map_writer_process: no points_out");
  if (rows_dev && ((uintptr_t)rows_dev & 15) != 0) return ctx->fail(DL_ERR_ARG, "dl_map_writer_process: rows must be 16-byte aligned");
  *num_points_out = 0;
  dl_map_writer_info local{};
  local.pass = pass;
  local.final_pass = final_pass() ? 1 : 0;
  local.num_rows = n;
  local.messages_without_batch = num_messages;
  if (n == 0) {
    if (origins_out) for (int64_t k = 0; k < 3 * (int64_t)num_messages; ++k) origins_out[k] = NAN;
    started = true;
    if (info) *info = local;
    return DL_OK;
  }
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  DL_TRY(upload_tables());
  const unsigned tiles = tiles_of(n);
  SelectArgs a{};
  float4* up_rows = nullptr;
  MsgRec* d_msgs = nullptr;
  int32_t* d_ints = nullptr;  // [0] runs, [1] kept, [2] gate survivors
  float* d_out = nullptr;
  int32_t* gate_tiles = nullptr;
  // X-ray and grid stages: the message of every output point; X-ray stages: the sort of one chunk's (stage, column) keys
  const bool with_xray = final_pass() && !xrays.empty();
  const bool with_grid = final_pass() && !grids.empty();
  GridBoxes boxes{};
  const int64_t sort_items = with_xray ? std::min<int64_t>(n, kXrayChunk) * (int64_t)sum_stage.size() : 0;
  size_t sort_bytes = 0;
  if (sort_items > 0) {
    cub::DoubleBuffer<unsigned long long> k(nullptr, nullptr);
    cub::DoubleBuffer<int32_t> v(nullptr, nullptr);
    DL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, k, v, (int)sort_items, 0, 64, ctx->stream));
  }
  int32_t* out_msg = nullptr;
  unsigned long long* sort_keys = nullptr;
  int32_t* sort_vals = nullptr;
  void* sort_scratch = nullptr;
  DL_TRY(carve_scratch(ctx, [&](Arena& ar) {
    if (with_xray || with_grid) out_msg = ar.take<int32_t>((size_t)n);
    if (with_grid) {
      boxes.keys = ar.take<uint32_t>(4 * (size_t)num_messages);
      boxes.first = ar.take<int32_t>((size_t)num_messages);
      boxes.last = ar.take<int32_t>((size_t)num_messages);
      boxes.nonfinite = ar.take<unsigned long long>(1);
    }
    if (with_xray) {
      sort_keys = ar.take<unsigned long long>(2 * (size_t)sort_items);
      sort_vals = ar.take<int32_t>(2 * (size_t)sort_items);
      sort_scratch = ar.take<char>(sort_bytes);
    }
    if (rows_host) up_rows = ar.take<float4>((size_t)num_rows);
    d_msgs = ar.take<MsgRec>((size_t)num_messages);
    a.head_tiles = ar.take<int32_t>(tiles);
    a.keep_tiles = ar.take<int32_t>(tiles);
    gate_tiles = ar.take<int32_t>(tiles);
    a.run_of_row = ar.take<int32_t>((size_t)n);
    a.msg_last_run = ar.take<int32_t>((size_t)num_messages);
    a.origins = ar.take<float>(3 * (size_t)num_messages);
    a.counters = ar.take<unsigned long long>(kNumCounters);
    d_ints = ar.take<int32_t>(3);
    a.compact = ar.take<float4>((size_t)n);
    if (points_host) d_out = ar.take<float>(3 * (size_t)n);
  }));
  if (rows_host) {
    DL_CUDA(ctx, cudaMemcpyAsync(up_rows, rows_host, (size_t)num_rows * 16, cudaMemcpyHostToDevice, ctx->stream));
    a.rows = up_rows;
  } else {
    a.rows = reinterpret_cast<const float4*>(rows_dev);
  }
  if (!d_out) d_out = points_dev;
  DL_CUDA(ctx, cudaMemcpyAsync(d_msgs, msgs.data(), (size_t)num_messages * sizeof(MsgRec), cudaMemcpyHostToDevice, ctx->stream));
  DL_CUDA(ctx, cudaMemsetAsync(a.msg_last_run, 0xff, (size_t)num_messages * sizeof(int32_t), ctx->stream));
  DL_CUDA(ctx, cudaMemsetAsync(a.counters, 0, kNumCounters * sizeof(unsigned long long), ctx->stream));
  a.num_rows = num_rows;
  a.msgs = d_msgs;
  a.num_msgs = num_messages;
  a.n = n;
  a.times = d_times.get();
  a.nodes = d_nodes.get();
  a.trajs = d_trajs.get();
  a.num_runs = d_ints;
  a.num_keep = d_ints + 1;
  a.range_filter = options.range_filter;
  a.min_range = options.min_range;
  a.max_range = options.max_range;
  a.resolution = resolution;
  a.check_extent = options.outlier_voxel_size > 0 && pass == 0;

  // runs and their poses: the number of runs is counted before the pose table is sized
  mw_heads_count<<<tiles, kBlock, 0, ctx->stream>>>(a);
  DL_LAUNCH_CHECK(ctx, "mw_heads_count");
  mw_tile_prefix<<<1, kBlock, 0, ctx->stream>>>(a.head_tiles, (int)tiles, a.num_runs);
  DL_LAUNCH_CHECK(ctx, "mw_tile_prefix");
  int32_t num_runs = 0;
  DL_CUDA(ctx, cudaMemcpyAsync(&num_runs, a.num_runs, sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
  DL_CUDA(ctx, ctx->wait_stream());
  DL_TRY(reserve_runs(num_runs));
  a.runs = d_runs.get();
  mw_run_poses<<<tiles, kBlock, 0, ctx->stream>>>(a);
  DL_LAUNCH_CHECK(ctx, "mw_run_poses");
  mw_origins<<<(num_messages + 127) / 128, 128, 0, ctx->stream>>>(a);
  DL_LAUNCH_CHECK(ctx, "mw_origins");
  // transform, Has, range gate, ordered compaction
  mw_select<0><<<tiles, kBlock, 0, ctx->stream>>>(a);
  DL_LAUNCH_CHECK(ctx, "mw_select<0>");
  mw_tile_prefix<<<1, kBlock, 0, ctx->stream>>>(a.keep_tiles, (int)tiles, a.num_keep);
  DL_LAUNCH_CHECK(ctx, "mw_tile_prefix");
  const bool direct = final_pass() && options.outlier_voxel_size <= 0;
  SelectArgs s = a;
  if (direct) {
    s.compact = nullptr;
    s.out_xyz = d_out;
    s.out_msg = out_msg;
  }
  mw_select<1><<<tiles, kBlock, 0, ctx->stream>>>(s);
  DL_LAUNCH_CHECK(ctx, "mw_select<1>");
  unsigned long long counters[kNumCounters];
  int32_t kept = 0;
  std::vector<int32_t> last_run((size_t)num_messages);
  DL_CUDA(ctx, cudaMemcpyAsync(counters, a.counters, sizeof(counters), cudaMemcpyDeviceToHost, ctx->stream));
  DL_CUDA(ctx, cudaMemcpyAsync(&kept, a.num_keep, sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
  DL_CUDA(ctx, cudaMemcpyAsync(last_run.data(), a.msg_last_run, (size_t)num_messages * sizeof(int32_t), cudaMemcpyDeviceToHost,
                               ctx->stream));
  if (origins_out)
    DL_CUDA(ctx, cudaMemcpyAsync(origins_out, a.origins, 3 * (size_t)num_messages * sizeof(float), cudaMemcpyDeviceToHost,
                                 ctx->stream));
  DL_CUDA(ctx, ctx->wait_stream());
  if (counters[kOutside] > 0)
    return ctx->fail(DL_ERR_ARG, "dl_map_writer_process: a point's or its batch origin's cell lies beyond +-8192 cells (the hybrid "
                                 "grid's largest extent)");
  local.dropped_no_pose = (int64_t)counters[kNoPose];
  local.dropped_range = (int64_t)counters[kRange];
  local.messages_without_batch = std::count(last_run.begin(), last_run.end(), -1);

  if (options.outlier_voxel_size > 0) DL_TRY(reserve_table(&table, num_cells, pass == 0 ? kept : 0, false));
  const Table t = table.view();
  int64_t out_count = 0;
  if (direct) {
    out_count = kept;
  } else if (pass == 0) {
    if (kept > 0) {
      mw_insert_hits<<<tiles_of(kept), kBlock, 0, ctx->stream>>>(t, a.compact, kept, resolution);
      DL_LAUNCH_CHECK(ctx, "mw_insert_hits");
    }
  } else if (pass == 1) {
    if (kept > 0) {
      mw_rays<<<tiles_of(kept), kBlock, 0, ctx->stream>>>(t, a.compact, kept, a.origins, resolution, options.outlier_voxel_size,
                                                          a.counters);
      DL_LAUNCH_CHECK(ctx, "mw_rays");
    }
  } else if (kept > 0) {
    const unsigned gt = tiles_of(kept);
    mw_gate<0><<<gt, kBlock, 0, ctx->stream>>>(t, a.compact, kept, resolution, gate_tiles, nullptr, nullptr);
    DL_LAUNCH_CHECK(ctx, "mw_gate<0>");
    mw_tile_prefix<<<1, kBlock, 0, ctx->stream>>>(gate_tiles, (int)gt, d_ints + 2);
    DL_LAUNCH_CHECK(ctx, "mw_tile_prefix");
    mw_gate<1><<<gt, kBlock, 0, ctx->stream>>>(t, a.compact, kept, resolution, gate_tiles, d_out, out_msg);
    DL_LAUNCH_CHECK(ctx, "mw_gate<1>");
    int32_t survivors = 0;
    DL_CUDA(ctx, cudaMemcpyAsync(&survivors, d_ints + 2, sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
    DL_CUDA(ctx, ctx->wait_stream());
    out_count = survivors;
    local.dropped_moving = kept - survivors;
  }
  // every stage checks its input before any of them changes: the grids' growth first, then the X-ray cells
  GridCall grid_call;
  if (with_grid) DL_TRY(plan_grids(d_out, out_msg, out_count, a.origins, num_messages, last_run, boxes, &grid_call));
  if (with_xray && out_count > 0)
    DL_TRY(insert_xray(d_out, out_msg, d_msgs, out_count, sort_scratch, sort_bytes, sort_keys, sort_vals, a.counters + kOutside));
  if (with_grid) DL_TRY(apply_grids(d_out, &grid_call));
  DL_CUDA(ctx, cudaMemcpyAsync(counters, a.counters, sizeof(counters), cudaMemcpyDeviceToHost, ctx->stream));
  int32_t cells = 0;
  if (t.num_cells) DL_CUDA(ctx, cudaMemcpyAsync(&cells, t.num_cells, sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
  if (points_host && out_count > 0)
    DL_CUDA(ctx, cudaMemcpyAsync(points_host, d_out, 3 * (size_t)out_count * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  DL_CUDA(ctx, ctx->wait_stream());
  num_cells = cells;
  local.num_samples = (int64_t)counters[kSamples];
  local.num_points_out = out_count;
  *num_points_out = out_count;
  started = true;
  if (info) *info = local;
  return DL_OK;
}

// The final pass's output points [0, n) of one call into every X-ray stage. Every cell is checked before anything changes; then
// chunks of kXrayChunk points, each with its table reservation (two new entries per point and stage at most), insert, sort and
// fold, so that the colour sums take the points in stream order across chunks and calls.
int dl_map_writer::insert_xray(const float* points, const int32_t* point_msg, const MsgRec* msgs, int64_t n, void* sort_scratch,
                               size_t sort_bytes, unsigned long long* keys, int32_t* vals, unsigned long long* outside) {
  XrayArgs a = xray_args();
  a.points = points;
  a.point_msg = point_msg;
  a.msgs = msgs;
  a.outside = outside;
  a.n = n;
  DL_CUDA(ctx, cudaMemsetAsync(outside, 0, sizeof(unsigned long long), ctx->stream));
  mw_xray_check<<<tiles_of(n), kBlock, 0, ctx->stream>>>(a);
  DL_LAUNCH_CHECK(ctx, "mw_xray_check");
  unsigned long long num_outside = 0;
  DL_CUDA(ctx, cudaMemcpyAsync(&num_outside, outside, sizeof(num_outside), cudaMemcpyDeviceToHost, ctx->stream));
  DL_CUDA(ctx, ctx->wait_stream());
  if (num_outside > 0)
    return ctx->fail(DL_ERR_ARG, "dl_map_writer_process: a point's X-ray cell lies beyond +-8192 cells (the hybrid grid's largest "
                                 "extent)");
  const int64_t num_sums = (int64_t)sum_stage.size();
  const int64_t items_cap = std::min<int64_t>(n, kXrayChunk) * num_sums;  // the carve's size of each sort buffer
  int sum_bits = 0;
  while ((1 << sum_bits) < num_sums) ++sum_bits;
  for (int64_t first = 0; first < n; first += kXrayChunk) {
    const int64_t m = std::min(kXrayChunk, n - first);
    DL_TRY(reserve_table(&xray, xray_entries, 2 * m * (int64_t)xrays.size(), true));
    const Table t = xray.view();
    a.first = first;
    a.n = m;
    a.slot_bits = 64 - t.shift;
    a.sort_keys = keys;
    a.sort_vals = vals;
    mw_xray_insert<<<tiles_of(m), kBlock, 0, ctx->stream>>>(t, a);
    DL_LAUNCH_CHECK(ctx, "mw_xray_insert");
    if (num_sums > 0) {
      const int items = (int)(m * num_sums);
      cub::DoubleBuffer<unsigned long long> k(keys, keys + items_cap);
      cub::DoubleBuffer<int32_t> v(vals, vals + items_cap);
      // the scratch was sized for all 64 bits and items_cap items, the most any chunk sorts
      DL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(sort_scratch, sort_bytes, k, v, items, 0, a.slot_bits + sum_bits, ctx->stream));
      mw_xray_fold<<<tiles_of(items), kBlock, 0, ctx->stream>>>(t, a, k.Current(), v.Current(), items);
      DL_LAUNCH_CHECK(ctx, "mw_xray_fold");
    }
    int32_t entries = 0;
    DL_CUDA(ctx, cudaMemcpyAsync(&entries, t.num_cells, sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
    DL_CUDA(ctx, ctx->wait_stream());
    xray_entries = entries;
  }
  return DL_OK;
}

// The grid stages' half of a final-pass call that changes nothing: one reduction of every batch's float box and point range over
// the call's output points, one read-back, then GrowAsNeeded replayed on the host for every stage and batch in order. A stage
// whose grid grows (or gets its first batch) gets its buffers at the call's final limits here, so that apply_grids cannot fail
// halfway.
int dl_map_writer::plan_grids(const float* points, const int32_t* point_msg, int64_t n, const float* origins, int num_messages,
                              const std::vector<int32_t>& last_run, const GridBoxes& b, GridCall* call) {
  std::vector<int32_t> batch_msgs;
  for (int m = 0; m < num_messages; ++m)
    if (last_run[m] >= 0) batch_msgs.push_back(m);
  if (batch_msgs.empty()) return DL_OK;
  const size_t nm = (size_t)num_messages;
  DL_CUDA(ctx, cudaMemsetAsync(b.keys, 0, 4 * nm * sizeof(uint32_t), ctx->stream));
  DL_CUDA(ctx, cudaMemsetAsync(b.first, 0x7f, nm * sizeof(int32_t), ctx->stream));
  DL_CUDA(ctx, cudaMemsetAsync(b.last, 0xff, nm * sizeof(int32_t), ctx->stream));
  DL_CUDA(ctx, cudaMemsetAsync(b.nonfinite, 0, sizeof(unsigned long long), ctx->stream));
  if (n > 0) {
    const int64_t per_block = (int64_t)kBlock * kGridBoxChunk;
    mw_grid_boxes<<<(unsigned)((n + per_block - 1) / per_block), kBlock, 0, ctx->stream>>>(points, point_msg, n, b);
    DL_LAUNCH_CHECK(ctx, "mw_grid_boxes");
  }
  std::vector<uint32_t> keys(4 * nm);
  std::vector<int32_t> first(nm), last(nm);
  std::vector<float> org(3 * nm);
  unsigned long long nonfinite = 0;
  DL_CUDA(ctx, cudaMemcpyAsync(keys.data(), b.keys, keys.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  DL_CUDA(ctx, cudaMemcpyAsync(first.data(), b.first, nm * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
  DL_CUDA(ctx, cudaMemcpyAsync(last.data(), b.last, nm * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
  DL_CUDA(ctx, cudaMemcpyAsync(org.data(), origins, org.size() * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  DL_CUDA(ctx, cudaMemcpyAsync(&nonfinite, b.nonfinite, sizeof(nonfinite), cudaMemcpyDeviceToHost, ctx->stream));
  DL_CUDA(ctx, ctx->wait_stream());
  if (nonfinite > 0) return ctx->fail(DL_ERR_ARG, "dl_map_writer_process: a point's x or y is not finite (probability grid stage)");
  // GrowAsNeeded's float box: the origin, extended by every point (min / max do not depend on the order)
  std::vector<float> lo(2 * batch_msgs.size()), hi(2 * batch_msgs.size());
  for (size_t j = 0; j < batch_msgs.size(); ++j) {
    const int m = batch_msgs[j];
    float x0 = org[3 * m], y0 = org[3 * m + 1], x1 = x0, y1 = y0;
    const bool points_in = first[m] <= last[m];
    if (points_in) {
      x0 = std::min(x0, key_float(~keys[4 * m]));
      y0 = std::min(y0, key_float(~keys[4 * m + 1]));
      x1 = std::max(x1, key_float(keys[4 * m + 2]));
      y1 = std::max(y1, key_float(keys[4 * m + 3]));
    }
    const float pad = 1e-6f;  // kPadding
    lo[2 * j] = x0 - pad;
    lo[2 * j + 1] = y0 - pad;
    hi[2 * j] = x1 + pad;
    hi[2 * j + 1] = y1 + pad;
    call->first.push_back(points_in ? first[m] : 0);
    call->count.push_back(points_in ? last[m] - first[m] + 1 : 0);
    call->origins.push_back(org[3 * m]);
    call->origins.push_back(org[3 * m + 1]);
  }
  for (const GridStage& g : grids) {
    GridPlan p;
    p.final_limits = g.limits;
    std::vector<int2> at_growth;
    for (size_t j = 0; j < batch_msgs.size(); ++j) {
      if (!grid_grow_limits(&p.final_limits, g.resolution, lo[2 * j], lo[2 * j + 1], &p.grow_x, &p.grow_y) ||
          !grid_grow_limits(&p.final_limits, g.resolution, hi[2 * j], hi[2 * j + 1], &p.grow_x, &p.grow_y))
        return ctx->fail(DL_ERR_ARG, "dl_map_writer_process: a batch would grow a probability grid beyond "
                                     "DL_MAP_WRITER_MAX_GRID_CELLS cells per axis");
      p.at.push_back(p.final_limits);
      at_growth.push_back(make_int2(p.grow_x, p.grow_y));
    }
    for (const int2& c : at_growth) p.offset.push_back(make_int2(p.grow_x - c.x, p.grow_y - c.y));
    call->plans.push_back(std::move(p));
  }
  for (size_t s = 0; s < grids.size(); ++s) {
    GridPlan& p = call->plans[s];
    if (grids[s].cells.get() && p.grow_x == 0 && p.grow_y == 0) continue;
    const size_t cells = (size_t)p.final_limits.nx * (size_t)p.final_limits.ny;
    DL_TRY(alloc(ctx, p.cells, cells));
    DL_TRY(alloc(ctx, p.stamps, cells));
  }
  return DL_OK;
}

// Moves grown grids into their new buffers, then per stage and batch in order one launch for the hits and one for the walks.
int dl_map_writer::apply_grids(const float* points, GridCall* call) {
  for (size_t s = 0; s < grids.size() && !call->count.empty(); ++s) {
    GridStage& g = grids[s];
    GridPlan& p = call->plans[s];
    const GridLimits& l = p.final_limits;
    if (p.cells.get()) {
      const size_t cells = (size_t)l.nx * (size_t)l.ny;
      DL_CUDA(ctx, cudaMemsetAsync(p.cells.get(), 0, cells * sizeof(uint16_t), ctx->stream));
      DL_CUDA(ctx, cudaMemsetAsync(p.stamps.get(), 0, cells * sizeof(uint32_t), ctx->stream));  // below every claim
      if (g.cells.get()) {
        DL_CUDA(ctx, cudaMemcpy2DAsync(p.cells.get() + (size_t)p.grow_y * l.nx + p.grow_x, (size_t)l.nx * sizeof(uint16_t),
                                       g.cells.get(), (size_t)g.limits.nx * sizeof(uint16_t), (size_t)g.limits.nx * sizeof(uint16_t),
                                       (size_t)g.limits.ny, cudaMemcpyDeviceToDevice, ctx->stream));
        DL_CUDA(ctx, ctx->wait_stream());  // the copy out of the old buffers has ended
      }
      g.cells = std::move(p.cells);
      g.stamps = std::move(p.stamps);
    }
    g.limits = l;
    const double superscaled = g.resolution / kSubpixel;
    for (size_t j = 0; j < call->count.size(); ++j) {
      const int64_t k = ++g.batches;
      GridBatch gb{};
      gb.pts = points + 3 * (size_t)call->first[j];
      gb.n = call->count[j];
      long bx, by;
      grid_cell_index(p.at[j], superscaled, call->origins[2 * j], call->origins[2 * j + 1], &bx, &by);
      gb.begin_x = (int32_t)bx;
      gb.begin_y = (int32_t)by;
      gb.off_x = p.offset[j].x;
      gb.off_y = p.offset[j].y;
      gb.stride = l.nx;
      gb.max_x = p.at[j].max_x;
      gb.max_y = p.at[j].max_y;
      gb.resolution = superscaled;
      gb.cells = g.cells.get();
      gb.stamps = g.stamps.get();
      if (gb.n == 0) continue;  // the batch only grew the grid
      gb.table = g.tables.get();
      gb.claim = (uint32_t)(2 * k + 1);
      mw_grid_hits<<<tiles_of(gb.n), kBlock, 0, ctx->stream>>>(gb);
      DL_LAUNCH_CHECK(ctx, "mw_grid_hits");
      if (!g.insert_free_space) continue;
      gb.table = g.tables.get() + 32768;
      gb.claim = (uint32_t)(2 * k);
      mw_grid_walks<<<tiles_of(gb.n), kBlock, 0, ctx->stream>>>(gb);
      DL_LAUNCH_CHECK(ctx, "mw_grid_walks");
    }
  }
  return DL_OK;
}

int dl_map_writer_create(dl_context* ctx, const dl_map_writer_options* options, dl_map_writer** out) {
  if (!ctx || !options || !out) return DL_ERR_ARG;
  const dl_map_writer_options& o = *options;
  if (o.range_filter != 0 && o.range_filter != 1) return ctx->fail(DL_ERR_ARG, "range_filter must be 0 or 1");
  if (o.range_filter && (std::isnan(o.min_range) || std::isnan(o.max_range)))
    return ctx->fail(DL_ERR_ARG, "min_range / max_range must not be NaN");
  if (!(o.outlier_voxel_size >= 0) || !std::isfinite(o.outlier_voxel_size) ||
      (o.outlier_voxel_size > 0 && !((float)o.outlier_voxel_size > 0.f)))
    return ctx->fail(DL_ERR_ARG, "outlier_voxel_size must be finite and >= 0");
  std::unique_ptr<dl_map_writer> w(new dl_map_writer());
  w->ctx = ctx;
  w->options = o;
  w->resolution = (float)o.outlier_voxel_size;
  if (o.outlier_voxel_size > 0) {
    DL_CUDA(ctx, cudaSetDevice(ctx->device));
    DL_TRY(alloc(ctx, w->table.num_cells, 1, 0));
  }
  *out = w.release();
  return DL_OK;
}

void dl_map_writer_destroy(dl_map_writer* w) {
  if (!w) return;
  cudaSetDevice(w->ctx->device);
  w->ctx->wait_stream();
  delete w;
}

int dl_map_writer_add_trajectory(dl_map_writer* w, int32_t trajectory_id, int32_t num_nodes, const int64_t* times,
                                 const double* poses) {
  if (!w) return DL_ERR_ARG;
  dl_context* ctx = w->ctx;
  if (num_nodes < 0 || (num_nodes > 0 && (!times || !poses))) return ctx->fail(DL_ERR_ARG, "dl_map_writer_add_trajectory: bad arguments");
  if (w->started || w->finished) return ctx->fail(DL_ERR_ARG, "dl_map_writer_add_trajectory: processing has begun");
  if (w->slot_of.count(trajectory_id)) return ctx->fail(DL_ERR_ARG, "dl_map_writer_add_trajectory: trajectory added twice");
  for (int32_t i = 0; i < num_nodes; ++i) {
    if (!valid_pose7(poses + 7 * (size_t)i)) return ctx->fail(DL_ERR_ARG, "dl_map_writer_add_trajectory: a pose is not finite");
    // TransformInterpolationBuffer::Push: CHECK_GE(time, latest_time())
    if (i > 0 && times[i] < times[i - 1]) return ctx->fail(DL_ERR_ARG, "dl_map_writer_add_trajectory: node times decrease");
  }
  const int64_t first = (int64_t)w->nodes.size();
  for (int32_t i = 0; i < num_nodes; ++i) {
    NodeRec r{};
    r.pose = pose_from7(poses + 7 * (size_t)i);
    if (i > 0) {
      r.slerp = slerp_constants(w->nodes.back().pose.q, r.pose.q);  // the interval-constant half, with the host's acos / sin
    }
    w->nodes.push_back(r);
    w->times.push_back(times[i]);
  }
  w->slot_of[trajectory_id] = (int32_t)w->trajs.size();
  w->trajs.push_back(TrajRec{first, num_nodes});
  w->tables_dirty = true;
  return DL_OK;
}

int dl_map_writer_process(dl_map_writer* w, int32_t num_messages, const dl_map_message* messages, const float* xyzt_rows,
                          int64_t num_rows, float* points_out, int64_t* num_points_out, float* origins_out,
                          dl_map_writer_info* info) {
  if (!w) return DL_ERR_ARG;
  return w->process(num_messages, messages, xyzt_rows, nullptr, num_rows, points_out, nullptr, num_points_out, origins_out, info);
}

int dl_map_writer_process_dev(dl_map_writer* w, int32_t num_messages, const dl_map_message* messages, const float* xyzt_rows_dev,
                              int64_t num_rows, float* points_out_dev, int64_t* num_points_out, float* origins_out,
                              dl_map_writer_info* info) {
  if (!w) return DL_ERR_ARG;
  return w->process(num_messages, messages, nullptr, xyzt_rows_dev, num_rows, nullptr, points_out_dev, num_points_out, origins_out,
                    info);
}

int dl_map_writer_flush(dl_map_writer* w, int32_t* restart) {
  if (!w || !restart) return DL_ERR_ARG;
  if (w->finished) return w->ctx->fail(DL_ERR_ARG, "dl_map_writer_flush: the final pass was flushed");
  if (w->final_pass()) {
    w->finished = true;
    *restart = 0;
  } else {
    ++w->pass;
    *restart = 1;
  }
  return DL_OK;
}

int dl_map_writer_voxels(const dl_map_writer* w, int64_t capacity, int32_t* cells_xyz, int32_t* hits, int32_t* rays, int64_t* count) {
  if (!w || !count || capacity < 0) return DL_ERR_ARG;
  dl_context* ctx = w->ctx;
  *count = w->num_cells;
  if (!cells_xyz) return DL_OK;
  if (capacity < w->num_cells || !hits || !rays) return ctx->fail(DL_ERR_ARG, "dl_map_writer_voxels: capacity below the cell count");
  const size_t cap = w->table.keys.cap;
  if (cap == 0) return DL_OK;
  std::vector<unsigned long long> keys(cap);
  std::vector<int32_t> h(cap), r(cap);
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  DL_TRY(d2h(ctx, keys.data(), w->table.keys.get(), cap));
  DL_TRY(d2h(ctx, h.data(), w->table.hits.get(), cap));
  DL_TRY(d2h(ctx, r.data(), w->table.rays.get(), cap));
  DL_TRY(sync(ctx));
  std::vector<size_t> order;
  for (size_t i = 0; i < cap; ++i)
    if (keys[i] != kEmpty) order.push_back(i);
  std::sort(order.begin(), order.end(), [&](size_t a, size_t b) { return keys[a] < keys[b]; });  // key order = (x, y, z) order
  for (size_t k = 0; k < order.size(); ++k) {
    const unsigned long long key = keys[order[k]];
    cells_xyz[3 * k] = (int32_t)((key >> 28) & 0x3fff) - kGridHalf;
    cells_xyz[3 * k + 1] = (int32_t)((key >> 14) & 0x3fff) - kGridHalf;
    cells_xyz[3 * k + 2] = (int32_t)(key & 0x3fff) - kGridHalf;
    hits[k] = h[order[k]];
    rays[k] = r[order[k]];
  }
  *count = (int64_t)order.size();
  return DL_OK;
}

int dl_map_writer_add_color(dl_map_writer* w, const dl_map_writer_color* color) {
  if (!w) return DL_ERR_ARG;
  dl_context* ctx = w->ctx;
  if (!color) return ctx->fail(DL_ERR_ARG, "dl_map_writer_add_color: bad arguments");
  if (w->started || w->finished) return ctx->fail(DL_ERR_ARG, "dl_map_writer_add_color: processing has begun");
  if (w->num_stages() >= kMaxStages)
    return ctx->fail(DL_ERR_ARG, "dl_map_writer_add_color: more than DL_MAP_WRITER_MAX_STAGES stages");
  // ToFloatColor: Uint8ComponentToFloat(c) = c / 255.f
  w->colors.push_back(ColorStage{color->frame_id, color->rgb[0] / 255.f, color->rgb[1] / 255.f, color->rgb[2] / 255.f});
  return DL_OK;
}

int dl_map_writer_add_xray(dl_map_writer* w, const dl_map_writer_xray* xray, int32_t* stage) {
  if (!w) return DL_ERR_ARG;
  dl_context* ctx = w->ctx;
  if (!xray || !stage) return ctx->fail(DL_ERR_ARG, "dl_map_writer_add_xray: bad arguments");
  if (w->started || w->finished) return ctx->fail(DL_ERR_ARG, "dl_map_writer_add_xray: processing has begun");
  if (w->num_stages() >= kMaxStages)
    return ctx->fail(DL_ERR_ARG, "dl_map_writer_add_xray: more than DL_MAP_WRITER_MAX_STAGES stages");
  if (!(xray->voxel_size > 0) || !std::isfinite(xray->voxel_size) || !((float)xray->voxel_size > 0.f))
    return ctx->fail(DL_ERR_ARG, "dl_map_writer_add_xray: voxel_size must be finite and > 0");
  if (!valid_pose7(xray->transform)) return ctx->fail(DL_ERR_ARG, "dl_map_writer_add_xray: transform is not finite");
  const double* q = xray->transform + 3;  // Eigen's squaredNorm order
  const double norm = std::sqrt(q[1] * q[1] + q[2] * q[2] + q[3] * q[3] + q[0] * q[0]);
  if (!(std::fabs(norm - 1.0) <= 1e-9)) return ctx->fail(DL_ERR_ARG, "dl_map_writer_add_xray: the rotation is not a unit quaternion");
  DL_TRY(w->init_xray());
  XrayStage s{};
  s.transform = to_float(pose_from7(xray->transform));
  s.resolution = (float)xray->voxel_size;
  s.num_colors = (int32_t)w->colors.size();
  s.sum_index = -1;
  if (s.num_colors > 0) {
    s.sum_index = (int32_t)w->sum_stage.size();
    w->sum_stage.push_back((int32_t)w->xrays.size());
  }
  *stage = (int32_t)w->xrays.size();
  w->xrays.push_back(s);
  return DL_OK;
}

int dl_map_writer_xray_image(const dl_map_writer* w, int32_t stage, int64_t capacity, uint32_t* argb, int32_t* width,
                             int32_t* height) {
  if (!w || !width || !height) return DL_ERR_ARG;
  dl_context* ctx = w->ctx;
  if (stage < 0 || stage >= (int32_t)w->xrays.size()) return ctx->fail(DL_ERR_ARG, "dl_map_writer_xray_image: unknown stage");
  if (!w->finished) return ctx->fail(DL_ERR_ARG, "dl_map_writer_xray_image: the final pass has not been flushed");
  int32_t box[6];
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  DL_TRY(d2h(ctx, box, w->d_bbox.get() + 6 * stage, 6));
  DL_TRY(sync(ctx));
  const bool empty = box[1] > box[4];  // Eigen::AlignedBox::isEmpty
  const int32_t wd = empty ? 0 : box[4] - box[1] + 1, ht = empty ? 0 : box[5] - box[2] + 1;
  *width = wd;
  *height = ht;
  if (!argb || empty) return DL_OK;
  const int64_t pixels = (int64_t)wd * ht;
  if (capacity < pixels) return ctx->fail(DL_ERR_ARG, "dl_map_writer_xray_image: capacity below width * height");
  int32_t* d_max = nullptr;
  uint32_t* d_img = nullptr;
  DL_TRY(carve_scratch(ctx, [&](Arena& ar) {
    d_max = ar.take<int32_t>(1);
    d_img = ar.take<uint32_t>((size_t)pixels);
  }));
  const Table xray = w->xray.view();
  const int64_t xray_capacity = (int64_t)w->xray.keys.cap;
  const unsigned tiles = tiles_of(xray_capacity);
  DL_CUDA(ctx, cudaMemsetAsync(d_max, 0, sizeof(int32_t), ctx->stream));
  DL_CUDA(ctx, cudaMemsetAsync(d_img, 0xff, (size_t)pixels * sizeof(uint32_t), ctx->stream));  // white
  mw_xray_max_voxels<<<tiles, kBlock, 0, ctx->stream>>>(xray, xray_capacity, stage, d_max);
  DL_LAUNCH_CHECK(ctx, "mw_xray_max_voxels");
  int32_t max_voxels = 0;
  DL_CUDA(ctx, cudaMemcpyAsync(&max_voxels, d_max, sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
  DL_CUDA(ctx, ctx->wait_stream());
  // IntoImage: max starts at numeric_limits<float>::min() and takes std::max<float>(max, log(n)); log is monotone, so the
  // largest n gives the largest (float)log(n)
  const float max_log = std::max<float>(FLT_MIN, (float)log_table()[max_voxels]);
  mw_xray_pixels<<<tiles, kBlock, 0, ctx->stream>>>(xray, xray_capacity, stage, w->d_log.get(), max_log, box[4], box[5], wd,
                                                     d_img);
  DL_LAUNCH_CHECK(ctx, "mw_xray_pixels");
  DL_CUDA(ctx, cudaMemcpyAsync(argb, d_img, (size_t)pixels * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  DL_CUDA(ctx, ctx->wait_stream());
  return DL_OK;
}

int dl_map_writer_add_probability_grid(dl_map_writer* w, const dl_map_writer_grid_options* options, int32_t* stage) {
  if (!w) return DL_ERR_ARG;
  dl_context* ctx = w->ctx;
  if (!options || !stage) return ctx->fail(DL_ERR_ARG, "dl_map_writer_add_probability_grid: bad arguments");
  if (w->started || w->finished) return ctx->fail(DL_ERR_ARG, "dl_map_writer_add_probability_grid: processing has begun");
  if (w->num_stages() >= kMaxStages)
    return ctx->fail(DL_ERR_ARG, "dl_map_writer_add_probability_grid: more than DL_MAP_WRITER_MAX_STAGES stages");
  const dl_map_writer_grid_options& o = *options;
  if (!(o.resolution > 0) || !std::isfinite(o.resolution))
    return ctx->fail(DL_ERR_ARG, "dl_map_writer_add_probability_grid: resolution must be finite and > 0");
  // CreateProbabilityGridRangeDataInserterOptions2D: CHECK_GT(hit_probability, 0.5), CHECK_LT(miss_probability, 0.5)
  if (!(o.hit_probability > 0.5) || !std::isfinite(o.hit_probability) || !(o.miss_probability < 0.5) ||
      !std::isfinite(o.miss_probability))
    return ctx->fail(DL_ERR_ARG, "dl_map_writer_add_probability_grid: hit_probability must be > 0.5 and miss_probability < 0.5");
  if (o.insert_free_space != 0 && o.insert_free_space != 1)
    return ctx->fail(DL_ERR_ARG, "dl_map_writer_add_probability_grid: insert_free_space must be 0 or 1");
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  std::vector<uint16_t> tables(2 * 32768);
  compute_correspondence_cost_table(o.hit_probability, tables.data());
  compute_correspondence_cost_table(o.miss_probability, tables.data() + 32768);
  const std::vector<uint8_t> colors = grid_color_table();
  GridStage g{};
  DeviceBuffer<uint8_t> d_colors;
  DL_TRY(alloc(ctx, g.tables, tables.size()));
  DL_TRY(h2d(ctx, g.tables.get(), tables.data(), tables.size()));
  if (!w->d_grid_colors.get()) {
    DL_TRY(alloc(ctx, d_colors, colors.size()));
    DL_TRY(h2d(ctx, d_colors.get(), colors.data(), colors.size()));
  }
  DL_TRY(sync(ctx));  // `tables` and `colors` are pageable and local
  if (d_colors.get()) w->d_grid_colors = std::move(d_colors);
  g.resolution = o.resolution;
  g.insert_free_space = o.insert_free_space;
  // CreateProbabilityGrid (probability_grid_points_processor.cc:150-158): 100 x 100 cells, max = 0.5 * 100 * resolution
  const double max = 0.5 * 100 * o.resolution;
  g.limits = GridLimits{max, max, 100, 100};
  *stage = (int32_t)w->grids.size();
  w->grids.push_back(std::move(g));
  return DL_OK;
}

int dl_map_writer_probability_grid(const dl_map_writer* w, int32_t stage, dl_map_writer_grid_info* info, int64_t capacity,
                                   uint16_t* cells, uint8_t* pixels) {
  if (!w || !info) return DL_ERR_ARG;
  dl_context* ctx = w->ctx;
  if (stage < 0 || stage >= (int32_t)w->grids.size()) return ctx->fail(DL_ERR_ARG, "dl_map_writer_probability_grid: unknown stage");
  if (!w->finished) return ctx->fail(DL_ERR_ARG, "dl_map_writer_probability_grid: the final pass has not been flushed");
  const GridStage& g = w->grids[stage];
  const int64_t num_cells = (int64_t)g.limits.nx * g.limits.ny;
  int32_t box[4] = {INT_MAX, INT_MAX, INT_MIN, INT_MIN};
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  if (g.cells.get()) {
    int32_t* d_box = nullptr;
    DL_TRY(carve_scratch(ctx, [&](Arena& ar) { d_box = ar.take<int32_t>(4); }));
    DL_CUDA(ctx, cudaMemcpyAsync(d_box, box, sizeof(box), cudaMemcpyHostToDevice, ctx->stream));
    mw_grid_known_box<<<tiles_of(num_cells), kBlock, 0, ctx->stream>>>(g.cells.get(), g.limits.nx, num_cells, d_box);
    DL_LAUNCH_CHECK(ctx, "mw_grid_known_box");
    DL_CUDA(ctx, cudaMemcpyAsync(box, d_box, sizeof(box), cudaMemcpyDeviceToHost, ctx->stream));
    DL_CUDA(ctx, ctx->wait_stream());
  }
  dl_map_writer_grid_info r{};
  r.resolution = g.resolution;
  r.max_x = g.limits.max_x;
  r.max_y = g.limits.max_y;
  r.num_x_cells = g.limits.nx;
  r.num_y_cells = g.limits.ny;
  const bool empty = box[0] > box[2];  // ComputeCroppedLimits: an empty box gives offset 0 and 1 x 1
  r.offset_x = empty ? 0 : box[0];
  r.offset_y = empty ? 0 : box[1];
  r.width = empty ? 1 : box[2] - box[0] + 1;
  r.height = empty ? 1 : box[3] - box[1] + 1;
  *info = r;
  if (!cells && !pixels) return DL_OK;
  const int64_t count = (int64_t)r.width * r.height;
  if (capacity < count) return ctx->fail(DL_ERR_ARG, "dl_map_writer_probability_grid: capacity below width * height");
  if (!g.cells.get()) {  // no batch reached the stage: cell (0, 0) of the initial grid, unknown
    if (cells) cells[0] = 0;
    if (pixels) pixels[0] = 128;
    return DL_OK;
  }
  uint16_t* d_cells = nullptr;
  uint8_t* d_pixels = nullptr;
  DL_TRY(carve_scratch(ctx, [&](Arena& ar) {
    d_cells = ar.take<uint16_t>((size_t)count);
    d_pixels = ar.take<uint8_t>((size_t)count);
  }));
  mw_grid_crop<<<tiles_of(count), kBlock, 0, ctx->stream>>>(g.cells.get(), g.limits.nx, r.offset_x, r.offset_y, r.width,
                                                             count, w->d_grid_colors.get(), d_cells, d_pixels);
  DL_LAUNCH_CHECK(ctx, "mw_grid_crop");
  if (cells) DL_CUDA(ctx, cudaMemcpyAsync(cells, d_cells, (size_t)count * sizeof(uint16_t), cudaMemcpyDeviceToHost, ctx->stream));
  if (pixels) DL_CUDA(ctx, cudaMemcpyAsync(pixels, d_pixels, (size_t)count, cudaMemcpyDeviceToHost, ctx->stream));
  DL_CUDA(ctx, ctx->wait_stream());
  return DL_OK;
}
