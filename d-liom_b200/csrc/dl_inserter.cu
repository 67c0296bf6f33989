// Range-data insertion into the device-resident probability grid (SURVEY 8f-1: the step right after the hot path).
//
// Replaces RangeDataInserter3D::Insert + InsertMissesIntoGrid (C/mapping/3d/range_data_inserter_3d.cc:27-51, :76-92),
// HybridGrid::ApplyLookupTable / FinishUpdate (C/mapping/3d/hybrid_grid.h:494-520) and the growth path of
// DynamicGrid / NestedGrid::mutable_value (hybrid_grid.h:285-300, :165-176, :389-407) so that the device grid is the
// PRIMARY copy: no per-scan host insert + dirty-brick upload.
//
// Semantics preserved exactly: within one Insert every cell is updated at most once (the update marker, bit 15);
// all hits are applied before any miss, so a hit wins over a miss in the same cell; all hits use one table and all
// misses another, so the order inside each group is irrelevant and the two groups parallelise freely:
//     cell' = hit_table[cell]  if the cell is a hit cell, else miss_table[cell] if it is a miss cell, else cell.
// Concurrent updates of one uint16 cell go through a 32-bit compare-and-swap on the containing word.
// Structure growth is lock-free and spin-free: (1) claim missing top entries, (2) claim missing node entries — one
// kernel each, so nobody ever waits for an allocation made in the same kernel — then (3) hits, (4) misses,
// (5) FinishUpdate over the list of touched cells.
// One call inserts into many grids (a list of jobs, blockIdx.y = job): jobs of distinct grids touch distinct cells, so they run
// side by side, and the host steps (bounding boxes, pool growth) are taken once for all of them.
#include <algorithm>
#include <cstring>
#include <vector>

#include "dl_internal.cuh"
#include "dl_pipeline.cuh"

namespace dl {
namespace {

constexpr int kBlock = 256;

struct InsertArgs {
  const float* returns;  // n x 3, already in the grid's frame
  int n;
  const int32_t* n_dev;  // bounding-box pass only, optional: the point count on the device (n is then an upper bound)
  Vec3f origin;
  float resolution;
  int bits;
  int num_free;
  int32_t* top;
  int32_t* nodes;
  uint16_t* bricks;
  int32_t* counters;     // [0] nodes in use, [1] bricks in use, [2] update-list length, [3] nodes / [4] bricks this Insert adds
  int32_t* bbox;         // min xyz, max xyz
  uint32_t* update_list;
  const uint16_t* hit_table;
  const uint16_t* miss_table;
};

__device__ __forceinline__ Int3 hit_cell(const InsertArgs& a, int i) {
  return cell_index(Vec3f{a.returns[3 * i], a.returns[3 * i + 1], a.returns[3 * i + 2]}, a.resolution);
}

// CHECK_LT(num_samples, 1 << 15) of range_data_inserter_3d.cc:37: the host refuses a job with a longer ray before any grid
// changes, so that delta * position below stays inside int.
constexpr int kMaxSamples = 1 << 15;

// Sample `position` of a ray from cell o with delta d: origin_cell + delta * position / num_samples, C++ truncating division.
__device__ __forceinline__ Int3 miss_cell(const Int3& o, const Int3& d, int num_samples, int position) {
  return Int3{o.x + d.x * position / num_samples, o.y + d.y * position / num_samples, o.z + d.z * position / num_samples};
}

// Visits the hit cell (phase 0) or the miss cells (phase 1) of ray i, exactly as range_data_inserter_3d.cc:33-50.
template <typename F>
__device__ __forceinline__ void for_each_cell(const InsertArgs& a, int i, int phase, F f) {
  const Int3 h = hit_cell(a, i);
  if (phase == 0) {
    f(h);
    return;
  }
  const Int3 o = cell_index(a.origin, a.resolution);
  const Int3 d{h.x - o.x, h.y - o.y, h.z - o.z};
  const int num_samples = max(abs(d.x), max(abs(d.y), abs(d.z)));
  for (int position = max(0, num_samples - a.num_free); position < num_samples; ++position) f(miss_cell(o, d, num_samples, position));
}

// The box of every cell the job touches, in bbox[0..5], and its longest ray (num_samples) in bbox[7]. A ray touches its hit
// cell and samples max(0, num_samples - num_free) .. num_samples - 1; sample cells move monotonically along each axis, so the
// first of them and the hit cell bound them all (the origin cell only counts when it is a sample).
__global__ void ins_bbox_kernel(const InsertArgs* __restrict__ jobs) {
  const InsertArgs a = jobs[blockIdx.y];
  const int n = a.n_dev ? *a.n_dev : a.n;
  const Int3 o = cell_index(a.origin, a.resolution);
  int lo[3] = {0x7fffffff, 0x7fffffff, 0x7fffffff}, hi[3] = {-0x7fffffff, -0x7fffffff, -0x7fffffff};
  int longest = 0;
  auto add = [&](const Int3& c) {
    lo[0] = min(lo[0], c.x); lo[1] = min(lo[1], c.y); lo[2] = min(lo[2], c.z);
    hi[0] = max(hi[0], c.x); hi[1] = max(hi[1], c.y); hi[2] = max(hi[2], c.z);
  };
  for (int i = blockIdx.x * kBlock + threadIdx.x; i < n; i += gridDim.x * kBlock) {
    const Int3 h = hit_cell(a, i);
    add(h);
    const Int3 d{h.x - o.x, h.y - o.y, h.z - o.z};
    const int num_samples = max(abs(d.x), max(abs(d.y), abs(d.z)));
    longest = max(longest, num_samples);
    if (a.num_free > 0 && num_samples > 0 && num_samples < kMaxSamples)  // a longer ray fails the call: its box is not needed
      add(miss_cell(o, d, num_samples, max(0, num_samples - a.num_free)));
  }
  for (int k = 0; k < 3; ++k) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      lo[k] = min(lo[k], __shfl_xor_sync(0xffffffffu, lo[k], d));
      hi[k] = max(hi[k], __shfl_xor_sync(0xffffffffu, hi[k], d));
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) longest = max(longest, __shfl_xor_sync(0xffffffffu, longest, d));
  if ((threadIdx.x & 31) == 0) {
    for (int k = 0; k < 3; ++k) {
      atomicMin(a.bbox + k, lo[k]);
      atomicMax(a.bbox + 3 + k, hi[k]);
    }
    atomicMax(a.bbox + 7, longest);
  }
}

// Grow(): every axis doubles, the old content moves to the centre (hybrid_grid.h:389-407).
__global__ void grid_grow_kernel(const int32_t* old_top, int old_bits, int32_t* new_top) {
  const int n = 1 << old_bits;
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n * n * n) return;
  const int x = e & (n - 1), y = (e >> old_bits) & (n - 1), z = e >> (2 * old_bits);
  const int o = 1 << (old_bits - 1), nb = old_bits + 1;
  new_top[((((z + o) << nb) + (y + o)) << nb) + (x + o)] = old_top[e];
}

__device__ __forceinline__ void shifted(const InsertArgs& a, const Int3& c, unsigned* sx, unsigned* sy, unsigned* sz) {
  const int half = (64 << a.bits) >> 1;
  *sx = (unsigned)(c.x + half); *sy = (unsigned)(c.y + half); *sz = (unsigned)(c.z + half);
}

// level 0: make sure the top entry has a node; level 1: make sure the node entry has a brick. Two passes per level so that the
// pools are reserved for EXACTLY the entries this Insert creates (round 1 reserved the worst case, one node and one brick per
// touched cell: ~400 MB per grid for a 30k-point scan with two free-space voxels, a few hundred bricks actually used):
//   ASSIGN = 0  mark every missing entry this Insert touches (-1 -> -2) and count them in counters[3 + LEVEL];
//   ASSIGN = 1  after the host has grown the pool by that count: give every marked entry its slot (-2 -> index).
template <int LEVEL, int ASSIGN>
__global__ void __launch_bounds__(kBlock) ins_claim_kernel(const InsertArgs* __restrict__ jobs, int phase) {
  const InsertArgs a = jobs[blockIdx.y];
  for (int i = blockIdx.x * kBlock + threadIdx.x; i < a.n; i += gridDim.x * kBlock) {
    for_each_cell(a, i, phase, [&](const Int3& c) {
      unsigned sx, sy, sz;
      shifted(a, c, &sx, &sy, &sz);
      int32_t* entry = a.top + ((((sz >> 6) << a.bits) + (sy >> 6)) << a.bits) + (sx >> 6);
      if (LEVEL == 1) {
        const int node = *(volatile int32_t*)entry;  // assigned by the previous level
        entry = a.nodes + (size_t)node * 512 + ((((sz >> 3) & 7) << 6) | (((sy >> 3) & 7) << 3) | ((sx >> 3) & 7));
      }
      if (ASSIGN == 0) {
        if (*(volatile int32_t*)entry == -1 && atomicCAS(entry, -1, -2) == -1) atomicAdd(a.counters + 3 + LEVEL, 1);
      } else {
        if (*(volatile int32_t*)entry == -2 && atomicCAS(entry, -2, -3) == -2) {
          const int idx = atomicAdd(a.counters + LEVEL, 1);  // pool slots are pre-initialised (-1 nodes / 0 bricks)
          *(volatile int32_t*)entry = idx;
        }
      }
    });
  }
}

__global__ void __launch_bounds__(kBlock) ins_apply_kernel(const InsertArgs* __restrict__ jobs, int phase) {
  const InsertArgs a = jobs[blockIdx.y];
  const uint16_t* table = phase == 0 ? a.hit_table : a.miss_table;
  for (int i = blockIdx.x * kBlock + threadIdx.x; i < a.n; i += gridDim.x * kBlock) {
    for_each_cell(a, i, phase, [&](const Int3& c) {
      unsigned sx, sy, sz;
      shifted(a, c, &sx, &sy, &sz);
      const int node = a.top[((((sz >> 6) << a.bits) + (sy >> 6)) << a.bits) + (sx >> 6)];
      const int brick = a.nodes[(size_t)node * 512 + ((((sz >> 3) & 7) << 6) | (((sy >> 3) & 7) << 3) | ((sx >> 3) & 7))];
      const uint32_t cell = (uint32_t)brick * 512u + (((sz & 7) << 6) | ((sy & 7) << 3) | (sx & 7));
      unsigned* word = (unsigned*)a.bricks + (cell >> 1);
      const int shift = (cell & 1) * 16;
      unsigned old = *(volatile unsigned*)word;
      for (;;) {
        const uint16_t v = (uint16_t)(old >> shift);
        if (v >= 32768) return;  // already updated in this Insert (ApplyLookupTable returns false)
        const unsigned desired = (old & ~(0xFFFFu << shift)) | ((unsigned)table[v] << shift);
        const unsigned seen = atomicCAS(word, old, desired);
        if (seen == old) {
          a.update_list[atomicAdd(a.counters + 2, 1)] = cell;
          return;
        }
        old = seen;
      }
    });
  }
}

// FinishUpdate: remove the update marker from every cell touched by this Insert.
__global__ void ins_finish_kernel(const InsertArgs* __restrict__ jobs) {
  const InsertArgs a = jobs[blockIdx.y];
  const int count = a.counters[2];
  for (int k = blockIdx.x * kBlock + threadIdx.x; k < count; k += gridDim.x * kBlock) {
    const uint32_t cell = a.update_list[k];
    atomicSub((unsigned*)a.bricks + (cell >> 1), 32768u << ((cell & 1) * 16));  // the two halves of a word are different cells
  }
}

__global__ void transform_filter_kernel(const TransformJob* __restrict__ jobs, int pass) {
  // pass 0: transform + per-tile count of in-range points; pass 1: ordered scatter of the in-range ones. blockIdx.y = job.
  const TransformJob& job = jobs[blockIdx.y];
  const int n = job.n;
  if ((int)blockIdx.x * kBlock >= max(n, 1)) return;  // the launch covers the longest job (whole CTAs: the ballots below)
  const float* __restrict__ in = job.in;
  const Rigidf to_submap = job.to_submap;
  const Vec3f origin_submap = job.origin_submap;
  const float max_range = job.max_range;
  float* __restrict__ all = job.all;
  float* __restrict__ near = job.near;
  int32_t* tile_counts = job.tile_counts;
  __shared__ int warp_sums[kBlock / 32];
  const int i = blockIdx.x * kBlock + threadIdx.x;
  Vec3f p{0, 0, 0};
  int flag = 0;
  if (i < n) {
    p = apply(to_submap, Vec3f{in[3 * i], in[3 * i + 1], in[3 * i + 2]});
    flag = norm3(sub(p, origin_submap)) <= max_range;   // FilterRangeDataByMaxRange, submap_3d.cc:42-51
    if (pass == 0) { all[3 * i] = p.x; all[3 * i + 1] = p.y; all[3 * i + 2] = p.z; }
  }
  const unsigned ballot = __ballot_sync(0xffffffffu, flag);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) warp_sums[warp] = __popc(ballot);
  __syncthreads();
  int base = 0, total = 0;
  for (int w = 0; w < kBlock / 32; ++w) {
    if (w < warp) base += warp_sums[w];
    total += warp_sums[w];
  }
  if (pass == 0) {
    if (threadIdx.x == 0) tile_counts[blockIdx.x] = total;
    return;
  }
  int tile_base = 0;
  for (int t = 0; t < (int)blockIdx.x; ++t) tile_base += tile_counts[t];
  if (flag) {
    float* o = near + 3 * (size_t)(tile_base + base + __popc(ballot & ((1u << lane) - 1)));
    o[0] = p.x; o[1] = p.y; o[2] = p.z;
  }
  if ((int)blockIdx.x == (max(n, 1) + kBlock - 1) / kBlock - 1 && threadIdx.x == 0) *job.near_count = tile_base + total;
}

// range_data_in_local = opt_pose * returns / misses (LTB:559-560) and the gravity-aligned returns of the histogram
// (Rotation(gravity_alignment) * returns, LTB:605-610), float arithmetic of dl_math.cuh without contraction: the bits of the
// host loop it replaces. blockIdx.y = job; x covers returns, then misses.
__global__ void local_frame_kernel(const LocalFrameJob* __restrict__ jobs) {
  const LocalFrameJob& job = jobs[blockIdx.y];
  const int n = job.num_returns + job.num_misses;
  for (int i = blockIdx.x * kBlock + threadIdx.x; i < n; i += gridDim.x * kBlock) {
    const bool ret = i < job.num_returns;
    const int k = ret ? i : i - job.num_returns;
    const float* src = (ret ? job.returns : job.misses) + 3 * (size_t)k;
    const Vec3f p{src[0], src[1], src[2]};
    const Vec3f l = apply(job.pose, p);
    float* dst = (ret ? job.returns_local : job.misses_local) + 3 * (size_t)k;
    dst[0] = l.x; dst[1] = l.y; dst[2] = l.z;
    if (ret) {
      const Vec3f g = apply(job.gravity_alignment, p);
      float* d = job.returns_aligned + 3 * (size_t)k;
      d[0] = g.x; d[1] = g.y; d[2] = g.z;
    }
  }
}

}  // namespace

// ComputeLookupTableToApplyOdds (probability_values.cc:70-80), host float arithmetic (-ffp-contract=off).
void compute_odds_table(float probability, uint16_t* table) {
  auto clampf = [](float v, float lo, float hi) { return v > hi ? hi : (v < lo ? lo : v); };
  auto to_value = [&](float p) {
    const float lo = 0.1f, hi = 1.f - 0.1f;
    return (uint16_t)((int)lroundf((clampf(p, lo, hi) - lo) * (32766.f / (hi - lo))) + 1);
  };
  const float odds = probability / (1.f - probability);
  auto from_odds = [](float o) { return o / (o + 1.f); };
  table[0] = to_value(from_odds(odds)) + 32768;
  for (int cell = 1; cell != 32768; ++cell) {
    const float p = value_to_probability((uint16_t)cell);
    table[cell] = to_value(from_odds(odds * (p / (1.f - p)))) + 32768;
  }
}

size_t insert_args_bytes(int jobs) { return sizeof(InsertArgs) * (size_t)jobs; }

namespace {

// Grows every job's node pool (level 0) or brick pool (level 1) by exactly the number of entries its Insert marked
// (counters[3 + level], written by ins_claim_kernel<level, 0>). The grids' counters are gathered on the device into d_gather
// (8 ints per job) and read back in one copy: one host wait for all grids.
int reserve_pools(dl_context* ctx, std::vector<InsertArgs>& args, const std::vector<dl_grid*>& grids, int level, int32_t* d_gather) {
  for (size_t j = 0; j < grids.size(); ++j)
    DL_CUDA(ctx, cudaMemcpyAsync(d_gather + 8 * j, grids[j]->d_counters.get(), 5 * sizeof(int32_t), cudaMemcpyDeviceToDevice, ctx->stream));
  std::vector<int32_t> counters(8 * grids.size());
  DL_CUDA(ctx, cudaMemcpyAsync(counters.data(), d_gather, counters.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
  DL_CUDA(ctx, ctx->wait_stream());
  for (size_t j = 0; j < grids.size(); ++j) {
    dl_grid* g = grids[j];
    const int32_t* c = counters.data() + 8 * j;
    DL_TRY(grid_grow_pool(g, level, (size_t)c[level], (size_t)c[3 + level]));
    if (level == 0) args[j].nodes = g->d_nodes.get();
    else args[j].bricks = g->d_bricks.get();
  }
  return DL_OK;
}

// One round of insert_range_data_device: every grid at most once. bbox holds each job's box (8 ints, ins_bbox_kernel).
int insert_round(dl_context* ctx, std::vector<InsertArgs> args, const std::vector<dl_grid*>& grids, const std::vector<int32_t>& bbox,
                 int num_free, int32_t* d_bbox, InsertArgs* d_args) {
  const unsigned K = (unsigned)args.size();
  auto upload = [&]() -> int {
    DL_CUDA(ctx, cudaMemcpyAsync(d_args, args.data(), sizeof(InsertArgs) * K, cudaMemcpyHostToDevice, ctx->stream));
    return DL_OK;
  };
  int widest = 0;
  for (const InsertArgs& a : args) widest = std::max(widest, a.n);
  const dim3 blocks(std::min(kNumSMs * 8, (widest + kBlock - 1) / kBlock), K);
  // 1. top-level growth of whichever grids need it
  for (unsigned j = 0; j < K; ++j) {
    dl_grid* g = grids[j];
    const int32_t* bb = bbox.data() + 8 * j;
    for (;;) {
      const int half = (64 << g->bits) >> 1;
      bool fits = true;
      for (int k = 0; k < 3; ++k) fits = fits && bb[k] >= -half && bb[3 + k] < half;
      if (fits) break;
      if (g->bits + 1 > 8) return ctx->fail(DL_ERR_GRID_RANGE, "cell index outside +-8192 cells");
      const size_t new_size = (size_t)8 << (3 * g->bits);
      DeviceBuffer<int32_t> grown;
      DL_TRY(alloc(ctx, grown, new_size, 0xFF));
      const int old_cells = 1 << (3 * g->bits);
      grid_grow_kernel<<<(old_cells + 255) / 256, 256, 0, ctx->stream>>>(g->d_top.get(), g->bits, grown.get());
      DL_LAUNCH_CHECK(ctx, "grid_grow_kernel");
      DL_CUDA(ctx, ctx->wait_stream());
      g->d_top = std::move(grown);
      g->bits += 1;
      // from here on the device copy is ahead of the host mirror, whatever happens next: a later failure (range, out of
      // memory) must not leave g->bits describing a host `top` of the old size
      g->mirror_stale = true;
      g->version++;
    }
  }
  // 2. structure growth with exact reservations: mark + count the missing nodes, grow the node pools by those counts, assign;
  //    then the same for the bricks (whose node entries now exist)
  for (unsigned j = 0; j < K; ++j) {
    dl_grid* g = grids[j];
    InsertArgs& a = args[j];
    a.bits = g->bits; a.top = g->d_top.get(); a.nodes = g->d_nodes.get(); a.bricks = g->d_bricks.get(); a.counters = g->d_counters.get();
    DL_CUDA(ctx, cudaMemsetAsync(g->d_counters.get() + 2, 0, 3 * sizeof(int32_t), ctx->stream));
  }
  DL_TRY(upload());
  const int phases = num_free > 0 ? 2 : 1;
  for (int phase = 0; phase < phases; ++phase) {
    ins_claim_kernel<0, 0><<<blocks, kBlock, 0, ctx->stream>>>(d_args, phase);
    DL_LAUNCH_CHECK(ctx, "ins_claim_kernel<0,0>");
  }
  for (dl_grid* g : grids) {  // top entries are marked: the device copy is the only consistent one until the Insert completes
    g->mirror_stale = true;
    g->version++;
  }
  DL_TRY(reserve_pools(ctx, args, grids, 0, d_bbox));
  DL_TRY(upload());
  for (int phase = 0; phase < phases; ++phase) {
    ins_claim_kernel<0, 1><<<blocks, kBlock, 0, ctx->stream>>>(d_args, phase);
    DL_LAUNCH_CHECK(ctx, "ins_claim_kernel<0,1>");
  }
  for (int phase = 0; phase < phases; ++phase) {
    ins_claim_kernel<1, 0><<<blocks, kBlock, 0, ctx->stream>>>(d_args, phase);
    DL_LAUNCH_CHECK(ctx, "ins_claim_kernel<1,0>");
  }
  DL_TRY(reserve_pools(ctx, args, grids, 1, d_bbox));
  DL_TRY(upload());
  for (int phase = 0; phase < phases; ++phase) {
    ins_claim_kernel<1, 1><<<blocks, kBlock, 0, ctx->stream>>>(d_args, phase);
    DL_LAUNCH_CHECK(ctx, "ins_claim_kernel<1,1>");
  }
  ins_apply_kernel<<<blocks, kBlock, 0, ctx->stream>>>(d_args, 0);
  DL_LAUNCH_CHECK(ctx, "ins_apply_kernel(hits)");
  if (num_free > 0) {
    ins_apply_kernel<<<blocks, kBlock, 0, ctx->stream>>>(d_args, 1);
    DL_LAUNCH_CHECK(ctx, "ins_apply_kernel(misses)");
  }
  ins_finish_kernel<<<blocks, kBlock, 0, ctx->stream>>>(d_args);
  DL_LAUNCH_CHECK(ctx, "ins_finish_kernel");
  for (dl_grid* g : grids) {
    g->mirror_stale = true;
    g->version++;
  }
  return DL_OK;
}

}  // namespace

int insert_range_data_device(dl_context* ctx, const InsertJob* jobs, int count, int num_free, const uint16_t* d_hit_table,
                             const uint16_t* d_miss_table, int32_t* d_bbox, void* d_args_raw) {
  InsertArgs* d_args = (InsertArgs*)d_args_raw;
  std::vector<InsertArgs> args;
  std::vector<dl_grid*> grids;
  int widest = 0;
  for (int j = 0; j < count; ++j) {
    const InsertJob& job = jobs[j];
    if (job.n <= 0) continue;
    DL_TRY(grid_ensure_device_state(job.grid));
    InsertArgs a{};
    a.returns = job.returns; a.n = job.n; a.n_dev = job.n_dev; a.origin = job.origin; a.resolution = job.grid->resolution;
    a.num_free = num_free; a.bbox = d_bbox + 8 * args.size(); a.update_list = job.update_list;
    a.hit_table = d_hit_table; a.miss_table = d_miss_table;
    args.push_back(a);
    grids.push_back(job.grid);
    widest = std::max(widest, job.n);
  }
  if (args.empty()) return DL_OK;
  const unsigned J = (unsigned)args.size();
  // 1. which cells will be touched, and how long the rays are: one pass over every job of every round, one read-back
  std::vector<int32_t> bbox(8 * J);
  for (unsigned j = 0; j < J; ++j) {
    const int32_t init[8] = {0x7fffffff, 0x7fffffff, 0x7fffffff, -0x7fffffff, -0x7fffffff, -0x7fffffff, 0, 0};
    std::memcpy(bbox.data() + 8 * j, init, sizeof(init));
  }
  DL_CUDA(ctx, cudaMemcpyAsync(d_bbox, bbox.data(), sizeof(int32_t) * 8 * J, cudaMemcpyHostToDevice, ctx->stream));
  DL_CUDA(ctx, cudaMemcpyAsync(d_args, args.data(), sizeof(InsertArgs) * J, cudaMemcpyHostToDevice, ctx->stream));
  ins_bbox_kernel<<<dim3(std::min(kNumSMs * 8, (widest + kBlock - 1) / kBlock), J), kBlock, 0, ctx->stream>>>(d_args);
  DL_LAUNCH_CHECK(ctx, "ins_bbox_kernel");
  // the device counts ride in the unused seventh int of each job's box: one read-back, one host wait for every job
  for (unsigned j = 0; j < J; ++j)
    if (args[j].n_dev)
      DL_CUDA(ctx, cudaMemcpyAsync(d_bbox + 8 * j + 6, args[j].n_dev, sizeof(int32_t), cudaMemcpyDeviceToDevice, ctx->stream));
  DL_CUDA(ctx, cudaMemcpyAsync(bbox.data(), d_bbox, sizeof(int32_t) * 8 * J, cudaMemcpyDeviceToHost, ctx->stream));
  DL_CUDA(ctx, ctx->wait_stream());
  // jobs whose count on the device is zero drop out; the others carry their exact count from here on
  {
    std::vector<InsertArgs> kept_args;
    std::vector<dl_grid*> kept_grids;
    std::vector<int32_t> kept_bbox;
    for (unsigned j = 0; j < J; ++j) {
      if (args[j].n_dev) args[j].n = bbox[8 * j + 6];
      args[j].n_dev = nullptr;
      if (args[j].n <= 0) continue;
      kept_args.push_back(args[j]);
      kept_grids.push_back(grids[j]);
      kept_bbox.insert(kept_bbox.end(), bbox.begin() + 8 * j, bbox.begin() + 8 * j + 8);
    }
    args.swap(kept_args);
    grids.swap(kept_grids);
    bbox.swap(kept_bbox);
  }
  // 2. the checks that refuse a call run before any grid changes: CHECK_LT(num_samples, 1 << 15) (range_data_inserter_3d.cc:37)
  //    and CHECK_LE(new_bits, 8) (hybrid_grid.h:391), i.e. every touched cell within +-8192 cells
  const unsigned K = (unsigned)args.size();
  for (unsigned j = 0; j < K; ++j) {
    const int32_t* bb = bbox.data() + 8 * j;
    if (bb[7] >= kMaxSamples) return ctx->fail(DL_ERR_ARG, "a ray crosses 2^15 cells or more (CHECK_LT(num_samples, 1 << 15))");
    for (int k = 0; k < 3; ++k)
      if (bb[k] < -8192 || bb[3 + k] >= 8192) return ctx->fail(DL_ERR_GRID_RANGE, "cell index outside +-8192 cells");
  }
  // 3. a grid named by several jobs takes them in list order, one round each: a round takes the first pending job of every grid
  std::vector<char> done(K, 0);
  for (unsigned left = K; left > 0;) {
    std::vector<InsertArgs> round_args;
    std::vector<dl_grid*> round_grids;
    std::vector<int32_t> round_bbox;
    for (unsigned j = 0; j < K; ++j) {
      if (done[j] || std::find(round_grids.begin(), round_grids.end(), grids[j]) != round_grids.end()) continue;
      done[j] = 1;
      --left;
      round_args.push_back(args[j]);
      round_grids.push_back(grids[j]);
      round_bbox.insert(round_bbox.end(), bbox.begin() + 8 * j, bbox.begin() + 8 * j + 8);
    }
    DL_TRY(insert_round(ctx, round_args, round_grids, round_bbox, num_free, d_bbox, d_args));
  }
  return DL_OK;
}

size_t transform_jobs_bytes(int jobs) { return sizeof(TransformJob) * (size_t)jobs; }

int launch_transform_filter(dl_context* ctx, const TransformJob* jobs, int count, void* d_jobs) {
  int widest = 0;
  for (int j = 0; j < count; ++j) widest = std::max(widest, jobs[j].n);
  if (widest <= 0) return DL_OK;
  DL_CUDA(ctx, cudaMemcpyAsync(d_jobs, jobs, sizeof(TransformJob) * (size_t)count, cudaMemcpyHostToDevice, ctx->stream));
  const dim3 tiles((widest + kBlock - 1) / kBlock, count);
  for (int pass = 0; pass < 2; ++pass) {
    transform_filter_kernel<<<tiles, kBlock, 0, ctx->stream>>>((const TransformJob*)d_jobs, pass);
    DL_LAUNCH_CHECK(ctx, "transform_filter_kernel");
  }
  return DL_OK;
}

size_t local_frame_jobs_bytes(int jobs) { return sizeof(LocalFrameJob) * (size_t)jobs; }

int launch_local_frame(dl_context* ctx, const LocalFrameJob* jobs, int count, void* d_jobs) {
  int widest = 0;
  for (int j = 0; j < count; ++j) widest = std::max(widest, jobs[j].num_returns + jobs[j].num_misses);
  if (widest <= 0) return DL_OK;
  DL_CUDA(ctx, cudaMemcpyAsync(d_jobs, jobs, sizeof(LocalFrameJob) * (size_t)count, cudaMemcpyHostToDevice, ctx->stream));
  local_frame_kernel<<<dim3(std::min(64, (widest + kBlock - 1) / kBlock), count), kBlock, 0, ctx->stream>>>((const LocalFrameJob*)d_jobs);
  DL_LAUNCH_CHECK(ctx, "local_frame_kernel");
  return DL_OK;
}

}  // namespace dl

// ------------------------------------------------------------------------------------------------ grid write side
using namespace dl;

namespace {
uint32_t* take_update_list(Arena& a, const dl_range_data_inserter_options& o, int64_t n) {
  return a.take<uint32_t>((size_t)n * (size_t)(1 + std::max(o.num_free_space_voxels, 0)));
}
}  // namespace

namespace dl {
// The scratch every insert_range_data_device call of `jobs` jobs shares; each job's update list is carved by take_update_list.
void carve_insert(Arena& a, int jobs, InsertScratch* s) {
  s->hit_table = a.take<uint16_t>(32768);
  s->miss_table = a.take<uint16_t>(32768);
  s->bbox = a.take<int32_t>(8 * (size_t)std::max(jobs, 1));
  s->args = a.take<char>(insert_args_bytes(std::max(jobs, 1)));
}
void carve_submap_insert(Arena& a, const dl_range_data_inserter_options& o, int64_t n, SubmapInsertScratch* s) {
  s->all = a.take<float>(3 * (size_t)n);
  s->near = a.take<float>(3 * (size_t)n);
  s->near_count = a.take<int32_t>(1);
  s->tiles = a.take<int32_t>((size_t)(n + 255) / 256 + 1);
  s->update_hi = take_update_list(a, o, n);
  s->update_lo = take_update_list(a, o, n);
}
// Submap3D::InsertRangeData of `returns` (n points, local frame, device) into the submap at `submap_local_pose`: the transform
// job that moves them into the submap frame and the two Insert jobs that read its output.
void submap_insert_jobs(dl_grid* hi, dl_grid* lo, const double* submap_local_pose, int32_t high_resolution_max_range,
                        const float* origin, const float* d_returns, int n, const SubmapInsertScratch& s, TransformJob* transform,
                        InsertJob* inserts) {
  // TransformRangeData(range_data, local_pose().inverse().cast<float>())
  const Rigidf to_submap = to_float(inverse(pose_from7(submap_local_pose)));
  const Vec3f origin_submap = apply(to_submap, Vec3f{origin[0], origin[1], origin[2]});
  *transform = TransformJob{d_returns, n, to_submap, origin_submap, (float)high_resolution_max_range, s.all, s.near, s.near_count, s.tiles};
  inserts[0] = InsertJob{hi, origin_submap, s.near, n, s.near_count, s.update_hi};
  inserts[1] = InsertJob{lo, origin_submap, s.all, n, nullptr, s.update_lo};
}
int upload_odds_tables(dl_context* ctx, const dl_range_data_inserter_options& o, const InsertScratch& s) {
  static thread_local std::vector<uint16_t> tables(65536);
  static thread_local double cached_hit = -1, cached_miss = -1;
  if (cached_hit != o.hit_probability || cached_miss != o.miss_probability) {
    compute_odds_table((float)o.hit_probability, tables.data());           // Odds(options.hit_probability()) takes a float
    compute_odds_table((float)o.miss_probability, tables.data() + 32768);
    cached_hit = o.hit_probability;
    cached_miss = o.miss_probability;
  }
  DL_TRY(h2d(ctx, s.hit_table, tables.data(), 32768));
  DL_TRY(h2d(ctx, s.miss_table, tables.data() + 32768, 32768));
  return DL_OK;
}
int check_inserter(dl_context* ctx, const dl_range_data_inserter_options* o) {
  if (!o) return DL_ERR_ARG;
  if (!(o->hit_probability > 0.5) || !(o->miss_probability < 0.5) || o->num_free_space_voxels < 0)
    return ctx->fail(DL_ERR_ARG, "hit_probability must be > 0.5 and miss_probability < 0.5 (CHECK_GT / CHECK_LT)");
  return DL_OK;
}
}  // namespace dl

extern "C" {

int dl_grid_insert_range_data(dl_context* ctx, dl_grid* grid, const dl_range_data_inserter_options* options,
                              const float* origin, const float* returns, int64_t n) {
  if (!ctx || !grid || !origin || n < 0 || n > 0x3fffffff || (n > 0 && !returns)) return DL_ERR_ARG;  // CHECK_NOTNULL(hybrid_grid)
  DL_TRY(check_inserter(ctx, options));
  if (n == 0) return DL_OK;
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  float* d_returns;
  uint32_t* update_list;
  InsertScratch s;
  DL_TRY(carve_scratch(ctx, [&](Arena& a) {
    d_returns = a.take<float>(3 * n);
    carve_insert(a, 1, &s);
    update_list = take_update_list(a, *options, n);
  }));
  DL_TRY(h2d(ctx, d_returns, returns, 3 * n));
  DL_TRY(upload_odds_tables(ctx, *options, s));
  const InsertJob job{grid, Vec3f{origin[0], origin[1], origin[2]}, d_returns, (int)n, nullptr, update_list};
  DL_TRY(insert_range_data_device(ctx, &job, 1, options->num_free_space_voxels, s.hit_table, s.miss_table, s.bbox, s.args));
  return sync(ctx);
}

int dl_submap_insert_range_data(dl_context* ctx, dl_grid* hi, dl_grid* lo, const dl_range_data_inserter_options* options,
                                const double* submap_local_pose, int32_t high_resolution_max_range, const float* origin,
                                const float* returns, int64_t n) {
  if (!ctx || !hi || !lo || !submap_local_pose || !origin || n < 0 || n > 0x3fffffff || (n > 0 && !returns)) return DL_ERR_ARG;
  DL_TRY(check_inserter(ctx, options));
  if (n == 0) return DL_OK;
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  float* d_in;
  void* d_transform;
  SubmapInsertScratch t;
  InsertScratch s;
  DL_TRY(carve_scratch(ctx, [&](Arena& a) {
    d_in = a.take<float>(3 * n);
    d_transform = a.take<char>(transform_jobs_bytes(1));
    carve_submap_insert(a, *options, n, &t);
    carve_insert(a, 2, &s);
  }));
  DL_TRY(h2d(ctx, d_in, returns, 3 * n));
  TransformJob transform;
  InsertJob jobs[2];
  submap_insert_jobs(hi, lo, submap_local_pose, high_resolution_max_range, origin, d_in, (int)n, t, &transform, jobs);
  DL_TRY(launch_transform_filter(ctx, &transform, 1, d_transform));
  DL_TRY(upload_odds_tables(ctx, *options, s));
  DL_TRY(insert_range_data_device(ctx, jobs, 2, options->num_free_space_voxels, s.hit_table, s.miss_table, s.bbox, s.args));
  return sync(ctx);
}

}  // extern "C"
