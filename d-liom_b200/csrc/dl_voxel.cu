// Voxel hashing kernels: first-point-per-voxel filter and its adaptive (bisection) variant.
//
// Replaces sensor::VoxelFilter::Filter / AdaptiveVoxelFilter::Filter
// (C/sensor/internal/voxel_filter.cc:28-131,147-150). The reference inserts 96-bit keys into a
// std::unordered_set in input order and keeps a point iff its insertion succeeded. Here every point
// atomically proposes its input index to an open-addressing table slot keyed by the voxel; the slot keeps
// the MINIMUM index (atomicMin), so the survivor of each voxel is the first point in input order regardless
// of thread scheduling, and an order-preserving compaction returns exactly the reference's output.
// The table stores only point indices (4 B/slot): a slot's key is the voxel of whichever point currently owns
// it, which is invariant under atomicMin among points of the same voxel.
//
// HBM traffic per pass (algorithmic): read stride*4 B per point, write 4 B per survivor. The table (8 B per
// point) lives in L2. Compile with -fmad=false: index = lroundf(x / resolution) must match the CPU bit for bit.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "dl_internal.cuh"

namespace dl {
namespace {

constexpr uint32_t kEmpty = 0xFFFFFFFFu;
constexpr int kBlock = 256;

__device__ __forceinline__ uint32_t hash_cell(const Int3& c) {
  uint32_t h = (uint32_t)c.x * 73856093u ^ (uint32_t)c.y * 19349663u ^ (uint32_t)c.z * 83492791u;
  h ^= h >> 15;
  h *= 0x2c1b3c6du;
  h ^= h >> 12;
  return h;
}
__device__ __forceinline__ Int3 row_cell(const float* __restrict__ pts, int stride, uint32_t row, float res) {
  const float* p = pts + (size_t)row * stride;
  return cell_index(Vec3f{p[0], p[1], p[2]}, res);
}

// Proposes `id` (position in the filter's input order) for the voxel `c`. `row_of(id)` maps ids to rows.
template <typename RowOf>
__device__ __forceinline__ uint32_t table_insert(uint32_t* table, uint32_t mask, const float* pts, int stride,
                                                 float res, const Int3& c, uint32_t id, RowOf row_of) {
  uint32_t h = hash_cell(c) & mask;
  for (;;) {
    const uint32_t prev = atomicCAS(table + h, kEmpty, id);
    if (prev == kEmpty) return h;
    const Int3 o = row_cell(pts, stride, row_of(prev), res);
    if (o.x == c.x && o.y == c.y && o.z == c.z) {
      atomicMin(table + h, id);
      return h;
    }
    h = (h + 1) & mask;
  }
}

// ------------------------------------------------------------------------------------------- plain filter
__global__ void __launch_bounds__(kBlock) voxel_insert_kernel(const float* __restrict__ points, int stride,
                                                              int64_t cap, const int32_t* __restrict__ counts,
                                                              float res, uint32_t* table, int64_t table_cap,
                                                              uint32_t* slot) {
  const int b = blockIdx.y;
  const int n = counts[b];
  const float* pts = points + (size_t)b * cap * stride;
  uint32_t* tab = table + (size_t)b * table_cap;
  const uint32_t mask = (uint32_t)table_cap - 1;
  for (int i = blockIdx.x * kBlock + threadIdx.x; i < n; i += gridDim.x * kBlock) {
    const Int3 c = row_cell(pts, stride, i, res);
    slot[(size_t)b * cap + i] = table_insert(tab, mask, pts, stride, res, c, (uint32_t)i, [](uint32_t id) { return id; });
  }
}

__device__ __forceinline__ int block_exclusive_scan(int value, int* total) {
  __shared__ int warp_sums[kBlock / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int inc = value;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int o = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc += o;
  }
  __syncthreads();  // protects warp_sums across successive calls
  if (lane == 31) warp_sums[warp] = inc;
  __syncthreads();
  int base = 0, sum = 0;
#pragma unroll
  for (int w = 0; w < kBlock / 32; ++w) {
    const int s = warp_sums[w];
    if (w < warp) base += s;
    sum += s;
  }
  *total = sum;
  return base + inc - value;
}

// Per 256-row tile: number of survivors (a row survives iff it owns its slot).
__global__ void __launch_bounds__(kBlock) voxel_count_kernel(const int32_t* __restrict__ counts, int64_t cap,
                                                             const uint32_t* __restrict__ table, int64_t table_cap,
                                                             const uint32_t* __restrict__ slot, int32_t* block_counts,
                                                             int tiles) {
  const int b = blockIdx.y;
  const int n = counts[b];
  const int i = blockIdx.x * kBlock + threadIdx.x;
  int flag = 0;
  if (i < n) flag = __ldcg(table + (size_t)b * table_cap + slot[(size_t)b * cap + i]) == (uint32_t)i;
  int total;
  block_exclusive_scan(flag, &total);
  if (threadIdx.x == 0) block_counts[(size_t)b * tiles + blockIdx.x] = total;
}

__global__ void __launch_bounds__(kBlock) voxel_scatter_kernel(const int32_t* __restrict__ counts, int64_t cap,
                                                               const uint32_t* __restrict__ table, int64_t table_cap,
                                                               const uint32_t* __restrict__ slot,
                                                               const int32_t* __restrict__ block_counts, int tiles,
                                                               int32_t* keep, int32_t* keep_counts) {
  const int b = blockIdx.y;
  const int n = counts[b];
  __shared__ int tile_base;
  // prefix over the preceding tiles of this cloud (<= 1024 tiles for 262 144 rows)
  int partial = 0;
  for (int t = threadIdx.x; t < (int)blockIdx.x; t += kBlock) partial += block_counts[(size_t)b * tiles + t];
  int total;
  block_exclusive_scan(partial, &total);
  if (threadIdx.x == 0) tile_base = total;
  __syncthreads();
  const int i = blockIdx.x * kBlock + threadIdx.x;
  int flag = 0;
  if (i < n) flag = __ldcg(table + (size_t)b * table_cap + slot[(size_t)b * cap + i]) == (uint32_t)i;
  const int off = block_exclusive_scan(flag, &total);
  if (flag) keep[(size_t)b * cap + tile_base + off] = i;
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) keep_counts[b] = tile_base + total;
}

__global__ void voxel_indices_kernel(const float* __restrict__ points, int stride, int64_t n, float res,
                                     int32_t* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  // the reciprocal-multiply fast path with its exact fallback (dl_math.cuh round_div): what the fused front end uses
  const float* p = points + (size_t)i * stride;
  const Int3 c = cell_index(Vec3f{p[0], p[1], p[2]}, make_divider(res));
  out[3 * i] = c.x;
  out[3 * i + 1] = c.y;
  out[3 * i + 2] = c.z;
}

// ------------------------------------------------------------------------------------------- adaptive filter
// One CTA runs the whole data-dependent pass sequence of AdaptivelyVoxelFiltered for one (cloud, filter) pair, so the bisection
// needs no host round trip. Every pair takes this search, the already sparse ones and those that stop at the first edge
// included: a cloud that passes through costs two sweeps (the crop count, then the ordered copy). The CTA is small (512
// threads, 34 KiB of shared memory, two per SM): a sub-batch's pairs run in one wave and share their SMs with the kernels that overlap them. Nothing of the cloud is cached; every sweep streams the pair's rows (they stay in
// L2) and repeats the range crop.
//
// The search passes only need the NUMBER of voxels at an edge (voxel_filter.cc:47,57,63), a pure function of the edge, so one sweep
// counts several edges: each gets a byte map over the cloud's cell box at that edge (cell_index is monotone per axis, so every cell
// lies in [cell(min corner), cell(max corner)]), a point stores a 1 into its cell's byte (a plain store: all writers write the same
// value, so no atomics and no read), and the count is the number of non-zero bytes. The search
// (adaptive_search, unchanged) then replays on the stored counts. The first edge it asks for that has not been counted ends the
// replay and the next sweep counts it. While the search is still halving, that sweep also counts the next halving e/2 and the
// midpoint (e/2 + e)/2 that the bisection of [e/2, e] asks for first. On the front end's clouds that is {L, L/2, 3L/4} and then one
// sweep per further step of the bisection of [L/2, L]: a sweep costs about as much as loading and cropping the cloud plus one edge,
// so counting every midpoint the bisection can reach ahead (up to 9 edges in one sweep instead of 3 sweeps) measured slower. A last sweep at the result edge inserts every point into a small hash table (packed key, min row);
// its minima are the survivors. Rows rather than cropped positions identify points: the crop keeps input
// order, so the first point of a voxel is the same either way.
//
// What shared memory cannot hold (one edge's box beyond the whole byte-map budget, more voxels than the result table, a key that
// does not pack) sends the pair to generic mode: the same search on an index-only table in global memory.
constexpr int kSearchBlock = 512;
constexpr int kSearchWarps = kSearchBlock / 32;
constexpr int kMapBytes = 32768;    // 32 KiB of byte maps, shared by the edges of one sweep
constexpr int kResultSlots = 2048;  // result table: packed key 8 B + min row 4 B per slot, and 4 B per survivor to order them
constexpr int kMaxAhead = 3;        // edges counted by one sweep
constexpr int kKnownEdges = 64;     // counted edges of one search
constexpr unsigned long long kEmptyKey = 0xFFFFFFFFFFFFFFFFull;

__device__ __forceinline__ int block_sum(int v) {
  __shared__ int ws[kSearchWarps];
  __shared__ int result;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  __syncthreads();
  if (lane == 0) ws[warp] = v;
  __syncthreads();
  if (warp == 0) {
    int s = lane < kSearchWarps ? ws[lane] : 0;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
    if (lane == 0) result = s;
  }
  __syncthreads();
  return result;
}

// Exclusive prefix of one value per warp over the warps of the CTA (value must be warp-uniform); *total = the sum.
__device__ __forceinline__ int warp_bases(int warp_value, int* total) {
  __shared__ int ws[kSearchWarps], wb[kSearchWarps + 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();  // protects ws / wb across successive calls
  if (lane == 0) ws[warp] = warp_value;
  __syncthreads();
  if (warp == 0) {
    const int v = lane < kSearchWarps ? ws[lane] : 0;
    int inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int o = __shfl_up_sync(0xffffffffu, inc, d);
      if (lane >= d) inc += o;
    }
    if (lane < kSearchWarps) wb[lane] = inc - v;
    if (lane == 31) wb[kSearchWarps] = inc;
  }
  __syncthreads();
  *total = wb[kSearchWarps];
  return wb[warp];
}

// Order-preserving compaction of ids [0, n) with predicate flags computed by `pred` (pure: it is evaluated twice). Every warp
// owns a contiguous chunk of ids: it counts its flags (no barrier between its rounds, so the loads behind `pred` pipeline), ONE
// block scan turns the per-warp counts into bases, and a second sweep writes. block_compact runs the three steps and returns the
// count; the adaptive search runs them apart, with its first sweep as the counting one.
template <typename Pred>
__device__ __forceinline__ int warp_chunk_count(int n, Pred pred) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int chunk = ((n + kSearchBlock - 1) / kSearchBlock) * 32;  // ids per warp, a multiple of 32
  const int begin = warp * chunk, end = min(n, begin + chunk);
  // four 32-id rounds per iteration: the four loads behind `pred` are in flight together (a ballot per round would serialise them)
  int count = 0;
  for (int base = begin; base < end; base += 128) {
    bool f[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int i = base + 32 * u + lane;
      f[u] = i < end && pred(i);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) count += __popc(__ballot_sync(0xffffffffu, f[u]));
  }
  return count;
}
// `pos`: the warp's base from warp_bases over the counts of warp_chunk_count.
template <typename Pred, typename Emit>
__device__ __forceinline__ void warp_chunk_emit(int n, int pos, Pred pred, Emit emit) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int chunk = ((n + kSearchBlock - 1) / kSearchBlock) * 32;
  const int begin = warp * chunk, end = min(n, begin + chunk);
  for (int base = begin; base < end; base += 128) {
    bool f[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int i = base + 32 * u + lane;
      f[u] = i < end && pred(i);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const unsigned ballot = __ballot_sync(0xffffffffu, f[u]);
      if (f[u]) emit(pos + __popc(ballot & ((1u << lane) - 1)), base + 32 * u + lane);
      pos += __popc(ballot);
    }
  }
  __syncthreads();  // the emitted list is complete for every reader
}
template <typename Pred, typename Emit>
__device__ __forceinline__ int block_compact(int n, Pred pred, Emit emit) {
  int total;
  const int pos = warp_bases(warp_chunk_count(n, pred), &total);
  warp_chunk_emit(n, pos, pred, emit);
  return total;
}

// The reference's search over voxel edge lengths (AdaptivelyVoxelFiltered, voxel_filter.cc:40-77), statement for
// statement, parameterised by `run_pass(edge) -> number of voxels` (negative = the pass could not be run in the
// current mode). Returns false if a pass failed; otherwise *result_edge is the edge whose survivors are the result.
template <typename RunPass>
__device__ __forceinline__ bool adaptive_search(const AdaptiveParams& opt, RunPass run_pass, float* result_edge) {
  *result_edge = opt.max_length;
  int result_count = run_pass(opt.max_length);
  if (result_count < 0) return false;
  if ((float)result_count >= opt.min_num_points) return true;
  for (float high_length = opt.max_length; high_length > 1e-2f * opt.max_length; high_length /= 2.f) {
    float low_length = high_length / 2.f;
    result_count = run_pass(low_length);
    if (result_count < 0) return false;
    *result_edge = low_length;
    if ((float)result_count >= opt.min_num_points) {
      while ((high_length - low_length) / low_length > 1e-1f) {
        const float mid_length = (low_length + high_length) / 2.f;
        const int candidate = run_pass(mid_length);
        if (candidate < 0) return false;
        if ((float)candidate >= opt.min_num_points) {
          low_length = mid_length;
          *result_edge = mid_length;
        } else {
          high_length = mid_length;
        }
      }
      return true;
    }
  }
  return true;
}

__device__ __forceinline__ bool pack_cell(const Int3& c, unsigned long long* key) {
  const int lim = 1 << 20;
  if (c.x < -lim || c.x >= lim - 1 || c.y < -lim || c.y >= lim - 1 || c.z < -lim || c.z >= lim - 1) return false;
  *key = ((unsigned long long)(c.x + lim) << 42) | ((unsigned long long)(c.y + lim) << 21) | (unsigned long long)(c.z + lim);
  return true;
}
__device__ __forceinline__ uint32_t hash_key(unsigned long long k) {
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdull;
  k ^= k >> 29;
  return (uint32_t)k;
}

union SearchShared {
  uint4 maps[kMapBytes / 16];
  struct {
    unsigned long long keys[kResultSlots];
    uint32_t mins[kResultSlots];
    uint32_t rows[kResultSlots];  // the survivors, unordered
  } result;
};
struct EdgeBox {  // one edge of a sweep: its byte map covers cells lo + [0, nx) x [0, ny) x [0, cells / (nx ny))
  CellDivider div;
  int lo[3], nx, ny, cells, map0;  // map0: offset of the map in sixteen-byte words
};
struct SearchState {
  float lo[3], hi[3];  // bounding box of the cropped cloud
  float box_warp[6][kSearchWarps];
  int num_set, words;  // the edges of the next sweep and the sixteen-byte words their maps take
  EdgeBox set[kMaxAhead];
  int set_count[kMaxAhead];
  int num_known;  // every edge counted so far, with its number of voxels
  float known_edge[kKnownEdges];
  int known_count[kKnownEdges];
  int fail, survivors;
};

__device__ __forceinline__ int find_edge(const float* edges, int num, float edge) {
  for (int k = 0; k < num; ++k)
    if (__float_as_uint(edges[k]) == __float_as_uint(edge)) return k;
  return -1;
}

// Adds `edge` to the next sweep unless it is counted or queued already; false if its byte map does not fit in what is left.
__device__ bool place_edge(SearchState& st, float edge) {
  if (find_edge(st.known_edge, st.num_known, edge) >= 0) return true;
  for (int k = 0; k < st.num_set; ++k)
    if (__float_as_uint(st.set[k].div.resolution) == __float_as_uint(edge)) return true;
  if (st.num_set == kMaxAhead || st.num_known + st.num_set == kKnownEdges) return false;
  const CellDivider div = make_divider(edge);
  const Int3 lo = cell_index(Vec3f{st.lo[0], st.lo[1], st.lo[2]}, div), hi = cell_index(Vec3f{st.hi[0], st.hi[1], st.hi[2]}, div);
  const long long nx = (long long)hi.x - lo.x + 1, ny = (long long)hi.y - lo.y + 1, nz = (long long)hi.z - lo.z + 1;
  const long long budget = 16LL * (kMapBytes / 16 - st.words);
  if (nx <= 0 || ny <= 0 || nz <= 0 || nx > budget || ny > budget || nz > budget || nx * ny * nz > budget) return false;
  EdgeBox& b = st.set[st.num_set++];
  b.div = div;
  b.lo[0] = lo.x; b.lo[1] = lo.y; b.lo[2] = lo.z;
  b.nx = (int)nx; b.ny = (int)ny; b.cells = (int)(nx * ny * nz);
  b.map0 = st.words;
  st.words += (b.cells + 15) >> 4;
  return true;
}

// cell_index(p, d) when no axis needs round_div's division: round_div's fast path for the three axes as straight-line code, so
// that the compiler can interleave the axes and the points of a batch. Returns false (and leaves *c unset) when an axis lies too
// close to a rounding boundary or out of the fast path's range; the caller then takes cell_index, which divides.
__device__ __forceinline__ bool cell_index_fast(const Vec3f& p, const CellDivider& d, Int3* c) {
  const float v[3] = {p.x, p.y, p.z};
  int k[3];
  bool ok = true;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float q = v[a] * d.inverse;
    const float aq = fabsf(q);
    const float t = aq + 12582912.f;
    const float dist = fabsf(aq - (t - 12582912.f));
    ok = ok && aq < 4194304.f && 0.5f - dist > aq * 4.8e-7f + 1e-30f;
    const int r = __float_as_int(t) - 0x4B400000;
    k[a] = q < 0.f ? -r : r;
  }
  *c = Int3{k[0], k[1], k[2]};
  return ok;
}

// One sweep over the pair's rows: every cropped point marks its cell in the byte map of every queued edge; the edges and their
// numbers of voxels are then appended to the known ones.
__device__ void count_sweep(SearchShared& sm, SearchState& st, const float* __restrict__ pts, int stride, int n, float max_range) {
  for (int i = threadIdx.x; i < st.words; i += kSearchBlock) sm.maps[i] = make_uint4(0u, 0u, 0u, 0u);
  if (threadIdx.x < kMaxAhead) st.set_count[threadIdx.x] = 0;
  __syncthreads();
  const int num_set = st.num_set;
  constexpr int kBatch = 3;
  for (int base = 0; base < n; base += kBatch * kSearchBlock) {
    Vec3f v[kBatch];
    bool in[kBatch];
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {  // the loads of a batch are in flight together
      const int i = base + u * kSearchBlock + threadIdx.x;
      in[u] = false;
      v[u] = Vec3f{0.f, 0.f, 0.f};
      if (i < n) {
        const float* p = pts + (size_t)i * stride;
        v[u] = Vec3f{p[0], p[1], p[2]};
        in[u] = norm3(v[u]) <= max_range;  // FilterByMaxRange (voxel_filter.cc:28-38)
      }
    }
    for (int k = 0; k < num_set; ++k) {
      const EdgeBox b = st.set[k];
      unsigned idx[kBatch];
#pragma unroll
      for (int u = 0; u < kBatch; ++u) {
        Int3 c;
        if (!cell_index_fast(v[u], b.div, &c) && in[u]) c = cell_index(v[u], b.div);
        idx[u] = (unsigned)(((c.z - b.lo[2]) * b.ny + (c.y - b.lo[1])) * b.nx + (c.x - b.lo[0]));
      }
      uint8_t* map = reinterpret_cast<uint8_t*>(sm.maps + b.map0);
#pragma unroll
      for (int u = 0; u < kBatch; ++u) {
        if (!in[u]) continue;
        if (idx[u] < (unsigned)b.cells) map[idx[u]] = 1;
        else st.fail = 1;  // cannot happen (monotone cell_index)
      }
    }
  }
  __syncthreads();
  for (int k = 0; k < num_set; ++k) {
    const EdgeBox& b = st.set[k];
    int local = 0;
    for (int i = threadIdx.x; i < (b.cells + 15) >> 4; i += kSearchBlock) {
      const uint4 v = sm.maps[b.map0 + i];  // every byte is 0 or 1
      local += __popc(v.x) + __popc(v.y) + __popc(v.z) + __popc(v.w);
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) local += __shfl_xor_sync(0xffffffffu, local, d);
    if ((threadIdx.x & 31) == 0 && local) atomicAdd(&st.set_count[k], local);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 0; k < num_set; ++k) {  // place_edge keeps num_known + num_set <= kKnownEdges
      st.known_edge[st.num_known] = st.set[k].div.resolution;
      st.known_count[st.num_known++] = st.set_count[k];
    }
  }
  __syncthreads();
}

// One sweep at `edge`: every cropped point proposes its row to its voxel's slot, where the lowest row stays. Lanes of a warp in
// the same voxel are merged with match.any first, and only the lowest lane (= lowest row) touches the table. Sets st.fail when a
// key does not pack or the table is full.
__device__ void result_sweep(SearchShared& sm, SearchState& st, const float* __restrict__ pts, int stride, int n, float max_range,
                             float edge) {
  for (int i = threadIdx.x; i < kResultSlots; i += kSearchBlock) {
    sm.result.keys[i] = kEmptyKey;
    sm.result.mins[i] = kEmpty;
  }
  if (threadIdx.x == 0) st.survivors = 0;
  __syncthreads();
  const CellDivider div = make_divider(edge);
  const int lane = threadIdx.x & 31;
  constexpr int kBatch = 4;
  for (int base = 0; base < n; base += kBatch * kSearchBlock) {  // the same trip count for every lane: match.any needs them all
    unsigned long long key[kBatch];
    bool have[kBatch];
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {  // the loads of a batch are in flight together
      const int i = base + u * kSearchBlock + threadIdx.x;
      key[u] = kEmptyKey - 1 - lane;  // distinct dummy for idle lanes (packed keys leave bit 63 clear)
      have[u] = false;
      if (i < n) {
        const float* p = pts + (size_t)i * stride;
        const Vec3f v{p[0], p[1], p[2]};
        if (norm3(v) <= max_range) {
          Int3 c;
          if (!cell_index_fast(v, div, &c)) c = cell_index(v, div);
          have[u] = pack_cell(c, &key[u]);
          if (!have[u]) st.fail = 1;
        }
      }
    }
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {
      const unsigned peers = __match_any_sync(0xffffffffu, key[u]);
      if (have[u] && (__ffs(peers) - 1) == lane) {
        uint32_t h = hash_key(key[u]) & (kResultSlots - 1);
        for (int probes = 0;;) {
          const unsigned long long prev = atomicCAS(&sm.result.keys[h], kEmptyKey, key[u]);
          if (prev == kEmptyKey || prev == key[u]) {
            atomicMin(&sm.result.mins[h], (uint32_t)(base + u * kSearchBlock + threadIdx.x));
            break;
          }
          h = (h + 1) & (kResultSlots - 1);
          if (++probes >= kResultSlots) {  // table full
            st.fail = 1;
            break;
          }
        }
      }
    }
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kSearchBlock, 2) adaptive_voxel_kernel(
    const float* __restrict__ points, int stride, int64_t cap, const int32_t* __restrict__ counts,
    const AdaptiveParams* __restrict__ filters, int num_filters, uint32_t* table, int64_t table_cap,
    uint32_t* scratch /* per pair: cap cropped rows + cap slots */, int32_t* keep, int32_t* keep_counts,
    float* passes, int32_t* num_passes, int32_t* cropped_counts) {
  __shared__ SearchShared sm;
  __shared__ SearchState st;
  const int pair = blockIdx.x;
  const int b = pair / num_filters;
  const AdaptiveParams opt = filters[pair % num_filters];
  const int n = counts[b];
  const float* pts = points + (size_t)b * cap * stride;
  int32_t* out = keep + (size_t)pair * cap;
  float* pass_log = passes + (size_t)pair * 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // FilterByMaxRange (voxel_filter.cc:28-38): norm = sqrt(x^2 + (y^2 + z^2)) <= max_range
  auto in_range = [&](int i) {
    const float* p = pts + (size_t)i * stride;
    return norm3(Vec3f{p[0], p[1], p[2]}) <= opt.max_range;
  };

  // first sweep: the number of cropped points and their bounding box, counted as block_compact counts
  {
    float lo3[3] = {3.4e38f, 3.4e38f, 3.4e38f}, hi3[3] = {-3.4e38f, -3.4e38f, -3.4e38f};
    const int count = warp_chunk_count(n, [&](int i) {
      const float* p = pts + (size_t)i * stride;
      const float v[3] = {p[0], p[1], p[2]};
      if (!(norm3(Vec3f{v[0], v[1], v[2]}) <= opt.max_range)) return false;
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        lo3[a] = fminf(lo3[a], v[a]);
        hi3[a] = fmaxf(hi3[a], v[a]);
      }
      return true;
    });
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) {
        lo3[a] = fminf(lo3[a], __shfl_xor_sync(0xffffffffu, lo3[a], d));
        hi3[a] = fmaxf(hi3[a], __shfl_xor_sync(0xffffffffu, hi3[a], d));
      }
    if (lane == 0)
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        st.box_warp[a][warp] = lo3[a];
        st.box_warp[3 + a][warp] = hi3[a];
      }
    if (threadIdx.x == 0) {
      st.fail = 0;
      st.num_known = 0;
    }
    int m;
    const int pos = warp_bases(count, &m);  // its barriers publish box_warp
    if (threadIdx.x < 6) {
      float v = st.box_warp[threadIdx.x][0];
      for (int w = 1; w < kSearchWarps; ++w) v = threadIdx.x < 3 ? fminf(v, st.box_warp[threadIdx.x][w]) : fmaxf(v, st.box_warp[threadIdx.x][w]);
      if (threadIdx.x < 3) st.lo[threadIdx.x] = v;
      else st.hi[threadIdx.x - 3] = v;
    }
    if (threadIdx.x == 0 && cropped_counts) cropped_counts[pair] = m;
    if ((float)m <= opt.min_num_points) {  // 'point_cloud' is already sparse enough
      warp_chunk_emit(n, pos, in_range, [&](int pos, int i) { out[pos] = i; });
      if (threadIdx.x == 0) {
        keep_counts[pair] = m;
        num_passes[pair] = 0;
      }
      return;
    }
  }
  int npass = 0;
  auto log_pass = [&](float edge) {
    if (threadIdx.x == 0 && npass < 32) pass_log[npass] = edge;
    ++npass;
  };

  // ---------------- the search on counted edges
  float result_edge = 0.f;
  for (;;) {
    __syncthreads();  // the box, the known edges and st.fail are visible
    if (st.fail) break;
    // Replay. The search bisects from its first edge with enough voxels on; before that it halves.
    npass = 0;
    bool bisecting = false, missed = false;
    float missing = 0.f;
    adaptive_search(
        opt,
        [&](float edge) -> int {
          const int k = find_edge(st.known_edge, st.num_known, edge);
          if (k < 0) {
            missed = true;
            missing = edge;
            return -1;
          }
          log_pass(edge);
          const int count = st.known_count[k];
          if ((float)count >= opt.min_num_points) bisecting = true;
          return count;
        },
        &result_edge);
    if (!missed) break;
    __syncthreads();  // every thread has read the known edges
    if (threadIdx.x == 0) {
      st.num_set = st.words = 0;
      if (!place_edge(st, missing)) {
        st.fail = 1;  // generic mode
      } else if (!bisecting) {  // as far as they fit: the next halving, and the bisection's first midpoint if that suffices
        const float low = missing / 2.f;
        if (place_edge(st, low)) place_edge(st, (low + missing) / 2.f);
      }
    }
    __syncthreads();
    if (st.fail) break;
    count_sweep(sm, st, pts, stride, n, opt.max_range);
  }
  if (!st.fail) result_sweep(sm, st, pts, stride, n, opt.max_range, result_edge);
  if (!st.fail) {
    // the survivors are the table's minima; each goes to its rank among them
    for (int s = threadIdx.x; s < kResultSlots; s += kSearchBlock) {
      const uint32_t r = sm.result.mins[s];
      if (r != kEmpty) sm.result.rows[atomicAdd(&st.survivors, 1)] = r;
    }
    __syncthreads();
    const int kept = st.survivors;
    for (int a = threadIdx.x; a < kept; a += kSearchBlock) {
      const uint32_t r = sm.result.rows[a];
      int rank = 0;
      for (int c = 0; c < kept; ++c) rank += sm.result.rows[c] < r;
      out[rank] = (int32_t)r;
    }
    if (threadIdx.x == 0) {
      keep_counts[pair] = kept;
      num_passes[pair] = npass;
    }
    return;
  }

  // ---------------- generic mode: index-only table in global memory, any number of points, any coordinates
  uint32_t* tab = table + (size_t)pair * table_cap;
  uint32_t* rows = scratch + (size_t)pair * 2 * cap;  // cropped cloud: id -> row
  uint32_t* slot = rows + cap;
  const int m = block_compact(n, in_range, [&](int pos, int i) { rows[pos] = (uint32_t)i; });
  npass = 0;
  uint32_t eff_cap = 64;
  while (eff_cap < 2u * (uint32_t)m) eff_cap <<= 1;
  if (eff_cap > (uint32_t)table_cap) eff_cap = (uint32_t)table_cap;
  const uint32_t mask = eff_cap - 1;
  float last_edge = -1.f;
  auto run_pass = [&](float edge) -> int {
    for (uint32_t i = threadIdx.x; i < eff_cap; i += kSearchBlock) tab[i] = kEmpty;
    __syncthreads();
    for (int j = threadIdx.x; j < m; j += kSearchBlock) {
      const Int3 c = row_cell(pts, stride, rows[j], edge);
      slot[j] = table_insert(tab, mask, pts, stride, edge, c, (uint32_t)j, [&](uint32_t id) { return rows[id]; });
    }
    __syncthreads();
    int local = 0;
    for (int j = threadIdx.x; j < m; j += kSearchBlock) local += __ldcg(tab + slot[j]) == (uint32_t)j;  // L2 read: atomics bypass L1
    last_edge = edge;
    return block_sum(local);
  };
  adaptive_search(
      opt,
      [&](float edge) {
        log_pass(edge);
        return run_pass(edge);
      },
      &result_edge);
  if (last_edge != result_edge) run_pass(result_edge);  // the table must hold the pass that produced `result`
  const int kept = block_compact(
      m, [&](int j) { return __ldcg(tab + slot[j]) == (uint32_t)j; }, [&](int pos, int j) { out[pos] = (int32_t)rows[j]; });
  if (threadIdx.x == 0) {
    keep_counts[pair] = kept;
    num_passes[pair] = npass;
  }
}

}  // namespace

// Voxel filter over `batch` clouds. Cloud b = rows [b * cap, b * cap + counts[b]) of `points` (stride floats per row).
// keep[b * cap ...] receives the surviving row indices (relative to the cloud) in input order, keep_counts[b] their number.
// table: batch * table_cap uint32 (table_cap a power of two >= 2 * max count); slot: batch * cap uint32.
int launch_voxel_filter(dl_context* ctx, const float* points, int stride, int64_t cap, const int32_t* counts, int batch,
                        float resolution, uint32_t* table, int64_t table_cap, uint32_t* slot, int32_t* keep,
                        int32_t* keep_counts, int32_t* block_counts) {
  if (batch <= 0 || cap <= 0) return DL_OK;
  DL_CUDA(ctx, cudaMemsetAsync(table, 0xFF, (size_t)batch * table_cap * sizeof(uint32_t), ctx->stream));
  const int tiles = (int)((cap + kBlock - 1) / kBlock);
  const dim3 grid(tiles, batch);
  voxel_insert_kernel<<<grid, kBlock, 0, ctx->stream>>>(points, stride, cap, counts, resolution, table, table_cap, slot);
  DL_LAUNCH_CHECK(ctx, "voxel_insert_kernel");
  voxel_count_kernel<<<grid, kBlock, 0, ctx->stream>>>(counts, cap, table, table_cap, slot, block_counts, tiles);
  DL_LAUNCH_CHECK(ctx, "voxel_count_kernel");
  voxel_scatter_kernel<<<grid, kBlock, 0, ctx->stream>>>(counts, cap, table, table_cap, slot, block_counts, tiles, keep,
                                                         keep_counts);
  DL_LAUNCH_CHECK(ctx, "voxel_scatter_kernel");
  return DL_OK;
}

int launch_voxel_indices(dl_context* ctx, const float* points, int stride, int64_t n, float resolution, int32_t* out) {
  if (n <= 0) return DL_OK;
  voxel_indices_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(points, stride, n, resolution, out);
  DL_LAUNCH_CHECK(ctx, "voxel_indices_kernel");
  return DL_OK;
}

int launch_adaptive_voxel_filter(dl_context* ctx, const float* points, int stride, int64_t cap, const int32_t* counts,
                                 int batch, const AdaptiveParams* filters_dev, int num_filters, uint32_t* table,
                                 int64_t table_cap, uint32_t* scratch, int32_t* keep, int32_t* keep_counts,
                                 float* passes, int32_t* num_passes, int32_t* cropped_counts) {
  if (batch <= 0 || num_filters <= 0) return DL_OK;
  adaptive_voxel_kernel<<<batch * num_filters, kSearchBlock, 0, ctx->stream>>>(
      points, stride, cap, counts, filters_dev, num_filters, table, table_cap, scratch, keep, keep_counts, passes,
      num_passes, cropped_counts);
  DL_LAUNCH_CHECK(ctx, "adaptive_voxel_kernel");
  return DL_OK;
}

}  // namespace dl

// ------------------------------------------------------------------------------------------------ voxel filters
namespace dl {
int64_t next_pow2(int64_t v) {
  int64_t p = 64;
  while (p < v) p <<= 1;
  return p;
}
}  // namespace dl

using namespace dl;

extern "C" {

int dl_voxel_indices(dl_context* ctx, const float* points, int64_t n, int stride, float resolution, int32_t* out) {
  if (!ctx || n < 0 || stride < 3 || !(resolution > 0.f) || (n > 0 && (!points || !out))) return DL_ERR_ARG;
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  float* d_pts;
  int32_t* d_out;
  DL_TRY(carve_scratch(ctx, [&](Arena& a) {
    d_pts = a.take<float>(n * stride);
    d_out = a.take<int32_t>(3 * n);
  }));
  DL_TRY(h2d(ctx, d_pts, points, n * stride));
  DL_TRY(launch_voxel_indices(ctx, d_pts, stride, n, resolution, d_out));
  DL_TRY(d2h(ctx, out, d_out, 3 * n));
  return sync(ctx);
}

int dl_voxel_filter(dl_context* ctx, const float* points, int64_t n, int stride, float resolution, int64_t* keep_out,
                    int64_t* n_keep) {
  if (!ctx || n < 0 || stride < 3 || !(resolution > 0.f) || !n_keep || (n > 0 && (!points || !keep_out)))
    return DL_ERR_ARG;
  *n_keep = 0;
  if (n == 0) return DL_OK;
  if (n > 0x7fffffff) return ctx->fail(DL_ERR_ARG, "more than 2^31-1 points");
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  const int64_t tcap = next_pow2(2 * n);
  const int tiles = (int)((n + 255) / 256);
  float* d_pts;
  uint32_t *d_table, *d_slot;
  int32_t *d_keep, *d_blocks, *d_counts;
  DL_TRY(carve_scratch(ctx, [&](Arena& a) {
    d_pts = a.take<float>(n * stride);
    d_table = a.take<uint32_t>(tcap);
    d_slot = a.take<uint32_t>(n);
    d_keep = a.take<int32_t>(n);
    d_blocks = a.take<int32_t>(tiles);
    d_counts = a.take<int32_t>(2);  // [0] = n, [1] = survivors
  }));
  const int32_t n32 = (int32_t)n;
  DL_TRY(h2d(ctx, d_pts, points, n * stride));
  DL_TRY(h2d(ctx, d_counts, &n32, 1));
  DL_TRY(launch_voxel_filter(ctx, d_pts, stride, n, d_counts, 1, resolution, d_table, tcap, d_slot, d_keep, d_counts + 1,
                             d_blocks));
  int32_t kept = 0;
  DL_TRY(d2h(ctx, &kept, d_counts + 1, 1));
  DL_TRY(sync(ctx));
  std::vector<int32_t> keep32(kept);
  DL_TRY(d2h(ctx, keep32.data(), d_keep, kept));
  DL_TRY(sync(ctx));
  for (int32_t i = 0; i < kept; ++i) keep_out[i] = keep32[i];
  *n_keep = kept;
  return DL_OK;
}

int dl_adaptive_voxel_filter(dl_context* ctx, const dl_adaptive_voxel_filter_options* options, const float* points,
                             int64_t n, int stride, int64_t* keep_out, int64_t* n_keep, float* passes_out,
                             int* n_passes) {
  if (!ctx || !options || n < 0 || stride < 3 || !n_keep || (n > 0 && (!points || !keep_out))) return DL_ERR_ARG;
  *n_keep = 0;
  if (n_passes) *n_passes = 0;
  if (n == 0) return DL_OK;
  if (n > 0x7fffffff) return ctx->fail(DL_ERR_ARG, "more than 2^31-1 points");
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  const int64_t tcap = next_pow2(2 * n);
  float *d_pts, *d_passes;
  uint32_t *d_table, *d_scratch;
  int32_t *d_keep, *d_counts;
  AdaptiveParams* d_params;
  DL_TRY(carve_scratch(ctx, [&](Arena& a) {
    d_pts = a.take<float>(n * stride);
    d_table = a.take<uint32_t>(tcap);
    d_scratch = a.take<uint32_t>(2 * n);
    d_keep = a.take<int32_t>(n);
    d_counts = a.take<int32_t>(3);  // n, survivors, passes
    d_params = a.take<AdaptiveParams>(1);
    d_passes = a.take<float>(32);
  }));
  const int32_t n32 = (int32_t)n;
  const AdaptiveParams params{options->max_length, options->min_num_points, options->max_range};
  DL_TRY(h2d(ctx, d_pts, points, n * stride));
  DL_TRY(h2d(ctx, d_counts, &n32, 1));
  DL_TRY(h2d(ctx, d_params, &params, 1));
  DL_TRY(launch_adaptive_voxel_filter(ctx, d_pts, stride, n, d_counts, 1, d_params, 1, d_table, tcap, d_scratch, d_keep,
                                      d_counts + 1, d_passes, d_counts + 2, nullptr));
  int32_t res[2] = {0, 0};
  float passes[32];
  DL_TRY(d2h(ctx, res, d_counts + 1, 2));
  DL_TRY(d2h(ctx, passes, d_passes, 32));
  DL_TRY(sync(ctx));
  std::vector<int32_t> keep32(res[0]);
  DL_TRY(d2h(ctx, keep32.data(), d_keep, res[0]));
  DL_TRY(sync(ctx));
  for (int32_t i = 0; i < res[0]; ++i) keep_out[i] = keep32[i];
  *n_keep = res[0];
  if (n_passes) *n_passes = res[1];
  if (passes_out) std::memcpy(passes_out, passes, sizeof(float) * std::min(res[1], 32));
  return DL_OK;
}

}  // extern "C"
