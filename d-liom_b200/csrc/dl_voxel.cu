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
// One CTA runs the whole data-dependent pass sequence of AdaptivelyVoxelFiltered for one (cloud, filter) pair,
// so the bisection needs no host round trip: every pass clears the table, re-inserts the range-cropped cloud and
// block-reduces the survivor count; the control flow below is the reference's, statement for statement.
constexpr int kAdaptiveBlock = 1024;  // 64 registers per thread: 8 cached points each, the rest in shared memory
constexpr int kAdaptiveWarps = kAdaptiveBlock / 32;

__device__ __forceinline__ int block_sum_1024(int v) {
  __shared__ int ws[32];
  __shared__ int result;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  __syncthreads();
  if (lane == 0) ws[warp] = v;
  __syncthreads();
  if (warp == 0) {
    int s = lane < kAdaptiveWarps ? ws[lane] : 0;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
    if (lane == 0) result = s;
  }
  __syncthreads();
  return result;
}

// Exclusive prefix of one value per warp over the 32 warps of the CTA (value must be warp-uniform); *total = the sum.
__device__ __forceinline__ int warp_bases_1024(int warp_value, int* total) {
  __shared__ int ws[kAdaptiveWarps], wb[kAdaptiveWarps + 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();  // protects ws / wb across successive calls
  if (lane == 0) ws[warp] = warp_value;
  __syncthreads();
  if (warp == 0) {
    const int v = ws[lane];
    int inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int o = __shfl_up_sync(0xffffffffu, inc, d);
      if (lane >= d) inc += o;
    }
    wb[lane] = inc - v;
    if (lane == 31) wb[kAdaptiveWarps] = inc;
  }
  __syncthreads();
  *total = wb[kAdaptiveWarps];
  return wb[warp];
}

// Order-preserving compaction of ids [0, n) with predicate flags computed by `pred` (pure: it is evaluated twice); returns the
// count. Every warp owns a contiguous chunk of ids: it counts its flags (no barrier between its rounds, so the loads behind
// `pred` pipeline), ONE block scan turns the 32 counts into bases, and a second sweep writes. (Round 1 walked the ids 1024 at a
// time with three barriers and a 32-step shared-memory sum per round: 19 % of the kernel's stall samples.)
template <typename Pred, typename Emit>
__device__ __forceinline__ int block_compact_1024(int n, Pred pred, Emit emit) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int chunk = ((n + kAdaptiveBlock - 1) / kAdaptiveBlock) * 32;  // ids per warp, a multiple of 32
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
  int total;
  int pos = warp_bases_1024(count, &total);
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

// ---- fast mode: the cropped cloud lives in registers (<= 16 points per thread), the hash table in shared memory
// (packed 63-bit voxel keys + min index), duplicates inside a warp are merged with match.any before touching the
// table. A pass is then ~16 ALU iterations + shared-memory atomics: no global traffic at all.
constexpr int kFastPoints = 8;                        // points per thread held in registers (x 1024 threads = 8 192)
constexpr int kFastSlots = 4096;                      // shared-memory table slots (12 B each = 48 KiB)
constexpr int kFastExtra = 14336;                     // further points cached in shared memory (12 B each = 168 KiB)
constexpr int kFastCapacity = kFastPoints * 1024 + kFastExtra;  // 22 528 points
static_assert(kFastCapacity / 1024 <= 32, "the compaction keeps one round count per lane");
constexpr unsigned long long kEmptyKey = 0xFFFFFFFFFFFFFFFFull;

struct FastTable {
  unsigned long long keys[kFastSlots];
  uint32_t mins[kFastSlots];
  float extra[kFastExtra * 3];  // points with id >= kFastPoints * kAdaptiveBlock
};

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

// One point of a pass (all 32 lanes of the warp call this together): lanes that fall into the same voxel are
// merged with match.any and only the lowest lane (= lowest id) touches the table. Returns 1 for a new voxel.
__device__ __forceinline__ int fast_insert(FastTable& tab, bool have, float x, float y, float z, int j,
                                           const CellDivider& edge, int* fail_flag) {
  const int lane = threadIdx.x & 31;
  unsigned long long key = kEmptyKey - 1 - lane;  // distinct dummy for idle lanes
  bool ok = true;
  if (have) ok = pack_cell(cell_index(Vec3f{x, y, z}, edge), &key);
  if (!ok) *fail_flag = 1;
  const unsigned peers = __match_any_sync(0xffffffffu, key);
  int claimed = 0;
  if (have && ok && (__ffs(peers) - 1) == lane) {
    uint32_t h = hash_key(key) & (kFastSlots - 1);
    int probes = 0;
    for (;;) {
      const unsigned long long prev = atomicCAS(&tab.keys[h], kEmptyKey, key);
      if (prev == kEmptyKey) claimed = 1;
      if (prev == kEmptyKey || prev == key) {
        atomicMin(&tab.mins[h], (uint32_t)j);
        break;
      }
      h = (h + 1) & (kFastSlots - 1);
      if (++probes >= kFastSlots) {  // table full
        *fail_flag = 1;
        break;
      }
    }
  }
  return claimed;
}

// Returns the number of distinct voxels, or -1 if the table overflowed / a key could not be packed.
__device__ __forceinline__ int fast_pass(FastTable& tab, const float (&px)[kFastPoints], const float (&py)[kFastPoints],
                                         const float (&pz)[kFastPoints], int m, float edge_length, int* fail_flag) {
  const CellDivider edge = make_divider(edge_length);
  for (int i = threadIdx.x; i < kFastSlots; i += kAdaptiveBlock) {
    tab.keys[i] = kEmptyKey;
    tab.mins[i] = 0xFFFFFFFFu;
  }
  __syncthreads();
  int claims = 0;
#pragma unroll
  for (int k = 0; k < kFastPoints; ++k) {
    if (k * kAdaptiveBlock >= m) break;  // uniform
    const int j = k * kAdaptiveBlock + threadIdx.x;
    claims += fast_insert(tab, j < m, px[k], py[k], pz[k], j, edge, fail_flag);
  }
  for (int base = kFastPoints * kAdaptiveBlock; base < m; base += kAdaptiveBlock) {
    const int j = base + threadIdx.x;
    const float* e = tab.extra + (size_t)(j - kFastPoints * kAdaptiveBlock) * 3;
    const bool have = j < m;
    claims += fast_insert(tab, have, have ? e[0] : 0.f, have ? e[1] : 0.f, have ? e[2] : 0.f, j, edge, fail_flag);
  }
  const int total = block_sum_1024(claims);  // contains the barriers that publish fail_flag
  return *fail_flag ? -1 : total;
}

// ---- count-only passes of the search on a BYTE MAP instead of the hash table.
// The search only needs the NUMBER of voxels a pass produces (voxel_filter.cc:47,57,63); the survivors are needed for the result
// pass alone. cell_index is monotone per axis, so every cell of the pass lies in the box [cell(min corner), cell(max corner)] of
// the cropped cloud; when that box has at most kByteCells cells each point simply stores a 1 into its cell's byte (plain shared-
// memory stores: all writers write the same value, no atomics, no probing, no warp matching) and the count is the number of
// non-zero bytes. The map aliases the hash table (which is rebuilt by the result pass anyway). ~3x fewer instructions per point
// than a hash pass and none of its shared-memory atomics. Returns -2 when the box is too large (the caller runs a hash pass).
constexpr int kByteCells = (int)((sizeof(unsigned long long) + sizeof(uint32_t)) * kFastSlots);  // 48 KiB
struct CloudBox {
  float lo[3], hi[3];
};
__device__ __forceinline__ int byte_map_pass(FastTable& tab, const CloudBox& box, const float (&px)[kFastPoints],
                                             const float (&py)[kFastPoints], const float (&pz)[kFastPoints], int m, float edge_length,
                                             int* fail_flag) {
  const CellDivider edge = make_divider(edge_length);
  const Int3 lo = cell_index(Vec3f{box.lo[0], box.lo[1], box.lo[2]}, edge), hi = cell_index(Vec3f{box.hi[0], box.hi[1], box.hi[2]}, edge);
  const long long nx = (long long)hi.x - lo.x + 1, ny = (long long)hi.y - lo.y + 1, nz = (long long)hi.z - lo.z + 1;
  if (nx <= 0 || ny <= 0 || nz <= 0 || nx > kByteCells || ny > kByteCells || nz > kByteCells || nx * ny * nz > kByteCells) return -2;
  const int inx = (int)nx, iny = (int)ny, cells = (int)(nx * ny * nz);
  uint8_t* map = reinterpret_cast<uint8_t*>(&tab);
  uint4* map4 = reinterpret_cast<uint4*>(&tab);
  const int words16 = (cells + 15) >> 4;
  for (int i = threadIdx.x; i < words16; i += kAdaptiveBlock) map4[i] = make_uint4(0u, 0u, 0u, 0u);
  __syncthreads();
  auto mark = [&](float x, float y, float z) {
    const Int3 c = cell_index(Vec3f{x, y, z}, edge);
    const unsigned idx = (unsigned)(((c.z - lo.z) * iny + (c.y - lo.y)) * inx + (c.x - lo.x));
    if (idx < (unsigned)cells) map[idx] = 1;
    else *fail_flag = 1;  // cannot happen (monotone cell_index); checked by the closing test of *fail_flag
  };
#pragma unroll
  for (int k = 0; k < kFastPoints; ++k) {
    if (k * kAdaptiveBlock >= m) break;  // uniform
    if (k * kAdaptiveBlock + (int)threadIdx.x < m) mark(px[k], py[k], pz[k]);
  }
  for (int j = kFastPoints * kAdaptiveBlock + threadIdx.x; j < m; j += kAdaptiveBlock) {
    const float* e = tab.extra + (size_t)(j - kFastPoints * kAdaptiveBlock) * 3;
    mark(e[0], e[1], e[2]);
  }
  __syncthreads();
  int local = 0;
  for (int i = threadIdx.x; i < words16; i += kAdaptiveBlock) {
    const uint4 v = map4[i];  // every byte is 0 or 1
    local += __popc(v.x) + __popc(v.y) + __popc(v.z) + __popc(v.w);
  }
  const int total = block_sum_1024(local);
  return *fail_flag ? -1 : total;
}

__device__ __forceinline__ bool fast_survives(const FastTable& tab, float x, float y, float z, float edge, int j) {
  unsigned long long key;
  pack_cell(cell_index(Vec3f{x, y, z}, make_divider(edge)), &key);
  uint32_t h = hash_key(key) & (kFastSlots - 1);
  while (tab.keys[h] != key) h = (h + 1) & (kFastSlots - 1);
  return tab.mins[h] == (uint32_t)j;
}

__global__ void __launch_bounds__(kAdaptiveBlock) adaptive_voxel_kernel(
    const float* __restrict__ points, int stride, int64_t cap, const int32_t* __restrict__ counts,
    const AdaptiveParams* __restrict__ filters, int num_filters, uint32_t* table, int64_t table_cap,
    uint32_t* scratch /* per pair: cap cropped rows + cap slots */, int32_t* keep, int32_t* keep_counts,
    float* passes, int32_t* num_passes, int32_t* cropped_counts, const int32_t* __restrict__ need) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  FastTable& fast = *reinterpret_cast<FastTable*>(smem_raw);
  __shared__ int fail_flag;
  const int pair = blockIdx.x;
  if (need && need[4 * pair] == 0) return;  // EdgeMeta::need of this pair: the grid-wide first pass already produced its result
  const int b = pair / num_filters;
  const AdaptiveParams opt = filters[pair % num_filters];
  const int n = counts[b];
  const float* pts = points + (size_t)b * cap * stride;
  uint32_t* tab = table + (size_t)pair * table_cap;
  uint32_t* rows = scratch + (size_t)pair * 2 * cap;  // cropped cloud: id -> row
  uint32_t* slot = rows + cap;
  int32_t* out = keep + (size_t)pair * cap;
  float* pass_log = passes + (size_t)pair * 32;
  int npass = 0;
  if (threadIdx.x == 0) fail_flag = 0;

  // FilterByMaxRange (voxel_filter.cc:28-38): norm = sqrt(x^2 + (y^2 + z^2)) <= max_range
  const int m = block_compact_1024(
      n,
      [&](int i) {
        const float* p = pts + (size_t)i * stride;
        return norm3(Vec3f{p[0], p[1], p[2]}) <= opt.max_range;
      },
      [&](int pos, int i) { rows[pos] = (uint32_t)i; });
  if (threadIdx.x == 0 && cropped_counts) cropped_counts[pair] = m;

  if ((float)m <= opt.min_num_points) {  // 'point_cloud' is already sparse enough
    for (int j = threadIdx.x; j < m; j += kAdaptiveBlock) out[j] = (int32_t)rows[j];
    if (threadIdx.x == 0) {
      keep_counts[pair] = m;
      num_passes[pair] = 0;
    }
    return;
  }
  auto log_pass = [&](float edge) {
    if (threadIdx.x == 0 && npass < 32) pass_log[npass] = edge;
    ++npass;
  };

  // ---------------- fast mode
  if (m <= kFastCapacity) {
    float px[kFastPoints], py[kFastPoints], pz[kFastPoints];
#pragma unroll
    for (int k = 0; k < kFastPoints; ++k) {
      const int j = k * kAdaptiveBlock + threadIdx.x;
      px[k] = py[k] = pz[k] = 0.f;
      if (j < m) {
        const float* p = pts + (size_t)rows[j] * stride;
        px[k] = p[0]; py[k] = p[1]; pz[k] = p[2];
      }
    }
    for (int j = kFastPoints * kAdaptiveBlock + threadIdx.x; j < m; j += kAdaptiveBlock) {
      const float* p = pts + (size_t)rows[j] * stride;
      float* e = fast.extra + (size_t)(j - kFastPoints * kAdaptiveBlock) * 3;
      e[0] = p[0]; e[1] = p[1]; e[2] = p[2];
    }
    // bounding box of the cropped cloud, for the byte-map passes
    __shared__ CloudBox box;
    __shared__ float box_warp[6][kAdaptiveWarps];
    {
      float lo3[3] = {3.4e38f, 3.4e38f, 3.4e38f}, hi3[3] = {-3.4e38f, -3.4e38f, -3.4e38f};
      auto grow = [&](float x, float y, float z) {
        lo3[0] = fminf(lo3[0], x); lo3[1] = fminf(lo3[1], y); lo3[2] = fminf(lo3[2], z);
        hi3[0] = fmaxf(hi3[0], x); hi3[1] = fmaxf(hi3[1], y); hi3[2] = fmaxf(hi3[2], z);
      };
#pragma unroll
      for (int k = 0; k < kFastPoints; ++k)
        if (k * kAdaptiveBlock + (int)threadIdx.x < m) grow(px[k], py[k], pz[k]);
      for (int j = kFastPoints * kAdaptiveBlock + threadIdx.x; j < m; j += kAdaptiveBlock) {
        const float* p = pts + (size_t)rows[j] * stride;
        grow(p[0], p[1], p[2]);
      }
#pragma unroll
      for (int a3 = 0; a3 < 3; ++a3)
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
          lo3[a3] = fminf(lo3[a3], __shfl_xor_sync(0xffffffffu, lo3[a3], d));
          hi3[a3] = fmaxf(hi3[a3], __shfl_xor_sync(0xffffffffu, hi3[a3], d));
        }
      const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
      if (lane == 0)
#pragma unroll
        for (int a3 = 0; a3 < 3; ++a3) {
          box_warp[a3][warp] = lo3[a3];
          box_warp[3 + a3][warp] = hi3[a3];
        }
      __syncthreads();
      if (threadIdx.x < 6) {
        float v = box_warp[threadIdx.x][0];
        for (int w = 1; w < kAdaptiveWarps; ++w) v = threadIdx.x < 3 ? fminf(v, box_warp[threadIdx.x][w]) : fmaxf(v, box_warp[threadIdx.x][w]);
        if (threadIdx.x < 3) box.lo[threadIdx.x] = v; else box.hi[threadIdx.x - 3] = v;
      }
    }
    __syncthreads();
    float last_edge = -1.f, result_edge = 0.f;  // last_edge: the edge whose survivors the hash table holds
    const bool ok = adaptive_search(
        opt,
        [&](float edge) {
          log_pass(edge);
          const int count = byte_map_pass(fast, box, px, py, pz, m, edge, &fail_flag);
          if (count != -2) {
            last_edge = -1.f;  // the byte map overwrote the table
            return count;
          }
          last_edge = edge;
          return fast_pass(fast, px, py, pz, m, edge, &fail_flag);
        },
        &result_edge);
    bool done = ok;
    if (ok && last_edge != result_edge) done = fast_pass(fast, px, py, pz, m, result_edge, &fail_flag) >= 0;
    if (done) {
      // Ordered compaction of the survivors. Id j = k * 1024 + t belongs to round k, warp t / 32: the output order is (round, warp,
      // lane). Every warp counts its survivors per round (lane k keeps round k's count: at most kFastCapacity / 1024 = 22 rounds), ONE block
      // scan over the (round, warp) sequence gives every warp its base per round, then the warps write.
      __shared__ int seq[32 * kAdaptiveWarps];
      const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
      const int rounds = (m + kAdaptiveBlock - 1) / kAdaptiveBlock;
      uint32_t flags = 0;
      int my_round_count = 0;
      auto test_round = [&](int k, float x, float y, float z) {
        const int j = k * kAdaptiveBlock + threadIdx.x;
        const bool f = j < m && fast_survives(fast, x, y, z, result_edge, j);
        const unsigned ballot = __ballot_sync(0xffffffffu, f);
        if (f) flags |= 1u << k;
        if (lane == k) my_round_count = __popc(ballot);
      };
#pragma unroll
      for (int k = 0; k < kFastPoints; ++k) {
        if (k >= rounds) break;
        test_round(k, px[k], py[k], pz[k]);
      }
      for (int k = kFastPoints; k < rounds; ++k) {
        const float* e = fast.extra + (size_t)(min(k * kAdaptiveBlock + (int)threadIdx.x, m - 1) - kFastPoints * kAdaptiveBlock) * 3;
        test_round(k, e[0], e[1], e[2]);
      }
      if (lane < rounds) seq[lane * kAdaptiveWarps + warp] = my_round_count;
      __syncthreads();
      // exclusive scan of seq[0 .. rounds * 32): one entry per thread
      const int entries = rounds * kAdaptiveWarps;
      const int v = (int)threadIdx.x < entries ? seq[threadIdx.x] : 0;
      int inc = v;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int o = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc += o;
      }
      int kept;
      const int wbase = warp_bases_1024(__shfl_sync(0xffffffffu, inc, 31), &kept);
      if ((int)threadIdx.x < entries) seq[threadIdx.x] = wbase + inc - v;
      __syncthreads();
      for (int k = 0; k < rounds; ++k) {
        const bool f = (flags >> k) & 1u;
        const unsigned ballot = __ballot_sync(0xffffffffu, f);
        if (f) out[seq[k * kAdaptiveWarps + warp] + __popc(ballot & ((1u << lane) - 1))] = (int32_t)rows[k * kAdaptiveBlock + threadIdx.x];
      }
      if (threadIdx.x == 0) {
        keep_counts[pair] = kept;
        num_passes[pair] = npass;
      }
      return;
    }
    // a pass overflowed the shared table or met an unpackable key: redo everything in generic mode
    npass = 0;
    __syncthreads();
  }

  // ---------------- generic mode: index-only table in global memory, any number of points, any coordinates
  uint32_t eff_cap = 64;
  while (eff_cap < 2u * (uint32_t)m) eff_cap <<= 1;
  if (eff_cap > (uint32_t)table_cap) eff_cap = (uint32_t)table_cap;
  const uint32_t mask = eff_cap - 1;
  float last_edge = -1.f;
  auto run_pass = [&](float edge) -> int {
    for (uint32_t i = threadIdx.x; i < eff_cap; i += kAdaptiveBlock) tab[i] = kEmpty;
    __syncthreads();
    for (int j = threadIdx.x; j < m; j += kAdaptiveBlock) {
      const Int3 c = row_cell(pts, stride, rows[j], edge);
      slot[j] = table_insert(tab, mask, pts, stride, edge, c, (uint32_t)j, [&](uint32_t id) { return rows[id]; });
    }
    __syncthreads();
    int local = 0;
    for (int j = threadIdx.x; j < m; j += kAdaptiveBlock) local += __ldcg(tab + slot[j]) == (uint32_t)j;  // L2 read: atomics bypass L1
    last_edge = edge;
    return block_sum_1024(local);
  };
  float result_edge = 0.f;
  adaptive_search(
      opt,
      [&](float edge) {
        log_pass(edge);
        return run_pass(edge);
      },
      &result_edge);
  if (last_edge != result_edge) run_pass(result_edge);  // the table must hold the pass that produced `result`
  const int kept = block_compact_1024(
      m, [&](int j) { return __ldcg(tab + slot[j]) == (uint32_t)j; }, [&](int pos, int j) { out[pos] = (int32_t)rows[j]; });
  if (threadIdx.x == 0) {
    keep_counts[pair] = kept;
    num_passes[pair] = npass;
  }
}

// ------------------------------------------------------------------------------------------- adaptive filter, common case
// In the front end the FIRST pass of the search (edge = max_length) almost always yields >= min_num_points voxels: the result
// is then simply the voxel filter at max_length of the range-cropped cloud. That case needs no bisection and no single-CTA
// sequencing, so it runs grid-wide for every (cloud, filter) pair of the batch: crop + insert (packed 63-bit key, min index),
// mark the winners, count per tile, prefix per pair, ordered scatter. adaptive_voxel_kernel (one CTA per pair, whole
// search) then runs only for the pairs whose first pass fell short, whose table overflowed or whose keys do not pack.
// Round 1 ran every pair through the single CTA: 190 us per 74 scans, mostly barrier latency of its 1024-id compaction rounds.
constexpr int kEdgeSlots = 8192;  // slots of the first-pass table per pair (keys 8 B + min index 4 B)
struct EdgeMeta {
  int32_t cropped, voxels, fail, need;
};
__device__ __forceinline__ unsigned long long* edge_keys(uint32_t* table, int64_t table_cap, int pair) {
  return reinterpret_cast<unsigned long long*>(table + (size_t)pair * table_cap);
}
__device__ __forceinline__ uint32_t* edge_mins(uint32_t* table, int64_t table_cap, int pair) {
  return table + (size_t)pair * table_cap + 2 * kEdgeSlots;
}

__global__ void __launch_bounds__(kBlock) adaptive_first_insert_kernel(const float* __restrict__ points, int stride, int64_t cap,
                                                                       const int32_t* __restrict__ counts,
                                                                       const AdaptiveParams* __restrict__ filters, int num_filters,
                                                                       uint32_t* table, int64_t table_cap, uint8_t* win, EdgeMeta* meta) {
  const int pair = blockIdx.y, b = pair / num_filters;
  const AdaptiveParams opt = filters[pair % num_filters];
  const int n = counts[b];
  const float* pts = points + (size_t)b * cap * stride;
  unsigned long long* keys = edge_keys(table, table_cap, pair);
  uint32_t* mins = edge_mins(table, table_cap, pair);
  uint8_t* w = win + (size_t)pair * cap;
  const CellDivider edge = make_divider(opt.max_length);
  int cropped = 0;
  for (int base = blockIdx.x * kBlock; base < n; base += gridDim.x * kBlock) {
    const int i = base + threadIdx.x;
    bool in = false;
    Vec3f p{0.f, 0.f, 0.f};
    if (i < n) {
      const float* q = pts + (size_t)i * stride;
      p = {q[0], q[1], q[2]};
      in = norm3(p) <= opt.max_range;  // FilterByMaxRange (voxel_filter.cc:28-38)
      w[i] = in ? 2 : 0;
    }
    cropped += in;
    if (in) {
      unsigned long long key;
      if (!pack_cell(cell_index(p, edge), &key)) {
        meta[pair].fail = 1;
      } else {
        uint32_t h = hash_key(key) & (kEdgeSlots - 1);
        int probes = 0;
        for (;;) {
          const unsigned long long prev = atomicCAS(keys + h, kEmptyKey, key);
          if (prev == kEmptyKey || prev == key) {
            atomicMin(mins + h, (uint32_t)i);
            break;
          }
          h = (h + 1) & (kEdgeSlots - 1);
          if (++probes >= kEdgeSlots) {
            meta[pair].fail = 1;
            break;
          }
        }
      }
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) cropped += __shfl_xor_sync(0xffffffffu, cropped, d);
  if ((threadIdx.x & 31) == 0 && cropped) atomicAdd(&meta[pair].cropped, cropped);
}

__global__ void __launch_bounds__(kBlock) adaptive_first_mark_kernel(uint32_t* table, int64_t table_cap, int64_t cap, uint8_t* win,
                                                                     EdgeMeta* meta) {
  const int pair = blockIdx.y;
  const uint32_t* mins = edge_mins(table, table_cap, pair);
  const int h = blockIdx.x * kBlock + threadIdx.x;
  const uint32_t m = __ldcg(mins + h);
  const bool used = m != kEmpty;
  if (used) win[(size_t)pair * cap + m] = 3;  // cropped + owner of its voxel; one writer per point
  const int c = __syncthreads_count(used);
  if (threadIdx.x == 0 && c) atomicAdd(&meta[pair].voxels, c);
}

// 1 = keep. Decided per pair from the finished counts: sparse enough already -> every cropped point; first pass sufficient ->
// the voxel owners; otherwise nothing here (the single-CTA search takes over).
__device__ __forceinline__ int edge_mode(const EdgeMeta& m, const AdaptiveParams& opt) {
  if (m.fail) return 0;
  if ((float)m.cropped <= opt.min_num_points) return 2;
  if ((float)m.voxels >= opt.min_num_points) return 1;
  return 0;
}

__global__ void __launch_bounds__(kBlock) adaptive_first_count_kernel(const int32_t* __restrict__ counts,
                                                                      const AdaptiveParams* __restrict__ filters, int num_filters,
                                                                      int64_t cap, const uint8_t* __restrict__ win,
                                                                      const EdgeMeta* __restrict__ meta, int32_t* tile_counts, int tiles) {
  const int pair = blockIdx.y, b = pair / num_filters;
  const int n = counts[b];
  if ((int)blockIdx.x * kBlock >= n) return;
  const int mode = edge_mode(meta[pair], filters[pair % num_filters]);
  const int i = blockIdx.x * kBlock + threadIdx.x;
  const int wv = i < n ? win[(size_t)pair * cap + i] : 0;
  const int c = __syncthreads_count(mode && (wv & mode) != 0);
  if (threadIdx.x == 0) tile_counts[(size_t)pair * tiles + blockIdx.x] = c;
}

// One CTA per pair: exclusive prefix of the tile counts (in place) and the pair's bookkeeping.
__global__ void __launch_bounds__(kBlock) adaptive_first_prefix_kernel(const int32_t* __restrict__ counts,
                                                                       const AdaptiveParams* __restrict__ filters, int num_filters,
                                                                       EdgeMeta* meta, int32_t* tile_counts, int tiles,
                                                                       int32_t* keep_counts, float* passes, int32_t* num_passes,
                                                                       int32_t* cropped_counts, int32_t* stats) {
  const int pair = blockIdx.x, b = pair / num_filters;
  const AdaptiveParams opt = filters[pair % num_filters];
  const int n = counts[b];
  const int mode = edge_mode(meta[pair], opt);
  if (threadIdx.x == 0 && stats) {
    atomicAdd(stats + 1, 1);
    if (mode == 0) atomicAdd(stats, 1);
  }
  if (mode == 0) {  // falls through to adaptive_voxel_kernel, which writes all of this pair's outputs
    if (threadIdx.x == 0) meta[pair].need = 1;
    return;
  }
  const int my_tiles = (n + kBlock - 1) / kBlock;
  int32_t* tc = tile_counts + (size_t)pair * tiles;
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < my_tiles; base += kBlock) {
    const int t = base + threadIdx.x;
    const int v = t < my_tiles ? tc[t] : 0;
    int total;
    const int ex = block_exclusive_scan(v, &total);
    if (t < my_tiles) tc[t] = carry + ex;
    __syncthreads();
    if (threadIdx.x == 0) carry += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    meta[pair].need = 0;
    keep_counts[pair] = carry;
    num_passes[pair] = mode == 2 ? 0 : 1;
    if (mode == 1) passes[(size_t)pair * 32] = opt.max_length;
    if (cropped_counts) cropped_counts[pair] = meta[pair].cropped;
  }
}

__global__ void __launch_bounds__(kBlock) adaptive_first_scatter_kernel(const int32_t* __restrict__ counts,
                                                                        const AdaptiveParams* __restrict__ filters, int num_filters,
                                                                        int64_t cap, const uint8_t* __restrict__ win,
                                                                        const EdgeMeta* __restrict__ meta,
                                                                        const int32_t* __restrict__ tile_counts, int tiles, int32_t* keep) {
  const int pair = blockIdx.y, b = pair / num_filters;
  const int n = counts[b];
  if ((int)blockIdx.x * kBlock >= n || meta[pair].need) return;
  const int mode = edge_mode(meta[pair], filters[pair % num_filters]);
  const int i = blockIdx.x * kBlock + threadIdx.x;
  const int wv = i < n ? win[(size_t)pair * cap + i] : 0;
  const int flag = (wv & mode) != 0;
  int total;
  const int off = block_exclusive_scan(flag, &total);
  if (flag) keep[(size_t)pair * cap + tile_counts[(size_t)pair * tiles + blockIdx.x] + off] = i;
}

}  // namespace

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

size_t adaptive_first_pass_bytes(int pairs, int64_t cap) {
  const size_t tiles = (size_t)((cap + kBlock - 1) / kBlock);
  return (((size_t)pairs * cap + 255) & ~size_t(255)) + (size_t)pairs * tiles * 4 + (size_t)pairs * sizeof(EdgeMeta) + 256;
}

int launch_adaptive_voxel_filter(dl_context* ctx, const float* points, int stride, int64_t cap, const int32_t* counts,
                                 int batch, const AdaptiveParams* filters_dev, int num_filters, uint32_t* table,
                                 int64_t table_cap, uint32_t* scratch, int32_t* keep, int32_t* keep_counts,
                                 float* passes, int32_t* num_passes, int32_t* cropped_counts, void* first_pass_scratch) {
  if (batch <= 0 || num_filters <= 0) return DL_OK;
  const int pairs = batch * num_filters;
  const int tiles = (int)((cap + kBlock - 1) / kBlock);
  // The grid-wide first pass keeps its keys + min indices in the head of each pair's table region (the single-CTA search only
  // touches that region afterwards, for its own pair) and its winner bytes, tile counts and bookkeeping in first_pass_scratch
  // (adaptive_first_pass_bytes). Tables too small for it (tiny clouds) go straight to the single-CTA search.
  bool first_pass = first_pass_scratch && (size_t)table_cap * 4 >= (size_t)kEdgeSlots * 12;
  // Self-tuning: the grid-wide pass only pays when the first edge usually suffices. The share of pairs that fell through to the
  // single-CTA search in the last probed launch is read from a pinned counter (no synchronisation: a stale or half-updated
  // value only changes which of two exact paths runs); when most pairs fall through, skip the pass and re-probe every 16th call.
  if (first_pass && !ctx->h_adaptive_stats) {
    if (cudaMallocHost((void**)&ctx->h_adaptive_stats, 2 * sizeof(int32_t)) != cudaSuccess ||
        cudaMalloc((void**)&ctx->d_adaptive_stats, 2 * sizeof(int32_t)) != cudaSuccess) {
      cudaGetLastError();
      ctx->h_adaptive_stats = nullptr;
    } else {
      ctx->h_adaptive_stats[0] = ctx->h_adaptive_stats[1] = 0;
    }
  }
  int32_t* stats = nullptr;
  if (first_pass && ctx->h_adaptive_stats) {
    const int32_t fell = ctx->h_adaptive_stats[0], probed = ctx->h_adaptive_stats[1];
    const bool probe = (ctx->adaptive_calls++ % 16) == 0;
    if (!probe && probed > 0 && 2 * fell > probed) first_pass = false;
    if (first_pass && probe) stats = ctx->d_adaptive_stats;
  }
  const int32_t* need = nullptr;
  if (first_pass) {
    uint8_t* win = reinterpret_cast<uint8_t*>(first_pass_scratch);                        // pairs * cap bytes
    int32_t* tile_counts = reinterpret_cast<int32_t*>(win + (((size_t)pairs * cap + 255) & ~size_t(255)));  // pairs * tiles
    EdgeMeta* meta = reinterpret_cast<EdgeMeta*>(tile_counts + (size_t)pairs * tiles);
    DL_CUDA(ctx, cudaMemset2DAsync(table, (size_t)table_cap * 4, 0xFF, (size_t)kEdgeSlots * 12, (size_t)pairs, ctx->stream));
    DL_CUDA(ctx, cudaMemsetAsync(meta, 0, sizeof(EdgeMeta) * pairs, ctx->stream));
    if (stats) DL_CUDA(ctx, cudaMemsetAsync(stats, 0, 2 * sizeof(int32_t), ctx->stream));
    const int insert_tiles = std::min(tiles, 96);
    adaptive_first_insert_kernel<<<dim3(insert_tiles, pairs), kBlock, 0, ctx->stream>>>(points, stride, cap, counts, filters_dev,
                                                                                         num_filters, table, table_cap, win, meta);
    DL_LAUNCH_CHECK(ctx, "adaptive_first_insert_kernel");
    adaptive_first_mark_kernel<<<dim3(kEdgeSlots / kBlock, pairs), kBlock, 0, ctx->stream>>>(table, table_cap, cap, win, meta);
    DL_LAUNCH_CHECK(ctx, "adaptive_first_mark_kernel");
    adaptive_first_count_kernel<<<dim3(tiles, pairs), kBlock, 0, ctx->stream>>>(counts, filters_dev, num_filters, cap, win, meta,
                                                                                 tile_counts, tiles);
    DL_LAUNCH_CHECK(ctx, "adaptive_first_count_kernel");
    adaptive_first_prefix_kernel<<<pairs, kBlock, 0, ctx->stream>>>(counts, filters_dev, num_filters, meta, tile_counts, tiles,
                                                                    keep_counts, passes, num_passes, cropped_counts, stats);
    DL_LAUNCH_CHECK(ctx, "adaptive_first_prefix_kernel");
    if (stats)
      DL_CUDA(ctx, cudaMemcpyAsync(ctx->h_adaptive_stats, stats, 2 * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
    adaptive_first_scatter_kernel<<<dim3(tiles, pairs), kBlock, 0, ctx->stream>>>(counts, filters_dev, num_filters, cap, win, meta,
                                                                                   tile_counts, tiles, keep);
    DL_LAUNCH_CHECK(ctx, "adaptive_first_scatter_kernel");
    need = &meta->need;  // stride sizeof(EdgeMeta): see the kernel's indexing below
  }
  DL_CUDA(ctx, cudaFuncSetAttribute(adaptive_voxel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(FastTable)));
  adaptive_voxel_kernel<<<pairs, kAdaptiveBlock, sizeof(FastTable), ctx->stream>>>(
      points, stride, cap, counts, filters_dev, num_filters, table, table_cap, scratch, keep, keep_counts, passes,
      num_passes, cropped_counts, need);
  DL_LAUNCH_CHECK(ctx, "adaptive_voxel_kernel");
  return DL_OK;
}

}  // namespace dl
