// Fused scan front half of the batched front end and of dl_ingest_scan: 5 launches per sub-batch (6 with per-run deskew poses),
// then the small glue kernels of the batched front end (cloud gathers, pose algebra, result records).
//
//   A  fe_first_filter_tile     first voxel filter (LTB:393-395), per tile of 2048 rows: the tile's lowest row per voxel in
//                               shared memory; the tile stores its words of the scan's survivor bitmap and writes its winners
//                               to the scan's hash partitions.
//   A2 fe_merge_partitions      per (scan, partition): the lowest row per voxel over all tiles, in shared memory; clears the
//                               bits of the tile winners that lost.
//   B0 fe_run_poses             12-byte rows with the point times as runs: the deskew pose (fp64 slerp + composition, LTB:430-445) once
//                               per RUN instead of once per survivor; kernel B then loads the finished Rigid3f.
//   B  fe_ingest_tile           per tile, the first-filter survivors in index order (from the bitmap): deskew + transform +
//                               range gate (LTB:426-472) and the SECOND voxel filter (LTB:479-484) keyed on the local-frame
//                               voxel, again per tile in shared memory first — no compaction in between: ids stay the original
//                               input indices, which preserves "first point in input order wins" for free. Its tile winners
//                               end as two per-scan bitmaps (returns, misses; 4 KiB per 32 k points) and go to partitions as
//                               kernel A's do.
//   B2 fe_merge_partitions      as A2, for the second filter's words.
//   C  fe_emit_tracking        ordered compaction straight from the bitmaps (popcount prefix; no per-point class map, no
//                               tile counts), fused with the scan's current pose (hits_poses.back(), LTB:476) and the frame
//                               change back to tracking (TransformRangeData with current_pose^-1, LTB:485-487); output rows
//                               are written coalesced.
//
// The second filter's entries are ONE 64-bit word: [miss | voxel key relative to the scan's pose | point index]. The key sits
// above the index, so for equal keys atomicMin keeps the lowest index ("first point in input order", voxel_filter.cc:81-131)
// and a claimed word's key never changes: a collision compares keys inside the word. The key holds 3 x axis_bits
// (axis_bits = min(21, (63 - index_bits) / 3): 15 bits for scans up to 256 k points) of the voxel index RELATIVE to the voxel of
// the scan's predicted pose: every output point lies within max_range of the (moving) sensor origin, so the reachable span is
// 2 max_range / voxel_filter_size cells — +-2.4 km at 0.15 m. A point outside it sets the scan's error flag and the scan's
// result is invalid (ok = -1); the generic dl_voxel_filter has no such limit. Returns and misses share the table (bit 63).
//
// Algorithmic traffic per raw point: A reads 12/16 B and writes 1 bit (+16 B entry per tile winner, read back by A2); B reads
// 1 bit (+12/16 B row + 4 B time, writes 16 B record for survivors, 8 B entry per tile winner, read back by B2) and writes
// 2 bits; C reads 16 B and writes 12 B per output point.
#include <type_traits>
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <vector>

#include "dl_internal.cuh"
#include "dl_pipeline.cuh"

namespace dl {
namespace {

constexpr uint32_t kEmpty32 = 0xFFFFFFFFu;
constexpr unsigned long long kEmpty64 = 0xFFFFFFFFFFFFFFFFull;
constexpr int kBlock = 256;

__device__ __forceinline__ uint32_t hash_cell(const Int3& c) {
  uint32_t h = (uint32_t)c.x * 73856093u ^ (uint32_t)c.y * 19349663u ^ (uint32_t)c.z * 83492791u;
  h ^= h >> 15;
  h *= 0x2c1b3c6du;
  h ^= h >> 12;
  return h;
}

// Slot of a 32-bit hash in a table of `tcap` slots, tcap arbitrary (multiply-shift range reduction: no power-of-two padding).
__device__ __forceinline__ uint32_t table_slot(uint32_t hash, uint32_t tcap) { return __umulhi(hash, tcap); }

__device__ __forceinline__ Vec3f load_xyz(const float* __restrict__ rows, int row_floats, uint32_t i) {
  if (row_floats == 3) {
    const float* p = rows + (size_t)i * 3;
    return {p[0], p[1], p[2]};
  }
  const float4 v = __ldg((const float4*)(rows + (size_t)i * row_floats));  // rows are 16- or 32-byte records
  return {v.x, v.y, v.z};
}

// 12-byte rows: index (into the batch's run arrays) of the time run that contains row i, searched among runs [lo, hi] (the last
// run whose first row is <= i). The ingest kernel bounds the search to the runs of its tile, a few dozen L1-resident starts:
// expanding the run index of every row once per batch (4 B per row, one more kernel and 17 MB of writes per step) made the
// ingest kernel faster but the step slower.
__device__ __forceinline__ int run_search(const FrontendArgs& a, int lo, int hi, int i) {
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(a.run_first_row + mid) <= i) lo = mid; else hi = mid - 1;
  }
  return lo;
}
__device__ __forceinline__ int run_index(const FrontendArgs& a, int b, int i) {
  return run_search(a, a.run_offsets[b], a.run_offsets[b + 1] - 1, i);
}

// Time of row i of scan b: the row's fourth float, or (12-byte rows) the value of the run that contains the row.
__device__ __forceinline__ float point_time(const FrontendArgs& a, int b, const float* __restrict__ rows, int rf, int i) {
  if (rf != 3) return rows[(size_t)i * rf + 3];
  return a.run_value[run_index(a, b, i)];
}

__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  return v;
}
__device__ __forceinline__ int warp_exclusive(int v) {
  const int lane = threadIdx.x & 31;
  int inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int o = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc += o;
  }
  return inc - v;
}

// Both voxel filters keep the lowest input index per voxel, and a minimum can be taken in any grouping: within each tile of kTile
// consecutive rows (shared memory), then over the tile winners of one hash partition (shared memory again, see "partitions"
// below). The survivors are the same for any input order and any tiling; what the tiles buy is that rows arrive in firing order,
// so most duplicates of a voxel lie in the same tile (first filter: 93 %, second filter: 91.5 % of a 64-beam sweep's duplicates,
// tools/frontend_locality.py). A tile table has 2 * kTile slots and holds at most kTile voxels: it cannot fill.
constexpr int kTile = kFrontendTile;
constexpr int kTileSlots = 2 * kTile;

// Appends the index of every non-empty entry of a tile table to `list` (any order) and returns how many there are. The whole CTA
// calls it; kTileSlots is a multiple of the block size, so every warp runs the same number of rounds.
template <typename T>
__device__ __forceinline__ int list_occupied(const T* table, T empty, uint16_t* list, int* count) {
  const int lane = threadIdx.x & 31;
  for (int k = threadIdx.x; k < kTileSlots; k += blockDim.x) {
    const bool used = table[k] != empty;
    const unsigned ballot = __ballot_sync(0xffffffffu, used);
    int at = 0;
    if (lane == 0 && ballot) at = atomicAdd(count, __popc(ballot));
    at = __shfl_sync(0xffffffffu, at, 0);
    if (used) list[at + __popc(ballot & ((1u << lane) - 1))] = (uint16_t)k;
  }
  __syncthreads();
  return *count;
}

// ---------------------------------------------------------------------------------------------------- partitions
// The tile winners of a scan meet by hash partition, not in a scan-wide table. A tile writes its winners to its own kTile-entry
// segment of the scan's stage, grouped by partition, and the end of every partition to its row of part_ends: it writes the whole
// row, so nothing needs clearing. Then one CTA per (scan, partition) (kernels A2 and B2, fe_merge_partitions) reads that
// partition's entries from every tile and keeps the lowest index per voxel in a shared table, as the tiles did; every entry that
// loses there clears its bit in the scan's bitmap, whose words the tiles stored whole. The kernel boundary orders the clears
// after the stores.
//
// A scan has two partitions per row tile (at most kParts), so a partition expects at most half of its shared table's kTile
// entries even when every row is its own voxel. A partition with more entries than that (hash collisions, or scans of more than
// kParts / 2 tiles) runs the same protocol in a global table of 2 slots per entry, carved from the scan's `spill` and cleared by
// the CTA itself. The partition takes hash bits that the tile table's slot does not use, and the merge's table takes the slot's
// bits, which vary freely within a partition.
//
// A tile counts its winners per partition in 16-bit halves of 32-bit words (a count, start or cursor is at most kTile), so that
// kernel B's count fits in its tile's bitmap words once they are stored.
constexpr int kParts = kFrontendParts;
static_assert(kParts % 64 == 0 && kParts / 2 <= 2 * kTile / 32, "kernel B counts partitions in its tile's bitmap words");

__device__ __forceinline__ int num_parts(int n) { return min(2 * ((n + kTile - 1) / kTile), kParts); }
__device__ __forceinline__ size_t row_tiles(const FrontendArgs& a) { return (size_t)((a.cap + kTile - 1) / kTile); }
__device__ __forceinline__ int4* scan_stage(const FrontendArgs& a, int b) { return a.stage + (size_t)b * row_tiles(a) * kTile; }
__device__ __forceinline__ int32_t* part_ends(const FrontendArgs& a, int b, int tile) {
  return a.part_ends + ((size_t)b * row_tiles(a) + tile) * kParts;
}
// First filter: the tile slot is the hash's top 12 bits (table_slot), the partition its low 20 bits.
__device__ __forceinline__ int first_part(uint32_t hash, int parts) { return (int)__umulhi(hash << 12, (uint32_t)parts); }

// Adds one to the 16-bit counter of partition q in hist[kParts / 2] and returns its value before.
__device__ __forceinline__ int part_add(uint32_t* hist, int q) {
  const int shift = (q & 1) * 16;
  return (int)(atomicAdd(hist + (q >> 1), 1u << shift) >> shift) & 0xFFFF;
}

// The whole CTA calls this once hist holds the tile's winners per partition: warp 0 turns the counts into the start of every
// partition in the tile's segment (hist) and stores their ends to the tile's row of part_ends. The caller then places each
// winner at part_add(hist, partition).
__device__ __forceinline__ void partition_starts(uint32_t* hist, int parts, int32_t* ends) {
  if (threadIdx.x < 32) {
    constexpr int kWords = kParts / 64;  // per lane: 2 partitions per word
    uint32_t c[kWords];
    int sum = 0;
#pragma unroll
    for (int j = 0; j < kWords; ++j) {
      c[j] = hist[threadIdx.x * kWords + j];
      sum += (int)(c[j] & 0xFFFF) + (int)(c[j] >> 16);
    }
    int run = warp_exclusive(sum);
#pragma unroll
    for (int j = 0; j < kWords; ++j) {
      const int q = 2 * (threadIdx.x * kWords + j);
      const int lo = run, hi = run + (int)(c[j] & 0xFFFF);
      run = hi + (int)(c[j] >> 16);
      hist[threadIdx.x * kWords + j] = (uint32_t)lo | ((uint32_t)hi << 16);
      if (q < parts) ends[q] = hi;
      if (q + 1 < parts) ends[q + 1] = run;
    }
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------------- A
// One CTA per tile: the rows' cells go to shared memory (consecutive lanes read consecutive rows, so every sector of the tile is
// fetched once), and a shared table keeps the lowest row per cell (comparing cells in shared memory). The tile stores its words
// of the scan's first-filter bitmap, one bit per tile winner, and writes each winner to its partition as {cell x, y, z, row}.
constexpr int kTileBlock = 512;
__global__ void __launch_bounds__(kTileBlock) fe_first_filter_tile(FrontendArgs a) {
  __shared__ Int3 cell[kTile];
  __shared__ uint32_t owner[kTileSlots];
  __shared__ uint16_t winners[kTile];
  __shared__ uint32_t tile_bits[kTile / 32];
  __shared__ uint32_t hist[kParts / 2];
  __shared__ int num_winners;
  const int b = a.first_scan + blockIdx.y;
  const int n = a.counts[b];
  const int base = blockIdx.x * kTile;
  if (base >= n) return;
  const int rows_here = min(kTile, n - base);
  const float* rows = a.ranges + (size_t)b * a.in_cap * a.row_floats;
  const CellDivider res = make_divider(a.first_resolution);
  for (int k = threadIdx.x; k < kTileSlots; k += kTileBlock) owner[k] = kEmpty32;
  if (threadIdx.x == 0) num_winners = 0;
  if (threadIdx.x < kTile / 32) tile_bits[threadIdx.x] = 0;
  if (threadIdx.x < kParts / 2) hist[threadIdx.x] = 0;
  for (int k = threadIdx.x; k < rows_here; k += kTileBlock) cell[k] = cell_index(load_xyz(rows, a.row_floats, base + k), res);
  __syncthreads();
  for (int k = threadIdx.x; k < rows_here; k += kTileBlock) {
    const Int3 c = cell[k];
    uint32_t hh = table_slot(hash_cell(c), kTileSlots);
    uint32_t p = atomicCAS(owner + hh, kEmpty32, (uint32_t)k);
    while (p != kEmpty32) {  // the slot has an owner: same voxel -> the lower row stays; else probe on
      const Int3 o = cell[p];
      if (o.x == c.x && o.y == c.y && o.z == c.z) {
        if ((uint32_t)k < p) atomicMin(owner + hh, (uint32_t)k);  // the owner only ever decreases
        break;
      }
      hh = (hh + 1) & (kTileSlots - 1);
      p = atomicCAS(owner + hh, kEmpty32, (uint32_t)k);
    }
  }
  __syncthreads();
  const int m = list_occupied(owner, kEmpty32, winners, &num_winners);
  // One bit per tile winner; the merge (A2) clears the bits of the winners that lose to another tile's (4 % of the tile winners
  // on a bench sweep).
  const int parts = num_parts(n);
  for (int k = threadIdx.x; k < m; k += kTileBlock) {
    const uint32_t w = owner[winners[k]];
    atomicOr(tile_bits + (w >> 5), 1u << (w & 31));
    part_add(hist, first_part(hash_cell(cell[w]), parts));
  }
  __syncthreads();
  if (threadIdx.x < ((rows_here + 31) >> 5))
    a.first_bits[(size_t)b * a.bit_words + (base >> 5) + threadIdx.x] = tile_bits[threadIdx.x];
  partition_starts(hist, parts, part_ends(a, b, blockIdx.x));
  int4* seg = scan_stage(a, b) + base;
  for (int k = threadIdx.x; k < m; k += kTileBlock) {
    const uint32_t w = owner[winners[k]];
    const Int3 c = cell[w];
    seg[part_add(hist, first_part(hash_cell(c), parts))] = make_int4(c.x, c.y, c.z, base + (int)w);
  }
}

// ---------------------------------------------------------------------------------------------------- B
__device__ __forceinline__ Rigidd interpolate_pose(double s, const ScanConstants& c) {
  Rigidd out;
  out.q = slerp(Quatd{1.0, 0.0, 0.0, 0.0}, c.rel.q, s, c.slerp);
  out.t = mul(s, c.rel.t);
  return out;
}

// pose applied to the point with per-point time t (LTB:430-445)
__device__ __forceinline__ Rigidf point_pose(const ScanConstants& sc, bool no_deskew, double scan_period, float t) {
  if (no_deskew) return to_float(sc.cur);
  const double s = (scan_period + (double)t) / scan_period;
  return to_float(compose(sc.prev, interpolate_pose(s, sc)));
}

// Every point of a time run has the same deskew pose (LTB:430-445 depends on the point's time only): with the times given as
// runs (~2 k firing columns per sweep) the double-precision slerp + composition is done once per RUN here, and the ingest kernel
// loads the finished Rigid3f (32 bytes, L2-resident) instead of ~600 fp64-heavy instructions per survivor. Same arithmetic on the
// same float time -> bit-identical poses.
__global__ void __launch_bounds__(128) fe_run_poses(FrontendArgs a) {
  const int b = a.first_scan + blockIdx.y;
  const int n = a.counts[b];
  const int r = a.run_offsets[b] + blockIdx.x * 128 + threadIdx.x;
  if (n == 0 || r >= a.run_offsets[b + 1]) return;
  const float* rows = a.ranges + (size_t)b * a.in_cap * a.row_floats;
  const bool no_deskew = (double)fabsf(point_time(a, b, rows, a.row_floats, 0)) < 1e-3;  // LTB:430-433
  const Rigidf pose = point_pose(a.scans[b], no_deskew, a.scan_period, a.run_value[r]);
  float4* out = (float4*)(a.run_pose + (size_t)8 * r);
  out[0] = make_float4(pose.t.x, pose.t.y, pose.t.z, pose.q.w);
  out[1] = make_float4(pose.q.x, pose.q.y, pose.q.z, 0.f);
}

// Second-filter slot word of point i in voxel c (see the file header). false: c is outside the key range of this scan.
struct KeyLayout {
  uint32_t bx, by, bz;  // voxel of the scan's predicted pose minus half the key span, per axis (wrapping 32-bit arithmetic)
  int axis_bits, idx_bits;
};
__device__ __forceinline__ KeyLayout key_layout(const FrontendArgs& a, const ScanConstants& sc) {
  const Int3 centre = cell_index(to_float(sc.cur).t, make_divider(a.second_resolution));
  const uint32_t half = 1u << (a.axis_bits - 1);
  return {(uint32_t)centre.x - half, (uint32_t)centre.y - half, (uint32_t)centre.z - half, a.axis_bits, a.idx_bits};
}
__device__ __forceinline__ bool pack_slot(const KeyLayout& k, const Int3& c, bool miss, uint32_t i, unsigned long long* slot) {
  const uint32_t lim = (1u << k.axis_bits) - 1;  // lim itself excluded: the word is never all ones
  const uint32_t rx = (uint32_t)c.x - k.bx, ry = (uint32_t)c.y - k.by, rz = (uint32_t)c.z - k.bz;  // negative -> huge
  if (rx >= lim || ry >= lim || rz >= lim) return false;
  const unsigned long long key = ((unsigned long long)rx << (2 * k.axis_bits)) | ((unsigned long long)ry << k.axis_bits) | (unsigned long long)rz;
  *slot = (miss ? (1ull << 63) : 0ull) | (key << k.idx_bits) | (unsigned long long)i;
  return true;
}
// The voxel of a slot word (inverse of pack_slot's key).
__device__ __forceinline__ Int3 unpack_cell(const KeyLayout& k, unsigned long long slot) {
  const unsigned long long key = slot >> k.idx_bits;  // the miss bit lies above the three axes and is masked off
  const uint32_t m = (1u << k.axis_bits) - 1;
  return {(int)(((uint32_t)(key >> (2 * k.axis_bits)) & m) + k.bx), (int)(((uint32_t)(key >> k.axis_bits) & m) + k.by),
          (int)(((uint32_t)key & m) + k.bz)};
}
// Second-filter hash of a slot word in voxel c: returns and misses apart. The tile slot is its low 12 bits, the partition the 20
// bits above.
__device__ __forceinline__ uint32_t second_hash(const Int3& c, unsigned long long slot) {
  return hash_cell(c) ^ ((slot >> 63) ? 0x9e3779b9u : 0u);
}
__device__ __forceinline__ int second_part(uint32_t hash, int parts) { return (int)__umulhi(hash & 0xFFFFF000u, (uint32_t)parts); }

// Second-filter insert of a slot word into the tile's table: CAS claim; among equal keys (same class and voxel) atomicMin keeps
// the lowest index.
__device__ __forceinline__ void slot_insert(unsigned long long* slots, int idx_bits, const Int3& c, unsigned long long slot) {
  uint32_t hh = second_hash(c, slot) & (kTileSlots - 1);
  for (;;) {
    const unsigned long long prev = atomicCAS(slots + hh, kEmpty64, slot);
    if (prev == kEmpty64) return;
    if ((prev >> idx_bits) == (slot >> idx_bits)) {
      if (slot < prev) atomicMin(slots + hh, slot);  // the owner only ever decreases
      return;
    }
    hh = (hh + 1) & (kTileSlots - 1);
  }
}

// Per-survivor work of kernel B: deskew, transform, range gate, the local-frame record and the second filter's insert into the
// tile table. [run_lo, run_hi]: the tile's time runs (12-byte rows).
template <bool kRunPose>
__device__ __forceinline__ int ingest_survivor(const FrontendArgs& a, int b, const float* rows, int rf, const ScanConstants& sc,
                                               bool no_deskew, const KeyLayout& kl, int run_lo, int run_hi,
                                               unsigned long long* tile_slots, int i) {
  float4 h;
  Rigidf pose;
  if (kRunPose) {  // 12-byte rows, per-run pose table
    const float* p = rows + (size_t)i * 3;
    h = make_float4(p[0], p[1], p[2], 0.f);
    const float4* rp = (const float4*)(a.run_pose + (size_t)8 * run_search(a, run_lo, run_hi, i));
    const float4 p0 = __ldg(rp), p1 = __ldg(rp + 1);
    pose = Rigidf{{p0.x, p0.y, p0.z}, {p0.w, p1.x, p1.y, p1.z}};
  } else if (rf == 3) {
    const float* p = rows + (size_t)i * 3;
    h = make_float4(p[0], p[1], p[2], a.run_value[run_search(a, run_lo, run_hi, i)]);
  } else {
    h = __ldg((const float4*)(rows + (size_t)i * rf));
  }
  const unsigned long long origin_index = rf >= 8 ? *(const unsigned long long*)(rows + (size_t)i * rf + 4) : 0ull;
  const float* o = a.origins + 3 * (origin_index + (unsigned long long)a.origin_base[b]);
  if (!kRunPose) pose = point_pose(sc, no_deskew, a.scan_period, h.w);
  const Vec3f hit = apply(pose, Vec3f{h.x, h.y, h.z});
  const Vec3f org = apply(pose, Vec3f{o[0], o[1], o[2]});
  const Vec3f delta = sub(hit, org);
  const float range = norm3(delta);
  Vec3f outp = hit;
  int cls = 0;
  if (range >= a.min_range) {
    if (range <= a.max_range) {
      cls = 1;
    } else {
      cls = 2;
      outp = add(org, mul(a.max_range / range, delta));
    }
  }
  if (cls) {
    // one aligned 16-byte record per survivor: local-frame point (+ class in .w, which dl_ingest_scan reads for returns_local)
    ((float4*)a.local)[(size_t)b * a.cap + i] = make_float4(outp.x, outp.y, outp.z, __int_as_float(cls));
    const Int3 c = cell_index(outp, make_divider(a.second_resolution));
    unsigned long long slot;
    if (!pack_slot(kl, c, cls == 2, (uint32_t)i, &slot)) {
      a.error_flag[b] = 1;  // per scan: only this scan's result is invalidated
      cls = 0;
    } else {
      slot_insert(tile_slots, kl.idx_bits, c, slot);
    }
  }
  return cls;
}

// One CTA per tile of kTile rows. Warp 0 expands the tile's first-filter bitmap words into a shared list of survivors in index
// order (only ~40 % of the rows survive, so the heavy path runs over the list with all lanes busy): rows are read and local-frame
// records written at nearly consecutive addresses, and the run search of 12-byte rows covers only the tile's few dozen runs
// (L1-resident starts and poses). The survivors' second-filter words meet in the tile table. The CTA stores its tile's words of
// the scan's two bitmaps (returns, misses), one bit per tile winner, and writes the winners' words (self-describing: miss | key
// | index) to their partitions, where B2 clears the bits of those that lose to another tile's.
constexpr int kWordsPerLane = kTile / 32 / 32;  // bitmap words of a tile per lane of warp 0
constexpr int kTileWords = kTile / 32;

__device__ __forceinline__ uint32_t* scan_bits(const FrontendArgs& a, int b, int miss) {
  return a.bits + ((size_t)b * 2 + miss) * a.bit_words;
}

template <bool kRunPose>
__global__ void __launch_bounds__(kBlock, kRunPose ? 6 : 4) fe_ingest_tile(FrontendArgs a) {  // <= 40 / 64 registers
  __shared__ unsigned long long tile_slots[kTileSlots];
  __shared__ uint16_t list[kTile];
  __shared__ uint32_t tile_bits[2][kTileWords];  // the tile winners: returns, misses
  __shared__ int listed, num_winners, run_lo, run_hi;
  const int b = a.first_scan + blockIdx.y;
  const int n = a.counts[b];
  const int base = blockIdx.x * kTile;
  if (base >= n) return;
  const int rows_here = min(kTile, n - base);
  const int rf = a.row_floats;
  const float* rows = a.ranges + (size_t)b * a.in_cap * rf;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int k = threadIdx.x; k < kTileSlots; k += kBlock) tile_slots[k] = kEmpty64;
  if (threadIdx.x < 2 * kTileWords) tile_bits[threadIdx.x / kTileWords][threadIdx.x % kTileWords] = 0u;
  if (warp == 0) {
    const uint32_t* bits = a.first_bits + (size_t)b * a.bit_words + (base >> 5);
    const int words = (rows_here + 31) >> 5;
    uint32_t w[kWordsPerLane];
    int count = 0;
#pragma unroll
    for (int j = 0; j < kWordsPerLane; ++j) {
      const int q = lane * kWordsPerLane + j;
      w[j] = q < words ? __ldcg(bits + q) : 0u;
      count += __popc(w[j]);
    }
    int pos = warp_exclusive(count);
#pragma unroll
    for (int j = 0; j < kWordsPerLane; ++j)
      for (uint32_t x = w[j]; x; x &= x - 1) list[pos++] = (uint16_t)((lane * kWordsPerLane + j) * 32 + __ffs(x) - 1);
    if (lane == 31) listed = pos;
    if (lane == 0) num_winners = 0;
  } else if (threadIdx.x == 32) {
    run_lo = run_hi = 0;
    if (rf == 3) {
      run_lo = run_index(a, b, base);
      run_hi = run_index(a, b, base + rows_here - 1);
    }
  }
  const ScanConstants& sc = a.scans[b];
  const KeyLayout kl = key_layout(a, sc);
  const bool no_deskew = !kRunPose && (double)fabsf(point_time(a, b, rows, rf, 0)) < 1e-3;  // LTB:430-433
  __syncthreads();
  if (threadIdx.x == 0 && listed > 0) {  // survivor count and the LAST survivor (hits_poses.back(), LTB:476)
    atomicAdd(a.n_first + b, listed);
    atomicMax(a.last_index + b, base + list[listed - 1]);
  }
  int returns = 0;
  for (int k = threadIdx.x; k < listed; k += kBlock)  // (shared operands read where used: fewer registers across the loop)
    returns += ingest_survivor<kRunPose>(a, b, rows, rf, sc, no_deskew, kl, run_lo, run_hi, tile_slots, base + list[k]) == 1;
  __syncthreads();
  const int won = list_occupied(tile_slots, kEmpty64, list, &num_winners);
  const unsigned long long idx_mask = (1ull << kl.idx_bits) - 1;
  for (int k = threadIdx.x; k < won; k += kBlock) {
    const unsigned long long s = tile_slots[list[k]];
    const uint32_t w = (uint32_t)(s & idx_mask) - (uint32_t)base;
    atomicOr(&tile_bits[s >> 63][w >> 5], 1u << (w & 31));
  }
  __syncthreads();
  if (threadIdx.x < 2 * kTileWords) {
    const int miss = threadIdx.x / kTileWords, q = threadIdx.x % kTileWords;
    if (q < ((rows_here + 31) >> 5)) __stcg(scan_bits(a, b, miss) + (base >> 5) + q, tile_bits[miss][q]);
  }
  __syncthreads();
  uint32_t* hist = &tile_bits[0][0];  // stored: the words count the winners per partition now (6 CTAs per SM leave no room)
  if (threadIdx.x < kParts / 2) hist[threadIdx.x] = 0;
  __syncthreads();
  const int parts = num_parts(n);
  for (int k = threadIdx.x; k < won; k += kBlock) {
    const unsigned long long s = tile_slots[list[k]];
    part_add(hist, second_part(second_hash(unpack_cell(kl, s), s), parts));
  }
  __syncthreads();
  partition_starts(hist, parts, part_ends(a, b, blockIdx.x));
  unsigned long long* seg = reinterpret_cast<unsigned long long*>(scan_stage(a, b)) + base;
  for (int k = threadIdx.x; k < won; k += kBlock) {
    const unsigned long long s = tile_slots[list[k]];
    seg[part_add(hist, second_part(second_hash(unpack_cell(kl, s), s), parts))] = s;
  }
  returns = warp_sum(returns);
  if (lane == 0 && returns) atomicAdd(a.n_returns_local + b, returns);
}

// ---------------------------------------------------------------------------------------------------- A2, B2
// Merge of entry k into a table of n slots that holds entry positions (Slot: 16 bits in shared memory, 32 in the spill): CAS
// claim; an equal voxel keeps the lower index in the claimer's entry (atomicMin) and clears the bit of the one that lost, the
// newcomer or the index it replaced. A voxel with k entries sees k - 1 meetings, each with a different loser, so exactly the
// lowest index keeps its bit. An entry's index changes only once it has claimed a slot, so entry k is read unchanged here.
template <typename Slot>
__device__ __forceinline__ void merge_entry(const FrontendArgs& a, int b, const KeyLayout&, int4* ent, uint32_t k, Slot* table,
                                            uint32_t n) {
  const int4 e = ent[k];
  const uint32_t i = (uint32_t)e.w;
  uint32_t hh = __umulhi(hash_cell(Int3{e.x, e.y, e.z}), n);  // the top bits: the partition took the low ones
  for (;;) {
    const Slot o = atomicCAS(table + hh, (Slot)~0u, (Slot)k);
    if (o == (Slot)~0u) return;
    const int4 f = ent[o];
    if (f.x == e.x && f.y == e.y && f.z == e.z) {
      const uint32_t loser = max(atomicMin(reinterpret_cast<unsigned*>(&ent[o].w), i), i);
      atomicAnd(a.first_bits + (size_t)b * a.bit_words + (loser >> 5), ~(1u << (loser & 31)));
      return;
    }
    hh = hh + 1 == n ? 0u : hh + 1;
  }
}
template <typename Slot>
__device__ __forceinline__ void merge_entry(const FrontendArgs& a, int b, const KeyLayout& kl, unsigned long long* ent, uint32_t k,
                                            Slot* table, uint32_t n) {
  const unsigned long long s = ent[k];
  const uint32_t h = second_hash(unpack_cell(kl, s), s);
  uint32_t hh = __umulhi(__funnelshift_l(h, h, 20), n);  // the low 12 bits first: the partition took the ones above
  for (;;) {
    const Slot o = atomicCAS(table + hh, (Slot)~0u, (Slot)k);
    if (o == (Slot)~0u) return;
    if ((ent[o] >> kl.idx_bits) == (s >> kl.idx_bits)) {  // the key bits of a claimed entry never change
      const unsigned long long loser = max(atomicMin(ent + o, s), s);
      const uint32_t i = (uint32_t)(loser & ((1ull << kl.idx_bits) - 1));
      atomicAnd(scan_bits(a, b, (int)(loser >> 63)) + (i >> 5), ~(1u << (i & 31)));
      return;
    }
    hh = hh + 1 == n ? 0u : hh + 1;
  }
}

// One CTA per (scan, partition), kSecond: B2, else A2. The partition's entries are copied from every tile's segment into shared
// memory and merged there; when they exceed kTile they are merged where they lie, through a table in the scan's spill.
constexpr int kMergeBlock = 256;
template <bool kSecond>
__global__ void __launch_bounds__(kMergeBlock) fe_merge_partitions(FrontendArgs a) {
  using Entry = typename std::conditional<kSecond, unsigned long long, int4>::type;
  __shared__ Entry ent[kTile];
  __shared__ uint32_t table[kTileSlots / 2];  // kTileSlots 16-bit slots
  __shared__ int fill;
  __shared__ uint32_t* spill;
  const int b = a.first_scan + blockIdx.y;
  const int n = a.counts[b];
  const int p = blockIdx.x;
  if (p >= num_parts(n)) return;
  const int tiles = (n + kTile - 1) / kTile;
  const int32_t* ends = part_ends(a, b, 0) + p;  // tile t: ends[t * kParts]
  Entry* stage = reinterpret_cast<Entry*>(scan_stage(a, b));
  const KeyLayout kl = kSecond ? key_layout(a, a.scans[b]) : KeyLayout{};
  if (threadIdx.x == 0) fill = 0;
  for (int k = threadIdx.x; k < kTileSlots / 2; k += kMergeBlock) table[k] = kEmpty32;
  __syncthreads();
  // a thread per tile reserves room for the tile's entries and copies them while the partition still fits (kCopy loads in
  // flight: a tile holds a few entries of a partition)
  constexpr int kCopy = 4;
  for (int t = threadIdx.x; t < tiles; t += kMergeBlock) {
    const int from = p ? ends[(size_t)t * kParts - 1] : 0, to = ends[(size_t)t * kParts];
    const int at = atomicAdd(&fill, to - from) - from;
    if (at + to > kTile) continue;
    for (int j = from; j < to; j += kCopy) {
      Entry v[kCopy];
#pragma unroll
      for (int u = 0; u < kCopy; ++u)
        if (j + u < to) v[u] = stage[(size_t)t * kTile + j + u];
#pragma unroll
      for (int u = 0; u < kCopy; ++u)
        if (j + u < to) ent[at + j + u] = v[u];
    }
  }
  __syncthreads();
  const int count = fill;
  if (count <= kTile) {
    for (int k = threadIdx.x; k < count; k += kMergeBlock)
      merge_entry(a, b, kl, ent, (uint32_t)k, reinterpret_cast<uint16_t*>(table), (uint32_t)kTileSlots);
    return;
  }
  const uint32_t slots = 2u * (uint32_t)count;
  if (threadIdx.x == 0) spill = a.spill + (size_t)b * 2 * row_tiles(a) * kTile + atomicAdd(a.spill_used + 2 * b + kSecond, (int)slots);
  __syncthreads();
  uint32_t* tab = spill;
  for (uint32_t k = threadIdx.x; k < slots; k += kMergeBlock) tab[k] = kEmpty32;
  __syncthreads();
  for (int t = threadIdx.x; t < tiles; t += kMergeBlock) {
    const int from = p ? ends[(size_t)t * kParts - 1] : 0, to = ends[(size_t)t * kParts];
    for (int j = from; j < to; ++j) merge_entry(a, b, kl, stage, (uint32_t)(t * kTile + j), tab, slots);
  }
}

// ---------------------------------------------------------------------------------------------------- C
constexpr int kEmitBlock = 512, kEmitWarps = kEmitBlock / 32;
constexpr int kChunkPoints = 1024;  // one warp handles 32 bitmap words = 1024 consecutive point indices at a time

// C: gridDim.x CTAs per scan. Every CTA counts the bits of all 1024-point chunks of its scan (32 words per chunk: a few KiB from
// L2), scans the chunk counts, and emits the chunks it owns: the warp expands a chunk's set bits into a shared-memory list and
// then walks the list with all lanes, so that output rows k, k+1, ... are written by neighbouring lanes (coalesced 12-byte rows).
__global__ void __launch_bounds__(kEmitBlock) fe_emit_tracking(FrontendArgs a, int max_chunks) {
  extern __shared__ __align__(16) unsigned char emit_smem[];
  int* off_r = reinterpret_cast<int*>(emit_smem);           // [max_chunks + 1] exclusive prefix of the returns per chunk
  int* off_m = off_r + max_chunks + 1;                       // ... misses
  uint16_t* lists = reinterpret_cast<uint16_t*>(off_m + max_chunks + 1);  // [kEmitWarps][kChunkPoints]
  __shared__ Rigidf back_s;
  __shared__ int warp_tot[2][kEmitWarps];
  __shared__ int carry[2];
  const int b = a.first_scan + blockIdx.y;
  const int n = a.counts[b];
  if (n == 0) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int words = (n + 31) >> 5, chunks = (words + 31) >> 5;
  const uint32_t* bits_r = scan_bits(a, b, 0);
  const uint32_t* bits_m = scan_bits(a, b, 1);
  if (threadIdx.x == 0) {
    // current_pose = pose of the LAST first-filter survivor (hits_poses.back(), LTB:476) and its inverse
    const int rf = a.row_floats;
    const float* rows = a.ranges + (size_t)b * a.in_cap * rf;
    const int last = a.last_index[b];
    Rigidf cur = to_float(a.scans[b].cur);
    if (last >= 0) {
      const bool no_deskew = (double)fabsf(point_time(a, b, rows, rf, 0)) < 1e-3;
      cur = point_pose(a.scans[b], no_deskew, a.scan_period, point_time(a, b, rows, rf, last));
    }
    back_s = inverse(cur);
    if (blockIdx.x == 0) {
      float* cp = a.current_pose + 7 * b;
      cp[0] = cur.t.x; cp[1] = cur.t.y; cp[2] = cur.t.z; cp[3] = cur.q.w; cp[4] = cur.q.x; cp[5] = cur.q.y; cp[6] = cur.q.z;
    }
    carry[0] = carry[1] = 0;
  }
  // per-chunk counts
  for (int c = warp; c < chunks; c += kEmitWarps) {
    const int w = c * 32 + lane;
    const int cr = warp_sum(w < words ? __popc(__ldcg(bits_r + w)) : 0), cm = warp_sum(w < words ? __popc(__ldcg(bits_m + w)) : 0);
    if (lane == 0) {
      off_r[c] = cr;
      off_m[c] = cm;
    }
  }
  __syncthreads();
  // exclusive prefix over the chunks, kEmitBlock at a time
  for (int base = 0; base < chunks; base += kEmitBlock) {
    const int c = base + threadIdx.x;
    const int vr = c < chunks ? off_r[c] : 0, vm = c < chunks ? off_m[c] : 0;
    const int er = warp_exclusive(vr), em = warp_exclusive(vm);
    if (lane == 31) {
      warp_tot[0][warp] = er + vr;
      warp_tot[1][warp] = em + vm;
    }
    __syncthreads();
    int br = carry[0], bm = carry[1];
    for (int w2 = 0; w2 < warp; ++w2) {
      br += warp_tot[0][w2];
      bm += warp_tot[1][w2];
    }
    if (c < chunks) {
      off_r[c] = br + er;
      off_m[c] = bm + em;
    }
    __syncthreads();
    if (threadIdx.x == kEmitBlock - 1) {
      carry[0] = br + er + vr;
      carry[1] = bm + em + vm;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    off_r[chunks] = carry[0];
    off_m[chunks] = carry[1];
    if (blockIdx.x == 0) {
      a.n_returns[b] = carry[0];
      a.n_misses[b] = carry[1];
    }
  }
  __syncthreads();
  const Rigidf back = back_s;
  uint16_t* list = lists + warp * kChunkPoints;
  const float4* local = (const float4*)a.local + (size_t)b * a.cap;
  for (int c = blockIdx.x * kEmitWarps + warp; c < chunks; c += gridDim.x * kEmitWarps) {
#pragma unroll
    for (int cls = 0; cls < 2; ++cls) {
      const int* off = cls ? off_m : off_r;
      const int first = off[c], count = off[c + 1] - first;
      if (count == 0) continue;  // warp-uniform
      const int w = c * 32 + lane;
      uint32_t word = w < words ? __ldcg((cls ? bits_m : bits_r) + w) : 0u;
      int pos = warp_exclusive(__popc(word));
      while (word) {
        const int bit = __ffs(word) - 1;
        word &= word - 1;
        list[pos++] = (uint16_t)(lane * 32 + bit);
      }
      __syncwarp();
      float* dst = (cls ? a.misses_tracking : a.returns_tracking) + ((size_t)b * a.cap + first) * 3;
      for (int k = lane; k < count; k += 32) {
        const float4 l = __ldcg(local + (size_t)c * kChunkPoints + list[k]);
        const Vec3f q = apply(back, Vec3f{l.x, l.y, l.z});
        dst[3 * k] = q.x; dst[3 * k + 1] = q.y; dst[3 * k + 2] = q.z;
      }
      __syncwarp();
    }
  }
}

__global__ void fe_reset_counters(FrontendArgs a, int batch) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch) return;
  a.n_first[b] = 0;
  a.n_returns_local[b] = 0;
  a.last_index[b] = -1;
  if (a.counts[b] == 0) {  // nothing will write these for an empty scan
    a.n_returns[b] = 0;
    a.n_misses[b] = 0;
    const Rigidf cur = to_float(a.scans[b].cur);
    float* cp = a.current_pose + 7 * b;
    cp[0] = cur.t.x; cp[1] = cur.t.y; cp[2] = cur.t.z; cp[3] = cur.q.w; cp[4] = cur.q.x; cp[5] = cur.q.y; cp[6] = cur.q.z;
  }
  a.error_flag[b] = 0;
  a.spill_used[2 * b] = a.spill_used[2 * b + 1] = 0;
}

// ---------------------------------------------------------------------------------------------------- glue
// Plain gather of selected rows (adaptive filter survivors) into a dense cloud.
__global__ void __launch_bounds__(kBlock) gather_rows_kernel(const float* __restrict__ in, int64_t cap_in, int pairs_per_cloud,
                                                             const int32_t* __restrict__ keep, const int32_t* __restrict__ keep_counts,
                                                             int64_t cap_out, float* __restrict__ out) {
  const int pair = blockIdx.y;
  const int b = pair / pairs_per_cloud;
  const int count = keep_counts[pair];
  // grid-stride: the survivors are a few hundred rows, so a handful of CTAs per cloud replaces one per 256 rows of capacity
  for (int j = blockIdx.x * kBlock + threadIdx.x; j < count; j += gridDim.x * kBlock) {
    const float* p = in + ((size_t)b * cap_in + keep[(size_t)pair * cap_in + j]) * 3;
    float* o = out + ((size_t)pair * cap_out + j) * 3;
    o[0] = p[0]; o[1] = p[1]; o[2] = p[2];
  }
}

// initial_ceres_pose = submap.local_pose^-1 * pose_prediction, pose_prediction = current_pose.cast<double>() (LTB:476-487, :504-505)
__global__ void initial_pose_kernel(int batch, const float* __restrict__ current_pose, const Rigidd* __restrict__ submap_inverse,
                                    double* __restrict__ initial_pose, double* __restrict__ target_translation) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch) return;
  const float* cp = current_pose + 7 * b;
  const Rigidd prediction = to_double(Rigidf{{cp[0], cp[1], cp[2]}, {cp[3], cp[4], cp[5], cp[6]}});
  const Rigidd init = compose(submap_inverse[b], prediction);
  pose_to7(init, initial_pose + 7 * b);
  target_translation[3 * b] = init.t.x;
  target_translation[3 * b + 1] = init.t.y;
  target_translation[3 * b + 2] = init.t.z;
}

__global__ void finalize_results_kernel(ResultArgs a) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= a.batch) return;
  dl_scan_result& r = a.results[b];
  const int n_hi = a.adaptive_counts[2 * b], n_lo = a.adaptive_counts[2 * b + 1];
  r.num_first_filter = a.first_counts[b];
  r.num_returns = a.return_counts[b];
  r.num_misses = a.miss_counts[b];
  r.num_high_resolution = n_hi;
  r.num_low_resolution = n_lo;
  r.num_cropped_high = a.adaptive_cropped[2 * b];
  r.num_cropped_low = a.adaptive_cropped[2 * b + 1];
  r.num_passes_high = a.adaptive_passes[2 * b];
  r.num_passes_low = a.adaptive_passes[2 * b + 1];
  r.rtcsm_score = a.rtcsm_scores ? a.rtcsm_scores[b] : 0.f;
  r.reserved = 0;
  // the reference drops the scan when any of the three clouds is empty (LTB:497-500, :510-513, :531-534)
  r.ok = (a.return_counts[b] > 0 && n_hi > 0 && n_lo > 0) ? 1 : 0;
  if (a.error_flag && a.error_flag[b]) r.ok = -1;  // a point fell outside +-2^20 voxels: results are not valid
  if (a.imu_ok && a.imu_ok[b] == 0) r.ok = -2;   // no IMU factor (no samples / covariance not positive definite): no solve ran
  const double* pose = a.fused ? a.fused[b].state : a.nls[b].pose;
  r.summary = a.fused ? a.fused[b].summary : a.nls[b].summary;
  for (int i = 0; i < 7; ++i) r.pose_observation_in_submap[i] = pose[i];
  const Rigidd submap = a.submap[b];
  const Rigidd est = compose(submap, pose_from7(pose));  // LTB:553-554
  pose_to7(est, r.pose_estimate_local);
  if (a.fused && a.states_out) {  // solver state (submap frame) -> dl_nav_state in the local frame
    dl_nav_state& o = a.states_out[b];
    const Vec3d v = rotate(submap.q, Vec3d{pose[7], pose[8], pose[9]});
    o.p[0] = est.t.x; o.p[1] = est.t.y; o.p[2] = est.t.z;
    o.q[0] = est.q.w; o.q[1] = est.q.x; o.q[2] = est.q.y; o.q[3] = est.q.z;
    o.v[0] = v.x; o.v[1] = v.y; o.v[2] = v.z;
    for (int k = 0; k < 3; ++k) { o.ba[k] = pose[10 + k]; o.bg[k] = pose[13 + k]; }
  }
}

}  // namespace

// Nothing of the front half needs clearing: the tiles store every bitmap word and part_ends row that is read, and a spilled
// partition clears its own table.
int launch_fe_prepare(dl_context* ctx, const FrontendArgs& a, int batch) {
  fe_reset_counters<<<(batch + 127) / 128, 128, 0, ctx->stream>>>(a, batch);
  DL_LAUNCH_CHECK(ctx, "fe_reset_counters");
  return DL_OK;
}

static int launch_merge(dl_context* ctx, const FrontendArgs& a, int row_tiles, int num_scans, bool second) {
  const dim3 grid(std::min(2 * row_tiles, kParts), num_scans);
  if (second) fe_merge_partitions<true><<<grid, kMergeBlock, 0, ctx->stream>>>(a);
  else fe_merge_partitions<false><<<grid, kMergeBlock, 0, ctx->stream>>>(a);
  DL_LAUNCH_CHECK(ctx, "fe_merge_partitions");
  return DL_OK;
}

// Kernels A and A2 for scans [first_scan, first_scan + num_scans): lets the host overlap the upload of later scans.
int launch_fe_first_filter(dl_context* ctx, FrontendArgs a, int first_scan, int num_scans) {
  if (num_scans <= 0) return DL_OK;
  a.first_scan = first_scan;
  const int row_tiles = (int)((a.cap + kTile - 1) / kTile);
  fe_first_filter_tile<<<dim3(row_tiles, num_scans), kTileBlock, 0, ctx->stream>>>(a);
  DL_LAUNCH_CHECK(ctx, "fe_first_filter_tile");
  return launch_merge(ctx, a, row_tiles, num_scans, false);
}

int launch_fe_rest(dl_context* ctx, FrontendArgs a, int first_scan, int batch) {
  if (batch <= 0) return DL_OK;
  a.first_scan = first_scan;
  const int row_tiles = (int)((a.cap + kTile - 1) / kTile);
  if (a.run_pose && a.max_runs > 0) {
    fe_run_poses<<<dim3((a.max_runs + 127) / 128, batch), 128, 0, ctx->stream>>>(a);
    DL_LAUNCH_CHECK(ctx, "fe_run_poses");
    fe_ingest_tile<true><<<dim3(row_tiles, batch), kBlock, 0, ctx->stream>>>(a);
  } else {
    fe_ingest_tile<false><<<dim3(row_tiles, batch), kBlock, 0, ctx->stream>>>(a);
  }
  DL_LAUNCH_CHECK(ctx, "fe_ingest_tile");
  if (const int st = launch_merge(ctx, a, row_tiles, batch, true)) return st;
  const int max_chunks = (int)((a.bit_words + 31) / 32);
  const size_t smem = (size_t)2 * (max_chunks + 1) * sizeof(int) + (size_t)kEmitWarps * kChunkPoints * sizeof(uint16_t);
  if (smem > 200 * 1024) return ctx->fail(DL_ERR_ARG, "scan too large for the front end's compaction (> 20 M points)");
  static bool emit_attr = false;  // dynamic shared memory above 48 KiB needs the opt-in once per process
  if (smem > 48 * 1024 && !emit_attr) {
    DL_CUDA(ctx, cudaFuncSetAttribute(fe_emit_tracking, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    emit_attr = true;
  }
  const int parts = 4;  // CTAs per scan: a 74-scan sub-batch x 4 = 296 CTAs of 512 threads, about two per SM of an H100
  fe_emit_tracking<<<dim3(parts, batch), kEmitBlock, smem, ctx->stream>>>(a, max_chunks);
  DL_LAUNCH_CHECK(ctx, "fe_emit_tracking");
  return DL_OK;
}

int launch_gather_rows(dl_context* ctx, const float* in, int64_t cap_in, int pairs_per_cloud, const int32_t* keep,
                       const int32_t* keep_counts, int64_t cap_out, float* out, int pairs) {
  if (pairs <= 0) return DL_OK;
  const dim3 grid((unsigned)std::min<int64_t>((cap_out + kBlock - 1) / kBlock, 8), pairs);
  gather_rows_kernel<<<grid, kBlock, 0, ctx->stream>>>(in, cap_in, pairs_per_cloud, keep, keep_counts, cap_out, out);
  DL_LAUNCH_CHECK(ctx, "gather_rows_kernel");
  return DL_OK;
}

int launch_initial_pose(dl_context* ctx, int batch, const float* current_pose, const Rigidd* submap_inverse,
                        double* initial_pose, double* target_translation) {
  if (batch <= 0) return DL_OK;
  initial_pose_kernel<<<(batch + 127) / 128, 128, 0, ctx->stream>>>(batch, current_pose, submap_inverse, initial_pose,
                                                                    target_translation);
  DL_LAUNCH_CHECK(ctx, "initial_pose_kernel");
  return DL_OK;
}

int launch_finalize_results(dl_context* ctx, const ResultArgs& a) {
  if (a.batch <= 0) return DL_OK;
  finalize_results_kernel<<<(a.batch + 127) / 128, 128, 0, ctx->stream>>>(a);
  DL_LAUNCH_CHECK(ctx, "finalize_results_kernel");
  return DL_OK;
}

}  // namespace dl

// ------------------------------------------------------------------------------------------------ batched front end
using namespace dl;

namespace {

// Device scratch of one front-end run.
void carve(Arena& a, int batch, int64_t cap, int num_origins, FrontendBuffers* f) {
  const size_t B = (size_t)batch, C = (size_t)cap;
  f->batch = batch;
  f->cap = cap;
  f->tcap = next_pow2(2 * cap);
  f->counts0 = a.take<int32_t>(B); f->n1 = a.take<int32_t>(B); f->n_ret = a.take<int32_t>(B);
  f->n2 = a.take<int32_t>(B); f->n3 = a.take<int32_t>(B); f->countsA = a.take<int32_t>(2 * B); f->npassesA = a.take<int32_t>(2 * B);
  f->croppedA = a.take<int32_t>(2 * B);
  f->tableA = a.take<uint32_t>(B * 2 * f->tcap); f->scratchA = a.take<uint32_t>(B * 4 * C);
  f->keepA = a.take<int32_t>(B * 2 * C);
  f->returns_tracking = a.take<float>(B * C * 3); f->misses_tracking = a.take<float>(B * C * 3);
  f->clouds = a.take<float>(B * 2 * C * 3); f->current_pose = a.take<float>(B * 7); f->origins = a.take<float>((size_t)num_origins * 3);
  f->passesA = a.take<float>(B * 2 * 32); f->rtcsm_scores = a.take<float>(B);
  f->scans = a.take<ScanConstants>(B); f->filters = a.take<AdaptiveParams>(2);
  f->submap = a.take<Rigidd>(B); f->submap_inverse = a.take<Rigidd>(B); f->origin_base = a.take<int32_t>(B);
  f->initial_pose = a.take<double>(B * 7); f->target = a.take<double>(B * 3);
  f->problems = a.take<NlsProblem>(B); f->nls_out = a.take<NlsOutput>(B);
  f->bit_words = (int64_t)((C + 31) / 32);
  f->bits = a.take<uint32_t>(B * 2 * f->bit_words);
  f->first_bits = a.take<uint32_t>(B * f->bit_words);
  const size_t tiles = (C + kFrontendTile - 1) / kFrontendTile;
  f->stage = a.take<int4>(B * tiles * kFrontendTile);
  f->part_ends = a.take<int32_t>(B * tiles * kFrontendParts);
  f->spill = a.take<uint32_t>(B * 2 * tiles * kFrontendTile);
  f->spill_used = a.take<int32_t>(2 * B);
  f->last_index = a.take<int32_t>(B); f->error_flag = a.take<int32_t>(B);
  f->local4 = a.take<float>(B * C * 4);
}

// Device copies of the time_run_* arrays of 12-byte rows (validated by check_frontend) and, with many runs per scan, the table
// of per-run deskew poses: one pose per run (fe_run_poses) instead of one per survivor.
void carve_time_runs(Arena& a, const dl_frontend_options& o, int num_scans, FrontendBuffers* f) {
  if (o.range_row_floats != 3) return;
  const size_t runs = (size_t)o.time_run_offsets[num_scans];
  f->run_offsets = a.take<int32_t>((size_t)num_scans + 1);
  f->run_first_row = a.take<int32_t>(runs);
  f->run_value = a.take<float>(runs);
  if (runs > (size_t)8 * num_scans) f->run_pose = a.take<float>(runs * 8);
}

// The pre-match's per-scan flags, carved last so that every other buffer sits where it does without the pre-match.
void carve_prematch(Arena& a, const dl_frontend_options& o, int num_scans, FrontendBuffers* f) {
  if (o.use_online_correlative_scan_matching) f->rtcsm_nonpositive = a.take<int32_t>((size_t)num_scans);
}

FrontendArgs make_frontend_args(const dl_frontend_options& o, const FrontendBuffers& f, const float* d_ranges,
                                int64_t in_cap, int row_floats) {
  FrontendArgs fa{};
  fa.ranges = d_ranges; fa.in_cap = in_cap; fa.row_floats = row_floats; fa.counts = f.counts0; fa.scans = f.scans;
  fa.origins = f.origins; fa.origin_base = f.origin_base; fa.cap = f.cap;
  fa.first_resolution = 0.5f * o.voxel_filter_size;  // LTB:394
  fa.second_resolution = o.voxel_filter_size;        // LTB:479-484
  fa.min_range = o.min_range; fa.max_range = o.max_range; fa.scan_period = o.scan_period;
  fa.first_bits = f.first_bits; fa.bits = f.bits; fa.bit_words = f.bit_words;
  fa.stage = f.stage; fa.part_ends = f.part_ends; fa.spill = f.spill; fa.spill_used = f.spill_used;
  fa.idx_bits = 1;
  while (((int64_t)1 << fa.idx_bits) < f.cap) ++fa.idx_bits;      // point indices are < cap
  fa.axis_bits = std::min(21, (63 - fa.idx_bits) / 3);             // 15 bits per axis up to 256 k points per scan
  fa.local = f.local4;
  fa.returns_tracking = f.returns_tracking; fa.misses_tracking = f.misses_tracking;
  fa.n_first = f.n1; fa.n_returns_local = f.n_ret; fa.n_returns = f.n2; fa.n_misses = f.n3; fa.last_index = f.last_index;
  fa.current_pose = f.current_pose; fa.error_flag = f.error_flag;
  return fa;
}

int row_floats_of(const dl_frontend_options& o) { return o.range_row_floats == 4 ? 4 : (o.range_row_floats == 3 ? 3 : 8); }

ScanConstants make_scan_constants(const double* prev7, const double* cur7) {  // dl_pipeline.cuh has the arithmetic
  return dl::make_scan_constants(pose_from7(prev7), pose_from7(cur7));
}

// The pinned staging block of a front-end batch: the small per-call tables, then the results and estimated IMU states that a
// submitted batch downloads (dl_frontend_submit*, collected by dl_frontend_collect*).
struct Staging {
  int32_t* counts;
  ScanConstants* scans;
  float* origins;
  AdaptiveParams* filters;
  NlsProblem* problems;
  dl_scan_result* results;
  dl_nav_state* states;
  Rigidd* submaps;      // per scan: pose, inverse
  int32_t* origin_base;
};
void carve_staging(Arena& h, int batch, int num_origins, Staging* s) {
  const size_t B = (size_t)batch;
  s->counts = h.take<int32_t>(B);
  s->submaps = h.take<Rigidd>(2 * B);
  s->origin_base = h.take<int32_t>(B);
  s->scans = h.take<ScanConstants>(B);
  s->origins = h.take<float>((size_t)num_origins * 3);
  s->filters = h.take<AdaptiveParams>(2);
  s->problems = h.take<NlsProblem>(B);
  s->results = h.take<dl_scan_result>(B);
  s->states = h.take<dl_nav_state>(B);
}

// Uploads the small per-call tables (counts, deskew constants, origins, filter options, NLS problem records, matching
// submaps) through the pinned staging block. No host synchronisation: the block is reused only after `staging_done`.
// origin_base (optional, per scan): where each scan's origins start in `origins`; without it every scan uses them all.
int frontend_upload_small(dl_context* ctx, const dl_frontend_options& o, const FrontendBuffers& f, const int64_t* sizes,
                          const float* origins, int num_origins, const double* prev_poses, const double* cur_poses,
                          const SubmapSet* submaps, const int32_t* origin_base = nullptr, const int32_t* enabled_dev = nullptr) {
  const size_t B = (size_t)f.batch;
  Staging s;
  Arena count(nullptr);
  carve_staging(count, f.batch, num_origins, &s);
  DL_TRY(ctx->reserve_pinned(count.off));
  DL_CUDA(ctx, cudaEventSynchronize(ctx->staging_done));
  Arena h(ctx->h_pinned.get());
  carve_staging(h, f.batch, num_origins, &s);
  for (int b = 0; b < f.batch; ++b) {
    s.counts[b] = (int32_t)sizes[b];
    s.origin_base[b] = origin_base ? origin_base[b] : 0;
    if (prev_poses) s.scans[b] = make_scan_constants(prev_poses + 7 * b, cur_poses + 7 * b);
    NlsProblem& p = s.problems[b];
    std::memset(&p, 0, sizeof(p));
    if (submaps) {
      const Rigidd pose = pose_from7(submaps->pose(b));
      s.submaps[2 * b] = pose;
      s.submaps[2 * b + 1] = inverse(pose);
      for (int k = 0; k < 2; ++k) {
        p.cloud[k] = f.clouds + (size_t)(2 * b + k) * f.cap * 3;
        p.count_dev[k] = f.countsA + 2 * b + k;
        p.grid[k] = k == 0 ? submaps->high(b)->view() : submaps->low(b)->view();
      }
      p.initial_dev = f.initial_pose + 7 * b;
      p.target_dev = f.target + 3 * b;
      if (enabled_dev) p.enabled_dev = enabled_dev + b;  // scans whose IMU factor could not be formed are not solved
    }
  }
  std::memcpy(s.origins, origins, (size_t)num_origins * 12);
  s.filters[0] = {o.high_resolution_adaptive_voxel_filter.max_length, o.high_resolution_adaptive_voxel_filter.min_num_points,
                  o.high_resolution_adaptive_voxel_filter.max_range};
  s.filters[1] = {o.low_resolution_adaptive_voxel_filter.max_length, o.low_resolution_adaptive_voxel_filter.min_num_points,
                  o.low_resolution_adaptive_voxel_filter.max_range};
  DL_TRY(h2d(ctx, f.counts0, s.counts, B));
  if (prev_poses) DL_TRY(h2d(ctx, f.scans, s.scans, B));  // otherwise imu_prepare_kernel writes them on the device
  DL_TRY(h2d(ctx, f.origins, s.origins, (size_t)num_origins * 3));
  DL_TRY(h2d(ctx, f.filters, s.filters, 2));
  DL_TRY(h2d(ctx, f.problems, s.problems, B));
  DL_TRY(h2d(ctx, f.origin_base, s.origin_base, B));
  if (submaps) {
    DL_CUDA(ctx, cudaMemcpy2DAsync(f.submap, sizeof(Rigidd), s.submaps, 2 * sizeof(Rigidd), sizeof(Rigidd), B, cudaMemcpyHostToDevice,
                                   ctx->stream));
    DL_CUDA(ctx, cudaMemcpy2DAsync(f.submap_inverse, sizeof(Rigidd), s.submaps + 1, 2 * sizeof(Rigidd), sizeof(Rigidd), B,
                                   cudaMemcpyHostToDevice, ctx->stream));
  }
  DL_CUDA(ctx, cudaEventRecord(ctx->staging_done, ctx->stream));
  return DL_OK;
}

void carve_imu(Arena& a, int num_scans, ImuRun* r) {
  r->d_terms = a.take<ImuTerm>(num_scans);
  r->d_init16 = a.take<double>((size_t)num_scans * 16);
  r->d_fused = a.take<FusedOutput>(num_scans);
  r->d_states = r->d_states_out ? r->d_states_out : a.take<dl_nav_state>(num_scans);
  if (!r->samples) return;
  const size_t ns = (size_t)r->samples->offsets[num_scans];
  r->d_off = a.take<int32_t>(num_scans + 1);
  r->d_dt = a.take<double>(ns);
  r->d_acc = a.take<double>(3 * ns);
  r->d_gyr = a.take<double>(3 * ns);
  r->d_si = a.take<dl_nav_state>(num_scans);
  r->d_pre = a.take<dl_preintegration>(num_scans);
  r->d_predicted = a.take<dl_nav_state>(num_scans);
  r->d_ok = a.take<int32_t>(num_scans);
}

// CTAs per least-squares problem. The pipeline's adaptive filters hand the matcher a few hundred points: one CTA. With the filters
// opened up (min_num_points in the thousands: SURVEY 8d's full-cloud mode F, tens of thousands of points per solve) one 256-thread
// CTA per problem is latency-bound and leaves half the SMs idle, so the problem is spread over a thread-block cluster — as many
// CTAs as keep the launch within one wave of the SMs (on an H100's 132 SMs: 2 for sub-batches of up to 66 problems, 1 for the
// bench's 74), at most the portable 8.
// DLIOM_NLS_CLUSTER=n forces n (1 = never).
int solve_cluster_size(dl_context* ctx, const dl_frontend_options& o, int problems) {
  if (const char* env = std::getenv("DLIOM_NLS_CLUSTER")) return std::max(1, std::min(8, std::atoi(env)));
  const float few = 4096.f;
  if (o.high_resolution_adaptive_voxel_filter.min_num_points < few && o.low_resolution_adaptive_voxel_filter.min_num_points < few) return 1;
  int sms = kNumSMs;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, ctx->device);
  int cs = 1;
  while (cs < 8 && problems * cs * 2 <= sms) cs *= 2;
  return cs;
}

// The batch is processed as `chunks` sub-batches that alternate between two streams, so that
//   - with host scans (host_ranges != nullptr) the upload of sub-batch k+1 (copy stream) overlaps the kernels of k;
//   - the latency-bound tail of sub-batch k (adaptive filter: 2 CTAs per scan, LM solve: 1 CTA per scan) overlaps the
//     bandwidth-bound front half of sub-batch k+1.
// Every kernel launcher enqueues on ctx->stream, which is pointed at the sub-batch's stream while it is enqueued.
int frontend_run(dl_context* ctx, const dl_frontend_options& o, int num_scans, float* d_ranges, int64_t in_cap,
                 const void* const* host_ranges, const int64_t* sizes, const float* origins, int num_origins,
                 const int32_t* origin_base, const double* prev_poses, const double* cur_poses, const SubmapSet& submaps,
                 const FrontendBuffers& f, Arena& a, dl_scan_result* d_results, ImuRun* imu_run = nullptr) {
  // optional IMU coupling: one pre-integration factor per scan, the 15-parameter solve instead of the 6-parameter one
  const ImuRun no_imu;
  const ImuRun& m = imu_run ? *imu_run : no_imu;
  const dl_frontend_imu* imu = m.host;
  const dl_frontend_imu_samples* raw = m.samples;
  if (imu) {
    std::vector<ImuTerm> terms(num_scans);
    std::vector<double> init16((size_t)num_scans * 16);
    for (int b = 0; b < num_scans; ++b)
      if (!build_imu_term(inverse(pose_from7(submaps.pose(b))), imu->states_i[b], imu->predicted_states[b], imu->preintegrations[b], imu->gravity,
                          imu->imu_weight, &terms[b], init16.data() + 16 * b))
        return ctx->fail(DL_ERR_ARG, "pre-integration covariance is not positive definite");
    DL_TRY(h2d(ctx, m.d_terms, terms.data(), num_scans));
    DL_TRY(h2d(ctx, m.d_init16, init16.data(), (size_t)num_scans * 16));
    DL_TRY(sync(ctx));  // the staging vectors are pageable and local
  }
  if (imu || raw) DL_CUDA(ctx, cudaMemsetAsync(m.d_fused, 0, sizeof(FusedOutput) * num_scans, ctx->stream));
  const int rf = row_floats_of(o);
  DL_TRY(frontend_upload_small(ctx, o, f, sizes, origins, num_origins, raw ? nullptr : prev_poses, cur_poses, &submaps, origin_base,
                               m.d_ok));
  FrontendArgs fa = make_frontend_args(o, f, d_ranges, in_cap, rf);
  if (rf == 3) {  // per-point times as runs: validated by check_frontend, uploaded next to the scans
    const size_t runs = (size_t)o.time_run_offsets[num_scans];
    DL_TRY(h2d(ctx, f.run_offsets, o.time_run_offsets, (size_t)num_scans + 1));
    DL_TRY(h2d(ctx, f.run_first_row, o.time_run_first_row, runs));
    DL_TRY(h2d(ctx, f.run_value, o.time_run_value, runs));
    fa.run_offsets = f.run_offsets; fa.run_first_row = f.run_first_row; fa.run_value = f.run_value;
    if (f.run_pose) {
      int max_runs = 0;
      for (int b = 0; b < num_scans; ++b) max_runs = std::max(max_runs, (int)(o.time_run_offsets[b + 1] - o.time_run_offsets[b]));
      fa.run_pose = f.run_pose;  // filled per sub-batch by fe_run_poses once the scans' deskew constants exist
      fa.max_runs = max_runs;
    }
  }
  DL_TRY(launch_fe_prepare(ctx, fa, f.batch));
  const float hi_resolution = submaps.high(0)->resolution;  // one for the batch (check_frontend)
  const bool rtcsm = o.use_online_correlative_scan_matching != 0;
  int chunks = rtcsm ? 1 : (host_ranges ? 5 : 2);
  if (f.batch < 8 * chunks) chunks = std::max(1, f.batch / 8);
  // Sub-batches alternate between two equal-priority streams. Every back half (latency-bound, one or two CTAs per scan) on one
  // high-priority stream behind its front half would serialise the back halves, which costs more than the priority gains.
  // DLIOM_SERIAL=1: every sub-batch on the main stream, nothing overlaps (bench.py's per-stage roofline pass: the stage events then
  // bracket the kernels' own durations at the sub-batch size the step really uses)
  const bool serial = std::getenv("DLIOM_SERIAL") != nullptr;
  cudaStream_t main_stream = ctx->stream;
  cudaEvent_t prepared = ctx->take_event();
  DL_CUDA(ctx, cudaEventRecord(prepared, main_stream));
  DL_CUDA(ctx, cudaStreamWaitEvent(ctx->aux_stream, prepared, 0));
  DL_CUDA(ctx, cudaStreamWaitEvent(ctx->tail_stream, prepared, 0));
  if (host_ranges) DL_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream, prepared, 0));  // the upload target may be in use
  ctx->event_pool.push_back(prepared);
  cudaEvent_t imu_ready = nullptr;
  if (raw) {
    // Raw samples: pre-integration, prediction, deskew constants, factor and information matrix all on the device; the
    // only host work is the upload of the samples and of the states at the previous scans. The chain runs on its own
    // stream next to the first voxel filter (which needs none of it); the ingest kernels wait for `imu_ready`.
    ctx->stream = ctx->tail_stream;
    auto chain = [&]() -> int {
      StageScope st(ctx, "imu_preintegrate_predict");
      const size_t ns = (size_t)raw->offsets[num_scans];
      DL_TRY(h2d(ctx, m.d_off, raw->offsets, (size_t)num_scans + 1));
      DL_TRY(h2d(ctx, m.d_dt, raw->dt, ns));
      DL_TRY(h2d(ctx, m.d_acc, raw->acc, 3 * ns));
      DL_TRY(h2d(ctx, m.d_gyr, raw->gyr, 3 * ns));
      DL_TRY(h2d(ctx, m.d_si, raw->states_i, (size_t)num_scans));
      DL_TRY(launch_imu_preintegrate(ctx, num_scans, m.d_off, m.d_dt, m.d_acc, m.d_gyr, (const double*)m.d_si + 10, 16, raw->noise,
                                     m.d_pre));
      ImuPrepareArgs pa{};
      pa.count = num_scans; pa.preint = m.d_pre; pa.states_i = m.d_si; pa.to_submap = f.submap_inverse;
      for (int k = 0; k < 3; ++k) pa.gravity[k] = raw->gravity[k];
      pa.imu_weight = raw->imu_weight; pa.scans = f.scans; pa.terms = m.d_terms; pa.init16 = m.d_init16; pa.predicted = m.d_predicted;
      pa.ok = m.d_ok;
      return launch_imu_prepare(ctx, pa);
    };
    const int st_imu = chain();
    ctx->stream = main_stream;
    DL_TRY(st_imu);
    imu_ready = ctx->take_event();
    DL_CUDA(ctx, cudaEventRecord(imu_ready, ctx->tail_stream));  // recycled once every sub-batch's wait is enqueued
  }
  std::vector<float> rtcsm_scores;
  bool have_scores = false;
  int status = DL_OK;
  // Sub-batch boundaries. Device-resident scans: equal parts. Host scans: the upload is the long pole and the kernels of
  // the LAST sub-batch are exposed after its copy ends, so the last parts shrink (shares 1 : ... : 1 : 1/2 : 1/4) — their
  // back halves are latency-bound (~0.6 ms however few scans), so only the front-half time shrinks with them.
  std::vector<int> bounds(chunks + 1, 0);
  {
    std::vector<double> share(chunks, 1.0);
    if (host_ranges && chunks >= 3) {
      share[chunks - 2] = 0.5;
      share[chunks - 1] = 0.25;
    }
    double total = 0, acc = 0;
    for (double v : share) total += v;
    for (int k = 0; k < chunks; ++k) {
      acc += share[k];
      bounds[k + 1] = k + 1 == chunks ? f.batch : (int)std::lround(f.batch * acc / total);
    }
  }
  for (int k = 0; k < chunks && status == DL_OK; ++k) {
    const int b0 = bounds[k], b1 = bounds[k + 1], nb = b1 - b0;
    if (nb <= 0) continue;
    ctx->stream = (!serial && (k & 1)) ? ctx->aux_stream : main_stream;
    auto run = [&]() -> int {
      {
        StageScope st(ctx, "voxel_filter_first");
        if (host_ranges && o.host_scan_stride_rows > 0) {
          int64_t widest = 0;
          for (int b = b0; b < b1; ++b) widest = std::max(widest, sizes[b]);
          if (widest > 0)
            DL_CUDA(ctx, cudaMemcpy2DAsync(d_ranges + (size_t)b0 * in_cap * rf, (size_t)in_cap * rf * 4, host_ranges[b0],
                                           (size_t)o.host_scan_stride_rows * rf * 4, (size_t)widest * rf * 4, (size_t)nb,
                                           cudaMemcpyHostToDevice, ctx->copy_stream));
        } else if (host_ranges) {
          for (int b = b0; b < b1; ++b)
            if (sizes[b] > 0)
              DL_CUDA(ctx, cudaMemcpyAsync(d_ranges + (size_t)b * in_cap * rf, host_ranges[b], (size_t)sizes[b] * rf * 4,
                                           cudaMemcpyHostToDevice, ctx->copy_stream));
        }
        if (host_ranges) {
          cudaEvent_t ev = ctx->take_event();
          DL_CUDA(ctx, cudaEventRecord(ev, ctx->copy_stream));
          DL_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ev, 0));
          ctx->event_pool.push_back(ev);  // safe to recycle: the wait has been enqueued
        }
        DL_TRY(launch_fe_first_filter(ctx, fa, b0, nb));
      }
      if (imu_ready) DL_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, imu_ready, 0));
      {
        StageScope st(ctx, "ingest_second_filter");
        DL_TRY(launch_fe_rest(ctx, fa, b0, nb));
      }
      {
        // adaptive voxel filters (high, low resolution) on the tracking-frame returns: one CTA per (scan, filter)
        StageScope st(ctx, "adaptive_voxel_filter");
        DL_TRY(launch_adaptive_voxel_filter(ctx, f.returns_tracking + (size_t)b0 * f.cap * 3, 3, f.cap, f.n2 + b0, nb, f.filters, 2,
                                            f.tableA + (size_t)2 * b0 * f.tcap, f.tcap, f.scratchA + (size_t)4 * b0 * f.cap,
                                            f.keepA + (size_t)2 * b0 * f.cap, f.countsA + 2 * b0, f.passesA + 64 * b0,
                                            f.npassesA + 2 * b0, f.croppedA + 2 * b0));
      }
      DL_TRY(launch_gather_rows(ctx, f.returns_tracking + (size_t)b0 * f.cap * 3, f.cap, 2, f.keepA + (size_t)2 * b0 * f.cap,
                                f.countsA + 2 * b0, f.cap, f.clouds + (size_t)2 * b0 * f.cap * 3, 2 * nb));
      DL_TRY(launch_initial_pose(ctx, nb, f.current_pose + 7 * b0, f.submap_inverse + b0, f.initial_pose + 7 * b0, f.target + 3 * b0));
      if (rtcsm) {
        // The angular window depends on the farthest point of each cloud through acosf, which must be the host's to stay
        // bit-exact: ONE synchronisation per batch brings back the clouds' sizes, farthest points and initial poses; the
        // candidate tables of all scans then go up in one copy and one launch scores every (scan, rotation, translation),
        // each scan against its own matching submap's high-resolution grid. The best poses are written into f.initial_pose on
        // the device, where the solve reads them (the fused solve takes them as the pose part of state j's initial value);
        // f.target keeps the prediction's translation (LTB:536).
        std::vector<int32_t> countsA(2 * f.batch);
        std::vector<double> init(7 * f.batch);
        std::vector<float> far(f.batch);
        float* d_far = a.take<float>(f.batch);
        DL_TRY(launch_max_range_batch(ctx, f.clouds, (int64_t)2 * f.cap * 3, f.countsA, 2, f.batch, 3.f * hi_resolution, d_far));
        DL_TRY(d2h(ctx, countsA.data(), f.countsA, 2 * f.batch));
        DL_TRY(d2h(ctx, init.data(), f.initial_pose, 7 * f.batch));
        DL_TRY(d2h(ctx, far.data(), d_far, f.batch));
        DL_TRY(sync(ctx));
        StageScope st(ctx, "rtcsm");
        std::vector<RtcsmBatchItem> items;
        std::vector<int32_t> slots;
        for (int b = 0; b < f.batch; ++b) {
          if (countsA[2 * b] <= 0) continue;
          items.push_back(RtcsmBatchItem{submaps.high(b), f.clouds + (size_t)(2 * b) * f.cap * 3, countsA[2 * b],
                                         pose_from7(init.data() + 7 * b), far[b], nullptr, f.rtcsm_nonpositive + b});
          slots.push_back(b);
        }
        DL_CUDA(ctx, cudaMemsetAsync(f.rtcsm_scores, 0, sizeof(float) * f.batch, ctx->stream));
        DL_CUDA(ctx, cudaMemsetAsync(f.rtcsm_nonpositive, 0, sizeof(int32_t) * f.batch, ctx->stream));
        if (!items.empty()) {
          RtcsmBatchPlan plan;
          DL_TRY(plan_rtcsm_batch(ctx, o.real_time_correlative_scan_matcher, hi_resolution, items, &plan));
          plan.take(a);
          if (a.off > ctx->d_scratch.cap) return ctx->fail(DL_ERR_ARG, "internal: RT-CSM scratch underestimated");
          DL_TRY(run_rtcsm_batch(ctx, items, plan));
          int32_t* d_slots = a.take<int32_t>(items.size());
          DL_TRY(h2d(ctx, d_slots, slots.data(), slots.size()));
          DL_TRY(launch_rtcsm_pick(ctx, plan.d_scans, (int)items.size(), f.initial_pose, d_slots, f.rtcsm_scores, d_slots));
          DL_TRY(sync(ctx));  // `slots` is pageable and local
        }
        have_scores = true;
      }
      {
        StageScope st(ctx, "nls_solve");
        NlsOptions no = to_nls_options(o.ceres_scan_matcher, 2);
        no.cluster = solve_cluster_size(ctx, o, nb);
        if (imu || raw)  // pose part of the initial state comes from problems[].initial_dev like the plain solve's
          DL_TRY(launch_nls_fused(ctx, no, f.problems + b0, m.d_terms + b0, m.d_init16 + 16 * b0, nb, m.d_fused + b0));
        else
          DL_TRY(launch_nls(ctx, no, f.problems + b0, nb, f.nls_out + b0));
      }
      ResultArgs ra{};
      ra.batch = nb; ra.first_counts = f.n1 + b0; ra.return_counts = f.n2 + b0; ra.miss_counts = f.n3 + b0;
      ra.adaptive_counts = f.countsA + 2 * b0; ra.adaptive_cropped = f.croppedA + 2 * b0; ra.adaptive_passes = f.npassesA + 2 * b0;
      ra.rtcsm_scores = have_scores ? f.rtcsm_scores + b0 : nullptr; ra.nls = f.nls_out + b0; ra.fused = (imu || raw) ? m.d_fused + b0 : nullptr; ra.submap = f.submap + b0;
      ra.results = d_results + b0; ra.error_flag = f.error_flag + b0;
      ra.imu_ok = m.d_ok ? m.d_ok + b0 : nullptr; ra.states_out = m.d_states ? m.d_states + b0 : nullptr;
      DL_TRY(launch_finalize_results(ctx, ra));
      return DL_OK;
    };
    status = run();
  }
  ctx->stream = main_stream;
  if (imu_ready) ctx->event_pool.push_back(imu_ready);
  if (chunks > 1) {  // later work on the main stream (result copies, the next call) waits for the other stream
    cudaEvent_t joined = ctx->take_event();
    DL_CUDA(ctx, cudaEventRecord(joined, ctx->aux_stream));
    DL_CUDA(ctx, cudaStreamWaitEvent(main_stream, joined, 0));
    ctx->event_pool.push_back(joined);
  }
  return status;
}

int check_frontend(dl_context* ctx, const dl_frontend_options* o, int num_scans, const int64_t* sizes,
                   const SubmapSet& submaps, int64_t* max_size) {
  if (!o || num_scans < 0 || !submaps.hi || !submaps.lo || (num_scans > 0 && !sizes)) return DL_ERR_ARG;
  for (int b = 0; b < (submaps.per_scan ? num_scans : 1); ++b) {
    if (!submaps.high(b) || !submaps.low(b)) return DL_ERR_ARG;
    if (submaps.high(b)->structure_dirty || submaps.low(b)->structure_dirty)
      return ctx->fail(DL_ERR_ARG, "dl_grid_sync not called after dl_grid_set_cells");
    // the pre-match's candidate tables and the 3 * resolution floor of the farthest point take one resolution per batch
    if (o->use_online_correlative_scan_matching && submaps.high(b)->resolution != submaps.high(0)->resolution)
      return ctx->fail(DL_ERR_ARG, "the correlative pre-match takes one high-resolution grid resolution per batch");
  }
  DL_TRY(check_ceres_options(ctx, &o->ceres_scan_matcher, 2));
  int64_t m = 0;
  for (int b = 0; b < num_scans; ++b) {
    if (sizes[b] < 0 || sizes[b] > 0x3fffffff) return ctx->fail(DL_ERR_ARG, "scan size out of range");
    m = std::max(m, sizes[b]);
  }
  *max_size = m;
  if (o->range_row_floats == 3 && num_scans > 0) {
    if (!o->time_run_offsets || !o->time_run_first_row || !o->time_run_value)
      return ctx->fail(DL_ERR_ARG, "range_row_floats = 3 needs the time_run_* arrays");
    if (o->time_run_offsets[0] != 0) return ctx->fail(DL_ERR_ARG, "time_run_offsets[0] must be 0");
    for (int b = 0; b < num_scans; ++b) {
      const int32_t r0 = o->time_run_offsets[b], r1 = o->time_run_offsets[b + 1];
      if (r1 < r0 || (sizes[b] > 0 && r1 == r0)) return ctx->fail(DL_ERR_ARG, "every non-empty scan needs at least one time run");
      // O(scans) checks only (this runs on the issue path of every batch): first run at row 0, last run inside the scan. The
      // kernels clamp every run to its scan, so a table that does not ascend gives wrong times, never a wild access.
      if (r1 > r0 && (o->time_run_first_row[r0] != 0 || o->time_run_first_row[r1 - 1] >= std::max<int64_t>(sizes[b], 1) ||
                      o->time_run_first_row[r1 - 1] < 0))
        return ctx->fail(DL_ERR_ARG, "time_run_first_row must start at 0 and stay inside the scan");
    }
  }
  return DL_OK;
}

}  // namespace

namespace dl {

int frontend_enqueue(dl_context* ctx, const dl_frontend_options* options, int num_scans, const FrontendScans& in,
                     const int64_t* sizes, const float* origins, int num_origins, const double* prev_poses,
                     const double* predicted_poses, const SubmapSet& submaps, dl_scan_result** d_results_out, ImuRun* imu,
                     FrontendBuffers* buffers_out, const int32_t* origin_base, const std::function<void(Arena&)>* more) {
  int64_t max_size = 0;
  DL_TRY(check_frontend(ctx, options, num_scans, sizes, submaps, &max_size));
  if (num_scans == 0) return DL_OK;
  const bool raw = imu && imu->samples;
  if (!origins || num_origins < 1 || (!raw && (!prev_poses || !predicted_poses)) || !submaps.poses) return DL_ERR_ARG;
  if (in.on_device) {
    if (!in.dev || !in.results_dev || (imu && !imu->d_states_out) || in.cap_rows < max_size || in.cap_rows < 1) return DL_ERR_ARG;
  } else {
    if (!in.host) return DL_ERR_ARG;
    for (int b = 0; b < num_scans; ++b)
      if (sizes[b] > 0 && !in.host[b]) return DL_ERR_ARG;
    if (options->host_scan_stride_rows != 0) {
      const int64_t stride = options->host_scan_stride_rows;
      const size_t row_bytes = (size_t)row_floats_of(*options) * 4;
      if (stride < max_size) return ctx->fail(DL_ERR_ARG, "host_scan_stride_rows is smaller than a scan");
      for (int b = 0; b < num_scans; ++b)
        if ((const char*)in.host[b] != (const char*)in.host[0] + (size_t)b * stride * row_bytes)
          return ctx->fail(DL_ERR_ARG, "host_scan_stride_rows does not describe the ranges pointers");
    }
  }
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  const int64_t cap = in.on_device ? in.cap_rows : std::max<int64_t>(max_size, 1);
  // The correlative pre-match takes its candidate tables after the carve (see rtcsm_scratch_bound).
  const size_t rtcsm_extra = options->use_online_correlative_scan_matching
      ? (size_t)num_scans * rtcsm_scratch_bound(options->real_time_correlative_scan_matcher, submaps.high(0)->resolution,
                                                options->high_resolution_adaptive_voxel_filter.max_range)
      : 0;
  float* d_ranges;
  dl_scan_result* d_results;
  FrontendBuffers f;
  Arena rest(nullptr);
  DL_TRY(carve_scratch(ctx, [&](Arena& a) {
    d_ranges = in.on_device ? (float*)in.dev : a.take<float>((size_t)num_scans * cap * 8);
    d_results = in.on_device ? in.results_dev : a.take<dl_scan_result>(num_scans);
    carve(a, num_scans, cap, num_origins, &f);
    if (imu) carve_imu(a, num_scans, imu);
    carve_time_runs(a, *options, num_scans, &f);
    if (more) (*more)(a);
    carve_prematch(a, *options, num_scans, &f);
  }, rtcsm_extra, &rest));
  if (d_results_out) *d_results_out = d_results;
  if (buffers_out) *buffers_out = f;
  return frontend_run(ctx, *options, num_scans, d_ranges, cap, in.host, sizes, origins, num_origins, origin_base, prev_poses,
                      predicted_poses, submaps, f, rest, d_results, imu);
}

int check_imu_options(dl_context* ctx, const dl_frontend_options* options) {
  if (options && options->ceres_scan_matcher.only_optimize_yaw)
    return ctx->fail(DL_ERR_ARG, "only_optimize_yaw is not supported by the fused solve");
  return DL_OK;
}

int check_imu_samples(dl_context* ctx, const dl_frontend_options* options, const dl_frontend_imu_samples* imu, int num_scans) {
  if (!imu || num_scans < 0) return DL_ERR_ARG;
  if (num_scans == 0) return DL_OK;
  if (!imu->states_i || !imu->offsets || !(imu->imu_weight >= 0.)) return DL_ERR_ARG;
  if (imu->offsets[0] != 0) return ctx->fail(DL_ERR_ARG, "offsets[0] must be 0");
  for (int k = 0; k < num_scans; ++k)
    if (imu->offsets[k + 1] < imu->offsets[k]) return ctx->fail(DL_ERR_ARG, "offsets must be non-decreasing");
  if (imu->offsets[num_scans] > 0 && (!imu->dt || !imu->acc || !imu->gyr)) return DL_ERR_ARG;
  return check_imu_options(ctx, options);
}

}  // namespace dl

extern "C" {

int dl_frontend_match_batch_dev(dl_context* ctx, const dl_frontend_options* options, int32_t num_scans,
                                const void* ranges_dev, int64_t cap_rows, const int64_t* sizes, const float* origins,
                                int32_t num_origins, const double* prev_poses, const double* predicted_poses,
                                const double* submap_local_pose, const dl_grid* hi, const dl_grid* lo,
                                dl_scan_result* results_dev) {
  if (!ctx) return DL_ERR_ARG;
  FrontendScans in;
  in.on_device = true;
  in.dev = ranges_dev;
  in.cap_rows = cap_rows;
  in.results_dev = results_dev;
  return frontend_enqueue(ctx, options, num_scans, in, sizes, origins, num_origins, prev_poses, predicted_poses,
                          OneSubmap(submap_local_pose, hi, lo), nullptr);
}

int dl_frontend_fetch_results(dl_context* ctx, const dl_scan_result* results_dev, int32_t num_scans,
                              dl_scan_result* results) {
  if (!ctx || num_scans < 0 || (num_scans > 0 && (!results_dev || !results))) return DL_ERR_ARG;
  DL_TRY(d2h(ctx, results, results_dev, num_scans));
  return sync(ctx);
}

int dl_frontend_match_batch(dl_context* ctx, const dl_frontend_options* options, int32_t num_scans,
                            const void* const* ranges, const int64_t* sizes, const float* origins, int32_t num_origins,
                            const double* prev_poses, const double* predicted_poses, const double* submap_local_pose,
                            const dl_grid* hi, const dl_grid* lo, dl_scan_result* results) {
  if (!ctx) return DL_ERR_ARG;
  if (num_scans == 0) {
    int64_t m = 0;
    return check_frontend(ctx, options, num_scans, sizes, OneSubmap(submap_local_pose, hi, lo), &m);
  }
  if (!results) return DL_ERR_ARG;
  dl_scan_result* d_results = nullptr;
  DL_TRY(frontend_enqueue(ctx, options, num_scans, FrontendScans{ranges}, sizes, origins, num_origins, prev_poses, predicted_poses,
                          OneSubmap(submap_local_pose, hi, lo), &d_results));
  DL_TRY(d2h(ctx, results, d_results, num_scans));
  return sync(ctx);
}

int dl_frontend_match_batch_imu(dl_context* ctx, const dl_frontend_options* options, const dl_frontend_imu* imu,
                                int32_t num_scans, const void* const* ranges, const int64_t* sizes, const float* origins,
                                int32_t num_origins, const double* submap_local_pose, const dl_grid* hi, const dl_grid* lo,
                                dl_scan_result* results) {
  if (!ctx || !imu) return DL_ERR_ARG;
  if (num_scans == 0) return DL_OK;
  if (num_scans < 0 || !results || !imu->states_i || !imu->predicted_states || !imu->preintegrations || !imu->states_out ||
      !(imu->imu_weight >= 0.))
    return DL_ERR_ARG;
  DL_TRY(check_imu_options(ctx, options));
  std::vector<double> prev((size_t)num_scans * 7), pred((size_t)num_scans * 7);
  for (int b = 0; b < num_scans; ++b) {
    const dl_nav_state& si = imu->states_i[b];
    const dl_nav_state& sj = imu->predicted_states[b];
    for (int k = 0; k < 3; ++k) { prev[7 * b + k] = si.p[k]; pred[7 * b + k] = sj.p[k]; }
    for (int k = 0; k < 4; ++k) { prev[7 * b + 3 + k] = si.q[k]; pred[7 * b + 3 + k] = sj.q[k]; }
  }
  dl_scan_result* d_results = nullptr;
  ImuRun run;
  run.host = imu;
  DL_TRY(frontend_enqueue(ctx, options, num_scans, FrontendScans{ranges}, sizes, origins, num_origins, prev.data(), pred.data(),
                          OneSubmap(submap_local_pose, hi, lo), &d_results, &run));
  DL_TRY(d2h(ctx, results, d_results, num_scans));
  DL_TRY(d2h(ctx, imu->states_out, run.d_states, num_scans));
  return sync(ctx);
}

int dl_frontend_match_batch_imu_samples(dl_context* ctx, const dl_frontend_options* options, const dl_frontend_imu_samples* imu,
                                        int32_t num_scans, const void* const* ranges, const int64_t* sizes, const float* origins,
                                        int32_t num_origins, const double* submap_local_pose, const dl_grid* hi,
                                        const dl_grid* lo, dl_scan_result* results, dl_nav_state* states_out,
                                        dl_nav_state* predicted_states_out) {
  if (!ctx) return DL_ERR_ARG;
  DL_TRY(check_imu_samples(ctx, options, imu, num_scans));
  if (num_scans == 0) return DL_OK;
  if (!results || !states_out) return DL_ERR_ARG;
  dl_scan_result* d_results = nullptr;
  ImuRun run;
  run.samples = imu;
  DL_TRY(frontend_enqueue(ctx, options, num_scans, FrontendScans{ranges}, sizes, origins, num_origins, nullptr, nullptr,
                          OneSubmap(submap_local_pose, hi, lo), &d_results, &run));
  DL_TRY(d2h(ctx, results, d_results, num_scans));
  DL_TRY(d2h(ctx, states_out, run.d_states, num_scans));
  if (predicted_states_out) DL_TRY(d2h(ctx, predicted_states_out, run.d_predicted, num_scans));
  return sync(ctx);
}

int dl_frontend_match_batch_imu_samples_dev(dl_context* ctx, const dl_frontend_options* options,
                                            const dl_frontend_imu_samples* imu, int32_t num_scans, const void* ranges_dev,
                                            int64_t cap_rows, const int64_t* sizes, const float* origins, int32_t num_origins,
                                            const double* submap_local_pose, const dl_grid* hi, const dl_grid* lo,
                                            dl_scan_result* results_dev, dl_nav_state* states_out_dev) {
  if (!ctx) return DL_ERR_ARG;
  DL_TRY(check_imu_samples(ctx, options, imu, num_scans));
  FrontendScans in;
  in.on_device = true;
  in.dev = ranges_dev;
  in.cap_rows = cap_rows;
  in.results_dev = results_dev;
  ImuRun run;
  run.samples = imu;
  run.d_states_out = states_out_dev;
  return frontend_enqueue(ctx, options, num_scans, in, sizes, origins, num_origins, nullptr, nullptr, OneSubmap(submap_local_pose, hi, lo),
                          nullptr, &run);
}

// Tail of a submit: the results (and, with the IMU, the estimated states) go to pinned staging behind the batch.
static int submit_finish(dl_context* ctx, int num_scans, int num_origins, const dl_scan_result* d_results,
                         const dl_nav_state* d_states) {
  Staging s;
  Arena h(ctx->h_pinned.get());  // the block frontend_upload_small reserved for this batch
  carve_staging(h, num_scans, num_origins, &s);
  DL_CUDA(ctx, cudaMemcpyAsync(s.results, d_results, (size_t)num_scans * sizeof(dl_scan_result), cudaMemcpyDeviceToHost,
                               ctx->stream));
  if (d_states)
    DL_CUDA(ctx, cudaMemcpyAsync(s.states, d_states, (size_t)num_scans * sizeof(dl_nav_state), cudaMemcpyDeviceToHost, ctx->stream));
  DL_CUDA(ctx, cudaEventRecord(ctx->batch_done, ctx->stream));
  ctx->in_flight = num_scans;
  ctx->in_flight_states = d_states != nullptr;
  ctx->staged_results = s.results;
  ctx->staged_states = s.states;
  return DL_OK;
}

int dl_frontend_submit(dl_context* ctx, const dl_frontend_options* options, int32_t num_scans, const void* const* ranges,
                       const int64_t* sizes, const float* origins, int32_t num_origins, const double* prev_poses,
                       const double* predicted_poses, const double* submap_local_pose, const dl_grid* hi, const dl_grid* lo) {
  if (!ctx || num_scans < 1) return DL_ERR_ARG;
  if (ctx->in_flight) return ctx->fail(DL_ERR_ARG, "a submitted batch is already in flight on this context");
  dl_scan_result* d_results = nullptr;
  DL_TRY(frontend_enqueue(ctx, options, num_scans, FrontendScans{ranges}, sizes, origins, num_origins, prev_poses, predicted_poses,
                          OneSubmap(submap_local_pose, hi, lo), &d_results));
  return submit_finish(ctx, num_scans, num_origins, d_results, nullptr);
}

int dl_frontend_submit_imu_samples(dl_context* ctx, const dl_frontend_options* options, const dl_frontend_imu_samples* imu,
                                   int32_t num_scans, const void* const* ranges, const int64_t* sizes, const float* origins,
                                   int32_t num_origins, const double* submap_local_pose, const dl_grid* hi, const dl_grid* lo) {
  if (!ctx || num_scans < 1) return DL_ERR_ARG;
  if (ctx->in_flight) return ctx->fail(DL_ERR_ARG, "a submitted batch is already in flight on this context");
  DL_TRY(check_imu_samples(ctx, options, imu, num_scans));
  dl_scan_result* d_results = nullptr;
  ImuRun run;
  run.samples = imu;
  DL_TRY(frontend_enqueue(ctx, options, num_scans, FrontendScans{ranges}, sizes, origins, num_origins, nullptr, nullptr, OneSubmap(submap_local_pose, hi, lo), &d_results, &run));
  return submit_finish(ctx, num_scans, num_origins, d_results, run.d_states);
}

static int collect_common(dl_context* ctx, int32_t num_scans, dl_scan_result* results, dl_nav_state* states_out) {
  if (!ctx || !results) return DL_ERR_ARG;
  if (!ctx->in_flight) return ctx->fail(DL_ERR_ARG, "no submitted batch on this context");
  if (num_scans != ctx->in_flight) return ctx->fail(DL_ERR_ARG, "num_scans differs from the submitted batch");
  if (states_out && !ctx->in_flight_states) return ctx->fail(DL_ERR_ARG, "the submitted batch carries no IMU states");
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  const cudaError_t e = cudaEventSynchronize(ctx->batch_done);
  ctx->in_flight = 0;
  if (e != cudaSuccess) return ctx->cuda_fail(e, "dl_frontend_collect");
  std::memcpy(results, ctx->staged_results, (size_t)num_scans * sizeof(dl_scan_result));
  if (states_out) std::memcpy(states_out, ctx->staged_states, (size_t)num_scans * sizeof(dl_nav_state));
  return DL_OK;
}
int dl_frontend_collect(dl_context* ctx, int32_t num_scans, dl_scan_result* results) {
  return collect_common(ctx, num_scans, results, nullptr);
}
int dl_frontend_collect_imu(dl_context* ctx, int32_t num_scans, dl_scan_result* results, dl_nav_state* states_out) {
  if (!states_out) return DL_ERR_ARG;
  return collect_common(ctx, num_scans, results, states_out);
}

int dl_ingest_scan(dl_context* ctx, const dl_frontend_options* options, const void* ranges, int64_t n,
                   const float* origins, int32_t num_origins, const double* prev_pose, const double* predicted_pose,
                   int64_t* first_keep_out, float* returns_local_out, float* returns_tracking_out,
                   float* misses_tracking_out, float* current_pose7f_out, int64_t* counts_out) {
  if (!ctx || !options || !ranges || n < 1 || n > 0x3fffffff || !origins || num_origins < 1 || !prev_pose || !predicted_pose ||
      !counts_out)
    return DL_ERR_ARG;
  if (row_floats_of(*options) != 8) return ctx->fail(DL_ERR_ARG, "dl_ingest_scan takes RangeMeasurement rows (range_row_floats = 8)");
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  float* d_ranges;
  FrontendBuffers f;
  DL_TRY(carve_scratch(ctx, [&](Arena& a) {
    d_ranges = a.take<float>((size_t)n * 8);
    carve(a, 1, n, num_origins, &f);
  }));
  DL_TRY(h2d(ctx, d_ranges, (const float*)ranges, (size_t)n * 8));
  DL_TRY(frontend_upload_small(ctx, *options, f, &n, origins, num_origins, prev_pose, predicted_pose, nullptr, nullptr));
  // fe_ingest_tile writes the local record of a return or a miss only: zeroed records read as class 0 for every other row
  DL_CUDA(ctx, cudaMemsetAsync(f.local4, 0, (size_t)n * 4 * sizeof(float), ctx->stream));
  const FrontendArgs fa = make_frontend_args(*options, f, d_ranges, n, 8);
  DL_TRY(launch_fe_prepare(ctx, fa, 1));
  DL_TRY(launch_fe_first_filter(ctx, fa, 0, 1));
  DL_TRY(launch_fe_rest(ctx, fa, 0, 1));
  int32_t c[4], error_flag;
  DL_TRY(d2h(ctx, &c[0], f.n1, 1));
  DL_TRY(d2h(ctx, &c[1], f.n_ret, 1));
  DL_TRY(d2h(ctx, &c[2], f.n2, 1));
  DL_TRY(d2h(ctx, &c[3], f.n3, 1));
  DL_TRY(d2h(ctx, &error_flag, f.error_flag, 1));
  std::vector<uint32_t> first_bits(f.bit_words);
  DL_TRY(d2h(ctx, first_bits.data(), f.first_bits, first_bits.size()));
  std::vector<float> local(returns_local_out ? (size_t)n * 4 : 0);  // float4 per row: local-frame point, class in .w
  DL_TRY(d2h(ctx, local.data(), f.local4, local.size()));
  DL_TRY(sync(ctx));
  for (int i = 0; i < 4; ++i) counts_out[i] = c[i];
  if (error_flag)
    return ctx->fail(DL_ERR_ARG, "a point lies outside the voxel-key span of the second voxel filter (dl_scan_result.ok = -1)");
  if (returns_tracking_out) DL_TRY(d2h(ctx, returns_tracking_out, f.returns_tracking, (size_t)c[2] * 3));
  if (misses_tracking_out) DL_TRY(d2h(ctx, misses_tracking_out, f.misses_tracking, (size_t)c[3] * 3));
  if (current_pose7f_out) DL_TRY(d2h(ctx, current_pose7f_out, f.current_pose, 7));
  DL_TRY(sync(ctx));
  // first_keep: the rows of the first filter's bitmap in index order; returns_local: those of them in class 1 (a return)
  int64_t kept = 0, returns = 0;
  for (int64_t i = 0; i < n; ++i) {
    if (!(first_bits[i >> 5] >> (i & 31) & 1u)) continue;
    if (first_keep_out) first_keep_out[kept++] = i;
    if (!returns_local_out) continue;
    int32_t cls;
    std::memcpy(&cls, &local[4 * i + 3], sizeof(cls));
    if (cls == 1) std::memcpy(returns_local_out + 3 * returns++, &local[4 * i], 3 * sizeof(float));
  }
  return DL_OK;
}

}  // extern "C"
