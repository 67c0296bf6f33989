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
