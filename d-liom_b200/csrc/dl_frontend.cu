// Fused scan front half for the batched front end: 4 launches per sub-batch (5 with per-run deskew poses) instead of the 11 of the stage-wise path
// (dl_voxel.cu + dl_ingest.cu, which stay as the standalone filter API and as a cross-check in the tests).
//
//   A  fe_first_filter_insert   first voxel filter (LTB:393-395): every point proposes its index for its voxel
//                               (atomicCAS claim + atomicMin), one 128-bit load per point.
//   B0 fe_run_poses             12-byte rows with the point times as runs: the deskew pose (fp64 slerp + composition, LTB:430-445) once
//                               per RUN instead of once per survivor; kernel B then loads the finished Rigid3f.
//   B  fe_ingest_second_insert  for each first-filter survivor: deskew + transform + range gate (LTB:426-472) and
//                               immediately the SECOND voxel filter's insert (LTB:479-484) keyed on the local-frame
//                               voxel — no compaction in between: ids stay the original input indices, which
//                               preserves "first point in input order wins" for free.
//   C1 fe_mark_bits             the second filter's winners (the index field of every non-empty slot) become bits of two
//                               per-scan bitmaps (returns, misses): 4 KiB per 32 k points, L2-resident.
//   C2 fe_emit_tracking         ordered compaction straight from the bitmaps (popcount prefix; no per-point class map, no
//                               tile counts), fused with the scan's current pose (hits_poses.back(), LTB:476) and the frame
//                               change back to tracking (TransformRangeData with current_pose^-1, LTB:485-487); output rows
//                               are written coalesced.
//
// The second filter's table has ONE 64-bit word per slot: [miss | voxel key relative to the scan's pose | point index]. The
// key sits above the index, so for equal keys atomicMin keeps the lowest index ("first point in input order", voxel_filter.cc:
// 81-131) and a slot's key never changes once claimed: a collision compares keys inside the word, never reads another thread's
// point, and a survivor touches one 8-byte slot (round 1: an 8-byte key slot + a 4-byte min slot). The key holds 3 x axis_bits
// (axis_bits = min(21, (63 - index_bits) / 3): 15 bits for scans up to 256 k points) of the voxel index RELATIVE to the voxel of
// the scan's predicted pose: every output point lies within max_range of the (moving) sensor origin, so the reachable span is
// 2 max_range / voxel_filter_size cells — +-2.4 km at 0.15 m. A point outside it sets the scan's error flag and the scan's
// result is invalid (ok = -1); the generic dl_voxel_filter has no such limit. Returns and misses share the table (bit 63).
//
// Algorithmic traffic per raw point: A reads 12/16 B; B reads 4 B slot (+12/16 B row + 4 B time, writes 16 B record + 8 B slot
// for survivors); C1 reads 8 B per slot; C2 reads 16 B and writes 12 B per output point.
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

// 12-byte rows: index (into the batch's run arrays) of the time run that contains row i of scan b. A binary search of the scan's
// ~2 k run starts (L1-resident) per survivor: expanding the run index of every row once per batch (4 B per row, one more kernel
// and 17 MB of writes per step) made the ingest kernel faster but the step slower.
__device__ __forceinline__ int run_index(const FrontendArgs& a, int b, int i) {
  int lo = a.run_offsets[b], hi = a.run_offsets[b + 1] - 1;  // last run whose first row is <= i
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(a.run_first_row + mid) <= i) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// Time of row i of scan b: the row's fourth float, or (12-byte rows) the value of the run that contains the row.
__device__ __forceinline__ float point_time(const FrontendArgs& a, int b, const float* __restrict__ rows, int rf, int i) {
  if (rf != 3) return rows[(size_t)i * rf + 3];
  return a.run_value[run_index(a, b, i)];
}

// ---------------------------------------------------------------------------------------------------- A
// One point in flight per thread: the kernel runs at the L2's atomic throughput, and 2 or 4 points per thread (more outstanding
// atomics) measured slower because they only lengthen the L2 queues.
__global__ void __launch_bounds__(kBlock, 8) fe_first_filter_insert(FrontendArgs a) {
  const int b = a.first_scan + blockIdx.y;
  const int n = a.counts[b];
  const float* rows = a.ranges + (size_t)b * a.in_cap * a.row_floats;
  uint32_t* tab = a.table1 + (size_t)b * a.tcap1;
  const uint32_t tcap = (uint32_t)a.tcap1;  // any size (not a power of two): slot = hash * tcap >> 32
  const CellDivider res = make_divider(a.first_resolution);
  const int stride = gridDim.x * kBlock;
  for (int i = blockIdx.x * kBlock + threadIdx.x; i < n; i += stride) {
    const Int3 c = cell_index(load_xyz(rows, a.row_floats, i), res);
    uint32_t hh = table_slot(hash_cell(c), tcap);
    uint32_t p = atomicCAS(tab + hh, kEmpty32, (uint32_t)i);
    while (p != kEmpty32) {  // the slot has an owner: same voxel -> the lower index stays; else probe on
      const Int3 o = cell_index(load_xyz(rows, a.row_floats, p), res);
      if (o.x == c.x && o.y == c.y && o.z == c.z) {
        if ((uint32_t)i < p) atomicMin(tab + hh, (uint32_t)i);  // the owner only ever decreases
        break;
      }
      hh = hh + 1 == tcap ? 0u : hh + 1;
      p = atomicCAS(tab + hh, kEmpty32, (uint32_t)i);
    }
  }
}

// ---------------------------------------------------------------------------------------------------- B
__device__ __forceinline__ Rigidd interpolate_pose(double s, const ScanConstants& c) {
  double scale0, scale1;
  if (c.linear_slerp) {
    scale0 = 1.0 - s;
    scale1 = s;
  } else {
    scale0 = sin((1.0 - s) * c.theta) / c.sin_theta;
    scale1 = sin(s * c.theta) / c.sin_theta;
  }
  if (c.negative_dot) scale1 = -scale1;
  Rigidd out;
  out.q = {scale0 * 1.0 + scale1 * c.rel.q.w, scale0 * 0.0 + scale1 * c.rel.q.x, scale0 * 0.0 + scale1 * c.rel.q.y,
           scale0 * 0.0 + scale1 * c.rel.q.z};
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

// Heavy per-survivor work of kernel B (double slerp, pose composition, transform, gate, second-filter insert).
template <bool kRunPose>
__device__ __forceinline__ int ingest_survivor(const FrontendArgs& a, int b, const float* rows, int rf, const ScanConstants& sc,
                                               bool no_deskew, const KeyLayout& kl, unsigned long long* slots, uint32_t mask2, int i) {
  float4 h;
  Rigidf pose;
  if (kRunPose) {  // 12-byte rows, per-run pose table
    const float* p = rows + (size_t)i * 3;
    h = make_float4(p[0], p[1], p[2], 0.f);
    const float4* rp = (const float4*)(a.run_pose + (size_t)8 * run_index(a, b, i));
    const float4 p0 = __ldg(rp), p1 = __ldg(rp + 1);
    pose = Rigidf{{p0.x, p0.y, p0.z}, {p0.w, p1.x, p1.y, p1.z}};
  } else if (rf == 3) {
    const float* p = rows + (size_t)i * 3;
    h = make_float4(p[0], p[1], p[2], point_time(a, b, rows, rf, i));
  } else {
    h = __ldg((const float4*)(rows + (size_t)i * rf));
  }
  const unsigned long long origin_index = rf >= 8 ? *(const unsigned long long*)(rows + (size_t)i * rf + 4) : 0ull;
  const float* o = a.origins + 3 * origin_index;
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
    // one aligned 16-byte record per survivor: local-frame point (+ class in .w, for debugging only)
    ((float4*)a.local)[(size_t)b * a.cap + i] = make_float4(outp.x, outp.y, outp.z, __int_as_float(cls));
    const Int3 c = cell_index(outp, make_divider(a.second_resolution));
    unsigned long long slot;
    if (!pack_slot(kl, c, cls == 2, (uint32_t)i, &slot)) {
      a.error_flag[b] = 1;  // per scan: only this scan's result is invalidated
      cls = 0;
    } else {
      uint32_t hh = (hash_cell(c) ^ (cls == 2 ? 0x9e3779b9u : 0u)) & mask2;
      for (;;) {
        const unsigned long long prev = atomicCAS(slots + hh, kEmpty64, slot);
        if (prev == kEmpty64) break;
        if ((prev >> kl.idx_bits) == (slot >> kl.idx_bits)) {  // same class and voxel: the lowest index stays
          if (slot < prev) atomicMin(slots + hh, slot);
          break;
        }
        hh = (hh + 1) & mask2;
      }
    }
  }
  return cls;
}

// Only ~30 % of the raw points survive the first filter, so running the heavy path under the survivor predicate
// would leave most lanes idle. Each warp instead appends its survivors to a small shared-memory queue and drains
// it 32 at a time with all lanes busy.
template <bool kRunPose>
__global__ void __launch_bounds__(kBlock, kRunPose ? 6 : 4) fe_ingest_second_insert(FrontendArgs a) {  // <= 40 / 64 registers
  __shared__ int queue[kBlock / 32][64];
  const int b = a.first_scan + blockIdx.y;
  const int n = a.counts[b];
  const int rf = a.row_floats;
  const float* rows = a.ranges + (size_t)b * a.in_cap * rf;
  const uint32_t* tab = a.table1 + (size_t)b * a.tcap1;
  unsigned long long* slots = a.slots2 + (size_t)b * a.tcap2;
  const uint32_t mask2 = (uint32_t)a.tcap2 - 1;
  const ScanConstants& sc = a.scans[b];
  const KeyLayout kl = key_layout(a, sc);
  const bool no_deskew = n > 0 && (double)fabsf(point_time(a, b, rows, rf, 0)) < 1e-3;  // first survivor is row 0 (LTB:430-433)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int* q = queue[warp];
  int queued = 0, survivors = 0, returns = 0, last = -1;
  // The first filter's survivors are exactly the non-empty table slots: stream the table (coalesced) instead of
  // probing it once per raw point. Order does not matter here: the second filter keys on the original index.
  if (n == 0) return;
  // (four slots per thread and step through one 16-byte load: same kernel time in the serial launch list, slightly slower in the
  //  overlapped step, so the stream stays one slot per thread)
  for (int h = blockIdx.x * kBlock + threadIdx.x; h < (int)a.tcap1; h += gridDim.x * kBlock) {
    const uint32_t owner = __ldcg(tab + h);
    const bool surv = owner != kEmpty32;
    const unsigned ballot = __ballot_sync(0xffffffffu, surv);
    if (surv) {
      q[queued + __popc(ballot & ((1u << lane) - 1))] = (int)owner;
      last = max(last, (int)owner);
    }
    queued += __popc(ballot);
    survivors += surv;
    __syncwarp();
    if (queued >= 32) {
      returns += ingest_survivor<kRunPose>(a, b, rows, rf, sc, no_deskew, kl, slots, mask2, q[lane]) == 1;
      __syncwarp();
      const int rest = queued - 32;
      const int moved = lane < rest ? q[32 + lane] : 0;
      __syncwarp();
      if (lane < rest) q[lane] = moved;
      queued = rest;
      __syncwarp();
    }
  }
  if (lane < queued) returns += ingest_survivor<kRunPose>(a, b, rows, rf, sc, no_deskew, kl, slots, mask2, q[lane]) == 1;
  // bookkeeping: survivor counts and the LAST first-filter survivor (hits_poses.back(), LTB:476)
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    survivors += __shfl_xor_sync(0xffffffffu, survivors, d);
    returns += __shfl_xor_sync(0xffffffffu, returns, d);
    last = max(last, __shfl_xor_sync(0xffffffffu, last, d));
  }
  if (lane == 0) {
    if (survivors) atomicAdd(a.n_first + b, survivors);
    if (returns) atomicAdd(a.n_returns_local + b, returns);
    if (last >= 0) atomicMax(a.last_index + b, last);
  }
}

// ---------------------------------------------------------------------------------------------------- C
constexpr int kEmitBlock = 512, kEmitWarps = kEmitBlock / 32;
constexpr int kChunkPoints = 1024;  // one warp handles 32 bitmap words = 1024 consecutive point indices at a time

__device__ __forceinline__ uint32_t* scan_bits(const FrontendArgs& a, int b, int miss) {
  return a.bits + ((size_t)b * 2 + miss) * a.bit_words;
}

// C1: the second filter's survivors are the index fields of its non-empty slots: stream the table once, set one bit each.
__global__ void __launch_bounds__(kBlock) fe_mark_bits(FrontendArgs a) {
  const int b = a.first_scan + blockIdx.y;
  if (a.counts[b] == 0) return;
  const unsigned long long* slots = a.slots2 + (size_t)b * a.tcap2;
  const unsigned long long idx_mask = (1ull << a.idx_bits) - 1;
  for (int h = blockIdx.x * kBlock + threadIdx.x; h < (int)a.tcap2; h += gridDim.x * kBlock) {
    const unsigned long long s = __ldcg(slots + h);
    if (s != kEmpty64) {
      const uint32_t i = (uint32_t)(s & idx_mask);
      atomicOr(scan_bits(a, b, (int)(s >> 63)) + (i >> 5), 1u << (i & 31));  // result unused: a reduction, no round trip
    }
  }
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

// C2: gridDim.x CTAs per scan. Every CTA counts the bits of all 1024-point chunks of its scan (32 words per chunk: a few KiB from
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
}

}  // namespace

int launch_fe_prepare(dl_context* ctx, const FrontendArgs& a, int batch) {
  DL_CUDA(ctx, cudaMemsetAsync(a.table1, 0xFF, (size_t)batch * a.tcap1 * sizeof(uint32_t), ctx->stream));
  DL_CUDA(ctx, cudaMemsetAsync(a.slots2, 0xFF, (size_t)batch * a.tcap2 * sizeof(unsigned long long), ctx->stream));
  DL_CUDA(ctx, cudaMemsetAsync(a.bits, 0, (size_t)batch * 2 * a.bit_words * sizeof(uint32_t), ctx->stream));
  fe_reset_counters<<<(batch + 127) / 128, 128, 0, ctx->stream>>>(a, batch);
  DL_LAUNCH_CHECK(ctx, "fe_reset_counters");
  return DL_OK;
}

// Kernel A for scans [first_scan, first_scan + num_scans): lets the host overlap the upload of later scans.
int launch_fe_first_filter(dl_context* ctx, FrontendArgs a, int first_scan, int num_scans) {
  if (num_scans <= 0) return DL_OK;
  a.first_scan = first_scan;
  const int tiles = (int)std::min<int64_t>((a.cap + kBlock - 1) / kBlock, 128);
  fe_first_filter_insert<<<dim3(tiles, num_scans), kBlock, 0, ctx->stream>>>(a);
  DL_LAUNCH_CHECK(ctx, "fe_first_filter_insert");
  return DL_OK;
}

int launch_fe_rest(dl_context* ctx, FrontendArgs a, int first_scan, int batch) {
  if (batch <= 0) return DL_OK;
  a.first_scan = first_scan;
  const int tiles = (int)std::min<int64_t>((a.cap + kBlock - 1) / kBlock, 128);
  const int per_scan = 48;  // measured best of {8, 20, 32, 48, 64}: enough CTAs in flight to hide the random-access latency
  if (a.run_pose && a.max_runs > 0) {
    fe_run_poses<<<dim3((a.max_runs + 127) / 128, batch), 128, 0, ctx->stream>>>(a);
    DL_LAUNCH_CHECK(ctx, "fe_run_poses");
    fe_ingest_second_insert<true><<<dim3(per_scan, batch), kBlock, 0, ctx->stream>>>(a);
  } else {
    fe_ingest_second_insert<false><<<dim3(per_scan, batch), kBlock, 0, ctx->stream>>>(a);
  }
  DL_LAUNCH_CHECK(ctx, "fe_ingest_second_insert");
  fe_mark_bits<<<dim3(tiles, batch), kBlock, 0, ctx->stream>>>(a);
  DL_LAUNCH_CHECK(ctx, "fe_mark_bits");
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

}  // namespace dl
