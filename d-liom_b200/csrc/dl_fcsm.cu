// Loop-closure coarse matcher (SURVEY 8f-2): FastCorrelativeScanMatcher3D::MatchWith3DofInitial
// (SM/fast_correlative_scan_matcher_3d.cc:165-196) without the branch and bound.
//
// The reference prunes the (x, y, z) translation window with a stack of max-pooled 8-bit "precomputation" grids
// (PrecomputationGridStack3D, :57-77; PrecomputeGrid, precomputation_grid_3d.cc:62-81) because a CPU cannot afford the
// ~10^5 leaves x 10^3 points of the full window. The bounds are exact, so branch and bound returns the best-scoring
// leaf that passes the low-resolution gate — which is also what scoring EVERY leaf returns. On the GPU the brute-force
// cube is L1/L2-resident integer gathers, needs no precomputation stack at all (the
// 8-bit value is derived from the uint16 cell on the fly with the reference's float expression,
// precomputation_grid_3d.cc:50-53) and has no data-dependent control flow:
//   cells      c_i = GetCellIndex(pose * p_i)                                 (float, exact)
//   leaf score s(o) = ToProbability( sum_i V8[c_i + o] / float(N) )           (integer sum: order-independent, exact)
//   result     argmax_o s(o) subject to s(o) > min_score and the low-resolution gate (low_resolution_matcher.cc:24-36),
//              lowest linear index (z, y, x order) among equal scores; the reference's own tie order is that of an
//              unstable std::sort.
//
// Pruned form (default when the submap has a search index): the reference's depth-3 bound, kept exact. For a block of
// 8 x 8 x 8 translations starting at o0 the sum over points of M8[c_i + o0], M8[x] = max of V8 over [x, x + 8)^3 (the
// sliding maximum PrecomputeGrid builds, stored here as one dense byte volume per finished submap), dominates every leaf
// sum of the block. Blocks are opened in two rounds — first those within 1/8 of the largest bound, then every remaining
// block whose bound still reaches the best leaf found (>=, so equal-score leaves with a lower index are not lost) — and
// everything else is provably below the answer. On street scenes ~3-5 % of the blocks are opened
// (tools/fcsm_pruning_study.py); results are identical to the exhaustive kernel, which stays as the fallback.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <vector>

#include "dl_internal.cuh"

namespace dl {
namespace {

constexpr int kBlock = 256;
constexpr int kTile = 1024;
constexpr int kLutSize = 32768;  // uint16 cell value (marker bit dropped) -> 8-bit precomputation-grid value

// GetPoseFromCandidate: Translation(resolution * offset) * discrete_scan.pose (cc:423-430); Rigid3 * Rigid3 re-normalises
__device__ __forceinline__ Rigidf candidate_pose(const Rigidf& pose, float res, int ox, int oy, int oz) {
  return compose(Rigidf{{res * (float)ox, res * (float)oy, res * (float)oz}, {1.f, 0.f, 0.f, 0.f}}, pose);
}

// ConvertToPrecomputationGrid's per-cell expression (precomputation_grid_3d.cc:50-53)
__device__ __forceinline__ int precomputation_value(uint16_t v) {
  const float kMin = 0.1f, kMax = 1.f - 0.1f;
  return round_to_int((value_to_probability(v) - kMin) * (255.f / (kMax - kMin)));
}

// DiscretizeScan at full resolution (cc:253-266) + the candidate-independent half of the low-resolution match: every
// candidate pose shares the rotation, so R * p is formed once per point and a candidate only adds its translation.
__global__ void fcsm_prepare_kernel(const FcsmPair* __restrict__ pairs) {
  const FcsmPair& pr = pairs[blockIdx.y];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < pr.n_hi) {
    const Int3 c = cell_index(apply(pr.pose, Vec3f{pr.hi_pts[3 * i], pr.hi_pts[3 * i + 1], pr.hi_pts[3 * i + 2]}), pr.hi.resolution);
    pr.cells[3 * i] = c.x; pr.cells[3 * i + 1] = c.y; pr.cells[3 * i + 2] = c.z;
  }
  if (i < pr.n_lo) {
    const Quatf q = candidate_pose(pr.pose, pr.hi.resolution, 0, 0, 0).q;
    const Vec3f r = rotate(q, Vec3f{pr.lo_pts[3 * i], pr.lo_pts[3 * i + 1], pr.lo_pts[3 * i + 2]});
    pr.lo_rot[3 * i] = r.x; pr.lo_rot[3 * i + 1] = r.y; pr.lo_rot[3 * i + 2] = r.z;
  }
}

// Brick row (8 voxels along x, 16 bytes, 16-byte aligned) that holds shifted cell (sx, sy, sz), or nullptr when the
// cell is outside the grid or its brick was never allocated (HybridGrid::value() -> 0 in both cases).
__device__ __forceinline__ const uint4* brick_row(const GridView& g, int sx, int sy, int sz) {
  const int gs = 64 << g.bits;
  if ((unsigned)sx >= (unsigned)gs || (unsigned)sy >= (unsigned)gs || (unsigned)sz >= (unsigned)gs) return nullptr;
  const int node = __ldg(g.top + ((((sz >> 6) << g.bits) + (sy >> 6)) << g.bits) + (sx >> 6));
  if (node < 0) return nullptr;
  const int brick = __ldg(g.nodes + (size_t)node * 512 + ((((sz >> 3) & 7) << 6) | (((sy >> 3) & 7) << 3) | ((sx >> 3) & 7)));
  if (brick < 0) return nullptr;
  return reinterpret_cast<const uint4*>(g.bricks + (size_t)brick * 512 + (((sz & 7) << 6) | ((sy & 7) << 3)));
}

constexpr int kRun = 8;  // leaves per thread: one brick-row-aligned span of x offsets

// The 8-bit value of every possible cell value, built once per context with the reference's float expression and
// staged in shared memory by every CTA: one shared-memory load per voxel instead of ~12 float/convert instructions.
__global__ void fcsm_lut_kernel(uint8_t* __restrict__ lut) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < kLutSize) lut[v] = (uint8_t)precomputation_value((uint16_t)v);
}

template <int A>
__device__ __forceinline__ void add_run(const uint4& r0, const uint4& r1, const uint8_t* __restrict__ lut, int (&sum)[kRun]) {
  const unsigned w[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
#pragma unroll
  for (int k = 0; k < kRun; ++k) {
    const int e = A + k;
    const unsigned v = (e & 1) ? (w[e >> 1] >> 16) : (w[e >> 1] & 0xFFFFu);
    sum[k] += lut[v & (kLutSize - 1)];  // value_to_probability ignores the update marker (bit 15)
  }
}

// One thread per run of 8 consecutive x offsets of the translation window (one (y, z) offset): for every
// high-resolution cell the 8 leaves read 8 consecutive voxels = at most two 16-byte brick rows, so the three-level
// walk is paid twice per point instead of eight times and the values arrive as 128-bit loads. The phase of the run
// inside a brick row depends on the point only (runs start 8 apart), i.e. it is uniform across the block.
// Integer correlation sums -> score; only leaves above min_score run the low-resolution gate
// (low_resolution_matcher.cc:24-36: float sum in point order); one packed atomicMax per warp.
__global__ void __launch_bounds__(kBlock) fcsm_search_kernel(const FcsmPair* __restrict__ pairs, unsigned long long* __restrict__ best,
                                                             float* __restrict__ all_scores, const uint8_t* __restrict__ lut_global) {
  __shared__ int tile[kTile * 3];
  __shared__ __align__(16) uint8_t lut[kLutSize];
  const FcsmPair& pr = pairs[blockIdx.y];
  const int side = 2 * pr.wxy + 1;
  const int runs = (side + kRun - 1) / kRun;
  const int rows = side * (2 * pr.wz + 1);
  if ((long long)blockIdx.x * kBlock >= (long long)rows * runs) return;
  for (int j = threadIdx.x; j < kLutSize / 16; j += kBlock)
    reinterpret_cast<uint4*>(lut)[j] = __ldg(reinterpret_cast<const uint4*>(lut_global) + j);
  const int tid = blockIdx.x * kBlock + threadIdx.x;
  const bool active = tid < rows * runs;
  const int run = active ? tid % runs : 0, row = active ? tid / runs : 0;
  const int ox0 = -pr.wxy + kRun * run, oy = row % side - pr.wxy, oz = row / side - pr.wz;
  const int half = (64 << pr.hi.bits) >> 1;
  int sum[kRun] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int base = 0; base < pr.n_hi; base += kTile) {
    const int count = min(kTile, pr.n_hi - base);
    __syncthreads();
    for (int j = threadIdx.x; j < count * 3; j += kBlock) tile[j] = pr.cells[base * 3 + j];
    __syncthreads();
    if (active)
      for (int j = 0; j < count; ++j) {
        const int sx = tile[3 * j] + ox0 + half, sy = tile[3 * j + 1] + oy + half, sz = tile[3 * j + 2] + oz + half;
        const int phase = sx & 7;  // block-uniform
        const uint4* p0 = brick_row(pr.hi, sx - phase, sy, sz);
        const uint4* p1 = phase ? brick_row(pr.hi, sx - phase + 8, sy, sz) : nullptr;
        if (!p0 && !p1) continue;
        const uint4 zero = make_uint4(0, 0, 0, 0);
        const uint4 r0 = p0 ? __ldg(p0) : zero, r1 = p1 ? __ldg(p1) : zero;
        switch (phase) {
          case 0: add_run<0>(r0, r1, lut, sum); break;
          case 1: add_run<1>(r0, r1, lut, sum); break;
          case 2: add_run<2>(r0, r1, lut, sum); break;
          case 3: add_run<3>(r0, r1, lut, sum); break;
          case 4: add_run<4>(r0, r1, lut, sum); break;
          case 5: add_run<5>(r0, r1, lut, sum); break;
          case 6: add_run<6>(r0, r1, lut, sum); break;
          default: add_run<7>(r0, r1, lut, sum); break;
        }
      }
  }
  const float kMin = 0.1f, kMax = 1.f - 0.1f;
  float score[kRun];
  unsigned cand = 0;
#pragma unroll
  for (int k = 0; k < kRun; ++k) {
    score[k] = kMin + ((float)sum[k] / (float)pr.n_hi) * ((kMax - kMin) / 255.f);  // ToProbability(sum / float(n))
    const bool leaf = active && ox0 + k <= pr.wxy;
    if (leaf && all_scores) all_scores[((long long)row * side) + (ox0 + k + pr.wxy)] = score[k];
    if (leaf && score[k] > pr.min_score) cand |= 1u << k;
  }
  float low[kRun] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  float* ftile = reinterpret_cast<float*>(tile);
  const bool any = __syncthreads_or(cand != 0);
  if (!any) return;
  for (int base = 0; base < pr.n_lo; base += kTile) {
    const int count = min(kTile, pr.n_lo - base);
    __syncthreads();
    for (int j = threadIdx.x; j < count * 3; j += kBlock) ftile[j] = pr.lo_rot[base * 3 + j];
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kRun; ++k) {
      if (!(cand >> k & 1)) continue;
      const Vec3f t = candidate_pose(pr.pose, pr.hi.resolution, ox0 + k, oy, oz).t;
      float acc = low[k];
      for (int j = 0; j < count; ++j) {
        const Int3 c = cell_index(add(Vec3f{ftile[3 * j], ftile[3 * j + 1], ftile[3 * j + 2]}, t), pr.lo.resolution);
        acc += value_to_probability(grid_value(pr.lo, c.x, c.y, c.z));
      }
      low[k] = acc;
    }
  }
  unsigned long long packed = 0ull;
#pragma unroll
  for (int k = 0; k < kRun; ++k) {
    if (!(cand >> k & 1) || !((double)(low[k] / (float)pr.n_lo) >= pr.min_low)) continue;
    const unsigned long long idx = (unsigned long long)row * side + (ox0 + k + pr.wxy);
    const unsigned long long p = ((unsigned long long)__float_as_uint(score[k]) << 32) | (0xFFFFFFFFull - idx);
    packed = p > packed ? p : packed;
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    const unsigned long long o = __shfl_xor_sync(0xffffffffu, packed, d);
    packed = o > packed ? o : packed;
  }
  if ((threadIdx.x & 31) == 0 && packed) atomicMax(best + blockIdx.y, packed);
}

// ------------------------------------------------------------------------------------------- search index (per submap)
// pass X: A[x, y, z] = max of V8 over x .. x+7 (grid read through brick rows: 16 cells -> 8 outputs per thread)
__global__ void __launch_bounds__(256) m8_pass_x_kernel(GridView g, const uint8_t* __restrict__ lut, int ox, int oy, int oz, int nx,
                                                        int ny, int nz, uint8_t* __restrict__ out) {
  // ox is chosen so that (ox + half) % 8 == 0: every thread's 8 outputs start on a brick-row boundary
  const long long t = (long long)blockIdx.x * 256 + threadIdx.x;
  const int runs = nx / 8;
  if (t >= (long long)runs * ny * nz) return;
  const int rx = (int)(t % runs), y = (int)((t / runs) % ny), z = (int)(t / ((long long)runs * ny));
  const int half = (64 << g.bits) >> 1;
  const int sx = ox + 8 * rx + half, sy = oy + y + half, sz = oz + z + half;
  const uint4* p0 = brick_row(g, sx, sy, sz);
  const uint4* p1 = brick_row(g, sx + 8, sy, sz);
  const uint4 zero = make_uint4(0, 0, 0, 0);
  const uint4 r0 = p0 ? __ldg(p0) : zero, r1 = p1 ? __ldg(p1) : zero;
  const unsigned w[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
  int v[16];
#pragma unroll
  for (int e = 0; e < 16; ++e) {
    const unsigned c = (e & 1) ? (w[e >> 1] >> 16) : (w[e >> 1] & 0xFFFFu);
    v[e] = c ? (int)__ldg(lut + (c & (kLutSize - 1))) : 0;
  }
#pragma unroll
  for (int e = 0; e < 15; ++e) v[e] = max(v[e], v[e + 1]);   // window 2
#pragma unroll
  for (int e = 0; e < 13; ++e) v[e] = max(v[e], v[e + 2]);   // window 4
#pragma unroll
  for (int e = 0; e < 9; ++e) v[e] = max(v[e], v[e + 4]);    // window 8
  unsigned lo = 0, hi = 0;
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    lo |= (unsigned)v[e] << (8 * e);
    hi |= (unsigned)v[4 + e] << (8 * e);
  }
  uint2* dst = reinterpret_cast<uint2*>(out + ((size_t)z * ny + y) * nx + 8 * rx);
  *dst = make_uint2(lo, hi);
}

// pass along a strided axis: out[i] = max(in[i], in[i + stride], ..., in[i + 7 stride]) with zeros past the end
__global__ void __launch_bounds__(256) m8_pass_axis_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, long long total,
                                                           long long stride, int extent_index_div, int extent) {
  // element i has coordinate (i / extent_index_div) % extent along the axis being filtered
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= total) return;
  const int c = (int)((i / extent_index_div) % extent);
  int m = 0;
#pragma unroll
  for (int d = 0; d < 8; ++d)
    if (c + d < extent) m = max(m, (int)in[i + d * stride]);
  out[i] = (uint8_t)m;
}

// ------------------------------------------------------------------------------------------- pruned search
constexpr int kSub = 8;  // block edge

__device__ __forceinline__ float sum_to_score(int sum, int n) {
  const float kMin = 0.1f, kMax = 1.f - 0.1f;
  return kMin + ((float)sum / (float)n) * ((kMax - kMin) / 255.f);  // PrecomputationGrid3D::ToProbability(sum / float(n))
}

__device__ __forceinline__ void block_dims(const FcsmPair& pr, int* bx, int* by, int* bz) {
  *bx = (2 * pr.wxy + 1 + kSub - 1) / kSub;
  *by = *bx;
  *bz = (2 * pr.wz + 1 + kSub - 1) / kSub;
}

// bound of every 8^3 block of the window: sum over points of the sliding maximum at the block's first offset.
// One WARP per block: the lanes split the points (integer sum: order-independent), so the dependent byte gathers of a block
// run 32 wide instead of one after the other (round 1: one thread per block, 93 us for 8 pairs).
__global__ void __launch_bounds__(128) fcsm_bounds_kernel(const FcsmPair* __restrict__ pairs, int* __restrict__ bounds, int stride,
                                                          int* __restrict__ max_bound) {
  const FcsmPair& pr = pairs[blockIdx.y];
  int bx, by, bz;
  block_dims(pr, &bx, &by, &bz);
  const int blocks = bx * by * bz;
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (b >= blocks) return;  // warp-uniform
  const int ox = -pr.wxy + kSub * (b % bx), oy = -pr.wxy + kSub * ((b / bx) % by), oz = -pr.wz + kSub * (b / (bx * by));
  int sum = 0;
  for (int i = lane; i < pr.n_hi; i += 32) {
    const int x = pr.cells[3 * i] + ox - pr.m8_org[0], y = pr.cells[3 * i + 1] + oy - pr.m8_org[1], z = pr.cells[3 * i + 2] + oz - pr.m8_org[2];
    if ((unsigned)x < (unsigned)pr.m8_dim[0] && (unsigned)y < (unsigned)pr.m8_dim[1] && (unsigned)z < (unsigned)pr.m8_dim[2])
      sum += __ldg(pr.m8 + ((size_t)z * pr.m8_dim[1] + y) * pr.m8_dim[0] + x);
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, d);
  if (lane == 0) {
    bounds[(size_t)blockIdx.y * stride + b] = sum;
    if (sum > 0) atomicMax(max_bound + blockIdx.y, sum);
  }
}

// Low-resolution gate of ONE candidate leaf, evaluated by the whole CTA (low_resolution_matcher.cc:24-36): the threads gather the
// probabilities of the rotated low-resolution points in parallel (the three-level walks are the expensive part), then thread 0
// adds them up in point order, which is what keeps the float sum bit-identical to the reference's sequential loop.
// prob: shared scratch of kTile floats. Returns (to every thread) whether the leaf passes.
template <int THREADS>
__device__ bool low_resolution_gate(const FcsmPair& pr, const Vec3f& t, float* prob, float* low_out) {
  __shared__ float acc_s;
  __shared__ int pass_s;
  if (threadIdx.x == 0) acc_s = 0.f;
  for (int base = 0; base < pr.n_lo; base += kTile) {
    const int count = min(kTile, pr.n_lo - base);
    __syncthreads();
    for (int j = threadIdx.x; j < count; j += THREADS) {
      const float* r = pr.lo_rot + 3 * (size_t)(base + j);
      const Int3 c = cell_index(add(Vec3f{r[0], r[1], r[2]}, t), pr.lo.resolution);
      prob[j] = value_to_probability(grid_value(pr.lo, c.x, c.y, c.z));
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      float acc = acc_s;
      for (int j = 0; j < count; ++j) acc += prob[j];
      acc_s = acc;
    }
  }
  if (threadIdx.x == 0) {
    const float low = acc_s / (float)pr.n_lo;
    *low_out = low;
    pass_s = (double)low >= pr.min_low ? 1 : 0;
  }
  __syncthreads();
  return pass_s != 0;
}

// One CTA per (block, pair): 64 leaf threads (one (y, z) offset of the block with its 8 x offsets each) x kPointGroups groups that
// share the node's points (group g takes points g, g + kPointGroups, ...; the leaf sums are integers, so adding the groups' partial
// sums is exact and order-free). A search is a handful of open blocks, i.e. its time is ONE CTA's walk over the cloud — the
// groups cut that walk's length, which is what the exchange step waits for. round 0 opens the blocks within 1/8 of the pair's
// largest bound; round 1 every other block whose bound still reaches the best leaf so far.
constexpr int kPointGroups = 4;
__global__ void __launch_bounds__(64 * kPointGroups) fcsm_block_kernel(const FcsmPair* __restrict__ pairs, const int* __restrict__ bounds, int stride,
                                                        const int* __restrict__ max_bound, unsigned long long* __restrict__ best,
                                                        const uint8_t* __restrict__ lut, int round) {
  __shared__ int tile[kTile * 3];
  const FcsmPair& pr = pairs[blockIdx.y];
  int bx, by, bz;
  block_dims(pr, &bx, &by, &bz);
  const int b = blockIdx.x;
  if (b >= bx * by * bz) return;
  __shared__ int skip;
  if (threadIdx.x == 0) {  // one decision for the whole CTA: `best` moves while the round runs
    const int bound = bounds[(size_t)blockIdx.y * stride + b];
    const int top = max_bound[blockIdx.y];
    const bool first_round = bound >= top - (top >> 3);
    const float bound_score = sum_to_score(bound, pr.n_hi);
    bool s = !(bound_score > pr.min_score);  // no leaf of the block can exceed min_score
    if (round == 0) {
      s = s || !first_round;
    } else {
      const unsigned long long cur = *reinterpret_cast<volatile const unsigned long long*>(best + blockIdx.y);
      // strictly below the best leaf so far: nothing in the block can win or tie
      s = s || first_round || (cur != 0ull && bound_score < __uint_as_float((unsigned)(cur >> 32)));
    }
    skip = s ? 1 : 0;
  }
  __syncthreads();
  if (skip) return;
  const int side = 2 * pr.wxy + 1;
  const int leaf = threadIdx.x & 63, group = threadIdx.x >> 6;
  const int ox0 = -pr.wxy + kSub * (b % bx);
  const int oy = -pr.wxy + kSub * ((b / bx) % by) + (leaf & 7);
  const int oz = -pr.wz + kSub * (b / (bx * by)) + (leaf >> 3);
  const bool active = oy <= pr.wxy && oz <= pr.wz;
  const int half = (64 << pr.hi.bits) >> 1;
  int sum[kRun] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int base = 0; base < pr.n_hi; base += kTile) {
    const int count = min(kTile, pr.n_hi - base);
    __syncthreads();
    for (int j = threadIdx.x; j < count * 3; j += 64 * kPointGroups) tile[j] = pr.cells[base * 3 + j];
    __syncthreads();
    if (active)
      for (int j = group; j < count; j += kPointGroups) {
        const int sx = tile[3 * j] + ox0 + half, sy = tile[3 * j + 1] + oy + half, sz = tile[3 * j + 2] + oz + half;
        const int phase = sx & 7;  // block-uniform
        const uint4* p0 = brick_row(pr.hi, sx - phase, sy, sz);
        const uint4* p1 = phase ? brick_row(pr.hi, sx - phase + 8, sy, sz) : nullptr;
        if (!p0 && !p1) continue;
        const uint4 zero = make_uint4(0, 0, 0, 0);
        const uint4 r0 = p0 ? __ldg(p0) : zero, r1 = p1 ? __ldg(p1) : zero;
        switch (phase) {
          case 0: add_run<0>(r0, r1, lut, sum); break;
          case 1: add_run<1>(r0, r1, lut, sum); break;
          case 2: add_run<2>(r0, r1, lut, sum); break;
          case 3: add_run<3>(r0, r1, lut, sum); break;
          case 4: add_run<4>(r0, r1, lut, sum); break;
          case 5: add_run<5>(r0, r1, lut, sum); break;
          case 6: add_run<6>(r0, r1, lut, sum); break;
          default: add_run<7>(r0, r1, lut, sum); break;
        }
      }
  }
  // fold the groups' partial sums into group 0 (integers: exact), then only the 64 leaf threads go on
  __shared__ int partial[kPointGroups - 1][64][kRun];
  if (group > 0) {
#pragma unroll
    for (int k = 0; k < kRun; ++k) partial[group - 1][leaf][k] = sum[k];
  }
  __syncthreads();  // also: everyone is done with `tile`
  if (group > 0) return;  // whole warps leave; the barriers below count the remaining threads only
#pragma unroll
  for (int g = 0; g < kPointGroups - 1; ++g)
#pragma unroll
    for (int k = 0; k < kRun; ++k) sum[k] += partial[g][leaf][k];
  // Candidate leaves of this block, best first: (score bits << 32 | ~index), the same key `best` is maximised with. Only the
  // best candidate that PASSES the low-resolution gate can win, so the CTA walks its candidates in descending key order,
  // evaluates the gate cooperatively (low_resolution_gate) and stops at the first pass — or as soon as the remaining keys
  // are below the best leaf any CTA has published. Round 1 ran the gate inside each thread, serially per candidate
  // (~150 us per leaf of three-level walks): the dominant cost of the whole search.
  __shared__ unsigned long long cand[64 * kRun];
  __shared__ unsigned long long pick_s;
#pragma unroll
  for (int k = 0; k < kRun; ++k) {
    const float sc = sum_to_score(sum[k], pr.n_hi);
    unsigned long long key = 0ull;
    if (active && ox0 + k <= pr.wxy && sc > pr.min_score) {
      const unsigned long long idx = ((unsigned long long)(oz + pr.wz) * side + (oy + pr.wxy)) * side + (ox0 + k + pr.wxy);
      key = ((unsigned long long)__float_as_uint(sc) << 32) | (0xFFFFFFFFull - idx);
    }
    cand[threadIdx.x * kRun + k] = key;
  }
  float* prob = reinterpret_cast<float*>(tile);
  for (;;) {
    __syncthreads();
    unsigned long long m = 0ull;
    for (int e = threadIdx.x; e < 64 * kRun; e += 64) m = cand[e] > m ? cand[e] : m;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      const unsigned long long o = __shfl_xor_sync(0xffffffffu, m, d);
      m = o > m ? o : m;
    }
    if (threadIdx.x == 0) pick_s = 0ull;
    __syncthreads();
    if ((threadIdx.x & 31) == 0 && m) atomicMax(&pick_s, m);
    __syncthreads();
    const unsigned long long key = pick_s;
    if (!key) return;
    const unsigned long long seen = *reinterpret_cast<volatile const unsigned long long*>(best + blockIdx.y);
    if (key < seen) return;  // keys are unique per leaf: everything left in this block loses to a published leaf
    const long long idx = (long long)(0xFFFFFFFFull - (key & 0xFFFFFFFFull));
    const int lx = (int)(idx % side) - pr.wxy, ly = (int)((idx / side) % side) - pr.wxy, lz = (int)(idx / ((long long)side * side)) - pr.wz;
    const Vec3f t = candidate_pose(pr.pose, pr.hi.resolution, lx, ly, lz).t;
    float low;
    if (low_resolution_gate<64>(pr, t, prob, &low)) {
      if (threadIdx.x == 0) atomicMax(best + blockIdx.y, key);
      return;
    }
    // rejected by the gate: drop it and try the next best
    for (int e = threadIdx.x; e < 64 * kRun; e += 64)
      if (cand[e] == key) cand[e] = 0ull;
  }
}

// Decode the winner of each pair: Result{score, pose_estimate, rotational_score, low_resolution_score} (cc:186-195) and the
// switch + initial pose the refinement kernel reads. One CTA per pair; the winner's low-resolution score is recomputed with
// the cooperative gate (parallel gathers, sequential float sum) — round 1 walked the cloud with one thread per pair (262 us).
__global__ void __launch_bounds__(128) fcsm_finish_kernel(const FcsmPair* __restrict__ pairs, const unsigned long long* __restrict__ best,
                                                          int count, FcsmPick* __restrict__ picks) {
  __shared__ float prob[kTile];
  const int p = blockIdx.x;
  if (p >= count) return;
  const FcsmPair& pr = pairs[p];
  FcsmPick out{};
  const int side = 2 * pr.wxy + 1;
  out.num_candidates = (long long)side * side * (2 * pr.wz + 1);
  const unsigned long long b = best[p];
  Rigidf pose = pr.pose;
  if (b) {  // block-uniform
    const long long idx = (long long)(0xFFFFFFFFull - (b & 0xFFFFFFFFull));
    out.found = 1;
    out.score = __uint_as_float((unsigned)(b >> 32));
    out.offset[0] = (int)(idx % side) - pr.wxy;
    out.offset[1] = (int)((idx / side) % side) - pr.wxy;
    out.offset[2] = (int)(idx / ((long long)side * side)) - pr.wz;
    pose = candidate_pose(pr.pose, pr.hi.resolution, out.offset[0], out.offset[1], out.offset[2]);
    __shared__ float low_s;
    low_resolution_gate<128>(pr, pose.t, prob, &low_s);
    __syncthreads();
    out.low_resolution_score = low_s;
  }
  if (threadIdx.x == 0) {
    pose_to7(to_double(pose), out.pose);
    picks[p] = out;
  }
}

}  // namespace

int ensure_fcsm_lut(dl_context* ctx) {
  if (!ctx->d_fcsm_lut.get()) {
    DL_TRY(alloc(ctx, ctx->d_fcsm_lut, kLutSize));
    fcsm_lut_kernel<<<kLutSize / 256, 256, 0, ctx->stream>>>(ctx->d_fcsm_lut.get());
    DL_LAUNCH_CHECK(ctx, "fcsm_lut_kernel");
  }
  return DL_OK;
}

// Dense sliding-maximum volume of one grid: out has nx * ny * nz bytes, element (0, 0, 0) = cell (ox, oy, oz); tmp same size.
// nx is a multiple of 8 and (ox + grid_size / 2) % 8 == 0.
int launch_fcsm_index(dl_context* ctx, const GridView& g, int ox, int oy, int oz, int nx, int ny, int nz, uint8_t* tmp, uint8_t* out) {
  DL_TRY(ensure_fcsm_lut(ctx));
  const long long total = (long long)nx * ny * nz, runs = total / 8;
  m8_pass_x_kernel<<<(unsigned)((runs + 255) / 256), 256, 0, ctx->stream>>>(g, ctx->d_fcsm_lut.get(), ox, oy, oz, nx, ny, nz, out);
  DL_LAUNCH_CHECK(ctx, "m8_pass_x_kernel");
  m8_pass_axis_kernel<<<(unsigned)((total + 255) / 256), 256, 0, ctx->stream>>>(out, tmp, total, nx, nx, ny);
  DL_LAUNCH_CHECK(ctx, "m8_pass_axis_kernel(y)");
  m8_pass_axis_kernel<<<(unsigned)((total + 255) / 256), 256, 0, ctx->stream>>>(tmp, out, total, (long long)nx * ny, nx * ny, nz);
  DL_LAUNCH_CHECK(ctx, "m8_pass_axis_kernel(z)");
  return DL_OK;
}

// Pruned search: bounds of every 8^3 block, then two rounds of block evaluation. bounds_dev: count * stride ints.
int launch_fcsm_pruned(dl_context* ctx, const FcsmPair* pairs_dev, int count, int max_points, int max_blocks, int* bounds_dev,
                       int* max_bound_dev, unsigned long long* best_dev, FcsmPick* picks_dev) {
  DL_TRY(ensure_fcsm_lut(ctx));
  DL_CUDA(ctx, cudaMemsetAsync(best_dev, 0, sizeof(unsigned long long) * count, ctx->stream));
  DL_CUDA(ctx, cudaMemsetAsync(max_bound_dev, 0, sizeof(int) * count, ctx->stream));
  fcsm_prepare_kernel<<<dim3((max_points + 255) / 256, count), 256, 0, ctx->stream>>>(pairs_dev);
  DL_LAUNCH_CHECK(ctx, "fcsm_prepare_kernel");
  fcsm_bounds_kernel<<<dim3((max_blocks + 3) / 4, count), 128, 0, ctx->stream>>>(pairs_dev, bounds_dev, max_blocks, max_bound_dev);
  DL_LAUNCH_CHECK(ctx, "fcsm_bounds_kernel");
  for (int round = 0; round < 2; ++round) {
    fcsm_block_kernel<<<dim3(max_blocks, count), 64 * kPointGroups, 0, ctx->stream>>>(pairs_dev, bounds_dev, max_blocks, max_bound_dev, best_dev,
                                                                       ctx->d_fcsm_lut.get(), round);
    DL_LAUNCH_CHECK(ctx, "fcsm_block_kernel");
  }
  fcsm_finish_kernel<<<count, 128, 0, ctx->stream>>>(pairs_dev, best_dev, count, picks_dev);
  DL_LAUNCH_CHECK(ctx, "fcsm_finish_kernel");
  return DL_OK;
}

namespace {
// Constraint{submap_id, node_id, pose, weights} (constraint_builder_3d.cc:328-333) for every searched pair, written where the
// all-gather reads it: no host round trip between the refinement and the exchange.
__global__ void pack_constraint_rows_kernel(int n, const FcsmPick* __restrict__ picks, const NlsOutput* __restrict__ refined,
                                            const int32_t* __restrict__ submap_ids, const int32_t* __restrict__ node_ids,
                                            double translation_weight, double rotation_weight, int rank, dl_constraint_row* rows) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  dl_constraint_row r;
  r.submap_id = submap_ids[k];
  r.node_id = node_ids[k];
  r.found = picks[k].found ? 1 : 0;
  r.rank = rank;
  r.score = picks[k].found ? picks[k].score : 0.f;
  r.low_resolution_score = picks[k].found ? picks[k].low_resolution_score : 0.f;
  for (int i = 0; i < 7; ++i) r.pose[i] = picks[k].found ? refined[k].pose[i] : picks[k].pose[i];
  r.translation_weight = translation_weight;
  r.rotation_weight = rotation_weight;
  rows[k] = r;
}
}  // namespace

int launch_pack_constraint_rows(dl_context* ctx, int n, const FcsmPick* picks, const NlsOutput* refined, const int32_t* submap_ids,
                                const int32_t* node_ids, double translation_weight, double rotation_weight, int rank,
                                dl_constraint_row* rows) {
  if (n <= 0) return DL_OK;
  pack_constraint_rows_kernel<<<(n + 127) / 128, 128, 0, ctx->stream>>>(n, picks, refined, submap_ids, node_ids, translation_weight,
                                                                         rotation_weight, rank, rows);
  DL_LAUNCH_CHECK(ctx, "pack_constraint_rows_kernel");
  return DL_OK;
}

int launch_fcsm(dl_context* ctx, const FcsmPair* pairs_dev, int count, int max_points, long long max_threads,
                unsigned long long* best_dev, FcsmPick* picks_dev, float* all_scores_dev) {
  DL_TRY(ensure_fcsm_lut(ctx));
  DL_CUDA(ctx, cudaMemsetAsync(best_dev, 0, sizeof(unsigned long long) * count, ctx->stream));
  fcsm_prepare_kernel<<<dim3((max_points + 255) / 256, count), 256, 0, ctx->stream>>>(pairs_dev);
  DL_LAUNCH_CHECK(ctx, "fcsm_prepare_kernel");
  fcsm_search_kernel<<<dim3((unsigned)((max_threads + kBlock - 1) / kBlock), count), kBlock, 0, ctx->stream>>>(pairs_dev, best_dev,
                                                                                                           all_scores_dev, ctx->d_fcsm_lut.get());
  DL_LAUNCH_CHECK(ctx, "fcsm_search_kernel");
  fcsm_finish_kernel<<<count, 128, 0, ctx->stream>>>(pairs_dev, best_dev, count, picks_dev);
  DL_LAUNCH_CHECK(ctx, "fcsm_finish_kernel");
  return DL_OK;
}

}  // namespace dl

// ------------------------------------------------------------------------------------------------ loop closure
using namespace dl;

namespace {
struct CoarseSearch {  // device state of one chunk of (node, submap) pairs
  bool pruned;     // pruned search (plan_coarse); otherwise exhaustive
  int max_blocks;  // most pruning blocks of any pair of the chunk (pruned search)
  float *d_hi, *d_lo;  // uploaded clouds (null when device-resident)
  int* d_cells;
  float* d_rot;
  FcsmPair* d_pairs;
  FcsmPick* d_picks;
  unsigned long long* d_best;
  int *d_bounds, *d_max_bound;  // pruned search only
  std::vector<const float*> hi, lo;  // per pair of the chunk: its clouds on the device (uploaded or resident)
};
int check_fcsm_options(dl_context* ctx, const dl_fcsm_options& o) {
  if (o.branch_and_bound_depth < 1 || o.full_resolution_depth < 1)
    return ctx->fail(DL_ERR_ARG, "branch_and_bound_depth and full_resolution_depth must be >= 1 (CHECK_GE)");
  if (o.linear_xy_search_window < 0 || o.linear_z_search_window < 0) return ctx->fail(DL_ERR_ARG, "negative search window");
  return DL_OK;
}
// Loop-closure search index of a grid (dense sliding 8^3 maximum over the bounding box of its bricks), cached in the grid
// and rebuilt when the grid changed. Returns false (no error) when the grid is empty or the volume would be unreasonably
// large: the caller then searches exhaustively.
int ensure_search_index(dl_context* ctx, dl_grid* g, bool* have) {
  std::lock_guard<std::mutex> lock(g->index_mutex);  // grids are shared read-only between contexts: build once
  *have = false;
  if (g->m8_version == g->version && g->d_m8.get()) {
    *have = true;
    return DL_OK;
  }
  if (g->mirror_stale) DL_TRY(grid_download(g));
  const int side = 1 << g->bits;
  int lo[3] = {INT_MAX, INT_MAX, INT_MAX}, hi[3] = {INT_MIN, INT_MIN, INT_MIN};
  for (int tz = 0; tz < side; ++tz)
    for (int ty = 0; ty < side; ++ty)
      for (int tx = 0; tx < side; ++tx) {
        const int node = g->top[top_flat(tx, ty, tz, g->bits)];
        if (node < 0) continue;
        for (int k = 0; k < 512; ++k) {
          if (g->nodes[(size_t)node * 512 + k] < 0) continue;
          const int b[3] = {(tx << 3) | (k & 7), (ty << 3) | ((k >> 3) & 7), (tz << 3) | (k >> 6)};  // brick coordinates
          for (int a = 0; a < 3; ++a) { lo[a] = std::min(lo[a], b[a]); hi[a] = std::max(hi[a], b[a]); }
        }
      }
  if (hi[0] < lo[0]) return DL_OK;  // empty grid
  const int half = (64 << g->bits) >> 1;
  int org[3], dim[3];
  for (int a = 0; a < 3; ++a) {
    org[a] = lo[a] * 8 - half - 8;                 // one brick of margin below: M8 is non-zero from 7 cells before the data
    dim[a] = (hi[a] - lo[a] + 1) * 8 + 8;           // (org + half) % 8 == 0 and dim % 8 == 0 by construction
  }
  const size_t bytes = (size_t)dim[0] * dim[1] * dim[2];
  if (bytes > ((size_t)3 << 30)) return DL_OK;    // > 3 GiB per submap: stay exhaustive
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  if (g->d_m8.cap < bytes) DL_TRY(grow(ctx, g->d_m8, bytes));
  DeviceBuffer<uint8_t> tmp;
  DL_TRY(alloc(ctx, tmp, bytes));
  const int st = launch_fcsm_index(ctx, g->view(), org[0], org[1], org[2], dim[0], dim[1], dim[2], tmp.get(), g->d_m8.get());
  ctx->wait_stream();  // tmp is freed on return
  DL_TRY(st);
  for (int a = 0; a < 3; ++a) { g->m8_org[a] = org[a]; g->m8_dim[a] = dim[a]; }
  g->m8_version = g->version;
  *have = true;
  return DL_OK;
}

// Window half-widths in cells of a search in `hi` (double / float -> double, common::RoundToInt, cc:174-176).
void search_window(const dl_fcsm_options& o, const dl_grid* hi, int* wxy, int* wz) {
  *wxy = (int)std::lround(o.linear_xy_search_window / hi->resolution);
  *wz = (int)std::lround(o.linear_z_search_window / hi->resolution);
}
// Decides, before the scratch is carved, whether pairs [first, first + n) get the pruned search and how many pruning blocks
// its bounds table needs per pair. The pruned search needs the index of every high-resolution grid of the chunk
// (DLIOM_FCSM_EXHAUSTIVE=1 or allow_pruned = false forces the fallback, and then no index is built) and at most 60 000 blocks
// per pair (one CTA per block and pair in grid.x).
int plan_coarse(dl_context* ctx, const dl_fcsm_options& o, int first, int n, const dl_grid* const* hi_grids, CoarseSearch* cs,
                bool allow_pruned = true) {
  cs->pruned = allow_pruned && std::getenv("DLIOM_FCSM_EXHAUSTIVE") == nullptr;
  cs->max_blocks = 1;
  for (int k = 0; k < n && cs->pruned; ++k) {
    bool have = false;
    DL_TRY(ensure_search_index(ctx, const_cast<dl_grid*>(hi_grids[first + k]), &have));
    cs->pruned = have;
  }
  for (int k = 0; k < n; ++k) {
    int wxy, wz;
    search_window(o, hi_grids[first + k], &wxy, &wz);
    const long long side = 2ll * wxy + 1, K = side * side * (2ll * wz + 1);
    if (K >= 0xFFFFFFFFll) return ctx->fail(DL_ERR_ARG, "more than 2^32-1 translation candidates");
    if (cs->pruned) {
      const long long bxy = (side + 7) / 8, bz = (2ll * wz + 1 + 7) / 8;
      if (bxy * bxy * bz > 60000) cs->pruned = false;
      cs->max_blocks = (int)std::max<long long>(cs->max_blocks, bxy * bxy * bz);
    }
  }
  return DL_OK;
}
// The device buffers of the coarse search of pairs [first, first + n), as plan_coarse decided it.
void carve_coarse(Arena& a, const PairClouds& pc, int first, int n, CoarseSearch* cs) {
  const int64_t n_hi = pc.hi_off[first + n] - pc.hi_off[first], n_lo = pc.lo_off[first + n] - pc.lo_off[first];
  const bool resident = pc.hi_store != nullptr;
  cs->d_hi = resident ? nullptr : a.take<float>(3 * n_hi);
  cs->d_lo = resident ? nullptr : a.take<float>(3 * n_lo);
  cs->d_cells = a.take<int>(3 * n_hi);
  cs->d_rot = a.take<float>(3 * n_lo);
  cs->d_pairs = a.take<FcsmPair>(n);
  cs->d_picks = a.take<FcsmPick>(n);
  cs->d_best = a.take<unsigned long long>(n);
  cs->d_bounds = cs->pruned ? a.take<int>((size_t)n * cs->max_blocks) : nullptr;
  cs->d_max_bound = cs->pruned ? a.take<int>(n) : nullptr;
}

// Runs the coarse search for pairs [first, first + n) in the buffers carve_coarse took, uploading their clouds first unless they
// are device-resident; leaves the picks on the device. all_scores_dev (exhaustive search of one pair only): every leaf score.
int coarse_search(dl_context* ctx, const dl_fcsm_options& o, float min_score, int first, int n, const double* guesses,
                  const PairClouds& pc, const dl_grid* const* hi_grids, const dl_grid* const* lo_grids, CoarseSearch* out,
                  float* all_scores_dev = nullptr) {
  const int64_t* hi_off = pc.hi_off;
  const int64_t* lo_off = pc.lo_off;
  const int64_t hi0 = hi_off[first], lo0 = lo_off[first];
  const int64_t n_hi = hi_off[first + n] - hi0, n_lo = lo_off[first + n] - lo0;
  const bool resident = pc.hi_store != nullptr;
  out->hi.resize(n);
  out->lo.resize(n);
  for (int k = 0; k < n; ++k) {
    const int g = first + k;
    out->hi[k] = resident ? pc.hi_store + 3 * pc.hi_begin[g] : out->d_hi + 3 * (hi_off[g] - hi0);
    out->lo[k] = resident ? pc.lo_store + 3 * pc.lo_begin[g] : out->d_lo + 3 * (lo_off[g] - lo0);
  }
  if (!resident) {
    DL_TRY(h2d(ctx, out->d_hi, pc.hi_pts + 3 * hi0, 3 * n_hi));
    DL_TRY(h2d(ctx, out->d_lo, pc.lo_pts + 3 * lo0, 3 * n_lo));
  }
  std::vector<FcsmPair> pairs(n);
  int max_points = 1;
  long long max_candidates = 1;
  for (int k = 0; k < n; ++k) {
    const int g = first + k;
    FcsmPair& p = pairs[k];
    std::memset(&p, 0, sizeof(p));
    p.hi = hi_grids[g]->view();
    p.lo = lo_grids[g]->view();
    p.hi_pts = out->hi[k];
    p.lo_pts = out->lo[k];
    p.cells = out->d_cells + 3 * (hi_off[g] - hi0);
    p.lo_rot = out->d_rot + 3 * (lo_off[g] - lo0);
    p.n_hi = (int)(hi_off[g + 1] - hi_off[g]);
    p.n_lo = (int)(lo_off[g + 1] - lo_off[g]);
    p.pose = to_float(pose_from7(guesses + 7 * g));
    search_window(o, hi_grids[g], &p.wxy, &p.wz);
    p.min_score = min_score;
    p.min_low = o.min_low_resolution_score;
    if (out->pruned) {
      p.m8 = hi_grids[g]->d_m8.get();
      for (int a3 = 0; a3 < 3; ++a3) { p.m8_org[a3] = hi_grids[g]->m8_org[a3]; p.m8_dim[a3] = hi_grids[g]->m8_dim[a3]; }
    }
    const long long side = 2ll * p.wxy + 1;
    max_candidates = std::max(max_candidates, side * (2ll * p.wz + 1) * ((side + kFcsmRun - 1) / kFcsmRun));  // search threads
    max_points = std::max(max_points, std::max(p.n_hi, p.n_lo));
  }
  DL_TRY(h2d(ctx, out->d_pairs, pairs.data(), n));
  DL_TRY(sync(ctx));  // `pairs` is pageable host memory
  StageScope st(ctx, "loop_closure_search");
  if (out->pruned)
    return launch_fcsm_pruned(ctx, out->d_pairs, n, max_points, out->max_blocks, out->d_bounds, out->d_max_bound, out->d_best,
                              out->d_picks);
  return launch_fcsm(ctx, out->d_pairs, n, max_points, max_candidates, out->d_best, out->d_picks, all_scores_dev);
}
int check_pairs(dl_context* ctx, int count, const double* guesses, const float* hi_pts, const int64_t* hi_off, const float* lo_pts,
                const int64_t* lo_off, const dl_grid* const* hi_grids, const dl_grid* const* lo_grids) {
  if (!guesses || !hi_off || !lo_off || !hi_grids || !lo_grids || !hi_pts || !lo_pts) return DL_ERR_ARG;
  for (int k = 0; k < count; ++k) {
    if (!hi_grids[k] || !lo_grids[k]) return DL_ERR_ARG;
    if (hi_off[k + 1] < hi_off[k] || lo_off[k + 1] < lo_off[k]) return ctx->fail(DL_ERR_ARG, "offsets must be non-decreasing");
    if (hi_off[k + 1] == hi_off[k] || lo_off[k + 1] == lo_off[k]) return ctx->fail(DL_ERR_EMPTY, "empty point cloud");
    if (hi_grids[k]->structure_dirty || lo_grids[k]->structure_dirty)
      return ctx->fail(DL_ERR_ARG, "dl_grid_sync not called after dl_grid_set_cells");
  }
  return DL_OK;
}
// RotateHistogram / MatchHistograms (rotational_scan_matcher.cc:123-155), float arithmetic in the reference's order
std::vector<float> rotate_histogram(const float* h, int n, float angle) {
  const float rotate_by_buckets = (float)(-angle * n / M_PI);
  int full_buckets = (int)std::lround(rotate_by_buckets - 0.5f);
  const float fraction = rotate_by_buckets - full_buckets;
  while (full_buckets < 0) full_buckets += n;
  std::vector<float> out(n);
  for (int i = 0; i < n; ++i) out[i] = fraction * h[(i + 1 + full_buckets) % n] + (1.f - fraction) * h[(i + full_buckets) % n];
  return out;
}
float match_histograms(const float* submap, const float* scan, int n) {
  float ss = 0.f, sm = 0.f, dot = 0.f;
  for (int i = 0; i < n; ++i) ss += scan[i] * scan[i];
  for (int i = 0; i < n; ++i) sm += submap[i] * submap[i];
  const float normalization = std::sqrt(ss) * std::sqrt(sm);
  if (normalization < 1e-3f) return 1.f;
  for (int i = 0; i < n; ++i) dot += submap[i] * scan[i];
  return dot / normalization;
}
Quatf eigen_quaternion_inverse_f(const Quatf& q) {  // Eigen::Quaternion::inverse(): conjugate / squared norm
  const float n2 = (q.x * q.x + q.y * q.y) + (q.z * q.z + q.w * q.w);
  return {q.w / n2, -q.x / n2, -q.y / n2, -q.z / n2};
}
Quatd eigen_quaternion_inverse_d(const Quatd& q) {
  const double n2 = (q.x * q.x + q.y * q.y) + (q.z * q.z + q.w * q.w);
  return {q.w / n2, -q.x / n2, -q.y / n2, -q.z / n2};
}
}  // namespace

namespace dl {
int check_constraint_options(dl_context* ctx, const dl_constraint_options& o) {
  DL_TRY(check_fcsm_options(ctx, o.fast_correlative_scan_matcher_3d));
  return check_ceres_options(ctx, &o.ceres_scan_matcher_3d, 2);
}
int constraint_search(dl_context* ctx, const dl_constraint_options& o, int count, const double* guesses, const PairClouds& pc,
                      const dl_grid* const* hi_grids, const dl_grid* const* lo_grids, dl_constraint* constraints) {
  const dl_constraint_options* options = &o;
  const int64_t* hi_off = pc.hi_off;
  const int64_t* lo_off = pc.lo_off;
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  const NlsOptions nls = to_nls_options(options->ceres_scan_matcher_3d, 2);
  constexpr int kChunk = 1024;  // pairs per launch set: bounds the scratch, keeps every grid dimension legal
  for (int first = 0; first < count; first += kChunk) {
    const int n = std::min(kChunk, count - first);
    CoarseSearch cs;
    NlsProblem* d_problems;
    NlsOutput* d_out;
    DL_TRY(plan_coarse(ctx, options->fast_correlative_scan_matcher_3d, first, n, hi_grids, &cs));
    DL_TRY(carve_scratch(ctx, [&](Arena& a) {
      carve_coarse(a, pc, first, n, &cs);
      d_problems = a.take<NlsProblem>(n);
      d_out = a.take<NlsOutput>(n);
    }));
    DL_TRY(coarse_search(ctx, options->fast_correlative_scan_matcher_3d, (float)options->min_score, first, n, guesses, pc,
                         hi_grids, lo_grids, &cs));
    // refinement: initial pose = translation target = the coarse pose, read from the pick record on the device
    std::vector<NlsProblem> problems(n);
    for (int k = 0; k < n; ++k) {
      const int g = first + k;
      NlsProblem& p = problems[k];
      std::memset(&p, 0, sizeof(p));
      p.cloud[0] = cs.hi[k];
      p.cloud[1] = cs.lo[k];
      p.count[0] = (int32_t)(hi_off[g + 1] - hi_off[g]);
      p.count[1] = (int32_t)(lo_off[g + 1] - lo_off[g]);
      p.grid[0] = hi_grids[g]->view();
      p.grid[1] = lo_grids[g]->view();
      p.initial_dev = cs.d_picks[k].pose;  // address arithmetic only
      p.enabled_dev = &cs.d_picks[k].found;
    }
    DL_TRY(h2d(ctx, d_problems, problems.data(), n));
    DL_CUDA(ctx, cudaMemsetAsync(d_out, 0, sizeof(NlsOutput) * n, ctx->stream));
    {
      StageScope st(ctx, "loop_closure_refine");
      DL_TRY(launch_nls(ctx, nls, d_problems, n, d_out));
    }
    std::vector<FcsmPick> picks(n);
    std::vector<NlsOutput> out(n);
    DL_TRY(d2h(ctx, picks.data(), cs.d_picks, n));
    DL_TRY(d2h(ctx, out.data(), d_out, n));
    DL_TRY(sync(ctx));
    for (int k = 0; k < n; ++k) {
      dl_constraint& c = constraints[first + k];
      std::memset(&c, 0, sizeof(c));
      std::memcpy(c.coarse_pose, picks[k].pose, sizeof(c.coarse_pose));
      if (!picks[k].found) continue;
      c.found = 1;
      c.score = picks[k].score;
      c.rotational_score = (float)(options->fast_correlative_scan_matcher_3d.min_rotational_score + 0.01);
      c.low_resolution_score = picks[k].low_resolution_score;
      std::memcpy(c.pose, out[k].pose, sizeof(c.pose));
      c.translation_weight = options->loop_closure_translation_weight;
      c.rotation_weight = options->loop_closure_rotation_weight;
      c.summary = out[k].summary;
    }
  }
  return DL_OK;
}
}  // namespace dl

extern "C" {

int dl_fcsm_match_3dof(dl_context* ctx, const dl_fcsm_options* o, const double* guess, const float* hi_pts, int64_t n_hi,
                       const float* lo_pts, int64_t n_lo, const dl_grid* hi, const dl_grid* lo, float min_score,
                       dl_fcsm_result* result, float* all_scores, int64_t all_scores_capacity) {
  if (!ctx || !o || !result || n_hi < 0 || n_lo < 0) return DL_ERR_ARG;
  const int64_t hi_off[2] = {0, n_hi}, lo_off[2] = {0, n_lo};
  if (guess && hi && lo && (n_hi == 0 || n_lo == 0)) return ctx->fail(DL_ERR_EMPTY, "empty point cloud");
  DL_TRY(check_pairs(ctx, 1, guess, hi_pts, hi_off, lo_pts, lo_off, &hi, &lo));
  DL_TRY(check_fcsm_options(ctx, *o));
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  CoarseSearch cs;
  PairClouds pc;
  pc.hi_pts = hi_pts;
  pc.lo_pts = lo_pts;
  pc.hi_off = hi_off;
  pc.lo_off = lo_off;
  int wxy, wz;
  search_window(*o, hi, &wxy, &wz);
  const int64_t K = (2ll * wxy + 1) * (2ll * wxy + 1) * (2ll * wz + 1);
  if (all_scores && all_scores_capacity < K) return ctx->fail(DL_ERR_ARG, "all_scores has room for fewer than num_candidates floats");
  DL_TRY(plan_coarse(ctx, *o, 0, 1, &hi, &cs, all_scores == nullptr));  // only the exhaustive kernel scores every leaf
  float* d_scores = nullptr;
  DL_TRY(carve_scratch(ctx, [&](Arena& a) {
    carve_coarse(a, pc, 0, 1, &cs);
    d_scores = all_scores ? a.take<float>(K) : nullptr;
  }));
  DL_TRY(coarse_search(ctx, *o, min_score, 0, 1, guess, pc, &hi, &lo, &cs, d_scores));
  FcsmPick pick;
  DL_TRY(d2h(ctx, &pick, cs.d_picks, 1));
  if (all_scores) DL_TRY(d2h(ctx, all_scores, d_scores, K));
  DL_TRY(sync(ctx));
  std::memset(result, 0, sizeof(*result));
  result->num_candidates = pick.num_candidates;
  if (!pick.found) return DL_OK;  // nothing above min_score passes the low-resolution gate: the reference returns nullptr
  result->found = 1;
  result->score = pick.score;
  std::memcpy(result->pose_estimate, pick.pose, sizeof(pick.pose));
  result->rotational_score = (float)(o->min_rotational_score + 0.01);  // what MatchWith3DofInitial reports (cc:179-181)
  result->low_resolution_score = pick.low_resolution_score;
  std::memcpy(result->offset, pick.offset, sizeof(pick.offset));
  return DL_OK;
}

int dl_fcsm_match(dl_context* ctx, const dl_fcsm_options* o, const float* submap_histogram, const float* scan_histogram,
                  int32_t histogram_size, const double* global_node_pose, const double* global_submap_pose,
                  const double* gravity_alignment, const float* hi_pts, int64_t n_hi, const float* lo_pts, int64_t n_lo,
                  const dl_grid* hi, const dl_grid* lo, float min_score, dl_fcsm_result* result) {
  if (!ctx || !o || !result || !submap_histogram || !scan_histogram || histogram_size < 1 || !global_node_pose ||
      !global_submap_pose || !gravity_alignment || !hi || !lo || n_hi < 0 || n_lo < 0 || (n_hi > 0 && !hi_pts) || (n_lo > 0 && !lo_pts))
    return DL_ERR_ARG;
  if (n_hi == 0 || n_lo == 0) return ctx->fail(DL_ERR_EMPTY, "empty point cloud");
  DL_TRY(check_fcsm_options(ctx, *o));
  std::memset(result, 0, sizeof(*result));
  const float res = hi->resolution;
  const Rigidf node = to_float(pose_from7(global_node_pose)), submap = to_float(pose_from7(global_submap_pose));
  // GenerateDiscreteScans (cc:296-350)
  float max_scan_range = 3.f * res;
  for (int64_t i = 0; i < n_hi; ++i) max_scan_range = std::max(norm3(Vec3f{hi_pts[3 * i], hi_pts[3 * i + 1], hi_pts[3 * i + 2]}), max_scan_range);
  const float angular_step_size = (1.f - 1e-2f) * std::acos(1.f - (res * res) / (2.f * (max_scan_range * max_scan_range)));
  const int angular_window_size = (int)std::lround(o->angular_search_window / angular_step_size);
  if (angular_window_size < 0 || angular_window_size > 100000) return ctx->fail(DL_ERR_ARG, "angular window out of range");
  const Rigidf node_to_submap = compose(inverse(submap), node);
  const Quatd ga_inv_d = eigen_quaternion_inverse_d(Quatd{gravity_alignment[0], gravity_alignment[1], gravity_alignment[2], gravity_alignment[3]});
  const Quatf ga_inv{(float)ga_inv_d.w, (float)ga_inv_d.x, (float)ga_inv_d.y, (float)ga_inv_d.z};
  const Vec3f dir = rotate(qmul(node_to_submap.q, ga_inv), Vec3f{1.f, 0.f, 0.f});
  const float initial_angle = std::atan2(dir.y, dir.x);  // transform::GetYaw
  std::vector<double> guesses;
  std::vector<float> scores;
  for (int rz = -angular_window_size; rz <= angular_window_size; ++rz) {
    const float angle = rz * angular_step_size;
    const std::vector<float> rotated = rotate_histogram(scan_histogram, histogram_size, initial_angle + angle);
    const float score = match_histograms(submap_histogram, rotated.data(), histogram_size);
    if (score < o->min_rotational_score) continue;
    const Quatf q = qmul(qmul(eigen_quaternion_inverse_f(submap.q), angle_axis_to_quat(Vec3f{0.f, 0.f, angle})), node.q);
    const double g[7] = {node_to_submap.t.x, node_to_submap.t.y, node_to_submap.t.z, q.w, q.x, q.y, q.z};  // floats widen exactly
    guesses.insert(guesses.end(), g, g + 7);
    scores.push_back(score);
  }
  const int n = (int)scores.size();
  if (n == 0) return DL_OK;  // no yaw step passes the rotational score: the reference returns nullptr
  std::vector<float> hi_all((size_t)n * n_hi * 3), lo_all((size_t)n * n_lo * 3);
  std::vector<int64_t> hi_off(n + 1), lo_off(n + 1);
  std::vector<const dl_grid*> his(n, hi), los(n, lo);
  for (int k = 0; k < n; ++k) {
    std::memcpy(hi_all.data() + (size_t)k * n_hi * 3, hi_pts, (size_t)n_hi * 12);
    std::memcpy(lo_all.data() + (size_t)k * n_lo * 3, lo_pts, (size_t)n_lo * 12);
    hi_off[k] = k * n_hi; lo_off[k] = k * n_lo;
  }
  hi_off[n] = n * n_hi; lo_off[n] = n * n_lo;
  DL_TRY(check_pairs(ctx, n, guesses.data(), hi_all.data(), hi_off.data(), lo_all.data(), lo_off.data(), his.data(), los.data()));
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  FcsmPick best{};
  int best_scan = -1;
  constexpr int kChunk = 1024;
  for (int first = 0; first < n; first += kChunk) {
    const int m = std::min(kChunk, n - first);
    CoarseSearch cs;
    PairClouds pc;
    pc.hi_pts = hi_all.data();
    pc.lo_pts = lo_all.data();
    pc.hi_off = hi_off.data();
    pc.lo_off = lo_off.data();
    DL_TRY(plan_coarse(ctx, *o, first, m, his.data(), &cs));
    DL_TRY(carve_scratch(ctx, [&](Arena& a) { carve_coarse(a, pc, first, m, &cs); }));
    DL_TRY(coarse_search(ctx, *o, min_score, first, m, guesses.data(), pc, his.data(), los.data(), &cs));
    std::vector<FcsmPick> picks(m);
    DL_TRY(d2h(ctx, picks.data(), cs.d_picks, m));
    DL_TRY(sync(ctx));
    for (int k = 0; k < m; ++k) {
      result->num_candidates += picks[k].num_candidates;
      if (picks[k].found && (best_scan < 0 || picks[k].score > best.score)) {  // first of equal scores: lowest yaw step
        best = picks[k];
        best_scan = first + k;
      }
    }
  }
  if (best_scan < 0) return DL_OK;
  result->found = 1;
  result->score = best.score;
  std::memcpy(result->pose_estimate, best.pose, sizeof(best.pose));
  result->rotational_score = scores[best_scan];
  result->low_resolution_score = best.low_resolution_score;
  std::memcpy(result->offset, best.offset, sizeof(best.offset));
  result->scan_index = best_scan;
  return DL_OK;
}

int dl_constraint_search_batch(dl_context* ctx, const dl_constraint_options* options, int32_t count, const double* guesses,
                               const float* hi_pts, const int64_t* hi_off, const float* lo_pts, const int64_t* lo_off,
                               const dl_grid* const* hi_grids, const dl_grid* const* lo_grids, dl_constraint* constraints) {
  if (!ctx || !options || count < 0) return DL_ERR_ARG;
  if (count == 0) return DL_OK;
  if (!constraints) return DL_ERR_ARG;
  DL_TRY(check_pairs(ctx, count, guesses, hi_pts, hi_off, lo_pts, lo_off, hi_grids, lo_grids));
  DL_TRY(check_constraint_options(ctx, *options));
  PairClouds pc;
  pc.hi_pts = hi_pts;
  pc.lo_pts = lo_pts;
  pc.hi_off = hi_off;
  pc.lo_off = lo_off;
  return constraint_search(ctx, *options, count, guesses, pc, hi_grids, lo_grids, constraints);
}

int dl_constraint_search_exchange(dl_context* ctx, dl_comm* comm, const dl_constraint_options* options, int32_t count,
                                  int32_t capacity, const int32_t* submap_ids, const int32_t* node_ids, const double* guesses,
                                  const float* hi_pts, const int64_t* hi_off, const float* lo_pts, const int64_t* lo_off,
                                  const dl_grid* const* hi_grids, const dl_grid* const* lo_grids, dl_constraint_row* table,
                                  dl_exchange_info* info) {
  if (!ctx || !comm || !options || count < 0 || capacity < 1 || count > capacity || !table) return DL_ERR_ARG;
  if (capacity > 1024) return ctx->fail(DL_ERR_ARG, "capacity > 1024 pairs per rank and exchange: split the call");
  if (count > 0 && (!submap_ids || !node_ids)) return DL_ERR_ARG;
  if (count > 0) DL_TRY(check_pairs(ctx, count, guesses, hi_pts, hi_off, lo_pts, lo_off, hi_grids, lo_grids));
  DL_TRY(check_constraint_options(ctx, *options));
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  const int world = dl_comm_world_size(comm), rank = dl_comm_rank(comm);
  const size_t row_bytes = sizeof(dl_constraint_row), block = (size_t)capacity * row_bytes;
  DL_TRY(comm_reserve(comm, block));
  dl_constraint_row* d_send = (dl_constraint_row*)comm_send_buffer(comm);
  dl_constraint_row* d_recv = (dl_constraint_row*)comm_recv_buffer(comm);
  // padding rows: found = -1 (every int32 of the row is -1; the doubles are NaN and never read)
  DL_CUDA(ctx, cudaMemsetAsync(d_send, 0xFF, block, ctx->stream));
  if (count > 0) {
    const NlsOptions nls = to_nls_options(options->ceres_scan_matcher_3d, 2);
    const int n = count;
    CoarseSearch cs;
    PairClouds pc;
    pc.hi_pts = hi_pts;
    pc.lo_pts = lo_pts;
    pc.hi_off = hi_off;
    pc.lo_off = lo_off;
    NlsProblem* d_problems;
    NlsOutput* d_out;
    int32_t* d_ids;
    DL_TRY(plan_coarse(ctx, options->fast_correlative_scan_matcher_3d, 0, n, hi_grids, &cs));
    DL_TRY(carve_scratch(ctx, [&](Arena& a) {
      carve_coarse(a, pc, 0, n, &cs);
      d_problems = a.take<NlsProblem>(n);
      d_out = a.take<NlsOutput>(n);
      d_ids = a.take<int32_t>(2 * (size_t)n);
    }));
    DL_TRY(coarse_search(ctx, options->fast_correlative_scan_matcher_3d, (float)options->min_score, 0, n, guesses, pc,
                         hi_grids, lo_grids, &cs));
    std::vector<NlsProblem> problems(n);
    for (int k = 0; k < n; ++k) {
      NlsProblem& p = problems[k];
      std::memset(&p, 0, sizeof(p));
      p.cloud[0] = cs.hi[k];
      p.cloud[1] = cs.lo[k];
      p.count[0] = (int32_t)(hi_off[k + 1] - hi_off[k]);
      p.count[1] = (int32_t)(lo_off[k + 1] - lo_off[k]);
      p.grid[0] = hi_grids[k]->view();
      p.grid[1] = lo_grids[k]->view();
      p.initial_dev = cs.d_picks[k].pose;  // address arithmetic only
      p.enabled_dev = &cs.d_picks[k].found;
    }
    DL_TRY(h2d(ctx, d_problems, problems.data(), n));
    DL_TRY(h2d(ctx, d_ids, submap_ids, n));
    DL_TRY(h2d(ctx, d_ids + n, node_ids, n));
    DL_CUDA(ctx, cudaMemsetAsync(d_out, 0, sizeof(NlsOutput) * n, ctx->stream));
    {
      StageScope st(ctx, "loop_closure_refine");
      DL_TRY(launch_nls(ctx, nls, d_problems, n, d_out));
    }
    DL_TRY(launch_pack_constraint_rows(ctx, n, cs.d_picks, d_out, d_ids, d_ids + n, options->loop_closure_translation_weight,
                                       options->loop_closure_rotation_weight, rank, d_send));
    DL_TRY(sync(ctx));  // `problems` is pageable host memory; also keeps the search out of the collective's timing
  }
  float ms = 0.f;
  {
    StageScope st(ctx, "constraint_all_gather");
    DL_TRY(comm_all_gather(comm, d_send, d_recv, block, &ms));
  }
  DL_TRY(d2h(ctx, table, d_recv, (size_t)world * capacity));
  DL_TRY(sync(ctx));
  if (info) {
    info->bytes_sent = (int64_t)block;
    info->bytes_received = (int64_t)block * world;
    info->collective_ms = ms;
    int found = 0;
    for (int i = 0; i < world * capacity; ++i) found += table[i].found == 1;
    info->found_total = found;
  }
  return DL_OK;
}

}  // extern "C"
