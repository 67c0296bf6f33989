// RotationalScanMatcher::ComputeHistogram on the device (SURVEY 8a a13 / VERDICT "missing" 4): the histogram of horizontal
// directions between angular neighbours that LocalTrajectoryBuilder3D::InsertIntoSubmap stores with every inserted node
// (LTB:605-610) and the loop-closure matcher compares (SM/rotational_scan_matcher.cc:31-121, :159-170).
//
// The reference buckets the cloud into 0.2 m slices (std::map -> ascending slice order, points in input order), sorts each
// slice by the angle around its centroid (SortSlice, :94-121) and walks the SORTED slice (AddPointCloudSliceToHistogram,
// :63-92), which takes the centroid again, of the points SortSlice kept and in their sorted order; it adds into ONE float
// histogram. Every float sum here keeps the reference's order:
//   1. key = (slice, input index) -> bitonic sort: slices contiguous, ascending, input order inside        (whole CTA)
//   2. first centroid of a slice = sequential float sum over its points in input order, one thread per slice (:54-61)
//   3. key = (slice, atan2 of the offset from the first centroid, index); points closer than 0.2 m dropped -> sort (:94-121)
//   4. one thread per slice: exact-angle fix-up of the sort, second centroid = sequential float sum over the kept points in
//      sorted order, then the walk with the reference's `last`-point logic, one (bucket, value) event per point     (:63-92)
//   5. one thread per bucket adds its events in (slice, point) order = the order of the reference's += chain (:31-52)
// One CTA per cloud (several clouds in one launch through an argument array); the sorts run in global memory (the arrays are L2-resident: 8 B per point).
// Float parity: compiled -fmad=false, so every sqrt, division and sum is the reference's IEEE operation in the reference's
// order, and the histogram is bit-identical to the reference's except through atan2f. The device's atan2f and glibc's are
// each within a few ulps of the true angle, so only a point whose angle lies within a few ulps of another point's angle in
// its slice (the sort) or of a bucket boundary (the walk) can be decided differently. Equal angles keep input order (the
// order libstdc++'s insertion sort gives slices of at most 16 points; std::sort leaves it unspecified beyond), with -0 and +0
// equal as std::sort's operator< sees them. tests/test_gpu_rotational_histogram.py checks bit equality on clouds cleared of
// such points and, on scene clouds, that any difference comes from one.
#include <algorithm>
#include <vector>

#include "dl_internal.cuh"

namespace dl {
namespace {

constexpr int kThreads = 1024;
constexpr unsigned long long kPad = 0xFFFFFFFFFFFFFFFFull;

struct HistogramArgs {
  const float* points;  // n x 3, already rotated into the gravity-aligned frame
  int n, np2;           // np2 = n rounded up to a power of two
  int size;             // histogram buckets
  unsigned long long* keys;   // np2
  int* slice_first;     // n + 1: first sorted position of each distinct slice (compact list), then the end
  float* centroid;      // 2 per distinct slice
  int* ev_bucket;       // n
  float* ev_value;      // n
  int* counters;        // [0] number of distinct slices, [1] error
  float* histogram;     // size
};

__device__ __forceinline__ unsigned order_bits(float f) {  // monotone map float -> unsigned
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ void bitonic_sort(unsigned long long* keys, int np2) {
  for (int k = 2; k <= np2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < np2; i += kThreads) {
        const int partner = i ^ j;
        if (partner > i) {
          const unsigned long long a = keys[i], b = keys[partner];
          const bool ascending = (i & k) == 0;
          if ((a > b) == ascending) {
            keys[i] = b;
            keys[partner] = a;
          }
        }
      }
      __syncthreads();
    }
  }
}

// boundaries of the runs of equal `slice` (top 20 bits of the key) in the sorted array -> compact, ordered list of run starts.
// Every thread scans one contiguous chunk; a block-wide exclusive scan of the per-chunk run counts places them in order.
__device__ void find_slices(const HistogramArgs& a, int count) {
  __shared__ int warp_sums[kThreads / 32];
  __shared__ int total_s;
  const int chunk = (count + kThreads - 1) / kThreads;
  const int begin = min(count, (int)threadIdx.x * chunk), end = min(count, begin + chunk);
  auto starts_run = [&](int i) { return i == 0 || (a.keys[i] >> 44) != (a.keys[i - 1] >> 44); };
  int mine = 0;
  for (int i = begin; i < end; ++i) mine += starts_run(i);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int inc = mine;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int o = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc += o;
  }
  if (lane == 31) warp_sums[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    int v = warp_sums[lane];
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int o = __shfl_up_sync(0xffffffffu, v, d);
      if (lane >= d) v += o;
    }
    warp_sums[lane] = v;  // inclusive over warps
    if (lane == 31) total_s = v;
  }
  __syncthreads();
  int pos = inc - mine + (warp ? warp_sums[warp - 1] : 0);
  for (int i = begin; i < end; ++i)
    if (starts_run(i)) a.slice_first[pos++] = i;
  if (threadIdx.x == 0) {
    a.slice_first[total_s] = count;
    a.counters[0] = total_s;
  }
  __syncthreads();
}

// many == nullptr: the one cloud `one`; otherwise cloud blockIdx.x of `many`.
__global__ void __launch_bounds__(kThreads) rotational_histogram_kernel(HistogramArgs one, const HistogramArgs* __restrict__ many) {
  const HistogramArgs a = many ? many[blockIdx.x] : one;
  const float kSliceHeight = 0.2f, kMinDistance = 0.2f, kMaxDistance = 0.9f;
  const float kPi = 3.14159274101257324f;  // (float)M_PI
  // ---- 1. (slice, index) keys
  for (int i = threadIdx.x; i < a.np2; i += kThreads) {
    unsigned long long key = kPad;
    if (i < a.n) {
      const int slice = round_to_int(a.points[3 * i + 2] / kSliceHeight);
      if (slice < -(1 << 19) || slice >= (1 << 19)) a.counters[1] = 1;
      key = ((unsigned long long)(unsigned)(slice + (1 << 19)) << 44) | (unsigned long long)i;
    }
    a.keys[i] = key;
  }
  if (threadIdx.x < a.size) a.histogram[threadIdx.x] = 0.f;
  __syncthreads();
  bitonic_sort(a.keys, a.np2);
  find_slices(a, a.n);
  const int num_slices = a.counters[0];
  // ---- 2. first centroids (sequential float sums in input order, per slice)
  for (int s = threadIdx.x; s < num_slices; s += kThreads) {
    float sx = 0.f, sy = 0.f;
    const int b = a.slice_first[s], e = a.slice_first[s + 1];
    for (int k = b; k < e; ++k) {
      const int i = (int)(a.keys[k] & 0xFFFFFFFFFFFull);
      sx += a.points[3 * i];
      sy += a.points[3 * i + 1];
    }
    const float cnt = (float)(e - b);
    a.centroid[2 * s] = sx / cnt;
    a.centroid[2 * s + 1] = sy / cnt;
  }
  __syncthreads();
  // ---- 3. (slice, angle, index) keys of the points far enough from their slice's centroid
  for (int s = 0; s < num_slices; ++s) {
    const int b = a.slice_first[s], e = a.slice_first[s + 1];
    const float cx = a.centroid[2 * s], cy = a.centroid[2 * s + 1];
    for (int k = b + threadIdx.x; k < e; k += kThreads) {
      const unsigned long long key = a.keys[k];
      const int i = (int)(key & 0xFFFFFFFFFFFull);
      const float dx = a.points[3 * i] - cx, dy = a.points[3 * i + 1] - cy;
      unsigned long long out = kPad;
      if (!(sqrtf(dx * dx + dy * dy) < kMinDistance)) {
        float angle = atan2f(dy, dx);
        if (angle == 0.f) angle = 0.f;  // -0 sorts with +0 (std::sort's operator< sees them equal): input order decides
        out = ((unsigned long long)s << 44) | ((unsigned long long)(order_bits(angle) >> 8) << 20) | (unsigned long long)(k - b);
      }
      // 20 bits slice ordinal | 24 bits angle | 20 bits position inside the slice (ties and the lost low angle bits resolve
      // towards input order; std::sort leaves that order unspecified)
      a.keys[k] = out;
      a.ev_bucket[k] = i;  // position in the first sort -> point index (the second key carries the position inside the slice)
    }
  }
  __syncthreads();
  // 24 angle bits cannot order nearly equal angles: runs that tie on them are fixed up below with the exact float compare
  bitonic_sort(a.keys, a.np2);
  // ---- 4. per slice: sequential walk in sorted order
  for (int s = threadIdx.x; s < num_slices; s += kThreads) {
    const int b0 = a.slice_first[s];
    // sorted segment of slice s: find it by binary search on the leading 20 bits
    int lo = 0, hi = a.n;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if ((a.keys[mid] >> 44) < (unsigned long long)s) lo = mid + 1; else hi = mid;
    }
    const int begin = lo;
    hi = a.n;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if ((a.keys[mid] >> 44) <= (unsigned long long)s) lo = mid + 1; else hi = mid;
    }
    const int end = lo;
    if (begin >= end) continue;
    const float cx = a.centroid[2 * s], cy = a.centroid[2 * s + 1];
    auto point_of = [&](int k) { return a.ev_bucket[b0 + (int)(a.keys[k] & 0xFFFFFull)]; };
    // insertion-sort fix-up inside runs whose 24-bit angle prefix ties: exact float angle, then input order
    // (runs are short: neighbouring points of one slice rarely share 24 leading angle bits)
    for (int k = begin + 1; k < end; ++k) {
      int m = k;
      while (m > begin && ((a.keys[m] >> 20) == (a.keys[m - 1] >> 20))) {
        const int im = point_of(m), ip = point_of(m - 1);
        const float am = atan2f(a.points[3 * im + 1] - cy, a.points[3 * im] - cx);
        const float ap = atan2f(a.points[3 * ip + 1] - cy, a.points[3 * ip] - cx);
        if (am < ap) {
          const unsigned long long t = a.keys[m];
          a.keys[m] = a.keys[m - 1];
          a.keys[m - 1] = t;
          --m;
        } else {
          break;
        }
      }
    }
    // the walk's centroid: AddPointCloudSliceToHistogram takes it of the sorted slice (kept points, sorted order)
    float sx = 0.f, sy = 0.f;
    for (int k = begin; k < end; ++k) {
      const int i = point_of(k);
      sx += a.points[3 * i];
      sy += a.points[3 * i + 1];
    }
    const float wx = sx / (float)(end - begin), wy = sy / (float)(end - begin);
    int il = point_of(begin);
    float lx = a.points[3 * il], ly = a.points[3 * il + 1];
    for (int k = begin; k < end; ++k) {
      const int i = point_of(k);
      const float px = a.points[3 * i], py = a.points[3 * i + 1];
      const float dx = px - lx, dy = py - ly;
      const float ccx = px - wx, ccy = py - wy;
      const float distance = sqrtf(dx * dx + dy * dy);
      const float direction_norm = sqrtf(ccx * ccx + ccy * ccy);
      int bucket = -1;
      float value = 0.f;
      if (!(distance < kMinDistance || direction_norm < kMinDistance)) {
        if (distance > kMaxDistance) {
          lx = px; ly = py;
        } else {
          float angle = atan2f(dy, dx);
          const float dot = (dx / distance) * (ccx / direction_norm) + (dy / distance) * (ccy / direction_norm);
          value = fmaxf(0.f, 1.f - fabsf(dot));
          while (angle > kPi) angle -= kPi;
          while (angle < 0.f) angle += kPi;
          const float zero_to_one = angle / kPi;
          bucket = min(max(round_to_int((float)a.size * zero_to_one - 0.5f), 0), a.size - 1);
        }
      }
      // events are stored at the sorted position: (slice, point) order = array order
      a.ev_value[k] = value;
      reinterpret_cast<int*>(a.centroid + 2 * a.n)[k] = bucket;  // second half of the centroid buffer: bucket per sorted position
    }
  }
  __syncthreads();
  // ---- 5. per bucket: sequential float sum in (slice, point) order
  const int* ev_b = reinterpret_cast<const int*>(a.centroid + 2 * a.n);
  // number of kept points = first padded key
  __shared__ int kept;
  if (threadIdx.x == 0) {
    int lo = 0, hi = a.n;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (a.keys[mid] != kPad) lo = mid + 1; else hi = mid;
    }
    kept = lo;
  }
  __syncthreads();
  if (threadIdx.x < a.size) {
    float sum = 0.f;
    for (int k = 0; k < kept; ++k)
      if (ev_b[k] == (int)threadIdx.x) sum += a.ev_value[k];
    a.histogram[threadIdx.x] = sum;
  }
}

}  // namespace

static int64_t histogram_np2(int64_t n) {
  int64_t np2 = 64;
  while (np2 < n) np2 <<= 1;
  return np2;
}

void carve_rotational_histogram(Arena& a, int64_t n, HistogramScratch* s) {
  s->keys = a.take<unsigned long long>(histogram_np2(n));
  s->slice_first = a.take<int>(n + 1);
  s->centroid = a.take<float>(4 * (size_t)n + 4);  // 2 n centroid floats (upper bound) + n bucket ints
  s->ev_bucket = a.take<int>(n + 1);
  s->ev_value = a.take<float>(n + 1);
  s->counters = a.take<int>(2);
}

static HistogramArgs histogram_args(const HistogramScratch& s, const float* d_points, int64_t n, int size, float* d_histogram) {
  HistogramArgs h{};
  h.points = d_points;
  h.n = (int)n;
  h.np2 = (int)histogram_np2(n);
  h.size = size;
  h.keys = s.keys;
  h.slice_first = s.slice_first;
  h.centroid = s.centroid;
  h.ev_bucket = s.ev_bucket;
  h.ev_value = s.ev_value;
  h.counters = s.counters;
  h.histogram = d_histogram;
  return h;
}

// d_points: n x 3 floats on the device. d_histogram: `size` floats (size <= 1024). `s` is carved for n points.
int launch_rotational_histogram(dl_context* ctx, const HistogramScratch& s, const float* d_points, int64_t n, int size,
                                float* d_histogram, int32_t** d_error_out) {
  if (size < 1 || size > kThreads) return ctx->fail(DL_ERR_ARG, "histogram size must be in [1, 1024]");
  if (n > (1 << 20)) return ctx->fail(DL_ERR_ARG, "more than 2^20 points in a rotational histogram");
  const HistogramArgs h = histogram_args(s, d_points, n, size, d_histogram);
  DL_CUDA(ctx, cudaMemsetAsync(h.counters, 0, 2 * sizeof(int), ctx->stream));
  if (n == 0) {
    DL_CUDA(ctx, cudaMemsetAsync(d_histogram, 0, sizeof(float) * size, ctx->stream));
  } else {
    rotational_histogram_kernel<<<1, kThreads, 0, ctx->stream>>>(h, nullptr);
    DL_LAUNCH_CHECK(ctx, "rotational_histogram_kernel");
  }
  if (d_error_out) *d_error_out = h.counters + 1;
  return DL_OK;
}

size_t rotational_histograms_args_bytes(int count) { return sizeof(HistogramArgs) * (size_t)count; }

int launch_rotational_histograms(dl_context* ctx, const HistogramScratch* s, const float* const* d_points, const int64_t* n,
                                 int count, int size, float* const* d_histograms, void* d_args) {
  if (count <= 0) return DL_OK;
  if (size < 1 || size > kThreads) return ctx->fail(DL_ERR_ARG, "histogram size must be in [1, 1024]");
  std::vector<HistogramArgs> h(count);
  for (int k = 0; k < count; ++k) {
    if (n[k] < 1 || n[k] > (1 << 20)) return ctx->fail(DL_ERR_ARG, "every cloud of a histogram batch needs 1 to 2^20 points");
    h[k] = histogram_args(s[k], d_points[k], n[k], size, d_histograms[k]);
    DL_CUDA(ctx, cudaMemsetAsync(h[k].counters, 0, 2 * sizeof(int), ctx->stream));
  }
  DL_CUDA(ctx, cudaMemcpyAsync(d_args, h.data(), sizeof(HistogramArgs) * (size_t)count, cudaMemcpyHostToDevice, ctx->stream));
  rotational_histogram_kernel<<<count, kThreads, 0, ctx->stream>>>(h[0], (const HistogramArgs*)d_args);
  DL_LAUNCH_CHECK(ctx, "rotational_histogram_kernel");
  return DL_OK;
}

}  // namespace dl

// ------------------------------------------------------------------------------------------------ rotational histogram
using namespace dl;

extern "C" int dl_rotational_histogram(dl_context* ctx, const float* points, int64_t n, int32_t size, float* histogram_out) {
  if (!ctx || n < 0 || (n > 0 && !points) || !histogram_out) return DL_ERR_ARG;
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  float *d_pts, *d_hist;
  HistogramScratch hs;
  DL_TRY(carve_scratch(ctx, [&](Arena& a) {
    d_pts = a.take<float>(3 * (size_t)std::max<int64_t>(n, 1));
    d_hist = a.take<float>(std::max(size, 1));
    carve_rotational_histogram(a, n, &hs);
  }));
  DL_TRY(h2d(ctx, d_pts, points, 3 * (size_t)n));
  int32_t* d_err = nullptr;
  DL_TRY(launch_rotational_histogram(ctx, hs, d_pts, n, size, d_hist, &d_err));
  int32_t err = 0;
  DL_TRY(d2h(ctx, histogram_out, d_hist, (size_t)size));
  DL_TRY(d2h(ctx, &err, d_err, 1));
  DL_TRY(sync(ctx));
  if (err) return ctx->fail(DL_ERR_ARG, "a point lies outside +-2^19 slices of 0.2 m");
  return DL_OK;
}
