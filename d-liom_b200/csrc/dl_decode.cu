// Wire format -> TimedPointCloud rows in the tracking frame (SURVEY 8f-5): SensorBridge::HandlePointCloud2Message's
// per-sensor-type loops (cartographer_ros/sensor_bridge.cc:176-240) + HandleRangefinder's TransformTimedPointCloud
// (:286-300, cartographer/sensor/point_cloud.cc:35-46) on the raw sensor_msgs/PointCloud2 bytes, so a driver's message can
// be uploaded as it arrives and decoded where the front end reads it (the 16-byte rows are dl_frontend_match_batch_dev's
// input layout). NaN / Inf points are dropped in order: tile counts -> per-message prefix -> decode + transform + scatter.
//
// HBM-bound byte work: reads point_step bytes per point (22-48 for the drivers the reference knows) twice, writes 16 per
// kept point. Fields may sit at any byte offset (the velodyne driver packs its point into 22 bytes), so they are assembled
// from bytes unless the layout is 4-byte aligned.
#include <cstdint>

#include "dl_internal.cuh"

namespace dl {
namespace {

constexpr int kBlock = 256;

template <typename T>
__device__ __forceinline__ T read_field(const uint8_t* p, bool aligned) {
  T v;
  if (aligned) {
    v = *reinterpret_cast<const T*>(p);
  } else {
    uint8_t* b = reinterpret_cast<uint8_t*>(&v);
#pragma unroll
    for (int i = 0; i < (int)sizeof(T); ++i) b[i] = p[i];
  }
  return v;
}

__device__ __forceinline__ bool finite3(float x, float y, float z) {
  return !(isnan(x) || isnan(y) || isnan(z) || isinf(x) || isinf(y) || isinf(z));  // sensor_bridge.h:100-107
}

// rel_time_last (a double in every branch of the reference) from the LAST point of the message, valid or not
__device__ __forceinline__ double time_of_last(const DecodeArgs& a) {
  if (a.n <= 0) return 0.;
  const uint8_t* p = a.data + (size_t)(a.n - 1) * a.point_step + a.offset_time;
  const bool al = a.time_aligned;
  if (a.time_type == DL_TIME_FLOAT32_SECONDS) return (double)read_field<float>(p, al);
  if (a.time_type == DL_TIME_UINT32_NANOSECONDS) return (double)((float)read_field<uint32_t>(p, al) * 1e-9f);
  if (a.time_type == DL_TIME_FLOAT64_SECONDS) return read_field<double>(p, al);
  return 0.;
}

__global__ void __launch_bounds__(kBlock) decode_count_kernel(DecodeArgs a) {
  const int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  bool ok = false;
  if (i < a.n) {
    const uint8_t* p = a.data + (size_t)i * a.point_step;
    ok = finite3(read_field<float>(p + a.offset_x, a.xyz_aligned), read_field<float>(p + a.offset_y, a.xyz_aligned),
                 read_field<float>(p + a.offset_z, a.xyz_aligned));
  }
  const int c = __syncthreads_count(ok);
  if (threadIdx.x == 0) a.tile_counts[blockIdx.x] = c;
}

// exclusive prefix of the tile counts in place (one CTA), total -> *num_out, stamp offset -> *stamp_offset
__global__ void __launch_bounds__(kBlock) decode_prefix_kernel(DecodeArgs a, int tiles) {
  __shared__ int warp_sums[kBlock / 32];
  __shared__ int carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < tiles; base += kBlock) {
    const int t = base + threadIdx.x;
    const int v = t < tiles ? a.tile_counts[t] : 0;
    int inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int o = __shfl_up_sync(0xffffffffu, inc, d);
      if (lane >= d) inc += o;
    }
    if (lane == 31) warp_sums[warp] = inc;
    __syncthreads();
    int before = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kBlock / 32; ++w) {
      if (w < warp) before += warp_sums[w];
      total += warp_sums[w];
    }
    if (t < tiles) a.tile_counts[t] = carry + before + inc - v;
    __syncthreads();
    if (threadIdx.x == 0) carry += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    *a.num_out = carry;
    const double last = time_of_last(a);
    *a.stamp_offset = (a.time_type == DL_TIME_FLOAT32_SECONDS || a.time_type == DL_TIME_UINT32_NANOSECONDS) ? last : 0.;
  }
}

__global__ void __launch_bounds__(kBlock) decode_scatter_kernel(DecodeArgs a) {
  __shared__ int warp_counts[kBlock / 32];
  const int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float x = 0.f, y = 0.f, z = 0.f, t = 0.f;
  bool ok = false;
  if (i < a.n) {
    const uint8_t* p = a.data + (size_t)i * a.point_step;
    x = read_field<float>(p + a.offset_x, a.xyz_aligned);
    y = read_field<float>(p + a.offset_y, a.xyz_aligned);
    z = read_field<float>(p + a.offset_z, a.xyz_aligned);
    ok = finite3(x, y, z);
    if (ok && a.time_type != DL_TIME_NONE) {
      const double last = time_of_last(a);  // same few bytes for every thread: cache-resident
      const uint8_t* q = p + a.offset_time;
      // Eigen::Vector4f(x, y, z, <double expression>): the difference is formed in double and narrowed to float
      if (a.time_type == DL_TIME_FLOAT32_SECONDS) t = (float)((double)read_field<float>(q, a.time_aligned) - last);
      if (a.time_type == DL_TIME_UINT32_NANOSECONDS) t = (float)((double)((float)read_field<uint32_t>(q, a.time_aligned) * 1e-9f) - last);
      if (a.time_type == DL_TIME_FLOAT64_SECONDS) t = (float)(read_field<double>(q, a.time_aligned) - last);
    }
  }
  const unsigned ballot = __ballot_sync(0xffffffffu, ok);
  if (lane == 0) warp_counts[warp] = __popc(ballot);
  __syncthreads();
  if (!ok) return;
  int pos = a.tile_counts[blockIdx.x];
  for (int w = 0; w < warp; ++w) pos += warp_counts[w];
  pos += __popc(ballot & ((1u << lane) - 1));
  const Vec3f q = apply(a.sensor_to_tracking, Vec3f{x, y, z});  // transform * point.head<3>()
  reinterpret_cast<float4*>(a.rows_out)[pos] = make_float4(q.x, q.y, q.z, t);
}

}  // namespace

int launch_decode_point_cloud2(dl_context* ctx, const DecodeArgs& a) {
  const int tiles = (int)((a.n + kBlock - 1) / kBlock);
  if (tiles > 0) {
    decode_count_kernel<<<tiles, kBlock, 0, ctx->stream>>>(a);
    DL_LAUNCH_CHECK(ctx, "decode_count_kernel");
  }
  decode_prefix_kernel<<<1, kBlock, 0, ctx->stream>>>(a, tiles);
  DL_LAUNCH_CHECK(ctx, "decode_prefix_kernel");
  if (tiles > 0) {
    decode_scatter_kernel<<<tiles, kBlock, 0, ctx->stream>>>(a);
    DL_LAUNCH_CHECK(ctx, "decode_scatter_kernel");
  }
  return DL_OK;
}

}  // namespace dl

// ------------------------------------------------------------------------------------------------ decode
using namespace dl;

namespace {
int decode_common(dl_context* ctx, const dl_point_cloud2_layout* l, const void* data_host, const void* data_dev, int64_t n,
                  const double* sensor_to_tracking, float* rows_host, float* rows_dev, int64_t* num_rows_out,
                  double* stamp_offset_seconds) {
  if (!ctx || !l || !sensor_to_tracking || !num_rows_out || !stamp_offset_seconds || n < 0 || n >= (1ll << 31)) return DL_ERR_ARG;
  const int time_bytes = l->time_type == DL_TIME_FLOAT64_SECONDS ? 8 : (l->time_type == DL_TIME_NONE ? 0 : 4);
  if (l->time_type < DL_TIME_NONE || l->time_type > DL_TIME_FLOAT64_SECONDS) return ctx->fail(DL_ERR_ARG, "unknown time_type");
  if (l->point_step < 12 || l->offset_x < 0 || l->offset_y < 0 || l->offset_z < 0 || l->offset_x + 4 > l->point_step ||
      l->offset_y + 4 > l->point_step || l->offset_z + 4 > l->point_step ||
      (time_bytes && (l->offset_time < 0 || l->offset_time + time_bytes > l->point_step)))
    return ctx->fail(DL_ERR_ARG, "field offsets do not fit point_step");
  *num_rows_out = 0;
  *stamp_offset_seconds = 0.;
  if (n == 0) return DL_OK;
  if ((!data_host && !data_dev) || (!rows_host && !rows_dev)) return DL_ERR_ARG;
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t bytes = (size_t)n * l->point_step;
  const size_t tiles = (size_t)((n + 255) / 256);
  DecodeArgs d{};
  uint8_t* up = nullptr;
  DL_TRY(carve_scratch(ctx, [&](Arena& a) {
    if (data_host) up = a.take<uint8_t>(bytes);
    d.rows_out = rows_host ? a.take<float>((size_t)n * 4) : rows_dev;
    d.tile_counts = a.take<int32_t>(tiles);
    d.num_out = a.take<int32_t>(1);
    d.stamp_offset = a.take<double>(1);
  }));
  if (data_host) {
    DL_TRY(h2d(ctx, up, (const uint8_t*)data_host, bytes));
    d.data = up;
  } else {
    d.data = (const uint8_t*)data_dev;
  }
  if (((uintptr_t)d.rows_out & 15) != 0) return ctx->fail(DL_ERR_ARG, "rows_out must be 16-byte aligned");
  d.n = n;
  d.point_step = l->point_step; d.offset_x = l->offset_x; d.offset_y = l->offset_y; d.offset_z = l->offset_z;
  d.offset_time = l->offset_time; d.time_type = l->time_type;
  const bool base4 = ((uintptr_t)d.data & 3) == 0 && l->point_step % 4 == 0;
  d.xyz_aligned = base4 && l->offset_x % 4 == 0 && l->offset_y % 4 == 0 && l->offset_z % 4 == 0;
  d.time_aligned = time_bytes == 8 ? (((uintptr_t)d.data & 7) == 0 && l->point_step % 8 == 0 && l->offset_time % 8 == 0)
                                   : (base4 && l->offset_time % 4 == 0);
  d.sensor_to_tracking = to_float(pose_from7(sensor_to_tracking));  // sensor_to_tracking->cast<float>()
  DL_TRY(launch_decode_point_cloud2(ctx, d));
  int32_t kept = 0;
  DL_TRY(d2h(ctx, &kept, d.num_out, 1));
  DL_TRY(d2h(ctx, stamp_offset_seconds, d.stamp_offset, 1));
  DL_TRY(sync(ctx));
  *num_rows_out = kept;
  if (rows_host && kept > 0) {
    DL_TRY(d2h(ctx, rows_host, d.rows_out, (size_t)kept * 4));
    DL_TRY(sync(ctx));
  }
  return DL_OK;
}
}  // namespace

extern "C" {

int dl_decode_point_cloud2(dl_context* ctx, const dl_point_cloud2_layout* layout, const void* data, int64_t num_points,
                           const double* sensor_to_tracking, float* rows_out, int64_t* num_rows_out, double* stamp_offset_seconds) {
  return decode_common(ctx, layout, data, nullptr, num_points, sensor_to_tracking, rows_out, nullptr, num_rows_out, stamp_offset_seconds);
}
int dl_decode_point_cloud2_dev(dl_context* ctx, const dl_point_cloud2_layout* layout, const void* data_dev, int64_t num_points,
                               const double* sensor_to_tracking, float* rows_out_dev, int64_t* num_rows_out,
                               double* stamp_offset_seconds) {
  return decode_common(ctx, layout, nullptr, data_dev, num_points, sensor_to_tracking, nullptr, rows_out_dev, num_rows_out,
                       stamp_offset_seconds);
}

}  // extern "C"
