// Submap images from the device grids (include/dliom_b200.h, "submap images"): the X-ray textures of Submap3D::ToResponseProto
// (C/mapping/3d/submap_3d.cc:53-178, :253-262) and the loop detector's ProjectToCvMat (:381-464), for many (grid, pose) queries
// per call. Every query's cells are read in place from its GridView; the host waits three times per call whatever the count (once
// more when the call's device scratch has to grow), and the pool sizes are read with one 8-byte copy per query.
//
// The pipeline, all queries at once:
//   1. node_top_kernel / brick_key_kernel: every occupied brick gets the key (query, top cell, node slot); a radix sort of those
//      keys puts the bricks in HybridGrid::Iterator order (top cells, then node slots, then the brick's z-major cells), which is
//      lexicographic in (z/64, y/64, x/64, z/8 % 8, y/8 % 8, x/8 % 8, z % 8, y % 8, x % 8) of the cell index.
//   2. image_cells_kernel<false>: one CTA per sorted brick filters and transforms its 512 cells (ExtractVoxelData, :82-112):
//      count per brick, and the integer bounding box and count per query. Read-back -> image sizes.
//   3. image_cells_kernel<true>: the same cells again, written compacted in iterator order as (pixel, probability | z) pairs; a
//      stable radix sort by pixel keeps iterator order inside every pixel, so image_runs_kernel's one thread per pixel sums the
//      probabilities in the reference's order (AccumulatePixelData, :53-77) and writes the texture's or projection's bytes.
#include <cub/cub.cuh>

#include <algorithm>
#include <cmath>
#include <mutex>
#include <vector>

#include "dl_internal.cuh"
#include "dl_log_odds.h"

namespace dl {
namespace {

constexpr int kTexture = 0, kProjection = 1;
constexpr uint64_t kNoBrick = ~0ull;  // brick-key of a pool slot no node entry refers to: sorts last, yields no cells
constexpr int kKeyQueryShift = 33;    // brick key = query << 33 | top cell (< 2^24) << 9 | node slot (< 2^9)

struct ImageQuery {  // one query, on the device
  GridView grid;
  Rigidf transform;
  float inverse;  // 1.f / resolution: the reference multiplies by it (ExtractVoxelData's resolution_inverse)
  int32_t num_nodes, num_bricks;
  int64_t node_off, brick_off;
  // the image, known after the bounding-box read-back
  int64_t pixel_off;
  int32_t min_x, min_y, max_x, max_y, width;
};

struct Thresholds {
  float t[kLogOddsThresholds];
};

__global__ void node_top_kernel(const ImageQuery* qs, int32_t* node_top) {
  const ImageQuery& q = qs[blockIdx.x];
  const int64_t top_cells = (int64_t)1 << (3 * q.grid.bits);
  for (int64_t t = (int64_t)blockIdx.y * blockDim.x + threadIdx.x; t < top_cells; t += (int64_t)gridDim.y * blockDim.x) {
    const int node = q.grid.top[t];
    if (node >= 0 && node < q.num_nodes) node_top[q.node_off + node] = (int32_t)t;
  }
}

__global__ void brick_key_kernel(const ImageQuery* qs, const int32_t* node_top, uint64_t* keys, int32_t* bricks) {
  const ImageQuery& q = qs[blockIdx.x];
  const int64_t entries = (int64_t)q.num_nodes * 512;
  for (int64_t e = (int64_t)blockIdx.y * blockDim.x + threadIdx.x; e < entries; e += (int64_t)gridDim.y * blockDim.x) {
    const int32_t t = node_top[q.node_off + (e >> 9)];
    const int brick = q.grid.nodes[e];
    if (t < 0 || brick < 0 || brick >= q.num_bricks) continue;
    keys[q.brick_off + brick] = ((uint64_t)blockIdx.x << kKeyQueryShift) | ((uint64_t)t << 9) | (uint64_t)(e & 511);
    bricks[q.brick_off + brick] = brick;
  }
}

__device__ __forceinline__ int64_t pixel_of(const ImageQuery& q, int mode, int ix, int iy) {
  if (mode == kTexture) return (int64_t)(q.max_x - ix) * q.width + (q.max_y - iy);  // AccumulatePixelData :65-67
  return (int64_t)(iy - q.min_y) * q.width + (ix - q.min_x);                        // ProjectToCvMat :443-445
}

// One CTA of 512 threads per sorted brick, one cell per thread. kEmit = false: per-brick counts, per-query bounding box and
// count (bbox: 8 ints per query, min x y z, max x y z, count). kEmit = true: the brick's cells at brick_first[brick] onwards.
template <bool kEmit>
__global__ void __launch_bounds__(512) image_cells_kernel(const ImageQuery* qs, const uint64_t* brick_keys, const int32_t* bricks,
                                                          int mode, int32_t* bbox, int32_t* brick_count,
                                                          const int32_t* brick_first, uint64_t* cell_key, uint64_t* cell_val) {
  const uint64_t key = brick_keys[blockIdx.x];
  if (key == kNoBrick) {
    if (!kEmit && threadIdx.x == 0) brick_count[blockIdx.x] = 0;
    return;
  }
  const int qi = (int)(key >> kKeyQueryShift);
  const ImageQuery& q = qs[qi];
  const int t = (int)((key >> 9) & 0xFFFFFF), l = (int)(key & 511), c = threadIdx.x;
  const uint16_t value = q.grid.bricks[(size_t)bricks[blockIdx.x] * 512 + c];
  const float probability = value_to_probability(value);
  const bool valid = value != 0 && !(probability < 0.501f);  // kXrayObstructedCellProbabilityLimit
  int ix = 0, iy = 0, iz = 0;
  if (valid) {
    const int bits = q.grid.bits, mask = (1 << bits) - 1, half = 32 << bits;
    const int x = (t & mask) * 64 + (l & 7) * 8 + (c & 7) - half;
    const int y = ((t >> bits) & mask) * 64 + ((l >> 3) & 7) * 8 + ((c >> 3) & 7) - half;
    const int z = (t >> (2 * bits)) * 64 + (l >> 6) * 8 + (c >> 6) - half;
    const float r = q.grid.resolution;  // GetCenterOfCell: index.cast<float>() * resolution
    const Vec3f p = apply(q.transform, Vec3f{(float)x * r, (float)y * r, (float)z * r});
    ix = round_to_int(p.x * q.inverse);
    iy = round_to_int(p.y * q.inverse);
    iz = round_to_int(p.z * q.inverse);
  }
  if (!kEmit) {
    __shared__ int s[7];
    if (c < 3) s[c] = INT_MAX;
    else if (c < 6) s[c] = INT_MIN;
    else if (c == 6) s[c] = 0;
    __syncthreads();
    if (valid) {
      atomicMin(&s[0], ix); atomicMin(&s[1], iy); atomicMin(&s[2], iz);
      atomicMax(&s[3], ix); atomicMax(&s[4], iy); atomicMax(&s[5], iz);
      atomicAdd(&s[6], 1);
    }
    __syncthreads();
    if (c == 0) {
      brick_count[blockIdx.x] = s[6];
      if (s[6] > 0) {
        int32_t* b = bbox + 8 * qi;
        atomicMin(b + 0, s[0]); atomicMin(b + 1, s[1]); atomicMin(b + 2, s[2]);
        atomicMax(b + 3, s[3]); atomicMax(b + 4, s[4]); atomicMax(b + 5, s[5]);
        atomicAdd(b + 6, s[6]);
      }
    }
  } else {
    using Scan = cub::BlockScan<int, 512>;
    __shared__ typename Scan::TempStorage scan;
    int rank;
    Scan(scan).ExclusiveSum(valid ? 1 : 0, rank);
    if (valid) {
      const int64_t at = (int64_t)brick_first[blockIdx.x] + rank;
      cell_key[at] = (uint64_t)(q.pixel_off + pixel_of(q, mode, ix, iy));
      cell_val[at] = ((uint64_t)__float_as_uint(probability) << 32) | (uint32_t)iz;
    }
  }
}

// One thread per pixel run of the pixel-sorted cells: PixelData over the run in iterator order, then the pixel's bytes.
__global__ void image_runs_kernel(const uint64_t* keys, const uint64_t* vals, int64_t n, int mode, Thresholds th, uint8_t* out) {
  __shared__ float table[kLogOddsThresholds];
  for (int k = threadIdx.x; k < kLogOddsThresholds; k += blockDim.x) table[k] = th.t[k];
  __syncthreads();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || (i > 0 && keys[i - 1] == keys[i])) return;
  const uint64_t pixel = keys[i];
  int count = 0, min_z = INT_MAX, max_z = INT_MIN;
  float sum = 0.f, max_probability = 0.5f;
  for (int64_t j = i; j < n && keys[j] == pixel; ++j) {
    const float probability = __uint_as_float((uint32_t)(vals[j] >> 32));
    const int z = (int)(uint32_t)vals[j];
    ++count;
    min_z = min(min_z, z);
    max_z = max(max_z, z);
    sum += probability;
    max_probability = max_probability < probability ? probability : max_probability;  // std::max
  }
  if (mode == kProjection) {  // ProjectToCvMat :455-461: int -> uchar wraps
    out[pixel] = (uint8_t)round_to_int((sum - kMinProbability) * (255.f / (kMaxProbability - kMinProbability)));
    return;
  }
  // ComputePixelValues (:116-146); count > 0 here
  const float z_difference = (float)(max_z - min_z);
  if (z_difference < 3.f) return;  // (0, 0), the buffer's initial bytes
  const float free_space = fmaxf(z_difference - (float)count, 0.f);
  const float free_space_weight = 0.15f * free_space;
  const float total_weight = (float)count + free_space_weight;
  const float free_space_probability = 1.f - max_probability;
  float average = (sum + free_space_probability * free_space_weight) / total_weight;
  if (average > kMaxProbability) average = kMaxProbability;  // ClampProbability
  if (average < kMinProbability) average = kMinProbability;
  const int delta = 128 - log_odds_integer_from_table(table, average);
  const uint8_t alpha = delta > 0 ? 0 : -delta;
  const uint8_t value = delta > 0 ? delta : 0;
  out[2 * pixel] = value;
  out[2 * pixel + 1] = (value || alpha) ? alpha : 1;
}

const Thresholds& log_odds_thresholds() {
  static Thresholds th;
  static std::once_flag once;
  std::call_once(once, [] { build_log_odds_thresholds(th.t); });
  return th;
}

// The float rotation of ProjectToCvMat (:384-390): Rigid3d::Rotation(q).cast<float>() with its yaw removed,
// Embed3D(Rigid2d::Rotation(-yaw)).cast<float>() * that, as Rigid3f products.
Rigidf projection_transform(const Rigidd& pose) {
  const Rigidf rotation{{0.f, 0.f, 0.f}, {(float)pose.q.w, (float)pose.q.x, (float)pose.q.y, (float)pose.q.z}};
  const Vec3d direction = rotate(pose.q, Vec3d{1.0, 0.0, 0.0});  // GetYaw (transform.h:42-47)
  const double yaw = std::atan2(direction.y, direction.x);
  const double half = 0.5 * -yaw;  // Quaternion(AngleAxis(-yaw, UnitZ))
  const double s = std::sin(half);
  const Rigidd inverse_yaw{{0.0, 0.0, 0.0}, {std::cos(half), s * 0.0, s * 0.0, s * 1.0}};
  return compose(to_float(inverse_yaw), rotation);
}

int bits_for(int64_t n) {  // least b >= 1 with n <= 2^b
  int b = 1;
  while (((int64_t)1 << b) < n) ++b;
  return b;
}

struct ImageResult {
  int32_t width, height;
  int32_t max_x, max_y, min_x, min_y;
  int64_t offset;  // byte offset in the call's output
};

// Both entry points: mode kTexture or kProjection. results[k] is filled for every query; *num_bytes is the total output size.
int submap_images(dl_context* ctx, int mode, int32_t count, const dl_submap_image_query* queries, std::vector<ImageResult>& results,
                  int64_t capacity, uint8_t* out, int64_t* num_bytes) {
  if (!ctx || count < 0 || (count > 0 && !queries) || !num_bytes || capacity < 0) return DL_ERR_ARG;
  for (int k = 0; k < count; ++k) {
    const dl_grid* g = queries[k].grid;
    if (!g) return ctx->fail(DL_ERR_ARG, "submap image query without a grid");
    if (g->structure_dirty || !g->d_counters.get()) return ctx->fail(DL_ERR_ARG, "dl_grid_sync not called after dl_grid_set_cells");
    if (g->ctx->device != ctx->device) return ctx->fail(DL_ERR_ARG, "submap image query of a grid on another device");
  }
  // the pinned block below holds a submitted front-end batch's staged results until dl_frontend_collect
  if (ctx->in_flight) return ctx->fail(DL_ERR_ARG, "a submitted batch is in flight on this context: call dl_frontend_collect first");
  results.assign(count, ImageResult{0, 0, 0, 0, 0, 0, 0});
  *num_bytes = 0;
  if (count == 0) return DL_OK;
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  StageScope stage(ctx, mode == kTexture ? "submap_textures" : "submap_projections");

  // 1. the pools' sizes: a grid the device inserter grew is ahead of its host mirror
  DL_TRY(ctx->reserve_pinned((size_t)count * 8 * sizeof(int32_t)));
  int32_t* h_words = (int32_t*)ctx->h_pinned.get();
  for (int k = 0; k < count; ++k)
    DL_CUDA(ctx, cudaMemcpyAsync(h_words + 2 * k, queries[k].grid->d_counters.get(), 2 * sizeof(int32_t), cudaMemcpyDeviceToHost,
                                 ctx->stream));
  DL_CUDA(ctx, ctx->wait_stream());
  std::vector<ImageQuery> qs(count);
  int64_t nodes = 0, bricks = 0, max_top = 0, max_entries = 0;
  for (int k = 0; k < count; ++k) {
    const dl_grid* g = queries[k].grid;
    const Rigidd pose = pose_from7(queries[k].pose);
    ImageQuery& q = qs[k];
    q = ImageQuery{};
    q.grid = g->view();
    q.transform = mode == kTexture ? to_float(pose) : projection_transform(pose);
    q.inverse = 1.f / g->resolution;
    q.num_nodes = h_words[2 * k];
    q.num_bricks = h_words[2 * k + 1];
    q.node_off = nodes;
    q.brick_off = bricks;
    nodes += q.num_nodes;
    bricks += q.num_bricks;
    max_top = std::max<int64_t>(max_top, (int64_t)1 << (3 * g->bits));
    max_entries = std::max<int64_t>(max_entries, (int64_t)q.num_nodes * 512);
  }
  // brick_first counts cells in int32: at most 512 per brick
  if (bricks >= (1 << 22)) return ctx->fail(DL_ERR_ARG, "submap images: more than 2^22 bricks in one call");
  const int num_bricks = (int)std::max<int64_t>(bricks, 1);

  // 2. sorted bricks, per-brick counts, bounding boxes
  const int brick_end_bit = kKeyQueryShift + bits_for(count);
  size_t sort_bricks_bytes = 0, scan_bytes = 0;
  DL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(nullptr, sort_bricks_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                                               (const int32_t*)nullptr, (int32_t*)nullptr, num_bricks, 0, brick_end_bit, ctx->stream));
  DL_CUDA(ctx, cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (const int32_t*)nullptr, (int32_t*)nullptr, num_bricks + 1,
                                             ctx->stream));
  ImageQuery* d_qs;
  int32_t *d_node_top, *d_bricks_in, *d_bricks, *d_bbox, *d_brick_count, *d_brick_first;
  uint64_t *d_keys_in, *d_keys;
  void *d_sort_bricks, *d_scan;
  auto carve_a = [&](Arena& a) {
    d_qs = a.take<ImageQuery>(count);
    d_node_top = a.take<int32_t>(std::max<int64_t>(nodes, 1));
    d_keys_in = a.take<uint64_t>(num_bricks);
    d_bricks_in = a.take<int32_t>(num_bricks);
    d_keys = a.take<uint64_t>(num_bricks);
    d_bricks = a.take<int32_t>(num_bricks);
    d_sort_bricks = a.take<char>(sort_bricks_bytes);
    d_bbox = a.take<int32_t>(8 * (size_t)count);
    d_brick_count = a.take<int32_t>(num_bricks + 1);
    d_brick_first = a.take<int32_t>(num_bricks + 1);
    d_scan = a.take<char>(scan_bytes);
  };
  Arena counted_a(nullptr);  // the bytes phase 4 must keep
  carve_a(counted_a);
  DL_TRY(carve_scratch(ctx, carve_a));
  DL_CUDA(ctx, cudaMemcpyAsync(d_qs, qs.data(), count * sizeof(ImageQuery), cudaMemcpyHostToDevice, ctx->stream));
  DL_CUDA(ctx, cudaMemsetAsync(d_node_top, 0xFF, std::max<int64_t>(nodes, 1) * sizeof(int32_t), ctx->stream));
  DL_CUDA(ctx, cudaMemsetAsync(d_keys_in, 0xFF, (size_t)num_bricks * sizeof(uint64_t), ctx->stream));
  DL_CUDA(ctx, cudaMemsetAsync(d_bricks_in, 0, (size_t)num_bricks * sizeof(int32_t), ctx->stream));
  std::vector<int32_t> bbox_init(8 * (size_t)count);
  for (int k = 0; k < count; ++k) {
    int32_t* b = bbox_init.data() + 8 * k;
    b[0] = b[1] = b[2] = INT_MAX;
    b[3] = b[4] = b[5] = INT_MIN;
    b[6] = b[7] = 0;
  }
  DL_CUDA(ctx, cudaMemcpyAsync(d_bbox, bbox_init.data(), bbox_init.size() * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
  const int top_blocks = (int)std::min<int64_t>((max_top + 255) / 256, 1024);
  node_top_kernel<<<dim3(count, std::max(top_blocks, 1)), 256, 0, ctx->stream>>>(d_qs, d_node_top);
  DL_LAUNCH_CHECK(ctx, "node_top_kernel");
  const int entry_blocks = (int)std::min<int64_t>((max_entries + 255) / 256, 4096);
  brick_key_kernel<<<dim3(count, std::max(entry_blocks, 1)), 256, 0, ctx->stream>>>(d_qs, d_node_top, d_keys_in, d_bricks_in);
  DL_LAUNCH_CHECK(ctx, "brick_key_kernel");
  DL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(d_sort_bricks, sort_bricks_bytes, d_keys_in, d_keys, d_bricks_in, d_bricks,
                                               num_bricks, 0, brick_end_bit, ctx->stream));
  DL_LAUNCH_CHECK(ctx, "image brick sort");
  image_cells_kernel<false><<<num_bricks, 512, 0, ctx->stream>>>(d_qs, d_keys, d_bricks, mode, d_bbox, d_brick_count, nullptr,
                                                                 nullptr, nullptr);
  DL_LAUNCH_CHECK(ctx, "image_cells_kernel<count>");
  DL_CUDA(ctx, cub::DeviceScan::ExclusiveSum(d_scan, scan_bytes, d_brick_count, d_brick_first, num_bricks + 1, ctx->stream));
  DL_LAUNCH_CHECK(ctx, "image cell scan");
  DL_CUDA(ctx, cudaMemcpyAsync(h_words, d_bbox, 8 * (size_t)count * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
  DL_CUDA(ctx, ctx->wait_stream());

  // 3. image sizes
  int64_t pixels = 0, cells = 0;
  const int bytes_per_pixel = mode == kTexture ? 2 : 1;
  for (int k = 0; k < count; ++k) {
    const int32_t* b = h_words + 8 * k;
    ImageQuery& q = qs[k];
    ImageResult& r = results[k];
    q.pixel_off = pixels;
    if (b[6] == 0) continue;  // no obstructed cell: 0 x 0
    cells += b[6];
    q.min_x = b[0]; q.min_y = b[1]; q.max_x = b[3]; q.max_y = b[4];
    r.min_x = b[0]; r.min_y = b[1]; r.max_x = b[3]; r.max_y = b[4];
    if (mode == kTexture) {
      r.width = b[4] - b[1] + 1;
      r.height = b[3] - b[0] + 1;
    } else {
      r.width = b[3] - b[0] + 1;
      r.height = b[4] - b[1] + 1;
    }
    q.width = r.width;
    r.offset = pixels * bytes_per_pixel;
    pixels += (int64_t)r.width * r.height;
  }
  *num_bytes = pixels * bytes_per_pixel;
  if (!out) return DL_OK;
  if (capacity < *num_bytes) return ctx->fail(DL_ERR_ARG, "submap images: output capacity below the images' size");
  if (pixels == 0) return DL_OK;

  // 4. cells in iterator order -> sorted by pixel (stable) -> one thread per pixel
  const int n = (int)cells;
  const int pixel_end_bit = bits_for(pixels);
  size_t sort_cells_bytes = 0;
  DL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(nullptr, sort_cells_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                                               (const uint64_t*)nullptr, (uint64_t*)nullptr, n, 0, pixel_end_bit, ctx->stream));
  uint64_t *d_cell_key_in, *d_cell_val_in, *d_cell_key, *d_cell_val;
  void* d_sort_cells;
  uint8_t* d_out;
  auto carve_b = [&](Arena& a) {
    carve_a(a);
    d_cell_key_in = a.take<uint64_t>(n);
    d_cell_val_in = a.take<uint64_t>(n);
    d_cell_key = a.take<uint64_t>(n);
    d_cell_val = a.take<uint64_t>(n);
    d_sort_cells = a.take<char>(sort_cells_bytes);
    d_out = a.take<uint8_t>(*num_bytes);
  };
  Arena counted_b(nullptr);
  carve_b(counted_b);
  // the call's scratch bytes in use so far are kept when it has to grow (reserve_device would drop them)
  if (counted_b.off > ctx->d_scratch.cap) DL_TRY(grow(ctx, ctx->d_scratch, counted_b.off + counted_b.off / 4, counted_a.off));
  Arena arena(ctx->d_scratch.get());
  carve_b(arena);
  DL_CUDA(ctx, cudaMemcpyAsync(d_qs, qs.data(), count * sizeof(ImageQuery), cudaMemcpyHostToDevice, ctx->stream));
  image_cells_kernel<true><<<num_bricks, 512, 0, ctx->stream>>>(d_qs, d_keys, d_bricks, mode, nullptr, nullptr, d_brick_first,
                                                                d_cell_key_in, d_cell_val_in);
  DL_LAUNCH_CHECK(ctx, "image_cells_kernel<emit>");
  DL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(d_sort_cells, sort_cells_bytes, d_cell_key_in, d_cell_key, d_cell_val_in, d_cell_val,
                                               n, 0, pixel_end_bit, ctx->stream));
  DL_LAUNCH_CHECK(ctx, "image cell sort");
  // the bytes of a pixel without cells: texture (0, 0); projection lround((0 - 0.1f) * 318.75f) = -32 -> 224
  DL_CUDA(ctx, cudaMemsetAsync(d_out, mode == kTexture ? 0 : 224, (size_t)*num_bytes, ctx->stream));
  image_runs_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(d_cell_key, d_cell_val, n, mode, log_odds_thresholds(), d_out);
  DL_LAUNCH_CHECK(ctx, "image_runs_kernel");
  DL_CUDA(ctx, cudaMemcpyAsync(out, d_out, (size_t)*num_bytes, cudaMemcpyDeviceToHost, ctx->stream));
  DL_CUDA(ctx, ctx->wait_stream());
  return DL_OK;
}

}  // namespace
}  // namespace dl

using namespace dl;

extern "C" {

int dl_submap_textures(dl_context* ctx, int32_t count, const dl_submap_image_query* queries, dl_submap_texture* textures,
                       int64_t capacity, uint8_t* cells, int64_t* num_bytes) {
  if (!ctx || (count > 0 && !textures)) return DL_ERR_ARG;
  std::vector<ImageResult> rs;
  const int st = submap_images(ctx, kTexture, count, queries, rs, capacity, cells, num_bytes);
  if (st != DL_OK) return st;
  for (int k = 0; k < count; ++k) {
    dl_submap_texture& t = textures[k];
    const float resolution = queries[k].grid->resolution;
    t.resolution = resolution;
    t.width = rs[k].width;
    t.height = rs[k].height;
    t.reserved = 0;
    t.offset = rs[k].offset;
    if (rs[k].width == 0) {
      std::fill(t.slice_pose, t.slice_pose + 7, 0.0);
      continue;
    }
    // global_submap_pose.inverse() * Translation(max_x * resolution, max_y * resolution, global z): float products (:173-177)
    const Rigidd global = pose_from7(queries[k].pose);
    const Rigidd translation{{(double)(rs[k].max_x * resolution), (double)(rs[k].max_y * resolution), global.t.z},
                             {1.0, 0.0, 0.0, 0.0}};
    pose_to7(compose(inverse(global), translation), t.slice_pose);
  }
  return DL_OK;
}

int dl_submap_projections(dl_context* ctx, int32_t count, const dl_submap_image_query* queries, dl_submap_projection* projections,
                          int64_t capacity, uint8_t* pixels, int64_t* num_bytes) {
  if (!ctx || (count > 0 && !projections)) return DL_ERR_ARG;
  std::vector<ImageResult> rs;
  const int st = submap_images(ctx, kProjection, count, queries, rs, capacity, pixels, num_bytes);
  if (st != DL_OK) return st;
  for (int k = 0; k < count; ++k) {
    dl_submap_projection& p = projections[k];
    const double resolution = queries[k].grid->resolution;
    p.resolution = queries[k].grid->resolution;
    p.width = rs[k].width;
    p.height = rs[k].height;
    p.reserved = 0;
    p.offset = rs[k].offset;
    p.ox = rs[k].width == 0 ? 0.0 : rs[k].min_x * resolution;  // ox = min_index.x() * resolution (a double)
    p.oy = rs[k].width == 0 ? 0.0 : rs[k].min_y * resolution;
  }
  return DL_OK;
}

}  // extern "C"
