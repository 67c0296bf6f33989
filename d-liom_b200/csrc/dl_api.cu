// C-ABI of libdliom_b200.so (declared in include/dliom_b200.h): contexts, the device grid mirror, and the host
// orchestration of the kernels in dl_voxel.cu / dl_rtcsm.cu / dl_nls.cu / dl_frontend.cu.
// There is deliberately no CPU implementation of anything here: without a CUDA device every call fails.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <climits>
#include <cstring>
#include <functional>
#include <mutex>
#include <new>

#include "dl_internal.cuh"
#include "dl_pipeline.cuh"

using namespace dl;

// ------------------------------------------------------------------------------------------------ context
int dl_context::reserve_device(size_t bytes) {
  if (in_flight) return fail(DL_ERR_ARG, "a submitted batch is in flight on this context: call dl_frontend_collect first");
  if (bytes <= d_scratch.cap) return DL_OK;
  return grow(this, d_scratch, bytes + bytes / 4);
}
int dl_context::reserve_pinned(size_t bytes) {
  if (bytes <= h_pinned.cap) return DL_OK;
  return grow(this, h_pinned, bytes + bytes / 4);
}

int dl_context::stage_id(const char* name) {
  for (size_t i = 0; i < stage_names.size(); ++i)
    if (stage_names[i] == name) return (int)i;
  stage_names.push_back(name);
  stage_ms.push_back(0.0);
  stage_calls.push_back(0);
  return (int)stage_names.size() - 1;
}
cudaEvent_t dl_context::take_event() {
  if (!event_pool.empty()) {
    cudaEvent_t e = event_pool.back();
    event_pool.pop_back();
    return e;
  }
  cudaEvent_t e;
  cudaEventCreate(&e);
  return e;
}

namespace {
thread_local std::string g_create_error;

int64_t next_pow2(int64_t v) {
  int64_t p = 64;
  while (p < v) p <<= 1;
  return p;
}

}  // namespace

extern "C" {

static cudaError_t create_high_priority_stream(cudaStream_t* s) {
  int least = 0, greatest = 0;
  cudaError_t e = cudaDeviceGetStreamPriorityRange(&least, &greatest);
  if (e != cudaSuccess) return e;
  return cudaStreamCreateWithPriority(s, cudaStreamNonBlocking, greatest);
}

int dl_context_create(int device_ordinal, dl_context** out) {
  if (!out) return DL_ERR_ARG;
  *out = nullptr;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || device_ordinal < 0 || device_ordinal >= count) {
    g_create_error = e != cudaSuccess ? cudaGetErrorString(e) : "no such CUDA device";
    return DL_ERR_CUDA;
  }
  dl_context* ctx = new (std::nothrow) dl_context();
  if (!ctx) return DL_ERR_ARG;
  ctx->device = device_ordinal;
  if ((e = cudaSetDevice(device_ordinal)) != cudaSuccess ||
      (e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking)) != cudaSuccess ||
      (e = cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking)) != cudaSuccess ||
      (e = cudaStreamCreateWithFlags(&ctx->aux_stream, cudaStreamNonBlocking)) != cudaSuccess ||
      (e = create_high_priority_stream(&ctx->tail_stream)) != cudaSuccess ||
      (e = cudaEventCreateWithFlags(&ctx->batch_done, cudaEventDisableTiming)) != cudaSuccess ||
      (e = cudaEventCreateWithFlags(&ctx->staging_done, cudaEventDisableTiming)) != cudaSuccess) {
    g_create_error = cudaGetErrorString(e);
    delete ctx;
    return DL_ERR_CUDA;
  }
  *out = ctx;
  return DL_OK;
}

void dl_context_destroy(dl_context* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  if (ctx->stream) ctx->wait_stream();
  for (const dl_context::Mark& m : ctx->marks) { cudaEventDestroy(m.begin); cudaEventDestroy(m.end); }
  for (cudaEvent_t e : ctx->event_pool) cudaEventDestroy(e);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
  if (ctx->aux_stream) cudaStreamDestroy(ctx->aux_stream);
  if (ctx->tail_stream) cudaStreamDestroy(ctx->tail_stream);
  if (ctx->batch_done) cudaEventDestroy(ctx->batch_done);
  if (ctx->sync_event) cudaEventDestroy(ctx->sync_event);
  if (ctx->staging_done) cudaEventDestroy(ctx->staging_done);
  delete ctx;
}

const char* dl_last_error(const dl_context* ctx) { return ctx ? ctx->error.c_str() : g_create_error.c_str(); }

const char* dl_status_string(int status) {
  switch (status) {
    case DL_OK: return "ok";
    case DL_ERR_CUDA: return "CUDA error";
    case DL_ERR_ARG: return "invalid argument";
    case DL_ERR_GRID_RANGE: return "cell index outside the growable grid range";
    case DL_ERR_EMPTY: return "empty point cloud";
    case DL_ERR_SCORE: return "non-positive correlative score";
    default: return "unknown status";
  }
}
int64_t dl_context_kernel_launches(const dl_context* ctx) { return ctx ? ctx->launches : 0; }
uint64_t dl_context_stream(const dl_context* ctx) { return ctx ? (uint64_t)(uintptr_t)ctx->stream : 0; }
int dl_context_synchronize(dl_context* ctx) {
  if (!ctx) return DL_ERR_ARG;
  return sync(ctx);
}
int dl_context_set_blocking_sync(dl_context* ctx, int enabled) {
  if (!ctx) return DL_ERR_ARG;
  ctx->blocking_sync = enabled != 0;
  return DL_OK;
}
int dl_context_set_profiling(dl_context* ctx, int enabled) {
  if (!ctx) return DL_ERR_ARG;
  ctx->profiling = enabled != 0;
  return DL_OK;
}
int dl_context_read_profile(dl_context* ctx, dl_stage_time* out, int32_t capacity, int32_t* num_stages) {
  if (!ctx || !num_stages || capacity < 0 || (capacity > 0 && !out)) return DL_ERR_ARG;
  DL_CUDA(ctx, ctx->wait_stream());
  for (const dl_context::Mark& m : ctx->marks) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, m.begin, m.end) == cudaSuccess) {
      ctx->stage_ms[m.stage] += ms;
      ctx->stage_calls[m.stage] += 1;
    }
    ctx->event_pool.push_back(m.begin);
    ctx->event_pool.push_back(m.end);
  }
  ctx->marks.clear();
  const int n = (int)std::min<size_t>(ctx->stage_names.size(), (size_t)capacity);
  for (int i = 0; i < n; ++i) {
    std::memset(out[i].name, 0, sizeof(out[i].name));
    std::strncpy(out[i].name, ctx->stage_names[i].c_str(), sizeof(out[i].name) - 1);
    out[i].ms = ctx->stage_ms[i];
    out[i].calls = ctx->stage_calls[i];
    ctx->stage_ms[i] = 0.0;
    ctx->stage_calls[i] = 0;
  }
  *num_stages = n;
  return DL_OK;
}

int dl_device_alloc(dl_context* ctx, int64_t bytes, void** out_dev) {
  if (!ctx || !out_dev || bytes < 0) return DL_ERR_ARG;
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  DL_CUDA(ctx, cudaMalloc(out_dev, (size_t)std::max<int64_t>(bytes, 1)));
  return DL_OK;
}
int dl_device_free(dl_context* ctx, void* dev) {
  if (!ctx) return DL_ERR_ARG;
  DL_CUDA(ctx, cudaFree(dev));
  return DL_OK;
}
int dl_copy_to_device(dl_context* ctx, void* dst_dev, const void* src_host, int64_t bytes) {
  if (!ctx || bytes < 0) return DL_ERR_ARG;
  DL_CUDA(ctx, cudaMemcpyAsync(dst_dev, src_host, (size_t)bytes, cudaMemcpyHostToDevice, ctx->stream));
  return sync(ctx);
}
int dl_copy_to_host(dl_context* ctx, void* dst_host, const void* src_dev, int64_t bytes) {
  if (!ctx || bytes < 0) return DL_ERR_ARG;
  DL_CUDA(ctx, cudaMemcpyAsync(dst_host, src_dev, (size_t)bytes, cudaMemcpyDeviceToHost, ctx->stream));
  return sync(ctx);
}

// ------------------------------------------------------------------------------------------------ grid
int dl_grid_create(dl_context* ctx, float resolution, dl_grid** out) {
  if (!ctx || !out || !(resolution > 0.f)) return DL_ERR_ARG;
  dl_grid* g = new (std::nothrow) dl_grid();
  if (!g) return ctx->fail(DL_ERR_ARG, "out of memory");
  g->ctx = ctx;
  g->resolution = resolution;
  g->bits = 1;  // DynamicGrid starts with 2^3 top cells (hybrid_grid.h:255)
  g->top.assign(8, -1);
  *out = g;
  return DL_OK;
}

void dl_grid_destroy(dl_grid* g) {
  if (!g) return;
  cudaSetDevice(g->ctx->device);
  g->ctx->wait_stream();
  delete g;
}

float dl_grid_resolution(const dl_grid* g) { return g ? g->resolution : 0.f; }
// After a device insert the host mirror is behind until the next download: the device's brick counter is then the count in use.
int64_t dl_grid_num_bricks(const dl_grid* g) {
  if (!g) return 0;
  if (!g->mirror_stale) return (int64_t)(g->bricks.size() / 512);
  int32_t used = 0;
  if (cudaSetDevice(g->ctx->device) != cudaSuccess ||
      cudaMemcpyAsync(&used, g->d_counters.get() + 1, sizeof(int32_t), cudaMemcpyDeviceToHost, g->ctx->stream) != cudaSuccess ||
      g->ctx->wait_stream() != cudaSuccess)
    return -1;
  return used;
}

static int grid_download(dl_grid* g);
static inline size_t top_flat(int x, int y, int z, int bits) { return ((((size_t)z << bits) + y) << bits) + x; }

// Grow(): double every axis, old content moves to the centre (hybrid_grid.h:389-407).
static int grid_grow(dl_grid* g) {
  const int nb = g->bits + 1;
  if (nb > 8) return DL_ERR_GRID_RANGE;
  std::vector<int32_t> grown((size_t)8 * g->top.size(), -1);
  const int n = 1 << g->bits, o = 1 << (g->bits - 1);
  for (int z = 0; z < n; ++z)
    for (int y = 0; y < n; ++y)
      for (int x = 0; x < n; ++x) grown[top_flat(x + o, y + o, z + o, nb)] = g->top[top_flat(x, y, z, g->bits)];
  g->top.swap(grown);
  g->bits = nb;
  g->structure_dirty = true;
  return DL_OK;
}

int dl_grid_set_cells(dl_grid* g, int64_t n, const int32_t* xs, const int32_t* ys, const int32_t* zs,
                      const uint16_t* values) {
  if (g) g->version++;
  if (!g || n < 0 || (n > 0 && (!xs || !ys || !zs || !values))) return DL_ERR_ARG;
  if (g->mirror_stale) {
    const int st = grid_download(g);
    if (st != DL_OK) return st;
  }
  for (int64_t i = 0; i < n; ++i) {
    for (;;) {
      const int gs = 64 << g->bits, half = gs >> 1;
      const unsigned sx = (unsigned)(xs[i] + half), sy = (unsigned)(ys[i] + half), sz = (unsigned)(zs[i] + half);
      if (sx >= (unsigned)gs || sy >= (unsigned)gs || sz >= (unsigned)gs) {
        if (grid_grow(g) != DL_OK) return g->ctx->fail(DL_ERR_GRID_RANGE, "cell index outside +-8192 cells");
        continue;
      }
      int32_t& node = g->top[top_flat(sx >> 6, sy >> 6, sz >> 6, g->bits)];
      if (node < 0) {
        node = (int32_t)(g->nodes.size() / 512);
        g->nodes.insert(g->nodes.end(), 512, -1);
        g->structure_dirty = true;
      }
      int32_t& brick = g->nodes[(size_t)node * 512 + ((((sz >> 3) & 7) << 6) | (((sy >> 3) & 7) << 3) | ((sx >> 3) & 7))];
      if (brick < 0) {
        brick = (int32_t)(g->bricks.size() / 512);
        g->bricks.insert(g->bricks.end(), 512, 0);
        g->brick_dirty.push_back(1);
        g->structure_dirty = true;
      }
      g->bricks[(size_t)brick * 512 + (((sz & 7) << 6) | ((sy & 7) << 3) | (sx & 7))] = values[i];
      g->brick_dirty[brick] = 1;
      break;
    }
  }
  return DL_OK;
}

// Host mirror <- device (after device-side insertion the device copy is ahead).
static int grid_download(dl_grid* g) {
  if (!g->mirror_stale) return DL_OK;
  dl_context* ctx = g->ctx;
  int32_t counters[2] = {0, 0};
  DL_TRY(d2h(ctx, counters, g->d_counters.get(), 2));
  DL_TRY(sync(ctx));
  g->top.resize((size_t)1 << (3 * g->bits));
  g->nodes.resize((size_t)counters[0] * 512);
  g->bricks.resize((size_t)counters[1] * 512);
  g->brick_dirty.assign(counters[1], 0);
  DL_TRY(d2h(ctx, g->top.data(), g->d_top.get(), g->top.size()));
  DL_TRY(d2h(ctx, g->nodes.data(), g->d_nodes.get(), g->nodes.size()));
  DL_TRY(d2h(ctx, g->bricks.data(), g->d_bricks.get(), g->bricks.size()));
  DL_TRY(sync(ctx));
  g->mirror_stale = false;
  g->structure_dirty = false;
  return DL_OK;
}

int dl_grid_sync(dl_grid* g) {
  if (g) g->version++;
  if (!g) return DL_ERR_ARG;
  dl_context* ctx = g->ctx;
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  if (g->mirror_stale) return ctx->fail(DL_ERR_ARG, "internal: host mirror is behind the device grid");
  const size_t nbricks = g->bricks.size() / 512;
  if (!g->d_counters.get()) DL_TRY(alloc(ctx, g->d_counters, 8));
  if (g->structure_dirty) {
    if (g->top.size() > g->d_top.cap) DL_TRY(grow(ctx, g->d_top, g->top.size()));
    DL_TRY(grid_grow_pool(g, 0, 0, std::max<size_t>(g->nodes.size() / 512, 1)));
    const size_t old_cap = g->d_bricks.cap;
    DL_TRY(grid_grow_pool(g, 1, 0, std::max<size_t>(nbricks, 1)));
    if (g->d_bricks.cap != old_cap) std::fill(g->brick_dirty.begin(), g->brick_dirty.end(), 1);  // reallocated
    DL_TRY(h2d(ctx, g->d_top.get(), g->top.data(), g->top.size()));
    DL_TRY(h2d(ctx, g->d_nodes.get(), g->nodes.data(), g->nodes.size()));
    g->structure_dirty = false;
  }
  // upload dirty bricks, coalescing runs of consecutive dirty bricks into one copy
  size_t b = 0;
  while (b < nbricks) {
    if (!g->brick_dirty[b]) { ++b; continue; }
    size_t e = b;
    while (e < nbricks && g->brick_dirty[e]) g->brick_dirty[e++] = 0;
    DL_TRY(h2d(ctx, g->d_bricks.get() + b * 512, g->bricks.data() + b * 512, (e - b) * 512));
    b = e;
  }
  const int32_t counters[8] = {(int32_t)(g->nodes.size() / 512), (int32_t)nbricks, 0, 0, 0, 0, 0, 0};
  DL_TRY(h2d(ctx, g->d_counters.get(), counters, 8));
  return sync(ctx);
}

int dl_grid_lookup(dl_context* ctx, const dl_grid* g, int64_t n, const int32_t* xyz, uint16_t* value_out) {
  if (!ctx || !g || n < 0 || (n > 0 && (!xyz || !value_out))) return DL_ERR_ARG;
  if (g->structure_dirty) return ctx->fail(DL_ERR_ARG, "dl_grid_sync not called after dl_grid_set_cells");
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  int32_t* d_xyz;
  uint16_t* d_out;
  DL_TRY(carve_scratch(ctx, [&](Arena& a) {
    d_xyz = a.take<int32_t>(3 * n);
    d_out = a.take<uint16_t>(n);
  }));
  DL_TRY(h2d(ctx, d_xyz, xyz, 3 * n));
  DL_TRY(launch_grid_lookup(ctx, g->view(), n, d_xyz, d_out));
  DL_TRY(d2h(ctx, value_out, d_out, n));
  return sync(ctx);
}

int dl_grid_interpolate(dl_context* ctx, const dl_grid* g, int64_t n, const double* xyz, double* out) {
  if (!ctx || !g || n < 0 || (n > 0 && (!xyz || !out))) return DL_ERR_ARG;
  if (g->structure_dirty) return ctx->fail(DL_ERR_ARG, "dl_grid_sync not called after dl_grid_set_cells");
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  double *d_xyz, *d_out;
  DL_TRY(carve_scratch(ctx, [&](Arena& a) {
    d_xyz = a.take<double>(3 * n);
    d_out = a.take<double>(4 * n);
  }));
  DL_TRY(h2d(ctx, d_xyz, xyz, 3 * n));
  DL_TRY(launch_interpolate(ctx, g->view(), n, d_xyz, d_out));
  DL_TRY(d2h(ctx, out, d_out, 4 * n));
  return sync(ctx);
}

// ------------------------------------------------------------------------------------------------ grid write side
}  // extern "C"

namespace dl {
int grid_ensure_device_state(dl_grid* g) {
  if (g->mirror_stale) return DL_OK;  // the device copy is authoritative and complete
  bool dirty = g->structure_dirty || !g->d_counters.get();
  for (size_t b = 0; b < g->brick_dirty.size() && !dirty; ++b) dirty = g->brick_dirty[b] != 0;
  return dirty ? dl_grid_sync(g) : DL_OK;
}
// Grows the node pool (level 0) or the brick pool (level 1) from `used` entries in use by `add` more (dl_inserter.cu counts
// them exactly: the entries the running Insert marked), to the exact need + 25 % headroom, keeping the entries in use. Free
// node slots must read -1 and free brick slots 0 for the lock-free device-side growth.
int grid_grow_pool(dl_grid* g, int level, size_t used, size_t add) {
  const size_t need = (used + add) * 512;
  auto grow_pool = [&](auto& pool, int fill) {
    return need <= pool.cap ? DL_OK : grow(g->ctx, pool, need + need / 4 + 16 * 512, used * 512, fill);
  };
  return level == 0 ? grow_pool(g->d_nodes, 0xFF) : grow_pool(g->d_bricks, 0);
}
}  // namespace dl

namespace {
struct InsertScratch {
  uint16_t *hit_table, *miss_table;
  int32_t* bbox;
  void* args;
};
// The scratch every insert_range_data_device call of `jobs` jobs shares; each job's update list is carved by take_update_list.
void carve_insert(Arena& a, int jobs, InsertScratch* s) {
  s->hit_table = a.take<uint16_t>(32768);
  s->miss_table = a.take<uint16_t>(32768);
  s->bbox = a.take<int32_t>(8 * (size_t)std::max(jobs, 1));
  s->args = a.take<char>(insert_args_bytes(std::max(jobs, 1)));
}
uint32_t* take_update_list(Arena& a, const dl_range_data_inserter_options& o, int64_t n) {
  return a.take<uint32_t>((size_t)n * (size_t)(1 + std::max(o.num_free_space_voxels, 0)));
}
// The submap-frame transform and range filter of Submap3D::InsertRangeData for one cloud (carve_transform) and its two Inserts.
struct SubmapInsertScratch {
  float *all, *near;
  int32_t *near_count, *tiles;
  uint32_t *update_hi, *update_lo;
};
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
}  // namespace

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

int dl_grid_export_cells(dl_grid* g, int64_t capacity, int32_t* xs, int32_t* ys, int32_t* zs, uint16_t* vs, int64_t* n_cells) {
  if (!g || !n_cells || capacity < 0 || (capacity > 0 && (!xs || !ys || !zs || !vs))) return DL_ERR_ARG;
  DL_CUDA(g->ctx, cudaSetDevice(g->ctx->device));
  DL_TRY(grid_download(g));
  const int bits = g->bits, tmask = (1 << bits) - 1, half_top = (1 << (bits - 1)) * 64;
  int64_t count = 0;
  for (size_t t = 0; t < g->top.size(); ++t) {
    if (g->top[t] < 0) continue;
    const int tx = (int)t & tmask, ty = ((int)t >> bits) & tmask, tz = ((int)t >> bits) >> bits;
    const int32_t* node = g->nodes.data() + (size_t)g->top[t] * 512;
    for (int l = 0; l < 512; ++l) {
      if (node[l] < 0) continue;
      const uint16_t* brick = g->bricks.data() + (size_t)node[l] * 512;
      for (int c = 0; c < 512; ++c) {
        if (brick[c] == 0) continue;
        if (count < capacity) {
          xs[count] = tx * 64 + (l & 7) * 8 + (c & 7) - half_top;
          ys[count] = ty * 64 + ((l >> 3) & 7) * 8 + ((c >> 3) & 7) - half_top;
          zs[count] = tz * 64 + (l >> 6) * 8 + (c >> 6) - half_top;
          vs[count] = brick[c];
        }
        ++count;
      }
    }
  }
  *n_cells = count;
  return DL_OK;
}

// ------------------------------------------------------------------------------------------------ voxel filters
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

// ------------------------------------------------------------------------------------------------ RT-CSM (host part)
namespace {

// AngleAxisVectorToRotationQuaternion<float> (C/transform/transform.h:85-99): the cutoff compare and sin/cos run
// in double, results narrow to float.
Quatf angle_axis_to_quat(const Vec3f& aa) {
  float s = 0.5f, w = 1.f;
  if ((double)dot3(aa, aa) > 1e-8) {
    const float n = norm3(aa);
    s = (float)(std::sin((double)n / 2.) / (double)n);
    w = (float)std::cos((double)n / 2.);
  }
  return {w, s * aa.x, s * aa.y, s * aa.z};
}
float rotation_angle(const Quatf& q) {  // transform.h:33-37
  return 2.f * std::atan2(norm3(Vec3f{q.x, q.y, q.z}), std::fabs(q.w));
}

struct RtcsmTables {
  int linear = 0, angular = 0;
  float step = 0.f;
  std::vector<Quatf> cand_q;
  std::vector<Vec3f> cand_t;
  std::vector<double> pen_r, pen_t;
};

// GenerateExhaustiveSearchTransforms (SM/real_time_correlative_scan_matcher_3d.cc:55-95), factored into the
// R rotations and L translations it is the outer product of, each composed with the initial pose.
void build_rtcsm_tables(const dl_rtcsm_options& opt, float resolution, float max_scan_range, const Rigidf& initial,
                        RtcsmTables* t) {
  t->linear = (int)std::lround(opt.linear_search_window / resolution);  // double / float -> double
  const float kSafetyMargin = 1.f - 1e-3f;
  t->step = kSafetyMargin * std::acos(1.f - (resolution * resolution) / (2.f * (max_scan_range * max_scan_range)));
  t->angular = (int)std::lround(opt.angular_search_window / t->step);
  const int L = t->linear, A = t->angular;
  for (int rz = -A; rz <= A; ++rz)
    for (int ry = -A; ry <= A; ++ry)
      for (int rx = -A; rx <= A; ++rx) {
        const Quatf q = angle_axis_to_quat(Vec3f{rx * t->step, ry * t->step, rz * t->step});
        t->cand_q.push_back(qnormalized(qmul(initial.q, q)));
        t->pen_r.push_back(rotation_angle(q) * opt.rotation_delta_cost_weight);
      }
  for (int z = -L; z <= L; ++z)
    for (int y = -L; y <= L; ++y)
      for (int x = -L; x <= L; ++x) {
        const Vec3f off{x * resolution, y * resolution, z * resolution};
        t->cand_t.push_back(add(rotate(initial.q, off), initial.t));
        t->pen_t.push_back(norm3(off) * opt.translation_delta_cost_weight);
      }
}

// One batched correlative search. Clouds are on the device: cloud k = points[k] with counts[k] rows (host-known). The tables
// of every scan (R rotations, L translations, their penalties) are built on the host with the reference's float operations
// — the angular window depends on each cloud's farthest point through acosf, which must be the host's to stay bit-exact —
// and go up in ONE copy; one launch scores all (scan, rotation, translation) candidates.
struct RtcsmBatchItem {
  const dl_grid* grid;  // the grid this scan is scored against; every grid of a batch has the plan's resolution
  const float* d_points;
  int64_t n;
  Rigidd initial;
  float max_scan_range;
  float* d_scores;          // optional
  int32_t* d_nonpositive;   // optional: set to 1 when a candidate's score is not > 0
};
// plan_rtcsm_batch builds the tables and lays out the one upload (every scan's tables, the descriptors, the CTA prefix); take()
// carves that upload and the argmax words, so a caller can count the scratch before it reserves it; run_rtcsm_batch uploads
// and launches.
struct RtcsmBatchPlan {
  std::vector<RtcsmTables> tables;
  std::vector<size_t> off_q, off_t, off_pr, off_pt;
  std::vector<int32_t> prefix;
  size_t off_scans = 0, off_prefix = 0, blob = 0;
  unsigned char* d_blob = nullptr;
  RtcsmScan* d_scans = nullptr;
  unsigned long long* d_best = nullptr;
  void take(Arena& a) {
    d_blob = a.take<unsigned char>(blob);
    d_best = a.take<unsigned long long>(tables.size());
    d_scans = (RtcsmScan*)(d_blob + off_scans);
  }
};
int plan_rtcsm_batch(dl_context* ctx, const dl_rtcsm_options& opt, float resolution, const std::vector<RtcsmBatchItem>& items,
                     RtcsmBatchPlan* plan) {
  const int B = (int)items.size();
  plan->tables.assign(B, RtcsmTables{});
  plan->off_q.resize(B); plan->off_t.resize(B); plan->off_pr.resize(B); plan->off_pt.resize(B);
  plan->prefix.assign(B + 1, 0);
  auto align16 = [](size_t v) { return (v + 15) & ~size_t(15); };
  size_t blob = 0;
  for (int k = 0; k < B; ++k) {
    build_rtcsm_tables(opt, resolution, items[k].max_scan_range, to_float(items[k].initial), &plan->tables[k]);
    const RtcsmTables& t = plan->tables[k];
    const int64_t R = (int64_t)t.cand_q.size(), L = (int64_t)t.cand_t.size();
    if (R * L >= 0xFFFFFFFFll) return ctx->fail(DL_ERR_ARG, "more than 2^32-1 correlative candidates");
    plan->off_q[k] = blob; blob = align16(blob + R * sizeof(Quatf));
    plan->off_t[k] = blob; blob = align16(blob + L * sizeof(Vec3f));
    plan->off_pr[k] = blob; blob = align16(blob + R * sizeof(double));
    plan->off_pt[k] = blob; blob = align16(blob + L * sizeof(double));
    plan->prefix[k + 1] = plan->prefix[k] + rtcsm_ctas_for(R, L);
  }
  plan->off_scans = blob; blob = align16(blob + (size_t)B * sizeof(RtcsmScan));
  plan->off_prefix = blob; blob = align16(blob + (size_t)(B + 1) * sizeof(int32_t));
  plan->blob = blob;
  return DL_OK;
}
// `plan` has taken its scratch; items[k].d_points / d_scores / d_nonpositive are read here.
int run_rtcsm_batch(dl_context* ctx, const std::vector<RtcsmBatchItem>& items, const RtcsmBatchPlan& plan) {
  const int B = (int)items.size();
  if (B == 0) return DL_OK;
  std::vector<unsigned char> host(plan.blob);
  for (int k = 0; k < B; ++k) {
    const RtcsmTables& t = plan.tables[k];
    std::memcpy(host.data() + plan.off_q[k], t.cand_q.data(), t.cand_q.size() * sizeof(Quatf));
    std::memcpy(host.data() + plan.off_t[k], t.cand_t.data(), t.cand_t.size() * sizeof(Vec3f));
    std::memcpy(host.data() + plan.off_pr[k], t.pen_r.data(), t.pen_r.size() * sizeof(double));
    std::memcpy(host.data() + plan.off_pt[k], t.pen_t.data(), t.pen_t.size() * sizeof(double));
    RtcsmScan sc{};
    sc.grid = items[k].grid->view();
    sc.points = items[k].d_points;
    sc.n = (int32_t)items[k].n;
    sc.cand_q = (const Quatf*)(plan.d_blob + plan.off_q[k]);
    sc.cand_t = (const Vec3f*)(plan.d_blob + plan.off_t[k]);
    sc.pen_r = (const double*)(plan.d_blob + plan.off_pr[k]);
    sc.pen_t = (const double*)(plan.d_blob + plan.off_pt[k]);
    sc.R = (int32_t)t.cand_q.size();
    sc.L = (int32_t)t.cand_t.size();
    sc.scores = items[k].d_scores;
    sc.best = plan.d_best + k;
    sc.nonpositive = items[k].d_nonpositive;
    std::memcpy(host.data() + plan.off_scans + (size_t)k * sizeof(RtcsmScan), &sc, sizeof(sc));
  }
  std::memcpy(host.data() + plan.off_prefix, plan.prefix.data(), (size_t)(B + 1) * sizeof(int32_t));
  DL_TRY(h2d(ctx, plan.d_blob, host.data(), plan.blob));
  DL_CUDA(ctx, cudaMemsetAsync(plan.d_best, 0, sizeof(unsigned long long) * B, ctx->stream));
  DL_TRY(sync(ctx));  // `host` is pageable and local
  return launch_rtcsm_batch(ctx, plan.d_scans, (const int32_t*)(plan.d_blob + plan.off_prefix), B, plan.prefix[B]);
}

// The farthest point of a host cloud, floored at 3 * resolution (cc:63-71), with the norm the device reduction uses.
float max_scan_range_host(const float* points, int64_t n, float resolution) {
  float m = 3.f * resolution;
  for (int64_t i = 0; i < n; ++i) m = std::max(m, norm3(Vec3f{points[3 * i], points[3 * i + 1], points[3 * i + 2]}));
  return m;
}

// Upper bound of the scratch one scan of the front end's correlative pre-match takes (tables, descriptor, prefix, argmax word).
// The tables' size follows from the cloud's farthest point, which a device reduction finds after the front end has carved its
// scratch, so it is bounded from the options. Every point the pre-match sees has passed the high-resolution filter's
// norm3(p) <= max_range, so max_scan_range <= max(3 * resolution, max_range). The float step does not grow with the range, so
// A is largest at that range, until the argument of acosf rounds to 1 (about 4096 resolutions): there the step is 0 and A is 0,
// and below it the step is never smaller than 0.999f * acosf(1 - 2^-24). So A is bounded by its value at max_range, or by the
// smallest positive step when max_range is past that cliff.
size_t rtcsm_scratch_bound(const dl_rtcsm_options& opt, float resolution, float max_range) {
  const int L1 = 2 * (int)std::lround(opt.linear_search_window / resolution) + 1;
  const float r = max_range > 3.f * resolution ? max_range : 3.f * resolution;
  const float kSafetyMargin = 1.f - 1e-3f;
  float step = kSafetyMargin * std::acos(1.f - (resolution * resolution) / (2.f * (r * r)));
  if (!(step > 0.f)) step = kSafetyMargin * std::acos(std::nextafter(1.f, 0.f));
  const int A1 = 2 * (int)std::lround(opt.angular_search_window / step) + 1;
  const size_t R = (size_t)A1 * A1 * A1, L = (size_t)L1 * L1 * L1;
  Arena bound(nullptr);  // the plan's takes at the largest tables, with room for the blob's 16-byte alignment
  bound.take<unsigned char>(R * 16 + L * 12 + R * 8 + L * 8 + 256 + sizeof(RtcsmScan) + 64);
  bound.take<unsigned long long>(1);
  return bound.off + 4096;
}

}  // namespace

extern "C" {

int dl_rtcsm_match(dl_context* ctx, const dl_rtcsm_options* options, const double* initial_pose, const float* points,
                   int64_t n, const dl_grid* grid, double* pose_out, float* score_out, dl_rtcsm_info* info,
                   float* all_scores) {
  if (!ctx || !options || !initial_pose || !grid || !pose_out || n < 0 || (n > 0 && !points)) return DL_ERR_ARG;  // CHECK_NOTNULL(pose_estimate)
  if (n == 0) return ctx->fail(DL_ERR_EMPTY, "empty point cloud");
  if (grid->structure_dirty) return ctx->fail(DL_ERR_ARG, "dl_grid_sync not called after dl_grid_set_cells");
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  // The cloud is on the host: its farthest point, hence the tables and the exact scratch, are known before the carve.
  const float max_scan_range = max_scan_range_host(points, n, grid->resolution);
  std::vector<RtcsmBatchItem> items{RtcsmBatchItem{grid, nullptr, n, pose_from7(initial_pose), max_scan_range, nullptr, nullptr}};
  RtcsmBatchPlan plan;
  DL_TRY(plan_rtcsm_batch(ctx, *options, grid->resolution, items, &plan));
  const RtcsmTables& t = plan.tables[0];
  const int64_t R = (int64_t)t.cand_q.size(), K = R * (int64_t)t.cand_t.size();
  float* d_pts;
  float* d_scores = nullptr;
  DL_TRY(carve_scratch(ctx, [&](Arena& c) {
    d_pts = c.take<float>(3 * n);
    if (all_scores) d_scores = c.take<float>(K);
    plan.take(c);
  }));
  DL_TRY(h2d(ctx, d_pts, points, 3 * n));
  items[0].d_points = d_pts;
  items[0].d_scores = d_scores;
  DL_TRY(run_rtcsm_batch(ctx, items, plan));
  unsigned long long best = 0;
  DL_TRY(d2h(ctx, &best, plan.d_best, 1));
  if (all_scores) DL_TRY(d2h(ctx, all_scores, d_scores, K));
  DL_TRY(sync(ctx));
  if (best == 0) return ctx->fail(DL_ERR_SCORE, "no candidate with a positive score (CHECK_GT(score, 0))");
  const uint32_t score_bits = (uint32_t)(best >> 32);
  const int64_t index = (int64_t)(0xFFFFFFFFull - (best & 0xFFFFFFFFull));
  float score;
  std::memcpy(&score, &score_bits, 4);
  const int64_t l = index / R, r = index - l * R;
  pose_to7(to_double(Rigidf{t.cand_t[l], t.cand_q[r]}), pose_out);
  if (score_out) *score_out = score;
  if (info) {
    info->best_index = index;
    info->num_candidates = K;
    info->linear_window = t.linear;
    info->angular_window = t.angular;
    info->angular_step = t.step;
    info->max_scan_range = max_scan_range;
  }
  return DL_OK;
}

// ------------------------------------------------------------------------------------------------ Ceres-equivalent matcher
static int check_ceres_options(dl_context* ctx, const dl_ceres_options* o, int num_pairs) {
  if (!o) return DL_ERR_ARG;
  if (num_pairs < 1 || num_pairs > DL_MAX_PAIRS) return ctx->fail(DL_ERR_ARG, "num_pairs out of range");
  if (o->num_occupied_space_weights != num_pairs)
    return ctx->fail(DL_ERR_ARG, "occupied_space_weight count != number of (cloud, grid) pairs (CHECK_EQ)");
  for (int i = 0; i < num_pairs; ++i)
    if (!(o->occupied_space_weight[i] > 0.)) return ctx->fail(DL_ERR_ARG, "occupied_space_weight must be > 0 (CHECK_GT)");
  if (o->max_num_iterations <= 0) return ctx->fail(DL_ERR_ARG, "max_num_iterations must be > 0 (CHECK_GT)");
  return DL_OK;
}
static NlsOptions to_nls_options(const dl_ceres_options& o, int num_pairs) {
  NlsOptions n{};
  n.num_pairs = num_pairs;
  for (int i = 0; i < num_pairs; ++i) n.occ_weight[i] = o.occupied_space_weight[i];
  n.trans_weight = o.translation_weight;
  n.rot_weight = o.rotation_weight;
  n.only_yaw = o.only_optimize_yaw;
  n.nonmono = o.use_nonmonotonic_steps;
  n.max_iter = o.max_num_iterations;
  return n;
}

int dl_ceres_match_batch(dl_context* ctx, const dl_ceres_options* options, int32_t count, int32_t num_pairs,
                         const double* target_translations, const double* initial_poses, const float* const* clouds,
                         const int64_t* sizes, const dl_grid* const* grids, double* poses_out,
                         dl_solve_summary* summaries) {
  if (!ctx) return DL_ERR_ARG;
  DL_TRY(check_ceres_options(ctx, options, num_pairs));
  if (count < 0 || (count > 0 && (!target_translations || !initial_poses || !clouds || !sizes || !grids || !poses_out)))
    return DL_ERR_ARG;
  if (count == 0) return DL_OK;
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  for (int i = 0; i < count * num_pairs; ++i) {
    if (sizes[i] < 0 || !grids[i] || (sizes[i] > 0 && !clouds[i])) return DL_ERR_ARG;
    if (sizes[i] == 0) return ctx->fail(DL_ERR_EMPTY, "empty point cloud");
    if (grids[i]->structure_dirty) return ctx->fail(DL_ERR_ARG, "dl_grid_sync not called after dl_grid_set_cells");
  }
  std::vector<float*> d_clouds(count * num_pairs);
  NlsProblem* d_problems;
  NlsOutput* d_out;
  DL_TRY(carve_scratch(ctx, [&](Arena& a) {
    for (int i = 0; i < count * num_pairs; ++i) d_clouds[i] = a.take<float>(3 * sizes[i]);
    d_problems = a.take<NlsProblem>(count);
    d_out = a.take<NlsOutput>(count);
  }));
  std::vector<NlsProblem> problems(count);
  for (int c = 0; c < count; ++c) {
    NlsProblem& p = problems[c];
    std::memset(&p, 0, sizeof(p));
    for (int k = 0; k < num_pairs; ++k) {
      const int i = c * num_pairs + k;
      DL_TRY(h2d(ctx, d_clouds[i], clouds[i], 3 * sizes[i]));
      p.cloud[k] = d_clouds[i];
      p.count[k] = (int32_t)sizes[i];
      p.grid[k] = grids[i]->view();
    }
    for (int j = 0; j < 3; ++j) p.target_t[j] = target_translations[3 * c + j];
    for (int j = 0; j < 7; ++j) p.initial[j] = initial_poses[7 * c + j];
  }
  DL_TRY(h2d(ctx, d_problems, problems.data(), count));
  DL_TRY(launch_nls(ctx, to_nls_options(*options, num_pairs), d_problems, count, d_out));
  std::vector<NlsOutput> out(count);
  DL_TRY(d2h(ctx, out.data(), d_out, count));
  DL_TRY(sync(ctx));
  for (int c = 0; c < count; ++c) {
    std::memcpy(poses_out + 7 * c, out[c].pose, 7 * sizeof(double));
    if (summaries) summaries[c] = out[c].summary;
  }
  return DL_OK;
}

int dl_ceres_match(dl_context* ctx, const dl_ceres_options* options, const double* target_translation,
                   const double* initial_pose, int32_t num_pairs, const float* const* clouds, const int64_t* sizes,
                   const dl_grid* const* grids, double* pose_out, dl_solve_summary* summary) {
  return dl_ceres_match_batch(ctx, options, 1, num_pairs, target_translation, initial_pose, clouds, sizes, grids,
                              pose_out, summary);
}

int dl_ceres_normal_equations(dl_context* ctx, const dl_ceres_options* options, const double* target_translation,
                              const double* reference_pose, const double* at_pose, int32_t num_pairs,
                              const float* const* clouds, const int64_t* sizes, const dl_grid* const* grids,
                              double* cost, double* gradient6, double* hessian36) {
  if (!ctx) return DL_ERR_ARG;
  DL_TRY(check_ceres_options(ctx, options, num_pairs));
  if (!target_translation || !reference_pose || !at_pose || !clouds || !sizes || !grids || !cost || !gradient6 || !hessian36)
    return DL_ERR_ARG;
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  float* d_clouds[DL_MAX_PAIRS];
  NlsProblem* d_p;
  double *d_at, *d_out;
  DL_TRY(carve_scratch(ctx, [&](Arena& a) {
    for (int k = 0; k < num_pairs; ++k) d_clouds[k] = a.take<float>(3 * sizes[k]);
    d_p = a.take<NlsProblem>(1);
    d_at = a.take<double>(7);
    d_out = a.take<double>(28);
  }));
  NlsProblem p;
  std::memset(&p, 0, sizeof(p));
  for (int k = 0; k < num_pairs; ++k) {
    DL_TRY(h2d(ctx, d_clouds[k], clouds[k], 3 * sizes[k]));
    p.cloud[k] = d_clouds[k];
    p.count[k] = (int32_t)sizes[k];
    p.grid[k] = grids[k]->view();
  }
  for (int j = 0; j < 3; ++j) p.target_t[j] = target_translation[j];
  for (int j = 0; j < 7; ++j) p.initial[j] = reference_pose[j];
  DL_TRY(h2d(ctx, d_p, &p, 1));
  DL_TRY(h2d(ctx, d_at, at_pose, 7));
  DL_TRY(launch_nls_normal_equations(ctx, to_nls_options(*options, num_pairs), d_p, d_at, d_out));
  double out[28];
  DL_TRY(d2h(ctx, out, d_out, 28));
  DL_TRY(sync(ctx));
  *cost = out[0];
  for (int i = 0; i < 6; ++i) gradient6[i] = out[1 + i];
  int t = 7;
  for (int r = 0; r < 6; ++r)
    for (int c = r; c < 6; ++c) hessian36[r * 6 + c] = hessian36[c * 6 + r] = out[t++];
  return DL_OK;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------ IMU
// ------------------------------------------------------------------------------------------------ loop closure
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
}  // namespace

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

namespace {
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

}  // extern "C"

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

namespace {
using HostImuTerm = dl::ImuTerm;  // prepared here on the host for the calls that take finished pre-integrations

// W = weight^2 * Sigma^-1 by Cholesky (Sigma = L L^T, W = L^-T L^-1). False if Sigma is not positive definite.
bool information_matrix(const double* sigma, double weight, double* W) {
  double L[15][15] = {};
  for (int i = 0; i < 15; ++i)
    for (int j = 0; j <= i; ++j) {
      double s = sigma[i * 15 + j];
      for (int k = 0; k < j; ++k) s -= L[i][k] * L[j][k];
      if (i == j) {
        if (!(s > 0)) return false;
        L[i][i] = std::sqrt(s);
      } else {
        L[i][j] = s / L[j][j];
      }
    }
  double Li[15][15] = {};  // L^-1 (lower)
  for (int c = 0; c < 15; ++c) {
    for (int i = c; i < 15; ++i) {
      double s = i == c ? 1.0 : 0.0;
      for (int k = c; k < i; ++k) s -= L[i][k] * Li[k][c];
      Li[i][c] = s / L[i][i];
    }
  }
  for (int a = 0; a < 15; ++a)
    for (int b = 0; b < 15; ++b) {
      double s = 0;
      for (int k = std::max(a, b); k < 15; ++k) s += Li[k][a] * Li[k][b];
      W[a * 15 + b] = weight * weight * s;
    }
  return true;
}
// One pre-integration factor in the submap frame (the grids live there and the solve is frame-invariant) + the initial
// 16-vector of state j. False if the covariance is not positive definite.
bool build_imu_term(const Rigidd& to_submap, const dl_nav_state& si, const dl_nav_state& sj, const dl_preintegration& m,
                    const double* gravity, double imu_weight, HostImuTerm* t, double* x16) {
  const Rigidd pose_i = compose(to_submap, Rigidd{{si.p[0], si.p[1], si.p[2]}, {si.q[0], si.q[1], si.q[2], si.q[3]}});
  const Rigidd pose_j = compose(to_submap, Rigidd{{sj.p[0], sj.p[1], sj.p[2]}, {sj.q[0], sj.q[1], sj.q[2], sj.q[3]}});
  const Vec3d vi = rotate(to_submap.q, Vec3d{si.v[0], si.v[1], si.v[2]});
  const Vec3d vj = rotate(to_submap.q, Vec3d{sj.v[0], sj.v[1], sj.v[2]});
  const Vec3d G = rotate(to_submap.q, Vec3d{gravity[0], gravity[1], gravity[2]});
  t->pi[0] = pose_i.t.x; t->pi[1] = pose_i.t.y; t->pi[2] = pose_i.t.z;
  t->qi[0] = pose_i.q.w; t->qi[1] = pose_i.q.x; t->qi[2] = pose_i.q.y; t->qi[3] = pose_i.q.z;
  t->vi[0] = vi.x; t->vi[1] = vi.y; t->vi[2] = vi.z;
  imu_term_deltas(m, si.ba, si.bg, t);
  t->G[0] = G.x; t->G[1] = G.y; t->G[2] = G.z;
  t->sum_dt = m.sum_dt;
  if (!information_matrix(m.covariance, imu_weight, t->W)) return false;
  pose_to7(pose_j, x16);
  x16[7] = vj.x; x16[8] = vj.y; x16[9] = vj.z;
  for (int k = 0; k < 3; ++k) { x16[10 + k] = sj.ba[k]; x16[13 + k] = sj.bg[k]; }
  return true;
}
// Solver state (submap frame) -> dl_nav_state in the local frame.
void state_to_local(const Rigidd& submap, const double* x, dl_nav_state* o) {
  const Rigidd pose = compose(submap, pose_from7(x));
  const Vec3d v = rotate(submap.q, Vec3d{x[7], x[8], x[9]});
  o->p[0] = pose.t.x; o->p[1] = pose.t.y; o->p[2] = pose.t.z;
  o->q[0] = pose.q.w; o->q[1] = pose.q.x; o->q[2] = pose.q.y; o->q[3] = pose.q.z;
  o->v[0] = v.x; o->v[1] = v.y; o->v[2] = v.z;
  for (int k = 0; k < 3; ++k) { o->ba[k] = x[10 + k]; o->bg[k] = x[13 + k]; }
}
}  // namespace

extern "C" {

int dl_imu_preintegrate(dl_context* ctx, const dl_imu_noise* noise, int32_t count, const int32_t* offsets,
                        const double* dt, const double* acc, const double* gyr, const double* biases,
                        dl_preintegration* out) {
  if (!ctx || !noise || count < 0 || (count > 0 && (!offsets || !dt || !acc || !gyr || !biases || !out))) return DL_ERR_ARG;
  if (count == 0) return DL_OK;
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t n = (size_t)offsets[count];
  for (int k = 0; k < count; ++k)
    if (offsets[k + 1] < offsets[k]) return ctx->fail(DL_ERR_ARG, "offsets must be non-decreasing");
  int32_t* d_off;
  double *d_dt, *d_acc, *d_gyr, *d_bias;
  dl_preintegration* d_out;
  DL_TRY(carve_scratch(ctx, [&](Arena& a) {
    d_off = a.take<int32_t>(count + 1);
    d_dt = a.take<double>(n);
    d_acc = a.take<double>(3 * n);
    d_gyr = a.take<double>(3 * n);
    d_bias = a.take<double>(6 * (size_t)count);
    d_out = a.take<dl_preintegration>(count);
  }));
  DL_TRY(h2d(ctx, d_off, offsets, count + 1));
  DL_TRY(h2d(ctx, d_dt, dt, n));
  DL_TRY(h2d(ctx, d_acc, acc, 3 * n));
  DL_TRY(h2d(ctx, d_gyr, gyr, 3 * n));
  DL_TRY(h2d(ctx, d_bias, biases, 6 * (size_t)count));
  DL_TRY(launch_imu_preintegrate(ctx, count, d_off, d_dt, d_acc, d_gyr, d_bias, 6, *noise, d_out));
  DL_TRY(d2h(ctx, out, d_out, count));
  return sync(ctx);
}

int dl_imu_predict(const dl_nav_state* si, const dl_preintegration* m, const double* gravity, dl_nav_state* sj) {
  if (!si || !m || !gravity || !sj) return DL_ERR_ARG;
  const double T = m->sum_dt;
  const Quatd qi{si->q[0], si->q[1], si->q[2], si->q[3]};
  const Vec3d G{gravity[0], gravity[1], gravity[2]};
  const Vec3d p = add(sub(add(Vec3d{si->p[0], si->p[1], si->p[2]}, mul(T, Vec3d{si->v[0], si->v[1], si->v[2]})), mul(0.5 * T * T, G)),
                      rotate(qi, Vec3d{m->delta_p[0], m->delta_p[1], m->delta_p[2]}));
  const Vec3d v = add(sub(Vec3d{si->v[0], si->v[1], si->v[2]}, mul(T, G)), rotate(qi, Vec3d{m->delta_v[0], m->delta_v[1], m->delta_v[2]}));
  const Quatd q = qnormalized(qmul(qi, Quatd{m->delta_q[0], m->delta_q[1], m->delta_q[2], m->delta_q[3]}));
  *sj = *si;
  sj->p[0] = p.x; sj->p[1] = p.y; sj->p[2] = p.z;
  sj->v[0] = v.x; sj->v[1] = v.y; sj->v[2] = v.z;
  sj->q[0] = q.w; sj->q[1] = q.x; sj->q[2] = q.y; sj->q[3] = q.z;
  return DL_OK;
}

int dl_imu_factor_evaluate(dl_context* ctx, int32_t count, const dl_nav_state* states_i, const dl_preintegration* preintegrations,
                           const double* submap_local_poses, const double* gravity, double imu_weight, const double* x16,
                           int32_t* ok, dl_nav_state* predicted, double* information, double* residual, double* hessian,
                           double* gradient, double* cost2) {
  if (!ctx || count < 0 || !gravity || !(imu_weight >= 0.) ||
      (count > 0 && (!states_i || !preintegrations || !submap_local_poses || !ok || !predicted || !information || !residual ||
                     !hessian || !gradient || !cost2)))
    return DL_ERR_ARG;
  if (count == 0) return DL_OK;
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  dl_preintegration* d_pre;
  dl_nav_state *d_si, *d_pred;
  Rigidd* d_to_submap;
  ScanConstants* d_scans;
  HostImuTerm* d_terms;
  double *d_init, *d_x, *d_out;
  int32_t* d_ok;
  DL_TRY(carve_scratch(ctx, [&](Arena& a) {
    d_pre = a.take<dl_preintegration>(count);
    d_si = a.take<dl_nav_state>(count);
    d_pred = a.take<dl_nav_state>(count);
    d_to_submap = a.take<Rigidd>(count);
    d_scans = a.take<ScanConstants>(count);
    d_terms = a.take<HostImuTerm>(count);
    d_init = a.take<double>((size_t)count * 16);
    d_x = x16 ? a.take<double>((size_t)count * 16) : nullptr;
    d_out = a.take<double>((size_t)count * kImuFactorOutDoubles);
    d_ok = a.take<int32_t>(count);
  }));
  std::vector<Rigidd> to_submap(count);
  for (int c = 0; c < count; ++c) to_submap[c] = inverse(pose_from7(submap_local_poses + 7 * c));
  DL_TRY(h2d(ctx, d_pre, preintegrations, count));
  DL_TRY(h2d(ctx, d_si, states_i, count));
  DL_TRY(h2d(ctx, d_to_submap, to_submap.data(), count));
  if (x16) DL_TRY(h2d(ctx, d_x, x16, (size_t)count * 16));
  ImuPrepareArgs pa{};
  pa.count = count; pa.preint = d_pre; pa.states_i = d_si; pa.to_submap = d_to_submap;
  for (int k = 0; k < 3; ++k) pa.gravity[k] = gravity[k];
  pa.imu_weight = imu_weight; pa.scans = d_scans; pa.terms = d_terms; pa.init16 = d_init; pa.predicted = d_pred; pa.ok = d_ok;
  DL_TRY(launch_imu_prepare(ctx, pa));
  DL_TRY(launch_imu_factor_evaluate(ctx, count, d_terms, d_ok, x16 ? d_x : d_init, d_out));
  std::vector<HostImuTerm> terms(count);
  std::vector<double> out((size_t)count * kImuFactorOutDoubles);
  DL_TRY(d2h(ctx, ok, d_ok, count));
  DL_TRY(d2h(ctx, predicted, d_pred, count));
  DL_TRY(d2h(ctx, terms.data(), d_terms, count));
  DL_TRY(d2h(ctx, out.data(), d_out, out.size()));
  DL_TRY(sync(ctx));
  for (int c = 0; c < count; ++c) {
    const double* o = out.data() + (size_t)c * kImuFactorOutDoubles;
    const bool good = ok[c] != 0;
    for (int e = 0; e < 225; ++e) {
      information[225 * (size_t)c + e] = good ? terms[c].W[e] : 0.0;
      hessian[225 * (size_t)c + e] = good ? o[15 + e] : 0.0;
    }
    for (int e = 0; e < 15; ++e) {
      residual[15 * (size_t)c + e] = good ? o[e] : 0.0;
      gradient[15 * (size_t)c + e] = good ? o[240 + e] : 0.0;
    }
    cost2[c] = good ? o[255] : 0.0;
  }
  return DL_OK;
}

int dl_fused_match_batch(dl_context* ctx, const dl_ceres_options* options, double imu_weight, const double* gravity,
                         int32_t count, int32_t num_pairs, const double* submap_local_poses,
                         const dl_nav_state* states_i, const dl_nav_state* initial_states_j,
                         const dl_preintegration* preints, const float* const* clouds, const int64_t* sizes,
                         const dl_grid* const* grids, dl_nav_state* states_j_out, dl_solve_summary* summaries) {
  if (!ctx) return DL_ERR_ARG;
  DL_TRY(check_ceres_options(ctx, options, num_pairs));
  if (options->only_optimize_yaw) return ctx->fail(DL_ERR_ARG, "only_optimize_yaw is not supported by the fused solve");
  if (count < 0 || !gravity || !(imu_weight >= 0.) ||
      (count > 0 && (!submap_local_poses || !states_i || !initial_states_j || !preints || !clouds || !sizes || !grids || !states_j_out)))
    return DL_ERR_ARG;
  if (count == 0) return DL_OK;
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  for (int i = 0; i < count * num_pairs; ++i) {
    if (sizes[i] < 0 || !grids[i] || (sizes[i] > 0 && !clouds[i])) return DL_ERR_ARG;
    if (sizes[i] == 0) return ctx->fail(DL_ERR_EMPTY, "empty point cloud");
    if (grids[i]->structure_dirty) return ctx->fail(DL_ERR_ARG, "dl_grid_sync not called after dl_grid_set_cells");
  }
  std::vector<float*> d_clouds(count * num_pairs);
  NlsProblem* d_problems;
  HostImuTerm* d_terms;
  double* d_init;
  FusedOutput* d_out;
  DL_TRY(carve_scratch(ctx, [&](Arena& a) {
    for (int i = 0; i < count * num_pairs; ++i) d_clouds[i] = a.take<float>(3 * sizes[i]);
    d_problems = a.take<NlsProblem>(count);
    d_terms = a.take<HostImuTerm>(count);
    d_init = a.take<double>((size_t)count * 16);
    d_out = a.take<FusedOutput>(count);
  }));
  std::vector<NlsProblem> problems(count);
  std::vector<HostImuTerm> terms(count);
  std::vector<double> init16((size_t)count * 16);
  for (int c = 0; c < count; ++c) {
    const Rigidd to_submap = inverse(pose_from7(submap_local_poses + 7 * c));
    double* x = init16.data() + 16 * c;
    if (!build_imu_term(to_submap, states_i[c], initial_states_j[c], preints[c], gravity, imu_weight, &terms[c], x))
      return ctx->fail(DL_ERR_ARG, "pre-integration covariance is not positive definite");
    NlsProblem& p = problems[c];
    std::memset(&p, 0, sizeof(p));
    for (int k = 0; k < num_pairs; ++k) {
      const int i = c * num_pairs + k;
      DL_TRY(h2d(ctx, d_clouds[i], clouds[i], 3 * sizes[i]));
      p.cloud[k] = d_clouds[i];
      p.count[k] = (int32_t)sizes[i];
      p.grid[k] = grids[i]->view();
    }
    for (int k = 0; k < 7; ++k) p.initial[k] = x[k];
    for (int k = 0; k < 3; ++k) p.target_t[k] = x[k];  // the translation prior (if weighted) pulls to the IMU prediction
  }
  DL_TRY(h2d(ctx, d_problems, problems.data(), count));
  DL_TRY(h2d(ctx, d_terms, terms.data(), count));
  DL_TRY(h2d(ctx, d_init, init16.data(), (size_t)count * 16));
  DL_TRY(launch_nls_fused(ctx, to_nls_options(*options, num_pairs), d_problems, d_terms, d_init, count, d_out));
  std::vector<FusedOutput> out(count);
  DL_TRY(d2h(ctx, out.data(), d_out, count));
  DL_TRY(sync(ctx));
  for (int c = 0; c < count; ++c) {
    state_to_local(pose_from7(submap_local_poses + 7 * c), out[c].state, &states_j_out[c]);
    if (summaries) summaries[c] = out[c].summary;
  }
  return DL_OK;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------ batched front end
namespace {

// The submaps a front-end batch matches against: one for every scan (the public front-end entry points) or one per scan
// (dl_ltb_add_range_data_batch, whose scans come from different trajectories).
struct SubmapSet {
  const double* poses = nullptr;             // 7 doubles: the local pose, once or per scan
  const dl_grid* const* hi = nullptr;        // one grid, or one per scan
  const dl_grid* const* lo = nullptr;
  bool per_scan = false;
  const double* pose(int b) const { return poses + (per_scan ? 7 * b : 0); }
  const dl_grid* high(int b) const { return hi[per_scan ? b : 0]; }
  const dl_grid* low(int b) const { return lo[per_scan ? b : 0]; }
};
// The single-submap form; the grid pointers must outlive the call.
struct OneSubmap : SubmapSet {
  const dl_grid* h;
  const dl_grid* l;
  OneSubmap(const double* pose7, const dl_grid* hi_grid, const dl_grid* lo_grid) : h(hi_grid), l(lo_grid) {
    poses = pose7;
    hi = &h;
    lo = &l;
  }
  OneSubmap(const OneSubmap&) = delete;
};

struct FrontendBuffers {
  int batch = 0;
  int64_t cap = 0, tcap = 0;
  int32_t *counts0, *n1, *n_ret, *n2, *n3, *countsA, *npassesA, *croppedA;
  uint32_t *tableA, *scratchA;
  int32_t* keepA;
  float *returns_tracking, *misses_tracking, *clouds, *current_pose, *origins, *passesA, *rtcsm_scores;
  int32_t* rtcsm_nonpositive = nullptr;  // pre-match only (carve_prematch): per scan, a candidate scored <= 0 (CHECK_GT)
  // fused front half
  int64_t bit_words = 0;
  uint32_t* bits;              // two survivor bitmaps per scan
  uint32_t* first_bits;        // the first filter's survivor bitmap per scan
  int4* stage;                 // tile winners by hash partition, and their ends per tile (dl_frontend.cu)
  int32_t *part_ends, *spill_used;
  uint32_t* spill;
  int32_t *last_index, *error_flag;
  float* local4;
  ScanConstants* scans;
  AdaptiveParams* filters;
  Rigidd *submap, *submap_inverse;  // per scan: its matching submap's local pose and the inverse (host arithmetic)
  int32_t* origin_base;             // per scan: its first origin in `origins`
  double *initial_pose, *target;
  NlsProblem* problems;
  NlsOutput* nls_out;
  // 12-byte rows only (carve_time_runs)
  int32_t *run_offsets = nullptr, *run_first_row = nullptr;
  float *run_value = nullptr, *run_pose = nullptr;
};

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

// IMU coupling of one front-end run: either finished pre-integrations (`host`, factors built on the host) or raw samples
// (`samples`, everything on the device), and its device buffers (carve_imu).
struct ImuRun {
  const dl_frontend_imu* host = nullptr;
  const dl_frontend_imu_samples* samples = nullptr;
  dl_nav_state* d_states_out = nullptr;  // in: optional caller-provided device buffer for the estimated states
  HostImuTerm* d_terms = nullptr;
  double* d_init16 = nullptr;
  FusedOutput* d_fused = nullptr;
  dl_nav_state* d_states = nullptr;      // estimated states, local frame
  // raw samples only
  int32_t* d_off = nullptr;
  double *d_dt = nullptr, *d_acc = nullptr, *d_gyr = nullptr;
  dl_nav_state* d_si = nullptr;
  dl_preintegration* d_pre = nullptr;
  dl_nav_state* d_predicted = nullptr;   // predicted states, local frame
  int32_t* d_ok = nullptr;               // per scan: its IMU factor could be formed
};
void carve_imu(Arena& a, int num_scans, ImuRun* r) {
  r->d_terms = a.take<HostImuTerm>(num_scans);
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
    std::vector<HostImuTerm> terms(num_scans);
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

// Where the scans of a batch are: host rows, one pointer per scan, which the batch uploads into its scratch; or device rows
// (scan b at row b * cap_rows) with a caller-provided device buffer for the results (and, with raw IMU samples, one for the
// estimated states in ImuRun::d_states_out).
struct FrontendScans {
  const void* const* host = nullptr;
  bool on_device = false;
  const void* dev = nullptr;
  int64_t cap_rows = 0;
  dl_scan_result* results_dev = nullptr;
};

// Validates, reserves, carves and enqueues one front-end batch: the one place that sizes a batch's scratch. On return
// *d_results_out holds the device results (not yet synchronised).
// `more` (optional) carves the caller's own buffers into the same reservation, after the batch's: they stay valid as long as the
// batch's (the trajectory builders' batch keeps the tracking-frame clouds on the device until insertion has read them).
// origin_base (optional): per scan, where its origins start in `origins`.
int frontend_enqueue(dl_context* ctx, const dl_frontend_options* options, int num_scans, const FrontendScans& in,
                     const int64_t* sizes, const float* origins, int num_origins, const double* prev_poses,
                     const double* predicted_poses, const SubmapSet& submaps, dl_scan_result** d_results_out, ImuRun* imu = nullptr,
                     FrontendBuffers* buffers_out = nullptr, const int32_t* origin_base = nullptr,
                     const std::function<void(Arena&)>* more = nullptr) {
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

}  // namespace

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

static int check_imu_options(dl_context* ctx, const dl_frontend_options* options) {
  if (options && options->ceres_scan_matcher.only_optimize_yaw)
    return ctx->fail(DL_ERR_ARG, "only_optimize_yaw is not supported by the fused solve");
  return DL_OK;
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

static int check_imu_samples(dl_context* ctx, const dl_frontend_options* options, const dl_frontend_imu_samples* imu, int num_scans) {
  if (!imu || num_scans < 0) return DL_ERR_ARG;
  if (num_scans == 0) return DL_OK;
  if (!imu->states_i || !imu->offsets || !(imu->imu_weight >= 0.)) return DL_ERR_ARG;
  if (imu->offsets[0] != 0) return ctx->fail(DL_ERR_ARG, "offsets[0] must be 0");
  for (int k = 0; k < num_scans; ++k)
    if (imu->offsets[k + 1] < imu->offsets[k]) return ctx->fail(DL_ERR_ARG, "offsets must be non-decreasing");
  if (imu->offsets[num_scans] > 0 && (!imu->dt || !imu->acc || !imu->gyr)) return DL_ERR_ARG;
  return check_imu_options(ctx, options);
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


// ------------------------------------------------------------------------------------------------ rotational histogram
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

// ------------------------------------------------------------------------------------------------ LocalTrajectoryBuilder3D
// The per-trajectory object of the reference front end (local_trajectory_builder_3d.h:81-113) over the device path:
// AddImuData buffers the samples of the running interval, AddRangeData runs a scan through the IMU-coupled front end
// against the matching submap (active_submaps_.submaps().front(), LTB:502-505) — the scans of many builders in one batch
// (dl_ltb_add_range_data_batch; the single calls are its batch of one) — then does what AddAccumulatedRangeData /
// InsertIntoSubmap do after the match: motion filter (motion_filter.cc:37-57), insertion into both active submaps on the
// device (submap_3d.cc:264-279, :300-326 incl. the submap hand-over), rotational histogram of the inserted scan (LTB:605-610).
// Differences, all stated in the header: the fused solve replaces the match + GTSAM window (so `local_pose` is the solve's
// pose), num_accumulated_range_data = 1, a single range sensor (the synchroniser for several is the host-side
// dliom::sensor::RangeDataSynchronizer of the C++ shim), initialisation = InitializeStatic or a state given by the caller.
namespace {
// Device buffers of `count` window updates (carve_window) and the upload / launch / read-back of dl_window_optimize_batch on them,
// shared with the trajectory builders' batch, which carves them next to its front end's buffers.
struct WindowBuffers {
  dl_nav_state *si, *init, *si_out, *sj_out;
  double *prior, *z, *info;
  dl_preintegration* pre;
  dl_solve_summary* sum;
};
void carve_window(Arena& a, int count, WindowBuffers* w) {
  const size_t n = (size_t)count;
  w->si = a.take<dl_nav_state>(n);
  w->prior = a.take<double>(n * 225);
  w->pre = a.take<dl_preintegration>(n);
  w->z = a.take<double>(n * 7);
  w->init = a.take<dl_nav_state>(n);
  w->si_out = a.take<dl_nav_state>(n);
  w->sj_out = a.take<dl_nav_state>(n);
  w->info = a.take<double>(n * 225);
  w->sum = a.take<dl_solve_summary>(n);
}
int window_optimize(dl_context* ctx, const dl_window_options& options, int count, const WindowBuffers& w, const dl_nav_state* states_i,
                    const double* prior_information, const dl_preintegration* preintegrations, const double* matched_poses,
                    const dl_nav_state* initial_states_j, dl_nav_state* states_i_out, dl_nav_state* states_j_out,
                    double* information_out, dl_solve_summary* summaries) {
  const size_t n = (size_t)count;
  DL_TRY(h2d(ctx, w.si, states_i, n));
  DL_TRY(h2d(ctx, w.prior, prior_information, n * 225));
  DL_TRY(h2d(ctx, w.pre, preintegrations, n));
  DL_TRY(h2d(ctx, w.z, matched_poses, n * 7));
  if (initial_states_j) DL_TRY(h2d(ctx, w.init, initial_states_j, n));
  DL_CUDA(ctx, cudaMemsetAsync(w.sj_out, 0, n * sizeof(dl_nav_state), ctx->stream));
  DL_CUDA(ctx, cudaMemsetAsync(w.info, 0, n * 225 * 8, ctx->stream));
  DL_TRY(launch_window_optimize(ctx, count, w.si, w.prior, w.pre, w.z, initial_states_j ? w.init : nullptr, options, w.si_out, w.sj_out,
                                w.info, w.sum));
  DL_TRY(d2h(ctx, states_j_out, w.sj_out, n));
  if (states_i_out) DL_TRY(d2h(ctx, states_i_out, w.si_out, n));
  DL_TRY(d2h(ctx, information_out, w.info, n * 225));
  std::vector<dl_solve_summary> sums(n);
  DL_TRY(d2h(ctx, sums.data(), w.sum, n));
  DL_TRY(sync(ctx));
  if (summaries) std::memcpy(summaries, sums.data(), n * sizeof(dl_solve_summary));
  return DL_OK;
}
// The options of dl_window_optimize_batch and dl_window_evaluate as the kernels take them: sigmas and the IMU weight positive and,
// with the gravity factor on, both directions finite and non-zero. Only their orientation enters the factor (Unit3 normalises
// too), so both are normalised here, the one place that does it.
int window_options_checked(dl_context* ctx, const dl_window_options& in, dl_window_options* out) {
  if (!(in.pose_sigma_translation > 0.) || !(in.pose_sigma_rotation > 0.) || !(in.imu_weight > 0.) ||
      (in.use_gravity_factor && !(in.gravity_sigma > 0.)))
    return ctx->fail(DL_ERR_ARG, "dl_window_options: sigmas and the IMU weight must be positive");
  *out = in;
  if (!in.use_gravity_factor) return DL_OK;
  for (double* d : {out->gravity_direction, out->body_reference_direction}) {
    const double n = std::sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    if (!std::isfinite(n) || !(n > 0.))
      return ctx->fail(DL_ERR_ARG, "dl_window_options: the gravity and body reference directions must be finite and non-zero");
    for (int k = 0; k < 3; ++k) d[k] /= n;
  }
  return DL_OK;
}

}  // namespace

struct LtbSubmap {
  dl_grid* hi = nullptr;
  dl_grid* lo = nullptr;
  Rigidd local_pose{{0, 0, 0}, {1, 0, 0, 0}};
  int num_range_data = 0;
  int finished = 0;
  int index = 0;
};
struct dl_local_trajectory_builder {
  dl_context* ctx = nullptr;
  dl_ltb_options opt{};
  bool initialized = false;
  int accumulated_frames = 0;
  std::vector<double> init_acc, init_gyr;  // xyz per sample
  dl_nav_state prev_state{};
  double last_imu_time = -1.0;
  std::vector<double> dt, acc, gyr;        // the running interval; sample 0 is the latch
  std::vector<LtbSubmap> active, finished;
  int next_index = 0;
  int64_t motion_total = 0;
  double motion_last_time = 0;
  Rigidd motion_last_pose{{0, 0, 0}, {1, 0, 0, 0}};
  std::vector<float> clouds[4];            // returns / misses in the local frame, high / low resolution cloud in the tracking frame
  std::vector<float> histogram;
  double window_information[225];          // two-stage mode: the marginal of the previous key (prior of the next window update)
  void reset_window_information() {        // prior_pose_noise_, prior_vel_noise_, prior_bias_noise_ (LTB:84-90)
    for (double& v : window_information) v = 0.;
    const double sp = opt.prior_pose_noise > 0 ? opt.prior_pose_noise : 1e-2, sv = opt.prior_velocity_noise > 0 ? opt.prior_velocity_noise : 1e4,
                 sb = opt.prior_bias_noise > 0 ? opt.prior_bias_noise : 1e-2;
    for (int k = 0; k < 15; ++k) {
      const double s = k < 6 ? sp : (k < 9 ? sv : sb);
      window_information[k * 15 + k] = 1.0 / (s * s);
    }
  }
};

namespace {
// The empty grids of a new submap; on failure nothing is left allocated.
int ltb_make_grids(const dl_local_trajectory_builder* b, LtbSubmap* s) {
  int st = dl_grid_create(b->ctx, b->opt.high_resolution, &s->hi);
  if (st == DL_OK) st = dl_grid_create(b->ctx, b->opt.low_resolution, &s->lo);
  if (st == DL_OK) st = dl_grid_sync(s->hi);
  if (st == DL_OK) st = dl_grid_sync(s->lo);
  if (st != DL_OK) {
    dl_grid_destroy(s->hi);
    dl_grid_destroy(s->lo);
    s->hi = s->lo = nullptr;
  }
  return st;
}
// ActiveSubmaps3D::AddSubmap (submap_3d.cc:315-326) with the grids of `s` (ltb_make_grids).
void ltb_add_submap(dl_local_trajectory_builder* b, const Rigidd& pose, LtbSubmap s) {
  if (b->active.size() > 1) {
    b->active.front().finished = 1;
    b->finished.push_back(b->active.front());
    b->active.erase(b->active.begin());
  }
  s.local_pose = pose;
  s.index = b->next_index++;
  b->active.push_back(s);
}
double rotation_angle_d(const Quatd& q) {  // transform::GetAngle (transform.h:33-37)
  return 2.0 * std::atan2(std::sqrt(q.x * q.x + q.y * q.y + q.z * q.z), std::fabs(q.w));
}
// InitializeStatic after frames_for_static_initialization scans (LTB:372-381, :203-229): the mean specific force fixes roll /
// pitch, the residual of the two the accelerometer bias, the mean rate the gyroscope bias.
void ltb_initialize_static(dl_local_trajectory_builder* b) {
  if (!(b->accumulated_frames++ > b->opt.frames_for_static_initialization && !b->init_acc.empty())) return;
  const size_t m = b->init_acc.size() / 3;
  double am[3] = {0, 0, 0}, gm[3] = {0, 0, 0};
  for (size_t k = 0; k < m; ++k)
    for (int c = 0; c < 3; ++c) { am[c] += b->init_acc[3 * k + c]; gm[c] += b->init_gyr[3 * k + c]; }
  for (int c = 0; c < 3; ++c) { am[c] /= (double)m; gm[c] /= (double)m; }
  // R = FromTwoVectors(accel_mean, (0, 0, g)): the rotation taking the measured up direction to +z
  const double an = std::sqrt(am[0] * am[0] + am[1] * am[1] + am[2] * am[2]);
  Quatd q{1, 0, 0, 0};
  if (an > 0) {
    const Vec3d u{am[0] / an, am[1] / an, am[2] / an}, v{0, 0, 1};
    const double c = dot3(u, v);
    if (c > -1.0 + 1e-12) {
      const Vec3d ax = cross3(u, v);
      const double s2 = std::sqrt((1.0 + c) * 2.0);
      q = qnormalized(Quatd{s2 * 0.5, ax.x / s2, ax.y / s2, ax.z / s2});
    } else {
      q = Quatd{0, 1, 0, 0};
    }
  }
  dl_nav_state st{};
  st.q[0] = q.w; st.q[1] = q.x; st.q[2] = q.y; st.q[3] = q.z;
  const Vec3d g_body = rotate(qconj(q), Vec3d{0, 0, -b->opt.gravity});  // R^T g_vec
  st.ba[0] = g_body.x + am[0]; st.ba[1] = g_body.y + am[1]; st.ba[2] = g_body.z + am[2];
  for (int c = 0; c < 3; ++c) st.bg[c] = gm[c];
  b->prev_state = st;
  b->initialized = true;
  b->reset_window_information();
  b->init_acc.clear(); b->init_gyr.clear();
}

// The batched front end takes one options block and one IMU noise, so the members of a batch must agree on every field the
// builder reads (bit for bit; the frontend's row layout and host stride are the builder's own and always equal).
bool same_ltb_options(const dl_ltb_options& a, const dl_ltb_options& b) {
#define DL_SAME(field) (std::memcmp(&a.field, &b.field, sizeof(a.field)) == 0)
  const bool frontend = DL_SAME(frontend.min_range) && DL_SAME(frontend.max_range) && DL_SAME(frontend.voxel_filter_size) &&
      DL_SAME(frontend.high_resolution_adaptive_voxel_filter) && DL_SAME(frontend.low_resolution_adaptive_voxel_filter) &&
      DL_SAME(frontend.use_online_correlative_scan_matching) && DL_SAME(frontend.range_row_floats) &&
      DL_SAME(frontend.scan_period) && DL_SAME(frontend.real_time_correlative_scan_matcher) &&
      DL_SAME(frontend.ceres_scan_matcher.num_occupied_space_weights) && DL_SAME(frontend.ceres_scan_matcher.occupied_space_weight) &&
      DL_SAME(frontend.ceres_scan_matcher.translation_weight) && DL_SAME(frontend.ceres_scan_matcher.rotation_weight) &&
      DL_SAME(frontend.ceres_scan_matcher.only_optimize_yaw) && DL_SAME(frontend.ceres_scan_matcher.use_nonmonotonic_steps) &&
      DL_SAME(frontend.ceres_scan_matcher.max_num_iterations) && DL_SAME(frontend.host_scan_stride_rows);
  return frontend && DL_SAME(imu_noise) && DL_SAME(imu_weight) && DL_SAME(gravity) && DL_SAME(high_resolution) &&
         DL_SAME(low_resolution) && DL_SAME(num_range_data) && DL_SAME(high_resolution_max_range) &&
         DL_SAME(range_data_inserter.hit_probability) && DL_SAME(range_data_inserter.miss_probability) &&
         DL_SAME(range_data_inserter.num_free_space_voxels) && DL_SAME(motion_filter_max_time_seconds) &&
         DL_SAME(motion_filter_max_distance_meters) && DL_SAME(motion_filter_max_angle_radians) &&
         DL_SAME(rotational_histogram_size) && DL_SAME(frames_for_static_initialization) && DL_SAME(two_stage) &&
         DL_SAME(ceres_pose_noise_t) && DL_SAME(ceres_pose_noise_r) && DL_SAME(prior_pose_noise) &&
         DL_SAME(prior_velocity_noise) && DL_SAME(prior_bias_noise);
#undef DL_SAME
}

// One member of dl_ltb_add_range_data_batch: what the device work found for it and what its builder takes over at the commit.
struct LtbMember {
  dl_local_trajectory_builder* b = nullptr;
  const dl_ltb_batch_item* item = nullptr;
  int slot = -1;                       // its scan in the front-end batch; -1: an early return applies
  dl_matching_result out{};
  dl_preintegration m{};               // two-stage mode: the interval's pre-integration and the predicted state
  dl_nav_state pred{};
  dl_nav_state state{};                // the node's state (has_result)
  bool window_reset = false;           // two-stage: FailureDetection fell back and re-seeds the carried information
  std::vector<double> window_information;
  bool motion_filtered = false;
  Rigidd opt_pose{{0, 0, 0}, {1, 0, 0, 0}};
  std::vector<float> clouds[4];
  std::vector<float> histogram;
  bool hands_over = false;             // this insert completes the newest submap: `next` holds the grids of the one it adds
  LtbSubmap next;
};

// The builder takes over what the device work found for its member (the single call's tail, LTB:553-622). Cannot fail: the
// grids of a hand-over were made beforehand.
void ltb_commit(dl_local_trajectory_builder* b, LtbMember& m, double time) {
  if (m.out.scan.ok != 1) return;  // dropped like the reference's nullptr (LTB:497-534); the interval keeps integrating
  if (b->opt.two_stage) {
    if (m.window_reset) b->reset_window_information();
    else std::memcpy(b->window_information, m.window_information.data(), sizeof(b->window_information));
  }
  // the estimate becomes the previous state; the last sample of the interval latches the next one
  b->prev_state = m.state;
  {
    const size_t last = b->dt.size() - 1;
    const double ldt = b->dt[last];
    const double la[3] = {b->acc[3 * last], b->acc[3 * last + 1], b->acc[3 * last + 2]};
    const double lg[3] = {b->gyr[3 * last], b->gyr[3 * last + 1], b->gyr[3 * last + 2]};
    b->dt.assign(1, ldt);
    b->acc.assign(la, la + 3);
    b->gyr.assign(lg, lg + 3);
  }
  for (int c = 0; c < 4; ++c) b->clouds[c].swap(m.clouds[c]);
  ++b->motion_total;
  if (m.motion_filtered) return;  // insertion_result == nullptr
  b->motion_last_time = time;
  b->motion_last_pose = m.opt_pose;
  for (LtbSubmap& sm : b->active) sm.num_range_data++;
  if (m.hands_over)  // ActiveSubmaps3D::InsertRangeData (submap_3d.cc:300-313)
    ltb_add_submap(b, Rigidd{{(double)m.out.origin_in_local[0], (double)m.out.origin_in_local[1], (double)m.out.origin_in_local[2]},
                             m.opt_pose.q}, m.next);
  b->histogram.swap(m.histogram);
}

// The device work of a batch: the front end over every participating member's scan, each against its own matching submap, then
// (two-stage) the window update of all of them, the local frame and the histogram input, insertion into every inserted member's
// active submaps and their histograms. The host waits a fixed number of times, whatever the number of members, except once for
// each grid pool or top level that has to grow.
int ltb_batch_device(dl_context* ctx, const dl_ltb_options& opt, bool two_stage, const double* gravity, std::vector<LtbMember>& ms,
                     const std::vector<int>& part) {
  const int P = (int)part.size();
  // ---- the scans' rows: one layout for the batch (4-float rows become RangeMeasurement rows of origin index 0 when mixed)
  bool mixed = false;
  for (int i : part) mixed = mixed || ms[i].item->row_floats != ms[part[0]].item->row_floats;
  const int rf = mixed ? 8 : ms[part[0]].item->row_floats;
  std::vector<std::vector<float>> widened(P);
  std::vector<const void*> ranges(P);
  std::vector<int64_t> sizes(P);
  std::vector<int32_t> origin_base(P);
  std::vector<float> origins;
  for (int s = 0; s < P; ++s) {
    const dl_ltb_batch_item& it = *ms[part[s]].item;
    ranges[s] = it.rows;
    sizes[s] = it.n;
    origin_base[s] = (int32_t)(origins.size() / 3);
    origins.insert(origins.end(), it.origins, it.origins + 3 * (size_t)it.num_origins);
    if (it.row_floats != rf) {
      std::vector<float>& w = widened[s];
      w.assign((size_t)it.n * 8, 0.f);
      for (int64_t r = 0; r < it.n; ++r) std::memcpy(&w[8 * r], (const float*)it.rows + 4 * r, 4 * sizeof(float));
      ranges[s] = w.data();
    }
  }
  // ---- matching submaps (active_submaps_.submaps().front(), LTB:502-505)
  std::vector<double> submap_poses(7 * (size_t)P);
  std::vector<const dl_grid*> his(P), los(P);
  for (int s = 0; s < P; ++s) {
    const LtbSubmap& matching = ms[part[s]].b->active.front();
    pose_to7(matching.local_pose, submap_poses.data() + 7 * s);
    his[s] = matching.hi;
    los[s] = matching.lo;
  }
  SubmapSet submaps;
  submaps.poses = submap_poses.data();
  submaps.hi = his.data();
  submaps.lo = los.data();
  submaps.per_scan = true;
  // ---- the IMU intervals, concatenated
  std::vector<int32_t> offsets(P + 1, 0);
  std::vector<double> dt, acc, gyr;
  std::vector<dl_nav_state> states_i(P);
  for (int s = 0; s < P; ++s) {
    const dl_local_trajectory_builder* b = ms[part[s]].b;
    dt.insert(dt.end(), b->dt.begin(), b->dt.end());
    acc.insert(acc.end(), b->acc.begin(), b->acc.end());
    gyr.insert(gyr.end(), b->gyr.begin(), b->gyr.end());
    offsets[s + 1] = (int32_t)dt.size();
    states_i[s] = b->prev_state;
  }
  dl_frontend_options fo = opt.frontend;
  fo.range_row_floats = rf;
  dl_frontend_imu_samples imu{};
  imu.noise = opt.imu_noise;
  imu.imu_weight = opt.imu_weight;
  imu.gravity[0] = gravity[0]; imu.gravity[1] = gravity[1]; imu.gravity[2] = gravity[2];
  imu.states_i = states_i.data();
  imu.offsets = offsets.data();
  imu.dt = dt.data(); imu.acc = acc.data(); imu.gyr = gyr.data();
  std::vector<double> prev7, pred7;
  if (two_stage) {
    // the reference's chain: predict (AddImuData, LTB:188-199) -> plain match from the prediction (LTB:535-542) -> window (LTB:555)
    std::vector<double> bias(6 * (size_t)P);
    for (int s = 0; s < P; ++s)
      for (int c = 0; c < 3; ++c) { bias[6 * s + c] = states_i[s].ba[c]; bias[6 * s + 3 + c] = states_i[s].bg[c]; }
    std::vector<dl_preintegration> pre(P);
    DL_TRY(dl_imu_preintegrate(ctx, &opt.imu_noise, P, offsets.data(), dt.data(), acc.data(), gyr.data(), bias.data(), pre.data()));
    prev7.resize(7 * (size_t)P);
    pred7.resize(7 * (size_t)P);
    for (int s = 0; s < P; ++s) {
      LtbMember& m = ms[part[s]];
      m.m = pre[s];
      DL_TRY(dl_imu_predict(&states_i[s], &m.m, imu.gravity, &m.pred));
      for (int k = 0; k < 3; ++k) { prev7[7 * s + k] = states_i[s].p[k]; pred7[7 * s + k] = m.pred.p[k]; }
      for (int k = 0; k < 4; ++k) { prev7[7 * s + 3 + k] = states_i[s].q[k]; pred7[7 * s + 3 + k] = m.pred.q[k]; }
    }
  } else {
    DL_TRY(check_imu_samples(ctx, &fo, &imu, P));
  }
  // ---- scratch of everything after the front end, carved into the front end's reservation: its tracking-frame clouds stay
  //      valid until insertion and the histograms have read them. Sizes are the scans' row counts (bounds of every cloud).
  const dl_range_data_inserter_options& io = opt.range_data_inserter;
  const int H = opt.rotational_histogram_size;
  struct Slot {
    float *returns_local, *misses_local, *aligned, *histogram;
    HistogramScratch hs;
    SubmapInsertScratch ins[2];
  };
  std::vector<Slot> slots(P);
  InsertScratch is;
  void *d_local_jobs, *d_transform_jobs, *d_hist_args;
  int32_t* d_hist_err;
  float* d_gather;
  size_t gather_floats = 0;
  for (int s = 0; s < P; ++s) gather_floats += 12 * (size_t)sizes[s] + (size_t)H;
  WindowBuffers w{};
  const std::function<void(Arena&)> more = [&](Arena& a) {
    for (int s = 0; s < P; ++s) {
      const int64_t n = sizes[s];
      Slot& sl = slots[s];
      sl.returns_local = a.take<float>(3 * (size_t)n);
      sl.misses_local = a.take<float>(3 * (size_t)n);
      sl.aligned = a.take<float>(3 * (size_t)n);
      sl.histogram = a.take<float>((size_t)H);
      carve_rotational_histogram(a, n, &sl.hs);
      for (int k = 0; k < (int)ms[part[s]].b->active.size() && k < 2; ++k) carve_submap_insert(a, io, n, &sl.ins[k]);
    }
    carve_insert(a, 4 * P, &is);
    d_local_jobs = a.take<char>(local_frame_jobs_bytes(P));
    d_transform_jobs = a.take<char>(transform_jobs_bytes(2 * P));
    d_hist_args = a.take<char>(rotational_histograms_args_bytes(P));
    d_hist_err = a.take<int32_t>((size_t)P);
    d_gather = a.take<float>(gather_floats);
    if (two_stage) carve_window(a, P, &w);
  };
  // ---- the front end: every scan against its own matching submap
  dl_scan_result* d_results = nullptr;
  FrontendBuffers f;
  ImuRun run;
  run.samples = &imu;
  DL_TRY(frontend_enqueue(ctx, &fo, P, FrontendScans{ranges.data()}, sizes.data(), origins.data(), (int)(origins.size() / 3),
                          two_stage ? prev7.data() : nullptr, two_stage ? pred7.data() : nullptr, submaps, &d_results,
                          two_stage ? nullptr : &run, &f, origin_base.data(), &more));
  std::vector<dl_scan_result> r(P);
  std::vector<dl_nav_state> fused_states(P);
  std::vector<float> cur7(7 * (size_t)P);
  std::vector<int32_t> nonpositive(fo.use_online_correlative_scan_matching ? P : 0, 0);
  DL_TRY(d2h(ctx, r.data(), d_results, P));
  if (!two_stage) DL_TRY(d2h(ctx, fused_states.data(), run.d_states, P));
  DL_TRY(d2h(ctx, cur7.data(), f.current_pose, 7 * (size_t)P));
  DL_TRY(d2h(ctx, nonpositive.data(), f.rtcsm_nonpositive, nonpositive.size()));
  DL_TRY(sync(ctx));
  // The reference CHECK-fails on a pre-match candidate whose score is not > 0 (real_time_correlative_scan_matcher_3d.cc:111).
  // The pre-match runs before the insertion, so no grid has changed yet: the call fails and no builder is committed.
  for (int32_t flag : nonpositive)
    if (flag) return ctx->fail(DL_ERR_SCORE, "a correlative pre-match candidate scored <= 0 (CHECK_GT(score, 0))");
  std::vector<int> ok;  // slots whose scan was matched (scan.ok == 1)
  for (int s = 0; s < P; ++s) {
    LtbMember& m = ms[part[s]];
    m.out.scan = r[s];
    if (r[s].ok == 1) ok.push_back(s);
    if (!two_stage) m.state = fused_states[s];
  }
  if (ok.empty()) return DL_OK;
  if (two_stage) {
    // WindowOptimize(pose_estimate) (LTB:555): the matched pose is a prior on the new key next to the IMU factor and the carried
    // marginal of the previous key; one solve per member, all in one launch (dl_window_optimize_batch's kernel).
    dl_window_options wo{};
    wo.pose_sigma_translation = opt.ceres_pose_noise_t > 0 ? opt.ceres_pose_noise_t : 1e-2;
    wo.pose_sigma_rotation = opt.ceres_pose_noise_r > 0 ? opt.ceres_pose_noise_r : 1e-2;
    wo.imu_weight = opt.imu_weight > 0 ? opt.imu_weight : 1.0;
    wo.gravity[2] = opt.gravity;
    wo.max_num_iterations = 10;
    const size_t n = ok.size();
    std::vector<dl_nav_state> si(n), init(n), sj(n);
    std::vector<double> prior(n * 225), z(n * 7), info(n * 225);
    std::vector<dl_preintegration> pre(n);
    std::vector<dl_solve_summary> sums(n);
    for (size_t j = 0; j < n; ++j) {
      const LtbMember& m = ms[part[ok[j]]];
      si[j] = m.b->prev_state;
      init[j] = m.pred;
      pre[j] = m.m;
      std::memcpy(prior.data() + 225 * j, m.b->window_information, 225 * sizeof(double));
      std::memcpy(z.data() + 7 * j, m.out.scan.pose_estimate_local, 7 * sizeof(double));
    }
    DL_TRY(window_optimize(ctx, wo, (int)n, w, si.data(), prior.data(), pre.data(), z.data(), init.data(), nullptr, sj.data(),
                           info.data(), sums.data()));
    for (size_t j = 0; j < n; ++j) {
      LtbMember& m = ms[part[ok[j]]];
      if (sums[j].termination == 2) {  // the reference's FailureDetection path (LTB:856-859): matched pose + predicted rest, re-seed
        m.state = m.pred;
        for (int k = 0; k < 3; ++k) m.state.p[k] = m.out.scan.pose_estimate_local[k];
        for (int k = 0; k < 4; ++k) m.state.q[k] = m.out.scan.pose_estimate_local[3 + k];
        m.window_reset = true;
      } else {
        m.state = sj[j];
        m.window_information.assign(info.data() + 225 * j, info.data() + 225 * (j + 1));
      }
    }
  }
  // ---- per matched member: the node, the motion filter, the local frame and the histogram input
  std::vector<LocalFrameJob> local_jobs;
  std::vector<int> inserted;  // slots
  for (int s : ok) {
    LtbMember& m = ms[part[s]];
    const dl_local_trajectory_builder* b = m.b;
    const dl_scan_result& rs = r[s];
    dl_matching_result& out = m.out;
    out.has_result = 1;
    out.state = m.state;
    const Rigidd opt_pose{{m.state.p[0], m.state.p[1], m.state.p[2]}, {m.state.q[0], m.state.q[1], m.state.q[2], m.state.q[3]}};
    m.opt_pose = opt_pose;
    pose_to7(opt_pose, out.local_pose);
    // filtered_range_data_in_local = TransformRangeData(filtered_range_data_in_tracking, opt_pose.cast<float>()) (LTB:559-560)
    const Rigidf opt_f = to_float(opt_pose);
    const float* c7 = cur7.data() + 7 * s;
    const Rigidf cur{{c7[0], c7[1], c7[2]}, {c7[3], c7[4], c7[5], c7[6]}};
    const Vec3f origin_tracking = apply(inverse(cur), cur.t);  // LTB:485-487: the origin back in the tracking frame
    const Vec3f origin_local = apply(opt_f, origin_tracking);
    out.origin_in_local[0] = origin_local.x; out.origin_in_local[1] = origin_local.y; out.origin_in_local[2] = origin_local.z;
    out.num_returns = rs.num_returns; out.num_misses = rs.num_misses;
    out.num_high_resolution = rs.num_high_resolution; out.num_low_resolution = rs.num_low_resolution;
    // MotionFilter::IsSimilar (motion_filter.cc:37-57), against the builder's memory before this scan
    m.motion_filtered = b->motion_total + 1 > 1 && m.item->time - b->motion_last_time <= opt.motion_filter_max_time_seconds &&
        norm3(sub(opt_pose.t, b->motion_last_pose.t)) <= opt.motion_filter_max_distance_meters &&
        rotation_angle_d(compose(inverse(opt_pose), b->motion_last_pose).q) <= opt.motion_filter_max_angle_radians;
    const Slot& sl = slots[s];
    const Quatf gq{(float)opt_pose.q.w, (float)opt_pose.q.x, (float)opt_pose.q.y, (float)opt_pose.q.z};
    local_jobs.push_back(LocalFrameJob{f.returns_tracking + (size_t)s * f.cap * 3, f.misses_tracking + (size_t)s * f.cap * 3,
                                       rs.num_returns, rs.num_misses, opt_f, Rigidf{{0.f, 0.f, 0.f}, gq}, sl.returns_local,
                                       sl.misses_local, sl.aligned});
    if (m.motion_filtered) continue;
    // InsertIntoSubmap (LTB:584-622): the insertion submaps are queried BEFORE the insert
    out.num_insertion_submaps = (int32_t)b->active.size();
    for (size_t k = 0; k < b->active.size() && k < 2; ++k) out.insertion_submap_index[k] = b->active[k].index;
    out.inserted = 1;
    inserted.push_back(s);
  }
  DL_TRY(launch_local_frame(ctx, local_jobs.data(), (int)local_jobs.size(), d_local_jobs));
  // ---- ComputeHistogram(TransformPointCloud(returns in tracking, Rotation(gravity_alignment.cast<float>())), size): one launch,
  //      before the insertion, so that a cloud the histogram refuses fails the call while every grid is still untouched
  std::vector<HistogramScratch> hs;
  std::vector<const float*> hpts;
  std::vector<int64_t> hn;
  std::vector<float*> hout;
  for (int s : inserted) {
    if (r[s].num_returns > (1 << 20)) return ctx->fail(DL_ERR_ARG, "more than 2^20 points in a rotational histogram");
    hs.push_back(slots[s].hs);
    hpts.push_back(slots[s].aligned);
    hn.push_back(r[s].num_returns);
    hout.push_back(slots[s].histogram);
  }
  DL_TRY(launch_rotational_histograms(ctx, hs.data(), hpts.data(), hn.data(), (int)hs.size(), H, hout.data(), d_hist_args));
  if (!inserted.empty()) {  // the error flags, gathered on the device: one read-back
    for (size_t j = 0; j < inserted.size(); ++j)
      DL_CUDA(ctx, cudaMemcpyAsync(d_hist_err + j, hs[j].counters + 1, sizeof(int32_t), cudaMemcpyDeviceToDevice, ctx->stream));
    std::vector<int32_t> hist_err(inserted.size(), 0);
    DL_TRY(d2h(ctx, hist_err.data(), d_hist_err, hist_err.size()));
    DL_TRY(sync(ctx));
    for (int32_t e : hist_err)
      if (e) return ctx->fail(DL_ERR_ARG, "a point lies outside +-2^19 slices of 0.2 m");
  }
  // ---- insertion into both active submaps of every inserted member at both resolutions (Submap3D::InsertRangeData): no grid
  //      appears twice (distinct builders, distinct submaps), so all jobs run side by side
  std::vector<TransformJob> transforms;
  std::vector<InsertJob> inserts;
  for (int s : inserted) {
    const LtbMember& m = ms[part[s]];
    int k = 0;
    for (const LtbSubmap& sm : m.b->active) {
      double sp[7];
      pose_to7(sm.local_pose, sp);
      TransformJob t;
      InsertJob ij[2];
      submap_insert_jobs(sm.hi, sm.lo, sp, opt.high_resolution_max_range, m.out.origin_in_local, slots[s].returns_local,
                         m.out.num_returns, slots[s].ins[k++], &t, ij);
      transforms.push_back(t);
      inserts.insert(inserts.end(), ij, ij + 2);
    }
  }
  if (!inserts.empty()) {
    DL_TRY(launch_transform_filter(ctx, transforms.data(), (int)transforms.size(), d_transform_jobs));
    DL_TRY(upload_odds_tables(ctx, io, is));
    DL_TRY(insert_range_data_device(ctx, inserts.data(), (int)inserts.size(), io.num_free_space_voxels, is.hit_table, is.miss_table,
                                    is.bbox, is.args));
  }
  // ---- the nodes' clouds and the histograms, gathered on the device and read back in one copy
  struct Piece {
    std::vector<float>* dst;
    const float* src;
  };
  std::vector<Piece> pieces;
  for (int s : ok) {
    LtbMember& m = ms[part[s]];
    const Slot& sl = slots[s];
    const int32_t counts[4] = {r[s].num_returns, r[s].num_misses, r[s].num_high_resolution, r[s].num_low_resolution};
    const float* src[4] = {sl.returns_local, sl.misses_local, f.clouds + (size_t)(2 * s) * f.cap * 3,
                           f.clouds + (size_t)(2 * s + 1) * f.cap * 3};
    for (int c = 0; c < 4; ++c) {
      m.clouds[c].resize((size_t)counts[c] * 3);
      pieces.push_back(Piece{&m.clouds[c], src[c]});
    }
  }
  for (int s : inserted) {
    LtbMember& m = ms[part[s]];
    m.histogram.assign(H, 0.f);
    pieces.push_back(Piece{&m.histogram, slots[s].histogram});
  }
  size_t at = 0;
  for (const Piece& p : pieces) {
    if (!p.dst->empty())
      DL_CUDA(ctx, cudaMemcpyAsync(d_gather + at, p.src, p.dst->size() * sizeof(float), cudaMemcpyDeviceToDevice, ctx->stream));
    at += p.dst->size();
  }
  std::vector<float> gathered(at);
  DL_TRY(d2h(ctx, gathered.data(), d_gather, at));
  DL_TRY(sync(ctx));
  at = 0;
  for (const Piece& p : pieces) {
    if (!p.dst->empty()) std::memcpy(p.dst->data(), gathered.data() + at, p.dst->size() * sizeof(float));
    at += p.dst->size();
  }
  return DL_OK;
}
}  // namespace

extern "C" {

int dl_ltb_create(dl_context* ctx, const dl_ltb_options* options, dl_local_trajectory_builder** out) {
  if (!ctx || !options || !out) return DL_ERR_ARG;
  if (!(options->high_resolution > 0.f) || !(options->low_resolution > 0.f) || options->num_range_data < 1 ||
      options->rotational_histogram_size < 1 || options->rotational_histogram_size > 1024)
    return ctx->fail(DL_ERR_ARG, "dl_ltb_options: resolutions, num_range_data or rotational_histogram_size out of range");
  DL_TRY(check_ceres_options(ctx, &options->frontend.ceres_scan_matcher, 2));
  DL_TRY(check_inserter(ctx, &options->range_data_inserter));
  if (!options->two_stage) DL_TRY(check_imu_options(ctx, &options->frontend));  // the two-stage chain's plain solve takes only_optimize_yaw
  dl_local_trajectory_builder* b = new dl_local_trajectory_builder;
  b->ctx = ctx;
  b->opt = *options;
  b->opt.frontend.range_row_floats = 4;
  b->opt.frontend.host_scan_stride_rows = 0;
  // "We always want to have at least one submap ... create it at the origin" (submap_3d.cc:286-295)
  LtbSubmap first;
  const int st = ltb_make_grids(b, &first);
  if (st != DL_OK) {
    delete b;
    return st;
  }
  ltb_add_submap(b, Rigidd{{0, 0, 0}, {1, 0, 0, 0}}, first);
  *out = b;
  return DL_OK;
}

void dl_ltb_destroy(dl_local_trajectory_builder* b) {
  if (!b) return;
  for (auto* list : {&b->active, &b->finished})
    for (LtbSubmap& s : *list) {
      dl_grid_destroy(s.hi);
      dl_grid_destroy(s.lo);
    }
  delete b;
}

int dl_ltb_set_initial_state(dl_local_trajectory_builder* b, const dl_nav_state* state) {
  if (!b || !state) return DL_ERR_ARG;
  b->prev_state = *state;
  b->initialized = true;
  b->dt.clear(); b->acc.clear(); b->gyr.clear();
  b->reset_window_information();
  return DL_OK;
}

int dl_ltb_add_imu_data(dl_local_trajectory_builder* b, double time, const double* linear_acceleration, const double* angular_velocity) {
  if (!b || !linear_acceleration || !angular_velocity) return DL_ERR_ARG;
  if (!b->initialized) {  // init_imu_buffer_opt_ (LTB:165-176)
    b->init_acc.insert(b->init_acc.end(), linear_acceleration, linear_acceleration + 3);
    b->init_gyr.insert(b->init_gyr.end(), angular_velocity, angular_velocity + 3);
    return DL_OK;
  }
  const double dt = b->last_imu_time < 0 ? 1.0 / 500.0 : time - b->last_imu_time;  // LTB:183-185
  b->last_imu_time = time;
  b->dt.push_back(dt);
  b->acc.insert(b->acc.end(), linear_acceleration, linear_acceleration + 3);
  b->gyr.insert(b->gyr.end(), angular_velocity, angular_velocity + 3);
  return DL_OK;
}

int dl_ltb_add_range_data(dl_local_trajectory_builder* b, double time, const float* xyzt, int64_t n, const float* origin,
                          dl_matching_result* out) {
  return dl_ltb_add_synchronized_range_data(b, time, xyzt, n, 4, origin, 1, out);
}

int dl_ltb_add_synchronized_range_data(dl_local_trajectory_builder* b, double time, const void* rows, int64_t n, int32_t row_floats,
                                       const float* origin, int32_t num_origins, dl_matching_result* out) {
  if (!b) return DL_ERR_ARG;
  const dl_ltb_batch_item item{b, time, rows, n, row_floats, num_origins, origin};
  return dl_ltb_add_range_data_batch(1, &item, out);
}

int dl_ltb_add_range_data_batch(int32_t count, const dl_ltb_batch_item* items, dl_matching_result* results) {
  if (count < 0) return DL_ERR_ARG;
  if (count == 0) return DL_OK;
  if (!items || !results) return DL_ERR_ARG;
  // ---- validation: nothing is touched before every member has passed
  dl_context* ctx = items[0].builder ? items[0].builder->ctx : nullptr;
  for (int k = 0; k < count; ++k) {
    const dl_ltb_batch_item& it = items[k];
    dl_local_trajectory_builder* b = it.builder;
    if (!b || it.n < 0 || it.n > 0x3fffffff || (it.n > 0 && !it.rows) || !it.origins || it.num_origins < 1 ||
        (it.row_floats != 4 && it.row_floats != 8))
      return DL_ERR_ARG;
    if (it.row_floats == 4 && it.num_origins != 1) return b->ctx->fail(DL_ERR_ARG, "x y z t rows carry no origin index: one origin only");
    if (b->ctx != ctx) return b->ctx->fail(DL_ERR_ARG, "the builders of a batch must share one dl_context");
    for (int j = 0; j < k; ++j)
      if (items[j].builder == b) return ctx->fail(DL_ERR_ARG, "a builder appears twice in one batch");
    if (!same_ltb_options(b->opt, items[0].builder->opt))
      return ctx->fail(DL_ERR_ARG, "the builders of a batch must have equal dl_ltb_options");
  }
  const dl_ltb_options& opt = items[0].builder->opt;
  const bool two_stage = opt.two_stage != 0;
  const double gravity[3] = {0, 0, opt.gravity};
  // ---- who takes part in the device work: the members none of the single call's early returns applies to
  std::vector<LtbMember> ms(count);
  std::vector<int> part;  // members with a front-end scan, in batch order
  for (int k = 0; k < count; ++k) {
    LtbMember& m = ms[k];
    m.b = items[k].builder;
    m.item = &items[k];
    std::memset(&m.out, 0, sizeof(m.out));
    m.out.time = items[k].time;
    // "Range data collator filling buffer" (LTB:366-369); initialising (LTB:372-381); predicted_states_.empty(): no IMU since
    // the last scan (LTB:426)
    if (items[k].n == 0 || !m.b->initialized || m.b->dt.size() < 2) continue;
    m.slot = (int)part.size();
    part.push_back(k);
  }
  const int P = (int)part.size();
  if (P > 0) DL_TRY(ltb_batch_device(ctx, opt, two_stage, gravity, ms, part));
  // ---- the grids of the submaps this call hands over to, made before any builder changes: the commit below cannot fail
  for (LtbMember& m : ms) {
    if (m.slot < 0 || !m.out.inserted || m.b->active.back().num_range_data + 1 != opt.num_range_data) continue;
    const int st = ltb_make_grids(m.b, &m.next);
    if (st != DL_OK) {
      for (LtbMember& o : ms)
        if (o.hands_over) {
          dl_grid_destroy(o.next.hi);
          dl_grid_destroy(o.next.lo);
        }
      return st;
    }
    m.hands_over = true;
  }
  // ---- commit: every builder's host state, now that the device work has succeeded
  for (int k = 0; k < count; ++k) {
    LtbMember& m = ms[k];
    dl_local_trajectory_builder* b = m.b;
    if (items[k].n > 0 && !b->initialized) ltb_initialize_static(b);
    if (m.slot >= 0) ltb_commit(b, m, items[k].time);
    results[k] = m.out;
  }
  return DL_OK;
}

int dl_ltb_get_cloud(const dl_local_trajectory_builder* b, int32_t which, float* out, int64_t capacity_points, int64_t* num_points) {
  if (!b || which < 0 || which > 3 || !num_points) return DL_ERR_ARG;
  const std::vector<float>& c = b->clouds[which];
  *num_points = (int64_t)c.size() / 3;
  if (out && capacity_points >= *num_points) std::memcpy(out, c.data(), c.size() * sizeof(float));
  return DL_OK;
}

int dl_ltb_get_histogram(const dl_local_trajectory_builder* b, float* out, int32_t capacity) {
  if (!b || !out || capacity < (int32_t)b->histogram.size()) return DL_ERR_ARG;
  std::memcpy(out, b->histogram.data(), b->histogram.size() * sizeof(float));
  return DL_OK;
}

int32_t dl_ltb_num_submaps(const dl_local_trajectory_builder* b) { return b ? (int32_t)(b->finished.size() + b->active.size()) : 0; }

int dl_ltb_get_submap(dl_local_trajectory_builder* b, int32_t index, dl_grid** high_resolution_grid, dl_grid** low_resolution_grid,
                      double* local_pose, int32_t* num_range_data, int32_t* finished) {
  if (!b) return DL_ERR_ARG;
  for (auto* list : {&b->finished, &b->active})
    for (LtbSubmap& s : *list)
      if (s.index == index) {
        if (high_resolution_grid) *high_resolution_grid = s.hi;
        if (low_resolution_grid) *low_resolution_grid = s.lo;
        if (local_pose) pose_to7(s.local_pose, local_pose);
        if (num_range_data) *num_range_data = s.num_range_data;
        if (finished) *finished = s.finished;
        return DL_OK;
      }
  return b->ctx->fail(DL_ERR_ARG, "no submap with this index");
}

int dl_ltb_release_submap(dl_local_trajectory_builder* b, int32_t index) {
  if (!b) return DL_ERR_ARG;
  for (LtbSubmap& s : b->finished)
    if (s.index == index) {
      if (!s.hi) return b->ctx->fail(DL_ERR_ARG, "the submap's grids were already released");
      dl_grid_destroy(s.hi);
      dl_grid_destroy(s.lo);
      s.hi = s.lo = nullptr;
      return DL_OK;
    }
  for (const LtbSubmap& s : b->active)
    if (s.index == index) return b->ctx->fail(DL_ERR_ARG, "an active submap cannot be released");
  return b->ctx->fail(DL_ERR_ARG, "no submap with this index");
}

int dl_ltb_get_state(const dl_local_trajectory_builder* b, dl_nav_state* state, int32_t* initialized) {
  if (!b) return DL_ERR_ARG;
  if (state) *state = b->prev_state;
  if (initialized) *initialized = b->initialized ? 1 : 0;
  return DL_OK;
}

}  // extern "C"


// ------------------------------------------------------------------------------------------------ two-stage window (dl_window.cu)
extern "C" int dl_window_optimize_batch(dl_context* ctx, const dl_window_options* options, int32_t count, const dl_nav_state* states_i,
                                        const double* prior_information, const dl_preintegration* preintegrations,
                                        const double* matched_poses, const dl_nav_state* initial_states_j, dl_nav_state* states_i_out,
                                        dl_nav_state* states_j_out, double* information_out, dl_solve_summary* summaries) {
  if (!ctx || !options || count < 0) return DL_ERR_ARG;
  if (count == 0) return DL_OK;
  if (!states_i || !prior_information || !preintegrations || !matched_poses || !states_j_out || !information_out) return DL_ERR_ARG;
  dl_window_options o;
  DL_TRY(window_options_checked(ctx, *options, &o));
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  WindowBuffers w;
  DL_TRY(carve_scratch(ctx, [&](Arena& a) { carve_window(a, count, &w); }));
  return window_optimize(ctx, o, count, w, states_i, prior_information, preintegrations, matched_poses, initial_states_j,
                         states_i_out, states_j_out, information_out, summaries);
}

extern "C" int dl_window_evaluate(dl_context* ctx, const dl_window_options* options, int32_t count, const dl_nav_state* states_i,
                                  const double* prior_information, const dl_preintegration* preintegrations, const double* matched_poses,
                                  const dl_nav_state* x_i, const dl_nav_state* x_j, int32_t* ok, double* residuals, double* jacobians,
                                  double* weights) {
  if (!ctx || !options || count < 0) return DL_ERR_ARG;
  if (count == 0) return DL_OK;
  if (!states_i || !prior_information || !preintegrations || !matched_poses || !x_i || !x_j || !ok || !residuals || !jacobians ||
      !weights)
    return DL_ERR_ARG;
  dl_window_options o;
  DL_TRY(window_options_checked(ctx, *options, &o));
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t n = (size_t)count;
  dl_nav_state* d_si;
  dl_preintegration* d_pre;
  double *d_prior, *d_z, *d_x, *d_out;
  int32_t* d_ok;
  DL_TRY(carve_scratch(ctx, [&](Arena& a) {
    d_si = a.take<dl_nav_state>(n);
    d_prior = a.take<double>(n * 225);
    d_pre = a.take<dl_preintegration>(n);
    d_z = a.take<double>(n * 7);
    d_x = a.take<double>(n * 32);
    d_out = a.take<double>(n * kWindowEvalDoubles);
    d_ok = a.take<int32_t>(n);
  }));
  std::vector<double> x(n * 32);
  for (size_t k = 0; k < n; ++k)
    for (int s = 0; s < 2; ++s) {
      const dl_nav_state& v = (s == 0 ? x_i : x_j)[k];
      double* d = x.data() + 32 * k + 16 * s;
      for (int c = 0; c < 3; ++c) { d[c] = v.p[c]; d[7 + c] = v.v[c]; d[10 + c] = v.ba[c]; d[13 + c] = v.bg[c]; }
      for (int c = 0; c < 4; ++c) d[3 + c] = v.q[c];
    }
  DL_TRY(h2d(ctx, d_si, states_i, n));
  DL_TRY(h2d(ctx, d_prior, prior_information, n * 225));
  DL_TRY(h2d(ctx, d_pre, preintegrations, n));
  DL_TRY(h2d(ctx, d_z, matched_poses, n * 7));
  DL_TRY(h2d(ctx, d_x, x.data(), n * 32));
  DL_TRY(launch_window_evaluate(ctx, count, d_si, d_prior, d_pre, d_z, o, d_x, d_ok, d_out));
  std::vector<double> out(n * kWindowEvalDoubles);
  DL_TRY(d2h(ctx, ok, d_ok, n));
  DL_TRY(d2h(ctx, out.data(), d_out, out.size()));
  DL_TRY(sync(ctx));
  for (size_t k = 0; k < n; ++k) {
    const double* s = out.data() + k * kWindowEvalDoubles;
    std::memcpy(residuals + 38 * k, s, 38 * sizeof(double));
    std::memcpy(jacobians + 38 * 30 * k, s + 38, 38 * 30 * sizeof(double));
    std::memcpy(weights + 38 * 38 * k, s + 38 + 38 * 30, 38 * 38 * sizeof(double));
  }
  return DL_OK;
}
