// C-ABI of libdliom_b200.so (declared in include/dliom_b200.h): contexts, device memory and the device grid mirror. Every other
// subsystem keeps its entry points in the unit that holds its kernels.
// There is deliberately no CPU implementation of anything here: without a CUDA device every call fails.
#include <algorithm>
#include <cstring>
#include <new>

#include "dl_internal.cuh"

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

}  // extern "C"

namespace dl {
// Host mirror <- device (after device-side insertion the device copy is ahead).
int grid_download(dl_grid* g) {
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
