// Multi-GPU exchange steps of the path, issued from the C-ABI over NCCL (NVLink / NVSwitch within a box).
//
// One process per GPU; the scan-to-submap problems are independent, so the front end itself needs no collective. The steps
// that do exchange data are the ones the reference hands to its constraint-builder thread pool and its pose graph
// (SURVEY 8e): every rank searches the (node, submap) pairs whose submap it OWNS (constraint_builder_3d.cc:189-197) and the
// found constraints (constraint_builder_3d.cc:328-333) are all-gathered so that every rank holds the same table for the
// replicated pose graph; the pose graph's normal-equation blocks are all-reduced in fp64 (dl_posegraph_sparse.cu); a finished submap
// moves between ranks by one broadcast of its brick arrays.
//
// NCCL is bound at run time (dlopen of libnccl.so.2, the library the host process already uses when it is a
// torch.distributed program), so single-GPU users do not need it installed. The communicator is created from a 128-byte
// unique id that the host program distributes however it likes (MPI, a file, torch.distributed's store).
#include <dlfcn.h>
#include <nccl.h>

#include <cstring>

#include "dl_internal.cuh"

namespace {

struct NcclApi {
  void* handle = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  std::string error;
};

NcclApi* nccl_api() {
  static NcclApi* api = [] {
    NcclApi* a = new NcclApi;
    a->handle = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!a->handle) {
      a->error = std::string("libnccl.so.2 could not be loaded: ") + dlerror();
      return a;
    }
    auto sym = [&](const char* name) {
      void* p = dlsym(a->handle, name);
      if (!p && a->error.empty()) a->error = std::string("libnccl.so.2 lacks ") + name;
      return p;
    };
    a->GetUniqueId = (decltype(a->GetUniqueId))sym("ncclGetUniqueId");
    a->CommInitRank = (decltype(a->CommInitRank))sym("ncclCommInitRank");
    a->CommDestroy = (decltype(a->CommDestroy))sym("ncclCommDestroy");
    a->AllGather = (decltype(a->AllGather))sym("ncclAllGather");
    a->AllReduce = (decltype(a->AllReduce))sym("ncclAllReduce");
    a->Broadcast = (decltype(a->Broadcast))sym("ncclBroadcast");
    a->GetErrorString = (decltype(a->GetErrorString))sym("ncclGetErrorString");
    return a;
  }();
  return api;
}

thread_local std::string g_comm_error;

int nccl_fail(dl_context* ctx, ncclResult_t r, const char* what) {
  NcclApi* a = nccl_api();
  const std::string msg = std::string(what) + ": " + (a->GetErrorString ? a->GetErrorString(r) : "NCCL error");
  if (ctx) ctx->error = msg;
  g_comm_error = msg;
  return DL_ERR_CUDA;
}

#define DL_NCCL(ctx, call)                                  \
  do {                                                      \
    const ncclResult_t r__ = (call);                        \
    if (r__ != ncclSuccess) return nccl_fail(ctx, r__, #call); \
  } while (0)

}  // namespace

struct dl_comm {
  dl_context* ctx = nullptr;
  ncclComm_t comm = nullptr;
  int rank = 0, world = 1;
  dl::DeviceBuffer<uint8_t> d_send;   // staging for the constraint exchange
  dl::DeviceBuffer<uint8_t> d_recv;   // world times d_send's bytes
  cudaEvent_t e0 = nullptr, e1 = nullptr;
};

namespace dl {

int comm_reserve(dl_comm* c, size_t bytes_per_rank) {
  if (bytes_per_rank <= c->d_send.cap && bytes_per_rank * c->world <= c->d_recv.cap) return DL_OK;
  const size_t want = bytes_per_rank + bytes_per_rank / 2 + 1024;
  DL_TRY(grow(c->ctx, c->d_recv, want * (size_t)c->world));
  return grow(c->ctx, c->d_send, want);
}
void* comm_send_buffer(dl_comm* c) { return c->d_send.get(); }
void* comm_recv_buffer(dl_comm* c) { return c->d_recv.get(); }

// recv[r * bytes .. (r+1) * bytes) = rank r's send[0 .. bytes); device-timed with events on the context's stream.
int comm_all_gather(dl_comm* c, const void* send_dev, void* recv_dev, size_t bytes, float* ms) {
  dl_context* ctx = c->ctx;
  NcclApi* a = nccl_api();
  if (ms) DL_CUDA(ctx, cudaEventRecord(c->e0, ctx->stream));
  DL_NCCL(ctx, a->AllGather(send_dev, recv_dev, bytes, ncclChar, c->comm, ctx->stream));
  if (ms) {
    DL_CUDA(ctx, cudaEventRecord(c->e1, ctx->stream));
    DL_CUDA(ctx, ctx->blocking_sync ? ctx->wait_stream() : cudaEventSynchronize(c->e1));
    DL_CUDA(ctx, cudaEventElapsedTime(ms, c->e0, c->e1));
  }
  return DL_OK;
}

}  // namespace dl

extern "C" {

const char* dl_comm_last_error(void) { return g_comm_error.c_str(); }

int dl_comm_unique_id(uint8_t* id128) {
  if (!id128) return DL_ERR_ARG;
  NcclApi* a = nccl_api();
  if (!a->error.empty()) {
    g_comm_error = a->error;
    return DL_ERR_CUDA;
  }
  ncclUniqueId id;
  const ncclResult_t r = a->GetUniqueId(&id);
  if (r != ncclSuccess) return nccl_fail(nullptr, r, "ncclGetUniqueId");
  static_assert(sizeof(id) == DL_COMM_ID_BYTES, "ncclUniqueId size");
  std::memcpy(id128, &id, sizeof(id));
  return DL_OK;
}

int dl_comm_create(dl_context* ctx, const uint8_t* id128, int32_t rank, int32_t world, dl_comm** out) {
  if (!ctx || !id128 || !out || world < 1 || rank < 0 || rank >= world) return DL_ERR_ARG;
  NcclApi* a = nccl_api();
  if (!a->error.empty()) return ctx->fail(DL_ERR_CUDA, a->error);
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  dl_comm* c = new dl_comm;
  c->ctx = ctx;
  c->rank = rank;
  c->world = world;
  ncclUniqueId id;
  std::memcpy(&id, id128, sizeof(id));
  const ncclResult_t r = a->CommInitRank(&c->comm, world, id, rank);
  if (r != ncclSuccess) {
    delete c;
    return nccl_fail(ctx, r, "ncclCommInitRank");
  }
  cudaEventCreate(&c->e0);
  cudaEventCreate(&c->e1);
  *out = c;
  return DL_OK;
}

void dl_comm_destroy(dl_comm* c) {
  if (!c) return;
  cudaSetDevice(c->ctx->device);
  c->ctx->wait_stream();
  if (c->comm) nccl_api()->CommDestroy(c->comm);
  if (c->e0) cudaEventDestroy(c->e0);
  if (c->e1) cudaEventDestroy(c->e1);
  delete c;
}

int32_t dl_comm_rank(const dl_comm* c) { return c ? c->rank : -1; }
int32_t dl_comm_world_size(const dl_comm* c) { return c ? c->world : 0; }

int dl_comm_all_gather_dev(dl_comm* c, const void* send_dev, void* recv_dev, int64_t bytes_per_rank) {
  if (!c || !send_dev || !recv_dev || bytes_per_rank < 0) return DL_ERR_ARG;
  if (bytes_per_rank == 0) return DL_OK;
  DL_CUDA(c->ctx, cudaSetDevice(c->ctx->device));
  return dl::comm_all_gather(c, send_dev, recv_dev, (size_t)bytes_per_rank, nullptr);
}

int dl_comm_all_reduce_f64_dev(dl_comm* c, double* buffer_dev, int64_t count) {
  if (!c || !buffer_dev || count < 0) return DL_ERR_ARG;
  if (count == 0) return DL_OK;
  dl_context* ctx = c->ctx;
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  DL_NCCL(ctx, nccl_api()->AllReduce(buffer_dev, buffer_dev, (size_t)count, ncclDouble, ncclSum, c->comm, ctx->stream));
  return DL_OK;
}

int dl_comm_broadcast_dev(dl_comm* c, void* buffer_dev, int64_t bytes, int32_t root) {
  if (!c || !buffer_dev || bytes < 0 || root < 0 || root >= c->world) return DL_ERR_ARG;
  if (bytes == 0) return DL_OK;
  dl_context* ctx = c->ctx;
  DL_CUDA(ctx, cudaSetDevice(ctx->device));
  DL_NCCL(ctx, nccl_api()->Broadcast(buffer_dev, buffer_dev, (size_t)bytes, ncclChar, root, c->comm, ctx->stream));
  return DL_OK;
}

}  // extern "C"
