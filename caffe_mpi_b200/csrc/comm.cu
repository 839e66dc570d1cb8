// comm.cu -- gradient exchange over NCCL (NVLink 4 / NVSwitch), one communicator per process.
//
// Replaces the NCCL use of P2PManager / P2PSync (reference src/caffe/parallel.cpp:36-87,
// 145-253: ncclGetUniqueId + MPI_Bcast, ncclCommInitRank between MPI_Barriers, ncclBcast of the
// initial weights, in-place ncclSum ncclAllReduce of each diff bucket followed by a host
// cudaStreamSynchronize) and the MPI bootstrap of src/caffe/clusters.cpp:8-16.  Differences by
// design: one process per GPU (no solver threads, no boost barriers, no GPUMemory write-lock),
// every call is asynchronous on the caller's stream -- ordering against the backward pass and the
// SGD kernel is done with CUDA events by the caller (caffe_mpi_b200/host), never by host syncs.
#include <nccl.h>
#include "b2c_common.cuh"

#include <stdlib.h>
#include <vector>

struct b2c_comm {
  ncclComm_t comm;
  int nranks, rank;
  std::vector<void*> handles;      // ncclCommRegister handles, released at destroy
};

#define B2C_NCCL_OK(expr)                                                                          \
  do {                                                                                             \
    ncclResult_t r__ = (expr);                                                                     \
    if (r__ != ncclSuccess)                                                                        \
      return ::b2c::fail(B2C_ERR_NCCL, "%s:%d %s: %s", __FILE__, __LINE__, #expr, ncclGetErrorString(r__)); \
  } while (0)

static_assert(sizeof(ncclUniqueId) == B2C_UNIQUE_ID_BYTES, "ncclUniqueId size");

extern "C" int b2c_comm_get_unique_id(void* id_out) {
  if (!id_out) return b2c::fail(B2C_ERR_INVALID, "b2c_comm_get_unique_id: null");
  ncclUniqueId id;
  B2C_NCCL_OK(ncclGetUniqueId(&id));
  memcpy(id_out, &id, sizeof(id));
  return B2C_OK;
}

extern "C" int b2c_comm_init(int nranks, int rank, const void* id, b2c_comm** out) {
  if (!id || !out || nranks < 1 || rank < 0 || rank >= nranks)
    return b2c::fail(B2C_ERR_INVALID, "b2c_comm_init: bad argument");
  ncclUniqueId uid;
  memcpy(&uid, id, sizeof(uid));
  b2c_comm* c = new b2c_comm{nullptr, nranks, rank, {}};
  // B2C_NCCL_MAX_CTAS: cap the CTAs NCCL may use per collective.  The tensor-core conv kernels are persistent with one CTA per
  // SM, so an allreduce overlapped with backward only gets SMs at kernel tails; fewer, NVLS-fed CTAs disturb them less.
  ncclConfig_t cfg = NCCL_CONFIG_INITIALIZER;
  if (const char* e = getenv("B2C_NCCL_MAX_CTAS")) { const int v = atoi(e); if (v > 0) cfg.maxCTAs = v; }
  if (const char* e = getenv("B2C_NCCL_MIN_CTAS")) { const int v = atoi(e); if (v > 0) cfg.minCTAs = v; }
  ncclResult_t r = ncclCommInitRankConfig(&c->comm, nranks, uid, rank, &cfg);
  if (r != ncclSuccess) {
    delete c;
    return b2c::fail(B2C_ERR_NCCL, "ncclCommInitRank: %s", ncclGetErrorString(r));
  }
  *out = c;
  return B2C_OK;
}

extern "C" int b2c_comm_destroy(b2c_comm* c) {
  if (!c) return B2C_OK;
  for (void* h : c->handles) ncclCommDeregister(c->comm, h);
  ncclCommDestroy(c->comm);
  delete c;
  return B2C_OK;
}

extern "C" int b2c_comm_nranks(const b2c_comm* c) { return c ? c->nranks : 0; }

extern "C" int b2c_comm_bcast(b2c_comm* c, float* buf, size_t count, int root, void* stream) {
  if (!c || !buf) return b2c::fail(B2C_ERR_INVALID, "b2c_comm_bcast: null");
  B2C_NCCL_OK(ncclBroadcast(buf, buf, count, ncclFloat, root, c->comm, b2c::as_stream(stream)));
  return B2C_OK;
}

extern "C" int b2c_comm_allreduce_sum(b2c_comm* c, float* buf, size_t count, void* stream) {
  if (!c || !buf) return b2c::fail(B2C_ERR_INVALID, "b2c_comm_allreduce_sum: null");
  B2C_NCCL_OK(ncclAllReduce(buf, buf, count, ncclFloat, ncclSum, c->comm, b2c::as_stream(stream)));
  return B2C_OK;
}

// ---- NVLS-friendly buffers ------------------------------------------------------------------------------------------------
// ncclMemAlloc hands out memory that can be mapped into the NVSwitch multicast space, ncclCommRegister registers it with a
// communicator: an in-place allreduce on such a buffer can use NVLS (in-switch reduction) without staging through NCCL's own
// buffers.  The host layer allocates the contiguous diff arena this way (ParamArena) and registers it in P2PSync::on_start.
extern "C" int b2c_comm_mem_alloc(void** ptr, size_t bytes) {
  if (!ptr || !bytes) return b2c::fail(B2C_ERR_INVALID, "b2c_comm_mem_alloc: bad argument");
  B2C_NCCL_OK(ncclMemAlloc(ptr, bytes));
  return B2C_OK;
}
extern "C" int b2c_comm_mem_free(void* ptr) {
  if (!ptr) return B2C_OK;
  B2C_NCCL_OK(ncclMemFree(ptr));
  return B2C_OK;
}
extern "C" int b2c_comm_register(b2c_comm* c, void* buf, size_t bytes) {
  if (!c || !buf || !bytes) return b2c::fail(B2C_ERR_INVALID, "b2c_comm_register: bad argument");
  void* h = nullptr;
  B2C_NCCL_OK(ncclCommRegister(c->comm, buf, bytes, &h));
  c->handles.push_back(h);
  return B2C_OK;
}
