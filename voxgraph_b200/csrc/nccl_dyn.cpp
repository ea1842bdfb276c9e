// NCCL binding resolved at run time (dlopen): the library uses whichever libnccl.so.2 the
// process already has (torch's bundled one under torchrun) or the system one, and has no
// link-time dependency on it.  Only the four entry points the path needs are declared.
#include <dlfcn.h>
#include <string.h>

#include <string>

#include "vgx_internal.h"

typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
typedef int ncclResult_t;
enum { ncclFloat64 = 8, ncclSum = 0 };

static struct {
  void* handle;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*);
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int);
  ncclResult_t (*CommDestroy)(ncclComm_t);
  ncclResult_t (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t);
  const char* (*GetErrorString)(ncclResult_t);
} g_nccl;

static bool nccl_load(std::string* err) {
  if (g_nccl.handle) return true;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  void* h = nullptr;
  for (const char* n : names) {
    h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (h) break;
  }
  if (!h) {
    if (err) *err = std::string("dlopen libnccl.so.2 failed: ") + dlerror();
    return false;
  }
  g_nccl.GetUniqueId = (ncclResult_t(*)(ncclUniqueId*))dlsym(h, "ncclGetUniqueId");
  g_nccl.CommInitRank = (ncclResult_t(*)(ncclComm_t*, int, ncclUniqueId, int))dlsym(h, "ncclCommInitRank");
  g_nccl.CommDestroy = (ncclResult_t(*)(ncclComm_t))dlsym(h, "ncclCommDestroy");
  g_nccl.AllReduce = (ncclResult_t(*)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t))dlsym(h, "ncclAllReduce");
  g_nccl.GetErrorString = (const char* (*)(ncclResult_t))dlsym(h, "ncclGetErrorString");
  if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.CommDestroy || !g_nccl.AllReduce) {
    if (err) *err = "libnccl is missing required symbols";
    dlclose(h);
    return false;
  }
  g_nccl.handle = h;
  return true;
}

extern "C" int vgx_comm_unique_id(uint8_t id[128]) {
  return vgx_entry_noctx([&] {
    if (!id) return VGX_ERR_INVALID;
    if (!nccl_load(nullptr)) return VGX_ERR_NCCL;
    ncclUniqueId u;
    if (g_nccl.GetUniqueId(&u) != 0) return VGX_ERR_NCCL;
    memcpy(id, u.internal, 128);
    return VGX_OK;
  });
}

extern "C" int vgx_comm_init(vgx_ctx* c, int nranks, int rank, const uint8_t id[128]) {
  return vgx_entry(c, __func__, [&] {
    if (!id || nranks < 1 || rank < 0 || rank >= nranks) return VGX_ERR_INVALID;
    std::string err;
    if (!nccl_load(&err)) VGX_FAIL(c, VGX_ERR_NCCL, err);
    vgx_comm_destroy(c);
    ncclUniqueId u;
    memcpy(u.internal, id, 128);
    ncclComm_t comm = nullptr;
    ncclResult_t r = g_nccl.CommInitRank(&comm, nranks, u, rank);
    if (r != 0)
      VGX_FAIL(c, VGX_ERR_NCCL, std::string("ncclCommInitRank: ") +
                                    (g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "error"));
    c->nccl_comm = comm;
    c->nranks = nranks;
    c->rank = rank;
    vgx_graph_invalidate_registration(c);
    return VGX_OK;
  });
}

extern "C" int vgx_comm_destroy(vgx_ctx* c) {
  return vgx_entry(c, __func__, [&] {
    if (c->nccl_comm && g_nccl.handle) {
      vgx_drain(c);
      g_nccl.CommDestroy((ncclComm_t)c->nccl_comm);
    }
    c->nccl_comm = nullptr;
    c->nranks = 1;
    c->rank = 0;
    return VGX_OK;
  });
}

int vgx_nccl_allreduce_sum_f64(vgx_ctx* c, double* d_buf, size_t count) {
  if (c->nranks <= 1) return VGX_OK;
  if (!c->nccl_comm) VGX_FAIL(c, VGX_ERR_NCCL, "communicator not initialised");
  ncclResult_t r = g_nccl.AllReduce(d_buf, d_buf, count, ncclFloat64, ncclSum,
                                    (ncclComm_t)c->nccl_comm, c->stream);
  if (r != 0)
    VGX_FAIL(c, VGX_ERR_NCCL, std::string("ncclAllReduce: ") +
                                  (g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "error"));
  return VGX_OK;
}
