// One-shot all-gather-reduce of the packed normal equations over NVLink peer memory (CUDA IPC):
// PUSH variant with tagged 16-byte words.  See vgx_comm_p2p_export / vgx_comm_p2p_import in
// include/voxgraph_b200.h and the protocol description in vgx_internal.h.
//
// Two parities suffice: a rank can only push epoch e+2 after its own gather of e+1 has finished
// (stream order), which needs every rank's elements of e+1, which a rank pushes only after its
// gather of e.
#include <stdlib.h>
#include <string.h>

#include "vgx_internal.h"

#define P2P_FLAG_BYTES 256
#define P2P_MAX_RANKS 8
#define P2P_ELEM_BYTES 16   // {value.lo32, tag, value.hi32, tag}

// separate-launch gather (VGX_P2P_FUSED=0): spin on the tagged elements, add them in rank order
__global__ void __launch_bounds__(256)
p2p_gather_kernel(VgxP2PGather G, double* __restrict__ out, size_t count,
                  const unsigned char* __restrict__ block_mask, int N) {
  vgx_ll_gather(G, out, count, (size_t)blockIdx.x * blockDim.x + threadIdx.x, (size_t)gridDim.x * blockDim.x,
                block_mask, N);
}

void vgx_p2p_free(vgx_ctx* c) {
  if (!c->p2p_base) return;
  vgx_drain(c);
  for (int r = 0; r < 8; ++r)
    if (c->p2p_peer[r] && c->p2p_peer[r] != c->p2p_base) cudaIpcCloseMemHandle(c->p2p_peer[r]);
  cudaFree(c->p2p_base);
  c->p2p_base = nullptr;
  memset(c->p2p_peer, 0, sizeof(c->p2p_peer));
  c->p2p_ready = false;
  c->p2p_cap = 0;
}

extern "C" int vgx_comm_p2p_export(vgx_ctx* c, uint64_t capacity_doubles, uint8_t handle[64]) {
  return vgx_entry(c, __func__, [&] {
    if (!handle || capacity_doubles == 0) return VGX_ERR_INVALID;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    vgx_p2p_free(c);
    const size_t cap = ((size_t)capacity_doubles + 31) & ~(size_t)31;
    // the rank count is not known yet: room for the 8 source ranks of one node, two parities
    const size_t bytes = P2P_FLAG_BYTES + 2 * (size_t)P2P_MAX_RANKS * cap * P2P_ELEM_BYTES;
    VGX_CUDA(c, cudaMalloc(&c->p2p_base, bytes));
    // zero before the handle leaves: the exchange protocol relies on a region that starts zeroed
    VGX_TRY(vgx_fill(c, static_cast<uint8_t*>(c->p2p_base), bytes));
    VGX_TRY(vgx_sync(c));
    cudaIpcMemHandle_t h;
    VGX_CUDA(c, cudaIpcGetMemHandle(&h, c->p2p_base));
    memcpy(handle, &h, 64);
    c->p2p_cap = cap;
    c->p2p_epoch = 0;
    return VGX_OK;
  });
}

extern "C" int vgx_comm_p2p_import(vgx_ctx* c, int nranks, int rank, const uint8_t* handles) {
  return vgx_entry(c, __func__, [&] {
    if (!handles || nranks < 1 || nranks > P2P_MAX_RANKS || rank < 0 || rank >= nranks) return VGX_ERR_INVALID;
    if (!c->p2p_base) VGX_FAIL(c, VGX_ERR_INVALID, "call vgx_comm_p2p_export first");
    if (c->nccl_comm && (c->nranks != nranks || c->rank != rank))
      VGX_FAIL(c, VGX_ERR_INVALID, "rank layout differs from vgx_comm_init");
    for (int r = 0; r < nranks; ++r) {
      if (r == rank) { c->p2p_peer[r] = c->p2p_base; continue; }
      cudaIpcMemHandle_t h;
      memcpy(&h, handles + 64 * (size_t)r, 64);
      void* p = nullptr;
      VGX_CUDA(c, cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
      c->p2p_peer[r] = p;
    }
    c->nranks = nranks;
    c->rank = rank;
    c->p2p_ready = true;
    {
      // one launch (assemble + push + wait + reduce) by default; VGX_P2P_FUSED=0 selects two launches
      const char* f = getenv("VGX_P2P_FUSED");
      c->p2p_fused = !(f && f[0] == '0');
      // a rank that lags (first-launch module load, table builds, uploads) must not look dead:
      // generous default, VGX_P2P_TIMEOUT_S overrides; callers barrier before the first exchange
      const char* t = getenv("VGX_P2P_TIMEOUT_S");
      double secs = t ? atof(t) : 30.0;
      if (!(secs > 0)) secs = 30.0;
      int khz = 1965000;
      cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, c->device);
      c->p2p_timeout_cycles = (long long)(secs * 1e3 * (double)khz);
    }
    vgx_graph_invalidate_registration(c);
    return VGX_OK;
  });
}

int vgx_p2p_check(vgx_ctx* c) {
  if (!c->p2p_ready) return VGX_OK;
  int t = 0;
  int* d_t = (int*)((char*)c->p2p_base + 128);
  VGX_TRY(vgx_read(c, &t, d_t));
  if (t) {
    VGX_TRY(vgx_fill(c, d_t, 1));   // not sticky: the next call starts clean
    VGX_FAIL(c, VGX_ERR_NCCL, "peer exchange timed out waiting for a rank (NVLink all-gather-reduce); "
                              "the result of that evaluation is NaN");
  }
  return VGX_OK;
}

static inline char* p2p_slot(void* region, size_t cap, unsigned long long epoch, int src_rank) {
  return (char*)region + P2P_FLAG_BYTES + ((epoch & 1) * P2P_MAX_RANKS + (size_t)src_rank) * cap * P2P_ELEM_BYTES;
}

int vgx_p2p_begin(vgx_ctx* c, size_t count, VgxP2PPush* push, VgxP2PGather* gat) {
  if (!c->p2p_ready) VGX_FAIL(c, VGX_ERR_INVALID, "peer exchange not initialised");
  if (count > c->p2p_cap) VGX_FAIL(c, VGX_ERR_CAPACITY, "packed normal equations exceed the exported peer buffer");
  unsigned long long e = ++c->p2p_epoch;
  if ((unsigned)e == 0u) e = (c->p2p_epoch += 2);   // tag 0 means "never written"; keep the parity alternating
  memset(push, 0, sizeof(*push));
  memset(gat, 0, sizeof(*gat));
  push->n = c->nranks;
  push->tag = (unsigned)e;
  gat->timeout_flag = (int*)((char*)c->p2p_base + 128);  // local word of the page, peers never touch it
  gat->timeout_cycles = c->p2p_timeout_cycles;
  gat->tag = (unsigned)e;
  gat->nranks = c->nranks;
  for (int r = 0; r < c->nranks; ++r) {
    push->dst[r] = (double*)p2p_slot(c->p2p_peer[r], c->p2p_cap, e, c->rank);   // my slot in rank r's region
    gat->slot[r] = p2p_slot(c->p2p_base, c->p2p_cap, e, r);                    // rank r's slot in my region
  }
  return VGX_OK;
}

int vgx_p2p_gather(vgx_ctx* c, const VgxP2PGather& gat, double* d_out, size_t count,
                   const unsigned char* d_block_mask, int N) {
  VgxProfileScope s(c, VGX_SLOT_OTHER);
  const int blocks = (int)((count + 1023) / 1024) > 0 ? (int)((count + 1023) / 1024) : 1;
  return vgx_launch(c, p2p_gather_kernel, blocks < 64 ? blocks : 64, 256, 0, VgxLaunch::plain, gat, d_out, count,
                    d_block_mask, N);
}

extern "C" int vgx_comm_suspend(vgx_ctx* c, int on) {
  return vgx_entry(c, __func__, [&] {
    if (on) {
      if (c->saved_nranks == 0) {
        c->saved_nranks = c->nranks;
        c->saved_rank = c->rank;
        c->nranks = 1;
        c->rank = 0;
        vgx_graph_invalidate_registration(c);
      }
    } else if (c->saved_nranks != 0) {
      c->nranks = c->saved_nranks;
      c->rank = c->saved_rank;
      c->saved_nranks = 0;
      c->saved_rank = 0;
      vgx_graph_invalidate_registration(c);
    }
    return VGX_OK;
  });
}
