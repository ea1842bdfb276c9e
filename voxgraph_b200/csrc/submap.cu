// Context + brick store: voxblox::Layer/Block/AnyIndexHash replacement in HBM.
// Reference semantics: SURVEY.md Appendix A.2 (voxblox core) as used by
// voxgraph/src/frontend/submap_collection/voxgraph_submap.cpp.
#include <math.h>
#include <string.h>

#include <limits.h>

#include <algorithm>
#include <new>
#include <stdexcept>
#include <string>
#include <vector>

#include "layer_access.cuh"

// ------------------------------------------------------------------ context
extern "C" int vgx_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  return n;
}

extern "C" int vgx_ctx_create(int device, vgx_ctx** out) {
  return vgx_entry_noctx([&] {
    if (!out) return VGX_ERR_INVALID;
    *out = nullptr;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0 || device < 0 || device >= n)
      return VGX_ERR_CUDA;  // no CPU fallback: the product path needs a GPU
    if (cudaSetDevice(device) != cudaSuccess) return VGX_ERR_CUDA;
    vgx_ctx* c = new vgx_ctx();
    c->device = device;
    if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreate(&c->ev0) != cudaSuccess || cudaEventCreate(&c->ev1) != cudaSuccess) {
      delete c;
      return VGX_ERR_CUDA;
    }
    *out = c;
    return VGX_OK;
  });
}

extern "C" void vgx_ctx_destroy(vgx_ctx* c) {
  vgx_entry_noctx([&] {
    if (!c) return VGX_OK;
    vgx_comm_destroy(c);   // as an entry point, it selects the context's device
    vgx_drain(c);
    vgx_p2p_free(c);
    vgx_graph_free(c);
    for (auto& kv : c->submaps) delete kv.second;
    cudaEventDestroy(c->ev0);
    cudaEventDestroy(c->ev1);
    cudaStreamDestroy(c->stream);
    delete c;
    return VGX_OK;
  });
}

extern "C" const char* vgx_last_error(const vgx_ctx* c) { return c ? c->error.c_str() : "null context"; }
extern "C" void* vgx_ctx_stream(vgx_ctx* c) { return c ? (void*)c->stream : nullptr; }
extern "C" int vgx_ctx_synchronize(vgx_ctx* c) {
  return vgx_entry(c, __func__, [&] { return vgx_sync(c); });
}

extern "C" int vgx_profile_enable(vgx_ctx* c, int on) {
  return vgx_entry(c, __func__, [&] {
    c->profile = on != 0;
    return VGX_OK;
  });
}
extern "C" int vgx_profile_reset(vgx_ctx* c) {
  return vgx_entry(c, __func__, [&] {
    vgx_reset_counts(c);
    return VGX_OK;
  });
}
extern "C" int vgx_profile_get(vgx_ctx* c, int which, double* total_ms, int64_t* launches) {
  return vgx_entry(c, __func__, [&] {
    if (which < 0 || which >= VGX_PROFILE_SLOTS) return VGX_ERR_INVALID;
    if (total_ms) *total_ms = c->prof[which].total_ms;
    if (launches) *launches = c->prof[which].launches;
    return VGX_OK;
  });
}
extern "C" int64_t vgx_launch_count(vgx_ctx* c) { return c ? c->launches : 0; }

const char* vgx_status_name(int rc) {
  static const char* const names[] = {"invalid argument", "CUDA error", "not found", "out of memory",
                                      "NCCL error", "capacity exceeded"};   // VGX_ERR_INVALID ... VGX_ERR_CAPACITY
  return rc <= VGX_ERR_INVALID && rc >= VGX_ERR_CAPACITY ? names[VGX_ERR_INVALID - rc] : "error";
}

int vgx_caught(vgx_ctx* c) noexcept {
  int rc = VGX_ERR_NOMEM;
  const char* what = "out of host memory";
  try {
    throw;
  } catch (const std::bad_alloc&) {
  } catch (const std::length_error&) {
  } catch (const std::exception& e) {
    rc = VGX_ERR_INVALID;
    what = e.what();
  } catch (...) {
    rc = VGX_ERR_INVALID;
    what = "unknown exception";
  }
  try {
    if (c) c->set_error(what);
  } catch (...) {   // no memory for the message either: the status alone tells
  }
  return rc;
}

int vgx_submap_get(vgx_ctx* c, uint32_t id, VgxSubmap** out, VgxNeed need) {
  VgxSubmap* s = c->find(id);
  if (!s) VGX_FAIL(c, VGX_ERR_NOT_FOUND, "unknown submap " + std::to_string(id));
  if (need != VgxNeed::any && s->finished != (need == VgxNeed::finished))
    VGX_FAIL(c, VGX_ERR_INVALID, "submap " + std::to_string(id) + (s->finished ? " is finished" : " is not finished"));
  *out = s;
  return VGX_OK;
}

// ------------------------------------------------------------------ kernels
__global__ void hash_clear_kernel(VgxHashEntry* entries, uint32_t size) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < size) {
    VgxHashEntry e;
    e.key = VGX_EMPTY_KEY;
    e.val = -1;
    e.pad = 0;
    entries[i] = e;
  }
}

// Insert n blocks (slot = position in the list).  With `bad` non-null the list is caller input:
// a block index outside [VGX_BLOCK_INDEX_MIN, VGX_BLOCK_INDEX_MAX] sets bit 2 and is not inserted,
// a repeated index sets bit 1 (the writers race, so which slot it maps to is undefined).
__global__ void hash_insert_kernel(VgxHash h, const int32_t* block_idx, int n, int* bad) {
  int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const int bx = block_idx[3 * s], by = block_idx[3 * s + 1], bz = block_idx[3 * s + 2];
  if (bad && !(vgx_block_index_ok(bx) && vgx_block_index_ok(by) && vgx_block_index_ok(bz))) {
    atomicOr(bad, 2);
    return;
  }
  const uint64_t key = vgx_pack_key(bx, by, bz);
  uint32_t i = vgx_hash_index(bx, by, bz, h.mask);
  for (;;) {
    unsigned long long prev =
        atomicCAS((unsigned long long*)&h.entries[i].key, (unsigned long long)VGX_EMPTY_KEY,
                  (unsigned long long)key);
    if (prev == VGX_EMPTY_KEY || prev == key) {
      if (prev == key && bad) atomicOr(bad, 1);
      h.entries[i].val = s;
      return;
    }
    i = (i + 1) & h.mask;
  }
}

// Reads back hash_insert_kernel's input flag of an upload (d_counters[2]); on a bad block list the
// new submap is dropped and the upload fails.
static int check_uploaded_blocks(vgx_ctx* c, VgxSubmap* s) {
  int bad = 0;
  VGX_TRY(vgx_read(c, &bad, s->d_counters.get() + 2));
  if (!bad) return VGX_OK;
  vgx_submap_drop(c, s->id);
  VGX_FAIL(c, VGX_ERR_INVALID, (bad & 2) ? "block index outside the accepted range" : "repeated block index");
}

// (distance[], weight[]) -> interleaved float2 bricks.
__global__ void interleave_kernel(const float* __restrict__ d, const float* __restrict__ w,
                                  float2* __restrict__ dw, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  dw[i] = make_float2(d[i], w[i]);
}

// Registration view: one thread per voxel gathers its 2x2x2 forward neighbourhood (across
// brick faces through the hash) and stores the 8 distances, NaN where
// utils::isObservedVoxel (weight > 1e-6) fails or the neighbour block does not exist.
__global__ void __launch_bounds__(256)
build_view_kernel(LayerDev L, float* __restrict__ view) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= vgx_voxel_count(L.n_blocks, L.sh)) return;
  int v[3];
  const int slot = vgx_voxel_of(i, L.sh, v);
  const int b[3] = {L.block_idx[3 * slot], L.block_idx[3 * slot + 1], L.block_idx[3 * slot + 2]};
  int s[8];
  vgx_forward_slots(L.hash, b, v, slot, L.sh, s);
  float o[8];
#pragma unroll
  for (int m = 0; m < 8; ++m) {   // offset m = (x, y, z) bits (0, 1, 2) is corner x = bit 2, y = bit 1, z = bit 0
    float d = __int_as_float(0x7fc00000);
    if (s[m] >= 0) {
      const float2 q = L.dw[vgx_voxel_index(s[m], vgx_voxel_in_block(v[0] + (m & 1), L.sh),
                                            vgx_voxel_in_block(v[1] + ((m >> 1) & 1), L.sh),
                                            vgx_voxel_in_block(v[2] + (m >> 2), L.sh), L.sh)];
      if (q.y > 1e-6f) d = q.x;
    }
    o[((m & 1) << 2) | (m & 2) | (m >> 2)] = d;
  }
  float4* dst = reinterpret_cast<float4*>(view + i * 8);
  dst[0] = make_float4(o[0], o[1], o[2], o[3]);
  dst[1] = make_float4(o[4], o[5], o[6], o[7]);
}

__global__ void deinterleave_kernel(const float2* __restrict__ dw, float* __restrict__ d,
                                    float* __restrict__ w, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float2 v = dw[i];
  d[i] = v.x;
  w[i] = v.y;
}

// Dense block index over the blocks' AABB (host-built: off the hot path, once per finished submap).
#define VGX_GRID_MAX_CELLS 4096
int vgx_submap_build_grid(vgx_ctx* c, VgxSubmap* s) {
  s->d_grid.reset();
  s->d_grid16.reset();
  s->grid_dim[0] = s->grid_dim[1] = s->grid_dim[2] = 0;
  const int n = s->n_blocks;
  if (n <= 0) return VGX_OK;
  std::vector<int32_t> idx(3 * (size_t)n);
  VGX_TRY(vgx_read(c, idx.data(), s->d_block_idx.get(), idx.size()));
  int lo[3] = {INT_MAX, INT_MAX, INT_MAX}, hi[3] = {INT_MIN, INT_MIN, INT_MIN};
  for (int i = 0; i < n; ++i)
    for (int a = 0; a < 3; ++a) {
      lo[a] = std::min(lo[a], idx[3 * i + a]);
      hi[a] = std::max(hi[a], idx[3 * i + a]);
    }
  const long long cells = (long long)(hi[0] - lo[0] + 1) * (hi[1] - lo[1] + 1) * (hi[2] - lo[2] + 1);
  // sparse / huge: registration uses the hash (the kernel stages the grid as 16-bit slots)
  if (cells > VGX_GRID_MAX_CELLS || n >= 0xFFFF) return VGX_OK;
  std::vector<int32_t> grid((size_t)cells, -1);
  const int dx = hi[0] - lo[0] + 1, dy = hi[1] - lo[1] + 1;
  for (int i = 0; i < n; ++i)
    grid[(size_t)(idx[3 * i + 2] - lo[2]) * dy * dx + (size_t)(idx[3 * i + 1] - lo[1]) * dx +
         (idx[3 * i] - lo[0])] = i;
  VGX_TRY(s->d_grid.alloc(c, sizeof(int32_t) * cells, "dense block grid"));
  VGX_TRY(vgx_upload(c, s->d_grid.get(), grid.data(), grid.size()));
  // 16-bit copy for the registration kernel's shared-memory grid (one bulk copy per tile)
  std::vector<uint16_t> g16(((size_t)cells + 7) & ~(size_t)7, 0xFFFF);
  for (long long k = 0; k < cells; ++k) g16[(size_t)k] = grid[(size_t)k] < 0 ? 0xFFFF : (uint16_t)grid[(size_t)k];
  VGX_TRY(s->d_grid16.alloc(c, sizeof(uint16_t) * g16.size(), "dense block grid"));
  VGX_TRY(vgx_upload(c, s->d_grid16.get(), g16.data(), g16.size()));
  VGX_TRY(vgx_sync(c));
  for (int a = 0; a < 3; ++a) { s->grid_min[a] = lo[a]; s->grid_dim[a] = hi[a] - lo[a] + 1; }
  return VGX_OK;
}

int vgx_submap_build_view(vgx_ctx* c, VgxSubmap* s, int which) {
  const size_t used = (size_t)s->n_blocks * s->vox_per_block;
  if (used == 0) return VGX_OK;
  return vgx_launch(c, build_view_kernel, (unsigned)((used + 255) / 256), 256, 0, VgxLaunch::plain, layer_of(s, which),
                    which == VGX_LAYER_ESDF ? s->d_view_esdf.get() : s->d_view.get());
}

int vgx_submap_rebuild_hash(vgx_ctx* c, VgxSubmap* s) {
  const uint32_t tsize = s->hash_mask + 1;
  VGX_TRY(vgx_launch(c, hash_clear_kernel, (tsize + 255) / 256, 256, 0, VgxLaunch::plain, s->d_hash.get(), tsize));
  if (s->n_blocks == 0) return VGX_OK;
  return vgx_launch(c, hash_insert_kernel, (s->n_blocks + 127) / 128, 128, 0, VgxLaunch::plain, s->hash(),
                    s->d_block_idx.get(), s->n_blocks, nullptr);
}

// ------------------------------------------------------------------ submap management
static uint32_t table_size_for(int cap) {
  uint32_t t = 64;
  while (t < (uint32_t)cap * 2u) t <<= 1;
  return t;
}

int vgx_submap_alloc(vgx_ctx* c, uint32_t id, float voxel_size, int vps, int cap, bool with_view,
                        VgxSubmap** out) {
  if (!(voxel_size > 0) || !vgx_vps_ok(vps) || cap < 0)
    VGX_FAIL(c, VGX_ERR_INVALID, "invalid voxel_size / voxels_per_side / capacity");
  VgxSubmap* old = c->find(id);
  if (old) {
    VGX_TRY(vgx_sync(c));
    delete old;
    c->submaps.erase(id);
    vgx_graph_invalidate_registration(c);
  }
  VgxSubmap* s = new VgxSubmap();
  s->id = id;
  s->voxel_size = voxel_size;
  // voxblox Layer ctor: inverses by double division, stored as float
  s->voxel_size_inv = (float)(1.0 / (double)voxel_size);
  s->block_size = voxel_size * (float)vps;
  s->block_size_inv = (float)(1.0 / (double)s->block_size);
  s->vps = vps;
  s->sh = 0;
  while ((1 << s->sh) < vps) s->sh++;
  s->vox_per_block = vps * vps * vps;
  s->cap_blocks = cap > 0 ? cap : 1;
  const uint32_t tsize = table_size_for(s->cap_blocks);
  s->hash_mask = tsize - 1;
  const size_t nvox = (size_t)s->cap_blocks * s->vox_per_block;
  const char* what = "submap allocation";
  int rc = s->d_hash.alloc(c, sizeof(VgxHashEntry) * tsize, what, VGX_ERR_NOMEM);
  if (rc == VGX_OK) rc = s->d_block_idx.alloc(c, sizeof(int32_t) * 3 * s->cap_blocks, what, VGX_ERR_NOMEM);
  if (rc == VGX_OK) rc = s->d_dw.alloc(c, sizeof(float2) * nvox, what, VGX_ERR_NOMEM);
  if (rc == VGX_OK && with_view) rc = s->d_view.alloc(c, sizeof(float) * 8 * nvox, what, VGX_ERR_NOMEM);
  if (rc == VGX_OK) rc = s->d_counters.alloc(c, sizeof(int) * 4, what, VGX_ERR_NOMEM);
  if (rc == VGX_OK)
    rc = vgx_launch(c, hash_clear_kernel, (tsize + 255) / 256, 256, 0, VgxLaunch::plain, s->d_hash.get(), tsize);
  if (rc != VGX_OK) {
    delete s;
    return rc;
  }
  VGX_TRY(vgx_fill(c, s->d_counters.get(), 4));
  c->submaps[id] = s;
  *out = s;
  return VGX_OK;
}

extern "C" int vgx_submap_upload(vgx_ctx* c, uint32_t id, float voxel_size, int vps, int n_blocks,
                                 const int32_t* block_idx, const float* distance,
                                 const float* weight) {
  return vgx_entry(c, __func__, [&] {
    if (n_blocks < 0 || (n_blocks > 0 && (!block_idx || !distance || !weight)))
      VGX_FAIL(c, VGX_ERR_INVALID, "null input");
    VgxSubmap* s = nullptr;
    VGX_TRY(vgx_submap_alloc(c, id, voxel_size, vps, n_blocks, true, &s));
    s->n_blocks = n_blocks;
    s->finished = true;
    if (n_blocks == 0) return VGX_OK;
    const size_t nvox = (size_t)n_blocks * s->vox_per_block;
    float *tmp_d, *tmp_w;
    VGX_TRY(vgx_carve(c, c->d_scratch, vgx_part(tmp_d, nvox), vgx_part(tmp_w, nvox)));
    VGX_TRY(vgx_upload(c, tmp_d, distance, nvox));
    VGX_TRY(vgx_upload(c, tmp_w, weight, nvox));
    VGX_TRY(vgx_upload(c, s->d_block_idx.get(), block_idx, 3 * (size_t)n_blocks));
    VGX_TRY(vgx_launch(c, interleave_kernel, (unsigned)((nvox + 255) / 256), 256, 0, VgxLaunch::plain, tmp_d, tmp_w,
                       s->d_dw.get(), nvox));
    // synchronises: the host buffers are the caller's
    return vgx_submap_upload_finish(c, s);
  });
}

extern "C" int vgx_submap_peek_device(vgx_ctx* c, uint32_t id, const int32_t** d_block_idx,
                                      const float** d_dw, int* n_blocks) {
  return vgx_entry(c, __func__, [&] {
    VgxSubmap* s;
    VGX_TRY(vgx_submap_get(c, id, &s));
    VGX_TRY(vgx_sync(c));   // the caller reads the bricks on its own stream
    if (d_block_idx) *d_block_idx = s->d_block_idx.get();
    if (d_dw) *d_dw = reinterpret_cast<const float*>(s->d_dw.get());
    if (n_blocks) *n_blocks = s->n_blocks;
    return VGX_OK;
  });
}

extern "C" int vgx_submap_upload_device(vgx_ctx* c, uint32_t id, float voxel_size, int vps, int n_blocks,
                                        const int32_t* d_block_idx, const float* d_dw) {
  return vgx_entry(c, __func__, [&] {
    if (n_blocks < 0 || (n_blocks > 0 && (!d_block_idx || !d_dw))) VGX_FAIL(c, VGX_ERR_INVALID, "null input");
    VgxSubmap* s = nullptr;
    VGX_TRY(vgx_submap_alloc(c, id, voxel_size, vps, n_blocks, true, &s));
    s->n_blocks = n_blocks;
    s->finished = true;
    if (n_blocks == 0) return VGX_OK;
    const size_t nvox = (size_t)n_blocks * s->vox_per_block;
    VGX_TRY(vgx_copy(c, s->d_block_idx.get(), d_block_idx, 3 * (size_t)n_blocks));
    VGX_TRY(vgx_copy(c, s->d_dw.get(), reinterpret_cast<const float2*>(d_dw), nvox));   // (distance, weight) pairs
    // synchronises: the source buffers are the caller's
    return vgx_submap_upload_finish(c, s);
  });
}

// ------------------------------------------------------------------ colour channel
int vgx_submap_ensure_colour(vgx_ctx* c, VgxSubmap* s) {
  if (s->d_rgba.get()) return VGX_OK;
  const size_t words = (size_t)s->cap_blocks * s->vox_per_block;
  VgxBuffer<uint32_t> q;
  VGX_TRY(q.alloc(c, sizeof(uint32_t) * words, "submap colour channel", VGX_ERR_NOMEM));
  VGX_TRY(vgx_fill(c, q.get(), words));
  s->d_rgba = std::move(q);
  return VGX_OK;
}

extern "C" int vgx_submap_has_colour(vgx_ctx* c, uint32_t id, int* has) {
  return vgx_entry(c, __func__, [&] {
    if (!has) return VGX_ERR_INVALID;
    VgxSubmap* s;
    VGX_TRY(vgx_submap_get(c, id, &s));
    *has = s->d_rgba.get() ? 1 : 0;
    return VGX_OK;
  });
}

extern "C" int vgx_submap_download_colour(vgx_ctx* c, uint32_t id, int max_blocks, uint32_t* rgba, int* n_out) {
  return vgx_entry(c, __func__, [&] {
    VgxSubmap* s;
    VGX_TRY(vgx_submap_get(c, id, &s));
    const int n = s->n_blocks;
    if (n_out) *n_out = n;
    if (n > max_blocks) VGX_FAIL(c, VGX_ERR_CAPACITY, "max_blocks too small");
    if (n == 0 || !rgba) return VGX_OK;
    const size_t words = (size_t)n * s->vox_per_block;
    if (!s->d_rgba.get()) {
      memset(rgba, 0, sizeof(uint32_t) * words);
      return VGX_OK;
    }
    return vgx_read(c, rgba, s->d_rgba.get(), words);
  });
}

// the channel of submap id from n_blocks x vps^3 words in host or device memory; the submap keeps its
// previous channel (or none) when anything fails
static int upload_colour(vgx_ctx* c, uint32_t id, int n_blocks, const uint32_t* rgba, bool on_device) {
  VgxSubmap* s;
  VGX_TRY(vgx_submap_get(c, id, &s));
  if (n_blocks != s->n_blocks) VGX_FAIL(c, VGX_ERR_INVALID, "n_blocks differs from the submap's");
  if (n_blocks > 0 && !rgba) VGX_FAIL(c, VGX_ERR_INVALID, "null input");
  const size_t cap_words = (size_t)s->cap_blocks * s->vox_per_block;
  const size_t words = (size_t)n_blocks * s->vox_per_block;
  VgxBuffer<uint32_t> q;
  VGX_TRY(q.alloc(c, sizeof(uint32_t) * cap_words, "colour channel", VGX_ERR_NOMEM));
  VGX_TRY(vgx_fill(c, q.get(), cap_words));
  if (words) VGX_TRY(on_device ? vgx_copy(c, q.get(), rgba, words) : vgx_upload(c, q.get(), rgba, words));
  // synchronises: the source is the caller's, and the stream may still read the old channel
  VGX_TRY(vgx_sync(c));
  s->d_rgba = std::move(q);
  return VGX_OK;
}

extern "C" int vgx_submap_upload_colour(vgx_ctx* c, uint32_t id, int n_blocks, const uint32_t* rgba) {
  return vgx_entry(c, __func__, [&] { return upload_colour(c, id, n_blocks, rgba, false); });
}

extern "C" int vgx_submap_peek_device_colour(vgx_ctx* c, uint32_t id, const uint32_t** d_rgba) {
  return vgx_entry(c, __func__, [&] {
    if (!d_rgba) return VGX_ERR_INVALID;
    VgxSubmap* s;
    VGX_TRY(vgx_submap_get(c, id, &s));
    VGX_TRY(vgx_sync(c));   // the caller reads the channel on its own stream
    *d_rgba = s->d_rgba.get();
    return VGX_OK;
  });
}

extern "C" int vgx_submap_upload_device_colour(vgx_ctx* c, uint32_t id, int n_blocks, const uint32_t* d_rgba) {
  return vgx_entry(c, __func__, [&] { return upload_colour(c, id, n_blocks, d_rgba, true); });
}

int vgx_submap_upload_finish(vgx_ctx* c, VgxSubmap* s) {
  if (s->n_blocks == 0) return VGX_OK;
  VGX_TRY(vgx_upload(c, s->d_counters.get(), &s->n_blocks, 1));
  VGX_TRY(vgx_launch(c, hash_insert_kernel, (s->n_blocks + 127) / 128, 128, 0, VgxLaunch::plain, s->hash(),
                     s->d_block_idx.get(), s->n_blocks, s->d_counters.get() + 2));
  VGX_TRY(vgx_submap_build_view(c, s, VGX_LAYER_TSDF));
  VGX_TRY(check_uploaded_blocks(c, s));
  return vgx_submap_build_grid(c, s);
}

extern "C" int vgx_submap_create(vgx_ctx* c, uint32_t id, float voxel_size, int vps, int capacity) {
  return vgx_entry(c, __func__, [&] {
    if (capacity <= 0) VGX_FAIL(c, VGX_ERR_INVALID, "capacity must be > 0");
    VgxSubmap* s = nullptr;
    VGX_TRY(vgx_submap_alloc(c, id, voxel_size, vps, capacity, false, &s));
    // new voxblox blocks are zero-initialised (distance 0, weight 0)
    VGX_TRY(vgx_fill(c, s->d_dw.get(), (size_t)capacity * s->vox_per_block));
    s->finished = false;
    return VGX_OK;
  });
}

extern "C" int vgx_submap_finish(vgx_ctx* c, uint32_t id) {
  return vgx_entry(c, __func__, [&] {
    VgxSubmap* s;
    VGX_TRY(vgx_submap_get(c, id, &s));
    // the layer is frozen from here on: the view only needs the blocks that exist, not the
    // integration capacity (128 KiB per brick)
    const size_t used = (size_t)s->n_blocks * s->vox_per_block;
    if (!s->d_view.get()) {
      VGX_TRY(s->d_view.alloc(c, sizeof(float) * 8 * (used > 0 ? used : 1), "registration view"));
    }
    VGX_TRY(vgx_submap_build_view(c, s, VGX_LAYER_TSDF));
    s->finished = true;
    vgx_graph_invalidate_registration(c);
    return vgx_submap_build_grid(c, s);
  });
}

extern "C" int vgx_submap_free(vgx_ctx* c, uint32_t id) {
  return vgx_entry(c, __func__, [&] {
    VgxSubmap* s;
    VGX_TRY(vgx_submap_get(c, id, &s));
    VGX_TRY(vgx_sync(c));
    delete s;
    c->submaps.erase(id);
    vgx_graph_invalidate_registration(c);
    return VGX_OK;
  });
}

void vgx_submap_drop(vgx_ctx* c, uint32_t id) {
  if (c->find(id)) vgx_submap_free(c, id);
}

int vgx_submap_move(vgx_ctx* c, uint32_t from_id, uint32_t id) {
  VgxSubmap* s;
  VGX_TRY(vgx_submap_get(c, from_id, &s));
  VGX_TRY(vgx_sync(c));
  VgxSubmap* old = c->find(id);
  delete old;
  c->submaps.erase(from_id);
  s->id = id;
  c->submaps[id] = s;
  vgx_graph_invalidate_registration(c);
  return VGX_OK;
}

uint32_t vgx_scratch_id(vgx_ctx* c) {
  uint32_t id = 0xFFFFFFFEu;
  while (c->find(id)) --id;
  return id;
}

extern "C" int vgx_submap_block_count(vgx_ctx* c, uint32_t id, int* n) {
  return vgx_entry(c, __func__, [&] {
    if (!n) return VGX_ERR_INVALID;
    VgxSubmap* s;
    VGX_TRY(vgx_submap_get(c, id, &s));
    *n = s->n_blocks;
    return VGX_OK;
  });
}

extern "C" int vgx_submap_info(vgx_ctx* c, uint32_t id, float* voxel_size, int* vps, int* n_blocks,
                               int* finished) {
  return vgx_entry(c, __func__, [&] {
    VgxSubmap* s;
    VGX_TRY(vgx_submap_get(c, id, &s));
    if (voxel_size) *voxel_size = s->voxel_size;
    if (vps) *vps = s->vps;
    if (n_blocks) *n_blocks = s->n_blocks;
    if (finished) *finished = s->finished ? 1 : 0;
    return VGX_OK;
  });
}

extern "C" int vgx_submap_download(vgx_ctx* c, uint32_t id, int max_blocks, int32_t* block_idx,
                                   float* distance, float* weight, int* n_out) {
  return vgx_entry(c, __func__, [&] {
    VgxSubmap* s;
    VGX_TRY(vgx_submap_get(c, id, &s));
    const int n = s->n_blocks;
    if (n_out) *n_out = n;
    if (n > max_blocks) VGX_FAIL(c, VGX_ERR_CAPACITY, "max_blocks too small");
    if (n == 0) return VGX_OK;
    const size_t nvox = (size_t)n * s->vox_per_block;
    if (block_idx) VGX_TRY(vgx_download(c, block_idx, s->d_block_idx.get(), 3 * (size_t)n));
    if (distance || weight) {
      float *tmp_d, *tmp_w;
      VGX_TRY(vgx_carve(c, c->d_scratch, vgx_part(tmp_d, nvox), vgx_part(tmp_w, nvox)));
      VGX_TRY(vgx_launch(c, deinterleave_kernel, (unsigned)((nvox + 255) / 256), 256, 0, VgxLaunch::plain,
                         s->d_dw.get(), tmp_d, tmp_w, nvox));
      if (distance) VGX_TRY(vgx_download(c, distance, tmp_d, nvox));
      if (weight) VGX_TRY(vgx_download(c, weight, tmp_w, nvox));
    }
    return vgx_sync(c);
  });
}

extern "C" int vgx_submap_upload_points(vgx_ctx* c, uint32_t id, int type, int n, const float* xyz,
                                        const float* distance, const float* weight) {
  return vgx_entry(c, __func__, [&] {
    if (type < 0 || type > 1 || n < 0 || (n > 0 && (!xyz || !distance || !weight)))
      VGX_FAIL(c, VGX_ERR_INVALID, "invalid argument");
    VgxSubmap* s;
    VGX_TRY(vgx_submap_get(c, id, &s));
    VGX_TRY(vgx_sync(c));
    VgxPoints& p = s->points[type];
    p = VgxPoints();
    vgx_graph_invalidate_registration(c);
    if (n == 0) return VGX_OK;
    // unit-major AoSoA staging on the host (pinned): unit u = {x[32], y[32], z[32], d[32], w[32]}
    const size_t units = ((size_t)n + VGX_PT_UNIT - 1) / VGX_PT_UNIT;
    const size_t floats = units * VGX_PT_UNIT_FLOATS;
    float* h;
    VGX_TRY(vgx_carve(c, c->h_pinned, vgx_part(h, floats)));
    memset(h, 0, floats * sizeof(float));
    double sum_w = 0;
    std::vector<double> cumulative((size_t)n);
    for (int i = 0; i < n; ++i) {
      float* u = h + vgx_pt_index((size_t)i, 0);
      u[0] = xyz[3 * (size_t)i];
      u[32] = xyz[3 * (size_t)i + 1];
      u[64] = xyz[3 * (size_t)i + 2];
      u[96] = distance[i];
      u[128] = weight[i];
      sum_w += (double)weight[i];  // cpp:124, in point order
      cumulative[i] = sum_w;       // WeightedSampler::addItem (weighted_sampler_inl.h:6-17)
    }
    VgxBuffer<float> d;
    VGX_TRY(d.alloc(c, floats * sizeof(float), "points upload"));
    VGX_TRY(vgx_upload(c, d.get(), h, floats));
    VGX_TRY(vgx_sync(c));
    p.n = n;
    p.data = std::move(d);
    p.sum_w = sum_w;
    p.cumulative_w.swap(cumulative);
    return VGX_OK;
  });
}

// ------------------------------------------------------------------ WeightedSampler
// weighted_sampler_inl.h:19-28: r = uniform_real_distribution<double>(0,1)(mt19937),
// index = upper_bound(cumulative, r * cumulative.back()).  std::mt19937's default seed (5489)
// and uniform_real_distribution are what the reference instantiates (weighted_sampler.h:34-36).
// fl(r * back) can round up to back itself, where upper_bound returns end(): the reference then
// indexes one past the last item; clamped here.
void vgx_points_draw(VgxPoints& p, int count, int32_t* idx) {
  std::uniform_real_distribution<double> uniform(0.0, 1.0);
  const std::vector<double>& cw = p.cumulative_w;
  for (int i = 0; i < count; ++i) {
    const double r = uniform(p.rng);
    const double t = r * cw.back();
    size_t k = (size_t)(std::upper_bound(cw.begin(), cw.end(), t) - cw.begin());
    if (k >= cw.size()) k = cw.size() - 1;
    idx[i] = (int32_t)k;
  }
}

extern "C" int vgx_submap_draw_samples(vgx_ctx* c, uint32_t id, int type, int n, int32_t* indices) {
  return vgx_entry(c, __func__, [&] {
    if (type < 0 || type > 1 || n < 0 || (n > 0 && !indices)) VGX_FAIL(c, VGX_ERR_INVALID, "invalid argument");
    VgxSubmap* s;
    VGX_TRY(vgx_submap_get(c, id, &s));
    VgxPoints& p = s->points[type];
    if (p.n == 0) VGX_FAIL(c, VGX_ERR_INVALID, "the submap has no registration points");
    vgx_points_draw(p, n, indices);
    return VGX_OK;
  });
}
