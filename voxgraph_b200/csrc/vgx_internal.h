// Internal declarations shared by the translation units of libvoxgraph_b200.so.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <map>
#include <random>
#include <string>
#include <utility>
#include <vector>

#include "voxgraph_b200.h"

// ------------------------------------------------------------------ error handling
// Both set the context's message through vgx_ctx::set_error, which prefixes the entry point's name.
#define VGX_CUDA(ctx, expr)                                                            \
  do {                                                                                 \
    cudaError_t _e = (expr);                                                           \
    if (_e != cudaSuccess) {                                                           \
      (ctx)->set_error(std::string(#expr) + ": " + cudaGetErrorString(_e));            \
      return VGX_ERR_CUDA;                                                             \
    }                                                                                  \
  } while (0)

#define VGX_FAIL(ctx, code, msg) \
  do {                           \
    (ctx)->set_error(msg);       \
    return (code);               \
  } while (0)

// returns the status of a call that did not return VGX_OK (its message is already set)
#define VGX_TRY(expr)              \
  do {                             \
    const int _rc = (expr);        \
    if (_rc != VGX_OK) return _rc; \
  } while (0)

// ------------------------------------------------------------------ memory owner
// The one owner of device (cudaMalloc) and page-locked host (cudaMallocHost) allocations: a buffer
// of T that is freed by reset(), by its destructor or by a new allocation.  Move-only.  Freeing a
// buffer the stream may still read is the owner's caller's concern: it synchronises first.
// Kernel-facing structs hold the raw pointer, taken with get().
enum class VgxMem { device, pinned };
struct vgx_ctx;

template <class T = char>
class VgxBuffer {
 public:
  VgxBuffer() = default;
  explicit VgxBuffer(VgxMem kind) : kind_(kind) {}
  VgxBuffer(VgxBuffer&& o) noexcept { *this = std::move(o); }
  VgxBuffer& operator=(VgxBuffer&& o) noexcept {
    if (this != &o) {
      reset();
      std::swap(p_, o.p_);
      std::swap(bytes_, o.bytes_);
      std::swap(kind_, o.kind_);
    }
    return *this;
  }
  VgxBuffer(const VgxBuffer&) = delete;
  VgxBuffer& operator=(const VgxBuffer&) = delete;
  ~VgxBuffer() { reset(); }

  T* get() const { return p_; }
  size_t bytes() const { return bytes_; }
  void reset() {
    if (p_) kind_ == VgxMem::pinned ? cudaFreeHost(p_) : cudaFree(p_);
    p_ = nullptr;
    bytes_ = 0;
  }
  // frees what it holds and allocates `bytes`.  On failure the owner is empty, the context's error
  // reads "<what>: <CUDA error>" and the status is VGX_ERR_CUDA (`nomem` when out of memory).
  int alloc(vgx_ctx* c, size_t bytes, const char* what, int nomem = VGX_ERR_CUDA);
  // discard-and-grow: when it holds fewer than `need` bytes, a new allocation of need + need / 4
  // bytes replaces the old one and its contents
  int grow(vgx_ctx* c, size_t need, const char* what) {
    return need <= bytes_ ? VGX_OK : alloc(c, need + need / 4, what);
  }
  // grow-and-keep: as grow, but the first `used` bytes are copied over on the context's stream, which
  // is synchronised before the old allocation is freed; a failed allocation leaves the old one in place
  int grow_keep(vgx_ctx* c, size_t need, size_t used, const char* what);

 private:
  T* p_ = nullptr;
  size_t bytes_ = 0;
  VgxMem kind_ = VgxMem::device;
};

// ------------------------------------------------------------------ block hash
// voxblox AnyIndexHash (block_hash.h): x + 17191*y + 17191^2*z, then masked into an
// open-addressing table with linear probing. Keys pack the three 21-bit biased indices.
#define VGX_EMPTY_KEY 0xFFFFFFFFFFFFFFFFull

__host__ __device__ __forceinline__ uint64_t vgx_pack_key(int bx, int by, int bz) {
  return ((uint64_t)((uint32_t)(bx + (1 << 20)) & 0x1FFFFFu)) |
         ((uint64_t)((uint32_t)(by + (1 << 20)) & 0x1FFFFFu) << 21) |
         ((uint64_t)((uint32_t)(bz + (1 << 20)) & 0x1FFFFFu) << 42);
}
// the block index a key packs (the inverse of vgx_pack_key inside the range)
__host__ __device__ __forceinline__ void vgx_unpack_key(uint64_t key, int b[3]) {
  b[0] = (int)(key & 0x1FFFFFu) - (1 << 20);
  b[1] = (int)((key >> 21) & 0x1FFFFFu) - (1 << 20);
  b[2] = (int)((key >> 42) & 0x1FFFFFu) - (1 << 20);
}
// an uploaded block index component whose +-1 neighbours pack to keys of their own
__host__ __device__ __forceinline__ bool vgx_block_index_ok(int b) {
  return b >= VGX_BLOCK_INDEX_MIN && b <= VGX_BLOCK_INDEX_MAX;
}
// The range rule: no block exists outside [VGX_BLOCK_INDEX_MIN, VGX_BLOCK_INDEX_MAX] on any axis
// (uploads refuse one, integration never allocates one), so a lookup there is a miss without a probe.
// Inside the range vgx_pack_key is injective; outside it a key aliases a block 2^21 away.
__host__ __device__ __forceinline__ bool vgx_block_in_range(int bx, int by, int bz) {
  return vgx_block_index_ok(bx) && vgx_block_index_ok(by) && vgx_block_index_ok(bz);
}
__host__ __device__ __forceinline__ uint32_t vgx_hash_index(int bx, int by, int bz, uint32_t mask) {
  uint64_t h = (uint64_t)(int64_t)bx + (uint64_t)(int64_t)by * 17191ull +
               (uint64_t)(int64_t)bz * (17191ull * 17191ull);
  h ^= h >> 15;  // fold the high bits so power-of-two masking sees all three axes
  return (uint32_t)h & mask;
}

// One 16-byte entry per table slot so a probe is a single 128-bit load.
struct __align__(16) VgxHashEntry {
  uint64_t key;   // VGX_EMPTY_KEY when free
  int32_t val;    // brick slot (-1 while unmapped)
  int32_t pad;
};

struct VgxHash {
  VgxHashEntry* entries;
  uint32_t mask;    // table_size - 1
};

#ifdef __CUDACC__
// Read-only lookup (finished layers / kernels that do not insert concurrently).  At most
// table-size probes: a completely full table (capacity overflow) ends the search instead of
// spinning.  Entries with val < 0 (unmapped / overflowed) read as "no block", and so does an index
// outside the range (vgx_block_in_range).
__device__ __forceinline__ int vgx_hash_find(const VgxHash& h, int bx, int by, int bz) {
  if (!vgx_block_in_range(bx, by, bz)) return -1;
  const uint64_t key = vgx_pack_key(bx, by, bz);
  uint32_t i = vgx_hash_index(bx, by, bz, h.mask);
  for (uint32_t n = 0; n <= h.mask; ++n) {
    const int4 e = __ldg(reinterpret_cast<const int4*>(h.entries + i));
    const uint64_t k = (uint64_t)(uint32_t)e.x | ((uint64_t)(uint32_t)e.y << 32);
    if (k == key) return e.z < 0 ? -1 : e.z;
    if (k == VGX_EMPTY_KEY) return -1;
    i = (i + 1) & h.mask;
  }
  return -1;
}
#endif

// ------------------------------------------------------------------ submap store
// WeightedSampler<RegistrationPoint> in HBM, "unit-major" AoSoA: 32 points per unit,
// unit u = float[5][32] = {x[32], y[32], z[32], distance[32], weight[32]} = 640 contiguous
// bytes, so one cp.async.bulk (TMA 1-D) brings a warp's whole unit into shared memory and a warp
// reading lane-wise is coalesced.  Zero padded to a whole unit (weight 0 = no contribution).
#define VGX_PT_UNIT 32
#define VGX_PT_UNIT_FLOATS 160
struct VgxPoints {
  int n = 0;
  VgxBuffer<float> data;        // ceil(n / 32) units
  double sum_w = 0;             // summed_reference_weight (cpp:124), sequential double sum
  std::vector<double> cumulative_w;  // WeightedSampler::cumulative_item_weights_ (host, sampling mode)
  std::mt19937 rng;                  // WeightedSampler::random_number_generator_ (default seed)
};
__host__ __device__ __forceinline__ size_t vgx_pt_index(size_t i, int component) {
  return (i >> 5) * VGX_PT_UNIT_FLOATS + (size_t)component * VGX_PT_UNIT + (i & 31);
}

struct VgxSubmap {
  uint32_t id = 0;
  float voxel_size = 0, voxel_size_inv = 0, block_size = 0, block_size_inv = 0;
  int vps = 16, vox_per_block = 4096;
  int sh = 4;                  // log2(vps)
  int cap_blocks = 0;
  int n_blocks = 0;            // host mirror (valid after upload / integrate sync)
  bool finished = false;
  VgxBuffer<VgxHashEntry> d_hash;   // hash_mask + 1 entries
  uint32_t hash_mask = 0;
  VgxBuffer<int32_t> d_block_idx;  // cap x 3
  VgxBuffer<float2> d_dw;          // cap x vps^3 (distance, weight)
  // Optional colour channel, cap x vps^3 words in the layout of colour.cuh; empty (get() == nullptr) until
  // a coloured integration, vgx_submap_upload_colour / _upload_device_colour or the colour-keeping
  // collection loader creates it (vgx_submap_ensure_colour).  A submap without it runs every call as a
  // colour-free layer does.  +4 B per voxel.
  VgxBuffer<uint32_t> d_rgba;
  // Registration view ("octets"): for every voxel the distances of its 2x2x2 forward
  // neighbourhood (corner i: x = bit2, y = bit1, z = bit0; apron across bricks baked in),
  // NaN where the voxel is unobserved or its block missing. One 32-byte sector per point.
  VgxBuffer<float> d_view;         // cap x vps^3 x 8
  VgxBuffer<float2> d_esdf;        // ESDF bricks (distance, observed 1/0), n_blocks x vps^3 (vgx_submap_generate_esdf)
  VgxBuffer<float> d_view_esdf;    // registration view of the ESDF bricks
  VgxBuffer<int> d_counters;       // [0] = n_blocks (device), [1] = overflow flag, [2] = bad upload input
  // Dense block index over the AABB of the allocated blocks (finished submaps): slot or -1.
  // Small enough to be staged in shared memory by the registration kernel; the hash stays
  // the general structure (integration, view construction, sparse/huge submaps).
  VgxBuffer<int32_t> d_grid;
  VgxBuffer<uint16_t> d_grid16;   // 16-bit copy (0xFFFF = no block), padded to a multiple of 16 bytes
  int grid_min[3] = {0, 0, 0};
  int grid_dim[3] = {0, 0, 0};
  VgxPoints points[2];
  // vgx_submap_extract_points: surface OBB (cpp:280-324) and isosurface block slots (cpp:237-240)
  bool surface_obb_valid = false;
  float surface_obb_min[3] = {0, 0, 0}, surface_obb_max[3] = {0, 0, 0};
  std::vector<int> iso_blocks;
  bool points_extracted = false;
  VgxBuffer<int32_t> d_iso_idx;   // block indices of the isosurface blocks (n_iso x 3)
  int n_iso = 0;

  VgxHash hash() const { return {d_hash.get(), hash_mask}; }
};

// ------------------------------------------------------------------ pose graph
struct VgxRelEdge {
  int a, b;
  double t_obs[3], yaw_obs, L[16];
};

struct VgxGraph;  // defined in graph.h

struct VgxProfileSlot {   // one per VgxProfileSlotId (voxgraph_b200.h)
  double total_ms = 0;
  int64_t launches = 0;
};

struct vgx_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  std::string error;
  std::map<uint32_t, VgxSubmap*> submaps;
  VgxGraph* graph = nullptr;
  // profiling
  bool profile = false;
  VgxProfileSlot prof[VGX_PROFILE_SLOTS];
  int64_t launches = 0;
  int slot = -1;              // the slot of the innermost open VgxProfileScope, -1 outside every scope
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  // Scratch arenas.  They grow (discard-and-grow) and never shrink; a call lays its parts out in one
  // with vgx_carve, and the parts are valid until the next vgx_carve of the same arena.  A function
  // may hold parts of several arenas at once, but a callee must not carve an arena its caller holds
  // parts of: the arena may move.  A function that carves the same arena twice re-sends what the
  // first parts held.
  VgxBuffer<> d_scratch;   // a call's inputs and outputs on their way to or from the host
  VgxBuffer<> d_work;      // a pass's working buffers: counts, offsets, flags, scan and sort temp
  VgxBuffer<> d_work2;     // the second set of a pass that holds d_work parts (sort tuples, candidates)
  VgxBuffer<> h_pinned{VgxMem::pinned};   // page-locked host staging of copies to and from the device
  // NCCL
  void* nccl_comm = nullptr;
  int nranks = 1, rank = 0;
  int saved_nranks = 0, saved_rank = 0;   // vgx_comm_suspend
  // NVLink peer exchange (CUDA IPC): region = [flags 256 B | buf0 | buf1]
  void* p2p_base = nullptr;        // own region
  void* p2p_peer[8] = {nullptr};   // mapped regions of all ranks (own entry = p2p_base)
  size_t p2p_cap = 0;              // doubles per buffer
  unsigned long long p2p_epoch = 0;
  bool p2p_ready = false;
  bool p2p_fused = true;           // one-launch assemble + exchange (VGX_P2P_FUSED=0: two launches)
  long long p2p_timeout_cycles = 0;
  // separated submap mesh of the last vgx_mesh_build (mesh.cu)
  VgxBuffer<float> d_mesh_xyz;        // n_vertices x 3
  VgxBuffer<uint32_t> d_mesh_tri;     // n_triangles x 3
  VgxBuffer<uint32_t> d_mesh_rgba;    // n_vertices colour words; empty unless a submap of the build has a colour channel
  std::vector<uint8_t> mesh_has_colour;   // per submap of the build: it has a colour channel
  int64_t mesh_nv = 0, mesh_nt = 0;
  std::vector<uint32_t> mesh_ids;     // the submaps of the build, in build order
  std::vector<int64_t> mesh_voff;     // their first vertices (+ the total)
  bool mesh_table_ready = false;      // triangle table in this device's constant memory
  // the entry point the caller called, while it runs (vgx_entry); nullptr between calls
  const char* entry = nullptr;

  void set_error(const std::string& e) { error = std::string(entry ? entry : "voxgraph_b200") + ": " + e; }
  VgxSubmap* find(uint32_t id) {
    auto it = submaps.find(id);
    return it == submaps.end() ? nullptr : it->second;
  }
};

// ------------------------------------------------------------------ C-ABI guard
// Every extern "C" entry point with a context runs its body through vgx_entry.  The outermost call on a
// context records its name, clears the message, selects the context's device and runs the body inside
// try: std::bad_alloc and std::length_error become VGX_ERR_NOMEM, any other exception VGX_ERR_INVALID with
// its what().  A failure the body left without a message reads "<name>: <status>"; VGX_OK leaves the
// message empty.  An entry point called from inside another one only runs its body, so its messages name
// the outer call and its exceptions reach the outer guard.  A null context is VGX_ERR_INVALID.
int vgx_caught(vgx_ctx* c) noexcept;   // the status (and message, with c) of the exception being handled
const char* vgx_status_name(int rc);

template <class F>
int vgx_entry(vgx_ctx* c, const char* name, F&& body) {
  if (!c) return VGX_ERR_INVALID;
  if (c->entry) return body();
  c->entry = name;
  int rc;
  try {
    c->error.clear();
    rc = [&] {
      VGX_CUDA(c, cudaSetDevice(c->device));
      return body();
    }();
    if (rc == VGX_OK) c->error.clear();
    else if (rc < 0 && c->error.empty()) c->set_error(vgx_status_name(rc));
  } catch (...) {
    rc = vgx_caught(c);
  }
  c->entry = nullptr;
  return rc;
}

// the same for the entry points without a context: exceptions become a status, with no message
template <class F>
int vgx_entry_noctx(F&& body) noexcept {
  try {
    return body();
  } catch (...) {
    return vgx_caught(nullptr);
  }
}

// The submap `id`: VGX_ERR_NOT_FOUND ("unknown submap <id>") when the context has none, VGX_ERR_INVALID
// when it is not finished (need = finished) or is finished (need = active).
enum class VgxNeed { any, finished, active };
int vgx_submap_get(vgx_ctx* c, uint32_t id, VgxSubmap** out, VgxNeed need = VgxNeed::any);

template <class T>
int VgxBuffer<T>::alloc(vgx_ctx* c, size_t bytes, const char* what, int nomem) {
  reset();
  void* p = nullptr;
  const cudaError_t e = kind_ == VgxMem::pinned ? cudaMallocHost(&p, bytes) : cudaMalloc(&p, bytes);
  if (e != cudaSuccess) {
    c->set_error(std::string(what) + ": " + cudaGetErrorString(e));
    return e == cudaErrorMemoryAllocation ? nomem : VGX_ERR_CUDA;
  }
  p_ = static_cast<T*>(p);
  bytes_ = bytes;
  return VGX_OK;
}

// ------------------------------------------------------------------ scratch layout
// one part of a vgx_carve layout: n elements of T at *at
template <class T>
struct VgxPart {
  T*& at;
  size_t bytes;
};
template <class T>
VgxPart<T> vgx_part(T*& at, size_t n) { return {at, sizeof(T) * n}; }
static inline size_t vgx_part_span(size_t bytes) { return (bytes + 255) & ~(size_t)255; }

// Lays the parts out in `arena` in order, each rounded up to 256 bytes (so every part starts
// 256-byte aligned), growing the arena to the total first; no CUDA call when it is large enough.
template <class... T>
int vgx_carve(vgx_ctx* c, VgxBuffer<>& arena, VgxPart<T>... parts) {
  VGX_TRY(arena.grow(c, (vgx_part_span(parts.bytes) + ...), "scratch arena"));
  char* at = arena.get();
  ((parts.at = reinterpret_cast<T*>(at), at += vgx_part_span(parts.bytes)), ...);
  return VGX_OK;
}

// ------------------------------------------------------------------ kernel launches
// The one place that counts launches and writes the profile slots.  A profile scope names the slot of the
// launches inside it and, while profiling is enabled, times its region into that slot with two events on the
// context's stream.  A launch outside every scope counts in the total only.
struct VgxProfileScope {
  vgx_ctx* c;
  int slot, outer;
  VgxProfileScope(vgx_ctx* ctx, int s) : c(ctx), slot(s), outer(ctx->slot) {
    c->slot = s;
    if (c->profile) cudaEventRecord(c->ev0, c->stream);
  }
  ~VgxProfileScope() {
    if (c->profile) {
      cudaEventRecord(c->ev1, c->stream);
      cudaEventSynchronize(c->ev1);
      float ms = 0;
      cudaEventElapsedTime(&ms, c->ev0, c->ev1);
      c->prof[slot].total_ms += ms;
    }
    c->slot = outer;
  }
};

// one launch into the total and the open scope's slot; a library call that launches kernels of its own
// (a cub sort) counts as one launch through this call
static inline void vgx_count_launch(vgx_ctx* c) {
  ++c->launches;
  if (c->slot >= 0) ++c->prof[c->slot].launches;
}

// vgx_profile_reset: every slot and the total back to zero
static inline void vgx_reset_counts(vgx_ctx* c) {
  for (auto& p : c->prof) p = VgxProfileSlot();
  c->launches = 0;
}

// plain: as <<<>>>.  pdl: programmatic stream serialisation, the kernel may be scheduled while the one
// ahead of it on the stream is still running and waits for it at griddepcontrol.wait.  cooperative: the
// grid is co-resident as a whole (grid-wide synchronisation).
enum class VgxLaunch { plain, pdl, cooperative };

// Every kernel of the library is launched here, on the context's stream, with its arguments converted
// as <<<>>> converts them.  A launch that fails leaves no last error behind for a later check to find:
// the message is set as VGX_CUDA sets it and the status is VGX_ERR_CUDA.
template <class... P, class... A>
int vgx_launch(vgx_ctx* c, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, VgxLaunch mode,
               A&&... args) {
  cudaLaunchAttribute attr = {};
  if (mode == VgxLaunch::pdl) {
    attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr.val.programmaticStreamSerializationAllowed = 1;
  } else if (mode == VgxLaunch::cooperative) {
    attr.id = cudaLaunchAttributeCooperative;
    attr.val.cooperative = 1;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = c->stream;
  cfg.attrs = &attr;
  cfg.numAttrs = mode == VgxLaunch::plain ? 0 : 1;
  vgx_count_launch(c);
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, std::forward<A>(args)...);
  if (e != cudaSuccess) {
    cudaGetLastError();
    c->set_error(std::string("kernel launch: ") + cudaGetErrorString(e));
    return VGX_ERR_CUDA;
  }
  return VGX_OK;
}

// ------------------------------------------------------------------ host-device copies
// The one place that calls the runtime's copies, memsets and stream synchronises.  A transfer states its element
// count once and takes the element type from its pointers (two sides of different types are written in uint8_t
// bytes at the call site).  It runs on the context's stream unless one is passed, and a failure sets the message
// as VGX_CUDA sets it and returns VGX_ERR_CUDA.  Copies are asynchronous; vgx_read is a download that ends in a
// synchronise, the idiom of a count read back from the device.
static inline int vgx_cuda_status(vgx_ctx* c, cudaError_t e, const char* call) {
  if (e == cudaSuccess) return VGX_OK;
  c->set_error(std::string(call) + ": " + cudaGetErrorString(e));
  return VGX_ERR_CUDA;
}
template <class T>
int vgx_upload(vgx_ctx* c, T* d, const T* h, size_t n) {
  return vgx_cuda_status(c, cudaMemcpyAsync(d, h, sizeof(T) * n, cudaMemcpyHostToDevice, c->stream),
                         "cudaMemcpyAsync host to device");
}
template <class T>
int vgx_download(vgx_ctx* c, T* h, const T* d, size_t n, cudaStream_t st) {
  return vgx_cuda_status(c, cudaMemcpyAsync(h, d, sizeof(T) * n, cudaMemcpyDeviceToHost, st),
                         "cudaMemcpyAsync device to host");
}
template <class T>
int vgx_download(vgx_ctx* c, T* h, const T* d, size_t n) { return vgx_download(c, h, d, n, c->stream); }
// device to device, or pinned to pinned
template <class T>
int vgx_copy(vgx_ctx* c, T* dst, const T* src, size_t n) {
  return vgx_cuda_status(c, cudaMemcpyAsync(dst, src, sizeof(T) * n, cudaMemcpyDefault, c->stream), "cudaMemcpyAsync");
}
// every byte of the n elements at d set to `byte`
template <class T>
int vgx_fill(vgx_ctx* c, T* d, size_t n, int byte = 0) {
  return vgx_cuda_status(c, cudaMemsetAsync(d, byte, sizeof(T) * n, c->stream), "cudaMemsetAsync");
}
static inline int vgx_sync(vgx_ctx* c, cudaStream_t st) {
  return vgx_cuda_status(c, cudaStreamSynchronize(st), "cudaStreamSynchronize");
}
static inline int vgx_sync(vgx_ctx* c) { return vgx_sync(c, c->stream); }
template <class T>
int vgx_read(vgx_ctx* c, T* h, const T* d, size_t n = 1) {
  VGX_TRY(vgx_download(c, h, d, n));
  return vgx_sync(c);
}
// unchecked synchronise for the void teardown paths: it leaves the context's message alone
static inline void vgx_drain(vgx_ctx* c) { cudaStreamSynchronize(c->stream); }

template <class T>
int VgxBuffer<T>::grow_keep(vgx_ctx* c, size_t need, size_t used, const char* what) {
  if (need <= bytes_) return VGX_OK;
  VgxBuffer q(kind_);
  VGX_TRY(q.alloc(c, need + need / 4, what));
  if (used) {   // bytes
    VGX_TRY(vgx_copy(c, reinterpret_cast<uint8_t*>(q.p_), reinterpret_cast<const uint8_t*>(p_), used));
    VGX_TRY(vgx_sync(c));
  }
  *this = std::move(q);
  return VGX_OK;
}

// ------------------------------------------------------------------ passes shared by the translation units
int vgx_submap_build_grid(vgx_ctx* ctx, VgxSubmap* s);
// a new, empty submap (replaces submap_id) with room for cap blocks; with_view: registration view storage
int vgx_submap_alloc(vgx_ctx* ctx, uint32_t submap_id, float voxel_size, int vps, int cap, bool with_view,
                     VgxSubmap** out);
// the rest of an upload once s->n_blocks block indices and bricks are in place on the device: block
// hash, registration view, the upload rules (a bad block list drops the submap: VGX_ERR_INVALID) and
// the dense grid.  Synchronises.
int vgx_submap_upload_finish(vgx_ctx* ctx, VgxSubmap* s);
// gives the submap its colour channel if it has none: cap_blocks x vps^3 words, zero (voxblox Color())
int vgx_submap_ensure_colour(vgx_ctx* ctx, VgxSubmap* s);
// frees submap_id if it exists and keeps the error message of the failure that leads to the drop
void vgx_submap_drop(vgx_ctx* ctx, uint32_t submap_id);
// moves the submap from_id to id (whose previous content is freed); from_id no longer exists.  Synchronises.
int vgx_submap_move(vgx_ctx* ctx, uint32_t from_id, uint32_t id);
// an id for a scratch submap: the first unused one counting down from 2^32 - 2 (2^32 - 1 is a valid cblox id)
uint32_t vgx_scratch_id(vgx_ctx* ctx);
// registration view (octets) of the layer `which` (VGX_LAYER_TSDF: d_dw into d_view, VGX_LAYER_ESDF: d_esdf into
// d_view_esdf)
int vgx_submap_build_view(vgx_ctx* ctx, VgxSubmap* s, int which);
// clears the block hash and re-inserts the first s->n_blocks blocks (after a capacity overflow
// left keys without a brick behind)
int vgx_submap_rebuild_hash(vgx_ctx* ctx, VgxSubmap* s);
// hand-written exclusive scan (extract.cu): out[0..n], out[n] = total; d_tmp: vgx_scan_tmp_count(n) words
int vgx_exclusive_scan_u32(vgx_ctx* c, const unsigned* d_in, unsigned* d_out, size_t n, unsigned* d_tmp);
size_t vgx_scan_tmp_count(size_t n);
// TSDF integration over points that are already in device memory (tsdf.cu): the core behind
// vgx_tsdf_integrate, vgx_tsdf_integrate_device and vgx_tsdf_integrate_cloud.
//   check:    the argument rules the three share (null pose, unknown / finished submap, mode) -> the submap
//             and the configuration with defaults filled in.
//   resident: integrates the n point slots d_pts (a slot with a non-finite coordinate is skipped and not
//             counted) with ray colours d_ray_rgba (r, g, b, a bytes per slot, or NULL), ends in the one
//             synchronising copy that brings the statistics back.  The caller lays out, in d_scratch,
//             d_stats (VGX_TSDF_STAT_WORDS words, cleared on the stream before anything it enqueues itself) and
//             d_sets (vgx_tsdf_set_words words); word VGX_TSDF_STAT_CALLER of d_stats is the caller's own counter
//             and comes back through *n_points.  Carves d_work and d_work2.
#define VGX_TSDF_STAT_WORDS 32
#define VGX_TSDF_STAT_CALLER 4
static inline size_t vgx_tsdf_set_words(const vgx_tsdf_config& cfg) { return cfg.mode == 1 ? (size_t)2 << 20 : 0; }
int vgx_tsdf_check(vgx_ctx* c, uint32_t id, const float T_G_C[7], const vgx_tsdf_config* cfg, VgxSubmap** out,
                   vgx_tsdf_config* resolved);
int vgx_tsdf_integrate_resident(vgx_ctx* c, VgxSubmap* s, const float T_G_C[7], const vgx_tsdf_config& cfg, int n,
                                const float* d_pts, const uint32_t* d_ray_rgba, unsigned long long* d_stats,
                                unsigned long long* d_sets, vgx_tsdf_stats* stats, int* n_points);
// WeightedSampler::getRandomItem x count on the sampler's own generator (host)
void vgx_points_draw(VgxPoints& p, int count, int32_t* idx);
void vgx_graph_free(vgx_ctx* ctx);
void vgx_graph_invalidate_registration(vgx_ctx* ctx);
// releases the separated mesh buffer (mesh.cu)
void vgx_mesh_free(vgx_ctx* ctx);

// NCCL (dlopen'ed, nccl_dyn.cpp)
int vgx_nccl_allreduce_sum_f64(vgx_ctx* ctx, double* d_buf, size_t count);

// NVLink peer exchange (p2p.cu): PUSH all-gather + local reduce with TAGGED WORDS (the low-latency
// protocol of NCCL's LL transport, restated for doubles).
// Every rank owns a CUDA-IPC exported region [page 256 B | slot[parity 2][source rank 8][cap x 16 B]].
// An element travels as one 16-byte store {value.lo32, tag, value.hi32, tag}, tag = the evaluation's
// epoch (never 0; the region starts zeroed).  An evaluation (epoch e, parity e & 1): the assembly kernel
// stores every element of the rank's partial straight into slot[parity][rank] of EVERY rank's region
// while it is produced (posted NVLink writes) - no fence, no ticket, no flag.  The receiver spins on
// each element of its n local slots until both tags read e, and adds the n values in rank order (no
// load ever crosses NVLink; bit-identical on all ranks).  8-byte halves of a store are each atomic,
// which is all the tag check relies on.
struct VgxP2PPush {
  double* dst[8];   // where this rank's partial goes: one destination per rank (n == 1: local buffer)
  int n;
  unsigned tag;     // != 0: the destinations are tagged 16-byte slots; 0: plain doubles
};
struct VgxP2PGather {
  const void* slot[8];           // this epoch's local slots, one per source rank (16 bytes per element)
  int* timeout_flag;
  long long timeout_cycles;
  unsigned tag;
  int nranks;
};
int vgx_p2p_begin(vgx_ctx* ctx, size_t count, VgxP2PPush* push, VgxP2PGather* gat);
int vgx_p2p_gather(vgx_ctx* ctx, const VgxP2PGather& gat, double* d_out, size_t count,
                   const unsigned char* d_block_mask, int N);  // separate-launch variant
void vgx_p2p_free(vgx_ctx* ctx);
int vgx_p2p_check(vgx_ctx* ctx);   // VGX_ERR_NCCL if a gather timed out (the flag is cleared)
#ifdef __CUDACC__
__device__ __forceinline__ void vgx_push_store(const VgxP2PPush& P, int k, size_t idx, double v) {
  if (P.tag == 0) { P.dst[k][idx] = v; return; }
  const unsigned long long b = (unsigned long long)__double_as_longlong(v);
  asm volatile("st.volatile.global.v4.u32 [%0], {%1, %2, %3, %2};"
               ::"l"(reinterpret_cast<uint4*>(P.dst[k]) + idx), "r"((unsigned)b), "r"(P.tag), "r"((unsigned)(b >> 32))
               : "memory");
}
// element idx of source rank r: spins until both tags match; false on timeout
__device__ __forceinline__ bool vgx_ll_load(const VgxP2PGather& G, int r, size_t idx, long long t0, double& v) {
  const uint4* p = reinterpret_cast<const uint4*>(G.slot[r]) + idx;
  for (;;) {
    unsigned x, y, z, w;
    asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(x), "=r"(y), "=r"(z), "=r"(w) : "l"(p) : "memory");
    if (y == G.tag && w == G.tag) {
      v = __longlong_as_double((long long)(((unsigned long long)z << 32) | x));
      return true;
    }
    if (clock64() - t0 > G.timeout_cycles) return false;
  }
}
// out[i] = sum over the CONTRIBUTING ranks of element i, in rank order; NaN-poisoned when a rank never
// delivered.  block_mask[ob] (bit r: rank r has items for output block ob; identical on all ranks,
// the constraint -> rank partition is global knowledge) tells which slots hold this epoch's value: a
// rank does not push blocks it has nothing for.  Packed layout: [4 header | 4 N gradient | 16 N
// diagonal | 16 E off-diagonal]; the header comes from every rank.  All the loads of an element are
// issued before the first tag is checked.
__device__ __forceinline__ void vgx_ll_gather(const VgxP2PGather& G, double* __restrict__ out, size_t count,
                                              size_t first, size_t stride,
                                              const unsigned char* __restrict__ block_mask, int N) {
  const long long t0 = clock64();
  const unsigned all = (1u << G.nranks) - 1u;
  for (size_t i = first; i < count; i += stride) {
    unsigned m = all;
    if (block_mask && i >= 4) {
      const size_t j = i - 4;
      m = j < 4 * (size_t)N ? block_mask[j >> 2] : block_mask[(j - 4 * (size_t)N) >> 4];
    }
    unsigned x[8], y[8], z[8], w[8];
#pragma unroll
    for (int r = 0; r < 8; ++r)
      if (r < G.nranks && ((m >> r) & 1u)) {
        const uint4* p = reinterpret_cast<const uint4*>(G.slot[r]) + i;
        asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];"
                     : "=r"(x[r]), "=r"(y[r]), "=r"(z[r]), "=r"(w[r]) : "l"(p) : "memory");
      }
    double s = 0.0;
    bool ok = true;
#pragma unroll
    for (int r = 0; r < 8; ++r)
      if (r < G.nranks && ((m >> r) & 1u)) {
        double v = 0.0;
        if (y[r] == G.tag && w[r] == G.tag) v = __longlong_as_double((long long)(((unsigned long long)z[r] << 32) | x[r]));
        else if (ok && !vgx_ll_load(G, r, i, t0, v)) { ok = false; *G.timeout_flag = 1; }
        s += v;
      }
    out[i] = ok ? s : __longlong_as_double(0x7ff8000000000000ll);   // the LM sees an invalid step
  }
}
#endif
