// Internal declarations shared by the translation units of libvoxgraph_b200.so.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <map>
#include <random>
#include <string>
#include <vector>

#include "voxgraph_b200.h"

// ------------------------------------------------------------------ error handling
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

// ------------------------------------------------------------------ block hash
// voxblox AnyIndexHash (block_hash.h): x + 17191*y + 17191^2*z, then masked into an
// open-addressing table with linear probing. Keys pack the three 21-bit biased indices.
#define VGX_EMPTY_KEY 0xFFFFFFFFFFFFFFFFull

__host__ __device__ __forceinline__ uint64_t vgx_pack_key(int bx, int by, int bz) {
  return ((uint64_t)((uint32_t)(bx + (1 << 20)) & 0x1FFFFFu)) |
         ((uint64_t)((uint32_t)(by + (1 << 20)) & 0x1FFFFFu) << 21) |
         ((uint64_t)((uint32_t)(bz + (1 << 20)) & 0x1FFFFFu) << 42);
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
// spinning.  Entries with val < 0 (unmapped / overflowed) read as "no block".
__device__ __forceinline__ int vgx_hash_find(const VgxHash& h, int bx, int by, int bz) {
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
  float* data = nullptr;        // ceil(n / 32) units
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
  int cap_blocks = 0;
  int n_blocks = 0;            // host mirror (valid after upload / integrate sync)
  bool finished = false;
  VgxHash hash{nullptr, 0};
  int32_t* d_block_idx = nullptr;  // cap x 3
  float2* d_dw = nullptr;          // cap x vps^3 (distance, weight)
  // Registration view ("octets"): for every voxel the distances of its 2x2x2 forward
  // neighbourhood (corner i: x = bit2, y = bit1, z = bit0; apron across bricks baked in),
  // NaN where the voxel is unobserved or its block missing. One 32-byte sector per point.
  float* d_view = nullptr;         // cap x vps^3 x 8
  float2* d_esdf = nullptr;        // ESDF bricks (distance, observed 1/0), n_blocks x vps^3 (vgx_submap_generate_esdf)
  float* d_view_esdf = nullptr;    // registration view of the ESDF bricks
  int* d_counters = nullptr;       // [0] = n_blocks (device), [1] = overflow flag
  // Dense block index over the AABB of the allocated blocks (finished submaps): slot or -1.
  // Small enough to be staged in shared memory by the registration kernel; the hash stays
  // the general structure (integration, view construction, sparse/huge submaps).
  int32_t* d_grid = nullptr;
  uint16_t* d_grid16 = nullptr;   // 16-bit copy (0xFFFF = no block), padded to a multiple of 16 bytes
  int grid_min[3] = {0, 0, 0};
  int grid_dim[3] = {0, 0, 0};
  VgxPoints points[2];
  // vgx_submap_extract_points: surface OBB (cpp:280-324) and isosurface block slots (cpp:237-240)
  bool surface_obb_valid = false;
  float surface_obb_min[3] = {0, 0, 0}, surface_obb_max[3] = {0, 0, 0};
  std::vector<int> iso_blocks;
  bool points_extracted = false;
  int32_t* d_iso_idx = nullptr;   // block indices of the isosurface blocks (n_iso x 3)
  int n_iso = 0;
};

// ------------------------------------------------------------------ pose graph
struct VgxRelEdge {
  int a, b;
  double t_obs[3], yaw_obs, L[16];
};

struct VgxGraph;  // defined in graph.h

struct VgxProfileSlot {
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
  VgxProfileSlot prof[10];
  int64_t launches = 0;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  // scratch
  void* d_scratch = nullptr;
  size_t scratch_bytes = 0;
  void* h_pinned = nullptr;
  size_t pinned_bytes = 0;
  void* d_sort = nullptr;    // TSDF deterministic path: counts / offsets / scan temp
  size_t sort_bytes = 0;
  void* d_sort2 = nullptr;   // ... tuple buffers + radix-sort temp
  size_t sort2_bytes = 0;
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

  void set_error(const std::string& e) { error = e; }
  VgxSubmap* find(uint32_t id) {
    auto it = submaps.find(id);
    return it == submaps.end() ? nullptr : it->second;
  }
  int ensure_scratch(size_t bytes);
  int ensure_pinned(size_t bytes);
  int ensure_sort(size_t bytes);
  int ensure_sort2(size_t bytes);
};

// RAII-less helper to bracket kernel launches for accounting.
struct VgxLaunchScope {
  vgx_ctx* c;
  int which;
  VgxLaunchScope(vgx_ctx* ctx, int w, int n_launches = 1) : c(ctx), which(w) {
    c->launches += n_launches;
    c->prof[which].launches += n_launches;
    if (c->profile) cudaEventRecord(c->ev0, c->stream);
  }
  ~VgxLaunchScope() {
    if (c->profile) {
      cudaEventRecord(c->ev1, c->stream);
      cudaEventSynchronize(c->ev1);
      float ms = 0;
      cudaEventElapsedTime(&ms, c->ev0, c->ev1);
      c->prof[which].total_ms += ms;
    }
  }
};

int vgx_submap_build_grid(vgx_ctx* ctx, VgxSubmap* s);
// registration view (octets) of `bricks` (n_blocks x vps^3 (distance, weight/observed)) into `view`
int vgx_submap_build_view(vgx_ctx* ctx, VgxSubmap* s, const float2* bricks, float* view);
// clears the block hash and re-inserts the first s->n_blocks blocks (after a capacity overflow
// left keys without a brick behind)
int vgx_submap_rebuild_hash(vgx_ctx* ctx, VgxSubmap* s);
// hand-written exclusive scan (extract.cu): out[0..n], out[n] = total; d_tmp: vgx_scan_tmp_count(n) words
int vgx_exclusive_scan_u32(vgx_ctx* c, const unsigned* d_in, unsigned* d_out, size_t n, unsigned* d_tmp);
size_t vgx_scan_tmp_count(size_t n);
// WeightedSampler::getRandomItem x count on the sampler's own generator (host)
void vgx_points_draw(VgxPoints& p, int count, int32_t* idx);
void vgx_graph_free(vgx_ctx* ctx);
void vgx_graph_invalidate_registration(vgx_ctx* ctx);

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
