// Registration-point extraction from resident bricks (SURVEY §8 rows a9 / f1):
//   VoxgraphSubmap::findRelevantVoxelIndices  voxgraph/src/frontend/submap_collection/voxgraph_submap.cpp:144-201
//   VoxgraphSubmap::findIsosurfaceVertices    voxgraph_submap.cpp:203-243
//   VoxgraphSubmap::getSubmapFrameSurfaceObb  voxgraph_submap.cpp:280-324
// so that a submap integrated on the GPU becomes a registration constraint's reference without its
// voxels ever leaving the device (finishSubmap, voxgraph_submap.cpp:84-107).
//
// findIsosurfaceVertices = voxblox MeshIntegrator::generateMesh + MeshLayer::getConnectedMesh +
// Interpolator::getVoxel.  Only the mesh VERTICES are used by voxgraph, and the set of vertices of
// a marching-cubes mesh is table independent: one vertex per cube edge whose end points differ in
// sign, for every cube whose 8 corners have weight > min_weight.  The connected mesh keeps the
// first vertex of each round(vertex / (0.5 voxel)) bucket; "first" is fixed canonically (blocks in
// allocation order, voxels in linear order, cube edges 0..11 - the reference walks a hash map).
// Data-parallel form: count -> scan -> emit candidates in canonical order -> bucket table with
// atomicMin(candidate index) -> the winners are interpolated -> scan -> compact.
// Compiled with -fmad=false (float expressions restated operation by operation, see oracle).
#include <math.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "layer_access.cuh"

// ------------------------------------------------------------------ exclusive scan (hand-written)
// out[i] = sum_{j<i} in[j] for i in [0, n]; out has n + 1 entries (out[n] = total).
#define SCAN_THREADS 256
#define SCAN_ITEMS 8
#define SCAN_TILE (SCAN_THREADS * SCAN_ITEMS)

__global__ void __launch_bounds__(SCAN_THREADS)
scan_tile_kernel(const unsigned* __restrict__ in, unsigned* __restrict__ out, unsigned* __restrict__ tile_sums,
                 size_t n) {
  __shared__ unsigned s_warp[SCAN_THREADS / 32];
  const size_t base = (size_t)blockIdx.x * SCAN_TILE + (size_t)threadIdx.x * SCAN_ITEMS;
  unsigned v[SCAN_ITEMS], sum = 0;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; ++k) {
    v[k] = (base + k < n) ? in[base + k] : 0u;
    sum += v[k];
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned incl = sum;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const unsigned t = __shfl_up_sync(0xffffffffu, incl, off);
    if (lane >= off) incl += t;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    unsigned w = lane < SCAN_THREADS / 32 ? s_warp[lane] : 0u;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const unsigned t = __shfl_up_sync(0xffffffffu, w, off);
      if (lane >= off) w += t;
    }
    if (lane < SCAN_THREADS / 32) s_warp[lane] = w;  // inclusive over warps
  }
  __syncthreads();
  unsigned run = incl - sum + (warp > 0 ? s_warp[warp - 1] : 0u);
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; ++k) {
    if (base + k < n) out[base + k] = run;
    run += v[k];
  }
  if (threadIdx.x == SCAN_THREADS - 1) tile_sums[blockIdx.x] = run;
}

// single CTA: exclusive scan of the tile sums in place, chunk by chunk with a running carry
__global__ void __launch_bounds__(1024) scan_sums_kernel(unsigned* __restrict__ sums, size_t m,
                                                          unsigned* __restrict__ total) {
  __shared__ unsigned s_warp[32];
  __shared__ unsigned s_carry;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (size_t c0 = 0; c0 < m; c0 += 1024) {
    const size_t i = c0 + threadIdx.x;
    const unsigned v = i < m ? sums[i] : 0u;
    unsigned incl = v;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const unsigned t = __shfl_up_sync(0xffffffffu, incl, off);
      if (lane >= off) incl += t;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      unsigned w = s_warp[lane];
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const unsigned t = __shfl_up_sync(0xffffffffu, w, off);
        if (lane >= off) w += t;
      }
      s_warp[lane] = w;
    }
    __syncthreads();
    const unsigned carry = s_carry;
    const unsigned excl = carry + incl - v + (warp > 0 ? s_warp[warp - 1] : 0u);
    if (i < m) sums[i] = excl;
    __syncthreads();
    if (threadIdx.x == 1023) s_carry = carry + s_warp[31];
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = s_carry;
}

__global__ void __launch_bounds__(SCAN_THREADS)
scan_add_kernel(unsigned* __restrict__ out, const unsigned* __restrict__ tile_sums, size_t n,
                const unsigned* __restrict__ total) {
  const size_t base = (size_t)blockIdx.x * SCAN_TILE + (size_t)threadIdx.x * SCAN_ITEMS;
  const unsigned add = tile_sums[blockIdx.x];
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; ++k)
    if (base + k < n) out[base + k] += add;
  if (blockIdx.x == 0 && threadIdx.x == 0) out[n] = *total;
}

// d_tmp: (tiles + 1) unsigned of scratch.  3 launches.
int vgx_exclusive_scan_u32(vgx_ctx* c, const unsigned* d_in, unsigned* d_out, size_t n, unsigned* d_tmp) {
  if (n == 0) return vgx_fill(c, d_out, 1);
  const size_t tiles = (n + SCAN_TILE - 1) / SCAN_TILE;
  VGX_TRY(vgx_launch(c, scan_tile_kernel, (unsigned)tiles, SCAN_THREADS, 0, VgxLaunch::plain, d_in, d_out, d_tmp, n));
  VGX_TRY(vgx_launch(c, scan_sums_kernel, 1, 1024, 0, VgxLaunch::plain, d_tmp, tiles, d_tmp + tiles));
  return vgx_launch(c, scan_add_kernel, (unsigned)tiles, SCAN_THREADS, 0, VgxLaunch::plain, d_out, d_tmp, n,
                    d_tmp + tiles);
}
size_t vgx_scan_tmp_count(size_t n) { return (n + SCAN_TILE - 1) / SCAN_TILE + 2; }

// ------------------------------------------------------------------ layer access on the device
// (LayerDev, the cube gather ex_cube, the interpolator ex_interp_voxel and the cube tables live in
// layer_access.cuh)

// ------------------------------------------------------------------ relevant voxels (cpp:144-201)
__global__ void __launch_bounds__(256)
relevant_count_kernel(LayerDev L, double min_w, double max_d, unsigned* __restrict__ counts) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= vgx_voxel_count(L.n_blocks, L.sh)) return;
  const float2 x = L.dw[i];
  counts[i] = ((double)x.y > min_w && fabs((double)x.x) < max_d) ? 1u : 0u;  // cpp:177-178
}

__device__ __forceinline__ float atomicMinFloat(float* addr, float v) {
  return (v >= 0) ? __int_as_float(atomicMin((int*)addr, __float_as_int(v)))
                  : __uint_as_float(atomicMax((unsigned*)addr, __float_as_uint(v)));
}
__device__ __forceinline__ float atomicMaxFloat(float* addr, float v) {
  return (v >= 0) ? __int_as_float(atomicMax((int*)addr, __float_as_int(v)))
                  : __uint_as_float(atomicMin((unsigned*)addr, __float_as_uint(v)));
}

// scatter into the unit-major point layout + surface OBB (cpp:280-324: centre -+ half voxel)
__global__ void __launch_bounds__(256)
relevant_emit_kernel(LayerDev L, const unsigned* __restrict__ counts, const unsigned* __restrict__ offsets,
                     const float2* __restrict__ esdf /* null: TSDF distance */, float* __restrict__ pts,
                     float* __restrict__ obb /* min[3], max[3] */) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= vgx_voxel_count(L.n_blocks, L.sh) || counts[i] == 0) return;
  int v[3];
  const int slot = vgx_voxel_of(i, L.sh, v);
  const float2 x = L.dw[i];
  float cpos[3];
  const float half = 0.5f * L.voxel_size;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    cpos[a] = vgx_voxel_centre(L.block_idx[3 * slot + a], v[a], L.block_size, L.voxel_size);
    atomicMinFloat(obb + a, cpos[a] - half);
    atomicMaxFloat(obb + 3 + a, cpos[a] + half);
  }
  float* u = pts + vgx_pt_index((size_t)offsets[i], 0);
  // cpp:183-191: the ESDF distance when use_esdf_distance, the weight is always the TSDF weight
  u[0] = cpos[0]; u[32] = cpos[1]; u[64] = cpos[2]; u[96] = esdf ? esdf[i].x : x.x; u[128] = x.y;
}

// ------------------------------------------------------------------ isosurface vertices (cpp:203-243)
__global__ void __launch_bounds__(128)
iso_count_kernel(LayerDev L, float min_weight, unsigned* __restrict__ counts) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= vgx_voxel_count(L.n_blocks, L.sh)) return;
  float sdf[8], coords[3];
  unsigned n = 0;
  if (ex_cube(L, i, min_weight, sdf, coords)) {
#pragma unroll
    for (int e = 0; e < 12; ++e) n += ex_edge_crosses(sdf[c_edge[e][0]], sdf[c_edge[e][1]]) ? 1u : 0u;
  }
  counts[i] = n;
}

struct __align__(16) IsoBucket {
  unsigned long long key;   // packed bucket coordinates, VGX_EMPTY_KEY when free
  unsigned first;           // smallest candidate index seen
  unsigned pad;
};

__global__ void iso_table_clear_kernel(IsoBucket* t, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { t[i].key = VGX_EMPTY_KEY; t[i].first = 0xFFFFFFFFu; t[i].pad = 0; }
}

__device__ __forceinline__ unsigned long long iso_bucket_key(const float p[3], double threshold_inv) {
  // createConnectedMesh: round(double(vertex) * threshold_inv) per axis, 21 bits each (biased)
  unsigned long long k = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const long long r = llround((double)p[a] * threshold_inv);
    k |= ((unsigned long long)((r + (1ll << 20)) & 0x1FFFFF)) << (21 * a);
  }
  return k;
}

__device__ __forceinline__ size_t iso_slot_of(unsigned long long key, size_t mask) {
  unsigned long long h = key * 0x9E3779B97F4A7C15ull;
  h ^= h >> 29;
  return (size_t)h & mask;
}

// candidates in canonical order; each registers itself in its bucket (atomicMin of its index)
__global__ void __launch_bounds__(128)
iso_emit_kernel(LayerDev L, float min_weight, double threshold_inv, const unsigned* __restrict__ counts,
                const unsigned* __restrict__ offsets, float* __restrict__ cand /* M x 3 */,
                unsigned long long* __restrict__ cand_key, IsoBucket* __restrict__ table, size_t mask) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= vgx_voxel_count(L.n_blocks, L.sh) || counts[i] == 0) return;
  float sdf[8], coords[3];
  if (!ex_cube(L, i, min_weight, sdf, coords)) return;
  unsigned o = offsets[i];
#pragma unroll
  for (int e = 0; e < 12; ++e) {
    const int e0 = c_edge[e][0], e1 = c_edge[e][1];
    const float s1 = sdf[e0], s2 = sdf[e1];
    if (!ex_edge_crosses(s1, s2)) continue;
    float p[3];
    const float diff = s1 - s2;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      // corner_coords = coords + cube_coord_offsets (index offset * voxel_size)
      const float c0 = coords[a] + (float)c_cube_off[e0][a] * L.voxel_size;
      const float c1 = coords[a] + (float)c_cube_off[e1][a] * L.voxel_size;
      if (fabsf(diff) >= 1e-6f) {
        const float t = s1 / diff;
        p[a] = c0 + t * (c1 - c0);
      } else {
        p[a] = 0.5f * (c0 + c1);
      }
    }
    cand[3 * (size_t)o] = p[0]; cand[3 * (size_t)o + 1] = p[1]; cand[3 * (size_t)o + 2] = p[2];
    const unsigned long long key = iso_bucket_key(p, threshold_inv);
    cand_key[o] = key;
    size_t h = iso_slot_of(key, mask);
    for (;;) {
      const unsigned long long prev = atomicCAS(&table[h].key, (unsigned long long)VGX_EMPTY_KEY, key);
      if (prev == VGX_EMPTY_KEY || prev == key) { atomicMin(&table[h].first, o); break; }
      h = (h + 1) & mask;
    }
    ++o;
  }
}

// the first candidate of every bucket is a connected-mesh vertex; interpolate (distance, weight)
__global__ void __launch_bounds__(128)
iso_select_kernel(LayerDev L, const float* __restrict__ cand, const unsigned long long* __restrict__ cand_key,
                  const IsoBucket* __restrict__ table, size_t mask, unsigned M, unsigned* __restrict__ keep,
                  float2* __restrict__ cand_dw) {
  const unsigned c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= M) return;
  const unsigned long long key = cand_key[c];
  size_t h = iso_slot_of(key, mask);
  while (table[h].key != key) h = (h + 1) & mask;
  unsigned k = 0;
  if (table[h].first == c) {
    float d, w;
    if (ex_interp_voxel(L, cand[3 * (size_t)c], cand[3 * (size_t)c + 1], cand[3 * (size_t)c + 2], d, w)) {
      k = 1;
      cand_dw[c] = make_float2(d, w);
    }
  }
  keep[c] = k;
}

__global__ void __launch_bounds__(128)
iso_compact_kernel(LayerDev L, const float* __restrict__ cand, const float2* __restrict__ cand_dw,
                   const unsigned* __restrict__ keep, const unsigned* __restrict__ offsets, unsigned M,
                   float* __restrict__ pts, unsigned* __restrict__ iso_block_flags) {
  const unsigned c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= M || keep[c] == 0) return;
  const float p[3] = {cand[3 * (size_t)c], cand[3 * (size_t)c + 1], cand[3 * (size_t)c + 2]};
  float* u = pts + vgx_pt_index((size_t)offsets[c], 0);
  const float2 dw = cand_dw[c];
  u[0] = p[0]; u[32] = p[1]; u[64] = p[2]; u[96] = dw.x; u[128] = dw.y;
  // isosurface_blocks_ (cpp:237-240): computeBlockIndexFromCoordinates(vertex)
  const int b0 = ex_floor(p[0] * L.block_size_inv + 1e-6f), b1 = ex_floor(p[1] * L.block_size_inv + 1e-6f),
            b2 = ex_floor(p[2] * L.block_size_inv + 1e-6f);
  const int slot = vgx_hash_find(L.hash, b0, b1, b2);
  if (slot >= 0) iso_block_flags[slot] = 1u;
}

__global__ void gather_weights_kernel(const float* __restrict__ pts, int n, float* __restrict__ w) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) w[i] = pts[vgx_pt_index((size_t)i, 4)];
}

__global__ void unpack_points_kernel(const float* __restrict__ pts, int n, float* __restrict__ xyz,
                                     float* __restrict__ d, float* __restrict__ w) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* u = pts + vgx_pt_index((size_t)i, 0);
  if (xyz) { xyz[3 * (size_t)i] = u[0]; xyz[3 * (size_t)i + 1] = u[32]; xyz[3 * (size_t)i + 2] = u[64]; }
  if (d) d[i] = u[96];
  if (w) w[i] = u[128];
}

// ------------------------------------------------------------------ host orchestration
// takes d_pts (n points, unit-major, zero padded) over; weights come back to the host once for the
// sampler's cumulative sums and summed_reference_weight (cpp:124), in point order
static int install_points(vgx_ctx* c, VgxSubmap* s, int type, VgxBuffer<float>&& d_pts, int n) {
  VgxPoints& p = s->points[type];
  p = VgxPoints();
  if (n == 0) {
    d_pts.reset();
    return VGX_OK;
  }
  std::vector<float> w((size_t)n);
  float* d_w;
  VGX_TRY(vgx_carve(c, c->d_scratch, vgx_part(d_w, (size_t)n)));
  VGX_TRY(vgx_launch(c, gather_weights_kernel, (n + 255) / 256, 256, 0, VgxLaunch::plain, d_pts.get(), n, d_w));
  VGX_TRY(vgx_read(c, w.data(), d_w, (size_t)n));
  p.cumulative_w.resize((size_t)n);
  double sum = 0;
  for (int i = 0; i < n; ++i) { sum += (double)w[i]; p.cumulative_w[i] = sum; }
  p.n = n;
  p.data = std::move(d_pts);
  p.sum_w = sum;
  return VGX_OK;
}

static int alloc_points(vgx_ctx* c, int n, VgxBuffer<float>& out) {
  const size_t units = ((size_t)std::max(n, 1) + VGX_PT_UNIT - 1) / VGX_PT_UNIT;
  VGX_TRY(out.alloc(c, units * VGX_PT_UNIT_FLOATS * sizeof(float), "registration points"));
  return vgx_fill(c, out.get(), units * VGX_PT_UNIT_FLOATS);
}

extern "C" void vgx_registration_filter_default(vgx_registration_filter* f) {
  if (!f) return;
  f->min_voxel_weight = 1.0;     // voxgraph_submap.h:27
  f->max_voxel_distance = 0.3;   // voxgraph_submap.h:28
  f->use_esdf_distance = 0;      // reference default true; the ESDF branch needs an ESDF layer
}

extern "C" int vgx_submap_extract_points(vgx_ctx* c, uint32_t id, const vgx_registration_filter* filter) {
  return vgx_entry(c, __func__, [&] {
    VgxSubmap* s;
    VGX_TRY(vgx_submap_get(c, id, &s, VgxNeed::finished));
    vgx_registration_filter f;
    vgx_registration_filter_default(&f);
    if (filter) f = *filter;
    if (f.use_esdf_distance && !s->d_esdf.get() && s->n_blocks > 0)
      VGX_FAIL(c, VGX_ERR_INVALID, "use_esdf_distance needs the submap's ESDF "
                                   "(vgx_submap_generate_esdf first, as finishSubmap does)");
    vgx_graph_invalidate_registration(c);
    const LayerDev L = layer_of(s);
    const size_t nvox = (size_t)s->n_blocks * s->vox_per_block;
    s->surface_obb_valid = false;
    s->iso_blocks.clear();
    s->d_iso_idx.reset();
    s->n_iso = 0;
    s->points_extracted = true;
    if (nvox == 0) {
      VGX_TRY(install_points(c, s, VGX_POINTS_VOXELS, VgxBuffer<float>(), 0));
      return install_points(c, s, VGX_POINTS_ISOSURFACE, VgxBuffer<float>(), 0);
    }
    if (nvox >= 0xFFFFFFFFull / 12) VGX_FAIL(c, VGX_ERR_CAPACITY, "submap too large for 32-bit candidate indices");
    unsigned *d_counts, *d_offsets, *d_tmp, *d_flags;
    float* d_obb;
    VGX_TRY(vgx_carve(c, c->d_work, vgx_part(d_counts, nvox + 1), vgx_part(d_offsets, nvox + 1),
                      vgx_part(d_tmp, vgx_scan_tmp_count(nvox * 12)), vgx_part(d_obb, 6),
                      vgx_part(d_flags, (size_t)s->n_blocks)));
    const unsigned grid256 = (unsigned)((nvox + 255) / 256), grid128 = (unsigned)((nvox + 127) / 128);

    // ---- relevant voxels + surface OBB
    {
      const float inf = INFINITY;
      const float init[6] = {inf, inf, inf, -inf, -inf, -inf};
      VGX_TRY(vgx_upload(c, d_obb, init, std::size(init)));
      VGX_TRY(vgx_launch(c, relevant_count_kernel, grid256, 256, 0, VgxLaunch::plain, L, f.min_voxel_weight,
                         f.max_voxel_distance, d_counts));
      VGX_TRY(vgx_exclusive_scan_u32(c, d_counts, d_offsets, nvox, d_tmp));
      unsigned total = 0;
      VGX_TRY(vgx_read(c, &total, d_offsets + nvox));
      VgxBuffer<float> d_pts;
      VGX_TRY(alloc_points(c, (int)total, d_pts));
      VGX_TRY(vgx_launch(c, relevant_emit_kernel, grid256, 256, 0, VgxLaunch::plain, L, d_counts, d_offsets,
                         f.use_esdf_distance ? s->d_esdf.get() : nullptr, d_pts.get(), d_obb));
      float obb[6];
      VGX_TRY(vgx_read(c, obb, d_obb, std::size(obb)));
      for (int a = 0; a < 3; ++a) { s->surface_obb_min[a] = obb[a]; s->surface_obb_max[a] = obb[3 + a]; }
      s->surface_obb_valid = total > 0;
      VGX_TRY(install_points(c, s, VGX_POINTS_VOXELS, std::move(d_pts), (int)total));
    }
    // ---- isosurface vertices
    {
      const float min_weight = (float)f.min_voxel_weight;                 // cpp:211-212
      const float threshold = (float)(0.5 * (double)s->voxel_size);       // cpp:220
      const double threshold_inv = 1.0 / (double)threshold;               // createConnectedMesh
      VGX_TRY(vgx_launch(c, iso_count_kernel, grid128, 128, 0, VgxLaunch::plain, L, min_weight, d_counts));
      VGX_TRY(vgx_exclusive_scan_u32(c, d_counts, d_offsets, nvox, d_tmp));
      unsigned M = 0;
      VGX_TRY(vgx_read(c, &M, d_offsets + nvox));
      unsigned kept = 0;
      VgxBuffer<float> d_pts;
      if (M > 0) {
        size_t tsize = 1024;
        while (tsize < 2 * (size_t)M) tsize <<= 1;
        IsoBucket* d_table;
        float* d_cand;
        unsigned long long* d_key;
        unsigned *d_keep, *d_koff, *d_tmp2;
        float2* d_cdw;
        VGX_TRY(vgx_carve(c, c->d_work2, vgx_part(d_table, tsize), vgx_part(d_cand, (size_t)M * 3), vgx_part(d_key, M),
                          vgx_part(d_keep, (size_t)M + 1), vgx_part(d_koff, (size_t)M + 1), vgx_part(d_cdw, M),
                          vgx_part(d_tmp2, vgx_scan_tmp_count(M))));
        VGX_TRY(vgx_launch(c, iso_table_clear_kernel, (unsigned)((tsize + 255) / 256), 256, 0, VgxLaunch::plain, d_table,
                           tsize));
        VGX_TRY(vgx_launch(c, iso_emit_kernel, grid128, 128, 0, VgxLaunch::plain, L, min_weight, threshold_inv, d_counts,
                           d_offsets, d_cand, d_key, d_table, tsize - 1));
        VGX_TRY(vgx_launch(c, iso_select_kernel, (M + 127) / 128, 128, 0, VgxLaunch::plain, L, d_cand, d_key, d_table,
                           tsize - 1, M, d_keep, d_cdw));
        VGX_TRY(vgx_exclusive_scan_u32(c, d_keep, d_koff, M, d_tmp2));
        VGX_TRY(vgx_read(c, &kept, d_koff + M));
        VGX_TRY(alloc_points(c, (int)kept, d_pts));
        VGX_TRY(vgx_fill(c, d_flags, (size_t)s->n_blocks));
        VGX_TRY(vgx_launch(c, iso_compact_kernel, (M + 127) / 128, 128, 0, VgxLaunch::plain, L, d_cand, d_cdw, d_keep,
                           d_koff, M, d_pts.get(), d_flags));
        // isosurface block list (slots, ascending) for overlapsWith
        std::vector<unsigned> flags((size_t)s->n_blocks);
        VGX_TRY(vgx_read(c, flags.data(), d_flags, flags.size()));
        for (int b = 0; b < s->n_blocks; ++b)
          if (flags[b]) s->iso_blocks.push_back(b);
        if (!s->iso_blocks.empty()) {
          std::vector<int32_t> bidx(3 * (size_t)s->n_blocks), iso(3 * s->iso_blocks.size());
          VGX_TRY(vgx_read(c, bidx.data(), s->d_block_idx.get(), bidx.size()));
          for (size_t k = 0; k < s->iso_blocks.size(); ++k)
            for (int a = 0; a < 3; ++a) iso[3 * k + a] = bidx[3 * (size_t)s->iso_blocks[k] + a];
          VGX_TRY(s->d_iso_idx.alloc(c, sizeof(int32_t) * iso.size(), "isosurface block list"));
          VGX_TRY(vgx_upload(c, s->d_iso_idx.get(), iso.data(), iso.size()));
          VGX_TRY(vgx_sync(c));
          s->n_iso = (int)s->iso_blocks.size();
        }
      } else {
        VGX_TRY(alloc_points(c, 0, d_pts));
      }
      VGX_TRY(install_points(c, s, VGX_POINTS_ISOSURFACE, std::move(d_pts), (int)kept));
    }
    return VGX_OK;
  });
}

extern "C" int vgx_submap_finish_ex(vgx_ctx* c, uint32_t id, const vgx_registration_filter* filter) {
  return vgx_entry(c, __func__, [&] {
    VGX_TRY(vgx_submap_finish(c, id));
    return vgx_submap_extract_points(c, id, filter);
  });
}

extern "C" int vgx_submap_num_points(vgx_ctx* c, uint32_t id, int type, int* n) {
  return vgx_entry(c, __func__, [&] {
    if (!n || type < 0 || type > 1) return VGX_ERR_INVALID;
    VgxSubmap* s;
    VGX_TRY(vgx_submap_get(c, id, &s));
    *n = s->points[type].n;
    return VGX_OK;
  });
}

extern "C" int vgx_submap_download_points(vgx_ctx* c, uint32_t id, int type, int max_n, float* xyz,
                                          float* distance, float* weight, int* n_out) {
  return vgx_entry(c, __func__, [&] {
    if (type < 0 || type > 1) return VGX_ERR_INVALID;
    VgxSubmap* s;
    VGX_TRY(vgx_submap_get(c, id, &s));
    const VgxPoints& p = s->points[type];
    if (n_out) *n_out = p.n;
    if (p.n > max_n) VGX_FAIL(c, VGX_ERR_CAPACITY, "max_n too small");
    if (p.n == 0) return VGX_OK;
    const size_t n = (size_t)p.n;
    float *d_xyz, *d_d, *d_w;
    VGX_TRY(vgx_carve(c, c->d_scratch, vgx_part(d_xyz, 3 * n), vgx_part(d_d, n), vgx_part(d_w, n)));
    VGX_TRY(vgx_launch(c, unpack_points_kernel, (unsigned)((n + 255) / 256), 256, 0, VgxLaunch::plain, p.data.get(), p.n,
                       d_xyz, d_d, d_w));
    if (xyz) VGX_TRY(vgx_download(c, xyz, d_xyz, 3 * n));
    if (distance) VGX_TRY(vgx_download(c, distance, d_d, n));
    if (weight) VGX_TRY(vgx_download(c, weight, d_w, n));
    return vgx_sync(c);
  });
}

extern "C" int vgx_submap_surface_obb(vgx_ctx* c, uint32_t id, float obb_min[3], float obb_max[3]) {
  return vgx_entry(c, __func__, [&] {
    if (!obb_min || !obb_max) return VGX_ERR_INVALID;
    VgxSubmap* s;
    VGX_TRY(vgx_submap_get(c, id, &s));
    if (!s->surface_obb_valid) return VGX_ZERO_WEIGHT;  // no voxel qualifies: the box stays +-inf
    for (int a = 0; a < 3; ++a) { obb_min[a] = s->surface_obb_min[a]; obb_max[a] = s->surface_obb_max[a]; }
    return VGX_OK;
  });
}
