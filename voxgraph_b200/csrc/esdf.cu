// ESDF generation for a finished submap from its resident TSDF bricks (SURVEY §8 row f2):
//   cblox::TsdfEsdfSubmap::generateEsdf, called by VoxgraphSubmap::finishSubmap
//   (voxgraph/src/frontend/submap_collection/voxgraph_submap.cpp:86) =
//   voxblox::EsdfIntegrator::updateFromTsdfLayerBatch (upstream, absent here; restated from the
//   published algorithm as its fixed point; the CPU checker restates the same definition).
// The ESDF feeds the reference's default registration branch (use_esdf_distance = true,
// registration_cost_function.h:35; cpp:133-140) and findRelevantVoxelIndices' ESDF distance.
//
// GPU form: voxblox pops a bucketed priority queue on one thread; here every observed, non-fixed
// voxel repeatedly PULLS  d <- min(d, d_neighbour + |offset| voxel_size)  over its 26 neighbours
// (max on the negative side) in place until a sweep changes nothing.  The update is monotone, so
// any interleaving reaches the same least fixed point = the exact shortest quasi-Euclidean path in
// float arithmetic; max_distance / voxel_size sweeps (10-20) over the bricks suffice.
// Compiled with -fmad=false.
#include <math.h>
#include <string.h>

#include <vector>

#include "layer_access.cuh"

struct EsdfParams {
  float max_distance, default_distance, min_distance, min_weight;
};

// (distance, observed) from the TSDF brick + "fixed" mask
__global__ void __launch_bounds__(256)
esdf_init_kernel(EsdfParams P, LayerDev L, float2* __restrict__ esdf, unsigned char* __restrict__ fixed) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= vgx_voxel_count(L.n_blocks, L.sh)) return;
  const float2 t = L.dw[i];
  float2 e = make_float2(0.f, 0.f);
  unsigned char f = 0;
  if (!(t.y < P.min_weight)) {
    e.y = 1.f;
    if (fabsf(t.x) < P.min_distance) { f = 1; e.x = t.x; }
    else e.x = (t.x > 0.f ? 1.f : -1.f) * P.default_distance;
  }
  esdf[i] = e;
  fixed[i] = f;
}

// 27 neighbour slots per block (centre included), -1 where the block does not exist
__global__ void esdf_neighbours_kernel(LayerDev L, int* __restrict__ nb) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 27 * L.n_blocks) return;
  const int b = t / 27, k = t % 27;
  nb[t] = vgx_hash_find(L.hash, L.block_idx[3 * b] + (k % 3) - 1, L.block_idx[3 * b + 1] + ((k / 3) % 3) - 1,
                        L.block_idx[3 * b + 2] + (k / 9) - 1);
}

__global__ void __launch_bounds__(256)
esdf_sweep_kernel(EsdfParams P, LayerDev L, float2* esdf, const unsigned char* __restrict__ fixed,
                  const int* __restrict__ nb, int* __restrict__ changed) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= vgx_voxel_count(L.n_blocks, L.sh)) return;
  volatile float2* ev = esdf;
  const float2 me = make_float2(ev[i].x, ev[i].y);
  if (me.y == 0.f || fixed[i]) return;
  int v[3];
  const int b = vgx_voxel_of(i, L.sh, v);
  const float s1 = 1.0f * L.voxel_size, s2 = sqrtf(2.0f) * L.voxel_size, s3 = sqrtf(3.0f) * L.voxel_size;
  float d = me.x;
#pragma unroll 1
  for (int dz = -1; dz <= 1; ++dz)
#pragma unroll 1
    for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
      for (int dx = -1; dx <= 1; ++dx) {
        if (!dx && !dy && !dz) continue;
        int q0 = v[0] + dx, q1 = v[1] + dy, q2 = v[2] + dz, bo0 = 1, bo1 = 1, bo2 = 1;
        if (q0 < 0) { q0 += L.vps; bo0 = 0; } else if (q0 >= L.vps) { q0 -= L.vps; bo0 = 2; }
        if (q1 < 0) { q1 += L.vps; bo1 = 0; } else if (q1 >= L.vps) { q1 -= L.vps; bo1 = 2; }
        if (q2 < 0) { q2 += L.vps; bo2 = 0; } else if (q2 >= L.vps) { q2 -= L.vps; bo2 = 2; }
        const int s = nb[27 * b + bo0 + 3 * bo1 + 9 * bo2];
        if (s < 0) continue;
        const size_t j = vgx_voxel_index(s, q0, q1, q2, L.sh);
        const float ny = ev[j].y;
        if (ny == 0.f) continue;
        const float dn = ev[j].x;
        const int m = (dx != 0) + (dy != 0) + (dz != 0);
        const float step = m == 1 ? s1 : (m == 2 ? s2 : s3);
        if (d > 0.f && dn > 0.f) {
          const float cand = dn + step;
          if (cand < P.max_distance && cand < d) d = cand;
        } else if (d < 0.f && dn < 0.f) {
          const float cand = dn - step;
          if (cand > -P.max_distance && cand > d) d = cand;
        }
      }
  if (d != me.x) {
    ev[i].x = d;
    *changed = 1;
  }
}

extern "C" void vgx_esdf_config_default(vgx_esdf_config* c) {
  if (!c) return;
  c->max_distance_m = 2.0f;       // voxblox::EsdfIntegrator::Config defaults
  c->default_distance_m = 2.0f;
  c->min_distance_m = 0.2f;
  c->min_weight = 1e-6f;
}

extern "C" int vgx_submap_generate_esdf(vgx_ctx* c, uint32_t id, const vgx_esdf_config* cfg, int* sweeps_out) {
  return vgx_entry(c, __func__, [&] {
    VgxSubmap* s;
    VGX_TRY(vgx_submap_get(c, id, &s, VgxNeed::finished));
    vgx_esdf_config dc;
    vgx_esdf_config_default(&dc);
    if (cfg) dc = *cfg;
    if (!(dc.max_distance_m > 0) || !(dc.min_distance_m >= 0))
      VGX_FAIL(c, VGX_ERR_INVALID, "invalid distances");
    vgx_graph_invalidate_registration(c);
    s->d_esdf.reset();
    s->d_view_esdf.reset();
    const size_t nvox = (size_t)s->n_blocks * s->vox_per_block;
    if (sweeps_out) *sweeps_out = 0;
    if (nvox == 0) return s->d_view_esdf.alloc(c, 32, "ESDF registration view");
    EsdfParams P;
    P.max_distance = dc.max_distance_m; P.default_distance = dc.default_distance_m;
    P.min_distance = dc.min_distance_m; P.min_weight = dc.min_weight;
    const LayerDev L = layer_of(s);
    VGX_TRY(s->d_esdf.alloc(c, sizeof(float2) * nvox, "ESDF bricks"));
    unsigned char* d_fixed;
    int *d_nb, *d_changed;
    VGX_TRY(vgx_carve(c, c->d_work, vgx_part(d_fixed, nvox), vgx_part(d_nb, (size_t)27 * s->n_blocks),
                      vgx_part(d_changed, 1)));
    const unsigned grid = (unsigned)((nvox + 255) / 256);
    VGX_TRY(vgx_launch(c, esdf_init_kernel, grid, 256, 0, VgxLaunch::plain, P, L, s->d_esdf.get(), d_fixed));
    VGX_TRY(vgx_launch(c, esdf_neighbours_kernel, (27 * s->n_blocks + 127) / 128, 128, 0, VgxLaunch::plain, L, d_nb));
    // relax to convergence: the flag is read back every other sweep
    int sweeps = 0;
    const int max_sweeps = 4 * (int)ceilf(dc.max_distance_m / s->voxel_size) + 16;
    for (;;) {
      VGX_TRY(vgx_fill(c, d_changed, 1));
      for (int k = 0; k < 2; ++k) {
        VGX_TRY(vgx_launch(c, esdf_sweep_kernel, grid, 256, 0, VgxLaunch::plain, P, L, s->d_esdf.get(), d_fixed, d_nb,
                           d_changed));
        ++sweeps;
      }
      int changed = 0;
      VGX_TRY(vgx_read(c, &changed, d_changed));
      if (!changed) break;
      if (sweeps > max_sweeps) VGX_FAIL(c, VGX_ERR_INVALID, "relaxation did not converge");
    }
    if (sweeps_out) *sweeps_out = sweeps;
    // registration view of the ESDF layer (observed <=> weight 1), same octet layout as the TSDF view
    VGX_TRY(s->d_view_esdf.alloc(c, sizeof(float) * 8 * nvox, "ESDF registration view"));
    VGX_TRY(vgx_submap_build_view(c, s, VGX_LAYER_ESDF));
    return vgx_sync(c);
  });
}

extern "C" int vgx_submap_download_esdf(vgx_ctx* c, uint32_t id, int max_blocks, float* distance,
                                        float* observed, int* n_out) {
  return vgx_entry(c, __func__, [&] {
    VgxSubmap* s;
    VGX_TRY(vgx_submap_get(c, id, &s));
    if (!s->d_esdf.get() && s->n_blocks > 0) VGX_FAIL(c, VGX_ERR_INVALID, "no ESDF generated");
    const int n = s->n_blocks;
    if (n_out) *n_out = n;
    if (n > max_blocks) VGX_FAIL(c, VGX_ERR_CAPACITY, "max_blocks too small");
    if (n == 0) return VGX_OK;
    const size_t nvox = (size_t)n * s->vox_per_block;
    std::vector<float2> h(nvox);
    VGX_TRY(vgx_read(c, h.data(), s->d_esdf.get(), nvox));
    for (size_t i = 0; i < nvox; ++i) {
      if (distance) distance[i] = h[i].x;
      if (observed) observed[i] = h[i].y;
    }
    return VGX_OK;
  });
}
