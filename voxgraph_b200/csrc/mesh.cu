// Separated submap meshes on the device (SURVEY §8 visualisation rows):
//   SubmapVisuals::publishSeparatedMesh / saveSeparatedMesh  voxgraph/src/tools/visualization/submap_visuals.cpp:68-97
//   = cblox SubmapMesher::generateSeparatedMesh + voxblox::outputMeshLayerAsPly, over
//     voxblox MeshIntegrator<TsdfVoxel>::generateMesh(false, false) (a full re-mesh of every submap)
// so that a map can be looked at without its voxels leaving the GPU.
//
// The mesh (the contract the restatement in tests/mesh_exact.py follows bit for bit):
//   * a cube at voxel g has corners g + c_cube_off[k]; it is meshed when all 8 are valid (ex_cube:
//     allocated and weight > min_weight); bit k of its configuration is set iff sdf_k < 0;
//   * one vertex per lattice edge (low voxel, axis) of a meshed cube whose ends differ in sign, shared by
//     every cube that uses the edge (watertight by construction), interpolated from the low end;
//   * triangles by the face-walk rule: the crossings of a cube are joined across its faces into loops
//     (a face with 4 crossings joins the pairs that meet at the same negative corner, so neighbouring
//     cubes agree on every face), each loop is directed so that its front faces the positive side, starts
//     at its lowest edge and is fanned; the 256-row table is built once on the host from that rule;
//   * vertices in (slot, linear voxel index, axis) order, triangles in (slot, linear index, loop, fan)
//     order; submaps in the order given, vertices moved to the mission frame by T_M_S.
// This is not voxblox's classic table (not available here): the vertex set, the meshed cubes and the
// surface topology on every unambiguous face carry over, and the ambiguous faces cannot crack.
//
// Passes, each one launch over every submap of a batch (batches only split lists whose per-voxel scratch
// exceeds VGX_MESH_BATCH_VOXELS): count (triangles per cube, mark the crossing edges of meshed cubes with
// an idempotent atomicOr) -> scan -> count marked edges -> scan -> emit vertices -> emit triangles.
// Deterministic: no result depends on the order in which threads run.  Compiled with -fmad=false.
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "layer_access.cuh"

#define VGX_MESH_BATCH_VOXELS ((size_t)1 << 27)   // 16 B of scratch per voxel: 2 GiB per batch

static __constant__ uint8_t c_mesh_ntri[256];
static __constant__ uint8_t c_mesh_tri[256][15];   // up to 5 triangles of 3 cube edges
static __constant__ uint8_t c_mesh_edge[12];       // low corner | axis << 3

// ------------------------------------------------------------------ the triangle table (host)
namespace {

const int kCubeOff[8][3] = VGX_CUBE_OFF;
const int kEdge[12][2] = VGX_CUBE_EDGE;

struct MeshTable {
  uint8_t ntri[256];
  uint8_t tri[256][15];
  uint8_t edge[12];
};

int edge_axis(int e) {
  for (int a = 0; a < 3; ++a)
    if (kCubeOff[kEdge[e][0]][a] != kCubeOff[kEdge[e][1]][a]) return a;
  return -1;
}

// the face-walk rule of the file comment, for one configuration; false if the rule breaks down
bool walk(int cfg, uint8_t* ntri, uint8_t tri[15]) {
  bool neg[8], cross[12];
  for (int k = 0; k < 8; ++k) neg[k] = (cfg >> k) & 1;
  for (int e = 0; e < 12; ++e) cross[e] = neg[kEdge[e][0]] != neg[kEdge[e][1]];
  int nbr[12][2], nn[12] = {0};
  auto join = [&](int a, int b) {
    if (nn[a] >= 2 || nn[b] >= 2) return false;
    nbr[a][nn[a]++] = b;
    nbr[b][nn[b]++] = a;
    return true;
  };
  for (int a = 0; a < 3; ++a) {
    for (int side = 0; side < 2; ++side) {
      int corners[4], nc = 0, ce[4], nce = 0;
      for (int k = 0; k < 8; ++k)
        if (kCubeOff[k][a] == side) corners[nc++] = k;
      for (int e = 0; e < 12; ++e) {
        const bool on = kCubeOff[kEdge[e][0]][a] == side && kCubeOff[kEdge[e][1]][a] == side;
        if (on && cross[e]) ce[nce++] = e;
      }
      if (nce == 2) {
        if (!join(ce[0], ce[1])) return false;
      } else if (nce == 4) {   // ambiguous face: pair the crossings at each negative corner
        for (int q = 0; q < 4; ++q) {
          const int k = corners[q];
          if (!neg[k]) continue;
          int inc[2], ni = 0;
          for (int j = 0; j < 4; ++j)
            if ((kEdge[ce[j]][0] == k || kEdge[ce[j]][1] == k) && ni < 2) inc[ni++] = ce[j];
          if (ni != 2 || !join(inc[0], inc[1])) return false;
        }
      } else if (nce != 0) {
        return false;
      }
    }
  }
  bool seen[12] = {false};
  int nt = 0;
  for (int start = 0; start < 12; ++start) {
    if (!cross[start] || seen[start]) continue;
    if (nn[start] != 2) return false;
    int lp[12], m = 0, prev = -1, cur = start;
    lp[m++] = start;
    seen[start] = true;
    for (;;) {
      int nxt = (prev < 0) ? std::min(nbr[cur][0], nbr[cur][1]) : (nbr[cur][0] != prev ? nbr[cur][0] : nbr[cur][1]);
      if (nxt == start) break;
      if (seen[nxt] || nn[nxt] != 2 || m >= 12) return false;
      lp[m++] = nxt;
      seen[nxt] = true;
      prev = cur;
      cur = nxt;
    }
    if (m < 3) return false;
    // Newell normal of the doubled edge midpoints against sum(positive corner - negative corner)
    long n[3] = {0, 0, 0}, g[3] = {0, 0, 0};
    for (int i = 0; i < m; ++i) {
      const int e = lp[i], f = lp[(i + 1) % m];
      long p[3], q[3];
      for (int a = 0; a < 3; ++a) {
        p[a] = kCubeOff[kEdge[e][0]][a] + kCubeOff[kEdge[e][1]][a];
        q[a] = kCubeOff[kEdge[f][0]][a] + kCubeOff[kEdge[f][1]][a];
      }
      n[0] += p[1] * q[2] - p[2] * q[1];
      n[1] += p[2] * q[0] - p[0] * q[2];
      n[2] += p[0] * q[1] - p[1] * q[0];
      const int c0 = kEdge[e][0], c1 = kEdge[e][1];
      const int pos = neg[c0] ? c1 : c0, ng = neg[c0] ? c0 : c1;
      for (int a = 0; a < 3; ++a) g[a] += kCubeOff[pos][a] - kCubeOff[ng][a];
    }
    const long dot = n[0] * g[0] + n[1] * g[1] + n[2] * g[2];
    if (dot == 0) return false;
    if (dot < 0)
      for (int i = 1, j = m - 1; i < j; ++i, --j) std::swap(lp[i], lp[j]);
    for (int j = 1; j + 1 < m; ++j) {
      if (nt >= 5) return false;
      tri[3 * nt] = (uint8_t)lp[0];
      tri[3 * nt + 1] = (uint8_t)lp[j];
      tri[3 * nt + 2] = (uint8_t)lp[j + 1];
      ++nt;
    }
  }
  *ntri = (uint8_t)nt;
  return true;
}

bool build_table(MeshTable* t) {
  memset(t, 0, sizeof(*t));
  for (int e = 0; e < 12; ++e) {
    const int a = edge_axis(e), c0 = kEdge[e][0], c1 = kEdge[e][1];
    const int low = kCubeOff[c0][a] < kCubeOff[c1][a] ? c0 : c1;
    t->edge[e] = (uint8_t)(low | (a << 3));
  }
  for (int cfg = 0; cfg < 256; ++cfg)
    if (!walk(cfg, &t->ntri[cfg], t->tri[cfg])) return false;
  return true;
}

int ensure_table(vgx_ctx* c) {
  if (c->mesh_table_ready) return VGX_OK;
  static MeshTable table;
  static bool built = false, ok = false;
  if (!built) {
    ok = build_table(&table);
    built = true;
  }
  if (!ok) VGX_FAIL(c, VGX_ERR_INVALID, "the face-walk rule failed to build its table");
  uint8_t *ntri, (*tri)[15], *edge;
  VGX_CUDA(c, cudaGetSymbolAddress(reinterpret_cast<void**>(&ntri), c_mesh_ntri));
  VGX_CUDA(c, cudaGetSymbolAddress(reinterpret_cast<void**>(&tri), c_mesh_tri));
  VGX_CUDA(c, cudaGetSymbolAddress(reinterpret_cast<void**>(&edge), c_mesh_edge));
  VGX_TRY(vgx_upload(c, ntri, table.ntri, std::size(table.ntri)));
  VGX_TRY(vgx_upload(c, tri, table.tri, std::size(table.tri)));
  VGX_TRY(vgx_upload(c, edge, table.edge, std::size(table.edge)));
  VGX_TRY(vgx_sync(c));   // the host table outlives the copies anyway
  c->mesh_table_ready = true;
  return VGX_OK;
}

// voxblox rainbowColorMap (color.h), the default colour of a submap: h = (id mod 20) / 20
void rainbow(uint32_t id, uint8_t rgba[4]) {
  double h = (double)(id % 20u) / 20.0;
  h -= floor(h);
  h *= 6;
  const int i = (int)floor(h);
  double f = h - i;
  if (!(i & 1)) f = 1 - f;
  const double n = 1 - f;
  double r, g, b;
  switch (i) {
    case 6:
    case 0: r = 1; g = n; b = 0; break;
    case 1: r = n; g = 1; b = 0; break;
    case 2: r = 0; g = 1; b = n; break;
    case 3: r = 0; g = n; b = 1; break;
    case 4: r = n; g = 0; b = 1; break;
    default: r = 1; g = 0; b = n; break;
  }
  rgba[0] = (uint8_t)(255 * r);
  rgba[1] = (uint8_t)(255 * g);
  rgba[2] = (uint8_t)(255 * b);
  rgba[3] = 255;
}

struct MeshJob {
  LayerDev L;
  size_t vox_base;   // first voxel of the submap in the batch's voxel numbering
  float T[7];        // T_M_S
  int has_T;
};

}  // namespace

// ------------------------------------------------------------------ kernels
// the job holding batch voxel i: the last job whose vox_base <= i (empty jobs share their successor's base)
__device__ __forceinline__ const MeshJob& mesh_job_of(const MeshJob* __restrict__ jobs, int n, size_t i) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (jobs[mid].vox_base <= i) lo = mid; else hi = mid - 1;
  }
  return jobs[lo];
}

// a[k] for a runtime k without indexing the array (which would move it to local memory)
__device__ __forceinline__ size_t mesh_pick8(const size_t a[8], unsigned k) {
  size_t r = a[0];
#pragma unroll
  for (unsigned c = 1; c < 8; ++c) r = (k == c) ? a[c] : r;
  return r;
}

__device__ __forceinline__ unsigned mesh_config(const float sdf[8]) {
  unsigned cfg = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) cfg |= (sdf[k] < 0 ? 1u : 0u) << k;
  return cfg;
}

// pass 1: triangles of the cube at every voxel; marks the crossing edges of meshed cubes at their low voxel
__global__ void __launch_bounds__(128)
mesh_count_kernel(const MeshJob* __restrict__ jobs, int n_jobs, size_t n_vox, float min_weight,
                  unsigned* __restrict__ tri_cnt, unsigned* __restrict__ vflag) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_vox) return;
  const MeshJob& J = mesh_job_of(jobs, n_jobs, i);
  float sdf[8], coords[3];
  size_t corner[8];
  unsigned nt = 0;
  if (ex_cube(J.L, i - J.vox_base, min_weight, sdf, coords, corner)) {
    const unsigned cfg = mesh_config(sdf);
    nt = c_mesh_ntri[cfg];
    if (nt) {
#pragma unroll
      for (int e = 0; e < 12; ++e) {
        if (!(((cfg >> c_edge[e][0]) ^ (cfg >> c_edge[e][1])) & 1u)) continue;
        const unsigned code = c_mesh_edge[e];
        atomicOr(vflag + J.vox_base + mesh_pick8(corner, code & 7u), 1u << (code >> 3));
      }
    }
  }
  tri_cnt[i] = nt;
}

__global__ void __launch_bounds__(256)
mesh_popc_kernel(const unsigned* __restrict__ vflag, size_t n, unsigned* __restrict__ cnt) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) cnt[i] = (unsigned)__popc(vflag[i]);
}

// per job: its first triangle and first vertex in the batch; the batch totals at the end
__global__ void mesh_offsets_kernel(const MeshJob* __restrict__ jobs, int n_jobs, size_t n_vox,
                                    const unsigned* __restrict__ tri_off, const unsigned* __restrict__ vert_off,
                                    unsigned* __restrict__ out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k > n_jobs) return;
  const size_t at = k < n_jobs ? jobs[k].vox_base : n_vox;
  out[2 * k] = tri_off[at];
  out[2 * k + 1] = vert_off[at];
}

// pass 5: the vertices owned by every voxel (one per marked axis), interpolated from the low end.
// kColour (some submap of the build has a colour channel): also the vertex colour, voxblox
// MeshIntegrator::updateMeshColor with use_color = true, restated from the published sources and not
// checked against a compiled voxblox: a vertex takes the colour word of the voxel that contains it, voxel
// index floor(p / voxel_size + 1e-6) of its position in the layer's own frame (before T_M_S).  The vertex
// sits on a lattice edge whose two end voxels both have weight > min_weight, and the containing voxel is
// one of the two, so it always exists and qualifies: no neighbour search is needed (a voxel the hash does
// not find would give 0).  Vertices of a submap without a channel get 0.
template <bool kColour>
__global__ void __launch_bounds__(128)
mesh_vertex_kernel(const MeshJob* __restrict__ jobs, int n_jobs, size_t n_vox, const unsigned* __restrict__ vflag,
                   const unsigned* __restrict__ vert_off, size_t vbase, float* __restrict__ xyz,
                   uint32_t* __restrict__ vcol) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_vox) return;
  const unsigned f = vflag[i];
  if (!f) return;
  const MeshJob& J = mesh_job_of(jobs, n_jobs, i);
  const LayerDev& L = J.L;
  const size_t local = i - J.vox_base;
  int v[3];
  const int slot = vgx_voxel_of(local, L.sh, v);
  const int b[3] = {L.block_idx[3 * slot], L.block_idx[3 * slot + 1], L.block_idx[3 * slot + 2]};
  const float s_lo = L.dw[local].x;
  float c_lo[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) c_lo[a] = vgx_voxel_centre(b[a], v[a], L.block_size, L.voxel_size);
  size_t o = vbase + vert_off[i];
#pragma unroll
  for (int ax = 0; ax < 3; ++ax) {
    if (!((f >> ax) & 1u)) continue;
    int nv[3] = {v[0], v[1], v[2]};
    int s = slot;
    if (++nv[ax] == L.vps) {   // the high end lies in the next block (allocated: a meshed cube uses it)
      nv[ax] = 0;
      int nb[3] = {b[0], b[1], b[2]};
      ++nb[ax];
      s = vgx_hash_find(L.hash, nb[0], nb[1], nb[2]);
    }
    const float s_hi = L.dw[vgx_voxel_index(s, nv[0], nv[1], nv[2], L.sh)].x;
    float c_hi[3] = {c_lo[0], c_lo[1], c_lo[2]};
    c_hi[ax] = c_lo[ax] + L.voxel_size;
    const float d = s_lo - s_hi;
    float p[3];
    if (fabsf(d) >= 1e-6f) {
      const float t = s_lo / d;
#pragma unroll
      for (int a = 0; a < 3; ++a) p[a] = c_lo[a] + t * (c_hi[a] - c_lo[a]);
    } else {
#pragma unroll
      for (int a = 0; a < 3; ++a) p[a] = 0.5f * (c_lo[a] + c_hi[a]);
    }
    float q[3] = {p[0], p[1], p[2]};
    if (J.has_T) ov_transform(J.T, p, q);
    xyz[3 * o] = q[0]; xyz[3 * o + 1] = q[1]; xyz[3 * o + 2] = q[2];
    if (kColour) {
      uint32_t col = 0;
      if (L.rgba) {
        const int g[3] = {ex_floor(p[0] * L.voxel_size_inv + 1e-6f), ex_floor(p[1] * L.voxel_size_inv + 1e-6f),
                          ex_floor(p[2] * L.voxel_size_inv + 1e-6f)};
        int gb[3];
        const int cs = vgx_global_block(g, L.sh, gb) ? vgx_hash_find(L.hash, gb[0], gb[1], gb[2]) : -1;
        if (cs >= 0) col = L.rgba[vgx_voxel_index(cs, vgx_global_voxel(g, L.sh), L.sh)];
      }
      vcol[o] = col;
    }
    ++o;
  }
}

// pass 6: the triangles of every meshed cube as global vertex indices
__global__ void __launch_bounds__(128)
mesh_triangle_kernel(const MeshJob* __restrict__ jobs, int n_jobs, size_t n_vox, float min_weight,
                     const unsigned* __restrict__ tri_off, const unsigned* __restrict__ vflag,
                     const unsigned* __restrict__ vert_off, size_t vbase, size_t tbase, uint32_t* __restrict__ tri) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_vox) return;
  const unsigned t0 = tri_off[i];
  if (tri_off[i + 1] == t0) return;
  const MeshJob& J = mesh_job_of(jobs, n_jobs, i);
  float sdf[8], coords[3];
  size_t corner[8];
  if (!ex_cube(J.L, i - J.vox_base, min_weight, sdf, coords, corner)) return;   // counted, so never taken
  const unsigned cfg = mesh_config(sdf);
  const int nt = c_mesh_ntri[cfg];
  uint32_t* out = tri + 3 * (tbase + t0);
  for (int k = 0; k < 3 * nt; ++k) {
    const unsigned code = c_mesh_edge[c_mesh_tri[cfg][k]];
    const size_t g = J.vox_base + mesh_pick8(corner, code & 7u);
    const unsigned below = vflag[g] & ((1u << (code >> 3)) - 1u);
    out[k] = (uint32_t)(vbase + vert_off[g] + (unsigned)__popc(below));
  }
}

// binary PLY body: vertex records {float x, y, z; uchar r, g, b, a} then face records {uchar 3; int i[3]}.
// vcol (may be NULL): the vertices' colour words; a submap with voxel[k] != 0 writes them (bytes r, g, b, a =
// the stored word reversed), the others the submap's colour rgba[k].
__global__ void __launch_bounds__(256)
mesh_ply_kernel(const float* __restrict__ xyz, const uint32_t* __restrict__ tri, int64_t nv, int64_t nt,
                const int64_t* __restrict__ voff, int n_sub, const uint32_t* __restrict__ rgba,
                const uint32_t* __restrict__ vcol, const uint32_t* __restrict__ voxel, uint8_t* __restrict__ body) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < nv) {
    int lo = 0, hi = n_sub - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (voff[mid] <= r) lo = mid; else hi = mid - 1;
    }
    uint4 rec;
    rec.x = __float_as_uint(xyz[3 * r]);
    rec.y = __float_as_uint(xyz[3 * r + 1]);
    rec.z = __float_as_uint(xyz[3 * r + 2]);
    rec.w = (vcol && voxel[lo]) ? __byte_perm(vcol[r], 0, 0x0123) : rgba[lo];
    reinterpret_cast<uint4*>(body)[r] = rec;
  } else if (r < nv + nt) {
    const int64_t t = r - nv;
    uint8_t* o = body + 16 * nv + 13 * t;
    o[0] = 3;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const uint32_t x = tri[3 * t + k];
#pragma unroll
      for (int j = 0; j < 4; ++j) o[1 + 4 * k + j] = (uint8_t)(x >> (8 * j));
    }
  }
}

// ------------------------------------------------------------------ host
void vgx_mesh_free(vgx_ctx* c) {
  c->d_mesh_xyz.reset();
  c->d_mesh_tri.reset();
  c->d_mesh_rgba.reset();
  c->mesh_has_colour.clear();
  c->mesh_nv = c->mesh_nt = 0;
  c->mesh_ids.clear();
  c->mesh_voff.assign(1, 0);
}


extern "C" void vgx_mesh_config_default(vgx_mesh_config* cfg) {
  if (!cfg) return;
  cfg->min_weight = 2.0f;   // voxgraph_mapper.yaml:52 mesh_min_weight
}

// one batch of jobs (their vox_base set, n_vox voxels in all) appended to the context's mesh
static int mesh_batch(vgx_ctx* c, std::vector<MeshJob>& jobs, size_t n_vox, float min_weight, bool coloured,
                      std::vector<int64_t>& voff, std::vector<int64_t>& toff) {
  const int nj = (int)jobs.size();
  unsigned *d_cnt, *d_toff, *d_flag, *d_voff, *d_tmp, *d_offs;
  MeshJob* d_jobs;
  VGX_TRY(vgx_carve(c, c->d_work, vgx_part(d_cnt, n_vox + 1), vgx_part(d_toff, n_vox + 1),
                    vgx_part(d_flag, n_vox + 1), vgx_part(d_voff, n_vox + 1),
                    vgx_part(d_tmp, vgx_scan_tmp_count(n_vox)), vgx_part(d_jobs, (size_t)nj),
                    vgx_part(d_offs, 2 * ((size_t)nj + 1))));
  VGX_TRY(vgx_upload(c, d_jobs, jobs.data(), (size_t)nj));
  VGX_TRY(vgx_fill(c, d_flag, n_vox));
  const unsigned g128 = (unsigned)((n_vox + 127) / 128), g256 = (unsigned)((n_vox + 255) / 256);
  {
    VgxProfileScope scope(c, VGX_SLOT_MESH);
    VGX_TRY(vgx_launch(c, mesh_count_kernel, g128, 128, 0, VgxLaunch::plain, d_jobs, nj, n_vox, min_weight, d_cnt,
                       d_flag));
  }
  {
    VgxProfileScope scope(c, VGX_SLOT_MESH);
    VGX_TRY(vgx_exclusive_scan_u32(c, d_cnt, d_toff, n_vox, d_tmp));
  }
  {
    VgxProfileScope scope(c, VGX_SLOT_MESH);
    VGX_TRY(vgx_launch(c, mesh_popc_kernel, g256, 256, 0, VgxLaunch::plain, d_flag, n_vox, d_cnt));
  }
  {
    VgxProfileScope scope(c, VGX_SLOT_MESH);
    VGX_TRY(vgx_exclusive_scan_u32(c, d_cnt, d_voff, n_vox, d_tmp));
  }
  {
    VgxProfileScope scope(c, VGX_SLOT_MESH);
    VGX_TRY(vgx_launch(c, mesh_offsets_kernel, (nj + 1 + 127) / 128, 128, 0, VgxLaunch::plain, d_jobs, nj, n_vox, d_toff,
                       d_voff, d_offs));
  }
  std::vector<unsigned> offs(2 * ((size_t)nj + 1));
  VGX_TRY(vgx_read(c, offs.data(), d_offs, offs.size()));
  const size_t vbase = (size_t)c->mesh_nv, tbase = (size_t)c->mesh_nt;
  const size_t nv = vbase + offs[2 * (size_t)nj + 1], nt = tbase + offs[2 * (size_t)nj];
  if (nv > (size_t)INT32_MAX || nt > (size_t)INT32_MAX)
    VGX_FAIL(c, VGX_ERR_CAPACITY, "more than 2^31 - 1 vertices or triangles");
  for (int k = 0; k < nj; ++k) {
    toff.push_back((int64_t)(tbase + offs[2 * (size_t)k]));
    voff.push_back((int64_t)(vbase + offs[2 * (size_t)k + 1]));
  }
  VGX_TRY(c->d_mesh_xyz.grow_keep(c, 3 * sizeof(float) * std::max(nv, (size_t)1), 3 * sizeof(float) * vbase,
                                  "mesh vertices"));
  VGX_TRY(c->d_mesh_tri.grow_keep(c, 3 * sizeof(uint32_t) * std::max(nt, (size_t)1), 3 * sizeof(uint32_t) * tbase,
                                  "mesh triangles"));
  if (coloured) {
    VGX_TRY(c->d_mesh_rgba.grow_keep(c, sizeof(uint32_t) * std::max(nv, (size_t)1), sizeof(uint32_t) * vbase,
                                     "mesh vertex colours"));
  }
  {
    VgxProfileScope scope(c, VGX_SLOT_MESH);
    VGX_TRY(vgx_launch(c, coloured ? mesh_vertex_kernel<true> : mesh_vertex_kernel<false>, g128, 128, 0, VgxLaunch::plain,
                       d_jobs, nj, n_vox, d_flag, d_voff, vbase, c->d_mesh_xyz.get(),
                       coloured ? c->d_mesh_rgba.get() : nullptr));
  }
  {
    VgxProfileScope scope(c, VGX_SLOT_MESH);
    VGX_TRY(vgx_launch(c, mesh_triangle_kernel, g128, 128, 0, VgxLaunch::plain, d_jobs, nj, n_vox, min_weight, d_toff,
                       d_flag, d_voff, vbase, tbase, c->d_mesh_tri.get()));
  }
  VGX_TRY(vgx_sync(c));   // the scratch is reused by the next batch
  c->mesh_nv = (int64_t)nv;
  c->mesh_nt = (int64_t)nt;
  return VGX_OK;
}

static int mesh_build(vgx_ctx* c, int n, const uint32_t* ids, const float* T_M_S, const vgx_mesh_config& f,
                      std::vector<int64_t>& voff, std::vector<int64_t>& toff) {
  std::vector<VgxSubmap*> subs((size_t)n);
  for (int k = 0; k < n; ++k) VGX_TRY(vgx_submap_get(c, ids[k], &subs[k]));
  VGX_TRY(vgx_sync(c));   // n_blocks of an active submap is final after its integration
  VGX_TRY(ensure_table(c));
  // the build carries vertex colours iff one of its submaps has a colour channel
  bool coloured = false;
  for (int k = 0; k < n; ++k) {
    c->mesh_has_colour.push_back(subs[k]->d_rgba.get() ? 1 : 0);
    coloured = coloured || subs[k]->d_rgba.get();
  }
  std::vector<MeshJob> jobs;
  size_t n_vox = 0;
  for (int k = 0; k <= n; ++k) {
    const size_t sv = k < n ? (size_t)subs[k]->n_blocks * (size_t)subs[k]->vox_per_block : 0;
    if (k == n || (!jobs.empty() && n_vox + sv > VGX_MESH_BATCH_VOXELS)) {   // run the batch so far
      if (n_vox > 0) {
        if (n_vox > (size_t)0xFFFFFFFFu / 5)
          VGX_FAIL(c, VGX_ERR_CAPACITY, "a submap too large for 32-bit triangle counts");
        VGX_TRY(mesh_batch(c, jobs, n_vox, f.min_weight, coloured, voff, toff));
      } else {
        for (size_t j = 0; j < jobs.size(); ++j) {
          voff.push_back(c->mesh_nv);
          toff.push_back(c->mesh_nt);
        }
      }
      jobs.clear();
      n_vox = 0;
      if (k == n) break;
    }
    MeshJob J;
    memset(&J, 0, sizeof(J));
    J.L = layer_of(subs[k]);
    J.vox_base = n_vox;
    J.has_T = T_M_S != nullptr;
    for (int a = 0; a < 7; ++a) J.T[a] = T_M_S ? T_M_S[7 * (size_t)k + a] : 0.0f;
    jobs.push_back(J);
    n_vox += sv;
  }
  voff.push_back(c->mesh_nv);
  toff.push_back(c->mesh_nt);
  return VGX_OK;
}

extern "C" int vgx_mesh_build(vgx_ctx* c, int n, const uint32_t* ids, const float* T_M_S,
                              const vgx_mesh_config* cfg, int64_t* vertex_offsets, int64_t* triangle_offsets) {
  return vgx_entry(c, __func__, [&] {
    if (n < 0 || (n > 0 && !ids)) VGX_FAIL(c, VGX_ERR_INVALID, "invalid argument");
    vgx_mesh_free(c);
    vgx_mesh_config f;
    vgx_mesh_config_default(&f);
    if (cfg) f = *cfg;
    std::vector<int64_t> voff, toff;
    const int rc = mesh_build(c, n, ids, T_M_S, f, voff, toff);
    if (rc != VGX_OK) {
      vgx_mesh_free(c);
      voff.assign((size_t)n + 1, 0);
      toff.assign((size_t)n + 1, 0);
    } else {
      c->mesh_ids.assign(ids, ids + n);
      c->mesh_voff = voff;
    }
    if (vertex_offsets) memcpy(vertex_offsets, voff.data(), voff.size() * sizeof(int64_t));
    if (triangle_offsets) memcpy(triangle_offsets, toff.data(), toff.size() * sizeof(int64_t));
    return rc;
  });
}

extern "C" int vgx_mesh_download(vgx_ctx* c, int64_t max_vertices, float* xyz, int64_t max_triangles,
                                 uint32_t* triangles, int64_t* n_vertices, int64_t* n_triangles) {
  return vgx_entry(c, __func__, [&] {
    if (n_vertices) *n_vertices = c->mesh_nv;
    if (n_triangles) *n_triangles = c->mesh_nt;
    if ((xyz && c->mesh_nv > max_vertices) || (triangles && c->mesh_nt > max_triangles))
      VGX_FAIL(c, VGX_ERR_CAPACITY, "output too small");
    if (xyz && c->mesh_nv) VGX_TRY(vgx_download(c, xyz, c->d_mesh_xyz.get(), 3 * (size_t)c->mesh_nv));
    if (triangles && c->mesh_nt) VGX_TRY(vgx_download(c, triangles, c->d_mesh_tri.get(), 3 * (size_t)c->mesh_nt));
    return vgx_sync(c);
  });
}

extern "C" int vgx_mesh_download_colours(vgx_ctx* c, int64_t max_vertices, uint32_t* rgba, int64_t* n_vertices) {
  return vgx_entry(c, __func__, [&] {
    if (n_vertices) *n_vertices = c->mesh_nv;
    if (!rgba || c->mesh_nv == 0) return VGX_OK;
    if (c->mesh_nv > max_vertices) VGX_FAIL(c, VGX_ERR_CAPACITY, "output too small");
    if (!c->d_mesh_rgba.get()) {   // no submap of the build has a colour channel
      memset(rgba, 0, sizeof(uint32_t) * (size_t)c->mesh_nv);
      return VGX_OK;
    }
    return vgx_read(c, rgba, c->d_mesh_rgba.get(), (size_t)c->mesh_nv);
  });
}

extern "C" int vgx_mesh_ply(vgx_ctx* c, const uint8_t* rgba, uint8_t* out, uint64_t capacity, uint64_t* size) {
  return vgx_entry(c, __func__, [&] { return vgx_mesh_ply_ex(c, rgba, 0, out, capacity, size); });
}

extern "C" int vgx_mesh_ply_ex(vgx_ctx* c, const uint8_t* rgba, int voxel_colours, uint8_t* out, uint64_t capacity,
                               uint64_t* size) {
  return vgx_entry(c, __func__, [&] {
    if (!size) VGX_FAIL(c, VGX_ERR_INVALID, "invalid argument");
    char hdr[512];
    const int hn = snprintf(hdr, sizeof(hdr),
                            "ply\nformat binary_little_endian 1.0\nelement vertex %lld\nproperty float x\n"
                            "property float y\nproperty float z\nproperty uchar red\nproperty uchar green\n"
                            "property uchar blue\nproperty uchar alpha\nelement face %lld\n"
                            "property list uchar int vertex_indices\nend_header\n",
                            (long long)c->mesh_nv, (long long)c->mesh_nt);
    const uint64_t body = 16 * (uint64_t)c->mesh_nv + 13 * (uint64_t)c->mesh_nt;
    *size = (uint64_t)hn + body;
    if (!out) return VGX_OK;
    if (capacity < *size) VGX_FAIL(c, VGX_ERR_CAPACITY, "capacity too small");
    memcpy(out, hdr, (size_t)hn);
    if (body == 0) return VGX_OK;
    const int ns = (int)c->mesh_ids.size();
    std::vector<uint32_t> col((size_t)ns);
    for (int k = 0; k < ns; ++k) {
      uint8_t q[4];
      if (rgba) memcpy(q, rgba + 4 * (size_t)k, 4); else rainbow(c->mesh_ids[k], q);
      col[k] = (uint32_t)q[0] | ((uint32_t)q[1] << 8) | ((uint32_t)q[2] << 16) | ((uint32_t)q[3] << 24);
    }
    const bool voxel = voxel_colours && c->d_mesh_rgba.get();
    std::vector<uint32_t> use((size_t)ns, 0u);
    for (int k = 0; voxel && k < ns; ++k) use[k] = c->mesh_has_colour[k];
    uint8_t* d_body;
    int64_t* d_voff;
    uint32_t *d_col, *d_use;
    VGX_TRY(vgx_carve(c, c->d_scratch, vgx_part(d_body, (size_t)body), vgx_part(d_voff, c->mesh_voff.size()),
                      vgx_part(d_col, col.size()), vgx_part(d_use, voxel ? use.size() : 0)));
    if (voxel) VGX_TRY(vgx_upload(c, d_use, use.data(), use.size()));
    VGX_TRY(vgx_upload(c, d_voff, c->mesh_voff.data(), c->mesh_voff.size()));
    VGX_TRY(vgx_upload(c, d_col, col.data(), col.size()));
    const int64_t recs = c->mesh_nv + c->mesh_nt;
    {
      VgxProfileScope scope(c, VGX_SLOT_MESH);
      VGX_TRY(vgx_launch(c, mesh_ply_kernel, (unsigned)((recs + 255) / 256), 256, 0, VgxLaunch::plain, c->d_mesh_xyz.get(),
                         c->d_mesh_tri.get(), c->mesh_nv, c->mesh_nt, d_voff, ns, d_col,
                         voxel ? c->d_mesh_rgba.get() : nullptr, d_use, d_body));
    }
    return vgx_read(c, out + hn, d_body, (size_t)body);
  });
}
