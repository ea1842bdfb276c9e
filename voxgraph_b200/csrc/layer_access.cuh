// Device access to a resident block layer shared by the kernels that sweep marching cubes over it
// (extract.cu: isosurface vertices, mesh.cu: submap meshes), the trilinear interpolator shared by
// extract.cu and project.cu, and the minkindr float transform and its inverse shared by overlap.cu,
// mesh.cu, project.cu and evaluate.cu.  Compiled with -fmad=false by every includer.
#pragma once

#include "vgx_internal.h"

struct LayerDev {
  VgxHash hash;
  const float2* dw;
  const int32_t* block_idx;
  float voxel_size, voxel_size_inv, block_size, block_size_inv;
  int vps, sh, n_blocks;
};

static inline LayerDev layer_of(const VgxSubmap* s) {
  LayerDev L;
  L.hash = s->hash();
  L.dw = s->d_dw.get();
  L.block_idx = s->d_block_idx.get();
  L.voxel_size = s->voxel_size; L.voxel_size_inv = s->voxel_size_inv;
  L.block_size = s->block_size; L.block_size_inv = s->block_size_inv;
  L.vps = s->vps;
  L.sh = s->sh;
  L.n_blocks = s->n_blocks;
  return L;
}

// Cube corner offsets and edges (voxblox MarchingCubes order); host copies use the same initialisers.
#define VGX_CUBE_OFF {{0, 0, 0}, {1, 0, 0}, {1, 1, 0}, {0, 1, 0}, {0, 0, 1}, {1, 0, 1}, {1, 1, 1}, {0, 1, 1}}
#define VGX_CUBE_EDGE {{0, 1}, {1, 2}, {2, 3}, {3, 0}, {4, 5}, {5, 6}, {6, 7}, {7, 4}, {0, 4}, {1, 5}, {2, 6}, {3, 7}}
static __constant__ int c_cube_off[8][3] = VGX_CUBE_OFF;
static __constant__ int c_edge[12][2] = VGX_CUBE_EDGE;

__device__ __forceinline__ int ex_floor(float v) { return __float2int_rd(v); }

// gathers the cube of voxel i: returns false unless all 8 corners have weight > min_weight.
// corner (may be null): the layer-wide voxel index (slot << 3 sh | linear index) of every corner.
__device__ __forceinline__ bool ex_cube(const LayerDev& L, size_t i, float min_weight, float sdf[8],
                                        float coords[3], size_t* corner = nullptr) {
  const int slot = (int)(i >> (3 * L.sh));
  const int lin = (int)(i & (((size_t)1 << (3 * L.sh)) - 1));
  const int v[3] = {lin & (L.vps - 1), (lin >> L.sh) & (L.vps - 1), lin >> (2 * L.sh)};
  const int b[3] = {L.block_idx[3 * slot], L.block_idx[3 * slot + 1], L.block_idx[3 * slot + 2]};
#pragma unroll
  for (int a = 0; a < 3; ++a) coords[a] = (float)b[a] * L.block_size + ((float)v[a] + 0.5f) * L.voxel_size;
  int nslot[8];
  nslot[0] = slot;
#pragma unroll
  for (int k = 1; k < 8; ++k) {  // k bit0 = x overflow, bit1 = y, bit2 = z
    const bool ux = (k & 1) && v[0] == L.vps - 1, uy = (k & 2) && v[1] == L.vps - 1,
               uz = (k & 4) && v[2] == L.vps - 1;
    const int j = (ux ? 1 : 0) | (uy ? 2 : 0) | (uz ? 4 : 0);
    nslot[k] = (j == k) ? vgx_hash_find(L.hash, b[0] + (ux ? 1 : 0), b[1] + (uy ? 1 : 0), b[2] + (uz ? 1 : 0))
                        : nslot[j];
  }
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int ox = c_cube_off[c][0], oy = c_cube_off[c][1], oz = c_cube_off[c][2];
    const int s = nslot[ox | (oy << 1) | (oz << 2)];
    if (s < 0) return false;
    const int x = (v[0] + ox) & (L.vps - 1), y = (v[1] + oy) & (L.vps - 1), z = (v[2] + oz) & (L.vps - 1);
    const size_t at = ((size_t)s << (3 * L.sh)) + x + (y << L.sh) + (z << (2 * L.sh));
    const float2 q = L.dw[at];
    if (q.y <= min_weight) return false;  // utils::getSdfIfValid
    sdf[c] = q.x;
    if (corner) corner[c] = at;
  }
  return true;
}

__device__ __forceinline__ bool ex_edge_crosses(float s1, float s2) {
  return (s1 < 0 && s2 >= 0) || (s1 >= 0 && s2 < 0);
}

// Interpolator::getVoxel(pos, &voxel, interpolate = true): same steps as vgx_locate (registration.cuh)
// on the raw bricks, distance AND weight.  Restates oracle vgo_interp_voxel operation by operation.
__device__ inline bool ex_interp_voxel(const LayerDev& L, float p0, float p1, float p2, float& out_d, float& out_w) {
  const int vps = L.vps;
  const float p[3] = {p0, p1, p2};
  int b[3], v[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) b[a] = ex_floor(p[a] * L.block_size_inv + 1e-6f);
  if (vgx_hash_find(L.hash, b[0], b[1], b[2]) < 0) return false;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float origin = (float)b[a] * L.block_size;
    int vi = ex_floor((p[a] - origin) * L.voxel_size_inv + 1e-6f);
    vi = max(min(vi, vps - 1), 0);
    const float centre = origin + ((float)vi + 0.5f) * L.voxel_size;
    if (p[a] - centre < 0) {
      if (--vi < 0) { --b[a]; vi += vps; }
    }
    v[a] = vi;
  }
  float d[8], w[8], q[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int cv[3] = {v[0] + ((i >> 2) & 1), v[1] + ((i >> 1) & 1), v[2] + (i & 1)};
    int cb[3] = {b[0], b[1], b[2]};
    if (vgx_hash_find(L.hash, b[0], b[1], b[2]) < 0) return false;
#pragma unroll
    for (int a = 0; a < 3; ++a)
      if (cv[a] >= vps) { cb[a]++; cv[a] -= vps; }
    const int slot = vgx_hash_find(L.hash, cb[0], cb[1], cb[2]);
    if (slot < 0) return false;
    if (i == 0) {
      float off[3];
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        const float centre = (float)b[a] * L.block_size + ((float)cv[a] + 0.5f) * L.voxel_size;
        off[a] = (p[a] - centre) * L.voxel_size_inv;
      }
      q[0] = 1.0f; q[1] = off[0]; q[2] = off[1]; q[3] = off[2];
      q[4] = off[0] * off[1]; q[5] = off[1] * off[2]; q[6] = off[2] * off[0];
      q[7] = off[0] * off[1] * off[2];
    }
    const float2 x = L.dw[((size_t)slot << (3 * L.sh)) + cv[0] + (cv[1] << L.sh) + (cv[2] << (2 * L.sh))];
    d[i] = x.x;
    w[i] = x.y;
    if (!(x.y > 1e-6f)) return false;
  }
  float res[2];
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const float* x = k == 0 ? d : w;
    float a[8];
    a[0] = x[0];
    a[1] = -x[0] + x[4];
    a[2] = -x[0] + x[2];
    a[3] = -x[0] + x[1];
    a[4] = x[0] - x[2] - x[4] + x[6];
    a[5] = x[0] - x[1] - x[2] + x[3];
    a[6] = x[0] - x[1] - x[4] + x[5];
    a[7] = -x[0] + x[1] + x[2] - x[3] + x[4] - x[5] - x[6] + x[7];
    float r = q[0] * a[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) r = r + q[i] * a[i];
    res[k] = r;
  }
  out_d = res[0];
  out_w = res[1];
  return true;
}

// Eigen Quaternion::_transformVector (minkindr RotationQuaternion::rotate), float
__host__ __device__ inline void ov_rotate(const float q[4], const float v[3], float o[3]) {
  const float w = q[0], x = q[1], y = q[2], z = q[3];
  float uv0 = y * v[2] - z * v[1], uv1 = z * v[0] - x * v[2], uv2 = x * v[1] - y * v[0];
  uv0 += uv0; uv1 += uv1; uv2 += uv2;
  const float c0 = y * uv2 - z * uv1, c1 = z * uv0 - x * uv2, c2 = x * uv1 - y * uv0;
  o[0] = (v[0] + w * uv0) + c0;
  o[1] = (v[1] + w * uv1) + c1;
  o[2] = (v[2] + w * uv2) + c2;
}
__host__ __device__ inline void ov_transform(const float T[7], const float p[3], float o[3]) {
  float r[3];
  ov_rotate(T, p, r);
  o[0] = r[0] + T[4]; o[1] = r[1] + T[5]; o[2] = r[2] + T[6];
}
// minkindr QuatTransformation::inverse, float (oracle vgo_T_inverse)
__host__ __device__ inline void ov_inverse(const float T[7], float o[7]) {
  const float qi[4] = {T[0], -T[1], -T[2], -T[3]};
  float r[3];
  ov_rotate(qi, T + 4, r);
  o[0] = qi[0]; o[1] = qi[1]; o[2] = qi[2]; o[3] = qi[3];
  o[4] = -r[0]; o[5] = -r[1]; o[6] = -r[2];
}
