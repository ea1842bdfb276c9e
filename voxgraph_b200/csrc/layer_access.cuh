// Device access to a resident block layer.  Brick addressing: how a voxel is found in a layer's bricks, for every
// kernel that reads or writes them (the registration path keeps its own, see registration.cuh).  LayerDev: the one
// kernel-facing view of a resident layer.  The cube gather shared by the kernels that sweep marching cubes over a
// layer (extract.cu: isosurface vertices, mesh.cu: submap meshes), the trilinear interpolator shared by extract.cu
// and project.cu, and the minkindr float transform and its inverse shared by overlap.cu, mesh.cu, project.cu,
// evaluate.cu and tsdf.cu.  Every kernel that uses the float helpers is compiled with -fmad=false.
#pragma once

#include "vgx_internal.h"

// ------------------------------------------------------------------ brick addressing
// A brick holds vps^3 voxels, vps = 2^sh, voxel (x, y, z) at the linear index x + vps (y + vps z).  The layer-wide
// index of a voxel is slot vps^3 + linear index, slot being its brick's.  A global voxel index (per axis, in voxels
// from the origin) lies in block g >> sh at voxel g mod vps.

// the voxels_per_side a layer accepts
__host__ __device__ __forceinline__ bool vgx_vps_ok(long long vps) {
  return vps >= 2 && vps <= 32 && (vps & (vps - 1)) == 0;
}
// voxels in one brick, and in n_blocks bricks
__host__ __device__ __forceinline__ int vgx_voxels_per_block(int sh) { return 1 << (3 * sh); }
__host__ __device__ __forceinline__ size_t vgx_voxel_count(int n_blocks, int sh) { return (size_t)n_blocks << (3 * sh); }
// linear index in its brick of voxel (x, y, z), and back
__host__ __device__ __forceinline__ int vgx_voxel_linear(int x, int y, int z, int sh) {
  return x + (y << sh) + (z << (2 * sh));
}
__host__ __device__ __forceinline__ void vgx_voxel_xyz(int lin, int sh, int v[3]) {
  const int m = (1 << sh) - 1;
  v[0] = lin & m;
  v[1] = (lin >> sh) & m;
  v[2] = lin >> (2 * sh);
}
// layer-wide index of the voxel with linear index lin, or (x, y, z), in the brick at slot
__host__ __device__ __forceinline__ size_t vgx_voxel_index(int slot, int lin, int sh) {
  return ((size_t)slot << (3 * sh)) + lin;
}
__host__ __device__ __forceinline__ size_t vgx_voxel_index(int slot, int x, int y, int z, int sh) {
  return ((size_t)slot << (3 * sh)) + x + (y << sh) + (z << (2 * sh));
}
// layer-wide voxel index i -> its brick's slot (returned) and the voxel (x, y, z) in the brick
__host__ __device__ __forceinline__ int vgx_voxel_of(size_t i, int sh, int v[3]) {
  vgx_voxel_xyz((int)(i & (((size_t)1 << (3 * sh)) - 1)), sh, v);
  return (int)(i >> (3 * sh));
}
// one axis of the centre of voxel v of block b (voxblox Block::computeCoordinatesFromLinearIndex)
__host__ __device__ __forceinline__ float vgx_voxel_centre(int b, int v, float block_size, float voxel_size) {
  return (float)b * block_size + ((float)v + 0.5f) * voxel_size;
}
// one axis of a global voxel index (int or 64-bit) -> the voxel's index in its block; also the index in its own
// block of a neighbour one voxel past the brick's face
template <class I>
__host__ __device__ __forceinline__ int vgx_voxel_in_block(I g, int sh) {
  return (int)(g & (((I)1 << sh) - 1));
}
// global voxel index g -> the linear index of the voxel in its block
template <class I>
__host__ __device__ __forceinline__ int vgx_global_voxel(const I g[3], int sh) {
  return vgx_voxel_linear(vgx_voxel_in_block(g[0], sh), vgx_voxel_in_block(g[1], sh), vgx_voxel_in_block(g[2], sh), sh);
}
// global voxel index g -> its block b.  False when a component lies outside [VGX_BLOCK_INDEX_MIN, VGX_BLOCK_INDEX_MAX]:
// no such block exists (vgx_block_in_range).  The test is made on the index as given, before the cast to int could
// wrap a 64-bit one.
template <class I>
__host__ __device__ __forceinline__ bool vgx_global_block(const I g[3], int sh, int b[3]) {
  const I c0 = g[0] >> sh, c1 = g[1] >> sh, c2 = g[2] >> sh;
  b[0] = (int)c0; b[1] = (int)c1; b[2] = (int)c2;
  return c0 >= VGX_BLOCK_INDEX_MIN && c0 <= VGX_BLOCK_INDEX_MAX && c1 >= VGX_BLOCK_INDEX_MIN &&
         c1 <= VGX_BLOCK_INDEX_MAX && c2 >= VGX_BLOCK_INDEX_MIN && c2 <= VGX_BLOCK_INDEX_MAX;
}
// Slots of the bricks that hold the 2x2x2 forward neighbourhood of voxel v of block b (in brick `slot`): nslot[m]
// for the offset m (bit 0 = +x, bit 1 = +y, bit 2 = +z), -1 where the brick does not exist.  An offset leaves the
// brick only on an axis where v is the brick's last voxel, so there is one hash lookup per distinct brick.
__device__ __forceinline__ void vgx_forward_slots(const VgxHash& hash, const int b[3], const int v[3], int slot, int sh,
                                                  int nslot[8]) {
  const int last = (1 << sh) - 1;
  const bool lx = v[0] == last, ly = v[1] == last, lz = v[2] == last;   // an offset along the axis leaves the brick
  nslot[0] = slot;
#pragma unroll
  for (int m = 1; m < 8; ++m) {   // offset m is in the brick of m without an axis that stays, or in a new one
    if ((m & 1) && !lx) nslot[m] = nslot[m ^ 1];
    else if ((m & 2) && !ly) nslot[m] = nslot[m ^ 2];
    else if ((m & 4) && !lz) nslot[m] = nslot[m ^ 4];
    else nslot[m] = vgx_hash_find(hash, b[0] + (m & 1), b[1] + ((m >> 1) & 1), b[2] + (m >> 2));
  }
}

// ------------------------------------------------------------------ layer view
// dw: the (distance, weight) bricks, or the ESDF bricks (distance, observed 1 / 0) of a view of the ESDF layer
struct LayerDev {
  VgxHash hash;
  const float2* dw;
  const int32_t* block_idx;
  const uint32_t* rgba;   // the colour channel (colour.cuh), or NULL
  float voxel_size, voxel_size_inv, block_size, block_size_inv;
  int vps, sh, n_blocks;
};

// which: VGX_LAYER_TSDF or VGX_LAYER_ESDF (the bricks dw points at)
static inline LayerDev layer_of(const VgxSubmap* s, int which = VGX_LAYER_TSDF) {
  LayerDev L;
  L.hash = s->hash();
  L.dw = which == VGX_LAYER_ESDF ? s->d_esdf.get() : s->d_dw.get();
  L.block_idx = s->d_block_idx.get();
  L.rgba = s->d_rgba.get();
  L.voxel_size = s->voxel_size; L.voxel_size_inv = s->voxel_size_inv;
  L.block_size = s->block_size; L.block_size_inv = s->block_size_inv;
  L.vps = s->vps;
  L.sh = s->sh;
  L.n_blocks = s->n_blocks;
  return L;
}

// ------------------------------------------------------------------ cube gather and interpolation
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
  int v[3];
  const int slot = vgx_voxel_of(i, L.sh, v);
  const int b[3] = {L.block_idx[3 * slot], L.block_idx[3 * slot + 1], L.block_idx[3 * slot + 2]};
#pragma unroll
  for (int a = 0; a < 3; ++a) coords[a] = vgx_voxel_centre(b[a], v[a], L.block_size, L.voxel_size);
  int nslot[8];
  vgx_forward_slots(L.hash, b, v, slot, L.sh, nslot);
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int ox = c_cube_off[c][0], oy = c_cube_off[c][1], oz = c_cube_off[c][2];
    const int s = nslot[ox | (oy << 1) | (oz << 2)];
    if (s < 0) return false;
    const size_t at = vgx_voxel_index(s, vgx_voxel_in_block(v[0] + ox, L.sh), vgx_voxel_in_block(v[1] + oy, L.sh),
                                      vgx_voxel_in_block(v[2] + oz, L.sh), L.sh);
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
// kColour (L.rgba != NULL): also Interpolator::interpVoxel's colour, restated from the published voxblox
// sources and not checked against a compiled voxblox: every channel is interpolated like the distance,
// q . (B1 . channel^T) over the 8 neighbours as floats, and converted to uint8 by truncation (an implicit
// float -> uint8 conversion, not round).  The sum can leave [0, 255] by rounding only (the neighbours lie
// inside it); the kernel clamps to [0, 255] before truncating, NaN to 0, where the reference's conversion
// is undefined.
template <bool kColour>
__device__ inline bool ex_interp_voxel_impl(const LayerDev& L, float p0, float p1, float p2, float& out_d,
                                            float& out_w, uint32_t& out_c) {
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
    const float centre = vgx_voxel_centre(b[a], vi, L.block_size, L.voxel_size);
    if (p[a] - centre < 0) {
      if (--vi < 0) { --b[a]; vi += vps; }
    }
    v[a] = vi;
  }
  float d[8], w[8], q[8];
  uint32_t col[kColour ? 8 : 1];
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
        const float centre = vgx_voxel_centre(b[a], cv[a], L.block_size, L.voxel_size);
        off[a] = (p[a] - centre) * L.voxel_size_inv;
      }
      q[0] = 1.0f; q[1] = off[0]; q[2] = off[1]; q[3] = off[2];
      q[4] = off[0] * off[1]; q[5] = off[1] * off[2]; q[6] = off[2] * off[0];
      q[7] = off[0] * off[1] * off[2];
    }
    const size_t at = vgx_voxel_index(slot, cv[0], cv[1], cv[2], L.sh);
    const float2 x = L.dw[at];
    if (kColour) col[i] = L.rgba[at];
    d[i] = x.x;
    w[i] = x.y;
    if (!(x.y > 1e-6f)) return false;
  }
  float res[kColour ? 6 : 2];
#pragma unroll
  for (int k = 0; k < (kColour ? 6 : 2); ++k) {
    float ch[8];
    if (kColour && k >= 2) {
#pragma unroll
      for (int i = 0; i < 8; ++i) ch[i] = (float)((col[i] >> (8 * (k - 2))) & 0xffu);
    }
    const float* x = k == 0 ? d : k == 1 ? w : ch;
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
  if (kColour) {
    out_c = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) out_c |= (uint32_t)fminf(fmaxf(res[2 + k], 0.0f), 255.0f) << (8 * k);
  }
  return true;
}
__device__ inline bool ex_interp_voxel(const LayerDev& L, float p0, float p1, float p2, float& out_d, float& out_w) {
  uint32_t unused;
  return ex_interp_voxel_impl<false>(L, p0, p1, p2, out_d, out_w, unused);
}

// ------------------------------------------------------------------ minkindr float transform
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
