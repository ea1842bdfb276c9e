// Device-side restatement of RegistrationCostFunction::Evaluate
// (voxgraph/src/backend/constraint/cost_functions/registration_cost_function.cpp:58-298)
// and voxblox Interpolator::getVoxelsAndQVector (SURVEY.md Appendix A.3).
//
// This translation unit family is compiled with -fmad=false: every float expression of
// the reference is evaluated operation by operation (IEEE RN, no contraction) so that
// voxel/block indices are bit-exact and residuals/Jacobians match the reference's float
// path.  FMAs are used explicitly (fma()) only where the product is exact in double.
#pragma once

#include <math.h>

#include "vgx_internal.h"

#define VGX_COORD_EPS 1e-6f

// Per-constraint, per-evaluation pose block (cpp:61-110).
struct __align__(16) RegPoseConst {   // 64 bytes: staged by one cp.async.bulk
  float qw, qz;                          // T_reading__reference rotation (yaw-only quaternion)
  float tx, ty, tz;                      // T_reading__reference translation
  float cos_e, sin_e, cos_emo, sin_emo;  // cpp:91-96
  float dxs, dyc, dxc, dys;              // (xe-xo)*sin_e, (ye-yo)*cos_e, (xe-xo)*cos_e, (ye-yo)*sin_e
};

// Reading-submap view + reference points of one residual block.
struct __align__(16) RegConstraintDev {   // 160 bytes: staged by one cp.async.bulk
  const float* pts;    // reference registration points, unit-major AoSoA (vgx_internal.h VgxPoints)
  int n;
  int ref_node, read_node;
  VgxHash hash;        // reading submap block hash
  const float* view;   // reading octets: 8 floats per voxel, NaN where unobserved / missing
  float voxel_size, voxel_size_inv, block_size, block_size_inv;
  int vps, vps_shift;
  const int32_t* grid;  // dense block index over the reading submap's block AABB (or null)
  const uint16_t* grid16;  // the same as 16-bit slots (0xFFFF = no block), padded to 16 bytes: TMA source
  int gmin0, gmin1, gmin2, gd0, gd1, gd2;
  double factor;       // num_residuals / summed_reference_weight (cpp:274)
  double no_corr;      // config.no_correspondence_cost
};

struct TrigHostLibm {  // host: the reference's own calls, std::cos(float) -> cosf
  static __host__ __device__ float cosf_(float x) {
#ifdef __CUDA_ARCH__
    return (float)cos((double)x);
#else
    return ::cosf(x);
#endif
  }
  static __host__ __device__ float sinf_(float x) {
#ifdef __CUDA_ARCH__
    return (float)sin((double)x);
#else
    return ::sinf(x);
#endif
  }
};
struct TrigDevice {  // double evaluation rounded once to float
  static __host__ __device__ float cosf_(float x) { return (float)cos((double)x); }
  static __host__ __device__ float sinf_(float x) { return (float)sin((double)x); }
};

// Eigen Quaternion::_transformVector specialised to q = (w, 0, 0, z) (minkindr rotate()).
__host__ __device__ __forceinline__ void vgx_rotate_yaw(float w, float z, float v0, float v1,
                                                        float v2, float& o0, float& o1, float& o2) {
  float uv0 = -(z * v1);
  float uv1 = z * v0;
  uv0 += uv0;
  uv1 += uv1;
  const float c0 = -(z * uv1);
  const float c1 = z * uv0;
  o0 = (v0 + w * uv0) + c0;
  o1 = (v1 + w * uv1) + c1;
  o2 = v2;
}

// minkindr RotationQuaternion::exp for a pure-yaw rotation vector (Appendix A.1).
__host__ __device__ __forceinline__ void vgx_yaw_quat(float yaw, float& qw, float& qz) {
  const float sq = yaw * yaw;
  const double theta = (double)sqrtf(sq);
  double na;
  if (theta < 1.220703125e-4) {  // eps^(1/4) for double
    na = 0.5 + (theta * theta) * (1.0 / 48.0);
  } else {
    na = sin(theta * 0.5) / theta;
  }
  qw = (float)cos(theta * 0.5);
  qz = (float)((double)yaw * na);
}

template <class Trig>
__host__ __device__ inline void vgx_reg_pose_setup(const double* ref, const double* read,
                                                   RegPoseConst& P) {
  const float xo = (float)ref[0], yo = (float)ref[1], zo = (float)ref[2], tho = (float)ref[3];
  const float xe = (float)read[0], ye = (float)read[1], ze = (float)read[2], the = (float)read[3];
  float wo, qo, we, qe;
  vgx_yaw_quat(tho, wo, qo);
  vgx_yaw_quat(the, we, qe);
  P.cos_e = Trig::cosf_(the);
  P.sin_e = Trig::sinf_(the);
  P.cos_emo = Trig::cosf_(the - tho);
  P.sin_emo = Trig::sinf_(the - tho);
  P.dxs = (xe - xo) * P.sin_e;
  P.dyc = (ye - yo) * P.cos_e;
  P.dxc = (xe - xo) * P.cos_e;
  P.dys = (ye - yo) * P.sin_e;
  // T_mission__reading.inverse(): q^-1 = (we, -qe), t = -(q^-1 rotate t_read)
  const float iw = we, iz = -qe;
  float r0, r1, r2;
  vgx_rotate_yaw(iw, iz, xe, ye, ze, r0, r1, r2);
  const float ti0 = -r0, ti1 = -r1, ti2 = -r2;
  // inverse * T_mission__reference
  P.qw = iw * wo - iz * qo;
  P.qz = iw * qo + iz * wo;
  vgx_rotate_yaw(iw, iz, xo, yo, zo, r0, r1, r2);
  P.tx = ti0 + r0;
  P.ty = ti1 + r1;
  P.tz = ti2 + r2;
}

#ifdef __CUDACC__
// Result of evaluating one registration point.
struct RegPointResult {
  double r;        // unnormalised residual (cpp:161-166)
  float jr[4];     // unnormalised dResidual/dReferencePose (cpp:234-235)
  float je3;       // dResidual/dReadingYaw; je[0..2] == -jr[0..2] exactly
  bool ok;         // interpolation possible
};

// floor(v) as int: single F2I.FLOOR (== (int)floorf(v) for in-range v).
__device__ __forceinline__ int vgx_floor_idx(float v) { return __float2int_rd(v); }

// getVoxelsAndQVector on the octet view, split into phases so that a thread working on several
// points can keep their loads in flight together:
//   locate : base corner voxel (the one whose centre is <= pos on every axis, possibly in the
//            lower neighbour block) and the q-vector offsets
//   probe  : hash path only: first hash probe issued (vgx_probe_start), then the probe sequence
//            finished -> brick slot (vgx_resolve); the block grid path looks the slot up instead
//   fetch  : the voxel's 2x2x2 octet (two 128-bit loads), NaN test
// Returns false when the base block is missing or any corner is unobserved / in a missing
// block (NaN baked into the view).  The reference's first lookup of the block containing pos
// is implied: that block always holds one of the 8 corners.
struct RegLocate {
  float ox, oy, oz;   // q-vector offsets
  int lin;            // voxel index inside the brick
  int b0, b1, b2;     // block of the base corner voxel
};
struct RegProbe {
  uint32_t h;         // current hash table index
  uint64_t key;
  int4 e;             // probed entry
};

// step (1) of getVoxelsAndQVector: index of the block that contains pos
__device__ __forceinline__ void vgx_block_index(const RegConstraintDev& C, float p0, float p1, float p2,
                                                int& b0, int& b1, int& b2) {
  b0 = vgx_floor_idx(p0 * C.block_size_inv + VGX_COORD_EPS);
  b1 = vgx_floor_idx(p1 * C.block_size_inv + VGX_COORD_EPS);
  b2 = vgx_floor_idx(p2 * C.block_size_inv + VGX_COORD_EPS);
}

// shared-memory block grid, 16-bit slots (0xFFFF = no block) -> brick slot or -1
__device__ __forceinline__ int vgx_grid_slot(const RegConstraintDev& C, const uint16_t* __restrict__ s_grid,
                                             int b0, int b1, int b2) {
  const int g0 = b0 - C.gmin0, g1 = b1 - C.gmin1, g2 = b2 - C.gmin2;
  const bool in = (unsigned)g0 < (unsigned)C.gd0 && (unsigned)g1 < (unsigned)C.gd1 &&
                  (unsigned)g2 < (unsigned)C.gd2;
  const int gs = in ? (int)s_grid[(g2 * C.gd1 + g1) * C.gd0 + g0] : 0xFFFF;
  return gs == 0xFFFF ? -1 : gs;
}

// One axis of the base-corner selection.  In: b = the block that contains p.  Out: v = the voxel of
// the base corner, b moved to the lower neighbour block when that corner lies in it, o = the q-vector
// offset from the corner.  The reference moves the voxel index down by one when p lies below the
// voxel centre and then recomputes the corner's centre from the moved indices; here the moved centre
// is selected instead, computed from the same float values:
//   (float)(v - 1) + 0.5f == fv - 0.5f       v is a small integer: both are exact
//   (float)(b - 1) == fb - 1.0f              b is the floor of a float, so fb == b exactly and both
//                                            are b - 1 rounded once (a saturated b has no block)
//   (float)(vps - 1) + 0.5f == vps - 0.5f    exact
// so every corner coordinate, and with it o, is bit-identical to the reference's.
__device__ __forceinline__ void vgx_corner_axis(const RegConstraintDev& C, float p, int& b, int& v, float& o) {
  const int vps = C.vps;
  const float fb = (float)b;
  const float orb = fb * C.block_size;
  v = vgx_floor_idx((p - orb) * C.voxel_size_inv + VGX_COORD_EPS);
  v = max(min(v, vps - 1), 0);
  const float fv = (float)v;
  const float cv = (fv + 0.5f) * C.voxel_size;
  const bool down = p - (orb + cv) < 0;   // the corner is the voxel below
  const bool wrap = down && v == 0;       // ... and it lies in block b - 1
  const float ob = wrap ? (fb - 1.0f) * C.block_size : orb;
  const float oc = down ? ((wrap ? (float)vps : fv) - 0.5f) * C.voxel_size : cv;
  b = wrap ? b - 1 : b;
  v = down ? (wrap ? vps - 1 : v - 1) : v;
  o = (p - (ob + oc)) * C.voxel_size_inv;
}

// b0..b2: the block that contains p (vgx_block_index) -> L (base corner block, voxel, q offsets)
__device__ __forceinline__ void vgx_locate_in_block(const RegConstraintDev& C, float p0, float p1,
                                                    float p2, int b0, int b1, int b2, RegLocate& L) {
  int v0, v1, v2;
  vgx_corner_axis(C, p0, b0, v0, L.ox);
  vgx_corner_axis(C, p1, b1, v1, L.oy);
  vgx_corner_axis(C, p2, b2, v2, L.oz);
  L.b0 = b0; L.b1 = b1; L.b2 = b2;
  const int sh = C.vps_shift;
  L.lin = v0 + (v1 << sh) + (v2 << (2 * sh));
}

__device__ __forceinline__ void vgx_locate(const RegConstraintDev& C, float p0, float p1, float p2,
                                           RegLocate& L) {
  int b0, b1, b2;
  vgx_block_index(C, p0, p1, p2, b0, b1, b2);
  vgx_locate_in_block(C, p0, p1, p2, b0, b1, b2, L);
}

// first probe of the base corner's block in the reading submap's hash (load issued)
__device__ __forceinline__ RegProbe vgx_probe_start(const RegConstraintDev& C, const RegLocate& L) {
  RegProbe H;
  H.key = vgx_pack_key(L.b0, L.b1, L.b2);
  H.h = vgx_hash_index(L.b0, L.b1, L.b2, C.hash.mask);
  H.e = __ldg(reinterpret_cast<const int4*>(C.hash.entries + H.h));
  return H;
}

__device__ __forceinline__ int vgx_resolve(const RegConstraintDev& C, RegProbe& H) {
  for (;;) {
    const uint64_t k = (uint64_t)(uint32_t)H.e.x | ((uint64_t)(uint32_t)H.e.y << 32);
    if (k == H.key) return H.e.z;
    if (k == VGX_EMPTY_KEY) return -1;
    H.h = (H.h + 1) & C.hash.mask;
    H.e = __ldg(reinterpret_cast<const int4*>(C.hash.entries + H.h));
  }
}

__device__ __forceinline__ bool vgx_octet_ok(const float d[8]) {
  // isObservedVoxel failed / block missing <=> NaN in the octet: the sum is NaN iff any is
  const float chk = ((d[0] + d[1]) + (d[2] + d[3])) + ((d[4] + d[5]) + (d[6] + d[7]));
  return chk == chk || !(isnan(d[0]) || isnan(d[1]) || isnan(d[2]) || isnan(d[3]) || isnan(d[4]) ||
                         isnan(d[5]) || isnan(d[6]) || isnan(d[7]));
}

__device__ __forceinline__ bool vgx_interp_gather(const RegConstraintDev& C, float p0, float p1,
                                                  float p2, float d[8], float& ox, float& oy,
                                                  float& oz) {
  RegLocate L;
  vgx_locate(C, p0, p1, p2, L);
  RegProbe H = vgx_probe_start(C, L);
  const int slot = vgx_resolve(C, H);
  if (slot < 0) return false;
  ox = L.ox; oy = L.oy; oz = L.oz;
  const size_t lin = ((size_t)slot << (3 * C.vps_shift)) + L.lin;
  const float4* o = reinterpret_cast<const float4*>(C.view) + 2 * lin;
  const float4 lo = __ldg(o), hi = __ldg(o + 1);
  d[0] = lo.x; d[1] = lo.y; d[2] = lo.z; d[3] = lo.w;
  d[4] = hi.x; d[5] = hi.y; d[6] = hi.z; d[7] = hi.w;
  return vgx_octet_ok(d);
}

// Everything after the gather: B1 coefficients, interpolation, residual, Jacobian.
template <bool kJacobian>
__device__ __forceinline__ RegPointResult vgx_reg_math(const RegConstraintDev& C,
                                                       const RegPoseConst& P, float xi, float yi,
                                                       float dist, float w, bool ok,
                                                       const float d[8], float ox, float oy,
                                                       float oz) {
  RegPointResult R;
  R.ok = ok;
  R.jr[0] = R.jr[1] = R.jr[2] = R.jr[3] = 0.f;
  R.je3 = 0.f;
  if (!R.ok) {
    R.r = (double)w * C.no_corr;  // cpp:164-166
    return R;
  }
  // a = B1 * distances^T (registration_cost_function.h:73-81)
  float a[8];
  a[0] = d[0];
  a[1] = -d[0] + d[4];
  a[2] = -d[0] + d[2];
  a[3] = -d[0] + d[1];
  a[4] = d[0] - d[2] - d[4] + d[6];
  a[5] = d[0] - d[1] - d[2] + d[3];
  a[6] = d[0] - d[1] - d[4] + d[5];
  a[7] = -d[0] + d[1] + d[2] - d[3] + d[4] - d[5] - d[6] + d[7];
  float q[8];
  q[0] = 1.0f; q[1] = ox; q[2] = oy; q[3] = oz;
  q[4] = ox * oy; q[5] = oy * oz; q[6] = oz * ox; q[7] = ox * oy * oz;
  float interp = q[0] * a[0];
#pragma unroll
  for (int k = 1; k < 8; ++k) interp = interp + q[k] * a[k];
  R.r = ((double)dist - (double)interp) * (double)w;  // cpp:158-163
  if (kJacobian) {
    // cpp:183-202: double deltas, float entries
    // (float)(inv * Dx): the double product of two floats is exact, so rounding it to float
    // is the float product; the triple products round once in double first, kept in double.
    const float finv = C.voxel_size_inv;
    const float iDx = finv * q[1], iDy = finv * q[2], iDz = finv * q[3];
    const double inv = (double)finv;
    const double Dx = (double)q[1], Dy = (double)q[2], Dz = (double)q[3];
    const double iDyd = inv * Dy, iDxd = inv * Dx;
    const float iDyDz = (float)(iDyd * Dz), iDxDz = (float)(iDxd * Dz), iDxDy = (float)(iDxd * Dy);
    // cpp:204-205: pInterp_pr = a * pQ_pr summed k = 0..7; the structurally zero entries of
    // pQ_pr add (+-0) and are skipped (value-identical)
    float g0 = a[1] * finv;
    g0 = g0 + a[4] * iDy; g0 = g0 + a[6] * iDz; g0 = g0 + a[7] * iDyDz;
    float g1 = a[2] * finv;
    g1 = g1 + a[4] * iDx; g1 = g1 + a[5] * iDz; g1 = g1 + a[7] * iDxDz;
    float g2 = a[3] * finv;
    g2 = g2 + a[5] * iDy; g2 = g2 + a[6] * iDx; g2 = g2 + a[7] * iDxDy;
    // cpp:214-227
    const float ar03 = xi * P.sin_emo - yi * P.cos_emo;
    const float ar13 = xi * P.cos_emo + yi * P.sin_emo;
    const float ae03 = -xi * P.sin_emo + yi * P.cos_emo + P.dxs - P.dyc;
    const float ae13 = -xi * P.cos_emo - yi * P.sin_emo + P.dxc + P.dys;
    // cpp:234-239: (-w * pInterp_pr) * A, row sums (k0 + k1) + k2
    const float m0 = -w * g0, m1 = -w * g1, m2 = -w * g2;
    R.jr[0] = m0 * P.cos_e + m1 * (-P.sin_e);
    R.jr[1] = m0 * P.sin_e + m1 * P.cos_e;
    R.jr[2] = m2;
    R.jr[3] = m0 * ar03 + m1 * ar13;
    R.je3 = m0 * ae03 + m1 * ae13;
  }
  return R;
}

// cpp:128-129  reading_coordinate = T_reading__reference * reference_coordinate
__device__ __forceinline__ void vgx_reg_transform(const RegPoseConst& P, float xi, float yi, float zi,
                                                  float& p0, float& p1, float& p2) {
  float r0, r1, r2;
  vgx_rotate_yaw(P.qw, P.qz, xi, yi, zi, r0, r1, r2);
  p0 = r0 + P.tx; p1 = r1 + P.ty; p2 = r2 + P.tz;
}

template <bool kJacobian>
__device__ __forceinline__ RegPointResult vgx_reg_point(const RegConstraintDev& C,
                                                        const RegPoseConst& P, float xi, float yi,
                                                        float zi, float dist, float w) {
  float p0, p1, p2;
  vgx_reg_transform(P, xi, yi, zi, p0, p1, p2);
  float d[8], ox = 0, oy = 0, oz = 0;
  const bool ok = vgx_interp_gather(C, p0, p1, p2, d, ox, oy, oz);
  return vgx_reg_math<kJacobian>(C, P, xi, yi, dist, w, ok, d, ox, oy, oz);
}
#endif  // __CUDACC__
