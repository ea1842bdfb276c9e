// TSDF ray-cast integration into the HBM brick store (boundary b3).
// Restates voxblox TsdfIntegratorBase::{isPointValid, getVoxelWeight, computeDistance,
// updateTsdfVoxel}, RayCaster and the Simple/Fast scheduling (SURVEY.md Appendix A.4) as
// driven by PointcloudIntegrator::integratePointcloud
// (voxgraph/src/frontend/measurement_processors/pointcloud_integrator.cpp:66-84).
// Compiled with -fmad=false (the float expressions are restated operation by operation).
//
// mode 0 (Simple scheduling, every ray, every voxel) is RAY ORDERED: bit-identical to the
//   single-threaded reference.  allocate pass (blocks of whole rays) -> per-ray update counts ->
//   scan -> emit (voxel address, sdf, update weight) at the ray's offset -> stable radix sort by
//   voxel address -> one thread (short segments) or one warp (long ones) applies a voxel's
//   updates in ray order.
// mode 1 (FastTsdfIntegrator scheduling, what voxgraph runs): one kernel, one thread per ray;
//   blocks are allocated ON DEMAND for the voxels that are actually updated (as
//   allocateStorageAndGetVoxelPtr does), the update is a lock-free 64-bit CAS read-modify-write of
//   the interleaved (distance, weight) pair (replaces the per-voxel mutex); the order in which
//   rays hit a voxel is unspecified, as in the multi-threaded reference.
//
// Colour (rgba != NULL; colour.cuh has the word layout and the blend).  updateTsdfVoxel, restated from the
// published voxblox sources and not checked against a compiled voxblox: with w the voxel's weight BEFORE
// the update and uw the update weight, after the new_weight < 1e-6 early-out,
//   if (|sdf| < truncation) colour = blendTwoColors(colour, w, ray colour, uw).
// Every update outside the band leaves the colour alone.  The rule looks at |sdf| only, so clearing rays
// follow it too: a clearing ray ends at norm - truncation, and the centre of its last voxel can lie
// further along, within truncation of the point (a point just beyond max_ray_length_m); that update is in
// the band and blends the ray's colour.  The colourless call (rgba == NULL)
// runs the kernels it always ran (the <false> instantiations below) and leaves an existing channel
// untouched - the one place this differs from voxblox, which would blend in its default Color().
//   mode 0: the emitted tuple carries the ray's colour (16 bytes instead of 8 through the sort) and the
//     replay applies the rule next to the (distance, weight) recurrence: colour, distance and weight are
//     bit-identical to a sequential replay of the rays, and distance and weight to the colourless call.
//   mode 1: the (distance, weight) update stays the single 64-bit CAS; for a band update the thread first
//     applies the rule to the colour word in a 32-bit CAS loop, with the weight it read for its first CAS
//     attempt (see update_tsdf_voxel for why the colour step leads).  The reference does both under one
//     voxel mutex; here two rays that hit a voxel in one call may apply their colour steps in the other
//     order than their weight steps (the reference's Fast integrator is itself race dependent).  The
//     weight the rule uses is one the voxel held at some point during the call; with other updates of
//     the voxel in flight it need not be the one this ray's CAS replaces.  The fence ordering argument
//     in update_tsdf_voxel rests on reasoning: no test forces the contended interleavings.
//     Contract: (a) a voxel with a single update in a call holds the exact
//     result of the rule; (b) otherwise every channel lies within the closed range spanned by the
//     voxel's previous colour and the colours of the rays that updated it in the band, and is exactly c
//     when those are all one colour c: previous colour c, or previous weight 0 and every update of the
//     voxel in the call inside the band (an update outside it raises the weight of a still default-
//     coloured voxel, and the reference too then blends c with black); (c) distance, weight,
//     statistics and the block set do not depend on the presence of colours.
#include <math.h>
#include <string.h>

#include <type_traits>

#include <cub/cub.cuh>

#include "colour.cuh"
#include "layer_access.cuh"

#define VGX_EPS 1e-6f

struct TsdfParams {
  float q[4], t[3];  // T_G_C
  float voxel_size, voxel_size_inv;
  int sh;            // log2(voxels_per_side)
  vgx_tsdf_config cfg;
  int n;
};

struct DevRay {
  long long cur[3];
  int sign[3];
  float t_next[3], t_step[3];
  long long steps, step;
};

__device__ __forceinline__ void ray_setup(DevRay& rc, const float s[3], const float e[3]) {
  rc.step = 0;
  if (isnan(s[0]) || isnan(s[1]) || isnan(s[2]) || isnan(e[0]) || isnan(e[1]) || isnan(e[2])) {
    rc.steps = -1;
    return;
  }
  rc.steps = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    rc.cur[a] = (long long)floorf(s[a] + VGX_EPS);
    const long long end = (long long)floorf(e[a] + VGX_EPS);
    const long long d = end - rc.cur[a];
    rc.steps += d < 0 ? -d : d;
    const float ray = e[a] - s[a];
    rc.sign[a] = (ray > 0.f) - (ray < 0.f);
    const int corrected = rc.sign[a] > 0 ? rc.sign[a] : 0;
    const float shifted = s[a] - (float)rc.cur[a];
    const float dist = (float)corrected - shifted;
    if (ray == 0.f) {
      rc.t_next[a] = 2.0f;
      rc.t_step[a] = 2.0f;
    } else {
      rc.t_next[a] = dist / ray;
      rc.t_step[a] = (float)rc.sign[a] / ray;
    }
  }
}

__device__ __forceinline__ bool ray_next(DevRay& rc, long long g[3]) {
  if (rc.step++ > rc.steps) return false;
  g[0] = rc.cur[0]; g[1] = rc.cur[1]; g[2] = rc.cur[2];
  // minCoeff: first strictly smallest
  const float t0 = rc.t_next[0], t1 = rc.t_next[1], t2 = rc.t_next[2];
  if (t1 < t0) {
    if (t2 < t1) { rc.cur[2] += rc.sign[2]; rc.t_next[2] = t2 + rc.t_step[2]; }
    else { rc.cur[1] += rc.sign[1]; rc.t_next[1] = t1 + rc.t_step[1]; }
  } else {
    if (t2 < t0) { rc.cur[2] += rc.sign[2]; rc.t_next[2] = t2 + rc.t_step[2]; }
    else { rc.cur[0] += rc.sign[0]; rc.t_next[0] = t0 + rc.t_step[0]; }
  }
  return true;
}

// isPointValid + transform + RayCaster ctor. Returns false for skipped points.
__device__ __forceinline__ bool point_to_ray(const TsdfParams& P, const float* __restrict__ pts, int i,
                                             DevRay& rc, float origin[3], float pG[3], float& weight) {
  const float pC[3] = {pts[3 * (size_t)i], pts[3 * (size_t)i + 1], pts[3 * (size_t)i + 2]};
  // a NaN or infinite coordinate makes the point invalid (undefined in the reference: NaN ray
  // direction, non-finite start key); a finite point whose squared norm overflows stays valid
  if (!(isfinite(pC[0]) && isfinite(pC[1]) && isfinite(pC[2]))) return false;
  const float ray_distance = sqrtf(pC[0] * pC[0] + pC[1] * pC[1] + pC[2] * pC[2]);
  bool clearing = false;
  if (ray_distance < P.cfg.min_ray_length_m) return false;
  if (ray_distance > P.cfg.max_ray_length_m) {
    if (P.cfg.allow_clear) clearing = true;
    else return false;
  }
  origin[0] = P.t[0]; origin[1] = P.t[1]; origin[2] = P.t[2];
  float r[3];
  ov_rotate(P.q, pC, r);
  pG[0] = r[0] + P.t[0]; pG[1] = r[1] + P.t[1]; pG[2] = r[2] + P.t[2];
  // getVoxelWeight
  if (P.cfg.use_const_weight) weight = 1.0f;
  else {
    const float dz = fabsf(pC[2]);
    weight = dz > VGX_EPS ? 1.0f / (dz * dz) : 0.0f;
  }
  const float d[3] = {pG[0] - origin[0], pG[1] - origin[1], pG[2] - origin[2]};
  const float norm = sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
  float u[3] = {d[0], d[1], d[2]};
  if (norm > 0.f) { u[0] = d[0] / norm; u[1] = d[1] / norm; u[2] = d[2] / norm; }
  const float trunc = P.cfg.default_truncation_distance;
  float rs[3], re[3];
  if (clearing) {
    float len = norm - trunc;
    if (len < 0.f) len = 0.f;
    if (len > P.cfg.max_ray_length_m) len = P.cfg.max_ray_length_m;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      re[a] = origin[a] + u[a] * len;
      rs[a] = P.cfg.voxel_carving_enabled ? origin[a] : re[a];
    }
  } else {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      re[a] = pG[a] + u[a] * trunc;
      rs[a] = P.cfg.voxel_carving_enabled ? origin[a] : (pG[a] - u[a] * trunc);
    }
  }
  const float ss[3] = {rs[0] * P.voxel_size_inv, rs[1] * P.voxel_size_inv, rs[2] * P.voxel_size_inv};
  const float es[3] = {re[0] * P.voxel_size_inv, re[1] * P.voxel_size_inv, re[2] * P.voxel_size_inv};
  if (P.cfg.mode == 1) ray_setup(rc, es, ss);  // Fast: cast_from_origin = false
  else ray_setup(rc, ss, es);
  return true;
}

__device__ __forceinline__ unsigned long long any_index_hash64(long long x, long long y, long long z) {
  return (unsigned long long)x + (unsigned long long)y * 17191ull +
         (unsigned long long)z * (17191ull * 17191ull);
}

// Fast scheduling: start-voxel de-duplication at start_voxel_subsampling_factor x resolution.
__device__ __forceinline__ bool fast_start_ok(const TsdfParams& P, const float pG[3],
                                              unsigned long long* start_set) {
  const float inv = P.cfg.start_voxel_subsampling_factor * P.voxel_size_inv;
  const long long k0 = (long long)floorf(pG[0] * inv + VGX_EPS);
  const long long k1 = (long long)floorf(pG[1] * inv + VGX_EPS);
  const long long k2 = (long long)floorf(pG[2] * inv + VGX_EPS);
  const unsigned long long h = any_index_hash64(k0, k1, k2);
  const unsigned long long old = atomicExch(start_set + (h & ((1ull << 20) - 1)), h);
  return old != h;
}

// Block lookup with on-demand allocation (allocateStorageAndGetVoxelPtr): returns the brick slot,
// or -1 when the submap's capacity is exhausted (counters[1] is raised; the key stays behind with
// val = -2 until the host rebuilds the table).  Probe and wait loops are bounded: a full table or
// a lost publisher ends in the overflow flag, never in a hang.
template <bool kWait>
__device__ __forceinline__ int tsdf_get_or_alloc(const VgxHash& hash, int32_t* __restrict__ block_idx,
                                                 int* __restrict__ counters, int capacity, int b0,
                                                 int b1, int b2) {
  const uint64_t key = vgx_pack_key(b0, b1, b2);
  uint32_t h = vgx_hash_index(b0, b1, b2, hash.mask);
  for (uint32_t probes = 0; probes <= hash.mask; ++probes) {
    uint64_t k = *((volatile uint64_t*)&hash.entries[h].key);
    if (k == VGX_EMPTY_KEY) {
      const unsigned long long prev = atomicCAS((unsigned long long*)&hash.entries[h].key,
                                                (unsigned long long)VGX_EMPTY_KEY, (unsigned long long)key);
      if (prev == VGX_EMPTY_KEY) {
        const int slot = atomicAdd(counters, 1);
        if (slot < capacity) {
          block_idx[3 * slot] = b0; block_idx[3 * slot + 1] = b1; block_idx[3 * slot + 2] = b2;
          __threadfence();
          *((volatile int*)&hash.entries[h].val) = slot;
          return slot;
        }
        counters[1] = 1;
        *((volatile int*)&hash.entries[h].val) = -2;
        return -1;
      }
      k = prev;
    }
    if (k == key) {
      if (!kWait) return -1;  // insert-only pass: the slot is not needed yet
      // another thread owns the insertion: wait until it publishes the slot.  The owner may be a
      // lane of this very warp on a divergent path: __nanosleep suspends this lane so the
      // scheduler runs the owner (plain spinning can starve it).
      unsigned ns = 8;
      for (int spin = 0; spin < (1 << 20); ++spin) {
        const int v = *((volatile int*)&hash.entries[h].val);
        if (v >= 0) return v;
        if (v == -2) return -1;
        __nanosleep(ns);
        if (ns < 256) ns <<= 1;
      }
      counters[1] = 1;
      return -1;
    }
    h = (h + 1) & hash.mask;
  }
  counters[1] = 1;
  return -1;
}

// ------------------------------------------------------------------ pass 1: allocate
__global__ void __launch_bounds__(128)
tsdf_allocate_kernel(TsdfParams P, const float* __restrict__ pts, VgxHash hash,
                     int32_t* __restrict__ block_idx, int* __restrict__ counters, int capacity) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P.n) return;
  DevRay rc;
  float origin[3], pG[3], weight;
  if (!point_to_ray(P, pts, i, rc, origin, pG, weight)) return;
  long long g[3];
  int lb0 = INT_MIN, lb1 = 0, lb2 = 0;   // INT_MIN: no block (outside the range)
  while (ray_next(rc, g)) {
    int b[3];
    // a block outside the range is never allocated and its voxels are skipped (its key would alias a block
    // 2^21 away)
    if (!vgx_global_block(g, P.sh, b)) { lb0 = INT_MIN; continue; }
    if (b[0] == lb0 && b[1] == lb1 && b[2] == lb2) continue;
    lb0 = b[0]; lb1 = b[1]; lb2 = b[2];
    tsdf_get_or_alloc<false>(hash, block_idx, counters, capacity, b[0], b[1], b[2]);
  }
}

// ------------------------------------------------------------------ pass 2: integrate
// updateTsdfVoxel, part 1: projective sdf (computeDistance) and the update weight
// (drop-off + sparsity compensation).
__device__ __forceinline__ void tsdf_update_terms(const TsdfParams& P, const float origin[3],
                                                  const float pG[3], const long long g[3],
                                                  float weight, float& sdf, float& uw) {
  const float vs = P.voxel_size;
  const float c0 = ((float)g[0] + 0.5f) * vs, c1 = ((float)g[1] + 0.5f) * vs, c2 = ((float)g[2] + 0.5f) * vs;
  const float vv0 = c0 - origin[0], vv1 = c1 - origin[1], vv2 = c2 - origin[2];
  const float vp0 = pG[0] - origin[0], vp1 = pG[1] - origin[1], vp2 = pG[2] - origin[2];
  const float dist_G = sqrtf(vp0 * vp0 + vp1 * vp1 + vp2 * vp2);
  const float dot = vv0 * vp0 + vv1 * vp1 + vv2 * vp2;
  const float dist_G_V = dot / dist_G;
  sdf = dist_G - dist_G_V;
  uw = weight;
  const float trunc = P.cfg.default_truncation_distance;
  const float dropoff_eps = vs;
  if (P.cfg.use_weight_dropoff && sdf < -dropoff_eps) {
    uw = weight * (trunc + sdf) / (trunc - dropoff_eps);
    uw = uw > 0.0f ? uw : 0.0f;
  }
  if (P.cfg.use_sparsity_compensation_factor) {
    if (fabsf(sdf) < trunc) uw *= P.cfg.sparsity_compensation_factor;
  }
}

// updateTsdfVoxel, part 2: the weighted running average with clamping. Returns false when the
// voxel is left untouched (new_weight < kFloatEpsilon).
__device__ __forceinline__ bool tsdf_apply(float trunc, float max_weight, float sdf, float uw,
                                           float& vd, float& vw) {
  // branch-free: the long-segment replay runs tens of thousands of these back to back
  const float new_weight = vw + uw;
  const bool skip = new_weight < VGX_EPS;
  const float new_sdf = (sdf * uw + vd * vw) / new_weight;
  const float nd = (new_sdf > 0.0f) ? fminf(trunc, new_sdf) : fmaxf(-trunc, new_sdf);
  const float nw = fminf(max_weight, new_weight);
  vd = skip ? vd : nd;
  vw = skip ? vw : nw;
  return !skip;
}

// updateTsdfVoxel's colour rule for one update; vw = the voxel's weight before the update
__device__ __forceinline__ void tsdf_colour_step(float trunc, float sdf, float uw, float vw, uint32_t ray,
                                                 uint32_t& colour) {
  if (vw + uw < VGX_EPS) return;
  if (fabsf(sdf) < trunc) colour = vgx_colour_blend(colour, vw, ray, uw);
}

// kColour: `colour` is the voxel's colour word and `ray` the ray's colour
template <bool kColour>
__device__ __forceinline__ void update_tsdf_voxel(const TsdfParams& P, const float origin[3],
                                                  const float pG[3], const long long g[3],
                                                  float weight, float2* voxel, uint32_t* colour, uint32_t ray) {
  float sdf, uw;
  tsdf_update_terms(P, origin, pG, g, weight, sdf, uw);
  unsigned long long* addr = (unsigned long long*)voxel;
  unsigned long long old = *((volatile unsigned long long*)addr);
  bool colour_pending = kColour && fabsf(sdf) < P.cfg.default_truncation_distance;
  for (;;) {
    float vd = __uint_as_float((unsigned)(old & 0xffffffffull));
    float vw = __uint_as_float((unsigned)(old >> 32));
    const float w_seen = vw;
    if (!tsdf_apply(P.cfg.default_truncation_distance, P.cfg.max_weight, sdf, uw, vd, vw)) return;
    if (colour_pending) {
      // The colour step comes BEFORE this ray's weight step and is made once, with the weight first read
      // (a weight the voxel did hold; another ray may replace it before the CAS below lands).  Hence a
      // thread that reads a weight > 0 finds the colour steps of every band update behind that weight already
      // applied (the fences order colour before weight on the writer and weight before colour on the
      // reader), and a thread that reads weight 0 sets its ray's colour exactly: band updates
      // of one colour c alone, into a voxel of weight 0 or of colour c, can only leave c.
      colour_pending = false;
      __threadfence();
      unsigned c_old = *((volatile unsigned*)colour);
      for (;;) {
        const unsigned c_prev = atomicCAS(colour, c_old, vgx_colour_blend(c_old, w_seen, ray, uw));
        if (c_prev == c_old) break;
        c_old = c_prev;
      }
      __threadfence();
    }
    const unsigned long long nv =
        (unsigned long long)__float_as_uint(vd) | ((unsigned long long)__float_as_uint(vw) << 32);
    const unsigned long long prev = atomicCAS(addr, old, nv);
    if (prev == old) return;
    old = prev;
  }
}

// ------------------------------------------------------------------ deterministic path
// Ray-ordered integration, bit-identical to the single-threaded reference: every ray emits its
// (voxel address, sdf, update weight) tuples at a precomputed offset (ray-major), a stable
// radix sort groups them by voxel keeping ray order, and one thread per voxel applies its
// updates sequentially.
__global__ void __launch_bounds__(128)
tsdf_count_kernel(TsdfParams P, const float* __restrict__ pts, unsigned* __restrict__ counts) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P.n) return;
  DevRay rc;
  float origin[3], pG[3], weight;
  unsigned c = 0;
  if (point_to_ray(P, pts, i, rc, origin, pG, weight) && rc.steps >= 0) c = (unsigned)(rc.steps + 1);
  counts[i] = c;
}

// The tuple a ray emits per voxel: (sdf, update weight), and with colours the ray's colour word
// beside them (16 bytes, so the sort moves one aligned vector per tuple).
template <bool kColour> struct TsdfTuple { typedef float2 type; };
template <> struct TsdfTuple<true> { typedef uint4 type; };
__device__ __forceinline__ float tuple_sdf(const float2& u) { return u.x; }
__device__ __forceinline__ float tuple_uw(const float2& u) { return u.y; }
__device__ __forceinline__ float tuple_sdf(const uint4& u) { return __uint_as_float(u.x); }
__device__ __forceinline__ float tuple_uw(const uint4& u) { return __uint_as_float(u.y); }
__device__ __forceinline__ uint32_t tuple_ray(const float2&) { return 0; }
__device__ __forceinline__ uint32_t tuple_ray(const uint4& u) { return u.z; }
__device__ __forceinline__ void tuple_make(float2& u, float sdf, float uw, uint32_t) { u = make_float2(sdf, uw); }
__device__ __forceinline__ void tuple_make(uint4& u, float sdf, float uw, uint32_t ray) {
  u = make_uint4(__float_as_uint(sdf), __float_as_uint(uw), ray, 0u);
}

template <bool kColour>
__global__ void __launch_bounds__(128)
tsdf_emit_kernel(TsdfParams P, const float* __restrict__ pts, const uint32_t* __restrict__ ray_rgba, VgxHash hash,
                 const unsigned* __restrict__ offsets, unsigned sentinel, unsigned* __restrict__ keys,
                 typename TsdfTuple<kColour>::type* __restrict__ vals, unsigned long long* __restrict__ stats) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long n_valid = 0, n_upd = 0;
  if (i < P.n) {
    DevRay rc;
    float origin[3], pG[3], weight;
    if (point_to_ray(P, pts, i, rc, origin, pG, weight)) {
      n_valid = 1;
      unsigned o = offsets[i];
      const uint32_t ray = kColour ? vgx_colour_pack(ray_rgba[i]) : 0u;
      long long g[3];
      int lb0 = INT_MIN, lb1 = 0, lb2 = 0, slot = -1;
      while (ray_next(rc, g)) {
        int b[3];
        if (!vgx_global_block(g, P.sh, b)) {
          lb0 = INT_MIN; slot = -1;            // outside the range: the voxel is skipped
        } else if (!(b[0] == lb0 && b[1] == lb1 && b[2] == lb2)) {
          lb0 = b[0]; lb1 = b[1]; lb2 = b[2];
          slot = vgx_hash_find(hash, b[0], b[1], b[2]);
        }
        unsigned key = sentinel;
        float sdf = 0.f, uw = 0.f;
        if (slot >= 0) {
          key = (unsigned)vgx_voxel_index(slot, vgx_global_voxel(g, P.sh), P.sh);
          tsdf_update_terms(P, origin, pG, g, weight, sdf, uw);
          ++n_upd;
        }
        keys[o] = key;
        tuple_make(vals[o], sdf, uw, ray);
        ++o;
      }
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    n_valid += __shfl_xor_sync(0xffffffffu, n_valid, off);
    n_upd += __shfl_xor_sync(0xffffffffu, n_upd, off);
  }
  if ((threadIdx.x & 31) == 0) {
    if (n_valid) { atomicAdd(stats + 0, n_valid); atomicAdd(stats + 1, n_valid); }
    if (n_upd) atomicAdd(stats + 2, n_upd);
  }
}

// Segment heads apply their voxel's updates in order. Short segments (the vast majority) are
// handled by the head's thread; long ones (voxels near the sensor collect one update per ray)
// are queued for the warp-cooperative kernel below.
#define VGX_TSDF_LONG_SEGMENT 64
template <bool kColour>
__global__ void __launch_bounds__(256)
tsdf_apply_kernel(const unsigned* __restrict__ keys, const typename TsdfTuple<kColour>::type* __restrict__ vals,
                  unsigned total, unsigned sentinel, float2* __restrict__ dw, uint32_t* __restrict__ rgba,
                  float trunc, float max_weight, unsigned* __restrict__ long_heads, unsigned* __restrict__ n_long) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const unsigned key = keys[i];
  if (key >= sentinel) return;
  if (i > 0 && keys[i - 1] == key) return;  // not the head of its voxel's segment
  // short segment? (bounded look-ahead keeps the loads independent of the recurrence)
  const unsigned probe = i + VGX_TSDF_LONG_SEGMENT;
  if (probe < total && keys[probe] == key) {
    long_heads[atomicAdd(n_long, 1u)] = i;
    return;
  }
  float2 v = dw[key];
  uint32_t col = kColour ? rgba[key] : 0u;
  for (unsigned j = i; j < total && keys[j] == key; ++j) {
    const typename TsdfTuple<kColour>::type u = vals[j];
    if (kColour) tsdf_colour_step(trunc, tuple_sdf(u), tuple_uw(u), v.y, tuple_ray(u), col);
    tsdf_apply(trunc, max_weight, tuple_sdf(u), tuple_uw(u), v.x, v.y);
  }
  dw[key] = v;
  if (kColour) rgba[key] = col;
}

// One warp per long segment: lanes fetch 32 consecutive tuples (coalesced), then every lane
// replays them in order through shuffles, so the serial chain is pure ALU latency.
//
// Saturated batches are not replayed at all.  The voxels next to the sensor collect one update
// per ray (65 k for a 64 x 1024 scan), all of them far in front of the surface (sdf >> trunc):
// once the voxel's distance sits at +trunc, an update with sdf >= 2 trunc leaves it there
//   new_sdf = (sdf uw + trunc w) / (w + uw) >= trunc (1 + uw / (w + uw)) (1 - 4.1 eps) > trunc
// (float rounding of the two products, the sum, the weight sum and the division; needs
// uw / (w + uw) > 4.2 eps, guaranteed by uw >= 2^-20 max_weight) -> fminf(trunc, .) = trunc exactly.
// The weight recurrence w <- min(max_weight, w + uw) is an exact integer sum when w and all uw of
// the batch are integer valued and stay below 2^24 (voxgraph integrates with constant weight 1):
// a whole batch collapses to w <- min(max_weight, w + sum(uw)) - exact partial sums until the cap
// is crossed, pinned at the cap from then on (a voxel already at the cap simply stays there).
// Everything else (first updates, dropped-off weights, fractional weights) takes the sequential replay, so
// the result stays bit-identical to the single-threaded reference
// (tests/test_gpu_tsdf_exact.py::test_dense_scans_bit_exact).
// With colours the shortcut stays valid and is still taken: it needs sdf >= 2 trunc on every lane, and
// the colour rule acts only where |sdf| < trunc, so a saturated batch changes no colour.
template <bool kColour>
__global__ void __launch_bounds__(128)
tsdf_apply_long_kernel(const unsigned* __restrict__ keys, const typename TsdfTuple<kColour>::type* __restrict__ vals,
                       unsigned total, float2* __restrict__ dw, uint32_t* __restrict__ rgba, float trunc,
                       float max_weight, const unsigned* __restrict__ long_heads,
                       const unsigned* __restrict__ n_long, unsigned long long* __restrict__ fast_batches) {
  const unsigned w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const unsigned lane = threadIdx.x & 31;
  if (w >= *n_long) return;
  const unsigned head = long_heads[w];
  const unsigned key = keys[head];
  float2 v = dw[key];
  uint32_t col = kColour ? rgba[key] : 0u;
  const float uw_floor = max_weight * 9.5367431640625e-07f;  // 2^-20 max_weight
  unsigned n_fast = 0;
  // software pipeline: the next batch's tuples are in flight while the current batch is replayed
  typedef typename TsdfTuple<kColour>::type Tuple;
  unsigned j = head + lane;
  bool mine = j < total && keys[j] == key;
  float2 u = make_float2(0.f, 0.f);
  uint32_t uc = 0;     // the ray colour of this lane's tuple
  if (mine) { const Tuple t = vals[j]; u = make_float2(tuple_sdf(t), tuple_uw(t)); uc = tuple_ray(t); }
  for (unsigned base = head; base < total; base += 32) {
    const unsigned jn = base + 32 + lane;
    const bool mine_n = jn < total && keys[jn] == key;
    float2 u_n = make_float2(0.f, 0.f);
    uint32_t uc_n = 0;
    if (mine_n) { const Tuple t = vals[jn]; u_n = make_float2(tuple_sdf(t), tuple_uw(t)); uc_n = tuple_ray(t); }
    const unsigned m = __ballot_sync(0xffffffffu, mine);
    const int cnt = __popc(m);  // the matching lanes form a prefix (keys are sorted)
    if (cnt == 32) {
      // ---- saturated batch? (warp-uniform test)
      bool fast = false;
      const bool capped = v.y == max_weight;   // w <- min(max_weight, w + uw) is stuck at the cap
      if (v.x == trunc && (capped || (v.y == rintf(v.y) && v.y >= 0.f && max_weight < 16777216.0f))) {
        const bool lane_ok = u.x >= 2.0f * trunc && u.y >= uw_floor && (capped || u.y == rintf(u.y));
        if (__all_sync(0xffffffffu, lane_ok)) {
          if (!capped) {
            float sum = u.y;   // integers: every partial sum below the cap is exact (< 2^24)
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
            // step k: w_k = min(max_weight, w_{k-1} + u_k); exact until the cap is crossed, then pinned
            v.y = fminf(max_weight, v.y + sum);
          }
          fast = true;
        }
      }
      if (fast) {
        ++n_fast;
      } else {
        // full batch: stage all 32 tuples in registers first so the shuffles stay off the
        // serial (distance, weight) recurrence
        float sx[32], sy[32];
        uint32_t sc[32];
#pragma unroll
        for (int k = 0; k < 32; ++k) {
          sx[k] = __shfl_sync(0xffffffffu, u.x, k);
          sy[k] = __shfl_sync(0xffffffffu, u.y, k);
          if (kColour) sc[k] = __shfl_sync(0xffffffffu, uc, k);
        }
#pragma unroll
        for (int k = 0; k < 32; ++k) {
          if (kColour) tsdf_colour_step(trunc, sx[k], sy[k], v.y, sc[k], col);
          tsdf_apply(trunc, max_weight, sx[k], sy[k], v.x, v.y);
        }
      }
    } else {
      for (int k = 0; k < cnt; ++k) {
        const float sx = __shfl_sync(0xffffffffu, u.x, k);
        const float sy = __shfl_sync(0xffffffffu, u.y, k);
        if (kColour) tsdf_colour_step(trunc, sx, sy, v.y, __shfl_sync(0xffffffffu, uc, k), col);
        tsdf_apply(trunc, max_weight, sx, sy, v.x, v.y);
      }
      break;
    }
    mine = mine_n;
    u = u_n;
    uc = uc_n;
  }
  if (lane == 0) {
    dw[key] = v;
    if (kColour) rgba[key] = col;
    if (n_fast && fast_batches) atomicAdd(fast_batches, (unsigned long long)n_fast);
  }
}

template <bool kColour>
__global__ void __launch_bounds__(128)
tsdf_integrate_kernel(TsdfParams P, const float* __restrict__ pts, const uint32_t* __restrict__ ray_rgba,
                      VgxHash hash, int32_t* __restrict__ block_idx, int* __restrict__ counters, int capacity,
                      float2* __restrict__ dw, uint32_t* __restrict__ rgba, unsigned long long* __restrict__ stats,
                      unsigned long long* __restrict__ start_set,
                      unsigned long long* __restrict__ obs_set) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long n_valid = 0, n_cast = 0, n_upd = 0;
  if (i < P.n) {
    DevRay rc;
    float origin[3], pG[3], weight;
    if (point_to_ray(P, pts, i, rc, origin, pG, weight)) {
      n_valid = 1;
      bool cast = true;
      if (P.cfg.mode == 1) cast = fast_start_ok(P, pG, start_set);
      if (cast) {
        n_cast = 1;
        const uint32_t ray = kColour ? vgx_colour_pack(ray_rgba[i]) : 0u;
        long long g[3];
        int lb0 = INT_MIN, lb1 = 0, lb2 = 0, slot = -1;
        long long collisions = 0;
        while (ray_next(rc, g)) {
          if (P.cfg.mode == 1) {
            const unsigned long long h = any_index_hash64(g[0], g[1], g[2]);
            const unsigned long long old = atomicExch(obs_set + (h & ((1ull << 20) - 1)), h);
            if (old == h) ++collisions; else collisions = 0;
            if (collisions > P.cfg.max_consecutive_ray_collisions) break;
          }
          int b[3];
          if (!vgx_global_block(g, P.sh, b)) {
            lb0 = INT_MIN; slot = -1;          // outside the range: the voxel is skipped
          } else if (!(b[0] == lb0 && b[1] == lb1 && b[2] == lb2)) {
            lb0 = b[0]; lb1 = b[1]; lb2 = b[2];
            slot = tsdf_get_or_alloc<true>(hash, block_idx, counters, capacity, b[0], b[1], b[2]);
          }
          if (slot < 0) continue;  // outside the range, or capacity exhausted (reported by the host)
          const size_t at = vgx_voxel_index(slot, vgx_global_voxel(g, P.sh), P.sh);
          update_tsdf_voxel<kColour>(P, origin, pG, g, weight, dw + at, kColour ? rgba + at : nullptr, ray);
          ++n_upd;
        }
      }
    }
  }
  // warp-aggregated statistics
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    n_valid += __shfl_xor_sync(0xffffffffu, n_valid, off);
    n_cast += __shfl_xor_sync(0xffffffffu, n_cast, off);
    n_upd += __shfl_xor_sync(0xffffffffu, n_upd, off);
  }
  if ((threadIdx.x & 31) == 0) {
    if (n_valid) atomicAdd(stats + 0, n_valid);
    if (n_cast) atomicAdd(stats + 1, n_cast);
    if (n_upd) atomicAdd(stats + 2, n_upd);
  }
}

// ------------------------------------------------------------------ C-ABI: b3
extern "C" void vgx_tsdf_config_default(vgx_tsdf_config* c) {
  if (!c) return;
  // voxblox defaults overridden by voxgraph/config/voxgraph_mapper.yaml:21-28
  c->default_truncation_distance = 0.6f;
  c->max_weight = 10000.0f;
  c->voxel_carving_enabled = 1;
  c->min_ray_length_m = 0.1f;
  c->max_ray_length_m = 16.0f;
  c->use_const_weight = 1;
  c->allow_clear = 1;
  c->use_weight_dropoff = 1;
  c->use_sparsity_compensation_factor = 1;
  c->sparsity_compensation_factor = 20.0f;
  c->start_voxel_subsampling_factor = 2.0f;
  c->max_consecutive_ray_collisions = 2;
  c->mode = 0;
  c->deterministic = 1;  // ignored: mode 0 is always ray ordered
}

// mode 0 after the scan: emit -> stable sort by voxel -> apply, over `total` tuples whose ray offsets are
// in d_offsets (d_work); the tuple buffers and the sort's scratch go to d_work2
template <bool kColour>
static int tsdf_sort_and_apply(vgx_ctx* c, VgxSubmap* s, const TsdfParams& P, const float* d_pts,
                               const uint32_t* d_ray_rgba, const unsigned* d_offsets, unsigned total,
                               unsigned long long* d_stats) {
  typedef typename TsdfTuple<kColour>::type Tuple;
  // cub moves the tuple as one value of its size
  typedef typename std::conditional<kColour, uint4, unsigned long long>::type SortValue;
  static_assert(sizeof(SortValue) == sizeof(Tuple), "the sort moves whole tuples");
  cudaStream_t stream = c->stream;
  const int n = P.n;
  const unsigned grid = (unsigned)((n + 127) / 128);
  // keys = slot * 4096 + voxel; the sentinel (unmapped block) is one past the largest key
  const unsigned long long sent64 = vgx_voxel_count(s->cap_blocks, P.sh);
  if (sent64 >= 0xFFFFFFFFull) VGX_FAIL(c, VGX_ERR_CAPACITY, "submap too large for 32-bit voxel keys");
  const unsigned sentinel = (unsigned)sent64;
  int end_bit = 1;
  while (end_bit < 32 && (1ull << end_bit) <= sent64) end_bit++;
  size_t sort_tmp = 0;
  VGX_CUDA(c, cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (unsigned*)nullptr, (unsigned*)nullptr,
                                              (SortValue*)nullptr, (SortValue*)nullptr, (int)total, 0, end_bit, stream));
  unsigned *k_in, *k_out, *d_nlong, *d_heads;
  Tuple *v_in, *v_out;
  char* d_sort_tmp;
  VGX_TRY(vgx_carve(c, c->d_work2, vgx_part(k_in, total), vgx_part(k_out, total), vgx_part(v_in, total),
                    vgx_part(v_out, total), vgx_part(d_nlong, 64),
                    vgx_part(d_heads, (size_t)total / VGX_TSDF_LONG_SEGMENT + 2), vgx_part(d_sort_tmp, sort_tmp)));
  uint32_t* d_rgba = kColour ? s->d_rgba.get() : nullptr;
  VgxProfileScope scope(c, VGX_SLOT_TSDF_INTEGRATE);
  VGX_TRY(vgx_fill(c, d_nlong, 64));
  VGX_TRY(vgx_launch(c, tsdf_emit_kernel<kColour>, grid, 128, 0, VgxLaunch::plain, P, d_pts, d_ray_rgba, s->hash(),
                     d_offsets, sentinel, k_in, v_in, d_stats));
  VGX_CUDA(c, cub::DeviceRadixSort::SortPairs(d_sort_tmp, sort_tmp, k_in, k_out, (SortValue*)v_in, (SortValue*)v_out,
                                              (int)total, 0, end_bit, stream));
  vgx_count_launch(c);
  VGX_TRY(vgx_launch(c, tsdf_apply_kernel<kColour>, (total + 255) / 256, 256, 0, VgxLaunch::plain, k_out, v_out, total,
                     sentinel, s->d_dw.get(), d_rgba, P.cfg.default_truncation_distance, P.cfg.max_weight, d_heads,
                     d_nlong));
  // at most total / 64 long segments; launch enough warps, the surplus exits
  const unsigned max_long = total / VGX_TSDF_LONG_SEGMENT + 1;
  return vgx_launch(c, tsdf_apply_long_kernel<kColour>, (max_long + 3) / 4, 128, 0, VgxLaunch::plain, k_out, v_out, total,
                    s->d_dw.get(), d_rgba, P.cfg.default_truncation_distance, P.cfg.max_weight, d_heads, d_nlong,
                    d_stats + 3);
}

int vgx_tsdf_check(vgx_ctx* c, uint32_t id, const float T_G_C[7], const vgx_tsdf_config* cfg, VgxSubmap** out,
                   vgx_tsdf_config* resolved) {
  if (!T_G_C) return VGX_ERR_INVALID;
  VGX_TRY(vgx_submap_get(c, id, out, VgxNeed::active));
  vgx_tsdf_config_default(resolved);
  if (cfg) *resolved = *cfg;
  if (resolved->mode != 0 && resolved->mode != 1) VGX_FAIL(c, VGX_ERR_INVALID, "invalid mode");
  return VGX_OK;
}

int vgx_tsdf_integrate_resident(vgx_ctx* c, VgxSubmap* s, const float T_G_C[7], const vgx_tsdf_config& cfg, int n,
                                const float* d_pts, const uint32_t* d_ray_rgba, unsigned long long* d_stats,
                                unsigned long long* d_start, vgx_tsdf_stats* stats, int* n_points) {
  TsdfParams P;
  memset(&P, 0, sizeof(P));
  P.cfg = cfg;
  for (int k = 0; k < 4; ++k) P.q[k] = T_G_C[k];
  for (int k = 0; k < 3; ++k) P.t[k] = T_G_C[4 + k];
  P.voxel_size = s->voxel_size;
  P.voxel_size_inv = s->voxel_size_inv;
  P.sh = s->sh;
  P.n = n;
  vgx_tsdf_stats st;
  memset(&st, 0, sizeof(st));
  const bool rgba = d_ray_rgba != nullptr;
  int rc;
  // the first coloured scan gives the submap its colour channel, once its scratch is in place; a call that
  // fails later (block capacity) or whose points are all rejected still leaves the channel, all zero
  if (rgba) VGX_TRY(vgx_submap_ensure_colour(c, s));
  unsigned long long* d_obs = d_start + (1u << 20);
  if (P.cfg.mode == 1) VGX_TRY(vgx_fill(c, d_start, vgx_tsdf_set_words(P.cfg), 0xff));
  const int blocks_before = s->n_blocks;
  const unsigned grid = (unsigned)((n + 127) / 128);
  if (P.cfg.mode == 0) {
    // ---- ray-ordered path: allocate -> count -> scan -> emit -> stable sort by voxel -> apply
    {
      VgxProfileScope scope(c, VGX_SLOT_TSDF_ALLOCATE);
      VGX_TRY(vgx_launch(c, tsdf_allocate_kernel, grid, 128, 0, VgxLaunch::plain, P, d_pts, s->hash(), s->d_block_idx.get(),
                         s->d_counters.get(), s->cap_blocks));
    }
    unsigned *d_counts, *d_offsets, *d_scan_tmp;
    VGX_TRY(vgx_carve(c, c->d_work, vgx_part(d_counts, (size_t)n + 2), vgx_part(d_offsets, (size_t)n + 2),
                      vgx_part(d_scan_tmp, vgx_scan_tmp_count((size_t)n))));
    unsigned total = 0;
    {
      VgxProfileScope scope(c, VGX_SLOT_TSDF_INTEGRATE);
      VGX_TRY(vgx_launch(c, tsdf_count_kernel, grid, 128, 0, VgxLaunch::plain, P, d_pts, d_counts));
      VGX_TRY(vgx_exclusive_scan_u32(c, d_counts, d_offsets, (size_t)n, d_scan_tmp));   // hand-written, 3 launches
    }
    VGX_TRY(vgx_read(c, &total, d_offsets + n));
    if (total > 0) {
      VGX_TRY(rgba ? tsdf_sort_and_apply<true>(c, s, P, d_pts, d_ray_rgba, d_offsets, total, d_stats)
                                               : tsdf_sort_and_apply<false>(c, s, P, d_pts, nullptr, d_offsets, total, d_stats));
    }
  } else {
    // ---- Fast scheduling: one kernel, blocks allocated on demand
    VgxProfileScope scope(c, VGX_SLOT_TSDF_INTEGRATE);
    VGX_TRY(vgx_launch(c, rgba ? tsdf_integrate_kernel<true> : tsdf_integrate_kernel<false>, grid, 128, 0,
                       VgxLaunch::plain, P, d_pts, d_ray_rgba, s->hash(), s->d_block_idx.get(), s->d_counters.get(),
                       s->cap_blocks, s->d_dw.get(), rgba ? s->d_rgba.get() : nullptr, d_stats, d_start, d_obs));
  }
  unsigned long long h_stats[VGX_TSDF_STAT_CALLER + 1];
  int h_counters[2];
  VGX_TRY(vgx_download(c, h_stats, d_stats, std::size(h_stats)));
  VGX_TRY(vgx_download(c, h_counters, s->d_counters.get(), std::size(h_counters)));
  VGX_TRY(vgx_sync(c));
  const bool overflow = h_counters[1] != 0 || h_counters[0] > s->cap_blocks;
  s->n_blocks = h_counters[0] < s->cap_blocks ? h_counters[0] : s->cap_blocks;
  st.rays_valid = (int64_t)h_stats[0];
  st.rays_cast = (int64_t)h_stats[1];
  st.voxel_updates = (int64_t)h_stats[2];
  st.blocks_allocated = s->n_blocks - blocks_before;
  st.saturated_batches = (int64_t)h_stats[3];
  if (stats) *stats = st;
  if (n_points) *n_points = (int)h_stats[VGX_TSDF_STAT_CALLER];
  if (overflow) {
    // keys without a brick must not stay in the table: rebuild it from the blocks that exist.  A repair that
    // fails leaves the hash in an unknown state, so its status and message are the call's.
    const int fixed[2] = {s->n_blocks, 0};
    VGX_TRY(vgx_upload(c, s->d_counters.get(), fixed, std::size(fixed)));
    VGX_TRY(vgx_submap_rebuild_hash(c, s));
    VGX_TRY(vgx_sync(c));
    VGX_FAIL(c, VGX_ERR_CAPACITY, "submap block capacity exhausted");
  }
  return VGX_OK;
}

extern "C" int vgx_tsdf_integrate(vgx_ctx* c, uint32_t id, const float T_G_C[7], int n,
                                  const float* points_C, const uint8_t* rgba,
                                  const vgx_tsdf_config* cfg, vgx_tsdf_stats* stats) {
  return vgx_entry(c, __func__, [&] {
    if (!T_G_C || n < 0 || (n > 0 && !points_C)) return VGX_ERR_INVALID;
    VgxSubmap* s;
    vgx_tsdf_config rcfg;
    VGX_TRY(vgx_tsdf_check(c, id, T_G_C, cfg, &s, &rcfg));
    if (n == 0) {
      if (stats) memset(stats, 0, sizeof(*stats));
      return VGX_OK;
    }
    // scratch: points | stats (cleared as 256 bytes) | (fast) two 2^20-entry approximate sets | ray colours
    float* d_pts;
    unsigned long long *d_stats, *d_start;
    uint32_t* d_ray_rgba;   // r, g, b, a bytes per point, as the caller has them
    VGX_TRY(vgx_carve(c, c->d_scratch, vgx_part(d_pts, 3 * (size_t)n), vgx_part(d_stats, VGX_TSDF_STAT_WORDS),
                      vgx_part(d_start, vgx_tsdf_set_words(rcfg)), vgx_part(d_ray_rgba, rgba ? (size_t)n : 0)));
    VGX_TRY(vgx_upload(c, d_pts, points_C, 3 * (size_t)n));
    // the caller's r, g, b, a bytes into the device's colour words: written in bytes
    if (rgba) VGX_TRY(vgx_upload(c, reinterpret_cast<uint8_t*>(d_ray_rgba), rgba, 4 * (size_t)n));
    VGX_TRY(vgx_fill(c, d_stats, VGX_TSDF_STAT_WORDS));
    return vgx_tsdf_integrate_resident(c, s, T_G_C, rcfg, n, d_pts, rgba ? d_ray_rgba : nullptr, d_stats, d_start, stats,
                                       nullptr);
  });
}

extern "C" int vgx_tsdf_integrate_device(vgx_ctx* c, uint32_t id, const float T_G_C[7], int n,
                                         const float* d_points_C, const uint32_t* d_rgba,
                                         const vgx_tsdf_config* cfg, vgx_tsdf_stats* stats) {
  return vgx_entry(c, __func__, [&] {
    if (!T_G_C || n < 0 || (n > 0 && !d_points_C)) return VGX_ERR_INVALID;
    VgxSubmap* s;
    vgx_tsdf_config rcfg;
    VGX_TRY(vgx_tsdf_check(c, id, T_G_C, cfg, &s, &rcfg));
    if (n == 0) {
      if (stats) memset(stats, 0, sizeof(*stats));
      return VGX_OK;
    }
    // the kernels dereference these: refuse host memory and memory of another GPU before any launch
    for (const void* p : {(const void*)d_points_C, (const void*)d_rgba}) {
      if (!p) continue;
      cudaPointerAttributes at;
      VGX_CUDA(c, cudaPointerGetAttributes(&at, p));
      const bool device = at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged;
      if (!device || (at.type == cudaMemoryTypeDevice && at.device != c->device))
        VGX_FAIL(c, VGX_ERR_INVALID, "not device memory of this context's GPU");
    }
    unsigned long long *d_stats, *d_start;
    VGX_TRY(vgx_carve(c, c->d_scratch, vgx_part(d_stats, VGX_TSDF_STAT_WORDS), vgx_part(d_start, vgx_tsdf_set_words(rcfg))));
    VGX_TRY(vgx_fill(c, d_stats, VGX_TSDF_STAT_WORDS));
    return vgx_tsdf_integrate_resident(c, s, T_G_C, rcfg, n, d_points_C, d_rgba, d_stats, d_start, stats, nullptr);
  });
}
