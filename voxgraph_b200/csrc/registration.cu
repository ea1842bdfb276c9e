// Registration kernels: emit mode (Ceres layout, boundary b1) and fused reduce mode
// (per-constraint normal-equation sums, boundary b2).  Compiled with -fmad=false.
#include "registration.cuh"
#include "registration_kernels.h"

#include <type_traits>

// ------------------------------------------------------------------ emit mode
// One thread per registration point; writes the normalised residual and the two 1x4
// Jacobian rows exactly as Evaluate leaves them for Ceres (cpp:254-291).
__global__ void __launch_bounds__(256)
reg_emit_kernel(RegConstraintDev C, RegPoseConst P, double* __restrict__ residuals,
                double* __restrict__ jac_ref, double* __restrict__ jac_read) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= C.n) return;
  const float* pp = C.pts + vgx_pt_index((size_t)i, 0);
  const float xi = __ldg(pp), yi = __ldg(pp + 32), zi = __ldg(pp + 64);
  const float dist = __ldg(pp + 96), w = __ldg(pp + 128);
  RegPointResult R;
  if (jac_ref || jac_read) R = vgx_reg_point<true>(C, P, xi, yi, zi, dist, w);
  else R = vgx_reg_point<false>(C, P, xi, yi, zi, dist, w);
  residuals[i] = R.r * C.factor;
  if (jac_ref) {
    double4 v;
    v.x = (double)R.jr[0] * C.factor; v.y = (double)R.jr[1] * C.factor;
    v.z = (double)R.jr[2] * C.factor; v.w = (double)R.jr[3] * C.factor;
    reinterpret_cast<double4*>(jac_ref)[i] = v;
  }
  if (jac_read) {
    double4 v;
    v.x = (double)(-R.jr[0]) * C.factor; v.y = (double)(-R.jr[1]) * C.factor;
    v.z = (double)(-R.jr[2]) * C.factor; v.w = (double)R.je3 * C.factor;
    reinterpret_cast<double4*>(jac_read)[i] = v;
  }
}

// ------------------------------------------------------------------ reduce mode
// Sums per tile, in double (products of float-valued doubles are exact, so fma == mul+add):
//   S[15] = upper triangle of sum j j^T over j = (jr0, jr1, jr2, jr3, je3)
//   g[5]  = sum j * r,   c = sum r^2
// The 8x8 block of the residual block follows from je[0..2] == -jr[0..2].

// The sums are the 6x6 Gram matrix of v = (jr0, jr1, jr2, jr3, je3, r) over the points, formed
// on the FP64 tensor cores: each warp stages its 32 points' vectors in shared memory and issues
// eight mma.sync.m8n8k4.f64 (A = B^T = 4 points x 8 components), so the reduction over points
// happens inside the MMA and each lane keeps just two accumulators.
__device__ __forceinline__ void dmma_8x8x4(double& d0, double& d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(d0), "+d"(d1)
               : "d"(a), "d"(b));
}

// Half of an octet through the read-only path, marked evict-first in L2.  The gathers are what the kernel spends
// its HBM bandwidth on (asking L2 to fetch 128 or 256 bytes around each sector made a config 2 step 7 and 12 %
// slower); the reading submap's view is far larger than L2 and its sectors are rarely met again before
// they would be evicted, while the point units, block grids and descriptors are re-read by every tile of
// their constraints.  Evict-first keeps the gathers from pushing those out.
__device__ __forceinline__ float4 ldg_evict_first(const float4* p, uint64_t policy) {
  float4 v;
  asm volatile("ld.global.nc.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p), "l"(policy));
  return v;
}

#define VGX_STAGE_STRIDE 36  // doubles per component row (32 points + pad: 2-way = optimal for 8 B)

// ---- TMA (1-D bulk copy) + mbarrier primitives, sm_90a PTX
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "VGX_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra VGX_DONE;\n"
      "bra VGX_WAIT;\n"
      "VGX_DONE:\n"
      "}" ::"r"(bar), "r"(parity) : "memory");
}
// global -> shared bulk copy completing on an mbarrier (SASS UBLKCP); 16-byte aligned, size % 16 == 0
__device__ __forceinline__ void tma_load_1d(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

// ---- unit culling
// A point contributes to the sums only if the block that contains it exists in the reading submap:
// otherwise its octet is missing (early-out in stage A) or holds NaN, and with
// no_correspondence_cost == 0 it adds nothing.  A unit none of whose points can reach an existing
// block is therefore skipped as a whole, before its points are fetched; the sums do not change by a
// bit (a whole unit of zero contributions leaves every accumulator as it was).  Points of weight 0
// with finite coordinates and distance, such as the zero padding of the last unit, are left out of
// the bounds: with the reading submap's distances finite or NaN, such a point adds only +-0.
__global__ void __launch_bounds__(128)
reg_unit_bounds_kernel(const RegTile* __restrict__ tiles, float4* __restrict__ bounds) {
  const RegTile T = tiles[blockIdx.x];
  const int lane = threadIdx.x & 31;
  const int n_units = (T.count + VGX_REG_UNIT - 1) / VGX_REG_UNIT;
  for (int u = threadIdx.x >> 5; u < n_units; u += blockDim.x >> 5) {
    const float* p = T.pts + (size_t)u * VGX_PT_UNIT_FLOATS + lane;
    const float x = p[0], y = p[32], z = p[64], d = p[96], w = p[128];
    const bool finite = isfinite(x) && isfinite(y) && isfinite(z);
    const bool in = !(w == 0.f && finite && isfinite(d));
    float lo0 = in ? x : INFINITY, lo1 = in ? y : INFINITY, lo2 = in ? z : INFINITY;
    float hi0 = in ? x : -INFINITY, hi1 = in ? y : -INFINITY, hi2 = in ? z : -INFINITY;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      lo0 = fminf(lo0, __shfl_xor_sync(0xffffffffu, lo0, off));
      lo1 = fminf(lo1, __shfl_xor_sync(0xffffffffu, lo1, off));
      lo2 = fminf(lo2, __shfl_xor_sync(0xffffffffu, lo2, off));
      hi0 = fmaxf(hi0, __shfl_xor_sync(0xffffffffu, hi0, off));
      hi1 = fmaxf(hi1, __shfl_xor_sync(0xffffffffu, hi1, off));
      hi2 = fmaxf(hi2, __shfl_xor_sync(0xffffffffu, hi2, off));
    }
    const float c0 = 0.5f * (lo0 + hi0), c1 = 0.5f * (lo1 + hi1), c2 = 0.5f * (lo2 + hi2);
    // distance to the (rounded) centre in double, radius rounded up to float
    const double e0 = (double)x - c0, e1 = (double)y - c1, e2 = (double)z - c2;
    double r2 = in ? e0 * e0 + e1 * e1 + e2 * e2 : 0.0;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) r2 = fmax(r2, __shfl_xor_sync(0xffffffffu, r2, off));
    const bool never = __any_sync(0xffffffffu, in && !finite) || !__any_sync(0xffffffffu, in);
    if (lane == 0)
      bounds[T.unit0 + u] = make_float4(c0, c1, c2, never ? INFINITY : __double2float_ru(__dsqrt_ru(r2)));
  }
}

int vgx_launch_reg_unit_bounds(vgx_ctx* c, const RegTile* tiles, int n_tiles, float4* bounds) {
  if (n_tiles <= 0) return VGX_OK;
  return vgx_launch(c, reg_unit_bounds_kernel, n_tiles, 128, 0, VgxLaunch::plain, tiles, bounds);
}

// May a point of the unit with bounding sphere b (reference frame) lie in an existing block?  One
// lane per unit; false only when the answer is provably no.
//
// Why the test is conservative.  Stage A computes, per point x, p = vgx_reg_transform(x) in float and
// then b = floor(p * block_size_inv + VGX_COORD_EPS) (vgx_block_index).  Every one of those last
// operations is monotone in p (round-to-nearest and floor are monotone), so if L <= p <= H on an
// axis, b lies between the block indices of L and H computed by the same expression.  It remains to
// bound p.  With n = qw^2 + qz^2, the transform is p = M x + t exactly, where M is n times a rotation
// in x-y (|M| <= 1 + 2|n - 1|) and the identity in z; so |M x + t - (M c + t)| <= (1 + 2|n - 1|) r on
// every axis.  The float evaluation (six roundings, every intermediate at most 5 (|x| + |t|)) adds
// under 32 ulp-units of (|x| + |t|) for x and again for the centre c, and S below bounds |x| + |t|
// and |c| + |t|; the margin S * 2^-16 = 256 u S (u = 2^-24) covers both with the rounding of L and H
// themselves, and r * 2^-10 covers the rounding of the radius and of |n - 1|.  Non-finite values make
// the unit live.
__device__ __forceinline__ bool reg_unit_may_hit(const RegConstraintDev& C, const RegPoseConst& P,
                                                 const uint16_t* __restrict__ s_grid, const float4 b) {
  float c0, c1, c2;
  vgx_reg_transform(P, b.x, b.y, b.z, c0, c1, c2);
  const float n1 = fabsf(P.qw * P.qw + P.qz * P.qz - 1.0f);
  const float S = ((fabsf(b.x) + fabsf(b.y)) + (fabsf(b.z) + 3.0f * b.w)) +
                  ((fabsf(P.tx) + fabsf(P.ty)) + fabsf(P.tz));
  const float R = b.w + (b.w * (2.0f * n1 + 0x1p-10f) + S * 0x1p-16f);
  if (!isfinite((c0 + c1) + (c2 + R))) return true;
  int l0, l1, l2, h0, h1, h2;
  vgx_block_index(C, c0 - R, c1 - R, c2 - R, l0, l1, l2);
  vgx_block_index(C, c0 + R, c1 + R, c2 + R, h0, h1, h2);
  // box of grid cells, clipped to the grid (64-bit: the indices may be saturated)
  const long long a0 = max((long long)min(l0, h0) - C.gmin0, 0ll), z0 = min((long long)max(l0, h0) - C.gmin0, (long long)C.gd0 - 1);
  const long long a1 = max((long long)min(l1, h1) - C.gmin1, 0ll), z1 = min((long long)max(l1, h1) - C.gmin1, (long long)C.gd1 - 1);
  const long long a2 = max((long long)min(l2, h2) - C.gmin2, 0ll), z2 = min((long long)max(l2, h2) - C.gmin2, (long long)C.gd2 - 1);
  if (a0 > z0 || a1 > z1 || a2 > z2) return false;   // entirely outside the grid
  if ((z0 - a0 + 1) * (z1 - a1 + 1) * (z2 - a2 + 1) > 27) return true;
  for (int g2 = (int)a2; g2 <= (int)z2; ++g2)
    for (int g1 = (int)a1; g1 <= (int)z1; ++g1)
      for (int g0 = (int)a0; g0 <= (int)z0; ++g0)
        if (s_grid[(g2 * C.gd1 + g1) * C.gd0 + g0] != 0xFFFF) return true;
  return false;
}

// Registration reduce kernel, v5.  One CTA per tile; a tile is a run of 32-point units inside one
// residual block (graph.cu cuts them).  CTA b runs tile tile_order[b], the longest-first order
// from the cost measured by an earlier evaluation: the hardware hands CTAs out in index order, so
// the expensive tiles start first and the tail of the grid is made of cheap ones.  The CTA writes
// the tile's 21 sums to partials[tile] and its cost in SM cycles to tile_cost[tile].  Inside the
// tile every warp runs its own software pipeline over the units u = warp, warp + W, ...:
//   * the unit's points (640 contiguous bytes of the unit-major AoSoA layout) are brought into a
//     per-warp 4-slot shared-memory ring by ONE cp.async.bulk (TMA 1-D) completing on an
//     mbarrier, three units ahead - the point loads never touch the LSU path of the math warps;
//   * stage A(u+1): transform -> voxel index -> block-grid lookup (shared memory) -> the octet's
//     two LDG.128 are ISSUED;  stage B(u): the octet issued one iteration earlier is consumed:
//     B1 coefficients, residual, Jacobian, Gram staging + 8 DMMA.  The gather latency of unit
//     u+1 is hidden behind the arithmetic of unit u inside the same warp.
// The last unit is zero-padded to 32 points (weight 0 -> zero contribution), so the
// loop carries no "active" predicate.  Warps never synchronise with each other before the epilogue.
// Block-grid tiles without a no-correspondence cost first test every unit's bounding sphere against
// the block grid (one lane per unit, reg_unit_may_hit); the ring then carries only the units that
// may hit, in the same order, so the per-warp sums are those of the full walk.
template <bool kJacobian>
__global__ void __launch_bounds__(VGX_REG_THREADS, VGX_REG_MIN_BLOCKS)
reg_reduce_kernel(const RegConstraintDev* __restrict__ constraints,
                  const RegPoseConst* __restrict__ poses, const RegTile* __restrict__ tiles,
                  const int* __restrict__ tile_order, int* __restrict__ tile_cost,
                  double* __restrict__ partials, int grid_capacity, const float4* __restrict__ unit_bounds,
                  const int* __restrict__ skip) {
  if (skip && *skip) return;   // evaluation enqueued ahead of a solve that has already ended
  constexpr int kWarps = VGX_REG_THREADS / 32;
  constexpr int kRing = VGX_REG_RING;
  __shared__ __align__(128) float s_ring[kWarps][kRing][5][32];
  __shared__ __align__(8) unsigned long long s_bar[kWarps][kRing];
  __shared__ __align__(8) unsigned long long s_tbar;   // tile barrier: descriptor + pose block + grid
  __shared__ long long s_clk0;   // tile start, SM cycles (thread 0; in a register it spills at 72)
  __shared__ double s_stage[kWarps][6][VGX_STAGE_STRIDE];
  __shared__ double s_gram[kWarps][64];
  __shared__ __align__(16) RegConstraintDev s_C;
  __shared__ __align__(16) RegPoseConst s_P;
  extern __shared__ __align__(16) uint16_t s_grid[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int grp = lane >> 2, tig = lane & 3;
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < kRing; ++k) mbar_init(smem_u32(&s_bar[warp][k]), 1);
    if (warp == 0) mbar_init(smem_u32(&s_tbar), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // the assembly kernel may be scheduled as soon as every CTA of this grid has started; it blocks in
  // griddepcontrol.wait until this grid has completed and its partials are visible
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  __syncthreads();
  const uint32_t ring0 = smem_u32(&s_ring[warp][0][0][0]);
  const uint32_t bar0 = smem_u32(&s_bar[warp][0]);
  const uint32_t tbar = smem_u32(&s_tbar);
  const float* ringf = &s_ring[warp][0][0][0];
  double* stage_w = &s_stage[warp][0][lane];
  const double* stage_r = &s_stage[warp][grp < 6 ? grp : 0][tig];
  uint32_t it = 0;   // units consumed by this warp so far: ring slot = it % kRing, parity = (it / kRing) & 1

  const int tile = __ldg(tile_order + blockIdx.x);
  // the 32-byte tile record is all a thread needs to start the bulk copies
  const int4 rec0 = __ldg(reinterpret_cast<const int4*>(tiles + tile));
  const ulonglong2 rec1 = __ldg(reinterpret_cast<const ulonglong2*>(tiles + tile) + 1);
  RegTile T;
  T.constraint = rec0.x; T.unit0 = rec0.y; T.count = rec0.z; T.grid_bytes = rec0.w;
  T.pts = reinterpret_cast<const float*>(rec1.x);
  T.grid16 = reinterpret_cast<const uint16_t*>(rec1.y);
  const bool use_grid = T.grid_bytes > 0 && T.grid_bytes <= 2 * grid_capacity;
  // ---- descriptor (160 B), pose block (64 B) and the 16-bit block grid: three bulk copies on the
  //      tile barrier; the warps' first point units follow on their own barriers
  if (threadIdx.x == 0) {
    const uint32_t bytes = (uint32_t)sizeof(RegConstraintDev) + (uint32_t)sizeof(RegPoseConst) +
                           (use_grid ? (uint32_t)T.grid_bytes : 0u);
    mbar_expect_tx(tbar, bytes);
    tma_load_1d(smem_u32(&s_C), constraints + T.constraint, (uint32_t)sizeof(RegConstraintDev), tbar);
    if (use_grid) tma_load_1d(smem_u32(s_grid), T.grid16, (uint32_t)T.grid_bytes, tbar);
    // the pose blocks are the only input the preceding kernel (pose set-up) writes: everything
    // above was independent of it (programmatic dependent launch)
    asm volatile("griddepcontrol.wait;" ::: "memory");
    tma_load_1d(smem_u32(&s_P), poses + T.constraint, (uint32_t)sizeof(RegPoseConst), tbar);
  }
  const int n_units = (T.count + 31) >> 5;
  const int my_units = warp < n_units ? (n_units - warp + kWarps - 1) / kWarps : 0;
  // culling needs the pose block, so a tile that may cull issues its first units after the tile
  // barrier; lane j tests unit j of this warp
  const bool may_cull = unit_bounds && use_grid && my_units <= 32;
  float4 bnd = make_float4(0.f, 0.f, 0.f, 0.f);
  if (may_cull && lane < my_units) bnd = __ldg(unit_bounds + T.unit0 + warp + lane * kWarps);
  uint32_t live = 0;   // may_cull: units of this warp not yet issued that may hit (bit j: unit j)
  int next = 0;        // otherwise: next unit to issue
  // producer (lane 0): bring the next unit of this warp into ring slot seq % kRing
  auto issue = [&](uint32_t seq) {
    int j = next++;
    if (may_cull) { j = __ffs(live) - 1; live &= live - 1; }
    if (lane == 0) {
      const uint32_t slot = seq % kRing;
      const uint32_t bar = bar0 + 8u * slot, dst = ring0 + 640u * slot;
      mbar_expect_tx(bar, 640u);
      tma_load_1d(dst, T.pts + (size_t)(warp + j * kWarps) * VGX_PT_UNIT_FLOATS, 640u, bar);
    }
  };
  int n_live = my_units;   // units this warp consumes
  if (!may_cull) {
#pragma unroll
    for (int j = 0; j < kRing - 1; ++j)
      if (j < n_live) issue(it + j);
  }
  mbar_wait(tbar, 0);   // descriptor, pose block and grid have landed
  if (threadIdx.x == 0) s_clk0 = clock64();
  // The tile's constants are read from shared memory once, here, into locals whose address is never
  // taken.  Every ring wait below keeps its "memory" clobber, because it is what orders the reads of a
  // ring slot after the bulk copy that filled it; but a clobber reaches only memory, so these values
  // are not reloaded per unit.  They are the same for the whole CTA, and ptxas holds them in uniform
  // registers, which the 64-register budget of __launch_bounds__ does not count.
  const RegConstraintDev C = s_C;
  const RegPoseConst P = s_P;
  const bool gram_always = C.no_corr != 0.0;  // r = w * no_correspondence_cost without a match
  if (may_cull) {
    live = __ballot_sync(0xffffffffu, lane < my_units && (gram_always || reg_unit_may_hit(C, P, s_grid, bnd)));
    n_live = __popc(live);
#pragma unroll
    for (int j = 0; j < kRing - 1; ++j)
      if (j < n_live) issue(it + j);
  }
  double d0 = 0.0, d1 = 0.0;
  uint64_t octet_policy;
  asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(octet_policy));

  // a lane without a correspondence carries an all-NaN octet
  struct Pipe { float4 lo, hi; float ox, oy, oz; };
  // stage B: consume the octet issued by stage A
  auto stage_b = [&](uint32_t seq, const Pipe& R) {
    const float* sp = ringf + 160 * (seq % kRing) + lane;
    const float d[8] = {R.lo.x, R.lo.y, R.lo.z, R.lo.w, R.hi.x, R.hi.y, R.hi.z, R.hi.w};
    // a unit without a single correspondence adds nothing unless a missing one costs something
    const bool ok = vgx_octet_ok(d);
    if (gram_always || __any_sync(0xffffffffu, ok)) {
      const float xi = sp[0], yi = sp[32], dist = sp[96], w = sp[128];
      const RegPointResult Q = vgx_reg_math<kJacobian>(C, P, xi, yi, dist, w, ok, d, R.ox, R.oy, R.oz);
      if (kJacobian) {
        stage_w[0 * VGX_STAGE_STRIDE] = (double)Q.jr[0];
        stage_w[1 * VGX_STAGE_STRIDE] = (double)Q.jr[1];
        stage_w[2 * VGX_STAGE_STRIDE] = (double)Q.jr[2];
        stage_w[3 * VGX_STAGE_STRIDE] = (double)Q.jr[3];
        stage_w[4 * VGX_STAGE_STRIDE] = (double)Q.je3;
        stage_w[5 * VGX_STAGE_STRIDE] = Q.r;
        __syncwarp();
        // lanes of groups 6 and 7 feed rows 6 and 7 of A with a copy of row 0: those rows reach only row
        // and column 6 and 7 of the Gram matrix, which the epilogue never reads
#pragma unroll
        for (int t4 = 0; t4 < 8; ++t4) {
          const double a = stage_r[4 * t4];
          dmma_8x8x4(d0, d1, a, a);
        }
      } else {
        d0 = fma(Q.r, Q.r, d0);
      }
    }
    __syncwarp();  // every lane is done with this unit's ring slot and the Gram staging buffer
  };

  // The tile's pipeline, instantiated once per lookup path (use_grid is uniform across the CTA):
  // kGrid, the reading submap's block grid staged in shared memory, or its hash in global memory.
  // kShift > 0 fixes the reading submap's brick at 2^kShift voxels per side, so that the voxel clamp,
  // the block wrap and the octet address fold to constants; 0 reads the brick size from the descriptor.
  auto run_tile = [&](auto path, auto brick) {
    constexpr bool kGrid = decltype(path)::value;
    constexpr int kShift = decltype(brick)::value;
    RegConstraintDev K = C;
    if constexpr (kShift > 0) {
      K.vps = 1 << kShift;
      K.vps_shift = kShift;
    }
    // stage A: everything up to the ISSUE of the octet load
    auto stage_a = [&](uint32_t seq, Pipe& R) {
      const uint32_t slot = seq % kRing;
      mbar_wait(bar0 + 8u * slot, (seq / kRing) & 1u);
      const float* sp = ringf + 160 * slot + lane;
      float p0, p1, p2;
      vgx_reg_transform(P, sp[0], sp[32], sp[64], p0, p1, p2);
      const float qnan = __int_as_float(0x7fc00000);
      R.lo = make_float4(qnan, qnan, qnan, qnan);
      R.hi = R.lo;
      R.ox = R.oy = R.oz = 0.f;
      int b0, b1, b2;
      vgx_block_index(K, p0, p1, p2, b0, b1, b2);
      RegLocate L;
      int slot_b;
      if constexpr (kGrid) {
        // getVoxelsAndQVector fails right away when the block that contains pos does not exist;
        // overlapping submaps share only part of their surface and consecutive points are
        // spatially coherent: most warps miss with all 32 lanes and skip the rest of the unit
        const int slot_c = vgx_grid_slot(K, s_grid, b0, b1, b2);
        if (!__any_sync(0xffffffffu, slot_c >= 0)) return;
        vgx_locate_in_block(K, p0, p1, p2, b0, b1, b2, L);
        // the base corner lies in another block only when it moved into a lower neighbour
        const bool moved = (L.b0 != b0) | (L.b1 != b1) | (L.b2 != b2);
        const int slot_m = moved ? vgx_grid_slot(K, s_grid, L.b0, L.b1, L.b2) : slot_c;
        slot_b = slot_c >= 0 ? slot_m : -1;
      } else {
        vgx_probe_range(b0, b1, b2);
        vgx_locate_in_block(K, p0, p1, p2, b0, b1, b2, L);
        RegProbe H = vgx_probe_start(K, L);
        slot_b = vgx_resolve(K, H);
      }
      R.ox = L.ox; R.oy = L.oy; R.oz = L.oz;
      if (slot_b >= 0) {
        const float4* o = reinterpret_cast<const float4*>(K.view) +
                          2 * (((size_t)slot_b << (3 * K.vps_shift)) + (size_t)L.lin);
        // the whole 32-byte octet = one sector = two 128-bit loads (sm_90 has no 256-bit LDG)
        R.lo = ldg_evict_first(o, octet_policy); R.hi = ldg_evict_first(o + 1, octet_policy);
      }
    };
    // two register sets alternate (loop unrolled by two): the in-flight octet is never copied
    Pipe Ra, Rb;
    stage_a(it, Ra);
    int j = 0;
    for (; j + 2 <= n_live; j += 2, it += 2) {
      if (j + kRing - 1 < n_live) issue(it + kRing - 1);
      stage_a(it + 1, Rb);
      stage_b(it, Ra);
      if (j + kRing < n_live) issue(it + kRing);
      if (j + 2 < n_live) stage_a(it + 2, Ra);
      stage_b(it + 1, Rb);
    }
    if (j < n_live) stage_b(it++, Ra);
  };
  // 16 voxels per side: voxblox's default brick, which voxgraph and both bench workloads use
  if (n_live > 0) {
    if (!use_grid) run_tile(std::false_type(), std::integral_constant<int, 0>());
    else if (C.vps_shift == 4) run_tile(std::true_type(), std::integral_constant<int, 4>());
    else run_tile(std::true_type(), std::integral_constant<int, 0>());
  }
  // ---- tile epilogue: warp Gram fragments -> 21 sums -> partials[tile]
  if (kJacobian) {
    s_gram[warp][grp * 8 + 2 * tig] = d0;
    s_gram[warp][grp * 8 + 2 * tig + 1] = d1;
  } else {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) d0 += __shfl_xor_sync(0xffffffffu, d0, off);
    if (lane == 0) s_gram[warp][0] = d0;
  }
  __syncthreads();
  if (threadIdx.x < VGX_REG_NSUM) {
    // entry e of the 21 sums -> (row, col) of the Gram matrix
    int row = 5, col = 5;
    const int e = threadIdx.x;
    if (e < 15) {
      int p = 0, rem = e;
      while (rem >= 5 - p) { rem -= 5 - p; ++p; }
      row = p; col = p + rem;
    } else if (e < 20) {
      row = e - 15; col = 5;
    }
    double s = 0;
    if (kJacobian) {
#pragma unroll
      for (int wv = 0; wv < kWarps; ++wv) s += s_gram[wv][row * 8 + col];
    } else if (e == 20) {
#pragma unroll
      for (int wv = 0; wv < kWarps; ++wv) s += s_gram[wv][0];
    }
    // The tile's sums are final here: no ticket, no fence.  The assembly kernel (a programmatic
    // dependent of this one) adds a constraint's tiles in tile order and applies factor^2
    // (cpp:274-291) - bit-reproducible whatever order the tiles ran in.
    partials[(size_t)tile * VGX_REG_NSTRIDE + e] = s;
    if (e == 0) tile_cost[tile] = (int)min(clock64() - s_clk0, (long long)0x3fffffff);
  }
}

// Longest-processing-time-first order of the tiles from their measured cost (SM cycles of an earlier
// evaluation at nearly the same poses): counting sort into 1024 cost classes, most expensive first.
// One CTA; the order inside a class is arbitrary (the results do not depend on the execution order).
__global__ void __launch_bounds__(1024)
reg_order_kernel(const int* __restrict__ cost, int n, int* __restrict__ order) {
  __shared__ int s_hist[1024];
  __shared__ int s_scan[1024];
  __shared__ int s_max;
  const int t = threadIdx.x;
  s_hist[t] = 0;
  if (t == 0) s_max = 1;
  __syncthreads();
  int m = 1;
  for (int i = t; i < n; i += 1024) m = max(m, cost[i]);
  atomicMax(&s_max, m);
  __syncthreads();
  const float scale = 1023.0f / (float)s_max;
  for (int i = t; i < n; i += 1024) atomicAdd(&s_hist[1023 - min(1023, (int)((float)cost[i] * scale))], 1);
  __syncthreads();
  // exclusive scan of the 1024 classes (Hillis-Steele)
  int v = s_hist[t];
  s_scan[t] = v;
  __syncthreads();
  for (int off = 1; off < 1024; off <<= 1) {
    const int add = t >= off ? s_scan[t - off] : 0;
    __syncthreads();
    s_scan[t] += add;
    __syncthreads();
  }
  s_hist[t] = s_scan[t] - v;
  __syncthreads();
  for (int i = t; i < n; i += 1024)
    order[atomicAdd(&s_hist[1023 - min(1023, (int)((float)cost[i] * scale))], 1)] = i;
}

int vgx_launch_reg_order(vgx_ctx* c, const int* tile_cost, int n_tiles, int* tile_order) {
  if (n_tiles <= 0) return VGX_OK;
  return vgx_launch(c, reg_order_kernel, 1, 1024, 0, VgxLaunch::plain, tile_cost, n_tiles, tile_order);
}

// The pose blocks of one evaluation, one thread per constraint.  The kernel is a programmatic
// dependent of what precedes it, and the pose arithmetic (eight double sin / cos) is most of its
// time, so it is done speculatively BEFORE griddepcontrol.wait from the poses as they read then.
// After the wait the poses are read again (through L2), and the block is recomputed only if one of
// them differs bit for bit: the block written is always the one of the poses the predecessor left,
// and when they did not change (consecutive evaluations at the same poses) the arithmetic is off the
// critical path.  The pose blocks themselves are written after the wait: they were read by the
// previous evaluation's reduce kernel, which has completed once the assembly (its dependent) has.
__device__ __forceinline__ void reg_load_pose(const double* x, int node, double* p) {
  const double2* q = reinterpret_cast<const double2*>(x + 4 * (size_t)node);   // 32-byte aligned rows
  const double2 a = __ldcg(q), b = __ldcg(q + 1);
  p[0] = a.x; p[1] = a.y; p[2] = b.x; p[3] = b.y;
}
__global__ void reg_pose_setup_kernel(const RegConstraintDev* __restrict__ constraints, const double* x,
                                      RegPoseConst* __restrict__ poses, int n_constraints,
                                      const int* __restrict__ skip) {
  // programmatic dependent launch: the reduce kernel may start its prologue (tile records, TMA of the
  // descriptors, block grids and first point units) while the pose blocks are still being computed
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const bool active = c < n_constraints;
  int na = 0, nb = 0;
  double ref[4] = {0, 0, 0, 0}, read[4] = {0, 0, 0, 0};
  RegPoseConst P;
  if (active) {
    na = __ldg(&constraints[c].ref_node);
    nb = __ldg(&constraints[c].read_node);
    reg_load_pose(x, na, ref);
    reg_load_pose(x, nb, read);
    vgx_reg_pose_setup<TrigDevice>(ref, read, P);
  }
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (skip && *skip) return;
  if (!active) return;
  double ref1[4], read1[4];
  reg_load_pose(x, na, ref1);
  reg_load_pose(x, nb, read1);
  bool same = true;
#pragma unroll
  for (int k = 0; k < 4; ++k)
    same = same && __double_as_longlong(ref1[k]) == __double_as_longlong(ref[k]) &&
           __double_as_longlong(read1[k]) == __double_as_longlong(read[k]);
  if (!same) vgx_reg_pose_setup<TrigDevice>(ref1, read1, P);
  poses[c] = P;
}

// ------------------------------------------------------------------ launch helpers
int vgx_launch_reg_pose_setup(vgx_ctx* c, const RegConstraintDev* cons, const double* x, RegPoseConst* poses, int n,
                              const int* skip) {
  if (n <= 0) return VGX_OK;
  return vgx_launch(c, reg_pose_setup_kernel, (unsigned)((n + 127) / 128), 128, 0, VgxLaunch::pdl, cons, x, poses, n,
                    skip);
}

int vgx_launch_reg_reduce(vgx_ctx* c, const RegConstraintDev* cons, const RegPoseConst* poses, const RegTile* tiles,
                          int n_tiles, const int* tile_order, int* tile_cost, double* partials, int grid_capacity,
                          const float4* unit_bounds, bool jacobian, const int* skip) {
  if (n_tiles <= 0) return VGX_OK;
  // its CTAs may start while the pose set-up kernel is still running; they block at
  // griddepcontrol.wait before touching the pose blocks
  return vgx_launch(c, jacobian ? reg_reduce_kernel<true> : reg_reduce_kernel<false>, (unsigned)n_tiles,
                    VGX_REG_THREADS, sizeof(uint16_t) * (size_t)grid_capacity, VgxLaunch::pdl, cons, poses, tiles,
                    tile_order, tile_cost, partials, grid_capacity, unit_bounds, skip);
}

// cpp:45-55: num_residuals = int(sampling_ratio * size()) (float product) or size()
static int reg_num_residuals(const VgxPoints& p, const vgx_reg_config* cfg) {
  if (cfg->sampling_ratio != -1.0f) return (int)(cfg->sampling_ratio * (float)(size_t)p.n);
  return p.n;
}

__global__ void reg_gather_samples_kernel(const float* __restrict__ src, const int32_t* __restrict__ idx,
                                          int n, float* __restrict__ dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ((n + 31) & ~31)) return;
  float x = 0.f, y = 0.f, z = 0.f, d = 0.f, w = 0.f;
  if (i < n) {
    const float* sp = src + vgx_pt_index((size_t)idx[i], 0);
    x = sp[0]; y = sp[32]; z = sp[64]; d = sp[96];
    w = 1.0f;  // cpp:121 registration_point.weight = 1
  }
  float* dp = dst + vgx_pt_index((size_t)i, 0);
  dp[0] = x; dp[32] = y; dp[64] = z; dp[96] = d; dp[128] = w;
}

int vgx_launch_reg_gather_samples(vgx_ctx* c, const float* src, const int32_t* d_idx, int n, float* dst) {
  if (n <= 0) return VGX_OK;
  const int padded = (n + 31) & ~31;
  return vgx_launch(c, reg_gather_samples_kernel, (padded + 255) / 256, 256, 0, VgxLaunch::plain, src, d_idx, n, dst);
}

int vgx_fill_constraint(vgx_ctx* c, uint32_t ref_id, uint32_t read_id, const vgx_reg_config* cfg,
                        RegConstraintDev* out, bool* sampled) {
  if (!cfg) VGX_FAIL(c, VGX_ERR_INVALID, "null registration config");
  if (cfg->registration_point_type < 0 || cfg->registration_point_type > 1)
    VGX_FAIL(c, VGX_ERR_INVALID, "invalid registration_point_type");
  if (cfg->sampling_ratio != -1.0f && !(cfg->sampling_ratio >= 0.0f))
    VGX_FAIL(c, VGX_ERR_INVALID, "sampling_ratio must be -1 (all points) or >= 0");
  if (ref_id == read_id) VGX_FAIL(c, VGX_ERR_INVALID, "cannot constrain a submap to itself");
  VgxSubmap *ref, *rd;
  VGX_TRY(vgx_submap_get(c, ref_id, &ref));
  VGX_TRY(vgx_submap_get(c, read_id, &rd));
  if (!rd->finished || !rd->d_view.get())
    VGX_FAIL(c, VGX_ERR_INVALID, "registration constraint: reading submap is not finished");
  if (cfg->use_esdf_distance && !rd->d_view_esdf.get())
    VGX_FAIL(c, VGX_ERR_INVALID, "registration constraint: use_esdf_distance needs the reading submap's ESDF "
                                 "(vgx_submap_generate_esdf)");
  const VgxPoints& p = ref->points[cfg->registration_point_type];
  const bool is_sampled = cfg->sampling_ratio != -1.0f;
  RegConstraintDev C;
  C.pts = is_sampled ? nullptr : p.data.get();
  C.n = reg_num_residuals(p, cfg);
  C.ref_node = -1; C.read_node = -1;
  C.hash = rd->hash();
  C.view = cfg->use_esdf_distance ? rd->d_view_esdf.get() : rd->d_view.get();   // cpp:133-153
  C.voxel_size = rd->voxel_size; C.voxel_size_inv = rd->voxel_size_inv;
  C.block_size = rd->block_size; C.block_size_inv = rd->block_size_inv;
  C.vps = rd->vps;
  C.grid = rd->d_grid.get();
  C.grid16 = rd->d_grid16.get();
  C.gmin0 = rd->grid_min[0]; C.gmin1 = rd->grid_min[1]; C.gmin2 = rd->grid_min[2];
  C.gd0 = rd->grid_dim[0]; C.gd1 = rd->grid_dim[1]; C.gd2 = rd->grid_dim[2];
  C.vps_shift = rd->sh;
  // cpp:274 factor = num_residuals / summed_reference_weight; sampled points all weigh 1
  if (is_sampled) C.factor = (C.n > 0 && p.n > 0) ? 1.0 : 0.0;
  else C.factor = (p.sum_w != 0.0) ? (double)p.n / p.sum_w : 0.0;
  C.no_corr = cfg->no_correspondence_cost;
  *out = C;
  if (sampled) *sampled = is_sampled;
  return VGX_OK;
}

// ------------------------------------------------------------------ C-ABI: b1
extern "C" void vgx_reg_config_default(vgx_reg_config* cfg) {
  if (!cfg) return;
  cfg->registration_point_type = VGX_POINTS_ISOSURFACE;  // h:20-21
  cfg->no_correspondence_cost = 0.0;                      // h:32
  cfg->sampling_ratio = -1.0f;                            // h:28
  cfg->use_esdf_distance = 0;                             // h:35 defaults to true; needs an ESDF
}

extern "C" int vgx_reg_num_residuals(vgx_ctx* c, uint32_t ref_id, const vgx_reg_config* cfg, int* n) {
  return vgx_entry(c, __func__, [&] {
    if (!cfg || !n) return VGX_ERR_INVALID;
    VgxSubmap* ref;
    VGX_TRY(vgx_submap_get(c, ref_id, &ref));
    if (cfg->registration_point_type < 0 || cfg->registration_point_type > 1) return VGX_ERR_INVALID;
    if (cfg->sampling_ratio != -1.0f && !(cfg->sampling_ratio >= 0.0f)) return VGX_ERR_INVALID;
    *n = reg_num_residuals(ref->points[cfg->registration_point_type], cfg);
    return VGX_OK;
  });
}

extern "C" int vgx_reg_eval_emit(vgx_ctx* c, uint32_t ref_id, uint32_t read_id,
                                 const vgx_reg_config* cfg, const double ref_pose[4],
                                 const double read_pose[4], double* residuals, double* jac_ref,
                                 double* jac_read) {
  return vgx_entry(c, __func__, [&] {
    if (!ref_pose || !read_pose || !residuals) return VGX_ERR_INVALID;
    RegConstraintDev C;
    bool sampled = false;
    VGX_TRY(vgx_fill_constraint(c, ref_id, read_id, cfg, &C, &sampled));
    if (C.n == 0) return VGX_ZERO_WEIGHT;  // summed weight 0 -> Evaluate returns false
    if (C.factor == 0.0) return VGX_ZERO_WEIGHT;
    const size_t K = (size_t)C.n;
    const size_t Kp = (K + 3) & ~(size_t)3;  // keep the Jacobian blocks 32-byte aligned
    const size_t units = (K + 31) / 32;
    // scratch: residuals and both Jacobians (9 x Kp) | (sampling mode) the drawn points and their indices
    double* d_r;
    float* d_pts;
    int32_t* d_idx;
    VGX_TRY(vgx_carve(c, c->d_scratch, vgx_part(d_r, 9 * Kp), vgx_part(d_pts, sampled ? units * VGX_PT_UNIT_FLOATS : 0),
                      vgx_part(d_idx, sampled ? Kp : 0)));
    if (sampled) {
      // cpp:118-122: every Evaluate draws its points anew from the reference submap's sampler
      VgxPoints& p = c->submaps.at(ref_id)->points[cfg->registration_point_type];
      int32_t* h_idx;
      VGX_TRY(vgx_carve(c, c->h_pinned, vgx_part(h_idx, Kp)));
      VGX_TRY(vgx_sync(c));
      vgx_points_draw(p, (int)K, h_idx);
      VGX_TRY(vgx_upload(c, d_idx, h_idx, K));
      VGX_TRY(vgx_launch_reg_gather_samples(c, p.data.get(), d_idx, (int)K, d_pts));
      C.pts = d_pts;
    }
    RegPoseConst P;
    vgx_reg_pose_setup<TrigHostLibm>(ref_pose, read_pose, P);
    double* d_jr = jac_ref ? d_r + Kp : nullptr;
    double* d_je = jac_read ? d_r + 5 * Kp : nullptr;
    {
      VgxProfileScope scope(c, VGX_SLOT_REG_EMIT);
      VGX_TRY(vgx_launch(c, reg_emit_kernel, (unsigned)((K + 255) / 256), 256, 0, VgxLaunch::plain, C, P, d_r, d_jr,
                         d_je));
    }
    VGX_TRY(vgx_download(c, residuals, d_r, K));
    if (jac_ref) VGX_TRY(vgx_download(c, jac_ref, d_jr, 4 * K));
    if (jac_read) VGX_TRY(vgx_download(c, jac_read, d_je, 4 * K));
    return vgx_sync(c);
  });
}
