// Registration kernels: emit mode (Ceres layout, boundary b1) and fused reduce mode
// (per-constraint normal-equation sums, boundary b2).  Compiled with -fmad=false.
#include "registration.cuh"
#include "registration_kernels.h"

#include <stdlib.h>
#include <string.h>

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

// Registration reduce kernel, v4.  Persistent CTAs; the local residual index space is cut into
// 32-point units that are dealt evenly to the CTAs (a tile = a CTA's run of units inside one
// residual block).  Inside a tile every warp runs its own software pipeline over the units
// u = warp, warp + W, ...:
//   * the unit's points (640 contiguous bytes of the unit-major AoSoA layout) are brought into a
//     per-warp 4-slot shared-memory ring by ONE cp.async.bulk (TMA 1-D) completing on an
//     mbarrier, three units ahead - the point loads never touch the LSU path of the math warps;
//   * stage A(u+1): transform -> voxel index -> block-grid lookup (shared memory) -> the octet's
//     two LDG.128 are ISSUED;  stage B(u): the octet issued one iteration earlier is consumed:
//     B1 coefficients, residual, Jacobian, Gram staging + 8 DMMA.  The gather latency of unit
//     u+1 is hidden behind the arithmetic of unit u inside the same warp.
// The last unit is zero-padded to 32 points (weight 0 -> zero contribution), so the
// loop carries no "active" predicate.  Warps never synchronise with each other inside a tile.
template <bool kJacobian>
__global__ void __launch_bounds__(VGX_REG_THREADS, VGX_REG_MIN_BLOCKS)
reg_reduce_kernel(const RegConstraintDev* __restrict__ constraints,
                  const RegPoseConst* __restrict__ poses, const RegTile* __restrict__ tiles,
                  const int* __restrict__ cta_tile_begin, const int* __restrict__ tile_order,
                  int* __restrict__ tile_cost, double* __restrict__ partials, int grid_capacity,
                  const int* __restrict__ skip) {
  if (skip && *skip) return;   // evaluation enqueued ahead of a solve that has already ended
  constexpr int kWarps = VGX_REG_THREADS / 32;
  constexpr int kRing = VGX_REG_RING;
  __shared__ __align__(128) float s_ring[kWarps][kRing][5][32];
  __shared__ __align__(8) unsigned long long s_bar[kWarps][kRing];
  __shared__ __align__(8) unsigned long long s_tbar;   // tile barrier: descriptor + pose block + grid
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
  int grid_of = -1;  // constraint whose block grid is currently staged

  uint32_t tseq = 0;  // tiles staged by this CTA (parity of the tile barrier)
  // one CTA per tile: CTA b runs tile_order[b] (longest-first order from the measured cost of an earlier
  // evaluation: the hardware hands CTAs out in index order, so the expensive tiles start first and the
  // tail of the grid is made of cheap ones); persistent mode: CTA b walks its run of tiles
  int tile_first, tile_end;
  if (tile_order) { tile_first = __ldg(tile_order + blockIdx.x); tile_end = tile_first + 1; }
  else { tile_first = cta_tile_begin[blockIdx.x]; tile_end = cta_tile_begin[blockIdx.x + 1]; }
  for (int tile = tile_first; tile < tile_end; ++tile, ++tseq) {
    // the 32-byte tile record is all a thread needs to start the bulk copies
    const int4 rec0 = __ldg(reinterpret_cast<const int4*>(tiles + tile));
    const ulonglong2 rec1 = __ldg(reinterpret_cast<const ulonglong2*>(tiles + tile) + 1);
    RegTile T;
    T.constraint = rec0.x; T.start = rec0.y; T.count = rec0.z; T.grid_bytes = rec0.w;
    T.pts = reinterpret_cast<const float*>(rec1.x);
    T.grid16 = reinterpret_cast<const uint16_t*>(rec1.y);
    const bool use_grid = T.grid_bytes > 0 && T.grid_bytes <= 2 * grid_capacity;
    const bool stage_grid = use_grid && grid_of != T.constraint;
    __syncthreads();  // previous tile: every warp is out of its loop (s_C / s_P / s_grid readers)
    // ---- descriptor (160 B), pose block (64 B) and the 16-bit block grid: three bulk copies on the
    //      tile barrier; the warps' first point units follow on their own barriers
    if (threadIdx.x == 0) {
      const uint32_t bytes = (uint32_t)sizeof(RegConstraintDev) + (uint32_t)sizeof(RegPoseConst) +
                             (stage_grid ? (uint32_t)T.grid_bytes : 0u);
      mbar_expect_tx(tbar, bytes);
      tma_load_1d(smem_u32(&s_C), constraints + T.constraint, (uint32_t)sizeof(RegConstraintDev), tbar);
      if (stage_grid) tma_load_1d(smem_u32(s_grid), T.grid16, (uint32_t)T.grid_bytes, tbar);
      // the pose blocks are the only input the preceding kernel (pose set-up) writes: everything
      // above was independent of it (programmatic dependent launch)
      asm volatile("griddepcontrol.wait;" ::: "memory");
      tma_load_1d(smem_u32(&s_P), poses + T.constraint, (uint32_t)sizeof(RegPoseConst), tbar);
    }
    if (stage_grid) grid_of = T.constraint;
    const int n_units = (T.count + 31) >> 5;
    const int my_units = warp < n_units ? (n_units - warp + kWarps - 1) / kWarps : 0;
    // producer (lane 0): bring unit j of this warp into ring slot seq % kRing
    auto issue = [&](int j, uint32_t seq) {
      if (lane == 0) {
        const uint32_t slot = seq % kRing;
        const uint32_t bar = bar0 + 8u * slot, dst = ring0 + 640u * slot;
        mbar_expect_tx(bar, 640u);
        tma_load_1d(dst, T.pts + (size_t)(warp + j * kWarps) * VGX_PT_UNIT_FLOATS, 640u, bar);
      }
    };
    if (my_units > 0) {
#pragma unroll
      for (int j = 0; j < kRing - 1; ++j)
        if (j < my_units) issue(j, it + j);
    }
    mbar_wait(tbar, tseq & 1u);   // descriptor, pose block and grid have landed
    const long long clk0 = clock64();
    const RegPoseConst P = s_P;
    double d0 = 0.0, d1 = 0.0;
    const size_t vox_shift = 3 * s_C.vps_shift;
    const float4* view = reinterpret_cast<const float4*>(s_C.view);

    // stage A: everything up to the ISSUE of the octet load
    struct Pipe { float4 lo, hi; float ox, oy, oz; bool found; };
    const bool gram_always = s_C.no_corr != 0.0;  // r = w * no_correspondence_cost without a match
    auto stage_a = [&](uint32_t seq, Pipe& R) {
      const uint32_t slot = seq % kRing;
      mbar_wait(bar0 + 8u * slot, (seq / kRing) & 1u);
      const float* sp = ringf + 160 * slot + lane;
      float p0, p1, p2;
      vgx_reg_transform(P, sp[0], sp[32], sp[64], p0, p1, p2);
      const float qnan = __int_as_float(0x7fc00000);
      R.lo = make_float4(qnan, qnan, qnan, qnan);
      R.hi = R.lo;
      R.found = false;
      R.ox = R.oy = R.oz = 0.f;
      int b0, b1, b2;
      vgx_block_index(s_C, p0, p1, p2, b0, b1, b2);
      RegLocate L;
      int slot_b;
      if (use_grid) {
#if VGX_REG_EARLYOUT
        // getVoxelsAndQVector fails right away when the block that contains pos does not exist;
        // overlapping submaps share only part of their surface and consecutive points are
        // spatially coherent: most warps miss with all 32 lanes and skip the rest of the unit
        const bool hit = vgx_grid_slot(s_C, s_grid, b0, b1, b2) >= 0;
        if (!__any_sync(0xffffffffu, hit)) return;
        vgx_locate_in_block<true>(s_C, p0, p1, p2, b0, b1, b2, L, s_grid);
        slot_b = hit ? L.slot : -1;
#else
        vgx_locate_in_block<true>(s_C, p0, p1, p2, b0, b1, b2, L, s_grid);
        slot_b = L.slot;
#endif
      } else {
        vgx_locate_in_block<false>(s_C, p0, p1, p2, b0, b1, b2, L);
        slot_b = vgx_resolve(s_C, L);
      }
      R.found = slot_b >= 0;
      R.ox = L.ox; R.oy = L.oy; R.oz = L.oz;
      if (R.found) {
        const float4* o = view + 2 * (((size_t)slot_b << vox_shift) + (size_t)L.lin);
        // the whole 32-byte octet = one sector = two 128-bit loads (sm_90 has no 256-bit LDG)
        R.lo = __ldg(o); R.hi = __ldg(o + 1);
      }
    };
    // stage B: consume the octet issued one unit ago
    auto stage_b = [&](uint32_t seq, const Pipe& R) {
      const float* sp = ringf + 160 * (seq % kRing) + lane;
      const float d[8] = {R.lo.x, R.lo.y, R.lo.z, R.lo.w, R.hi.x, R.hi.y, R.hi.z, R.hi.w};
#if VGX_REG_SKIPGRAM
      bool ok = false;
      if (__any_sync(0xffffffffu, R.found)) ok = R.found && vgx_octet_ok(d);
      const bool work = gram_always || __any_sync(0xffffffffu, ok);
#else
      const bool ok = R.found && vgx_octet_ok(d);
      const bool work = true;
#endif
      if (work) {
        const float xi = sp[0], yi = sp[32], dist = sp[96], w = sp[128];
        const RegPointResult Q = vgx_reg_math<kJacobian>(s_C, P, xi, yi, dist, w, ok, d, R.ox, R.oy, R.oz);
#if defined(VGX_X_NOGRAM)
        // timing ablation only (scripts/build_variants.py x_nogram): no staging, no MMA - results are wrong
        d0 = fma(Q.r, (double)Q.jr[0] + (double)Q.jr[3] + (double)Q.je3, d0);
        if (false) {
#else
        if (kJacobian) {
#endif
          stage_w[0 * VGX_STAGE_STRIDE] = (double)Q.jr[0];
          stage_w[1 * VGX_STAGE_STRIDE] = (double)Q.jr[1];
          stage_w[2 * VGX_STAGE_STRIDE] = (double)Q.jr[2];
          stage_w[3 * VGX_STAGE_STRIDE] = (double)Q.jr[3];
          stage_w[4 * VGX_STAGE_STRIDE] = (double)Q.je3;
          stage_w[5 * VGX_STAGE_STRIDE] = Q.r;
          __syncwarp();
#pragma unroll
          for (int t4 = 0; t4 < 8; ++t4) {
            const double a = (grp < 6) ? stage_r[4 * t4] : 0.0;
            dmma_8x8x4(d0, d1, a, a);
          }
        } else {
          d0 = fma(Q.r, Q.r, d0);
        }
      }
      __syncwarp();  // every lane is done with this unit's ring slot and the Gram staging buffer
    };

    if (my_units > 0) {
      // two register sets alternate (loop unrolled by two): the in-flight octet is never copied
      Pipe Ra, Rb;
      stage_a(it, Ra);
      int j = 0;
      for (; j + 2 <= my_units; j += 2, it += 2) {
        if (j + kRing - 1 < my_units) issue(j + kRing - 1, it + kRing - 1);
        stage_a(it + 1, Rb);
        stage_b(it, Ra);
        if (j + kRing < my_units) issue(j + kRing, it + kRing);
        if (j + 2 < my_units) stage_a(it + 2, Ra);
        stage_b(it + 1, Rb);
      }
      if (j < my_units) {
        stage_b(it, Ra);
        ++it;
      }
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
      if (e == 0 && tile_cost) tile_cost[tile] = (int)min(clock64() - clk0, (long long)0x3fffffff);
    }
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

void vgx_launch_reg_order(cudaStream_t st, const int* tile_cost, int n_tiles, int* tile_order) {
  if (n_tiles > 0) reg_order_kernel<<<1, 1024, 0, st>>>(tile_cost, n_tiles, tile_order);
}

__global__ void reg_pose_setup_kernel(const RegConstraintDev* __restrict__ constraints,
                                      const double* __restrict__ x, RegPoseConst* __restrict__ poses,
                                      int n_constraints, const int* __restrict__ skip) {
  // programmatic dependent launch: the reduce kernel may start its prologue (tile records, TMA of the
  // descriptors, block grids and first point units) while the pose blocks are still being computed
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  // ... and this kernel may itself have been scheduled while the previous evaluation's assembly was
  // still running: the pose blocks it overwrites were read by that evaluation's reduce kernel, which
  // has completed once the assembly (its dependent) has
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (skip && *skip) return;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_constraints) return;
  RegPoseConst P;
  vgx_reg_pose_setup<TrigDevice>(x + 4 * constraints[c].ref_node, x + 4 * constraints[c].read_node, P);
  poses[c] = P;
}

// ------------------------------------------------------------------ launch helpers
void vgx_launch_reg_pose_setup(cudaStream_t st, const RegConstraintDev* cons, const double* x,
                               RegPoseConst* poses, int n, const int* skip) {
  if (n <= 0) return;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)((n + 127) / 128));
  cfg.blockDim = dim3(128);
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  static const char* no_pdl = getenv("VGX_NO_PDL");
  cfg.attrs = attr;
  cfg.numAttrs = (no_pdl && no_pdl[0] == '1') ? 0 : 1;
  cudaLaunchKernelEx(&cfg, reg_pose_setup_kernel, cons, x, poses, n, skip);
}

void vgx_launch_reg_reduce(cudaStream_t st, const RegConstraintDev* cons, const RegPoseConst* poses,
                           const RegTile* tiles, int n_ctas, const int* cta_tile_begin,
                           const int* tile_order, int* tile_cost, double* partials, int grid_capacity,
                           bool jacobian, const int* skip) {
  if (n_ctas <= 0) return;
  // launched with programmatic stream serialisation: its CTAs may start while the pose set-up kernel
  // is still running; they block at griddepcontrol.wait before touching the pose blocks
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)n_ctas);
  cfg.blockDim = dim3(VGX_REG_THREADS);
  cfg.dynamicSmemBytes = sizeof(uint16_t) * (size_t)grid_capacity;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  static const char* no_pdl = getenv("VGX_NO_PDL");
  cfg.attrs = attr;
  cfg.numAttrs = (no_pdl && no_pdl[0] == '1') ? 0 : 1;
  if (jacobian)
    cudaLaunchKernelEx(&cfg, reg_reduce_kernel<true>, cons, poses, tiles, cta_tile_begin, tile_order, tile_cost,
                       partials, grid_capacity, skip);
  else
    cudaLaunchKernelEx(&cfg, reg_reduce_kernel<false>, cons, poses, tiles, cta_tile_begin, tile_order, tile_cost,
                       partials, grid_capacity, skip);
}

int vgx_reg_resident_ctas(int device, int grid_capacity) {
  int sms = 132, per_sm = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
  const size_t smem = sizeof(uint16_t) * (size_t)grid_capacity;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, reg_reduce_kernel<true>, VGX_REG_THREADS,
                                                    smem) != cudaSuccess || per_sm <= 0)
    per_sm = VGX_REG_MIN_BLOCKS;
  static const char* env = getenv("VGX_REG_CTAS_PER_SM");  // tuning override
  if (env && atoi(env) > 0) per_sm = atoi(env);
  return sms * per_sm;
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

void vgx_launch_reg_gather_samples(cudaStream_t st, const float* src, const int32_t* d_idx, int n,
                                   float* dst) {
  if (n <= 0) return;
  const int padded = (n + 31) & ~31;
  reg_gather_samples_kernel<<<(padded + 255) / 256, 256, 0, st>>>(src, d_idx, n, dst);
}

int vgx_fill_constraint(vgx_ctx* c, uint32_t ref_id, uint32_t read_id, const vgx_reg_config* cfg,
                        RegConstraintDev* out, bool* sampled) {
  if (!cfg) VGX_FAIL(c, VGX_ERR_INVALID, "null registration config");
  if (cfg->registration_point_type < 0 || cfg->registration_point_type > 1)
    VGX_FAIL(c, VGX_ERR_INVALID, "invalid registration_point_type");
  if (cfg->sampling_ratio != -1.0f && !(cfg->sampling_ratio >= 0.0f))
    VGX_FAIL(c, VGX_ERR_INVALID, "sampling_ratio must be -1 (all points) or >= 0");
  if (ref_id == read_id) VGX_FAIL(c, VGX_ERR_INVALID, "cannot constrain a submap to itself");
  VgxSubmap* ref = c->find(ref_id);
  VgxSubmap* rd = c->find(read_id);
  if (!ref || !rd) VGX_FAIL(c, VGX_ERR_NOT_FOUND, "registration constraint: unknown submap");
  if (!rd->finished || !rd->d_view)
    VGX_FAIL(c, VGX_ERR_INVALID, "registration constraint: reading submap is not finished");
  if (cfg->use_esdf_distance && !rd->d_view_esdf)
    VGX_FAIL(c, VGX_ERR_INVALID, "registration constraint: use_esdf_distance needs the reading submap's ESDF "
                                 "(vgx_submap_generate_esdf)");
  const VgxPoints& p = ref->points[cfg->registration_point_type];
  const bool is_sampled = cfg->sampling_ratio != -1.0f;
  RegConstraintDev C;
  C.pts = is_sampled ? nullptr : p.data;
  C.n = reg_num_residuals(p, cfg);
  C.ref_node = -1; C.read_node = -1;
  C.hash = rd->hash;
  C.view = cfg->use_esdf_distance ? rd->d_view_esdf : rd->d_view;   // cpp:133-153
  C.voxel_size = rd->voxel_size; C.voxel_size_inv = rd->voxel_size_inv;
  C.block_size = rd->block_size; C.block_size_inv = rd->block_size_inv;
  C.vps = rd->vps;
  C.grid = rd->d_grid;
  C.grid16 = rd->d_grid16;
  C.gmin0 = rd->grid_min[0]; C.gmin1 = rd->grid_min[1]; C.gmin2 = rd->grid_min[2];
  C.gd0 = rd->grid_dim[0]; C.gd1 = rd->grid_dim[1]; C.gd2 = rd->grid_dim[2];
  C.vps_shift = 0;
  while ((1 << C.vps_shift) < rd->vps) C.vps_shift++;
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
  if (!c || !cfg || !n) return VGX_ERR_INVALID;
  VgxSubmap* ref = c->find(ref_id);
  if (!ref) VGX_FAIL(c, VGX_ERR_NOT_FOUND, "vgx_reg_num_residuals: unknown submap");
  if (cfg->registration_point_type < 0 || cfg->registration_point_type > 1) return VGX_ERR_INVALID;
  if (cfg->sampling_ratio != -1.0f && !(cfg->sampling_ratio >= 0.0f)) return VGX_ERR_INVALID;
  *n = reg_num_residuals(ref->points[cfg->registration_point_type], cfg);
  return VGX_OK;
}

extern "C" int vgx_reg_eval_emit(vgx_ctx* c, uint32_t ref_id, uint32_t read_id,
                                 const vgx_reg_config* cfg, const double ref_pose[4],
                                 const double read_pose[4], double* residuals, double* jac_ref,
                                 double* jac_read) {
  if (!c || !ref_pose || !read_pose || !residuals) return VGX_ERR_INVALID;
  VGX_CUDA(c, cudaSetDevice(c->device));
  RegConstraintDev C;
  bool sampled = false;
  int rc = vgx_fill_constraint(c, ref_id, read_id, cfg, &C, &sampled);
  if (rc != VGX_OK) return rc;
  if (C.n == 0) return VGX_ZERO_WEIGHT;  // summed weight 0 -> Evaluate returns false
  if (C.factor == 0.0) return VGX_ZERO_WEIGHT;
  const size_t K = (size_t)C.n;
  const size_t Kp = (K + 3) & ~(size_t)3;  // keep the Jacobian blocks 32-byte aligned
  const size_t units = (K + 31) / 32;
  const size_t sample_bytes = sampled ? ((units * VGX_PT_UNIT_FLOATS * sizeof(float) + Kp * sizeof(int32_t) + 255) & ~(size_t)255) : 0;
  rc = c->ensure_scratch(9 * Kp * sizeof(double) + sample_bytes);
  if (rc != VGX_OK) return rc;
  if (sampled) {
    // cpp:118-122: every Evaluate draws its points anew from the reference submap's sampler
    VgxPoints& p = c->find(ref_id)->points[cfg->registration_point_type];
    rc = c->ensure_pinned(Kp * sizeof(int32_t));
    if (rc != VGX_OK) return rc;
    VGX_CUDA(c, cudaStreamSynchronize(c->stream));
    vgx_points_draw(p, (int)K, (int32_t*)c->h_pinned);
    float* d_pts = (float*)((char*)c->d_scratch + 9 * Kp * sizeof(double));
    int32_t* d_idx = (int32_t*)(d_pts + units * VGX_PT_UNIT_FLOATS);
    VGX_CUDA(c, cudaMemcpyAsync(d_idx, c->h_pinned, K * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
    vgx_launch_reg_gather_samples(c->stream, p.data, d_idx, (int)K, d_pts);
    c->launches++;
    C.pts = d_pts;
  }
  RegPoseConst P;
  vgx_reg_pose_setup<TrigHostLibm>(ref_pose, read_pose, P);
  double* d_r = (double*)c->d_scratch;
  double* d_jr = jac_ref ? d_r + Kp : nullptr;
  double* d_je = jac_read ? d_r + 5 * Kp : nullptr;
  {
    VgxLaunchScope scope(c, 1);
    reg_emit_kernel<<<(unsigned)((K + 255) / 256), 256, 0, c->stream>>>(C, P, d_r, d_jr, d_je);
  }
  VGX_CUDA(c, cudaGetLastError());
  VGX_CUDA(c, cudaMemcpyAsync(residuals, d_r, K * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  if (jac_ref)
    VGX_CUDA(c, cudaMemcpyAsync(jac_ref, d_jr, 4 * K * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  if (jac_read)
    VGX_CUDA(c, cudaMemcpyAsync(jac_read, d_je, 4 * K * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  VGX_CUDA(c, cudaStreamSynchronize(c->stream));
  return VGX_OK;
}
