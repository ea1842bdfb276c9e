// Device-resident Levenberg-Marquardt over the packed normal equations of graph.cu, with Ceres'
// default trust-region schedule, that runs one iteration ahead of the host; the dense Cholesky
// kernels behind its steps; and the edge covariances, which factor J^T J with the same kernels.
//
// Reference: voxgraph/src/backend/pose_graph.cpp:48-163 (optimize(), getEdgeCovarianceMap()),
// Ceres 1.x TrustRegionMinimizer/LevenbergMarquardtStrategy defaults (SURVEY.md A.6).
#include <math.h>
#include <stdio.h>
#include <string.h>
#include <time.h>

#include <algorithm>

#include <cooperative_groups.h>

#include "graph.h"

namespace cg = cooperative_groups;

struct LmOpts {
  int max_num_iterations;
  double parameter_tolerance, function_tolerance, gradient_tolerance;
  double max_radius, min_radius, min_relative_decrease, min_lm_diagonal, max_lm_diagonal;
  int jacobi_scaling;
};

// ------------------------------------------------------------------ kernels: LM
// Reduced, Jacobi-scaled normal matrix, lower triangle, column-major with leading
// dimension M = n + 1; row n carries the scaled gradient (forward substitution for free).
__global__ void lm_build_kernel(const double* __restrict__ packed, const int* __restrict__ red,
                                const int* __restrict__ block_nodes, int N, int E, int n,
                                double* __restrict__ A, double* __restrict__ scale,
                                double* __restrict__ diag, double* __restrict__ gs,
                                LmState* __restrict__ st, LmOpts o) {
  if (st->done) return;   // an iteration enqueued ahead of the host's look at the previous one
  const int M = n + 1;
  const double* g = packed + PACK_HDR;
  const double* D = packed + PACK_HDR + 4 * (size_t)N;
  const double* O = D + 16 * (size_t)N;
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  const int stride = gridDim.x * blockDim.x;
  const bool first = st->scale_ready == 0;
  const bool reuse = st->reuse_diagonal != 0;
  const double radius = st->radius;
  // scale from the first Jacobian's column norms (TrustRegionMinimizer, iteration 0)
  auto sc = [&](int node, int k) -> double {
    if (!o.jacobi_scaling) return 1.0;
    if (first) return 1.0 / (1.0 + sqrt(D[16 * (size_t)node + 5 * k]));
    return scale[red[node] + k];
  };
  // diagonal blocks
  for (int t = tid; t < N * 16; t += stride) {
    const int node = t >> 4, r = (t >> 2) & 3, c = t & 3;
    const int off = red[node];
    if (off < 0 || r < c) continue;
    const double sr = sc(node, r), scc = sc(node, c);
    double v = sr * scc * D[16 * (size_t)node + 4 * r + c];
    if (r == c) {
      double d;
      if (reuse) d = diag[off + r];
      else d = fmin(fmax(v, o.min_lm_diagonal), o.max_lm_diagonal);
      // lm_diagonal = sqrt(diag / radius); added squared
      const double lm = sqrt(d / radius);
      v += lm * lm;
    }
    A[(size_t)(off + c) * M + off + r] = v;
  }
  // off-diagonal blocks: rows = node i (smaller index), cols = node j
  for (int t = tid; t < E * 16; t += stride) {
    const int b = t >> 4, r = (t >> 2) & 3, c = t & 3;
    const int ni = block_nodes[2 * b], nj = block_nodes[2 * b + 1];
    const int oi = red[ni], oj = red[nj];
    if (oi < 0 || oj < 0) continue;
    const double v = sc(ni, r) * sc(nj, c) * O[16 * (size_t)b + 4 * r + c];
    // lower triangle: row index must be the larger one (oj > oi because nj > ni)
    A[(size_t)(oi + r) * M + (oj + c)] = v;
  }
  // gradient row + bookkeeping vectors
  for (int t = tid; t < N * 4; t += stride) {
    const int node = t >> 2, k = t & 3;
    const int off = red[node];
    if (off < 0) continue;
    const double s = sc(node, k);
    const double gsv = s * g[4 * node + k];
    A[(size_t)(off + k) * M + n] = gsv;
    gs[off + k] = gsv;
  }
}

// Second pass (after lm_build): persist scale / diag. Separate so every thread of
// lm_build sees the old values.
__global__ void lm_persist_kernel(const double* __restrict__ packed, const int* __restrict__ red,
                                  int N, double* __restrict__ scale, double* __restrict__ diag,
                                  LmState* __restrict__ st, LmOpts o) {
  if (st->done) return;
  const double* D = packed + PACK_HDR + 4 * (size_t)N;
  const bool first = st->scale_ready == 0;
  const bool reuse = st->reuse_diagonal != 0;
  for (int t = threadIdx.x; t < N * 4; t += blockDim.x) {
    const int node = t >> 2, k = t & 3;
    const int off = red[node];
    if (off < 0) continue;
    double s = 1.0;
    if (o.jacobi_scaling) s = first ? 1.0 / (1.0 + sqrt(D[16 * (size_t)node + 5 * k])) : scale[off + k];
    if (first) scale[off + k] = s;
    if (!reuse) {
      const double v = s * s * D[16 * (size_t)node + 5 * k];
      diag[off + k] = fmin(fmax(v, o.min_lm_diagonal), o.max_lm_diagonal);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) st->scale_ready = 1;
}

// 1/sqrt(d) to double precision from the float MUFU seed + Newton (the fp64 sqrt/div
// routines cost several hundred cycles each on the serial pivot path).
__device__ __forceinline__ double fast_rsqrt(double d) {
  // rsqrtf is good to ~2^-22; each Newton step squares the error: two steps reach double precision
  double r = (double)rsqrtf((float)d);
  const double hd = -0.5 * d;
#pragma unroll
  for (int it = 0; it < 3; ++it) r = r * fma(hd, r * r, 1.5);
  return r;
}

// Small systems (n <= ~230, i.e. BASELINE configs[0..1]): the whole packed lower triangle of
// the (n+1) x (n+1) augmented matrix lives in shared memory; one CTA factors it column by
// column (pivot via fast_rsqrt, warps over trailing columns, lanes over rows), the rhs row
// gives the forward substitution for free, then the back substitution writes x = (L L^T)^-1 g.
__device__ __forceinline__ int tri_off(int j, int M) { return j * M - (j * (j - 1)) / 2; }

__device__ __forceinline__ void dmma_sub_8x8x4(double& c0, double& c1, double a, double b) {
  // C += A * B on the FP64 tensor core (callers negate)
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

// Left-looking, panel width 8: (1) the block column is updated with all previous columns by
// m8n8k4 FP64 MMAs (warps over 8-row tiles), (2) warp 0 factors the 8x8 diagonal block,
// (3) one thread per row solves the panel.  Then back substitution in place.
#define CS_NB 8
__global__ void __launch_bounds__(512)
chol_solve_smem_kernel(const double* __restrict__ A, int n, double* __restrict__ xsol,
                       LmState* __restrict__ st, const int* __restrict__ red,
                       const int* __restrict__ block_nodes, int N, int E, long long* __restrict__ dbg) {
  extern __shared__ double S[];  // packed columns: column j holds rows j..n
  __shared__ int s_fail;
  if (st->done) return;
  const int M = n + 1;
  const int tid = threadIdx.x, T = blockDim.x, lane = tid & 31, warp = tid >> 5, nw = T >> 5;
  const int g = lane >> 2, t = lane & 3;
  double* rinv = S + tri_off(M, M);  // n reciprocals of the diagonal of L
  if (tid == 0) s_fail = 0;
  long long tk0 = clock64(), tk_upd = 0, tk_fac = 0;   // phase cycles (thread 0, VGX_CHOL_DEBUG=1)
  // Only the 4x4 blocks lm_build wrote are read (N diagonal, E off-diagonal, the gradient row):
  // ~5 k loads instead of the dense (n+1)^2, and the matrix in global memory needs no clearing.
  for (int i = tid; i < tri_off(M, M); i += T) S[i] = 0.0;
  __syncthreads();
  for (int t0 = tid; t0 < N * 16; t0 += T) {
    const int node = t0 >> 4, r = (t0 >> 2) & 3, c = t0 & 3;
    const int off = red[node];
    if (off < 0 || r < c) continue;
    S[tri_off(off + c, M) + (r - c)] = A[(size_t)(off + c) * M + off + r];
  }
  for (int t0 = tid; t0 < E * 16; t0 += T) {
    const int b = t0 >> 4, r = (t0 >> 2) & 3, c = t0 & 3;
    const int oi = red[block_nodes[2 * b]], oj = red[block_nodes[2 * b + 1]];
    if (oi < 0 || oj < 0) continue;
    S[tri_off(oi + r, M) + (oj + c) - (oi + r)] = A[(size_t)(oi + r) * M + (oj + c)];
  }
  for (int k = tid; k < n; k += T) S[tri_off(k, M) + n - k] = A[(size_t)k * M + n];
  __syncthreads();
  const long long tk_load = clock64() - tk0;
  for (int J0 = 0; J0 < n; J0 += CS_NB) {
    const int nb = min(CS_NB, n - J0);
    const long long tp0 = clock64();
    // (1) A[J0.., J0..J0+8) -= L[J0.., 0..J0) * L[J0..J0+8, 0..J0)^T
    if (J0 > 0) {
      const int ntiles = (M - J0 + 7) >> 3;
      for (int tile = warp; tile < ntiles; tile += nw) {
        const int i0 = J0 + 8 * tile;
        const int ra = i0 + g;        // row of this lane's A fragment element
        const int rb = J0 + g;        // row (= column of the block) of its B fragment element
        // four independent accumulator pairs: the k-loop is a chain of dependent MMAs otherwise
        double c0 = 0.0, c1 = 0.0, e0 = 0.0, e1 = 0.0, f0 = 0.0, f1 = 0.0, h0 = 0.0, h1 = 0.0;
        const bool va = ra < M, vb = rb < n;
        int k0 = 0;
        for (; k0 + 16 <= J0; k0 += 16) {
          const int kc = k0 + t;      // J0 is a multiple of 8, so every kc below is < J0
          const int o0 = tri_off(kc, M) - kc, o1 = tri_off(kc + 4, M) - (kc + 4),
                    o2 = tri_off(kc + 8, M) - (kc + 8), o3 = tri_off(kc + 12, M) - (kc + 12);
          const double a0 = va ? S[o0 + ra] : 0.0, b0 = vb ? S[o0 + rb] : 0.0;
          const double a1 = va ? S[o1 + ra] : 0.0, b1 = vb ? S[o1 + rb] : 0.0;
          const double a2 = va ? S[o2 + ra] : 0.0, b2 = vb ? S[o2 + rb] : 0.0;
          const double a3 = va ? S[o3 + ra] : 0.0, b3 = vb ? S[o3 + rb] : 0.0;
          dmma_sub_8x8x4(c0, c1, a0, b0);
          dmma_sub_8x8x4(e0, e1, a1, b1);
          dmma_sub_8x8x4(f0, f1, a2, b2);
          dmma_sub_8x8x4(h0, h1, a3, b3);
        }
        for (; k0 < J0; k0 += 4) {
          const int kc = k0 + t;
          const int ok = tri_off(kc, M) - kc;
          const double a = va ? S[ok + ra] : 0.0;
          const double b = vb ? S[ok + rb] : 0.0;
          dmma_sub_8x8x4(c0, c1, a, b);
        }
        c0 = (c0 + e0) + (f0 + h0);
        c1 = (c1 + e1) + (f1 + h1);
        // lane holds C[g][2t], C[g][2t+1] -> element (row i0+g, col J0+2t(+1)), lower part only
        const int r = i0 + g;
        if (r < M) {
          const int cA = J0 + 2 * t, cB = cA + 1;
          if (cA < n && cA < J0 + nb && r >= cA) S[tri_off(cA, M) + r - cA] -= c0;
          if (cB < n && cB < J0 + nb && r >= cB) S[tri_off(cB, M) + r - cB] -= c1;
        }
      }
    }
    __syncthreads();
    const long long tp1 = clock64();
    tk_upd += tp1 - tp0;
    // (2)+(3) EVERY thread factors the 8x8 diagonal block redundantly in registers - no serial warp,
    // no shuffles on the pivot chain (chain per column: rsqrt, mul, fma) - and then forward-substitutes
    // its own row (thread t owns row J0 + t; the block's own rows come out of the same recurrence,
    // restricted to the lower triangle, bit-identical to the register factor).
    {
      const int r = J0 + tid;
      const int i = tid;            // row inside / below the block
      const bool act = r < M;
      double Lb[CS_NB][CS_NB], x[CS_NB], ri[CS_NB];
#pragma unroll
      for (int c = 0; c < CS_NB; ++c) {
#pragma unroll
        for (int q = 0; q < CS_NB; ++q)
          if (q >= c) Lb[q][c] = (q < nb && c < nb) ? S[tri_off(J0 + c, M) + q - c] : (q == c ? 1.0 : 0.0);
        x[c] = (act && c < nb && (i >= nb || c <= i)) ? S[tri_off(J0 + c, M) + r - (J0 + c)] : 0.0;
      }
      __syncthreads();   // every thread has read the unfactored block before any row is written back
      bool bad = false;
      // only the warps that own a row run the recurrence (the FP64 pipe of the one SM is the limiter:
      // 16 redundant copies cost more than the chain itself)
      if (tid < ((M - J0 + 31) & ~31)) {
#pragma unroll
      for (int k = 0; k < CS_NB; ++k) {
        double d = Lb[k][k];
        if (k < nb && (!(d > 0.0) || !isfinite(d))) { bad = true; d = 1.0; }
        const double rs = fast_rsqrt(d);
        ri[k] = rs;
        Lb[k][k] = d * rs;
#pragma unroll
        for (int q = k + 1; q < CS_NB; ++q) Lb[q][k] *= rs;
#pragma unroll
        for (int c = k + 1; c < CS_NB; ++c)
#pragma unroll
          for (int q = c; q < CS_NB; ++q) Lb[q][c] = fma(-Lb[q][k], Lb[c][k], Lb[q][c]);
      }
#pragma unroll
      for (int c = 0; c < CS_NB; ++c) {
        double v = x[c];
#pragma unroll
        for (int k = 0; k < CS_NB; ++k)
          if (k < c) v = fma(-x[k], Lb[c][k], v);
        x[c] = v * ri[c];
      }
      }
      if (act) {
#pragma unroll
        for (int c = 0; c < CS_NB; ++c)
          if (c < nb && (i >= nb || c <= i)) S[tri_off(J0 + c, M) + r - (J0 + c)] = x[c];
      }
      if (tid == 0) {
#pragma unroll
        for (int k = 0; k < CS_NB; ++k)
          if (k < nb) rinv[J0 + k] = ri[k];
        if (bad) s_fail = 1;
      }
    }
    __syncthreads();
    tk_fac += clock64() - tp1;
  }
  const long long tk_back0 = clock64();
  // back substitution L^T x = y (y = row n of L, element n of each column): ONE warp, y in
  // registers (lane l owns unknowns l, l + 32, ...).  Step j: the owner scales its y_j, one shuffle
  // broadcasts x_j, every lane folds it into its remaining unknowns with loads that do not depend
  // on the chain - n steps of (FMA, MUL, SHFL) instead of n/8 block steps with barriers.
  constexpr int kSlots = 8;   // n <= 256 (the shared-memory variant holds ~230 unknowns)
  if (warp == 0) {
    double y[kSlots];
    int base[kSlots];
#pragma unroll
    for (int m = 0; m < kSlots; ++m) {
      const int i = lane + 32 * m;
      base[m] = i < n ? tri_off(i, M) - i : 0;
      y[m] = i < n ? S[base[m] + n] : 0.0;
    }
#pragma unroll
    for (int m = kSlots - 1; m >= 0; --m) {
      if (32 * m < n) {   // warp-uniform
        for (int l = min(31, n - 1 - 32 * m); l >= 0; --l) {
          const int j = 32 * m + l;
          const double xj = __shfl_sync(0xffffffffu, y[m] * rinv[j], l);
          if (lane == l) y[m] = xj;
#pragma unroll
          for (int mm = 0; mm <= m; ++mm) {
            const int i = lane + 32 * mm;
            if (i < j) y[mm] = fma(-S[base[mm] + j], xj, y[mm]);
          }
        }
      }
    }
#pragma unroll
    for (int m = 0; m < kSlots; ++m) {
      const int i = lane + 32 * m;
      if (i < n) xsol[i] = y[m];
    }
  }
  if (tid == 0 && s_fail) st->step_valid = 0;
  if (dbg && tid == 0) {
    dbg[0] = tk_load; dbg[1] = tk_upd; dbg[2] = tk_fac; dbg[3] = clock64() - tk_back0; dbg[4] = clock64() - tk0;
  }
}

// Blocked right-looking Cholesky of the (n+1) x (n+1) lower-triangular system on a cooperative
// grid (grid-wide barriers): every CTA factors the 32x32 diagonal block redundantly in shared
// memory (deterministic, saves a barrier), the panel rows and the 32x32 trailing tiles are spread
// over the grid.  Two grid syncs per panel.
// A pivot d_k fails when !(d_k > 0); with diag0 (the unfactored diagonal, covariances only) it also
// fails when d_k <= rank_tol * diag0[k] (see VGX_COV_RANK_TOL).
#define CH_NB 32
__global__ void __launch_bounds__(256) chol_coop_kernel(double* __restrict__ A, int n,
                                                        LmState* __restrict__ st,
                                                        const double* __restrict__ diag0, double rank_tol) {
  cg::grid_group grid = cg::this_grid();
  if (st->done) return;   // uniform over the grid
  __shared__ double sD[CH_NB * 33];
  __shared__ double sPi[CH_NB * 33];
  __shared__ double sPj[CH_NB * 33];
  __shared__ double sDinv[CH_NB];
  __shared__ int s_fail;
  const int M = n + 1;
  const int tid = threadIdx.x, T = blockDim.x;
  const int gsize = gridDim.x * T, gid = blockIdx.x * T + tid;
  if (tid == 0) s_fail = 0;
  __syncthreads();
  for (int j0 = 0; j0 < n; j0 += CH_NB) {
    const int nb = min(CH_NB, n - j0);
    for (int t = tid; t < nb * nb; t += T) {
      const int r = t % nb, c = t / nb;
      if (r >= c) sD[r * 33 + c] = A[(size_t)(j0 + c) * M + j0 + r];
    }
    __syncthreads();
    if (tid < 32) {
      const int r = tid;
      for (int k = 0; k < nb; ++k) {
        double d = sD[k * 33 + k];
        const double floor_k = diag0 ? rank_tol * diag0[j0 + k] : 0.0;
        if (!(d > floor_k) || !isfinite(d)) { if (r == 0) s_fail = 1; d = 1.0; }
        const double rs = fast_rsqrt(d);
        __syncwarp();
        if (r == k) { sD[k * 33 + k] = d * rs; sDinv[k] = rs; }
        if (r > k && r < nb) sD[r * 33 + k] *= rs;
        __syncwarp();
        if (r > k && r < nb) {
          const double lrk = sD[r * 33 + k];
          for (int c = k + 1; c <= r; ++c) sD[r * 33 + c] -= lrk * sD[c * 33 + k];
        }
        __syncwarp();
      }
    }
    __syncthreads();
    if (blockIdx.x == 0)
      for (int t = tid; t < nb * nb; t += T) {
        const int r = t % nb, c = t / nb;
        if (r >= c) A[(size_t)(j0 + c) * M + j0 + r] = sD[r * 33 + c];
      }
    // panel solve: one thread of the grid per row below the block (incl. the rhs row n)
    const int r0 = j0 + nb;
    const int rows = M - r0;
    for (int rr = gid; rr < rows; rr += gsize) {
      double x[CH_NB];
#pragma unroll
      for (int c = 0; c < CH_NB; ++c) {
        if (c < nb) {
          double v = A[(size_t)(j0 + c) * M + r0 + rr];
#pragma unroll
          for (int k = 0; k < CH_NB; ++k)
            if (k < c) v -= x[k] * sD[c * 33 + k];
          v *= sDinv[c];
          x[c] = v;
          A[(size_t)(j0 + c) * M + r0 + rr] = v;
        }
      }
    }
    grid.sync();
    // trailing update over 32x32 tiles (bi >= bj) of rows/cols [r0, M) x [r0, n)
    const int tc = n - r0;
    if (tc > 0) {
      const int ntr = (rows + CH_NB - 1) / CH_NB;   // tile rows (incl. rhs row)
      const int ntc = (tc + CH_NB - 1) / CH_NB;     // tile cols
      for (int tile = blockIdx.x; tile < ntr * ntc; tile += gridDim.x) {
        const int bi = tile / ntc, bj = tile % ntc;
        if (bi < bj) continue;
        __syncthreads();
        for (int t = tid; t < CH_NB * CH_NB; t += T) {
          const int r = t % CH_NB, k = t / CH_NB;
          const int ri = bi * CH_NB + r, rj = bj * CH_NB + r;
          sPi[r * 33 + k] = (ri < rows) ? A[(size_t)(j0 + k) * M + r0 + ri] : 0.0;
          sPj[r * 33 + k] = (rj < rows) ? A[(size_t)(j0 + k) * M + r0 + rj] : 0.0;
        }
        __syncthreads();
        // 256 threads x 4 outputs: thread owns column cj = tid / 8, rows (tid % 8) + 8 * q
        const int cj = tid >> 3, rb = tid & 7;
        double acc[4] = {0, 0, 0, 0};
#pragma unroll 8
        for (int k = 0; k < CH_NB; ++k) {
          const double pj = sPj[cj * 33 + k];
#pragma unroll
          for (int q = 0; q < 4; ++q) acc[q] = fma(sPi[(rb + 8 * q) * 33 + k], pj, acc[q]);
        }
        const int gc = bj * CH_NB + cj;
        if (gc < tc) {
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int gr = bi * CH_NB + rb + 8 * q;
            if (gr < rows && gr >= gc) A[(size_t)(r0 + gc) * M + r0 + gr] -= acc[q];
          }
        }
      }
    }
    grid.sync();
  }
  if (blockIdx.x == 0 && tid == 0 && s_fail) st->step_valid = 0;
}

// Back substitution L^T x = y (y = row n of L), step = -x, model cost change, candidate.
__global__ void __launch_bounds__(1024)
lm_step_kernel(const double* __restrict__ A, int n, int N, const int* __restrict__ red,
               const double* __restrict__ scale, const double* __restrict__ diag,
               const double* __restrict__ gs, const double* __restrict__ x,
               double* __restrict__ xc, double* __restrict__ step, LmState* __restrict__ st,
               const double* __restrict__ presolved) {
  extern __shared__ double sy[];  // n
  __shared__ double s_red[3][32];
  if (st->done) return;
  const int M = n + 1;
  const int tid = threadIdx.x, T = blockDim.x, lane = tid & 31, warp = tid >> 5, nw = T >> 5;
  for (int i = tid; i < n; i += T) sy[i] = presolved ? presolved[i] : A[(size_t)i * M + n];
  __syncthreads();
  const int nblk = presolved ? 0 : (n + CH_NB - 1) / CH_NB;
  for (int b = nblk - 1; b >= 0; --b) {
    const int j0 = b * CH_NB, nb = min(CH_NB, n - j0);
    // solve the nb x nb upper-triangular block (warp 0)
    if (warp == 0) {
      for (int k = nb - 1; k >= 0; --k) {
        const double xk = sy[j0 + k] / A[(size_t)(j0 + k) * M + j0 + k];
        __syncwarp();
        if (lane == 0) sy[j0 + k] = xk;
        if (lane < k) sy[j0 + lane] -= A[(size_t)(j0 + lane) * M + j0 + k] * xk;
        __syncwarp();
      }
    }
    __syncthreads();
    // y_i -= sum_k L[j0+k][i] x_k for i < j0: one warp per column i, lanes over k
    for (int i = warp; i < j0; i += nw) {
      double v = (lane < nb) ? A[(size_t)i * M + j0 + lane] * sy[j0 + lane] : 0.0;
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
      if (lane == 0) sy[i] -= v;
    }
    __syncthreads();
  }
  // step = -x ; model_cost_change = 1/2 sum x_i (gs_i + D_i x_i), D = diag / radius
  const double radius = st->radius;
  double mcc = 0;
  int bad = 0;
  for (int i = tid; i < n; i += T) {
    const double xi = sy[i];
    if (!isfinite(xi)) bad = 1;
    step[i] = -xi;
    mcc += 0.5 * xi * (gs[i] + (diag[i] / radius) * xi);
  }
  // candidate = Plus(x, step .* scale)
  double sn2 = 0, xn2 = 0;
  for (int t = tid; t < 4 * N; t += T) {
    const int node = t >> 2, k = t & 3;
    const int off = red[node];
    const double xv = x[t];
    double cv = xv;
    if (off >= 0) {
      const double d = -sy[off + k] * scale[off + k];
      cv = (k == 3) ? normalize_angle(xv + d) : xv + d;
      const double dd = xv - cv;
      sn2 += dd * dd;
      xn2 += xv * xv;
    }
    xc[t] = cv;
  }
  // block reduce (fixed order)
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    mcc += __shfl_xor_sync(0xffffffffu, mcc, off);
    sn2 += __shfl_xor_sync(0xffffffffu, sn2, off);
    xn2 += __shfl_xor_sync(0xffffffffu, xn2, off);
    bad |= __shfl_xor_sync(0xffffffffu, bad, off);
  }
  __shared__ int s_bad;
  if (tid == 0) s_bad = 0;
  __syncthreads();
  if (lane == 0) { s_red[0][warp] = mcc; s_red[1][warp] = sn2; s_red[2][warp] = xn2; if (bad) atomicOr(&s_bad, 1); }
  __syncthreads();
  if (tid == 0) {
    double a = 0, b2 = 0, c2 = 0;
    for (int w = 0; w < nw; ++w) { a += s_red[0][w]; b2 += s_red[1][w]; c2 += s_red[2][w]; }
    st->model_cost_change = a;
    st->step_norm = sqrt(b2);
    st->x_norm = sqrt(c2);
    if (s_bad || !(a > 0.0)) st->step_valid = 0;
  }
}

// max |g_k| over the free parameters of the packed gradient: warp shuffles, then the warps' maxima in
// warp order.  The result is valid in thread 0.
__device__ __forceinline__ double free_gradient_max_norm(const double* __restrict__ packed,
                                                         const int* __restrict__ red, int N) {
  __shared__ double s_g[32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double gm = 0;
  for (int t = tid; t < 4 * N; t += blockDim.x)
    if (red[t >> 2] >= 0) gm = fmax(gm, fabs(packed[PACK_HDR + t]));
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) gm = fmax(gm, __shfl_xor_sync(0xffffffffu, gm, off));
  if (lane == 0) s_g[warp] = gm;
  __syncthreads();
  gm = 0;
  if (tid == 0)
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) gm = fmax(gm, s_g[w]);
  return gm;
}

// Accept / reject and termination tests of TrustRegionMinimizer (A.6).
__global__ void lm_decide_kernel(const double* __restrict__ packed_cur,
                                 const double* __restrict__ packed_cand,
                                 const int* __restrict__ red, int N, double* __restrict__ x,
                                 const double* __restrict__ xc, LmState* __restrict__ st, LmOpts o,
                                 int cand_eval_ok, LmState* __restrict__ snapshot) {
  if (st->done) {   // no-op iteration: the snapshot still tells the host the solve has ended
    if (threadIdx.x == 0) *snapshot = *st;
    return;
  }
  const int tid = threadIdx.x;
  const double gm = free_gradient_max_norm(packed_cand, red, N);   // at the candidate (used if accepted)
  __shared__ int s_accept;
  if (tid == 0) {
    LmState S = *st;
    S.accepted = 0;
    S.iterations++;
    const double cost = packed_cur[0];
    const double cand = packed_cand[0];
    S.cost = cost;
    S.cand_cost = cand;
    bool invalid = (S.step_valid == 0);
    if (!invalid) { S.evals++; if (!cand_eval_ok) invalid = true; }
    if (invalid) {
      // HandleInvalidStep
      if (++S.consecutive_invalid >= 5) { S.termination = 6; S.done = 1; }
      S.radius /= S.decrease_factor; S.decrease_factor *= 2; S.reuse_diagonal = 1;
    } else {
      S.consecutive_invalid = 0;
      if (S.step_norm <= o.parameter_tolerance * (S.x_norm + o.parameter_tolerance)) {
        S.termination = 0; S.done = 1;  // ParameterToleranceReached (x is not updated)
      } else {
        const double cost_change = cost - cand;
        if (fabs(cost_change) <= o.function_tolerance * cost) {
          S.termination = 1; S.done = 1;  // FunctionToleranceReached
        } else {
          const double rel = cost_change / S.model_cost_change;
          if (rel > o.min_relative_decrease) {
            S.accepted = 1; S.successful++;
            S.cost = cand;
            S.gmax = gm;
            const double q = 2.0 * rel - 1.0;
            S.radius = S.radius / fmax(1.0 / 3.0, 1.0 - q * q * q);
            S.radius = fmin(o.max_radius, S.radius);
            S.decrease_factor = 2.0; S.reuse_diagonal = 0;
          } else {
            S.radius /= S.decrease_factor; S.decrease_factor *= 2; S.reuse_diagonal = 1;
          }
        }
      }
    }
    if (!S.done) {
      // FinalizeIterationAndCheckIfMinimizerCanContinue for the next iteration
      if (S.iterations >= o.max_num_iterations) { S.termination = 3; S.done = 1; }
      else if (S.gmax <= o.gradient_tolerance) { S.termination = 2; S.done = 1; }
      else if (S.radius <= o.min_radius) { S.termination = 5; S.done = 1; }
    }
    S.step_valid = 1;
    s_accept = S.accepted;
    *st = S;
    *snapshot = S;   // what the host reads (the live state is rewritten by the next iteration's kernels)
  }
  __syncthreads();
  if (s_accept)
    for (int t = tid; t < 4 * N; t += blockDim.x) x[t] = xc[t];
}

// The candidate's normal equations become the current ones when the step was accepted (slot 1 ->
// slot 0), so every kernel of an iteration has fixed arguments whatever the decisions were.
__global__ void lm_accept_kernel(const double* __restrict__ cand, double* __restrict__ cur, size_t len,
                                 const LmState* __restrict__ st) {
  if (!st->accepted) return;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < len; i += (size_t)gridDim.x * blockDim.x)
    cur[i] = cand[i];
}

__global__ void lm_init_kernel(const double* __restrict__ packed, const int* __restrict__ red, int N,
                               LmState* __restrict__ st, double radius, LmOpts o) {
  const double gm = free_gradient_max_norm(packed, red, N);
  if (threadIdx.x == 0) {
    LmState S;
    memset(&S, 0, sizeof(S));
    S.radius = radius; S.decrease_factor = 2.0;
    S.cost = packed[0];
    S.gmax = gm;
    S.evals = 1;
    S.step_valid = 1;
    S.termination = 3;
    if (o.max_num_iterations <= 0) { S.termination = 3; S.done = 1; }
    else if (gm <= o.gradient_tolerance) { S.termination = 2; S.done = 1; }
    *st = S;
  }
}

// ------------------------------------------------------------------ dense solve dispatch
// Which Cholesky factors an n-unknown system (n > 0).  smem_ok (the LM): chol_solve_smem_kernel, which
// factors and solves the whole packed system in one CTA's shared memory, when it fits; *smem_bytes is
// then its dynamic shared memory.  Otherwise, and always for the covariances, which need L itself:
// chol_coop_kernel on *coop_grid co-resident CTAs.
static int chol_dispatch(vgx_ctx* c, int n, bool smem_ok, size_t* smem_bytes, int* coop_grid) {
  *smem_bytes = 0;
  *coop_grid = 0;
  const size_t smem_chol_bytes = sizeof(double) * ((size_t)(n + 1) * (n + 2) / 2 + n + 2);
  const bool use_smem_chol = n > 0 && n <= 256 && smem_chol_bytes <= 220 * 1024;
  if (smem_ok && use_smem_chol) {
    VGX_CUDA(c, cudaFuncSetAttribute(chol_solve_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)smem_chol_bytes));
    *smem_bytes = smem_chol_bytes;
    return VGX_OK;
  }
  int coop = 0, sms = 0, per_sm = 0;
  cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, c->device);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device);
  if (!coop)
    VGX_FAIL(c, VGX_ERR_CAPACITY, "dense pose-graph Cholesky: the device does not support cooperative launches");
  VGX_CUDA(c, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, chol_coop_kernel, 256, 0));
  if (per_sm == 0)
    VGX_FAIL(c, VGX_ERR_CAPACITY, "dense pose-graph Cholesky: chol_coop_kernel cannot be resident on this device");
  const int tiles = ((n + 1 + CH_NB - 1) / CH_NB) * ((n + CH_NB - 1) / CH_NB);
  *coop_grid = std::max(1, std::min(sms * std::min(per_sm, 2), std::max(tiles / 2, (n + 256) / 256)));
  return VGX_OK;
}

static cudaError_t launch_chol_coop(cudaStream_t st, int grid, double* A, int n, LmState* state,
                                    const double* diag0, double rank_tol) {
  void* args[] = {(void*)&A, (void*)&n, (void*)&state, (void*)&diag0, (void*)&rank_tol};
  return cudaLaunchCooperativeKernel((void*)chol_coop_kernel, dim3(grid), dim3(256), args, 0, st);
}

// lm_build_kernel + lm_persist_kernel on the normal equations in d_packed[0]
static void enqueue_lm_build(cudaStream_t st, VgxGraph* g, int n, const LmOpts& lo) {
  const int N = g->N;
  const int nthreads = std::max(16 * (N + g->E), 4 * N);
  lm_build_kernel<<<std::min(296, (nthreads + 255) / 256), 256, 0, st>>>(
      g->d_packed[0], g->d_red_offset, g->d_block_nodes, N, g->E, n, g->d_A, g->d_scale, g->d_diag,
      g->d_gs, g->d_state, lo);
  lm_persist_kernel<<<1, 256, 0, st>>>(g->d_packed[0], g->d_red_offset, N, g->d_scale, g->d_diag,
                                       g->d_state, lo);
}

// ------------------------------------------------------------------ edge covariances
// PoseGraph::getEdgeCovarianceMap (pose_graph.cpp:117-163): ceres::Covariance blocks
// Cov(x_a, x_b) = rows of a, columns of b of (J^T J)^-1 over the free parameter blocks at the current
// poses (no LM damping, no Jacobi scaling, no loss function); constant blocks have zero covariance.
// Dense reduced H -> chol_coop_kernel -> two triangular solves per requested column.
//
// ceres::Covariance::Compute returns false when J^T J is rank deficient.  A plain sign test on the
// pivots cannot decide that: on a graph without a constant node (a 4-dimensional gauge null space)
// the null-space pivots come out within ~1e-14 of 0 relative to their diagonal, with either sign,
// so the result would be the error or finite covariances of ~1e14 depending on rounding.  A pivot
// d_k <= VGX_COV_RANK_TOL * H_kk is therefore taken as rank deficient.  1e-10 lies 4 orders above
// that rounding noise and 7 below the smallest relative pivot of anchored chains (4e-3 for
// 64..250-node chains with condition numbers up to 4e8; tests/test_host_dense_solve.py checks both
// margins).  It approximates Ceres' rank decision (SPARSE_QR's) rather than restating it.
#define VGX_COV_RANK_TOL 1e-10
// one CTA per requested column c: x = (L L^T)^-1 e_c.  L: lower, column-major, leading dimension n+1.
__global__ void __launch_bounds__(256)
cov_column_kernel(const double* __restrict__ A, int n, const int* __restrict__ cols, double* __restrict__ X) {
  extern __shared__ double sx[];   // n
  __shared__ double s_red[8];
  const int M = n + 1, c = cols[blockIdx.x];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < n; i += blockDim.x) sx[i] = (i == c) ? 1.0 : 0.0;
  __syncthreads();
  // forward: L y = e_c (y_i = 0 for i < c)
  for (int i = c; i < n; ++i) {
    double acc = 0;
    for (int k = c + tid; k < i; k += blockDim.x) acc += A[(size_t)k * M + i] * sx[k];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if (lane == 0) s_red[warp] = acc;
    __syncthreads();
    if (tid == 0) {
      double t = 0;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += s_red[w];
      sx[i] = (sx[i] - t) / A[(size_t)i * M + i];
    }
    __syncthreads();
  }
  // backward: L^T x = y
  for (int i = n - 1; i >= 0; --i) {
    double acc = 0;
    for (int k = i + 1 + tid; k < n; k += blockDim.x) acc += A[(size_t)i * M + k] * sx[k];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if (lane == 0) s_red[warp] = acc;
    __syncthreads();
    if (tid == 0) {
      double t = 0;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += s_red[w];
      sx[i] = (sx[i] - t) / A[(size_t)i * M + i];
    }
    __syncthreads();
  }
  for (int i = tid; i < n; i += blockDim.x) X[(size_t)blockIdx.x * n + i] = sx[i];
}

extern "C" int vgx_graph_edge_covariances(vgx_ctx* c, int m, const uint32_t* ids_a, const uint32_t* ids_b,
                                          double* cov) {
  VgxGraph* g = nullptr;
  int rc = prepare(c, &g);
  if (rc != VGX_OK) return rc;
  if (m < 0 || (m > 0 && (!ids_a || !ids_b || !cov))) return VGX_ERR_INVALID;
  if (m == 0) return VGX_OK;
  if (g->zero_weight) VGX_FAIL(c, VGX_ZERO_WEIGHT, "a registration constraint has zero summed weight (Evaluate == false)");
  const int N = g->N, n = g->n_free;
  const std::vector<int>& red = g->red;
  // distinct columns: the 4 parameters of every second node that is free
  std::vector<int> col_of(N, -1), cols;
  std::vector<std::pair<int, int>> pr(m);
  for (int k = 0; k < m; ++k) {
    auto ia = g->index.find(ids_a[k]);
    auto ib = g->index.find(ids_b[k]);
    if (ia == g->index.end() || ib == g->index.end())
      VGX_FAIL(c, VGX_ERR_NOT_FOUND, "vgx_graph_edge_covariances: graph contains no node for a requested submap");
    pr[k] = {ia->second, ib->second};
    const int b = ib->second;
    if (red[b] >= 0 && col_of[b] < 0) {
      col_of[b] = (int)cols.size();
      for (int q = 0; q < 4; ++q) cols.push_back(red[b] + q);
    }
  }
  for (int k = 0; k < 16 * m; ++k) cov[k] = 0.0;   // constant blocks: zero covariance
  if (n == 0 || cols.empty()) return VGX_OK;
  cudaStream_t st = c->stream;
  rc = eval_enqueue(c, g, g->d_x, g->d_packed[0], true, false);
  if (rc != VGX_OK) return rc;
  const size_t M = (size_t)n + 1;
  // scratch: requested column indices | X (ncols x n)
  const size_t ncols = cols.size();
  const size_t x_off = (sizeof(int) * ncols + 255) & ~(size_t)255;
  rc = c->ensure_scratch(x_off + sizeof(double) * ncols * (size_t)n);
  if (rc != VGX_OK) return rc;
  int* d_cols = (int*)c->d_scratch;
  double* d_X = (double*)((char*)c->d_scratch + x_off);
  size_t no_smem = 0;
  int coop_grid = 0;
  rc = chol_dispatch(c, n, false, &no_smem, &coop_grid);
  if (rc != VGX_OK) return rc;
  // J^T J is the LM system without Jacobi scaling or damping: with scaling off, a [0, inf] diagonal
  // clamp and an infinite radius lm_build_kernel writes exactly H_ff (and the gradient as row n, which
  // no column of L depends on), and lm_persist_kernel stores the unfactored diagonal H_kk in d_diag.
  LmOpts lo;
  memset(&lo, 0, sizeof(lo));
  lo.min_lm_diagonal = 0.0;
  lo.max_lm_diagonal = INFINITY;
  lo.jacobi_scaling = 0;
  LmState* init = g->h_state;   // pinned: the copy stays asynchronous (the stream is synchronised below)
  memset(init, 0, sizeof(*init));
  init->radius = INFINITY;
  init->step_valid = 1;
  VGX_CUDA(c, cudaMemsetAsync(g->d_A, 0, sizeof(double) * M * M, st));
  VGX_CUDA(c, cudaMemcpyAsync(g->d_state, init, sizeof(*init), cudaMemcpyHostToDevice, st));
  {
    VgxLaunchScope s(c, 4, 3);
    enqueue_lm_build(st, g, n, lo);
    VGX_CUDA(c, launch_chol_coop(st, coop_grid, g->d_A, n, g->d_state, g->d_diag, VGX_COV_RANK_TOL));
  }
  VGX_CUDA(c, cudaGetLastError());
  // inverse columns
  VGX_CUDA(c, cudaMemcpyAsync(d_cols, cols.data(), sizeof(int) * ncols, cudaMemcpyHostToDevice, st));
  if (sizeof(double) * (size_t)n > 48 * 1024)
    VGX_CUDA(c, cudaFuncSetAttribute(cov_column_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)(sizeof(double) * (size_t)n)));
  {
    VgxLaunchScope s(c, 4);
    cov_column_kernel<<<(unsigned)ncols, 256, sizeof(double) * (size_t)n, st>>>(g->d_A, n, d_cols, d_X);
  }
  VGX_CUDA(c, cudaGetLastError());
  std::vector<double> X(ncols * (size_t)n);
  LmState hs;
  VGX_CUDA(c, cudaMemcpyAsync(X.data(), d_X, sizeof(double) * X.size(), cudaMemcpyDeviceToHost, st));
  VGX_CUDA(c, cudaMemcpyAsync(&hs, g->d_state, sizeof(hs), cudaMemcpyDeviceToHost, st));
  VGX_CUDA(c, cudaStreamSynchronize(st));
  if (!hs.step_valid)   // a pivot failed the rank rule above (ceres::Covariance::Compute returns false)
    VGX_FAIL(c, VGX_ERR_INVALID, "vgx_graph_edge_covariances: J^T J is not positive definite (rank deficient)");
  for (int k = 0; k < m; ++k) {
    const int a = pr[k].first, b = pr[k].second;
    if (red[a] < 0 || red[b] < 0) continue;
    for (int r = 0; r < 4; ++r)
      for (int q = 0; q < 4; ++q)
        cov[16 * (size_t)k + 4 * r + q] = X[(size_t)(col_of[b] + q) * n + red[a] + r];
  }
  return VGX_OK;
}

extern "C" void vgx_solver_options_default(vgx_solver_options* o) {
  if (!o) return;
  o->max_num_iterations = 50;
  o->parameter_tolerance = 3e-3;  // pose_graph.cpp:93
  o->function_tolerance = 1e-6;
  o->gradient_tolerance = 1e-10;
  o->initial_trust_region_radius = 1e4;
  o->max_trust_region_radius = 1e16;
  o->min_trust_region_radius = 1e-32;
  o->min_relative_decrease = 1e-3;
  o->min_lm_diagonal = 1e-6;
  o->max_lm_diagonal = 1e32;
  o->max_solver_time_s = 4.0;     // pose_graph.cpp:95
  o->jacobi_scaling = 1;
  o->exclude_registration = 0;
}

static double wall_s() {
  struct timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}

extern "C" int vgx_graph_solve(vgx_ctx* c, const vgx_solver_options* opts, double* xyzyaw_out,
                               vgx_solver_summary* summary) {
  const double t0 = wall_s();
  VgxGraph* g = nullptr;
  int rc = prepare(c, &g);
  if (rc != VGX_OK) return rc;
  vgx_solver_options od;
  vgx_solver_options_default(&od);
  const vgx_solver_options* o = opts ? opts : &od;
  const bool excl = o->exclude_registration != 0;
  vgx_solver_summary S;
  memset(&S, 0, sizeof(S));
  const int N = g->N, n = g->n_free;
  cudaStream_t st = c->stream;
  if (!excl && g->zero_weight) {
    S.termination = 6;
    if (summary) *summary = S;
    VGX_FAIL(c, VGX_ZERO_WEIGHT, "a registration constraint has zero summed weight (Evaluate == false)");
  }
  // dense Cholesky: whole system in shared memory when it fits (configs[0..1]), else the
  // cooperative multi-CTA kernel
  size_t smem_chol_bytes = 0;
  int coop_grid = 0;
  if (n > 0) {
    rc = chol_dispatch(c, n, true, &smem_chol_bytes, &coop_grid);
    if (rc != VGX_OK) return rc;
  }
  const bool use_smem_chol = smem_chol_bytes > 0;

  LmOpts lo;
  lo.max_num_iterations = o->max_num_iterations;
  lo.parameter_tolerance = o->parameter_tolerance;
  lo.function_tolerance = o->function_tolerance;
  lo.gradient_tolerance = o->gradient_tolerance;
  lo.max_radius = o->max_trust_region_radius;
  lo.min_radius = o->min_trust_region_radius;
  lo.min_relative_decrease = o->min_relative_decrease;
  lo.min_lm_diagonal = o->min_lm_diagonal;
  lo.max_lm_diagonal = o->max_lm_diagonal;
  lo.jacobi_scaling = o->jacobi_scaling;

  // Slot 0 of d_packed always holds the normal equations at the current poses, slot 1 the candidate's;
  // an accepted step copies 1 -> 0 on the device, so an iteration is a fixed sequence of launches
  // that needs nothing from the host.  The host therefore runs ONE ITERATION AHEAD: iteration k + 1
  // is enqueued before the 144-byte outcome of iteration k has been read (on a second stream, from
  // a snapshot the decide kernel writes); every kernel of an iteration returns at once when the
  // solve has ended, so the speculative iteration after the last one is a row of empty launches
  // that drain while the host already returns.  Multi-rank: no run-ahead (the ranks stay in step).
  rc = eval_enqueue(c, g, g->d_x, g->d_packed[0], true, excl);
  if (rc != VGX_OK) return rc;
  {
    VgxLaunchScope s(c, 4);
    lm_init_kernel<<<1, 256, 0, st>>>(g->d_packed[0], g->d_red_offset, N, g->d_state,
                                      o->initial_trust_region_radius, lo);
  }
  VGX_CUDA(c, cudaMemcpyAsync(g->h_state, g->d_state, sizeof(LmState), cudaMemcpyDeviceToHost, st));
  VGX_CUDA(c, cudaStreamSynchronize(st));
  S.initial_cost = g->h_state->cost;
  bool timed_out = false;
  static const char* no_spec = getenv("VGX_LM_NO_RUNAHEAD");
  const int ahead = (c->nranks == 1 && !(no_spec && no_spec[0] == '1')) ? 1 : 0;
  // VGX_CHOL_DEBUG=1: phase cycle counts of the last shared-memory Cholesky, printed after the solve
  static const char* chol_dbg_env = getenv("VGX_CHOL_DEBUG");
  long long* d_chol_dbg = nullptr;
  if (chol_dbg_env && chol_dbg_env[0] == '1' && use_smem_chol) cudaMalloc((void**)&d_chol_dbg, 8 * sizeof(long long));
  const int* skip = &g->d_state->done;
  auto enqueue_iteration = [&](int k) -> int {
    {
      VgxLaunchScope s(c, 4, 4);
      if (!use_smem_chol)   // the shared-memory solver reads the written blocks only
        VGX_CUDA(c, cudaMemsetAsync(g->d_A, 0, sizeof(double) * (size_t)(n + 1) * (n + 1), st));
      enqueue_lm_build(st, g, n, lo);
      if (use_smem_chol) {
        chol_solve_smem_kernel<<<1, 512, smem_chol_bytes, st>>>(g->d_A, n, g->d_step, g->d_state, g->d_red_offset,
                                                                g->d_block_nodes, N, g->E, d_chol_dbg);
      } else {
        // LM: sign test only (as Eigen's LLT in the reference)
        VGX_CUDA(c, launch_chol_coop(st, coop_grid, g->d_A, n, g->d_state, nullptr, 0.0));
      }
      lm_step_kernel<<<1, 1024, sizeof(double) * n, st>>>(g->d_A, n, N, g->d_red_offset, g->d_scale,
                                                         g->d_diag, g->d_gs, g->d_x, g->d_xc, g->d_step,
                                                         g->d_state, use_smem_chol ? g->d_step : nullptr);
    }
    VGX_CUDA(c, cudaGetLastError());
    // candidate evaluated with Jacobians so an accepted step needs no second pass
    int rc2 = eval_enqueue(c, g, g->d_xc, g->d_packed[1], true, excl, skip);
    if (rc2 != VGX_OK) return rc2;
    {
      VgxLaunchScope s(c, 4, 2);
      lm_decide_kernel<<<1, 256, 0, st>>>(g->d_packed[0], g->d_packed[1], g->d_red_offset, N, g->d_x,
                                          g->d_xc, g->d_state, lo, 1, g->d_snap + (k & 1));
      lm_accept_kernel<<<std::max(1, std::min(64, (int)(g->packed_len / 2048))), 256, 0, st>>>(
          g->d_packed[1], g->d_packed[0], g->packed_len, g->d_state);
    }
    VGX_CUDA(c, cudaGetLastError());
    // outcome of iteration k -> host, on the copy stream (the main stream keeps running ahead)
    VGX_CUDA(c, cudaEventRecord(g->ev_iter[k & 1], st));
    VGX_CUDA(c, cudaStreamWaitEvent(g->copy_stream, g->ev_iter[k & 1], 0));
    VGX_CUDA(c, cudaMemcpyAsync(g->h_snap + (k & 1), g->d_snap + (k & 1), sizeof(LmState),
                                cudaMemcpyDeviceToHost, g->copy_stream));
    VGX_CUDA(c, cudaEventRecord(g->ev_copy[k & 1], g->copy_stream));
    return VGX_OK;
  };
  bool run = !g->h_state->done && n > 0;
  if (run) {
    int enq = 0, k = 0;   // iterations enqueued / the one whose outcome is awaited
    for (;;) {
      while (enq <= k + ahead) {
        // (single-rank only: ranks must take identical decisions or the exchange would hang)
        if (enq > k && c->nranks == 1 && wall_s() - t0 >= o->max_solver_time_s) break;
        rc = enqueue_iteration(enq);
        if (rc != VGX_OK) return rc;
        ++enq;
      }
      VGX_CUDA(c, cudaEventSynchronize(g->ev_copy[k & 1]));
      *g->h_state = g->h_snap[k & 1];
      if (g->h_state->done) break;
      if (c->nranks == 1 && wall_s() - t0 >= o->max_solver_time_s) { timed_out = true; break; }
      ++k;
    }
    if (timed_out) VGX_CUDA(c, cudaStreamSynchronize(st));   // iterations in flight still move x
    // final poses: the main stream may still be draining the empty launches of the speculative
    // iteration; the copy stream is ordered after the deciding iteration only
    VGX_CUDA(c, cudaMemcpyAsync(g->h_x, g->d_x, sizeof(double) * 4 * N, cudaMemcpyDeviceToHost,
                                timed_out ? st : g->copy_stream));
    VGX_CUDA(c, cudaStreamSynchronize(timed_out ? st : g->copy_stream));
    if (timed_out) {
      VGX_CUDA(c, cudaMemcpyAsync(g->h_state, g->d_state, sizeof(LmState), cudaMemcpyDeviceToHost, st));
      VGX_CUDA(c, cudaStreamSynchronize(st));
    }
    memcpy(g->x.data(), g->h_x, sizeof(double) * 4 * N);
  } else {
    VGX_CUDA(c, cudaMemcpyAsync(g->x.data(), g->d_x, sizeof(double) * 4 * N, cudaMemcpyDeviceToHost, st));
    VGX_CUDA(c, cudaStreamSynchronize(st));
  }
  if (n == 0) { g->h_state->termination = 2; }
  if (d_chol_dbg) {
    long long h[5] = {0, 0, 0, 0, 0};
    cudaStreamSynchronize(st);
    cudaMemcpy(h, d_chol_dbg, sizeof(h), cudaMemcpyDeviceToHost);
    fprintf(stderr, "[vgx] chol n=%d cycles: load %lld update %lld factor+solve %lld back %lld total %lld\n", n, h[0],
            h[1], h[2], h[3], h[4]);
    cudaFree(d_chol_dbg);
  }
  S.iterations = g->h_state->iterations;
  S.num_successful_steps = g->h_state->successful;
  S.num_residual_evals = g->h_state->evals;
  S.termination = timed_out ? 4 : g->h_state->termination;
  S.final_cost = g->h_state->cost;
  S.total_time_s = wall_s() - t0;
  if (xyzyaw_out) memcpy(xyzyaw_out, g->x.data(), sizeof(double) * 4 * N);
  if (summary) *summary = S;
  if (c->nranks > 1) {
    rc = vgx_p2p_check(c);
    if (rc != VGX_OK) return rc;
  }
  if (S.termination == 6) VGX_FAIL(c, VGX_ERR_INVALID, "solver failure: too many consecutive invalid steps");
  return VGX_OK;
}
