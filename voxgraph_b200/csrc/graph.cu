// Pose graph on the device: fused evaluation of all residual blocks into packed
// normal-equation blocks (pose set-up -> reduce -> per-constraint sums -> assembly, chained by
// programmatic dependent launches), exchange across ranks inside the assembly kernel (tagged
// push over NVLink peer memory; NCCL all-reduce as the fallback), and a device-resident
// Levenberg-Marquardt with Ceres' default trust-region schedule that runs one iteration ahead of
// the host.
//
// Reference: voxgraph/src/backend/pose_graph.cpp:48-106 (constraints, optimize()),
// include/voxgraph/backend/constraint/cost_functions/relative_pose_cost_function_inl.h:8-70,
// src/backend/node/node_collection.cpp:8-12 (x,y,z additive, yaw wrapped),
// Ceres 1.x TrustRegionMinimizer/LevenbergMarquardtStrategy defaults (SURVEY.md A.6).
#include <limits.h>
#include <math.h>
#include <string.h>
#include <time.h>

#include <algorithm>
#include <new>
#include <numeric>

#include <cooperative_groups.h>

#include "registration.cuh"
#include "registration_kernels.h"

namespace cg = cooperative_groups;

#define PACK_HDR 4      // [0] cost, [1..3] reserved

struct LmState {
  double radius, decrease_factor;
  double cost, cand_cost, model_cost_change;
  double x_norm, step_norm, gmax;
  int reuse_diagonal, consecutive_invalid;
  int iterations, successful, evals;
  int termination, done, accepted, step_valid, scale_ready;
};

struct LmOpts {
  int max_num_iterations;
  double parameter_tolerance, function_tolerance, gradient_tolerance;
  double max_radius, min_radius, min_relative_decrease, min_lm_diagonal, max_lm_diagonal;
  int jacobi_scaling;
};

struct VgxGraph {
  int N = 0;
  std::vector<uint32_t> ids;
  std::vector<double> x;
  std::vector<uint8_t> constant;
  std::map<uint32_t, int> index;
  std::vector<VgxRelEdge> rel;
  std::vector<uint32_t> reg_ref, reg_read;
  std::vector<vgx_reg_config> reg_cfgs;              // one per residual block
  std::vector<std::vector<int32_t>> samples;         // sampling mode: indices in use per block
  std::vector<std::vector<int32_t>> sample_override; // vgx_graph_set_sample_indices
  bool dirty = true;

  // derived
  std::vector<int> local;  // global indices of this rank's registration constraints
  std::vector<int> block_nodes;  // E x 2 (host copy)
  int n_local = 0, n_tiles = 0, n_rel_local = 0, n_ctas = 0, grid_capacity = 0;
  int E = 0;               // off-diagonal blocks
  int n_free = 0;          // reduced dimension 4 * (non-constant nodes)
  int64_t residuals_local = 0, residuals_global = 0;
  bool zero_weight = false;
  size_t packed_len = 0;

  // device
  RegConstraintDev* d_cons = nullptr;
  RegPoseConst* d_poses = nullptr;
  RegTile* d_tiles = nullptr;
  int* d_tile_begin = nullptr;
  int* d_cta_tile_begin = nullptr;
  double* d_partials = nullptr;
  double* d_csum = nullptr;
  VgxRelEdge* d_rel = nullptr;
  int* d_counters = nullptr;    // (unused)
  unsigned char* d_block_mask = nullptr;   // per output block: bit r = rank r contributes (peer exchange)
  int* d_tile_order = nullptr;  // one-CTA-per-tile mode: CTA b runs tile d_tile_order[b] (longest first)
  int* d_tile_cost = nullptr;   // SM cycles each tile took in the latest evaluation
  bool hw_tiles = false;
  int evals_since_order = -1;   // -1: no cost measured yet since the tables were built
  int* d_csr_begin = nullptr;   // N + E + 1
  int4* d_csr_items = nullptr;  // (source, role, first tile, end tile)
  int* d_block_nodes = nullptr; // E x 2
  int* d_red_offset = nullptr;  // N: reduced offset or -1
  double* d_x = nullptr;
  double* d_xc = nullptr;
  double* d_packed[2] = {nullptr, nullptr};
  double* d_A = nullptr;
  double* d_scale = nullptr;
  double* d_diag = nullptr;
  double* d_gs = nullptr;
  double* d_step = nullptr;
  LmState* d_state = nullptr;
  LmState* h_state = nullptr;
  LmState* d_snap = nullptr;    // [2] outcome of iteration k (written by lm_decide), parity k & 1
  LmState* h_snap = nullptr;    // [2] pinned
  double* h_x = nullptr;        // pinned, 4 * h_x_cap
  int h_x_cap = 0;
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ev_iter[2] = {nullptr, nullptr}, ev_copy[2] = {nullptr, nullptr};
  float* d_sample_pts = nullptr;   // gathered unit-major points of the local sampled blocks
  int32_t* d_sample_idx = nullptr;
};

static void free_tables(VgxGraph* g) {
  cudaFree(g->d_cons); cudaFree(g->d_poses); cudaFree(g->d_tiles); cudaFree(g->d_tile_begin); cudaFree(g->d_cta_tile_begin);
  cudaFree(g->d_partials); cudaFree(g->d_csum); cudaFree(g->d_rel); cudaFree(g->d_counters);
  cudaFree(g->d_tile_order); cudaFree(g->d_tile_cost); cudaFree(g->d_block_mask);
  g->d_tile_order = nullptr; g->d_tile_cost = nullptr; g->d_block_mask = nullptr;
  cudaFree(g->d_csr_begin); cudaFree(g->d_csr_items); cudaFree(g->d_block_nodes);
  cudaFree(g->d_red_offset); cudaFree(g->d_x); cudaFree(g->d_xc);
  cudaFree(g->d_packed[0]); cudaFree(g->d_packed[1]);
  cudaFree(g->d_A); cudaFree(g->d_scale); cudaFree(g->d_diag); cudaFree(g->d_gs); cudaFree(g->d_step);
  cudaFree(g->d_state);
  cudaFree(g->d_sample_pts); cudaFree(g->d_sample_idx);
  g->d_sample_pts = nullptr; g->d_sample_idx = nullptr;
  cudaFree(g->d_snap); g->d_snap = nullptr;
  // the pinned host buffers (h_state, h_snap, h_x) outlive the tables: cudaMallocHost costs ~0.2 ms each
  g->d_cons = nullptr; g->d_poses = nullptr; g->d_tiles = nullptr; g->d_tile_begin = nullptr; g->d_cta_tile_begin = nullptr;
  g->d_partials = nullptr; g->d_csum = nullptr; g->d_rel = nullptr; g->d_counters = nullptr;
  g->d_csr_begin = nullptr; g->d_csr_items = nullptr; g->d_block_nodes = nullptr;
  g->d_red_offset = nullptr; g->d_x = nullptr; g->d_xc = nullptr;
  g->d_packed[0] = g->d_packed[1] = nullptr;
  g->d_A = nullptr; g->d_scale = nullptr; g->d_diag = nullptr; g->d_gs = nullptr; g->d_step = nullptr;
  g->d_state = nullptr;
}

void vgx_graph_free(vgx_ctx* c) {
  if (!c->graph) return;
  cudaStreamSynchronize(c->stream);
  free_tables(c->graph);
  if (c->graph->h_state) cudaFreeHost(c->graph->h_state);
  if (c->graph->h_snap) cudaFreeHost(c->graph->h_snap);
  if (c->graph->h_x) cudaFreeHost(c->graph->h_x);
  if (c->graph->copy_stream) {
    cudaStreamDestroy(c->graph->copy_stream);
    for (int k = 0; k < 2; ++k) { cudaEventDestroy(c->graph->ev_iter[k]); cudaEventDestroy(c->graph->ev_copy[k]); }
  }
  delete c->graph;
  c->graph = nullptr;
}

void vgx_graph_invalidate_registration(vgx_ctx* c) {
  if (c->graph) c->graph->dirty = true;
}

static VgxGraph* graph_of(vgx_ctx* c) {
  if (!c->graph) {
    c->graph = new (std::nothrow) VgxGraph();
  }
  return c->graph;
}

// ------------------------------------------------------------------ kernels: blocks
__device__ __forceinline__ double normalize_angle(double a) {
  const double two_pi = 6.283185307179586476925286766559;
  return a - two_pi * floor((a + 3.14159265358979323846) / two_pi);
}

// RelativePoseCostFunction (inl.h:8-70) with the analytic Jacobians autodiff yields:
// r (4) and J = [dr/dA | dr/dB] (4 x 8), both already multiplied by sqrt_information.
struct RelEval {
  double r[4];
  double J[4][8];
};

__device__ __forceinline__ void rel_eval(const VgxRelEdge& E, const double* __restrict__ x, RelEval& o) {
  const double* A = x + 4 * E.a;
  const double* B = x + 4 * E.b;
  const double c = cos(A[3]), s = sin(A[3]);
  const double dx = B[0] - A[0], dy = B[1] - A[1], dz = B[2] - A[2];
  double err[4];
  err[0] = (c * dx + s * dy) - E.t_obs[0];
  err[1] = (-s * dx + c * dy) - E.t_obs[1];
  err[2] = dz - E.t_obs[2];
  err[3] = normalize_angle((B[3] - A[3]) - E.yaw_obs);
  const double ja[16] = {-c, -s, 0, -s * dx + c * dy, s, -c, 0, -c * dx - s * dy,
                         0, 0, -1, 0, 0, 0, 0, -1};
  const double jb[16] = {c, s, 0, 0, -s, c, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    double acc = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) acc += E.L[4 * i + k] * err[k];
    o.r[i] = acc;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      double sa = 0, sb = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        sa += E.L[4 * i + k] * ja[4 * k + j];
        sb += E.L[4 * i + k] * jb[4 * k + j];
      }
      o.J[i][j] = sa;
      o.J[i][4 + j] = sb;
    }
  }
}

// The reduce kernel leaves one row of 21 sums per TILE; a constraint's sums are its tiles' rows added
// in tile order, times factor^2 (cpp:274-291).  Doing this here, in the consumer, keeps tickets and
// fences out of the hot kernel and is bit-reproducible whatever order the tiles ran in.
struct RegSums {
  const double* partials;
  const int* tile_begin;
  const RegConstraintDev* cons;
};
// entry e of the tiles [t0, t1), added in tile order (four loads in flight)
__device__ __forceinline__ double reg_tile_sum(const double* __restrict__ partials, int t0, int t1, int e) {
  const double* p = partials + (size_t)t0 * VGX_REG_NSTRIDE + e;
  double s = 0;
  int t = t0;
  for (; t + 4 <= t1; t += 4, p += 4 * VGX_REG_NSTRIDE) {
    const double v0 = __ldcg(p), v1 = __ldcg(p + VGX_REG_NSTRIDE), v2 = __ldcg(p + 2 * VGX_REG_NSTRIDE),
                 v3 = __ldcg(p + 3 * VGX_REG_NSTRIDE);
    s = (((s + v0) + v1) + v2) + v3;
  }
  for (; t < t1; ++t, p += VGX_REG_NSTRIDE) s += __ldcg(p);
  return s;
}
__device__ __forceinline__ double reg_constraint_sum(const RegSums& R, int c, int e) {
  const double f = R.cons[c].factor;
  return reg_tile_sum(R.partials, R.tile_begin[c], R.tile_begin[c + 1], e) * (f * f);
}

// Per-constraint sums csum[c][21] from the tile rows: one warp per constraint, a programmatic
// dependent of the reduce kernel (and the assembly kernel is one of this).  A separate, massively
// parallel stage: inside the assembly the same loop is a chain of dependent L2 latencies per item.
// The tiles are added in tile-index order, never in completion order: every evaluation at the same
// poses is bit-identical, which the parity tests and bench.py --dump-outputs rely on.
__global__ void __launch_bounds__(128)
reg_csum_kernel(RegSums R, int n, double* __restrict__ csum, const int* __restrict__ skip) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (skip && *skip) return;
  const int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (c < n && lane < VGX_REG_NSUM) csum[(size_t)c * VGX_REG_NSTRIDE + lane] = reg_constraint_sum(R, c, lane);
}

// Assembly of the packed normal equations, one 4-warp CTA per output block (N diagonal, E
// off-diagonal, +1 for the cost). Lanes 0..15 own the 4x4 entries, lanes 16..19 the
// gradient of a diagonal block. Contributions are summed in list order -> bit-reproducible.
// A registration item reads the constraint's 21 sums (csum) and expands them with
// je[0..2] == -jr[0..2]; a relative-pose item is evaluated on the fly.
// item = (source, role): source >= 0 registration constraint, < 0 relative edge -(e+1);
// role 0: A-A, 1: B-B, 2: rows A / cols B, 3: rows B / cols A.
// Work of one output block `ob` (N diagonal, E off-diagonal, ob == N + E: the cost) by one
// 4-warp CTA: warp w sums items w, w+4, ...; the four partial sums are combined in warp order
// -> bit-reproducible. Ends with a __syncthreads() so it can be called in a loop.
__device__ __forceinline__ void assemble_block(int ob, const double* __restrict__ csum,
                                               const VgxRelEdge* __restrict__ rel,
                                               const double* __restrict__ x,
                                               const int* __restrict__ csr_begin,
                                               const int4* __restrict__ items,
                                               const VgxP2PPush& push, int N, int E, int n_reg,
                                               int n_rel, int exclude_reg, double (*s_part)[20]) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (ob == N + E) {
    // cost = 1/2 sum r^2
    double a = 0;
    if (!exclude_reg)
      for (int c = threadIdx.x; c < n_reg; c += 128) a += __ldcg(csum + (size_t)c * VGX_REG_NSTRIDE + 20);
    for (int e = threadIdx.x; e < n_rel; e += 128) {
      RelEval R;
      rel_eval(rel[e], x, R);
      a += R.r[0] * R.r[0] + R.r[1] * R.r[1] + R.r[2] * R.r[2] + R.r[3] * R.r[3];
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) a += __shfl_xor_sync(0xffffffffu, a, off);
    if (lane == 0) s_part[warp][0] = a;
    __syncthreads();
    if (threadIdx.x == 0) {
      const double cst = 0.5 * (((s_part[0][0] + s_part[1][0]) + s_part[2][0]) + s_part[3][0]);
      for (int k = 0; k < push.n; ++k) {
        vgx_push_store(push, k, 0, cst);
        vgx_push_store(push, k, 1, 0.0); vgx_push_store(push, k, 2, 0.0); vgx_push_store(push, k, 3, 0.0);
      }
    }
    __syncthreads();
    return;
  }
  const int i0 = csr_begin[ob], i1 = csr_begin[ob + 1];
  // peer exchange: a block this rank has nothing for is not pushed (the receivers know from the
  // block's rank mask that this slot holds no value of this epoch)
  if (push.tag != 0 && i0 == i1) return;
  const bool diag = ob < N;
  const int r4 = (lane >> 2) & 3, c4 = lane & 3;
  double acc = 0;
  // warp w expands items w, w + 4, ... in list order; two items per trip so their loads overlap
  for (int i = i0 + warp; i < i1; i += 8) {
    const bool two = i + 4 < i1;
    const int4 itA = __ldg(items + i);
    const int4 itB = two ? __ldg(items + i + 4) : make_int4(-1, 0, 0, 0);
    double svA = 0.0, svB = 0.0;
    if (!exclude_reg && lane < VGX_REG_NSUM) {
      if (itA.x >= 0) svA = __ldcg(csum + (size_t)itA.x * VGX_REG_NSTRIDE + lane);
      if (two && itB.x >= 0) svB = __ldcg(csum + (size_t)itB.x * VGX_REG_NSTRIDE + lane);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (h == 1 && !two) break;
      const int4 it = h ? itB : itA;
      const double sv = h ? svB : svA;
      // (row, col) of the residual block's 8x8 this lane needs; lanes 16..19: gradient row
      int row, col;
      if (lane < 16) {
        switch (it.y) {
          case 0: row = r4; col = c4; break;
          case 1: row = 4 + r4; col = 4 + c4; break;
          case 2: row = r4; col = 4 + c4; break;
          default: row = 4 + r4; col = c4; break;
        }
      } else {
        row = (it.y == 0 ? 0 : 4) + (lane & 3);
        col = -1;
      }
      if (it.x >= 0) {
        if (exclude_reg) continue;
        // 8-vector j8 = (j0, j1, j2, j3, -j0, -j1, -j2, j4): map component a -> (m, sign)
        const int ma = (row < 4) ? row : (row == 7 ? 4 : row - 4);
        const double sa = (row >= 4 && row < 7) ? -1.0 : 1.0;
        int idx;
        double sgn = sa;
        if (col >= 0) {
          const int mb = (col < 4) ? col : (col == 7 ? 4 : col - 4);
          sgn *= (col >= 4 && col < 7) ? -1.0 : 1.0;
          const int p = min(ma, mb), q = max(ma, mb);
          idx = p * 5 - (p * (p - 1)) / 2 + (q - p);
        } else {
          idx = 15 + ma;
        }
        const double v = __shfl_sync(0xffffffffu, sv, idx);
        acc += sgn * v;
      } else {
        RelEval R;
        rel_eval(rel[-it.x - 1], x, R);
        double v = 0;
        if (col >= 0) {
#pragma unroll
          for (int k = 0; k < 4; ++k) v += R.J[k][row] * R.J[k][col];
        } else {
#pragma unroll
          for (int k = 0; k < 4; ++k) v += R.J[k][row] * R.r[k];
        }
        acc += v;
      }
    }
  }
  if (lane < 20) s_part[warp][lane] = acc;
  __syncthreads();
  if (warp == 0 && lane < 20) {
    const double tot = ((s_part[0][lane] + s_part[1][lane]) + s_part[2][lane]) + s_part[3][lane];
    // single rank: one local destination; peer exchange: the value goes to this rank's slot in
    // every rank's region (posted stores over NVLink)
    for (int k = 0; k < push.n; ++k) {
      if (lane < 16) vgx_push_store(push, k, PACK_HDR + 4 * (size_t)N + 16 * (size_t)ob + lane, tot);
      else if (diag) vgx_push_store(push, k, PACK_HDR + 4 * (size_t)ob + (lane - 16), tot);
    }
  }
  __syncthreads();
}

__global__ void __launch_bounds__(128)
assemble_kernel(const double* __restrict__ csum, const VgxRelEdge* __restrict__ rel,
                const double* __restrict__ x, const int* __restrict__ csr_begin,
                const int4* __restrict__ items, VgxP2PPush push, int N, int E, int n_reg,
                int n_rel, int exclude_reg, const int* __restrict__ skip) {
  __shared__ double s_part[4][20];
  if (skip && *skip) return;   // evaluation enqueued ahead of a solve that has already ended
  // programmatic dependent of the constraint-sum kernel (itself one of the reduce kernel): scheduled
  // while those grids drain, blocked here until the sums are visible
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // next evaluation's pose set-up
  assemble_block(blockIdx.x, csum, rel, x, csr_begin, items, push, N, E, n_reg, n_rel, exclude_reg, s_part);
}

// Fused compute + collective (multi-rank, peer exchange): ONE launch assembles this rank's
// partial and PUSHES every element, tagged with the evaluation's epoch, into its slot of every rank's
// NVLink-mapped region while it is produced; the same CTAs then spin on the tagged elements of the n
// local slots and add them in rank order.  No fence, ticket or flag sits between producing a value
// and a peer consuming it.  The grid is persistent and sized to be fully co-resident, so spinning
// CTAs can never starve a CTA (here or on a peer) that still has to produce.
__global__ void __launch_bounds__(128)
assemble_exchange_kernel(const double* __restrict__ csum, const VgxRelEdge* __restrict__ rel,
                         const double* __restrict__ x, const int* __restrict__ csr_begin,
                         const int4* __restrict__ items, VgxP2PPush push, int N, int E,
                         int n_reg, int n_rel, int exclude_reg, VgxP2PGather gat,
                         double* __restrict__ out, int count, const int* __restrict__ skip,
                         const unsigned char* __restrict__ block_mask) {
  if (skip && *skip) return;   // identical on every rank (the ranks' solver states are bit-identical)
  __shared__ double s_part[4][20];
  asm volatile("griddepcontrol.wait;" ::: "memory");   // see assemble_kernel
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  for (int ob = blockIdx.x; ob <= N + E; ob += gridDim.x)
    assemble_block(ob, csum, rel, x, csr_begin, items, push, N, E, n_reg, n_rel, exclude_reg, s_part);
  vgx_ll_gather(gat, out, (size_t)count, (size_t)blockIdx.x * blockDim.x + threadIdx.x,
                (size_t)gridDim.x * blockDim.x, block_mask, N);
}

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

// Blocked right-looking Cholesky of the (n+1) x (n+1) lower-triangular system, one CTA.
// smem: sD[32][33] diagonal block, sP[(M - 32)][33] panel.
#define CH_NB 32
__global__ void __launch_bounds__(1024) chol_kernel(double* __restrict__ A, int n,
                                                    LmState* __restrict__ st) {
  extern __shared__ double smem[];
  if (st->done) return;
  double* sD = smem;                 // 32 x 33
  double* sP = smem + CH_NB * 33;    // rows x 33
  const int M = n + 1;
  const int tid = threadIdx.x, T = blockDim.x;
  __shared__ int s_fail;
  __shared__ double sDinv[CH_NB];
  if (tid == 0) s_fail = 0;
  __syncthreads();
  for (int j0 = 0; j0 < n; j0 += CH_NB) {
    const int nb = min(CH_NB, n - j0);
    // 1. diagonal block -> smem
    for (int t = tid; t < nb * nb; t += T) {
      const int r = t % nb, c = t / nb;
      if (r >= c) sD[r * 33 + c] = A[(size_t)(j0 + c) * M + j0 + r];
    }
    __syncthreads();
    // 2. factor it (warp 0, lane = row)
    if (tid < 32) {
      const int r = tid;
      for (int k = 0; k < nb; ++k) {
        double d = sD[k * 33 + k];
        if (!(d > 0.0) || !isfinite(d)) { if (r == 0) s_fail = 1; d = 1.0; }
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
    // write the factored diagonal block back
    for (int t = tid; t < nb * nb; t += T) {
      const int r = t % nb, c = t / nb;
      if (r >= c) A[(size_t)(j0 + c) * M + j0 + r] = sD[r * 33 + c];
    }
    // 3. panel solve, one thread per row below the block (includes the rhs row n)
    const int r0 = j0 + nb;
    const int rows = M - r0;
    for (int rr = tid; rr < rows; rr += T) {
      double* p = sP + (size_t)rr * 33;
      for (int c = 0; c < nb; ++c) {
        double v = A[(size_t)(j0 + c) * M + r0 + rr];
        for (int k = 0; k < c; ++k) v -= p[k] * sD[c * 33 + k];
        v *= sDinv[c];
        p[c] = v;
        A[(size_t)(j0 + c) * M + r0 + rr] = v;
      }
    }
    __syncthreads();
    // 4. trailing update: A[i][j] -= sum_k P[i][k] P[j][k], i >= j, columns r0..n-1
    const int tc = n - r0;  // trailing columns
    if (tc > 0) {
      // element (ri, cj) with cj in [0,tc), ri in [cj, rows)
      const long long total = (long long)tc * rows - (long long)tc * (tc - 1) / 2;
      // enumerate column by column so consecutive threads share the column
      int cj = 0;
      long long base = 0;  // elements before column cj
      for (long long t = tid; t < total; t += T) {
        while (t >= base + (rows - cj)) { base += rows - cj; ++cj; }
        const int ri = cj + (int)(t - base);
        const double* pi = sP + (size_t)ri * 33;
        const double* pj = sP + (size_t)cj * 33;
        double acc = 0;
#pragma unroll 8
        for (int k = 0; k < CH_NB; ++k) acc = fma(pi[k], pj[k], acc);
        // nb < 32 only happens in the last panel, where tc == 0
        A[(size_t)(r0 + cj) * M + r0 + ri] -= acc;
      }
    }
    __syncthreads();
  }
  if (tid == 0 && s_fail) st->step_valid = 0;
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

// Multi-CTA variant (cooperative launch, grid-wide barriers): every CTA factors the 32x32
// diagonal block redundantly in shared memory (deterministic, saves a barrier), the panel rows
// and the 32x32 trailing tiles are spread over the grid.  Two grid syncs per panel.
__global__ void __launch_bounds__(256) chol_coop_kernel(double* __restrict__ A, int n,
                                                        LmState* __restrict__ st) {
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
        if (!(d > 0.0) || !isfinite(d)) { if (r == 0) s_fail = 1; d = 1.0; }
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

// Accept / reject and termination tests of TrustRegionMinimizer (A.6).
__global__ void lm_decide_kernel(const double* __restrict__ packed_cur,
                                 const double* __restrict__ packed_cand,
                                 const int* __restrict__ red, int N, double* __restrict__ x,
                                 const double* __restrict__ xc, LmState* __restrict__ st, LmOpts o,
                                 int cand_eval_ok, LmState* __restrict__ snapshot) {
  __shared__ double s_g[32];
  if (st->done) {   // no-op iteration: the snapshot still tells the host the solve has ended
    if (threadIdx.x == 0) *snapshot = *st;
    return;
  }
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // gradient max norm at the candidate (used if accepted)
  double gm = 0;
  for (int t = tid; t < 4 * N; t += blockDim.x)
    if (red[t >> 2] >= 0) gm = fmax(gm, fabs(packed_cand[PACK_HDR + t]));
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) gm = fmax(gm, __shfl_xor_sync(0xffffffffu, gm, off));
  if (lane == 0) s_g[warp] = gm;
  __syncthreads();
  __shared__ int s_accept;
  if (tid == 0) {
    gm = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) gm = fmax(gm, s_g[w]);
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
  __shared__ double s_g[32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double gm = 0;
  for (int t = tid; t < 4 * N; t += blockDim.x)
    if (red[t >> 2] >= 0) gm = fmax(gm, fabs(packed[PACK_HDR + t]));
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) gm = fmax(gm, __shfl_xor_sync(0xffffffffu, gm, off));
  if (lane == 0) s_g[warp] = gm;
  __syncthreads();
  if (tid == 0) {
    gm = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) gm = fmax(gm, s_g[w]);
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

// ------------------------------------------------------------------ sharding (host only)
extern "C" int vgx_shard_constraints(int nranks, int n, const int32_t* num_residuals,
                                     const uint32_t* locality_keys, int32_t* owner) {
  if (nranks < 1 || n < 0 || (n > 0 && (!num_residuals || !owner))) return VGX_ERR_INVALID;
  std::vector<int> order(n);
  std::iota(order.begin(), order.end(), 0);
  if (locality_keys)
    std::stable_sort(order.begin(), order.end(),
                     [&](int a, int b) { return locality_keys[a] < locality_keys[b]; });
  int64_t total = 0;
  for (int i = 0; i < n; ++i) total += std::max(num_residuals[i], 0);
  int64_t before = 0;
  for (int i : order) {
    const int64_t cnt = std::max(num_residuals[i], 0);
    // rank whose share [r * total / nranks, (r + 1) * total / nranks) holds the midpoint
    int r = total > 0 ? (int)(((2 * before + cnt) * nranks) / (2 * total)) : 0;
    owner[i] = std::min(std::max(r, 0), nranks - 1);
    before += cnt;
  }
  return VGX_OK;
}

// ------------------------------------------------------------------ table construction
template <class T>
static cudaError_t upload_vec(T** dptr, const std::vector<T>& v, cudaStream_t st) {
  *dptr = nullptr;
  const size_t bytes = sizeof(T) * std::max<size_t>(v.size(), 1);
  cudaError_t e = cudaMalloc((void**)dptr, bytes);
  if (e != cudaSuccess) return e;
  if (!v.empty()) e = cudaMemcpyAsync(*dptr, v.data(), sizeof(T) * v.size(), cudaMemcpyHostToDevice, st);
  return e;
}

static int build_tables(vgx_ctx* c, VgxGraph* g) {
  VGX_CUDA(c, cudaSetDevice(c->device));
  VGX_CUDA(c, cudaStreamSynchronize(c->stream));
  free_tables(g);
  const int N = g->N;
  const int P = (int)g->reg_ref.size();
  // ---- shard registration constraints over ranks: greedy by descending point count
  std::vector<RegConstraintDev> all(P);
  std::vector<uint8_t> is_sampled(P, 0);
  g->zero_weight = false;
  g->residuals_global = 0;
  g->samples.assign(P, std::vector<int32_t>());
  g->sample_override.resize(P);
  for (int i = 0; i < P; ++i) {
    bool sampled = false;
    int rc = vgx_fill_constraint(c, g->reg_ref[i], g->reg_read[i], &g->reg_cfgs[i], &all[i], &sampled);
    if (rc != VGX_OK) return rc;
    auto ia = g->index.find(g->reg_ref[i]);
    auto ib = g->index.find(g->reg_read[i]);
    if (ia == g->index.end() || ib == g->index.end())
      VGX_FAIL(c, VGX_ERR_NOT_FOUND, "registration constraint references a submap without a node");
    all[i].ref_node = ia->second;
    all[i].read_node = ib->second;
    if (all[i].n == 0 || all[i].factor == 0.0) g->zero_weight = true;
    g->residuals_global += all[i].n;
    if (sampled && all[i].n > 0) {
      // Sampling mode: one draw per (re)build of the constraint list, on EVERY rank and in list
      // order, so the per-submap generators advance identically everywhere (see the header).
      is_sampled[i] = 1;
      VgxPoints& p = c->find(g->reg_ref[i])->points[g->reg_cfgs[i].registration_point_type];
      if ((int)g->sample_override[i].size() == all[i].n) {
        g->samples[i] = g->sample_override[i];
        for (int32_t v : g->samples[i])
          if (v < 0 || v >= p.n) VGX_FAIL(c, VGX_ERR_INVALID, "vgx_graph_set_sample_indices: index out of range");
      } else {
        g->samples[i].resize(all[i].n);
        vgx_points_draw(p, all[i].n, g->samples[i].data());
      }
    }
  }
  std::vector<int32_t> owner(P, 0), counts(P, 0);
  for (int i = 0; i < P; ++i) counts[i] = all[i].n;
  vgx_shard_constraints(c->nranks, P, counts.data(), g->reg_read.data(), owner.data());
  g->local.clear();
  std::vector<RegConstraintDev> cons;
  std::vector<RegTile> tiles;
  std::vector<int> tile_begin;
  g->residuals_local = 0;
  for (int i = 0; i < P; ++i) {
    if (owner[i] != c->rank) continue;
    g->local.push_back(i);
    cons.push_back(all[i]);
    g->residuals_local += all[i].n;
  }
  g->n_local = (int)cons.size();
  // gather the drawn points of the local sampled blocks into their own unit-major buffers
  {
    size_t units = 0, nidx = 0;
    for (int k = 0; k < g->n_local; ++k)
      if (is_sampled[g->local[k]]) { units += ((size_t)cons[k].n + 31) / 32; nidx += (size_t)cons[k].n; }
    if (units > 0) {
      VGX_CUDA(c, cudaMalloc((void**)&g->d_sample_pts, units * VGX_PT_UNIT_FLOATS * sizeof(float)));
      VGX_CUDA(c, cudaMalloc((void**)&g->d_sample_idx, nidx * sizeof(int32_t)));
      size_t uo = 0, io = 0;
      for (int k = 0; k < g->n_local; ++k) {
        const int i = g->local[k];
        if (!is_sampled[i]) continue;
        const VgxPoints& p = c->find(g->reg_ref[i])->points[g->reg_cfgs[i].registration_point_type];
        VGX_CUDA(c, cudaMemcpyAsync(g->d_sample_idx + io, g->samples[i].data(), sizeof(int32_t) * cons[k].n,
                                    cudaMemcpyHostToDevice, c->stream));
        float* dst = g->d_sample_pts + uo * VGX_PT_UNIT_FLOATS;
        vgx_launch_reg_gather_samples(c->stream, p.data, g->d_sample_idx + io, cons[k].n, dst);
        c->launches++;
        cons[k].pts = dst;
        uo += ((size_t)cons[k].n + 31) / 32;
        io += (size_t)cons[k].n;
      }
      VGX_CUDA(c, cudaStreamSynchronize(c->stream));  // g->samples[] are pageable host vectors
    }
  }
  // Cut the local residual index space into 32-point units and deal them evenly to the resident
  // CTAs; a tile is the part of one CTA's run of units that lies inside one residual block (tiles
  // never straddle constraints and start on a unit boundary = 128-byte aligned SoA slices for TMA).
  g->grid_capacity = 0;
  for (const auto& cc : cons)
    if (cc.grid) g->grid_capacity = std::max(g->grid_capacity, (cc.gd0 * cc.gd1 * cc.gd2 + 7) & ~7);  // 16-byte multiple
  const int n_ctas_max = std::max(vgx_reg_resident_ctas(c->device, g->grid_capacity), 1);
  int64_t U = 0;  // total units
  for (const auto& cc : cons) U += (cc.n + VGX_REG_UNIT - 1) / VGX_REG_UNIT;
  g->n_ctas = (int)std::min<int64_t>(n_ctas_max, U);
  std::vector<int> cta_tile_begin;
  // Scheduling of the reduce kernel.  The cost of a unit varies ~4x with the share of its points
  // that land in the reading submap, so a static equal cut leaves SMs idle while the hit-heavy
  // ones finish (measured: max SM busy time 16 % above the mean).  hw_units > 0: fixed tiles of
  // that many units, ONE CTA PER TILE, dealt to the SMs by the hardware block scheduler as
  // resident CTAs retire (dynamic balancing at no instruction cost; the per-CTA set-up latency
  // hides behind the other resident CTAs).  0: persistent CTAs with an equal static cut.
  // Tile size: at most VGX_REG_HW_TILE_UNITS units, fewer when the problem is small, so that there
  // are at least ~2 tiles per resident CTA slot (a 3-pair streaming graph still fills the machine).
  int hw_units = VGX_REG_HW_TILE_UNITS;
  if (hw_units > 0)
    hw_units = (int)std::min<int64_t>(hw_units, std::max<int64_t>(4, (U + 2 * (int64_t)n_ctas_max - 1) / (2 * (int64_t)n_ctas_max)));
  if (const char* e = getenv("VGX_REG_HW_TILE_UNITS")) hw_units = atoi(e);
  g->hw_tiles = false;
  g->evals_since_order = -1;
  if (hw_units > 0) {
    for (int k = 0; k < g->n_local; ++k) {
      tile_begin.push_back((int)tiles.size());
      const int tile_pts = hw_units * VGX_REG_UNIT;
      for (int s0 = 0; s0 < cons[k].n; s0 += tile_pts) {
        RegTile t;
        t.constraint = k; t.start = s0; t.count = std::min(tile_pts, cons[k].n - s0);
        tiles.push_back(t);
      }
    }
    g->n_ctas = (int)tiles.size();
    g->hw_tiles = true;
    cta_tile_begin.resize(tiles.size() + 1);
    for (size_t k = 0; k <= tiles.size(); ++k) cta_tile_begin[k] = (int)k;
  } else {
    int64_t ubase = 0;  // unit index of the current constraint's first unit
    int cta = 0;
    auto cta_end = [&](int k) { return (int64_t)(((__int128)U * (k + 1)) / std::max(g->n_ctas, 1)); };
    if (g->n_ctas > 0) cta_tile_begin.push_back(0);
    for (int k = 0; k < g->n_local; ++k) {
      tile_begin.push_back((int)tiles.size());
      const int64_t uc = (cons[k].n + VGX_REG_UNIT - 1) / VGX_REG_UNIT;
      int64_t u = 0;
      while (u < uc) {
        while (cta + 1 < g->n_ctas && ubase + u >= cta_end(cta)) { cta_tile_begin.push_back((int)tiles.size()); ++cta; }
        const int64_t take = std::min<int64_t>(uc - u, cta_end(cta) - (ubase + u));
        RegTile t;
        t.constraint = k;
        t.start = (int)(u * VGX_REG_UNIT);
        t.count = (int)std::min<int64_t>(take * VGX_REG_UNIT, (int64_t)cons[k].n - t.start);
        tiles.push_back(t);
        u += take;
      }
      ubase += uc;
    }
    while ((int)cta_tile_begin.size() <= g->n_ctas) cta_tile_begin.push_back((int)tiles.size());
  }
  tile_begin.push_back((int)tiles.size());
  g->n_tiles = (int)tiles.size();
  for (auto& t : tiles) {   // what the CTA needs to start its bulk copies without a dependent load
    const RegConstraintDev& cc = cons[t.constraint];
    const int cells = cc.gd0 * cc.gd1 * cc.gd2;
    t.pts = cc.pts + (size_t)(t.start / VGX_REG_UNIT) * VGX_PT_UNIT_FLOATS;
    t.grid16 = cc.grid16;
    t.grid_bytes = (cc.grid16 && cells > 0) ? (int)((((size_t)cells + 7) & ~(size_t)7) * sizeof(uint16_t)) : 0;
  }
  g->n_rel_local = (c->rank == 0) ? (int)g->rel.size() : 0;

  // ---- off-diagonal block index over ALL edges (identical on every rank)
  std::map<std::pair<int, int>, int> block_of;
  std::vector<int>& block_nodes = g->block_nodes;
  block_nodes.clear();
  auto block_id = [&](int a, int b) {
    std::pair<int, int> key(std::min(a, b), std::max(a, b));
    auto it = block_of.find(key);
    if (it != block_of.end()) return it->second;
    int id = (int)block_of.size();
    block_of[key] = id;
    block_nodes.push_back(key.first);
    block_nodes.push_back(key.second);
    return id;
  };
  for (const auto& e : g->rel) block_id(e.a, e.b);
  for (int i = 0; i < P; ++i) block_id(all[i].ref_node, all[i].read_node);
  g->E = (int)block_of.size();

  // ---- CSR of contributions per output block (local blocks only)
  std::vector<std::vector<int2>> lists(N + g->E);
  auto add_items = [&](int blk, int a, int b) {
    lists[a].push_back(make_int2(blk, 0));
    lists[b].push_back(make_int2(blk, 1));
    const int ob = N + block_id(a, b);
    lists[ob].push_back(make_int2(blk, a < b ? 2 : 3));
  };
  for (int e = 0; e < g->n_rel_local; ++e) add_items(-(e + 1), g->rel[e].a, g->rel[e].b);
  for (int k = 0; k < g->n_local; ++k) add_items(k, cons[k].ref_node, cons[k].read_node);
  // which ranks have items for an output block (every rank computes the same table: the partition
  // of the constraints is global knowledge; relative edges live on rank 0)
  std::vector<unsigned char> block_mask(N + g->E, 0);
  for (const auto& e : g->rel) {
    block_mask[e.a] |= 1; block_mask[e.b] |= 1;
    block_mask[N + block_id(e.a, e.b)] |= 1;
  }
  for (int i = 0; i < P; ++i) {
    const unsigned char bit = (unsigned char)(1u << owner[i]);
    block_mask[all[i].ref_node] |= bit; block_mask[all[i].read_node] |= bit;
    block_mask[N + block_id(all[i].ref_node, all[i].read_node)] |= bit;
  }
  std::vector<int> csr_begin(N + g->E + 1, 0);
  std::vector<int4> items;   // a registration item carries its constraint's tile range
  for (int ob = 0; ob < N + g->E; ++ob) {
    csr_begin[ob] = (int)items.size();
    for (const int2& it : lists[ob])
      items.push_back(it.x >= 0 ? make_int4(it.x, it.y, tile_begin[it.x], tile_begin[it.x + 1])
                                : make_int4(it.x, it.y, 0, 0));
  }
  csr_begin[N + g->E] = (int)items.size();

  // ---- reduced offsets
  std::vector<int> red(N, -1);
  int n = 0;
  for (int i = 0; i < N; ++i)
    if (!g->constant[i]) { red[i] = n; n += 4; }
  g->n_free = n;
  g->packed_len = PACK_HDR + 20 * (size_t)N + 16 * (size_t)g->E;

  cudaError_t e = cudaSuccess;
  cudaStream_t st = c->stream;
  if (e == cudaSuccess) e = upload_vec(&g->d_cons, cons, st);
  if (e == cudaSuccess) e = upload_vec(&g->d_tiles, tiles, st);
  if (e == cudaSuccess) e = upload_vec(&g->d_tile_begin, tile_begin, st);
  if (e == cudaSuccess) e = upload_vec(&g->d_cta_tile_begin, cta_tile_begin, st);
  static const char* lpt_env = getenv("VGX_REG_LPT");
  if (g->hw_tiles && !(lpt_env && lpt_env[0] == '0')) {
    std::vector<int> ident(tiles.size()), zero(tiles.size(), 0);
    for (size_t k = 0; k < tiles.size(); ++k) ident[k] = (int)k;
    if (e == cudaSuccess) e = upload_vec(&g->d_tile_order, ident, st);
    if (e == cudaSuccess) e = upload_vec(&g->d_tile_cost, zero, st);
  }
  if (e == cudaSuccess) e = upload_vec(&g->d_rel, g->rel, st);
  if (e == cudaSuccess) e = upload_vec(&g->d_csr_begin, csr_begin, st);
  if (e == cudaSuccess) e = upload_vec(&g->d_csr_items, items, st);
  if (e == cudaSuccess) e = upload_vec(&g->d_block_mask, block_mask, st);
  if (e == cudaSuccess) e = upload_vec(&g->d_block_nodes, block_nodes, st);
  if (e == cudaSuccess) e = upload_vec(&g->d_red_offset, red, st);
  if (e == cudaSuccess) e = upload_vec(&g->d_x, g->x, st);
  auto dmalloc = [&](void** p, size_t bytes) {
    if (e == cudaSuccess) e = cudaMalloc(p, std::max<size_t>(bytes, 8));
  };
  dmalloc((void**)&g->d_poses, sizeof(RegPoseConst) * g->n_local);
  dmalloc((void**)&g->d_partials, sizeof(double) * VGX_REG_NSTRIDE * (size_t)g->n_tiles);
  dmalloc((void**)&g->d_csum, sizeof(double) * VGX_REG_NSTRIDE * (size_t)g->n_local);
  dmalloc((void**)&g->d_xc, sizeof(double) * 4 * N);
  dmalloc((void**)&g->d_packed[0], sizeof(double) * g->packed_len);
  dmalloc((void**)&g->d_packed[1], sizeof(double) * g->packed_len);
  dmalloc((void**)&g->d_A, sizeof(double) * (size_t)(n + 1) * (n + 1));
  dmalloc((void**)&g->d_scale, sizeof(double) * n);
  dmalloc((void**)&g->d_diag, sizeof(double) * n);
  dmalloc((void**)&g->d_gs, sizeof(double) * n);
  dmalloc((void**)&g->d_step, sizeof(double) * n);
  dmalloc((void**)&g->d_state, sizeof(LmState));
  if (e == cudaSuccess && !g->h_state) e = cudaMallocHost((void**)&g->h_state, sizeof(LmState));
  dmalloc((void**)&g->d_snap, 2 * sizeof(LmState));
  if (e == cudaSuccess && !g->h_snap) e = cudaMallocHost((void**)&g->h_snap, 2 * sizeof(LmState));
  if (e == cudaSuccess && g->h_x_cap < N) {
    if (g->h_x) cudaFreeHost(g->h_x);
    g->h_x = nullptr;
    g->h_x_cap = std::max(2 * N, 64);
    e = cudaMallocHost((void**)&g->h_x, sizeof(double) * 4 * (size_t)g->h_x_cap);
    if (e != cudaSuccess) g->h_x_cap = 0;
  }
  if (e == cudaSuccess && !g->copy_stream) {
    e = cudaStreamCreateWithFlags(&g->copy_stream, cudaStreamNonBlocking);
    for (int k = 0; k < 2 && e == cudaSuccess; ++k) {
      e = cudaEventCreateWithFlags(&g->ev_iter[k], cudaEventDisableTiming);
      if (e == cudaSuccess) e = cudaEventCreateWithFlags(&g->ev_copy[k], cudaEventDisableTiming);
    }
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) {
    free_tables(g);
    c->set_error(std::string("graph table build: ") + cudaGetErrorString(e));
    return e == cudaErrorMemoryAllocation ? VGX_ERR_NOMEM : VGX_ERR_CUDA;
  }
  g->dirty = false;
  return VGX_OK;
}

// ------------------------------------------------------------------ evaluation pipeline
static int eval_enqueue(vgx_ctx* c, VgxGraph* g, const double* d_x, double* d_packed, bool jacobian,
                        bool exclude_reg, const int* skip = nullptr) {
  cudaStream_t st = c->stream;
  const bool do_reg = !exclude_reg && g->n_local > 0;
  if (do_reg) {
    // refresh the longest-first tile order from the cost measured by the previous evaluation: before
    // the second evaluation on new tables, then every 32nd (the poses move little inside a solve)
    if (g->d_tile_order && g->n_tiles > 1 && (g->evals_since_order == -2 || g->evals_since_order >= 32)) {
      VgxLaunchScope s(c, 5);
      vgx_launch_reg_order(st, g->d_tile_cost, g->n_tiles, g->d_tile_order);
      g->evals_since_order = 0;
    }
    if (g->evals_since_order >= 0) ++g->evals_since_order;
    {
      VgxLaunchScope s(c, 6);
      vgx_launch_reg_pose_setup(st, g->d_cons, d_x, g->d_poses, g->n_local, skip);
    }
    {
      VgxLaunchScope s(c, 0);
      vgx_launch_reg_reduce(st, g->d_cons, g->d_poses, g->d_tiles, g->n_ctas, g->d_cta_tile_begin,
                            g->d_tile_order, g->d_tile_cost, g->d_partials, g->grid_capacity, jacobian, skip);
    }
    if (g->evals_since_order < 0) g->evals_since_order = -2;   // a cost has been measured now
  }
  // multi-rank peer path: the assembly pushes this rank's partial into every rank's region
  const bool p2p = c->nranks > 1 && c->p2p_ready;
  VgxP2PPush push;
  VgxP2PGather gat;
  memset(&push, 0, sizeof(push));
  memset(&gat, 0, sizeof(gat));
  push.n = 1;
  push.dst[0] = d_packed;
  // the assembly kernels and the constraint-sum kernel are launched as programmatic dependents of
  // what precedes them on the stream
  cudaLaunchAttribute pdl[1];
  pdl[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  pdl[0].val.programmaticStreamSerializationAllowed = 1;
  static const char* no_pdl = getenv("VGX_NO_PDL");
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.blockDim = dim3(128);
  cfg.stream = st;
  cfg.attrs = pdl;
  cfg.numAttrs = (no_pdl && no_pdl[0] == '1') ? 0 : 1;
  const int excl = do_reg ? 0 : 1;
  if (do_reg) {
    RegSums sums;
    sums.partials = g->d_partials; sums.tile_begin = g->d_tile_begin; sums.cons = g->d_cons;
    VgxLaunchScope s(c, 7);
    cfg.gridDim = dim3((unsigned)((g->n_local + 3) / 4));
    cudaLaunchKernelEx(&cfg, reg_csum_kernel, sums, g->n_local, g->d_csum, skip);
  }
  if (p2p) {
    int rc = vgx_p2p_begin(c, g->packed_len, &push, &gat);
    if (rc != VGX_OK) return rc;
  }
  if (p2p && c->p2p_fused && g->packed_len < (size_t)INT_MAX) {
    // one launch: assemble + push -> signal -> wait -> local reduce (grid fully co-resident)
    static int resident = 0;
    if (resident == 0) {
      int sms = 0, per_sm = 0;
      cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device);
      if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, assemble_exchange_kernel, 128, 0) != cudaSuccess)
        per_sm = 1;
      resident = std::max(1, sms * std::max(per_sm, 1));
    }
    const int grid = std::min(g->N + g->E + 1, resident);
    {
      VgxLaunchScope s(c, 8);
      cfg.gridDim = dim3((unsigned)grid);
      cudaLaunchKernelEx(&cfg, assemble_exchange_kernel, (const double*)g->d_csum, (const VgxRelEdge*)g->d_rel, d_x,
                         (const int*)g->d_csr_begin, (const int4*)g->d_csr_items, push, g->N, g->E, g->n_local,
                         g->n_rel_local, excl, gat, d_packed, (int)g->packed_len, skip,
                         (const unsigned char*)g->d_block_mask);
    }
    VGX_CUDA(c, cudaGetLastError());
    return VGX_OK;
  }
  {
    VgxLaunchScope s(c, 8);
    cfg.gridDim = dim3((unsigned)(g->N + g->E + 1));
    cudaLaunchKernelEx(&cfg, assemble_kernel, (const double*)g->d_csum, (const VgxRelEdge*)g->d_rel, d_x, (const int*)g->d_csr_begin,
                       (const int4*)g->d_csr_items, push, g->N, g->E, g->n_local, g->n_rel_local, excl, skip);
  }
  VGX_CUDA(c, cudaGetLastError());
  if (p2p) return vgx_p2p_gather(c, gat, d_packed, g->packed_len, g->d_block_mask, g->N);
  return vgx_nccl_allreduce_sum_f64(c, d_packed, g->packed_len);
}

static int prepare(vgx_ctx* c, VgxGraph** out) {
  if (!c) return VGX_ERR_INVALID;
  VgxGraph* g = graph_of(c);
  if (!g) return VGX_ERR_NOMEM;
  if (g->N == 0) VGX_FAIL(c, VGX_ERR_INVALID, "pose graph has no nodes");
  VGX_CUDA(c, cudaSetDevice(c->device));
  if (g->dirty) {
    int rc = build_tables(c, g);
    if (rc != VGX_OK) return rc;
  }
  *out = g;
  return VGX_OK;
}

// ------------------------------------------------------------------ C-ABI: b2
extern "C" int vgx_graph_set_nodes(vgx_ctx* c, int n, const uint32_t* ids, const double* xyzyaw,
                                   const uint8_t* constant) {
  if (!c || n < 0 || (n > 0 && (!ids || !xyzyaw))) return VGX_ERR_INVALID;
  VgxGraph* g = graph_of(c);
  if (!g) return VGX_ERR_NOMEM;
  std::map<uint32_t, int> index;
  for (int i = 0; i < n; ++i) {
    if (index.count(ids[i])) VGX_FAIL(c, VGX_ERR_INVALID, "duplicate submap id in node list");
    index[ids[i]] = i;
  }
  g->N = n;
  g->ids.assign(ids, ids + n);
  g->x.assign(xyzyaw, xyzyaw + 4 * (size_t)n);
  g->constant.assign(n, 0);
  if (constant)
    for (int i = 0; i < n; ++i) g->constant[i] = constant[i] ? 1 : 0;
  g->index.swap(index);
  g->rel.clear();
  g->reg_ref.clear();
  g->reg_read.clear();
  g->reg_cfgs.clear();
  g->sample_override.clear();
  g->dirty = true;
  return VGX_OK;
}

extern "C" int vgx_graph_set_poses(vgx_ctx* c, const double* xyzyaw) {
  if (!c || !xyzyaw) return VGX_ERR_INVALID;
  VgxGraph* g = graph_of(c);
  if (!g || g->N == 0) VGX_FAIL(c, VGX_ERR_INVALID, "pose graph has no nodes");
  g->x.assign(xyzyaw, xyzyaw + 4 * (size_t)g->N);
  if (!g->dirty) {
    VGX_CUDA(c, cudaSetDevice(c->device));
    // stage through pinned memory so the copy is a true async H2D
    int rc = c->ensure_pinned(sizeof(double) * 4 * g->N);
    if (rc != VGX_OK) return rc;
    VGX_CUDA(c, cudaStreamSynchronize(c->stream));
    memcpy(c->h_pinned, xyzyaw, sizeof(double) * 4 * g->N);
    VGX_CUDA(c, cudaMemcpyAsync(g->d_x, c->h_pinned, sizeof(double) * 4 * g->N, cudaMemcpyHostToDevice,
                                c->stream));
  }
  return VGX_OK;
}

extern "C" int vgx_graph_get_poses(vgx_ctx* c, double* xyzyaw) {
  if (!c || !xyzyaw) return VGX_ERR_INVALID;
  VgxGraph* g = graph_of(c);
  if (!g) return VGX_ERR_NOMEM;
  memcpy(xyzyaw, g->x.data(), sizeof(double) * 4 * g->N);
  return VGX_OK;
}

extern "C" int vgx_graph_set_relative_edges(vgx_ctx* c, int m, const uint32_t* ids_a,
                                            const uint32_t* ids_b, const double* t_obs,
                                            const double* sqrt_info) {
  if (!c || m < 0 || (m > 0 && (!ids_a || !ids_b || !t_obs || !sqrt_info))) return VGX_ERR_INVALID;
  VgxGraph* g = graph_of(c);
  if (!g) return VGX_ERR_NOMEM;
  std::vector<VgxRelEdge> rel(m);
  for (int i = 0; i < m; ++i) {
    auto ia = g->index.find(ids_a[i]);
    auto ib = g->index.find(ids_b[i]);
    if (ia == g->index.end() || ib == g->index.end())
      VGX_FAIL(c, VGX_ERR_NOT_FOUND, "relative-pose edge references a submap without a node");
    if (ia->second == ib->second) VGX_FAIL(c, VGX_ERR_INVALID, "relative-pose edge from a node to itself");
    rel[i].a = ia->second;
    rel[i].b = ib->second;
    rel[i].t_obs[0] = t_obs[4 * i]; rel[i].t_obs[1] = t_obs[4 * i + 1]; rel[i].t_obs[2] = t_obs[4 * i + 2];
    rel[i].yaw_obs = t_obs[4 * i + 3];
    memcpy(rel[i].L, sqrt_info + 16 * (size_t)i, sizeof(double) * 16);
  }
  g->rel.swap(rel);
  g->dirty = true;
  return VGX_OK;
}

static int set_registration(vgx_ctx* c, int p, const uint32_t* ref_ids, const uint32_t* read_ids,
                            const vgx_reg_config* cfgs, bool per_constraint) {
  if (!c || p < 0 || (p > 0 && (!ref_ids || !read_ids))) return VGX_ERR_INVALID;
  if (per_constraint && p > 0 && !cfgs) return VGX_ERR_INVALID;
  VgxGraph* g = graph_of(c);
  if (!g) return VGX_ERR_NOMEM;
  for (int i = 0; i < p; ++i) {
    if (ref_ids[i] == read_ids[i]) VGX_FAIL(c, VGX_ERR_INVALID, "cannot constrain a submap to itself");
    if (!g->index.count(ref_ids[i]) || !g->index.count(read_ids[i]))
      VGX_FAIL(c, VGX_ERR_NOT_FOUND, "graph contains no node for a registration constraint's submap");
  }
  vgx_reg_config dflt;
  vgx_reg_config_default(&dflt);
  g->reg_ref.assign(ref_ids, ref_ids + p);
  g->reg_read.assign(read_ids, read_ids + p);
  g->reg_cfgs.resize(p);
  for (int i = 0; i < p; ++i) g->reg_cfgs[i] = per_constraint ? cfgs[i] : (cfgs ? cfgs[0] : dflt);
  g->sample_override.assign(p, std::vector<int32_t>());
  g->dirty = true;
  return VGX_OK;
}

extern "C" int vgx_graph_set_registration_constraints(vgx_ctx* c, int p, const uint32_t* ref_ids,
                                                      const uint32_t* read_ids,
                                                      const vgx_reg_config* cfg) {
  return set_registration(c, p, ref_ids, read_ids, cfg, false);
}

extern "C" int vgx_graph_set_registration_constraints_v(vgx_ctx* c, int p, const uint32_t* ref_ids,
                                                        const uint32_t* read_ids,
                                                        const vgx_reg_config* cfgs) {
  return set_registration(c, p, ref_ids, read_ids, cfgs, true);
}

extern "C" int vgx_graph_set_sample_indices(vgx_ctx* c, int constraint, int n, const int32_t* indices) {
  if (!c) return VGX_ERR_INVALID;
  VgxGraph* g = graph_of(c);
  if (!g) return VGX_ERR_NOMEM;
  if (constraint < 0 || constraint >= (int)g->reg_ref.size() || n < 0 || (n > 0 && !indices))
    VGX_FAIL(c, VGX_ERR_INVALID, "vgx_graph_set_sample_indices: invalid argument");
  if (g->reg_cfgs[constraint].sampling_ratio == -1.0f)
    VGX_FAIL(c, VGX_ERR_INVALID, "vgx_graph_set_sample_indices: the constraint is not in sampling mode");
  g->sample_override.resize(g->reg_ref.size());
  g->sample_override[constraint].assign(indices, indices + n);
  g->dirty = true;
  return VGX_OK;
}

extern "C" int vgx_graph_num_registration_residuals(vgx_ctx* c, int64_t* local, int64_t* global) {
  VgxGraph* g = nullptr;
  int rc = prepare(c, &g);
  if (rc != VGX_OK) return rc;
  if (local) *local = g->residuals_local;
  if (global) *global = g->residuals_global;
  return VGX_OK;
}

extern "C" int vgx_graph_get_sample_indices(vgx_ctx* c, int constraint, int max_n, int32_t* indices, int* n) {
  VgxGraph* g = nullptr;
  int rc = prepare(c, &g);
  if (rc != VGX_OK) return rc;
  if (constraint < 0 || constraint >= (int)g->samples.size())
    VGX_FAIL(c, VGX_ERR_INVALID, "vgx_graph_get_sample_indices: invalid constraint index");
  const std::vector<int32_t>& v = g->samples[constraint];
  if (n) *n = (int)v.size();
  if ((int)v.size() > max_n) VGX_FAIL(c, VGX_ERR_CAPACITY, "vgx_graph_get_sample_indices: max_n too small");
  if (indices && !v.empty()) memcpy(indices, v.data(), sizeof(int32_t) * v.size());
  return VGX_OK;
}

extern "C" int vgx_graph_eval_async(vgx_ctx* c, int exclude_registration) {
  VgxGraph* g = nullptr;
  int rc = prepare(c, &g);
  if (rc != VGX_OK) return rc;
  return eval_enqueue(c, g, g->d_x, g->d_packed[0], true, exclude_registration != 0);
}

extern "C" int vgx_graph_eval(vgx_ctx* c, int exclude_registration, double* cost, double* gradient,
                              double* H) {
  VgxGraph* g = nullptr;
  int rc = prepare(c, &g);
  if (rc != VGX_OK) return rc;
  rc = eval_enqueue(c, g, g->d_x, g->d_packed[0], true, exclude_registration != 0);
  if (rc != VGX_OK) return rc;
  rc = c->ensure_pinned(sizeof(double) * g->packed_len);
  if (rc != VGX_OK) return rc;
  double* h = (double*)c->h_pinned;
  VGX_CUDA(c, cudaMemcpyAsync(h, g->d_packed[0], sizeof(double) * g->packed_len, cudaMemcpyDeviceToHost,
                              c->stream));
  VGX_CUDA(c, cudaStreamSynchronize(c->stream));
  const int N = g->N, dim = 4 * N;
  if (cost) *cost = h[0];
  if (gradient) memcpy(gradient, h + PACK_HDR, sizeof(double) * dim);
  if (H) {
    memset(H, 0, sizeof(double) * (size_t)dim * dim);
    const double* D = h + PACK_HDR + dim;
    const double* O = D + 16 * (size_t)N;
    for (int i = 0; i < N; ++i)
      for (int r = 0; r < 4; ++r)
        for (int q = 0; q < 4; ++q) H[(size_t)(4 * i + r) * dim + 4 * i + q] = D[16 * (size_t)i + 4 * r + q];
    const std::vector<int>& bn = g->block_nodes;
    for (int b = 0; b < g->E; ++b) {
      const int i = bn[2 * b], j = bn[2 * b + 1];
      for (int r = 0; r < 4; ++r)
        for (int q = 0; q < 4; ++q) {
          const double v = O[16 * (size_t)b + 4 * r + q];
          H[(size_t)(4 * i + r) * dim + 4 * j + q] = v;
          H[(size_t)(4 * j + q) * dim + 4 * i + r] = v;
        }
    }
  }
  if (c->nranks > 1) {
    rc = vgx_p2p_check(c);
    if (rc != VGX_OK) return rc;
  }
  if (!exclude_registration && g->zero_weight) return VGX_ZERO_WEIGHT;
  return VGX_OK;
}

extern "C" int vgx_graph_registration_costs(vgx_ctx* c, double* per_constraint) {
  VgxGraph* g = nullptr;
  int rc = prepare(c, &g);
  if (rc != VGX_OK) return rc;
  if (!per_constraint) return VGX_ERR_INVALID;
  rc = eval_enqueue(c, g, g->d_x, g->d_packed[1], false, false);
  if (rc != VGX_OK) return rc;
  const int P = (int)g->reg_ref.size();
  std::vector<double> cs((size_t)g->n_local * VGX_REG_NSTRIDE + 1);
  if (g->n_local > 0)
    VGX_CUDA(c, cudaMemcpyAsync(cs.data(), g->d_csum, sizeof(double) * VGX_REG_NSTRIDE * g->n_local,
                                cudaMemcpyDeviceToHost, c->stream));
  VGX_CUDA(c, cudaStreamSynchronize(c->stream));
  for (int i = 0; i < P; ++i) per_constraint[i] = 0.0;
  for (int k = 0; k < g->n_local; ++k) per_constraint[g->local[k]] = cs[(size_t)k * VGX_REG_NSTRIDE + 20];
  return VGX_OK;
}

// ------------------------------------------------------------------ edge covariances
// PoseGraph::getEdgeCovarianceMap (pose_graph.cpp:117-163): ceres::Covariance blocks
// Cov(x_a, x_b) = rows of a, columns of b of (J^T J)^-1 over the free parameter blocks at the current
// poses (no LM damping, no Jacobi scaling, no loss function); constant blocks have zero covariance.
// Dense reduced H -> Cholesky (the solver's factorisation kernels) -> two triangular solves per
// requested column.
__global__ void cov_build_kernel(const double* __restrict__ packed, const int* __restrict__ red,
                                 const int* __restrict__ block_nodes, int N, int E, int n,
                                 double* __restrict__ A) {
  const int M = n + 1;
  const double* D = packed + PACK_HDR + 4 * (size_t)N;
  const double* O = D + 16 * (size_t)N;
  const int tid = blockIdx.x * blockDim.x + threadIdx.x, stride = gridDim.x * blockDim.x;
  for (int t = tid; t < N * 16; t += stride) {
    const int node = t >> 4, r = (t >> 2) & 3, c = t & 3;
    const int off = red[node];
    if (off < 0 || r < c) continue;
    A[(size_t)(off + c) * M + off + r] = D[16 * (size_t)node + 4 * r + c];
  }
  for (int t = tid; t < E * 16; t += stride) {
    const int b = t >> 4, r = (t >> 2) & 3, c = t & 3;
    const int ni = block_nodes[2 * b], nj = block_nodes[2 * b + 1];
    const int oi = red[ni], oj = red[nj];
    if (oi < 0 || oj < 0) continue;
    A[(size_t)(oi + r) * M + (oj + c)] = O[16 * (size_t)b + 4 * r + c];   // lower triangle: oj > oi
  }
}

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
  std::vector<int> red(N, -1);
  {
    int o = 0;
    for (int i = 0; i < N; ++i)
      if (!g->constant[i]) { red[i] = o; o += 4; }
  }
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
  VGX_CUDA(c, cudaMemsetAsync(g->d_A, 0, sizeof(double) * M * M, st));
  {
    VgxLaunchScope s(c, 4);
    const int nthreads = 16 * (N + g->E);
    cov_build_kernel<<<std::min(296, (nthreads + 255) / 256), 256, 0, st>>>(g->d_packed[0], g->d_red_offset,
                                                                          g->d_block_nodes, N, g->E, n, g->d_A);
  }
  // factorise with the solver's kernels (the rhs row n of the augmented matrix stays zero)
  VGX_CUDA(c, cudaMemsetAsync(g->d_state, 0, sizeof(LmState), st));
  {
    LmState init;
    memset(&init, 0, sizeof(init));
    init.step_valid = 1;
    VGX_CUDA(c, cudaMemcpyAsync(g->d_state, &init, sizeof(init), cudaMemcpyHostToDevice, st));
    VGX_CUDA(c, cudaStreamSynchronize(st));
  }
  {
    VgxLaunchScope s(c, 4);
    int coop = 0, sms = 0, per_sm = 0, coop_grid = 0;
    cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, c->device);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device);
    const size_t chol_smem = sizeof(double) * ((size_t)CH_NB * 33 + (size_t)std::max(n + 1 - CH_NB, 1) * 33);
    if (n > 256 && coop &&
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, chol_coop_kernel, 256, 0) == cudaSuccess && per_sm > 0) {
      const int tiles = ((n + 1 + CH_NB - 1) / CH_NB) * ((n + CH_NB - 1) / CH_NB);
      coop_grid = std::max(1, std::min(sms * std::min(per_sm, 2), std::max(tiles / 2, (n + 256) / 256)));
    }
    if (coop_grid > 0) {
      int n_arg = n;
      void* args[] = {(void*)&g->d_A, (void*)&n_arg, (void*)&g->d_state};
      VGX_CUDA(c, cudaLaunchCooperativeKernel((void*)chol_coop_kernel, dim3(coop_grid), dim3(256), args, 0, st));
    } else {
      if (chol_smem > 227 * 1024)
        VGX_FAIL(c, VGX_ERR_CAPACITY, "pose graph too large for the single-CTA dense factorisation");
      VGX_CUDA(c, cudaFuncSetAttribute(chol_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)chol_smem));
      chol_kernel<<<1, 1024, chol_smem, st>>>(g->d_A, n, g->d_state);
    }
  }
  VGX_CUDA(c, cudaGetLastError());
  // inverse columns
  const size_t ncols = cols.size();
  rc = c->ensure_scratch(sizeof(int) * ncols + 256 + sizeof(double) * ncols * (size_t)n);
  if (rc != VGX_OK) return rc;
  int* d_cols = (int*)c->d_scratch;
  double* d_X = (double*)((char*)c->d_scratch + ((sizeof(int) * ncols + 255) & ~(size_t)255));
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
  if (!hs.step_valid)   // ceres::Covariance::Compute returns false on a rank-deficient Jacobian
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
  // cooperative multi-CTA kernel, else one CTA streaming from global memory
  const size_t smem_chol_bytes = sizeof(double) * ((size_t)(n + 1) * (n + 2) / 2 + n + 2);
  const bool use_smem_chol = n > 0 && n <= 256 && smem_chol_bytes <= 220 * 1024;
  if (use_smem_chol)
    VGX_CUDA(c, cudaFuncSetAttribute(chol_solve_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)smem_chol_bytes));
  int coop_grid = 0;
  if (!use_smem_chol) {
    int coop = 0, sms = 0, per_sm = 0;
    cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, c->device);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device);
    if (coop && cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, chol_coop_kernel, 256, 0) == cudaSuccess &&
        per_sm > 0) {
      const int tiles = ((n + 1 + CH_NB - 1) / CH_NB) * ((n + CH_NB - 1) / CH_NB);
      coop_grid = std::max(1, std::min(sms * std::min(per_sm, 2), std::max(tiles / 2, (n + 256) / 256)));
    }
  }
  const size_t chol_smem = sizeof(double) * ((size_t)CH_NB * 33 + (size_t)std::max(n + 1 - CH_NB, 1) * 33);
  if (coop_grid == 0) {
    if (chol_smem > 227 * 1024)
      VGX_FAIL(c, VGX_ERR_CAPACITY, "pose graph too large for the single-CTA dense solver (max ~219 free nodes)");
    VGX_CUDA(c, cudaFuncSetAttribute(chol_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)chol_smem));
  }

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
      const int nthreads = std::max(16 * (N + g->E), 4 * N);
      lm_build_kernel<<<std::min(296, (nthreads + 255) / 256), 256, 0, st>>>(
          g->d_packed[0], g->d_red_offset, g->d_block_nodes, N, g->E, n, g->d_A, g->d_scale, g->d_diag,
          g->d_gs, g->d_state, lo);
      lm_persist_kernel<<<1, 256, 0, st>>>(g->d_packed[0], g->d_red_offset, N, g->d_scale, g->d_diag,
                                           g->d_state, lo);
      if (use_smem_chol) {
        chol_solve_smem_kernel<<<1, 512, smem_chol_bytes, st>>>(g->d_A, n, g->d_step, g->d_state, g->d_red_offset,
                                                                g->d_block_nodes, N, g->E, d_chol_dbg);
      } else if (coop_grid > 0) {
        int n_arg = n;
        void* args[] = {(void*)&g->d_A, (void*)&n_arg, (void*)&g->d_state};
        VGX_CUDA(c, cudaLaunchCooperativeKernel((void*)chol_coop_kernel, dim3(coop_grid), dim3(256), args, 0, st));
      } else {
        chol_kernel<<<1, 1024, chol_smem, st>>>(g->d_A, n, g->d_state);
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
