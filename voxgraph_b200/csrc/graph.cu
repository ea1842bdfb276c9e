// Pose graph on the device: fused evaluation of all residual blocks into packed
// normal-equation blocks (pose set-up -> reduce -> per-constraint sums -> assembly, chained by
// programmatic dependent launches) and exchange across ranks inside the assembly kernel (tagged
// push over NVLink peer memory; NCCL all-reduce as the fallback).  The solver that consumes the
// packed equations is in solve.cu.
//
// Reference: voxgraph/src/backend/pose_graph.cpp:48-106 (constraints, optimize()),
// include/voxgraph/backend/constraint/cost_functions/relative_pose_cost_function_inl.h:8-70,
// src/backend/node/node_collection.cpp:8-12 (x,y,z additive, yaw wrapped).
#include <limits.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <new>
#include <numeric>

#include "graph.h"
#include "registration.cuh"
#include "registration_kernels.h"

static void free_tables(VgxGraph* g) {
  cudaFree(g->d_cons); cudaFree(g->d_poses); cudaFree(g->d_tiles); cudaFree(g->d_tile_begin);
  cudaFree(g->d_unit_bounds); g->d_unit_bounds = nullptr;
  cudaFree(g->d_partials); cudaFree(g->d_csum); cudaFree(g->d_rel);
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
  g->d_cons = nullptr; g->d_poses = nullptr; g->d_tiles = nullptr; g->d_tile_begin = nullptr;
  g->d_partials = nullptr; g->d_csum = nullptr; g->d_rel = nullptr;
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
  // Scheduling of the reduce kernel.  The cost of a unit varies ~4x with the share of its points
  // that land in the reading submap, so a static equal cut of the units over the resident CTAs
  // leaves SMs idle while the hit-heavy ones finish (measured: max SM busy time 16 % above the
  // mean).  Instead each residual block is cut into fixed tiles of hw_units 32-point units, ONE CTA
  // PER TILE, dealt to the SMs by the hardware block scheduler as resident CTAs retire (dynamic
  // balancing at no instruction cost; the per-CTA set-up latency hides behind the other resident
  // CTAs).  Tiles never straddle constraints and start on a unit boundary (128-byte aligned SoA
  // slices for TMA).
  g->grid_capacity = 0;
  for (const auto& cc : cons)
    if (cc.grid) g->grid_capacity = std::max(g->grid_capacity, (cc.gd0 * cc.gd1 * cc.gd2 + 7) & ~7);  // 16-byte multiple
  const int resident_ctas = std::max(vgx_reg_resident_ctas(c->device, g->grid_capacity), 1);
  int64_t U = 0;  // total units
  for (const auto& cc : cons) U += (cc.n + VGX_REG_UNIT - 1) / VGX_REG_UNIT;
  // Tile size: at most VGX_REG_HW_TILE_UNITS units, fewer when the problem is small, so that there
  // are at least ~2 tiles per resident CTA slot (a 3-pair streaming graph still fills the machine).
  // The environment variable of the same name forces a size (n >= 1; tests use it for shapes the
  // formula never produces).
  int hw_units = (int)std::min<int64_t>(VGX_REG_HW_TILE_UNITS,
                                        std::max<int64_t>(4, (U + 2 * (int64_t)resident_ctas - 1) / (2 * (int64_t)resident_ctas)));
  if (const char* env = getenv("VGX_REG_HW_TILE_UNITS"))
    if (atoi(env) >= 1) hw_units = atoi(env);
  g->evals_since_order = -1;
  const int tile_pts = hw_units * VGX_REG_UNIT;
  for (int k = 0; k < g->n_local; ++k) {
    tile_begin.push_back((int)tiles.size());
    for (int s0 = 0; s0 < cons[k].n; s0 += tile_pts) {
      RegTile t;
      t.constraint = k; t.count = std::min(tile_pts, cons[k].n - s0);
      t.pts = cons[k].pts + (size_t)(s0 / VGX_REG_UNIT) * VGX_PT_UNIT_FLOATS;
      tiles.push_back(t);
    }
  }
  tile_begin.push_back((int)tiles.size());
  g->n_tiles = (int)tiles.size();
  int n_units = 0;   // units of all tiles = entries of the unit-bound table
  for (auto& t : tiles) {   // what the CTA needs to start its bulk copies without a dependent load
    const RegConstraintDev& cc = cons[t.constraint];
    const int cells = cc.gd0 * cc.gd1 * cc.gd2;
    t.unit0 = n_units;
    n_units += (t.count + VGX_REG_UNIT - 1) / VGX_REG_UNIT;
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
  std::vector<int>& red = g->red;
  red.assign(N, -1);
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
  {
    std::vector<int> ident(tiles.size()), zero(tiles.size(), 0);
    std::iota(ident.begin(), ident.end(), 0);
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
  dmalloc((void**)&g->d_unit_bounds, sizeof(float4) * (size_t)n_units);
  if (e == cudaSuccess && g->n_tiles > 0) {
    vgx_launch_reg_unit_bounds(st, g->d_tiles, g->n_tiles, g->d_unit_bounds);
    c->launches++;
    e = cudaGetLastError();
  }
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
int eval_enqueue(vgx_ctx* c, VgxGraph* g, const double* d_x, double* d_packed, bool jacobian, bool exclude_reg,
                 const int* skip) {
  cudaStream_t st = c->stream;
  const bool do_reg = !exclude_reg && g->n_local > 0;
  if (do_reg) {
    // refresh the longest-first tile order from the cost measured by the previous evaluation: before
    // the second evaluation on new tables, then every 32nd (the poses move little inside a solve)
    if (g->n_tiles > 1 && (g->evals_since_order == -2 || g->evals_since_order >= 32)) {
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
      vgx_launch_reg_reduce(st, g->d_cons, g->d_poses, g->d_tiles, g->n_tiles, g->d_tile_order,
                            g->d_tile_cost, g->d_partials, g->grid_capacity, g->d_unit_bounds, jacobian, skip);
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
  VgxPdlLaunch L(st, dim3(1), dim3(128));
  const int excl = do_reg ? 0 : 1;
  if (do_reg) {
    RegSums sums;
    sums.partials = g->d_partials; sums.tile_begin = g->d_tile_begin; sums.cons = g->d_cons;
    VgxLaunchScope s(c, 7);
    L.cfg.gridDim = dim3((unsigned)((g->n_local + 3) / 4));
    cudaLaunchKernelEx(&L.cfg, reg_csum_kernel, sums, g->n_local, g->d_csum, skip);
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
      L.cfg.gridDim = dim3((unsigned)grid);
      cudaLaunchKernelEx(&L.cfg, assemble_exchange_kernel, (const double*)g->d_csum, (const VgxRelEdge*)g->d_rel, d_x,
                         (const int*)g->d_csr_begin, (const int4*)g->d_csr_items, push, g->N, g->E, g->n_local,
                         g->n_rel_local, excl, gat, d_packed, (int)g->packed_len, skip,
                         (const unsigned char*)g->d_block_mask);
    }
    VGX_CUDA(c, cudaGetLastError());
    return VGX_OK;
  }
  {
    VgxLaunchScope s(c, 8);
    L.cfg.gridDim = dim3((unsigned)(g->N + g->E + 1));
    cudaLaunchKernelEx(&L.cfg, assemble_kernel, (const double*)g->d_csum, (const VgxRelEdge*)g->d_rel, d_x, (const int*)g->d_csr_begin,
                       (const int4*)g->d_csr_items, push, g->N, g->E, g->n_local, g->n_rel_local, excl, skip);
  }
  VGX_CUDA(c, cudaGetLastError());
  if (p2p) return vgx_p2p_gather(c, gat, d_packed, g->packed_len, g->d_block_mask, g->N);
  return vgx_nccl_allreduce_sum_f64(c, d_packed, g->packed_len);
}

int prepare(vgx_ctx* c, VgxGraph** out) {
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

