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
#include <numeric>

#include "graph.h"
#include "registration.cuh"
#include "registration_kernels.h"

void vgx_graph_free(vgx_ctx* c) {
  if (!c->graph) return;
  vgx_drain(c);
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
  if (!c->graph) c->graph = new VgxGraph();
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

// Per-constraint sums csum[c][21] from the tile rows: one warp per constraint, a programmatic
// dependent of the reduce kernel (and the assembly kernel is one of this).  A separate, massively
// parallel stage: inside the assembly the same loop is a chain of dependent L2 latencies per item.
// The tiles are added in tile-index order, never in completion order: every evaluation at the same
// poses is bit-identical, which the parity tests and bench.py --dump-outputs rely on.
__global__ void __launch_bounds__(128)
reg_csum_kernel(RegSums R, int n, double* __restrict__ csum, const int* __restrict__ skip) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  const bool active = c < n && lane < VGX_REG_NSUM;
  // the tile range and factor are tables built with the graph: read before the wait
  int t0 = 0, t1 = 0;
  double f = 0.0;
  if (active) { t0 = __ldg(R.tile_begin + c); t1 = __ldg(R.tile_begin + c + 1); f = __ldg(&R.cons[c].factor); }
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (skip && *skip) return;
  if (active) csum[(size_t)c * VGX_REG_NSTRIDE + lane] = reg_tile_sum(R.partials, t0, t1, lane) * (f * f);
}

// Single-rank assembly: wait for the constraint sums (programmatic dependent of the constraint-sum
// kernel, itself one of the reduce kernel), then let the next evaluation's pose set-up be scheduled.
__device__ __forceinline__ void vgx_assemble_wait() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
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
                                               int n_rel, int exclude_reg, double (*s_part)[20],
                                               bool wait) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (ob == N + E) {
    if (wait) vgx_assemble_wait();
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
  const int i0 = __ldg(csr_begin + ob), i1 = __ldg(csr_begin + ob + 1);
  // the CSR and its items are tables built with the graph: this warp's first two items are read
  // before the wait, the next trip's during the current one
  int4 nA = make_int4(-1, 0, 0, 0), nB = make_int4(-1, 0, 0, 0);
  if (i0 + warp < i1) nA = __ldg(items + i0 + warp);
  if (i0 + warp + 4 < i1) nB = __ldg(items + i0 + warp + 4);
  if (wait) vgx_assemble_wait();
  // peer exchange: a block this rank has nothing for is not pushed (the receivers know from the
  // block's rank mask that this slot holds no value of this epoch)
  if (push.tag != 0 && i0 == i1) return;
  const bool diag = ob < N;
  const int r4 = (lane >> 2) & 3, c4 = lane & 3;
  double acc = 0;
  // warp w expands items w, w + 4, ... in list order; two items per trip so their loads overlap
  for (int i = i0 + warp; i < i1; i += 8) {
    const bool two = i + 4 < i1;
    const int4 itA = nA;
    const int4 itB = two ? nB : make_int4(-1, 0, 0, 0);
    if (i + 8 < i1) nA = __ldg(items + i + 8);
    if (i + 12 < i1) nB = __ldg(items + i + 12);
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
  // scheduled while the constraint-sum grid drains; assemble_block reads this block's CSR range and
  // first items, then blocks in vgx_assemble_wait until the sums are visible
  assemble_block(blockIdx.x, csum, rel, x, csr_begin, items, push, N, E, n_reg, n_rel, exclude_reg, s_part, true);
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
    assemble_block(ob, csum, rel, x, csr_begin, items, push, N, E, n_reg, n_rel, exclude_reg, s_part, false);
  vgx_ll_gather(gat, out, (size_t)count, (size_t)blockIdx.x * blockDim.x + threadIdx.x,
                (size_t)gridDim.x * blockDim.x, block_mask, N);
}

// ------------------------------------------------------------------ host only: sharding, square-root information
extern "C" int vgx_shard_constraints(int nranks, int n, const int32_t* num_residuals,
                                     const uint32_t* locality_keys, int32_t* owner) {
  return vgx_entry_noctx([&] {
    if (nranks < 1 || n < 0 || (n > 0 && (!num_residuals || !owner))) return VGX_ERR_INVALID;
    vgx_partition_constraints(nranks, n, num_residuals, locality_keys, owner);
    return VGX_OK;
  });
}

extern "C" int vgx_sqrt_information(const double information[16], int allow_semi_definite,
                                    double sqrt_information[16]) {
  return vgx_entry_noctx([&] {
    if (!information || !sqrt_information) return VGX_ERR_INVALID;
    return vgx_sqrt_information_factor(information, allow_semi_definite != 0, sqrt_information) ? VGX_OK
                                                                                                : VGX_ERR_INVALID;
  });
}

// ------------------------------------------------------------------ table construction
// A build collects the constraints, plans the layout (graph_plan.cpp) and uploads the plan.

// d <- n elements of T (at least 8 bytes: an empty table has an address too)
template <class T>
static int table_alloc(vgx_ctx* c, VgxBuffer<T>& d, size_t n) {
  return d.alloc(c, std::max<size_t>(sizeof(T) * n, 8), "graph table build", VGX_ERR_NOMEM);
}

// d <- a copy of v
template <class T>
static int table_upload(vgx_ctx* c, VgxBuffer<T>& d, const std::vector<T>& v) {
  VGX_TRY(table_alloc(c, d, std::max<size_t>(v.size(), 1)));
  return v.empty() ? VGX_OK : vgx_upload(c, d.get(), v.data(), v.size());
}

// The device tables of `plan`; all[i] is the descriptor of constraint i, is_sampled[i] whether its points are the
// draws in g->samples[i].  Every buffer is t's, so a failure leaves nothing behind.
static int upload_tables(vgx_ctx* c, VgxGraph* g, const VgxGraphPlan& plan, const std::vector<RegConstraintDev>& all,
                         const std::vector<uint8_t>& is_sampled, int sms, VgxGraphTables& t) {
  const int N = g->N, n_local = plan.n_local(), n_tiles = plan.n_tiles(), n = plan.n_free;
  std::vector<RegConstraintDev> cons(n_local);
  for (int k = 0; k < n_local; ++k) cons[k] = all[plan.local[k]];
  // gather the drawn points of the local sampled blocks into their own unit-major buffers
  size_t units = 0, nidx = 0;
  for (int k = 0; k < n_local; ++k)
    if (is_sampled[plan.local[k]]) { units += ((size_t)cons[k].n + 31) / 32; nidx += (size_t)cons[k].n; }
  if (units > 0) {
    VGX_TRY(t.d_sample_pts.alloc(c, units * VGX_PT_UNIT_FLOATS * sizeof(float), "registration sample points"));
    VGX_TRY(t.d_sample_idx.alloc(c, nidx * sizeof(int32_t), "registration sample points"));
    size_t uo = 0, io = 0;
    for (int k = 0; k < n_local; ++k) {
      const int i = plan.local[k];
      if (!is_sampled[i]) continue;
      const VgxPoints& p = c->find(g->reg_ref[i])->points[g->reg_cfgs[i].registration_point_type];
      VGX_TRY(vgx_upload(c, t.d_sample_idx.get() + io, g->samples[i].data(), (size_t)cons[k].n));
      float* dst = t.d_sample_pts.get() + uo * VGX_PT_UNIT_FLOATS;
      VGX_TRY(vgx_launch_reg_gather_samples(c, p.data.get(), t.d_sample_idx.get() + io, cons[k].n, dst));
      cons[k].pts = dst;
      uo += ((size_t)cons[k].n + 31) / 32;
      io += (size_t)cons[k].n;
    }
    VGX_TRY(vgx_sync(c));  // g->samples[] are pageable host vectors
  }
  // what the CTA of a tile needs to start its bulk copies without a dependent load
  std::vector<RegTile> tiles(n_tiles);
  for (int j = 0; j < n_tiles; ++j) {
    const VgxPlanTile& pt = plan.tiles[j];
    const RegConstraintDev& cc = cons[pt.constraint];
    tiles[j].constraint = pt.constraint;
    tiles[j].unit0 = pt.unit0;
    tiles[j].count = pt.count;
    tiles[j].grid_bytes = pt.grid_bytes;
    tiles[j].pts = cc.pts + (size_t)(pt.first / VGX_REG_UNIT) * VGX_PT_UNIT_FLOATS;
    tiles[j].grid16 = cc.grid16;
  }
  std::vector<int> ident(n_tiles), zero(n_tiles, 0);
  std::iota(ident.begin(), ident.end(), 0);
  VGX_TRY(table_upload(c, t.d_cons, cons));
  VGX_TRY(table_upload(c, t.d_tiles, tiles));
  VGX_TRY(table_upload(c, t.d_tile_begin, plan.tile_begin));
  VGX_TRY(table_upload(c, t.d_tile_order, ident));
  VGX_TRY(table_upload(c, t.d_tile_cost, zero));
  VGX_TRY(table_upload(c, t.d_rel, g->rel));
  VGX_TRY(table_upload(c, t.d_csr_begin, plan.csr_begin));
  VGX_TRY(table_upload(c, t.d_csr_items, plan.items));
  VGX_TRY(table_upload(c, t.d_block_mask, plan.block_mask));
  VGX_TRY(table_upload(c, t.d_block_nodes, plan.block_nodes));
  VGX_TRY(table_upload(c, t.d_red_offset, plan.red));
  VGX_TRY(table_upload(c, t.d_x, g->x));
  VGX_TRY(table_alloc(c, t.d_unit_bounds, plan.n_units));
  VGX_TRY(vgx_launch_reg_unit_bounds(c, t.d_tiles.get(), n_tiles, t.d_unit_bounds.get()));
  VGX_TRY(table_alloc(c, t.d_poses, n_local));
  VGX_TRY(table_alloc(c, t.d_partials, VGX_REG_NSTRIDE * (size_t)n_tiles));
  VGX_TRY(table_alloc(c, t.d_csum, VGX_REG_NSTRIDE * (size_t)n_local));
  VGX_TRY(table_alloc(c, t.d_xc, 4 * (size_t)N));
  VGX_TRY(table_alloc(c, t.d_packed[0], plan.packed_len));
  VGX_TRY(table_alloc(c, t.d_packed[1], plan.packed_len));
  VGX_TRY(table_alloc(c, t.d_A, (size_t)(n + 1) * (n + 1)));
  VGX_TRY(table_alloc(c, t.d_scale, n));
  VGX_TRY(table_alloc(c, t.d_diag, n));
  VGX_TRY(table_alloc(c, t.d_gs, n));
  VGX_TRY(table_alloc(c, t.d_step, n));
  VGX_TRY(table_alloc(c, t.d_state, 1));
  const char* what = "graph table build";
  if (!g->h_state.get()) VGX_TRY(g->h_state.alloc(c, sizeof(LmState), what, VGX_ERR_NOMEM));
  VGX_TRY(table_alloc(c, t.d_snap, 2));
  if (!g->h_snap.get()) VGX_TRY(g->h_snap.alloc(c, 2 * sizeof(LmState), what, VGX_ERR_NOMEM));
  if (g->h_x.bytes() < sizeof(double) * 4 * (size_t)N)
    VGX_TRY(g->h_x.alloc(c, sizeof(double) * 4 * (size_t)std::max(2 * N, 64), what, VGX_ERR_NOMEM));
  if (!g->copy_stream) {
    VGX_CUDA(c, cudaStreamCreateWithFlags(&g->copy_stream, cudaStreamNonBlocking));
    for (int k = 0; k < 2; ++k) {
      VGX_CUDA(c, cudaEventCreateWithFlags(&g->ev_iter[k], cudaEventDisableTiming));
      VGX_CUDA(c, cudaEventCreateWithFlags(&g->ev_copy[k], cudaEventDisableTiming));
    }
  }
  VGX_TRY(vgx_sync(c));
  // the fused assembly and exchange spins on its peers, so its grid must be co-resident as a whole
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, assemble_exchange_kernel, 128, 0) != cudaSuccess)
    per_sm = 1;
  t.exchange_grid = std::min(N + plan.E + 1, std::max(1, sms * std::max(per_sm, 1)));
  return VGX_OK;
}

static int build_tables(vgx_ctx* c, VgxGraph* g) {
  VGX_TRY(vgx_sync(c));
  g->dev = VgxGraphTables();   // before the new tables are allocated: a rebuild needs no more device memory
  // ---- collect: the descriptors, nodes and sampling draws of all constraints, and their partition over ranks
  const int P = (int)g->reg_ref.size();
  std::vector<RegConstraintDev> all(P);
  std::vector<VgxPlanConstraint> facts(P);
  std::vector<uint8_t> is_sampled(P, 0);
  std::vector<int32_t> counts(P), owner(P, 0);
  g->zero_weight = false;
  g->residuals_global = 0;
  g->samples.assign(P, std::vector<int32_t>());
  g->sample_override.resize(P);
  for (int i = 0; i < P; ++i) {
    bool sampled = false;
    VGX_TRY(vgx_fill_constraint(c, g->reg_ref[i], g->reg_read[i], &g->reg_cfgs[i], &all[i], &sampled));
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
          if (v < 0 || v >= p.n) VGX_FAIL(c, VGX_ERR_INVALID, "sample index out of range");
      } else {
        g->samples[i].resize(all[i].n);
        vgx_points_draw(p, all[i].n, g->samples[i].data());
      }
    }
    const RegConstraintDev& cc = all[i];
    facts[i] = {cc.n, cc.ref_node, cc.read_node, cc.gd0 * cc.gd1 * cc.gd2, cc.grid16 != nullptr};
    counts[i] = cc.n;
  }
  vgx_partition_constraints(c->nranks, P, counts.data(), g->reg_read.data(), owner.data());
  // ---- plan
  std::vector<int2> rel(g->rel.size());
  for (size_t e = 0; e < rel.size(); ++e) rel[e] = make_int2(g->rel[e].a, g->rel[e].b);
  int sms = 132;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device);
  const char* tile_units = getenv("VGX_REG_HW_TILE_UNITS");
  VgxGraphPlan plan = vgx_graph_plan(facts, owner, rel, g->N, g->constant, c->rank, sms,
                                     tile_units ? atoi(tile_units) : 0);
  // ---- upload
  VgxGraphTables t;
  VGX_TRY(upload_tables(c, g, plan, all, is_sampled, sms, t));
  g->plan = std::move(plan);
  g->dev = std::move(t);
  g->dirty = false;
  return VGX_OK;
}

// ------------------------------------------------------------------ evaluation pipeline
int eval_enqueue(vgx_ctx* c, VgxGraph* g, const double* d_x, double* d_packed, bool jacobian, bool exclude_reg,
                 const int* skip) {
  const VgxGraphPlan& plan = g->plan;
  VgxGraphTables& dev = g->dev;
  const bool do_reg = !exclude_reg && plan.n_local() > 0;
  if (do_reg) {
    // refresh the longest-first tile order from the cost measured by the previous evaluation: before
    // the second evaluation on new tables, then every 32nd (the poses move little inside a solve)
    if (plan.n_tiles() > 1 && (dev.evals_since_order == -2 || dev.evals_since_order >= 32)) {
      VgxProfileScope s(c, VGX_SLOT_OTHER);
      VGX_TRY(vgx_launch_reg_order(c, dev.d_tile_cost.get(), plan.n_tiles(), dev.d_tile_order.get()));
      dev.evals_since_order = 0;
    }
    if (dev.evals_since_order >= 0) ++dev.evals_since_order;
    {
      VgxProfileScope s(c, VGX_SLOT_REG_POSE_SETUP);
      VGX_TRY(vgx_launch_reg_pose_setup(c, dev.d_cons.get(), d_x, dev.d_poses.get(), plan.n_local(), skip));
    }
    {
      VgxProfileScope s(c, VGX_SLOT_REG_REDUCE);
      VGX_TRY(vgx_launch_reg_reduce(c, dev.d_cons.get(), dev.d_poses.get(), dev.d_tiles.get(), plan.n_tiles(),
                                    dev.d_tile_order.get(), dev.d_tile_cost.get(), dev.d_partials.get(),
                                    plan.grid_capacity, dev.d_unit_bounds.get(), jacobian, skip));
    }
    if (dev.evals_since_order < 0) dev.evals_since_order = -2;   // a cost has been measured now
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
  const int excl = do_reg ? 0 : 1;
  if (do_reg) {
    RegSums sums;
    sums.partials = dev.d_partials.get(); sums.tile_begin = dev.d_tile_begin.get();
    sums.cons = dev.d_cons.get();
    VgxProfileScope s(c, VGX_SLOT_REG_SUMS);
    VGX_TRY(vgx_launch(c, reg_csum_kernel, (unsigned)((plan.n_local() + 3) / 4), 128, 0, VgxLaunch::pdl, sums,
                       plan.n_local(), dev.d_csum.get(), skip));
  }
  if (p2p) {
    VGX_TRY(vgx_p2p_begin(c, plan.packed_len, &push, &gat));
  }
  if (p2p && c->p2p_fused && plan.packed_len < (size_t)INT_MAX) {
    // one launch: assemble + push -> signal -> wait -> local reduce (grid fully co-resident)
    VgxProfileScope s(c, VGX_SLOT_ASSEMBLY);
    return vgx_launch(c, assemble_exchange_kernel, (unsigned)dev.exchange_grid, 128, 0, VgxLaunch::pdl,
                      (const double*)dev.d_csum.get(), (const VgxRelEdge*)dev.d_rel.get(), d_x,
                      (const int*)dev.d_csr_begin.get(), (const int4*)dev.d_csr_items.get(), push, g->N, plan.E,
                      plan.n_local(), plan.n_rel_local, excl, gat, d_packed, (int)plan.packed_len, skip,
                      (const unsigned char*)dev.d_block_mask.get());
  }
  {
    VgxProfileScope s(c, VGX_SLOT_ASSEMBLY);
    VGX_TRY(vgx_launch(c, assemble_kernel, (unsigned)(g->N + plan.E + 1), 128, 0, VgxLaunch::pdl,
                       (const double*)dev.d_csum.get(), (const VgxRelEdge*)dev.d_rel.get(), d_x,
                       (const int*)dev.d_csr_begin.get(), (const int4*)dev.d_csr_items.get(), push, g->N, plan.E,
                       plan.n_local(), plan.n_rel_local, excl, skip));
  }
  if (p2p) return vgx_p2p_gather(c, gat, d_packed, plan.packed_len, dev.d_block_mask.get(), g->N);
  return vgx_nccl_allreduce_sum_f64(c, d_packed, plan.packed_len);
}

int prepare(vgx_ctx* c, VgxGraph** out) {
  VgxGraph* g = graph_of(c);
  if (g->N == 0) VGX_FAIL(c, VGX_ERR_INVALID, "pose graph has no nodes");
  if (g->dirty) {
    VGX_TRY(build_tables(c, g));
  }
  *out = g;
  return VGX_OK;
}

// ------------------------------------------------------------------ C-ABI: b2
extern "C" int vgx_graph_set_nodes(vgx_ctx* c, int n, const uint32_t* ids, const double* xyzyaw,
                                   const uint8_t* constant) {
  return vgx_entry(c, __func__, [&] {
    if (n < 0 || (n > 0 && (!ids || !xyzyaw))) return VGX_ERR_INVALID;
    VgxGraph* g = graph_of(c);
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
  });
}

extern "C" int vgx_graph_set_poses(vgx_ctx* c, const double* xyzyaw) {
  return vgx_entry(c, __func__, [&] {
    if (!xyzyaw) return VGX_ERR_INVALID;
    VgxGraph* g = graph_of(c);
    if (g->N == 0) VGX_FAIL(c, VGX_ERR_INVALID, "pose graph has no nodes");
    g->x.assign(xyzyaw, xyzyaw + 4 * (size_t)g->N);
    if (!g->dirty) {
      // stage through pinned memory so the copy is a true async H2D
      double* h;
      VGX_TRY(vgx_carve(c, c->h_pinned, vgx_part(h, 4 * (size_t)g->N)));
      VGX_TRY(vgx_sync(c));
      memcpy(h, xyzyaw, sizeof(double) * 4 * g->N);
      return vgx_upload(c, g->dev.d_x.get(), h, 4 * (size_t)g->N);
    }
    return VGX_OK;
  });
}

extern "C" int vgx_graph_get_poses(vgx_ctx* c, double* xyzyaw) {
  return vgx_entry(c, __func__, [&] {
    if (!xyzyaw) return VGX_ERR_INVALID;
    VgxGraph* g = graph_of(c);
    memcpy(xyzyaw, g->x.data(), sizeof(double) * 4 * g->N);
    return VGX_OK;
  });
}

extern "C" int vgx_graph_set_relative_edges(vgx_ctx* c, int m, const uint32_t* ids_a,
                                            const uint32_t* ids_b, const double* t_obs,
                                            const double* sqrt_info) {
  return vgx_entry(c, __func__, [&] {
    if (m < 0 || (m > 0 && (!ids_a || !ids_b || !t_obs || !sqrt_info))) return VGX_ERR_INVALID;
    VgxGraph* g = graph_of(c);
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
  });
}

static int set_registration(vgx_ctx* c, int p, const uint32_t* ref_ids, const uint32_t* read_ids,
                            const vgx_reg_config* cfgs, bool per_constraint) {
  if (p < 0 || (p > 0 && (!ref_ids || !read_ids))) return VGX_ERR_INVALID;
  if (per_constraint && p > 0 && !cfgs) return VGX_ERR_INVALID;
  VgxGraph* g = graph_of(c);
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
  return vgx_entry(c, __func__, [&] { return set_registration(c, p, ref_ids, read_ids, cfg, false); });
}

extern "C" int vgx_graph_set_registration_constraints_v(vgx_ctx* c, int p, const uint32_t* ref_ids,
                                                        const uint32_t* read_ids,
                                                        const vgx_reg_config* cfgs) {
  return vgx_entry(c, __func__, [&] { return set_registration(c, p, ref_ids, read_ids, cfgs, true); });
}

extern "C" int vgx_graph_set_sample_indices(vgx_ctx* c, int constraint, int n, const int32_t* indices) {
  return vgx_entry(c, __func__, [&] {
    VgxGraph* g = graph_of(c);
    if (constraint < 0 || constraint >= (int)g->reg_ref.size() || n < 0 || (n > 0 && !indices))
      VGX_FAIL(c, VGX_ERR_INVALID, "invalid argument");
    if (g->reg_cfgs[constraint].sampling_ratio == -1.0f)
      VGX_FAIL(c, VGX_ERR_INVALID, "the constraint is not in sampling mode");
    g->sample_override.resize(g->reg_ref.size());
    g->sample_override[constraint].assign(indices, indices + n);
    g->dirty = true;
    return VGX_OK;
  });
}

extern "C" int vgx_graph_num_registration_residuals(vgx_ctx* c, int64_t* local, int64_t* global) {
  return vgx_entry(c, __func__, [&] {
    VgxGraph* g = nullptr;
    VGX_TRY(prepare(c, &g));
    if (local) *local = g->plan.residuals_local;
    if (global) *global = g->residuals_global;
    return VGX_OK;
  });
}

extern "C" int vgx_graph_get_sample_indices(vgx_ctx* c, int constraint, int max_n, int32_t* indices, int* n) {
  return vgx_entry(c, __func__, [&] {
    VgxGraph* g = nullptr;
    VGX_TRY(prepare(c, &g));
    if (constraint < 0 || constraint >= (int)g->samples.size())
      VGX_FAIL(c, VGX_ERR_INVALID, "invalid constraint index");
    const std::vector<int32_t>& v = g->samples[constraint];
    if (n) *n = (int)v.size();
    if ((int)v.size() > max_n) VGX_FAIL(c, VGX_ERR_CAPACITY, "max_n too small");
    if (indices && !v.empty()) memcpy(indices, v.data(), sizeof(int32_t) * v.size());
    return VGX_OK;
  });
}

extern "C" int vgx_graph_eval_async(vgx_ctx* c, int exclude_registration) {
  return vgx_entry(c, __func__, [&] {
    VgxGraph* g = nullptr;
    VGX_TRY(prepare(c, &g));
    return eval_enqueue(c, g, g->dev.d_x.get(), g->dev.d_packed[0].get(), true, exclude_registration != 0);
  });
}

extern "C" int vgx_graph_eval(vgx_ctx* c, int exclude_registration, double* cost, double* gradient,
                              double* H) {
  return vgx_entry(c, __func__, [&] {
    VgxGraph* g = nullptr;
    VGX_TRY(prepare(c, &g));
    VGX_TRY(eval_enqueue(c, g, g->dev.d_x.get(), g->dev.d_packed[0].get(), true, exclude_registration != 0));
    double* h;
    VGX_TRY(vgx_carve(c, c->h_pinned, vgx_part(h, g->plan.packed_len)));
    VGX_TRY(vgx_read(c, h, g->dev.d_packed[0].get(), g->plan.packed_len));
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
      const std::vector<int>& bn = g->plan.block_nodes;
      for (int b = 0; b < g->plan.E; ++b) {
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
      VGX_TRY(vgx_p2p_check(c));
    }
    if (!exclude_registration && g->zero_weight) return VGX_ZERO_WEIGHT;
    return VGX_OK;
  });
}

extern "C" int vgx_graph_registration_costs(vgx_ctx* c, double* per_constraint) {
  return vgx_entry(c, __func__, [&] {
    VgxGraph* g = nullptr;
    VGX_TRY(prepare(c, &g));
    if (!per_constraint) return VGX_ERR_INVALID;
    VGX_TRY(eval_enqueue(c, g, g->dev.d_x.get(), g->dev.d_packed[1].get(), false, false));
    const int P = (int)g->reg_ref.size(), n_local = g->plan.n_local();
    std::vector<double> cs((size_t)n_local * VGX_REG_NSTRIDE + 1);
    if (n_local > 0) VGX_TRY(vgx_download(c, cs.data(), g->dev.d_csum.get(), VGX_REG_NSTRIDE * (size_t)n_local));
    VGX_TRY(vgx_sync(c));
    for (int i = 0; i < P; ++i) per_constraint[i] = 0.0;
    for (int k = 0; k < n_local; ++k) per_constraint[g->plan.local[k]] = cs[(size_t)k * VGX_REG_NSTRIDE + 20];
    return VGX_OK;
  });
}
