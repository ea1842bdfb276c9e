// Pose-graph state shared by the evaluation pipeline (graph.cu) and the dense solver (solve.cu).
#pragma once

#include "graph_plan.h"
#include "registration_kernels.h"

struct LmState {
  double radius, decrease_factor;
  double cost, cand_cost, model_cost_change;
  double x_norm, step_norm, gmax;
  int reuse_diagonal, consecutive_invalid;
  int iterations, successful, evals;
  int termination, done, accepted, step_valid, scale_ready;
};

// The device buffers of one table build, and the state that belongs to them: all of it is released when the
// tables are rebuilt.
struct VgxGraphTables {
  VgxBuffer<RegConstraintDev> d_cons;
  VgxBuffer<RegPoseConst> d_poses;
  VgxBuffer<RegTile> d_tiles;
  VgxBuffer<float4> d_unit_bounds;   // bounding sphere per 32-point unit of the tiles (RegTile::unit0)
  VgxBuffer<int> d_tile_begin;
  VgxBuffer<double> d_partials;
  VgxBuffer<double> d_csum;
  VgxBuffer<VgxRelEdge> d_rel;
  VgxBuffer<unsigned char> d_block_mask;   // per output block: bit r = rank r contributes (peer exchange)
  VgxBuffer<int> d_tile_order;  // CTA b of the reduce kernel runs tile d_tile_order[b] (longest first)
  VgxBuffer<int> d_tile_cost;   // SM cycles each tile took in the latest evaluation
  VgxBuffer<int> d_csr_begin;   // N + E + 1
  VgxBuffer<int4> d_csr_items;  // (source, role, first tile, end tile)
  VgxBuffer<int> d_block_nodes; // E x 2
  VgxBuffer<int> d_red_offset;  // N: reduced offset or -1
  VgxBuffer<double> d_x;
  VgxBuffer<double> d_xc;
  VgxBuffer<double> d_packed[2];
  VgxBuffer<double> d_A;
  VgxBuffer<double> d_scale;
  VgxBuffer<double> d_diag;
  VgxBuffer<double> d_gs;
  VgxBuffer<double> d_step;
  VgxBuffer<LmState> d_state;
  VgxBuffer<LmState> d_snap;    // [2] outcome of iteration k (written by lm_decide), parity k & 1
  VgxBuffer<float> d_sample_pts;   // gathered unit-major points of the local sampled blocks
  VgxBuffer<int32_t> d_sample_idx;
  int evals_since_order = -1;   // -1: no cost measured yet since the tables were built
  int exchange_grid = 0;        // CTAs of the fused assembly and exchange: all co-resident on this device
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

  // derived, by the table build
  bool zero_weight = false;       // some registration constraint has no points or zero weight
  int64_t residuals_global = 0;
  VgxGraphPlan plan;              // the layout, host copy
  VgxGraphTables dev;
  // pinned; they outlive the tables: a page-locked allocation costs ~0.2 ms
  VgxBuffer<LmState> h_state{VgxMem::pinned};
  VgxBuffer<LmState> h_snap{VgxMem::pinned};    // [2]
  VgxBuffer<double> h_x{VgxMem::pinned};        // 4 x (at least N)
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ev_iter[2] = {nullptr, nullptr}, ev_copy[2] = {nullptr, nullptr};
};

__device__ __forceinline__ double normalize_angle(double a) {
  const double two_pi = 6.283185307179586476925286766559;
  return a - two_pi * floor((a + 3.14159265358979323846) / two_pi);
}

// graph.cu: the tables (rebuilt when the graph changed) and one evaluation of the packed normal
// equations at the poses d_x into d_packed (skip: device flag, the launches return at once when set)
int prepare(vgx_ctx* c, VgxGraph** out);
int eval_enqueue(vgx_ctx* c, VgxGraph* g, const double* d_x, double* d_packed, bool jacobian, bool exclude_reg,
                 const int* skip = nullptr);
