// Pose-graph state shared by the evaluation pipeline (graph.cu) and the dense solver (solve.cu).
#pragma once

#include "registration_kernels.h"

// Packed normal equations, the output of one evaluation (doubles):
//   [PACK_HDR header: [0] cost, [1..3] reserved | 4 N gradient, node-major |
//    16 N diagonal 4x4 blocks, row-major, node order |
//    16 E off-diagonal 4x4 blocks, row-major: rows node block_nodes[2b] (the smaller index), cols block_nodes[2b + 1]]
#define PACK_HDR 4

struct LmState {
  double radius, decrease_factor;
  double cost, cand_cost, model_cost_change;
  double x_norm, step_norm, gmax;
  int reuse_diagonal, consecutive_invalid;
  int iterations, successful, evals;
  int termination, done, accepted, step_valid, scale_ready;
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
  std::vector<int> red;    // N: reduced offset or -1 (host copy of d_red_offset)
  int n_local = 0, n_tiles = 0, n_rel_local = 0, grid_capacity = 0;
  int E = 0;               // off-diagonal blocks
  int n_free = 0;          // reduced dimension 4 * (non-constant nodes)
  int64_t residuals_local = 0, residuals_global = 0;
  bool zero_weight = false;
  size_t packed_len = 0;

  // device
  RegConstraintDev* d_cons = nullptr;
  RegPoseConst* d_poses = nullptr;
  RegTile* d_tiles = nullptr;
  float4* d_unit_bounds = nullptr;   // bounding sphere per 32-point unit of the tiles (RegTile::unit0)
  int* d_tile_begin = nullptr;
  double* d_partials = nullptr;
  double* d_csum = nullptr;
  VgxRelEdge* d_rel = nullptr;
  unsigned char* d_block_mask = nullptr;   // per output block: bit r = rank r contributes (peer exchange)
  int* d_tile_order = nullptr;  // CTA b of the reduce kernel runs tile d_tile_order[b] (longest first)
  int* d_tile_cost = nullptr;   // SM cycles each tile took in the latest evaluation
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

__device__ __forceinline__ double normalize_angle(double a) {
  const double two_pi = 6.283185307179586476925286766559;
  return a - two_pi * floor((a + 3.14159265358979323846) / two_pi);
}

// graph.cu: the tables (rebuilt when the graph changed) and one evaluation of the packed normal
// equations at the poses d_x into d_packed (skip: device flag, the launches return at once when set)
int prepare(vgx_ctx* c, VgxGraph** out);
int eval_enqueue(vgx_ctx* c, VgxGraph* g, const double* d_x, double* d_packed, bool jacobian, bool exclude_reg,
                 const int* skip = nullptr);
