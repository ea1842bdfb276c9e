// Host-visible declarations of the registration kernels (registration.cu).
#pragma once

#include "graph_plan.h"   // the tile constants
#include "vgx_internal.h"

struct RegConstraintDev;
struct RegPoseConst;

#define VGX_REG_THREADS 128        // 4 warps per CTA, each with its own TMA ring + software pipeline
#define VGX_REG_MIN_BLOCKS 8       // resident CTAs per SM the register budget is sized for (64 registers)
#define VGX_REG_RING 4             // point-slice ring slots per warp (units in flight = RING - 1)
#define VGX_REG_NSUM 21            // 15 (upper 5x5) + 5 (gradient) + 1 (cost)
#define VGX_REG_NSTRIDE 24

struct __align__(16) RegTile {   // 32 bytes: everything a CTA needs to start its bulk copies
  int constraint;
  int unit0;                 // index of the tile's first unit in the unit-bound table
  int count;
  int grid_bytes;            // bytes of the 16-bit block grid to stage (multiple of 16), 0: hash path
  const float* pts;          // first unit of the tile (unit-major points)
  const uint16_t* grid16;
};

// skip (device flag, may be null): when set, the kernel returns at once (an evaluation enqueued
// ahead of a solve that has ended in the meantime)
int vgx_launch_reg_pose_setup(vgx_ctx* c, const RegConstraintDev* cons, const double* x, RegPoseConst* poses, int n,
                              const int* skip = nullptr);
// One CTA per tile, CTA b running tile tile_order[b] -> partials[tile][21] and tile_cost[tile]; the
// consumer adds a constraint's tiles in tile order (graph.cu: reg_csum_kernel).  unit_bounds (may be
// null: no culling): the table vgx_launch_reg_unit_bounds fills, indexed by RegTile::unit0 + unit.
int vgx_launch_reg_reduce(vgx_ctx* c, const RegConstraintDev* cons, const RegPoseConst* poses, const RegTile* tiles,
                          int n_tiles, const int* tile_order, int* tile_cost, double* partials, int grid_capacity,
                          const float4* unit_bounds, bool jacobian, const int* skip = nullptr);
// bounds[tile.unit0 + u] <- a sphere (centre xyz, radius w) around the points of unit u of every tile
// that can contribute (radius +inf: the unit is never culled)
int vgx_launch_reg_unit_bounds(vgx_ctx* c, const RegTile* tiles, int n_tiles, float4* bounds);
// tile_order <- tiles sorted by measured cost, most expensive first
int vgx_launch_reg_order(vgx_ctx* c, const int* tile_cost, int n_tiles, int* tile_order);
// Fills the descriptor of one (reference -> reading) residual block.  Deterministic mode: pts / n /
// factor describe all registration points.  Sampling mode (*sampled = true): n = int(ratio * K),
// factor = 1 (all weights forced to 1) and pts is left null for the caller, who draws the
// indices (vgx_points_draw) and gathers them (vgx_launch_reg_gather_samples).
int vgx_fill_constraint(vgx_ctx* c, uint32_t ref_id, uint32_t read_id, const vgx_reg_config* cfg,
                        RegConstraintDev* out, bool* sampled = nullptr);
// dst (unit-major, ceil(n/32) units) <- the n points of src selected by d_idx, weight forced to 1
int vgx_launch_reg_gather_samples(vgx_ctx* c, const float* src, const int32_t* d_idx, int n, float* dst);
