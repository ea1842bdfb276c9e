// Host-visible declarations of the registration kernels (registration.cu).
#pragma once

#include "vgx_internal.h"

struct RegConstraintDev;
struct RegPoseConst;

#ifndef VGX_REG_THREADS
#define VGX_REG_THREADS 128        // 4 warps per CTA, each with its own TMA ring + software pipeline
#endif
#ifndef VGX_REG_MIN_BLOCKS
#define VGX_REG_MIN_BLOCKS 6       // resident CTAs per SM the register budget is sized for (80 registers;
                                   // sm_90a spills at the 72 that 7 would allow, for the same step time)
#endif
#ifndef VGX_REG_RING
#define VGX_REG_RING 4             // point-slice ring slots per warp (units in flight = RING - 1)
#endif
#ifndef VGX_REG_EARLYOUT
#define VGX_REG_EARLYOUT 1         // a warp whose 32 points all miss the containing block skips the unit
#endif
#ifndef VGX_REG_SKIPGRAM
#define VGX_REG_SKIPGRAM 1         // no Gram stage for a unit without a single correspondence
#endif
#ifndef VGX_REG_HW_TILE_UNITS
#define VGX_REG_HW_TILE_UNITS 64   // > 0: one CTA per tile of that many units (hardware scheduling); 0: persistent
#endif
#define VGX_REG_UNIT 32            // points per unit = one warp iteration; tiles are cut on unit boundaries
#ifndef VGX_REG_STREAM_OCTETS
#define VGX_REG_STREAM_OCTETS 0   // ld.global.cs for the octet fetch
#endif
#define VGX_REG_NSUM 21            // 15 (upper 5x5) + 5 (gradient) + 1 (cost)
#define VGX_REG_NSTRIDE 24

struct __align__(16) RegTile {   // 32 bytes: everything a CTA needs to start its bulk copies
  int constraint;
  int start;
  int count;
  int grid_bytes;            // bytes of the 16-bit block grid to stage (multiple of 16), 0: hash path
  const float* pts;          // first unit of the tile (unit-major points)
  const uint16_t* grid16;
};

// skip (device flag, may be null): when set, the kernel returns at once (an evaluation enqueued
// ahead of a solve that has ended in the meantime)
void vgx_launch_reg_pose_setup(cudaStream_t st, const RegConstraintDev* cons, const double* x,
                               RegPoseConst* poses, int n, const int* skip = nullptr);
// One CTA per tile (or persistent CTAs walking their tiles) -> partials[tile][21]; the consumer adds
// a constraint's tiles in tile order (graph.cu: reg_constraint_sum).
void vgx_launch_reg_reduce(cudaStream_t st, const RegConstraintDev* cons, const RegPoseConst* poses,
                           const RegTile* tiles, int n_ctas, const int* cta_tile_begin,
                           const int* tile_order, int* tile_cost, double* partials, int grid_capacity,
                           bool jacobian, const int* skip = nullptr);
// tile_order <- tiles sorted by measured cost, most expensive first (one-CTA-per-tile mode)
void vgx_launch_reg_order(cudaStream_t st, const int* tile_cost, int n_tiles, int* tile_order);
// persistent grid size: SMs x CTAs that are co-resident with `grid_capacity` cells of dynamic smem
int vgx_reg_resident_ctas(int device, int grid_capacity);
// Fills the descriptor of one (reference -> reading) residual block.  Deterministic mode: pts / n /
// factor describe all registration points.  Sampling mode (*sampled = true): n = int(ratio * K),
// factor = 1 (all weights forced to 1) and pts is left null for the caller, who draws the
// indices (vgx_points_draw) and gathers them (vgx_launch_reg_gather_samples).
int vgx_fill_constraint(vgx_ctx* c, uint32_t ref_id, uint32_t read_id, const vgx_reg_config* cfg,
                        RegConstraintDev* out, bool* sampled = nullptr);
// dst (unit-major, ceil(n/32) units) <- the n points of src selected by d_idx, weight forced to 1
void vgx_launch_reg_gather_samples(cudaStream_t st, const float* src, const int32_t* d_idx, int n,
                                   float* dst);
