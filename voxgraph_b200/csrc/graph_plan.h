// Layout of the pose-graph tables (graph_plan.cpp): which registration constraints this rank owns, how their
// points are cut into reduce tiles, how the output blocks are numbered and which items each block sums; and the
// square-root information factor of a relative-pose edge.  Host only, no CUDA runtime: graph.cu collects the
// inputs, calls vgx_graph_plan and uploads what it returns.
#pragma once

#include <stddef.h>
#include <stdint.h>
#include <vector_types.h>   // int2, int4

#include <vector>

#define VGX_REG_TILE_SLOTS_PER_SM 7  // CTA slots per SM the tile size is cut for.  A fixed count, not the
                                     // resident one: the tiles, and with them the last bits of every sum, do
                                     // not follow the occupancy (7 CTAs per SM when the rule was set)
#define VGX_REG_HW_TILE_UNITS 64   // largest tile, in units (smaller on small problems)
#define VGX_REG_UNIT 32            // points per unit = one warp iteration; tiles are cut on unit boundaries

// Packed normal equations, the output of one evaluation (doubles):
//   [PACK_HDR header: [0] cost, [1..3] reserved | 4 N gradient, node-major |
//    16 N diagonal 4x4 blocks, row-major, node order |
//    16 E off-diagonal 4x4 blocks, row-major: rows node block_nodes[2b] (the smaller index), cols block_nodes[2b + 1]]
#define PACK_HDR 4

// What the layout needs of one registration constraint (reference -> reading submap).
struct VgxPlanConstraint {
  int n;                   // points (residuals)
  int ref_node, read_node;
  int grid_cells;          // cells of the reading submap's dense block grid
  bool grid16;             // the reading submap has the 16-bit copy of that grid
};

// A tile: points [first, first + count) of local constraint `constraint`, one reduce CTA.
struct VgxPlanTile {
  int constraint, first, count;
  int unit0;        // index of the tile's first unit in the unit-bound table
  int grid_bytes;   // bytes of the 16-bit block grid the CTA stages (multiple of 16), 0: hash path
};

struct VgxGraphPlan {
  std::vector<int> local;          // global indices of this rank's constraints, in list order
  int64_t residuals_local = 0;
  int n_rel_local = 0;             // relative edges evaluated here: all of them on rank 0, none elsewhere
  int tile_units = 0;              // tile size in units
  std::vector<VgxPlanTile> tiles;  // local constraint by constraint, each cut in point order
  std::vector<int> tile_begin;     // n_local + 1: local constraint k owns tiles [tile_begin[k], tile_begin[k + 1])
  int n_units = 0;                 // units of all tiles = entries of the unit-bound table
  int grid_capacity = 0;           // 16-bit cells of the largest local block grid, a multiple of 8
  int E = 0;                       // off-diagonal blocks
  std::vector<int> block_nodes;    // E x 2: (smaller, larger) node of each
  std::vector<int> csr_begin;      // N + E + 1: items of output block ob are [csr_begin[ob], csr_begin[ob + 1])
  std::vector<int4> items;         // (source, role, first tile, end tile); source >= 0: local constraint,
                                   // < 0: relative edge -(e + 1); role 0: A-A, 1: B-B, 2: A-B, 3: B-A
  std::vector<unsigned char> block_mask;   // N + E: bit r = rank r has items for the block
  std::vector<int> red;            // N: reduced offset of a free node, -1 for a constant one
  int n_free = 0;                  // reduced dimension 4 * (free nodes)
  size_t packed_len = 0;           // doubles of the packed normal equations

  int n_local() const { return (int)local.size(); }
  int n_tiles() const { return (int)tiles.size(); }
};

// owner[i] <- the rank of constraint i.  Constraints are taken in order of locality key (list order without
// keys, stable) and each goes to the rank whose equal share of the total residual count holds its midpoint.
void vgx_partition_constraints(int nranks, int n, const int32_t* num_residuals, const uint32_t* locality_keys,
                               int32_t* owner);

// The square-root information factor of a relative-pose edge (see vgx_sqrt_information); false when the matrix
// is rejected.
bool vgx_sqrt_information_factor(const double info[16], bool allow_semi_definite, double S[16]);

// The tables of rank `rank` for the constraints `cons` partitioned by `owner` (identical on every rank), the
// relative edges' node pairs `rel`, and N nodes of which constant[i] != 0 are held fixed.  sms: the device's SM
// count; tile_units_override >= 1 forces the tile size.
VgxGraphPlan vgx_graph_plan(const std::vector<VgxPlanConstraint>& cons, const std::vector<int32_t>& owner,
                            const std::vector<int2>& rel, int N, const std::vector<uint8_t>& constant, int rank,
                            int sms, int tile_units_override);
