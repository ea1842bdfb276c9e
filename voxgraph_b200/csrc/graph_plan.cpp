// Layout of the pose-graph tables and the square-root information factor (see graph_plan.h).  Plain C++: every
// decision here can be checked without a GPU.
#include "graph_plan.h"

#include <algorithm>
#include <cmath>
#include <map>
#include <numeric>
#include <utility>

void vgx_partition_constraints(int nranks, int n, const int32_t* num_residuals, const uint32_t* locality_keys,
                               int32_t* owner) {
  std::vector<int> order(n);
  std::iota(order.begin(), order.end(), 0);
  if (locality_keys)
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return locality_keys[a] < locality_keys[b]; });
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
}

bool vgx_sqrt_information_factor(const double info[16], bool allow_semi_definite, double S[16]) {
  std::fill(S, S + 16, 0.0);
  if (!allow_semi_definite) {
    for (int j = 0; j < 4; ++j) {
      double d = info[5 * j];
      for (int k = 0; k < j; ++k) d -= S[4 * j + k] * S[4 * j + k];
      if (!(d > 0)) return false;
      S[5 * j] = std::sqrt(d);
      for (int i = j + 1; i < 4; ++i) {
        double v = info[4 * i + j];
        for (int k = 0; k < j; ++k) v -= S[4 * i + k] * S[4 * j + k];
        S[4 * i + j] = v / S[5 * j];
      }
    }
    return true;
  }
  double A[4][4];
  int perm[4] = {0, 1, 2, 3};
  double scale = 0;
  for (int i = 0; i < 4; ++i) {
    scale = std::max(scale, std::fabs(info[5 * i]));
    for (int j = 0; j < 4; ++j) A[i][j] = info[4 * i + j];
  }
  for (int k = 0; k < 4; ++k) {
    int piv = k;
    for (int i = k + 1; i < 4; ++i)
      if (std::fabs(A[i][i]) > std::fabs(A[piv][piv])) piv = i;
    if (piv != k) {
      for (int j = 0; j < 4; ++j) std::swap(A[k][j], A[piv][j]);
      for (int i = 0; i < 4; ++i) std::swap(A[i][k], A[i][piv]);
      std::swap(perm[k], perm[piv]);
    }
    const double d = A[k][k];
    if (d < -1e-12 * (1.0 + scale)) return false;
    for (int i = k + 1; i < 4; ++i) A[i][k] = std::fabs(d) > 0 ? A[i][k] / d : 0.0;
    for (int i = k + 1; i < 4; ++i)
      for (int j = k + 1; j < 4; ++j) A[i][j] -= A[i][k] * d * A[j][k];
    for (int j = k + 1; j < 4; ++j) A[k][j] = 0;
  }
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j <= i; ++j) {
      const double l = (i == j) ? 1.0 : A[i][j];
      S[4 * perm[i] + perm[j]] = l * (A[j][j] > 0 ? std::sqrt(A[j][j]) : 0.0);
    }
  return true;
}

VgxGraphPlan vgx_graph_plan(const std::vector<VgxPlanConstraint>& cons, const std::vector<int32_t>& owner,
                            const std::vector<int2>& rel, int N, const std::vector<uint8_t>& constant, int rank,
                            int sms, int tile_units_override) {
  VgxGraphPlan p;
  const int P = (int)cons.size();
  for (int i = 0; i < P; ++i)
    if (owner[i] == rank) {
      p.local.push_back(i);
      p.residuals_local += cons[i].n;
    }
  p.n_rel_local = rank == 0 ? (int)rel.size() : 0;

  // Scheduling of the reduce kernel.  The cost of a unit varies ~4x with the share of its points that land in
  // the reading submap, so a static equal cut of the units over the resident CTAs leaves SMs idle while the
  // hit-heavy ones finish (measured: max SM busy time 16 % above the mean).  Instead each residual block is cut
  // into fixed tiles of tile_units 32-point units, ONE CTA PER TILE, dealt to the SMs by the hardware block
  // scheduler as resident CTAs retire (dynamic balancing at no instruction cost; the per-CTA set-up latency
  // hides behind the other resident CTAs).  Tiles never straddle constraints and start on a unit boundary
  // (128-byte aligned SoA slices for TMA).  The cut also fixes the order in which a constraint's tile rows
  // are added, and with it the last bits of every sum.
  int64_t U = 0;   // local units
  for (int i : p.local) {
    U += (cons[i].n + VGX_REG_UNIT - 1) / VGX_REG_UNIT;
    if (cons[i].grid16) p.grid_capacity = std::max(p.grid_capacity, (cons[i].grid_cells + 7) & ~7);
  }
  // At most VGX_REG_HW_TILE_UNITS units, fewer when the problem is small, so that there are at least ~2 tiles
  // per CTA slot (a 3-pair streaming graph still fills the machine).  The slots are a fixed count per SM, not
  // the resident CTAs, so that the tiles do not follow the occupancy.  The override is the environment
  // variable VGX_REG_HW_TILE_UNITS (tests use it for shapes the formula never produces).
  const int64_t slots = (int64_t)std::max(sms, 1) * VGX_REG_TILE_SLOTS_PER_SM;
  p.tile_units = (int)std::min<int64_t>(VGX_REG_HW_TILE_UNITS, std::max<int64_t>(4, (U + 2 * slots - 1) / (2 * slots)));
  if (tile_units_override >= 1) p.tile_units = tile_units_override;
  const int tile_pts = p.tile_units * VGX_REG_UNIT;
  for (int k = 0; k < p.n_local(); ++k) {
    const VgxPlanConstraint& cc = cons[p.local[k]];
    p.tile_begin.push_back(p.n_tiles());
    for (int s0 = 0; s0 < cc.n; s0 += tile_pts) {
      VgxPlanTile t;
      t.constraint = k;
      t.first = s0;
      t.count = std::min(tile_pts, cc.n - s0);
      t.unit0 = p.n_units;
      p.n_units += (t.count + VGX_REG_UNIT - 1) / VGX_REG_UNIT;
      t.grid_bytes = (cc.grid16 && cc.grid_cells > 0)
                         ? (int)((((size_t)cc.grid_cells + 7) & ~(size_t)7) * sizeof(uint16_t)) : 0;
      p.tiles.push_back(t);
    }
  }
  p.tile_begin.push_back(p.n_tiles());

  // off-diagonal blocks over ALL edges of all ranks, numbered in order of first appearance
  std::map<std::pair<int, int>, int> block_of;
  auto block_id = [&](int a, int b) {
    std::pair<int, int> key(std::min(a, b), std::max(a, b));
    auto it = block_of.find(key);
    if (it != block_of.end()) return it->second;
    int id = (int)block_of.size();
    block_of[key] = id;
    p.block_nodes.push_back(key.first);
    p.block_nodes.push_back(key.second);
    return id;
  };
  for (const int2& e : rel) block_id(e.x, e.y);
  for (const VgxPlanConstraint& cc : cons) block_id(cc.ref_node, cc.read_node);
  p.E = (int)block_of.size();

  // items per output block, in list order: this rank's relative edges, then its constraints
  std::vector<std::vector<int2>> lists(N + p.E);
  auto add_items = [&](int src, int a, int b) {
    lists[a].push_back({src, 0});
    lists[b].push_back({src, 1});
    lists[N + block_id(a, b)].push_back({src, a < b ? 2 : 3});
  };
  for (int e = 0; e < p.n_rel_local; ++e) add_items(-(e + 1), rel[e].x, rel[e].y);
  for (int k = 0; k < p.n_local(); ++k) add_items(k, cons[p.local[k]].ref_node, cons[p.local[k]].read_node);
  for (int ob = 0; ob < N + p.E; ++ob) {
    p.csr_begin.push_back((int)p.items.size());
    for (const int2& it : lists[ob])   // a registration item carries its constraint's tile range
      p.items.push_back(it.x >= 0 ? int4{it.x, it.y, p.tile_begin[it.x], p.tile_begin[it.x + 1]}
                                  : int4{it.x, it.y, 0, 0});
  }
  p.csr_begin.push_back((int)p.items.size());

  // which ranks have items for an output block: every rank computes the same table, the partition of the
  // constraints being global knowledge and the relative edges living on rank 0
  p.block_mask.assign(N + p.E, 0);
  auto mark = [&](int a, int b, unsigned char bit) {
    p.block_mask[a] |= bit;
    p.block_mask[b] |= bit;
    p.block_mask[N + block_id(a, b)] |= bit;
  };
  for (const int2& e : rel) mark(e.x, e.y, 1);
  for (int i = 0; i < P; ++i) mark(cons[i].ref_node, cons[i].read_node, (unsigned char)(1u << owner[i]));

  p.red.assign(N, -1);
  for (int i = 0; i < N; ++i)
    if (!constant[i]) { p.red[i] = p.n_free; p.n_free += 4; }
  p.packed_len = PACK_HDR + 20 * (size_t)N + 16 * (size_t)p.E;
  return p;
}
