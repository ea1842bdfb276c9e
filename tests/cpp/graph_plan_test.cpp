// Runs the pose-graph table layout (voxgraph_b200/csrc/graph_plan.cpp) on cases read from stdin and prints, per
// case, one JSON line: the partition the library computes and the plan of every rank.  No CUDA runtime.
// A case, as whitespace-separated integers:
//   nranks N P M sms tile_units_override
//   constant[N]
//   P x (n ref_node read_node grid_cells grid16 locality_key)
//   M x (a b)                                          relative edges
#include <cstdio>
#include <iostream>
#include <vector>

#include "graph_plan.h"

static void ints(const char* key, const std::vector<int>& v) {
  std::printf("\"%s\": [", key);
  for (size_t i = 0; i < v.size(); ++i) std::printf(i ? ", %d" : "%d", v[i]);
  std::printf("], ");
}

static void plan_json(const VgxGraphPlan& p) {
  std::printf("{");
  ints("local", p.local);
  std::printf("\"tiles\": [");
  for (size_t i = 0; i < p.tiles.size(); ++i) {
    const VgxPlanTile& t = p.tiles[i];
    std::printf("%s[%d, %d, %d, %d, %d]", i ? ", " : "", t.constraint, t.first, t.count, t.unit0, t.grid_bytes);
  }
  std::printf("], ");
  ints("tile_begin", p.tile_begin);
  ints("block_nodes", p.block_nodes);
  ints("csr_begin", p.csr_begin);
  std::printf("\"items\": [");
  for (size_t i = 0; i < p.items.size(); ++i) {
    const int4& it = p.items[i];
    std::printf("%s[%d, %d, %d, %d]", i ? ", " : "", it.x, it.y, it.z, it.w);
  }
  std::printf("], ");
  ints("block_mask", std::vector<int>(p.block_mask.begin(), p.block_mask.end()));
  ints("red", p.red);
  std::printf("\"residuals_local\": %lld, \"n_rel_local\": %d, \"tile_units\": %d, \"n_units\": %d, "
              "\"grid_capacity\": %d, \"E\": %d, \"n_free\": %d, \"packed_len\": %zu}",
              (long long)p.residuals_local, p.n_rel_local, p.tile_units, p.n_units, p.grid_capacity, p.E, p.n_free,
              p.packed_len);
}

int main() {
  int nranks, N, P, M, sms, override_units;
  while (std::cin >> nranks >> N >> P >> M >> sms >> override_units) {
    std::vector<uint8_t> constant(N);
    for (auto& v : constant) { int x; std::cin >> x; v = (uint8_t)x; }
    std::vector<VgxPlanConstraint> cons(P);
    std::vector<int32_t> counts(P), owner(P);
    std::vector<uint32_t> keys(P);
    for (int i = 0; i < P; ++i) {
      int grid16;
      std::cin >> cons[i].n >> cons[i].ref_node >> cons[i].read_node >> cons[i].grid_cells >> grid16 >> keys[i];
      cons[i].grid16 = grid16 != 0;
      counts[i] = cons[i].n;
    }
    std::vector<int2> rel(M);
    for (auto& e : rel) std::cin >> e.x >> e.y;
    if (!std::cin) return 2;
    vgx_partition_constraints(nranks, P, counts.data(), keys.data(), owner.data());
    std::printf("{\"owner\": [");
    for (int i = 0; i < P; ++i) std::printf(i ? ", %d" : "%d", owner[i]);
    std::printf("], \"plans\": [");
    for (int r = 0; r < nranks; ++r) {
      if (r) std::printf(", ");
      plan_json(vgx_graph_plan(cons, owner, rel, N, constant, r, sms, override_units));
    }
    std::printf("]}\n");
  }
  return 0;
}
