// Exercises the C++ mirror of voxgraph's combined-mesh service (ProjectMap / GenerateCombinedMesh /
// SaveCombinedMesh in voxgraph_b200/host/voxgraph_b200.hpp) on a GPU: loads the collection argv[1], writes
// the combined mesh of its submaps at their stored poses as a PLY to argv[2] (default colour and
// MeshIntegratorConfig).  Prints "COMBINED_OK" with the counts on success; the caller compares the file
// with the Python writer's.
#include <cstdio>
#include <vector>

#include "voxgraph_b200.hpp"

using namespace voxgraph_b200;

int main(int argc, char** argv) {
  if (argc != 3) { std::printf("usage: combined_mesh_test collection out.ply\n"); return 1; }
  try {
    Context ctx(0);
    std::vector<SubmapID> ids;
    std::vector<std::array<float, 7>> poses;
    LoadSubmapCollection(ctx, argv[1], &ids, &poses);
    const int n_blocks = ProjectMap(ctx, ids, poses, 777u);
    float vs = 0;
    int vps = 0, nb = 0, finished = 0;
    ctx.check(vgx_submap_info(ctx.get(), 777u, &vs, &vps, &nb, &finished));
    if (nb != n_blocks || !finished) { std::printf("projected submap inconsistent\n"); return 1; }
    ctx.check(vgx_submap_free(ctx.get(), 777u));
    // the submap set is unchanged after every combined-mesh call: the inputs are there, and neither the
    // projection nor the scratch submap (the fixture holds id 2^32 - 1, so the first free id is 2^32 - 2) is
    const auto unchanged = [&] {
      for (SubmapID id : ids)
        if (vgx_submap_info(ctx.get(), id, nullptr, nullptr, nullptr, nullptr) != VGX_OK) return false;
      for (SubmapID id : {777u, 0xFFFFFFFEu})
        if (vgx_submap_info(ctx.get(), id, nullptr, nullptr, nullptr, nullptr) != VGX_ERR_NOT_FOUND) return false;
      return true;
    };
    const SeparatedMesh m = GenerateCombinedMesh(ctx, ids, poses);
    if ((size_t)m.vertex_offsets.back() * 3 != m.xyz.size() || (size_t)m.triangle_offsets.back() * 3 != m.triangles.size()) {
      std::printf("inconsistent offsets\n");
      return 1;
    }
    if (!unchanged()) { std::printf("submap set changed\n"); return 1; }
    bool threw = false;
    try { GenerateCombinedMesh(ctx, {ids[0], 12345u}, {poses[0], poses[0]}); }
    catch (const Error& e) { threw = e.code() == VGX_ERR_NOT_FOUND; }
    if (!threw) { std::printf("unknown id not refused\n"); return 1; }
    if (!unchanged()) { std::printf("submap set changed\n"); return 1; }
    SaveCombinedMesh(ctx, argv[2], ids, poses);
    if (!unchanged()) { std::printf("submap set changed\n"); return 1; }
    std::printf("COMBINED_OK submaps=%zu blocks=%d vertices=%zu triangles=%zu\n", ids.size(), n_blocks,
                m.xyz.size() / 3, m.triangles.size() / 3);
    return 0;
  } catch (const std::exception& e) {
    std::printf("exception: %s\n", e.what());
    return 2;
  }
}
