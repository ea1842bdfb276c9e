// oracle/_ref recipe: compiles the REFERENCE's own WeightedSampler template
// (voxgraph/include/voxgraph/frontend/submap_collection/weighted_sampler.h and
// weighted_sampler_inl.h - header-only, no third-party dependency) behind a C interface, so the
// oracle's restatement (vgo_sampler_*) and the product's sampling mode can be pinned against the
// real reference code.  TEST INFRASTRUCTURE ONLY; built into oracle/_ref/ (git-ignored) when
// VOXGRAPH_SRC names a voxgraph checkout; its sources are included from where they lie, never copied.
#include <stdint.h>

#include "voxgraph/frontend/submap_collection/weighted_sampler.h"

namespace {
struct Item {
  int32_t index;
};
}  // namespace

extern "C" {
void* vgref_sampler_create(const float* weights, int n) {
  auto* s = new voxgraph::WeightedSampler<Item>();
  // VoxgraphSubmap::findIsosurfaceVertices / findRelevantVoxelIndices: addItem(point, voxel.weight)
  for (int i = 0; i < n; ++i) s->addItem(Item{i}, weights[i]);
  return s;
}
void vgref_sampler_destroy(void* h) { delete static_cast<voxgraph::WeightedSampler<Item>*>(h); }
// getRandomItem x count
void vgref_sampler_draw(void* h, int count, int32_t* idx) {
  auto* s = static_cast<voxgraph::WeightedSampler<Item>*>(h);
  for (int i = 0; i < count; ++i) idx[i] = s->getRandomItem().index;
}
}
