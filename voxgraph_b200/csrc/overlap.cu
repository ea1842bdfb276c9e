// Overlap detection / registration pair list on resident submaps (SURVEY §8 rows a20 / f3):
//   VoxgraphSubmap::overlapsWith                      voxgraph/src/frontend/submap_collection/voxgraph_submap.cpp:245-278
//   BoundingBox::getAabbFromObbAndPose                src/frontend/submap_collection/bounding_box.cpp:28-42
//   PoseGraphInterface::updateOverlappingSubmapList   src/frontend/pose_graph_interface/pose_graph_interface.cpp:109-147
// Mission-frame surface AABBs and the N(N-1)/2 rejection tests are a few thousand float compares
// (host, the reference's arithmetic restated in float: minkindr quaternion transform);
// "any isosurface block centre of A lands in an allocated block of B" runs on the device against
// B's block hash, one CTA per surviving pair.  Compiled with -fmad=false.
#include <math.h>
#include <string.h>

#include <vector>

#include "layer_access.cuh"

namespace {

inline void ov_compose(const float A[7], const float B[7], float o[7]) {
  const float aw = A[0], ax = A[1], ay = A[2], az = A[3];
  const float bw = B[0], bx = B[1], by = B[2], bz = B[3];
  o[0] = aw * bw - ax * bx - ay * by - az * bz;
  o[1] = aw * bx + ax * bw + ay * bz - az * by;
  o[2] = aw * by + ay * bw + az * bx - ax * bz;
  o[3] = aw * bz + az * bw + ax * by - ay * bx;
  float r[3];
  ov_rotate(A, B + 4, r);
  o[4] = A[4] + r[0]; o[5] = A[5] + r[1]; o[6] = A[6] + r[2];
}

struct OverlapJob {
  VgxHash other_hash;
  const int32_t* iso_idx;   // isosurface blocks of the current submap (n x 3)
  int n_iso;
  float block_size;         // of the current submap
  float other_block_size_inv;
  float T[7];               // T_other_submap__current_submap
};

}  // namespace

// cpp:263-273: one CTA per pair; a hit anywhere sets the pair's flag
__global__ void __launch_bounds__(128)
overlap_pairs_kernel(const OverlapJob* __restrict__ jobs, int* __restrict__ flags) {
  const OverlapJob J = jobs[blockIdx.x];
  __shared__ int s_hit;
  if (threadIdx.x == 0) s_hit = 0;
  __syncthreads();
  for (int k = threadIdx.x; k < J.n_iso; k += blockDim.x) {
    if (s_hit) break;
    // getCenterPointFromGridIndex(block_index, block_size) = (index + 0.5) * block_size
    const float cpt[3] = {((float)J.iso_idx[3 * k] + 0.5f) * J.block_size,
                          ((float)J.iso_idx[3 * k + 1] + 0.5f) * J.block_size,
                          ((float)J.iso_idx[3 * k + 2] + 0.5f) * J.block_size};
    float p[3];
    ov_transform(J.T, cpt, p);
    const int b0 = __float2int_rd(p[0] * J.other_block_size_inv + 1e-6f);
    const int b1 = __float2int_rd(p[1] * J.other_block_size_inv + 1e-6f);
    const int b2 = __float2int_rd(p[2] * J.other_block_size_inv + 1e-6f);
    if (vgx_hash_find(J.other_hash, b0, b1, b2) >= 0) s_hit = 1;   // hasBlock
  }
  __syncthreads();
  if (threadIdx.x == 0) flags[blockIdx.x] = s_hit;
}

extern "C" int vgx_find_overlapping_pairs(vgx_ctx* c, int n, const uint32_t* ids, const float* poses,
                                          int max_pairs, uint32_t* pairs, int* n_pairs) {
  return vgx_entry(c, __func__, [&] {
    if (n < 0 || (n > 0 && (!ids || !poses)) || !n_pairs || max_pairs < 0 || (max_pairs > 0 && !pairs))
      return VGX_ERR_INVALID;
    *n_pairs = 0;
    std::vector<VgxSubmap*> sm(n);
    std::vector<float> amin(3 * (size_t)n), amax(3 * (size_t)n);
    for (int i = 0; i < n; ++i) {
      VGX_TRY(vgx_submap_get(c, ids[i], &sm[i]));
      if (!sm[i]->finished || !sm[i]->points_extracted)
        VGX_FAIL(c, VGX_ERR_INVALID, "run vgx_submap_extract_points / "
                                     "vgx_submap_finish_ex on every submap first (surface OBB + isosurface blocks)");
      // getMissionFrameSurfaceAabb = getAabbFromObbAndPose(surface OBB, pose): an OBB that was never
      // updated stays (+inf, -inf) and so does the AABB, which then fails every interval test
      float* mn = &amin[3 * (size_t)i];
      float* mx = &amax[3 * (size_t)i];
      for (int a = 0; a < 3; ++a) { mn[a] = INFINITY; mx[a] = -INFINITY; }
      const float* T = poses + 7 * (size_t)i;
      const float omin[3] = {sm[i]->surface_obb_valid ? sm[i]->surface_obb_min[0] : INFINITY,
                             sm[i]->surface_obb_valid ? sm[i]->surface_obb_min[1] : INFINITY,
                             sm[i]->surface_obb_valid ? sm[i]->surface_obb_min[2] : INFINITY};
      const float omax[3] = {sm[i]->surface_obb_valid ? sm[i]->surface_obb_max[0] : -INFINITY,
                             sm[i]->surface_obb_valid ? sm[i]->surface_obb_max[1] : -INFINITY,
                             sm[i]->surface_obb_valid ? sm[i]->surface_obb_max[2] : -INFINITY};
      for (unsigned k = 0; k < 8; ++k) {
        // getCornerCoordinates: bit set -> min, clear -> max
        const float corner[3] = {(k & 1) ? omin[0] : omax[0], (k & 2) ? omin[1] : omax[1],
                                 (k & 4) ? omin[2] : omax[2]};
        float m[3];
        ov_transform(T, corner, m);
        for (int a = 0; a < 3; ++a) {
          if (m[a] < mn[a]) mn[a] = m[a];   // cwiseMin / cwiseMax (NaN never replaces)
          if (m[a] > mx[a]) mx[a] = m[a];
        }
      }
    }
    // pose_graph_interface.cpp:115-146: every i against the subsequent j
    std::vector<OverlapJob> jobs;
    std::vector<std::pair<int, int>> cand;
    for (int i = 0; i < n; ++i) {
      for (int j = i + 1; j < n; ++j) {
        bool sep = false;
        for (int a = 0; a < 3; ++a)   // cpp:251-256
          if (amax[3 * (size_t)i + a] < amin[3 * (size_t)j + a] || amin[3 * (size_t)i + a] > amax[3 * (size_t)j + a]) sep = true;
        if (sep || sm[i]->n_iso == 0) continue;
        OverlapJob J;
        J.other_hash = sm[j]->hash();
        J.iso_idx = sm[i]->d_iso_idx.get();
        J.n_iso = sm[i]->n_iso;
        J.block_size = sm[i]->block_size;
        J.other_block_size_inv = sm[j]->block_size_inv;
        float inv[7];
        ov_inverse(poses + 7 * (size_t)j, inv);              // cpp:261-262
        ov_compose(inv, poses + 7 * (size_t)i, J.T);
        jobs.push_back(J);
        cand.emplace_back(i, j);
      }
    }
    if (jobs.empty()) return VGX_OK;
    OverlapJob* d_jobs;
    int* d_flags;
    VGX_TRY(vgx_carve(c, c->d_scratch, vgx_part(d_jobs, jobs.size()), vgx_part(d_flags, jobs.size())));
    VGX_TRY(vgx_upload(c, d_jobs, jobs.data(), jobs.size()));
    VGX_TRY(vgx_launch(c, overlap_pairs_kernel, (unsigned)jobs.size(), 128, 0, VgxLaunch::plain, d_jobs, d_flags));
    std::vector<int> flags(jobs.size());
    VGX_TRY(vgx_read(c, flags.data(), d_flags, flags.size()));
    int np = 0;
    for (size_t k = 0; k < jobs.size(); ++k) {
      if (!flags[k]) continue;
      if (np < max_pairs) { pairs[2 * np] = ids[cand[k].first]; pairs[2 * np + 1] = ids[cand[k].second]; }
      ++np;
    }
    *n_pairs = np;
    if (np > max_pairs) VGX_FAIL(c, VGX_ERR_CAPACITY, "max_pairs too small");
    return VGX_OK;
  });
}
