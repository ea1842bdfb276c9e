// Map evaluation on the device (voxgraph MapEvaluation, src/tools/evaluation/map_evaluation.cpp:59-161):
//   vgx_evaluate_layers_rmse = voxblox utils::evaluateLayersRmse, mode kIgnoreErrorBehindTestSurface
//   vgx_map_evaluate         = MapEvaluation::evaluate: projection, finish, alignment on a private pose
//                              graph, vgx_submap_transform of the ground truth, RMSE
//
// The RMSE rule (restated from the published voxblox sources; see the header for the full statement):
//   test block without a ground-truth block -> its observed test voxels are non-overlapping;
//   shared block, per voxel: either side unobserved -> non-overlapping; d_test < 0 -> ignored + overlapping;
//     else evaluated + overlapping, e = d_test - d_gt (float), fl32(e * e) into a double sum,
//     max_error = std::max(max_error, |e|) (NaN never replaces it), min_error stays 0;
//   ground-truth block without a test block -> its observed ground-truth voxels are non-overlapping.
//
// Passes: rmse_block_kernel, one CTA per test block then one per ground-truth block, one hash lookup of the
// other layer per CTA; each thread walks its voxels in order, the CTA reduces counts, the maximum and the
// double sum in a fixed tree and writes one partial per CTA.  rmse_total_kernel (one CTA) adds the partials:
// thread t sums partials t, t + 256, ... in order, then the same fixed tree.  No float atomics, so two calls
// are bit-identical.  Compiled with -fmad=false.
#include <math.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "layer_access.cuh"

#define RMSE_THREADS 256

struct RmsePartial {
  double sum;
  float max_error;
  uint32_t pad;
  unsigned long long n_eval, n_ign, n_ovl, n_non;
};

struct RmseLayer {
  LayerDev L;   // L.dw: (distance, weight) or, esdf, (distance, observed 1 / 0)
  int esdf;     // observed: esdf ? flag != 0 : weight > 1e-6
};

__device__ __forceinline__ bool rmse_observed(int esdf, float2 q) {
  return esdf ? q.y != 0.0f : q.y > 1e-6f;
}

// fixed-tree CTA reduction of one partial per thread (blockDim.x a power of two); result in thread 0
__device__ void rmse_cta_reduce(RmsePartial& p) {
  __shared__ double s_sum[RMSE_THREADS];
  __shared__ float s_max[RMSE_THREADS];
  __shared__ unsigned long long s_cnt[4][RMSE_THREADS];
  const int t = threadIdx.x;
  s_sum[t] = p.sum;
  s_max[t] = p.max_error;
  s_cnt[0][t] = p.n_eval; s_cnt[1][t] = p.n_ign; s_cnt[2][t] = p.n_ovl; s_cnt[3][t] = p.n_non;
  __syncthreads();
  for (int h = blockDim.x >> 1; h > 0; h >>= 1) {
    if (t < h) {
      s_sum[t] = s_sum[t] + s_sum[t + h];
      s_max[t] = fmaxf(s_max[t], s_max[t + h]);
#pragma unroll
      for (int k = 0; k < 4; ++k) s_cnt[k][t] += s_cnt[k][t + h];
    }
    __syncthreads();
  }
  if (t == 0) {
    p.sum = s_sum[0];
    p.max_error = s_max[0];
    p.n_eval = s_cnt[0][0]; p.n_ign = s_cnt[1][0]; p.n_ovl = s_cnt[2][0]; p.n_non = s_cnt[3][0];
  }
}

__global__ void __launch_bounds__(RMSE_THREADS)
rmse_block_kernel(RmseLayer gt, RmseLayer test, RmsePartial* __restrict__ out) {
  const bool test_side = blockIdx.x < (unsigned)test.L.n_blocks;
  // the layer whose block this CTA owns (a_*) and the other one (field by field: no local copy)
  const int32_t* a_idx = test_side ? test.L.block_idx : gt.L.block_idx;
  const float2* a_dw = test_side ? test.L.dw : gt.L.dw;
  const int a_esdf = test_side ? test.esdf : gt.esdf;
  const VgxHash b_hash = test_side ? gt.L.hash : test.L.hash;
  const int slot = test_side ? (int)blockIdx.x : (int)blockIdx.x - test.L.n_blocks;
  const int other = vgx_hash_find(b_hash, a_idx[3 * slot], a_idx[3 * slot + 1], a_idx[3 * slot + 2]);
  RmsePartial p;
  p.sum = 0.0;
  p.max_error = 0.0f;
  p.pad = 0;
  p.n_eval = p.n_ign = p.n_ovl = p.n_non = 0;
  const int vpb = vgx_voxels_per_block(test.L.sh);   // the two layers share vps
  const float2* a = a_dw + (size_t)slot * vpb;
  if (other < 0) {   // a block of one layer only: its observed voxels are non-overlapping
    for (int v = threadIdx.x; v < vpb; v += blockDim.x) p.n_non += rmse_observed(a_esdf, a[v]) ? 1 : 0;
  } else if (test_side) {   // shared block (counted once, from the test side)
    const float2* g = gt.L.dw + (size_t)other * vpb;
    for (int v = threadIdx.x; v < vpb; v += blockDim.x) {
      const float2 qt = a[v], qg = g[v];
      if (!rmse_observed(test.esdf, qt) || !rmse_observed(gt.esdf, qg)) {
        p.n_non++;
      } else if (qt.x < 0.0f) {
        p.n_ign++;
        p.n_ovl++;
      } else {
        const float e = qt.x - qg.x;
        const float e2 = e * e;
        p.sum += (double)e2;
        p.max_error = fmaxf(p.max_error, fabsf(e));   // std::max(max, |e|): a NaN |e| is dropped
        p.n_eval++;
        p.n_ovl++;
      }
    }
  }
  rmse_cta_reduce(p);
  if (threadIdx.x == 0) out[blockIdx.x] = p;
}

__global__ void __launch_bounds__(RMSE_THREADS)
rmse_total_kernel(const RmsePartial* __restrict__ part, int n, RmsePartial* __restrict__ out) {
  RmsePartial p;
  p.sum = 0.0;
  p.max_error = 0.0f;
  p.pad = 0;
  p.n_eval = p.n_ign = p.n_ovl = p.n_non = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const RmsePartial q = part[i];
    p.sum = p.sum + q.sum;
    p.max_error = fmaxf(p.max_error, q.max_error);
    p.n_eval += q.n_eval; p.n_ign += q.n_ign; p.n_ovl += q.n_ovl; p.n_non += q.n_non;
  }
  rmse_cta_reduce(p);
  if (threadIdx.x == 0) *out = p;
}

// ------------------------------------------------------------------ host
static int rmse_layer(vgx_ctx* c, VgxSubmap* s, int which, const char* name, RmseLayer* L) {
  if (which != VGX_LAYER_TSDF && which != VGX_LAYER_ESDF)
    VGX_FAIL(c, VGX_ERR_INVALID, std::string("unknown layer selector for the ") + name);
  if (!s->finished) VGX_FAIL(c, VGX_ERR_INVALID, std::string("the ") + name + " is not finished");
  if (which == VGX_LAYER_ESDF && !s->d_view_esdf.get())
    VGX_FAIL(c, VGX_ERR_INVALID, std::string("the ") + name + " has no ESDF");
  L->L = layer_of(s, which);
  L->esdf = which == VGX_LAYER_ESDF;
  return VGX_OK;
}

extern "C" int vgx_evaluate_layers_rmse(vgx_ctx* c, uint32_t gt_id, int gt_layer, uint32_t test_id, int test_layer,
                                        vgx_voxel_evaluation_details* out) {
  return vgx_entry(c, __func__, [&] {
    if (!out) VGX_FAIL(c, VGX_ERR_INVALID, "invalid argument");
    memset(out, 0, sizeof(*out));
    VgxSubmap *g, *t;
    VGX_TRY(vgx_submap_get(c, gt_id, &g));
    VGX_TRY(vgx_submap_get(c, test_id, &t));
    if (g->voxel_size != t->voxel_size || g->vps != t->vps)
      VGX_FAIL(c, VGX_ERR_INVALID, "the layers differ in voxel size or voxels_per_side");
    RmseLayer G, T;
    VGX_TRY(rmse_layer(c, g, gt_layer, "ground truth", &G));
    VGX_TRY(rmse_layer(c, t, test_layer, "test layer", &T));
    const size_t n_part = (size_t)G.L.n_blocks + (size_t)T.L.n_blocks;
    if (n_part > (size_t)INT32_MAX) VGX_FAIL(c, VGX_ERR_CAPACITY, "too many blocks");
    RmsePartial total;
    memset(&total, 0, sizeof(total));
    if (n_part > 0) {
      RmsePartial* d_part;
      VGX_TRY(vgx_carve(c, c->d_work, vgx_part(d_part, n_part + 1)));
      const int threads = std::min(RMSE_THREADS, g->vox_per_block);
      {
        VgxProfileScope scope(c, VGX_SLOT_EVAL);
        VGX_TRY(vgx_launch(c, rmse_block_kernel, (unsigned)n_part, threads, 0, VgxLaunch::plain, G, T, d_part));
      }
      {
        VgxProfileScope scope(c, VGX_SLOT_EVAL);
        VGX_TRY(vgx_launch(c, rmse_total_kernel, 1, RMSE_THREADS, 0, VgxLaunch::plain, d_part, (int)n_part,
                           d_part + n_part));
      }
      VGX_TRY(vgx_read(c, &total, d_part + n_part));
    }
    out->rmse = (float)sqrt(total.sum / (double)total.n_eval);
    out->max_error = total.max_error;
    out->min_error = 0.0f;
    out->num_evaluated_voxels = total.n_eval;
    out->num_ignored_voxels = total.n_ign;
    out->num_overlapping_voxels = total.n_ovl;
    out->num_non_overlapping_voxels = total.n_non;
    return VGX_OK;
  });
}

// ------------------------------------------------------------------ MapEvaluation::evaluate
// minkindr QuatTransformation::exp([x y z 0 0 yaw]) in float: translation as given, rotation
// RotationQuaternion::exp of the yaw vector (angle |yaw| about +-z)
static void eval_exp_xyzyaw(const double pose[4], float T[7]) {
  const float yaw = (float)pose[3];
  const float half = 0.5f * fabsf(yaw);
  T[0] = cosf(half);
  T[1] = 0.0f;
  T[2] = 0.0f;
  T[3] = yaw == 0.0f ? 0.0f : (yaw < 0.0f ? -sinf(half) : sinf(half));
  T[4] = (float)pose[0];
  T[5] = (float)pose[1];
  T[6] = (float)pose[2];
}

// the projected map: view, ESDF (defaults), relevant voxels with the reference's registration filter
// (voxgraph_submap.h:26-30), the registration points of the alignment's reference side
static int eval_finish_projected(vgx_ctx* c, uint32_t id) {
  VGX_TRY(vgx_submap_finish(c, id));
  VGX_TRY(vgx_submap_generate_esdf(c, id, nullptr, nullptr));
  vgx_registration_filter f;
  f.min_voxel_weight = 1.0;
  f.max_voxel_distance = 0.3;
  f.use_esdf_distance = 1;
  return vgx_submap_extract_points(c, id, &f);
}

// the ground truth (the alignment's reading side): view and ESDF (defaults)
static int eval_finish_gt(vgx_ctx* c, uint32_t id) {
  VGX_TRY(vgx_submap_finish(c, id));
  return vgx_submap_generate_esdf(c, id, nullptr, nullptr);
}

// MapEvaluation::alignSubmapAtoSubmapB on a private pose graph (the context's graph is set aside)
static int eval_align(vgx_ctx* c, uint32_t projected, uint32_t gt, double pose[4], vgx_solver_summary* S) {
  VgxGraph* saved = c->graph;
  const int saved_nranks = c->nranks, saved_rank = c->rank;
  c->graph = nullptr;
  c->nranks = 1;   // the alignment is one residual block, evaluated on this rank alone
  c->rank = 0;
  const uint32_t ids[2] = {projected, gt};
  const double x0[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  const uint8_t constant[2] = {1, 0};
  vgx_reg_config rc_cfg;
  rc_cfg.registration_point_type = VGX_POINTS_VOXELS;
  rc_cfg.no_correspondence_cost = 0.0;
  rc_cfg.sampling_ratio = -1.0f;
  rc_cfg.use_esdf_distance = 1;
  vgx_solver_options o;
  vgx_solver_options_default(&o);
  o.max_num_iterations = 200;   // map_evaluation.cpp:127-128; every other option is Ceres' default
  o.parameter_tolerance = 1e-12;
  o.function_tolerance = 1e-6;
  o.gradient_tolerance = 1e-10;
  o.max_solver_time_s = 1e9;
  double x[8];
  memset(S, 0, sizeof(*S));
  int rc = vgx_graph_set_nodes(c, 2, ids, x0, constant);
  if (rc == VGX_OK) rc = vgx_graph_set_registration_constraints(c, 1, &ids[0], &ids[1], &rc_cfg);
  if (rc == VGX_OK) {
    rc = vgx_graph_solve(c, &o, x, S);
    if (rc == VGX_OK) {
      memcpy(pose, x + 4, 4 * sizeof(double));
    } else if (rc == VGX_ZERO_WEIGHT || (rc == VGX_ERR_INVALID && S->termination == 6)) {
      // Ceres reports FAILURE and leaves the parameters where they started
      S->termination = 6;
      memset(pose, 0, 4 * sizeof(double));
      rc = VGX_OK;
    }
  }
  vgx_graph_free(c);
  c->graph = saved;
  c->nranks = saved_nranks;
  c->rank = saved_rank;
  vgx_graph_invalidate_registration(c);
  return rc;
}

extern "C" int vgx_map_evaluate(vgx_ctx* c, uint32_t gt_id, int n, const uint32_t* ids, const float* T_M_S,
                                vgx_map_evaluation* out) {
  return vgx_entry(c, __func__, [&] {
    if (!out || n < 1 || !ids || !T_M_S) VGX_FAIL(c, VGX_ERR_INVALID, "invalid argument");
    memset(out, 0, sizeof(*out));
    VgxSubmap *g, *s;
    VGX_TRY(vgx_submap_get(c, gt_id, &g));
    for (int k = 0; k < n; ++k) {
      if (ids[k] == gt_id) VGX_FAIL(c, VGX_ERR_INVALID, "the ground truth is one of the submaps");
      VGX_TRY(vgx_submap_get(c, ids[k], &s));
      if (s->voxel_size != g->voxel_size || s->vps != g->vps)   // map_evaluation.cpp:66 CHECK_EQ
        VGX_FAIL(c, VGX_ERR_INVALID,
                 "the ground truth and the submaps differ in voxel size or voxels_per_side");
    }
    // 1. the projected map, in a scratch submap freed on every exit
    const uint32_t pid = vgx_scratch_id(c);
    VGX_TRY(vgx_project_map(c, n, ids, T_M_S, pid, nullptr));
    // 2.-3. finish both
    int rc = eval_finish_projected(c, pid);
    if (rc == VGX_OK) rc = eval_finish_gt(c, gt_id);
    // 4. align the ground truth (reading, free) to the projected map (reference, constant)
    if (rc == VGX_OK) rc = eval_align(c, pid, gt_id, out->aligned_pose, &out->summary);
    // 5. move the ground truth into the map's frame and finish it again
    if (rc == VGX_OK) {
      eval_exp_xyzyaw(out->aligned_pose, out->T_projected_map__ground_truth);
      ov_inverse(out->T_projected_map__ground_truth, out->T_ground_truth__reading);
      rc = vgx_submap_transform(c, gt_id, out->T_projected_map__ground_truth);
    }
    if (rc == VGX_OK) rc = eval_finish_gt(c, gt_id);
    // 6. RMSE of the projected map's ESDF against the ground truth's
    if (rc == VGX_OK) rc = vgx_evaluate_layers_rmse(c, gt_id, VGX_LAYER_ESDF, pid, VGX_LAYER_ESDF, &out->details);
    // 7.
    vgx_submap_drop(c, pid);
    return rc;
  });
}
