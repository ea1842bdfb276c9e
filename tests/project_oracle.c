/*
 * project_oracle.c — CPU restatement of cblox SubmapCollection::getProjectedMap for the tests (the checker of
 * vgx_project_map).  Built at test time by tests/project_oracle.py against oracle/libvg_oracle.so, whose public
 * functions it reuses for everything voxblox does per point: vgo_interp_voxel (Interpolator::getVoxel),
 * vgo_T_inverse / vgo_T_transform (minkindr float) and vgo_grid_index_from_point (getGridIndexFromPoint).
 *
 * getProjectedMap = voxblox mergeLayerAintoLayerB(layer, T_M_S, &global) (merge_integration.h:
 * transformLayer, then the untransformed merge) for every submap in increasing id order.  voxblox and cblox
 * are not in the reference tree: restated from the published sources, not checked against a compiled
 * voxblox.  Operation by operation with the same float forms; build with -ffp-contract=off.
 *   transformLayer: per block b of the input, c = T * ((b + 0.5) * block_size), offset =
 *   kUnitCubeDiagonalLength (sqrt(3)) * block_size * 0.5; for x = c.x - offset; x < c.x + offset;
 *   x += block_size (same for y, z) the block getGridIndexFromPoint(x, y, z) is a candidate; every voxel
 *   centre of a candidate block, moved by T.inverse(), is interpolated; a failure leaves (0, 0); candidate
 *   blocks without any success are removed.
 *   merge: every voxel of every remaining block into the global layer (new blocks start at (0, 0)):
 *   w = wA + wB; if (w > 0) { d = (dA * wA + dB * wB) / w; weight = w; }
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "oracle_harness.h"

#define VGP_BLOCK_INDEX_MIN (-(1 << 20) + 1)
#define VGP_BLOCK_INDEX_MAX ((1 << 20) - 2)

/* the global layer: blocks in first-touch order, found through an index layer (a vgo_layer used as a set:
 * its slots are assigned 0, 1, 2, ... in insertion order, the same numbering as the arrays here) */
typedef struct {
  vgo_layer* index;
  int n, cap, vpb;
  int32_t* idx;
  float* d;
  float* w;
} vgp_global;

static int global_slot(vgp_global* G, const int32_t b[3]) {
  int s = vgo_layer_find_block(G->index, b);
  if (s >= 0) return s;
  s = vgo_layer_add_block(G->index, b, NULL, NULL);
  if (G->n == G->cap) {
    G->cap = G->cap ? 2 * G->cap : 64;
    G->idx = (int32_t*)realloc(G->idx, sizeof(int32_t) * 3 * (size_t)G->cap);
    G->d = (float*)realloc(G->d, sizeof(float) * (size_t)G->vpb * G->cap);
    G->w = (float*)realloc(G->w, sizeof(float) * (size_t)G->vpb * G->cap);
  }
  memcpy(G->idx + 3 * (size_t)s, b, 3 * sizeof(int32_t));
  memset(G->d + (size_t)s * G->vpb, 0, sizeof(float) * (size_t)G->vpb);
  memset(G->w + (size_t)s * G->vpb, 0, sizeof(float) * (size_t)G->vpb);
  G->n++;
  return s;
}

/* mergeVoxelAIntoVoxelB<TsdfVoxel> (merge_integration.h), distance and weight */
static void merge_voxel(float dA, float wA, float* dB, float* wB) {
  const float combined_weight = wA + *wB;
  if (combined_weight > 0) {
    *dB = (dA * wA + *dB * *wB) / combined_weight;
    *wB = combined_weight;
  }
}

/* transformLayer(S, T, out) then mergeLayerAintoLayerB(out, G).  Returns 0 when a candidate block index is out
 * of range. */
static int project_one(const vgo_layer* S, float vs, int vps, const float T[7], vgp_global* G) {
  const float bs = vs * (float)vps; /* Layer ctor: block_size_ = voxel_size_ * voxels_per_side_ */
  const float bs_inv = vgo_layer_block_size_inv(S);
  const int vpb = vps * vps * vps;
  const int nb = vgo_layer_num_blocks(S);
  int32_t* in_idx = (int32_t*)malloc(sizeof(int32_t) * 3 * (size_t)(nb > 0 ? nb : 1));
  vgo_layer_export(S, in_idx, NULL, NULL);
  vgo_layer* cand = vgo_layer_create(1.0f, 2); /* candidate set, insertion order */
  int32_t* cidx = NULL;
  int nc = 0, ccap = 0, ok = 1;
  for (int b = 0; b < nb && ok; ++b) {
    const int32_t* bi = in_idx + 3 * b;
    const float c_in[3] = {((float)bi[0] + 0.5f) * bs, ((float)bi[1] + 0.5f) * bs, ((float)bi[2] + 0.5f) * bs};
    float c_out[3];
    vgo_T_transform(T, c_in, c_out);
    const float offset = (float)((double)(1.7320508075688772f * bs) * 0.5);
    for (float x = c_out[0] - offset; x < c_out[0] + offset && ok; x += bs)
      for (float y = c_out[1] - offset; y < c_out[1] + offset && ok; y += bs)
        for (float z = c_out[2] - offset; z < c_out[2] + offset && ok; z += bs) {
          const float p[3] = {x, y, z};
          for (int a = 0; a < 3; ++a) {
            const float f = floorf(p[a] * bs_inv + 1e-6f);
            if (!(f >= (float)VGP_BLOCK_INDEX_MIN && f <= (float)VGP_BLOCK_INDEX_MAX)) ok = 0;
          }
          if (!ok) break;
          int32_t q[3];
          vgo_grid_index_from_point(p, bs_inv, q);
          if (vgo_layer_find_block(cand, q) >= 0) continue;
          vgo_layer_add_block(cand, q, NULL, NULL);
          if (nc == ccap) {
            ccap = ccap ? 2 * ccap : 64;
            cidx = (int32_t*)realloc(cidx, sizeof(int32_t) * 3 * (size_t)ccap);
          }
          memcpy(cidx + 3 * (size_t)nc++, q, sizeof(q));
        }
  }
  vgo_layer_destroy(cand);
  free(in_idx);
  if (!ok) {
    free(cidx);
    return 0;
  }
  /* resampling at the voxel centres of the candidate blocks; merge of the blocks that got data */
  float T_in_out[7];
  vgo_T_inverse(T, T_in_out);
  float* xd = (float*)malloc(sizeof(float) * (size_t)vpb);
  float* xw = (float*)malloc(sizeof(float) * (size_t)vpb);
  for (int c = 0; c < nc; ++c) {
    const int32_t* bi = cidx + 3 * c;
    int has_data = 0;
    for (int lin = 0; lin < vpb; ++lin) {
      const int v[3] = {lin % vps, (lin / vps) % vps, lin / (vps * vps)};
      float centre[3], p_in[3];
      for (int a = 0; a < 3; ++a) centre[a] = (float)bi[a] * bs + ((float)v[a] + 0.5f) * vs;
      vgo_T_transform(T_in_out, centre, p_in);
      float d, w;
      xd[lin] = 0.0f;
      xw[lin] = 0.0f;
      if (vgo_interp_voxel(S, p_in, &d, &w)) {
        xd[lin] = d;
        xw[lin] = w;
        has_data = 1;
      }
    }
    if (!has_data) continue; /* removeBlock */
    const int g = global_slot(G, bi);
    float* gd = G->d + (size_t)g * vpb;
    float* gw = G->w + (size_t)g * vpb;
    for (int lin = 0; lin < vpb; ++lin) merge_voxel(xd[lin], xw[lin], gd + lin, gw + lin);
  }
  free(xd);
  free(xw);
  free(cidx);
  return 1;
}

typedef struct {
  uint64_t key;
  int slot;
} vgp_entry;

static int entry_cmp(const void* a, const void* b) {
  const uint64_t x = ((const vgp_entry*)a)->key, y = ((const vgp_entry*)b)->key;
  return (x > y) - (x < y);
}

/* layers: n layers, voxel_sizes / vps their geometry (one voxel size and voxels_per_side); poses: n x 7 T_M_S
 * [qw qx qy qz tx ty tz]; ids: the submap ids (distinct; they fix the merge order).  Returns a new layer with
 * the global blocks in ascending packed key order ((z + 2^20) << 42 | (y + 2^20) << 21 | (x + 2^20)), or
 * NULL when n < 1, an id repeats, the geometry is mixed or a candidate block index leaves
 * [-(2^20) + 1, 2^20 - 2]. */
vgo_layer* vgp_project_layers(int n, const vgo_layer* const* layers, const float* voxel_sizes, const int* vps,
                              const float* poses, const uint32_t* ids) {
  if (n < 1) return NULL;
  for (int k = 1; k < n; ++k)
    if (voxel_sizes[k] != voxel_sizes[0] || vps[k] != vps[0]) return NULL;
  /* the submaps in increasing id order (cblox iterates a std::map) */
  int* order = (int*)malloc(sizeof(int) * (size_t)n);
  for (int k = 0; k < n; ++k) {
    int j = k;
    while (j > 0 && ids[order[j - 1]] > ids[k]) {
      order[j] = order[j - 1];
      --j;
    }
    order[j] = k;
  }
  int ok = 1;
  for (int k = 1; k < n; ++k)
    if (ids[order[k]] == ids[order[k - 1]]) ok = 0;
  vgp_global G;
  memset(&G, 0, sizeof(G));
  G.index = vgo_layer_create(1.0f, 2);
  G.vpb = vps[0] * vps[0] * vps[0];
  for (int k = 0; k < n && ok; ++k)
    ok = project_one(layers[order[k]], voxel_sizes[0], vps[0], poses + 7 * (size_t)order[k], &G);
  free(order);
  vgo_layer* out = NULL;
  if (ok) {
    /* canonical block order: ascending packed key */
    vgp_entry* e = (vgp_entry*)malloc(sizeof(vgp_entry) * (size_t)(G.n > 0 ? G.n : 1));
    for (int b = 0; b < G.n; ++b) {
      const int32_t* bi = G.idx + 3 * b;
      e[b].key = (uint64_t)(uint32_t)(bi[0] + (1 << 20)) | ((uint64_t)(uint32_t)(bi[1] + (1 << 20)) << 21) |
                 ((uint64_t)(uint32_t)(bi[2] + (1 << 20)) << 42);
      e[b].slot = b;
    }
    qsort(e, (size_t)G.n, sizeof(vgp_entry), entry_cmp);
    out = vgo_layer_create(voxel_sizes[0], vps[0]);
    for (int b = 0; b < G.n; ++b) {
      const int s = e[b].slot;
      vgo_layer_add_block(out, G.idx + 3 * s, G.d + (size_t)s * G.vpb, G.w + (size_t)s * G.vpb);
    }
    free(e);
  }
  vgo_layer_destroy(G.index);
  free(G.idx);
  free(G.d);
  free(G.w);
  return out;
}
