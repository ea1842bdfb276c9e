/*
 * transform_oracle.c — CPU restatement of voxblox transformLayer(old copy, T_new_old, &own layer) as
 * VoxgraphSubmap::transformSubmap (voxgraph_submap.cpp:38-58) calls it: the checker of vgx_submap_transform.
 * Built at test time by tests/transform_oracle.py against oracle/libvg_oracle.so, whose public functions it
 * reuses for everything voxblox does per point (vgo_interp_voxel, vgo_T_inverse / vgo_T_transform,
 * vgo_grid_index_from_point).  Restated from the published voxblox sources, not checked against a compiled
 * voxblox.  Operation by operation with the same float forms as tests/project_oracle.c; build with
 * -ffp-contract=off.
 *   candidates: per old block b, c = T * ((b + 0.5) * block_size), offset = sqrt(3) * block_size * 0.5; for
 *   x = c.x - offset; x < c.x + offset; x += block_size (same for y, z) the block getGridIndexFromPoint(x, y,
 *   z) is a candidate (as in getProjectedMap's transformLayer);
 *   resampling into the uncleared output layer (= the old layer): every voxel centre of a candidate block,
 *   moved by T.inverse(), is interpolated in the old copy; a success writes (d, w); a failure leaves the
 *   output voxel as it was: the old voxel where the block existed, (0, 0) in a new block; a new block with no
 *   success is removed, an old block never is (bricks carry no has_data flag).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "oracle_harness.h"

#define VGT_BLOCK_INDEX_MIN (-(1 << 20) + 1)
#define VGT_BLOCK_INDEX_MAX ((1 << 20) - 2)

typedef struct {
  uint64_t key;
  int slot;
} vgt_entry;

static int entry_cmp(const void* a, const void* b) {
  const uint64_t x = ((const vgt_entry*)a)->key, y = ((const vgt_entry*)b)->key;
  return (x > y) - (x < y);
}

static uint64_t pack_key(const int32_t* bi) {
  return (uint64_t)(uint32_t)(bi[0] + (1 << 20)) | ((uint64_t)(uint32_t)(bi[1] + (1 << 20)) << 21) |
         ((uint64_t)(uint32_t)(bi[2] + (1 << 20)) << 42);
}

/* S: the old layer (voxel size vs, vps); T: T_new_old [qw qx qy qz tx ty tz].  Returns the transformed layer
 * with its blocks in ascending packed key order, or NULL when a candidate block index leaves
 * [-(2^20) + 1, 2^20 - 2]. */
vgo_layer* vgt_transform_layer(const vgo_layer* S, float vs, int vps, const float T[7]) {
  const float bs = vs * (float)vps;
  const float bs_inv = vgo_layer_block_size_inv(S);
  const int vpb = vps * vps * vps;
  const int nb = vgo_layer_num_blocks(S);
  const size_t nb1 = (size_t)(nb > 0 ? nb : 1);
  int32_t* in_idx = (int32_t*)malloc(sizeof(int32_t) * 3 * nb1);
  float* in_d = (float*)malloc(sizeof(float) * (size_t)vpb * nb1);
  float* in_w = (float*)malloc(sizeof(float) * (size_t)vpb * nb1);
  vgo_layer_export(S, in_idx, in_d, in_w);
  /* output blocks: the old ones (slots 0 .. nb - 1), then new candidates in first-touch order */
  vgo_layer* cand = vgo_layer_create(1.0f, 2);
  int nc = nb, ccap = nb + 64, ok = 1;
  int32_t* cidx = (int32_t*)malloc(sizeof(int32_t) * 3 * (size_t)ccap);
  for (int b = 0; b < nb; ++b) {
    vgo_layer_add_block(cand, in_idx + 3 * b, NULL, NULL);
    memcpy(cidx + 3 * b, in_idx + 3 * b, 3 * sizeof(int32_t));
  }
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
            if (!(f >= (float)VGT_BLOCK_INDEX_MIN && f <= (float)VGT_BLOCK_INDEX_MAX)) ok = 0;
          }
          if (!ok) break;
          int32_t q[3];
          vgo_grid_index_from_point(p, bs_inv, q);
          if (vgo_layer_find_block(cand, q) >= 0) continue;
          vgo_layer_add_block(cand, q, NULL, NULL);
          if (nc == ccap) {
            ccap *= 2;
            cidx = (int32_t*)realloc(cidx, sizeof(int32_t) * 3 * (size_t)ccap);
          }
          memcpy(cidx + 3 * (size_t)nc++, q, sizeof(q));
        }
  }
  vgo_layer_destroy(cand);
  vgo_layer* out = NULL;
  if (ok) {
    float T_old_new[7];
    vgo_T_inverse(T, T_old_new);
    float* od = (float*)malloc(sizeof(float) * (size_t)vpb * (size_t)nc);
    float* ow = (float*)malloc(sizeof(float) * (size_t)vpb * (size_t)nc);
    int* keep = (int*)malloc(sizeof(int) * (size_t)nc);
    for (int c = 0; c < nc; ++c) {
      const int32_t* bi = cidx + 3 * c;
      float* xd = od + (size_t)c * vpb;
      float* xw = ow + (size_t)c * vpb;
      keep[c] = c < nb;
      for (int lin = 0; lin < vpb; ++lin) {
        const int v[3] = {lin % vps, (lin / vps) % vps, lin / (vps * vps)};
        float centre[3], p_in[3];
        for (int a = 0; a < 3; ++a) centre[a] = (float)bi[a] * bs + ((float)v[a] + 0.5f) * vs;
        vgo_T_transform(T_old_new, centre, p_in);
        float d, w;
        if (vgo_interp_voxel(S, p_in, &d, &w)) {
          xd[lin] = d;
          xw[lin] = w;
          keep[c] = 1;
        } else {
          xd[lin] = c < nb ? in_d[(size_t)c * vpb + lin] : 0.0f;
          xw[lin] = c < nb ? in_w[(size_t)c * vpb + lin] : 0.0f;
        }
      }
    }
    vgt_entry* e = (vgt_entry*)malloc(sizeof(vgt_entry) * (size_t)(nc > 0 ? nc : 1));
    int ne = 0;
    for (int c = 0; c < nc; ++c)
      if (keep[c]) {
        e[ne].key = pack_key(cidx + 3 * c);
        e[ne].slot = c;
        ++ne;
      }
    qsort(e, (size_t)ne, sizeof(vgt_entry), entry_cmp);
    out = vgo_layer_create(vs, vps);
    for (int k = 0; k < ne; ++k) {
      const int s = e[k].slot;
      vgo_layer_add_block(out, cidx + 3 * s, od + (size_t)s * vpb, ow + (size_t)s * vpb);
    }
    free(e);
    free(keep);
    free(od);
    free(ow);
  }
  free(cidx);
  free(in_idx);
  free(in_d);
  free(in_w);
  return out;
}
