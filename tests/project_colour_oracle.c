/*
 * project_colour_oracle.c — CPU restatement of the colour that cblox SubmapCollection::getProjectedMap carries,
 * beside tests/project_oracle.c (which restates its distance and weight and is unchanged).  Built at test time by
 * tests/project_colour_oracle.py against oracle/libvg_oracle.so.  Restated from the published voxblox sources, not
 * checked against a compiled voxblox; build with -ffp-contract=off.
 *
 *   Interpolator::interpVoxel: every colour channel is interpolated like the distance, q . (B1 . channel^T) over
 *   the 8 neighbours as floats, and converted to uint8 by truncation (clamped to [0, 255] here, NaN to 0).  The
 *   oracle's vgo_interp_voxel is that very expression for the distance, so a channel is interpolated by calling it
 *   on a layer whose distances are the channel's values as floats (and whose weights are the submap's).
 *   mergeVoxelAIntoVoxelB: w = wA + wB; if (w > 0) { colourB = blendTwoColors(colourA, wA, colourB, wB); weight w }.
 *   blendTwoColors(c1, w1, c2, w2): t = w1 + w2; w1 /= t; w2 /= t; channel = (uint8) round(c1 w1 + c2 w2).
 *
 * Which output blocks a submap's transformed layer holds (transformLayer's candidate enumeration, which can miss
 * blocks at the edge of a rotated submap, and the removal of candidates without data) is not restated again: the
 * caller passes it in, taken from tests/project_oracle.c run on that submap alone.  Inside such a block a voxel
 * whose interpolation fails merges with weight 0: blendTwoColors(cA, 0, cB, wB) is cB exactly and wB + 0 is wB.
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#include "oracle_harness.h"

static uint32_t to_u8(float v) {
  if (!(v == v)) return 0;
  if (v < 0.0f) v = 0.0f;
  if (v > 255.0f) v = 255.0f;
  return (uint32_t)v; /* truncation */
}

static uint32_t blend(uint32_t c1, float w1, uint32_t c2, float w2) {
  const float t = w1 + w2;
  w1 = w1 / t;
  w2 = w2 / t;
  uint32_t out = 0;
  for (int sh = 0; sh < 32; sh += 8) {
    const float a = (float)((c1 >> sh) & 0xffu), b = (float)((c2 >> sh) & 0xffu);
    out |= to_u8(roundf(a * w1 + b * w2)) << sh;
  }
  return out;
}

/* layers: n submaps IN INCREASING ID ORDER; channels: 4 n layers (byte k of the colour word of submap s at
 * channels[4 s + k], distances = channel values), or NULL entries for a submap without a colour channel; poses:
 * n x 7 T_M_S; holds[s * n_blocks + b] != 0: submap s's transformed layer holds output block b.  For the n_blocks
 * output blocks block_idx (as the distance / weight projection found them): out_rgba and out_weight,
 * n_blocks x vps^3. */
void vgpc_project_colour(int n, const vgo_layer* const* layers, const vgo_layer* const* channels, float vs, int vps,
                         const float* poses, int n_blocks, const int32_t* block_idx, const uint8_t* holds,
                         uint32_t* out_rgba, float* out_weight) {
  const float bs = vs * (float)vps;
  const int vpb = vps * vps * vps;
  for (int b = 0; b < n_blocks; ++b) {
    const int32_t* bi = block_idx + 3 * b;
    for (int lin = 0; lin < vpb; ++lin) {
      const int v[3] = {lin % vps, (lin / vps) % vps, lin / (vps * vps)};
      float centre[3];
      for (int a = 0; a < 3; ++a) centre[a] = (float)bi[a] * bs + ((float)v[a] + 0.5f) * vs;
      uint32_t cB = 0;
      float wB = 0.0f;
      for (int s = 0; s < n; ++s) {
        if (!holds[(size_t)s * n_blocks + b]) continue;
        float T_inv[7], p[3], d, w;
        vgo_T_inverse(poses + 7 * s, T_inv);
        vgo_T_transform(T_inv, centre, p);
        if (!vgo_interp_voxel(layers[s], p, &d, &w)) continue;
        uint32_t cA = 0;
        if (channels[4 * s])
          for (int k = 0; k < 4; ++k) {
            float ch, wk;
            vgo_interp_voxel(channels[4 * s + k], p, &ch, &wk);
            cA |= to_u8(ch) << (8 * k);
          }
        if (w + wB > 0) {
          cB = blend(cA, w, cB, wB);
          wB = w + wB;
        }
      }
      out_rgba[(size_t)b * vpb + lin] = cB;
      out_weight[(size_t)b * vpb + lin] = wB;
    }
  }
}
