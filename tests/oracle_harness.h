/*
 * oracle_harness.h — the entry points of the three C harnesses built on the CPU oracle
 * (project_oracle.c, project_colour_oracle.c, transform_oracle.c).  TEST INFRASTRUCTURE ONLY.
 * Each harness's ctypes loader declares its function in a SIGNATURES table, which
 * tests/test_host_binding_signatures.py compares with these prototypes.
 */
#ifndef VG_ORACLE_HARNESS_H_
#define VG_ORACLE_HARNESS_H_

#include <stdint.h>

#include "vg_oracle.h"

/* project_oracle.c: cblox SubmapCollection::getProjectedMap -> a new layer, NULL where refused */
vgo_layer* vgp_project_layers(int n, const vgo_layer* const* layers, const float* voxel_sizes, const int* vps,
                              const float* poses, const uint32_t* ids);

/* project_colour_oracle.c: the colour words and weights of the projected map's blocks */
void vgpc_project_colour(int n, const vgo_layer* const* layers, const vgo_layer* const* channels, float vs, int vps,
                         const float* poses, int n_blocks, const int32_t* block_idx, const uint8_t* holds,
                         uint32_t* out_rgba, float* out_weight);

/* transform_oracle.c: voxblox transformLayer into a new layer, NULL where refused */
vgo_layer* vgt_transform_layer(const vgo_layer* S, float vs, int vps, const float T[7]);

#endif /* VG_ORACLE_HARNESS_H_ */
