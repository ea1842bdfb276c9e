/*
 * voxgraph_b200.h — C-ABI of the H100-native voxgraph hot paths.
 *
 * Drop-in boundary for (paths relative to voxgraph/ of the reference, ethz-asl/voxgraph):
 *   b1  RegistrationCostFunction::Evaluate
 *         include/voxgraph/backend/constraint/cost_functions/registration_cost_function.h:47-48
 *         src/backend/constraint/cost_functions/registration_cost_function.cpp:58-298
 *   b2  PoseGraph  (include/voxgraph/backend/pose_graph.h:21-55, src/backend/pose_graph.cpp)
 *   b3  voxblox::TsdfIntegratorBase::integratePointCloud as driven by
 *         PointcloudIntegrator::integratePointcloud
 *         (src/frontend/measurement_processors/pointcloud_integrator.cpp:66-84), and the message
 *         conversion in front of it (cpp:29-63)
 *
 * Conventions: plain pointers and sizes, caller owns every host buffer, the context
 * owns all device memory, every function returns an int status (no exceptions or
 * aborts cross the boundary: a host allocation failure is VGX_ERR_NOMEM).  Every
 * call on a context selects the context's device first.  vgx_last_error() gives the
 * message of the last call on the context, prefixed with the name of the function the
 * caller called.  One context per GPU; a context is not thread-safe.  There is NO CPU
 * fallback: every entry point needs a CUDA device and fails with VGX_ERR_CUDA without one.
 */
#ifndef VOXGRAPH_B200_H_
#define VOXGRAPH_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VGX_OK 0
#define VGX_ZERO_WEIGHT 1      /* Evaluate() would return false (cpp:273) */
#define VGX_ERR_INVALID (-1)
#define VGX_ERR_CUDA (-2)
#define VGX_ERR_NOT_FOUND (-3)
#define VGX_ERR_NOMEM (-4)
#define VGX_ERR_NCCL (-5)
#define VGX_ERR_CAPACITY (-6)

typedef struct vgx_ctx vgx_ctx;

/* ------------------------------------------------------------------ context */
int vgx_device_count(void);
int vgx_ctx_create(int device, vgx_ctx** out);
void vgx_ctx_destroy(vgx_ctx* ctx);
/* The message of the last call on ctx: "<function>: <reason>" after a failure, the
 * function being the one the caller called; empty after a call that returned VGX_OK. */
const char* vgx_last_error(const vgx_ctx* ctx);
/* cudaStream_t all work of this context is enqueued on (for event timing). */
void* vgx_ctx_stream(vgx_ctx* ctx);
int vgx_ctx_synchronize(vgx_ctx* ctx);

/* Kernel accounting: the library runs its kernels in regions, each of one slot (vgx_profile_get's `which`).
 * A slot counts the launches inside its regions, a library sort counting as one launch; a launch outside
 * every region counts in vgx_launch_count only.  When enabled the library also brackets each region with
 * CUDA events on the context stream and adds its time to the slot. */
enum VgxProfileSlotId {
  VGX_SLOT_REG_REDUCE = 0,       /* registration reduce kernel */
  VGX_SLOT_REG_EMIT = 1,         /* registration emit kernel */
  VGX_SLOT_TSDF_INTEGRATE = 2,   /* TSDF integrate kernels (mode 0: count, scan, emit, sort and apply) */
  VGX_SLOT_TSDF_ALLOCATE = 3,    /* TSDF allocate kernel */
  VGX_SLOT_SOLVE = 4,            /* Cholesky / LM kernels */
  VGX_SLOT_OTHER = 5,            /* everything else */
  VGX_SLOT_REG_POSE_SETUP = 6,   /* registration pose set-up */
  VGX_SLOT_REG_SUMS = 7,         /* per-constraint sums */
  VGX_SLOT_ASSEMBLY = 8,         /* assembly of the normal equations (+ the peer exchange when it is fused into it) */
  VGX_SLOT_COLL_CODEC = 9,       /* submap collection codec kernels (decode / encode) */
  VGX_SLOT_COLL_COPY = 10,       /* submap collection stream copies (host <-> device) */
  VGX_SLOT_COLL_UPLOAD = 11,     /* submap collection upload (block hash, registration view, grid) */
  VGX_SLOT_MESH = 12,            /* mesh kernels (vgx_mesh_build's passes and scans, the PLY pack of vgx_mesh_ply) */
  VGX_SLOT_PROJECT = 13,         /* projection kernels (vgx_project_map's passes, sort and scans; the upload of
                                    the result is not included) */
  VGX_SLOT_EVAL = 14,            /* map evaluation kernels (vgx_submap_transform's resampling kernel, the two
                                    vgx_evaluate_layers_rmse kernels) */
  VGX_SLOT_CLOUD_DECODE = 15,    /* point-cloud message decode kernel (vgx_cloud_decode, vgx_tsdf_integrate_cloud;
                                    vgx_cloud_decode's compaction is included, the upload of the bytes is not) */
  VGX_PROFILE_SLOTS = 16
};
int vgx_profile_enable(vgx_ctx* ctx, int on);
int vgx_profile_reset(vgx_ctx* ctx);
int vgx_profile_get(vgx_ctx* ctx, int which, double* total_ms, int64_t* launches);
/* total kernels launched by the library since reset (counted even when disabled) */
int64_t vgx_launch_count(vgx_ctx* ctx);

/* ------------------------------------------------------------------ submaps */
/* Replaces voxblox::Layer<TsdfVoxel|EsdfVoxel> + Block + block hash: dense 16^3 bricks
 * in HBM behind a GPU open-addressing hash keyed on the voxblox block index.
 * A voxel is (distance, weight); observed <=> weight > 1e-6 (upload an ESDF layer with
 * weight = observed ? 1 : 0).  Voxel order inside a block: x + vps*(y + vps*z). */

/* Upload a finished layer (replaces any previous content of submap_id).  Block indices must be
 * distinct and every component within [VGX_BLOCK_INDEX_MIN, VGX_BLOCK_INDEX_MAX], so that the
 * +-1 neighbours every kernel looks up have their own 21-bit hash key; otherwise the upload
 * fails with VGX_ERR_INVALID and submap_id holds no submap afterwards.  The same rules hold for
 * vgx_submap_upload_device. */
#define VGX_BLOCK_INDEX_MIN (-(1 << 20) + 1)
#define VGX_BLOCK_INDEX_MAX ((1 << 20) - 2)
int vgx_submap_upload(vgx_ctx* ctx, uint32_t submap_id, float voxel_size, int voxels_per_side,
                      int n_blocks, const int32_t* block_idx /* n x 3 */,
                      const float* distance /* n x vps^3 */,
                      const float* weight /* n x vps^3 */);
/* Create an empty (active) submap that vgx_tsdf_integrate fills. */
int vgx_submap_create(vgx_ctx* ctx, uint32_t submap_id, float voxel_size, int voxels_per_side,
                      int capacity_blocks);
/* VoxgraphSubmap::finishSubmap (voxgraph_submap.cpp:84-107), device part: freezes the
 * layer and builds the registration view of the bricks. */
int vgx_submap_finish(vgx_ctx* ctx, uint32_t submap_id);
/* The rest of finishSubmap (voxgraph_submap.cpp:84-107) on the device, so that a submap integrated
 * on the GPU never leaves it between HP1 and HP2:
 *   findRelevantVoxelIndices (cpp:144-201)  -> registration points of type VGX_POINTS_VOXELS
 *   findIsosurfaceVertices   (cpp:203-243)  -> registration points of type VGX_POINTS_ISOSURFACE
 *                                              (+ the isosurface block list overlapsWith uses)
 *   getSubmapFrameSurfaceObb (cpp:280-324)
 * Order of the points: blocks in allocation order, voxels in linear order, cube edges 0..11 (the
 * reference iterates a hash map; see oracle/vg_oracle.h vgo_find_isosurface_vertices). */
typedef struct vgx_registration_filter {   /* VoxgraphSubmap::Config::RegistrationFilter (h:26-30) */
  double min_voxel_weight;                 /* 1 */
  double max_voxel_distance;               /* 0.3 */
  int use_esdf_distance;                   /* reference default true: relevant voxels carry the ESDF
                                              distance (cpp:185-189; needs vgx_submap_generate_esdf);
                                              vgx_registration_filter_default sets 0 = TSDF distance */
} vgx_registration_filter;
void vgx_registration_filter_default(vgx_registration_filter* f);
/* On a finished submap (uploaded or integrated). filter may be NULL (defaults). */
int vgx_submap_extract_points(vgx_ctx* ctx, uint32_t submap_id, const vgx_registration_filter* filter);
/* vgx_submap_finish + vgx_submap_extract_points. */
int vgx_submap_finish_ex(vgx_ctx* ctx, uint32_t submap_id, const vgx_registration_filter* filter);
int vgx_submap_num_points(vgx_ctx* ctx, uint32_t submap_id, int point_type, int* n);
/* Copies the registration points back (inspection / parity); any output may be NULL. */
int vgx_submap_download_points(vgx_ctx* ctx, uint32_t submap_id, int point_type, int max_n,
                               float* xyz /* n x 3 */, float* distance, float* weight, int* n);
/* Submap-frame surface OBB; VGX_ZERO_WEIGHT when no voxel qualified (box stays +-inf). */
int vgx_submap_surface_obb(vgx_ctx* ctx, uint32_t submap_id, float obb_min[3], float obb_max[3]);
/* TsdfEsdfSubmap::generateEsdf (finishSubmap, voxgraph_submap.cpp:86) on the device: ESDF bricks
 * + their registration view from the resident TSDF bricks of a finished submap, so that the
 * reference's default registration branch (use_esdf_distance = true,
 * registration_cost_function.h:35, cpp:133-140) has a device producer.  Restates
 * voxblox::EsdfIntegrator's batch update as its fixed point: observed <=> TSDF weight >=
 * min_weight; |tsdf| < min_distance_m is copied (fixed); elsewhere the quasi-Euclidean distance
 * propagated through the 26-neighbourhood of same-sign observed voxels, clipped at max_distance_m
 * (default_distance_m where nothing reaches).  sweeps (may be NULL): relaxation sweeps run. */
typedef struct vgx_esdf_config {      /* voxblox::EsdfIntegrator::Config subset */
  float max_distance_m;               /* 2.0 */
  float default_distance_m;           /* 2.0 */
  float min_distance_m;               /* 0.2 */
  float min_weight;                   /* 1e-6 */
} vgx_esdf_config;
void vgx_esdf_config_default(vgx_esdf_config* cfg);
int vgx_submap_generate_esdf(vgx_ctx* ctx, uint32_t submap_id, const vgx_esdf_config* cfg, int* sweeps);
/* ESDF bricks in block (allocation) order: distance and observed (1 / 0) per voxel. */
int vgx_submap_download_esdf(vgx_ctx* ctx, uint32_t submap_id, int max_blocks, float* distance,
                             float* observed, int* n_blocks);

/* PoseGraphInterface::updateOverlappingSubmapList (pose_graph_interface.cpp:109-147) over
 * VoxgraphSubmap::overlapsWith (voxgraph_submap.cpp:245-278): mission-frame surface-AABB rejection,
 * then "any isosurface block centre of the first submap lands in an allocated block of the second",
 * for every i < j of the list.  poses: n x 7 = T_mission_submap [qw qx qy qz tx ty tz] (float, as
 * cblox stores them).  Needs vgx_submap_extract_points on every submap.  pairs: 2 ids per pair. */
int vgx_find_overlapping_pairs(vgx_ctx* ctx, int n, const uint32_t* submap_ids, const float* poses,
                               int max_pairs, uint32_t* pairs, int* n_pairs);
int vgx_submap_free(vgx_ctx* ctx, uint32_t submap_id);
int vgx_submap_block_count(vgx_ctx* ctx, uint32_t submap_id, int* n_blocks);
/* Layer geometry and state (any output may be NULL). */
int vgx_submap_info(vgx_ctx* ctx, uint32_t submap_id, float* voxel_size, int* voxels_per_side,
                    int* n_blocks, int* finished);
/* Copies blocks back in allocation order (parity checks / saving). */
int vgx_submap_download(vgx_ctx* ctx, uint32_t submap_id, int max_blocks, int32_t* block_idx,
                        float* distance, float* weight, int* n_blocks);

/* Device-to-device hand-over of a finished submap between two contexts (BASELINE configs[4]: one
 * GPU integrates, the other registers; the finished submap crosses NVLink once).  peek: read-only
 * device pointers of the resident bricks (block indices n x 3 int32, voxels n x vps^3 x
 * {distance, weight} float) - valid until the submap is modified or freed; the caller moves them
 * with its own transport (ncclSend / cudaMemcpyPeer).  upload_device: same as vgx_submap_upload but
 * from device memory of this context's GPU, interleaved (distance, weight) voxels. */
int vgx_submap_peek_device(vgx_ctx* ctx, uint32_t submap_id, const int32_t** d_block_idx,
                           const float** d_distance_weight, int* n_blocks);
int vgx_submap_upload_device(vgx_ctx* ctx, uint32_t submap_id, float voxel_size, int voxels_per_side,
                             int n_blocks, const int32_t* d_block_idx, const float* d_distance_weight);

/* Voxel colour (voxblox Color: 4 x uint8 r, g, b, a; default 0, 0, 0, 0).  A submap has NO colour channel
 * until something gives it one: the first vgx_tsdf_integrate with rgba != NULL, vgx_submap_upload_colour /
 * vgx_submap_upload_device_colour, or vgx_collection_load_ex with VGX_COLLECTION_KEEP_COLOUR.  A submap without
 * a channel runs every call exactly as before colour existed (same kernels, same bytes, same statistics).  The
 * channel costs 4 bytes per voxel of the submap's capacity, starts zero, survives vgx_submap_finish*, and is
 * released with the submap.  One uint32 per voxel, in block (allocation) order and linear voxel order, held
 * exactly as the third word of a voxel in a collection file; restated from the published voxblox sources and
 * not checked against a compiled voxblox, that word is   a | b << 8 | g << 16 | r << 24.
 * Colour follows the data: vgx_collection_save writes it, vgx_project_map gives its output a channel when an
 * input has one, vgx_mesh_build computes vertex colours for submaps that have one.  vgx_layer_load does not
 * read it, and vgx_submap_transform (used only on the evaluation path) drops it: its result has no channel.
 *   has:            *has = 1 when the submap has a channel, else 0.
 *   download:       n_blocks x vps^3 words (zeros when there is no channel); VGX_ERR_CAPACITY when max_blocks is
 *                   too small (*n_blocks is set either way); rgba may be NULL to query the count.
 *   upload:         replaces (or creates) the channel of an existing submap; n_blocks must equal the submap's.
 *   peek / upload_device: the same from device memory of this context's GPU, for the device-to-device
 *                   hand-over of vgx_submap_peek_device / vgx_submap_upload_device; peek gives NULL when there
 *                   is no channel (valid until the submap is modified or freed). */
int vgx_submap_has_colour(vgx_ctx* ctx, uint32_t submap_id, int* has);
int vgx_submap_download_colour(vgx_ctx* ctx, uint32_t submap_id, int max_blocks, uint32_t* rgba /* n x vps^3 */,
                               int* n_blocks);
int vgx_submap_upload_colour(vgx_ctx* ctx, uint32_t submap_id, int n_blocks, const uint32_t* rgba);
int vgx_submap_peek_device_colour(vgx_ctx* ctx, uint32_t submap_id, const uint32_t** d_rgba);
int vgx_submap_upload_device_colour(vgx_ctx* ctx, uint32_t submap_id, int n_blocks, const uint32_t* d_rgba);

/* ------------------------------------------------------------------ submap collection files */
/* cblox::SubmapCollection::saveToFile / cblox::io::LoadSubmapCollection (TSDF layers), as byte
 * buffers.  The stream is a sequence of varint-length-delimited proto2 messages: one
 * SubmapCollectionProto {1 voxel_size: double, 2 voxels_per_side, 3 num_submaps}, then per submap in
 * increasing id order one SubmapProto {1 id, 2 num_blocks, 3 transform: T_M_S} followed by num_blocks
 * BlockProto {1 voxels_per_side, 2 voxel_size, 3-5 origin, 6 has_data, 7 voxel_data: 3 words per voxel
 * = distance bits, weight bits, colour}.  The format is restated from the published voxblox / cblox
 * sources and has not been checked against a file written by cblox; the reader is strict
 * (VGX_ERR_INVALID on any deviation, unknown fields skipped; see csrc/collection.cu).  Colour:
 * vgx_collection_save writes the colour word of every submap that has a colour channel and 0 (voxblox's default
 * Color()) for the others; vgx_collection_load drops the colour words, vgx_collection_load_ex keeps them on
 * request, so a foreign file then round-trips bit-exactly, colour included.  The voxel payload is decoded
 * and encoded on the device; the host walks message headers only. */
typedef struct vgx_collection_entry {
  uint32_t id;
  uint32_t num_blocks;
  float voxel_size;
  int32_t voxels_per_side;
  float T_M_S[7];              /* qw qx qy qz tx ty tz (cblox stores doubles; the library uses float) */
} vgx_collection_entry;
/* Host only (no context, no GPU): validates the framing of the whole stream and describes its
 * submaps in stream order.  *n_submaps is set on success and on VGX_ERR_CAPACITY (max_submaps too
 * small; out may be NULL when max_submaps is 0). */
int vgx_collection_scan(const uint8_t* bytes, uint64_t n, int max_submaps, vgx_collection_entry* out,
                        int* n_submaps);
/* Creates every submap of the stream under its stored id as a finished upload (the rules of
 * vgx_submap_upload apply); the caller runs vgx_submap_finish_ex and, where wanted,
 * vgx_submap_generate_esdf, as finishSubmap does after VoxgraphSubmap::LoadFromStream.  All or
 * nothing: if an id of the stream already exists in the context or anything fails, VGX_ERR_INVALID
 * (or the CUDA error) is returned and no submap of the stream is left; other submaps are untouched. */
int vgx_collection_load(vgx_ctx* ctx, const uint8_t* bytes, uint64_t n, int* n_submaps);
/* vgx_collection_load with flags (0: the same call).  VGX_COLLECTION_KEEP_COLOUR: a submap of the stream gets
 * a colour channel holding its colour words iff any of them is non-zero.  Other bits give VGX_ERR_INVALID. */
#define VGX_COLLECTION_KEEP_COLOUR 1
int vgx_collection_load_ex(vgx_ctx* ctx, const uint8_t* bytes, uint64_t n, int flags, int* n_submaps);
/* Writes the n submaps (active or finished; one voxel size and voxels_per_side) in increasing id
 * order with poses T_M_S (n x 7, qw qx qy qz tx ty tz; ids[i] goes with row i).  Blocks are written in
 * allocation order, voxel_data unpacked.  out == NULL: only *size is set.  capacity < *size:
 * VGX_ERR_CAPACITY with *size set. */
int vgx_collection_save(vgx_ctx* ctx, int n, const uint32_t* ids, const float* T_M_S, uint8_t* out,
                        uint64_t capacity, uint64_t* size);

/* ------------------------------------------------------------------ submap meshes */
/* SubmapVisuals::publishSeparatedMesh / saveSeparatedMesh (voxgraph src/tools/visualization/
 * submap_visuals.cpp:68-97): cblox SubmapMesher::generateSeparatedMesh over voxblox
 * MeshIntegrator::generateMesh (a full re-mesh), then voxblox::outputMeshLayerAsPly.  The mesh is a
 * watertight shared-vertex marching-cubes mesh: a cube is meshed when its 8 corners have weight >
 * min_weight, one vertex per crossing lattice edge interpolated from its low end, triangles by a
 * face-walk rule (ambiguous faces join the crossings at their negative corners; fronts face the
 * positive side), which is not voxblox's table (see csrc/mesh.cu for the full rule and order).
 * Vertices are float32 in the mission frame, triangle indices uint32 into the whole mesh. */
typedef struct vgx_mesh_config {   /* voxblox::MeshIntegratorConfig subset */
  float min_weight;                /* voxgraph_mapper.yaml:52 mesh_min_weight: 2.0 */
} vgx_mesh_config;
void vgx_mesh_config_default(vgx_mesh_config* cfg);
/* Separated mesh of n submaps (active or finished), in the order given, into the context's mesh buffer,
 * which the next build or vgx_ctx_destroy releases; n = 0 releases it.  T_M_S: n x 7 [qw qx qy qz tx ty
 * tz] or NULL (submap frames); cfg may be NULL (defaults).  vertex_offsets / triangle_offsets: n + 1
 * entries each (submap k owns [offsets[k], offsets[k + 1])), may be NULL.  An unknown id gives
 * VGX_ERR_NOT_FOUND and an empty mesh; more than 2^31 - 1 vertices or triangles VGX_ERR_CAPACITY. */
int vgx_mesh_build(vgx_ctx* ctx, int n, const uint32_t* submap_ids, const float* T_M_S,
                   const vgx_mesh_config* cfg, int64_t* vertex_offsets, int64_t* triangle_offsets);
/* Copies the mesh of the last build: xyz n_vertices x 3, triangles n_triangles x 3 (either may be
 * NULL; the counts are always set).  VGX_ERR_CAPACITY when a non-NULL output is too small. */
int vgx_mesh_download(vgx_ctx* ctx, int64_t max_vertices, float* xyz, int64_t max_triangles,
                      uint32_t* triangles, int64_t* n_vertices, int64_t* n_triangles);
/* Binary little-endian PLY of the last build: vertex {float x, y, z; uchar red, green, blue, alpha},
 * face {list uchar int vertex_indices}.  rgba: one colour per submap of the build (n x 4), or NULL for
 * voxblox's rainbowColorMap((id mod 20) / 20).  out == NULL: only *size is set.  capacity < *size:
 * VGX_ERR_CAPACITY with *size set. */
int vgx_mesh_ply(vgx_ctx* ctx, const uint8_t* rgba, uint8_t* out, uint64_t capacity, uint64_t* size);
/* Vertex colours (voxblox MeshIntegrator::updateMeshColor, use_color = true; restated, not checked against a
 * compiled voxblox): when a submap of the build has a colour channel, vgx_mesh_build also gives every vertex the
 * colour word of the voxel that contains it, voxel index floor(p / voxel_size + 1e-6) of the vertex in the submap's
 * own frame (before T_M_S); a build without such a submap launches the kernels it always launched.
 * download_colours: one colour word per vertex (the layout of vgx_submap_download_colour), 0 for the vertices of
 * submaps without a channel; rgba may be NULL to query the count; VGX_ERR_CAPACITY when max_vertices is too small.
 * ply_ex: vgx_mesh_ply (voxel_colours = 0), or with voxel_colours != 0 the PLY in which the vertices of submaps
 * with a channel carry their voxel colour and the others the per-submap colour given (what
 * SubmapVisuals::saveCombinedMesh writes for the projected map). */
int vgx_mesh_download_colours(vgx_ctx* ctx, int64_t max_vertices, uint32_t* rgba, int64_t* n_vertices);
int vgx_mesh_ply_ex(vgx_ctx* ctx, const uint8_t* rgba, int voxel_colours, uint8_t* out, uint64_t capacity,
                    uint64_t* size);

/* ------------------------------------------------------------------ projected global map */
/* cblox SubmapCollection::getProjectedMap: every submap merged, at its pose, into one mission-frame TSDF
 * layer (voxblox mergeLayerAintoLayerB = transformLayer + the untransformed merge).  What
 * save_combined_mesh / publish_combined_mesh (cblox generateCombinedMesh: vgx_mesh_build_combined below),
 * ProjectedMapServer and MapEvaluation consume.  The rule is restated from the published voxblox / cblox
 * sources and has not been checked against a compiled voxblox (see csrc/project.cu; the CPU restatement
 * tests/project_oracle.c pins it bit for bit):
 *   - all submaps share one voxel size and voxels_per_side (cblox never mixes them; voxblox's resampling
 *     branch is not ported); they are merged in increasing id order whatever the order of submap_ids;
 *   - candidate output blocks: per allocated block b, c = T_M_S * ((b + 0.5) * block_size), and per axis
 *     the samples x = c - sqrt(3) * block_size / 2, x + block_size (a float loop while x < c + offset), so
 *     8 sample points whose blocks floor(p / block_size + 1e-6) are candidates (this can miss blocks at the
 *     edge of a rotated submap, as the reference does);
 *   - every voxel centre of a candidate block is moved by T_M_S.inverse() and interpolated trilinearly
 *     (Interpolator::getVoxel, all 8 neighbours observed); a failure leaves (0, 0); a candidate block
 *     with no success does not exist for that submap;
 *   - every voxel of an existing block, (0, 0) ones included, is merged: w = wA + wB; if w > 0:
 *     d = (dA * wA + dB * wB) / w and weight w (float, no FMA; no float atomics, so the result does not
 *     depend on thread order).
 * Colour: when an input has a colour channel the output gets one: the resampling interpolates every channel like
 * the distance and truncates to uint8 (clamped to [0, 255]), the merge does, inside its if (w > 0), colourB =
 * blendTwoColors(colourA, wA, colourB, wB); an input without a channel contributes colour 0 with its weight.  With
 * no coloured input the launches and the output are the colour-free ones.  T_M_S: n x 7 [qw qx qy qz tx ty tz], row i for submap_ids[i]; inputs may be
 * active or finished.  Creates out_id as a finished upload (the state vgx_collection_load leaves: run
 * vgx_submap_finish_ex / vgx_submap_generate_esdf / vgx_mesh_build / vgx_collection_save /
 * vgx_submap_download on it) with its blocks in ascending packed key order ((z + 2^20) << 42 |
 * (y + 2^20) << 21 | (x + 2^20)); *n_blocks (may be NULL) its block count, 0 when nothing projects.
 * An unknown id gives VGX_ERR_NOT_FOUND; n < 1, a repeated id, out_id among the inputs or already
 * existing, mixed voxel geometry, or a candidate block index outside [VGX_BLOCK_INDEX_MIN,
 * VGX_BLOCK_INDEX_MAX] give VGX_ERR_INVALID.  On any error no out_id is left and no other submap
 * changes.  Device memory besides the new submap: 8 (key, submap) pairs per input block and the sort's
 * scratch. */
int vgx_project_map(vgx_ctx* ctx, int n, const uint32_t* submap_ids, const float* T_M_S /* n x 7 */,
                    uint32_t out_id, int* n_blocks);
/* cblox SubmapMesher::generateCombinedMesh: vgx_project_map of the n submaps at T_M_S (n x 7) into a scratch
 * submap (the first unused id counting down from 2^32 - 2), vgx_mesh_build of that one submap with cfg (may be
 * NULL: defaults), and the scratch submap freed on every exit, so the context's submaps are unchanged.  The mesh
 * is left in the context's mesh buffer for vgx_mesh_download / vgx_mesh_ply_ex; SubmapVisuals::saveCombinedMesh
 * is vgx_mesh_ply_ex with voxel_colours = 1 and one colour.  Errors are those of the two calls. */
int vgx_mesh_build_combined(vgx_ctx* ctx, int n, const uint32_t* submap_ids, const float* T_M_S /* n x 7 */,
                            const vgx_mesh_config* cfg);

/* Registration points of a submap = WeightedSampler<RegistrationPoint> items
 * (include/voxgraph/frontend/submap_collection/registration_point.h:6-12).
 * point_type: 0 = kVoxels, 1 = kIsosurfacePoints (voxgraph_submap.h RegistrationPointType). */
#define VGX_POINTS_VOXELS 0
#define VGX_POINTS_ISOSURFACE 1
int vgx_submap_upload_points(vgx_ctx* ctx, uint32_t submap_id, int point_type, int n,
                             const float* xyz /* n x 3 */, const float* distance,
                             const float* weight);

/* ------------------------------------------------------------------ b3: TSDF integration */
typedef struct vgx_tsdf_config {          /* voxblox::TsdfIntegratorBase::Config */
  float default_truncation_distance;      /* voxgraph_mapper.yaml:23  0.6 */
  float max_weight;                       /* 10000 */
  int voxel_carving_enabled;              /* 1 */
  float min_ray_length_m;                 /* 0.1 */
  float max_ray_length_m;                 /* yaml:24  16 */
  int use_const_weight;                   /* yaml:25  1 */
  int allow_clear;                        /* 1 */
  int use_weight_dropoff;                 /* yaml:26  1 */
  int use_sparsity_compensation_factor;   /* yaml:27  1 */
  float sparsity_compensation_factor;     /* yaml:28  20 */
  float start_voxel_subsampling_factor;   /* FastTsdfIntegrator, 2 */
  int max_consecutive_ray_collisions;     /* FastTsdfIntegrator, 2.  Both approximate sets start each
                                             call filled with ~0, which index (-1, 0, 0) also hashes to:
                                             its first visit counts as a collision, and a point whose
                                             start cell is (-1, 0, 0) is never cast.  A point with a NaN
                                             or infinite coordinate touches neither set. */
  int mode;                               /* 0 simple (every ray, every voxel; the updates of each
                                             voxel are applied in ray order = bit-identical to the
                                             single-threaded reference), 1 fast (FastTsdfIntegrator
                                             scheduling, what voxgraph runs) */
  int deterministic;                      /* ignored (kept for layout compatibility): mode 0 is always
                                             ray ordered */
} vgx_tsdf_config;

typedef struct vgx_tsdf_stats {
  int64_t rays_valid;
  int64_t rays_cast;
  int64_t voxel_updates;
  int64_t blocks_allocated;
  int64_t saturated_batches;   /* mode 0: 32-update batches of sensor-adjacent voxels collapsed in
                                  closed form (distance pinned at +trunc, exact integer weight sum) */
} vgx_tsdf_stats;

void vgx_tsdf_config_default(vgx_tsdf_config* cfg);
/* integratePointCloud(T_G_C, points_C, colors): T_G_C = [qw qx qy qz tx ty tz].
 * Host buffers; copies are part of the call.
 * rgba: one r, g, b, a byte quadruple per point, or NULL.  With colours the submap gets a colour channel (see
 * vgx_submap_has_colour) and every update inside the truncation band blends the ray's colour into the voxel
 * (updateTsdfVoxel: colour = blendTwoColors(colour, weight before the update, ray colour, update weight) when
 * |sdf| < truncation; restated, not checked against a compiled voxblox).  Distance, weight, statistics and
 * the block set never depend on rgba.  mode 0: the colour too is bit-identical to a sequential replay of the
 * rays.  mode 1: a voxel with a single update in the call holds the exact result (in general the weight the
 * rule uses is one the voxel held at some point during the call); otherwise every
 * channel lies within the closed range spanned by the voxel's previous colour and the colours of the rays
 * that updated it in the band; exactly c when the previous colour is c, or the previous weight is 0 and
 * every update of the voxel in the call is a band update of colour c (csrc/tsdf.cu).  NULL on a submap
 * that has a channel leaves the channel untouched (voxblox would blend in its default Color()).
 * Index range (both modes): a block with a component outside [VGX_BLOCK_INDEX_MIN,
 * VGX_BLOCK_INDEX_MAX] (in the submap frame, |coordinate| beyond about 2^20 block sizes) is never
 * allocated.  Its voxels are skipped: not updated, not counted in voxel_updates, no capacity error;
 * the ray still counts in rays_valid / rays_cast.  Every downloaded block index is therefore one
 * vgx_submap_upload accepts. */
int vgx_tsdf_integrate(vgx_ctx* ctx, uint32_t submap_id, const float T_G_C[7], int n,
                       const float* points_C /* n x 3 */, const uint8_t* rgba /* n x 4 or NULL */,
                       const vgx_tsdf_config* cfg, vgx_tsdf_stats* stats /* may be NULL */);

/* vgx_tsdf_integrate with the points (n x 3 float) and the optional colours (n words, bytes r g b a in memory
 * order) already in device memory of this context's GPU: no copy of the points is made.  The work is enqueued
 * on the context's stream (vgx_ctx_stream); the caller makes sure whatever produced the buffers has finished, or
 * is ordered before that stream, and keeps them alive until the call returns (it returns after the statistics
 * are back, so the kernels are done).  Host memory or memory of another GPU gives VGX_ERR_INVALID before any
 * launch.  Everything else - modes, colour rule, index range, statistics, launches - is vgx_tsdf_integrate's. */
int vgx_tsdf_integrate_device(vgx_ctx* ctx, uint32_t submap_id, const float T_G_C[7], int n,
                              const float* d_points_C /* n x 3 */, const uint32_t* d_rgba /* n or NULL */,
                              const vgx_tsdf_config* cfg, vgx_tsdf_stats* stats /* may be NULL */);

/* ------------------------------------------------------------------ b3: point-cloud messages */
/* The first half of PointcloudIntegrator::integratePointcloud (pointcloud_integrator.cpp:29-63): a
 * sensor_msgs::PointCloud2 becomes voxblox::Pointcloud + voxblox::Colors through pcl::fromROSMsg and
 * voxblox::convertPointcloud.  Restated here from the published ROS message definition and the published PCL /
 * voxblox sources; nothing is copied from them and nothing was checked against a compiled PCL or voxblox.  The
 * raw message bytes are uploaded once and decoded by a kernel; the host never walks the records.
 * vgx_cloud_layout is the part of the message fromROSMsg reads, the caller having matched the fields by name
 * (the front ends do: `rgb` makes an XYZRGB cloud, else `intensity` an XYZI cloud, else XYZ; cpp:33-63).  Little
 * endian only.  Offsets are byte offsets inside one record. */
typedef struct vgx_cloud_layout {
  uint32_t width, height;        /* width * height records; height > 1 = organised cloud */
  uint32_t point_step, row_step; /* bytes per record / per row (row_step >= width * point_step) */
  int32_t x_offset, y_offset, z_offset;   /* FLOAT32 each */
  int32_t rgb_offset;            /* -1: none.  4 bytes b, g, r, a (PCL's packed rgb) */
  int32_t intensity_offset;      /* -1: none.  FLOAT32.  Ignored when rgb_offset >= 0 (cpp:45-56) */
} vgx_cloud_layout;
/* Rules (record i = row i / width, column i mod width, at byte row * row_step + column * point_step):
 *   Finite filter.  A record is kept iff x, y and z are all finite (voxblox isPointFinite).  Kept records keep
 *     their message order; n_points is their count.
 *   Colours.  rgb: Color(r, g, b, a) = bytes 2, 1, 0, 3 of the packed word; the alpha byte is carried as the
 *     message has it, not forced to 255.  intensity: h = clamp(intensity, 0, colour_map_max) / colour_map_max in
 *     float, every channel round(h * 255), alpha 255 (GrayscaleColorMap; the reference sets the maximum to 10000,
 *     cpp:14).  A NaN intensity on a finite point is black: voxblox clamps with std::min(max, std::max(min,
 *     value)), and std::max(0, NaN) is 0 by the standard's definition (a < b ? b : a); this is restated, not
 *     observed.  Neither field: colorLookup(0) = (0, 0, 0, 255).
 *   Validation, all VGX_ERR_INVALID with nothing changed: a NULL layout; point_step == 0; an x, y or z offset
 *     that is negative or ends (offset + 4) beyond point_step; an rgb or intensity offset that is neither -1 nor
 *     inside the record; row_step < width * point_step; n_bytes < height * row_step; width * height > INT_MAX;
 *     data == NULL with records to read; colour_map_max not a finite value > 0.  Offsets, point_step and
 *     row_step need not be multiples of 4: PCL's layouts are, the message format does not promise it, and
 *     records of up to 128 bytes at any alignment take the same kernel path (a warp stages its 32 records in
 *     shared memory with 16-byte loads); longer records are read field by field.
 *
 * vgx_cloud_decode: convertPointcloud's result brought back (inspection / parity, like vgx_submap_draw_samples):
 *   the kept points compacted in message order (points_C n x 3, rgba n x 4 r g b a; either may be NULL) and
 *   *n_points.  More kept points than max_points with a non-NULL output: VGX_ERR_CAPACITY, *n_points set.
 *
 * vgx_tsdf_integrate_cloud: PointcloudIntegrator::integratePointcloud, decode and integration in one call with
 *   one upload of height * row_step message bytes and no host pass over the points.  colours != 0: as the
 *   reference, every cloud type yields colours (an XYZ cloud's are (0, 0, 0, 255)) and the submap gets a colour
 *   channel; colours == 0: the points are integrated without colours and the channel is neither created nor
 *   touched.  The result is the one vgx_tsdf_integrate gives for the kept points and their colours: the
 *   dropped records stay in place as non-finite points, which integration skips and does not count (see
 *   max_consecutive_ray_collisions above), so in mode 0 every voxel still sees its updates in message order and
 *   the result is bit-identical; in mode 1 the usual contract between two runs of one scan holds.  Submap
 *   errors are vgx_tsdf_integrate's (unknown: VGX_ERR_NOT_FOUND; finished: VGX_ERR_INVALID), and so are modes,
 *   block-index range and colour blending.  An empty cloud (width * height == 0) is VGX_OK with zero statistics
 *   and creates no colour channel; a cloud whose records are all dropped still does when colours != 0.
 *   *n_points (may be NULL): the kept records; it arrives in the copy that brings the statistics back.
 *   One launch more than vgx_tsdf_integrate whatever the size (profiling slot VGX_SLOT_CLOUD_DECODE). */
int vgx_cloud_decode(vgx_ctx* ctx, const vgx_cloud_layout* layout, const uint8_t* data, uint64_t n_bytes,
                     float colour_map_max, int max_points, float* points_C, uint8_t* rgba, int* n_points);
int vgx_tsdf_integrate_cloud(vgx_ctx* ctx, uint32_t submap_id, const float T_G_C[7], const vgx_cloud_layout* layout,
                             const uint8_t* data, uint64_t n_bytes, int colours, float colour_map_max,
                             const vgx_tsdf_config* cfg, vgx_tsdf_stats* stats /* may be NULL */,
                             int* n_points /* may be NULL */);

/* ------------------------------------------------------------------ b1: cost function */
typedef struct vgx_reg_config {           /* RegistrationCostFunction::Config (h:17-41) */
  int registration_point_type;            /* VGX_POINTS_* ; default isosurface */
  double no_correspondence_cost;          /* 0 */
  float sampling_ratio;                   /* -1: every registration point, in order (cpp:115-117).
                                             Otherwise (voxgraph_mapper.yaml:34 uses 0.05):
                                             num_residuals = int(ratio * K) points are drawn with
                                             probability proportional to their weight from the
                                             reference submap's WeightedSampler (a default-seeded
                                             std::mt19937 per submap and point type,
                                             weighted_sampler_inl.h:19-28) and their weight is
                                             forced to 1 (cpp:118-122). */
  int use_esdf_distance;                  /* h:35 (reference default true): interpolate the reading
                                             submap's ESDF (vgx_submap_generate_esdf) instead of its
                                             TSDF (cpp:133-153).  vgx_reg_config_default sets 0. */
} vgx_reg_config;
void vgx_reg_config_default(vgx_reg_config* cfg);

/* Number of residuals of the (reference -> reading) cost function (cpp:45-55). */
int vgx_reg_num_residuals(vgx_ctx* ctx, uint32_t reference_submap_id, const vgx_reg_config* cfg,
                          int* num_residuals);
/* Evaluate(parameters, residuals, jacobians): Ceres layout, residuals[K] and two K x 4
 * row-major Jacobian blocks (either may be NULL). Returns VGX_OK, or VGX_ZERO_WEIGHT
 * where Evaluate returns false.  In sampling mode every call draws a fresh sample from the
 * reference submap's generator, exactly as every Evaluate does in the reference.
 * Index range (here and in vgx_graph_eval): no block exists outside [VGX_BLOCK_INDEX_MIN,
 * VGX_BLOCK_INDEX_MAX], so a point whose block lies outside it has no correspondence, as in the
 * reference, whose blocks can never be there (uploads and integration refuse them). */
int vgx_reg_eval_emit(vgx_ctx* ctx, uint32_t reference_submap_id, uint32_t reading_submap_id,
                      const vgx_reg_config* cfg, const double reference_pose[4],
                      const double reading_pose[4], double* residuals, double* jac_reference,
                      double* jac_reading);

/* WeightedSampler::getRandomItem (weighted_sampler_inl.h:19-28) n times on the submap's
 * generator: writes the n drawn point indices and advances the generator (inspection / parity
 * tests; the same routine feeds the sampling mode of b1 and b2). */
int vgx_submap_draw_samples(vgx_ctx* ctx, uint32_t submap_id, int point_type, int n,
                            int32_t* indices);

/* ------------------------------------------------------------------ b2: pose graph */
/* addSubmapNode for every node (replaces the node set). xyzyaw: n x 4 [x,y,z,yaw]. */
int vgx_graph_set_nodes(vgx_ctx* ctx, int n, const uint32_t* submap_ids, const double* xyzyaw,
                        const uint8_t* constant);
int vgx_graph_set_poses(vgx_ctx* ctx, const double* xyzyaw);
int vgx_graph_get_poses(vgx_ctx* ctx, double* xyzyaw);
/* add{Relative,Absolute}PoseConstraint: m edges, observed [tx,ty,tz,yaw], sqrt-information
 * (vgx_sqrt_information of the edge's information matrix, row-major 4x4). */
int vgx_graph_set_relative_edges(vgx_ctx* ctx, int m, const uint32_t* ids_a, const uint32_t* ids_b,
                                 const double* t_obs_xyzyaw, const double* sqrt_info);
/* Host-only: the Constraint constructor's square-root information factor (constraint.cpp:4-38) of a
 * row-major 4x4 information matrix.  allow_semi_definite = 0: the lower LLT factor, rejected when a pivot
 * is not > 0.  allow_semi_definite != 0: Eigen's LDLT with diagonal pivoting, sqrt = P^T L sqrt(D) P,
 * rejected when a pivot is below -1e-12 * (1 + max |diagonal entry|); a pivot between that bound and 0 gives a zero column.
 * A rejected matrix or a NULL pointer gives VGX_ERR_INVALID. */
int vgx_sqrt_information(const double information[16], int allow_semi_definite, double sqrt_information[16]);
/* One entry per registration residual block (reference -> reading). The caller adds the
 * mirrored block for isosurface points as PoseGraph::addRegistrationConstraint does
 * (pose_graph.cpp:63-71). Replaces the previous list (resetRegistrationConstraints). */
int vgx_graph_set_registration_constraints(vgx_ctx* ctx, int p, const uint32_t* reference_ids,
                                           const uint32_t* reading_ids, const vgx_reg_config* cfg);
/* Same with one config per residual block (the reference keeps a Config per constraint,
 * registration_constraint.h:15-21). */
int vgx_graph_set_registration_constraints_v(vgx_ctx* ctx, int p, const uint32_t* reference_ids,
                                             const uint32_t* reading_ids,
                                             const vgx_reg_config* cfgs /* p entries */);
/* Sampling mode inside the fused evaluation: the reference re-draws on every Evaluate, i.e. the
 * cost Ceres compares between two LM iterations is stochastic.  The fused path draws ONCE per
 * constraint when the constraint list is (re)built - PoseGraphInterface resets and re-adds the
 * registration constraints before every optimize() (pose_graph_interface.cpp:149-175), so every
 * solve gets a fresh draw from the submap's generator - and keeps it for all evaluations of
 * that solve.  Every rank draws for every constraint, so the streams stay identical across
 * ranks.  get: the indices in use (n = num_residuals of that block); set: replace them
 * (parity tests against an oracle fed with the same list). constraint = index in the list. */
int vgx_graph_get_sample_indices(vgx_ctx* ctx, int constraint, int max_n, int32_t* indices, int* n);
int vgx_graph_set_sample_indices(vgx_ctx* ctx, int constraint, int n, const int32_t* indices);
int vgx_graph_num_registration_residuals(vgx_ctx* ctx, int64_t* local, int64_t* global);

/* Whole-problem evaluation at the current poses, fused on the device: cost = 1/2 sum r^2,
 * gradient = J^T r (4 per node), H = J^T J (dense 4N x 4N row-major). Outputs may be NULL.
 * With a communicator the result is the all-reduced global one. */
int vgx_graph_eval(vgx_ctx* ctx, int exclude_registration, double* cost, double* gradient,
                   double* H);
/* Enqueue only (no device->host copy, no sync): for device-side timing. */
int vgx_graph_eval_async(vgx_ctx* ctx, int exclude_registration);
/* Sum of squared residuals per registration constraint (pose_graph.cpp:194-207). */
int vgx_graph_registration_costs(vgx_ctx* ctx, double* per_constraint);

typedef struct vgx_solver_options {       /* ceres::Solver::Options subset, pose_graph.cpp:91-97 */
  int max_num_iterations;                 /* 50 */
  double parameter_tolerance;             /* 3e-3 */
  double function_tolerance;              /* 1e-6 */
  double gradient_tolerance;              /* 1e-10 */
  double initial_trust_region_radius;     /* 1e4 */
  double max_trust_region_radius;         /* 1e16 */
  double min_trust_region_radius;         /* 1e-32 */
  double min_relative_decrease;           /* 1e-3 */
  double min_lm_diagonal;                 /* 1e-6 */
  double max_lm_diagonal;                 /* 1e32 */
  double max_solver_time_s;               /* 4 */
  int jacobi_scaling;                     /* 1 */
  int exclude_registration;               /* PoseGraph::optimize(bool) */
} vgx_solver_options;

typedef struct vgx_solver_summary {       /* what voxgraph reads off ceres::Solver::Summary */
  int iterations;
  int num_successful_steps;
  int num_residual_evals;  /* 1 (the start) + one per candidate evaluated; Ceres also counts the
                             re-evaluation after an accepted step, which the device fuses into the
                             candidate's */
  int termination;  /* 0 parameter tol, 1 function tol, 2 gradient tol, 3 max iterations,
                       4 max time, 5 min radius, 6 failure */
  double initial_cost, final_cost;
  double total_time_s;
} vgx_solver_summary;

void vgx_solver_options_default(vgx_solver_options* o);
/* PoseGraph::optimize: Levenberg-Marquardt with Ceres' default trust-region schedule,
 * device resident; optimised poses are written to xyzyaw_out (n x 4, may be NULL) and
 * stay the graph's current poses. */
int vgx_graph_solve(vgx_ctx* ctx, const vgx_solver_options* opts, double* xyzyaw_out,
                    vgx_solver_summary* summary);

/* PoseGraph::getEdgeCovarianceMap (pose_graph.cpp:117-163): the 4 x 4 covariance blocks
 * Cov(x_a, x_b) (row-major, rows = parameters of a) that ceres::Covariance reports for the requested
 * submap pairs: blocks of (J^T J)^-1 over the free nodes at the current poses; zero for a constant
 * node.  Fails (VGX_ERR_INVALID) where Covariance::Compute returns false (rank-deficient J). */
int vgx_graph_edge_covariances(vgx_ctx* ctx, int m, const uint32_t* ids_a, const uint32_t* ids_b,
                               double* covariances /* m x 16 */);

/* ------------------------------------------------------------------ map evaluation */
/* voxblox::io::LoadLayer<TsdfVoxel> from a byte buffer: a varint32 message count (utils::
 * writeProtoMsgCountToStream), one LayerProto {1 voxel_size: double, 2 voxels_per_side, 3 type: string},
 * then count - 1 BlockProto messages (the collection files' block messages).  The format is restated from
 * the published voxblox sources and has not been checked against a file voxblox wrote.  Rules: type must be
 * "tsdf"; every block's voxels_per_side and voxel_size equal the header's; a repeated block index is an error
 * (BlockMergingStrategy::kProhibit); the stream ends right after the last block; colour is dropped.
 * Creates submap_id as a finished upload (the state vgx_collection_load leaves).  submap_id must not exist.
 * Any deviation gives VGX_ERR_INVALID and leaves no submap behind. */
int vgx_layer_load(vgx_ctx* ctx, uint32_t submap_id, const uint8_t* bytes, uint64_t n, int* n_blocks);

/* VoxgraphSubmap::transformSubmap's layer part (voxgraph_submap.cpp:38-58): voxblox transformLayer(old copy,
 * T_new_old, &own layer), i.e. written into the submap's own, uncleared layer.  Restated rule:
 *   - candidate output blocks are enumerated as vgx_project_map does (8 sample points per old block);
 *   - every voxel centre of a candidate block is moved by T_new_old.inverse() and interpolated trilinearly
 *     in the old copy (all 8 neighbours observed); on success the voxel takes the interpolated (d, w), on a
 *     failure it keeps its old value where the block already existed and is (0, 0) otherwise;
 *   - output blocks: every old block (none is removed; bricks carry no has_data flag, so every old block
 *     counts as holding data) plus every candidate block with at least one success, in ascending packed key
 *     order; no merge, no (d w) / w rounding.
 * The identity transform therefore changes no bit of a layer whose distances are finite and carry no -0.0
 * (0 * NaN is NaN, so a NaN spreads to the neighbours interpolated over it, and -0.0 + 0.0 is +0.0), and the
 * result differs from vgx_project_map with n = 1, which
 * merges.  T_new_old: [qw qx qy qz tx ty tz].  The submap (active or finished) becomes a finished upload:
 * its ESDF and registration points are dropped; run vgx_submap_generate_esdf / vgx_submap_extract_points
 * again.  A candidate block index outside [VGX_BLOCK_INDEX_MIN, VGX_BLOCK_INDEX_MAX] gives VGX_ERR_INVALID
 * and leaves the submap unchanged.  Profiling: the kernels count in slot 13 (the shared projection passes)
 * and slot 14 (the transform's own resampling kernel). */
int vgx_submap_transform(vgx_ctx* ctx, uint32_t submap_id, const float T_new_old[7]);

/* voxblox utils::VoxelEvaluationDetails */
typedef struct vgx_voxel_evaluation_details {
  float rmse;
  float max_error;
  float min_error;
  float pad;
  uint64_t num_evaluated_voxels;
  uint64_t num_ignored_voxels;
  uint64_t num_overlapping_voxels;
  uint64_t num_non_overlapping_voxels;
} vgx_voxel_evaluation_details;
#define VGX_LAYER_TSDF 0   /* the resident (distance, weight) bricks; observed <=> weight > 1e-6 */
#define VGX_LAYER_ESDF 1   /* the ESDF bricks of vgx_submap_generate_esdf; observed <=> the observed flag */
/* voxblox utils::evaluateLayersRmse with VoxelEvaluationMode::kIgnoreErrorBehindTestSurface (the only mode
 * ported).  Restated rule:
 *   - a test block missing from the ground truth: every observed test voxel is non-overlapping;
 *   - a shared block, per voxel in this order: either side unobserved (both included) -> non-overlapping;
 *     d_test < 0.0 -> ignored and overlapping; otherwise evaluated and overlapping with e = d_test - d_gt in
 *     float, fl32(e * e) added to a double sum, max_error = std::max(max_error, |e|) (a NaN never replaces
 *     it); min_error starts at 0 and keeps std::min(min_error, |e|), so it is always 0;
 *   - a ground-truth block missing from the test layer: every observed ground-truth voxel is non-overlapping;
 *   - rmse = (float)sqrt(sum / num_evaluated): NaN when nothing was evaluated.
 * Both layers need the same voxel size and voxels_per_side (VGX_ERR_INVALID), and an ESDF selector a
 * generated ESDF (VGX_ERR_INVALID).  No float atomics: per-block partials are added in block order, so two
 * calls are bit-identical; the double sum is not the sequential one (it lies within n 2^-53 of the exact
 * sum of the terms).  Profiling slot 14. */
int vgx_evaluate_layers_rmse(vgx_ctx* ctx, uint32_t gt_id, int gt_layer, uint32_t test_id, int test_layer,
                             vgx_voxel_evaluation_details* out);

typedef struct vgx_map_evaluation {
  vgx_voxel_evaluation_details details;
  double aligned_pose[4];               /* [x y z yaw] of the ground truth after the alignment */
  float T_projected_map__ground_truth[7];   /* exp([x y z 0 0 yaw]) in float, applied to the ground truth */
  float T_ground_truth__reading[7];     /* its inverse, as MapEvaluation::EvaluationDetails reports it */
  vgx_solver_summary summary;           /* the alignment; termination 6 when the solve failed */
} vgx_map_evaluation;
/* MapEvaluation::evaluate (voxgraph src/tools/evaluation/map_evaluation.cpp:59-161), with the reference's
 * fixed settings:
 *   1. vgx_project_map of the n submaps at T_M_S (n x 7) into an id the context does not use;
 *   2. the projected map: vgx_submap_generate_esdf (defaults) and VGX_POINTS_VOXELS with the reference's
 *      registration filter (min_voxel_weight 1, max_voxel_distance 0.3, use_esdf_distance 1);
 *   3. the ground truth gt_id: vgx_submap_finish and vgx_submap_generate_esdf (defaults);
 *   4. alignment on a private pose graph: node B = projected map (constant, 0), node A = ground truth (free,
 *      0), one residual block reference = projected, reading = ground truth {kVoxels, no_correspondence_cost
 *      0, sampling -1, use_esdf_distance 1}; solver defaults except max_num_iterations 200,
 *      parameter_tolerance 1e-12 and max_solver_time_s 1e9;
 *   5. vgx_submap_transform(gt_id, T) with T = exp([x y z 0 0 yaw]) (minkindr: translation as given,
 *      rotation quaternion of the yaw), in float, then its ESDF again;
 *   6. vgx_evaluate_layers_rmse(gt ESDF, projected ESDF);
 *   7. the projected map is freed.
 * A failed solve (e.g. no relevant voxels in the projected map) leaves the pose at 0 and still reports the
 * evaluation, as the reference does; summary.termination says so.  Only gt_id changes: it ends transformed
 * and finished with an ESDF, so a second call starts from the moved ground truth, as in the reference.  The
 * context's own pose graph keeps its nodes, poses, edges and constraints (its tables are rebuilt on next
 * use).  Errors: an unknown id VGX_ERR_NOT_FOUND; gt_id among submap_ids, a voxel size or voxels_per_side
 * that differs between the ground truth and the submaps, or any vgx_project_map refusal VGX_ERR_INVALID.
 * On any refusal (VGX_ERR_NOT_FOUND, VGX_ERR_INVALID, including a transform refused for its index range) the
 * ground truth's voxels are unchanged; on every error no temporary submap is left.  A CUDA or capacity error
 * after step 3 can leave the ground truth finished with a new ESDF, and one after step 5 transformed. */
int vgx_map_evaluate(vgx_ctx* ctx, uint32_t gt_id, int n, const uint32_t* submap_ids,
                     const float* T_M_S /* n x 7 */, vgx_map_evaluation* out);

/* ------------------------------------------------------------------ multi-GPU */
/* One process per GPU. Registration constraints are sharded over the ranks of the
 * communicator (every rank passes the same full list and holds the submaps it needs);
 * the per-node / per-edge normal-equation blocks are summed with one ncclAllReduce per
 * evaluation. */
/* Host-only: the constraint -> rank partition the library uses. Constraints are ordered by
 * locality key (the reading submap id; NULL = input order; ties keep input order) and that
 * sequence is cut into nranks contiguous pieces of equal residual count, so a rank gathers from
 * few reading submaps (L2 locality) and loads differ by at most one constraint.
 * owner[i] in [0, nranks). */
int vgx_shard_constraints(int nranks, int n, const int32_t* num_residuals,
                          const uint32_t* locality_keys, int32_t* owner);
int vgx_comm_unique_id(uint8_t id[128]);
int vgx_comm_init(vgx_ctx* ctx, int nranks, int rank, const uint8_t id[128]);
int vgx_comm_destroy(vgx_ctx* ctx);
/* NVLink peer-memory exchange (single node, <= 8 ranks): replaces the NCCL all-reduce of the
 * packed normal equations by a one-shot all-gather-reduce over CUDA-IPC mapped peer buffers:
 * the assembly kernel PUSHES every element of the rank's partial, tagged with the evaluation's
 * epoch (one 16-byte store {lo32, tag, hi32, tag}), into its slot of every peer's exported
 * region while it is produced; each rank then spins on the tagged elements of its own region and
 * sums the partials in rank order (no load crosses NVLink, no fence or flag; bit-identical on all
 * ranks).  export: allocate 2 parities x 8 ranks x capacity_doubles x 16 bytes + get the 64-byte
 * IPC handle; import: map the peers (handles = nranks x 64 bytes, own entry ignored). Works with
 * or without vgx_comm_init; when both are set the peer path is used. */
/* Self-check of the sharded evaluation: while suspended (on = 1) the context behaves as a
 * single-rank context - it evaluates EVERY constraint locally and skips the exchange - so a rank
 * can compare the all-reduced result with the full problem computed on one GPU (all submaps are
 * replicated anyway).  Local to the calling rank; on = 0 restores the rank layout. */
int vgx_comm_suspend(vgx_ctx* ctx, int on);
int vgx_comm_p2p_export(vgx_ctx* ctx, uint64_t capacity_doubles, uint8_t handle[64]);
int vgx_comm_p2p_import(vgx_ctx* ctx, int nranks, int rank, const uint8_t* handles);

#ifdef __cplusplus
}
#endif
#endif /* VOXGRAPH_B200_H_ */
