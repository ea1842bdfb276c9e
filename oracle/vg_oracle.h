/*
 * vg_oracle.h — CPU ORACLE for the voxgraph hot paths.  TEST INFRASTRUCTURE ONLY.
 *
 * This is a plain-C restatement of the reference algorithm used as the checker for
 * the CUDA product path.  Nothing under voxgraph_b200/ may include, link or call it;
 * only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs do.
 *
 * PARITY UNPINNED: the reference (ethz-asl/voxgraph @ bd802b5) ships no tests, golden
 * vectors or fixtures, and its arithmetic dependencies (voxblox, cblox, minkindr,
 * Ceres, Eigen) are neither vendored nor installed, so neither the reference nor its
 * dependencies can be compiled here.  The restatement follows the reference sources
 * line by line where they exist in the reference, ethz-asl/voxgraph (cited per function below) and
 * the published upstream algorithms (SURVEY.md Appendix A) elsewhere; it is pinned
 * by analytic known-answer tests (tests/test_oracle_*.py) and by golden vectors
 * generated from the reference's own sympy derivation
 * (voxgraph/scripts/jacobians_xyz_yaw.py -> tests/golden/).
 *
 * Paths are relative to voxgraph/ of the reference.
 */
#ifndef VG_ORACLE_H_
#define VG_ORACLE_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------- */
/* Layer = voxblox::Layer<Voxel> + Block<Voxel> + AnyIndexHash (Appendix A.2) */
/* A voxel carries (distance, weight); observed <=> weight > 1e-6.            */
/* For an ESDF layer upload weight = observed ? 1 : 0.                        */
/* ------------------------------------------------------------------------- */
typedef struct vgo_layer vgo_layer;

vgo_layer* vgo_layer_create(float voxel_size, int voxels_per_side);
void vgo_layer_destroy(vgo_layer* layer);
/* Adds (or overwrites) a block. distance/weight may be NULL (zero-filled).
 * Returns the block slot. */
int vgo_layer_add_block(vgo_layer* layer, const int32_t idx[3], const float* distance,
                        const float* weight);
int vgo_layer_num_blocks(const vgo_layer* layer);
int vgo_layer_find_block(const vgo_layer* layer, const int32_t idx[3]);
/* Copies all blocks out in slot (= allocation) order. */
void vgo_layer_export(const vgo_layer* layer, int32_t* idx, float* distance, float* weight);
float vgo_layer_voxel_size_inv(const vgo_layer* layer);
float vgo_layer_block_size_inv(const vgo_layer* layer);

/* ------------------------------------------------------------------------- */
/* Index math (voxblox/core/common.h, Appendix A.2)                           */
/* ------------------------------------------------------------------------- */
/* floor(p * inv + 1e-6) per axis, float arithmetic. */
void vgo_grid_index_from_point(const float p[3], float grid_size_inv, int32_t out[3]);
/* global voxel index -> (block index, local voxel index), upstream float/bitmask forms */
void vgo_block_and_local_from_global(const int64_t g[3], int vps, int32_t block[3],
                                     int32_t local[3]);

/* ------------------------------------------------------------------------- */
/* Interpolator<V>::getVoxelsAndQVector (voxblox interpolator_inl.h, A.3)     */
/* ------------------------------------------------------------------------- */
/* Returns 1 when all 8 neighbours exist and are observed. On success (and on
 * failure as far as computed) fills: base block index, the 8 (slot, linear
 * voxel index) pairs, the 8 distances and the q vector. */
int vgo_interp_voxels_and_q(const vgo_layer* layer, const float pos[3], int32_t base_block[3],
                            int32_t base_voxel[3], int32_t slots[8], int32_t linear[8],
                            float distances[8], float q[8]);

/* ------------------------------------------------------------------------- */
/* minkindr QuatTransformationTemplate<float> (Appendix A.1)                  */
/* T = [qw qx qy qz tx ty tz]                                                 */
/* ------------------------------------------------------------------------- */
void vgo_T_exp(const float v6[6], float T[7]);
void vgo_T_inverse(const float T[7], float out[7]);
void vgo_T_compose(const float A[7], const float B[7], float out[7]);
void vgo_T_transform(const float T[7], const float p[3], float out[3]);

/* ------------------------------------------------------------------------- */
/* RegistrationCostFunction::Evaluate                                         */
/* src/backend/constraint/cost_functions/registration_cost_function.cpp:58-298 */
/* ------------------------------------------------------------------------- */
/* points: n x {x,y,z}, distance[n], weight[n] (RegistrationPoint AoS split in 3 arrays).
 * residuals: n doubles. jac_ref/jac_read: n x 4 row-major doubles, each may be NULL.
 * Returns 1 (true) or 0 (false: summed weight == 0, cpp:273). Deterministic mode
 * (sampling_ratio == -1) only. */
int vgo_reg_evaluate(const vgo_layer* reading_layer, int n, const float* xyz,
                     const float* distance, const float* weight, double no_correspondence_cost,
                     const double ref_pose[4], const double read_pose[4], double* residuals,
                     double* jac_ref, double* jac_read);

/* The float pose-setup block of Evaluate (cpp:61-110): fills
 * T_reading_reference [7] and {cos_e, sin_e, cos_emo, sin_emo, xe, ye, xo, yo}. */
void vgo_reg_pose_setup(const double ref_pose[4], const double read_pose[4], float T_rr[7],
                        float trig[8]);

/* ------------------------------------------------------------------------- */
/* RelativePoseCostFunction::operator()                                       */
/* include/voxgraph/backend/constraint/cost_functions/relative_pose_cost_function_inl.h:8-70 */
/* Jacobians are the analytic derivatives autodiff would produce.             */
/* ------------------------------------------------------------------------- */
void vgo_relpose_evaluate(const double pose_a[4], const double pose_b[4], const double t_obs[3],
                          double yaw_obs, const double sqrt_info[16], double r[4],
                          double jac_a[16], double jac_b[16]);
/* Constraint ctor (src/backend/constraint/constraint.cpp:4-38): LLT lower factor.
 * Returns 0 ok, -1 not positive definite. */
int vgo_sqrt_information(const double info[16], double sqrt_info[16]);
/* Constraint ctor, allow_semi_definite_information_matrix branch (constraint.cpp:15-37):
 * Eigen LDLT with diagonal pivoting; sqrt_information = P^T L sqrt(D) P.
 * Returns 0 ok, -1 if the matrix is not positive semi-definite. */
int vgo_sqrt_information_ldlt(const double info[16], double sqrt_info[16]);
/* NormalizeAngle (include/voxgraph/backend/local_parameterization/normalize_angle.h:11-16) */
double vgo_normalize_angle(double a);

/* ------------------------------------------------------------------------- */
/* Pose graph + Ceres-default Levenberg-Marquardt (pose_graph.cpp:85-106, A.6) */
/* ------------------------------------------------------------------------- */
typedef struct vgo_graph vgo_graph;

typedef struct vgo_solver_options {
  int max_num_iterations;        /* Ceres default 50 */
  double parameter_tolerance;    /* pose_graph.cpp:93 -> 3e-3 (Ceres default 1e-8) */
  double function_tolerance;     /* 1e-6 */
  double gradient_tolerance;     /* 1e-10 */
  double initial_trust_region_radius; /* 1e4 */
  double max_trust_region_radius;     /* 1e16 */
  double min_trust_region_radius;     /* 1e-32 */
  double min_relative_decrease;       /* 1e-3 */
  double min_lm_diagonal;             /* 1e-6 */
  double max_lm_diagonal;             /* 1e32 */
  double max_solver_time_s;           /* pose_graph.cpp:95 -> 4 */
  int jacobi_scaling;                 /* 1 */
  int num_threads;                    /* pose_graph.cpp:96 -> 4 */
  int exclude_registration;           /* PoseGraph::optimize(bool) */
} vgo_solver_options;

typedef struct vgo_solver_summary {
  int iterations;            /* LM iterations performed (incl. unsuccessful) */
  int num_successful_steps;
  int num_residual_evals;    /* full-problem evaluations */
  int termination;           /* 0 parameter tol, 1 function tol, 2 gradient tol,
                                3 max iterations, 4 max time, 5 min radius, 6 failure */
  double initial_cost, final_cost;
  double total_time_s;
  double eval_time_s;        /* time inside residual/Jacobian evaluation */
  double linear_solver_time_s;
} vgo_solver_summary;

void vgo_solver_options_default(vgo_solver_options* o);

vgo_graph* vgo_graph_create(void);
void vgo_graph_destroy(vgo_graph* g);
/* addSubmapNode (pose_graph.cpp:12-14). Returns node index. */
int vgo_graph_add_node(vgo_graph* g, uint32_t id, const double xyzyaw[4], int constant);
/* addRelativePoseConstraint (pose_graph.cpp:41-46). sqrt_info row-major 4x4. */
int vgo_graph_add_relative(vgo_graph* g, uint32_t id_a, uint32_t id_b, const double t_obs[3],
                           double yaw_obs, const double sqrt_info[16]);
/* One registration residual block: reference points (not copied; caller keeps them
 * alive) registered against reading layer. PoseGraph::addRegistrationConstraint's
 * mirroring (pose_graph.cpp:63-71) is done by the caller. */
int vgo_graph_add_registration(vgo_graph* g, uint32_t ref_id, uint32_t read_id,
                               const vgo_layer* reading_layer, int n, const float* xyz,
                               const float* distance, const float* weight,
                               double no_correspondence_cost);
void vgo_graph_reset_registration(vgo_graph* g);
int vgo_graph_num_nodes(const vgo_graph* g);
int vgo_graph_num_registration_residuals(const vgo_graph* g);
void vgo_graph_get_poses(const vgo_graph* g, double* xyzyaw);
void vgo_graph_set_poses(vgo_graph* g, const double* xyzyaw);

/* Evaluates the whole problem at the current poses the way Ceres would:
 * cost = 1/2 sum r^2, gradient g = J^T r (4 per node, node order), H = J^T J
 * dense (4N x 4N row-major). Constant nodes are included in the layout (their
 * rows/cols are simply what the Jacobians give); any output may be NULL.
 * Returns 1 ok, 0 if some registration Evaluate returned false. */
int vgo_graph_eval(vgo_graph* g, int num_threads, int exclude_registration, double* cost,
                   double* gradient, double* H);
/* Per-registration-constraint summed squared residual (pose_graph.cpp:194-207). */
void vgo_graph_registration_costs(vgo_graph* g, double* per_constraint_sq_sum);

int vgo_graph_solve(vgo_graph* g, const vgo_solver_options* opts, vgo_solver_summary* summary);

/* ------------------------------------------------------------------------- */
/* "Next" rows of SURVEY §8f, restated ahead of their GPU versions            */
/* (src/frontend/submap_collection/voxgraph_submap.cpp, bounding_box.cpp)    */
/* ------------------------------------------------------------------------- */
/* VoxgraphSubmap::findRelevantVoxelIndices (voxgraph_submap.cpp:144-201), TSDF-distance branch:
 * every voxel with weight > min_voxel_weight and |distance| < max_voxel_distance becomes a
 * RegistrationPoint {voxel centre, distance, weight}, blocks in allocation order, voxels in
 * linear order. Writes at most max_n entries, returns the total count. */
int vgo_find_relevant_voxels(const vgo_layer* layer, double min_voxel_weight,
                             double max_voxel_distance, float* xyz, float* distance,
                             float* weight, int max_n);
/* VoxgraphSubmap::findIsosurfaceVertices (voxgraph_submap.cpp:203-243):
 *   MeshIntegrator(min_weight = min_voxel_weight, use_color = false).generateMesh  (upstream voxblox
 *   mesh_integrator.h / marching_cubes.h, restated from the published algorithm: every voxel is the
 *   origin of a cube over its 2x2x2 forward neighbourhood - corner order (0,0,0),(1,0,0),(1,1,0),
 *   (0,1,0),(0,0,1),(1,0,1),(1,1,1),(0,1,1) - meshed only when all 8 corners have weight >
 *   min_weight; a vertex is interpolated on every cube edge whose end points differ in sign (sdf < 0):
 *   v1 + sdf1 / (sdf1 - sdf2) * (v2 - v1), or the mid point when |sdf1 - sdf2| < 1e-6),
 *   MeshLayer::getConnectedMesh(0.5 * voxel_size) (vertices are bucketed by
 *   round(vertex / threshold) in double; the first vertex of a bucket is kept),
 *   Interpolator::getVoxel(vertex, interpolate = true) -> trilinear (distance, weight); vertices whose
 *   8 neighbours are not all observed are dropped.
 * The marching-cubes triangle table only decides how often and in which order an edge vertex is
 * emitted, not which vertices exist; the order decides which member of a bucket survives.  The
 * reference walks blocks in hash-map order; this restatement (and the GPU path) fixes the order
 * canonically: blocks in allocation order, voxels in linear order, cube edges 0..11.
 * Writes at most max_n points / max_blocks isosurface block indices (cpp:237-240), returns the
 * vertex count, *n_blocks the number of distinct isosurface blocks (first-occurrence order). */
int vgo_find_isosurface_vertices(const vgo_layer* layer, double min_voxel_weight, float* xyz,
                                 float* distance, float* weight, int max_n, int32_t* iso_blocks,
                                 int max_blocks, int* n_blocks);
/* Interpolator::getVoxel(pos, &voxel, true): trilinear distance and weight; 0 when impossible. */
int vgo_interp_voxel(const vgo_layer* layer, const float pos[3], float* distance, float* weight);

/* cblox::TsdfEsdfSubmap::generateEsdf (finishSubmap, voxgraph_submap.cpp:86) =
 * voxblox::EsdfIntegrator::updateFromTsdfLayerBatch, restated from the published algorithm as its
 * fixed point (parity unpinned; upstream is absent):
 *   a TSDF voxel with weight >= min_weight is observed; |tsdf| < min_distance_m -> fixed, ESDF
 *   distance = TSDF distance; otherwise the distance starts at sign(tsdf) * default_distance_m and
 *   is lowered (raised on the negative side) through the 26-neighbourhood,
 *   d(n) <- d(v) + |offset| * voxel_size for same-sign observed non-fixed neighbours while it stays
 *   below max_distance_m (quasi-Euclidean, full_euclidean_distance = false).
 * voxblox pops a bucketed priority queue once; this restatement (and the GPU path) relaxes to
 * convergence, i.e. the exact shortest quasi-Euclidean path in float arithmetic, which is
 * independent of the processing order.  Output per voxel of the layer's blocks (slot order):
 * distance and observed (1 / 0). */
typedef struct vgo_esdf_config {
  float max_distance_m;      /* 2.0 */
  float default_distance_m;  /* 2.0 */
  float min_distance_m;      /* 0.2 */
  float min_weight;          /* 1e-6 */
} vgo_esdf_config;
void vgo_esdf_config_default(vgo_esdf_config* c);
/* returns the number of relaxation sweeps */
int vgo_generate_esdf(const vgo_layer* tsdf, const vgo_esdf_config* cfg, float* distance, float* observed);

/* VoxgraphSubmap::getSubmapFrameSurfaceObb (voxgraph_submap.cpp:280-324). Returns 0 when no
 * voxel qualifies (box stays +-inf). */
int vgo_surface_obb(const vgo_layer* layer, double min_voxel_weight, double max_voxel_distance,
                    float obb_min[3], float obb_max[3]);
/* BoundingBox::getAabbFromObbAndPose (bounding_box.cpp:28-42); pose = [qw qx qy qz tx ty tz]. */
void vgo_aabb_from_obb_and_pose(const float obb_min[3], const float obb_max[3], const float pose[7],
                                float aabb_min[3], float aabb_max[3]);
/* VoxgraphSubmap::overlapsWith (voxgraph_submap.cpp:245-278): mission-frame surface AABB
 * rejection, then "any isosurface block centre of the current submap lands in an allocated block
 * of the other". isosurface_blocks: n x 3 block indices of the current submap. */
int vgo_submaps_overlap(const float aabb_min[3], const float aabb_max[3],
                        const float other_aabb_min[3], const float other_aabb_max[3],
                        const float pose_current[7], const float pose_other[7],
                        const int32_t* isosurface_blocks, int n, float block_size_current,
                        const vgo_layer* other_layer);

/* ------------------------------------------------------------------------- */
/* WeightedSampler<RegistrationPoint>::getRandomItem                          */
/* (include/voxgraph/frontend/submap_collection/weighted_sampler_inl.h:19-28, */
/*  weighted_sampler.h:34-36): std::mt19937 (default seed 5489) through        */
/*  std::uniform_real_distribution<double>(0, 1) = generate_canonical<double,  */
/*  53> = two 32-bit draws, then upper_bound over the cumulative weights.      */
/* ------------------------------------------------------------------------- */
typedef struct vgo_sampler {
  uint32_t mt[624];
  int idx;
} vgo_sampler;
void vgo_sampler_init(vgo_sampler* s);                 /* default-constructed std::mt19937 */
uint32_t vgo_sampler_next_u32(vgo_sampler* s);         /* std::mt19937::operator() */
double vgo_sampler_canonical(vgo_sampler* s);          /* uniform_real_distribution<double>(0,1)(gen) */
/* cumulative = WeightedSampler::cumulative_item_weights_ (double prefix sums of the float
 * weights, addItem inl.h:6-17); writes `count` drawn indices. */
void vgo_sampler_draw(vgo_sampler* s, const double* cumulative, int n, int count, int32_t* idx);

/* ------------------------------------------------------------------------- */
/* TSDF integration (voxblox tsdf_integrator.cc / integrator_utils, A.4)      */
/* ------------------------------------------------------------------------- */
typedef struct vgo_tsdf_config {
  float default_truncation_distance; /* voxgraph_mapper.yaml:23 -> 0.6 */
  float max_weight;                  /* 10000 */
  int voxel_carving_enabled;         /* 1 */
  float min_ray_length_m;            /* 0.1 */
  float max_ray_length_m;            /* yaml:24 -> 16 */
  int use_const_weight;              /* yaml:25 -> 1 */
  int allow_clear;                   /* 1 */
  int use_weight_dropoff;            /* yaml:26 -> 1 */
  int use_sparsity_compensation_factor; /* yaml:27 -> 1 */
  float sparsity_compensation_factor;   /* yaml:28 -> 20 */
  /* FastTsdfIntegrator only */
  float start_voxel_subsampling_factor; /* 2 */
  int max_consecutive_ray_collisions;   /* 2 */
  int mode;                             /* 0 = simple (every ray, every voxel), 1 = fast */
} vgo_tsdf_config;

typedef struct vgo_tsdf_stats {
  int64_t rays_valid;      /* rays that passed isPointValid */
  int64_t rays_cast;       /* rays actually cast (fast mode skips some) */
  int64_t voxel_updates;   /* updateTsdfVoxel calls */
  int64_t blocks_allocated;
} vgo_tsdf_stats;

void vgo_tsdf_config_default(vgo_tsdf_config* c);
/* T_G_C = [qw qx qy qz tx ty tz]. Single-threaded, points in order. */
void vgo_tsdf_integrate(vgo_layer* layer, const vgo_tsdf_config* cfg, const float T_G_C[7],
                        int n, const float* points_C, vgo_tsdf_stats* stats);
/* Multi-threaded form, as voxblox runs its integrators (integrator_threads = hardware_concurrency;
 * points dealt to the threads round robin, per-voxel locks, block allocation under a mutex,
 * ApproxHashSet = atomic exchange).  Order dependent like the reference's; used as the CPU baseline
 * of the TSDF timing leg, the single-threaded form above stays the parity checker. */
void vgo_tsdf_integrate_mt(vgo_layer* layer, const vgo_tsdf_config* cfg, const float T_G_C[7],
                           int n, const float* points_C, int num_threads, vgo_tsdf_stats* stats);
/* RayCaster restatement: writes up to max_out global voxel indices (int64 x 3);
 * returns the number the caster emits. cast_from_origin=1 -> start->end. */
int vgo_raycast(const float origin[3], const float point_G[3], int is_clearing,
                int voxel_carving, float max_ray_length_m, float voxel_size_inv,
                float truncation_distance, int cast_from_origin, int64_t* out, int max_out);

#ifdef __cplusplus
}
#endif
#endif /* VG_ORACLE_H_ */
