/*
 * vg_oracle.c — CPU ORACLE (test infrastructure; see vg_oracle.h header comment).
 * PARITY UNPINNED against the real reference binaries (they cannot be built here);
 * pinned by known-answer tests and sympy-derived golden vectors.
 *
 * Build with -ffp-contract=off: the reference float expressions are restated
 * operation by operation and must not be fused.
 */
#include "vg_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <pthread.h>
#include <sched.h>
#include <stdatomic.h>
#include <stdint.h>

#define VGO_COORD_EPS 1e-6f  /* voxblox kCoordinateEpsilon */
#define VGO_FLOAT_EPS 1e-6f  /* voxblox kFloatEpsilon / kEpsilon */

static double now_s(void) {
  struct timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}

/* ========================================================================= */
/* Layer                                                                     */
/* ========================================================================= */
struct vgo_layer {
  float voxel_size, voxel_size_inv, block_size, block_size_inv;
  int vps, vox_per_block;
  float vps_inv;
  int n_blocks, cap_blocks;
  int32_t* idx;     /* n x 3 */
  float* distance;  /* n x vps^3 */
  float* weight;    /* n x vps^3 */
  int32_t* table;   /* open addressing, slot or -1 */
  uint32_t table_size; /* power of two */
  int mt_zeroed_from, mt_zeroed_to; /* spare bricks [from, to) zeroed for the multi-threaded integrator */
};

/* voxblox AnyIndexHash: x + y*17191 + z*17191^2 (block_hash.h) */
static inline uint64_t any_index_hash(int64_t x, int64_t y, int64_t z) {
  const uint64_t sl = 17191u, sl2 = 17191u * 17191u;
  return (uint64_t)x + (uint64_t)y * sl + (uint64_t)z * sl2;
}

vgo_layer* vgo_layer_create(float voxel_size, int vps) {
  vgo_layer* l = (vgo_layer*)calloc(1, sizeof(vgo_layer));
  l->voxel_size = voxel_size;
  /* Layer ctor: voxel_size_inv_ = 1.0 / voxel_size_; block_size_ = voxel_size_ * vps;
   * block_size_inv_ = 1.0 / block_size_ (double division, stored as float) */
  l->voxel_size_inv = (float)(1.0 / (double)voxel_size);
  l->block_size = voxel_size * (float)vps;
  l->block_size_inv = (float)(1.0 / (double)l->block_size);
  l->vps = vps;
  l->vps_inv = (float)(1.0 / (double)vps);
  l->vox_per_block = vps * vps * vps;
  l->table_size = 1024;
  l->table = (int32_t*)malloc(sizeof(int32_t) * l->table_size);
  for (uint32_t i = 0; i < l->table_size; ++i) l->table[i] = -1;
  return l;
}

void vgo_layer_destroy(vgo_layer* l) {
  if (!l) return;
  free(l->idx); free(l->distance); free(l->weight); free(l->table); free(l);
}

static void layer_table_insert(vgo_layer* l, int slot) {
  const int32_t* k = l->idx + 3 * slot;
  uint32_t h = (uint32_t)(any_index_hash(k[0], k[1], k[2]) & (l->table_size - 1));
  while (l->table[h] >= 0) h = (h + 1) & (l->table_size - 1);
  l->table[h] = slot;
}

int vgo_layer_find_block(const vgo_layer* l, const int32_t k[3]) {
  uint32_t h = (uint32_t)(any_index_hash(k[0], k[1], k[2]) & (l->table_size - 1));
  for (;;) {
    int s = l->table[h];
    if (s < 0) return -1;
    const int32_t* q = l->idx + 3 * s;
    if (q[0] == k[0] && q[1] == k[1] && q[2] == k[2]) return s;
    h = (h + 1) & (l->table_size - 1);
  }
}

int vgo_layer_add_block(vgo_layer* l, const int32_t k[3], const float* distance,
                        const float* weight) {
  int s = vgo_layer_find_block(l, k);
  if (s < 0) {
    if (l->n_blocks == l->cap_blocks) {
      int nc = l->cap_blocks ? 2 * l->cap_blocks : 64;
      l->idx = (int32_t*)realloc(l->idx, sizeof(int32_t) * 3 * (size_t)nc);
      l->distance = (float*)realloc(l->distance, sizeof(float) * (size_t)l->vox_per_block * nc);
      l->weight = (float*)realloc(l->weight, sizeof(float) * (size_t)l->vox_per_block * nc);
      l->cap_blocks = nc;
    }
    s = l->n_blocks++;
    l->idx[3 * s + 0] = k[0]; l->idx[3 * s + 1] = k[1]; l->idx[3 * s + 2] = k[2];
    if ((uint32_t)l->n_blocks * 2 > l->table_size) {
      l->table_size *= 2;
      l->table = (int32_t*)realloc(l->table, sizeof(int32_t) * l->table_size);
      for (uint32_t i = 0; i < l->table_size; ++i) l->table[i] = -1;
      for (int i = 0; i < l->n_blocks - 1; ++i) layer_table_insert(l, i);
    }
    layer_table_insert(l, s);
  }
  float* d = l->distance + (size_t)s * l->vox_per_block;
  float* w = l->weight + (size_t)s * l->vox_per_block;
  if (distance) memcpy(d, distance, sizeof(float) * l->vox_per_block);
  else memset(d, 0, sizeof(float) * l->vox_per_block);
  if (weight) memcpy(w, weight, sizeof(float) * l->vox_per_block);
  else memset(w, 0, sizeof(float) * l->vox_per_block);
  return s;
}

int vgo_layer_num_blocks(const vgo_layer* l) { return l->n_blocks; }
float vgo_layer_voxel_size_inv(const vgo_layer* l) { return l->voxel_size_inv; }
float vgo_layer_block_size_inv(const vgo_layer* l) { return l->block_size_inv; }

void vgo_layer_export(const vgo_layer* l, int32_t* idx, float* distance, float* weight) {
  if (idx) memcpy(idx, l->idx, sizeof(int32_t) * 3 * (size_t)l->n_blocks);
  if (distance)
    memcpy(distance, l->distance, sizeof(float) * (size_t)l->vox_per_block * l->n_blocks);
  if (weight) memcpy(weight, l->weight, sizeof(float) * (size_t)l->vox_per_block * l->n_blocks);
}

/* ========================================================================= */
/* Index math                                                                */
/* ========================================================================= */
/* getGridIndexFromPoint(point, grid_size_inv): floor(p * inv + eps)  (common.h) */
void vgo_grid_index_from_point(const float p[3], float inv, int32_t out[3]) {
  out[0] = (int32_t)floorf(p[0] * inv + VGO_COORD_EPS);
  out[1] = (int32_t)floorf(p[1] * inv + VGO_COORD_EPS);
  out[2] = (int32_t)floorf(p[2] * inv + VGO_COORD_EPS);
}

/* getBlockIndexFromGlobalVoxelIndex: floor(float(g) * vps_inv);
 * getLocalFromGlobalVoxelIndex: (g + 2^31) & (vps - 1)   (common.h) */
void vgo_block_and_local_from_global(const int64_t g[3], int vps, int32_t block[3],
                                     int32_t local[3]) {
  const float vps_inv = (float)(1.0 / (double)vps);
  for (int a = 0; a < 3; ++a) {
    block[a] = (int32_t)floorf((float)g[a] * vps_inv);
    const int64_t offset = (int64_t)1 << 31;
    local[a] = (int32_t)((g[a] + offset) & (int64_t)(vps - 1));
  }
}

/* ========================================================================= */
/* Interpolator (A.3)                                                        */
/* ========================================================================= */
int vgo_interp_voxels_and_q(const vgo_layer* l, const float pos[3], int32_t base_block[3],
                            int32_t base_voxel[3], int32_t slots[8], int32_t linear[8],
                            float distances[8], float q[8]) {
  const int vps = l->vps;
  /* setIndexes: block_index = layer.computeBlockIndexFromCoordinates(pos) */
  int32_t bi[3];
  vgo_grid_index_from_point(pos, l->block_size_inv, bi);
  base_block[0] = bi[0]; base_block[1] = bi[1]; base_block[2] = bi[2];
  if (vgo_layer_find_block(l, bi) < 0) return 0;
  /* block origin = block_index * block_size (getOriginPointFromGridIndex) */
  float origin[3] = {(float)bi[0] * l->block_size, (float)bi[1] * l->block_size,
                     (float)bi[2] * l->block_size};
  /* Block::computeVoxelIndexFromCoordinates: floor((p - origin) * vsi + eps), clamped */
  int32_t vi[3];
  float rel[3] = {pos[0] - origin[0], pos[1] - origin[1], pos[2] - origin[2]};
  vgo_grid_index_from_point(rel, l->voxel_size_inv, vi);
  for (int a = 0; a < 3; ++a) {
    if (vi[a] > vps - 1) vi[a] = vps - 1;
    if (vi[a] < 0) vi[a] = 0;
  }
  /* shift to the bottom-left corner voxel: centre = origin + (vi + 0.5) * voxel_size */
  for (int a = 0; a < 3; ++a) {
    float centre = origin[a] + ((float)vi[a] + 0.5f) * l->voxel_size;
    float off = pos[a] - centre;
    if (off < 0) {
      vi[a]--;
      if (vi[a] < 0) {
        bi[a]--;
        vi[a] += vps;
      }
    }
  }
  base_block[0] = bi[0]; base_block[1] = bi[1]; base_block[2] = bi[2];
  base_voxel[0] = vi[0]; base_voxel[1] = vi[1]; base_voxel[2] = vi[2];
  /* getVoxelsAndQVector(block_index, voxel_indexes, pos, ...) */
  for (int i = 0; i < 8; ++i) {
    /* columns of [0 0 0 0 1 1 1 1; 0 0 1 1 0 0 1 1; 0 1 0 1 0 1 0 1] */
    int32_t v[3] = {vi[0] + ((i >> 2) & 1), vi[1] + ((i >> 1) & 1), vi[2] + (i & 1)};
    int slot = vgo_layer_find_block(l, bi);
    if (slot < 0) return 0;
    if (v[0] >= vps || v[1] >= vps || v[2] >= vps) {
      int32_t nb[3] = {bi[0], bi[1], bi[2]};
      for (int a = 0; a < 3; ++a)
        if (v[a] >= vps) { nb[a]++; v[a] -= vps; }
      slot = vgo_layer_find_block(l, nb);
      if (slot < 0) return 0;
      if (i == 0) { /* cannot happen: corner 0 is always inside the base block */ }
    }
    if (i == 0) {
      /* getQVector(block->computeCoordinatesFromVoxelIndex(v), pos, vsi) */
      float bo[3] = {(float)bi[0] * l->block_size, (float)bi[1] * l->block_size,
                     (float)bi[2] * l->block_size};
      float off[3];
      for (int a = 0; a < 3; ++a) {
        float centre = bo[a] + ((float)v[a] + 0.5f) * l->voxel_size;
        off[a] = (pos[a] - centre) * l->voxel_size_inv;
      }
      q[0] = 1.0f; q[1] = off[0]; q[2] = off[1]; q[3] = off[2];
      q[4] = off[0] * off[1]; q[5] = off[1] * off[2]; q[6] = off[2] * off[0];
      q[7] = off[0] * off[1] * off[2];
    }
    const int lin = v[0] + vps * (v[1] + vps * v[2]);
    slots[i] = slot; linear[i] = lin;
    const size_t o = (size_t)slot * l->vox_per_block + lin;
    distances[i] = l->distance[o];
    /* utils::isObservedVoxel: weight > 1e-6 */
    if (!(l->weight[o] > 1e-6f)) return 0;
  }
  return 1;
}

/* ========================================================================= */
/* minkindr float transformation (A.1)                                       */
/* ========================================================================= */
/* RotationQuaternion::exp (Grassia) — double internals, float result */
static void rot_exp(const float dx[3], float q[4]) {
  float sq = dx[0] * dx[0] + dx[1] * dx[1] + dx[2] * dx[2];
  double theta = (double)sqrtf(sq);
  double na;
  /* isLessThenEpsilons4thRoot(theta): theta < eps^(1/4) */
  if (theta < pow(2.220446049250313e-16, 0.25)) {
    na = 0.5 + (theta * theta) * (1.0 / 48.0);
  } else {
    na = sin(theta * 0.5) / theta;
  }
  double ct = cos(theta * 0.5);
  q[0] = (float)ct;
  q[1] = (float)((double)dx[0] * na);
  q[2] = (float)((double)dx[1] * na);
  q[3] = (float)((double)dx[2] * na);
}

/* Eigen Quaternion::_transformVector: uv = vec x v; uv += uv; v + w*uv + vec x uv */
static void quat_rotate(const float q[4], const float v[3], float out[3]) {
  const float w = q[0], x = q[1], y = q[2], z = q[3];
  float uv[3] = {y * v[2] - z * v[1], z * v[0] - x * v[2], x * v[1] - y * v[0]};
  uv[0] += uv[0]; uv[1] += uv[1]; uv[2] += uv[2];
  float c[3] = {y * uv[2] - z * uv[1], z * uv[0] - x * uv[2], x * uv[1] - y * uv[0]};
  out[0] = (v[0] + w * uv[0]) + c[0];
  out[1] = (v[1] + w * uv[1]) + c[1];
  out[2] = (v[2] + w * uv[2]) + c[2];
}

void vgo_T_exp(const float v6[6], float T[7]) {
  rot_exp(v6 + 3, T);
  T[4] = v6[0]; T[5] = v6[1]; T[6] = v6[2];
}

void vgo_T_inverse(const float T[7], float out[7]) {
  float qi[4] = {T[0], -T[1], -T[2], -T[3]};
  float r[3];
  quat_rotate(qi, T + 4, r);
  out[0] = qi[0]; out[1] = qi[1]; out[2] = qi[2]; out[3] = qi[3];
  out[4] = -r[0]; out[5] = -r[1]; out[6] = -r[2];
}

void vgo_T_compose(const float A[7], const float B[7], float out[7]) {
  const float aw = A[0], ax = A[1], ay = A[2], az = A[3];
  const float bw = B[0], bx = B[1], by = B[2], bz = B[3];
  float q[4];
  q[0] = aw * bw - ax * bx - ay * by - az * bz;
  q[1] = aw * bx + ax * bw + ay * bz - az * by;
  q[2] = aw * by + ay * bw + az * bx - ax * bz;
  q[3] = aw * bz + az * bw + ax * by - ay * bx;
  float r[3];
  quat_rotate(A, B + 4, r);
  out[0] = q[0]; out[1] = q[1]; out[2] = q[2]; out[3] = q[3];
  out[4] = A[4] + r[0]; out[5] = A[5] + r[1]; out[6] = A[6] + r[2];
}

void vgo_T_transform(const float T[7], const float p[3], float out[3]) {
  float r[3];
  quat_rotate(T, p, r);
  out[0] = r[0] + T[4]; out[1] = r[1] + T[5]; out[2] = r[2] + T[6];
}

/* ========================================================================= */
/* RegistrationCostFunction::Evaluate (registration_cost_function.cpp:58-298) */
/* ========================================================================= */
void vgo_reg_pose_setup(const double ref_pose[4], const double read_pose[4], float T_rr[7],
                        float trig[8]) {
  /* cpp:69-88 — doubles cast to float Vector6, exp() */
  float v_ref[6] = {(float)ref_pose[0], (float)ref_pose[1], (float)ref_pose[2], 0.f, 0.f,
                    (float)ref_pose[3]};
  float v_read[6] = {(float)read_pose[0], (float)read_pose[1], (float)read_pose[2], 0.f, 0.f,
                     (float)read_pose[3]};
  float T_ref[7], T_read[7], T_read_inv[7];
  vgo_T_exp(v_ref, T_ref);
  vgo_T_exp(v_read, T_read);
  /* cpp:91-100 — float trig */
  trig[0] = cosf(v_read[5]);
  trig[1] = sinf(v_read[5]);
  trig[2] = cosf(v_read[5] - v_ref[5]);
  trig[3] = sinf(v_read[5] - v_ref[5]);
  trig[4] = v_read[0]; trig[5] = v_read[1]; trig[6] = v_ref[0]; trig[7] = v_ref[1];
  /* cpp:109-110 — T_reading__reference = T_mission__reading.inverse() * T_mission__reference */
  vgo_T_inverse(T_read, T_read_inv);
  vgo_T_compose(T_read_inv, T_ref, T_rr);
}

int vgo_reg_evaluate(const vgo_layer* layer, int n, const float* xyz, const float* distance,
                     const float* weight, double no_correspondence_cost,
                     const double ref_pose[4], const double read_pose[4], double* residuals,
                     double* jac_ref, double* jac_read) {
  float T_rr[7], trig[8];
  vgo_reg_pose_setup(ref_pose, read_pose, T_rr, trig);
  const float cos_e = trig[0], sin_e = trig[1], cos_emo = trig[2], sin_emo = trig[3];
  const float xe = trig[4], ye = trig[5], xo = trig[6], yo = trig[7];
  double summed_reference_weight = 0;

  for (int i = 0; i < n; ++i) {
    const float* p = xyz + 3 * (size_t)i;
    const float w = weight[i];
    summed_reference_weight += (double)w; /* cpp:124 */
    float rc[3];
    vgo_T_transform(T_rr, p, rc); /* cpp:128-129 */
    int32_t bb[3], bv[3], slots[8], lin[8];
    float d[8], q[8];
    int ok = vgo_interp_voxels_and_q(layer, rc, bb, bv, slots, lin, d, q);

    /* a = B1 * distances^T (h:73-81); shared by cpp:159 and cpp:204-205 */
    float a[8];
    if (ok) {
      a[0] = d[0];
      a[1] = -d[0] + d[4];
      a[2] = -d[0] + d[2];
      a[3] = -d[0] + d[1];
      a[4] = d[0] - d[2] - d[4] + d[6];
      a[5] = d[0] - d[1] - d[2] + d[3];
      a[6] = d[0] - d[1] - d[4] + d[5];
      a[7] = -d[0] + d[1] + d[2] - d[3] + d[4] - d[5] - d[6] + d[7];
      /* cpp:158-163 */
      float interp = q[0] * a[0];
      for (int k = 1; k < 8; ++k) interp = interp + q[k] * a[k];
      const double reading_distance = (double)interp;
      residuals[i] = ((double)distance[i] - reading_distance) * (double)w;
    } else {
      residuals[i] = (double)w * no_correspondence_cost; /* cpp:164-166 */
    }

    if (jac_ref || jac_read) {
      float jr[4] = {0, 0, 0, 0}, je[4] = {0, 0, 0, 0};
      if (ok) {
        /* cpp:183-202 — double deltas, float matrix entries */
        const double inv = (double)layer->voxel_size_inv;
        const double Dx = (double)q[1], Dy = (double)q[2], Dz = (double)q[3];
        float pQ[8][3] = {
            {0.f, 0.f, 0.f},
            {(float)inv, 0.f, 0.f},
            {0.f, (float)inv, 0.f},
            {0.f, 0.f, (float)inv},
            {(float)(inv * Dy), (float)(inv * Dx), 0.f},
            {0.f, (float)(inv * Dz), (float)(inv * Dy)},
            {(float)(inv * Dz), 0.f, (float)(inv * Dx)},
            {(float)(inv * Dy * Dz), (float)(inv * Dx * Dz), (float)(inv * Dx * Dy)}};
        /* cpp:204-205 — pInterp_pr = (distances * B1^T) * pQ_pr */
        float g[3];
        for (int c = 0; c < 3; ++c) {
          float s = a[0] * pQ[0][c];
          for (int k = 1; k < 8; ++k) s = s + a[k] * pQ[k][c];
          g[c] = s;
        }
        const float xi = p[0], yi = p[1]; /* cpp:208-209 */
        /* cpp:214-218 */
        const float Aref[3][4] = {{cos_e, sin_e, 0.f, xi * sin_emo - yi * cos_emo},
                                  {-sin_e, cos_e, 0.f, xi * cos_emo + yi * sin_emo},
                                  {0.f, 0.f, 1.f, 0.f}};
        /* cpp:223-227 */
        const float Aread[3][4] = {
            {-cos_e, -sin_e, 0.f,
             -xi * sin_emo + yi * cos_emo + (xe - xo) * sin_e - (ye - yo) * cos_e},
            {sin_e, -cos_e, 0.f,
             -xi * cos_emo - yi * sin_emo + (xe - xo) * cos_e + (ye - yo) * sin_e},
            {0.f, 0.f, -1.f, 0.f}};
        /* cpp:234-239 — (-w * pInterp_pr) * A */
        const float mg[3] = {-w * g[0], -w * g[1], -w * g[2]};
        for (int c = 0; c < 4; ++c) {
          jr[c] = (mg[0] * Aref[0][c] + mg[1] * Aref[1][c]) + mg[2] * Aref[2][c];
          je[c] = (mg[0] * Aread[0][c] + mg[1] * Aread[1][c]) + mg[2] * Aread[2][c];
        }
      }
      if (jac_ref)
        for (int c = 0; c < 4; ++c) jac_ref[4 * (size_t)i + c] = (double)jr[c];
      if (jac_read)
        for (int c = 0; c < 4; ++c) jac_read[4 * (size_t)i + c] = (double)je[c];
    }
  }
  /* cpp:272-291 */
  if (summed_reference_weight == 0) return 0;
  const double factor = (double)n / summed_reference_weight;
  for (int i = 0; i < n; ++i) {
    residuals[i] *= factor;
    if (jac_ref)
      for (int c = 0; c < 4; ++c) jac_ref[4 * (size_t)i + c] *= factor;
    if (jac_read)
      for (int c = 0; c < 4; ++c) jac_read[4 * (size_t)i + c] *= factor;
  }
  return 1;
}

/* ========================================================================= */
/* Relative pose cost (relative_pose_cost_function_inl.h:8-70)               */
/* ========================================================================= */
double vgo_normalize_angle(double a) {
  const double two_pi = 2.0 * M_PI;
  return a - two_pi * floor((a + M_PI) / two_pi);
}

void vgo_relpose_evaluate(const double A[4], const double B[4], const double t_obs[3],
                          double yaw_obs, const double L[16], double r[4], double JA[16],
                          double JB[16]) {
  const double c = cos(A[3]), s = sin(A[3]);
  const double dx = B[0] - A[0], dy = B[1] - A[1], dz = B[2] - A[2];
  double e[4];
  /* inl.h:21-24 — R_z(yaw_A)^T (t_B - t_A) - t_obs */
  e[0] = (c * dx + s * dy) - t_obs[0];
  e[1] = (-s * dx + c * dy) - t_obs[1];
  e[2] = dz - t_obs[2];
  /* inl.h:27-28 */
  e[3] = vgo_normalize_angle((B[3] - A[3]) - yaw_obs);
  /* unscaled Jacobians (what AutoDiffCostFunction<.,4,4,4> yields) */
  double ja[16] = {-c, -s, 0, -s * dx + c * dy,
                   s, -c, 0, -c * dx - s * dy,
                   0, 0, -1, 0,
                   0, 0, 0, -1};
  double jb[16] = {c, s, 0, 0,
                   -s, c, 0, 0,
                   0, 0, 1, 0,
                   0, 0, 0, 1};
  /* inl.h:59 — residuals = sqrt_information * residuals */
  for (int i = 0; i < 4; ++i) {
    double acc = 0;
    for (int k = 0; k < 4; ++k) acc += L[4 * i + k] * e[k];
    r[i] = acc;
    for (int j = 0; j < 4; ++j) {
      double sa = 0, sb = 0;
      for (int k = 0; k < 4; ++k) {
        sa += L[4 * i + k] * ja[4 * k + j];
        sb += L[4 * i + k] * jb[4 * k + j];
      }
      if (JA) JA[4 * i + j] = sa;
      if (JB) JB[4 * i + j] = sb;
    }
  }
}

/* Constraint ctor, LLT branch (constraint.cpp:8-14): sqrt_information = L (lower) */
int vgo_sqrt_information(const double info[16], double L[16]) {
  memset(L, 0, sizeof(double) * 16);
  for (int j = 0; j < 4; ++j) {
    double d = info[4 * j + j];
    for (int k = 0; k < j; ++k) d -= L[4 * j + k] * L[4 * j + k];
    if (!(d > 0)) return -1;
    L[4 * j + j] = sqrt(d);
    for (int i = j + 1; i < 4; ++i) {
      double v = info[4 * i + j];
      for (int k = 0; k < j; ++k) v -= L[4 * i + k] * L[4 * j + k];
      L[4 * i + j] = v / L[4 * j + j];
    }
  }
  return 0;
}

/* Constraint ctor, LDLT branch (constraint.cpp:15-37). Eigen's LDLT (lower, in place) picks
 * the largest remaining |diagonal| as pivot and applies it as a symmetric transposition. */
int vgo_sqrt_information_ldlt(const double info[16], double S[16]) {
  double A[4][4];
  int tr[4];
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) A[i][j] = info[4 * i + j];
  int sign_pos = 1;
  for (int k = 0; k < 4; ++k) {
    int piv = k;
    double best = fabs(A[k][k]);
    for (int i = k + 1; i < 4; ++i)
      if (fabs(A[i][i]) > best) { best = fabs(A[i][i]); piv = i; }
    tr[k] = piv;
    if (piv != k) {
      /* symmetric swap of rows/columns k and piv (full matrix kept symmetric) */
      for (int j = 0; j < 4; ++j) { double t = A[k][j]; A[k][j] = A[piv][j]; A[piv][j] = t; }
      for (int i = 0; i < 4; ++i) { double t = A[i][k]; A[i][k] = A[i][piv]; A[i][piv] = t; }
    }
    /* eliminate: A = L D L^T step on the trailing block */
    const double d = A[k][k];
    if (d < -1e-12 * (1.0 + best)) sign_pos = 0;
    if (fabs(d) > 0) {
      for (int i = k + 1; i < 4; ++i) A[i][k] /= d;
      for (int i = k + 1; i < 4; ++i)
        for (int j = k + 1; j < 4; ++j) A[i][j] -= A[i][k] * d * A[j][k];
    } else {
      for (int i = k + 1; i < 4; ++i) A[i][k] = 0;
    }
    for (int j = k + 1; j < 4; ++j) A[k][j] = 0; /* keep L strictly lower */
  }
  if (!sign_pos) return -1;
  /* M = L * sqrt(D) */
  double M[4][4];
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      const double l = (i == j) ? 1.0 : (i > j ? A[i][j] : 0.0);
      const double d = A[j][j] > 0 ? sqrt(A[j][j]) : 0.0;
      M[i][j] = l * d;
    }
  /* S = P^T M P with P = product of the transpositions (applied in order) */
  int perm[4] = {0, 1, 2, 3};
  for (int k = 0; k < 4; ++k) { int t = perm[k]; perm[k] = perm[tr[k]]; perm[tr[k]] = t; }
  /* (P x)[k] = x[perm[k]]  =>  S[perm[i]][perm[j]] = M[i][j] */
  memset(S, 0, sizeof(double) * 16);
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) S[4 * perm[i] + perm[j]] = M[i][j];
  return 0;
}

/* ========================================================================= */
/* Pose graph + LM                                                           */
/* ========================================================================= */
typedef struct {
  int a, b; /* node indices */
  double t_obs[3], yaw_obs, L[16];
} rel_edge;

typedef struct {
  int ref, read; /* node indices */
  const vgo_layer* layer;
  int n;
  const float *xyz, *distance, *weight;
  double no_corr;
} reg_edge;

struct vgo_graph {
  int n_nodes, cap_nodes;
  uint32_t* ids;
  double* x; /* n x 4 */
  int* constant;
  int n_rel, cap_rel;
  rel_edge* rel;
  int n_reg, cap_reg;
  reg_edge* reg;
};

vgo_graph* vgo_graph_create(void) { return (vgo_graph*)calloc(1, sizeof(vgo_graph)); }
void vgo_graph_destroy(vgo_graph* g) {
  if (!g) return;
  free(g->ids); free(g->x); free(g->constant); free(g->rel); free(g->reg); free(g);
}
static int node_index(const vgo_graph* g, uint32_t id) {
  for (int i = 0; i < g->n_nodes; ++i)
    if (g->ids[i] == id) return i;
  return -1;
}
int vgo_graph_add_node(vgo_graph* g, uint32_t id, const double x[4], int constant) {
  if (g->n_nodes == g->cap_nodes) {
    g->cap_nodes = g->cap_nodes ? 2 * g->cap_nodes : 64;
    g->ids = (uint32_t*)realloc(g->ids, sizeof(uint32_t) * g->cap_nodes);
    g->x = (double*)realloc(g->x, sizeof(double) * 4 * g->cap_nodes);
    g->constant = (int*)realloc(g->constant, sizeof(int) * g->cap_nodes);
  }
  int i = g->n_nodes++;
  g->ids[i] = id;
  memcpy(g->x + 4 * i, x, sizeof(double) * 4);
  g->constant[i] = constant;
  return i;
}
int vgo_graph_add_relative(vgo_graph* g, uint32_t id_a, uint32_t id_b, const double t_obs[3],
                           double yaw_obs, const double L[16]) {
  int a = node_index(g, id_a), b = node_index(g, id_b);
  if (a < 0 || b < 0) return -1;
  if (g->n_rel == g->cap_rel) {
    g->cap_rel = g->cap_rel ? 2 * g->cap_rel : 64;
    g->rel = (rel_edge*)realloc(g->rel, sizeof(rel_edge) * g->cap_rel);
  }
  rel_edge* e = &g->rel[g->n_rel++];
  e->a = a; e->b = b;
  memcpy(e->t_obs, t_obs, sizeof(double) * 3);
  e->yaw_obs = yaw_obs;
  memcpy(e->L, L, sizeof(double) * 16);
  return g->n_rel - 1;
}
int vgo_graph_add_registration(vgo_graph* g, uint32_t ref_id, uint32_t read_id,
                               const vgo_layer* layer, int n, const float* xyz,
                               const float* distance, const float* weight, double no_corr) {
  int a = node_index(g, ref_id), b = node_index(g, read_id);
  if (a < 0 || b < 0 || a == b) return -1; /* pose_graph.cpp:50-57 CHECKs */
  if (g->n_reg == g->cap_reg) {
    g->cap_reg = g->cap_reg ? 2 * g->cap_reg : 64;
    g->reg = (reg_edge*)realloc(g->reg, sizeof(reg_edge) * g->cap_reg);
  }
  reg_edge* e = &g->reg[g->n_reg++];
  e->ref = a; e->read = b; e->layer = layer; e->n = n;
  e->xyz = xyz; e->distance = distance; e->weight = weight; e->no_corr = no_corr;
  return g->n_reg - 1;
}
void vgo_graph_reset_registration(vgo_graph* g) { g->n_reg = 0; }
int vgo_graph_num_nodes(const vgo_graph* g) { return g->n_nodes; }
int vgo_graph_num_registration_residuals(const vgo_graph* g) {
  int s = 0;
  for (int i = 0; i < g->n_reg; ++i) s += g->reg[i].n;
  return s;
}
void vgo_graph_get_poses(const vgo_graph* g, double* x) {
  memcpy(x, g->x, sizeof(double) * 4 * g->n_nodes);
}
void vgo_graph_set_poses(vgo_graph* g, const double* x) {
  memcpy(g->x, x, sizeof(double) * 4 * g->n_nodes);
}

/* One residual block per task across threads, as Ceres' evaluator does. */
typedef struct {
  vgo_graph* g;
  const double* x;
  double* blk;
  int want_j, kmax;
  atomic_int next;
} reg_job;

/* Persistent worker pool: Ceres keeps its evaluation threads alive between iterations, so the
 * baseline must not pay thread creation per evaluation. Workers sleep on a condition variable;
 * an evaluation publishes a job, wakes them and waits until all have finished. */
static struct {
  pthread_mutex_t mu;
  pthread_cond_t wake, done;
  pthread_t* threads;
  int n_threads;      /* workers created so far */
  int active;         /* workers taking part in the current job */
  int remaining;      /* workers that have not finished the current job */
  unsigned long generation;
  void* (*fn)(void*);
  void* arg;
} g_pool = {PTHREAD_MUTEX_INITIALIZER, PTHREAD_COND_INITIALIZER, PTHREAD_COND_INITIALIZER,
            NULL, 0, 0, 0, 0, NULL, NULL};

/* Worker t is pinned to the t-th CPU of the process's affinity mask (round robin): without it
 * the evaluation time of the same problem varied 5x between runs on the shared GPU hosts
 * (threads migrating between sockets / sharing cores).  VGO_PIN=0 disables it. */
static void pool_pin_self(int id) {
  const char* e = getenv("VGO_PIN");
  if (e && e[0] == '0') return;
  cpu_set_t all;
  CPU_ZERO(&all);
  if (sched_getaffinity(0, sizeof(all), &all) != 0) return;
  const int n = CPU_COUNT(&all);
  if (n <= 0) return;
  int want = id % n, seen = 0;
  for (int c = 0; c < CPU_SETSIZE; ++c) {
    if (!CPU_ISSET(c, &all)) continue;
    if (seen++ == want) {
      cpu_set_t one;
      CPU_ZERO(&one);
      CPU_SET(c, &one);
      pthread_setaffinity_np(pthread_self(), sizeof(one), &one);
      return;
    }
  }
}

static void* pool_main(void* p) {
  const int id = (int)(intptr_t)p;
  unsigned long seen = 0;
  pool_pin_self(id);
  pthread_mutex_lock(&g_pool.mu);
  for (;;) {
    while (g_pool.generation == seen) pthread_cond_wait(&g_pool.wake, &g_pool.mu);
    seen = g_pool.generation;
    if (id >= g_pool.active) continue;
    void* (*fn)(void*) = g_pool.fn;
    void* arg = g_pool.arg;
    pthread_mutex_unlock(&g_pool.mu);
    fn(arg);
    pthread_mutex_lock(&g_pool.mu);
    if (--g_pool.remaining == 0) pthread_cond_signal(&g_pool.done);
  }
  return NULL;
}

/* Runs fn(arg) on nt pool threads and returns when all are done. */
static void pool_run(int nt, void* (*fn)(void*), void* arg) {
  pthread_mutex_lock(&g_pool.mu);
  if (nt > g_pool.n_threads) {
    g_pool.threads = (pthread_t*)realloc(g_pool.threads, sizeof(pthread_t) * nt);
    for (int t = g_pool.n_threads; t < nt; ++t) {
      pthread_create(&g_pool.threads[t], NULL, pool_main, (void*)(intptr_t)t);
      pthread_detach(g_pool.threads[t]);
    }
    g_pool.n_threads = nt;
  }
  g_pool.fn = fn; g_pool.arg = arg;
  g_pool.active = nt; g_pool.remaining = nt;
  g_pool.generation++;
  pthread_cond_broadcast(&g_pool.wake);
  while (g_pool.remaining > 0) pthread_cond_wait(&g_pool.done, &g_pool.mu);
  pthread_mutex_unlock(&g_pool.mu);
}

static void* reg_worker(void* arg) {
  reg_job* job = (reg_job*)arg;
  vgo_graph* g = job->g;
  const int kmax = job->kmax, want_j = job->want_j;
  /* per-thread scratch survives between evaluations (Ceres preallocates its Jacobian too) */
  static __thread double* tl_buf = NULL;
  static __thread size_t tl_cap = 0;
  const size_t need = 9 * (size_t)(kmax > 0 ? kmax : 1);
  if (need > tl_cap) {
    free(tl_buf);
    tl_buf = (double*)malloc(sizeof(double) * need);
    tl_cap = need;
  }
  double* r = tl_buf;
  double* J = want_j ? tl_buf + (size_t)(kmax > 0 ? kmax : 1) : NULL;
  for (;;) {
    const int e = atomic_fetch_add(&job->next, 1);
    if (e >= g->n_reg) break;
    const reg_edge* ge = &g->reg[e];
    double* Jr = J;
    double* Je = J ? J + 4 * (size_t)ge->n : NULL;
    int ok = vgo_reg_evaluate(ge->layer, ge->n, ge->xyz, ge->distance, ge->weight, ge->no_corr,
                              job->x + 4 * ge->ref, job->x + 4 * ge->read, r, Jr, Je);
    double* o = job->blk + 74 * (size_t)e;
    memset(o, 0, sizeof(double) * 74);
    o[73] = ok;
    if (!ok) continue;
    double c = 0;
    for (int i = 0; i < ge->n; ++i) c += r[i] * r[i];
    o[72] = c;
    if (!want_j) continue;
    /* J^T J and J^T r of this residual block, accumulated in double like Ceres */
    for (int i = 0; i < ge->n; ++i) {
      double row[8];
      for (int k = 0; k < 4; ++k) { row[k] = Jr[4 * (size_t)i + k]; row[4 + k] = Je[4 * (size_t)i + k]; }
      for (int a = 0; a < 8; ++a) {
        o[64 + a] += row[a] * r[i];
        for (int b = a; b < 8; ++b) o[8 * a + b] += row[a] * row[b];
      }
    }
    for (int a = 0; a < 8; ++a)
      for (int b = 0; b < a; ++b) o[8 * a + b] = o[8 * b + a];
  }
  return NULL;
}

/* Evaluate at poses x (n x 4). Jacobian-free when gradient == H == NULL. */
static int graph_eval_at(vgo_graph* g, const double* x, int num_threads, int exclude_reg,
                         double* cost_out, double* gradient, double* H, double* per_reg) {
  const int N = g->n_nodes, dim = 4 * N;
  const int want_j = (gradient != NULL) || (H != NULL);
  double cost = 0;
  if (gradient) memset(gradient, 0, sizeof(double) * dim);
  if (H) memset(H, 0, sizeof(double) * (size_t)dim * dim);
  int all_ok = 1;

  /* relative pose residual blocks */
  for (int e = 0; e < g->n_rel; ++e) {
    const rel_edge* re = &g->rel[e];
    double r[4], JA[16], JB[16];
    vgo_relpose_evaluate(x + 4 * re->a, x + 4 * re->b, re->t_obs, re->yaw_obs, re->L, r,
                         want_j ? JA : NULL, want_j ? JB : NULL);
    for (int i = 0; i < 4; ++i) cost += 0.5 * r[i] * r[i];
    if (!want_j) continue;
    const int oa = 4 * re->a, ob = 4 * re->b;
    for (int i = 0; i < 4; ++i) {
      for (int c = 0; c < 4; ++c) {
        if (gradient) {
          gradient[oa + c] += JA[4 * i + c] * r[i];
          gradient[ob + c] += JB[4 * i + c] * r[i];
        }
        if (H)
          for (int d = 0; d < 4; ++d) {
            H[(size_t)(oa + c) * dim + oa + d] += JA[4 * i + c] * JA[4 * i + d];
            H[(size_t)(ob + c) * dim + ob + d] += JB[4 * i + c] * JB[4 * i + d];
            H[(size_t)(oa + c) * dim + ob + d] += JA[4 * i + c] * JB[4 * i + d];
            H[(size_t)(ob + d) * dim + oa + c] += JA[4 * i + c] * JB[4 * i + d];
          }
      }
    }
  }

  if (!exclude_reg && g->n_reg > 0) {
    int kmax = 0;
    for (int e = 0; e < g->n_reg; ++e)
      if (g->reg[e].n > kmax) kmax = g->reg[e].n;
    double* blk = (double*)malloc(sizeof(double) * 74 * (size_t)g->n_reg); /* 64 H + 8 g + cost + ok */
    int nt = num_threads > 0 ? num_threads : 1;
    if (nt > g->n_reg) nt = g->n_reg;
    reg_job job;
    job.g = g; job.x = x; job.blk = blk; job.want_j = want_j; job.kmax = kmax; job.next = 0;
    if (nt <= 1) {
      reg_worker(&job);
    } else {
      pool_run(nt, reg_worker, &job);
    }
    for (int e = 0; e < g->n_reg; ++e) {
      const reg_edge* ge = &g->reg[e];
      const double* o = blk + 74 * (size_t)e;
      if (o[73] == 0) { all_ok = 0; if (per_reg) per_reg[e] = 0; continue; }
      cost += 0.5 * o[72];
      if (per_reg) per_reg[e] = o[72];
      if (!want_j) continue;
      const int off[2] = {4 * ge->ref, 4 * ge->read};
      for (int a = 0; a < 8; ++a) {
        const int ia = off[a >> 2] + (a & 3);
        if (gradient) gradient[ia] += o[64 + a];
        if (H)
          for (int b = 0; b < 8; ++b) {
            const int ib = off[b >> 2] + (b & 3);
            H[(size_t)ia * dim + ib] += o[8 * a + b];
          }
      }
    }
    free(blk);
  }
  if (cost_out) *cost_out = cost;
  return all_ok;
}

int vgo_graph_eval(vgo_graph* g, int num_threads, int exclude_reg, double* cost,
                   double* gradient, double* H) {
  return graph_eval_at(g, g->x, num_threads, exclude_reg, cost, gradient, H, NULL);
}

void vgo_graph_registration_costs(vgo_graph* g, double* per) {
  double c;
  graph_eval_at(g, g->x, 1, 0, &c, NULL, NULL, per);
}

void vgo_solver_options_default(vgo_solver_options* o) {
  o->max_num_iterations = 50;
  o->parameter_tolerance = 3e-3; /* pose_graph.cpp:93 */
  o->function_tolerance = 1e-6;
  o->gradient_tolerance = 1e-10;
  o->initial_trust_region_radius = 1e4;
  o->max_trust_region_radius = 1e16;
  o->min_trust_region_radius = 1e-32;
  o->min_relative_decrease = 1e-3;
  o->min_lm_diagonal = 1e-6;
  o->max_lm_diagonal = 1e32;
  o->max_solver_time_s = 4.0; /* pose_graph.cpp:95 */
  o->jacobi_scaling = 1;
  o->num_threads = 4; /* pose_graph.cpp:96 */
  o->exclude_registration = 0;
}

/* dense Cholesky solve of A x = b (A n x n SPD, row-major, destroyed). 0 ok. */
static int chol_solve(double* A, double* b, int n) {
  for (int j = 0; j < n; ++j) {
    double d = A[(size_t)j * n + j];
    for (int k = 0; k < j; ++k) d -= A[(size_t)j * n + k] * A[(size_t)j * n + k];
    if (!(d > 0) || !isfinite(d)) return -1;
    d = sqrt(d);
    A[(size_t)j * n + j] = d;
    for (int i = j + 1; i < n; ++i) {
      double v = A[(size_t)i * n + j];
      const double* ri = A + (size_t)i * n;
      const double* rj = A + (size_t)j * n;
      for (int k = 0; k < j; ++k) v -= ri[k] * rj[k];
      A[(size_t)i * n + j] = v / d;
    }
  }
  for (int i = 0; i < n; ++i) {
    double v = b[i];
    for (int k = 0; k < i; ++k) v -= A[(size_t)i * n + k] * b[k];
    b[i] = v / A[(size_t)i * n + i];
  }
  for (int i = n - 1; i >= 0; --i) {
    double v = b[i];
    for (int k = i + 1; k < n; ++k) v -= A[(size_t)k * n + i] * b[k];
    b[i] = v / A[(size_t)i * n + i];
  }
  return 0;
}

/* Ceres 1.x TrustRegionMinimizer + LevenbergMarquardtStrategy on the normal
 * equations (A.6). Constant nodes are removed from the reduced problem. */
int vgo_graph_solve(vgo_graph* g, const vgo_solver_options* o, vgo_solver_summary* sum) {
  const double t0 = now_s();
  const int N = g->n_nodes, dim = 4 * N;
  int* map = (int*)malloc(sizeof(int) * dim); /* reduced index -> full index */
  int n = 0;
  for (int i = 0; i < N; ++i)
    if (!g->constant[i])
      for (int c = 0; c < 4; ++c) map[n++] = 4 * i + c;

  double* x = (double*)malloc(sizeof(double) * dim);
  double* xc = (double*)malloc(sizeof(double) * dim);
  double* grad = (double*)malloc(sizeof(double) * dim);
  double* H = (double*)malloc(sizeof(double) * (size_t)dim * dim);
  double* Hs = (double*)malloc(sizeof(double) * (size_t)(n ? n : 1) * (n ? n : 1));
  double* A = (double*)malloc(sizeof(double) * (size_t)(n ? n : 1) * (n ? n : 1));
  double* gs = (double*)malloc(sizeof(double) * (n ? n : 1));
  double* step = (double*)malloc(sizeof(double) * (n ? n : 1));
  double* scale = (double*)malloc(sizeof(double) * (n ? n : 1));
  double* diag = (double*)malloc(sizeof(double) * (n ? n : 1));
  memcpy(x, g->x, sizeof(double) * dim);

  vgo_solver_summary S;
  memset(&S, 0, sizeof(S));
  S.termination = 3;
  double cost = 0, t_eval = 0, t_lin = 0;
  double te = now_s();
  int ok = graph_eval_at(g, x, o->num_threads, o->exclude_registration, &cost, grad, H, NULL);
  t_eval += now_s() - te;
  S.num_residual_evals = 1;
  S.initial_cost = cost;
  int ret = 0;
  if (!ok) { S.termination = 6; ret = -1; goto done; }

  /* Jacobi scaling from the initial Jacobian column norms */
  for (int i = 0; i < n; ++i) {
    double cn = H[(size_t)map[i] * dim + map[i]];
    scale[i] = o->jacobi_scaling ? 1.0 / (1.0 + sqrt(cn)) : 1.0;
  }
  double radius = o->initial_trust_region_radius, decrease_factor = 2.0;
  int reuse_diagonal = 0, consecutive_invalid = 0;

  for (;;) {
    /* FinalizeIterationAndCheckIfMinimizerCanContinue */
    double gmax = 0;
    for (int i = 0; i < n; ++i) {
      double v = fabs(grad[map[i]]);
      if (v > gmax) gmax = v;
    }
    if (now_s() - t0 >= o->max_solver_time_s) { S.termination = 4; break; }
    if (S.iterations >= o->max_num_iterations) { S.termination = 3; break; }
    if (gmax <= o->gradient_tolerance) { S.termination = 2; break; }
    if (radius <= o->min_trust_region_radius) { S.termination = 5; break; }
    S.iterations++;

    /* scaled normal equations */
    for (int i = 0; i < n; ++i) {
      gs[i] = scale[i] * grad[map[i]];
      for (int j = 0; j < n; ++j)
        Hs[(size_t)i * n + j] = scale[i] * scale[j] * H[(size_t)map[i] * dim + map[j]];
    }
    if (!reuse_diagonal)
      for (int i = 0; i < n; ++i) {
        double d = Hs[(size_t)i * n + i];
        if (d < o->min_lm_diagonal) d = o->min_lm_diagonal;
        if (d > o->max_lm_diagonal) d = o->max_lm_diagonal;
        diag[i] = d;
      }
    memcpy(A, Hs, sizeof(double) * (size_t)n * n);
    for (int i = 0; i < n; ++i) {
      double lm = sqrt(diag[i] / radius);
      A[(size_t)i * n + i] += lm * lm;
      step[i] = gs[i];
    }
    double tl = now_s();
    int lin_ok = chol_solve(A, step, n) == 0;
    t_lin += now_s() - tl;
    double model_cost_change = 0;
    if (lin_ok) {
      for (int i = 0; i < n; ++i) {
        step[i] = -step[i];
        if (!isfinite(step[i])) lin_ok = 0;
      }
    }
    if (lin_ok) {
      /* model_cost_change = -step^T gs - 1/2 step^T Hs step */
      for (int i = 0; i < n; ++i) {
        double hv = 0;
        for (int j = 0; j < n; ++j) hv += Hs[(size_t)i * n + j] * step[j];
        model_cost_change += -step[i] * (gs[i] + 0.5 * hv);
      }
    }
    if (!lin_ok || !(model_cost_change > 0)) {
      /* HandleInvalidStep */
      if (++consecutive_invalid >= 5) { S.termination = 6; ret = -1; break; }
      radius /= decrease_factor; decrease_factor *= 2; reuse_diagonal = 1;
      continue;
    }
    consecutive_invalid = 0;
    /* candidate = Plus(x, step .* scale): xyz additive, yaw wrapped */
    memcpy(xc, x, sizeof(double) * dim);
    double step_norm2 = 0, x_norm2 = 0;
    for (int i = 0; i < n; ++i) {
      const int f = map[i];
      const double d = step[i] * scale[i];
      xc[f] = ((f & 3) == 3) ? vgo_normalize_angle(x[f] + d) : x[f] + d;
      const double dd = x[f] - xc[f];
      step_norm2 += dd * dd;
      x_norm2 += x[f] * x[f];
    }
    double cand_cost = 0;
    te = now_s();
    int cok = graph_eval_at(g, xc, o->num_threads, o->exclude_registration, &cand_cost, NULL,
                            NULL, NULL);
    t_eval += now_s() - te;
    S.num_residual_evals++;
    if (!cok) {
      if (++consecutive_invalid >= 5) { S.termination = 6; ret = -1; break; }
      radius /= decrease_factor; decrease_factor *= 2; reuse_diagonal = 1;
      continue;
    }
    /* ParameterToleranceReached */
    const double x_norm = sqrt(x_norm2);
    if (sqrt(step_norm2) <= o->parameter_tolerance * (x_norm + o->parameter_tolerance)) {
      S.termination = 0;
      break;
    }
    /* FunctionToleranceReached */
    const double cost_change = cost - cand_cost;
    if (fabs(cost_change) <= o->function_tolerance * cost) { S.termination = 1; break; }
    const double rel_decrease = cost_change / model_cost_change;
    if (rel_decrease > o->min_relative_decrease) {
      /* HandleSuccessfulStep */
      memcpy(x, xc, sizeof(double) * dim);
      te = now_s();
      ok = graph_eval_at(g, x, o->num_threads, o->exclude_registration, &cost, grad, H, NULL);
      t_eval += now_s() - te;
      S.num_residual_evals++;
      S.num_successful_steps++;
      if (!ok) { S.termination = 6; ret = -1; break; }
      double q = 2.0 * rel_decrease - 1.0;
      double den = 1.0 - q * q * q;
      if (den < 1.0 / 3.0) den = 1.0 / 3.0;
      radius = radius / den;
      if (radius > o->max_trust_region_radius) radius = o->max_trust_region_radius;
      decrease_factor = 2.0;
      reuse_diagonal = 0;
    } else {
      radius /= decrease_factor; decrease_factor *= 2; reuse_diagonal = 1;
    }
  }
done:
  memcpy(g->x, x, sizeof(double) * dim);
  S.final_cost = cost;
  S.total_time_s = now_s() - t0;
  S.eval_time_s = t_eval;
  S.linear_solver_time_s = t_lin;
  if (sum) *sum = S;
  free(map); free(x); free(xc); free(grad); free(H); free(Hs); free(A); free(gs);
  free(step); free(scale); free(diag);
  return ret;
}

/* ========================================================================= */
/* SURVEY §8f rows: registration-voxel extraction, OBB/AABB, overlap test    */
/* ========================================================================= */
int vgo_find_relevant_voxels(const vgo_layer* l, double min_w, double max_d, float* xyz,
                             float* distance, float* weight, int max_n) {
  int n = 0;
  const int vps = l->vps;
  for (int b = 0; b < l->n_blocks; ++b) {
    const int32_t* bi = l->idx + 3 * b;
    const float origin[3] = {(float)bi[0] * l->block_size, (float)bi[1] * l->block_size,
                             (float)bi[2] * l->block_size};
    for (int lin = 0; lin < l->vox_per_block; ++lin) {
      const size_t o = (size_t)b * l->vox_per_block + lin;
      /* cpp:177-178 (double comparison of float members) */
      if ((double)l->weight[o] > min_w && fabs((double)l->distance[o]) < max_d) {
        if (n < max_n) {
          /* Block::computeCoordinatesFromLinearIndex: origin + (voxel_index + 0.5) * voxel_size */
          const int vx = lin % vps, vy = (lin / vps) % vps, vz = lin / (vps * vps);
          xyz[3 * n + 0] = origin[0] + ((float)vx + 0.5f) * l->voxel_size;
          xyz[3 * n + 1] = origin[1] + ((float)vy + 0.5f) * l->voxel_size;
          xyz[3 * n + 2] = origin[2] + ((float)vz + 0.5f) * l->voxel_size;
          distance[n] = l->distance[o];
          weight[n] = l->weight[o];
        }
        ++n;
      }
    }
  }
  return n;
}

/* Interpolator::getVoxel(pos, &voxel, interpolate = true) -> getInterpVoxel: distance and weight
 * are each q * (interp_table * values^T) with the B1 table of the cost function (A.3) */
int vgo_interp_voxel(const vgo_layer* l, const float pos[3], float* distance, float* weight) {
  int32_t bb[3], bv[3], slots[8], lin[8];
  float d[8], q[8], w[8];
  if (!vgo_interp_voxels_and_q(l, pos, bb, bv, slots, lin, d, q)) return 0;
  for (int i = 0; i < 8; ++i) w[i] = l->weight[(size_t)slots[i] * l->vox_per_block + lin[i]];
  const float* v[2] = {d, w};
  float out[2];
  for (int k = 0; k < 2; ++k) {
    const float* x = v[k];
    float a[8];
    a[0] = x[0];
    a[1] = -x[0] + x[4];
    a[2] = -x[0] + x[2];
    a[3] = -x[0] + x[1];
    a[4] = x[0] - x[2] - x[4] + x[6];
    a[5] = x[0] - x[1] - x[2] + x[3];
    a[6] = x[0] - x[1] - x[4] + x[5];
    a[7] = -x[0] + x[1] + x[2] - x[3] + x[4] - x[5] - x[6] + x[7];
    float r = q[0] * a[0];
    for (int i = 1; i < 8; ++i) r = r + q[i] * a[i];
    out[k] = r;
  }
  *distance = out[0];
  *weight = out[1];
  return 1;
}

/* marching cubes corner offsets and edge end points (voxblox marching_cubes.h) */
static const int kCubeOffset[8][3] = {{0, 0, 0}, {1, 0, 0}, {1, 1, 0}, {0, 1, 0},
                                      {0, 0, 1}, {1, 0, 1}, {1, 1, 1}, {0, 1, 1}};
static const int kEdgePairs[12][2] = {{0, 1}, {1, 2}, {2, 3}, {3, 0}, {4, 5}, {5, 6},
                                      {6, 7}, {7, 4}, {0, 4}, {1, 5}, {2, 6}, {3, 7}};

/* The marching cube whose origin is voxel `lin` of block slot `b`: corner distances and coordinates.
 * Returns 0 unless all 8 corners exist and have weight > min_weight. */
static int iso_cube(const vgo_layer* l, int b, int lin, float min_weight, float sdf[8], float cc[8][3]) {
  const int vps = l->vps;
  const int32_t* bi = l->idx + 3 * b;
  const float origin[3] = {(float)bi[0] * l->block_size, (float)bi[1] * l->block_size,
                           (float)bi[2] * l->block_size};
  const int v[3] = {lin % vps, (lin / vps) % vps, lin / (vps * vps)};
  /* cube origin coordinates = voxel centre (Block::computeCoordinatesFromVoxelIndex) */
  const float coords[3] = {origin[0] + ((float)v[0] + 0.5f) * l->voxel_size,
                           origin[1] + ((float)v[1] + 0.5f) * l->voxel_size,
                           origin[2] + ((float)v[2] + 0.5f) * l->voxel_size};
  for (int i = 0; i < 8; ++i) {
    int cv[3], cb[3];
    for (int a = 0; a < 3; ++a) {
      cv[a] = v[a] + kCubeOffset[i][a];
      cb[a] = bi[a];
      if (cv[a] >= vps) { cv[a] -= vps; cb[a] += 1; }
    }
    const int32_t cbi[3] = {cb[0], cb[1], cb[2]};
    const int slot = vgo_layer_find_block(l, cbi);
    if (slot < 0) return 0;
    const size_t o = (size_t)slot * l->vox_per_block + cv[0] + vps * (cv[1] + vps * cv[2]);
    /* utils::getSdfIfValid: weight <= min_weight -> invalid */
    if (l->weight[o] <= min_weight) return 0;
    sdf[i] = l->distance[o];
    /* corner_coords = coords + cube_coord_offsets (offset = index offset * voxel_size) */
    for (int a = 0; a < 3; ++a) cc[i][a] = coords[a] + (float)kCubeOffset[i][a] * l->voxel_size;
  }
  return 1;
}

static inline int iso_edge_crosses(float s1, float s2) { return (s1 < 0 && s2 >= 0) || (s1 >= 0 && s2 < 0); }

int vgo_find_isosurface_vertices(const vgo_layer* l, double min_w, float* xyz, float* distance,
                                 float* weight, int max_n, int32_t* iso_blocks, int max_blocks,
                                 int* n_blocks_out) {
  const float min_weight = (float)min_w; /* cpp:211-212 static_cast<float> */
  /* createConnectedMesh: threshold_inv = 1. / double(float threshold), threshold = 0.5 * voxel_size */
  const float threshold = (float)(0.5 * (double)l->voxel_size);
  const double threshold_inv = 1.0 / (double)threshold;
  /* count the candidate vertices first: the bucket set holds at most one key per candidate, and
   * open addressing needs a free slot to end every probe */
  size_t n_cand = 0;
  for (int b = 0; b < l->n_blocks; ++b)
    for (int lin = 0; lin < l->vox_per_block; ++lin) {
      float sdf[8], cc[8][3];
      if (!iso_cube(l, b, lin, min_weight, sdf, cc)) continue;
      for (int e = 0; e < 12; ++e) n_cand += (size_t)iso_edge_crosses(sdf[kEdgePairs[e][0]], sdf[kEdgePairs[e][1]]);
    }
  /* bucket set: open addressing on the three int64 bucket coordinates */
  size_t cap = 1024;
  while (cap < 2 * n_cand) cap <<= 1;
  int64_t* keys = (int64_t*)malloc(sizeof(int64_t) * 3 * cap);
  uint8_t* used = (uint8_t*)calloc(cap, 1);
  /* isosurface block set: a vertex lies in its cube's block or one of the 7 forward neighbours */
  size_t bcap = 64;
  while (bcap < 16 * (size_t)l->n_blocks) bcap <<= 1;
  int32_t* bkeys = (int32_t*)malloc(sizeof(int32_t) * 3 * bcap);
  uint8_t* bused = (uint8_t*)calloc(bcap, 1);
  int n = 0, nb = 0;
  for (int b = 0; b < l->n_blocks; ++b) {
    for (int lin = 0; lin < l->vox_per_block; ++lin) {
      float sdf[8], cc[8][3];
      if (!iso_cube(l, b, lin, min_weight, sdf, cc)) continue;
      for (int e = 0; e < 12; ++e) {
        const int e0 = kEdgePairs[e][0], e1 = kEdgePairs[e][1];
        const float s1 = sdf[e0], s2 = sdf[e1];
        if (!iso_edge_crosses(s1, s2)) continue;
        /* MarchingCubes::interpolateVertex */
        float p[3];
        const float diff = s1 - s2;
        if (fabsf(diff) >= 1e-6f) {
          const float t = s1 / diff;
          for (int a = 0; a < 3; ++a) p[a] = cc[e0][a] + t * (cc[e1][a] - cc[e0][a]);
        } else {
          for (int a = 0; a < 3; ++a) p[a] = 0.5f * (cc[e0][a] + cc[e1][a]);
        }
        /* createConnectedMesh: bucket = round(double(vertex) * threshold_inv) */
        int64_t k3[3];
        for (int a = 0; a < 3; ++a) k3[a] = (int64_t)llround((double)p[a] * threshold_inv);
        uint64_t h = any_index_hash(k3[0], k3[1], k3[2]);
        h ^= h >> 29;
        size_t pos = (size_t)(h * 0x9E3779B97F4A7C15ull) & (cap - 1);
        int dup = 0;
        while (used[pos]) {
          if (keys[3 * pos] == k3[0] && keys[3 * pos + 1] == k3[1] && keys[3 * pos + 2] == k3[2]) { dup = 1; break; }
          pos = (pos + 1) & (cap - 1);
        }
        if (dup) continue;
        used[pos] = 1;
        keys[3 * pos] = k3[0]; keys[3 * pos + 1] = k3[1]; keys[3 * pos + 2] = k3[2];
        /* voxgraph_submap.cpp:226-241 */
        float vd, vw;
        if (!vgo_interp_voxel(l, p, &vd, &vw)) continue;
        if (n < max_n) {
          xyz[3 * n] = p[0]; xyz[3 * n + 1] = p[1]; xyz[3 * n + 2] = p[2];
          distance[n] = vd;
          weight[n] = vw;
        }
        ++n;
        int32_t ib[3];
        vgo_grid_index_from_point(p, l->block_size_inv, ib);
        size_t bp = (size_t)any_index_hash(ib[0], ib[1], ib[2]) & (bcap - 1);
        int seen = 0;
        while (bused[bp]) {
          if (bkeys[3 * bp] == ib[0] && bkeys[3 * bp + 1] == ib[1] && bkeys[3 * bp + 2] == ib[2]) { seen = 1; break; }
          bp = (bp + 1) & (bcap - 1);
        }
        if (!seen) {
          bused[bp] = 1;
          bkeys[3 * bp] = ib[0]; bkeys[3 * bp + 1] = ib[1]; bkeys[3 * bp + 2] = ib[2];
          if (nb < max_blocks) { iso_blocks[3 * nb] = ib[0]; iso_blocks[3 * nb + 1] = ib[1]; iso_blocks[3 * nb + 2] = ib[2]; }
          ++nb;
        }
      }
    }
  }
  free(keys);
  free(used);
  free(bkeys);
  free(bused);
  if (n_blocks_out) *n_blocks_out = nb;
  return n;
}

/* ========================================================================= */
/* ESDF generation (fixed point of EsdfIntegrator's batch update)            */
/* ========================================================================= */
void vgo_esdf_config_default(vgo_esdf_config* c) {
  c->max_distance_m = 2.0f;
  c->default_distance_m = 2.0f;
  c->min_distance_m = 0.2f;
  c->min_weight = 1e-6f;
}

int vgo_generate_esdf(const vgo_layer* l, const vgo_esdf_config* c, float* dist, float* obs) {
  const int vps = l->vps, vpb = l->vox_per_block;
  const size_t nvox = (size_t)l->n_blocks * vpb;
  uint8_t* fixed = (uint8_t*)calloc(nvox ? nvox : 1, 1);
  for (size_t i = 0; i < nvox; ++i) {
    const float w = l->weight[i], d = l->distance[i];
    if (w < c->min_weight) { dist[i] = 0.f; obs[i] = 0.f; continue; }
    obs[i] = 1.f;
    if (fabsf(d) < c->min_distance_m) { fixed[i] = 1; dist[i] = d; }
    else dist[i] = (d > 0.f ? 1.f : -1.f) * c->default_distance_m;   /* signum(tsdf) * default */
  }
  /* neighbour slots of every block (27, centre included) */
  int* nb = (int*)malloc(sizeof(int) * 27 * (size_t)(l->n_blocks ? l->n_blocks : 1));
  for (int b = 0; b < l->n_blocks; ++b)
    for (int k = 0; k < 27; ++k) {
      const int32_t q[3] = {l->idx[3 * b] + (k % 3) - 1, l->idx[3 * b + 1] + ((k / 3) % 3) - 1,
                            l->idx[3 * b + 2] + (k / 9) - 1};
      nb[27 * b + k] = vgo_layer_find_block(l, q);
    }
  int sweeps = 0, changed = 1;
  while (changed) {
    changed = 0;
    ++sweeps;
    for (int b = 0; b < l->n_blocks; ++b)
      for (int lin = 0; lin < vpb; ++lin) {
        const size_t i = (size_t)b * vpb + lin;
        if (obs[i] == 0.f || fixed[i]) continue;
        const int v[3] = {lin % vps, (lin / vps) % vps, lin / (vps * vps)};
        float d = dist[i];
        for (int dz = -1; dz <= 1; ++dz)
          for (int dy = -1; dy <= 1; ++dy)
            for (int dx = -1; dx <= 1; ++dx) {
              if (!dx && !dy && !dz) continue;
              int q[3] = {v[0] + dx, v[1] + dy, v[2] + dz}, bo[3] = {1, 1, 1};
              for (int a = 0; a < 3; ++a) {
                if (q[a] < 0) { q[a] += vps; bo[a] = 0; }
                else if (q[a] >= vps) { q[a] -= vps; bo[a] = 2; }
              }
              const int s = nb[27 * b + bo[0] + 3 * bo[1] + 9 * bo[2]];
              if (s < 0) continue;
              const size_t j = (size_t)s * vpb + q[0] + vps * (q[1] + vps * q[2]);
              if (obs[j] == 0.f) continue;
              const float dn = dist[j];
              /* |offset| * voxel_size: 1, sqrt(2), sqrt(3) in float */
              const int m = abs(dx) + abs(dy) + abs(dz);
              const float step = (m == 1 ? 1.0f : (m == 2 ? sqrtf(2.0f) : sqrtf(3.0f))) * l->voxel_size;
              if (d > 0.f && dn > 0.f) {
                const float cand = dn + step;
                if (cand < c->max_distance_m && cand < d) d = cand;
              } else if (d < 0.f && dn < 0.f) {
                const float cand = dn - step;
                if (cand > -c->max_distance_m && cand > d) d = cand;
              }
            }
        if (d != dist[i]) { dist[i] = d; changed = 1; }
      }
  }
  free(nb); free(fixed);
  return sweeps;
}

int vgo_surface_obb(const vgo_layer* l, double min_w, double max_d, float mn[3], float mx[3]) {
  const int vps = l->vps;
  const float half = 0.5f * l->voxel_size;
  int any = 0;
  for (int a = 0; a < 3; ++a) { mn[a] = INFINITY; mx[a] = -INFINITY; }
  for (int b = 0; b < l->n_blocks; ++b) {
    const int32_t* bi = l->idx + 3 * b;
    const float origin[3] = {(float)bi[0] * l->block_size, (float)bi[1] * l->block_size,
                             (float)bi[2] * l->block_size};
    for (int lin = 0; lin < l->vox_per_block; ++lin) {
      const size_t o = (size_t)b * l->vox_per_block + lin;
      if ((double)l->weight[o] > min_w && fabs((double)l->distance[o]) < max_d) {
        const int v[3] = {lin % vps, (lin / vps) % vps, lin / (vps * vps)};
        for (int a = 0; a < 3; ++a) {
          const float c = origin[a] + ((float)v[a] + 0.5f) * l->voxel_size;
          if (c - half < mn[a]) mn[a] = c - half;
          if (c + half > mx[a]) mx[a] = c + half;
        }
        any = 1;
      }
    }
  }
  return any;
}

void vgo_aabb_from_obb_and_pose(const float omin[3], const float omax[3], const float pose[7],
                                float amin[3], float amax[3]) {
  for (int a = 0; a < 3; ++a) { amin[a] = INFINITY; amax[a] = -INFINITY; }
  for (unsigned i = 0; i < 8; ++i) {
    /* getCornerCoordinates: bit set -> min, clear -> max */
    const float corner[3] = {(i & 1) ? omin[0] : omax[0], (i & 2) ? omin[1] : omax[1],
                             (i & 4) ? omin[2] : omax[2]};
    float m[3];
    vgo_T_transform(pose, corner, m);
    for (int a = 0; a < 3; ++a) {
      if (m[a] < amin[a]) amin[a] = m[a];
      if (m[a] > amax[a]) amax[a] = m[a];
    }
  }
}

int vgo_submaps_overlap(const float amin[3], const float amax[3], const float bmin[3],
                        const float bmax[3], const float pose_current[7], const float pose_other[7],
                        const int32_t* blocks, int n, float block_size, const vgo_layer* other) {
  /* cpp:251-256 */
  for (int a = 0; a < 3; ++a)
    if (amax[a] < bmin[a] || amin[a] > bmax[a]) return 0;
  /* cpp:261-262: T_other_submap__current_submap = other.getPose().inverse() * getPose() */
  float inv[7], T[7];
  vgo_T_inverse(pose_other, inv);
  vgo_T_compose(inv, pose_current, T);
  for (int i = 0; i < n; ++i) {
    /* getCenterPointFromGridIndex(block_index, block_size) */
    const float c[3] = {((float)blocks[3 * i] + 0.5f) * block_size,
                        ((float)blocks[3 * i + 1] + 0.5f) * block_size,
                        ((float)blocks[3 * i + 2] + 0.5f) * block_size};
    float p[3];
    vgo_T_transform(T, c, p);
    int32_t ob[3];
    vgo_grid_index_from_point(p, other->block_size_inv, ob);
    if (vgo_layer_find_block(other, ob) >= 0) return 1;
  }
  return 0;
}

/* ========================================================================= */
/* WeightedSampler::getRandomItem (weighted_sampler_inl.h:19-28)             */
/* ========================================================================= */
void vgo_sampler_init(vgo_sampler* s) {
  /* std::mersenne_twister_engine<uint32, 32, 624, 397, 31, 0x9908b0df, 11, 0xffffffff, 7,
   * 0x9d2c5680, 15, 0xefc60000, 18, 1812433253>, default_seed = 5489 */
  s->mt[0] = 5489u;
  for (int i = 1; i < 624; ++i)
    s->mt[i] = 1812433253u * (s->mt[i - 1] ^ (s->mt[i - 1] >> 30)) + (uint32_t)i;
  s->idx = 624;
}

uint32_t vgo_sampler_next_u32(vgo_sampler* s) {
  if (s->idx >= 624) {
    for (int i = 0; i < 624; ++i) {
      const uint32_t y = (s->mt[i] & 0x80000000u) | (s->mt[(i + 1) % 624] & 0x7fffffffu);
      uint32_t v = s->mt[(i + 397) % 624] ^ (y >> 1);
      if (y & 1u) v ^= 0x9908b0dfu;
      s->mt[i] = v;
    }
    s->idx = 0;
  }
  uint32_t y = s->mt[s->idx++];
  y ^= y >> 11;
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  y ^= y >> 18;
  return y;
}

double vgo_sampler_canonical(vgo_sampler* s) {
  /* std::generate_canonical<double, 53>: k = ceil(53 / 32) = 2 draws, sum in double,
   * divided by 2^64; a result of 1.0 is replaced by nextafter(1, 0) */
  const double g1 = (double)vgo_sampler_next_u32(s);
  const double g2 = (double)vgo_sampler_next_u32(s);
  double r = (g1 + g2 * 4294967296.0) / 18446744073709551616.0;
  if (r >= 1.0) r = nextafter(1.0, 0.0);
  return r;
}

void vgo_sampler_draw(vgo_sampler* s, const double* cum, int n, int count, int32_t* idx) {
  for (int i = 0; i < count; ++i) {
    const double t = vgo_sampler_canonical(s) * cum[n - 1];
    /* std::upper_bound: first element > t */
    int lo = 0, hi = n;
    while (lo < hi) {
      const int mid = lo + (hi - lo) / 2;
      if (cum[mid] > t) hi = mid; else lo = mid + 1;
    }
    if (lo >= n) lo = n - 1; /* the reference would read one past the end here */
    idx[i] = lo;
  }
}

/* ========================================================================= */
/* TSDF integration (A.4)                                                    */
/* ========================================================================= */
void vgo_tsdf_config_default(vgo_tsdf_config* c) {
  /* voxblox defaults overridden by voxgraph/config/voxgraph_mapper.yaml:21-28 */
  c->default_truncation_distance = 0.6f;
  c->max_weight = 10000.0f;
  c->voxel_carving_enabled = 1;
  c->min_ray_length_m = 0.1f;
  c->max_ray_length_m = 16.0f;
  c->use_const_weight = 1;
  c->allow_clear = 1;
  c->use_weight_dropoff = 1;
  c->use_sparsity_compensation_factor = 1;
  c->sparsity_compensation_factor = 20.0f;
  c->start_voxel_subsampling_factor = 2.0f;
  c->max_consecutive_ray_collisions = 2;
  c->mode = 0;
}

typedef struct {
  int64_t cur[3];
  int sign[3];
  float t_next[3], t_step[3];
  int64_t steps, current_step;
} raycaster;

static inline int signum_f(float v) { return (v > 0.f) - (v < 0.f); }

/* RayCaster::setupRayCaster (integrator_utils.cc). Degenerate axis (ray component
 * exactly 0): upstream intends t = 2.0 ("never chosen"); restated as such. */
static void raycaster_setup(raycaster* rc, const float s[3], const float e[3]) {
  if (isnan(s[0]) || isnan(s[1]) || isnan(s[2]) || isnan(e[0]) || isnan(e[1]) || isnan(e[2])) {
    rc->steps = -1; rc->current_step = 0;
    return;
  }
  int64_t end_idx[3];
  rc->steps = 0;
  for (int a = 0; a < 3; ++a) {
    rc->cur[a] = (int64_t)floorf(s[a] + VGO_COORD_EPS);
    end_idx[a] = (int64_t)floorf(e[a] + VGO_COORD_EPS);
    int64_t d = end_idx[a] - rc->cur[a];
    rc->steps += d < 0 ? -d : d;
  }
  rc->current_step = 0;
  for (int a = 0; a < 3; ++a) {
    const float ray = e[a] - s[a];
    rc->sign[a] = signum_f(ray);
    const int corrected = rc->sign[a] > 0 ? rc->sign[a] : 0;
    const float shifted = s[a] - (float)rc->cur[a];
    const float dist = (float)corrected - shifted;
    if (ray == 0.f) {
      rc->t_next[a] = 2.0f; rc->t_step[a] = 2.0f;
    } else {
      rc->t_next[a] = dist / ray;
      rc->t_step[a] = (float)rc->sign[a] / ray;
    }
  }
}

static int raycaster_next(raycaster* rc, int64_t out[3]) {
  if (rc->current_step++ > rc->steps) return 0;
  out[0] = rc->cur[0]; out[1] = rc->cur[1]; out[2] = rc->cur[2];
  /* minCoeff: first strictly-smallest */
  int m = 0;
  if (rc->t_next[1] < rc->t_next[m]) m = 1;
  if (rc->t_next[2] < rc->t_next[m]) m = 2;
  rc->cur[m] += rc->sign[m];
  rc->t_next[m] += rc->t_step[m];
  return 1;
}

/* RayCaster ctor (integrator_utils.cc) */
static void raycaster_init(raycaster* rc, const float origin[3], const float pG[3],
                           int is_clearing, int carving, float max_ray, float vsi, float trunc,
                           int cast_from_origin) {
  float d[3] = {pG[0] - origin[0], pG[1] - origin[1], pG[2] - origin[2]};
  float norm = sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
  /* Eigen normalized(): v / norm (when norm > 0) */
  float u[3] = {d[0], d[1], d[2]};
  if (norm > 0.f) { u[0] = d[0] / norm; u[1] = d[1] / norm; u[2] = d[2] / norm; }
  float rs[3], re[3];
  if (is_clearing) {
    float len = norm - trunc;
    if (len < 0.f) len = 0.f;
    if (len > max_ray) len = max_ray;
    for (int a = 0; a < 3; ++a) {
      re[a] = origin[a] + u[a] * len;
      rs[a] = carving ? origin[a] : re[a];
    }
  } else {
    for (int a = 0; a < 3; ++a) {
      re[a] = pG[a] + u[a] * trunc;
      rs[a] = carving ? origin[a] : (pG[a] - u[a] * trunc);
    }
  }
  float ss[3] = {rs[0] * vsi, rs[1] * vsi, rs[2] * vsi};
  float es[3] = {re[0] * vsi, re[1] * vsi, re[2] * vsi};
  if (cast_from_origin) raycaster_setup(rc, ss, es);
  else raycaster_setup(rc, es, ss);
}

int vgo_raycast(const float origin[3], const float pG[3], int is_clearing, int carving,
                float max_ray, float vsi, float trunc, int cast_from_origin, int64_t* out,
                int max_out) {
  raycaster rc;
  raycaster_init(&rc, origin, pG, is_clearing, carving, max_ray, vsi, trunc, cast_from_origin);
  int n = 0;
  int64_t g[3];
  while (raycaster_next(&rc, g)) {
    if (n < max_out) { out[3 * n] = g[0]; out[3 * n + 1] = g[1]; out[3 * n + 2] = g[2]; }
    n++;
  }
  return n;
}

/* Update trace (test code): the ray-ordered (voxel, sdf, update weight) tuples of an integration */
static void trace_push(vgo_tsdf_trace* tr, const int64_t g[3], float sdf, float uw) {
  if (tr->n == tr->cap) {
    tr->cap = tr->cap ? 2 * tr->cap : 4096;
    tr->g = (int64_t*)realloc(tr->g, sizeof(int64_t) * 3 * (size_t)tr->cap);
    tr->sdf = (float*)realloc(tr->sdf, sizeof(float) * (size_t)tr->cap);
    tr->uw = (float*)realloc(tr->uw, sizeof(float) * (size_t)tr->cap);
  }
  tr->g[3 * tr->n] = g[0]; tr->g[3 * tr->n + 1] = g[1]; tr->g[3 * tr->n + 2] = g[2];
  tr->sdf[tr->n] = sdf; tr->uw[tr->n] = uw;
  tr->n++;
}

void vgo_tsdf_trace_free(vgo_tsdf_trace* tr) {
  free(tr->g); free(tr->sdf); free(tr->uw);
  memset(tr, 0, sizeof(*tr));
}

/* A point with a non-finite coordinate is invalid (voxblox leaves it undefined: its ray direction
 * is NaN, and the Fast start key casts a non-finite float to an integer). */
static inline int point_finite(const float* p) {
  return isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]);
}

/* (int64_t)floorf(v), saturating at the int64 range and NaN -> 0 as the device's float -> integer
 * conversion does (a finite point whose start key overflows, e.g. a huge "no return" coordinate). */
static inline int64_t floor_to_i64(float v) {
  const float f = floorf(v);
  if (f != f) return 0;
  if (f >= 9223372036854775808.0f) return INT64_MAX;
  if (f < -9223372036854775808.0f) return INT64_MIN;
  return (int64_t)f;
}

/* updateTsdfVoxel + computeDistance (tsdf_integrator.cc) */
static void update_tsdf_voxel(const vgo_layer* l, const vgo_tsdf_config* c, const float origin[3],
                              const float pG[3], const int64_t g[3], float weight, float* vd,
                              float* vw, vgo_tsdf_trace* tr) {
  const float vs = l->voxel_size;
  /* getCenterPointFromGridIndex(global_idx, voxel_size) */
  float centre[3] = {((float)g[0] + 0.5f) * vs, ((float)g[1] + 0.5f) * vs,
                     ((float)g[2] + 0.5f) * vs};
  float vvo[3] = {centre[0] - origin[0], centre[1] - origin[1], centre[2] - origin[2]};
  float vpo[3] = {pG[0] - origin[0], pG[1] - origin[1], pG[2] - origin[2]};
  float dist_G = sqrtf(vpo[0] * vpo[0] + vpo[1] * vpo[1] + vpo[2] * vpo[2]);
  float dot = vvo[0] * vpo[0] + vvo[1] * vpo[1] + vvo[2] * vpo[2];
  float dist_G_V = dot / dist_G;
  float sdf = dist_G - dist_G_V;
  float uw = weight;
  const float trunc = c->default_truncation_distance;
  const float dropoff_eps = vs;
  if (c->use_weight_dropoff && sdf < -dropoff_eps) {
    uw = weight * (trunc + sdf) / (trunc - dropoff_eps);
    uw = uw > 0.0f ? uw : 0.0f;
  }
  if (c->use_sparsity_compensation_factor) {
    if (fabsf(sdf) < trunc) uw *= c->sparsity_compensation_factor;
  }
  if (tr) trace_push(tr, g, sdf, uw);
  const float new_weight = *vw + uw;
  if (new_weight < VGO_FLOAT_EPS) return;
  const float new_sdf = (sdf * uw + *vd * *vw) / new_weight;
  /* std::min(a, b) = (b < a) ? b : a, std::max(a, b) = (a < b) ? b : a: a NaN new_sdf (a point at
   * the sensor origin, 0/0 in computeDistance) clamps to -trunc */
  *vd = (new_sdf > 0.0f) ? (new_sdf < trunc ? new_sdf : trunc)
                         : (-trunc < new_sdf ? new_sdf : -trunc);
  *vw = new_weight < c->max_weight ? new_weight : c->max_weight;
}

static void tsdf_integrate(vgo_layer* l, const vgo_tsdf_config* c, const float T_G_C[7], int n,
                           const float* pts, vgo_tsdf_stats* st, vgo_tsdf_trace* tr) {
  vgo_tsdf_stats S;
  memset(&S, 0, sizeof(S));
  const int blocks_before = l->n_blocks;
  const float origin[3] = {T_G_C[4], T_G_C[5], T_G_C[6]};
  /* FastTsdfIntegrator approximate sets: 2^20 slots, cleared every scan */
  const uint64_t mask = ((uint64_t)1 << 20) - 1;
  uint64_t* start_set = NULL;
  uint64_t* obs_set = NULL;
  if (c->mode == 1) {
    start_set = (uint64_t*)malloc(sizeof(uint64_t) * (mask + 1));
    obs_set = (uint64_t*)malloc(sizeof(uint64_t) * (mask + 1));
    /* "empty" marker ~0, as on the device.  It is a real hash: index (-1, 0, 0) (and (17190, -1, 0))
     * hashes to ~0, so the first visit of that voxel counts as a collision and a point whose start
     * cell is (-1, 0, 0) is never cast (tests/fast_schedule.py) */
    for (uint64_t i = 0; i <= mask; ++i) { start_set[i] = ~(uint64_t)0; obs_set[i] = ~(uint64_t)0; }
  }
  for (int i = 0; i < n; ++i) {
    const float* pC = pts + 3 * (size_t)i;
    if (!point_finite(pC)) continue;
    /* isPointValid */
    const float ray_distance = sqrtf(pC[0] * pC[0] + pC[1] * pC[1] + pC[2] * pC[2]);
    int is_clearing = 0;
    if (ray_distance < c->min_ray_length_m) continue;
    else if (ray_distance > c->max_ray_length_m) {
      if (c->allow_clear) is_clearing = 1;
      else continue;
    }
    S.rays_valid++;
    float pG[3];
    vgo_T_transform(T_G_C, pC, pG);
    if (c->mode == 1) {
      float inv = c->start_voxel_subsampling_factor * l->voxel_size_inv;
      int64_t k[3] = {floor_to_i64(pG[0] * inv + VGO_COORD_EPS),
                      floor_to_i64(pG[1] * inv + VGO_COORD_EPS),
                      floor_to_i64(pG[2] * inv + VGO_COORD_EPS)};
      uint64_t h = any_index_hash(k[0], k[1], k[2]);
      if (start_set[h & mask] == h) continue;
      start_set[h & mask] = h;
    }
    S.rays_cast++;
    raycaster rc;
    raycaster_init(&rc, origin, pG, is_clearing, c->voxel_carving_enabled, c->max_ray_length_m,
                   l->voxel_size_inv, c->default_truncation_distance, c->mode == 1 ? 0 : 1);
    /* getVoxelWeight */
    float weight;
    if (c->use_const_weight) weight = 1.0f;
    else {
      float dz = fabsf(pC[2]);
      weight = dz > VGO_FLOAT_EPS ? 1.0f / (dz * dz) : 0.0f;
    }
    int64_t g[3];
    int64_t collisions = 0;
    while (raycaster_next(&rc, g)) {
      if (c->mode == 1) {
        uint64_t h = any_index_hash(g[0], g[1], g[2]);
        if (obs_set[h & mask] == h) ++collisions;
        else { obs_set[h & mask] = h; collisions = 0; }
        if (collisions > c->max_consecutive_ray_collisions) break;
      }
      /* allocateStorageAndGetVoxelPtr */
      int32_t b[3], loc[3];
      vgo_block_and_local_from_global(g, l->vps, b, loc);
      int slot = vgo_layer_find_block(l, b);
      if (slot < 0) slot = vgo_layer_add_block(l, b, NULL, NULL);
      const size_t o = (size_t)slot * l->vox_per_block + loc[0] + l->vps * (loc[1] + l->vps * loc[2]);
      update_tsdf_voxel(l, c, origin, pG, g, weight, l->distance + o, l->weight + o, tr);
      S.voxel_updates++;
    }
  }
  S.blocks_allocated = l->n_blocks - blocks_before;
  free(start_set); free(obs_set);
  if (st) *st = S;
}

void vgo_tsdf_integrate(vgo_layer* l, const vgo_tsdf_config* c, const float T_G_C[7], int n,
                        const float* pts, vgo_tsdf_stats* st) {
  tsdf_integrate(l, c, T_G_C, n, pts, st, NULL);
}

void vgo_tsdf_integrate_trace(vgo_layer* l, const vgo_tsdf_config* c, const float T_G_C[7], int n,
                              const float* pts, vgo_tsdf_stats* st, vgo_tsdf_trace* tr) {
  tsdf_integrate(l, c, T_G_C, n, pts, st, tr);
}


/* ========================================================================= */
/* Multi-threaded integrator (timing baseline)                               */
/* ========================================================================= */
#define VGO_MT_LOCKS 65536
typedef struct {
  vgo_layer* l;
  const vgo_tsdf_config* c;
  const float* T;
  const float* pts;
  int n, nt;
  atomic_int next_id;
  pthread_mutex_t alloc_mu;
  atomic_flag* locks;
  _Atomic uint64_t* start_set;
  _Atomic uint64_t* obs_set;
  _Atomic int64_t rays_valid, rays_cast, voxel_updates;
} tsdf_mt_job;

/* capacity for `extra` more blocks without any reallocation; the new bricks are zeroed up front */
static void layer_reserve(vgo_layer* l, int extra) {
  if (l->cap_blocks - l->n_blocks >= extra / 2 && l->mt_zeroed_from <= l->n_blocks && l->mt_zeroed_to >= l->cap_blocks)
    return;  /* enough zeroed spare bricks from an earlier call */
  const int need = l->n_blocks + extra;
  if (need > l->cap_blocks) {
    l->idx = (int32_t*)realloc(l->idx, sizeof(int32_t) * 3 * (size_t)need);
    l->distance = (float*)realloc(l->distance, sizeof(float) * (size_t)l->vox_per_block * need);
    l->weight = (float*)realloc(l->weight, sizeof(float) * (size_t)l->vox_per_block * need);
    l->cap_blocks = need;
  }
  memset(l->distance + (size_t)l->n_blocks * l->vox_per_block, 0,
         sizeof(float) * (size_t)l->vox_per_block * (l->cap_blocks - l->n_blocks));
  memset(l->weight + (size_t)l->n_blocks * l->vox_per_block, 0,
         sizeof(float) * (size_t)l->vox_per_block * (l->cap_blocks - l->n_blocks));
  l->mt_zeroed_from = l->n_blocks;
  l->mt_zeroed_to = l->cap_blocks;
  uint32_t ts = l->table_size;
  while ((uint32_t)l->cap_blocks * 2 > ts) ts *= 2;
  if (ts != l->table_size) {
    l->table_size = ts;
    l->table = (int32_t*)realloc(l->table, sizeof(int32_t) * ts);
    for (uint32_t i = 0; i < ts; ++i) l->table[i] = -1;
    for (int i = 0; i < l->n_blocks; ++i) layer_table_insert(l, i);
  }
}

static int layer_get_or_add_mt(tsdf_mt_job* J, const int32_t b[3]) {
  vgo_layer* l = J->l;
  int slot = vgo_layer_find_block(l, b);
  if (slot >= 0) return slot;
  pthread_mutex_lock(&J->alloc_mu);
  slot = vgo_layer_find_block(l, b);
  if (slot < 0 && l->n_blocks < l->cap_blocks) {
    slot = l->n_blocks;
    l->idx[3 * slot] = b[0]; l->idx[3 * slot + 1] = b[1]; l->idx[3 * slot + 2] = b[2];
    atomic_thread_fence(memory_order_release);
    l->n_blocks = slot + 1;
    layer_table_insert(l, slot);   /* the brick was zeroed by layer_reserve */
  }
  pthread_mutex_unlock(&J->alloc_mu);
  return slot;
}

static void* tsdf_mt_worker(void* arg) {
  tsdf_mt_job* J = (tsdf_mt_job*)arg;
  vgo_layer* l = J->l;
  const vgo_tsdf_config* c = J->c;
  const int id = atomic_fetch_add(&J->next_id, 1);
  const float origin[3] = {J->T[4], J->T[5], J->T[6]};
  const uint64_t mask = ((uint64_t)1 << 20) - 1;
  int64_t n_valid = 0, n_cast = 0, n_upd = 0;
  for (int i = id; i < J->n; i += J->nt) {
    const float* pC = J->pts + 3 * (size_t)i;
    if (!point_finite(pC)) continue;
    const float ray_distance = sqrtf(pC[0] * pC[0] + pC[1] * pC[1] + pC[2] * pC[2]);
    int is_clearing = 0;
    if (ray_distance < c->min_ray_length_m) continue;
    else if (ray_distance > c->max_ray_length_m) {
      if (c->allow_clear) is_clearing = 1;
      else continue;
    }
    n_valid++;
    float pG[3];
    vgo_T_transform(J->T, pC, pG);
    if (c->mode == 1) {
      float inv = c->start_voxel_subsampling_factor * l->voxel_size_inv;
      int64_t k[3] = {floor_to_i64(pG[0] * inv + VGO_COORD_EPS),
                      floor_to_i64(pG[1] * inv + VGO_COORD_EPS),
                      floor_to_i64(pG[2] * inv + VGO_COORD_EPS)};
      uint64_t h = any_index_hash(k[0], k[1], k[2]);
      if (atomic_exchange(&J->start_set[h & mask], h) == h) continue;
    }
    n_cast++;
    raycaster rc;
    raycaster_init(&rc, origin, pG, is_clearing, c->voxel_carving_enabled, c->max_ray_length_m,
                   l->voxel_size_inv, c->default_truncation_distance, c->mode == 1 ? 0 : 1);
    float weight;
    if (c->use_const_weight) weight = 1.0f;
    else {
      float dz = fabsf(pC[2]);
      weight = dz > VGO_FLOAT_EPS ? 1.0f / (dz * dz) : 0.0f;
    }
    int64_t g[3];
    int64_t collisions = 0;
    int32_t lb[3] = {INT32_MIN, 0, 0};
    int slot = -1;
    while (raycaster_next(&rc, g)) {
      if (c->mode == 1) {
        uint64_t h = any_index_hash(g[0], g[1], g[2]);
        if (atomic_exchange(&J->obs_set[h & mask], h) == h) ++collisions;
        else collisions = 0;
        if (collisions > c->max_consecutive_ray_collisions) break;
      }
      int32_t b[3], loc[3];
      vgo_block_and_local_from_global(g, l->vps, b, loc);
      if (b[0] != lb[0] || b[1] != lb[1] || b[2] != lb[2]) {
        slot = layer_get_or_add_mt(J, b);
        lb[0] = b[0]; lb[1] = b[1]; lb[2] = b[2];
      }
      if (slot < 0) continue;
      const size_t o = (size_t)slot * l->vox_per_block + loc[0] + l->vps * (loc[1] + l->vps * loc[2]);
      atomic_flag* lk = &J->locks[(o * 0x9E3779B1u) & (VGO_MT_LOCKS - 1)];
      while (atomic_flag_test_and_set_explicit(lk, memory_order_acquire)) { }
      update_tsdf_voxel(l, c, origin, pG, g, weight, l->distance + o, l->weight + o, NULL);
      atomic_flag_clear_explicit(lk, memory_order_release);
      n_upd++;
    }
  }
  atomic_fetch_add(&J->rays_valid, n_valid);
  atomic_fetch_add(&J->rays_cast, n_cast);
  atomic_fetch_add(&J->voxel_updates, n_upd);
  return NULL;
}

void vgo_tsdf_integrate_mt(vgo_layer* l, const vgo_tsdf_config* c, const float T_G_C[7], int n,
                           const float* pts, int num_threads, vgo_tsdf_stats* st) {
  tsdf_mt_job J;
  memset(&J, 0, sizeof(J));
  const int nt = num_threads > 1 ? num_threads : 1;
  const int blocks_before = l->n_blocks;
  layer_reserve(l, 4096);
  J.l = l; J.c = c; J.T = T_G_C; J.pts = pts; J.n = n; J.nt = nt;
  atomic_init(&J.next_id, 0);
  pthread_mutex_init(&J.alloc_mu, NULL);
  J.locks = (atomic_flag*)calloc(VGO_MT_LOCKS, sizeof(atomic_flag));
  if (c->mode == 1) {
    const size_t m = (size_t)1 << 20;
    J.start_set = (_Atomic uint64_t*)malloc(sizeof(uint64_t) * m);
    J.obs_set = (_Atomic uint64_t*)malloc(sizeof(uint64_t) * m);
    for (size_t i = 0; i < m; ++i) { atomic_init(&J.start_set[i], ~(uint64_t)0); atomic_init(&J.obs_set[i], ~(uint64_t)0); }
  }
  if (nt <= 1) tsdf_mt_worker(&J);
  else pool_run(nt, tsdf_mt_worker, &J);
  vgo_tsdf_stats S;
  memset(&S, 0, sizeof(S));
  S.rays_valid = J.rays_valid; S.rays_cast = J.rays_cast; S.voxel_updates = J.voxel_updates;
  S.blocks_allocated = l->n_blocks - blocks_before;
  free(J.locks); free((void*)J.start_set); free((void*)J.obs_set);
  pthread_mutex_destroy(&J.alloc_mu);
  if (st) *st = S;
}
