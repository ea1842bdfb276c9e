// C++ host-side mirror of the reference's interface for the two hot paths, header only, on top
// of the C-ABI (include/voxgraph_b200.h).  Same names, argument meaning and CHECK behaviour
// (as exceptions) as:
//   voxgraph::PoseGraph                    include/voxgraph/backend/pose_graph.h:15-65
//   voxgraph::SubmapNode::Config           include/voxgraph/backend/node/{node,submap_node}.h
//   voxgraph::RelativePoseConstraint::Config / RegistrationConstraint::Config
//                                          include/voxgraph/backend/constraint/*.h
//   voxgraph::PointcloudIntegrator         include/voxgraph/frontend/measurement_processors/pointcloud_integrator.h
// Poses are the reference's 4-DoF optimisation vectors [x, y, z, yaw] (pose_4d.cpp:4-11); Eigen /
// minkindr types are not available in this image, so plain arrays stand in for them.
#pragma once

#include <algorithm>
#include <array>
#include <cstdint>
#include <fstream>
#include <iterator>
#include <map>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "voxgraph_b200.h"

namespace voxgraph_b200 {

using SubmapID = uint32_t;                       // cblox::SubmapID
using Pose4 = std::array<double, 4>;             // x, y, z, yaw
using InformationMatrix = std::array<double, 16>;  // row-major 4x4 (Constraint::InformationMatrix)

inline InformationMatrix IdentityInformation() {
  InformationMatrix m{};
  for (int i = 0; i < 4; ++i) m[5 * i] = 1.0;
  return m;
}

class Error : public std::runtime_error {
 public:
  Error(int code, const std::string& what) : std::runtime_error(what), code_(code) {}
  int code() const { return code_; }
 private:
  int code_;
};

// One GPU's brick store + pose-graph state.
class Context {
 public:
  explicit Context(int device = 0) {
    const int rc = vgx_ctx_create(device, &ctx_);
    if (rc != VGX_OK) throw Error(rc, "vgx_ctx_create failed: a CUDA device is required (no CPU fallback)");
  }
  ~Context() { vgx_ctx_destroy(ctx_); }
  Context(const Context&) = delete;
  Context& operator=(const Context&) = delete;
  vgx_ctx* get() const { return ctx_; }
  void check(int rc) const {
    if (rc < 0) throw Error(rc, vgx_last_error(ctx_));
  }

  // voxblox::Layer upload (finished submap) + its WeightedSampler<RegistrationPoint> items
  void uploadSubmap(SubmapID id, float voxel_size, int vps, int n_blocks, const int32_t* block_idx,
                    const float* distance, const float* weight) {
    check(vgx_submap_upload(ctx_, id, voxel_size, vps, n_blocks, block_idx, distance, weight));
  }
  void uploadRegistrationPoints(SubmapID id, int point_type, int n, const float* xyz, const float* distance,
                                const float* weight) {
    check(vgx_submap_upload_points(ctx_, id, point_type, n, xyz, distance, weight));
  }

 private:
  vgx_ctx* ctx_ = nullptr;
};

// RegistrationCostFunction (registration_cost_function.h:11-82): drop-in Evaluate.
class RegistrationCostFunction {
 public:
  struct Config {  // h:17-41
    int registration_point_type = VGX_POINTS_ISOSURFACE;
    float sampling_ratio = -1;
    double no_correspondence_cost = 0;
    bool use_esdf_distance = false;  // h:35 (reference default true): needs Context-side generateEsdf
  };
  RegistrationCostFunction(const Context& ctx, SubmapID reference, SubmapID reading, const Config& config)
      : ctx_(ctx), reference_(reference), reading_(reading) {
    vgx_reg_config_default(&cfg_);
    cfg_.registration_point_type = config.registration_point_type;
    cfg_.sampling_ratio = config.sampling_ratio;
    cfg_.no_correspondence_cost = config.no_correspondence_cost;
    cfg_.use_esdf_distance = config.use_esdf_distance ? 1 : 0;
    ctx_.check(vgx_reg_num_residuals(ctx_.get(), reference_, &cfg_, &num_residuals_));
  }
  int num_residuals() const { return num_residuals_; }
  // bool Evaluate(double const* const* parameters, double* residuals, double** jacobians) const
  bool Evaluate(double const* const* parameters, double* residuals, double** jacobians) const {
    const int rc = vgx_reg_eval_emit(ctx_.get(), reference_, reading_, &cfg_, parameters[0], parameters[1],
                                     residuals, jacobians ? jacobians[0] : nullptr,
                                     jacobians ? jacobians[1] : nullptr);
    ctx_.check(rc);
    return rc == VGX_OK;  // VGX_ZERO_WEIGHT -> false (registration_cost_function.cpp:273)
  }

 private:
  const Context& ctx_;
  SubmapID reference_, reading_;
  vgx_reg_config cfg_;
  int num_residuals_ = 0;
};

struct SubmapNodeConfig {  // SubmapNode::Config
  bool set_constant = false;
  Pose4 T_mission_node_initial{};
  SubmapID submap_id = 0;
};
struct RelativePoseConstraintConfig {  // RelativePoseConstraint::Config
  InformationMatrix information_matrix = IdentityInformation();
  SubmapID origin_submap_id = 0, destination_submap_id = 0;
  Pose4 T_origin_destination{};  // [t, yaw]
};
struct ReferenceFrameNodeConfig {  // ReferenceFrameNode::Config
  bool set_constant = true;
  Pose4 T_mission_node_initial{};
  uint32_t reference_frame_id = 0;
};
struct AbsolutePoseConstraintConfig {  // AbsolutePoseConstraint::Config
  InformationMatrix information_matrix = IdentityInformation();
  bool allow_semi_definite_information_matrix = false;
  uint32_t reference_frame_id = 0;
  SubmapID submap_id = 0;
  Pose4 T_ref_submap{};  // [t, yaw]
};
// reference-frame nodes share the C-ABI's uint32 node id space
constexpr uint32_t kFrameNodeIdBase = 0x80000000u;

// Constraint ctor (constraint.cpp:4-38): LLT lower factor, or Eigen's pivoted LDLT
// (sqrt = P^T L sqrt(D) P) when semi-definite matrices are allowed (vgx_sqrt_information). Throws like the CHECKs.
inline std::array<double, 16> SqrtInformation(const InformationMatrix& info, bool allow_semi_definite) {
  std::array<double, 16> S{};
  if (vgx_sqrt_information(info.data(), allow_semi_definite ? 1 : 0, S.data()) != VGX_OK)
    throw std::invalid_argument(allow_semi_definite ? "The information matrix must be positive semi-definite"
                                                    : "The square root of the information matrix could not be "
                                                      "computed, make sure it is symmetric and positive definite");
  return S;
}

struct RegistrationConstraintConfig {  // RegistrationConstraint::Config
  InformationMatrix information_matrix = IdentityInformation();
  SubmapID first_submap_id = 0, second_submap_id = 0;
  RegistrationCostFunction::Config registration;
};
struct SolverSummary {  // what voxgraph reads off ceres::Solver::Summary
  int iterations = 0, num_successful_steps = 0, termination = 0;
  double initial_cost = 0, final_cost = 0, total_time_in_seconds = 0;
};

class PoseGraph {
 public:
  typedef std::map<const SubmapID, const Pose4> PoseMap;
  explicit PoseGraph(Context& ctx) : ctx_(ctx) { vgx_solver_options_default(&options_); }

  void addSubmapNode(const SubmapNodeConfig& config) {
    nodes_[config.submap_id] = config;
    dirty_ = true;
  }
  bool hasSubmapNode(SubmapID id) const { return nodes_.count(id) != 0; }

  void addRelativePoseConstraint(const RelativePoseConstraintConfig& config) {
    // Constraint ctor (constraint.cpp:8-14): sqrt_information = LLT lower factor
    relative_.push_back({config, SqrtInformation(config.information_matrix, false)});
    dirty_ = true;
  }

  void addReferenceFrameNode(const ReferenceFrameNodeConfig& config) {  // pose_graph.cpp:21-24
    SubmapNodeConfig n;
    n.submap_id = kFrameNodeIdBase + config.reference_frame_id;
    n.set_constant = config.set_constant;
    n.T_mission_node_initial = config.T_mission_node_initial;
    nodes_[n.submap_id] = n;
    dirty_ = true;
  }
  bool hasReferenceFrameNode(uint32_t frame_id) const { return nodes_.count(kFrameNodeIdBase + frame_id) != 0; }

  // pose_graph.cpp:33-39 + absolute_pose_constraint.cpp:6-35 (height / GPS measurements)
  void addAbsolutePoseConstraint(const AbsolutePoseConstraintConfig& config) {
    if (!hasReferenceFrameNode(config.reference_frame_id))
      throw std::invalid_argument("Graph contains no reference frame node " + std::to_string(config.reference_frame_id));
    if (!hasSubmapNode(config.submap_id))
      throw std::invalid_argument("Graph contains no node for submap " + std::to_string(config.submap_id));
    RelativePoseConstraintConfig r;
    r.information_matrix = config.information_matrix;
    r.origin_submap_id = kFrameNodeIdBase + config.reference_frame_id;
    r.destination_submap_id = config.submap_id;
    r.T_origin_destination = config.T_ref_submap;
    relative_.push_back({r, SqrtInformation(config.information_matrix, config.allow_semi_definite_information_matrix)});
    dirty_ = true;
  }

  void addRegistrationConstraint(const RegistrationConstraintConfig& config) {
    if (config.first_submap_id == config.second_submap_id)  // pose_graph.cpp:50-51
      throw std::invalid_argument("Cannot constrain submap " + std::to_string(config.first_submap_id) + " to itself");
    for (SubmapID id : {config.first_submap_id, config.second_submap_id})  // pose_graph.cpp:54-57
      if (!hasSubmapNode(id)) throw std::invalid_argument("Graph contains no node for submap " + std::to_string(id));
    if (config.information_matrix != IdentityInformation())  // registration_constraint.h:32-34
      throw std::invalid_argument("Registration constraint information matrices that differ from the identity "
                                  "matrix are not yet supported.");
    // the reference keeps one Config per constraint (registration_constraint.h:15-21)
    registration_.emplace_back(config.first_submap_id, config.second_submap_id);
    registration_cfgs_.push_back(config.registration);
    if (config.registration.registration_point_type == VGX_POINTS_ISOSURFACE) {  // pose_graph.cpp:63-71
      registration_.emplace_back(config.second_submap_id, config.first_submap_id);
      registration_cfgs_.push_back(config.registration);
    }
    dirty_ = true;
  }
  void resetRegistrationConstraints() {
    registration_.clear();
    registration_cfgs_.clear();
    dirty_ = true;
  }

  void optimize(bool exclude_registration_constraints = false) {  // pose_graph.cpp:85-106
    sync();
    options_.exclude_registration = exclude_registration_constraints ? 1 : 0;
    std::vector<double> x(4 * nodes_.size());
    vgx_solver_summary s;
    ctx_.check(vgx_graph_solve(ctx_.get(), &options_, x.data(), &s));
    size_t k = 0;
    for (auto& kv : nodes_) {
      for (int c = 0; c < 4; ++c) kv.second.T_mission_node_initial[c] = x[4 * k + c];
      ++k;
    }
    SolverSummary out;
    out.iterations = s.iterations; out.num_successful_steps = s.num_successful_steps;
    out.termination = s.termination; out.initial_cost = s.initial_cost; out.final_cost = s.final_cost;
    out.total_time_in_seconds = s.total_time_s;
    solver_summaries_.push_back(out);
  }

  PoseMap getSubmapPoses() const {
    PoseMap m;
    for (const auto& kv : nodes_)
      if (kv.first < kFrameNodeIdBase) m.emplace(kv.first, kv.second.T_mission_node_initial);
    return m;
  }
  const std::vector<SolverSummary>& getSolverSummaries() const { return solver_summaries_; }
  vgx_solver_options& solverOptions() { return options_; }

  // pose_graph.cpp:117-163: the keys of the map are the submap pairs whose 4 x 4 covariance blocks are
  // wanted; false where ceres::Covariance::Compute would fail (rank-deficient Jacobian)
  typedef std::pair<SubmapID, SubmapID> SubmapIdPair;
  typedef std::array<double, 16> EdgeCovarianceMatrix;   // row-major, rows = parameters of the first submap
  typedef std::map<SubmapIdPair, EdgeCovarianceMatrix> EdgeCovarianceMap;
  bool getEdgeCovarianceMap(EdgeCovarianceMap* edge_covariance_map) {
    if (!edge_covariance_map) throw std::invalid_argument("edge_covariance_map is null");   // CHECK_NOTNULL
    sync();
    std::vector<uint32_t> first, second;
    for (const auto& kv : *edge_covariance_map) {
      for (SubmapID id : {kv.first.first, kv.first.second})
        if (!hasSubmapNode(id)) throw std::invalid_argument("Graph contains no node for submap " + std::to_string(id));
      first.push_back(kv.first.first);
      second.push_back(kv.first.second);
    }
    std::vector<double> cov(16 * first.size());
    const int rc = vgx_graph_edge_covariances(ctx_.get(), (int)first.size(), first.data(), second.data(), cov.data());
    if (rc == VGX_ERR_INVALID) return false;
    ctx_.check(rc);
    size_t k = 0;
    for (auto& kv : *edge_covariance_map) {
      for (int e = 0; e < 16; ++e) kv.second[e] = cov[16 * k + e];
      ++k;
    }
    return true;
  }
  // per-edge summed squared residual (getVisualizationEdges, pose_graph.cpp:194-207)
  std::vector<double> getRegistrationEdgeResiduals() {
    sync();
    std::vector<double> r(registration_.size());
    if (!r.empty()) ctx_.check(vgx_graph_registration_costs(ctx_.get(), r.data()));
    return r;
  }

 private:
  void sync() {
    if (!dirty_) return;
    std::vector<uint32_t> ids; std::vector<double> x; std::vector<uint8_t> cst;
    for (const auto& kv : nodes_) {
      ids.push_back(kv.first);
      x.insert(x.end(), kv.second.T_mission_node_initial.begin(), kv.second.T_mission_node_initial.end());
      cst.push_back(kv.second.set_constant ? 1 : 0);
    }
    ctx_.check(vgx_graph_set_nodes(ctx_.get(), (int)ids.size(), ids.data(), x.data(), cst.data()));
    std::vector<uint32_t> a, b; std::vector<double> t, L;
    for (const auto& r : relative_) {
      a.push_back(r.first.origin_submap_id); b.push_back(r.first.destination_submap_id);
      t.insert(t.end(), r.first.T_origin_destination.begin(), r.first.T_origin_destination.end());
      L.insert(L.end(), r.second.begin(), r.second.end());
    }
    ctx_.check(vgx_graph_set_relative_edges(ctx_.get(), (int)a.size(), a.data(), b.data(), t.data(), L.data()));
    std::vector<uint32_t> ra, rb;
    for (const auto& r : registration_) { ra.push_back(r.first); rb.push_back(r.second); }
    std::vector<vgx_reg_config> rcs(registration_cfgs_.size());
    for (size_t k = 0; k < rcs.size(); ++k) {
      vgx_reg_config_default(&rcs[k]);
      rcs[k].registration_point_type = registration_cfgs_[k].registration_point_type;
      rcs[k].sampling_ratio = registration_cfgs_[k].sampling_ratio;
      rcs[k].no_correspondence_cost = registration_cfgs_[k].no_correspondence_cost;
      rcs[k].use_esdf_distance = registration_cfgs_[k].use_esdf_distance ? 1 : 0;
    }
    ctx_.check(vgx_graph_set_registration_constraints_v(ctx_.get(), (int)ra.size(), ra.data(), rb.data(),
                                                        rcs.data()));
    dirty_ = false;
  }

  Context& ctx_;
  std::map<SubmapID, SubmapNodeConfig> nodes_;
  std::vector<std::pair<RelativePoseConstraintConfig, std::array<double, 16>>> relative_;
  std::vector<std::pair<SubmapID, SubmapID>> registration_;
  std::vector<RegistrationCostFunction::Config> registration_cfgs_;
  vgx_solver_options options_;
  std::vector<SolverSummary> solver_summaries_;
  bool dirty_ = true;
};

// PoseGraphInterface::updateOverlappingSubmapList (pose_graph_interface.cpp:109-147) over
// VoxgraphSubmap::overlapsWith (voxgraph_submap.cpp:245-278).  poses: T_mission_submap as
// [qw qx qy qz tx ty tz] per submap (float, as cblox stores them).
inline std::vector<std::pair<SubmapID, SubmapID>> findOverlappingSubmaps(
    Context& ctx, const std::vector<SubmapID>& ids, const std::vector<std::array<float, 7>>& poses) {
  if (ids.size() != poses.size()) throw std::invalid_argument("findOverlappingSubmaps: one pose per submap");
  const int n = (int)ids.size();
  const int cap = std::max(1, n * (n - 1) / 2);
  std::vector<uint32_t> out(2 * (size_t)cap);
  int np = 0;
  ctx.check(vgx_find_overlapping_pairs(ctx.get(), n, ids.data(), n ? poses[0].data() : nullptr, cap, out.data(), &np));
  std::vector<std::pair<SubmapID, SubmapID>> pairs;
  for (int k = 0; k < np; ++k) pairs.emplace_back(out[2 * k], out[2 * k + 1]);
  return pairs;
}

// cblox::io::LoadSubmapCollection: creates the file's submaps (TSDF only; finish them with
// PointcloudIntegrator::finishSubmap as VoxgraphSubmap::LoadFromStream's caller does) and returns
// their ids and poses T_M_S [qw qx qy qz tx ty tz].  All or nothing; throws Error on failure.
inline void LoadSubmapCollection(Context& ctx, const std::string& path, std::vector<SubmapID>* ids,
                                 std::vector<std::array<float, 7>>* poses) {
  std::ifstream f(path, std::ios::binary);
  if (!f) throw Error(VGX_ERR_INVALID, "LoadSubmapCollection: cannot open " + path);
  const std::vector<uint8_t> data((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
  int n = 0;
  int rc = vgx_collection_scan(data.data(), data.size(), 0, nullptr, &n);
  if (rc != VGX_OK && rc != VGX_ERR_CAPACITY) throw Error(rc, "LoadSubmapCollection: malformed stream " + path);
  std::vector<vgx_collection_entry> entries((size_t)n);
  if (n > 0) {
    rc = vgx_collection_scan(data.data(), data.size(), n, entries.data(), &n);
    if (rc != VGX_OK) throw Error(rc, "LoadSubmapCollection: malformed stream " + path);
  }
  ctx.check(vgx_collection_load(ctx.get(), data.data(), data.size(), &n));
  if (ids) ids->clear();
  if (poses) poses->clear();
  for (const vgx_collection_entry& e : entries) {
    if (ids) ids->push_back(e.id);
    if (poses) {
      std::array<float, 7> T;
      std::copy(e.T_M_S, e.T_M_S + 7, T.begin());
      poses->push_back(T);
    }
  }
}

// cblox::SubmapCollection::saveToFile: the submaps with their poses T_M_S, in increasing id order.
inline void SaveSubmapCollection(Context& ctx, const std::string& path, const std::vector<SubmapID>& ids,
                                 const std::vector<std::array<float, 7>>& poses) {
  if (ids.size() != poses.size()) throw std::invalid_argument("SaveSubmapCollection: one pose per submap");
  const int n = (int)ids.size();
  const float* T = n ? poses[0].data() : nullptr;
  uint64_t size = 0;
  ctx.check(vgx_collection_save(ctx.get(), n, ids.data(), T, nullptr, 0, &size));
  std::vector<uint8_t> data(size);
  ctx.check(vgx_collection_save(ctx.get(), n, ids.data(), T, data.data(), size, &size));
  std::ofstream f(path, std::ios::binary);
  f.write(reinterpret_cast<const char*>(data.data()), (std::streamsize)size);
  if (!f) throw Error(VGX_ERR_INVALID, "SaveSubmapCollection: cannot write " + path);
}

// voxblox::MeshIntegratorConfig, the part voxgraph sets (voxgraph_mapper.yaml:52-53; mesh_use_color is
// false there; vertex colours are computed for submaps with a colour channel and used by vgx_mesh_ply_ex only).
struct MeshIntegratorConfig {
  float min_weight = 2.0f;
  vgx_mesh_config c() const {
    vgx_mesh_config m;
    vgx_mesh_config_default(&m);
    m.min_weight = min_weight;
    return m;
  }
};

// A separated submap mesh on the host: vertices in the mission frame, triangles indexing them, and the
// first vertex / triangle of every submap (n + 1 entries each).
struct SeparatedMesh {
  std::vector<float> xyz;            // n_vertices x 3
  std::vector<uint32_t> triangles;   // n_triangles x 3
  std::vector<int64_t> vertex_offsets, triangle_offsets;
};

// cblox::SubmapMesher::generateSeparatedMesh on the device: the submaps in the given order, each at its
// pose T_M_S [qw qx qy qz tx ty tz] (poses empty: the submap frames).
inline SeparatedMesh GenerateSeparatedMesh(Context& ctx, const std::vector<SubmapID>& ids,
                                           const std::vector<std::array<float, 7>>& poses,
                                           const MeshIntegratorConfig& config = MeshIntegratorConfig()) {
  if (!poses.empty() && ids.size() != poses.size())
    throw std::invalid_argument("GenerateSeparatedMesh: one pose per submap");
  const int n = (int)ids.size();
  const vgx_mesh_config cfg = config.c();
  SeparatedMesh m;
  m.vertex_offsets.resize((size_t)n + 1);
  m.triangle_offsets.resize((size_t)n + 1);
  ctx.check(vgx_mesh_build(ctx.get(), n, ids.data(), poses.empty() ? nullptr : poses[0].data(), &cfg,
                           m.vertex_offsets.data(), m.triangle_offsets.data()));
  int64_t nv = 0, nt = 0;
  ctx.check(vgx_mesh_download(ctx.get(), 0, nullptr, 0, nullptr, &nv, &nt));
  m.xyz.resize(3 * (size_t)nv);
  m.triangles.resize(3 * (size_t)nt);
  ctx.check(vgx_mesh_download(ctx.get(), nv, m.xyz.data(), nt, m.triangles.data(), &nv, &nt));
  return m;
}

// SubmapVisuals::saveSeparatedMesh: the separated mesh as a binary PLY, one colour per submap (rgba, n x 4;
// empty: voxblox's rainbowColorMap((id mod 20) / 20)).
inline void SaveSeparatedMesh(Context& ctx, const std::string& path, const std::vector<SubmapID>& ids,
                              const std::vector<std::array<float, 7>>& poses,
                              const MeshIntegratorConfig& config = MeshIntegratorConfig(),
                              const std::vector<std::array<uint8_t, 4>>& colours = {}) {
  if (!poses.empty() && ids.size() != poses.size())
    throw std::invalid_argument("SaveSeparatedMesh: one pose per submap");
  if (!colours.empty() && colours.size() != ids.size())
    throw std::invalid_argument("SaveSeparatedMesh: one colour per submap");
  const vgx_mesh_config cfg = config.c();
  ctx.check(vgx_mesh_build(ctx.get(), (int)ids.size(), ids.data(), poses.empty() ? nullptr : poses[0].data(), &cfg,
                           nullptr, nullptr));
  const uint8_t* rgba = colours.empty() ? nullptr : colours[0].data();
  uint64_t size = 0;
  ctx.check(vgx_mesh_ply(ctx.get(), rgba, nullptr, 0, &size));
  std::vector<uint8_t> data(size);
  ctx.check(vgx_mesh_ply(ctx.get(), rgba, data.data(), size, &size));
  std::ofstream f(path, std::ios::binary);
  f.write(reinterpret_cast<const char*>(data.data()), (std::streamsize)size);
  if (!f) throw Error(VGX_ERR_INVALID, "SaveSeparatedMesh: cannot write " + path);
}

// cblox SubmapCollection::getProjectedMap: the submaps merged at their poses T_M_S [qw qx qy qz tx ty tz], in
// increasing id order, into the new finished submap out_id (mission frame).  Returns its block count.
inline int ProjectMap(Context& ctx, const std::vector<SubmapID>& ids, const std::vector<std::array<float, 7>>& poses,
                      SubmapID out_id) {
  if (ids.size() != poses.size()) throw std::invalid_argument("ProjectMap: one pose per submap");
  int n_blocks = 0;
  ctx.check(vgx_project_map(ctx.get(), (int)ids.size(), ids.data(), ids.empty() ? nullptr : poses[0].data(), out_id,
                            &n_blocks));
  return n_blocks;
}

// cblox SubmapMesher::generateCombinedMesh on the device: the mesh of the projected global map.  The mesh is
// left in the context's mesh buffer (vgx_mesh_download / vgx_mesh_ply read it).
inline void BuildCombinedMesh(Context& ctx, const std::vector<SubmapID>& ids,
                              const std::vector<std::array<float, 7>>& poses, const MeshIntegratorConfig& config) {
  if (ids.size() != poses.size()) throw std::invalid_argument("BuildCombinedMesh: one pose per submap");
  const vgx_mesh_config cfg = config.c();
  ctx.check(vgx_mesh_build_combined(ctx.get(), (int)ids.size(), ids.data(), ids.empty() ? nullptr : poses[0].data(),
                                    &cfg));
}

// The combined mesh on the host: vertices in the mission frame and triangles indexing them.
inline SeparatedMesh GenerateCombinedMesh(Context& ctx, const std::vector<SubmapID>& ids,
                                          const std::vector<std::array<float, 7>>& poses,
                                          const MeshIntegratorConfig& config = MeshIntegratorConfig()) {
  BuildCombinedMesh(ctx, ids, poses, config);
  SeparatedMesh m;
  int64_t nv = 0, nt = 0;
  ctx.check(vgx_mesh_download(ctx.get(), 0, nullptr, 0, nullptr, &nv, &nt));
  m.xyz.resize(3 * (size_t)nv);
  m.triangles.resize(3 * (size_t)nt);
  ctx.check(vgx_mesh_download(ctx.get(), nv, m.xyz.data(), nt, m.triangles.data(), &nv, &nt));
  m.vertex_offsets = {0, nv};
  m.triangle_offsets = {0, nt};
  return m;
}

// voxgraph's save_combined_mesh service: the combined mesh as a binary PLY with the voxel colours of the projected
// map where a submap had a colour channel, else in the one colour given (default opaque white).
inline void SaveCombinedMesh(Context& ctx, const std::string& path, const std::vector<SubmapID>& ids,
                             const std::vector<std::array<float, 7>>& poses,
                             const MeshIntegratorConfig& config = MeshIntegratorConfig(),
                             const std::array<uint8_t, 4>& colour = {255, 255, 255, 255}) {
  BuildCombinedMesh(ctx, ids, poses, config);
  uint64_t size = 0;
  ctx.check(vgx_mesh_ply_ex(ctx.get(), colour.data(), 1, nullptr, 0, &size));
  std::vector<uint8_t> data(size);
  ctx.check(vgx_mesh_ply_ex(ctx.get(), colour.data(), 1, data.data(), size, &size));
  std::ofstream f(path, std::ios::binary);
  f.write(reinterpret_cast<const char*>(data.data()), (std::streamsize)size);
  if (!f) throw Error(VGX_ERR_INVALID, "SaveCombinedMesh: cannot write " + path);
}

// voxgraph MapEvaluation (src/tools/evaluation/map_evaluation.cpp) minus the ROS publishers: the constructor
// loads the ground-truth voxblox TSDF layer file into submap gt_id; evaluate() projects the submaps at their
// poses T_M_S, aligns the ground truth to the projection, moves it there (it stays moved, as in the reference)
// and returns voxblox's evaluateLayersRmse details with T_ground_truth__reading.
class MapEvaluation {
 public:
  struct EvaluationDetails {
    vgx_voxel_evaluation_details reconstruction;
    std::array<float, 7> T_ground_truth__reading;
    std::array<double, 4> aligned_pose;
    vgx_solver_summary summary;
  };

  MapEvaluation(Context& ctx, const std::string& ground_truth_tsdf_file_path, SubmapID gt_id)
      : ctx_(ctx), gt_id_(gt_id) {
    std::ifstream f(ground_truth_tsdf_file_path, std::ios::binary);
    if (!f) throw Error(VGX_ERR_INVALID, "MapEvaluation: cannot read " + ground_truth_tsdf_file_path);
    const std::vector<uint8_t> data((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    int n_blocks = 0;
    ctx_.check(vgx_layer_load(ctx_.get(), gt_id_, data.data(), data.size(), &n_blocks));
  }

  EvaluationDetails evaluate(const std::vector<SubmapID>& ids, const std::vector<std::array<float, 7>>& poses) {
    if (ids.size() != poses.size()) throw std::invalid_argument("MapEvaluation::evaluate: one pose per submap");
    vgx_map_evaluation r;
    ctx_.check(vgx_map_evaluate(ctx_.get(), gt_id_, (int)ids.size(), ids.data(),
                                ids.empty() ? nullptr : poses[0].data(), &r));
    EvaluationDetails out;
    out.reconstruction = r.details;
    std::copy(r.T_ground_truth__reading, r.T_ground_truth__reading + 7, out.T_ground_truth__reading.begin());
    std::copy(r.aligned_pose, r.aligned_pose + 4, out.aligned_pose.begin());
    out.summary = r.summary;
    return out;
  }

  SubmapID groundTruthId() const { return gt_id_; }

 private:
  Context& ctx_;
  SubmapID gt_id_;
};

// A sensor_msgs::PointCloud2 without ROS: the members pcl::fromROSMsg reads, the data not owned.
struct PointField {  // sensor_msgs::PointField
  enum : uint8_t { UINT32 = 6, FLOAT32 = 7 };
  std::string name;
  uint32_t offset = 0;
  uint8_t datatype = 0;
  uint32_t count = 1;
};
struct PointCloud2View {
  std::vector<PointField> fields;
  uint32_t width = 0, height = 0, point_step = 0, row_step = 0;
  bool is_bigendian = false;
  const uint8_t* data = nullptr;   // at least height * row_step bytes
  uint64_t size = 0;
};

// The field matching of PointcloudIntegrator::integratePointcloud (pointcloud_integrator.cpp:33-63) and
// pcl::fromROSMsg: x, y, z must be FLOAT32; a field named rgb makes an XYZRGB cloud (FLOAT32 or UINT32: the
// reference overwrites its datatype, cpp:36-39), else a field named intensity (FLOAT32) an XYZI cloud, else XYZ.
// Throws std::invalid_argument for a big-endian message, a missing coordinate or another datatype; sizes are
// checked by the library.
inline vgx_cloud_layout CloudLayout(const PointCloud2View& msg) {
  if (msg.is_bigendian) throw std::invalid_argument("CloudLayout: big-endian messages are not supported");
  const auto find = [&](const char* name) -> const PointField* {
    for (const PointField& f : msg.fields)
      if (f.name == name) return &f;
    return nullptr;
  };
  const auto need = [&](const char* name, bool uint32_too) -> int32_t {
    const PointField* f = find(name);
    if (!f) throw std::invalid_argument(std::string("CloudLayout: the message has no field ") + name);
    if (!(f->datatype == PointField::FLOAT32 || (uint32_too && f->datatype == PointField::UINT32)) || f->count != 1)
      throw std::invalid_argument(std::string("CloudLayout: field ") + name + " has the wrong datatype or count");
    return (int32_t)f->offset;
  };
  vgx_cloud_layout L;
  L.width = msg.width; L.height = msg.height; L.point_step = msg.point_step; L.row_step = msg.row_step;
  L.x_offset = need("x", false); L.y_offset = need("y", false); L.z_offset = need("z", false);
  L.rgb_offset = find("rgb") ? need("rgb", true) : -1;
  L.intensity_offset = L.rgb_offset < 0 && find("intensity") ? need("intensity", false) : -1;
  return L;
}

// PointcloudIntegrator::integratePointcloud (pointcloud_integrator.cpp:23-90): from the sensor message
// (PointCloud2View; decoded on the device), or from a voxblox::Pointcloud already converted (points_C, n x 3
// floats, sensor frame).
class PointcloudIntegrator {
 public:
  explicit PointcloudIntegrator(Context& ctx) : ctx_(ctx) { vgx_tsdf_config_default(&config_); config_.mode = 1; }
  vgx_tsdf_config& config() { return config_; }  // voxblox::TsdfIntegratorBase::Config
  void createSubmap(SubmapID id, float voxel_size, int vps = 16, int capacity_blocks = 16384) {
    ctx_.check(vgx_submap_create(ctx_.get(), id, voxel_size, vps, capacity_blocks));
  }
  // T_submap_sensor = [qw qx qy qz tx ty tz]; rgba: the voxblox::Colors of the cloud (n x 4 bytes r, g, b, a),
  // or nullptr for a cloud without colours (the submap then gets no colour channel)
  vgx_tsdf_stats integratePointcloud(SubmapID submap, const float T_submap_sensor[7], int n,
                                     const float* points_C, const uint8_t* rgba = nullptr) {
    vgx_tsdf_stats st;
    ctx_.check(vgx_tsdf_integrate(ctx_.get(), submap, T_submap_sensor, n, points_C, rgba, &config_, &st));
    return st;
  }
  // The reference's call: the message is decoded on the device (records with a non-finite coordinate dropped;
  // colours from rgb, the grey of intensity with maximum colorMapMax(), or black) and integrated in the same
  // call.  colours = false integrates without colours.  n_points (may be null): the records kept.
  vgx_tsdf_stats integratePointcloud(SubmapID submap, const float T_submap_sensor[7], const PointCloud2View& msg,
                                     bool colours = true, int* n_points = nullptr) {
    const vgx_cloud_layout layout = CloudLayout(msg);
    vgx_tsdf_stats st;
    ctx_.check(vgx_tsdf_integrate_cloud(ctx_.get(), submap, T_submap_sensor, &layout, msg.data, msg.size,
                                        colours ? 1 : 0, color_map_max_, &config_, &st, n_points));
    return st;
  }
  float& colorMapMax() { return color_map_max_; }   // GrayscaleColorMap::setMaxValue (cpp:14)
  // VoxgraphSubmap::finishSubmap (voxgraph_submap.cpp:84-107): registration view, then - with a
  // filter - the registration points (relevant voxels + isosurface vertices), the surface OBB and
  // the isosurface block list, all on the device
  void finishSubmap(SubmapID id) { ctx_.check(vgx_submap_finish(ctx_.get(), id)); }
  void finishSubmap(SubmapID id, const vgx_registration_filter& filter) {
    ctx_.check(vgx_submap_finish(ctx_.get(), id));
    if (filter.use_esdf_distance) ctx_.check(vgx_submap_generate_esdf(ctx_.get(), id, nullptr, nullptr));  // cpp:86
    ctx_.check(vgx_submap_extract_points(ctx_.get(), id, &filter));
  }

 private:
  Context& ctx_;
  vgx_tsdf_config config_;
  float color_map_max_ = 10000.0f;
};

}  // namespace voxgraph_b200
