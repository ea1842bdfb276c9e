"""ctypes front-end for the CPU oracle (oracle/vg_oracle.c).

TEST INFRASTRUCTURE ONLY. May be imported by tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline / --impl reference legs — never by voxgraph_b200/.
Parity unpinned against the real reference binaries (see vg_oracle.h).
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libvg_oracle.so")


def build(force=False):
    """Compile the C restatement with the committed Makefile."""
    src = [os.path.join(_HERE, f) for f in ("vg_oracle.c", "vg_oracle.h", "Makefile")]
    if (not force and os.path.exists(_LIB_PATH)
            and all(os.path.getmtime(_LIB_PATH) >= os.path.getmtime(s) for s in src)):
        return _LIB_PATH
    env = dict(os.environ)
    env.pop("CC", None)
    subprocess.run(["make", "-C", _HERE, "-B"], check=True, env=env,
                   stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    return _LIB_PATH


_REF_SAMPLER_PATH = os.path.join(_HERE, "_ref", "libvgref_sampler.so")
_ref_sampler = None


def ref_sampler_lib():
    """oracle/_ref/libvgref_sampler.so: the REFERENCE's own WeightedSampler template compiled from a
    voxgraph checkout (oracle/ref_sampler_shim.cpp + Makefile target `ref`, VOXGRAPH_SRC=<voxgraph/>).
    Returns None when it has not been built."""
    global _ref_sampler
    if _ref_sampler is None:
        if not os.path.exists(_REF_SAMPLER_PATH):
            return None
        L = C.CDLL(_REF_SAMPLER_PATH)
        L.vgref_sampler_create.restype = C.c_void_p
        L.vgref_sampler_create.argtypes = [C.POINTER(C.c_float), C.c_int]
        L.vgref_sampler_destroy.argtypes = [C.c_void_p]
        L.vgref_sampler_draw.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int32)]
        _ref_sampler = L
    return _ref_sampler


class RefWeightedSampler:
    """The reference's voxgraph::WeightedSampler (compiled, oracle/_ref)."""

    def __init__(self, weights):
        L = ref_sampler_lib()
        if L is None:
            raise RuntimeError("oracle/_ref/libvgref_sampler.so is not built")
        w = np.ascontiguousarray(weights, np.float32)
        self._L = L
        self._h = L.vgref_sampler_create(_p(w, C.c_float), len(w))

    def draw(self, count):
        idx = np.zeros(count, np.int32)
        self._L.vgref_sampler_draw(self._h, int(count), _p(idx, C.c_int32))
        return idx

    def __del__(self):
        try:
            self._L.vgref_sampler_destroy(self._h)
        except Exception:
            pass


class SolverOptions(C.Structure):
    _fields_ = [("max_num_iterations", C.c_int),
                ("parameter_tolerance", C.c_double),
                ("function_tolerance", C.c_double),
                ("gradient_tolerance", C.c_double),
                ("initial_trust_region_radius", C.c_double),
                ("max_trust_region_radius", C.c_double),
                ("min_trust_region_radius", C.c_double),
                ("min_relative_decrease", C.c_double),
                ("min_lm_diagonal", C.c_double),
                ("max_lm_diagonal", C.c_double),
                ("max_solver_time_s", C.c_double),
                ("jacobi_scaling", C.c_int),
                ("num_threads", C.c_int),
                ("exclude_registration", C.c_int)]


class SolverSummary(C.Structure):
    _fields_ = [("iterations", C.c_int),
                ("num_successful_steps", C.c_int),
                ("num_residual_evals", C.c_int),
                ("termination", C.c_int),
                ("initial_cost", C.c_double),
                ("final_cost", C.c_double),
                ("total_time_s", C.c_double),
                ("eval_time_s", C.c_double),
                ("linear_solver_time_s", C.c_double)]


class TsdfConfig(C.Structure):
    _fields_ = [("default_truncation_distance", C.c_float),
                ("max_weight", C.c_float),
                ("voxel_carving_enabled", C.c_int),
                ("min_ray_length_m", C.c_float),
                ("max_ray_length_m", C.c_float),
                ("use_const_weight", C.c_int),
                ("allow_clear", C.c_int),
                ("use_weight_dropoff", C.c_int),
                ("use_sparsity_compensation_factor", C.c_int),
                ("sparsity_compensation_factor", C.c_float),
                ("start_voxel_subsampling_factor", C.c_float),
                ("max_consecutive_ray_collisions", C.c_int),
                ("mode", C.c_int)]


class EsdfConfig(C.Structure):
    _fields_ = [("max_distance_m", C.c_float), ("default_distance_m", C.c_float),
                ("min_distance_m", C.c_float), ("min_weight", C.c_float)]


class TsdfStats(C.Structure):
    _fields_ = [("rays_valid", C.c_int64), ("rays_cast", C.c_int64),
                ("voxel_updates", C.c_int64), ("blocks_allocated", C.c_int64)]


class TsdfTrace(C.Structure):
    _fields_ = [("n", C.c_int64), ("cap", C.c_int64), ("g", C.POINTER(C.c_int64)),
                ("sdf", C.POINTER(C.c_float)), ("uw", C.POINTER(C.c_float))]


class Sampler(C.Structure):
    _fields_ = [("mt", C.c_uint32 * 624), ("idx", C.c_int)]


_P = C.POINTER
_vp, _i32, _u32, _f32, _f64 = C.c_void_p, C.c_int, C.c_uint32, C.c_float, C.c_double
_pi32, _pi64, _pf, _pd = _P(C.c_int32), _P(C.c_int64), _P(C.c_float), _P(C.c_double)

# (restype, argtypes) of every function vg_oracle.h declares, in the header's order.  c_void_p stands only for
# the opaque vgo_layer* and vgo_graph*; tests/test_host_binding_signatures.py compares every entry with the header.
SIGNATURES = {
    # layer, index math, interpolation
    "vgo_layer_create": (_vp, [_f32, _i32]),
    "vgo_layer_destroy": (None, [_vp]),
    "vgo_layer_add_block": (_i32, [_vp, _pi32, _pf, _pf]),
    "vgo_layer_num_blocks": (_i32, [_vp]),
    "vgo_layer_find_block": (_i32, [_vp, _pi32]),
    "vgo_layer_export": (None, [_vp, _pi32, _pf, _pf]),
    "vgo_layer_voxel_size_inv": (_f32, [_vp]),
    "vgo_layer_block_size_inv": (_f32, [_vp]),
    "vgo_grid_index_from_point": (None, [_pf, _f32, _pi32]),
    "vgo_block_and_local_from_global": (None, [_pi64, _i32, _pi32, _pi32]),
    "vgo_interp_voxels_and_q": (_i32, [_vp, _pf, _pi32, _pi32, _pi32, _pi32, _pf, _pf]),
    # transforms
    "vgo_T_exp": (None, [_pf, _pf]),
    "vgo_T_inverse": (None, [_pf, _pf]),
    "vgo_T_compose": (None, [_pf, _pf, _pf]),
    "vgo_T_transform": (None, [_pf, _pf, _pf]),
    # cost functions
    "vgo_reg_evaluate": (_i32, [_vp, _i32, _pf, _pf, _pf, _f64, _pd, _pd, _pd, _pd, _pd]),
    "vgo_reg_pose_setup": (None, [_pd, _pd, _pf, _pf]),
    "vgo_relpose_evaluate": (None, [_pd, _pd, _pd, _f64, _pd, _pd, _pd, _pd]),
    "vgo_sqrt_information": (_i32, [_pd, _pd]),
    "vgo_sqrt_information_ldlt": (_i32, [_pd, _pd]),
    "vgo_normalize_angle": (_f64, [_f64]),
    # pose graph
    "vgo_solver_options_default": (None, [_P(SolverOptions)]),
    "vgo_graph_create": (_vp, []),
    "vgo_graph_destroy": (None, [_vp]),
    "vgo_graph_add_node": (_i32, [_vp, _u32, _pd, _i32]),
    "vgo_graph_add_relative": (_i32, [_vp, _u32, _u32, _pd, _f64, _pd]),
    "vgo_graph_add_registration": (_i32, [_vp, _u32, _u32, _vp, _i32, _pf, _pf, _pf, _f64]),
    "vgo_graph_reset_registration": (None, [_vp]),
    "vgo_graph_num_nodes": (_i32, [_vp]),
    "vgo_graph_num_registration_residuals": (_i32, [_vp]),
    "vgo_graph_get_poses": (None, [_vp, _pd]),
    "vgo_graph_set_poses": (None, [_vp, _pd]),
    "vgo_graph_eval": (_i32, [_vp, _i32, _i32, _pd, _pd, _pd]),
    "vgo_graph_registration_costs": (None, [_vp, _pd]),
    "vgo_graph_solve": (_i32, [_vp, _P(SolverOptions), _P(SolverSummary)]),
    # submap finishing, bounding boxes, overlap
    "vgo_find_relevant_voxels": (_i32, [_vp, _f64, _f64, _pf, _pf, _pf, _i32]),
    "vgo_find_isosurface_vertices": (_i32, [_vp, _f64, _pf, _pf, _pf, _i32, _pi32, _i32, _pi32]),
    "vgo_interp_voxel": (_i32, [_vp, _pf, _pf, _pf]),
    "vgo_esdf_config_default": (None, [_P(EsdfConfig)]),
    "vgo_generate_esdf": (_i32, [_vp, _P(EsdfConfig), _pf, _pf]),
    "vgo_surface_obb": (_i32, [_vp, _f64, _f64, _pf, _pf]),
    "vgo_aabb_from_obb_and_pose": (None, [_pf, _pf, _pf, _pf, _pf]),
    "vgo_submaps_overlap": (_i32, [_pf, _pf, _pf, _pf, _pf, _pf, _pi32, _i32, _f32, _vp]),
    # weighted sampler
    "vgo_sampler_init": (None, [_P(Sampler)]),
    "vgo_sampler_next_u32": (_u32, [_P(Sampler)]),
    "vgo_sampler_canonical": (_f64, [_P(Sampler)]),
    "vgo_sampler_draw": (None, [_P(Sampler), _pd, _i32, _i32, _pi32]),
    # TSDF integration
    "vgo_tsdf_config_default": (None, [_P(TsdfConfig)]),
    "vgo_tsdf_integrate": (None, [_vp, _P(TsdfConfig), _pf, _i32, _pf, _P(TsdfStats)]),
    "vgo_tsdf_integrate_trace": (None, [_vp, _P(TsdfConfig), _pf, _i32, _pf, _P(TsdfStats), _P(TsdfTrace)]),
    "vgo_tsdf_trace_free": (None, [_P(TsdfTrace)]),
    "vgo_tsdf_integrate_mt": (None, [_vp, _P(TsdfConfig), _pf, _i32, _pf, _i32, _P(TsdfStats)]),
    "vgo_raycast": (_i32, [_pf, _pf, _i32, _i32, _f32, _f32, _f32, _i32, _pi64, _i32]),
}

_lib = None


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t)) if a is not None else None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    build()
    L = C.CDLL(_LIB_PATH)
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = restype, argtypes
    _lib = L
    return L


def f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


class Layer:
    """voxblox::Layer restatement holding (distance, weight) voxels."""

    def __init__(self, voxel_size, vps=16):
        self.voxel_size = float(np.float32(voxel_size))
        self.vps = int(vps)
        self._h = lib().vgo_layer_create(voxel_size, vps)

    def __del__(self):
        if getattr(self, "_h", None):
            lib().vgo_layer_destroy(self._h)
            self._h = None

    @classmethod
    def from_blocks(cls, voxel_size, vps, block_idx, distance, weight):
        l = cls(voxel_size, vps)
        l.add_blocks(block_idx, distance, weight)
        return l

    @classmethod
    def adopt(cls, h, voxel_size, vps):
        """A Layer that owns the vgo_layer* h made elsewhere (a C harness): it is destroyed with the Layer."""
        l = cls.__new__(cls)
        l.voxel_size = float(np.float32(voxel_size))
        l.vps = int(vps)
        l._h = h
        return l

    def add_blocks(self, block_idx, distance, weight):
        bi = np.ascontiguousarray(block_idx, dtype=np.int32).reshape(-1, 3)
        n = bi.shape[0]
        if n == 0:
            return
        d = f32(distance).reshape(n, -1)
        w = f32(weight).reshape(n, -1)
        assert d.shape[1] == self.vps ** 3
        for i in range(n):
            lib().vgo_layer_add_block(self._h, _p(bi[i], C.c_int32), _p(d[i], C.c_float),
                                      _p(w[i], C.c_float))

    @property
    def num_blocks(self):
        return lib().vgo_layer_num_blocks(self._h)

    @property
    def voxel_size_inv(self):
        return lib().vgo_layer_voxel_size_inv(self._h)

    @property
    def block_size_inv(self):
        return lib().vgo_layer_block_size_inv(self._h)

    def find_block(self, idx):
        k = np.ascontiguousarray(idx, dtype=np.int32)
        return lib().vgo_layer_find_block(self._h, _p(k, C.c_int32))

    def export(self):
        n = self.num_blocks
        v = self.vps ** 3
        idx = np.zeros((n, 3), np.int32)
        d = np.zeros((n, v), np.float32)
        w = np.zeros((n, v), np.float32)
        lib().vgo_layer_export(self._h, _p(idx, C.c_int32), _p(d, C.c_float), _p(w, C.c_float))
        return idx, d, w

    def interp(self, pos):
        """getVoxelsAndQVector -> dict."""
        pos = f32(pos)
        bb = np.zeros(3, np.int32); bv = np.zeros(3, np.int32)
        slots = np.full(8, -1, np.int32); lin = np.full(8, -1, np.int32)
        d = np.zeros(8, np.float32); q = np.zeros(8, np.float32)
        ok = lib().vgo_interp_voxels_and_q(self._h, _p(pos, C.c_float), _p(bb, C.c_int32),
                                           _p(bv, C.c_int32), _p(slots, C.c_int32),
                                           _p(lin, C.c_int32), _p(d, C.c_float), _p(q, C.c_float))
        return dict(ok=bool(ok), base_block=bb, base_voxel=bv, slots=slots, linear=lin,
                    distances=d, q=q)


def reg_evaluate(layer, xyz, distance, weight, ref_pose, read_pose, no_correspondence_cost=0.0,
                 jacobians=True):
    """RegistrationCostFunction::Evaluate -> (ok, residuals, J_ref, J_read)."""
    xyz = f32(xyz).reshape(-1, 3)
    n = xyz.shape[0]
    distance = f32(distance); weight = f32(weight)
    r = np.zeros(n, np.float64)
    jr = np.zeros((n, 4), np.float64) if jacobians else None
    je = np.zeros((n, 4), np.float64) if jacobians else None
    ref_pose = f64(ref_pose); read_pose = f64(read_pose)
    ok = lib().vgo_reg_evaluate(layer._h, n, _p(xyz, C.c_float), _p(distance, C.c_float),
                                _p(weight, C.c_float), float(no_correspondence_cost),
                                _p(ref_pose, C.c_double), _p(read_pose, C.c_double),
                                _p(r, C.c_double), _p(jr, C.c_double), _p(je, C.c_double))
    return bool(ok), r, jr, je


def reg_pose_setup(ref_pose, read_pose):
    T = np.zeros(7, np.float32); trig = np.zeros(8, np.float32)
    ref_pose = f64(ref_pose); read_pose = f64(read_pose)
    lib().vgo_reg_pose_setup(_p(ref_pose, C.c_double), _p(read_pose, C.c_double),
                             _p(T, C.c_float), _p(trig, C.c_float))
    return T, trig


def relpose_evaluate(pose_a, pose_b, t_obs, yaw_obs, sqrt_info):
    r = np.zeros(4); ja = np.zeros((4, 4)); jb = np.zeros((4, 4))
    pa = f64(pose_a); pb = f64(pose_b); to = f64(t_obs); L = f64(sqrt_info).reshape(16)
    lib().vgo_relpose_evaluate(_p(pa, C.c_double), _p(pb, C.c_double), _p(to, C.c_double),
                               float(yaw_obs), _p(L, C.c_double), _p(r, C.c_double),
                               _p(ja, C.c_double), _p(jb, C.c_double))
    return r, ja, jb


def sqrt_information(info):
    info = f64(info).reshape(16)
    out = np.zeros(16)
    rc = lib().vgo_sqrt_information(_p(info, C.c_double), _p(out, C.c_double))
    if rc != 0:
        raise ValueError("information matrix not positive definite")
    return out.reshape(4, 4)


def sqrt_information_ldlt(info):
    """allow_semi_definite_information_matrix branch (constraint.cpp:15-37)."""
    info = f64(info).reshape(16)
    out = np.zeros(16)
    rc = lib().vgo_sqrt_information_ldlt(_p(info, C.c_double), _p(out, C.c_double))
    if rc != 0:
        raise ValueError("information matrix must be positive semi-definite")
    return out.reshape(4, 4)


def normalize_angle(a):
    return lib().vgo_normalize_angle(float(a))


def T_exp(v6):
    v = f32(v6); T = np.zeros(7, np.float32)
    lib().vgo_T_exp(_p(v, C.c_float), _p(T, C.c_float))
    return T


def T_inverse(T):
    T = f32(T); o = np.zeros(7, np.float32)
    lib().vgo_T_inverse(_p(T, C.c_float), _p(o, C.c_float))
    return o


def T_compose(A, B):
    A = f32(A); B = f32(B); o = np.zeros(7, np.float32)
    lib().vgo_T_compose(_p(A, C.c_float), _p(B, C.c_float), _p(o, C.c_float))
    return o


def T_transform(T, p):
    T = f32(T); p = f32(p); o = np.zeros(3, np.float32)
    lib().vgo_T_transform(_p(T, C.c_float), _p(p, C.c_float), _p(o, C.c_float))
    return o


def grid_index_from_point(p, inv):
    p = f32(p); o = np.zeros(3, np.int32)
    lib().vgo_grid_index_from_point(_p(p, C.c_float), float(inv), _p(o, C.c_int32))
    return o


def block_and_local_from_global(g, vps):
    g = np.ascontiguousarray(g, dtype=np.int64)
    b = np.zeros(3, np.int32); l = np.zeros(3, np.int32)
    lib().vgo_block_and_local_from_global(_p(g, C.c_int64), int(vps), _p(b, C.c_int32),
                                          _p(l, C.c_int32))
    return b, l


def solver_options(**kw):
    o = SolverOptions()
    lib().vgo_solver_options_default(C.byref(o))
    for k, v in kw.items():
        setattr(o, k, v)
    return o


class Graph:
    """PoseGraph restatement: nodes, relative-pose and registration residual blocks."""

    def __init__(self):
        self._h = lib().vgo_graph_create()
        self._keep = []

    def __del__(self):
        if getattr(self, "_h", None):
            lib().vgo_graph_destroy(self._h)
            self._h = None

    def add_node(self, node_id, xyzyaw, constant=False):
        x = f64(xyzyaw)
        return lib().vgo_graph_add_node(self._h, int(node_id), _p(x, C.c_double), int(constant))

    def add_relative(self, id_a, id_b, t_obs, yaw_obs, sqrt_info):
        to = f64(t_obs); L = f64(sqrt_info).reshape(16)
        rc = lib().vgo_graph_add_relative(self._h, int(id_a), int(id_b), _p(to, C.c_double),
                                          float(yaw_obs), _p(L, C.c_double))
        assert rc >= 0
        return rc

    def add_registration(self, ref_id, read_id, reading_layer, xyz, distance, weight,
                         no_correspondence_cost=0.0):
        xyz = f32(xyz).reshape(-1, 3); distance = f32(distance); weight = f32(weight)
        self._keep += [reading_layer, xyz, distance, weight]
        rc = lib().vgo_graph_add_registration(self._h, int(ref_id), int(read_id),
                                              reading_layer._h, xyz.shape[0],
                                              _p(xyz, C.c_float), _p(distance, C.c_float),
                                              _p(weight, C.c_float),
                                              float(no_correspondence_cost))
        assert rc >= 0
        return rc

    def reset_registration(self):
        lib().vgo_graph_reset_registration(self._h)

    @property
    def num_nodes(self):
        return lib().vgo_graph_num_nodes(self._h)

    @property
    def num_registration_residuals(self):
        return lib().vgo_graph_num_registration_residuals(self._h)

    def poses(self):
        x = np.zeros((self.num_nodes, 4))
        lib().vgo_graph_get_poses(self._h, _p(x, C.c_double))
        return x

    def set_poses(self, x):
        x = f64(x).reshape(self.num_nodes, 4)
        lib().vgo_graph_set_poses(self._h, _p(x, C.c_double))

    def eval(self, num_threads=1, exclude_registration=False, want_gradient=True, want_H=True):
        n = 4 * self.num_nodes
        cost = C.c_double(0)
        g = np.zeros(n) if want_gradient else None
        H = np.zeros((n, n)) if want_H else None
        ok = lib().vgo_graph_eval(self._h, int(num_threads), int(exclude_registration),
                                  C.byref(cost), _p(g, C.c_double), _p(H, C.c_double))
        return bool(ok), cost.value, g, H

    def registration_costs(self, n_constraints):
        out = np.zeros(n_constraints)
        lib().vgo_graph_registration_costs(self._h, _p(out, C.c_double))
        return out

    def solve(self, options=None):
        o = options if options is not None else solver_options()
        s = SolverSummary()
        rc = lib().vgo_graph_solve(self._h, C.byref(o), C.byref(s))
        return rc, s


class WeightedSampler:
    """WeightedSampler<RegistrationPoint> (weighted_sampler.h:10-37): cumulative double weights +
    a default-seeded mt19937; draw(count) = getRandomItem x count -> item indices."""

    def __init__(self, weights):
        w = np.asarray(weights, np.float32)
        self.cumulative = np.cumsum(w.astype(np.float64))   # addItem: sequential double sums
        self._state = Sampler()
        lib().vgo_sampler_init(C.byref(self._state))

    def next_u32(self):
        return int(lib().vgo_sampler_next_u32(C.byref(self._state)))

    def canonical(self):
        return float(lib().vgo_sampler_canonical(C.byref(self._state)))

    def draw(self, count):
        idx = np.zeros(count, np.int32)
        cum = np.ascontiguousarray(self.cumulative)
        lib().vgo_sampler_draw(C.byref(self._state), _p(cum, C.c_double), len(cum), int(count),
                               _p(idx, C.c_int32))
        return idx


def sampled_num_residuals(sampling_ratio, n_points):
    """registration_cost_function.cpp:45-55: int(float ratio * size())."""
    if sampling_ratio == -1:
        return int(n_points)
    return int(np.float32(sampling_ratio) * np.float32(n_points))


def reg_evaluate_sampled(layer, xyz, distance, indices, ref_pose, read_pose,
                         no_correspondence_cost=0.0, jacobians=True):
    """Evaluate in sampling mode (cpp:118-122) for a given draw: residual j uses point
    indices[j] with its weight forced to 1."""
    idx = np.asarray(indices, np.int64)
    return reg_evaluate(layer, np.asarray(xyz, np.float32)[idx], np.asarray(distance, np.float32)[idx],
                        np.ones(len(idx), np.float32), ref_pose, read_pose,
                        no_correspondence_cost=no_correspondence_cost, jacobians=jacobians)


def find_relevant_voxels(layer, min_voxel_weight=1.0, max_voxel_distance=0.3):
    """findRelevantVoxelIndices -> (xyz (n,3), distance (n,), weight (n,))."""
    n = lib().vgo_find_relevant_voxels(layer._h, float(min_voxel_weight), float(max_voxel_distance),
                                       None, None, None, 0)
    xyz = np.zeros((n, 3), np.float32); d = np.zeros(n, np.float32); w = np.zeros(n, np.float32)
    lib().vgo_find_relevant_voxels(layer._h, float(min_voxel_weight), float(max_voxel_distance),
                                   _p(xyz, C.c_float), _p(d, C.c_float), _p(w, C.c_float), n)
    return xyz, d, w


def find_isosurface_vertices(layer, min_voxel_weight=1.0):
    """findIsosurfaceVertices -> (xyz (n,3), distance (n,), weight (n,), isosurface_blocks (m,3))."""
    # counted first, as find_relevant_voxels does; a vertex lies in its cube's block or in one of the
    # 7 forward neighbours, so 8 block indices per block always suffice
    blk = np.zeros((max(1, layer.num_blocks) * 8, 3), np.int32); nb = C.c_int(0)
    n = lib().vgo_find_isosurface_vertices(layer._h, float(min_voxel_weight), None, None, None, 0,
                                           _p(blk, C.c_int32), blk.shape[0], C.byref(nb))
    xyz = np.zeros((n, 3), np.float32); d = np.zeros(n, np.float32); w = np.zeros(n, np.float32)
    got = lib().vgo_find_isosurface_vertices(layer._h, float(min_voxel_weight), _p(xyz, C.c_float),
                                             _p(d, C.c_float), _p(w, C.c_float), n, _p(blk, C.c_int32),
                                             blk.shape[0], C.byref(nb))
    assert got == n and nb.value <= blk.shape[0]
    return xyz, d, w, blk[:nb.value].copy()


def interp_voxel(layer, pos):
    """Interpolator::getVoxel(pos, interpolate=True) -> (ok, distance, weight)."""
    p = f32(pos); d = C.c_float(0); w = C.c_float(0)
    ok = lib().vgo_interp_voxel(layer._h, _p(p, C.c_float), C.byref(d), C.byref(w))
    return bool(ok), d.value, w.value


def esdf_config(**kw):
    c = EsdfConfig()
    lib().vgo_esdf_config_default(C.byref(c))
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def generate_esdf(layer, cfg=None):
    """generateEsdf -> (distance (n_blocks, vps^3), observed (n_blocks, vps^3), sweeps), slot order."""
    cfg = cfg or esdf_config()
    n = layer.num_blocks
    vpb = layer.vps ** 3
    d = np.zeros((max(n, 1), vpb), np.float32); ob = np.zeros((max(n, 1), vpb), np.float32)
    sweeps = lib().vgo_generate_esdf(layer._h, C.byref(cfg), _p(d, C.c_float), _p(ob, C.c_float))
    return d[:n], ob[:n], sweeps


def surface_obb(layer, min_voxel_weight=1.0, max_voxel_distance=0.3):
    mn = np.zeros(3, np.float32); mx = np.zeros(3, np.float32)
    ok = lib().vgo_surface_obb(layer._h, float(min_voxel_weight), float(max_voxel_distance),
                               _p(mn, C.c_float), _p(mx, C.c_float))
    return bool(ok), mn, mx


def aabb_from_obb_and_pose(obb_min, obb_max, pose_T):
    a = f32(obb_min); b = f32(obb_max); T = f32(pose_T)
    mn = np.zeros(3, np.float32); mx = np.zeros(3, np.float32)
    lib().vgo_aabb_from_obb_and_pose(_p(a, C.c_float), _p(b, C.c_float), _p(T, C.c_float),
                                     _p(mn, C.c_float), _p(mx, C.c_float))
    return mn, mx


def submaps_overlap(aabb, other_aabb, pose_T, other_pose_T, isosurface_blocks, block_size, other_layer):
    blk = np.ascontiguousarray(isosurface_blocks, np.int32).reshape(-1, 3)
    a0, a1 = f32(aabb[0]), f32(aabb[1]); b0, b1 = f32(other_aabb[0]), f32(other_aabb[1])
    T = f32(pose_T); To = f32(other_pose_T)
    return bool(lib().vgo_submaps_overlap(_p(a0, C.c_float), _p(a1, C.c_float), _p(b0, C.c_float),
                                          _p(b1, C.c_float), _p(T, C.c_float), _p(To, C.c_float),
                                          _p(blk, C.c_int32), blk.shape[0], float(block_size),
                                          other_layer._h))


def tsdf_config(**kw):
    c = TsdfConfig()
    lib().vgo_tsdf_config_default(C.byref(c))
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def tsdf_integrate(layer, cfg, T_G_C, points_C):
    T = f32(T_G_C); pts = f32(points_C).reshape(-1, 3)
    st = TsdfStats()
    lib().vgo_tsdf_integrate(layer._h, C.byref(cfg), _p(T, C.c_float), pts.shape[0],
                             _p(pts, C.c_float), C.byref(st))
    return st


def tsdf_integrate_trace(layer, cfg, T_G_C, points_C):
    """tsdf_integrate that also returns its voxel updates in the order they were applied:
    (stats, g (m, 3) int64 global voxel indices, sdf (m,) float32, update weight (m,) float32)."""
    T = f32(T_G_C); pts = f32(points_C).reshape(-1, 3)
    st = TsdfStats(); tr = TsdfTrace()
    lib().vgo_tsdf_integrate_trace(layer._h, C.byref(cfg), _p(T, C.c_float), pts.shape[0],
                                   _p(pts, C.c_float), C.byref(st), C.byref(tr))
    m = int(tr.n)
    try:
        if m == 0:
            return st, np.zeros((0, 3), np.int64), np.zeros(0, np.float32), np.zeros(0, np.float32)
        g = np.ctypeslib.as_array(tr.g, shape=(m * 3,)).reshape(m, 3).copy()
        sdf = np.ctypeslib.as_array(tr.sdf, shape=(m,)).copy()
        uw = np.ctypeslib.as_array(tr.uw, shape=(m,)).copy()
    finally:
        lib().vgo_tsdf_trace_free(C.byref(tr))
    return st, g, sdf, uw


def tsdf_integrate_mt(layer, cfg, T_G_C, points_C, num_threads):
    """Multi-threaded integrator (voxblox runs hardware_concurrency threads): timing baseline."""
    T = f32(T_G_C); pts = f32(points_C).reshape(-1, 3)
    st = TsdfStats()
    lib().vgo_tsdf_integrate_mt(layer._h, C.byref(cfg), _p(T, C.c_float), pts.shape[0],
                                _p(pts, C.c_float), int(num_threads), C.byref(st))
    return st


def raycast(origin, point_G, voxel_size_inv, truncation_distance, is_clearing=False,
            voxel_carving=True, max_ray_length_m=16.0, cast_from_origin=True, max_out=4096):
    o = f32(origin); p = f32(point_G)
    out = np.zeros((max_out, 3), np.int64)
    n = lib().vgo_raycast(_p(o, C.c_float), _p(p, C.c_float), int(is_clearing),
                          int(voxel_carving), float(max_ray_length_m), float(voxel_size_inv),
                          float(truncation_distance), int(cast_from_origin), _p(out, C.c_int64),
                          max_out)
    return out[:min(n, max_out)], n
