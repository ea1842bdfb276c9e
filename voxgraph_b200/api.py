"""Host-side mirror of the reference's interface for the two hot paths, on top of the C-ABI.

Names, argument meaning and error behaviour follow the reference:
  PoseGraph                 voxgraph/include/voxgraph/backend/pose_graph.h:15-65
  RegistrationCostFunction  .../cost_functions/registration_cost_function.h:11-82
  PointcloudIntegrator      voxgraph/include/voxgraph/frontend/measurement_processors/pointcloud_integrator.h
(the C++ mirror of the same surface lives in voxgraph_b200/host/; this module is what the
pytest parity tests and bench.py drive).
"""
import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from . import _lib
from ._lib import (CloudLayout, CollectionEntry, EsdfConfig, MapEvaluationResult, MeshConfig, RegConfig, RegistrationFilter,
                   SolverOptions, SolverSummary, TsdfConfig, TsdfStats, VoxelEvaluationDetails)

# sensor_msgs/PointField datatypes the message front end looks at
POINTFIELD_UINT32 = 6
POINTFIELD_FLOAT32 = 7

K_VOXELS = 0            # VoxgraphSubmap::RegistrationPointType::kVoxels
K_ISOSURFACE_POINTS = 1  # ...::kIsosurfacePoints


class VgxError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("vgx error %d: %s" % (code, msg))
        self.code = code


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t)) if a is not None else None


def _ref(x):
    """An optional struct by reference: NULL for None."""
    return C.byref(x) if x is not None else None


def _config(struct, default_fn, **kw):
    """A config struct holding the library's defaults, then the fields given."""
    c = struct()
    default_fn(C.byref(c))
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def _ids_poses(submap_ids, poses_T, what, optional=False):
    """uint32 submap ids (n,) and float32 poses (n, 7), one per submap; poses_T may be None when optional."""
    ids = np.ascontiguousarray(submap_ids, np.uint32).reshape(-1)
    if optional and poses_T is None:
        return ids, None
    T = _f32(poses_T).reshape(-1, 7)
    if T.shape[0] != ids.shape[0]:
        raise ValueError("%s: one pose per submap" % what)
    return ids, T


def _call_noctx(name, *args, allow=(0,)):
    """An entry point without a context, so without a vgx_last_error message: a status outside allow raises."""
    rc = getattr(_lib.load(), name)(*args)
    if rc not in allow:
        raise VgxError(rc, "%s failed" % name)


def _bytes_arg(data):
    """A bytes-like object as a C buffer without copying it (read-only views other than bytes are copied)."""
    if isinstance(data, bytes):
        return data, len(data)
    mv = memoryview(data).cast("B")
    if mv.readonly or mv.nbytes == 0:
        b = mv.tobytes()
        return b, len(b)
    return (C.c_char * mv.nbytes).from_buffer(mv), mv.nbytes


@dataclass
class PointCloud2:
    """A sensor_msgs/PointCloud2 without ROS: fields is a list of (name, offset, datatype, count), data any
    bytes-like object of at least height * row_step bytes."""
    fields: list
    width: int
    height: int
    point_step: int
    row_step: int
    data: object
    is_bigendian: bool = False


def cloud_layout(msg):
    """The field matching of PointcloudIntegrator::integratePointcloud (pointcloud_integrator.cpp:33-63) and
    pcl::fromROSMsg -> CloudLayout.  x, y and z must be FLOAT32 fields; a field named rgb makes the cloud an
    XYZRGB one (FLOAT32 or UINT32: the reference overwrites its datatype, cpp:36-39), else a field named intensity
    (FLOAT32) an XYZI one, else it is XYZ.  Other fields are ignored.  ValueError for a big-endian message, a
    missing coordinate or a datatype the reference's point types do not have; sizes are checked by the library."""
    if msg.is_bigendian:
        raise ValueError("cloud_layout: big-endian messages are not supported")
    by_name = {}
    for name, offset, datatype, count in msg.fields:
        by_name.setdefault(name, (int(offset), int(datatype), int(count)))

    def need(name, datatypes, what):
        offset, datatype, count = by_name[name]
        if datatype not in datatypes or count != 1:
            raise ValueError("cloud_layout: field %s must be one %s" % (name, what))
        return offset

    for name in "xyz":
        if name not in by_name:
            raise ValueError("cloud_layout: the message has no field %s" % name)
    L = CloudLayout(width=msg.width, height=msg.height, point_step=msg.point_step, row_step=msg.row_step,
                    rgb_offset=-1, intensity_offset=-1)
    L.x_offset, L.y_offset, L.z_offset = (need(name, (POINTFIELD_FLOAT32,), "FLOAT32") for name in "xyz")
    if "rgb" in by_name:
        L.rgb_offset = need("rgb", (POINTFIELD_FLOAT32, POINTFIELD_UINT32), "FLOAT32 or UINT32")
    elif "intensity" in by_name:
        L.intensity_offset = need("intensity", (POINTFIELD_FLOAT32,), "FLOAT32")
    return L


def _device_array(a, dtype, shape_ok, device, what):
    """Pointer of a device array (anything with __cuda_array_interface__, e.g. a torch CUDA tensor) after
    checking dtype, shape, contiguity and, where the object tells, its device."""
    try:   # a torch CPU tensor has the attribute and raises from it
        cai = a.__cuda_array_interface__
    except Exception:
        raise TypeError("%s: not an array in device memory (no __cuda_array_interface__)" % what)
    if np.dtype(cai["typestr"]) != np.dtype(dtype):
        raise TypeError("%s: dtype must be %s" % (what, np.dtype(dtype).name))
    shape = tuple(cai["shape"])
    if not shape_ok(shape):
        raise ValueError("%s: bad shape %s" % (what, shape))
    if cai.get("strides") is not None:
        expect = tuple(np.dtype(dtype).itemsize * int(np.prod(shape[k + 1:])) for k in range(len(shape)))
        if tuple(cai["strides"]) != expect and int(np.prod(shape)) > 0:
            raise ValueError("%s: must be C-contiguous" % what)
    dev = getattr(getattr(a, "device", None), "index", getattr(getattr(a, "device", None), "id", None))
    if dev is not None and int(dev) != int(device):
        raise ValueError("%s: lives on device %d, the context on device %d" % (what, dev, device))
    return int(cai["data"][0]), shape


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


class Context:
    """One GPU's brick store + pose graph state (vgx_ctx)."""

    def __init__(self, device=0):
        self._L = _lib.load()
        h = C.c_void_p()
        rc = self._L.vgx_ctx_create(int(device), C.byref(h))
        if rc != 0:
            raise VgxError(rc, "vgx_ctx_create failed (a CUDA device is required; no CPU fallback)")
        self._h = h
        self.device = device

    def close(self):
        if getattr(self, "_h", None):
            self._L.vgx_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, allow=(0,)):
        if rc not in allow:
            raise VgxError(rc, self._L.vgx_last_error(self._h).decode())
        return rc

    def _sized_bytes(self, call):
        """call(out, capacity, size*) once with no buffer to learn the size, then into a bytearray of that size."""
        size = C.c_uint64(0)
        self._check(call(None, 0, C.byref(size)))
        out = bytearray(size.value)
        buf = (C.c_char * size.value).from_buffer(out) if size.value else None
        self._check(call(buf, size.value, C.byref(size)))
        return out

    # ---- stream / accounting
    @property
    def stream_ptr(self):
        return self._L.vgx_ctx_stream(self._h)

    def synchronize(self):
        self._check(self._L.vgx_ctx_synchronize(self._h))

    def profile_enable(self, on=True):
        self._check(self._L.vgx_profile_enable(self._h, int(on)))

    def profile_reset(self):
        self._check(self._L.vgx_profile_reset(self._h))

    def profile_get(self, which):
        ms = C.c_double(0); n = C.c_int64(0)
        self._check(self._L.vgx_profile_get(self._h, which, C.byref(ms), C.byref(n)))
        return ms.value, n.value

    @property
    def launch_count(self):
        return self._L.vgx_launch_count(self._h)

    # ---- submaps
    def submap_upload(self, submap_id, voxel_size, vps, block_idx, distance, weight):
        bi = np.ascontiguousarray(block_idx, dtype=np.int32).reshape(-1, 3)
        n = bi.shape[0]
        d = _f32(distance).reshape(n, vps ** 3); w = _f32(weight).reshape(n, vps ** 3)
        self._check(self._L.vgx_submap_upload(self._h, int(submap_id), float(voxel_size), int(vps), n,
                                              _p(bi, C.c_int32), _p(d, C.c_float), _p(w, C.c_float)))

    def submap_create(self, submap_id, voxel_size, vps, capacity_blocks):
        self._check(self._L.vgx_submap_create(self._h, int(submap_id), float(voxel_size), int(vps),
                                              int(capacity_blocks)))

    def submap_finish(self, submap_id):
        self._check(self._L.vgx_submap_finish(self._h, int(submap_id)))

    def submap_peek_device(self, submap_id):
        """(device pointer of block indices, device pointer of (distance, weight) voxels, n_blocks)."""
        pi = C.c_void_p(); pd = C.c_void_p(); n = C.c_int(0)
        self._check(self._L.vgx_submap_peek_device(self._h, int(submap_id), C.byref(pi), C.byref(pd), C.byref(n)))
        return pi.value, pd.value, n.value

    def submap_upload_device(self, submap_id, voxel_size, vps, n_blocks, d_block_idx_ptr, d_dw_ptr):
        self._check(self._L.vgx_submap_upload_device(self._h, int(submap_id), float(voxel_size), int(vps),
                                                     int(n_blocks), C.c_void_p(d_block_idx_ptr), C.c_void_p(d_dw_ptr)))

    # ---- voxel colour (one uint32 per voxel: a | b << 8 | g << 16 | r << 24, see include/voxgraph_b200.h)
    def submap_has_colour(self, submap_id):
        has = C.c_int(0)
        self._check(self._L.vgx_submap_has_colour(self._h, int(submap_id), C.byref(has)))
        return bool(has.value)

    def submap_download_colour(self, submap_id):
        """The colour words (n_blocks, vps^3) uint32 in the block order of submap_download; zeros when the
        submap has no colour channel."""
        _, vps, n, _ = self.submap_info(submap_id)
        out = np.zeros((n, vps ** 3), np.uint32); got = C.c_int(0)
        self._check(self._L.vgx_submap_download_colour(self._h, int(submap_id), n, _p(out, C.c_uint32), C.byref(got)))
        return out

    def submap_upload_colour(self, submap_id, rgba):
        """Give an existing submap the colour words rgba (n_blocks, vps^3) uint32."""
        _, vps, _, _ = self.submap_info(submap_id)
        w = np.ascontiguousarray(rgba, np.uint32).reshape(-1, vps ** 3)
        self._check(self._L.vgx_submap_upload_colour(self._h, int(submap_id), w.shape[0], _p(w, C.c_uint32)))

    def submap_peek_device_colour(self, submap_id):
        """Device pointer of the colour words, or None when the submap has no colour channel."""
        p = C.c_void_p()
        self._check(self._L.vgx_submap_peek_device_colour(self._h, int(submap_id), C.byref(p)))
        return p.value

    def submap_upload_device_colour(self, submap_id, n_blocks, d_rgba_ptr):
        self._check(self._L.vgx_submap_upload_device_colour(self._h, int(submap_id), int(n_blocks),
                                                            C.c_void_p(d_rgba_ptr)))

    # ---- submap collection files (cblox SubmapCollection::saveToFile / io::LoadSubmapCollection)
    @staticmethod
    def collection_scan(data):
        """Framing check of a collection stream, host only (no GPU) -> list of dicts with id,
        num_blocks, voxel_size, voxels_per_side and T_M_S ([qw qx qy qz tx ty tz], float32)."""
        buf, nbytes = _bytes_arg(data)
        n = C.c_int(0)
        _call_noctx("vgx_collection_scan", buf, nbytes, 0, None, C.byref(n), allow=(0, _lib.VGX_ERR_CAPACITY))
        out = (CollectionEntry * max(n.value, 1))()
        _call_noctx("vgx_collection_scan", buf, nbytes, n.value, out, C.byref(n))
        return [dict(id=e.id, num_blocks=e.num_blocks, voxel_size=e.voxel_size,
                     voxels_per_side=e.voxels_per_side, T_M_S=np.array(e.T_M_S[:], np.float32))
                for e in out[:n.value]]

    def collection_load(self, data, keep_colour=False):
        """Create every submap of the stream as a finished upload (all or nothing) -> submap count.
        keep_colour: a submap whose colour words are not all zero gets them as its colour channel."""
        buf, nbytes = _bytes_arg(data)
        n = C.c_int(0)
        if keep_colour:
            self._check(self._L.vgx_collection_load_ex(self._h, buf, nbytes, _lib.VGX_COLLECTION_KEEP_COLOUR,
                                                       C.byref(n)))
        else:
            self._check(self._L.vgx_collection_load(self._h, buf, nbytes, C.byref(n)))
        return n.value

    def collection_save(self, submap_ids, poses_T):
        """Serialise the submaps with poses T_M_S (n, 7) [qw qx qy qz tx ty tz] -> bytearray."""
        ids, T = _ids_poses(submap_ids, poses_T, "collection_save")
        return self._sized_bytes(lambda *a: self._L.vgx_collection_save(self._h, len(ids), _p(ids, C.c_uint32),
                                                                        _p(T, C.c_float), *a))

    # ---- submap meshes (SubmapVisuals::publishSeparatedMesh / saveSeparatedMesh)
    def mesh_config(self, **kw):
        return _config(MeshConfig, self._L.vgx_mesh_config_default, **kw)

    def mesh_build(self, submap_ids, poses_T=None, cfg=None):
        """Separated mesh of the submaps (in the order given) into the context's mesh buffer; poses_T
        (n, 7) [qw qx qy qz tx ty tz] or None (submap frames) -> (vertex_offsets, triangle_offsets),
        n + 1 entries each.  An empty list releases the buffer."""
        ids, T = _ids_poses(submap_ids, poses_T, "mesh_build", optional=True)
        vo = np.zeros(len(ids) + 1, np.int64); to = np.zeros(len(ids) + 1, np.int64)
        self._check(self._L.vgx_mesh_build(self._h, len(ids), _p(ids, C.c_uint32), _p(T, C.c_float),
                                           _ref(cfg), _p(vo, C.c_int64), _p(to, C.c_int64)))
        return vo, to

    def mesh_download(self):
        """The last build's mesh -> (xyz (V, 3) float32, triangles (T, 3) uint32)."""
        nv = C.c_int64(0); nt = C.c_int64(0)
        self._check(self._L.vgx_mesh_download(self._h, 0, None, 0, None, C.byref(nv), C.byref(nt)))
        xyz = np.zeros((nv.value, 3), np.float32); tri = np.zeros((nt.value, 3), np.uint32)
        self._check(self._L.vgx_mesh_download(self._h, nv.value, _p(xyz, C.c_float), nt.value,
                                              _p(tri, C.c_uint32), C.byref(nv), C.byref(nt)))
        return xyz, tri

    def mesh_ply(self, rgba=None, voxel_colours=False):
        """Binary PLY of the last build; rgba (n, 4) uint8 per submap or None (the default palette)
        -> bytearray.  voxel_colours: vertices of submaps with a colour channel carry their voxel colour."""
        col = np.ascontiguousarray(rgba, np.uint8).reshape(-1, 4) if rgba is not None else None
        if voxel_colours:
            return self._sized_bytes(lambda *a: self._L.vgx_mesh_ply_ex(self._h, _p(col, C.c_uint8), 1, *a))
        return self._sized_bytes(lambda *a: self._L.vgx_mesh_ply(self._h, _p(col, C.c_uint8), *a))

    def mesh_colours(self):
        """The last build's vertex colour words (V,) uint32 (the layout of submap_download_colour); 0 for the
        vertices of submaps without a colour channel."""
        nv = C.c_int64(0)
        self._check(self._L.vgx_mesh_download_colours(self._h, 0, None, C.byref(nv)))
        out = np.zeros(nv.value, np.uint32)
        self._check(self._L.vgx_mesh_download_colours(self._h, nv.value, _p(out, C.c_uint32), C.byref(nv)))
        return out

    # ---- projected global map (cblox SubmapCollection::getProjectedMap)
    def project_map(self, submap_ids, poses_T, out_id):
        """Merge the submaps at their poses T_M_S (n, 7) [qw qx qy qz tx ty tz], in increasing id order,
        into a new finished submap out_id in the mission frame -> its block count."""
        ids, T = _ids_poses(submap_ids, poses_T, "project_map")
        n = C.c_int(0)
        self._check(self._L.vgx_project_map(self._h, len(ids), _p(ids, C.c_uint32), _p(T, C.c_float),
                                            int(out_id), C.byref(n)))
        return n.value

    def mesh_build_combined(self, submap_ids, poses_T, cfg=None):
        """cblox SubmapMesher::generateCombinedMesh: the mesh of the submaps' projected map (T_M_S (n, 7)) into the
        context's mesh buffer, through a scratch submap that is freed again."""
        ids, T = _ids_poses(submap_ids, poses_T, "mesh_build_combined")
        self._check(self._L.vgx_mesh_build_combined(self._h, len(ids), _p(ids, C.c_uint32), _p(T, C.c_float),
                                                    _ref(cfg)))

    # ---- map evaluation (voxgraph MapEvaluation)
    def layer_load(self, submap_id, data):
        """voxblox::io::LoadLayer<TsdfVoxel> of a layer file's bytes into a new finished submap -> block count."""
        buf, nbytes = _bytes_arg(data)
        n = C.c_int(0)
        self._check(self._L.vgx_layer_load(self._h, int(submap_id), buf, nbytes, C.byref(n)))
        return n.value

    def submap_transform(self, submap_id, T_new_old):
        """VoxgraphSubmap::transformSubmap's layer part (voxblox transformLayer into the submap's own layer);
        T_new_old [qw qx qy qz tx ty tz].  The submap becomes a finished upload without ESDF or points."""
        T = _f32(T_new_old).reshape(7)
        self._check(self._L.vgx_submap_transform(self._h, int(submap_id), _p(T, C.c_float)))

    def evaluate_layers_rmse(self, gt_id, test_id, gt_layer=_lib.VGX_LAYER_ESDF, test_layer=_lib.VGX_LAYER_ESDF):
        """voxblox utils::evaluateLayersRmse (kIgnoreErrorBehindTestSurface) -> VoxelEvaluationDetails."""
        d = VoxelEvaluationDetails()
        self._check(self._L.vgx_evaluate_layers_rmse(self._h, int(gt_id), int(gt_layer), int(test_id),
                                                     int(test_layer), C.byref(d)))
        return d

    def map_evaluate(self, gt_id, submap_ids, poses_T):
        """MapEvaluation::evaluate: align the ground truth gt_id to the projection of the submaps at T_M_S
        (n, 7), move it there and report the RMSE -> MapEvaluationResult.  gt_id ends transformed."""
        ids, T = _ids_poses(submap_ids, poses_T, "map_evaluate")
        r = MapEvaluationResult()
        self._check(self._L.vgx_map_evaluate(self._h, int(gt_id), len(ids), _p(ids, C.c_uint32), _p(T, C.c_float),
                                             C.byref(r)))
        return r

    def registration_filter(self, **kw):
        return _config(RegistrationFilter, self._L.vgx_registration_filter_default, **kw)

    def submap_extract_points(self, submap_id, filt=None):
        """findRelevantVoxelIndices + findIsosurfaceVertices + surface OBB on the device."""
        self._check(self._L.vgx_submap_extract_points(self._h, int(submap_id), _ref(filt)))

    def submap_finish_ex(self, submap_id, filt=None):
        self._check(self._L.vgx_submap_finish_ex(self._h, int(submap_id), _ref(filt)))

    def submap_num_points(self, submap_id, point_type):
        n = C.c_int(0)
        self._check(self._L.vgx_submap_num_points(self._h, int(submap_id), int(point_type), C.byref(n)))
        return n.value

    def submap_download_points(self, submap_id, point_type):
        n = self.submap_num_points(submap_id, point_type)
        xyz = np.zeros((n, 3), np.float32); d = np.zeros(n, np.float32); w = np.zeros(n, np.float32)
        got = C.c_int(0)
        self._check(self._L.vgx_submap_download_points(self._h, int(submap_id), int(point_type), n,
                                                       _p(xyz, C.c_float), _p(d, C.c_float),
                                                       _p(w, C.c_float), C.byref(got)))
        return xyz, d, w

    def submap_surface_obb(self, submap_id):
        mn = np.zeros(3, np.float32); mx = np.zeros(3, np.float32)
        rc = self._check(self._L.vgx_submap_surface_obb(self._h, int(submap_id), _p(mn, C.c_float),
                                                        _p(mx, C.c_float)), allow=(0, 1))
        return rc == 0, mn, mx

    def esdf_config(self, **kw):
        return _config(EsdfConfig, self._L.vgx_esdf_config_default, **kw)

    def submap_generate_esdf(self, submap_id, cfg=None):
        """TsdfEsdfSubmap::generateEsdf on the device -> number of relaxation sweeps."""
        n = C.c_int(0)
        self._check(self._L.vgx_submap_generate_esdf(self._h, int(submap_id), _ref(cfg), C.byref(n)))
        return n.value

    def submap_download_esdf(self, submap_id):
        _, vps, n, _ = self.submap_info(submap_id)
        d = np.zeros((n, vps ** 3), np.float32); ob = np.zeros((n, vps ** 3), np.float32)
        got = C.c_int(0)
        self._check(self._L.vgx_submap_download_esdf(self._h, int(submap_id), n, _p(d, C.c_float),
                                                     _p(ob, C.c_float), C.byref(got)))
        return d, ob

    def find_overlapping_pairs(self, submap_ids, poses_T):
        """updateOverlappingSubmapList: poses_T (n,7) = [qw qx qy qz tx ty tz] -> list of (id_i, id_j)."""
        ids, T = _ids_poses(submap_ids, poses_T, "find_overlapping_pairs")
        cap = max(1, len(ids) * (len(ids) - 1) // 2)
        out = np.zeros((cap, 2), np.uint32); n = C.c_int(0)
        self._check(self._L.vgx_find_overlapping_pairs(self._h, len(ids), _p(ids, C.c_uint32),
                                                       _p(T, C.c_float), cap, _p(out, C.c_uint32),
                                                       C.byref(n)))
        return [tuple(int(v) for v in out[k]) for k in range(n.value)]

    def submap_free(self, submap_id):
        self._check(self._L.vgx_submap_free(self._h, int(submap_id)))

    def submap_block_count(self, submap_id):
        n = C.c_int(0)
        self._check(self._L.vgx_submap_block_count(self._h, int(submap_id), C.byref(n)))
        return n.value

    def submap_info(self, submap_id):
        """(voxel_size, voxels_per_side, n_blocks, finished)"""
        vs = C.c_float(0); vps = C.c_int(0); n = C.c_int(0); fin = C.c_int(0)
        self._check(self._L.vgx_submap_info(self._h, int(submap_id), C.byref(vs), C.byref(vps),
                                            C.byref(n), C.byref(fin)))
        return vs.value, vps.value, n.value, bool(fin.value)

    def submap_draw_samples(self, submap_id, point_type, n):
        """WeightedSampler::getRandomItem n times on the submap's generator -> indices."""
        idx = np.zeros(n, np.int32)
        self._check(self._L.vgx_submap_draw_samples(self._h, int(submap_id), int(point_type), int(n),
                                                    _p(idx, C.c_int32)))
        return idx

    def submap_download(self, submap_id):
        _, vps, n, _ = self.submap_info(submap_id)
        idx = np.zeros((n, 3), np.int32)
        d = np.zeros((n, vps ** 3), np.float32); w = np.zeros((n, vps ** 3), np.float32)
        got = C.c_int(0)
        self._check(self._L.vgx_submap_download(self._h, int(submap_id), n, _p(idx, C.c_int32),
                                                _p(d, C.c_float), _p(w, C.c_float), C.byref(got)))
        return idx, d, w

    def submap_upload_points(self, submap_id, point_type, xyz, distance, weight):
        xyz = _f32(xyz).reshape(-1, 3); distance = _f32(distance); weight = _f32(weight)
        self._check(self._L.vgx_submap_upload_points(self._h, int(submap_id), int(point_type),
                                                     xyz.shape[0], _p(xyz, C.c_float),
                                                     _p(distance, C.c_float), _p(weight, C.c_float)))

    def upload_synth_submap(self, s, point_type=K_ISOSURFACE_POINTS):
        """Upload a voxgraph_b200.synth.Submap (bricks + registration points)."""
        self.submap_upload(s.submap_id, s.voxel_size, s.vps, s.block_idx, s.distance, s.weight)
        if s.points_xyz is not None:
            self.submap_upload_points(s.submap_id, point_type, s.points_xyz, s.points_distance,
                                      s.points_weight)

    # ---- b3
    def tsdf_config(self, **kw):
        return _config(TsdfConfig, self._L.vgx_tsdf_config_default, **kw)

    def tsdf_integrate(self, submap_id, T_G_C, points_C, cfg=None, rgba=None):
        """integratePointCloud; rgba (n, 4) uint8 [r g b a] per point, or None (no colour)."""
        T = _f32(T_G_C); pts = _f32(points_C).reshape(-1, 3)
        st = TsdfStats()
        col = np.ascontiguousarray(rgba, np.uint8).reshape(-1, 4) if rgba is not None else None
        if col is not None and col.shape[0] != pts.shape[0]:
            raise ValueError("tsdf_integrate: one colour per point")
        self._check(self._L.vgx_tsdf_integrate(self._h, int(submap_id), _p(T, C.c_float), pts.shape[0],
                                               _p(pts, C.c_float), _p(col, C.c_uint8), _ref(cfg), C.byref(st)))
        return st

    def tsdf_integrate_device(self, submap_id, T_G_C, d_points_C, cfg=None, d_rgba=None):
        """tsdf_integrate with the points (n, 3) float32, and optionally the colours (n, 4) uint8 [r g b a] or (n,)
        uint32 words of those bytes, already on this context's GPU: any C-contiguous object with
        __cuda_array_interface__ (a torch CUDA tensor).  The work runs on the context's stream: whatever produced
        the arrays must have finished (torch.cuda.current_stream().synchronize())."""
        T = _f32(T_G_C)
        ptr, shape = _device_array(d_points_C, np.float32, lambda s: len(s) == 2 and s[1] == 3, self.device,
                                   "tsdf_integrate_device: points")
        n = shape[0]
        col = None
        if d_rgba is not None:
            words = getattr(d_rgba, "ndim", 2) == 1
            col, _ = _device_array(d_rgba, np.uint32 if words else np.uint8,
                                   (lambda s: s == (n,)) if words else (lambda s: s == (n, 4)), self.device,
                                   "tsdf_integrate_device: colours")
        st = TsdfStats()
        self._check(self._L.vgx_tsdf_integrate_device(self._h, int(submap_id), _p(T, C.c_float), n,
                                                      C.c_void_p(ptr if n else None), C.c_void_p(col),
                                                      _ref(cfg), C.byref(st)))
        return st

    # ---- b3, from the sensor message (PointcloudIntegrator::integratePointcloud, cpp:23-90)
    def cloud_decode(self, msg, colour_map_max=10000.0):
        """pcl::fromROSMsg + voxblox::convertPointcloud of a PointCloud2 on the device -> (points (n, 3) float32,
        colours (n, 4) uint8 [r g b a]): the records with finite coordinates, in message order."""
        L = cloud_layout(msg)
        buf, nbytes = _bytes_arg(msg.data)
        n = C.c_int(0)
        decode = lambda cap, pts, col: self._check(self._L.vgx_cloud_decode(
            self._h, C.byref(L), buf, nbytes, float(colour_map_max), cap, _p(pts, C.c_float), _p(col, C.c_uint8),
            C.byref(n)))
        decode(0, None, None)                    # validates, and counts: the outputs are sized from the answer
        pts = np.zeros((n.value, 3), np.float32); col = np.zeros((n.value, 4), np.uint8)
        if n.value:
            decode(n.value, pts, col)
        return pts, col

    def tsdf_integrate_cloud(self, submap_id, T_G_C, msg, cfg=None, colours=True, colour_map_max=10000.0):
        """Decode a PointCloud2 and integrate it, in one call on the device -> (TsdfStats, number of records with
        finite coordinates).  colours: as the reference every cloud type carries colours (rgb, the grey of its
        intensity, or black); False integrates without them and leaves the submap's colour channel alone."""
        T = _f32(T_G_C)
        L = cloud_layout(msg)
        buf, nbytes = _bytes_arg(msg.data)
        st = TsdfStats(); n = C.c_int(0)
        self._check(self._L.vgx_tsdf_integrate_cloud(self._h, int(submap_id), _p(T, C.c_float), C.byref(L), buf,
                                                     nbytes, int(bool(colours)), float(colour_map_max),
                                                     _ref(cfg), C.byref(st), C.byref(n)))
        return st, n.value

    # ---- b1
    def reg_config(self, **kw):
        return _config(RegConfig, self._L.vgx_reg_config_default, **kw)

    def reg_num_residuals(self, ref_id, cfg=None):
        cfg = cfg or self.reg_config()
        n = C.c_int(0)
        self._check(self._L.vgx_reg_num_residuals(self._h, int(ref_id), C.byref(cfg), C.byref(n)))
        return n.value

    def reg_eval_emit(self, ref_id, read_id, ref_pose, read_pose, cfg=None, jacobians=True):
        """RegistrationCostFunction::Evaluate -> (ok, residuals, J_ref, J_read)."""
        cfg = cfg or self.reg_config()
        K = self.reg_num_residuals(ref_id, cfg)
        r = np.zeros(K); jr = np.zeros((K, 4)) if jacobians else None
        je = np.zeros((K, 4)) if jacobians else None
        a = _f64(ref_pose); b = _f64(read_pose)
        rc = self._check(self._L.vgx_reg_eval_emit(self._h, int(ref_id), int(read_id), C.byref(cfg),
                                                   _p(a, C.c_double), _p(b, C.c_double),
                                                   _p(r, C.c_double), _p(jr, C.c_double),
                                                   _p(je, C.c_double)), allow=(0, 1))
        return rc == 0, r, jr, je

    # ---- b2 (raw)
    def graph_set_nodes(self, ids, xyzyaw, constant):
        ids = np.ascontiguousarray(ids, np.uint32); x = _f64(xyzyaw).reshape(-1, 4)
        cst = np.ascontiguousarray(constant, np.uint8)
        self._check(self._L.vgx_graph_set_nodes(self._h, len(ids), _p(ids, C.c_uint32),
                                                _p(x, C.c_double), _p(cst, C.c_uint8)))

    def graph_set_poses(self, xyzyaw):
        x = _f64(xyzyaw)
        self._check(self._L.vgx_graph_set_poses(self._h, _p(x, C.c_double)))

    def graph_get_poses(self, n):
        x = np.zeros((n, 4))
        self._check(self._L.vgx_graph_get_poses(self._h, _p(x, C.c_double)))
        return x

    def graph_set_relative_edges(self, ids_a, ids_b, t_obs_xyzyaw, sqrt_info):
        a = np.ascontiguousarray(ids_a, np.uint32); b = np.ascontiguousarray(ids_b, np.uint32)
        t = _f64(t_obs_xyzyaw).reshape(-1, 4); L = _f64(sqrt_info).reshape(-1, 16)
        self._check(self._L.vgx_graph_set_relative_edges(self._h, len(a), _p(a, C.c_uint32),
                                                         _p(b, C.c_uint32), _p(t, C.c_double),
                                                         _p(L, C.c_double)))

    def graph_set_registration_constraints(self, ref_ids, read_ids, cfg=None):
        a = np.ascontiguousarray(ref_ids, np.uint32); b = np.ascontiguousarray(read_ids, np.uint32)
        cfg = cfg or self.reg_config()
        self._check(self._L.vgx_graph_set_registration_constraints(self._h, len(a), _p(a, C.c_uint32),
                                                                   _p(b, C.c_uint32), C.byref(cfg)))

    def graph_set_registration_constraints_v(self, ref_ids, read_ids, cfgs):
        a = np.ascontiguousarray(ref_ids, np.uint32); b = np.ascontiguousarray(read_ids, np.uint32)
        arr = (RegConfig * len(a))(*cfgs)
        self._check(self._L.vgx_graph_set_registration_constraints_v(self._h, len(a), _p(a, C.c_uint32),
                                                                     _p(b, C.c_uint32), arr))

    def graph_get_sample_indices(self, constraint, max_n):
        idx = np.zeros(max(max_n, 1), np.int32); n = C.c_int(0)
        self._check(self._L.vgx_graph_get_sample_indices(self._h, int(constraint), int(max_n),
                                                         _p(idx, C.c_int32), C.byref(n)))
        return idx[:n.value].copy()

    def graph_set_sample_indices(self, constraint, indices):
        idx = np.ascontiguousarray(indices, np.int32)
        self._check(self._L.vgx_graph_set_sample_indices(self._h, int(constraint), len(idx),
                                                         _p(idx, C.c_int32)))

    def graph_num_registration_residuals(self):
        a = C.c_int64(0); b = C.c_int64(0)
        self._check(self._L.vgx_graph_num_registration_residuals(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def graph_eval(self, n_nodes, exclude_registration=False, want_H=True):
        dim = 4 * n_nodes
        cost = C.c_double(0); g = np.zeros(dim); H = np.zeros((dim, dim)) if want_H else None
        rc = self._check(self._L.vgx_graph_eval(self._h, int(exclude_registration), C.byref(cost),
                                                _p(g, C.c_double), _p(H, C.c_double)), allow=(0, 1))
        return rc == 0, cost.value, g, H

    def graph_eval_async(self, exclude_registration=False):
        self._check(self._L.vgx_graph_eval_async(self._h, int(exclude_registration)))

    def graph_registration_costs(self, n_constraints):
        out = np.zeros(n_constraints)
        self._check(self._L.vgx_graph_registration_costs(self._h, _p(out, C.c_double)))
        return out

    def graph_edge_covariances(self, ids_a, ids_b):
        a = np.ascontiguousarray(ids_a, np.uint32); b = np.ascontiguousarray(ids_b, np.uint32)
        cov = np.zeros((len(a), 4, 4))
        self._check(self._L.vgx_graph_edge_covariances(self._h, len(a), _p(a, C.c_uint32), _p(b, C.c_uint32),
                                                       _p(cov, C.c_double)))
        return cov

    def solver_options(self, **kw):
        return _config(SolverOptions, self._L.vgx_solver_options_default, **kw)

    def graph_solve(self, n_nodes, options=None):
        o = options or self.solver_options()
        x = np.zeros((n_nodes, 4)); s = SolverSummary()
        self._check(self._L.vgx_graph_solve(self._h, C.byref(o), _p(x, C.c_double), C.byref(s)))
        return x, s

    # ---- multi-GPU
    def comm_suspend(self, on=True):
        """Behave as a single-rank context (full problem locally, no exchange) while on."""
        self._check(self._L.vgx_comm_suspend(self._h, int(bool(on))))

    def comm_init(self, nranks, rank, unique_id):
        u = np.ascontiguousarray(unique_id, np.uint8)
        if u.size != 128:
            raise ValueError("comm_init: the unique id has 128 bytes")
        self._check(self._L.vgx_comm_init(self._h, int(nranks), int(rank), _p(u, C.c_uint8)))

    def comm_p2p_export(self, capacity_doubles):
        h = np.zeros(64, np.uint8)
        self._check(self._L.vgx_comm_p2p_export(self._h, int(capacity_doubles), _p(h, C.c_uint8)))
        return h

    def comm_p2p_import(self, nranks, rank, handles):
        hs = np.ascontiguousarray(handles, np.uint8).reshape(-1)
        if hs.size != 64 * nranks:
            raise ValueError("comm_p2p_import: 64 handle bytes per rank")
        self._check(self._L.vgx_comm_p2p_import(self._h, int(nranks), int(rank), _p(hs, C.c_uint8)))


def p2p_setup(ctx, nranks, rank, all_gather_bytes, capacity_doubles=1 << 20):
    """Bring up the NVLink peer exchange: export this rank's buffer, all-gather the 64-byte IPC
    handles with the caller's collective (all_gather_bytes(np.uint8[64]) -> np.uint8[nranks, 64]),
    map the peers."""
    h = ctx.comm_p2p_export(capacity_doubles)
    handles = np.ascontiguousarray(all_gather_bytes(h), np.uint8).reshape(nranks, 64)
    ctx.comm_p2p_import(nranks, rank, handles)


def shard_constraints(nranks, num_residuals, locality_keys=None):
    """Constraint -> rank partition used by the library (host only, no GPU needed)."""
    cnt = np.ascontiguousarray(num_residuals, np.int32)
    owner = np.zeros(len(cnt), np.int32)
    keys = np.ascontiguousarray(locality_keys, np.uint32) if locality_keys is not None else None
    _call_noctx("vgx_shard_constraints", int(nranks), len(cnt), _p(cnt, C.c_int32), _p(keys, C.c_uint32),
                _p(owner, C.c_int32))
    return owner


def grayscale_colours(intensity, max_value=10000.0):
    """The colours PointcloudIntegrator gives an XYZI cloud (pointcloud_integrator.cpp:12-14: a voxblox
    GrayscaleColorMap with max value 10000).  Restated from the published voxblox sources, not checked
    against a compiled voxblox: h = clamp(intensity, 0, max) / max in float, every channel round(h * 255)
    in double, alpha 255 -> (n, 4) uint8 [r g b a]."""
    x = np.asarray(intensity, np.float32).reshape(-1)
    h = np.clip(x, np.float32(0), np.float32(max_value)) / np.float32(max_value)
    g = np.floor(h.astype(np.float64) * 255.0 + 0.5).astype(np.uint8)
    return np.stack([g, g, g, np.full_like(g, 255)], -1)


def load_submap_collection(ctx, path, keep_colour=False):
    """cblox::io::LoadSubmapCollection: create the file's submaps in ctx (TSDF only; run
    submap_finish_ex / submap_generate_esdf as finishSubmap does) -> (ids uint32 (n,), poses T_M_S
    float32 (n, 7) [qw qx qy qz tx ty tz]).  keep_colour: as Context.collection_load."""
    with open(path, "rb") as f:
        data = f.read()
    entries = Context.collection_scan(data)
    ctx.collection_load(data, keep_colour)
    ids = np.array([e["id"] for e in entries], np.uint32)
    poses = np.array([e["T_M_S"] for e in entries], np.float32).reshape(-1, 7)
    return ids, poses


def save_submap_collection(ctx, path, submap_ids, poses_T):
    """cblox::SubmapCollection::saveToFile: the submaps with their poses T_M_S (n, 7)."""
    data = ctx.collection_save(submap_ids, poses_T)
    with open(path, "wb") as f:
        f.write(data)
    return len(data)


def separated_mesh(ctx, submap_ids, poses_T=None, min_weight=2.0):
    """cblox SubmapMesher::generateSeparatedMesh on the device -> (xyz (V, 3) float32 in the mission
    frame, triangles (T, 3) uint32, vertex_offsets (n + 1,), triangle_offsets (n + 1,))."""
    vo, to = ctx.mesh_build(submap_ids, poses_T, ctx.mesh_config(min_weight=min_weight))
    xyz, tri = ctx.mesh_download()
    return xyz, tri, vo, to


def save_separated_mesh(ctx, path, submap_ids, poses_T, colours=None, min_weight=2.0):
    """SubmapVisuals::saveSeparatedMesh: the submaps at poses T_M_S (n, 7) as a binary PLY, one colour
    per submap (rgba (n, 4); default: the library's palette, voxblox rainbowColorMap((id mod 20) / 20)).
    Returns the file size in bytes."""
    ctx.mesh_build(submap_ids, poses_T, ctx.mesh_config(min_weight=min_weight))
    data = ctx.mesh_ply(colours)
    with open(path, "wb") as f:
        f.write(data)
    return len(data)


def combined_mesh(ctx, submap_ids, poses_T, min_weight=2.0):
    """cblox SubmapMesher::generateCombinedMesh on the device: the mesh of the projected global map (one
    surface where submaps overlap) -> (xyz (V, 3) float32 in the mission frame, triangles (T, 3) uint32)."""
    ctx.mesh_build_combined(submap_ids, poses_T, ctx.mesh_config(min_weight=min_weight))
    return ctx.mesh_download()


def save_combined_mesh(ctx, path, submap_ids, poses_T, colour=None, min_weight=2.0):
    """voxgraph's save_combined_mesh service: the combined mesh as a binary PLY, as SubmapVisuals::saveCombinedMesh
    writes it: the voxel colours of the projected map where a submap had a colour channel, else the one colour
    given (rgba, default opaque white).  Returns the file size in bytes."""
    ctx.mesh_build_combined(submap_ids, poses_T, ctx.mesh_config(min_weight=min_weight))
    rgba = np.array([255, 255, 255, 255] if colour is None else colour, np.uint8).reshape(1, 4)
    data = ctx.mesh_ply(rgba, voxel_colours=True)
    with open(path, "wb") as f:
        f.write(data)
    return len(data)


@dataclass
class EvaluationDetails:
    """MapEvaluation::EvaluationDetails: the voxblox evaluation details and T_ground_truth__reading
    ([qw qx qy qz tx ty tz], float32), plus the aligned pose and the alignment's solver summary."""
    reconstruction: VoxelEvaluationDetails
    T_ground_truth__reading: np.ndarray
    aligned_pose: np.ndarray = None
    summary: SolverSummary = None


class MapEvaluation:
    """voxgraph MapEvaluation (src/tools/evaluation/map_evaluation.cpp): loads the ground-truth TSDF layer
    file into submap gt_id of ctx; evaluate() aligns it to the projected map of the submaps and reports the
    RMSE.  As in the reference the ground truth stays where the alignment moved it, so a second evaluate()
    starts from there."""

    def __init__(self, ctx, ground_truth_tsdf_file_path, gt_id):
        self.ctx = ctx
        self.gt_id = int(gt_id)
        with open(ground_truth_tsdf_file_path, "rb") as f:
            ctx.layer_load(self.gt_id, f.read())

    def evaluate(self, submap_ids, poses_T):
        r = self.ctx.map_evaluate(self.gt_id, submap_ids, poses_T)
        return EvaluationDetails(reconstruction=r.details,
                                 T_ground_truth__reading=np.array(r.T_ground_truth__reading[:], np.float32),
                                 aligned_pose=np.array(r.aligned_pose[:], np.float64), summary=r.summary)


def comm_unique_id():
    u = np.zeros(128, np.uint8)
    _call_noctx("vgx_comm_unique_id", _p(u, C.c_uint8))
    return u


# --------------------------------------------------------------------------- PoseGraph mirror
@dataclass
class SubmapNodeConfig:        # SubmapNode::Config (submap_node.h:16-18, node.h:17-21)
    submap_id: int
    T_mission_node_initial: np.ndarray  # [x, y, z, yaw] (Pose4D, pose_4d.cpp:4-11)
    set_constant: bool = False


@dataclass
class RelativePoseConstraintConfig:   # relative_pose_constraint.h:13-18
    origin_submap_id: int
    destination_submap_id: int
    T_origin_destination: np.ndarray  # [tx, ty, tz, yaw]
    information_matrix: np.ndarray = field(default_factory=lambda: np.eye(4))


@dataclass
class ReferenceFrameNodeConfig:       # ReferenceFrameNode::Config (reference_frame_node.h:15-17)
    reference_frame_id: int
    T_mission_node_initial: np.ndarray = field(default_factory=lambda: np.zeros(4))
    set_constant: bool = True


@dataclass
class AbsolutePoseConstraintConfig:   # absolute_pose_constraint.h:13-18
    reference_frame_id: int
    submap_id: int
    T_ref_submap: np.ndarray          # [tx, ty, tz, yaw]
    information_matrix: np.ndarray = field(default_factory=lambda: np.eye(4))
    allow_semi_definite_information_matrix: bool = False


def sqrt_information_matrix(information_matrix, allow_semi_definite=False):
    """Constraint ctor (constraint.cpp:4-38): the LLT lower factor, or for semi-definite matrices
    Eigen's pivoted LDLT, sqrt = P^T L sqrt(D) P (vgx_sqrt_information). Raises like the reference CHECKs."""
    info = _f64(information_matrix).reshape(4, 4)
    S = np.zeros((4, 4))
    rc = _lib.load().vgx_sqrt_information(_p(info, C.c_double), int(bool(allow_semi_definite)), _p(S, C.c_double))
    if rc != _lib.VGX_OK:
        raise ValueError("The information matrix must be positive semi-definite" if allow_semi_definite else
                         "The square root of the information matrix could not be computed, "
                         "make sure it is symmetric and positive definite")
    return S


FRAME_NODE_ID_BASE = 0x80000000   # reference-frame nodes share the C-ABI's uint32 node id space


@dataclass
class RegistrationConstraintConfig:   # registration_constraint.h:15-21
    first_submap_id: int
    second_submap_id: int
    registration_point_type: int = K_ISOSURFACE_POINTS
    no_correspondence_cost: float = 0.0
    sampling_ratio: float = -1.0
    information_matrix: np.ndarray = field(default_factory=lambda: np.eye(4))
    use_esdf_distance: bool = False       # registration_cost_function.h:35 (reference default true)


class PoseGraph:
    """voxgraph::PoseGraph over the GPU path (pose_graph.h:15-65). Submaps are referred to by id
    and must have been uploaded to the Context (bricks + registration points)."""

    def __init__(self, ctx):
        self.ctx = ctx
        self._nodes = {}
        self._frames = set()
        self._relative = []
        self._registration = []   # (ref_id, read_id) residual blocks, mirrored ones included
        self._reg_cfgs = []       # one RegistrationCostFunction::Config per residual block
        self._dirty = True
        self.solver_summaries = []
        self.solver_options = ctx.solver_options()   # pose_graph.cpp:91-97 defaults

    def addSubmapNode(self, config):
        self._nodes[int(config.submap_id)] = [np.asarray(config.T_mission_node_initial, np.float64).copy(),
                                              bool(config.set_constant)]
        self._dirty = True

    def hasSubmapNode(self, submap_id):
        return int(submap_id) in self._nodes

    def addReferenceFrameNode(self, config):
        """pose_graph.cpp:21-24; the frame node lives at id FRAME_NODE_ID_BASE + frame id."""
        nid = FRAME_NODE_ID_BASE + int(config.reference_frame_id)
        self._nodes[nid] = [np.asarray(config.T_mission_node_initial, np.float64).copy(),
                            bool(config.set_constant)]
        self._frames.add(int(config.reference_frame_id))
        self._dirty = True

    def hasReferenceFrameNode(self, frame_id):
        return int(frame_id) in self._frames

    def addAbsolutePoseConstraint(self, config):
        """pose_graph.cpp:33-39 + absolute_pose_constraint.cpp:6-35: a RelativePoseCostFunction between
        the reference-frame node and the submap node (e.g. the height constraint, information zz only)."""
        if int(config.reference_frame_id) not in self._frames:
            raise ValueError("Graph contains no reference frame node %d" % int(config.reference_frame_id))
        if int(config.submap_id) not in self._nodes:
            raise ValueError("Graph contains no node for submap %d" % int(config.submap_id))
        L = sqrt_information_matrix(config.information_matrix,
                                    config.allow_semi_definite_information_matrix)
        self._relative.append((FRAME_NODE_ID_BASE + int(config.reference_frame_id), int(config.submap_id),
                               np.asarray(config.T_ref_submap, np.float64).copy(), L))
        self._dirty = True

    def addRelativePoseConstraint(self, config):
        # Constraint ctor (constraint.cpp:8-14): LLT lower factor, CHECK on failure
        L = sqrt_information_matrix(config.information_matrix,
                                    getattr(config, "allow_semi_definite_information_matrix", False))
        self._relative.append((int(config.origin_submap_id), int(config.destination_submap_id),
                               np.asarray(config.T_origin_destination, np.float64).copy(), L))
        self._dirty = True

    def addRegistrationConstraint(self, config):
        a, b = int(config.first_submap_id), int(config.second_submap_id)
        if a == b:   # pose_graph.cpp:50-51
            raise ValueError("Cannot constrain submap %d to itself" % a)
        for s in (a, b):   # pose_graph.cpp:54-57
            if s not in self._nodes:
                raise ValueError("Graph contains no node for submap %d" % s)
        if not np.array_equal(np.asarray(config.information_matrix), np.eye(4)):
            raise ValueError("Registration constraint information matrices that differ from the "
                             "identity matrix are not yet supported.")   # registration_constraint.h:32-34
        cfg = self.ctx.reg_config(registration_point_type=int(config.registration_point_type),
                                  no_correspondence_cost=float(config.no_correspondence_cost),
                                  sampling_ratio=float(config.sampling_ratio),
                                  use_esdf_distance=int(bool(getattr(config, "use_esdf_distance", False))))
        self._registration.append((a, b)); self._reg_cfgs.append(cfg)
        if config.registration_point_type == K_ISOSURFACE_POINTS:   # pose_graph.cpp:63-71
            self._registration.append((b, a)); self._reg_cfgs.append(cfg)
        self._dirty = True

    def resetRegistrationConstraints(self):
        self._registration = []
        self._reg_cfgs = []
        self._dirty = True

    def _sync(self):
        ids = sorted(self._nodes)
        if self._dirty:
            x = np.array([self._nodes[i][0] for i in ids]).reshape(-1, 4)
            cst = np.array([self._nodes[i][1] for i in ids], np.uint8)
            self.ctx.graph_set_nodes(ids, x, cst)
            if self._relative:
                self.ctx.graph_set_relative_edges([r[0] for r in self._relative],
                                                  [r[1] for r in self._relative],
                                                  np.array([r[2] for r in self._relative]),
                                                  np.array([r[3] for r in self._relative]))
            if self._registration:
                self.ctx.graph_set_registration_constraints_v([r[0] for r in self._registration],
                                                              [r[1] for r in self._registration],
                                                              self._reg_cfgs)
            self._dirty = False
        return ids

    def optimize(self, exclude_registration_constraints=False):
        ids = self._sync()
        o = self.solver_options
        o.exclude_registration = int(exclude_registration_constraints)
        x, s = self.ctx.graph_solve(len(ids), o)
        for k, i in enumerate(ids):
            self._nodes[i][0] = x[k].copy()
        self.solver_summaries.append(s)
        return s

    def evaluate(self, exclude_registration_constraints=False, want_H=True):
        ids = self._sync()
        return self.ctx.graph_eval(len(ids), exclude_registration_constraints, want_H)

    def getSubmapPoses(self):
        return {i: v[0].copy() for i, v in self._nodes.items() if i < FRAME_NODE_ID_BASE}

    def getEdgeCovarianceMap(self, submap_id_pairs):
        """pose_graph.cpp:117-163: {(first, second): 4x4 covariance} for the requested pairs."""
        self._sync()
        pairs = [(int(a), int(b)) for (a, b) in submap_id_pairs]
        cov = self.ctx.graph_edge_covariances([p[0] for p in pairs], [p[1] for p in pairs])
        return {p: cov[k] for k, p in enumerate(pairs)}

    def getSolverSummaries(self):
        return self.solver_summaries

    def getVisualizationEdgeResiduals(self):
        """Summed squared residual per registration residual block (pose_graph.cpp:194-207)."""
        self._sync()
        return self.ctx.graph_registration_costs(len(self._registration))

    @property
    def registration_blocks(self):
        return list(self._registration)
