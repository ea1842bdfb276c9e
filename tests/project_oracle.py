"""ctypes front-end of tests/project_oracle.c, the CPU restatement of cblox SubmapCollection::getProjectedMap
that vgx_project_map is checked against.  The C file is compiled on first use into a temporary directory
(never into the tree) and linked against oracle/libvg_oracle.so, whose layers it reads."""
import ctypes as C

import numpy as np

from oracle import oracle as o
from support import build_oracle_harness

# its prototype is in tests/oracle_harness.h
SIGNATURES = {"vgp_project_layers": (C.c_void_p, [C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_float),
                                                  C.POINTER(C.c_int), C.POINTER(C.c_float), C.POINTER(C.c_uint32)])}
_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = build_oracle_harness("project_oracle.c", "libvg_project_oracle.so", SIGNATURES)
    return _lib


def project_layers(layers, poses_T, ids):
    """SubmapCollection::getProjectedMap: the oracle Layers merged at their poses T_M_S (n, 7) [qw qx qy qz tx
    ty tz] in increasing id order -> a new oracle Layer, blocks in ascending packed key order.  Raises
    ValueError where the restatement refuses (no layer, repeated id, mixed geometry, index out of range)."""
    T = np.ascontiguousarray(poses_T, np.float32).reshape(-1, 7)
    ids = np.ascontiguousarray(ids, np.uint32).reshape(-1)
    n = len(layers)
    if T.shape[0] != n or ids.shape[0] != n:
        raise ValueError("project_layers: one pose and one id per layer")
    hs = (C.c_void_p * max(n, 1))(*[l._h for l in layers])
    vs = np.array([l.voxel_size for l in layers] or [0], np.float32)
    vps = np.array([l.vps for l in layers] or [0], np.intc)
    h = lib().vgp_project_layers(n, hs, vs.ctypes.data_as(C.POINTER(C.c_float)),
                                 vps.ctypes.data_as(C.POINTER(C.c_int)), T.ctypes.data_as(C.POINTER(C.c_float)),
                                 ids.ctypes.data_as(C.POINTER(C.c_uint32)))
    if not h:
        raise ValueError("vgp_project_layers refused the input")
    return o.Layer.adopt(h, layers[0].voxel_size, layers[0].vps)
