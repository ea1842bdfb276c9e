"""ctypes front-end of tests/transform_oracle.c, the CPU restatement of voxblox transformLayer into a submap's
own layer (VoxgraphSubmap::transformSubmap) that vgx_submap_transform is checked against.  Compiled on first use
into a temporary directory (never into the tree) and linked against oracle/libvg_oracle.so."""
import ctypes as C

import numpy as np

from oracle import oracle as o
from support import build_oracle_harness

# its prototype is in tests/oracle_harness.h
SIGNATURES = {"vgt_transform_layer": (C.c_void_p, [C.c_void_p, C.c_float, C.c_int, C.POINTER(C.c_float)])}
_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = build_oracle_harness("transform_oracle.c", "libvg_transform_oracle.so", SIGNATURES)
    return _lib


def transform_layer(layer, T_new_old):
    """transformLayer(layer copy, T_new_old, &layer) -> a new oracle Layer, blocks in ascending packed key
    order.  Raises ValueError where a candidate block index leaves the accepted range."""
    T = np.ascontiguousarray(T_new_old, np.float32).reshape(7)
    h = lib().vgt_transform_layer(layer._h, layer.voxel_size, layer.vps, T.ctypes.data_as(C.POINTER(C.c_float)))
    if not h:
        raise ValueError("vgt_transform_layer refused the input")
    return o.Layer.adopt(h, layer.voxel_size, layer.vps)
