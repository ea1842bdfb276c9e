"""ctypes front-end of tests/project_colour_oracle.c, the CPU restatement of the colour of the projected map
(rules: interpolate every channel like the distance and truncate; blend in the merge).  Compiled on first use into
a temporary directory and linked against oracle/libvg_oracle.so."""
import ctypes as C

import numpy as np

import project_oracle as po
from oracle import oracle as o
from support import build_oracle_harness

# its prototype is in tests/oracle_harness.h
SIGNATURES = {"vgpc_project_colour": (None, [C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_float, C.c_int,
                                             C.POINTER(C.c_float), C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_uint8),
                                             C.POINTER(C.c_uint32), C.POINTER(C.c_float)])}
_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = build_oracle_harness("project_colour_oracle.c", "libvg_project_colour_oracle.so", SIGNATURES)
    return _lib


def channel_layers(vs, vps, idx, weight, words):
    """The four oracle Layers whose distances are the bytes of the colour words (as floats), weights the submap's."""
    w = np.asarray(words, np.uint32).reshape(len(idx), -1)
    return [o.Layer.from_blocks(vs, vps, idx, ((w >> (8 * k)) & 255).astype(np.float32), weight) for k in range(4)]


def project(vs, vps, submaps, poses_T, ids, block_idx):
    """submaps [(idx, d, w, words or None)], poses T_M_S (n, 7), ids (n,), output blocks (B, 3) -> (colour words
    (B, vps^3) uint32, weights (B, vps^3) float32), the submaps merged in increasing id order.  Which output
    blocks a submap's transformed layer holds comes from project_oracle on that submap alone."""
    order = np.argsort(np.asarray(ids, np.uint32), kind="stable")
    T = np.ascontiguousarray(np.asarray(poses_T, np.float32).reshape(-1, 7)[order])
    layers, chans = [], []
    for k in order:
        idx, d, w, words = submaps[k]
        layers.append(o.Layer.from_blocks(vs, vps, idx, d, w))
        chans += channel_layers(vs, vps, idx, w, words) if words is not None else [None] * 4
    n = len(layers)
    bi = np.ascontiguousarray(block_idx, np.int32).reshape(-1, 3)
    holds = np.zeros((n, len(bi)), np.uint8)
    for s in range(n):
        own = set(map(tuple, po.project_layers([layers[s]], T[s:s + 1], [0]).export()[0].tolist()))
        holds[s] = [tuple(b) in own for b in bi.tolist()]
    hs = (C.c_void_p * n)(*[l._h for l in layers])
    cs = (C.c_void_p * (4 * n))(*[(c._h if c is not None else None) for c in chans])
    out = np.zeros((len(bi), vps ** 3), np.uint32); ow = np.zeros((len(bi), vps ** 3), np.float32)
    lib().vgpc_project_colour(n, hs, cs, float(np.float32(vs)), int(vps), T.ctypes.data_as(C.POINTER(C.c_float)),
                              len(bi), bi.ctypes.data_as(C.POINTER(C.c_int32)), holds.ctypes.data_as(C.POINTER(C.c_uint8)),
                              out.ctypes.data_as(C.POINTER(C.c_uint32)), ow.ctypes.data_as(C.POINTER(C.c_float)))
    return out, ow
