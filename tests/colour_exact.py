"""Exact numpy-float32 models of the voxel colour rules (csrc/colour.cuh, csrc/tsdf.cu), for
tests/test_oracle_colour.py, tests/test_gpu_tsdf_exact.py and tests/test_gpu_colour*.py.  The rules are
restated from the published voxblox sources; like the kernels they have not been checked against a compiled
voxblox.

* `pack`: r, g, b, a bytes -> the stored word  a | b << 8 | g << 16 | r << 24  (the third word of a voxel
  in a collection file).  `colours`: test colours whose four channels differ.
* `blend`: Color::blendTwoColors.
* `trace_rays`: the oracle's statistics and update trace with the ray each tuple belongs to (one oracle
  call per point: in mode 0, and in mode 1 with every ray cast, the rays do not interact except through
  the voxels).
* `replay`: updateTsdfVoxel's colour rule applied voxel by voxel in ray order next to tsdf_exact's
  (distance, weight) update: the sequential coloured integrator.  `expected_words` lays its result out
  as a downloaded layer's colour words.
* `merge`: mergeVoxelAIntoVoxelB's colour and weight.  `interp_channels`: Interpolator::interpVoxel's colour from
  the 8 neighbour words and the offset of the point in the cell.  `containing_voxel` / `vertex_colours`:
  MeshIntegrator::updateMeshColor's rule, the colour of the voxel that contains a vertex.
"""
import numpy as np

import tsdf_exact as tx

F32 = np.float32
_EPS = F32(1e-6)


def pack(rgba):
    """(n, 4) uint8 [r g b a] -> (n,) uint32 stored words."""
    c = np.asarray(rgba, np.uint8).reshape(-1, 4).astype(np.uint32)
    return (c[:, 3] | (c[:, 2] << 8) | (c[:, 1] << 16) | (c[:, 0] << 24)).astype(np.uint32)


def unpack(words):
    """(n,) uint32 stored words -> (n, 4) uint8 [r g b a]."""
    w = np.asarray(words, np.uint32).reshape(-1)
    return np.stack([w >> 24, (w >> 16) & 255, (w >> 8) & 255, w & 255], -1).astype(np.uint8)


def colours(rs, n):
    """n colours [r g b a] from the RandomState rs, the four channels of each one distinct."""
    return np.argsort(rs.rand(n, 256), 1)[:, :4].astype(np.uint8)


def blend(c1, w1, c2, w2):
    """blendTwoColors elementwise: t = w1 + w2; w1 /= t; w2 /= t; channel = (uint8) round(c1 w1 + c2 w2) with
    round half away from zero; clamped to [0, 255], NaN -> 0 (vgx_colour_blend)."""
    c1 = np.asarray(c1, np.uint32); c2 = np.asarray(c2, np.uint32)
    w1 = np.asarray(w1, F32); w2 = np.asarray(w2, F32)
    with np.errstate(all="ignore"):
        t = (w1 + w2).astype(F32)
        a = (w1 / t).astype(F32); b = (w2 / t).astype(F32)
        out = np.zeros(np.broadcast(c1, c2, a).shape, np.uint32)
        for sh in (0, 8, 16, 24):
            x = ((c1 >> sh) & 255).astype(F32); y = ((c2 >> sh) & 255).astype(F32)
            v = ((x * a).astype(F32) + (y * b).astype(F32)).astype(F32)
            r = np.floor(v.astype(np.float64) + 0.5)          # v >= 0: half away from zero, exact in double
            r = np.where(np.isnan(r), 0.0, np.clip(r, 0.0, 255.0))
            out |= r.astype(np.uint32) << sh
    return out


def colour_step(trunc, sdf, uw, vw, ray, colour):
    """The colour rule of one update, elementwise; vw = the weights before the update."""
    with np.errstate(all="ignore"):
        live = ~((vw + uw).astype(F32) < _EPS) & (np.abs(sdf) < F32(trunc))
    return np.where(live, blend(colour, vw, ray, uw), colour).astype(np.uint32)


def trace_rays(oracle, layer, cfg, T, pts):
    """oracle.tsdf_integrate_trace point by point (it integrates into `layer`) -> ((rays_valid, rays_cast,
    voxel_updates, blocks_allocated) summed over the points, g (m, 3), sdf (m,), uw (m,), ray (m,) point index)."""
    pts = np.asarray(pts, F32).reshape(-1, 3)
    st = np.zeros(4, np.int64)
    G, S, U, R = [np.zeros((0, 3), np.int64)], [np.zeros(0, F32)], [np.zeros(0, F32)], [np.zeros(0, np.int64)]
    for i in range(len(pts)):
        o, g, s, u = oracle.tsdf_integrate_trace(layer, cfg, T, pts[i:i + 1])
        st += (o.rays_valid, o.rays_cast, o.voxel_updates, o.blocks_allocated)
        G.append(g); S.append(s); U.append(u); R.append(np.full(len(s), i, np.int64))
    return tuple(int(v) for v in st), np.concatenate(G), np.concatenate(S), np.concatenate(U), np.concatenate(R)


class State(tx.State):
    """tsdf_exact.State with the colour word of every voxel touched so far."""

    def __init__(self):
        super().__init__()
        self.c = np.zeros(0, np.uint32)

    def get_colour(self, keys):
        c = np.zeros(len(keys), np.uint32)
        if len(self.keys):
            pos = np.minimum(np.searchsorted(self.keys, keys), len(self.keys) - 1)
            hit = self.keys[pos] == keys
            c[hit] = self.c[pos[hit]]
        return c

    def put_colour(self, keys, d, w, c):
        k = np.concatenate([keys, self.keys])
        cc = np.concatenate([c, self.c])
        _, first = np.unique(k, return_index=True)
        self.put(keys, d, w)
        self.c = cc[first]


def replay(keys, sdf, uw, ray_words, trunc, max_weight, state):
    """Apply the tuples (voxel key, sdf, uw, ray colour word) voxel by voxel in the listed (ray) order, starting
    from `state` (a State), which receives the results.  Returns (voxel keys, distance, weight, colour)."""
    keys = np.asarray(keys, np.int64); sdf = np.asarray(sdf, F32); uw = np.asarray(uw, F32)
    ray_words = np.asarray(ray_words, np.uint32)
    trunc = F32(trunc); M = F32(max_weight)
    o = np.argsort(keys, kind="stable")
    k, s, u, rw = keys[o], sdf[o], uw[o], ray_words[o]
    uniq, start, cnt = np.unique(k, return_index=True, return_counts=True)
    d0, w0 = state.get(uniq)
    c0 = state.get_colour(uniq)
    by = np.argsort(-cnt, kind="stable")
    cnt_s, start_s = cnt[by], start[by]
    dd, ww, cc = d0[by].copy(), w0[by].copy(), c0[by].copy()
    neg = -cnt_s
    for r in range(int(cnt_s[0]) if len(cnt_s) else 0):
        n = int(np.searchsorted(neg, -r, side="left"))   # voxels with more than r updates
        j = start_s[:n] + r
        b = np.nonzero(np.abs(s[j]) < trunc)[0]     # colour_step changes nothing outside the band
        if b.size:
            cc[b] = colour_step(trunc, s[j[b]], u[j[b]], ww[b], rw[j[b]], cc[b])
        dd[:n], ww[:n] = tx.apply_update(s[j], u[j], dd[:n], ww[:n], trunc, M)
    inv = np.empty_like(by); inv[by] = np.arange(len(by))
    d_out, w_out, c_out = dd[inv], ww[inv], cc[inv]
    state.put_colour(uniq, d_out, w_out, c_out)
    return uniq, d_out, w_out, c_out


def layer_colours(idx, words, vps):
    """Downloaded block indices and colour words -> (voxel keys, words), sorted by key (as tx.layer_voxels)."""
    idx = np.asarray(idx, np.int64).reshape(-1, 3)
    lin = np.arange(vps ** 3)
    loc = np.stack([lin % vps, (lin // vps) % vps, lin // (vps * vps)], -1)
    k = tx.voxel_keys((idx[:, None, :] * vps + loc[None]).reshape(-1, 3))
    o = np.argsort(k, kind="stable")
    return k[o], np.asarray(words, np.uint32).reshape(-1)[o]


def expected_words(idx, vps, state):
    """The colours of `state` (a State) laid out as the voxels of the downloaded blocks `idx` sorted by key (as
    layer_colours); 0 where never touched.  Every voxel of `state` must lie in those blocks."""
    keys = layer_colours(idx, np.zeros((len(idx), vps ** 3), np.uint32), vps)[0]
    exp = np.zeros(len(keys), np.uint32)
    pos = np.searchsorted(keys, state.keys)
    assert np.array_equal(keys[pos], state.keys)
    exp[pos] = state.c
    return exp


def merge(cA, wA, cB, wB):
    """mergeVoxelAIntoVoxelB elementwise -> (colourB, weightB): w = wA + wB; if w > 0 the blend and w."""
    wA = np.asarray(wA, F32); wB = np.asarray(wB, F32)
    w = (wA + wB).astype(F32)
    live = w > 0
    return np.where(live, blend(cA, wA, cB, wB), cB).astype(np.uint32), np.where(live, w, wB).astype(F32)


def interp_channels(words, off):
    """Interpolator::interpVoxel's colour: words = the 8 neighbours' colour words in the interpolator's order
    (index = 4 dx + 2 dy + dz), off = the point's offset from neighbour 0's centre in voxels (3,).  Every channel
    is q . (B1 . channel^T) in float32, operation by operation as vgo_interp_voxel sums it, then truncated to
    uint8 (clamped to [0, 255])."""
    o = np.asarray(off, F32)
    q = [F32(1), o[0], o[1], o[2], o[0] * o[1], o[1] * o[2], o[2] * o[0], o[0] * o[1] * o[2]]
    out = 0
    for k in range(4):
        x = [F32((int(w) >> (8 * k)) & 255) for w in words]
        a = [x[0], -x[0] + x[4], -x[0] + x[2], -x[0] + x[1], x[0] - x[2] - x[4] + x[6], x[0] - x[1] - x[2] + x[3],
             x[0] - x[1] - x[4] + x[5], -x[0] + x[1] + x[2] - x[3] + x[4] - x[5] - x[6] + x[7]]
        r = F32(q[0] * a[0])
        for i in range(1, 8):
            r = F32(r + F32(q[i] * a[i]))
        out |= int(min(max(float(r), 0.0), 255.0)) << (8 * k)
    return np.uint32(out)


def containing_voxel(p, voxel_size):
    """Global voxel index floor(p / voxel_size + 1e-6) of points (n, 3) in the layer's frame, in float32 with
    the layer's voxel_size_inv (a double division stored as float)."""
    inv = F32(1.0 / float(F32(voxel_size)))
    return np.floor(np.asarray(p, F32) * inv + F32(1e-6)).astype(np.int64)


def vertex_colours(xyz, voxel_size, vps, idx, words):
    """The colour word of the voxel containing every vertex (layer frame); 0 where that voxel's block is missing."""
    k, c = layer_colours(idx, words, vps)
    g = containing_voxel(xyz, voxel_size)
    key = tx.voxel_keys(g)
    pos = np.minimum(np.searchsorted(k, key), len(k) - 1)
    return np.where(k[pos] == key, c[pos], 0).astype(np.uint32)
