"""Exact models of the TSDF integrator for the GPU parity tests (tests/test_gpu_tsdf_exact.py, with
tests/colour_exact.py for the colour of the same updates), and the scans, configurations and crafted
points they run.

* `replay` applies a list of ray-ordered (voxel, sdf, update weight) tuples, as the oracle's
  `tsdf_integrate_trace` records them, with the integrator's float32 update (updateTsdfVoxel's
  weighted running average, fminf/fmaxf clamps).  In ray order it reproduces the oracle bit for bit;
  in any other order it is one serialisation of the Fast schedule's CAS updates.
* It also counts the batches that `tsdf_apply_long_kernel` must collapse in closed form (mode 0,
  `saturated_batches`): segments longer than VGX_TSDF_LONG_SEGMENT = 64 are cut into 32-tuple
  batches; a full batch is saturated when the voxel sits at +trunc with an integer weight below
  2^24 (or at the cap) and every tuple has sdf >= 2 trunc, uw >= 2^-20 max_weight and an integer
  uw (unless capped).
* `check_fast` is the serialisation check of the Fast schedule (mode 1 with every ray cast): with
  integer update weights the weight min(max_weight, sum uw) does not depend on the order, so a lost
  or duplicated update moves it by at least 1; the distance is checked where it is order free
  (one update; +trunc when every sdf >= 2 trunc) and against a rounding bound elsewhere.

Rounding bound of the running mean (C_MEAN).  With integer weights below 2^24 the weight sums
W_k are exact, and one step computes d_k = fl(fl(fl(s_k u_k) + fl(d_{k-1} W_{k-1})) / W_k): every
term passes through at most three roundings (a product, the sum, the quotient), each a relative
error of at most u = 2^-24.  With m_k the exact weighted mean of the first k updates and
S = max |s_i|, e_k = d_k - m_k obeys
    e_k = (W_{k-1} / W_k) e_{k-1} + r_k,   |r_k| <= ((1 + u)^3 - 1) (|s_k| u_k + |d_{k-1}| W_{k-1}) / W_k
                                                 <= 3 u (1 + 2u) (S + |e_{k-1}|),
so |e_n| <= 3 n u S (1 + 3 n u) (W_{k-1}/W_k <= 1 and the second-order terms are folded into the
last factor).  Clamping to [-trunc, trunc] is a projection onto an interval that holds m_n (every
|s_i| <= trunc there) and cannot increase the error.  Hence C_MEAN = 3:
    |d - m| <= 3 n u S (1 + 3 n u).
"""
import math

import numpy as np

U = 2.0 ** -24
C_MEAN = 3
LONG_SEGMENT = 64
F32 = np.float32
_EPS = F32(1e-6)            # VGX_EPS / kFloatEpsilon
_UW_FLOOR = F32(9.5367431640625e-07)  # 2^-20


def voxel_keys(g):
    """(m, 3) int64 global voxel indices -> one sortable int64 per voxel (21 bits per axis)."""
    g = np.asarray(g, np.int64).reshape(-1, 3) + (1 << 20)
    assert g.min(initial=0) >= 0 and g.max(initial=0) < (1 << 21)
    return g[:, 0] | (g[:, 1] << 21) | (g[:, 2] << 42)


def layer_voxels(idx, d, w, vps):
    """Exported layer -> (keys, distance, weight) of every voxel of every block, sorted by key."""
    idx = np.asarray(idx, np.int64).reshape(-1, 3)
    lin = np.arange(vps ** 3)
    loc = np.stack([lin % vps, (lin // vps) % vps, lin // (vps * vps)], -1)
    g = (idx[:, None, :] * vps + loc[None]).reshape(-1, 3)
    k = voxel_keys(g)
    o = np.argsort(k, kind="stable")
    return k[o], np.asarray(d, F32).reshape(-1)[o], np.asarray(w, F32).reshape(-1)[o]


def _sorted_blocks(idx, d, w):
    idx = np.asarray(idx).reshape(-1, 3)
    o = np.lexsort((idx[:, 2], idx[:, 1], idx[:, 0]))
    return idx[o], np.asarray(d)[o], np.asarray(w)[o]


def assert_layers_bit_equal(exp, got):
    """Same block set, and every voxel's distance and weight equal bit for bit."""
    ie, de, we = _sorted_blocks(*exp)
    ig, dg, wg = _sorted_blocks(*got)
    assert ie.shape == ig.shape and np.array_equal(ie, ig), "block sets differ"
    bad_w = np.nonzero(wg.view(np.uint32) != we.view(np.uint32))
    assert bad_w[0].size == 0, ("weights differ", ie[bad_w[0][0]], bad_w[1][0], we[bad_w][0], wg[bad_w][0])
    bad_d = np.nonzero(dg.view(np.uint32) != de.view(np.uint32))
    assert bad_d[0].size == 0, ("distances differ", ie[bad_d[0][0]], bad_d[1][0], de[bad_d][0], dg[bad_d][0])


def apply_update(s, u, vd, vw, trunc, max_weight):
    """tsdf_apply (csrc/tsdf.cu), elementwise in float32; returns the new (distance, weight)."""
    with np.errstate(all="ignore"):
        nw = vw + u
        skip = nw < _EPS
        ns = (s * u + vd * vw) / nw
        nd = np.where(ns > F32(0), np.fmin(trunc, ns), np.fmax(-trunc, ns)).astype(F32)
        nww = np.fmin(max_weight, nw).astype(F32)
    return np.where(skip, vd, nd), np.where(skip, vw, nww)


class State:
    """(distance, weight) of the voxels touched so far, sorted by voxel key."""

    def __init__(self):
        self.keys = np.zeros(0, np.int64)
        self.d = np.zeros(0, F32)
        self.w = np.zeros(0, F32)

    def get(self, keys):
        d = np.zeros(len(keys), F32); w = np.zeros(len(keys), F32)
        if len(self.keys):
            pos = np.minimum(np.searchsorted(self.keys, keys), len(self.keys) - 1)
            hit = self.keys[pos] == keys
            d[hit] = self.d[pos[hit]]; w[hit] = self.w[pos[hit]]
        return d, w

    def put(self, keys, d, w):
        k = np.concatenate([keys, self.keys])
        dd = np.concatenate([d, self.d]); ww = np.concatenate([w, self.w])
        k, first = np.unique(k, return_index=True)    # the new values come first
        self.keys, self.d, self.w = k, dd[first], ww[first]


def replay(keys, sdf, uw, trunc, max_weight, state=None, order=None):
    """Apply the tuples (voxel key, sdf, uw) voxel by voxel in the given order (default: as listed,
    i.e. ray order).  Returns (voxel keys, distance, weight, saturated batches); `state` (a State)
    supplies the starting values and receives the results."""
    keys = np.asarray(keys, np.int64); sdf = np.asarray(sdf, F32); uw = np.asarray(uw, F32)
    if order is not None:
        keys, sdf, uw = keys[order], sdf[order], uw[order]
    trunc = F32(trunc); M = F32(max_weight)
    o = np.argsort(keys, kind="stable")
    k, s, u = keys[o], sdf[o], uw[o]
    uniq, start, cnt = np.unique(k, return_index=True, return_counts=True)
    d0, w0 = state.get(uniq) if state is not None else (np.zeros(len(uniq), F32), np.zeros(len(uniq), F32))
    by = np.argsort(-cnt, kind="stable")
    cnt_s, start_s = cnt[by], start[by]
    dd, ww = d0[by].copy(), w0[by].copy()
    n_long = int(np.count_nonzero(cnt_s > LONG_SEGMENT))
    two_t = F32(2) * trunc
    floor = F32(M * _UW_FLOOR)
    sat = 0
    neg = -cnt_s
    for r in range(int(cnt_s[0]) if len(cnt_s) else 0):
        n_act = int(np.searchsorted(neg, -r, side="left"))   # voxels with more than r updates
        if r % 32 == 0 and n_long:
            full = np.nonzero(cnt_s[:n_long] - r >= 32)[0]
            if full.size:
                j = start_s[full][:, None] + r + np.arange(32)
                bs, bu = s[j], u[j]
                vx, vy = dd[full], ww[full]
                capped = vy == M
                pre = (vx == trunc) & (capped | ((vy == np.rint(vy)) & (vy >= 0) & (M < F32(16777216.0))))
                lanes = ((bs >= two_t).all(1) & (bu >= floor).all(1)
                         & (capped | (bu == np.rint(bu)).all(1)))
                sat += int(np.count_nonzero(pre & lanes))
        j = start_s[:n_act] + r
        dd[:n_act], ww[:n_act] = apply_update(s[j], u[j], dd[:n_act], ww[:n_act], trunc, M)
    inv = np.empty_like(by); inv[by] = np.arange(len(by))
    d_out, w_out = dd[inv], ww[inv]
    if state is not None:
        state.put(uniq, d_out, w_out)
    return uniq, d_out, w_out, sat


# ---------------------------------------------------------------------- the parity matrix
# Scans, configurations and crafted points that tests/test_gpu_tsdf_exact.py runs into a coloured
# submap and a colourless twin.
MW24 = 2.0 ** 24
# Mode 1 with every ray cast (start keys all distinct, unlimited ray collisions) and integer update
# weights (no drop-off): the set of updates is fixed, as check_fast needs.
FAST_ALL = dict(mode=1, start_voxel_subsampling_factor=1e3, max_consecutive_ray_collisions=1 << 30,
                use_weight_dropoff=0)
CONFIGS = [
    dict(),
    dict(use_const_weight=0),
    dict(use_weight_dropoff=0),
    dict(use_sparsity_compensation_factor=0),
    dict(sparsity_compensation_factor=1.0),
    dict(sparsity_compensation_factor=2.5),
    dict(allow_clear=0),
    dict(voxel_carving_enabled=0),
    dict(use_const_weight=0, use_weight_dropoff=0),
    dict(use_const_weight=0, sparsity_compensation_factor=2.5, allow_clear=0),
    dict(voxel_carving_enabled=0, use_weight_dropoff=0, use_sparsity_compensation_factor=0),
    dict(min_ray_length_m=1.5, max_ray_length_m=9.0),
    dict(default_truncation_distance=0.1),
    dict(default_truncation_distance=0.2),    # = voxel size: the drop-off denominator is 0
    dict(default_truncation_distance=2.0),
    dict(max_weight=3.0),
    dict(max_weight=40.0),
    dict(max_weight=100.5),
    dict(max_weight=MW24 - 8),
    dict(max_weight=MW24),
]


def config_id(kw):
    return ",".join("%s=%r" % i for i in kw.items()) or "default"


def scans(world, n_beams=16, n_azimuth=256, origin=(0.0, 0.0, 0.0)):
    """Three scans from different poses (two with clearing rays), sensor poses offset by `origin`."""
    from voxgraph_b200 import synth
    out = []
    for k, (px, py, yaw) in enumerate([(15.0, 15.0, 0.4), (16.5, 14.0, 1.9), (13.0, 16.0, -2.6)]):
        pts = synth.lidar_scan(world, np.array([px, py, 1.2, yaw]), n_beams=n_beams, n_azimuth=n_azimuth,
                               seed=k, miss_range=40.0 if k != 1 else None)
        T = synth.pose_to_T([px - 15.0 + origin[0], py - 15.0 + origin[1], 0.1 * k + origin[2], yaw])
        out.append((T, pts))
    return out


def ring(n, z, ranges, az0=0.1):
    """n points around the sensor at height z (sensor frame) and the given horizontal ranges."""
    a = az0 + 2 * np.pi * np.arange(n) / n
    r = np.resize(np.asarray(ranges, np.float64), n)
    zz = np.resize(np.asarray(z, np.float64), n)
    return np.stack([r * np.cos(a), r * np.sin(a), zz], -1).astype(np.float32)


def edge_points():
    """Crafted points for 0.25 m voxels: the ray-length limits and one ulp either side, the sensor
    point, NaN, inf and huge finite points, points on voxel faces, in one voxel, and clearing rays."""
    f = np.float32
    up = lambda v: np.nextafter(f(v), f(np.inf)); dn = lambda v: np.nextafter(f(v), f(-np.inf))
    p = []
    for r in (0.5, 8.0):                       # min / max ray length exactly, and one ulp either side
        for v in (dn(r), f(r), up(r)):
            p += [[v, 0, 0], [0, -v, 0], [0, 0, v]]     # axis-aligned: t = 2 on the degenerate axes
    p += [[0, 0, 0]]                           # sdf = 0/0 at the sensor voxel when min_ray_length_m = 0
    p += [[np.nan, 0, 0], [1, np.nan, 2], [np.inf, 0, 0], [-np.inf, 0, 0], [0, np.inf, 1]]
    p += [[3e19, 0, 0], [-2e19, 2e19, 0], [1.1e19, 1.1e19, 1.1e19], [1e19, -1e19, 1e19]]
    p += [[2.0, 0.5, 0.25], [4.0, -2.0, 1.0], [-2.0, 2.0, -0.75], [6.0, 4.0, 0.0], [0.0, -4.0, 2.0]]
    p += [[3.1 + 0.02 * k, 1.3 + 0.01 * k, -0.6 + 0.015 * k] for k in range(5)]   # one voxel
    p += [[12.0, 3.0, -1.0], [-9.0, 10.0, 0.5], [0.3, -15.0, 2.0]]             # clearing rays
    return np.array(p, np.float32)


EDGE_CFGS = [dict(min_ray_length_m=0.5, max_ray_length_m=8.0),
             dict(min_ray_length_m=0.0, max_ray_length_m=8.0, voxel_carving_enabled=0),
             dict(min_ray_length_m=0.0, max_ray_length_m=8.0, allow_clear=0),
             dict(min_ray_length_m=0.0, max_ray_length_m=8.0, use_weight_dropoff=0)]


def clearing_points(vs, n=400, seed=0):
    """n points 8 m + U(0.001, 0.6 m + one voxel) away in random directions: with max_ray_length_m = 8
    and the default trunc of 0.6 m every one is a clearing ray, cut at norm - trunc, and its last voxels
    can have their centres inside the band."""
    rs = np.random.RandomState(seed)
    d = rs.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1)[:, None]
    return (d * (8.0 + rs.uniform(0.001, 0.6 + vs, n))[:, None]).astype(F32)


def check_fast(cand, keys, sdf, uw, trunc, max_weight, exact=None):
    """Serialisation check of one Fast integration into an empty layer.

    cand = (keys, distance, weight) of every voxel of the candidate layer (layer_voxels);
    (keys, sdf, uw) = the scan's update tuples, every uw an integer; exact = (keys, distance, weight)
    of the oracle's result, used where a voxel has one update.  Raises AssertionError."""
    ck, cd, cw = cand
    keys = np.asarray(keys, np.int64); sdf = np.asarray(sdf, F32); uw = np.asarray(uw, F32)
    assert np.array_equal(uw, np.rint(uw)), "check_fast needs integer update weights"
    trunc = F32(trunc); M = F32(max_weight)
    o = np.argsort(keys, kind="stable")
    k, s, u = keys[o], sdf[o].astype(np.float64), uw[o].astype(np.float64)
    uniq, start, cnt = np.unique(k, return_index=True, return_counts=True)
    # visited voxels: exactly the voxels with an update (uw >= 1 here)
    visited = ck[cw > 0]
    assert np.array_equal(visited, uniq), "visited voxel sets differ"
    assert not np.any(cd[cw == 0]), "unvisited voxel with a distance"
    pos = np.searchsorted(ck, uniq)
    gd, gw = cd[pos], cw[pos]
    wsum = np.add.reduceat(u, start)            # integers below 2^53: exact
    w_exp = np.minimum(wsum, float(M)).astype(F32)
    bad = np.nonzero(gw != w_exp)[0]
    assert bad.size == 0, ("weight", uniq[bad[0]], int(cnt[bad[0]]), float(w_exp[bad[0]]), float(gw[bad[0]]))
    abs_s = np.abs(s)
    s_min = np.minimum.reduceat(s, start)
    s_absmax = np.maximum.reduceat(np.where(np.isnan(s), np.inf, abs_s), start)
    if exact is not None:
        ek, ed, _ = exact
        one = np.nonzero(cnt == 1)[0]
        ed1 = ed[np.searchsorted(ek, uniq[one])]
        bad = one[gd[one].view(np.uint32) != ed1.view(np.uint32)]
        assert bad.size == 0, ("single update", uniq[bad[0]])
    far = np.nonzero(s_min >= 2.0 * float(trunc))[0]
    bad = far[gd[far] != trunc]
    assert bad.size == 0, ("not +trunc", uniq[bad[0]], float(gd[bad[0]]))
    inner = np.nonzero((s_absmax <= float(trunc)) & (wsum <= float(M)) & (cnt > 1))[0]
    for i in inner:
        a, b = start[i], start[i] + cnt[i]
        m = math.fsum(s[a:b] * u[a:b]) / wsum[i]
        n = int(cnt[i])
        bound = C_MEAN * n * U * s_absmax[i] * (1.0 + C_MEAN * n * U)
        assert abs(float(gd[i]) - m) <= bound, ("mean", uniq[i], n, float(gd[i]), m, bound)
    return dict(voxels=len(uniq), single=int(np.count_nonzero(cnt == 1)), far=len(far), inner=len(inner),
                max_updates=int(cnt.max(initial=0)))
