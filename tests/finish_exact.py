"""Exact models of finishSubmap on the device (ESDF, relevant voxels, surface OBB, isosurface vertices)
for tests/test_oracle_finish.py and tests/test_gpu_finish_exact.py.  Test support, not product code.
MATRIX (the layer matrix), FILTERS and ESDF_CASES are the cases that the finishSubmap, mesh, projection,
registration-lookup and map evaluation tests run over.

Every model works on `Grid`, a dense embedding of a block layer over its block AABB with "absent"
cells, so neighbour logic owes nothing to block tables, hashes or slot order.  Block coordinates are
compressed per axis (runs of consecutive indices keep their spacing, any larger gap becomes one empty
block), which keeps adjacency exact and lets layers with blocks at both ends of the index range
embed in a small grid; positions are always computed from the original block indices.  All float
arithmetic is float32 operation by operation (numpy rounds every operation, as the kernels do under
-fmad=false), unless stated otherwise.

ESDF (`esdf`): the greatest fixed point of the device's rule, by float32 Jacobi relaxation
(np.minimum / np.maximum over the 26 shifted views of the grid):
  * a voxel is observed when !(w < min_weight); unobserved voxels read (0, 0) and are skipped as
    neighbours;
  * an observed voxel is fixed when |d| < min_distance and keeps d (so -0.0 and 0.0 stay);
  * every other observed voxel starts at +default when d > 0 and at -default otherwise (0 counts as
    negative);
  * a positive voxel pulls only from positive neighbours, cand = d_n + step, accepted when
    cand < max_distance and cand < d; a negative one only from negative neighbours, cand = d_n - step,
    accepted when cand > -max_distance and cand > d; a voxel at exactly 0 pulls from nothing and seeds
    nothing;
  * step = 1, sqrtf(2), sqrtf(3) times the voxel size in float32 for face, edge and corner neighbours.
  This is the device's rule restated; it is not voxblox's, which stays parity-unpinned.
  Sweep bound.  The update is monotone (cand is non-decreasing in d_n and the acceptance test only
  compares), so every fair order reaches the same point, and by induction on the sweep every value the
  in-place device sweeps hold is at least as far along as the Jacobi iterate of the same sweep.  Jacobi
  iterate k holds the best path of at most k steps.  An accepted path starts at a seed of the same
  sign and every step adds at least one voxel size, so a path of k steps has |value| >= k voxel sizes
  less k roundings of at most half an ulp of max_distance each; it is accepted only below
  max_distance, so it has at most ceil(max_distance / voxel_size) steps (the rounding can buy at most
  the step that lands exactly on max_distance).  Jacobi is therefore final after
  F = ceil(max_distance / voxel_size) + 1 sweeps, and so is the device.  The device reads its change
  flag after every second sweep and stops at the first pair of sweeps that changed nothing, so
      sweeps <= 2 ceil(F / 2) + 2                                            (`sweep_bound`).

Relevant voxels and surface OBB (`relevant`): slot order, then linear voxel order; a voxel qualifies
when double(w) > min_voxel_weight and |double(d)| < max_voxel_distance (voxgraph_submap.cpp:177-178),
centre = float(b) * block_size + (float(v) + 0.5f) * voxel_size, OBB = [min(c - h), max(c + h)],
h = 0.5f * voxel_size.

Isosurface vertices (`isosurface`): every voxel is the origin of a cube over its 2x2x2 forward
neighbourhood, valid when all 8 corners exist with w > float(min_voxel_weight).  Candidates in
canonical order: slot, linear voxel index, edge 0..11; a candidate per edge whose end points differ in
sign (s < 0 against s >= 0, so -0.0 is non-negative), interpolated as MarchingCubes::interpolateVertex
does (t = s1 / (s1 - s2), p = c0 + t (c1 - c0), or the midpoint when |s1 - s2| < 1e-6).  Bucket keys
are round(double(p) / threshold) with threshold = float(0.5 double(voxel_size)), rounded half away from
zero exactly: the fraction is taken against floor(|x|), which is exact in double.  The first candidate
of each bucket wins; a winner is kept when Interpolator::getVoxel succeeds (all 8 trilinear neighbours
exist with w > 1e-6f).  Its (distance, weight) is restated in float32 as vgo_interp_voxel evaluates it,
and also computed in float64 from the textbook trilinear formula on the same grid values.
  Interpolation bound.  Let u = 2^-24 and X = max |x_i| over the 8 values.  The float32 offset
  off = (p - centre) * inv differs from the exact (p - centre_exact) / voxel_size by at most
  E = u (3 |b| vps + 2 vps + 4) (centre: two products and a sum, each rounded relative to at most
  |b| vps + vps voxel sizes; the difference, the product and the rounded inverse each add u |off|,
  |off| <= 1 + E).  The q entries (products of up to three offsets, each |.| <= 1 + E) are off by at
  most 3 E + 2 u each, so sum |dq| <= 24 E + 16 u.  Each coefficient a_k is a sum of at most 8 values
  of size <= X: |a_k| <= 8 X with a rounding error of at most 7 u 8 X.  The sum r = q0 a0 + ... rounds
  8 products and 7 sums of terms bounded by 8 X (1 + E)^3.  Altogether, to first order and with
  E, u <= 2^-8 folding the higher orders into a factor 2,
      |r32 - r64| <= 2 X (8 (24 E + 16 u) + 64 * 8 * 7 u + 15 * 8 * 8 u)      (`interp_bound`).
"""
import math

import numpy as np

F32 = np.float32
U = 2.0 ** -24
_EPS = F32(1e-6)
CUBE_OFF = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0], [0, 0, 1], [1, 0, 1], [1, 1, 1], [0, 1, 1]])
EDGES = np.array([[0, 1], [1, 2], [2, 3], [3, 0], [4, 5], [5, 6], [6, 7], [7, 4], [0, 4], [1, 5], [2, 6], [3, 7]])
INDEX_MIN, INDEX_MAX = -(1 << 20) + 1, (1 << 20) - 2     # VGX_BLOCK_INDEX_MIN / _MAX


def _compress(v):
    """Sorted unique axis values -> compressed coordinates (spacing 1 kept, larger gaps become 2)."""
    u = np.unique(v)
    c = np.zeros(len(u), np.int64)
    if len(u) > 1:
        c[1:] = np.cumsum(np.minimum(np.diff(u), 2))
    return u, c


class Grid:
    """Dense embedding of the layer (voxel_size, vps, block_idx (n,3), distance, weight (n, vps^3))."""

    def __init__(self, voxel_size, vps, block_idx, distance, weight):
        self.vs = F32(voxel_size)
        self.vps = int(vps)
        self.bs = F32(self.vs * F32(vps))
        self.vsi = F32(1.0 / np.float64(self.vs))
        self.bsi = F32(1.0 / np.float64(self.bs))
        self.idx = np.asarray(block_idx, np.int64).reshape(-1, 3)
        n, vpb = len(self.idx), self.vps ** 3
        self.n = n
        self.d = np.asarray(distance, F32).reshape(n, vpb)
        self.w = np.asarray(weight, F32).reshape(n, vpb)
        assert len(np.unique(self.idx, axis=0)) == n, "repeated block index"
        vps = self.vps
        self.axes = [_compress(self.idx[:, a]) if n else (np.zeros(0, np.int64), np.zeros(0, np.int64))
                     for a in range(3)]
        nb = [int(c[-1]) + 1 if len(c) else 0 for _, c in self.axes]
        # padded by one voxel on every side: shifts never wrap
        self.shape = (nb[2] * vps + 2, nb[1] * vps + 2, nb[0] * vps + 2)    # [z, y, x]
        Z, Y, X = self.shape
        self.D = np.zeros(Z * Y * X, F32)
        self.W = np.zeros(Z * Y * X, F32)
        self.P = np.zeros(Z * Y * X, bool)
        lin = np.arange(vpb)
        self.loc = np.stack([lin % vps, (lin // vps) % vps, lin // (vps * vps)], -1)    # x, y, z
        if n:
            cb = np.stack([self.axes[a][1][np.searchsorted(self.axes[a][0], self.idx[:, a])] for a in range(3)], -1)
            g = cb[:, None, :] * vps + self.loc[None] + 1
            self.flat = ((g[..., 2] * Y + g[..., 1]) * X + g[..., 0]).reshape(-1)     # slot, lin order
        else:
            self.flat = np.zeros(0, np.int64)
        self.D[self.flat] = self.d.reshape(-1)
        self.W[self.flat] = self.w.reshape(-1)
        self.P[self.flat] = True

    def shift(self, dx, dy, dz):
        return (dz * self.shape[1] + dy) * self.shape[2] + dx

    def lookup(self, b, v):
        """Original block indices b (m,3) and local voxel indices v (m,3) -> flat cell, -1 if absent."""
        b = np.asarray(b, np.int64); v = np.asarray(v, np.int64)
        ok = np.ones(len(b), bool)
        g = np.zeros_like(b)
        for a in range(3):
            u, c = self.axes[a]
            if len(u) == 0:
                return np.full(len(b), -1, np.int64)
            k = np.minimum(np.searchsorted(u, b[:, a]), len(u) - 1)
            ok &= u[k] == b[:, a]
            g[:, a] = c[k] * self.vps + v[:, a] + 1
        Z, Y, X = self.shape
        f = (g[:, 2] * Y + g[:, 1]) * X + g[:, 0]
        f = np.where(ok, f, 0)
        ok &= self.P[f]
        return np.where(ok, f, -1)

    def centres(self):
        """Voxel centres (n * vps^3, 3) in slot / linear order, float32 as the kernels compute them."""
        origin = self.idx.astype(F32) * self.bs                              # (n, 3)
        off = (self.loc.astype(F32) + F32(0.5)) * self.vs                    # (vpb, 3)
        return (origin[:, None, :] + off[None]).reshape(-1, 3)


# --------------------------------------------------------------------------- ESDF
def sweep_bound(max_distance, voxel_size):
    F = math.ceil(float(F32(max_distance)) / float(F32(voxel_size))) + 1
    return 2 * ((F + 1) // 2) + 2, F


def esdf(grid, max_distance=2.0, default_distance=2.0, min_distance=0.2, min_weight=1e-6):
    """-> (distance (n, vps^3), observed (n, vps^3), Jacobi sweeps until final)."""
    g = grid
    mx, df, mn, mw = F32(max_distance), F32(default_distance), F32(min_distance), F32(min_weight)
    obs = g.P & ~(g.W < mw)
    fixed = obs & (np.abs(g.D) < mn)
    E = np.where(obs, np.where(fixed, g.D, np.where(g.D > 0, df, -df)), F32(0)).astype(F32)
    free = obs & ~fixed
    cells = np.nonzero(free)[0]
    steps = [F32(1.0) * g.vs, F32(np.sqrt(F32(2.0))) * g.vs, F32(np.sqrt(F32(3.0))) * g.vs]
    offs = [(dx, dy, dz) for dz in (-1, 0, 1) for dy in (-1, 0, 1) for dx in (-1, 0, 1) if dx or dy or dz]
    sweeps = 0
    while True:
        d = E[cells]
        pos, neg = d > 0, d < 0
        best = d.copy()
        for dx, dy, dz in offs:
            j = cells + g.shift(dx, dy, dz)
            dn = E[j]
            on = obs[j]
            step = steps[abs(dx) + abs(dy) + abs(dz) - 1]
            cp = (dn + step).astype(F32)
            cn = (dn - step).astype(F32)
            best = np.where(pos & on & (dn > 0) & (cp < mx) & (cp < best), cp, best)
            best = np.where(neg & on & (dn < 0) & (cn > -mx) & (cn > best), cn, best)
        if np.array_equal(best.view(np.uint32), d.view(np.uint32)):
            break
        E[cells] = best
        sweeps += 1
    vpb = g.vps ** 3
    return (E[g.flat].reshape(g.n, vpb), obs[g.flat].astype(F32).reshape(g.n, vpb), sweeps)


# --------------------------------------------------------------------------- relevant voxels + OBB
def relevant(grid, min_voxel_weight=1.0, max_voxel_distance=0.3, esdf_distance=None):
    """-> (xyz (m,3), distance (m,), weight (m,), (obb ok, min, max))."""
    g = grid
    d = g.d.reshape(-1); w = g.w.reshape(-1)
    sel = (w.astype(np.float64) > float(min_voxel_weight)) & (np.abs(d.astype(np.float64)) < float(max_voxel_distance))
    c = g.centres()[sel]
    dd = (np.asarray(esdf_distance, F32).reshape(-1) if esdf_distance is not None else d)[sel]
    half = F32(0.5) * g.vs
    if len(c):
        obb = (True, (c - half).min(0).astype(F32), (c + half).max(0).astype(F32))
    else:
        obb = (False, None, None)
    return c, dd.copy(), w[sel].copy(), obb


# --------------------------------------------------------------------------- isosurface vertices
def round_half_away(x):
    """llround on doubles, exactly: the fraction against floor(|x|) is exact in binary64."""
    a = np.abs(x)
    f = np.floor(a)
    r = f + (a - f >= 0.5)
    return (np.sign(x) * r).astype(np.int64)


def bucket_keys(p, voxel_size):
    thr = F32(0.5 * np.float64(F32(voxel_size)))
    return round_half_away(np.asarray(p, F32).astype(np.float64) * (1.0 / np.float64(thr)))


def candidates(grid, min_voxel_weight):
    """Candidate vertices in canonical order -> (xyz (M,3) float32, row (M,) voxel, edge (M,))."""
    g = grid
    mw = F32(min_voxel_weight)
    f = g.flat
    sdf = np.zeros((len(f), 8), F32)
    ok = np.ones(len(f), bool)
    for i, (ox, oy, oz) in enumerate(CUBE_OFF):
        j = f + g.shift(ox, oy, oz)
        ok &= g.P[j] & ~(g.W[j] <= mw)
        sdf[:, i] = g.D[j]
    s1, s2 = sdf[:, EDGES[:, 0]], sdf[:, EDGES[:, 1]]
    cross = ok[:, None] & (((s1 < 0) & (s2 >= 0)) | ((s1 >= 0) & (s2 < 0)))
    row, edge = np.nonzero(cross)                 # row-major: voxel order, then edge order
    coords = g.centres()[row]
    e0, e1 = EDGES[edge, 0], EDGES[edge, 1]
    a, b = s1[row, edge], s2[row, edge]
    diff = (a - b).astype(F32)
    big = np.abs(diff) >= _EPS
    with np.errstate(all="ignore"):
        t = (a / diff).astype(F32)
    p = np.zeros((len(row), 3), F32)
    for ax in range(3):
        c0 = (coords[:, ax] + CUBE_OFF[e0, ax].astype(F32) * g.vs).astype(F32)
        c1 = (coords[:, ax] + CUBE_OFF[e1, ax].astype(F32) * g.vs).astype(F32)
        lerp = (c0 + (t * (c1 - c0)).astype(F32)).astype(F32)
        mid = (F32(0.5) * (c0 + c1).astype(F32)).astype(F32)
        p[:, ax] = np.where(big, lerp, mid)
    return p, row, edge


def first_of_bucket(keys):
    """Index of the first candidate of every bucket, ascending."""
    if len(keys) == 0:
        return np.zeros(0, np.int64)
    packed = np.zeros(len(keys), np.int64)
    for a in range(3):
        u, inv = np.unique(keys[:, a], return_inverse=True)
        packed = packed * len(u) + inv.reshape(-1)
    _, first = np.unique(packed, return_index=True)
    return np.sort(first)


def _floor_i(x):
    return np.floor(x).astype(np.int64)


def interp(grid, p):
    """Interpolator::getVoxel at float32 points p (m,3) -> (ok, d32, w32, d64, w64, bound_d, bound_w)."""
    g = grid
    p = np.asarray(p, F32)
    m = len(p)
    vps = g.vps
    b = _floor_i(((p * g.bsi).astype(F32) + _EPS).astype(F32))
    ok = _blocks_exist(g, b)
    v = np.zeros_like(b)
    for a in range(3):
        origin = (b[:, a].astype(F32) * g.bs).astype(F32)
        vi = _floor_i(((p[:, a] - origin).astype(F32) * g.vsi + _EPS).astype(F32))
        vi = np.clip(vi, 0, vps - 1)
        centre = (origin + ((vi.astype(F32) + F32(0.5)) * g.vs).astype(F32)).astype(F32)
        dn = (p[:, a] - centre).astype(F32) < 0
        vi = np.where(dn, vi - 1, vi)
        wrap = vi < 0
        b[:, a] = np.where(wrap, b[:, a] - 1, b[:, a])
        v[:, a] = np.where(wrap, vi + vps, vi)
    ok &= _blocks_exist(g, b)
    off = np.zeros((m, 3), F32)
    off64 = np.zeros((m, 3))
    for a in range(3):
        centre = (((b[:, a].astype(F32) * g.bs).astype(F32)
                   + ((v[:, a].astype(F32) + F32(0.5)) * g.vs).astype(F32))).astype(F32)
        off[:, a] = ((p[:, a] - centre).astype(F32) * g.vsi).astype(F32)
        exact = (b[:, a] * vps + v[:, a] + 0.5) * np.float64(g.vs)
        off64[:, a] = (p[:, a].astype(np.float64) - exact) / np.float64(g.vs)
    x = np.zeros((m, 8), F32); wv = np.zeros((m, 8), F32)
    for i in range(8):
        cv = v + np.array([(i >> 2) & 1, (i >> 1) & 1, i & 1])
        cb = b + (cv >= vps)
        cv = cv % vps
        f = g.lookup(cb, cv)
        ok &= f >= 0
        fi = np.maximum(f, 0)
        x[:, i] = g.D[fi]; wv[:, i] = g.W[fi]
        ok &= wv[:, i] > _EPS
    q = np.stack([np.ones(m, F32), off[:, 0], off[:, 1], off[:, 2], (off[:, 0] * off[:, 1]).astype(F32),
                  (off[:, 1] * off[:, 2]).astype(F32), (off[:, 2] * off[:, 0]).astype(F32),
                  ((off[:, 0] * off[:, 1]).astype(F32) * off[:, 2]).astype(F32)], -1)
    out32, out64, bound = [], [], []
    E = U * (3 * np.abs(b).max(1, initial=0) * vps + 2 * vps + 4)
    for xs in (x, wv):
        c = [xs[:, k] for k in range(8)]
        a = [c[0], -c[0] + c[4], -c[0] + c[2], -c[0] + c[1],
             ((c[0] - c[2]) - c[4]) + c[6], ((c[0] - c[1]) - c[2]) + c[3], ((c[0] - c[1]) - c[4]) + c[5],
             ((((((-c[0] + c[1]) + c[2]) - c[3]) + c[4]) - c[5]) - c[6]) + c[7]]
        r = q[:, 0] * a[0]
        for k in range(1, 8):
            r = (r + (q[:, k] * a[k]).astype(F32)).astype(F32)
        out32.append(r.astype(F32))
        xd = xs.astype(np.float64)
        fx, fy, fz = off64[:, 0], off64[:, 1], off64[:, 2]
        r64 = np.zeros(m)
        for i in range(8):
            wx = fx if (i >> 2) & 1 else 1 - fx
            wy = fy if (i >> 1) & 1 else 1 - fy
            wz = fz if i & 1 else 1 - fz
            r64 += wx * wy * wz * xd[:, i]
        out64.append(r64)
        X = np.abs(xd).max(1, initial=0)
        bound.append(interp_bound(X, E))
    return ok, out32[0], out32[1], out64[0], out64[1], bound[0], bound[1]


def interp_bound(X, E):
    return 2 * X * (8 * (24 * E + 16 * U) + 64 * 8 * 7 * U + 15 * 8 * 8 * U)


def _blocks_exist(g, b):
    return g.lookup(b, np.zeros_like(b)) >= 0 if len(b) else np.zeros(0, bool)


def isosurface(grid, min_voxel_weight=1.0):
    """-> dict(xyz, distance, weight, blocks (first-occurrence order), cand, keys, winners, d64, w64,
    bound_d, bound_w) with the isosurface vertices in canonical order."""
    g = grid
    cand, row, edge = candidates(g, min_voxel_weight)
    keys = bucket_keys(cand, g.vs).reshape(-1, 3)
    win = first_of_bucket(keys)
    ok, d32, w32, d64, w64, bd, bw = interp(g, cand[win])
    keep = win[ok]
    xyz = cand[keep]
    blocks = _floor_i((xyz * g.bsi + _EPS).astype(F32)) if len(xyz) else np.zeros((0, 3), np.int64)
    if len(blocks):
        _, first = np.unique(blocks, axis=0, return_index=True)
        blocks = blocks[np.sort(first)]
    return dict(xyz=xyz, distance=d32[ok], weight=w32[ok], blocks=blocks.astype(np.int32), cand=cand,
                keys=keys, winners=win, kept=keep, d64=d64[ok], w64=w64[ok], bound_d=bd[ok], bound_w=bw[ok])


# --------------------------------------------------------------------------- comparisons
def assert_bits(exp, got, what):
    exp = np.asarray(exp); got = np.asarray(got)
    assert exp.shape == got.shape, (what, "shape", exp.shape, got.shape)
    e = np.ascontiguousarray(exp, F32).view(np.uint32); g = np.ascontiguousarray(got, F32).view(np.uint32)
    bad = np.nonzero(e != g)
    assert bad[0].size == 0, (what, "first difference at", tuple(int(k[0]) for k in bad),
                              float(exp[bad][0]), float(got[bad][0]), "differences", bad[0].size)


def assert_points(exp, got, what):
    """(xyz, distance, weight) triples equal bit for bit, in the same order."""
    for k, name in enumerate(("xyz", "distance", "weight")):
        assert_bits(exp[k], got[k], "%s %s" % (what, name))


# --------------------------------------------------------------------------- the layer matrix
RESOLUTIONS = [(0.05, 2), (0.1, 4), (0.15, 8), (0.2, 16), (0.05, 32), (0.125, 16), (0.25, 8)]
EXACT_RESOLUTIONS = [(0.125, 16), (0.25, 8)]
_HI = INDEX_MAX


def layout(name, rs=None):
    """Block index sets of the matrix (slot order as listed)."""
    box = lambda x, y, z: [(i, j, k) for k in range(z[0], z[1] + 1) for j in range(y[0], y[1] + 1)
                           for i in range(x[0], x[1] + 1)]
    if name == "box":
        b = box((0, 1), (0, 1), (-1, 0))
    elif name == "checker":
        b = [q for q in box((0, 2), (0, 2), (0, 1)) if sum(q) % 2 == 0]
    elif name == "edge":        # two groups that meet only along one block edge
        b = [(0, 0, 0), (1, 0, 0), (2, 1, 0), (3, 1, 0)]
    elif name == "corner":      # ... only at one block corner
        b = [(0, 0, 0), (1, 0, 0), (2, 1, 1), (3, 1, 1)]
    elif name == "negative":
        b = box((-3, -2), (-2, -1), (-2, -1))
    elif name == "straddle":
        b = box((-1, 0), (-1, 0), (-1, 0))
    elif name == "range_edges":  # both ends of the accepted index range, on every axis
        h = _HI
        b = [(h - 1, 0, 0), (h, 0, 0), (h, 1, 0), (-h, -h, -h), (-h + 1, -h, -h), (-h, -h + 1, -h),
             (0, h, -h), (0, h, -h + 1)]
    elif name == "shuffled":
        b = box((0, 1), (0, 1), (-1, 0))
        b = [b[k] for k in np.random.RandomState(7).permutation(len(b))]
    elif name == "one":
        b = [(0, 0, 0)]
    elif name == "zero":
        b = []
    else:
        raise KeyError(name)
    return np.asarray(b, np.int32).reshape(-1, 3)


LAYOUTS = ["box", "checker", "edge", "corner", "negative", "straddle", "range_edges", "shuffled", "one", "zero"]


def voxel_global(idx, vps):
    """(n, vps^3, 3) int64 global voxel indices."""
    lin = np.arange(vps ** 3)
    loc = np.stack([lin % vps, (lin // vps) % vps, lin // (vps * vps)], -1)
    return np.asarray(idx, np.int64)[:, None, :] * vps + loc[None]


def field(name, voxel_size, vps, idx, seed=0):
    """(distance, weight) of a named field at the voxel centres of the blocks idx."""
    vs = F32(voxel_size)
    g = voxel_global(idx, vps)
    n = len(idx)
    local = (g - g.reshape(-1, 3).min(0)) if n else g      # fields are placed relative to the layer
    if n and local.max() > 8 * vps:
        local = np.mod(g, 2 * vps)                         # ... or repeat where the layer is huge
    lc = (local + 0.5) * float(vs)
    w = np.full((n, vps ** 3), 2.0, F32)
    if name == "plane":
        d = lc[..., 2] - 0.37 * float(vs) * vps
    elif name == "tilted":
        d = lc @ np.array([0.3, -0.2, 0.93]) - 0.6 * float(vs) * vps
    elif name == "sphere":
        ext = lc.reshape(-1, 3).max(0, initial=1.0) if n else np.ones(3)
        d = np.linalg.norm(lc - 0.5 * ext, axis=-1) - 0.3 * float(ext.min())
    elif name == "noise":
        d = np.random.RandomState(seed).uniform(-0.05, 0.05, (n, vps ** 3))
    elif name == "crafted":
        d, w = crafted(g, vs)
        return d, w
    else:
        raise KeyError(name)
    return np.clip(d, -0.6, 0.6).astype(F32).reshape(n, vps ** 3), w


def crafted(g, vs):
    """Exact-binary field at voxel size 0.25 or 0.125 on global voxel indices g (n, vpb, 3): per
    column (x + 3y) mod 7 the two voxels around the layer's middle z plane are (-0.25, 0.75) [t = 0.25: the vertex lies
    exactly on a bucket half-boundary with an odd integer part], (-0.75, 0.25) [t = 0.75: even integer
    part, where llround and rint differ], (-1e-7, 5e-7) [the midpoint branch], (-0.0, 0.0),
    (-0.5, 0.0) [t = 1], (0.0, -0.0) and (-1e-6f, 0.0) [|s1 - s2| exactly 1e-6f: interpolated, t = 1];
    further away a ramp of whole voxel sizes."""
    gz = g[..., 2] - ((g[..., 2].min() + g[..., 2].max() + 1) // 2 if g.size else 0)   # z = 0 mid-layer
    col = (g[..., 0] + 3 * g[..., 1]) % 7
    pairs = np.array([[-0.25, 0.75], [-0.75, 0.25], [-1e-7, 5e-7], [-0.0, 0.0], [-0.5, 0.0], [0.0, -0.0],
                      [-1e-6, 0.0]], F32)
    lo = pairs[col, 0]; hi = pairs[col, 1]
    ramp = (np.clip(gz, -4, 4).astype(F32) * F32(vs)).astype(F32)
    d = np.where(gz == -1, lo, np.where(gz == 0, hi, np.where(gz < -1, ramp - F32(0.5), ramp + F32(0.5)))).astype(F32)
    return d.reshape(len(g), g.shape[1]), np.full(d.shape, 2.0, F32).reshape(len(g), g.shape[1])


def layer(res, lay, fld, seed=0):
    vs, vps = res
    idx = layout(lay)
    d, w = field(fld, vs, vps, idx, seed)
    return vs, vps, idx, d, w


def matrix():
    """(id, (voxel size, vps, idx, distance, weight)) over resolutions x layouts, the field rotating
    with the layout so every layout meets planes, spheres and noise; the crafted field runs on the
    exact-binary resolutions."""
    out = []
    fields = ["tilted", "sphere", "plane", "noise"]
    for r, res in enumerate(RESOLUTIONS):
        for k, lay in enumerate(LAYOUTS):
            fld = fields[(r + k) % len(fields)]
            if res in EXACT_RESOLUTIONS and lay in ("box", "straddle", "negative", "shuffled"):
                fld = "crafted"
            out.append(("%g/%d-%s-%s" % (res[0], res[1], lay, fld), layer(res, lay, fld, seed=r * 31 + k)))
    return out


def noise_layer(vs, vps, nblocks_xyz, seed=0, origin=(0, 0, 0)):
    """Random-sign noise (distance uniform in +-0.05, weight 2) over a box of blocks."""
    nx, ny, nz = nblocks_xyz
    idx = np.array([(origin[0] + i, origin[1] + j, origin[2] + k) for k in range(nz) for j in range(ny)
                    for i in range(nx)], np.int32)
    d = np.random.RandomState(seed).uniform(-0.05, 0.05, (len(idx), vps ** 3)).astype(F32)
    return vs, vps, idx, d, np.full(d.shape, 2.0, F32)


# filters: min_voxel_weight 0 / 0.1 with weights 0.1f / 0.5 / 1, weights at 1e-6, zero-weight slabs,
# max_voxel_distance 0, 0.3 and exactly a voxel's value
def filter_cases():
    out = []
    for res in [(0.25, 8), (0.2, 16)]:
        vs, vps, idx, d, w = layer(res, "box", "tilted")
        w01 = np.full_like(w, np.float32(0.1))
        wz = w.copy().reshape(len(idx), vps, vps, vps)
        wz[:, :, 3, :] = 0.0                      # a zero-weight slab (y = 3) in every block
        wz[:, 5, :, :] = np.float32(1e-6)         # ... and a slab at the observation threshold
        wz = wz.reshape(len(idx), -1)
        v = float(d.reshape(-1)[len(d.reshape(-1)) // 2])
        for mw, ww, md in [(0.0, w, 0.3), (0.1, w01, 0.3), (0.5, w, 0.3), (1.0, w, 0.3), (0.0, wz, 0.3),
                           (1.0, w, 0.0), (1.0, w, abs(v)), (0.0, wz, 0.6)]:
            out.append(("%g/%d-minw%g-maxd%g-%s" % (res[0], res[1], mw, md, "slabs" if ww is wz else
                                                     "w0.1f" if ww is w01 else "w2"),
                        (vs, vps, idx, d, ww, mw, md)))
    return out


def esdf_cases():
    sph = layer((0.2, 16), "box", "sphere")
    pl = layer((0.25, 8), "edge", "plane")
    cr = layer((0.125, 16), "straddle", "crafted")
    long = layer((0.05, 32), "one", "plane")
    idx5 = np.array([(i, 0, 0) for i in range(4)], np.int32)
    d5 = np.full((4, 32 ** 3), 0.6, np.float32)
    d5.reshape(4, 32, 32, 32)[0, :, :, 0] = 0.01          # one seed plane at x = 0: 127 voxels to go
    far = (0.05, 32, idx5, d5, np.full_like(d5, 2.0))
    de = np.full((1, 8 ** 3), 0.5, np.float32)
    de.reshape(8, 8, 8)[:, :, 0] = 0.25                   # seeds at x = 0: 0.25 + 3 * 0.25 is exactly 1.0
    exact_max = (0.25, 8, np.zeros((1, 3), np.int32), de, np.full_like(de, 2.0))
    return [("defaults-sphere", sph, {}), ("max<vs", sph, dict(max_distance_m=0.15)),
            ("max-not-multiple", sph, dict(max_distance_m=0.93)),
            ("default<max", sph, dict(default_distance_m=0.5, max_distance_m=2.0)),
            ("min0", sph, dict(min_distance_m=0.0)), ("min>=trunc", sph, dict(min_distance_m=0.7)),
            ("edge-join", pl, {}), ("crafted-zeros", cr, dict(min_distance_m=0.3)),
            ("crafted-min0", cr, dict(min_distance_m=0.0)),
            ("weights-1e-6", (long[0], long[1], long[2], long[3], np.full_like(long[4], np.float32(1e-6))), {}),
            ("5m-at-0.05", far, dict(max_distance_m=5.0, default_distance_m=5.0)),
            ("max-reached-exactly", exact_max, dict(min_distance_m=0.3, max_distance_m=1.0))]


MATRIX = matrix()
FILTERS = filter_cases()
ESDF_CASES = esdf_cases()
