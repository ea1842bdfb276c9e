"""Test support for the fused registration reduction (not product code).

Three pieces:

* Poses whose pose blocks are the same on the host and on the device.  The oracle (and emit mode)
  evaluates cos_e, sin_e, cos(the - tho), sin(the - tho) with libm cosf/sinf; the device pose set-up
  rounds a double cos/sin to float, and both evaluate vgx_yaw_quat with a double sin/cos.  For the
  poses drawn here every one of those values rounds to the same float on either side, so the fused
  kernel sees exactly the pose block the oracle uses and its per-point terms are the oracle's.
* An exact reference of cost, gradient and H: the oracle's per-point residuals and Jacobians placed
  at the node columns and summed per entry with math.fsum, with the error bound the fused sums must
  meet (only double summation order and a few ulps of `factor` per term separate them).
* A float32 restatement of the reduce kernel's transform, block index, unit bounds and unit cull test
  (vgx_reg_transform, vgx_block_index, reg_unit_bounds_kernel, reg_unit_may_hit), operation by
  operation and without FMA, used to build units on the cull decision and to check its margin.
"""
import ctypes
import ctypes.util
import math
from fractions import Fraction

import numpy as np

F32 = np.float32
SERIES_THETA = 1.220703125e-4     # vgx_yaw_quat: series branch below eps^(1/4)
MID_MARGIN = 2.0 ** -40           # relative distance a rounded double keeps from a float midpoint

_libm = ctypes.CDLL(ctypes.util.find_library("m"))
_libm.cosf.restype = ctypes.c_float
_libm.cosf.argtypes = [ctypes.c_float]
_libm.sinf.restype = ctypes.c_float
_libm.sinf.argtypes = [ctypes.c_float]


# --------------------------------------------------------------------------- exact-trig poses
def _far_from_midpoint(v):
    """v rounds to the same float32 under any perturbation below MID_MARGIN relative."""
    if v == 0.0:
        return True
    f = F32(v)
    for nb in (np.nextafter(f, F32(np.inf)), np.nextafter(f, F32(-np.inf))):
        mid = (float(f) + float(nb)) * 0.5      # exact in double
        if abs(v - mid) < MID_MARGIN * abs(v):
            return False
    return True


def _trig_ok(v):
    """libm cosf/sinf(v) == float(cos/sin(v)), and the double values sit clear of a midpoint."""
    v = F32(v)
    c, s = math.cos(float(v)), math.sin(float(v))
    return (_libm.cosf(float(v)) == float(F32(c)) and _libm.sinf(float(v)) == float(F32(s))
            and _far_from_midpoint(c) and _far_from_midpoint(s))


def _yaw_quat_ok(y):
    """Both roundings of vgx_yaw_quat (double sin/cos of theta / 2) sit clear of a midpoint."""
    y = F32(y)
    theta = float(np.sqrt(F32(y * y)))
    if not _far_from_midpoint(math.cos(theta * 0.5)):
        return False
    if theta < SERIES_THETA:
        return True        # 0.5 + theta^2 / 48: the same double operations on both sides
    return _far_from_midpoint(float(y) * (math.sin(theta * 0.5) / theta))


def node_pose_ok(pose):
    return _trig_ok(pose[3]) and _yaw_quat_ok(pose[3])


def pair_ok(ref_pose, read_pose):
    """the - tho, in float as the pose set-up computes it."""
    return _trig_ok(F32(read_pose[3]) - F32(ref_pose[3]))


def exact_trig_poses(base, constraints, rng, sigma=(0.05, 0.05, 0.02, 0.03), fixed=None, tries=2000):
    """Node poses (float32-representable x, y, z, yaw) near `base` (N, 4) whose pose blocks are the
    same on the host and the device for every constraint (ref, read) of `constraints` (node indices).
    Drawn by rejection, node by node.  fixed: {node: pose} used as drawn, without noise (still
    checked)."""
    base = np.asarray(base, np.float64)
    fixed = fixed or {}
    out = np.zeros_like(base)
    for k in range(base.shape[0]):
        for t in range(tries):
            if k in fixed:
                cand = np.asarray(fixed[k], np.float64)
            else:
                cand = base[k] + rng.normal(0.0, 1.0, 4) * np.asarray(sigma)
                cand[3] = cand[3] - 2 * np.pi * np.floor((cand[3] + np.pi) / (2 * np.pi))
            cand = cand.astype(F32).astype(np.float64)
            if not node_pose_ok(cand):
                ok = False
            else:
                ok = True
                for (a, b) in constraints:
                    if max(a, b) == k and min(a, b) <= k:
                        pa = cand if a == k else out[a]
                        pb = cand if b == k else out[b]
                        if not pair_ok(pa, pb):
                            ok = False
                            break
            if ok:
                out[k] = cand
                break
            if k in fixed:
                raise AssertionError("fixed pose %d fails the exact-trig condition" % k)
        else:
            raise AssertionError("no exact-trig pose found for node %d" % k)
    return out


def _rotate_yaw(w, z, v0, v1, v2):
    """vgx_rotate_yaw (Eigen _transformVector for q = (w, 0, 0, z)), float32, no FMA."""
    uv0 = -(z * v1)
    uv1 = z * v0
    uv0 = uv0 + uv0
    uv1 = uv1 + uv1
    c0 = -(z * uv1)
    c1 = z * uv0
    return (v0 + w * uv0) + c0, (v1 + w * uv1) + c1, v2


def yaw_quat(yaw):
    y = F32(yaw)
    theta = float(np.sqrt(F32(y * y)))
    if theta < SERIES_THETA:
        na = 0.5 + (theta * theta) * (1.0 / 48.0)
    else:
        na = math.sin(theta * 0.5) / theta
    return F32(math.cos(theta * 0.5)), F32(float(y) * na)


def pose_block(ref, read):
    """The device pose set-up (vgx_reg_pose_setup<TrigDevice>): dict of float32 values."""
    xo, yo, zo, tho = (F32(v) for v in ref)
    xe, ye, ze, the = (F32(v) for v in read)
    wo, qo = yaw_quat(tho)
    we, qe = yaw_quat(the)
    v = the - tho
    P = dict(cos_e=F32(math.cos(float(the))), sin_e=F32(math.sin(float(the))),
             cos_emo=F32(math.cos(float(v))), sin_emo=F32(math.sin(float(v))))
    iw, iz = we, -qe
    r0, r1, r2 = _rotate_yaw(iw, iz, xe, ye, ze)
    ti0, ti1, ti2 = -r0, -r1, -r2
    P["qw"] = iw * wo - iz * qo
    P["qz"] = iw * qo + iz * wo
    r0, r1, r2 = _rotate_yaw(iw, iz, xo, yo, zo)
    P["tx"], P["ty"], P["tz"] = ti0 + r0, ti1 + r1, ti2 + r2
    return P


def check_pose_block(oracle, ref, read):
    """oracle.reg_pose_setup (libm trig) == the device restatement, value for value."""
    T, trig = oracle.reg_pose_setup(ref, read)
    P = pose_block(ref, read)
    got = [T[0], T[3], T[4], T[5], T[6], trig[0], trig[1], trig[2], trig[3]]
    want = [P[k] for k in ("qw", "qz", "tx", "ty", "tz", "cos_e", "sin_e", "cos_emo", "sin_emo")]
    assert all(F32(g) == w for g, w in zip(got, want)), (ref, read, got, want)
    return P


# --------------------------------------------------------------------------- exact reference
BOUND_ULP = 2.0 ** -50


class Exact:
    """Exact per-entry sums of the registration terms: cost, g (4N), H (4N x 4N), per-block costs.
    Each entry keeps its exact sum, the exact sum of |terms| and the number of contributing
    residuals."""

    def __init__(self, n_nodes):
        self.N = n_nodes
        self._terms = {}      # key -> list of term arrays
        self._count = {}
        self.block_cost = []  # (exact, sum|t|, n) per residual block

    def _add(self, key, t, n):
        self._terms.setdefault(key, []).append(t)
        self._count[key] = self._count.get(key, 0) + n

    def add_block(self, ia, ib, r, jr, je):
        """One residual block with node indices (ia: reference, ib: reading) and the oracle's
        normalised residuals / Jacobians."""
        n = len(r)
        J = np.concatenate([jr, je], axis=1)
        cols = [4 * ia + k for k in range(4)] + [4 * ib + k for k in range(4)]
        rr = r * r
        self.block_cost.append((math.fsum(rr.tolist()), math.fsum(rr.tolist()), n))
        self._add(("c",), 0.5 * rr, n)
        for i in range(8):
            self._add(("g", cols[i]), J[:, i] * r, n)
            for j in range(i, 8):
                p, q = min(cols[i], cols[j]), max(cols[i], cols[j])
                self._add(("H", p, q), J[:, i] * J[:, j], n)

    def finish(self):
        """-> dict key -> (exact sum, sum |t|, n)"""
        out = {}
        for key, arrs in self._terms.items():
            t = np.concatenate(arrs).tolist()
            out[key] = (math.fsum(t), math.fsum(abs(v) for v in t), self._count[key])
        self.sums = out
        return out


def _ratio(fused, exact, abs_sum, n):
    """|fused - exact| / bound; an entry without terms must be exactly 0 (ratio 0 or inf)."""
    if abs_sum == 0.0:
        return 0.0 if fused == 0.0 else math.inf
    d = abs(Fraction(fused) - Fraction(exact))
    return float(d / (Fraction(BOUND_ULP) * (n + 64) * Fraction(abs_sum)))


def check_bound(ex, cost, g, H, per_block=None, label=""):
    """Cost, every g and H entry and (optionally) every per-block cost of the fused evaluation within
    2^-50 (n + 64) sum|t| of the exact sums.  Returns the largest ratio to the bound."""
    s = ex.sums
    dim = 4 * ex.N
    worst = 0.0
    where = None

    def upd(r, w):
        nonlocal worst, where
        if r > worst:
            worst, where = r, w

    c = s.get(("c",), (0.0, 0.0, 0))
    upd(_ratio(cost, *c), "cost")
    for p in range(dim):
        upd(_ratio(g[p], *s.get(("g", p), (0.0, 0.0, 0))), ("g", p))
        for q in range(dim):
            upd(_ratio(H[p, q], *s.get(("H", min(p, q), max(p, q)), (0.0, 0.0, 0))), ("H", p, q))
    if per_block is not None:
        assert len(per_block) == len(ex.block_cost)
        for k, (e, a, n) in enumerate(ex.block_cost):
            upd(_ratio(per_block[k], e, a, n), ("block", k))
    assert worst <= 1.0, "%s: fused sum beyond the exact-sum bound at %s (ratio %.3g)" % (label, where, worst)
    return worst


def check_costs_bound(ex, per_block, label=""):
    worst = 0.0
    assert len(per_block) == len(ex.block_cost)
    for k, (e, a, n) in enumerate(ex.block_cost):
        r = _ratio(per_block[k], e, a, n)
        assert r <= 1.0, "%s: per-constraint cost %d beyond the bound (ratio %.3g)" % (label, k, r)
        worst = max(worst, r)
    return worst


# --------------------------------------------------------------------------- cull restatement
COORD_EPS = F32(1e-6)
MARGIN_S = F32(2.0 ** -16)     # reg_unit_may_hit: S * 2^-16
MARGIN_R = F32(2.0 ** -10)     # reg_unit_may_hit: r * 2^-10


def transform(P, x):
    """vgx_reg_transform on (n, 3) float32 points."""
    x = np.asarray(x, F32)
    r0, r1, r2 = _rotate_yaw(P["qw"], P["qz"], x[:, 0], x[:, 1], x[:, 2])
    return np.stack([r0 + P["tx"], r1 + P["ty"], r2 + P["tz"]], -1)


def block_index(p, block_size_inv):
    """vgx_block_index on (n, 3) float32 points -> int64 block indices."""
    p = np.asarray(p, F32)
    return np.floor(p * F32(block_size_inv) + COORD_EPS).astype(np.int64)


def _square_below(s, v):
    """s * s < v exactly, for float64 arrays (Dekker's product: no FMA, no rounding)."""
    c = 134217729.0 * s
    hi = c - (c - s)
    lo = s - hi
    p = s * s
    e = ((hi * hi - p) + 2.0 * hi * lo) + lo * lo
    return (p < v) | ((p == v) & (e < 0))


def unit_bounds(pts, w, d=None):
    """reg_unit_bounds_kernel for (U, 32, 3) points and (U, 32) weights -> (U, 4) float32 spheres.
    Points of weight 0 with finite values are left out; a unit without any point, or with a counted
    non-finite point, gets radius inf (never culled)."""
    pts = np.asarray(pts, F32)
    w = np.asarray(w, F32)
    d = np.zeros(w.shape, F32) if d is None else np.asarray(d, F32)
    fin = np.isfinite(pts).all(2)
    inn = ~((w == 0) & fin & np.isfinite(d))
    never = (inn & ~fin).any(1) | ~inn.any(1)
    with np.errstate(invalid="ignore", over="ignore"):
        lo = np.where(inn[..., None], pts, F32(np.inf)).min(1)
        hi = np.where(inn[..., None], pts, F32(-np.inf)).max(1)
        c = F32(0.5) * (lo + hi)
        e = pts.astype(np.float64) - c[:, None, :].astype(np.float64)
        r2 = np.where(inn, (e[..., 0] * e[..., 0] + e[..., 1] * e[..., 1]) + e[..., 2] * e[..., 2], 0.0).max(1)
        r2 = np.where(never, 0.0, r2)
        s = np.sqrt(r2)                                   # __dsqrt_ru
        s = np.where(_square_below(s, r2), np.nextafter(s, np.inf), s)
        f = s.astype(F32)                                 # __double2float_ru
        f = np.where(f.astype(np.float64) < s, np.nextafter(f, F32(np.inf)), f)
    out = np.concatenate([c, f[:, None]], 1).astype(F32)
    out[never] = [np.nan, np.nan, np.nan, np.inf]
    return out


def cull_box(P, b, margin=True, margin_s=None):
    """The reading-frame box reg_unit_may_hit tests for (U, 4) spheres: (centre - R, centre + R) in
    float32, as the kernel rounds them.  margin=False: R = radius.  -> (centre, R, low, high, S)"""
    b = np.asarray(b, F32)
    c = transform(P, b[:, :3])
    n1 = np.abs(P["qw"] * P["qw"] + P["qz"] * P["qz"] - F32(1.0))
    ms = MARGIN_S if margin_s is None else F32(margin_s)
    S = ((np.abs(b[:, 0]) + np.abs(b[:, 1])) + (np.abs(b[:, 2]) + F32(3.0) * b[:, 3])) + \
        ((np.abs(P["tx"]) + np.abs(P["ty"])) + np.abs(P["tz"]))
    with np.errstate(invalid="ignore", over="ignore"):
        R = b[:, 3] + (b[:, 3] * (F32(2.0) * n1 + MARGIN_R) + S * ms) if margin else b[:, 3]
        return c, R, c - R[:, None], c + R[:, None], S


def may_hit(P, grid, b, margin=True, margin_s=None):
    """reg_unit_may_hit for (U, 4) spheres.  grid: dict(gmin (3,), occ (gd2, gd1, gd0) bool,
    block_size_inv).  margin=False drops both margin terms (R = radius): the test a unit would get
    without the float error argument."""
    c, R, L, H, _ = cull_box(P, b, margin, margin_s)
    with np.errstate(invalid="ignore", over="ignore"):
        fin = np.isfinite((c[:, 0] + c[:, 1]) + (c[:, 2] + R))
        lo = block_index(L, grid["block_size_inv"])
        hi = block_index(H, grid["block_size_inv"])
    occ = grid["occ"]
    gd = np.array([occ.shape[2], occ.shape[1], occ.shape[0]])
    out = np.ones(len(b), bool)
    for u in range(len(b)):
        if not fin[u]:
            continue
        a = np.maximum(np.minimum(lo[u], hi[u]) - grid["gmin"], 0)
        z = np.minimum(np.maximum(lo[u], hi[u]) - grid["gmin"], gd - 1)
        if (a > z).any():
            out[u] = False
            continue
        if np.prod(z - a + 1) > 27:
            continue
        out[u] = bool(occ[a[2]:z[2] + 1, a[1]:z[1] + 1, a[0]:z[0] + 1].any())
    return out


def make_grid(block_idx, block_size_inv):
    """The reading submap's block grid over its block AABB (vgx_submap_build_grid)."""
    bi = np.asarray(block_idx, np.int64)
    gmin = bi.min(0); gdim = bi.max(0) - gmin + 1
    occ = np.zeros((gdim[2], gdim[1], gdim[0]), bool)
    occ[bi[:, 2] - gmin[2], bi[:, 1] - gmin[1], bi[:, 0] - gmin[0]] = True
    return dict(gmin=gmin, occ=occ, block_size_inv=F32(block_size_inv))


def in_grid_blocks(grid, blk):
    """(n, 3) block indices -> bool: the block exists."""
    g = np.asarray(blk, np.int64) - grid["gmin"]
    occ = grid["occ"]
    inside = ((g >= 0) & (g < np.array([occ.shape[2], occ.shape[1], occ.shape[0]]))).all(1)
    out = np.zeros(len(g), bool)
    gi = g[inside]
    out[inside] = occ[gi[:, 2], gi[:, 1], gi[:, 0]]
    return out


# --------------------------------------------------------------------------- culling-edge scene
CULL_VS, CULL_VPS = 0.2, 16
CULL_BLOCKS = [(x, y, z) for z in range(2) for y in range(4) for x in range(4)]
CULL_HOLES = {(1, 1, 0), (2, 1, 0), (1, 2, 1), (2, 2, 1), (0, 3, 0), (3, 0, 1)}
CULL_NORMAL = (0.0, 0.3, 0.953939201416946)


def _inverse(P, p):
    """Reference-frame float32 points that the restated transform maps near p (double inverse)."""
    w, z = float(P["qw"]), float(P["qz"])
    n = w * w + z * z
    c, s = (w * w - z * z) / n, 2 * w * z / n
    q = np.asarray(p, np.float64) - np.array([float(P["tx"]), float(P["ty"]), float(P["tz"])])
    x = np.stack([(c * q[:, 0] + s * q[:, 1]) / n, (-s * q[:, 0] + c * q[:, 1]) / n, q[:, 2]], -1)
    return x.astype(F32)


def _nudge_into(P, p, axis, sign, target, bsi):
    """Points whose restated block index is `target` (n, 3), as close to the face as the float grid
    allows: p moved along axis by sign * k * step for the smallest k that lands in the target."""
    p = np.asarray(p, np.float64)
    step = np.abs(p).max() * 2.0 ** -24 + 1e-7
    best = np.full(len(p), -1)
    cand = None
    out = np.zeros((len(p), 3), F32)
    for k in range(-16, 128):
        q = p.copy()
        q[:, axis] += sign * k * step
        x = _inverse(P, q)
        hit = (block_index(transform(P, x), bsi) == target).all(1) & (best < 0)
        out[hit] = x[hit]
        best[hit] = k
    assert (best >= 0).all()
    return out


def cull_scene(P, offset_blocks, rng, layer_bsi):
    """Reading blocks (4 x 4 x 2 with six holes, shifted by offset_blocks along x) and reference units
    built on the cull decision for the pose block P.  Returns dict(block_idx, distance, weight,
    xyz, d, w (reference points, whole units), kinds (per unit))."""
    vs, vps = CULL_VS, CULL_VPS
    bs = float(F32(vs) * F32(vps))
    blocks = [(x + offset_blocks, y, z) for (x, y, z) in CULL_BLOCKS if (x, y, z) not in CULL_HOLES]
    lo = (offset_blocks, 0, 0)
    from voxgraph_b200 import synth
    idx, dist, wt = synth.plane_layer_blocks(CULL_NORMAL, 0.9, vs, vps,
                                             ((lo[0], lo[0] + 3), (0, 3), (0, 1)))
    keep = np.array([tuple(b) in set(blocks) for b in idx.tolist()])
    idx, dist, wt = idx[keep], dist[keep], wt[keep]
    grid = make_grid(idx, layer_bsi)
    exist = set(map(tuple, idx.tolist()))
    # faces between an existing block E and a missing neighbour M inside the AABB
    faces = []
    for (hx, hy, hz) in sorted(CULL_HOLES):
        m = (hx + offset_blocks, hy, hz)
        for axis in range(3):
            for sgn in (-1, 1):
                e = list(m); e[axis] += sgn
                if tuple(e) in exist:
                    faces.append((np.array(e), np.array(m), axis, sgn))

    def field(p):
        return (p @ np.asarray(CULL_NORMAL) - 0.9).astype(F32)

    units, kinds = [], []

    def unit(x, kind, w=None):
        x = np.asarray(x, F32)
        p = transform(P, x).astype(np.float64)
        d = field(p) + rng.normal(0, 0.02, len(x)).astype(F32)
        w = rng.uniform(0.5, 2.0, len(x)).astype(F32) if w is None else np.asarray(w, F32)
        units.append((x, d, w)); kinds.append(kind)

    def in_block(b, n, inset=0.3):
        return (np.asarray(b, np.float64) + rng.uniform(inset / bs, 1 - inset / bs, (n, 3))) * bs

    S_margin = 2.0 ** -16 * (3 * bs * (abs(offset_blocks) + 4) + 8)
    for (e, m, axis, sgn) in faces:
        face = (max(e[axis], m[axis])) * bs      # coordinate of the shared face
        into_e = sgn                             # direction from the face into E
        # (1) face huggers: 12 points a few ulps inside E, 20 outside in M by up to 5 cm
        base = in_block(e, 1)[0]
        p = np.repeat(base[None], 32, 0) + rng.uniform(-0.05, 0.05, (32, 3))
        p[:, axis] = face
        x_in = _nudge_into(P, p[:12], axis, into_e, e, layer_bsi)
        q = p[12:].copy(); q[:, axis] = face - into_e * rng.uniform(1e-4, 0.05, 20)
        unit(np.concatenate([x_in, _inverse(P, q)]), "hug")
        # (2) radius 0 just outside E, within the margin: live only because of the margin
        q = base.copy(); q[axis] = face - into_e * 0.25 * S_margin
        unit(np.repeat(_inverse(P, q[None]), 32, 0), "r0_margin")
        # (3) radius 0 a few ulps inside E (no correspondence: the base corner is in M)
        q = base.copy(); q[axis] = face
        unit(np.repeat(_nudge_into(P, q[None], axis, into_e, e, layer_bsi), 32, 0), "r0_inside")
        # (4) one live point inside E, 31 weight-0 points far away
        x = np.concatenate([_inverse(P, in_block(e, 1)), np.full((31, 3), 5.0e3, F32) + np.arange(31, dtype=F32)[:, None]])
        w = np.zeros(32, F32); w[0] = 1.5
        unit(x, "one_live", w)
    for (hx, hy, hz) in sorted(CULL_HOLES):
        m = (hx + offset_blocks, hy, hz)
        # radius 0 in the middle of a hole, and a small unit there: culled
        c = (np.asarray(m, np.float64) + 0.5) * bs
        unit(np.repeat(_inverse(P, c[None]), 32, 0), "r0_hole")
        unit(_inverse(P, c + rng.uniform(-0.3, 0.3, (32, 3))), "hole")
    for b in blocks[::2]:
        unit(_inverse(P, in_block(b, 32, 0.05)), "inside")
    order = rng.permutation(len(units))
    units = [units[k] for k in order]; kinds = [kinds[k] for k in order]
    xyz = np.concatenate([u[0] for u in units]); d = np.concatenate([u[1] for u in units])
    w = np.concatenate([u[2] for u in units])
    # a single-point last unit, inside an existing block
    x1 = _inverse(P, in_block(blocks[0], 1))
    xyz = np.concatenate([xyz, x1]); d = np.concatenate([d, field(transform(P, x1).astype(np.float64))])
    w = np.concatenate([w, np.ones(1, F32)]); kinds.append("last")
    return dict(block_idx=idx, distance=dist, weight=wt, xyz=xyz, d=d, w=w, kinds=kinds, grid=grid)


def split_units(xyz, d, w):
    """(n, 3) points -> (U, 32, ...) units, the last one zero-padded as the device pads it."""
    n = len(w)
    U = (n + 31) // 32
    X = np.zeros((U * 32, 3), F32); D = np.zeros(U * 32, F32); W = np.zeros(U * 32, F32)
    X[:n] = xyz; D[:n] = d; W[:n] = w
    return X.reshape(U, 32, 3), D.reshape(U, 32), W.reshape(U, 32)


def cull_report(P, scene):
    """Restated cull decision per unit: (may_hit, may_hit without margin, some counted point lies in
    an existing block)."""
    X, D, W = split_units(scene["xyz"], scene["d"], scene["w"])
    b = unit_bounds(X, W, D)
    grid = scene["grid"]
    mh = may_hit(P, grid, b)
    mh0 = may_hit(P, grid, b, margin=False)
    blk = block_index(transform(P, X.reshape(-1, 3)), grid["block_size_inv"])
    counted = ~((W.reshape(-1) == 0) & np.isfinite(X.reshape(-1, 3)).all(1) & np.isfinite(D.reshape(-1)))
    hits = (in_grid_blocks(grid, blk) & counted).reshape(X.shape[0], 32).any(1)
    return mh, mh0, hits


CULL_BASE_POSES = ((0.5, -0.3, 0.2, 2.5), (1.0, 0.4, -0.1, -1.0), (-0.4, 0.6, 0.3, -2.9), (0.2, 0.1, 0.0, 0.7))
CULL_PAIRS = ((0, 1, 0), (2, 3, 625))   # (reference node, reading node, block offset along x)


def cull_problem_scenes(bsi, seed=5):
    """The culling-edge problem: four exact-trig node poses and two reference/reading pairs built by
    cull_scene, one near the origin and one 2 km away whose pose block has qw^2 + qz^2 != 1 in float.
    Returns (poses (4, 4), [(ref node, read node, P, scene), ...])."""
    rng = np.random.default_rng(seed)
    base = np.array(CULL_BASE_POSES)
    for _ in range(100):
        x = exact_trig_poses(base, [(0, 1), (1, 0), (2, 3), (3, 2)], rng)
        P_far = pose_block(x[2], x[3])
        if P_far["qw"] * P_far["qw"] + P_far["qz"] * P_far["qz"] != F32(1.0):
            break
    else:
        raise AssertionError("no far pose with qw^2 + qz^2 != 1 in float")
    out = []
    for (ref, read, off) in CULL_PAIRS:
        P = pose_block(x[ref], x[read])
        out.append((ref, read, P, cull_scene(P, off, rng, bsi)))
    return x, out
