"""Race-aware model of one Fast TSDF integration call (mode 1, FastTsdfIntegrator scheduling), for
tests/test_oracle_fast_schedule.py and tests/test_gpu_fast_schedule.py.

The Fast schedule (csrc/tsdf.cu tsdf_integrate_kernel) keeps two approximate sets of 2^20 buckets, both
filled with the marker ~0 at the start of every call:
* start set: a valid point's start key floor(pG * (factor / voxel_size) + 1e-6) (float) is exchanged
  into bucket h & (2^20 - 1), h its AnyIndexHash; the ray is cast only when the old value differs from h;
* observation set: a cast ray walks its voxel sequence (from beyond the point back to the sensor,
  cast_from_origin = false) and exchanges every voxel's hash into its bucket.  An old value equal to the
  hash is a collision, anything else resets the count, and the ray stops before updating the voxel at
  which the count exceeds max_consecutive_ray_collisions (m).

The marker is itself a hash: voxel or start key (-1, 0, 0) hashes to 2^64 - 1 (so does (17190, -1, 0)).
The first visit of such a voxel already counts as a collision, and a point whose start cell is (-1, 0, 0)
is never cast.  Device and oracle agree on this.

A cast ray therefore updates a prefix v_1..v_p of its sequence: p = L (the whole ray) or m <= p < L (a
break at v_{p+1}).  `Scene` holds per valid point its start key, its full sequence (oracle.raycast) and
the (sdf, update weight) of every voxel of it (oracle.tsdf_integrate_trace with every ray cast), and:
* `simulate(order)`: the outcome of one sequential order of the points; it equals the oracle's mode-1
  integration of the points fed in that order, bit for bit;
* `reachable()`: every outcome {(cast_r, p_r)} over all interleavings of the start and observation
  exchanges.  The atomics of one call are executed in one order at the L2, and a ray issues its next
  exchange only after the previous one returned (the loop decision depends on it), so every device
  outcome is one of these.  The search is exact, aliasing included: it carries the contents of every
  bucket that two rays touch, and runs the exchanges on a bucket that only one ray touches eagerly
  (they commute with every other step);
* `check(layer, stats)`: for scenes whose rays carry distinct power-of-four weights (1/z^2 with z = 2^j;
  identical points share one), the weight of a voxel spells out which rays updated it, and the checker
  asserts, for any interleaving: (a) each ray's updated voxels are a prefix of its sequence; (b) p = L or
  m <= p < L; (c) after a break, the last m updated voxels and the break voxel were also reached by
  another ray or hash to ~0; (d) the cast counts of the start keys can be produced by one order of the
  start exchanges of each bucket; (e) rays_valid, rays_cast, voxel_updates, blocks_allocated and the block
  set are those of the decoded prefixes (the break voxel allocates nothing); (f) a voxel with one update
  holds it bit for bit, one with k <= 3 updates equals the float32 replay of one of the k! orders, and
  above that the distance lies within tsdf_exact's running-mean bound.
"""
import itertools
import math

import numpy as np

import tsdf_exact as tx

F32 = np.float32
MASK = (1 << 20) - 1
MARKER = (1 << 64) - 1
EPS = F32(1e-6)
SENSORS = {"origin": (0.0, 0.0, 0.0), "negative": (-1.25, -2.5, -0.5)}


def any_index_hash(x, y, z):
    """voxblox AnyIndexHash x + 17191 y + 17191^2 z as uint64."""
    return (int(x) + int(y) * 17191 + int(z) * 17191 * 17191) & MARKER


def pose(t):
    return np.array([1, 0, 0, 0, *t], F32)


class Ray:
    def __init__(self, index, point):
        self.index = index
        self.point = point
        self.valid = False
        self.slot = -1


def start_key(v, inv):
    """Start key of a point: floor(pG * inv + 1e-6) per axis in float, inv = factor / voxel_size."""
    with np.errstate(all="ignore"):
        return tuple(int(np.floor(F32(F32(c) * inv) + EPS)) for c in v)


class Scene:
    """One call's points (sensor frame) at pose T = [1 0 0 0 tx ty tz] or any other pose, and the mode-1
    configuration `cfg` (oracle.tsdf_config keywords; mode is forced to 1).  `m` may be changed
    afterwards: the sequences do not depend on it."""

    def __init__(self, oracle, vs, vps, T, pts, **cfg):
        cfg = dict(cfg, mode=1)
        self.kw = cfg
        c = oracle.tsdf_config(**cfg)
        self.vs, self.vps = vs, int(vps)
        self.sh = int(vps).bit_length() - 1
        self.T = np.asarray(T, F32)
        self.pts = np.ascontiguousarray(pts, F32).reshape(-1, 3)
        self.trunc = F32(c.default_truncation_distance)
        self.M = F32(c.max_weight)
        self.m = int(c.max_consecutive_ray_collisions)
        layer = oracle.Layer(vs, vps)
        vsi = F32(layer.voxel_size_inv)
        inv = F32(F32(c.start_voxel_subsampling_factor) * vsi)
        origin = self.T[4:7]
        self.rays = []
        for i, p in enumerate(self.pts):
            r = Ray(i, p)
            self.rays.append(r)
            if not np.all(np.isfinite(p)):
                continue
            with np.errstate(all="ignore"):
                rd = np.sqrt(F32(F32(F32(p[0] * p[0]) + F32(p[1] * p[1])) + F32(p[2] * p[2])))
            if rd < F32(c.min_ray_length_m):
                continue
            r.clearing = bool(rd > F32(c.max_ray_length_m))
            if r.clearing and not c.allow_clear:
                continue
            r.valid = True
            r.pG = oracle.T_transform(self.T, p)
            r.key = start_key(r.pG, inv)
            r.kh = any_index_hash(*r.key)
            g, n = oracle.raycast(origin, r.pG, vsi, self.trunc, r.clearing, c.voxel_carving_enabled,
                                  c.max_ray_length_m, cast_from_origin=False, max_out=8192)
            assert n <= 8192
            r.seq = [tuple(int(a) for a in v) for v in g]
            r.vh = [any_index_hash(*v) for v in r.seq]
            r.pos = {v: k for k, v in enumerate(r.seq)}
        self.valid = [r.index for r in self.rays if r.valid]
        # identical points share a slot (and a weight); every other pair is told apart by its weight
        slots = {}
        for i in self.valid:
            r = self.rays[i]
            r.slot = slots.setdefault(r.point.tobytes(), len(slots))
        self.slots = [[] for _ in slots]
        for i in self.valid:
            self.slots[self.rays[i].slot].append(i)
        self._trace(oracle, cfg)

    def _trace(self, oracle, cfg):
        """(sdf, update weight) of every voxel of every slot's full sequence: one trace with every ray
        cast (tiny start cells, unlimited collisions), split by sequence length; point by point when two
        slots still share a start cell."""
        every = dict(cfg, start_voxel_subsampling_factor=1e3, max_consecutive_ray_collisions=1 << 30)
        reps = [self.rays[s[0]] for s in self.slots]
        if not reps:
            return
        ocfg = oracle.tsdf_config(**every)
        st, g, s, u = oracle.tsdf_integrate_trace(oracle.Layer(self.vs, self.vps), ocfg, self.T,
                                                  np.array([r.point for r in reps]))
        if st.rays_cast == len(reps):
            parts = np.cumsum([len(r.seq) for r in reps])[:-1]
            traces = zip(np.split(g, parts), np.split(s, parts), np.split(u, parts))
        else:
            traces = [oracle.tsdf_integrate_trace(oracle.Layer(self.vs, self.vps), ocfg, self.T,
                                                  r.point[None])[1:] for r in reps]
        for r, (gg, ss, uu) in zip(reps, traces):
            assert [tuple(v) for v in gg.tolist()] == r.seq, "trace and raycast sequences differ"
            for i in self.slots[r.slot]:
                self.rays[i].sdf, self.rays[i].uw = ss, uu

    # ------------------------------------------------------------------ sequential outcome
    def simulate(self, order=None):
        """The outcome of the points taken one after another in `order` (default: as listed):
        {ray index: (cast, p)}."""
        order = range(len(self.rays)) if order is None else order
        start, obs, out = {}, {}, {}
        for i in order:
            r = self.rays[i]
            if not r.valid:
                continue
            b = r.kh & MASK
            old = start.get(b, MARKER); start[b] = r.kh
            if old == r.kh:
                out[i] = (False, 0)
                continue
            p, coll = len(r.vh), 0
            for k, h in enumerate(r.vh):
                b = h & MASK
                old = obs.get(b, MARKER); obs[b] = h
                coll = coll + 1 if old == h else 0
                if coll > self.m:
                    p = k
                    break
            out[i] = (True, p)
        return out

    def updates(self, outcome, order=None):
        """(ray, position) updates of an outcome in the order a sequential run applies them."""
        order = range(len(self.rays)) if order is None else order
        return [(i, k) for i in order if i in outcome for k in range(outcome[i][1])]

    def stats(self, outcome, extra_blocks=()):
        ups = self.updates(outcome)
        return (len(self.valid), sum(c for c, _ in outcome.values()), len(ups),
                len(self.blocks_of(ups) | set(extra_blocks)))

    def block(self, g):
        return tuple(a >> self.sh for a in g)

    def blocks_of(self, ups):
        return {self.block(self.rays[i].seq[k]) for i, k in ups}

    def layer(self, ups, extra_blocks=()):
        """Layer (block indices, distance, weight) after applying the updates in the order listed into an
        empty submap, with every block of an updated voxel plus `extra_blocks` allocated."""
        vox = {}
        for i, k in ups:
            r = self.rays[i]
            g = r.seq[k]
            d, w = vox.get(g, (F32(0), F32(0)))
            d, w = tx.apply_update(r.sdf[k], r.uw[k], d, w, self.trunc, self.M)
            vox[g] = (F32(d), F32(w))
        blocks = sorted({self.block(g) for g in vox} | set(extra_blocks))
        slot = {b: n for n, b in enumerate(blocks)}
        n3 = self.vps ** 3
        idx = np.array(blocks, np.int32).reshape(-1, 3)
        dd = np.zeros((len(blocks), n3), F32); ww = np.zeros((len(blocks), n3), F32)
        mask = self.vps - 1
        for g, (d, w) in vox.items():
            lin = (g[0] & mask) + self.vps * ((g[1] & mask) + self.vps * (g[2] & mask))
            dd[slot[self.block(g)], lin] = d; ww[slot[self.block(g)], lin] = w
        return idx, dd, ww

    # ------------------------------------------------------------------ all interleavings
    def reachable(self, max_states=1_000_000):
        """Every outcome over all interleavings of the exchanges: a set of tuples ((cast, p) per valid
        ray, in self.valid order)."""
        R = [self.rays[i] for i in self.valid]
        users = {}
        for ri, r in enumerate(R):
            users.setdefault(("s", r.kh & MASK), set()).add(ri)
            for h in r.vh:
                users.setdefault(("o", h & MASK), set()).add(ri)
        shared = sorted(b for b, u in users.items() if len(u) > 1)
        sid = {b: n for n, b in enumerate(shared)}
        s_op = [sid.get(("s", r.kh & MASK), -1) for r in R]
        o_op = [[sid.get(("o", h & MASK), -1) for h in r.vh] for r in R]
        prev = []          # old value of a local exchange: the ray's own last write to that bucket
        for r in R:
            last, pv = {}, []
            for h in r.vh:
                pv.append(last.get(h & MASK, MARKER)); last[h & MASK] = h
            prev.append(pv)
        m = self.m

        def step(ri, rs, sh):
            """Run ray ri's next exchange; status 0 = before its start exchange, 1 = walking, 2 = done
            (p = pos), 3 = skipped."""
            r = R[ri]
            pos, coll, st = rs
            if st == 0:
                b = s_op[ri]
                old = MARKER
                if b >= 0:
                    old = sh[b]; sh = sh[:b] + (r.kh,) + sh[b + 1:]
                if old == r.kh:
                    return (0, 0, 3), sh
                return ((0, 0, 1) if r.vh else (0, 0, 2)), sh
            h = r.vh[pos]; b = o_op[ri][pos]
            if b >= 0:
                old = sh[b]; sh = sh[:b] + (h,) + sh[b + 1:]
            else:
                old = prev[ri][pos]
            coll = coll + 1 if old == h else 0
            if coll > m:
                return (pos, 0, 2), sh
            pos += 1
            return ((pos, 0, 2) if pos == len(r.vh) else (pos, coll, 1)), sh

        def local_next(ri, rs):
            pos, _, st = rs
            if st == 0:
                return s_op[ri] < 0
            return st == 1 and o_op[ri][pos] < 0

        def close(ri, rs, sh):
            while local_next(ri, rs):
                rs, sh = step(ri, rs, sh)
            return rs, sh

        sh0 = (MARKER,) * len(shared)
        rs0 = []
        for ri in range(len(R)):
            rs, sh0 = close(ri, (0, 0, 0), sh0)
            rs0.append(rs)
        init = (tuple(rs0), sh0)
        seen, stack, out = {init}, [init], set()
        while stack:
            rss, sh = stack.pop()
            live = [ri for ri, rs in enumerate(rss) if rs[2] < 2]
            if not live:
                out.add(tuple((rs[2] == 2, rs[0] if rs[2] == 2 else 0) for rs in rss))
                continue
            for ri in live:
                rs, sh2 = step(ri, rss[ri], sh)
                rs, sh2 = close(ri, rs, sh2)
                nxt = (rss[:ri] + (rs,) + rss[ri + 1:], sh2)
                if nxt not in seen:
                    seen.add(nxt); stack.append(nxt)
                    assert len(seen) <= max_states, "interleaving search too large"
        return out

    def canonical(self, outcome):
        """(updates per slot, rays cast) of an outcome: what a decoded layer and its stats show.  An
        outcome in which two rays of one slot update voxels shows as -1 (the decoder rejects it)."""
        if not isinstance(outcome, dict):
            outcome = dict(zip(self.valid, outcome))
        ps = []
        for s in self.slots:
            nz = [outcome[i][1] for i in s if outcome[i][1] > 0]
            ps.append(-1 if len(nz) > 1 else sum(nz))
        return tuple(ps), sum(c for c, _ in outcome.values())

    # ------------------------------------------------------------------ decoding and checking
    def slot_weight(self, s):
        r = self.rays[self.slots[s][0]]
        w = float(r.uw[0])
        assert np.all(r.uw == r.uw[0]), "a ray's update weight varies along it"
        mant, e = math.frexp(w)
        assert mant == 0.5 and (e - 1) % 2 == 0, ("not a power of four", w)
        return w

    def decodable(self):
        ws = [self.slot_weight(s) for s in range(len(self.slots))]
        return len(set(ws)) == len(ws)

    def decode(self, layer):
        """Layer -> ({voxel: (distance, weight)} of the touched voxels, updated prefix length per slot).
        Raises AssertionError when a weight is not a sum of distinct slot weights (a duplicated update)
        or a slot's voxels are not a prefix of its sequence."""
        idx, d, w = (np.asarray(a) for a in layer)
        vps, n3 = self.vps, self.vps ** 3
        lin = np.arange(n3)
        loc = np.stack([lin % vps, (lin // vps) % vps, lin // (vps * vps)], -1)
        vox = {}
        for b in range(len(idx)):
            hit = np.nonzero((w[b] != 0) | (d[b] != 0))[0]
            for v in hit:
                g = tuple(int(a) for a in idx[b].astype(np.int64) * vps + loc[v])
                vox[g] = (F32(d[b, v]), F32(w[b, v]))
        ws = [self.slot_weight(s) for s in range(len(self.slots))]
        emin = min((math.frexp(x)[1] for x in ws), default=0) - 1
        bit = [int(math.log2(x)) - emin for x in ws]
        sets = [set() for _ in ws]
        for g, (dv, wv) in vox.items():
            x = float(wv) * 2.0 ** -emin
            assert x == int(x) and x > 0, ("weight is not a sum of ray weights", g, float(wv))
            n = int(x)
            for s, bb in enumerate(bit):
                if n >> bb & 1:
                    sets[s].add(g); n &= ~(1 << bb)
            assert n == 0, ("weight is not a sum of distinct ray weights", g, float(wv))
        ps = []
        for s, vs in enumerate(sets):
            r = self.rays[self.slots[s][0]]
            pos = sorted(r.pos.get(g, -1) for g in vs)
            assert pos == list(range(len(vs))), ("(a) updated voxels are not a prefix of the ray", s, pos[:8])
            ps.append(len(vs))
        return vox, ps

    def check(self, layer, stats, reach=None):
        """Assert rules (a)-(f) for a layer (block indices, distance, weight) integrated into an empty
        submap and its stats (rays_valid, rays_cast, voxel_updates, blocks_allocated), and, given the
        canonical reachable outcomes `reach`, that the decoded outcome is one of them.  Returns the
        decoded (updates per slot, rays_cast) and counts of breaks, skips and ~0 collisions."""
        vox, ps = self.decode(layer)
        m = self.m
        p = {i: 0 for i in self.valid}
        for s, pp in enumerate(ps):
            p[self.slots[s][0]] = pp
        valid, cast, n_upd, n_blk = (int(v) for v in stats)
        assert valid == len(self.valid), ("(e) rays_valid", valid, len(self.valid))
        # (b)
        for i in self.valid:
            L = len(self.rays[i].seq)
            assert p[i] == 0 or p[i] == L or m <= p[i] < L, ("(b) prefix length", i, p[i], L, m)
        # (c) voxels another ray (possibly) exchanged: a ray with p = 0 may have been cast when m = 0
        visited = {}
        for i in self.valid:
            r = self.rays[i]
            n = len(r.vh) if p[i] == len(r.vh) else p[i] + 1
            if p[i] == 0 and m > 0:
                n = 0
            visited[i] = set(r.vh[:n])
        breaks = marker = 0
        for i in self.valid:
            r = self.rays[i]
            if not 0 < p[i] < len(r.vh):
                continue
            breaks += 1
            others = set().union(*(visited[j] for j in self.valid if j != i))
            for k in range(p[i] - m, p[i] + 1):
                h = r.vh[k]
                assert h == MARKER or h in others or h in r.vh[:k], \
                    ("(c) break without a collision", i, k, r.seq[k], p[i], m)
        for i in self.valid:
            marker += MARKER in visited[i]
        # (d) start keys, bucket by bucket: which cast counts can one order of the exchanges give?
        buckets = {}
        for i in self.valid:
            r = self.rays[i]
            buckets.setdefault(r.kh & MASK, {}).setdefault(r.kh, []).append(i)
        totals = {0}
        for keys in buckets.values():
            lo = {h: sum(p[i] > 0 for i in rays) for h, rays in keys.items()}
            exact = m > 0
            poss = {sum(c) for c in _bucket_casts(keys) if all(
                (c[n] == lo[h]) if exact else (c[n] >= lo[h]) for n, h in enumerate(keys))}
            assert poss, ("(d) start-key casts", {h: len(v) for h, v in keys.items()}, lo)
            totals = {a + b for a in totals for b in poss}
        assert cast in totals, ("(d)/(e) rays_cast", cast, sorted(totals))
        marker += sum(len(v) for k in buckets.values() for h, v in k.items() if h == MARKER)
        # (e) updates and blocks
        ups = [(i, k) for i in self.valid for k in range(p[i])]
        assert n_upd == len(ups), ("(e) voxel_updates", n_upd, len(ups))
        blocks = self.blocks_of(ups)
        assert n_blk == len(blocks), ("(e) blocks_allocated", n_blk, len(blocks))
        got_blocks = {tuple(int(a) for a in b) for b in np.asarray(layer[0]).reshape(-1, 3)}
        assert got_blocks == blocks, ("(e) block set", sorted(got_blocks ^ blocks)[:4])
        # (f) distances
        per = {}
        for i, k in ups:
            r = self.rays[i]
            per.setdefault(r.seq[k], []).append((r.sdf[k], r.uw[k]))
        assert set(per) == set(vox), "(f) touched voxels differ from the decoded updates"
        for g, u in per.items():
            dv, wv = vox[g]
            if len(u) <= 3:
                cands = set()
                for perm in itertools.permutations(u):
                    d0, w0 = F32(0), F32(0)
                    for s, uw in perm:
                        d0, w0 = tx.apply_update(s, uw, d0, w0, self.trunc, self.M)
                    cands.add((F32(d0).tobytes(), F32(w0).tobytes()))
                assert (dv.tobytes(), wv.tobytes()) in cands, ("(f) distance", g, len(u), float(dv))
            else:
                s = np.array([a for a, _ in u], np.float64); uw = np.array([b for _, b in u], np.float64)
                if s.min() >= 2.0 * float(self.trunc):
                    assert dv == self.trunc, ("(f) not +trunc", g, float(dv))
                elif np.abs(s).max() <= float(self.trunc) and uw.sum() <= float(self.M):
                    mean = math.fsum(s * uw) / math.fsum(uw)
                    n = len(u)
                    bound = tx.C_MEAN * n * tx.U * np.abs(s).max() * (1 + tx.C_MEAN * n * tx.U)
                    assert abs(float(dv) - mean) <= bound, ("(f) mean", g, n, float(dv), mean)
        decoded = (tuple(ps), cast)
        assert reach is None or decoded in reach, ("outcome no interleaving produces", decoded, sorted(reach)[:6])
        return dict(decoded=decoded, breaks=breaks, skips=valid - cast, marker=marker)


def _bucket_casts(keys):
    """Cast counts per key (tuple in `keys` order) that one order of the start exchanges of one bucket
    can give.  The exchanges form runs of one key; a run's first exchange casts unless the bucket held
    the same hash before, which happens only for the first run when the key hashes to the marker ~0."""
    hs = list(keys)
    n = [len(keys[h]) for h in hs]
    out = set()
    for runs in itertools.product(*(range(1, k + 1) for k in n)):
        tot = sum(runs)
        for first in range(len(hs)):
            # runs with no two neighbours equal and key `first` leading
            if runs[first] > tot - runs[first] + 1:
                continue
            if any(runs[j] > tot - runs[j] for j in range(len(hs)) if j != first):
                continue
            out.add(tuple(r - (j == first and hs[j] == MARKER) for j, r in enumerate(runs)))
    return out


# ---------------------------------------------------------------------- scenes
FACTORS = [1, 2, 4]
MS = [0, 1, 2, 7]
RES = [(0.05, 8), (0.1, 16), (0.2, 16)]

def random_scene(oracle, rs, n_max=11):
    """A decoded scene: up to n_max rays with distinct power-of-four weights (z = 2^j, j in -9..1),
    random directions within a cone, a few exact duplicates and near twins in one start cell, random
    collision limit, start-cell factor, resolution and sensor."""
    vs, vps = RES[rs.randint(len(RES))]
    factor = FACTORS[rs.randint(3)]
    m = MS[rs.randint(4)]
    t = SENSORS[["origin", "negative"][rs.randint(2)]]
    u = float(F32(vs))
    n = rs.randint(2, n_max + 1)
    js = rs.permutation(np.arange(-9, 2))[:n]
    az0 = rs.uniform(0, 2 * np.pi)
    spread = rs.choice([0.05, 0.3, 1.5, 6.3])
    pts = []
    for j in js:
        if pts and rs.rand() < 0.15:
            pts.append(pts[rs.randint(len(pts))])          # an exact duplicate (same slot)
            continue
        if pts and rs.rand() < 0.15 and j <= -7:
            x, y, _ = pts[rs.randint(len(pts))]              # a near twin: same x, y, other small z
        else:
            a = az0 + rs.uniform(-spread, spread) / 2
            d = rs.uniform(3.0, 25.0) * u
            x, y = d * np.cos(a), d * np.sin(a)
        pts.append((x, y, 2.0 ** j))
    cfg = dict(BASE, default_truncation_distance=float(rs.choice([2, 3, 5])) * u,
               start_voxel_subsampling_factor=float(factor), max_consecutive_ray_collisions=m,
               voxel_carving_enabled=int(rs.rand() < 0.85))
    sc = Scene(oracle, vs, vps, pose(t), np.array(pts, F32), **cfg)
    assert sc.decodable()
    return sc


MICRO_NAMES = ["collinear", "crossing", "duplicates", "one_cell", "one_bucket", "marker", "clearing",
               "carving_off"]
BASE = dict(use_const_weight=0, use_weight_dropoff=0, use_sparsity_compensation_factor=0,
            max_weight=float(2 ** 23))


def micro_scene(name, vs, factor, sensor):
    """(T, points in the sensor frame, cfg) of a micro scene.  Geometry in voxel units u around the
    sensor; every point's sensor-frame z is 2^-8, 2^-9 or 2^-10 (weights 4^8, 4^9, 4^10, told apart in
    any sum), small enough that points a few voxels apart in x and y share their z start cell."""
    t = SENSORS[sensor]
    T = pose(t)
    u = float(F32(vs))
    cell = u / factor
    z8, z9, z10 = 2.0 ** -8, 2.0 ** -9, 2.0 ** -10
    cfg = dict(BASE, default_truncation_distance=3 * u, start_voxel_subsampling_factor=float(factor))

    def at_cell(cx, cy, fx, fy):
        """Sensor-frame x, y of a point at fraction (fx, fy) of the start cell (cx, cy) counted from the
        sensor's own cell."""
        kx, ky = math.floor(t[0] / cell), math.floor(t[1] / cell)
        return (kx + cx + fx) * cell - t[0], (ky + cy + fy) * cell - t[1]

    if name == "collinear":        # the short ray's sequence lies inside the long one's
        a, b = 14.3 * u, 5.7 * u
        pts = [(a, b, z9), (a / 2, b / 2, z10)]
    elif name == "crossing":       # two rays at a wide angle: they meet at the sensor voxels only
        pts = [(9.3 * u, 2.2 * u, z8), (-1.7 * u, 10.4 * u, z9)]
    elif name == "duplicates":     # one of the two equal points is cast, the other is skipped
        pts = [(7.6 * u, -6.1 * u, z8), (7.6 * u, -6.1 * u, z8), (-8.2 * u, -3.3 * u, z9)]
    elif name == "one_cell":       # two distinct points in one start cell
        x1, y1 = at_cell(10, 4, 0.3, 0.6)
        x2, y2 = at_cell(10, 4, 0.65, 0.3)
        pts = [(x1, y1, z8), (x2, y2, z9), (-6.0 * u, 5.0 * u, z10)]
    elif name == "one_bucket":     # start keys (75, -61, 0) apart: hashes 2^20 apart, one bucket
        x1, y1 = at_cell(37, -31, 0.5, 0.5)
        x2, y2 = at_cell(-38, 30, 0.5, 0.5)
        pts = [(x1, y1, z8), (x2, y2, z9)]
        cfg["max_ray_length_m"] = 40.0
    elif name == "marker":         # at the origin: a ray through voxel (-1, 0, 0), a start cell (-1, 0, 0)
        pts = [(-4.3 * u, 0.45 * u, z9), (-0.5 * cell, 0.5 * cell, z10), (3.2 * u, -5.1 * u, z8)]
        cfg["min_ray_length_m"] = 0.0
    elif name == "marker_block":   # sensor at (-5.5u, 0.5u, 0): a ray enters block (-1, 0, 0) at voxel (-1, 0, 0)
        T = pose((-5.5 * u, 0.5 * u, 0.0))
        pts = [(8.8 * u, -0.1 * u, z8), (8.8 * u, -0.1 * u, z8)]     # every other ray would end in that block
    elif name == "clearing":       # a clearing ray over a short ray in nearly its direction
        pts = [(13.1 * u, 3.3 * u, z8), (5.2 * u, 1.1 * u, z9)]
        cfg["max_ray_length_m"] = 8 * u
    elif name == "carving_off":    # three overlapping truncation bands without carving
        pts = [(8.1 * u, 2.9 * u, z8), (8.6 * u, 3.3 * u, z9), (7.7 * u, 2.6 * u, z10)]
        cfg["voxel_carving_enabled"] = 0
    else:
        raise KeyError(name)
    return T, np.array(pts, F32), cfg


def assert_micro_property(sc, name, sensor):
    """The property the micro scene was built for holds (so a scene cannot silently test less)."""
    R = [sc.rays[i] for i in sc.valid]
    if name == "duplicates":
        assert R[0].key == R[1].key
    elif name == "one_cell":
        assert R[0].key == R[1].key and not np.array_equal(R[0].point, R[1].point)
    elif name == "one_bucket":
        assert R[0].key != R[1].key and R[0].kh & MASK == R[1].kh & MASK
    elif name == "marker" and sensor == "origin":
        assert R[1].kh == MARKER and MARKER in R[0].vh
    elif name == "marker_block":
        k = R[0].seq.index((-1, 0, 0))
        assert all(sc.block(g) != sc.block((-1, 0, 0)) for g in R[0].seq[:k])
    elif name == "marker_block":   # sensor at (-5.5u, 0.5u, 0): a ray enters block (-1, 0, 0) at voxel (-1, 0, 0)
        T = pose((-5.5 * u, 0.5 * u, 0.0))
        pts = [(8.8 * u, -0.1 * u, z8), (8.8 * u, -0.1 * u, z8)]     # every other ray would end in that block
    elif name == "clearing":
        assert R[0].clearing and not R[1].clearing
    assert len(R) == len(sc.pts)
