"""Registration lookup points over the finishSubmap layer matrix (tests/finish_exact.py), for
tests/test_oracle_registration_layers.py and tests/test_gpu_registration_layers.py.  Test support, not
product code.

`points(layer)` builds, in reading-frame coordinates (float32), the places where the interpolator's
block and voxel selection can go wrong:
  * voxel centres (a seeded subset, at most CENTRES per layer);
  * voxel corners, where 8 voxels meet;
  * points on block faces and on voxel-centre planes, and one float ulp either side (np.nextafter);
  * points inside missing blocks that border existing ones (face, edge and corner neighbours);
  * random points over the block AABB grown by one block;
  * far points: inside every real block shifted by +-2^21 on each axis (the shift that aliases in the
    21-bit hash key), and inside blocks just beyond both ends of the index range.
Far points are kept only where the block that contains them, computed as the kernels compute it, lies
outside [INDEX_MIN, INDEX_MAX]: no block can exist there, so the reference finds no correspondence.
Every block index stays below 2^31 in magnitude (the oracle's (int32_t)floorf is undefined beyond).
"""
import numpy as np

import finish_exact as fx

F32 = np.float32
CENTRES = 20000
ALIAS = 1 << 21          # block index shift that packs to the same 21-bit key field


def contain_block(p, bsi):
    """vgx_block_index / getGridIndexFromPoint on float32 points -> int64 block indices."""
    p = np.asarray(p, F32)
    return np.floor((p * F32(bsi)).astype(F32) + fx._EPS).astype(np.int64)


def in_range(b):
    b = np.asarray(b, np.int64)
    return ((b >= fx.INDEX_MIN) & (b <= fx.INDEX_MAX)).all(1)


def _key(b):
    """vgx_pack_key on int64 block indices."""
    b = (np.asarray(b, np.int64) + (1 << 20)) & ((1 << 21) - 1)
    return b[:, 0] | (b[:, 1] << 21) | (b[:, 2] << 42)


def aliases(b, idx):
    """(m, 3) blocks -> bool: outside the range, with the packed key of one of the real blocks idx."""
    if len(idx) == 0:
        return np.zeros(len(b), bool)
    return ~in_range(b) & np.isin(_key(b), _key(idx))


def _in_blocks(blocks, bs, rng, n_per, lo=0.02, hi=0.98):
    """n_per points inside each block (float64 position, then rounded to float32)."""
    blocks = np.asarray(blocks, np.int64).reshape(-1, 3)
    if len(blocks) == 0:
        return np.zeros((0, 3), F32)
    u = rng.uniform(lo, hi, (len(blocks), n_per, 3))
    return ((blocks[:, None, :] + u) * float(bs)).reshape(-1, 3).astype(F32)


def _ulps(p, axis):
    """p and its one-ulp neighbours along `axis`."""
    up = p.copy(); up[:, axis] = np.nextafter(p[:, axis], F32(np.inf))
    dn = p.copy(); dn[:, axis] = np.nextafter(p[:, axis], F32(-np.inf))
    return np.concatenate([p, up, dn])


def points(vs, vps, idx, d, w, seed=0, centres=CENTRES):
    """-> dict(xyz (m, 3) float32, kind (m,) str array, far (m,) bool)."""
    g = fx.Grid(vs, vps, idx, d, w)
    rng = np.random.default_rng(seed)
    bs = g.bs
    idx = np.asarray(idx, np.int64).reshape(-1, 3)
    parts = []

    def add(p, kind):
        p = np.asarray(p, F32).reshape(-1, 3)
        if len(p):
            parts.append((p, kind))

    if len(idx):
        c = g.centres()
        sel = rng.choice(len(c), min(centres, len(c)), replace=False)
        add(c[sel], "centre")
        m = min(centres // 4, len(c))
        corners = (c[rng.choice(len(c), m, replace=False)] - F32(0.5) * g.vs).astype(F32)
        add(corners, "corner")
        # block faces and voxel-centre planes, +-1 ulp
        base = _in_blocks(idx[rng.integers(0, len(idx), 3000)], bs, rng, 1)
        for axis in range(3):
            b = contain_block(base, g.bsi)
            face = base.copy()
            face[:, axis] = (b[:, axis].astype(F32) * bs).astype(F32)
            add(_ulps(face, axis), "face")
            v = rng.integers(0, vps, len(base))
            plane = base.copy()
            plane[:, axis] = ((b[:, axis].astype(F32) * bs).astype(F32)
                              + ((v.astype(F32) + F32(0.5)) * g.vs).astype(F32)).astype(F32)
            add(_ulps(plane, axis), "plane")
        # missing blocks next to existing ones (26 neighbours)
        have = set(map(tuple, idx.tolist()))
        miss = sorted({tuple(np.add(b, (i - 1, j - 1, k - 1)))
                       for b in idx.tolist() for i in range(3) for j in range(3) for k in range(3)} - have)
        miss = np.array(miss, np.int64).reshape(-1, 3)
        miss = miss[in_range(miss)]
        if len(miss) > 400:
            miss = miss[rng.choice(len(miss), 400, replace=False)]
        add(_in_blocks(miss, bs, rng, 8, 0.0, 1.0), "missing")
        # random points over the AABB grown by one block (per compressed group where it is huge)
        lo, hi = idx.min(0) - 1, idx.max(0) + 2
        if np.prod(hi - lo) <= 4096:
            add(((lo + rng.uniform(0, 1, (4000, 3)) * (hi - lo)) * float(bs)).astype(F32), "random")
        else:
            add(_in_blocks(idx, bs, rng, 4000 // len(idx) + 1, -1.0, 2.0), "random")
        # far: every real block shifted by +-2^21 on each axis
        far = []
        for axis in range(3):
            for s in (ALIAS, -ALIAS):
                sh = idx.copy(); sh[:, axis] += s
                far.append(sh)
        far = np.concatenate(far)
        add(_in_blocks(far, bs, rng, 16), "far_alias")
    # just beyond both ends of the range, on every axis
    ends = []
    for axis in range(3):
        for b in (fx.INDEX_MAX + 1, fx.INDEX_MAX + 2, fx.INDEX_MIN - 1, fx.INDEX_MIN - 2):
            q = np.zeros(3, np.int64); q[axis] = b
            ends.append(q)
    add(_in_blocks(np.array(ends), bs, rng, 16), "far_end")
    xyz = np.concatenate([p for p, _ in parts])
    kind = np.concatenate([np.full(len(p), k) for p, k in parts])
    cb = contain_block(xyz, g.bsi)
    is_far = np.char.startswith(kind.astype(str), "far")
    keep = ~is_far | ~in_range(cb)       # a far candidate that rounded into the range is dropped
    assert np.abs(cb).max(initial=0) < (1 << 31) // max(vps, 1)
    xyz, kind, is_far = xyz[keep], kind[keep], is_far[keep]
    return dict(xyz=xyz, kind=kind, far=is_far, grid=g, block=cb[keep])
