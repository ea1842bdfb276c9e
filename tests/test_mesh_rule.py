"""The submap mesh rule (tests/mesh_exact.py, restated by vgx_mesh_build) on the CPU: the face-walk
triangulation over all 256 cube configurations, closed and consistently oriented surfaces on analytic
fields, vertex accuracy, open boundaries only where the valid region ends, the shared-edge property
over the finishSubmap layer matrix, and the palette."""
import numpy as np
import pytest

import finish_exact as fx
import mesh_exact as me
from finish_exact import MATRIX
from voxgraph_b200 import synth


# --------------------------------------------------------------------------- the rule over 256 configurations
def _trilinear_grad(vals, p, h=1e-4):
    """Central-difference gradient of the trilinear interpolant of the 8 corner values at p."""
    def f(q):
        r = 0.0
        for k, o in enumerate(me.CUBE_OFF):
            w = np.prod([q[a] if o[a] else 1 - q[a] for a in range(3)])
            r += w * vals[k]
        return r
    return np.array([(f(p + h * e) - f(p - h * e)) / (2 * h) for e in np.eye(3)])


def test_rule_over_all_configurations():
    """Every crossing edge lies on exactly one loop with its two face neighbours next to it, a loop
    has 3 to 7 edges, a cube at most 4 loops and 5 triangles, and every loop faces the positive side by
    the numerical gradient of the corner field (summed over its edge midpoints)."""
    counts = []
    for cfg in range(256):
        neg = [(cfg >> k) & 1 for k in range(8)]
        cross = {e for e in range(12) if neg[me.EDGES[e][0]] != neg[me.EDGES[e][1]]}
        loops = me.loops(cfg)
        flat = [e for lp in loops for e in lp]
        assert sorted(flat) == sorted(cross), cfg
        assert len(loops) <= 4 and all(3 <= len(lp) <= 7 for lp in loops)
        assert [lp[0] for lp in loops] == sorted(lp[0] for lp in loops)
        assert all(lp[0] == min(lp) for lp in loops)
        vals = np.where(np.array(neg) == 1, -1.0, 1.0)
        for lp in loops:
            for i in range(len(lp)):      # consecutive edges share a cube face
                a, b = lp[i], lp[(i + 1) % len(lp)]
                assert any(a in f[1] and b in f[1] for f in me.FACES), (cfg, lp)
            mid = [(me.CUBE_OFF[me.EDGES[e][0]] + me.CUBE_OFF[me.EDGES[e][1]]) / 2.0 for e in lp]
            n = sum(np.cross(mid[i], mid[(i + 1) % len(lp)]) for i in range(len(lp)))
            g = sum(_trilinear_grad(vals, m) for m in mid)
            assert n @ g > 0, (cfg, lp)
        tri = me.triangles(cfg)
        assert len(tri) == sum(len(lp) - 2 for lp in loops) <= 5
        counts.append(len(tri))
    assert max(counts) == 5 and counts[0] == counts[255] == 0
    # complementary configurations have the same crossing edges
    for cfg in range(256):
        assert sorted(e for lp in me.loops(cfg) for e in lp) == sorted(e for lp in me.loops(255 - cfg) for e in lp)


# --------------------------------------------------------------------------- topology helpers
def _edge_use(tri):
    """{(a, b) undirected: [directed uses]}."""
    use = {}
    for t in tri:
        for k in range(3):
            a, b = int(t[k]), int(t[(k + 1) % 3])
            use.setdefault((min(a, b), max(a, b)), []).append((a, b))
    return use


def _check_shared_edges(tri):
    """Every undirected edge is used once or twice, and twice only in opposite directions."""
    use = _edge_use(tri)
    for k, u in use.items():
        assert len(u) <= 2, (k, u)
        if len(u) == 2:
            assert u[0] == (u[1][1], u[1][0]), (k, u)
    return use


def _closed(xyz, tri):
    use = _check_shared_edges(tri)
    assert all(len(u) == 2 for u in use.values())
    V = len(np.unique(tri))
    assert V == len(xyz)
    return V - len(use) + len(tri)


def _normals(xyz, tri):
    p = xyz.astype(np.float64)
    return np.cross(p[tri[:, 1]] - p[tri[:, 0]], p[tri[:, 2]] - p[tri[:, 0]])


def _sphere(vs, vps, centre, r, blocks):
    fn = lambda p: np.linalg.norm(p - np.asarray(centre), axis=-1) - r
    idx, d, w = synth.field_layer_blocks(fn, vs, vps, blocks, weight=3.0)
    return fx.Grid(vs, vps, idx, d, w)


@pytest.mark.parametrize("vs,vps", [(0.1, 8), (0.05, 16), (0.2, 4)])
def test_sphere_is_a_closed_outward_manifold(vs, vps):
    bs = vs * vps
    r = 1.3 * bs
    c = np.array([1.0, 1.0, 1.0]) * bs + 0.013
    g = _sphere(vs, vps, c, r, ((-1, 2), (-1, 2), (-1, 2)))
    xyz, tri = me.mesh(g, 2.0)
    assert len(tri) > 100
    assert _closed(xyz, tri) == 2
    n = _normals(xyz, tri)
    cen = xyz.astype(np.float64)[tri].mean(1)
    assert np.all(np.einsum("ij,ij->i", n, cen - c) > 0)
    # vertices on the surface within the interpolation bound of a distance field: |f(p)| <= s^2 / (8 (r - s))
    err = np.abs(np.linalg.norm(xyz.astype(np.float64) - c, axis=1) - r)
    assert err.max() <= vs * vs / (8 * (r - vs)) + 1e-5 * r
    # area within 5 % of 4 pi r^2 (the chords of a convex surface cut it slightly short)
    area = 0.5 * np.linalg.norm(n, axis=1).sum()
    assert abs(area / (4 * np.pi * r * r) - 1) < 0.05


def test_box_and_two_spheres_are_closed():
    """A box (flat faces, sharp edges) is one closed surface; two disjoint spheres have Euler
    characteristic 4."""
    vs, vps = 0.1, 8
    lo, hi = np.array([0.23, 0.31, 0.27]), np.array([1.37, 1.12, 1.29])
    fn = lambda p: synth.box_sdf(p, (lo + hi) / 2, (hi - lo) / 2)
    idx, d, w = synth.field_layer_blocks(fn, vs, vps, ((-1, 2), (-1, 2), (-1, 2)), weight=3.0)
    xyz, tri = me.mesh(fx.Grid(vs, vps, idx, d, w), 2.0)
    assert _closed(xyz, tri) == 2
    c = (lo + hi) / 2
    assert np.all(np.einsum("ij,ij->i", _normals(xyz, tri), xyz.astype(np.float64)[tri].mean(1) - c) > 0)
    fn2 = lambda p: np.minimum(np.linalg.norm(p - [0.5, 0.5, 0.5], axis=-1) - 0.35,
                               np.linalg.norm(p - [1.6, 1.5, 1.4], axis=-1) - 0.3)
    idx, d, w = synth.field_layer_blocks(fn2, vs, vps, ((-1, 3), (-1, 3), (-1, 3)), weight=3.0)
    xyz, tri = me.mesh(fx.Grid(vs, vps, idx, d, w), 2.0)
    assert _closed(xyz, tri) == 4


def test_open_layout_boundary_only_where_the_valid_region_ends():
    """A tilted plane through one block: the mesh is open, and each boundary edge lies on a face of the
    meshed region (cube origins span voxel centres 0 .. vps - 2 per axis)."""
    vs, vps = 0.1, 8
    vs32 = np.float32(vs)
    idx, d, w = synth.plane_layer_blocks([0.3, -0.2, 0.93], 0.35, vs, vps, ((0, 0), (0, 0), (0, 0)), weight=3.0)
    xyz, tri = me.mesh(fx.Grid(vs, vps, idx, d, w), 2.0)
    use = _check_shared_edges(tri)
    boundary = [k for k, u in use.items() if len(u) == 1]
    assert boundary
    lo = np.float32(0.5) * vs32
    hi = (np.float32(vps - 1) + np.float32(0.5)) * vs32
    for a, b in boundary:
        pa, pb = xyz[a], xyz[b]
        on = [(pa[ax] == v and pb[ax] == v) for ax in range(3) for v in (lo, hi)]
        assert any(on), (pa, pb)
    # with one voxel slab invalid the surface splits there and gains boundary on both sides
    w2 = w.copy().reshape(1, vps, vps, vps)
    w2[:, :, :, 4] = 1.0                     # x = 4 below min_weight
    xyz2, tri2 = me.mesh(fx.Grid(vs, vps, idx, d, w2.reshape(1, -1)), 2.0)
    assert 0 < len(tri2) < len(tri)
    use2 = _check_shared_edges(tri2)
    assert sum(len(u) == 1 for u in use2.values()) > len(boundary)


@pytest.mark.parametrize("case", range(0, len(MATRIX), 3), ids=[m[0] for m in MATRIX][::3])
def test_shared_edges_over_the_layer_matrix(case):
    """On every layer of the finishSubmap matrix (noise, crafted exact values, blocks joined through an
    edge or a corner, both ends of the index range) the mesh is watertight: the uses of an edge in its
    two directions differ by at most one (one only on the boundary); every vertex is used."""
    vs, vps, idx, d, w = MATRIX[case][1]
    g = fx.Grid(vs, vps, idx, d, w)
    xyz, tri = me.mesh(g, 1.0)
    for k, u in _edge_use(tri).items():
        fwd = sum(1 for x in u if x == k)
        # a fan diagonal across an ambiguous face can be drawn by both cubes of the face: two sheets
        # then touch along it (4 uses), still balanced
        assert fwd <= 2 and len(u) - fwd <= 2 and abs(2 * fwd - len(u)) <= 1, (k, u)
    assert len(np.unique(tri)) == len(xyz)
    # at most one vertex per crossing edge of a meshed cube (finishSubmap's candidates count every cube's
    # copy of a shared edge)
    cand, _, _ = fx.candidates(g, 1.0)
    assert len(xyz) <= len(cand)
    assert (len(xyz) == 0) == (len(cand) == 0)


def test_separated_offsets_and_transform():
    gs = [_sphere(0.1, 8, [0.4, 0.4, 0.4], 0.25, ((0, 0), (0, 0), (0, 0))),
          _sphere(0.2, 4, [0.4, 0.4, 0.4], 0.3, ((0, 0), (0, 0), (0, 0)))]
    T = np.array([[1, 0, 0, 0, 0, 0, 0], [np.cos(0.15), 0, 0, np.sin(0.15), 1.0, -2.0, 0.5]], np.float32)
    xyz, tri, vo, to = me.separated(gs, T, 2.0)
    x0, t0 = me.mesh(gs[0], 2.0)
    x1, t1 = me.mesh(gs[1], 2.0)
    assert vo.tolist() == [0, len(x0), len(x0) + len(x1)] and to.tolist() == [0, len(t0), len(t0) + len(t1)]
    assert np.array_equal(tri[len(t0):], (t1 + len(x0)).astype(np.uint32))
    R = np.array([[np.cos(0.3), -np.sin(0.3), 0], [np.sin(0.3), np.cos(0.3), 0], [0, 0, 1]])
    assert np.allclose(xyz[len(x0):], x1.astype(np.float64) @ R.T + [1.0, -2.0, 0.5], atol=1e-5)
    assert np.array_equal(xyz[:len(x0)], x0)


def test_palette():
    """The default submap colour, rainbowColorMap((id mod 20) / 20): id 0 is red, the 20 colours of a cycle
    differ, and the largest id wraps like any other."""
    colour = lambda i: me.rainbow((i % 20) / 20.0)   # noqa: E731
    assert colour(0) == [255, 0, 0, 255]
    assert colour(20) == colour(0) and colour(2 ** 32 - 1) == colour(15)
    assert len({tuple(colour(i)) for i in range(20)}) == 20
