"""The fused registration reduction (reg_reduce_kernel -> reg_csum_kernel -> assembly) against an exact
sum of the oracle's per-point terms.

At exact-trig poses (reduce_exact.exact_trig_poses) the device pose block equals the oracle's bit for
bit, so every per-point residual and Jacobian the kernel forms is the oracle's, and the fused cost, g,
H and per-constraint costs may differ from the exact sums only by double summation rounding:
|fused - exact| <= 2^-50 (n + 64) sum|t| per entry.  One dropped point, one point moved by an ulp or a
residual rounded to float breaks that bound, where the 1e-7 tolerance of the oracle tests does not.
"""
import numpy as np
import pytest

import reduce_exact as RX
from reduce_exact import GRID_MAX_CELLS, Problem, check_eval
from support import ctx, oracle_layer  # noqa: F401
from voxgraph_b200 import synth

pytestmark = pytest.mark.gpu

RAGGED = (1, 31, 32, 33, 95, 2047, 2048, 2049, 3000, 5000)
PI_F = float(np.float32(np.pi))


# --------------------------------------------------------------------------- scenes
def _small(ctx, oracle, small_scene):
    pb = Problem(ctx, oracle)
    for i, s in enumerate(small_scene.submaps):
        pb.synth_submap(s, sid=i)
        pb.node(i, small_scene.poses_init[i], constant=(i == 0))
    for (i, j) in small_scene.pairs:
        pb.constrain(i, j)
    return pb


def _with_dummy_block(s, dims):
    """s's bricks plus one unobserved block at the far corner of a block AABB of `dims` cells."""
    lo = s.block_idx.min(0)
    assert np.all(s.block_idx.max(0) - lo + 1 <= dims)
    idx = np.concatenate([s.block_idx, (lo + np.asarray(dims) - 1)[None].astype(np.int32)])
    d = np.concatenate([s.distance, np.zeros((1, s.distance.shape[1]), np.float32)])
    w = np.concatenate([s.weight, np.zeros((1, s.weight.shape[1]), np.float32)])
    cells = int(np.prod(idx.max(0) - idx.min(0) + 1))
    return idx, d, w, cells


def _tile_scene(ctx, oracle, small_scene):
    """Every small_scene pair both ways, ten K_VOXELS constraints of ragged point counts, and a
    hash-path constraint in the middle of the list: 30 + 2 + 10 residual blocks, ~78k residuals."""
    from voxgraph_b200 import api
    sc = small_scene
    pb = _small(ctx, oracle, sc)
    pairs = list(sc.pairs)
    cons_iso = pb.cons
    pb.cons = []
    half = len(cons_iso) // 2
    pb.cons += cons_iso[:half]
    # hash path: a copy of submap 1 whose block AABB is too large for the block grid
    idx, d, w, cells = _with_dummy_block(sc.submaps[1], (21, 21, 16))
    assert cells > GRID_MAX_CELLS
    s1 = sc.submaps[1]
    pb.submap(40, s1.voxel_size, s1.vps, idx, d, w, iso=(s1.points_xyz, s1.points_distance, s1.points_weight))
    pb.node(40, sc.poses_init[1])
    pb.constrain(0, 40)
    pb.cons += cons_iso[half:]
    # ragged counts: copies of the reference submap of a pair, points repeated cyclically, each read
    # against its own copy of the reading submap whose block grid has other dimensions (a CTA that
    # moves on to the next constraint must restage the grid)
    for k, n in enumerate(RAGGED):
        i, j = pairs[k % len(pairs)]
        s = sc.submaps[i]
        sel = np.arange(n) % len(s.points_weight)
        sid = 20 + k
        pb.submap(sid, s.voxel_size, s.vps, s.block_idx[:1], s.distance[:1], s.weight[:1],
                  vox=(s.points_xyz[sel], s.points_distance[sel], s.points_weight[sel]))
        pb.node(sid, sc.poses_init[i])
        sj = sc.submaps[j]
        idx, d, w, cells = _with_dummy_block(sj, (7 + k, 6, 3))
        assert cells <= GRID_MAX_CELLS
        pb.submap(50 + k, sj.voxel_size, sj.vps, idx, d, w)
        pb.node(50 + k, sc.poses_init[j])
        pb.constrain(sid, 50 + k, registration_point_type=api.K_VOXELS)
    return pb


# --------------------------------------------------------------------------- 1. baseline
def test_baseline_small_scene(ctx, oracle, small_scene):
    """All pairs both ways; yaws at 0, +-pi (float) and in vgx_yaw_quat's series branch."""
    sc = small_scene
    pb = _small(ctx, oracle, sc)
    fixed = {0: sc.poses_init[0]}
    for k, yaw in ((2, PI_F), (3, -PI_F), (5, 5e-5)):
        fixed[k] = np.array([*sc.poses_init[k][:3], yaw])
    pb.build(seed=1, fixed=fixed)
    assert pb.x[0, 3] == 0.0 and abs(pb.x[5, 3]) < RX.SERIES_THETA
    ex = pb.exact()
    check_eval(pb, ex, "baseline")


# --------------------------------------------------------------------------- 2. tile shapes
@pytest.fixture(scope="module")
def tile_problem(ctx, oracle, small_scene):
    pb = _tile_scene(ctx, oracle, small_scene)
    pb.build(seed=2, fixed={0: small_scene.poses_init[0]})
    ex = pb.exact()
    n_units = sum((n + 31) // 32 for n in (len(pb.sub[a]["pts"][c.registration_point_type][2])
                                           for (a, _), c in zip(pb.pg.registration_blocks, pb.pg._reg_cfgs)))
    assert len(pb.pg.registration_blocks) >= 20 and n_units * 32 > 132 * 7 * 32
    return pb, ex


@pytest.mark.parametrize("tile_units", ["1", "2", "3", "5", "17", "64", "128", "129", "256"])
def test_tile_shapes(ctx, tile_problem, monkeypatch, tile_units):
    """VGX_REG_HW_TILE_UNITS is read at every table build: small tiles below the ring depth,
    tiles above 128 units (no culling)."""
    from voxgraph_b200 import api
    pb, ex = tile_problem
    monkeypatch.setenv("VGX_REG_HW_TILE_UNITS", tile_units)
    pg0 = pb.pg
    pg = api.PoseGraph(ctx)
    for s in sorted(pb.nodes):
        pg.addSubmapNode(api.SubmapNodeConfig(s, pb.x[pb.col[s]], set_constant=pb.nodes[s][1]))
    for c in pb.cons:
        pg.addRegistrationConstraint(c)
    assert pg.registration_blocks == pg0.registration_blocks
    pb.pg = pg
    try:
        check_eval(pb, ex, "tile_units=%s" % tile_units, costs=(tile_units in ("1", "2", "129")))
    finally:
        pb.pg = pg0


# --------------------------------------------------------------------------- 6. reproducibility
def test_bits_stable_across_lpt_refreshes(ctx, tile_problem, monkeypatch):
    """The longest-first tile order is refreshed at the start of the 2nd evaluation call on new
    tables and then whenever 32 calls have run since the last refresh; cost-only calls
    (getVisualizationEdgeResiduals) count as calls.  Here the calls are 32 evaluations, one cost-only
    call, and 8 more evaluations: the refreshes come before calls 2 and 34, and the one before call 34
    orders the tiles by the costs the cost-only kernel measured.  Every evaluation is bit-identical
    to the first, and the cost-only sums are within the exact-sum bound."""
    from voxgraph_b200 import api
    monkeypatch.delenv("VGX_REG_HW_TILE_UNITS", raising=False)
    pb, ex = tile_problem
    pg = api.PoseGraph(ctx)
    for s in sorted(pb.nodes):
        pg.addSubmapNode(api.SubmapNodeConfig(s, pb.x[pb.col[s]], set_constant=pb.nodes[s][1]))
    for c in pb.cons:
        pg.addRegistrationConstraint(c)
    first = None
    for call in range(1, 42):
        if call == 33:
            RX.check_costs_bound(ex, pg.getVisualizationEdgeResiduals(), "cost-only before a re-order")
            continue
        ok, cost, g, H = pg.evaluate()
        assert ok
        if first is None:
            first = (cost, g, H)
            pb_pg, pb.pg = pb.pg, pg
            try:
                RX.check_bound(ex, cost, g, H, label="evaluation 1")
            finally:
                pb.pg = pb_pg
        else:
            assert cost == first[0] and g.tobytes() == first[1].tobytes() and H.tobytes() == first[2].tobytes(), \
                "call %d differs from evaluation 1" % call


# --------------------------------------------------------------------------- 3. culling edges
def cull_problem(ctx, oracle):
    """The pairs of reduce_exact.cull_problem_scenes (the scene test_host_cull_margin checks on the
    host) as submaps 60..63 with K_VOXELS constraints (one block each)."""
    from voxgraph_b200 import api
    pb = Problem(ctx, oracle)
    bsi = oracle.Layer(RX.CULL_VS, RX.CULL_VPS).block_size_inv
    x, scenes = RX.cull_problem_scenes(bsi)
    for (ref, read, P, sc) in scenes:
        mh, mh0, hits = RX.cull_report(P, sc)
        assert mh.any() and (~mh).any(), "units on both sides of the cull decision"
        assert (mh & ~mh0).any(), "units live only because of the margin"
        assert not (hits & ~mh).any()
        pb.submap(60 + read, RX.CULL_VS, RX.CULL_VPS, sc["block_idx"], sc["distance"], sc["weight"])
        pb.submap(60 + ref, RX.CULL_VS, RX.CULL_VPS, sc["block_idx"][:1], sc["distance"][:1], sc["weight"][:1],
                  vox=(sc["xyz"], sc["d"], sc["w"]))
        pb.node(60 + ref, x[ref]); pb.node(60 + read, x[read], constant=(read == 1))
        pb.constrain(60 + ref, 60 + read, registration_point_type=api.K_VOXELS)
    pb.build(seed=0, fixed={60 + k: x[k] for k in range(4)})
    return pb, scenes


def test_culling_edges(ctx, oracle):
    pb, _ = cull_problem(ctx, oracle)
    ex = pb.exact()
    check_eval(pb, ex, "culling edges")


# --------------------------------------------------------------------------- 4. options
def _grid_pair(pb, s, sid, dims):
    idx, d, w, cells = _with_dummy_block(s, dims)
    pb.submap(sid, s.voxel_size, s.vps, idx, d, w, iso=(s.points_xyz, s.points_distance, s.points_weight))
    return cells


def test_constraint_options(ctx, oracle, small_scene):
    """no_correspondence_cost, ESDF distances, K_VOXELS points, sampling 0.05 / 0.5, four voxel
    sizes, non-uniform weights, two constraints on one pair, a constant node, and reading submaps
    with exactly 4096 (block grid) and 4100 (hash) block-AABB cells, in one graph."""
    from voxgraph_b200 import api
    sc = small_scene
    pb = Problem(ctx, oracle)
    for i in range(4):
        s = sc.submaps[i]
        vx, vd, vw = oracle.find_relevant_voxels(oracle_layer(oracle, s), 1.0, 0.3)
        pb.submap(100 + i, s.voxel_size, s.vps, s.block_idx, s.distance, s.weight,
                  iso=(s.points_xyz, s.points_distance, s.points_weight), vox=(vx, vd, vw), esdf=True)
        pb.node(100 + i, sc.poses_init[i], constant=(i == 0))
        assert len(np.unique(s.points_weight)) > 1    # factor != 1
    pb.constrain(100, 101, no_correspondence_cost=0.3)
    pb.constrain(100, 101)                                   # same pair, other options
    pb.constrain(101, 102, use_esdf_distance=True)
    pb.constrain(102, 103, registration_point_type=api.K_VOXELS)
    pb.constrain(100, 102, sampling_ratio=0.05)
    pb.constrain(101, 103, sampling_ratio=0.5)
    # exactly 4096 block-AABB cells (block grid) and 4100 (hash)
    assert _grid_pair(pb, sc.submaps[2], 110, (16, 16, 16)) == GRID_MAX_CELLS
    assert _grid_pair(pb, sc.submaps[2], 111, (10, 10, 41)) == GRID_MAX_CELLS + 4
    pb.node(110, sc.poses_init[2]); pb.node(111, sc.poses_init[2])
    pb.constrain(100, 110)
    pb.constrain(100, 111)
    # other voxel sizes / voxels per side
    world = synth.make_world(7, size_xy=(16.0, 14.0), n_clutter=20, n_walls=2)
    for k, (vs, vps) in enumerate(((0.05, 8), (0.1, 16), (0.2, 16), (0.4, 32))):
        r = 3.0 if vs < 0.2 else 6.0
        pa, pr = np.array([8.0, 7.0, 1.0, 0.2]), np.array([8.6, 7.3, 1.0, -0.4])
        a = synth.make_submap(world, 0, pa, vs, vps, r, n_points=1500)
        b = synth.make_submap(world, 0, pr, vs, vps, r, n_points=1500)
        pb.synth_submap(a, sid=200 + 2 * k); pb.synth_submap(b, sid=201 + 2 * k)
        pb.node(200 + 2 * k, pa + np.array([0.03, -0.02, 0.01, 0.01])); pb.node(201 + 2 * k, pr)
        pb.constrain(200 + 2 * k, 201 + 2 * k)
    pb.build(seed=4, fixed={100: sc.poses_init[0]})
    ex = pb.exact()
    check_eval(pb, ex, "constraint options")
