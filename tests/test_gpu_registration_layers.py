"""Registration lookups and TSDF allocation over the finishSubmap layer matrix and at block indices far
outside the accepted range, on the device.

1. Emit mode, every layer of finish_exact.matrix() as the reading submap, the points of
   tests/registration_layers.py (far points included): residuals and both Jacobians equal the oracle's
   bit for bit (Jacobian zeros up to their sign) at identity, at a translation by whole block sizes (exact-binary resolutions) and at two
   exact-trig random poses, one with a yaw near +-pi.
2. The fused evaluation, one graph per resolution with one constraint per layout, each layout read as
   is (block grid when its AABB has at most 4096 cells) and with one unobserved block far away (hash
   loop): cost, g, H and per-constraint costs within the exact-sum bound (tests/reduce_exact.py).  A read
   node moved by exactly -2^21 block sizes puts every reference point on a block whose 21-bit key is a
   real block's: both loops must report no correspondence.
3. TSDF integration with points whose truncation bands alias near blocks (2^21 block sizes away), lie
   beyond +-2^20 blocks, or sit at 2^32 block sizes (where an int cast of the block index wraps to 0):
   no block outside the range is allocated and no in-range voxel changes.  Mode 0 bit for bit against the
   oracle's in-range blocks; mode 1 by the serialisation check of tests/tsdf_exact.py.
"""
import itertools

import numpy as np
import pytest

import finish_exact as fx
import reduce_exact as RX
import registration_layers as RL
import tsdf_exact as tx
from finish_exact import MATRIX
from reduce_exact import GRID_MAX_CELLS, Problem, check_eval
from support import ctx  # noqa: F401

pytestmark = pytest.mark.gpu

_ids = itertools.count(3000)
PI_F = float(np.float32(np.pi))


def _reference_points(xyz, ref, read):
    """Reference-frame points that the pose pair maps to (near) the reading-frame points xyz."""
    if not np.any(ref) and not np.any(read):
        return np.asarray(xyz, np.float32)
    P = RX.pose_block(ref, read)
    return RX._inverse(P, xyz)


def _poses(res, bs, seed):
    """(label, ref pose, read pose): identity, whole block sizes (exact-binary), two exact-trig poses."""
    out = [("identity", np.zeros(4), np.zeros(4))]
    if res in fx.EXACT_RESOLUTIONS:
        out.append(("blocks", np.array([3 * bs, -2 * bs, bs, 0.0]), np.zeros(4)))
    rng = np.random.default_rng(seed)
    for k, base in enumerate(([[0.3, -0.2, 0.1, 0.5], [-0.1, 0.2, 0.05, PI_F - 0.02]],
                              [[0.05, 0.1, -0.1, -1.2], [0.2, -0.3, 0.0, 0.4]])):
        x = RX.exact_trig_poses(np.array(base), [(0, 1), (1, 0)], rng, sigma=(0.05, 0.05, 0.02, 0.01))
        out.append(("random%d" % k, x[0], x[1]))
    assert abs(out[-2][2][3]) > 3.0        # the yaw near +-pi
    return out


# --------------------------------------------------------------------------- 1. emit
@pytest.mark.parametrize("case", range(len(MATRIX)), ids=[m[0] for m in MATRIX])
def test_emit_matrix_bit_exact(ctx, oracle, case):
    from voxgraph_b200 import api
    vs, vps, idx, d, w = MATRIX[case][1]
    P = RL.points(vs, vps, idx, d, w, seed=case)
    xyz = P["xyz"]
    n = len(xyz)
    rng = np.random.default_rng(case)
    dist = rng.uniform(-0.1, 0.1, n).astype(np.float32)
    wt = np.ones(n, np.float32)
    L = oracle.Layer.from_blocks(vs, vps, idx, d, w)
    ref_sid, read_sid = next(_ids), next(_ids)
    one = fx.layer((vs, vps), "one", "plane")
    ctx.submap_upload(ref_sid, vs, vps, *one[2:])
    ctx.submap_upload(read_sid, vs, vps, idx, d, w)
    try:
        for label, ref, read in _poses((vs, vps), P["grid"].bs, case):
            x = _reference_points(xyz, ref, read)
            ctx.submap_upload_points(ref_sid, api.K_ISOSURFACE_POINTS, x, dist, wt)
            RX.check_pose_block(oracle, ref, read)
            ok_o, r_o, jr_o, je_o = oracle.reg_evaluate(L, x, dist, wt, ref, read)
            ok_g, r_g, jr_g, je_g = ctx.reg_eval_emit(ref_sid, read_sid, ref, read)
            assert ok_o and ok_g
            # residuals bit for bit; Jacobians bit for bit with the sign of zero folded (emit mode writes
            # J_read[0..2] = -J_ref[0..2], so a point without a correspondence reads -0.0 where the oracle
            # writes +0.0; a zero's sign never changes a sum)
            for what, a, b in (("residual", r_o, r_g), ("J_ref", jr_o + 0.0, jr_g + 0.0),
                               ("J_read", je_o + 0.0, je_g + 0.0)):
                bad = np.nonzero((a.view(np.uint64) != b.view(np.uint64)).reshape(n, -1).any(1))[0]
                assert bad.size == 0, (label, what, "first at", int(bad[0]), P["kind"][bad[0]],
                                       x[bad[0]].tolist(), bad.size)
            if label == "identity":
                # the far points: no correspondence (r = 0 at no_correspondence_cost 0, zero Jacobians)
                far = P["far"]
                assert not np.any(r_g[far]) and not np.any(jr_g[far]) and not np.any(je_g[far])
    finally:
        ctx.submap_free(ref_sid)
        ctx.submap_free(read_sid)


# --------------------------------------------------------------------------- 2. fused
def _fused_points(P, rng, cap=5000, far=True):
    """Every far point (far=True) and a seeded subset of the others."""
    near = np.nonzero(~P["far"])[0]
    if len(near) > cap:
        near = rng.choice(near, cap, replace=False)
    sel = np.sort(np.concatenate([near, np.nonzero(P["far"])[0] if far else np.zeros(0, np.int64)]))
    return P["xyz"][sel]


def _dummy(idx, d, w):
    """The layer plus one unobserved block far away in the range: its block AABB exceeds the block grid
    limit, so the reduce kernel takes the hash loop.  None when the layer already takes it (or has no
    blocks)."""
    if len(idx) == 0:
        return None
    lo, hi = idx.min(0).astype(np.int64), idx.max(0).astype(np.int64)
    if np.prod(hi - lo + 1) > GRID_MAX_CELLS:
        return None
    far = (hi + np.array([20, 20, 15]))[None].astype(np.int32)
    cells = int(np.prod(np.maximum(hi, far[0]) - lo + 1))
    assert cells > GRID_MAX_CELLS
    vpb = d.shape[1]
    return (np.concatenate([idx, far]), np.concatenate([d, np.zeros((1, vpb), np.float32)]),
            np.concatenate([w, np.zeros((1, vpb), np.float32)]))


def _layout_problem(ctx, oracle, res, point_type, nc, read_offset=None):
    """One constraint per layout of the resolution, read as is and through the hash loop.  Returns
    (Problem, {sid: pose}, n_hash) with reference nodes at 0 and read nodes at 0 or read_offset."""
    from voxgraph_b200 import api
    vs, vps = res
    pb = Problem(ctx, oracle)
    poses = {}
    rng = np.random.default_rng(int(vs * 1000) + vps)
    n_hash = 0
    for k, lay in enumerate(fx.LAYOUTS):
        fld = "crafted" if res in fx.EXACT_RESOLUTIONS and lay in ("box", "straddle", "negative", "shuffled") \
            else ["tilted", "sphere", "plane", "noise"][k % 4]
        _, _, idx, d, w = fx.layer(res, lay, fld, seed=k)
        P = RL.points(vs, vps, idx, d, w, seed=k, centres=3000)
        # moved by 2^21 blocks, the far points would land back on real blocks: left out there
        xyz = _fused_points(P, rng, far=read_offset is None)
        n = len(xyz)
        if n == 0:
            continue            # the zero-block layout has only far points

        dist = rng.uniform(-0.1, 0.1, n).astype(np.float32)
        wt = rng.uniform(0.5, 2.0, n).astype(np.float32)
        ref_sid = 400 + 10 * k
        one = fx.layer(res, "one", "plane")
        half = n // 2
        # a constraint is evaluated both ways: every submap carries the layout's points of both types
        pts = dict(iso=(xyz, dist, wt), vox=(xyz[half:], dist[half:], np.ones(n - half, np.float32)))
        pb.submap(ref_sid, vs, vps, *one[2:], **pts)
        pb.node(ref_sid, np.zeros(4)); poses[ref_sid] = np.zeros(4)
        reads = [(ref_sid + 1, (idx, d, w))]
        dm = _dummy(idx, d, w)
        if dm is not None:
            reads.append((ref_sid + 2, dm))
        for sid, lyr in reads:
            cells = int(np.prod(lyr[0].max(0).astype(np.int64) - lyr[0].min(0) + 1)) if len(lyr[0]) else 0
            n_hash += cells > GRID_MAX_CELLS or cells == 0
            pb.submap(sid, vs, vps, *lyr, **pts)
            pose = np.zeros(4) if read_offset is None else np.asarray(read_offset, np.float64)
            pb.node(sid, pose); poses[sid] = pose
            pb.constrain(ref_sid, sid, registration_point_type=point_type, no_correspondence_cost=nc)
    return pb, poses, n_hash


@pytest.mark.parametrize("res", fx.RESOLUTIONS, ids=["%g/%d" % r for r in fx.RESOLUTIONS])
def test_fused_layouts_both_loops(ctx, oracle, res):
    from voxgraph_b200 import api
    for point_type, nc in ((api.K_ISOSURFACE_POINTS, 0.0), (api.K_VOXELS, 0.3)):
        pb, poses, n_hash = _layout_problem(ctx, oracle, res, point_type, nc)
        assert n_hash >= 8
        for label, fixed in (("identity", poses), ("random", {400: np.zeros(4)})):
            pb.build(seed=7, fixed=fixed)
            ex = pb.exact()
            check_eval(pb, ex, "%g/%d %s type=%d nc=%g" % (res[0], res[1], label, point_type, nc))


@pytest.mark.parametrize("nc", [0.0, 0.3])
def test_fused_far_translation_aliases_nothing(ctx, oracle, nc):
    """Read nodes at exactly -2^21 block sizes on x (0.125 m / 16, yaw 0): every reference point lands
    2^21 blocks from where it was, on blocks whose 21-bit keys are the reading layer's own.  The oracle
    finds no correspondence anywhere; the fused sums of both loops must agree (exactly 0 at cost 0)."""
    from voxgraph_b200 import api
    res = (0.125, 16)
    bs = 2.0
    shift = -(2.0 ** 21) * bs
    pb, poses, n_hash = _layout_problem(ctx, oracle, res, api.K_ISOSURFACE_POINTS, nc,
                                        read_offset=[shift, 0.0, 0.0, 0.0])
    assert n_hash >= 8
    pb.build(seed=3, fixed=poses)
    ex = pb.exact()
    for k, ((a, b), cfg) in enumerate(zip(pb.pg.registration_blocks, pb.pg._reg_cfgs)):
        xyz, d, w = pb.sub[a]["pts"][cfg.registration_point_type]
        ok, r, _, _ = oracle.reg_evaluate(pb.sub[b]["layer"], xyz, d, w, pb.x[pb.col[a]], pb.x[pb.col[b]],
                                          no_correspondence_cost=float("nan"), jacobians=False)
        assert ok and np.isnan(r).all(), "block %d: a correspondence 2^21 blocks away" % k
    check_eval(pb, ex, "far translation nc=%g" % nc)
    if nc == 0.0:
        ok, cost, g, H = pb.pg.evaluate()
        assert ok and cost == 0.0 and not np.any(g) and not np.any(H)


# --------------------------------------------------------------------------- 3. TSDF far field
TVS, TVPS, TBS = 0.125, 16, 2.0
FAR_CFG = dict(voxel_carving_enabled=0, max_ray_length_m=1.0e11)
T_ID = np.array([1, 0, 0, 0, 0, 0, 0], np.float32)


def _far_scan():
    """(near, far, p32): near points 2.5-6 m around the sensor; far = the near points moved by 2^21
    block sizes on x (their bands alias the near blocks) and points beyond +-2^20 blocks on every axis;
    p32 = one point at 2^32 block sizes on x."""
    rng = np.random.default_rng(11)
    n = 400
    a = rng.uniform(-np.pi, np.pi, n)
    r = rng.uniform(2.5, 6.0, n)
    near = np.stack([r * np.cos(a), r * np.sin(a), rng.uniform(-1.0, 1.0, n)], -1).astype(np.float32)
    alias = (near.astype(np.float64) + [2.0 ** 21 * TBS, 0, 0]).astype(np.float32)
    beyond = []
    for axis in range(3):
        for s in (1, -1):
            for k in (3, 37, 1000):
                p = rng.uniform(-3, 3, 3)
                p[axis] = s * ((1 << 20) + k) * TBS + rng.uniform(0.2, 1.8)
                beyond.append(p)
    far = np.concatenate([alias, np.array(beyond, np.float32)])
    p32 = np.array([[2.0 ** 32 * TBS, 0.0, 0.0]], np.float32)
    return near, far, p32


def _in_range_blocks(idx):
    return RL.in_range(np.asarray(idx, np.int64).reshape(-1, 3))


def _oracle_in_range(layer):
    oi, od, ow = layer.export()
    k = _in_range_blocks(oi)
    return oi[k], od[k], ow[k]


def _trace_in_range(g, s, u):
    k = RL.in_range(np.floor_divide(np.asarray(g, np.int64), TVPS))
    return g[k], s[k], u[k]


def test_tsdf_far_field_simple(ctx, oracle):
    near, far, p32 = _far_scan()
    pts = np.concatenate([near, far])
    layer = oracle.Layer(TVS, TVPS)
    st, g, s, u = oracle.tsdf_integrate_trace(layer, oracle.tsdf_config(**FAR_CFG), T_ID, pts)
    assert (~RL.in_range(np.floor_divide(g, TVPS))).sum() > 1000      # the far bands were traced
    oi, od, ow = _oracle_in_range(layer)
    gi_, _, _ = _trace_in_range(g, s, u)
    # the aliasing is real: far voxels whose block key field is a near block's
    fb = np.floor_divide(g, TVPS)
    assert RL.aliases(fb[~RL.in_range(fb)], oi).sum() > 100
    sids = []
    try:
        got = {}
        for name, scan in (("near", near), ("far", pts), ("far+p32", np.concatenate([pts, p32]))):
            sid = next(_ids); sids.append(sid)
            ctx.submap_create(sid, TVS, TVPS, len(oi))
            sg = ctx.tsdf_integrate(sid, T_ID, scan, ctx.tsdf_config(**FAR_CFG))
            got[name] = (sg, ctx.submap_download(sid), sid)
        sg, dl, _ = got["far"]
        assert (sg.rays_valid, sg.rays_cast) == (st.rays_valid, st.rays_cast)
        assert sg.voxel_updates == len(gi_) < st.voxel_updates
        assert sg.blocks_allocated == len(oi)
        tx.assert_layers_bit_equal((oi, od, ow), dl)
        # device only: the 2^32 point (block 2^32 wraps to 0 in an int) changes nothing
        sg32, dl32, sid32 = got["far+p32"]
        assert (sg32.rays_valid, sg32.rays_cast, sg32.voxel_updates, sg32.blocks_allocated) == \
            (sg.rays_valid + 1, sg.rays_cast + 1, sg.voxel_updates, sg.blocks_allocated)
        tx.assert_layers_bit_equal(got["near"][1], dl32)
        tx.assert_layers_bit_equal(dl, dl32)
        assert _in_range_blocks(dl32[0]).all()
        sid = next(_ids); sids.append(sid)
        ctx.submap_upload(sid, TVS, TVPS, *dl32)
        tx.assert_layers_bit_equal(dl32, ctx.submap_download(sid))
    finally:
        for sid in sids:
            ctx.submap_free(sid)


def test_tsdf_far_field_fast(ctx, oracle):
    near, far, p32 = _far_scan()
    pts = np.concatenate([near, far])
    ocfg = oracle.tsdf_config(**{**FAR_CFG, **tx.FAST_ALL})
    layer = oracle.Layer(TVS, TVPS)
    st, g, s, u = oracle.tsdf_integrate_trace(layer, ocfg, T_ID, pts)
    assert st.rays_cast == st.rays_valid
    oi, od, ow = _oracle_in_range(layer)
    gi_, si_, ui_ = _trace_in_range(g, s, u)
    sid = next(_ids)
    ctx.submap_create(sid, TVS, TVPS, len(oi))
    try:
        sg = ctx.tsdf_integrate(sid, T_ID, np.concatenate([pts, p32]), ctx.tsdf_config(**{**FAR_CFG, **tx.FAST_ALL}))
        assert (sg.rays_valid, sg.rays_cast, sg.voxel_updates, sg.blocks_allocated) == \
            (st.rays_valid + 1, st.rays_cast + 1, len(gi_), len(oi))
        gi, gd, gw = ctx.submap_download(sid)
    finally:
        ctx.submap_free(sid)
    assert _in_range_blocks(gi).all()
    assert np.array_equal(np.unique(gi, axis=0), np.unique(oi, axis=0))
    tx.check_fast(tx.layer_voxels(gi, gd, gw, TVPS), tx.voxel_keys(gi_), si_, ui_,
                  ocfg.default_truncation_distance, ocfg.max_weight, tx.layer_voxels(oi, od, ow, TVPS))
