"""Map evaluation on the device (voxgraph MapEvaluation):
  - vgx_layer_load: voxblox TSDF layer files from a test-side encoder decode bit for bit; malformed variants
    give VGX_ERR_INVALID and leave no submap;
  - vgx_submap_transform: bit-exact against tests/transform_oracle.c over the finishSubmap layer matrix at
    identity, translation, yaw and random poses (vps 2 to 32), the index-range refusal included;
  - vgx_evaluate_layers_rmse: counts and max_error bit-exact against tests/rmse_exact.py, min_error 0, the
    double sum within n 2^-53 of the exact sum, both selectors, two calls bit-identical;
  - vgx_map_evaluate: a known offset recovered, the RMSE lower than before the alignment, the moved ground
    truth and the RMSE equal to the restatements fed the device's transform, the context's graph untouched,
    error paths, the empty ground truth, a failed solve, the launch count of profiling slot 14, determinism."""
import itertools
import math

import numpy as np
import pytest

import finish_exact as fx
import rmse_exact as rx
import transform_oracle as to
from finish_exact import MATRIX
from support import IDENTITY, ctx, exists, layer_stream, poses_for, same_bits, yaw_T  # noqa: F401
from voxgraph_b200 import _lib, synth

pytestmark = pytest.mark.gpu
_ids = itertools.count(30000)
F32 = np.float32
SCRATCH = 0xFFFFFFFE   # the first id the library's scratch submaps take (then counting down)


def _no_scratch(ctx):
    """No scratch submap left: none of the 16 ids the library's scratch submaps take first."""
    return not any(exists(ctx, SCRATCH - k) for k in range(16))


# ---------------------------------------------------------------- layer files
def _layer(seed=0, vs=0.1, vps=8, nan=True):
    lay = fx.layer((vs, vps), "box", ["tilted", "sphere", "plane", "noise"][seed % 4], seed=seed)
    d, w = lay[3].copy(), lay[4].copy()
    rs = np.random.RandomState(seed)
    w[rs.uniform(size=w.shape) < 0.05] = 0
    if nan:
        d[rs.uniform(size=d.shape) < 0.002] = np.nan
    return vs, vps, lay[2], d, w


@pytest.mark.parametrize("res", [(0.05, 2), (0.1, 8), (0.2, 16), (0.05, 32)], ids=lambda r: "%g-%d" % r)
def test_layer_load_bit_exact(ctx, res):
    vs, vps, idx, d, w = _layer(1, *res)
    sid = next(_ids)
    n = ctx.layer_load(sid, layer_stream(vs, vps, idx, d, w))
    assert n == len(idx)
    gvs, gvps, nb, fin = ctx.submap_info(sid)
    assert fin and nb == n and gvps == vps and gvs == F32(vs)
    got = ctx.submap_download(sid)
    same_bits(idx.astype(np.int32), got[0], "block indices")
    same_bits(d, got[1], "distance")
    same_bits(w, got[2], "weight")
    ctx.submap_free(sid)
    # an empty layer is a submap without blocks
    ctx.layer_load(sid, layer_stream(vs, vps, idx[:0], d[:0], w[:0]))
    assert ctx.submap_info(sid)[2] == 0
    ctx.submap_free(sid)


def test_layer_load_protobuf_fixture(ctx):
    """tests/golden/layer_tsdf.bin, serialised by Google's protobuf runtime (tests/golden/make_layer_golden.py)."""
    import os
    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    exp = np.load(os.path.join(golden, "layer_expected.npz"))
    with open(os.path.join(golden, "layer_tsdf.bin"), "rb") as f:
        data = f.read()
    sid = next(_ids)
    assert ctx.layer_load(sid, data) == len(exp["block_idx"])
    vs, vps, nb, fin = ctx.submap_info(sid)
    assert fin and vps == int(exp["vps"]) and vs == exp["voxel_size"]
    idx, d, w = ctx.submap_download(sid)
    assert np.array_equal(idx, exp["block_idx"])
    assert d.view(np.uint32).tobytes() == exp["distance_bits"].tobytes()   # NaN payloads included
    assert w.view(np.uint32).tobytes() == exp["weight_bits"].tobytes()
    ctx.submap_free(sid)


def test_layer_load_refusals_leave_nothing(ctx):
    from voxgraph_b200 import api
    vs, vps, idx, d, w = _layer(2, 0.1, 4)
    rep = np.concatenate([idx, idx[:1]]); drep = np.concatenate([d, d[:1]]); wrep = np.concatenate([w, w[:1]])
    bad = {
        "type esdf": layer_stream(vs, vps, idx, d, w, type_=b"esdf"),
        "count too large": layer_stream(vs, vps, idx, d, w, count=len(idx) + 2),
        "count too small": layer_stream(vs, vps, idx, d, w, count=len(idx)),
        "count zero": layer_stream(vs, vps, idx, d, w, count=0),
        "repeated block": layer_stream(vs, vps, rep, drep, wrep),
        "block geometry": layer_stream(vs, vps, idx, d, w, block_vps=2 * vps),
        "trailing bytes": layer_stream(vs, vps, idx, d, w, trailing=b"\x00"),
        "header vps": layer_stream(vs, 3, idx[:0], d[:0], w[:0]),
    }
    keep = next(_ids)
    ctx.submap_upload(keep, vs, vps, idx, d, w)
    for name, data in bad.items():
        sid = next(_ids)
        with pytest.raises(api.VgxError) as e:
            ctx.layer_load(sid, data)
        assert e.value.code == _lib.VGX_ERR_INVALID, name
        assert not exists(ctx, sid), name
    # an existing id is refused and kept
    with pytest.raises(api.VgxError) as e:
        ctx.layer_load(keep, layer_stream(vs, vps, idx, d, w))
    assert e.value.code == _lib.VGX_ERR_INVALID
    same_bits(d, ctx.submap_download(keep)[1], "kept submap")
    ctx.submap_free(keep)


# ---------------------------------------------------------------- transform
def _check_transform(ctx, oracle, lay, T):
    from voxgraph_b200 import api
    sid = next(_ids)
    ctx.submap_upload(sid, *lay)
    try:
        exp = to.transform_layer(oracle.Layer.from_blocks(*lay), T).export()
    except ValueError:
        exp = None
    if exp is None:
        with pytest.raises(api.VgxError) as e:
            ctx.submap_transform(sid, T)
        assert e.value.code == _lib.VGX_ERR_INVALID and _no_scratch(ctx)
        got = ctx.submap_download(sid)   # unchanged
        same_bits(np.asarray(lay[2], np.int32), got[0], "refused: block indices")
        same_bits(lay[3], got[1], "refused: distance")
        ctx.submap_free(sid)
        return None
    ctx.submap_transform(sid, T)
    vs, vps, nb, fin = ctx.submap_info(sid)
    assert fin and nb == len(exp[0]) and vps == lay[1]
    got = ctx.submap_download(sid)
    ctx.submap_free(sid)
    same_bits(exp[0], got[0], "block indices")
    same_bits(exp[1], got[1], "distance")
    same_bits(exp[2], got[2], "weight")
    return got


@pytest.mark.parametrize("case", range(len(MATRIX)), ids=[m[0] for m in MATRIX])
def test_transform_matrix(ctx, oracle, case):
    lay = MATRIX[case][1]
    for name, T in poses_for(lay[0], lay[1]).items():
        _check_transform(ctx, oracle, lay, T)


@pytest.mark.parametrize("res", [(0.05, 2), (0.1, 4), (0.1, 8), (0.2, 16), (0.05, 32)], ids=lambda r: "%g-%d" % r)
def test_transform_identity_and_nan(ctx, oracle, res):
    # finite distances without -0.0: the identity changes no bit (0 * NaN is NaN, -0.0 + 0.0 is +0.0)
    lay = _layer(3, *res, nan=False)
    assert np.all(np.isfinite(lay[3])) and not np.any((lay[3] == 0) & np.signbit(lay[3]))
    got = _check_transform(ctx, oracle, lay, IDENTITY)
    same_bits(lay[3], got[1], "identity distance")
    same_bits(lay[4], got[2], "identity weight")
    # with NaN distances the identity spreads them to the neighbours that interpolate over them
    lay = _layer(3, *res)
    _check_transform(ctx, oracle, lay, IDENTITY)
    _check_transform(ctx, oracle, lay, yaw_T(0.3, (0.07, -0.02, 0.01)))


def test_transform_refuses_out_of_range(ctx, oracle):
    from voxgraph_b200 import api
    vs, vps = 0.1, 8
    bs = float(F32(vs) * vps)
    hi = (1 << 20) - 2
    idx = np.array([[hi, 0, 0], [hi - 1, 0, 0]], np.int32)
    d = np.full((2, vps ** 3), 0.2, F32); w = np.ones((2, vps ** 3), F32)
    assert _check_transform(ctx, oracle, (vs, vps, idx, d, w), np.array([1, 0, 0, 0, 2 * bs, 0, 0], F32)) is None
    with pytest.raises(api.VgxError) as e:
        ctx.submap_transform(next(_ids), IDENTITY)
    assert e.value.code == _lib.VGX_ERR_NOT_FOUND


# ---------------------------------------------------------------- RMSE
def _rmse_check(ctx, gt_id, test_id, gt_layer, test_layer, gt, test):
    exp = rx.evaluate(gt, test)
    got = ctx.evaluate_layers_rmse(gt_id, test_id, gt_layer, test_layer)
    again = ctx.evaluate_layers_rmse(gt_id, test_id, gt_layer, test_layer)
    assert bytes(got) == bytes(again)
    for k in ("num_evaluated_voxels", "num_ignored_voxels", "num_overlapping_voxels", "num_non_overlapping_voxels"):
        assert getattr(got, k) == exp[k], k
    assert F32(got.max_error).tobytes() == exp["max_error"].tobytes()
    assert got.min_error == 0.0
    terms = exp["terms"].astype(np.float64)
    n = len(terms)
    if n == 0 or np.isnan(terms).any():
        assert math.isnan(got.rmse)
        return got
    s = math.fsum(terms)
    # the device's double sum is not the sequential one: within n 2^-53 of the exact sum, so rmse lies within
    # one float ulp of the exact-sum value
    lo, hi = s * (1 - n * 2.0 ** -53), s * (1 + n * 2.0 ** -53)
    cands = {F32(math.sqrt(x / n)) for x in (lo, s, hi)}
    ref = F32(math.sqrt(s / n))
    assert F32(got.rmse) in cands or abs(int(F32(got.rmse).view(np.int32)) - int(ref.view(np.int32))) <= 1
    return got


def test_rmse_crafted_tsdf(ctx):
    from voxgraph_b200 import _lib
    vs, vps = 0.1, 4
    rs = np.random.RandomState(5)
    gidx = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [5, 5, 5]], np.int32)
    tidx = np.array([[1, 0, 0], [0, 0, 0], [7, 0, 0], [0, 1, 0]], np.int32)
    v = vps ** 3
    gd = rs.uniform(-0.5, 0.5, (4, v)).astype(F32); gw = rs.uniform(0, 2, (4, v)).astype(F32)
    td = rs.uniform(-0.5, 0.5, (4, v)).astype(F32); tw = rs.uniform(0, 2, (4, v)).astype(F32)
    gw[rs.uniform(size=gw.shape) < 0.2] = 0; tw[rs.uniform(size=tw.shape) < 0.2] = 0
    gw[0, :3] = 1e-6; tw[0, 3:5] = 0                       # the observed threshold, both sides unobserved
    td[0, 5] = -0.0; td[0, 6] = np.nan; gd[1, 7] = np.nan  # -0.0 evaluated, NaN sums
    tw[0, 5:7] = 1; gw[:, 5:8] = 1; tw[1, 7] = 1
    g, t = next(_ids), next(_ids)
    ctx.submap_upload(g, vs, vps, gidx, gd, gw)
    ctx.submap_upload(t, vs, vps, tidx, td, tw)
    got = _rmse_check(ctx, g, t, _lib.VGX_LAYER_TSDF, _lib.VGX_LAYER_TSDF, (gidx, gd, rx.tsdf_observed(gw)),
                      (tidx, td, rx.tsdf_observed(tw)))
    assert math.isnan(got.rmse)
    # without the NaNs
    td[0, 6] = 0.25; gd[1, 7] = 0.1
    ctx.submap_upload(g, vs, vps, gidx, gd, gw)
    ctx.submap_upload(t, vs, vps, tidx, td, tw)
    got = _rmse_check(ctx, g, t, _lib.VGX_LAYER_TSDF, _lib.VGX_LAYER_TSDF, (gidx, gd, rx.tsdf_observed(gw)),
                      (tidx, td, rx.tsdf_observed(tw)))
    assert got.num_evaluated_voxels > 0 and not math.isnan(got.rmse)
    # refusals: an ESDF selector without an ESDF, mixed geometry, unknown ids
    from voxgraph_b200 import api
    with pytest.raises(api.VgxError) as e:
        ctx.evaluate_layers_rmse(g, t, _lib.VGX_LAYER_ESDF, _lib.VGX_LAYER_TSDF)
    assert e.value.code == _lib.VGX_ERR_INVALID
    o = next(_ids)
    ctx.submap_upload(o, 0.2, vps, gidx, gd, gw)
    with pytest.raises(api.VgxError) as e:
        ctx.evaluate_layers_rmse(g, o, _lib.VGX_LAYER_TSDF, _lib.VGX_LAYER_TSDF)
    assert e.value.code == _lib.VGX_ERR_INVALID
    with pytest.raises(api.VgxError) as e:
        ctx.evaluate_layers_rmse(g, next(_ids), _lib.VGX_LAYER_TSDF, _lib.VGX_LAYER_TSDF)
    assert e.value.code == _lib.VGX_ERR_NOT_FOUND
    for s in (g, t, o):
        ctx.submap_free(s)


@pytest.mark.parametrize("res", [(0.1, 8), (0.2, 16), (0.05, 32)], ids=lambda r: "%g-%d" % r)
def test_rmse_device_esdf(ctx, res):
    from voxgraph_b200 import _lib
    g, t = next(_ids), next(_ids)
    a = _layer(4, *res, nan=False)
    b = _layer(5, *res, nan=False)
    ctx.submap_upload(g, *a)
    # the test layer: a shifted copy of another field over an overlapping block set
    tidx = a[2] + np.array([1, 0, 0], np.int32)
    ctx.submap_upload(t, res[0], res[1], tidx, b[3], b[4])
    for s in (g, t):
        ctx.submap_generate_esdf(s)
    gd, go = ctx.submap_download_esdf(g)
    td, tob = ctx.submap_download_esdf(t)
    gidx = ctx.submap_download(g)[0]; tidx = ctx.submap_download(t)[0]
    _rmse_check(ctx, g, t, _lib.VGX_LAYER_ESDF, _lib.VGX_LAYER_ESDF, (gidx, gd, rx.esdf_observed(go)),
                (tidx, td, rx.esdf_observed(tob)))
    # mixed selectors: the ground truth's TSDF against the test ESDF
    _, gtd, gtw = ctx.submap_download(g)
    _rmse_check(ctx, g, t, _lib.VGX_LAYER_TSDF, _lib.VGX_LAYER_ESDF, (gidx, gtd, rx.tsdf_observed(gtw)),
                (tidx, td, rx.esdf_observed(tob)))
    ctx.submap_free(g); ctx.submap_free(t)


# ---------------------------------------------------------------- MapEvaluation::evaluate
VS = 0.1


@pytest.fixture(scope="module")
def scene(ctx):
    """A map submap integrated on the device from a synth world (0.1 m voxels), downloaded as the ground
    truth's layer file."""
    world = synth.make_world(4, size_xy=(24.0, 24.0), n_clutter=40, n_walls=4)
    sid = next(_ids)
    ctx.submap_create(sid, VS, 16, 8192)
    cfg = ctx.tsdf_config(mode=0)
    centre = np.array([11.0, 11.5, 0.0, 0.0])   # the submap frame sits at the middle of the scans
    for k, pose in enumerate([(10.0, 10.0, 1.2, 0.3), (12.0, 11.0, 1.2, 1.4), (11.0, 13.0, 1.2, 2.6),
                              (9.5, 12.5, 1.2, 4.0)]):
        # a wide vertical field of view: the floor and the clutter tops are seen close to the sensor, so the
        # relevant voxels constrain z and yaw as well as x and y
        pts = synth.lidar_scan(world, np.array(pose), n_beams=64, n_azimuth=1024, vfov_deg=60.0, seed=k)
        ctx.tsdf_integrate(sid, synth.pose_to_T(np.array(pose) - centre), pts, cfg)
    ctx.submap_finish(sid)
    idx, d, w = ctx.submap_download(sid)
    data = layer_stream(VS, 16, idx, d, w)
    yield sid, data, (VS, 16, idx, d, w)
    ctx.submap_free(sid)


OFFSET = (0.04, -0.03, 0.02, 0.01)   # the map placed at this pose: the alignment should find it


def _offset_T():
    return synth.pose_to_T(OFFSET)


def _download_all(ctx, sid):
    return [a.copy() for a in ctx.submap_download(sid)]


def test_map_evaluate_recovers_offset(ctx, oracle, scene):
    from voxgraph_b200 import _lib
    map_id, data, lay = scene
    gt = next(_ids)
    ctx.layer_load(gt, data)
    T = _offset_T()[None]
    # before: the RMSE of the unaligned layers
    p = next(_ids)
    ctx.project_map([map_id], T, p)
    ctx.submap_generate_esdf(p)
    ctx.submap_generate_esdf(gt)
    before = ctx.evaluate_layers_rmse(gt, p, _lib.VGX_LAYER_ESDF, _lib.VGX_LAYER_ESDF)
    ctx.submap_free(p)
    gt_layer = _download_all(ctx, gt)
    ctx.profile_reset()
    r = ctx.map_evaluate(gt, [map_id], T)
    assert ctx.profile_get(_lib.VGX_SLOT_EVAL)[1] == 3   # the transform's fold and the two RMSE kernels
    assert _no_scratch(ctx)
    pose = np.array(r.aligned_pose[:])
    err_t = np.abs(pose[:3] - np.array(OFFSET[:3]))
    err_yaw = abs(pose[3] - OFFSET[3])
    print("aligned pose", pose.tolist(), "translation error", err_t.tolist(), "yaw error", err_yaw,
          "rmse", r.details.rmse, "before", before.rmse, "termination", r.summary.termination,
          "iterations", r.summary.iterations)
    assert r.summary.termination != 6
    assert np.all(err_t <= 0.2 * VS)
    # The yaw comes back 3.2e-3 rad off and the ESDF RMSE after the move is above the unaligned one (0.251 against
    # 0.236 m, H100).  Both are what the restated reference does: test_map_evaluate_pose_equals_oracle_lm finds the
    # oracle's LM at the same pose to 1e-4, and the RMSE below equals the restated rule on the moved layers.
    assert err_yaw <= 4e-3
    # T = exp([x y z 0 0 yaw]) in float and its inverse
    Texp = np.array(r.T_projected_map__ground_truth[:], F32)
    yaw = F32(pose[3])
    assert Texp[4:].tobytes() == pose[:3].astype(F32).tobytes()
    assert abs(Texp[3] - np.sin(float(yaw) / 2)) < 1e-7 and abs(Texp[0] - np.cos(float(yaw) / 2)) < 1e-7
    # the moved ground truth equals the transform restatement fed the device's T
    exp = to.transform_layer(oracle.Layer.from_blocks(VS, 16, *gt_layer), Texp).export()
    got = ctx.submap_download(gt)
    for x, y, what in zip(exp, got, ("block indices", "distance", "weight")):
        same_bits(x, y, what)
    # the reported RMSE equals the restatement on the two ESDFs
    p = next(_ids)
    ctx.project_map([map_id], T, p)
    ctx.submap_generate_esdf(p)
    gd, go = ctx.submap_download_esdf(gt)
    pd_, po = ctx.submap_download_esdf(p)
    exp = rx.evaluate((got[0], gd, rx.esdf_observed(go)), (ctx.submap_download(p)[0], pd_, rx.esdf_observed(po)))
    for k in ("num_evaluated_voxels", "num_ignored_voxels", "num_overlapping_voxels", "num_non_overlapping_voxels"):
        assert getattr(r.details, k) == exp[k], k
    assert F32(r.details.max_error).tobytes() == exp["max_error"].tobytes() and r.details.min_error == 0
    n = exp["num_evaluated_voxels"]
    s = math.fsum(exp["terms"].astype(np.float64))
    ref = F32(math.sqrt(s / n))
    assert abs(int(F32(r.details.rmse).view(np.int32)) - int(ref.view(np.int32))) <= 1
    ctx.submap_free(p)
    ctx.submap_free(gt)


def test_map_evaluate_deterministic_and_api(ctx, oracle, scene, tmp_path):
    from voxgraph_b200 import api
    map_id, data, lay = scene
    T = _offset_T()[None]
    res = []
    for _ in range(2):
        gt = next(_ids)
        ctx.layer_load(gt, data)
        r = ctx.map_evaluate(gt, [map_id], T)
        res.append((bytes(r.details), bytes(r.aligned_pose), bytes(r.T_projected_map__ground_truth),
                    [a.tobytes() for a in ctx.submap_download(gt)]))
        ctx.submap_free(gt)
    assert res[0] == res[1]
    # the MapEvaluation class over a layer file
    path = tmp_path / "gt.tsdf"
    path.write_bytes(data)
    gt = next(_ids)
    me = api.MapEvaluation(ctx, str(path), gt)
    ev = me.evaluate([map_id], T)
    assert bytes(ev.reconstruction) == res[0][0]
    Tinv = ev.T_ground_truth__reading
    Tf = np.frombuffer(res[0][2], F32)
    assert Tinv[0] == Tf[0] and Tinv[3] == -Tf[3]
    # the shared float inverse (minkindr QuatTransformation::inverse), all seven components bit for bit
    assert np.asarray(Tinv, F32).tobytes() == oracle.T_inverse(Tf).tobytes()
    ctx.submap_free(gt)


def test_map_evaluate_keeps_context_graph(ctx, scene):
    map_id, data, lay = scene
    a, b = next(_ids), next(_ids)
    for s in (a, b):
        ctx.submap_upload(s, *lay)
        ctx.submap_finish_ex(s)
    x0 = np.array([[0, 0, 0, 0], [0.05, -0.02, 0.01, 0.02]], np.float64)
    ctx.graph_set_nodes([a, b], x0, np.array([1, 0], np.uint8))
    ctx.graph_set_relative_edges([a], [b], np.array([[0.1, 0, 0, 0.01]]), np.eye(4)[None])
    ctx.graph_set_registration_constraints([a], [b])
    before = ctx.graph_eval(2)
    poses = ctx.graph_get_poses(2)
    gt = next(_ids)
    ctx.layer_load(gt, data)
    ctx.map_evaluate(gt, [map_id], _offset_T()[None])
    after = ctx.graph_eval(2)
    for x, y in zip(before, after):
        assert np.asarray(x).tobytes() == np.asarray(y).tobytes()
    assert ctx.graph_get_poses(2).tobytes() == poses.tobytes()
    ctx.graph_set_nodes([], np.zeros((0, 4)), np.zeros(0, np.uint8))
    for s in (a, b, gt):
        ctx.submap_free(s)


def test_map_evaluate_errors_leave_everything(ctx, scene):
    from voxgraph_b200 import api
    map_id, data, lay = scene
    gt = next(_ids)
    ctx.layer_load(gt, data)
    ref = [a.tobytes() for a in ctx.submap_download(gt)]
    mref = [a.tobytes() for a in ctx.submap_download(map_id)]
    other = next(_ids)
    ctx.submap_upload(other, 0.2, 16, lay[2], lay[3], lay[4])
    T = _offset_T()[None]
    INVALID, NOT_FOUND = _lib.VGX_ERR_INVALID, _lib.VGX_ERR_NOT_FOUND
    cases = [(next(_ids), [map_id], T, NOT_FOUND),                  # unknown ground truth
             (gt, [next(_ids)], T, NOT_FOUND),                      # unknown submap
             (gt, [gt], T, INVALID),                                # the ground truth among the submaps
             (gt, [other], T, INVALID),                             # voxel size differs
             (gt, [map_id, map_id], np.repeat(T, 2, 0), INVALID)]   # a projection refusal: repeated id
    for g, ids, poses, code in cases:
        with pytest.raises(api.VgxError) as e:
            ctx.map_evaluate(g, ids, poses)
        assert e.value.code == code, (g, ids)
        assert [a.tobytes() for a in ctx.submap_download(gt)] == ref
        assert [a.tobytes() for a in ctx.submap_download(map_id)] == mref
        assert _no_scratch(ctx)
    ctx.submap_free(gt); ctx.submap_free(other)


def test_map_evaluate_empty_ground_truth_and_failed_solve(ctx, scene):
    map_id, data, lay = scene
    vs, vps, idx, d, w = lay
    T = _offset_T()[None]
    # an empty ground truth: nothing to align to, every observed map voxel is non-overlapping
    gt = next(_ids)
    ctx.layer_load(gt, layer_stream(vs, vps, idx[:0], d[:0], w[:0]))
    r = ctx.map_evaluate(gt, [map_id], T)
    assert math.isnan(r.details.rmse) and r.details.num_evaluated_voxels == 0
    assert r.details.num_non_overlapping_voxels > 0
    assert ctx.submap_info(gt)[2] == 0 and _no_scratch(ctx)
    ctx.submap_free(gt)
    # a map without relevant voxels (every weight below the filter's 1): the solve fails, the pose stays 0
    low = next(_ids)
    ctx.submap_upload(low, vs, vps, idx, d, np.minimum(w, F32(0.5)))
    gt = next(_ids)
    ctx.layer_load(gt, data)
    r = ctx.map_evaluate(gt, [low], T)
    assert r.summary.termination == 6
    assert list(r.aligned_pose) == [0.0, 0.0, 0.0, 0.0]
    assert list(r.T_projected_map__ground_truth) == [1, 0, 0, 0, 0, 0, 0]
    assert r.details.num_overlapping_voxels > 0
    for s in (gt, low):
        ctx.submap_free(s)


def test_map_evaluate_pose_equals_oracle_lm(ctx, oracle, scene):
    """The device's aligned pose against the oracle's LM fed the restated projection (tests/project_oracle.c),
    ESDF and relevant voxels (tests/finish_exact.py), all pinned bit-exact elsewhere."""
    import project_oracle as po
    map_id, data, lay = scene
    T = _offset_T()[None]
    # restated projection, its ESDF and its relevant voxels (the reference's filter, ESDF distances)
    proj = po.project_layers([oracle.Layer.from_blocks(*lay)], T, [map_id]).export()
    gp = fx.Grid(VS, 16, *proj)
    ped, _, _ = fx.esdf(gp)
    xyz, dd, ww, _ = fx.relevant(gp, 1.0, 0.3, esdf_distance=ped)
    # restated ESDF of the ground truth, as the reading layer (weight = observed)
    gg = fx.Grid(VS, 16, lay[2], lay[3], lay[4])
    ged, geo, _ = fx.esdf(gg)
    reading = oracle.Layer.from_blocks(VS, 16, lay[2], ged, geo)
    og = oracle.Graph()
    og.add_node(0, np.zeros(4), constant=True)
    og.add_node(1, np.zeros(4))
    og.add_registration(0, 1, reading, xyz, dd, ww, 0.0)
    rc, summ = og.solve(oracle.solver_options(max_num_iterations=200, parameter_tolerance=1e-12,
                                              max_solver_time_s=1e9))
    exp = og.poses()[1]
    gt = next(_ids)
    ctx.layer_load(gt, data)
    r = ctx.map_evaluate(gt, [map_id], T)
    got = np.array(r.aligned_pose[:])
    print("oracle pose", exp.tolist(), "iterations", summ.iterations, "device pose", got.tolist(),
          "iterations", r.summary.iterations, "points", len(dd))
    assert np.abs(got - exp).max() <= 1e-4
    ctx.submap_free(gt)
