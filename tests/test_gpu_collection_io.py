"""Submap collection files on the device: the committed fixtures (serialised by Google's protobuf
runtime) decode to the expected bricks bit for bit, the writer reproduces the unpacked fixture byte for
byte, malformed voxel payloads fail with nothing of the stream left behind, and a map built on the
device (mapper, Fast integration) or a config-2-sized collection survives save -> load bit for bit
through finishSubmap, the ESDF, overlap detection and the pose-graph evaluation."""
import os
import sys

import numpy as np
import pytest

import collection_stream as cs
from voxgraph_b200 import _lib

pytestmark = pytest.mark.gpu
INVALID = _lib.VGX_ERR_INVALID


@pytest.fixture(scope="module")
def exp():
    return cs.expected()


def _expected_blocks(exp):
    """{id: {block index tuple: (distance bits, weight bits)}}"""
    out, first = {}, 0
    for k, sid in enumerate(exp["ids"]):
        nb = int(exp["num_blocks"][k])
        out[int(sid)] = {tuple(int(v) for v in exp["block_idx"][first + b]):
                         (exp["distance_bits"][first + b], exp["weight_bits"][first + b]) for b in range(nb)}
        first += nb
    return out


def _check_loaded(ctx, exp):
    want = _expected_blocks(exp)
    for sid, blocks in want.items():
        vs, vps, n, finished = ctx.submap_info(sid)
        assert finished and vs == exp["voxel_size"] and vps == exp["vps"] and n == len(blocks)
        idx, d, w = ctx.submap_download(sid)
        got = {tuple(int(v) for v in idx[b]): (d[b].view(np.uint32), w[b].view(np.uint32)) for b in range(n)}
        assert set(got) == set(blocks)
        for key, (db, wb) in blocks.items():
            assert np.array_equal(got[key][0], db) and np.array_equal(got[key][1], wb), (sid, key)


def _absent(ctx, ids):
    from voxgraph_b200 import api
    for sid in ids:
        with pytest.raises(api.VgxError):
            ctx.submap_info(int(sid))


@pytest.mark.parametrize("case", cs.CASES)
def test_load_fixture(exp, case):
    from voxgraph_b200 import api
    ctx = api.Context(0)
    assert ctx.collection_load(cs.read(case)) == len(exp["ids"])
    _check_loaded(ctx, exp)
    # every one of them saves as the unpacked, colour-free stream
    entries = api.Context.collection_scan(cs.read(case))
    ids = [e["id"] for e in entries]
    T = np.array([e["T_M_S"] for e in entries])
    assert ctx.collection_save(ids, T) == cs.read("unpacked")
    ctx.close()


def test_load_empty_collection():
    from voxgraph_b200 import api
    ctx = api.Context(0)
    assert ctx.collection_load(cs.read("empty")) == 0
    data = ctx.collection_save([], np.zeros((0, 7), np.float32))
    assert api.Context.collection_scan(data) == []
    ctx.close()


def test_save_is_byte_identical_to_protobuf(exp, tmp_path):
    from voxgraph_b200 import api
    ctx = api.Context(0)
    ctx.collection_load(cs.read("unpacked"))
    # ids in any order: the file lists them in increasing id order
    perm = [2, 0, 1]
    ids = exp["ids"][perm]
    path = str(tmp_path / "c.bin")
    n = api.save_submap_collection(ctx, path, ids, exp["poses"][perm])
    data = open(path, "rb").read()
    assert n == len(data) and data == cs.read("unpacked")
    # the size query and the capacity rule
    import ctypes as C
    L = ctx._L
    size = C.c_uint64(0)
    ids32 = np.ascontiguousarray(exp["ids"], np.uint32); T = np.ascontiguousarray(exp["poses"], np.float32)
    args = (ctx._h, 3, ids32.ctypes.data_as(C.POINTER(C.c_uint32)), T.ctypes.data_as(C.POINTER(C.c_float)))
    small = C.create_string_buffer(len(data) - 1)
    assert L.vgx_collection_save(*args, small, len(data) - 1, C.byref(size)) == _lib.VGX_ERR_CAPACITY
    assert size.value == len(data)
    try:
        sys.path.insert(0, cs.GOLDEN)
        import make_collection_golden as g
        P = g._classes()
    except ImportError:
        P = None
    finally:
        sys.path.remove(cs.GOLDEN)
    if P is not None:   # parse the saved bytes with Google's runtime as well
        msgs = cs.messages(data)
        head = P["SubmapCollectionProto"].FromString(msgs[0])
        assert head.num_submaps == 3 and head.voxels_per_side == exp["vps"]
        sm = P["SubmapProto"].FromString(msgs[1])
        assert sm.id == 0 and sm.num_blocks == exp["num_blocks"][0]
        blk = P["BlockProto"].FromString(msgs[2])
        words = np.array(blk.voxel_data, np.uint32).reshape(-1, 3)
        assert np.array_equal(words[:, 0], exp["distance_bits"][0]) and not words[:, 2].any()
    ctx.close()


def _corrupt_last_block(fn):
    def voxel_data(k, b, words):
        return fn(words) if (k, b) == (2, 2) else cs.unpacked_voxel_data(words)
    return voxel_data


def _packed(words, extra=0):
    body = b"".join(cs.varint(int(w)) for w in words)
    return b"\x3a" + cs.varint(len(body) + extra) + body


def _overlong(words):   # the block's first value as a 6-byte varint
    return b"\x38\x80\x80\x80\x80\x80\x00" + cs.unpacked_voxel_data(words[1:])


PAYLOAD_ERRORS = {
    "tag": lambda w: cs.unpacked_voxel_data(w[:10]) + b"\x40" + cs.unpacked_voxel_data(w[10:])[1:],
    "overlong_varint": _overlong,
    "one_value_too_many": lambda w: cs.unpacked_voxel_data(w) + b"\x38\x00",
    "one_value_too_few": lambda w: cs.unpacked_voxel_data(w[:-1]),
    "packed_length_overruns": lambda w: _packed(w, extra=1),
    "packed_length_short": lambda w: _packed(w, extra=-1),
}


@pytest.mark.parametrize("kind", sorted(PAYLOAD_ERRORS) + ["repeated_index", "index_out_of_range", "packed_ok"])
def test_payload_errors_leave_nothing(exp, kind):
    from voxgraph_b200 import api
    bidx = exp["block_idx"].copy()
    if kind in PAYLOAD_ERRORS:
        data = cs.build(exp, voxel_data=_corrupt_last_block(PAYLOAD_ERRORS[kind]))
    elif kind == "packed_ok":
        data = cs.build(exp, voxel_data=lambda k, b, w: _packed(w))
    else:
        if kind == "repeated_index":
            bidx[-1] = bidx[-2]
        else:
            bidx[-1] = [(1 << 20), 0, 0]
        data = cs.build(exp, block_idx=bidx)
    if kind != "packed_length_overruns":   # the host framing reads that length too
        assert len(api.Context.collection_scan(data)) == 3
    ctx = api.Context(0)
    ctx.submap_upload(99, 0.1, 8, [[1, 2, 3]], np.full(512, 0.25, np.float32), np.ones(512, np.float32))
    if kind == "packed_ok":
        ctx.collection_load(data)
        _check_loaded(ctx, exp)
    else:
        with pytest.raises(api.VgxError) as e:
            ctx.collection_load(data)
        assert e.value.code == INVALID
        _absent(ctx, exp["ids"])
    idx, d, w = ctx.submap_download(99)
    assert idx.tolist() == [[1, 2, 3]] and (d == 0.25).all() and (w == 1).all()
    ctx.close()


def test_existing_id_blocks_the_load(exp):
    from voxgraph_b200 import api
    ctx = api.Context(0)
    ctx.submap_upload(7, 0.1, 8, [[4, 5, 6]], np.full(512, -0.5, np.float32), np.full(512, 2.0, np.float32))
    with pytest.raises(api.VgxError) as e:
        ctx.collection_load(cs.read("unpacked"))
    assert e.value.code == INVALID
    _absent(ctx, [0, 2 ** 32 - 1])
    vs, vps, n, _ = ctx.submap_info(7)
    idx, d, w = ctx.submap_download(7)
    assert (vs, vps, n) == (np.float32(0.1), 8, 1) and idx.tolist() == [[4, 5, 6]]
    assert (d == -0.5).all() and (w == 2.0).all()
    ctx.close()


def _finished_state(ctx, ids, poses_T, xyzyaw):
    """finish_ex + ESDF of every submap, then everything registration reads."""
    filt = ctx.registration_filter()
    out = {}
    for sid in ids:
        ctx.submap_finish_ex(sid, filt)
        ctx.submap_generate_esdf(sid)
        pts = [ctx.submap_download_points(sid, t) for t in (0, 1)]
        out[sid] = (ctx.submap_download(sid), pts, ctx.submap_download_esdf(sid), ctx.submap_surface_obb(sid))
    pairs = ctx.find_overlapping_pairs(ids, poses_T)
    ctx.graph_set_nodes(ids, xyzyaw, [1] + [0] * (len(ids) - 1))
    ctx.graph_set_relative_edges([], [], np.zeros((0, 4)), np.zeros((0, 16)))   # registration only
    if pairs:
        a = [p[0] for p in pairs] + [p[1] for p in pairs]
        b = [p[1] for p in pairs] + [p[0] for p in pairs]
        ctx.graph_set_registration_constraints(a, b)
    ok, cost, g, H = ctx.graph_eval(len(ids))
    return out, pairs, (ok, cost, g, H)


def _identical(a, b):
    if isinstance(a, (tuple, list)):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            _identical(x, y)
    elif isinstance(a, np.ndarray):
        assert a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()
    else:
        assert a == b or (a != a and b != b)


def test_mapper_round_trip(tmp_path):
    from voxgraph_b200 import api, mapper as vm, synth
    ctx = api.Context(0)
    world = synth.make_world(7, size_xy=(40.0, 30.0), n_clutter=60, n_walls=5)
    n = 10
    s_arc = np.arange(n) * 0.6
    gt = np.stack([8.0 + s_arc, 12.0 + 0.5 * np.sin(s_arc / 3.0), np.full(n, 1.2), 0.05 * s_arc], -1)
    cfg = vm.MapperConfig(voxel_size=0.2, submap_creation_interval=4 / 10.0, capacity_blocks=4096,
                          tsdf=dict(max_ray_length_m=12.0))
    m = vm.VoxgraphMapper(ctx, cfg)
    for k in range(n):
        m.pointcloudCallback(k / 10.0, gt[k], synth.lidar_scan(world, gt[k], n_beams=24, n_azimuth=360,
                                                               seed=k, max_range=12.0))
    assert len(m.submap_ids) == 3   # two finished, one active
    path = str(tmp_path / "mapper.cblox")
    size = m.saveToFile(path)
    assert size == os.path.getsize(path)
    ctx2 = api.Context(0)
    ids, poses = api.load_submap_collection(ctx2, path)
    assert ids.tolist() == sorted(m.submap_ids)
    want = np.array([vm._pose4_to_T(m.submap_pose[i]) for i in ids.tolist()], np.float32)
    assert poses.tobytes() == want.tobytes()
    ids_l = ids.tolist()
    xyzyaw = np.array([m.submap_pose[i] for i in ids_l])
    a = _finished_state(ctx, ids_l, want, xyzyaw)
    b = _finished_state(ctx2, ids_l, poses, xyzyaw)
    assert a[1] and a[1] == b[1]   # overlapping pairs
    for sid in ids_l:
        _identical(a[0][sid], b[0][sid])
    _identical(a[2], b[2])
    assert a[2][0] and a[2][1] > 0
    ctx.close()
    ctx2.close()


def test_config2_sized_round_trip():
    from voxgraph_b200 import api, synth
    sc = synth.make_scene(seed=2, n_submaps=50, n_points=100, radius=8.0, size_xy=(48.0, 32.0),
                          n_clutter=80, n_walls=6, workers=8)
    ctx = api.Context(0)
    for s in sc.submaps:
        ctx.submap_upload(s.submap_id, s.voxel_size, s.vps, s.block_idx, s.distance, s.weight)
    ids = [s.submap_id for s in sc.submaps]
    T = np.array([synth.pose_to_T(p) for p in sc.poses_init], np.float32)
    data = ctx.collection_save(ids, T)
    ctx2 = api.Context(0)
    assert ctx2.collection_load(data) == 50
    for s in sc.submaps:
        i1, d1, w1 = ctx.submap_download(s.submap_id)
        i2, d2, w2 = ctx2.submap_download(s.submap_id)
        assert i1.tobytes() == i2.tobytes() and d1.tobytes() == d2.tobytes() and w1.tobytes() == w2.tobytes()
    assert ctx2.collection_save(ids, T) == data
    ctx.close()
    ctx2.close()
