"""The 6-DoF streaming front end on the device: a tilted sensor through pointcloudMessageCallback, a closed loop
with drifting 6-DoF odometry and loop closures from ground truth, height constraints, the loop-closure edge
list, finishMap, and the equivalence of yaw-only 7-vector poses with the 4-DoF path."""
import numpy as np
import pytest

from voxgraph_b200 import api, synth
from voxgraph_b200 import mapper as vm
from voxgraph_b200 import transform as tf

pytestmark = pytest.mark.gpu

F32 = np.float32
# an 8 degree pitch and a lever arm, like the Arche config's T_base_sensor (voxgraph_mapper.yaml:15-19)
T_B_C = np.array([np.cos(np.deg2rad(4)), 0, np.sin(np.deg2rad(4)), 0, 0.1, 0.0, 0.2], F32)


def base_pose(x, y, z, yaw, roll=0.0, pitch=0.0):
    """T_W_B [qw qx qy qz tx ty tz] of R_z(yaw) R_y(pitch) R_x(roll)."""
    qz = tf.exp([0, 0, 0, 0, 0, yaw]); qy = tf.exp([0, 0, 0, 0, pitch, 0]); qx = tf.exp([0, 0, 0, roll, 0, 0])
    T = tf.compose(tf.compose(qz, qy), qx)
    T[4:] = [x, y, z]
    return T


def scan(world, T_W_B, seed, T_B_C=T_B_C, **kw):
    """A LiDAR scan from the sensor at T_W_B * T_B_C, in the sensor frame."""
    T_W_C = tf.compose(T_W_B, T_B_C)
    args = dict(n_beams=24, n_azimuth=360, max_range=10.0)
    args.update(kw)
    return synth.lidar_scan(world, np.r_[T_W_C[4:], 0.0], seed=seed, R_world_sensor=synth.quat_to_matrix(T_W_C[:4]),
                            **args)


def to_mission(m, sid, xyz):
    T = vm._pose4_to_T(m.submap_pose[sid])
    R = synth.quat_to_matrix(T[:4])
    return np.asarray(xyz, np.float64) @ R.T + T[4:]


def by_block(ctx, sid):
    """Block indices, distance, weight and colour bits of a submap, blocks sorted by index."""
    idx, d, w = ctx.submap_download(sid)
    order = np.lexsort(idx.T[::-1])
    return idx[order], d[order].view(np.uint32), w[order].view(np.uint32), ctx.submap_download_colour(sid)[order]


def record_solves(m):
    """Wrap m.pose_graph.optimize: every call appends (exclude_registration, nodes {id: (pose, constant)} and
    relative edges it started from, the poses it left)."""
    pg = m.pose_graph
    optimize = pg.optimize
    log = []

    def recording(exclude_registration_constraints=False):
        nodes = {i: (v[0].copy(), v[1]) for i, v in pg._nodes.items()}
        rel = list(pg._relative)
        s = optimize(exclude_registration_constraints)
        log.append((bool(exclude_registration_constraints), nodes, rel, {i: v[0].copy() for i, v in pg._nodes.items()}))
        return s
    pg.optimize = recording
    return log


def oracle_solve(oracle, nodes, rel, exclude_registration):
    """The oracle's LM over the same nodes (in id order, as the device graph holds them) and relative edges."""
    og = oracle.Graph()
    ids = sorted(nodes)
    for i in ids:
        og.add_node(i, nodes[i][0], constant=nodes[i][1])
    for (i, j, t, L) in rel:
        og.add_relative(i, j, t[:3], t[3], L)
    rc, _ = og.solve(oracle.solver_options(exclude_registration=int(exclude_registration)))
    assert rc == 0
    return ids, og.poses()


def test_tilted_sensor_message(oracle):
    world = synth.make_world(7, size_xy=(40.0, 30.0), n_clutter=60, n_walls=5)
    T_O_B = base_pose(12.0, 14.0, 1.1, 0.4, roll=0.03, pitch=-0.05)
    msg = synth.pack_pointcloud2(scan(world, T_O_B, seed=1, n_beams=32, n_azimuth=512))
    ctx = api.Context(0)
    try:
        tsdf = dict(mode=0, max_ray_length_m=10.0)
        m = vm.VoxgraphMapper(ctx, vm.MapperConfig(capacity_blocks=4096, tsdf=tsdf, T_base_sensor=T_B_C))
        m.pointcloudMessageCallback(0.0, T_O_B, msg)
        # T_S_C = gravity_align(T_O_B)^-1 * T_O_B * T_B_C, composed by the oracle
        G = tf.gravity_align(T_O_B)
        want = oracle.T_compose(oracle.T_compose(oracle.T_inverse(G), T_O_B), T_B_C)
        assert np.abs(m.last_T_S_C - want).max() <= 1e-6
        # the submap is the direct integration of the message at that T_S_C
        ctx.submap_create(900, 0.2, 16, 4096)
        ctx.tsdf_integrate_cloud(900, m.last_T_S_C, msg, ctx.tsdf_config(**tsdf))
        assert ctx.submap_has_colour(0)
        for a, b in zip(by_block(ctx, 0), by_block(ctx, 900)):
            assert np.array_equal(a, b)
        # the same scan as a 4-vector [sensor position, sensor yaw] ignores the tilt
        T_W_C = tf.compose(T_O_B, T_B_C)
        m4 = vm.VoxgraphMapper(ctx, vm.MapperConfig(capacity_blocks=4096, tsdf=tsdf), first_submap_id=10)
        m4.pointcloudMessageCallback(0.0, np.r_[T_W_C[4:], tf.log(T_W_C)[5]], msg)
        m.finishMap(); m4.finishMap()
        err = {}
        for mm, sid in ((m, 0), (m4, 10)):
            xyz, _, _ = ctx.submap_download_points(sid, api.K_ISOSURFACE_POINTS)
            assert len(xyz) > 500
            err[sid] = float(np.mean(np.abs(synth.world_sdf(world, to_mission(mm, sid, xyz)))))
        print("isosurface distance to the world: 6-DoF %.4f m, yaw only %.4f m" % (err[0], err[10]))
        assert err[0] < 0.15 and err[0] < 0.5 * err[10]
    finally:
        ctx.close()


# --------------------------------------------------------------------------- the loop
N_PER_SUBMAP = 6
N_SUBMAPS = 7


def loop_trajectory():
    """Ground truth around a loop that ends where it started, and an odometry whose yaw and position drift."""
    n = N_PER_SUBMAP * N_SUBMAPS
    s = 2 * np.pi * np.arange(n) / (N_PER_SUBMAP * (N_SUBMAPS - 1))     # back at the start as the last submap begins
    gt, odo = [], []
    for k in range(n):
        x, y = 15.0 + 7.0 * np.cos(s[k]), 12.0 + 5.0 * np.sin(s[k])
        yaw = np.arctan2(5.0 * np.cos(s[k]), -7.0 * np.sin(s[k]))
        T = base_pose(x, y, 1.2, yaw, roll=0.03 * np.sin(3 * s[k]), pitch=0.04 * np.cos(2 * s[k]))
        gt.append(T)
        D = tf.exp([0.012 * k, -0.008 * k, 0.0, 0.0, 0.0, 0.004 * k])       # drift about the start
        odo.append(tf.compose(tf.compose(gt[0], D), tf.compose(tf.inverse(gt[0]), T)))
    return gt, odo


@pytest.fixture(scope="module")
def loop_world():
    world = synth.make_world(11, size_xy=(30.0, 24.0), n_clutter=50, n_walls=3)
    gt, odo = loop_trajectory()
    scans = [scan(world, T, seed=k) for k, T in enumerate(gt)]
    return world, gt, odo, scans


def run_loop(loop_world, loop_closure):
    world, gt, odo, scans = loop_world
    ctx = api.Context(0)
    cfg = vm.MapperConfig(submap_creation_interval=N_PER_SUBMAP / 10.0 - 0.05, capacity_blocks=4096,
                          tsdf=dict(max_ray_length_m=10.0), T_base_sensor=T_B_C,
                          loop_closure_information=np.diag([100.0, 100.0, 100.0, 1000.0]))
    m = vm.VoxgraphMapper(ctx, cfg)
    solves = record_solves(m)
    lc = None
    k_lc = N_PER_SUBMAP * (N_SUBMAPS - 1) - 1           # the last scan before the last submap, near the start
    for k in range(len(gt)):
        m.pointcloudCallback(k / 10.0, odo[k], scans[k])
        if loop_closure and k == k_lc:
            # a loop closure from scan 1 to now, from the ground truth
            T = tf.compose(tf.inverse(gt[1]), gt[k])
            lc = (k, m.loopClosureCallback(0.1, k / 10.0, T), T)
    m.finishMap()
    return ctx, m, lc, solves


def gt_submap_pose(gt, m, sid):
    k = int(round(m.submap_start[sid] * 10.0))
    return tf.to_pose4(tf.gravity_align(gt[k]))


def test_loop_closure_stream(loop_world, oracle):
    world, gt, odo, scans = loop_world
    ctx0, m0, _, solves0 = run_loop(loop_world, False)
    ctx, m, (k_lc, ab, T_lc), solves = run_loop(loop_world, True)
    try:
        assert len(m.submap_ids) == N_SUBMAPS and m.submap_ids == m0.submap_ids
        a, b = ab
        assert a == 0 and b == N_SUBMAPS - 2 == m.lookupActiveSubmapByTime(k_lc / 10.0)
        assert not m.loop_closure_warnings
        # the A -> B edge: T_A_t1 * T_t1_t2 * T_B_t2^-1 as [t, yaw]
        T_AB = oracle.T_compose(oracle.T_compose(m.lookupPoseByTime(a, 0.1), T_lc),
                                oracle.T_inverse(m.lookupPoseByTime(b, k_lc / 10.0)))
        edge = [r for r in m.pose_graph._relative if r[:2] == (a, b)]
        assert len(edge) == 1 and np.abs(edge[0][2] - tf.to_pose4(T_AB)).max() <= 1e-6
        # the first optimisation after it (the switch to the last submap): two solves, the first without
        # registration; every other optimisation one solve with registration
        assert [s[0] for s in solves0] == [False] * N_SUBMAPS
        assert [s[0] for s in solves] == [False] * (N_SUBMAPS - 2) + [True, False, False]
        rec = [t for t in m.timings if "preoptimize_ms" in t]
        assert len(rec) == 1 and rec[0] is m.timings[N_SUBMAPS - 1] and rec[0]["pre_lm_iterations"] >= 1
        _, nodes, rel, solved = solves[N_SUBMAPS - 2]
        ids, xo = oracle_solve(oracle, nodes, rel, True)
        xg = np.array([solved[i] for i in ids])
        print("pre-solve vs oracle: max |dx| %.3g" % np.abs(xg - xo).max())
        assert np.abs(xg - xo).max() < 1e-6
        # the loop closure pulls the last submap back to the ground truth
        last = m.submap_ids[-1]
        errs = []
        for mm in (m, m0):
            d = mm.submap_pose[last] - gt_submap_pose(gt, mm, last)
            errs.append(float(np.hypot(d[0], d[1]) + abs(np.angle(np.exp(1j * d[3])))))
        print("last submap pose error to the ground truth: with the loop closure %.4f, without %.4f" % tuple(errs))
        assert errs[0] < errs[1]
        # finishMap: the last submap has isosurface points, overlaps others and is registered
        assert ctx.submap_num_points(last, api.K_ISOSURFACE_POINTS) > 0
        assert any(last in p for p in m.overlapping_submap_list)
        assert any(last in blk for blk in m.pose_graph.registration_blocks)
        # the loop-closure edge list
        edges = m.loopClosureEdges()
        pairs = m.overlapping_submap_list
        assert len(edges) == len(pairs) > 0
        try:
            cov = m.pose_graph.getEdgeCovarianceMap(pairs)
        except api.VgxError:
            cov = None
        for (pa, pb), (ta, tb, T_A_B, c6) in zip(pairs, edges):
            assert (ta, tb) == (m.submap_start[pa], m.submap_start[pb])
            T_M_A = oracle.T_compose(vm._pose4_to_T(m.submap_pose[pa]), m.lookupPoseByTime(pa, ta))
            T_M_B = oracle.T_compose(vm._pose4_to_T(m.submap_pose[pb]), m.lookupPoseByTime(pb, tb))
            assert np.abs(T_A_B - oracle.T_compose(oracle.T_inverse(T_M_A), T_M_B)).max() <= 1e-6
            if cov is None:
                assert np.array_equal(c6, np.eye(6))
            else:
                idx = [0, 1, 2, 5]
                assert np.array_equal(c6[np.ix_(idx, idx)], cov[(pa, pb)])
                rest = np.ones((6, 6), bool); rest[np.ix_(idx, idx)] = False
                assert np.all(c6[rest] == 1e4)
    finally:
        ctx.close(); ctx0.close()


def test_height_constraints_match_the_oracle(oracle):
    world = synth.make_world(5, size_xy=(30.0, 24.0), n_clutter=40, n_walls=3)
    n = 16
    gt = [base_pose(6.0 + 0.8 * k, 12.0 + 0.3 * np.sin(0.4 * k), 1.2, 0.05 * k, roll=0.02, pitch=-0.03)
          for k in range(n)]
    odo = [tf.compose(T, tf.exp([0, 0, 0.02 * k, 0, 0, 0.003 * k])) for k, T in enumerate(gt)]   # drifting height
    ctx = api.Context(0)
    try:
        m = vm.VoxgraphMapper(ctx, vm.MapperConfig(submap_creation_interval=0.35, capacity_blocks=4096,
                                                   tsdf=dict(max_ray_length_m=10.0), T_base_sensor=T_B_C,
                                                   height_constraints_enabled=True,
                                                   registration_constraints_enabled=False))
        solves = record_solves(m)
        for k in range(n):
            m.pointcloudCallback(k / 10.0, odo[k], scan(world, gt[k], seed=k, n_beams=12, n_azimuth=180))
        frame = api.FRAME_NODE_ID_BASE
        assert m.pose_graph.hasReferenceFrameNode(0) and len(m.submap_ids) == 4 and len(solves) == 3
        for exclude, nodes, rel, solved in solves:
            assert not exclude and nodes[frame][1] and sum(r[0] == frame for r in rel) == len(nodes) - 2
            ids, xo = oracle_solve(oracle, nodes, rel, False)
            xg = np.array([solved[i] for i in ids])
            print("height solve vs oracle: max |dz| %.3g, max |dx| %.3g"
                  % (np.abs(xg[:, 2] - xo[:, 2]).max(), np.abs(xg - xo).max()))
            assert np.abs(xg - xo).max() < 1e-6
    finally:
        ctx.close()


def test_yaw_only_7_vectors_match_4_vectors():
    """Registration is off: its LM stopping rule would turn last-bit differences of the two paths' float and
    float64 algebra into differences as large as its parameter tolerance."""
    world = synth.make_world(7, size_xy=(40.0, 30.0), n_clutter=60, n_walls=5)
    n = 16
    s_arc = np.arange(n) * 0.6
    p4 = np.stack([8.0 + s_arc, 12.0 + 0.5 * np.sin(s_arc / 3.0), np.full(n, 1.2), 0.05 * s_arc], -1)
    scans = [synth.lidar_scan(world, p4[k], n_beams=24, n_azimuth=360, seed=k, max_range=10.0) for k in range(n)]
    out = []
    for as_7 in (False, True):
        ctx = api.Context(0)
        try:
            m = vm.VoxgraphMapper(ctx, vm.MapperConfig(submap_creation_interval=0.35, capacity_blocks=4096,
                                                       tsdf=dict(mode=0, max_ray_length_m=10.0),
                                                       registration_constraints_enabled=False))
            for k in range(n):
                pose = np.r_[np.cos(p4[k, 3] / 2), 0, 0, np.sin(p4[k, 3] / 2), p4[k, :3]] if as_7 else p4[k]
                m.pointcloudCallback(k / 10.0, pose, scans[k])
            blocks = {i: set(map(tuple, ctx.submap_download(i)[0])) for i in m.submap_ids}
            out.append((list(m.submap_ids), blocks, np.array([m.submap_pose[i] for i in m.submap_ids])))
        finally:
            ctx.close()
    (ids4, b4, x4), (ids7, b7, x7) = out
    assert ids4 == ids7 and len(ids4) == 4
    assert b4 == b7
    print("4-vector vs 7-vector poses: max |dx| %.3g" % np.abs(x4 - x7).max())
    assert np.abs(x4 - x7).max() < 1e-5
