"""Host logic of the 6-DoF front end without a GPU: the float transforms (voxgraph_b200/transform.py) against the
oracle's minkindr restatement, the MapTracker algebra of VoxgraphMapper (map_tracker.cpp:30-126), the submap
timeline and pose history, loop closures (voxgraph_mapper.cpp:267-340), the pre-optimisation after them
(pose_graph_interface.cpp:177-198), height constraints, finishMap and the loop-closure edge list, all driven
through the recording stand-in for the Context of test_host_mapper.py."""
import numpy as np
import pytest

from test_host_mapper import FakeCtx
from voxgraph_b200 import _lib, api, synth
from voxgraph_b200 import mapper as vm
from voxgraph_b200 import transform as tf

F32 = np.float32
LC_INFO = np.diag([100.0, 100.0, 100.0, 1000.0])


class Ctx(FakeCtx):
    """FakeCtx that also records each solve's exclude_registration and each edge set's square roots, answers
    edge covariances, and (still=True) leaves the poses where they are."""

    def __init__(self, still=False, covariance_rc=0):
        super().__init__()
        self.still = still
        self.covariance_rc = covariance_rc
        self.edges = None

    def graph_set_relative_edges(self, a, b, t, L):
        self.edges = (list(a), list(b), np.array(t), np.array(L))
        super().graph_set_relative_edges(a, b, t, L)

    def graph_solve(self, n, o):
        self.calls.append(("solve_excl", int(o.exclude_registration)))
        if self.still:
            self.calls.append(("solve", n))
            return self.nodes[1].copy(), type("S", (), {"iterations": 3})()
        return super().graph_solve(n, o)

    def graph_edge_covariances(self, a, b):
        if self.covariance_rc:
            raise api.VgxError(self.covariance_rc, "rank-deficient")
        return np.array([np.arange(16.0).reshape(4, 4) + 100 * k for k in range(len(a))])


def rot_T(axis, angle, t=(0, 0, 0)):
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    return np.array([np.cos(angle / 2), *(np.sin(angle / 2) * axis), *t], F32)


def tilted_poses(n, seed=0):
    """A drifting 6-DoF odometry: forward along a curve with a few degrees of roll and pitch."""
    rs = np.random.RandomState(seed)
    out = []
    for k in range(n):
        yaw = 0.05 * k
        roll, pitch = 0.06 * np.sin(0.3 * k), 0.04 * np.cos(0.2 * k) + 0.01 * rs.normal()
        R = synth.rot_z(yaw) @ _rot_y(pitch) @ _rot_x(roll)
        M = np.eye(4); M[:3, :3] = R; M[:3, 3] = [0.3 * k, 0.1 * k + 0.02 * rs.normal(), 1.0 + 0.01 * k]
        out.append(tf.from_matrix(M))
    return out


def _rot_x(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[1, 0, 0], [0, c, -s], [0, s, c]])


def _rot_y(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])


T_BASE_SENSOR = tf.from_matrix(np.array([[-0.9908275, -0.0196803, 0.1336922, -0.024],     # voxgraph_mapper.yaml:15-19
                                         [0.0202159, -0.9997921, 0.0026504, -0.011],
                                         [0.1336122, 0.0053288, 0.9910194, -0.131],
                                         [0.0, 0.0, 0.0, 1.0]]))


# --------------------------------------------------------------------------- transforms
def test_transforms_match_the_oracle(oracle):
    rs = np.random.RandomState(1)
    for _ in range(300):
        v = rs.uniform(-4, 4, 6).astype(F32)
        w = rs.uniform(-4, 4, 6).astype(F32)
        A, B = oracle.T_exp(v), oracle.T_exp(w)
        assert np.abs(tf.exp(v) - A).max() <= 1e-6
        assert np.abs(tf.compose(A, B) - oracle.T_compose(A, B)).max() <= 1e-6
        assert np.abs(tf.inverse(A) - oracle.T_inverse(A)).max() <= 1e-6
    # the small-angle branch of exp
    v = np.array([1, 2, 3, 1e-6, -2e-6, 3e-6], F32)
    assert np.abs(tf.exp(v) - oracle.T_exp(v)).max() <= 1e-7


def test_log_closed_forms_and_round_trip():
    rs = np.random.RandomState(2)
    for _ in range(300):
        T = tf.exp(np.concatenate([rs.uniform(-5, 5, 3), rs.uniform(-1, 1, 3) * rs.uniform(0, np.pi)]))
        back = tf.exp(tf.log(T))
        back[:4] *= np.sign(back[0] * T[0])          # a rotation vector longer than pi comes back as -q
        assert np.abs(back - T).max() <= 2e-6
    # [t; yaw] of a yaw-only pose, [t; angle * axis] of a rotation about x, and -q == q
    assert np.allclose(tf.log(rot_T([0, 0, 1], 0.7, (1, 2, 3))), [1, 2, 3, 0, 0, 0.7], atol=1e-6)
    assert np.allclose(tf.log(rot_T([1, 0, 0], -2.5)), [0, 0, 0, -2.5, 0, 0], atol=1e-6)
    q = rot_T([0, 1, 1], 1.2, (4, 5, 6))
    neg = np.concatenate([-q[:4], q[4:]])
    assert np.allclose(tf.log(neg), tf.log(q), atol=1e-6)
    # a yaw beyond pi comes back on (-pi, pi]
    assert np.allclose(tf.log(rot_T([0, 0, 1], 3.5))[5], 3.5 - 2 * np.pi, atol=1e-6)
    assert np.array_equal(tf.log(tf.IDENTITY), np.zeros(6, F32))


def test_gravity_align():
    for yaw in (-3.0, -0.4, 0.0, 1.3, 3.1):
        T = rot_T([0, 0, 1], yaw, (1.5, -2.0, 0.7))
        assert np.abs(tf.gravity_align(T) - T).max() <= 1e-6
    T = tf.compose(rot_T([0, 0, 1], 0.8, (3, 4, 5)), rot_T([1, 0.3, 0], 0.14))
    G = tf.gravity_align(T)
    v = tf.log(G)
    assert abs(v[3]) < 1e-7 and abs(v[4]) < 1e-7
    assert np.allclose(v[[0, 1, 2, 5]], tf.log(T)[[0, 1, 2, 5]], atol=1e-6)
    assert np.abs(tf.log(T)[3:5]).max() > 0.05


def test_as_transform():
    assert np.allclose(tf.as_transform([1, 2, 3, 0.5]), rot_T([0, 0, 1], 0.5, (1, 2, 3)), atol=1e-7)
    T = rot_T([0.2, -1, 0.4], 2.2, (1, 2, 3))
    M = np.eye(4); M[:3, :3] = synth.quat_to_matrix(T[:4]); M[:3, 3] = T[4:]
    got = tf.as_transform(M)
    assert np.abs(got[:4] * np.sign(got[0]) - T[:4] * np.sign(T[0])).max() < 1e-6
    assert np.array_equal(got[4:], T[4:])
    for R in (np.diag([1.0, -1, -1]), np.diag([-1.0, 1, -1]), np.diag([-1.0, -1, 1])):   # every branch of the trace test
        M = np.eye(4); M[:3, :3] = R
        assert np.allclose(synth.quat_to_matrix(tf.as_transform(M)[:4]), R, atol=1e-6)
    with pytest.raises(ValueError, match="unit norm"):
        tf.as_transform([1, 2, 3, 0, 0, 0, 1])        # [t; x y z w] by mistake is refused
    with pytest.raises(ValueError, match="shape"):
        tf.as_transform([1, 2, 3])


# --------------------------------------------------------------------------- the 6-DoF tracker
def _restated_tracker(poses, times, interval, T_B_C, submap_pose_of):
    """MapTracker + switchToNewSubmap restated with the oracle-checked primitives -> per scan the expected
    T_S_C, per switch the new node pose and the odometry edge."""
    init = tf.IDENTITY
    start = None
    T_S_C, nodes, edges = [], [], []
    for k, (t, T_O_B) in enumerate(zip(times, poses)):
        T_S_B = tf.compose(init, T_O_B)
        if start is None or t >= start + interval:
            T_M_B = T_O_B if start is None else tf.compose(vm._pose4_to_T(submap_pose_of(len(nodes) - 1)), T_S_B)
            nodes.append(tf.to_pose4(tf.gravity_align(T_M_B)))
            T_S1_B = T_S_B
            init = tf.inverse(tf.gravity_align(T_O_B))
            T_S_B = tf.compose(init, T_O_B)
            if start is not None:
                edges.append(tf.to_pose4(tf.compose(T_S1_B, tf.inverse(T_S_B))))
            start = t
        T_S_C.append(tf.compose(T_S_B, T_B_C))
    return T_S_C, nodes, edges


def test_6dof_run_frames_nodes_and_odometry_edges():
    ctx = Ctx(still=True)
    m = vm.VoxgraphMapper(ctx, vm.MapperConfig(submap_creation_interval=1.0, T_base_sensor=T_BASE_SENSOR))
    poses = tilted_poses(25)
    times = [0.1 * k for k in range(25)]
    pts = np.zeros((3, 3), F32)
    for t, T in zip(times, poses):
        m.pointcloudCallback(t, T, pts)
    assert m.submap_ids == [0, 1, 2]
    exp_T_S_C, exp_nodes, exp_edges = _restated_tracker(poses, times, 1.0, T_BASE_SENSOR, lambda i: m.submap_pose[i])
    integ = [c for c in ctx.calls if c[0] == "integrate"]
    assert len(integ) == 25
    for k, c in enumerate(integ):
        assert np.abs(c[2] - exp_T_S_C[k]).max() <= 1e-6, k
    assert np.array_equal(m.last_T_S_C, integ[-1][2])
    # the first scan of each submap: gravity_align(T_O_B)^-1 * T_O_B * T_B_C, which is not the identity
    for first in (0, 10, 20):
        want = tf.compose(tf.compose(tf.inverse(tf.gravity_align(poses[first])), poses[first]), T_BASE_SENSOR)
        assert np.abs(integ[first][2] - want).max() <= 1e-6
        assert np.abs(integ[first][2] - tf.IDENTITY).max() > 0.1
        # ... and the submap frame is level while the base link is not
        assert np.abs(tf.log(tf.compose(tf.inverse(tf.gravity_align(poses[first])), poses[first]))[3:5]).max() > 0.01
    # node poses [t, yaw] of the gravity-aligned submap poses (the fake solver leaves them in place)
    assert ctx.nodes[0] == [0, 1, 2]
    assert np.abs(ctx.nodes[1] - np.array(exp_nodes)).max() <= 1e-6
    assert np.allclose(ctx.nodes[1][0][:3], poses[0][4:], atol=1e-6)
    # odometry edges T_S1_B * T_S2_B^-1 reduced to [t, log()[5]]
    assert ctx.edges[0] == [0, 1] and ctx.edges[1] == [1, 2]
    assert np.abs(ctx.edges[2] - np.array(exp_edges)).max() <= 1e-6
    # the odometry edge is the relative pose of the two base-link poses seen from the level submap frames
    # (T_S1_B = G0^-1 T_O_B and T_S2_B = G10^-1 T_O_B at the switch, G the gravity-aligned submap frames)
    E = tf.compose(tf.inverse(tf.gravity_align(poses[0])), tf.gravity_align(poses[10]))
    assert np.abs(ctx.edges[2][0] - tf.to_pose4(E)).max() <= 1e-6


def test_6dof_without_extrinsic_and_4x4_input():
    """A 4x4 T_O_B and no extrinsic: T_S_C = T_S_B; a 4-vector after 6-DoF poses counts as zero roll/pitch."""
    ctx = Ctx(still=True)
    m = vm.VoxgraphMapper(ctx, vm.MapperConfig(submap_creation_interval=1.0))
    T = tilted_poses(3)[2]
    M = np.eye(4); M[:3, :3] = synth.quat_to_matrix(T[:4]); M[:3, 3] = T[4:]
    m.pointcloudCallback(0.0, M, np.zeros((1, 3), F32))
    want = tf.compose(tf.inverse(tf.gravity_align(T)), T)
    assert np.abs(m.last_T_S_C - want).max() <= 1e-6
    m.pointcloudCallback(0.1, [0.0, 0.0, 1.0, 0.3], np.zeros((1, 3), F32))
    want = tf.compose(tf.inverse(tf.gravity_align(T)), tf.exp([0, 0, 1, 0, 0, 0.3]))
    assert np.abs(m.last_T_S_C - want).max() <= 1e-6
    # a mapper that started on 4-DoF poses refuses a 6-DoF one
    m4 = vm.VoxgraphMapper(Ctx(), vm.MapperConfig())
    m4.pointcloudCallback(0.0, [0, 0, 0, 0], np.zeros((1, 3), F32))
    with pytest.raises(ValueError, match="4-DoF"):
        m4.pointcloudCallback(0.1, tf.IDENTITY, np.zeros((1, 3), F32))


def test_4dof_path_makes_the_same_calls():
    """[x y z yaw] poses and no extrinsic: the calls and arrays of the 4-DoF float64 algebra, nothing more."""
    ctx = Ctx()
    cfg = vm.MapperConfig(voxel_size=0.15, submap_creation_interval=1.0, capacity_blocks=64)
    m = vm.VoxgraphMapper(ctx, cfg, first_submap_id=10)
    rs = np.random.RandomState(4)
    poses = [np.array([0.1 * k, 0.05 * k, 0.01 * k, 0.02 * k]) + rs.normal(0, 0.01, 4) for k in range(25)]
    pts = np.zeros((4, 3), F32)
    for k in range(25):
        m.pointcloudCallback(0.1 * k, poses[k], pts)
    # restated: the old algebra, with the fake optimiser's +0.5 m on every free node at every solve
    want, sub_pose, odom, sids = [], {}, None, []
    for k in range(25):
        p = poses[k]
        if not sids or 0.1 * k >= 0.1 * (10 * (len(sids) - 1)) + 1.0:
            sid = 10 + len(sids)
            if sids:
                want += [("finish", sids[-1]), ("extract", sids[-1])]
                if len(sids) >= 2:
                    want.append(("overlap", list(sids)))
            want.append(("create", sid))
            if not sids:
                sub_pose[sid] = p.copy()
            else:
                T_S1_S2 = vm._compose4(vm._inverse4(odom), p)
                sub_pose[sid] = vm._compose4(sub_pose[sids[-1]], T_S1_S2)
                want += [("nodes",), ("rel", T_S1_S2)] + [("reg",)] * (len(sids) >= 2) + [("solve_excl", 0), ("solve",)]
            sids.append(sid)
            odom = p.copy()
            if len(sids) >= 2:
                for i in sids[1:]:
                    sub_pose[i] = sub_pose[i].copy(); sub_pose[i][0] += 0.5
        want.append(("integrate", sids[-1], vm._pose4_to_T(vm._compose4(vm._inverse4(odom), p))))
    got = [c for c in ctx.calls if c[0] in ("finish", "extract", "overlap", "reg", "create", "nodes", "rel",
                                            "solve_excl", "solve", "integrate")]
    assert [c[0] for c in got] == [w[0] for w in want]
    for g, w in zip(got, want):
        if w[0] == "integrate":
            assert g[1] == w[1] and np.array_equal(g[2], w[2])
        elif w[0] == "rel":
            assert np.array_equal(g[3][-1], w[1])
        elif w[0] in ("finish", "extract", "create"):
            assert g[1] == w[1]
    assert not m.pose_graph._frames and "preoptimize_ms" not in m.timings[-1]
    assert [k for k in m.timings[-1]] == ["finish_ms", "overlap_ms", "pairs", "view_ms", "finished_blocks",
                                          "isosurface_points", "optimize_ms", "lm_iterations", "registration_blocks"]
    # the history holds the 4-DoF T_S_C as a yaw quaternion
    assert np.array_equal(m.lookupPoseByTime(12, 0.1 * 24), want[-1][2])


# --------------------------------------------------------------------------- timeline and history
def test_timeline_and_pose_history_are_step_lookups():
    ctx = Ctx(still=True)
    m = vm.VoxgraphMapper(ctx, vm.MapperConfig(submap_creation_interval=1.0), first_submap_id=3)
    assert m.lookupActiveSubmapByTime(0.0) is None
    times = [0.5 + 0.25 * k for k in range(9)]          # submaps 3, 4, 5 start at 0.5, 1.5, 2.5
    poses = tilted_poses(9)
    for t, T in zip(times, poses):
        m.pointcloudCallback(t, T, np.zeros((1, 3), F32))
    assert [m.submap_start[i] for i in m.submap_ids] == [0.5, 1.5, 2.5]
    assert m.lookupActiveSubmapByTime(0.4999) is None                      # before the first scan
    assert m.lookupActiveSubmapByTime(0.5) == 3                            # a creation time belongs to its submap
    assert m.lookupActiveSubmapByTime(1.4999) == 3
    assert m.lookupActiveSubmapByTime(1.5) == 4
    assert m.lookupActiveSubmapByTime(1e9) == 5
    assert m.lookupPoseByTime(3, 0.49) is None
    # step lookups: the pose of the last scan at or before t
    integ = [c[2] for c in ctx.calls if c[0] == "integrate"]
    assert np.array_equal(m.lookupPoseByTime(3, 0.5), integ[0])            # no extrinsic: T_S_B == T_S_C
    assert np.array_equal(m.lookupPoseByTime(3, 0.74), integ[0])
    assert np.array_equal(m.lookupPoseByTime(3, 0.75), integ[1])
    assert np.array_equal(m.lookupPoseByTime(3, 1.4), integ[3])
    assert np.array_equal(m.lookupPoseByTime(4, 1.6), integ[4])
    assert m.lookupPoseByTime(5, 2.4) is None
    # the history in the mission frame: submaps in id order, each in time order, T_M_S * T_S_B
    hist = m.getPoseHistory()
    assert [h[0] for h in hist] == times
    for (t, T_M_B), sid, T_S_B in zip(hist, [3] * 4 + [4] * 4 + [5], integ):
        assert np.abs(T_M_B - tf.compose(vm._pose4_to_T(m.submap_pose[sid]), T_S_B)).max() <= 1e-6
        # ... which is the odometry pose again, up to the submap frame's float round trip
        assert np.abs(T_M_B[4:] - poses[times.index(t)][4:]).max() < 1e-4
    # a repeated timestamp keeps the first pose, as std::map::emplace
    first = m.lookupPoseByTime(5, 2.5)
    m._add_pose_to_history(5, 2.5, tf.IDENTITY)
    assert m.lookupPoseByTime(5, 2.5) is first


# --------------------------------------------------------------------------- loop closures
def _two_submap_mapper(**cfg):
    ctx = Ctx(still=True)
    m = vm.VoxgraphMapper(ctx, vm.MapperConfig(submap_creation_interval=1.0, **cfg))
    for k, T in enumerate(tilted_poses(15)):
        m.pointcloudCallback(0.1 * k, T, np.zeros((1, 3), F32))
    return ctx, m


def test_loop_closure_refusals_in_the_reference_order():
    ctx, m = _two_submap_mapper(loop_closure_information=LC_INFO)
    assert m.submap_ids == [0, 1]
    ok = np.array([1, 0, 0, 0, 0.5, 0, 0])
    bad_q = np.array([0.9, 0, 0, 0, 0.5, 0, 0])
    # before the first submap -> no submap; that check comes before the quaternion's
    assert m.loopClosureCallback(-1.0, 1.2, bad_q) is None
    # the same submap (also before the quaternion check)
    assert m.loopClosureCallback(0.2, 0.3, bad_q) is None
    # no pose: a time inside submap 1 but before its first recorded pose (moved from 1.0 to 1.05 to make one)
    m._history[1][0][0] = 1.05
    assert m.loopClosureCallback(0.2, 1.02, bad_q) is None
    m._history[1][0][0] = 1.0
    assert m.loopClosureCallback(0.2, 1.2, bad_q) is None
    w = m.loop_closure_warnings
    assert len(w) == 4
    assert w[0] == "Could not add loop closure from timestamp -1.0 to 1.2: timestamp A or B has no corresponding submap"
    assert w[1].endswith(": timestamp A and B fall within the same submap")
    assert w[2].endswith(": timestamp A or B has no corresponding robot pose")
    assert w[3].endswith(": supplied transform quaternion is invalid")
    n_rel = len(m.pose_graph._relative)
    assert m.loopClosureCallback(0.2, 1.2, ok) == (0, 1)
    assert len(m.pose_graph._relative) == n_rel + 1 and len(w) == 4
    # a quaternion off unit norm by less than the tolerance is normalised
    assert m.loopClosureCallback(0.2, 1.2, np.array([1.0004, 0, 0, 0, 0.5, 0, 0])) == (0, 1)
    assert np.array_equal(m.pose_graph._relative[-1][2], m.pose_graph._relative[-2][2])


def test_loop_closure_needs_its_information_matrix():
    ctx, m = _two_submap_mapper()
    with pytest.raises(ValueError, match="loop_closure_information"):
        m.loopClosureCallback(0.2, 1.2, [1, 0, 0, 0, 0, 0, 0])


def test_loop_closure_constraint_and_preoptimisation():
    ctx, m = _two_submap_mapper(loop_closure_information=LC_INFO)
    T_t1_t2 = rot_T([0, 0, 1], 0.3, (0.4, -0.2, 0.05))
    assert m.loopClosureCallback(0.25, 1.35, T_t1_t2) == (0, 1)
    a, b, t_obs, L = m.pose_graph._relative[-1]
    T_AB = tf.compose(tf.compose(m.lookupPoseByTime(0, 0.25), T_t1_t2), tf.inverse(m.lookupPoseByTime(1, 1.35)))
    assert (a, b) == (0, 1) and np.abs(t_obs - tf.to_pose4(T_AB)).max() <= 1e-6
    assert np.allclose(L, np.linalg.cholesky(LC_INFO))
    ctx.calls.clear()
    for k in range(15, 25):                          # the next switch: pre-solve, then the full solve
        m.pointcloudCallback(0.1 * k, tilted_poses(25)[k], np.zeros((1, 3), F32))
    assert [c[1] for c in ctx.calls if c[0] == "solve_excl"] == [1, 0]
    assert m.timings[-1]["pre_lm_iterations"] == 3 and m.timings[-1]["preoptimize_ms"] >= 0
    ctx.calls.clear()
    for k in range(25, 35):                          # and the one after it: the full solve alone
        m.pointcloudCallback(0.1 * k, tilted_poses(35)[k], np.zeros((1, 3), F32))
    assert [c[1] for c in ctx.calls if c[0] == "solve_excl"] == [0]
    assert "preoptimize_ms" not in m.timings[-1]


# --------------------------------------------------------------------------- height constraints
def test_height_constraints():
    ctx = Ctx(still=True)
    m = vm.VoxgraphMapper(ctx, vm.MapperConfig(submap_creation_interval=1.0, height_constraints_enabled=True))
    poses = tilted_poses(35)
    for k, T in enumerate(poses):
        m.pointcloudCallback(0.1 * k, T, np.zeros((1, 3), F32))
    assert m.submap_ids == [0, 1, 2, 3]
    frame = api.FRAME_NODE_ID_BASE + 0
    ids, x, cst = ctx.nodes
    assert ids == [0, 1, 2, 3, frame] and cst == [1, 0, 0, 0, 1] and np.array_equal(x[-1], np.zeros(4))
    a, b, t, L = ctx.edges
    absolute = [k for k in range(len(a)) if a[k] == frame]
    assert [b[k] for k in absolute] == [1, 2, 3]
    for k, s in zip(absolute, (10, 20, 30)):
        assert np.array_equal(t[k], [0, 0, np.float64(poses[s][6]), 0])
        assert np.array_equal(L[k], np.diag([0, 0, 50.0, 0]))      # semi-definite sqrt of diag(0, 0, 2500, 0)
    # odometry edges stay where they were: one per switch, before that switch's height edge
    assert [(a[k], b[k]) for k in range(len(a)) if a[k] != frame] == [(0, 1), (1, 2), (2, 3)]
    assert [a[k] == frame for k in range(len(a))] == [False, True] * 3
    assert list(m.pose_graph.getSubmapPoses()) == [0, 1, 2, 3]


# --------------------------------------------------------------------------- finishMap and the edge list
def test_finish_map_order_and_later_scan():
    ctx = Ctx(still=True)
    m = vm.VoxgraphMapper(ctx, vm.MapperConfig(submap_creation_interval=1.0))
    for k, T in enumerate(tilted_poses(25)):
        m.pointcloudCallback(0.1 * k, T, np.zeros((1, 3), F32))
    ctx.calls.clear()
    m.finishMap()
    names = [c[0] for c in ctx.calls]
    assert names == ["finish", "extract", "overlap", "nodes", "rel", "reg", "solve_excl", "solve"]
    assert ctx.calls[0][1] == 2 and ctx.calls[2][1] == [0, 1, 2]
    assert m.timings[-1]["finish_map"] and m.timings[-1]["pairs"] == 2 and "optimize_ms" in m.timings[-1]
    assert m.overlapping_submap_list == [(0, 1), (1, 2)]
    with pytest.raises(RuntimeError, match="no active submap"):
        m.pointcloudCallback(2.5, tilted_poses(26)[25], np.zeros((1, 3), F32))
    with pytest.raises(RuntimeError):
        m.finishMap()


@pytest.mark.parametrize("rc", [0, _lib.VGX_ERR_INVALID])
def test_loop_closure_edges(rc):
    ctx = Ctx(still=True, covariance_rc=rc)
    m = vm.VoxgraphMapper(ctx, vm.MapperConfig(submap_creation_interval=1.0))
    poses = tilted_poses(25)
    for k, T in enumerate(poses):
        m.pointcloudCallback(0.1 * k, T, np.zeros((1, 3), F32))
    m.finishMap()
    edges = m.loopClosureEdges()
    assert [(e[0], e[1]) for e in edges] == [(0.0, 1.0), (1.0, 2.0)]
    for k, ((a, b), (ta, tb, T_A_B, c6)) in enumerate(zip(m.overlapping_submap_list, edges)):
        T_M_A = tf.compose(vm._pose4_to_T(m.submap_pose[a]), m.lookupPoseByTime(a, ta))
        T_M_B = tf.compose(vm._pose4_to_T(m.submap_pose[b]), m.lookupPoseByTime(b, tb))
        assert np.abs(T_A_B - tf.compose(tf.inverse(T_M_A), T_M_B)).max() <= 1e-6
        # the robot poses at the submaps' first scans are the odometry poses there
        assert np.abs(tf.compose(tf.inverse(poses[10 * a]), poses[10 * b])[4:] - T_A_B[4:]).max() < 1e-4
        if rc:
            assert np.array_equal(c6, np.eye(6))
        else:
            want = np.full((6, 6), 1e4)
            block = np.arange(16.0).reshape(4, 4) + 100 * k
            for i, mi in enumerate((0, 1, 2, 5)):
                for j, mj in enumerate((0, 1, 2, 5)):
                    want[mi, mj] = block[i, j]
            assert np.array_equal(c6, want)
    ctx.covariance_rc = _lib.VGX_ERR_CUDA                 # any other failure is not swallowed
    with pytest.raises(api.VgxError):
        m.loopClosureEdges()
