"""Host-side mirror of the reference's front end for the streaming path (HP1 -> HP2 online):

  VoxgraphMapper::pointcloudCallback        voxgraph/src/frontend/voxgraph_mapper.cpp:202-265
  VoxgraphMapper::loopClosureCallback       voxgraph_mapper.cpp:267-340
  VoxgraphMapper::finishMapCallback         voxgraph_mapper.cpp:378-404
  VoxgraphMapper::switchToNewSubmap         voxgraph_mapper.cpp:457-510
  VoxgraphMapper::optimizePoseGraph         voxgraph_mapper.cpp:512-524
  VoxgraphMapper::saveToFileCallback        voxgraph_mapper.cpp:412-417
  VoxgraphMapper::saveSeparatedMeshCallback / publishActiveSubmapMeshCallback
                                            voxgraph_mapper.cpp:342-368, 428-433
  MapTracker (odometry T_O_B, extrinsic T_B_C, T_S_B, T_S_C)
                                            src/frontend/map_tracker/map_tracker.cpp:30-126
  PoseGraphInterface::updateRegistrationConstraints / addSubmap / addOdometryMeasurement /
  addLoopClosureMeasurement / addHeightMeasurement / optimize
                                            src/frontend/pose_graph_interface/pose_graph_interface.cpp:24-198
  VoxgraphSubmapCollection::shouldCreateNewSubmap / gravityAlignPose / getPoseHistory, SubmapTimeline,
  VoxgraphSubmap::addPoseToHistory / lookupPoseByTime
  LoopClosureEdgeServer::publishLoopClosureEdges   src/tools/data_servers/loop_closure_edge_server.cpp:31-139

Everything heavy happens behind the C-ABI on the device: the scan is ray-cast into the active
submap (vgx_tsdf_integrate, or vgx_tsdf_integrate_cloud when the scan arrives as a sensor message), a
finished submap gets its registration view, registration points,
surface OBB and isosurface blocks without leaving the GPU (vgx_submap_finish_ex), overlapping pairs
come from vgx_find_overlapping_pairs and the pose graph is solved by vgx_graph_solve.

Two odometry paths.  A 4-vector [x y z yaw] pose with no sensor extrinsic configured is the 4-DoF path,
in float64.  A 7-vector [qw qx qy qz tx ty tz], a 4x4 matrix, or any pose once MapperConfig.T_base_sensor
is set is the 6-DoF odometry pose T_O_B of the base link, and runs the MapTracker algebra in float, as the
reference does (voxgraph_b200.transform): gravity-aligned submaps, T_S_C = T_S_B * T_B_C.  The first scan
decides the path.  ROS, TF lookups and the visualisation/publishing code of the reference are out of
scope: poses and loop closures arrive as arguments.
"""
import bisect
import time
from dataclasses import dataclass, field

import numpy as np

from . import _lib, api
from . import transform as tf


def _pose4_to_T(p):
    """[x, y, z, yaw] -> [qw qx qy qz tx ty tz] (minkindr exp of [t, 0, 0, yaw])."""
    p = np.asarray(p, np.float64)
    return np.array([np.cos(0.5 * p[3]), 0.0, 0.0, np.sin(0.5 * p[3]), p[0], p[1], p[2]], np.float32)


def _compose4(a, b):
    """4-DoF pose a composed with b (b expressed in a's frame)."""
    c, s = np.cos(a[3]), np.sin(a[3])
    out = np.array([a[0] + c * b[0] - s * b[1], a[1] + s * b[0] + c * b[1], a[2] + b[2], a[3] + b[3]])
    out[3] = out[3] - 2 * np.pi * np.floor((out[3] + np.pi) / (2 * np.pi))
    return out


def _inverse4(a):
    c, s = np.cos(a[3]), np.sin(a[3])
    return np.array([-(c * a[0] + s * a[1]), -(-s * a[0] + c * a[1]), -a[2], -a[3]])


@dataclass
class MapperConfig:
    voxel_size: float = 0.2                      # voxgraph_mapper.yaml:21
    voxels_per_side: int = 16
    submap_creation_interval: float = 10.0       # seconds (voxgraph_mapper.yaml submap_creation_interval)
    capacity_blocks: int = 16384
    tsdf: dict = field(default_factory=dict)     # overrides of vgx_tsdf_config (mode 1 = Fast by default)
    registration_filter: dict = field(default_factory=dict)
    registration: dict = field(default_factory=dict)   # RegistrationConstraintConfig overrides
    odometry_information: np.ndarray = field(default_factory=lambda: np.diag([1.0, 1.0, 2500.0, 2500.0]))
    registration_constraints_enabled: bool = True
    odometry_constraints_enabled: bool = True
    mesh_min_weight: float = 2.0                 # voxgraph_mapper.yaml:52 (MeshIntegratorConfig::min_weight)
    colour_map_max: float = 10000.0              # pointcloud_integrator.cpp:14 (GrayscaleColorMap::setMaxValue)
    message_colours: bool = True                 # pointcloudMessageCallback integrates the message's colours
    T_base_sensor: object = None                 # T_base_link_sensor rosparam: [qw qx qy qz tx ty tz] or 4x4;
                                                 # setting it makes every pose a 6-DoF T_O_B
    loop_closure_information: object = None      # measurements/loop_closure/information_matrix (4x4); needed
                                                 # by loopClosureCallback
    height_constraints_enabled: bool = False     # voxgraph_mapper.yaml:48-50
    height_information_zz: float = 2500.0


MISSION_FRAME_ID = 0      # NodeTemplates::kMissionFrame: the frame node of the height constraints


class VoxgraphMapper:
    """Streaming driver: integrate scans, switch submaps on a timer, register online."""

    def __init__(self, ctx, config=None, first_submap_id=0):
        self.ctx = ctx
        self.cfg = config or MapperConfig()
        self.pose_graph = api.PoseGraph(ctx)
        self.submap_ids = []            # creation order
        self.submap_pose = {}           # id -> T_mission_submap [x y z yaw] (optimised)
        self.submap_start = {}
        self._next_id = first_submap_id
        self._last_robot_pose_in_submap = None
        self.timings = []               # one dict per submap switch (and one for finishMap)
        self.scan_stats = []
        self.scan_points = []           # finite points of every message pointcloudMessageCallback integrated
        self.overlapping_submap_list = []
        self.last_T_S_C = None          # [qw qx qy qz tx ty tz] the last scan was integrated at
        self.loop_closure_warnings = []  # why loopClosureCallback refused a loop closure, one line each
        kw = dict(mode=1)
        kw.update(self.cfg.tsdf)
        self.tsdf_cfg = ctx.tsdf_config(**kw)
        self.filter = ctx.registration_filter(**self.cfg.registration_filter)
        # MapTracker state of the 6-DoF path
        self._six_dof = None            # decided by the first scan
        self._T_B_C = (tf.IDENTITY if self.cfg.T_base_sensor is None
                       else tf.as_transform(self.cfg.T_base_sensor, "MapperConfig.T_base_sensor"))
        self._initial_T_S_O = tf.IDENTITY
        self._T_O_B = None
        self._T_S_B = None
        self._history = {}              # id -> ([t], [T_S_B]) in time order (VoxgraphSubmap::pose_history_)
        self._new_loop_closures = False
        self._map_finished = False

    # ---- VoxgraphSubmapCollection
    def empty(self):
        return not self.submap_ids

    @property
    def active_id(self):
        return self.submap_ids[-1]

    def shouldCreateNewSubmap(self, t):
        return self.empty() or t >= self.submap_start[self.active_id] + self.cfg.submap_creation_interval

    def _T_M_S(self, sid):
        """The submap's pose as a transform: its (optimised) 4-DoF pose with zero roll and pitch."""
        return _pose4_to_T(self.submap_pose[sid])

    # ---- SubmapTimeline::lookupActiveSubmapByTime
    def lookupActiveSubmapByTime(self, t):
        """The submap that was active at time t (the last one created at or before t), or None before the first."""
        k = bisect.bisect_right([self.submap_start[i] for i in self.submap_ids], t)
        return self.submap_ids[k - 1] if k else None

    # ---- VoxgraphSubmap::addPoseToHistory / lookupPoseByTime
    def _add_pose_to_history(self, sid, t, T_S_B):
        times, poses = self._history.setdefault(sid, ([], []))
        if times and t <= times[-1]:
            k = bisect.bisect_left(times, t)
            if times[k] == t:          # std::map::emplace keeps the first pose of a timestamp
                return
            times.insert(k, t); poses.insert(k, T_S_B)
        else:
            times.append(t); poses.append(T_S_B)

    def lookupPoseByTime(self, sid, t):
        """T_S_B of submap sid at time t: the last pose recorded at or before t (no interpolation), or None."""
        times, poses = self._history.get(sid, ((), ()))
        k = bisect.bisect_right(times, t)
        return poses[k - 1] if k else None

    # ---- VoxgraphSubmapCollection::getPoseHistory
    def getPoseHistory(self):
        """[(t, T_M_B)] of every integrated scan: submaps in id order, each in time order, moved to the mission
        frame by the submap's current (optimised) pose."""
        out = []
        for sid in sorted(self._history):
            T_M_S = self._T_M_S(sid)
            out += [(t, tf.compose(T_M_S, T)) for t, T in zip(*self._history[sid])]
        return out

    # ---- VoxgraphMapper::pointcloudCallback
    def pointcloudCallback(self, timestamp, T_mission_sensor, points_C, colours=None):
        """T_mission_sensor: 4-DoF odometry pose of the sensor [x, y, z, yaw], or the 6-DoF odometry pose
        T_O_B of the base link (see the module docstring); points_C: (n, 3); colours:
        (n, 4) uint8 [r g b a] per point (an RGB cloud's colours, or api.grayscale_colours of an intensity
        cloud's), or None.  Coloured scans give the submaps a colour channel, which saveToFile writes."""
        extra = {} if colours is None else {"rgba": colours}      # a colourless scan is the call it always was
        return self._integrate(timestamp, T_mission_sensor,
                               lambda sid, T_S_C: self.ctx.tsdf_integrate(sid, T_S_C, points_C, self.tsdf_cfg, **extra))

    def pointcloudMessageCallback(self, timestamp, T_mission_sensor, msg):
        """pointcloudCallback with the sensor message itself (an api.PointCloud2) instead of arrays, as the
        reference's callback takes it: the records are decoded on the device, those with a non-finite coordinate
        are dropped, and (config message_colours) the message's rgb, the grey of its intensity or black is
        integrated as colour.  No host pass over the points."""
        def integrate(sid, T_S_C):
            st, n_points = self.ctx.tsdf_integrate_cloud(sid, T_S_C, msg, self.tsdf_cfg, self.cfg.message_colours,
                                                         self.cfg.colour_map_max)
            self.scan_points.append(n_points)
            return st
        return self._integrate(timestamp, T_mission_sensor, integrate)

    def _integrate(self, timestamp, pose, integrate):
        """The part of the callback around the integration: integrate(active submap id, T_S_C) -> TsdfStats."""
        if self._map_finished:
            raise RuntimeError("finishMap() finished the last submap: there is no active submap to integrate into")
        if self._takes_6dof(pose):
            self._T_O_B = tf.as_transform(pose, "T_O_B")
            self._T_S_B = tf.compose(self._initial_T_S_O, self._T_O_B)    # MapTracker::updateToTime
        else:
            pose = np.asarray(pose, np.float64)
        if self.shouldCreateNewSubmap(timestamp):
            self.switchToNewSubmap(timestamp, pose)
            self.optimizePoseGraph()
        sid = self.active_id
        # map_tracker_.get_T_S_C(): the sensor in the active submap's frame (odometry, not optimised)
        if self._six_dof:
            T_S_B = self._T_S_B
            T_S_C = tf.compose(T_S_B, self._T_B_C)
        else:
            self._last_T_S_B = _compose4(_inverse4(self._odom_submap_pose), pose)
            T_S_B = T_S_C = _pose4_to_T(self._last_T_S_B)
        st = integrate(sid, T_S_C)
        self.last_T_S_C = T_S_C
        self._add_pose_to_history(sid, timestamp, T_S_B)                # voxgraph_mapper.cpp:253
        self.scan_stats.append(st)
        return st

    def _takes_6dof(self, pose):
        six = self.cfg.T_base_sensor is not None or np.shape(pose) != (4,)
        if self._six_dof is None:
            self._six_dof = six
        elif six and not self._six_dof:
            raise ValueError("this mapper runs on 4-DoF [x y z yaw] poses (its first scan had one); got a pose "
                             "of shape %s" % (np.shape(pose),))
        return self._six_dof

    # ---- VoxgraphMapper::switchToNewSubmap
    def switchToNewSubmap(self, timestamp, T_mission_sensor=None):
        """T_mission_sensor: the scan's 4-DoF pose on the 4-DoF path; the 6-DoF path reads the tracker's T_O_B."""
        rec = {"finish_ms": 0.0, "overlap_ms": 0.0, "pairs": 0}
        ctx = self.ctx
        if not self.empty():
            self._finish_active(rec)
        if self.cfg.registration_constraints_enabled and len(self.submap_ids) >= 2:
            t0 = time.time()
            rec["pairs"] = self.updateRegistrationConstraints()
            rec["overlap_ms"] = (time.time() - t0) * 1e3
        # createNewSubmap(T_M_B): the new submap's frame is the robot's current (odometry) pose
        sid = self._next_id
        self._next_id += 1
        ctx.submap_create(sid, self.cfg.voxel_size, self.cfg.voxels_per_side, self.cfg.capacity_blocks)
        prev = self.submap_ids[-1] if self.submap_ids else None
        if self._six_dof:
            # get_T_M_B(), gravity aligned; the node is its Pose4D [t, log()[5]]
            T_M_B = self._T_O_B if prev is None else tf.compose(self._T_M_S(prev), self._T_S_B)
            pose = tf.to_pose4(tf.gravity_align(T_M_B))
            height = float(self._T_O_B[6])
        elif prev is None:
            pose = T_mission_sensor.copy()
            height = T_mission_sensor[2]
        else:
            # the optimised pose of the previous submap composed with the odometry since its creation
            T_S1_S2 = _compose4(_inverse4(self._odom_submap_pose), T_mission_sensor)
            pose = _compose4(self.submap_pose[prev], T_S1_S2)
            height = T_mission_sensor[2]
        self.submap_ids.append(sid)
        self.submap_pose[sid] = pose
        self.submap_start[sid] = timestamp
        self.pose_graph.addSubmapNode(api.SubmapNodeConfig(sid, pose, set_constant=(prev is None)))   # addSubmap
        if self._six_dof:
            # MapTracker::switchToNewSubmap; the odometry edge T_S1_S2 = T_S1_B * T_S2_B^-1
            T_S1_B = self._T_S_B
            self._initial_T_S_O = tf.inverse(tf.gravity_align(self._T_O_B))
            self._T_S_B = tf.compose(self._initial_T_S_O, self._T_O_B)
            T_S1_S2 = tf.to_pose4(tf.compose(T_S1_B, tf.inverse(self._T_S_B)))
        if self.cfg.odometry_constraints_enabled and prev is not None:
            self.pose_graph.addRelativePoseConstraint(api.RelativePoseConstraintConfig(
                prev, sid, T_S1_S2, self.cfg.odometry_information))                                   # addOdometryMeasurement
        if self.cfg.height_constraints_enabled and len(self.submap_ids) > 1:
            self.addHeightMeasurement(sid, height)
        if not self._six_dof:
            self._odom_submap_pose = T_mission_sensor.copy()
        self.timings.append(rec)

    def _finish_active(self, rec):
        """finishSubmap() of the active submap, timed into the switch record rec."""
        ctx = self.ctx
        t0 = time.time()
        ctx.submap_finish(self.active_id)                          # finishSubmap(): registration view + grid
        ctx.synchronize()
        t1 = time.time()
        ctx.submap_extract_points(self.active_id, self.filter)    # ... registration points, OBB, isosurface blocks
        ctx.synchronize()
        rec["finish_ms"] = (time.time() - t0) * 1e3
        rec["view_ms"] = (t1 - t0) * 1e3
        rec["finished_blocks"] = ctx.submap_block_count(self.active_id)
        rec["isosurface_points"] = ctx.submap_num_points(self.active_id, api.K_ISOSURFACE_POINTS)

    # ---- PoseGraphInterface::addHeightMeasurement (pose_graph_interface.cpp:94-107)
    def addHeightMeasurement(self, submap_id, height):
        """An absolute constraint from the constant mission-frame node (added when missing) on the submap's
        height alone: information diag(0, 0, height_information_zz, 0)."""
        pg = self.pose_graph
        if not pg.hasReferenceFrameNode(MISSION_FRAME_ID):
            pg.addReferenceFrameNode(api.ReferenceFrameNodeConfig(MISSION_FRAME_ID, np.zeros(4), set_constant=True))
        pg.addAbsolutePoseConstraint(api.AbsolutePoseConstraintConfig(
            MISSION_FRAME_ID, submap_id, np.array([0.0, 0.0, float(height), 0.0]),
            np.diag([0.0, 0.0, float(self.cfg.height_information_zz), 0.0]),
            allow_semi_definite_information_matrix=True))

    # ---- VoxgraphMapper::loopClosureCallback
    def loopClosureCallback(self, from_timestamp, to_timestamp, T_t1_t2):
        """A loop closure from an external source: the robot at to_timestamp seen from the robot at
        from_timestamp.  T_t1_t2 = [qw qx qy qz tx ty tz]; a geometry_msgs/Transform (translation x y z,
        rotation x y z w) is [rotation.w, rotation.x, rotation.y, rotation.z, translation.x, translation.y,
        translation.z].  The message's own information matrix is not used (neither does the reference):
        MapperConfig.loop_closure_information is.  Returns (submap A, submap B) of the new A -> B constraint, or
        None when the loop closure is refused; the reason is appended to loop_closure_warnings."""
        info = self.cfg.loop_closure_information
        if info is None:
            raise ValueError("loopClosureCallback: MapperConfig.loop_closure_information "
                             "(measurements/loop_closure/information_matrix) is not set")
        prefix = "Could not add loop closure from timestamp %r to %r" % (from_timestamp, to_timestamp)

        def refuse(why):
            self.loop_closure_warnings.append(prefix + ": " + why)
            return None

        a = self.lookupActiveSubmapByTime(from_timestamp)
        b = self.lookupActiveSubmapByTime(to_timestamp)
        if a is None or b is None:
            return refuse("timestamp A or B has no corresponding submap")
        if a == b:
            return refuse("timestamp A and B fall within the same submap")
        T_A_t1 = self.lookupPoseByTime(a, from_timestamp)
        T_B_t2 = self.lookupPoseByTime(b, to_timestamp)
        if T_A_t1 is None or T_B_t2 is None:
            return refuse("timestamp A or B has no corresponding robot pose")
        T = np.asarray(T_t1_t2, np.float64).reshape(7)
        q = T[:4]
        if abs(q @ q - 1.0) > 1e-3:
            return refuse("supplied transform quaternion is invalid")
        T_t1_t2 = np.concatenate([q / np.linalg.norm(q), T[4:]]).astype(np.float32)
        T_AB = tf.compose(tf.compose(T_A_t1, T_t1_t2), tf.inverse(T_B_t2))
        self.pose_graph.addRelativePoseConstraint(api.RelativePoseConstraintConfig(
            a, b, tf.to_pose4(T_AB), info))                                      # addLoopClosureMeasurement
        self._new_loop_closures = True
        return a, b

    # ---- VoxgraphMapper::finishMapCallback
    def finishMap(self):
        """Finish the last submap, bring the registration constraints up to date with it and optimise.  The
        map is then complete: a later scan raises, as there is no active submap left to integrate into."""
        if self._map_finished:
            raise RuntimeError("finishMap() was already called")
        rec = {"finish_ms": 0.0, "overlap_ms": 0.0, "pairs": 0, "finish_map": True}
        if not self.empty():
            self._finish_active(rec)
        if self.cfg.registration_constraints_enabled and len(self.submap_ids) >= 2:
            t0 = time.time()
            rec["pairs"] = self.updateRegistrationConstraints()
            rec["overlap_ms"] = (time.time() - t0) * 1e3
        self.timings.append(rec)
        self._map_finished = True
        return self.optimizePoseGraph()

    # ---- PoseGraphInterface::updateRegistrationConstraints
    def updateRegistrationConstraints(self):
        pg = self.pose_graph
        pg.resetRegistrationConstraints()
        finished = self.submap_ids        # all of them are finished at this point (the new one does not exist yet)
        T = np.array([_pose4_to_T(self.submap_pose[i]) for i in finished], np.float32)
        pairs = self.ctx.find_overlapping_pairs(finished, T)             # updateOverlappingSubmapList
        for (a, b) in pairs:
            pg.addRegistrationConstraint(api.RegistrationConstraintConfig(a, b, **self.cfg.registration))
        self.overlapping_submap_list = pairs
        return len(pairs)

    # ---- VoxgraphMapper::optimizePoseGraph -> PoseGraphInterface::optimize (pose_graph_interface.cpp:177-198)
    def optimizePoseGraph(self):
        """After new loop closures, a solve without the registration constraints comes first (its time and
        iterations go to the switch record as preoptimize_ms / pre_lm_iterations), then the full solve."""
        if len(self.submap_ids) < 2:
            return None
        if self._new_loop_closures:
            t0 = time.time()
            pre = self.pose_graph.optimize(exclude_registration_constraints=True)
            self.timings[-1]["preoptimize_ms"] = (time.time() - t0) * 1e3
            self.timings[-1]["pre_lm_iterations"] = pre.iterations
            self._new_loop_closures = False
        t0 = time.time()
        summ = self.pose_graph.optimize()
        ms = (time.time() - t0) * 1e3
        for i, p in self.pose_graph.getSubmapPoses().items():            # updateSubmapCollectionPoses
            self.submap_pose[i] = p
        self.timings[-1]["optimize_ms"] = ms
        self.timings[-1]["lm_iterations"] = summ.iterations
        self.timings[-1]["registration_blocks"] = len(self.pose_graph.registration_blocks)
        return summ

    # ---- LoopClosureEdgeServer::publishLoopClosureEdges
    def loopClosureEdges(self):
        """One edge per overlapping submap pair: (start time of A, start time of B, T_A_B [qw qx qy qz tx ty tz],
        6x6 covariance over [x y z roll pitch yaw]).  T_A_B joins the robot poses at the two submaps' first scans
        (kFake6dofTransforms).  The covariance holds PoseGraph.getEdgeCovarianceMap's 4x4 block, its yaw row and
        column at index 5, and 1e4 in the entries it does not know; when the covariance cannot be computed (a
        rank-deficient problem) every edge gets the 6x6 identity, as in the reference."""
        pairs = list(self.overlapping_submap_list)
        cov = None
        if pairs:
            try:
                cov = self.pose_graph.getEdgeCovarianceMap(pairs)
            except api.VgxError as e:
                if e.code != _lib.VGX_ERR_INVALID:
                    raise
        idx = [0, 1, 2, 5]
        edges = []
        for (a, b) in pairs:
            T_M_A = tf.compose(self._T_M_S(a), self._history[a][1][0])
            T_M_B = tf.compose(self._T_M_S(b), self._history[b][1][0])
            if cov is None:
                c6 = np.eye(6)
            else:
                c6 = np.full((6, 6), 1e4)
                c6[np.ix_(idx, idx)] = cov[(a, b)]
            edges.append((self.submap_start[a], self.submap_start[b], tf.compose(tf.inverse(T_M_A), T_M_B), c6))
        return edges

    # ---- VoxgraphMapper::saveToFileCallback -> cblox::SubmapCollection::saveToFile
    def saveToFile(self, path):
        """Write every submap (the active one included) with its current optimised pose; the 4-DoF
        pose is stored as a yaw-only quaternion.  Returns the file size in bytes."""
        ids = list(self.submap_ids)
        T = np.array([_pose4_to_T(self.submap_pose[i]) for i in ids], np.float32).reshape(-1, 7)
        return api.save_submap_collection(self.ctx, path, ids, T)

    # ---- VoxgraphMapper::saveSeparatedMeshCallback -> SubmapVisuals::saveSeparatedMesh
    def saveSeparatedMesh(self, path):
        """Mesh every submap (the active one included) at its current optimised pose and write the
        separated mesh as a binary PLY, each submap in its default colour.  Returns the file size."""
        ids = list(self.submap_ids)
        T = np.array([_pose4_to_T(self.submap_pose[i]) for i in ids], np.float32).reshape(-1, 7)
        return api.save_separated_mesh(self.ctx, path, ids, T, min_weight=self.cfg.mesh_min_weight)

    # ---- VoxgraphMapper::saveCombinedMeshCallback -> SubmapVisuals::saveCombinedMesh
    def saveCombinedMesh(self, path):
        """Project every submap (the active one included) at its current optimised pose into one global
        TSDF and write its mesh as a binary PLY (opaque white).  Returns the file size in bytes."""
        ids = list(self.submap_ids)
        T = np.array([_pose4_to_T(self.submap_pose[i]) for i in ids], np.float32).reshape(-1, 7)
        return api.save_combined_mesh(self.ctx, path, ids, T, min_weight=self.cfg.mesh_min_weight)

    # ---- VoxgraphMapper::publishCombinedMeshCallback
    def combinedMesh(self):
        """-> (xyz (V, 3) float32 in the mission frame, triangles (T, 3) uint32) of the projected map."""
        ids = list(self.submap_ids)
        T = np.array([_pose4_to_T(self.submap_pose[i]) for i in ids], np.float32).reshape(-1, 7)
        return api.combined_mesh(self.ctx, ids, T, self.cfg.mesh_min_weight)

    # ---- VoxgraphMapper::evaluateMapCallback -> MapEvaluation::evaluate
    def evaluateMap(self, map_evaluation):
        """Evaluate every submap (the active one included) at its current optimised pose against the
        ground truth of map_evaluation (an api.MapEvaluation on this mapper's context) -> EvaluationDetails."""
        ids = list(self.submap_ids)
        T = np.array([_pose4_to_T(self.submap_pose[i]) for i in ids], np.float32).reshape(-1, 7)
        return map_evaluation.evaluate(ids, T)

    # ---- VoxgraphMapper::publishActiveSubmapMeshCallback (the active submap in its own frame)
    def activeSubmapMesh(self):
        """-> (xyz (V, 3) float32 in the active submap's frame, triangles (T, 3) uint32)."""
        xyz, tri, _, _ = api.separated_mesh(self.ctx, [self.active_id], None, self.cfg.mesh_min_weight)
        return xyz, tri
