"""Seeded synthetic inputs for the voxgraph hot paths (SURVEY.md §8d).

A "world" is a set of axis-aligned boxes (floor slab, outer walls, interior walls,
crates/pillars).  A submap is the truncated signed distance to that world sampled
at voxel centres of a gravity-aligned, yawed submap frame, cut into voxblox-style
16^3 blocks; its registration points are the marching-cubes edge vertices of the
zero level set (what VoxgraphSubmap::findIsosurfaceVertices yields,
voxgraph/src/frontend/submap_collection/voxgraph_submap.cpp:203-243), kept in
block-coherent order like a voxblox mesh.  Nothing here is on the product's hot
path: it only produces host arrays that are fed through the C-ABI.
"""
from dataclasses import dataclass, field

import numpy as np


# --------------------------------------------------------------------------- world
@dataclass
class World:
    boxes: np.ndarray  # (M, 6) cx, cy, cz, hx, hy, hz   (float64)
    size_xy: tuple
    height: float


def make_world(seed=0, size_xy=(120.0, 80.0), height=5.0, n_clutter=400, n_walls=24):
    rng = np.random.default_rng(seed)
    sx, sy = size_xy
    boxes = []
    # floor slab (top face at z = 0) and ceiling-less outer walls
    boxes.append([sx / 2, sy / 2, -1.0, sx / 2 + 2, sy / 2 + 2, 1.0])
    t = 0.4
    boxes.append([sx / 2, -t, height / 2, sx / 2 + 2, t, height / 2 + 1])
    boxes.append([sx / 2, sy + t, height / 2, sx / 2 + 2, t, height / 2 + 1])
    boxes.append([-t, sy / 2, height / 2, t, sy / 2 + 2, height / 2 + 1])
    boxes.append([sx + t, sy / 2, height / 2, t, sy / 2 + 2, height / 2 + 1])
    # interior wall segments
    for _ in range(n_walls):
        cx, cy = rng.uniform(5, sx - 5), rng.uniform(5, sy - 5)
        length = rng.uniform(4, 14)
        if rng.random() < 0.5:
            boxes.append([cx, cy, height / 2, length / 2, 0.2, height / 2])
        else:
            boxes.append([cx, cy, height / 2, 0.2, length / 2, height / 2])
    # clutter: crates, pillars, shelves
    for _ in range(n_clutter):
        cx, cy = rng.uniform(1, sx - 1), rng.uniform(1, sy - 1)
        hx, hy = rng.uniform(0.3, 1.8), rng.uniform(0.3, 1.8)
        hz = rng.uniform(0.3, 1.6)
        boxes.append([cx, cy, hz, hx, hy, hz])
    return World(np.asarray(boxes, np.float64), (sx, sy), height)


def box_sdf(p, c, h):
    """Exact signed distance from points p (...,3) to the box centre c half-size h."""
    q = np.abs(p - c) - h
    outside = np.linalg.norm(np.maximum(q, 0.0), axis=-1)
    inside = np.minimum(np.max(q, axis=-1), 0.0)
    return outside + inside


def world_sdf(world, p):
    d = np.full(p.shape[:-1], np.inf)
    for b in world.boxes:
        d = np.minimum(d, box_sdf(p, b[:3], b[3:]))
    return d


# --------------------------------------------------------------------------- poses
def rot_z(yaw):
    c, s = np.cos(yaw), np.sin(yaw)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def pose_to_T(xyzyaw):
    """[x,y,z,yaw] -> [qw,qx,qy,qz,tx,ty,tz] (float32)."""
    x, y, z, yaw = [float(v) for v in xyzyaw]
    return np.array([np.cos(yaw / 2), 0, 0, np.sin(yaw / 2), x, y, z], np.float32)


def relative_pose(pa, pb):
    """T_a_b for 4-DoF poses: (t_obs[3], yaw_obs)."""
    pa = np.asarray(pa, np.float64); pb = np.asarray(pb, np.float64)
    t = rot_z(pa[3]).T @ (pb[:3] - pa[:3])
    yaw = pb[3] - pa[3]
    yaw = yaw - 2 * np.pi * np.floor((yaw + np.pi) / (2 * np.pi))
    return t, yaw


# --------------------------------------------------------------------------- submaps
@dataclass
class Submap:
    submap_id: int
    pose_gt: np.ndarray            # (4,) x y z yaw of the submap frame in the mission frame
    voxel_size: float
    vps: int
    block_idx: np.ndarray          # (B,3) int32
    distance: np.ndarray           # (B, vps^3) float32
    weight: np.ndarray             # (B, vps^3) float32
    points_xyz: np.ndarray = None  # (K,3) float32 submap frame
    points_distance: np.ndarray = None
    points_weight: np.ndarray = None
    surface_blocks: np.ndarray = None  # (S,3) int32 blocks containing isosurface vertices
    meta: dict = field(default_factory=dict)

    @property
    def num_blocks(self):
        return self.block_idx.shape[0]


def make_submap(world, submap_id, pose_gt, voxel_size=0.2, vps=16, radius=12.0,
                z_world=(-0.8, 4.0), trunc=None, n_points=None):
    """Sample the world TSDF in the frame `pose_gt` and extract isosurface points."""
    pose_gt = np.asarray(pose_gt, np.float64)
    vs = float(voxel_size)
    trunc = 3 * vs if trunc is None else float(trunc)
    bs = vs * vps
    R = rot_z(pose_gt[3])
    t = pose_gt[:3]
    # block range in the submap frame
    zlo, zhi = z_world[0] - t[2], z_world[1] - t[2]
    bmin = np.floor(np.array([-radius, -radius, zlo]) / bs).astype(int)
    bmax = np.floor(np.array([radius, radius, zhi]) / bs).astype(int)
    nb = bmax - bmin + 1
    dims = nb * vps
    ax = [((np.arange(dims[a]) + 0.5) * vs + bmin[a] * bs) for a in range(3)]
    dist = np.full(dims, np.inf, np.float64)
    # stamp each nearby box into the grid slice it can influence
    margin = trunc + 2 * vs
    for b in world.boxes:
        c, h = b[:3], b[3:]
        corners = np.array([[sx, sy, sz] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)],
                           np.float64) * (h + margin) + c
        cs = (corners - t) @ R  # world -> submap frame: R^T (p - t)
        lo = cs.min(0); hi = cs.max(0)
        i0 = np.maximum(np.floor((lo - bmin * bs) / vs).astype(int), 0)
        i1 = np.minimum(np.ceil((hi - bmin * bs) / vs).astype(int) + 1, dims)
        if np.any(i1 <= i0):
            continue
        gx, gy, gz = np.meshgrid(ax[0][i0[0]:i1[0]], ax[1][i0[1]:i1[1]], ax[2][i0[2]:i1[2]],
                                 indexing="ij")
        pw = np.stack([gx, gy, gz], -1) @ R.T + t
        sl = (slice(i0[0], i1[0]), slice(i0[1], i1[1]), slice(i0[2], i1[2]))
        dist[sl] = np.minimum(dist[sl], box_sdf(pw, c, h))
    gx, gy = np.meshgrid(ax[0], ax[1], indexing="ij")
    r_xy = np.sqrt(gx ** 2 + gy ** 2)[:, :, None]
    observed = (r_xy <= radius) & (dist > -trunc)
    wz = (ax[2] + t[2] >= z_world[0]) & (ax[2] + t[2] <= z_world[1])
    observed &= wz[None, None, :]
    weight = np.where(observed, 1.0 + 9.0 / (1.0 + (r_xy / 6.0) ** 2), 0.0).astype(np.float32)
    tsdf = np.clip(dist, -trunc, trunc).astype(np.float32)
    tsdf = np.where(observed, tsdf, np.float32(0)).astype(np.float32)

    # ---- isosurface vertices: sign-change edges between observed neighbours
    verts = []
    for a in range(3):
        s0 = [slice(None)] * 3; s1 = [slice(None)] * 3
        s0[a] = slice(0, dims[a] - 1); s1[a] = slice(1, dims[a])
        s0 = tuple(s0); s1 = tuple(s1)
        d0, d1 = tsdf[s0], tsdf[s1]
        m = observed[s0] & observed[s1] & ((d0 < 0) != (d1 < 0))
        ii = np.argwhere(m)
        if ii.shape[0] == 0:
            continue
        e0 = d0[m].astype(np.float32); e1 = d1[m].astype(np.float32)
        tt = e0 / (e0 - e1)
        pos = np.stack([ax[k][ii[:, k]] for k in range(3)], -1).astype(np.float32)
        pos[:, a] += tt * np.float32(vs)
        w0, w1 = weight[s0][m], weight[s1][m]
        vd = (e0 + tt * (e1 - e0)).astype(np.float32)
        vw = (w0 + tt * (w1 - w0)).astype(np.float32)
        blk = ii // vps
        loc = ii % vps
        key = (((blk[:, 2] * nb[1] + blk[:, 1]) * nb[0] + blk[:, 0]) * (vps ** 3)
               + (loc[:, 2] * vps + loc[:, 1]) * vps + loc[:, 0]) * 3 + a
        verts.append((key, pos, vd, vw, blk + bmin))
    if verts:
        key = np.concatenate([v[0] for v in verts])
        order = np.argsort(key, kind="stable")
        pos = np.concatenate([v[1] for v in verts])[order]
        vd = np.concatenate([v[2] for v in verts])[order]
        vw = np.concatenate([v[3] for v in verts])[order]
        vb = np.concatenate([v[4] for v in verts])[order]
    else:
        pos = np.zeros((0, 3), np.float32); vd = np.zeros(0, np.float32)
        vw = np.zeros(0, np.float32); vb = np.zeros((0, 3), int)
    n_all = pos.shape[0]
    if n_points is not None and n_all > 0:
        if n_all >= n_points:
            sel = np.floor(np.arange(n_points) * (n_all / n_points)).astype(int)
        else:
            sel = np.arange(n_points) % n_all
        pos, vd, vw = pos[sel], vd[sel], vw[sel]
    surface_blocks = np.unique(vb, axis=0).astype(np.int32) if n_all else np.zeros((0, 3), np.int32)

    # ---- cut into blocks (linear index x + vps*(y + vps*z))
    def to_blocks(arr):
        a6 = arr.reshape(nb[0], vps, nb[1], vps, nb[2], vps)
        return a6.transpose(4, 2, 0, 5, 3, 1).reshape(nb[2] * nb[1] * nb[0], vps ** 3)

    bd = to_blocks(tsdf); bw = to_blocks(weight)
    bz, by, bx = np.meshgrid(np.arange(nb[2]), np.arange(nb[1]), np.arange(nb[0]), indexing="ij")
    bidx = (np.stack([bx, by, bz], -1).reshape(-1, 3) + bmin).astype(np.int32)
    keep = (bw > 1e-6).any(axis=1)
    return Submap(submap_id=int(submap_id), pose_gt=pose_gt.copy(), voxel_size=vs, vps=vps,
                  block_idx=np.ascontiguousarray(bidx[keep]),
                  distance=np.ascontiguousarray(bd[keep]),
                  weight=np.ascontiguousarray(bw[keep]),
                  points_xyz=np.ascontiguousarray(pos), points_distance=vd, points_weight=vw,
                  surface_blocks=surface_blocks,
                  meta=dict(trunc=trunc, radius=radius, n_vertices_all=int(n_all)))


# --------------------------------------------------------------------------- overlap (a20)
def submaps_overlap(a, b, pose_a, pose_b):
    """VoxgraphSubmap::overlapsWith restated on the host (voxgraph_submap.cpp:245-278):
    mission-frame AABB rejection, then 'any isosurface block centre of A lands in an
    allocated block of B'."""
    def aabb(s, pose):
        bs = s.voxel_size * s.vps
        if s.surface_blocks.shape[0] == 0:
            return None
        lo = s.surface_blocks.min(0) * bs; hi = (s.surface_blocks.max(0) + 1) * bs
        cs = np.array([[x, y, z] for x in (lo[0], hi[0]) for y in (lo[1], hi[1])
                       for z in (lo[2], hi[2])])
        cw = cs @ rot_z(pose[3]).T + pose[:3]
        return cw.min(0), cw.max(0)
    A = aabb(a, pose_a); B = aabb(b, pose_b)
    if A is None or B is None:
        return False
    if np.any(A[1] < B[0]) or np.any(A[0] > B[1]):
        return False
    bs_a = a.voxel_size * a.vps
    centres = (a.surface_blocks.astype(np.float64) + 0.5) * bs_a
    cw = centres @ rot_z(pose_a[3]).T + pose_a[:3]
    cb = (cw - pose_b[:3]) @ rot_z(pose_b[3])
    bs_b = np.float32(b.voxel_size * b.vps)
    inv = np.float32(1.0 / float(bs_b))
    other = np.floor(cb.astype(np.float32) * inv + np.float32(1e-6)).astype(np.int64)
    have = set(map(tuple, b.block_idx.astype(np.int64)))
    return any(tuple(o) in have for o in other)


# --------------------------------------------------------------------------- scenes
@dataclass
class Scene:
    world: World
    submaps: list
    poses_gt: np.ndarray       # (N,4)
    poses_init: np.ndarray     # (N,4) noisy initial estimates (node 0 = ground truth)
    pairs: list                # overlapping (i, j), i < j  (submap indices)
    odometry: list             # (i, j, t_obs[3], yaw_obs)
    odom_information: np.ndarray  # (4,4)
    meta: dict = field(default_factory=dict)


def figure8(n, size_xy, margin=16.0):
    sx, sy = size_xy
    s = np.linspace(0.0, 2 * np.pi, n, endpoint=False)
    x = sx / 2 + (sx / 2 - margin) * np.sin(s)
    y = sy / 2 + (sy / 2 - margin) * np.sin(2 * s) * 0.9
    dx = (sx / 2 - margin) * np.cos(s)
    dy = (sy / 2 - margin) * 2 * np.cos(2 * s) * 0.9
    yaw = np.arctan2(dy, dx)
    return x, y, yaw


def compose_pose(p, t_rel, yaw_rel):
    """4-DoF pose p composed with a relative transform expressed in p's frame."""
    p = np.asarray(p, np.float64)
    out = np.empty(4)
    out[:3] = p[:3] + rot_z(p[3]) @ np.asarray(t_rel, np.float64)
    y = p[3] + yaw_rel
    out[3] = y - 2 * np.pi * np.floor((y + np.pi) / (2 * np.pi))
    return out


def _make_submap_job(job):
    world, i, pose, voxel_size, vps, radius, n_points, trunc = job
    return make_submap(world, i, pose, voxel_size, vps, radius, n_points=n_points, trunc=trunc)


def make_scene(seed=2, n_submaps=50, n_points=10000, voxel_size=0.2, vps=16, radius=12.0,
               size_xy=(120.0, 80.0), max_pairs=None, pose_noise=(0.2, 0.05, 0.02),
               n_clutter=400, n_walls=24, trunc=None, trajectory=None, drift=None, workers=1):
    """Config-2 style scene: N submaps along a figure-8 through a cluttered hall.

    drift=(sigma_xy, sigma_z, sigma_yaw) per odometry step: the initial poses are the integrated
    noisy odometry (what voxgraph starts from) and the odometry edges are those noisy relative
    transforms; otherwise independent pose noise with near-exact odometry."""
    rng = np.random.default_rng(seed)
    world = make_world(seed, size_xy=size_xy, n_clutter=n_clutter, n_walls=n_walls)
    if trajectory is None:
        x, y, yaw = figure8(n_submaps, size_xy)
    else:
        x, y, yaw = trajectory
    poses_gt = np.stack([x, y, np.full(n_submaps, 1.0), yaw], -1)
    yaw_w = poses_gt[:, 3]
    poses_gt[:, 3] = yaw_w - 2 * np.pi * np.floor((yaw_w + np.pi) / (2 * np.pi))
    jobs = [(world, i, poses_gt[i], voxel_size, vps, radius, n_points, trunc) for i in range(n_submaps)]
    if workers > 1 and n_submaps > 1:
        # host-side numpy sampling of the analytic world; one process per submap (fork: call this
        # before the process initialises CUDA)
        import multiprocessing as mp
        with mp.get_context("fork").Pool(min(workers, n_submaps)) as pool:
            submaps = pool.map(_make_submap_job, jobs, chunksize=1)
    else:
        submaps = [_make_submap_job(j) for j in jobs]
    odometry = []
    if drift is None:
        noise = np.concatenate([rng.normal(0, pose_noise[0], (n_submaps, 2)),
                                rng.normal(0, pose_noise[1], (n_submaps, 1)),
                                rng.normal(0, pose_noise[2], (n_submaps, 1))], -1)
        noise[0] = 0
        poses_init = poses_gt + noise
        for i in range(n_submaps - 1):
            t_obs, yaw_obs = relative_pose(poses_gt[i], poses_gt[i + 1])
            t_obs = t_obs + rng.normal(0, 0.05, 3) * np.array([1, 1, 0.1])
            yaw_obs = yaw_obs + rng.normal(0, 0.005)
            odometry.append((i, i + 1, t_obs, float(yaw_obs)))
    else:
        poses_init = poses_gt.copy()
        for i in range(n_submaps - 1):
            t_obs, yaw_obs = relative_pose(poses_gt[i], poses_gt[i + 1])
            t_obs = t_obs + rng.normal(0, 1.0, 3) * np.array([drift[0], drift[0], drift[1]])
            yaw_obs = float(yaw_obs + rng.normal(0, drift[2]))
            odometry.append((i, i + 1, t_obs, yaw_obs))
            poses_init[i + 1] = compose_pose(poses_init[i], t_obs, yaw_obs)
    pairs = []
    for i in range(n_submaps):
        for j in range(i + 1, n_submaps):
            if np.hypot(*(poses_gt[i, :2] - poses_gt[j, :2])) > 2 * radius + 4:
                continue
            if submaps_overlap(submaps[i], submaps[j], poses_init[i], poses_init[j]):
                pairs.append((i, j))
    if max_pairs is not None and len(pairs) > max_pairs:
        sel = np.sort(rng.choice(len(pairs), max_pairs, replace=False))
        pairs = [pairs[k] for k in sel]
    info = np.diag([1.0, 1.0, 2500.0, 2500.0])  # voxgraph_mapper.yaml:41-47
    return Scene(world, submaps, poses_gt, poses_init, pairs, odometry, info,
                 meta=dict(seed=seed, n_points=n_points, voxel_size=voxel_size, radius=radius))


def make_pair_scene(seed=1, n_points=1000, voxel_size=0.2, vps=16, radius=6.0,
                    perturbation=(0.3, -0.3, 0.15, 0.1)):
    """Config-1: two box-room submaps of the same place, reading perturbed."""
    world = make_world(seed, size_xy=(24.0, 20.0), n_clutter=30, n_walls=3)
    p0 = np.array([12.0, 10.0, 1.0, 0.0])
    p1 = np.array([13.5, 10.5, 1.0, 0.3])
    s0 = make_submap(world, 0, p0, voxel_size, vps, radius, n_points=n_points)
    s1 = make_submap(world, 1, p1, voxel_size, vps, radius, n_points=n_points)
    poses_gt = np.stack([p0, p1])
    poses_init = poses_gt.copy()
    poses_init[1] += np.asarray(perturbation)
    t_obs, yaw_obs = relative_pose(p0, p1)
    return Scene(world, [s0, s1], poses_gt, poses_init, [(0, 1)],
                 [(0, 1, t_obs, float(yaw_obs))], np.diag([1.0, 1.0, 2500.0, 2500.0]),
                 meta=dict(seed=seed, n_points=n_points, voxel_size=voxel_size, radius=radius))


# --------------------------------------------------------------------------- sensors
def ray_world_range(world, origin, dirs, max_range):
    """Nearest hit distance of rays (origin, unit dirs (n,3)) with the world boxes."""
    best = np.full(dirs.shape[0], np.inf)
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / dirs
    for b in world.boxes:
        c, h = b[:3], b[3:]
        if np.linalg.norm(np.maximum(np.abs(origin - c) - h, 0)) > max_range:
            continue
        t1 = (c - h - origin) * inv
        t2 = (c + h - origin) * inv
        tmin = np.nanmax(np.minimum(t1, t2), axis=1)
        tmax = np.nanmin(np.maximum(t1, t2), axis=1)
        hit = (tmax >= np.maximum(tmin, 0.0))
        tt = np.where(tmin > 0, tmin, tmax)  # origin inside the box -> exit distance
        best = np.where(hit & (tt < best), tt, best)
    return best


def quat_to_matrix(q):
    """Unit quaternion [qw qx qy qz] -> 3x3 rotation matrix (float64)."""
    w, x, y, z = [float(v) for v in q]
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def lidar_scan(world, sensor_pose, n_beams=64, n_azimuth=1024, vfov_deg=16.6, max_range=16.0,
               range_noise=0.02, seed=0, miss_range=None, R_world_sensor=None):
    """64x1024 spinning LiDAR (config 3). Returns points in the sensor frame (n,3) f32.
    Rays that hit nothing within max_range are dropped unless miss_range is given
    (then they are reported at miss_range, producing voxblox clearing rays).
    R_world_sensor: the sensor's full 3x3 orientation (a tilted sensor); sensor_pose[3] (yaw) is then
    not used, and only sensor_pose[:3] places the sensor."""
    rng = np.random.default_rng(seed)
    el = np.deg2rad(np.linspace(-vfov_deg, vfov_deg, n_beams))
    az = np.linspace(-np.pi, np.pi, n_azimuth, endpoint=False)
    E, A = np.meshgrid(el, az, indexing="ij")
    dirs_c = np.stack([np.cos(E) * np.cos(A), np.cos(E) * np.sin(A), np.sin(E)], -1).reshape(-1, 3)
    Rw = rot_z(sensor_pose[3]) if R_world_sensor is None else np.asarray(R_world_sensor, np.float64)
    dirs_w = dirs_c @ Rw.T
    rng_m = ray_world_range(world, np.asarray(sensor_pose[:3], np.float64), dirs_w, max_range * 2)
    rng_m = rng_m + rng.normal(0, range_noise, rng_m.shape)
    if miss_range is None:
        keep = np.isfinite(rng_m) & (rng_m <= max_range)
        return (dirs_c[keep] * rng_m[keep, None]).astype(np.float32)
    rng_m = np.where(np.isfinite(rng_m) & (rng_m <= max_range), rng_m, miss_range)
    return (dirs_c * rng_m[:, None]).astype(np.float32)


def depth_scan(world, sensor_pose, width=640, height=480, fx=525.0, fy=525.0, max_depth=5.0,
               noise=0.005, seed=0):
    """Pinhole depth camera looking along +x of the sensor frame (config 5)."""
    rng = np.random.default_rng(seed)
    u = (np.arange(width) - width / 2 + 0.5) / fx
    v = (np.arange(height) - height / 2 + 0.5) / fy
    V, U = np.meshgrid(v, u, indexing="ij")
    dirs_c = np.stack([np.ones_like(U), -U, -V], -1).reshape(-1, 3)
    norm = np.linalg.norm(dirs_c, axis=1, keepdims=True)
    dirs_c = dirs_c / norm
    dirs_w = dirs_c @ rot_z(sensor_pose[3]).T
    r = ray_world_range(world, np.asarray(sensor_pose[:3], np.float64), dirs_w, max_depth * 3)
    depth = r * dirs_c[:, 0]
    keep = np.isfinite(r) & (depth <= max_depth)
    r = r + rng.normal(0, noise, r.shape)
    return (dirs_c[keep] * r[keep, None]).astype(np.float32)


def surface_colours(points_C, sensor_pose, cell=0.5):
    """A deterministic colour for every point of a scan (lidar_scan / depth_scan output, sensor frame): the
    world is painted in `cell`-sized cubes, each with a colour of its own whose four channels differ, so a
    coloured stream sees the same colour on a surface from every pose -> (n, 4) uint8 [r g b a]."""
    p = np.asarray(points_C, np.float64).reshape(-1, 3) @ rot_z(sensor_pose[3]).T + np.asarray(sensor_pose[:3])
    i = np.floor(p / cell).astype(np.int64)
    h = (i[:, 0] * 73856093) ^ (i[:, 1] * 19349663) ^ (i[:, 2] * 83492791)
    return np.stack([40 + h % 200, 30 + (h >> 8) % 220, 20 + (h >> 16) % 230, 128 + (h >> 24) % 128], -1).astype(np.uint8)


def pack_pointcloud2(points, rgba=None, intensity=None, point_step=None, pad_rows=0, organised=None):
    """A scan (lidar_scan / depth_scan output, (n, 3) float32) as the sensor message a driver would publish ->
    api.PointCloud2, in PCL's layouts: XYZ (point_step 16), XYZI with intensity (n,) float32 at byte 16 (32) or
    XYZRGB with rgba (n, 4) uint8 [r g b a] packed b, g, r, a at byte 16 (32).  point_step: a longer (or, down to
    the fields' 16 / 20 bytes, shorter) record, the extra bytes filled with 0xA5.  organised = (height, width)
    with height * width == n, else one row; pad_rows: 0xA5 bytes appended to every row."""
    from .api import POINTFIELD_FLOAT32, PointCloud2
    pts = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
    n = len(pts)
    fields = [("x", 0, POINTFIELD_FLOAT32, 1), ("y", 4, POINTFIELD_FLOAT32, 1), ("z", 8, POINTFIELD_FLOAT32, 1)]
    used, step = 12, 16
    if rgba is not None:
        fields.append(("rgb", 16, POINTFIELD_FLOAT32, 1)); used, step = 20, 32
    elif intensity is not None:
        fields.append(("intensity", 16, POINTFIELD_FLOAT32, 1)); used, step = 20, 32
    step = step if point_step is None else int(point_step)
    if step < used:
        raise ValueError("pack_pointcloud2: point_step %d is shorter than the fields (%d bytes)" % (step, used))
    rec = np.full((n, step), 0xA5, np.uint8)
    rec[:, :12] = pts.view(np.uint8).reshape(n, 12)
    if rgba is not None:
        rec[:, 16:20] = np.ascontiguousarray(rgba, np.uint8).reshape(n, 4)[:, [2, 1, 0, 3]]
    elif intensity is not None:
        rec[:, 16:20] = np.ascontiguousarray(intensity, np.float32).reshape(n).view(np.uint8).reshape(n, 4)
    height, width = (1, n) if organised is None else organised
    if height * width != n:
        raise ValueError("pack_pointcloud2: organised %s does not hold %d points" % (organised, n))
    rows = np.full((height, width * step + pad_rows), 0xA5, np.uint8)
    rows[:, :width * step] = rec.reshape(height, width * step)
    return PointCloud2(fields=fields, width=width, height=height, point_step=step, row_step=width * step + pad_rows,
                       data=rows.tobytes())


# --------------------------------------------------------------------------- analytic layers
def plane_layer_blocks(normal, offset, voxel_size, vps, block_range, trunc=None, weight=1.0):
    """Blocks sampling d(p) = n.p - c at voxel centres (KA1). block_range = ((x0,x1),(y0,y1),(z0,z1))
    inclusive block indices. Returns (block_idx, distance, weight)."""
    n = np.asarray(normal, np.float64)
    idx, dist, wts = [], [], []
    vs = np.float32(voxel_size)
    for bz in range(block_range[2][0], block_range[2][1] + 1):
        for by in range(block_range[1][0], block_range[1][1] + 1):
            for bx in range(block_range[0][0], block_range[0][1] + 1):
                o = np.array([bx, by, bz], np.float32) * (vs * np.float32(vps))
                lz, ly, lx = np.meshgrid(np.arange(vps), np.arange(vps), np.arange(vps),
                                         indexing="ij")
                c = np.stack([lx, ly, lz], -1).reshape(-1, 3).astype(np.float32)
                p = o + (c + np.float32(0.5)) * vs
                d = p.astype(np.float64) @ n - offset
                if trunc is not None:
                    d = np.clip(d, -trunc, trunc)
                idx.append([bx, by, bz]); dist.append(d.astype(np.float32))
                wts.append(np.full(vps ** 3, weight, np.float32))
    return (np.asarray(idx, np.int32), np.asarray(dist, np.float32), np.asarray(wts, np.float32))


def field_layer_blocks(fn, voxel_size, vps, block_range, weight=1.0):
    """Blocks sampling an arbitrary scalar field fn(p (n,3) float64) at voxel centres."""
    idx, dist, wts = [], [], []
    vs = np.float32(voxel_size)
    for bz in range(block_range[2][0], block_range[2][1] + 1):
        for by in range(block_range[1][0], block_range[1][1] + 1):
            for bx in range(block_range[0][0], block_range[0][1] + 1):
                o = np.array([bx, by, bz], np.float32) * (vs * np.float32(vps))
                lz, ly, lx = np.meshgrid(np.arange(vps), np.arange(vps), np.arange(vps),
                                         indexing="ij")
                c = np.stack([lx, ly, lz], -1).reshape(-1, 3).astype(np.float32)
                p = o + (c + np.float32(0.5)) * vs
                idx.append([bx, by, bz]); dist.append(fn(p.astype(np.float64)).astype(np.float32))
                wts.append(np.full(vps ** 3, weight, np.float32))
    return (np.asarray(idx, np.int32), np.asarray(dist, np.float32), np.asarray(wts, np.float32))
