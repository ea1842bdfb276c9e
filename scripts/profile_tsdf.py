"""One 64 x 1024 LiDAR scan through both TSDF schedulers and one finishSubmap on the device - a
workload to profile the HP1 / extraction kernels on."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from voxgraph_b200 import api, synth  # noqa: E402

ctx = api.Context(0)
world = synth.make_world(3, size_xy=(40.0, 40.0), n_clutter=60, n_walls=6)
pts = synth.lidar_scan(world, np.array([20.0, 20.0, 1.2, 0.4]), n_beams=64, n_azimuth=1024, seed=1)
T = synth.pose_to_T([0.0, 0.0, 0.0, 0.0])
for sid, mode, vs in ((1, 1, 0.15), (2, 0, 0.15)):
    ctx.submap_create(sid, vs, 16, 16384)
    cfg = ctx.tsdf_config(mode=mode, default_truncation_distance=3 * vs, max_ray_length_m=16.0)
    for k in range(2):   # second pass: blocks exist, pure update
        st = ctx.tsdf_integrate(sid, T, pts, cfg)
    print("mode", mode, "voxel updates", st.voxel_updates, "blocks", ctx.submap_block_count(sid))
ctx.submap_finish_ex(1, ctx.registration_filter())
print("isosurface vertices", ctx.submap_num_points(1, api.K_ISOSURFACE_POINTS))
sweeps = ctx.submap_generate_esdf(1, None)
print("esdf sweeps", sweeps)
ctx.close()
