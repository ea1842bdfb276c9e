"""Build separated submap meshes on the GPU (vgx_mesh_build) and report where the time goes.

    python scripts/mesh_extract.py [--workload config2|config4] [--submaps N] [--repeats 5]
                                   [--restate-submaps 3] [--min-weight 2.0] [--out FILE]

Two inputs: bench.py's synthetic scene (config2: 50 submaps at 0.2 m voxels; config4: 200 at 0.10 m),
meshed as one separated mesh at the scene's poses; and the active submap at the end of a short mapper
stream (lidar scans into a 0.2 m submap, Fast integration), meshed in its own frame as the active-mesh
callback does.  For each: the build time (CUDA events around the call, and a host clock that ends in a
synchronise), the per-kernel time of profiling slot 12 from a separate profiled build and its launch
count, vertices and triangles, voxels swept per second, the download and PLY times, and the time of the
numpy restatement (tests/mesh_exact.py, one process) on the first --restate-submaps submaps, labelled as
the restated reference.  min_weight defaults to voxgraph's mesh_min_weight 2.0 (synthetic weights are
1 to 10).  The card's name and power limit are read in the same run.  Needs a GPU.
"""
import argparse
import os
import sys
import time

import numpy as np

import _measure as M

sys.path.insert(0, os.path.join(M.ROOT, "tests"))


def measure(ctx, ids, T, min_weight, repeats, restate_layers):
    from voxgraph_b200 import _lib, api
    cfg = ctx.mesh_config(min_weight=min_weight)
    n_vox = 0
    for i in ids:
        _, vps, nb, _ = ctx.submap_info(i)
        n_vox += nb * vps ** 3
    ctx.mesh_build(ids, T, cfg)   # warm-up: table upload, scratch and output buffers
    host, dev = [], []
    for _ in range(repeats):
        h, d, _ = M.timed(ctx, lambda: ctx.mesh_build(ids, T, cfg))
        host.append(h)
        dev.append(d)
    kern_ms, launches, _ = M.profiled(ctx, _lib.VGX_SLOT_MESH, lambda: ctx.mesh_build(ids, T, cfg))
    t_dl, _, (xyz, tri) = M.timed(ctx, ctx.mesh_download)
    t_ply, _, ply = M.timed(ctx, ctx.mesh_ply)
    res = dict(submaps=len(ids), voxels=n_vox, min_weight=min_weight, vertices=len(xyz), triangles=len(tri),
               build_host_ms=[round(x, 3) for x in host], build_event_ms=[round(x, 3) for x in dev],
               build_best_ms=round(min(host), 3), voxels_per_s=float("%.4g" % (n_vox / (min(host) / 1e3))),
               profiled_kernels_ms=round(kern_ms, 3), kernel_launches=launches,
               download_ms=round(t_dl, 3), ply_ms=round(t_ply, 3), ply_bytes=len(ply))
    if restate_layers:
        import finish_exact as fx
        import mesh_exact as me
        k = len(restate_layers)
        t = time.perf_counter()
        ex, et, _, _ = me.separated([fx.Grid(*lay) for lay in restate_layers], None if T is None else T[:k],
                                    min_weight)
        dt = time.perf_counter() - t
        rv = sum(len(lay[2]) * lay[1] ** 3 for lay in restate_layers)
        gx, gt, _, _ = api.separated_mesh(ctx, ids[:k], None if T is None else T[:k], min_weight)
        res["restated_reference"] = dict(what="numpy restatement tests/mesh_exact.py, one process", submaps=k,
                                         voxels=rv, seconds=round(dt, 3), voxels_per_s=float("%.4g" % (rv / dt)),
                                         equal=bool(np.array_equal(et.astype(np.uint32), gt)
                                                    and ex.tobytes() == gx.tobytes()))
    return res


def stream_active(min_weight, repeats):
    from voxgraph_b200 import api, mapper as vm, synth
    ctx = api.Context(0)
    world = synth.make_world(7, size_xy=(60.0, 40.0), n_clutter=120, n_walls=8)
    n = 40
    s_arc = np.arange(n) * 0.5
    gt = np.stack([10.0 + s_arc, 15.0 + 2.0 * np.sin(s_arc / 5.0), np.full(n, 1.2), 0.05 * s_arc], -1)
    cfg = vm.MapperConfig(voxel_size=0.2, submap_creation_interval=15 / 10.0, capacity_blocks=16384,
                          mesh_min_weight=min_weight)
    m = vm.VoxgraphMapper(ctx, cfg)
    for k in range(n):
        m.pointcloudCallback(k / 10.0, gt[k], synth.lidar_scan(world, gt[k], n_beams=64, n_azimuth=1024, seed=k))
    sid = m.active_id
    idx, d, w = ctx.submap_download(sid)
    res = measure(ctx, [sid], None, min_weight, repeats, [(0.2, 16, idx, d, w)])
    res["stream_scans"] = n
    ctx.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="config2", choices=sorted(M.WORKLOADS))
    ap.add_argument("--submaps", type=int, default=None)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--restate-submaps", type=int, default=3)
    ap.add_argument("--min-weight", type=float, default=2.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    w = M.WORKLOADS[a.workload]
    ctx, sc, ids, T = M.upload_scene(w, a.submaps)
    layers = [(s.voxel_size, s.vps, s.block_idx, s.distance, s.weight) for s in sc.submaps[:a.restate_submaps]]
    scene = measure(ctx, ids, T, a.min_weight, a.repeats, layers)
    ctx.close()
    M.emit(dict(gpu=M.gpu_info(), workload=a.workload, voxel_size=w["voxel_size"], scene=scene,
                active_submap=stream_active(a.min_weight, a.repeats)), a.out)


if __name__ == "__main__":
    main()
